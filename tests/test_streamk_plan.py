"""CPU checks of the stream-K work split (tests/streamk_model.py, a restatement of ao_b200/csrc/streamk.cuh):

* partition invariants of the split, exhaustively over small problems and every grid;
* the ring of every format policy (streamk_model.ring), pinned, so that a change to a policy's stage layout fails here
  first;
* coverage: the case lists of the exact GPU sweeps (test_exact_gemm_gpu.GRID_CASES and TAILS, the staged-gather
  cases, the grouped cases of the int4, nvfp4, fp8 weight-only, int8 and int8 weight-only grouped tests, and of the
  rowwise and blockwise e4m3 grouped tests) reach every segment pattern and every owner gather the kernel has, for
  every token-tile width of every format, so that an edit of a case list or of the walk that loses a pattern fails
  here, before a GPU run.  Where a kernel stages partials in its ring, the gather's boundaries are counted from S, its
  stage count: owners with 1, S - 1, S and S + 1 contributors, every remainder (c - S) mod GB of the register path
  behind the staged ones, more than 32 (and 64) flags polled after staging, and an owner tile with fewer valid token
  columns than the width.  Where it does not, the register gather's: 1 to 5 contributors, every c mod GB, more than
  32 and 64.
"""
import pytest

import grouped_model as gm
import streamk_model as sk


@pytest.mark.parametrize("KT", list(range(1, 65)))
def test_partition_invariants(KT):
    for tiles in range(1, 17):
        U = tiles * KT
        for G in range(1, min(U, 132) + 1):
            owned = [0] * U
            owners = {}
            for b in range(G):
                u0, u1 = sk.unit_begin(b, U, G), sk.unit_begin(b + 1, U, G)
                assert u1 > u0, f"empty CTA {b} (KT={KT} tiles={tiles} G={G})"
                segs = sk.walk(u0, u1 - u0, KT)
                u = u0
                for i, s in enumerate(segs):
                    assert s.tile * KT + s.kc0 == u and s.count > 0
                    for v in range(u, u + s.count):
                        owned[v] += 1
                        assert sk.cta_of_unit(v, U, G) == b
                    u += s.count
                    if s.kind == sk.CONTRIB:
                        assert i == 0 and s.kc0 > 0, "CONTRIB is only ever a CTA's first segment"
                    if s.kind == sk.OWNER:
                        assert i == len(segs) - 1 and s.kc0 == 0, "OWNER is only ever a CTA's last segment"
                        assert s.tile not in owners
                        owners[s.tile] = b
                    if s.kind == sk.FULL:
                        assert s.kc0 == 0 and s.count == KT
                assert u == u1
            assert owned == [1] * U, "every unit is computed exactly once"
            for t in range(tiles):
                first, last = sk.cta_of_unit(t * KT, U, G), sk.cta_of_unit(t * KT + KT - 1, U, G)
                if first == last:
                    assert t not in owners
                    continue
                # a split tile: its owner is the CTA of chunk 0, its contributors are CTAs owner+1 .. b_last, each of
                # which holds the tile as its first (CONTRIB) segment
                assert owners.get(t) == first
                for c in range(first + 1, last + 1):
                    seg0 = sk.walk(sk.unit_begin(c, U, G), sk.unit_begin(c + 1, U, G) - sk.unit_begin(c, U, G), KT)[0]
                    assert seg0.tile == t and seg0.kind == sk.CONTRIB


# S at token-tile widths 16 / 32 / 64 / 128, and the widths whose partials are staged, of the dense kernels and of the
# grouped ones (None: no grouped kernel); from the policy structs of ao_b200/csrc
RINGS = {
    "int4": ((7, 6, 7, 4), (16, 32), (12, 11, 7, 4)),
    "int8": ((6, 5, 8, 6), (16, 32), (11, 10, 8, 6)),
    "fp8": ((11, 10, 8), (), ()),
    "mxfp8": ((9, 8, 6, 4), (16, 32, 64), None),
    "mxfp4": ((12, 11, 8, 4), (16, 32), None),
    "nvfp4": ((12, 11, 8, 4), (16, 32), (12, 11, 8, 4)),
    "int8wo": ((5, 4, 6, 4), (16, 32, 64), (10, 8, 6, 4)),
    "fp8wo": ((9, 8, 6, 4), (16, 32, 64), (9, 8, 6, 4)),
    "fp8_sparse": ((9, 7, 11, 7), (16,), None),
    "fp8_blockwise": ((10, 9, 8), (), (10, 9, 8)),
}
TWO_CTAS = {("int4", 16), ("int4", 32), ("int8", 16), ("int8", 32), ("int8wo", 16), ("int8wo", 32),
            ("fp8_sparse", 16), ("fp8_sparse", 32)}


@pytest.mark.parametrize("fmt", sorted(RINGS))
def test_ring_of_every_policy(fmt):
    dense, staged, grouped = RINGS[fmt]
    assert sorted(sk.POLICIES) == sorted(RINGS) == sorted(sk.WIDTHS)
    for w, S in zip(sk.WIDTHS[fmt], dense):
        stage, ctas, stages, staging = sk.ring(fmt, w)
        assert stages == S, f"{fmt} at N_MMA={w}: S = {stages}, pinned {S}"
        assert ctas == (2 if (fmt, w) in TWO_CTAS else 1), f"{fmt} at N_MMA={w}: {ctas} CTAs per SM"
        assert staging == (w in staged), f"{fmt} at N_MMA={w}: STAGE_PARTIALS = {staging}"
        assert ctas * (sk.ring_smem(fmt, w) + sk.RESERVED_PER_CTA) <= sk.SMEM_PER_SM
    if grouped:
        for w, S in zip(sk.WIDTHS[fmt], grouped):
            stage, ctas, stages, staging = sk.ring(fmt, w, grouped=True)
            assert (stages, ctas) == (S, 1), f"grouped {fmt} at N_MMA={w}: S = {stages}, pinned {S}"
            assert staging == (w in staged), f"grouped {fmt} at N_MMA={w}: STAGE_PARTIALS = {staging}"
    # int8 weight-only at width 64: the partial (64 x 128 fp32) fills the whole stage
    assert sk.ring("int8wo", 64)[0] == 64 * sk.ROWS * 4


def _staged(p, grouped):
    return sk.ring(p.fmt, p.width, grouped)


def _gather_features(p, grouped=False):
    """The owner gathers of one plan: for a staging kernel the boundaries of the staged gather, else the register
    gather's (c = 1 .. 5, c % GB, c > 32, c > 64)."""
    f = set()
    _, _, S, staging = _staged(p, grouped)
    gb = sk.group_width(p.width)
    for t, (_, contrib) in p.owners.items():
        c = len(contrib)
        if not staging:
            if 1 <= c <= 5:
                f.add(f"contributors_{c}")
            f.add(f"rem_{c % gb}")
            if c > 32:
                f.add("contributors_gt32")
            if c > 64:
                f.add("contributors_gt64")
            continue
        n_staged, n_reg = p.gather_split(c)
        assert n_staged == min(c, S)
        for name, k in (("1", 1), ("S-1", S - 1), ("S", S), ("S+1", S + 1)):
            if c == k:
                f.add(f"c=" + name)
        if n_reg:
            f.add(f"(c-S)%GB={n_reg % gb}")
        if n_reg > 32:
            f.add("c-S>32")
        if n_reg > 64:
            f.add("c-S>64")
        if p.owner_cols(t) < p.width:
            f.add("ragged_owner")
    return f


def _required_gather(fmt, width, grouped=False, gt64=True):
    gb = sk.group_width(width)
    if not sk.ring(fmt, width, grouped)[3]:
        return ({"contributors_gt32", "contributors_gt64"} | {f"contributors_{c}" for c in range(1, 6)}
                | {f"rem_{r}" for r in range(gb)})
    return ({"c=1", "c=S-1", "c=S", "c=S+1", "c-S>32", "ragged_owner"} | ({"c-S>64"} if gt64 else set())
            | {f"(c-S)%GB={r}" for r in range(gb)})


def _missing(what, fmt, width, grouped, required, reached):
    missing = required - reached
    S = sk.ring(fmt, width, grouped)[2]
    return f"{what} at N_MMA={width} (S={S}): never reach {sorted(missing)}" if missing else None


def _features(p):
    """Which of the patterns the coverage check asks for one launch plan reaches."""
    f = _gather_features(p)
    for segs in p.ctas:
        kinds = [s.kind for s in segs]
        if kinds and all(k == sk.FULL for k in kinds):
            f.add("all_full")
        if kinds[:1] == [sk.CONTRIB] and kinds[-1:] == [sk.OWNER] and sk.FULL in kinds:
            f.add("contrib_full_owner")
        for s in segs:
            if s.kind == sk.CONTRIB and s.kc0 + s.count < p.KT:
                f.add("contrib_inside_tile")
    return f


def _required(fmt, width):
    return {"all_full", "contrib_inside_tile", "contrib_full_owner"} | _required_gather(fmt, width)


def _dense_runs():
    """(op, M, N, K, grid) of every launch of the dense exact sweeps: GRID_CASES, TAILS and the staged-gather cases."""
    import test_exact_gemm_gpu as suite
    import test_staged_gather_gpu as staged

    for op in suite.OPS:
        fmt = suite.OP_FORMAT[op]
        for M, N, K, grids in suite.GRID_CASES:
            if suite.shape_supported(op, M, N, K):
                for G in suite.grids_of(fmt, M, N, K, grids):
                    yield op, M, N, K, G
    for op, M, N, K, n_out in suite.TAILS:
        n = n_out or N
        U = sk.plan(suite.OP_FORMAT[op], M, n, K, grid=1).U
        for G in (None, 1, min(U, 132)):
            yield op, M, n, K, G
    for op, width, Ms, grids in staged.DENSE_CASES:
        for M in Ms:
            for G in grids:
                yield op, M, staged.N, staged.K, G


def test_exact_suite_grid_cases_cover_every_split_pattern():
    import test_exact_gemm_gpu as suite

    reached = {}
    for op, M, N, K, G in _dense_runs():
        p = sk.plan(suite.OP_FORMAT[op], M, N, K, grid=G)
        reached.setdefault((op, p.width), set()).update(_features(p))
    for op in suite.OPS:
        fmt = suite.OP_FORMAT[op]
        for width in sk.WIDTHS[fmt]:
            msg = _missing(op, fmt, width, False, _required(fmt, width), reached.get((op, width), set()))
            assert not msg, "the dense exact sweeps: " + msg


def test_staged_gather_cases_reach_every_staged_boundary():
    """The staged-gather test on its own reaches every boundary of every staging op and width, dense and grouped."""
    import test_exact_gemm_gpu as suite
    import test_staged_gather_gpu as staged

    dense = {}
    for op, width, Ms, grids in staged.DENSE_CASES:
        for M in Ms:
            for G in grids:
                p = sk.plan(suite.OP_FORMAT[op], M, staged.N, staged.K, grid=G)
                assert p.width == width
                dense.setdefault((op, width), set()).update(_gather_features(p))
    for op in staged.STAGED_OPS:
        fmt = suite.OP_FORMAT[op]
        for width in sk.WIDTHS[fmt]:
            if sk.ring(fmt, width)[3]:
                msg = _missing(op, fmt, width, False, _required_gather(fmt, width, gt64=False), dense.get((op, width), set()))
                assert not msg, "the staged-gather cases: " + msg
    for op in staged.CONTROL_OPS:
        assert not any(sk.ring(suite.OP_FORMAT[op], w)[3] for w in sk.WIDTHS[suite.OP_FORMAT[op]]), op
    grouped = {}
    for fmt, width, rows, grids, found in staged.GROUPED_CASES:
        for G in grids:
            p = gm.plan(gm.cumulative(rows), sum(rows), staged.N, staged.K, grid=G, fmt=fmt)
            grouped.setdefault((fmt, width), set()).update(_gather_features(p, grouped=True))
    for fmt in staged.GROUPED_FORMATS:
        for width in sk.WIDTHS[fmt]:
            if sk.ring(fmt, width, grouped=True)[3]:
                msg = _missing(f"grouped {fmt}", fmt, width, True, _required_gather(fmt, width, True, gt64=False),
                               grouped.get((fmt, width), set()))
                assert not msg, "the staged-gather cases: " + msg


def _grouped_suite_features(fmt, module):
    """{width: gather features} of the grid sweep of a grouped test module's GROUPED_CASES."""
    import importlib

    suite = importlib.import_module(module)
    reached = {}
    for case in suite.GROUPED_CASES:
        rows, N, K, tail, grids = (case[0], case[1], case[2], case[-2], case[-1])
        offs, M = gm.cumulative(rows), sum(rows) + tail
        args = (rows, N, K, tail, grids, 132)
        for G in [None] + (suite.grids_of(fmt, *args) if module == "test_grouped_int8_gpu" else suite.grids_of(*args)):
            p = gm.plan(offs, M, N, K, grid=G, fmt=fmt)
            reached.setdefault(p.width, set()).update(_gather_features(p, grouped=True))
    return reached


@pytest.mark.parametrize("fmt,module", [("int4", "test_grouped_int4_gpu"), ("nvfp4", "test_grouped_nvfp4_gpu"),
                                        ("fp8wo", "test_grouped_fp8_weight_only_gpu"), ("int8", "test_grouped_int8_gpu"),
                                        ("int8wo", "test_grouped_int8_gpu")])
def test_grouped_cases_reach_every_staged_boundary(fmt, module):
    """The grouped sweeps of a format (its GROUPED_CASES and the staged-gather cases) reach every boundary of the
    staged gather at every width whose partials are staged."""
    import test_staged_gather_gpu as staged

    reached = _grouped_suite_features(fmt, module)
    for f, width, rows, grids, found in staged.GROUPED_CASES:
        if f == fmt:
            for G in grids:
                p = gm.plan(gm.cumulative(rows), sum(rows), staged.N, staged.K, grid=G, fmt=fmt)
                reached.setdefault(p.width, set()).update(_gather_features(p, grouped=True))
    for width in sk.WIDTHS[fmt]:
        if sk.ring(fmt, width, grouped=True)[3]:
            msg = _missing(f"grouped {fmt}", fmt, width, True, _required_gather(fmt, width, True, gt64=False),
                           reached.get(width, set()))
            assert not msg, f"{module}.GROUPED_CASES and the staged-gather cases: " + msg


@pytest.mark.parametrize("fmt,module", [("fp8", "test_grouped_mm_gpu"),
                                        ("fp8_blockwise", "test_grouped_fp8_blockwise_gpu")])
def test_grouped_cases_reach_every_register_gather(fmt, module):
    """The grouped e4m3 kernels do not stage (PROMOTE): every owner reads its contributors' partials from L2.  Their
    GROUPED_CASES reach owners with 1 to 5 contributors, every remainder c mod GB of the partial groups, and more than
    32 and 64 contributors (flags polled 32 at a time), at every token-tile width."""
    reached = _grouped_suite_features(fmt, module)
    for width in sk.WIDTHS[fmt]:
        assert not sk.ring(fmt, width, grouped=True)[3], (fmt, width)
        msg = _missing(f"grouped {fmt}", fmt, width, True, _required_gather(fmt, width, True), reached.get(width, set()))
        assert not msg, f"{module}.GROUPED_CASES: " + msg
