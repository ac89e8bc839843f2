"""CPU checks of the stream-K work split (tests/streamk_model.py, a restatement of ao_b200/csrc/streamk.cuh):

* partition invariants of the split, exhaustively over small problems and every grid;
* coverage: the grid cases of the exact GPU suite (test_exact_gemm_gpu.GRID_CASES) reach every segment pattern and
  every owner gather the kernel has, for every token-tile width of every format, so that an edit of the case list or
  of the walk that loses a pattern fails here, before a GPU run.
"""
import pytest

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


def _features(p):
    """Which of the patterns the coverage check asks for one launch plan reaches."""
    f = set()
    for segs in p.ctas:
        kinds = [s.kind for s in segs]
        if kinds and all(k == sk.FULL for k in kinds):
            f.add("all_full")
        if kinds[:1] == [sk.CONTRIB] and kinds[-1:] == [sk.OWNER] and sk.FULL in kinds:
            f.add("contrib_full_owner")
        for s in segs:
            if s.kind == sk.CONTRIB and s.kc0 + s.count < p.KT:
                f.add("contrib_inside_tile")
    for c in p.contributor_counts():
        if 1 <= c <= 5:
            f.add(f"contributors_{c}")
        f.add(f"rem_{c % p.gb}")
        if c > 32:
            f.add("contributors_gt32")
        if c > 64:
            f.add("contributors_gt64")
    return f


def _required(width):
    gb = sk.group_width(width)
    return ({"all_full", "contrib_inside_tile", "contrib_full_owner", "contributors_gt32", "contributors_gt64"}
            | {f"contributors_{c}" for c in range(1, 6)} | {f"rem_{r}" for r in range(gb)})


def test_exact_suite_grid_cases_cover_every_split_pattern():
    import test_exact_gemm_gpu as suite

    reached = {}
    for op in suite.OPS:
        fmt = suite.OP_FORMAT[op]
        for M, N, K, grids in suite.GRID_CASES:
            if not suite.shape_supported(op, M, N, K):
                continue
            for G in suite.grids_of(fmt, M, N, K, grids):
                p = sk.plan(fmt, M, N, K, grid=G)
                reached.setdefault((op, p.width), set()).update(_features(p))
    for op in suite.OPS:
        fmt = suite.OP_FORMAT[op]
        for width in sk.WIDTHS[fmt]:
            missing = _required(width) - reached.get((op, width), set())
            assert not missing, f"{op} at N_MMA={width}: the grid cases never reach {sorted(missing)}"
