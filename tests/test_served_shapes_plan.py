"""On the CPU: every case of test_served_shapes_exact_gpu.py is exact by construction, and the served shapes keep
reaching the parts of the schedule that the toy cases of test_exact_gemm_gpu.py never do.

* the analytic bound of each case's value windows (tests/exact_operands.py bound()): K max|X| max|W| times the
  epilogue's scales plus the bias below 2^24 output quanta, and the e4m3 128-k chunk sums below 2^13;
* the stream-K split (tests/streamk_model.py, tests/grouped_model.py at 132 SMs): the largest KT, n-tile and m-block
  counts and the (expert, m-block) pair count J of the prefill routings are asserted, for every grouped expert kind,
  so shrinking the cases back to toy sizes fails here;
* the DeepSeek-V3 expert stacks and the 32-expert torch.bmm stack stay larger than 2^31 bytes.
"""
import exact_operands as ex
import grouped_model as gm
import streamk_model as sk
from test_exact_gemm_gpu import GRID_CASES
from test_served_shapes_exact_gpu import (BMM_LARGE, GATHER_GRIDS, GATHER_SHAPE, MOE_OP, MOE_TAIL,
                                          MOE_TOKENS, OP_FORMAT, OPS, PRIME_GRID, TOKENS, bmm_cases, dense_cases,
                                          moe_cases, routing)

# the grouped expert kinds added after the first MoE sweep, and the toy suite that checks each under every grid
NEW_KINDS = ("int8", "int8wo", "fp8wo", "fp8_blockwise", "mxfp8", "mxfp4")
TOY_SUITE = {"int8": "test_grouped_int8_gpu", "int8wo": "test_grouped_int8_gpu",
             "fp8wo": "test_grouped_fp8_weight_only_gpu", "fp8_blockwise": "test_grouped_fp8_blockwise_gpu",
             "mxfp8": "test_grouped_mx_gpu", "mxfp4": "test_grouped_mx_gpu"}


def test_every_dense_case_is_exact_by_its_windows():
    for op, g, name, N, K in dense_cases():
        win = ex.window(op, K)
        s, c = ex.bound(op, K, win)
        assert s < 2.0**24, (op, name, s)
        assert c is None or c < 2.0**13, (op, name, c)


def test_every_moe_case_is_exact_by_its_windows():
    for kind, name, E, topk, N, K in moe_cases():
        s, c = ex.bound(MOE_OP[kind], K, ex.window(MOE_OP[kind], K))
        assert s < 2.0**24 and (c is None or c < 2.0**13), (kind, name, s, c)


def test_every_bmm_case_is_exact_by_its_window():
    for layout, name, B, K, N, Ms in bmm_cases():
        s, c = ex.bound("fp8", K, ex.window("fp8", K))
        assert s < 2.0**24 and c < 2.0**13, (layout, name, s, c)


def _has_mantissa(values):
    return any(ex.span([v])[0] / ex.span([v])[1] > 1 for v in values)


def test_windows_shrink_only_where_k_needs_it():
    """At K = 1024 every format but int8 and nvfp4 keeps its widest window; at the largest served K int4, int8, fp8
    and mxfp8 need a narrower one; every chosen window keeps scales with mantissa bits."""
    for op in ("int4", "fp8", "mxfp8", "nvfp4w"):
        assert ex.window(op, 1024) == ex.served_candidates(op)[0], op
    for op in ("int4", "int8_dyn", "fp8", "mxfp8"):
        assert ex.window(op, 28672) != ex.served_candidates(op)[0], op
    for K in (1024, 4096, 8192, 14336, 28672):
        for op in ("fp8", "nvfp4w_xs", "nvfp4w_rowpts"):
            assert _has_mantissa([o * 2.0**-8 for o in ex.window(op, K)["odd"]]), (op, K)
        for op in ("nvfp4", "nvfp4w", "nvfp4w_xs", "nvfp4w_rowpts"):
            assert _has_mantissa([ex._e4m3(b) for b in ex.window(op, K)["wb"]]), (op, K)


def _dense_maxima(cases):
    kt = nt = mb = gather = 0
    for fmt, M, N, K, grids in cases:
        for G in grids:
            p = sk.plan(fmt, M, N, K, grid=G)
            kt, nt, mb = max(kt, p.KT), max(nt, p.n_tiles), max(mb, p.m_blocks)
            gather = max([gather] + p.contributor_counts())
    return kt, nt, mb, gather


def test_served_dense_shapes_reach_past_the_toy_cases():
    served = _dense_maxima([(OP_FORMAT[op], M, N, K, (None, 1, PRIME_GRID))
                            for op, g, name, N, K in dense_cases() for M in TOKENS])
    toy = _dense_maxima([(f, M, N, K, [None] + list(grids or range(1, 133)))
                         for f in ("int4", "fp8") for M, N, K, grids in GRID_CASES])
    kt, nt, mb, gather = served
    assert kt == 224 and nt == 224 and mb == 32, served   # 70B down K = 28672; 8B gate|up N = 28672; fp8 2048 / 64
    assert kt > toy[0] and nt > toy[1] and mb > toy[2], (served, toy)
    assert gather == 4, served   # whole projections on 132 SMs: a tile is split across at most 5 CTAs
    # the default grid at served sizes: the MIN_UNITS rule never binds, every SM gets a CTA
    assert all(sk.plan(OP_FORMAT[op], M, N, K).G == 132 for op, g, name, N, K in dense_cases() for M in TOKENS)


def test_moe_routings_reach_past_the_toy_cases():
    j_prefill, experts, empty_all = 0, 0, True
    for kind, name, E, topk, N, K in moe_cases():
        for T in MOE_TOKENS:
            rows = routing(E, topk, T, seed=T + E)
            assert sum(rows) == T * topk
            empty_all &= rows.count(0) > 0
            offs = gm.cumulative(rows)
            p = gm.plan(offs, offs[-1] + MOE_TAIL, N, K, fmt=kind)
            assert p.mbp[-1] >= len([r for r in rows if r])
            if T == max(MOE_TOKENS):
                j_prefill = max(j_prefill, p.mbp[-1])
            experts = max(experts, E)
    assert empty_all, "every routing leaves some experts empty"
    assert experts == gm.MAX_EXPERTS
    assert j_prefill >= 700, j_prefill   # E = 1024 prefill: hundreds of (expert, m-block) pairs


def test_the_tile_case_reaches_gathers_of_more_than_32():
    """test_owner_gathers_of_many_contributors_at_served_k_bit_exact: one 128-feature tile at K = 28672 split across
    up to 132 CTAs, so the owner gathers 32 and more partials (131 at one token), which the whole projections do not."""
    name, N, K = GATHER_SHAPE
    per_op = {}
    for op in OPS:
        p = [sk.plan(OP_FORMAT[op], M, N, K, grid=G) for M in TOKENS for G in GATHER_GRIDS]
        per_op[op] = max(max(q.contributor_counts() or [0]) for q in p)
        assert any(32 < max(q.contributor_counts() or [0]) <= 64 for q in p), op
    assert min(per_op.values()) == 131, per_op


def _grouped_maxima(kind, cases):
    """(largest E, J, KT, n-tile count) over grouped launches (offs, M, N, K) of kind at 132 SMs."""
    E = j = kt = nt = 0
    for offs, M, N, K in cases:
        p = gm.plan(offs, M, N, K, fmt=kind)
        E, j, kt, nt = max(E, len(offs)), max(j, p.mbp[-1]), max(kt, p.KT), max(nt, p.n_tiles)
    return E, j, kt, nt


def test_every_new_expert_kind_reaches_past_its_toy_cases():
    """Each grouped kind added after the first sweep, at its served prefill routings: E = MAX_EXPERTS (the kernel's
    s_end / s_mbp arrays full), hundreds of (expert, m-block) pairs, KT = 112 (Mixtral down) and 112 n-tiles (Mixtral
    gate|up), more than its toy GROUPED_CASES reach.  The blockwise toy cases already run single tiles at K = 16384
    (KT = 128, the owner gathers of many contributors), so only its n-tiles must exceed them."""
    import importlib

    T = max(MOE_TOKENS)
    for kind in NEW_KINDS:
        served = []
        for k, name, E, topk, N, K in moe_cases():
            if k == kind:
                offs = gm.cumulative(routing(E, topk, T, seed=T + E))
                served.append((offs, offs[-1] + MOE_TAIL, N, K))
        toy = [(gm.cumulative(rows), sum(rows) + tail, N, K)
               for rows, N, K, tail, _ in importlib.import_module(TOY_SUITE[kind]).GROUPED_CASES]
        E, j, kt, nt = _grouped_maxima(kind, served)
        toy_E, toy_j, toy_kt, toy_nt = _grouped_maxima(kind, toy)
        assert E == gm.MAX_EXPERTS and j >= 700, (kind, E, j)
        assert kt == 112 and nt == 112, (kind, kt, nt)
        assert E > toy_E and j > toy_j and nt > toy_nt, (kind, (E, j, nt), (toy_E, toy_j, toy_nt))
        assert kt > toy_kt or kind == "fp8_blockwise", (kind, kt, toy_kt)


def test_the_largest_weight_stacks_pass_2_31_bytes():
    """The DeepSeek-V3 expert stacks (one byte per e4m3 weight) and the 32-expert [B, K, N] bmm stack are the cases
    whose weight offsets and tensor-map extents need more than 31 bits; no other case does."""
    big = {(kind, name) for kind, name, E, topk, N, K in moe_cases() if E * N * K >= 2**31}
    assert big == {(kind, name) for kind in ("fp8", "fp8_blockwise") for name in ("dsv3_gate_up", "dsv3_down")}, big
    layout, name, B, K, N, Ms = BMM_LARGE
    assert BMM_LARGE in bmm_cases() and layout == "kn" and B * K * N >= 2**31, BMM_LARGE
    assert all(B * K * N < 2**31 for layout, name, B, K, N, Ms in bmm_cases() if name != BMM_LARGE[1])


def test_bmm_cases_reach_past_the_toy_cases():
    """The served bmm shapes against test_fp8_bmm_gpu.py's exact cases (K <= 2048, N <= 272, B <= 4)."""
    from test_fp8_bmm_gpu import EXACT_CASES

    served = bmm_cases()
    assert {layout for layout, *_ in served} == {"nk", "kn"}
    assert min(K for *_, K, N, Ms in served) > max(K for B, M, K, N in EXACT_CASES)
    assert min(N for *_, N, Ms in served) > max(N for B, M, K, N in EXACT_CASES)
    assert min(B for _, _, B, *_ in served) > max(B for B, M, K, N in EXACT_CASES)
