"""On the CPU: every case of test_served_shapes_exact_gpu.py is exact by construction, and the served shapes keep
reaching the parts of the schedule that the toy cases of test_exact_gemm_gpu.py never do.

* the analytic bound of each case's value windows (tests/exact_operands.py bound()): K max|X| max|W| times the
  epilogue's scales plus the bias below 2^24 output quanta, and the e4m3 128-k chunk sums below 2^13;
* the stream-K split (tests/streamk_model.py, tests/grouped_model.py at 132 SMs): the largest KT, n-tile and m-block
  counts and the (expert, m-block) pair count J of the prefill routings are asserted, so shrinking the cases back to
  toy sizes fails here.
"""
import exact_operands as ex
import grouped_model as gm
import grouped_nvfp4_model as gnm
import streamk_model as sk
from test_exact_gemm_gpu import GRID_CASES
from test_served_shapes_exact_gpu import (GATHER_GRIDS, GATHER_SHAPE, MOE_OP, MOE_TAIL, MOE_TOKENS, OP_FORMAT, OPS,
                                          PRIME_GRID, TOKENS, dense_cases, moe_cases, routing)


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
            p = (gm if kind == "fp8" else gnm).plan(offs, offs[-1] + MOE_TAIL, N, K)
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
