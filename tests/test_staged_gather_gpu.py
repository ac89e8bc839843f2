"""The owner's gather through ring stages (ts_gemm.cuh, Cfg::STAGE_PARTIALS), checked bit for bit at its boundaries.

An owner with c contributors stages the partials of the first min(c, S) of them in freed ring stages (S = the ring's
stage count, streamk_model.ring: 4 .. 12 by format, token-tile width and whether the kernel is grouped) and reads the
other c - S from L2: their flags polled 32 at a time, their partials loaded in groups of GB.  For every format and
width that stages, the forced grids give owners with c = 1, S - 1, S (the last staged copy lands in the stage of the
owner's own last chunk), S + 1 .. S + GB (every remainder of (c - S) mod GB) and S + 33 (more than 32 flags polled
after staging), over owner tiles whose valid token columns fill the width and fall short of it.

* dense: one 128-row tile at K = 8192 (64 chunks) over G = c + 1 CTAs, at M = the width, the width - 1 and (width 16)
  M = 1, through tests/exact_operands.py and the shared sweep of test_exact_gemm_gpu.py.  int8 weight-only at width 64
  copies a partial that fills its stage exactly; 2:4-sparse e4m3 stages at width 16 only, two CTAs per SM.  fp8 and
  blockwise fp8 (e4m3 x e4m3, PROMOTE) do not stage: they run the register path at the same counts, as controls.
* grouped (int4, nvfp4, fp8 weight-only, int8, int8 weight-only): experts of width - 1 and 1 rows, and one of width rows, so the copy length
  comes from each owner's expert; each file's exact grouped case and flag-checking sweep.

* every count at once: one tile at K = 4096 (32 chunks) over G = 2 .. 14 and 32 CTAs, so each format runs one owner
  with 1 to 13 and 31 contributors, at M = 1, 5, 16, 17 and 32 (two CTAs per SM at the decode widths of int4, int8
  and 2:4-sparse e4m3).

Every run asserts through tests/streamk_model.py that it has the contributor counts it claims, and
tests/test_streamk_plan.py checks on the CPU that the boundary cases reach every boundary.
"""
import pytest

import exact_operands as ex
import grouped_model as gm
import streamk_model as sk
from test_exact_gemm_gpu import OP_FORMAT, _sweep

pytestmark = pytest.mark.gpu

N, K = 128, 8192
STAGED_OPS = ("int4", "int8_dyn", "mxfp8", "nvfp4", "nvfp4w", "mxfp4", "int8wo", "fp8wo", "fp8_sparse")
CONTROL_OPS = ("fp8", "fp8_blockwise")
GROUPED_FORMATS = ("int4", "nvfp4", "fp8wo", "int8", "int8wo")
K_COUNTS, GRIDS_COUNTS = 4096, list(range(2, 15)) + [32]


def counts(S, width):
    """The contributor counts an owner is forced to: 1, S - 1, S, S + 1 .. S + GB and S + 33."""
    return sorted({1, S - 1, S} | {S + r for r in range(1, sk.group_width(width) + 1)} | {S + 33})


def dense_cases():
    """(op, width, token counts, forced grids) of every staging op and width, and of the fp8 control."""
    out = []
    for op in STAGED_OPS + CONTROL_OPS:
        fmt = OP_FORMAT[op]
        for w in sk.WIDTHS[fmt]:
            _, _, S, staging = sk.ring(fmt, w)
            if staging or op in CONTROL_OPS:
                out.append((op, w, [w, w - 1] + ([1] if w == 16 else []), [c + 1 for c in counts(S, w)]))
    return out


DENSE_CASES = dense_cases()


def grouped_cases(sm=132):
    """(fmt, width, rows per expert, forced grids, {(owner columns, contributors): grid}) of every staging grouped
    width: for each owner column count of the layout and each count of counts(), the first grid that has such an
    owner."""
    out = []
    for fmt in GROUPED_FORMATS:
        for w in sk.WIDTHS[fmt]:
            _, _, S, staging = sk.ring(fmt, w, grouped=True)
            if not staging:
                continue
            for rows in ([w - 1, 1], [w]):
                offs, M = gm.cumulative(rows), sum(rows)
                want = {(cols, c) for cols in rows for c in counts(S, w)}
                found = {}
                for G in range(1, min(gm.plan(offs, M, N, K, grid=1, sm=sm, fmt=fmt).U_bound, sm) + 1):
                    p = gm.plan(offs, M, N, K, grid=G, sm=sm, fmt=fmt)
                    assert p.width == w
                    for t, (_, contrib) in p.owners.items():
                        key = (p.owner_cols(t), len(contrib))
                        if key in want and key not in found:
                            found[key] = G
                out.append((fmt, w, rows, sorted(set(found.values())), found))
    return out


GROUPED_CASES = grouped_cases()


@pytest.fixture(scope="module")
def ops():
    return ex.ops()


@pytest.fixture
def set_ctas(ops):
    """Forces the stream-K CTA count; always restores the heuristic."""
    try:
        yield ops.debug_set_streamk_ctas
    finally:
        ops.debug_set_streamk_ctas(0)


@pytest.mark.parametrize("op,width,Ms,grids", DENSE_CASES, ids=lambda v: str(v))
def test_dense_staged_gather_boundaries_bit_exact(ops, set_ctas, op, width, Ms, grids):
    fmt = OP_FORMAT[op]
    for M in Ms:
        for G in grids:
            p = sk.plan(fmt, M, N, K, grid=G, sm=ex.sm_count())
            assert p.width == width and p.contributor_counts() == [G - 1], (M, G, p.width, p.contributor_counts())
    _sweep(ops, set_ctas, ex.build(op, width, N, K), grids, Ms=Ms)


def _grouped_case(fmt, offs, M, seed):
    if fmt == "int4":
        from test_grouped_int4_gpu import GroupedCase, _sweep as sweep

        return GroupedCase(offs, M, N, K, 128, seed), sweep
    if fmt in ("int8", "int8wo"):
        from test_grouped_int8_gpu import GroupedCase, _sweep as sweep

        return GroupedCase(fmt, offs, M, N, K, seed), sweep
    if fmt == "nvfp4":
        from test_grouped_nvfp4_gpu import GroupedCase, _sweep as sweep
    else:
        from test_grouped_fp8_weight_only_gpu import GroupedCase, _sweep as sweep
    return GroupedCase(offs, M, N, K, seed), sweep


@pytest.mark.parametrize("ci", range(len(GROUPED_CASES)), ids=lambda ci: "{}-{}-{}".format(*GROUPED_CASES[ci][:3]))
def test_grouped_staged_gather_boundaries_bit_exact(ops, set_ctas, ci):
    fmt, width, rows, grids, found = GROUPED_CASES[ci]
    offs, M = gm.cumulative(rows), sum(rows)
    for (cols, c), G in found.items():
        p = gm.plan(offs, M, N, K, grid=G, sm=ex.sm_count(), fmt=fmt)
        assert (cols, c) in {(p.owner_cols(t), len(cs)) for t, (_, cs) in p.owners.items()}, (cols, c, G)
    case, sweep = _grouped_case(fmt, offs, M, seed=ci)
    sweep(ops, set_ctas, case, grids, f"{fmt} width {width} rows {rows}")


@pytest.mark.parametrize("M", [1, 5, 16, 17, 32])
@pytest.mark.parametrize("op", ["int4", "int8_dyn", "fp8", "nvfp4", "fp8_sparse"])
def test_owner_contributor_counts_bit_exact(ops, set_ctas, op, M):
    for G in GRIDS_COUNTS:
        p = sk.plan(OP_FORMAT[op], M, N, K_COUNTS, grid=G, sm=ex.sm_count())
        assert p.contributor_counts() == [G - 1], (G, p.contributor_counts())
    _sweep(ops, set_ctas, ex.build(op, M, N, K_COUNTS), GRIDS_COUNTS)
