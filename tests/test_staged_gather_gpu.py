"""The owner's gather through ring stages (ts_gemm.cuh, Cfg::STAGE_PARTIALS), checked bit for bit.

An owner stages the partials of its first S contributors (S = the ring's stage count, 5 .. 12 depending on format and
token-tile width) in shared memory and reads the rest from L2.  One 128-row tile at K = 4096 (32 chunks) forced over
G CTAs has one owner and G - 1 contributors; G = 2 .. 14 gives every owner from one contributor to more than any ring
holds, so each format and width runs with fewer contributors than stages, exactly as many, and more.  G = 32 (one
chunk per CTA) stages partials in ring stages that never held a chunk; G = 2 (16 chunks each) in stages the owner's
chunks have already cycled through more than once.  fp8 (e4m3 x e4m3) does not stage: its runs check the register
path at the same counts.  The operands are
tests/exact_operands.py's: the output must equal the fp64 reference rounded once, and the flags must be re-armed.
"""
import pytest

import exact_operands as ex
import streamk_model as sk
from test_exact_gemm_gpu import OP_FORMAT, _sweep

pytestmark = pytest.mark.gpu

N, K = 128, 4096
GRIDS = list(range(2, 15)) + [32]


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


@pytest.mark.parametrize("M", [1, 5, 16, 17, 32])
@pytest.mark.parametrize("op", ["int4", "int8_dyn", "fp8", "nvfp4"])
def test_owner_contributor_counts_bit_exact(ops, set_ctas, op, M):
    for G in GRIDS:
        p = sk.plan(OP_FORMAT[op], M, N, K, grid=G, sm=ex.sm_count())
        assert p.contributor_counts() == [G - 1], (G, p.contributor_counts())
    _sweep(ops, set_ctas, ex.build(op, M, N, K), GRIDS)
