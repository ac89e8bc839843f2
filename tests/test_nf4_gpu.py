"""NF4 weights on the H100: the in-kernel conversion (every code byte in every fragment position, with the real table,
and scalers from every class of factor and mean) against torch's get_original_weight() on the same device; the GEMM bit
for bit on exact operands under every forced stream-K grid, token tile, K and N tail, block size and scaler-block
boundary, at a row pitch of the scalers that is not 16-byte aligned and at the Llama-3-8B projections; the handler's
accuracy and launch count, CUDA-graph replay, a PDL chain against a serialized run and AO_B200_NO_PDL=1, opcheck, and a
model quantized on the CPU and moved with .cuda()."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from test_nf4_host import restated_weight

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
GRIDS = (0, 1, 2, 3, 7, 64, 132)


@pytest.fixture(scope="module")
def ops():
    import ao_b200  # noqa: F401

    return torch.ops.ao_b200


@pytest.fixture
def set_ctas(ops):
    try:
        yield ops.debug_set_streamk_ctas
    finally:
        ops.debug_set_streamk_ctas(0)


def bits(t):
    return t.contiguous().view(torch.int16)


def make_nf4(qd, qs, f, mean, table, N, K, bs, sbs):
    from ao_b200.quantization import NF4Tensor
    from ao_b200.quantization.quantize_.workflows.nf4.nf4_tensor import SubclassTensorArgs

    meta = SubclassTensorArgs(torch.Size([N, K]), (K, 1), 0, torch.bfloat16, qd.device, False)
    return NF4Tensor(meta, bs, N * K // bs, sbs, qs, f, mean, qd, table)


def dequantized(t):
    return restated_weight(t.quantized_data, t.quantized_scalers, t.quantization_factor, t.scaler_mean, t.nf4,
                           tuple(t.shape), t.block_size, t.scaler_block_size)


class Exact:
    """Stored tensors whose products and sums are exact in fp32: a table of multiples of 1/8, scalers qs / f + 1/2 with
    f in {1/2, 1, 2}, activations in -2..2, so every output is one rounding of an exact sum, whatever the order."""

    def __init__(self, M, N, K, bs=64, sbs=256, bias=True, seed=0):
        g = torch.Generator().manual_seed(seed)
        nb = N * K // bs
        self.t = make_nf4(torch.randint(0, 256, (N * K // 2,), generator=g, dtype=torch.uint8).to(DEV),
                          torch.randint(-6, 7, (nb,), generator=g, dtype=torch.int8).to(DEV),
                          torch.pow(2.0, torch.randint(-1, 2, (nb // sbs,), generator=g).float()).to(torch.bfloat16).to(DEV),
                          torch.tensor(0.5, dtype=torch.bfloat16, device=DEV),
                          ((torch.arange(16) - 8) / 8).to(torch.bfloat16).to(DEV), N, K, bs, sbs)
        self.x = torch.randint(-2, 3, (M, K), generator=g).to(torch.bfloat16).to(DEV)
        self.bias = torch.randint(-64, 65, (N,), generator=g).to(torch.bfloat16).to(DEV) * 0.25 if bias else None
        w = dequantized(self.t)
        y = (self.x.double() @ w.double().t()).to(torch.bfloat16)
        self.ref = y if self.bias is None else y + self.bias


def run(case):
    return F.linear(case.x, case.t, case.bias)


def same_with_nans(a, b):
    na, nb = torch.isnan(a.float()), torch.isnan(b.float())
    return torch.equal(na, nb) and torch.equal(bits(a)[~na], bits(b)[~nb])


def test_every_byte_in_every_fragment_position_and_scaler_classes(ops):
    """512 rows x 256 k, row r holding byte (r + j) % 256 at code byte j: rows 0..255 put every byte in every position
    of both chunks, with the real NF4 table (the quantizer's).  One factor per scaler: bf16 values whose division
    rounds, powers of two that make bf16-subnormal scalers, and negative factors; in every fourth of rows 256..511, 0
    (scalers +-inf, NaN for qs = 0) and inf (scaler = mean).  Means 0, one that rounds in the add, and a subnormal one.
    One-hot activations read every w~ back: bf16(1 * w~) exactly, and a row with a non-finite weight is NaN everywhere
    (0 * inf), as torch computes it."""
    from ao_b200.quantization import to_nf4

    N, K, bs = 512, 256, 16
    nb = N * K // bs
    g = torch.Generator().manual_seed(1)
    qd = ((torch.arange(N)[:, None] + torch.arange(K // 2)[None, :]) % 256).to(torch.uint8).flatten()
    qs = torch.randint(-128, 128, (nb,), generator=g, dtype=torch.int8)
    f = (torch.randn(nb, generator=g) * 30).to(torch.bfloat16)
    blk, row = torch.arange(nb) % 4, torch.arange(nb) // (K // bs)
    tiny = blk == 1
    f[tiny] = torch.pow(2.0, torch.randint(120, 134, (int(tiny.sum()),), generator=g).float()).to(torch.bfloat16)
    f[blk == 2] = -f[blk == 2].abs()
    special = (row >= 256) & (row % 4 == 0)
    f[special & (blk == 0)] = 0.0
    f[special & (blk == 3)] = float("inf")
    table = to_nf4(torch.randn(256, 64, dtype=torch.bfloat16)).nf4
    for mean in (0.0, 0.3137, -1e-38):
        t = make_nf4(qd.to(DEV), qs.to(DEV), f.to(DEV), torch.tensor(mean, dtype=torch.bfloat16, device=DEV),
                     table.to(DEV), N, K, bs, 1)
        w = t.get_original_weight()
        assert same_with_nans(w, dequantized(t))
        eye = torch.eye(K, dtype=torch.bfloat16, device=DEV)
        y = F.linear(eye, t)
        # the reference's own linear of the same w~ on the same device: every bit, NaN as NaN
        ref = F.linear(eye, w)
        bad = ~((y.float() == ref.float()) | (torch.isnan(y.float()) & torch.isnan(ref.float())))
        assert same_with_nans(y, ref), (mean, int(bad.sum()), y[bad][:8].tolist(), ref[bad][:8].tolist())
        # the values of w~ themselves in every row without a non-finite weight (-0 reads back as the sum's +0)
        finite = torch.isfinite(w.float()).all(dim=1)
        assert finite[:256].all() and not finite[256::4].any()
        assert torch.equal(y[:, finite].float(), w[finite].t().float()), mean
        assert torch.isnan(y[:, ~finite].float()).all()
        if mean != 0.3137:
            sub = (w.float().abs() < 2.0**-126) & (w.float() != 0)
            assert sub[:256].any(), "no subnormal weight exercised"


@pytest.mark.parametrize("M", [1, 16, 17, 32, 64, 128, 129])
def test_every_forced_grid_bit_exact(ops, set_ctas, M):
    case = Exact(M, 384, 1024, seed=M)
    for grid in GRIDS:
        set_ctas(grid)
        assert torch.equal(bits(run(case)), bits(case.ref)), (M, grid)


@pytest.mark.parametrize("M", [512, 4096])
def test_prefill_tiles_bit_exact(ops, set_ctas, M):
    case = Exact(M, 640, 2048, seed=M)
    for grid in (0, 5, 132):
        set_ctas(grid)
        assert torch.equal(bits(run(case)), bits(case.ref)), (M, grid)


@pytest.mark.parametrize("bs,sbs,N,K", [(16, 4, 200, 160), (64, 3, 130, 576), (128, 5, 136, 1280), (192, 2, 256, 576),
                                         (256, 1, 72, 768), (64, 256, 256, 11008)])
@pytest.mark.parametrize("bias", [True, False])
def test_block_sizes_tails_and_scaler_blocks_bit_exact(ops, set_ctas, bs, sbs, N, K, bias):
    """Block sizes 16..256 (192: a block across two chunks), K and N tails, scaler blocks of a few scalers (their
    boundaries inside every tile), and K = 11008, whose scaler row pitch 172 bytes is not a multiple of 16."""
    for M in (1, 33):
        case = Exact(M, N, K, bs=bs, sbs=sbs, bias=bias, seed=bs + M)
        for grid in (0, 1, 3, 64):
            set_ctas(grid)
            assert torch.equal(bits(run(case)), bits(case.ref)), (bs, sbs, N, K, M, grid)


@pytest.mark.parametrize("N,K", [(6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336)])
def test_llama3_8b_shapes_bit_exact(ops, N, K):
    for M in (1, 32, 512):
        case = Exact(M, N, K, seed=N + M)
        assert torch.equal(bits(run(case)), bits(case.ref)), (N, K, M)


def test_row_strided_and_3d_activations(ops):
    case = Exact(8, 256, 512, seed=3)
    wide = torch.zeros(8, 768, dtype=torch.bfloat16, device=DEV)
    wide[:, 128:640] = case.x
    assert torch.equal(bits(F.linear(wide[:, 128:640], case.t, case.bias)), bits(case.ref))
    y3 = F.linear(case.x.view(2, 4, 512), case.t, case.bias)
    assert y3.shape == (2, 4, 256) and torch.equal(bits(y3.view(8, 256)), bits(case.ref))


def _quantized_model(K=4096, N=4096, bias=True, device=DEV):
    from ao_b200.prototype._nf4tensor_api import NF4WeightOnlyConfig
    from ao_b200.quantization import quantize_

    torch.manual_seed(0)
    m = nn.Sequential(nn.Linear(K, N, bias=bias)).to(torch.bfloat16).to(device)
    w = m[0].weight.detach().clone()
    quantize_(m, NF4WeightOnlyConfig())
    return m, w


def test_handler_accuracy_and_one_launch(ops):
    from ao_b200.quantization import NF4Tensor
    from ao_b200.quantization.utils import compute_error

    m, w = _quantized_model()
    t = m[0].weight
    assert isinstance(t, NF4Tensor) and t.is_cuda
    torch.testing.assert_close(t.get_original_weight(), w, atol=0.13, rtol=0.13)   # the reference's own bound
    for M in (1, 32, 512):
        x = torch.randn(M, 4096, dtype=torch.bfloat16, device=DEV)
        with torch.no_grad():
            torch.cuda.synchronize()
            n0 = ops.launch_count()
            y = m(x)
            assert ops.launch_count() - n0 == 1   # one kernel per linear: the scalers are decoded inside it
            recipe = F.linear(x, t.get_original_weight()) + m[0].bias
        assert compute_error(F.linear(x, w, m[0].bias), y) > 15.0
        # the reference's recipe, up to the order of the fp32 sums: within a few bf16 ulps of its magnitude
        assert (y.float() - recipe.float()).abs().max() <= 2e-2 * recipe.float().abs().max()


def test_cuda_graph_replay(ops):
    case, other = Exact(32, 384, 1024, seed=5), Exact(32, 384, 1024, seed=6)
    x = case.x.clone()
    run(case)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = F.linear(x, case.t, case.bias)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(bits(y), bits(case.ref))
    x.copy_(other.x)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(bits(y), bits(F.linear(other.x, case.t, case.bias)))


CHAIN = """
import sys, torch, torch.nn as nn
sys.path.insert(0, {root!r})
from ao_b200.prototype._nf4tensor_api import NF4WeightOnlyConfig
from ao_b200.quantization import quantize_
torch.manual_seed(7)
ls = [nn.Linear(2048, 2048, bias=True, device="cuda", dtype=torch.bfloat16) for _ in range(3)]
for l in ls:
    quantize_(l, NF4WeightOnlyConfig())
outs = []
with torch.no_grad():
    for M in (1, 32, 300):
        x = torch.randn(M, 2048, device="cuda", dtype=torch.bfloat16)
        outs.append(ls[2](ls[1](ls[0](x))))
torch.cuda.synchronize()
sys.stdout.buffer.write(b"".join(o.view(torch.int16).cpu().numpy().tobytes() for o in outs))
"""


def test_pdl_chain_matches_serialized_and_no_pdl():
    """Three NF4 linears back to back (each GEMM prefetches its weights under the previous one) against the same
    launches separated by synchronisations, and against a process that launches without PDL."""
    from ao_b200.prototype._nf4tensor_api import NF4WeightOnlyConfig
    from ao_b200.quantization import quantize_

    torch.manual_seed(7)
    ls = [nn.Linear(2048, 2048, bias=True, device=DEV, dtype=torch.bfloat16) for _ in range(3)]
    for l in ls:
        quantize_(l, NF4WeightOnlyConfig())
    outs = []
    with torch.no_grad():
        for M in (1, 32, 300):
            x = torch.randn(M, 2048, device=DEV, dtype=torch.bfloat16)
            chained = ls[2](ls[1](ls[0](x)))
            a = ls[0](x)
            torch.cuda.synchronize()
            b = ls[1](a)
            torch.cuda.synchronize()
            serial = ls[2](b)
            torch.cuda.synchronize()
            assert torch.equal(bits(chained), bits(serial)), f"M={M}"
            outs.append(chained)
    here = b"".join(o.view(torch.int16).cpu().numpy().tobytes() for o in outs)
    for no_pdl in ("0", "1"):
        env = dict(os.environ, AO_B200_NO_PDL=no_pdl)
        r = subprocess.run([sys.executable, "-c", CHAIN.format(root=ROOT)], env=env, stdout=subprocess.PIPE, check=True)
        assert r.stdout == here, f"AO_B200_NO_PDL={no_pdl}: the chain's outputs differ"


def test_opcheck(ops):
    case = Exact(17, 256, 512, seed=9)
    t = case.t
    args = (case.x, t.quantized_data, t.quantized_scalers, t.quantization_factor, t.scaler_mean, t.nf4, 64, 256)
    torch.library.opcheck(ops.nf4_linear.default, args + (case.bias,))
    torch.library.opcheck(ops.nf4_linear.default, args + (None,))


def test_cpu_quantized_model_moved_with_cuda(ops):
    from ao_b200.quantization import NF4Tensor

    m, w = _quantized_model(K=1024, N=512, device="cpu")
    cpu_w = m[0].weight.get_original_weight()
    m = m.cuda()
    t = m[0].weight
    assert isinstance(t, NF4Tensor) and t.is_cuda and t.quantized_data.is_cuda and t.nf4.is_cuda
    assert t.shape == (512, 1024) and t.dtype == torch.bfloat16 and t.block_size == 64 and t.scaler_block_size == 256
    assert torch.equal(t.get_original_weight().cpu(), cpu_w)
    x = torch.randn(4, 1024, dtype=torch.bfloat16, device=DEV)
    with torch.no_grad():
        y = m(x)
    recipe = F.linear(x, t.get_original_weight()) + m[0].bias
    assert (y.float() - recipe.float()).abs().max() <= 2e-2 * recipe.float().abs().max()
    back = t.cpu()
    assert isinstance(back, NF4Tensor) and not back.quantized_data.is_cuda and back.device.type == "cpu"
