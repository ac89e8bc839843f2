// HQQ (half-quadratic quantization) qparams + codes for int4 weights, on the GPU (SURVEY §8f-2).
// Replaces `_choose_qparams_and_quantize_affine_hqq` + `optimize_weights_proximal_legacy`
// (torchao/quantization/quant_primitives.py:1797-2002) as called by Int4TilePackedTo4dTensor.from_hp
// (quantize_/workflows/int4/int4_tile_packed_to_4d_tensor.py:149-167): nbits 4, groups of g along K, lp_norm 0.7,
// beta 10 (x1.01 per iteration), at most 20 iterations, early stop when the tensor-wide mean |W - W_r| stops falling,
// zero converted to the tinygemm convention ((8 - zero) / scale), scale and zero returned in bf16.
//
// The reference runs ~15 elementwise / reduction torch kernels per iteration plus a host sync for the early stop
// (on CUDA in fp16).  Here: one warp owns one group (its g elements live in registers: g/32 per lane), the group
// reductions are warp shuffles, the solver runs in fp32 (the reference's CPU arithmetic) with explicit IEEE
// operations (no FMA contraction), and the early-stop decision stays on the device: every iteration is one update
// kernel that also leaves per-block sums of |W - W_r|, and a one-block kernel that adds them in a fixed order,
// compares with the best error so far and raises a stop flag that turns the remaining launches into no-ops.
// Setup-time code: ~40 tiny launches per weight, no host synchronisation, CUDA-graph friendly.
#include <cuda_bf16.h>

#include "common.h"

namespace ao {
namespace hqq {

constexpr int WARPS = 8;  // groups per block

struct Ctrl {
  double best;
  int stop;
  int iters;
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

template <int EPL>  // elements per lane = g / 32
__global__ void __launch_bounds__(WARPS * 32) init_kernel(const __nv_bfloat16* __restrict__ w, float* __restrict__ scale,
                                                          float* __restrict__ zero, long long groups, Ctrl* ctrl) {
  const long long gi = (long long)blockIdx.x * WARPS + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    ctrl->best = 1e4;
    ctrl->stop = 0;
    ctrl->iters = 0;
  }
  if (gi >= groups) return;
  float mn = INFINITY, mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < EPL; ++j) {
    const float v = __bfloat162float(w[gi * (EPL * 32) + j * 32 + lane]);
    mn = fminf(mn, v);
    mx = fmaxf(mx, v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if (lane == 0) {
    const float s = fminf(__fdiv_rn(15.0f, __fsub_rn(mx, mn)), 2e4f);
    scale[gi] = s;
    zero[gi] = rintf(__fmul_rn(-mn, s));
  }
}

template <int EPL>
__global__ void __launch_bounds__(WARPS * 32) iter_kernel(const __nv_bfloat16* __restrict__ w, const float* __restrict__ scale,
                                                          float* __restrict__ zero, long long groups, float inv_beta,
                                                          double* __restrict__ partial, const Ctrl* __restrict__ ctrl) {
  if (ctrl->stop) return;
  __shared__ float err_s[WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long gi = (long long)blockIdx.x * WARPS + warp;
  float err = 0.f;
  if (gi < groups) {
    const float s = scale[gi], z = zero[gi];
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < EPL; ++j) {
      const float W = __bfloat162float(w[gi * (EPL * 32) + j * 32 + lane]);
      float wq = rintf(__fadd_rn(__fmul_rn(W, s), z));
      wq = fminf(fmaxf(wq, 0.f), 15.f);
      const float wr = __fdiv_rn(__fsub_rn(wq, z), s);
      const float d = __fsub_rn(W, wr), a = fabsf(d);
      // shrinkage operator: sign(d) * relu(|d| - |d|^(p-1) / beta), p = 0.7; |d| = 0 gives 0
      float shr = a > 0.f ? __fsub_rn(a, __fmul_rn(inv_beta, powf(a, -0.3f))) : 0.f;
      shr = fmaxf(shr, 0.f);
      const float we = d > 0.f ? shr : -shr;
      acc = __fadd_rn(acc, __fsub_rn(wq, __fmul_rn(__fsub_rn(W, we), s)));
      err = __fadd_rn(err, a);
    }
    acc = warp_sum(acc);
    if (lane == 0) zero[gi] = __fdiv_rn(acc, (float)(EPL * 32));
  }
  err = warp_sum(err);
  if (lane == 0) err_s[warp] = err;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
#pragma unroll
    for (int i = 0; i < WARPS; ++i) t += (double)err_s[i];
    partial[blockIdx.x] = t;
  }
}

// one block: fixed-order sum of the per-block errors, early-stop bookkeeping
__global__ void __launch_bounds__(256) decide_kernel(const double* __restrict__ partial, int nblocks, double numel, Ctrl* ctrl) {
  if (ctrl->stop) return;
  __shared__ double sm[256];
  double t = 0.0;
  for (int i = threadIdx.x; i < nblocks; i += 256) t += partial[i];
  sm[threadIdx.x] = t;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) sm[threadIdx.x] += sm[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double cur = (double)(float)(sm[0] / numel);
    ctrl->iters += 1;
    if (cur < ctrl->best) ctrl->best = cur;
    else ctrl->stop = 1;
  }
}

template <int EPL>
__global__ void __launch_bounds__(WARPS * 32) final_kernel(const __nv_bfloat16* __restrict__ w, const float* __restrict__ scale,
                                                           const float* __restrict__ zero, long long groups,
                                                           uint8_t* __restrict__ q, __nv_bfloat16* __restrict__ scale_out,
                                                           __nv_bfloat16* __restrict__ zero_out) {
  const long long gi = (long long)blockIdx.x * WARPS + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (gi >= groups) return;
  const float s = scale[gi], z = zero[gi];
#pragma unroll
  for (int j = 0; j < EPL; ++j) {
    const long long e = gi * (EPL * 32) + j * 32 + lane;
    float wq = rintf(__fadd_rn(__fmul_rn(__bfloat162float(w[e]), s), z));
    q[e] = (uint8_t)fminf(fmaxf(wq, 0.f), 15.f);
  }
  if (lane == 0) {
    const float s_inv = __fdiv_rn(1.0f, s);
    scale_out[gi] = __float2bfloat16_rn(s_inv);
    zero_out[gi] = __float2bfloat16_rn(__fmul_rn(__fsub_rn(8.0f, z), s_inv));
  }
}

// Workspace layout: fp32 scale[G] and zero[G], then partial[nblocks] doubles at align16(8 G), then Ctrl.  The tests
// read all of it back after a call (tests/test_hqq_exact_gpu.py, layout in tests/hqq_model.py workspace_layout), so a
// change here needs the same change there.
template <int EPL>
static int run(const uint16_t* w, int N, int K, uint8_t* q, uint16_t* scale_out, uint16_t* zero_out, void* ws,
               cudaStream_t st) {
  const long long groups = (long long)N * K / (EPL * 32);
  const int nblocks = (int)((groups + WARPS - 1) / WARPS);
  float* scale = reinterpret_cast<float*>(ws);
  float* zero = scale + groups;
  double* partial = reinterpret_cast<double*>(reinterpret_cast<uint8_t*>(ws) + ((2 * groups * sizeof(float) + 15) / 16) * 16);
  Ctrl* ctrl = reinterpret_cast<Ctrl*>(partial + nblocks);
  const __nv_bfloat16* wb = reinterpret_cast<const __nv_bfloat16*>(w);
  AO_CUDA_CHECK(launch(init_kernel<EPL>, dim3(nblocks), dim3(WARPS * 32), 0, st, false, wb, scale, zero, groups, ctrl));
  double beta = 10.0;
  for (int it = 0; it < 20; ++it) {
    AO_CUDA_CHECK(launch(iter_kernel<EPL>, dim3(nblocks), dim3(WARPS * 32), 0, st, false, wb, (const float*)scale, zero, groups,
                         (float)(1.0 / beta), partial, (const Ctrl*)ctrl));
    AO_CUDA_CHECK(launch(decide_kernel, dim3(1), dim3(256), 0, st, false, (const double*)partial, nblocks,
                         (double)N * (double)K, ctrl));
    beta *= 1.01;
  }
  AO_CUDA_CHECK(launch(final_kernel<EPL>, dim3(nblocks), dim3(WARPS * 32), 0, st, false, wb, (const float*)scale, (const float*)zero,
                       groups, q, reinterpret_cast<__nv_bfloat16*>(scale_out), reinterpret_cast<__nv_bfloat16*>(zero_out)));
  return AO_OK;
}

}  // namespace hqq
}  // namespace ao

extern "C" size_t ao_int4_hqq_workspace_bytes(int N, int K, int group_size) {
  const size_t groups = (size_t)N * K / group_size;
  const size_t nblocks = (groups + ao::hqq::WARPS - 1) / ao::hqq::WARPS;
  return ((2 * groups * sizeof(float) + 15) / 16) * 16 + nblocks * sizeof(double) + 64;
}

extern "C" int ao_int4_hqq_quantize(const uint16_t* w, int N, int K, int group_size, uint8_t* q, uint16_t* scale,
                                    uint16_t* zero, void* workspace, size_t workspace_bytes, void* stream) {
  using namespace ao;
  AO_REQUIRE(N > 0 && K > 0, "int4 hqq: bad sizes N=%d K=%d", N, K);
  AO_REQUIRE(group_size == 32 || group_size == 64 || group_size == 128 || group_size == 256,
             "int4 hqq: group_size=%d not in {32,64,128,256}", group_size);
  AO_REQUIRE(K % group_size == 0, "int4 hqq: K=%d must be a multiple of group_size=%d", K, group_size);
  AO_REQUIRE(w && q && scale && zero && workspace, "int4 hqq: null pointer");
  AO_REQUIRE(workspace_bytes >= ao_int4_hqq_workspace_bytes(N, K, group_size), "int4 hqq: workspace too small");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  switch (group_size) {
    case 32: return hqq::run<1>(w, N, K, q, scale, zero, workspace, st);
    case 64: return hqq::run<2>(w, N, K, q, scale, zero, workspace, st);
    case 128: return hqq::run<4>(w, N, K, q, scale, zero, workspace, st);
    default: return hqq::run<8>(w, N, K, q, scale, zero, workspace, st);
  }
}
