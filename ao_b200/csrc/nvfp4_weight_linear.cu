// NVFP4 weight (e2m1 + e4m3 block-16 scales + f32 per-tensor scale) x bf16 activation linear.
//
// Semantics = F.linear(x, NVFP4Tensor.dequantize()) (torchao/prototype/mx_formats/nvfp4_tensor.py:199-231,
// weight-only handler inference_workflow.py:356-400), with an optional per-token activation scale applied in
// the epilogue so that e4m3-rowwise-quantised activations (BASELINE config 5; SURVEY section 0-5) run on the
// same kernel: their values are exact in bf16, the scale is a row factor.
// Hopper has no fp4 tensor-core kind, so the weights are dequantised in-kernel to the bf16 wgmma A fragment (exact,
// nvfp4_fmt.cuh) and run through the int4 path's kernel (ts_gemm.cuh); the per-tensor scale is applied in fp32 in
// the epilogue.
#include <cuda_bf16.h>
#include <cuda_fp8.h>

#include "common.h"
#include "nvfp4_fmt.cuh"
#include "ptx.cuh"
#include "ts_gemm.cuh"

namespace ao {
namespace nvf4w {

using tsg::ROWS;

template <int N_MMA>
static int launch_tc(const uint16_t* x, int ldx, const float* x_scale, int M, int K, const uint8_t* wq, const uint8_t* w_sf,
                     const float* b_pts, int b_pts_per_row, int N, const uint16_t* bias, uint16_t* y, void* ws,
                     size_t ws_bytes, cudaStream_t stream) {
  CUtensorMap tm_w, tm_sf, tm_x;
  if (int rc = make_weight_maps(wq, w_sf, N, K, &tm_w, &tm_sf)) return rc;
  {
    const uint64_t dims[2] = {(uint64_t)K, (uint64_t)M};
    const uint64_t str[1] = {(uint64_t)ldx * 2};
    const uint32_t box[2] = {64, (uint32_t)N_MMA};
    int rc = make_tmap(&tm_x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, x, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  tsg::Params p{};
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  p.row_scale = x_scale;
  p.out_scale = b_pts;
  p.out_scale_per_row = b_pts_per_row;
  p.y = reinterpret_cast<__nv_bfloat16*>(y);
  p.epi = tsg::EPI_FLOAT;
  p.acc_exp2 = Nvfp4Fmt::ACC_EXP2;
  p.aux_col_blocks = ceil_div(K / 16, 4);
  p.M = M; p.N = N; p.N_out = N; p.K = K; p.group_size = 16;
  p.n_tiles = ceil_div(N, ROWS);
  p.m_blocks = ceil_div(M, N_MMA);
  p.KT = K / 128;
  return tsg::launch_gemm<Nvfp4Fmt, N_MMA>(p, tm_w, tm_sf, tm_x, ws, ws_bytes, "nvfp4 weight linear", stream);
}

// per-token e4m3 "fake quantisation": x -> bf16(e4m3(x / s)) and s = f32(bf16(amax/448)); the bf16 values
// are exactly the e4m3 codes Float8Tensor.from_hp(x, PerRow()) would store (quant_primitives.py:2172-2287).
__global__ void __launch_bounds__(256) fp8_fakequant_rowwise_kernel(const __nv_bfloat16* __restrict__ x, int ldx, int K,
                                                                    __nv_bfloat16* __restrict__ xq,
                                                                    float* __restrict__ scale) {
  __shared__ float sh[8];
  // PDL: let the linear that consumes this output become resident and start its weight stream now; our own input may be
  // the previous kernel's output, so wait for it before the first read
  pdl_launch_dependents();
  pdl_wait();
  const int m = blockIdx.x;
  const uint4* xr = reinterpret_cast<const uint4*>(x + (size_t)m * ldx);
  const int nv = K / 8;
  float amax = 0.f;
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const uint4 v = xr[i];
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __bfloat1622float2(h[j]);
      amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
    }
  }
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = amax;
  __syncthreads();
  amax = sh[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) amax = fmaxf(amax, sh[i]);
  const float s = __bfloat162float(__float2bfloat16_rn(amax / 448.0f));
  if (threadIdx.x == 0) scale[m] = s;
  uint4* qr = reinterpret_cast<uint4*>(xq + (size_t)m * K);
  for (int i = threadIdx.x; i < nv; i += blockDim.x) {
    const uint4 v = xr[i];
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
    __nv_bfloat16 o[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __bfloat1622float2(h[j]);
      float a = fminf(fmaxf(f.x / s, -448.f), 448.f), b = fminf(fmaxf(f.y / s, -448.f), 448.f);
      if (s == 0.f) { a = 0.f; b = 0.f; }  // all-zero row: the reference yields NaN (0/0); we keep zeros
      const __nv_fp8_storage_t qa = __nv_cvt_float_to_fp8(a, __NV_SATFINITE, __NV_E4M3);
      const __nv_fp8_storage_t qb = __nv_cvt_float_to_fp8(b, __NV_SATFINITE, __NV_E4M3);
      o[2 * j] = __float2bfloat16_rn(__half2float(__half(__nv_cvt_fp8_to_halfraw(qa, __NV_E4M3))));
      o[2 * j + 1] = __float2bfloat16_rn(__half2float(__half(__nv_cvt_fp8_to_halfraw(qb, __NV_E4M3))));
    }
    qr[i] = *reinterpret_cast<const uint4*>(o);
  }
}

}  // namespace nvf4w
}  // namespace ao

using namespace ao;

extern "C" int ao_fp8_fakequant_rowwise_ld(const uint16_t* x, int ldx, int M, int K, uint16_t* xq_bf16, float* scale,
                                           void* stream) {
  AO_REQUIRE(M >= 0 && K > 0 && K % 8 == 0, "fp8 fakequant: bad sizes M=%d K=%d", M, K);
  if (M == 0) return AO_OK;
  AO_REQUIRE(x && xq_bf16 && scale, "fp8 fakequant: null pointer");
  AO_REQUIRE(ldx >= K && ldx % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0,
             "fp8 fakequant: ldx=%d must be >= K=%d, a multiple of 8, x 16-byte aligned", ldx, K);
  AO_CUDA_CHECK(ao::launch(nvf4w::fp8_fakequant_rowwise_kernel, dim3(M), dim3(256), 0,
                           reinterpret_cast<cudaStream_t>(stream), pdl_enabled(), reinterpret_cast<const __nv_bfloat16*>(x), ldx, K,
                           reinterpret_cast<__nv_bfloat16*>(xq_bf16), scale));
  return AO_OK;
}
extern "C" int ao_fp8_fakequant_rowwise(const uint16_t* x, int M, int K, uint16_t* xq_bf16, float* scale, void* stream) {
  return ao_fp8_fakequant_rowwise_ld(x, K, M, K, xq_bf16, scale, stream);
}

extern "C" int ao_nvfp4_weight_linear_ex(const uint16_t* x, int ldx, const float* x_scale, int M, int K, const uint8_t* wq,
                                         const uint8_t* w_scale_blocked, const float* b_pts, int b_pts_per_row, int N,
                                         const uint16_t* bias, uint16_t* y, void* workspace, size_t workspace_bytes,
                                         void* stream) {
  AO_REQUIRE(M >= 0 && K > 0 && N > 0, "nvfp4 weight linear: bad sizes M=%d K=%d N=%d", M, K, N);
  AO_REQUIRE(K % 128 == 0, "nvfp4 weight linear: K=%d must be a multiple of 128", K);
  AO_REQUIRE(N % 16 == 0, "nvfp4 weight linear: N=%d must be a multiple of 16 (inference_workflow.py:248-251)", N);
  AO_REQUIRE(ldx >= K && ldx % 8 == 0, "nvfp4 weight linear: ldx=%d must be >= K=%d and a multiple of 8", ldx, K);
  if (M == 0) return AO_OK;
  AO_REQUIRE(x && wq && w_scale_blocked && y, "nvfp4 weight linear: null pointer");
  AO_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0, "nvfp4 weight linear: x must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (M <= 16) return nvf4w::launch_tc<16>(x, ldx, x_scale, M, K, wq, w_scale_blocked, b_pts, b_pts_per_row, N, bias, y, workspace, workspace_bytes, st);
  if (M <= 32) return nvf4w::launch_tc<32>(x, ldx, x_scale, M, K, wq, w_scale_blocked, b_pts, b_pts_per_row, N, bias, y, workspace, workspace_bytes, st);
  if (M <= 64) return nvf4w::launch_tc<64>(x, ldx, x_scale, M, K, wq, w_scale_blocked, b_pts, b_pts_per_row, N, bias, y, workspace, workspace_bytes, st);
  return nvf4w::launch_tc<128>(x, ldx, x_scale, M, K, wq, w_scale_blocked, b_pts, b_pts_per_row, N, bias, y, workspace, workspace_bytes, st);
}

extern "C" int ao_nvfp4_weight_linear(const uint16_t* x, const float* x_scale, int M, int K, const uint8_t* wq,
                                      const uint8_t* w_scale_blocked, const float* b_pts, int N,
                                      const uint16_t* bias, uint16_t* y, void* workspace, size_t workspace_bytes,
                                      void* stream) {
  return ao_nvfp4_weight_linear_ex(x, K, x_scale, M, K, wq, w_scale_blocked, b_pts, 0, N, bias, y, workspace, workspace_bytes,
                                   stream);
}
