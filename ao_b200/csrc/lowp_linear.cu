// Swap-AB streaming GEMMs for 8-bit / 4-bit operands on Hopper wgmma (sm_90a), all on the kernel of ts_gemm.cuh:
//   int8 x int8 -> int32  (wgmma s8, both operands TMA tiles)      replaces aten._int_mm + the scale epilogue
//   e4m3 x e4m3 -> f32    (wgmma e4m3, both operands TMA tiles)    replaces torch._scaled_mm rowwise
//   mxfp8 block-32 e8m0   (bf16 wgmma on exactly dequantised operands)   replaces torch._scaled_mm block-scaled
//   nvfp4 block-16 e4m3   (bf16 wgmma on exactly dequantised operands)   replaces torch._scaled_mm fp4 + pts/bias kernels
//   nvfp4 weight x bf16   (bf16 wgmma, weights dequantised exactly)      replaces F.linear on the dequantised weight
// Reference call sites: int8/kernels.py:18-76,114-144 + int8_tensor.py:305-359;
// float8/inference.py:86-123; mx_formats/mx_tensor.py:759-843; nvfp4_tensor.py:487-578.
//
// The weight matrix W[N,K] (K-major, exactly the stored qdata) is the wgmma A operand: 128 output features per tile;
// the activations are the B operand (N_MMA tokens).  Hopper's tensor cores have no block-scaled kinds, so for mxfp8 and
// nvfp4 every element is multiplied by its block scale BEFORE the MMA, in bf16: the weights inside the kernel
// (register-A fragments), the activations by a pre-pass into a bf16 slab of the workspace.  The fp32 sums then see the
// same products a block-scaled MMA sees, as long as the scaled element is exact in bf16:
//   * e2m1 x e4m3 (at most 6 significant bits, >= 2^-10): exact for every finite non-negative scale byte, the
//     subnormal and zero bytes included (nvfp4_fmt.cuh);
//   * e4m3 x 2^(e-127) (4 significant bits, every code a multiple of 2^-9): exact for e8m0 bytes e >= 3.  For
//     e = 0, 1, 2 the codes whose lowest set bit lies below 2^-(6+e) need bits under 2^-133, the smallest bf16
//     subnormal, and round.
#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <stdlib.h>

#include <type_traits>

#include "common.h"
#include "nvfp4_fmt.cuh"
#include "ptx.cuh"
#include "streamk.cuh"
#include "ts_gemm.cuh"

namespace ao {
namespace lowp {

enum Kind { KIND_I8 = 0, KIND_F8 = 1, KIND_MXF8 = 2, KIND_NVF4 = 3 };

using tsg::KCHUNK;
using tsg::ROWS;

// K-major byte weights W[N][K] in 128-row x 128-k boxes, 128-byte swizzle (int8, e4m3, mxfp8)
static int kmajor_byte_map(const uint8_t* wq, int N, int K, CUtensorMap* tm) {
  const uint64_t dims[2] = {(uint64_t)K, (uint64_t)N};
  const uint64_t str[1] = {(uint64_t)K};
  const uint32_t box[2] = {KCHUNK, ROWS};
  return make_tmap(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, wq, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

// int8 / e4m3: both operands straight from the TMA tiles (128-byte swizzle, 128 k per chunk = four k32 wgmmas)
template <int KIND>
struct SsFmt {
  static constexpr bool SS = true;
  static constexpr bool PROMOTE = KIND == KIND_F8;   // int8 sums are exact in s32
  // e4m3 waits for each chunk's wgmmas (PROMOTE) and measured 14 % slower per decode step at two CTAs per SM
  static constexpr bool DECODE_2CTA = !PROMOTE;
  static constexpr int X_ELEM_BYTES = 1;
  static constexpr int W_BYTES = ROWS * KCHUNK;   // 16 KiB
  static constexpr int AUX_BYTES = 0;
  static constexpr int EPI = KIND == KIND_I8 ? tsg::EPI_I8 : tsg::EPI_F8;
  static constexpr int ACC_EXP2 = 0;
  static constexpr int MAX_N_MMA = KIND == KIND_F8 ? 64 : 128;   // e4m3 keeps a second accumulator per chunk
  // no aux operand: the weight map stands in for it, so that the kernel's descriptor prefetch reads a valid map
  static int make_maps(const uint8_t* wq, int N, int K, CUtensorMap* tm_w, CUtensorMap* tm_aux) {
    if (int rc = kmajor_byte_map(wq, N, K, tm_w)) return rc;
    *tm_aux = *tm_w;
    return AO_OK;
  }
  __device__ static __forceinline__ uint32_t w_tx_bytes(const tsg::Params&) { return W_BYTES; }
  __device__ static __forceinline__ void issue_w(const CUtensorMap* tm_w, const CUtensorMap*, const tsg::Params&,
                                                 uint8_t* w_dst, uint8_t*, uint64_t* bar, int n_tile, int kc,
                                                 uint64_t policy) {
    tma_load_2d(w_dst, tm_w, bar, kc * KCHUNK, n_tile * ROWS, policy);
  }
  // grouped kernels: 128 rows from `row` of the [E * N, K] map of all experts' weights
  __device__ static __forceinline__ void issue_w_rows(const CUtensorMap* tm_w, const CUtensorMap*, const tsg::Params&,
                                                      uint8_t* w_dst, uint8_t*, uint64_t* bar, int row, int kc,
                                                      uint64_t policy) {
    tma_load_2d(w_dst, tm_w, bar, kc * KCHUNK, row, policy);
  }
  template <int N_MMA>
  __device__ static __forceinline__ void mma(uint32_t (&acc)[N_MMA / 2], uint32_t w_s, uint32_t x_s, int wg,
                                             uint32_t scale_d) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const uint64_t ad = wgmma_desc_k_sw128(w_s + wg * (64 * 128) + kk * 32);
      const uint64_t bd = wgmma_desc_k_sw128(x_s + kk * 32);
      if (KIND == KIND_I8) Wgmma<N_MMA>::ss_s8(acc, ad, bd, kk == 0 ? scale_d : 1u);
      else Wgmma<N_MMA>::ss_e4m3(acc, ad, bd, kk == 0 ? scale_d : 1u);
    }
  }
};

// 2^(e - 127) for an e8m0 byte (0xFF = NaN)
__device__ __forceinline__ float e8m0_to_f32(uint32_t e) {
  return __uint_as_float(e == 0xFFu ? 0x7FC00000u : (e ? e << 23 : 0x00400000u));
}

// mxfp8 weights as the register-A operand: e4m3 pairs x their block-32 e8m0 scale -> bf16 (exact)
struct Mxfp8Fmt {
  static constexpr bool SS = false;
  // at 104 consumer registers the dequant of a chunk spills inside the chunk loop: one CTA per SM
  static constexpr bool DECODE_2CTA = false;
  static constexpr bool PROMOTE = false;
  static constexpr int X_ELEM_BYTES = 2;
  static constexpr int W_BYTES = ROWS * KCHUNK;   // 128 rows x 128 bytes, 128-byte swizzle
  static constexpr int AUX_BYTES = 512;           // one blocked scale tile (4 scales = 128 k per row)
  static constexpr int EPI = tsg::EPI_FLOAT;
  static constexpr int ACC_EXP2 = 0;
  static constexpr int MAX_N_MMA = 128;
  // the weights and the blocked scale tiles, one 512-byte tile per box
  static int make_maps(const uint8_t* wq, const uint8_t* w_sf, int N, int K, CUtensorMap* tm_w, CUtensorMap* tm_sf) {
    if (int rc = kmajor_byte_map(wq, N, K, tm_w)) return rc;
    const uint64_t dims[2] = {128, (uint64_t)ceil_div(N, ROWS) * (uint64_t)ceil_div(K / 32, 4)};
    const uint64_t str[1] = {512};
    const uint32_t box[2] = {128, 1};
    return make_tmap(tm_sf, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, w_sf, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE);
  }
  __device__ static __forceinline__ uint32_t w_tx_bytes(const tsg::Params&) { return W_BYTES + AUX_BYTES; }
  __device__ static __forceinline__ void issue_w(const CUtensorMap* tm_w, const CUtensorMap* tm_sf, const tsg::Params& p,
                                                 uint8_t* w_dst, uint8_t* aux_dst, uint64_t* bar, int n_tile, int kc,
                                                 uint64_t policy) {
    tma_load_2d(w_dst, tm_w, bar, kc * KCHUNK, n_tile * ROWS, policy);
    tma_load_2d(aux_dst, tm_sf, bar, 0, n_tile * p.aux_col_blocks + kc, policy);
  }
  // the thread's two fragment rows: for k16 step kk the e4m3 pair at k 16kk + 2t (low half) and + 8 (high half)
  struct Raw {
    uint32_t v[2][8];
    uint32_t sc[2];
  };
  __device__ static __forceinline__ void load(const tsg::Params&, uint32_t w_smem, uint32_t aux_smem, int row_lo, int lane,
                                              Raw& raw) {
    const int t = lane & 3;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = row_lo + 8 * h;
      raw.sc[h] = tsg::lds32(aux_smem + (uint32_t)(r & 31) * 16u + (uint32_t)(r >> 5) * 4u);
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        const uint32_t a = w_smem + (uint32_t)r * 128u + ((uint32_t)(kk ^ (r & 7)) << 4) + 2 * t;   // TMA 128B swizzle
        raw.v[h][kk] = tsg::lds16(a) | (tsg::lds16(a + 8) << 16);
      }
    }
  }
  __device__ static __forceinline__ uint32_t deq(uint32_t pair, float s) {
    const __half2_raw hr = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)pair, __NV_E4M3);
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hr));
    __nv_bfloat162 b = __floats2bfloat162_rn(f.x * s, f.y * s);
    return *reinterpret_cast<uint32_t*>(&b);
  }
  __device__ static __forceinline__ void frag(const tsg::Params&, const Raw& raw, int kk, uint32_t (&a)[4]) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float s = e8m0_to_f32((raw.sc[h] >> (8 * (kk >> 1))) & 0xFFu);   // the 32-k block of step kk
      a[h] = deq(raw.v[h][kk] & 0xFFFFu, s);
      a[h + 2] = deq(raw.v[h][kk] >> 16, s);
    }
  }
};

// Activation pre-pass of the block-scaled kinds: rows [m0, m0 + rows) of the quantised activations -> bf16 [rows][K],
// every element times its block scale (exact in bf16).  One thread per 16 elements.
template <int KIND>
__global__ void __launch_bounds__(256) dequant_act_kernel(const uint8_t* __restrict__ xq, const uint8_t* __restrict__ x_sf,
                                                          int m0, int rows, int K, int sf_col_blocks,
                                                          __nv_bfloat16* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();   // the slab may still be read by the previous GEMM; the activations may be the previous kernel's output
  const int per_row = K / 16;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)rows * per_row) return;
  const int mr = (int)(idx / per_row), k0 = (int)(idx % per_row) * 16, m = m0 + mr;
  const int kb = KIND == KIND_NVF4 ? k0 / 16 : k0 / 32;
  const size_t tile = (size_t)(m / 128) * sf_col_blocks + kb / 4;
  const uint32_t sbyte = x_sf[tile * 512 + (m % 32) * 16 + ((m % 128) / 32) * 4 + kb % 4];
  __nv_bfloat16 o[16];
  if (KIND == KIND_NVF4) {
    const __half_raw sh = __nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)sbyte, __NV_E4M3);
    const float s = __half2float(*reinterpret_cast<const __half*>(&sh));
    const uint2 v = *reinterpret_cast<const uint2*>(xq + (size_t)m * (K / 2) + k0 / 2);
    const float lut[8] = {0.f, 0.5f, 1.f, 1.5f, 2.f, 3.f, 4.f, 6.f};
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const uint32_t nib = ((j < 8 ? v.x : v.y) >> (4 * (j & 7))) & 0xFu;
      const float x = lut[nib & 7] * s;
      o[j] = __float2bfloat16_rn(nib & 8 ? -x : x);
    }
  } else {
    const float s = e8m0_to_f32(sbyte);
    const uint4 v = *reinterpret_cast<const uint4*>(xq + (size_t)m * K + k0);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const __half2_raw hr = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(w[j >> 1] >> (16 * (j & 1))), __NV_E4M3);
      const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hr));
      o[2 * j] = __float2bfloat16_rn(f.x * s);
      o[2 * j + 1] = __float2bfloat16_rn(f.y * s);
    }
  }
  uint4* dst = reinterpret_cast<uint4*>(out + (size_t)mr * K + k0);
  dst[0] = reinterpret_cast<const uint4*>(o)[0];
  dst[1] = reinterpret_cast<const uint4*>(o)[1];
}

// int8 / fp8 rowwise
template <int KIND>
static int rowwise(const uint8_t* xq, const float* x_scale, int M, int K, const uint8_t* wq, const float* w_scale, int N,
                   const uint16_t* bias, uint16_t* y, int32_t* i32_out, void* ws, size_t ws_bytes, void* stream) {
  using Fmt = SsFmt<KIND>;
  CUtensorMap tm_w, tm_aux;
  if (int rc = Fmt::make_maps(wq, N, K, &tm_w, &tm_aux)) return rc;
  tsg::Params p{};
  p.row_scale = x_scale;
  p.w_scale = w_scale;
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  p.y = reinterpret_cast<__nv_bfloat16*>(y);
  p.i32_out = i32_out;
  p.M = M; p.N = N; p.N_out = N; p.K = K;
  return tsg::run<Fmt>(p, tm_w, tm_aux, xq, K, ws, ws_bytes, "lowp linear", reinterpret_cast<cudaStream_t>(stream));
}

// mxfp8 / nvfp4: activation slabs dequantised into the workspace behind the partial slots, one GEMM per slab
template <int KIND>
static int block_scaled(const uint8_t* xq, const uint8_t* x_sf, const float* a_pts, int M, int K, const uint8_t* wq,
                        const uint8_t* w_sf, const float* b_pts, int N, const uint16_t* bias, uint16_t* y, void* ws,
                        size_t ws_bytes, void* stream) {
  using Fmt = std::conditional_t<KIND == KIND_NVF4, nvf4w::Nvfp4Fmt, Mxfp8Fmt>;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int sf_per_row = KIND == KIND_MXF8 ? K / 32 : K / 16;
  const int sf_col_blocks = ceil_div(sf_per_row, 4);
  CUtensorMap tm_w, tm_sf;
  if (int rc = Fmt::make_maps(wq, w_sf, N, K, &tm_w, &tm_sf)) return rc;
  // the partial slots take at most (SMs x 128 x 128) words; the slab starts on the next MiB (restated by
  // tests/test_exact_gemm_gpu.py::test_block_scaled_activation_slabs, which sizes workspaces to given slab heights)
  const size_t act_off = (streamk::WS_PARTIAL_OFF + (size_t)sm_count() * ROWS * 128 * 4 + (1u << 20) - 1) & ~(size_t)((1u << 20) - 1);
  const size_t row_bytes = (size_t)K * 2;
  long long slab = ws && ws_bytes > act_off ? (long long)((ws_bytes - act_off) / row_bytes) : 0;
  if (slab >= 128) slab &= ~127LL;
  if (slab < 1)
    return fail(AO_ERR_WORKSPACE, "block-scaled linear: workspace too small for one bf16 activation row (K=%d)", K);
  __nv_bfloat16* xb = reinterpret_cast<__nv_bfloat16*>(reinterpret_cast<uint8_t*>(ws) + act_off);
  for (int m0 = 0; m0 < M; m0 += (int)slab) {
    const int rows = (int)(M - m0 < slab ? M - m0 : slab);
    const long long threads = (long long)rows * (K / 16);
    AO_CUDA_CHECK(ao::launch(dequant_act_kernel<KIND>, dim3((unsigned)((threads + 255) / 256)), dim3(256), 0, st,
                             pdl_enabled(), xq, x_sf, m0, rows, K, sf_col_blocks, xb));
    tsg::Params p{};
    p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
    p.y = reinterpret_cast<__nv_bfloat16*>(y) + (size_t)m0 * N;
    p.out_scale = KIND == KIND_NVF4 ? b_pts : nullptr;
    p.out_scale2 = KIND == KIND_NVF4 ? a_pts : nullptr;
    p.aux_col_blocks = sf_col_blocks;
    p.M = rows; p.N = N; p.N_out = N; p.K = K;
    if (int rc = tsg::run<Fmt>(p, tm_w, tm_sf, xb, K, ws, act_off, "lowp linear", st)) return rc;
  }
  return AO_OK;
}

}  // namespace lowp
}  // namespace ao

using namespace ao;

extern "C" int ao_int8_dyn_linear(const int8_t* xq, const float* x_scale, int M, int K,
                                  const int8_t* wq, const float* w_scale, int N,
                                  const uint16_t* bias, uint16_t* y, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  AO_REQUIRE(M >= 0 && K > 0 && N > 0, "int8 linear: bad sizes M=%d K=%d N=%d", M, K, N);
  AO_REQUIRE(K % 16 == 0, "int8 linear: K=%d must be a multiple of 16 (TMA row pitch)", K);
  AO_REQUIRE(N % 8 == 0, "int8 linear: N=%d must be a multiple of 8 (reference: int8/kernels.py:48-58)", N);
  if (M == 0) return AO_OK;
  AO_REQUIRE(xq && x_scale && wq && w_scale && y, "int8 linear: null pointer");
  return lowp::rowwise<lowp::KIND_I8>(reinterpret_cast<const uint8_t*>(xq), x_scale, M, K,
                                      reinterpret_cast<const uint8_t*>(wq), w_scale, N, bias, y, nullptr, workspace,
                                      workspace_bytes, stream);
}

extern "C" int ao_int8_mm_i32(const int8_t* xq, int M, int K, const int8_t* wq, int N, int32_t* acc,
                              void* workspace, size_t workspace_bytes, void* stream) {
  AO_REQUIRE(M >= 0 && K > 0 && N > 0 && K % 16 == 0, "int8 mm: bad sizes M=%d K=%d N=%d (K%%16==0)", M, K, N);
  if (M == 0) return AO_OK;
  AO_REQUIRE(xq && wq && acc, "int8 mm: null pointer");
  return lowp::rowwise<lowp::KIND_I8>(reinterpret_cast<const uint8_t*>(xq), nullptr, M, K,
                                      reinterpret_cast<const uint8_t*>(wq), nullptr, N, nullptr, nullptr, acc, workspace,
                                      workspace_bytes, stream);
}

extern "C" int ao_fp8_rowwise_linear(const uint8_t* xq, const float* x_scale, int M, int K,
                                     const uint8_t* wq, const float* w_scale, int N,
                                     const uint16_t* bias, uint16_t* y, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  AO_REQUIRE(M >= 0 && K > 0 && N > 0, "fp8 linear: bad sizes M=%d K=%d N=%d", M, K, N);
  AO_REQUIRE(K % 16 == 0, "fp8 linear: K=%d must be a multiple of 16 (reference: quantization/utils.py:663-687)", K);
  AO_REQUIRE(N % 16 == 0, "fp8 linear: N=%d must be a multiple of 16 (reference: quantization/utils.py:663-687)", N);
  if (M == 0) return AO_OK;
  AO_REQUIRE(xq && x_scale && wq && w_scale && y, "fp8 linear: null pointer");
  return lowp::rowwise<lowp::KIND_F8>(xq, x_scale, M, K, wq, w_scale, N, bias, y, nullptr, workspace, workspace_bytes,
                                      stream);
}

// torch._grouped_mm(x, W.transpose(-2, -1), offs) on rowwise e4m3 operands: expert e's rows [offs[e-1], offs[e]) of
// xq against its weights wq[e] (the stored [E, N, K] qdata), the dense kernel's epilogue with w_scale[e, :].  offs
// stays on the device (grouped schedule, ts_gemm.cuh).
extern "C" int ao_fp8_rowwise_grouped_mm(const uint8_t* xq, const float* x_scale, int M, int K,
                                         const uint8_t* wq, const float* w_scale, int E, int N,
                                         const int32_t* offs, uint16_t* y, void* workspace,
                                         size_t workspace_bytes, void* stream) {
  AO_REQUIRE(M >= 0 && K > 0 && N > 0, "fp8 grouped mm: bad sizes M=%d K=%d N=%d", M, K, N);
  AO_REQUIRE(E >= 1 && E <= tsg::MAX_EXPERTS, "fp8 grouped mm: E=%d experts must be in [1, %d]", E, tsg::MAX_EXPERTS);
  AO_REQUIRE(K % 16 == 0, "fp8 grouped mm: K=%d must be a multiple of 16 (TMA row pitch)", K);
  AO_REQUIRE(N % 16 == 0, "fp8 grouped mm: N=%d must be a multiple of 16", N);
  AO_REQUIRE((long long)E * N <= 0x7FFFFFFF, "fp8 grouped mm: E*N=%lld weight rows exceed the int32 range", (long long)E * N);
  if (M == 0) return AO_OK;
  AO_REQUIRE(xq && x_scale && wq && w_scale && offs && y && workspace, "fp8 grouped mm: null pointer");
  using Fmt = tsg::Grouped<lowp::SsFmt<lowp::KIND_F8>>;
  CUtensorMap tm_w, tm_aux;
  if (int rc = Fmt::make_maps(wq, E * N, K, &tm_w, &tm_aux)) return rc;
  tsg::Params p{};
  p.row_scale = x_scale;
  p.w_scale = w_scale;
  p.y = reinterpret_cast<__nv_bfloat16*>(y);
  p.offs = offs;
  p.E = E;
  p.M = M; p.N = N; p.N_out = N; p.K = K;
  return tsg::run<Fmt>(p, tm_w, tm_aux, xq, K, workspace, workspace_bytes, "fp8 grouped mm",
                             reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int ao_mxfp8_linear(const uint8_t* xq, const uint8_t* x_scale_blocked, int M, int K,
                               const uint8_t* wq, const uint8_t* w_scale_blocked, int N,
                               const uint16_t* bias, uint16_t* y, void* workspace,
                               size_t workspace_bytes, void* stream) {
  AO_REQUIRE(M >= 0 && K > 0 && N > 0, "mxfp8 linear: bad sizes M=%d K=%d N=%d", M, K, N);
  AO_REQUIRE(K % 32 == 0, "mxfp8 linear: K=%d must be a multiple of 32 (mx_tensor.py:244-246)", K);
  if (M == 0) return AO_OK;
  AO_REQUIRE(xq && x_scale_blocked && wq && w_scale_blocked && y, "mxfp8 linear: null pointer");
  return lowp::block_scaled<lowp::KIND_MXF8>(xq, x_scale_blocked, nullptr, M, K, wq, w_scale_blocked, nullptr, N, bias,
                                             y, workspace, workspace_bytes, stream);
}

extern "C" int ao_nvfp4_linear(const uint8_t* xq, const uint8_t* x_scale_blocked, const float* a_pts,
                               int M, int K, const uint8_t* wq, const uint8_t* w_scale_blocked,
                               const float* b_pts, int N, const uint16_t* bias, uint16_t* y,
                               void* workspace, size_t workspace_bytes, void* stream) {
  AO_REQUIRE(M >= 0 && K > 0 && N > 0, "nvfp4 linear: bad sizes M=%d K=%d N=%d", M, K, N);
  AO_REQUIRE(K % 256 == 0, "nvfp4 linear: K=%d must be a multiple of 256", K);
  AO_REQUIRE(N % 16 == 0, "nvfp4 linear: N=%d must be a multiple of 16 (inference_workflow.py:248-251)", N);
  if (M == 0) return AO_OK;
  AO_REQUIRE(xq && x_scale_blocked && wq && w_scale_blocked && y, "nvfp4 linear: null pointer");
  return lowp::block_scaled<lowp::KIND_NVF4>(xq, x_scale_blocked, a_pts, M, K, wq, w_scale_blocked, b_pts, N, bias, y,
                                             workspace, workspace_bytes, stream);
}

// nvfp4 weights x bf16 activations = F.linear(x, NVFP4Tensor.dequantize()) (nvfp4_tensor.py:199-231, weight-only
// handler inference_workflow.py:356-400).  The optional per-token x_scale is applied in the epilogue, so that
// e4m3-rowwise activations (ao_fp8_fakequant_rowwise: values exact in bf16, the scale a row factor) run on the same
// kernel; b_pts is one per-tensor scale or (b_pts_per_row) one per output feature.
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
  CUtensorMap tm_w, tm_sf;
  if (int rc = nvf4w::Nvfp4Fmt::make_maps(wq, w_scale_blocked, N, K, &tm_w, &tm_sf)) return rc;
  tsg::Params p{};
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  p.row_scale = x_scale;
  p.out_scale = b_pts;
  p.out_scale_per_row = b_pts_per_row;
  p.y = reinterpret_cast<__nv_bfloat16*>(y);
  p.aux_col_blocks = ceil_div(K / 16, 4);
  p.M = M; p.N = N; p.N_out = N; p.K = K;
  return tsg::run<nvf4w::Nvfp4Fmt>(p, tm_w, tm_sf, x, ldx, workspace, workspace_bytes, "nvfp4 weight linear",
                                   reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int ao_nvfp4_weight_linear(const uint16_t* x, const float* x_scale, int M, int K, const uint8_t* wq,
                                      const uint8_t* w_scale_blocked, const float* b_pts, int N,
                                      const uint16_t* bias, uint16_t* y, void* workspace, size_t workspace_bytes,
                                      void* stream) {
  return ao_nvfp4_weight_linear_ex(x, K, x_scale, M, K, wq, w_scale_blocked, b_pts, 0, N, bias, y, workspace, workspace_bytes,
                                   stream);
}

// torch._grouped_mm(x, W.transpose(-2, -1), offs) on NVFP4 expert weights (nvfp4_tensor.py:709-753), 2-D x 3-D:
// expert e's rows [offs[e-1], offs[e]) of x (bf16; for NVFP4 activations the exactly dequantised codes of
// ao_nvfp4_fakequant_grouped) against wq[e] (the stored [E, N, K/2] qdata) with its blocked scales, the nvfp4-weight
// epilogue y = acc * x_scale[m] * w_pts[e].  offs stays on the device (grouped schedule, ts_gemm.cuh).
extern "C" int ao_nvfp4_grouped_mm(const uint16_t* x, const float* x_scale, int M, int K, const uint8_t* wq,
                                   const uint8_t* w_scale_blocked, const float* w_pts, int E, int N,
                                   const int32_t* offs, uint16_t* y, void* workspace, size_t workspace_bytes,
                                   void* stream) {
  AO_REQUIRE(M >= 0 && K > 0 && N > 0, "nvfp4 grouped mm: bad sizes M=%d K=%d N=%d", M, K, N);
  AO_REQUIRE(E >= 1 && E <= tsg::MAX_EXPERTS, "nvfp4 grouped mm: E=%d experts must be in [1, %d]", E, tsg::MAX_EXPERTS);
  AO_REQUIRE(K % 128 == 0, "nvfp4 grouped mm: K=%d must be a multiple of 128", K);
  // every expert's weights and scales start on a 128-row block of the stacked [E * N, ..] tensors
  AO_REQUIRE(N % 128 == 0, "nvfp4 grouped mm: N=%d must be a multiple of 128", N);
  AO_REQUIRE((long long)E * N <= 0x7FFFFFFF, "nvfp4 grouped mm: E*N=%lld weight rows exceed the int32 range", (long long)E * N);
  if (M == 0) return AO_OK;
  AO_REQUIRE(x && wq && w_scale_blocked && w_pts && offs && y && workspace, "nvfp4 grouped mm: null pointer");
  AO_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0, "nvfp4 grouped mm: x must be 16-byte aligned");
  using Fmt = tsg::Grouped<nvf4w::Nvfp4Fmt>;
  CUtensorMap tm_w, tm_sf;
  if (int rc = Fmt::make_maps(wq, w_scale_blocked, E * N, K, &tm_w, &tm_sf)) return rc;
  tsg::Params p{};
  p.row_scale = x_scale;
  p.out_scale = w_pts;
  p.y = reinterpret_cast<__nv_bfloat16*>(y);
  p.offs = offs;
  p.E = E;
  p.aux_col_blocks = ceil_div(K / 16, 4);
  p.M = M; p.N = N; p.N_out = N; p.K = K;
  return tsg::run<Fmt>(p, tm_w, tm_sf, x, K, workspace, workspace_bytes, "nvfp4 grouped mm",
                       reinterpret_cast<cudaStream_t>(stream));
}
