// Swap-AB streaming GEMMs for 8-bit / 4-bit operands on Hopper wgmma (sm_90a), all on the kernel of ts_gemm.cuh:
//   int8 x int8 -> int32  (wgmma s8, both operands TMA tiles)      replaces aten._int_mm + the scale epilogue
//                         and, per expert, aten._int_mm on select()ed int8 expert weights
//   e4m3 x e4m3 -> f32    (wgmma e4m3, both operands TMA tiles)    replaces torch._scaled_mm rowwise
//                         and, 1x128 x 128x128 block scales, the reference's blockwise Triton GEMM
//                         and, 2:4-sparse weights (wgmma.sp), the reference's CUTLASS sparse GEMM
//   mxfp8 block-32 e8m0   (bf16 wgmma on exactly dequantised operands)   replaces torch._scaled_mm block-scaled
//                         and, mxfp8 and mxfp4 per expert, torch._grouped_mm on 3-D MX expert weights
//   nvfp4 block-16 e4m3   (bf16 wgmma on exactly dequantised operands)   replaces torch._scaled_mm fp4 + pts/bias kernels
//   nvfp4 weight x bf16   (bf16 wgmma, weights dequantised exactly)      replaces F.linear on the dequantised weight
//   mxfp4 block-32 e8m0   (bf16 wgmma on exactly dequantised operands)   replaces F.linear on both dequantize()s
//   int8 weight x bf16    (bf16 wgmma, weights converted exactly)        replaces torch.mm on qdata.to(bf16) + the scale
//                         and, per expert, the same on select()ed int8 expert weights
//   e4m3 weight x bf16    (bf16 wgmma, weights dequantised per element)  replaces torch.matmul on the dequantised weight
//                         and, per expert, torch._grouped_mm on the dequantised expert weights
//   nf4 weight x bf16     (bf16 wgmma, weights dequantised per element)  replaces F.linear on get_original_weight()
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
//   * e2m1 x 2^(e-127) (at most 2 significant bits, every code a multiple of 2^-1): exact for every e8m0 byte
//     0x00..0xFE, the smallest product 2^-128 being a bf16 subnormal; the products at or above 2^128 (|code| >= 4 at
//     byte 253, |code| >= 2 at byte 254) are inf, as in the reference's fp32 dequantize, and byte 0xFF is NaN;
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

enum Kind { KIND_I8 = 0, KIND_F8 = 1, KIND_MXF8 = 2, KIND_NVF4 = 3, KIND_MXF4 = 4 };

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
  // PROMOTE (e4m3): the rowwise scales stay in the epilogue, each chunk's partial is added as it is
  struct NoScales {};
  template <int N_MMA>
  __device__ static __forceinline__ NoScales chunk_scales(const tsg::Params&, uint32_t, int, int, int, int) { return {}; }
  template <int N_MMA>
  __device__ static __forceinline__ void promote(uint32_t (&acc)[N_MMA / 2], const uint32_t (&part)[N_MMA / 2],
                                                 uint32_t accumulate, NoScales) {
#pragma unroll
    for (int j = 0; j < N_MMA / 2; ++j)
      acc[j] = accumulate ? __float_as_uint(__uint_as_float(acc[j]) + __uint_as_float(part[j])) : part[j];
  }
};

// Static e4m3 activations (PrototypeFloat8Tensor): the operands, wgmmas and promotion of SsFmt<KIND_F8>, and the EPI_F8
// output with a per-tensor weight scale read as one value, followed, with output_act_quant_scale, by its e4m3
// quantize-dequantize (EPI_F8_STATIC)
struct F8StaticFmt : SsFmt<KIND_F8> {
  static constexpr int EPI = tsg::EPI_F8_STATIC;
};

// Rowwise e4m3 expert weights stored [E, K, N] (N-major: torch.bmm(x, w) on Llama-4-style experts), under the grouped
// schedule only: the operands, wgmmas, promotion and EPI_F8 epilogue of SsFmt<KIND_F8>, with w_scale [E, N].  A stage
// holds a [128 k][128 n] box of a 3-D map over [E, K, N] (128-byte swizzle): k past K and n past N are zero-filled,
// never read from the next expert.  Each consumer warpgroup transposes its 64 n of it into the K-major 128-byte-swizzled
// [64 n][128 k] layout SsFmt::mma reads (W_XPOSE_BYTES, ts_gemm.cuh).
struct F8NMajorFmt : SsFmt<KIND_F8> {
  static constexpr int W_XPOSE_BYTES = ROWS * KCHUNK;   // 8 KiB per consumer warpgroup
  static int make_maps(const uint8_t* wq, int E, int K, int N, CUtensorMap* tm_w, CUtensorMap* tm_aux) {
    const uint64_t dims[3] = {(uint64_t)N, (uint64_t)K, (uint64_t)E};
    const uint64_t str[2] = {(uint64_t)N, (uint64_t)K * N};
    const uint32_t box[3] = {ROWS, KCHUNK, 1};
    if (int rc = make_tmap(tm_w, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, wq, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B))
      return rc;
    *tm_aux = *tm_w;
    return AO_OK;
  }
  __device__ static __forceinline__ void issue_w_rows(const CUtensorMap* tm_w, const CUtensorMap*, const tsg::Params& p,
                                                      uint8_t* w_dst, uint8_t*, uint64_t* bar, int row, int kc,
                                                      uint64_t policy) {
    const int e = row / p.N;
    tma_load_3d(w_dst, tm_w, bar, row - e * p.N, kc * KCHUNK, e, policy);
  }
  // Thread t of warpgroup wg: warp w = t / 32 reads the 16 n of column chunk c = 4wg + w, lane (kg = lane % 8, ng =
  // lane / 8) the 4 n at 16c + 4ng of k rows 16kg .. 16kg + 15, one 32-bit word per row, and stores the 16 k of each of
  // its 4 n as one 16-byte chunk of that n's row.  Byte (k, n) of the stage is at k*128 + ((n/16) ^ (k%8))*16 + n%16,
  // byte (n, k) of the buffer at n*128 + ((k/16) ^ (n%8))*16 + k%16.  Word j of a thread is row 16kg + (j ^ kg): the 8
  // lanes of one ng then read 8 distinct swizzle phases, so each load's 32 words fall in 32 banks, and the 8 lanes of
  // a quarter-warp store 8 distinct 16-byte chunks of one row.  That load order is undone in the byte transposes: word
  // (4q + t) ^ kg = 4(q ^ (kg/4)) + (t ^ kg%4), a byte permutation within each 4x4 block (the prmt selectors) and a
  // swap of neighbouring blocks (kg >= 4).
  __device__ static __forceinline__ void xpose(uint32_t src, uint32_t dst, int wg, int t) {
    const int w = t >> 5, lane = t & 31;
    const int kg = lane & 7, ng = lane >> 3, c = 4 * wg + w;
    uint32_t r[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int k = 16 * kg + (j ^ kg);
      r[j] = tsg::lds32(src + k * 128 + ((c ^ (k & 7)) << 4) + 4 * ng);
    }
    // stage 2 selectors: byte t of [a0 b0 c0 d0] (0x5410) taken from byte t ^ (kg % 4); [a1 b1 c1 d1] is 0x2222 above
    const int m = kg & 3;
    uint32_t s_lo = 0;
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int u = b ^ m;
      s_lo |= (uint32_t)((u & 1) | ((u & 2) << 1)) << (4 * b);
    }
    const uint32_t s_hi = s_lo + 0x2222u;
    uint32_t o[4][4];   // o[i][q]: the bytes of n 16c + 4ng + i, k 16kg + 4(q ^ (kg/4)) ..
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t lo01 = __byte_perm(r[4 * q], r[4 * q + 1], 0x5140), hi01 = __byte_perm(r[4 * q], r[4 * q + 1], 0x7362);
      const uint32_t lo23 = __byte_perm(r[4 * q + 2], r[4 * q + 3], 0x5140);
      const uint32_t hi23 = __byte_perm(r[4 * q + 2], r[4 * q + 3], 0x7362);
      o[0][q] = __byte_perm(lo01, lo23, s_lo);
      o[1][q] = __byte_perm(lo01, lo23, s_hi);
      o[2][q] = __byte_perm(hi01, hi23, s_lo);
      o[3][q] = __byte_perm(hi01, hi23, s_hi);
    }
    const bool swap = kg >= 4;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int n = 16 * w + 4 * ng + i;   // the row within the warpgroup's 64
      const uint32_t a = dst + wg * (64 * 128) + n * 128 + ((kg ^ (n & 7)) << 4);
      const uint32_t v0 = swap ? o[i][1] : o[i][0], v1 = swap ? o[i][0] : o[i][1];
      const uint32_t v2 = swap ? o[i][3] : o[i][2], v3 = swap ? o[i][2] : o[i][3];
      asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(v0), "r"(v1), "r"(v2), "r"(v3) : "memory");
    }
  }
};

// Blockwise e4m3 (Float8DynamicActivationFloat8WeightConfig with PerBlock([1, 128]) activations and PerBlock([128,
// 128]) weights; reference float8_tensor.py:431-447 and its Triton loop, kernels.py:86-97): the operands, wgmmas and
// per-chunk promotion of SsFmt<KIND_F8>.  A tile is 128 weight rows and a chunk 128 k, i.e. exactly one weight block
// and one activation block per token, so each chunk's partial is scaled as it is promoted, in the loop's order:
//   acc = fma(part * a_s[m][kc], w_s[n_tile][kc], acc)      (acc = 0 before a segment's first chunk)
// The multiply-add is fused (what Triton's default fp-fusion contracts `acc += dot * a_s * w_s` to).  The epilogue is
// EPI_BF16: bf16(acc), then a bf16 add of the bias.  Stream-K partials are such scaled sums and are gathered in the
// fixed CTA order as for every format.
// Scales: w_s from w_scale [N/128][K/128] (Params::w_scale), one value per chunk read by every thread; a_s from the
// transposed activation scales [K/128][ldm] (ldm = M rounded up to 4, ao_fp8_quantize_1x128): one 256-byte TMA box of
// 64 tokens per chunk, requested with the activation tile into the stage's aux slot (the 64-token box serves every
// token tile: tokens past the tile or past M are never stored).
struct BlockwiseF8Fmt : SsFmt<KIND_F8> {
  static constexpr int X_AUX_BYTES = MAX_N_MMA * 4;
  static constexpr int AUX_BYTES = X_AUX_BYTES;
  static constexpr int EPI = tsg::EPI_BF16;
  static int make_maps(const uint8_t* wq, const float* x_scale_t, int M, int N, int K, CUtensorMap* tm_w,
                       CUtensorMap* tm_xs) {
    if (int rc = kmajor_byte_map(wq, N, K, tm_w)) return rc;
    return scale_map(x_scale_t, M, K, MAX_N_MMA, tm_xs);
  }
  // the transposed token scales [K/128][round_up(M, 4)], one box of `tokens` scales of one chunk
  static int scale_map(const float* x_scale_t, int M, int K, uint32_t tokens, CUtensorMap* tm_xs) {
    const uint64_t ldm = ((uint64_t)M + 3) & ~3ull;
    const uint64_t dims[2] = {ldm, (uint64_t)K / KCHUNK};
    const uint64_t str[1] = {ldm * 4};
    const uint32_t box[2] = {tokens, 1};
    return make_tmap(tm_xs, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, x_scale_t, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE);
  }
  __device__ static __forceinline__ void issue_x_aux(const CUtensorMap* tm_xs, uint8_t* aux_dst, uint64_t* bar, int m0,
                                                     int kc, uint64_t policy) {
    tma_load_2d(aux_dst, tm_xs, bar, m0, kc, policy);
  }
  // the weight block's scale and the activation scales of the thread's tokens 8q + 2t, + 1 (accumulator value
  // 4q + 2h + c is token 8q + 2t + c)
  template <int N_MMA>
  struct Scales {
    float w;
    float2 a[N_MMA / 8];
  };
  template <int N_MMA>
  __device__ static __forceinline__ Scales<N_MMA> chunk_scales(const tsg::Params& p, uint32_t aux_s, int w_blk, int,
                                                               int kc, int lane) {
    Scales<N_MMA> cs;
    cs.w = p.w_scale[(size_t)w_blk * p.KT + kc];
    const uint32_t t = lane & 3;
#pragma unroll
    for (int q = 0; q < N_MMA / 8; ++q) {
      const uint2 v = tsg::lds64(aux_s + (8 * q + 2 * t) * 4);
      cs.a[q] = make_float2(__uint_as_float(v.x), __uint_as_float(v.y));
    }
    return cs;
  }
  template <int N_MMA>
  __device__ static __forceinline__ void promote(uint32_t (&acc)[N_MMA / 2], const uint32_t (&part)[N_MMA / 2],
                                                 uint32_t accumulate, const Scales<N_MMA>& cs) {
#pragma unroll
    for (int j = 0; j < N_MMA / 2; ++j) {
      const float a = (j & 1) ? cs.a[j / 4].y : cs.a[j / 4].x;
      const float prev = accumulate ? __uint_as_float(acc[j]) : 0.f;
      acc[j] = __float_as_uint(__fmaf_rn(__fmul_rn(__uint_as_float(part[j]), a), cs.w, prev));
    }
  }
};

// Blockwise e4m3 under the grouped schedule (torch._grouped_mm on [E, N, K] experts, ts_gemm_kernel<Grouped<...>>): the
// weights come from SsFmt::issue_w_rows, row e*N + 128t of the [E*N, K] map; the scales [E, N/128, K/128] are
// [E*N/128][KT], indexed by the block e*(N/128) + t the kernel passes (W_BLOCK_SCALES).  A tile starts at its expert's
// first row, any row, and a TMA box whose first element is off a 16-byte boundary faulted on the H100 (an illegal
// instruction; DESIGN §2a): the token scale box starts at row0 & ~3, 4 scales before the tile at most, and holds
// MAX_N_MMA + 4 scales, read from row0 & 3 on.  Rows of other experts in it are never stored.
struct BlockwiseF8GroupedFmt : BlockwiseF8Fmt {
  static constexpr int X_AUX_BYTES = (MAX_N_MMA + 4) * 4;
  static constexpr int AUX_BYTES = X_AUX_BYTES;
  static constexpr bool W_BLOCK_SCALES = true;
  static int make_maps(const uint8_t* wq, const float* x_scale_t, int M, int N, int K, CUtensorMap* tm_w,
                       CUtensorMap* tm_xs) {
    if (int rc = kmajor_byte_map(wq, N, K, tm_w)) return rc;
    return scale_map(x_scale_t, M, K, MAX_N_MMA + 4, tm_xs);
  }
  __device__ static __forceinline__ void issue_x_aux(const CUtensorMap* tm_xs, uint8_t* aux_dst, uint64_t* bar, int m0,
                                                     int kc, uint64_t policy) {
    tma_load_2d(aux_dst, tm_xs, bar, m0 & ~3, kc, policy);
  }
  template <int N_MMA>
  __device__ static __forceinline__ Scales<N_MMA> chunk_scales(const tsg::Params& p, uint32_t aux_s, int w_blk, int m0,
                                                               int kc, int lane) {
    Scales<N_MMA> cs;
    cs.w = p.w_scale[(size_t)w_blk * p.KT + kc];
    const uint32_t base = aux_s + (uint32_t)((m0 & 3) + 2 * (lane & 3)) * 4;   // 4-byte aligned only: two 32-bit loads
#pragma unroll
    for (int q = 0; q < N_MMA / 8; ++q)
      cs.a[q] = make_float2(__uint_as_float(tsg::lds32(base + 32 * q)), __uint_as_float(tsg::lds32(base + 32 * q + 4)));
    return cs;
  }
};

// 2:4-sparse e4m3 (Float8DynamicActivationFloat8WeightConfig with packing_format SPARSE_2D_DATA_2D_METADATA; reference
// float8_sparse_2x4_2d_data_2d_metadata_tensor.py and its CUTLASS GEMM rowwise_scaled_linear_sparse_cutlass.cuh).
// Weights: the compressed codes wq [N][K/2] (each 4-k group keeps its two stored codes) and the metadata wm as CUTLASS's
// Sm90 sparse compressor writes it: atoms of 64 rows x 128 k, 16 bytes per row (one 4-bit nibble per 4-k group, the
// two kept positions in bits 1:0 and 3:2), atoms along N first, then along K, so that the metadata of column block kc
// starts at byte kc * round_up(N, 64) * 16 and a tile's two atoms are 2 KiB in a row.
// Per 128-k chunk a stage holds the tile's compressed codes (128 rows x 64 bytes, 64-byte swizzle), its two metadata
// atoms in the aux slot (one 2 KiB box of 8-byte words; past round_up(N, 64) zero-filled) and the e4m3 activation tile.
// MMA: two wgmma.sp k64 per chunk.  PTX ISA, sparse wgmma metadata for 8-bit types: thread (warp w, lane l) of the
// warpgroup supplies the 32 k of row 16w + l/4 + 8(l%2), k 32((l/2)%2) .. + 31 of the k64 step, group j at bits 4j+3:4j.
// The chunks of a segment accumulate in the wgmma accumulator (the reference's FP8FastAccum mainloop: no promotion),
// each chunk's wgmmas completing before the next chunk's are issued (ts_gemm.cuh), and the epilogue is EPI_F8_SPARSE.
// Metadata nibbles 0b0000, 0b0101, 0b1010, 0b1111 (both positions equal) are undefined behaviour for the MMA.  The
// reference's compressor writes 0b0000 for an all-zero group and for its padding, and its allocation leaves any bytes
// it did not write as they were, so meta() replaces every word of rows >= N or k >= K by 0x44444444 (positions 0, 1)
// and every 0b0000 nibble by 0b0100.  A 0b0000 group's two stored codes are zero, so the product is unchanged.
struct SparseF8Fmt {
  static constexpr bool SS = true;
  static constexpr bool SPARSE_A = true;
  static constexpr bool PROMOTE = false;
  static constexpr bool DECODE_2CTA = true;
  static constexpr int X_ELEM_BYTES = 1;
  static constexpr int W_BYTES = ROWS * KCHUNK / 2;   // 8 KiB of compressed codes
  static constexpr int META_BYTES = 2 * 64 * 16;      // two metadata atoms
  static constexpr int AUX_BYTES = META_BYTES;
  static constexpr int EPI = tsg::EPI_F8_SPARSE;
  static constexpr int ACC_EXP2 = 0;
  static constexpr int MAX_N_MMA = 128;
  static int make_maps(const uint8_t* wq, const uint8_t* wm, int N, int K, CUtensorMap* tm_w, CUtensorMap* tm_m) {
    {
      const uint64_t dims[2] = {(uint64_t)K / 2, (uint64_t)N};
      const uint64_t str[1] = {(uint64_t)K / 2};
      const uint32_t box[2] = {64, ROWS};
      if (int rc = make_tmap(tm_w, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, wq, dims, str, box, CU_TENSOR_MAP_SWIZZLE_64B))
        return rc;
    }
    // [KT][round_up(N, 64) * 16 bytes] as 8-byte words, one box = one tile's two atoms
    const uint64_t row_words = (uint64_t)ceil_div(N, 64) * 64 * 16 / 8;
    const uint64_t dims[2] = {row_words, (uint64_t)ceil_div(K, KCHUNK)};
    const uint64_t str[1] = {row_words * 8};
    const uint32_t box[2] = {META_BYTES / 8, 1};
    return make_tmap(tm_m, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, wm, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE);
  }
  __device__ static __forceinline__ uint32_t w_tx_bytes(const tsg::Params&) { return W_BYTES + META_BYTES; }
  __device__ static __forceinline__ void issue_w(const CUtensorMap* tm_w, const CUtensorMap* tm_m, const tsg::Params&,
                                                 uint8_t* w_dst, uint8_t* aux_dst, uint64_t* bar, int n_tile, int kc,
                                                 uint64_t policy) {
    tma_load_2d(w_dst, tm_w, bar, kc * (KCHUNK / 2), n_tile * ROWS, policy);
    tma_load_2d(aux_dst, tm_m, bar, n_tile * (META_BYTES / 8), kc, policy);
  }
  // valid words as they are except 0b0000 nibbles -> 0b0100; words of rows >= N or k >= K: 0x44444444
  __device__ static __forceinline__ uint32_t sanitize(uint32_t w, bool valid) {
    w = valid ? w : 0x44444444u;
    uint32_t z = w | (w >> 1);
    z |= z >> 2;
    return w | ((~z & 0x11111111u) << 2);
  }
  // the thread's metadata words of k64 steps 0 and 1 (row: its metadata row 0..127 of the tile)
  __device__ static __forceinline__ uint2 meta(const tsg::Params& p, uint32_t aux_s, int n_tile, int kc, int row,
                                               int lane) {
    const int half = (lane >> 1) & 1;
    const uint32_t a = aux_s + (uint32_t)(row >> 6) * 1024u + (uint32_t)(row & 63) * 16u + 4u * half;
    const bool row_ok = n_tile * ROWS + row < p.N;
    const int k0 = kc * KCHUNK + 32 * half;
    return make_uint2(sanitize(tsg::lds32(a), row_ok && k0 < p.K), sanitize(tsg::lds32(a + 8), row_ok && k0 + 64 < p.K));
  }
  template <int N_MMA>
  __device__ static __forceinline__ void mma(uint32_t (&acc)[N_MMA / 2], uint32_t w_s, uint32_t x_s,
                                             const uint32_t (&mt)[2], int wg, uint32_t scale_d) {
    // k64 step j: 32 bytes of each compressed row, 64 bytes of each activation row
    Wgmma<N_MMA>::sp_e4m3(acc, wgmma_desc_k_sw64(w_s + wg * (64 * 64)), wgmma_desc_k_sw128(x_s), mt[0], scale_d);
    Wgmma<N_MMA>::sp_e4m3(acc, wgmma_desc_k_sw64(w_s + wg * (64 * 64) + 32), wgmma_desc_k_sw128(x_s + 64), mt[1], 1u);
  }
};

// the blocked e8m0 scales of block-32 weights W[N][K] as a 2-D tensor of 128 words x 512-byte tiles, one tile (4
// scales x 128 rows = 128 k) per box
static int e8m0_tile_map(const uint8_t* w_sf, int N, int K, CUtensorMap* tm_sf) {
  const uint64_t dims[2] = {128, (uint64_t)ceil_div(N, ROWS) * (uint64_t)ceil_div(K / 32, 4)};
  const uint64_t str[1] = {512};
  const uint32_t box[2] = {128, 1};
  return make_tmap(tm_sf, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, w_sf, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE);
}

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
  static constexpr bool EXPERT_SCALE = false;   // grouped: y = acc, the dense MX epilogue without bias
  // the weights and the blocked scale tiles, one 512-byte tile per box
  static int make_maps(const uint8_t* wq, const uint8_t* w_sf, int N, int K, CUtensorMap* tm_w, CUtensorMap* tm_sf) {
    if (int rc = kmajor_byte_map(wq, N, K, tm_w)) return rc;
    return e8m0_tile_map(w_sf, N, K, tm_sf);
  }
  __device__ static __forceinline__ uint32_t w_tx_bytes(const tsg::Params&) { return W_BYTES + AUX_BYTES; }
  __device__ static __forceinline__ void issue_w(const CUtensorMap* tm_w, const CUtensorMap* tm_sf, const tsg::Params& p,
                                                 uint8_t* w_dst, uint8_t* aux_dst, uint64_t* bar, int n_tile, int kc,
                                                 uint64_t policy) {
    tma_load_2d(w_dst, tm_w, bar, kc * KCHUNK, n_tile * ROWS, policy);
    tma_load_2d(aux_dst, tm_sf, bar, 0, n_tile * p.aux_col_blocks + kc, policy);
  }
  // grouped kernels: the 128 weight rows from `row` = e*N + 128t of the [E * N, K] map of all experts' weights, and
  // their scale tile at row block row / 128 of the blocked [E * N, K / 32] scales.  The launcher requires N % 128 == 0,
  // which keeps every expert's weights and scales in whole 128-row blocks, so no tile has a tail (Nvfp4Fmt::issue_w_rows)
  __device__ static __forceinline__ void issue_w_rows(const CUtensorMap* tm_w, const CUtensorMap* tm_sf,
                                                      const tsg::Params& p, uint8_t* w_dst, uint8_t* aux_dst,
                                                      uint64_t* bar, int row, int kc, uint64_t policy) {
    tma_load_2d(w_dst, tm_w, bar, kc * KCHUNK, row, policy);
    tma_load_2d(aux_dst, tm_sf, bar, 0, (row / ROWS) * p.aux_col_blocks + kc, policy);
  }
  // the thread's two fragment rows: for k16 step kk the e4m3 pair at k 16kk + 2t (low half) and + 8 (high half)
  struct Raw {
    uint32_t v[2][8];
    uint32_t sc[2];
  };
  // row r's e4m3 pairs of k16 step kk: k 16kk + 2t, + 1 at bits 15:0 and k 16kk + 2t + 8, + 9 at bits 31:16
  __device__ static __forceinline__ uint32_t lds_pairs(uint32_t w_smem, int r, int kk, int t) {
    const uint32_t a = w_smem + (uint32_t)r * 128u + ((uint32_t)(kk ^ (r & 7)) << 4) + 2 * t;   // TMA 128B swizzle
    return tsg::lds16(a) | (tsg::lds16(a + 8) << 16);
  }
  __device__ static __forceinline__ void load(const tsg::Params&, uint32_t w_smem, uint32_t aux_smem, int row_lo, int lane,
                                              Raw& raw) {
    const int t = lane & 3;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = row_lo + 8 * h;
      raw.sc[h] = tsg::lds32(aux_smem + (uint32_t)(r & 31) * 16u + (uint32_t)(r >> 5) * 4u);
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) raw.v[h][kk] = lds_pairs(w_smem, r, kk, t);
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

// mxfp4 weights as the register-A operand: packed e2m1 pairs (the stored [N, K/2] qdata, even k in the low nibble,
// loaded as nvf4w::Nvfp4Fmt loads them) x their block-32 e8m0 scale (one blocked tile per chunk, as Mxfp8Fmt) -> bf16.
// A nibble placed at bf16 bits 15|8:6 is value * 2^-126 (Nvfp4Fmt::deq); one exact multiply by 2^126 gives the value and
// a second one by the bf16 scale 2^(e-127) the element, exact for every byte (see the top of this file): the e8m0
// range is the bf16 exponent range, 2^-127 a bf16 subnormal, and bf16 multiplies keep subnormals.  The scales are
// decoded once per chunk; the thread keeps only the 16 code bytes of its two fragment rows that its steps read.
struct Mxfp4Fmt {
  static constexpr bool SS = false;
  // at 80 registers (two CTAs per SM) the N_MMA = 32 decode tile keeps 8 bytes of stack, a spill and refill in every
  // chunk: one CTA per SM, as mxfp8 and nvfp4 (DESIGN.md, mxfp4)
  static constexpr bool DECODE_2CTA = false;
  static constexpr bool PROMOTE = false;
  static constexpr int X_ELEM_BYTES = 2;
  static constexpr int W_BYTES = ROWS * KCHUNK / 2;   // 128 rows x 64 bytes, 64-byte swizzle
  static constexpr int AUX_BYTES = 512;               // one blocked scale tile (4 scales = 128 k per row)
  static constexpr int EPI = tsg::EPI_FLOAT;
  static constexpr int ACC_EXP2 = 0;
  static constexpr int MAX_N_MMA = 128;
  static constexpr bool EXPERT_SCALE = false;   // grouped: y = acc, the dense MX epilogue without bias
  static int make_maps(const uint8_t* wq, const uint8_t* w_sf, int N, int K, CUtensorMap* tm_w, CUtensorMap* tm_sf) {
    const uint64_t dims[2] = {(uint64_t)K / 2, (uint64_t)N};
    const uint64_t str[1] = {(uint64_t)K / 2};
    const uint32_t box[2] = {64, 128};
    if (int rc = make_tmap(tm_w, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, wq, dims, str, box, CU_TENSOR_MAP_SWIZZLE_64B))
      return rc;
    return e8m0_tile_map(w_sf, N, K, tm_sf);
  }
  __device__ static __forceinline__ uint32_t w_tx_bytes(const tsg::Params&) { return W_BYTES + AUX_BYTES; }
  __device__ static __forceinline__ void issue_w(const CUtensorMap* tm_w, const CUtensorMap* tm_sf, const tsg::Params& p,
                                                 uint8_t* w_dst, uint8_t* aux_dst, uint64_t* bar, int n_tile, int kc,
                                                 uint64_t policy) {
    tma_load_2d(w_dst, tm_w, bar, kc * 64, n_tile * ROWS, policy);
    tma_load_2d(aux_dst, tm_sf, bar, 0, n_tile * p.aux_col_blocks + kc, policy);
  }
  // grouped kernels: Mxfp8Fmt::issue_w_rows on the [E * N, K / 2] map of all experts' packed weights
  __device__ static __forceinline__ void issue_w_rows(const CUtensorMap* tm_w, const CUtensorMap* tm_sf,
                                                      const tsg::Params& p, uint8_t* w_dst, uint8_t* aux_dst,
                                                      uint64_t* bar, int row, int kc, uint64_t policy) {
    tma_load_2d(w_dst, tm_w, bar, kc * 64, row, policy);
    tma_load_2d(aux_dst, tm_sf, bar, 0, (row / ROWS) * p.aux_col_blocks + kc, policy);
  }
  // c[h][j]: row h's code bytes of k16 steps 2j, 2j + 1 (step kk reads byte t of bytes 8kk..8kk+3, the k pair
  // 16kk + 2t, and byte t of 8kk+4..8kk+7, the pair 8 further), as bytes (2j lo, 2j hi, 2j+1 lo, 2j+1 hi);
  // s[h][i]: bf16x2 of the scales of 32-k blocks 2i, 2i + 1
  struct Raw {
    uint32_t c[2][4];
    uint32_t s[2][2];
  };
  // Raw::c[h][j] of row r from the 64-byte-swizzled stage (the byte selector sel of thread t, see load)
  __device__ static __forceinline__ uint32_t lds_codes(uint32_t w_smem, int r, int j, uint32_t sel) {
    const uint32_t off = (uint32_t)r * 64u + j * 16;
    const uint4 v = tsg::lds128(w_smem + (off ^ (((off >> 7) & 3) << 4)));   // undo the TMA 64B swizzle
    return __byte_perm(__byte_perm(v.x, v.y, sel), __byte_perm(v.z, v.w, sel), 0x5410);
  }
  __device__ static __forceinline__ void load(const tsg::Params&, uint32_t w_smem, uint32_t aux_smem, int row_lo, int lane,
                                              Raw& raw) {
    const uint32_t t = lane & 3;
    const uint32_t sel = t | (t + 4) << 4 | t << 8 | (t + 4) << 12;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = row_lo + 8 * h;
      const uint32_t sc = tsg::lds32(aux_smem + (uint32_t)(r & 31) * 16u + (uint32_t)(r >> 5) * 4u);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const __nv_bfloat162 s2 = __floats2bfloat162_rn(e8m0_to_f32((sc >> (16 * i)) & 0xFFu),
                                                        e8m0_to_f32((sc >> (16 * i + 8)) & 0xFFu));
        raw.s[h][i] = *reinterpret_cast<const uint32_t*>(&s2);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) raw.c[h][j] = lds_codes(w_smem, r, j, sel);
    }
  }
  __device__ static __forceinline__ uint32_t deq(uint32_t byte, __nv_bfloat162 s2) {
    const uint32_t hh = (byte | (byte << 12)) & 0x000F000Fu;   // even k nibble at bits 3:0, odd k at 19:16
    const uint32_t bits = (hh * 0x1040u) & 0x81C081C0u;         // sign | e1 e0 m at bf16 bits 15 | 8:6 = value * 2^-126
    __nv_bfloat162 x = *reinterpret_cast<const __nv_bfloat162*>(&bits);
    x = __hmul2(__hmul2(x, __nv_bfloat162(__ushort_as_bfloat16(0x7E80), __ushort_as_bfloat16(0x7E80))), s2);   // * 2^126
    return *reinterpret_cast<uint32_t*>(&x);
  }
  __device__ static __forceinline__ void frag(const tsg::Params&, const Raw& raw, int kk, uint32_t (&a)[4]) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      // the scale of the 32-k block of step kk, in both halves
      const uint32_t s_bits = __byte_perm(raw.s[h][kk >> 2], 0u, ((kk >> 1) & 1) ? 0x3232u : 0x1010u);
      const __nv_bfloat162 s2 = *reinterpret_cast<const __nv_bfloat162*>(&s_bits);
      const uint32_t cw = raw.c[h][kk >> 1] >> (16 * (kk & 1));
      a[h] = deq(cw & 0xFFu, s2);
      a[h + 2] = deq((cw >> 8) & 0xFFu, s2);
    }
  }
};

// int8 weights x bf16 activations (Int8WeightOnlyConfig; reference int8_tensor.py:336-359, per-row and per-tensor
// scales): the stored [N, K] qdata in the stage and map of SsFmt<KIND_I8>, each byte converted exactly to bf16 in the
// register-A fragment.  The scale stays out of the K loop: bf16 x int8 products are exact in fp32, and the epilogue
// (EPI_BF16_WSCALE) applies the reference's three roundings.
// Conversion: a byte b of two's complement q gives bf16 0x4300 | (b & 0x7F) = 128 + (b & 0x7F) and
// 0x4300 | (b & 0x80) = 128 (q >= 0) or 256 (q < 0); their difference is q, exact (|q| <= 128 has 8 significant bits).
struct Int8WoFmt {
  static constexpr bool SS = false;
  // ptxas, sm_90a: no stack at 80 registers for the 16- and 32-token tiles (DESIGN.md §2c)
  static constexpr bool DECODE_2CTA = true;
  static constexpr bool PROMOTE = false;
  static constexpr int X_ELEM_BYTES = 2;
  static constexpr int W_BYTES = ROWS * KCHUNK;   // 128 rows x 128 bytes, 128-byte swizzle
  static constexpr int AUX_BYTES = 0;
  static constexpr int EPI = tsg::EPI_BF16_WSCALE;
  static constexpr int ACC_EXP2 = 0;
  static constexpr int MAX_N_MMA = 128;
  // no aux operand: the weight map stands in for it (see SsFmt)
  static int make_maps(const uint8_t* wq, int N, int K, CUtensorMap* tm_w, CUtensorMap* tm_aux) {
    return SsFmt<KIND_I8>::make_maps(wq, N, K, tm_w, tm_aux);
  }
  __device__ static __forceinline__ uint32_t w_tx_bytes(const tsg::Params&) { return W_BYTES; }
  __device__ static __forceinline__ void issue_w(const CUtensorMap* tm_w, const CUtensorMap*, const tsg::Params&,
                                                 uint8_t* w_dst, uint8_t*, uint64_t* bar, int n_tile, int kc,
                                                 uint64_t policy) {
    tma_load_2d(w_dst, tm_w, bar, kc * KCHUNK, n_tile * ROWS, policy);
  }
  // grouped kernels: 128 rows from `row` = e*N + 128t of the [E * N, K] map of all experts' weights.  No aux box: the
  // EPI_BF16_WSCALE epilogue reads w_scale[e*N + n] itself, so N needs no alignment.  A tile past N reads the next
  // expert's rows (or the map's zero fill); each output row depends on its own weight row only, and the epilogue skips
  // the features >= N
  __device__ static __forceinline__ void issue_w_rows(const CUtensorMap* tm_w, const CUtensorMap*, const tsg::Params&,
                                                      uint8_t* w_dst, uint8_t*, uint64_t* bar, int row, int kc,
                                                      uint64_t policy) {
    tma_load_2d(w_dst, tm_w, bar, kc * KCHUNK, row, policy);
  }
  // the thread's two fragment rows: for k16 step kk the bytes of k 16kk + 2t + (0, 8, 1, 9), so that each bf16x2 lane
  // finds its byte at its own bits 7:0 (k 2t, 2t + 1) or 15:8 (k 2t + 8, 2t + 9)
  struct Raw {
    uint32_t v[2][8];
  };
  __device__ static __forceinline__ void load(const tsg::Params&, uint32_t w_smem, uint32_t, int row_lo, int lane,
                                              Raw& raw) {
    const int t = lane & 3;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = row_lo + 8 * h;
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        const uint32_t a = w_smem + (uint32_t)r * 128u + ((uint32_t)(kk ^ (r & 7)) << 4) + 2 * t;   // TMA 128B swizzle
        raw.v[h][kk] = __byte_perm(tsg::lds16(a), tsg::lds16(a + 8), 0x5140);
      }
    }
  }
  // bf16x2 of the int8 at bits 7:0 of each 16-bit lane (the other bits are ignored)
  __device__ static __forceinline__ uint32_t cvt(uint32_t w, uint32_t magic) {
    uint32_t v, c;
    asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(v) : "r"(w), "r"(0x007F007Fu), "r"(magic));   // (w & mask) | magic
    asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(c) : "r"(w), "r"(0x00800080u), "r"(magic));
    const __nv_bfloat162 d = __hsub2(*reinterpret_cast<const __nv_bfloat162*>(&v), *reinterpret_cast<const __nv_bfloat162*>(&c));
    return *reinterpret_cast<const uint32_t*>(&d);
  }
  __device__ static __forceinline__ void frag(const tsg::Params&, const Raw& raw, int kk, uint32_t (&a)[4]) {
    uint32_t magic = 0x43004300u;
    asm volatile("" : "+r"(magic));   // keep it in a register
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      a[h] = cvt(raw.v[h][kk], magic);
      a[h + 2] = cvt(raw.v[h][kk] >> 8, magic);
    }
  }
};

// e4m3 weights x bf16 activations (Float8WeightOnlyConfig; reference float8_tensor.py:459-469, per-row and per-tensor
// scales): the stored [N, K] qdata in the stage and map of Mxfp8Fmt, plus the tile's 128 fp32 row scales, one 512-byte
// TMA box of w_scale [N] per chunk (rows past N zero-filled).  The reference dequantizes before the matmul,
// w~ = bf16(fp32(e4m3(q) * s)): an e4m3 code has 4 significant bits and a bf16 scale 8, so the product rounds per
// element and the scale cannot leave the K loop.  Each element is Mxfp8Fmt::deq with the row's fp32 scale in place of
// the block's power of two (e4m3 -> half -> fp32 exactly, one fp32 multiply, one bf16 rounding; the build has no
// flush-to-zero, so subnormal products stay), every bf16 x w~ product is exact in fp32, and the epilogue (EPI_BF16)
// rounds the sum to bf16 and adds the bias in bf16, as torch.matmul and `+ bias` do.
struct Fp8WoFmt {
  static constexpr bool SS = false;
  // ptxas, sm_90a: at 80 registers (two CTAs per SM) the N_MMA = 32 tile keeps 8 bytes of stack: one CTA per SM, as
  // mxfp8 (DESIGN.md §2d)
  static constexpr bool DECODE_2CTA = false;
  static constexpr bool PROMOTE = false;
  static constexpr int X_ELEM_BYTES = 2;
  static constexpr int W_BYTES = ROWS * KCHUNK;   // 128 rows x 128 bytes, 128-byte swizzle
  static constexpr int AUX_BYTES = ROWS * 4;      // the tile's fp32 row scales
  static constexpr int EPI = tsg::EPI_BF16;
  static constexpr int ACC_EXP2 = 0;
  static constexpr int MAX_N_MMA = 128;
  static int make_maps(const uint8_t* wq, const float* w_scale, int N, int K, CUtensorMap* tm_w, CUtensorMap* tm_s) {
    if (int rc = kmajor_byte_map(wq, N, K, tm_w)) return rc;
    const uint64_t dims[1] = {(uint64_t)N};
    const uint32_t box[1] = {ROWS};
    return make_tmap(tm_s, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 1, w_scale, dims, nullptr, box, CU_TENSOR_MAP_SWIZZLE_NONE);
  }
  __device__ static __forceinline__ uint32_t w_tx_bytes(const tsg::Params&) { return W_BYTES + AUX_BYTES; }
  __device__ static __forceinline__ void issue_w(const CUtensorMap* tm_w, const CUtensorMap* tm_s, const tsg::Params&,
                                                 uint8_t* w_dst, uint8_t* aux_dst, uint64_t* bar, int n_tile, int kc,
                                                 uint64_t policy) {
    tma_load_2d(w_dst, tm_w, bar, kc * KCHUNK, n_tile * ROWS, policy);
    tma_load_1d(aux_dst, tm_s, bar, n_tile * ROWS, policy);
  }
  // grouped kernels: the 128 weight rows from `row` = e*N + 128t of the [E * N, K] map and their scales, the 512-byte
  // box from element `row` of the 1-D map over w_scale [E * N] (N % 8 == 0: a box that started off a 16-byte boundary
  // of w_scale faulted on the H100).  A tile past N reads the next expert's rows and scales, or the maps' zero fill
  // after the last expert; each output row depends on its own weight row only, and the epilogue skips the features >= N
  __device__ static __forceinline__ void issue_w_rows(const CUtensorMap* tm_w, const CUtensorMap* tm_s,
                                                      const tsg::Params&, uint8_t* w_dst, uint8_t* aux_dst,
                                                      uint64_t* bar, int row, int kc, uint64_t policy) {
    tma_load_2d(w_dst, tm_w, bar, kc * KCHUNK, row, policy);
    tma_load_1d(aux_dst, tm_s, bar, row, policy);
  }
  // the pairs of Mxfp8Fmt::Raw and the scales of the thread's two fragment rows
  struct Raw {
    uint32_t v[2][8];
    float s[2];
  };
  __device__ static __forceinline__ void load(const tsg::Params&, uint32_t w_smem, uint32_t aux_smem, int row_lo, int lane,
                                              Raw& raw) {
    const int t = lane & 3;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = row_lo + 8 * h;
      raw.s[h] = __uint_as_float(tsg::lds32(aux_smem + (uint32_t)r * 4u));
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) raw.v[h][kk] = Mxfp8Fmt::lds_pairs(w_smem, r, kk, t);
    }
  }
  __device__ static __forceinline__ void frag(const tsg::Params&, const Raw& raw, int kk, uint32_t (&a)[4]) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      a[h] = Mxfp8Fmt::deq(raw.v[h][kk] & 0xFFFFu, raw.s[h]);
      a[h + 2] = Mxfp8Fmt::deq(raw.v[h][kk] >> 16, raw.s[h]);
    }
  }
};

// NF4 weights x bf16 activations (NF4Tensor, QLoRA; reference nf4_tensor.py get_original_weight and LinearNF4): the
// stored codes [N*K/2] viewed as [N, K/2] bytes (even k in the high nibble) in the stage and map of Mxfp4Fmt, and per
// flat block b = (n*K + k) / block_size the double-quantized scaler
//   s[b] = bf16(bf16(qs[b] / f[b / sbs]) + mean),  w~[n,k] = bf16(nf4[code] * s[b])
// with qs int8, f, mean and the 16-entry table nf4 bf16 tensors of the weight.  The scalers are decoded in the GEMM, by
// the aux fillers of ts_gemm.cuh (AUX_FILL): one chunk's scaler bytes are 2 per row at block_size 64, under TMA's
// 16-byte box minimum, and their row pitch K / block_size is a multiple of 16 bytes only when K % 1024 == 0.  A filler
// warp reads them with ordinary loads (each block once), divides as torch does (IEEE division, then a separate add) and
// writes one bf16 scaler per (row, k16 step) into the stage's aux slot, with the table behind them.
// Conversion: the four codes of a thread's 16-bit code word select their table entries with byte permutes, the low and
// the high bytes of the bf16 values separately (entries 0..7 and 8..15, then bit 3 of the code picks one), and one bf16x2
// multiply by the step's scaler rounds each element once, as torch's bf16 multiply does.  Every bf16 x w~ product is exact
// in fp32, and the epilogue (EPI_BF16) rounds the sum to bf16 and adds the bias in bf16, as F.linear and `+ bias` do.
// Params: the fields its EPI_BF16 epilogue never reads carry the NF4 tensors, so Params (and the code of every other
// kernel) stays as it is: row_scale = quantized_scalers (int8), out_scale = quantization_factor (bf16), out_scale2 =
// scaler_mean (bf16), w_scale = nf4 (bf16), group_size = block_size, aux_col_blocks = scaler_block_size.
// Shapes: block_size % 16 == 0 (a k16 step lies in one block), K % block_size == 0 (no block spans two rows; then every
// row has its block boundaries at the same k), K % 32 == 0 (the TMA row pitch of the codes), any N.
struct Nf4Fmt {
  static constexpr bool SS = false;
  // one CTA per SM: the aux fillers hold a chunk's loads in registers (ts_gemm.cuh, AuxFill)
  static constexpr bool DECODE_2CTA = false;
  static constexpr bool PROMOTE = false;
  static constexpr bool AUX_FILL = true;
  static constexpr int X_ELEM_BYTES = 2;
  static constexpr int W_BYTES = ROWS * KCHUNK / 2;   // 128 rows x 64 bytes, 64-byte swizzle
  // the scalers [128 rows][8 k16 steps] bf16, then the table as byte planes: words 0..3 the low bytes of entries 0..15,
  // words 4..7 their high bytes
  static constexpr int LUT_OFF = ROWS * 16;
  static constexpr int AUX_BYTES = LUT_OFF + 32;
  static constexpr int EPI = tsg::EPI_BF16;
  static constexpr int ACC_EXP2 = 0;
  static constexpr int MAX_N_MMA = 128;
  // no aux map: the weight map stands in for it (the aux slot is written by the fillers)
  static int make_maps(const uint8_t* qdata, int N, int K, CUtensorMap* tm_w, CUtensorMap* tm_aux) {
    const uint64_t dims[2] = {(uint64_t)K / 2, (uint64_t)N};
    const uint64_t str[1] = {(uint64_t)K / 2};
    const uint32_t box[2] = {64, 128};
    if (int rc = make_tmap(tm_w, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, qdata, dims, str, box, CU_TENSOR_MAP_SWIZZLE_64B))
      return rc;
    *tm_aux = *tm_w;
    return AO_OK;
  }
  __device__ static __forceinline__ uint32_t w_tx_bytes(const tsg::Params&) { return W_BYTES; }
  __device__ static __forceinline__ void issue_w(const CUtensorMap* tm_w, const CUtensorMap*, const tsg::Params&,
                                                 uint8_t* w_dst, uint8_t*, uint64_t* bar, int n_tile, int kc,
                                                 uint64_t policy) {
    tma_load_2d(w_dst, tm_w, bar, kc * 64, n_tile * ROWS, policy);
  }
  // the reference's dequantize_scalers: an int8 / bf16 division rounded to bf16, then a bf16 add of the mean
  __device__ static __forceinline__ uint32_t scaler_bits(int8_t q, __nv_bfloat16 f, float mean) {
    const float d = __bfloat162float(__float2bfloat16_rn(__fdiv_rn((float)q, __bfloat162float(f))));
    return __bfloat16_as_ushort(__float2bfloat16_rn(__fadd_rn(d, mean)));
  }
  // one warp: the aux slot of chunk kc of tile n_tile; lane l writes rows l, l + 32, l + 64, l + 96
  __device__ static __forceinline__ void fill_aux(const tsg::Params& p, uint8_t* aux, int n_tile, int kc, int lane) {
    const int bs = p.group_size, k0 = kc * KCHUNK;
    const uint32_t per_row = (uint32_t)(p.K / bs), o0 = (uint32_t)(k0 / bs), sbs = (uint32_t)p.aux_col_blocks;
    // step kk lies in block o0 + ob[kk] of its row and starts a block (fresh) at kk == 0 and where k0 + 16kk is a
    // multiple of bs.  Steps past K get the scaler 0: their codes are TMA zero fill (code 0 = -1), and a 0 keeps them
    // out of the sums even in a row whose scalers are inf or NaN
    int ob[8];
    bool fresh[8], in_k[8];
    {
      int o = 0, pos = k0 - (int)o0 * bs;
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        if (kk > 0 && (pos += 16) == bs) {
          pos = 0;
          ++o;
        }
        ob[kk] = o;
        fresh[kk] = kk == 0 || pos == 0;
        in_k[kk] = k0 + 16 * kk < p.K;
      }
    }
    // every load of the chunk first (each block once), then the arithmetic
    int8_t q[4][8];
    __nv_bfloat16 f[4][8];
#pragma unroll
    for (int rr = 0; rr < 4; ++rr) {
      const int n = n_tile * ROWS + lane + 32 * rr;
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        q[rr][kk] = 0;
        f[rr][kk] = __ushort_as_bfloat16(0x3F80);
        if (fresh[kk] && in_k[kk] && n < p.N) {
          const uint32_t b = (uint32_t)n * per_row + o0 + ob[kk];
          q[rr][kk] = reinterpret_cast<const int8_t*>(p.row_scale)[b];
          f[rr][kk] = reinterpret_cast<const __nv_bfloat16*>(p.out_scale)[b / sbs];
        }
      }
    }
    const float mean = __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(p.out_scale2));
#pragma unroll
    for (int rr = 0; rr < 4; ++rr) {
      const int r = lane + 32 * rr;
      const bool row_ok = n_tile * ROWS + r < p.N;
      uint32_t w[4] = {0u, 0u, 0u, 0u}, s = 0u;
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        if (fresh[kk]) s = in_k[kk] && row_ok ? scaler_bits(q[rr][kk], f[rr][kk], mean) : 0u;
        w[kk >> 1] |= s << (16 * (kk & 1));
      }
      *reinterpret_cast<uint4*>(aux + r * 16) = make_uint4(w[0], w[1], w[2], w[3]);
    }
    if (lane < 8) {
      const uint16_t* e = reinterpret_cast<const uint16_t*>(p.w_scale) + 4 * (lane & 3);
      const uint32_t lo = e[0] | (uint32_t)e[1] << 16, hi = e[2] | (uint32_t)e[3] << 16;
      *reinterpret_cast<uint32_t*>(aux + LUT_OFF + 4 * lane) = __byte_perm(lo, hi, lane < 4 ? 0x6420 : 0x7531);
    }
  }
  // c: the code words of Mxfp4Fmt::Raw (the same bytes; here the even k is the high nibble); s[h][i]: the bf16 scalers
  // of row h's steps 2i, 2i + 1; lut: the table's byte planes
  struct Raw {
    uint32_t c[2][4];
    uint32_t s[2][4];
    uint32_t lut[8];
  };
  __device__ static __forceinline__ void load(const tsg::Params&, uint32_t w_smem, uint32_t aux_smem, int row_lo, int lane,
                                              Raw& raw) {
    const uint32_t t = lane & 3;
    const uint32_t sel = t | (t + 4) << 4 | t << 8 | (t + 4) << 12;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = row_lo + 8 * h;
      const uint4 sv = tsg::lds128(aux_smem + (uint32_t)r * 16u);
      raw.s[h][0] = sv.x;
      raw.s[h][1] = sv.y;
      raw.s[h][2] = sv.z;
      raw.s[h][3] = sv.w;
#pragma unroll
      for (int j = 0; j < 4; ++j) raw.c[h][j] = Mxfp4Fmt::lds_codes(w_smem, r, j, sel);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const uint4 l = tsg::lds128(aux_smem + LUT_OFF + 16 * i);
      raw.lut[4 * i] = l.x;
      raw.lut[4 * i + 1] = l.y;
      raw.lut[4 * i + 2] = l.z;
      raw.lut[4 * i + 3] = l.w;
    }
  }
  __device__ static __forceinline__ void frag(const tsg::Params&, const Raw& raw, int kk, uint32_t (&a)[4]) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t s_bits = __byte_perm(raw.s[h][kk >> 1], 0u, (kk & 1) ? 0x3232u : 0x1010u);
      const __nv_bfloat162 s2 = *reinterpret_cast<const __nv_bfloat162*>(&s_bits);
      // nibbles 0..3: the odd and the even k of the pair 16kk + 2t, then of the pair 8 further
      const uint32_t w = raw.c[h][kk >> 1] >> (16 * (kk & 1));
      const uint32_t sel7 = w & 0x7777u, pick = ((w >> 1) & 0x4444u) | 0x3210u;
      const uint32_t lo = __byte_perm(__byte_perm(raw.lut[0], raw.lut[1], sel7), __byte_perm(raw.lut[2], raw.lut[3], sel7), pick);
      const uint32_t hi = __byte_perm(__byte_perm(raw.lut[4], raw.lut[5], sel7), __byte_perm(raw.lut[6], raw.lut[7], sel7), pick);
      const uint32_t v0 = __byte_perm(lo, hi, 0x4051), v1 = __byte_perm(lo, hi, 0x6273);
      const __nv_bfloat162 d0 = __hmul2(*reinterpret_cast<const __nv_bfloat162*>(&v0), s2);
      const __nv_bfloat162 d1 = __hmul2(*reinterpret_cast<const __nv_bfloat162*>(&v1), s2);
      a[h] = *reinterpret_cast<const uint32_t*>(&d0);
      a[h + 2] = *reinterpret_cast<const uint32_t*>(&d1);
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
  if (KIND == KIND_NVF4 || KIND == KIND_MXF4) {
    float s;
    if (KIND == KIND_NVF4) {
      const __half_raw sh = __nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)sbyte, __NV_E4M3);
      s = __half2float(*reinterpret_cast<const __half*>(&sh));
    } else {
      s = e8m0_to_f32(sbyte);   // code x 2^(e-127) is exact in fp32 (subnormals kept) and then in bf16
    }
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

// mxfp8 / nvfp4: activation slabs dequantised into the workspace behind the partial slots, one GEMM per slab
template <int KIND>
static int block_scaled(const char* what, const uint8_t* xq, const uint8_t* x_sf, const float* a_pts, int M, int K,
                        const uint8_t* wq, const uint8_t* w_sf, const float* b_pts, int N, const uint16_t* bias,
                        uint16_t* y, void* ws, size_t ws_bytes, void* stream) {
  using Fmt = std::conditional_t<KIND == KIND_NVF4, nvf4w::Nvfp4Fmt,
                                 std::conditional_t<KIND == KIND_MXF4, Mxfp4Fmt, Mxfp8Fmt>>;
  tsg::Params p{};
  if (int rc = tsg::dense_params(p, what, "xq", xq, K, M, K, N, N, bias, y)) return rc;
  if (M == 0) return AO_OK;
  AO_REQUIRE(x_sf && wq && w_sf, "%s: null pointer", what);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int sf_per_row = KIND == KIND_NVF4 ? K / 16 : K / 32;
  const int sf_col_blocks = ceil_div(sf_per_row, 4);
  CUtensorMap tm_w, tm_sf;
  if (int rc = Fmt::make_maps(wq, w_sf, N, K, &tm_w, &tm_sf)) return rc;
  p.out_scale = KIND == KIND_NVF4 ? b_pts : nullptr;
  p.out_scale2 = KIND == KIND_NVF4 ? a_pts : nullptr;
  p.aux_col_blocks = sf_col_blocks;
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
    tsg::Params ps = p;
    ps.y = p.y + (size_t)m0 * N;
    ps.M = rows;
    if (int rc = tsg::run<Fmt>(ps, tm_w, tm_sf, xb, K, ws, act_off, what, st)) return rc;
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
  AO_REQUIRE(K % 16 == 0, "int8 linear: K=%d must be a multiple of 16 (TMA row pitch)", K);
  AO_REQUIRE(N % 8 == 0, "int8 linear: N=%d must be a multiple of 8 (reference: int8/kernels.py:48-58)", N);
  using Fmt = lowp::SsFmt<lowp::KIND_I8>;
  return tsg::run_dense<Fmt>("int8 linear", "xq", xq, K, M, K, N, N, bias, y, workspace, workspace_bytes, stream,
                             [&](tsg::Params& p, CUtensorMap* tm_w, CUtensorMap* tm_aux) {
    AO_REQUIRE(x_scale && wq && w_scale, "int8 linear: null pointer");
    p.row_scale = x_scale;
    p.w_scale = w_scale;
    return Fmt::make_maps(reinterpret_cast<const uint8_t*>(wq), N, K, tm_w, tm_aux);
  });
}

extern "C" int ao_int8_mm_i32(const int8_t* xq, int M, int K, const int8_t* wq, int N, int32_t* acc,
                              void* workspace, size_t workspace_bytes, void* stream) {
  AO_REQUIRE(K % 16 == 0, "int8 mm: K=%d must be a multiple of 16 (TMA row pitch)", K);
  using Fmt = lowp::SsFmt<lowp::KIND_I8>;
  return tsg::run_dense<Fmt>("int8 mm", "xq", xq, K, M, K, N, N, nullptr, acc, workspace, workspace_bytes, stream,
                             [&](tsg::Params& p, CUtensorMap* tm_w, CUtensorMap* tm_aux) {
    AO_REQUIRE(wq, "int8 mm: null pointer");
    p.i32_out = acc;   // the raw s32 sums instead of y
    p.y = nullptr;
    return Fmt::make_maps(reinterpret_cast<const uint8_t*>(wq), N, K, tm_w, tm_aux);
  });
}

// F.linear(x, Int8Tensor without act_quant_kwargs), per-row or per-tensor scale (int8_tensor.py:336-359):
// y = bf16(bf16(bf16(x wq^T) * bf16(w_scale[n])) + bias[n]); one launch, no activation quantizer
extern "C" int ao_int8_weight_linear(const uint16_t* x, int ldx, int M, int K, const int8_t* wq, const float* w_scale,
                                     int N, const uint16_t* bias, uint16_t* y, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  AO_REQUIRE(K % 16 == 0, "int8 weight linear: K=%d must be a multiple of 16 (TMA row pitch)", K);
  using Fmt = lowp::Int8WoFmt;
  return tsg::run_dense<Fmt>("int8 weight linear", "x", x, ldx, M, K, N, N, bias, y, workspace, workspace_bytes, stream,
                             [&](tsg::Params& p, CUtensorMap* tm_w, CUtensorMap* tm_aux) {
    AO_REQUIRE(wq && w_scale, "int8 weight linear: null pointer");
    p.w_scale = w_scale;
    return Fmt::make_maps(reinterpret_cast<const uint8_t*>(wq), N, K, tm_w, tm_aux);
  });
}

// F.linear(x, Float8Tensor without act_quant_kwargs), per-row or per-tensor scale (float8_tensor.py:459-469):
// y = bf16(bf16(sum_k x[m,k] * bf16(fp32(e4m3(wq[n,k]) * w_scale[n]))) + bias[n]); one launch, no activation quantizer
extern "C" int ao_fp8_weight_linear(const uint16_t* x, int ldx, int M, int K, const uint8_t* wq, const float* w_scale,
                                    int N, const uint16_t* bias, uint16_t* y, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  AO_REQUIRE(K % 16 == 0, "fp8 weight linear: K=%d must be a multiple of 16 (TMA row pitch)", K);
  using Fmt = lowp::Fp8WoFmt;
  return tsg::run_dense<Fmt>("fp8 weight linear", "x", x, ldx, M, K, N, N, bias, y, workspace, workspace_bytes, stream,
                             [&](tsg::Params&, CUtensorMap* tm_w, CUtensorMap* tm_s) {
    AO_REQUIRE(wq && w_scale, "fp8 weight linear: null pointer");
    AO_REQUIRE((reinterpret_cast<uintptr_t>(w_scale) & 15) == 0,
               "fp8 weight linear: w_scale must be 16-byte aligned (it is loaded by TMA)");
    return Fmt::make_maps(wq, w_scale, N, K, tm_w, tm_s);
  });
}

// F.linear(x, NF4Tensor) (nf4_tensor.py LinearNF4 and the F.linear override): y = bf16(bf16(sum_k x[m,k] * w~[n,k]) +
// bias[n]), w~ = the reference's get_original_weight(); one launch, the scalers decoded in the kernel (Nf4Fmt)
extern "C" int ao_nf4_linear(const uint16_t* x, int ldx, int M, int K, const uint8_t* quantized_data,
                             const int8_t* quantized_scalers, const uint16_t* quantization_factor,
                             const uint16_t* scaler_mean, const uint16_t* nf4, int block_size, int scaler_block_size,
                             int N, const uint16_t* bias, uint16_t* y, void* workspace, size_t workspace_bytes,
                             void* stream) {
  AO_REQUIRE(block_size > 0 && block_size % 16 == 0, "nf4 linear: block_size=%d must be a positive multiple of 16",
             block_size);
  AO_REQUIRE(K % block_size == 0, "nf4 linear: K=%d must be a multiple of block_size=%d", K, block_size);
  AO_REQUIRE(K % 32 == 0, "nf4 linear: K=%d must be a multiple of 32 (TMA row pitch of the codes)", K);
  const long long n_blocks = N > 0 ? (long long)N * (K / block_size) : 0;
  AO_REQUIRE(n_blocks <= 0x7FFFFFFF, "nf4 linear: N*K/block_size=%lld scalers exceed the int32 range", n_blocks);
  AO_REQUIRE(scaler_block_size > 0 && n_blocks % scaler_block_size == 0,
             "nf4 linear: scaler_block_size=%d must divide the %lld scalers", scaler_block_size, n_blocks);
  using Fmt = lowp::Nf4Fmt;
  return tsg::run_dense<Fmt>("nf4 linear", "x", x, ldx, M, K, N, N, bias, y, workspace, workspace_bytes, stream,
                             [&](tsg::Params& p, CUtensorMap* tm_w, CUtensorMap* tm_aux) {
    AO_REQUIRE(quantized_data && quantized_scalers && quantization_factor && scaler_mean && nf4,
               "nf4 linear: null pointer");
    p.row_scale = reinterpret_cast<const float*>(quantized_scalers);   // the fields of Nf4Fmt (see there)
    p.out_scale = reinterpret_cast<const float*>(quantization_factor);
    p.out_scale2 = reinterpret_cast<const float*>(scaler_mean);
    p.w_scale = reinterpret_cast<const float*>(nf4);
    p.group_size = block_size;
    p.aux_col_blocks = scaler_block_size;
    return Fmt::make_maps(quantized_data, N, K, tm_w, tm_aux);
  });
}

extern "C" int ao_fp8_rowwise_linear(const uint8_t* xq, const float* x_scale, int M, int K,
                                     const uint8_t* wq, const float* w_scale, int N,
                                     const uint16_t* bias, uint16_t* y, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  AO_REQUIRE(K % 16 == 0, "fp8 linear: K=%d must be a multiple of 16 (reference: quantization/utils.py:663-687)", K);
  AO_REQUIRE(N % 16 == 0, "fp8 linear: N=%d must be a multiple of 16 (reference: quantization/utils.py:663-687)", N);
  using Fmt = lowp::SsFmt<lowp::KIND_F8>;
  return tsg::run_dense<Fmt>("fp8 linear", "xq", xq, K, M, K, N, N, bias, y, workspace, workspace_bytes, stream,
                             [&](tsg::Params& p, CUtensorMap* tm_w, CUtensorMap* tm_aux) {
    AO_REQUIRE(x_scale && wq && w_scale, "fp8 linear: null pointer");
    p.row_scale = x_scale;
    p.w_scale = w_scale;
    return Fmt::make_maps(wq, N, K, tm_w, tm_aux);
  });
}

// F.linear(x, PrototypeFloat8Tensor) (prototype_float8_tensor.py:329-474) on the static quantizer's codes: the output of
// ao_fp8_rowwise_linear, y = bf16(acc * (x_scale[m] * w_scale[n]) + bias[n]), with w_scale[0] for every n when
// w_scale_per_row == 0; with out_scale, y is then quantized to e4m3 with the output scale and dequantized:
// bf16(fp32(e4m3(clamp(y / s, -448, 448))) * s), s = out_scale[0] or (out_scale_per_row) out_scale[m]
extern "C" int ao_fp8_static_linear(const uint8_t* xq, const float* x_scale, int M, int K, const uint8_t* wq,
                                    const float* w_scale, int w_scale_per_row, int N, const uint16_t* bias,
                                    const float* out_scale, int out_scale_per_row, uint16_t* y, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  AO_REQUIRE(K % 16 == 0, "fp8 static linear: K=%d must be a multiple of 16 (reference: quantization/utils.py:663-687)", K);
  AO_REQUIRE(N % 16 == 0, "fp8 static linear: N=%d must be a multiple of 16 (reference: quantization/utils.py:663-687)", N);
  using Fmt = lowp::F8StaticFmt;
  return tsg::run_dense<Fmt>("fp8 static linear", "xq", xq, K, M, K, N, N, bias, y, workspace, workspace_bytes, stream,
                             [&](tsg::Params& p, CUtensorMap* tm_w, CUtensorMap* tm_aux) {
    AO_REQUIRE(x_scale && wq && w_scale, "fp8 static linear: null pointer");
    p.row_scale = x_scale;
    p.w_scale = w_scale;
    p.out_scale = out_scale;
    p.out_scale_per_row = (out_scale_per_row ? tsg::F8S_OUT_PER_TOKEN : 0) | (w_scale_per_row ? 0 : tsg::F8S_W_PER_TENSOR);
    return Fmt::make_maps(wq, N, K, tm_w, tm_aux);
  });
}

// F.linear(x, Float8Tensor with 128x128 weight blocks and 1x128 activation blocks) (float8_tensor.py:431-447):
// y = bf16(bf16(acc) + bias[n]), acc summed chunk by chunk as BlockwiseF8Fmt states.  x_scale_t: the transposed
// activation scales [K/128][round_up(M, 4)] of ao_fp8_quantize_1x128; w_scale [N/128][K/128].
extern "C" int ao_fp8_blockwise_linear(const uint8_t* xq, const float* x_scale_t, int M, int K, const uint8_t* wq,
                                       const float* w_scale, int N, const uint16_t* bias, uint16_t* y, void* workspace,
                                       size_t workspace_bytes, void* stream) {
  AO_REQUIRE(K % 128 == 0, "fp8 blockwise linear: K=%d must be a multiple of 128 (one scale per 128 k)", K);
  AO_REQUIRE(N % 128 == 0, "fp8 blockwise linear: N=%d must be a multiple of 128 (one scale per 128 rows)", N);
  using Fmt = lowp::BlockwiseF8Fmt;
  return tsg::run_dense<Fmt>("fp8 blockwise linear", "xq", xq, K, M, K, N, N, bias, y, workspace, workspace_bytes,
                             stream, [&](tsg::Params& p, CUtensorMap* tm_w, CUtensorMap* tm_xs) {
    AO_REQUIRE(x_scale_t && wq && w_scale, "fp8 blockwise linear: null pointer");
    AO_REQUIRE((reinterpret_cast<uintptr_t>(x_scale_t) & 15) == 0,
               "fp8 blockwise linear: x_scale must be 16-byte aligned (it is loaded by TMA)");
    p.w_scale = w_scale;
    return Fmt::make_maps(wq, x_scale_t, M, N, K, tm_w, tm_xs);
  });
}

// F.linear(x, Float8Sparse2x4_2DData2DMetadataTensor) (float8_sparse_2x4_2d_data_2d_metadata_tensor.py): per-token
// e4m3 xq with x_scale [M], the 2:4-compressed weights wq [N][K/2] with the CUTLASS metadata w_meta
// (round_up(N, 64) x round_up(K, 128) / 8 bytes, SparseF8Fmt) and w_scale [N]:
// y = bf16(fma(acc * w_scale[n], x_scale[m], bias[n])), acc summed without promotion (SparseF8Fmt)
extern "C" int ao_fp8_sparse_linear(const uint8_t* xq, const float* x_scale, int M, int K, const uint8_t* wq,
                                    const uint8_t* w_meta, const float* w_scale, int N, const uint16_t* bias, uint16_t* y,
                                    void* workspace, size_t workspace_bytes, void* stream) {
  AO_REQUIRE(K % 32 == 0, "fp8 sparse linear: K=%d must be a multiple of 32 (16-byte rows of compressed codes)", K);
  AO_REQUIRE(N % 16 == 0, "fp8 sparse linear: N=%d must be a multiple of 16", N);
  using Fmt = lowp::SparseF8Fmt;
  return tsg::run_dense<Fmt>("fp8 sparse linear", "xq", xq, K, M, K, N, N, bias, y, workspace, workspace_bytes, stream,
                             [&](tsg::Params& p, CUtensorMap* tm_w, CUtensorMap* tm_m) {
    AO_REQUIRE(x_scale && wq && w_meta && w_scale, "fp8 sparse linear: null pointer");
    AO_REQUIRE((reinterpret_cast<uintptr_t>(wq) & 15) == 0, "fp8 sparse linear: wq must be 16-byte aligned");
    AO_REQUIRE((reinterpret_cast<uintptr_t>(w_meta) & 15) == 0,
               "fp8 sparse linear: w_meta must be 16-byte aligned (it is loaded by TMA)");
    p.row_scale = x_scale;
    p.w_scale = w_scale;
    return Fmt::make_maps(wq, w_meta, N, K, tm_w, tm_m);
  });
}

// torch._grouped_mm(x, W.transpose(-2, -1), offs) on rowwise e4m3 operands: expert e's rows [offs[e-1], offs[e]) of
// xq against its weights wq[e] (the stored [E, N, K] qdata), the dense kernel's epilogue with w_scale[e, :].  offs
// stays on the device (grouped schedule, ts_gemm.cuh).
extern "C" int ao_fp8_rowwise_grouped_mm(const uint8_t* xq, const float* x_scale, int M, int K,
                                         const uint8_t* wq, const float* w_scale, int E, int N,
                                         const int32_t* offs, uint16_t* y, void* workspace,
                                         size_t workspace_bytes, void* stream) {
  AO_REQUIRE(K % 16 == 0, "fp8 grouped mm: K=%d must be a multiple of 16 (TMA row pitch)", K);
  AO_REQUIRE(N % 16 == 0, "fp8 grouped mm: N=%d must be a multiple of 16", N);
  using Fmt = lowp::SsFmt<lowp::KIND_F8>;
  return tsg::run_grouped<Fmt>("fp8 grouped mm", xq, M, K, E, N, N, offs, y, workspace, workspace_bytes, stream,
                               [&](tsg::Params& p, CUtensorMap* tm_w, CUtensorMap* tm_aux) {
    AO_REQUIRE(x_scale && wq && w_scale, "fp8 grouped mm: null pointer");
    p.row_scale = x_scale;
    p.w_scale = w_scale;
    return Fmt::make_maps(wq, E * N, K, tm_w, tm_aux);
  });
}

namespace ao {
namespace lowp {
// torch.bmm runs as the grouped schedule with B groups of M rows: offs[b] = (b + 1) * M, written on the device (no
// host copy: a CUDA graph replays it) between the stream-K flags and the partial slots of the workspace.  It waits for
// the previous kernel first, which may be a batched GEMM still reading the last offs.
constexpr size_t BMM_OFFS_OFF = streamk::WS_FLAGS_BYTES;
static_assert(BMM_OFFS_OFF + 4 * tsg::MAX_EXPERTS <= streamk::WS_PARTIAL_OFF, "bmm offs do not fit the workspace");
__global__ void bmm_offs_kernel(int32_t* offs, int B, int M) {
  pdl_launch_dependents();
  pdl_wait();
  for (int b = threadIdx.x; b < B; b += blockDim.x) offs[b] = (b + 1) * M;
}
}  // namespace lowp
}  // namespace ao

// torch.bmm(x, w) on rowwise e4m3 operands, w a [B, K, N] Float8Tensor: xq [B*M, K] (x's rows, batch-major) with
// x_scale [B*M], against batch b's weights with w_scale [B, N], y [B*M, N] = bf16(acc * x_scale[m] * w_scale[b, n]),
// no bias.  w_kn = 0: wq is stored [B, N, K] (K-major, w the transposed view: the grouped kernel of
// ao_fp8_rowwise_grouped_mm); w_kn = 1: wq is stored [B, K, N] (N-major: F8NMajorFmt, no transposed copy).
extern "C" int ao_fp8_rowwise_bmm(const uint8_t* xq, const float* x_scale, int B, int M, int K, const uint8_t* wq,
                                  const float* w_scale, int N, int w_kn, uint16_t* y, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  AO_REQUIRE(B >= 1 && B <= tsg::MAX_EXPERTS, "fp8 bmm: B=%d must be in [1, %d]", B, tsg::MAX_EXPERTS);
  AO_REQUIRE(M >= 0 && K > 0 && N > 0, "fp8 bmm: bad sizes M=%d K=%d N=%d", M, K, N);
  AO_REQUIRE((long long)B * M <= 0x7FFFFFFF, "fp8 bmm: B*M=%lld rows exceed the int32 range", (long long)B * M);
  AO_REQUIRE(K % 16 == 0, "fp8 bmm: K=%d must be a multiple of 16 (TMA row pitch)", K);
  AO_REQUIRE(N % 16 == 0, "fp8 bmm: N=%d must be a multiple of 16", N);
  AO_REQUIRE(w_kn == 0 || w_kn == 1, "fp8 bmm: w_kn=%d must be 0 ([B, N, K] weights) or 1 ([B, K, N])", w_kn);
  if (M == 0) return AO_OK;
  AO_REQUIRE(xq && x_scale && wq && w_scale && y && workspace, "fp8 bmm: null pointer");
  AO_REQUIRE(workspace_bytes >= streamk::WS_PARTIAL_OFF, "fp8 bmm: workspace too small (%zu bytes)", workspace_bytes);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int32_t* offs = reinterpret_cast<int32_t*>(reinterpret_cast<uint8_t*>(workspace) + lowp::BMM_OFFS_OFF);
  AO_CUDA_CHECK(ao::launch(lowp::bmm_offs_kernel, dim3(1), dim3(256), 0, st, pdl_enabled(), offs, B, M));
  auto setup = [&](tsg::Params& p, CUtensorMap* tm_w, CUtensorMap* tm_aux) {
    p.row_scale = x_scale;
    p.w_scale = w_scale;
    return w_kn ? lowp::F8NMajorFmt::make_maps(wq, B, K, N, tm_w, tm_aux)
                : lowp::SsFmt<lowp::KIND_F8>::make_maps(wq, B * N, K, tm_w, tm_aux);
  };
  if (w_kn)
    return tsg::run_grouped<lowp::F8NMajorFmt>("fp8 bmm", xq, B * M, K, B, N, N, offs, y, workspace, workspace_bytes,
                                               stream, setup);
  return tsg::run_grouped<lowp::SsFmt<lowp::KIND_F8>>("fp8 bmm", xq, B * M, K, B, N, N, offs, y, workspace,
                                                      workspace_bytes, stream, setup);
}

// torch._grouped_mm(x, W.transpose(-2, -1), offs) on blockwise e4m3 operands: expert e's rows [offs[e-1], offs[e]) of
// xq (x_scale_t [K/128][round_up(M, 4)] of ao_fp8_quantize_1x128 over all M rows) against wq[e] (the stored [E, N, K]
// qdata) with its 128x128 block scales w_scale[e] ([E, N/128, K/128]), summed and rounded as the dense
// ao_fp8_blockwise_linear does, without bias.  offs stays on the device (grouped schedule, ts_gemm.cuh).
extern "C" int ao_fp8_blockwise_grouped_mm(const uint8_t* xq, const float* x_scale_t, int M, int K, const uint8_t* wq,
                                           const float* w_scale, int E, int N, const int32_t* offs, uint16_t* y,
                                           void* workspace, size_t workspace_bytes, void* stream) {
  AO_REQUIRE(K % 128 == 0, "fp8 blockwise grouped mm: K=%d must be a multiple of 128 (one scale per 128 k)", K);
  AO_REQUIRE(N % 128 == 0, "fp8 blockwise grouped mm: N=%d must be a multiple of 128 (one scale per 128 rows)", N);
  using Fmt = lowp::BlockwiseF8GroupedFmt;
  return tsg::run_grouped<Fmt>("fp8 blockwise grouped mm", xq, M, K, E, N, N, offs, y, workspace, workspace_bytes,
                               stream, [&](tsg::Params& p, CUtensorMap* tm_w, CUtensorMap* tm_xs) {
    AO_REQUIRE(x_scale_t && wq && w_scale, "fp8 blockwise grouped mm: null pointer");
    AO_REQUIRE((reinterpret_cast<uintptr_t>(x_scale_t) & 15) == 0,
               "fp8 blockwise grouped mm: x_scale must be 16-byte aligned (it is loaded by TMA)");
    p.w_scale = w_scale;
    return Fmt::make_maps(wq, x_scale_t, M, E * N, K, tm_w, tm_xs);
  });
}

// torch._grouped_mm(x, W.transpose(-2, -1), offs) on weight-only e4m3 expert weights (float8_tensor.py:1085-1122,
// weight-only branch: torch._grouped_mm on W.dequantize()), 2-D x 3-D: expert e's rows [offs[e-1], offs[e]) of the
// bf16 x against wq[e] (the stored [E, N, K] qdata), each weight dequantized as the dense fp8 weight-only linear does
// with w_scale[e, n], y = bf16(sum).  No bias.  offs stays on the device (grouped schedule, ts_gemm.cuh).
extern "C" int ao_fp8_weight_grouped_mm(const uint16_t* x, int M, int K, const uint8_t* wq, const float* w_scale, int E,
                                        int N, const int32_t* offs, uint16_t* y, void* workspace,
                                        size_t workspace_bytes, void* stream) {
  AO_REQUIRE(K % 16 == 0, "fp8 weight grouped mm: K=%d must be a multiple of 16 (TMA row pitch)", K);
  // every scale box (element e*N + 128t of w_scale) starts on 32 bytes and every weight box on a row multiple of 8
  AO_REQUIRE(N % 8 == 0, "fp8 weight grouped mm: N=%d must be a multiple of 8", N);
  using Fmt = lowp::Fp8WoFmt;
  return tsg::run_grouped<Fmt>("fp8 weight grouped mm", x, M, K, E, N, N, offs, y, workspace, workspace_bytes, stream,
                               [&](tsg::Params&, CUtensorMap* tm_w, CUtensorMap* tm_s) {
    AO_REQUIRE(wq && w_scale, "fp8 weight grouped mm: null pointer");
    AO_REQUIRE((reinterpret_cast<uintptr_t>(w_scale) & 15) == 0,
               "fp8 weight grouped mm: w_scale must be 16-byte aligned (it is loaded by TMA)");
    return Fmt::make_maps(wq, w_scale, E * N, K, tm_w, tm_s);
  });
}

// torch._grouped_mm(x, W.transpose(-2, -1), offs) on weight-only int8 expert weights, 2-D x 3-D: expert e's rows
// [offs[e-1], offs[e]) of the bf16 x against wq[e] (the stored [E, N, K] qdata), the dense int8 weight-only epilogue
// with w_scale[e, n] and no bias, y = bf16(bf16(bf16(x wq[e]^T) * bf16(w_scale[e, n]))), which is what select + the
// dense linear computes per expert.  offs stays on the device (grouped schedule, ts_gemm.cuh).
extern "C" int ao_int8_weight_grouped_mm(const uint16_t* x, int M, int K, const int8_t* wq, const float* w_scale, int E,
                                         int N, const int32_t* offs, uint16_t* y, void* workspace,
                                         size_t workspace_bytes, void* stream) {
  AO_REQUIRE(K % 16 == 0, "int8 weight grouped mm: K=%d must be a multiple of 16 (TMA row pitch)", K);
  // no N rule: weight boxes may start on any row of the [E * N, K] map, and the scales are read by the epilogue
  using Fmt = lowp::Int8WoFmt;
  return tsg::run_grouped<Fmt>("int8 weight grouped mm", x, M, K, E, N, N, offs, y, workspace, workspace_bytes, stream,
                               [&](tsg::Params& p, CUtensorMap* tm_w, CUtensorMap* tm_aux) {
    AO_REQUIRE(wq && w_scale, "int8 weight grouped mm: null pointer");
    p.w_scale = w_scale;
    return Fmt::make_maps(reinterpret_cast<const uint8_t*>(wq), E * N, K, tm_w, tm_aux);
  });
}

// torch._grouped_mm(x, W.transpose(-2, -1), offs) on int8 expert weights with per-token int8 activations: expert e's
// rows [offs[e-1], offs[e]) of xq (x_scale [M] per row) against wq[e], s32 sums, the dense int8 epilogue
// y = bf16(bf16(acc * x_scale[m]) * w_scale[e, n]) without bias.  offs stays on the device (grouped schedule,
// ts_gemm.cuh).
extern "C" int ao_int8_dyn_grouped_mm(const int8_t* xq, const float* x_scale, int M, int K, const int8_t* wq,
                                      const float* w_scale, int E, int N, const int32_t* offs, uint16_t* y,
                                      void* workspace, size_t workspace_bytes, void* stream) {
  AO_REQUIRE(K % 16 == 0, "int8 grouped mm: K=%d must be a multiple of 16 (TMA row pitch)", K);
  AO_REQUIRE(N % 8 == 0, "int8 grouped mm: N=%d must be a multiple of 8 (reference: int8/kernels.py:48-58)", N);
  using Fmt = lowp::SsFmt<lowp::KIND_I8>;
  return tsg::run_grouped<Fmt>("int8 grouped mm", xq, M, K, E, N, N, offs, y, workspace, workspace_bytes, stream,
                               [&](tsg::Params& p, CUtensorMap* tm_w, CUtensorMap* tm_aux) {
    AO_REQUIRE(x_scale && wq && w_scale, "int8 grouped mm: null pointer");
    p.row_scale = x_scale;
    p.w_scale = w_scale;
    return Fmt::make_maps(reinterpret_cast<const uint8_t*>(wq), E * N, K, tm_w, tm_aux);
  });
}

extern "C" int ao_mxfp8_linear(const uint8_t* xq, const uint8_t* x_scale_blocked, int M, int K,
                               const uint8_t* wq, const uint8_t* w_scale_blocked, int N,
                               const uint16_t* bias, uint16_t* y, void* workspace,
                               size_t workspace_bytes, void* stream) {
  AO_REQUIRE(K % 32 == 0, "mxfp8 linear: K=%d must be a multiple of 32 (mx_tensor.py:244-246)", K);
  return lowp::block_scaled<lowp::KIND_MXF8>("mxfp8 linear", xq, x_scale_blocked, nullptr, M, K, wq, w_scale_blocked,
                                             nullptr, N, bias, y, workspace, workspace_bytes, stream);
}

extern "C" int ao_mxfp4_linear(const uint8_t* xq, const uint8_t* x_scale_blocked, int M, int K,
                               const uint8_t* wq, const uint8_t* w_scale_blocked, int N,
                               const uint16_t* bias, uint16_t* y, void* workspace,
                               size_t workspace_bytes, void* stream) {
  // K / 2 bytes per weight row: a multiple of 16, the TMA row pitch; a K tail of the last chunk is zero-filled
  AO_REQUIRE(K % 32 == 0, "mxfp4 linear: K=%d must be a multiple of 32 (mx_tensor.py:244-246)", K);
  return lowp::block_scaled<lowp::KIND_MXF4>("mxfp4 linear", xq, x_scale_blocked, nullptr, M, K, wq, w_scale_blocked,
                                             nullptr, N, bias, y, workspace, workspace_bytes, stream);
}

extern "C" int ao_nvfp4_linear(const uint8_t* xq, const uint8_t* x_scale_blocked, const float* a_pts,
                               int M, int K, const uint8_t* wq, const uint8_t* w_scale_blocked,
                               const float* b_pts, int N, const uint16_t* bias, uint16_t* y,
                               void* workspace, size_t workspace_bytes, void* stream) {
  AO_REQUIRE(K % 256 == 0, "nvfp4 linear: K=%d must be a multiple of 256", K);
  AO_REQUIRE(N % 16 == 0, "nvfp4 linear: N=%d must be a multiple of 16 (inference_workflow.py:248-251)", N);
  return lowp::block_scaled<lowp::KIND_NVF4>("nvfp4 linear", xq, x_scale_blocked, a_pts, M, K, wq, w_scale_blocked,
                                             b_pts, N, bias, y, workspace, workspace_bytes, stream);
}

// nvfp4 weights x bf16 activations = F.linear(x, NVFP4Tensor.dequantize()) (nvfp4_tensor.py:199-231, weight-only
// handler inference_workflow.py:356-400).  The optional per-token x_scale is applied in the epilogue, so that
// e4m3-rowwise activations (ao_fp8_fakequant_rowwise: values exact in bf16, the scale a row factor) run on the same
// kernel; b_pts is one per-tensor scale or (b_pts_per_row) one per output feature.
extern "C" int ao_nvfp4_weight_linear_ex(const uint16_t* x, int ldx, const float* x_scale, int M, int K, const uint8_t* wq,
                                         const uint8_t* w_scale_blocked, const float* b_pts, int b_pts_per_row, int N,
                                         const uint16_t* bias, uint16_t* y, void* workspace, size_t workspace_bytes,
                                         void* stream) {
  AO_REQUIRE(K % 128 == 0, "nvfp4 weight linear: K=%d must be a multiple of 128", K);
  AO_REQUIRE(N % 16 == 0, "nvfp4 weight linear: N=%d must be a multiple of 16 (inference_workflow.py:248-251)", N);
  using Fmt = nvf4w::Nvfp4Fmt;
  return tsg::run_dense<Fmt>("nvfp4 weight linear", "x", x, ldx, M, K, N, N, bias, y, workspace, workspace_bytes,
                             stream, [&](tsg::Params& p, CUtensorMap* tm_w, CUtensorMap* tm_sf) {
    AO_REQUIRE(wq && w_scale_blocked, "nvfp4 weight linear: null pointer");
    p.row_scale = x_scale;
    p.out_scale = b_pts;
    p.out_scale_per_row = b_pts_per_row;
    p.aux_col_blocks = ceil_div(K / 16, 4);
    return Fmt::make_maps(wq, w_scale_blocked, N, K, tm_w, tm_sf);
  });
}

extern "C" int ao_nvfp4_weight_linear(const uint16_t* x, const float* x_scale, int M, int K, const uint8_t* wq,
                                      const uint8_t* w_scale_blocked, const float* b_pts, int N,
                                      const uint16_t* bias, uint16_t* y, void* workspace, size_t workspace_bytes,
                                      void* stream) {
  return ao_nvfp4_weight_linear_ex(x, K, x_scale, M, K, wq, w_scale_blocked, b_pts, 0, N, bias, y, workspace, workspace_bytes,
                                   stream);
}

// torch._grouped_mm(x, W.transpose(-2, -1), offs) on MX expert weights, 2-D x 3-D: expert e's rows [offs[e-1], offs[e])
// of x (bf16: the exactly dequantised activation codes of ao_mx*_fakequant) against wq[e] with its blocked e8m0 scales,
// y = bf16(acc), the dense MX linear's epilogue without bias.  offs stays on the device (grouped schedule, ts_gemm.cuh).
template <class Fmt>
static int mx_grouped_mm(const char* what, const uint16_t* x, int M, int K, const uint8_t* wq,
                         const uint8_t* w_scale_blocked, int E, int N, const int32_t* offs, uint16_t* y, void* workspace,
                         size_t workspace_bytes, void* stream) {
  AO_REQUIRE(K % 32 == 0, "%s: K=%d must be a multiple of 32 (mx_tensor.py:244-246)", what, K);
  // every expert's weights and scales start on a 128-row block of the stacked [E * N, ..] tensors
  AO_REQUIRE(N % 128 == 0, "%s: N=%d must be a multiple of 128", what, N);
  return tsg::run_grouped<Fmt>(what, x, M, K, E, N, N, offs, y, workspace, workspace_bytes, stream,
                               [&](tsg::Params& p, CUtensorMap* tm_w, CUtensorMap* tm_sf) {
    AO_REQUIRE(wq && w_scale_blocked, "%s: null pointer", what);
    p.aux_col_blocks = ceil_div(K / 32, 4);
    return Fmt::make_maps(wq, w_scale_blocked, E * N, K, tm_w, tm_sf);
  });
}

extern "C" int ao_mxfp8_grouped_mm(const uint16_t* x, int M, int K, const uint8_t* wq, const uint8_t* w_scale_blocked,
                                   int E, int N, const int32_t* offs, uint16_t* y, void* workspace,
                                   size_t workspace_bytes, void* stream) {
  return mx_grouped_mm<lowp::Mxfp8Fmt>("mxfp8 grouped mm", x, M, K, wq, w_scale_blocked, E, N, offs, y, workspace,
                                       workspace_bytes, stream);
}

extern "C" int ao_mxfp4_grouped_mm(const uint16_t* x, int M, int K, const uint8_t* wq, const uint8_t* w_scale_blocked,
                                   int E, int N, const int32_t* offs, uint16_t* y, void* workspace,
                                   size_t workspace_bytes, void* stream) {
  return mx_grouped_mm<lowp::Mxfp4Fmt>("mxfp4 grouped mm", x, M, K, wq, w_scale_blocked, E, N, offs, y, workspace,
                                       workspace_bytes, stream);
}

// torch._grouped_mm(x, W.transpose(-2, -1), offs) on NVFP4 expert weights (nvfp4_tensor.py:709-753), 2-D x 3-D:
// expert e's rows [offs[e-1], offs[e]) of x (bf16; for NVFP4 activations the exactly dequantised codes of
// ao_nvfp4_fakequant_grouped) against wq[e] (the stored [E, N, K/2] qdata) with its blocked scales, the nvfp4-weight
// epilogue y = acc * x_scale[m] * w_pts[e].  offs stays on the device (grouped schedule, ts_gemm.cuh).
extern "C" int ao_nvfp4_grouped_mm(const uint16_t* x, const float* x_scale, int M, int K, const uint8_t* wq,
                                   const uint8_t* w_scale_blocked, const float* w_pts, int E, int N,
                                   const int32_t* offs, uint16_t* y, void* workspace, size_t workspace_bytes,
                                   void* stream) {
  AO_REQUIRE(K % 128 == 0, "nvfp4 grouped mm: K=%d must be a multiple of 128", K);
  // every expert's weights and scales start on a 128-row block of the stacked [E * N, ..] tensors
  AO_REQUIRE(N % 128 == 0, "nvfp4 grouped mm: N=%d must be a multiple of 128", N);
  using Fmt = nvf4w::Nvfp4Fmt;
  return tsg::run_grouped<Fmt>("nvfp4 grouped mm", x, M, K, E, N, N, offs, y, workspace, workspace_bytes, stream,
                               [&](tsg::Params& p, CUtensorMap* tm_w, CUtensorMap* tm_sf) {
    AO_REQUIRE(wq && w_scale_blocked && w_pts, "nvfp4 grouped mm: null pointer");
    p.row_scale = x_scale;
    p.out_scale = w_pts;
    p.aux_col_blocks = ceil_div(K / 16, 4);
    return Fmt::make_maps(wq, w_scale_blocked, E * N, K, tm_w, tm_sf);
  });
}
