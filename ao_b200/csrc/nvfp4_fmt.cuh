// NVFP4 weights (e2m1 pairs, even k in the low nibble; e4m3 block-16 scales in the blocked 128 x 4 tile layout)
// as the register-A operand of ts_gemm.cuh: each consumer thread turns the bytes of its two fragment rows into the
// bf16 wgmma A fragment.  Used by the nvfp4-weight linear, the nvfp4 x nvfp4 linear and (Grouped<Nvfp4Fmt>) the nvfp4
// expert GEMM.
//
// e2m1 -> bf16 without a table: nibble x = (s e1 e0 m) placed at bf16 bits 15|8:6 is the bf16 number
// value(x) * 2^-126 (denormal for e = 0, which bf16 multiplies handle exactly); ONE exact multiply by
// (block_scale * 2^66) gives value(x) * block_scale * 2^-60, and the 2^60 is taken back out of the fp32 accumulator in the
// epilogue (ACC_EXP2; power-of-two factors commute with every rounding on the way).  The scale byte placed at
// bf16 bits 10:4 is the bf16 number block_scale * 2^-120 for EVERY byte 0x00..0x7E: normal bytes map exponent to
// exponent, and the subnormal bytes 0x01..0x07 (m * 2^-9) and the zero byte become bf16 subnormals / zero, which bf16
// multiplies handle exactly.  Two exact multiplies (by 2^127, then 2^59) give bf16(block_scale * 2^66), once per
// chunk in load() for two scales at a time rather than once per k16 step in frag(); this is
// (byte << 4) + 0x5D00 only for the normal bytes >= 0x08, and quantizers without a lower clamp on the scale (such as
// the TransformerEngine NVFP4 recipe) do write 0x00..0x07.  The product with an e2m1 value has at most 6 significant
// bits and, when not zero, lies between 2^-70 and 2^-48 (normal), so the bf16 A operand is exact.  Bytes with the sign bit and 0x7F (NaN) are not
// decoded: no quantizer writes them.
#pragma once
#include <cuda_bf16.h>

#include "ptx.cuh"
#include "ts_gemm.cuh"

namespace ao {
namespace nvf4w {

struct Nvfp4Fmt {
  static constexpr bool SS = false;
  // at 104 consumer registers the dequant of a chunk spills inside the chunk loop: one CTA per SM
  static constexpr bool DECODE_2CTA = false;
  static constexpr bool PROMOTE = false;
  static constexpr int X_ELEM_BYTES = 2;
  static constexpr int W_BYTES = tsg::ROWS * tsg::KCHUNK / 2;   // 128 rows x 64 bytes, 64-byte swizzle
  static constexpr int AUX_BYTES = 1024;                        // two blocked scale tiles (64 k each)
  static constexpr int EPI = tsg::EPI_FLOAT;
  static constexpr int ACC_EXP2 = 60;   // the accumulators hold the result * 2^-60
  static constexpr int MAX_N_MMA = 128;
  // the packed weights (128 rows x 64 bytes, 64B swizzle) and the blocked scale tiles
  static int make_maps(const uint8_t* wq, const uint8_t* w_sf, int N, int K, CUtensorMap* tm_w, CUtensorMap* tm_sf) {
    {
      const uint64_t dims[2] = {(uint64_t)K / 2, (uint64_t)N};
      const uint64_t str[1] = {(uint64_t)K / 2};
      const uint32_t box[2] = {64, 128};
      int rc = make_tmap(tm_w, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, wq, dims, str, box, CU_TENSOR_MAP_SWIZZLE_64B);
      if (rc) return rc;
    }
    const uint64_t dims[2] = {128, (uint64_t)ceil_div(N, tsg::ROWS) * (uint64_t)ceil_div(K / 16, 4)};
    const uint64_t str[1] = {512};
    const uint32_t box[2] = {128, 2};
    return make_tmap(tm_sf, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, w_sf, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE);
  }
  __device__ static __forceinline__ uint32_t w_tx_bytes(const tsg::Params&) { return W_BYTES + AUX_BYTES; }
  __device__ static __forceinline__ void issue_w(const CUtensorMap* tm_w, const CUtensorMap* tm_sf, const tsg::Params& p,
                                                 uint8_t* w_dst, uint8_t* aux_dst, uint64_t* bar, int n_tile, int kc,
                                                 uint64_t policy) {
    tma_load_2d(w_dst, tm_w, bar, kc * 64, n_tile * tsg::ROWS, policy);
    // two consecutive blocked scale tiles (128 rows x 4 scales each = 64 k per tile): the blocked scale tensor is a
    // [row block][column block] array of contiguous 512-byte tiles = a 2-D tensor of 128 words x tiles
    tma_load_2d(aux_dst, tm_sf, bar, 0, n_tile * p.aux_col_blocks + kc * 2, policy);
  }
  // grouped kernels: the 128 weight rows from `row` of the [E * N, K / 2] map of all experts' weights, and their scale
  // tiles at row block row / 128 of the blocked [E * N, K / 16] scales.  Expert e's n-tile t is row e * N + 128 t, so
  // this is row block e * N / 128 + t: the launcher requires N % 128 == 0, which is also what keeps every expert's
  // scales in whole 128-row blocks of one blocked tensor
  __device__ static __forceinline__ void issue_w_rows(const CUtensorMap* tm_w, const CUtensorMap* tm_sf,
                                                      const tsg::Params& p, uint8_t* w_dst, uint8_t* aux_dst,
                                                      uint64_t* bar, int row, int kc, uint64_t policy) {
    tma_load_2d(w_dst, tm_w, bar, kc * 64, row, policy);
    tma_load_2d(aux_dst, tm_sf, bar, 0, (row / tsg::ROWS) * p.aux_col_blocks + kc * 2, policy);
  }
  // the thread's two fragment rows: bytes 8kk .. 8kk+7 of each (k16 step kk: byte 8kk + t holds k pair 16kk + 2t,
  // byte 8kk + 4 + t the pair 8 further), and the eight block scales of each row, decoded once per chunk: s2[h][j] =
  // bf16x2 of (scale of step 2j, scale of step 2j + 1) * 2^66
  struct Raw {
    uint2 v[2][8];
    uint32_t s2[2][4];
  };
  __device__ static __forceinline__ void load(const tsg::Params&, uint32_t w_smem, uint32_t aux_smem, int row_lo, int,
                                              Raw& raw) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = row_lo + 8 * h;
      const uint32_t sc_off = (uint32_t)(r & 31) * 16u + (uint32_t)(r >> 5) * 4u;
      const uint32_t sc[2] = {tsg::lds32(aux_smem + sc_off), tsg::lds32(aux_smem + 512 + sc_off)};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        // scale bytes 2j, 2j + 1 at bf16 bits 10:4 of each half = scale * 2^-120, then two exact multiplies
        const uint32_t bits = __byte_perm(sc[j >> 1], 0u, (j & 1) ? 0x4342u : 0x4140u) << 4;
        __nv_bfloat162 s2 = *reinterpret_cast<const __nv_bfloat162*>(&bits);
        s2 = __hmul2(__hmul2(s2, __nv_bfloat162(__ushort_as_bfloat16(0x7F00), __ushort_as_bfloat16(0x7F00))),
                     __nv_bfloat162(__ushort_as_bfloat16(0x5D00), __ushort_as_bfloat16(0x5D00)));   // * 2^127 * 2^59
        raw.s2[h][j] = *reinterpret_cast<const uint32_t*>(&s2);
      }
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        const uint32_t off = (uint32_t)r * 64u + kk * 8;
        raw.v[h][kk] = tsg::lds64(w_smem + (off ^ (((off >> 7) & 3) << 4)));  // undo the TMA 64B swizzle
      }
    }
  }
  __device__ static __forceinline__ uint32_t deq(uint32_t byte, __nv_bfloat162 s2) {
    const uint32_t hh = (byte | (byte << 12)) & 0x000F000Fu;   // even k nibble at bits 3:0, odd k at 19:16
    const uint32_t bits = (hh * 0x1040u) & 0x81C081C0u;         // sign | e1 e0 m at bf16 bits 15 | 8:6 = value * 2^-126
    __nv_bfloat162 x = *reinterpret_cast<const __nv_bfloat162*>(&bits);
    x = __hmul2(x, s2);
    return *reinterpret_cast<uint32_t*>(&x);
  }
  __device__ static __forceinline__ void frag(const tsg::Params&, const Raw& raw, int kk, uint32_t (&a)[4]) {
    const int t = threadIdx.x & 3;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      // the decoded scale of the 16-k block of step kk, in both halves
      const uint32_t s_bits = __byte_perm(raw.s2[h][kk >> 1], 0u, (kk & 1) ? 0x3232u : 0x1010u);
      const __nv_bfloat162 s2 = *reinterpret_cast<const __nv_bfloat162*>(&s_bits);
      a[h] = deq((raw.v[h][kk].x >> (8 * t)) & 0xFFu, s2);
      a[h + 2] = deq((raw.v[h][kk].y >> (8 * t)) & 0xFFu, s2);
    }
  }
};

}  // namespace nvf4w
}  // namespace ao
