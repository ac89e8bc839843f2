// NVFP4 weights (e2m1 pairs, even k in the low nibble; e4m3 block-16 scales in the blocked 128 x 4 tile layout)
// as the register-A operand of ts_gemm.cuh: each consumer thread turns the bytes of its two fragment rows into the
// bf16 wgmma A fragment.  Used by the nvfp4-weight linear and by the nvfp4 x nvfp4 linear.
//
// e2m1 -> bf16 without a table: nibble x = (s e1 e0 m) placed at bf16 bits 15|8:6 is the bf16 number
// value(x) * 2^-126 (denormal for e = 0, which bf16 multiplies handle exactly); ONE exact multiply by
// (block_scale * 2^66) gives value(x) * block_scale * 2^-60, and the 2^60 is taken back out of the fp32 accumulator in the
// epilogue (Params::acc_exp2; power-of-two factors commute with every rounding on the way).  bf16(block_scale * 2^66) =
// (byte << 4) + 0x5D00 for the (always normal, >= 2^-6) e4m3 scale bytes.  The product has at most 6 significant
// bits, so the bf16 A operand is exact.
#pragma once
#include <cuda_bf16.h>

#include "ptx.cuh"
#include "ts_gemm.cuh"

namespace ao {
namespace nvf4w {

struct Nvfp4Fmt {
  static constexpr bool SS = false;
  static constexpr bool PROMOTE = false;
  static constexpr int X_ELEM_BYTES = 2;
  static constexpr int W_BYTES = tsg::ROWS * tsg::KCHUNK / 2;   // 128 rows x 64 bytes, 64-byte swizzle
  static constexpr int AUX_BYTES = 1024;                        // two blocked scale tiles (64 k each)
  static constexpr int ACC_EXP2 = 60;   // the accumulators hold the result * 2^-60 (Params::acc_exp2)
  __device__ static __forceinline__ uint32_t w_tx_bytes(const tsg::Params&) { return W_BYTES + AUX_BYTES; }
  __device__ static __forceinline__ void issue_w(const CUtensorMap* tm_w, const CUtensorMap* tm_sf, const tsg::Params& p,
                                                 uint8_t* w_dst, uint8_t* aux_dst, uint64_t* bar, int n_tile, int kc,
                                                 uint64_t policy) {
    tma_load_2d(w_dst, tm_w, bar, kc * 64, n_tile * tsg::ROWS, policy);
    // two consecutive blocked scale tiles (128 rows x 4 scales each = 64 k per tile): the blocked scale tensor is a
    // [row block][column block] array of contiguous 512-byte tiles = a 2-D tensor of 128 words x tiles
    tma_load_2d(aux_dst, tm_sf, bar, 0, n_tile * p.aux_col_blocks + kc * 2, policy);
  }
  // the thread's two fragment rows: bytes 8kk .. 8kk+7 of each (k16 step kk: byte 8kk + t holds k pair 16kk + 2t,
  // byte 8kk + 4 + t the pair 8 further), and the two scale words (four e4m3 bytes = four 16-k blocks each)
  struct Raw {
    uint2 v[2][8];
    uint32_t sc[2][2];
  };
  __device__ static __forceinline__ void load(const tsg::Params&, uint32_t w_smem, uint32_t aux_smem, int row_lo, int,
                                              Raw& raw) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = row_lo + 8 * h;
      const uint32_t sc_off = (uint32_t)(r & 31) * 16u + (uint32_t)(r >> 5) * 4u;
      raw.sc[h][0] = tsg::lds32(aux_smem + sc_off);
      raw.sc[h][1] = tsg::lds32(aux_smem + 512 + sc_off);
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
      const uint32_t sb = (raw.sc[h][kk >> 2] >> (8 * (kk & 3))) & 0xFFu;   // the 16-k block of step kk
      const uint32_t s_bits = ((sb << 4) + 0x5D00u) * 0x00010001u;          // bf16x2 of scale * 2^66
      const __nv_bfloat162 s2 = *reinterpret_cast<const __nv_bfloat162*>(&s_bits);
      a[h] = deq((raw.v[h][kk].x >> (8 * t)) & 0xFFu, s2);
      a[h + 2] = deq((raw.v[h][kk].y >> (8 * t)) & 0xFFu, s2);
    }
  }
};

// tensor maps of the packed weights (128 rows x 64 bytes, 64B swizzle) and of the blocked scale tiles
inline int make_weight_maps(const uint8_t* wq, const uint8_t* w_sf, int N, int K, CUtensorMap* tm_w, CUtensorMap* tm_sf) {
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

}  // namespace nvf4w
}  // namespace ao
