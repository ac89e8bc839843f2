// int4 weight-only linear on the tinygemm "tile_packed_to_4d" format, sm_90a.
//
//   Y[M,N] = X[M,K] * W^[N,K]^T (+bias),  W^ = bf16((q-8)*s + z)   (group-wise s,z)
//
// Replaces aten._weight_int4pack_mm as called from the reference handler
// (torchao/quantization/quantize_/workflows/int4/int4_tile_packed_to_4d_tensor.py:243-299).
// The GEMM itself is the persistent wgmma kernel of ts_gemm.cuh; this file supplies the int4 format policy (how a
// 128-row x 128-k chunk is fetched and turned into bf16 wgmma A fragments) and the C entry point.
//
// qdata layout (int32 [N/8][K/128][32][4], inner_k_tiles = 8), word `wd` of lane `t`:
//   row n = 8*n8 + t/4;  k0 = 128*ko + 32*wd + 2*(t%4);
//   bits [4e,4e+4)   = q[n, k0 + 8e]      e = 0..3
//   bits [16+4e, ..) = q[n, k0 + 8e + 1]
// which is the m16n8k16 fragment layout: lane t of n8 tile j holds, for its row, exactly the k pairs that lane t of
// the wgmma A fragment needs (k 2(t%4) + {0,1} and + 8 of every k16 step).  A 128-row chunk is 16 runs of 512 B,
// fetched by ONE 3-D TMA box {32 words, 4 row-pairs, 16 n8-tiles} with 128-byte swizzle; a consumer thread reads
// the 16 bytes of its lane in the n8 tiles of its two fragment rows (conflict-free ld.shared.v4).
#include <cuda_bf16.h>
#include <stdlib.h>

#include "common.h"
#include "ptx.cuh"
#include "ts_gemm.cuh"

namespace ao {
namespace int4k {

using tsg::KCHUNK;
using tsg::ROWS;

// (128+q) bf16x2 bits -> bf16x2 of fma(q-8, s, z), single rounding, = oracle W^.
__device__ __forceinline__ uint32_t deq_pair(uint32_t magic_bits, __nv_bfloat162 s2, __nv_bfloat162 z2) {
  const __nv_bfloat162 c136 = __floats2bfloat162_rn(136.f, 136.f);
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&magic_bits);
  v = __hsub2(v, c136);    // exact: (128+q) - 136 = q - 8
  v = __hfma2(v, s2, z2);  // bf16(fma(q-8, s, z))
  return *reinterpret_cast<uint32_t*>(&v);
}

struct Int4Fmt {
  static constexpr bool SS = false;
  static constexpr bool DECODE_2CTA = true;
  static constexpr bool PROMOTE = false;
  static constexpr int X_ELEM_BYTES = 2;
  static constexpr int W_BYTES = ROWS * KCHUNK / 2;   // 8 KiB of 4-bit weights per chunk
  static constexpr int AUX_BYTES = 2048;              // (s, z) pairs: up to 4 groups x 128 rows x 4 B
  static constexpr int EPI = tsg::EPI_FLOAT;
  static constexpr int ACC_EXP2 = 0;
  static constexpr int MAX_N_MMA = 128;
  // the packed weights ({32 words, 4 row-pairs, 16 n8-tiles} box, 128-byte swizzle) and the (scale, zero) pairs
  static int make_maps(const int32_t* qdata, const uint16_t* sz, int N, int K, int g, CUtensorMap* tm_w,
                       CUtensorMap* tm_sz) {
    const int KT = K / 128;
    {
      const uint64_t dims[3] = {32, (uint64_t)4 * KT, (uint64_t)N / 8};
      const uint64_t str[2] = {128, (uint64_t)KT * 512};
      const uint32_t box[3] = {32, 4, 16};
      int rc = make_tmap(tm_w, CU_TENSOR_MAP_DATA_TYPE_INT32, 3, qdata, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B);
      if (rc) return rc;
    }
    const int gpc = g <= 128 ? 128 / g : 1;
    const uint64_t dims[2] = {(uint64_t)N, (uint64_t)K / g};
    const uint64_t str[1] = {(uint64_t)N * 4};
    const uint32_t box[2] = {128, (uint32_t)gpc};
    return make_tmap(tm_sz, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, sz, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE);
  }
  __device__ static __forceinline__ uint32_t w_tx_bytes(const tsg::Params& p) {
    const int gpc = p.group_size <= KCHUNK ? KCHUNK / p.group_size : 1;
    return W_BYTES + gpc * 512;
  }
  __device__ static __forceinline__ void issue_w(const CUtensorMap* tm_w, const CUtensorMap* tm_sz,
                                                 const tsg::Params& p, uint8_t* w_dst, uint8_t* aux_dst,
                                                 uint64_t* bar, int n_tile, int kc, uint64_t policy) {
    tma_load_3d(w_dst, tm_w, bar, 0, 4 * kc, n_tile * (ROWS / 8), policy);
    tma_load_2d(aux_dst, tm_sz, bar, n_tile * ROWS, (kc * KCHUNK) / p.group_size, policy);
  }
  // the thread's two fragment rows: 16 bytes (4 tinygemm words = 128 k) each, and the (s, z) pair of every 32-k word
  struct Raw {
    uint4 v[2];
    uint32_t sz[2][4];
  };
  __device__ static __forceinline__ void load(const tsg::Params& p, uint32_t w_smem, uint32_t aux_smem, int row_lo,
                                              int lane, Raw& raw) {
    const int gshift = p.group_size == 32 ? 0 : (p.group_size == 64 ? 1 : 2);  // 32-k word -> group of the chunk
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = row_lo + 8 * h;
      const uint32_t off = (uint32_t)(r >> 3) * 512u + (uint32_t)lane * 16u;
      raw.v[h] = tsg::lds128(w_smem + (off ^ (((off >> 7) & 7) << 4)));  // undo the TMA 128B swizzle
#pragma unroll
      for (int w = 0; w < 4; ++w) raw.sz[h][w] = tsg::lds32(aux_smem + r * 4 + (w >> gshift) * 512);
    }
  }
  // k16 step kk = half (kk & 1) of tinygemm word kk / 2: a[0] / a[1] = rows lo / hi at k 2t + {0,1} (nibble e),
  // a[2] / a[3] = the same rows at k + 8 (nibble e + 1)
  __device__ static __forceinline__ void frag(const tsg::Params&, const Raw& raw, int kk, uint32_t (&a)[4]) {
    uint32_t magic = 0x43004300u;
    asm volatile("" : "+r"(magic));  // keep it in a register
    const int wd = kk >> 1, e0 = 2 * (kk & 1);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t sz = raw.sz[h][wd];
      const uint32_t s_bits = __byte_perm(sz, sz, 0x1010);
      const uint32_t z_bits = __byte_perm(sz, sz, 0x3232);
      const __nv_bfloat162 s2 = *reinterpret_cast<const __nv_bfloat162*>(&s_bits);
      const __nv_bfloat162 z2 = *reinterpret_cast<const __nv_bfloat162*>(&z_bits);
      const uint32_t word = wd == 0 ? raw.v[h].x : wd == 1 ? raw.v[h].y : wd == 2 ? raw.v[h].z : raw.v[h].w;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        // bf16x2 of 128+q = ((word >> 4e) & 0x000F000F) | 0x43004300 as ONE lop3
        uint32_t m;
        asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(m) : "r"(word >> (4 * (e0 + e))), "r"(0x000F000Fu), "r"(magic));
        a[h + 2 * e] = deq_pair(m, s2, z2);
      }
    }
  }
};

// ---------------------------------------------------------------------------------------
// Reference-grade CUDA-core kernel (impl = 2): one warp per weight row, lanes stride over
// k-tiles, fp32 accumulation.  Slow; used as an on-device cross-check and for odd shapes.
template <int MT>
__global__ void int4_linear_simple_kernel(const __nv_bfloat16* __restrict__ x,
                                          const int32_t* __restrict__ qdata,
                                          const __nv_bfloat16* __restrict__ sz,
                                          const __nv_bfloat16* __restrict__ bias,
                                          __nv_bfloat16* __restrict__ y, int M, int N, int N_out,
                                          int K, int g, int ldx) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x * 8 + warp;
  const int m0 = blockIdx.y * MT;
  if (n >= N) return;
  const int KT = K / 128;
  float acc[MT];
#pragma unroll
  for (int m = 0; m < MT; ++m) acc[m] = 0.f;
  for (int ko = lane; ko < KT; ko += 32) {
    const uint4* wp = reinterpret_cast<const uint4*>(qdata + (((size_t)(n >> 3) * KT + ko) * 32 + (n & 7) * 4) * 4);
    for (int tq = 0; tq < 4; ++tq) {
      const uint4 v = wp[tq];
      const uint32_t words[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int wd = 0; wd < 4; ++wd) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int k = ko * 128 + 32 * wd + 2 * tq + 8 * e + h;
            const int q = (words[wd] >> (4 * e + 16 * h)) & 15;
            const size_t gi = ((size_t)(k / g) * N + n) * 2;
            const __nv_bfloat16 wv = __hfma(__int2bfloat16_rn(q - 8), sz[gi], sz[gi + 1]);
            const float wf = __bfloat162float(wv);
#pragma unroll
            for (int m = 0; m < MT; ++m)
              if (m0 + m < M) acc[m] += __bfloat162float(x[(size_t)(m0 + m) * ldx + k]) * wf;
          }
        }
      }
    }
  }
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    float v = acc[m];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0 && m0 + m < M && n < N_out)
      y[(size_t)(m0 + m) * N_out + n] = __float2bfloat16_rn(v + (bias ? __bfloat162float(bias[n]) : 0.f));
  }
}

}  // namespace int4k
}  // namespace ao

extern "C" int ao_int4_tilepacked_linear_strided(const uint16_t* x, int ldx, int M, int K, const int32_t* qdata,
                                                 const uint16_t* scale_and_zero, int group_size, int N,
                                                 const uint16_t* bias, uint16_t* y, int N_out,
                                                 void* workspace, size_t workspace_bytes, int impl,
                                                 void* stream) {
  using namespace ao;
  AO_REQUIRE(M >= 0 && K > 0 && N > 0, "int4 linear: bad sizes M=%d K=%d N=%d", M, K, N);
  AO_REQUIRE(K % 1024 == 0, "int4 linear: K=%d must be a multiple of 1024 (format pads K)", K);
  AO_REQUIRE(N % 8 == 0, "int4 linear: N=%d must be a multiple of 8", N);
  AO_REQUIRE(N_out > 0 && N_out <= N, "int4 linear: N_out=%d out of range (N=%d)", N_out, N);
  AO_REQUIRE(group_size == 32 || group_size == 64 || group_size == 128 || group_size == 256,
             "int4 linear: group_size=%d not in {32,64,128,256}", group_size);
  AO_REQUIRE(ldx >= K && ldx % 8 == 0, "int4 linear: ldx=%d must be >= K=%d and a multiple of 8", ldx, K);
  if (M == 0) return AO_OK;
  AO_REQUIRE(x && qdata && scale_and_zero && y, "int4 linear: null pointer");
  AO_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0, "int4 linear: x must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (impl == 2) {
    constexpr int MT = 8;
    dim3 grid(ceil_div(N, 8), ceil_div(M, MT));
    AO_CUDA_CHECK(launch(int4k::int4_linear_simple_kernel<MT>, grid, dim3(256), 0, st, false,
                         reinterpret_cast<const __nv_bfloat16*>(x), qdata,
                         reinterpret_cast<const __nv_bfloat16*>(scale_and_zero),
                         reinterpret_cast<const __nv_bfloat16*>(bias),
                         reinterpret_cast<__nv_bfloat16*>(y), M, N, N_out, K, group_size, ldx));
    return AO_OK;
  }
  CUtensorMap tm_w, tm_sz;
  if (int rc = int4k::Int4Fmt::make_maps(qdata, scale_and_zero, N, K, group_size, &tm_w, &tm_sz)) return rc;
  tsg::Params p{};
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  p.y = reinterpret_cast<__nv_bfloat16*>(y);
  p.M = M; p.N = N; p.N_out = N_out; p.K = K; p.group_size = group_size;
  return tsg::run<int4k::Int4Fmt>(p, tm_w, tm_sz, x, ldx, workspace, workspace_bytes, "int4 linear", st);
}

extern "C" int ao_int4_tilepacked_linear(const uint16_t* x, int M, int K, const int32_t* qdata,
                                         const uint16_t* scale_and_zero, int group_size, int N,
                                         const uint16_t* bias, uint16_t* y, int N_out,
                                         void* workspace, size_t workspace_bytes, int impl,
                                         void* stream) {
  return ao_int4_tilepacked_linear_strided(x, K, M, K, qdata, scale_and_zero, group_size, N, bias, y, N_out, workspace,
                                           workspace_bytes, impl, stream);
}
