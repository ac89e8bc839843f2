// Persistent stream-K GEMM on Hopper wgmma (sm_90a) for every quantized linear of the library.
//
//   Y[M,N] = X[M,K] * W^[N,K]^T (+bias),   W^ = the weights, dequantised in-kernel where the format needs it
//
// Swap-AB: 128 weight rows of a tile are the wgmma M dimension (two consumer warpgroups of 64 rows each), the tokens
// are the wgmma N dimension (N_MMA = 16..128).  A format policy (Fmt) decides how the weights reach the tensor core:
//   * register-A (Fmt::SS == false): int4 tinygemm, nvfp4, mxfp8 weights.  Each consumer thread loads the packed
//     weights of its two fragment rows straight from the TMA-filled stage and dequantises them into the bf16 A
//     fragment of wgmma.m64nNk16 (4 x bf16x2 per k16 step); the activations (bf16) are the shared-memory B operand
//   * shared-memory A (Fmt::SS == true): int8 x int8 -> s32 and e4m3 x e4m3 -> f32 (wgmma k32), both operands are
//     the TMA tiles themselves
// Roles (384 threads): warpgroup 0 = one TMA producer warp (weights first: they never depend on the previous kernel;
// activations after griddepcontrol.wait), warpgroups 1 and 2 = consumers (dequant, wgmma, epilogue).  A stage holds
// one 128-k chunk: weights + scales (wfull) and the activation tile (xfull); the 8 consumer warps hand it back
// (sempty) once the wgmmas that read it have completed.  The wgmmas of chunk i run while chunk i+1 is dequantised.
//
// Work split (streamk.cuh): the (tile, chunk) units are split evenly over the CTAs; the accumulator of a segment lives
// in registers and is finished by the consumers right after the segment's last chunk (FULL: outputs, CONTRIB: publish
// the partial + flag, OWNER: add the contributors' partials in CTA order, then outputs).
#pragma once
#include <cuda_bf16.h>

#include "common.h"
#include "ptx.cuh"
#include "streamk.cuh"
#include "wgmma.cuh"

namespace ao {
namespace tsg {

using streamk::ROWS;
constexpr int KCHUNK = 128;
constexpr int NUM_THREADS = 384;
constexpr int CONSUMER_WARPS = 8;
constexpr int SMEM_BUDGET = 200 * 1024;   // of the 227 KB a block may use on H100: one CTA per SM
constexpr int MAX_STAGES = 12;

// Epilogue arithmetic, per kind (must stay what each format's reference computes, see Params)
enum Epi { EPI_FLOAT = 0, EPI_I8 = 1, EPI_F8 = 2 };

struct Params {
  const __nv_bfloat16* bias;
  const float* row_scale;   // EPI_FLOAT: optional per-token scale [M]; EPI_I8 / EPI_F8: the activation scale [M]
  const float* out_scale;   // EPI_FLOAT: optional device scalar, or (out_scale_per_row) one value per output feature
  const float* out_scale2;  // EPI_FLOAT: optional second device scalar multiplied into out_scale (nvfp4 a_pts * b_pts)
  int out_scale_per_row;
  int acc_exp2;             // the accumulators hold the result * 2^-acc_exp2 (format policy folds a power of two into
                            // its dequant multiply); undone in the epilogue together with out_scale
  const float* w_scale;     // EPI_I8 / EPI_F8: per-output-feature weight scale [N]
  int epi;
  __nv_bfloat16* y;         // [M, N_out]
  int32_t* i32_out;         // EPI_I8: raw int32 accumulators [M, N] instead of y
  float* ws_partial;        // [grid][N_MMA*128]   CTA b's CONTRIB partial (streamk.cuh)
  unsigned int* ws_flag;    // [grid]              CTA b's partial is published
  int M, N, N_out, K, group_size;
  int n_tiles, m_blocks, KT;   // KT = chunks of 128 k
  int aux_col_blocks;          // blocked block-scale layouts: 4-scale column blocks per 128-row block
};

template <class Fmt, int N_MMA>
struct Cfg {
  static constexpr int X_BYTES = N_MMA * KCHUNK * Fmt::X_ELEM_BYTES;   // activation tile of one chunk
  static constexpr int X_ATOMS = Fmt::X_ELEM_BYTES;                    // 128-byte-wide swizzle atoms per chunk
  static constexpr int AUX_SLOT = (Fmt::AUX_BYTES + 1023) & ~1023;
  static constexpr int STAGE_BYTES = Fmt::W_BYTES + AUX_SLOT + X_BYTES;
  static constexpr int STAGES_FIT = SMEM_BUDGET / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT > MAX_STAGES ? MAX_STAGES : STAGES_FIT;
  static_assert(STAGES >= 2, "stage does not fit");
  static constexpr int BAR_OFF = STAGES * STAGE_BYTES;
  static constexpr int BAR_BYTES = 3 * STAGES * 8;   // wfull, xfull, sempty per stage
  static constexpr size_t SMEM_BYTES = (size_t)BAR_OFF + BAR_BYTES + 1024;   // + the 1024-byte alignment of the base
};

__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint2 lds64(uint32_t addr) {
  uint2 v;
  asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint32_t lds16(uint32_t addr) {
  unsigned short v;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(addr));
  return v;
}

// Fmt policy:
//   SS, PROMOTE (SS only: sum each chunk's wgmmas into the fp32 registers), X_ELEM_BYTES (2: bf16 activations,
//   1: 8-bit), W_BYTES, AUX_BYTES (per stage)
//   static void issue_w(tm_w, tm_aux, p, w smem dst, aux smem dst, full barrier, n_tile, kc, policy)  (one thread)
//   static uint32_t w_tx_bytes(p)
//   SS:  static void mma(acc, w smem, x smem, wg, scale_d)          the 4 k32 wgmmas of a chunk for rows 64wg..
//   RA:  struct Raw; static void load(p, w smem, aux smem, row_lo, lane, Raw&)   rows row_lo and row_lo + 8
//        static void frag(p, raw, kk, a[4])                        bf16 A fragment of k16 step kk (0..7)
template <class Fmt, int N_MMA>
__global__ void __launch_bounds__(NUM_THREADS, 1)
ts_gemm_kernel(const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_aux,
               const __grid_constant__ CUtensorMap tm_x, const Params p) {
  using C = Cfg<Fmt, N_MMA>;
  using MMA = Wgmma<N_MMA>;
  constexpr int S = C::STAGES;
  constexpr int NACC = N_MMA / 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::BAR_OFF);
  uint64_t* wfull = bars;        // [S] weights + scales landed
  uint64_t* xfull = wfull + S;   // [S] activation tile landed
  uint64_t* sempty = xfull + S;  // [S] the 8 consumer warps are done with the stage

  // warp and warpgroup indices through a shuffle: the compiler then knows that the role branches below are
  // warp-uniform and warpgroup-uniform (wgmma in code it must treat as divergent is serialised)
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const int wgi = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
  const int G = gridDim.x, b = blockIdx.x;
  const long long U = (long long)p.n_tiles * p.m_blocks * p.KT;
  const int u0 = streamk::unit_begin(b, U, G), u1 = streamk::unit_begin(b + 1, U, G);
  const int nunits = u1 - u0;
  const streamk::Walk walk(u0, nunits, p.KT);
  auto tile_of = [&](int i) { return (u0 + i) / p.KT; };
  auto kc_of = [&](int i) { return (u0 + i) % p.KT; };
  auto stage = [&](int s) { return smem + (size_t)s * C::STAGE_BYTES; };

  if (threadIdx.x == 0) {
    for (int i = 0; i < S; ++i) {
      mbar_init(&wfull[i], 1);
      mbar_init(&xfull[i], 1);
      mbar_init(&sempty[i], CONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tm_w);
    tma_prefetch_desc(&tm_aux);
    tma_prefetch_desc(&tm_x);
  }
  __syncthreads();
  pdl_launch_dependents();

  const int seg_last = walk.nseg - 1;
  const bool last_is_owner = walk.seg_kind(seg_last) == streamk::SEG_OWNER;

  if (wgi == 0) {
    if (warp != 0) goto done;
    // ------------------------------------------------------------ TMA producer
    const uint64_t pol_w = policy_evict_first();
    const uint64_t pol_x = policy_evict_last();
    auto issue_w = [&](int i) {
      const int s = i % S;
      uint8_t* st = stage(s);
      mbar_expect_tx(&wfull[s], Fmt::w_tx_bytes(p));
      Fmt::issue_w(&tm_w, &tm_aux, p, st, st + Fmt::W_BYTES, &wfull[s], tile_of(i) % p.n_tiles, kc_of(i), pol_w);
    };
    auto issue_x = [&](int i) {
      const int s = i % S;
      uint8_t* xs = stage(s) + Fmt::W_BYTES + C::AUX_SLOT;
      const int m0 = (tile_of(i) / p.n_tiles) * N_MMA;
      mbar_expect_tx(&xfull[s], C::X_BYTES);
#pragma unroll
      for (int a = 0; a < C::X_ATOMS; ++a)
        tma_load_2d(xs + a * (N_MMA * 128), &tm_x, &xfull[s], kc_of(i) * KCHUNK + a * (KCHUNK / C::X_ATOMS), m0, pol_x);
    };
    const int pre = nunits < S ? nunits : S;
    for (int i = 0; i < pre; ++i) {
      if (elect_one()) issue_w(i);   // weights never depend on the previous kernel
      __syncwarp();
    }
    pdl_wait();   // activations are the previous kernel's output
    for (int i = 0; i < pre; ++i) {
      if (elect_one()) issue_x(i);
      __syncwarp();
    }
    for (int i = S; i < nunits; ++i) {
      mbar_wait(&sempty[i % S], ((i / S) & 1) ^ 1);
      if (elect_one()) {
        issue_w(i);
        issue_x(i);
      }
      __syncwarp();
    }
  } else {
    // ------------------------------------------------------------ consumers: warpgroup wg owns rows 64wg .. 64wg+63
    const int wg = wgi - 1, wq = warp & 3;
    const int g = lane >> 2, t = lane & 3;
    const int row_lo = wg * 64 + wq * 16 + g;   // fragment rows row_lo and row_lo + 8 (accumulator rows as well)
    pdl_wait();   // outputs, workspace and scales belong to the previous kernel's stream order

    uint32_t acc[NACC];
    uint32_t a[8][4];   // register-A formats: the bf16 fragments of one chunk (read by the wgmmas until they complete)
    int pending = -1;   // stage whose wgmmas may still be in flight
    auto release = [&](int s) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&sempty[s]);
    };

    // ---- epilogue of segment `seg` from v = the accumulator, once its wgmmas completed (wait_group 0 + operand fence,
    // in warpgroup-uniform code: no wgmma is in flight while the epilogue's divergent code touches it).  Value
    // j = 4q + 2h + c of this thread is (weight row row_lo + 8h, token 8q + 2t + c) of the tile (wgmma m64nN fragment)
    auto epilogue = [&](int seg, uint32_t (&v)[NACC]) {
      const int tile = walk.seg_tile(seg);
      const int kind = walk.seg_kind(seg);
      const int n_tile = tile % p.n_tiles, m_blk = tile / p.n_tiles;
      const int m0 = m_blk * N_MMA;
      if (kind == streamk::SEG_CONTRIB) {
        // publish the partial (column-major slot: word (token j, row r) at j * 128 + r), then one gpu-scope release
        uint32_t* slot = reinterpret_cast<uint32_t*>(p.ws_partial) + (size_t)b * (N_MMA * ROWS);
#pragma unroll
        for (int q = 0; q < NACC / 4; ++q)
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              const int col = 8 * q + 2 * t + c, r = row_lo + 8 * h;
              if (m0 + col < p.M) __stcg(&slot[col * ROWS + r], v[4 * q + 2 * h + c]);
            }
        asm volatile("bar.sync 1, 256;" ::: "memory");   // all 128 rows stored (cta-scope order) ...
        if (warp == 4 && lane == 0) streamk::st_release_u32(p.ws_flag + b, 1u);   // ... then one gpu-scope release
        return;
      }
      if (kind == streamk::SEG_OWNER) {
        // own partial + the partials of CTAs b+1 .. b_last in that order (fixed: bit-reproducible run to run)
        const int b_last = streamk::cta_of_unit((long long)tile * p.KT + p.KT - 1, U, G);
        for (int c = b + 1; c <= b_last; ++c)
          while (streamk::ld_acquire_u32(p.ws_flag + c) == 0u) __nanosleep(64);
#pragma unroll 1
        for (int c = b + 1; c <= b_last; ++c) {
          const uint32_t* slot = reinterpret_cast<const uint32_t*>(p.ws_partial) + (size_t)c * (N_MMA * ROWS);
#pragma unroll
          for (int q = 0; q < NACC / 4; ++q)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int cc = 0; cc < 2; ++cc) {
                const int col = 8 * q + 2 * t + cc, r = row_lo + 8 * h, j = 4 * q + 2 * h + cc;
                if (m0 + col < p.M) {
                  const uint32_t o = __ldcg(slot + col * ROWS + r);
                  if (p.epi == EPI_I8) v[j] = (uint32_t)((int32_t)v[j] + (int32_t)o);
                  else v[j] = __float_as_uint(__uint_as_float(v[j]) + __uint_as_float(o));
                }
              }
        }
      }
      // outputs
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int n = n_tile * ROWS + row_lo + 8 * h;
        if (n >= p.N_out) continue;
        const float bias = p.bias ? __bfloat162float(p.bias[n]) : 0.f;
        float osc = 1.f, sw = 1.f;
        if (p.epi == EPI_FLOAT) {
          osc = (p.out_scale ? (p.out_scale_per_row ? p.out_scale[n] : *p.out_scale) : 1.f);
          if (p.out_scale2) osc *= *p.out_scale2;
          osc *= __int_as_float((127 + p.acc_exp2) << 23);
        } else {
          sw = p.w_scale ? p.w_scale[n] : 1.f;
        }
#pragma unroll
        for (int q = 0; q < NACC / 4; ++q)
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int m = m0 + 8 * q + 2 * t + c;
            if (m >= p.M) continue;
            const uint32_t raw = v[4 * q + 2 * h + c];
            __nv_bfloat16* dst = p.y ? p.y + (size_t)m * p.N_out + n : nullptr;
            if (p.epi == EPI_FLOAT) {
              float x = __uint_as_float(raw);
              if (p.row_scale) x *= p.row_scale[m];
              *dst = __float2bfloat16_rn(x * osc + bias);
            } else if (p.epi == EPI_I8) {
              if (p.i32_out) {
                p.i32_out[(size_t)m * p.N_out + n] = (int32_t)raw;
              } else {
                // int8 reference: bf16 round between the activation and the weight scale
                const float x = __bfloat162float(__float2bfloat16_rn((float)(int32_t)raw * p.row_scale[m]));
                *dst = __float2bfloat16_rn(x * sw + bias);
              }
            } else {
              *dst = __float2bfloat16_rn(__uint_as_float(raw) * (p.row_scale[m] * sw) + bias);
            }
          }
      }
    };

    int i = 0;
    for (int seg = 0; seg < walk.nseg; ++seg) {
      const int cnt = walk.seg_count(seg);
      for (int c = 0; c < cnt; ++c, ++i) {
        const uint32_t scale_d = c > 0;   // the first wgmma of a segment overwrites the accumulator
        const int s = i % S;
        const uint32_t ph = (i / S) & 1;
        uint8_t* st = stage(s);
        const uint32_t w_s = smem_u32(st), aux_s = w_s + Fmt::W_BYTES, x_s = aux_s + C::AUX_SLOT;
        mbar_wait(&wfull[s], ph);
        if constexpr (Fmt::PROMOTE) {
          // e4m3: a chain of wgmmas accumulates in the tensor core's reduced-precision adder; each chunk's four k32
          // wgmmas go to a fresh accumulator that is added to the fp32 registers here (fp32 accuracy across K)
          mbar_wait(&xfull[s], ph);
          uint32_t part[NACC];
          wgmma_fence();
          Fmt::template mma<N_MMA>(part, w_s, x_s, wg, 0u);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_fence_operand(part);
          release(s);
#pragma unroll
          for (int j = 0; j < NACC; ++j)
            acc[j] = scale_d ? __float_as_uint(__uint_as_float(acc[j]) + __uint_as_float(part[j])) : part[j];
          continue;
        } else if constexpr (Fmt::SS) {
          mbar_wait(&xfull[s], ph);
          wgmma_fence_operand(acc);
          wgmma_fence();
          Fmt::template mma<N_MMA>(acc, w_s, x_s, wg, scale_d);
        } else {
          typename Fmt::Raw raw;
          Fmt::load(p, w_s, aux_s, row_lo, lane, raw);
          // the previous chunk's wgmmas still read a[]: they complete (their stage goes back) before a[] is rewritten,
          // and the operand fence keeps the old fragment registers alive up to that point.  The wgmmas overlap this
          // chunk's weight loads and barrier waits, not its dequant arithmetic
          wgmma_wait<0>();
#pragma unroll
          for (int kk = 0; kk < 8; ++kk) wgmma_fence_operand(a[kk]);
          if (pending >= 0) release(pending);
          pending = -1;
#pragma unroll
          for (int kk = 0; kk < 8; ++kk) Fmt::frag(p, raw, kk, a[kk]);
          mbar_wait(&xfull[s], ph);
          wgmma_fence_operand(acc);
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < 8; ++kk) {
            // k16 step kk of the bf16 B tile: atom kk / 4 (64 k each), 32 bytes per step inside the 128-byte row
            const uint64_t bd = wgmma_desc_k_sw128(x_s + (kk >> 2) * (N_MMA * 128) + (kk & 3) * 32);
            MMA::ra_bf16(acc, a[kk], bd, kk == 0 ? scale_d : 1u);
          }
        }
        wgmma_commit();
        wgmma_fence_operand(acc);
        wgmma_wait<1>();   // the wgmmas of the previous chunk are done: its stage goes back to the producer
        if (pending >= 0) release(pending);
        pending = s;
      }
      wgmma_wait<0>();
      wgmma_fence_operand(acc);
      if (pending >= 0) release(pending);
      pending = -1;
      epilogue(seg, acc);
    }
  }

done:
  __syncthreads();
  if (last_is_owner && warp == 4) {
    // every consumer has read the contributors' partials: re-arm their flags for the next launch
    const int b_last = streamk::cta_of_unit((long long)walk.seg_tile(seg_last) * p.KT + p.KT - 1, U, G);
    for (int c = b + 1 + lane; c <= b_last; c += 32) p.ws_flag[c] = 0u;
  }
}

// ------------------------------------------------------------------------------------------------ host side
// Grid choice + workspace carve-up shared by the launchers of this kernel.
//   * at most one CTA per SM (the stage ring takes most of the shared memory): the grid stays within the resident
//     capacity, which the owner protocol needs for forward progress (streamk.cuh)
//   * never fewer than `min_units` chunks per CTA: splitting a tile over more CTAs shortens the streaming phase but
//     lengthens the owner's gather
template <class Fmt, int N_MMA>
inline int launch_gemm(Params& p, const CUtensorMap& tm_w, const CUtensorMap& tm_aux, const CUtensorMap& tm_x,
                       void* ws, size_t ws_bytes, const char* what, cudaStream_t stream) {
  using C = Cfg<Fmt, N_MMA>;
  const long long units = (long long)p.n_tiles * p.m_blocks * p.KT;
  int grid = sm_count();
  const int min_units = ts_min_units() ? ts_min_units() : 4;
  if (units / min_units < grid) grid = units / min_units > 0 ? (int)(units / min_units) : 1;
  const size_t need = streamk::WS_PARTIAL_OFF + (size_t)grid * N_MMA * ROWS * 4;
  if (!ws || ws_bytes < need || (size_t)grid * 4 > streamk::WS_FLAGS_BYTES)
    return fail(AO_ERR_WORKSPACE, "%s: workspace too small (%zu < %zu)", what, ws_bytes, need);
  p.ws_flag = reinterpret_cast<unsigned int*>(ws);
  p.ws_partial = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(ws) + streamk::WS_PARTIAL_OFF);
  auto kern = ts_gemm_kernel<Fmt, N_MMA>;
  AO_CUDA_CHECK(ensure_dynamic_smem(reinterpret_cast<const void*>(kern), C::SMEM_BYTES));
  AO_CUDA_CHECK(launch(kern, dim3(grid), dim3(NUM_THREADS), C::SMEM_BYTES, stream, pdl_enabled(), tm_w, tm_aux, tm_x, p));
  return AO_OK;
}

}  // namespace tsg
}  // namespace ao
