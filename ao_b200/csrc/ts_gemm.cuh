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
// (sempty) once the wgmmas that read it have completed.  The wgmmas of chunk i overlap chunk i+1's weight loads.
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
constexpr int MAX_STAGES = 12;
// Residency.  Decode tiles (N_MMA <= 32) of the formats with Fmt::DECODE_2CTA fit two CTAs per SM: the next linear's
// CTA (PDL) becomes resident beside the running one and fills its ring with weights during that kernel's tail,
// instead of starting after it on an empty pipeline.  Each CTA then has half of the SM's 228 KB (less the 1 KB the driver reserves per CTA) and 80 registers
// per thread at launch; the producer warpgroup gives registers back to the consumers (setmaxnreg).  Prefill tiles
// keep one CTA per SM and up to 200 KB of ring.
constexpr int SMEM_PER_SM = 228 * 1024, SMEM_RESERVED_PER_CTA = 1024;
template <class Fmt, int N_MMA>
constexpr int ctas_per_sm() { return N_MMA <= 32 && Fmt::DECODE_2CTA ? 2 : 1; }
constexpr int PRODUCER_REGS = 24, CONSUMER_REGS = 104;   // 128 * 24 + 256 * 104 <= 384 * 80

// Epilogue arithmetic, per kind (Fmt::EPI; must stay what each format's reference computes, see Params)
enum Epi { EPI_FLOAT = 0, EPI_I8 = 1, EPI_F8 = 2 };

struct Params {
  const __nv_bfloat16* bias;
  const float* row_scale;   // EPI_FLOAT: optional per-token scale [M]; EPI_I8 / EPI_F8: the activation scale [M]
  const float* out_scale;   // EPI_FLOAT: optional device scalar, or (out_scale_per_row) one value per output feature;
                            // Grouped<Fmt>: one value per expert [E] (nvfp4: the per-expert weight scale)
  // The grouped fields share storage and padding with the dense ones, so Params keeps its 120 bytes: a larger
  // parameter block changed the code ptxas generates for every dense instantiation.
  union {
    const float* out_scale2;  // EPI_FLOAT: optional second device scalar multiplied into out_scale (nvfp4 a_pts * b_pts)
    const int* offs;          // Grouped<Fmt>: [E] on the device, see below (the grouped epilogue never reads out_scale2)
  };
  int out_scale_per_row;
  int grid_forced;          // Grouped<Fmt>: the host grid was forced (ao_b200_debug_set_streamk_ctas): no MIN_UNITS rule
  const float* w_scale;     // EPI_I8 / EPI_F8: per-output-feature weight scale [N]
  __nv_bfloat16* y;         // [M, N_out]
  int32_t* i32_out;         // EPI_I8: raw int32 accumulators [M, N] instead of y
  float* ws_partial;        // [grid][N_MMA*128]   CTA b's CONTRIB partial (streamk.cuh)
  unsigned int* ws_flag;    // [grid]              CTA b's partial is published
  int M, N, N_out, K, group_size;
  int n_tiles, m_blocks, KT;   // KT = chunks of 128 k
  int aux_col_blocks;          // blocked block-scale layouts: 4-scale column blocks per 128-row block
  // Grouped<Fmt> (see Grouped schedule below): expert e < E owns rows [offs[e-1], offs[e]) of x and y (offs[-1] = 0), its
  // weights are rows e*N .. e*N+N-1 of the weight map and its weight scales w_scale[e*N ..]
  int E;
};
static_assert(sizeof(Params) == 120, "Params layout (see above)");

// Grouped schedule (torch._grouped_mm, 2-D x 3-D).  The m-blocks are per expert: ceil(rows_e / N_MMA) blocks of
// N_MMA tokens starting at the expert's first row, so a tile never mixes two experts' weights.  Only the device knows
// offs, so every CTA derives the split from it after griddepcontrol.wait: the tile index stays j * n_tiles + n_tile,
// with j enumerating the (expert, m-block) pairs, U = n_tiles * J * KT and the grid the host heuristic would have
// picked for that U (streamk.cuh, "Device-side grid").
constexpr int MAX_EXPERTS = 1024;   // one row end and one m-block prefix per expert in shared memory
constexpr int MIN_UNITS = 4;        // never fewer chunks per CTA (launch_gemm)

// ts_gemm_kernel<Grouped<Fmt>, N_MMA>: Fmt under the grouped schedule, for a shared-memory A format (fp8) or a
// register-A one (nvfp4).  A wrapper rather than a kernel template parameter, so the dense kernels keep their names and
// their code.
template <class F>
struct Grouped : F {};
template <class F>
struct IsGrouped {
  static constexpr bool value = false;
};
template <class F>
struct IsGrouped<Grouped<F>> {
  static constexpr bool value = true;
};

struct GroupTile {
  int e, row0, row_end;   // the expert, the tile's first row and the expert's end row (rows >= row_end: not stored)
};

// One warp: end[e] = min(M, max(0, offs[0..e])) (each offs[e] clamped into [end[e-1], M]: a malformed offs never
// reaches a row outside [0, M)) and mbp[e] = the m-blocks of experts 0 .. e-1, mbp[E] = J
template <int N_MMA>
__device__ __forceinline__ void grouped_schedule(const Params& p, int* end, int* mbp, int lane) {
  int run_end = 0, run_mb = 0;
  for (int base = 0; base < p.E; base += 32) {
    const int e = base + lane;
    int r = e < p.E ? p.offs[e] : 0;
    r = r > run_end ? r : run_end;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int o = __shfl_up_sync(0xffffffffu, r, d);
      if (lane >= d && o > r) r = o;
    }
    if (r > p.M) r = p.M;
    int start = __shfl_up_sync(0xffffffffu, r, 1);
    if (lane == 0) start = run_end;
    const int mb = e < p.E ? (r - start + N_MMA - 1) / N_MMA : 0;
    int s = mb;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int o = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += o;
    }
    if (e < p.E) {
      end[e] = r;
      mbp[e + 1] = run_mb + s;
    }
    run_end = __shfl_sync(0xffffffffu, r, 31);
    run_mb += __shfl_sync(0xffffffffu, s, 31);
  }
  if (lane == 0) mbp[0] = 0;
}

// The (expert, m-block) pair j < J: the largest e with mbp[e] <= j (an empty expert shares its prefix with the next)
template <int N_MMA>
__device__ __forceinline__ GroupTile group_tile(const int* end, const int* mbp, int E, int j) {
  int lo = 0, hi = E - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (mbp[mid] <= j) lo = mid;
    else hi = mid - 1;
  }
  return {lo, (lo > 0 ? end[lo - 1] : 0) + (j - mbp[lo]) * N_MMA, end[lo]};
}

// The grid of a grouped launch once U is known: what launch_gemm picks for U units, never above the launched grid
// (sized from an upper bound of U), never a CTA without units, no CTA at all when every expert is empty
__device__ __forceinline__ int grouped_grid(int G, long long U, int forced) {
  if (U == 0) return 0;
  const long long cap = forced ? U : (U / MIN_UNITS > 0 ? U / MIN_UNITS : 1);
  return cap < G ? (int)cap : G;
}

template <class Fmt, int N_MMA>
struct Cfg {
  static constexpr int X_BYTES = N_MMA * KCHUNK * Fmt::X_ELEM_BYTES;   // activation tile of one chunk
  static constexpr int X_ATOMS = Fmt::X_ELEM_BYTES;                    // 128-byte-wide swizzle atoms per chunk
  static constexpr int AUX_SLOT = (Fmt::AUX_BYTES + 1023) & ~1023;
  static constexpr int STAGE_BYTES = Fmt::W_BYTES + AUX_SLOT + X_BYTES;
  static constexpr int CTAS = ctas_per_sm<Fmt, N_MMA>();
  // one CTA per SM: a 200 KB ring; two: the CTA's share less its barriers (3 x 8 bytes per stage) and alignment pad
  static constexpr int STAGES_FIT = CTAS == 1 ? 200 * 1024 / STAGE_BYTES
                                              : (SMEM_PER_SM / 2 - SMEM_RESERVED_PER_CTA - 1024) / (STAGE_BYTES + 24);
  static constexpr int STAGES = STAGES_FIT > MAX_STAGES ? MAX_STAGES : STAGES_FIT;
  static_assert(STAGES >= 2, "stage does not fit");
  static constexpr int BAR_OFF = STAGES * STAGE_BYTES;
  static constexpr int BAR_BYTES = 3 * STAGES * 8;   // wfull, xfull, sempty per stage
  static constexpr size_t SMEM_BYTES = (size_t)BAR_OFF + BAR_BYTES + 1024;   // + the 1024-byte alignment of the base
  static_assert(CTAS * (SMEM_BYTES + SMEM_RESERVED_PER_CTA) <= SMEM_PER_SM, "CTAs per SM do not fit");
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
//   SS, PROMOTE (SS only: sum each chunk's wgmmas into the fp32 registers), DECODE_2CTA (two decode CTAs per SM, see
//   Residency), X_ELEM_BYTES (2: bf16 activations, 1: 8-bit), W_BYTES, AUX_BYTES (per stage), EPI (epilogue kind),
//   ACC_EXP2 (the accumulators hold the result * 2^-ACC_EXP2: a power of two folded into the dequant multiply, undone
//   in the EPI_FLOAT epilogue together with out_scale), MAX_N_MMA (widest token tile: 64 or 128)
//   static int make_maps(...)  host: the weight and aux tensor maps of one GEMM (arguments per format)
//   static void issue_w(tm_w, tm_aux, p, w smem dst, aux smem dst, full barrier, n_tile, kc, policy)  (one thread)
//   static uint32_t w_tx_bytes(p)
//   static void issue_w_rows(tm_w, tm_aux, p, w smem dst, aux smem dst, full barrier, row, kc, policy)
//                                                                  grouped only: the 128 weight rows from `row` of the
//                                                                  [E * N, K] map of all experts, and their aux tiles
//   SS:  static void mma(acc, w smem, x smem, wg, scale_d)          the 4 k32 wgmmas of a chunk for rows 64wg..
//   RA:  struct Raw; static void load(p, w smem, aux smem, row_lo, lane, Raw&)   rows row_lo and row_lo + 8
//        static void frag(p, raw, kk, a[4])                        bf16 A fragment of k16 step kk (0..7)
// Grouped<Fmt>: the grouped schedule above; the dense kernels compile without any of it.
template <class Fmt, int N_MMA>
__global__ void __launch_bounds__(NUM_THREADS, ctas_per_sm<Fmt, N_MMA>())
ts_gemm_kernel(const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_aux,
               const __grid_constant__ CUtensorMap tm_x, const Params p) {
  constexpr bool GROUPED = IsGrouped<Fmt>::value;
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
  const int b = blockIdx.x;
  int G = gridDim.x;
  long long U;
  const int* g_end = nullptr;   // grouped: the schedule table in shared memory
  const int* g_mbp = nullptr;
  if constexpr (GROUPED) {
    // which weights a unit needs depends on offs, the previous kernel's output: no weight request before the wait
    __shared__ int s_end[MAX_EXPERTS], s_mbp[MAX_EXPERTS + 1];
    // the static tables sit beside the ring, which Cfg::SMEM_BYTES does not count: both within the 227 KB a CTA may use
    static_assert(C::SMEM_BYTES + sizeof(s_end) + sizeof(s_mbp) <= 227 * 1024, "grouped tables do not fit beside the ring");
    pdl_launch_dependents();
    pdl_wait();
    if (warp == 0) grouped_schedule<N_MMA>(p, s_end, s_mbp, lane);
    __syncthreads();
    g_end = s_end;
    g_mbp = s_mbp;
    U = (long long)p.n_tiles * s_mbp[p.E] * p.KT;
    G = grouped_grid(G, U, p.grid_forced);
    if (b >= G) return;   // a CTA past the device-side grid has no units and owns no flag
  } else {
    U = (long long)p.n_tiles * p.m_blocks * p.KT;
  }
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
  if constexpr (!GROUPED) pdl_launch_dependents();

  const int seg_last = walk.nseg - 1;
  const bool last_is_owner = walk.seg_kind(seg_last) == streamk::SEG_OWNER;

  if (wgi == 0) {
    if constexpr (C::CTAS > 1) setmaxnreg_dec<PRODUCER_REGS>();   // all four warps, before three of them leave
    if (warp != 0) goto done;
    // ------------------------------------------------------------ TMA producer
    const uint64_t pol_w = policy_evict_first();
    const uint64_t pol_x = policy_evict_last();
    auto issue_w = [&](int i) {
      const int s = i % S;
      uint8_t* st = stage(s);
      mbar_expect_tx(&wfull[s], Fmt::w_tx_bytes(p));
      if constexpr (GROUPED) {
        // expert e's feature n is weight row e * N + n; a tile tail past N reads the next expert's rows (or the
        // map's zero fill), whose outputs the epilogue skips (n >= N_out)
        const int tile = tile_of(i), n_tile = tile % p.n_tiles;
        const int e = group_tile<N_MMA>(g_end, g_mbp, p.E, tile / p.n_tiles).e;
        Fmt::issue_w_rows(&tm_w, &tm_aux, p, st, st + Fmt::W_BYTES, &wfull[s], e * p.N + n_tile * ROWS, kc_of(i), pol_w);
      } else {
        Fmt::issue_w(&tm_w, &tm_aux, p, st, st + Fmt::W_BYTES, &wfull[s], tile_of(i) % p.n_tiles, kc_of(i), pol_w);
      }
    };
    auto issue_x = [&](int i) {
      const int s = i % S;
      uint8_t* xs = stage(s) + Fmt::W_BYTES + C::AUX_SLOT;
      int m0 = (tile_of(i) / p.n_tiles) * N_MMA;
      // grouped: from the expert's rows on (rows of the next expert in the box are loaded but never stored)
      if constexpr (GROUPED) m0 = group_tile<N_MMA>(g_end, g_mbp, p.E, tile_of(i) / p.n_tiles).row0;
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
    if constexpr (C::CTAS > 1) setmaxnreg_inc<CONSUMER_REGS>();
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
      int m0 = m_blk * N_MMA, m_end = p.M;   // tokens m0 .. min(m0 + N_MMA, m_end) - 1 are this tile's
      const float* w_scale = p.w_scale;
      const float* out_scale = p.out_scale;
      if constexpr (GROUPED) {
        const GroupTile gt = group_tile<N_MMA>(g_end, g_mbp, p.E, m_blk);
        m0 = gt.row0;
        m_end = gt.row_end;
        w_scale += (size_t)gt.e * p.N;
        out_scale += gt.e;
      }
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
              if (m0 + col < m_end) __stcg(&slot[col * ROWS + r], v[4 * q + 2 * h + c]);
            }
        asm volatile("bar.sync 1, 256;" ::: "memory");   // all 128 rows stored (cta-scope order) ...
        if (warp == 4 && lane == 0) streamk::st_release_u32(p.ws_flag + b, 1u);   // ... then one gpu-scope release
        return;
      }
      if (kind == streamk::SEG_OWNER) {
        // own partial + the partials of CTAs b+1 .. b_last in that order (fixed: bit-reproducible run to run)
        // One warp polls the flags, on distinct lanes at once (one L2 round trip when they are up, not one per
        // contributor), and the consumer barrier passes its acquire on; narrow tiles then load the partials of GB
        // contributors before adding any of them
        const int b_last = streamk::cta_of_unit((long long)tile * p.KT + p.KT - 1, U, G);
        if (warp == 4) streamk::wait_flags(p.ws_flag + b + 1, b_last - b, lane);
        asm volatile("bar.sync 1, 256;" ::: "memory");
        // registers: GB x NACC words of partials (restated by tests/streamk_model.py::group_width)
        constexpr int GB = NACC <= 8 ? 4 : (NACC <= 16 ? 2 : 1);
#pragma unroll 1
        for (int c = b + 1; c <= b_last && GB == 1; ++c) {
          const uint32_t* slot = reinterpret_cast<const uint32_t*>(p.ws_partial) + (size_t)c * (N_MMA * ROWS);
#pragma unroll
          for (int q = 0; q < NACC / 4; ++q) {
            // a warp-uniform exit every 16 tokens (the rest of the tile is past M).  The branch also bounds the loads the
            // compiler hoists above their adds to 8 words; hoisting all NACC of them spills at N_MMA = 128
            if (q % 2 == 0 && m0 + 8 * q >= m_end) break;
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int cc = 0; cc < 2; ++cc) {
                const int col = 8 * q + 2 * t + cc, r = row_lo + 8 * h, j = 4 * q + 2 * h + cc;
                if (m0 + col < m_end) {
                  const uint32_t o = __ldcg(slot + col * ROWS + r);
                  if constexpr (Fmt::EPI == EPI_I8) v[j] = (uint32_t)((int32_t)v[j] + (int32_t)o);
                  else v[j] = __float_as_uint(__uint_as_float(v[j]) + __uint_as_float(o));
                }
              }
          }
        }
#pragma unroll 1
        for (int c0 = b + 1; c0 <= b_last && GB > 1; c0 += GB) {
          uint32_t o[GB][NACC];
#pragma unroll
          for (int gi = 0; gi < GB; ++gi) {
            if (c0 + gi > b_last) break;
            const uint32_t* slot = reinterpret_cast<const uint32_t*>(p.ws_partial) + (size_t)(c0 + gi) * (N_MMA * ROWS);
#pragma unroll
            for (int q = 0; q < NACC / 4; ++q)
#pragma unroll
              for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int cc = 0; cc < 2; ++cc) {
                  const int col = 8 * q + 2 * t + cc, r = row_lo + 8 * h, j = 4 * q + 2 * h + cc;
                  o[gi][j] = m0 + col < m_end ? __ldcg(slot + col * ROWS + r) : 0u;
                }
          }
#pragma unroll
          for (int gi = 0; gi < GB; ++gi) {
            if (c0 + gi > b_last) break;
#pragma unroll
            for (int q = 0; q < NACC / 4; ++q)
#pragma unroll
              for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int cc = 0; cc < 2; ++cc) {
                  // tokens past M add the 0 loaded for them and are never written
                  const int j = 4 * q + 2 * h + cc;
                  if constexpr (Fmt::EPI == EPI_I8) v[j] = (uint32_t)((int32_t)v[j] + (int32_t)o[gi][j]);
                  else v[j] = __float_as_uint(__uint_as_float(v[j]) + __uint_as_float(o[gi][j]));
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
        if constexpr (Fmt::EPI == EPI_FLOAT) {
          if constexpr (GROUPED) {
            // the expert's own scale (required); never out_scale2, whose storage holds offs
            osc = *out_scale;
          } else {
            osc = (p.out_scale ? (p.out_scale_per_row ? p.out_scale[n] : *p.out_scale) : 1.f);
            if (p.out_scale2) osc *= *p.out_scale2;
          }
          osc *= __int_as_float((127 + Fmt::ACC_EXP2) << 23);
        } else {
          sw = w_scale ? w_scale[n] : 1.f;
        }
#pragma unroll
        for (int q = 0; q < NACC / 4; ++q)
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int m = m0 + 8 * q + 2 * t + c;
            if (m >= m_end) continue;
            const uint32_t raw = v[4 * q + 2 * h + c];
            __nv_bfloat16* dst = p.y ? p.y + (size_t)m * p.N_out + n : nullptr;
            if constexpr (Fmt::EPI == EPI_FLOAT) {
              float x = __uint_as_float(raw);
              if (p.row_scale) x *= p.row_scale[m];
              *dst = __float2bfloat16_rn(x * osc + bias);
            } else if constexpr (Fmt::EPI == EPI_I8) {
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
          // two halves: the wgmmas of k16 steps 0..3 run while steps 4..7 are dequantised (same wgmmas, same order)
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) Fmt::frag(p, raw, kk, a[kk]);
          mbar_wait(&xfull[s], ph);
          wgmma_fence_operand(acc);
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            if (half == 1) {
              // the raw words pass through here after the first half is issued, so its dequant cannot move above
              uint32_t(&rw)[sizeof(raw) / 4] = *reinterpret_cast<uint32_t(*)[sizeof(raw) / 4]>(&raw);
              wgmma_fence_operand(rw);
#pragma unroll
              for (int kk = 4; kk < 8; ++kk) Fmt::frag(p, raw, kk, a[kk]);
            }
            wgmma_fence();   // orders the fragment registers just written before the wgmmas that read them
#pragma unroll
            for (int kk = 4 * half; kk < 4 * half + 4; ++kk) {
              // k16 step kk of the bf16 B tile: atom kk / 4 (64 k each), 32 bytes per step inside the 128-byte row
              const uint64_t bd = wgmma_desc_k_sw128(x_s + (kk >> 2) * (N_MMA * 128) + (kk & 3) * 32);
              MMA::ra_bf16(acc, a[kk], bd, kk == 0 ? scale_d : 1u);
            }
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
// Activation tensor map, grid choice, workspace carve-up and launch at one token-tile width.
//   * at most one CTA of the grid per SM: the grid stays within the resident capacity, which the owner protocol needs
//     for forward progress (streamk.cuh), and a decode SM keeps room for the next kernel's CTA
//   * never fewer than MIN_UNITS chunks per CTA: splitting a tile over more CTAs shortens the streaming phase but
//     lengthens the owner's gather
//   * Grouped<Fmt>: the grid and the partial slots are sized for an upper bound of the units (each expert adds at most
//     one partial m-block); the kernel cuts the grid to the same rule for the units offs gives (grouped_grid)
template <class Fmt, int N_MMA>
inline int launch_gemm(Params& p, const CUtensorMap& tm_w, const CUtensorMap& tm_aux, const void* x, int ldx,
                       void* ws, size_t ws_bytes, const char* what, cudaStream_t stream) {
  using C = Cfg<Fmt, N_MMA>;
  CUtensorMap tm_x;   // box: 128 bytes of k (one swizzle atom) x N_MMA tokens
  {
    const uint64_t dims[2] = {(uint64_t)p.K, (uint64_t)p.M};
    const uint64_t str[1] = {(uint64_t)ldx * Fmt::X_ELEM_BYTES};
    const uint32_t box[2] = {128 / Fmt::X_ELEM_BYTES, N_MMA};
    int rc = make_tmap(&tm_x, Fmt::X_ELEM_BYTES == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8,
                       2, x, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  p.m_blocks = ceil_div(p.M, N_MMA);
  if constexpr (IsGrouped<Fmt>::value) p.m_blocks += p.E < p.M ? p.E : p.M;   // >= sum over experts of ceil(rows_e / N_MMA)
  const long long units = (long long)p.n_tiles * p.m_blocks * p.KT;
  int grid = sm_count();
  if (units / MIN_UNITS < grid) grid = units / MIN_UNITS > 0 ? (int)(units / MIN_UNITS) : 1;
  const int forced = streamk_ctas_override();
  p.grid_forced = forced != 0;
  if (forced) {
    // tests only: at most one CTA per SM (forward progress, see above) and never a CTA without units (its epilogue
    // would run on an accumulator no wgmma wrote)
    const int cap = units < sm_count() ? (int)units : sm_count();
    grid = forced < 1 ? 1 : (forced > cap ? cap : forced);
  }
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

// Y = X * W^T for every format: the caller sets M, N, N_out, K and its format's Params fields and builds the weight
// and aux maps (Fmt::make_maps); x is [M][ldx] activations of Fmt::X_ELEM_BYTES each.  The token count picks the
// token tile; more than Fmt::MAX_N_MMA tokens run as several blocks of that width.
// Grouped<Fmt> (Params::offs, E): an expert never holds more than M rows, so the width chosen from M streams each
// active expert's weights once for M <= 64.
template <class Fmt>
inline int run(Params& p, const CUtensorMap& tm_w, const CUtensorMap& tm_aux, const void* x, int ldx, void* ws,
               size_t ws_bytes, const char* what, cudaStream_t stream) {
  static_assert(Fmt::MAX_N_MMA == 64 || Fmt::MAX_N_MMA == 128, "token tile");
  p.n_tiles = ceil_div(p.N_out, ROWS);
  p.KT = ceil_div(p.K, KCHUNK);   // a K tail is zero-filled by TMA (out-of-bounds box elements) on both operands
  if (p.M <= 16) return launch_gemm<Fmt, 16>(p, tm_w, tm_aux, x, ldx, ws, ws_bytes, what, stream);
  if (p.M <= 32) return launch_gemm<Fmt, 32>(p, tm_w, tm_aux, x, ldx, ws, ws_bytes, what, stream);
  if (p.M <= 64) return launch_gemm<Fmt, 64>(p, tm_w, tm_aux, x, ldx, ws, ws_bytes, what, stream);
  return launch_gemm<Fmt, Fmt::MAX_N_MMA>(p, tm_w, tm_aux, x, ldx, ws, ws_bytes, what, stream);
}

}  // namespace tsg
}  // namespace ao
