// Persistent stream-K GEMM on Hopper wgmma (sm_90a) for every quantized linear of the library.
//
//   Y[M,N] = X[M,K] * W^[N,K]^T (+bias),   W^ = the weights, dequantised in-kernel where the format needs it
//
// Swap-AB: 128 weight rows of a tile are the wgmma M dimension (two consumer warpgroups of 64 rows each), the tokens
// are the wgmma N dimension (N_MMA = 16..128).  A format policy (Fmt) decides how the weights reach the tensor core:
//   * register-A (Fmt::SS == false): int4 tinygemm, nvfp4, mxfp8, mxfp4, int8, fp8 and nf4 weight-only.  Each consumer thread loads the packed
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
#include <cuda_fp8.h>

#include <type_traits>

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
// keep one CTA per SM and up to 200 KB of ring.  Grouped<Fmt> kernels (below) always run one CTA per SM: they cannot
// request weights before griddepcontrol.wait (which weights depends on offs), so a second resident CTA gains nothing,
// and their 8 KB schedule tables do not fit beside a ring sized to half of the SM.
constexpr int SMEM_PER_SM = 228 * 1024, SMEM_RESERVED_PER_CTA = 1024;

// ts_gemm_kernel<Grouped<Fmt>, N_MMA>: Fmt under the grouped schedule (see Grouped schedule below), for a shared-memory
// A format (fp8) or a register-A one (nvfp4, int4).  A wrapper rather than a kernel template parameter, so the dense
// kernels keep their names and their code.
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

// Fmt::X_AUX_BYTES (optional, default 0): bytes of the stage's aux slot that arrive with the activation tile (xfull,
// after griddepcontrol.wait: per-token values the previous kernel wrote), requested by Fmt::issue_x_aux
template <class F, class = void>
struct XAux {
  static constexpr int BYTES = 0;
};
template <class F>
struct XAux<F, std::void_t<decltype(F::X_AUX_BYTES)>> {
  static constexpr int BYTES = F::X_AUX_BYTES;
};

// Fmt::W_BLOCK_SCALES (optional, default false): Fmt::chunk_scales reads a scale per 128-row weight block, so a grouped
// kernel passes it the block of the expert's weights (e * n_tiles + n_tile), looked up once per segment
template <class F, class = void>
struct WBlockScales {
  static constexpr bool value = false;
};
template <class F>
struct WBlockScales<F, std::void_t<decltype(F::W_BLOCK_SCALES)>> {
  static constexpr bool value = F::W_BLOCK_SCALES;
};

// Fmt::SPARSE_A (optional, default false): a shared-memory A format whose weights are 2:4 sparse (wgmma.sp); the
// consumer passes its metadata words (Fmt::meta) to Fmt::mma
template <class F, class = void>
struct SparseA {
  static constexpr bool value = false;
};
template <class F>
struct SparseA<F, std::void_t<decltype(F::SPARSE_A)>> {
  static constexpr bool value = F::SPARSE_A;
};

// Fmt::W_XPOSE_BYTES (optional, default 0): a PROMOTE format whose stage holds its weights N-major ([128 k][128 n]);
// e4m3 wgmma reads K-major shared-memory operands only, so each consumer warpgroup transposes its 64 rows of every
// chunk (Fmt::xpose) into its half of a W_XPOSE_BYTES buffer beside the ring, and its wgmmas read them there
template <class F, class = void>
struct WXpose {
  static constexpr int BYTES = 0;
};
template <class F>
struct WXpose<F, std::void_t<decltype(F::W_XPOSE_BYTES)>> {
  static constexpr int BYTES = F::W_XPOSE_BYTES;
};

// Fmt::AUX_FILL (optional, default false): a register-A format whose aux slot is not loaded by TMA but written by
// warps 1..3 of the producer warpgroup, which the other formats leave idle.  Unit i belongs to warp 1 + i % 3: it waits
// for the stage as the producer does, runs Fmt::fill_aux(p, aux smem, n_tile, kc, lane) on all 32 lanes and arrives on
// the stage's wfull, which then expects two arrivals (the producer's with the weight bytes, and this one).  Three warps
// keep three stages' global loads in flight, and the weight TMAs never wait for them
template <class F, class = void>
struct AuxFill {
  static constexpr bool value = false;
};
template <class F>
struct AuxFill<F, std::void_t<decltype(F::AUX_FILL)>> {
  static constexpr bool value = F::AUX_FILL;
};

template <class Fmt, int N_MMA>
constexpr int ctas_per_sm() { return N_MMA <= 32 && Fmt::DECODE_2CTA && !IsGrouped<Fmt>::value ? 2 : 1; }
constexpr int PRODUCER_REGS = 24, CONSUMER_REGS = 104;   // 128 * 24 + 256 * 104 <= 384 * 80

// Epilogue arithmetic, per kind (Fmt::EPI; must stay what each format's reference computes, see Params)
enum Epi { EPI_FLOAT = 0, EPI_I8 = 1, EPI_F8 = 2, EPI_BF16_WSCALE = 3, EPI_BF16 = 4, EPI_F8_SPARSE = 5, EPI_F8_STATIC = 6 };
// EPI_F8_STATIC: Params::out_scale_per_row is a set of these flags
enum F8StaticFlags { F8S_OUT_PER_TOKEN = 1, F8S_W_PER_TENSOR = 2 };

// The output fake-quant of PrototypeFloat8Tensor (EPI_F8_STATIC), on the bf16 value y of the EPI_F8 epilogue:
// fp32(e4m3(clamp(y / s, -448, 448))) * s, the division a true one (torch divides by the scale tensor) and a NaN
// quotient kept NaN by the clamp (x / 0 = +-inf gives +-448, 0 / 0 NaN).  The caller rounds the product to bf16.
__device__ __forceinline__ float e4m3_qdq(float y, float s) {
  float v = __fdiv_rn(y, s);
  if (!isnan(v)) v = fminf(fmaxf(v, -448.f), 448.f);
  const __half_raw h = __nv_cvt_fp8_to_halfraw(__nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E4M3), __NV_E4M3);
  return __half2float(__half(h)) * s;
}

struct Params {
  const __nv_bfloat16* bias;
  const float* row_scale;   // EPI_FLOAT: optional per-token scale [M]; EPI_I8 / EPI_F8 / EPI_F8_SPARSE / EPI_F8_STATIC: the
                            // activation scale [M]
  const float* out_scale;   // EPI_FLOAT: optional device scalar, or (out_scale_per_row) one value per output feature;
                            // Grouped<Fmt>: one value per expert [E] (nvfp4: the per-expert weight scale);
                            // EPI_F8_STATIC: the output fake-quant scale (nullptr: none), one value or one per token [M]
  // The grouped fields share storage and padding with the dense ones, so Params keeps its 120 bytes: a larger
  // parameter block changed the code ptxas generates for every dense instantiation.
  union {
    const float* out_scale2;  // EPI_FLOAT: optional second device scalar multiplied into out_scale (nvfp4 a_pts * b_pts)
    const int* offs;          // Grouped<Fmt>: [E] on the device, see below (the grouped epilogue never reads out_scale2)
  };
  int out_scale_per_row;     // EPI_F8_STATIC: F8StaticFlags
  int grid_forced;          // Grouped<Fmt>: the host grid was forced (ao_b200_debug_set_streamk_ctas): no MIN_UNITS rule
  const float* w_scale;     // EPI_I8 / EPI_F8 / EPI_F8_SPARSE / EPI_F8_STATIC / EPI_BF16_WSCALE: per-output-feature weight
                            // scale [N] (EPI_F8_STATIC with F8S_W_PER_TENSOR: one value)
                            // (EPI_BF16 never
                            // reads it: its format applies the scale per weight, from the aux operand, or, blockwise
                            // e4m3, per 128x128 block [N/128][KT] in its promotion; grouped: [E * N/128][KT])
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
  static constexpr int XPOSE_BYTES = WXpose<Fmt>::BYTES;   // after the ring (1024-aligned: stages are 1 KiB multiples)
  static_assert(XPOSE_BYTES == 0 || CTAS == 1, "the transpose buffer is sized for one CTA per SM");
  // one CTA per SM: a 200 KB ring (less the transpose buffer); two: the CTA's share less its barriers (3 x 8 bytes per
  // stage) and alignment pad
  static constexpr int STAGES_FIT = CTAS == 1 ? (200 * 1024 - XPOSE_BYTES) / STAGE_BYTES
                                              : (SMEM_PER_SM / 2 - SMEM_RESERVED_PER_CTA - 1024) / (STAGE_BYTES + 24);
  static constexpr int STAGES = STAGES_FIT > MAX_STAGES ? MAX_STAGES : STAGES_FIT;
  static_assert(STAGES >= 2, "stage does not fit");
  static constexpr int XPOSE_OFF = STAGES * STAGE_BYTES;
  static constexpr int BAR_OFF = XPOSE_OFF + XPOSE_BYTES;
  static constexpr int BAR_BYTES = 3 * STAGES * 8;   // wfull, xfull, sempty per stage
  static constexpr size_t SMEM_BYTES = (size_t)BAR_OFF + BAR_BYTES + 1024;   // + the 1024-byte alignment of the base
  static_assert(CTAS * (SMEM_BYTES + SMEM_RESERVED_PER_CTA) <= SMEM_PER_SM, "CTAs per SM do not fit");
  // the owner's gather stages up to STAGES contributors' partials in the ring (see the producer) when one fits a stage;
  // not for PROMOTE (e4m3 x e4m3): its bs=32 decode stack measured 5 % slower with it (DESIGN §4)
  static constexpr bool STAGE_PARTIALS = !Fmt::PROMOTE && N_MMA * ROWS * 4 <= STAGE_BYTES;
  // the aux fillers keep a stage's loads in registers: they run at the kernel's register count, not PRODUCER_REGS
  static_assert(!AuxFill<Fmt>::value || CTAS == 1, "AUX_FILL formats run one CTA per SM");
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
//                                                                  (row = e * N + n)
//   W_XPOSE_BYTES: static void xpose(w smem, buffer, wg, t)      thread t < 128 of warpgroup wg: its share of the
//                                                                  stage's rows 64wg.. into buffer + 64wg rows, K-major
//   EXPERT_SCALE (grouped EPI_FLOAT only): the epilogue multiplies by out_scale[e] (nvfp4: yes, int4: no scale at all)
//   SS:  static void mma(acc, w smem, x smem, wg, scale_d)          the 4 k32 wgmmas of a chunk for rows 64wg..
//   SPARSE_A: mt = meta(p, aux smem, n_tile, kc, row, lane)        the thread's metadata words of the chunk (row: its
//                                                                  metadata row of the tile)
//             static void mma(acc, w smem, x smem, mt[2], wg, scale_d)  the 2 k64 wgmma.sp of a chunk for rows 64wg..
//   PROMOTE: cs = chunk_scales<N_MMA>(p, aux smem, w_blk, m0, kc, lane)  the chunk's scales (before its wgmmas); w_blk
//                                                                  is the weight's 128-row block: n_tile, or under the
//                                                                  grouped schedule (W_BLOCK_SCALES) e * n_tiles +
//                                                                  n_tile; m0 the tile's first token row
//            static void promote<N_MMA>(acc, part, accumulate, cs)   acc (+)= the chunk's partial sums, scaled by cs
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
    // the static tables sit beside the ring, which Cfg::SMEM_BYTES does not count: both within the 227 KB a CTA may use,
    // and every resident CTA's ring, tables and reserve within the SM
    static_assert(C::SMEM_BYTES + sizeof(s_end) + sizeof(s_mbp) <= 227 * 1024, "grouped tables do not fit beside the ring");
    static_assert(C::CTAS * (C::SMEM_BYTES + sizeof(s_end) + sizeof(s_mbp) + SMEM_RESERVED_PER_CTA) <= SMEM_PER_SM,
                  "grouped CTAs per SM do not fit");
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
      mbar_init(&wfull[i], AuxFill<Fmt>::value ? 2 : 1);
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
    if constexpr (AuxFill<Fmt>::value) {
      if (warp != 0) {
        // the aux fillers (see AuxFill): their stores, then the warp barrier, then one arrival on the stage
        for (int i = warp - 1; i < nunits; i += 3) {
          const int s = i % S;
          if (i >= S) mbar_wait(&sempty[s], ((i / S) & 1) ^ 1);
          Fmt::fill_aux(p, stage(s) + Fmt::W_BYTES, tile_of(i) % p.n_tiles, kc_of(i), lane);
          __syncwarp();
          if (lane == 0) mbar_arrive(&wfull[s]);
        }
        goto done;
      }
    }
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
      mbar_expect_tx(&xfull[s], C::X_BYTES + XAux<Fmt>::BYTES);
#pragma unroll
      for (int a = 0; a < C::X_ATOMS; ++a)
        tma_load_2d(xs + a * (N_MMA * 128), &tm_x, &xfull[s], kc_of(i) * KCHUNK + a * (KCHUNK / C::X_ATOMS), m0, pol_x);
      if constexpr (XAux<Fmt>::BYTES > 0) Fmt::issue_x_aux(&tm_aux, stage(s) + Fmt::W_BYTES, &xfull[s], m0, kc_of(i), pol_x);
    };
    const int pre = nunits < S ? nunits : S;
    for (int i = 0; i < pre; ++i) {
      if (elect_one()) issue_w(i);   // weights are complete before the previous kernel starts (ao_b200_pdl_fence)
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
    if constexpr (C::STAGE_PARTIALS) {
      // The gatherer: the partial of contributor b+1+k goes into ring position nunits + k (after the last chunk) as
      // soon as that stage comes back and the flag is up, while the consumers still run the last chunks.  The
      // consumers add them from shared memory in CTA order (epilogue, OWNER); contributors past the ring take the
      // register path there.  Only the owner's valid token columns are copied
      if (last_is_owner) {
        const int tile = walk.seg_tile(seg_last);
        const int b_last = streamk::cta_of_unit((long long)tile * p.KT + p.KT - 1, U, G);
        const int n_staged = b_last - b < S ? b_last - b : S;
        int m0 = (tile / p.n_tiles) * N_MMA, m_end = p.M;
        if constexpr (GROUPED) {
          const GroupTile gt = group_tile<N_MMA>(g_end, g_mbp, p.E, tile / p.n_tiles);
          m0 = gt.row0;
          m_end = gt.row_end;
        }
        const int cols = m_end - m0 < N_MMA ? m_end - m0 : N_MMA;
        // one lane per contributor: the flags are polled at once, not one round trip after another
        static_assert(S <= 32, "one gatherer lane per staged partial");
        if (lane < n_staged) {
          const int i = nunits + lane, s = i % S;
          mbar_wait(&sempty[s], ((i / S) & 1) ^ 1);
          while (streamk::ld_acquire_u32(p.ws_flag + b + 1 + lane) == 0u) __nanosleep(64);
          fence_proxy_async_global();   // the contributor's st.cg stores, acquired above, before the bulk reads
          mbar_expect_tx(&wfull[s], cols * ROWS * 4);
          bulk_load(stage(s), p.ws_partial + (size_t)(b + 1 + lane) * (N_MMA * ROWS), cols * ROWS * 4, &wfull[s]);
          if constexpr (AuxFill<Fmt>::value) mbar_arrive(&wfull[s]);   // the arrival no filler makes for this stage
        }
        __syncwarp();
      }
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
        // publish the partial (column-major slot, streamk::part_word), then one gpu-scope release
        uint32_t* slot = reinterpret_cast<uint32_t*>(p.ws_partial) + (size_t)b * (N_MMA * ROWS);
#pragma unroll
        for (int q = 0; q < NACC / 4; ++q)
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              const int col = 8 * q + 2 * t + c, r = row_lo + 8 * h;
              if (m0 + col < m_end) __stcg(&slot[streamk::part_word<C::STAGE_PARTIALS>(col, r)], v[4 * q + 2 * h + c]);
            }
        asm volatile("bar.sync 1, 256;" ::: "memory");   // all 128 rows stored (cta-scope order) ...
        if (warp == 4 && lane == 0) streamk::st_release_u32(p.ws_flag + b, 1u);   // ... then one gpu-scope release
        return;
      }
      if (kind == streamk::SEG_OWNER) {
        // own partial + the partials of CTAs b+1 .. b_last in that order (fixed: bit-reproducible run to run).
        // The first n_staged arrive in ring stages (the producer's gatherer): each is added once its stage is full.
        // For the rest, one warp polls the flags, on distinct lanes at once (one L2 round trip when they are up, not
        // one per contributor), and the consumer barrier passes its acquire on; narrow tiles then load the partials of
        // GB contributors before adding any of them
        const int b_last = streamk::cta_of_unit((long long)tile * p.KT + p.KT - 1, U, G);
        const int n_staged = !C::STAGE_PARTIALS ? 0 : (b_last - b < S ? b_last - b : S);
        if (warp == 4) streamk::wait_flags(p.ws_flag + b + 1 + n_staged, b_last - b - n_staged, lane);
        asm volatile("bar.sync 1, 256;" ::: "memory");
#pragma unroll 1
        for (int k = 0; k < n_staged; ++k) {
          const int i = nunits + k, s = i % S;
          mbar_wait(&wfull[s], (i / S) & 1);
          const uint32_t part = smem_u32(stage(s));
#pragma unroll
          for (int q = 0; q < NACC / 4; ++q)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int cc = 0; cc < 2; ++cc) {
                const int col = 8 * q + 2 * t + cc, r = row_lo + 8 * h, j = 4 * q + 2 * h + cc;
                if (m0 + col < m_end) {
                  const uint32_t o = lds32(part + streamk::part_word<C::STAGE_PARTIALS>(col, r) * 4);
                  if constexpr (Fmt::EPI == EPI_I8) v[j] = (uint32_t)((int32_t)v[j] + (int32_t)o);
                  else v[j] = __float_as_uint(__uint_as_float(v[j]) + __uint_as_float(o));
                }
              }
        }
        // registers: GB x NACC words of partials (restated by tests/streamk_model.py::group_width)
        constexpr int GB = NACC <= 8 ? 4 : (NACC <= 16 ? 2 : 1);
#pragma unroll 1
        for (int c = b + 1 + n_staged; c <= b_last && GB == 1; ++c) {
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
                  const uint32_t o = __ldcg(slot + streamk::part_word<C::STAGE_PARTIALS>(col, r));
                  if constexpr (Fmt::EPI == EPI_I8) v[j] = (uint32_t)((int32_t)v[j] + (int32_t)o);
                  else v[j] = __float_as_uint(__uint_as_float(v[j]) + __uint_as_float(o));
                }
              }
          }
        }
#pragma unroll 1
        for (int c0 = b + 1 + n_staged; c0 <= b_last && GB > 1; c0 += GB) {
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
                  o[gi][j] = m0 + col < m_end ? __ldcg(slot + streamk::part_word<C::STAGE_PARTIALS>(col, r)) : 0u;
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
            // the expert's own scale where the format has one (required then); never out_scale2, whose storage holds
            // offs
            if constexpr (Fmt::EXPERT_SCALE) osc = *out_scale;
          } else {
            osc = (p.out_scale ? (p.out_scale_per_row ? p.out_scale[n] : *p.out_scale) : 1.f);
            if (p.out_scale2) osc *= *p.out_scale2;
          }
          osc *= __int_as_float((127 + Fmt::ACC_EXP2) << 23);
        } else if constexpr (Fmt::EPI == EPI_F8_STATIC) {
          sw = w_scale[p.out_scale_per_row & F8S_W_PER_TENSOR ? 0 : n];
        } else if constexpr (Fmt::EPI != EPI_BF16) {
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
            } else if constexpr (Fmt::EPI == EPI_BF16_WSCALE) {
              // int8 weight-only reference: torch.mm returns bf16, a bf16 multiply by the weight scale cast to bf16,
              // then a bf16 add of the bias (absent: no add).  The product of two bf16 is exact in fp32
              const float s = __bfloat162float(__float2bfloat16_rn(sw));
              __nv_bfloat16 o = __float2bfloat16_rn(__bfloat162float(__float2bfloat16_rn(__uint_as_float(raw))) * s);
              if (p.bias) o = __float2bfloat16_rn(__bfloat162float(o) + bias);
              *dst = o;
            } else if constexpr (Fmt::EPI == EPI_BF16) {
              // fp8 weight-only reference: torch.matmul returns bf16, then a bf16 add of the bias (absent: no add)
              __nv_bfloat16 o = __float2bfloat16_rn(__uint_as_float(raw));
              if (p.bias) o = __float2bfloat16_rn(__bfloat162float(o) + bias);
              *dst = o;
            } else if constexpr (Fmt::EPI == EPI_F8_SPARSE) {
              // 2:4-sparse e4m3 reference (CUTLASS EVT, rowwise_scaled_linear_sparse_cutlass.cuh): fp32 nodes
              // ((acc * w_scale[n]) * x_scale[m]) + bias[n] (0 without bias), then one bf16 rounding.  Its build
              // contracts the last multiply and the add into one FFMA (its SASS has no FADD: DESIGN §2g)
              const float t = __fmul_rn(__uint_as_float(raw), sw);
              *dst = __float2bfloat16_rn(__fmaf_rn(t, p.row_scale[m], bias));
            } else if constexpr (Fmt::EPI == EPI_F8_STATIC) {
              // EPI_F8's bf16 output; with out_scale, then the output fake-quant with the token's (or the one) scale
              const __nv_bfloat16 y = __float2bfloat16_rn(__uint_as_float(raw) * (p.row_scale[m] * sw) + bias);
              *dst = p.out_scale ? __float2bfloat16_rn(e4m3_qdq(__bfloat162float(y),
                                                               p.out_scale[p.out_scale_per_row & F8S_OUT_PER_TOKEN ? m : 0]))
                                 : y;
            } else {
              *dst = __float2bfloat16_rn(__uint_as_float(raw) * (p.row_scale[m] * sw) + bias);
            }
          }
      }
    };

    // the ring's shared-memory address, converted once: converting a stage's generic pointer in the chunk loop costs
    // a dozen uniform instructions per chunk
    const uint32_t ring_s = smem_u32(smem);
    int i = 0;
    for (int seg = 0; seg < walk.nseg; ++seg) {
      const int cnt = walk.seg_count(seg);
      // grouped, W_BLOCK_SCALES: the 128-row weight block of the segment's tile in [E * N / 128], and its first row
      int w_blk = 0, row0 = 0;
      if constexpr (GROUPED && WBlockScales<Fmt>::value) {
        const int tile = walk.seg_tile(seg);
        const GroupTile gt = group_tile<N_MMA>(g_end, g_mbp, p.E, tile / p.n_tiles);
        w_blk = gt.e * p.n_tiles + tile % p.n_tiles;
        row0 = gt.row0;
      }
      for (int c = 0; c < cnt; ++c, ++i) {
        const uint32_t scale_d = c > 0;   // the first wgmma of a segment overwrites the accumulator
        const int s = i % S;
        const uint32_t ph = (i / S) & 1;
        const uint32_t w_s = ring_s + s * C::STAGE_BYTES, aux_s = w_s + Fmt::W_BYTES, x_s = aux_s + C::AUX_SLOT;
        mbar_wait(&wfull[s], ph);
        if constexpr (Fmt::PROMOTE) {
          // e4m3: a chain of wgmmas accumulates in the tensor core's reduced-precision adder; each chunk's four k32
          // wgmmas go to a fresh accumulator that is added to the fp32 registers here (fp32 accuracy across K).  The
          // format's chunk scales (none for rowwise) are read before the wgmmas, so their loads overlap them, and
          // before the stage goes back
          uint32_t a_s = w_s;
          if constexpr (WXpose<Fmt>::BYTES > 0) {
            // N-major weights: the warpgroup's 64 rows, K-major, into its half of the transpose buffer.  Its wgmmas of
            // the previous chunk have completed (wait_group 0 below), so none reads the buffer any more.  Its 128
            // threads' stores (generic proxy), then the proxy fence, then the wgmmas (async proxy) that read them.  The
            // stage goes back after those wgmmas, long after the loads of the transpose, whose values the stores used
            a_s = smem_u32(smem + C::XPOSE_OFF);
            Fmt::xpose(w_s, a_s, wg, threadIdx.x & 127);
            asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
            fence_proxy_async();
          }
          mbar_wait(&xfull[s], ph);
          const auto cs = Fmt::template chunk_scales<N_MMA>(p, aux_s, GROUPED ? w_blk : tile_of(i) % p.n_tiles,
                                                            GROUPED ? row0 : (tile_of(i) / p.n_tiles) * N_MMA,
                                                            kc_of(i), lane);
          uint32_t part[NACC];
          wgmma_fence();
          Fmt::template mma<N_MMA>(part, a_s, x_s, wg, 0u);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_fence_operand(part);
          release(s);
          Fmt::template promote<N_MMA>(acc, part, scale_d, cs);
          continue;
        } else if constexpr (SparseA<Fmt>::value) {
          // the metadata words arrived with the weights.  A wgmma.sp reads its metadata register while it runs, and
          // ptxas reuses that register once the instruction is issued: each chunk's wgmmas complete before the next
          // chunk's metadata is loaded (no wgmma in flight across chunks, as CUTLASS's sparse mainloop does)
          uint32_t mt[2];
          {
            const uint2 m2 = Fmt::meta(p, aux_s, tile_of(i) % p.n_tiles, kc_of(i), row_lo + 8 * (lane & 1), lane);
            mt[0] = m2.x;
            mt[1] = m2.y;
          }
          mbar_wait(&xfull[s], ph);
          wgmma_fence_operand(acc);
          wgmma_fence();
          Fmt::template mma<N_MMA>(acc, w_s, x_s, mt, wg, scale_d);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_fence_operand(acc);
          wgmma_fence_operand(mt);
          release(s);
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
          const uint64_t x_desc = wgmma_desc_k_sw128(x_s);
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
              // k16 step kk of the bf16 B tile: atom kk / 4 (64 k each), 32 bytes per step inside the 128-byte row.
              // The step's byte offset goes straight into the start-address field (16-byte units) of the chunk's
              // descriptor: shared addresses stay below 2^18 bytes, so the 14-bit field never carries
              const uint64_t bd = x_desc + (uint32_t)(((kk >> 2) * (N_MMA * 128) + (kk & 3) * 32) >> 4);
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

// The checks every dense linear shares, made once the caller has checked its format's K, N and group rules: x [M][ldx]
// (byte codes pass ldx = K) into the output y [M][N_out].  Returns at M == 0 before any pointer is looked at; then x
// and y must be set and x (named x_name in the message) start on 16 bytes, and p gets bias, y, M, N, N_out and K.
inline int dense_params(Params& p, const char* what, const char* x_name, const void* x, int ldx, int M, int K, int N,
                        int N_out, const uint16_t* bias, void* y) {
  AO_REQUIRE(M >= 0 && K > 0 && N > 0, "%s: bad sizes M=%d K=%d N=%d", what, M, K, N);
  AO_REQUIRE(ldx >= K && ldx % 8 == 0, "%s: ldx=%d must be >= K=%d and a multiple of 8", what, ldx, K);
  if (M == 0) return AO_OK;
  AO_REQUIRE(x && y, "%s: null pointer", what);
  AO_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0, "%s: %s must be 16-byte aligned", what, x_name);
  p.bias = reinterpret_cast<const __nv_bfloat16*>(bias);
  p.y = reinterpret_cast<__nv_bfloat16*>(y);
  p.M = M; p.N = N; p.N_out = N_out; p.K = K;
  return AO_OK;
}

// Y = X * W^T for one dense linear: dense_params, then `setup(p, &tm_w, &tm_aux)` checks the format's own pointers,
// sets its Params fields and builds its two maps, and the GEMM runs on x.
template <class Fmt, class Setup>
inline int run_dense(const char* what, const char* x_name, const void* x, int ldx, int M, int K, int N, int N_out,
                     const uint16_t* bias, void* y, void* ws, size_t ws_bytes, void* stream, Setup setup) {
  Params p{};
  if (int rc = dense_params(p, what, x_name, x, ldx, M, K, N, N_out, bias, y)) return rc;
  if (M == 0) return AO_OK;
  CUtensorMap tm_w, tm_aux;
  if (int rc = setup(p, &tm_w, &tm_aux)) return rc;
  return run<Fmt>(p, tm_w, tm_aux, x, ldx, ws, ws_bytes, what, reinterpret_cast<cudaStream_t>(stream));
}

// torch._grouped_mm(x, W.transpose(-2, -1), offs), 2-D x 3-D, for every format: expert e's rows [offs[e-1], offs[e])
// of x [M][K] (dense rows) against rows e*N .. e*N+N-1 of the weight map, into y [M][N_out] under Grouped<Fmt>.  The
// caller has checked its format's K and N rules.  This checks what every grouped launch needs, returns at M == 0
// before any pointer is looked at, then `setup(p, &tm_w, &tm_aux)` checks the format's own pointers, sets its Params
// fields and builds its two maps.
template <class Fmt, class Setup>
inline int run_grouped(const char* what, const void* x, int M, int K, int E, int N, int N_out, const int32_t* offs,
                       uint16_t* y, void* ws, size_t ws_bytes, void* stream, Setup setup) {
  AO_REQUIRE(M >= 0 && K > 0 && N > 0, "%s: bad sizes M=%d K=%d N=%d", what, M, K, N);
  AO_REQUIRE(E >= 1 && E <= MAX_EXPERTS, "%s: E=%d experts must be in [1, %d]", what, E, MAX_EXPERTS);
  AO_REQUIRE((long long)E * N <= 0x7FFFFFFF, "%s: E*N=%lld weight rows exceed the int32 range", what, (long long)E * N);
  if (M == 0) return AO_OK;
  AO_REQUIRE(x && offs && y && ws, "%s: null pointer", what);
  AO_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0, "%s: x must be 16-byte aligned", what);
  Params p{};
  p.y = reinterpret_cast<__nv_bfloat16*>(y);
  p.offs = offs;
  p.E = E;
  p.M = M; p.N = N; p.N_out = N_out; p.K = K;
  CUtensorMap tm_w, tm_aux;
  if (int rc = setup(p, &tm_w, &tm_aux)) return rc;
  return run<Grouped<Fmt>>(p, tm_w, tm_aux, x, K, ws, ws_bytes, what, reinterpret_cast<cudaStream_t>(stream));
}

}  // namespace tsg
}  // namespace ao
