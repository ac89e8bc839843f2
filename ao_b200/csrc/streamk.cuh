// Persistent stream-K work split and the split-tile ("fix-up") protocol shared by the decode GEMM kernels
// (ts_gemm.cuh, for every weight format).
//
// Work split.  The GEMM is n_tiles x m_blocks output tiles (128 weight rows x N_MMA tokens) times KT chunks of
// 128 k: U = tiles * KT units, unit u = (tile u / KT, chunk u % KT).  CTA b of G owns the contiguous range
// [U*b/G, U*(b+1)/G): every SM streams the same number of bytes whatever N and K are.  A CTA's range is a
// sequence of SEGMENTS (maximal runs of units of one tile), each accumulated in registers in turn:
//   FULL     all KT chunks of the tile: the epilogue writes the outputs directly
//   CONTRIB  starts at chunk > 0 (only ever the CTA's FIRST segment): the CTA is not the tile's first
//            contributor; it publishes its partial sums to its workspace slot and raises its flag
//   OWNER    starts at chunk 0 but the CTA's range ends before the tile does (only ever the CTA's LAST
//            segment): the remaining chunks belong to CTAs b+1 .. b_last, each of which holds them as its
//            CONTRIB segment.  The owner keeps its partial in registers, waits for the contributors' flags, adds
//            their partials in CTA order (= k order: fixed, so results are bit-reproducible run to run) and
//            writes the outputs.
// Compared with a symmetric "last arriver reduces" protocol this takes the owner's own partial, every atomic
// and all but one gpu-scope fence off the critical path at the end of the kernel: a CONTRIB segment is the
// first thing a CTA computes, so in long ranges its partial has been in L2 for a long time when the owner
// (which finishes that tile last) looks for it; only when the tile is split so finely that its contributors
// have no other work do publish and gather run back to back.
//
// Staged gather (ts_gemm.cuh, where a partial fits a ring stage: Cfg::STAGE_PARTIALS).  Once the producer warp of an
// owner has issued its last chunk, lane k of it waits for ring stage nunits + k to come back, acquires contributor
// b+1+k's flag, and bulk-copies (cp.async.bulk, after fence.proxy.async) that partial's valid token columns into
// the stage, for k < n_staged = min(b_last - b, STAGES).  These copies run while the consumers finish the owner's
// last chunks.  The consumers add the staged partials from shared memory, then the rest from L2, in CTA order.
//
// Workspace (caller-owned, zero-initialised once): flags uint32[grid] at +0 (0 = empty, 1 = published; the owner
// resets the flags it consumed, so the flags are all-zero again when the kernel ends), partial slots [grid][N_MMA * 128] 32-bit words at +64 KiB (slot b = CTA b's CONTRIB partial,
// column-major: token j's 128 rows at j * 128, in the row order of part_word below).
//
// Forward progress: an owner spins on flags of CTAs with HIGHER block indices, of its own grid only.  The launchers
// keep the grid at or below the SM count.  Decode kernels fit two CTAs per SM, so grid j+1 (PDL) shares the SMs with
// grid j:
//   * every CTA triggers its dependents first thing, so grid j is entirely resident before any CTA of j+1 launches;
//     an owner of j therefore only waits on CTAs that are already running;
//   * a CTA of j+1 touches the workspace, the flags and the activations only after griddepcontrol.wait, i.e. after
//     grid j has completed; before that it only streams weights into its own shared memory, and j never waits on it
//     (the weights must be complete before grid j starts: a weight quantized by this library is separated from its
//     first linear by ao_b200_pdl_fence, which quantize_ launches);
//   * CTAs of j+1 that did not find room become resident as CTAs of j exit, which they do without waiting on j+1.
// The staged gather adds no wait on another grid: its flags are the same flags of the same grid, polled by the
// producer warp after its griddepcontrol.wait.  Inside the CTA, the stages it waits for are released by consumers
// that wait on nothing but the ring before their last segment's epilogue, so the gatherer and the consumers cannot
// wait on each other.
//
// Device-side grid (grouped GEMM, ts_gemm.cuh Grouped<Fmt>).  The units per expert come from offs, which only the
// device reads, so the host launches a grid sized for an upper bound of U.  With more CTAs than units, unit_begin
// gives some CTA an empty range: an owner would then wait for a flag that CTA never raises, and that CTA's epilogue
// would run on an accumulator no wgmma wrote.  So every CTA first derives U from offs and the effective grid the host
// would have picked for it, G_eff = min(G, max(1, U / MIN_UNITS)) (forced grids: min(G, U); U = 0: no CTA).  CTAs
// b >= G_eff leave at once, before they touch the workspace; the split uses G_eff, and G_eff <= U gives every
// remaining CTA at least one unit.  All CTAs compute the same G_eff, so owners and contributors agree on the split.
// The forward-progress argument above holds unchanged for the CTAs below G_eff.
//
// tests/streamk_model.py restates unit_begin, cta_of_unit and Walk on the CPU (and GB, the owner's gather group of
// ts_gemm.cuh); a change here needs the same change there.
#pragma once
#include <stdint.h>

namespace ao {
namespace streamk {

constexpr int ROWS = 128;
constexpr size_t WS_FLAGS_BYTES = 16 * 1024;      // up to 4096 CTAs
constexpr size_t WS_PARTIAL_OFF = 64 * 1024;

__device__ __forceinline__ int unit_begin(int b, long long U, int G) { return (int)((U * b) / G); }
// the CTA whose range contains unit u
__device__ __forceinline__ int cta_of_unit(long long u, long long U, int G) {
  return (int)(((u + 1) * G + U - 1) / U) - 1;
}

enum SegKind { SEG_FULL = 0, SEG_CONTRIB = 1, SEG_OWNER = 2 };

// The segments of one CTA's unit range.  Everything is derived from (u0, nunits, KT), so every warp role computes
// the same walk without talking to the others.
struct Walk {
  int u0, nunits, KT;
  int cnt0;   // units of the first segment
  int nseg;
  __device__ __forceinline__ Walk(int u0_, int nunits_, int KT_) : u0(u0_), nunits(nunits_), KT(KT_) {
    const int kc0 = u0 % KT;
    cnt0 = KT - kc0 < nunits ? KT - kc0 : nunits;
    nseg = 1 + (nunits - cnt0 + KT - 1) / KT;
  }
  __device__ __forceinline__ int seg_begin(int s) const { return s == 0 ? 0 : cnt0 + (s - 1) * KT; }
  __device__ __forceinline__ int seg_count(int s) const {
    if (s == 0) return cnt0;
    const int rest = nunits - seg_begin(s);
    return rest < KT ? rest : KT;
  }
  __device__ __forceinline__ int seg_tile(int s) const { return u0 / KT + s; }
  __device__ __forceinline__ int seg_kind(int s) const {
    if (seg_count(s) == KT) return SEG_FULL;
    return (s == 0 && (u0 % KT) != 0) ? SEG_CONTRIB : SEG_OWNER;
  }
};

// Word (token j, row r) of a partial slot.  STAGED (kernels that stage partials in shared memory): the rows of a token
// column are XOR-permuted in blocks of 8 by bits 1..2 of j, so the four columns 2t + c (t = 0..3) of one fragment
// access land on distinct shared-memory banks when the owner reads a slot copied verbatim into a ring stage
template <bool STAGED>
__device__ __forceinline__ int part_word(int j, int r) { return j * ROWS + (STAGED ? r ^ (((j >> 1) & 3) << 3) : r); }

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_u32(unsigned* p, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// All lanes of the calling warp: wait until flags[0 .. n) are raised (lanes poll distinct flags, backing off while a
// flag is down so that the polling does not compete with the contributors still streaming).
__device__ __forceinline__ void wait_flags(const unsigned* flags, int n, int lane) {
  for (int base = 0; base < n; base += 32) {
    if (base + lane < n) {
      const unsigned* f = flags + base + lane;
      while (ld_acquire_u32(f) == 0u) __nanosleep(64);
    }
  }
  __syncwarp();
}

}  // namespace streamk
}  // namespace ao
