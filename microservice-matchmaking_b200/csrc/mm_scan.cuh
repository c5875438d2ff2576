// mm_scan.cuh — phase 2 of the tick: column scan of the histogram matrix + the tail (matched prefix per bin, policies S0 / S1)
#pragma once
#include "mm_common.cuh"

namespace mm {

// ---------------------------------------------------------------------------------------
// k_colscan: exclusive prefix down every column of M.  A column CTA is 32 bins wide
// (lanes = consecutive bins, coalesced) and 16 row-slices deep (warps): every thread sums
// its slice of rows, the slices are scanned through shared memory, then the slice is
// rewritten as running prefixes — one round trip of latency instead of R.
// The LAST CTA of the grid runs concurrently as the "tail": bin totals (accumulated by
// k_hist with global reductions) -> sorted position of every bin -> how many players of every
// bin are matched under the tick's policy (always a PREFIX of the bin in enqueue order) ->
//   outbase[v] = member slot of bin v's first player (exclusive scan of the matched counts)
//   binlim[v]  = outbase[v] + matched players of bin v; a player at or past it stays queued.
// ---------------------------------------------------------------------------------------
constexpr int kScanBlock = 512;
constexpr uint32_t kColScratchWords = (kScanBlock / 32) * 33;      // column CTA scratch
constexpr uint32_t kTailScratchWords = 64 + 4 + 9 * kMaxSegs + 12;  // tail CTA scratch, fixed part

// One 32-bin column group: exclusive prefix down the rows of M (scratch: kColScratchWords).  Bin b belongs to one
// partition, and only the rows holding that partition's tiles wrote M[.][b] (mm_hist.cuh): the scan of a column is
// confined to rows [rlo, rhi] of its partition — about R / partitions rows instead of R.  The prefixes go to P; M
// keeps the raw counts (a row's own count is M[row][b]).  Only run when geo_use_colscan(g): otherwise every row sums
// the few rows before it by itself (mm_place.cuh).
__device__ __forceinline__ void colscan_cols_body(uint32_t* scratch, const Geo& g, uint32_t group, uint32_t Kp, uint32_t K,
                                                  const uint16_t* __restrict__ bin_seg, const uint32_t* __restrict__ M,
                                                  uint32_t* __restrict__ P) {
  uint32_t(*s_part)[33] = reinterpret_cast<uint32_t(*)[33]>(scratch);
  const uint32_t tid = threadIdx.x, x = tid & 31, y = tid >> 5;
  constexpr uint32_t NY = kScanBlock / 32;
  const uint32_t b = group * 32 + x;
  uint32_t rlo = 0, rhi = 0;
  const bool on = b < K && geo_rows_of(g, bin_seg[b], rlo, rhi);
  const uint32_t nrows = on ? rhi - rlo + 1 : 0u;
  const uint32_t rp = (nrows + NY - 1) / NY;
  const uint32_t r0 = rlo + (y * rp < nrows ? y * rp : nrows), r1 = rlo + ((y + 1) * rp < nrows ? (y + 1) * rp : nrows);
  constexpr int kU = 4;  // independent loads in flight per thread
  uint32_t sum = 0;
  for (uint32_t r = r0; r < r1; r += kU) {
    uint32_t v[kU];
#pragma unroll
    for (int k = 0; k < kU; ++k) v[k] = (r + k < r1) ? __ldcg(M + (size_t)(r + k) * Kp + b) : 0u;
#pragma unroll
    for (int k = 0; k < kU; ++k) sum += v[k];
  }
  s_part[y][x] = sum;
  __syncthreads();
  uint32_t run = 0;
  for (uint32_t yy = 0; yy < y; ++yy) run += s_part[yy][x];
  for (uint32_t r = r0; r < r1; r += kU) {
    uint32_t v[kU];
#pragma unroll
    for (int k = 0; k < kU; ++k) v[k] = (r + k < r1) ? __ldcg(M + (size_t)(r + k) * Kp + b) : 0u;
#pragma unroll
    for (int k = 0; k < kU; ++k) {
      if (r + k < r1) P[(size_t)(r + k) * Kp + b] = run;
      run += v[k];
    }
  }
  __syncthreads();  // scratch may be reused by the next group
}

// arguments of the tail (shared by k_colscan and the fused k_tick)
struct TailArgs {
  uint32_t Kp, K, n_segs;
  uint32_t n_cut;                     // (mode, group) cut segments; each is a run of partitions
  const uint16_t* part_cut;           // [n_segs] partition -> cut segment
  const uint32_t* cut_lp_lo;          // [n_cut + 1] first partition of the cut segment
  uint32_t layout;                    // bit 0: matched counts in shared memory; bit 1: bin keys too (tail_words)
  int32_t max_spread;                 // < 0: unlimited (policy S0); >= 0: policy S1, rating order only
  const uint32_t* tot;                // [Kp] bin totals of the pool being matched (kept up to date by ingest / remove / tick)
  const uint32_t* seg_bin_lo;         // [n_segs + 1]
  const uint32_t* seg_L;              // [n_segs]
  const uint16_t* bin_seg;            // [Kp] bin -> segment
  const uint16_t* bin_key;            // [Kp] bin -> clamp key (rating order: ascending inside a segment)
  uint32_t* outbase;                  // [Kp] out: member slot of the bin's first player
  uint32_t* binlim;                   // [Kp] out: outbase + matched players of the bin
  SegInfo* seg;                       // [n_segs] out
  TickCtr* ctr;
  const uint32_t* fill;               // [n_segs] partition fills of the pool being matched
  PoolMeta dst;                       // out: layout of the compacted pool (fill, chunk table, chunks used)
  // lobby budget (flow control), read only by the tail instantiations with kBudget / kCountOnly
  const uint32_t* bud_queue;          // [n_cut] lobbies a (mode, group) queue may emit this tick (0xFFFFFFFF: no limit), or null
  const uint32_t* bud_mode;           // [n_cut / n_groups] lobbies a mode may emit this tick, or null
  uint32_t n_groups;                  // cut segment c = mode * n_groups + group
  uint32_t* cand;                     // [n_cut] out (budgeted tick, count-only tail): lobbies the queue has, budgets ignored
};
// shared-memory words of the tail for a layout: bases | matched counts (bit 0) | keys (bit 1)
__host__ __device__ constexpr uint32_t tail_words(uint32_t Kp, uint32_t layout) {
  return kTailScratchWords + (Kp + 2) + ((layout & 1u) ? (Kp + 2) : 0u) + ((layout & 2u) ? (Kp + 3) / 2 : 0u);
}

// The S1 walk on a histogram (oracle: orc_run_windowed), one bin v of a segment [.., hi) at a time.  bb holds the
// sorted position of every bin's first player (bb[v + 1] = b1 ends bin v); `keys` indexes like an array of the bins'
// ascending keys.  Off the carry chain:
//   reach = sorted position where keys exceed key_v + W (binary search over the segment's keys)
//   rsel  = min(reach, b1 - 1 + L): the seeds of bin v are cur, cur + L, ... < min(b1, reach - L + 1)
template <class Keys>
__device__ __forceinline__ uint32_t s1_rsel(const uint32_t* bb, const Keys& keys, uint32_t v, uint32_t hi, int32_t W,
                                            uint32_t L, uint32_t b1) {
  const int32_t lim = (int32_t)keys[v] + W;
  uint32_t a = v, e = hi;  // last bin in [v, hi) with key <= lim
  while (e - a > 1) { const uint32_t mid = (a + e) >> 1; if ((int32_t)keys[mid] <= lim) a = mid; else e = mid; }
  const uint32_t reach = bb[a + 1], cap = b1 - 1 + L;
  return reach < cap ? reach : cap;
}
// On the chain: pos = next unconsumed position; bin [B0, B1) with rsel RS.  With a = RS - cur the bin seeds a / L
// lobbies and p2 = RS - a mod L is the next unconsumed position (a mod L by a reciprocal multiply, Mrec =
// 0xFFFFFFFF / L).  -> matched players of the bin (always a prefix of it); pos advances.  An empty or padding bin
// (B0 = B1 <= pos) leaves pos alone and matches nothing.
__device__ __forceinline__ uint32_t s1_step(uint32_t& pos, uint32_t B0, uint32_t B1, uint32_t RS, uint32_t L,
                                            uint32_t Mrec) {
  const uint32_t cur = pos > B0 ? pos : B0;
  const uint32_t a = RS - cur;                      // meaningful when cur < B1 (then RS > cur)
  uint32_t rem = a - __umulhi(a, Mrec) * L;         // a mod L, or a mod L + L
  rem = rem < rem - L ? rem : rem - L;              // unsigned: picks the one below L
  const uint32_t p2 = RS - rem;                     // next unconsumed position after this bin's lobbies
  const bool inside = cur < B1, full = p2 >= B1;
  const uint32_t m = (!inside || full) ? B1 - B0 : p2 - B0;
  pos = !inside ? pos : (full ? p2 : B1);           // the rest of a partly matched bin stays queued
  return m;
}

// Tables of the tail in its scratch (word offsets; the per-bin arrays follow at kTailScratchWords)
constexpr uint32_t kTailLo = 68 + 3 * kMaxSegs;           // s_lo  [kMaxSegs + 1] first bin of the partition
constexpr uint32_t kTailNch = kTailLo + kMaxSegs + 1;     // s_nch [kMaxSegs + 1]
constexpr uint32_t kTailL = kTailNch + kMaxSegs + 1;      // s_L   [kMaxSegs] lobby size of the partition
constexpr uint32_t kTailClp = kTailL + 2 * kMaxSegs;      // s_clp [kMaxSegs + 1] first partition of the cut segment
constexpr uint32_t kTailMs = kTailClp + kMaxSegs + 1;     // s_ms  [kMaxSegs + 1]
// The lobby budget keeps two per-queue arrays where the partition table later puts s_ms / s_nch (they are spent by then):
constexpr uint32_t kTailCand = kTailMs;    // s_c  [n_cut] lobbies of the queue, budgets ignored
constexpr uint32_t kTailAllot = kTailNch;  // s_al [n_cut] lobbies it may emit

// Lobbies of every (mode, group) queue from the tail's tables -> out[c] (shared or global).  S0: the queue's players /
// L, from the bases s_bb; S1 (s_m: the bins' matched counts after the walk): its matched players / L, one warp per queue.
__device__ __forceinline__ void tail_count_lobbies(const uint32_t* scratch, const uint32_t* s_m, uint32_t n_cut,
                                                   bool windowed, uint32_t* out) {
  const uint32_t *s_lo = scratch + kTailLo, *s_L = scratch + kTailL, *s_clp = scratch + kTailClp;
  const uint32_t* s_bb = scratch + kTailScratchWords;
  const uint32_t lane = threadIdx.x & 31;
  if (!windowed) {
    for (uint32_t c = threadIdx.x; c < n_cut; c += kScanBlock)
      out[c] = (s_bb[s_lo[s_clp[c + 1]]] - s_bb[s_lo[s_clp[c]]]) / s_L[s_clp[c]];
    return;
  }
  for (uint32_t c = threadIdx.x >> 5; c < n_cut; c += kScanBlock / 32) {
    uint32_t sum = 0;
    for (uint32_t v = s_lo[s_clp[c]] + lane; v < s_lo[s_clp[c + 1]]; v += 32) sum += s_m[v];
    sum = __reduce_add_sync(0xFFFFFFFFu, sum);
    if (lane == 0) out[c] = sum / s_L[s_clp[c]];
  }
}

// The allowances of mode m's queues q = m * G + g, one warp (<= 64 groups: two per lane, remainder ranks by
// comparison): s_c[q] lobbies the queue has -> s_al[q] lobbies it may emit.  c' = min(c, bud_queue[q]); if the mode's
// sum C of c' exceeds its budget B, B is apportioned by largest remainder: floor(B c' / C) each, and the B - sum groups
// with the largest (B c') mod C get one more, ties to the lower group.  Restated on the host by shard.apportion.  The
// tick's tail and the off-tick calls' k_wd_allot both apportion with it.
__device__ __forceinline__ void budget_apportion(const uint32_t* s_c, uint32_t* s_al, uint32_t m, uint32_t G,
                                                 const uint32_t* bud_queue, const uint32_t* bud_mode) {
  const uint32_t lane = threadIdx.x & 31;
  uint32_t c[2], al[2], C = 0;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const uint32_t g = lane + 32 * j;
    c[j] = g < G ? s_c[m * G + g] : 0u;
    if (g < G && bud_queue) { const uint32_t b = bud_queue[m * G + g]; c[j] = c[j] < b ? c[j] : b; }
    al[j] = c[j];
    C += c[j];
  }
  C = __reduce_add_sync(0xFFFFFFFFu, C);  // < 2^31: every lobby has a player of its own
  const uint32_t B = bud_mode ? bud_mode[m] : 0xFFFFFFFFu;
  if (C > B) {  // (uniform over the warp)
    uint32_t rem[2], fl = 0;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const uint64_t p = (uint64_t)B * c[j];
      al[j] = (uint32_t)(p / C); rem[j] = (uint32_t)(p % C);
      fl += al[j];
    }
    const uint32_t extra = B - __reduce_add_sync(0xFFFFFFFFu, fl);  // fewer than the groups with a remainder
    uint32_t rank[2] = {0u, 0u};  // groups that come before this one by (remainder descending, group ascending)
    for (int l = 0; l < 32; ++l)
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const uint32_t r = __shfl_sync(0xFFFFFFFFu, rem[k], l), g2 = l + 32 * k;
#pragma unroll
        for (int j = 0; j < 2; ++j) rank[j] += (r > rem[j] || (r == rem[j] && g2 < lane + 32 * j)) ? 1u : 0u;
      }
#pragma unroll
    for (int j = 0; j < 2; ++j) al[j] += rank[j] < extra ? 1u : 0u;
  }
#pragma unroll
  for (int j = 0; j < 2; ++j)
    if (lane + 32 * j < G) s_al[m * G + lane + 32 * j] = al[j];
}

// Lobby budget, the whole block, called with the tail's tables and (S1) matched counts in place:
//   s_c[q]  = lobbies queue q = m * G + g would emit (also written to cand[q])
//   s_al[q] = lobbies it may emit (budget_apportion, one warp per mode)
//   S0 clip: the queue's matched end moves to its (a_q L)-th sorted position: the partitions' matched counts s_mt,
//             which the caller has filled for the unbudgeted cut, are written again.
//   S1 clip: one warp per queue, bin v keeps the matched players that come before the queue's (a_q L)-th matched
//             player: m'_v = clamp(a_q L - matched players of the queue's earlier bins, 0, m_v).
// Not inlined, and no argument is passed by address: the budget instantiation of the fused kernel keeps the register
// allocation of its placement loops.
__device__ __noinline__ void tail_budget(uint32_t* scratch, uint32_t* s_m, uint32_t n_cut, uint32_t n_segs, uint32_t G,
                                         bool windowed,
                                         const uint32_t* bud_queue, const uint32_t* bud_mode, uint32_t* cand) {
  const uint32_t *s_lo = scratch + kTailLo, *s_L = scratch + kTailL, *s_clp = scratch + kTailClp;
  uint32_t *s_c = scratch + kTailCand, *s_al = scratch + kTailAllot;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  tail_count_lobbies(scratch, s_m, n_cut, windowed, s_c);
  __syncthreads();
  if (warp < n_cut / G) budget_apportion(s_c, s_al, warp, G, bud_queue, bud_mode);
  for (uint32_t q = threadIdx.x; q < n_cut; q += kScanBlock) cand[q] = s_c[q];
  __syncthreads();
  if (!windowed) {  // the partitions' matched counts again, with the queue's matched end at a_q L
    const uint32_t *s_bb = scratch + kTailScratchWords, *s_pc = scratch + kTailL + kMaxSegs;
    uint32_t* s_mt = scratch + 68 + 2 * kMaxSegs;
    for (uint32_t sg = threadIdx.x; sg < n_segs; sg += kScanBlock) {
      const uint32_t q = s_pc[sg], mend = s_bb[s_lo[s_clp[q]]] + s_al[q] * s_L[sg];
      const uint32_t a = s_bb[s_lo[sg]], b = s_bb[s_lo[sg + 1]];
      s_mt[sg] = (mend < a ? a : (mend > b ? b : mend)) - a;
    }
    return;
  }
  for (uint32_t q = warp; q < n_cut; q += kScanBlock / 32) {
    if (s_al[q] == s_c[q]) continue;
    const uint32_t lo = s_lo[s_clp[q]], hi = s_lo[s_clp[q + 1]], limit = s_al[q] * s_L[s_clp[q]];
    uint32_t before = 0;
    for (uint32_t off = lo; off < hi; off += 32) {
      const uint32_t v = off + lane, m = v < hi ? s_m[v] : 0u;
      uint32_t incl = m;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t up = __shfl_up_sync(0xFFFFFFFFu, incl, d);
        if (lane >= (uint32_t)d) incl += up;
      }
      const uint32_t b = before + incl - m, room = b < limit ? limit - b : 0u;
      if (v < hi) s_m[v] = m < room ? m : room;
      before += __shfl_sync(0xFFFFFFFFu, incl, 31);
    }
  }
  __syncthreads();
}

// The tail.  One pipeline for both policies:
//   bin totals -> bases s_bb -> matched prefix of every bin -> member slot of the bin's first player.
// S0 (reference behaviour): a (mode, group) partition of n players emits floor(n/L) lobbies, the n mod L
//   highest-ranked players stay queued: member slot = sorted position - leftovers of earlier partitions,
//   clipped at the partition's matched end (closed form, only a scan over the partitions).
// S1 (extension): greedy windowed walk over the partition (oracle: orc_run_windowed).  Players of one bin have
//   the same key, so the walk runs on the histogram: from position cur in bin v, lobbies are seeded at
//   cur, cur+L, ... while the seed is still in bin v and its L-th player has key <= key_v + W; whatever is
//   left of bin v afterwards cannot seed and stays queued.  Two-pointer over the bins of the segment.
// Very large key domains (layout bit 0 clear) park m_v in global memory and scan it in place of the bases.
// Lobby budget (t.bud_queue / t.bud_mode): under both policies the first a lobbies of a cut segment are its first a L
// matched players in sorted order, so an allowance a_q clips the matched counts — S0: the segment's matched end; S1:
// the bins' matched counts past a_q L, before they are scanned into member slots — and everything downstream sees a
// smaller matched prefix per bin.  kBudget selects the tail with the budget code: a tick without a budget runs the
// instantiation without it, instruction for instruction the tail it has always run.  kCountOnly (k_lobby_candidates): stop at the per-queue lobby counts, write t.cand
// (and, for layout bit 0 clear, the parked counts in t.binlim) and nothing else.
// kPreview (mm_locate): the whole cut, budget included when kBudget, into the caller's own scratch: t.outbase, t.binlim,
// t.cand (kBudget) and, in t.dst.tot, the sorted position of every bin's first player ([Kp + 1]: the bases s_bb).
// Nothing else is written: not t.seg, t.ctr or the rest of t.dst.
template <bool kCountOnly = false, bool kBudget = false, bool kPreview = false>
__device__ __forceinline__ void colscan_tail_body(uint32_t* scratch, const TailArgs t) {
  constexpr uint32_t NW = kScanBlock / 32;
  uint32_t* s_tmp = scratch;            // [64]
  uint32_t* s_misc = scratch + 64;      // [4] heavy flag | n_matched | lobbies | chunks of the compacted pool
  uint32_t* s_a = scratch + 68;         // [kMaxSegs] leftovers of earlier segments
  uint32_t* s_ns = s_a + kMaxSegs;      // [kMaxSegs] alive players of the segment
  uint32_t* s_mt = s_ns + kMaxSegs;     // [kMaxSegs] matched players of the segment
  uint32_t* s_lo = scratch + kTailLo;      // [kMaxSegs + 1] first bin of the segment
  uint32_t* s_nch = scratch + kTailNch;    // [kMaxSegs + 1] first chunk of the segment in the compacted pool
  uint32_t* s_L = scratch + kTailL;        // [kMaxSegs] lobby size of the segment
  uint32_t* s_pc = s_L + kMaxSegs;         // [kMaxSegs] cut segment of the partition
  uint32_t* s_clp = scratch + kTailClp;    // [kMaxSegs + 1] first partition of the cut segment
  uint32_t* s_ms = scratch + kTailMs;      // [kMaxSegs + 1] member slot of the partition's first matched player
  uint32_t* s_bb = scratch + kTailScratchWords;  // [Kp + 1] sorted position of the bin's first player
  static_assert(kTailMs + kMaxSegs + 1 <= kTailScratchWords, "the tail's tables end before its per-bin arrays");
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, Kp = t.Kp, K = t.K, n_segs = t.n_segs;
  if (tid == 0) s_misc[0] = 0;
  for (uint32_t sg = tid; sg <= n_segs; sg += kScanBlock) s_lo[sg] = t.seg_bin_lo[sg];  // all the cold loads at once
  for (uint32_t sg = tid; sg < n_segs; sg += kScanBlock) { s_L[sg] = t.seg_L[sg]; s_pc[sg] = t.part_cut[sg]; }
  for (uint32_t c = tid; c <= t.n_cut; c += kScanBlock) s_clp[c] = t.cut_lp_lo[c];
  for (uint32_t i = tid; i < Kp; i += kScanBlock) s_bb[i] = __ldcg(&t.tot[i]);  // coalesced, independent loads
  __syncthreads();
  // list-ranked partitions only: does some bin expect > 8 players per tile of its partition?
  for (uint32_t sg = warp; !kCountOnly && sg < n_segs; sg += NW) {
    if (s_lo[sg + 1] - s_lo[sg] <= kFastBins) continue;
    uint32_t mx = 0;
    for (uint32_t v = s_lo[sg] + lane; v < s_lo[sg + 1]; v += 32) mx = s_bb[v] > mx ? s_bb[v] : mx;
    mx = __reduce_max_sync(0xFFFFFFFFu, mx);
    if (lane == 0 && (uint64_t)mx * kTile > 8ull * __ldcg(&t.fill[sg])) s_misc[0] = 1;
  }
  __syncthreads();
  const uint32_t total = block_excl_scan<kScanBlock>(s_bb, Kp, s_tmp);
  if (tid == 0) s_bb[Kp] = total;
  __syncthreads();
  if constexpr (kPreview)
    for (uint32_t v = tid; v <= Kp; v += kScanBlock) t.dst.tot[v] = s_bb[v];
  const uint32_t alive = s_bb[K], dead = total - alive;
  const bool windowed = t.max_spread >= 0;
  const bool m_smem = (t.layout & 1u) != 0, key_smem = (t.layout & 2u) != 0;
  uint32_t* s_m = m_smem ? s_bb + Kp + 2 : t.binlim;  // S1: [Kp + 1] matched players of the bin

  if (!windowed) {
    if (kCountOnly) { tail_count_lobbies(scratch, nullptr, t.n_cut, false, t.cand); return; }
    // S0: a cut segment of n players gives n / L lobbies: its first (n / L) * L sorted positions are matched; a partition holds the part of that prefix that falls into its own position range.
    for (uint32_t sg = tid; sg < n_segs; sg += kScanBlock) {
      const uint32_t c = s_pc[sg], cs = s_bb[s_lo[s_clp[c]]], ce = s_bb[s_lo[s_clp[c + 1]]], L = s_L[sg];
      const uint32_t mend = cs + (ce - cs) / L * L;
      const uint32_t a = s_bb[s_lo[sg]], b = s_bb[s_lo[sg + 1]];
      s_ns[sg] = b - a;
      s_mt[sg] = (mend < a ? a : (mend > b ? b : mend)) - a;
    }
    if constexpr (kBudget) tail_budget(scratch, nullptr, t.n_cut, t.n_segs, t.n_groups, false, t.bud_queue, t.bud_mode, t.cand);
  } else {
    uint16_t* s_key = reinterpret_cast<uint16_t*>(s_bb + (m_smem ? 2 : 1) * (Kp + 2));
    const uint16_t* keys = key_smem ? s_key : t.bin_key;
    if (key_smem)
      for (uint32_t v = tid; v < K; v += kScanBlock) s_key[v] = t.bin_key[v];
    for (uint32_t v = K + tid; v < Kp; v += kScanBlock) s_m[v] = 0;
    __syncthreads();
    const int32_t W = t.max_spread;
    // One warp walks TWO partitions at a time (two independent carry chains in flight).  Per bin, off the chain:
    // s1_rsel; on the chain only: s1_step.  Empty bins fall out of the same arithmetic (cur >= b1), so the 32 bins
    // of a batch are visited by an unrolled loop.
    for (uint32_t sg = tid; sg < n_segs; sg += kScanBlock) s_ns[sg] = s_bb[s_lo[sg + 1]] - s_bb[s_lo[sg]];
    // the walk runs over whole CUT segments (a window may span the partitions of a wide rating group)
    for (uint32_t sg0 = warp; sg0 < t.n_cut; sg0 += 2 * NW) {
      uint32_t lo[2], hi[2], L[2], Mrec[2], pos[2];
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const uint32_t sg = sg0 + q * NW;
        const bool on = sg < t.n_cut;
        lo[q] = on ? s_lo[s_clp[sg]] : 0u; hi[q] = on ? s_lo[s_clp[sg + 1]] : 0u; L[q] = on ? s_L[s_clp[sg]] : 1u;
        Mrec[q] = 0xFFFFFFFFu / L[q];  // umulhi(a, Mrec) is a / L or a / L - 1 for every 32-bit a
        pos[q] = s_bb[lo[q]];
      }
      const uint32_t span0 = hi[0] - lo[0], span1 = hi[1] - lo[1], span = span0 > span1 ? span0 : span1;
      for (uint32_t off = 0; off < span; off += 32) {
        uint32_t b0[2], b1[2], rs[2], mine[2];
        bool valid[2];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const uint32_t v = lo[q] + off + lane;
          valid[q] = v < hi[q];
          b0[q] = b1[q] = rs[q] = 0u; mine[q] = 0u;
          if (valid[q]) {
            b0[q] = s_bb[v]; b1[q] = s_bb[v + 1];
            rs[q] = s1_rsel(s_bb, keys, v, hi[q], W, L[q], b1[q]);
          }
        }
#pragma unroll 8
        for (int l = 0; l < 32; ++l) {
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            const uint32_t B0 = __shfl_sync(0xFFFFFFFFu, b0[q], l), B1 = __shfl_sync(0xFFFFFFFFu, b1[q], l);
            const uint32_t RS = __shfl_sync(0xFFFFFFFFu, rs[q], l);
            const uint32_t m = s1_step(pos[q], B0, B1, RS, L[q], Mrec[q]);
            if ((int)lane == l) mine[q] = m;
          }
        }
#pragma unroll
        for (int q = 0; q < 2; ++q)
          if (valid[q]) s_m[lo[q] + off + lane] = mine[q];
      }
    }
    __syncthreads();
    if (!m_smem) {  // very large key domain: the counts were parked in global memory; scan them in place of the bases
      for (uint32_t v = tid; v < Kp; v += kScanBlock) s_bb[v] = s_m[v];
      s_m = s_bb;
      __syncthreads();
    }
    if (kCountOnly) { tail_count_lobbies(scratch, s_m, t.n_cut, true, t.cand); return; }
    if constexpr (kBudget) tail_budget(scratch, s_m, t.n_cut, t.n_segs, t.n_groups, true, t.bud_queue, t.bud_mode, t.cand);
    // member slots = exclusive scan of the matched counts (members of successive partitions are contiguous)
    const uint32_t nm = block_excl_scan<kScanBlock>(s_m, Kp, s_tmp);
    if (tid == 0) s_m[Kp] = nm;
    __syncthreads();
    for (uint32_t v = tid; v < Kp; v += kScanBlock) {
      t.outbase[v] = s_m[v];
      t.binlim[v] = s_m[v + 1];  // = outbase + matched players of the bin
      // bin totals of the compacted pool: what was there minus the matched prefix; removed players are gone
      if constexpr (!kPreview) t.dst.tot[v] = v < K ? __ldcg(&t.tot[v]) - (s_m[v + 1] - s_m[v]) : 0u;
    }
    for (uint32_t sg = tid; sg < n_segs; sg += kScanBlock) s_mt[sg] = s_m[s_lo[sg + 1]] - s_m[s_lo[sg]];
  }
  __syncthreads();
  // Partition table, by ONE warp (<= 512 partitions, 32 per step with carries; no block-wide scans): member / lobby
  // bases, and the layout of the compacted pool — partition sg keeps n_left players in ceil(n_left / kTile) fresh
  // chunks handed out in partition order from chunk 0 (the epilogue moves the players).
  if (warp == 0) {
    uint32_t c_mem = 0, c_left = 0, c_ch = 0;
    for (uint32_t base = 0; base < n_segs; base += 32) {
      const uint32_t sg = base + lane;
      const bool on = sg < n_segs;
      const uint32_t ns = on ? s_ns[sg] : 0u, mt = on ? s_mt[sg] : 0u;
      const uint32_t nleft = ns - mt, nch = (nleft + kTile - 1) / kTile;
      uint32_t i_mem = mt, i_left = nleft, i_ch = nch;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const uint32_t a = __shfl_up_sync(0xFFFFFFFFu, i_mem, off);
        const uint32_t c = __shfl_up_sync(0xFFFFFFFFu, i_left, off), d = __shfl_up_sync(0xFFFFFFFFu, i_ch, off);
        if (lane >= (uint32_t)off) { i_mem += a; i_left += c; i_ch += d; }
      }
      if (on) {
        s_ms[sg] = c_mem + i_mem - mt;
        s_a[sg] = c_left + i_left - nleft;
        s_nch[sg] = c_ch + i_ch - nch;
        if constexpr (!kPreview) t.dst.fill[sg] = nleft;
      }
      c_mem += __shfl_sync(0xFFFFFFFFu, i_mem, 31);
      c_left += __shfl_sync(0xFFFFFFFFu, i_left, 31); c_ch += __shfl_sync(0xFFFFFFFFu, i_ch, 31);
    }
    __syncwarp();
    // Lobbies are cut per CUT segment: lobby k of segment c = member slots [mb_c + k L, + L).  A partition is
    // credited with the lobbies that START inside its member-slot range, so the header writers can loop per partition.
    uint32_t c_lob = 0;
    for (uint32_t base = 0; base < n_segs; base += 32) {
      const uint32_t sg = base + lane;
      const bool on = sg < n_segs;
      uint32_t nl = 0, hb = 0;
      if (on) {
        const uint32_t L = s_L[sg], mb = s_ms[s_clp[s_pc[sg]]], m0 = s_ms[sg] - mb, m1 = m0 + s_mt[sg];
        const uint32_t k0 = (m0 + L - 1) / L, k1 = (m1 + L - 1) / L;
        nl = k1 - k0; hb = mb + k0 * L;
      }
      uint32_t i_lob = nl;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const uint32_t b = __shfl_up_sync(0xFFFFFFFFu, i_lob, off);
        if (lane >= (uint32_t)off) i_lob += b;
      }
      if (on) {
        SegInfo si;
        si.n = s_ns[sg]; si.n_lobbies = nl; si.member_base = hb; si.lobby_base = c_lob + i_lob - nl;
        si.left_base = s_a[sg]; si.new_chunk = s_nch[sg]; si.n_left = s_ns[sg] - s_mt[sg]; si.reserved = 0;
        if constexpr (!kPreview) t.seg[sg] = si;
      }
      c_lob += __shfl_sync(0xFFFFFFFFu, i_lob, 31);
    }
    if (lane == 0) {
      s_nch[n_segs] = c_ch;
      s_misc[1] = c_mem; s_misc[2] = c_lob;
      if constexpr (!kPreview) {
        *t.dst.bump = c_ch;
        t.ctr->n_lobbies = c_lob; t.ctr->n_matched = c_mem; t.ctr->n_alive = alive; t.ctr->n_dead = dead;
        t.ctr->n_resid = c_left;
        t.ctr->heavy = s_misc[0];
      }
    }
  }
  __syncthreads();
  const uint32_t n_matched = s_misc[1];
  if (!windowed) {
    // S0: member slot = sorted position - leftovers of earlier partitions, clipped at the partition's matched end
    for (uint32_t sg = warp; sg < n_segs; sg += NW) {  // one warp per partition: no bin -> segment lookups
      const uint32_t lo = s_lo[sg], hi = s_lo[sg + 1], start = s_bb[lo], shift = s_a[sg];
      const uint32_t mend = start + s_mt[sg];  // end of the partition's matched positions
      for (uint32_t v = lo + lane; v < hi; v += 32) {
        const uint32_t b0 = s_bb[v], b1 = s_bb[v + 1];
        const uint32_t o = (b0 < mend ? b0 : mend), l = (b1 < mend ? b1 : mend);
        t.outbase[v] = o - shift;
        t.binlim[v] = l - shift;
        if constexpr (!kPreview) t.dst.tot[v] = (b1 - b0) - (l - o);  // bin totals of the compacted pool: the unmatched tail of the bin
      }
    }
    for (uint32_t v = K + tid; v < Kp; v += kScanBlock) {
      t.outbase[v] = n_matched; t.binlim[v] = n_matched;
      if constexpr (!kPreview) t.dst.tot[v] = 0;
    }
  }
  if constexpr (!kPreview)
    for (uint32_t sg = warp; sg < n_segs; sg += NW) {  // chunk lists of the compacted pool
      const uint32_t c0 = s_nch[sg], c1 = s_nch[sg + 1];
      for (uint32_t k = lane; k < c1 - c0; k += 32) t.dst.chunk_tab[(size_t)sg * t.dst.max_ch + k] = c0 + k;
    }
  __syncthreads();
}

template <bool kBudget>
__global__ void __launch_bounds__(kScanBlock) k_colscan(uint32_t R, const uint32_t* __restrict__ M, uint32_t* __restrict__ P,
                                                        const TailArgs t) {
  extern __shared__ __align__(16) uint32_t scratch[];  // max(kColScratchWords, tail_words(Kp, layout)) words
  __shared__ Geo geo;
  __shared__ uint32_t s_gtmp[33];
  if (blockIdx.x + 1 < gridDim.x) {
    geo_build<kScanBlock>(geo, t.fill, t.n_segs, R, s_gtmp);
    if (geo_use_colscan(geo)) colscan_cols_body(scratch, geo, blockIdx.x, t.Kp, t.K, t.bin_seg, M, P);
  } else {
    colscan_tail_body<false, kBudget>(scratch, t);
  }
}

// mm_lobby_candidates: the tail up to the per-queue lobby counts, on the resident bin totals (tail_words words)
__global__ void __launch_bounds__(kScanBlock) k_lobby_candidates(const TailArgs t) {
  extern __shared__ __align__(16) uint32_t scratch[];
  colscan_tail_body<true>(scratch, t);
}

}  // namespace mm
