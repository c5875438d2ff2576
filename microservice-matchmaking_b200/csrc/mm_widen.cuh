// mm_widen.cuh — widening search on the device (mm_widen, DESIGN §4): lobbies formed around the players who have waited
// longest, each in a rating window that grows with its anchor's wait.
//
// Anchors (k_wd_anchors, two passes over the tiles of the enabled queues' partitions, shaped like k_expire): the first
// counts the live players whose WAIT reaches their queue's min_wait per CTA and per partition; the second writes their
// slots and ages at the CTA's scanned offset in tile order, so every partition's anchors form one run in storage (=
// age) order.  k_wd_rank gives each anchor its rank among the live players of its bin in enqueue order (bin_rank, the
// computation of k_locate).
//
// Plan (k_wd_plan): one warp per enabled queue serves the queue's anchors oldest first, merging the runs of its
// partitions by age.  rem[bin] starts from tot and counts the bin's players no earlier lobby of the call took; lobbies
// take the oldest untaken players of a bin, so the taken players of a bin are its rank prefix [0, tot - rem) and an
// anchor whose rank lies in it is absorbed.  Otherwise the warp walks the bins outward from the anchor's own bin in
// (distance, rating) order inside the anchor's window (bf_walk, k_bf_plan's walk): a first walk only counts, and only
// when it reaches the lobby size L does a second walk take the players, one PIECE per (lobby, bin) with its offset
// inside the lobby in member order (rating, then enqueue order).
//
// Off-tick budget: k_wd_allot turns the plan's per-queue lobby counts into allowances; when one falls short, the host
// resets the plan's state and runs it again with the allowances as caps (WdArgs::cap).
//
// Take and output: k_bf_keys turns the taken prefixes into keys and the band pipeline takes them into staging, as for
// mm_backfill; k_wd_bases scans the per-queue lobby counts, k_wd_hdr writes the headers and every lobby's member base,
// and k_bf_out copies the pieces into place.
#pragma once

#include "mm_backfill.cuh"
#include "mm_locate.cuh"
#include "mm_stats.cuh"

namespace mm {

static_assert(sizeof(mm_widen_rule) == 24, "mm_widen_rule is 24 bytes (include/mm_engine.h)");
static_assert(sizeof(mm_widen_stats) == 32, "mm_widen_stats is 32 bytes (include/mm_engine.h)");

constexpr uint32_t kWdBlock = 256;  // 8 slots per thread: one tile per CTA step
static_assert(kWdBlock * 8 == kTile, "a CTA step covers one tile");
constexpr uint32_t kWdPlanWarps = 4;

// ctr words of one call (zeroed by the host); the first kBfWords are k_bf_keys' and the pieces' (BfCtr)
enum WdCtr : uint32_t { kWdLobbies = kBfWords, kWdAbsorbed, kWdWords };

struct WdRule {       // one per queue, as the device reads it
  uint32_t min_wait;  // MM_WIDEN_OFF: the queue is not served
  uint32_t step;
  int32_t w0, inc, w_max;
  uint32_t L;         // lobby size of the queue's mode
};

struct WdArgs {
  PoolView pool;
  PoolMeta meta;
  uint32_t n_segs, n_cut, n_groups, now, seq_next;
  const WdRule* rule;          // [n_cut]
  const uint16_t* part_cut;    // [n_segs] partition -> queue
  const uint32_t* cut_lp_lo;   // [n_cut + 1] first partition of the queue
  const uint32_t* seg_bin_lo;  // [n_segs + 1]
  const uint16_t* bin_seg;     // [Kp]
  const uint16_t* bin_key;     // [Kp] clamp key of the bin
  const uint32_t* tot;         // the pool's per-bin totals
  uint32_t* rem;               // [K] tot minus what this call took so far
  const uint32_t* rmap;        // k_loc_rmap
  uint32_t* cta;               // [grid] anchors per CTA (first pass)
  uint32_t* part;              // [n_segs + 1] anchors per partition -> exclusive scan (k_wd_part_scan)
  uint32_t* cur;               // [n_segs] plan: next anchor of the partition's run
  uint32_t n_anchors;
  uint32_t* a_slot;            // [n_anchors] in (partition, age) order
  uint32_t* a_age;             // [n_anchors] (seq - seq_next) mod 2^32
  uint32_t* a_rank;            // [n_anchors] rank in the bin
  uint2* rec;                  // [n_anchors] lobby record: (queue, index inside the queue)
  uint32_t* qlob;              // [n_cut] lobbies of the queue (0 for a queue not served)
  const uint32_t* cap;         // [n_cut] lobbies the queue may emit (the off-tick budget's allowance), or null
  uint32_t* qlbase;            // [n_cut] first lobby of the queue
  uint32_t* qmbase;            // [n_cut] first member slot of the queue
  BfPiece* piece;              // pieces: req = lobby record
  uint32_t* mbase;             // [n_anchors] member slot of the record's first member
  mm_lobby_hdr* hdr;
  uint32_t* ctr;               // [kWdWords]
};

// Anchors: `write` = 0 counts per CTA (cta[]) and per partition (part[]); 1 writes each CTA's anchors from the sum of
// the counts of the CTAs before it.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_wd_anchors(const WdArgs a, uint32_t write) {
  __shared__ Geo geo;
  __shared__ uint32_t s_gtmp[33];
  __shared__ uint32_t s_warp[BLOCK / 32];
  const uint32_t tid = threadIdx.x;
  uint32_t s0, s1;
  if (!geo_cta_run<BLOCK>(geo, a.meta.fill, a.n_segs, s_gtmp, s0, s1)) return;  // (uniform)
  uint32_t base = 0, counted = 0;
  if (write) {
    for (uint32_t c = tid; c < blockIdx.x; c += BLOCK) base += a.cta[c];
    base = __reduce_add_sync(0xFFFFFFFFu, base);
    block_warp_offsets<BLOCK>(base, counted, s_warp);  // lane 31 gives its warp's sum
    base = counted;
  }
  const uint32_t o = tid * 8;
  for (uint32_t s = s0; s < s1; ++s) {
    const TileDesc d = geo_tile(geo, a.meta, s);
    const uint32_t min_wait = a.rule[a.part_cut[d.seg]].min_wait;
    if (min_wait == MM_WIDEN_OFF) continue;  // (uniform)
    const size_t tb = (size_t)d.phys * kTile + o;
    uint32_t hit = 0;  // bit j: slot tb + j is an anchor
    if (o < d.nvalid) {
      const uint2 m2 = __ldcs(reinterpret_cast<const uint2*>(a.pool.mode + tb));
      uint32_t ts[8];
      ld_stamps8(a.pool.ts + tb, ts);
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (o + j < d.nvalid && mode8_at(m2, j) != MM_MODE_DEAD && stat_wait(a.now, ts[j]) >= min_wait) hit |= 1u << j;
    }
    const uint32_t k = __popc(hit);
    const uint32_t incl = warp_incl_scan(k);
    uint32_t total;
    const uint32_t before = block_warp_offsets<BLOCK>(__shfl_sync(0xFFFFFFFFu, incl, 31), total, s_warp);
    if (!write) {
      if (tid == 0 && total) atomicAdd(&a.part[d.seg], total);
      counted += total;
      continue;
    }
    uint32_t q = base + before + incl - k;
    for (int j = 0; j < 8; ++j) {
      if (!((hit >> j) & 1u)) continue;
      const uint32_t slot = (uint32_t)(tb + j);
      a.a_slot[q] = slot;
      a.a_age[q] = a.pool.seq[slot] - a.seq_next;
      ++q;
    }
    base += total;
  }
  if (!write && tid == 0) a.cta[blockIdx.x] = counted;
}

// One CTA: part[] -> its exclusive scan (part[n_segs] = the anchors), cur[] = the first anchor of every partition.
__global__ void __launch_bounds__(1024) k_wd_part_scan(const WdArgs a) {
  __shared__ uint32_t s_tmp[33];
  uint32_t carry = 0;
  for (uint32_t i0 = 0; i0 < a.n_segs; i0 += 1024) {
    const uint32_t i = i0 + threadIdx.x;
    const uint32_t v = i < a.n_segs ? a.part[i] : 0u;
    const uint32_t x = block_scan_step<1024>(v, carry, s_tmp);
    if (i < a.n_segs) { a.part[i] = x; a.cur[i] = x; }
  }
  if (threadIdx.x == 0) a.part[a.n_segs] = carry;
}

// One warp per anchor: its rank in its bin.
__global__ void __launch_bounds__(256) k_wd_rank(const WdArgs a) {
  const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= a.n_anchors) return;  // (uniform over the warp)
  const uint32_t slot = a.a_slot[i], v = a.pool.bin[slot];
  const uint32_t r = bin_rank(a.pool, a.meta, a.seg_bin_lo, a.rmap, slot, v, a.bin_seg[v]);
  if ((threadIdx.x & 31) == 0) a.a_rank[i] = r;
}

__global__ void __launch_bounds__(kWdPlanWarps * 32) k_wd_plan(const WdArgs a) {
  __shared__ uint32_t s_bin[kWdPlanWarps][32];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, c = blockIdx.x * kWdPlanWarps + warp;
  if (c >= a.n_cut) return;
  const WdRule u = a.rule[c];
  if (u.min_wait == MM_WIDEN_OFF) { if (lane == 0) a.qlob[c] = 0; return; }
  const uint32_t p0 = a.cut_lp_lo[c], p1 = a.cut_lp_lo[c + 1];
  const uint32_t lo = a.seg_bin_lo[p0], hi = a.seg_bin_lo[p1];
  const uint32_t cap = a.cap ? a.cap[c] : 0xFFFFFFFFu;
  uint32_t n_lob = 0, n_abs = 0;
  while (n_lob < cap) {  // a capped queue stops after its cap-th lobby: the rest of its anchors stay queued
    // the oldest anchor not yet served: the least age over the heads of the partitions' runs (ages are unique)
    unsigned long long best = ~0ull;
    for (uint32_t p = p0 + lane; p < p1; p += 32) {
      const uint32_t i = a.cur[p];
      if (i < a.part[p + 1]) best = min(best, ((unsigned long long)a.a_age[i] << 32) | p);
    }
#pragma unroll
    for (int s = 16; s; s >>= 1) best = min(best, __shfl_xor_sync(0xFFFFFFFFu, best, s));
    if (best == ~0ull) break;
    const uint32_t p = (uint32_t)best, i = a.cur[p];
    __syncwarp();
    if (lane == 0) a.cur[p] = i + 1;
    __syncwarp();
    const uint32_t slot = a.a_slot[i], v = a.pool.bin[slot];
    if (a.a_rank[i] < a.tot[v] - a.rem[v]) { ++n_abs; continue; }  // an earlier lobby of the call took it
    const uint32_t wait = stat_wait(a.now, a.pool.ts[slot]);
    const long long w = min((long long)u.w_max, (long long)u.w0 + (long long)((wait - u.min_wait) / u.step) * u.inc);
    const uint32_t win = (uint32_t)min(w, (long long)kBfFar - 1);
    uint32_t left = 0;
    const int32_t target = (int32_t)a.bin_key[v];
    if (bf_walk<false>(a, s_bin[warp], target, v, lo, hi, win, u.L, left, 0) < u.L) continue;  // all or nothing
    uint32_t r = 0;
    if (lane == 0) r = atomicAdd(&a.ctr[kWdLobbies], 1u);
    r = __shfl_sync(0xFFFFFFFFu, r, 0);
    if (lane == 0) a.rec[r] = make_uint2(c, n_lob);
    ++n_lob;
    bf_walk<true>(a, s_bin[warp], target, v, lo, hi, win, u.L, left, r);
  }
  if (lane == 0) {
    a.qlob[c] = n_lob;
    if (n_abs) atomicAdd(&a.ctr[kWdAbsorbed], n_abs);
  }
}

// One CTA, the off-tick budget (mm_set_offtick_budget) of an mm_widen / mm_party_match call after its unbudgeted plan:
// cand[q] = qlob[q] (c_q), allot[q] = a_q by the tick's apportionment (budget_apportion, one warp per mode) of bud_queue
// [n_cut] / bud_mode [n_modes] (either null: unlimited), *cut = 1 if some a_q < c_q (the plan runs again, capped).
__global__ void __launch_bounds__(kScanBlock) k_wd_allot(const WdArgs a, const uint32_t* bud_queue,
                                                         const uint32_t* bud_mode, uint32_t* cand, uint32_t* allot,
                                                         uint32_t* cut) {
  const uint32_t G = a.n_groups;
  for (uint32_t q = threadIdx.x; q < a.n_cut; q += kScanBlock) cand[q] = a.qlob[q];
  __syncthreads();
  for (uint32_t m = threadIdx.x >> 5; m < a.n_cut / G; m += kScanBlock / 32)
    budget_apportion(cand, allot, m, G, bud_queue, bud_mode);
  __syncthreads();
  bool less = false;
  for (uint32_t q = threadIdx.x; q < a.n_cut; q += kScanBlock) less |= allot[q] < cand[q];
  const int any = __syncthreads_or(less);
  if (threadIdx.x == 0) *cut = any ? 1u : 0u;
}

// One warp: the lobby and member bases of every queue (queue order = (mode, group) order).
__global__ void k_wd_bases(const WdArgs a) {
  const uint32_t lane = threadIdx.x & 31;
  uint32_t cl = 0, cm = 0;
  for (uint32_t c0 = 0; c0 < a.n_cut; c0 += 32) {
    const uint32_t c = c0 + lane;
    const uint32_t nl = c < a.n_cut && a.rule[c].min_wait != MM_WIDEN_OFF ? a.qlob[c] : 0u;
    const uint32_t nm = c < a.n_cut ? nl * a.rule[c].L : 0u;
    const uint32_t il = warp_incl_scan(nl), im = warp_incl_scan(nm);
    if (c < a.n_cut) { a.qlbase[c] = cl + il - nl; a.qmbase[c] = cm + im - nm; }
    cl += __shfl_sync(0xFFFFFFFFu, il, 31);
    cm += __shfl_sync(0xFFFFFFFFu, im, 31);
  }
}

// One thread per lobby record: its header and member base.
__global__ void k_wd_hdr(const WdArgs a, uint32_t n_rec) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rec) return;
  const uint2 x = a.rec[r];
  const uint32_t L = a.rule[x.x].L, mb = a.qmbase[x.x] + x.y * L;
  a.mbase[r] = mb;
  a.hdr[a.qlbase[x.x] + x.y] = mm_lobby_hdr{mb, (uint16_t)L, (uint8_t)(x.x / a.n_groups), (uint8_t)(x.x % a.n_groups)};
}

}  // namespace mm
