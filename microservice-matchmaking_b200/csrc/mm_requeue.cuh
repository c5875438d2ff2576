// mm_requeue.cuh — requeue (mm_requeue): players of a lobby that did not start go back into their queue at the
// position their enqueue sequence number gives them.
//
// The call is an in-engine export, merge and import of the partitions it touches:
//   k_rq_check  checks every entry (the checks of img_player, clamp_key for the group, strict age order, one copy per id
//               through seen_insert) and classifies its active-set entry: 0 = a live queued player (gen << 32 |
//               slot on a live slot, the test of k_img_active), 1 = active and not queued (matched, taken), 4 = not
//               active.  Code-1 entries are counted per (ingest-sized block, partition).
//   k_rq_scan   turns the block counts into each block's first index among its partition's code-1 entries, the
//               partitions' offsets, and the selection of touched partitions.
//   (export passes 1 and 2 of mm_image.cuh gather the live players of the touched partitions, in enqueue order)
//   k_rq_group  writes the code-1 entries partition by partition, in age order (a stable counting sort).
//   k_rq_merge  gives every player of a touched partition its index in the merged list: a live player's index plus the
//               requeued entries of its partition that are older, a requeued entry's rank plus the live players that
//               are older (binary searches: last_le, first_not).  An equal sequence number is a collision.
//   k_rq_layout puts the touched partitions on fresh chunks (the host's layout, as import_image) and rebuilds their bin
//               totals; k_img_load then writes the merged columns, and k_restamp points the entries at the new slots.
#pragma once

#include "mm_image.cuh"

namespace mm {

constexpr uint32_t kRqItems = 1024;  // entries per k_rq_check / k_rq_group block: 256 threads x 4, warp-striped

// error bits of a requeue (the host names them in mm_last_error)
constexpr uint32_t kRqBadId = 1, kRqBadMode = 2, kRqBadRating = 4, kRqOrder = 8, kRqSeqNext = 16, kRqDup = 32,
                   kRqSeqLive = 64;

struct RqCheckArgs {
  const uint64_t* id;
  const int32_t* rating;
  const uint8_t* mode;
  const uint32_t* seq;
  uint32_t n, n_segs, nblk;
  BinMap bm;
  const uint8_t* grp_lut;
  const uint16_t* bin_seg;
  uint32_t n_modes, seq_next;
  uint64_t id_limit;
  ActiveView act;
  const uint8_t* pool_mode;
  uint32_t n_slots, gen;
  unsigned long long* seen;  // empty scratch id set of seen_mask + 1 keys, at most half full
  uint64_t seen_mask;
  uint8_t* code;             // [n] 0 / 1 / 4
  uint16_t* part;            // [n] partition of a code-1 entry, kNoPart otherwise
  uint32_t* blockhist;       // [n_segs][nblk] code-1 entries of the block in the partition
  uint32_t* err;
};

__global__ void __launch_bounds__(256) k_rq_check(const RqCheckArgs a) {
  __shared__ uint32_t s_hist[kMaxSegs];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (uint32_t p = tid; p < a.n_segs; p += 256) s_hist[p] = 0;
  __syncthreads();
  uint32_t bad = 0;
#pragma unroll 1
  for (int j = 0; j < 4; ++j) {
    const uint32_t i = blockIdx.x * kRqItems + warp * 128 + j * 32 + lane;
    if (i >= a.n) continue;
    const uint64_t pid = a.id[i];
    const uint32_t md = a.mode[i], u = a.seq[i] - a.seq_next;
    uint32_t b = 0, p = kNoPart;
    if (pid >= a.id_limit) b |= kRqBadId;
    if (md >= a.n_modes) {
      b |= kRqBadMode;
    } else {
      if (a.grp_lut[clamp_key(a.bm.key_lo, a.bm.KR, a.rating[i])] == 0xFF) b |= kRqBadRating;
      else p = a.bin_seg[bin_of(a.bm, a.bm.lut, a.rating[i], md)];
    }
    if (u == 0) b |= kRqSeqNext;
    if (i + 1 < a.n && a.seq[i + 1] - a.seq_next <= u) b |= kRqOrder;
    uint8_t c = 4;
    if (!(b & kRqBadId)) {
      if (!seen_insert(a.seen, a.seen_mask, pid)) b |= kRqDup;
      const uint64_t h = act_find(a.act, pid);
      const unsigned long long v = h == ~0ull ? kFreeVal : *a.act.val(h);
      if (v < kPending) {
        const uint32_t slot = (uint32_t)v;
        const bool live = ((uint32_t)(v >> 32) == a.gen && slot < a.n_slots && a.pool_mode[slot] != MM_MODE_DEAD) ||
                          pt_queued(v);  // queued in a party
        c = live ? 0 : 1;
      }
    }
    bad |= b;
    if (c != 1 || p == kNoPart) p = kNoPart;
    else atomicAdd(&s_hist[p], 1u);
    a.code[i] = c;
    a.part[i] = (uint16_t)p;
  }
  bad = __reduce_or_sync(0xFFFFFFFFu, bad);
  if (lane == 0 && bad) atomicOr(a.err, bad);
  __syncthreads();
  for (uint32_t p = tid; p < a.n_segs; p += 256) a.blockhist[(size_t)p * a.nblk + blockIdx.x] = s_hist[p];
}

// One CTA: per partition (one warp each) the exclusive scan of its block counts; the partitions' offsets rq_off[0 ..
// n_segs] among all code-1 entries; every block count then becomes the block's first index in the grouped list.
// sel[p] = the partition receives players.  n_segs may be kMaxSegs + 1 (mm_import_regroup adds a reject bucket).
__global__ void __launch_bounds__(512) k_rq_scan(uint32_t n_segs, uint32_t nblk, uint32_t* __restrict__ blockhist,
                                                 uint32_t* __restrict__ rq_off, uint8_t* __restrict__ sel) {
  __shared__ uint32_t s_off[kMaxSegs + 1], s_tmp[64];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (uint32_t p = warp; p < n_segs; p += 16) {
    uint32_t* hrow = blockhist + (size_t)p * nblk;
    const uint32_t carry = warp_col_scan(hrow, hrow, nblk);
    if (lane == 0) { s_off[p] = carry; sel[p] = carry != 0; }
  }
  __syncthreads();
  const uint32_t total = block_excl_scan<512>(s_off, n_segs, s_tmp);
  for (uint32_t p = tid; p < n_segs; p += 512) rq_off[p] = s_off[p];
  if (tid == 0) rq_off[n_segs] = total;
  __syncthreads();
  for (uint32_t p = warp; p < n_segs; p += 16) {
    uint32_t* hrow = blockhist + (size_t)p * nblk;
    for (uint32_t b = lane; b < nblk; b += 32) hrow[b] += s_off[p];
  }
}

// The code-1 entries partition by partition, in age order: grp_src[k] = the entry, grp_u[k] = its age (seq - seq_next).
// The rank inside the block is stable: peers of a partition in a warp by __match_any_sync, per-warp counters in shared
// memory, a prefix over the block's 8 warps (each warp holds 128 consecutive entries).  n_segs <= kMaxSegs + 1, as in
// k_rq_scan.
__global__ void __launch_bounds__(256) k_rq_group(uint32_t n, uint32_t n_segs, uint32_t nblk,
                                                  const uint16_t* __restrict__ part, const uint32_t* __restrict__ seq,
                                                  uint32_t seq_next, const uint32_t* __restrict__ blockbase,
                                                  uint32_t* __restrict__ grp_src, uint32_t* __restrict__ grp_u) {
  __shared__ uint16_t s_wc[8][kMaxSegs + 2];
  __shared__ uint32_t s_base[kMaxSegs + 1];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t S1 = n_segs + 1;  // digit n_segs = not a code-1 entry
  for (uint32_t k = tid; k < 8 * (kMaxSegs + 2); k += 256) (&s_wc[0][0])[k] = 0;
  for (uint32_t p = tid; p < n_segs; p += 256) s_base[p] = blockbase[(size_t)p * nblk + blockIdx.x];
  __syncthreads();
  uint32_t dg[4], rk[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t i = blockIdx.x * kRqItems + warp * 128 + j * 32 + lane;
    const uint32_t p = i < n ? part[i] : kNoPart;
    dg[j] = p == kNoPart ? n_segs : p;
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, dg[j]);
    const uint32_t leader = __ffs(peers) - 1;
    uint32_t old = 0;
    if (lane == leader) { old = s_wc[warp][dg[j]]; s_wc[warp][dg[j]] = (uint16_t)(old + __popc(peers)); }
    __syncwarp();
    old = __shfl_sync(0xFFFFFFFFu, old, leader);
    rk[j] = old + __popc(peers & ((1u << lane) - 1u));
  }
  __syncthreads();
  for (uint32_t p = tid; p < S1; p += 256) {  // prefix over the 8 warps
    uint32_t run = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) { const uint32_t v = s_wc[w][p]; s_wc[w][p] = (uint16_t)run; run += v; }
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (dg[j] >= n_segs) continue;
    const uint32_t i = blockIdx.x * kRqItems + warp * 128 + j * 32 + lane;
    const uint32_t k = s_base[dg[j]] + s_wc[warp][dg[j]] + rk[j];
    grp_src[k] = i;
    grp_u[k] = seq[i] - seq_next;
  }
}

struct RqMergeArgs {
  ImgCols live;              // the touched partitions' live players (export pass 2), partition by partition
  const uint32_t* live_cnt;  // [n_segs] live players per partition (export pass 1; 0 for untouched partitions)
  uint32_t n_segs, seq_next;
  const uint32_t* rq_off;    // [n_segs + 1] (k_rq_scan)
  const uint32_t* grp_src;   // [n_rq] (k_rq_group)
  const uint32_t* grp_u;
  const uint64_t* id;        // the caller's entries
  const int32_t* rating;
  const uint8_t* mode;
  const uint32_t* ts;
  const uint32_t* seq;
  ImgCols out;               // the merged list, partition by partition, in enqueue order
  uint32_t* m_off;           // [n_segs + 1] out: first merged index of the partition (CTA 0 writes it)
  uint32_t* err;
};

// One merged player per thread: t < n_live a live player, else requeued entry t - n_live.  Both counts come from the
// device (the scans of the partition counts), so the host launches a grid for an upper bound before it reads them.
__global__ void __launch_bounds__(256) k_rq_merge(const RqMergeArgs a) {
  __shared__ uint32_t s_live[kMaxSegs + 1], s_rq[kMaxSegs + 1], s_tmp[64];
  for (uint32_t p = threadIdx.x; p <= a.n_segs; p += blockDim.x) {
    s_live[p] = p < a.n_segs ? a.live_cnt[p] : 0u;
    s_rq[p] = a.rq_off[p];
  }
  __syncthreads();
  const uint32_t n_live = block_excl_scan<256>(s_live, a.n_segs, s_tmp), n_rq = s_rq[a.n_segs];
  if (threadIdx.x == 0) s_live[a.n_segs] = n_live;
  __syncthreads();
  if (blockIdx.x == 0)
    for (uint32_t p = threadIdx.x; p <= a.n_segs; p += blockDim.x) a.m_off[p] = s_live[p] + s_rq[p];
  const uint32_t n = n_live + n_rq;
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
    const bool is_live = t < n_live;
    const uint32_t x = is_live ? t : t - n_live;
    const uint32_t p = last_le(is_live ? s_live : s_rq, 0, a.n_segs, x);
    if (is_live) {  // + the requeued entries of p that are older
      const uint32_t u = a.live.seq[x] - a.seq_next;
      const uint32_t l = first_not(s_rq[p], s_rq[p + 1], [&](uint32_t k) { return a.grp_u[k] < u; });
      img_copy(a.out, s_live[p] + s_rq[p] + (x - s_live[p]) + (l - s_rq[p]), a.live, x);
    } else {  // + the live players of p that are older; one of the same age is a collision
      const uint32_t u = a.grp_u[x];
      const uint32_t l = first_not(s_live[p], s_live[p + 1], [&](uint32_t k) { return a.live.seq[k] - a.seq_next < u; });
      if (l < s_live[p + 1] && a.live.seq[l] - a.seq_next == u) { atomicOr(a.err, kRqSeqLive); continue; }
      const uint32_t dst = s_live[p] + s_rq[p] + (x - s_rq[p]) + (l - s_live[p]);
      const uint32_t i = a.grp_src[x];
      img_set_id(a.out, dst, a.id[i]);
      a.out.rating[dst] = a.rating[i]; a.out.ts[dst] = a.ts ? a.ts[i] : 0u; a.out.seq[dst] = a.seq[i];
      a.out.mode[dst] = a.mode[i];
    }
  }
}

// One CTA per partition; only the touched ones (sel) change: the fill becomes the merged count, the chunk list the
// fresh chunks from slot_base[p] / kTile on (zeroed histograms), the bin totals of the partition zero (k_img_load adds
// the players back).  CTA 0 also takes the touched partitions' dead slots out of the dead bin and sets the bump.
__global__ void k_rq_layout(PoolMeta meta, uint32_t n_segs, const uint8_t* __restrict__ sel,
                            const uint32_t* __restrict__ m_off, const uint32_t* __restrict__ slot_base,
                            const uint32_t* __restrict__ seg_bin_lo, uint32_t dead_bin, uint32_t dead, uint32_t bump) {
  const uint32_t p = blockIdx.x;
  if (p == 0 && threadIdx.x == 0) {
    meta.tot[dead_bin] -= dead;
    *meta.bump = bump;
  }
  if (p >= n_segs || !sel[p]) return;
  const uint32_t cnt = m_off[p + 1] - m_off[p], nch = (cnt + kTile - 1) / kTile, c0 = slot_base[p] / kTile;
  if (threadIdx.x == 0) meta.fill[p] = cnt;
  for (uint32_t k = threadIdx.x; k < nch; k += blockDim.x) meta.chunk_tab[(size_t)p * meta.max_ch + k] = c0 + k;
  if (meta.chist)
    for (size_t w = threadIdx.x; w < (size_t)nch * kChunkHist; w += blockDim.x) meta.chist[(size_t)c0 * kChunkHist + w] = 0;
  for (uint32_t b = seg_bin_lo[p] + threadIdx.x; b < seg_bin_lo[p + 1]; b += blockDim.x) meta.tot[b] = 0;
}

}  // namespace mm
