// mm_regroup.cuh — mm_import_regroup: an mm_export image written under another config (rating groups, default group,
// modes, order, MM_F_WIDE_PARTITIONS) re-filed into this engine's layout partitions, every player keeping its id,
// rating, mode, stamp and sequence number.
//
//   k_rg_classify  one pass over the image columns: every player checked under the IMAGE's layout (img_player, the
//                  checks of k_img_load), then given its partition under the ENGINE's layout, or the reject bucket
//                  n_segs (no group, or a mode the engine does not have); a player of a partition `keep` does not
//                  select (mm_import_regroup_many) is skipped: counted, and left out like a player that failed a check.
//                  Counts per (1024-player block, bucket) for
//                  the stable counting scatter of mm_requeue.cuh (k_rq_scan, k_rq_group), and per (image partition,
//                  new partition) pair: the sorted runs each new partition will hold.
//   k_rg_dups      one copy per id over the players and the active section (what k_img_insert refuses), before
//                  anything is written.
//   k_rq_scan / k_rq_group   the stable scatter by bucket: a new partition is then k runs in image-partition order, each
//                  in age order (an image partition is age-sorted); the reject bucket is in ascending image order.
//   k_rg_plan      per new partition, the position of each run (by its ordinal among the runs) and the ordinal of each
//                  image partition; the largest run count k_max.
//   k_rg_merge     round t merges super-runs 2s and 2s+1 of 2^t runs each: every player finds its place by one binary
//                  search in the partner super-run (ties: the left one first).  ceil(log2 k_max) rounds do work, so
//                  the cost per player is O(log n log k): no round when groups only split or their bounds move.
//   k_rg_finish    equal adjacent ages inside a new partition (a duplicate sequence number) -> refusal; the kept
//                  players' columns gathered in the new order; the reject bucket copied out.
// The host reads the counters once, decides every refusal, and only then runs the load tail that mm_import runs.
#pragma once

#include "mm_image.cuh"
#include "mm_requeue.cuh"

namespace mm {

struct RgClassifyArgs {
  ImgCols in;
  uint32_t n, nblk;
  const uint32_t* part_off;   // [n_img_segs + 1] first image index of the image partition
  uint32_t n_img_segs;
  BinMap bm_img;              // the image's layout
  const uint8_t* grp_img;
  const uint16_t* bin_seg_img;
  uint32_t n_modes_img, seq_next;
  uint64_t id_limit;
  BinMap bm;                  // the engine's layout
  const uint8_t* grp_lut;
  const uint16_t* bin_seg;
  uint32_t n_modes, n_segs;
  const uint8_t* keep;        // [n_segs] selected new partitions; null: all
  uint32_t* n_skip;           // players of unselected partitions (keep != null)
  uint16_t* part;             // [n] new partition; n_segs = rejected; kNoPart = failed a check or skipped
  uint16_t* pimg;             // [n] image partition
  uint32_t* blockhist;        // [n_segs + 1][nblk]
  uint32_t* pair;             // [n_img_segs][n_segs] kept players per (image partition, new partition)
  uint32_t* err;
};

// The block geometry of k_rq_check / k_rq_group: block b holds entries b * kRqItems + warp * 128 + j * 32 + lane.
__global__ void __launch_bounds__(256) k_rg_classify(const RgClassifyArgs a) {
  __shared__ uint32_t s_off[kMaxSegs + 1], s_hist[kMaxSegs + 1];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (uint32_t p = tid; p <= a.n_img_segs; p += 256) s_off[p] = a.part_off[p];
  for (uint32_t p = tid; p <= a.n_segs; p += 256) s_hist[p] = 0;
  __syncthreads();
  uint32_t bad = 0, skip = 0;
#pragma unroll 1
  for (int j = 0; j < 4; ++j) {
    const uint32_t i = blockIdx.x * kRqItems + warp * 128 + j * 32 + lane;
    uint32_t key = ~0u;  // (image partition, new partition) of a kept player
    if (i < a.n) {
      const ImgPlayer x = img_player(a.in, i, s_off, a.n_img_segs, a.bm_img, a.grp_img, a.bin_seg_img, a.n_modes_img,
                                     a.seq_next, a.id_limit);
      uint32_t q = kNoPart;
      if (x.bad) {
        bad |= x.bad;
      } else if (x.md >= a.n_modes) {
        q = a.n_segs;
      } else {
        q = a.grp_lut[clamp_key(a.bm.key_lo, a.bm.KR, x.rt)] == 0xFF ? a.n_segs : a.bin_seg[bin_of(a.bm, a.bm.lut, x.rt, x.md)];
        if (a.keep && q < a.n_segs && !a.keep[q]) { q = kNoPart; ++skip; }
      }
      if (q != kNoPart) atomicAdd(&s_hist[q], 1u);
      if (q < a.n_segs) key = x.p * a.n_segs + q;
      a.part[i] = (uint16_t)q;
      a.pimg[i] = (uint16_t)x.p;
    }
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, key);
    if (key != ~0u && lane == __ffs(peers) - 1) atomicAdd(&a.pair[key], (uint32_t)__popc(peers));
  }
  bad = __reduce_or_sync(0xFFFFFFFFu, bad);
  if (lane == 0 && bad) atomicOr(a.err, bad);
  skip = __reduce_add_sync(0xFFFFFFFFu, skip);
  if (lane == 0 && skip) atomicAdd(a.n_skip, skip);
  __syncthreads();
  for (uint32_t p = tid; p <= a.n_segs; p += 256) a.blockhist[(size_t)p * a.nblk + blockIdx.x] = s_hist[p];
}

// Every copy of an id after the first, over the players (n) and the active section (m), into *count (`seen`: an empty
// scratch set of seen_mask + 1 keys, at most half full).
__global__ void k_rg_dups(const void* ids, const void* act_ids, uint32_t id_bytes, uint32_t n, uint32_t m,
                          unsigned long long* seen, uint64_t seen_mask, uint32_t* __restrict__ count) {
  uint32_t dup = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n + m; i += gridDim.x * blockDim.x) {
    const void* col = i < n ? ids : act_ids;
    const uint32_t k = i < n ? i : i - n;
    const uint64_t pid = id_bytes == 8 ? static_cast<const uint64_t*>(col)[k] : static_cast<const uint32_t*>(col)[k];
    if (!seen_insert(seen, seen_mask, pid)) ++dup;
  }
  dup = __reduce_add_sync(0xFFFFFFFFu, dup);
  if ((threadIdx.x & 31) == 0 && dup) atomicAdd(count, dup);
}

// One CTA, one warp per new partition q: its runs are the image partitions with pair[p][q] > 0, in p order, at
// rq_off[q] + the players of the runs before.  ord[p][q] = the run's ordinal; run_start[q][0 .. k_q] = the runs'
// first positions and the partition's end; kq[q] = k_q; *kmax = the largest k_q.
__global__ void __launch_bounds__(1024) k_rg_plan(uint32_t n_img_segs, uint32_t n_segs, const uint32_t* __restrict__ pair,
                                                  const uint32_t* __restrict__ rq_off, uint16_t* __restrict__ ord,
                                                  uint32_t* __restrict__ run_start, uint32_t* __restrict__ kq,
                                                  uint32_t* __restrict__ kmax) {
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (uint32_t q = warp; q < n_segs; q += 32) {
    uint32_t carry = rq_off[q], k = 0;
    uint32_t* rs = run_start + (size_t)q * (n_img_segs + 1);
    for (uint32_t p0 = 0; p0 < n_img_segs; p0 += 32) {
      const uint32_t p = p0 + lane;
      const uint32_t c = p < n_img_segs ? pair[(size_t)p * n_segs + q] : 0u;
      const uint32_t incl = warp_incl_scan(c);
      const uint32_t nz = __ballot_sync(0xFFFFFFFFu, c != 0);
      if (c) {
        const uint32_t j = k + __popc(nz & ((1u << lane) - 1u));
        ord[(size_t)p * n_segs + q] = (uint16_t)j;
        rs[j] = carry + incl - c;
      }
      carry += __shfl_sync(0xFFFFFFFFu, incl, 31);
      k += __popc(nz);
    }
    if (lane == 0) {
      rs[k] = carry;
      kq[q] = k;
      atomicMax(kmax, k);
    }
  }
}

// rounds of k_rg_merge that do work for k_max runs
__device__ __forceinline__ uint32_t rg_rounds(uint32_t kmax) { return kmax <= 1 ? 0u : 32u - __clz(kmax - 1); }

template <class Key>
struct RgMergeArgsT {
  const uint32_t* rq_off;     // [n_segs + 2] (k_rq_scan over n_segs + 1 buckets)
  uint32_t n_segs, n_img_segs, round;
  const uint16_t* pimg;
  const uint16_t* ord;
  const uint32_t* run_start;
  const uint32_t* kq;
  const uint32_t* kmax;
  const uint32_t* src_in;     // image index of the player at a position
  const Key* u_in;            // its key: the age (mm_import_regroup), an RcKey (mm_recut.cuh)
  uint32_t* src_out;
  Key* u_out;
};
using RgMergeArgs = RgMergeArgsT<uint32_t>;

// Key: ordered by < and ==; every run must be sorted by it.
template <class Key>
__global__ void __launch_bounds__(256) k_rg_merge(const RgMergeArgsT<Key> a) {
  __shared__ uint32_t s_off[kMaxSegs + 1];
  if ((1u << a.round) >= *a.kmax) return;  // (uniform) every partition is one sorted run already
  for (uint32_t p = threadIdx.x; p <= a.n_segs; p += blockDim.x) s_off[p] = a.rq_off[p];
  __syncthreads();
  const uint32_t kept = s_off[a.n_segs], t = a.round;
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < kept; k += gridDim.x * blockDim.x) {
    const uint32_t q = last_le(s_off, 0, a.n_segs, k);
    const uint32_t src = a.src_in[k];
    const Key u = a.u_in[k];
    const uint32_t s = a.ord[(size_t)a.pimg[src] * a.n_segs + q] >> t, ps = s ^ 1u, K = a.kq[q];
    const uint32_t* rs = a.run_start + (size_t)q * (a.n_img_segs + 1);
    uint32_t dst = k;
    if ((ps << t) < K) {
      const uint32_t A = rs[s << t], C = rs[ps << t], D = rs[min((ps + 1) << t, K)];
      const bool left = !(s & 1u);  // left: the partner's players older than u; right: older or of the same age
      const uint32_t l = first_not(C, D, [&](uint32_t m) {
        const Key v = a.u_in[m];
        return v < u || (!left && v == u);
      });
      dst = left ? k + (l - C) : k - A + l;
    }
    a.src_out[dst] = src;
    a.u_out[dst] = u;
  }
}

struct RgFinishArgs {
  const uint32_t* rq_off;
  uint32_t n_segs, n;
  const uint32_t* kmax;
  const uint32_t* src[2];  // the merge buffers: the result is in src[rounds & 1]; the reject bucket in src[0]
  const uint32_t* u[2];
  ImgCols in, out;         // image columns -> the kept players' columns in the new order
  uint32_t* rejected;      // [rejects] ascending image indices
  uint32_t* err;
};

__global__ void __launch_bounds__(256) k_rg_finish(const RgFinishArgs a) {
  __shared__ uint32_t s_off[kMaxSegs + 2];
  for (uint32_t p = threadIdx.x; p <= a.n_segs + 1; p += blockDim.x) s_off[p] = a.rq_off[p];
  __syncthreads();
  const uint32_t kept = s_off[a.n_segs], total = s_off[a.n_segs + 1], b = rg_rounds(*a.kmax) & 1u;
  const uint32_t* src = a.src[b];
  const uint32_t* age = a.u[b];
  bool bad = false;
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < total; k += gridDim.x * blockDim.x) {
    if (k >= kept) { a.rejected[k - kept] = a.src[0][k]; continue; }
    const uint32_t q = last_le(s_off, 0, a.n_segs, k), i = src[k];
    if (k + 1 < s_off[q + 1] && age[k + 1] == age[k]) bad = true;
    if (i >= a.n) { bad = true; continue; }  // only after a failed check: the merge had holes
    img_copy(a.out, k, a.in, i);
  }
  if (__any_sync(0xFFFFFFFFu, bad) && (threadIdx.x & 31) == 0) atomicOr(a.err, kImgBadSeq);
}

}  // namespace mm
