// mm_recut.cuh — mm_import_regroup_many: K mm_export images written under one config (the old ranks of a sharded
// deployment) re-filed into this engine's layout partitions and merged.  Each image first runs the regroup pipeline
// of mm_regroup.cuh on its own (classify with the `keep` selection, the stable scatter, the age merge); then, for
// K > 1:
//   k_rc_sum       per new partition q: the kept players of every image, their offsets, the (image, q) run counts.
//   k_rg_plan      (again) the image runs of every new partition: run ordinals and starts.
//   k_rc_gather    per image: refuses a repeated age inside a new partition (as k_rg_finish), and writes its players
//                  of q as one run, at the run's start, keyed by (stamp, image, age).
//   k_rc_runmax / k_rc_carry / k_rc_apply   the running maximum of the stamps along every (image, q) run: a
//                  segmented inclusive max scan, block by block, then across the blocks.
//   k_rg_merge<RcKey>   ceil(log2 K) rounds merge the image runs of each q by (running max, image, age): the order of
//                  a classic head-comparison merge by running-max stamp, ties to the lower image.
//   k_rc_finish    the kept players' columns in that order; each player's position.
//   k_rg_merge<RcKey>   ceil(log2 S) more rounds over the S partition lists (each sorted by the same key) give the
//                  one global order; k_rc_number writes each player's position in it as its new sequence number.
#pragma once

#include "mm_regroup.cuh"

namespace mm {

constexpr uint32_t kRcMaxImages = 64;
constexpr uint32_t kRcBlock = 1024;  // k_rc_runmax: 256 threads x 4 consecutive positions

// the order key of a player among the images' runs: hi = running-max stamp << 32 | image, lo = age in its image
struct __align__(16) RcKey {
  uint64_t hi;
  uint32_t lo, pad;
};
__device__ __forceinline__ bool operator<(const RcKey& a, const RcKey& b) {
  return a.hi < b.hi || (a.hi == b.hi && a.lo < b.lo);
}
__device__ __forceinline__ bool operator==(const RcKey& a, const RcKey& b) { return a.hi == b.hi && a.lo == b.lo; }

// One CTA.  rq_img[k][0 .. S+1]: image k's kept offsets per new partition (k_rq_scan).  -> rq_glob[0 .. S] the
// offsets of all kept players, rq_one = {0, kept}, pair[k][q] = image k's players of q.
__global__ void __launch_bounds__(1024) k_rc_sum(uint32_t K, uint32_t S, const uint32_t* __restrict__ rq_img,
                                                 uint32_t* __restrict__ rq_glob, uint32_t* __restrict__ rq_one,
                                                 uint32_t* __restrict__ pair) {
  for (uint32_t q = threadIdx.x; q <= S; q += blockDim.x) {
    uint32_t s = 0;
    for (uint32_t k = 0; k < K; ++k) {
      const uint32_t* r = rq_img + (size_t)k * (S + 2);
      s += r[q];
      if (q < S) pair[(size_t)k * S + q] = r[q + 1] - r[q];
    }
    rq_glob[q] = s;
    if (q == S) { rq_one[0] = 0; rq_one[1] = s; }
  }
}

struct RcGatherArgs {
  uint32_t k, base, n, n_segs, n_img;  // image, its first virtual index, its players, S, K
  const uint32_t* rq_off;              // [S + 2] the image's kept offsets per new partition
  const uint32_t* kmax;                // the age merge's: its result is in src[rounds & 1]
  const uint32_t* src[2];
  const uint32_t* age[2];
  const uint16_t* ord;                 // [K][S] ordinal of image k's run among q's image runs
  const uint32_t* run_start;           // [S][K + 1]
  const uint32_t* ts;                  // the image's stamps
  uint32_t* src_out;                   // virtual index (base + image index) at a position
  RcKey* key_out;
  uint8_t* head;                       // 1: the first position of an (image, q) run
  uint16_t* img;                       // [virtual index] image
  uint16_t* qv;                        // [virtual index] new partition
  uint32_t* err;
};

__global__ void __launch_bounds__(256) k_rc_gather(const RcGatherArgs a) {
  __shared__ uint32_t s_off[kMaxSegs + 1];
  for (uint32_t p = threadIdx.x; p <= a.n_segs; p += blockDim.x) s_off[p] = a.rq_off[p];
  __syncthreads();
  const uint32_t kept = s_off[a.n_segs], b = rg_rounds(*a.kmax) & 1u;
  const uint32_t* src = a.src[b];
  const uint32_t* age = a.age[b];
  bool bad = false;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < kept; i += gridDim.x * blockDim.x) {
    const uint32_t q = last_le(s_off, 0, a.n_segs, i), local = src[i];
    if (i + 1 < s_off[q + 1] && age[i + 1] == age[i]) bad = true;
    if (local >= a.n) { bad = true; continue; }  // only after a failed check: the merge had holes
    const uint32_t v = a.base + local;
    const uint32_t dst = a.run_start[(size_t)q * (a.n_img + 1) + a.ord[(size_t)a.k * a.n_segs + q]] + (i - s_off[q]);
    a.src_out[dst] = v;
    RcKey key;
    key.hi = ((uint64_t)a.ts[local] << 32) | a.k;
    key.lo = age[i];
    key.pad = 0;
    a.key_out[dst] = key;
    a.head[dst] = i == s_off[q];
    a.img[v] = (uint16_t)a.k;
    a.qv[v] = (uint16_t)q;
  }
  if (__any_sync(0xFFFFFFFFu, bad) && (threadIdx.x & 31) == 0) atomicOr(a.err, kImgBadSeq);
}

// ---- the running stamp maximum: a segmented inclusive max scan over the kept positions ----------------------------
// (f, v): f = a run starts inside the span, v = the max since the last run start (or of the whole span)
struct RcSeg {
  uint32_t f, v;
};
__device__ __forceinline__ RcSeg rc_seg(RcSeg a, RcSeg b) { return RcSeg{a.f | b.f, b.f ? b.v : max(a.v, b.v)}; }
__device__ __forceinline__ RcSeg shfl_up(const RcSeg& s, int off) { return RcSeg{shfl_up(s.f, off), shfl_up(s.v, off)}; }
// the CTA scans' combine operator (block_excl_scan_op)
struct RcSegOp {
  __device__ __forceinline__ RcSeg operator()(RcSeg a, RcSeg b) const { return rc_seg(a, b); }
};

// Block b scans positions [b * kRcBlock, (b + 1) * kRcBlock) of the n = *kept: the stamp field of key.hi becomes the
// max since the last run start inside the block; agg[b] = the block's (f, v), first[b] = its first run start (or its
// end).
__global__ void __launch_bounds__(256) k_rc_runmax(const uint32_t* __restrict__ kept, RcKey* __restrict__ key,
                                                   const uint8_t* __restrict__ head, RcSeg* __restrict__ agg,
                                                   uint32_t* __restrict__ first) {
  __shared__ RcSeg s_warp[8];
  __shared__ uint32_t s_first;
  const uint32_t n = *kept, b0 = blockIdx.x * kRcBlock;
  if (b0 >= n) return;
  if (threadIdx.x == 0) s_first = min(kRcBlock, n - b0);
  __syncthreads();
  const uint32_t p0 = b0 + threadIdx.x * 4;
  RcSeg t{0, 0};
  uint32_t f[4], v[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t p = p0 + j;
    f[j] = p < n ? head[p] : 0u;
    v[j] = p < n ? (uint32_t)(key[p].hi >> 32) : 0u;
    t = rc_seg(t, RcSeg{f[j], v[j]});
    if (f[j]) atomicMin(&s_first, p - b0);
  }
  RcSeg run = block_excl_scan_op<256>(t, RcSeg{0, 0}, RcSegOp{}, s_warp);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t p = p0 + j;
    run = rc_seg(run, RcSeg{f[j], v[j]});
    if (p < n) key[p].hi = ((uint64_t)run.v << 32) | (key[p].hi & 0xFFFFFFFFull);
  }
  if (threadIdx.x == (min(kRcBlock, n - b0) - 1) / 4) agg[blockIdx.x] = run;  // it holds the block's last position
  __syncthreads();
  if (threadIdx.x == 0) first[blockIdx.x] = s_first;
}

// One CTA: carry[b] = the exclusive scan of agg over the blocks before b.
__global__ void __launch_bounds__(1024) k_rc_carry(const uint32_t* __restrict__ kept, const RcSeg* __restrict__ agg,
                                                   RcSeg* __restrict__ carry) {
  __shared__ RcSeg s_warp[32];
  const uint32_t nb = (*kept + kRcBlock - 1) / kRcBlock, per = (nb + 1023) / 1024;
  const uint32_t b0 = threadIdx.x * per, b1 = min(nb, b0 + per);
  RcSeg t{0, 0};
  for (uint32_t b = b0; b < b1; ++b) t = rc_seg(t, agg[b]);
  RcSeg run = block_excl_scan_op<1024>(t, RcSeg{0, 0}, RcSegOp{}, s_warp);
  for (uint32_t b = b0; b < b1; ++b) {
    carry[b] = run;
    run = rc_seg(run, agg[b]);
  }
}

// The positions of block b before its first run start continue the run of the blocks before.
__global__ void __launch_bounds__(256) k_rc_apply(const uint32_t* __restrict__ kept, RcKey* __restrict__ key,
                                                  const RcSeg* __restrict__ carry, const uint32_t* __restrict__ first) {
  const uint32_t n = *kept, b0 = blockIdx.x * kRcBlock;
  if (blockIdx.x == 0 || b0 >= n) return;
  const uint32_t c = carry[blockIdx.x].v, end = b0 + first[blockIdx.x];
  for (uint32_t p = b0 + threadIdx.x; p < end; p += blockDim.x) {
    const uint32_t v = max(c, (uint32_t)(key[p].hi >> 32));
    key[p].hi = ((uint64_t)v << 32) | (key[p].hi & 0xFFFFFFFFull);
  }
}

struct RcFinishArgs {
  const uint32_t* rq_glob;   // [S + 1]
  uint32_t n_segs;
  const uint32_t* kmax;      // the image-run merge's: its result is in src[rounds & 1]
  uint32_t* src[2];
  RcKey* key[2];
  const ImgCols* imgs;       // [K] every image's columns
  const uint16_t* img;       // [virtual index] image
  const uint32_t* base;      // [K] first virtual index of the image
  ImgCols out;
  uint32_t* pos;             // [virtual index] position in the new order
};

// The kept players' columns in the merged order, and the order moved to buffer 0 for the numbering rounds.
__global__ void __launch_bounds__(256) k_rc_finish(const RcFinishArgs a) {
  const uint32_t kept = a.rq_glob[a.n_segs], b = rg_rounds(*a.kmax) & 1u;
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < kept; p += gridDim.x * blockDim.x) {
    const uint32_t v = a.src[b][p], k = a.img[v], i = v - a.base[k];
    const ImgCols& in = a.imgs[k];
    if (in.id_bytes == 8) static_cast<uint64_t*>(a.out.id)[p] = static_cast<const uint64_t*>(in.id)[i];
    else static_cast<uint32_t*>(a.out.id)[p] = static_cast<const uint32_t*>(in.id)[i];
    a.out.rating[p] = in.rating[i]; a.out.ts[p] = in.ts[i]; a.out.mode[p] = in.mode[i];
    a.pos[v] = p;
    if (b) { a.src[0][p] = v; a.key[0][p] = a.key[1][p]; }
  }
}

// the player at global position g gets sequence number g
__global__ void __launch_bounds__(256) k_rc_number(const uint32_t* __restrict__ kept, const uint32_t* __restrict__ gsrc,
                                                   const uint32_t* __restrict__ pos, uint32_t* __restrict__ seq) {
  const uint32_t n = *kept;
  for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < n; g += gridDim.x * blockDim.x) seq[pos[gsrc[g]]] = g;
}

}  // namespace mm
