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

#include "mm_party.cuh"
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
  uint16_t* qv;                        // [virtual index] new partition + qoff
  uint32_t qoff;                       // 0 for the solos' partitions, S for the parties' queues
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
    a.qv[v] = (uint16_t)(q + a.qoff);
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

// ---- parties (mm_import_regroup_many_parties) ----------------------------------------------------------------------
// Party image k's parties take virtual indices N + pbase[k] + j after the N solos.  Per image:
//   k_rp_classify  the malformed-image checks, R, and the bucket: queue c = mode * n_groups + group(R), n_cut =
//                  rejected, kNoPart = failed a check or skipped; block counts for k_rq_scan / k_rq_group (the same
//                  stable scatter as the solos: a queue's parties stay in age order, the rejects in index order); each
//                  party's (image, age) into the sequence-number set.
//   k_rp_probe     a solo of image k whose (image, age) a party holds.
// n_images == 1: k_rp_rows1 gives the kept parties rows in image order and keeps their numbers.  n_images > 1: the
// queues' image runs go through the solos' machinery (k_rc_gather with qoff = S, the running maximum, k_rg_merge<RcKey>
// by queue), k_rp_norm, ceil(log2 n_cut) rounds merge the queue lists into the parties' order (= their rows), k_rp_place
// puts that list after the solos' global list, and one k_rg_merge round of the two lists gives the global order that
// k_rc_number numbers.  After the solos' load, k_rp_write writes the table rows, members and active-set values.
enum RpErr : uint32_t { kRpBadSize = 1, kRpBadSum = 2, kRpBadSeq = 4, kRpBadId = 8 };
enum RpCtr : uint32_t { kRpErrBits = 0, kRpSeqDup, kRpWords };  // then skip[K], kept members[K], member sums[K]

__device__ __forceinline__ uint64_t rp_seq_key(uint32_t k, uint32_t age) { return ((uint64_t)k << 32) | age; }

__device__ __forceinline__ bool seen_has(const unsigned long long* seen, uint64_t mask, uint64_t key) {
  for (uint64_t s = hash64(key) & mask;; s = (s + 1) & mask) {
    const unsigned long long k = seen[s];
    if (k == key) return true;
    if (k == kEmptyKey) return false;
  }
}

// floor(sum / s) of a party's member ratings, as k_pt_resolve computes it
__device__ __forceinline__ int32_t rp_rating(const int32_t* rating, uint32_t o, uint32_t s) {
  long long sum = 0;
  for (uint32_t k = 0; k < s; ++k) sum += rating[o + k];
  long long R = sum / (long long)s;
  if (R * (long long)s > sum) --R;
  return (int32_t)R;
}

__device__ __forceinline__ uint64_t rp_id(const PtImgCols& c, uint32_t m) {
  return c.id_bytes == 8 ? reinterpret_cast<const uint64_t*>(c.id)[m] : reinterpret_cast<const uint32_t*>(c.id)[m];
}

__global__ void k_rp_sizes(uint32_t n, const uint8_t* __restrict__ size, uint32_t* __restrict__ msz) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) msz[j] = size[j];
}

struct RpClassifyArgs {
  PtImgCols in;
  uint32_t k, n, m, nblk, seq_next;  // image, its parties, members, blocks, seq_next
  const uint32_t* moff;              // [n] member offsets (exclusive scan of the sizes)
  uint64_t id_limit;
  BinMap bm;
  const uint8_t* grp_lut;
  const uint8_t* mode_tsize;
  uint32_t n_modes, n_groups, n_cut;
  const uint8_t* keep;               // [n_cut] or null
  unsigned long long* seqset;
  uint64_t seq_mask;
  uint16_t* part;                    // [n] bucket
  uint16_t* pk;                      // [n] image
  int32_t* R;                        // [n]
  uint32_t* flag;                    // [n] 1: kept
  uint8_t* size;                     // [n] copy of the sizes, by party index
  uint32_t* blockhist;               // [n_cut + 1][nblk]
  uint32_t* ctr;                     // RpCtr words
  uint32_t* skip;                    // this image's skipped parties
  uint32_t* kmem;                    // this image's kept members
};

__global__ void __launch_bounds__(256) k_rp_classify(const RpClassifyArgs a) {
  __shared__ uint32_t s_hist[kMaxSegs + 1];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (uint32_t p = tid; p <= a.n_cut; p += 256) s_hist[p] = 0;
  __syncthreads();
  uint32_t bad = 0, skip = 0, kmem = 0, dup = 0;
#pragma unroll 1
  for (int j = 0; j < 4; ++j) {
    const uint32_t i = blockIdx.x * kRqItems + warp * 128 + j * 32 + lane;
    if (i >= a.n) continue;
    const uint32_t s = a.in.size[i], o = a.moff[i], md = a.in.mode[i], u = a.in.seq[i] - a.seq_next;
    uint32_t b = 0;
    if (s < 2) b |= kRpBadSize;
    if (o + s > a.m || o + s < o) b |= kRpBadSum;
    if (u == 0 || (i + 1 < a.n && a.in.seq[i + 1] - a.seq_next <= u)) b |= kRpBadSeq;
    uint32_t q = kNoPart;
    int32_t R = 0;
    if (!b) {
      for (uint32_t x = 0; x < s; ++x) b |= rp_id(a.in, o + x) >= a.id_limit ? (uint32_t)kRpBadId : 0u;
      R = rp_rating(a.in.rating, o, s);
    }
    if (b) {
      bad |= b;
    } else {
      const uint32_t g = a.grp_lut[clamp_key(a.bm.key_lo, a.bm.KR, R)];
      if (md >= a.n_modes || s > a.mode_tsize[md] || g == 0xFF) {
        q = a.n_cut;
      } else {
        q = md * a.n_groups + g;
        if (a.keep && !a.keep[q]) { q = kNoPart; ++skip; }
      }
    }
    if (q != kNoPart) atomicAdd(&s_hist[q], 1u);
    if (q < a.n_cut) kmem += s;
    if (!seen_insert(a.seqset, a.seq_mask, rp_seq_key(a.k, u))) ++dup;
    a.part[i] = (uint16_t)q;
    a.pk[i] = (uint16_t)a.k;
    a.R[i] = R;
    a.flag[i] = q < a.n_cut;
    a.size[i] = (uint8_t)s;
  }
  bad = __reduce_or_sync(0xFFFFFFFFu, bad);
  skip = __reduce_add_sync(0xFFFFFFFFu, skip);
  kmem = __reduce_add_sync(0xFFFFFFFFu, kmem);
  dup = __reduce_add_sync(0xFFFFFFFFu, dup);
  if (lane == 0) {
    if (bad) atomicOr(&a.ctr[kRpErrBits], bad);
    if (dup) atomicAdd(&a.ctr[kRpSeqDup], dup);
    if (skip) atomicAdd(a.skip, skip);
    if (kmem) atomicAdd(a.kmem, kmem);
  }
  __syncthreads();
  for (uint32_t p = tid; p <= a.n_cut; p += 256) a.blockhist[(size_t)p * a.nblk + blockIdx.x] = s_hist[p];
}

// image k's solos whose (image, age) a party of image k holds -> *count
__global__ void k_rp_probe(uint32_t k, uint32_t n, const uint32_t* __restrict__ seq, uint32_t seq_next,
                           const unsigned long long* __restrict__ seqset, uint64_t seq_mask, uint32_t* __restrict__ count) {
  uint32_t dup = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    dup += seen_has(seqset, seq_mask, rp_seq_key(k, seq[i] - seq_next));
  dup = __reduce_add_sync(0xFFFFFFFFu, dup);
  if ((threadIdx.x & 31) == 0 && dup) atomicAdd(count, dup);
}

// n_images == 1: kept party pv (row = the exclusive scan of the kept flags) -> its row, its own number
__global__ void k_rp_rows1(uint32_t n, const uint16_t* __restrict__ part, uint32_t n_cut, const uint32_t* __restrict__ row,
                           const uint8_t* __restrict__ size, const uint32_t* __restrict__ seq, uint32_t* __restrict__ rsrc,
                           uint32_t* __restrict__ rsz, uint32_t* __restrict__ rseq) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n || part[j] >= n_cut) return;
  const uint32_t r = row[j];
  rsrc[r] = j; rsz[r] = size[j]; rseq[r] = seq[j];
}

// The queue merge's result (in buffer rg_rounds(*kmax) & 1) into buffer 0, for the rounds that merge the queues.
__global__ void __launch_bounds__(256) k_rp_norm(const uint32_t* __restrict__ kept, const uint32_t* __restrict__ kmax,
                                                 uint32_t* src0, const uint32_t* src1, RcKey* key0, const RcKey* key1) {
  if (!(rg_rounds(*kmax) & 1u)) return;
  const uint32_t n = *kept;
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
    src0[p] = src1[p];
    key0[p] = key1[p];
  }
}

struct RpPlaceArgs {
  const uint32_t* kept_p;   // parties kept
  const uint32_t* kept_s;   // solos kept
  const uint32_t* psrc;     // [kept_p] the parties' order: virtual indices
  const RcKey* pkey;
  uint32_t n_solo;          // N: the first party virtual index
  const uint8_t* size;      // [P] by party index (virtual index - N)
  uint32_t* gsrc;           // the solos' global list: the parties go after it
  RcKey* gkey;
  uint32_t* pos;            // [virtual index] -> N + row for a party
  uint32_t* rsrc;           // [row] party index
  uint32_t* rsz;            // [row] size
  uint32_t* fin;            // {0, total} | {0, kept_s, total} | {2}
};

__global__ void __launch_bounds__(256) k_rp_place(const RpPlaceArgs a) {
  const uint32_t np = *a.kept_p, ns = *a.kept_s;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    a.fin[0] = 0; a.fin[1] = ns + np;
    a.fin[2] = 0; a.fin[3] = ns; a.fin[4] = ns + np;
    a.fin[5] = 2;
  }
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < np; r += gridDim.x * blockDim.x) {
    const uint32_t v = a.psrc[r], j = v - a.n_solo;
    a.pos[v] = a.n_solo + r;
    a.rsrc[r] = j;
    a.rsz[r] = a.size[j];
    a.gsrc[ns + r] = v;
    a.gkey[ns + r] = a.pkey[r];
  }
}

struct RpWriteArgs {
  const PtImgCols* imgs;    // [K]
  const uint32_t* pbase;    // [K] first party index of the image
  const uint16_t* pk;       // [P] image
  const uint32_t* moff;     // [P] member offset in its image
  const int32_t* R;         // [P]
  const uint32_t* rsrc;     // [rows] party index
  const uint32_t* rseq;     // [rows] number
  const uint32_t* roff;     // [rows] first member entry (exclusive scan of the sizes)
  uint32_t rows;
  BinMap bm;
  const uint8_t* grp_lut;
  PartyView pt;
  ActiveView act;
};

// One thread per row of the new table: the row, its members, their active-set values kPtVal(row).  The ids were
// checked unique against everything loaded, and the room decided, before the load.
__global__ void __launch_bounds__(256) k_rp_write(const RpWriteArgs a) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.rows) return;
  const uint32_t j = a.rsrc[r], k = a.pk[j], i = j - a.pbase[k], o = a.roff[r], mo = a.moff[j];
  const PtImgCols& c = a.imgs[k];
  const uint32_t s = c.size[i], md = c.mode[i];
  const int32_t R = a.R[j];
  a.pt.seq[r] = a.rseq[r]; a.pt.ts[r] = c.ts[i]; a.pt.off[r] = o; a.pt.R[r] = R;
  a.pt.bin[r] = (uint16_t)bin_of(a.bm, a.bm.lut, R, md);
  a.pt.mode[r] = (uint8_t)md;
  a.pt.grp[r] = a.grp_lut[clamp_key(a.bm.key_lo, a.bm.KR, R)];
  a.pt.size[r] = (uint8_t)s;
  a.pt.dead[r] = 0;
  for (uint32_t x = 0; x < s; ++x) {
    const uint64_t pid = rp_id(c, mo + x);
    a.pt.mid[o + x] = pid;
    a.pt.mrat[o + x] = c.rating[mo + x];
    if (a.act.dcap) { *a.act.val(pid) = kPtVal(r); continue; }
    for (uint64_t h = hash64(pid) & a.act.mask;; h = (h + 1) & a.act.mask) {
      const unsigned long long kk = atomicCAS(a.act.key(h), kEmptyKey, (unsigned long long)pid);
      if (kk == kEmptyKey || kk == pid) { *a.act.val(h) = kPtVal(r); break; }
    }
  }
}

}  // namespace mm
