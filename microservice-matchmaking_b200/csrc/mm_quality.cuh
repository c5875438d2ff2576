// mm_quality.cuh — mm_match_quality: rating spread and team imbalance of the last tick's lobbies, per lobby and per
// (mode, group) queue, from the pool buffer the last tick read (pool[cur ^ 1], which no call writes until the next
// tick) and its left bits.  The tick's results (d_members, d_hdr) and scratch (d_outbase, d_binlim) are not read:
// other calls hand out or reuse them between ticks.
//
// A slot of that buffer was matched when it is live (not in the removed bin) and its left bit is clear.  The matched
// players of a queue, in the tick's order, are its lobbies' members in member order, L at a time, and a queue's
// lobbies sit at consecutive header positions from the exclusive scan of the per-queue lobby counts.
//   k_mq_count     one pass over the bin column and the left bits: matched players per bin (warp-aggregated atomics)
//   k_mq_scan      one CTA per queue: each bin's first member inside its queue and, in rating order, the 64-bit prefix
//                  of count x c over the queue's bins (a queue's bins are consecutive, across its partitions too);
//                  the queue's lobbies = its matched players / L
//   k_mq_base      one CTA: lobby base and team-sum base of every queue (exclusive scans)
// MM_ORDER_RATING: every player of a bin has c = key_lo + bin_key[bin], so no player is read again —
//   k_mq_lobby<false>  one thread per lobby: min and max from the bins of its first and last member, the rating sum
//                      and every team sum as differences of the prefix F(x) = sum of c over the queue's first x members
// MM_ORDER_ARRIVAL: a bin is a whole group and a queue one partition, whose matched players are its first a_q L live
//   players in storage order; mm_export's live-slot count (k_img_tiles) and k_scan_small give every tile's first live
//   rank, then
//   k_mq_arrival       one warp step per 32 slots: live rank -> lobby and team, segmented warp reductions of
//                      c - key_lo (never negative) and exact integer atomics into per-lobby scratch
//   k_mq_lobby<true>   one thread per lobby: the record from its scratch
// Both: k_mq_queue     the per-queue records: shared-memory histograms, flushed with atomics per queue run
// A lobby of a mode the last tick balanced (team_balance, mm_balance.cuh) has other teams than the pool's order gives:
// its imbalance is the one k_tb_lobby stored for its header position, and every other value is order-free.
#pragma once
#include <cstddef>

#include "mm_image.cuh"
#include "mm_stats.cuh"

namespace mm {

static_assert(sizeof(mm_lobby_quality) == 24 && offsetof(mm_lobby_quality, rating_sum) == 8 &&
                  offsetof(mm_lobby_quality, imbalance) == 16,
              "mm_lobby_quality is 24 bytes (include/mm_engine.h)");
static_assert(sizeof(mm_queue_quality) == 992 && offsetof(mm_queue_quality, n_lobbies) == 4 &&
                  offsetof(mm_queue_quality, sum_spread) == 16 && offsetof(mm_queue_quality, spread_hist) == 32 &&
                  offsetof(mm_queue_quality, imbalance_hist) == 512,
              "mm_queue_quality is 992 bytes (include/mm_engine.h)");

constexpr uint32_t kMqBlock = 256;
constexpr uint32_t kMqNone = 0xFFFFu;  // k_mq_count: not a matched player

// mm_queue_stats' bucket of a rating-point value; 2^31 and more count in the last bucket
__device__ __forceinline__ uint32_t mq_bucket(uint32_t v) { return v >= 0x80000000u ? kWaitBuckets - 1 : stat_bucket(v); }

struct MqArgs {
  PoolView pool;                // the pool buffer the last tick read
  PoolMeta meta;                // its partitions
  const uint32_t* left_bits;    // the last tick's: a set bit = stayed queued (virtual position)
  uint32_t n_segs, n_cut, n_groups, K;
  int32_t key_lo;
  uint32_t KR;
  const uint16_t* bin_key;      // [Kp] rating order: c = key_lo + bin_key[bin]
  const uint32_t* seg_bin_lo;   // [n_segs + 1]
  const uint32_t* seg_L;        // [n_segs]
  const uint16_t* part_cut;     // [n_segs] partition -> queue
  const uint32_t* cut_lp_lo;    // [n_cut + 1] first partition of the queue
  const uint8_t* mode_tsize;    // [MM_MAX_MODES] S of a mode
  uint32_t* cnt;                // [Kp] matched players of the bin -> (k_mq_scan) its first member inside its queue
  long long* csum;              // [Kp] rating order: sum of c over the queue's members before the bin
  uint32_t* qlob;               // [n_cut + 1] lobbies of the queue -> (k_mq_base) its first header position
  uint32_t* qteam;              // [n_cut + 1] arrival order: first team-sum word of the queue
  const uint32_t* tile_off;     // arrival order: live slots of the virtual tiles before this one
  uint32_t* lmin;               // [lobbies] arrival order: min of c - key_lo (starts all ones)
  uint32_t* lmax;               // [lobbies] arrival order: max of c - key_lo (starts 0)
  uint32_t* tsum;               // [teams] arrival order: team sums of c - key_lo (start 0)
  mm_lobby_quality* lob;        // [lobbies]
  uint32_t n_lob;               // the tick's lobbies
  mm_queue_quality* qrec;       // [n_cut], zeroed before k_mq_queue
  uint32_t tb_mask;             // the modes the last tick balanced (mm_balance.cuh): their S > 1 lobbies' imbalance
  const uint32_t* tb_imb;       // [lobbies] ... is the balanced one, per header position
};

// lobby size L and team size S of queue q
__device__ __forceinline__ void mq_shape(const MqArgs& a, uint32_t q, uint32_t& L, uint32_t& S) {
  L = a.seg_L[a.cut_lp_lo[q]];
  S = a.mode_tsize[q / a.n_groups];
}
// queue of header position h: the last q with qlob[q] <= h (queues without lobbies share their successor's base)
__device__ __forceinline__ uint32_t mq_queue_of(const MqArgs& a, uint32_t h) { return last_le(a.qlob, 0, a.n_cut, h); }

// matched players per bin (cnt zeroed by the host).  CTAs take contiguous runs of the virtual tile sequence.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_mq_count(const MqArgs a) {
  __shared__ Geo geo;
  __shared__ uint32_t s_gtmp[33];
  uint32_t s0, s1;
  if (!geo_cta_run<BLOCK>(geo, a.meta.fill, a.n_segs, s_gtmp, s0, s1)) return;  // (uniform)
  const uint32_t o = threadIdx.x * 8;
  for (uint32_t s = s0; s < s1; ++s) {
    const TileDesc d = geo_tile(geo, a.meta, s);
    uint32_t b[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) b[j] = kMqNone;
    if (o < d.nvalid) {
      uint32_t v[8];
      ld_bins8(a.pool.bin + (size_t)d.phys * kTile + o, v);
      const uint32_t left = (__ldcs(&a.left_bits[((size_t)s * kTile + o) >> 5]) >> (o & 31)) & 0xFFu;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (o + j < d.nvalid && v[j] < a.K && !((left >> j) & 1u)) b[j] = v[j];
    }
    warp_hist8_add(a.cnt, b, kMqNone);
  }
}

// (members, sum of c) of a run of bins, scanned together by k_mq_scan
struct MqSum {
  uint32_t c;
  long long w;
};
__device__ __forceinline__ MqSum operator+(const MqSum& x, const MqSum& y) { return MqSum{x.c + y.c, x.w + y.w}; }
__device__ __forceinline__ MqSum operator-(const MqSum& x, const MqSum& y) { return MqSum{x.c - y.c, x.w - y.w}; }
__device__ __forceinline__ MqSum shfl_up(const MqSum& v, int off) { return MqSum{shfl_up(v.c, off), shfl_up(v.w, off)}; }

// One CTA per queue: cnt -> each bin's first member inside the queue, csum -> the sum of c before it (rating order),
// qlob[q] = the queue's lobbies.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_mq_scan(const MqArgs a, bool rating) {
  __shared__ MqSum s_tmp[BLOCK / 32 + 1];
  const uint32_t q = blockIdx.x, tid = threadIdx.x;
  const uint32_t b0 = a.seg_bin_lo[a.cut_lp_lo[q]], b1 = a.seg_bin_lo[a.cut_lp_lo[q + 1]];
  MqSum run{0u, 0ll};
  for (uint32_t base = b0; base < b1; base += BLOCK) {
    const uint32_t b = base + tid;
    const uint32_t c = b < b1 ? a.cnt[b] : 0u;
    const MqSum v{c, rating && c ? (long long)c * (a.key_lo + (int32_t)a.bin_key[b]) : 0ll};
    const MqSum x = block_scan_step<BLOCK>(v, run, s_tmp);
    if (b < b1) {
      a.cnt[b] = x.c;
      if (rating) a.csum[b] = x.w;
    }
  }
  if (tid == 0) {
    uint32_t L, S;
    mq_shape(a, q, L, S);
    a.qlob[q] = run.c / L;
  }
}

// One CTA: qlob -> exclusive scan (first header position of every queue), qteam -> first team-sum word.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_mq_base(const MqArgs a) {
  __shared__ uint32_t s_l[kMaxSegs + 1], s_t[kMaxSegs + 1];
  __shared__ uint32_t s_tmp[33];
  for (uint32_t q = threadIdx.x; q < a.n_cut; q += BLOCK) {
    uint32_t L, S;
    mq_shape(a, q, L, S);
    s_l[q] = a.qlob[q];
    s_t[q] = a.qlob[q] * (L / S);
  }
  __syncthreads();
  const uint32_t nl = block_excl_scan<BLOCK>(s_l, a.n_cut, s_tmp);
  const uint32_t nt = block_excl_scan<BLOCK>(s_t, a.n_cut, s_tmp);
  for (uint32_t q = threadIdx.x; q < a.n_cut; q += BLOCK) { a.qlob[q] = s_l[q]; a.qteam[q] = s_t[q]; }
  if (threadIdx.x == 0) { a.qlob[a.n_cut] = nl; a.qteam[a.n_cut] = nt; }
}

// Arrival order: every matched player's live rank rho in its partition -> lobby rho / L, team rho / S; the minimum,
// maximum and team sums of c - key_lo reduce over runs of equal keys in the warp, then one atomic per run.  A slot
// that is not matched carries the keys of the next live rank and a neutral value, so the keys never decrease along
// the lanes and equal keys are consecutive.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_mq_arrival(const MqArgs a) {
  __shared__ Geo geo;
  __shared__ uint32_t s_gtmp[33];
  __shared__ uint32_t s_warp[BLOCK / 32];
  const uint32_t lane = threadIdx.x & 31;
  uint32_t s0, s1;
  if (!geo_cta_run<BLOCK>(geo, a.meta.fill, a.n_segs, s_gtmp, s0, s1)) return;  // (uniform)
  auto all = [](const TileDesc&) { return true; };
  live_rank_walk<BLOCK>(geo, a.meta, a.pool.mode, a.left_bits, a.tile_off, s0, s1, s_warp, all,
                        [&](const TileDesc& d, size_t slot, bool matched, uint32_t rho) {
      const uint32_t q = a.part_cut[d.seg];
      uint32_t L, S;
      mq_shape(a, q, L, S);
      const uint32_t n_q = a.qlob[q + 1] - a.qlob[q], T = L / S;
      const uint32_t v = matched ? clamp_key(a.key_lo, a.KR, a.pool.rating[slot]) : 0u;
      const uint32_t lk = rho / L, tk = rho / S;
      uint32_t mn = matched ? v : 0xFFFFFFFFu, mx = v, sm = v;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const uint32_t o_lk = __shfl_down_sync(0xFFFFFFFFu, lk, off), o_tk = __shfl_down_sync(0xFFFFFFFFu, tk, off);
        const uint32_t o_mn = __shfl_down_sync(0xFFFFFFFFu, mn, off), o_mx = __shfl_down_sync(0xFFFFFFFFu, mx, off);
        const uint32_t o_sm = __shfl_down_sync(0xFFFFFFFFu, sm, off);
        if (lane + off < 32 && o_lk == lk) { mn = o_mn < mn ? o_mn : mn; mx = o_mx > mx ? o_mx : mx; }
        if (lane + off < 32 && o_tk == tk) sm += o_sm;
      }
      const uint32_t p_lk = __shfl_up_sync(0xFFFFFFFFu, lk, 1), p_tk = __shfl_up_sync(0xFFFFFFFFu, tk, 1);
      if (lk < n_q && mn != 0xFFFFFFFFu && (lane == 0 || p_lk != lk)) {  // head of a run with a matched player
        const uint32_t h = a.qlob[q] + lk;
        atomicMin(&a.lmin[h], mn);
        atomicMax(&a.lmax[h], mx);
      }
      if (tk < n_q * T && sm && (lane == 0 || p_tk != tk)) atomicAdd(&a.tsum[a.qteam[q] + tk], sm);
    });
}

// One thread per lobby: its record.  Rating order: from the per-bin prefixes; arrival order: from k_mq_arrival.
template <bool ARRIVAL>
__global__ void __launch_bounds__(256) k_mq_lobby(const MqArgs a) {
  const uint32_t h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= a.n_lob) return;
  const uint32_t q = mq_queue_of(a, h), ord = h - a.qlob[q];
  uint32_t L, S;
  mq_shape(a, q, L, S);
  const uint32_t T = L / S;
  mm_lobby_quality r{};
  long long smin = 0, smax = 0;
  if (ARRIVAL) {
    r.min_rating = a.key_lo + (int32_t)a.lmin[h];
    r.max_rating = a.key_lo + (int32_t)a.lmax[h];
    const uint32_t* ts = a.tsum + a.qteam[q] + (size_t)ord * T;
    long long sum = 0;
    for (uint32_t t = 0; t < T; ++t) {
      const long long v = ts[t];
      sum += v;
      smin = t == 0 || v < smin ? v : smin;
      smax = t == 0 || v > smax ? v : smax;
    }
    r.rating_sum = sum + (long long)L * a.key_lo;
  } else {
    const uint32_t b0 = a.seg_bin_lo[a.cut_lp_lo[q]], b1 = a.seg_bin_lo[a.cut_lp_lo[q + 1]];
    // bin of the queue's member x: the last bin whose first member is <= x (empty bins share their successor's)
    uint32_t from = b0;
    auto bin_at = [&](uint32_t x) {
      from = last_le(a.cnt, from, b1, x);  // members are asked for in ascending order
      return from;
    };
    auto c_of = [&](uint32_t b) { return (long long)a.key_lo + a.bin_key[b]; };
    // F(x): sum of c over the queue's members [0, x), x > 0
    auto F = [&](uint32_t x) {
      const uint32_t b = bin_at(x - 1);
      return a.csum[b] + (long long)(x - a.cnt[b]) * c_of(b);
    };
    const uint32_t x0 = ord * L;
    const long long f0 = x0 ? F(x0) : 0ll;  // (member x0 - 1 comes before member x0)
    r.min_rating = (int32_t)c_of(bin_at(x0));
    long long prev = f0;
    for (uint32_t t = 0; t < T; ++t) {
      const long long f = F(x0 + (t + 1) * S), v = f - prev;
      prev = f;
      smin = t == 0 || v < smin ? v : smin;
      smax = t == 0 || v > smax ? v : smax;
    }
    r.max_rating = (int32_t)c_of(bin_at(x0 + L - 1));
    r.rating_sum = prev - f0;
  }
  const unsigned long long imb = (unsigned long long)(smax - smin);
  r.imbalance = imb > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)imb;
  if (((a.tb_mask >> (q / a.n_groups)) & 1u) && S > 1) r.imbalance = a.tb_imb[h];  // the teams actually emitted
  a.lob[h] = r;
}

// The per-queue records.  CTA k takes a contiguous run of header positions; per queue inside it, the histograms
// build in shared memory and flush with global atomics (the record is zeroed by the host).
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_mq_queue(const MqArgs a) {
  __shared__ uint32_t s_hs[kWaitBuckets], s_hi[kWaitBuckets];
  __shared__ unsigned long long s_ss, s_si;
  __shared__ uint32_t s_ms, s_mi;
  const uint32_t tid = threadIdx.x, lane = tid & 31;
  const uint32_t per = (a.n_lob + gridDim.x - 1) / gridDim.x;
  uint32_t h = blockIdx.x * per;
  const uint32_t h1 = h + per < a.n_lob ? h + per : a.n_lob;
  for (uint32_t i = tid; i < kWaitBuckets; i += BLOCK) { s_hs[i] = 0; s_hi[i] = 0; }
  if (tid == 0) { s_ss = 0; s_si = 0; s_ms = 0; s_mi = 0; }
  __syncthreads();
  while (h < h1) {  // (uniform)
    const uint32_t q = mq_queue_of(a, h), end = a.qlob[q + 1] < h1 ? a.qlob[q + 1] : h1;
    unsigned long long ss = 0, si = 0;
    uint32_t ms = 0, mi = 0;
    for (uint32_t base = h; base < end; base += BLOCK) {  // (uniform)
      const uint32_t k = base + tid;
      uint32_t bs = kMqNone, bi = kMqNone;
      if (k < end) {
        const mm_lobby_quality r = a.lob[k];
        const uint32_t sp = (uint32_t)(r.max_rating - r.min_rating);
        ss += sp; si += r.imbalance;
        ms = sp > ms ? sp : ms; mi = r.imbalance > mi ? r.imbalance : mi;
        bs = mq_bucket(sp); bi = mq_bucket(r.imbalance);
      }
      const uint32_t m1 = __match_any_sync(0xFFFFFFFFu, bs);
      if (bs != kMqNone && lane == (uint32_t)(__ffs(m1) - 1)) atomicAdd(&s_hs[bs], (uint32_t)__popc(m1));
      const uint32_t m2 = __match_any_sync(0xFFFFFFFFu, bi);
      if (bi != kMqNone && lane == (uint32_t)(__ffs(m2) - 1)) atomicAdd(&s_hi[bi], (uint32_t)__popc(m2));
    }
#pragma unroll
    for (int off = 16; off; off >>= 1) {
      ss += __shfl_xor_sync(0xFFFFFFFFu, ss, off);
      si += __shfl_xor_sync(0xFFFFFFFFu, si, off);
    }
    ms = __reduce_max_sync(0xFFFFFFFFu, ms);
    mi = __reduce_max_sync(0xFFFFFFFFu, mi);
    if (lane == 0) {
      if (ss) atomicAdd(&s_ss, ss);
      if (si) atomicAdd(&s_si, si);
      if (ms) atomicMax(&s_ms, ms);
      if (mi) atomicMax(&s_mi, mi);
    }
    __syncthreads();
    mm_queue_quality* rec = a.qrec + q;
    for (uint32_t i = tid; i < kWaitBuckets; i += BLOCK) {
      if (s_hs[i]) { atomicAdd(&rec->spread_hist[i], s_hs[i]); s_hs[i] = 0; }
      if (s_hi[i]) { atomicAdd(&rec->imbalance_hist[i], s_hi[i]); s_hi[i] = 0; }
    }
    if (tid == 0) {
      atomicAdd(&rec->n_lobbies, end - h);
      if (s_ss) atomicAdd(reinterpret_cast<unsigned long long*>(&rec->sum_spread), s_ss);
      if (s_si) atomicAdd(reinterpret_cast<unsigned long long*>(&rec->sum_imbalance), s_si);
      if (s_ms) atomicMax(&rec->max_spread, s_ms);
      if (s_mi) atomicMax(&rec->max_imbalance, s_mi);
      s_ss = 0; s_si = 0; s_ms = 0; s_mi = 0;
    }
    __syncthreads();
    h = end;
  }
}

}  // namespace mm
