// mm_backfill.cuh — backfill on the device (mm_backfill, DESIGN §4): k open slots of a running lobby filled from its
// queue, nearest rating first (or oldest first on an arrival-order engine).
//
// Plan (k_bf_plan): the host sorts the requests by queue, stably; one warp per queue serves that queue's requests in
// order on the resident per-bin totals (tot).  rem[bin] starts from tot and counts the bin's players no earlier request
// of the call took.  A rating-order request finds its target among the queue's bins (bf_seek) and walks them outward
// from it in (distance, rating) order (bf_walk, the one outward walk of every off-tick call: mm_widen, mm_party_match
// and mm_backfill_party walk with it too).  Every (request, bin) take is
// one PIECE: the request, the bin, its rank offset inside the bin (the bin's players taken so far in this call), the
// count and its offset inside the request's output.  Every request takes a bin's oldest untaken players, so the call
// takes a prefix of every bin in enqueue order: what the band pipeline places with klim = the bin's taken count.
//
// Keys (k_bf_keys): every bin with a take becomes a key (ascending bin order) with klim = its taken count and kbase =
// the exclusive scan of those counts; the counters give the keys, the players and the size of the per-(key, tile)
// count columns.  The gather and take is then k_band_prep (BfKeyBins) / k_band_count / k_band_scan / k_band_limit /
// k_band_place (take = 1) into a staging array at kbase[key] + rank, and k_bf_out copies the pieces from staging into
// request order.
#pragma once

#include "mm_band.cuh"

namespace mm {

constexpr uint32_t kBfPlanWarps = 4;
constexpr uint32_t kBfKeysBlock = 1024;
constexpr uint32_t kBfFar = 0xFFFFFFFFu;  // distance of a bin outside the run or the window

// ctr words of one call (zeroed by the host)
enum BfCtr : uint32_t { kBfKeys = 0, kBfPlayers, kBfCols, kBfPieces, kBfWords };

struct BfReq {        // one request, in queue order
  uint32_t idx;       // its index in the caller's array
  uint32_t count;
  int32_t target;     // rating order: the target's clamp key (rating - key_lo, clamped to the key range)
  int32_t window;     // < 0: no limit
};
struct BfPiece { uint32_t req, bin, roff, cnt, poff; };

struct BfArgs {
  const uint32_t* tot;       // the pool's per-bin totals
  uint32_t* rem;             // [K] tot minus what this call took so far
  const uint16_t* bin_key;   // [Kp] clamp key of the bin (rating order)
  const uint32_t* seg_bin_lo;
  const uint32_t* cut_lp_lo;  // [n_cut + 1] first partition of the queue
  const uint16_t* bin_seg;
  const uint32_t* fill;      // the pool's partition fills
  uint32_t rating_order, K;
  const BfReq* req;          // [n] sorted by queue
  const uint32_t* qr;        // [n_cut + 1] first sorted request of the queue
  const uint32_t* queues;    // [nq] the queues with requests
  uint32_t nq;
  uint32_t* n_taken;         // [n] by caller index
  BfPiece* piece;            // [cap_pieces]
  uint32_t* key_bin;         // [K] key -> bin
  uint32_t* kbase;           // [K]
  uint32_t* klim;            // [K]
  uint32_t* ctr;             // [kBfWords]
};

// the count of lanes j whose sorted value v_j is below x (below or equal with `le`), v nondecreasing over the lanes
__device__ __forceinline__ uint32_t bf_rank(uint32_t v, uint32_t x, bool le) {
  uint32_t c = 0;
#pragma unroll
  for (uint32_t s = 16; s; s >>= 1) {
    const uint32_t u = __shfl_sync(0xFFFFFFFFu, v, c + s - 1);
    if (le ? u <= x : u < x) c += s;
  }
  const uint32_t last = __shfl_sync(0xFFFFFFFFu, v, 31);
  if (c == 31 && (le ? last <= x : last < x)) c = 32;
  return c;
}

// The first bin of [lo, hi) whose key is >= target (hi: none): the answer lies in [l, h]; each round samples 32 bins of
// it by a ballot and keeps one slice.  Uniform over the warp.
__device__ __forceinline__ uint32_t bf_seek(const uint16_t* bin_key, uint32_t lo, uint32_t hi, int32_t target) {
  const uint32_t lane = threadIdx.x & 31;
  uint32_t l = lo, h = hi;
  while (l < h) {
    const uint32_t step = (h - l + 31) / 32, b = l + lane * step;
    const uint32_t nb = __popc(__ballot_sync(0xFFFFFFFFu, b < h && (int32_t)bin_key[b] < target));
    if (nb == 0) break;
    const uint32_t l0 = l;
    l = l0 + (nb - 1) * step + 1;
    h = min(h, l0 + nb * step);
  }
  return l;
}

// The outward walk from `target` over the queue's bins [lo, hi), pos = bf_seek's first bin at or above it, within
// distance win: the first `need` players in (distance, rating, enqueue order).  The bins below pos (distance growing
// downwards) and the bins from pos on (growing upwards) are two sorted runs; each step merges the next 32 bins of the two
// runs by their distances (a tie goes to the lower rating), takes a warp prefix sum of their rem and consumes bins until
// need or the window runs out.  Without by_rating (arrival order: the queue's one bin) every distance is 0.  Returns how
// many it found (at most need) and, in left, how many of them lie below pos.  kTake: the players are taken (rem) and
// written as pieces of record r, each at its offset in member order (the left bins ascending, then the right bins, from
// offset `left`); kWalkOrder: in walk order instead, from offset `left`.  A: BfArgs or WdArgs (bin_key, tot, rem,
// piece, ctr).  Uniform over the warp.
template <bool kTake, bool kWalkOrder = false, class A>
__device__ __forceinline__ uint32_t bf_walk(const A& a, uint32_t* s_bin, int32_t target, uint32_t pos, uint32_t lo,
                                            uint32_t hi, uint32_t win, uint32_t need, uint32_t& left, uint32_t r,
                                            bool by_rating = true) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t nL = pos - lo, nR = hi - pos;
  const uint32_t left_all = left;  // kTake: the players below pos that the record takes
  uint32_t got = 0, used_l = 0, used_r = 0, got_l = 0, got_r = 0;
  while (need) {
    // the next 32 bins of each run and their distances (kBfFar past the run or the window)
    const uint32_t il = used_l + lane, ir = used_r + lane;
    uint32_t dl = kBfFar, dr = kBfFar;
    if (il < nL) {
      const uint32_t d = (uint32_t)(target - (int32_t)a.bin_key[pos - 1 - il]);
      dl = d <= win ? d : kBfFar;
    }
    if (ir < nR) {
      const uint32_t d = by_rating ? (uint32_t)((int32_t)a.bin_key[pos + ir] - target) : 0u;
      dr = d <= win ? d : kBfFar;
    }
    // merged positions: a lower bin goes before an upper bin of the same distance
    const uint32_t pl = lane + bf_rank(dr, dl, false), pr = lane + bf_rank(dl, dr, true);
    const bool okl = dl != kBfFar && pl < 32, okr = dr != kBfFar && pr < 32;
    if (okl) s_bin[pl] = pos - 1 - il;
    if (okr) s_bin[pr] = pos + ir;
    const uint32_t nl = __popc(__ballot_sync(0xFFFFFFFFu, okl)), nr = __popc(__ballot_sync(0xFFFFFFFFu, okr));
    const uint32_t nv = nl + nr;
    __syncwarp();
    uint32_t bin = 0, v = 0;
    if (lane < nv) { bin = s_bin[lane]; v = a.rem[bin]; }
    const uint32_t incl = warp_incl_scan(v);
    const uint32_t excl = incl - v, before = min(excl, need), take = min(v, need - before);
    const bool is_l = lane < nv && bin < pos;
    const uint32_t tl = is_l ? take : 0u, tr = is_l ? 0u : take;
    const uint32_t il_incl = warp_incl_scan(tl), ir_incl = warp_incl_scan(tr);
    if (kTake) {
      const uint32_t at = warp_append(&a.ctr[kBfPieces], take != 0);
      if (take) {
        // member order: the left bins in ascending rating (reverse walk order), then the right bins in walk order
        const uint32_t poff = kWalkOrder ? left_all + got + before
                                         : (is_l ? left_all - (got_l + il_incl) : left_all + got_r + ir_incl - tr);
        a.piece[at] = BfPiece{r, bin, a.tot[bin] - v, take, poff};
        a.rem[bin] = v - take;
      }
    }
    got_l += __shfl_sync(0xFFFFFFFFu, il_incl, 31);
    got_r += __shfl_sync(0xFFFFFFFFu, ir_incl, 31);
    const uint32_t took = min(__shfl_sync(0xFFFFFFFFu, incl, 31), need);
    need -= took; got += took;
    __syncwarp();  // rem and s_bin are read again by the next step
    if (nv < 32) break;  // both runs (or the window) exhausted
    used_l += nl; used_r += nr;
  }
  left = got_l;
  return got;
}

__global__ void __launch_bounds__(kBfPlanWarps * 32) k_bf_plan(const BfArgs a) {
  __shared__ uint32_t s_bin[kBfPlanWarps][32];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, qi = blockIdx.x * kBfPlanWarps + warp;
  if (qi >= a.nq) return;
  const uint32_t c = a.queues[qi];
  const uint32_t lo = a.seg_bin_lo[a.cut_lp_lo[c]], hi = a.seg_bin_lo[a.cut_lp_lo[c + 1]];
  for (uint32_t s = a.qr[c]; s < a.qr[c + 1]; ++s) {
    const BfReq r = a.req[s];
    const uint32_t win = r.window < 0 ? kBfFar - 1 : (uint32_t)r.window;
    // arrival order: the queue's one bin, at distance 0
    const uint32_t pos = a.rating_order ? bf_seek(a.bin_key, lo, hi, r.target) : lo;
    uint32_t left = 0;
    const uint32_t got =
        bf_walk<true, true>(a, s_bin[warp], r.target, pos, lo, hi, win, r.count, left, r.idx, a.rating_order != 0);
    if (lane == 0) a.n_taken[r.idx] = got;
  }
}

// One CTA: every bin with a take -> a key (ascending bin order), klim = its taken count, kbase = the exclusive scan of
// those; ctr = keys, players, and the count-column words of the keys' partitions.  Each thread owns a run of bins.
__global__ void __launch_bounds__(kBfKeysBlock) k_bf_keys(const BfArgs a) {
  __shared__ uint32_t s_tmp[33];
  const uint32_t tid = threadIdx.x, per = (a.K + kBfKeysBlock - 1) / kBfKeysBlock;
  const uint32_t b0 = min(a.K, tid * per), b1 = min(a.K, b0 + per);
  uint32_t nk = 0, np = 0, cols = 0;
  for (uint32_t b = b0; b < b1; ++b) {
    const uint32_t t = a.tot[b] - a.rem[b];
    if (t) { ++nk; np += t; cols += (__ldcg(&a.fill[a.bin_seg[b]]) + kTile - 1) / kTile; }
  }
  __shared__ uint32_t s_val[kBfKeysBlock];
  s_val[tid] = nk;
  __syncthreads();
  const uint32_t n_keys = block_excl_scan<kBfKeysBlock>(s_val, kBfKeysBlock, s_tmp);
  uint32_t q = s_val[tid];
  __syncthreads();
  s_val[tid] = np;
  __syncthreads();
  const uint32_t n_players = block_excl_scan<kBfKeysBlock>(s_val, kBfKeysBlock, s_tmp);
  uint32_t base = s_val[tid];
  for (uint32_t b = b0; b < b1; ++b) {
    const uint32_t t = a.tot[b] - a.rem[b];
    if (t) { a.key_bin[q] = b; a.klim[q] = t; a.kbase[q] = base; ++q; base += t; }
  }
  cols = __reduce_add_sync(0xFFFFFFFFu, cols);
  if ((tid & 31) == 0 && cols) atomicAdd(&a.ctr[kBfCols], cols);
  if (tid == 0) { a.ctr[kBfKeys] = n_keys; a.ctr[kBfPlayers] = n_players; }
}

// The backfill numbering for k_band_prep: key q is the bin k_bf_keys gave it, always local.
struct BfKeyBins {
  const uint32_t* key_bin;
  __device__ __forceinline__ uint32_t operator()(const BandArgs&, uint32_t q, bool& local) const {
    local = true;
    return key_bin[q];
  }
};

// Pieces to request order: piece p's cnt players sit in staging at kbase[key of its bin] + roff; they go to the request's
// output at req_base[req] + poff.  One warp per piece.  T: the ids, or (the off-tick report) the stamps beside them.
template <class T>
__global__ void k_bf_out(uint32_t n_pieces, const BfPiece* __restrict__ piece, const uint32_t* __restrict__ map,
                         const uint32_t* __restrict__ kbase, const uint32_t* __restrict__ req_base,
                         const T* __restrict__ staging, T* __restrict__ members) {
  const uint32_t lane = threadIdx.x & 31, p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (p >= n_pieces) return;
  const BfPiece c = piece[p];
  const T* src = staging + kbase[map[c.bin]] + c.roff;
  T* dst = members + req_base[c.req] + c.poff;
  for (uint32_t i = lane; i < c.cnt; i += 32) dst[i] = src[i];
}

}  // namespace mm
