// mm_offtick.cuh — the off-tick match report (mm_offtick_report, include/mm_engine.h): waits and rating quality of the
// lobbies one mm_party_match or mm_widen call formed, captured on the device inside that call, after its members are
// final (after the balance pass when one runs).  After the call the host holds only ids, and the next tick or party
// call compacts the taken slots and rows away, so the report cannot be rebuilt later.
//
// Inputs, per member slot of the call (the member order the plan produced, before any balance split):
//   cval  c - key_lo: a solo's from its piece's bin (k_tb_pieces), a party member's from its own rating (k_tb_parties)
//   ts    enq_ts: a solo's from its pool slot (k_band_place's stamp column, placed by k_bf_out), a party member's its
//         party's (k_tb_parties)
// and the queues' lobby and member bases the call scanned (k_wd_bases).
//   k_ot_bases   one CTA: the bases as [n_cut + 1] arrays, the totals at the end
//   k_ot_lobby   one warp per lobby: min, max, 64-bit sum and the team sums over its L member slots -> mm_lobby_quality;
//                a lobby the balance pass re-split takes the imbalance that pass stored for its header position
//   k_mq_queue   (mm_quality.cuh) the per-queue quality records from the lobby records and the lobby bases
//   k_ot_waits   the per-queue wait records: CTA k takes a contiguous run of member slots; per queue inside it the
//                histogram builds in shared memory and flushes with global atomics (the records are zeroed by the host)
// Every value but the imbalance is order-free, so the balance pass's permutation of the ids needs no permutation here.
#pragma once
#include <climits>
#include <cstddef>

#include "mm_quality.cuh"

namespace mm {

static_assert(sizeof(mm_match_waits) == 496 && offsetof(mm_match_waits, n_lobbies) == 4 &&
                  offsetof(mm_match_waits, max_match_wait) == 12 && offsetof(mm_match_waits, match_wait_hist) == 16,
              "mm_match_waits is 496 bytes (include/mm_engine.h)");

constexpr uint32_t kOtBlock = 256;

struct OtArgs {
  const mm_lobby_hdr* hdr;     // [n_lob] the call's headers
  uint32_t n_lob, n_mem, n_cut, n_groups, now;
  int32_t key_lo;
  const uint8_t* mode_tsize;   // [MM_MAX_MODES]
  const uint32_t* cval;        // [n_mem] c - key_lo per member slot
  const uint32_t* ts;          // [n_mem] enq_ts per member slot
  uint32_t bal_mask;           // the modes the call's balance pass split (S > 1 lobbies) ...
  const uint32_t* bal_imb;     // ... and their imbalance per header position
  const uint32_t* qlbase;      // [n_cut] first header position of the queue (k_wd_bases)
  const uint32_t* qmbase;      // [n_cut] first member slot of the queue
  uint32_t* qb;                // [n_cut + 1] out: lobby bases, n_lob at the end
  uint32_t* qm;                // [n_cut + 1] out: member bases, n_mem at the end
  mm_lobby_quality* lob;       // [n_lob]
  mm_match_waits* waits;       // [n_cut], zeroed by the host
};

__global__ void __launch_bounds__(kOtBlock) k_ot_bases(const OtArgs a) {
  for (uint32_t c = threadIdx.x; c <= a.n_cut; c += kOtBlock) {
    a.qb[c] = c < a.n_cut ? a.qlbase[c] : a.n_lob;
    a.qm[c] = c < a.n_cut ? a.qmbase[c] : a.n_mem;
  }
}

// One warp per lobby (grid-stride): lanes stride over the members for min / max / sum and over the teams for the team
// sums (team t = members [tS, (t + 1)S)).
__global__ void __launch_bounds__(kOtBlock) k_ot_lobby(const OtArgs a) {
  const uint32_t lane = threadIdx.x & 31, nw = gridDim.x * (blockDim.x >> 5);
  for (uint32_t h = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; h < a.n_lob; h += nw) {
    const mm_lobby_hdr hd = a.hdr[h];
    const uint32_t L = hd.n_members, S = a.mode_tsize[hd.mode], T = L / S;
    const uint32_t* c = a.cval + hd.first_member;
    uint32_t mn = 0xFFFFFFFFu, mx = 0;
    long long sum = 0;
    for (uint32_t i = lane; i < L; i += 32) {
      const uint32_t v = c[i];
      mn = v < mn ? v : mn;
      mx = v > mx ? v : mx;
      sum += v;
    }
    long long tmin = LLONG_MAX, tmax = LLONG_MIN;
    for (uint32_t t = lane; t < T; t += 32) {
      long long s = 0;
      for (uint32_t i = t * S; i < (t + 1) * S; ++i) s += c[i];
      tmin = s < tmin ? s : tmin;
      tmax = s > tmax ? s : tmax;
    }
    mn = __reduce_min_sync(0xFFFFFFFFu, mn);
    mx = __reduce_max_sync(0xFFFFFFFFu, mx);
#pragma unroll
    for (int off = 16; off; off >>= 1) {
      sum += __shfl_xor_sync(0xFFFFFFFFu, sum, off);
      const long long omin = __shfl_xor_sync(0xFFFFFFFFu, tmin, off), omax = __shfl_xor_sync(0xFFFFFFFFu, tmax, off);
      tmin = omin < tmin ? omin : tmin;
      tmax = omax > tmax ? omax : tmax;
    }
    if (lane == 0) {
      mm_lobby_quality r{};
      r.min_rating = a.key_lo + (int32_t)mn;
      r.max_rating = a.key_lo + (int32_t)mx;
      r.rating_sum = sum + (long long)L * a.key_lo;
      const unsigned long long imb = (unsigned long long)(tmax - tmin);  // every lobby has T >= 1 teams
      r.imbalance = imb > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)imb;
      if (((a.bal_mask >> hd.mode) & 1u) && S > 1) r.imbalance = a.bal_imb[h];  // the teams actually emitted
      a.lob[h] = r;
    }
  }
}

// The per-queue wait records over the member slots, shaped like k_mq_queue over the header positions.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_ot_waits(const OtArgs a) {
  __shared__ uint32_t s_h[kWaitBuckets];
  __shared__ uint32_t s_mx;
  const uint32_t tid = threadIdx.x, lane = tid & 31;
  const uint32_t per = (a.n_mem + gridDim.x - 1) / gridDim.x;
  uint32_t m = blockIdx.x * per;
  const uint32_t m1 = m + per < a.n_mem ? m + per : a.n_mem;
  for (uint32_t i = tid; i < kWaitBuckets; i += BLOCK) s_h[i] = 0;
  if (tid == 0) s_mx = 0;
  __syncthreads();
  while (m < m1) {  // (uniform)
    const uint32_t q = last_le(a.qm, 0, a.n_cut, m), end = a.qm[q + 1] < m1 ? a.qm[q + 1] : m1;
    uint32_t mx = 0;
    for (uint32_t base = m; base < end; base += BLOCK) {  // (uniform)
      const uint32_t k = base + tid;
      uint32_t b = kMqNone;
      if (k < end) {
        const uint32_t w = stat_wait(a.now, a.ts[k]);
        mx = w > mx ? w : mx;
        b = stat_bucket(w);
      }
      const uint32_t peers = __match_any_sync(0xFFFFFFFFu, b);
      if (b != kMqNone && lane == (uint32_t)(__ffs(peers) - 1)) atomicAdd(&s_h[b], (uint32_t)__popc(peers));
    }
    mx = __reduce_max_sync(0xFFFFFFFFu, mx);
    if (lane == 0 && mx) atomicMax(&s_mx, mx);
    __syncthreads();
    mm_match_waits* rec = a.waits + q;
    for (uint32_t i = tid; i < kWaitBuckets; i += BLOCK)
      if (s_h[i]) { atomicAdd(&rec->match_wait_hist[i], s_h[i]); s_h[i] = 0; }
    if (tid == 0) {
      atomicAdd(&rec->n_matched, end - m);
      if (s_mx) atomicMax(&rec->max_match_wait, s_mx);
      s_mx = 0;
    }
    __syncthreads();
    m = end;
  }
}

}  // namespace mm
