// mm_party_status.cuh — party search status on the device (mm_party_queue_stats / mm_party_locate, DESIGN §4): the
// waiting section of mm_queue_stats for the queued parties, and one party member's place and next mm_party_match lobby.
//
// Stats (k_pst_stats): one thread per table row; dead rows count nowhere.  Per warp, __match_any_sync groups the rows
// of one queue (parties, members, max wait) and of one (queue, bucket) (the two histograms), and the first lane of a
// group adds it in.  Rows are in age order, not by queue, so a CTA keeps every queue's record in shared memory (the
// per-queue histograms of mm_stats.cuh, all at once) and flushes the non-zero words with global atomics; when the
// records do not fit the opt-in shared memory (up to 8 x 64 queues of 560 bytes), the groups add into the global
// records directly.
//
// Locate: mm_party_match's path up to the point where it changes anything — compaction, the (bin, age) sort, the
// unbudgeted k_pt_plan (lob / pos of every placed row, rec of every lobby), k_wd_bases and, under an off-tick budget,
// k_wd_allot into the call's own words (a lobby at ordinal >= its queue's allowance stays: the capped plan's first
// a_q lobbies are the unbudgeted plan's).  k_pst_rank gives every row its rank among its queue's rows (rows are in age
// order after compaction).  With party_balance, the balance pass runs on tags: k_tb_pieces and k_tb_parties give
// every member slot its c and every lobby its continuation bits, k_tb_lobby<true, true> permutes member slots that hold
// their own index, and a tag's new slot is the member's index in the balanced lobby.  k_pst_answer: one warp per id.
#pragma once
#include <cstddef>

#include "mm_party.cuh"

namespace mm {

static_assert(sizeof(mm_party_queue_stat) == 560, "mm_party_queue_stat is 560 bytes (include/mm_engine.h)");
static_assert(sizeof(mm_party_member_status) == 48, "mm_party_member_status is 48 bytes (include/mm_engine.h)");

constexpr uint32_t kPstWords = sizeof(mm_party_queue_stat) / 4;
// word offsets inside mm_party_queue_stat
constexpr uint32_t kPstParties = 1, kPstMembers = 2, kPstMax = 3, kPstHist = 4, kPstSize = kPstHist + kWaitBuckets;
static_assert(offsetof(mm_party_queue_stat, n_parties) == kPstParties * 4 &&
                  offsetof(mm_party_queue_stat, max_wait) == kPstMax * 4 &&
                  offsetof(mm_party_queue_stat, wait_hist) == kPstHist * 4 &&
                  offsetof(mm_party_queue_stat, size_hist) == kPstSize * 4,
              "the kernel's word offsets follow mm_party_queue_stat");
constexpr uint32_t kPstNone = 0xFFFFFFFFu;
constexpr uint32_t kPstBlock = 256;

struct PstArgs {
  PartyView t;
  uint32_t n_rows, n_groups, n_cut, now;
  uint32_t* out;  // [n_cut] records as words, zeroed before the launch
};

template <bool kShared>
__global__ void __launch_bounds__(kPstBlock) k_pst_stats(const PstArgs a) {
  extern __shared__ uint32_t s_rec[];
  uint32_t* rec = kShared ? s_rec : a.out;
  const uint32_t words = a.n_cut * kPstWords, lane = threadIdx.x & 31;
  if (kShared) {
    for (uint32_t i = threadIdx.x; i < words; i += kPstBlock) s_rec[i] = 0;
    __syncthreads();
  }
  for (uint32_t r0 = blockIdx.x * kPstBlock + (threadIdx.x & ~31u); r0 < a.n_rows; r0 += gridDim.x * kPstBlock) {
    const uint32_t r = r0 + lane;  // (uniform loop: whole warps)
    const bool live = r < a.n_rows && a.t.dead[r] == 0;
    uint32_t q = kPstNone, w = 0, s = 0;
    if (live) {
      q = a.t.mode[r] * a.n_groups + a.t.grp[r];
      w = stat_wait(a.now, a.t.ts[r]);
      s = a.t.size[r];
    }
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, q);
    const uint32_t members = __reduce_add_sync(peers, s), mx = __reduce_max_sync(peers, w);
    const uint32_t hk = live ? (q << 8 | stat_bucket(w)) : kPstNone, hpeers = __match_any_sync(0xFFFFFFFFu, hk);
    const uint32_t sk = live ? (q << 8 | min(s, MM_PARTY_SIZE_BUCKETS - 1)) : kPstNone;
    const uint32_t speers = __match_any_sync(0xFFFFFFFFu, sk);
    if (!live) continue;
    uint32_t* x = rec + (size_t)q * kPstWords;
    if ((__ffs(peers) - 1) == lane) {
      atomicAdd(&x[kPstParties], __popc(peers));
      atomicAdd(&x[kPstMembers], members);
      if (mx) atomicMax(&x[kPstMax], mx);
    }
    if ((__ffs(hpeers) - 1) == lane) atomicAdd(&x[kPstHist + (hk & 0xFFu)], __popc(hpeers));
    if ((__ffs(speers) - 1) == lane) atomicAdd(&x[kPstSize + (sk & 0xFFu)], __popc(speers));
  }
  if (kShared) {
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < words; i += kPstBlock) {
      const uint32_t v = s_rec[i];
      if (!v) continue;
      if (i % kPstWords == kPstMax) atomicMax(&a.out[i], v);
      else atomicAdd(&a.out[i], v);
    }
  }
}

// One CTA over the rows in tiles of 1024: rank[r] = the live rows of r's queue before it, depth[q] = the live rows of
// queue q.  A row's rank is its queue's rows of the earlier tiles (s_cur) + its queue's rows in the warps before it
// (the warps' run tables, as in k_pt_scatter) + its rank among its warp's peers.
constexpr uint32_t kPstRankBlock = 1024;
__global__ void __launch_bounds__(kPstRankBlock) k_pst_rank(const PartyView t, uint32_t n_rows, uint32_t n_groups,
                                                             uint32_t n_cut, uint32_t* __restrict__ rank,
                                                             uint32_t* __restrict__ depth) {
  constexpr uint32_t W = kPstRankBlock / 32;
  __shared__ uint32_t s_q[W][32], s_cnt[W][32], s_cur[MM_MAX_MODES * MM_MAX_GROUPS];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (uint32_t i = threadIdx.x; i < n_cut; i += kPstRankBlock) s_cur[i] = 0;
  __syncthreads();
  for (uint32_t r0 = 0; r0 < n_rows; r0 += kPstRankBlock) {
    const uint32_t r = r0 + threadIdx.x;
    const uint32_t q = r < n_rows && t.dead[r] == 0 ? t.mode[r] * n_groups + t.grp[r] : kPstNone;
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, q), first = __ffs(peers) - 1;
    const bool lead = first == lane && q != kPstNone;
    s_q[warp][lane] = lead ? q : kPstNone;
    s_cnt[warp][lane] = __popc(peers);
    __syncthreads();
    uint32_t before = 0;
    if (lead) {
      before = s_cur[q];
      for (uint32_t w = 0; w < warp; ++w)
        for (uint32_t l = 0; l < 32; ++l)
          if (s_q[w][l] == q) { before += s_cnt[w][l]; break; }
    }
    before = __shfl_sync(0xFFFFFFFFu, before, first);
    if (q != kPstNone) rank[r] = before + __popc(peers & ((1u << lane) - 1u));
    __syncthreads();  // every count is read before a queue's count moves on
    if (lead) atomicAdd(&s_cur[q], __popc(peers));
    __syncthreads();
  }
  for (uint32_t i = threadIdx.x; i < n_cut; i += kPstRankBlock) depth[i] = s_cur[i];
}

struct PlocArgs {
  uint32_t n;
  const uint64_t* id;           // [n] queried ids (handles on MM_F_DENSE_IDS engines)
  ActiveView act;
  PoolView pool;                // states 1 and 2 as mm_locate decides them
  uint32_t n_slots, gen;
  PartyView t;                  // the compacted table
  uint32_t n_groups, now;
  const WdRule* rule;           // [n_cut]
  const uint32_t* rank;         // [rows] k_pst_rank
  const uint32_t* depth;        // [n_cut] k_pst_rank
  const uint32_t* lob;          // [rows] the plan's lobby record of a placed row, or null: no plan ran
  const uint32_t* pos;          // [rows] the plan's member offset inside the lobby
  const uint2* rec;             // [records] (queue, ordinal inside the queue)
  const uint32_t* allot;        // [n_cut] the off-tick budget's allowances, or null
  const uint32_t* mbase;        // party_balance: [records] member slot of the lobby's first member, or null
  const uint64_t* tags;         // party_balance: the member slots' tags after k_tb_lobby
  uint32_t pb_mask;
  mm_party_member_status* out;  // [n]
};

__global__ void __launch_bounds__(256) k_pst_answer(const PlocArgs a) {
  const uint32_t lane = threadIdx.x & 31, i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= a.n) return;  // (uniform over the warp)
  const uint64_t pid = a.id[i];
  uint32_t state = 0, row = 0;
  if (lane == 0) state = loc_state(a.act, a.pool, a.n_slots, a.gen, pid, row);
  state = __shfl_sync(0xFFFFFFFFu, state, 0);
  row = __shfl_sync(0xFFFFFFFFu, row, 0);
  mm_party_member_status r{};
  r.state = (uint8_t)state;
  r.window = -1;
  r.lobby = MM_LOCATE_STAYS;
  r.member = 0xFFFFu;
  if (state == 3) {
    const uint32_t o = a.t.off[row], s = a.t.size[row];
    uint32_t k = kPstNone;
    for (uint32_t j = lane; j < s; j += 32)
      if (a.t.mid[o + j] == pid) k = j;
    k = __reduce_min_sync(0xFFFFFFFFu, k);  // the row holds the id once
    const uint32_t md = a.t.mode[row], q = md * a.n_groups + a.t.grp[row];
    const WdRule u = a.rule[q];
    r.mode = (uint8_t)md;
    r.group = a.t.grp[row];
    r.size = (uint8_t)s;
    r.index = (uint8_t)k;
    r.rating = a.t.mrat[o + k];
    r.party_rating = a.t.R[row];
    r.enq_ts = a.t.ts[row];
    r.seq = a.t.seq[row];
    r.wait = stat_wait(a.now, r.enq_ts);
    if (u.min_wait != MM_WIDEN_OFF && r.wait >= u.min_wait) {  // k_pt_plan's anchor test and window
      r.anchor = 1;
      r.window = (int32_t)min((long long)u.w_max, (long long)u.w0 + (long long)((r.wait - u.min_wait) / u.step) * u.inc);
    }
    r.ahead = a.rank[row];
    r.depth = a.depth[q];
    const uint32_t l = a.lob ? a.lob[row] : kPtNone;
    const uint2 x = l != kPtNone ? a.rec[l] : make_uint2(0u, 0u);
    if (l != kPtNone && (!a.allot || x.y < a.allot[x.x])) {
      uint32_t m = a.pos[row] + k;
      if (a.tags && ((a.pb_mask >> md) & 1u)) {  // (uniform) a balanced lobby: L <= 16, where did slot m go
        const uint32_t L = a.rule[x.x].L, b = a.mbase[l];
        const bool hit = lane < L && a.tags[b + lane] == (uint64_t)(b + m);
        m = __ffs(__ballot_sync(0xFFFFFFFFu, hit)) - 1;
      }
      r.lobby = x.y;
      r.member = (uint16_t)m;
    }
  }
  if (lane == 0) a.out[i] = r;
}

// tags[j] = j: every member slot holds its own index before the balance pass
__global__ void k_pst_tags(uint32_t n, uint64_t* __restrict__ tags) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) tags[j] = j;
}

}  // namespace mm
