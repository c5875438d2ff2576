// mm_locate.cuh — mm_locate: the search status of single players, answered on the device from the resident pool
//
// Three launches, none of which writes anything but the call's own scratch:
//   k_locate_preview  the tick's tail (mm_scan.cuh, kPreview) on the resident bin totals with the engine's max_spread
//                     and lobby budget: the sorted position of every bin's first player (pos), and the member slots
//                     of every bin's matched prefix (outbase / binlim) the next tick would use
//   k_loc_rmap        physical chunk -> its index in its partition's chunk list (one entry per chunk in use)
//   k_locate          one warp per query: the active-set probe (mm_remove's test), then the player's rank among the
//                     live players of its bin that the tick places before it, and the answer
// The tick places the players of a bin in partition storage order, so a player's rank is the live players of its bin
// in the partition's earlier chunks plus those before it in its own chunk.  With resident chunk histograms the earlier
// chunks cost one 4-byte read each; without them (MM_F_WIDE_PARTITIONS, or more than kMaxSegs partitions) the warp
// counts the bin column of the earlier chunks.  The own chunk is counted from the bin column (at most 4 KB).
// With team_balance set for the player's mode, the predicted lobby is split as the tick's balance pass will split it
// (tb_split): its members' c from the preview's per-bin member ranges (rating order), or from the L consecutive live
// players of the partition around the player (arrival order), found by walking the mode and rating columns.
#pragma once
#include "mm_balance.cuh"
#include "mm_kernels.cuh"

namespace mm {

static_assert(sizeof(mm_player_status) == 36, "mm_player_status is 36 bytes (include/mm_engine.h)");

// Always the budget form of the tail: with no budget set (null t.bud_queue / t.bud_mode) every queue is allotted all
// of its lobbies and the cut is the unbudgeted one.  (The form without the budget code spills at this launch bound.)
__global__ void __launch_bounds__(kScanBlock) k_locate_preview(const TailArgs t) {
  extern __shared__ __align__(16) uint32_t scratch[];
  colscan_tail_body<false, true, true>(scratch, t);
}

// rmap[chunk_tab[sg][k]] = k for the chunks of every partition in use (one CTA per partition)
__global__ void k_loc_rmap(const PoolMeta m, uint32_t* __restrict__ rmap) {
  const uint32_t sg = blockIdx.x, nch = (__ldg(&m.fill[sg]) + kTile - 1) / kTile;
  for (uint32_t k = threadIdx.x; k < nch; k += blockDim.x) rmap[__ldg(&m.chunk_tab[(size_t)sg * m.max_ch + k])] = k;
}

// One warp: the live players of bin v (partition sg) stored before `slot` in the partition — the player's rank in its
// bin in enqueue order.  Every lane gets the answer.
__device__ __forceinline__ uint32_t bin_rank(const PoolView& pool, const PoolMeta& meta, const uint32_t* seg_bin_lo,
                                             const uint32_t* rmap, uint32_t slot, uint32_t v, uint32_t sg) {
  const uint32_t lane = threadIdx.x & 31, chunk = slot / kTile, off = slot % kTile;
  const uint32_t k = rmap[chunk];
  const uint32_t* tab = meta.chunk_tab + (size_t)sg * meta.max_ch;
  uint32_t rank = 0;
  if (meta.chist) {
    const uint32_t key = v - seg_bin_lo[sg];
    for (uint32_t j = lane; j < k; j += 32) rank += meta.chist[(size_t)tab[j] * kChunkHist + key];
  } else {
    for (uint32_t j = 0; j < k; ++j) {
      const uint16_t* b = pool.bin + (size_t)tab[j] * kTile;
      for (uint32_t o = lane; o < kTile; o += 32) rank += b[o] == v ? 1u : 0u;
    }
  }
  const uint16_t* own = pool.bin + (size_t)chunk * kTile;
  for (uint32_t o = lane; o < off; o += 32) rank += own[o] == v ? 1u : 0u;
  return __reduce_add_sync(0xFFFFFFFFu, rank);
}

// The state of id pid (one thread, an engine with an active set): 0 not in the active set, 1 a live player of the
// current pool generation (slot = its pool slot: mm_remove's test), 3 a member of a queued party (slot = the party's
// row), 2 otherwise.
__device__ __forceinline__ uint32_t loc_state(const ActiveView& act, const PoolView& pool, uint32_t n_slots,
                                              uint32_t gen, uint64_t pid, uint32_t& slot) {
  uint32_t state = 0;
  const uint64_t h = act_find(act, pid);
  if (h != ~0ull) {
    const unsigned long long v = *act.val(h);
    state = (act.dcap && v == kFreeVal) ? 0u : 2u;  // a hashed key is found only while it is active
    slot = (uint32_t)v;
    if (v < kPending && (uint32_t)(v >> 32) == gen && slot < n_slots && pool.id[slot] == pid &&
        pool.mode[slot] != MM_MODE_DEAD)
      state = 1;
    else if (v < kPending && pt_queued(v))
      state = 3;
  }
  return state;
}

struct LocateArgs {
  uint32_t n;
  const uint64_t* id;        // [n] queried ids (handles on MM_F_DENSE_IDS engines)
  ActiveView act;
  PoolView pool;
  PoolMeta meta;             // the resident pool's partitions
  uint32_t n_slots, gen, n_groups, now;
  const uint16_t* bin_seg;   // [Kp] bin -> partition
  const uint32_t* seg_bin_lo;  // [n_segs + 1]
  const uint32_t* seg_L;     // [n_segs]
  const uint16_t* part_cut;  // [n_segs] partition -> (mode, group) queue
  const uint32_t* cut_lp_lo; // [n_cut + 1] first partition of the queue
  const uint32_t* rmap;      // k_loc_rmap
  const uint32_t* pos;       // [Kp + 1] k_locate_preview: sorted position of the bin's first player
  const uint32_t* outbase;   // [Kp] k_locate_preview: member slot of the bin's first player
  const uint32_t* binlim;    // [Kp] k_locate_preview: end of the bin's matched member slots
  mm_player_status* out;     // [n]
  uint32_t tb_mask;          // team_balance: modes whose lobbies the next tick balances
  bool arrival;              // MM_ORDER_ARRIVAL
  const uint8_t* mode_tsize; // [MM_MAX_MODES]
  const uint16_t* bin_key;   // [Kp] c - key_lo of the bin
  PartyView pt;              // the party table (state 3)
  int32_t key_lo;
  uint32_t KR;
};

// Arrival order, one warp: the lobby of the player at `slot` (partition sg) is L consecutive live players of the
// partition in storage order, the player being member j.  c - key_lo of member i goes to cw[i].
__device__ __forceinline__ void loc_arrival_lobby(const LocateArgs& a, uint32_t slot, uint32_t sg, uint32_t j,
                                                  uint32_t L, uint32_t* cw) {
  const uint32_t lane = threadIdx.x & 31, fill = a.meta.fill[sg];
  const uint32_t* tab = a.meta.chunk_tab + (size_t)sg * a.meta.max_ch;
  auto at = [&](uint32_t p) { return (size_t)tab[p / kTile] * kTile + p % kTile; };
  auto c_of = [&](size_t s) { return clamp_key(a.key_lo, a.KR, a.pool.rating[s]); };
  const uint32_t p0 = a.rmap[slot / kTile] * kTile + slot % kTile;  // the player's index in its partition
  if (lane == 0) cw[j] = c_of(slot);
  // members j - 1 .. 0: the nearest live players before it (lane l looks at index p - 1 - l)
  for (uint32_t need = j, p = p0; need && p;) {  // (uniform)
    const bool live = p > lane && a.pool.mode[at(p - 1 - lane)] != MM_MODE_DEAD;
    const uint32_t bal = __ballot_sync(0xFFFFFFFFu, live), k = __popc(bal & ((1u << lane) - 1u));
    if (live && k < need) cw[need - 1 - k] = c_of(at(p - 1 - lane));
    need -= __popc(bal) < need ? __popc(bal) : need;
    p = p > 32 ? p - 32 : 0;
  }
  // members j + 1 .. L - 1: the nearest live players after it
  for (uint32_t need = L - 1 - j, p = p0 + 1; need && p < fill;) {  // (uniform)
    const bool live = p + lane < fill && a.pool.mode[at(p + lane)] != MM_MODE_DEAD;
    const uint32_t bal = __ballot_sync(0xFFFFFFFFu, live), k = __popc(bal & ((1u << lane) - 1u));
    if (live && k < need) cw[L - need + k] = c_of(at(p + lane));
    need -= __popc(bal) < need ? __popc(bal) : need;
    p += 32;
  }
}

__global__ void __launch_bounds__(256) k_locate(const LocateArgs a) {
  __shared__ uint32_t s_c[8][16];  // team_balance: c - key_lo of the predicted lobby's members, per warp
  const uint32_t lane = threadIdx.x & 31, q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (q >= a.n) return;  // (uniform over the warp)
  const uint64_t pid = a.id[q];
  uint32_t state = 0, slot = 0;
  if (lane == 0 && a.act.on()) state = loc_state(a.act, a.pool, a.n_slots, a.gen, pid, slot);
  state = __shfl_sync(0xFFFFFFFFu, state, 0);
  slot = __shfl_sync(0xFFFFFFFFu, slot, 0);
  mm_player_status r{};
  r.lobby = MM_LOCATE_STAYS;
  r.member = 0xFFFFu;
  if (state == 3) {  // queued in a party: the member's own rating, the party's queue, stamp, seq and wait
    const uint32_t o = a.pt.off[slot], n = a.pt.size[slot];
    for (uint32_t k = lane; k < n; k += 32)
      if (a.pt.mid[o + k] == pid) r.rating = a.pt.mrat[o + k];
    r.rating = __reduce_or_sync(0xFFFFFFFFu, (uint32_t)r.rating);  // one lane holds the id
    r.state = 3;
    r.mode = a.pt.mode[slot];
    r.group = a.pt.grp[slot];
    r.enq_ts = a.pt.ts[slot];
    r.seq = a.pt.seq[slot];
    const int32_t w = (int32_t)(a.now - r.enq_ts);
    r.wait = w < 0 ? 0u : (uint32_t)w;
    if (lane == 0) a.out[q] = r;
    return;
  }
  if (state != 1) {
    r.state = (uint8_t)state;
    if (lane == 0) a.out[q] = r;
    return;
  }
  const uint32_t v = a.pool.bin[slot], sg = a.bin_seg[v];
  const uint32_t rank = bin_rank(a.pool, a.meta, a.seg_bin_lo, a.rmap, slot, v, sg);
  const uint32_t c = a.part_cut[sg], b0 = a.seg_bin_lo[a.cut_lp_lo[c]], b1 = a.seg_bin_lo[a.cut_lp_lo[c + 1]];
  r.state = 1;
  r.mode = a.pool.mode[slot];
  r.group = (uint8_t)(c % a.n_groups);
  r.rating = a.pool.rating[slot];
  r.enq_ts = a.pool.ts[slot];
  r.seq = a.pool.seq[slot];
  const int32_t w = (int32_t)(a.now - r.enq_ts);
  r.wait = w < 0 ? 0u : (uint32_t)w;
  r.ahead = a.pos[v] - a.pos[b0] + rank;
  r.depth = a.pos[b1] - a.pos[b0];
  const uint32_t m = a.outbase[v] + rank;  // the member slot the tick gives the player
  if (m < a.binlim[v]) {
    const uint32_t rel = m - a.outbase[b0], L = a.seg_L[sg];  // the queue's lobby k = its member slots [k L, k L + L)
    r.lobby = rel / L;
    r.member = (uint16_t)(rel % L);
    const uint32_t S = a.mode_tsize[r.mode];
    if (((a.tb_mask >> r.mode) & 1u) && S > 1) {  // (uniform) the balance pass reorders the lobby
      uint32_t* cw = s_c[(threadIdx.x >> 5) & 7];
      if (a.arrival) {
        loc_arrival_lobby(a, slot, sg, r.member, L, cw);
      } else if (lane < L) {
        const uint32_t x = a.outbase[b0] + r.lobby * L + lane;  // member slot of the lobby's member `lane`
        cw[lane] = a.bin_key[last_le(a.outbase, b0, b1, x)];
      }
      __syncwarp();
      unsigned long long imb;
      const uint32_t mf = tb_split(lane < L ? cw[lane] : 0u, L, S, 0u, &imb);
      r.member = (uint16_t)tb_new_index(mf, r.member, S);
    }
  }
  if (lane == 0) a.out[q] = r;
}

}  // namespace mm
