// mm_party_backfill.cuh — party backfill on the device (mm_backfill_party, DESIGN §4): the open team slots of running
// lobbies filled with whole queued parties, then with the nearest solos.
//
// The host sorts the requests by queue (stably, as mm_backfill does) and the party table by (bin, age) (mm_party_match's
// compaction, k_pt_count / k_scan_small / k_pt_scatter).  Plan (k_pbf_plan): one warp per queue with requests serves
// them in order on rem (copied from tot) and the sorted table.  A request finds its target's first bin (bf_seek), runs
// the co-party walk from the target (pt_walk: every placed row gets lob = the request's index and pos = t * S + (S -
// room[t]) before its placement), then one solo walk per team with open slots, in team order (bf_walk<true, walk
// order>), each from offset (team base + the team's party members) of the request's output; a team's base is the sum
// of the earlier teams' fills, known when its walk starts.  Every walk takes a bin's oldest untaken solos, so the call
// takes a prefix of every bin, as mm_backfill does.  The plan writes each team's fill and base; k_pbf_pos then turns a
// placed row's pos into its offset inside the request's output (team base + the party members placed in its team
// before it).  The solos go through k_bf_keys, the band pipeline and k_bf_out; k_pt_out copies the party members with
// mbase = the requests' output bases.
#pragma once

#include "mm_party.cuh"

namespace mm {

struct PbfArgs {
  const BfReq* req;        // [n] sorted by queue
  const uint32_t* qr;      // [n_cut + 1] first sorted request of the queue
  const uint32_t* queues;  // [nq] the queues with requests
  uint32_t nq;
  const uint32_t* roff;    // [n + 1] request j's teams are entries roff[j] .. roff[j + 1] - 1 of room / filled / tbase
  const uint16_t* room;    // [roff[n]] open slots per team
  uint32_t* filled;        // [roff[n]] members the team received
  uint32_t* tbase;         // [roff[n]] the team's first member inside the request's output
  uint32_t* n_taken;       // [n] by caller index
};

__global__ void __launch_bounds__(kPtPlanWarps * 32, 1) k_pbf_plan(const PtArgs p, const WdArgs a, const PbfArgs q) {
  __shared__ uint32_t s_bin[kPtPlanWarps][32];
  __shared__ uint16_t s_room[kPtPlanWarps][kPtMaxTeams];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, qi = blockIdx.x * kPtPlanWarps + warp;
  if (qi >= q.nq) return;
  const uint32_t c = q.queues[qi];
  const uint32_t lo = a.seg_bin_lo[a.cut_lp_lo[c]], hi = a.seg_bin_lo[a.cut_lp_lo[c + 1]];
  const uint32_t S = p.mode_tsize[c / a.n_groups];
  const bool parties = p.pb[hi] != p.pb[lo];
  uint16_t* room = s_room[warp];
  uint32_t n_placed = 0;  // (pt_walk counts; the host counts the members instead)
  for (uint32_t s = q.qr[c]; s < q.qr[c + 1]; ++s) {
    const BfReq r = q.req[s];
    const uint32_t o = q.roff[r.idx], T = q.roff[r.idx + 1] - o;  // the host refuses T > kPtMaxTeams
    const uint32_t win = r.window < 0 ? kBfFar - 1 : (uint32_t)r.window;
    const uint32_t pos = bf_seek(a.bin_key, lo, hi, r.target);
    for (uint32_t t = lane; t < T; t += 32) room[t] = q.room[o + t];
    __syncwarp();
    if (parties) pt_walk(p, a, kPtNone, r.target, pos, lo, hi, win, room, T, S, r.count, true, r.idx, n_placed);
    uint32_t base = 0;
    for (uint32_t t = 0; t < T; ++t) {  // the solos fill the open slots team by team, in their rank order
      const uint32_t open = q.room[o + t], need = room[t];
      uint32_t got = 0;
      if (need) {
        uint32_t left = base + (open - need);
        got = bf_walk<true, true>(a, s_bin[warp], r.target, pos, lo, hi, win, need, left, r.idx);
      }
      const uint32_t f = open - need + got;
      if (lane == 0) { q.filled[o + t] = f; q.tbase[o + t] = base; }
      base += f;
    }
    if (lane == 0) q.n_taken[r.idx] = base;
    __syncwarp();  // room is rewritten by the next request
  }
}

// One thread per row: a placed row's pos (t * S + S - room[t] at its placement) -> its offset inside its request's
// output, tbase of its team + the members placed in the team before it.
__global__ void k_pbf_pos(const PtArgs p, const PbfArgs q) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= p.n_rows || p.lob[r] == kPtNone) return;
  const uint32_t j = p.lob[r], S = p.mode_tsize[p.t.mode[r]], x = p.pos[r], t = x / S, e = q.roff[j] + t;
  p.pos[r] = q.tbase[e] + (x - t * S) - (S - q.room[e]);
}

}  // namespace mm
