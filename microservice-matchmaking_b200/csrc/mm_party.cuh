// mm_party.cuh — parties on the device (mm_enqueue_party / mm_party_match, DESIGN §4): players who queue together are
// matched into one lobby and one team.  Parties live in a table of their own beside the pool, which the tick never
// reads.
//
// Table: one row per party, the LIVE rows in age order (every party of an accepted batch consumes one enqueue sequence
// number, so rows and solos share the numbering of emit_seq), its members in a member array at the row's offset.  Dead
// rows need not be in order with the live ones: mm_merge_parties(MM_PARTY_KEEP_SEQ) on a table whose parties were all
// released appends the image's (older) numbers after the released rows.  A queued member's active-set value is kPtVal(row) (pool generation 0, which no pool ever has); a matched
// member's is kPtMatched (a slot past every pool), which every call reads as a matched player.  Rows of matched,
// dissolved and expired parties stay in place, `dead`, until the next compaction (k_pt_keep / k_pt_move: stable, by age).
//
// Enqueue: k_pt_claim claims every member id in the active set as k_enq_claim does (the lowest batch index wins);
// k_pt_resolve gives every party its code 2 (invalid) or 0 (a member was queued before the call, or belongs to an
// earlier party of the batch, accepted or not) from its own members alone; the candidates' member counts are scanned
// (k_scan_small) and k_pt_commit cuts the last parties that do not fit (code 3) and writes the rows; k_pt_members
// writes the member rows and active-set values, and frees every id whose first occurrence lost.
//
// Match: after compaction the rows are counting-sorted by (bin, age) — bins are the solo pool's, so a queue's parties
// are the runs of its bins — and k_pt_plan serves one queue per warp.  The warp takes the queue's anchors in age
// order, walks the bins outward from the anchor's bin in (distance, rating) order for co-parties (sequential: every
// placement changes the rooms), then counts the solos of the open slots with bf_walk<false>.  Only a full lobby commits:
// the same co-party walk again, then one bf_walk<true, walk order> per team with open slots, so the solos fill team 0,
// then team 1, ... in their rank order.  The solo pieces go through k_bf_keys, the band pipeline and k_bf_out like
// mm_widen's; k_wd_bases / k_wd_hdr write the headers and bases and k_pt_out copies the party members.
//
// Balance (mm_set_option "party_balance", mm_balance.cuh): after k_pt_out, k_tb_pieces gives every solo its c and
// k_tb_parties every placed member its own c and its party's stamp (the off-tick report, mm_offtick.cuh) and, in a
// masked mode, its lobby the party's continuation bits; then k_tb_lobby<true, true> splits each lobby of a masked
// mode, every party kept whole.
//
// Hand-over (mm_export_parties / mm_merge_parties): k_pt_sel and two k_scan_small give every selected live row its
// image index and member offset, k_pt_export gathers the columns in age order and releases the row (pt_release, as
// k_pt_dissolve does).  The merge is the enqueue pipeline with the image's numbers (PtEnqArgs::seq) or new ones; its
// refusal for room comes before k_pt_commit, and k_pt_unclaim gives the claims back.
//
// Requeue (mm_requeue_party): matched parties back into the table at their age position, a merge of the live rows and
// the requeued parties into the other buffer (k_pq_*, "requeue" below).
#pragma once

#include "mm_widen.cuh"

namespace mm {

static_assert(sizeof(mm_party_stats) == 32, "mm_party_stats is 32 bytes (include/mm_engine.h)");

constexpr uint32_t kPtPlanWarps = 4;
constexpr uint32_t kPtMaxTeams = 256;
constexpr uint32_t kPtNone = 0xFFFFFFFFu;

// the counters of one party call (zeroed by the host)
enum PtCtr : uint32_t { kPtAccepted = 0, kPtReleased, kPtRows, kPtMembers, kPtGone, kPtAnchors, kPtPlaced, kPtWords };

// ---- enqueue ----------------------------------------------------------------------------------------------------------
struct PtEnqArgs {
  uint32_t n, m;                 // parties, members
  const uint8_t* size;           // [n]
  const uint32_t* moff;          // [n] first member of the party in the batch
  const uint32_t* mparty;        // [m] member -> party
  const uint64_t* id;            // [m]
  const int32_t* rating;         // [m]
  const uint8_t* mode;           // [n]
  const uint32_t* ts;            // [n] or null
  ActiveView act;
  BinMap bm;
  const uint8_t* grp_lut;
  const uint8_t* mode_tsize;
  uint32_t n_modes;
  uint64_t* hslot;               // [m] active-set slot of the member's id (~0: invalid id)
  uint8_t* pre;                  // [m] 1: the id was committed before the call
  uint8_t* code;                 // [n]
  uint32_t* msz;                 // [n] candidates' member counts -> exclusive scan
  uint32_t* one;                 // [n] candidates: 1 -> exclusive scan
  uint32_t* tot;                 // [2] scan totals (zeroed)
  uint32_t room;                 // members the table still holds
  uint32_t rows0, mem0, seq0;    // first free row and member entry, seq of party 0
  const uint32_t* seq;           // [n] the parties' own numbers (mm_merge_parties, MM_PARTY_KEEP_SEQ), or null
  PartyView pt;
  uint32_t* ctr;
};

__global__ void k_pt_claim(const PtEnqArgs a) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= a.m) return;
  const uint64_t pid = a.id[j];
  const uint32_t p = a.mparty[j];
  a.pre[j] = 0;
  a.hslot[j] = ~0ull;
  if (a.act.dcap ? pid >= a.act.dcap : pid >= kTombKey) return;
  if (a.act.dcap) {
    a.pre[j] = atomicMin(a.act.val(pid), kPending | p) < kPending;
    a.hslot[j] = pid;
    return;
  }
  uint64_t h = hash64(pid) & a.act.mask;
  for (uint64_t probe = 0; probe <= a.act.mask; ++probe) {
    unsigned long long k = *a.act.key(h);
    if (k == kEmptyKey) {
      k = atomicCAS(a.act.key(h), kEmptyKey, pid);
      if (k == kEmptyKey) k = pid;
    }
    if (k == pid) {
      a.pre[j] = atomicMin(a.act.val(h), kPending | p) < kPending;
      a.hslot[j] = h;
      return;
    }
    h = (h + 1) & a.act.mask;
  }
}

// One thread per party: 2 (invalid) before 0 (a member taken before the call or by an earlier party) before 1.
__global__ void k_pt_resolve(const PtEnqArgs a) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.n) return;
  const uint32_t s = a.size[p], o = a.moff[p], md = a.mode[p];
  bool bad = md >= a.n_modes || s < 2 || s > a.mode_tsize[md < a.n_modes ? md : 0], taken = false;
  long long sum = 0;
  for (uint32_t k = 0; k < s; ++k) {
    const uint64_t h = a.hslot[o + k];
    sum += a.rating[o + k];
    if (h == ~0ull) { bad = true; continue; }
    for (uint32_t k2 = 0; k2 < k; ++k2) bad |= a.id[o + k2] == a.id[o + k];
    taken |= a.pre[o + k] || *a.act.val(h) != (kPending | p);
  }
  long long R = 0;
  if (s) {
    R = sum / (long long)s;
    if (R * (long long)s > sum) --R;  // floor toward minus infinity
  }
  const int32_t Rc = R < INT32_MIN ? INT32_MIN : (R > INT32_MAX ? INT32_MAX : (int32_t)R);
  if (!bad && a.grp_lut[clamp_key(a.bm.key_lo, a.bm.KR, Rc)] == 0xFF) bad = true;
  const uint8_t c = bad ? 2 : (taken ? 0 : 1);
  a.code[p] = c;
  a.msz[p] = c == 1 ? s : 0u;
  a.one[p] = c == 1;
}

// One thread per party after the scans: the cut, then the accepted rows.
__global__ void k_pt_commit(const PtEnqArgs a) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.n || a.code[p] != 1) return;
  const uint32_t s = a.size[p], o = a.moff[p];
  if (a.msz[p] + s > a.room) { a.code[p] = 3; return; }
  const uint32_t row = a.rows0 + a.one[p], md = a.mode[p];
  long long sum = 0;
  for (uint32_t k = 0; k < s; ++k) sum += a.rating[o + k];
  long long R = sum / (long long)s;
  if (R * (long long)s > sum) --R;
  const int32_t Rc = (int32_t)R;  // the mean of 32-bit ratings
  a.pt.seq[row] = a.seq ? a.seq[p] : a.seq0 + p;
  a.pt.ts[row] = a.ts ? a.ts[p] : 0u;
  a.pt.off[row] = a.mem0 + a.msz[p];
  a.pt.R[row] = Rc;
  a.pt.bin[row] = (uint16_t)bin_of(a.bm, a.bm.lut, Rc, md);
  a.pt.mode[row] = (uint8_t)md;
  a.pt.grp[row] = a.grp_lut[clamp_key(a.bm.key_lo, a.bm.KR, Rc)];
  a.pt.size[row] = (uint8_t)s;
  a.pt.dead[row] = 0;
  atomicAdd(&a.ctr[kPtAccepted], s);
}

// One thread per member: accepted parties' member rows and active-set values; ids whose first occurrence lost are freed.
__global__ void k_pt_members(const PtEnqArgs a) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= a.m) return;
  const uint64_t h = a.hslot[j];
  if (h == ~0ull || a.pre[j]) return;
  const uint32_t p = a.mparty[j];
  if (*a.act.val(h) != (kPending | p)) return;  // an earlier party holds the id
  if (a.code[p] == 1) {
    const uint32_t m = a.mem0 + a.msz[p] + (j - a.moff[p]);
    a.pt.mid[m] = a.id[j];
    a.pt.mrat[m] = a.rating[j];
    *a.act.val(h) = kPtVal(a.rows0 + a.one[p]);
    return;
  }
  if (atomicExch(a.act.val(h), kFreeVal) != kFreeVal) {  // a repeat inside the party frees it once
    if (!a.act.dcap) *a.act.key(h) = kTombKey;
    atomicAdd(&a.ctr[kPtReleased], 1u);
  }
}

// ---- compaction -------------------------------------------------------------------------------------------------------
__global__ void k_pt_keep(uint32_t n_rows, PartyView t, uint32_t* __restrict__ keep, uint32_t* __restrict__ msz) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows) return;
  const bool k = t.dead[r] == 0;
  keep[r] = k;
  msz[r] = k ? t.size[r] : 0u;
}

// live row r of `s` -> row q of `d`, its members from entry o on; the members' active-set values follow the row
__device__ __forceinline__ void pt_move_row(const PartyView& s, uint32_t r, const PartyView& d, uint32_t q, uint32_t o,
                                            const ActiveView& act) {
  const uint32_t so = s.off[r], n = s.size[r];
  d.seq[q] = s.seq[r]; d.ts[q] = s.ts[r]; d.off[q] = o; d.R[q] = s.R[r]; d.bin[q] = s.bin[r];
  d.mode[q] = s.mode[r]; d.grp[q] = s.grp[r]; d.size[q] = (uint8_t)n; d.dead[q] = 0;
  for (uint32_t k = 0; k < n; ++k) {
    const uint64_t pid = s.mid[so + k];
    d.mid[o + k] = pid;
    d.mrat[o + k] = s.mrat[so + k];
    const uint64_t h = act_find(act, pid);
    if (h != ~0ull) *act.val(h) = kPtVal(q);
  }
}

// rows kept -> their place in `d` (keep / msz hold the exclusive scans)
__global__ void k_pt_move(uint32_t n_rows, PartyView s, PartyView d, const uint32_t* __restrict__ keep,
                          const uint32_t* __restrict__ msz, ActiveView act) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows || s.dead[r]) return;
  pt_move_row(s, r, d, keep[r], msz[r], act);
}

// ---- remove and expire ------------------------------------------------------------------------------------------------
// mm_remove, before k_remove: every party with a removed member is marked for dissolution.
__global__ void k_pt_mark(uint32_t n, const uint64_t* __restrict__ id, ActiveView act, PartyView t) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !act.on()) return;
  const uint64_t h = act_find(act, id[i]);
  if (h == ~0ull) return;
  const uint64_t v = *act.val(h);
  if (v != kFreeVal && pt_queued(v)) t.dead[(uint32_t)v] = 2;
}

// A party member's entry leaves the set if it still is the row's.  -> 1 if it did.
__device__ __forceinline__ uint32_t pt_free(ActiveView act, uint64_t pid, uint32_t row) {
  const uint64_t h = act_find(act, pid);
  if (h == ~0ull) return 0;
  if (act.dcap) return atomicCAS(act.val(h), kPtVal(row), kFreeVal) == kPtVal(row);
  if (*act.val(h) != kPtVal(row) || atomicCAS(act.key(h), (unsigned long long)pid, kTombKey) != pid) return 0;
  *act.val(h) = kFreeVal;
  return 1;
}

// Row r's members leave the active set (the entries that still are the row's) and the row is gone.  -> entries freed
__device__ __forceinline__ uint32_t pt_release(PartyView t, ActiveView act, uint32_t r) {
  uint32_t freed = 0;
  for (uint32_t k = 0; k < t.size[r]; ++k) freed += pt_free(act, t.mid[t.off[r] + k], r);
  t.dead[r] = 1;
  return freed;
}

// after k_remove: the other members of every marked party leave (counted with the removed ones), the row is gone
__global__ void k_pt_dissolve(uint32_t n_rows, PartyView t, ActiveView act, uint32_t* __restrict__ n_removed,
                              uint32_t* __restrict__ ctr) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows || t.dead[r] != 2) return;
  const uint32_t freed = pt_release(t, act, r);
  if (freed) atomicAdd(n_removed, freed);
  atomicAdd(&ctr[kPtGone], t.size[r]);
}

// ---- hand-over (mm_export_parties / mm_merge_parties) -----------------------------------------------------------------
// The party image's columns (include/mm_engine.h), from section 1 (size) on.
struct PtImgCols {
  uint8_t* size;
  uint32_t* seq;
  uint32_t* ts;
  uint8_t* mode;
  uint8_t* id;  // id_bytes per member
  int32_t* rating;
  uint32_t id_bytes;
};

// a live row of a selected queue (sel: one byte per (mode, group) queue, null: every queue)
__device__ __forceinline__ bool pt_selected(const PartyView& t, const uint8_t* sel, uint32_t n_groups, uint32_t r) {
  return t.dead[r] == 0 && (!sel || sel[t.mode[r] * n_groups + t.grp[r]]);
}

// the export's rows: 1 and the member count per selected row (k_pt_keep's shape), for the two scans
__global__ void k_pt_sel(uint32_t n_rows, PartyView t, const uint8_t* __restrict__ sel, uint32_t n_groups,
                         uint32_t* __restrict__ keep, uint32_t* __restrict__ msz) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows) return;
  const bool k = pt_selected(t, sel, n_groups, r);
  keep[r] = k;
  msz[r] = k ? t.size[r] : 0u;
}

// One thread per selected row, after the scans: its columns at its image index (age order), then its release.
__global__ void k_pt_export(uint32_t n_rows, PartyView t, const uint8_t* __restrict__ sel, uint32_t n_groups,
                            const uint32_t* __restrict__ keep, const uint32_t* __restrict__ msz, PtImgCols out,
                            ActiveView act, uint32_t* __restrict__ n_freed) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows || !pt_selected(t, sel, n_groups, r)) return;
  const uint32_t q = keep[r], o = msz[r], so = t.off[r], n = t.size[r];
  out.size[q] = (uint8_t)n; out.seq[q] = t.seq[r]; out.ts[q] = t.ts[r]; out.mode[q] = t.mode[r];
  for (uint32_t k = 0; k < n; ++k) {
    const uint64_t pid = t.mid[so + k];
    if (out.id_bytes == 8) reinterpret_cast<uint64_t*>(out.id)[o + k] = pid;
    else reinterpret_cast<uint32_t*>(out.id)[o + k] = (uint32_t)pid;
    out.rating[o + k] = t.mrat[so + k];
  }
  const uint32_t freed = pt_release(t, act, r);
  if (freed) atomicAdd(n_freed, freed);
}

// mm_merge_parties refused for room, after k_pt_claim and before any commit: every claim of the batch is undone.  An
// id claimed without `pre` was free before the call; hashed, k_pt_claim inserted its key into an empty slot (it never
// takes a tombstone), so the slot goes back to empty and every probe chain is what it was.
__global__ void k_pt_unclaim(const PtEnqArgs a) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= a.m) return;
  const uint64_t h = a.hslot[j];
  if (h == ~0ull || a.pre[j]) return;
  *a.act.val(h) = kFreeVal;
  if (!a.act.dcap) *a.act.key(h) = kEmptyKey;
}

// ---- requeue (mm_requeue_party) ---------------------------------------------------------------------------------------
// A merge of two age-sorted lists, the table's live rows and the requeued parties, into the other buffer (as a
// compaction).  k_pq_check classifies every member's entry, k_pq_party gives every party its checks and code, the scans
// (k_scan_small) number the code-1 parties and their members and, over k_pt_keep, the live rows and theirs; k_pq_live
// lists the live rows' seqs and member offsets in live-row order (= age order; the dead rows are left out, since they
// need not be in order with the live ones).  k_pq_seat finds each code-1 party's age in that list (one binary search:
// its rank among the live rows, and the collision with a live row of the same seq).  After the one counter read that decides every refusal, k_pq_move moves each live row to
// its own rank plus the code-1 parties older than it (one binary search over the call's ages) and k_pq_write writes the
// requeued rows, their members and active-set values.

// error bits (the host names them in mm_last_error)
constexpr uint32_t kPqBadId = 1, kPqBadMode = 2, kPqBadSize = 4, kPqBadRating = 8, kPqOrder = 16, kPqSeqNext = 32,
                   kPqDup = 64, kPqSeqLive = 128;
// the counters of one requeue (zeroed by the host): error bits, the code-1 parties' members and rows (scan totals), the
// live rows and their members (scan totals)
enum PqCtr : uint32_t { kPqErr = 0, kPqMem, kPqRows, kPqLiveRows, kPqLiveMem, kPqWords };

struct PqArgs {
  uint32_t n, m;                 // parties, members
  const uint8_t* size;           // [n]
  const uint32_t* moff;          // [n] first member of the party in the call
  const uint64_t* id;            // [m]
  const int32_t* rating;         // [m]
  const uint8_t* mode;           // [n]
  const uint32_t* ts;            // [n] or null
  const uint32_t* seq;           // [n]
  uint32_t seq_next;
  uint64_t id_limit;
  ActiveView act;
  const uint8_t* pool_mode;      // the live-slot test of k_rq_check
  uint32_t n_slots, gen;
  unsigned long long* seen;      // empty scratch id set of seen_mask + 1 keys, at most half full
  uint64_t seen_mask;
  BinMap bm;
  const uint8_t* grp_lut;
  const uint8_t* mode_tsize;
  uint32_t n_modes;
  uint64_t* hslot;               // [m] active-set slot of the member's id (~0: none)
  uint8_t* cls;                  // [m] 0 queued (a live solo or a queued party's member), 1 matched, 4 not active
  uint8_t* code;                 // [n]
  uint32_t* msz;                 // [n] code-1 member counts -> exclusive scan
  uint32_t* one;                 // [n] code-1: 1 -> exclusive scan
  uint32_t* at;                  // [2n] code-1 party p: its row (at[p]) and first member entry (at[n + p]) in d
  PartyView t;                   // the table (buffer cur)
  uint32_t n_rows;
  const uint32_t* keep;          // [n_rows] k_pt_keep -> exclusive scans
  const uint32_t* lmsz;
  uint32_t* lseq;                // [live rows] the live rows' seqs, in live-row order (k_pq_live)
  uint32_t* lmo;                 // [live rows] their first member entries among the live rows' members
  PartyView d;                   // buffer cur ^ 1
  uint32_t* ctr;                 // [kPqWords]
};

// floor(sum / s) of s >= 1 ratings (64-bit sum, toward minus infinity), clamped into int32 for a hostile s
__device__ __forceinline__ int32_t pq_mean(const int32_t* r, uint32_t s) {
  long long sum = 0;
  for (uint32_t k = 0; k < s; ++k) sum += r[k];
  long long R = sum / (long long)s;
  if (R * (long long)s > sum) --R;
  return R < INT32_MIN ? INT32_MIN : (R > INT32_MAX ? INT32_MAX : (int32_t)R);
}

// One thread per member: a repeated id (seen_insert), then its active-set entry: live solo or queued party member (0),
// matched (1), not active (4).
__global__ void k_pq_check(const PqArgs a) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= a.m) return;
  const uint64_t pid = a.id[j];
  uint64_t h = ~0ull;
  uint8_t c = 4;
  if (pid >= a.id_limit) {
    atomicOr(&a.ctr[kPqErr], kPqBadId);
  } else {
    if (!seen_insert(a.seen, a.seen_mask, pid)) atomicOr(&a.ctr[kPqErr], kPqDup);
    h = act_find(a.act, pid);
    const unsigned long long v = h == ~0ull ? kFreeVal : *a.act.val(h);
    if (v < kPending) {
      const uint32_t slot = (uint32_t)v;
      const bool queued = ((uint32_t)(v >> 32) == a.gen && slot < a.n_slots && a.pool_mode[slot] != MM_MODE_DEAD) ||
                          pt_queued(v);
      c = queued ? 0 : 1;
    }
  }
  a.hslot[j] = h;
  a.cls[j] = c;
}

// One thread per party: its argument checks and its code, 0 (a member queued) before 4 (a member not active) before 1.
__global__ void k_pq_party(const PqArgs a) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.n) return;
  const uint32_t s = a.size[p], o = a.moff[p], md = a.mode[p], u = a.seq[p] - a.seq_next;
  uint32_t bad = 0;
  if (md >= a.n_modes) bad |= kPqBadMode;
  if (s < 2 || (md < a.n_modes && s > a.mode_tsize[md])) bad |= kPqBadSize;
  if (u == 0) bad |= kPqSeqNext;
  if (p + 1 < a.n && a.seq[p + 1] - a.seq_next <= u) bad |= kPqOrder;
  if (s && a.grp_lut[clamp_key(a.bm.key_lo, a.bm.KR, pq_mean(a.rating + o, s))] == 0xFF) bad |= kPqBadRating;
  bool queued = false, gone = false;
  for (uint32_t k = 0; k < s; ++k) {
    queued |= a.cls[o + k] == 0;
    gone |= a.cls[o + k] == 4;
  }
  const uint8_t c = queued ? 0 : (gone ? 4 : 1);
  a.code[p] = c;
  a.msz[p] = c == 1 ? s : 0u;
  a.one[p] = c == 1;
  if (bad) atomicOr(&a.ctr[kPqErr], bad);
}

// age of a sequence number: (seq - seq_next) mod 2^32, the oldest first
__device__ __forceinline__ uint32_t pq_age(uint32_t seq, uint32_t seq_next) { return seq - seq_next; }

// One thread per live row, after the scans: its seq and member offset at its rank among the live rows.
__global__ void k_pq_live(const PqArgs a) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.n_rows || a.t.dead[r]) return;
  a.lseq[a.keep[r]] = a.t.seq[r];
  a.lmo[a.keep[r]] = a.lmsz[r];
}

// One thread per code-1 party, after k_pq_live: its row and first member entry in d = its rank among the code-1
// parties plus the live rows older than it; a live row of the same age is a collision.
__global__ void k_pq_seat(const PqArgs a) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.n || a.code[p] != 1) return;
  const uint32_t u = pq_age(a.seq[p], a.seq_next), L = a.ctr[kPqLiveRows];
  const uint32_t l = first_not(0, L, [&](uint32_t k) { return pq_age(a.lseq[k], a.seq_next) < u; });
  if (l < L && pq_age(a.lseq[l], a.seq_next) == u) atomicOr(&a.ctr[kPqErr], kPqSeqLive);
  a.at[p] = a.one[p] + l;
  a.at[a.n + p] = a.msz[p] + (l < L ? a.lmo[l] : a.ctr[kPqLiveMem]);
}

// One thread per live row: to its rank among the live rows (= its age rank) plus the code-1 parties older than it.
__global__ void k_pq_move(const PqArgs a) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.n_rows || a.t.dead[r]) return;
  const uint32_t u = pq_age(a.t.seq[r], a.seq_next);
  const uint32_t l = first_not(0, a.n, [&](uint32_t p) { return pq_age(a.seq[p], a.seq_next) < u; });
  const uint32_t q = a.keep[r] + (l < a.n ? a.one[l] : a.ctr[kPqRows]);
  const uint32_t o = a.lmsz[r] + (l < a.n ? a.msz[l] : a.ctr[kPqMem]);
  pt_move_row(a.t, r, a.d, q, o, a.act);
}

// One thread per code-1 party: its row and members in d, in the order given; its members' values become kPtVal(row).
__global__ void k_pq_write(const PqArgs a) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.n || a.code[p] != 1) return;
  const uint32_t s = a.size[p], o = a.moff[p], md = a.mode[p], q = a.at[p], mo = a.at[a.n + p];
  const int32_t R = pq_mean(a.rating + o, s);
  a.d.seq[q] = a.seq[p];
  a.d.ts[q] = a.ts ? a.ts[p] : 0u;
  a.d.off[q] = mo;
  a.d.R[q] = R;
  a.d.bin[q] = (uint16_t)bin_of(a.bm, a.bm.lut, R, md);
  a.d.mode[q] = (uint8_t)md;
  a.d.grp[q] = a.grp_lut[clamp_key(a.bm.key_lo, a.bm.KR, R)];
  a.d.size[q] = (uint8_t)s;
  a.d.dead[q] = 0;
  for (uint32_t k = 0; k < s; ++k) {
    a.d.mid[mo + k] = a.id[o + k];
    a.d.mrat[mo + k] = a.rating[o + k];
    *a.act.val(a.hslot[o + k]) = kPtVal(q);
  }
}

// mm_expire: whole parties whose WAIT >= max_wait, after k_expire on the same counters (ctr[0] the output cursor,
// ctr[1] the entries erased).  Without `commit` only ctr[0] counts.
__global__ void k_pt_expire(uint32_t n_rows, PartyView t, uint32_t now, uint32_t max_wait, uint32_t commit,
                            ActiveView act, uint64_t* __restrict__ out_id, uint32_t* __restrict__ out_handle,
                            uint32_t* __restrict__ out_seq, uint32_t* __restrict__ ctr, uint32_t* __restrict__ pctr) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows || t.dead[r] || stat_wait(now, t.ts[r]) < max_wait) return;
  const uint32_t n = t.size[r];
  const uint32_t q = atomicAdd(&ctr[0], n);
  if (!commit) return;
  uint32_t erased = 0;
  for (uint32_t k = 0; k < n; ++k) {
    const uint64_t pid = t.mid[t.off[r] + k];
    if (out_id) out_id[q + k] = pid;
    else if (out_handle) out_handle[q + k] = (uint32_t)pid;
    if (out_seq) out_seq[q + k] = t.seq[r];
    erased += pt_free(act, pid, r);
  }
  t.dead[r] = 1;
  if (erased) atomicAdd(&ctr[1], erased);
  atomicAdd(&pctr[kPtGone], n);
}

// ---- match ------------------------------------------------------------------------------------------------------------
struct PtArgs {
  PartyView t;
  uint32_t n_rows;
  const uint32_t* pb;      // [K + 1] first sorted party of the bin (exclusive scan of the bin counts)
  uint32_t* pcur;          // [K] scatter cursors, then the plan's first party of the bin not known to be placed
  uint32_t* sorted;        // [n_rows] rows by (bin, age)
  uint32_t* lob;           // [n_rows] lobby record of a placed party, kPtNone
  uint32_t* pos;           // [n_rows] member offset of a placed party inside its lobby
  const uint8_t* mode_tsize;  // [MM_MAX_MODES]
  uint64_t* members;       // lobby members (k_pt_out)
  uint32_t* ctr;           // [kPtWords]
};

__global__ void k_pt_count(const PtArgs p, uint32_t* __restrict__ cnt) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= p.n_rows) return;
  p.lob[r] = kPtNone;
  atomicAdd(&cnt[p.t.bin[r]], 1u);
}
// Stable scatter by bin (row order is age order), one CTA over tiles of 1024 rows in order.  Inside a tile, a row's
// place is the bin's cursor + its bin's rows in the warps before it (the warps' run tables in shared memory) + its
// rank among its warp's peers (__match_any_sync); the first warp holding a bin then advances the bin's cursor.
constexpr uint32_t kPtScatterBlock = 1024;
__global__ void __launch_bounds__(kPtScatterBlock) k_pt_scatter(const PtArgs p) {
  constexpr uint32_t W = kPtScatterBlock / 32;
  __shared__ uint32_t s_bin[W][32], s_cnt[W][32];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (uint32_t r0 = 0; r0 < p.n_rows; r0 += kPtScatterBlock) {
    const uint32_t r = r0 + threadIdx.x;
    const uint32_t b = r < p.n_rows ? p.t.bin[r] : 0xFFFFFFFFu;
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, b);
    const bool lead = (__ffs(peers) - 1) == lane;
    s_bin[warp][lane] = lead ? b : 0xFFFFFFFFu;
    s_cnt[warp][lane] = __popc(peers);
    __syncthreads();
    uint32_t before = 0, after = 0, base = 0;
    if (lead && b != 0xFFFFFFFFu) {
      for (uint32_t w = 0; w < W; ++w) {
        if (w == warp) continue;
        for (uint32_t l = 0; l < 32; ++l)
          if (s_bin[w][l] == b) { (w < warp ? before : after) += s_cnt[w][l]; break; }
      }
      base = p.pcur[b];
    }
    __syncthreads();  // every cursor is read before the first warp of a bin advances it
    if (lead && b != 0xFFFFFFFFu && before == 0) p.pcur[b] = base + __popc(peers) + after;
    const uint32_t at = __shfl_sync(0xFFFFFFFFu, base + before, __ffs(peers) - 1);
    if (b != 0xFFFFFFFFu) p.sorted[at + __popc(peers & ((1u << lane) - 1u))] = r;
    __syncthreads();
  }
}

// The co-party walk around clamp key `target` (pos: the first of the queue's bins [lo, hi) at or above it, window win)
// for anchor row `ar` (kPtNone: no anchor): every unplaced party of the window in (distance, rating, age) order goes to
// the lowest team with room for it.  room[] holds the teams' free slots on entry (the anchor's taken).  commit: the
// placed parties get lobby record r and member offsets t * S + (S - room[t]) (room[t] before the placement).
// Uniform over the warp; lane 0 writes.  -> the free slots left.
__device__ uint32_t pt_walk(const PtArgs& p, const WdArgs& a, uint32_t ar, int32_t target, uint32_t pos, uint32_t lo,
                            uint32_t hi, uint32_t win, uint16_t* room, uint32_t T, uint32_t S, uint32_t open, bool commit,
                            uint32_t r, uint32_t& n_placed) {
  const uint32_t lane = threadIdx.x & 31;
  uint32_t l = pos, h = pos;  // next bins: l - 1 below, h at or above
  while (open >= 2) {
    uint32_t d_l = kBfFar, d_h = kBfFar;
    if (l > lo) { const uint32_t d = (uint32_t)(target - (int32_t)a.bin_key[l - 1]); if (d <= win) d_l = d; }
    if (h < hi) { const uint32_t d = (uint32_t)((int32_t)a.bin_key[h] - target); if (d <= win) d_h = d; }
    if (d_l == kBfFar && d_h == kBfFar) break;
    const uint32_t b = d_l <= d_h ? --l : h++;  // a lower bin first at equal distance
    uint32_t i = p.pcur[b];
    while (i < p.pb[b + 1] && p.lob[p.sorted[i]] != kPtNone) ++i;  // the bin's placed prefix is skipped for good
    __syncwarp();
    if (lane == 0) p.pcur[b] = i;
    __syncwarp();
    for (; i < p.pb[b + 1] && open >= 2; ++i) {
      const uint32_t x = p.sorted[i];
      if (x == ar || p.lob[x] != kPtNone) continue;
      const uint32_t s = p.t.size[x];
      uint32_t t = 0;
      while (t < T && room[t] < s) ++t;
      if (t == T) continue;
      if (commit && lane == 0) { p.lob[x] = r; p.pos[x] = t * S + (S - room[t]); }
      __syncwarp();
      if (lane == 0) room[t] = (uint16_t)(room[t] - s);
      __syncwarp();
      open -= s;
      ++n_placed;
    }
  }
  return open;
}

__global__ void __launch_bounds__(kPtPlanWarps * 32) k_pt_plan(const PtArgs p, const WdArgs a) {
  __shared__ uint32_t s_bin[kPtPlanWarps][32];
  __shared__ uint16_t s_room[kPtPlanWarps][kPtMaxTeams];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, c = blockIdx.x * kPtPlanWarps + warp;
  if (c >= a.n_cut) return;
  const WdRule u = a.rule[c];
  if (u.min_wait == MM_WIDEN_OFF) return;
  const uint32_t lo = a.seg_bin_lo[a.cut_lp_lo[c]], hi = a.seg_bin_lo[a.cut_lp_lo[c + 1]];
  const uint32_t S = p.mode_tsize[c / a.n_groups], T = u.L / S;  // the host refuses T > kPtMaxTeams
  uint16_t* room = s_room[warp];
  const uint32_t cap = a.cap ? a.cap[c] : 0xFFFFFFFFu;  // a capped queue stops after its cap-th lobby
  uint32_t n_lob = 0, n_anc = 0, n_abs = 0, n_placed = 0;
  if (p.pb[hi] == p.pb[lo]) { if (lane == 0) a.qlob[c] = 0; return; }
  // the anchors: the queue's parties that waited long enough, by age
  for (uint32_t r0 = 0; r0 < p.n_rows && n_lob < cap; r0 += 32) {
    const uint32_t x = r0 + lane;
    const bool is_a = x < p.n_rows && p.t.bin[x] >= lo && p.t.bin[x] < hi && stat_wait(a.now, p.t.ts[x]) >= u.min_wait;
    uint32_t bal = __ballot_sync(0xFFFFFFFFu, is_a);
    while (bal && n_lob < cap) {
      const uint32_t ar = r0 + __ffs(bal) - 1;
      bal &= bal - 1;
      ++n_anc;
      if (p.lob[ar] != kPtNone) { ++n_abs; continue; }  // an earlier lobby of the call placed it
      const uint32_t wait = stat_wait(a.now, p.t.ts[ar]);
      const long long w = min((long long)u.w_max, (long long)u.w0 + (long long)((wait - u.min_wait) / u.step) * u.inc);
      const uint32_t win = (uint32_t)min(w, (long long)kBfFar - 1), pos = p.t.bin[ar], sa = p.t.size[ar];
      const int32_t target = (int32_t)a.bin_key[pos];
      for (uint32_t t = lane; t < T; t += 32) room[t] = (uint16_t)(t == 0 ? S - sa : S);
      __syncwarp();
      uint32_t np = 0;
      const uint32_t open = pt_walk(p, a, ar, target, pos, lo, hi, win, room, T, S, u.L - sa, false, 0, np);
      uint32_t left = 0;
      if (open && bf_walk<false>(a, s_bin[warp], target, pos, lo, hi, win, open, left, 0) < open) continue;  // all or nothing
      uint32_t r = 0;
      if (lane == 0) r = atomicAdd(&a.ctr[kWdLobbies], 1u);
      r = __shfl_sync(0xFFFFFFFFu, r, 0);
      if (lane == 0) { a.rec[r] = make_uint2(c, n_lob); p.lob[ar] = r; p.pos[ar] = 0; }
      ++n_lob;
      for (uint32_t t = lane; t < T; t += 32) room[t] = (uint16_t)(t == 0 ? S - sa : S);
      __syncwarp();
      pt_walk(p, a, ar, target, pos, lo, hi, win, room, T, S, u.L - sa, true, r, n_placed);
      ++n_placed;
      for (uint32_t t = 0; t < T; ++t) {  // the solos fill the open slots team by team, in their rank order
        const uint32_t need = room[t];
        if (!need) continue;
        left = t * S + (S - need);
        bf_walk<true, true>(a, s_bin[warp], target, pos, lo, hi, win, need, left, r);
      }
      __syncwarp();
    }
  }
  if (lane == 0) {
    a.qlob[c] = n_lob;
    atomicAdd(&p.ctr[kPtAnchors], n_anc);
    atomicAdd(&p.ctr[kPtPlaced], n_placed);
    if (n_abs) atomicAdd(&a.ctr[kWdAbsorbed], n_abs);
  }
}

// One thread per row: a placed party's members into its lobby; they become matched players and the row is gone.
__global__ void k_pt_out(const PtArgs p, const uint32_t* __restrict__ mbase, ActiveView act) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= p.n_rows || p.lob[r] == kPtNone) return;
  uint64_t* dst = p.members + mbase[p.lob[r]] + p.pos[r];
  const uint32_t o = p.t.off[r];
  for (uint32_t k = 0; k < p.t.size[r]; ++k) {
    const uint64_t pid = p.t.mid[o + k];
    dst[k] = pid;
    const uint64_t h = act_find(act, pid);
    if (h != ~0ull) *act.val(h) = kPtMatched;
  }
  p.t.dead[r] = 1;
}

// One thread per row placed in this call, every mode: its members' c - key_lo and the party's enq_ts at their member
// slots (the off-tick report, mm_offtick.cuh); for a lobby of a party_balance mode (mask), bits pos + 1 .. pos + size
// - 1 (member i continues member i - 1's party) in the continuation word of the lobby's header position (cont zeroed by
// the host).
__global__ void k_tb_parties(const PtArgs p, const WdArgs a, uint32_t mask, int32_t key_lo, uint32_t KR,
                             uint32_t* __restrict__ cval, uint32_t* __restrict__ cont, uint32_t* __restrict__ ts) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= p.n_rows || p.lob[r] == kPtNone) return;
  const uint32_t l = p.lob[r], at = p.pos[r], n = p.t.size[r], o = p.t.off[r], stamp = p.t.ts[r];
  const uint2 x = a.rec[l];
  uint32_t* dst = cval + a.mbase[l] + at;
  uint32_t* dts = ts + a.mbase[l] + at;
  for (uint32_t k = 0; k < n; ++k) {
    dst[k] = clamp_key(key_lo, KR, p.t.mrat[o + k]);
    dts[k] = stamp;
  }
  if ((mask >> p.t.mode[r]) & 1u) atomicOr(&cont[a.qlbase[x.x] + x.y], ((1u << (n - 1)) - 1u) << (at + 1));
}

}  // namespace mm
