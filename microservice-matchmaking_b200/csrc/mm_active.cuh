// mm_active.cuh — active set (GPU hash table / direct-mapped handle table) and pool ingest kernels
#pragma once
#include "mm_common.cuh"

namespace mm {

// =======================================================================================
// Active set (replaces the Mnesia table of models/active_user.ex) + pool ingest.
// Hashed mode: open addressing, linear probing; keys EMPTY / TOMB / id.  Direct mode (dense 32-bit host handles):
// the handle indexes the value array.  Values: FREE (all ones) when the id is not committed, PENDING|batch_index
// while an enqueue batch is being resolved, (pool_generation << 32 | pool_slot) once the player is queued.
// Generations are 31-bit (kGenMask), so a committed value is always below PENDING.  Generation 0 is never a pool's:
// (0 << 32 | row) = kPtVal(row) is a member of the queued party in that row of the party table (mm_party.cuh), and
// kPtMatched (generation kGenMask, slot 0xFFFFFFFF, past every pool) a matched party member, and any matched or taken
// player an image load put in the set.  Every pool-side test
// (generation == gen, slot < slots, id at the slot) reads both as "not a live pool slot".
//
// Ingest of one chunk of a batch = claim -> [count, scan, cut: only when the batch could overflow the pool]
// -> route -> alloc -> append.  The pool is segmented by (mode, group) partition: `route` counts every ingest
// block's winners per partition, `alloc` turns the counts into per-(partition, block) bases, extends the partition
// chunk lists from the bump allocator and advances the fills, `append` writes every winner to
// fill[partition] + its stable rank among the batch's winners of that partition — enqueue order is kept inside
// the partition, which is all the serialized reference defines (one queue per group, search/worker.ex:46-66).
// =======================================================================================
constexpr uint32_t kEnqChunk = 1u << 20;     // batch entries per ingest chunk when the columns arrive over PCIe (pipelined)
constexpr uint32_t kEnqChunkDev = 1u << 22;  // ... when they are already in HBM: fewer, fuller launches
constexpr uint32_t kIngestItems = 1024;  // batch entries per ingest block: 256 threads x 4, warp-striped
constexpr uint16_t kNoPart = 0xFFFFu;

// E1: validate + claim.  The lowest batch index wins a repeated id (atomicMin), which
// is what a serialized in_queue?/add_user sequence (middleware/worker.ex:65-70) yields.
__global__ void k_enq_claim(uint32_t base, uint32_t n, const uint64_t* __restrict__ id, const int32_t* __restrict__ rating,
                            const uint8_t* __restrict__ mode, const uint8_t* __restrict__ grp_lut, int32_t key_lo,
                            uint32_t KR, uint32_t n_modes, BinMap bm, const uint16_t* __restrict__ bin_seg, ActiveView act,
                            uint64_t* __restrict__ hslot, uint8_t* __restrict__ code, uint16_t* __restrict__ part) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;  // this launch covers batch indices [base, base + n)
  if (t >= n) return;
  const uint32_t i = base + t;
  const uint64_t pid = id[i];
  const int32_t hi = key_lo + (int32_t)KR - 1;
  const int32_t r = rating[i] < key_lo ? key_lo : (rating[i] > hi ? hi : rating[i]);
  const uint32_t grp = grp_lut[r - key_lo];
  const bool bad_id = act.dcap ? pid >= act.dcap : pid >= kTombKey;
  if (mode[i] >= n_modes || bad_id || grp == 0xFF) { code[i] = 2; hslot[i] = ~0ull; part[i] = kNoPart; return; }
  part[i] = bin_seg[bin_of(bm, bm.lut, rating[i], mode[i])];  // the layout partition that holds the player's sort key
  if (!act.on()) { code[i] = 1; hslot[i] = ~0ull; return; }
  if (act.dcap) {
    const unsigned long long old = atomicMin(act.val(pid), kPending | i);
    code[i] = (old < kPending) ? 0 : 1;
    hslot[i] = pid;
    return;
  }
  uint64_t h = hash64(pid) & act.mask;
  for (uint64_t probe = 0; probe <= act.mask; ++probe) {
    unsigned long long k = *act.key(h);
    if (k == kEmptyKey) {
      k = atomicCAS(act.key(h), kEmptyKey, pid);
      if (k == kEmptyKey) k = pid;
    }
    if (k == pid) {
      const unsigned long long old = atomicMin(act.val(h), kPending | i);
      code[i] = (old < kPending) ? 0 : 1;  // committed entry -> "already in the queue"
      hslot[i] = h;
      return;
    }
    h = (h + 1) & act.mask;
  }
  code[i] = 3; hslot[i] = ~0ull;  // table full
}

// ---- only when n_pool + batch could exceed the capacity: exact "the last ones do not fit" cut --------------------
// winners = entries whose PENDING index is their own; per-block winner counts.  A chunk's winners are final once
// every lower batch index has claimed.  A loser keeps PENDING | its winner's index in hslot (unused by the later
// kernels): k_enq_promote gives it the winner's final code.
__global__ void k_enq_count(uint32_t base, uint32_t n, ActiveView act, uint64_t* __restrict__ hslot,
                            uint8_t* __restrict__ code, uint32_t* __restrict__ blocksum) {
  __shared__ uint32_t s_cnt;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t i = base + t;
  bool win = false;
  if (t < n && code[i] == 1) {
    const unsigned long long v = act.on() ? *act.val(hslot[i]) : (kPending | i);
    win = v == (kPending | i);
    if (!win) { code[i] = 0; hslot[i] = v; }  // a lower batch index of this chunk holds the id
  }
  const uint32_t b = __ballot_sync(0xFFFFFFFFu, win);
  if ((threadIdx.x & 31) == 0 && b) atomicAdd(&s_cnt, (uint32_t)__popc(b));
  __syncthreads();
  if (threadIdx.x == 0) blocksum[blockIdx.x] = s_cnt;
}
// exclusive scan of blocksum (single CTA), continued from the running total of the earlier chunks (*total)
__global__ void __launch_bounds__(1024) k_scan_small(uint32_t nb, uint32_t* __restrict__ v, uint32_t* __restrict__ total) {
  __shared__ uint32_t s_sum[1024];
  const uint32_t tid = threadIdx.x;
  const uint32_t before = *total;
  const uint32_t per = (nb + 1023) / 1024;
  const uint32_t lo = tid * per, hi = (lo + per < nb) ? lo + per : nb;
  uint32_t local = 0;
  for (uint32_t i = lo; i < hi && i < nb; ++i) local += v[i];
  s_sum[tid] = local;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {
    uint32_t x = (tid >= (uint32_t)off) ? s_sum[tid - off] : 0;
    __syncthreads();
    s_sum[tid] += x;
    __syncthreads();
  }
  uint32_t run = before + s_sum[tid] - local;
  for (uint32_t i = lo; i < hi && i < nb; ++i) { const uint32_t x = v[i]; v[i] = run; run += x; }
  __syncthreads();  // everyone has read *total
  if (tid == 1023) *total = before + s_sum[1023];
}
// winners whose rank among the batch's winners does not fit the pool are rolled back with code 3
__global__ void k_enq_cut(uint32_t base, uint32_t n, ActiveView act, const uint64_t* __restrict__ hslot,
                          uint8_t* __restrict__ code, const uint32_t* __restrict__ blockoff, uint32_t room,
                          uint32_t* __restrict__ n_rejected_cap) {
  __shared__ uint32_t s_warp[32];
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t i = base + t;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool win = t < n && code[i] == 1;
  const uint32_t b = __ballot_sync(0xFFFFFFFFu, win);
  if (lane == 0) s_warp[warp] = __popc(b);
  __syncthreads();
  uint32_t woff = 0;
  for (uint32_t w = 0; w < warp; ++w) woff += s_warp[w];
  if (!win) return;
  const uint32_t grank = blockoff[blockIdx.x] + woff + __popc(b & ((1u << lane) - 1u));
  if (grank >= room) {
    code[i] = 3;
    if (act.on()) {
      *act.val(hslot[i]) = kFreeVal;
      if (!act.dcap) *act.key(hslot[i]) = kTombKey;
    }
    atomicAdd(n_rejected_cap, 1u);
  }
}
// a repeat whose batch winner was rolled back did not fit either: code 3, as if the repeat had been offered alone
// (it holds no active-set entry, so it is not counted in n_rejected_cap, which feeds the tombstone count)
__global__ void k_enq_promote(uint32_t base, uint32_t n, const uint64_t* __restrict__ hslot, uint8_t* __restrict__ code) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const uint32_t i = base + t;
  if (code[i] != 0) return;
  const uint64_t v = hslot[i];
  if (v >= kPending && code[(uint32_t)v] == 3) code[i] = 3;
}

// E2: winners per (ingest block, partition).  blockhist is [n_segs][nblk].
__global__ void __launch_bounds__(256) k_enq_route(uint32_t base, uint32_t n, ActiveView act,
                                                   const uint64_t* __restrict__ hslot, uint8_t* __restrict__ code,
                                                   const uint16_t* __restrict__ part, uint32_t n_segs, uint32_t nblk,
                                                   uint32_t* __restrict__ blockhist) {
  __shared__ uint32_t s_hist[kMaxSegs];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (uint32_t p = tid; p < n_segs; p += 256) s_hist[p] = 0;
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t t = blockIdx.x * kIngestItems + warp * 128 + j * 32 + lane;
    if (t < n) {
      const uint32_t i = base + t;
      if (code[i] == 1) {
        const bool win = !act.on() || *act.val(hslot[i]) == (kPending | i);
        if (win) atomicAdd(&s_hist[part[i]], 1u);
        else code[i] = 0;  // a lower batch index holds the id: "already in the queue"
      }
    }
  }
  __syncthreads();
  for (uint32_t p = tid; p < n_segs; p += 256) blockhist[(size_t)p * nblk + blockIdx.x] = s_hist[p];
}

// E3 (one CTA): blockhist -> per-(partition, block) append bases; new chunks from the bump allocator; fills advance.
// counters[0] += players accepted by this chunk.
__global__ void __launch_bounds__(512) k_enq_alloc(uint32_t n_segs, uint32_t nblk, uint32_t* __restrict__ blockhist,
                                                   PoolMeta meta, uint32_t* __restrict__ counters) {
  __shared__ uint32_t s_old[kMaxSegs], s_new[kMaxSegs], s_need[kMaxSegs], s_tmp[64];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (uint32_t p = warp; p < n_segs; p += 16) {  // one warp per partition: shuffle scan over the blocks, 32 at a time
    const uint32_t fill = meta.fill[p];
    uint32_t carry = fill;
    uint32_t* hrow = blockhist + (size_t)p * nblk;
    for (uint32_t b0 = 0; b0 < nblk; b0 += 1024) {  // 32 loads in flight per lane: one memory round trip per 1024 blocks
      uint32_t v[32];
#pragma unroll
      for (int k = 0; k < 32; ++k) { const uint32_t b = b0 + k * 32 + lane; v[k] = b < nblk ? hrow[b] : 0u; }
#pragma unroll
      for (int k = 0; k < 32; ++k) {
        if (b0 + (uint32_t)k * 32 >= nblk) break;
        const uint32_t b = b0 + k * 32 + lane;
        uint32_t incl = v[k];
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
          const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, incl, off);
          if (lane >= (uint32_t)off) incl += u;
        }
        if (b < nblk) hrow[b] = carry + incl - v[k];
        carry += __shfl_sync(0xFFFFFFFFu, incl, 31);
      }
    }
    if (lane == 0) {
      s_old[p] = fill; s_new[p] = carry;
      s_need[p] = (carry + kTile - 1) / kTile - (fill + kTile - 1) / kTile;
    }
  }
  __syncthreads();
  uint32_t added = 0;
  for (uint32_t p = tid; p < n_segs; p += 512) added += s_new[p] - s_old[p];
  added = __reduce_add_sync(0xFFFFFFFFu, added);
  if (lane == 0 && added) atomicAdd(&counters[0], added);
  const uint32_t total = block_excl_scan<512>(s_need, n_segs, s_tmp);  // -> first new chunk of the partition (relative)
  const uint32_t bump = *meta.bump;
  for (uint32_t p = warp; p < n_segs; p += 16) {
    const uint32_t have = (s_old[p] + kTile - 1) / kTile, want = (s_new[p] + kTile - 1) / kTile;
    for (uint32_t k = lane; k < want - have; k += 32) meta.chunk_tab[(size_t)p * meta.max_ch + have + k] = bump + s_need[p] + k;
    if (lane == 0) meta.fill[p] = s_new[p];
  }
  if (meta.chist)  // chunks come from a bump allocator that restarts every tick: a new chunk starts with an empty histogram
    for (size_t i = (size_t)bump * kChunkHist + tid; i < (size_t)(bump + total) * kChunkHist; i += 512) meta.chist[i] = 0;
  __syncthreads();
  if (tid == 0) *meta.bump = bump + total;
}

// E4: append winners to their partition in batch order (= enqueue order) and commit their active-set entries.
// Stable rank inside the block: peers of the same partition inside a warp by ballots over the partition index bits,
// per-warp counters in shared memory, prefix over the block's 8 warps.  The block's winners are then laid out by
// (partition, rank) in shared memory — only their batch-local index — and the write-back walks that order: consecutive
// threads write consecutive pool slots (one run per partition), the inputs are gathered from the block's 1024-entry
// window of the batch columns.
__global__ void __launch_bounds__(256) k_enq_append(uint32_t base, uint32_t n, const uint64_t* __restrict__ id,
                                                    const int32_t* __restrict__ rating, const uint8_t* __restrict__ mode,
                                                    const uint32_t* __restrict__ ts, const uint8_t* __restrict__ mode_tsize,
                                                    ActiveView act, const uint64_t* __restrict__ hslot,
                                                    const uint8_t* __restrict__ code, const uint16_t* __restrict__ part,
                                                    uint32_t n_segs, uint32_t nblk, const uint32_t* __restrict__ blockbase,
                                                    PoolView pool, PoolMeta meta, uint32_t gen, uint32_t seq_base, BinMap bm,
                                                    const uint32_t* __restrict__ seg_bin_lo) {
  extern __shared__ __align__(16) uint32_t s_dyn[];  // start[n_segs] | bbase[n_segs] | tmp[64] | wc[8][n_segs+1] u16 | src[1024] u16 | sp[1024] u16
  const uint32_t S1 = n_segs + 1;                     // digit n_segs = not a winner
  uint32_t* start = s_dyn;
  uint32_t* bbase = start + n_segs;
  uint32_t* s_tmp = bbase + n_segs;
  uint16_t* wc = reinterpret_cast<uint16_t*>(s_tmp + 64);
  uint16_t* src = wc + ((8 * S1 + 1) & ~1u);
  uint16_t* sp = src + kIngestItems;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t lt_mask = (1u << lane) - 1u;
  for (uint32_t k = tid; k < 8 * S1; k += 256) wc[k] = 0;
  for (uint32_t p = tid; p < n_segs; p += 256) bbase[p] = blockbase[(size_t)p * nblk + blockIdx.x];
  __syncthreads();
  const uint32_t nbits = 32u - __clz(n_segs);
  const uint32_t blk0 = base + blockIdx.x * kIngestItems;
  uint32_t dg[4], rk[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t li = warp * 128 + j * 32 + lane, t = blockIdx.x * kIngestItems + li;
    dg[j] = (t < n && code[blk0 + li] == 1) ? (uint32_t)part[blk0 + li] : n_segs;
    uint32_t peers = 0xFFFFFFFFu;
    for (uint32_t bit = 0; bit < nbits; ++bit) {
      const bool on = (dg[j] >> bit) & 1u;
      const uint32_t bal = __ballot_sync(0xFFFFFFFFu, on);
      peers &= on ? bal : ~bal;
    }
    const uint32_t leader = __ffs(peers) - 1;
    uint32_t old = 0;
    uint16_t* c = wc + warp * S1 + dg[j];
    if (lane == leader) { old = *c; *c = (uint16_t)(old + __popc(peers)); }
    __syncwarp();
    old = __shfl_sync(0xFFFFFFFFu, old, leader);
    rk[j] = old + __popc(peers & lt_mask);
  }
  __syncthreads();
  for (uint32_t p = tid; p < n_segs; p += 256) {  // prefix over the 8 warps; the partition's winners in this block
    uint32_t run = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) { const uint32_t v = wc[w * S1 + p]; wc[w * S1 + p] = (uint16_t)run; run += v; }
    start[p] = run;
  }
  __syncthreads();
  const uint32_t n_win = block_excl_scan<256>(start, n_segs, s_tmp);  // -> the partition's first sorted position
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (dg[j] >= n_segs) continue;
    const uint32_t q = start[dg[j]] + wc[warp * S1 + dg[j]] + rk[j];
    src[q] = (uint16_t)(warp * 128 + j * 32 + lane);
    sp[q] = (uint16_t)dg[j];
  }
  __syncthreads();
  for (uint32_t q0 = 0; q0 < n_win; q0 += 1024) {
    uint32_t slot[4], i[4], bin[4];
    uint64_t pid[4];
    int32_t rt[4];
    uint8_t md[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t q = q0 + j * 256 + tid;
      slot[j] = ~0u;
      if (q >= n_win) continue;
      const uint32_t p = sp[q];
      const uint32_t pos = bbase[p] + (q - start[p]);
      i[j] = blk0 + src[q];
      slot[j] = meta.chunk_tab[(size_t)p * meta.max_ch + pos / kTile] * kTile + pos % kTile;
      pid[j] = id[i[j]]; rt[j] = rating[i[j]]; md[j] = mode[i[j]];
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (slot[j] == ~0u) continue;
      bin[j] = bin_of(bm, bm.lut, rt[j], md[j]);  // the tick's sort key, derived once at ingest
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (slot[j] == ~0u) continue;
      const uint32_t s = slot[j];
      pool.id[s] = pid[j]; pool.rating[s] = rt[j]; pool.mode[s] = md[j];
      pool.tsize[s] = mode_tsize[md[j]]; pool.ts[s] = ts ? ts[i[j]] : 0u;
      pool.bin[s] = (uint16_t)bin[j];
      pool.seq[s] = seq_base + i[j];
      atomicAdd(&meta.tot[bin[j]], 1u);  // bin totals stay current: the tick needs no counting pass for them
      if (meta.chist) atomicAdd(&meta.chist[(size_t)(s / kTile) * kChunkHist + (bin[j] - seg_bin_lo[sp[q0 + j * 256 + tid]])], 1u);
      if (act.on()) *act.val(act.dcap ? pid[j] : hslot[i[j]]) = ((unsigned long long)gen << 32) | s;  // dense set: the handle is the slot
    }
  }
}

// ActiveUser.remove_user/1 (models/active_user.ex:57-66), batched.  A player still
// queued is tombstoned in the pool (mode byte = DEAD) so the next tick drops it the way
// remove_inactive_players/1 (search/worker.ex:267-280) filters it.
// bookkeeping of a queued player that turns "removed": bin totals, chunk histogram, sort key
__device__ __forceinline__ void pool_mark_dead(PoolView pool, const PoolMeta& meta, uint32_t slot, uint32_t dead_bin,
                                               const uint16_t* __restrict__ bin_seg, const uint32_t* __restrict__ seg_bin_lo) {
  const uint32_t b = pool.bin[slot];
  atomicSub(&meta.tot[b], 1u);
  atomicAdd(&meta.tot[dead_bin], 1u);
  if (meta.chist) atomicSub(&meta.chist[(size_t)(slot / kTile) * kChunkHist + (b - seg_bin_lo[bin_seg[b]])], 1u);
  pool.bin[slot] = (uint16_t)dead_bin;
}

__global__ void k_remove(uint32_t n, const uint64_t* __restrict__ id, ActiveView act, PoolView pool, PoolMeta meta,
                         uint32_t n_slots, uint32_t gen, uint32_t dead_bin, const uint16_t* __restrict__ bin_seg,
                         const uint32_t* __restrict__ seg_bin_lo, uint32_t* __restrict__ n_removed) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !act.on()) return;
  const uint64_t pid = id[i];
  const uint64_t h = act_find(act, pid);
  if (h == ~0ull) return;
  unsigned long long v;
  if (act.dcap) {
    v = atomicExch(act.val(h), kFreeVal);
    if (v == kFreeVal) return;  // not active (or a twin in this batch won)
  } else {
    v = *act.val(h);
    if (atomicCAS(act.key(h), (unsigned long long)pid, kTombKey) != pid) return;  // a twin in this batch won
    *act.val(h) = kFreeVal;
  }
  const uint32_t slot = (uint32_t)v, g = (uint32_t)(v >> 32);
  // a player taken since the tick (mm_take) is dead already: its bin totals and chunk histogram were updated then
  if (v < kPending && g == gen && slot < n_slots && pool.id[slot] == pid && pool.mode[slot] != MM_MODE_DEAD) {
    pool.mode[slot] = MM_MODE_DEAD;
    pool_mark_dead(pool, meta, slot, dead_bin, bin_seg, seg_bin_lo);
  }
  atomicAdd(n_removed, 1u);
}

// A queued slot leaves the pool the way mm_take takes it (its active-set entry is left as it is); false if it was dead
// already.  A twin in the same batch must not count twice: the mode byte is the claim.
__device__ __forceinline__ bool pool_take_slot(PoolView pool, const PoolMeta& meta, uint32_t slot, uint32_t dead_bin,
                                               const uint16_t* __restrict__ bin_seg,
                                               const uint32_t* __restrict__ seg_bin_lo) {
  const uint32_t word = slot & ~3u, sh = (slot & 3u) * 8;
  uint32_t* mw = reinterpret_cast<uint32_t*>(pool.mode + word);
  const uint32_t old = atomicOr(mw, 0xFFu << sh);
  if (((old >> sh) & 0xFFu) == MM_MODE_DEAD) return false;
  pool_mark_dead(pool, meta, slot, dead_bin, bin_seg, seg_bin_lo);
  return true;
}

// mm_take: queued players matched OUTSIDE this engine's tick (the cross-group boundary pass, shard.py) leave the pool
// but stay in the active set — exactly like members of an emitted lobby, who are "in the queue" until the lobby stage
// removes them (game-lobby/worker.ex:80).
__global__ void k_take(uint32_t n, const uint64_t* __restrict__ id, ActiveView act, PoolView pool, PoolMeta meta,
                       uint32_t n_slots, uint32_t gen, uint32_t dead_bin, const uint16_t* __restrict__ bin_seg,
                       const uint32_t* __restrict__ seg_bin_lo, uint32_t* __restrict__ n_taken) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !act.on()) return;
  const uint64_t pid = id[i];
  const uint64_t h = act_find(act, pid);
  if (h == ~0ull) return;
  const unsigned long long v = *act.val(h);
  const uint32_t slot = (uint32_t)v, g = (uint32_t)(v >> 32);
  if (v < kPending && g == gen && slot < n_slots && pool.id[slot] == pid &&
      pool_take_slot(pool, meta, slot, dead_bin, bin_seg, seg_bin_lo))
    atomicAdd(n_taken, 1u);
}

// ActiveUser.in_queue?/1 (models/active_user.ex:33-44), batched.
__global__ void k_lookup(uint32_t n, const uint64_t* __restrict__ id, ActiveView act, uint8_t* __restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint8_t found = 0;
  if (act.on()) {
    const uint64_t h = act_find(act, id[i]);
    if (h != ~0ull) found = act.dcap ? (*act.val(h) != kFreeVal) : 1;
  }
  out[i] = found;
}

// Rebuild without tombstones: re-insert every committed entry of the old table (hashed mode).
__global__ void k_rehash(ActiveView oldt, ActiveView newt) {
  for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s <= oldt.mask; s += (uint64_t)gridDim.x * blockDim.x) {
    const unsigned long long k = *oldt.key(s);
    if (k >= kTombKey) continue;
    uint64_t h = hash64(k) & newt.mask;
    for (;;) {
      if (atomicCAS(newt.key(h), kEmptyKey, k) == kEmptyKey) { *newt.val(h) = *oldt.val(s); break; }
      h = (h + 1) & newt.mask;
    }
  }
}

// After mm_restore / a generation wrap: point every queued player's entry at its slot again.
// grid = (chunks in use, partitions): block (k, p) handles the partition's k-th chunk.  sel (may be null): only the
// partitions with a non-zero byte (mm_requeue).
__global__ void k_restamp(PoolView pool, PoolMeta meta, ActiveView act, uint32_t gen, const uint8_t* __restrict__ sel) {
  const uint32_t p = blockIdx.y, k = blockIdx.x;
  if (sel && !sel[p]) return;
  const uint32_t fill = meta.fill[p];
  if ((uint64_t)k * kTile >= fill || !act.on()) return;
  const uint32_t cnt = fill - k * kTile < kTile ? fill - k * kTile : kTile;
  const uint32_t c = meta.chunk_tab[(size_t)p * meta.max_ch + k];
  for (uint32_t o = threadIdx.x; o < cnt; o += blockDim.x) {
    const uint32_t slot = c * kTile + o;
    if (pool.mode[slot] == MM_MODE_DEAD) continue;
    const uint64_t h = act_find(act, pool.id[slot]);
    if (h != ~0ull) *act.val(h) = ((unsigned long long)gen << 32) | slot;
  }
}

// empty hashed active set: every slot {EMPTY key, FREE value}
__global__ void k_fill_kv(ulonglong2* p, uint64_t n, unsigned long long k, unsigned long long v) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    p[i] = make_ulonglong2(k, v);
}

// batch indices whose code is not 1 ("queued"), compacted for the host (unordered): the ack / nack list of a batch
__global__ void k_compact_rejects(uint32_t n, const uint8_t* __restrict__ code, uint32_t cap, uint32_t* __restrict__ idx,
                                  uint8_t* __restrict__ rcode, uint32_t* __restrict__ count) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool rej = i < n && code[i] != 1;
  const uint32_t b = __ballot_sync(0xFFFFFFFFu, rej);
  if (!b) return;
  const uint32_t lane = threadIdx.x & 31;
  uint32_t base = 0;
  if (lane == 0) base = atomicAdd(count, (uint32_t)__popc(b));
  base = __shfl_sync(0xFFFFFFFFu, base, 0);
  if (rej) {
    const uint32_t o = base + __popc(b & ((1u << lane) - 1u));
    if (o < cap) { idx[o] = i; rcode[o] = code[i]; }
  }
}

// ---- packed host formats (mm_enqueue_packed / mm_tick_packed): 6 B per player up, 4 B per player down ----------
// key = mode << 13 | rating (0 .. 8191); the 32-bit host handle is the player id on the device
__global__ void k_unpack(uint32_t n, const uint32_t* __restrict__ handle, const uint16_t* __restrict__ key,
                         uint64_t* __restrict__ id, int32_t* __restrict__ rating, uint8_t* __restrict__ mode) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t k = key[i];
  id[i] = handle[i]; rating[i] = (int32_t)(k & 0x1FFFu); mode[i] = (uint8_t)(k >> 13);
}
__global__ void k_narrow(uint32_t n, const uint64_t* __restrict__ src, uint32_t* __restrict__ dst) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[i] = (uint32_t)src[i];
}

}  // namespace mm
