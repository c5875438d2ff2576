// mm_expire.cuh — search timeout (mm_expire): every live queued player whose wait at `now` is >= max_wait leaves the
// pool and the active set, as if mm_remove had been called with its id.
//
// One streaming pass over the mode byte and the 4-byte enqueue stamp of every slot in use (5 B per slot); an expired
// player adds its id, sequence number and bin reads, the bookkeeping of pool_mark_dead and one active-set probe.  CTAs
// take contiguous runs of the virtual tile sequence the tick uses (geo_build over the partition fills), as
// k_queue_stats does, so the grid never covers chunks that are not in use.  The same kernel without `commit` only
// counts: the host runs it first when the caller's output might be too small, so that a refused call changes nothing.
// mm_export_queues releases the players it exports with this kernel too: a partition selection, max_wait = 0 and no
// id output.
#pragma once

#include "mm_active.cuh"
#include "mm_stats.cuh"

namespace mm {

constexpr uint32_t kExpBlock = 256;  // 8 slots per thread: one tile per CTA step
static_assert(kExpBlock * 8 == kTile, "a CTA step covers one tile");

struct ExpireArgs {
  PoolView pool;
  PoolMeta meta;
  uint32_t n_segs;
  uint32_t now, max_wait;
  uint32_t commit;                 // 0: count only (nothing is written but ctr[0])
  ActiveView act;                  // off for MM_F_NO_DEDUPE engines
  uint32_t gen, dead_bin;          // the pool's generation (active-set values), bin K = removed while queued
  const uint16_t* bin_seg;
  const uint32_t* seg_bin_lo;
  uint64_t* out_id;                // one of out_id / out_handle receives the expired ids (unordered)
  uint32_t* out_handle;
  uint32_t* out_seq;               // may be null
  const uint8_t* sel;              // [n_segs] or null: only the partitions with a non-zero byte (mm_export_queues)
  uint32_t* ctr;                   // [0] expired (the output cursor)  [1] active-set entries erased; zeroed by the host
};

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_expire(const ExpireArgs a) {
  __shared__ Geo geo;
  __shared__ uint32_t s_gtmp[33];
  const uint32_t tid = threadIdx.x, lane = tid & 31;
  uint32_t s0, s1;
  if (!geo_cta_run<BLOCK>(geo, a.meta.fill, a.n_segs, s_gtmp, s0, s1)) return;  // (uniform)
  const uint32_t o = tid * 8;
  uint32_t counted = 0, erased = 0;
  for (uint32_t s = s0; s < s1; ++s) {
    const TileDesc d = geo_tile(geo, a.meta, s);
    const size_t base = (size_t)d.phys * kTile + o;
    uint2 m2 = make_uint2(0, 0);
    uint32_t hit = 0;  // bit j: slot base + j expires
    if (o < d.nvalid && (!a.sel || a.sel[d.seg])) {
      m2 = __ldcs(reinterpret_cast<const uint2*>(a.pool.mode + base));
      uint32_t ts[8];
      ld_stamps8(a.pool.ts + base, ts);
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (o + j < d.nvalid && mode8_at(m2, j) != MM_MODE_DEAD && stat_wait(a.now, ts[j]) >= a.max_wait) hit |= 1u << j;
    }
    const uint32_t k = __popc(hit);
    if (!a.commit) { counted += k; continue; }  // (uniform)
    uint32_t q = warp_append(&a.ctr[0], k);  // one global atomic per warp and tile
    if (!hit) continue;
    uint2 dead = m2;  // the thread's 8 mode bytes with the expired ones set to DEAD: one store
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if ((hit >> j) & 1u) (j < 4 ? dead.x : dead.y) |= 0xFFu << (8 * (j & 3));
    *reinterpret_cast<uint2*>(a.pool.mode + base) = dead;
#pragma unroll 1
    for (int j = 0; j < 8; ++j) {
      if (!((hit >> j) & 1u)) continue;
      const uint32_t slot = (uint32_t)(base + j);
      const uint64_t pid = a.pool.id[slot];
      if (a.out_id) a.out_id[q] = pid;
      else if (a.out_handle) a.out_handle[q] = (uint32_t)pid;
      if (a.out_seq) a.out_seq[q] = a.pool.seq[slot];
      ++q;
      pool_mark_dead(a.pool, a.meta, slot, a.dead_bin, a.bin_seg, a.seg_bin_lo);
      if (!a.act.on()) continue;
      // as k_remove: the id's entry leaves the set, if it is this slot's (generation and slot match)
      const uint64_t h = act_find(a.act, pid);
      if (h == ~0ull || *a.act.val(h) != (((unsigned long long)a.gen << 32) | slot)) continue;
      if (!a.act.dcap) *a.act.key(h) = kTombKey;
      *a.act.val(h) = kFreeVal;
      ++erased;
    }
  }
  if (!a.commit) {
    counted = __reduce_add_sync(0xFFFFFFFFu, counted);
    if (lane == 0 && counted) atomicAdd(&a.ctr[0], counted);
  } else {
    erased = __reduce_add_sync(0xFFFFFFFFu, erased);
    if (lane == 0 && erased) atomicAdd(&a.ctr[1], erased);
  }
}

}  // namespace mm
