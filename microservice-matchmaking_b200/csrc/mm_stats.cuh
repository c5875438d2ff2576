// mm_stats.cuh — per-queue status of the resident pool (mm_queue_stats): depth, removals and wait-time histograms per
// (mode, rating group) cut segment, for the players queued now and for the players the last tick matched.
//
// One streaming pass over the columns a section needs: the mode byte (dead slots) and the 4-byte enqueue stamp, plus
// one bit per player of the last tick's left_bits for the match section.  CTAs take contiguous runs of the virtual
// tile sequence the tick uses (geo_build over the partition fills), so a grid never covers chunks that are not in use
// and a CTA mostly stays inside one cut segment: it keeps the segment's histogram in shared memory and flushes the
// non-zero bins with global atomics whenever its run crosses into another segment.
#pragma once
#include <cstddef>

#include "mm_common.cuh"

namespace mm {

constexpr uint32_t kWaitBuckets = MM_WAIT_BUCKETS;
constexpr uint32_t kStatBlock = 256;             // 8 players per thread: one tile per CTA step
constexpr uint32_t kStatWords = sizeof(mm_queue_stat) / 4;
constexpr uint32_t kNoBucket = 0xFFFFu;          // dead / matched / past the fill: counted in no bucket
static_assert(kStatBlock * 8 == kTile, "a CTA step covers one tile");
static_assert(sizeof(mm_queue_stat) == 988, "mm_queue_stat layout");
static_assert(offsetof(mm_queue_stat, n_waiting) == 1 * 4 && offsetof(mm_queue_stat, n_removed) == 2 * 4 &&
                  offsetof(mm_queue_stat, max_wait) == 3 * 4 && offsetof(mm_queue_stat, wait_hist) == 4 * 4 &&
                  offsetof(mm_queue_stat, n_lobbies) == 124 * 4 && offsetof(mm_queue_stat, n_matched) == 125 * 4 &&
                  offsetof(mm_queue_stat, max_match_wait) == 126 * 4 && offsetof(mm_queue_stat, match_wait_hist) == 127 * 4,
              "the kernel's word offsets (o_cnt / o_dead / o_max / o_hist) follow mm_queue_stat");

// Wait of a slot: (now - enq_ts) mod 2^32 read as a signed value, "in the future" clamped to 0.
__device__ __forceinline__ uint32_t stat_wait(uint32_t now, uint32_t ts) {
  const int32_t w = (int32_t)(now - ts);
  return w < 0 ? 0u : (uint32_t)w;
}
// Bucket of a wait: exact below 8, then 4 sub-buckets per octave (include/mm_engine.h lists the bounds).
__device__ __forceinline__ uint32_t stat_bucket(uint32_t w) {
  if (w < 8) return w;
  const uint32_t e = 31 - __clz(w);
  return 8 + 4 * (e - 3) + ((w >> (e - 2)) & 3u);
}

struct StatSection {
  const uint8_t* mode;
  const uint32_t* ts;
  PoolMeta meta;               // fill + chunk table of the pool the section reads
  const uint32_t* left_bits;   // null: waiting section (pool now); else match section (pool the last tick matched)
  uint32_t now;
};
struct StatArgs {
  StatSection sec[2];          // blockIdx.y picks one
  uint32_t n_segs;
  const uint16_t* part_cut;    // [n_segs] partition -> cut segment
  uint32_t* out;               // [n_cut] mm_queue_stat records as words, zeroed before the launch
};

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_queue_stats(const StatArgs a) {
  __shared__ Geo geo;
  __shared__ uint32_t s_gtmp[33];
  __shared__ uint32_t s_hist[kWaitBuckets];
  __shared__ uint32_t s_cnt, s_dead, s_max;
  const bool match = blockIdx.y == 1;
  const StatSection sec = match ? a.sec[1] : a.sec[0];
  // word offsets inside the record (see mm_queue_stat)
  const uint32_t o_cnt = match ? 125u : 1u, o_max = match ? 126u : 3u, o_hist = match ? 127u : 4u, o_dead = 2u;
  const uint32_t tid = threadIdx.x, lane = tid & 31;
  geo_build<BLOCK>(geo, sec.meta.fill, a.n_segs, gridDim.x, s_gtmp);
  const uint32_t s0 = blockIdx.x * geo.tpr;
  if (s0 >= geo.NT) return;  // (uniform)
  const uint32_t s1 = s0 + geo.tpr < geo.NT ? s0 + geo.tpr : geo.NT;
  for (uint32_t i = tid; i < kWaitBuckets; i += BLOCK) s_hist[i] = 0;
  if (tid == 0) { s_cnt = 0; s_dead = 0; s_max = 0; }
  __syncthreads();
  auto flush = [&](uint32_t cut) {
    __syncthreads();
    uint32_t* rec = a.out + (size_t)cut * kStatWords;
    for (uint32_t i = tid; i < kWaitBuckets; i += BLOCK) {
      const uint32_t v = s_hist[i];
      if (v) { atomicAdd(&rec[o_hist + i], v); s_hist[i] = 0; }
    }
    if (tid == 0) {
      if (s_cnt) atomicAdd(&rec[o_cnt], s_cnt);
      if (s_dead && !match) atomicAdd(&rec[o_dead], s_dead);  // removed players only count in the pool now
      if (s_max) atomicMax(&rec[o_max], s_max);
      s_cnt = 0; s_dead = 0; s_max = 0;
    }
    __syncthreads();
  };
  uint32_t cur_cut = ~0u;
  const uint32_t o = tid * 8;
  for (uint32_t s = s0; s < s1; ++s) {
    const TileDesc d = geo_tile(geo, sec.meta, s);
    const uint32_t cut = a.part_cut[d.seg];
    if (cut != cur_cut) {  // (uniform: one tile is one partition)
      if (cur_cut != ~0u) flush(cur_cut);
      cur_cut = cut;
    }
    uint32_t b[8], cnt = 0, dead = 0, mx = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) b[j] = kNoBucket;
    if (o < d.nvalid) {
      const size_t slot = (size_t)d.phys * kTile + o;
      const uint2 m2 = __ldcs(reinterpret_cast<const uint2*>(sec.mode + slot));
      const uint4 t0 = __ldcs(reinterpret_cast<const uint4*>(sec.ts + slot));
      const uint4 t1 = __ldcs(reinterpret_cast<const uint4*>(sec.ts + slot) + 1);
      // match section: a set bit = stayed queued (virtual position s * kTile + o; 8 bits of one word)
      const uint32_t left = match ? (__ldcs(&sec.left_bits[((size_t)s * kTile + o) >> 5]) >> (o & 31)) & 0xFFu : 0u;
      const uint32_t ts[8] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (o + j >= d.nvalid) continue;
        const uint32_t md = ((j < 4 ? m2.x : m2.y) >> (8 * (j & 3))) & 0xFFu;
        if (md == MM_MODE_DEAD) { ++dead; continue; }
        if ((left >> j) & 1u) continue;
        const uint32_t w = stat_wait(sec.now, ts[j]);
        b[j] = stat_bucket(w);
        ++cnt;
        mx = w > mx ? w : mx;
      }
    }
    // warp-aggregated: one shared atomic per distinct bucket of the warp (one in all when the warp's 256 share it)
    const uint32_t b0 = __shfl_sync(0xFFFFFFFFu, b[0], 0);
    bool same = true;
#pragma unroll
    for (int j = 0; j < 8; ++j) same &= b[j] == b0;
    if (__all_sync(0xFFFFFFFFu, same)) {
      if (lane == 0 && b0 != kNoBucket) atomicAdd(&s_hist[b0], 8u * 32u);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint32_t m = __match_any_sync(0xFFFFFFFFu, b[j]);
        if (b[j] != kNoBucket && lane == (uint32_t)(__ffs(m) - 1)) atomicAdd(&s_hist[b[j]], (uint32_t)__popc(m));
      }
    }
    cnt = __reduce_add_sync(0xFFFFFFFFu, cnt);
    dead = __reduce_add_sync(0xFFFFFFFFu, dead);
    mx = __reduce_max_sync(0xFFFFFFFFu, mx);
    if (lane == 0) {
      if (cnt) atomicAdd(&s_cnt, cnt);
      if (dead) atomicAdd(&s_dead, dead);
      if (mx) atomicMax(&s_max, mx);
    }
  }
  flush(cur_cut);
}

}  // namespace mm
