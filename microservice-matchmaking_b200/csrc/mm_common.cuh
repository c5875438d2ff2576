// mm_common.cuh — shared types and device helpers of the search tick (sm_90a); see mm_kernels.cuh.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/mm_engine.h"

namespace mm {

constexpr int kBlock = 512;           // threads per CTA of every tick phase (two CTAs share an SM)
constexpr uint32_t kTile = 2048;      // players per pool chunk = per TMA tile (a tile never mixes partitions)
constexpr uint32_t kMaxRows = 2048;   // rows (CTAs) of the histogram matrix
constexpr uint32_t kMaxStages = 4;    // depth of the (bin, id) shared-memory ring
constexpr uint32_t kTileBytes = kTile * (8 + 2);
constexpr uint32_t kMaxSegs = MM_MAX_GROUPS * MM_MAX_MODES;  // (mode, group) partitions
constexpr uint32_t kChunkHist = 256;  // counters per chunk histogram row
constexpr uint32_t kFastBins = 255;   // partitions with <= 255 bins rank with warp ballots (8-bit digit + "dead")
constexpr uint64_t kEmptyKey = 0xFFFFFFFFFFFFFFFFull;
constexpr uint64_t kTombKey = 0xFFFFFFFFFFFFFFFEull;
constexpr uint64_t kFreeVal = 0xFFFFFFFFFFFFFFFFull;
constexpr uint64_t kPending = 0x8000000000000000ull;
constexpr uint32_t kGenMask = 0x7FFFFFFFu;  // pool generations live in 31 bits: committed values stay below kPending

// The resident pool: SoA columns over fixed-size chunks of kTile players.  Every (mode, group) partition — the
// reference's per-group queue (search/worker.ex:46-66) x the game_mode selector of LobbyState
// (models/lobby_state.ex:72-79) — owns an ordered list of chunks; inside a partition players sit in enqueue order.
struct PoolView {
  uint64_t* id;
  int32_t* rating;
  uint8_t* mode;
  uint8_t* tsize;
  uint32_t* ts;
  uint16_t* bin;  // derived at ingest: mode * stride + lut[clamp(rating)]; K = removed while queued
  uint32_t* seq;  // enqueue sequence number (mod 2^32): global arrival order across partitions
};
struct PoolMeta {
  uint32_t* fill;       // [n_segs] players of the partition (dead ones included)
  uint32_t* chunk_tab;  // [n_segs][max_ch] physical chunk of the partition's k-th chunk
  uint32_t* bump;       // chunks handed out so far
  uint32_t* tot;        // [K + 1] players per bin (K = removed while queued), kept up to date by ingest / remove / tick
  uint32_t* chist;      // [chunks][kChunkHist] live players of the chunk per key of its partition (key - first key of the
                        // partition), kept up to date by ingest / remove / tick; null when a partition has > 255 keys
  uint32_t max_ch;
};

struct BinMap {
  const uint16_t* lut;  // [KR] clamp key -> bin offset inside the mode
  int32_t key_lo;       // rmin - 1
  uint32_t KR;          // rmax - rmin + 3
  uint32_t stride;      // bins per mode
  uint32_t K;           // live bins; bin K = removed-while-queued players
};

struct SegInfo {        // one layout partition, written by the scan tail
  uint32_t n;           // alive players
  uint32_t n_lobbies;   // lobbies of the partition's cut segment that START in this partition
  uint32_t member_base; // member_ids slot of the first of them
  uint32_t lobby_base;  // first lobby index
  uint32_t left_base;   // leftover players of earlier partitions (rank base of the compaction)
  uint32_t new_chunk;   // first chunk of the partition in the compacted pool
  uint32_t n_left;      // players of the partition that stay queued
  uint32_t reserved;
};

struct TickCtr {
  uint32_t gbar;  // grid barrier of the fused tick kernel (zero at launch: re-armed by the previous tick, see k_tick)
  uint32_t done;  // CTAs that finished the fused tick
  uint32_t n_lobbies, n_matched, n_alive, n_dead, n_resid;
  uint32_t n_tiles;
  uint32_t heavy;  // some bin expects > 8 players per tile: the list ranking uses warp-aggregated nodes
  uint32_t chist_bad;  // placement tiles whose ranked key counts differ from their chunk histogram (must stay 0)
  uint32_t hdr_next;   // fused tick: lobby-header chunks claimed so far (headers_claimed)
  uint32_t left_bad;   // leftover players whose compacted-pool rank falls outside their partition (must stay 0)
  uint32_t clr_done;   // fused tick: CTAs done clearing the compacted pool's chunk histograms
  unsigned long long t[12]; // fused kernel: %globaltimer (ns) at phase boundaries, CTA 0; [3],[6]: max over CTAs;
                            // [3] last row done placing and compacting, [8] last row done with phase 1,
                            // [10] last row done placing; two-pipeline placement, max over rows: [4] first tile
                            // ranked, [7] first slot bases taken
  unsigned long long stall[2][4];  // two-pipeline placement, per half, SM clock cycles summed over the rows: waits on
                                   // [0] hand, [1] the tile's loads, [2] a stage's release before a re-issue; [3] tile loop
};

// Tile geometry of a tick, rebuilt by every CTA from the partition fills: the pool's tiles in (partition, chunk) order
// form the VIRTUAL tile sequence 0 .. NT-1; row r (= CTA r) owns tiles [r * tpr, (r + 1) * tpr).  Virtual position
// = tile * kTile + offset indexes left_bits / src_idx; only the pool loads translate a tile to its physical chunk.
struct Geo {
  uint32_t T0[kMaxSegs + 1];  // first virtual tile of the partition
  uint32_t NT, tpr, n_segs, max_rows;  // max_rows: most rows any partition spans
};

// Active set = {key, value} pairs (hashed: open addressing on the u64 player id) or a direct-mapped value array
// (dense 32-bit host handles, SURVEY §7.3).  value: FREE | PENDING|batch index | (pool generation << 32 | slot).
struct ActiveView {
  unsigned long long* kv;  // hashed: [cap] x {key, value} (one 16-byte pair = one sector); direct: value[dcap]
  uint64_t mask;           // hashed: capacity - 1
  uint64_t dcap;           // direct: handle capacity (mask = 0)
  __device__ __forceinline__ bool on() const { return mask != 0 || dcap != 0; }
  __device__ __forceinline__ unsigned long long* key(uint64_t h) const { return kv + 2 * h; }
  __device__ __forceinline__ unsigned long long* val(uint64_t h) const { return dcap ? kv + h : kv + 2 * h + 1; }
};

__device__ __forceinline__ uint64_t hash64(uint64_t x) {
  x ^= x >> 33; x *= 0xFF51AFD7ED558CCDull; x ^= x >> 33; x *= 0xC4CEB9FE1A85EC53ull; x ^= x >> 33;
  return x;
}
// slot of a resident id, ~0 when absent
__device__ __forceinline__ uint64_t act_find(const ActiveView& a, uint64_t pid) {
  if (a.dcap) return pid < a.dcap ? pid : ~0ull;
  if (pid >= kTombKey) return ~0ull;
  uint64_t h = hash64(pid) & a.mask;
  for (uint64_t probe = 0; probe <= a.mask; ++probe) {
    const unsigned long long k = *a.key(h);
    if (k == pid) return h;
    if (k == kEmptyKey) return ~0ull;
    h = (h + 1) & a.mask;
  }
  return ~0ull;
}

// L2 cache-policy hints: the input columns stream through once (evict_first); the histogram pass keeps the 2-byte bin
// column in L2 for the placement pass (evict_last).
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ void st_hint_u64(uint64_t* a, uint64_t v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.u64 [%0], %1, %2;" ::"l"(a), "l"(v), "l"(pol) : "memory");
}

// ---- TMA (1-D bulk copy) + mbarrier, CTA-local ------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// plain arrival (release, CTA scope): the thread's earlier shared-memory writes are visible to the phase's waiters
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_inval(uint64_t* bar) {
  asm volatile("mbarrier.inval.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// order earlier generic-proxy accesses to shared memory before later async-proxy (TMA) writes
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// barrier among the first `nthreads` threads of the CTA only (named barrier 1)
__device__ __forceinline__ void bar_sync_named(uint32_t nthreads) {
  asm volatile("bar.sync 1, %0;" ::"r"(nthreads) : "memory");
}
// barrier among the 256 threads of one half of the CTA (threads [256 h, 256 h + 256)): named barrier 2 + h
__device__ __forceinline__ void bar_sync_half(uint32_t h) {
  if (h) asm volatile("barrier.sync 3, 256;" ::: "memory");  // literal ids: ptxas reserves only the barriers it sees
  else asm volatile("barrier.sync 2, 256;" ::: "memory");
}
// Grid-wide barrier for the fused tick kernel (cooperative launch: all CTAs are co-resident).
__device__ __forceinline__ void grid_barrier(unsigned int* bar, unsigned int target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(bar, 1u);
    unsigned int v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory");
      if (v < target) __nanosleep(32);
    } while (v < target);
    __threadfence();
  }
  __syncthreads();
}
// The same barrier in two halves: work that needs nothing from the other CTAs can sit between arrive and wait.
__device__ __forceinline__ void grid_arrive(unsigned int* bar) {
  __syncthreads();
  if (threadIdx.x == 0) { __threadfence(); atomicAdd(bar, 1u); }
}
__device__ __forceinline__ void grid_wait(unsigned int* bar, unsigned int target) {
  if (threadIdx.x == 0) {
    unsigned int v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory");
      if (v < target) __nanosleep(32);
    } while (v < target);
    __threadfence();
  }
  __syncthreads();
}
// grid_wait for the 256 threads of half h of the CTA only (thread 0 of the half polls; then the half's named barrier)
__device__ __forceinline__ void grid_wait_half(unsigned int* bar, unsigned int target, uint32_t h) {
  if ((threadIdx.x & 255u) == 0) {
    unsigned int v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory");
      if (v < target) __nanosleep(32);
    } while (v < target);
    __threadfence();
  }
  bar_sync_half(h);
}
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// global -> shared bulk copy (SASS: UBLKCP), completion counted on `bar`, with an L2 cache-policy hint
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t pol) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
          smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
      : "memory");
}

// In-place exclusive scan of a shared-memory array a[0..n) by the whole CTA; returns the
// total.  s_tmp must hold >= 33 words.  Warp-shuffle scan: 3 barriers.
template <int BLOCK>
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t* a, uint32_t n, uint32_t* s_tmp) {
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t per = (n + BLOCK - 1) / BLOCK;
  const uint32_t lo = tid * per < n ? tid * per : n, hi = (lo + per < n) ? lo + per : n;
  uint32_t local = 0;
  for (uint32_t i = lo; i < hi; ++i) local += a[i];
  uint32_t incl = local;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, incl, off);
    if (lane >= (uint32_t)off) incl += v;
  }
  if (lane == 31) s_tmp[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = lane < BLOCK / 32 ? s_tmp[lane] : 0, wi = w;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, wi, off);
      if (lane >= (uint32_t)off) wi += v;
    }
    s_tmp[lane] = wi - w;                 // exclusive warp offsets
    if (lane == 31) s_tmp[32] = wi;       // grand total
  }
  __syncthreads();
  uint32_t run = s_tmp[warp] + incl - local;
  for (uint32_t i = lo; i < hi; ++i) { const uint32_t v = a[i]; a[i] = run; run += v; }
  const uint32_t total = s_tmp[32];
  __syncthreads();
  return total;
}

// Every CTA derives the tick's tile geometry from the partition fills (n_segs <= 512 values: one block scan).
template <int BLOCK>
__device__ __forceinline__ void geo_build(Geo& g, const uint32_t* __restrict__ fill, uint32_t n_segs, uint32_t R,
                                          uint32_t* s_tmp) {
  for (uint32_t p = threadIdx.x; p < n_segs; p += BLOCK) g.T0[p] = (__ldcg(&fill[p]) + kTile - 1) / kTile;
  __syncthreads();
  const uint32_t NT = block_excl_scan<BLOCK>(g.T0, n_segs, s_tmp);
  if (threadIdx.x == 0) {
    g.T0[n_segs] = NT;
    g.NT = NT;
    g.tpr = NT ? (NT + R - 1) / R : 1u;
    g.n_segs = n_segs;
    g.max_rows = 0;
  }
  __syncthreads();
  uint32_t mr = 0;
  for (uint32_t p = threadIdx.x; p < n_segs; p += BLOCK) {
    const uint32_t a = g.T0[p], b = g.T0[p + 1];
    if (b > a) { const uint32_t r = (b - 1) / g.tpr - a / g.tpr + 1; mr = r > mr ? r : mr; }
  }
  mr = __reduce_max_sync(0xFFFFFFFFu, mr);
  if ((threadIdx.x & 31) == 0 && mr) atomicMax(&g.max_rows, mr);
  __syncthreads();
}
// partition owning virtual tile s (s < NT): the last p with T0[p] <= s (empty partitions share their successor's T0)
__device__ __forceinline__ uint32_t geo_seg_of(const Geo& g, uint32_t s) {
  uint32_t a = 0, e = g.n_segs;
  while (e - a > 1) { const uint32_t mid = (a + e) >> 1; if (g.T0[mid] <= s) a = mid; else e = mid; }
  return a;
}
struct TileDesc { uint32_t phys, nvalid, seg; };
__device__ __forceinline__ TileDesc geo_tile(const Geo& g, const PoolMeta& m, uint32_t s) {
  TileDesc d;
  d.seg = geo_seg_of(g, s);
  const uint32_t k = s - g.T0[d.seg];
  d.phys = __ldcg(&m.chunk_tab[(size_t)d.seg * m.max_ch + k]);
  const uint32_t left = __ldcg(&m.fill[d.seg]) - k * kTile;
  d.nvalid = left < kTile ? left : kTile;
  return d;
}
// The descriptors of a row's tiles, computed by the whole CTA in parallel (each is a binary search + two global
// loads: far too slow for the one thread that feeds the TMA ring).  Covers tiles [base, base + kDescCap) of the row.
constexpr uint32_t kDescCap = 64;
struct DescCache {
  uint32_t phys[kDescCap];
  uint32_t nvsg[kDescCap];  // nvalid | seg << 16
};
template <int BLOCK>
__device__ __forceinline__ void desc_fill(DescCache& c, const Geo& g, const PoolMeta& m, uint32_t s_first, uint32_t s_end) {
  for (uint32_t k = threadIdx.x; k < kDescCap; k += BLOCK)
    if (s_first + k < s_end) {
      const TileDesc d = geo_tile(g, m, s_first + k);
      c.phys[k] = d.phys;
      c.nvsg[k] = d.nvalid | (d.seg << 16);
    }
}
// Row prefixes of the histogram matrix: with few rows per partition (R rows over tens of partitions) every row sums
// the rows before it on the fly; only when a partition spans many rows (one rating group over the whole pool) is the
// column-scan phase (and its grid barrier) worth it.  Uniform: every CTA derives the same answer from the geometry.
constexpr uint32_t kInlinePrefixRows = 24;
__device__ __forceinline__ bool geo_use_colscan(const Geo& g) {
  return g.NT > (uint64_t)g.tpr * kInlinePrefixRows && g.max_rows > kInlinePrefixRows;
}
// rows [rlo, rhi] holding tiles of partition p; false when the partition is empty
__device__ __forceinline__ bool geo_rows_of(const Geo& g, uint32_t p, uint32_t& rlo, uint32_t& rhi) {
  const uint32_t a = g.T0[p], b = g.T0[p + 1];
  if (b == a) return false;
  rlo = a / g.tpr; rhi = (b - 1) / g.tpr;
  return true;
}

__device__ __forceinline__ uint32_t bin_of(const BinMap& bm, const uint16_t* s_lut, int32_t rating, uint32_t mode) {
  if (mode == MM_MODE_DEAD) return bm.K;
  int32_t hi = bm.key_lo + (int32_t)bm.KR - 1;
  int32_t r = rating < bm.key_lo ? bm.key_lo : (rating > hi ? hi : rating);
  return mode * bm.stride + s_lut[r - bm.key_lo];
}

}  // namespace mm
