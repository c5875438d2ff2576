// mm_hist.cuh — phase 1 of the tick: row histograms of the resident bin column
#pragma once
#include "mm_common.cuh"

namespace mm {

// ---------------------------------------------------------------------------------------
// hist_body<BLOCK>: M[row][bin] = number of the row's players in that bin, straight from the resident 16-bit
// bin column (the sort key, derived once at ingest by k_enq_append, tombstoned by k_remove, carried through
// the compaction).  The row's tiles stream through a ring of TMA bulk copies (one 4 KB chunk of the bin
// column per tile, L2 evict-last: the placement pass re-reads the column from L2); shared-memory atomics
// build the row histogram.  Only the bins of the partitions the row touches are written to M — a row's tiles
// are consecutive in (partition, chunk) order, so that is one contiguous bin range.
// Shared memory: ring[8][kTile] u16 | mbarriers | tile descriptors per stage | hist[keys of one partition] | descriptor cache.
// ---------------------------------------------------------------------------------------
constexpr uint32_t kHistStages = 8;  // ring depth: two half-turns of 4 tiles (8 192 players each)

// max_nb = most sort keys any one partition has: the row histogram is kept per partition and flushed to M when the
// row moves on to the next one (tiles come in partition order), so shared memory does not grow with the key domain.
__host__ __device__ constexpr size_t hist_smem_bytes(uint32_t max_nb) {
  return (size_t)kHistStages * kTile * 2 + 256 + (size_t)((max_nb + 4) & ~3u) * 4 + sizeof(DescCache) + 16;
}

template <int BLOCK>
__device__ __forceinline__ void hist_body(unsigned char* smem_raw, const Geo& g, const uint16_t* __restrict__ bins16,
                                          const PoolMeta meta, uint32_t Kp, uint32_t max_nb,
                                          const uint32_t* __restrict__ seg_bin_lo, uint32_t* __restrict__ M) {
  constexpr uint32_t kBytes = kTile * 2, S = kHistStages, H = S / 2;
  uint16_t* ring = reinterpret_cast<uint16_t*>(smem_raw);                            // [S][kTile]
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + (size_t)S * kBytes);       // [S]
  uint32_t* s_nv = reinterpret_cast<uint32_t*>(smem_raw + (size_t)S * kBytes + 64);  // [S] valid players of the tile
  uint32_t* s_sg = s_nv + S;                                                         // [S] its partition
  uint32_t* s_b0 = s_sg + S;                                                         // [S] first key of the partition
  uint32_t* s_b1 = s_b0 + S;                                                         // [S] end key
  uint32_t* hist = reinterpret_cast<uint32_t*>(smem_raw + (size_t)S * kBytes + 256); // [max_nb + 1]
  DescCache& dc = *reinterpret_cast<DescCache*>(hist + ((max_nb + 4) & ~3u));
  const uint32_t tid = threadIdx.x, row = blockIdx.x;
  const uint64_t pol = policy_evict_last();
  const uint32_t s0 = row * g.tpr < g.NT ? row * g.tpr : g.NT;
  const uint32_t s1 = s0 + g.tpr < g.NT ? s0 + g.tpr : g.NT;
  const uint32_t n_tiles = s1 - s0;
  if (tid == 0) {
    for (uint32_t s = 0; s < S; ++s) mbar_init(&full[s], 1);
    mbar_fence_init();
  }
  fence_proxy_async();
  desc_fill<BLOCK>(dc, g, meta, s0, s1);
  __syncthreads();
  uint32_t dbase = 0;  // first row tile covered by the descriptor cache
  auto issue = [&](uint32_t stage, uint32_t t) {  // thread 0: the tile's bulk copy
    uint32_t phys, nvsg;
    if (t - dbase < kDescCap) { phys = dc.phys[t - dbase]; nvsg = dc.nvsg[t - dbase]; }
    else { const TileDesc d = geo_tile(g, meta, s0 + t); phys = d.phys; nvsg = d.nvalid | (d.seg << 16); }  // ahead of the cache
    s_nv[stage] = nvsg & 0xFFFFu;
    s_sg[stage] = nvsg >> 16;
    s_b0[stage] = seg_bin_lo[nvsg >> 16];
    s_b1[stage] = seg_bin_lo[(nvsg >> 16) + 1];
    mbar_expect_tx(&full[stage], kBytes);
    tma_load_1d(ring + (size_t)stage * kTile, bins16 + (size_t)phys * kTile, kBytes, &full[stage], pol);
  };
  if (tid == 0)
    for (uint32_t t = 0; t < S && t < n_tiles; ++t) issue(t, t);
  for (uint32_t i = tid; i <= max_nb; i += BLOCK) hist[i] = 0;
  __syncthreads();
  uint32_t* mrow = M + (size_t)row * Kp;
  uint32_t cur_sg = 0xFFFFFFFFu, cur_b0 = 0, cur_nb = 0;
  auto flush = [&]() {  // (uniform) the row leaves a partition: its histogram goes to M, the counters start over
    __syncthreads();
    for (uint32_t k = tid; k <= cur_nb; k += BLOCK) {  // slot cur_nb counted the removed players: dropped
      if (k < cur_nb) mrow[cur_b0 + k] = hist[k];
      hist[k] = 0;
    }
    __syncthreads();
  };
  // The ring is consumed half a turn at a time (4 tiles = up to 8 192 players between two CTA barriers) while the
  // other half's copies are in flight: the pass is latency-bound at this size, fewer and fatter steps win.
  for (uint32_t i = 0; i * H < n_tiles; ++i) {
    const uint32_t t0 = i * H, sb = (i & 1u) * H, parity = (i >> 1) & 1u;
    if (t0 >= dbase + kDescCap) {  // (uniform) next batch of descriptors; thread 0 is not issuing right now
      dbase = t0;
      desc_fill<BLOCK>(dc, g, meta, s0 + t0, s1);
      __syncthreads();
    }
    const uint32_t nt = n_tiles - t0 < H ? n_tiles - t0 : H;
    for (uint32_t k = 0; k < nt; ++k) {
      const uint16_t* tb = ring + (size_t)(sb + k) * kTile;
      mbar_wait(&full[sb + k], parity);
      if (s_sg[sb + k] != cur_sg) {
        if (cur_sg != 0xFFFFFFFFu) flush();
        cur_sg = s_sg[sb + k]; cur_b0 = s_b0[sb + k]; cur_nb = s_b1[sb + k] - cur_b0;
      }
      const uint32_t valid = s_nv[sb + k], b0 = cur_b0, nb = cur_nb;
      auto add = [&](uint32_t v) { const uint32_t d = v - b0; atomicAdd(&hist[d < nb ? d : nb], 1u); };  // slot nb: removed players
#pragma unroll
      for (uint32_t q = tid; q < kTile / 8; q += BLOCK) {  // 8 bins (128 bits) per thread per step
        const uint32_t o = q * 8;
        if (o + 8 <= valid) {
          const uint4 v = *reinterpret_cast<const uint4*>(tb + o);
          add(v.x & 0xFFFFu); add(v.x >> 16); add(v.y & 0xFFFFu); add(v.y >> 16);
          add(v.z & 0xFFFFu); add(v.z >> 16); add(v.w & 0xFFFFu); add(v.w >> 16);
        } else {
          for (uint32_t e = o; e < valid; ++e) add(tb[e]);
        }
      }
    }
    __syncthreads();
    if (tid == 0)
      for (uint32_t k = 0; k < H && t0 + S + k < n_tiles; ++k) issue(sb + k, t0 + S + k);
  }
  if (cur_sg != 0xFFFFFFFFu) flush();
  if (tid == 0)
    for (uint32_t s = 0; s < kHistStages; ++s) mbar_inval(&full[s]);
}

// ---------------------------------------------------------------------------------------
// rowsum_body<BLOCK>: the same M[row][bin] WITHOUT streaming the pool — when every partition has <= 255 keys the
// engine keeps a histogram per chunk current (PoolMeta::chist: +1 at ingest, -1 at remove / take, rebuilt for the
// compacted pool), so a row only adds up the histograms of its <= tiles-per-row chunks: ~1 KB per tile instead of the
// tile's 4 KB key column and no shared-memory atomics.  Thread k owns key k of the current partition.
// Shared memory: the tile descriptor cache only.
// ---------------------------------------------------------------------------------------
template <int BLOCK>
__device__ __forceinline__ void rowsum_body(unsigned char* smem_raw, const Geo& g, const PoolMeta meta, uint32_t Kp,
                                            const uint32_t* __restrict__ seg_bin_lo, uint32_t* __restrict__ M) {
  DescCache& dc = *reinterpret_cast<DescCache*>(smem_raw);
  const uint32_t tid = threadIdx.x, row = blockIdx.x;
  const uint32_t s0 = row * g.tpr < g.NT ? row * g.tpr : g.NT;
  const uint32_t s1 = s0 + g.tpr < g.NT ? s0 + g.tpr : g.NT;
  uint32_t* mrow = M + (size_t)row * Kp;
  uint32_t cur_sg = 0xFFFFFFFFu, acc = 0;
  for (uint32_t tb = s0; tb < s1; tb += kDescCap) {
    __syncthreads();
    desc_fill<BLOCK>(dc, g, meta, tb, s1);
    __syncthreads();
    const uint32_t nt = s1 - tb < kDescCap ? s1 - tb : kDescCap;
    constexpr uint32_t U = 8;  // loads in flight per thread: the histograms are cold in DRAM, one at a time serialises 17 round trips
    for (uint32_t t0 = 0; t0 < nt; t0 += U) {
      uint32_t v[U];
#pragma unroll
      for (uint32_t u = 0; u < U; ++u)
        v[u] = (t0 + u < nt && tid < kChunkHist) ? __ldcg(&meta.chist[(size_t)dc.phys[t0 + u] * kChunkHist + tid]) : 0u;
#pragma unroll
      for (uint32_t u = 0; u < U; ++u) {
        if (t0 + u >= nt) break;
        const uint32_t sg = dc.nvsg[t0 + u] >> 16;
        if (sg != cur_sg) {  // (uniform) the row leaves a partition: its sums go to M
          if (cur_sg != 0xFFFFFFFFu) {
            const uint32_t b0 = seg_bin_lo[cur_sg], nb = seg_bin_lo[cur_sg + 1] - b0;
            if (tid < nb) mrow[b0 + tid] = acc;
          }
          cur_sg = sg; acc = 0;
        }
        acc += v[u];
      }
    }
  }
  if (cur_sg != 0xFFFFFFFFu) {
    const uint32_t b0 = seg_bin_lo[cur_sg], nb = seg_bin_lo[cur_sg + 1] - b0;
    if (tid < nb) mrow[b0 + tid] = acc;
  }
  __syncthreads();
}

}  // namespace mm
