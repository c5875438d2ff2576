// mm_kernels.cuh — device code of the search tick (sm_90a).
//
// The tick replaces, for every queued player at once, the per-request loop of
// Search.Worker.consume/5 (reference matchmaking/lib/search/worker.ex:291-324).
// Under the serialized oracle (oracle/mm_oracle.c) that loop has the closed form
//   "drop inactive players, stable-partition the feed order by (mode, group), cut
//    each partition into lobbies of L".
// The resident pool is already partitioned by (mode, group) — the reference queues per rating group
// (search/worker.ex:46-66, generic/worker.ex:55-69) and selects partial lobbies by game mode
// (models/lobby_state.ex:72-79) — as per-partition chunk lists filled at ingest, so the tick is ONE stable counting
// sort by rating INSIDE every partition
//   bin(player) = mode * stride + lut[clamp(rating)]          (K bins, K ~ 5k * modes; ~K / partitions per tile)
// followed by the per-partition lobby cut.  One cooperative launch, k_tick<512>, runs the four phases
// (each also exists as a stand-alone kernel):
//   k_hist     row histograms M[row][bin]: sums of the resident per-chunk histograms (kept current by ingest / remove /
//              tick) when every partition has <= 255 keys, else from the 16-bit bin column (2 B/player, TMA ring)
//   k_colscan  the tail: per bin, how many players are matched (a prefix of the bin) and the member slot of the first
//              one — policy S0 (reference behaviour) or S1 (rating window, extension) — from the resident bin totals;
//              layout and bin totals of the compacted pool; column prefix of M only when a partition spans many rows
//   k_place    stable rank inside the row -> final lobby-major slot; tile-local counting sort staged in shared
//              memory, ids written to member_ids in whole sectors (reads 10 B/player, writes 8 B); players past
//              their bin's prefix: one bit in left_bits; then the row moves its own leftover players to the
//              compacted pool (enqueue order kept inside the partition; compact_row)
//   k_epilogue lobby headers
// Integer/HBM-bound work: no tensor cores (BASELINE.json north_star).
#pragma once
#include "mm_common.cuh"
#include "mm_hist.cuh"
#include "mm_scan.cuh"
#include "mm_place.cuh"
#include "mm_epilogue.cuh"
#include "mm_active.cuh"

namespace mm {

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, 2)
    k_hist(const uint16_t* __restrict__ bins16, const PoolMeta meta, uint32_t n_segs, uint32_t R, uint32_t Kp, uint32_t max_nb,
           const uint32_t* __restrict__ seg_bin_lo, uint32_t* __restrict__ M) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ Geo geo;
  __shared__ uint32_t s_gtmp[33];
  geo_build<BLOCK>(geo, meta.fill, n_segs, R, s_gtmp);
  if (meta.chist) rowsum_body<BLOCK>(smem_raw, geo, meta, Kp, seg_bin_lo, M);
  else hist_body<BLOCK>(smem_raw, geo, bins16, meta, Kp, max_nb, seg_bin_lo, M);
}

// placement + row compaction (the compacted pool's chunk histograms were cleared before the launch)
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, 2) k_place(const PlaceArgs a, const EpiArgs e, const uint32_t* __restrict__ fill,
                                                    uint32_t n_segs) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ Geo geo;
  __shared__ uint32_t s_gtmp[33];
  geo_build<BLOCK>(geo, fill, n_segs, a.R, s_gtmp);
  const uint32_t nres = place_body<BLOCK>(smem_raw, geo, a, [](uint32_t) {});
  compact_row<BLOCK>(reinterpret_cast<uint32_t*>(smem_raw), geo, a, e, nres, place_left_before(smem_raw, a), nullptr, 0u);
}

// ---------------------------------------------------------------------------------------
// k_tick<512>: the whole search tick in ONE cooperative launch ("fully matched in one
// launch", BASELINE.json).  G CTAs = R row CTAs + a few helper CTAs; the CTA's dynamic shared
// memory is re-used by every phase, the tile geometry is built once:
//   rows: histogram of their tiles      || helper 0: the tail (bin totals are resident, kept
//         (TMA ring of bin tiles)       ||   current by ingest / remove / the previous tick)         | barrier 1:
//   rows: placement prologue (descriptors, first bulk copies),              rows arrive before, each placement
//         ranking of each placement pipeline's first tile                   pipeline waits before its first slot bases
//   [only when a partition spans many rows: whole barrier 1, column scan of M by all CTAs            | barrier 1b]
//   rows: placement (TMA ring of bin/id tiles, tile sort, sector-complete stores), compaction of the
//         row's own leftovers, then lobby headers in chunks claimed by the rows that finish first
//                                       || helpers: clear the compacted pool's chunk histograms (clr_done)
//   [only when emission order was asked for: barrier 2, headers + emit_seq by all CTAs]
// ---------------------------------------------------------------------------------------
struct TickArgs {
  PoolView src;
  uint32_t R;      // row CTAs; the grid has R + helpers CTAs
  uint32_t* M;
  uint32_t* P;
  TailArgs tail;   // Kp, K, n_segs, src bin totals, segment tables, outbase / binlim, counters, src fill, dst meta
  PlaceArgs place;
  EpiArgs epi;
  TickCtr* next_ctr;  // the OTHER counter block (ticks alternate): re-armed by the last CTA so no memset precedes a launch
};

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, 2) k_tick(const TickArgs a) {
  static_assert(BLOCK == kScanBlock, "the column-scan phase is written for 512-thread CTAs");
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ Geo geo;
  __shared__ uint32_t s_gtmp[33];
  uint32_t* scratch = reinterpret_cast<uint32_t*>(smem_raw);
  const unsigned int G = gridDim.x;
  const uint32_t R = a.R, Kp = a.tail.Kp, K = a.tail.K;
  const bool is_row = blockIdx.x < R;
  const uint32_t helper = blockIdx.x - R, n_helpers = G - R;  // (helper valid when !is_row)
  TickCtr* ctr = a.tail.ctr;
  unsigned int bar = 0;
  auto stamp = [&](int k) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      ctr->t[k] = t;
    }
  };
  stamp(0);
  const bool tail_cta = blockIdx.x == G - 1;
  auto run_tail = [&]() {
    colscan_tail_body(scratch, a.tail);
    if (threadIdx.x == 0) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      ctr->t[5] = t;
    }
  };
  const bool tail_first = tail_cta && !is_row;
  if (tail_first) {  // the tail needs no tile geometry: it starts at once, beside the rows' pass, and signals the
    run_tail();      // barrier before it builds its own copy of the geometry (small ticks wait for the tail)
    grid_arrive(&ctr->gbar);
  }
  geo_build<BLOCK>(geo, a.place.meta.fill, a.tail.n_segs, R, s_gtmp);
  if (is_row) {
    if (a.place.meta.chist) rowsum_body<BLOCK>(smem_raw, geo, a.place.meta, Kp, a.tail.seg_bin_lo, a.M);
    else hist_body<BLOCK>(smem_raw, geo, a.src.bin, a.place.meta, Kp, a.place.max_nb, a.tail.seg_bin_lo, a.M);
  }
  if (tail_cta && is_row) run_tail();   // a grid without helpers: after its own row
  if (threadIdx.x == 0 && is_row) atomicMax(&ctr->t[8], global_ns());
  bar += G;
  // Barrier 1.  A row only arrives here: its placement prologue (descriptors, table zeroing, the first tiles' bulk
  // copies) and the ranking of each placement pipeline's first tile need nothing from the other CTAs and run before
  // the wait.  The column scan reads every row's M, so with it the barrier stays whole.  (uniform over the grid)
  const bool split_bar1 = is_row && !geo_use_colscan(geo);
  if (split_bar1) grid_arrive(&ctr->gbar);
  else if (tail_first) grid_wait(&ctr->gbar, bar);
  else grid_barrier(&ctr->gbar, bar);
  if (!split_bar1) {
    stamp(1);
    if (geo_use_colscan(geo)) {
      for (uint32_t grp = blockIdx.x; grp < (K + 31) / 32; grp += G) colscan_cols_body(scratch, geo, grp, Kp, K, a.tail.bin_seg, a.M, a.P);
      grid_barrier(&ctr->gbar, (bar += G));
    }
    stamp(2);
  }
  // the compacted pool's chunks start with empty histograms (the row compaction fills them): cleared by the helpers,
  // or by the rows when the grid has no helper; every clearing CTA then counts itself in clr_done
  const uint32_t n_clear = n_helpers ? n_helpers : G;
  auto clear_chist = [&]() {
    const uint32_t part = n_helpers ? helper : blockIdx.x;
    const size_t words = (size_t)__ldcg(a.epi.dst_meta.bump) * kChunkHist;
    for (size_t i = (size_t)part * BLOCK + threadIdx.x; i < words; i += (size_t)n_clear * BLOCK) a.epi.dst_meta.chist[i] = 0;
    grid_arrive(&ctr->clr_done);
  };
  if (a.epi.dst_meta.chist && !is_row) clear_chist();
  if (is_row) {
    const uint32_t nres = place_body<BLOCK>(smem_raw, geo, a.place, [&](uint32_t h) {
      if (split_bar1) { grid_wait_half(&ctr->gbar, bar, h); stamp(1); stamp(2); }
    });
    if (threadIdx.x == 0) atomicMax(&ctr->t[10], global_ns());
    if (a.epi.dst_meta.chist && n_helpers == 0) clear_chist();
    compact_row<BLOCK>(scratch, geo, a.place, a.epi, nres, place_left_before(smem_raw, a.place), &ctr->clr_done, n_clear);
    if (threadIdx.x == 0) atomicMax(&ctr->t[3], global_ns());
    if (!a.epi.write_headers) headers_claimed<BLOCK>(scratch, a.epi, &ctr->hdr_next);
  }
  if (a.epi.write_headers) {  // emission order: emit_seq reads the src_idx of every row, so barrier 2 stays
    grid_barrier(&ctr->gbar, (bar += G));
    epilogue_body<BLOCK>(scratch, geo, a.epi);
  }
  if (threadIdx.x == 0) {  // the last CTA to finish closes the epilogue phase
    unsigned long long tm;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(tm));
    atomicMax(&ctr->t[6], tm);
    __threadfence();
    if (atomicAdd(&ctr->done, 1u) == G - 1) {  // ... and arms the other counter block for the next tick
      TickCtr* nx = a.next_ctr;
      nx->gbar = 0; nx->done = 0; nx->chist_bad = 0; nx->hdr_next = 0; nx->left_bad = 0; nx->clr_done = 0;
      nx->t[3] = 0; nx->t[4] = 0; nx->t[6] = 0; nx->t[7] = 0; nx->t[8] = 0; nx->t[10] = 0;
      for (int i = 0; i < 8; ++i) nx->stall[i / 4][i % 4] = 0;
    }
  }
}

}  // namespace mm
