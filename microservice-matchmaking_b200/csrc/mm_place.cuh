// mm_place.cuh — phase 3 of the tick: stable rank inside the row -> final lobby-major slot of every player
#pragma once
#include "mm_common.cuh"

namespace mm {

// ---------------------------------------------------------------------------------------
// place_body<BLOCK>: the placement pass.  The row (= CTA) streams its tiles — 2 048 players of ONE (mode, group)
// partition each: (bin u16, id u64) chunks through a ring of TMA bulk copies (cp.async.bulk -> mbarrier),
// issued `stages` tiles ahead by one thread, L2 evict-first — computes every player's STABLE rank among the row's
// players of the same bin and stores the id to its final lobby-major slot
//     slot = outbase[bin] + (players of the bin in earlier rows: M) + rank inside the row.
// A player at or past binlim[bin] stays queued: one bit in left_bits (one ballot per 32 players, plain word stores).
//
// A pool with chunk histograms (every partition <= 255 keys) and rank_impl 3 takes place_halves: two tile pipelines
// per CTA whose slot bases come from the histograms, so no tile waits for another tile's ranking and no barrier spans
// the CTA (see there).  Otherwise (a partition with > 255 keys, or rank_impl 2) the whole CTA ranks one tile at a time
// and takes its slot bases from its own ranking; two ranking paths, chosen per tile (uniform for the CTA):
//  * FAST — the tile's partition has <= 255 bins (e.g. 5 001 rating values in 32 groups: 157): a one-pass 8-bit
//    counting sort of the tile in shared memory.  Warp w owns 128 consecutive tile positions; per 32 players the
//    peers with the same digit are found with <= 8 ballots (MATCH.ANY is a slow multi-pass warp instruction,
//    see tools/ubench/smem.cu), the lowest peer bumps the warp's private digit counter; 128 threads then scan the 16 x 256 counter
//    matrix (two 16-bit digits per word, packed adds) into tile-local sorted positions.  Ids are staged AT THEIR
//    SORTED POSITION in the tile's own ring stage together with their global slot, and the CTA writes the staged
//    tile back in sorted order: consecutive threads store consecutive slots of a bin's run (about 2048 / bins ids =
//    100+ contiguous bytes), so member_ids is written in whole 32-byte sectors instead of 8-byte fragments.
//  * LIST — larger key domains (one group of 5 001 rating values): one list node per player on a hashed,
//    epoch-tagged head table (shared-memory atomicExch), walk of the round-local list counting same-bin nodes with a
//    smaller tile position; ids are scattered straight from registers.  `heavy` ticks (some bin expects > 8
//    players per tile) aggregate the nodes per warp first (__match_any_sync) so a list never exceeds 64 nodes.
//
// Shared memory (whole CTA): ring_ids[stages][kTile] | ring_bins[stages][kTile] | mbarriers + tile descriptors |
//                cnt[keys of one partition] | union { LIST: head[kHeadSlots] node[kTile] nbin[kTile] ;
//                FAST: wmask[16][256], wcnt[16][256] u16, lgd[256], spd[kTile] }.
// Shared memory (two pipelines): ring_ids | ring_bins | ring_hist[stages][256] | mbarriers + tile descriptors | cnt |
//                2 x { wmask[8][256], wcnt[8][256] u16, lgd[256], spd[kTile] }.
// ---------------------------------------------------------------------------------------
constexpr uint32_t kHeadSlots = 4096;
constexpr uint32_t NW16 = 16;  // warps per 512-thread CTA
constexpr uint32_t kPlaceUnionBytes = NW16 * 256 * 4 + NW16 * 256 * 2 + 1024 + kTile * 4;  // FAST: 16 + 8 + 1 + 8 KB >= LIST: 28 KB

// max_nb = most sort keys any one partition has: the slot counters are kept per partition, not for the whole key domain
__host__ __device__ constexpr uint32_t place_cnt_cap(uint32_t max_nb) { return (max_nb > 1024u ? max_nb : 1024u); }
// Two tile pipelines per CTA (pools with chunk histograms): per pipeline wmask[8][256] u32 | wcnt[8][256] u16 |
// lgd[256] | spd[kTile]; every ring stage also carries the chunk's 1 KB histogram row.
constexpr uint32_t kHalfWarps = 8;
constexpr uint32_t kHalfBytes = kHalfWarps * 256 * 4 + kHalfWarps * 256 * 2 + 256 * 4 + kTile * 4;
constexpr uint32_t kHalvesHdr = 288;  // mbarriers, tile descriptors, flags, warp totals, stall counters
__host__ __device__ constexpr size_t place_smem_whole(uint32_t max_nb, uint32_t stages) {
  return (size_t)stages * kTileBytes + 128 + (size_t)((place_cnt_cap(max_nb) + 3) & ~3u) * 4 + kPlaceUnionBytes + sizeof(DescCache) + 16;
}
__host__ __device__ constexpr size_t place_smem_halves(uint32_t max_nb, uint32_t stages) {
  return (size_t)stages * (kTileBytes + kChunkHist * 4) + kHalvesHdr + (size_t)((place_cnt_cap(max_nb) + 3) & ~3u) * 4 +
         2 * kHalfBytes + sizeof(DescCache) + 16;
}
// max_nb <= kFastBins: the pool has chunk histograms and places on the two-pipeline path (or, with rank_impl = 2, on
// the whole-CTA path, whose layout fits in the same allocation)
__host__ __device__ constexpr size_t place_smem_bytes(uint32_t max_nb, uint32_t stages) {
  return max_nb <= kFastBins && place_smem_halves(max_nb, stages) > place_smem_whole(max_nb, stages)
             ? place_smem_halves(max_nb, stages)
             : place_smem_whole(max_nb, stages);
}

struct PlaceArgs {
  const uint16_t* bins16;
  const uint64_t* ids;
  PoolMeta meta;
  uint32_t K, Kp, R, stages, fast_ok, max_nb;
  const uint32_t* seg_bin_lo;
  const uint16_t* bin_seg;
  const uint32_t* M;     // [rows][Kp] row histograms (raw counts)
  const uint32_t* P;     // [rows][Kp] their column prefixes, only when the column-scan phase ran
  const uint32_t* outbase;
  const uint32_t* binlim;
  uint64_t* members;
  uint32_t* src_idx;    // optional: virtual pool position of every member (emission order in ARRIVAL mode)
  uint32_t* left_bits;  // one bit per virtual pool position: the player stays queued after this tick
  TickCtr* ctr;
  unsigned long long* trace;  // fused tick: TickCtr::t of the launch (first tile ranked / first slot bases taken); else null
};

// Shared memory of the two-pipeline placement (see the layout above); the row compaction after it reads the header.
constexpr uint32_t kLeftBeforeCap = 6;  // partitions of a row whose left_before the window loads keep (header words)
struct HalvesSmem {
  uint64_t* ring_ids;   // [S][kTile]
  uint16_t* ring_bins;  // [S][kTile]
  uint32_t* ring_hist;  // [S][kChunkHist]
  unsigned char* hdr;
  uint32_t* cnt;        // [cnt_cap]
  unsigned char* halves;
  DescCache* dc;
};
__device__ __forceinline__ HalvesSmem halves_smem(unsigned char* smem_raw, uint32_t S, uint32_t max_nb) {
  HalvesSmem m;
  m.ring_ids = reinterpret_cast<uint64_t*>(smem_raw);
  m.ring_bins = reinterpret_cast<uint16_t*>(smem_raw + (size_t)S * kTile * 8);
  m.ring_hist = reinterpret_cast<uint32_t*>(smem_raw + (size_t)S * kTileBytes);
  m.hdr = smem_raw + (size_t)S * (kTileBytes + kChunkHist * 4);
  m.cnt = reinterpret_cast<uint32_t*>(m.hdr + kHalvesHdr);
  m.halves = reinterpret_cast<unsigned char*>(m.cnt + ((place_cnt_cap(max_nb) + 3) & ~3u));
  m.dc = reinterpret_cast<DescCache*>(m.halves + 2 * kHalfBytes);
  return m;
}
// header words 66 .. 71: left_before(p0 + k), k < kLeftBeforeCap, of the row's partitions p0, p0 + 1, ...
__device__ __forceinline__ uint32_t* halves_left_before(unsigned char* hdr) { return reinterpret_cast<uint32_t*>(hdr + 264); }
static_assert(264 + 4 * kLeftBeforeCap <= kHalvesHdr, "left_before words fit in the placement header");
__device__ __forceinline__ bool place_on_halves(const PlaceArgs& a) { return a.meta.chist && a.fast_ok; }
// after place_body: the left_before words the two-pipeline placement left in shared memory, or null (whole-CTA path)
__device__ __forceinline__ const uint32_t* place_left_before(unsigned char* smem_raw, const PlaceArgs& a) {
  return place_on_halves(a) ? halves_left_before(halves_smem(smem_raw, a.stages, a.max_nb).hdr) : nullptr;
}

// place_halves<BLOCK>: the FAST ranking for a pool with chunk histograms (every partition <= 255 keys, rank_impl 3).
// The CTA runs two independent tile pipelines: half h (threads 256 h .. 256 h + 255, 8 warps, 8 players per thread)
// takes the row's tiles t = h, h + 2, ... and synchronises only on its own named barrier.  The halves share the ring
// and the row's running slot counters cnt[]; nothing waits for another tile's ranking:
//  * slot bases: the chunk's histogram row travels with the tile (third bulk copy into the stage).  Tile t takes
//    cnt[d] as the global slot of its first player of key d and advances cnt[d] by chist[d] — a 256-entry step,
//    passed from tile t-1 to tile t through the `hand` mbarrier (one phase per tile).  Tile-local first positions l0
//    are the exclusive scan of the same row.  Bit 31 of a slot base (some player of the (tile, key) cell is past the
//    key's matched prefix) comes from cnt[d] + chist[d] against binlim.
//  * ring: stage s has a `full` mbarrier (the three bulk copies) and an `empty` one (the 256 threads of the half that
//    wrote the tile back); thread 0 of that half waits on `empty` and issues the stage's next tile at once.
//  * per tile and half: rank (as below: match table / ballots, per-warp counters) | barrier | slot bases (hand) +
//    column scan of the 8 warps' counters + check of their totals against chist | barrier | stage the sorted order |
//    barrier | write back.
// A tile whose ranked key counts differ from its chunk histogram is not written at all and counted in
// TickCtr::chist_bad (the tick then fails): the slot bases of the row's later tiles rest on the histograms.
// The prologue (descriptors, table zeroing, the first tiles' bulk copies) and the ranking of a tile read only the pool
// being matched; the slot bases need the other CTAs' outputs.  So a tile ranks first and takes its bases after:
// `wait_inputs(h)`, called by the 256 threads of half h before its first slot bases, returns once the tail's outputs
// and every row's M are visible (the fused tick's grid barrier 1); it synchronises only the half.
// The window loads also sum left_before(p) (see compact_row) for the row's first kLeftBeforeCap partitions into the
// header (halves_left_before), where the row compaction reads them.
template <int BLOCK, class Wait>
__device__ __forceinline__ uint32_t place_halves(unsigned char* smem_raw, const Geo& g, const PlaceArgs a, Wait&& wait_inputs) {
  static_assert(BLOCK == 512 && kTile == 2048, "tile arrangement is written for 2 x 256 threads x 8 players");
  constexpr int J = 8;
  const uint32_t S = a.stages;
  const HalvesSmem m = halves_smem(smem_raw, S, a.max_nb);
  uint64_t* ring_ids = m.ring_ids;    // [S][kTile]
  uint16_t* ring_bins = m.ring_bins;  // [S][kTile]
  uint32_t* ring_hist = m.ring_hist;  // [S][kChunkHist]
  unsigned char* hdr = m.hdr;
  uint64_t* full = reinterpret_cast<uint64_t*>(hdr);  // [kMaxStages]
  uint64_t* empty = full + kMaxStages;                // [kMaxStages]
  uint64_t* hand = empty + kMaxStages;                // slot-base hand-off, one phase per tile
  uint32_t* s_nv = reinterpret_cast<uint32_t*>(hand + 1);  // [kMaxStages] valid players
  uint32_t* s_b0 = s_nv + kMaxStages;                      // [kMaxStages] first bin of the tile's partition
  uint32_t* s_b1 = s_b0 + kMaxStages;                      // [kMaxStages] its end bin
  uint32_t* s_sg = s_b1 + kMaxStages;                      // [kMaxStages] partition
  uint32_t* s_misc = s_sg + kMaxStages;  // [0] players of the row that stay queued, [1, 2] loaded counter window, [3 + h] tile flags of half h
  uint32_t* s_wt = s_misc + 8;           // [2][8] warp totals of the histogram-row scan
  uint32_t* s_ck = s_wt + 16;            // [2][4] stall counters of half h (cycles): hand, full, empty waits; loop
  uint32_t* s_lb = halves_left_before(hdr);  // [kLeftBeforeCap] left_before of the row's partitions p0, p0 + 1, ...
  uint32_t* cnt = m.cnt;  // [cnt_cap] slot of the next player of each window bin
  const uint32_t cnt_cap = place_cnt_cap(a.max_nb);
  unsigned char* halves = m.halves;
  DescCache& dc = *m.dc;

  const uint32_t tid = threadIdx.x, lane = tid & 31, h = tid >> 8, ht = tid & 255, hw = ht >> 5;
  const uint32_t lt_mask = (1u << lane) - 1u;
  uint32_t* wmask = reinterpret_cast<uint32_t*>(halves + h * kHalfBytes);  // [8][256] match masks (zero between items)
  uint16_t* wcnt = reinterpret_cast<uint16_t*>(wmask + kHalfWarps * 256);  // [8][256] per-warp digit counters
  uint32_t* lgd = reinterpret_cast<uint32_t*>(wcnt + kHalfWarps * 256);    // [256] (global slot base - l0) | flag
  uint32_t* spd = lgd + 256;                                                // [kTile] sorted pos -> tile pos | digit << 11
  const uint32_t row = blockIdx.x;
  const uint64_t pol_in = policy_evict_first();

  const uint32_t s0 = row * g.tpr < g.NT ? row * g.tpr : g.NT;
  const uint32_t s1 = s0 + g.tpr < g.NT ? s0 + g.tpr : g.NT;
  const uint32_t n_tiles = s1 - s0;

  auto issue = [&](uint32_t stage, uint32_t t) {  // descriptor + the tile's three bulk copies
    uint32_t phys, nvsg;
    if (t < kDescCap) { phys = dc.phys[t]; nvsg = dc.nvsg[t]; }
    else { const TileDesc d = geo_tile(g, a.meta, s0 + t); phys = d.phys; nvsg = d.nvalid | (d.seg << 16); }
    s_nv[stage] = nvsg & 0xFFFFu;
    s_sg[stage] = nvsg >> 16;
    s_b0[stage] = a.seg_bin_lo[nvsg >> 16];
    s_b1[stage] = a.seg_bin_lo[(nvsg >> 16) + 1];
    mbar_expect_tx(&full[stage], kTileBytes + kChunkHist * 4);
    tma_load_1d(ring_ids + (size_t)stage * kTile, a.ids + (size_t)phys * kTile, kTile * 8, &full[stage], pol_in);
    tma_load_1d(ring_bins + (size_t)stage * kTile, a.bins16 + (size_t)phys * kTile, kTile * 2, &full[stage], pol_in);
    tma_load_1d(ring_hist + (size_t)stage * kChunkHist, a.meta.chist + (size_t)phys * kChunkHist, kChunkHist * 4,
                &full[stage], pol_in);
  };

  if (tid == 0) {
    for (uint32_t s = 0; s < S; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 256); }
    mbar_init(hand, 256);
    mbar_fence_init();
    for (uint32_t i = 0; i < 8; ++i) { s_misc[i] = 0; s_ck[i] = 0; }
    for (uint32_t i = 0; i < kLeftBeforeCap; ++i) s_lb[i] = 0;
  }
  fence_proxy_async();
  desc_fill<BLOCK>(dc, g, a.meta, s0, s1);
  for (uint32_t i = tid; i < 2 * (kHalfWarps * 256 * 6 / 4); i += BLOCK) {  // both halves' match + counter tables
    const uint32_t hh = i / (kHalfWarps * 256 * 6 / 4), k = i % (kHalfWarps * 256 * 6 / 4);
    reinterpret_cast<uint32_t*>(halves + hh * kHalfBytes)[k] = 0;
  }
  __syncthreads();
  if (tid == 0)
    for (uint32_t t = 0; t < S && t < n_tiles; ++t) issue(t, t);

  uint32_t nleft = 0;  // lane 0: players of this warp's positions that stay queued
  const uint32_t row_p0 = n_tiles ? geo_seg_of(g, s0) : 0u;
  const uint32_t row_p_last = n_tiles ? geo_seg_of(g, s1 - 1) : 0u;
  const bool scanned = geo_use_colscan(g);  // the column-scan phase ran: P holds the row prefixes
  uint32_t* ck = s_ck + 4 * h;  // thread 0 of the half: stall counters, see TickCtr::stall
  if (ht == 0) ck[3] = (uint32_t)clock();
  for (uint32_t t = h; t < n_tiles; t += 2) {
    const uint32_t st = t % S, parity = (t / S) & 1u;
    const uint32_t vbase = (s0 + t) * kTile;  // virtual position of the tile's first player
    const uint16_t* tb = ring_bins + (size_t)st * kTile;
    const uint64_t* ti = ring_ids + (size_t)st * kTile;
    const uint32_t ck1 = (uint32_t)clock();
    mbar_wait(&full[st], parity);
    if (ht == 0) ck[1] += (uint32_t)clock() - ck1;
    const uint32_t valid = s_nv[st];
    const uint32_t bin0 = s_b0[st], nb = s_b1[st] - bin0;
    const uint32_t d = ht;  // this thread's key in the histogram-row steps
    const uint32_t ch = d < nb ? ring_hist[st * kChunkHist + d] : 0u;

    uint32_t incl = ch;  // inclusive scan of the histogram row inside the warp; the warp totals cross barrier A
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, incl, off);
      if (lane >= (uint32_t)off) incl += u;
    }
    if (lane == 31) s_wt[h * 8 + hw] = incl;

    // ---------------- rank inside the warp: warp hw owns tile positions 256 hw .. 256 hw + 255 ----------------
    uint32_t pk[J];  // digit | rank among the warp's players of the digit << 8
    {
      uint32_t* wm = wmask + hw * 256;
      uint16_t* wc = wcnt + hw * 256;
      uint32_t dg[J];
#pragma unroll
      for (int j = 0; j < J; ++j) {
        const uint32_t pos = hw * (32 * J) + j * 32 + lane;
        const uint32_t dd = (uint32_t)tb[pos] - bin0;  // digits 0 .. nb-1 live, nb = dead / past the tile's end
        dg[j] = (pos < valid && dd < nb) ? dd : nb;
      }
      const uint32_t lbit = 1u << lane;
      if (nb > 16) {
#pragma unroll
        for (int j = 0; j < J; ++j) {
          atomicOr(&wm[dg[j]], lbit);
          __syncwarp();
          const uint32_t peers = wm[dg[j]];
          const uint32_t cb = wc[dg[j]];
          __syncwarp();
          wm[dg[j]] = 0;
          wc[dg[j]] = (uint16_t)(cb + __popc(peers));
          __syncwarp();
          pk[j] = dg[j] | ((cb + __popc(peers & lt_mask)) << 8);
        }
      } else {  // a handful of keys (arrival order: one per partition): peers from <= 5 ballots
        const uint32_t nbits = 32u - __clz(nb);
#pragma unroll
        for (int j = 0; j < J; ++j) {
          uint32_t peers = 0xFFFFFFFFu;
#pragma unroll
          for (uint32_t bit = 0; bit < 5; ++bit)
            if (bit < nbits) {
              const bool on = (dg[j] >> bit) & 1u;
              const uint32_t bal = __ballot_sync(0xFFFFFFFFu, on);
              peers &= on ? bal : ~bal;
            }
          const uint32_t cb = wc[dg[j]];
          __syncwarp();
          wc[dg[j]] = (uint16_t)(cb + __popc(peers));
          __syncwarp();
          pk[j] = dg[j] | ((cb + __popc(peers & lt_mask)) << 8);
        }
      }
    }
    bar_sync_half(h);  // A: per-warp digit counts and histogram-row warp totals complete

    // ---------------- slot bases: the half's first tile waits for the other CTAs' outputs, every tile for t-1 ----------------
    if (t == h) {
      if (a.trace && tid == 0) atomicMax(&a.trace[4], global_ns());  // first tile ranked
      wait_inputs(h);
    }
    const uint32_t ck0 = (uint32_t)clock();
    if (t) mbar_wait(hand, (t - 1) & 1u);  // tile t-1 has taken its slot bases
    if (ht == 0) ck[0] += (uint32_t)clock() - ck0;
    const uint32_t lim = ch ? __ldcg(&a.binlim[bin0 + d]) : 0u;
    uint32_t wb = s_misc[1], we = s_misc[2];
    if (bin0 < wb || bin0 + nb > we) {
      // (uniform) the row enters a partition whose slot counters are not loaded: load a window of whole partitions
      // starting with this one (a row's tiles come in partition order; a row usually spans 1-3 partitions, which fit
      // at once).  cnt[b - wb] = slot of the (row, b) cell's first player.  Every partition of the row is loaded by
      // exactly one window, which also adds its bins' leftovers in earlier rows to left_before.
      wb = bin0; we = bin0 + nb;
      for (uint32_t p = s_sg[st] + 1; p <= row_p_last; ++p) {
        const uint32_t e = a.seg_bin_lo[p + 1];
        if (e - wb > cnt_cap) break;
        we = e;
      }
      for (uint32_t i = wb + ht; i < we; i += 256) {
        uint32_t rlo = 0, rhi = 0, v = 0;
        const uint32_t p = a.bin_seg[i];
        if (geo_rows_of(g, p, rlo, rhi) && row >= rlo && row <= rhi) {
          // __ldcg: these arrays are produced earlier in the same (fused) launch by other SMs
          uint32_t pre = 0;
          if (scanned) pre = __ldcg(&a.P[(size_t)row * a.Kp + i]);
          else
            for (uint32_t r = rlo; r < row; r += 8) {  // few rows per partition; 8 independent L2 loads in flight
              uint32_t v8[8];
#pragma unroll
              for (uint32_t u = 0; u < 8; ++u) v8[u] = r + u < row ? __ldcg(&a.M[(size_t)(r + u) * a.Kp + i]) : 0u;
#pragma unroll
              for (uint32_t u = 0; u < 8; ++u) pre += v8[u];
            }
          v = __ldcg(&a.outbase[i]) + pre;
          if (p - row_p0 < kLeftBeforeCap) {
            const uint32_t bl = __ldcg(&a.binlim[i]);
            if (v > bl) atomicAdd(&s_lb[p - row_p0], v - bl < pre ? v - bl : pre);
          }
        }
        cnt[i - wb] = v;
      }
      bar_sync_half(h);  // the window is loaded, and every thread of the half has read the old bounds
      if (ht == 0) { s_misc[1] = wb; s_misc[2] = we; }
    }
    uint32_t base = 0;  // global slot of the tile's first player of key d
    if (d < nb) { base = cnt[bin0 - wb + d]; cnt[bin0 - wb + d] = base + ch; }
    mbar_arrive(hand);  // tile t+1 may take its slot bases
    if (a.trace && t == 0 && tid == 0) atomicMax(&a.trace[7], global_ns());  // first slot bases taken

    uint32_t n_live = 0, l0 = 0;
#pragma unroll
    for (uint32_t w = 0; w < kHalfWarps; ++w) {
      const uint32_t v = s_wt[h * 8 + w];
      if (w < hw) l0 += v;
      n_live += v;
    }
    l0 += incl - ch;  // tile-local sorted position of the first player of key d
    uint32_t run = l0;
#pragma unroll
    for (uint32_t w = 0; w < kHalfWarps; ++w) {  // column scan: warp w's first sorted position of key d
      const uint32_t c = wcnt[w * 256 + d];
      wcnt[w * 256 + d] = (uint16_t)run;
      run += c;
    }
    const bool bad = d < nb && run - l0 != ch;  // the ranked count of key d differs from the chunk histogram
    const bool fl = ch != 0 && base + ch > lim;  // some player of the cell is past the key's matched prefix
    if (d < nb) lgd[d] = ((base - l0) & 0x7FFFFFFFu) | (fl ? 0x80000000u : 0u);
    if (fl || bad) atomicOr(&s_misc[3 + h], (fl ? 1u : 0u) | (bad ? 2u : 0u));
    bar_sync_half(h);  // B: run bases, slot bases and tile flags are complete

    const uint32_t tf = s_misc[3 + h];  // (uniform over the half)
    uint32_t lmask = 0;  // bit j: my j-th player stays queued
    if (!(tf & 2u)) {
#pragma unroll
      for (int j = 0; j < J; ++j) {
        const uint32_t dj = pk[j] & 0xFFu;
        if (dj < nb) {
          const uint32_t pos = hw * (32 * J) + j * 32 + lane;
          const uint32_t lpos = wcnt[hw * 256 + dj] + (pk[j] >> 8);
          bool matched = true;
          if ((tf & 1u) || a.src_idx) {
            const uint32_t e = lgd[dj];
            const uint32_t slot = (e + lpos) & 0x7FFFFFFFu;
            if (e >> 31) matched = slot < __ldcg(&a.binlim[bin0 + dj]);
            if (matched && a.src_idx) a.src_idx[slot] = vbase + pos;
          }
          // sorted position -> (tile position, digit); 255 = stays queued.  The ids stay where the TMA put them.
          spd[lpos] = pos | ((matched ? dj : 255u) << 11);
          if (!matched) lmask |= 1u << j;
        }
      }
    }
    {  // left_bits: the warp owns 256 consecutive positions = 8 words; lane j stores word j
      uint32_t mine = 0, all = 0;
      if (tf & 1u) {
#pragma unroll
        for (int j = 0; j < J; ++j) {
          const uint32_t wv = __ballot_sync(0xFFFFFFFFu, (lmask >> j) & 1u);
          if (lane == (uint32_t)j) mine = wv;
          all += __popc(wv);
        }
      }
      if (lane < (uint32_t)J) a.left_bits[(vbase >> 5) + hw * J + lane] = mine;
      if (lane == 0) nleft += all;
    }
    __syncwarp();  // the warp's counter row is read: all-zero again for the half's next tile (only this warp uses it)
    reinterpret_cast<uint4*>(wcnt + hw * 256)[lane] = make_uint4(0, 0, 0, 0);
    bar_sync_half(h);  // C: the sorted order of the tile is staged
    if (ht == 0) {
      s_misc[3 + h] = 0;
      if (tf & 2u) atomicAdd(&a.ctr->chist_bad, 1u);
    }
    if (!(tf & 2u)) {
#pragma unroll
      for (int i = 0; i < J; ++i) {
        const uint32_t k = i * 256 + ht;
        if (k < n_live) {
          const uint32_t v = spd[k], dk = v >> 11;
          if (dk != 255u) a.members[(lgd[dk] + k) & 0x7FFFFFFFu] = ti[v & 0x7FFu];
        }
      }
    }
    mbar_arrive(&empty[st]);  // this half is done with stage st
    if (ht == 0 && t + S < n_tiles) {
      const uint32_t ck2 = (uint32_t)clock();
      mbar_wait(&empty[st], parity);
      ck[2] += (uint32_t)clock() - ck2;
      issue(st, t + S);
    }
  }
  if (ht == 0) {
    ck[3] = (uint32_t)clock() - ck[3];
    for (uint32_t k = 0; k < 4; ++k) atomicAdd(&a.ctr->stall[h][k], (unsigned long long)ck[k]);
  }
  if (h == 0 && n_tiles == 0) wait_inputs(0u);  // a row without tiles still leaves with the inputs visible

  if (lane == 0 && nleft) atomicAdd(&s_misc[0], nleft);
  __syncthreads();
  const uint32_t n_res = s_misc[0];  // players of this row that stay queued
  if (tid == 0) {
    for (uint32_t s = 0; s < S; ++s) { mbar_inval(&full[s]); mbar_inval(&empty[s]); }
    mbar_inval(hand);
  }
  return n_res;
}

// wait_inputs(h): see place_halves (this path calls it for both halves at once, before its first tile)
template <int BLOCK, class Wait>
__device__ __forceinline__ uint32_t place_body(unsigned char* smem_raw, const Geo& g, const PlaceArgs a, Wait&& wait_inputs) {
  static_assert(BLOCK == 512 && kTile == 2048, "tile arrangement is written for 512 threads x 4 players");
  if (place_on_halves(a)) {  // (uniform) every partition has <= 255 keys
    return place_halves<BLOCK>(smem_raw, g, a, wait_inputs);
  }
  constexpr int J = kTile / BLOCK;
  constexpr int NW = BLOCK / 32;
  const uint32_t stages = a.stages, K = a.K, Kp = a.Kp;
  uint64_t* ring_ids = reinterpret_cast<uint64_t*>(smem_raw);                               // [stages][kTile]
  uint16_t* ring_bins = reinterpret_cast<uint16_t*>(smem_raw + (size_t)stages * kTile * 8);  // [stages][kTile]
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + (size_t)stages * kTileBytes);      // [kMaxStages]
  uint32_t* s_nv = reinterpret_cast<uint32_t*>(smem_raw + (size_t)stages * kTileBytes + 32); // [kMaxStages] valid players
  uint32_t* s_sg = s_nv + kMaxStages;                                                        // [kMaxStages] partition
  uint32_t* s_b0 = s_sg + kMaxStages;                                                        // [kMaxStages] its first bin
  uint32_t* s_b1 = s_b0 + kMaxStages;                                                        // [kMaxStages] its end bin
  uint32_t* s_misc = s_b1 + kMaxStages;                                                      // [8]
  uint32_t* cnt = reinterpret_cast<uint32_t*>(smem_raw + (size_t)stages * kTileBytes + 128); // [max_nb] of the current partition
  const uint32_t cnt_cap = place_cnt_cap(a.max_nb);
  unsigned char* uni = reinterpret_cast<unsigned char*>(cnt + ((cnt_cap + 3) & ~3u));
  DescCache& dc = *reinterpret_cast<DescCache*>(uni + kPlaceUnionBytes);
  // LIST
  uint32_t* head = reinterpret_cast<uint32_t*>(uni);           // [kHeadSlots]
  uint32_t* node = head + kHeadSlots;                          // [kTile]
  uint16_t* nbin = reinterpret_cast<uint16_t*>(node + kTile);  // [kTile] heavy path: bin of a group node
  // FAST
  uint32_t* wmask = reinterpret_cast<uint32_t*>(uni);          // [NW][256] per-warp match masks (all-zero between items)
  uint16_t* wcnt = reinterpret_cast<uint16_t*>(wmask + NW * 256);  // [NW][256] per-warp running digit counters
  uint32_t* wcnt32 = reinterpret_cast<uint32_t*>(wcnt);        // the same, two digits per word: [NW][128]
  uint32_t* lgd = wcnt32 + NW * 128;                           // [256] (global slot base - tile-local base) | flag
  uint32_t* spd = lgd + 256;                                   // [kTile] sorted position -> tile position | digit << 11

  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t lt_mask = (1u << lane) - 1u;
  const uint32_t row = blockIdx.x;
  const uint64_t pol_in = policy_evict_first();

  const uint32_t s0 = row * g.tpr < g.NT ? row * g.tpr : g.NT;
  const uint32_t s1 = s0 + g.tpr < g.NT ? s0 + g.tpr : g.NT;
  const uint32_t n_tiles = s1 - s0;

  uint32_t dbase = 0;  // first row tile covered by the descriptor cache
  auto issue = [&](uint32_t stage, uint32_t t) {  // thread 0: descriptor + the tile's two bulk copies
    uint32_t phys, nvsg;
    if (t - dbase < kDescCap) { phys = dc.phys[t - dbase]; nvsg = dc.nvsg[t - dbase]; }
    else { const TileDesc d = geo_tile(g, a.meta, s0 + t); phys = d.phys; nvsg = d.nvalid | (d.seg << 16); }
    s_nv[stage] = nvsg & 0xFFFFu;
    s_sg[stage] = nvsg >> 16;
    s_b0[stage] = a.seg_bin_lo[nvsg >> 16];
    s_b1[stage] = a.seg_bin_lo[(nvsg >> 16) + 1];
    mbar_expect_tx(&full[stage], kTileBytes);
    tma_load_1d(ring_ids + (size_t)stage * kTile, a.ids + (size_t)phys * kTile, kTile * 8, &full[stage], pol_in);
    tma_load_1d(ring_bins + (size_t)stage * kTile, a.bins16 + (size_t)phys * kTile, kTile * 2, &full[stage], pol_in);
  };

  if (tid == 0) {
    for (uint32_t s = 0; s < stages; ++s) mbar_init(&full[s], 1);
    mbar_fence_init();
    s_misc[0] = 0;  // players of the row that stay queued
    s_misc[2] = 0;  // FAST: the current tile has players past their bin's matched prefix
  }
  fence_proxy_async();
  desc_fill<BLOCK>(dc, g, a.meta, s0, s1);
  __syncthreads();
  if (tid == 0)
    for (uint32_t t = 0; t < stages && t < n_tiles; ++t) issue(t, t);
  for (uint32_t i = tid; i < kHeadSlots + NW * 128; i += BLOCK) head[i] = 0;  // LIST heads = FAST mask table; + FAST counters
  wait_inputs(tid >> 8);
  const bool heavy = __ldcg(&a.ctr->heavy) != 0;  // (written by the tail)
  __syncthreads();

  uint32_t st = 0, parity = 0;
  uint32_t nleft = 0;  // lane 0: players of this warp's positions that stay queued
  uint32_t wb = 0, we = 0;  // [wb, we): bins whose slot counters are loaded
  const uint32_t row_p_last = n_tiles ? geo_seg_of(g, s1 - 1) : 0u;
  uint32_t uni_st = 0;  // (uniform) who dirtied the union region: 0 nobody (all-zero), 1 LIST, 2 FAST
  for (uint32_t t = 0; t < n_tiles; ++t) {
    if (t == dbase + kDescCap) {  // (uniform) next batch of descriptors; thread 0 is not issuing right now
      dbase = t;
      desc_fill<BLOCK>(dc, g, a.meta, s0 + t, s1);
      __syncthreads();
    }
    const uint32_t vbase = (s0 + t) * kTile;  // virtual position of the tile's first player
    uint16_t* tb = ring_bins + (size_t)st * kTile;
    uint64_t* ti = ring_ids + (size_t)st * kTile;
    mbar_wait(&full[st], parity);
    const uint32_t valid = s_nv[st];
    const uint32_t bin0 = s_b0[st], nb = s_b1[st] - bin0;
    if (bin0 < wb || bin0 + nb > we) {
      // (uniform) the row enters a partition whose slot counters are not loaded: load a window of whole partitions
      // starting with this one (a row's tiles come in partition order; a row usually spans 1-3 partitions, which fit
      // at once).  cnt[b - wb] = slot of the (row, b) cell's first player; bit 31 flags a cell that reaches past
      // the bin's matched prefix (only those players look at binlim).
      wb = bin0; we = bin0 + nb;
      for (uint32_t p = s_sg[st] + 1; p <= row_p_last; ++p) {
        const uint32_t e = a.seg_bin_lo[p + 1];
        if (e - wb > cnt_cap) break;
        we = e;
      }
      const bool scanned = geo_use_colscan(g);  // the column-scan phase ran: P holds the row prefixes
      __syncthreads();
      for (uint32_t i = wb + tid; i < we; i += BLOCK) {
        uint32_t rlo = 0, rhi = 0, v = 0;
        if (geo_rows_of(g, a.bin_seg[i], rlo, rhi) && row >= rlo && row <= rhi) {
          // __ldcg: these arrays are produced earlier in the same (fused) launch by other SMs
          uint32_t pre = 0;
          if (scanned) pre = __ldcg(&a.P[(size_t)row * Kp + i]);
          else
            for (uint32_t r = rlo; r < row; r += 8) {  // few rows per partition; 8 independent L2 loads in flight
              uint32_t v[8];
#pragma unroll
              for (uint32_t u = 0; u < 8; ++u) v[u] = r + u < row ? __ldcg(&a.M[(size_t)(r + u) * Kp + i]) : 0u;
#pragma unroll
              for (uint32_t u = 0; u < 8; ++u) pre += v[u];
            }
          const uint32_t c = __ldcg(&a.M[(size_t)row * Kp + i]);
          const uint32_t start = __ldcg(&a.outbase[i]) + pre;
          v = start | ((start + c > __ldcg(&a.binlim[i])) ? 0x80000000u : 0u);
        }
        cnt[i - wb] = v;
      }
      __syncthreads();
    }
    uint32_t* cntp = cnt + (bin0 - wb);  // counters of this tile's partition
    const bool fast = a.fast_ok && nb <= kFastBins;
    uint32_t lmask = 0;  // bit j: my j-th player stays queued

    if (fast) {
      // ---------------- FAST: 8-bit counting sort of the tile in shared memory ----------------
      if (uni_st == 1) {  // the LIST path left head[] entries in the mask / counter tables
        for (uint32_t i = tid; i < NW * 256; i += BLOCK) wmask[i] = 0;
        for (uint32_t i = tid; i < NW * 128; i += BLOCK) wcnt32[i] = 0;
      }
      uint32_t dg[J], rk[J];
#pragma unroll
      for (int j = 0; j < J; ++j) {  // warp-striped: position = warp * 128 + j * 32 + lane
        const uint32_t pos = warp * (32 * J) + j * 32 + lane;
        const uint32_t d = (uint32_t)tb[pos] - bin0;  // digits 0 .. nb-1 live, nb = dead / past the tile's end
        dg[j] = (pos < valid && d < nb) ? d : nb;
      }
      if (uni_st == 1) __syncthreads();  // (uniform) the tables were just re-zeroed
      uni_st = 2;
      {   // the counter table is all-zero here (previous tile / prologue), the mask table always is between items
        // Peers of the same digit among the warp's 32 players: every lane ORs its bit into the warp's mask table
        // (shared-memory RED), reads the word back — that IS the match mask — and the peers reset the word
        // and bump the warp's running digit counter.  3 shared-memory instructions per 32 players instead of 8
        // ballots + selects (MATCH.ANY is a slow multi-pass warp instruction).
        uint32_t* wm = wmask + warp * 256;
        uint16_t* wc = wcnt + warp * 256;
        const uint32_t lbit = 1u << lane;
        if (nb > 16) {
#pragma unroll
          for (int j = 0; j < J; ++j) {
            atomicOr(&wm[dg[j]], lbit);
            __syncwarp();
            const uint32_t peers = wm[dg[j]];
            const uint32_t base = wc[dg[j]];
            __syncwarp();
            wm[dg[j]] = 0;                                    // every peer stores the same values: no leader election,
            wc[dg[j]] = (uint16_t)(base + __popc(peers));     // no divergence
            __syncwarp();
            rk[j] = base + __popc(peers & lt_mask);
          }
        } else {
          // a handful of keys (arrival order: ONE per partition): the 32 lanes would serialise on a few mask words,
          // so the peers come from <= 5 ballots instead
          const uint32_t nbits = 32u - __clz(nb);
#pragma unroll
          for (int j = 0; j < J; ++j) {
            uint32_t peers = 0xFFFFFFFFu;
#pragma unroll
            for (uint32_t bit = 0; bit < 5; ++bit)
              if (bit < nbits) {
                const bool on = (dg[j] >> bit) & 1u;
                const uint32_t bal = __ballot_sync(0xFFFFFFFFu, on);
                peers &= on ? bal : ~bal;
              }
            const uint32_t base = wc[dg[j]];
            __syncwarp();
            wc[dg[j]] = (uint16_t)(base + __popc(peers));
            __syncwarp();
            rk[j] = base + __popc(peers & lt_mask);
          }
        }
      }
      __syncthreads();  // B2: per-warp digit counts complete
      if (tid < 128) {
        // digits 2*tid, 2*tid+1: column scan over the 16 warps (packed 16-bit adds), exclusive scan over the digits,
        // global slot base from the row's running bin counters
        uint32_t v[NW], sum = 0;
#pragma unroll
        for (int w = 0; w < NW; ++w) { v[w] = wcnt32[w * 128 + tid]; sum += v[w]; }
        const uint32_t lo = sum & 0xFFFFu, hi = sum >> 16, both = lo + hi;
        uint32_t incl = both;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
          const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, incl, off);
          if (lane >= (uint32_t)off) incl += u;
        }
        if (lane == 31) s_misc[4 + warp] = incl;
        bar_sync_named(128);
        uint32_t wbase = 0;
        for (uint32_t w = 0; w < warp; ++w) wbase += s_misc[4 + w];
        const uint32_t l0 = wbase + incl - both, l1 = l0 + lo;  // tile-local sorted position of the digits' first players
        const uint32_t d0 = 2 * tid, d1 = d0 + 1;
        uint32_t fl = 0;
        if (d0 < nb) { const uint32_t base = cntp[d0]; cntp[d0] = base + lo; lgd[d0] = (((base & 0x7FFFFFFFu) - l0) & 0x7FFFFFFFu) | (base & 0x80000000u); if (lo) fl |= base; }
        if (d1 < nb) { const uint32_t base = cntp[d1]; cntp[d1] = base + hi; lgd[d1] = (((base & 0x7FFFFFFFu) - l1) & 0x7FFFFFFFu) | (base & 0x80000000u); if (hi) fl |= base; }
        if (fl >> 31) s_misc[2] = 1;   // some player of this tile sits in a cell that reaches past its bin's matched prefix
        if (d0 == nb) s_misc[1] = l0;  // live players of the tile (the dead digit sorts last)
        if (d1 == nb) s_misc[1] = l1;
        uint32_t run = l0 | (l1 << 16);
#pragma unroll
        for (int w = 0; w < NW; ++w) { wcnt32[w * 128 + tid] = run; run += v[w]; }
      }
      __syncthreads();  // B3: wcnt[w][d] = tile-local sorted position of warp w's first player of digit d
      const bool anyf = s_misc[2] != 0;  // (uniform)
#pragma unroll
      for (int j = 0; j < J; ++j) {
        if (dg[j] < nb) {
          const uint32_t lpos = wcnt[warp * 256 + dg[j]] + rk[j];
          bool matched = true;
          if (anyf || a.src_idx) {
            const uint32_t e = lgd[dg[j]];
            const uint32_t slot = (e + lpos) & 0x7FFFFFFFu;
            if (e >> 31) matched = slot < __ldcg(&a.binlim[bin0 + dg[j]]);
            if (matched && a.src_idx) a.src_idx[slot] = vbase + warp * (32 * J) + j * 32 + lane;
          }
          // sorted position -> (tile position, digit); 255 = stays queued.  The ids stay where the TMA put them.
          spd[lpos] = (warp * (32 * J) + j * 32 + lane) | ((matched ? dg[j] : 255u) << 11);
          if (!matched) lmask |= 1u << j;
        }
      }
      {  // left_bits: the warp owns 128 consecutive positions = 4 words; lane j stores word j
        uint32_t mine = 0, all = 0;
        if (anyf) {
#pragma unroll
          for (int j = 0; j < J; ++j) {
            const uint32_t wv = __ballot_sync(0xFFFFFFFFu, (lmask >> j) & 1u);
            if (lane == (uint32_t)j) mine = wv;
            all += __popc(wv);
          }
        }
        if (lane < (uint32_t)J) a.left_bits[(vbase >> 5) + warp * J + lane] = mine;
        if (lane == 0) nleft += all;
      }
      __syncthreads();  // B4: the sorted order of the tile is staged
      {
        const uint32_t n_live = s_misc[1];
#pragma unroll
        for (int i = 0; i < J; ++i) {
          const uint32_t k = i * BLOCK + tid;
          if (k < n_live) {
            const uint32_t v = spd[k], d = v >> 11;
            if (d != 255u) a.members[(lgd[d] + k) & 0x7FFFFFFFu] = ti[v & 0x7FFu];
          }
        }
        reinterpret_cast<uint4*>(wcnt32)[tid] = make_uint4(0, 0, 0, 0);  // counter table all-zero again (8 KB = 512 x 16 B)
        if (tid == 0) s_misc[2] = 0;
      }
    } else {
      // ---------------- LIST: hashed per-bin lists, ids scattered from registers ----------------
      if (uni_st == 2) {  // the FAST path left counters / slot bases in the head table
        for (uint32_t i = tid; i < kHeadSlots; i += BLOCK) head[i] = 0;
        __syncthreads();
      }
      uni_st = 1;
      const uint32_t epoch = t + 1;
      uint32_t bin[J], slot[J];
      uint64_t idv[J];
      bool flag[J];
#pragma unroll
      for (int j = 0; j < J; ++j) {  // strided: position = j * BLOCK + tid
        const uint32_t pos = j * BLOCK + tid;
        bin[j] = (pos < valid) ? (uint32_t)tb[pos] : 0xFFFFu;
        slot[j] = 0; flag[j] = false;
      }
      if (!heavy) {
        uint32_t snap[J];
#pragma unroll
        for (int j = 0; j < J; ++j) {
          const uint32_t pos = j * BLOCK + tid;
          snap[j] = 0;
          if (bin[j] < K) {
            snap[j] = cntp[bin[j] - bin0];
            const uint32_t prev = atomicExch(&head[bin[j] & (kHeadSlots - 1)], (epoch << 12) | pos);
            const uint32_t pn = ((prev >> 12) == epoch) ? (prev & 0xFFFu) : 0xFFFu;
            node[pos] = pn | (bin[j] << 12);
          }
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < J; ++j) idv[j] = ti[j * BLOCK + tid];  // ids early: their latency hides behind the walks
#pragma unroll
        for (int j = 0; j < J; ++j) {
          const uint32_t pos = j * BLOCK + tid;
          if (bin[j] < K) {
            uint32_t cur = head[bin[j] & (kHeadSlots - 1)] & 0xFFFu, lower = 0, total = 0;
            while (cur != 0xFFFu) {
              const uint32_t nd = node[cur];
              if ((nd >> 12) == bin[j]) {  // the slot is shared by bins congruent mod kHeadSlots
                ++total;
                lower += (cur < pos) ? 1u : 0u;
              }
              cur = nd & 0xFFFu;
            }
            slot[j] = (snap[j] & 0x7FFFFFFFu) + lower;
            flag[j] = (snap[j] >> 31) != 0;
            if (lower == 0) cntp[bin[j] - bin0] = snap[j] + total;  // the bin's earliest player of the tile
          }
        }
      } else {
        uint32_t snap[J], leader[J], rankw[J];
        bool isl[J];
#pragma unroll
        for (int j = 0; j < J; ++j) {
          const uint32_t pos = j * BLOCK + tid;
          const uint32_t mask = __match_any_sync(0xFFFFFFFFu, bin[j]);
          leader[j] = __ffs(mask) - 1;
          rankw[j] = __popc(mask & lt_mask);
          isl[j] = (lane == leader[j]) && (bin[j] < K);
          snap[j] = 0;
          if (isl[j]) {
            snap[j] = cntp[bin[j] - bin0];
            const uint32_t prev = atomicExch(&head[bin[j] & (kHeadSlots - 1)], (epoch << 12) | pos);
            const uint32_t pn = ((prev >> 12) == epoch) ? (prev & 0xFFFu) : 0xFFFu;
            node[pos] = pn | ((uint32_t)__popc(mask) << 12);
            nbin[pos] = (uint16_t)bin[j];
          }
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < J; ++j) {
          const uint32_t pos = j * BLOCK + tid;
          uint32_t bg = 0;
          if (isl[j]) {
            uint32_t cur = head[bin[j] & (kHeadSlots - 1)] & 0xFFFu, lower = 0, total = 0;
            while (cur != 0xFFFu) {
              const uint32_t nd = node[cur];
              if (nbin[cur] == bin[j]) {
                const uint32_t c = nd >> 12;
                total += c;
                if (cur < pos) lower += c;
              }
              cur = nd & 0xFFFu;
            }
            bg = snap[j] + lower;
            if (lower == 0) cntp[bin[j] - bin0] = snap[j] + total;
          }
          bg = __shfl_sync(0xFFFFFFFFu, bg, leader[j]);
          slot[j] = (bg & 0x7FFFFFFFu) + rankw[j];
          flag[j] = (bg >> 31) != 0;
        }
#pragma unroll
        for (int j = 0; j < J; ++j) idv[j] = ti[j * BLOCK + tid];
      }
#pragma unroll
      for (int j = 0; j < J; ++j) {
        if (bin[j] < K) {
          bool matched = true;
          if (flag[j]) matched = slot[j] < __ldcg(&a.binlim[bin[j]]);
          if (matched) {
            a.members[slot[j]] = idv[j];
            if (a.src_idx) a.src_idx[slot[j]] = vbase + j * BLOCK + tid;
          } else {
            lmask |= 1u << j;
          }
        }
      }
      {  // strided: batch j of the warp = positions j*BLOCK + 32*warp .. +31 = one word; lane j stores batch j's word
        uint32_t mine = 0, all = 0;
#pragma unroll
        for (int j = 0; j < J; ++j) {
          const uint32_t wv = __ballot_sync(0xFFFFFFFFu, (lmask >> j) & 1u);
          if (lane == (uint32_t)j) mine = wv;
          all += __popc(wv);
        }
        if (lane < (uint32_t)J) a.left_bits[(vbase + lane * BLOCK + warp * 32) >> 5] = mine;
        if (lane == 0) nleft += all;
      }
    }
    __syncthreads();  // everyone is done with stage st and with this tile's ranking state
    if (tid == 0 && t + stages < n_tiles) issue(st, t + stages);
    if (++st == stages) { st = 0; parity ^= 1u; }
  }

  if (lane == 0 && nleft) atomicAdd(&s_misc[0], nleft);
  __syncthreads();
  const uint32_t n_res = s_misc[0];  // players of this row that stay queued
  if (tid == 0)
    for (uint32_t s = 0; s < stages; ++s) mbar_inval(&full[s]);
  return n_res;
}

}  // namespace mm
