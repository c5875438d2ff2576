// mm_scan.cuh — phase 2 of the tick: column scan of the histogram matrix + the tail (matched prefix per bin, policies S0 / S1)
#pragma once
#include "mm_common.cuh"

namespace mm {

// ---------------------------------------------------------------------------------------
// k_colscan: exclusive prefix down every column of M.  A column CTA is 32 bins wide
// (lanes = consecutive bins, coalesced) and 16 row-slices deep (warps): every thread sums
// its slice of rows, the slices are scanned through shared memory, then the slice is
// rewritten as running prefixes — one round trip of latency instead of R.
// The LAST CTA of the grid runs concurrently as the "tail": bin totals (accumulated by
// k_hist with global reductions) -> sorted position of every bin -> how many players of every
// bin are matched under the tick's policy (always a PREFIX of the bin in enqueue order) ->
//   outbase[v] = member slot of bin v's first player (exclusive scan of the matched counts)
//   binlim[v]  = outbase[v] + matched players of bin v; a player at or past it stays queued.
// ---------------------------------------------------------------------------------------
constexpr int kScanBlock = 512;
constexpr uint32_t kColScratchWords = (kScanBlock / 32) * 33;      // column CTA scratch
constexpr uint32_t kTailScratchWords = 64 + 4 + 9 * kMaxSegs + 12;  // tail CTA scratch, fixed part

// One 32-bin column group: exclusive prefix down the rows of M (scratch: kColScratchWords).  Bin b belongs to one
// partition, and only the rows holding that partition's tiles wrote M[.][b] (mm_hist.cuh): the scan of a column is
// confined to rows [rlo, rhi] of its partition — about R / partitions rows instead of R.  The prefixes go to P; M
// keeps the raw counts (a row's own count is M[row][b]).  Only run when geo_use_colscan(g): otherwise every row sums
// the few rows before it by itself (mm_place.cuh).
__device__ __forceinline__ void colscan_cols_body(uint32_t* scratch, const Geo& g, uint32_t group, uint32_t Kp, uint32_t K,
                                                  const uint16_t* __restrict__ bin_seg, const uint32_t* __restrict__ M,
                                                  uint32_t* __restrict__ P) {
  uint32_t(*s_part)[33] = reinterpret_cast<uint32_t(*)[33]>(scratch);
  const uint32_t tid = threadIdx.x, x = tid & 31, y = tid >> 5;
  constexpr uint32_t NY = kScanBlock / 32;
  const uint32_t b = group * 32 + x;
  uint32_t rlo = 0, rhi = 0;
  const bool on = b < K && geo_rows_of(g, bin_seg[b], rlo, rhi);
  const uint32_t nrows = on ? rhi - rlo + 1 : 0u;
  const uint32_t rp = (nrows + NY - 1) / NY;
  const uint32_t r0 = rlo + (y * rp < nrows ? y * rp : nrows), r1 = rlo + ((y + 1) * rp < nrows ? (y + 1) * rp : nrows);
  constexpr int kU = 4;  // independent loads in flight per thread
  uint32_t sum = 0;
  for (uint32_t r = r0; r < r1; r += kU) {
    uint32_t v[kU];
#pragma unroll
    for (int k = 0; k < kU; ++k) v[k] = (r + k < r1) ? __ldcg(M + (size_t)(r + k) * Kp + b) : 0u;
#pragma unroll
    for (int k = 0; k < kU; ++k) sum += v[k];
  }
  s_part[y][x] = sum;
  __syncthreads();
  uint32_t run = 0;
  for (uint32_t yy = 0; yy < y; ++yy) run += s_part[yy][x];
  for (uint32_t r = r0; r < r1; r += kU) {
    uint32_t v[kU];
#pragma unroll
    for (int k = 0; k < kU; ++k) v[k] = (r + k < r1) ? __ldcg(M + (size_t)(r + k) * Kp + b) : 0u;
#pragma unroll
    for (int k = 0; k < kU; ++k) {
      if (r + k < r1) P[(size_t)(r + k) * Kp + b] = run;
      run += v[k];
    }
  }
  __syncthreads();  // scratch may be reused by the next group
}

// arguments of the tail (shared by k_colscan and the fused k_tick)
struct TailArgs {
  uint32_t Kp, K, n_segs;
  uint32_t n_cut;                     // (mode, group) cut segments; each is a run of partitions
  const uint16_t* part_cut;           // [n_segs] partition -> cut segment
  const uint32_t* cut_lp_lo;          // [n_cut + 1] first partition of the cut segment
  uint32_t layout;                    // bit 0: matched counts in shared memory; bit 1: bin keys too (tail_words)
  int32_t max_spread;                 // < 0: unlimited (policy S0); >= 0: policy S1, rating order only
  const uint32_t* tot;                // [Kp] bin totals of the pool being matched (kept up to date by ingest / remove / tick)
  const uint32_t* seg_bin_lo;         // [n_segs + 1]
  const uint32_t* seg_L;              // [n_segs]
  const uint16_t* bin_seg;            // [Kp] bin -> segment
  const uint16_t* bin_key;            // [Kp] bin -> clamp key (rating order: ascending inside a segment)
  uint32_t* outbase;                  // [Kp] out: member slot of the bin's first player
  uint32_t* binlim;                   // [Kp] out: outbase + matched players of the bin
  SegInfo* seg;                       // [n_segs] out
  TickCtr* ctr;
  const uint32_t* fill;               // [n_segs] partition fills of the pool being matched
  PoolMeta dst;                       // out: layout of the compacted pool (fill, chunk table, chunks used)
};
// shared-memory words of the tail for a layout: bases | matched counts (bit 0) | keys (bit 1)
__host__ __device__ constexpr uint32_t tail_words(uint32_t Kp, uint32_t layout) {
  return kTailScratchWords + (Kp + 2) + ((layout & 1u) ? (Kp + 2) : 0u) + ((layout & 2u) ? (Kp + 3) / 2 : 0u);
}

// The tail.  One pipeline for both policies:
//   bin totals -> bases s_bb -> matched prefix of every bin -> member slot of the bin's first player.
// S0 (reference behaviour): a (mode, group) partition of n players emits floor(n/L) lobbies, the n mod L
//   highest-ranked players stay queued: member slot = sorted position - leftovers of earlier partitions,
//   clipped at the partition's matched end (closed form, only a scan over the partitions).
// S1 (extension): greedy windowed walk over the partition (oracle: orc_run_windowed).  Players of one bin have
//   the same key, so the walk runs on the histogram: from position cur in bin v, lobbies are seeded at
//   cur, cur+L, ... while the seed is still in bin v and its L-th player has key <= key_v + W; whatever is
//   left of bin v afterwards cannot seed and stays queued.  Two-pointer over the bins of the segment.
// Very large key domains (layout bit 0 clear) park m_v in global memory and scan it in place of the bases.
__device__ __forceinline__ void colscan_tail_body(uint32_t* scratch, const TailArgs t) {
  constexpr uint32_t NW = kScanBlock / 32;
  uint32_t* s_tmp = scratch;            // [64]
  uint32_t* s_misc = scratch + 64;      // [4] heavy flag | n_matched | lobbies | chunks of the compacted pool
  uint32_t* s_a = scratch + 68;         // [kMaxSegs] leftovers of earlier segments
  uint32_t* s_ns = s_a + kMaxSegs;      // [kMaxSegs] alive players of the segment
  uint32_t* s_mt = s_ns + kMaxSegs;     // [kMaxSegs] matched players of the segment
  uint32_t* s_lo = s_mt + kMaxSegs;     // [kMaxSegs + 1] first bin of the segment
  uint32_t* s_nch = s_lo + kMaxSegs + 1;   // [kMaxSegs + 1] first chunk of the segment in the compacted pool
  uint32_t* s_L = s_nch + kMaxSegs + 1;    // [kMaxSegs] lobby size of the segment
  uint32_t* s_pc = s_L + kMaxSegs;         // [kMaxSegs] cut segment of the partition
  uint32_t* s_clp = s_pc + kMaxSegs;       // [kMaxSegs + 1] first partition of the cut segment
  uint32_t* s_ms = s_clp + kMaxSegs + 1;   // [kMaxSegs + 1] member slot of the partition's first matched player
  uint32_t* s_bb = scratch + kTailScratchWords;  // [Kp + 1] sorted position of the bin's first player
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, Kp = t.Kp, K = t.K, n_segs = t.n_segs;
  if (tid == 0) s_misc[0] = 0;
  for (uint32_t sg = tid; sg <= n_segs; sg += kScanBlock) s_lo[sg] = t.seg_bin_lo[sg];  // all the cold loads at once
  for (uint32_t sg = tid; sg < n_segs; sg += kScanBlock) { s_L[sg] = t.seg_L[sg]; s_pc[sg] = t.part_cut[sg]; }
  for (uint32_t c = tid; c <= t.n_cut; c += kScanBlock) s_clp[c] = t.cut_lp_lo[c];
  for (uint32_t i = tid; i < Kp; i += kScanBlock) s_bb[i] = __ldcg(&t.tot[i]);  // coalesced, independent loads
  __syncthreads();
  // list-ranked partitions only: does some bin expect > 8 players per tile of its partition?
  for (uint32_t sg = warp; sg < n_segs; sg += NW) {
    if (s_lo[sg + 1] - s_lo[sg] <= kFastBins) continue;
    uint32_t mx = 0;
    for (uint32_t v = s_lo[sg] + lane; v < s_lo[sg + 1]; v += 32) mx = s_bb[v] > mx ? s_bb[v] : mx;
    mx = __reduce_max_sync(0xFFFFFFFFu, mx);
    if (lane == 0 && (uint64_t)mx * kTile > 8ull * __ldcg(&t.fill[sg])) s_misc[0] = 1;
  }
  __syncthreads();
  const uint32_t total = block_excl_scan<kScanBlock>(s_bb, Kp, s_tmp);
  if (tid == 0) s_bb[Kp] = total;
  __syncthreads();
  const uint32_t alive = s_bb[K], dead = total - alive;
  const bool windowed = t.max_spread >= 0;
  const bool m_smem = (t.layout & 1u) != 0, key_smem = (t.layout & 2u) != 0;
  uint32_t* s_m = m_smem ? s_bb + Kp + 2 : t.binlim;  // S1: [Kp + 1] matched players of the bin

  if (!windowed) {
    // S0: a cut segment of n players gives n / L lobbies: its first (n / L) * L sorted positions are matched; a
    // partition holds the part of that prefix that falls into its own position range.
    for (uint32_t sg = tid; sg < n_segs; sg += kScanBlock) {
      const uint32_t c = s_pc[sg], cs = s_bb[s_lo[s_clp[c]]], ce = s_bb[s_lo[s_clp[c + 1]]], L = s_L[sg];
      const uint32_t mend = cs + (ce - cs) / L * L;
      const uint32_t a = s_bb[s_lo[sg]], b = s_bb[s_lo[sg + 1]];
      s_ns[sg] = b - a;
      s_mt[sg] = (mend < a ? a : (mend > b ? b : mend)) - a;
    }
  } else {
    uint16_t* s_key = reinterpret_cast<uint16_t*>(s_bb + (m_smem ? 2 : 1) * (Kp + 2));
    const uint16_t* keys = key_smem ? s_key : t.bin_key;
    if (key_smem)
      for (uint32_t v = tid; v < K; v += kScanBlock) s_key[v] = t.bin_key[v];
    for (uint32_t v = K + tid; v < Kp; v += kScanBlock) s_m[v] = 0;
    __syncthreads();
    const int32_t W = t.max_spread;
    // One warp walks TWO partitions at a time (two independent carry chains in flight).  Per bin, off the chain:
    //   reach  = sorted position where keys exceed key_v + W (binary search over the partition's keys)
    //   rsel   = min(reach, b1 - 1 + L): the seeds of bin v are cur, cur + L, ... < min(b1, reach - L + 1), so with
    //            a = rsel - cur the bin seeds a / L lobbies and p2 = rsel - a mod L is the next unconsumed position
    // and on the chain only: cur = max(pos, b0); a; a mod L by a reciprocal multiply; p2; select.  Empty bins
    // fall out of the same arithmetic (cur >= b1), so the 32 bins of a batch are visited by an unrolled loop.
    for (uint32_t sg = tid; sg < n_segs; sg += kScanBlock) s_ns[sg] = s_bb[s_lo[sg + 1]] - s_bb[s_lo[sg]];
    // the walk runs over whole CUT segments (a window may span the partitions of a wide rating group)
    for (uint32_t sg0 = warp; sg0 < t.n_cut; sg0 += 2 * NW) {
      uint32_t lo[2], hi[2], L[2], Mrec[2], pos[2];
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const uint32_t sg = sg0 + q * NW;
        const bool on = sg < t.n_cut;
        lo[q] = on ? s_lo[s_clp[sg]] : 0u; hi[q] = on ? s_lo[s_clp[sg + 1]] : 0u; L[q] = on ? s_L[s_clp[sg]] : 1u;
        Mrec[q] = 0xFFFFFFFFu / L[q];  // umulhi(a, Mrec) is a / L or a / L - 1 for every 32-bit a
        pos[q] = s_bb[lo[q]];
      }
      const uint32_t span0 = hi[0] - lo[0], span1 = hi[1] - lo[1], span = span0 > span1 ? span0 : span1;
      for (uint32_t off = 0; off < span; off += 32) {
        uint32_t b0[2], b1[2], rs[2], mine[2];
        bool valid[2];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const uint32_t v = lo[q] + off + lane;
          valid[q] = v < hi[q];
          b0[q] = b1[q] = rs[q] = 0u; mine[q] = 0u;
          if (valid[q]) {
            b0[q] = s_bb[v]; b1[q] = s_bb[v + 1];
            const int32_t lim = (int32_t)keys[v] + W;
            uint32_t a = v, e = hi[q];  // last bin in [v, hi) with key <= lim
            while (e - a > 1) { const uint32_t mid = (a + e) >> 1; if ((int32_t)keys[mid] <= lim) a = mid; else e = mid; }
            const uint32_t reach = s_bb[a + 1], cap = b1[q] - 1 + L[q];
            rs[q] = reach < cap ? reach : cap;
          }
        }
#pragma unroll 8
        for (int l = 0; l < 32; ++l) {
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            const uint32_t B0 = __shfl_sync(0xFFFFFFFFu, b0[q], l), B1 = __shfl_sync(0xFFFFFFFFu, b1[q], l);
            const uint32_t RS = __shfl_sync(0xFFFFFFFFu, rs[q], l);
            const uint32_t cur = pos[q] > B0 ? pos[q] : B0;
            const uint32_t a = RS - cur;                      // meaningful when cur < B1 (then RS > cur)
            uint32_t rem = a - __umulhi(a, Mrec[q]) * L[q];   // a mod L, or a mod L + L
            rem = rem < rem - L[q] ? rem : rem - L[q];        // unsigned: picks the one below L
            const uint32_t p2 = RS - rem;                     // next unconsumed position after this bin's lobbies
            const bool inside = cur < B1, full = p2 >= B1;
            const uint32_t m = (!inside || full) ? B1 - B0 : p2 - B0;  // matched players of the bin (a prefix)
            pos[q] = !inside ? pos[q] : (full ? p2 : B1);     // the rest of a partly matched bin stays queued
            if ((int)lane == l) mine[q] = m;
          }
        }
#pragma unroll
        for (int q = 0; q < 2; ++q)
          if (valid[q]) s_m[lo[q] + off + lane] = mine[q];
      }
    }
    __syncthreads();
    if (!m_smem) {  // very large key domain: the counts were parked in global memory; scan them in place of the bases
      for (uint32_t v = tid; v < Kp; v += kScanBlock) s_bb[v] = s_m[v];
      s_m = s_bb;
      __syncthreads();
    }
    // member slots = exclusive scan of the matched counts (members of successive partitions are contiguous)
    const uint32_t nm = block_excl_scan<kScanBlock>(s_m, Kp, s_tmp);
    if (tid == 0) s_m[Kp] = nm;
    __syncthreads();
    for (uint32_t v = tid; v < Kp; v += kScanBlock) {
      t.outbase[v] = s_m[v];
      t.binlim[v] = s_m[v + 1];  // = outbase + matched players of the bin
      // bin totals of the compacted pool: what was there minus the matched prefix; removed players are gone
      t.dst.tot[v] = v < K ? __ldcg(&t.tot[v]) - (s_m[v + 1] - s_m[v]) : 0u;
    }
    for (uint32_t sg = tid; sg < n_segs; sg += kScanBlock) s_mt[sg] = s_m[s_lo[sg + 1]] - s_m[s_lo[sg]];
  }
  __syncthreads();
  // Partition table, by ONE warp (<= 512 partitions, 32 per step with carries; no block-wide scans): member / lobby
  // bases, and the layout of the compacted pool — partition sg keeps n_left players in ceil(n_left / kTile) fresh
  // chunks handed out in partition order from chunk 0 (the epilogue moves the players).
  if (warp == 0) {
    uint32_t c_mem = 0, c_left = 0, c_ch = 0;
    for (uint32_t base = 0; base < n_segs; base += 32) {
      const uint32_t sg = base + lane;
      const bool on = sg < n_segs;
      const uint32_t ns = on ? s_ns[sg] : 0u, mt = on ? s_mt[sg] : 0u;
      const uint32_t nleft = ns - mt, nch = (nleft + kTile - 1) / kTile;
      uint32_t i_mem = mt, i_left = nleft, i_ch = nch;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const uint32_t a = __shfl_up_sync(0xFFFFFFFFu, i_mem, off);
        const uint32_t c = __shfl_up_sync(0xFFFFFFFFu, i_left, off), d = __shfl_up_sync(0xFFFFFFFFu, i_ch, off);
        if (lane >= (uint32_t)off) { i_mem += a; i_left += c; i_ch += d; }
      }
      if (on) {
        s_ms[sg] = c_mem + i_mem - mt;
        s_a[sg] = c_left + i_left - nleft;
        s_nch[sg] = c_ch + i_ch - nch;
        t.dst.fill[sg] = nleft;
      }
      c_mem += __shfl_sync(0xFFFFFFFFu, i_mem, 31);
      c_left += __shfl_sync(0xFFFFFFFFu, i_left, 31); c_ch += __shfl_sync(0xFFFFFFFFu, i_ch, 31);
    }
    __syncwarp();
    // Lobbies are cut per CUT segment: lobby k of segment c = member slots [mb_c + k L, + L).  A partition is
    // credited with the lobbies that START inside its member-slot range, so the header writers can loop per partition.
    uint32_t c_lob = 0;
    for (uint32_t base = 0; base < n_segs; base += 32) {
      const uint32_t sg = base + lane;
      const bool on = sg < n_segs;
      uint32_t nl = 0, hb = 0;
      if (on) {
        const uint32_t L = s_L[sg], mb = s_ms[s_clp[s_pc[sg]]], m0 = s_ms[sg] - mb, m1 = m0 + s_mt[sg];
        const uint32_t k0 = (m0 + L - 1) / L, k1 = (m1 + L - 1) / L;
        nl = k1 - k0; hb = mb + k0 * L;
      }
      uint32_t i_lob = nl;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const uint32_t b = __shfl_up_sync(0xFFFFFFFFu, i_lob, off);
        if (lane >= (uint32_t)off) i_lob += b;
      }
      if (on) {
        SegInfo si;
        si.n = s_ns[sg]; si.n_lobbies = nl; si.member_base = hb; si.lobby_base = c_lob + i_lob - nl;
        si.left_base = s_a[sg]; si.new_chunk = s_nch[sg]; si.n_left = s_ns[sg] - s_mt[sg]; si.reserved = 0;
        t.seg[sg] = si;
      }
      c_lob += __shfl_sync(0xFFFFFFFFu, i_lob, 31);
    }
    if (lane == 0) {
      s_nch[n_segs] = c_ch;
      s_misc[1] = c_mem; s_misc[2] = c_lob;
      *t.dst.bump = c_ch;
      t.ctr->n_lobbies = c_lob; t.ctr->n_matched = c_mem; t.ctr->n_alive = alive; t.ctr->n_dead = dead;
      t.ctr->n_resid = c_left;
      t.ctr->heavy = s_misc[0];
    }
  }
  __syncthreads();
  const uint32_t n_matched = s_misc[1];
  if (!windowed) {
    // S0: member slot = sorted position - leftovers of earlier partitions, clipped at the partition's matched end
    for (uint32_t sg = warp; sg < n_segs; sg += NW) {  // one warp per partition: no bin -> segment lookups
      const uint32_t lo = s_lo[sg], hi = s_lo[sg + 1], start = s_bb[lo], shift = s_a[sg];
      const uint32_t mend = start + s_mt[sg];  // end of the partition's matched positions
      for (uint32_t v = lo + lane; v < hi; v += 32) {
        const uint32_t b0 = s_bb[v], b1 = s_bb[v + 1];
        const uint32_t o = (b0 < mend ? b0 : mend), l = (b1 < mend ? b1 : mend);
        t.outbase[v] = o - shift;
        t.binlim[v] = l - shift;
        t.dst.tot[v] = (b1 - b0) - (l - o);  // bin totals of the compacted pool: the unmatched tail of the bin
      }
    }
    for (uint32_t v = K + tid; v < Kp; v += kScanBlock) { t.outbase[v] = n_matched; t.binlim[v] = n_matched; t.dst.tot[v] = 0; }
  }
  for (uint32_t sg = warp; sg < n_segs; sg += NW) {  // chunk lists of the compacted pool
    const uint32_t c0 = s_nch[sg], c1 = s_nch[sg + 1];
    for (uint32_t k = lane; k < c1 - c0; k += 32) t.dst.chunk_tab[(size_t)sg * t.dst.max_ch + k] = c0 + k;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kScanBlock) k_colscan(uint32_t R, const uint32_t* __restrict__ M, uint32_t* __restrict__ P,
                                                        const TailArgs t) {
  extern __shared__ __align__(16) uint32_t scratch[];  // max(kColScratchWords, tail_words(Kp, layout)) words
  __shared__ Geo geo;
  __shared__ uint32_t s_gtmp[33];
  if (blockIdx.x + 1 < gridDim.x) {
    geo_build<kScanBlock>(geo, t.fill, t.n_segs, R, s_gtmp);
    if (geo_use_colscan(geo)) colscan_cols_body(scratch, geo, blockIdx.x, t.Kp, t.K, t.bin_seg, M, P);
  } else {
    colscan_tail_body(scratch, t);
  }
}

}  // namespace mm
