// mm_epilogue.cuh — the end of the tick: pool compaction of the leftovers (per row) + lobby headers
#pragma once
#include "mm_common.cuh"
#include "mm_scan.cuh"
#include "mm_place.cuh"

namespace mm {

// ---------------------------------------------------------------------------------------
// Lobby headers from the segment table — lobby c of segment s = members [member_base + k*L, +L); replaces the payload
// assembly at search/worker.ex:315-319.
// Pool compaction, row by row and order-preserving (compact_row): right after placing its tiles, a row moves the
// players it left queued (one bit each in left_bits) into the alternate pool buffer and re-stamps their active-set
// entries.  Replaces save_new_state/3 (search/worker.ex:282-289): the "partial lobby" is the players left resident.
// ---------------------------------------------------------------------------------------
constexpr uint32_t kLeftList = 2048;  // leftover players handled per step of the compaction
constexpr uint32_t kEpiScratchWords = (kMaxSegs + 1) + 2 * kMaxSegs;
constexpr uint32_t kRowCompactWords = 64 + 4 * kMaxSegs + kLeftList;
static_assert(kRowCompactWords * 4 <= kPlaceUnionBytes, "the row compaction re-uses the placement's shared memory");

struct EpiArgs {
  PoolView src, dst;
  PoolMeta src_meta, dst_meta;  // dst_meta was filled in by the scan tail
  uint32_t new_gen, n_segs, n_groups, write_headers;
  ActiveView act;
  const SegInfo* seg;
  const uint32_t* seg_L;
  const uint16_t* part_cut;  // [n_segs] partition -> (mode, group) cut segment
  const uint32_t* seg_bin_lo;
  mm_lobby_hdr* hdr;
  const uint32_t* src_idx;
  uint32_t* emit_seq;
  TickCtr* ctr;
};

// Lobby headers from the segment table — lobby c of segment s = members [member_base + k*L, +L); replaces the payload
// assembly at search/worker.ex:315-319.  Written by `nparts` CTAs (part = 0 .. nparts-1), 8 B per lobby.
template <int BLOCK>
__device__ __forceinline__ void headers_body(const Geo& g, const EpiArgs& a, const uint32_t* s_lbase, const uint32_t* s_mbase,
                                             const uint32_t* s_L, uint32_t part, uint32_t nparts) {
  const uint32_t tid = threadIdx.x, n_segs = a.n_segs, n_groups = a.n_groups;
  const PoolMeta sm = a.src_meta;
  const uint32_t total_lob = __ldcg(&a.ctr->n_lobbies);
  for (uint32_t sg = 0; sg < n_segs; ++sg) {  // segment by segment: no per-lobby search, ~8 instructions per header
    const uint32_t l0 = s_lbase[sg], l1 = sg + 1 < n_segs ? s_lbase[sg + 1] : total_lob;
    const uint32_t L = s_L[sg], mb = s_mbase[sg];
    mm_lobby_hdr h;
    h.n_members = (uint16_t)L;
    const uint32_t cut = a.part_cut[sg];
    h.mode = (uint8_t)(cut / n_groups);
    h.group = (uint8_t)(cut % n_groups);
    for (uint32_t c = l0 + part * BLOCK + tid; c < l1; c += nparts * BLOCK) {
      h.first_member = mb + (c - l0) * L;
      a.hdr[c] = h;
      if (a.emit_seq) {  // enqueue sequence number of the member whose arrival completed the lobby
        const uint32_t v = __ldcg(&a.src_idx[h.first_member + L - 1]), p = geo_seg_of(g, v / kTile);
        a.emit_seq[c] = a.src.seq[__ldcg(&sm.chunk_tab[(size_t)p * sm.max_ch + (v / kTile - g.T0[p])]) * kTile + v % kTile];
      }
    }
  }
}
// Lobby headers in chunks of kHdrChunk lobbies, claimed from *next by whichever CTA asks (row CTAs of the fused tick
// once they have placed their tiles): the rows that finish first write them, and no CTA that shares an SM with a
// placing row streams stores beside it for the whole phase.  (With emission order asked for, the epilogue writes the
// headers: emit_seq needs every row's src_idx.)
constexpr uint32_t kHdrChunk = 8192;
template <int BLOCK>
__device__ __forceinline__ void headers_claimed(uint32_t* scratch, const EpiArgs& a, uint32_t* next) {
  uint32_t* s_lbase = scratch;                 // [kMaxSegs + 1]
  uint32_t* s_mbase = s_lbase + kMaxSegs + 1;  // [kMaxSegs]
  uint32_t* s_L = s_mbase + kMaxSegs;          // [kMaxSegs]
  uint32_t* s_claim = s_L + kMaxSegs;
  const uint32_t tid = threadIdx.x, n_segs = a.n_segs, n_groups = a.n_groups;
  const uint32_t total_lob = __ldcg(&a.ctr->n_lobbies);
  for (uint32_t s = tid; s < n_segs; s += BLOCK) {
    s_lbase[s] = __ldcg(&a.seg[s].lobby_base); s_mbase[s] = __ldcg(&a.seg[s].member_base); s_L[s] = a.seg_L[s];
  }
  for (;;) {
    if (tid == 0) *s_claim = atomicAdd(next, 1u);
    __syncthreads();  // the claim and (first pass) the segment tables are visible
    const uint32_t c0 = *s_claim * kHdrChunk;
    __syncthreads();  // everyone has read the claim before thread 0 overwrites it
    if (c0 >= total_lob) break;
    const uint32_t c1 = c0 + kHdrChunk < total_lob ? c0 + kHdrChunk : total_lob;
    for (uint32_t c = c0 + tid; c < c1; c += BLOCK) {
      uint32_t lo = 0, hi = n_segs;  // segment of lobby c: the last sg with s_lbase[sg] <= c (empty ones share a base)
      while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (s_lbase[mid] <= c) lo = mid; else hi = mid; }
      mm_lobby_hdr h;
      h.n_members = (uint16_t)s_L[lo];
      const uint32_t cut = a.part_cut[lo];
      h.mode = (uint8_t)(cut / n_groups);
      h.group = (uint8_t)(cut % n_groups);
      h.first_member = s_mbase[lo] + (c - s_lbase[lo]) * s_L[lo];
      a.hdr[c] = h;
    }
  }
}

// compact_row<BLOCK>: the row's leftover players -> compacted pool, run by the row right after it has placed its tiles.
// A bin's slots are handed out in row order — outbase[b] + players of b in earlier rows (pre_b) + rank inside the
// row — and a player at or past binlim[b] stays queued, so the leftovers of partition p that lie in earlier rows are
// a closed form of the prefixes the placement's window load uses:
//     left_before(p) = sum over the bins b of p of  min(pre_b, max(0, outbase[b] + pre_b - binlim[b])).
// Rows are contiguous in a partition's enqueue order: the leftover of rank k among the row's leftovers of p (in
// virtual-position order) goes to slot new_chunk[p] * kTile + left_before(p) + k of the compacted pool, which needs
// nothing from the other rows.  The row walks its own left_bits words (popcount prefix; slots of the set bits listed
// in shared memory), then one thread per listed player gathers its record from the old pool buffer into the alternate
// one, adds it to the compacted chunk histogram and re-stamps its active-set entry.  Rows without leftovers return at
// once (policy S0: only a partition's last row has any).  A rank outside [0, n_left) of its partition is not written;
// TickCtr::left_bad counts it and the tick fails.
// nres: the row's leftover players (place_body's result).  lb (may be null): left_before of the row's first
// kLeftBeforeCap partitions, summed by the placement's window loads (place_left_before; outside `scratch`); the
// others are summed here.  clr_done (may be null): the compacted pool's chunk histograms are cleared once it reaches
// clr_target.
static_assert(kRowCompactWords * 4 <= kTileBytes + kChunkHist * 4, "the row compaction leaves the placement header alone");
template <int BLOCK>
__device__ __forceinline__ void compact_row(uint32_t* scratch, const Geo& g, const PlaceArgs& pa, const EpiArgs& a,
                                            uint32_t nres, const uint32_t* lb, unsigned int* clr_done,
                                            unsigned int clr_target) {
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, row = blockIdx.x;
  constexpr uint32_t NW = BLOCK / 32;
  if (nres == 0) return;  // (uniform; place_body ended on a barrier: its shared memory is free)
  const PoolView& src = a.src;
  const PoolView& dst = a.dst;
  const PoolMeta sm = a.src_meta;
  const uint32_t s0 = row * g.tpr, s1 = s0 + g.tpr < g.NT ? s0 + g.tpr : g.NT;  // the row holds leftovers: s0 < s1
  const uint32_t p0 = geo_seg_of(g, s0), np = geo_seg_of(g, s1 - 1) - p0 + 1;  // partitions of the row's tiles
  uint32_t* s_tmp = scratch;           // [64]
  uint32_t* s_off = s_tmp + 64;        // [np] left_before(p) - row rank of p's first leftover
  uint32_t* s_cnt = s_off + kMaxSegs;  // [np] leftovers of p in the row -> row rank of p's first leftover
  uint32_t* s_nl = s_cnt + kMaxSegs;   // [np] players of p that stay queued
  uint32_t* s_nc = s_nl + kMaxSegs;    // [np] compacted-pool slot of p's first leftover
  uint32_t* s_list = s_nc + kMaxSegs;  // [kLeftList]
  const uint32_t nwords = (s1 - s0) * (kTile / 32);
  const uint32_t* bits = pa.left_bits + (size_t)s0 * (kTile / 32);  // 16-byte aligned: rows start on tile boundaries
  // 4 bit words (128 players) per thread and step of the walk below; the first step's words are loaded here, beside
  // the left_before loads (a row of up to 32 tiles is one step of a 512-thread CTA)
  const uint4 w4_first = 4 * tid < nwords ? __ldcg(reinterpret_cast<const uint4*>(bits + 4 * tid)) : make_uint4(0, 0, 0, 0);
  const uint32_t n_lb = lb ? kLeftBeforeCap : 0u;  // partitions p0 .. p0 + n_lb - 1 come with their left_before
  for (uint32_t k = tid; k < np; k += BLOCK) {
    s_off[k] = k < n_lb ? lb[k] : 0u; s_cnt[k] = 0;
    s_nl[k] = __ldcg(&a.seg[p0 + k].n_left); s_nc[k] = __ldcg(&a.seg[p0 + k].new_chunk) * kTile;
  }
  __syncthreads();
  if (np > n_lb) {  // left_before of the other partitions with leftovers: the window load's prefixes (P, or the few rows before this one)
    const bool scanned = geo_use_colscan(g);
    for (uint32_t i = a.seg_bin_lo[p0 + n_lb] + tid; i < a.seg_bin_lo[p0 + np]; i += BLOCK) {
      const uint32_t p = pa.bin_seg[i];
      uint32_t rlo = 0, rhi = 0;
      if (!s_nl[p - p0] || !geo_rows_of(g, p, rlo, rhi)) continue;
      uint32_t pre = 0;
      if (scanned) pre = __ldcg(&pa.P[(size_t)row * pa.Kp + i]);
      else
        for (uint32_t r = rlo; r < row; r += 8) {
          uint32_t v8[8];
#pragma unroll
          for (uint32_t u = 0; u < 8; ++u) v8[u] = r + u < row ? __ldcg(&pa.M[(size_t)(r + u) * pa.Kp + i]) : 0u;
#pragma unroll
          for (uint32_t u = 0; u < 8; ++u) pre += v8[u];
        }
      const uint32_t end = __ldcg(&pa.outbase[i]) + pre, lim = __ldcg(&pa.binlim[i]);
      if (end > lim) atomicAdd(&s_off[p - p0], end - lim < pre ? end - lim : pre);
    }
  }
  for (uint32_t w0 = 0; w0 < nwords; w0 += 4 * BLOCK) {  // the row's leftovers per partition (a tile is 64 words)
    const uint32_t wi = w0 + 4 * tid;
    const uint4 w4 = w0 == 0 ? w4_first : (wi < nwords ? __ldcg(reinterpret_cast<const uint4*>(bits + wi)) : make_uint4(0, 0, 0, 0));
    const uint32_t c = __popc(w4.x) + __popc(w4.y) + __popc(w4.z) + __popc(w4.w);
    if (c) atomicAdd(&s_cnt[geo_seg_of(g, s0 + wi / (kTile / 32)) - p0], c);
  }
  if (a.dst_meta.chist && clr_done) grid_wait(clr_done, clr_target);  // before the first chunk-histogram add
  else __syncthreads();
  block_excl_scan<BLOCK>(s_cnt, np, s_tmp);
  for (uint32_t k = tid; k < np; k += BLOCK) s_off[k] -= s_cnt[k];

  uint32_t tbase = 0, fill = 0;  // row rank of s_list[0]; entries in the list (uniform)
  auto flush = [&](uint32_t count) {
    __syncthreads();
    for (uint32_t e = tid; e < count; e += BLOCK) {
      const uint32_t v = s_list[e];  // virtual position in the old pool
      const uint32_t p = geo_seg_of(g, v / kTile), k = p - p0;  // a player never leaves its partition
      const uint32_t loc = tbase + e + s_off[k];
      if (loc >= s_nl[k]) { atomicAdd(&a.ctr->left_bad, 1u); continue; }
      const uint32_t i = __ldcg(&sm.chunk_tab[(size_t)p * sm.max_ch + (v / kTile - g.T0[p])]) * kTile + v % kTile;
      const uint32_t t = s_nc[k] + loc;
      // every column of the record is loaded before the first store (the two pool buffers may alias as far as the
      // compiler knows): one round trip instead of seven
      const uint64_t pid = src.id[i];
      const int32_t rating = src.rating[i];
      const uint8_t mode = src.mode[i], tsize = src.tsize[i];
      const uint32_t ts = src.ts[i], seq = src.seq[i];
      const uint32_t key = src.bin[i];
      dst.id[t] = pid; dst.rating[t] = rating; dst.mode[t] = mode;
      dst.tsize[t] = tsize; dst.ts[t] = ts; dst.seq[t] = seq;
      dst.bin[t] = (uint16_t)key;
      if (a.dst_meta.chist) atomicAdd(&a.dst_meta.chist[(size_t)(t / kTile) * kChunkHist + (key - a.seg_bin_lo[p])], 1u);
      if (a.act.on()) {
        const uint64_t h = act_find(a.act, pid);
        if (h != ~0ull) *a.act.val(h) = ((unsigned long long)a.new_gen << 32) | t;
      }
    }
    tbase += count;
    __syncthreads();
  };
  uint32_t run = 0;  // row rank of the step's first leftover player
  for (uint32_t w0 = 0; w0 < nwords && run < nres; w0 += 4 * BLOCK) {
    const uint32_t wi = w0 + 4 * tid;
    const uint4 w4 = w0 == 0 ? w4_first : (wi < nwords ? __ldcg(reinterpret_cast<const uint4*>(bits + wi)) : make_uint4(0, 0, 0, 0));
    const uint32_t wv[4] = {w4.x, w4.y, w4.z, w4.w};
    const uint32_t c = __popc(w4.x) + __popc(w4.y) + __popc(w4.z) + __popc(w4.w);
    uint32_t incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, incl, o);
      if (lane >= (uint32_t)o) incl += u;
    }
    if (lane == 31) s_tmp[warp] = incl;
    __syncthreads();
    uint32_t wbase = 0, wtot = 0;
    for (uint32_t k = 0; k < NW; ++k) { const uint32_t v = s_tmp[k]; if (k < warp) wbase += v; wtot += v; }
    const uint32_t lpre = run + wbase + incl - c;  // row rank of this thread's first leftover player
    for (uint32_t q = run; q < run + wtot;) {  // (uniform) ranks [q, q + take) of this step go to the list
      if (fill == kLeftList) { flush(fill); fill = 0; }
      const uint32_t room = kLeftList - fill, take = run + wtot - q < room ? run + wtot - q : room;
      if (c && lpre < q + take && lpre + c > q) {
        uint32_t r = lpre;
#pragma unroll
        for (int k4 = 0; k4 < 4; ++k4) {
          uint32_t ww = wv[k4];
          while (ww) {
            const uint32_t bpos = __ffs(ww) - 1;
            ww &= ww - 1;
            if (r >= q && r < q + take) s_list[fill + (r - q)] = s0 * kTile + ((wi + k4) << 5) + bpos;
            ++r;
          }
        }
      }
      fill += take;
      q += take;
    }
    run += wtot;
    __syncthreads();  // s_tmp is rewritten by the next step
  }
  if (fill) flush(fill);
}

// The lobby headers with emission order (emit_seq needs every row's src_idx, so this runs after the placement of the
// whole pool): written by all CTAs of the launch.
template <int BLOCK>
__device__ __forceinline__ void epilogue_body(uint32_t* scratch, const Geo& g, const EpiArgs a) {
  uint32_t* s_lbase = scratch;                 // [kMaxSegs + 1]
  uint32_t* s_mbase = s_lbase + kMaxSegs + 1;  // [kMaxSegs]
  uint32_t* s_L = s_mbase + kMaxSegs;          // [kMaxSegs]
  for (uint32_t s = threadIdx.x; s < a.n_segs; s += BLOCK) {
    s_lbase[s] = __ldcg(&a.seg[s].lobby_base); s_mbase[s] = __ldcg(&a.seg[s].member_base); s_L[s] = a.seg_L[s];
  }
  __syncthreads();
  headers_body<BLOCK>(g, a, s_lbase, s_mbase, s_L, blockIdx.x, gridDim.x);
}

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_epilogue(const EpiArgs a, uint32_t R) {
  __shared__ uint32_t scratch[kEpiScratchWords];
  __shared__ Geo geo;
  __shared__ uint32_t s_gtmp[33];
  geo_build<BLOCK>(geo, a.src_meta.fill, a.n_segs, R, s_gtmp);
  epilogue_body<BLOCK>(scratch, geo, a);
}

}  // namespace mm
