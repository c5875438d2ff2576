// mm_epilogue.cuh — phase 4 of the tick: pool compaction of the leftovers + lobby headers
#pragma once
#include "mm_common.cuh"
#include "mm_scan.cuh"

namespace mm {

// ---------------------------------------------------------------------------------------
// k_epilogue.  Lobby headers from the segment table — lobby c of segment s = members
// [member_base + k*L, +L); replaces the payload assembly at search/worker.ex:315-319.
// Pool compaction, row-parallel and order-preserving: the placement pass left one bit per
// player that stays queued (left_bits) and the count per row; every CTA scans the R row
// counts, then walks the bit words of its rows — popcount prefix, slots of the set bits
// enumerated into shared memory, one thread per leftover player gathers its record from the
// old pool buffer into the alternate one and re-stamps the player's active-set entry.
// Replaces save_new_state/3 (search/worker.ex:282-289): the "partial lobby" is the players
// left resident.
// ---------------------------------------------------------------------------------------
constexpr uint32_t kLeftList = 2048;  // leftover players handled per step of the compaction
constexpr uint32_t kEpiScratchWords = (kMaxRows + 1) + 64 + (kMaxSegs + 1) + 4 * kMaxSegs + kLeftList;

struct EpiArgs {
  PoolView src, dst;
  PoolMeta src_meta, dst_meta;  // dst_meta was filled in by the scan tail
  uint32_t R, new_gen, n_segs, n_groups, Kp, write_headers;
  const uint32_t* rescnt;
  const uint32_t* left_bits;
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

template <int BLOCK>
__device__ __forceinline__ void epilogue_body(uint32_t* scratch, const Geo& g, const EpiArgs a,
                                              unsigned long long* t_mid = nullptr) {
  const PoolView& src = a.src;
  const PoolView& dst = a.dst;
  const uint32_t R = a.R, n_segs = a.n_segs;
  const uint32_t* __restrict__ rescnt = a.rescnt;
  const uint32_t* __restrict__ left_bits = a.left_bits;
  const ActiveView act = a.act;
  const SegInfo* __restrict__ seg = a.seg;
  const uint32_t* __restrict__ seg_L = a.seg_L;
  TickCtr* ctr = a.ctr;
  const uint32_t new_gen = a.new_gen;
  const uint32_t n = g.NT * kTile;            // virtual positions of this tick
  const uint32_t chunk = g.tpr * kTile;       // virtual positions per row
  constexpr uint32_t NW = BLOCK / 32;
  const PoolMeta sm = a.src_meta;
  auto phys_of = [&](uint32_t v, uint32_t& p) -> uint32_t {  // virtual position of the old pool -> physical slot, partition
    p = geo_seg_of(g, v / kTile);
    return __ldcg(&sm.chunk_tab[(size_t)p * sm.max_ch + (v / kTile - g.T0[p])]) * kTile + v % kTile;
  };
  uint32_t* s_off = scratch;                   // [kMaxRows + 1]
  uint32_t* s_tmp = s_off + kMaxRows + 1;      // [64]
  uint32_t* s_lbase = s_tmp + 64;              // [kMaxSegs + 1]
  uint32_t* s_mbase = s_lbase + kMaxSegs + 1;  // [kMaxSegs]
  uint32_t* s_L = s_mbase + kMaxSegs;          // [kMaxSegs]
  uint32_t* s_leftb = s_L + kMaxSegs;          // [kMaxSegs] rank of the partition's first leftover player
  uint32_t* s_newch = s_leftb + kMaxSegs;      // [kMaxSegs] the partition's first chunk in the compacted pool
  uint32_t* s_list = s_newch + kMaxSegs;       // [kLeftList]
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (uint32_t s = tid; s < n_segs; s += BLOCK) {
    s_lbase[s] = __ldcg(&seg[s].lobby_base); s_mbase[s] = __ldcg(&seg[s].member_base); s_L[s] = seg_L[s];
    s_leftb[s] = __ldcg(&seg[s].left_base); s_newch[s] = __ldcg(&seg[s].new_chunk);
  }
  for (uint32_t r = tid; r < R; r += BLOCK) s_off[r] = __ldcg(&rescnt[r]);
  __syncthreads();
  const uint32_t total = block_excl_scan<BLOCK>(s_off, R, s_tmp);
  if (tid == 0) {
    s_off[R] = total;
    if (blockIdx.x == 0) ctr->n_resid = total;
  }
  __syncthreads();
  if (a.write_headers)  // fire-and-forget stores first: they drain while the compaction waits on its dependent chains
    headers_body<BLOCK>(g, a, s_lbase, s_mbase, s_L, blockIdx.x, gridDim.x);
  // Work is split by leftover RANK, not by row: under policy S0 the leftovers are the latest arrivals of every
  // partition and sit in the last rows of the pool.  CTA b moves the players with global rank [r0, r1); it walks
  // the bit words of the rows holding them (popcount prefix from the start of the row), enumerates the pool
  // slots of its ranks into a shared-memory list (no memory latency) and then, one thread per listed player,
  // gathers the record into the alternate pool buffer and re-stamps the player's active-set entry — all the
  // dependent gather / hash-probe chains run in parallel, neighbouring threads touch neighbouring slots.
  const uint32_t per = (total + gridDim.x - 1) / gridDim.x;
  const uint32_t r0 = (uint64_t)blockIdx.x * per < total ? blockIdx.x * per : total;
  const uint32_t r1 = r0 + per < total ? r0 + per : total;
  if (r1 > r0) {
    uint32_t tbase = r0, fill = 0;  // global rank of s_list[0]; entries in the list (uniform)
    uint32_t row_beg = 0;           // pool slot of the current row's first player
    auto flush = [&](uint32_t count, bool last) {
      __syncthreads();
      for (uint32_t e = tid; e < count; e += BLOCK) {
        const uint32_t v = s_list[e], r = tbase + e;  // virtual position in the old pool, global leftover rank
        uint32_t p;  // a player never leaves its partition
        const uint32_t i = phys_of(v, p);
        const uint32_t loc = r - s_leftb[p];
        const uint32_t t = (s_newch[p] + loc / kTile) * kTile + loc % kTile;
        const uint64_t pid = src.id[i];
        dst.id[t] = pid; dst.rating[t] = src.rating[i]; dst.mode[t] = src.mode[i];
        dst.tsize[t] = src.tsize[i]; dst.ts[t] = src.ts[i]; dst.seq[t] = src.seq[i];
        const uint32_t key = src.bin[i];
        dst.bin[t] = (uint16_t)key;
        if (a.dst_meta.chist) atomicAdd(&a.dst_meta.chist[(size_t)(t / kTile) * kChunkHist + (key - a.seg_bin_lo[p])], 1u);
        if (act.on()) {
          const uint64_t h = act_find(act, pid);
          if (h != ~0ull) *act.val(h) = ((unsigned long long)new_gen << 32) | t;
        }
      }
      tbase += count;
      if (!last) __syncthreads();  // the last flush runs on into the lobby headers: the few threads waiting on
                                   // their gather / probe chains do not hold up the others
    };
    uint32_t row = 0;
    {  // first row holding rank r0: smallest row with s_off[row + 1] > r0
      uint32_t a = 0, e = R;
      while (a < e) { const uint32_t mid = (a + e) >> 1; if (s_off[mid + 1] > r0) e = mid; else a = mid + 1; }
      row = a;
    }
    for (; row < R && s_off[row] < r1; ++row) {
      const uint32_t off = s_off[row], cnt = s_off[row + 1] - off;
      if (cnt == 0) continue;  // uniform for the CTA
      const uint64_t beg64 = (uint64_t)row * chunk;
      const uint32_t beg = beg64 < n ? (uint32_t)beg64 : n;
      const uint32_t end = (beg64 + chunk < n) ? (uint32_t)(beg64 + chunk) : n;
      const uint32_t nwords = (end - beg + 31) >> 5;  // beg is a multiple of 32 (chunk is a multiple of kRound)
      const uint32_t* bits = left_bits + (beg >> 5);
      row_beg = beg;
      const uint32_t lo_l = (r0 > off ? r0 : off) - off, hi_l = (r1 < off + cnt ? r1 : off + cnt) - off;  // row-local ranks
      uint32_t run_l = 0;  // row-local rank of the step's first leftover player
      // 4 bit words (128 players) per thread and step: a row of 17 tiles is one step of a 512-thread CTA.  nwords is a
      // multiple of 64 (whole tiles) and `bits` is 16-byte aligned (rows start on tile boundaries).
      for (uint32_t w0 = 0; w0 < nwords && run_l < hi_l; w0 += 4 * BLOCK) {
        const uint32_t wi = w0 + 4 * tid;
        const uint4 w4 = wi < nwords ? __ldcg(reinterpret_cast<const uint4*>(bits + wi)) : make_uint4(0, 0, 0, 0);
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
        const uint32_t lpre = run_l + wbase + incl - c;  // row-local rank of this thread's first leftover player
        uint32_t q = lo_l > run_l ? lo_l : run_l;
        const uint32_t q_end = hi_l < run_l + wtot ? hi_l : run_l + wtot;
        while (q < q_end) {  // (uniform) ranks [q, q_end) of this step are mine
          if (fill == kLeftList) { flush(fill, false); fill = 0; }
          const uint32_t room = kLeftList - fill, take = q_end - q < room ? q_end - q : room;
          if (c && lpre < q + take && lpre + c > q) {
            uint32_t r = lpre;
#pragma unroll
            for (int k4 = 0; k4 < 4; ++k4) {
              uint32_t ww = wv[k4];
              while (ww) {
                const uint32_t bpos = __ffs(ww) - 1;
                ww &= ww - 1;
                if (r >= q && r < q + take) s_list[fill + (r - q)] = row_beg + ((wi + k4) << 5) + bpos;
                ++r;
              }
            }
          }
          fill += take;
          q += take;
        }
        run_l += wtot;
        __syncthreads();  // s_tmp is rewritten by the next step
      }
    }
    if (fill) flush(fill, true);
  }
  if (t_mid && tid == 0) {
    unsigned long long tm;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(tm));
    atomicMax(t_mid, tm);
  }
}

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_epilogue(const EpiArgs a) {
  __shared__ uint32_t scratch[kEpiScratchWords];
  __shared__ Geo geo;
  __shared__ uint32_t s_gtmp[33];
  geo_build<BLOCK>(geo, a.src_meta.fill, a.n_segs, a.R, s_gtmp);
  epilogue_body<BLOCK>(scratch, geo, a);
}

}  // namespace mm
