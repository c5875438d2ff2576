// mm_band.cuh — the cross-group boundary pass on the device (mm_band_candidates / mm_band_match, DESIGN §6).
//
// BAND KEYS.  A call covers the boundaries g | g+1 for g_first <= g <= g_last and every mode: band b = (g - g_first)
// * n_modes + m, and band key q = b * 2W + j holds the rating hi_g - W + 1 + j — the lower side (group g) for j < W,
// the upper side (group g+1) for j >= W.  Ratings are consecutive integers, so j is the key of the walk, and q order
// is (boundary, mode, rating).  mm_band_candidates is the same numbering over the single boundary g-1 | g with only
// its upper side gathered: q order is then (mode, rating).
//
// Gather (k_band_prep, k_band_count, k_band_scan): every band key that lies in this pool has one sort-key bin (bin =
// mode * stride + lut[rating]); k_band_prep maps bin -> q, selects the partitions that hold such bins and gives every
// key a column of per-tile counts over its partition's tiles.  The key numbering is the caller's (BandKeyBins here,
// the backfill's own in mm_backfill.cuh); the rest of the gather and the place pass are shared.  The other partitions get a fill of 0 in the geometry
// the gather kernels build, so their tiles are never read.  k_band_count counts every tile's band players per key
// from the 2-byte bin column (dead slots sit in the removed bin, which maps to no key); k_band_scan turns each column
// into exclusive prefixes and the key's total.
//
// Walk (k_band_bases): one warp per band walks its 2W key counts with the tick's S1 arithmetic (s1_rsel / s1_step,
// mm_scan.cuh) -> matched players per key (a prefix in enqueue order), member slots, lobby bases.  Candidates take
// every player instead: key bases are the exclusive scan of the totals.
//
// Place (k_band_place): each band player lands at its key's base + its stable rank among the key's players (earlier
// tiles from the prefixes, earlier slots of its own tile by a warp-ordered pass), if that rank is below the key's
// limit; a match call takes the local players it places (pool_take_slot, as mm_take).  k_band_limit first cuts every
// selected partition after the tile of the last player any of its keys outputs, so the place pass reads no tile past it.  The caller's upper-side
// candidates (another rank's band) are checked, counted and placed by k_band_upper / k_band_upper_place.
#pragma once

#include "mm_active.cuh"
#include "mm_scan.cuh"

namespace mm {

constexpr uint32_t kBandBlock = 256;   // gather / place: one tile per warp at a time
constexpr uint32_t kBandWarps = kBandBlock / 32;
constexpr uint32_t kBandPrepBlock = 1024;
constexpr uint32_t kBandWalkBlock = 512;
constexpr uint32_t kBandNone = 0xFFFFFFFFu;

// k_band_upper error bits (mm_last_error names the first one that is set, in this order)
constexpr uint32_t kBandErrMode = 1, kBandErrRating = 2, kBandErrOrder = 4;

// ctr words written by the kernels of one call (zeroed by the host)
enum BandCtr : uint32_t { kBcKeys = 0, kBcLobbies, kBcMatched, kBcUpper, kBcTaken, kBcErr, kBcWords };

struct BandArgs {
  PoolView pool;
  PoolMeta meta;                  // meta.fill = the masked fills (written by k_band_prep)
  const uint32_t* fill;           // the pool's partition fills
  uint32_t n_segs, K;             // K = the removed bin
  BinMap bm;
  const uint16_t* bin_seg;
  const uint32_t* seg_bin_lo;
  int32_t W;
  uint32_t n_modes, g_first, n_bands, n_keys;
  uint32_t skip_lower;            // candidates: the lower sides are not gathered
  uint32_t remote_last;           // the upper side of the last boundary comes from the caller's columns
  int32_t hi[MM_MAX_GROUPS];      // group_hi of every group
  uint32_t L[MM_MAX_MODES];       // lobby size of every mode
  uint32_t* map;                  // [Kp] bin -> q (kBandNone: not a band key here)
  uint32_t* bfill;                // [n_segs] fills of the selected partitions, 0 for the others
  uint32_t* qoff;                 // [n_keys + 1] first count of the key's column
  uint32_t* qtiles;               // [n_keys] tiles of the key's partition
  uint32_t* qseg;                 // [n_keys] the key's partition (written for local keys)
  uint32_t* M;                    // per-(key, tile) counts -> exclusive prefixes -> running ranks (k_band_place)
  uint32_t* tot;                  // [n_keys] band players per key (local + caller's)
  uint32_t* pos;                  // [n_bands * (2W + 1)] walk: sorted position of every key's first player in its band
  uint32_t* kbase;                // [n_keys] output slot of the key's first player
  uint32_t* klim;                 // [n_keys] players of the key that are output (matched prefix, or all)
  uint32_t* band_mb;              // [n_bands + 1] first member slot of the band
  uint32_t* band_lb;              // [n_bands + 1] first lobby of the band
  uint32_t* ctr;                  // [kBcWords]
};

__device__ __forceinline__ uint32_t band_bin(const BandArgs& a, uint32_t q, bool& local) {
  const uint32_t twoW = 2u * (uint32_t)a.W, b = q / twoW, j = q - b * twoW;
  const uint32_t gi = b / a.n_modes, m = b - gi * a.n_modes;
  local = !(a.skip_lower && j < (uint32_t)a.W) && !(a.remote_last && gi + 1 == a.n_bands / a.n_modes && j >= (uint32_t)a.W);
  const int32_t r = a.hi[a.g_first + gi] - a.W + 1 + (int32_t)j;
  return m * a.bm.stride + a.bm.lut[r - a.bm.key_lo];
}

// The band numbering: key q -> its bin, local = the key's players are gathered from this pool.
struct BandKeyBins {
  __device__ __forceinline__ uint32_t operator()(const BandArgs& a, uint32_t q, bool& local) const {
    return band_bin(a, q, local);
  }
};

// One CTA: bin -> key map (a.map preset to kBandNone), partition selection, the keys' count columns.  KeyBins numbers
// the keys: kb(a, q, local) -> the bin of key q.
template <class KeyBins>
__global__ void __launch_bounds__(kBandPrepBlock) k_band_prep(const BandArgs a, const KeyBins kb) {
  __shared__ uint32_t s_sel[kMaxSegs];
  __shared__ uint32_t s_tmp[33];
  const uint32_t tid = threadIdx.x;
  for (uint32_t p = tid; p < a.n_segs; p += kBandPrepBlock) s_sel[p] = 0;
  __syncthreads();
  uint32_t carry = 0;
  for (uint32_t q0 = 0; q0 < a.n_keys; q0 += kBandPrepBlock) {  // a running exclusive scan of the column lengths
    const uint32_t q = q0 + tid;
    uint32_t tiles = 0;
    if (q < a.n_keys) {
      bool local;
      const uint32_t bin = kb(a, q, local);
      if (local) {
        const uint32_t p = a.bin_seg[bin];
        a.map[bin] = q;
        a.qseg[q] = p;
        s_sel[p] = 1;
        tiles = (__ldcg(&a.fill[p]) + kTile - 1) / kTile;
      }
      a.qtiles[q] = tiles;
    }
    const uint32_t off = block_scan_step<kBandPrepBlock>(tiles, carry, s_tmp);
    if (q < a.n_keys) a.qoff[q] = off;
  }
  if (tid == 0) a.qoff[a.n_keys] = carry;
  for (uint32_t p = tid; p < a.n_segs; p += kBandPrepBlock) a.bfill[p] = s_sel[p] ? __ldcg(&a.fill[p]) : 0u;
}

// The band keys of the 8 slots [o, o + 8) of a tile (kBandNone: not a band player, or past the tile's fill).
__device__ __forceinline__ void band_keys8(const BandArgs& a, size_t base, uint32_t o, uint32_t nvalid, uint32_t q[8]) {
  const uint4 b8 = o < nvalid ? __ldcs(reinterpret_cast<const uint4*>(a.pool.bin + base + o)) : make_uint4(~0u, ~0u, ~0u, ~0u);
  const uint32_t w[4] = {b8.x, b8.y, b8.z, b8.w};
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const uint32_t bin = (w[k >> 1] >> (16 * (k & 1))) & 0xFFFFu;
    q[k] = (o + k < nvalid && bin < a.K) ? __ldg(&a.map[bin]) : kBandNone;
  }
}

// Counting pass: M[qoff[q] + tile of the partition] += band players of key q in the tile.  One warp per tile; a warp
// adds once per distinct key of every 8-slot column.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_band_count(const BandArgs a) {
  __shared__ Geo geo;
  __shared__ uint32_t s_gtmp[33];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  geo_build<BLOCK>(geo, a.meta.fill, a.n_segs, 1, s_gtmp);
  for (uint32_t s = blockIdx.x * (BLOCK / 32) + warp; s < geo.NT; s += gridDim.x * (BLOCK / 32)) {
    const TileDesc d = geo_tile(geo, a.meta, s);
    const uint32_t t = s - geo.T0[d.seg];
    const size_t base = (size_t)d.phys * kTile;
    for (uint32_t o0 = 0; o0 < d.nvalid; o0 += 256) {
      uint32_t q[8];
      band_keys8(a, base, o0 + lane * 8, d.nvalid, q);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        if (!__any_sync(0xFFFFFFFFu, q[k] != kBandNone)) continue;
        const uint32_t peers = __match_any_sync(0xFFFFFFFFu, q[k]);
        if (q[k] != kBandNone && lane == (uint32_t)__ffs(peers) - 1) atomicAdd(&a.M[a.qoff[q[k]] + t], (uint32_t)__popc(peers));
      }
    }
  }
}

// Column scan: one warp per key, exclusive prefixes over the tiles of its partition in place; tot[q] = the total.
__global__ void __launch_bounds__(256) k_band_scan(const BandArgs a) {
  const uint32_t lane = threadIdx.x & 31, q = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (q >= a.n_keys) return;
  uint32_t* col = a.M + a.qoff[q];
  const uint32_t total = warp_col_scan(col, col, a.qtiles[q]);
  if (lane == 0) a.tot[q] = total;
}

// One CTA, once klim is known: the last tile of its partition that holds one of key q's first min(klim, tot) players
// (the last tile whose exclusive prefix is below that count), and every selected partition's fill cut after the last
// such tile of its keys (0: none of its players is output).  The place pass then skips the tiles past it without
// loading their key columns; the running ranks of the tiles it does place are unchanged.
__global__ void __launch_bounds__(kBandPrepBlock) k_band_limit(const BandArgs a) {
  __shared__ uint32_t s_lim[kMaxSegs];
  const uint32_t tid = threadIdx.x;
  for (uint32_t p = tid; p < a.n_segs; p += kBandPrepBlock) s_lim[p] = 0;
  __syncthreads();
  for (uint32_t q = tid; q < a.n_keys; q += kBandPrepBlock) {
    const uint32_t n = a.qtiles[q], lim = min(a.klim[q], a.tot[q]);
    if (n == 0 || lim == 0) continue;
    // the last tile with col[t] < lim (col[0] = 0 < lim)
    atomicMax(&s_lim[a.qseg[q]], last_le(a.M + a.qoff[q], 0, n, lim - 1) + 1);
  }
  __syncthreads();
  for (uint32_t p = tid; p < a.n_segs; p += kBandPrepBlock) a.bfill[p] = min(a.bfill[p], s_lim[p] * kTile);
}

// The caller's upper-side candidates of the last boundary: checked (mode, rating range, (mode, rating) order), then
// counted into tot and the first index of every key recorded in rstart.  Entries that fail a check count nothing: the
// host refuses the call before anything is placed.
__device__ __forceinline__ uint32_t band_upper_key(const BandArgs& a, uint8_t m, int32_t r) {
  const uint32_t b = (a.n_bands / a.n_modes - 1) * a.n_modes + m;
  return b * 2u * (uint32_t)a.W + (uint32_t)a.W + (uint32_t)(r - a.hi[a.g_first + a.n_bands / a.n_modes - 1] - 1);
}
__global__ void k_band_upper(const BandArgs a, uint32_t n, const int32_t* __restrict__ rating,
                             const uint8_t* __restrict__ mode, uint32_t* __restrict__ rstart) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t hi = a.hi[a.g_first + a.n_bands / a.n_modes - 1];
  const uint8_t m = mode[i];
  const int32_t r = rating[i];
  uint32_t err = 0;
  if (m >= a.n_modes) err |= kBandErrMode;
  if (r <= hi || (int64_t)r - hi > a.W) err |= kBandErrRating;
  if (i > 0 && (mode[i - 1] > m || (mode[i - 1] == m && rating[i - 1] > r))) err |= kBandErrOrder;
  if (err) { atomicOr(&a.ctr[kBcErr], err); return; }
  const uint32_t q = band_upper_key(a, m, r);
  atomicAdd(&a.tot[q], 1u);
  if (i == 0 || mode[i - 1] != m || rating[i - 1] != r) rstart[q] = i;
}

// Identity keys: the band key j is its rating offset.
struct BandKeys {
  __device__ __forceinline__ uint32_t operator[](uint32_t j) const { return j; }
};

// One CTA.  match = 0 (candidates): kbase = exclusive scan of tot, klim = all; ctr[kBcKeys] = the total.
// match = 1: the S1 walk of every band (one warp per band) -> klim = matched prefix per key, kbase = member slot of
// the key's first matched player; band_mb / band_lb = member / lobby bases per band; ctr = lobbies, matched, and the
// caller's candidates consumed.
__global__ void __launch_bounds__(kBandWalkBlock) k_band_bases(const BandArgs a, uint32_t match) {
  __shared__ uint32_t s_tmp[33];
  __shared__ uint32_t s_bm[kMaxSegs + 1], s_bl[kMaxSegs + 1];
  constexpr uint32_t NW = kBandWalkBlock / 32;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (!match) {
    uint32_t carry = 0;
    for (uint32_t q0 = 0; q0 < a.n_keys; q0 += kBandWalkBlock) {
      const uint32_t q = q0 + tid;
      const uint32_t base = block_scan_step<kBandWalkBlock>(q < a.n_keys ? a.tot[q] : 0u, carry, s_tmp);
      if (q < a.n_keys) { a.kbase[q] = base; a.klim[q] = kBandNone; }
    }
    if (tid == 0) a.ctr[kBcKeys] = carry;
    return;
  }
  const uint32_t twoW = 2u * (uint32_t)a.W, nb = a.n_bands;
  uint32_t upper = 0;  // the caller's candidates this warp's bands consume
  for (uint32_t b = warp; b < nb; b += NW) {
    const uint32_t q0 = b * twoW, L = a.L[b % a.n_modes], Mrec = 0xFFFFFFFFu / L;
    uint32_t* bb = a.pos + b * (twoW + 1);
    const uint32_t n_band = warp_col_scan(a.tot + q0, bb, twoW);  // sorted positions inside the band
    if (lane == 0) bb[twoW] = n_band;
    __syncwarp();
    const bool remote_band = a.remote_last && b / a.n_modes + 1 == nb / a.n_modes;
    uint32_t wpos = 0, mcarry = 0;
    for (uint32_t off = 0; off < twoW; off += 32) {
      const uint32_t v = off + lane;
      const bool valid = v < twoW;
      uint32_t b0 = 0, b1 = 0, rs = 0, mine = 0;
      if (valid) { b0 = bb[v]; b1 = bb[v + 1]; rs = s1_rsel(bb, BandKeys{}, v, twoW, a.W, L, b1); }
      for (int l = 0; l < 32; ++l) {
        const uint32_t B0 = __shfl_sync(0xFFFFFFFFu, b0, l), B1 = __shfl_sync(0xFFFFFFFFu, b1, l);
        const uint32_t RS = __shfl_sync(0xFFFFFFFFu, rs, l);
        const uint32_t m = s1_step(wpos, B0, B1, RS, L, Mrec);
        if ((int)lane == l) mine = m;
      }
      const uint32_t incl = warp_incl_scan(mine);
      if (valid) { a.klim[q0 + v] = mine; a.kbase[q0 + v] = mcarry + incl - mine; }  // relative to the band for now
      if (valid && remote_band && v >= (uint32_t)a.W) upper += mine;
      mcarry += __shfl_sync(0xFFFFFFFFu, incl, 31);
    }
    if (lane == 0) s_bm[b] = mcarry;
  }
  upper = __reduce_add_sync(0xFFFFFFFFu, upper);
  if (lane == 0 && upper) atomicAdd(&a.ctr[kBcUpper], upper);
  __syncthreads();
  if (warp == 0) {  // member and lobby bases of the bands, in band order = (boundary, mode)
    uint32_t cm = 0, cl = 0;
    for (uint32_t b0 = 0; b0 < nb; b0 += 32) {
      const uint32_t b = b0 + lane;
      const uint32_t m = b < nb ? s_bm[b] : 0u, l = b < nb ? m / a.L[b % a.n_modes] : 0u;
      const uint32_t im = warp_incl_scan(m), il = warp_incl_scan(l);
      if (b < nb) { s_bm[b] = cm + im - m; s_bl[b] = cl + il - l; }
      cm += __shfl_sync(0xFFFFFFFFu, im, 31);
      cl += __shfl_sync(0xFFFFFFFFu, il, 31);
    }
    if (lane == 0) {
      s_bm[nb] = cm; s_bl[nb] = cl;
      a.ctr[kBcMatched] = cm; a.ctr[kBcLobbies] = cl;
    }
  }
  __syncthreads();
  for (uint32_t b = tid; b <= nb; b += kBandWalkBlock) { a.band_mb[b] = s_bm[b]; a.band_lb[b] = s_bl[b]; }
  for (uint32_t q = tid; q < a.n_keys; q += kBandWalkBlock) a.kbase[q] += s_bm[q / twoW];
}

// Placing pass: the band players of every tile in slot order (= enqueue order inside the partition).  Per 256-slot
// step a warp lists its band players in order in shared memory, then ranks them 32 at a time: peers of one key by
// __match_any_sync, the key's running rank in M (the tile's exclusive prefix after k_band_scan; only this warp touches
// the tile's entries).  A player whose rank is below klim[q] goes to kbase[q] + rank: its id, rating and mode to the
// candidate columns, or its id to the members, and then it is taken (take = 1); its enqueue stamp beside the id when ts
// is not null (mm_widen / mm_party_match: the off-tick report, mm_offtick.cuh).
struct BandOut {
  uint64_t* id;
  int32_t* rating;  // candidates only
  uint8_t* mode;    // candidates only
  uint32_t take;
  uint32_t* ts = nullptr;
};
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_band_place(const BandArgs a, const BandOut out) {
  __shared__ Geo geo;
  __shared__ uint32_t s_gtmp[33];
  __shared__ uint32_t s_q[BLOCK / 32][256];
  __shared__ uint16_t s_o[BLOCK / 32][256];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, lt = (1u << lane) - 1u;
  geo_build<BLOCK>(geo, a.meta.fill, a.n_segs, 1, s_gtmp);
  uint32_t taken = 0;
  for (uint32_t s = blockIdx.x * (BLOCK / 32) + warp; s < geo.NT; s += gridDim.x * (BLOCK / 32)) {
    const TileDesc d = geo_tile(geo, a.meta, s);
    const uint32_t t = s - geo.T0[d.seg];
    const size_t base = (size_t)d.phys * kTile;
    for (uint32_t o0 = 0; o0 < d.nvalid; o0 += 256) {
      uint32_t q[8];
      const uint32_t o = o0 + lane * 8;
      band_keys8(a, base, o, d.nvalid, q);
      uint32_t cnt = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) cnt += q[k] != kBandNone;
      const uint32_t incl = warp_incl_scan(cnt);
      const uint32_t n = __shfl_sync(0xFFFFFFFFu, incl, 31);
      if (n == 0) continue;
      uint32_t w = incl - cnt;
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (q[k] != kBandNone) { s_q[warp][w] = q[k]; s_o[warp][w] = (uint16_t)(o + k); ++w; }
      __syncwarp();
      for (uint32_t e0 = 0; e0 < n; e0 += 32) {
        const uint32_t e = e0 + lane;
        const uint32_t qq = e < n ? s_q[warp][e] : kBandNone;
        const uint32_t peers = __match_any_sync(0xFFFFFFFFu, qq);
        const uint32_t leader = __ffs(peers) - 1;
        uint32_t run = 0;
        if (qq != kBandNone && lane == leader) {
          uint32_t* r = &a.M[a.qoff[qq] + t];
          run = *r;
          *r = run + __popc(peers);
        }
        run = __shfl_sync(0xFFFFFFFFu, run, leader);
        if (qq != kBandNone) {
          const uint32_t rank = run + __popc(peers & lt);
          if (rank < a.klim[qq]) {
            const uint32_t slot = (uint32_t)(base + s_o[warp][e]);
            const uint32_t at = a.kbase[qq] + rank;
            out.id[at] = a.pool.id[slot];
            if (out.rating) { out.rating[at] = a.pool.rating[slot]; out.mode[at] = a.pool.mode[slot]; }
            if (out.ts) out.ts[at] = a.pool.ts[slot];
            if (out.take && pool_take_slot(a.pool, a.meta, slot, a.K, a.bin_seg, a.seg_bin_lo)) ++taken;
          }
        }
        __syncwarp();  // the running ranks in M are read again by the next 32 entries
      }
    }
  }
  taken = __reduce_add_sync(0xFFFFFFFFu, taken);
  if (lane == 0 && taken) atomicAdd(&a.ctr[kBcTaken], taken);
}

// The caller's candidates: entry i is consumed when its rank inside its key is below the key's matched prefix.
__global__ void k_band_upper_place(const BandArgs a, uint32_t n, const uint64_t* __restrict__ id,
                                   const int32_t* __restrict__ rating, const uint8_t* __restrict__ mode,
                                   const uint32_t* __restrict__ rstart, uint64_t* __restrict__ members,
                                   uint8_t* __restrict__ taken) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t q = band_upper_key(a, mode[i], rating[i]), rank = i - rstart[q];
  const bool hit = rank < a.klim[q];
  if (hit) members[a.kbase[q] + rank] = id[i];
  taken[i] = hit ? 1 : 0;
}

// Lobby headers: lobby k of band b = member slots [band_mb[b] + (k - band_lb[b]) L, + L), group g_first + b / n_modes.
__global__ void k_band_hdr(const BandArgs a, uint32_t n_lobbies, mm_lobby_hdr* __restrict__ hdr) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_lobbies) return;
  const uint32_t lo = last_le(a.band_lb, 0, a.n_bands, k);
  const uint32_t m = lo % a.n_modes, L = a.L[m];
  mm_lobby_hdr h;
  h.first_member = a.band_mb[lo] + (k - a.band_lb[lo]) * L;
  h.n_members = (uint16_t)L;
  h.mode = (uint8_t)m;
  h.group = (uint8_t)(a.g_first + lo / a.n_modes);
  hdr[k] = h;
}

}  // namespace mm
