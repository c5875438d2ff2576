// mm_balance.cuh — balanced teams (mm_set_option "team_balance", include/mm_engine.h): every lobby of a masked two-team
// mode is split into the two teams with the least rating difference.  The tick's kernels are not touched: the pass runs
// on the tick's output (d_hdr, d_members) after the tick, and on mm_widen's output before it is copied out.
//
//   tb_split          one warp per lobby: L <= 16 values of c in, the balanced member order and its imbalance out.  The
//                     lanes take runs of the C(L - 1, S - 1) team-1 sets that hold member 0 (each lane's first set
//                     from a compile-time table, then Gosper-stepped), then a warp argmin on (|difference|, mask).
//                     k_tb_lobby and k_locate call it, so the emitted teams, mm_match_quality and mm_locate cannot
//                     disagree.
//   each member's c   rating order: the member slot's bin from the tick's per-bin member ranges (outbase, still valid
//                     right after the tick), c = key_lo + bin_key[bin] — no player is read;
//                     arrival order: k_tb_arrival walks the pool the tick read (live_rank_walk, as k_mq_arrival does)
//                     and writes every matched player's c - key_lo at its member slot;
//                     mm_widen: k_tb_pieces writes c - key_lo of every piece's bin at the piece's member slots.
//                     mm_party_match: k_tb_pieces for the solos, k_tb_parties (mm_party.cuh) for the party members.
//   k_tb_lobby        one warp per lobby of a masked mode with S > 1: reads the L ids, writes them back permuted (not
//                     when the permutation is the identity) and stores the lobby's imbalance.  mm_party_match's form
//                     (party_balance) reads each lobby's continuation word, so no split cuts a party, and sums the
//                     imbalances.
#pragma once
#include "mm_backfill.cuh"

namespace mm {

constexpr uint32_t kTbMaxS = 8;  // L <= 16: at most C(15, 7) = 6435 splits per lobby

constexpr uint32_t tb_binom(uint32_t n, uint32_t k) {
  if (k > n) return 0;
  uint32_t c = 1;
  for (uint32_t i = 0; i < k; ++i) c = c * (n - i) / (i + 1);
  return c;
}

// The k-subset of rank r in colex order (= ascending bitmask order) as a bitmask
constexpr uint32_t tb_unrank(uint32_t r, uint32_t k) {
  uint32_t x = 0;
  for (uint32_t i = k; i >= 1; --i) {  // the largest element e with C(e, i) <= r
    uint32_t e = i - 1;
    while (tb_binom(e + 1, i) <= r) ++e;
    x |= 1u << e;
    r -= tb_binom(e, i);
  }
  return x;
}

// Per team size S (L = 2S): the number of team-1 sets, C(2S - 1, S - 1), and each lane's first set (its run of ranks
// starts at lane x ceil(n / 32)), built at compile time: unranking per lobby costs more than the whole enumeration.
struct TbStarts {
  uint32_t n[kTbMaxS + 1];
  uint32_t x[kTbMaxS + 1][32];
};
constexpr TbStarts tb_starts() {
  TbStarts t{};
  for (uint32_t S = 1; S <= kTbMaxS; ++S) {
    const uint32_t n = tb_binom(2 * S - 1, S - 1), per = (n + 31) / 32;
    t.n[S] = n;
    for (uint32_t l = 0; l < 32; ++l) t.x[S][l] = l * per < n ? tb_unrank(l * per, S - 1) : 0u;
  }
  return t;
}
__device__ const TbStarts kTbStarts = tb_starts();

// One warp, every lane: lane i < L = 2S holds c_i (c - key_lo of member i in the lobby's current order).  Over the sets A of
// S members with member 0 in A, minimise |sum_A c - sum_rest c| (64-bit); ties go to the smallest M(A) = sum of 2^i
// over i in A, i > 0.  cont: bit i set when member i belongs to the same party as member i - 1; a set A is admissible
// when it holds all of every party or none of it, ((A ^ (A << 1)) & cont) == 0.  The identity (members [0, S)) is
// admissible whenever the lobby's parties do not straddle the teams, so some lane finds a winner; a lane that finds no
// admissible set keeps ~0.  cont == 0 (a compile-time constant for the tick, mm_widen and mm_locate) admits every set.
// Returns the mask of A (bit 0 set) on every lane and the imbalance in *imb.
__device__ __forceinline__ uint32_t tb_split(uint32_t ci, uint32_t L, uint32_t S, uint32_t cont,
                                             unsigned long long* imb) {
  const uint32_t lane = threadIdx.x & 31;
  uint32_t c[16];
  long long total = 0;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    c[j] = __shfl_sync(0xFFFFFFFFu, ci, j);
    total += (uint32_t)j < L ? (long long)c[j] : 0ll;
  }
  // team 1 besides member 0: an (S - 1)-subset x of members 1 .. L - 1, bit j of x = member j + 1
  const uint32_t n = kTbStarts.n[S], per = (n + 31) / 32;
  const uint32_t r0 = lane * per, r1 = r0 + per < n ? r0 + per : n;
  unsigned long long best_d = ~0ull;
  uint32_t best_m = ~0u;
  if (r0 < r1) {
    uint32_t x = kTbStarts.x[S][lane];
    for (uint32_t r = r0;;) {
      long long sa = c[0];
#pragma unroll
      for (int j = 0; j < 15; ++j) sa += ((x >> j) & 1u) ? (long long)c[j + 1] : 0ll;
      const long long d = 2 * sa - total;
      const unsigned long long ad = (unsigned long long)(d < 0 ? -d : d);
      const uint32_t m = x << 1, mf = m | 1u;
      if (((mf ^ (mf << 1)) & cont) == 0 && (ad < best_d || (ad == best_d && m < best_m))) { best_d = ad; best_m = m; }
      if (++r == r1) break;
      const uint32_t t = x | (x - 1);  // Gosper: the next larger mask with k bits
      x = (t + 1) | (((~t & (t + 1)) - 1) >> __ffs(x));
    }
  }
#pragma unroll
  for (int off = 16; off; off >>= 1) {
    const unsigned long long od = __shfl_xor_sync(0xFFFFFFFFu, best_d, off);
    const uint32_t om = __shfl_xor_sync(0xFFFFFFFFu, best_m, off);
    if (od < best_d || (od == best_d && om < best_m)) { best_d = od; best_m = om; }
  }
  *imb = best_d;
  return best_m | 1u;
}

// New index of member i under the split mask mf: A's members in their old order, then the others in theirs.
__device__ __forceinline__ uint32_t tb_new_index(uint32_t mf, uint32_t i, uint32_t S) {
  const uint32_t before = __popc(mf & ((1u << i) - 1u));
  return ((mf >> i) & 1u) ? before : S + i - before;
}

struct TbArgs {
  const mm_lobby_hdr* hdr;   // [n_lob]
  uint32_t n_lob;
  uint64_t* members;
  uint32_t mask;             // balanced modes
  const uint8_t* mode_tsize; // [MM_MAX_MODES]
  const uint32_t* cval;      // [member slots] c - key_lo (arrival-order tick, mm_widen), or null:
  const uint32_t* outbase;   // rating-order tick: [Kp] member slot of the bin's first player (ascending)
  const uint16_t* bin_key;   // [Kp] c - key_lo of the bin
  uint32_t K;                // live bins
  uint32_t* imb;             // [n_lob] imbalance per header position (saturated), or null
  const uint32_t* cont;      // kCont: [n_lob] continuation bits per header position (tb_split)
  unsigned long long* imb_sum;  // kCont: += the imbalances of the balanced lobbies
};

// The balanced teams of every lobby of a masked mode with S > 1 (one warp per lobby, grid-stride).  kCont: party
// lobbies (mm_party_match), whose splits keep every party whole.
template <bool kCval, bool kCont = false>
__global__ void __launch_bounds__(256) k_tb_lobby(const TbArgs a) {
  const uint32_t lane = threadIdx.x & 31, nw = gridDim.x * (blockDim.x >> 5);
  unsigned long long sum = 0;
  for (uint32_t h = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; h < a.n_lob; h += nw) {
    const mm_lobby_hdr hd = a.hdr[h];
    const uint32_t S = a.mode_tsize[hd.mode], L = hd.n_members;
    if (!((a.mask >> hd.mode) & 1u) || S < 2) continue;  // (uniform)
    const uint32_t m = hd.first_member + lane;
    uint64_t id = 0;
    uint32_t c = 0;
    if (lane < L) {
      id = a.members[m];
      c = kCval ? a.cval[m] : a.bin_key[last_le(a.outbase, 0, a.K, m)];
    }
    unsigned long long imb;
    const uint32_t mf = tb_split(c, L, S, kCont ? a.cont[h] : 0u, &imb);
    __syncwarp();  // every lane's load of its slot is ordered before another lane's store to it
    if (mf != (1u << S) - 1u && lane < L) a.members[hd.first_member + tb_new_index(mf, lane, S)] = id;
    if (a.imb && lane == 0) a.imb[h] = imb > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)imb;
    if (kCont) sum += imb;
  }
  if (kCont && lane == 0 && sum) atomicAdd(a.imb_sum, sum);
}

struct TbArrivalArgs {
  PoolView pool;              // the pool the tick read
  PoolMeta meta;
  const uint32_t* left_bits;  // the tick's
  const uint32_t* tile_off;   // live slots of the virtual tiles before each tile
  uint32_t n_segs, n_groups, mask;
  int32_t key_lo;
  uint32_t KR;
  const uint16_t* part_cut;   // [n_segs] partition -> queue
  const uint8_t* mode_tsize;
  const uint32_t* seg_bin_lo; // [n_segs + 1]
  const uint32_t* outbase;    // [Kp] the tick's: member slot of the bin's first player
  uint32_t* cval;             // out: [member slots] c - key_lo
};

// Arrival order: a queue is one partition and one bin, and its matched players are its first a_q L live players in
// storage order, so the matched player of live rank rho sits at member slot outbase[bin] + rho.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_tb_arrival(const TbArrivalArgs a) {
  __shared__ Geo geo;
  __shared__ uint32_t s_gtmp[33];
  __shared__ uint32_t s_warp[BLOCK / 32];
  uint32_t s0, s1;
  if (!geo_cta_run<BLOCK>(geo, a.meta.fill, a.n_segs, s_gtmp, s0, s1)) return;  // (uniform)
  auto want = [&](const TileDesc& d) {
    const uint32_t mode = a.part_cut[d.seg] / a.n_groups;
    return ((a.mask >> mode) & 1u) && a.mode_tsize[mode] > 1;
  };
  live_rank_walk<BLOCK>(geo, a.meta, a.pool.mode, a.left_bits, a.tile_off, s0, s1, s_warp, want,
                        [&](const TileDesc& d, size_t slot, bool matched, uint32_t rho) {
    if (matched) a.cval[a.outbase[a.seg_bin_lo[d.seg]] + rho] = clamp_key(a.key_lo, a.KR, a.pool.rating[slot]);
  });
}

// mm_widen: piece p's cnt players, all of bin p.bin, sit at member slots req_base[p.req] + p.poff + [0, cnt).
__global__ void k_tb_pieces(uint32_t n_pieces, const BfPiece* __restrict__ piece, const uint32_t* __restrict__ req_base,
                            const uint16_t* __restrict__ bin_key, uint32_t* __restrict__ cval) {
  const uint32_t lane = threadIdx.x & 31, p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (p >= n_pieces) return;
  const BfPiece c = piece[p];
  uint32_t* dst = cval + req_base[c.req] + c.poff;
  const uint32_t v = bin_key[c.bin];
  for (uint32_t i = lane; i < c.cnt; i += 32) dst[i] = v;
}

}  // namespace mm
