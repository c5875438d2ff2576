// mm_image.cuh — host image of the queue state (mm_export / mm_import; layout in include/mm_engine.h).
//
// Export: two passes over the tick's virtual tile sequence (geo_build over the partition fills, as k_expire and
// k_queue_stats walk it).  Pass 1 counts the live slots of every tile (and of every partition); k_scan_small turns the
// tile counts into offsets; pass 2 writes the live players of each tile at its offset, compacted and in order, into
// the image's columns in device memory — so the columns are partition by partition, in enqueue order inside a
// partition.  k_img_active compacts the active-set entries that are not queued (matched players awaiting mm_remove,
// players taken by mm_take) out of the hashed or direct-mapped table.
//
// Import: the layout is the engine's own (same config), so the host lays out every partition on consecutive chunks
// from the partition counts; k_img_load writes the columns into their slots, derives the sort key and team size,
// builds the bin totals and chunk histograms, and checks every player.  k_img_insert puts the ids of both sections
// into the active set (duplicate check) with the "not queued" value kPtMatched — a slot past every pool, so the entry
// never matches a slot, and not generation 0, which names a queued party's row — and k_restamp then points the queued
// players' entries at their slots.  A failed check sets a bit
// of one error word; the host then clears the engine.
//
// Queue move (mm_export_queues / mm_merge): the export passes with a partition selection; the merge kernels at the
// end of this file check a queue image and turn it into one ingest batch for a running engine.
#pragma once

#include "mm_active.cuh"

namespace mm {

constexpr uint32_t kImgBlock = 256;  // 8 slots per thread: one tile per CTA step
static_assert(kImgBlock * 8 == kTile, "a CTA step covers one tile");

// error bits of an import (the host names them in mm_last_error)
constexpr uint32_t kImgBadId = 1, kImgBadMode = 2, kImgBadRating = 4, kImgBadSeq = 8, kImgDup = 16, kImgFull = 32;

// the player columns of an image, in device memory (id: u64, or u32 handles when id_bytes == 4)
struct ImgCols {
  void* id;
  int32_t* rating;
  uint32_t* ts;
  uint32_t* seq;
  uint8_t* mode;
  uint32_t id_bytes;
};

__device__ __forceinline__ uint64_t img_id(const ImgCols& c, uint32_t i) {
  return c.id_bytes == 8 ? static_cast<const uint64_t*>(c.id)[i] : static_cast<const uint32_t*>(c.id)[i];
}
__device__ __forceinline__ void img_set_id(const ImgCols& c, uint32_t i, uint64_t pid) {
  if (c.id_bytes == 8) static_cast<uint64_t*>(c.id)[i] = pid;
  else static_cast<uint32_t*>(c.id)[i] = (uint32_t)pid;
}
// player s of `in` -> player d of `out`, every column
__device__ __forceinline__ void img_copy(const ImgCols& out, uint32_t d, const ImgCols& in, uint32_t s) {
  img_set_id(out, d, img_id(in, s));
  out.rating[d] = in.rating[s]; out.ts[d] = in.ts[s]; out.seq[d] = in.seq[s]; out.mode[d] = in.mode[s];
}

struct ImgExportArgs {
  PoolView pool;
  PoolMeta meta;
  uint32_t n_segs;
  uint32_t* tile_cnt;  // [virtual tiles] pass 1: live slots of the tile; pass 2: the tile's first output index
  uint32_t* part_cnt;  // [n_segs] pass 1: live slots of the partition (zeroed by the host)
  const uint8_t* sel;  // [n_segs] or null: only the partitions with a non-zero byte (mm_export_queues)
  ImgCols out;         // pass 2
};

// Pass 1 (WRITE = false) / pass 2 (WRITE = true).  CTAs take contiguous runs of the virtual tile sequence.
template <int BLOCK, bool WRITE>
__global__ void __launch_bounds__(BLOCK) k_img_tiles(const ImgExportArgs a) {
  __shared__ Geo geo;
  __shared__ uint32_t s_gtmp[33];
  __shared__ uint32_t s_warp[BLOCK / 32];
  const uint32_t tid = threadIdx.x;
  uint32_t s0, s1;
  if (!geo_cta_run<BLOCK>(geo, a.meta.fill, a.n_segs, s_gtmp, s0, s1)) return;  // (uniform)
  const uint32_t o = tid * 8;
  for (uint32_t s = s0; s < s1; ++s) {
    const TileDesc d = geo_tile(geo, a.meta, s);
    const size_t base = (size_t)d.phys * kTile + o;
    uint32_t live = 0;  // bit j: slot base + j holds a live player of a selected partition
    if (o < d.nvalid && (!a.sel || a.sel[d.seg])) {
      const uint2 m2 = __ldcs(reinterpret_cast<const uint2*>(a.pool.mode + base));
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (o + j < d.nvalid && mode8_at(m2, j) != MM_MODE_DEAD) live |= 1u << j;
      }
    }
    const uint32_t k = __popc(live), incl = warp_incl_scan(k);
    uint32_t total;
    const uint32_t before = block_warp_offsets<BLOCK>(incl, total, s_warp);
    if (!WRITE) {
      if (tid == 0) {
        a.tile_cnt[s] = total;
        if (total) atomicAdd(&a.part_cnt[d.seg], total);
      }
      continue;
    }
    if (!live) continue;
    uint32_t q = a.tile_cnt[s] + before + incl - k;
#pragma unroll 1
    for (int j = 0; j < 8; ++j) {
      if (!((live >> j) & 1u)) continue;
      const size_t slot = base + j;
      img_set_id(a.out, q, a.pool.id[slot]);
      a.out.rating[q] = a.pool.rating[slot];
      a.out.ts[q] = a.pool.ts[slot];
      a.out.seq[q] = a.pool.seq[slot];
      a.out.mode[q] = a.pool.mode[slot];
      ++q;
    }
  }
}

// The committed active-set entries that are not a live queued player's: a queued player's entry is exactly
// gen << 32 | slot with a slot that is not dead (k_expire's check); a taken player keeps such an entry on a dead slot.
// Output unordered, through a warp-aggregated cursor; at most `cap` are written (the host knows n_active).
__global__ void k_img_active(ActiveView act, uint64_t n_tab, const uint8_t* __restrict__ pool_mode, uint32_t n_slots,
                             uint32_t gen, void* out, uint32_t id_bytes, uint32_t cap, uint32_t* __restrict__ ctr) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t s0 = (uint64_t)blockIdx.x * blockDim.x; s0 < n_tab; s0 += stride) {  // uniform per CTA
    const uint64_t s = s0 + threadIdx.x;
    bool emit = false;
    uint64_t pid = 0;
    if (s < n_tab) {
      unsigned long long v;
      if (act.dcap) {
        pid = s;
        v = *act.val(s);
      } else {
        pid = *act.key(s);
        v = pid < kTombKey ? *act.val(s) : kFreeVal;
      }
      emit = v < kPending;
      const uint32_t slot = (uint32_t)v;
      if (emit && (uint32_t)(v >> 32) == gen && slot < n_slots && pool_mode[slot] != MM_MODE_DEAD) emit = false;
    }
    const uint32_t q = warp_append(ctr, emit);
    if (emit && q < cap) {
      if (id_bytes == 8) static_cast<uint64_t*>(out)[q] = pid;
      else static_cast<uint32_t*>(out)[q] = (uint32_t)pid;
    }
  }
}

struct ImgLoadArgs {
  PoolView pool;
  PoolMeta meta;
  ImgCols in;
  uint32_t n, n_segs;
  const uint32_t* part_off;   // [n_segs + 1] first image index of the partition
  const uint32_t* slot_base;  // [n_segs] pool slot of the partition's first player (its first chunk * kTile)
  BinMap bm;
  const uint8_t* grp_lut;
  const uint16_t* bin_seg;
  const uint32_t* seg_bin_lo;
  const uint8_t* mode_tsize;
  uint32_t n_modes;
  uint32_t seq_next;
  uint64_t id_limit;  // ids >= id_limit are invalid (the handle range, or the hashed set's reserved keys)
  uint32_t* err;
};

// Image player i as k_img_load and k_mrg_order check it.  p: its partition, the last whose first index in s_off is
// <= i (empty ones share it); u: its enqueue order, the distance of its sequence number above seq_next (0 is seq_next
// itself); bin: its sort key (valid when bad has no kImgBadMode); bad: the kImg* bits of the checks it fails.
struct ImgPlayer {
  uint64_t pid;
  int32_t rt;
  uint32_t p, md, u, bin, bad;
};
__device__ __forceinline__ ImgPlayer img_player(const ImgCols& in, uint32_t i, const uint32_t* s_off, uint32_t n_segs,
                                                const BinMap& bm, const uint8_t* grp_lut, const uint16_t* bin_seg,
                                                uint32_t n_modes, uint32_t seq_next, uint64_t id_limit) {
  ImgPlayer q;
  q.p = last_le(s_off, 0, n_segs, i);
  q.pid = img_id(in, i);
  q.md = in.mode[i];
  q.rt = in.rating[i];
  q.u = in.seq[i] - seq_next;
  q.bin = 0;
  q.bad = 0;
  if (q.pid >= id_limit) q.bad |= kImgBadId;
  if (q.md >= n_modes) {
    q.bad |= kImgBadMode;
  } else {
    q.bin = bin_of(bm, bm.lut, q.rt, q.md);
    if (grp_lut[clamp_key(bm.key_lo, bm.KR, q.rt)] == 0xFF || bin_seg[q.bin] != q.p) q.bad |= kImgBadRating;
  }
  if (q.u == 0 || (i + 1 < s_off[q.p + 1] && in.seq[i + 1] - seq_next <= q.u)) q.bad |= kImgBadSeq;
  return q;
}

// One image player per thread: check it, then write its slot (nothing is written for a player that fails a check).
__global__ void __launch_bounds__(256) k_img_load(const ImgLoadArgs a) {
  __shared__ uint32_t s_off[kMaxSegs + 1], s_base[kMaxSegs];
  for (uint32_t p = threadIdx.x; p <= a.n_segs; p += blockDim.x) {
    s_off[p] = a.part_off[p];
    if (p < a.n_segs) s_base[p] = a.slot_base[p];
  }
  __syncthreads();
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
    const ImgPlayer q =
        img_player(a.in, i, s_off, a.n_segs, a.bm, a.grp_lut, a.bin_seg, a.n_modes, a.seq_next, a.id_limit);
    if (q.bad) { atomicOr(a.err, q.bad); continue; }
    const uint32_t slot = s_base[q.p] + (i - s_off[q.p]);
    a.pool.id[slot] = q.pid; a.pool.rating[slot] = q.rt; a.pool.mode[slot] = (uint8_t)q.md;
    a.pool.tsize[slot] = a.mode_tsize[q.md]; a.pool.ts[slot] = a.in.ts[i];
    a.pool.bin[slot] = (uint16_t)q.bin; a.pool.seq[slot] = a.in.seq[i];
    atomicAdd(&a.meta.tot[q.bin], 1u);
    if (a.meta.chist) atomicAdd(&a.meta.chist[(size_t)(slot / kTile) * kChunkHist + (q.bin - a.seg_bin_lo[q.p])], 1u);
  }
}

// Ids of an image section into an empty active set with value kPtMatched ("active, not queued"); a second copy of an
// id — in the same section or the other — sets kImgDup.
__global__ void k_img_insert(const void* ids, uint32_t id_bytes, uint32_t n, uint64_t id_limit, ActiveView act,
                             uint32_t* __restrict__ err) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint64_t pid = id_bytes == 8 ? static_cast<const uint64_t*>(ids)[i] : static_cast<const uint32_t*>(ids)[i];
    if (pid >= id_limit) { atomicOr(err, kImgBadId); continue; }
    if (act.dcap) {
      if (atomicCAS(act.val(pid), kFreeVal, (unsigned long long)kPtMatched) != kFreeVal) atomicOr(err, kImgDup);
      continue;
    }
    uint64_t h = hash64(pid) & act.mask;
    bool placed = false;
    for (uint64_t probe = 0; probe <= act.mask && !placed; ++probe) {
      unsigned long long k = *act.key(h);
      if (k == kEmptyKey) {
        k = atomicCAS(act.key(h), kEmptyKey, (unsigned long long)pid);
        if (k == kEmptyKey) { *act.val(h) = kPtMatched; placed = true; break; }
      }
      if (k == pid) { atomicOr(err, kImgDup); placed = true; break; }
      h = (h + 1) & act.mask;
    }
    if (!placed) atomicOr(err, kImgFull);
  }
}

// ---- mm_merge: a queue image (mm_export_queues) into a running engine, through the ingest ----------------------------
// k_mrg_order checks every image player (as k_img_load) and writes the ingest batch: the players of each (mode, group)
// queue in the source's enqueue order.  A queue's partitions are consecutive in the image and each is sorted by
// sequence number, so a player's position in its queue is its index in its partition plus, for every other partition
// of the queue, the number of that partition's players enqueued before it (a binary search; equal numbers from a
// crafted image are ordered by partition, so the positions stay a permutation).  src[pos] = the image index.
struct MrgOrderArgs {
  ImgCols in;
  uint32_t n, n_segs;
  const uint32_t* part_off;   // [n_segs + 1] first image index of the partition
  const uint16_t* part_cut;   // [n_segs] partition -> (mode, group) queue
  const uint32_t* cut_lp_lo;  // [n_cut + 1] first partition of the queue
  BinMap bm;
  const uint8_t* grp_lut;
  const uint16_t* bin_seg;
  uint32_t n_modes, seq_next;
  uint64_t id_limit;
  uint64_t* out_id;  // the ingest batch columns
  int32_t* out_rating;
  uint8_t* out_mode;
  uint32_t* out_ts;
  uint32_t* src;
  uint32_t* err;
};

__global__ void __launch_bounds__(256) k_mrg_order(const MrgOrderArgs a) {
  __shared__ uint32_t s_off[kMaxSegs + 1];
  for (uint32_t p = threadIdx.x; p <= a.n_segs; p += blockDim.x) s_off[p] = a.part_off[p];
  __syncthreads();
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
    const ImgPlayer x =
        img_player(a.in, i, s_off, a.n_segs, a.bm, a.grp_lut, a.bin_seg, a.n_modes, a.seq_next, a.id_limit);
    if (x.bad) { atomicOr(a.err, x.bad); continue; }
    const uint32_t p = x.p, c = a.part_cut[p], q0 = a.cut_lp_lo[c], q1 = a.cut_lp_lo[c + 1];
    uint32_t pos = s_off[q0] + (i - s_off[p]);
    for (uint32_t q = q0; q < q1; ++q) {
      if (q == p) continue;
      // players of q enqueued before i: u' < u (u' <= u for q < p)
      pos += first_not(s_off[q], s_off[q + 1], [&](uint32_t k) {
               const uint32_t v = a.in.seq[k] - a.seq_next;
               return v < x.u || (q < p && v == x.u);
             }) - s_off[q];
    }
    a.out_id[pos] = x.pid; a.out_rating[pos] = x.rt; a.out_mode[pos] = (uint8_t)x.md; a.out_ts[pos] = a.in.ts[i];
    a.src[pos] = i;
  }
}

// Only when the caller's reject list or a capacity might be too small: the exact number of batch entries the ingest
// will not queue — ids already in the active set, and every copy of an id after the first (one copy wins the insert
// into `seen`, an empty scratch set of 2^k keys, at most half full).
__global__ void k_mrg_dups(const uint64_t* __restrict__ id, uint32_t n, ActiveView act, unsigned long long* seen,
                           uint64_t seen_mask, uint32_t* __restrict__ count) {
  uint32_t dup = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint64_t pid = id[i];
    const uint64_t h = act_find(act, pid);
    if (h != ~0ull && (!act.dcap || *act.val(h) != kFreeVal)) { ++dup; continue; }
    if (!seen_insert(seen, seen_mask, pid)) ++dup;
  }
  dup = __reduce_add_sync(0xFFFFFFFFu, dup);
  if ((threadIdx.x & 31) == 0 && dup) atomicAdd(count, dup);
}

// the batch entries the ingest did not queue -> their image indices (unordered)
__global__ void k_mrg_rejects(uint32_t n, const uint8_t* __restrict__ code, const uint32_t* __restrict__ src,
                              uint32_t* __restrict__ out, uint32_t* __restrict__ count) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool rej = i < n && code[i] != 1;
  const uint32_t at = warp_append(count, rej);
  if (rej) out[at] = src[i];
}

}  // namespace mm
