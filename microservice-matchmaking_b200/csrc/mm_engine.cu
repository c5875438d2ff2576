// mm_engine.cu — C ABI of the H100 opponent-search engine (include/mm_engine.h).
//
// Host side of the drop-in for the reference search stage
// (matchmaking/lib/search/worker.ex + models/{active_user,lobby_state}.ex).  The pool
// is a GPU-resident SoA (player_id u64 / rating i32 / game-mode u8 / team-size u8 /
// enqueue-time u32 + derived sort key u16 + enqueue sequence u32), segmented by
// (mode, rating group) partition into chunk lists, enqueue order kept inside a partition;
// all matching work runs in the kernels of mm_kernels.cuh.  There is no CPU path: every
// entry point either launches CUDA work or fails with MM_E_CUDA.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <vector>

#include "mm_kernels.cuh"
#include "mm_stats.cuh"

using namespace mm;

namespace {

struct Pool {
  PoolView v{};
  PoolMeta m{};
  uint32_t n = 0;  // host mirror of the sum of the partition fills (dead players included)
};

struct Table {
  unsigned long long* kv = nullptr;  // hashed: hcap x {key, value}; direct: dcap values
};

}  // namespace

struct mm_engine {
  mm_config cfg{};
  std::mutex mu;
  int device = 0;
  int n_sms = 0;
  int clock_khz = 0;  // peak SM clock (MM_TRACE: placement stall cycles -> µs)
  size_t smem_optin = 0, smem_sm = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = true;
  cudaStream_t copy_stream = nullptr;  // H2D of ingest chunks, overlapped with the ingest kernels
  cudaEvent_t ev_copy = nullptr;
  cudaStream_t d2h_stream = nullptr;   // async_results: a tick's host copies, overlapped with the next ingest
  bool async_results = false, results_pending = false;
  bool last_packed = false;  // the pending host copies read only d_hdr / d_members32
  cudaEvent_t ev[5]{};  // tick start | after hist | after colscan | after place | after epilogue
  char last_err[512] = {0};

  // key domain
  int32_t key_lo = 0;
  uint32_t KR = 0, stride = 0, K = 0, Kp = 0;
  uint32_t n_segs = 0;  // layout partitions (see build_tables)
  uint32_t n_cut = 0;   // (mode, group) cut segments
  uint16_t* d_part_cut = nullptr;   // [n_segs] partition -> cut segment
  uint32_t* d_cut_lp_lo = nullptr;  // [n_cut + 1] first partition of the cut segment
  uint16_t* d_lut = nullptr;
  uint8_t* d_grp_lut = nullptr;
  uint8_t* d_mode_tsize = nullptr;
  uint32_t* d_seg_bin_lo = nullptr;
  uint32_t* d_seg_L = nullptr;
  uint16_t* d_bin_seg = nullptr;  // [Kp] bin -> (mode, group) segment
  uint32_t min_L = 1;
  uint32_t max_nb = 1;  // most sort keys any one (mode, group) partition has

  // pool (double buffered) + snapshot
  uint32_t capacity = 0;
  uint32_t n_chunks = 0;  // physical chunks per pool buffer
  Pool pool[2];
  int cur = 0;
  uint32_t gen = 1;
  uint32_t seq_next = 0;  // enqueue sequence number of the next batch's first entry
  Pool snap;
  uint32_t snap_gen = 0, snap_seq = 0;
  bool has_snap = false;

  // active set
  bool use_active = true, dense_ids = false;
  uint64_t hcap = 0;  // hashed: slots (power of two); direct: handle capacity
  Table tab[2];
  int tcur = 0;
  uint64_t n_active = 0, n_tomb = 0;

  // tick scratch
  uint32_t R = 0;        // row CTAs of a tick
  uint32_t helpers = 0;  // extra CTAs of the fused launch: the tail, then the compacted pool's chunk histograms
  int rows_per_sm = 2;
  int rank_impl = 3;           // 3 = ballot tile sort for partitions of <= 255 bins + lists otherwise; 2 = lists only
  uint32_t place_stages = 0;
  int fused_ok = 0;  // k_tick<512> can be launched cooperatively with R CTAs
  int tick_impl = 1; // 1 = one fused cooperative launch when possible, 0 = four launches
  size_t tick_smem = 0;
  uint32_t *d_M = nullptr, *d_P = nullptr;  // row histograms, their column prefixes (only for many-row partitions)
  uint32_t *d_outbase = nullptr, *d_binlim = nullptr;
  uint16_t* d_bin_key = nullptr;
  int32_t max_spread = -1;  // < 0: policy S0 (reference behaviour); >= 0: policy S1 (extension)
  SegInfo* d_seg = nullptr;
  uint32_t* d_left_bits = nullptr;  // one bit per virtual pool position: stays queued after the tick
  uint64_t* d_members = nullptr;
  uint32_t* d_members32 = nullptr;  // mm_tick_packed: member handles narrowed for the host copy
  // async_results + mm_tick_packed: headers and narrowed handles alternate between two buffer sets, so the next
  // tick's kernels need not wait for this tick's host copies
  uint32_t* d_members32_alt = nullptr;
  mm_lobby_hdr* d_hdr_alt = nullptr;
  uint32_t* d_src_idx = nullptr;
  mm_lobby_hdr* d_hdr = nullptr;
  uint32_t* d_emit_seq = nullptr;
  uint32_t max_lobbies = 0;
  TickCtr* d_ctr2 = nullptr;  // two counter blocks, used alternately (the fused kernel re-arms the other one)
  TickCtr* d_ctr = nullptr;   // the block of the current / last tick
  int ctr_idx = 0;
  TickCtr* h_ctr = nullptr;  // pinned

  // enqueue scratch (grown on demand)
  uint32_t enq_cap = 0;
  uint64_t *d_in_id = nullptr, *d_hslot = nullptr;
  int32_t* d_in_rating = nullptr;
  uint8_t *d_in_mode = nullptr, *d_code = nullptr;
  uint16_t *d_part = nullptr, *d_in_key = nullptr;
  uint32_t *d_in_ts = nullptr, *d_in_handle = nullptr, *d_blocksum = nullptr, *d_blockhist = nullptr;
  uint32_t* d_small = nullptr;  // [0] accepted  [1] rejected: pool full  [2] removed  [3] running winner total (cut)
  uint32_t* h_small = nullptr;  // pinned
  uint32_t last_batch_n = 0;    // entries of the last ingest batch (their codes are still in d_code)
  uint32_t* d_rej_idx = nullptr; uint8_t* d_rej_code = nullptr; uint32_t rej_cap = 0;

  // mm_enqueue_packed_begin / _end: two staging slots for packed batches whose upload is in flight (FIFO)
  struct Stage {
    uint32_t *handle = nullptr, *ts = nullptr;
    uint16_t* key = nullptr;
    uint32_t cap = 0, n = 0;
    bool has_ts = false;
    cudaEvent_t ready = nullptr;  // recorded on the copy stream behind the slot's last copy
  } stage[2];
  int stage_head = 0, stage_count = 0;

  // last tick
  mm_tick_stats last{};
  bool last_fused = false;

  // mm_queue_stats: the match section reads pool[cur ^ 1] + d_left_bits, which describe the last tick until the next
  // one starts (its phase A writes the compacted pool's layout into pool[cur ^ 1].m)
  bool match_valid = false;  // the last tick completed and nothing since has invalidated its section
  uint32_t tick_now = 0;     // `now` of the tick in progress / the last tick (mod 2^32)
  uint32_t match_n = 0;      // players resident when that tick started: bounds its tile count
  uint32_t* d_qstat = nullptr;  // [n_cut] records
};

namespace {


int fail(mm_engine* e, cudaError_t err, const char* what) {
  if (e) std::snprintf(e->last_err, sizeof(e->last_err), "%s: %s", what, cudaGetErrorString(err));
  cudaGetLastError();  // clear sticky-free errors
  return MM_E_CUDA;
}
#define CK(call)                                          \
  do {                                                    \
    cudaError_t _err = (call);                            \
    if (_err != cudaSuccess) return fail(e, _err, #call); \
  } while (0)

// Allow a kernel the device's whole opt-in shared memory (minus its static part).  Function attributes are
// process-global: an engine with a small key domain must never lower the limit another engine relies on.
template <class F>
cudaError_t allow_max_smem(const mm_engine* e, F* func) {
  cudaFuncAttributes fa{};
  cudaError_t err = cudaFuncGetAttributes(&fa, func);
  if (err != cudaSuccess) return err;
  return cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              (int)(e->smem_optin - fa.sharedSizeBytes));
}

size_t pool_slots(const mm_engine* e) { return (size_t)e->n_chunks * kTile; }

int alloc_pool(mm_engine* e, Pool& p) {
  const size_t c = pool_slots(e);
  CK(cudaMalloc(&p.v.id, c * 8));
  CK(cudaMalloc(&p.v.rating, c * 4));
  CK(cudaMalloc(&p.v.mode, c));
  CK(cudaMalloc(&p.v.tsize, c));
  CK(cudaMalloc(&p.v.ts, c * 4));
  CK(cudaMalloc(&p.v.bin, c * 2));
  CK(cudaMalloc(&p.v.seq, c * 4));
  p.m.max_ch = e->n_chunks;
  CK(cudaMalloc(&p.m.fill, (size_t)e->n_segs * 4));
  CK(cudaMalloc(&p.m.chunk_tab, (size_t)e->n_segs * e->n_chunks * 4));
  CK(cudaMalloc(&p.m.bump, 4));
  CK(cudaMalloc(&p.m.tot, ((size_t)e->Kp + 1) * 4));
  p.m.chist = nullptr;
  if (e->max_nb <= kFastBins) {  // per-chunk key histograms: the tick skips its counting pass over the pool
    CK(cudaMalloc(&p.m.chist, (size_t)e->n_chunks * kChunkHist * 4));
    CK(cudaMemset(p.m.chist, 0, (size_t)e->n_chunks * kChunkHist * 4));
  }
  CK(cudaMemset(p.m.tot, 0, ((size_t)e->Kp + 1) * 4));
  CK(cudaMemset(p.m.fill, 0, (size_t)e->n_segs * 4));
  CK(cudaMemset(p.m.bump, 0, 4));
  // chunks are read whole by the TMA tiles: keep the bin column defined (and "dead") past the fills
  CK(cudaMemset(p.v.bin, 0xFF, c * 2));
  p.n = 0;
  return MM_OK;
}
void free_pool(Pool& p) {
  cudaFree(p.v.id); cudaFree(p.v.rating); cudaFree(p.v.mode); cudaFree(p.v.tsize); cudaFree(p.v.ts); cudaFree(p.v.bin);
  cudaFree(p.v.seq); cudaFree(p.m.fill); cudaFree(p.m.chunk_tab); cudaFree(p.m.bump); cudaFree(p.m.tot); cudaFree(p.m.chist);
  p = Pool{};
}
int copy_pool(mm_engine* e, Pool& dst, const Pool& src) {
  const size_t c = pool_slots(e);
  CK(cudaMemcpyAsync(dst.v.id, src.v.id, c * 8, cudaMemcpyDeviceToDevice, e->stream));
  CK(cudaMemcpyAsync(dst.v.rating, src.v.rating, c * 4, cudaMemcpyDeviceToDevice, e->stream));
  CK(cudaMemcpyAsync(dst.v.mode, src.v.mode, c, cudaMemcpyDeviceToDevice, e->stream));
  CK(cudaMemcpyAsync(dst.v.tsize, src.v.tsize, c, cudaMemcpyDeviceToDevice, e->stream));
  CK(cudaMemcpyAsync(dst.v.ts, src.v.ts, c * 4, cudaMemcpyDeviceToDevice, e->stream));
  CK(cudaMemcpyAsync(dst.v.bin, src.v.bin, c * 2, cudaMemcpyDeviceToDevice, e->stream));
  CK(cudaMemcpyAsync(dst.v.seq, src.v.seq, c * 4, cudaMemcpyDeviceToDevice, e->stream));
  CK(cudaMemcpyAsync(dst.m.fill, src.m.fill, (size_t)e->n_segs * 4, cudaMemcpyDeviceToDevice, e->stream));
  CK(cudaMemcpyAsync(dst.m.chunk_tab, src.m.chunk_tab, (size_t)e->n_segs * e->n_chunks * 4, cudaMemcpyDeviceToDevice, e->stream));
  CK(cudaMemcpyAsync(dst.m.bump, src.m.bump, 4, cudaMemcpyDeviceToDevice, e->stream));
  CK(cudaMemcpyAsync(dst.m.tot, src.m.tot, ((size_t)e->Kp + 1) * 4, cudaMemcpyDeviceToDevice, e->stream));
  if (src.m.chist)
    CK(cudaMemcpyAsync(dst.m.chist, src.m.chist, (size_t)e->n_chunks * kChunkHist * 4, cudaMemcpyDeviceToDevice, e->stream));
  dst.n = src.n;
  return MM_OK;
}

ActiveView act_view(mm_engine* e) {
  ActiveView a{};
  if (e->use_active) {
    a.kv = e->tab[e->tcur].kv;
    if (e->dense_ids) a.dcap = e->hcap;
    else a.mask = e->hcap - 1;
  }
  return a;
}

int clear_table(mm_engine* e, Table& t) {
  if (e->dense_ids) {
    CK(cudaMemsetAsync(t.kv, 0xFF, e->hcap * 8, e->stream));  // FREE = all ones
    return MM_OK;
  }
  k_fill_kv<<<1024, 256, 0, e->stream>>>(reinterpret_cast<ulonglong2*>(t.kv), e->hcap, kEmptyKey, kFreeVal);
  CK(cudaGetLastError());
  return MM_OK;
}

// generic/worker.ex:46-53 on the host (also exported as mm_group_of)
int group_of(const mm_config* cfg, int64_t rating) {
  for (uint32_t g = 0; g < cfg->n_groups; ++g)
    if (rating >= cfg->group_lo[g] && rating <= cfg->group_hi[g]) return (int)g;
  return cfg->default_group;
}

int check_config(const mm_config* c) {
  if (!c || c->abi_version != MM_ABI_VERSION) return MM_E_ARG;
  if (c->n_groups == 0 || c->n_groups > MM_MAX_GROUPS || c->n_modes == 0 || c->n_modes > MM_MAX_MODES) return MM_E_ARG;
  if (c->default_group >= (int32_t)c->n_groups || c->default_group < -1) return MM_E_ARG;
  if (c->order_mode > MM_ORDER_RATING) return MM_E_ARG;
  if (c->capacity == 0 || c->capacity > 0x7FFF0000u) return MM_E_ARG;
  if (c->flags & ~(MM_F_NO_DEDUPE | MM_F_DENSE_IDS | MM_F_WIDE_PARTITIONS)) return MM_E_ARG;
  for (uint32_t g = 0; g < c->n_groups; ++g) {
    if (c->group_lo[g] > c->group_hi[g]) return MM_E_ARG;
    if (c->group_lo[g] < -(1 << 30) || c->group_hi[g] > (1 << 30)) return MM_E_ARG;
  }
  for (uint32_t m = 0; m < c->n_modes; ++m) {
    const uint32_t L = (uint32_t)c->modes[m].teams * c->modes[m].team_size;
    if (L == 0 || L > 65535u || c->modes[m].team_size > 255) return MM_E_ARG;
  }
  return MM_OK;
}

// Shared-memory layout of the scan tail: everything on chip up to ~100 KB (so that it never exceeds the placement
// phase's footprint in the fused kernel), else keys from global memory, else matched counts parked in global too.
uint32_t tail_layout(const mm_engine* e) {
  if ((size_t)tail_words(e->Kp, 3) * 4 <= 100 * 1024) return 3;
  if ((size_t)tail_words(e->Kp, 1) * 4 + 1024 <= e->smem_optin) return 1;
  return 0;
}
size_t colscan_smem(const mm_engine* e) {
  return (size_t)std::max<uint32_t>(kColScratchWords, tail_words(e->Kp, tail_layout(e))) * 4;
}

// Build the key -> bin LUT and the (mode, group) segment table (see mm_kernels.cuh).
int build_tables(mm_engine* e) {
  const mm_config& c = e->cfg;
  int32_t rmin = c.group_lo[0], rmax = c.group_hi[0];
  for (uint32_t g = 1; g < c.n_groups; ++g) { rmin = std::min(rmin, c.group_lo[g]); rmax = std::max(rmax, c.group_hi[g]); }
  e->key_lo = rmin - 1;
  const uint64_t KR64 = (uint64_t)((int64_t)rmax - rmin + 3);
  if (KR64 > 65535u) return MM_E_ARG;  // rating span must fit the 16-bit LUT
  e->KR = (uint32_t)KR64;
  const uint32_t G = c.n_groups;
  std::vector<uint8_t> grp(e->KR);
  for (uint32_t k = 0; k < e->KR; ++k) {
    const int g = group_of(&c, (int64_t)e->key_lo + k);
    grp[k] = g < 0 ? 0xFF : (uint8_t)g;
  }
  std::vector<uint16_t> lut(e->KR, 0);
  std::vector<uint32_t> first(G + 1, 0);
  std::vector<uint16_t> key_of;  // rating order: bin (inside a mode) -> clamp key
  if (c.order_mode == MM_ORDER_RATING) {
    // bins ordered by (group, clamp key): the partition of a group is its keys ascending
    uint32_t next = 0;
    for (uint32_t g = 0; g < G; ++g) {
      first[g] = next;
      for (uint32_t k = 0; k < e->KR; ++k)
        if (grp[k] == g) { lut[k] = (uint16_t)next++; key_of.push_back((uint16_t)k); }
    }
    first[G] = next;
    e->stride = std::max(next, 1u);
  } else {
    for (uint32_t k = 0; k < e->KR; ++k) lut[k] = grp[k] == 0xFF ? 0 : grp[k];
    for (uint32_t g = 0; g <= G; ++g) first[g] = g;
    e->stride = G;
  }
  e->K = c.n_modes * e->stride;
  e->Kp = e->K + 1;
  if (e->Kp > 65535u) return MM_E_ARG;  // the resident sort key is 16 bits
  // Layout partitions: a (mode, group) CUT SEGMENT — the unit of the lobby cut — is stored as one or more PARTITIONS
  // of at most kFastBins consecutive sort keys each, so that every tile ranks on the 8-bit path and carries a chunk
  // histogram whatever the width of the rating group (the reference's default groups span 500 - 1 500 ratings,
  // config/config.exs:27-36).  Narrow groups: one partition per segment.
  e->n_cut = c.n_modes * G;
  std::vector<uint32_t> seg_lo, seg_L, cut_lp_lo(e->n_cut + 1);
  std::vector<uint16_t> part_cut;
  e->min_L = 0xFFFFFFFFu;
  std::vector<uint8_t> tsz(MM_MAX_MODES, 0);
  bool split = !(c.flags & MM_F_WIDE_PARTITIONS);
  for (int attempt = 0; attempt < 2; ++attempt) {
    seg_lo.clear(); seg_L.clear(); part_cut.clear();
    for (uint32_t m = 0; m < c.n_modes; ++m) {
      const uint32_t L = (uint32_t)c.modes[m].teams * c.modes[m].team_size;
      e->min_L = std::min(e->min_L, L);
      tsz[m] = (uint8_t)c.modes[m].team_size;
      for (uint32_t g = 0; g < G; ++g) {
        const uint32_t lo = m * e->stride + first[g], nk = first[g + 1] - first[g];
        const uint32_t nsub = split ? std::max(1u, (nk + kFastBins - 1) / kFastBins) : 1u;
        const uint32_t per = (nk + nsub - 1) / nsub;
        cut_lp_lo[m * G + g] = (uint32_t)seg_lo.size();
        for (uint32_t j = 0; j < nsub; ++j) {
          seg_lo.push_back(lo + std::min(nk, j * per)); seg_L.push_back(L); part_cut.push_back((uint16_t)(m * G + g));
        }
      }
    }
    if (seg_lo.size() <= kMaxSegs) break;
    split = false;  // too many partitions for the on-chip tables: whole segments, list ranking for the wide ones
  }
  e->n_segs = (uint32_t)seg_lo.size();
  if (e->n_segs > kMaxSegs) return MM_E_ARG;
  cut_lp_lo[e->n_cut] = e->n_segs;
  seg_lo.push_back(e->K);
  e->max_nb = 1;
  for (uint32_t sgi = 0; sgi < e->n_segs; ++sgi) e->max_nb = std::max(e->max_nb, seg_lo[sgi + 1] - seg_lo[sgi]);
  std::vector<uint16_t> bin_seg(e->Kp, 0);
  for (uint32_t sgi = 0; sgi < e->n_segs; ++sgi)
    for (uint32_t b = seg_lo[sgi]; b < seg_lo[sgi + 1]; ++b) bin_seg[b] = (uint16_t)sgi;
  CK(cudaMalloc(&e->d_part_cut, e->n_segs * 2));
  CK(cudaMemcpy(e->d_part_cut, part_cut.data(), e->n_segs * 2, cudaMemcpyHostToDevice));
  CK(cudaMalloc(&e->d_cut_lp_lo, (e->n_cut + 1) * 4));
  CK(cudaMemcpy(e->d_cut_lp_lo, cut_lp_lo.data(), (e->n_cut + 1) * 4, cudaMemcpyHostToDevice));
  std::vector<uint16_t> bin_key(e->Kp, 0);
  if (!key_of.empty())
    for (uint32_t b = 0; b < e->K; ++b) bin_key[b] = key_of[b % e->stride];
  CK(cudaMalloc(&e->d_bin_seg, e->Kp * 2));
  CK(cudaMemcpy(e->d_bin_seg, bin_seg.data(), e->Kp * 2, cudaMemcpyHostToDevice));
  CK(cudaMalloc(&e->d_bin_key, e->Kp * 2));
  CK(cudaMemcpy(e->d_bin_key, bin_key.data(), e->Kp * 2, cudaMemcpyHostToDevice));
  CK(cudaMalloc(&e->d_lut, e->KR * 2));
  CK(cudaMalloc(&e->d_grp_lut, e->KR));
  CK(cudaMalloc(&e->d_mode_tsize, MM_MAX_MODES));
  CK(cudaMalloc(&e->d_seg_bin_lo, (e->n_segs + 1) * 4));
  CK(cudaMalloc(&e->d_seg_L, e->n_segs * 4));
  CK(cudaMemcpy(e->d_lut, lut.data(), e->KR * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(e->d_grp_lut, grp.data(), e->KR, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(e->d_mode_tsize, tsz.data(), MM_MAX_MODES, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(e->d_seg_bin_lo, seg_lo.data(), (e->n_segs + 1) * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(e->d_seg_L, seg_L.data(), e->n_segs * 4, cudaMemcpyHostToDevice));
  return MM_OK;
}

BinMap bin_map(const mm_engine* e) {
  BinMap b{};
  b.lut = e->d_lut; b.key_lo = e->key_lo; b.KR = e->KR; b.stride = e->stride; b.K = e->K;
  return b;
}

int alloc_tick_scratch(mm_engine* e) {
  uint32_t total = (uint32_t)e->n_sms * (uint32_t)e->rows_per_sm;
  if (total > kMaxRows) total = kMaxRows;
  e->helpers = total >= 64 ? 4u : (total > 1 ? 1u : 0u);
  e->R = total - e->helpers;
  if (e->d_M) { cudaFree(e->d_M); cudaFree(e->d_P); }
  CK(cudaMalloc(&e->d_M, (size_t)(e->R + 1) * e->Kp * 4));
  CK(cudaMalloc(&e->d_P, (size_t)(e->R + 1) * e->Kp * 4));
  return MM_OK;
}

int ensure_enq_scratch(mm_engine* e, uint32_t n) {
  if (n <= e->enq_cap) return MM_OK;
  cudaFree(e->d_in_id); cudaFree(e->d_hslot); cudaFree(e->d_in_rating); cudaFree(e->d_in_mode);
  cudaFree(e->d_code); cudaFree(e->d_in_ts); cudaFree(e->d_blocksum); cudaFree(e->d_part); cudaFree(e->d_in_key);
  cudaFree(e->d_in_handle);
  e->enq_cap = 0;
  const size_t c = (size_t)n + 64;
  CK(cudaMalloc(&e->d_in_id, c * 8));
  CK(cudaMalloc(&e->d_hslot, c * 8));
  CK(cudaMalloc(&e->d_in_rating, c * 4));
  CK(cudaMalloc(&e->d_in_mode, c));
  CK(cudaMalloc(&e->d_code, c));
  CK(cudaMalloc(&e->d_part, c * 2));
  CK(cudaMalloc(&e->d_in_key, c * 2));
  CK(cudaMalloc(&e->d_in_handle, c * 4));
  CK(cudaMalloc(&e->d_in_ts, c * 4));
  CK(cudaMalloc(&e->d_blocksum, (std::min<size_t>(c, kEnqChunkDev) / 256 + 2) * 4));
  e->enq_cap = n;
  return MM_OK;
}

// Drop tombstones: re-insert the committed entries into the spare table (hashed mode).
int rehash(mm_engine* e) {
  Table& nt = e->tab[e->tcur ^ 1];
  int rc = clear_table(e, nt);
  if (rc) return rc;
  ActiveView oldv = act_view(e), newv{};
  newv.kv = nt.kv; newv.mask = e->hcap - 1;
  k_rehash<<<2048, 256, 0, e->stream>>>(oldv, newv);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(e->stream));
  e->tcur ^= 1;
  e->n_tomb = 0;
  return MM_OK;
}

// capacity checks + scratch for an ingest batch of n players
int enq_prepare(mm_engine* e, uint32_t n) {
  int rc = ensure_enq_scratch(e, n);
  if (rc) return rc;
  if (e->use_active && !e->dense_ids && (e->n_active + e->n_tomb + n) * 4 > e->hcap * 3) {
    if ((e->n_active + n) * 4 > e->hcap * 3) {
      std::snprintf(e->last_err, sizeof(e->last_err), "active set full: %llu ids resident, batch of %u, capacity %llu",
                    (unsigned long long)e->n_active, n, (unsigned long long)(e->hcap * 3 / 4));
      return MM_E_CAP;
    }
    if ((rc = rehash(e))) return rc;
  }
  CK(cudaMemsetAsync(e->d_small, 0, 16, e->stream));
  return MM_OK;
}

// one ingest chunk = batch indices [base, base + cnt): claim, (exact capacity cut), route, alloc, append
int enq_chunk(mm_engine* e, uint32_t base, uint32_t cnt, const uint64_t* id, const int32_t* rating, const uint8_t* mode,
              const uint32_t* ts, bool may_overflow) {
  Pool& p = e->pool[e->cur];
  ActiveView av = act_view(e);
  const uint32_t nb = (cnt + 255) / 256, nblk = (cnt + kIngestItems - 1) / kIngestItems;
  k_enq_claim<<<nb, 256, 0, e->stream>>>(base, cnt, id, rating, mode, e->d_grp_lut, e->key_lo, e->KR, e->cfg.n_modes,
                                         bin_map(e), e->d_bin_seg, av, e->d_hslot, e->d_code, e->d_part);
  if (may_overflow) {  // the batch might not fit: the winners past the pool capacity are rolled back (code 3)
    const uint32_t room = e->capacity > p.n ? e->capacity - p.n : 0u;
    k_enq_count<<<nb, 256, 0, e->stream>>>(base, cnt, av, e->d_hslot, e->d_code, e->d_blocksum);
    k_scan_small<<<1, 1024, 0, e->stream>>>(nb, e->d_blocksum, e->d_small + 3);
    k_enq_cut<<<nb, 256, 0, e->stream>>>(base, cnt, av, e->d_hslot, e->d_code, e->d_blocksum, room, e->d_small + 1);
  }
  k_enq_route<<<nblk, 256, 0, e->stream>>>(base, cnt, av, e->d_hslot, e->d_code, e->d_part, e->n_segs, nblk, e->d_blockhist);
  k_enq_alloc<<<1, 512, 0, e->stream>>>(e->n_segs, nblk, e->d_blockhist, p.m, e->d_small);
  const size_t smem = (size_t)(2 * e->n_segs + 64) * 4 + (size_t)(((8 * (e->n_segs + 1) + 1) & ~1u) + 2 * kIngestItems) * 2;
  k_enq_append<<<nblk, 256, smem, e->stream>>>(base, cnt, id, rating, mode, ts, e->d_mode_tsize, av, e->d_hslot, e->d_code,
                                               e->d_part, e->n_segs, nblk, e->d_blockhist, p.v, p.m, e->gen, e->seq_next,
                                               bin_map(e), e->d_seg_bin_lo);
  CK(cudaGetLastError());
  return MM_OK;
}

// counters of the finished batch -> host state
int enq_finish(mm_engine* e, uint32_t n, uint8_t* accepted_dev, uint32_t* n_accepted) {
  Pool& p = e->pool[e->cur];
  CK(cudaMemcpyAsync(e->h_small, e->d_small, 16, cudaMemcpyDeviceToHost, e->stream));
  if (accepted_dev) CK(cudaMemcpyAsync(accepted_dev, e->d_code, n, cudaMemcpyDeviceToDevice, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  const uint32_t acc = e->h_small[0], rej = e->h_small[1];
  p.n += acc;
  e->seq_next += n;
  e->last_batch_n = n;
  if (e->use_active) { e->n_active += acc; if (!e->dense_ids) e->n_tomb += rej; }
  if (n_accepted) *n_accepted = acc;
  return MM_OK;
}

// Device columns of a whole batch -> pool.  `upload` (may be null) queues the H2D copies of one chunk on the copy
// stream: the previous chunk's kernels run on the engine stream meanwhile, so the device side of the ingest hides
// behind the PCIe transfer except for the last chunk.
template <class Upload>
int enqueue_batch(mm_engine* e, uint32_t n, const uint64_t* id, const int32_t* rating, const uint8_t* mode,
                  const uint32_t* ts, uint32_t chunk, Upload upload) {
  int rc = enq_prepare(e, n);
  if (rc) return rc;
  const bool may_overflow = (uint64_t)e->pool[e->cur].n + n > e->capacity;
  for (uint32_t base = 0; base < n; base += chunk) {
    const uint32_t cnt = std::min(chunk, n - base);
    if ((rc = upload(base, cnt))) return rc;
    if ((rc = enq_chunk(e, base, cnt, id, rating, mode, ts, may_overflow))) return rc;
  }
  return MM_OK;
}

TailArgs tail_args(mm_engine* e) {
  TailArgs t{};
  t.Kp = e->Kp; t.K = e->K; t.n_segs = e->n_segs; t.max_spread = e->max_spread; t.layout = tail_layout(e);
  t.tot = e->pool[e->cur].m.tot; t.seg_bin_lo = e->d_seg_bin_lo; t.seg_L = e->d_seg_L; t.bin_seg = e->d_bin_seg;
  t.n_cut = e->n_cut; t.part_cut = e->d_part_cut; t.cut_lp_lo = e->d_cut_lp_lo;
  t.bin_key = e->d_bin_key; t.outbase = e->d_outbase; t.binlim = e->d_binlim; t.seg = e->d_seg; t.ctr = e->d_ctr;
  t.fill = e->pool[e->cur].m.fill;
  t.dst = e->pool[e->cur ^ 1].m;
  return t;
}
// Rows (CTAs) a tick uses: small pools do not pay the grid barriers and per-row set-up of the full grid.  About two
// tiles per row at least; the tile count is bounded from the host-side player count.
uint32_t tick_rows(const mm_engine* e) {
  const uint64_t tiles = (uint64_t)e->pool[e->cur].n / kTile + e->n_segs;
  // helper CTAs run the tail beside the rows' histograms and clear the compacted pool's chunk histograms; the rows
  // write the lobby headers after placing (headers_claimed).  Small lobbies keep more helpers, at the rows' expense
  const uint32_t total = e->R + e->helpers;
  const uint32_t want = std::min(32u, std::max(e->helpers, (total * 14 / 100 + e->min_L - 1) / e->min_L));
  return (uint32_t)std::min<uint64_t>(total - want, std::max<uint64_t>(1, (tiles + 1) / 2));
}

PlaceArgs place_args(mm_engine* e, bool want_seq) {
  const Pool& p = e->pool[e->cur];
  PlaceArgs a{};
  a.bins16 = p.v.bin; a.ids = p.v.id; a.meta = p.m;
  a.K = e->K; a.Kp = e->Kp; a.R = tick_rows(e); a.stages = e->place_stages; a.fast_ok = e->rank_impl == 3; a.max_nb = e->max_nb;
  a.seg_bin_lo = e->d_seg_bin_lo; a.bin_seg = e->d_bin_seg; a.M = e->d_M; a.P = e->d_P;
  a.outbase = e->d_outbase; a.binlim = e->d_binlim; a.members = e->d_members;
  a.src_idx = want_seq ? e->d_src_idx : nullptr;
  a.left_bits = e->d_left_bits; a.ctr = e->d_ctr;
  return a;
}
uint32_t next_gen(const mm_engine* e) { return e->gen >= kGenMask ? 1u : e->gen + 1; }
EpiArgs epi_args(mm_engine* e, bool want_seq, bool headers) {
  EpiArgs a{};
  a.src = e->pool[e->cur].v; a.dst = e->pool[e->cur ^ 1].v;
  a.src_meta = e->pool[e->cur].m; a.dst_meta = e->pool[e->cur ^ 1].m;
  a.new_gen = next_gen(e); a.n_segs = e->n_segs; a.n_groups = e->cfg.n_groups;
  a.write_headers = headers ? 1u : 0u;
  a.act = act_view(e); a.seg = e->d_seg; a.seg_L = e->d_seg_L; a.part_cut = e->d_part_cut;
  a.seg_bin_lo = e->d_seg_bin_lo;
  a.hdr = e->d_hdr; a.src_idx = want_seq ? e->d_src_idx : nullptr; a.emit_seq = want_seq ? e->d_emit_seq : nullptr;
  a.ctr = e->d_ctr;
  return a;
}

// launches k_hist + k_colscan (phase A of a tick): the counters are final afterwards
int tick_phase_a(mm_engine* e) {
  const Pool& p = e->pool[e->cur];
  CK(cudaMemsetAsync(e->d_ctr, 0, sizeof(TickCtr), e->stream));
  CK(cudaEventRecord(e->ev[0], e->stream));
  const uint32_t rows = tick_rows(e);
  k_hist<512><<<rows, 512, hist_smem_bytes(e->max_nb), e->stream>>>(p.v.bin, p.m, e->n_segs, rows, e->Kp, e->max_nb, e->d_seg_bin_lo, e->d_M);
  CK(cudaEventRecord(e->ev[1], e->stream));
  k_colscan<<<(e->K + 31) / 32 + 1, kScanBlock, colscan_smem(e), e->stream>>>(rows, e->d_M, e->d_P, tail_args(e));
  CK(cudaGetLastError());
  return MM_OK;
}

int tick_phase_b(mm_engine* e, bool want_seq) {
  const uint32_t rows = tick_rows(e);
  if (e->pool[e->cur ^ 1].m.chist)  // the compacted pool's chunk histograms start empty (the fused tick's helper CTAs do this)
    CK(cudaMemsetAsync(e->pool[e->cur ^ 1].m.chist, 0, (size_t)e->n_chunks * kChunkHist * 4, e->stream));
  CK(cudaEventRecord(e->ev[2], e->stream));
  k_place<512><<<rows, 512, place_smem_bytes(e->max_nb, e->place_stages), e->stream>>>(
      place_args(e, want_seq), epi_args(e, want_seq, true), e->pool[e->cur].m.fill, e->n_segs);
  CK(cudaEventRecord(e->ev[3], e->stream));
  k_epilogue<512><<<std::max<uint32_t>(1, std::min<uint32_t>((uint32_t)e->n_sms, 2 * rows)), 512, 0, e->stream>>>(
      epi_args(e, want_seq, true), rows);
  CK(cudaGetLastError());
  CK(cudaEventRecord(e->ev[4], e->stream));
  CK(cudaMemcpyAsync(e->h_ctr, e->d_ctr, sizeof(TickCtr), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return MM_OK;
}

bool use_fused(const mm_engine* e) { return e->tick_impl == 1 && e->fused_ok; }

// the whole tick in one cooperative launch (k_tick)
int tick_fused(mm_engine* e, bool want_seq) {
  TickArgs a{};
  const uint32_t rows = tick_rows(e);
  // a grid that does not fill the GPU spends the spare CTA slots on helpers: at a few tiles per row the lobby headers
  // (one per L players) are as much work as the placement
  const uint32_t helpers = rows >= 64 ? std::min(32u, e->helpers + (e->R - rows)) : (rows > 1 ? 1u : 0u);
  a.src = e->pool[e->cur].v;
  a.R = rows;
  a.M = e->d_M;
  a.P = e->d_P;
  e->ctr_idx ^= 1;
  e->d_ctr = e->d_ctr2 + e->ctr_idx;  // armed (barrier / stamps zero) by the previous fused tick or by mm_create
  a.tail = tail_args(e);
  a.place = place_args(e, want_seq);
  a.place.trace = e->d_ctr->t;  // device address of the launch's time stamps (not dereferenced here)
  a.epi = epi_args(e, want_seq, want_seq);  // emission order needs every row's src_idx first: barrier 2
  a.next_ctr = e->d_ctr2 + (e->ctr_idx ^ 1);
  CK(cudaEventRecord(e->ev[0], e->stream));
  void* params[] = {&a};
  CK(cudaLaunchCooperativeKernel((const void*)k_tick<512>, dim3(rows + helpers), dim3(512), params, e->tick_smem, e->stream));
  CK(cudaEventRecord(e->ev[4], e->stream));
  CK(cudaMemcpyAsync(e->h_ctr, e->d_ctr, sizeof(TickCtr), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return MM_OK;
}

int tick_commit(mm_engine* e, uint32_t n, mm_tick_stats* stats) {
  const TickCtr& c = *e->h_ctr;
  mm_tick_stats st{};
  st.pool_before = n; st.n_lobbies = c.n_lobbies; st.n_matched = c.n_matched; st.n_residual = c.n_resid;
  st.n_dead = c.n_dead; st.n_launches = 4;
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, e->ev[0], e->ev[4]));
  st.device_us = ms * 1000.f;
  if (e->last_fused) {  // one launch: phase times from %globaltimer stamps of CTA 0
    st.n_launches = 1;
    st.hist_us = (float)(c.t[1] - c.t[0]) * 1e-3f;
    st.scan_us = (float)(c.t[2] - c.t[1]) * 1e-3f;
    st.place_us = (float)(c.t[3] - c.t[2]) * 1e-3f;     // until the last row has placed and compacted
    st.epilogue_us = (float)(c.t[6] - c.t[3]) * 1e-3f;  // headers and counter re-arm, until the last CTA is done
    if (std::getenv("MM_TRACE")) {
      // placement stalls: per half, averaged over the rows, at the device's peak SM clock
      const double us = 1e3 / ((double)e->clock_khz * tick_rows(e));
      // first_ranked / first_bases: the last row to rank its first tile / take that tile's slot bases (two
      // pipelines only; 0 = not stamped)
      auto at = [&](int k) { return c.t[k] ? (c.t[k] - c.t[0]) * 1e-3 : 0.0; };
      std::fprintf(stderr, "[mm] t0=0 rows_p1_done=%.1f tail_done=%.1f first_ranked=%.1f bar1=%.1f place_start=%.1f first_bases=%.1f"
                   " rows_place_done=%.1f rows_compact_done=%.1f end=%.1f us"
                   " | place stall/row hand full empty loop: h0 %.1f %.1f %.1f %.1f h1 %.1f %.1f %.1f %.1f us\n",
                   at(8), at(5), at(4), at(1), at(2), at(7), at(10), at(3), at(6),
                   c.stall[0][0] * us, c.stall[0][1] * us, c.stall[0][2] * us, c.stall[0][3] * us,
                   c.stall[1][0] * us, c.stall[1][1] * us, c.stall[1][2] * us, c.stall[1][3] * us);
    }
  } else {
    CK(cudaEventElapsedTime(&ms, e->ev[0], e->ev[1]));
    st.hist_us = ms * 1000.f;
    CK(cudaEventElapsedTime(&ms, e->ev[1], e->ev[2]));
    st.scan_us = ms * 1000.f;
    CK(cudaEventElapsedTime(&ms, e->ev[2], e->ev[3]));
    st.place_us = ms * 1000.f;
    CK(cudaEventElapsedTime(&ms, e->ev[3], e->ev[4]));
    st.epilogue_us = ms * 1000.f;
  }
  e->gen = next_gen(e);
  e->cur ^= 1;
  e->pool[e->cur].n = c.n_resid;
  e->match_valid = true;  // pool[cur ^ 1] is now the pool this tick matched
  e->match_n = n;
  e->last = st;
  if (stats) *stats = st;
  if (c.chist_bad) {  // placement took slot bases from chunk histograms that disagree with the pool: results are wrong
    std::snprintf(e->last_err, sizeof(e->last_err), "%u placement tiles disagree with their chunk histograms", c.chist_bad);
    return MM_E_STATE;
  }
  if (c.left_bad) {  // the compaction found leftovers beyond their partition's share of the compacted pool
    std::snprintf(e->last_err, sizeof(e->last_err), "%u leftover players fall outside their partition's compacted range", c.left_bad);
    return MM_E_STATE;
  }
  return MM_OK;
}

// Every tick entry point: the tick's `now` is kept for mm_queue_stats, and the last tick's match section is void from
// here on (a tick that fails after its phase A — MM_E_CAP on the split path — has rewritten pool[cur ^ 1].m).
void tick_begin(mm_engine* e, uint64_t now) {
  e->tick_now = (uint32_t)now;
  e->match_valid = false;
}

// async_results: the previous tick's host copies must land before its device buffers are overwritten
int wait_results(mm_engine* e) {
  if (e->results_pending) {
    CK(cudaStreamSynchronize(e->d2h_stream));
    e->results_pending = false;
  }
  return MM_OK;
}

// mm_tick / mm_tick_packed: run the tick and copy lobbies + members (u64 ids or u32 handles) to host buffers
int tick_to_host(mm_engine* e, mm_lobby_hdr* lobbies, uint32_t lobby_cap, uint64_t* member_ids, uint32_t* member_handles,
                 uint64_t member_cap, uint32_t* emit_seq, mm_tick_stats* stats) {
  const uint32_t n = e->pool[e->cur].n;
  const bool want_members = member_ids || member_handles;
  int rc;
  // The previous tick's host copies read d_hdr / d_members32 (packed) or d_members / d_emit_seq.  A packed tick
  // switches to the other buffer set and lets its kernels run beside those copies; otherwise wait for them first.
  const bool defer = e->async_results && e->results_pending && member_handles && !member_ids && !emit_seq &&
                     e->last_packed && e->d_hdr_alt && e->d_members32_alt;
  if (defer) {
    std::swap(e->d_hdr, e->d_hdr_alt);
    std::swap(e->d_members32, e->d_members32_alt);
  } else if ((rc = wait_results(e))) {
    return rc;
  }
  // worst-case output sizes known up front -> the fused single launch is safe
  e->last_fused = use_fused(e) && (!lobbies || (uint64_t)lobby_cap >= n / e->min_L) && (!want_members || member_cap >= n);
  if (e->last_fused) {
    if ((rc = tick_fused(e, emit_seq != nullptr))) return rc;
  } else {
    if ((rc = tick_phase_a(e))) return rc;
    // the counts are final after phase A: check the caller's capacities before consuming
    CK(cudaMemcpyAsync(e->h_ctr, e->d_ctr, sizeof(TickCtr), cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    if ((lobbies && e->h_ctr->n_lobbies > lobby_cap) || (want_members && e->h_ctr->n_matched > member_cap)) {
      std::snprintf(e->last_err, sizeof(e->last_err), "need lobby_cap >= %u, member_cap >= %u", e->h_ctr->n_lobbies,
                    e->h_ctr->n_matched);
      return MM_E_CAP;
    }
    if ((rc = tick_phase_b(e, emit_seq != nullptr))) return rc;
  }
  if ((rc = tick_commit(e, n, stats))) return rc;
  const TickCtr& c = *e->h_ctr;
  if (member_handles && c.n_matched) {
    if (!e->d_members32) CK(cudaMalloc(&e->d_members32, ((size_t)e->capacity + 64) * 4));
    k_narrow<<<std::max(1, 4 * e->n_sms), 256, 0, e->stream>>>(c.n_matched, e->d_members, e->d_members32);
    CK(cudaGetLastError());
    if (e->async_results) CK(cudaStreamSynchronize(e->stream));  // the copy stream must see the narrowed handles
  }
  if ((rc = wait_results(e))) return rc;  // (deferred case) the caller's host arrays of the previous tick are complete
  e->last_packed = member_handles && !member_ids && !emit_seq;
  // the tick is complete here (tick_commit synchronised the engine stream); with async_results the copies run on
  // their own stream and the call returns: the caller may ingest the next batch meanwhile (PCIe is full duplex)
  cudaStream_t cs = e->async_results ? e->d2h_stream : e->stream;
  if (lobbies && c.n_lobbies)
    CK(cudaMemcpyAsync(lobbies, e->d_hdr, (size_t)c.n_lobbies * sizeof(mm_lobby_hdr), cudaMemcpyDeviceToHost, cs));
  if (member_ids && c.n_matched)
    CK(cudaMemcpyAsync(member_ids, e->d_members, (size_t)c.n_matched * 8, cudaMemcpyDeviceToHost, cs));
  if (member_handles && c.n_matched)
    CK(cudaMemcpyAsync(member_handles, e->d_members32, (size_t)c.n_matched * 4, cudaMemcpyDeviceToHost, cs));
  if (emit_seq && c.n_lobbies)
    CK(cudaMemcpyAsync(emit_seq, e->d_emit_seq, (size_t)c.n_lobbies * 4, cudaMemcpyDeviceToHost, cs));
  if (e->async_results) { e->results_pending = true; return MM_OK; }
  CK(cudaStreamSynchronize(e->stream));
  return MM_OK;
}

}  // namespace

// =======================================================================================
extern "C" {

uint32_t mm_abi_version(void) { return MM_ABI_VERSION; }

const char* mm_strerror(int s) {
  switch (s) {
    case MM_OK: return "ok";
    case MM_E_ARG: return "bad argument or config";
    case MM_E_CUDA: return "CUDA error or no CUDA device (no CPU fallback exists)";
    case MM_E_CAP: return "capacity exceeded";
    case MM_E_NCCL: return "NCCL error";
    case MM_E_STATE: return "invalid state for this call";
    default: return "unknown status";
  }
}

const char* mm_last_error(mm_engine* e) { return e ? e->last_err : ""; }

void mm_config_default(mm_config* c) {
  if (!c) return;
  std::memset(c, 0, sizeof(*c));
  c->abi_version = MM_ABI_VERSION;
  static const int32_t lo[7] = {0, 1500, 2000, 2500, 3000, 3500, 4000};  // config/config.exs:27-36
  static const int32_t hi[7] = {1499, 1999, 2499, 2999, 3499, 3999, 5000};
  c->n_groups = 7;
  for (int g = 0; g < 7; ++g) { c->group_lo[g] = lo[g]; c->group_hi[g] = hi[g]; }
  c->default_group = 7 / 2 + 1;  // generic/worker.ex:27 -> "diamond"
  c->n_modes = 2;
  c->modes[0].teams = 2; c->modes[0].team_size = 1;  // "1v1"
  c->modes[1].teams = 2; c->modes[1].team_size = 5;  // "5v5"
  c->order_mode = MM_ORDER_ARRIVAL;
  c->capacity = 1u << 20;
  c->active_capacity = 0;
  c->device = 0;
  c->flags = 0;
}

int mm_group_of(const mm_config* cfg, int32_t rating) {
  if (!cfg || cfg->n_groups == 0 || cfg->n_groups > MM_MAX_GROUPS) return MM_E_ARG;
  return group_of(cfg, rating);
}

int mm_create(const mm_config* cfg, mm_engine** out) {
  if (!out) return MM_E_ARG;
  *out = nullptr;
  int rc = check_config(cfg);
  if (rc) return rc;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0 || cfg->device < 0 || cfg->device >= ndev) {
    cudaGetLastError();
    return MM_E_CUDA;  // no CPU fallback
  }
  mm_engine* e = new (std::nothrow) mm_engine();
  if (!e) return MM_E_CAP;
  e->cfg = *cfg;
  e->device = cfg->device;
  e->capacity = cfg->capacity;
  e->use_active = !(cfg->flags & MM_F_NO_DEDUPE);
  e->dense_ids = e->use_active && (cfg->flags & MM_F_DENSE_IDS);
  auto bail = [&](int code) { mm_destroy(e); return code; };
  if (cudaSetDevice(e->device) != cudaSuccess) return bail(MM_E_CUDA);
  cudaDeviceProp prop{};
  if (cudaGetDeviceProperties(&prop, e->device) != cudaSuccess) return bail(MM_E_CUDA);
  e->n_sms = prop.multiProcessorCount;
  if (cudaDeviceGetAttribute(&e->clock_khz, cudaDevAttrClockRate, e->device) != cudaSuccess) return bail(MM_E_CUDA);
  e->smem_optin = prop.sharedMemPerBlockOptin;
  e->smem_sm = prop.sharedMemPerMultiprocessor;
  if (cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess) return bail(MM_E_CUDA);
  if (cudaStreamCreateWithFlags(&e->d2h_stream, cudaStreamNonBlocking) != cudaSuccess) return bail(MM_E_CUDA);
  if (cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->ev_copy, cudaEventDisableTiming) != cudaSuccess)
    return bail(MM_E_CUDA);
  for (auto& ev : e->ev)
    if (cudaEventCreate(&ev) != cudaSuccess) return bail(MM_E_CUDA);
  if ((rc = build_tables(e))) return bail(rc);
  {
    // Two 512-thread CTAs per SM when the placement phase's per-bin state allows it (one CTA's barrier phases
    // overlap the other's work), else one.  Function attributes are process-global:
    // every kernel gets the device's opt-in maximum.
    const size_t static_smem = sizeof(Geo) + 512;
    const uint32_t st_max = 2;  // measured on an H100 (config3, two tile pipelines): a third ring stage is slower
    for (uint32_t st = st_max; st >= 2 && !e->place_stages; --st)
      if (2 * (place_smem_bytes(e->max_nb, st) + static_smem + 1024) <= e->smem_sm) { e->place_stages = st; e->rows_per_sm = 2; }
    for (uint32_t st = kMaxStages; st >= 1 && !e->place_stages; --st)  // huge key domains: down to a single stage
      if (place_smem_bytes(e->max_nb, st) + static_smem + 1024 <= e->smem_optin) { e->place_stages = st; e->rows_per_sm = 1; }
    if (!e->place_stages || colscan_smem(e) + static_smem + 1024 > e->smem_optin) {
      std::snprintf(e->last_err, sizeof(e->last_err), "key domain too large for shared memory: %u bins", e->Kp);
      return bail(MM_E_ARG);
    }
    bool ok = allow_max_smem(e, k_colscan) == cudaSuccess && allow_max_smem(e, k_hist<512>) == cudaSuccess &&
              allow_max_smem(e, k_place<512>) == cudaSuccess && allow_max_smem(e, k_tick<512>) == cudaSuccess;
    if (!ok) return bail(fail(e, cudaGetLastError(), "cudaFuncSetAttribute"));
  }
  e->n_chunks = (e->capacity + kTile - 1) / kTile + e->n_segs + 2;
  if ((uint64_t)e->n_chunks * e->n_segs * 4 > (8ull << 30)) return bail(MM_E_CAP);
  if ((rc = alloc_pool(e, e->pool[0])) || (rc = alloc_pool(e, e->pool[1]))) return bail(rc);
  if (cudaMalloc(&e->d_left_bits, (pool_slots(e) / 32 + 64) * 4) != cudaSuccess) return bail(MM_E_CUDA);
  if (e->use_active) {
    const uint64_t want = cfg->active_capacity ? cfg->active_capacity : 2ull * cfg->capacity;
    if (e->dense_ids) {
      e->hcap = want;  // handles 0 .. active_capacity - 1
      for (auto& t : e->tab) t.kv = nullptr;
      if (cudaMalloc(&e->tab[0].kv, e->hcap * 8) != cudaSuccess) return bail(MM_E_CUDA);
    } else {
      uint64_t h = 1024;
      while (h * 3 < want * 4 + 64) h <<= 1;  // load factor <= 0.75 at active_capacity
      e->hcap = h;
      for (auto& t : e->tab)
        if (cudaMalloc(&t.kv, h * 16) != cudaSuccess) return bail(MM_E_CUDA);
    }
    if ((rc = clear_table(e, e->tab[0]))) return bail(rc);
  }
  const size_t cap = (size_t)e->capacity + 64;
  e->max_lobbies = e->capacity / e->min_L + 1;
  auto A = [&](void** p, size_t bytes) { return cudaMalloc(p, bytes) == cudaSuccess; };
  if (!A((void**)&e->d_outbase, (e->Kp + 1) * 4) ||
      !A((void**)&e->d_binlim, (e->Kp + 1) * 4) || !A((void**)&e->d_seg, e->n_segs * sizeof(SegInfo)) ||
      !A((void**)&e->d_members, cap * 8) || !A((void**)&e->d_src_idx, cap * 4) ||
      !A((void**)&e->d_hdr, (size_t)e->max_lobbies * sizeof(mm_lobby_hdr)) ||
      !A((void**)&e->d_emit_seq, (size_t)e->max_lobbies * 4) || !A((void**)&e->d_ctr2, 2 * sizeof(TickCtr)) ||
      !A((void**)&e->d_small, 64) ||
      !A((void**)&e->d_blockhist, (size_t)e->n_segs * (kEnqChunkDev / kIngestItems + 1) * 4))
    return bail(fail(e, cudaGetLastError(), "cudaMalloc"));
  if (cudaMemset(e->d_ctr2, 0, 2 * sizeof(TickCtr)) != cudaSuccess) return bail(MM_E_CUDA);
  e->d_ctr = e->d_ctr2;
  if (cudaMallocHost(&e->h_ctr, sizeof(TickCtr)) != cudaSuccess || cudaMallocHost(&e->h_small, 64) != cudaSuccess)
    return bail(MM_E_CUDA);
  if ((rc = alloc_tick_scratch(e))) return bail(rc);
  {
    size_t sz = std::max(hist_smem_bytes(e->max_nb), place_smem_bytes(e->max_nb, e->place_stages));
    sz = std::max<size_t>(sz, std::max<size_t>((size_t)std::max(kEpiScratchWords, kRowCompactWords) * 4, colscan_smem(e)));
    int coop = 0, nb = 0;
    cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, e->device);
    if (coop && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_tick<512>, 512, sz) == cudaSuccess &&
        (uint32_t)nb * (uint32_t)e->n_sms >= e->R + e->helpers) {
      e->fused_ok = 1;
      e->tick_smem = sz;
    }
    cudaGetLastError();
  }
  if (cudaStreamSynchronize(e->stream) != cudaSuccess) return bail(MM_E_CUDA);
  *out = e;
  return MM_OK;
}

int mm_destroy(mm_engine* e) {
  if (!e) return MM_OK;
  cudaSetDevice(e->device);
  if (e->stream) cudaStreamSynchronize(e->stream);
  if (e->d2h_stream) cudaStreamSynchronize(e->d2h_stream);
  free_pool(e->pool[0]); free_pool(e->pool[1]); free_pool(e->snap); cudaFree(e->d_left_bits);
  for (auto& t : e->tab) cudaFree(t.kv);
  cudaFree(e->d_lut); cudaFree(e->d_grp_lut); cudaFree(e->d_mode_tsize); cudaFree(e->d_seg_bin_lo); cudaFree(e->d_seg_L);
  cudaFree(e->d_part_cut); cudaFree(e->d_cut_lp_lo);
  cudaFree(e->d_M); cudaFree(e->d_P); cudaFree(e->d_outbase); cudaFree(e->d_binlim); cudaFree(e->d_bin_seg);
  cudaFree(e->d_bin_key); cudaFree(e->d_seg); cudaFree(e->d_members); cudaFree(e->d_members32); cudaFree(e->d_members32_alt); cudaFree(e->d_hdr_alt); cudaFree(e->d_src_idx);
  cudaFree(e->d_hdr); cudaFree(e->d_emit_seq); cudaFree(e->d_ctr2); cudaFree(e->d_small);
  cudaFree(e->d_in_id); cudaFree(e->d_hslot); cudaFree(e->d_in_rating); cudaFree(e->d_in_mode); cudaFree(e->d_code);
  cudaFree(e->d_in_ts); cudaFree(e->d_blocksum); cudaFree(e->d_blockhist); cudaFree(e->d_part); cudaFree(e->d_in_key);
  cudaFree(e->d_in_handle); cudaFree(e->d_rej_idx); cudaFree(e->d_rej_code);
  cudaFree(e->d_qstat);
  if (e->h_ctr) cudaFreeHost(e->h_ctr);
  if (e->h_small) cudaFreeHost(e->h_small);
  for (auto& ev : e->ev)
    if (ev) cudaEventDestroy(ev);
  if (e->stream && e->own_stream) cudaStreamDestroy(e->stream);
  for (auto& st : e->stage) { cudaFree(st.handle); cudaFree(st.key); cudaFree(st.ts); if (st.ready) cudaEventDestroy(st.ready); }
  if (e->d2h_stream) cudaStreamDestroy(e->d2h_stream);
  if (e->copy_stream) cudaStreamDestroy(e->copy_stream);
  if (e->ev_copy) cudaEventDestroy(e->ev_copy);
  cudaGetLastError();
  delete e;
  return MM_OK;
}

int mm_set_stream(mm_engine* e, void* s) {
  if (!e) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  cudaSetDevice(e->device);
  cudaStreamSynchronize(e->stream);
  if (e->own_stream && e->stream) cudaStreamDestroy(e->stream);
  e->stream = (cudaStream_t)s;
  e->own_stream = false;
  return MM_OK;
}

int mm_set_option(mm_engine* e, const char* name, int64_t value) {
  if (!e || !name) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  if (!std::strcmp(name, "rank_impl")) {
    if (value != 2 && value != 3) return MM_E_ARG;
    e->rank_impl = (int)value;
    return MM_OK;
  }
  if (!std::strcmp(name, "async_results")) {
    int rcw = wait_results(e);
    if (rcw) return rcw;
    e->async_results = value != 0;
    if (e->async_results) {  // second set of the packed result buffers, allocated here rather than inside a tick
      CK(cudaSetDevice(e->device));
      if (!e->d_hdr_alt) CK(cudaMalloc(&e->d_hdr_alt, (size_t)e->max_lobbies * sizeof(mm_lobby_hdr)));
      if (!e->d_members32) CK(cudaMalloc(&e->d_members32, ((size_t)e->capacity + 64) * 4));
      if (!e->d_members32_alt) CK(cudaMalloc(&e->d_members32_alt, ((size_t)e->capacity + 64) * 4));
    }
    return MM_OK;
  }
  if (!std::strcmp(name, "max_spread")) {
    // EXTENSION (policy S1): a lobby spans at most `value` rating points; < 0 restores the reference behaviour.
    // Defined on the rating-sorted partition, so MM_ORDER_RATING only (oracle: orc_run_windowed).
    if (value >= 0 && e->cfg.order_mode != MM_ORDER_RATING) return MM_E_ARG;
    if (value > 0x7FFFFFFF) return MM_E_ARG;
    e->max_spread = value < 0 ? -1 : (int32_t)value;
    return MM_OK;
  }
  if (!std::strcmp(name, "tick_impl")) { e->tick_impl = value != 0; return MM_OK; }
  return MM_E_ARG;
}

int mm_enqueue_device(mm_engine* e, uint32_t n, const uint64_t* id, const int32_t* rating, const uint8_t* mode,
                      const uint32_t* enq_ts, uint8_t* accepted, uint32_t* n_accepted) {
  if (n_accepted) *n_accepted = 0;
  if (!e || (n && (!id || !rating || !mode))) return MM_E_ARG;
  if (n == 0) return MM_OK;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  int rc = enqueue_batch(e, n, id, rating, mode, enq_ts, kEnqChunkDev, [](uint32_t, uint32_t) { return (int)MM_OK; });
  if (rc) return rc;
  return enq_finish(e, n, accepted, n_accepted);
}

int mm_enqueue(mm_engine* e, uint32_t n, const uint64_t* id, const int32_t* rating, const uint8_t* mode,
               const uint32_t* enq_ts, uint8_t* accepted) {
  if (!e || (n && (!id || !rating || !mode))) return MM_E_ARG;
  if (n == 0) return MM_OK;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  int rc = ensure_enq_scratch(e, n);
  if (rc) return rc;
  auto upload = [&](uint32_t base, uint32_t cnt) -> int {
    CK(cudaMemcpyAsync(e->d_in_id + base, id + base, (size_t)cnt * 8, cudaMemcpyHostToDevice, e->copy_stream));
    CK(cudaMemcpyAsync(e->d_in_rating + base, rating + base, (size_t)cnt * 4, cudaMemcpyHostToDevice, e->copy_stream));
    CK(cudaMemcpyAsync(e->d_in_mode + base, mode + base, (size_t)cnt, cudaMemcpyHostToDevice, e->copy_stream));
    if (enq_ts)
      CK(cudaMemcpyAsync(e->d_in_ts + base, enq_ts + base, (size_t)cnt * 4, cudaMemcpyHostToDevice, e->copy_stream));
    CK(cudaEventRecord(e->ev_copy, e->copy_stream));
    CK(cudaStreamWaitEvent(e->stream, e->ev_copy, 0));
    return MM_OK;
  };
  rc = enqueue_batch(e, n, e->d_in_id, e->d_in_rating, e->d_in_mode, enq_ts ? e->d_in_ts : nullptr, kEnqChunk, upload);
  if (rc) { cudaStreamSynchronize(e->copy_stream); return rc; }
  rc = enq_finish(e, n, nullptr, nullptr);
  if (rc) return rc;
  if (accepted) {
    CK(cudaMemcpyAsync(accepted, e->d_code, n, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
  }
  return MM_OK;
}

int mm_enqueue_packed(mm_engine* e, uint32_t n, const uint32_t* handle, const uint16_t* key, const uint32_t* enq_ts,
                      uint8_t* accepted) {
  if (!e || (n && (!handle || !key))) return MM_E_ARG;
  if (n == 0) return MM_OK;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  int rc = ensure_enq_scratch(e, n);
  if (rc) return rc;
  auto upload = [&](uint32_t base, uint32_t cnt) -> int {  // 6 B per player over PCIe, unpacked on the device
    CK(cudaMemcpyAsync(e->d_in_handle + base, handle + base, (size_t)cnt * 4, cudaMemcpyHostToDevice, e->copy_stream));
    CK(cudaMemcpyAsync(e->d_in_key + base, key + base, (size_t)cnt * 2, cudaMemcpyHostToDevice, e->copy_stream));
    if (enq_ts)
      CK(cudaMemcpyAsync(e->d_in_ts + base, enq_ts + base, (size_t)cnt * 4, cudaMemcpyHostToDevice, e->copy_stream));
    CK(cudaEventRecord(e->ev_copy, e->copy_stream));
    CK(cudaStreamWaitEvent(e->stream, e->ev_copy, 0));
    k_unpack<<<(cnt + 255) / 256, 256, 0, e->stream>>>(cnt, e->d_in_handle + base, e->d_in_key + base, e->d_in_id + base,
                                                       e->d_in_rating + base, e->d_in_mode + base);
    CK(cudaGetLastError());
    return MM_OK;
  };
  rc = enqueue_batch(e, n, e->d_in_id, e->d_in_rating, e->d_in_mode, enq_ts ? e->d_in_ts : nullptr, kEnqChunk, upload);
  if (rc) { cudaStreamSynchronize(e->copy_stream); return rc; }
  rc = enq_finish(e, n, nullptr, nullptr);
  if (rc) return rc;
  if (accepted) {
    CK(cudaMemcpyAsync(accepted, e->d_code, n, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
  }
  return MM_OK;
}

int mm_enqueue_packed_begin(mm_engine* e, uint32_t n, const uint32_t* handle, const uint16_t* key, const uint32_t* enq_ts) {
  if (!e || !n || !handle || !key) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  if (e->stage_count == 2) {
    std::snprintf(e->last_err, sizeof(e->last_err), "both staging slots hold a batch: call mm_enqueue_packed_end first");
    return MM_E_STATE;
  }
  mm_engine::Stage& st = e->stage[(e->stage_head + e->stage_count) & 1];
  if (n > st.cap) {  // the slot's previous batch was consumed by an _end that synchronised the engine stream
    cudaFree(st.handle); cudaFree(st.key); cudaFree(st.ts);
    st.handle = nullptr; st.key = nullptr; st.ts = nullptr; st.cap = 0;
    CK(cudaMalloc(&st.handle, ((size_t)n + 64) * 4));
    CK(cudaMalloc(&st.key, ((size_t)n + 64) * 2));
    CK(cudaMalloc(&st.ts, ((size_t)n + 64) * 4));
    st.cap = n;
  }
  if (!st.ready) CK(cudaEventCreateWithFlags(&st.ready, cudaEventDisableTiming));
  CK(cudaMemcpyAsync(st.handle, handle, (size_t)n * 4, cudaMemcpyHostToDevice, e->copy_stream));
  CK(cudaMemcpyAsync(st.key, key, (size_t)n * 2, cudaMemcpyHostToDevice, e->copy_stream));
  if (enq_ts) CK(cudaMemcpyAsync(st.ts, enq_ts, (size_t)n * 4, cudaMemcpyHostToDevice, e->copy_stream));
  CK(cudaEventRecord(st.ready, e->copy_stream));
  st.n = n; st.has_ts = enq_ts != nullptr;
  ++e->stage_count;
  return MM_OK;
}

int mm_enqueue_packed_end(mm_engine* e, uint8_t* accepted, uint32_t* n_accepted) {
  if (!e) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  if (e->stage_count == 0) {
    std::snprintf(e->last_err, sizeof(e->last_err), "no staged batch: call mm_enqueue_packed_begin first");
    return MM_E_STATE;
  }
  mm_engine::Stage& st = e->stage[e->stage_head];
  e->stage_head ^= 1; --e->stage_count;  // the slot is released whatever happens below
  const uint32_t n = st.n;
  int rc = ensure_enq_scratch(e, n);
  if (rc) return rc;
  CK(cudaStreamWaitEvent(e->stream, st.ready, 0));
  auto unpack = [&](uint32_t base, uint32_t cnt) -> int {
    k_unpack<<<(cnt + 255) / 256, 256, 0, e->stream>>>(cnt, st.handle + base, st.key + base, e->d_in_id + base,
                                                       e->d_in_rating + base, e->d_in_mode + base);
    CK(cudaGetLastError());
    return MM_OK;
  };
  rc = enqueue_batch(e, n, e->d_in_id, e->d_in_rating, e->d_in_mode, st.has_ts ? st.ts : nullptr, kEnqChunkDev, unpack);
  if (rc) { cudaStreamSynchronize(e->stream); return rc; }
  rc = enq_finish(e, n, nullptr, n_accepted);
  if (rc) return rc;
  if (accepted) {
    CK(cudaMemcpyAsync(accepted, e->d_code, n, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
  }
  return MM_OK;
}

int mm_enqueue_rejects(mm_engine* e, uint32_t cap, uint32_t* index, uint8_t* code, uint32_t* n_rejects) {
  if (!e || !n_rejects || (cap && (!index || !code))) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  *n_rejects = 0;
  const uint32_t n = e->last_batch_n;
  if (n == 0) return MM_OK;
  if (cap > e->rej_cap) {
    cudaFree(e->d_rej_idx); cudaFree(e->d_rej_code);
    e->rej_cap = 0;
    CK(cudaMalloc(&e->d_rej_idx, (size_t)cap * 4));
    CK(cudaMalloc(&e->d_rej_code, (size_t)cap));
    e->rej_cap = cap;
  }
  CK(cudaMemsetAsync(e->d_small + 4, 0, 4, e->stream));
  k_compact_rejects<<<(n + 255) / 256, 256, 0, e->stream>>>(n, e->d_code, cap, e->d_rej_idx, e->d_rej_code, e->d_small + 4);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(e->h_small + 4, e->d_small + 4, 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  const uint32_t cnt = e->h_small[4];
  *n_rejects = cnt;
  const uint32_t m = std::min(cnt, cap);
  if (m) {
    CK(cudaMemcpyAsync(index, e->d_rej_idx, (size_t)m * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(code, e->d_rej_code, m, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
  }
  return cnt > cap ? MM_E_CAP : MM_OK;
}

int mm_remove(mm_engine* e, uint32_t n, const uint64_t* id, uint32_t* n_removed) {
  if (n_removed) *n_removed = 0;
  if (!e || (n && !id)) return MM_E_ARG;
  if (!e->use_active) return MM_E_STATE;
  if (n == 0) return MM_OK;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  int rc = ensure_enq_scratch(e, n);
  if (rc) return rc;
  const Pool& p = e->pool[e->cur];
  CK(cudaMemcpyAsync(e->d_in_id, id, (size_t)n * 8, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemsetAsync(e->d_small, 0, 16, e->stream));
  k_remove<<<(n + 255) / 256, 256, 0, e->stream>>>(n, e->d_in_id, act_view(e), p.v, p.m, (uint32_t)pool_slots(e), e->gen, e->K,
                                                   e->d_bin_seg, e->d_seg_bin_lo, e->d_small + 2);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(e->h_small, e->d_small, 16, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  const uint32_t rem = e->h_small[2];
  e->n_active -= std::min<uint64_t>(rem, e->n_active);
  if (!e->dense_ids) e->n_tomb += rem;
  if (n_removed) *n_removed = rem;
  return MM_OK;
}

int mm_take(mm_engine* e, uint32_t n, const uint64_t* id, uint32_t* n_taken) {
  if (n_taken) *n_taken = 0;
  if (!e || (n && !id)) return MM_E_ARG;
  if (!e->use_active) return MM_E_STATE;
  if (n == 0) return MM_OK;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  int rc = ensure_enq_scratch(e, n);
  if (rc) return rc;
  const Pool& p = e->pool[e->cur];
  CK(cudaMemcpyAsync(e->d_in_id, id, (size_t)n * 8, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemsetAsync(e->d_small, 0, 16, e->stream));
  k_take<<<(n + 255) / 256, 256, 0, e->stream>>>(n, e->d_in_id, act_view(e), p.v, p.m, (uint32_t)pool_slots(e), e->gen, e->K,
                                                 e->d_bin_seg, e->d_seg_bin_lo, e->d_small + 2);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(e->h_small, e->d_small, 16, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  if (n_taken) *n_taken = e->h_small[2];
  return MM_OK;
}

int mm_remove_packed(mm_engine* e, uint32_t n, const uint32_t* handle, uint32_t* n_removed) {
  if (n_removed) *n_removed = 0;
  if (!e || (n && !handle)) return MM_E_ARG;
  std::vector<uint64_t> wide(handle, handle + n);
  return mm_remove(e, n, wide.data(), n_removed);
}

int mm_in_queue(mm_engine* e, uint32_t n, const uint64_t* id, uint8_t* out) {
  if (!e || (n && (!id || !out))) return MM_E_ARG;
  if (!e->use_active) return MM_E_STATE;
  if (n == 0) return MM_OK;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  int rc = ensure_enq_scratch(e, n);
  if (rc) return rc;
  CK(cudaMemcpyAsync(e->d_in_id, id, (size_t)n * 8, cudaMemcpyHostToDevice, e->stream));
  k_lookup<<<(n + 255) / 256, 256, 0, e->stream>>>(n, e->d_in_id, act_view(e), e->d_code);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, e->d_code, n, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return MM_OK;
}

int mm_pool_size(mm_engine* e, uint32_t* n) {
  if (!e || !n) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  *n = e->pool[e->cur].n;
  return MM_OK;
}

int mm_active_size(mm_engine* e, uint32_t* n) {
  if (!e || !n) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  *n = (uint32_t)std::min<uint64_t>(e->n_active, 0xFFFFFFFFu);
  return MM_OK;
}

int mm_results_wait(mm_engine* e) {
  if (!e) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  return wait_results(e);
}

int mm_tick_device(mm_engine* e, uint64_t now, mm_tick_stats* stats) {
  if (!e) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  tick_begin(e, now);
  { int rcw = wait_results(e); if (rcw) return rcw; }
  const uint32_t n = e->pool[e->cur].n;
  e->last_fused = use_fused(e);
  int rc;
  if (e->last_fused) {
    if ((rc = tick_fused(e, false))) return rc;
  } else {
    if ((rc = tick_phase_a(e))) return rc;
    if ((rc = tick_phase_b(e, false))) return rc;
  }
  return tick_commit(e, n, stats);
}

int mm_results_device(mm_engine* e, const mm_lobby_hdr** d_lobbies, const uint64_t** d_member_ids) {
  if (!e) return MM_E_ARG;
  if (d_lobbies) *d_lobbies = e->d_hdr;
  if (d_member_ids) *d_member_ids = e->d_members;
  return MM_OK;
}

int mm_tick(mm_engine* e, uint64_t now, mm_lobby_hdr* lobbies, uint32_t lobby_cap, uint64_t* member_ids,
            uint64_t member_cap, uint32_t* emit_seq, mm_tick_stats* stats) {
  if (!e) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  tick_begin(e, now);
  return tick_to_host(e, lobbies, lobby_cap, member_ids, nullptr, member_cap, emit_seq, stats);
}

int mm_tick_packed(mm_engine* e, uint64_t now, mm_lobby_hdr* lobbies, uint32_t lobby_cap, uint32_t* member_handles,
                   uint64_t member_cap, uint32_t* emit_seq, mm_tick_stats* stats) {
  if (!e) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  tick_begin(e, now);
  return tick_to_host(e, lobbies, lobby_cap, nullptr, member_handles, member_cap, emit_seq, stats);
}

int mm_pool_read(mm_engine* e, uint32_t cap, uint64_t* id, int32_t* rating, uint8_t* mode, uint8_t* team_size,
                 uint32_t* enq_ts, uint32_t* n_out) {
  if (!e || !n_out) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  const Pool& p = e->pool[e->cur];
  uint32_t bump = 0;
  std::vector<uint32_t> fill(e->n_segs);
  CK(cudaMemcpyAsync(&bump, p.m.bump, 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemcpyAsync(fill.data(), p.m.fill, (size_t)e->n_segs * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  const size_t n = (size_t)bump * kTile;  // chunks come from a bump allocator: the ones in use are [0, bump)
  std::vector<uint64_t> hid(n);
  std::vector<int32_t> hr(n);
  std::vector<uint8_t> hm(n), hs(n);
  std::vector<uint32_t> ht(n), hq(n), tab((size_t)e->n_segs * e->n_chunks);
  if (n) {
    CK(cudaMemcpyAsync(hid.data(), p.v.id, n * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(hr.data(), p.v.rating, n * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(hm.data(), p.v.mode, n, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(hs.data(), p.v.tsize, n, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(ht.data(), p.v.ts, n * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(hq.data(), p.v.seq, n * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(tab.data(), p.m.chunk_tab, tab.size() * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
  }
  // queued players in GLOBAL enqueue order: sort the partitions' lists by sequence number (distance below seq_next)
  std::vector<std::pair<uint32_t, uint32_t>> order;  // (seq - seq_next mod 2^32, slot)
  for (uint32_t sg = 0; sg < e->n_segs; ++sg)
    for (uint32_t k = 0; k < fill[sg]; ++k) {
      const uint32_t slot = tab[(size_t)sg * e->n_chunks + k / kTile] * kTile + k % kTile;
      if (hm[slot] == MM_MODE_DEAD) continue;  // removed while queued; the next tick drops it
      order.emplace_back(hq[slot] - e->seq_next, slot);
    }
  std::sort(order.begin(), order.end());
  if (order.size() > cap) return MM_E_CAP;
  uint32_t k = 0;
  for (const auto& o : order) {
    const uint32_t i = o.second;
    if (id) id[k] = hid[i];
    if (rating) rating[k] = hr[i];
    if (mode) mode[k] = hm[i];
    if (team_size) team_size[k] = hs[i];
    if (enq_ts) enq_ts[k] = ht[i];
    ++k;
  }
  *n_out = k;
  return MM_OK;
}

int mm_queue_stats(mm_engine* e, uint64_t now, mm_queue_stat* out, uint32_t cap, uint32_t* n_out) {
  if (!e || !out || !n_out) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  const uint32_t n_cut = e->n_cut;
  *n_out = n_cut;
  if (cap < n_cut) return MM_E_CAP;
  CK(cudaSetDevice(e->device));
  const size_t bytes = (size_t)n_cut * sizeof(mm_queue_stat);
  if (!e->d_qstat) CK(cudaMalloc(&e->d_qstat, bytes));
  CK(cudaMemsetAsync(e->d_qstat, 0, bytes, e->stream));
  StatArgs a{};
  const Pool& p = e->pool[e->cur];
  a.sec[0] = StatSection{p.v.mode, p.v.ts, p.m, nullptr, (uint32_t)now};
  const Pool& q = e->pool[e->cur ^ 1];
  a.sec[1] = StatSection{q.v.mode, q.v.ts, q.m, e->d_left_bits, e->tick_now};
  a.n_segs = e->n_segs; a.part_cut = e->d_part_cut; a.out = e->d_qstat;
  // CTAs: at most the tiles in use (the host-side player counts bound them), at most 8 per SM; each takes a
  // contiguous run of tiles
  const uint32_t n_max = std::max(p.n, e->match_valid ? e->match_n : 0u);
  const uint64_t tiles = (uint64_t)n_max / kTile + e->n_segs;
  const uint32_t ctas = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(tiles, 8ull * (uint32_t)e->n_sms));
  k_queue_stats<kStatBlock><<<dim3(ctas, e->match_valid ? 2 : 1), kStatBlock, 0, e->stream>>>(a);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, e->d_qstat, bytes, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  const uint32_t G = e->cfg.n_groups;
  for (uint32_t c = 0; c < n_cut; ++c) {
    const mm_mode_desc& md = e->cfg.modes[c / G];
    out[c].mode = (uint8_t)(c / G);
    out[c].group = (uint8_t)(c % G);
    out[c].n_lobbies = out[c].n_matched / ((uint32_t)md.teams * md.team_size);  // whole lobbies of L players
  }
  return MM_OK;
}

int mm_snapshot(mm_engine* e) {
  if (!e) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  if (!e->snap.v.id) {
    int rc = alloc_pool(e, e->snap);
    if (rc) return rc;
  }
  int rc = copy_pool(e, e->snap, e->pool[e->cur]);
  if (rc) return rc;
  CK(cudaStreamSynchronize(e->stream));
  e->snap_seq = e->seq_next;
  e->has_snap = true;
  return MM_OK;
}

int mm_restore(mm_engine* e) {
  if (!e) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->has_snap) return MM_E_STATE;
  CK(cudaSetDevice(e->device));
  Pool& p = e->pool[e->cur];
  int rc = copy_pool(e, p, e->snap);
  if (rc) return rc;
  e->seq_next = e->snap_seq;
  e->gen = next_gen(e);
  e->match_valid = false;  // the restored pool was not matched by the last tick
  if (e->use_active && p.n) {
    k_restamp<<<dim3(e->n_chunks, e->n_segs), 256, 0, e->stream>>>(p.v, p.m, act_view(e), e->gen);
    CK(cudaGetLastError());
  }
  CK(cudaStreamSynchronize(e->stream));
  return MM_OK;
}

}  // extern "C"
