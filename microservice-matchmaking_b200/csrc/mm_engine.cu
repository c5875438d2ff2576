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
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <utility>
#include <vector>

#include "mm_backfill.cuh"
#include "mm_balance.cuh"
#include "mm_band.cuh"
#include "mm_expire.cuh"
#include "mm_image.cuh"
#include "mm_kernels.cuh"
#include "mm_locate.cuh"
#include "mm_offtick.cuh"
#include "mm_party.cuh"
#include "mm_party_backfill.cuh"
#include "mm_party_status.cuh"
#include "mm_quality.cuh"
#include "mm_recut.cuh"
#include "mm_regroup.cuh"
#include "mm_requeue.cuh"
#include "mm_stats.cuh"
#include "mm_widen.cuh"

using namespace mm;

namespace {

// A device array the engine owns: n elements at p (one cudaMalloc), freed by reset() and the destructor.  reserve()
// grows it by free-then-allocate, so the old contents are lost; after a failed allocation the array is empty.  Kernels
// take the raw pointer (the conversion below).
template <class T>
struct DevArray {
  T* p = nullptr;
  size_t n = 0;

  DevArray() = default;
  DevArray(const DevArray&) = delete;
  DevArray& operator=(const DevArray&) = delete;
  DevArray(DevArray&& o) noexcept : p(std::exchange(o.p, nullptr)), n(std::exchange(o.n, 0)) {}
  DevArray& operator=(DevArray&& o) noexcept {
    if (this != &o) { reset(); p = std::exchange(o.p, nullptr); n = std::exchange(o.n, 0); }
    return *this;
  }
  ~DevArray() { reset(); }

  cudaError_t reserve(size_t want) {
    if (want <= n) return cudaSuccess;
    reset();
    const cudaError_t err = cudaMalloc(reinterpret_cast<void**>(&p), want * sizeof(T));
    if (err != cudaSuccess) { p = nullptr; return err; }
    n = want;
    return cudaSuccess;
  }
  void reset() {
    if (p) cudaFree(p);
    p = nullptr; n = 0;
  }
  operator T*() const { return p; }
  T* operator->() const { return p; }
};

struct Pool {
  PoolView v{};  // the arrays below, as the kernels take them
  PoolMeta m{};
  uint32_t n = 0;  // host mirror of the sum of the partition fills (dead players included)
  uint32_t held = 0;  // slots of the chunks mm_requeue left behind: in no partition's list, reclaimed by the next tick
  DevArray<uint64_t> id;
  DevArray<int32_t> rating;
  DevArray<uint8_t> mode, tsize;
  DevArray<uint32_t> ts, seq;
  DevArray<uint16_t> bin;
  DevArray<uint32_t> fill, chunk_tab, bump, tot, chist;
};

struct Table {
  DevArray<unsigned long long> kv;  // hashed: hcap x {key, value}; direct: dcap values
};

// The counters the kernels of one call write, in device memory with a pinned host mirror.  The fields of one line are
// zeroed together before their kernels run.
struct Counters {
  uint32_t accepted, pool_full, winners;  // ingest: queued; rolled back because the pool is full; running winner total
  uint32_t removed;                       // mm_remove / mm_take
  uint32_t rejects;                       // mm_enqueue_rejects / mm_merge: batch entries not queued, compacted
  uint32_t expired, erased;               // k_expire: players expired or released; active-set entries erased
  uint32_t img_players, img_active;       // export: live players; active ids outside the pool
  uint32_t img_err, mrg_dups;             // mm_import / mm_merge: kImg* error bits; batch entries that will not queue
                                          // (mm_import_regroup: repeated ids)
  uint32_t rg_kmax;                       // mm_import_regroup: most image partitions feeding one new partition
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
  cudaEvent_t ev[7]{};  // tick start | after hist | after colscan | after place | after epilogue | balance pass: start | end
  char last_err[512] = {0};

  // key domain
  int32_t key_lo = 0;
  uint32_t KR = 0, stride = 0, K = 0, Kp = 0;
  uint32_t n_segs = 0;  // layout partitions (see build_tables)
  uint32_t n_cut = 0;   // (mode, group) cut segments
  DevArray<uint16_t> d_part_cut;   // [n_segs] partition -> cut segment
  DevArray<uint32_t> d_cut_lp_lo;  // [n_cut + 1] first partition of the cut segment
  DevArray<uint16_t> d_lut;
  DevArray<uint8_t> d_grp_lut;
  DevArray<uint8_t> d_mode_tsize;
  DevArray<uint32_t> d_seg_bin_lo;
  DevArray<uint32_t> d_seg_L;
  DevArray<uint16_t> d_bin_seg;  // [Kp] bin -> (mode, group) segment
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
  Table snap_tab;  // mm_snapshot: the current table, with its counts
  uint64_t snap_active = 0, snap_tomb = 0;

  // tick scratch
  uint32_t R = 0;        // row CTAs of a tick
  uint32_t helpers = 0;  // extra CTAs of the fused launch: the tail, then the compacted pool's chunk histograms
  int rows_per_sm = 2;
  int rank_impl = 3;           // 3 = ballot tile sort for partitions of <= 255 bins + lists otherwise; 2 = lists only
  uint32_t place_stages = 0;
  int fused_ok = 0;  // k_tick<512> can be launched cooperatively with R CTAs
  int tick_impl = 1; // 1 = one fused cooperative launch when possible, 0 = four launches
  size_t tick_smem = 0;
  DevArray<uint32_t> d_M, d_P;  // row histograms, their column prefixes (only for many-row partitions)
  DevArray<uint32_t> d_outbase, d_binlim;
  DevArray<uint16_t> d_bin_key;
  int32_t max_spread = -1;  // < 0: policy S0 (reference behaviour); >= 0: policy S1 (extension)
  uint32_t tb_mask = 0;     // team_balance: bit m = lobbies of mode m are split into balanced teams (extension)
  uint32_t tb_last = 0;     // the mask the last tick's balance pass ran with (0: it did not run)
  uint32_t pb_mask = 0;     // party_balance: bit m = party lobbies of mode m are split, every party whole (extension)
  DevArray<SegInfo> d_seg;
  DevArray<uint32_t> d_left_bits;  // one bit per virtual pool position: stays queued after the tick
  DevArray<uint64_t> d_members;
  DevArray<uint32_t> d_members32;  // mm_tick_packed: member handles narrowed for the host copy
  // async_results + mm_tick_packed: headers and narrowed handles alternate between two buffer sets, so the next
  // tick's kernels need not wait for this tick's host copies
  DevArray<uint32_t> d_members32_alt;
  DevArray<mm_lobby_hdr> d_hdr_alt;
  DevArray<uint32_t> d_src_idx;
  DevArray<mm_lobby_hdr> d_hdr;
  DevArray<uint32_t> d_emit_seq;
  uint32_t max_lobbies = 0;
  DevArray<TickCtr> d_ctr2;  // two counter blocks, used alternately (the fused kernel re-arms the other one)
  TickCtr* d_ctr = nullptr;  // the block of the current / last tick
  int ctr_idx = 0;
  TickCtr* h_ctr = nullptr;  // pinned

  // enqueue scratch (grown on demand)
  DevArray<uint64_t> d_in_id, d_hslot;
  DevArray<int32_t> d_in_rating;
  DevArray<uint8_t> d_in_mode, d_lookup;
  DevArray<uint16_t> d_part, d_in_key;
  DevArray<uint32_t> d_in_ts, d_in_handle, d_blocksum, d_blockhist;
  DevArray<Counters> d_cnt;
  Counters* h_cnt = nullptr;  // pinned
  // codes of the last ingest batch: grown only by an ingest batch that passed its capacity check, written only by
  // ingest, so mm_enqueue_rejects reads them whatever ran since
  DevArray<uint8_t> d_code;
  uint32_t last_batch_n = 0;    // entries of the last ingest batch (their codes are still in d_code)
  DevArray<uint32_t> d_rej_idx;
  DevArray<uint8_t> d_rej_code;

  // mm_enqueue_packed_begin / _end: two staging slots for packed batches whose upload is in flight (FIFO)
  struct Stage {
    DevArray<uint32_t> handle, ts;
    DevArray<uint16_t> key;
    uint32_t n = 0;
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
  DevArray<uint32_t> d_qstat;  // [n_cut] records

  // lobby budget (mm_set_lobby_budget): lobbies a queue / a mode may emit per tick.  An empty host vector = no limit
  // anywhere; the device copy is brought up to date by the next tick.  Not part of images or snapshots.
  std::vector<uint32_t> bud_queue, bud_mode;  // [n_cut], [n_modes]
  bool bud_stale = false;
  DevArray<uint32_t> d_bud;       // [n_cut] per queue | [n_modes] per mode
  DevArray<uint32_t> d_cand;      // [n_cut] budgeted ticks: lobbies every queue had, budgets ignored
  DevArray<uint32_t> d_cand_dry;  // mm_lobby_candidates: [n_cut] counts | [Kp + 1] parked matched counts (tail layout 0)
  bool report_valid = false;      // the last tick completed: d_seg (and d_cand, if report_budgeted) describe it
  bool report_budgeted = false;

  // mm_expire output (grown on demand to the largest output a call could write; not d_members / d_hdr, which
  // mm_results_device hands out until the next tick)
  DevArray<uint64_t> d_exp_id;  // ids, or 32-bit handles in its first half
  DevArray<uint32_t> d_exp_seq;

  // mm_export / mm_import.  The image-sized buffers (d_img, d_img_act: about the image's size, 210 MB at 10 M queued
  // players) are freed at the end of every call, so a hand-over leaves no such footprint on either engine; the small
  // per-tile / per-partition arrays are kept.
  bool fresh = true;  // nothing ever enqueued, imported or restored: mm_import may load an image
  DevArray<uint8_t> d_img;  // the image from section 2 (id) on, as it lies in the host buffer
  DevArray<uint32_t> d_img_tile;  // export: live slots per virtual tile -> offsets
  DevArray<uint32_t> d_img_part;  // export: [n_segs] live slots per partition; import: part_off[n_segs+1] | slot_base[n_segs]
  DevArray<uint8_t> d_img_act;    // export: the active section

  // mm_export_queues / mm_merge.  Like the image buffers, the batch-sized merge scratch is freed by every call.
  std::vector<uint16_t> h_part_cut;   // host copies of d_part_cut / d_cut_lp_lo
  std::vector<uint32_t> h_cut_lp_lo;
  DevArray<uint8_t> d_sel;            // [n_segs] selected partitions
  DevArray<uint32_t> d_mrg_src;       // merge batch index -> image index
  DevArray<uint8_t> d_mrg_code;       // the merge batch's ingest codes (d_code keeps the last mm_enqueue* batch's)
  DevArray<unsigned long long> d_mrg_seen;  // duplicate count: scratch id set

  // mm_requeue: the entries go through the ingest scratch (d_in_*; seq in d_in_handle), their codes through d_mrg_code,
  // the id check through d_mrg_seen, the grouped entries through d_mrg_src and d_rq_u, the gathered and merged columns
  // through d_img (all freed by every call); the block counts and partition tables below are kept
  DevArray<uint32_t> d_rq_u;     // grouped entries: age (seq - seq_next)
  DevArray<uint32_t> d_rq_hist;  // [n_segs][blocks] code-1 entries -> the block's first grouped index
  DevArray<uint32_t> d_rq_seg;   // rq_off[n_segs + 1] | m_off[n_segs + 1] | slot_base[n_segs]

  // mm_import_regroup (mm_regroup.cuh): the image's layout tables and the re-filing scratch, carved from one
  // allocation that every call frees
  DevArray<uint8_t> d_rg;

  // mm_band_candidates / mm_band_match (mm_band.cuh): sized by the band keys and the candidates, grown on demand
  struct Band {
    DevArray<uint32_t> map, fill, qoff, qtiles, qseg, M, tot, pos, kbase, klim, band_mb, band_lb, rstart, ctr;
    DevArray<uint64_t> id;        // candidate ids / members
    DevArray<int32_t> rating;     // candidate ratings
    DevArray<uint8_t> mode;       // candidate modes
    DevArray<uint64_t> up_id;     // the caller's upper-side columns
    DevArray<int32_t> up_rating;
    DevArray<uint8_t> up_mode, up_taken;
    DevArray<mm_lobby_hdr> hdr;
  } band;

  // mm_backfill (mm_backfill.cuh): sized by the requests, the pieces, the bins and the players taken, grown on demand;
  // the gather runs on the band arrays above
  struct Backfill {
    DevArray<uint32_t> in;  // requests in queue order (BfReq) | first request of every queue | the queues with requests
    DevArray<uint32_t> rem, key_bin, kbase, klim, n_taken, req_base, ctr;
    DevArray<BfPiece> piece;
    DevArray<uint64_t> staging, members;
    DevArray<uint32_t> staging_ts;  // mm_widen / mm_party_match: the taken solos' stamps beside staging
    DevArray<uint32_t> teams;       // mm_backfill_party: roff [n + 1] | filled | tbase [room entries]
    DevArray<uint16_t> room;        // mm_backfill_party: [room entries]
  } bf;

  // mm_widen (mm_widen.cuh): the call's tables and the anchors, grown on demand; the plan's rem, the keys, the pieces,
  // the staging and the members are the backfill arrays above
  struct Widen {
    DevArray<uint32_t> tab;  // rules [n_cut] | qlbase | qmbase [n_cut] | part [n_segs + 1] | cur [n_segs] | cta
                             // [grid] | rmap [n_chunks] | ctr [kWdWords]
    DevArray<uint32_t> anc;  // rec (2 words) | slot | age | rank | mbase, each [anchors]
    DevArray<mm_lobby_hdr> hdr;
  } wd;

  // mm_locate (mm_locate.cuh): the queried ids, the records and the call's tables (preview bases, member slots,
  // budgets, reverse chunk map), grown on demand; no other call reads or writes them
  struct Locate {
    DevArray<uint64_t> id;
    DevArray<mm_player_status> out;
    DevArray<uint32_t> tab;  // pos [Kp + 2] | outbase [Kp + 2] | binlim [Kp + 2] | cand [n_cut] | budgets [n_cut + n_modes] | rmap [n_chunks]
  } loc;

  // mm_match_quality (mm_quality.cuh): allocated by the first call at the capacity's bounds and kept, so a polled call
  // never allocates; no other call reads or writes them
  struct Quality {
    DevArray<uint32_t> w;             // per-bin, per-queue, per-tile and (arrival order) per-lobby / per-team words
    DevArray<long long> csum;         // [Kp] rating order: per-bin prefix of count x c
    DevArray<mm_lobby_quality> lob;   // [max_lobbies]
    DevArray<mm_queue_quality> rec;   // [n_cut]
  } mq;

  // team_balance (mm_balance.cuh): allocated by the first balanced tick or mm_widen and kept.  imb is read only by
  // mm_match_quality and written only by a tick, so it describes the last tick's lobbies until the next one.
  struct Balance {
    DevArray<uint32_t> imb;   // [max_lobbies] the last tick's balanced imbalance per header position
    DevArray<uint32_t> cval;  // [capacity + 64, or a party call's members] c - key_lo per member slot (arrival-order
                              // ticks, mm_widen, mm_party_match)
    DevArray<uint32_t> w;     // arrival order: live slots per tile -> offsets [n_tiles] | per partition [n_segs] | total
    DevArray<uint32_t> cont;  // party_balance: [a party call's lobbies] continuation bits per header position
    DevArray<unsigned long long> sum;  // party_balance: [1] the call's summed imbalance
  } tb;

  // the off-tick report (mm_offtick.cuh): one kept report per source (MM_OFFTICK_PARTY_MATCH, MM_OFFTICK_WIDEN), written
  // only by that source's calls and read only by mm_offtick_report; the capture scratch is shared by the two calls.
  // Grown on demand, never shrunk.
  struct OffTick {
    DevArray<uint32_t> ts;   // [a call's members] enq_ts per member slot
    DevArray<uint32_t> imb;  // [a call's lobbies] the balance pass's imbalance per header position
    DevArray<uint32_t> qb;   // lobby bases [n_cut + 1] | member bases [n_cut + 1]
    struct Report {
      bool valid = false;    // the source's last call returned MM_OK
      uint32_t n_lob = 0;    // its lobbies
      DevArray<mm_lobby_quality> lob;
      DevArray<mm_queue_quality> quality;
      DevArray<mm_match_waits> waits;
    } rep[2];
  } ot;

  // off-tick budget (mm_set_offtick_budget), per source: the budgets (an empty host vector = no limit anywhere; options,
  // not part of images or snapshots) and the per-queue words of the source's last call, which only that source's calls
  // write and mm_offtick_budget_report reads
  struct OffBudget {
    std::vector<uint32_t> queue, mode;  // [n_cut], [n_modes]
    DevArray<uint32_t> tab;  // qlob (the plan's lobbies, emitted) | cand | allot [n_cut] | budgets [n_cut + n_modes] | cut
    bool ran = false;        // the last call ran its plan (set by the call, cleared before it)
    bool budgeted = false;   // ... under a budget: cand holds c_q
    bool valid = false;      // ... and returned MM_OK or MM_E_CAP: the report reads tab
  } ob[2];

  // parties (mm_party.cuh): the table in two buffers (compaction moves it from one to the other), sized by
  // party_capacity; the batch and match scratch grown on demand.  Not part of images or snapshots.
  struct Party {
    uint32_t cap = 0;                  // party_capacity: members the table holds (0: no table)
    uint32_t n_rows = 0, n_mem = 0;    // rows and member entries in use, gone parties included
    uint32_t live = 0;                 // members of queued parties
    struct Buf {
      DevArray<uint32_t> seq, ts, off;
      DevArray<int32_t> R, mrat;
      DevArray<uint16_t> bin;
      DevArray<uint8_t> mode, grp, size, dead;
      DevArray<uint64_t> mid;
    } buf[2];
    int cur = 0;
    DevArray<uint8_t> in_size, in_mode, in_pre, in_code;
    DevArray<uint32_t> in_ts, in_moff, in_mparty, in_msz, in_one, in_seq;
    DevArray<uint32_t> in_at, rq_ctr;  // mm_requeue_party: the requeued rows' places, the call's counters
    DevArray<uint64_t> in_id, in_hslot;
    DevArray<int32_t> in_rating;
    DevArray<uint32_t> pb, pcur, tmp, sorted, lob, pos;  // match: [K + 1], [K], then [rows] each (tmp: compaction)
    DevArray<uint32_t> ctr;                              // [kPtWords + 2]
  } pt;

  // mm_party_queue_stats / mm_party_locate (mm_party_status.cuh): the records, the queried ids and the locate's own
  // words (the match plan runs on the party scratch above and the mm_widen / mm_backfill scratch, which only hold a
  // call's state while it runs), grown on demand; no other call reads or writes them
  struct PartyStatus {
    DevArray<uint32_t> rec;  // mm_party_queue_stats: [n_cut] records as words
    DevArray<uint64_t> id;
    DevArray<mm_party_member_status> out;
    DevArray<uint32_t> tab;  // rank [rows] | depth [n_cut] | qlob [n_cut] | cand [n_cut] | allot [n_cut] | budgets
                             // [n_cut + n_modes] | cut [1]
    // party_balance: the balance pass on tags
    DevArray<mm_lobby_hdr> hdr;
    DevArray<uint64_t> tags;
    DevArray<uint32_t> bal;  // cval [members] | stamps [members] | cont [lobbies]
    DevArray<unsigned long long> sum;
  } pst;
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

// mm_last_error <- the formatted message; returns `code`
__attribute__((format(printf, 3, 4))) int set_err(mm_engine* e, int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  std::vsnprintf(e->last_err, sizeof(e->last_err), fmt, ap);
  va_end(ap);
  return code;
}

// the counters to their host mirror, once the engine stream's work is done
int read_counters(mm_engine* e) {
  CK(cudaMemcpyAsync(e->h_cnt, e->d_cnt, sizeof(Counters), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return MM_OK;
}

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
  CK(p.id.reserve(c));
  CK(p.rating.reserve(c));
  CK(p.mode.reserve(c));
  CK(p.tsize.reserve(c));
  CK(p.ts.reserve(c));
  CK(p.bin.reserve(c));
  CK(p.seq.reserve(c));
  CK(p.fill.reserve(e->n_segs));
  CK(p.chunk_tab.reserve((size_t)e->n_segs * e->n_chunks));
  CK(p.bump.reserve(1));
  CK(p.tot.reserve((size_t)e->Kp + 1));
  if (e->max_nb <= kFastBins) {  // per-chunk key histograms: the tick skips its counting pass over the pool
    CK(p.chist.reserve((size_t)e->n_chunks * kChunkHist));
    CK(cudaMemset(p.chist, 0, (size_t)e->n_chunks * kChunkHist * 4));
  }
  CK(cudaMemset(p.tot, 0, ((size_t)e->Kp + 1) * 4));
  CK(cudaMemset(p.fill, 0, (size_t)e->n_segs * 4));
  CK(cudaMemset(p.bump, 0, 4));
  // chunks are read whole by the TMA tiles: keep the bin column defined (and "dead") past the fills
  CK(cudaMemset(p.bin, 0xFF, c * 2));
  p.v = PoolView{p.id, p.rating, p.mode, p.tsize, p.ts, p.bin, p.seq};
  p.m = PoolMeta{p.fill, p.chunk_tab, p.bump, p.tot, p.chist, e->n_chunks};
  p.n = 0;
  p.held = 0;
  return MM_OK;
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
  dst.held = src.held;
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

// the party table in buffer b as the kernels take it (all null without party_capacity)
PartyView pt_view(mm_engine* e, int b) {
  auto& t = e->pt.buf[b];
  if (!e->pt.cap) return PartyView{};
  return PartyView{t.seq, t.ts, t.off, t.R, t.bin, t.mode, t.grp, t.size, t.dead, t.mid, t.mrat};
}

size_t table_bytes(const mm_engine* e) { return e->hcap * (e->dense_ids ? 8 : 16); }

int clear_table(mm_engine* e, Table& t) {
  if (e->dense_ids) {
    CK(cudaMemsetAsync(t.kv, 0xFF, e->hcap * 8, e->stream));  // FREE = all ones
    return MM_OK;
  }
  k_fill_kv<<<1024, 256, 0, e->stream>>>(reinterpret_cast<ulonglong2*>(t.kv.p), e->hcap, kEmptyKey, kFreeVal);
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

// a host table to a device array of its size
template <class T>
int upload_table(mm_engine* e, DevArray<T>& d, const std::vector<T>& h) {
  CK(d.reserve(h.size()));
  CK(cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
  return MM_OK;
}

// The layout of a config (see mm_kernels.cuh): the key -> bin LUT, the rating -> group table and the (mode, group)
// cut segments with their layout partitions.  A pure host function: mm_create uploads its tables (build_tables), and
// mm_import_regroup builds the layout of an image's config as well, to check the image against it.
struct Layout {
  int32_t key_lo = 0;
  uint32_t KR = 0, stride = 0, K = 0, Kp = 0;
  uint32_t n_segs = 0, n_cut = 0, min_L = 0xFFFFFFFFu, max_nb = 1;
  std::vector<uint8_t> grp, tsz;                        // [KR] clamp key -> group (0xFF: none); [MM_MAX_MODES]
  std::vector<uint16_t> lut, bin_seg, bin_key, part_cut;  // [KR], [Kp], [Kp], [n_segs]
  std::vector<uint32_t> seg_lo, seg_L, cut_lp_lo;       // [n_segs + 1], [n_segs], [n_cut + 1]
};

int build_layout(const mm_config& c, Layout& y) {
  int32_t rmin = c.group_lo[0], rmax = c.group_hi[0];
  for (uint32_t g = 1; g < c.n_groups; ++g) { rmin = std::min(rmin, c.group_lo[g]); rmax = std::max(rmax, c.group_hi[g]); }
  y.key_lo = rmin - 1;
  const uint64_t KR64 = (uint64_t)((int64_t)rmax - rmin + 3);
  if (KR64 > 65535u) return MM_E_ARG;  // rating span must fit the 16-bit LUT
  y.KR = (uint32_t)KR64;
  const uint32_t G = c.n_groups;
  y.grp.assign(y.KR, 0);
  for (uint32_t k = 0; k < y.KR; ++k) {
    const int g = group_of(&c, (int64_t)y.key_lo + k);
    y.grp[k] = g < 0 ? 0xFF : (uint8_t)g;
  }
  y.lut.assign(y.KR, 0);
  std::vector<uint32_t> first(G + 1, 0);
  std::vector<uint16_t> key_of;  // rating order: bin (inside a mode) -> clamp key
  if (c.order_mode == MM_ORDER_RATING) {
    // bins ordered by (group, clamp key): the partition of a group is its keys ascending
    uint32_t next = 0;
    for (uint32_t g = 0; g < G; ++g) {
      first[g] = next;
      for (uint32_t k = 0; k < y.KR; ++k)
        if (y.grp[k] == g) { y.lut[k] = (uint16_t)next++; key_of.push_back((uint16_t)k); }
    }
    first[G] = next;
    y.stride = std::max(next, 1u);
  } else {
    for (uint32_t k = 0; k < y.KR; ++k) y.lut[k] = y.grp[k] == 0xFF ? 0 : y.grp[k];
    for (uint32_t g = 0; g <= G; ++g) first[g] = g;
    y.stride = G;
  }
  y.K = c.n_modes * y.stride;
  y.Kp = y.K + 1;
  if (y.Kp > 65535u) return MM_E_ARG;  // the resident sort key is 16 bits
  // Layout partitions: a (mode, group) CUT SEGMENT — the unit of the lobby cut — is stored as one or more PARTITIONS
  // of at most kFastBins consecutive sort keys each, so that every tile ranks on the 8-bit path and carries a chunk
  // histogram whatever the width of the rating group (the reference's default groups span 500 - 1 500 ratings,
  // config/config.exs:27-36).  Narrow groups: one partition per segment.
  y.n_cut = c.n_modes * G;
  y.cut_lp_lo.assign(y.n_cut + 1, 0);
  y.min_L = 0xFFFFFFFFu;
  y.tsz.assign(MM_MAX_MODES, 0);
  bool split = !(c.flags & MM_F_WIDE_PARTITIONS);
  for (int attempt = 0; attempt < 2; ++attempt) {
    y.seg_lo.clear(); y.seg_L.clear(); y.part_cut.clear();
    for (uint32_t m = 0; m < c.n_modes; ++m) {
      const uint32_t L = (uint32_t)c.modes[m].teams * c.modes[m].team_size;
      y.min_L = std::min(y.min_L, L);
      y.tsz[m] = (uint8_t)c.modes[m].team_size;
      for (uint32_t g = 0; g < G; ++g) {
        const uint32_t lo = m * y.stride + first[g], nk = first[g + 1] - first[g];
        const uint32_t nsub = split ? std::max(1u, (nk + kFastBins - 1) / kFastBins) : 1u;
        const uint32_t per = (nk + nsub - 1) / nsub;
        y.cut_lp_lo[m * G + g] = (uint32_t)y.seg_lo.size();
        for (uint32_t j = 0; j < nsub; ++j) {
          y.seg_lo.push_back(lo + std::min(nk, j * per)); y.seg_L.push_back(L); y.part_cut.push_back((uint16_t)(m * G + g));
        }
      }
    }
    if (y.seg_lo.size() <= kMaxSegs) break;
    split = false;  // too many partitions for the on-chip tables: whole segments, list ranking for the wide ones
  }
  y.n_segs = (uint32_t)y.seg_lo.size();
  if (y.n_segs > kMaxSegs) return MM_E_ARG;
  y.cut_lp_lo[y.n_cut] = y.n_segs;
  y.seg_lo.push_back(y.K);
  y.max_nb = 1;
  for (uint32_t sgi = 0; sgi < y.n_segs; ++sgi) y.max_nb = std::max(y.max_nb, y.seg_lo[sgi + 1] - y.seg_lo[sgi]);
  y.bin_seg.assign(y.Kp, 0);
  for (uint32_t sgi = 0; sgi < y.n_segs; ++sgi)
    for (uint32_t b = y.seg_lo[sgi]; b < y.seg_lo[sgi + 1]; ++b) y.bin_seg[b] = (uint16_t)sgi;
  y.bin_key.assign(y.Kp, 0);
  if (!key_of.empty())
    for (uint32_t b = 0; b < y.K; ++b) y.bin_key[b] = key_of[b % y.stride];
  return MM_OK;
}

// The engine's layout (build_layout of its config) into its fields and device tables.
int build_tables(mm_engine* e) {
  Layout y;
  int rc = build_layout(e->cfg, y);
  if (rc) return rc;
  e->key_lo = y.key_lo; e->KR = y.KR; e->stride = y.stride; e->K = y.K; e->Kp = y.Kp;
  e->n_segs = y.n_segs; e->n_cut = y.n_cut; e->min_L = y.min_L; e->max_nb = y.max_nb;
  e->h_part_cut = y.part_cut;
  e->h_cut_lp_lo = y.cut_lp_lo;
  if ((rc = upload_table(e, e->d_part_cut, y.part_cut)) || (rc = upload_table(e, e->d_cut_lp_lo, y.cut_lp_lo)) ||
      (rc = upload_table(e, e->d_bin_seg, y.bin_seg)) || (rc = upload_table(e, e->d_bin_key, y.bin_key)) ||
      (rc = upload_table(e, e->d_lut, y.lut)) || (rc = upload_table(e, e->d_grp_lut, y.grp)) ||
      (rc = upload_table(e, e->d_mode_tsize, y.tsz)) || (rc = upload_table(e, e->d_seg_bin_lo, y.seg_lo)) ||
      (rc = upload_table(e, e->d_seg_L, y.seg_L)))
    return rc;
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
  CK(e->d_M.reserve((size_t)(e->R + 1) * e->Kp));
  CK(e->d_P.reserve((size_t)(e->R + 1) * e->Kp));
  return MM_OK;
}

// mm_create: both pool buffers, the active set, the tick's outputs and scratch, the counters
int alloc_buffers(mm_engine* e) {
  int rc;
  if ((rc = alloc_pool(e, e->pool[0])) || (rc = alloc_pool(e, e->pool[1]))) return rc;
  CK(e->d_left_bits.reserve(pool_slots(e) / 32 + 64));
  if (e->use_active) {
    const uint64_t want = e->cfg.active_capacity ? e->cfg.active_capacity : 2ull * e->cfg.capacity;
    if (e->dense_ids) {
      e->hcap = want;  // handles 0 .. active_capacity - 1
      CK(e->tab[0].kv.reserve(e->hcap));
    } else {
      uint64_t h = 1024;
      while (h * 3 < want * 4 + 64) h <<= 1;  // load factor <= 0.75 at active_capacity
      e->hcap = h;
      for (auto& t : e->tab) CK(t.kv.reserve(2 * h));  // {key, value} per slot
    }
    if ((rc = clear_table(e, e->tab[0]))) return rc;
  }
  const size_t cap = (size_t)e->capacity + 64;
  e->max_lobbies = e->capacity / e->min_L + 1;
  CK(e->d_outbase.reserve(e->Kp + 1));
  CK(e->d_binlim.reserve(e->Kp + 1));
  CK(e->d_seg.reserve(e->n_segs));
  CK(e->d_members.reserve(cap));
  CK(e->d_src_idx.reserve(cap));
  CK(e->d_hdr.reserve(e->max_lobbies));
  CK(e->d_emit_seq.reserve(e->max_lobbies));
  CK(e->d_ctr2.reserve(2));
  CK(e->d_cnt.reserve(1));
  CK(e->d_blockhist.reserve((size_t)e->n_segs * (kEnqChunkDev / kIngestItems + 1)));
  CK(cudaMemset(e->d_ctr2, 0, 2 * sizeof(TickCtr)));
  e->d_ctr = e->d_ctr2;
  CK(cudaMallocHost(&e->h_ctr, sizeof(TickCtr)));
  CK(cudaMallocHost(&e->h_cnt, sizeof(Counters)));
  return alloc_tick_scratch(e);
}

int ensure_enq_scratch(mm_engine* e, uint32_t n) {
  const size_t c = (size_t)n + 64;
  CK(e->d_in_id.reserve(c));
  CK(e->d_hslot.reserve(c));
  CK(e->d_in_rating.reserve(c));
  CK(e->d_in_mode.reserve(c));
  CK(e->d_lookup.reserve(c));
  CK(e->d_part.reserve(c));
  CK(e->d_in_key.reserve(c));
  CK(e->d_in_handle.reserve(c));
  CK(e->d_in_ts.reserve(c));
  CK(e->d_blocksum.reserve(std::min<size_t>(c, kEnqChunkDev) / 256 + 2));
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

// capacity checks + scratch for an ingest batch of n players, of which at most n_new can add an active-set entry
// (mm_merge counts them exactly; every other batch passes n)
// a hashed active set that could not take n_new more ids: rehashed, or MM_E_CAP (a batch of n entries)
int act_room(mm_engine* e, uint32_t n, uint32_t n_new) {
  if (e->use_active && !e->dense_ids && (e->n_active + e->n_tomb + n_new) * 4 > e->hcap * 3) {
    if ((e->n_active + n_new) * 4 > e->hcap * 3)
      return set_err(e, MM_E_CAP, "active set full: %llu ids resident, batch of %u, capacity %llu",
                     (unsigned long long)e->n_active, n, (unsigned long long)(e->hcap * 3 / 4));
    return rehash(e);
  }
  return MM_OK;
}

int enq_prepare(mm_engine* e, uint32_t n, uint32_t n_new) {
  e->fresh = false;
  int rc = ensure_enq_scratch(e, n);
  if (rc || (rc = act_room(e, n, n_new))) return rc;
  if ((size_t)n + 64 > e->d_code.n) {  // the batch is taken: the previous batch's codes may go
    e->last_batch_n = 0;
    CK(e->d_code.reserve((size_t)n + 64));
  }
  CK(cudaMemsetAsync(&e->d_cnt->accepted, 0, 3 * 4, e->stream));  // accepted, pool_full, winners
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
    const uint64_t used = (uint64_t)p.n + p.held;
    const uint32_t room = e->capacity > used ? (uint32_t)(e->capacity - used) : 0u;
    k_enq_count<<<nb, 256, 0, e->stream>>>(base, cnt, av, e->d_hslot, e->d_code, e->d_blocksum);
    k_scan_small<<<1, 1024, 0, e->stream>>>(nb, e->d_blocksum, &e->d_cnt->winners);
    k_enq_cut<<<nb, 256, 0, e->stream>>>(base, cnt, av, e->d_hslot, e->d_code, e->d_blocksum, room, &e->d_cnt->pool_full);
    if (e->use_active) k_enq_promote<<<nb, 256, 0, e->stream>>>(base, cnt, e->d_hslot, e->d_code);
  }
  k_enq_route<<<nblk, 256, 0, e->stream>>>(base, cnt, av, e->d_hslot, e->d_code, e->d_part, e->n_segs, nblk, e->d_blockhist);
  k_enq_alloc<<<1, 512, 0, e->stream>>>(e->n_segs, nblk, e->d_blockhist, p.m, &e->d_cnt->accepted);
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
  if (accepted_dev) CK(cudaMemcpyAsync(accepted_dev, e->d_code, n, cudaMemcpyDeviceToDevice, e->stream));
  int rc = read_counters(e);
  if (rc) return rc;
  const uint32_t acc = e->h_cnt->accepted, rej = e->h_cnt->pool_full;
  p.n += acc;
  e->seq_next += n;
  e->last_batch_n = n;
  if (e->use_active) { e->n_active += acc; if (!e->dense_ids) e->n_tomb += rej; }
  if (n_accepted) *n_accepted = acc;
  return MM_OK;
}

// The end of a batch uploaded from the host: the counters, then the codes to the caller's host array.  After a failed
// upload or ingest, the stream the batch's copies ran on is drained first.
int enq_finish_host(mm_engine* e, int rc, cudaStream_t drain, uint32_t n, uint8_t* accepted, uint32_t* n_accepted) {
  if (rc) { cudaStreamSynchronize(drain); return rc; }
  if ((rc = enq_finish(e, n, nullptr, n_accepted)) || !accepted) return rc;
  CK(cudaMemcpyAsync(accepted, e->d_code, n, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return MM_OK;
}

// the engine stream waits for the copies queued on the copy stream so far
int copy_fence(mm_engine* e) {
  CK(cudaEventRecord(e->ev_copy, e->copy_stream));
  CK(cudaStreamWaitEvent(e->stream, e->ev_copy, 0));
  return MM_OK;
}

// Device columns of a whole batch -> pool.  `upload` (may be null) queues the H2D copies of one chunk on the copy
// stream: the previous chunk's kernels run on the engine stream meanwhile, so the device side of the ingest hides
// behind the PCIe transfer except for the last chunk.
template <class Upload>
int enqueue_batch(mm_engine* e, uint32_t n, const uint64_t* id, const int32_t* rating, const uint8_t* mode,
                  const uint32_t* ts, uint32_t chunk, Upload upload) {
  int rc = enq_prepare(e, n, n);
  if (rc) return rc;
  const bool may_overflow = (uint64_t)e->pool[e->cur].n + e->pool[e->cur].held + n > e->capacity;
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
  t.n_groups = e->cfg.n_groups;
  t.bud_queue = e->bud_queue.empty() ? nullptr : e->d_bud.p;
  t.bud_mode = e->bud_mode.empty() ? nullptr : e->d_bud.p + e->n_cut;
  t.cand = e->d_cand;
  return t;
}
// the budgets set since the last tick -> their device copy (before a tick's launches)
int budget_upload(mm_engine* e) {
  e->report_budgeted = !e->bud_queue.empty() || !e->bud_mode.empty();
  if (!e->bud_stale) return MM_OK;
  e->bud_stale = false;
  if (!e->report_budgeted) return MM_OK;
  CK(e->d_bud.reserve(e->n_cut + e->cfg.n_modes));
  CK(e->d_cand.reserve(e->n_cut));
  if (!e->bud_queue.empty())
    CK(cudaMemcpyAsync(e->d_bud, e->bud_queue.data(), (size_t)e->n_cut * 4, cudaMemcpyHostToDevice, e->stream));
  if (!e->bud_mode.empty())
    CK(cudaMemcpyAsync(e->d_bud + e->n_cut, e->bud_mode.data(), (size_t)e->cfg.n_modes * 4, cudaMemcpyHostToDevice, e->stream));
  CK(cudaStreamSynchronize(e->stream));  // the host vectors may change as soon as the tick returns
  return MM_OK;
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
  a.src_idx = want_seq ? e->d_src_idx.p : nullptr;
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
  a.hdr = e->d_hdr; a.src_idx = want_seq ? e->d_src_idx.p : nullptr; a.emit_seq = want_seq ? e->d_emit_seq.p : nullptr;
  a.ctr = e->d_ctr;
  return a;
}

// launches k_hist + k_colscan (phase A of a tick): the counters are final afterwards
int tick_phase_a(mm_engine* e) {
  const Pool& p = e->pool[e->cur];
  { const int rc = budget_upload(e); if (rc) return rc; }
  CK(cudaMemsetAsync(e->d_ctr, 0, sizeof(TickCtr), e->stream));
  CK(cudaEventRecord(e->ev[0], e->stream));
  const uint32_t rows = tick_rows(e);
  k_hist<512><<<rows, 512, hist_smem_bytes(e->max_nb), e->stream>>>(p.v.bin, p.m, e->n_segs, rows, e->Kp, e->max_nb, e->d_seg_bin_lo, e->d_M);
  CK(cudaEventRecord(e->ev[1], e->stream));
  const uint32_t scan_ctas = (e->K + 31) / 32 + 1;
  if (e->report_budgeted) k_colscan<true><<<scan_ctas, kScanBlock, colscan_smem(e), e->stream>>>(rows, e->d_M, e->d_P, tail_args(e));
  else k_colscan<false><<<scan_ctas, kScanBlock, colscan_smem(e), e->stream>>>(rows, e->d_M, e->d_P, tail_args(e));
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
  { const int rc = budget_upload(e); if (rc) return rc; }
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
  const void* kernel = e->report_budgeted ? (const void*)k_tick<512, true> : (const void*)k_tick<512>;
  CK(cudaLaunchCooperativeKernel(kernel, dim3(rows + helpers), dim3(512), params, e->tick_smem, e->stream));
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
  e->pool[e->cur].held = 0;
  e->match_valid = true;  // pool[cur ^ 1] is now the pool this tick matched
  e->report_valid = true;
  e->match_n = n;
  e->last = st;
  if (stats) *stats = st;
  if (c.chist_bad)  // placement took slot bases from chunk histograms that disagree with the pool: results are wrong
    return set_err(e, MM_E_STATE, "%u placement tiles disagree with their chunk histograms", c.chist_bad);
  if (c.left_bad)  // the compaction found leftovers beyond their partition's share of the compacted pool
    return set_err(e, MM_E_STATE, "%u leftover players fall outside their partition's compacted range", c.left_bad);
  return MM_OK;
}

// Every tick entry point: the tick's `now` is kept for mm_queue_stats, and the last tick's match section is void from
// here on (a tick that fails after its phase A — MM_E_CAP on the split path — has rewritten pool[cur ^ 1].m).
void tick_begin(mm_engine* e, uint64_t now) {
  e->tick_now = (uint32_t)now;
  e->match_valid = false;
  e->report_valid = false;
}

// async_results: the previous tick's host copies must land before its device buffers are overwritten
int wait_results(mm_engine* e) {
  if (e->results_pending) {
    CK(cudaStreamSynchronize(e->d2h_stream));
    e->results_pending = false;
  }
  return MM_OK;
}

int balance_tick(mm_engine* e, mm_tick_stats* stats);  // (below)

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
    if ((lobbies && e->h_ctr->n_lobbies > lobby_cap) || (want_members && e->h_ctr->n_matched > member_cap))
      return set_err(e, MM_E_CAP, "need lobby_cap >= %u, member_cap >= %u", e->h_ctr->n_lobbies, e->h_ctr->n_matched);
    if ((rc = tick_phase_b(e, emit_seq != nullptr))) return rc;
  }
  if ((rc = tick_commit(e, n, stats))) return rc;
  if ((rc = balance_tick(e, stats))) return rc;
  const TickCtr& c = *e->h_ctr;
  if (member_handles && c.n_matched) {
    CK(e->d_members32.reserve((size_t)e->capacity + 64));
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

// The virtual tiles of a pool of n players (an upper bound: the host-side player count bounds them), and the CTAs of a
// tile walk over them: at most the tiles, at most 8 per SM; each CTA takes a contiguous run of tiles.
uint32_t tile_count(const mm_engine* e, uint32_t n) { return n / kTile + e->n_segs; }
// 1-D grid of 256-thread CTAs over n items: at most per_sm CTAs per SM, one at least.
uint32_t grid256(const mm_engine* e, uint64_t n, uint32_t per_sm) {
  return (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((n + 255) / 256, (uint64_t)per_sm * (uint32_t)e->n_sms));
}
// Keys of the scratch id set (seen_insert) for n ids: a power of two, at least 1024, at most half full.
uint64_t seen_keys(uint64_t n) {
  uint64_t sc = 1024;
  while (sc < 2 * n) sc <<= 1;
  return sc;
}
// The refusal of every call that reads or rewrites the pool while a packed batch is staged.
int staged_err(mm_engine* e) {
  return set_err(e, MM_E_STATE, "a packed batch is staged: call mm_enqueue_packed_end first");
}
// The refusal of the image calls and mm_snapshot while a party is queued.
int parties_err(mm_engine* e) {
  return set_err(e, MM_E_STATE, "%u party members are queued: images and snapshots do not carry parties", e->pt.live);
}
uint32_t tile_ctas(const mm_engine* e, uint32_t n) {
  return std::max<uint32_t>(1, std::min<uint32_t>(tile_count(e, n), 8u * (uint32_t)e->n_sms));
}

// team_balance: the balance pass over the results of the tick that has just committed (d_outbase and pool[cur ^ 1]
// still describe it).  Records the mask it ran with for mm_match_quality.  It returns with the engine stream idle, as
// the tick itself does: mm_results_device and the async_results copy stream read the members on streams of their own.
// Its CUDA-event time is added to the tick's device_us.
int balance_tick(mm_engine* e, mm_tick_stats* stats) {
  e->tb_last = 0;
  const uint32_t n_lob = e->last.n_lobbies;
  if (!e->tb_mask || !n_lob) return MM_OK;
  auto& s = e->tb;
  CK(s.imb.reserve(e->max_lobbies));
  TbArgs t{};
  t.hdr = e->d_hdr; t.n_lob = n_lob; t.members = e->d_members; t.mask = e->tb_mask; t.mode_tsize = e->d_mode_tsize;
  t.outbase = e->d_outbase; t.bin_key = e->d_bin_key; t.K = e->K; t.imb = s.imb;
  const uint32_t grid = grid256(e, (uint64_t)n_lob * 32, 8);
  CK(cudaEventRecord(e->ev[5], e->stream));
  if (e->cfg.order_mode == MM_ORDER_ARRIVAL) {
    const Pool& p = e->pool[e->cur ^ 1];  // the pool the tick read
    const size_t n_tiles = (size_t)e->n_chunks + e->n_segs;
    CK(s.cval.reserve((size_t)e->capacity + 64));
    CK(s.w.reserve(n_tiles + e->n_segs + 1));
    CK(cudaMemsetAsync(s.w + n_tiles, 0, ((size_t)e->n_segs + 1) * 4, e->stream));
    // live slots per virtual tile -> the live slots before each tile (mm_export's count and scan)
    ImgExportArgs x{};
    x.pool = p.v; x.meta = p.m; x.n_segs = e->n_segs; x.tile_cnt = s.w; x.part_cnt = s.w + n_tiles;
    const uint32_t ctas = tile_ctas(e, e->match_n);
    k_img_tiles<kImgBlock, false><<<ctas, kImgBlock, 0, e->stream>>>(x);
    k_scan_small<<<1, 1024, 0, e->stream>>>(tile_count(e, e->match_n), s.w, s.w + n_tiles + e->n_segs);
    TbArrivalArgs a{};
    a.pool = p.v; a.meta = p.m; a.left_bits = e->d_left_bits; a.tile_off = s.w;
    a.n_segs = e->n_segs; a.n_groups = e->cfg.n_groups; a.mask = e->tb_mask; a.key_lo = e->key_lo; a.KR = e->KR;
    a.part_cut = e->d_part_cut; a.mode_tsize = e->d_mode_tsize; a.seg_bin_lo = e->d_seg_bin_lo;
    a.outbase = e->d_outbase; a.cval = s.cval;
    k_tb_arrival<kMqBlock><<<ctas, kMqBlock, 0, e->stream>>>(a);
    t.cval = s.cval;
    k_tb_lobby<true><<<grid, 256, 0, e->stream>>>(t);
  } else {
    k_tb_lobby<false><<<grid, 256, 0, e->stream>>>(t);
  }
  CK(cudaGetLastError());
  CK(cudaEventRecord(e->ev[6], e->stream));
  CK(cudaStreamSynchronize(e->stream));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, e->ev[5], e->ev[6]));
  e->last.device_us += ms * 1000.f;
  if (stats) stats->device_us = e->last.device_us;
  e->tb_last = e->tb_mask;
  return MM_OK;
}

// active-set entries erased by mm_remove, mm_expire or an export release: a hashed set keeps a tombstone for each
void erase_active(mm_engine* e, uint32_t erased) {
  e->n_active -= std::min<uint64_t>(erased, e->n_active);
  if (e->use_active && !e->dense_ids) e->n_tomb += erased;
}

// k_expire over the current pool, with the counters expired / erased zeroed first.  The caller sets now, max_wait,
// commit, the outputs and the selection in `a`.
int launch_expire(mm_engine* e, ExpireArgs a) {
  const Pool& p = e->pool[e->cur];
  a.pool = p.v; a.meta = p.m; a.n_segs = e->n_segs;
  a.act = act_view(e); a.gen = e->gen; a.dead_bin = e->K; a.bin_seg = e->d_bin_seg; a.seg_bin_lo = e->d_seg_bin_lo;
  a.ctr = &e->d_cnt->expired;
  CK(cudaMemsetAsync(a.ctr, 0, 2 * 4, e->stream));  // expired, erased
  k_expire<kExpBlock><<<tile_ctas(e, p.n), kExpBlock, 0, e->stream>>>(a);
  if (e->pt.live && !a.sel) {  // whole parties, behind the solos
    CK(cudaMemsetAsync(e->pt.ctr, 0, kPtWords * 4, e->stream));
    k_pt_expire<<<(e->pt.n_rows + 255) / 256, 256, 0, e->stream>>>(e->pt.n_rows, pt_view(e, e->pt.cur), a.now,
                                                                    a.max_wait, a.commit, a.act, a.out_id, a.out_handle,
                                                                    a.out_seq, a.ctr, e->pt.ctr);
  }
  CK(cudaGetLastError());
  return MM_OK;
}

// mm_expire / mm_expire_packed (one of ids / handles).  A cap that holds every resident player cannot overflow: one
// pass.  Otherwise a counting pass decides first, so that a refused call leaves everything as it was.
int expire(mm_engine* e, uint64_t now, uint32_t max_wait, uint64_t* ids, uint32_t* handles, uint32_t* seq, uint32_t cap,
           uint32_t* n_expired) {
  const Pool& p = e->pool[e->cur];
  *n_expired = 0;
  const uint32_t most = p.n + e->pt.live;
  if (most == 0) return MM_OK;
  ExpireArgs a{};
  a.now = (uint32_t)now; a.max_wait = max_wait;
  uint32_t need = most;
  int rc;
  if (cap < most) {
    if ((rc = launch_expire(e, a)) || (rc = read_counters(e))) return rc;
    need = e->h_cnt->expired;
    *n_expired = need;
    if (need > cap) return set_err(e, MM_E_CAP, "need cap >= %u", need);
    if (need == 0) return MM_OK;
  }
  CK(e->d_exp_id.reserve(need));
  if (seq) CK(e->d_exp_seq.reserve(e->d_exp_id.n));
  a.commit = 1;
  a.out_id = ids ? e->d_exp_id.p : nullptr;
  a.out_handle = ids ? nullptr : reinterpret_cast<uint32_t*>(e->d_exp_id.p);
  a.out_seq = seq ? e->d_exp_seq.p : nullptr;
  uint32_t gone = 0;
  if ((rc = launch_expire(e, a))) return rc;
  if (e->pt.live) CK(cudaMemcpyAsync(&gone, e->pt.ctr + kPtGone, 4, cudaMemcpyDeviceToHost, e->stream));
  if ((rc = read_counters(e))) return rc;  // (synchronises the stream: `gone` has arrived)
  const uint32_t n = e->h_cnt->expired;
  e->pt.live -= gone;
  if (n) {
    if (ids) CK(cudaMemcpyAsync(ids, e->d_exp_id, (size_t)n * 8, cudaMemcpyDeviceToHost, e->stream));
    else CK(cudaMemcpyAsync(handles, e->d_exp_id, (size_t)n * 4, cudaMemcpyDeviceToHost, e->stream));
    if (seq) CK(cudaMemcpyAsync(seq, e->d_exp_seq, (size_t)n * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
  }
  erase_active(e, e->h_cnt->erased);
  *n_expired = n;
  return MM_OK;
}

// ---- mm_export / mm_import -------------------------------------------------------------------------------------------
// Section offsets of an image (include/mm_engine.h): off[0] part counts, [1] id, [2] rating, [3] enq_ts, [4] seq,
// [5] mode, [6] active, [7] total bytes.
struct ImgLayout { uint64_t off[8]; };
ImgLayout img_layout(uint32_t n_parts, uint32_t n, uint32_t m, uint32_t idb) {
  auto a8 = [](uint64_t x) { return (x + 7) & ~7ull; };
  const uint64_t bytes[7] = {4ull * n_parts, (uint64_t)idb * n, 4ull * n, 4ull * n, 4ull * n, (uint64_t)n,
                             (uint64_t)idb * m};
  ImgLayout l{};
  l.off[0] = sizeof(mm_image_header);
  for (int k = 0; k < 7; ++k) l.off[k + 1] = a8(l.off[k] + bytes[k]);
  return l;
}
ImgCols img_cols(uint8_t* body, const ImgLayout& l, uint32_t idb) {  // body = the image from section 2 (id) on
  ImgCols c{};
  c.id = body;
  c.rating = reinterpret_cast<int32_t*>(body + (l.off[2] - l.off[1]));
  c.ts = reinterpret_cast<uint32_t*>(body + (l.off[3] - l.off[1]));
  c.seq = reinterpret_cast<uint32_t*>(body + (l.off[4] - l.off[1]));
  c.mode = body + (l.off[5] - l.off[1]);
  c.id_bytes = idb;
  return c;
}
// Section offsets of a party image (include/mm_engine.h): [0] size, [1] seq, [2] enq_ts, [3] mode, [4] id, [5] rating,
// [6] total bytes.
struct PtImgLayout { uint64_t off[7]; };
PtImgLayout pt_img_layout(uint32_t P, uint32_t M, uint32_t W) {
  auto a8 = [](uint64_t x) { return (x + 7) & ~7ull; };
  const uint64_t bytes[6] = {(uint64_t)P, 4ull * P, 4ull * P, (uint64_t)P, (uint64_t)W * M, 4ull * M};
  PtImgLayout l{};
  l.off[0] = sizeof(mm_image_header);
  for (int k = 0; k < 6; ++k) l.off[k + 1] = a8(l.off[k] + bytes[k]);
  return l;
}

uint32_t id_bytes(const mm_engine* e) { return e->dense_ids ? 4u : 8u; }
uint64_t id_limit(const mm_engine* e) { return e->dense_ids ? e->hcap : kTombKey; }

// d_sel <- the partitions of the (mode, group) queues whose byte in `queues` (n_cut bytes) is non-zero
int upload_sel(mm_engine* e, const uint8_t* queues) {
  std::vector<uint8_t> sel(e->n_segs);
  for (uint32_t s = 0; s < e->n_segs; ++s) sel[s] = queues[e->h_part_cut[s]] != 0;
  CK(e->d_sel.reserve(kMaxSegs));
  CK(cudaMemcpyAsync(e->d_sel, sel.data(), e->n_segs, cudaMemcpyHostToDevice, e->stream));
  CK(cudaStreamSynchronize(e->stream));  // `sel` is pageable and goes out of scope
  return MM_OK;
}

// Export pass 1 over the current pool: the live slots of every virtual tile into d_img_tile and of every partition
// into d_img_part[0, n_segs), counting only the partitions in d_sel when `sel` is set.  `a` is left set for pass 2.
int count_tiles(mm_engine* e, bool sel, ImgExportArgs& a) {
  const Pool& p = e->pool[e->cur];
  const uint32_t tiles = tile_count(e, p.n);
  CK(e->d_img_tile.reserve(tiles));
  CK(e->d_img_part.reserve((size_t)3 * e->n_segs + 2));
  CK(cudaMemsetAsync(e->d_img_tile, 0, (size_t)tiles * 4, e->stream));
  CK(cudaMemsetAsync(e->d_img_part, 0, (size_t)e->n_segs * 4, e->stream));
  a = ImgExportArgs{};
  a.pool = p.v; a.meta = p.m; a.n_segs = e->n_segs; a.tile_cnt = e->d_img_tile; a.part_cnt = e->d_img_part;
  a.sel = sel ? e->d_sel.p : nullptr;
  if (p.n) k_img_tiles<kImgBlock, false><<<tile_ctas(e, p.n), kImgBlock, 0, e->stream>>>(a);
  CK(cudaGetLastError());
  return MM_OK;
}

// mm_export (queues = null) and mm_export_queues (queues: n_cut selection bytes; the image has no active section, and
// a call that writes it releases the exported players through k_expire with the same selection and max_wait = 0)
int export_image(mm_engine* e, void* buf, uint64_t cap, uint64_t* n_bytes, const uint8_t* queues) {
  if (e->stage_count) return staged_err(e);
  const Pool& p = e->pool[e->cur];
  const uint32_t idb = id_bytes(e);
  int rc;
  if (queues && (rc = upload_sel(e, queues))) return rc;
  // pass 1: live slots per tile and per partition, the tiles' offsets; the active section
  ImgExportArgs a;
  if ((rc = count_tiles(e, queues != nullptr, a))) return rc;
  CK(cudaMemsetAsync(&e->d_cnt->img_players, 0, 2 * 4, e->stream));  // img_players, img_active
  k_scan_small<<<1, 1024, 0, e->stream>>>(tile_count(e, p.n), e->d_img_tile, &e->d_cnt->img_players);
  const uint32_t act_cap = queues ? 0u : (uint32_t)std::min<uint64_t>(e->n_active, 0xFFFFFFFFu);
  if (e->use_active && act_cap) {
    CK(e->d_img_act.reserve((size_t)act_cap * idb));
    const uint64_t n_tab = e->hcap;
    const uint32_t nb = grid256(e, n_tab, 16);
    k_img_active<<<nb, 256, 0, e->stream>>>(act_view(e), n_tab, p.v.mode, (uint32_t)pool_slots(e), e->gen, e->d_img_act,
                                            idb, act_cap, &e->d_cnt->img_active);
  }
  CK(cudaGetLastError());
  if ((rc = read_counters(e))) return rc;
  const uint32_t n = e->h_cnt->img_players, m = e->h_cnt->img_active;
  if (m > act_cap) return set_err(e, MM_E_STATE, "%u active ids outside the pool, %u in the active set", m, act_cap);
  const ImgLayout l = img_layout(e->n_segs, n, m, idb);
  *n_bytes = l.off[7];
  if (!buf) return MM_OK;
  if (cap < l.off[7]) return set_err(e, MM_E_CAP, "need cap >= %llu", (unsigned long long)l.off[7]);
  // pass 2: the columns, laid out as in the image (padding zero)
  uint8_t* out = static_cast<uint8_t*>(buf);
  const uint64_t col_bytes = l.off[6] - l.off[1];
  CK(e->d_img.reserve(std::max<uint64_t>(col_bytes, 8)));
  if (n) {
    CK(cudaMemsetAsync(e->d_img, 0, col_bytes, e->stream));
    a.out = img_cols(e->d_img, l, idb);
    k_img_tiles<kImgBlock, true><<<tile_ctas(e, p.n), kImgBlock, 0, e->stream>>>(a);
    CK(cudaGetLastError());
  }
  mm_image_header h{};
  h.magic = queues ? MM_QUEUE_IMAGE_MAGIC : MM_IMAGE_MAGIC; h.version = MM_IMAGE_VERSION; h.abi_version = MM_ABI_VERSION; h.id_bytes = idb;
  h.total_bytes = l.off[7]; h.n_parts = e->n_segs; h.n_players = n; h.n_active = m; h.seq_next = e->seq_next;
  h.config = e->cfg;
  std::memcpy(out, &h, sizeof(h));
  std::memset(out + l.off[0], 0, l.off[1] - l.off[0]);  // the part counts' padding
  std::memset(out + l.off[6], 0, l.off[7] - l.off[6]);  // the active section and its padding
  CK(cudaMemcpyAsync(out + l.off[0], e->d_img_part, (size_t)e->n_segs * 4, cudaMemcpyDeviceToHost, e->stream));
  if (n) CK(cudaMemcpyAsync(out + l.off[1], e->d_img, col_bytes, cudaMemcpyDeviceToHost, e->stream));
  if (m) CK(cudaMemcpyAsync(out + l.off[6], e->d_img_act, (size_t)m * idb, cudaMemcpyDeviceToHost, e->stream));
  if (!(queues && n)) {
    CK(cudaStreamSynchronize(e->stream));
    return MM_OK;
  }
  // release the exported players, as mm_remove would: dead slots until the next tick (max_wait 0: every selected one)
  ExpireArgs x{};
  x.commit = 1; x.sel = e->d_sel;
  if ((rc = launch_expire(e, x)) || (rc = read_counters(e))) return rc;
  erase_active(e, e->h_cnt->erased);
  return MM_OK;
}

// the image-sized scratch of mm_export / mm_import / mm_merge (cudaFree waits for the work that uses it)
void free_img_scratch(mm_engine* e) {
  e->d_img.reset(); e->d_img_act.reset(); e->d_mrg_src.reset(); e->d_mrg_code.reset(); e->d_mrg_seen.reset();
  e->d_rq_u.reset(); e->d_rg.reset();
}

// The current pool buffer and the active set back to an empty engine's state.
int clear_engine(mm_engine* e) {
  Pool& p = e->pool[e->cur];
  CK(cudaMemsetAsync(p.m.fill, 0, (size_t)e->n_segs * 4, e->stream));
  CK(cudaMemsetAsync(p.m.bump, 0, 4, e->stream));
  CK(cudaMemsetAsync(p.m.tot, 0, ((size_t)e->Kp + 1) * 4, e->stream));
  if (p.m.chist) CK(cudaMemsetAsync(p.m.chist, 0, (size_t)e->n_chunks * kChunkHist * 4, e->stream));
  CK(cudaMemsetAsync(p.v.bin, 0xFF, pool_slots(e) * 2, e->stream));
  p.n = 0;
  p.held = 0;
  if (e->use_active) {
    int rc = clear_table(e, e->tab[e->tcur]);
    if (rc) return rc;
  }
  e->n_active = 0; e->n_tomb = 0;
  CK(cudaStreamSynchronize(e->stream));
  return MM_OK;
}

// the config fields an image must share with the engine that loads it (capacity, active_capacity, device may differ)
bool same_layout(const mm_config& a, const mm_config& c) {
  bool same = a.n_groups == c.n_groups && a.default_group == c.default_group && a.n_modes == c.n_modes &&
              a.order_mode == c.order_mode && a.flags == c.flags;
  for (uint32_t g = 0; same && g < c.n_groups; ++g) same = a.group_lo[g] == c.group_lo[g] && a.group_hi[g] == c.group_hi[g];
  for (uint32_t m = 0; same && m < c.n_modes; ++m)
    same = a.modes[m].teams == c.modes[m].teams && a.modes[m].team_size == c.modes[m].team_size;
  return same;
}

// The header checks of mm_import, mm_merge and mm_import_regroup.  `magic` is the image kind's, `prefix` starts every
// message, and `no_active` refuses an active section (null: one is allowed).  regroup = null: the image's config must
// be the engine's (same_layout); otherwise it may differ except on the id width and MM_F_NO_DEDUPE, must be a valid
// config (capacity aside), and *regroup receives its layout, whose partition count the image must have.
// -> the header, its layout and the partition counts
int check_header(mm_engine* e, const uint8_t* buf, uint64_t nb, uint32_t magic, const char* prefix,
                 const char* bad_magic, const char* no_active, mm_image_header& h, ImgLayout& l,
                 std::vector<uint32_t>& cnt, Layout* regroup = nullptr) {
  auto bad = [&](const char* what) { return set_err(e, MM_E_ARG, "%s: %s", prefix, what); };
  if (nb < sizeof(h)) return bad("shorter than its header");
  std::memcpy(&h, buf, sizeof(h));
  if (h.magic != magic) return bad(bad_magic);
  if (h.version != MM_IMAGE_VERSION || h.abi_version != MM_ABI_VERSION) return bad("unknown version");
  if (h.id_bytes != id_bytes(e)) return bad("id width differs from the engine's");
  uint32_t n_parts = e->n_segs;
  if (regroup) {
    if ((h.config.flags ^ e->cfg.flags) & (MM_F_NO_DEDUPE | MM_F_DENSE_IDS))
      return bad("MM_F_NO_DEDUPE or MM_F_DENSE_IDS differs from the engine's");
    mm_config c = h.config;
    c.capacity = 1;  // the writer's capacity does not matter here
    if (check_config(&c) || build_layout(c, *regroup)) return bad("the image's config is not a valid config");
    n_parts = regroup->n_segs;
  }
  if (h.n_parts != n_parts)
    return bad(regroup ? "partition count differs from the image config's layout"
                       : "partition count differs from the engine's layout");
  l = img_layout(h.n_parts, h.n_players, h.n_active, h.id_bytes);
  if (h.total_bytes != l.off[7] || nb != l.off[7]) return bad("length does not match the header's section counts");
  if (!regroup && !same_layout(h.config, e->cfg))
    return bad("config differs from the engine's (groups, default_group, modes, order_mode or flags)");
  if (no_active && h.n_active) return bad(no_active);
  cnt.resize(n_parts);
  std::memcpy(cnt.data(), buf + l.off[0], (size_t)n_parts * 4);
  uint64_t sum = 0;
  for (uint32_t q : cnt) sum += q;
  if (sum != h.n_players) return bad("partition counts do not add up to the player count");
  return MM_OK;
}

// the kImg* bits the device checks of an image's players set, named
int img_err(mm_engine* e, const char* prefix, uint32_t err) {
  return set_err(e, MM_E_ARG, "%s:%s%s%s%s%s%s", prefix, err & kImgBadId ? " id out of range" : "",
                 err & kImgBadMode ? " mode out of range" : "", err & kImgBadRating ? " rating outside its partition" : "",
                 err & kImgBadSeq ? " sequence numbers out of order" : "", err & kImgDup ? " duplicate id" : "",
                 err & kImgFull ? " active set full" : "");
}

// The capacity refusals of a load: n queued players and m active ids outside the pool.
int load_fits(mm_engine* e, uint64_t n, uint64_t m) {
  if (n > e->capacity) return set_err(e, MM_E_CAP, "%llu players, capacity %u", (unsigned long long)n, e->capacity);
  if (e->use_active && !e->dense_ids && (n + m) * 4 > e->hcap * 3)
    return set_err(e, MM_E_CAP, "%llu active ids, active set holds %llu", (unsigned long long)(n + m),
                   (unsigned long long)(e->hcap * 3 / 4));
  return MM_OK;
}

// The load tail of mm_import and mm_import_regroup: a fresh engine's pool and active set from image columns already in
// device memory — cnt[s] players of layout partition s, in `cols` partition by partition in enqueue order, and the m
// ids of the active section at `act`.  Every partition goes on consecutive chunks, in partition order; k_img_load
// checks every player under the engine's layout while it writes it, k_img_insert refuses a repeated id, and a failed
// check leaves the engine empty and fresh.
// k_img_load's arguments: n players of `in` into pool p, partition s's first at part_off[s], laid out from slot_base[s].
ImgLoadArgs load_args(mm_engine* e, const Pool& p, const ImgCols& in, uint32_t n, const uint32_t* part_off,
                      const uint32_t* slot_base, uint32_t seq_next) {
  ImgLoadArgs la{};
  la.pool = p.v; la.meta = p.m; la.in = in; la.n = n; la.n_segs = e->n_segs;
  la.part_off = part_off; la.slot_base = slot_base;
  la.bm = bin_map(e); la.grp_lut = e->d_grp_lut; la.bin_seg = e->d_bin_seg; la.seg_bin_lo = e->d_seg_bin_lo;
  la.mode_tsize = e->d_mode_tsize; la.n_modes = e->cfg.n_modes; la.seq_next = seq_next; la.id_limit = id_limit(e);
  la.err = &e->d_cnt->img_err;
  return la;
}

int load_columns(mm_engine* e, const std::vector<uint32_t>& cnt, const ImgCols& cols, uint32_t n, const void* act,
                 uint32_t m, uint32_t seq_next, const char* prefix) {
  std::vector<uint32_t> tab((size_t)e->n_segs * e->n_chunks, 0), off_base(2 * (size_t)e->n_segs + 1);
  uint32_t chunk = 0, idx = 0;
  for (uint32_t s = 0; s < e->n_segs; ++s) {
    const uint32_t nch = (cnt[s] + kTile - 1) / kTile;
    for (uint32_t k = 0; k < nch; ++k) tab[(size_t)s * e->n_chunks + k] = chunk + k;
    off_base[s] = idx;
    off_base[e->n_segs + 1 + s] = chunk * kTile;
    idx += cnt[s];
    chunk += nch;
  }
  off_base[e->n_segs] = idx;
  int rc;
  if ((rc = clear_engine(e))) return rc;
  Pool& p = e->pool[e->cur];
  CK(e->d_img_part.reserve((size_t)3 * e->n_segs + 2));
  CK(cudaMemcpyAsync(p.m.fill, cnt.data(), (size_t)e->n_segs * 4, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(p.m.chunk_tab, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(p.m.bump, &chunk, 4, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(e->d_img_part, off_base.data(), off_base.size() * 4, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemsetAsync(&e->d_cnt->img_err, 0, 4, e->stream));
  const uint32_t grid = grid256(e, n, 32);
  if (n)
    k_img_load<<<grid, 256, 0, e->stream>>>(
        load_args(e, p, cols, n, e->d_img_part, e->d_img_part + e->n_segs + 1, seq_next));
  if (e->use_active) {
    const ActiveView av = act_view(e);
    if (n) k_img_insert<<<grid, 256, 0, e->stream>>>(cols.id, cols.id_bytes, n, id_limit(e), av, &e->d_cnt->img_err);
    if (m) {
      const uint32_t g2 = grid256(e, m, 32);
      k_img_insert<<<g2, 256, 0, e->stream>>>(act, cols.id_bytes, m, id_limit(e), av, &e->d_cnt->img_err);
    }
  }
  CK(cudaGetLastError());
  if ((rc = read_counters(e))) return rc;
  if (const uint32_t err = e->h_cnt->img_err) {
    if ((rc = clear_engine(e))) return rc;
    return img_err(e, prefix, err);
  }
  p.n = n;
  e->seq_next = seq_next;
  if (e->use_active) e->n_active = (uint64_t)n + m;
  e->fresh = false;
  e->match_valid = false;
  e->last_batch_n = 0;
  if (e->use_active && n) {  // the queued players' entries point at their slots
    k_restamp<<<dim3(e->n_chunks, e->n_segs), 256, 0, e->stream>>>(p.v, p.m, act_view(e), e->gen, nullptr);
    CK(cudaGetLastError());
  }
  CK(cudaStreamSynchronize(e->stream));
  return MM_OK;
}

int import_image(mm_engine* e, const uint8_t* buf, uint64_t nb) {
  if (!e->fresh || e->stage_count)
    return set_err(e, MM_E_STATE, "mm_import needs a fresh engine (nothing enqueued, imported or restored)");
  mm_image_header h;
  ImgLayout l;
  std::vector<uint32_t> cnt;
  int rc = check_header(e, buf, nb, MM_IMAGE_MAGIC, "image rejected", "bad magic",
                        e->use_active ? nullptr : "active section in an image of an engine without an active set", h, l,
                        cnt);
  if (rc || (rc = load_fits(e, h.n_players, h.n_active))) return rc;
  const uint64_t body = nb - l.off[1];  // columns and active section
  CK(e->d_img.reserve(std::max<uint64_t>(body, 8)));
  if (body) CK(cudaMemcpyAsync(e->d_img, buf + l.off[1], body, cudaMemcpyHostToDevice, e->stream));
  return load_columns(e, cnt, img_cols(e->d_img, l, h.id_bytes), h.n_players, e->d_img + (l.off[6] - l.off[1]),
                      h.n_active, h.seq_next, "image rejected");
}

// live players per partition of the current pool, restricted to the partitions in d_sel (the export count pass)
int count_live(mm_engine* e, std::vector<uint32_t>& per_part) {
  per_part.assign(e->n_segs, 0);
  if (!e->pool[e->cur].n) return MM_OK;
  ImgExportArgs a;
  int rc = count_tiles(e, true, a);
  if (rc) return rc;
  CK(cudaMemcpyAsync(per_part.data(), e->d_img_part, (size_t)e->n_segs * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return MM_OK;
}

// mm_merge: every check first (header, config, the queues' live players here, the device pre-pass over the players,
// the capacities and the reject list's size), then one ingest batch through enq_prepare / enq_chunk / enq_finish with
// its codes in d_mrg_code, so that mm_enqueue_rejects still reads the last mm_enqueue* batch.
int merge_image(mm_engine* e, const uint8_t* buf, uint64_t nb, uint32_t cap, uint32_t* rejected, uint32_t* n_rejected) {
  if (e->stage_count) return staged_err(e);
  mm_image_header h;
  ImgLayout l;
  std::vector<uint32_t> cnt;
  int rc = check_header(e, buf, nb, MM_QUEUE_IMAGE_MAGIC, "queue image rejected",
                        "bad magic (not an mm_export_queues image)", "a queue image has no active section", h, l, cnt);
  if (rc) return rc;
  const uint32_t n = h.n_players;
  if (n == 0) return MM_OK;
  std::vector<uint32_t> off(e->n_segs + 1, n);  // first image index of each partition
  for (uint32_t s = 0, sum = 0; s < e->n_segs; ++s) { off[s] = sum; sum += cnt[s]; }
  // the queues the image fills must hold no live player here
  std::vector<uint8_t> touched(e->n_cut, 0);
  for (uint32_t s = 0; s < e->n_segs; ++s)
    if (cnt[s]) touched[e->h_part_cut[s]] = 1;
  if ((rc = upload_sel(e, touched.data()))) return rc;
  std::vector<uint32_t> live;
  if ((rc = count_live(e, live))) return rc;
  for (uint32_t s = 0; s < e->n_segs; ++s)
    if (live[s]) {
      const uint32_t c = e->h_part_cut[s];
      return set_err(e, MM_E_STATE, "queue (mode %u, group %u) holds %u live players here", c / e->cfg.n_groups,
                     c % e->cfg.n_groups, live[s]);
    }
  // upload once; the pre-pass checks every player and writes the ingest batch in the queues' enqueue order
  if ((rc = ensure_enq_scratch(e, n))) return rc;
  const uint64_t body = l.off[6] - l.off[1];
  CK(e->d_img.reserve(std::max<uint64_t>(body, 8)));
  CK(e->d_mrg_src.reserve((size_t)n + 64));
  CK(e->d_img_part.reserve((size_t)3 * e->n_segs + 2));
  CK(cudaMemcpyAsync(e->d_img, buf + l.off[1], body, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(e->d_img_part, off.data(), off.size() * 4, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemsetAsync(&e->d_cnt->img_err, 0, 2 * 4, e->stream));  // img_err, mrg_dups
  const uint32_t grid = grid256(e, n, 32);
  MrgOrderArgs oa{};
  oa.in = img_cols(e->d_img, l, h.id_bytes); oa.n = n; oa.n_segs = e->n_segs; oa.part_off = e->d_img_part;
  oa.part_cut = e->d_part_cut; oa.cut_lp_lo = e->d_cut_lp_lo; oa.bm = bin_map(e); oa.grp_lut = e->d_grp_lut;
  oa.bin_seg = e->d_bin_seg; oa.n_modes = e->cfg.n_modes; oa.seq_next = h.seq_next; oa.id_limit = id_limit(e);
  oa.out_id = e->d_in_id; oa.out_rating = e->d_in_rating; oa.out_mode = e->d_in_mode; oa.out_ts = e->d_in_ts;
  oa.src = e->d_mrg_src; oa.err = &e->d_cnt->img_err;
  k_mrg_order<<<grid, 256, 0, e->stream>>>(oa);
  CK(cudaGetLastError());
  // the exact reject count, when the reject list or a capacity could be too small for every player being queued
  const Pool& p = e->pool[e->cur];
  const bool hashed = e->use_active && !e->dense_ids;
  const bool tight = (uint64_t)p.n + p.held + n > e->capacity || (hashed && (e->n_active + n) * 4 > e->hcap * 3);
  if (e->use_active && (cap < n || tight)) {
    const uint64_t sc = seen_keys(n);
    CK(e->d_mrg_seen.reserve(sc));
    CK(cudaMemsetAsync(e->d_mrg_seen, 0xFF, sc * 8, e->stream));
    k_mrg_dups<<<grid, 256, 0, e->stream>>>(e->d_in_id, n, act_view(e), e->d_mrg_seen, sc - 1, &e->d_cnt->mrg_dups);
    CK(cudaGetLastError());
  }
  if ((rc = read_counters(e))) return rc;
  if (const uint32_t err = e->h_cnt->img_err) return img_err(e, "queue image rejected", err);
  const uint32_t n_rej = e->h_cnt->mrg_dups, accepted = n - n_rej;
  if (n_rej > cap) {
    *n_rejected = n_rej;
    return set_err(e, MM_E_CAP, "%u rejected players, cap %u", n_rej, cap);
  }
  if ((uint64_t)p.n + p.held + accepted > e->capacity)
    return set_err(e, MM_E_CAP, "%u players merged into %u slots in use, capacity %u", accepted, p.n + p.held,
                   e->capacity);
  if (hashed && (e->n_active + accepted) * 4 > e->hcap * 3)
    return set_err(e, MM_E_CAP, "active set full: %llu ids resident, %u merged, capacity %llu",
                   (unsigned long long)e->n_active, accepted, (unsigned long long)(e->hcap * 3 / 4));
  // the ingest, with the merge's own code buffer
  auto ingest = [&]() -> int {
    int r = enq_prepare(e, n, accepted);
    for (uint32_t base = 0; !r && base < n; base += kEnqChunkDev)
      r = enq_chunk(e, base, std::min(kEnqChunkDev, n - base), e->d_in_id, e->d_in_rating, e->d_in_mode, e->d_in_ts, false);
    uint32_t n_acc = 0;
    if (!r) r = enq_finish(e, n, nullptr, &n_acc);
    if (r || n_acc == n) return r;
    uint32_t* d_out = e->d_in_handle;  // free once the batch is in
    CK(cudaMemsetAsync(&e->d_cnt->rejects, 0, 4, e->stream));
    k_mrg_rejects<<<(n + 255) / 256, 256, 0, e->stream>>>(n, e->d_code, e->d_mrg_src, d_out, &e->d_cnt->rejects);
    CK(cudaGetLastError());
    if ((r = read_counters(e))) return r;
    const uint32_t k = std::min(e->h_cnt->rejects, cap);
    CK(cudaMemcpyAsync(rejected, d_out, (size_t)k * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    std::sort(rejected, rejected + k);
    *n_rejected = k;
    return MM_OK;
  };
  const uint32_t last_n = e->last_batch_n;
  std::swap(e->d_code, e->d_mrg_code);
  rc = ingest();
  std::swap(e->d_code, e->d_mrg_code);
  e->last_batch_n = last_n;
  return rc;
}

// mm_remove (take = false: the ids leave the active set too) and mm_take (they stay in it)
int remove_or_take(mm_engine* e, uint32_t n, const uint64_t* id, uint32_t* n_out, bool take) {
  if (n_out) *n_out = 0;
  if (!e || (n && !id)) return MM_E_ARG;
  if (!e->use_active) return MM_E_STATE;
  if (n == 0) return MM_OK;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  int rc = ensure_enq_scratch(e, n);
  if (rc) return rc;
  const Pool& p = e->pool[e->cur];
  CK(cudaMemcpyAsync(e->d_in_id, id, (size_t)n * 8, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemsetAsync(&e->d_cnt->removed, 0, 4, e->stream));
  const bool parties = !take && e->pt.live;  // a removed party member dissolves its whole party
  const PartyView t = pt_view(e, e->pt.cur);
  if (parties) {
    CK(cudaMemsetAsync(e->pt.ctr, 0, kPtWords * 4, e->stream));
    k_pt_mark<<<(n + 255) / 256, 256, 0, e->stream>>>(n, e->d_in_id, act_view(e), t);
  }
  (take ? k_take : k_remove)<<<(n + 255) / 256, 256, 0, e->stream>>>(
      n, e->d_in_id, act_view(e), p.v, p.m, (uint32_t)pool_slots(e), e->gen, e->K, e->d_bin_seg, e->d_seg_bin_lo,
      &e->d_cnt->removed);
  uint32_t gone = 0;
  if (parties) {
    k_pt_dissolve<<<(e->pt.n_rows + 255) / 256, 256, 0, e->stream>>>(e->pt.n_rows, t, act_view(e), &e->d_cnt->removed,
                                                                      e->pt.ctr);
    CK(cudaMemcpyAsync(&gone, e->pt.ctr + kPtGone, 4, cudaMemcpyDeviceToHost, e->stream));
  }
  CK(cudaGetLastError());
  if ((rc = read_counters(e))) return rc;  // (synchronises the stream: `gone` has arrived)
  e->pt.live -= gone;
  if (!take) erase_active(e, e->h_cnt->removed);
  if (n_out) *n_out = e->h_cnt->removed;
  return MM_OK;
}

// ---- mm_requeue (mm_requeue.cuh) ------------------------------------------------------------------------------------
// The columns of up to n players (8-byte ids) carved from `at`, which moves past them.
ImgCols carve_cols(uint8_t*& at, size_t n) {
  auto a8 = [](size_t x) { return (x + 7) & ~(size_t)7; };
  ImgCols c{};
  c.id = at; at += a8(8 * n);
  c.rating = reinterpret_cast<int32_t*>(at); at += a8(4 * n);
  c.ts = reinterpret_cast<uint32_t*>(at); at += a8(4 * n);
  c.seq = reinterpret_cast<uint32_t*>(at); at += a8(4 * n);
  c.mode = at; at += a8(n);
  c.id_bytes = 8;
  return c;
}
size_t cols_bytes(size_t n) { return 21 * n + 40; }

int rq_err(mm_engine* e, uint32_t err) {
  return set_err(e, MM_E_ARG, "requeue refused:%s%s%s%s%s%s%s", err & kRqBadId ? " id out of range" : "",
                 err & kRqBadMode ? " mode out of range" : "", err & kRqBadRating ? " rating without a group" : "",
                 err & kRqOrder ? " entries not in age order" : "",
                 err & kRqSeqNext ? " sequence number equal to seq_next" : "", err & kRqDup ? " duplicate id" : "",
                 err & kRqSeqLive ? " sequence number of a live player of the partition" : "");
}

// Three device phases, each ended by one read of the counters; the pool changes only in the third.
//   1. check and classify the entries, group them, count the touched partitions' live players: every refusal but the
//      sequence collision, and the exact sizes of the gather and the merge
//   2. gather the touched partitions' live players and merge: the collision refusal, then the capacity one
//   3. layout, load, restamp
// The gathered and merged columns are sized by the touched partitions' live players and the entries, never by the pool.
int requeue(mm_engine* e, uint32_t n, const uint64_t* id, const int32_t* rating, const uint8_t* mode, const uint32_t* ts,
            const uint32_t* seq, uint8_t* codes, uint32_t* n_requeued) {
  if (!e->use_active)
    return set_err(e, MM_E_STATE, "requeue needs the active set: an MM_F_NO_DEDUPE engine cannot tell matched from gone");
  if (e->stage_count) return staged_err(e);
  if (n == 0) return MM_OK;
  Pool& p = e->pool[e->cur];
  const uint32_t S = e->n_segs, nblk = (n + kRqItems - 1) / kRqItems;
  int rc;
  if ((rc = ensure_enq_scratch(e, n))) return rc;
  const uint64_t sc = seen_keys(n);
  CK(e->d_mrg_code.reserve((size_t)n + 64));
  CK(e->d_mrg_src.reserve((size_t)n + 64));
  CK(e->d_rq_u.reserve((size_t)n + 64));
  CK(e->d_mrg_seen.reserve(sc));
  CK(e->d_rq_hist.reserve((size_t)S * nblk));
  CK(e->d_rq_seg.reserve(3 * (size_t)S + 2));
  CK(e->d_sel.reserve(kMaxSegs));
  uint32_t* rq_off = e->d_rq_seg;
  uint32_t* m_off = rq_off + S + 1;
  uint32_t* slot_base = m_off + S + 1;
  uint32_t* d_seq = e->d_in_handle;
  CK(cudaMemcpyAsync(e->d_in_id, id, (size_t)n * 8, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(e->d_in_rating, rating, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(e->d_in_mode, mode, n, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(d_seq, seq, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
  if (ts) CK(cudaMemcpyAsync(e->d_in_ts, ts, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemsetAsync(e->d_mrg_seen, 0xFF, sc * 8, e->stream));
  CK(cudaMemsetAsync(&e->d_cnt->img_players, 0, 3 * 4, e->stream));  // img_players, img_active, img_err
  RqCheckArgs ca{};
  ca.id = e->d_in_id; ca.rating = e->d_in_rating; ca.mode = e->d_in_mode; ca.seq = d_seq;
  ca.n = n; ca.n_segs = S; ca.nblk = nblk; ca.bm = bin_map(e); ca.grp_lut = e->d_grp_lut; ca.bin_seg = e->d_bin_seg;
  ca.n_modes = e->cfg.n_modes; ca.seq_next = e->seq_next; ca.id_limit = id_limit(e);
  ca.act = act_view(e); ca.pool_mode = p.v.mode; ca.n_slots = (uint32_t)pool_slots(e); ca.gen = e->gen;
  ca.seen = e->d_mrg_seen; ca.seen_mask = sc - 1;
  ca.code = e->d_mrg_code; ca.part = e->d_part; ca.blockhist = e->d_rq_hist; ca.err = &e->d_cnt->img_err;
  k_rq_check<<<nblk, 256, 0, e->stream>>>(ca);
  k_rq_scan<<<1, 512, 0, e->stream>>>(S, nblk, e->d_rq_hist, rq_off, e->d_sel);
  // export pass 1 over the touched partitions (unselected tiles are skipped without a pool load)
  ImgExportArgs xa;
  if ((rc = count_tiles(e, true, xa))) return rc;
  k_scan_small<<<1, 1024, 0, e->stream>>>(tile_count(e, p.n), e->d_img_tile, &e->d_cnt->img_players);
  k_rq_group<<<nblk, 256, 0, e->stream>>>(n, S, nblk, e->d_part, d_seq, e->seq_next, e->d_rq_hist, e->d_mrg_src,
                                          e->d_rq_u);
  CK(cudaGetLastError());
  // read 1: counters, partition tables, fills, bump
  std::vector<uint32_t> h_rq(S + 1), live(S), fill(S);
  uint32_t bump = 0;
  CK(cudaMemcpyAsync(h_rq.data(), rq_off, (size_t)(S + 1) * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemcpyAsync(live.data(), e->d_img_part, (size_t)S * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemcpyAsync(fill.data(), p.m.fill, (size_t)S * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemcpyAsync(&bump, p.m.bump, 4, cudaMemcpyDeviceToHost, e->stream));
  if ((rc = read_counters(e))) return rc;
  if (const uint32_t err = e->h_cnt->img_err) return rq_err(e, err);
  const uint32_t n_rq = h_rq[S], n_live = e->h_cnt->img_players;
  ImgCols merged{};
  if (n_rq) {
    // export pass 2: the touched partitions' live players, partition by partition, in enqueue order; then the merge
    CK(e->d_img.reserve(cols_bytes(n_live) + cols_bytes((size_t)n_live + n_rq)));
    uint8_t* at = e->d_img;
    const ImgCols gath = carve_cols(at, n_live);
    merged = carve_cols(at, (size_t)n_live + n_rq);
    if (n_live) {
      xa.out = gath;
      k_img_tiles<kImgBlock, true><<<tile_ctas(e, p.n), kImgBlock, 0, e->stream>>>(xa);
    }
    RqMergeArgs ma{};
    ma.live = gath; ma.live_cnt = e->d_img_part; ma.n_segs = S; ma.seq_next = e->seq_next; ma.rq_off = rq_off;
    ma.grp_src = e->d_mrg_src; ma.grp_u = e->d_rq_u;
    ma.id = e->d_in_id; ma.rating = e->d_in_rating; ma.mode = e->d_in_mode; ma.ts = ts ? e->d_in_ts.p : nullptr;
    ma.seq = d_seq; ma.out = merged; ma.m_off = m_off; ma.err = &e->d_cnt->img_err;
    const uint64_t total = (uint64_t)n_live + n_rq;
    const uint32_t grid = grid256(e, total, 32);
    k_rq_merge<<<grid, 256, 0, e->stream>>>(ma);
    CK(cudaGetLastError());
    // read 2: the sequence collision
    if ((rc = read_counters(e))) return rc;
    if (const uint32_t err = e->h_cnt->img_err) return rq_err(e, err);
  }
  // the touched partitions on fresh chunks from the bump on, in partition order (import_image's layout)
  std::vector<uint32_t> base(S, 0);
  uint32_t chunk = bump;
  uint64_t dead = 0, left = 0;  // the touched partitions' dead slots; their chunks, left to the next tick
  for (uint32_t s = 0; s < S; ++s) {
    const uint32_t r = h_rq[s + 1] - h_rq[s];
    if (!r) continue;
    dead += fill[s] - live[s];
    left += (fill[s] + kTile - 1) / kTile;
    base[s] = chunk * kTile;
    chunk += (live[s] + r + kTile - 1) / kTile;
  }
  const uint64_t used = (uint64_t)p.n - dead + n_rq, held = p.held + left * kTile;
  if (used + held > e->capacity)
    return set_err(e, MM_E_CAP, "requeue needs %llu pool slots in use and %llu left to the next tick, capacity %u",
                   (unsigned long long)used, (unsigned long long)held, e->capacity);
  if (n_rq) {
    CK(cudaMemcpyAsync(slot_base, base.data(), (size_t)S * 4, cudaMemcpyHostToDevice, e->stream));
    k_rq_layout<<<S, 256, 0, e->stream>>>(p.m, S, e->d_sel, m_off, slot_base, e->d_seg_bin_lo, e->K, (uint32_t)dead, chunk);
    k_img_load<<<grid256(e, n_live + n_rq, 32), 256, 0, e->stream>>>(
        load_args(e, p, merged, n_live + n_rq, m_off, slot_base, e->seq_next));
    k_restamp<<<dim3(e->n_chunks, S), 256, 0, e->stream>>>(p.v, p.m, act_view(e), e->gen, e->d_sel);
    CK(cudaGetLastError());
  }
  if (codes) CK(cudaMemcpyAsync(codes, e->d_mrg_code, n, cudaMemcpyDeviceToHost, e->stream));
  if ((rc = read_counters(e))) return rc;
  if (n_rq) {
    p.n = (uint32_t)used;
    p.held = (uint32_t)held;
  }
  if (n_requeued) *n_requeued = n_rq;
  if (e->h_cnt->img_err)  // the merged list failed the load's own checks: nothing above lets that happen
    return set_err(e, MM_E_STATE, "requeue: the merged players failed the load checks (0x%x)", e->h_cnt->img_err);
  return MM_OK;
}

// ---- mm_import_regroup / mm_import_regroup_many (mm_regroup.cuh, mm_recut.cuh) -----------------------------------
// The party images of mm_import_regroup_many_parties, as their headers describe them.
struct RpImages {
  std::vector<uint32_t> pbase, mcount, pnblk;  // [K + 1] image k's first party; [K] its members; [K] classify blocks
  std::vector<PtImgLayout> pl;
  uint64_t P = 0, M = 0;                       // parties and members in all
};

// The party images' header checks on the host, against their engine images h (pp null: no party image).
int rp_headers(mm_engine* e, uint32_t K, mm_recut_parties* pp, const std::vector<mm_image_header>& h, RpImages& r) {
  r.pbase.assign(K + 1, 0); r.mcount.assign(K, 0); r.pnblk.assign(K, 0); r.pl.resize(K);
  if (!pp) return MM_OK;
  pp->n_rejected = pp->n_elsewhere = pp->n_loaded = 0;
  for (uint32_t k = 0; k < K; ++k) {
    r.pbase[k] = (uint32_t)r.P;
    const uint64_t nb = pp->n_bytes ? pp->n_bytes[k] : 0;
    const uint8_t* b = pp->bufs ? static_cast<const uint8_t*>(pp->bufs[k]) : nullptr;
    if (!b || !nb) continue;
    auto bad = [&](const char* what) { return set_err(e, MM_E_ARG, "party image %u rejected: %s", k, what); };
    mm_image_header ph;
    if (nb < sizeof(ph)) return bad("shorter than its header");
    std::memcpy(&ph, b, sizeof(ph));
    if (ph.magic != MM_PARTY_IMAGE_MAGIC) return bad("bad magic (not an mm_export_parties image)");
    if (ph.version != MM_IMAGE_VERSION || ph.abi_version != MM_ABI_VERSION) return bad("unknown version");
    if (ph.id_bytes != h[0].id_bytes) return bad("id width differs from the engine's");
    if (ph.config.flags & MM_F_NO_DEDUPE) return bad("written by an MM_F_NO_DEDUPE engine");
    r.pl[k] = pt_img_layout(ph.n_parts, ph.n_players, ph.id_bytes);
    if (ph.n_active || ph.total_bytes != r.pl[k].off[6] || nb != r.pl[k].off[6])
      return bad("length does not match the header's section counts");
    if (!same_layout(ph.config, h[k].config) || ph.seq_next != h[k].seq_next)
      return bad("config or seq_next differs from its engine image's (not written at the same stop)");
    r.P += ph.n_parts;
    r.M += ph.n_players;
    r.mcount[k] = ph.n_players;
    r.pnblk[k] = (ph.n_parts + kRqItems - 1) / kRqItems;
    if (r.P > 0x7FFFFFFFu || r.M > 0x7FFFFFFFu) return set_err(e, MM_E_CAP, "more than 2^31 - 1 parties or members");
  }
  r.pbase[K] = (uint32_t)r.P;
  if (r.P) {
    if (e->cfg.order_mode != MM_ORDER_RATING) return set_err(e, MM_E_ARG, "party images need MM_ORDER_RATING");
    if (!e->use_active) return set_err(e, MM_E_ARG, "an MM_F_NO_DEDUPE engine cannot hold parties");
    if (!e->pt.cap) return set_err(e, MM_E_STATE, "no party capacity: set the option party_capacity first");
  }
  return MM_OK;
}

// The buffers of one merge of K images' runs (mm_recut.cuh): the solos' over S partitions, the parties' over C queues.
// one = {0, kept, runs, kmax}; pair / ord / run / kq: k_rg_plan's; s2 / key: the ping-pong of virtual index and
// (stamp, image, age) key; head / agg / carry / first: the running-max scan.
struct RcRuns {
  uint32_t *glob, *one, *pair, *run, *kq, *s2[2], *first;
  uint16_t* ord;
  RcKey* key[2];
  uint8_t* head;
  RcSeg *agg, *carry;
};

// regroup_many's scratch in d_rg, one member per array; the carve in regroup_many gives each its count (0 where the
// call does not use it).  sr: K > 1, the solos' partition runs merged; pr: with parties too, their queue runs.
struct RgScratch {
  unsigned long long *seen, *seqset;
  uint8_t *grp, *sel, *keep, *out, *pbody, *psel, *pkeep, *psz;
  uint16_t *lut, *bseg, *ord, *part, *pimg, *ident, *img, *qv, *ppart, *pk;
  uint32_t *off, *rq, *skip, *hist, *pair, *run, *kq, *src[2], *age[2], *rej, *pos, *base;
  uint32_t *pbase, *pctr, *pmoff, *pflag, *phist, *rqp, *psrc, *page, *rsrc, *rsz, *fin;
  int32_t* pR;
  ImgCols* imgs;
  PtImgCols* pcols;
  RcRuns sr, pr;
};

// p <- the next n T at cursor o over base (null: only o moves), 16-byte aligned.
template <class T>
void rg_take(uint8_t* base, size_t& o, T*& p, size_t n) {
  p = base ? reinterpret_cast<T*>(base + o) : nullptr;
  o += (n * sizeof(T) + 15) & ~(size_t)15;
}

// The ⌈log2 runs⌉ rounds of k_rg_merge over ma's runs (ma.n_img_segs of them), ping-ponging between (src, key)[0] and
// [1] from [0]; the rounds past kmax's need return at once.  -> the index of the pair that holds the merged runs.
template <class U>
uint32_t rg_rounds(mm_engine* e, RgMergeArgsT<U> ma, uint32_t* const src[2], U* const key[2], uint32_t grid) {
  uint32_t t = 0;
  for (; (1u << t) < ma.n_img_segs; ++t) {
    ma.round = t;
    ma.src_in = src[t & 1]; ma.u_in = key[t & 1]; ma.src_out = src[(t + 1) & 1]; ma.u_out = key[(t + 1) & 1];
    k_rg_merge<<<grid, 256, 0, e->stream>>>(ma);
  }
  return t & 1;
}

// The runs of K images merged into one order per new partition or queue (runs n_segs).  Image k's kept runs are at
// rq[(n_segs + 2) * k] in src / age from first[k] on, its rows virtual indices vbase + first[k] on with stamps ts[k],
// and their runs new partitions qoff + run in qv.  The stamps become running maxima over each run; then the rounds over
// K, whose result k_rc_finish / k_rp_norm find by r.one[3].  rows: the length of r.s2; nrb, grid: the scan's blocks
// and the rounds' grid.
int rc_merge(mm_engine* e, uint32_t K, uint32_t n_segs, const uint32_t* rq, const std::vector<uint32_t>& first,
             const uint32_t* const src[2], const uint32_t* const age[2], const std::vector<const uint32_t*>& ts,
             uint32_t vbase, uint32_t qoff, uint16_t* img, uint16_t* qv, const RcRuns& r, size_t rows, uint32_t nrb,
             uint32_t grid) {
  const uint32_t n_kmax[2] = {n_segs, 0};  // one[2] = n_segs for the rounds into one list; one[3] = kmax
  CK(cudaMemcpyAsync(r.one + 2, n_kmax, 8, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemsetAsync(r.ord, 0, 2 * (size_t)K * n_segs, e->stream));
  CK(cudaMemsetAsync(r.s2[0], 0, 4 * rows, e->stream));  // holes (a refused image) stay in range
  CK(cudaMemsetAsync(r.s2[1], 0, 4 * rows, e->stream));
  k_rc_sum<<<1, 1024, 0, e->stream>>>(K, n_segs, rq, r.glob, r.one, r.pair);
  k_rg_plan<<<1, 1024, 0, e->stream>>>(K, n_segs, r.pair, r.glob, r.ord, r.run, r.kq, r.one + 3);
  for (uint32_t k = 0; k < K; ++k) {
    const uint32_t n = first[k + 1] - first[k];
    if (!n) continue;
    RcGatherArgs ga{};
    ga.k = k; ga.base = vbase + first[k]; ga.n = n; ga.n_segs = n_segs; ga.n_img = K; ga.rq_off = rq + (n_segs + 2) * k;
    ga.kmax = &e->d_cnt->rg_kmax; ga.src[0] = src[0] + first[k]; ga.src[1] = src[1] + first[k];
    ga.age[0] = age[0] + first[k]; ga.age[1] = age[1] + first[k]; ga.ord = r.ord; ga.run_start = r.run;
    ga.ts = ts[k]; ga.src_out = r.s2[0]; ga.key_out = r.key[0]; ga.head = r.head; ga.img = img; ga.qv = qv;
    ga.qoff = qoff; ga.err = &e->d_cnt->img_err;
    k_rc_gather<<<grid256(e, n, 32), 256, 0, e->stream>>>(ga);
  }
  if (nrb) {  // (no solo: parties only)
    k_rc_runmax<<<nrb, 256, 0, e->stream>>>(r.one + 1, r.key[0], r.head, r.agg, r.first);
    k_rc_carry<<<1, 1024, 0, e->stream>>>(r.one + 1, r.agg, r.carry);
    k_rc_apply<<<nrb, 256, 0, e->stream>>>(r.one + 1, r.key[0], r.carry, r.first);
  }
  rg_rounds(e, RgMergeArgsT<RcKey>{r.glob, n_segs, K, 0, img, r.ord, r.run, r.kq, r.one + 3}, r.s2, r.key, grid);
  return MM_OK;
}

// Each image's reject bucket (run n_segs of its rq row, in src from first[k]), in image order: (image, index)
// ascending; then rej_image, when asked for.
int rg_rejects(mm_engine* e, uint32_t K, uint32_t n_segs, const std::vector<uint32_t>& h_rq, const uint32_t* src,
               const std::vector<uint32_t>& first, uint32_t* rej_index, uint32_t* rej_image) {
  const size_t R = n_segs + 2;
  for (uint32_t k = 0, w = 0; k < K; ++k) {
    const uint32_t* r = h_rq.data() + R * k;
    if (r[n_segs + 1] > r[n_segs])
      CK(cudaMemcpyAsync(rej_index + w, src + first[k] + r[n_segs], (size_t)(r[n_segs + 1] - r[n_segs]) * 4,
                         cudaMemcpyDeviceToHost, e->stream));
    w += r[n_segs + 1] - r[n_segs];
  }
  CK(cudaStreamSynchronize(e->stream));
  if (rej_image)
    for (uint32_t k = 0, w = 0; k < K; ++k)
      for (uint32_t j = h_rq[R * k + n_segs]; j < h_rq[R * k + n_segs + 1]; ++j) rej_image[w++] = k;
  return MM_OK;
}

// K images of one config: each runs the regroup pipeline on its own; for K > 1 the images' runs are merged and the
// kept players renumbered on the device.  Every refusal is decided by one read of the counters, before the load tail
// writes the pool.  `who` names the call in the state refusal; keep_cut: n_cut selection bytes (null: all); act_img:
// the image whose active section is taken (>= K: none); pp: the party images (mm_import_regroup_many_parties) or
// null.  Without a non-empty party image every step is mm_import_regroup_many's.
int regroup_many(mm_engine* e, const char* who, uint32_t K, const uint8_t* const* bufs, const uint64_t* nbs,
                 const uint8_t* keep_cut, uint32_t act_img, uint32_t cap, uint32_t* rej_image, uint32_t* rej_index,
                 uint32_t* n_rejected, uint32_t* n_elsewhere, mm_recut_parties* pp) {
  if (!e->fresh || e->stage_count)
    return set_err(e, MM_E_STATE, "%s needs a fresh engine (nothing enqueued, imported or restored)", who);
  if (K == 0 || K > kRcMaxImages) return set_err(e, MM_E_ARG, "n_images must be 1 .. %u", kRcMaxImages);
  if (act_img != 0xFFFFFFFFu && act_img >= K) return set_err(e, MM_E_ARG, "active_image out of range");
  std::vector<mm_image_header> h(K);
  std::vector<ImgLayout> l(K);
  std::vector<std::vector<uint32_t>> cnt(K);
  Layout y;  // the images' layout
  int rc;
  for (uint32_t k = 0; k < K; ++k) {
    const char* no_active =
        k == act_img && !e->use_active ? "active section in an image of an engine without an active set" : nullptr;
    if ((rc = check_header(e, bufs[k], nbs[k], MM_IMAGE_MAGIC, "image rejected", "bad magic", no_active, h[k], l[k],
                           cnt[k], &y)))
      return rc;
    if (k && !same_layout(h[k].config, h[0].config))
      return set_err(e, MM_E_ARG, "image rejected: its config differs from image 0's");
  }
  const uint32_t S = e->n_segs, SI = y.n_segs, idb = h[0].id_bytes;
  const uint32_t m = act_img < K ? h[act_img].n_active : 0;
  RpImages ri;
  if ((rc = rp_headers(e, K, pp, h, ri))) return rc;
  const std::vector<uint32_t>& pbase = ri.pbase;
  const uint64_t P = ri.P;
  const bool parties = P != 0;
  const uint32_t C = e->n_cut;
  std::vector<uint32_t> base(K + 1, 0), nblk(K);
  uint64_t total = 0;
  for (uint32_t k = 0; k < K; ++k) {
    total += h[k].n_players;
    if (total > 0x7FFFFFFFu) return set_err(e, MM_E_CAP, "more than 2^31 - 1 players in the images");
    base[k + 1] = (uint32_t)total;
    nblk[k] = (h[k].n_players + kRqItems - 1) / kRqItems;
  }
  const uint32_t N = base[K];
  std::vector<uint64_t> boff(K + 1, 0);  // each image's body (section 2 on) in d_img, 16-byte aligned
  for (uint32_t k = 0; k < K; ++k) boff[k + 1] = boff[k] + ((nbs[k] - l[k].off[1] + 15) & ~(uint64_t)15);
  CK(e->d_img.reserve(std::max<uint64_t>(boff[K], 8)));
  for (uint32_t k = 0; k < K; ++k)
    if (nbs[k] > l[k].off[1])
      CK(cudaMemcpyAsync(e->d_img + boff[k], bufs[k] + l[k].off[1], nbs[k] - l[k].off[1], cudaMemcpyHostToDevice,
                         e->stream));
  std::vector<ImgCols> in(K);
  for (uint32_t k = 0; k < K; ++k) in[k] = img_cols(e->d_img + boff[k], l[k], idb);
  const void* act = act_img < K ? (const void*)(e->d_img + boff[act_img] + (l[act_img].off[6] - l[act_img].off[1]))
                                : (const void*)e->d_img.p;
  const uint32_t seq_next = K == 1 ? h[0].seq_next : 0;  // K > 1: renumbered, seq_next = the kept count
  if (n_elsewhere) *n_elsewhere = 0;
  if (N == 0 && !parties)
    return load_columns(e, std::vector<uint32_t>(S, 0), in[0], 0, act, m, seq_next, "image rejected");
  // scratch: the images' tables, the classification, the scatter and merge buffers, the gathered columns
  const uint64_t sc = e->use_active ? seen_keys((uint64_t)N + m + ri.M) : 0;  // the repeated-id set
  std::vector<uint32_t> off((size_t)K * (SI + 1), 0);
  for (uint32_t k = 0; k < K; ++k)
    for (uint32_t s = 0; s < SI; ++s) off[(size_t)k * (SI + 1) + s + 1] = off[(size_t)k * (SI + 1) + s] + cnt[k][s];
  std::vector<uint8_t> keep;  // per new partition
  if (keep_cut) {
    keep.resize(S);
    for (uint32_t q = 0; q < S; ++q) keep[q] = keep_cut[e->h_part_cut[q]] != 0;
  }
  uint64_t hist_n = 0, phist_n = 0;
  for (uint32_t k = 0; k < K; ++k) {
    hist_n += (uint64_t)(S + 1) * nblk[k];
    phist_n += (uint64_t)(C + 1) * ri.pnblk[k];
  }
  std::vector<uint64_t> pboff(K + 1, 0);  // each party image's body (section 1 on) in x.pbody, 16-byte aligned
  for (uint32_t k = 0; k < K; ++k)
    pboff[k + 1] = pboff[k] + (pbase[k + 1] > pbase[k] ? (ri.pl[k].off[6] - ri.pl[k].off[0] + 15) & ~(uint64_t)15 : 0);
  const bool many = K > 1;
  const size_t pair_n = (size_t)SI * S, R1 = S + 2, R2 = C + 2;  // per image: (image partition, new partition) pairs
  const uint32_t nrb = (N + kRcBlock - 1) / kRcBlock, nrbp = (uint32_t)((P + kRcBlock - 1) / kRcBlock);
  const uint64_t psc = parties ? seen_keys(P) : 0;
  RgScratch x;
  auto carve = [&](uint8_t* sb) {  // -> the bytes in use
    size_t o = 0;
    auto take = [&](auto*& p, size_t n) { rg_take(sb, o, p, n); };
    auto runs = [&](RcRuns& r, size_t on, size_t ns, size_t rows, size_t heads, size_t nb) {
      take(r.glob, on * (ns + 1)); take(r.one, on * 4); take(r.pair, on * K * ns); take(r.ord, on * K * ns);
      take(r.run, on * ns * (K + 1)); take(r.kq, on * ns);
      take(r.s2[0], on * rows); take(r.s2[1], on * rows); take(r.key[0], on * rows); take(r.key[1], on * rows);
      take(r.head, on * heads); take(r.agg, on * nb); take(r.carry, on * nb); take(r.first, on * nb);
    };
    const size_t M1 = many, P1 = parties, PM = parties && many, NP = N + P;
    take(x.seen, sc); take(x.lut, y.KR); take(x.grp, y.KR); take(x.bseg, y.Kp); take(x.off, off.size());
    take(x.rq, R1 * K); take(x.sel, S + 1); take(x.keep, keep.size()); take(x.skip, K); take(x.hist, hist_n);
    take(x.pair, pair_n * K); take(x.ord, pair_n * K); take(x.run, (size_t)S * (SI + 1) * K); take(x.kq, (size_t)S * K);
    take(x.part, N); take(x.pimg, N);
    take(x.src[0], N); take(x.src[1], N); take(x.age[0], N); take(x.age[1], N);
    take(x.rej, many ? 0 : N); take(x.out, cols_bytes(NP));
    runs(x.sr, M1, S, NP, N, nrb);
    take(x.ident, M1 * 2 * ((size_t)S + C)); take(x.img, M1 * NP); take(x.qv, M1 * NP); take(x.pos, M1 * NP);
    take(x.imgs, M1 * K); take(x.base, M1 * K);
    take(x.pbody, pboff[K]); take(x.pcols, P1 * K); take(x.pbase, P1 * (K + 1)); take(x.seqset, psc);
    take(x.pctr, P1 * (kRpWords + 3 * K));  // RpCtr | skip [K] | kept members [K] | member sums [K]
    take(x.pmoff, P); take(x.ppart, P); take(x.pk, P); take(x.pR, P);
    take(x.pflag, P); take(x.phist, phist_n * P1); take(x.rqp, P1 * R2 * K); take(x.psel, P1 * (C + 1));
    take(x.pkeep, keep_cut ? P1 * C : 0); take(x.psz, P);
    take(x.psrc, P); take(x.page, P); take(x.rsrc, P); take(x.rsz, P1 * (P + 2));
    runs(x.pr, PM, C, P, P, nrbp);
    take(x.fin, PM * 8);
    return o;
  };
  CK(e->d_rg.reserve(carve(nullptr)));
  carve(e->d_rg);
  uint8_t* ocur = x.out;
  ImgCols out = carve_cols(ocur, N + P);  // seq: the kept parties' numbers at N + row
  out.id_bytes = idb;
  CK(cudaMemcpyAsync(x.lut, y.lut.data(), (size_t)y.KR * 2, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(x.grp, y.grp.data(), y.KR, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(x.bseg, y.bin_seg.data(), (size_t)y.Kp * 2, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(x.off, off.data(), off.size() * 4, cudaMemcpyHostToDevice, e->stream));
  if (keep_cut) CK(cudaMemcpyAsync(x.keep, keep.data(), S, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemsetAsync(x.skip, 0, 4 * (size_t)K, e->stream));
  CK(cudaMemsetAsync(x.pair, 0, pair_n * 4 * K, e->stream));
  CK(cudaMemsetAsync(x.ord, 0, pair_n * 2 * K, e->stream));
  CK(cudaMemsetAsync(x.src[1], 0, (size_t)N * 4, e->stream));  // a merge that writes holes (a refused image) stays in range
  CK(cudaMemsetAsync(&e->d_cnt->img_err, 0, 3 * 4, e->stream));  // img_err, mrg_dups, rg_kmax
  if (e->use_active) CK(cudaMemsetAsync(x.seen, 0xFF, sc * 8, e->stream));
  // 1. per image: classify, repeated ids, the stable scatter by new partition (reject bucket S last), the run plan
  const uint32_t grid = grid256(e, N, 32);
  uint64_t hoff = 0;
  for (uint32_t k = 0; k < K; ++k) {
    const uint32_t n = h[k].n_players, b = base[k];
    uint32_t* bhist = x.hist + hoff;
    hoff += (uint64_t)(S + 1) * nblk[k];
    uint32_t* pair = x.pair + pair_n * k;
    const bool take_act = k == act_img && m;
    if (n) {
      RgClassifyArgs ca{};
      ca.in = in[k]; ca.n = n; ca.nblk = nblk[k]; ca.part_off = x.off + (size_t)k * (SI + 1); ca.n_img_segs = SI;
      ca.bm_img = BinMap{x.lut, y.key_lo, y.KR, y.stride, y.K};
      ca.grp_img = x.grp; ca.bin_seg_img = x.bseg; ca.n_modes_img = h[k].config.n_modes; ca.seq_next = h[k].seq_next;
      ca.id_limit = id_limit(e);
      ca.bm = bin_map(e); ca.grp_lut = e->d_grp_lut; ca.bin_seg = e->d_bin_seg; ca.n_modes = e->cfg.n_modes; ca.n_segs = S;
      ca.keep = keep_cut ? x.keep : nullptr; ca.n_skip = x.skip + k;
      ca.part = x.part + b; ca.pimg = x.pimg + b; ca.blockhist = bhist; ca.pair = pair; ca.err = &e->d_cnt->img_err;
      k_rg_classify<<<nblk[k], 256, 0, e->stream>>>(ca);
    }
    if (e->use_active && (n || take_act))
      k_rg_dups<<<grid, 256, 0, e->stream>>>(in[k].id, act, idb, n, take_act ? m : 0, x.seen, sc - 1,
                                              &e->d_cnt->mrg_dups);
    if (n) {
      k_rq_scan<<<1, 512, 0, e->stream>>>(S + 1, nblk[k], bhist, x.rq + R1 * k, x.sel);
      k_rq_group<<<nblk[k], 256, 0, e->stream>>>(n, S + 1, nblk[k], x.part + b, in[k].seq, h[k].seq_next, bhist,
                                                  x.src[0] + b, x.age[0] + b);
      k_rg_plan<<<1, 1024, 0, e->stream>>>(SI, S, pair, x.rq + R1 * k, x.ord + pair_n * k,
                                           x.run + (size_t)S * (SI + 1) * k, x.kq + (size_t)S * k, &e->d_cnt->rg_kmax);
    } else {
      CK(cudaMemsetAsync(x.rq + R1 * k, 0, 4 * R1, e->stream));
    }
  }
  // 1'. per party image: sizes -> member offsets, classify (and the seq set), the repeated ids, the stable scatter by
  // queue (reject bucket C last); then every solo of the image probes the seq set
  std::vector<PtImgCols> pc(K);
  if (parties) {
    for (uint32_t k = 0; k < K; ++k) {
      if (pbase[k + 1] == pbase[k]) continue;
      const PtImgLayout& pl = ri.pl[k];
      const uint8_t* b = static_cast<const uint8_t*>(pp->bufs[k]);
      uint8_t* d = x.pbody + pboff[k];
      CK(cudaMemcpyAsync(d, b + pl.off[0], pl.off[6] - pl.off[0], cudaMemcpyHostToDevice, e->stream));
      PtImgCols& c = pc[k];
      c.size = d; c.seq = reinterpret_cast<uint32_t*>(d + (pl.off[1] - pl.off[0]));
      c.ts = reinterpret_cast<uint32_t*>(d + (pl.off[2] - pl.off[0])); c.mode = d + (pl.off[3] - pl.off[0]);
      c.id = d + (pl.off[4] - pl.off[0]);
      c.rating = reinterpret_cast<int32_t*>(d + (pl.off[5] - pl.off[0])); c.id_bytes = idb;
    }
    CK(cudaMemcpyAsync(x.pcols, pc.data(), sizeof(PtImgCols) * K, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(x.pbase, pbase.data(), 4 * ((size_t)K + 1), cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemsetAsync(x.pctr, 0, 4 * (kRpWords + 3 * (size_t)K), e->stream));
    CK(cudaMemsetAsync(x.seqset, 0xFF, psc * 8, e->stream));
    CK(cudaMemsetAsync(x.rsz, 0, 4 * P + 8, e->stream));
    if (keep_cut) CK(cudaMemcpyAsync(x.pkeep, keep_cut, C, cudaMemcpyHostToDevice, e->stream));
    uint64_t phoff = 0;
    for (uint32_t k = 0; k < K; ++k) {
      const uint32_t np = pbase[k + 1] - pbase[k], pb = pbase[k];
      uint32_t* bhist = x.phist + phoff;
      phoff += (uint64_t)(C + 1) * ri.pnblk[k];
      if (np) {
        k_rp_sizes<<<(np + 255) / 256, 256, 0, e->stream>>>(np, pc[k].size, x.pmoff + pb);
        k_scan_small<<<1, 1024, 0, e->stream>>>(np, x.pmoff + pb, x.pctr + kRpWords + 2 * K + k);
        RpClassifyArgs ca{};
        ca.in = pc[k]; ca.k = k; ca.n = np; ca.m = ri.mcount[k]; ca.nblk = ri.pnblk[k]; ca.seq_next = h[k].seq_next;
        ca.moff = x.pmoff + pb; ca.id_limit = id_limit(e); ca.bm = bin_map(e); ca.grp_lut = e->d_grp_lut;
        ca.mode_tsize = e->d_mode_tsize; ca.n_modes = e->cfg.n_modes; ca.n_groups = e->cfg.n_groups; ca.n_cut = C;
        ca.keep = keep_cut ? x.pkeep : nullptr;
        ca.seqset = x.seqset; ca.seq_mask = psc - 1; ca.part = x.ppart + pb; ca.pk = x.pk + pb; ca.R = x.pR + pb;
        ca.flag = x.pflag + pb; ca.size = x.psz + pb; ca.blockhist = bhist; ca.ctr = x.pctr;
        ca.skip = x.pctr + kRpWords + k; ca.kmem = x.pctr + kRpWords + K + k;
        k_rp_classify<<<ri.pnblk[k], 256, 0, e->stream>>>(ca);
        if (ri.mcount[k])
          k_rg_dups<<<grid256(e, ri.mcount[k], 32), 256, 0, e->stream>>>(pc[k].id, nullptr, idb, ri.mcount[k], 0,
                                                                         x.seen, sc - 1, &e->d_cnt->mrg_dups);
        k_rq_scan<<<1, 512, 0, e->stream>>>(C + 1, ri.pnblk[k], bhist, x.rqp + R2 * k, x.psel);
        k_rq_group<<<ri.pnblk[k], 256, 0, e->stream>>>(np, C + 1, ri.pnblk[k], x.ppart + pb, pc[k].seq,
                                                        h[k].seq_next, bhist, x.psrc + pb, x.page + pb);
      } else {
        CK(cudaMemsetAsync(x.rqp + R2 * k, 0, 4 * R2, e->stream));
      }
      if (np && h[k].n_players)
        k_rp_probe<<<grid256(e, h[k].n_players, 32), 256, 0, e->stream>>>(k, h[k].n_players, in[k].seq, h[k].seq_next,
                                                                           x.seqset, psc - 1, x.pctr + kRpSeqDup);
    }
  }
  // 2. per image: the merge rounds by age (enough for any k_max <= SI)
  for (uint32_t k = 0; k < K; ++k) {
    const uint32_t b = base[k];
    if (!h[k].n_players) continue;
    uint32_t* const src[2] = {x.src[0] + b, x.src[1] + b};
    uint32_t* const age[2] = {x.age[0] + b, x.age[1] + b};
    rg_rounds(e, RgMergeArgs{x.rq + R1 * k, S, SI, 0, x.pimg + b, x.ord + pair_n * k, x.run + (size_t)S * (SI + 1) * k,
                             x.kq + (size_t)S * k, &e->d_cnt->rg_kmax}, src, age, grid);
  }
  if (!many) {
    // 3. one image: duplicate ages, the gathered columns, the reject list (mm_import_regroup's tail)
    RgFinishArgs fa{};
    fa.rq_off = x.rq; fa.n_segs = S; fa.n = N; fa.kmax = &e->d_cnt->rg_kmax;
    fa.src[0] = x.src[0]; fa.src[1] = x.src[1]; fa.u[0] = x.age[0]; fa.u[1] = x.age[1];
    fa.in = in[0]; fa.out = out; fa.rejected = x.rej; fa.err = &e->d_cnt->img_err;
    k_rg_finish<<<grid, 256, 0, e->stream>>>(fa);
    if (parties) {  // the kept parties keep their order and numbers
      k_scan_small<<<1, 1024, 0, e->stream>>>((uint32_t)P, x.pflag, x.rsz + P);
      k_rp_rows1<<<(uint32_t)((P + 255) / 256), 256, 0, e->stream>>>((uint32_t)P, x.ppart, C, x.pflag, x.psz, pc[0].seq,
                                                                     x.rsrc, x.rsz, out.seq + N);
    }
  } else {
    // 3'. several images: their runs of every new partition merged by (running-max stamp, image, age), then numbered
    const RcRuns& r = x.sr;
    // ident: run q of the numbering rounds is partition q, run S + c party queue c; with parties, then the side of
    // the final merge round (0: the solos' list, 1: the parties')
    std::vector<uint16_t> id16(parties ? 2 * ((size_t)S + C) : S);
    for (uint32_t q = 0; q < S; ++q) id16[q] = (uint16_t)q;
    if (parties)
      for (uint32_t c = 0; c < C; ++c) { id16[S + c] = (uint16_t)c; id16[2 * S + C + c] = 1; }
    CK(cudaMemcpyAsync(x.ident, id16.data(), id16.size() * 2, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(x.imgs, in.data(), sizeof(ImgCols) * K, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(x.base, base.data(), 4 * (size_t)K, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemsetAsync(x.img, 0, 2 * (N + P), e->stream));
    CK(cudaMemsetAsync(x.qv, 0, 2 * (N + P), e->stream));
    std::vector<const uint32_t*> ts(K);
    for (uint32_t k = 0; k < K; ++k) ts[k] = in[k].ts;
    if ((rc = rc_merge(e, K, S, x.rq, base, x.src, x.age, ts, 0, 0, x.img, x.qv, r, N + P, nrb, grid))) return rc;
    RcFinishArgs fa{};
    fa.rq_glob = r.glob; fa.n_segs = S; fa.kmax = r.one + 3; fa.src[0] = r.s2[0]; fa.src[1] = r.s2[1];
    fa.key[0] = r.key[0]; fa.key[1] = r.key[1]; fa.imgs = x.imgs; fa.img = x.img; fa.base = x.base; fa.out = out;
    fa.pos = x.pos;
    k_rc_finish<<<grid, 256, 0, e->stream>>>(fa);
    // the partitions' lists are the runs of one list: run q = partition q
    const uint32_t bs = rg_rounds(e, RgMergeArgsT<RcKey>{r.one, 1, S, 0, x.qv, x.ident, r.glob, r.one + 2, r.one + 2},
                                  r.s2, r.key, grid);
    if (!parties) {
      k_rc_number<<<grid, 256, 0, e->stream>>>(r.one + 1, r.s2[bs], x.pos, out.seq);
    } else {
      // the parties' queue runs: merged by (running max, image, age) as the solos' partition runs are
      const RcRuns& q = x.pr;
      const uint32_t gp = grid256(e, P, 32);
      const uint32_t* const psrc[2] = {x.psrc, x.psrc};
      const uint32_t* const page[2] = {x.page, x.page};
      for (uint32_t k = 0; k < K; ++k) ts[k] = pc[k].ts;
      if ((rc = rc_merge(e, K, C, x.rqp, pbase, psrc, page, ts, N, S, x.img, x.qv, q, P, nrbp, gp))) return rc;
      k_rp_norm<<<gp, 256, 0, e->stream>>>(q.one + 1, q.one + 3, q.s2[0], q.s2[1], q.key[0], q.key[1]);
      // the queues' lists into the parties' one order: their rows
      const uint32_t ps = rg_rounds(e, RgMergeArgsT<RcKey>{q.one, 1, C, 0, x.qv, x.ident, q.glob, q.one + 2, q.one + 2},
                                    q.s2, q.key, gp);
      // after the solos' global list, then one round merges the two lists; k_rc_number numbers both
      RpPlaceArgs pa{};
      pa.kept_p = q.one + 1; pa.kept_s = r.one + 1; pa.psrc = q.s2[ps]; pa.pkey = q.key[ps]; pa.n_solo = N;
      pa.size = x.psz; pa.gsrc = r.s2[bs]; pa.gkey = r.key[bs]; pa.pos = x.pos; pa.rsrc = x.rsrc; pa.rsz = x.rsz;
      pa.fin = x.fin;
      k_rp_place<<<gp, 256, 0, e->stream>>>(pa);
      uint32_t* const src[2] = {r.s2[bs], r.s2[bs ^ 1]};
      RcKey* const key[2] = {r.key[bs], r.key[bs ^ 1]};
      const uint32_t g2 = grid256(e, N + P, 32);
      rg_rounds(e, RgMergeArgsT<RcKey>{x.fin, 1, 2, 0, x.qv, x.ident + S + C, x.fin + 2, x.fin + 5, x.fin + 5}, src,
                key, g2);
      k_rc_number<<<g2, 256, 0, e->stream>>>(x.fin + 1, src[1], x.pos, out.seq);
    }
  }
  CK(cudaGetLastError());
  // 4. one read decides every refusal
  std::vector<uint32_t> h_off(R1 * K), h_skip(K), h_poff(parties ? R2 * K : 0), h_pctr(parties ? kRpWords + 3 * K : 0);
  CK(cudaMemcpyAsync(h_off.data(), x.rq, h_off.size() * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemcpyAsync(h_skip.data(), x.skip, 4 * (size_t)K, cudaMemcpyDeviceToHost, e->stream));
  if (parties) {
    CK(cudaMemcpyAsync(h_poff.data(), x.rqp, h_poff.size() * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(h_pctr.data(), x.pctr, h_pctr.size() * 4, cudaMemcpyDeviceToHost, e->stream));
  }
  if ((rc = read_counters(e))) return rc;
  if (const uint32_t err = e->h_cnt->img_err) return img_err(e, "image rejected", err);
  uint32_t p_kept = 0, p_rej = 0, p_skip = 0, p_mem = 0;
  if (parties) {
    const uint32_t err = h_pctr[kRpErrBits];
    for (uint32_t k = 0; k < K; ++k)
      if (h_pctr[kRpWords + 2 * K + k] != ri.mcount[k]) return set_err(e, MM_E_ARG, "party image %u rejected: party sizes do not add up to the member count", k);
    if (err)
      return set_err(e, MM_E_ARG, "party image rejected:%s%s%s", err & kRpBadSize ? " a party of fewer than 2 members" : "",
                     err & kRpBadSeq ? " sequence numbers out of order" : "", err & kRpBadId ? " id out of range" : "");
    if (h_pctr[kRpSeqDup]) return set_err(e, MM_E_ARG, "party image rejected: a party's sequence number is a solo's");
  }
  if (e->h_cnt->mrg_dups) return img_err(e, "image rejected", kImgDup);
  if (parties)
    for (uint32_t k = 0; k < K; ++k) {
      const uint32_t* r = h_poff.data() + R2 * k;
      const uint32_t np = pbase[k + 1] - pbase[k];
      if (r[C + 1] + h_pctr[kRpWords + k] != np)
        return set_err(e, MM_E_STATE, "regroup: %u parties kept or rejected and %u skipped of %u", r[C + 1],
                       h_pctr[kRpWords + k], np);
      p_kept += r[C]; p_rej += r[C + 1] - r[C]; p_skip += h_pctr[kRpWords + k]; p_mem += h_pctr[kRpWords + K + k];
    }
  uint32_t kept = 0, n_rej = 0, n_skip = 0;
  for (uint32_t k = 0; k < K; ++k) {
    const uint32_t* r = h_off.data() + R1 * k;
    if (r[S + 1] + h_skip[k] != h[k].n_players)  // every player that passed the checks is kept, skipped or rejected
      return set_err(e, MM_E_STATE, "regroup: %u kept or rejected and %u skipped of %u players", r[S + 1], h_skip[k],
                     h[k].n_players);
    kept += r[S]; n_rej += r[S + 1] - r[S]; n_skip += h_skip[k];
  }
  if (n_rej > cap) {
    *n_rejected = n_rej;
    return set_err(e, MM_E_CAP, "%u rejected players, cap %u", n_rej, cap);
  }
  if (parties && p_rej > pp->cap) {
    pp->n_rejected = p_rej;
    return set_err(e, MM_E_CAP, "%u rejected parties, cap %u", p_rej, pp->cap);
  }
  if (p_mem > e->pt.cap)
    return set_err(e, MM_E_CAP, "%u party members to load, party_capacity %u", p_mem, e->pt.cap);
  if ((rc = load_fits(e, kept, (uint64_t)m + p_mem))) return rc;
  if (n_rej && many && (rc = rg_rejects(e, K, S, h_off, x.src[0], base, rej_index, rej_image))) return rc;
  if (n_rej && !many) {  // one image: k_rg_finish's list
    CK(cudaMemcpyAsync(rej_index, x.rej, (size_t)n_rej * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    if (rej_image) std::fill_n(rej_image, n_rej, 0u);
  }
  if (p_rej && (rc = rg_rejects(e, K, C, h_poff, x.psrc, pbase, pp->rej_index, pp->rej_image))) return rc;
  std::vector<uint32_t> per(S, 0);
  for (uint32_t k = 0; k < K; ++k)
    for (uint32_t s = 0; s < S; ++s) per[s] += h_off[R1 * k + s + 1] - h_off[R1 * k + s];
  if ((rc = load_columns(e, per, out, kept, act, m, many ? kept + p_kept : seq_next, "image rejected"))) return rc;
  *n_rejected = n_rej;
  if (n_elsewhere) *n_elsewhere = n_skip;
  if (!parties) return MM_OK;
  pp->n_rejected = p_rej;
  pp->n_elsewhere = p_skip;
  if (p_kept) {  // the table rows in the new age order, members and active-set values
    auto& t = e->pt;
    k_scan_small<<<1, 1024, 0, e->stream>>>(p_kept, x.rsz, x.rsz + P + 1);
    RpWriteArgs wa{};
    wa.imgs = x.pcols; wa.pbase = x.pbase;
    wa.pk = x.pk; wa.moff = x.pmoff; wa.R = x.pR; wa.rsrc = x.rsrc; wa.rseq = out.seq + N; wa.roff = x.rsz;
    wa.rows = p_kept; wa.bm = bin_map(e); wa.grp_lut = e->d_grp_lut; wa.pt = pt_view(e, t.cur); wa.act = act_view(e);
    k_rp_write<<<(p_kept + 255) / 256, 256, 0, e->stream>>>(wa);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(e->stream));
    t.n_rows = p_kept; t.n_mem = p_mem; t.live = p_mem;
    e->n_active += p_mem;
  }
  pp->n_loaded = p_kept;
  return MM_OK;
}

// ---- boundary pass: mm_band_candidates / mm_band_match (mm_band.cuh) ----------------------------------------------
// The refusals both calls share (shard.check_bands' rules, then the engine's state).
int band_check(mm_engine* e, int32_t W) {
  const mm_config& c = e->cfg;
  if (W < 0) return set_err(e, MM_E_ARG, "W must be >= 0");
  if (c.order_mode != MM_ORDER_RATING) return set_err(e, MM_E_ARG, "the boundary pass needs MM_ORDER_RATING");
  for (uint32_t g = 0; g < c.n_groups; ++g) {
    if ((int64_t)c.group_hi[g] - c.group_lo[g] + 1 < 2 * (int64_t)W)
      return set_err(e, MM_E_ARG, "rating group %u is narrower than 2 x W: boundary bands would overlap", g);
    if (g && (int64_t)c.group_lo[g] != (int64_t)c.group_hi[g - 1] + 1)
      return set_err(e, MM_E_ARG, "the boundary pass needs contiguous ascending rating groups");
  }
  if (e->stage_count) return staged_err(e);
  if (!e->use_active) return set_err(e, MM_E_STATE, "an MM_F_NO_DEDUPE engine cannot take matched players");
  return MM_OK;
}

uint32_t band_ctas(const mm_engine* e, uint32_t n) {
  return std::max<uint32_t>(1, std::min<uint32_t>((tile_count(e, n) + kBandWarps - 1) / kBandWarps, 4u * (uint32_t)e->n_sms));
}

// The pool and table fields of the gather's arguments (every caller's)
BandArgs band_args(mm_engine* e) {
  const Pool& p = e->pool[e->cur];
  BandArgs a{};
  a.pool = p.v; a.meta = p.m; a.fill = p.m.fill;
  a.n_segs = e->n_segs; a.K = e->K; a.bm = bin_map(e); a.bin_seg = e->d_bin_seg; a.seg_bin_lo = e->d_seg_bin_lo;
  return a;
}

// The gather every caller shares, once a.n_keys is set: scratch of the per-key arrays and of `cols` per-(key, tile)
// counts, then the bin -> key map and count columns (k_band_prep with the caller's numbering kb), the per-(key, tile)
// counts, per-key prefixes and totals.
template <class KeyBins>
int band_gather(mm_engine* e, BandArgs& a, size_t cols, const KeyBins& kb) {
  auto& s = e->band;
  const size_t nk = std::max<size_t>(a.n_keys, 1);
  cols = std::max<size_t>(cols, 1);
  CK(s.map.reserve(e->Kp)); CK(s.fill.reserve(e->n_segs)); CK(s.qoff.reserve(nk + 1)); CK(s.qtiles.reserve(nk));
  CK(s.qseg.reserve(nk)); CK(s.M.reserve(cols)); CK(s.tot.reserve(nk)); CK(s.ctr.reserve(kBcWords));
  a.meta.fill = s.fill; a.map = s.map; a.bfill = s.fill; a.qoff = s.qoff; a.qtiles = s.qtiles; a.qseg = s.qseg;
  a.M = s.M; a.tot = s.tot; a.ctr = s.ctr;
  CK(cudaMemsetAsync(s.ctr, 0, kBcWords * 4, e->stream));
  CK(cudaMemsetAsync(s.tot, 0, nk * 4, e->stream));
  if (!a.n_keys) return MM_OK;
  CK(cudaMemsetAsync(s.map, 0xFF, (size_t)e->Kp * 4, e->stream));
  CK(cudaMemsetAsync(s.M, 0, cols * 4, e->stream));
  k_band_prep<<<1, kBandPrepBlock, 0, e->stream>>>(a, kb);
  k_band_count<kBandBlock><<<band_ctas(e, e->pool[e->cur].n), kBandBlock, 0, e->stream>>>(a);
  k_band_scan<<<(a.n_keys + 7) / 8, 256, 0, e->stream>>>(a);
  CK(cudaGetLastError());
  return MM_OK;
}

// Arguments and scratch of one call: n_bounds boundaries from g_first | g_first+1, every mode.  Every scratch array is
// sized by the band keys, the candidates or the per-key tile counts; none by the pool's capacity.
int band_setup(mm_engine* e, int32_t W, uint32_t g_first, uint32_t n_bounds, bool skip_lower, bool remote_last,
               BandArgs& a) {
  const mm_config& c = e->cfg;
  auto& s = e->band;
  a = band_args(e);
  a.W = W; a.n_modes = c.n_modes; a.g_first = g_first; a.n_bands = n_bounds * c.n_modes;
  a.n_keys = a.n_bands * 2u * (uint32_t)W;
  a.skip_lower = skip_lower; a.remote_last = remote_last;
  for (uint32_t g = 0; g < c.n_groups; ++g) a.hi[g] = c.group_hi[g];
  for (uint32_t m = 0; m < c.n_modes; ++m) a.L[m] = (uint32_t)c.modes[m].teams * c.modes[m].team_size;
  const size_t nk = std::max<size_t>(a.n_keys, 1);
  CK(s.kbase.reserve(nk)); CK(s.klim.reserve(nk));
  CK(s.rstart.reserve(nk)); CK(s.pos.reserve((size_t)a.n_bands * (2u * (uint32_t)W + 1)));
  CK(s.band_mb.reserve(a.n_bands + 1)); CK(s.band_lb.reserve(a.n_bands + 1));
  a.pos = s.pos; a.kbase = s.kbase; a.klim = s.klim; a.band_mb = s.band_mb; a.band_lb = s.band_lb;
  const size_t cols = (size_t)tile_count(e, e->pool[e->cur].n) * std::min<uint32_t>(e->max_nb, 2u * (uint32_t)W);
  return band_gather(e, a, cols, BandKeyBins{});
}

int band_read_ctr(mm_engine* e, uint32_t (&h)[kBcWords]) {
  CK(cudaMemcpyAsync(h, e->band.ctr, sizeof(h), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return MM_OK;
}

int band_candidates(mm_engine* e, int32_t W, uint32_t group, uint64_t* ids, int32_t* rating, uint8_t* mode,
                    uint32_t cap, uint32_t* n_out) {
  int rc = band_check(e, W);
  if (rc) return rc;
  if (group == 0 || group >= e->cfg.n_groups)
    return set_err(e, MM_E_ARG, "group %u has no low boundary: need 1 <= group < n_groups = %u", group, e->cfg.n_groups);
  if (W == 0) return MM_OK;
  BandArgs a;
  if ((rc = band_setup(e, W, group - 1, 1, true, false, a))) return rc;
  k_band_bases<<<1, kBandWalkBlock, 0, e->stream>>>(a, 0);
  CK(cudaGetLastError());
  uint32_t h[kBcWords];
  if ((rc = band_read_ctr(e, h))) return rc;
  const uint32_t n = h[kBcKeys];
  *n_out = n;
  if (n > cap) return set_err(e, MM_E_CAP, "need cap >= %u", n);
  if (n == 0) return MM_OK;
  auto& s = e->band;
  CK(s.id.reserve(n)); CK(s.rating.reserve(n)); CK(s.mode.reserve(n));
  k_band_limit<<<1, kBandPrepBlock, 0, e->stream>>>(a);
  k_band_place<kBandBlock><<<band_ctas(e, e->pool[e->cur].n), kBandBlock, 0, e->stream>>>(
      a, BandOut{s.id, s.rating, s.mode, 0u});
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(ids, s.id, (size_t)n * 8, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemcpyAsync(rating, s.rating, (size_t)n * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemcpyAsync(mode, s.mode, n, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return MM_OK;
}

int band_match(mm_engine* e, int32_t W, uint32_t g_first, uint32_t g_last, uint32_t upper_remote, const uint64_t* up_ids,
               const int32_t* up_rating, const uint8_t* up_mode, uint32_t n_upper, mm_lobby_hdr* lobbies,
               uint32_t lobby_cap, uint64_t* member_ids, uint64_t member_cap, uint8_t* upper_taken, mm_band_stats* st) {
  int rc = band_check(e, W);
  if (rc) return rc;
  const uint32_t G = e->cfg.n_groups;
  if (g_first > g_last || g_last + 1 >= G)
    return set_err(e, MM_E_ARG, "boundaries %u..%u: need g_first <= g_last < n_groups - 1 = %u", g_first, g_last, G - 1);
  if (!upper_remote && n_upper) return set_err(e, MM_E_ARG, "upper candidates given without upper_remote");
  if (upper_remote && e->dense_ids)
    return set_err(e, MM_E_ARG, "upper candidates on an MM_F_DENSE_IDS engine: another engine's handles are not ids here");
  auto& s = e->band;
  CK(cudaEventRecord(e->ev[0], e->stream));
  BandArgs a;
  if ((rc = band_setup(e, W, g_first, g_last - g_first + 1, false, upper_remote != 0, a))) return rc;
  if (n_upper) {  // the caller's columns: checked, counted into their keys
    CK(s.up_id.reserve(n_upper)); CK(s.up_rating.reserve(n_upper)); CK(s.up_mode.reserve(n_upper));
    CK(s.up_taken.reserve(n_upper));
    CK(cudaMemcpyAsync(s.up_id, up_ids, (size_t)n_upper * 8, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(s.up_rating, up_rating, (size_t)n_upper * 4, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(s.up_mode, up_mode, n_upper, cudaMemcpyHostToDevice, e->stream));
    k_band_upper<<<(n_upper + 255) / 256, 256, 0, e->stream>>>(a, n_upper, s.up_rating, s.up_mode, s.rstart);
  }
  if (a.n_keys) k_band_bases<<<1, kBandWalkBlock, 0, e->stream>>>(a, 1);
  CK(cudaGetLastError());
  uint32_t h[kBcWords];
  if ((rc = band_read_ctr(e, h))) return rc;
  if (h[kBcErr] & kBandErrMode) return set_err(e, MM_E_ARG, "an upper candidate's mode is >= n_modes");
  if (h[kBcErr] & kBandErrRating)
    return set_err(e, MM_E_ARG, "an upper candidate's rating is outside (%d, %lld]", e->cfg.group_hi[g_last],
                   (long long)e->cfg.group_hi[g_last] + W);
  if (h[kBcErr] & kBandErrOrder) return set_err(e, MM_E_ARG, "the upper candidates are not sorted by (mode, rating)");
  const uint32_t nl = h[kBcLobbies], nm = h[kBcMatched], nu = h[kBcUpper];
  st->n_lobbies = nl; st->n_matched = nm; st->n_upper_taken = nu; st->n_taken = nm - nu;
  if (lobby_cap < nl || member_cap < nm)
    return set_err(e, MM_E_CAP, "need lobby_cap >= %u and member_cap >= %u", nl, nm);
  // from here on the call changes the pool: the local members are taken as they are placed
  const uint32_t ctas = band_ctas(e, e->pool[e->cur].n);
  if (nm) {
    CK(s.id.reserve(nm));
    if (nm > nu) {
      k_band_limit<<<1, kBandPrepBlock, 0, e->stream>>>(a);
      k_band_place<kBandBlock><<<ctas, kBandBlock, 0, e->stream>>>(a, BandOut{s.id, nullptr, nullptr, 1u});
    }
  }
  if (n_upper)
    k_band_upper_place<<<(n_upper + 255) / 256, 256, 0, e->stream>>>(a, n_upper, s.up_id, s.up_rating, s.up_mode,
                                                                     s.rstart, s.id, s.up_taken);
  if (nl) {
    CK(s.hdr.reserve(nl));
    k_band_hdr<<<(nl + 255) / 256, 256, 0, e->stream>>>(a, nl, s.hdr);
  }
  CK(cudaGetLastError());
  CK(cudaEventRecord(e->ev[4], e->stream));
  if (nl) CK(cudaMemcpyAsync(lobbies, s.hdr, (size_t)nl * sizeof(mm_lobby_hdr), cudaMemcpyDeviceToHost, e->stream));
  if (nm) CK(cudaMemcpyAsync(member_ids, s.id, (size_t)nm * 8, cudaMemcpyDeviceToHost, e->stream));
  if (n_upper) CK(cudaMemcpyAsync(upper_taken, s.up_taken, n_upper, cudaMemcpyDeviceToHost, e->stream));
  if ((rc = band_read_ctr(e, h))) return rc;
  st->n_taken = h[kBcTaken];
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, e->ev[0], e->ev[4]));
  st->device_us = ms * 1000.f;
  return MM_OK;
}

// ---- mm_backfill (mm_backfill.cuh) ---------------------------------------------------------------------------------
// The prefixes k_bf_keys made keys (counters h) leave the pool: the band gather over the keys' partitions places them
// into bf.staging at kbase[key] + rank and takes them.  bf.members is sized for them too.
int bf_take(mm_engine* e, const uint32_t* h, bool stamps = false) {
  auto& s = e->bf;
  const uint32_t total = h[kBfPlayers];
  BandArgs a = band_args(e);
  a.n_keys = h[kBfKeys];
  a.kbase = s.kbase; a.klim = s.klim;
  int rc = band_gather(e, a, h[kBfCols], BfKeyBins{s.key_bin});
  if (rc) return rc;
  CK(s.staging.reserve(total)); CK(s.members.reserve(total));
  if (stamps) CK(s.staging_ts.reserve(total));
  k_band_limit<<<1, kBandPrepBlock, 0, e->stream>>>(a);
  k_band_place<kBandBlock><<<band_ctas(e, e->pool[e->cur].n), kBandBlock, 0, e->stream>>>(
      a, BandOut{s.staging, nullptr, nullptr, 1u, stamps ? s.staging_ts.p : nullptr});
  CK(cudaGetLastError());
  return MM_OK;
}

// The requests grouped by queue, stably (a counting sort), with the targets as clamp keys: in = the BfReqs in queue
// order | the first request of every queue [n_cut + 1] | the queues with requests.  -> the number of those queues.
uint32_t bf_sort(const mm_engine* e, uint32_t n, const mm_backfill_req* req, std::vector<uint32_t>& in) {
  const uint32_t G = e->cfg.n_groups, nc = e->n_cut;
  std::vector<uint32_t> qr(nc + 1, 0);
  for (uint32_t j = 0; j < n; ++j) ++qr[req[j].mode * G + req[j].group + 1];
  for (uint32_t q = 0; q < nc; ++q) qr[q + 1] += qr[q];
  const size_t rw = sizeof(BfReq) / 4;
  in.assign(rw * n + nc + 1, 0);
  std::copy(qr.begin(), qr.end(), in.begin() + rw * n);
  std::vector<uint32_t> at(qr.begin(), qr.end() - 1);
  for (uint32_t j = 0; j < n; ++j) {
    const mm_backfill_req& r = req[j];
    const int64_t t = std::min<int64_t>(std::max<int64_t>((int64_t)r.target - e->key_lo, 0), (int64_t)e->KR - 1);
    const BfReq b{j, r.count, (int32_t)t, r.window};
    std::memcpy(&in[rw * at[r.mode * G + r.group]++], &b, sizeof(b));
  }
  for (uint32_t q = 0; q < nc; ++q)
    if (qr[q + 1] > qr[q]) in.push_back(q);
  return (uint32_t)(in.size() - (rw * n + nc + 1));
}

// The refusals of request j that mm_backfill and mm_backfill_party share.
int bf_check_req(mm_engine* e, uint32_t j, const mm_backfill_req& r) {
  const mm_config& c = e->cfg;
  if (r.mode >= c.n_modes) return set_err(e, MM_E_ARG, "request %u: mode %u >= n_modes = %u", j, r.mode, c.n_modes);
  if (r.group >= c.n_groups)
    return set_err(e, MM_E_ARG, "request %u: group %u >= n_groups = %u", j, r.group, c.n_groups);
  if (r.reserved) return set_err(e, MM_E_ARG, "request %u: reserved must be 0", j);
  return MM_OK;
}

// The plan's scratch in e->bf for up to n_pieces pieces, with rem = the pool's per-bin totals.
int bf_plan_scratch(mm_engine* e, size_t n_pieces) {
  auto& b = e->bf;
  const size_t K = e->K;
  CK(b.rem.reserve(K)); CK(b.key_bin.reserve(K)); CK(b.kbase.reserve(K)); CK(b.klim.reserve(K));
  CK(b.piece.reserve(n_pieces));
  CK(cudaMemcpyAsync(b.rem, e->pool[e->cur].m.tot, K * 4, cudaMemcpyDeviceToDevice, e->stream));
  return MM_OK;
}

// k_bf_keys on e->bf's plan scratch: the bins with a take become keys, counted in ctr.
void bf_keys(mm_engine* e, uint32_t* ctr) {
  const Pool& p = e->pool[e->cur];
  auto& b = e->bf;
  BfArgs f{};
  f.tot = p.m.tot; f.rem = b.rem; f.bin_seg = e->d_bin_seg; f.fill = p.m.fill; f.K = e->K;
  f.key_bin = b.key_bin; f.kbase = b.kbase; f.klim = b.klim; f.ctr = ctr;
  k_bf_keys<<<1, kBfKeysBlock, 0, e->stream>>>(f);
}

// k_bf_out over np pieces of e->bf's plan: staging (the take's members or stamps) to out at req_base[piece.req] + offset.
template <class T>
void bf_out(mm_engine* e, uint32_t np, const uint32_t* req_base, const T* staging, T* out) {
  auto& b = e->bf;
  k_bf_out<<<(uint32_t)(((size_t)np * 32 + 255) / 256), 256, 0, e->stream>>>(np, b.piece, e->band.map, b.kbase, req_base,
                                                                             staging, out);
}

int backfill(mm_engine* e, uint32_t n, const mm_backfill_req* req, uint32_t* n_taken, uint64_t* member_ids,
             uint64_t member_cap, uint32_t* n_total) {
  const bool rating = e->cfg.order_mode == MM_ORDER_RATING;
  int rc;
  for (uint32_t j = 0; j < n; ++j) {
    if ((rc = bf_check_req(e, j, req[j]))) return rc;
    if (!rating && req[j].window >= 0)
      return set_err(e, MM_E_ARG, "request %u: a window on an MM_ORDER_ARRIVAL engine (pass window < 0)", j);
  }
  if (e->stage_count) return staged_err(e);
  if (!e->use_active) return set_err(e, MM_E_STATE, "an MM_F_NO_DEDUPE engine cannot hold taken players");
  if (n == 0) return MM_OK;
  const uint32_t nc = e->n_cut;
  const size_t rw = sizeof(BfReq) / 4;
  std::vector<uint32_t> in;
  const uint32_t nq = bf_sort(e, n, req, in);
  auto& s = e->bf;
  const Pool& p = e->pool[e->cur];
  CK(s.in.reserve(in.size())); CK(s.n_taken.reserve(n)); CK(s.req_base.reserve(n)); CK(s.ctr.reserve(kBfWords));
  // every bin a request reaches but the last is emptied: at most n + K pieces
  if ((rc = bf_plan_scratch(e, (size_t)n + e->K))) return rc;
  CK(cudaMemcpyAsync(s.in, in.data(), in.size() * 4, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemsetAsync(s.ctr, 0, kBfWords * 4, e->stream));
  BfArgs f{};
  f.tot = p.m.tot; f.rem = s.rem; f.bin_key = e->d_bin_key; f.seg_bin_lo = e->d_seg_bin_lo; f.cut_lp_lo = e->d_cut_lp_lo;
  f.bin_seg = e->d_bin_seg; f.fill = p.m.fill; f.rating_order = rating; f.K = e->K;
  f.req = reinterpret_cast<const BfReq*>(s.in.p); f.qr = s.in + rw * n; f.queues = s.in + rw * n + nc + 1; f.nq = nq;
  f.n_taken = s.n_taken; f.piece = s.piece; f.key_bin = s.key_bin; f.kbase = s.kbase; f.klim = s.klim; f.ctr = s.ctr;
  // plan: what every request takes, on the per-bin totals; then the bins with a take as keys
  k_bf_plan<<<(nq + kBfPlanWarps - 1) / kBfPlanWarps, kBfPlanWarps * 32, 0, e->stream>>>(f);
  k_bf_keys<<<1, kBfKeysBlock, 0, e->stream>>>(f);
  CK(cudaGetLastError());
  uint32_t h[kBfWords];
  CK(cudaMemcpyAsync(n_taken, s.n_taken, (size_t)n * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemcpyAsync(h, s.ctr, sizeof(h), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  const uint32_t total = h[kBfPlayers];
  *n_total = total;
  if (member_cap < total) return set_err(e, MM_E_CAP, "need member_cap >= %u", total);
  if (total == 0) return MM_OK;
  // from here on the call changes the pool
  if ((rc = bf_take(e, h))) return rc;
  std::vector<uint32_t> base(n);
  for (uint32_t j = 0, acc = 0; j < n; ++j) { base[j] = acc; acc += n_taken[j]; }
  CK(cudaMemcpyAsync(s.req_base, base.data(), (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
  bf_out(e, h[kBfPieces], s.req_base, s.staging.p, s.members.p);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(member_ids, s.members, (size_t)total * 8, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return MM_OK;
}

// ---- the off-tick report (mm_offtick.cuh) --------------------------------------------------------------------------
// Report `src` of a party / widen call with nl > 0 lobbies and nm members, from its headers and bases (w), the member
// slots' c - key_lo (tb.cval) and stamps (ot.ts), and the imbalances its balance pass (bal_mask) stored in ot.imb.
int ot_capture(mm_engine* e, uint32_t src, const WdArgs& w, uint32_t nl, uint32_t nm, uint32_t bal_mask) {
  auto& o = e->ot;
  auto& r = o.rep[src];
  const uint32_t nc = e->n_cut;
  CK(r.lob.reserve(nl)); CK(r.quality.reserve(nc)); CK(r.waits.reserve(nc)); CK(o.qb.reserve(2 * ((size_t)nc + 1)));
  CK(cudaMemsetAsync(r.quality, 0, nc * sizeof(mm_queue_quality), e->stream));
  CK(cudaMemsetAsync(r.waits, 0, nc * sizeof(mm_match_waits), e->stream));
  OtArgs a{};
  a.hdr = w.hdr; a.n_lob = nl; a.n_mem = nm; a.n_cut = nc; a.n_groups = e->cfg.n_groups; a.now = w.now;
  a.key_lo = e->key_lo; a.mode_tsize = e->d_mode_tsize; a.cval = e->tb.cval; a.ts = o.ts; a.bal_mask = bal_mask;
  a.bal_imb = o.imb; a.qlbase = w.qlbase; a.qmbase = w.qmbase; a.qb = o.qb; a.qm = o.qb + nc + 1; a.lob = r.lob;
  a.waits = r.waits;
  k_ot_bases<<<1, kOtBlock, 0, e->stream>>>(a);
  k_ot_lobby<<<grid256(e, (uint64_t)nl * 32, 8), kOtBlock, 0, e->stream>>>(a);
  MqArgs q{};  // k_mq_queue reads only the lobby records, their queue bases and the records it adds into
  q.n_cut = nc; q.qlob = a.qb; q.lob = r.lob; q.n_lob = nl; q.qrec = r.quality;
  const uint32_t qctas = std::max<uint32_t>(1, std::min<uint32_t>(nl / 1024 + 1, 8u * (uint32_t)e->n_sms));
  k_mq_queue<kMqBlock><<<qctas, kMqBlock, 0, e->stream>>>(q);
  const uint32_t wctas = std::max<uint32_t>(1, std::min<uint32_t>(nm / 4096 + 1, 8u * (uint32_t)e->n_sms));
  k_ot_waits<kOtBlock><<<wctas, kOtBlock, 0, e->stream>>>(a);
  CK(cudaGetLastError());
  r.n_lob = nl;
  return MM_OK;
}

// ---- the off-tick budget (mm_set_offtick_budget; k_wd_allot in mm_widen.cuh) ---------------------------------------
// Before the plan of source `src`: its lobby counts go to the source's own words, where mm_offtick_budget_report finds
// them.
int ob_begin(mm_engine* e, uint32_t src, WdArgs& a) {
  auto& o = e->ob[src];
  CK(o.tab.reserve(4 * (size_t)e->n_cut + e->cfg.n_modes + 1));
  a.qlob = o.tab;
  a.cap = nullptr;
  o.ran = true;
  o.budgeted = !o.queue.empty() || !o.mode.empty();
  return MM_OK;
}

// After the unbudgeted plan of a budgeted call: the allowances; when one is short of its queue's lobbies, a.cap points
// at them and the caller runs the plan again from its reset state.  Synchronizes the stream (the caller's copies of
// the first plan's counters land with it).
int ob_allot(mm_engine* e, uint32_t src, WdArgs& a) {
  auto& o = e->ob[src];
  const uint32_t nc = e->n_cut;
  uint32_t *cand = o.tab + nc, *allot = cand + nc, *bud = allot + nc, *cut = bud + nc + e->cfg.n_modes;
  if (!o.queue.empty()) CK(cudaMemcpyAsync(bud, o.queue.data(), nc * 4, cudaMemcpyHostToDevice, e->stream));
  if (!o.mode.empty()) CK(cudaMemcpyAsync(bud + nc, o.mode.data(), o.mode.size() * 4, cudaMemcpyHostToDevice, e->stream));
  k_wd_allot<<<1, kScanBlock, 0, e->stream>>>(a, o.queue.empty() ? nullptr : bud, o.mode.empty() ? nullptr : bud + nc,
                                              cand, allot, cut);
  CK(cudaGetLastError());
  uint32_t h = 0;
  CK(cudaMemcpyAsync(&h, cut, 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  a.cap = h ? allot : nullptr;
  return MM_OK;
}

// ---- mm_widen (mm_widen.cuh) ---------------------------------------------------------------------------------------
// The rules of mm_widen / mm_party_match as the device reads them, and the refusals both share.  any: a queue is served.
int wd_rules(mm_engine* e, const mm_widen_rule* rules, std::vector<WdRule>& rule, bool& any) {
  const mm_config& c = e->cfg;
  const uint32_t G = c.n_groups, nc = e->n_cut;
  rule.resize(nc);
  any = false;
  for (uint32_t q = 0; q < nc; ++q) {
    const mm_widen_rule& r = rules[q];
    const mm_mode_desc& md = c.modes[q / G];
    rule[q] = WdRule{r.min_wait, r.step, r.w0, r.inc, r.w_max, (uint32_t)md.teams * md.team_size};
    if (r.min_wait == MM_WIDEN_OFF) continue;
    if (r.step == 0 || r.w0 < 0 || r.inc < 0 || r.w_max < r.w0 || r.reserved)
      return set_err(e, MM_E_ARG, "rule %u (mode %u, group %u): need step > 0, w0 >= 0, inc >= 0, w_max >= w0 and "
                     "reserved = 0", q, q / G, q % G);
    any = true;
  }
  if (c.order_mode != MM_ORDER_RATING) return set_err(e, MM_E_ARG, "widening windows need MM_ORDER_RATING");
  if (!e->use_active) return set_err(e, MM_E_STATE, "an MM_F_NO_DEDUPE engine cannot hold taken players");
  if (e->stage_count) return staged_err(e);
  return MM_OK;
}

// What mm_widen and mm_party_match set up alike: wd.tab = the rules | qlbase [n_cut] | qmbase [n_cut] | `extra` words
// for the caller | the counters [kWdWords], zeroed, and the WdArgs fields that come from the engine and the pool.
int wd_setup(mm_engine* e, uint64_t now, const std::vector<WdRule>& rule, size_t extra, WdArgs& a) {
  const Pool& p = e->pool[e->cur];
  const uint32_t nc = e->n_cut;
  const size_t o_qlb = sizeof(WdRule) / 4 * nc, o_qmb = o_qlb + nc, o_ctr = o_qmb + nc + extra;
  auto& s = e->wd;
  CK(s.tab.reserve(o_ctr + kWdWords));
  uint32_t* t = s.tab;
  CK(cudaMemcpyAsync(t, rule.data(), nc * sizeof(WdRule), cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemsetAsync(t + o_ctr, 0, kWdWords * 4, e->stream));
  a = WdArgs{};
  a.pool = p.v; a.meta = p.m; a.n_segs = e->n_segs; a.n_cut = nc; a.n_groups = e->cfg.n_groups; a.now = (uint32_t)now;
  a.seq_next = e->seq_next; a.rule = reinterpret_cast<const WdRule*>(t); a.part_cut = e->d_part_cut;
  a.cut_lp_lo = e->d_cut_lp_lo; a.seg_bin_lo = e->d_seg_bin_lo; a.bin_seg = e->d_bin_seg; a.bin_key = e->d_bin_key;
  a.tot = p.m.tot; a.qlbase = t + o_qlb; a.qmbase = t + o_qmb; a.ctr = t + o_ctr;
  return MM_OK;
}

// The tail of mm_widen and mm_party_match once the balance pass ran: the report of source src, the end event, the
// lobbies and members (and party_balance's sum when imb_sum is given) to the host, and the call's device time.
int wd_finish(mm_engine* e, uint32_t src, const WdArgs& a, uint32_t nl, uint32_t nm, uint32_t bal_mask,
              mm_lobby_hdr* lobbies, uint64_t* member_ids, uint64_t* imb_sum, float* device_us) {
  if (int rc = ot_capture(e, src, a, nl, nm, bal_mask)) return rc;
  CK(cudaEventRecord(e->ev[4], e->stream));
  CK(cudaMemcpyAsync(lobbies, a.hdr, (size_t)nl * sizeof(mm_lobby_hdr), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemcpyAsync(member_ids, e->bf.members, (size_t)nm * 8, cudaMemcpyDeviceToHost, e->stream));
  if (imb_sum) CK(cudaMemcpyAsync(imb_sum, e->tb.sum, 8, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, e->ev[0], e->ev[4]));
  *device_us = ms * 1000.f;
  return MM_OK;
}

int widen(mm_engine* e, uint64_t now, const mm_widen_rule* rules, mm_lobby_hdr* lobbies, uint32_t lobby_cap,
          uint64_t* member_ids, uint64_t member_cap, mm_widen_stats* st) {
  const uint32_t nc = e->n_cut;
  std::vector<WdRule> rule;
  bool any = false;
  int rc = wd_rules(e, rules, rule, any);
  if (rc) return rc;
  const Pool& p = e->pool[e->cur];
  if (!any || p.n == 0) return MM_OK;
  auto& s = e->wd;
  auto& b = e->bf;
  CK(cudaEventRecord(e->ev[0], e->stream));
  const uint32_t ctas = tile_ctas(e, p.n);
  WdArgs a;
  if ((rc = wd_setup(e, now, rule, (size_t)2 * e->n_segs + 1 + ctas + e->n_chunks, a))) return rc;
  a.part = a.qmbase + nc; a.cur = a.part + e->n_segs + 1; a.cta = a.cur + e->n_segs; a.rmap = a.cta + ctas;
  CK(cudaMemsetAsync(a.part, 0, (size_t)(e->n_segs + 1) * 4, e->stream));
  CK(cudaMemsetAsync(a.cta, 0, (size_t)ctas * 4, e->stream));
  // anchors: counted, then written in (partition, age) order
  k_wd_anchors<kWdBlock><<<ctas, kWdBlock, 0, e->stream>>>(a, 0);
  k_wd_part_scan<<<1, 1024, 0, e->stream>>>(a);
  CK(cudaGetLastError());
  uint32_t na = 0;
  CK(cudaMemcpyAsync(&na, a.part + e->n_segs, 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  st->n_anchors = na;
  if (na == 0) return MM_OK;
  CK(s.anc.reserve((size_t)na * 6));
  a.n_anchors = na; a.rec = reinterpret_cast<uint2*>(s.anc.p);  // first: 8-byte aligned
  a.a_slot = s.anc + 2 * (size_t)na; a.a_age = s.anc + 3 * (size_t)na; a.a_rank = s.anc + 4 * (size_t)na;
  a.mbase = s.anc + 5 * (size_t)na;
  // every bin a lobby reaches but its last is emptied: at most lobbies + K pieces
  if ((rc = bf_plan_scratch(e, (size_t)na + e->K))) return rc;
  a.rem = b.rem; a.piece = b.piece;
  k_wd_anchors<kWdBlock><<<ctas, kWdBlock, 0, e->stream>>>(a, 1);
  k_loc_rmap<<<e->n_segs, 256, 0, e->stream>>>(p.m, a.cta + ctas);
  k_wd_rank<<<(uint32_t)(((size_t)na * 32 + 255) / 256), 256, 0, e->stream>>>(a);
  // plan on the per-bin totals, then the bins with a take as keys
  if ((rc = ob_begin(e, MM_OFFTICK_WIDEN, a))) return rc;
  const uint32_t plan_grid = (nc + kWdPlanWarps - 1) / kWdPlanWarps;
  k_wd_plan<<<plan_grid, kWdPlanWarps * 32, 0, e->stream>>>(a);
  uint32_t absorbed = 0;  // the unbudgeted plan's
  if (e->ob[MM_OFFTICK_WIDEN].budgeted) {
    CK(cudaMemcpyAsync(&absorbed, a.ctr + kWdAbsorbed, 4, cudaMemcpyDeviceToHost, e->stream));
    if ((rc = ob_allot(e, MM_OFFTICK_WIDEN, a))) return rc;
    if (a.cap) {  // again, capped, from the state the first plan started from
      CK(cudaMemcpyAsync(b.rem, p.m.tot, (size_t)e->K * 4, cudaMemcpyDeviceToDevice, e->stream));
      CK(cudaMemcpyAsync(a.cur, a.part, (size_t)e->n_segs * 4, cudaMemcpyDeviceToDevice, e->stream));
      CK(cudaMemsetAsync(a.ctr, 0, kWdWords * 4, e->stream));
      k_wd_plan<<<plan_grid, kWdPlanWarps * 32, 0, e->stream>>>(a);
    }
  }
  bf_keys(e, a.ctr);
  k_wd_bases<<<1, 32, 0, e->stream>>>(a);
  CK(cudaGetLastError());
  uint32_t h[kWdWords];
  CK(cudaMemcpyAsync(h, a.ctr, sizeof(h), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  const uint32_t nl = h[kWdLobbies], nm = h[kBfPlayers];
  st->n_lobbies = nl; st->n_matched = nm;
  st->n_absorbed = e->ob[MM_OFFTICK_WIDEN].budgeted ? absorbed : h[kWdAbsorbed];
  if (lobby_cap < nl || member_cap < nm)
    return set_err(e, MM_E_CAP, "need lobby_cap >= %u and member_cap >= %u", nl, nm);
  if (nl == 0) return MM_OK;
  // from here on the call changes the pool
  if ((rc = bf_take(e, h, true))) return rc;
  CK(s.hdr.reserve(nl));
  a.hdr = s.hdr;
  k_wd_hdr<<<(nl + 255) / 256, 256, 0, e->stream>>>(a, nl);
  const uint32_t np = h[kBfPieces], pgrid = (uint32_t)(((size_t)np * 32 + 255) / 256);
  bf_out(e, np, a.mbase, b.staging.p, b.members.p);
  // each member's stamp and c from its piece (the off-tick report; c also feeds team_balance)
  auto& o = e->ot;
  CK(e->tb.cval.reserve((size_t)e->capacity + 64));
  CK(o.ts.reserve(nm)); CK(o.imb.reserve(nl));
  bf_out(e, np, a.mbase, b.staging_ts.p, o.ts.p);
  k_tb_pieces<<<pgrid, 256, 0, e->stream>>>(np, b.piece, a.mbase, e->d_bin_key, e->tb.cval);
  if (e->tb_mask) {  // team_balance: the tick's balance kernel
    TbArgs t{};
    t.hdr = s.hdr; t.n_lob = nl; t.members = b.members; t.mask = e->tb_mask; t.mode_tsize = e->d_mode_tsize;
    t.cval = e->tb.cval; t.imb = o.imb;
    k_tb_lobby<true><<<grid256(e, (uint64_t)nl * 32, 8), 256, 0, e->stream>>>(t);
  }
  return wd_finish(e, MM_OFFTICK_WIDEN, a, nl, nm, e->tb_mask, lobbies, member_ids, nullptr, &st->device_us);
}

// ---- mm_locate (mm_locate.cuh) -------------------------------------------------------------------------------------
int locate(mm_engine* e, uint64_t now, uint32_t n, const uint64_t* id, mm_player_status* out) {
  auto& s = e->loc;
  const Pool& p = e->pool[e->cur];
  const size_t wb = (size_t)e->Kp + 2, nc = e->n_cut, nm = e->cfg.n_modes;
  CK(s.id.reserve(n)); CK(s.out.reserve(n)); CK(s.tab.reserve(3 * wb + 2 * nc + nm + e->n_chunks));
  uint32_t *pos = s.tab, *ob = pos + wb, *bl = ob + wb, *cand = bl + wb, *bud = cand + nc, *rmap = bud + nc + nm;
  CK(cudaMemcpyAsync(s.id, id, (size_t)n * 8, cudaMemcpyHostToDevice, e->stream));
  // the budgets as set now (the tick's device copy is brought up to date only by the next tick)
  if (!e->bud_queue.empty()) CK(cudaMemcpyAsync(bud, e->bud_queue.data(), nc * 4, cudaMemcpyHostToDevice, e->stream));
  if (!e->bud_mode.empty()) CK(cudaMemcpyAsync(bud + nc, e->bud_mode.data(), nm * 4, cudaMemcpyHostToDevice, e->stream));
  TailArgs t = tail_args(e);
  t.outbase = ob; t.binlim = bl; t.cand = cand; t.seg = nullptr; t.ctr = nullptr;
  t.dst = PoolMeta{}; t.dst.tot = pos;
  t.bud_queue = e->bud_queue.empty() ? nullptr : bud;
  t.bud_mode = e->bud_mode.empty() ? nullptr : bud + nc;
  const size_t smem = (size_t)tail_words(e->Kp, t.layout) * 4;
  k_locate_preview<<<1, kScanBlock, smem, e->stream>>>(t);
  k_loc_rmap<<<e->n_segs, 256, 0, e->stream>>>(p.m, rmap);
  LocateArgs a{};
  a.n = n; a.id = s.id; a.act = act_view(e); a.pool = p.v; a.meta = p.m;
  a.n_slots = (uint32_t)pool_slots(e); a.gen = e->gen; a.n_groups = e->cfg.n_groups; a.now = (uint32_t)now;
  a.bin_seg = e->d_bin_seg; a.seg_bin_lo = e->d_seg_bin_lo; a.seg_L = e->d_seg_L; a.part_cut = e->d_part_cut;
  a.cut_lp_lo = e->d_cut_lp_lo; a.rmap = rmap; a.pos = pos; a.outbase = ob; a.binlim = bl; a.out = s.out;
  a.tb_mask = e->tb_mask; a.arrival = e->cfg.order_mode == MM_ORDER_ARRIVAL; a.mode_tsize = e->d_mode_tsize;
  a.bin_key = e->d_bin_key; a.key_lo = e->key_lo; a.KR = e->KR; a.pt = pt_view(e, e->pt.cur);
  k_locate<<<(uint32_t)(((size_t)n * 32 + 255) / 256), 256, 0, e->stream>>>(a);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, s.out, (size_t)n * sizeof(mm_player_status), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return MM_OK;
}

// ---- mm_match_quality (mm_quality.cuh) -----------------------------------------------------------------------------
// The report of a valid last tick with n_lob lobbies (the caller has checked the capacities).
int match_quality(mm_engine* e, mm_queue_quality* per_queue, mm_lobby_quality* per_lobby, uint32_t n_lob) {
  auto& s = e->mq;
  const bool arrival = e->cfg.order_mode == MM_ORDER_ARRIVAL;
  const uint32_t n_cut = e->n_cut, G = e->cfg.n_groups;
  const size_t n_tiles = (size_t)e->n_chunks + e->n_segs;
  // word scratch: cnt [Kp] | qlob [n_cut + 1] | qteam [n_cut + 1] | arrival order: tile offsets [n_tiles] | partition
  // live counts [n_segs] | scan total [1] | lmin [max_lobbies] | lmax [max_lobbies] | team sums [capacity]
  const size_t o_qlob = e->Kp, o_qteam = o_qlob + n_cut + 1, o_tile = o_qteam + n_cut + 1, o_part = o_tile + n_tiles,
               o_tot = o_part + e->n_segs, o_lmin = o_tot + 1, o_lmax = o_lmin + e->max_lobbies,
               o_tsum = o_lmax + e->max_lobbies;
  CK(s.w.reserve(arrival ? o_tsum + e->capacity + 64 : o_tile));
  if (!arrival) CK(s.csum.reserve(e->Kp));
  CK(s.lob.reserve(e->max_lobbies));
  CK(s.rec.reserve(n_cut));
  CK(cudaMemsetAsync(s.rec, 0, (size_t)n_cut * sizeof(mm_queue_quality), e->stream));
  if (n_lob) {
    const Pool& p = e->pool[e->cur ^ 1];  // the pool the last tick read
    MqArgs a{};
    a.pool = p.v; a.meta = p.m; a.left_bits = e->d_left_bits;
    a.n_segs = e->n_segs; a.n_cut = n_cut; a.n_groups = G; a.K = e->K; a.key_lo = e->key_lo; a.KR = e->KR;
    a.bin_key = e->d_bin_key; a.seg_bin_lo = e->d_seg_bin_lo; a.seg_L = e->d_seg_L; a.part_cut = e->d_part_cut;
    a.cut_lp_lo = e->d_cut_lp_lo; a.mode_tsize = e->d_mode_tsize;
    a.cnt = s.w; a.csum = arrival ? nullptr : s.csum.p; a.qlob = s.w + o_qlob; a.qteam = s.w + o_qteam;
    a.lob = s.lob; a.n_lob = n_lob; a.qrec = s.rec;
    a.tb_mask = e->tb_last; a.tb_imb = e->tb.imb;
    CK(cudaMemsetAsync(a.cnt, 0, (size_t)e->Kp * 4, e->stream));
    const uint32_t ctas = tile_ctas(e, e->match_n);
    k_mq_count<kMqBlock><<<ctas, kMqBlock, 0, e->stream>>>(a);
    k_mq_scan<kMqBlock><<<n_cut, kMqBlock, 0, e->stream>>>(a, !arrival);
    k_mq_base<kMqBlock><<<1, kMqBlock, 0, e->stream>>>(a);
    if (arrival) {
      a.tile_off = s.w + o_tile; a.lmin = s.w + o_lmin; a.lmax = s.w + o_lmax; a.tsum = s.w + o_tsum;
      // every team holds at least one matched player: the tick's matched count bounds the team-sum words
      CK(cudaMemsetAsync(a.lmin, 0xFF, (size_t)n_lob * 4, e->stream));
      CK(cudaMemsetAsync(a.lmax, 0, (size_t)n_lob * 4, e->stream));
      CK(cudaMemsetAsync(a.tsum, 0, (size_t)e->last.n_matched * 4, e->stream));
      CK(cudaMemsetAsync(s.w + o_part, 0, ((size_t)e->n_segs + 1) * 4, e->stream));  // partition counts, scan total
      // live slots per virtual tile -> the live slots before each tile (mm_export's count and scan)
      ImgExportArgs x{};
      x.pool = p.v; x.meta = p.m; x.n_segs = e->n_segs; x.tile_cnt = s.w + o_tile; x.part_cnt = s.w + o_part;
      k_img_tiles<kImgBlock, false><<<ctas, kImgBlock, 0, e->stream>>>(x);
      k_scan_small<<<1, 1024, 0, e->stream>>>(tile_count(e, e->match_n), s.w + o_tile, s.w + o_tot);
      k_mq_arrival<kMqBlock><<<ctas, kMqBlock, 0, e->stream>>>(a);
      k_mq_lobby<true><<<(n_lob + 255) / 256, 256, 0, e->stream>>>(a);
    } else {
      k_mq_lobby<false><<<(n_lob + 255) / 256, 256, 0, e->stream>>>(a);
    }
    const uint32_t qctas = std::max<uint32_t>(1, std::min<uint32_t>(n_lob / 1024 + 1, 8u * (uint32_t)e->n_sms));
    k_mq_queue<kMqBlock><<<qctas, kMqBlock, 0, e->stream>>>(a);
    CK(cudaGetLastError());
    if (per_lobby) CK(cudaMemcpyAsync(per_lobby, s.lob, (size_t)n_lob * sizeof(mm_lobby_quality), cudaMemcpyDeviceToHost, e->stream));
  }
  uint32_t n_dev = 0;  // the lobbies the pool's matched players make up: the tick's own count
  if (n_lob) CK(cudaMemcpyAsync(&n_dev, s.w + o_qlob + n_cut, 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemcpyAsync(per_queue, s.rec, (size_t)n_cut * sizeof(mm_queue_quality), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  for (uint32_t c = 0; c < n_cut; ++c) {
    per_queue[c].mode = (uint8_t)(c / G);
    per_queue[c].group = (uint8_t)(c % G);
  }
  if (n_dev != n_lob)
    return set_err(e, MM_E_STATE, "the last tick's pool holds %u matched lobbies, the tick emitted %u", n_dev, n_lob);
  return MM_OK;
}

// ---- parties (mm_party.cuh) ----------------------------------------------------------------------------------------
uint32_t pt_rows_cap(const mm_engine* e) { return e->pt.cap / 2 + 1; }  // a party has at least two members

// The table's buffer b and the match scratch at the capacity's sizes (b's contents are lost).
int pt_alloc(mm_engine* e, int b) {
  auto& t = e->pt.buf[b];
  const size_t r = pt_rows_cap(e), m = (size_t)e->pt.cap + 1;
  t = mm_engine::Party::Buf{};
  CK(t.seq.reserve(r)); CK(t.ts.reserve(r)); CK(t.off.reserve(r)); CK(t.R.reserve(r)); CK(t.bin.reserve(r));
  CK(t.mode.reserve(r)); CK(t.grp.reserve(r)); CK(t.size.reserve(r)); CK(t.dead.reserve(r));
  CK(t.mid.reserve(m)); CK(t.mrat.reserve(m));
  auto& s = e->pt;
  for (auto* a : {&s.tmp, &s.sorted, &s.lob, &s.pos}) { a->reset(); CK(a->reserve(r)); }
  CK(s.pb.reserve((size_t)e->K + 1)); CK(s.pcur.reserve(e->K)); CK(s.ctr.reserve(kPtWords + 2));
  return MM_OK;
}

// Compaction: the queued parties' rows, stable, into the other buffer (their members' active-set values follow).
int pt_compact(mm_engine* e) {
  auto& s = e->pt;
  if (!s.n_rows) { s.n_mem = 0; return MM_OK; }
  const uint32_t n = s.n_rows, g = (n + 255) / 256;
  uint32_t* tot = s.ctr + kPtWords;
  CK(cudaMemsetAsync(tot, 0, 8, e->stream));
  k_pt_keep<<<g, 256, 0, e->stream>>>(n, pt_view(e, s.cur), s.tmp, s.sorted);
  k_scan_small<<<1, 1024, 0, e->stream>>>(n, s.tmp, tot);
  k_scan_small<<<1, 1024, 0, e->stream>>>(n, s.sorted, tot + 1);
  k_pt_move<<<g, 256, 0, e->stream>>>(n, pt_view(e, s.cur), pt_view(e, s.cur ^ 1), s.tmp, s.sorted, act_view(e));
  CK(cudaGetLastError());
  uint32_t h[2];
  CK(cudaMemcpyAsync(h, tot, 8, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  s.n_rows = h[0]; s.n_mem = h[1]; s.cur ^= 1;
  return MM_OK;
}

// mm_set_option("party_capacity", P): both buffers at the new size, the queued parties kept.
int pt_set_capacity(mm_engine* e, int64_t value) {
  auto& s = e->pt;
  if (value < 0 || value > 0x7FFF0000)
    return set_err(e, MM_E_ARG, "party_capacity %lld is out of range", (long long)value);
  if ((uint64_t)value < s.live)
    return set_err(e, MM_E_ARG, "party_capacity %lld is below the %u party members queued", (long long)value, s.live);
  if ((uint32_t)value == s.cap) return MM_OK;
  int rc;
  if (value == 0) {
    s = mm_engine::Party{};  // nothing is queued
    return MM_OK;
  }
  if (s.n_rows && (rc = pt_compact(e))) return rc;  // the queued parties now fill buffer cur from row 0
  const uint32_t old = s.cap;
  s.cap = (uint32_t)value;
  if ((rc = pt_alloc(e, s.cur ^ 1))) { s.cap = old; return rc; }
  if (s.n_rows) {
    const PartyView d = pt_view(e, s.cur ^ 1);
    s.cap = old;
    const PartyView o = pt_view(e, s.cur);
    s.cap = (uint32_t)value;
    const size_t r = s.n_rows, m = s.n_mem;
    CK(cudaMemcpyAsync(d.seq, o.seq, r * 4, cudaMemcpyDeviceToDevice, e->stream));
    CK(cudaMemcpyAsync(d.ts, o.ts, r * 4, cudaMemcpyDeviceToDevice, e->stream));
    CK(cudaMemcpyAsync(d.off, o.off, r * 4, cudaMemcpyDeviceToDevice, e->stream));
    CK(cudaMemcpyAsync(d.R, o.R, r * 4, cudaMemcpyDeviceToDevice, e->stream));
    CK(cudaMemcpyAsync(d.bin, o.bin, r * 2, cudaMemcpyDeviceToDevice, e->stream));
    CK(cudaMemcpyAsync(d.mode, o.mode, r, cudaMemcpyDeviceToDevice, e->stream));
    CK(cudaMemcpyAsync(d.grp, o.grp, r, cudaMemcpyDeviceToDevice, e->stream));
    CK(cudaMemcpyAsync(d.size, o.size, r, cudaMemcpyDeviceToDevice, e->stream));
    CK(cudaMemcpyAsync(d.dead, o.dead, r, cudaMemcpyDeviceToDevice, e->stream));
    CK(cudaMemcpyAsync(d.mid, o.mid, m * 8, cudaMemcpyDeviceToDevice, e->stream));
    CK(cudaMemcpyAsync(d.mrat, o.mrat, m * 4, cudaMemcpyDeviceToDevice, e->stream));
    CK(cudaStreamSynchronize(e->stream));
  }
  s.cur ^= 1;
  return pt_alloc(e, s.cur ^ 1);
}

// the refusals every party call shares
int pt_check(mm_engine* e) {
  if (e->cfg.order_mode != MM_ORDER_RATING) return set_err(e, MM_E_ARG, "parties need MM_ORDER_RATING");
  if (!e->pt.cap) return set_err(e, MM_E_STATE, "no party capacity: set the option party_capacity first");
  if (!e->use_active) return set_err(e, MM_E_STATE, "an MM_F_NO_DEDUPE engine cannot hold parties");
  if (e->stage_count) return staged_err(e);
  return MM_OK;
}

// The compacted table's rows by (bin, age), for mm_party_match and mm_backfill_party: x is set up over them, pb holds
// the bins' first sorted rows and pcur the plan's cursors (a copy of pb).
int pt_sort(mm_engine* e, PtArgs& x) {
  auto& s = e->pt;
  const uint32_t nr = s.n_rows, K = e->K;
  x = PtArgs{};
  x.t = pt_view(e, s.cur); x.n_rows = nr; x.pb = s.pb; x.pcur = s.pcur; x.sorted = s.sorted;
  x.lob = s.lob; x.pos = s.pos; x.mode_tsize = e->d_mode_tsize; x.ctr = s.ctr;
  CK(cudaMemsetAsync(s.pb, 0, ((size_t)K + 1) * 4, e->stream));
  CK(cudaMemsetAsync(s.ctr, 0, (kPtWords + 2) * 4, e->stream));
  if (nr) {
    k_pt_count<<<(nr + 255) / 256, 256, 0, e->stream>>>(x, s.pb);
    k_scan_small<<<1, 1024, 0, e->stream>>>(K + 1, s.pb, s.ctr + kPtWords);
    CK(cudaMemcpyAsync(s.pcur, s.pb, (size_t)K * 4, cudaMemcpyDeviceToDevice, e->stream));
    k_pt_scatter<<<1, kPtScatterBlock, 0, e->stream>>>(x);
    CK(cudaMemcpyAsync(s.pcur, s.pb, (size_t)K * 4, cudaMemcpyDeviceToDevice, e->stream));  // the plan's cursors
  }
  return MM_OK;
}

// The enqueue pipeline of mm_enqueue_party and mm_merge_parties (after pt_check, n > 0).  seq: every party's own
// number (MM_PARTY_KEEP_SEQ: seq_next does not move), else seq_next + index.  exact: MM_E_CAP with every claim undone
// if a party would get code 3, decided from the scanned member count of the code-1 parties (one counter read) before
// any row or active-set value is written.
int pt_enqueue(mm_engine* e, uint32_t n, const uint8_t* size, const uint64_t* ids, const int32_t* rating,
               const uint8_t* mode, const uint32_t* enq_ts, const uint32_t* seq, bool exact, uint8_t* accepted) {
  int rc;
  auto& s = e->pt;
  std::vector<uint32_t> moff(n), mparty;
  uint32_t m = 0;
  for (uint32_t j = 0; j < n; ++j) {
    moff[j] = m;
    m += size[j];
    mparty.insert(mparty.end(), size[j], j);
  }
  if ((rc = act_room(e, m, m))) return rc;
  if (!exact) e->fresh = false;
  if (s.n_mem + (uint64_t)m > s.cap && (rc = pt_compact(e))) return rc;
  CK(s.in_size.reserve(n)); CK(s.in_mode.reserve(n)); CK(s.in_code.reserve(n)); CK(s.in_ts.reserve(n));
  CK(s.in_moff.reserve(n)); CK(s.in_msz.reserve(n)); CK(s.in_one.reserve(n));
  if (seq) {
    CK(s.in_seq.reserve(n));
    CK(cudaMemcpyAsync(s.in_seq, seq, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
  }
  const size_t mm = std::max<uint32_t>(m, 1);
  CK(s.in_pre.reserve(mm)); CK(s.in_mparty.reserve(mm)); CK(s.in_id.reserve(mm)); CK(s.in_hslot.reserve(mm));
  CK(s.in_rating.reserve(mm));
  CK(cudaMemcpyAsync(s.in_size, size, n, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(s.in_mode, mode, n, cudaMemcpyHostToDevice, e->stream));
  if (enq_ts) CK(cudaMemcpyAsync(s.in_ts, enq_ts, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(s.in_moff, moff.data(), (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
  if (m) {
    CK(cudaMemcpyAsync(s.in_mparty, mparty.data(), (size_t)m * 4, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(s.in_id, ids, (size_t)m * 8, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(s.in_rating, rating, (size_t)m * 4, cudaMemcpyHostToDevice, e->stream));
  }
  CK(cudaMemsetAsync(s.ctr, 0, (kPtWords + 2) * 4, e->stream));
  PtEnqArgs a{};
  a.n = n; a.m = m; a.size = s.in_size; a.moff = s.in_moff; a.mparty = s.in_mparty; a.id = s.in_id;
  a.rating = s.in_rating; a.mode = s.in_mode; a.ts = enq_ts ? s.in_ts.p : nullptr; a.act = act_view(e);
  a.bm = bin_map(e); a.grp_lut = e->d_grp_lut; a.mode_tsize = e->d_mode_tsize; a.n_modes = e->cfg.n_modes;
  a.hslot = s.in_hslot; a.pre = s.in_pre; a.code = s.in_code; a.msz = s.in_msz; a.one = s.in_one;
  a.tot = s.ctr + kPtWords; a.room = s.cap - s.n_mem; a.rows0 = s.n_rows; a.mem0 = s.n_mem; a.seq0 = e->seq_next;
  a.seq = seq ? s.in_seq.p : nullptr; a.pt = pt_view(e, s.cur); a.ctr = s.ctr;
  const uint32_t gm = (m + 255) / 256, gn = (n + 255) / 256;
  if (m) k_pt_claim<<<gm, 256, 0, e->stream>>>(a);
  k_pt_resolve<<<gn, 256, 0, e->stream>>>(a);
  k_scan_small<<<1, 1024, 0, e->stream>>>(n, s.in_msz, a.tot);
  k_scan_small<<<1, 1024, 0, e->stream>>>(n, s.in_one, a.tot + 1);
  if (exact) {
    uint32_t want = 0;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(&want, a.tot, 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    if (want > a.room) {
      if (m) k_pt_unclaim<<<gm, 256, 0, e->stream>>>(a);
      CK(cudaGetLastError());
      CK(cudaStreamSynchronize(e->stream));
      return set_err(e, MM_E_CAP, "%u party members to merge, the party table has room for %u", want, a.room);
    }
    e->fresh = false;
  }
  k_pt_commit<<<gn, 256, 0, e->stream>>>(a);
  if (m) k_pt_members<<<gm, 256, 0, e->stream>>>(a);
  CK(cudaGetLastError());
  std::vector<uint8_t> code(n);
  uint32_t h[kPtWords];
  CK(cudaMemcpyAsync(code.data(), s.in_code, n, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemcpyAsync(h, s.ctr, sizeof(h), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  uint32_t rows = 0;
  for (uint32_t j = 0; j < n; ++j) rows += code[j] == 1;
  const uint32_t acc = h[kPtAccepted];
  s.n_rows += rows; s.n_mem += acc; s.live += acc;
  e->n_active += acc;
  if (!e->dense_ids) e->n_tomb += h[kPtReleased];
  if (!seq) e->seq_next += n;
  if (accepted) std::memcpy(accepted, code.data(), n);
  return MM_OK;
}

int enqueue_party(mm_engine* e, uint32_t n, const uint8_t* size, const uint64_t* ids, const int32_t* rating,
                  const uint8_t* mode, const uint32_t* enq_ts, uint8_t* accepted) {
  int rc = pt_check(e);
  if (rc || n == 0) return rc;
  return pt_enqueue(e, n, size, ids, rating, mode, enq_ts, nullptr, false, accepted);
}

// mm_export_parties: select and count (k_pt_sel, the scans, one counter read), then the columns gathered in age order
// into device scratch and released in the same pass (k_pt_export), one device-to-host copy.
int export_parties(mm_engine* e, const uint8_t* queues, void* buf, uint64_t cap, uint64_t* n_bytes) {
  int rc = pt_check(e);
  if (rc) return rc;
  auto& s = e->pt;
  const uint32_t nr = s.n_rows, W = id_bytes(e), g = (nr + 255) / 256;
  const PartyView t = pt_view(e, s.cur);
  const uint8_t* sel = nullptr;
  uint32_t h[2] = {0, 0};  // parties, members
  uint32_t* tot = s.ctr + kPtWords;
  if (nr) {
    if (queues) {
      CK(e->d_sel.reserve(kMaxSegs));
      CK(cudaMemcpyAsync(e->d_sel, queues, e->n_cut, cudaMemcpyHostToDevice, e->stream));
      sel = e->d_sel;
    }
    CK(cudaMemsetAsync(s.ctr, 0, (kPtWords + 2) * 4, e->stream));
    k_pt_sel<<<g, 256, 0, e->stream>>>(nr, t, sel, e->cfg.n_groups, s.tmp, s.sorted);
    k_scan_small<<<1, 1024, 0, e->stream>>>(nr, s.tmp, tot);
    k_scan_small<<<1, 1024, 0, e->stream>>>(nr, s.sorted, tot + 1);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(h, tot, 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
  }
  const uint32_t P = h[0], M = h[1];
  const PtImgLayout l = pt_img_layout(P, M, W);
  *n_bytes = l.off[6];
  if (!buf) return MM_OK;
  if (cap < l.off[6]) return set_err(e, MM_E_CAP, "need cap >= %llu", (unsigned long long)l.off[6]);
  uint8_t* out = static_cast<uint8_t*>(buf);
  mm_image_header hd{};
  hd.magic = MM_PARTY_IMAGE_MAGIC; hd.version = MM_IMAGE_VERSION; hd.abi_version = MM_ABI_VERSION; hd.id_bytes = W;
  hd.total_bytes = l.off[6]; hd.n_parts = P; hd.n_players = M; hd.n_active = 0; hd.seq_next = e->seq_next;
  hd.config = e->cfg;
  std::memcpy(out, &hd, sizeof(hd));
  if (!P) return MM_OK;
  const uint64_t body = l.off[6] - l.off[0];
  CK(e->d_img.reserve(body));
  uint8_t* d = e->d_img;
  CK(cudaMemsetAsync(d, 0, body, e->stream));
  PtImgCols c{};
  c.size = d; c.seq = reinterpret_cast<uint32_t*>(d + (l.off[1] - l.off[0]));
  c.ts = reinterpret_cast<uint32_t*>(d + (l.off[2] - l.off[0])); c.mode = d + (l.off[3] - l.off[0]);
  c.id = d + (l.off[4] - l.off[0]); c.rating = reinterpret_cast<int32_t*>(d + (l.off[5] - l.off[0])); c.id_bytes = W;
  k_pt_export<<<g, 256, 0, e->stream>>>(nr, t, sel, e->cfg.n_groups, s.tmp, s.sorted, c, act_view(e),
                                        s.ctr + kPtReleased);
  CK(cudaGetLastError());
  uint32_t freed = 0;
  CK(cudaMemcpyAsync(out + l.off[0], d, body, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemcpyAsync(&freed, s.ctr + kPtReleased, 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  s.live -= M;
  erase_active(e, freed);
  return MM_OK;
}

// mm_merge_parties: every image check on the host, then pt_enqueue with its exact room decision.
int merge_parties(mm_engine* e, const uint8_t* buf, uint64_t nb, uint32_t flags, uint8_t* code, uint32_t* n_merged) {
  int rc = pt_check(e);
  if (rc) return rc;
  auto bad = [&](const char* what) { return set_err(e, MM_E_ARG, "party image rejected: %s", what); };
  if (flags & ~MM_PARTY_KEEP_SEQ) return bad("unknown flags");
  mm_image_header h;
  if (nb < sizeof(h)) return bad("shorter than its header");
  std::memcpy(&h, buf, sizeof(h));
  if (h.magic != MM_PARTY_IMAGE_MAGIC) return bad("bad magic (not an mm_export_parties image)");
  if (h.version != MM_IMAGE_VERSION || h.abi_version != MM_ABI_VERSION) return bad("unknown version");
  if (h.id_bytes != id_bytes(e)) return bad("id width differs from the engine's");
  if (h.config.flags & MM_F_NO_DEDUPE) return bad("written by an MM_F_NO_DEDUPE engine");
  const uint32_t P = h.n_parts, M = h.n_players, W = h.id_bytes;
  const PtImgLayout l = pt_img_layout(P, M, W);
  if (h.n_active || h.total_bytes != l.off[6] || nb != l.off[6])
    return bad("length does not match the header's section counts");
  const uint8_t* size = buf + l.off[0];
  const uint8_t* mode = buf + l.off[3];
  std::vector<uint32_t> seq(P), ts(P);
  std::vector<int32_t> rating(M);
  std::vector<uint64_t> ids(M);
  std::memcpy(seq.data(), buf + l.off[1], (size_t)P * 4);
  std::memcpy(ts.data(), buf + l.off[2], (size_t)P * 4);
  std::memcpy(rating.data(), buf + l.off[5], (size_t)M * 4);
  uint64_t sum = 0;
  for (uint32_t j = 0; j < P; ++j) {
    if (size[j] < 2) return bad("a party of fewer than 2 members");
    sum += size[j];
  }
  if (sum != M) return bad("party sizes do not add up to the member count");
  const uint64_t lim = id_limit(e);
  for (uint32_t k = 0; k < M; ++k) {
    if (W == 8) std::memcpy(&ids[k], buf + l.off[4] + 8ull * k, 8);
    else { uint32_t x; std::memcpy(&x, buf + l.off[4] + 4ull * k, 4); ids[k] = x; }
    if (ids[k] >= lim) return bad("id out of range");
  }
  for (uint32_t j = 0; j < P; ++j) {
    const uint32_t age = seq[j] - h.seq_next;  // (seq - seq_next) mod 2^32: the oldest first
    if (age == 0 || (j && age <= seq[j - 1] - h.seq_next)) return bad("sequence numbers out of order");
  }
  const bool keep = flags & MM_PARTY_KEEP_SEQ;
  if (keep && (e->pt.live || e->seq_next != h.seq_next))
    return set_err(e, MM_E_STATE,
                   "MM_PARTY_KEEP_SEQ needs no queued party and seq_next %u (the image's): %u party members queued, "
                   "seq_next %u", h.seq_next, e->pt.live, e->seq_next);
  if (P == 0) return MM_OK;
  std::vector<uint8_t> c(P);
  if ((rc = pt_enqueue(e, P, size, ids.data(), rating.data(), mode, ts.data(), keep ? seq.data() : nullptr, true,
                       c.data())))
    return rc;
  uint32_t k = 0;
  for (uint8_t x : c) k += x == 1;
  *n_merged = k;
  if (code) std::memcpy(code, c.data(), P);
  return MM_OK;
}

int pq_err(mm_engine* e, uint32_t err) {
  return set_err(e, MM_E_ARG, "party requeue refused:%s%s%s%s%s%s%s%s", err & kPqBadId ? " id out of range" : "",
                 err & kPqBadMode ? " mode out of range" : "",
                 err & kPqBadSize ? " size below 2 or above the mode's team_size" : "",
                 err & kPqBadRating ? " party rating without a group" : "",
                 err & kPqOrder ? " parties not in age order" : "",
                 err & kPqSeqNext ? " sequence number equal to seq_next" : "", err & kPqDup ? " duplicate id" : "",
                 err & kPqSeqLive ? " sequence number of a queued party" : "");
}

// mm_requeue_party: check, code and seat on the device, one counter read that decides every refusal, then the merge of
// the live rows and the requeued parties into the other buffer (mm_party.cuh, "requeue").  The solo pool is not read
// beyond the mode byte of a member's own slot.
int requeue_party(mm_engine* e, uint32_t n, const uint8_t* size, const uint64_t* ids, const int32_t* rating,
                  const uint8_t* mode, const uint32_t* enq_ts, const uint32_t* seq, uint8_t* codes,
                  uint32_t* n_requeued) {
  int rc = pt_check(e);
  if (rc || n == 0) return rc;
  auto& s = e->pt;
  std::vector<uint32_t> moff(n);
  uint32_t m = 0;
  for (uint32_t j = 0; j < n; ++j) {
    moff[j] = m;
    m += size[j];
  }
  const size_t mm = std::max<uint32_t>(m, 1);
  const uint64_t sc = seen_keys(m);
  CK(s.in_size.reserve(n)); CK(s.in_mode.reserve(n)); CK(s.in_code.reserve(n)); CK(s.in_ts.reserve(n));
  CK(s.in_moff.reserve(n)); CK(s.in_msz.reserve(n)); CK(s.in_one.reserve(n)); CK(s.in_seq.reserve(n));
  CK(s.in_at.reserve(2 * (size_t)n));
  CK(s.in_pre.reserve(mm)); CK(s.in_id.reserve(mm)); CK(s.in_hslot.reserve(mm)); CK(s.in_rating.reserve(mm));
  CK(s.rq_ctr.reserve(kPqWords));
  CK(e->d_mrg_seen.reserve(sc));
  CK(cudaMemcpyAsync(s.in_size, size, n, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(s.in_mode, mode, n, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(s.in_seq, seq, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
  if (enq_ts) CK(cudaMemcpyAsync(s.in_ts, enq_ts, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(s.in_moff, moff.data(), (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
  if (m) {
    CK(cudaMemcpyAsync(s.in_id, ids, (size_t)m * 8, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(s.in_rating, rating, (size_t)m * 4, cudaMemcpyHostToDevice, e->stream));
  }
  CK(cudaMemsetAsync(e->d_mrg_seen, 0xFF, sc * 8, e->stream));
  CK(cudaMemsetAsync(s.rq_ctr, 0, kPqWords * 4, e->stream));
  const Pool& p = e->pool[e->cur];
  const uint32_t nr = s.n_rows;
  PqArgs a{};
  a.n = n; a.m = m; a.size = s.in_size; a.moff = s.in_moff; a.id = s.in_id; a.rating = s.in_rating;
  a.mode = s.in_mode; a.ts = enq_ts ? s.in_ts.p : nullptr; a.seq = s.in_seq; a.seq_next = e->seq_next;
  a.id_limit = id_limit(e); a.act = act_view(e); a.pool_mode = p.v.mode; a.n_slots = (uint32_t)pool_slots(e);
  a.gen = e->gen; a.seen = e->d_mrg_seen; a.seen_mask = sc - 1; a.bm = bin_map(e); a.grp_lut = e->d_grp_lut;
  a.mode_tsize = e->d_mode_tsize; a.n_modes = e->cfg.n_modes;
  a.hslot = s.in_hslot; a.cls = s.in_pre; a.code = s.in_code; a.msz = s.in_msz; a.one = s.in_one; a.at = s.in_at;
  a.t = pt_view(e, s.cur); a.n_rows = nr; a.keep = s.tmp; a.lmsz = s.sorted; a.lseq = s.lob; a.lmo = s.pos;
  a.d = pt_view(e, s.cur ^ 1);
  a.ctr = s.rq_ctr;
  const uint32_t gm = (m + 255) / 256, gn = (n + 255) / 256, gr = (nr + 255) / 256;
  if (m) k_pq_check<<<gm, 256, 0, e->stream>>>(a);
  k_pq_party<<<gn, 256, 0, e->stream>>>(a);
  k_scan_small<<<1, 1024, 0, e->stream>>>(n, s.in_msz, s.rq_ctr + kPqMem);
  k_scan_small<<<1, 1024, 0, e->stream>>>(n, s.in_one, s.rq_ctr + kPqRows);
  if (nr) {
    k_pt_keep<<<gr, 256, 0, e->stream>>>(nr, a.t, s.tmp, s.sorted);
    k_scan_small<<<1, 1024, 0, e->stream>>>(nr, s.tmp, s.rq_ctr + kPqLiveRows);
    k_scan_small<<<1, 1024, 0, e->stream>>>(nr, s.sorted, s.rq_ctr + kPqLiveMem);
    k_pq_live<<<gr, 256, 0, e->stream>>>(a);
  }
  k_pq_seat<<<gn, 256, 0, e->stream>>>(a);
  CK(cudaGetLastError());
  uint32_t h[kPqWords];
  CK(cudaMemcpyAsync(h, s.rq_ctr, sizeof(h), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  if (h[kPqErr]) return pq_err(e, h[kPqErr]);
  if (h[kPqMem] > s.cap - s.live)
    return set_err(e, MM_E_CAP, "%u party members to requeue, the party table has room for %u", h[kPqMem],
                   s.cap - s.live);
  if (h[kPqRows]) {
    if (nr) k_pq_move<<<gr, 256, 0, e->stream>>>(a);
    k_pq_write<<<gn, 256, 0, e->stream>>>(a);
    CK(cudaGetLastError());
  }
  if (codes) CK(cudaMemcpyAsync(codes, s.in_code, n, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  if (h[kPqRows]) {
    s.n_rows = h[kPqLiveRows] + h[kPqRows]; s.n_mem = h[kPqLiveMem] + h[kPqMem]; s.live += h[kPqMem];
    s.cur ^= 1;
  }
  if (n_requeued) *n_requeued = h[kPqRows];
  return MM_OK;
}

// The rules of mm_party_match and mm_party_locate: mm_widen's checks, the team limit and the refusals of every party
// call.
int pt_rules(mm_engine* e, const mm_widen_rule* rules, std::vector<WdRule>& rule, bool& any) {
  const mm_config& c = e->cfg;
  const uint32_t G = c.n_groups;
  int rc = wd_rules(e, rules, rule, any);
  if (rc) return rc;
  for (uint32_t q = 0; q < e->n_cut; ++q)
    if (rule[q].min_wait != MM_WIDEN_OFF && c.modes[q / G].teams > kPtMaxTeams)
      return set_err(e, MM_E_ARG, "rule %u: mode %u has %u teams (parties: at most %u)", q, q / G, c.modes[q / G].teams,
                     kPtMaxTeams);
  return pt_check(e);
}

int party_match(mm_engine* e, uint64_t now, const mm_widen_rule* rules, mm_lobby_hdr* lobbies, uint32_t lobby_cap,
                uint64_t* member_ids, uint64_t member_cap, mm_party_stats* st) {
  const mm_config& c = e->cfg;
  const uint32_t nc = e->n_cut;
  std::vector<WdRule> rule;
  bool any = false;
  int rc = pt_rules(e, rules, rule, any);
  if (rc) return rc;
  auto& s = e->pt;
  if (!any || !s.live) return MM_OK;
  CK(cudaEventRecord(e->ev[0], e->stream));
  if ((rc = pt_compact(e))) return rc;
  const Pool& p = e->pool[e->cur];
  const uint32_t nr = s.n_rows, K = e->K, gr = (nr + 255) / 256;
  PtArgs x;
  if ((rc = pt_sort(e, x))) return rc;
  // the plan, on the solo pool's per-bin totals (the mm_widen scratch)
  auto& w = e->wd;
  auto& b = e->bf;
  CK(w.anc.reserve((size_t)nr * 3));
  uint32_t maxT = 1;
  for (uint32_t m = 0; m < c.n_modes; ++m) maxT = std::max<uint32_t>(maxT, c.modes[m].teams);
  // each team's walk empties all bins but its last
  if ((rc = bf_plan_scratch(e, std::min<uint64_t>((uint64_t)nr * maxT, p.n) + K))) return rc;
  WdArgs a;
  if ((rc = wd_setup(e, now, rule, 0, a))) return rc;
  a.rem = b.rem; a.piece = b.piece;
  a.rec = reinterpret_cast<uint2*>(w.anc.p); a.mbase = w.anc + 2 * (size_t)nr;
  if ((rc = ob_begin(e, MM_OFFTICK_PARTY_MATCH, a))) return rc;
  CK(cudaMemsetAsync(a.qlob, 0, nc * 4, e->stream));
  const uint32_t plan_grid = (nc + kPtPlanWarps - 1) / kPtPlanWarps;
  k_pt_plan<<<plan_grid, kPtPlanWarps * 32, 0, e->stream>>>(x, a);
  uint32_t first[2] = {0u, 0u};  // the unbudgeted plan's anchors and absorbed anchors
  const bool budgeted = e->ob[MM_OFFTICK_PARTY_MATCH].budgeted;
  if (budgeted) {
    CK(cudaMemcpyAsync(first, s.ctr + kPtAnchors, 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(first + 1, a.ctr + kWdAbsorbed, 4, cudaMemcpyDeviceToHost, e->stream));
    if ((rc = ob_allot(e, MM_OFFTICK_PARTY_MATCH, a))) return rc;
    if (a.cap) {  // again, capped, from the state the first plan started from
      CK(cudaMemsetAsync(s.lob, 0xFF, (size_t)nr * 4, e->stream));  // kPtNone: no row placed
      CK(cudaMemcpyAsync(s.pcur, s.pb, (size_t)K * 4, cudaMemcpyDeviceToDevice, e->stream));
      CK(cudaMemcpyAsync(b.rem, p.m.tot, (size_t)K * 4, cudaMemcpyDeviceToDevice, e->stream));
      CK(cudaMemsetAsync(a.ctr, 0, kWdWords * 4, e->stream));
      CK(cudaMemsetAsync(s.ctr + kPtAnchors, 0, 2 * 4, e->stream));  // kPtAnchors, kPtPlaced
      k_pt_plan<<<plan_grid, kPtPlanWarps * 32, 0, e->stream>>>(x, a);
    }
  }
  bf_keys(e, a.ctr);
  k_wd_bases<<<1, 32, 0, e->stream>>>(a);
  CK(cudaGetLastError());
  CK(cudaEventRecord(e->ev[4], e->stream));
  uint32_t h[kWdWords], hp[kPtWords];
  std::vector<uint32_t> qlob(nc);
  CK(cudaMemcpyAsync(h, a.ctr, sizeof(h), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemcpyAsync(hp, s.ctr, sizeof(hp), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemcpyAsync(qlob.data(), a.qlob, nc * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  uint64_t nm = 0;
  for (uint32_t q = 0; q < nc; ++q)
    if (rule[q].min_wait != MM_WIDEN_OFF) nm += (uint64_t)qlob[q] * rule[q].L;
  const uint32_t nl = h[kWdLobbies], ns = h[kBfPlayers];
  st->n_anchors = budgeted ? first[0] : hp[kPtAnchors]; st->n_lobbies = nl; st->n_matched = (uint32_t)nm;
  st->n_parties = hp[kPtPlaced]; st->n_absorbed = budgeted ? first[1] : h[kWdAbsorbed];
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, e->ev[0], e->ev[4]));
  st->device_us = ms * 1000.f;  // a refused or empty call reports the table, sort and plan it ran
  if (lobby_cap < nl || member_cap < nm)
    return set_err(e, MM_E_CAP, "need lobby_cap >= %u and member_cap >= %llu", nl, (unsigned long long)nm);
  if (nl == 0) return MM_OK;
  // from here on the call changes the pool and the table
  if (ns && (rc = bf_take(e, h, true))) return rc;
  CK(b.members.reserve(nm));
  CK(w.hdr.reserve(nl));
  a.hdr = w.hdr;
  k_wd_hdr<<<(nl + 255) / 256, 256, 0, e->stream>>>(a, nl);
  const uint32_t np = h[kBfPieces], pgrid = (uint32_t)(((size_t)np * 32 + 255) / 256);
  if (np) bf_out(e, np, a.mbase, b.staging.p, b.members.p);
  x.members = b.members;
  k_pt_out<<<gr, 256, 0, e->stream>>>(x, a.mbase, act_view(e));
  // each member's stamp and c (solos from their piece, party members their own rating and their party's stamp) for
  // the off-tick report; c and the continuation bits also feed party_balance's split, which keeps every party whole
  auto& tb = e->tb;
  auto& o = e->ot;
  CK(tb.cval.reserve(std::max<size_t>((size_t)e->capacity + 64, nm)));
  CK(o.ts.reserve(nm)); CK(o.imb.reserve(nl));
  if (e->pb_mask) {
    CK(tb.cont.reserve(nl));
    CK(tb.sum.reserve(1));
    CK(cudaMemsetAsync(tb.cont, 0, (size_t)nl * 4, e->stream));
    CK(cudaMemsetAsync(tb.sum, 0, 8, e->stream));
  }
  if (np) {
    bf_out(e, np, a.mbase, b.staging_ts.p, o.ts.p);
    k_tb_pieces<<<pgrid, 256, 0, e->stream>>>(np, b.piece, a.mbase, e->d_bin_key, tb.cval);
  }
  k_tb_parties<<<gr, 256, 0, e->stream>>>(x, a, e->pb_mask, e->key_lo, e->KR, tb.cval, tb.cont, o.ts);
  if (e->pb_mask) {
    TbArgs v{};
    v.hdr = w.hdr; v.n_lob = nl; v.members = b.members; v.mask = e->pb_mask; v.mode_tsize = e->d_mode_tsize;
    v.cval = tb.cval; v.cont = tb.cont; v.imb_sum = tb.sum; v.imb = o.imb;
    k_tb_lobby<true, true><<<grid256(e, (uint64_t)nl * 32, 8), 256, 0, e->stream>>>(v);
  }
  if ((rc = wd_finish(e, MM_OFFTICK_PARTY_MATCH, a, nl, (uint32_t)nm, e->pb_mask, lobbies, member_ids,
                      e->pb_mask ? &st->sum_imbalance : nullptr, &st->device_us)))
    return rc;
  s.live -= (uint32_t)(nm - ns);
  return MM_OK;
}

// mm_backfill_party (mm_party_backfill.cuh): mm_backfill's request sort, mm_party_match's table sort, then k_pbf_plan;
// one read of the counters decides MM_E_CAP before the pool or the table changes.
int backfill_party(mm_engine* e, uint32_t n, const mm_backfill_req* req, const uint16_t* room, uint16_t* filled,
                   uint32_t* n_taken, uint64_t* member_ids, uint64_t member_cap, uint32_t* n_total) {
  const mm_config& c = e->cfg;
  std::vector<uint32_t> roff(n + 1, 0);
  int rc;
  for (uint32_t j = 0; j < n; ++j) {
    const mm_backfill_req& r = req[j];
    if ((rc = bf_check_req(e, j, r))) return rc;
    const mm_mode_desc& md = c.modes[r.mode];
    if (md.teams > kPtMaxTeams)
      return set_err(e, MM_E_ARG, "request %u: mode %u has %u teams (parties: at most %u)", j, r.mode, md.teams,
                     kPtMaxTeams);
    uint64_t sum = 0;
    for (uint32_t t = 0; t < md.teams; ++t) {
      const uint16_t v = room[roff[j] + t];
      if (v > md.team_size)
        return set_err(e, MM_E_ARG, "request %u: team %u has room %u > team_size %u", j, t, v, md.team_size);
      sum += v;
    }
    if (sum != r.count)
      return set_err(e, MM_E_ARG, "request %u: count %u is not the sum %llu of its room entries", j, r.count,
                     (unsigned long long)sum);
    roff[j + 1] = roff[j] + md.teams;
  }
  if ((rc = pt_check(e))) return rc;
  if (n == 0) return MM_OK;
  const uint32_t nc = e->n_cut, ne = roff[n];
  const size_t rw = sizeof(BfReq) / 4;
  std::vector<uint32_t> in;
  const uint32_t nq = bf_sort(e, n, req, in);
  // the table: compacted, then the rows by (bin, age)
  auto& s = e->pt;
  if ((rc = pt_compact(e))) return rc;
  const Pool& p = e->pool[e->cur];
  const uint32_t nr = s.n_rows, gr = (nr + 255) / 256;
  PtArgs x;
  if ((rc = pt_sort(e, x))) return rc;
  // the plan, on the solo pool's per-bin totals (the mm_backfill scratch)
  auto& b = e->bf;
  CK(b.in.reserve(in.size())); CK(b.n_taken.reserve(n)); CK(b.req_base.reserve(n)); CK(b.ctr.reserve(kBfWords));
  CK(b.teams.reserve((size_t)n + 1 + 2 * (size_t)ne)); CK(b.room.reserve(std::max<uint32_t>(ne, 1)));
  // every team walk empties all the bins it reaches but its last
  if ((rc = bf_plan_scratch(e, (size_t)ne + e->K))) return rc;
  CK(cudaMemcpyAsync(b.in, in.data(), in.size() * 4, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(b.teams, roff.data(), ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, e->stream));
  if (ne) CK(cudaMemcpyAsync(b.room, room, (size_t)ne * 2, cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemsetAsync(b.ctr, 0, kBfWords * 4, e->stream));
  WdArgs a{};
  a.n_groups = c.n_groups; a.cut_lp_lo = e->d_cut_lp_lo; a.seg_bin_lo = e->d_seg_bin_lo; a.bin_key = e->d_bin_key;
  a.tot = p.m.tot; a.rem = b.rem; a.piece = b.piece; a.ctr = b.ctr;
  PbfArgs q{};
  q.req = reinterpret_cast<const BfReq*>(b.in.p); q.qr = b.in + rw * n; q.queues = b.in + rw * n + nc + 1; q.nq = nq;
  q.roff = b.teams; q.room = b.room; q.filled = b.teams + n + 1; q.tbase = b.teams + n + 1 + ne; q.n_taken = b.n_taken;
  k_pbf_plan<<<(nq + kPtPlanWarps - 1) / kPtPlanWarps, kPtPlanWarps * 32, 0, e->stream>>>(x, a, q);
  bf_keys(e, b.ctr);
  CK(cudaGetLastError());
  uint32_t h[kBfWords];
  std::vector<uint32_t> fill32(ne);
  CK(cudaMemcpyAsync(n_taken, b.n_taken, (size_t)n * 4, cudaMemcpyDeviceToHost, e->stream));
  if (ne) CK(cudaMemcpyAsync(fill32.data(), q.filled, (size_t)ne * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemcpyAsync(h, b.ctr, sizeof(h), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  for (uint32_t i = 0; i < ne; ++i) filled[i] = (uint16_t)fill32[i];
  std::vector<uint32_t> base(n);
  uint32_t total = 0;
  for (uint32_t j = 0; j < n; ++j) { base[j] = total; total += n_taken[j]; }
  *n_total = total;
  if (member_cap < total) return set_err(e, MM_E_CAP, "need member_cap >= %u", total);
  if (total == 0) return MM_OK;
  // from here on the call changes the pool and the table
  const uint32_t ns = h[kBfPlayers], np = h[kBfPieces];
  if (ns && (rc = bf_take(e, h))) return rc;
  CK(b.members.reserve(total));
  CK(cudaMemcpyAsync(b.req_base, base.data(), (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
  if (np) bf_out(e, np, b.req_base, b.staging.p, b.members.p);
  if (total > ns) {
    x.members = b.members;
    k_pbf_pos<<<gr, 256, 0, e->stream>>>(x, q);
    k_pt_out<<<gr, 256, 0, e->stream>>>(x, b.req_base, act_view(e));
  }
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(member_ids, b.members, (size_t)total * 8, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  s.live -= total - ns;
  return MM_OK;
}

int party_read(mm_engine* e, uint32_t party_cap, uint32_t member_cap, uint8_t* size, uint32_t* seq, uint32_t* enq_ts,
               uint8_t* mode, uint8_t* group, int32_t* rating, uint64_t* member_ids, int32_t* member_rating,
               uint32_t* n_parties, uint32_t* n_members) {
  auto& s = e->pt;
  const uint32_t r = s.n_rows, m = s.n_mem;
  std::vector<uint32_t> hseq(r), hts(r), hoff(r);
  std::vector<int32_t> hR(r), hmr(m);
  std::vector<uint8_t> hmode(r), hgrp(r), hsize(r), hdead(r);
  std::vector<uint64_t> hmid(m);
  const PartyView t = pt_view(e, s.cur);
  if (r) {
    CK(cudaMemcpyAsync(hseq.data(), t.seq, r * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(hts.data(), t.ts, r * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(hoff.data(), t.off, r * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(hR.data(), t.R, r * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(hmode.data(), t.mode, r, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(hgrp.data(), t.grp, r, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(hsize.data(), t.size, r, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(hdead.data(), t.dead, r, cudaMemcpyDeviceToHost, e->stream));
  }
  if (m) {
    CK(cudaMemcpyAsync(hmid.data(), t.mid, (size_t)m * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(hmr.data(), t.mrat, (size_t)m * 4, cudaMemcpyDeviceToHost, e->stream));
  }
  CK(cudaStreamSynchronize(e->stream));
  uint32_t np = 0, nm = 0;
  for (uint32_t i = 0; i < r; ++i)
    if (!hdead[i]) { ++np; nm += hsize[i]; }
  *n_parties = np; *n_members = nm;
  if (np > party_cap || nm > member_cap)
    return set_err(e, MM_E_CAP, "need party_cap >= %u and member_cap >= %u", np, nm);
  for (uint32_t i = 0, k = 0, o = 0; i < r; ++i) {
    if (hdead[i]) continue;
    size[k] = hsize[i]; seq[k] = hseq[i]; enq_ts[k] = hts[i]; mode[k] = hmode[i]; group[k] = hgrp[i]; rating[k] = hR[i];
    for (uint32_t j = 0; j < hsize[i]; ++j, ++o) { member_ids[o] = hmid[hoff[i] + j]; member_rating[o] = hmr[hoff[i] + j]; }
    ++k;
  }
  return MM_OK;
}

// ---- party search status (mm_party_status.cuh) ----------------------------------------------------------------------
// mm_party_queue_stats after pt_check: one pass over the rows as they stand (no compaction), the records to out.
int party_queue_stats(mm_engine* e, uint64_t now, mm_party_queue_stat* out) {
  auto& s = e->pst;
  const uint32_t nc = e->n_cut, G = e->cfg.n_groups, nr = e->pt.n_rows;
  const size_t words = (size_t)nc * kPstWords;
  CK(s.rec.reserve(words));
  CK(cudaMemsetAsync(s.rec, 0, words * 4, e->stream));
  if (nr) {
    PstArgs a{};
    a.t = pt_view(e, e->pt.cur); a.n_rows = nr; a.n_groups = G; a.n_cut = nc; a.now = (uint32_t)now; a.out = s.rec;
    const uint32_t grid = grid256(e, nr, 2);
    if (words * 4 <= e->smem_optin) k_pst_stats<true><<<grid, kPstBlock, words * 4, e->stream>>>(a);
    else k_pst_stats<false><<<grid, kPstBlock, 0, e->stream>>>(a);
    CK(cudaGetLastError());
  }
  CK(cudaMemcpyAsync(out, s.rec, words * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  for (uint32_t c = 0; c < nc; ++c) {
    out[c].mode = (uint8_t)(c / G);
    out[c].group = (uint8_t)(c % G);
  }
  return MM_OK;
}

// mm_party_locate after pt_rules, n > 0: mm_party_match's compaction, sort and unbudgeted plan on the same scratch,
// stopped before the take; the budget's allotment and the balance pass into the call's own words; then the answers.
int party_locate(mm_engine* e, uint64_t now, const std::vector<WdRule>& rule, bool any, uint32_t n, const uint64_t* id,
                 mm_party_member_status* out) {
  const mm_config& c = e->cfg;
  const uint32_t nc = e->n_cut, nmodes = c.n_modes;
  auto& s = e->pt;
  auto& z = e->pst;
  int rc;
  if ((rc = pt_compact(e))) return rc;  // every row live, in age order
  const Pool& p = e->pool[e->cur];
  const uint32_t nr = s.n_rows, K = e->K;
  CK(z.id.reserve(n)); CK(z.out.reserve(n));
  CK(z.tab.reserve((size_t)nr + 5 * (size_t)nc + nmodes + 1));
  uint32_t *rank = z.tab, *depth = rank + nr, *qlob = depth + nc, *cand = qlob + nc, *allot = cand + nc,
           *bud = allot + nc, *cut = bud + nc + nmodes;
  CK(cudaMemcpyAsync(z.id, id, (size_t)n * 8, cudaMemcpyHostToDevice, e->stream));
  k_pst_rank<<<1, kPstRankBlock, 0, e->stream>>>(pt_view(e, s.cur), nr, c.n_groups, nc, rank, depth);
  WdArgs a;
  if ((rc = wd_setup(e, now, rule, 0, a))) return rc;  // the rules on the device, for the plan and the answers
  PlocArgs x{};
  if (any && s.live) {  // mm_party_match's plan, unbudgeted, its lobby counts in the call's own words
    auto& w = e->wd;
    auto& b = e->bf;
    PtArgs pa;
    if ((rc = pt_sort(e, pa))) return rc;
    CK(w.anc.reserve((size_t)nr * 3));
    uint32_t maxT = 1;
    for (uint32_t m = 0; m < nmodes; ++m) maxT = std::max<uint32_t>(maxT, c.modes[m].teams);
    if ((rc = bf_plan_scratch(e, std::min<uint64_t>((uint64_t)nr * maxT, p.n) + K))) return rc;
    a.rem = b.rem; a.piece = b.piece;
    a.rec = reinterpret_cast<uint2*>(w.anc.p); a.mbase = w.anc + 2 * (size_t)nr;
    a.qlob = qlob; a.cap = nullptr;
    CK(cudaMemsetAsync(qlob, 0, nc * 4, e->stream));
    k_pt_plan<<<(nc + kPtPlanWarps - 1) / kPtPlanWarps, kPtPlanWarps * 32, 0, e->stream>>>(pa, a);
    k_wd_bases<<<1, 32, 0, e->stream>>>(a);
    const auto& o = e->ob[MM_OFFTICK_PARTY_MATCH];
    if (!o.queue.empty() || !o.mode.empty()) {  // the allowances mm_party_match would cap the plan at (ob_allot's)
      if (!o.queue.empty()) CK(cudaMemcpyAsync(bud, o.queue.data(), nc * 4, cudaMemcpyHostToDevice, e->stream));
      if (!o.mode.empty()) CK(cudaMemcpyAsync(bud + nc, o.mode.data(), nmodes * 4, cudaMemcpyHostToDevice, e->stream));
      k_wd_allot<<<1, kScanBlock, 0, e->stream>>>(a, o.queue.empty() ? nullptr : bud, o.mode.empty() ? nullptr : bud + nc,
                                                  cand, allot, cut);
      x.allot = allot;
    }
    CK(cudaGetLastError());
    if (e->pb_mask) {  // party_balance: the split of every lobby, on member slots that hold their own index
      uint32_t h[kWdWords];
      std::vector<uint32_t> hq(nc);
      CK(cudaMemcpyAsync(h, a.ctr, sizeof(h), cudaMemcpyDeviceToHost, e->stream));
      CK(cudaMemcpyAsync(hq.data(), qlob, nc * 4, cudaMemcpyDeviceToHost, e->stream));
      CK(cudaStreamSynchronize(e->stream));
      uint64_t nm = 0;
      for (uint32_t q = 0; q < nc; ++q)
        if (rule[q].min_wait != MM_WIDEN_OFF) nm += (uint64_t)hq[q] * rule[q].L;
      const uint32_t nl = h[kWdLobbies], np = h[kBfPieces];
      if (nl) {
        CK(z.hdr.reserve(nl)); CK(z.tags.reserve(nm)); CK(z.bal.reserve(2 * nm + nl)); CK(z.sum.reserve(1));
        uint32_t *cval = z.bal, *ts = cval + nm, *cont = ts + nm;
        a.hdr = z.hdr;
        k_wd_hdr<<<(nl + 255) / 256, 256, 0, e->stream>>>(a, nl);  // headers and member bases
        k_pst_tags<<<(uint32_t)((nm + 255) / 256), 256, 0, e->stream>>>((uint32_t)nm, z.tags);
        CK(cudaMemsetAsync(cont, 0, (size_t)nl * 4, e->stream));
        CK(cudaMemsetAsync(z.sum, 0, 8, e->stream));
        if (np)
          k_tb_pieces<<<(uint32_t)(((size_t)np * 32 + 255) / 256), 256, 0, e->stream>>>(np, b.piece, a.mbase,
                                                                                        e->d_bin_key, cval);
        k_tb_parties<<<(nr + 255) / 256, 256, 0, e->stream>>>(pa, a, e->pb_mask, e->key_lo, e->KR, cval, cont, ts);
        TbArgs v{};
        v.hdr = z.hdr; v.n_lob = nl; v.members = z.tags; v.mask = e->pb_mask; v.mode_tsize = e->d_mode_tsize;
        v.cval = cval; v.cont = cont; v.imb_sum = z.sum;
        k_tb_lobby<true, true><<<grid256(e, (uint64_t)nl * 32, 8), 256, 0, e->stream>>>(v);
        CK(cudaGetLastError());
        x.mbase = a.mbase; x.tags = z.tags; x.pb_mask = e->pb_mask;
      }
    }
    x.lob = s.lob; x.pos = s.pos; x.rec = a.rec;
  }
  x.n = n; x.id = z.id; x.act = act_view(e); x.pool = p.v; x.n_slots = (uint32_t)pool_slots(e); x.gen = e->gen;
  x.t = pt_view(e, s.cur); x.n_groups = c.n_groups; x.now = (uint32_t)now; x.rule = a.rule; x.rank = rank;
  x.depth = depth; x.out = z.out;
  k_pst_answer<<<(uint32_t)(((size_t)n * 32 + 255) / 256), 256, 0, e->stream>>>(x);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, z.out, (size_t)n * sizeof(mm_party_member_status), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return MM_OK;
}

// The mask of team_balance / party_balance: set bits name modes < n_modes of two teams of at most kTbMaxS players.
int tb_check_mask(mm_engine* e, const char* name, int64_t value) {
  if (value < 0 || value >= (int64_t)1 << e->cfg.n_modes)
    return set_err(e, MM_E_ARG, "%s 0x%llx names a mode >= n_modes = %u", name, (unsigned long long)value,
                   e->cfg.n_modes);
  for (uint32_t m = 0; m < e->cfg.n_modes; ++m)
    if (((value >> m) & 1) && (e->cfg.modes[m].teams != 2 || e->cfg.modes[m].team_size > kTbMaxS))
      return set_err(e, MM_E_ARG, "%s: mode %u has %u teams of %u (two teams of at most %u only)", name, m,
                     e->cfg.modes[m].teams, e->cfg.modes[m].team_size, kTbMaxS);
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
    if (!e->place_stages || colscan_smem(e) + static_smem + 1024 > e->smem_optin)
      return bail(set_err(e, MM_E_ARG, "key domain too large for shared memory: %u bins", e->Kp));
    bool ok = allow_max_smem(e, k_colscan<false>) == cudaSuccess && allow_max_smem(e, k_colscan<true>) == cudaSuccess &&
              allow_max_smem(e, k_lobby_candidates) == cudaSuccess && allow_max_smem(e, k_hist<512>) == cudaSuccess &&
              allow_max_smem(e, k_place<512>) == cudaSuccess && allow_max_smem(e, k_tick<512>) == cudaSuccess &&
              allow_max_smem(e, k_tick<512, true>) == cudaSuccess &&
              allow_max_smem(e, k_locate_preview) == cudaSuccess && allow_max_smem(e, k_pst_stats<true>) == cudaSuccess;
    if (!ok) return bail(fail(e, cudaGetLastError(), "cudaFuncSetAttribute"));
  }
  e->n_chunks = (e->capacity + kTile - 1) / kTile + e->n_segs + 2;
  if ((uint64_t)e->n_chunks * e->n_segs * 4 > (8ull << 30)) return bail(MM_E_CAP);
  if ((rc = alloc_buffers(e))) return bail(rc);
  {
    size_t sz = std::max(hist_smem_bytes(e->max_nb), place_smem_bytes(e->max_nb, e->place_stages));
    sz = std::max<size_t>(sz, std::max<size_t>((size_t)std::max(kEpiScratchWords, kRowCompactWords) * 4, colscan_smem(e)));
    int coop = 0, nb = 0;
    cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, e->device);
    int nb_bud = 0;  // both forms of the fused kernel must fit: a budget must not change which tick form runs
    if (coop && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k_tick<512>, 512, sz) == cudaSuccess &&
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb_bud, k_tick<512, true>, 512, sz) == cudaSuccess &&
        (uint32_t)std::min(nb, nb_bud) * (uint32_t)e->n_sms >= e->R + e->helpers) {
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
  if (e->h_ctr) cudaFreeHost(e->h_ctr);
  if (e->h_cnt) cudaFreeHost(e->h_cnt);
  for (auto& ev : e->ev)
    if (ev) cudaEventDestroy(ev);
  if (e->stream && e->own_stream) cudaStreamDestroy(e->stream);
  for (auto& st : e->stage)
    if (st.ready) cudaEventDestroy(st.ready);
  if (e->d2h_stream) cudaStreamDestroy(e->d2h_stream);
  if (e->copy_stream) cudaStreamDestroy(e->copy_stream);
  if (e->ev_copy) cudaEventDestroy(e->ev_copy);
  delete e;  // frees the device arrays (on e->device, current here)
  cudaGetLastError();
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
      CK(e->d_hdr_alt.reserve(e->max_lobbies));
      CK(e->d_members32.reserve((size_t)e->capacity + 64));
      CK(e->d_members32_alt.reserve((size_t)e->capacity + 64));
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
  if (!std::strcmp(name, "team_balance")) {
    // EXTENSION (balanced teams, mm_balance.cuh): bit m splits every lobby of mode m into the two teams with the least
    // rating difference.  Exact two-way partitioning only: two teams of at most kTbMaxS players.
    if (int rc = tb_check_mask(e, name, value)) return rc;
    e->tb_mask = (uint32_t)value;
    return MM_OK;
  }
  if (!std::strcmp(name, "party_balance")) {
    // EXTENSION (balanced party lobbies, mm_balance.cuh): bit m splits every mm_party_match lobby of mode m into the
    // two teams with the least rating difference that keep every party whole.
    if (int rc = tb_check_mask(e, name, value)) return rc;
    e->pb_mask = (uint32_t)value;
    return MM_OK;
  }
  if (!std::strcmp(name, "tick_impl")) { e->tick_impl = value != 0; return MM_OK; }
  if (!std::strcmp(name, "party_capacity")) return pt_set_capacity(e, value);  // EXTENSION (parties, mm_party.cuh)
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
    return copy_fence(e);
  };
  rc = enqueue_batch(e, n, e->d_in_id, e->d_in_rating, e->d_in_mode, enq_ts ? e->d_in_ts.p : nullptr, kEnqChunk, upload);
  return enq_finish_host(e, rc, e->copy_stream, n, accepted, nullptr);
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
    int r = copy_fence(e);
    if (r) return r;
    k_unpack<<<(cnt + 255) / 256, 256, 0, e->stream>>>(cnt, e->d_in_handle + base, e->d_in_key + base, e->d_in_id + base,
                                                       e->d_in_rating + base, e->d_in_mode + base);
    CK(cudaGetLastError());
    return MM_OK;
  };
  rc = enqueue_batch(e, n, e->d_in_id, e->d_in_rating, e->d_in_mode, enq_ts ? e->d_in_ts.p : nullptr, kEnqChunk, upload);
  return enq_finish_host(e, rc, e->copy_stream, n, accepted, nullptr);
}

int mm_enqueue_packed_begin(mm_engine* e, uint32_t n, const uint32_t* handle, const uint16_t* key, const uint32_t* enq_ts) {
  if (!e || !n || !handle || !key) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  if (e->stage_count == 2)
    return set_err(e, MM_E_STATE, "both staging slots hold a batch: call mm_enqueue_packed_end first");
  mm_engine::Stage& st = e->stage[(e->stage_head + e->stage_count) & 1];
  // (a slot's previous batch was consumed by an _end that synchronised the engine stream: it may be reallocated)
  CK(st.handle.reserve((size_t)n + 64));
  CK(st.key.reserve((size_t)n + 64));
  CK(st.ts.reserve((size_t)n + 64));
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
  if (e->stage_count == 0) return set_err(e, MM_E_STATE, "no staged batch: call mm_enqueue_packed_begin first");
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
  rc = enqueue_batch(e, n, e->d_in_id, e->d_in_rating, e->d_in_mode, st.has_ts ? st.ts.p : nullptr, kEnqChunkDev, unpack);
  return enq_finish_host(e, rc, e->stream, n, accepted, n_accepted);
}

int mm_enqueue_rejects(mm_engine* e, uint32_t cap, uint32_t* index, uint8_t* code, uint32_t* n_rejects) {
  if (!e || !n_rejects || (cap && (!index || !code))) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  *n_rejects = 0;
  const uint32_t n = e->last_batch_n;
  if (n == 0) return MM_OK;
  CK(e->d_rej_idx.reserve(cap));
  CK(e->d_rej_code.reserve(cap));
  CK(cudaMemsetAsync(&e->d_cnt->rejects, 0, 4, e->stream));
  k_compact_rejects<<<(n + 255) / 256, 256, 0, e->stream>>>(n, e->d_code, cap, e->d_rej_idx, e->d_rej_code,
                                                             &e->d_cnt->rejects);
  CK(cudaGetLastError());
  int rc = read_counters(e);
  if (rc) return rc;
  const uint32_t cnt = e->h_cnt->rejects;
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
  return remove_or_take(e, n, id, n_removed, false);
}

int mm_take(mm_engine* e, uint32_t n, const uint64_t* id, uint32_t* n_taken) {
  return remove_or_take(e, n, id, n_taken, true);
}

int mm_requeue(mm_engine* e, uint32_t n, const uint64_t* id, const int32_t* rating, const uint8_t* mode,
               const uint32_t* enq_ts, const uint32_t* seq, uint8_t* codes, uint32_t* n_requeued) {
  if (n_requeued) *n_requeued = 0;
  if (!e || (n && (!id || !rating || !mode || !seq))) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  const int rc = requeue(e, n, id, rating, mode, enq_ts, seq, codes, n_requeued);
  free_img_scratch(e);
  return rc;
}

int mm_seq_next(mm_engine* e, uint32_t* seq_next) {
  if (!e || !seq_next) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  *seq_next = e->seq_next;
  return MM_OK;
}

int mm_band_candidates(mm_engine* e, int32_t W, uint32_t group, uint64_t* ids, int32_t* rating, uint8_t* mode,
                       uint32_t cap, uint32_t* n_out) {
  if (!e || !n_out || (cap && (!ids || !rating || !mode))) return MM_E_ARG;
  *n_out = 0;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  return band_candidates(e, W, group, ids, rating, mode, cap, n_out);
}

int mm_band_match(mm_engine* e, int32_t W, uint32_t g_first, uint32_t g_last, uint32_t upper_remote,
                  const uint64_t* up_ids, const int32_t* up_rating, const uint8_t* up_mode, uint32_t n_upper,
                  mm_lobby_hdr* lobbies, uint32_t lobby_cap, uint64_t* member_ids, uint64_t member_cap,
                  uint8_t* upper_taken, mm_band_stats* stats) {
  if (!e || !stats || (lobby_cap && !lobbies) || (member_cap && !member_ids) ||
      (n_upper && (!up_ids || !up_rating || !up_mode || !upper_taken)))
    return MM_E_ARG;
  std::memset(stats, 0, sizeof(*stats));
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  return band_match(e, W, g_first, g_last, upper_remote, up_ids, up_rating, up_mode, n_upper, lobbies, lobby_cap,
                    member_ids, member_cap, upper_taken, stats);
}

int mm_backfill(mm_engine* e, uint32_t n, const mm_backfill_req* req, uint32_t* n_taken, uint64_t* member_ids,
                uint64_t member_cap, uint32_t* n_total) {
  if (!e || !n_total || (n && (!req || !n_taken)) || (member_cap && !member_ids)) return MM_E_ARG;
  *n_total = 0;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  return backfill(e, n, req, n_taken, member_ids, member_cap, n_total);
}

int mm_backfill_party(mm_engine* e, uint32_t n, const mm_backfill_req* req, const uint16_t* room, uint16_t* filled,
                      uint32_t* n_taken, uint64_t* member_ids, uint64_t member_cap, uint32_t* n_total) {
  if (!e) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!n_total || (n && (!req || !room || !filled || !n_taken)) || (member_cap && !member_ids))
    return set_err(e, MM_E_ARG, "null n_total, or null req, room, filled, n_taken or member_ids with n = %u", n);
  *n_total = 0;
  CK(cudaSetDevice(e->device));
  return backfill_party(e, n, req, room, filled, n_taken, member_ids, member_cap, n_total);
}

int mm_widen(mm_engine* e, uint64_t now, const mm_widen_rule* rules, mm_lobby_hdr* lobbies, uint32_t lobby_cap,
             uint64_t* member_ids, uint64_t member_cap, mm_widen_stats* stats) {
  if (!e) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  auto& rep = e->ot.rep[MM_OFFTICK_WIDEN];  // void until this call returns MM_OK; its capture sets the lobby count
  rep.valid = false;
  rep.n_lob = 0;
  auto& ob = e->ob[MM_OFFTICK_WIDEN];  // zeros until a call that ran its plan returns MM_OK or MM_E_CAP
  ob.valid = ob.ran = false;
  if (!rules || !stats) return set_err(e, MM_E_ARG, "null rules or stats");
  std::memset(stats, 0, sizeof(*stats));
  if ((lobby_cap && !lobbies) || (member_cap && !member_ids))
    return set_err(e, MM_E_ARG, "null lobbies or member_ids with a non-zero capacity");
  CK(cudaSetDevice(e->device));
  const int rc = widen(e, now, rules, lobbies, lobby_cap, member_ids, member_cap, stats);
  rep.valid = rc == MM_OK;
  ob.valid = ob.ran && (rc == MM_OK || rc == MM_E_CAP);
  return rc;
}

int mm_enqueue_party(mm_engine* e, uint32_t n, const uint8_t* size, const uint64_t* ids, const int32_t* rating,
                     const uint8_t* mode, const uint32_t* enq_ts, uint8_t* accepted) {
  if (!e) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  if (n && (!size || !ids || !rating || !mode)) return set_err(e, MM_E_ARG, "null size, ids, rating or mode with n = %u", n);
  CK(cudaSetDevice(e->device));
  return enqueue_party(e, n, size, ids, rating, mode, enq_ts, accepted);
}

int mm_requeue_party(mm_engine* e, uint32_t n, const uint8_t* size, const uint64_t* ids, const int32_t* rating,
                     const uint8_t* mode, const uint32_t* enq_ts, const uint32_t* seq, uint8_t* codes,
                     uint32_t* n_requeued) {
  if (n_requeued) *n_requeued = 0;
  if (!e) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  if (n && (!size || !ids || !rating || !mode || !seq))
    return set_err(e, MM_E_ARG, "null size, ids, rating, mode or seq with n = %u", n);
  CK(cudaSetDevice(e->device));
  const int rc = requeue_party(e, n, size, ids, rating, mode, enq_ts, seq, codes, n_requeued);
  free_img_scratch(e);
  return rc;
}

int mm_party_match(mm_engine* e, uint64_t now, const mm_widen_rule* rules, mm_lobby_hdr* lobbies, uint32_t lobby_cap,
                   uint64_t* member_ids, uint64_t member_cap, mm_party_stats* stats) {
  if (!e) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  auto& rep = e->ot.rep[MM_OFFTICK_PARTY_MATCH];  // void until this call returns MM_OK; its capture sets the lobby count
  rep.valid = false;
  rep.n_lob = 0;
  auto& ob = e->ob[MM_OFFTICK_PARTY_MATCH];  // zeros until a call that ran its plan returns MM_OK or MM_E_CAP
  ob.valid = ob.ran = false;
  if (!rules || !stats) return set_err(e, MM_E_ARG, "null rules or stats");
  std::memset(stats, 0, sizeof(*stats));
  if ((lobby_cap && !lobbies) || (member_cap && !member_ids))
    return set_err(e, MM_E_ARG, "null lobbies or member_ids with a non-zero capacity");
  CK(cudaSetDevice(e->device));
  const int rc = party_match(e, now, rules, lobbies, lobby_cap, member_ids, member_cap, stats);
  rep.valid = rc == MM_OK;
  ob.valid = ob.ran && (rc == MM_OK || rc == MM_E_CAP);
  return rc;
}

int mm_party_read(mm_engine* e, uint32_t party_cap, uint32_t member_cap, uint8_t* size, uint32_t* seq, uint32_t* enq_ts,
                  uint8_t* mode, uint8_t* group, int32_t* rating, uint64_t* member_ids, int32_t* member_rating,
                  uint32_t* n_parties, uint32_t* n_members) {
  if (!e || !n_parties || !n_members || (party_cap && (!size || !seq || !enq_ts || !mode || !group || !rating)) ||
      (member_cap && (!member_ids || !member_rating)))
    return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  return party_read(e, party_cap, member_cap, size, seq, enq_ts, mode, group, rating, member_ids, member_rating,
                    n_parties, n_members);
}

int mm_party_queue_stats(mm_engine* e, uint64_t now, mm_party_queue_stat* out, uint32_t cap, uint32_t* n_out) {
  if (!e) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!out || !n_out) return set_err(e, MM_E_ARG, "null out or n_out");
  *n_out = e->n_cut;
  int rc = pt_check(e);
  if (rc) return rc;
  if (cap < e->n_cut) return set_err(e, MM_E_CAP, "need cap >= %u", e->n_cut);
  CK(cudaSetDevice(e->device));
  return party_queue_stats(e, now, out);
}

int mm_party_locate(mm_engine* e, uint64_t now, const mm_widen_rule* rules, uint32_t n, const uint64_t* id,
                    mm_party_member_status* out) {
  if (!e) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!rules) return set_err(e, MM_E_ARG, "null rules");
  if (n && (!id || !out)) return set_err(e, MM_E_ARG, "null id or out array with n = %u", n);
  std::vector<WdRule> rule;
  bool any = false;
  int rc = pt_rules(e, rules, rule, any);
  if (rc) return rc;
  if (n == 0) return MM_OK;
  CK(cudaSetDevice(e->device));
  return party_locate(e, now, rule, any, n, id, out);
}

int mm_export_parties(mm_engine* e, const uint8_t* queues, void* buf, uint64_t cap, uint64_t* n_bytes) {
  if (!e || !n_bytes || (cap && !buf)) return MM_E_ARG;
  *n_bytes = 0;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  const int rc = export_parties(e, queues, buf, cap, n_bytes);
  free_img_scratch(e);
  return rc;
}

int mm_merge_parties(mm_engine* e, const void* buf, uint64_t n_bytes, uint32_t flags, uint8_t* code,
                     uint32_t* n_merged) {
  if (!e || !n_merged || (n_bytes && !buf)) return MM_E_ARG;
  *n_merged = 0;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  return merge_parties(e, static_cast<const uint8_t*>(buf), n_bytes, flags, code, n_merged);
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
  k_lookup<<<(n + 255) / 256, 256, 0, e->stream>>>(n, e->d_in_id, act_view(e), e->d_lookup);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, e->d_lookup, n, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return MM_OK;
}

int mm_locate(mm_engine* e, uint64_t now, uint32_t n, const uint64_t* id, mm_player_status* out) {
  if (!e) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  if (n && (!id || !out)) return set_err(e, MM_E_ARG, "null id or out array with n = %u", n);
  if (!e->use_active) return set_err(e, MM_E_STATE, "an MM_F_NO_DEDUPE engine has no active set to find ids in");
  if (e->stage_count) return staged_err(e);
  if (n == 0) return MM_OK;
  CK(cudaSetDevice(e->device));
  return locate(e, now, n, id, out);
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
  if ((rc = tick_commit(e, n, stats))) return rc;
  return balance_tick(e, stats);
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
  CK(e->d_qstat.reserve(bytes / 4));
  CK(cudaMemsetAsync(e->d_qstat, 0, bytes, e->stream));
  StatArgs a{};
  const Pool& p = e->pool[e->cur];
  a.sec[0] = StatSection{p.v.mode, p.v.ts, p.m, nullptr, (uint32_t)now};
  const Pool& q = e->pool[e->cur ^ 1];
  a.sec[1] = StatSection{q.v.mode, q.v.ts, q.m, e->d_left_bits, e->tick_now};
  a.n_segs = e->n_segs; a.part_cut = e->d_part_cut; a.out = e->d_qstat;
  const uint32_t n_max = std::max(p.n, e->match_valid ? e->match_n : 0u);
  k_queue_stats<kStatBlock><<<dim3(tile_ctas(e, n_max), e->match_valid ? 2 : 1), kStatBlock, 0, e->stream>>>(a);
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

int mm_match_quality(mm_engine* e, mm_queue_quality* per_queue, uint32_t cap, uint32_t* n_out,
                     mm_lobby_quality* per_lobby, uint32_t lobby_cap, uint32_t* n_lobbies) {
  if (!e || !per_queue || !n_out || !n_lobbies) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  const uint32_t n_lob = e->match_valid ? e->last.n_lobbies : 0u;
  *n_out = e->n_cut;
  *n_lobbies = n_lob;
  if (cap < e->n_cut) return set_err(e, MM_E_CAP, "need cap >= %u", e->n_cut);
  if (per_lobby && lobby_cap < n_lob) return set_err(e, MM_E_CAP, "need lobby_cap >= %u", n_lob);
  if (!e->match_valid) {  // void: no tick, a failed one, or a pool loaded since (mm_queue_stats' match section)
    *n_out = 0;
    return MM_OK;
  }
  CK(cudaSetDevice(e->device));
  return match_quality(e, per_queue, per_lobby, n_lob);
}

int mm_offtick_report(mm_engine* e, uint32_t source, mm_match_waits* waits, mm_queue_quality* quality, uint32_t cap,
                      uint32_t* n_out, mm_lobby_quality* per_lobby, uint32_t lobby_cap, uint32_t* n_lobbies) {
  if (!e || !n_out || !n_lobbies) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  if (source > MM_OFFTICK_WIDEN) return set_err(e, MM_E_ARG, "unknown source %u", source);
  const auto& r = e->ot.rep[source];
  const uint32_t n_cut = e->n_cut, G = e->cfg.n_groups, n_lob = r.valid ? r.n_lob : 0u;
  *n_out = n_cut;
  *n_lobbies = n_lob;
  if ((waits || quality) && cap < n_cut) return set_err(e, MM_E_CAP, "need cap >= %u", n_cut);
  if (per_lobby && lobby_cap < n_lob) return set_err(e, MM_E_CAP, "need lobby_cap >= %u", n_lob);
  if (!r.valid) {  // no call of the source yet, or its last one did not return MM_OK
    *n_out = 0;
    return MM_OK;
  }
  if (n_lob) {
    CK(cudaSetDevice(e->device));
    if (waits) CK(cudaMemcpyAsync(waits, r.waits, (size_t)n_cut * sizeof(mm_match_waits), cudaMemcpyDeviceToHost, e->stream));
    if (quality)
      CK(cudaMemcpyAsync(quality, r.quality, (size_t)n_cut * sizeof(mm_queue_quality), cudaMemcpyDeviceToHost, e->stream));
    if (per_lobby)
      CK(cudaMemcpyAsync(per_lobby, r.lob, (size_t)n_lob * sizeof(mm_lobby_quality), cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
  } else {  // a valid call without lobbies: zero records
    if (waits) std::memset(waits, 0, (size_t)n_cut * sizeof(mm_match_waits));
    if (quality) std::memset(quality, 0, (size_t)n_cut * sizeof(mm_queue_quality));
  }
  for (uint32_t c = 0; c < n_cut; ++c) {
    const mm_mode_desc& md = e->cfg.modes[c / G];
    if (waits) {
      waits[c].mode = (uint8_t)(c / G);
      waits[c].group = (uint8_t)(c % G);
      waits[c].n_lobbies = waits[c].n_matched / ((uint32_t)md.teams * md.team_size);  // whole lobbies of L members
    }
    if (quality) {
      quality[c].mode = (uint8_t)(c / G);
      quality[c].group = (uint8_t)(c % G);
    }
  }
  return MM_OK;
}

int mm_set_lobby_budget(mm_engine* e, const uint32_t* per_queue, const uint32_t* per_mode) {
  if (!e) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  // an array without a limit in it is kept as "no array": the tick then takes its unbudgeted path
  auto keep = [](std::vector<uint32_t>& v, const uint32_t* src, uint32_t n) {
    v.clear();
    if (src && std::any_of(src, src + n, [](uint32_t b) { return b != MM_BUDGET_UNLIMITED; })) v.assign(src, src + n);
  };
  keep(e->bud_queue, per_queue, e->n_cut);
  keep(e->bud_mode, per_mode, e->cfg.n_modes);
  e->bud_stale = true;
  return MM_OK;
}

int mm_lobby_budget_report(mm_engine* e, uint32_t* candidates, uint32_t* emitted, uint32_t cap, uint32_t* n_out) {
  if (!e || !n_out || (cap && (!candidates || !emitted))) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  const uint32_t n_cut = e->n_cut;
  *n_out = n_cut;
  if (cap < n_cut) return set_err(e, MM_E_CAP, "need cap >= %u", n_cut);
  if (e->stage_count) return staged_err(e);
  std::fill(candidates, candidates + n_cut, 0u);
  std::fill(emitted, emitted + n_cut, 0u);
  if (!e->report_valid) return MM_OK;
  CK(cudaSetDevice(e->device));
  // emitted: the partition table the tick wrote (a queue's lobbies are credited to the partitions they start in)
  std::vector<SegInfo> seg(e->n_segs);
  CK(cudaMemcpyAsync(seg.data(), e->d_seg, (size_t)e->n_segs * sizeof(SegInfo), cudaMemcpyDeviceToHost, e->stream));
  if (e->report_budgeted) CK(cudaMemcpyAsync(candidates, e->d_cand, (size_t)n_cut * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  for (uint32_t s = 0; s < e->n_segs; ++s) emitted[e->h_part_cut[s]] += seg[s].n_lobbies;
  if (!e->report_budgeted) std::copy(emitted, emitted + n_cut, candidates);
  return MM_OK;
}

int mm_set_offtick_budget(mm_engine* e, uint32_t source, const uint32_t* per_queue, const uint32_t* per_mode) {
  if (!e) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  if (source > MM_OFFTICK_WIDEN) return set_err(e, MM_E_ARG, "unknown source %u", source);
  // as mm_set_lobby_budget: an array without a limit in it is "no array", and the call then runs unbudgeted
  auto keep = [](std::vector<uint32_t>& v, const uint32_t* src, uint32_t n) {
    v.clear();
    if (src && std::any_of(src, src + n, [](uint32_t b) { return b != MM_BUDGET_UNLIMITED; })) v.assign(src, src + n);
  };
  keep(e->ob[source].queue, per_queue, e->n_cut);
  keep(e->ob[source].mode, per_mode, e->cfg.n_modes);
  return MM_OK;
}

int mm_offtick_budget_report(mm_engine* e, uint32_t source, uint32_t* candidates, uint32_t* emitted, uint32_t cap,
                             uint32_t* n_out) {
  if (!e || !n_out || (cap && (!candidates || !emitted))) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  if (source > MM_OFFTICK_WIDEN) return set_err(e, MM_E_ARG, "unknown source %u", source);
  const uint32_t n_cut = e->n_cut;
  *n_out = n_cut;
  if (cap < n_cut) return set_err(e, MM_E_CAP, "need cap >= %u", n_cut);
  if (e->stage_count) return staged_err(e);
  std::fill(candidates, candidates + n_cut, 0u);
  std::fill(emitted, emitted + n_cut, 0u);
  const auto& o = e->ob[source];
  if (!o.valid) return MM_OK;
  CK(cudaSetDevice(e->device));
  CK(cudaMemcpyAsync(emitted, o.tab, (size_t)n_cut * 4, cudaMemcpyDeviceToHost, e->stream));
  if (o.budgeted) CK(cudaMemcpyAsync(candidates, o.tab + n_cut, (size_t)n_cut * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  if (!o.budgeted) std::copy(emitted, emitted + n_cut, candidates);
  return MM_OK;
}

int mm_lobby_candidates(mm_engine* e, uint32_t* candidates, uint32_t cap, uint32_t* n_out) {
  if (!e || !n_out || (cap && !candidates)) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  const uint32_t n_cut = e->n_cut;
  *n_out = n_cut;
  if (cap < n_cut) return set_err(e, MM_E_CAP, "need cap >= %u", n_cut);
  if (e->stage_count) return staged_err(e);
  CK(cudaSetDevice(e->device));
  const uint32_t layout = tail_layout(e);
  CK(e->d_cand_dry.reserve(n_cut + (layout & 1u ? 0u : e->Kp + 1)));
  TailArgs t = tail_args(e);
  // count only: the tail writes the counts (and, for a key domain too large for shared memory, its parked matched
  // counts) into this call's own scratch; the tick's outputs and the compacted pool's layout are not touched
  t.cand = e->d_cand_dry; t.binlim = e->d_cand_dry + n_cut;
  t.bud_queue = t.bud_mode = nullptr;
  t.outbase = nullptr; t.seg = nullptr; t.ctr = nullptr; t.dst = PoolMeta{};
  k_lobby_candidates<<<1, kScanBlock, (size_t)tail_words(e->Kp, layout) * 4, e->stream>>>(t);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(candidates, e->d_cand_dry, (size_t)n_cut * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return MM_OK;
}

int mm_expire(mm_engine* e, uint64_t now, uint32_t max_wait, uint64_t* ids, uint32_t* seq, uint32_t cap,
              uint32_t* n_expired) {
  if (!e || !n_expired || (cap && !ids)) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  return expire(e, now, max_wait, ids, nullptr, seq, cap, n_expired);
}

int mm_expire_packed(mm_engine* e, uint64_t now, uint32_t max_wait, uint32_t* handles, uint32_t* seq, uint32_t cap,
                     uint32_t* n_expired) {
  if (!e || !n_expired || (cap && !handles)) return MM_E_ARG;
  if (!(e->cfg.flags & MM_F_DENSE_IDS)) return MM_E_STATE;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  return expire(e, now, max_wait, nullptr, handles, seq, cap, n_expired);
}

int mm_export(mm_engine* e, void* buf, uint64_t cap, uint64_t* n_bytes) {
  if (!e || !n_bytes || (cap && !buf)) return MM_E_ARG;
  *n_bytes = 0;
  std::lock_guard<std::mutex> lk(e->mu);
  if (e->pt.live) return parties_err(e);
  CK(cudaSetDevice(e->device));
  const int rc = export_image(e, buf, cap, n_bytes, nullptr);
  free_img_scratch(e);
  return rc;
}

int mm_export_queues(mm_engine* e, const uint8_t* queues, void* buf, uint64_t cap, uint64_t* n_bytes) {
  if (!e || !queues || !n_bytes || (cap && !buf)) return MM_E_ARG;
  *n_bytes = 0;
  std::lock_guard<std::mutex> lk(e->mu);
  if (e->pt.live) return parties_err(e);
  CK(cudaSetDevice(e->device));
  const int rc = export_image(e, buf, cap, n_bytes, queues);
  free_img_scratch(e);
  return rc;
}

int mm_merge(mm_engine* e, const void* buf, uint64_t n_bytes, uint32_t cap, uint32_t* rejected, uint32_t* n_rejected) {
  if (!e || !n_rejected || (n_bytes && !buf) || (cap && !rejected)) return MM_E_ARG;
  *n_rejected = 0;
  std::lock_guard<std::mutex> lk(e->mu);
  if (e->pt.live) return parties_err(e);
  CK(cudaSetDevice(e->device));
  const int rc = merge_image(e, static_cast<const uint8_t*>(buf), n_bytes, cap, rejected, n_rejected);
  free_img_scratch(e);
  return rc;
}

int mm_import(mm_engine* e, const void* buf, uint64_t n_bytes) {
  if (!e || (n_bytes && !buf)) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  const int rc = import_image(e, static_cast<const uint8_t*>(buf), n_bytes);
  free_img_scratch(e);
  return rc;
}

int mm_import_regroup(mm_engine* e, const void* buf, uint64_t n_bytes, uint32_t cap, uint32_t* rejected,
                      uint32_t* n_rejected) {
  if (!e || !n_rejected || (n_bytes && !buf) || (cap && !rejected)) return MM_E_ARG;
  *n_rejected = 0;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  const uint8_t* b = static_cast<const uint8_t*>(buf);
  const int rc = regroup_many(e, "mm_import_regroup", 1, &b, &n_bytes, nullptr, 0, cap, nullptr, rejected, n_rejected,
                              nullptr, nullptr);
  free_img_scratch(e);
  return rc;
}

int mm_import_regroup_many(mm_engine* e, uint32_t n_images, const void* const* bufs, const uint64_t* n_bytes,
                           const uint8_t* keep, uint32_t active_image, uint32_t cap, uint32_t* rej_image,
                           uint32_t* rej_index, uint32_t* n_rejected, uint32_t* n_elsewhere) {
  return mm_import_regroup_many_parties(e, n_images, bufs, n_bytes, keep, active_image, cap, rej_image, rej_index,
                                        n_rejected, n_elsewhere, nullptr);
}

int mm_import_regroup_many_parties(mm_engine* e, uint32_t n_images, const void* const* bufs, const uint64_t* n_bytes,
                                   const uint8_t* keep, uint32_t active_image, uint32_t cap, uint32_t* rej_image,
                                   uint32_t* rej_index, uint32_t* n_rejected, uint32_t* n_elsewhere,
                                   mm_recut_parties* parties) {
  if (!e || !n_rejected || !n_elsewhere || (n_images && (!bufs || !n_bytes)) || (cap && (!rej_image || !rej_index)))
    return MM_E_ARG;
  if (parties && (parties->reserved || (parties->cap && (!parties->rej_image || !parties->rej_index)))) return MM_E_ARG;
  *n_rejected = 0;
  *n_elsewhere = 0;
  for (uint32_t k = 0; k < n_images && k < kRcMaxImages; ++k)
    if (n_bytes[k] && !bufs[k]) return MM_E_ARG;
  if (parties && n_images && parties->n_bytes && !parties->bufs) return MM_E_ARG;
  for (uint32_t k = 0; parties && parties->n_bytes && k < n_images && k < kRcMaxImages; ++k)
    if (parties->n_bytes[k] && !parties->bufs[k]) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  CK(cudaSetDevice(e->device));
  std::vector<const uint8_t*> b(n_images <= kRcMaxImages ? n_images : 0);
  for (size_t k = 0; k < b.size(); ++k) b[k] = static_cast<const uint8_t*>(bufs[k]);
  const int rc = regroup_many(e, "mm_import_regroup_many", n_images, b.data(), n_bytes, keep, active_image, cap,
                              rej_image, rej_index, n_rejected, n_elsewhere, parties);
  free_img_scratch(e);
  return rc;
}

int mm_snapshot(mm_engine* e) {
  if (!e) return MM_E_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  if (e->pt.live) return parties_err(e);
  CK(cudaSetDevice(e->device));
  if (!e->snap.v.id) {
    int rc = alloc_pool(e, e->snap);
    if (rc) return rc;
  }
  int rc = copy_pool(e, e->snap, e->pool[e->cur]);
  if (rc) return rc;
  if (e->use_active) {  // the active set as it stands: ids queued, matched and not yet removed, tombstones
    CK(e->snap_tab.kv.reserve(table_bytes(e) / 8));
    CK(cudaMemcpyAsync(e->snap_tab.kv, e->tab[e->tcur].kv, table_bytes(e), cudaMemcpyDeviceToDevice, e->stream));
    e->snap_active = e->n_active;
    e->snap_tomb = e->n_tomb;
  }
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
  if (e->use_active) {  // into whichever table is current: a rehash since the snapshot may have switched it
    CK(cudaMemcpyAsync(e->tab[e->tcur].kv, e->snap_tab.kv, table_bytes(e), cudaMemcpyDeviceToDevice, e->stream));
    e->n_active = e->snap_active;
    e->n_tomb = e->snap_tomb;
  }
  e->seq_next = e->snap_seq;
  e->gen = next_gen(e);
  e->fresh = false;
  e->pt.n_rows = e->pt.n_mem = e->pt.live = 0;  // a snapshot never holds parties
  e->match_valid = false;  // the restored pool was not matched by the last tick
  if (e->use_active && p.n) {
    k_restamp<<<dim3(e->n_chunks, e->n_segs), 256, 0, e->stream>>>(p.v, p.m, act_view(e), e->gen, nullptr);
    CK(cudaGetLastError());
  }
  CK(cudaStreamSynchronize(e->stream));
  return MM_OK;
}

}  // extern "C"
