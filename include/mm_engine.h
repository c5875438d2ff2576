/*
 * mm_engine.h — C ABI of the H100 opponent-search engine (libmm_engine.so).
 *
 * This is the drop-in boundary for the *search stage* of
 * OpenMatchmaking/microservice-matchmaking.  Every entry point names the
 * reference interface it replaces (paths relative to the reference tree,
 * matchmaking/lib/...).  The reference is Elixir; the binding a maintainer adds
 * is a dirty NIF (c_src/mm_nif.c, shown in INTEGRATION.md) — this header is what
 * that NIF, the Python ctypes host mirror and the tests all bind.
 *
 * Conventions
 *   - plain C, no torch / CUDA types in signatures; pointers + sizes only.
 *   - return 0 (MM_OK) or a negative mm_status; nothing throws or aborts
 *     (mirrors the tagged-tuple convention of models/active_user.ex:46-66 and
 *     models/lobby_state.ex:95-103,113).
 *   - caller owns every in/out HOST buffer; the engine owns device memory and
 *     its pinned staging.  *_device variants take/return DEVICE pointers.
 *   - an mm_engine is single-writer: enqueue/remove/tick are serialised by an
 *     internal mutex; all calls block until their result is valid.
 *   - there is NO CPU fallback: without a usable CUDA device mm_create fails
 *     with MM_E_CUDA.
 */
#ifndef MM_ENGINE_H
#define MM_ENGINE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MM_ABI_VERSION 2u

#define MM_MAX_GROUPS 64u   /* rating groups (reference default: 7, config.exs:27-36) */
#define MM_MAX_MODES 8u     /* game modes ("1v1", "5v5", ...)                         */
#define MM_MODE_DEAD 0xFFu  /* mode byte of a player removed while still queued        */

typedef enum mm_status {
  MM_OK = 0,
  MM_E_ARG = -1,   /* bad argument / bad config                                    */
  MM_E_CUDA = -2,  /* CUDA runtime error or no device (see mm_last_error)          */
  MM_E_CAP = -3,   /* pool / active-set / output capacity exceeded                 */
  MM_E_NCCL = -4,  /* reserved: boundary exchange (windowed extension)             */
  MM_E_STATE = -5  /* call not valid in the current state (e.g. no snapshot)       */
} mm_status;

/* Feed order of the serialized search loop (SURVEY §8c).
 *   ARRIVAL — enqueue order: the reference's queue serialized as-is
 *             (search/worker.ex:352-358 handled one delivery at a time).
 *   RATING  — (mode, clamp(rating), enqueue order): the canonical order
 *             BASELINE.json's north_star names ("sort by (mode, rating),
 *             tie-break by enqueue order").                                        */
typedef enum mm_order_mode { MM_ORDER_ARRIVAL = 0, MM_ORDER_RATING = 1 } mm_order_mode;

/* mm_config.flags */
#define MM_F_NO_DEDUPE 1u /* skip the "already in the queue" check (middleware/worker.ex:65-70) */
#define MM_F_DENSE_IDS 2u /* player ids are dense host handles 0 .. active_capacity-1 (SURVEY §7.3: the host owns the
                             UUID <-> handle table): the active set is a direct-mapped array instead of a hash
                             table, and the packed entry points (mm_enqueue_packed / mm_tick_packed) apply.        */
#define MM_F_WIDE_PARTITIONS 4u /* keep every (mode, group) queue ONE pool partition however many ratings it spans
                             (default: groups wider than 255 ratings are stored as several partitions of <= 255
                             sort keys so that every tile takes the 8-bit ranking path).  Results are identical;
                             this keeps the list-ranking path reachable for tests and comparisons.              */

typedef struct mm_mode_desc {
  uint16_t teams;     /* T: number of teams ("1v1" -> 2, "5v5" -> 2)   */
  uint16_t team_size; /* S: players per team ("1v1" -> 1, "5v5" -> 5)  */
} mm_mode_desc;

/* Replaces: config :matchmaking, RatingGroups (config/config.exs:27-36),
 * @default_rating_group (generic/worker.ex:27) and the strategist's mode table
 * (not in the repo; SURVEY F1 — policy S0).                                        */
typedef struct mm_config {
  uint32_t abi_version; /* MM_ABI_VERSION */
  uint32_t n_groups;
  int32_t group_lo[MM_MAX_GROUPS]; /* inclusive, generic/worker.ex:50 */
  int32_t group_hi[MM_MAX_GROUPS]; /* inclusive                        */
  int32_t default_group;           /* index used when no range matches; -1 = reject
                                      (generic/worker.ex:27: div(len,2)+1, nil for len<=2) */
  uint32_t n_modes;
  mm_mode_desc modes[MM_MAX_MODES];
  uint32_t order_mode;      /* mm_order_mode */
  uint32_t capacity;        /* max players resident in the pool           */
  uint32_t active_capacity; /* max ids in the active set (0 = 2*capacity); MM_F_DENSE_IDS: handle range */
  int32_t device;           /* CUDA device ordinal                        */
  uint32_t flags;
} mm_config;

/* One emitted lobby.  Members are member_ids[first_member .. first_member+n_members)
 * in join order; team t = members [t*S, (t+1)*S)  (policy S0: first team with room).
 * Replaces the payload built at search/worker.ex:315-319.                           */
typedef struct mm_lobby_hdr {
  uint32_t first_member;
  uint16_t n_members;
  uint8_t mode;
  uint8_t group;
} mm_lobby_hdr;

typedef struct mm_tick_stats {
  uint32_t pool_before;   /* players resident when the tick started (incl. dead)      */
  uint32_t n_lobbies;     /* lobbies emitted                                           */
  uint32_t n_matched;     /* players placed in emitted lobbies                         */
  uint32_t n_residual;    /* players left queued (< L per (mode, group))               */
  uint32_t n_dead;        /* removed-while-queued players dropped by this tick         */
  uint32_t n_launches;    /* kernels launched by this tick                             */
  float device_us;        /* CUDA-event time of the whole tick on the engine's stream  */
  float place_us;         /* CUDA-event time of the dominant kernel: placement + pool  */
                          /* compaction (fused tick: until the last row has compacted) */
  float hist_us;          /* ... of the histogram kernel                               */
  float scan_us;          /* ... of the column-scan kernel                             */
  float epilogue_us;      /* ... of the epilogue kernel: lobby headers (fused tick:    */
                          /* from the end of placement until the last CTA exits)       */
  uint32_t reserved;
} mm_tick_stats;

typedef struct mm_engine mm_engine;

/* ---- lifecycle ---------------------------------------------------------------
 * Replaces: Search.Worker.init/1 (search/worker.ex:220-237) state creation plus
 * ActiveUser.init_store/0 (models/active_user.ex:14-24) and
 * LobbyState.init_store/0 (models/lobby_state.ex:15-29).                           */
int mm_create(const mm_config* cfg, mm_engine** out);
int mm_destroy(mm_engine* e);

/* Fills cfg with the reference defaults: the 7 rating groups of
 * config/config.exs:27-36, default group index 4 ("diamond"), modes
 * {"1v1": 2x1, "5v5": 2x5}, ORDER_ARRIVAL.                                          */
void mm_config_default(mm_config* cfg);

/* rating -> group index.  Replaces Generic.Worker.find_rating_group_by_rating/1
 * (generic/worker.ex:46-53): first {from,to} in list order with from<=r<=to, else
 * default_group (may be -1).  Pure host function.                                   */
int mm_group_of(const mm_config* cfg, int32_t rating);

/* ---- active set + pool ingest -------------------------------------------------
 * mm_enqueue replaces, per player: Middleware dedupe + ActiveUser.add_user
 * (middleware/worker.ex:65-70, models/active_user.ex:46-55) and the publish of the
 * request to the group queue (generic/worker.ex:55-69).  Players are appended in
 * call order = enqueue order.  accepted[i]: 1 = queued, 0 = "already in the queue"
 * (also for a repeat inside the same batch: first occurrence wins), 2 = invalid
 * mode / id / rating without a default group, 3 = pool full (the LAST players of the
 * batch that do not fit).  A batch the active set cannot hold at all (more than
 * active_capacity ids resident) is refused as a whole with MM_E_CAP — nothing is
 * enqueued, the caller nacks / retries after mm_remove.  enq_ts may be NULL (stored 0).
 * Every offered player (accepted or not) consumes one enqueue sequence number.     */
int mm_enqueue(mm_engine* e, uint32_t n, const uint64_t* id, const int32_t* rating,
               const uint8_t* mode, const uint32_t* enq_ts, uint8_t* accepted);
/* Same, all five pointers are DEVICE pointers (accepted may be NULL).              */
int mm_enqueue_device(mm_engine* e, uint32_t n, const uint64_t* id, const int32_t* rating,
                      const uint8_t* mode, const uint32_t* enq_ts, uint8_t* accepted,
                      uint32_t* n_accepted);

/* Packed ingest for MM_F_DENSE_IDS engines — 6 bytes per player over PCIe instead of 17:
 * handle = the host's dense slot of the player (what the device stores as the id),
 * key = mode << 13 | rating with rating in 0 .. 8191 (other ratings: use mm_enqueue).
 * Same semantics and accepted codes as mm_enqueue.                                  */
int mm_enqueue_packed(mm_engine* e, uint32_t n, const uint32_t* handle, const uint16_t* key,
                      const uint32_t* enq_ts, uint8_t* accepted);

/* Split form of mm_enqueue_packed for a software-pipelined host loop (PCIe is full duplex and the copy engines run
 * beside the kernels): _begin starts the host-to-device copy of a batch into one of two staging slots and returns at
 * once; _end (oldest staged batch first) waits for that copy and runs the ingest.  Between the two the caller may run
 * mm_tick* / mm_enqueue_rejects of the PREVIOUS batch, so a step's upload hides behind the previous step's tick and
 * result copies.  The host arrays must stay valid until the matching _end returns.  MM_E_STATE: both slots staged
 * (_begin) / nothing staged (_end).  Replaces nothing in the reference: AMQP prefetch (search/worker.ex:36) is the
 * reference's own way of having the next deliveries in flight while one is consumed.                                */
int mm_enqueue_packed_begin(mm_engine* e, uint32_t n, const uint32_t* handle, const uint16_t* key,
                            const uint32_t* enq_ts);
int mm_enqueue_packed_end(mm_engine* e, uint8_t* accepted, uint32_t* n_accepted);

/* The ack / nack list of the LAST mm_enqueue* batch without a per-player transfer: the batch indices whose code is
 * not 1 (unordered) and their codes — pass accepted = NULL to mm_enqueue* and ack everything else
 * (search/worker.ex:323 acks per delivery).  MM_E_CAP if there are more than cap (n_rejects says how many).   */
int mm_enqueue_rejects(mm_engine* e, uint32_t cap, uint32_t* index, uint8_t* code, uint32_t* n_rejects);

/* Replaces ActiveUser.remove_user/1 (models/active_user.ex:57-66; callers
 * game-lobby/worker.ex:80,96).  A removed id that is still queued is dropped by the
 * next tick exactly as remove_inactive_players/1 filters it
 * (search/worker.ex:267-280).  Unknown ids are ignored, like Mnesia.delete.         */
int mm_remove(mm_engine* e, uint32_t n, const uint64_t* id, uint32_t* n_removed);
int mm_remove_packed(mm_engine* e, uint32_t n, const uint32_t* handle, uint32_t* n_removed);

/* EXTENSION (cross-group boundary pass, DESIGN.md §6): queued players that were matched outside this engine's tick
 * leave the pool but STAY in the active set — like the members of an emitted lobby, who are "in the queue" until
 * the lobby stage removes them (game-lobby/worker.ex:80).  Ids that are not queued are ignored.               */
int mm_take(mm_engine* e, uint32_t n, const uint64_t* id, uint32_t* n_taken);

/* Replaces ActiveUser.in_queue?/1 (models/active_user.ex:33-44), batched.          */
int mm_in_queue(mm_engine* e, uint32_t n, const uint64_t* id, uint8_t* out);

int mm_pool_size(mm_engine* e, uint32_t* n_players);
int mm_active_size(mm_engine* e, uint32_t* n_ids);

/* ---- the search tick ----------------------------------------------------------
 * Replaces the body of Search.Worker.consume/5 between decode and ack
 * (search/worker.ex:295-321) for EVERY queued player at once: LobbyState.get_state
 * (models/lobby_state.ex:61-104), the strategist RPC (search/worker.ex:296-306,
 * policy S0), remove_inactive_players (:267-280), prepare_game_lobby (:250-261) and
 * save_new_state (:282-289; the partial lobby = the residual players, who simply
 * stay resident in enqueue order).
 *
 * mm_tick copies results to host buffers: lobbies[0..n_lobbies) ordered by
 * (mode, group, emission order inside the (mode, group) partition) and
 * member_ids[0..n_matched).  emit_seq (may be NULL) receives, per lobby, the enqueue
 * sequence number (mod 2^32; the i-th player offered to the k-th mm_enqueue call has
 * number (players offered by earlier calls) + i) of the member whose arrival
 * completed it: sorting lobbies by emit_seq reproduces the serialized reference's
 * emission order in ORDER_ARRIVAL.
 * MM_E_CAP if lobby_cap / member_cap are too small (nothing is consumed).
 * now: the caller's clock, in the unit of the enq_ts stamps; it changes no result and is what mm_queue_stats
 * measures the matched players' waits against.                                        */
int mm_tick(mm_engine* e, uint64_t now, mm_lobby_hdr* lobbies, uint32_t lobby_cap,
            uint64_t* member_ids, uint64_t member_cap, uint32_t* emit_seq,
            mm_tick_stats* stats);

/* Same tick, members returned as 32-bit host handles (MM_F_DENSE_IDS engines): 4 bytes per
 * matched player over PCIe instead of 8.                                            */
int mm_tick_packed(mm_engine* e, uint64_t now, mm_lobby_hdr* lobbies, uint32_t lobby_cap,
                   uint32_t* member_handles, uint64_t member_cap, uint32_t* emit_seq,
                   mm_tick_stats* stats);

/* With mm_set_option("async_results", 1) mm_tick returns as soon as the tick is done and its host copies are
 * queued: the caller's buffers are valid only after mm_results_wait, or once the next mm_tick* call has returned (it
 * waits for them — a packed tick after its own kernels, which write a second set of device result buffers; the other
 * entry points before they start).  Give consecutive ticks different host arrays if tick k is read while tick k+1
 * runs.  mm_enqueue* / mm_remove / mm_in_queue may run meanwhile — the next batch's host-to-device transfer overlaps
 * the previous tick's device-to-host transfer.  What replaces it: nothing (the reference publishes lobby by lobby,
 * search/worker.ex:250-261); it is the batched hand-off of SURVEY §8f-1.  No-op when nothing is pending.            */
int mm_results_wait(mm_engine* e);

/* Same tick, results stay in HBM; pointers valid until the next tick/destroy.      */
int mm_tick_device(mm_engine* e, uint64_t now, mm_tick_stats* stats);
int mm_results_device(mm_engine* e, const mm_lobby_hdr** d_lobbies,
                      const uint64_t** d_member_ids);

/* Copy the queued players (global enqueue order, dead ones skipped) to host buffers; any
 * pointer may be NULL.  Test/diagnostic aid and the body of Search.Worker.status/0's
 * queue-depth report (search/worker.ex:326-334).                                    */
int mm_pool_read(mm_engine* e, uint32_t cap, uint64_t* id, int32_t* rating, uint8_t* mode,
                 uint8_t* team_size, uint32_t* enq_ts, uint32_t* n_out);

/* ---- per-queue status ----------------------------------------------------------
 * Replaces Search.Worker.status/0's queue depth (search/worker.ex:115-117,326-334: AMQP.Queue.status of the group's
 * queue) for the players the engine holds, plus what the reference stamps and never reads (created_at,
 * models/active_user.ex:47): how long they have waited.
 *
 * WAIT of a slot: w = (int32_t)((uint32_t)now - enq_ts), negative values clamped to 0.  The caller stamps enq_ts
 * (mm_enqueue*) and passes now (mm_tick*, mm_queue_stats) in one clock and unit; waits wrap modulo 2^32 and a stamp
 * "in the future" reads as 0.
 * BUCKET of a wait: w itself for w < 8; else, with e = 31 - clz(w) (3 <= e <= 30) and s = (w >> (e - 2)) & 3,
 * bucket 8 + 4 (e - 3) + s, which holds the waits [(4 + s) << (e - 2), (5 + s) << (e - 2)).  Four sub-buckets per
 * octave, at most 25 % relative width; bucket 119 ends at 2^31.  Buckets 0..7 = {0}..{7}, 8 = [8, 10), 11 = [14, 16),
 * 12 = [16, 20), 119 = [7 * 2^28, 2^31).                                                                        */
#define MM_WAIT_BUCKETS 120u

typedef struct mm_queue_stat {
  uint8_t mode, group;
  uint16_t reserved;
  /* the resident pool at `now` */
  uint32_t n_waiting;  /* live queued players of this (mode, group)                                     */
  uint32_t n_removed;  /* entries removed (mm_remove / mm_take) while queued; the next tick drops them    */
  uint32_t max_wait;   /* longest wait among the n_waiting players (0 if none)                          */
  uint32_t wait_hist[MM_WAIT_BUCKETS];
  /* the players the LAST tick matched, at that tick's `now` (all zero before the first tick, after a tick that
     failed, e.g. with MM_E_CAP, and after mm_restore) */
  uint32_t n_lobbies, n_matched, max_match_wait;
  uint32_t match_wait_hist[MM_WAIT_BUCKETS];
} mm_queue_stat; /* 988 bytes */

/* One record per (mode, group) queue, empty ones included, in mode * n_groups + group order: *n_out = n_modes *
 * n_groups.  MM_E_CAP (and *n_out = the count needed) if cap is smaller.  One pass over the resident mode and
 * enqueue-stamp columns on the device (and, for the match section, over the pool buffer the last tick read, which no
 * call writes until the next tick); only the records cross PCIe.  Runs on the engine's stream and leaves pending
 * async_results copies alone.                                                                                     */
int mm_queue_stats(mm_engine* e, uint64_t now, mm_queue_stat* out, uint32_t cap, uint32_t* n_out);

/* Device-side snapshot / restore of pool + active set (ram_copies analogue,
 * models/active_user.ex:20; used by bench.py to replay one pool K times).          */
int mm_snapshot(mm_engine* e);
int mm_restore(mm_engine* e);

/* Use an externally owned CUDA stream (cudaStream_t passed as void*).              */
int mm_set_stream(mm_engine* e, void* cuda_stream);

/* Options (name -> value); unknown name or bad value = MM_E_ARG.
 *   "tick_impl"     1 = whole tick in one cooperative launch (default when it fits), 0 = four launches
 *   "rank_impl"     3 = per tile: ballot counting sort staged in shared memory for partitions of <= 255 bins, hashed
 *                   lists otherwise (default); 2 = hashed lists for every tile (cross-check of the two rankings)
 *   "max_spread"    EXTENSION beyond the reference (strategist policy S1, SURVEY §8f-3): a lobby may span at most
 *                   `value` rating points — greedy walk over the rating-sorted partition, a player whose window cannot
 *                   be filled stays queued (oracle: orc_run_windowed).  < 0 (default) = reference behaviour (S0).
 *                   MM_ORDER_RATING only (MM_E_ARG otherwise).  Takes effect from the next tick.
 *   "async_results" 1 = mm_tick does not wait for its device-to-host copies (see mm_results_wait); default 0   */
int mm_set_option(mm_engine* e, const char* name, int64_t value);

const char* mm_strerror(int status);
const char* mm_last_error(mm_engine* e); /* last CUDA error text, "" if none */
uint32_t mm_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* MM_ENGINE_H */
