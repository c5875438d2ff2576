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
 * in join order; team t = members [t*S, (t+1)*S)  (policy S0: first team with room; with
 * mm_set_option("team_balance") the members of a balanced mode are reordered into the
 * two teams with the least rating difference, and team t is still [t*S, (t+1)*S)).
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
                          /* (with "team_balance": plus its balance pass)              */
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
 * call order = enqueue order.  accepted[i]: 1 = queued, 0 = "already in the queue",
 * 2 = invalid mode / id / rating without a default group, 3 = pool full (the LAST
 * players of the batch that do not fit).  A repeat inside the batch follows its first
 * occurrence: 0 if that was queued, 3 if it did not fit.  A removed or taken player
 * holds its pool slot until the next tick.  A batch the active set cannot hold at all
 * (more than active_capacity ids resident) is refused as a whole with MM_E_CAP —
 * nothing is enqueued and no sequence number is consumed; the caller nacks / retries
 * after mm_remove.  enq_ts may be NULL (stored 0).  Every offered player of an
 * accepted batch (queued or not) consumes one enqueue sequence number.             */
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
 * (search/worker.ex:323 acks per delivery).  MM_E_CAP if there are more than cap (n_rejects says how many).
 * mm_in_queue, mm_remove, mm_take and a refused batch in between do not change the list.                      */
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

/* EXTENSION (requeue): players of a lobby that did not start (a member declined the ready check, no game server
 * could be allocated: game-lobby/worker.ex:89-103) go back into their queue at their enqueue position, as the
 * reference keeps the remaining members of a partial lobby in place when one leaves (search/worker.ex:312-321).
 * Entry i carries what the player had when it was queued: id (a handle on MM_F_DENSE_IDS engines, as mm_enqueue
 * takes it), rating, mode, enq_ts (may be NULL: 0) and seq, its enqueue sequence number (the numbering of emit_seq;
 * an image's section 5).  The engine no longer has these once a tick has compacted the pool, so the caller keeps
 * them.  Entries are in AGE ORDER: (seq[i] - seq_next) mod 2^32 strictly ascending (the order of mm_pool_read).
 * codes[i] (may be NULL):
 *   1  requeued: the id was in the active set and is not a live queued player (matched by any earlier tick, taken by
 *      mm_take or mm_band_match).  It goes back into the partition its rating and mode map to, at the position its
 *      seq gives among that partition's live players, with its rating, enq_ts and seq: its wait and the search
 *      timeout count from its first enqueue.  mm_in_queue reads 1; mm_active_size does not change.
 *   0  already a live queued player: nothing changes.
 *   4  not in the active set (removed, expired, moved out, never queued): not requeued, the player left.
 * *n_requeued = the entries with code 1.  n = 0 does nothing.  Pending async_results copies, the last tick's match
 * section of mm_queue_stats, the snapshot and the mm_enqueue_rejects list are left alone.
 * Refusals, all decided before anything changes (mm_last_error names the cause):
 *   MM_E_ARG   a mode >= n_modes, a rating without a group, an id out of range, entries not in strict age order, a seq
 *              equal to seq_next, a seq equal to that of a live player of the partition a code-1 entry goes to, an id
 *              given twice;
 *   MM_E_STATE an MM_F_NO_DEDUPE engine (no active set tells matched from gone), a staged packed batch;
 *   MM_E_CAP   the pool does not hold the result.  The call writes every partition that receives a player (a TOUCHED
 *              partition) anew on fresh chunks and leaves its old chunks to the next tick, so with U = the slots in use
 *              (mm_pool_size) minus the touched partitions' dead slots plus the requeued players, and H = the slots of
 *              the chunks (2048 slots each) left behind by this and earlier requeues since the last tick (the touched
 *              partitions' old chunks: ceil(slots / 2048) each), the call needs U + H <= capacity.  Until the next
 *              tick, enqueue and mm_merge count H as slots in use.
 * Afterwards mm_pool_size = U.  Cost: the touched partitions' live players, read and written once.
 *
 * EQUIVALENCE.  Take mm_export of the engine just before the call, insert the code-1 entries into sections 2-6 in their
 * partition at their sequence position, remove their ids from section 7 and keep seq_next: every later call sequence
 * gives the same results on the engine as on a fresh engine that mm_import'ed that image.  What may differ is what
 * differs after mm_import (dead slots are not carried): mm_pool_size, the next tick's pool_before and n_dead,
 * mm_queue_stats' n_removed, and when a pool near capacity answers "full" (here H counts too).                 */
int mm_requeue(mm_engine* e, uint32_t n, const uint64_t* id, const int32_t* rating, const uint8_t* mode,
               const uint32_t* enq_ts, const uint32_t* seq, uint8_t* codes, uint32_t* n_requeued);
/* The enqueue sequence number the next offered player will get.                                                   */
int mm_seq_next(mm_engine* e, uint32_t* seq_next);

/* EXTENSION (cross-group boundary pass on the device, DESIGN.md §6): the band gather and the band walk of
 * shard.boundary_pass without reading the pool to the host.  Both calls need what shard.check_bands needs: W >= 0,
 * MM_ORDER_RATING, contiguous ascending groups, each at least 2W wide (else MM_E_ARG); MM_E_STATE with a staged
 * packed batch or on an MM_F_NO_DEDUPE engine.  Every refusal is decided before anything changes and sets
 * mm_last_error.  A player whose rating lies outside every group (a default-group fallback) is never a candidate.
 *
 * mm_band_candidates: the upper side of the boundary group-1 | group (1 <= group < n_groups, else MM_E_ARG): the live
 * queued players of group g with rating in (hi_{g-1}, hi_{g-1} + W], sorted by (mode, rating, enqueue order) — what a
 * rank sends to the owner of group g-1.  MM_E_CAP (and *n_out = the count) if cap is smaller; cap = 0 is a dry run.
 * Reads only the key column of the partitions that hold band keys; nothing changes.                              */
int mm_band_candidates(mm_engine* e, int32_t W, uint32_t group, uint64_t* ids, int32_t* rating, uint8_t* mode,
                       uint32_t cap, uint32_t* n_out);

typedef struct mm_band_stats {
  uint32_t n_lobbies, n_matched; /* boundary lobbies and their members                         */
  uint32_t n_taken;              /* local players taken out of this pool                       */
  uint32_t n_upper_taken;        /* upper-side candidates given by the caller and consumed     */
  float device_us;               /* CUDA-event time of the call's device work                  */
  uint32_t reserved[3];
} mm_band_stats; /* 32 bytes */

/* mm_band_match: the bands of the boundaries g|g+1 for g_first <= g <= g_last < n_groups - 1, every mode.  Band
 * (g, m): the live queued players of group g with rating in (hi_g - W, hi_g] and those of group g+1 with rating in
 * (hi_g, hi_g + W], matched by the S1 windowed walk (orc_run_windowed) in (rating, enqueue order) — the tick's walk
 * (mm_scan.cuh), run on the band's per-rating counts.  The upper side of boundary g_last|g_last+1 comes from the
 * caller's columns when upper_remote != 0 (another rank's mm_band_candidates; n_upper may be 0), otherwise from this
 * engine.  lobbies: ordered by (g, mode, emission), group = the LOWER group g, first_member into member_ids, members
 * in join order.  Local matched players leave the pool in the same call exactly as mm_take takes them (they stay in
 * the active set; the last tick's match section of mm_queue_stats is unaffected); upper_taken[i] = 1 for every
 * caller-given candidate a lobby consumed (the caller hands those ids back to the owner's mm_take).
 * MM_E_ARG also for: a boundary range out of bounds; upper columns without upper_remote, on an MM_F_DENSE_IDS engine
 * (another engine's handles are not ids here), not sorted by (mode, rating), with a rating outside
 * (hi_{g_last}, hi_{g_last} + W] or a mode >= n_modes (checked on the device).  MM_E_CAP if lobby_cap or member_cap
 * is too small: stats then holds the counts and nothing is taken (zero capacities: a dry run).  Only candidates,
 * headers, members and upper_taken cross PCIe.                                                                  */
int mm_band_match(mm_engine* e, int32_t W, uint32_t g_first, uint32_t g_last, uint32_t upper_remote,
                  const uint64_t* up_ids, const int32_t* up_rating, const uint8_t* up_mode, uint32_t n_upper,
                  mm_lobby_hdr* lobbies, uint32_t lobby_cap, uint64_t* member_ids, uint64_t member_cap,
                  uint8_t* upper_taken, mm_band_stats* stats);

/* EXTENSION (backfill, DESIGN.md §4): a running lobby that lost members (a player left during the loading screen, a
 * member declined and the rest should stay together) asks for k players from its queue instead of being disbanded —
 * the reference saves a partial lobby in its shrunken state and fills it with the next players of its queue
 * (search/worker.ex:312-321, models/lobby_state.ex).                                                              */
typedef struct mm_backfill_req {
  uint8_t mode, group; /* the (mode, group) queue to take from                                                  */
  uint16_t reserved;   /* 0                                                                                     */
  uint32_t count;      /* open slots: players wanted                                                            */
  int32_t target;      /* rating the slots should be filled around (MM_ORDER_RATING)                            */
  int32_t window;      /* max |rating - target| in clamped ratings; < 0 = no limit                              */
} mm_backfill_req;     /* 16 bytes */

/* mm_backfill: requests are served one at a time, in index order; request j is served against the live queued players
 * of its queue that no earlier request of the same call took.
 *   MM_ORDER_RATING  with c(x) = x clamped to [rmin - 1, rmax + 1] (the tick's key clamp), request j ranks the
 *                    candidates by (|c(rating) - c(target)|, c(rating), enqueue order) — at equal distance the lower
 *                    rating first, inside one rating the older player first — and takes the first
 *                    min(count, #{candidates with |c(rating) - c(target)| <= window}) of them (no limit when window < 0).
 *                    A request on the default group sees everything the tick files there, out-of-range players at their
 *                    clamped ratings; with overlapping groups a group's ratings need not be contiguous: distances are in
 *                    ratings, not in key indices.
 *   MM_ORDER_ARRIVAL request j takes the count oldest players of its queue; target is ignored, window must be < 0.
 * A request may be filled only in part: n_taken[j] says how many players it got (a caller that wants all or nothing
 * hands a short fill back to mm_requeue).  member_ids holds request 0's players, then request 1's, ..., each in the
 * rank order above (handles on MM_F_DENSE_IDS engines); *n_total = the sum of n_taken.  Taken players leave the pool
 * exactly as mm_take takes them and stay in the active set as matched players until mm_remove, so mm_requeue puts them
 * back (code 1).  The last tick's match section of mm_queue_stats, the lobby budget, pending async_results copies, the
 * snapshot and the mm_enqueue_rejects list are left alone.  n = 0 does nothing.
 * Refusals, all decided before anything changes (mm_last_error names the cause and the request index):
 *   MM_E_ARG   a mode >= n_modes, a group >= n_groups, reserved != 0, window >= 0 on an MM_ORDER_ARRIVAL engine;
 *   MM_E_STATE a staged packed batch, an MM_F_NO_DEDUPE engine (no active set holds matched players);
 *   MM_E_CAP   member_cap < *n_total.  n_taken and *n_total are still written: member_cap = 0 is a dry run.
 * Cost: the plan runs on the per-bin totals; the gather reads the key column of the partitions holding a taken player,
 * and places up to the tile of each partition's last taken player.  Only the requests, n_taken and member_ids cross
 * PCIe.
 *
 * EQUIVALENCE.  The call leaves the engine in the state mm_take of the returned ids would leave it in: every later
 * call sequence gives the same results on both engines.                                                           */
int mm_backfill(mm_engine* e, uint32_t n, const mm_backfill_req* req, uint32_t* n_taken, uint64_t* member_ids,
                uint64_t member_cap, uint32_t* n_total);

/* EXTENSION (widening search, DESIGN.md §6): the longer a player has waited, the wider the range of ratings it
 * accepts.  The tick's max_spread (policy S1) is one window for the whole pool; mm_widen forms lobbies around the
 * players who have waited longest, each in a window of its own that grows with its wait.  A separate call: the tick is
 * unchanged. */
#define MM_WIDEN_OFF 0xFFFFFFFFu
/* one rule per (mode, group) queue, in mm_queue_stats record order (mode * n_groups + group) */
typedef struct mm_widen_rule {
  uint32_t min_wait;  /* anchors: live queued players whose WAIT >= min_wait; MM_WIDEN_OFF = queue not touched     */
  uint32_t step;      /* > 0                                                                                       */
  int32_t w0;         /* >= 0: window (rating points, either side) of a player at exactly min_wait                 */
  int32_t inc;        /* >= 0: added per whole `step` of wait past min_wait                                        */
  int32_t w_max;      /* >= w0                                                                                     */
  uint32_t reserved;  /* 0                                                                                         */
} mm_widen_rule;      /* 24 bytes */

typedef struct mm_widen_stats {
  uint32_t n_anchors;   /* anchors considered                                              */
  uint32_t n_lobbies, n_matched;
  uint32_t n_absorbed;  /* anchors an earlier lobby of the call had already taken          */
  float device_us;      /* CUDA-event time of the call's device work                       */
  uint32_t reserved[3];
} mm_widen_stats;       /* 32 bytes */

/* mm_widen: WAIT is the definition of mm_queue_stats, c(x) the tick's key clamp (x clamped to [rmin - 1, rmax + 1], as
 * in mm_backfill) and AGE ORDER (seq - seq_next) mod 2^32 ascending.  Every queue q whose rule is not MM_WIDEN_OFF is
 * served on its own, with L = teams x team_size of its mode:
 *   U = the live queued players of q (across all partitions of a wide group)
 *   A = the players of U with WAIT >= min_wait, in age order
 *   for a in A:
 *     if a is not in U: a is ABSORBED (an earlier lobby took it); next
 *     w = min(w_max, w0 + floor((WAIT(a) - min_wait) / step) * inc)                (64-bit)
 *     C = the players x of U with |c(r_x) - c(r_a)| <= w, ranked by (|c(r_x) - c(r_a)|, c(r_x), age)
 *     if |C| < L: a stays queued; next                                             (all or nothing)
 *     the first L of C form a lobby and leave U
 * Only the anchor's window counts: widening favours the player who waited, and a lobby spans at most 2w.  Members of
 * a lobby are in (c(rating), age) order, so team t is members [tS, (t+1)S) (the tick's S0 member order in rating
 * order; "team_balance" then re-splits the lobbies of a balanced mode).  lobbies are ordered by (mode, group, emission
 * order within the queue), group = the queue's group,
 * first_member into member_ids (handles on MM_F_DENSE_IDS engines).  A default group holds its out-of-range players
 * at their clamped ratings; with overlapping groups distances are in ratings, not in key indices.  Widening never
 * crosses a group boundary.
 * THE ANCHOR IS IN ITS OWN LOBBY whenever stamps never decrease with age (an older anchor of the same rating that
 * failed would make this one fail too), which SearchPool's ingest and requeue keep.  Otherwise (e.g. after mm_merge) an
 * anchor with at least L older untaken players of its rating forms their lobby and stays queued itself.
 * Taken players leave the pool exactly as mm_take takes them: their slots are dead until the next tick and count in
 * n_removed; they stay in the active set as matched players (mm_locate state 2, mm_requeue code 1, mm_remove forgets
 * them).  The last tick's results, the match section of mm_queue_stats, mm_match_quality, the lobby budget and its
 * report, the snapshot, the mm_enqueue_rejects list, pending async_results copies and the options are left alone;
 * widen lobbies are outside the tick's lobby budget and inside mm_widen's own (mm_set_offtick_budget below).
 * Refusals, all decided before anything changes (mm_last_error names the cause):
 *   MM_E_ARG   a null e, rules or stats; on a queue that is not MM_WIDEN_OFF: step 0, w0 < 0, inc < 0, w_max < w0 or
 *              reserved != 0; an MM_ORDER_ARRIVAL engine (windows need rating order);
 *   MM_E_STATE an MM_F_NO_DEDUPE engine (no active set holds matched players), a staged packed batch;
 *   MM_E_CAP   lobby_cap or member_cap too small: stats holds the counts and nothing is taken (zero capacities: a dry
 *              run).
 * Cost: one pass over the mode and stamp columns of the served queues' partitions, a rank per anchor, one warp per
 * queue walking the per-bin totals sequentially over its anchors (a queue with very many anchors dominates the call),
 * and the backfill gather over the partitions holding a taken player.  Only the rules, headers, members and stats
 * cross PCIe.
 *
 * EQUIVALENCE.  The call leaves the engine in the state mm_take of the returned ids would leave it in: every later
 * call sequence gives the same results on both engines.                                                           */
int mm_widen(mm_engine* e, uint64_t now, const mm_widen_rule* rules, mm_lobby_hdr* lobbies, uint32_t lobby_cap,
             uint64_t* member_ids, uint64_t member_cap, mm_widen_stats* stats);

/* EXTENSION (parties, DESIGN.md §4): players who queue together are matched into one lobby and one team.  Parties live
 * in a table beside the pool that the tick never reads; mm_party_match, called before the tick, forms their lobbies, so
 * parties get the first pick of the solos.  mm_set_option("party_capacity", P) sets how many party members the table
 * holds (default 0: every party call is refused with MM_E_STATE; MM_E_ARG below the members queued now).
 *
 * mm_enqueue_party: party j's members are the next size[j] entries of ids / rating (handles on MM_F_DENSE_IDS
 * engines).  Its rating R = floor(sum(rating) / size) (64-bit sum, floor toward minus infinity), its group
 * mm_group_of(R) (with the default-group fallback).  Every offered party of an accepted batch consumes one enqueue
 * sequence number (the numbering of emit_seq: parties and solos share age order).  accepted[j] (may be null):
 *   2  invalid: mode >= n_modes, size < 2 or > the mode's team_size, an invalid id, an id twice in the party, R
 *      without a group;
 *   0  otherwise, if a member was in the active set before the call or is a member of an earlier party of the batch
 *      (accepted or not);
 *   3  otherwise, if the party does not fit the table: the last parties that do not fit;
 *   1  queued.
 * A queued member is in the active set (mm_in_queue 1, mm_active_size counts it) but not in the pool (mm_pool_size,
 * mm_queue_stats, the tick, mm_take, mm_widen, mm_backfill and the boundary pass do not see it).  mm_remove of any
 * member dissolves the whole party (every member leaves the active set and counts in n_removed); mm_expire expires
 * whole parties whose WAIT >= max_wait, listing every member with the party's seq (cap and the dry run count members;
 * the party members follow the solos); mm_locate reports state 3; mm_requeue gives a queued member code 0.
 * mm_export, mm_export_queues, mm_merge and mm_snapshot are refused with MM_E_STATE while a party is queued (images
 * do not carry parties); mm_restore empties the table.  Parties travel in a party image of their own
 * (mm_export_parties / mm_merge_parties below): release them, take the image, merge them back.
 * Refusals, decided before anything changes: MM_E_ARG null pointers with n > 0, an MM_ORDER_ARRIVAL engine;
 * MM_E_STATE no party capacity, an MM_F_NO_DEDUPE engine, a staged packed batch; MM_E_CAP a batch the active set
 * cannot hold at all.                                                                                                */
int mm_enqueue_party(mm_engine* e, uint32_t n_parties, const uint8_t* size, const uint64_t* ids, const int32_t* rating,
                     const uint8_t* mode, const uint32_t* enq_ts, uint8_t* accepted);

typedef struct mm_party_stats {
  uint32_t n_anchors;   /* anchors considered                                  */
  uint32_t n_lobbies, n_matched;
  uint32_t n_parties;   /* parties placed into lobbies                         */
  uint32_t n_absorbed;  /* anchors an earlier lobby of the call had placed     */
  float device_us;      /* CUDA-event time of the call's device work           */
  uint64_t sum_imbalance;  /* "party_balance": summed imbalance of the emitted lobbies of masked modes (0: off) */
} mm_party_stats;       /* 32 bytes */

/* mm_party_match: one mm_widen_rule per (mode, group) queue in mm_queue_stats order (MM_WIDEN_OFF: the queue is not
 * served); WAIT, c() and age order as in mm_widen; L = T x S of the queue's mode.  Every served queue q on its own:
 *   U = the live queued solos of q;  P = the queued parties of q
 *   A = the parties of P with WAIT >= min_wait, in age order
 *   for a in A:
 *     if an earlier lobby of the call placed a: a is ABSORBED; next
 *     w = min(w_max, w0 + floor((WAIT(a) - min_wait) / step) * inc)                                   (64-bit)
 *     room[t] = S for every team; a goes to team 0
 *     Q = the unplaced parties b != a of P with |c(R_b) - c(R_a)| <= w, by (|c(R_b) - c(R_a)|, c(R_b), age)
 *     for b in Q: b goes to the lowest team t with room[t] >= size(b); if there is none, b is skipped
 *     open = sum(room)
 *     C = the players x of U with |c(r_x) - c(R_a)| <= w, by (|c(r_x) - c(R_a)|, c(r_x), age)
 *     if |C| < open: a stays queued and nothing is placed; next                                  (all or nothing)
 *     a lobby is formed: its parties leave P, the first `open` of C leave U
 * Members are team-major (team t = members [tS, (t+1)S)): a team's parties in placement order, each with its members
 * in enqueue order, then the solos, which fill the open slots of team 0, then team 1, ... in C's order.  Lobbies are
 * ordered by (mode, group, emission within the queue), group = the queue's group.  Solos taken leave the pool exactly
 * as mm_take takes them; matched party members stay in the active set as matched players (mm_locate state 2,
 * mm_requeue code 1: back as a solo, with its own rating and the party's seq).  The members of a party share that one
 * seq, so mm_requeue takes at most one of them per call (two are not in strict age order: MM_E_ARG) and refuses a
 * member whose partition holds a co-member requeued earlier (the seq of a live player there: MM_E_ARG); a member whose
 * rating maps to another partition is requeued.  Only R needs a group, so a member whose own rating has none cannot be
 * requeued (MM_E_ARG).  To put a whole party back at its age position, use mm_requeue_party.  team_balance does not
 * split party lobbies; the last tick's results, mm_match_quality, the tick's lobby budget and pending async_results
 * copies are left alone (party lobbies are inside mm_party_match's own budget, mm_set_offtick_budget below).  With
 * mm_set_option("party_balance") a lobby of a masked mode is split into its most even teams with every party kept
 * whole, so its teams no longer read "a team's parties, then its solos": EQUIVALENCE, the call leaves
 * the engine exactly as the same call without the option would, and its member order is the party_balance rule
 * applied to that call's lobbies (each party's members stay contiguous and in enqueue order).
 * Refusals, all decided before anything changes (mm_last_error names the cause): MM_E_ARG the rule checks of mm_widen,
 * a served mode of more than 256 teams, an MM_ORDER_ARRIVAL engine; MM_E_STATE no party capacity, an MM_F_NO_DEDUPE
 * engine, a staged packed batch; MM_E_CAP lobby_cap or member_cap too small (stats holds the counts and nothing is
 * taken: zero capacities make a dry run).                                                                          */
int mm_party_match(mm_engine* e, uint64_t now, const mm_widen_rule* rules, mm_lobby_hdr* lobbies, uint32_t lobby_cap,
                   uint64_t* member_ids, uint64_t member_cap, mm_party_stats* stats);

/* mm_party_read: the queued parties in age order (a test and diagnostic aid, like mm_pool_read): size, seq, enq_ts,
 * mode, group and R per party, member ids and ratings in party order.  MM_E_CAP (with the counts) if party_cap or
 * member_cap is too small.                                                                                          */
int mm_party_read(mm_engine* e, uint32_t party_cap, uint32_t member_cap, uint8_t* size, uint32_t* seq, uint32_t* enq_ts,
                  uint8_t* mode, uint8_t* group, int32_t* rating, uint64_t* member_ids, int32_t* member_rating,
                  uint32_t* n_parties, uint32_t* n_members);

/* Party hand-over: the queued parties in a PARTY IMAGE, so that checkpoint / resume, regroup and queue moves carry them.
 * The image calls above keep refusing while a party is queued; a host layer releases the parties (mm_export_parties),
 * uses the image call, and merges the parties where they belong (mm_merge_parties).
 *
 * PARTY IMAGE LAYOUT (little-endian).  mm_image_header with magic MM_PARTY_IMAGE_MAGIC, n_parts = P parties, n_players
 * = M members, n_active = 0, the writer's seq_next and config; then six sections, each starting at the next multiple
 * of 8 bytes after the previous one ends, padding zero, total_bytes the end of the last rounded up to 8:
 *   1. size    u8[P]     2. seq   u32[P]     3. enq_ts  u32[P]     4. mode  u8[P]
 *   5. id      W * M     member ids (u64), or 32-bit handles on MM_F_DENSE_IDS engines
 *   6. rating  i32[M]
 * Parties in age order, members in party order.  R, group and bin are not stored: the loading engine derives them
 * under its own config (so a party image follows mm_import_regroup).
 *
 * mm_export_parties: `queues` = n_modes * n_groups bytes in mm_queue_stats order (non-zero: selected), NULL = every
 * queue.  buf = NULL with cap = 0 -> *n_bytes = the size, nothing changes; cap too small -> MM_E_CAP and *n_bytes,
 * nothing changes.  A call that writes the image RELEASES the selected parties in the same call, as mm_export_queues
 * does for solos: their members leave the active set (mm_in_queue 0) and their rows are gone.  Matched party members
 * are not in the image; they stay in this engine's active set, like matched solos.  Refusals, before anything
 * changes: MM_E_ARG an MM_ORDER_ARRIVAL engine; MM_E_STATE no party capacity, an MM_F_NO_DEDUPE engine, a staged
 * packed batch.  The image-sized device scratch is freed before the call returns.
 *
 * mm_merge_parties: without flags, exactly one mm_enqueue_party batch of the image's columns (the same codes, sequence
 * numbers seq_next + index, R / group / bin under THIS engine's config), except that it is all or nothing on room: if
 * any party would get code 3 the call returns MM_E_CAP and changes nothing (exact: decided after the codes 0 and 2).
 * code[j] (may be null) per image party: 1 merged; 0 a member is in the active set, or in an earlier party of the
 * image; 2 no place here (mode >= n_modes, a size above the mode's team_size, an id twice in the party, an R without a
 * group).  *n_merged counts the 1s.
 * flags = MM_PARTY_KEEP_SEQ (resume): every party keeps its image seq and seq_next does not move; allowed only when no
 * party is queued here and seq_next equals the image's (right after mm_import / mm_import_regroup of the image taken
 * at the same stop, or after the release on the source), else MM_E_STATE.
 * Refusals, before anything changes: MM_E_ARG bad magic, version or lengths, another id width, an image of an
 * MM_F_NO_DEDUPE engine, a size below 2, sizes that do not add up to M, an id or handle out of range, seq not strictly
 * increasing in age order ((seq - seq_next) mod 2^32) or equal to seq_next, unknown flags; MM_E_STATE as
 * mm_export_parties, and the MM_PARTY_KEEP_SEQ condition; MM_E_CAP the table or a hashed active set cannot take the
 * merged parties.
 *
 * EQUIVALENCE.  mm_export_parties leaves the engine as mm_remove of one member of each exported party would.  After
 * mm_import (or mm_import_regroup) of an mm_export image and mm_merge_parties(MM_PARTY_KEEP_SEQ) of the party image
 * taken at the same stop, every later call sequence gives what the source gives, on every output mm_import's
 * EQUIVALENCE names and on the party calls.                                                                          */
#define MM_PARTY_IMAGE_MAGIC 0x5954504Du /* "MPTY" */
#define MM_PARTY_KEEP_SEQ 1u
int mm_export_parties(mm_engine* e, const uint8_t* queues, void* buf, uint64_t cap, uint64_t* n_bytes);
int mm_merge_parties(mm_engine* e, const void* buf, uint64_t n_bytes, uint32_t flags, uint8_t* code,
                     uint32_t* n_merged);

/* mm_requeue_party: the parties of a party lobby that did not start (a declined ready check, no free game server) go
 * back into the party table as parties, at the position their enqueue sequence numbers give them, as mm_requeue does for
 * solos.  Arguments as mm_enqueue_party: party j's members are the next size[j] entries of ids / rating (handles on
 * MM_F_DENSE_IDS engines), plus what the party had when it was queued: enq_ts (may be NULL: 0) and seq.  R =
 * floor(sum / size) and its group mm_group_of(R), as at enqueue; a caller may pass only the members still willing,
 * which makes a smaller party with R from those members.  Parties are in AGE ORDER: (seq[j] - seq_next) mod 2^32
 * strictly ascending.  codes[j] (may be NULL), in this order:
 *   0  a member is queued (a live solo, or a member of a queued party): nothing changes for this party;
 *   4  otherwise, a member is not in the active set (removed, expired, moved out, never queued): not requeued;
 *   1  otherwise (every member active and matched: by a tick, mm_party_match, mm_widen, mm_backfill, mm_band_match,
 *      mm_take or the matched section of an image load): the party gets a row among the queued parties at its age
 *      position, with its seq, enq_ts, mode, R, group and its members in the order given.  mm_in_queue reads 1,
 *      mm_locate reports state 3 with the wait counted from enq_ts; mm_active_size and seq_next do not change; the next
 *      mm_party_match treats the row like any other queued party.
 * *n_requeued (may be NULL) = the code-1 parties.  n = 0 does nothing.  The engine trusts the columns, as mm_requeue
 * does.  The solo pool, the last tick's results, mm_match_quality, the match section of mm_queue_stats, the lobby
 * budget, the snapshot, the mm_enqueue_rejects list and pending async_results copies are left alone.  The call inserts
 * no key into a hashed active set.  Cost: one pass over the party table plus the call's members.
 * Refusals, all decided before anything changes (mm_last_error names the cause):
 *   MM_E_ARG   an MM_ORDER_ARRIVAL engine; null pointers with n > 0; a mode >= n_modes; a size < 2 or above the mode's
 *              team_size; an id out of range; an id given twice anywhere in the call; an R without a group; parties not
 *              in strict age order; a seq equal to seq_next; a code-1 party whose seq is that of a queued party;
 *   MM_E_STATE no party capacity, an MM_F_NO_DEDUPE engine, a staged packed batch;
 *   MM_E_CAP   the code-1 parties' members exceed party_capacity minus the party members queued now (exact: a table
 *              with exactly enough room takes them).
 *
 * EQUIVALENCE.  Take mm_export_parties(NULL) and then mm_export of the engine just before the call; insert the code-1
 * parties into the party image at their sequence position and remove their member ids from section 7 of the engine
 * image.  A fresh engine that mm_import's the engine image and then mm_merge_parties(MM_PARTY_KEEP_SEQ) the party image
 * gives the same results as this engine for every later call sequence, except what mm_import itself changes (dead
 * slots, the next tick's pool_before and n_dead, mm_queue_stats' n_removed).                                        */
int mm_requeue_party(mm_engine* e, uint32_t n_parties, const uint8_t* size, const uint64_t* ids, const int32_t* rating,
                     const uint8_t* mode, const uint32_t* enq_ts, const uint32_t* seq, uint8_t* codes,
                     uint32_t* n_requeued);

/* mm_backfill_party: mm_backfill with teams and parties.  A running lobby that lost members (a premade that left during
 * loading, a player who declined) gets its open team slots filled with whole queued parties of its queue first, then
 * with the nearest solos, each party kept on one team.  Requests are mm_backfill_req, as for mm_backfill; `room` holds
 * their open slots, flattened: request j owns the next T_j entries (T_j = teams of its mode), entry t the open slots of
 * team t (0 <= room <= team_size), and count must be the sum of its entries (room carries no lengths of its own).
 * DEFINITION.  c() is the tick's key clamp and age order (seq - seq_next) mod 2^32 ascending, as in mm_widen.  Requests
 * are served one at a time in index order, each against the live solos U and the queued parties P of its (mode, group)
 * queue that no earlier request of the call took:
 *   room[t] as given
 *   Q = the parties b of P with |c(R_b) - c(target)| <= window (no limit when window < 0),
 *       by (|c(R_b) - c(target)|, c(R_b), age)
 *   for b in Q: b goes to the lowest team t with room[t] >= size(b); if there is none, b is skipped
 *   C = the solos x of U with |c(r_x) - c(target)| <= window, by (|c(r_x) - c(target)|, c(r_x), age)
 *   for t = 0 .. T-1: the next room[t] players of C (as many as are left) fill team t
 * filled (parallel to room) gets the members each team received, n_taken[j] the sum of request j's filled entries and
 * *n_total the sum of n_taken.  member_ids holds request 0's members, then request 1's, ...; inside a request team-major
 * (team 0's members, then team 1's), inside a team its parties in placement order, each with its members in party
 * order, then its solos in C's order (handles on MM_F_DENSE_IDS engines).  A request may be filled in part, as in
 * mm_backfill: a caller that wants all or nothing hands a short fill back with mm_requeue (solos) and mm_requeue_party
 * (parties).  When no party of the queue lies inside the window, the member list is mm_backfill's with count =
 * sum(room) and the same target and window.  n = 0 does nothing.
 * Effects: taken solos leave the pool exactly as mm_take takes them; a placed party's row is gone and its members are
 * matched players (mm_locate state 2, mm_requeue and mm_requeue_party code 1).  The last tick's results,
 * mm_match_quality, the match section of mm_queue_stats, both mm_offtick_report sources, the lobby budget, the
 * snapshot, the mm_enqueue_rejects list, pending async_results copies and the options are left alone.  No balance pass
 * runs (team_balance and party_balance do not apply): the caller owns the running lobby's teams, as with mm_backfill.
 * Refusals, all decided before anything changes (mm_last_error names the cause and the request index):
 *   MM_E_ARG   null pointers with n > 0; a mode >= n_modes, a group >= n_groups, reserved != 0; a room entry above the
 *              mode's team_size; a count that is not the sum of its room entries; a mode of more than 256 teams; an
 *              MM_ORDER_ARRIVAL engine (party windows are rating distances, as for every party call);
 *   MM_E_STATE no party capacity, an MM_F_NO_DEDUPE engine, a staged packed batch;
 *   MM_E_CAP   member_cap < *n_total.  filled, n_taken and *n_total are still written: member_cap = 0 is a dry run.
 * Cost: the party table's compaction and (bin, age) sort (as mm_party_match), one warp per queue with requests walking
 * the party rows and the per-bin totals sequentially over its requests, and mm_backfill's gather over the partitions
 * holding a taken solo.  Only the requests, room, filled, n_taken and member_ids cross PCIe.
 *
 * EQUIVALENCE.  Take mm_export_parties(NULL) and then mm_export of the engine just before the call; delete the placed
 * parties from the party image, delete the taken solos from sections 2-6 of the engine image and from their partition
 * counts, and add every taken id (solos and party members alike) to section 7.  A fresh engine with the same
 * party_capacity that mm_import's that image and then mm_merge_parties(MM_PARTY_KEEP_SEQ) the party image gives the same
 * results as this engine for every later call sequence, except what mm_import itself changes (dead slots, the next
 * tick's pool_before and n_dead, mm_queue_stats' n_removed).                                                        */
int mm_backfill_party(mm_engine* e, uint32_t n, const mm_backfill_req* req, const uint16_t* room, uint16_t* filled,
                      uint32_t* n_taken, uint64_t* member_ids, uint64_t member_cap, uint32_t* n_total);

/* Replaces ActiveUser.in_queue?/1 (models/active_user.ex:33-44), batched.          */
int mm_in_queue(mm_engine* e, uint32_t n, const uint64_t* id, uint8_t* out);

/* EXTENSION (search status): where one player's search stands — the per-player counterpart of mm_queue_stats, for a
 * client that polls its search and an operator who asks why a player is not matched.  The reference answers only
 * ActiveUser.in_queue?/1 (models/active_user.ex:33-44), which mm_in_queue covers.                                 */
#define MM_LOCATE_STAYS 0xFFFFFFFFu
typedef struct mm_player_status {
  uint8_t state;        /* 0 not in the active set, 1 queued (live), 2 in the active set but not queued, 3 queued in a
                           party (its own rating; the party's mode, group, enq_ts, seq and wait; ahead = depth = 0,
                           lobby = MM_LOCATE_STAYS)                                                                   */
  uint8_t mode, group;  /* its (mode, group) queue; a default-group fallback reports the default group                */
  uint8_t reserved;     /* 0                                                                                          */
  int32_t rating;       /* as enqueued                                                                                */
  uint32_t enq_ts, seq; /* its stamp and enqueue sequence number (the numbering of emit_seq)                          */
  uint32_t wait;        /* WAIT at `now`, the definition of mm_queue_stats                                            */
  uint32_t ahead;       /* live players of its queue that the tick feeds before it                                    */
  uint32_t depth;       /* live players of its queue (= that queue's n_waiting in mm_queue_stats)                     */
  uint32_t lobby;       /* next tick: ordinal of its lobby among that queue's emitted lobbies; MM_LOCATE_STAYS        */
  uint16_t member;      /* next tick: index in the lobby (team = member / team_size); 0xFFFF if it stays              */
  uint16_t reserved2;   /* 0                                                                                          */
} mm_player_status;     /* 36 bytes */

/* mm_locate: out[i] describes id[i] (a handle on MM_F_DENSE_IDS engines, as mm_in_queue takes it).
 *   state 1  the active-set entry points at a live slot of the current pool generation that holds this id (the test
 *            of mm_remove): a queued player.
 *   state 2  the id is in the active set but is not a live queued player: matched by a tick, or taken by mm_take,
 *            mm_band_match or mm_backfill, and not yet removed (mm_requeue's code 1).
 *   state 0  every id mm_in_queue answers 0 for (removed, expired, moved out, never queued, a handle out of range).
 *   States 0 and 2 leave every other field 0, except lobby = MM_LOCATE_STAYS and member = 0xFFFF.  A repeated id gets
 *   the same record each time.
 * FEED ORDER of a queue: MM_ORDER_ARRIVAL enqueue order; MM_ORDER_RATING (c(rating), enqueue order) with c the tick's
 * key clamp to [rmin - 1, rmax + 1].  Enqueue order is age order, (seq - seq_next) mod 2^32 ascending; requeued,
 * merged and regrouped players sit where those calls put them.  ahead = the live players of the queue before the
 * player in this order (0 <= ahead < depth); a wide group stored as several partitions is one queue.
 * NEXT-TICK PREDICTION.  If the next call that changes the engine is an mm_tick* of any form (any `now`) and neither
 * the options nor the lobby budget change in between, that tick puts the player at member index `member` of the
 * `lobby`-th lobby it emits from the player's queue, counting from 0 in header order; MM_LOCATE_STAYS: the tick leaves
 * the player queued.  This holds under S0, S1 (max_spread), the per-queue and per-mode lobby budget and "team_balance"
 * (member is then the player's index in the balanced lobby).  Under S0
 * without a budget it reduces to lobby = ahead / L when ahead < floor(depth / L) * L.
 * No side effects: the pool, the active set, the snapshot, the mm_enqueue_rejects list, the last tick's results and
 * the match section of mm_queue_stats, mm_lobby_budget_report and pending async_results copies are left alone.  n = 0
 * does nothing.
 * Refusals, all decided before anything runs (mm_last_error names the cause):
 *   MM_E_ARG   null pointers with n > 0;
 *   MM_E_STATE an MM_F_NO_DEDUPE engine (no active set maps an id to its slot), a staged packed batch.
 * Cost: one warp per id.  A probe of the active set, then the player's rank in its bin: with resident chunk histograms
 * (every partition of <= 255 sort keys) one 4-byte read per earlier chunk of its partition plus at most 4 KB of its own
 * chunk's bin column; without them (MM_F_WIDE_PARTITIONS, or more than 512 partitions) the bin column of the partition
 * up to the player (2 B per slot).  Per call, a one-CTA dry run of the tick's lobby cut on the resident bin totals and
 * a reverse chunk map; scratch of 3 (Kp + 2) + 2 n_cut + n_modes + (chunks) words and 44 B per id.  Only the ids and the
 * records cross PCIe.                                                                                              */
int mm_locate(mm_engine* e, uint64_t now, uint32_t n, const uint64_t* id, mm_player_status* out);

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
  uint32_t n_removed;  /* entries removed (mm_remove / mm_take / mm_expire) while queued; the next tick drops them */
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

/* EXTENSION (party search status): the status pair of mm_queue_stats and mm_locate for queued parties, answered on the
 * device without copying the party table to the host.
 *
 * mm_party_queue_stats: the waiting section of mm_queue_stats for the queued parties.  A party's queue is its (mode,
 * group), the group that of R as at enqueue (the default-group fallback included); its WAIT is mm_queue_stats' WAIT of
 * the party's enq_ts (the wait mm_expire and mm_party_match use).  One record per (mode, group) queue, empty ones
 * included, in mode * n_groups + group order: *n_out = n_modes * n_groups, MM_E_CAP (with that count) if cap is
 * smaller.  Only queued parties count: rows of matched, dissolved, expired, released or requeued-away parties that
 * are still in the table count nowhere.  Read-only: the table is not compacted.  Refusals, decided before anything
 * runs: MM_E_ARG null pointers, an MM_ORDER_ARRIVAL engine; MM_E_STATE no party capacity, an MM_F_NO_DEDUPE engine, a
 * staged packed batch.  Cost: one pass over the table's rows on the device (per-queue records in shared memory when
 * n_modes * n_groups records fit it, else global atomics); only the records cross PCIe.                           */
#define MM_PARTY_SIZE_BUCKETS 16u
typedef struct mm_party_queue_stat {
  uint8_t mode, group;
  uint16_t reserved;                          /* 0                                                                */
  uint32_t n_parties;                         /* queued parties of this (mode, group) queue                       */
  uint32_t n_members;                         /* their members                                                    */
  uint32_t max_wait;                          /* longest party WAIT (0 if none)                                   */
  uint32_t wait_hist[MM_WAIT_BUCKETS];        /* one count per party, in the BUCKETS of mm_queue_stats            */
  uint32_t size_hist[MM_PARTY_SIZE_BUCKETS];  /* [k] parties of size k for 2 <= k <= 14, [15] size >= 15; [0], [1] = 0 */
} mm_party_queue_stat;                        /* 560 bytes */

int mm_party_queue_stats(mm_engine* e, uint64_t now, mm_party_queue_stat* out, uint32_t cap, uint32_t* n_out);

typedef struct mm_party_member_status {
  uint8_t state;         /* mm_locate's states: 0 not active, 1 queued solo, 2 matched, 3 queued in a party.  Only state
                            3 fills the fields below; otherwise they are 0, window = -1, lobby = MM_LOCATE_STAYS and
                            member = 0xFFFF                                                                           */
  uint8_t mode, group;   /* its party's queue                                                                        */
  uint8_t size;          /* members of its party                                                                     */
  uint8_t index;         /* its place in the party (party order, as mm_party_read lists it)                          */
  uint8_t anchor;        /* 1: the queue's rule is not MM_WIDEN_OFF and WAIT >= min_wait                             */
  uint16_t reserved;     /* 0                                                                                        */
  int32_t rating;        /* its own, as enqueued                                                                     */
  int32_t party_rating;  /* R                                                                                        */
  uint32_t enq_ts, seq, wait;  /* the party's stamp, sequence number and WAIT at now                                 */
  int32_t window;        /* the anchor window w of mm_party_match at now; -1 when anchor = 0                         */
  uint32_t ahead;        /* queued parties of its queue older than its party (age order)                             */
  uint32_t depth;        /* queued parties of its queue (= that queue's n_parties in mm_party_queue_stats)           */
  uint32_t lobby;        /* ordinal among its queue's lobbies of the next mm_party_match(now, rules); MM_LOCATE_STAYS */
  uint16_t member;       /* its index in that lobby (team = member / team_size); 0xFFFF if it stays                  */
  uint16_t reserved2;    /* 0                                                                                        */
} mm_party_member_status; /* 48 bytes */

/* mm_party_locate: out[i] describes id[i] (a handle on MM_F_DENSE_IDS engines); a repeated id gets the same record each
 * time.  rules: the mm_party_match layout and checks (one rule per queue, MM_WIDEN_OFF = not served).
 * NEXT-CALL PREDICTION.  If the next call that changes the engine is mm_party_match with the same `now` and `rules`,
 * and neither the options nor the off-tick budget change in between, that call puts the member at index `member` of
 * the `lobby`-th lobby it emits from the member's queue, counting from 0 in header order; MM_LOCATE_STAYS: its party
 * stays queued.  This holds under S0 whatever the anchor and absorbed-anchor sequence, all-or-nothing failures,
 * MM_WIDEN_OFF queues, the off-tick budget of MM_OFFTICK_PARTY_MATCH (a lobby of ordinal >= the queue's allowance
 * stays) and "party_balance" (member is then the index in the balanced lobby).  A dry run of mm_party_match (MM_E_CAP)
 * changes nothing, so it keeps the prediction.
 * No side effects: the pool, the party table as mm_party_read shows it, the active set, seq_next, the snapshot, the
 * mm_enqueue_rejects list, the last tick's results, mm_queue_stats, mm_match_quality, mm_lobby_budget_report, both
 * mm_offtick_report and both mm_offtick_budget_report sources, pending async_results copies and the options are left
 * alone.  The table may be compacted, as mm_party_match compacts it (invisible).  n = 0 does nothing after the
 * refusals.
 * Refusals, all decided before anything runs (mm_last_error names the cause): MM_E_ARG null pointers with n > 0, null
 * rules, the rule checks of mm_party_match (a served mode of more than 256 teams included), an MM_ORDER_ARRIVAL engine;
 * MM_E_STATE as mm_party_queue_stats.
 * Cost: mm_party_match's compaction, sort and unbudgeted plan (about one plan), one pass that ranks every row among its
 * queue's rows, under "party_balance" the balance pass on member-slot tags, and one warp per id.  Only the ids and the
 * records cross PCIe.                                                                                              */
int mm_party_locate(mm_engine* e, uint64_t now, const mm_widen_rule* rules, uint32_t n, const uint64_t* id,
                    mm_party_member_status* out);

/* ---- match quality -------------------------------------------------------------
 * EXTENSION (measurement): how even the last tick's lobbies are, the other half of the wait / quality trade-off that
 * mm_queue_stats reports the wait half of.  max_spread, a widening window schedule, the lobby budget and a new
 * rating-group table all move it; the tick itself returns only ids, and the ratings stay on the device.
 *
 * DEFINITION.  c(r) = min(max(r, rmin - 1), rmax + 1), rmin / rmax over all groups: the tick's key clamp (the c of
 * mm_backfill and mm_locate).  The rating of a player is the one the pool holds for it (what mm_pool_read returns).
 * Per lobby: take lobby h of the last completed tick, in the tick's header order; its mode has T teams of S players
 * (L = T S), its members are x_0 .. x_{L-1} in member order and r_i = c(rating(x_i)).  min_rating = min r_i,
 * max_rating = max r_i, SPREAD = max_rating - min_rating, rating_sum = sum r_i (64-bit), team sums
 * s_t = sum of r_i over i in [t S, (t + 1) S), IMBALANCE = max_t s_t - min_t s_t (0 when T = 1), saturated at
 * 2^32 - 1.  Per (mode, group) queue, over that queue's lobbies of the last tick: n_lobbies, the largest spread and
 * imbalance, their sums (64-bit, for means) and their histograms in the BUCKETS of mm_queue_stats applied to rating
 * points (a value of 2^31 or more counts in bucket 119).
 *
 * WHICH TICK: the last completed tick of any form — mm_tick, mm_tick_packed or mm_tick_device, fused or split
 * (tick_impl), with or without async_results and emit_seq, under S0 or S1 and any lobby budget.  per_lobby[h]
 * describes lobbies[h] of that tick; per_queue holds one record per queue, empty ones included, in the order of
 * mm_queue_stats (mode * n_groups + group).  The lobbies of mm_band_match and the players of mm_backfill are outside
 * the tick and not covered.  After a tick with "team_balance" (mm_set_option) the imbalance of a balanced lobby is
 * that of the teams it was emitted with.
 * VOID exactly when the match section of mm_queue_stats is (before the first tick, after a tick that failed, after
 * mm_restore and after the import loads): *n_out = 0 and *n_lobbies = 0, nothing is written.
 * READ-ONLY: no other call changes the report until the next tick, and the call changes nothing — not the pool, the
 * active set, the last tick's results, the snapshot, the reject list or pending async_results copies.
 * REFUSALS, decided before anything runs: MM_E_ARG for a null e, per_queue, n_out or n_lobbies; MM_E_CAP when
 * cap < n_modes * n_groups (*n_out = the records needed) or when per_lobby is not NULL and lobby_cap is below the
 * tick's lobby count (*n_lobbies = the count needed); nothing is written then.  per_lobby = NULL skips the per-lobby
 * output.
 * COST: one pass over the 2-byte sort-key column and the last tick's left bits of the pool it read (MM_ORDER_RATING;
 * the lobby values then come from per-key prefix sums), or over the mode and rating columns (MM_ORDER_ARRIVAL), plus
 * per-lobby work; only the records cross PCIe.  Device memory, allocated by the first call and kept: 24 bytes per
 * lobby the pool could hold (capacity / smallest L + 1), 12 bytes per sort key, 992 bytes per queue, 4 bytes per
 * chunk, and on MM_ORDER_ARRIVAL engines 8 more bytes per such lobby and 4 bytes per player of capacity.        */
typedef struct mm_lobby_quality {
  int32_t min_rating, max_rating; /* c(rating) of the lowest and highest member                    */
  int64_t rating_sum;             /* sum of the members' c(rating)                                  */
  uint32_t imbalance;             /* max - min team rating sum (0 for one team), saturated          */
  uint32_t reserved;              /* 0                                                              */
} mm_lobby_quality;               /* 24 bytes */

typedef struct mm_queue_quality {
  uint8_t mode, group;
  uint16_t reserved;
  uint32_t n_lobbies, max_spread, max_imbalance;
  uint64_t sum_spread, sum_imbalance;
  uint32_t spread_hist[MM_WAIT_BUCKETS];
  uint32_t imbalance_hist[MM_WAIT_BUCKETS];
} mm_queue_quality;               /* 992 bytes */

int mm_match_quality(mm_engine* e, mm_queue_quality* per_queue, uint32_t cap, uint32_t* n_out,
                     mm_lobby_quality* per_lobby, uint32_t lobby_cap, uint32_t* n_lobbies);

/* ---- off-tick match report -------------------------------------------------------
 * EXTENSION (measurement): the match section of mm_queue_stats and the mm_match_quality report for the lobbies formed
 * OUTSIDE the tick, by mm_party_match and mm_widen.  Widening matches exactly the players who waited longest, so the
 * tail of the queue -> match wait and the spread that widening trades for it show here and not in the tick's reports.
 *
 * WHICH CALL: the last call of `source` on this engine (MM_OFFTICK_PARTY_MATCH: mm_party_match, MM_OFFTICK_WIDEN:
 * mm_widen).  VOID before the first such call and after one that returned anything but MM_OK (a refusal, an MM_E_CAP
 * dry run): *n_out = 0 and *n_lobbies = 0, nothing is written.  A call that returned MM_OK without lobbies (no queue
 * served, no live party, no anchor filled a lobby) gives a valid, empty report: n_modes * n_groups zero records.
 * Nothing else changes a source's report: not ticks of any form, the other source, enqueue, remove, expire, requeue
 * (solo and party), backfill, the band pass, options, the lobby budget, snapshot / restore or export / merge.  Engines
 * loaded by mm_import* are fresh, so their reports start void.  MM_ORDER_ARRIVAL and MM_F_NO_DEDUPE engines refuse
 * both calls, so their reports are always void.
 * PER LOBBY: per_lobby[h] describes lobbies[h] of that call, in its header order, by the DEFINITION of
 * mm_match_quality: c(r) clamped to [rmin - 1, rmax + 1], min_rating, max_rating, rating_sum and the team imbalance.  A
 * solo's rating is its pool rating; a party member's is its own rating as enqueued (not the party's R).  Members are
 * taken in the order the call returned them, so with "team_balance" (mm_widen lobbies of masked modes) or
 * "party_balance" (mm_party_match lobbies of masked modes) the imbalance is that of the emitted teams.
 * WAIT of a member: the WAIT of mm_queue_stats at the call's `now`, from a solo's own enq_ts and from a party member's
 * party's enq_ts.
 * PER QUEUE, one record per (mode, group) queue, empty ones included, in mm_queue_stats order: waits[q] holds
 * n_lobbies, n_matched (members), max_match_wait and match_wait_hist over every member of the queue's lobbies of that
 * call, in the BUCKETS of mm_queue_stats; quality[q] every mm_queue_quality field as mm_match_quality defines it, over
 * those lobbies.  waits, quality and per_lobby may each be NULL, which skips that output.
 * READ-ONLY: the call changes nothing — not the pool, the party table, the active set, the results of any call, the
 * snapshot, the reject list or pending async_results copies.
 * REFUSALS, decided before anything is written: MM_E_ARG a null e, n_out or n_lobbies, or an unknown source; MM_E_CAP
 * cap < n_modes * n_groups while waits or quality is not NULL (*n_out = the records needed), or per_lobby not NULL
 * with lobby_cap below the call's lobby count (*n_lobbies = the count needed).
 * COST AND MEMORY: the capture runs inside mm_party_match / mm_widen, after the balance pass, and its device time is
 * part of their device_us: the enqueue stamp of every taken solo is written beside its id by the take, then one warp
 * per lobby over its member slots, one pass over the members for the waits and the per-queue quality records.  Kept
 * per source, allocated by the first call and grown to the largest call: 24 bytes per lobby and 1488 bytes per queue;
 * shared by the two calls: 8 bytes per member and 4 bytes per lobby of the largest call, 8 bytes per queue, and the c
 * column "team_balance" also uses (4 bytes per player of capacity).  mm_offtick_report itself is device-to-host copies of those records only.                                          */
#define MM_OFFTICK_PARTY_MATCH 0u
#define MM_OFFTICK_WIDEN 1u

typedef struct mm_match_waits {    /* the match section of mm_queue_stat, for one off-tick call */
  uint8_t mode, group;
  uint16_t reserved;               /* 0 */
  uint32_t n_lobbies, n_matched, max_match_wait;
  uint32_t match_wait_hist[MM_WAIT_BUCKETS];
} mm_match_waits;                  /* 496 bytes */

int mm_offtick_report(mm_engine* e, uint32_t source, mm_match_waits* waits, mm_queue_quality* quality, uint32_t cap,
                      uint32_t* n_out, mm_lobby_quality* per_lobby, uint32_t lobby_cap, uint32_t* n_lobbies);

/* ---- lobby budget: how many lobbies a tick may emit ------------------------------
 * EXTENSION (flow control).  The reference emits one lobby at a time behind prefetch_count: 10 (search/worker.ex:29),
 * and its lobby stage answers the players of a lobby it finds no game server for with an error
 * (game-lobby/worker.ex:89-103,118-141); a request the strategist does not add stays a queued player
 * (search/worker.ex:239-248,308-310).  Here the caller tells the tick how many lobbies it may emit — per (mode, group)
 * queue, to pause or drain a rating group, and per game mode, because game servers host modes — and the rest stays
 * queued, in order, with its waits and the search timeout running on.  Which players form a lobby, in which order and
 * on which team is untouched (S0 and S1 alike): the budget only decides how many of a queue's lobbies, in their
 * emission order, come out this tick.
 *
 * mm_set_lobby_budget: per_queue holds n_modes * n_groups entries in the record order of mm_queue_stats (mode *
 * n_groups + group), per_mode holds n_modes; either may be NULL (= all unlimited).  Values are lobbies per tick;
 * MM_BUDGET_UNLIMITED = no limit, 0 = the queue (mode) emits nothing.  Takes effect from the next tick and stays until
 * set again.  It is an option in the sense of NOT IN THE IMAGE below: mm_export does not carry it, mm_snapshot /
 * mm_restore leave it alone, an imported engine starts unlimited.  Default: unlimited, and then every result of every
 * call is bit for bit what it is without this section.
 *
 * DEFINITION.  For queue q = (m, g) let c_q be the lobbies the tick would emit from it with no budget (under the
 * current max_spread), c'_q = min(c_q, per_queue[q]) and C_m the sum of c'_q over the groups of mode m.  If C_m <=
 * per_mode[m], a_q = c'_q.  Otherwise the mode's budget B = per_mode[m] is apportioned by largest remainder, in 64-bit
 * integers: a_q = floor(B c'_q / C_m), and the B - sum(a_q) groups with the largest (B c'_q) mod C_m get one more, ties
 * to the lower group index (then a_q <= c'_q and the a_q of the mode add up to B).  The tick emits the FIRST a_q
 * LOBBIES of the queue in its emission order — the lobbies the unbudgeted tick would have put at the queue's first a_q
 * header positions, same members, same member order, same emit_seq — and every other player of the queue stays queued
 * in enqueue order, exactly as a residual player does.  Lobbies stay ordered by (mode, group, emission);
 * mm_tick_stats.n_lobbies / n_matched / n_residual and the match section of mm_queue_stats count what was emitted and
 * what stays.  The lobbies of mm_band_match are outside the tick and outside the budget.
 *
 * mm_lobby_budget_report: per queue, c_q (candidates) and a_q (emitted) of the last completed tick, zeros before the
 * first tick and after one that failed; c_q - a_q is what the budget held back.  mm_lobby_candidates: c_q for the pool
 * as it is now, budgets ignored — a dry run of the lobby cut on the resident per-key player counts that changes
 * nothing: not the pool, not the last tick's results or the match section of mm_queue_stats, not pending
 * async_results copies.  Removed-while-queued players are not counted, as the tick drops them.  It is what lets
 * several engines share one mode budget: gather every engine's c_q, apportion once, set each engine's per-queue
 * budgets.  Both: cap / n_out as in mm_queue_stats (MM_E_CAP and *n_out = n_modes * n_groups if cap is smaller);
 * MM_E_STATE while an mm_enqueue_packed_begin batch is staged.  Refusals are decided before anything changes.      */
#define MM_BUDGET_UNLIMITED 0xFFFFFFFFu
int mm_set_lobby_budget(mm_engine* e, const uint32_t* per_queue, const uint32_t* per_mode);
int mm_lobby_budget_report(mm_engine* e, uint32_t* candidates, uint32_t* emitted, uint32_t cap, uint32_t* n_out);
int mm_lobby_candidates(mm_engine* e, uint32_t* candidates, uint32_t cap, uint32_t* n_out);

/* ---- off-tick budget: how many lobbies mm_party_match and mm_widen may emit ------------------------------
 * EXTENSION (flow control).  Party and widen lobbies need game servers as the tick's do, so each of the two calls has
 * a lobby budget of its own, with the tick's rules: a step that runs party_match, the tick and widen can keep every
 * lobby it publishes within the free servers of a mode, and a paused queue emits nothing from any of them.
 *
 * mm_set_offtick_budget: source MM_OFFTICK_PARTY_MATCH or MM_OFFTICK_WIDEN; per_queue / per_mode, their units,
 * MM_BUDGET_UNLIMITED, NULL = all unlimited and "an array without a limit is no array" as in mm_set_lobby_budget.
 * Takes effect from the next call of that source and stays until set again.  Each source's budget is separate from the
 * other's and from the tick's.  Default: unlimited, and then every output of both calls is bit for bit what it is
 * without this section, from the same kernels.
 *
 * DEFINITION.  Let c_q be the lobbies the call would emit from queue q with no budget (same `now`, same rules).  The
 * allowance a_q follows the tick's DEFINITION: c'_q = min(c_q, per_queue[q]), then the per-mode largest remainder in
 * 64-bit integers, ties to the lower group.  The call emits the FIRST a_q LOBBIES of every queue in its emission order —
 * same members, same member order, same parties on the same teams — and everything else stays queued, as if the
 * queue's plan had stopped after its a_q-th lobby.  This is exact because both calls serve each queue on its own and
 * in order, so a lobby depends only on the lobbies of its queue formed before it.  Headers stay in (mode, group,
 * emission) order, first_member renumbered.
 * STATS: n_lobbies, n_matched, n_parties and sum_imbalance describe the emitted lobbies; n_anchors and n_absorbed are
 * those of the unbudgeted call.  MM_E_CAP checks lobby_cap / member_cap against the emitted counts; zero capacities
 * remain a dry run.
 * WHAT FOLLOWS THE CUT: "team_balance", "party_balance" and mm_offtick_report see only the emitted lobbies.
 * EQUIVALENCE.  A budgeted mm_widen leaves the engine as mm_take of the returned ids would.  A budgeted mm_party_match
 * leaves it as mm_party_match's own construction would with only the emitted lobbies: mm_export_parties and
 * mm_export, delete the placed parties and the taken solos, then import and mm_merge_parties(MM_PARTY_KEEP_SEQ).
 *
 * mm_offtick_budget_report: per queue, c_q (candidates) and a_q (emitted) of the last call of `source` that returned
 * MM_OK or MM_E_CAP (an MM_E_CAP dry run gives c_q without changing anything, which a later cross-engine share of a
 * mode budget needs; this is unlike mm_offtick_report, which is void after MM_E_CAP).  All zeros before the first such
 * call, after a call that served no queue or found no anchor, and after any other refusal.  With no budget set,
 * candidates equal emitted.  cap / n_out as in mm_queue_stats (MM_E_CAP and *n_out = n_modes * n_groups if cap is
 * smaller).
 * NOT IN THE IMAGE.  Budgets are options, as the tick's are: mm_export does not carry them, an imported engine starts
 * unlimited, and mm_snapshot / mm_restore leave them alone.
 * REFUSALS, decided before anything changes: mm_set_offtick_budget MM_E_ARG for a null e or an unknown source;
 * mm_offtick_budget_report MM_E_ARG for a null e or n_out, null arrays with cap > 0 or an unknown source, MM_E_CAP
 * as above, MM_E_STATE while an mm_enqueue_packed_begin batch is staged.
 * COST: with a budget set, one single-CTA kernel after the call's plan and one read of a flag; when some a_q < c_q the
 * plan runs again from its start, capped at a_q lobbies per queue (it stops serving a queue's anchors after its a_q-th
 * lobby).  Without a budget nothing is launched or copied.                                                          */
int mm_set_offtick_budget(mm_engine* e, uint32_t source, const uint32_t* per_queue, const uint32_t* per_mode);
int mm_offtick_budget_report(mm_engine* e, uint32_t source, uint32_t* candidates, uint32_t* emitted, uint32_t cap,
                             uint32_t* n_out);

/* ---- search timeout ------------------------------------------------------------
 * EXTENSION (search timeout): every live queued player whose WAIT at `now` (the definition of mm_queue_stats)
 * is >= max_wait leaves the pool AND the active set, as if mm_remove had been called with its id: mm_in_queue
 * reads 0, the id can be enqueued again, and the slot is dropped by the next tick (counted in its n_dead, and in
 * mm_queue_stats' n_removed until then).  Matched, removed and taken players are not affected.  max_wait = 0
 * expires every queued player; max_wait >= 2^31 expires none.  MM_F_NO_DEDUPE engines have no active set: only
 * the pool changes.  The caller tells each expired player so (the reference's answer to a player it cannot
 * serve: game-lobby/worker.ex:63-71,89-103, an error response and ActiveUser.remove_user).
 * ids[0..*n_expired): the expired ids (unordered); seq (may be NULL): the enqueue sequence number of each (the
 * numbering of emit_seq), which also tells apart the entries of a repeated id in an MM_F_NO_DEDUPE engine.
 * If more than `cap` would expire: MM_E_CAP, *n_expired = the number that would, and NOTHING changes
 * (so cap = 0 with ids = NULL is a dry run).  One pass over the resident mode and enqueue-stamp columns when cap
 * is at least mm_pool_size, else a counting pass first.  Runs on the engine's stream; pending async_results
 * copies are left alone; the last tick's match section of mm_queue_stats is unaffected.                        */
int mm_expire(mm_engine* e, uint64_t now, uint32_t max_wait, uint64_t* ids, uint32_t* seq, uint32_t cap,
              uint32_t* n_expired);
/* Same, ids returned as 32-bit handles (MM_F_DENSE_IDS engines; MM_E_STATE otherwise). */
int mm_expire_packed(mm_engine* e, uint64_t now, uint32_t max_wait, uint32_t* handles, uint32_t* seq,
                     uint32_t cap, uint32_t* n_expired);

/* Device-side snapshot / restore of pool + active set (ram_copies analogue,
 * models/active_user.ex:20; used by bench.py to replay one pool K times).
 * mm_snapshot copies the queued players, the enqueue sequence counter and the whole active set (every id queued or
 * matched and not yet removed, with the counts behind mm_active_size and the refusal rule of a hashed set).
 * mm_restore puts all of it back, any number of times: an id enqueued since the snapshot can be offered again, an id
 * removed since is queued and removable again.  The snapshot of the active set takes 16 B per hashed slot (8 B per
 * handle with MM_F_DENSE_IDS) of device memory beside the pool's copy; MM_F_NO_DEDUPE engines have no active set.
 * The last tick's match section of mm_queue_stats is void after mm_restore.                                          */
int mm_snapshot(mm_engine* e);
int mm_restore(mm_engine* e);

/* ---- hand-over: host image of the queue state ------------------------------------------
 * The copy_store analogue (models/active_user.ex:29-31, models/lobby_state.ex:31-40: mnesiam replicates ActiveUser and
 * LobbyState to every node, so a restarted node loses no queued player).  Here the engine is the only place a queued
 * player exists once its delivery is acked: mm_export writes what a new process needs into a host buffer (to disk, to
 * another host, to another GPU), mm_import loads it into a FRESH engine (nothing ever enqueued, imported or restored),
 * which then behaves exactly as the source would have.
 *
 * IMAGE LAYOUT (little-endian).  mm_image_header, then seven sections, each starting at the next multiple of 8 bytes
 * after the previous one ends (the first at offset sizeof(mm_image_header) = 624); total_bytes is the end of the last
 * section rounded up to 8.  Padding bytes are zero.  W = id_bytes, N = n_players, M = n_active:
 *   1. part_count  u32[n_parts]  queued players of each layout partition, in layout-partition order (the engine's
 *                                storage of a (mode, group) queue: one partition per queue, or several of <= 255 sort
 *                                keys each for a wide group without MM_F_WIDE_PARTITIONS)
 *   2. id          W * N         player ids (u64), or 32-bit handles for MM_F_DENSE_IDS engines
 *   3. rating      i32[N]
 *   4. enq_ts      u32[N]
 *   5. seq         u32[N]        enqueue sequence numbers (the numbering of emit_seq)
 *   6. mode        u8[N]
 *   7. active      W * M         ids in the active set that are not queued: players matched by a tick and not yet
 *                                removed, and players taken by mm_take (unordered)
 * Sections 2-6 are columns of one player list: partition by partition, in layout-partition order, enqueue order
 * inside a partition.
 *
 * NOT IN THE IMAGE: dead slots (players removed, taken or expired while queued: the next tick would drop them); the
 * last batch's reject list (mm_enqueue_rejects is empty after import); the last tick's match section of
 * mm_queue_stats (void after import, as after mm_restore); the mm_snapshot state; the options (max_spread, tick_impl,
 * rank_impl, async_results, the lobby budget and the off-tick budgets: the caller sets them again).
 *
 * EQUIVALENCE.  After mm_import, every sequence of calls gives the same results on the imported engine as on the
 * source: enqueue codes, remove / take / expire outputs, in_queue, active_size, pool_read, the ticks' lobbies,
 * members, emit_seq, n_lobbies, n_matched, n_residual, and the waiting section of mm_queue_stats.  What differs comes
 * from the dead slots that were not carried: mm_pool_size, the next tick's pool_before and n_dead, mm_queue_stats'
 * n_removed, and how soon a pool near capacity answers "full" (code 3): the imported pool has the dead slots' room.
 *
 * mm_export: buf = NULL with cap = 0 -> *n_bytes = the size the image needs, MM_OK.  cap smaller than that ->
 * MM_E_CAP and *n_bytes.  MM_E_STATE while an mm_enqueue_packed_begin batch is staged.  The source engine is never
 * changed (a checkpoint and a move are the same call); pending async_results copies are left alone.  The device
 * counts the live slots of every tile, scans the counts and writes the live players compacted, in order; the active
 * section is compacted from the active-set table.  About 21 B per queued player (17 with handles).  The size query
 * runs the counting passes too: a caller that wants one call passes a buffer of the layout's size with n_parts =
 * MM_MAX_GROUPS * MM_MAX_MODES, N = mm_pool_size, M = mm_active_size, W = 8 (an upper bound) and reads *n_bytes.
 * The image-sized device scratch of both calls is freed before they return.  mm_import moves the image to the device
 * in one host-to-device copy and runs the load kernels after it; it does not overlap them with a chunked upload as
 * ingest does (the kernels' share of the call is in DESIGN §5).
 * mm_import: MM_E_STATE if the engine is not fresh (or has a staged batch).  MM_E_ARG if the image's config differs
 * from the engine's on n_groups, group_lo / group_hi, default_group, n_modes, modes, order_mode or flags (capacity,
 * active_capacity and device may differ: a shard can grow or move to another GPU), and for an image that is truncated,
 * corrupted or hostile: bad magic / version / lengths / section counts, partition counts that do not add up, a mode
 * >= n_modes, a rating that does not map to the partition it is filed under, an id outside the id range (handles >=
 * active_capacity), a duplicate id within or across the sections, sequence numbers not strictly increasing in
 * enqueue order inside a partition (or equal to seq_next).  MM_E_CAP if the players do not fit the capacity (or a
 * hashed active set).  After any failure the engine is empty and still fresh.                                      */
#define MM_IMAGE_MAGIC 0x474D494Du /* "MIMG" */
#define MM_IMAGE_VERSION 1u

typedef struct mm_image_header {
  uint32_t magic;       /* MM_IMAGE_MAGIC                                                         */
  uint32_t version;     /* MM_IMAGE_VERSION                                                       */
  uint32_t abi_version; /* MM_ABI_VERSION of the writer                                           */
  uint32_t id_bytes;    /* 8: u64 ids; 4: 32-bit handles (MM_F_DENSE_IDS engines)                 */
  uint64_t total_bytes; /* the whole image, this header included                                  */
  uint32_t n_parts;     /* layout partitions: entries of section 1                                */
  uint32_t n_players;   /* queued players: entries of sections 2-6                                */
  uint32_t n_active;    /* active ids that are not queued: entries of section 7                   */
  uint32_t seq_next;    /* enqueue sequence number of the next offered player                     */
  mm_config config;     /* the writer's config (capacity, active_capacity, device: informational) */
  uint32_t reserved;    /* 0                                                                      */
} mm_image_header;      /* 624 bytes */

int mm_export(mm_engine* e, void* buf, uint64_t cap, uint64_t* n_bytes);
int mm_import(mm_engine* e, const void* buf, uint64_t n_bytes);

/* EXTENSION (regroup on import): load an mm_export image written under ANOTHER config into a fresh engine, so that a
 * new RatingGroups table (config/config.exs:27-36), a new default group, an added or dropped game mode, another
 * order_mode or MM_F_WIDE_PARTITIONS can be deployed without dropping the queue.  The image's config may differ from
 * the engine's on n_groups, group_lo / group_hi, default_group, n_modes, modes, order_mode and MM_F_WIDE_PARTITIONS;
 * it must match on the id width (MM_F_DENSE_IDS) and MM_F_NO_DEDUPE.
 * Each queued player goes to the layout partition its (rating, mode) maps to under the ENGINE's config, in age order
 * inside it ((seq - seq_next) mod 2^32 ascending: the order of mm_requeue and mm_pool_read), with its id, rating,
 * mode, enq_ts and seq; seq_next is kept, and the active section goes into the active set unchanged.  A player whose
 * rating has no group here (default_group = -1) or whose mode is >= n_modes is REJECTED: not queued, not in the
 * active set; its image index goes to rejected[] (ascending) and *n_rejected counts them — the caller answers those
 * players (they left).
 * Refusals, all decided by one read of the device's counters before the pool is written; after any of them the engine
 * is empty and still fresh:
 *   MM_E_STATE the engine is not fresh, or a packed batch is staged;
 *   MM_E_ARG   a queue image; another id width or MM_F_NO_DEDUPE; an image's config that is not a valid config
 *              (capacity aside); and everything mm_import refuses in an image on an engine created with the IMAGE's
 *              config, with mm_import's mm_last_error wording: bad lengths or counts, a mode >= the image's n_modes, a
 *              rating outside the partition it is filed under, an id out of the engine's id range or repeated
 *              anywhere in the image, sequence numbers out of order inside an image partition or equal to seq_next.
 *              Also two players the re-filing puts into one partition with the same seq ("sequence numbers out of
 *              order");
 *   MM_E_CAP   more than `cap` players would be rejected (*n_rejected = the count: cap = 0 with rejected = NULL is a
 *              dry run), or the kept players do not fit under mm_import's capacity rules.
 * Cost: one pass to classify, a stable counting scatter by new partition, and ceil(log2 k) merge rounds when up to
 * k image partitions feed one new partition (none when groups only split or their bounds move); then mm_import's load.
 *
 * EQUIVALENCE.  Let R be the image re-filed: header config = the engine's config, section 1 = the kept players per
 * layout partition of the engine, sections 2-6 = the kept players partition by partition in age order inside a
 * partition, section 7 unchanged, the same seq_next.  After mm_import_regroup(img), every later call sequence gives
 * the same results as on a fresh engine that called mm_import(R): as if each kept player had been enqueued into this
 * engine in its original order, with its original stamp and number.  When the configs are equal, R is the image itself.
 * Not covered: queue images (mm_merge still needs equal configs); a sharded deployment is re-cut with
 * mm_import_regroup_many below.                                                                                     */
int mm_import_regroup(mm_engine* e, const void* buf, uint64_t n_bytes, uint32_t cap, uint32_t* rejected,
                      uint32_t* n_rejected);

/* EXTENSION (re-cut of a sharded deployment): load up to 64 mm_export images (not queue images) into a FRESH engine.
 * All of them were written under ONE config, which may differ from the engine's exactly as mm_import_regroup allows
 * (typically: the old ranks of a deployment sharded by rating group, each exporting its engine, and the new ranks
 * taking the queues they own under a new group table and owner array).
 *   keep: n_modes * n_groups bytes of THIS engine's config in the record order of mm_queue_stats (mode * n_groups +
 *   group); NULL = every queue.  Each image player goes to the queue its (rating, mode) maps to under the engine's
 *   config: loaded if keep selects the queue; SKIPPED (counted in *n_elsewhere: another rank owns it) if the queue
 *   exists but is not selected; REJECTED if the engine has no queue for it — rej_image[i], rej_index[i] name the
 *   image and the player's index in it, ascending by (image, index).
 *   active_image: the image whose active section (section 7) goes into the active set; UINT32_MAX = none.  In a re-cut
 *   every rank takes its own: its matched-not-removed ids stay where the lobby stage's mm_remove goes.
 * ORDER inside a new queue (layout partition).  Take each image's players of that partition in the order
 * mm_import_regroup would give them (age order, (seq - seq_next) mod 2^32 ascending, with that image's seq_next).
 * Key each such sequence by the RUNNING MAXIMUM of enq_ts along it, and interleave the images as a stable merge by
 * that key, ties to the lower image index — the same as a classic head-comparison merge.  With stamps that never
 * decrease with age (what SearchPool writes) this is plain stamp order, ties by image and then age; with one image it
 * is mm_import_regroup's order whatever the stamps.
 * SEQUENCE NUMBERS.  n_images == 1: every number and seq_next are kept — the call is mm_import_regroup plus keep and
 * active_image.  n_images > 1: the numbers of different engines cannot be compared, so the kept players are numbered
 * 0 .. n_kept-1 by one global total order, (running-max stamp, image, age, then the lower partition), and seq_next =
 * n_kept: every partition stays strictly increasing and emit_seq stays an arrival order across queues.  Stamps are
 * kept, so waits, mm_expire and mm_queue_stats carry over unchanged.
 * Refusals, all decided by one read of the device's counters before the pool is written; after any of them the engine
 * is empty and still fresh:
 *   MM_E_STATE the engine is not fresh, or a packed batch is staged;
 *   MM_E_ARG   everything mm_import_regroup refuses in any image, with its wording; images whose configs differ from
 *              each other (groups, default_group, modes, order_mode, flags); n_images of 0 or more than 64;
 *              active_image out of range; an id repeated within or across the loaded images or the taken active
 *              section (engines with an active set);
 *   MM_E_CAP   more than `cap` rejects (*n_rejected = the count: cap = 0 with NULL outputs is a dry run), or the kept
 *              players do not fit under mm_import's capacity rules.
 * Cost: every image runs mm_import_regroup's passes; with n_images > 1, ceil(log2 n_images) merge rounds over the
 * kept players by (running-max stamp, image, age), a segmented max scan for the running maxima, and
 * ceil(log2 n_parts) rounds that merge the partitions' lists into the global order.  The images are uploaded once
 * each; the scratch is one allocation sized by the images, freed before the call returns.
 * EQUIVALENCE.  Let R be the restated image: header config = the engine's config, section 1 = the kept players per
 * layout partition, sections 2-6 = the kept players partition by partition in the merged order above with the numbers
 * above, section 7 = active_image's section (empty for none), seq_next as above.  After mm_import_regroup_many, every
 * later call sequence gives what a fresh engine gives after mm_import(R).
 * Not covered: a re-cut that changes the number of ranks; host records above the engine (SearchPool's player
 * documents and requeue records); requeue (mm_requeue) of players matched before a re-cut with n_images > 1, whose old
 * seq has no place in the new numbering.                                                                            */
int mm_import_regroup_many(mm_engine* e, uint32_t n_images, const void* const* bufs, const uint64_t* n_bytes,
                           const uint8_t* keep, uint32_t active_image, uint32_t cap, uint32_t* rej_image,
                           uint32_t* rej_index, uint32_t* n_rejected, uint32_t* n_elsewhere);

/* EXTENSION (re-cut with parties queued): mm_import_regroup_many that also takes, beside engine image k, the party
 * image (mm_export_parties) its rank wrote at the same stop: released first, then exported.  The solo arguments mean
 * what they mean for mm_import_regroup_many; `parties` may be NULL, and then (as with every party image NULL or empty)
 * the call IS mm_import_regroup_many, byte for byte.                                                                 */
typedef struct mm_recut_parties {
  const void* const* bufs;  /* [n_images] party image k, written at the same stop as engine image k; NULL = none   */
  const uint64_t* n_bytes;  /* [n_images] its length (0 with NULL)                                                 */
  uint32_t cap;             /* room in rej_image / rej_index, in parties                                           */
  uint32_t* rej_image;      /* out: rejected parties as (image, party index in its party image), ascending         */
  uint32_t* rej_index;
  uint32_t n_rejected;      /* out: parties this config has no queue for                                           */
  uint32_t n_elsewhere;     /* out: parties of an existing queue that `keep` does not select                       */
  uint32_t n_loaded;        /* out                                                                                 */
  uint32_t reserved;        /* 0                                                                                   */
} mm_recut_parties;

/* Party j of image k gets its R = floor(sum of member ratings / size) recomputed, as mm_merge_parties does, and is
 *   REJECTED if its mode is >= n_modes, its size is above its mode's team_size, or R has no group: its members do not
 *   enter the active set; the caller answers them (parties->rej_image / rej_index);
 *   SKIPPED (parties->n_elsewhere) if its queue (mode, group(R)) exists but `keep` does not select it;
 *   KEPT otherwise.
 * ORDER AND NUMBERS.  n_images == 1: every number and seq_next are kept; the call equals mm_import_regroup_many of the
 * one image followed by mm_merge_parties(MM_PARTY_KEEP_SEQ) of the kept parties.  n_images > 1: image k's kept parties
 * of one new queue, in age order, form a run keyed by the running maximum of enq_ts along it; kept solos keep their
 * keys (the running maximum along their (image, new partition) runs).  Every kept solo and kept party is numbered by
 * its position in ONE total order, (running-max stamp, image, age) — within one image solos and parties share the age
 * numbering — and seq_next = kept solos + kept parties.  With monotone stamps (what SearchPool writes) this is plain
 * stamp order, ties by image and then age.
 * LOAD.  The solos as mm_import_regroup_many loads them; the kept parties into the party table in the new age order,
 * with their new numbers, mode, stamp and members, and R / group / bin under this config; each member's active-set
 * value is its row's.  active_image's section 7 goes in as before (matched party members are already in it).
 * Refusals, all decided by one read of the device's counters before anything is written; after any of them the engine
 * is empty and still fresh, and its party table is empty:
 *   MM_E_ARG   everything mm_import_regroup_many refuses; a non-null party image mm_merge_parties would refuse as
 *              malformed (magic, version, lengths, a size below 2, sizes that do not add up to the member count,
 *              numbers not strictly increasing in age order, an id out of range); party image k whose config or
 *              seq_next differs from engine image k's (not written at the same stop); a party number equal to that of
 *              a solo of its image; an id repeated in a party, across parties, or against any loaded solo or the taken
 *              active section; a non-empty party image on an MM_ORDER_ARRIVAL or MM_F_NO_DEDUPE engine;
 *   MM_E_STATE what mm_import_regroup_many gives; a non-empty party image while party_capacity is 0;
 *   MM_E_CAP   the solo capacity rules; more rejected parties than parties->cap (parties->n_rejected = the count: cap
 *              0 with NULL outputs is a dry run); kept members above party_capacity (exactly enough room loads); solos
 *              plus party members past the 3/4 load of a hashed active set.
 * EQUIVALENCE.  Let R be the restated engine image, built as for mm_import_regroup_many but with the numbers and
 * seq_next above, and RP the restated party image: this engine's config, the kept parties in the new age order with
 * their new numbers, members in party order, R's seq_next.  After the call, every later call sequence gives what a
 * fresh engine with the same party_capacity gives after mm_import(R) and mm_merge_parties(RP, MM_PARTY_KEEP_SEQ).
 * Cost: mm_import_regroup_many's passes, plus per party image one classify pass and the stable scatter by queue; with
 * n_images > 1 the parties' queue runs go through the same running-max scan and merges, ceil(log2 n_queues) rounds
 * order the parties, and one more merge round interleaves them with the solos' global order.
 * Not covered: a re-cut that changes the number of ranks; mm_requeue / mm_requeue_party of players and parties matched
 * before a re-cut with n_images > 1 (their old numbers have no place in the new numbering); SearchPool host records. */
int mm_import_regroup_many_parties(mm_engine* e, uint32_t n_images, const void* const* bufs, const uint64_t* n_bytes,
                                   const uint8_t* keep, uint32_t active_image, uint32_t cap, uint32_t* rej_image,
                                   uint32_t* rej_index, uint32_t* n_rejected, uint32_t* n_elsewhere,
                                   mm_recut_parties* parties);

/* ---- queue move: part of an engine into another running engine ---------------------------
 * The reference's queues live in RabbitMQ and its state in replicated Mnesia tables, so any node's workers can serve
 * any rating group (application.ex:26-40).  Here a queued player lives in one engine: mm_export_queues releases
 * whole (mode, group) queues into an image, mm_merge loads that image into an engine that is already running (scale
 * out / in, rebalancing rating-group shards).
 *
 * mm_export_queues: `queues` holds n_modes * n_groups bytes in the record order of mm_queue_stats (mode * n_groups +
 * group); a non-zero byte selects the queue.  The image has the mm_image_header layout with magic
 * MM_QUEUE_IMAGE_MAGIC: part_count is zero for the partitions of unselected queues, sections 2-6 hold the selected
 * queues' live players (partition by partition, enqueue order inside a partition), and section 7 is EMPTY — an id that
 * is matched (or taken) and not yet removed cannot be attributed to a queue, so it stays in the source's active set
 * and its mm_remove goes to the source.  buf = NULL with cap = 0 -> *n_bytes = the size, nothing changes; cap too
 * small -> MM_E_CAP and *n_bytes, nothing changes.  A call that writes the image RELEASES its players in the same
 * call, exactly as mm_remove of their ids would (dead slots until the next tick, counted in n_removed): a tick between
 * an export and a release would match players who are already on their way.  MM_E_STATE while an
 * mm_enqueue_packed_begin batch is staged; pending async_results copies are left alone.
 *
 * mm_merge: refusals, all decided before anything changes:
 *   MM_E_ARG   bad magic (an mm_export image is refused here, and mm_import refuses a queue image), version, lengths,
 *              id width, a config that differs on the fields mm_import compares, a player whose mode is >= n_modes,
 *              whose rating has no group or does not map to its partition, whose id or handle is out of range, or
 *              sequence numbers out of order inside a partition (a device pre-pass over the image columns);
 *   MM_E_STATE a queue the image's players fall into holds a LIVE player here (dead slots are fine), or a staged
 *              packed batch;
 *   MM_E_CAP   the players that would be queued do not fit the capacity (pool slots in use + players queued), or the
 *              3/4 load of a hashed active set, or more players would be rejected than `cap` holds (*n_rejected then
 *              holds the count).  These are exact: the ids that would be rejected are counted first when needed.
 * The load is one ingest batch: each queue's players in the source's enqueue order, appended per partition, with the
 * image's enq_ts; they take this engine's next n_players sequence numbers in that order.  An id already in this
 * engine's active set, or a later copy of an id inside the image, is not queued: its image index goes to `rejected`
 * (ascending).  MM_F_NO_DEDUPE engines reject nothing.  mm_enqueue_rejects still describes the last mm_enqueue*
 * batch afterwards.
 *
 * EQUIVALENCE.  After a move, the source behaves like a twin that called mm_remove on the moved ids.  On the target,
 * every later call sequence gives, for the moved queues, what the source would have given: lobbies, members,
 * n_matched, in_queue, pool_read and the waiting section of mm_queue_stats; emit_seq as an order (sorting a moved
 * queue's lobbies by emit_seq gives the source's order; the numbers are the target's).  Queues never depend on each
 * other (S0 and S1 alike), so the unselected queues of both engines are unaffected.  Merging the image back into the
 * source restores the source's results; until the source's next tick the released players' dead slots still count
 * against its capacity, so a source that was nearly full may refuse it (MM_E_CAP) until then.                                                                               */
#define MM_QUEUE_IMAGE_MAGIC 0x5155514Du /* "MQUQ": same header and sections as an mm_export image */

int mm_export_queues(mm_engine* e, const uint8_t* queues, void* buf, uint64_t cap, uint64_t* n_bytes);
int mm_merge(mm_engine* e, const void* buf, uint64_t n_bytes, uint32_t cap, uint32_t* rejected, uint32_t* n_rejected);

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
 *   "team_balance"  EXTENSION (balanced teams): a mask, bit m = balance the lobbies of game mode m; 0 (default) = off.
 *                   MM_E_ARG if a set bit names a mode >= n_modes, a mode whose teams != 2 or whose team_size > 8
 *                   (L <= 16: at most C(15, 7) = 6435 splits per lobby).  A 1v1 mode is accepted and changes nothing.
 *                   Both feed orders.  For every lobby of a masked mode, with m_0 .. m_{L-1} its members in the order
 *                   the tick (or mm_widen) forms them and c_i = c(rating(m_i)) the tick's key clamp to [rmin - 1,
 *                   rmax + 1] (as in mm_match_quality): over the sets A of S members with m_0 in A, minimise
 *                   |sum_A c - sum_rest c| (64-bit); ties go to the smallest M(A) = sum of 2^i over i in A, i > 0.  The
 *                   lobby's members become A's members in their old relative order, then the others in theirs, so
 *                   team 1 is still members [0, S) and team 2 [S, 2S) (the team-major contract of mm_lobby_hdr).
 *                   Lobby membership, lobby order, headers and emit_seq do not change; with the option off every
 *                   output is what it was.  Applies to every lobby a tick of any form emits (mm_tick, mm_tick_packed,
 *                   async_results, mm_tick_device / mm_results_device, fused or split) and to every mm_widen lobby;
 *                   the mask in force when the call runs decides.  mm_backfill (the caller owns the running lobby's
 *                   teams) and mm_band_match are not balanced.  Not part of an image: mm_export / mm_import do not
 *                   carry it.  mm_match_quality: after a balanced tick, imbalance (per lobby, max_imbalance,
 *                   sum_imbalance, imbalance_hist) describes the teams emitted; spread and rating sums are unchanged.
 *                   mm_locate: under its condition (neither the options nor the lobby budget change before the tick),
 *                   member is the player's index in the balanced lobby.  Cost: after the tick, one warp per lobby of a
 *                   masked mode (the L ids read and, unless the split is the identity, written back); in arrival order
 *                   also one pass over the mode, rating and left bits of the pool the tick read.  The pass is part of
 *                   the tick: its CUDA-event time is added to mm_tick_stats.device_us (the phase times leave it out),
 *                   and mm_tick_device returns once it is done, so mm_results_device's members are final.  Device memory,
 *                   allocated by the first balanced call and kept: 4 bytes per lobby the pool could hold, 4 bytes per
 *                   player of capacity and, in arrival order, 4 bytes per chunk.
 *   "party_balance" EXTENSION (balanced party lobbies): a mask, bit m = balance the mm_party_match lobbies of game
 *                   mode m; 0 (default) = off.  team_balance's refusals (MM_E_ARG: a mode >= n_modes, teams != 2,
 *                   team_size > 8); a 1v1 mode is accepted and changes nothing; party_capacity need not be set.
 *                   Independent of team_balance: team_balance never splits party lobbies and party_balance splits
 *                   nothing else (tick, mm_widen, mm_backfill).  For every lobby of a masked mode that mm_party_match
 *                   forms, with m_0 .. m_{L-1} its members in the order the call forms them without the option and
 *                   c_i = c(rating of m_i) clamped to [rmin - 1, rmax + 1] (a party member's own rating, not the
 *                   party's R; a solo's pool rating): a set A of S members is admissible when it holds m_0 and, of
 *                   every party of the lobby, all members or none.  Over the admissible sets, minimise |sum_A c -
 *                   sum_rest c| (64-bit); ties go to the smallest M(A) = sum of 2^i over i in A, i > 0.  The lobby's
 *                   members become A's members in their old relative order, then the others in theirs (team 1 =
 *                   members [0, S)).  The lobby as formed is admissible, so its imbalance never grows.  Which lobbies
 *                   form, their headers and order, the solos taken, the parties placed, the party table, the active
 *                   set and seq_next do not change; with the option off every output is what it was.  A dry run or
 *                   an MM_E_CAP refusal runs no balance pass.  mm_party_stats.sum_imbalance sums the emitted
 *                   lobbies' imbalances.  Not part of an image: mm_export / mm_import do not carry it.  Cost: after
 *                   the call's member copy, one thread per placed party (its members' c and its lobby's continuation
 *                   bits), one warp per solo piece (as mm_widen) and one warp per lobby of a masked mode (the L ids
 *                   read and, unless the split is the identity, written back); the pass is inside device_us.
 *                   Device memory, allocated by the first balanced call and kept: 4 bytes per member slot of the
 *                   largest call (at least capacity + 64), 4 bytes per lobby of the largest call and 8 bytes.
 *   "async_results" 1 = mm_tick does not wait for its device-to-host copies (see mm_results_wait); default 0   */
int mm_set_option(mm_engine* e, const char* name, int64_t value);

const char* mm_strerror(int status);
const char* mm_last_error(mm_engine* e); /* last CUDA error text, "" if none */
uint32_t mm_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* MM_ENGINE_H */
