/*
 * mm_nif.c — dirty-NIF glue between the Elixir search stage and libmm_engine.so.
 *
 * NOT COMPILED IN THIS REPOSITORY'S CI: erl_nif.h is absent here (SURVEY F5).  It is the
 * binding a maintainer of OpenMatchmaking/microservice-matchmaking adds (see
 * INTEGRATION.md); it contains no logic — every function unpacks binaries, calls one
 * entry point of include/mm_engine.h and maps the status to {:ok, ...} | {:error, atom},
 * the convention of models/active_user.ex:46-66 and models/lobby_state.ex:95-103.
 * tick/enqueue/remove block on a CUDA stream sync, so they are registered
 * ERL_NIF_DIRTY_JOB_CPU_BOUND (> 1 ms rule).
 *
 * build:  cc -O2 -fPIC -shared -I$ERL_INCLUDE -I../../../include mm_nif.c \
 *            -L../../../microservice-matchmaking_b200/csrc -lmm_engine -o priv/mm_nif.so
 */
#include <erl_nif.h>
#include <stdlib.h>
#include <string.h>

#include "mm_engine.h"

static ErlNifResourceType* ENGINE_T;
typedef struct { mm_engine* e; } engine_res;

static void engine_dtor(ErlNifEnv* env, void* obj) { (void)env; mm_destroy(((engine_res*)obj)->e); }

static ERL_NIF_TERM atom(ErlNifEnv* env, const char* s) { return enif_make_atom(env, s); }
static ERL_NIF_TERM err(ErlNifEnv* env, int rc) {
  const char* a = rc == MM_E_ARG ? "badarg" : rc == MM_E_CUDA ? "cuda" : rc == MM_E_CAP ? "capacity"
                : rc == MM_E_STATE ? "state" : "unknown";
  return enif_make_tuple2(env, atom(env, "error"), atom(env, a));
}

static int load(ErlNifEnv* env, void** priv, ERL_NIF_TERM info) {
  (void)priv; (void)info;
  ENGINE_T = enif_open_resource_type(env, NULL, "mm_engine", engine_dtor, ERL_NIF_RT_CREATE, NULL);
  return ENGINE_T ? 0 : 1;
}

/* new(config_binary) — config_binary is an mm_config laid out by Matchmaking.Search.Engine.pack_config/1 */
static ERL_NIF_TERM nif_new(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  ErlNifBinary cfg;
  (void)argc;
  if (!enif_inspect_binary(env, argv[0], &cfg) || cfg.size != sizeof(mm_config)) return enif_make_badarg(env);
  mm_engine* e = NULL;
  int rc = mm_create((const mm_config*)cfg.data, &e);
  if (rc) return err(env, rc);
  engine_res* r = enif_alloc_resource(ENGINE_T, sizeof(engine_res));
  r->e = e;
  ERL_NIF_TERM t = enif_make_resource(env, r);
  enif_release_resource(r);
  return enif_make_tuple2(env, atom(env, "ok"), t);
}

/* enqueue(ref, ids :: binary(u64[]), ratings :: binary(i32[]), modes :: binary(u8[])) -> {:ok, accepted :: binary} */
static ERL_NIF_TERM nif_enqueue(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifBinary ids, rt, md;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_inspect_binary(env, argv[1], &ids) ||
      !enif_inspect_binary(env, argv[2], &rt) || !enif_inspect_binary(env, argv[3], &md))
    return enif_make_badarg(env);
  size_t n = md.size;
  if (ids.size != n * 8 || rt.size != n * 4) return enif_make_badarg(env);
  ERL_NIF_TERM out;
  unsigned char* acc = enif_make_new_binary(env, n, &out);
  int rc = mm_enqueue(r->e, (uint32_t)n, (const uint64_t*)ids.data, (const int32_t*)rt.data, md.data, NULL, acc);
  return rc ? err(env, rc) : enif_make_tuple2(env, atom(env, "ok"), out);
}

static ERL_NIF_TERM nif_remove(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifBinary ids; uint32_t removed = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_inspect_binary(env, argv[1], &ids))
    return enif_make_badarg(env);
  int rc = mm_remove(r->e, (uint32_t)(ids.size / 8), (const uint64_t*)ids.data, &removed);
  return rc ? err(env, rc) : enif_make_tuple2(env, atom(env, "ok"), enif_make_uint(env, removed));
}

static ERL_NIF_TERM nif_in_queue(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifUInt64 id; uint8_t f = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_get_uint64(env, argv[1], &id))
    return enif_make_badarg(env);
  uint64_t v = id;
  if (mm_in_queue(r->e, 1, &v, &f)) return atom(env, "false");  /* active_user.ex:39-43: errors read as false */
  return atom(env, f ? "true" : "false");
}

/* tick(ref, now_ms) -> {:ok, lobbies :: binary(mm_lobby_hdr[]), member_ids :: binary(u64[]), stats :: map} */
static ERL_NIF_TERM nif_tick(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifUInt64 now; uint32_t n = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_get_uint64(env, argv[1], &now))
    return enif_make_badarg(env);
  if (mm_pool_size(r->e, &n)) return err(env, MM_E_ARG);
  ErlNifBinary lob, mem;
  if (!enif_alloc_binary((size_t)n * sizeof(mm_lobby_hdr) + 8, &lob)) return err(env, MM_E_CAP);
  if (!enif_alloc_binary((size_t)n * 8 + 8, &mem)) { enif_release_binary(&lob); return err(env, MM_E_CAP); }
  mm_tick_stats st;
  int rc = mm_tick(r->e, now, (mm_lobby_hdr*)lob.data, n, (uint64_t*)mem.data, n, NULL, &st);
  if (rc) { enif_release_binary(&lob); enif_release_binary(&mem); return err(env, rc); }
  enif_realloc_binary(&lob, (size_t)st.n_lobbies * sizeof(mm_lobby_hdr));
  enif_realloc_binary(&mem, (size_t)st.n_matched * 8);
  ERL_NIF_TERM stats = enif_make_new_map(env);
  enif_make_map_put(env, stats, atom(env, "lobbies"), enif_make_uint(env, st.n_lobbies), &stats);
  enif_make_map_put(env, stats, atom(env, "matched"), enif_make_uint(env, st.n_matched), &stats);
  enif_make_map_put(env, stats, atom(env, "residual"), enif_make_uint(env, st.n_residual), &stats);
  enif_make_map_put(env, stats, atom(env, "dropped"), enif_make_uint(env, st.n_dead), &stats);
  enif_make_map_put(env, stats, atom(env, "device_us"), enif_make_double(env, st.device_us), &stats);
  return enif_make_tuple4(env, atom(env, "ok"), enif_make_binary(env, &lob), enif_make_binary(env, &mem), stats);
}

/* enqueue_packed(ref, handles :: binary(u32[]), keys :: binary(u16[]) [, enq_ts :: binary(u32[])])
 *   -> {:ok, accepted :: binary}   (6 B per player, 10 with the enqueue stamps mm_queue_stats measures waits from) */
static ERL_NIF_TERM nif_enqueue_packed(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifBinary hs, ks, ts;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_inspect_binary(env, argv[1], &hs) ||
      !enif_inspect_binary(env, argv[2], &ks) || hs.size != 2 * ks.size)
    return enif_make_badarg(env);
  size_t n = ks.size / 2;
  if (argc == 4 && (!enif_inspect_binary(env, argv[3], &ts) || ts.size != 4 * n)) return enif_make_badarg(env);
  ERL_NIF_TERM out;
  unsigned char* acc = enif_make_new_binary(env, n, &out);
  int rc = mm_enqueue_packed(r->e, (uint32_t)n, (const uint32_t*)hs.data, (const uint16_t*)ks.data,
                             argc == 4 ? (const uint32_t*)ts.data : NULL, acc);
  return rc ? err(env, rc) : enif_make_tuple2(env, atom(env, "ok"), out);
}

static ERL_NIF_TERM nif_remove_packed(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifBinary hs; uint32_t removed = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_inspect_binary(env, argv[1], &hs))
    return enif_make_badarg(env);
  int rc = mm_remove_packed(r->e, (uint32_t)(hs.size / 4), (const uint32_t*)hs.data, &removed);
  return rc ? err(env, rc) : enif_make_tuple2(env, atom(env, "ok"), enif_make_uint(env, removed));
}

/* tick_packed(ref, now_ms) -> {:ok, lobbies :: binary(mm_lobby_hdr[]), member_handles :: binary(u32[]), stats :: map} */
static ERL_NIF_TERM nif_tick_packed(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifUInt64 now; uint32_t n = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_get_uint64(env, argv[1], &now))
    return enif_make_badarg(env);
  if (mm_pool_size(r->e, &n)) return err(env, MM_E_ARG);
  ErlNifBinary lob, mem;
  if (!enif_alloc_binary((size_t)n * sizeof(mm_lobby_hdr) + 8, &lob)) return err(env, MM_E_CAP);
  if (!enif_alloc_binary((size_t)n * 4 + 8, &mem)) { enif_release_binary(&lob); return err(env, MM_E_CAP); }
  mm_tick_stats st;
  int rc = mm_tick_packed(r->e, now, (mm_lobby_hdr*)lob.data, n, (uint32_t*)mem.data, n, NULL, &st);
  if (rc) { enif_release_binary(&lob); enif_release_binary(&mem); return err(env, rc); }
  enif_realloc_binary(&lob, (size_t)st.n_lobbies * sizeof(mm_lobby_hdr));
  enif_realloc_binary(&mem, (size_t)st.n_matched * 4);
  ERL_NIF_TERM stats = enif_make_new_map(env);
  enif_make_map_put(env, stats, atom(env, "lobbies"), enif_make_uint(env, st.n_lobbies), &stats);
  enif_make_map_put(env, stats, atom(env, "matched"), enif_make_uint(env, st.n_matched), &stats);
  enif_make_map_put(env, stats, atom(env, "residual"), enif_make_uint(env, st.n_residual), &stats);
  enif_make_map_put(env, stats, atom(env, "device_us"), enif_make_double(env, st.device_us), &stats);
  return enif_make_tuple4(env, atom(env, "ok"), enif_make_binary(env, &lob), enif_make_binary(env, &mem), stats);
}

static ERL_NIF_TERM nif_status(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; uint32_t n = 0, a = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r)) return enif_make_badarg(env);
  mm_pool_size(r->e, &n); mm_active_size(r->e, &a);
  ERL_NIF_TERM m = enif_make_new_map(env);
  enif_make_map_put(env, m, atom(env, "message_count"), enif_make_uint(env, n), &m);
  enif_make_map_put(env, m, atom(env, "active_count"), enif_make_uint(env, a), &m);
  return enif_make_tuple2(env, atom(env, "ok"), m);
}

/* queue_stats(ref, now_ms) -> {:ok, records :: binary(mm_queue_stat[])}: one 988-byte record per (mode, group) queue,
 * mode * n_groups + group order — Search.Worker.status/0's per-queue depth plus wait histograms */
static ERL_NIF_TERM nif_queue_stats(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifUInt64 now; uint32_t n = 0; mm_queue_stat probe;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_get_uint64(env, argv[1], &now))
    return enif_make_badarg(env);
  int rc = mm_queue_stats(r->e, now, &probe, 0, &n);  /* MM_E_CAP: n = records needed */
  if (rc != MM_E_CAP) return err(env, rc ? rc : MM_E_STATE);
  ERL_NIF_TERM out;
  unsigned char* buf = enif_make_new_binary(env, (size_t)n * sizeof(mm_queue_stat), &out);
  rc = mm_queue_stats(r->e, now, (mm_queue_stat*)buf, n, &n);
  return rc ? err(env, rc) : enif_make_tuple2(env, atom(env, "ok"), out);
}

/* match_quality(ref) -> {:ok, records :: binary(mm_queue_quality[])}: one 992-byte record per (mode, group) queue,
 * mode * n_groups + group order — the rating spread and team imbalance of the last tick's lobbies (extension); an
 * empty binary while the report is void (no tick yet, a failed tick, a restore or an import since) */
static ERL_NIF_TERM nif_match_quality(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; uint32_t n = 0, n_lob = 0; mm_queue_quality probe;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r)) return enif_make_badarg(env);
  int rc = mm_match_quality(r->e, &probe, 0, &n, NULL, 0, &n_lob);  /* MM_E_CAP: n = records needed */
  if (rc != MM_E_CAP) return err(env, rc ? rc : MM_E_STATE);
  mm_queue_quality* tmp = (mm_queue_quality*)enif_alloc((size_t)n * sizeof(mm_queue_quality));
  if (!tmp) return err(env, MM_E_CAP);
  rc = mm_match_quality(r->e, tmp, n, &n, NULL, 0, &n_lob);  /* n = 0 when void */
  if (rc) { enif_free(tmp); return err(env, rc); }
  ERL_NIF_TERM out;
  unsigned char* buf = enif_make_new_binary(env, (size_t)n * sizeof(mm_queue_quality), &out);
  memcpy(buf, tmp, (size_t)n * sizeof(mm_queue_quality));
  enif_free(tmp);
  return enif_make_tuple2(env, atom(env, "ok"), out);
}

/* offtick_report(ref, source) -> {:ok, waits :: binary(mm_match_waits[]), quality :: binary(mm_queue_quality[])}:
 * one record of each per (mode, group) queue, mode * n_groups + group order — the waits and the rating quality of the
 * lobbies the last mm_party_match (source 0) or mm_widen (source 1) formed (extension); empty binaries while the report
 * is void (no such call yet, or its last one failed) */
static ERL_NIF_TERM nif_offtick_report(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; unsigned int source; uint32_t n = 0, n_lob = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_get_uint(env, argv[1], &source))
    return enif_make_badarg(env);
  int rc = mm_offtick_report(r->e, source, NULL, NULL, 0, &n, NULL, 0, &n_lob);  /* n = records, 0 when void */
  if (rc) return err(env, rc);
  ERL_NIF_TERM wout, qout;
  unsigned char* wb = enif_make_new_binary(env, (size_t)n * sizeof(mm_match_waits), &wout);
  unsigned char* qb = enif_make_new_binary(env, (size_t)n * sizeof(mm_queue_quality), &qout);
  /* nothing runs between the two calls: the engine's lock is taken per call, and only this engine's own calls change
     the report, which this process serialises */
  if (n) rc = mm_offtick_report(r->e, source, (mm_match_waits*)wb, (mm_queue_quality*)qb, n, &n, NULL, 0, &n_lob);
  return rc ? err(env, rc) : enif_make_tuple3(env, atom(env, "ok"), wout, qout);
}

/* expire_packed(ref, now_ms, max_wait_ms) -> {:ok, handles :: binary(u32[])}: search timeout (extension) — the
 * queued players who have waited >= max_wait_ms leave the pool and the active set; the caller answers each one */
static ERL_NIF_TERM nif_expire_packed(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifUInt64 now; unsigned int max_wait; uint32_t n = 0, got = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_get_uint64(env, argv[1], &now) ||
      !enif_get_uint(env, argv[2], &max_wait))
    return enif_make_badarg(env);
  if (mm_pool_size(r->e, &n)) return err(env, MM_E_ARG);
  ErlNifBinary hs;
  if (!enif_alloc_binary((size_t)n * 4 + 4, &hs)) return err(env, MM_E_CAP);
  /* cap = every resident player: the engine makes a single pass */
  int rc = mm_expire_packed(r->e, now, (uint32_t)max_wait, (uint32_t*)hs.data, NULL, n, &got);
  if (rc) { enif_release_binary(&hs); return err(env, rc); }
  enif_realloc_binary(&hs, (size_t)got * 4);
  return enif_make_tuple2(env, atom(env, "ok"), enif_make_binary(env, &hs));
}

/* export_image(ref) -> {:ok, image :: binary}: the queued players and the active set (mm_export; layout in
 * mm_engine.h).  One call: the binary is allocated at the layout's upper bound (mm_engine.h) and shrunk to the image. */
static ERL_NIF_TERM nif_export_image(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; uint32_t n = 0, a = 0; uint64_t size = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r)) return enif_make_badarg(env);
  if (mm_pool_size(r->e, &n) || mm_active_size(r->e, &a)) return err(env, MM_E_ARG);
  uint64_t bound = sizeof(mm_image_header), sec[7];
  sec[0] = 4ull * MM_MAX_GROUPS * MM_MAX_MODES; sec[1] = 8ull * n; sec[2] = sec[3] = sec[4] = 4ull * n; sec[5] = n;
  sec[6] = 8ull * a;
  for (int k = 0; k < 7; ++k) bound = (bound + sec[k] + 7) & ~7ull;
  ErlNifBinary img;
  if (!enif_alloc_binary((size_t)bound, &img)) return err(env, MM_E_CAP);
  int rc = mm_export(r->e, img.data, bound, &size);
  if (rc) { enif_release_binary(&img); return err(env, rc); }
  enif_realloc_binary(&img, (size_t)size);
  return enif_make_tuple2(env, atom(env, "ok"), enif_make_binary(env, &img));
}

/* import_image(ref, image :: binary) -> :ok | {:error, atom}: loads an image into a fresh engine (mm_import) */
static ERL_NIF_TERM nif_import_image(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifBinary img;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_inspect_binary(env, argv[1], &img))
    return enif_make_badarg(env);
  int rc = mm_import(r->e, img.data, img.size);
  return rc ? err(env, rc) : atom(env, "ok");
}

/* export_queues(ref, queues :: binary(u8[n_modes * n_groups])) -> {:ok, image :: binary}: the selected (mode, group)
 * queues leave the engine in a queue image (mm_export_queues; the players are released in the same call).  One call:
 * the binary is allocated at the layout's upper bound without an active section and shrunk to the image. */
static ERL_NIF_TERM nif_export_queues(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifBinary sel; uint32_t n = 0; uint64_t size = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_inspect_binary(env, argv[1], &sel) ||
      sel.size == 0 || sel.size > MM_MAX_GROUPS * MM_MAX_MODES)
    return enif_make_badarg(env);
  if (mm_pool_size(r->e, &n)) return err(env, MM_E_ARG);
  /* the engine reads n_modes * n_groups bytes: pad a short binary with "not selected" */
  uint8_t queues[MM_MAX_GROUPS * MM_MAX_MODES] = {0};
  memcpy(queues, sel.data, sel.size);
  uint64_t bound = sizeof(mm_image_header), sec[7];
  sec[0] = 4ull * MM_MAX_GROUPS * MM_MAX_MODES; sec[1] = 8ull * n; sec[2] = sec[3] = sec[4] = 4ull * n; sec[5] = n;
  sec[6] = 0;
  for (int k = 0; k < 7; ++k) bound = (bound + sec[k] + 7) & ~7ull;
  ErlNifBinary img;
  if (!enif_alloc_binary((size_t)bound, &img)) return err(env, MM_E_CAP);
  int rc = mm_export_queues(r->e, queues, img.data, bound, &size);
  if (rc) { enif_release_binary(&img); return err(env, rc); }
  enif_realloc_binary(&img, (size_t)size);
  return enif_make_tuple2(env, atom(env, "ok"), enif_make_binary(env, &img));
}

/* export_parties(ref, queues :: binary(u8[n_modes * n_groups]) | nil) -> {:ok, image :: binary}: the queued parties
 * of the selected queues (nil: every queue) leave the engine in a party image (mm_export_parties; released in the same
 * call).  Sized by the dry run, then written. */
static ERL_NIF_TERM nif_export_parties(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifBinary sel; uint64_t size = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r)) return enif_make_badarg(env);
  uint8_t queues[MM_MAX_GROUPS * MM_MAX_MODES] = {0};
  const uint8_t* q = NULL;
  if (enif_inspect_binary(env, argv[1], &sel)) {
    if (sel.size == 0 || sel.size > MM_MAX_GROUPS * MM_MAX_MODES) return enif_make_badarg(env);
    memcpy(queues, sel.data, sel.size);  /* padded with "not selected" */
    q = queues;
  }
  int rc = mm_export_parties(r->e, q, NULL, 0, &size);
  if (rc) return err(env, rc);
  ErlNifBinary img;
  if (!enif_alloc_binary((size_t)size, &img)) return err(env, MM_E_CAP);
  rc = mm_export_parties(r->e, q, img.data, size, &size);
  if (rc) { enif_release_binary(&img); return err(env, rc); }
  return enif_make_tuple2(env, atom(env, "ok"), enif_make_binary(env, &img));
}

/* merge_parties(ref, image :: binary, keep_seq :: boolean) -> {:ok, codes :: binary(u8[])} | {:error, atom}: merges a
 * party image (mm_merge_parties): codes per party 1 merged, 0 a member already active, 2 no queue here; keep_seq (after
 * import_image / import_regroup of the image taken at the same stop): every party keeps its sequence number. */
static ERL_NIF_TERM nif_merge_parties(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifBinary img, codes; uint32_t n = 0, got = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_inspect_binary(env, argv[1], &img))
    return enif_make_badarg(env);
  const uint32_t flags = enif_is_identical(argv[2], atom(env, "true")) ? MM_PARTY_KEEP_SEQ : 0u;
  if (img.size >= sizeof(mm_image_header)) {
    mm_image_header h;
    memcpy(&h, img.data, sizeof(h));
    n = h.n_parts < img.size ? h.n_parts : (uint32_t)img.size;  /* a corrupt count must not size the codes */
  }
  if (!enif_alloc_binary((size_t)n, &codes)) return err(env, MM_E_CAP);
  int rc = mm_merge_parties(r->e, img.data, img.size, flags, codes.data, &got);
  if (rc) { enif_release_binary(&codes); return err(env, rc); }
  return enif_make_tuple2(env, atom(env, "ok"), enif_make_binary(env, &codes));
}

/* merge_image(ref, image :: binary) -> {:ok, rejected :: binary(u32[])} | {:error, atom}: loads a queue image into
 * this running engine (mm_merge); `rejected` holds the image indices of players not queued (already active here). */
static ERL_NIF_TERM nif_merge_image(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifBinary img, rej; uint32_t cap = 0, got = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_inspect_binary(env, argv[1], &img))
    return enif_make_badarg(env);
  if (img.size >= sizeof(mm_image_header)) {
    mm_image_header h;
    memcpy(&h, img.data, sizeof(h));
    cap = h.n_players < img.size ? h.n_players : (uint32_t)img.size;  /* a corrupt count must not size the list */
  }
  if (!enif_alloc_binary((size_t)cap * 4, &rej)) return err(env, MM_E_CAP);
  int rc = mm_merge(r->e, img.data, img.size, cap, (uint32_t*)rej.data, &got);
  if (rc) { enif_release_binary(&rej); return err(env, rc); }
  enif_realloc_binary(&rej, (size_t)got * 4);
  return enif_make_tuple2(env, atom(env, "ok"), enif_make_binary(env, &rej));
}

/* import_regroup(ref, image :: binary) -> {:ok, rejected :: binary(u32[])} | {:error, atom}: loads an image written
 * under another config (groups, modes, order) into a fresh engine (mm_import_regroup); `rejected` holds the image
 * indices, ascending, of the players the engine's config has no queue for (not queued: the caller answers them). */
static ERL_NIF_TERM nif_import_regroup(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifBinary img, rej; uint32_t cap = 0, got = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_inspect_binary(env, argv[1], &img))
    return enif_make_badarg(env);
  if (img.size >= sizeof(mm_image_header)) {
    mm_image_header h;
    memcpy(&h, img.data, sizeof(h));
    cap = h.n_players < img.size ? h.n_players : (uint32_t)img.size;  /* a corrupt count must not size the list */
  }
  if (!enif_alloc_binary((size_t)cap * 4, &rej)) return err(env, MM_E_CAP);
  int rc = mm_import_regroup(r->e, img.data, img.size, cap, (uint32_t*)rej.data, &got);
  if (rc) { enif_release_binary(&rej); return err(env, rc); }
  enif_realloc_binary(&rej, (size_t)got * 4);
  return enif_make_tuple2(env, atom(env, "ok"), enif_make_binary(env, &rej));
}

/* import_regroup_many(ref, images :: [binary], keep :: binary | nil, active_image :: integer | nil) ->
 * {:ok, rejected :: binary((u32 image, u32 index)[]), n_elsewhere} | {:error, atom}: a re-cut of a sharded deployment
 * (mm_import_regroup_many): the old ranks' images, of one config, re-filed into this fresh engine; `keep` selects this
 * rank's queues (one byte per queue in queue_stats/2 record order; nil = all), `active_image` the image whose active
 * section it takes (nil = none).  `rejected` pairs name the players this config has no queue for, ascending. */
static ERL_NIF_TERM nif_import_regroup_many(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifBinary keep, out; unsigned len = 0; uint32_t cap = 0, got = 0, elsewhere = 0, act = UINT32_MAX;
  const void* bufs[64]; uint64_t sizes[64];
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_get_list_length(env, argv[1], &len) || len > 64)
    return enif_make_badarg(env);
  const int has_keep = !enif_is_identical(argv[2], atom(env, "nil"));
  if (has_keep && !enif_inspect_binary(env, argv[2], &keep)) return enif_make_badarg(env);
  if (!enif_is_identical(argv[3], atom(env, "nil")) && !enif_get_uint(env, argv[3], &act)) return enif_make_badarg(env);
  ERL_NIF_TERM head, tail = argv[1];
  for (unsigned k = 0; k < len; ++k) {
    ErlNifBinary img;
    if (!enif_get_list_cell(env, tail, &head, &tail) || !enif_inspect_binary(env, head, &img)) return enif_make_badarg(env);
    bufs[k] = img.data;
    sizes[k] = img.size;
    if (img.size >= sizeof(mm_image_header)) {
      mm_image_header h;
      memcpy(&h, img.data, sizeof(h));
      const uint32_t n = h.n_players < img.size ? h.n_players : (uint32_t)img.size;  /* a corrupt count must not size it */
      cap = cap + n < cap ? UINT32_MAX : cap + n;
    }
  }
  if (has_keep) {  /* one byte per queue: mm_queue_stats with cap 0 gives the queue count (it needs a record) */
    uint32_t n_cut = 0;
    mm_queue_stat probe;
    mm_queue_stats(r->e, 0, &probe, 0, &n_cut);
    if (keep.size != n_cut) return enif_make_badarg(env);
  }
  if (!enif_alloc_binary((size_t)cap * 8, &out)) return err(env, MM_E_CAP);
  uint32_t* img_of = (uint32_t*)enif_alloc((size_t)(cap ? cap : 1) * 4);
  if (!img_of) { enif_release_binary(&out); return err(env, MM_E_CAP); }
  uint32_t* idx = (uint32_t*)out.data;
  int rc = mm_import_regroup_many(r->e, len, bufs, sizes, has_keep ? keep.data : NULL, act, cap, img_of, idx, &got,
                                  &elsewhere);
  if (rc) { enif_free(img_of); enif_release_binary(&out); return err(env, rc); }
  for (uint32_t i = got; i-- > 0;) {  /* interleave in place, from the back: (image, index) pairs */
    const uint32_t v = idx[i];
    idx[2 * i + 1] = v;
    idx[2 * i] = img_of[i];
  }
  enif_free(img_of);
  enif_realloc_binary(&out, (size_t)got * 8);
  return enif_make_tuple3(env, atom(env, "ok"), enif_make_binary(env, &out), enif_make_uint(env, elsewhere));
}

/* import_regroup_many_parties(ref, images :: [binary], party_images :: [binary | nil], keep :: binary | nil,
 * active_image :: integer | nil) -> {:ok, rejected, n_elsewhere, party_rejected, party_elsewhere} | {:error, atom}: the
 * re-cut with the old ranks' queued parties (mm_import_regroup_many_parties); party_images[k] is the export_parties/2
 * image rank k took just before images[k] (nil or <<>> = none).  rejected / party_rejected: binaries of (u32 image,
 * u32 index) pairs, ascending — the players and the parties this config has no queue for. */
static int interleave(ErlNifBinary* out, uint32_t* img_of, uint32_t got) {
  uint32_t* idx = (uint32_t*)out->data;
  for (uint32_t i = got; i-- > 0;) {  /* (image, index) pairs, from the back */
    const uint32_t v = idx[i];
    idx[2 * i + 1] = v;
    idx[2 * i] = img_of[i];
  }
  return enif_realloc_binary(out, (size_t)got * 8);
}

static ERL_NIF_TERM nif_import_regroup_many_parties(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifBinary keep, out, pout; unsigned len = 0, plen = 0;
  uint32_t cap = 0, pcap = 0, got = 0, elsewhere = 0, act = UINT32_MAX;
  const void* bufs[64]; uint64_t sizes[64]; const void* pbufs[64]; uint64_t psizes[64];
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_get_list_length(env, argv[1], &len) || len > 64 ||
      !enif_get_list_length(env, argv[2], &plen) || plen != len)
    return enif_make_badarg(env);
  const int has_keep = !enif_is_identical(argv[3], atom(env, "nil"));
  if (has_keep && !enif_inspect_binary(env, argv[3], &keep)) return enif_make_badarg(env);
  if (!enif_is_identical(argv[4], atom(env, "nil")) && !enif_get_uint(env, argv[4], &act)) return enif_make_badarg(env);
  ERL_NIF_TERM head, tail = argv[1], ptail = argv[2];
  for (unsigned k = 0; k < len; ++k) {
    ErlNifBinary img;
    if (!enif_get_list_cell(env, tail, &head, &tail) || !enif_inspect_binary(env, head, &img)) return enif_make_badarg(env);
    bufs[k] = img.data;
    sizes[k] = img.size;
    if (img.size >= sizeof(mm_image_header)) {
      mm_image_header h;
      memcpy(&h, img.data, sizeof(h));
      const uint32_t n = h.n_players < img.size ? h.n_players : (uint32_t)img.size;  /* a corrupt count must not size it */
      cap = cap + n < cap ? UINT32_MAX : cap + n;
    }
    pbufs[k] = NULL;
    psizes[k] = 0;
    if (!enif_get_list_cell(env, ptail, &head, &ptail)) return enif_make_badarg(env);
    if (enif_is_identical(head, atom(env, "nil"))) continue;
    if (!enif_inspect_binary(env, head, &img)) return enif_make_badarg(env);
    if (img.size) { pbufs[k] = img.data; psizes[k] = img.size; }
    if (img.size >= sizeof(mm_image_header)) {
      mm_image_header h;
      memcpy(&h, img.data, sizeof(h));
      const uint32_t n = h.n_parts < img.size ? h.n_parts : (uint32_t)img.size;
      pcap = pcap + n < pcap ? UINT32_MAX : pcap + n;
    }
  }
  if (has_keep) {
    uint32_t n_cut = 0;
    mm_queue_stat probe;
    mm_queue_stats(r->e, 0, &probe, 0, &n_cut);
    if (keep.size != n_cut) return enif_make_badarg(env);
  }
  if (!enif_alloc_binary((size_t)cap * 8, &out)) return err(env, MM_E_CAP);
  if (!enif_alloc_binary((size_t)pcap * 8, &pout)) { enif_release_binary(&out); return err(env, MM_E_CAP); }
  uint32_t* img_of = (uint32_t*)enif_alloc((size_t)(cap ? cap : 1) * 4);
  uint32_t* pimg_of = (uint32_t*)enif_alloc((size_t)(pcap ? pcap : 1) * 4);
  if (!img_of || !pimg_of) {
    if (img_of) enif_free(img_of);
    if (pimg_of) enif_free(pimg_of);
    enif_release_binary(&out); enif_release_binary(&pout);
    return err(env, MM_E_CAP);
  }
  mm_recut_parties p;
  memset(&p, 0, sizeof(p));
  p.bufs = pbufs; p.n_bytes = psizes; p.cap = pcap; p.rej_image = pimg_of; p.rej_index = (uint32_t*)pout.data;
  int rc = mm_import_regroup_many_parties(r->e, len, bufs, sizes, has_keep ? keep.data : NULL, act, cap, img_of,
                                          (uint32_t*)out.data, &got, &elsewhere, &p);
  if (rc) {
    enif_free(img_of); enif_free(pimg_of); enif_release_binary(&out); enif_release_binary(&pout);
    return err(env, rc);
  }
  interleave(&out, img_of, got);
  interleave(&pout, pimg_of, p.n_rejected);
  enif_free(img_of);
  enif_free(pimg_of);
  ERL_NIF_TERM t[5] = {atom(env, "ok"), enif_make_binary(env, &out), enif_make_uint(env, elsewhere),
                       enif_make_binary(env, &pout), enif_make_uint(env, p.n_elsewhere)};
  return enif_make_tuple_from_array(env, t, 5);
}

/* seq_next(ref) -> {:ok, seq}: the enqueue sequence number the next offered player will get (mm_seq_next) */
static ERL_NIF_TERM nif_seq_next(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; uint32_t s = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r)) return enif_make_badarg(env);
  int rc = mm_seq_next(r->e, &s);
  return rc ? err(env, rc) : enif_make_tuple2(env, atom(env, "ok"), enif_make_uint(env, s));
}

/* qsort of (age, index) pairs by age: the age (seq - seq_next mod 2^32) is computed into the key first */
static int rq_cmp(const void* a, const void* b) {
  const uint32_t ux = *(const uint32_t*)a, uy = *(const uint32_t*)b;
  return ux < uy ? -1 : ux > uy;
}
/* requeue(ref, handles :: binary(u32[]), ratings :: binary(i32[]), modes :: binary(u8[]), enq_ts :: binary(u32[]),
 * seq :: binary(u32[])) -> {:ok, codes :: binary(u8[])} (1 requeued, 0 still queued, 4 gone; in the caller's order):
 * the members of a lobby that did not start go back into their queue at their enqueue position (mm_requeue).  The
 * entries are sorted by age here. */
static ERL_NIF_TERM nif_requeue(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifBinary hs, rt, md, ts, sq, codes; uint32_t got = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_inspect_binary(env, argv[1], &hs) ||
      !enif_inspect_binary(env, argv[2], &rt) || !enif_inspect_binary(env, argv[3], &md) ||
      !enif_inspect_binary(env, argv[4], &ts) || !enif_inspect_binary(env, argv[5], &sq))
    return enif_make_badarg(env);
  const size_t n = hs.size / 4;
  if (hs.size % 4 || rt.size != 4 * n || md.size != n || ts.size != 4 * n || sq.size != 4 * n) return enif_make_badarg(env);
  if (!enif_alloc_binary(n, &codes)) return err(env, MM_E_CAP);
  if (n == 0) return enif_make_tuple2(env, atom(env, "ok"), enif_make_binary(env, &codes));
  uint32_t* key = enif_alloc(n * 8);  /* (age, index) pairs */
  uint64_t* id = enif_alloc(n * 8);
  int32_t* rating = enif_alloc(n * 4);
  uint8_t* mode = enif_alloc(n);
  uint32_t *stamp = enif_alloc(n * 4), *seq = enif_alloc(n * 4);
  uint8_t* out = enif_alloc(n);
  int rc = MM_E_CAP;
  uint32_t seq_next = 0;
  if (key && id && rating && mode && stamp && seq && out && !(rc = mm_seq_next(r->e, &seq_next))) {
    for (size_t i = 0; i < n; ++i) {
      uint32_t s;
      memcpy(&s, sq.data + 4 * i, 4);
      key[2 * i] = s - seq_next;
      key[2 * i + 1] = (uint32_t)i;
    }
    qsort(key, n, 8, rq_cmp);
    for (size_t k = 0; k < n; ++k) {
      const uint32_t i = key[2 * k + 1];
      uint32_t h;
      memcpy(&h, hs.data + 4 * i, 4); id[k] = h;
      memcpy(&rating[k], rt.data + 4 * i, 4); mode[k] = md.data[i];
      memcpy(&stamp[k], ts.data + 4 * i, 4); memcpy(&seq[k], sq.data + 4 * i, 4);
    }
    rc = mm_requeue(r->e, (uint32_t)n, id, rating, mode, stamp, seq, out, &got);
    if (!rc)
      for (size_t k = 0; k < n; ++k) codes.data[key[2 * k + 1]] = out[k];
  }
  enif_free(key); enif_free(id); enif_free(rating); enif_free(mode); enif_free(stamp); enif_free(seq); enif_free(out);
  if (rc) { enif_release_binary(&codes); return err(env, rc); }
  return enif_make_tuple2(env, atom(env, "ok"), enif_make_binary(env, &codes));
}

/* backfill(ref, requests :: binary(mm_backfill_req[]: mode u8, group u8, 0 :: u16, count u32, target i32, window i32))
 * -> {:ok, n_taken :: binary(u32[]), handles :: binary(u32[])}: the open slots of running lobbies filled from their
 * queues, nearest rating first (mm_backfill); handles holds request 0's players, then request 1's, ...  The member
 * buffer is sized from the dry run's total (member_cap = 0). */
static ERL_NIF_TERM nif_backfill(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifBinary rq, taken, hs; uint32_t total = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_inspect_binary(env, argv[1], &rq))
    return enif_make_badarg(env);
  if (rq.size % sizeof(mm_backfill_req)) return enif_make_badarg(env);
  const uint32_t n = (uint32_t)(rq.size / sizeof(mm_backfill_req));
  mm_backfill_req* req = enif_alloc(rq.size + 1);
  if (!req || !enif_alloc_binary(4 * (size_t)n, &taken)) { enif_free(req); return err(env, MM_E_CAP); }
  memcpy(req, rq.data, rq.size);
  int rc = mm_backfill(r->e, n, req, (uint32_t*)taken.data, NULL, 0, &total);  /* the dry run: counts only */
  if (rc == MM_E_CAP || rc == MM_OK) {
    uint64_t* id = enif_alloc(8 * (size_t)total + 8);
    if (!id || !enif_alloc_binary(4 * (size_t)total, &hs)) rc = MM_E_CAP;
    else {
      rc = mm_backfill(r->e, n, req, (uint32_t*)taken.data, id, total, &total);
      if (rc) enif_release_binary(&hs);
      else for (uint32_t k = 0; k < total; ++k) { const uint32_t h = (uint32_t)id[k]; memcpy(hs.data + 4 * (size_t)k, &h, 4); }
    }
    enif_free(id);
  }
  enif_free(req);
  if (rc) { enif_release_binary(&taken); return err(env, rc); }
  return enif_make_tuple3(env, atom(env, "ok"), enif_make_binary(env, &taken), enif_make_binary(env, &hs));
}

/* backfill_party(ref, requests :: binary(mm_backfill_req[]), room :: binary(u16[]))
 * -> {:ok, filled :: binary(u16[]), handles :: binary(u32[])}: the open team slots of running lobbies filled with whole
 * queued parties, then the nearest solos (mm_backfill_party); room holds every request's open slots per team (teams of
 * its mode entries each, count = their sum), filled the members each team received, handles request 0's members team
 * by team, then request 1's, ...  The member buffer is sized from the dry run's total (member_cap = 0). */
static ERL_NIF_TERM nif_backfill_party(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifBinary rq, rm, filled, hs; uint32_t total = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_inspect_binary(env, argv[1], &rq) ||
      !enif_inspect_binary(env, argv[2], &rm))
    return enif_make_badarg(env);
  if (rq.size % sizeof(mm_backfill_req) || rm.size % 2) return enif_make_badarg(env);
  const uint32_t n = (uint32_t)(rq.size / sizeof(mm_backfill_req));
  mm_backfill_req* req = enif_alloc(rq.size + 1);
  uint16_t* room = enif_alloc(rm.size + 2);
  uint32_t* taken = enif_alloc(4 * (size_t)n + 4);
  if (!req || !room || !taken || !enif_alloc_binary(rm.size, &filled)) {
    enif_free(req); enif_free(room); enif_free(taken);
    return err(env, MM_E_CAP);
  }
  memcpy(req, rq.data, rq.size);
  memcpy(room, rm.data, rm.size);
  /* the dry run: counts only.  room must hold teams_of(mode) entries per request, as mm_backfill_party reads them;
   * Pool.backfill_teams/1 checks every request's list against its mode before the call. */
  int rc = mm_backfill_party(r->e, n, req, room, (uint16_t*)filled.data, taken, NULL, 0, &total);
  if (rc == MM_E_CAP || rc == MM_OK) {
    uint64_t* id = enif_alloc(8 * (size_t)total + 8);
    if (!id || !enif_alloc_binary(4 * (size_t)total, &hs)) rc = MM_E_CAP;
    else {
      rc = mm_backfill_party(r->e, n, req, room, (uint16_t*)filled.data, taken, id, total, &total);
      if (rc) enif_release_binary(&hs);
      else for (uint32_t k = 0; k < total; ++k) { const uint32_t h = (uint32_t)id[k]; memcpy(hs.data + 4 * (size_t)k, &h, 4); }
    }
    enif_free(id);
  }
  enif_free(req); enif_free(room); enif_free(taken);
  if (rc) { enif_release_binary(&filled); return err(env, rc); }
  return enif_make_tuple3(env, atom(env, "ok"), enif_make_binary(env, &filled), enif_make_binary(env, &hs));
}

/* widen(ref, now :: u64, rules :: binary(mm_widen_rule[n_modes * n_groups]))
 *   -> {:ok, lobbies :: binary(mm_lobby_hdr[]), handles :: binary(u32[])}: lobbies formed around the players who waited longest, each in a rating window that grows
 * with its wait (mm_widen).  badarg unless the binary holds exactly one rule per (mode, group) queue.  The buffers are
 * sized from the dry run's counts (zero capacities). */
static ERL_NIF_TERM nif_widen(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifUInt64 now; ErlNifBinary rb, lb, hs; mm_widen_stats st; uint32_t nq = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_get_uint64(env, argv[1], &now) ||
      !enif_inspect_binary(env, argv[2], &rb))
    return enif_make_badarg(env);
  mm_lobby_candidates(r->e, NULL, 0, &nq);  /* cap 0: only the number of queues; mm_widen reads one rule for each */
  if (rb.size != (size_t)nq * sizeof(mm_widen_rule)) return enif_make_badarg(env);
  mm_widen_rule* rules = enif_alloc(rb.size + 1);
  if (!rules) return err(env, MM_E_CAP);
  memcpy(rules, rb.data, rb.size);
  int rc = mm_widen(r->e, now, rules, NULL, 0, NULL, 0, &st);  /* the dry run: counts only */
  if (rc == MM_E_CAP || rc == MM_OK) {
    const uint32_t nl = st.n_lobbies, nm = st.n_matched;
    uint64_t* id = enif_alloc(8 * (size_t)nm + 8);
    if (!id || !enif_alloc_binary(sizeof(mm_lobby_hdr) * (size_t)nl, &lb)) rc = MM_E_CAP;
    else if (!enif_alloc_binary(4 * (size_t)nm, &hs)) { enif_release_binary(&lb); rc = MM_E_CAP; }
    else {
      rc = mm_widen(r->e, now, rules, (mm_lobby_hdr*)lb.data, nl, id, nm, &st);
      if (rc) { enif_release_binary(&lb); enif_release_binary(&hs); }
      else
        for (uint32_t k = 0; k < nm; ++k) { const uint32_t h = (uint32_t)id[k]; memcpy(hs.data + 4 * (size_t)k, &h, 4); }
    }
    enif_free(id);
  }
  enif_free(rules);
  if (rc) return err(env, rc);
  return enif_make_tuple3(env, atom(env, "ok"), enif_make_binary(env, &lb), enif_make_binary(env, &hs));
}

/* enqueue_party(ref, sizes :: binary(u8[]), handles :: binary(u32[]), ratings :: binary(i32[]), modes :: binary(u8[]),
 * enq_ts :: binary(u32[])) -> {:ok, codes :: binary(u8[])}: party j's members are the next sizes[j] handles and ratings
 * (mm_enqueue_party); codes 1 queued, 0 a member already queued, 2 invalid, 3 the party table is full.  badarg unless
 * the sizes add up to the handles and ratings and every per-party binary has one entry per party. */
static ERL_NIF_TERM nif_enqueue_party(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifBinary sb, hb, rtb, mb, tb, out;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_inspect_binary(env, argv[1], &sb) ||
      !enif_inspect_binary(env, argv[2], &hb) || !enif_inspect_binary(env, argv[3], &rtb) ||
      !enif_inspect_binary(env, argv[4], &mb) || !enif_inspect_binary(env, argv[5], &tb))
    return enif_make_badarg(env);
  const uint32_t n = (uint32_t)sb.size;
  size_t m = 0;
  for (uint32_t j = 0; j < n; ++j) m += sb.data[j];
  if (hb.size != 4 * m || rtb.size != 4 * m || mb.size != n || tb.size != 4 * (size_t)n) return enif_make_badarg(env);
  uint64_t* id = enif_alloc(8 * m + 8);
  if (!id || !enif_alloc_binary(n, &out)) { enif_free(id); return err(env, MM_E_CAP); }
  for (size_t k = 0; k < m; ++k) { uint32_t h; memcpy(&h, hb.data + 4 * k, 4); id[k] = h; }
  const int rc = mm_enqueue_party(r->e, n, sb.data, id, (const int32_t*)rtb.data, mb.data, (const uint32_t*)tb.data,
                                  out.data);
  enif_free(id);
  if (rc) { enif_release_binary(&out); return err(env, rc); }
  return enif_make_tuple2(env, atom(env, "ok"), enif_make_binary(env, &out));
}

/* requeue_party(ref, sizes :: binary(u8[]), handles :: binary(u32[]), ratings :: binary(i32[]), modes :: binary(u8[]),
 * enq_ts :: binary(u32[]), seq :: binary(u32[])) -> {:ok, codes :: binary(u8[])} (1 requeued, 0 a member still
 * queued, 4 a member gone; in the caller's order): the parties of a lobby that did not start go back into the party
 * table at their age position (mm_requeue_party).  Party j's members are the next sizes[j] handles and ratings; the
 * parties are sorted by age here.  badarg unless the sizes add up to the handles and ratings and every per-party
 * binary has one entry per party. */
static ERL_NIF_TERM nif_requeue_party(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifBinary sb, hb, rtb, mb, tb, qb, codes; uint32_t got = 0, seq_next = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_inspect_binary(env, argv[1], &sb) ||
      !enif_inspect_binary(env, argv[2], &hb) || !enif_inspect_binary(env, argv[3], &rtb) ||
      !enif_inspect_binary(env, argv[4], &mb) || !enif_inspect_binary(env, argv[5], &tb) ||
      !enif_inspect_binary(env, argv[6], &qb))
    return enif_make_badarg(env);
  const size_t n = sb.size;
  size_t m = 0;
  for (size_t j = 0; j < n; ++j) m += sb.data[j];
  if (hb.size != 4 * m || rtb.size != 4 * m || mb.size != n || tb.size != 4 * n || qb.size != 4 * n)
    return enif_make_badarg(env);
  if (!enif_alloc_binary(n, &codes)) return err(env, MM_E_CAP);
  if (n == 0) return enif_make_tuple2(env, atom(env, "ok"), enif_make_binary(env, &codes));
  uint32_t* key = enif_alloc(n * 8);  /* (age, index) pairs */
  uint32_t* off = enif_alloc(n * 4);  /* first member of party i in the caller's order */
  uint8_t *size = enif_alloc(n), *mode = enif_alloc(n), *out = enif_alloc(n);
  uint32_t *stamp = enif_alloc(n * 4), *seq = enif_alloc(n * 4);
  uint64_t* id = enif_alloc(m * 8 + 8);
  int32_t* rating = enif_alloc(m * 4 + 4);
  int rc = MM_E_CAP;
  if (key && off && size && mode && out && stamp && seq && id && rating && !(rc = mm_seq_next(r->e, &seq_next))) {
    for (size_t i = 0, o = 0; i < n; o += sb.data[i], ++i) {
      uint32_t q;
      memcpy(&q, qb.data + 4 * i, 4);
      key[2 * i] = q - seq_next;
      key[2 * i + 1] = (uint32_t)i;
      off[i] = (uint32_t)o;
    }
    qsort(key, n, 8, rq_cmp);
    for (size_t k = 0, o = 0; k < n; ++k) {
      const uint32_t i = key[2 * k + 1];
      size[k] = sb.data[i]; mode[k] = mb.data[i];
      memcpy(&stamp[k], tb.data + 4 * i, 4); memcpy(&seq[k], qb.data + 4 * i, 4);
      for (uint32_t x = 0; x < size[k]; ++x, ++o) {
        uint32_t h;
        memcpy(&h, hb.data + 4 * ((size_t)off[i] + x), 4); id[o] = h;
        memcpy(&rating[o], rtb.data + 4 * ((size_t)off[i] + x), 4);
      }
    }
    rc = mm_requeue_party(r->e, (uint32_t)n, size, id, rating, mode, stamp, seq, out, &got);
    if (!rc)
      for (size_t k = 0; k < n; ++k) codes.data[key[2 * k + 1]] = out[k];
  }
  enif_free(key); enif_free(off); enif_free(size); enif_free(mode); enif_free(out); enif_free(stamp); enif_free(seq);
  enif_free(id); enif_free(rating);
  if (rc) { enif_release_binary(&codes); return err(env, rc); }
  return enif_make_tuple2(env, atom(env, "ok"), enif_make_binary(env, &codes));
}

/* party_match(ref, now :: u64, rules :: binary(mm_widen_rule[n_modes * n_groups]))
 *   -> {:ok, lobbies :: binary(mm_lobby_hdr[]), handles :: binary(u32[])}: lobbies around the parties that waited
 * longest, each party whole on one team (mm_party_match).  badarg unless the binary holds exactly one rule per (mode,
 * group) queue.  The buffers are sized from the dry run's counts (zero capacities). */
static ERL_NIF_TERM nif_party_match(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifUInt64 now; ErlNifBinary rb, lb, hs; mm_party_stats st; uint32_t nq = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_get_uint64(env, argv[1], &now) ||
      !enif_inspect_binary(env, argv[2], &rb))
    return enif_make_badarg(env);
  mm_lobby_candidates(r->e, NULL, 0, &nq);
  if (rb.size != (size_t)nq * sizeof(mm_widen_rule)) return enif_make_badarg(env);
  mm_widen_rule* rules = enif_alloc(rb.size + 1);
  if (!rules) return err(env, MM_E_CAP);
  memcpy(rules, rb.data, rb.size);
  int rc = mm_party_match(r->e, now, rules, NULL, 0, NULL, 0, &st);  /* the dry run: counts only */
  if (rc == MM_E_CAP || rc == MM_OK) {
    const uint32_t nl = st.n_lobbies, nm = st.n_matched;
    uint64_t* id = enif_alloc(8 * (size_t)nm + 8);
    if (!id || !enif_alloc_binary(sizeof(mm_lobby_hdr) * (size_t)nl, &lb)) rc = MM_E_CAP;
    else if (!enif_alloc_binary(4 * (size_t)nm, &hs)) { enif_release_binary(&lb); rc = MM_E_CAP; }
    else {
      rc = mm_party_match(r->e, now, rules, (mm_lobby_hdr*)lb.data, nl, id, nm, &st);
      if (rc) { enif_release_binary(&lb); enif_release_binary(&hs); }
      else
        for (uint32_t k = 0; k < nm; ++k) { const uint32_t h = (uint32_t)id[k]; memcpy(hs.data + 4 * (size_t)k, &h, 4); }
    }
    enif_free(id);
  }
  enif_free(rules);
  if (rc) return err(env, rc);
  return enif_make_tuple3(env, atom(env, "ok"), enif_make_binary(env, &lb), enif_make_binary(env, &hs));
}

/* locate(ref, now :: u64, handles :: binary(u32[])) -> {:ok, records :: binary(mm_player_status[])}: where each
 * player's search stands (mm_locate): state, queue, wait at `now`, players ahead and queue depth, and the lobby ordinal
 * / member index the next tick gives it (0xFFFFFFFF: it stays queued). */
static ERL_NIF_TERM nif_locate(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifUInt64 now; ErlNifBinary hb, out;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_get_uint64(env, argv[1], &now) ||
      !enif_inspect_binary(env, argv[2], &hb) || hb.size % 4)
    return enif_make_badarg(env);
  const uint32_t n = (uint32_t)(hb.size / 4);
  uint64_t* id = enif_alloc(8 * (size_t)n + 8);
  if (!id || !enif_alloc_binary(sizeof(mm_player_status) * (size_t)n, &out)) { enif_free(id); return err(env, MM_E_CAP); }
  for (uint32_t k = 0; k < n; ++k) { uint32_t h; memcpy(&h, hb.data + 4 * (size_t)k, 4); id[k] = h; }
  const int rc = mm_locate(r->e, now, n, id, (mm_player_status*)out.data);
  enif_free(id);
  if (rc) { enif_release_binary(&out); return err(env, rc); }
  return enif_make_tuple2(env, atom(env, "ok"), enif_make_binary(env, &out));
}

/* party_queue_stats(ref, now_ms) -> {:ok, records :: binary(mm_party_queue_stat[])}: one 560-byte record per (mode,
 * group) queue, queue_stats/2 record order — the queued parties, their members, the longest party wait and the wait and
 * size histograms (mm_party_queue_stats, extension) */
static ERL_NIF_TERM nif_party_queue_stats(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifUInt64 now; uint32_t n = 0; mm_party_queue_stat probe;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_get_uint64(env, argv[1], &now))
    return enif_make_badarg(env);
  int rc = mm_party_queue_stats(r->e, now, &probe, 0, &n);  /* MM_E_CAP: n = records needed */
  if (rc != MM_E_CAP) return err(env, rc ? rc : MM_E_STATE);
  ERL_NIF_TERM out;
  unsigned char* buf = enif_make_new_binary(env, (size_t)n * sizeof(mm_party_queue_stat), &out);
  rc = mm_party_queue_stats(r->e, now, (mm_party_queue_stat*)buf, n, &n);
  return rc ? err(env, rc) : enif_make_tuple2(env, atom(env, "ok"), out);
}

/* party_locate(ref, now :: u64, rules :: binary(mm_widen_rule[n_modes * n_groups]), handles :: binary(u32[]))
 *   -> {:ok, records :: binary(mm_party_member_status[])}: where each party member's search stands and the lobby
 * ordinal / member index the next party_match(now, rules) gives it (0xFFFFFFFF: its party stays queued;
 * mm_party_locate, extension).  badarg unless the rules binary holds exactly one rule per (mode, group) queue. */
static ERL_NIF_TERM nif_party_locate(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifUInt64 now; ErlNifBinary rb, hb, out; uint32_t nq = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_get_uint64(env, argv[1], &now) ||
      !enif_inspect_binary(env, argv[2], &rb) || !enif_inspect_binary(env, argv[3], &hb) || hb.size % 4)
    return enif_make_badarg(env);
  mm_lobby_candidates(r->e, NULL, 0, &nq);
  if (rb.size != (size_t)nq * sizeof(mm_widen_rule)) return enif_make_badarg(env);
  const uint32_t n = (uint32_t)(hb.size / 4);
  mm_widen_rule* rules = enif_alloc(rb.size + 1);
  uint64_t* id = enif_alloc(8 * (size_t)n + 8);
  if (!rules || !id || !enif_alloc_binary(sizeof(mm_party_member_status) * (size_t)n, &out)) {
    enif_free(rules); enif_free(id);
    return err(env, MM_E_CAP);
  }
  memcpy(rules, rb.data, rb.size);
  for (uint32_t k = 0; k < n; ++k) { uint32_t h; memcpy(&h, hb.data + 4 * (size_t)k, 4); id[k] = h; }
  const int rc = mm_party_locate(r->e, now, rules, n, id, (mm_party_member_status*)out.data);
  enif_free(rules);
  enif_free(id);
  if (rc) { enif_release_binary(&out); return err(env, rc); }
  return enif_make_tuple2(env, atom(env, "ok"), enif_make_binary(env, &out));
}

/* set_lobby_budget(ref, per_queue :: binary(u32[n_modes * n_groups]) | <<>>, per_mode :: binary(u32[n_modes]) | <<>>)
 * -> :ok: lobbies every queue / every mode may emit per tick from the next tick on (mm_set_lobby_budget); an empty
 * binary = no limit, 0xFFFFFFFF in an entry = no limit for it.  The engine reads n_modes * n_groups / n_modes entries:
 * any other non-empty length is a badarg (status/1 gives neither count, so the lengths come from queue_stats). */
static ERL_NIF_TERM nif_set_lobby_budget(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifBinary pq, pm; uint32_t nq = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_inspect_binary(env, argv[1], &pq) ||
      !enif_inspect_binary(env, argv[2], &pm))
    return enif_make_badarg(env);
  mm_lobby_candidates(r->e, NULL, 0, &nq);  /* cap 0: only the number of queues */
  if ((pq.size && pq.size != (size_t)nq * 4) || pm.size % 4 || pm.size > 4 * MM_MAX_MODES || (pm.size && nq % (pm.size / 4)))
    return enif_make_badarg(env);
  uint32_t q[MM_MAX_GROUPS * MM_MAX_MODES], m[MM_MAX_MODES];
  memcpy(q, pq.data, pq.size);
  memcpy(m, pm.data, pm.size);
  int rc = mm_set_lobby_budget(r->e, pq.size ? q : NULL, pm.size ? m : NULL);
  return rc ? err(env, rc) : atom(env, "ok");
}

/* lobby_budget_report(ref) -> {:ok, candidates :: binary(u32[]), emitted :: binary(u32[])} per queue, of the last
 * completed tick (mm_lobby_budget_report); lobby_candidates(ref) -> {:ok, binary(u32[])} for the pool as it is now,
 * budgets ignored, nothing changes (mm_lobby_candidates). */
static ERL_NIF_TERM nif_lobby_budget_report(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifBinary c, a; uint32_t n = 0;
  const uint32_t cap = MM_MAX_GROUPS * MM_MAX_MODES;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r)) return enif_make_badarg(env);
  if (!enif_alloc_binary((size_t)cap * 4, &c)) return err(env, MM_E_CAP);
  if (!enif_alloc_binary((size_t)cap * 4, &a)) { enif_release_binary(&c); return err(env, MM_E_CAP); }
  int rc = mm_lobby_budget_report(r->e, (uint32_t*)c.data, (uint32_t*)a.data, cap, &n);
  if (rc) { enif_release_binary(&c); enif_release_binary(&a); return err(env, rc); }
  enif_realloc_binary(&c, (size_t)n * 4);
  enif_realloc_binary(&a, (size_t)n * 4);
  return enif_make_tuple3(env, atom(env, "ok"), enif_make_binary(env, &c), enif_make_binary(env, &a));
}
/* set_offtick_budget(ref, source, per_queue, per_mode) -> :ok: the lobby budget of mm_party_match (source 0) or mm_widen
 * (source 1) from its next call on (mm_set_offtick_budget); binaries as in set_lobby_budget.
 * offtick_budget_report(ref, source) -> {:ok, candidates, emitted} (binary(u32[]) per queue) of the source's last call
 * that returned MM_OK or was a dry run (mm_offtick_budget_report). */
static ERL_NIF_TERM nif_set_offtick_budget(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; unsigned int source; ErlNifBinary pq, pm; uint32_t nq = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_get_uint(env, argv[1], &source) ||
      !enif_inspect_binary(env, argv[2], &pq) || !enif_inspect_binary(env, argv[3], &pm))
    return enif_make_badarg(env);
  mm_lobby_candidates(r->e, NULL, 0, &nq);  /* cap 0: only the number of queues */
  if ((pq.size && pq.size != (size_t)nq * 4) || pm.size % 4 || pm.size > 4 * MM_MAX_MODES || (pm.size && nq % (pm.size / 4)))
    return enif_make_badarg(env);
  uint32_t q[MM_MAX_GROUPS * MM_MAX_MODES], m[MM_MAX_MODES];
  memcpy(q, pq.data, pq.size);
  memcpy(m, pm.data, pm.size);
  int rc = mm_set_offtick_budget(r->e, source, pq.size ? q : NULL, pm.size ? m : NULL);
  return rc ? err(env, rc) : atom(env, "ok");
}
static ERL_NIF_TERM nif_offtick_budget_report(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; unsigned int source; ErlNifBinary c, a; uint32_t n = 0;
  const uint32_t cap = MM_MAX_GROUPS * MM_MAX_MODES;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_get_uint(env, argv[1], &source))
    return enif_make_badarg(env);
  if (!enif_alloc_binary((size_t)cap * 4, &c)) return err(env, MM_E_CAP);
  if (!enif_alloc_binary((size_t)cap * 4, &a)) { enif_release_binary(&c); return err(env, MM_E_CAP); }
  int rc = mm_offtick_budget_report(r->e, source, (uint32_t*)c.data, (uint32_t*)a.data, cap, &n);
  if (rc) { enif_release_binary(&c); enif_release_binary(&a); return err(env, rc); }
  enif_realloc_binary(&c, (size_t)n * 4);
  enif_realloc_binary(&a, (size_t)n * 4);
  return enif_make_tuple3(env, atom(env, "ok"), enif_make_binary(env, &c), enif_make_binary(env, &a));
}
static ERL_NIF_TERM nif_lobby_candidates(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifBinary c; uint32_t n = 0;
  const uint32_t cap = MM_MAX_GROUPS * MM_MAX_MODES;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r)) return enif_make_badarg(env);
  if (!enif_alloc_binary((size_t)cap * 4, &c)) return err(env, MM_E_CAP);
  int rc = mm_lobby_candidates(r->e, (uint32_t*)c.data, cap, &n);
  if (rc) { enif_release_binary(&c); return err(env, rc); }
  enif_realloc_binary(&c, (size_t)n * 4);
  return enif_make_tuple2(env, atom(env, "ok"), enif_make_binary(env, &c));
}

/* set_max_spread(ref, w): extension knob (strategist policy S1); w < 0 restores the reference behaviour */
static ERL_NIF_TERM nif_set_max_spread(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifSInt64 w = -1;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_get_int64(env, argv[1], &w))
    return enif_make_badarg(env);
  int rc = mm_set_option(r->e, "max_spread", (int64_t)w);
  return rc ? err(env, rc) : atom(env, "ok");
}

/* set_team_balance(ref, mask): extension knob (balanced teams); bit m splits every lobby of mode m into the two teams
 * with the least rating difference, 0 = off; a mask naming a mode that cannot be balanced returns the engine error */
static ERL_NIF_TERM nif_set_team_balance(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifSInt64 mask = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_get_int64(env, argv[1], &mask))
    return enif_make_badarg(env);
  int rc = mm_set_option(r->e, "team_balance", (int64_t)mask);
  return rc ? err(env, rc) : atom(env, "ok");
}

/* set_party_balance(ref, mask): extension knob (balanced party lobbies); bit m splits every party_match lobby of mode
 * m into its most even teams that keep every party whole, 0 = off; a mask naming a mode that cannot be balanced
 * returns the engine error */
static ERL_NIF_TERM nif_set_party_balance(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifSInt64 mask = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_get_int64(env, argv[1], &mask))
    return enif_make_badarg(env);
  int rc = mm_set_option(r->e, "party_balance", (int64_t)mask);
  return rc ? err(env, rc) : atom(env, "ok");
}

/* set_party_capacity(ref, members): extension knob (parties); how many party members the engine holds */
static ERL_NIF_TERM nif_set_party_capacity(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifSInt64 cap = 0;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_get_int64(env, argv[1], &cap))
    return enif_make_badarg(env);
  int rc = mm_set_option(r->e, "party_capacity", (int64_t)cap);
  return rc ? err(env, rc) : atom(env, "ok");
}

static ErlNifFunc funcs[] = {
  {"new", 1, nif_new, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"enqueue", 4, nif_enqueue, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"remove", 2, nif_remove, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"in_queue?", 2, nif_in_queue, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"tick", 2, nif_tick, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"enqueue_packed", 3, nif_enqueue_packed, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"enqueue_packed", 4, nif_enqueue_packed, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"remove_packed", 2, nif_remove_packed, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"tick_packed", 2, nif_tick_packed, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"status", 1, nif_status, 0},
  {"queue_stats", 2, nif_queue_stats, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"match_quality", 1, nif_match_quality, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"offtick_report", 2, nif_offtick_report, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"expire_packed", 3, nif_expire_packed, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"export_image", 1, nif_export_image, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"import_image", 2, nif_import_image, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"export_queues", 2, nif_export_queues, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"merge_image", 2, nif_merge_image, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"export_parties", 2, nif_export_parties, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"merge_parties", 3, nif_merge_parties, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"import_regroup", 2, nif_import_regroup, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"import_regroup_many", 4, nif_import_regroup_many, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"import_regroup_many_parties", 5, nif_import_regroup_many_parties, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"requeue", 6, nif_requeue, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"requeue_party", 7, nif_requeue_party, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"backfill", 2, nif_backfill, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"backfill_party", 3, nif_backfill_party, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"widen", 3, nif_widen, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"enqueue_party", 6, nif_enqueue_party, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"party_match", 3, nif_party_match, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"set_party_capacity", 2, nif_set_party_capacity, 0},
  {"locate", 3, nif_locate, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"party_queue_stats", 2, nif_party_queue_stats, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"party_locate", 4, nif_party_locate, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"seq_next", 1, nif_seq_next, 0},
  {"set_max_spread", 2, nif_set_max_spread, 0},
  {"set_team_balance", 2, nif_set_team_balance, 0},
  {"set_party_balance", 2, nif_set_party_balance, 0},
  {"set_lobby_budget", 3, nif_set_lobby_budget, 0},
  {"lobby_budget_report", 1, nif_lobby_budget_report, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"lobby_candidates", 1, nif_lobby_candidates, ERL_NIF_DIRTY_JOB_CPU_BOUND},
  {"set_offtick_budget", 4, nif_set_offtick_budget, 0},
  {"offtick_budget_report", 2, nif_offtick_budget_report, ERL_NIF_DIRTY_JOB_CPU_BOUND},
};
ERL_NIF_INIT(Elixir.Matchmaking.Search.Engine, funcs, load, NULL, NULL, NULL)
