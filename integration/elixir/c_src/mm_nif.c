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

/* set_max_spread(ref, w): extension knob (strategist policy S1); w < 0 restores the reference behaviour */
static ERL_NIF_TERM nif_set_max_spread(ErlNifEnv* env, int argc, const ERL_NIF_TERM argv[]) {
  engine_res* r; ErlNifSInt64 w = -1;
  (void)argc;
  if (!enif_get_resource(env, argv[0], ENGINE_T, (void**)&r) || !enif_get_int64(env, argv[1], &w))
    return enif_make_badarg(env);
  int rc = mm_set_option(r->e, "max_spread", (int64_t)w);
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
  {"set_max_spread", 2, nif_set_max_spread, 0},
};
ERL_NIF_INIT(Elixir.Matchmaking.Search.Engine, funcs, load, NULL, NULL, NULL)
