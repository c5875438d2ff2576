"""Search timeout (mm_expire): the expired set against a numpy restatement over the test's own inputs (live queued
players — not removed, taken or matched — whose (int32)(now - ts), clamped at 0, is >= max_wait), expire against a
twin engine that removes the same ids, the refused call, the packed form, restore, and the SearchPool's error
responses on the CPU with an Engine double."""
import ctypes as C
import importlib
import json

import numpy as np
import pytest

from .fakes import FakeBroker, OracleEngine

sw = importlib.import_module("microservice-matchmaking_b200.search_worker")
eng_mod = importlib.import_module("microservice-matchmaking_b200.engine")
abi = importlib.import_module("microservice-matchmaking_b200.abi")

ARRIVAL, RATING = 0, 1
QUEUED, DEAD, GONE = 0, 1, 2


def r_wait(now, ts):
    d = (np.uint64(int(now) & 0xFFFFFFFF) - np.asarray(ts, np.uint64)) & np.uint64(0xFFFFFFFF)
    w = d.astype(np.int64)
    return np.where(w >= 2 ** 31, 0, w)


class Model:
    """Every entry the engine was given: id, stamp, enqueue sequence number and state."""

    def __init__(self, dedupe=True):
        self.dedupe = dedupe
        self.id = np.zeros(0, np.uint64); self.ts = np.zeros(0, np.uint32); self.seq = np.zeros(0, np.uint32)
        self.state = np.zeros(0, np.uint8)
        self.seq_next = 0

    def enqueue(self, ids, ts, acc):
        k = acc == 1
        seq = (self.seq_next + np.arange(len(ids), dtype=np.int64)).astype(np.uint32)
        self.seq_next += len(ids)
        self.id = np.concatenate([self.id, ids[k]]); self.ts = np.concatenate([self.ts, ts[k]])
        self.seq = np.concatenate([self.seq, seq[k]]); self.state = np.concatenate([self.state, np.zeros(k.sum(), np.uint8)])

    def remove(self, ids):  # mm_remove / mm_take on a dedupe engine
        self.state[np.isin(self.id, ids) & (self.state == QUEUED)] = DEAD

    def tick(self, mem):
        hit = np.isin(self.id, mem) & (self.state == QUEUED)
        assert hit.sum() == len(mem)
        self.state[hit] = GONE
        self.state[self.state == DEAD] = GONE

    def expire(self, now, max_wait):
        """-> (ids, seq) of the expiring entries in seq order; they turn dead."""
        k = (self.state == QUEUED) & (r_wait(now, self.ts) >= max_wait)
        self.state[k] = DEAD
        o = np.argsort(self.seq[k], kind="stable")
        return self.id[k][o], self.seq[k][o]


def same_set(got, want):
    ids, seq = got
    o = np.argsort(seq, kind="stable")
    assert np.array_equal(seq[o], want[1]), (len(seq), len(want[1]))
    assert np.array_equal(ids[o], want[0])


def make_players(rng, n, first, now, max_wait, dense):
    ids = (np.arange(first, first + n, dtype=np.uint64) * 7919 % (1 << 20)) if dense else \
        (np.arange(first, first + n, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(12345))
    rating = rng.integers(0, 5001, n).astype(np.int32)
    k = n // 50
    rating[rng.integers(0, n, k)] = rng.integers(-300, 5300, k)   # out of every range: the default group
    mode = rng.integers(0, 2, n).astype(np.uint8)
    wait = rng.integers(-200, 2 ** 31 - 1, n)                     # out of order; some stamped in the future
    near = rng.random(n) < 0.4
    wait[near] = max_wait + rng.integers(-3, 4, int(near.sum()))  # waits at, just below and just above the limit
    ts = ((int(now) - wait) % 2 ** 32).astype(np.uint32)          # most stamps lie "before 0": across the wrap
    return ids, rating, mode, ts


VARIANTS = {
    "hashed": dict(flags=0),
    "wide_partitions": dict(flags=abi.MM_F_WIDE_PARTITIONS),
    "dense_ids": dict(flags=abi.MM_F_DENSE_IDS, active_capacity=1 << 20),
}


def config(pkg, variant, order, capacity):
    return pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=order, capacity=capacity, **VARIANTS[variant])


def waiting_section(st):
    return {f: st[f].copy() for f in ("n_waiting", "n_removed", "max_wait", "wait_hist")}


def assert_same_state(a, b, all_ids, now):
    pa, pb = a.pool_read(), b.pool_read()
    for k in pa:
        assert np.array_equal(pa[k], pb[k]), k
    assert np.array_equal(a.in_queue(all_ids), b.in_queue(all_ids))
    assert a.active_size() == b.active_size() and a.pool_size() == b.pool_size()
    qa, qb = a.queue_stats(now), b.queue_stats(now)
    for f, v in waiting_section(qa).items():
        assert np.array_equal(v, waiting_section(qb)[f]), f


def assert_same_tick(ra, rb):
    for x, y in zip(ra[:3], rb[:3]):
        assert np.array_equal(x, y)
    for f in ("pool_before", "n_lobbies", "n_matched", "n_residual", "n_dead"):
        assert getattr(ra[3], f) == getattr(rb[3], f), f


# ---- GPU: the expired set, and expire == remove ---------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("order,spread", [(ARRIVAL, None), (RATING, None), (RATING, 25)])
@pytest.mark.parametrize("tick_impl", [0, 1])
def test_expire_equals_restatement_and_remove(pkg, variant, order, spread, tick_impl):
    rng = np.random.default_rng(31 + 7 * tick_impl + (spread or 0) + 3 * order)
    cfg = config(pkg, variant, order, 60_000)
    dense = variant == "dense_ids"
    m = Model()
    with pkg.Engine(cfg) as a, pkg.Engine(cfg) as b:
        for e in (a, b):
            e.set_option("tick_impl", tick_impl)
            if spread is not None:
                e.set_option("max_spread", spread)
        now, limit = 1000, 5000
        ids, rating, mode, ts = make_players(rng, 20_000, 0, now, limit, dense)
        acc = a.enqueue(ids, rating, mode, ts)
        assert np.array_equal(acc, b.enqueue(ids, rating, mode, ts))
        m.enqueue(ids, ts, acc)
        gone = ids[rng.random(len(ids)) < 0.05]
        assert a.remove(gone) == b.remove(gone); m.remove(gone)
        taken = ids[rng.random(len(ids)) < 0.03]
        assert a.take(taken) == b.take(taken); m.remove(taken)
        want = m.expire(now, limit)
        assert 0 < len(want[0]) < (m.state != GONE).sum()
        got = a.expire(now, limit)
        same_set(got, want)
        assert b.remove(want[0]) == len(want[0])
        all_ids = ids
        assert_same_state(a, b, all_ids, now)
        assert not a.in_queue(want[0]).any()
        ra, rb = a.tick(now + 1), b.tick(now + 1)
        assert_same_tick(ra, rb)
        assert ra[3].n_dead == len(want[0]) + len(np.unique(np.concatenate([gone, taken])))
        m.tick(ra[1])
        # second round: newcomers, expired ids coming back, matched leavers, then expire again
        t1 = now + 10_000
        ids2, rating2, mode2, ts2 = make_players(rng, 8_000, 20_000, t1, limit, dense)
        back = want[0][:500]
        ids2 = np.concatenate([ids2, back]); rating2 = np.concatenate([rating2, rng.integers(0, 5001, 500).astype(np.int32)])
        mode2 = np.concatenate([mode2, np.zeros(500, np.uint8)]); ts2 = np.concatenate([ts2, np.full(500, t1, np.uint32)])
        acc2 = a.enqueue(ids2, rating2, mode2, ts2)
        assert np.array_equal(acc2, b.enqueue(ids2, rating2, mode2, ts2))
        assert (acc2[-500:] == 1).all()  # an expired id is accepted again
        m.enqueue(ids2, ts2, acc2)
        left = rng.choice(ra[1], 50, replace=False)
        assert a.remove(left) == b.remove(left); m.remove(left)
        want2 = m.expire(t1, limit)
        got2 = a.expire(t1, limit, want_seq=True)
        same_set(got2, want2)
        b.remove(want2[0])
        all_ids = np.concatenate([ids, ids2])
        assert_same_state(a, b, all_ids, t1)
        assert_same_tick(a.tick(t1 + 1), b.tick(t1 + 1))
        assert_same_state(a, b, all_ids, t1 + 2)


@pytest.mark.gpu
@pytest.mark.parametrize("spread", [None, 25])
def test_no_dedupe_expires_every_entry(pkg, oracle, spread):
    """MM_F_NO_DEDUPE: no active set, a repeated id expires per entry (told apart by seq); the next tick equals the
    oracle over the survivors."""
    rng = np.random.default_rng(8 + (spread or 0))
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=RATING, capacity=50_000,
                                flags=abi.MM_F_NO_DEDUPE)
    n, now, limit = 30_000, 77, 300
    ids = rng.integers(0, n // 4, n).astype(np.uint64)  # about four entries per id
    _i, rating, mode, ts = make_players(rng, n, 0, now, limit, False)
    m = Model(dedupe=False)
    with pkg.Engine(cfg) as eng:
        if spread is not None:
            eng.set_option("max_spread", spread)
        acc = eng.enqueue(ids, rating, mode, ts)
        assert (acc == 1).all()
        m.enqueue(ids, ts, acc)
        want = m.expire(now, limit)
        got = eng.expire(now, limit)
        same_set(got, want)
        rep = np.unique(want[0], return_counts=True)[1]
        assert (rep > 1).any()  # some id expired with more than one of its entries
        alive = (m.state == QUEUED)
        pr = eng.pool_read()
        assert np.array_equal(pr["id"], ids[alive]) and np.array_equal(pr["enq_ts"], ts[alive])
        assert np.array_equal(pr["rating"], rating[alive]) and np.array_equal(pr["mode"], mode[alive])
        lob, mem, seq, st = eng.tick(now + 1)
        if spread is None:
            ref = oracle.run_closed_form(cfg, ids, rating, mode, alive=alive.astype(np.uint8))
        else:
            ref = oracle.run_windowed(cfg, spread, ids, rating, mode, alive=alive.astype(np.uint8))
        assert np.array_equal(lob, ref.lobbies) and np.array_equal(mem, ref.member_ids)
        assert np.array_equal(seq, ref.emit_seq)
        assert st.n_dead == len(want[0]) and st.n_matched == ref.n_matched
        assert np.array_equal(eng.pool_read()["id"], ref.residual_ids)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["hashed", "dense_ids"])
def test_limits_and_reenqueue(pkg, variant):
    rng = np.random.default_rng(9)
    cfg = config(pkg, variant, ARRIVAL, 20_000)
    with pkg.Engine(cfg) as eng:
        assert len(eng.expire(5, 0)[0]) == 0  # empty pool
        ids, rating, mode, ts = make_players(rng, 10_000, 0, 100, 50, variant == "dense_ids")
        ts[100:110] = 150  # stamped in the future: wait 0
        assert (eng.enqueue(ids, rating, mode, ts) == 1).all()
        assert len(eng.expire(100, 2 ** 31)[0]) == 0 and len(eng.expire(100, 2 ** 32 - 1)[0]) == 0
        assert eng.remove(ids[:100]) == 100
        w = r_wait(100, ts)
        live = np.arange(len(ids)) >= 100
        wmax = int(w[live].max())
        assert len(eng.expire(100, wmax + 1)[0]) == 0
        top, _ = eng.expire(100, wmax)
        assert np.array_equal(np.sort(top), np.sort(ids[live & (w == wmax)]))
        got, _ = eng.expire(100, 0)  # every queued player, however short its wait
        assert np.array_equal(np.sort(got), np.sort(ids[live & (w < wmax)]))
        assert (w[live] == 0).any()  # stamped "in the future" or at `now`: expired by max_wait 0 all the same
        assert eng.pool_size() == 10_000 and eng.active_size() == 0 and not eng.in_queue(ids).any()
        assert eng.remove(got[:50]) == 0  # an expired id is no longer in the active set
        assert (eng.enqueue(got[:10], rating[:10], mode[:10], ts[:10]) == 1).all()
        assert eng.in_queue(got[:10]).all() and eng.active_size() == 10
        st = eng.tick(200)[3]
        assert st.n_dead == 10_000 and st.pool_before == 10_010


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["hashed", "dense_ids"])
def test_cap_refusal_changes_nothing(pkg, variant):
    rng = np.random.default_rng(10)
    cfg = config(pkg, variant, RATING, 40_000)
    dense = variant == "dense_ids"
    with pkg.Engine(cfg) as a, pkg.Engine(cfg) as b:
        limit = 2 ** 30  # about half of the uniformly drawn waits
        ids, rating, mode, ts = make_players(rng, 20_000, 0, 500, limit, dense)
        for e in (a, b):
            assert (e.enqueue(ids, rating, mode, ts) == 1).all()
            e.remove(ids[:300])
            e.tick(450)
        ids2, rating2, mode2, ts2 = make_players(rng, 10_000, 20_000, 500, limit, dense)
        for e in (a, b):
            e.enqueue(ids2, rating2, mode2, ts2)
        qa0 = a.queue_stats(600)
        lib, n = a.lib, C.c_uint32(0)
        buf = np.empty(40_000, np.uint64)
        seq = np.empty(40_000, np.uint32)
        # dry run: cap 0, no output
        assert lib.mm_expire(a.h, 600, limit, None, None, 0, C.byref(n)) == abi.MM_E_CAP
        count = n.value
        assert 0 < count < a.pool_size()
        for cap in (1, count - 1):
            assert lib.mm_expire(a.h, 600, limit, buf.ctypes.data, seq.ctypes.data, cap, C.byref(n)) == abi.MM_E_CAP
            assert n.value == count
        all_ids = np.concatenate([ids, ids2])
        assert_same_state(a, b, all_ids, 600)
        qa = a.queue_stats(600)
        for f in qa.dtype.names:
            assert np.array_equal(qa[f], qa0[f]), f  # the match section too
        # a cap of exactly the count: the counting pass, then the expiry
        assert lib.mm_expire(a.h, 600, limit, buf.ctypes.data, seq.ctypes.data, count, C.byref(n)) == abi.MM_OK
        assert n.value == count
        want_ids, want_seq = b.expire(600, limit)
        assert np.array_equal(np.sort(buf[:count]), np.sort(want_ids))
        assert np.array_equal(np.sort(seq[:count]), np.sort(want_seq))
        assert_same_state(a, b, all_ids, 600)
        assert_same_tick(a.tick(700), b.tick(700))


@pytest.mark.gpu
def test_packed_handles_and_state(pkg):
    rng = np.random.default_rng(11)
    dense_cfg = config(pkg, "dense_ids", ARRIVAL, 20_000)
    hashed_cfg = config(pkg, "hashed", ARRIVAL, 20_000)
    ids, rating, mode, ts = make_players(rng, 10_000, 0, 900, 300, True)
    with pkg.Engine(dense_cfg) as d, pkg.Engine(hashed_cfg) as h:
        m = Model()
        m.enqueue(ids, ts, d.enqueue_packed(ids.astype(np.uint32), d.pack_key(rating.clip(0, 8191), mode), ts))
        assert h.enqueue(ids, rating, mode, ts).all()
        want = m.expire(900, 300)
        got = d.expire_packed(900, 300)
        assert got[0].dtype == np.uint32
        same_set((got[0].astype(np.uint64), got[1]), want)
        assert not d.in_queue(want[0]).any()
        with pytest.raises(pkg.EngineError) as ei:
            h.expire_packed(900, 300)
        assert ei.value.status == abi.MM_E_STATE
        n = C.c_uint32(0)
        assert d.lib.mm_expire(None, 0, 0, None, None, 0, C.byref(n)) == abi.MM_E_ARG
        assert d.lib.mm_expire(d.h, 0, 0, None, None, 5, C.byref(n)) == abi.MM_E_ARG
        assert d.lib.mm_expire(d.h, 0, 0, None, None, 0, None) == abi.MM_E_ARG


@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True])
def test_between_async_tick_and_results_wait(pkg, packed):
    rng = np.random.default_rng(12 + packed)
    cfg = config(pkg, "dense_ids", RATING, 40_000)
    ids, rating, mode, ts = make_players(rng, 30_000, 0, 2000, 1000, True)
    with pkg.Engine(cfg) as a, pkg.Engine(cfg) as b:
        for e in (a, b):
            e.set_option("async_results", 1)
            assert (e.enqueue(ids, rating, mode, ts) == 1).all()
        ref = b.tick_packed(2100) if packed else b.tick(2100)
        n = a.pool_size()
        lob = np.empty(n, eng_mod.LOBBY_DTYPE)
        mem = np.empty(n, np.uint32 if packed else np.uint64)
        seq = np.empty(n, np.uint32)
        st = a.tick_raw(lob.ctypes.data, n, mem.ctypes.data, n, seq.ctypes.data, now=2100, packed=packed)
        q0 = a.queue_stats(2200)
        got = a.expire_packed(2200, 1000) if packed else a.expire(2200, 1000)
        assert len(got[0]) > 0
        q1 = a.queue_stats(2200)
        for f in ("n_lobbies", "n_matched", "max_match_wait", "match_wait_hist"):
            assert np.array_equal(q0[f], q1[f]), f
        assert q1["n_removed"].sum() == q0["n_removed"].sum() + len(got[0])
        a.results_wait()
        assert np.array_equal(lob[:st.n_lobbies], ref[0]) and np.array_equal(mem[:st.n_matched], ref[1])
        assert np.array_equal(seq[:st.n_lobbies], ref[2])


@pytest.mark.gpu
def test_restore_brings_expired_players_back(pkg):
    rng = np.random.default_rng(13)
    cfg = config(pkg, "hashed", ARRIVAL, 30_000)
    ids, rating, mode, ts = make_players(rng, 20_000, 0, 50, 20, False)
    with pkg.Engine(cfg) as eng:
        assert eng.enqueue(ids, rating, mode, ts).all()
        eng.remove(ids[:100])
        eng.snapshot()
        before, inq, act = eng.pool_read(), eng.in_queue(ids), eng.active_size()
        got, _ = eng.expire(50, 20)
        assert len(got) > 0 and eng.active_size() == act - len(got)
        eng.restore()
        after = eng.pool_read()
        for k in before:
            assert np.array_equal(before[k], after[k]), k
        assert np.array_equal(eng.in_queue(ids), inq) and eng.active_size() == act
        again, _ = eng.expire(50, 20)  # the restored entries expire again
        assert np.array_equal(np.sort(again), np.sort(got))


@pytest.mark.gpu
def test_config3_ten_million(pkg):
    """BASELINE configs[2]: 10 M players with stamps i, about half of them expire."""
    cfg, mode_idx = pkg.synth.workload_config("config3_10m_g32_5v5", RATING, 10_000_000 + 65536)
    n = 10_000_000
    ids, rating, mode, ts = pkg.synth.gen_pool(1, n, mode=mode_idx)
    now, limit = n, n // 2
    with pkg.Engine(cfg) as a, pkg.Engine(cfg) as b:
        for e in (a, b):
            assert e.enqueue(ids, rating, mode, ts).all()
        got, seq = a.expire(now, limit)
        want = ids[np.arange(n) <= now - limit]
        assert len(got) == len(want) == n // 2 + 1
        assert np.array_equal(np.sort(got), np.sort(want)) and np.array_equal(np.sort(seq), np.arange(n // 2 + 1))
        assert b.remove(want) == len(want)
        assert a.active_size() == b.active_size() == n - len(want)
        assert_same_tick(a.tick(now + 1), b.tick(now + 1))
        assert np.array_equal(a.pool_read()["id"], b.pool_read()["id"])


# ---- CPU: the SearchPool with an Engine double ------------------------------------------------------------------------
class ExpiringEngine(OracleEngine):
    """The CPU fake with enqueue stamps and expire(): expired players leave like remove()."""

    def __init__(self, cfg):
        super().__init__(cfg)
        self.ts = {}
        self.expire_calls = []

    def enqueue(self, ids, rating, mode, enq_ts=None):
        acc = super().enqueue(ids, rating, mode, enq_ts)
        ts = np.zeros(len(ids), np.uint32) if enq_ts is None else np.asarray(enq_ts, np.uint32)
        for p, t, c in zip(np.asarray(ids, np.uint64).tolist(), ts.tolist(), acc.tolist()):
            if c == 1:
                self.ts[p] = t
        return acc

    def expire(self, now, max_wait, want_seq=True):
        self.expire_calls.append((now, max_wait))
        q = self.q[0][self.alive.astype(bool)].tolist()
        out = np.array([p for p in q if r_wait(now, self.ts[p]) >= max_wait], np.uint64)
        self.remove(out)
        return out, (np.zeros(len(out), np.uint32) if want_seq else None)


def boot(pkg, engine_cls, clock, timeout_ms):
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=ARRIVAL, capacity=1000)
    eng, broker = engine_cls(cfg), FakeBroker()
    pool = sw.SearchPool(eng, ["1v1", "5v5"], pkg.synth.REFERENCE_GROUP_NAMES, flush_every_s=3600, clock=clock,
                         timeout_ms=timeout_ms)
    for g in pkg.synth.REFERENCE_GROUP_NAMES:
        sw.SearchWorker.start_link(broker, pool, {"group_name": g, "channel_name": f"search.{g}"})
    broker.bind(sw.EXCHANGE_FORWARD, sw.QUEUE_FORWARD, sw.QUEUE_FORWARD)
    return cfg, eng, broker, pool


def publish(pkg, broker, cfg, pid, rating, mode="1v1"):
    from oracle import oracle as orc
    name = pkg.synth.REFERENCE_GROUP_NAMES[orc.find_rating_group(cfg, rating)]
    if f"resp.{pid}" not in broker.bindings.get((sw.EXCHANGE_RESPONSE, f"resp.{pid}"), []):
        broker.bind(sw.EXCHANGE_RESPONSE, f"resp.{pid}", f"resp.{pid}")
    broker.publish(sw.generate_exchange_name(name), sw.generate_queue_name(name),
                   json.dumps({"id": pid, "rating": rating, "game-mode": mode, "response-queue": f"resp.{pid}",
                               "event-name": f"find-{pid}"}))


def responses(broker, pid):
    return [(json.loads(p), pr) for p, pr in broker.queues[f"resp.{pid}"]]


def test_timeout_publishes_error_responses_and_releases_handles(pkg):
    now = [10.0]
    cfg, eng, broker, pool = boot(pkg, ExpiringEngine, lambda: now[0], timeout_ms=2000)
    publish(pkg, broker, cfg, "gm", 4500)          # grandmaster: nobody else
    publish(pkg, broker, cfg, "s1", 1600, "5v5")   # a 5v5 queue of one
    broker.deliver_all()
    assert pool.tick() == 0 and pool.stats["timed_out"] == 0
    now[0] += 1.999
    assert pool.tick() == 0 and pool.stats["timed_out"] == 0 and not responses(broker, "gm")
    now[0] += 0.001                                # waited exactly the limit
    assert pool.tick() == 0 and pool.stats["timed_out"] == 2
    for pid in ("gm", "s1"):
        (doc, props), = responses(broker, pid)
        assert doc == {"error": {"type": "MatchmakingError", "details": sw.TIMEOUT_DETAILS}, "event-name": f"find-{pid}"}
        assert props == {"persistent": True, "content_type": "application/json"}
        assert not pool.in_queue(pid)
    assert not pool.players and len(pool.handles) == 0 and eng.pool_size() == 0
    assert not broker.queues[sw.QUEUE_FORWARD]
    # the same player id queues again and is matched
    publish(pkg, broker, cfg, "gm", 4500)
    publish(pkg, broker, cfg, "gm2", 4600)
    broker.deliver_all()
    assert pool.tick() == 1 and pool.stats["timed_out"] == 2
    lobby = json.loads(broker.queues[sw.QUEUE_FORWARD][-1][0])
    assert sorted(p["id"] for t in lobby["teams"].values() for p in t) == ["gm", "gm2"]
    assert len(responses(broker, "gm")) == 1


def test_timeout_never_hits_players_the_tick_matched(pkg):
    now = [0.0]
    cfg, eng, broker, pool = boot(pkg, ExpiringEngine, lambda: now[0], timeout_ms=100)
    publish(pkg, broker, cfg, "a", 2100)
    broker.deliver_all()
    pool.flush()
    now[0] += 5.0                                  # "a" has waited far past the limit when its opponent arrives
    publish(pkg, broker, cfg, "b", 2200)
    publish(pkg, broker, cfg, "c", 4500)
    broker.deliver_all()
    pool.flush()
    now[0] += 5.0
    assert pool.tick() == 1
    assert not responses(broker, "a") and not responses(broker, "b")
    assert [d["event-name"] for d, _ in responses(broker, "c")] == ["find-c"]
    assert pool.stats["timed_out"] == 1 and pool.in_queue("a") and not pool.in_queue("c")


def run_traffic(pkg, engine_cls, timeout_ms):
    now = [0.0]
    cfg, eng, broker, pool = boot(pkg, engine_cls, lambda: now[0], timeout_ms)
    for step in range(4):
        for i in range(7):
            publish(pkg, broker, cfg, f"p{step}_{i}", 100 + 700 * i, "1v1" if i % 3 else "5v5")
        broker.deliver_all()
        now[0] += 60.0
        pool.tick()
    pool.remove_user("p0_1")
    pool.tick()
    return eng, broker, pool


def test_without_timeout_traffic_is_unchanged(pkg):
    eng, broker, pool = run_traffic(pkg, ExpiringEngine, None)
    ref_eng, ref_broker, ref_pool = run_traffic(pkg, OracleEngine, None)
    assert not eng.expire_calls and "timed_out" not in pool.stats and pool.stats == ref_pool.stats
    assert {q: list(v) for q, v in broker.queues.items()} == {q: list(v) for q, v in ref_broker.queues.items()}
    assert broker.acked == ref_broker.acked and broker.nacked == ref_broker.nacked
    _eng, t_broker, t_pool = run_traffic(pkg, ExpiringEngine, 1000)  # the same traffic with a limit does time out
    assert t_pool.stats["timed_out"] > 0
    assert sum(len(v) for q, v in t_broker.queues.items() if q.startswith("resp.")) == t_pool.stats["timed_out"]
