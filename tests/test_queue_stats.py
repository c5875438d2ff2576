"""Per-queue status (mm_queue_stats): wait buckets, the record layout, the worker's per-group status, and — on the
GPU — both sections of every record against a numpy restatement over the test's own inputs (ids, ratings, modes,
enqueue stamps, the removed / taken sets and the tick's member ids), exact."""
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
NB = 120


# ---- restatement (independent of the package's helpers) ---------------------------------------------------------
def r_wait(now, ts):
    d = (np.uint64(int(now) & 0xFFFFFFFF) - np.asarray(ts, np.uint64)) & np.uint64(0xFFFFFFFF)
    w = d.astype(np.int64)
    return np.where(w >= 2 ** 31, 0, w)  # negative as int32 -> 0


def r_bucket(w):
    w = np.asarray(w, np.int64)
    e = np.zeros_like(w)
    for k in range(31):
        e[w >= (1 << k)] = k
    return np.where(w < 8, w, 8 + 4 * (e - 3) + ((w >> np.maximum(e - 2, 0)) & 3))


def r_group(cfg, rating):
    g = np.full(len(rating), cfg.default_group, np.int64)
    for k in reversed(range(cfg.n_groups)):
        g[(rating >= cfg.group_lo[k]) & (rating <= cfg.group_hi[k])] = k
    return g


def r_section(cut, ts, now, n_cut):
    w = r_wait(now, ts)
    cnt = np.bincount(cut, minlength=n_cut)
    mx = np.zeros(n_cut, np.int64)
    np.maximum.at(mx, cut, w)
    hist = np.bincount(cut * NB + r_bucket(w), minlength=n_cut * NB).reshape(n_cut, NB)
    return cnt, mx, hist


class Model:
    """What the engine holds, restated: per player its queue (mode * G + group), stamp and state."""
    QUEUED, DEAD, GONE = 0, 1, 2

    def __init__(self, cfg):
        self.cfg, self.G = cfg, cfg.n_groups
        self.n_cut = cfg.n_modes * cfg.n_groups
        self.id = np.zeros(0, np.uint64); self.cut = np.zeros(0, np.int64); self.ts = np.zeros(0, np.uint32)
        self.state = np.zeros(0, np.uint8)
        self.match = None  # (cut, ts, now, lobbies per cut) of the last tick

    def enqueue(self, ids, rating, mode, ts, acc):
        k = acc == 1
        cut = mode[k].astype(np.int64) * self.G + r_group(self.cfg, rating[k])
        self.id = np.concatenate([self.id, ids[k]]); self.cut = np.concatenate([self.cut, cut])
        self.ts = np.concatenate([self.ts, ts[k]]); self.state = np.concatenate([self.state, np.zeros(k.sum(), np.uint8)])

    def remove(self, ids):  # mm_remove and mm_take alike: a queued player turns dead, anything else is untouched
        self.state[np.isin(self.id, ids) & (self.state == self.QUEUED)] = self.DEAD

    def tick(self, lob, mem, now):
        hit = np.isin(self.id, mem)
        assert hit.sum() == len(mem) and (self.state[hit] == self.QUEUED).all()
        lob_cut = lob["mode"].astype(np.int64) * self.G + lob["group"]
        self.match = (self.cut[hit], self.ts[hit], now, np.bincount(lob_cut, minlength=self.n_cut))
        self.state[hit] = self.GONE
        self.state[self.state == self.DEAD] = self.GONE

    def check(self, st, now):
        C_ = self.n_cut
        assert len(st) == C_
        assert np.array_equal(st["mode"], np.arange(C_) // self.G) and np.array_equal(st["group"], np.arange(C_) % self.G)
        q = self.state == self.QUEUED
        cnt, mx, hist = r_section(self.cut[q], self.ts[q], now, C_)
        assert np.array_equal(st["n_waiting"], cnt)
        assert np.array_equal(st["n_removed"], np.bincount(self.cut[self.state == self.DEAD], minlength=C_))
        assert np.array_equal(st["max_wait"], mx)
        assert np.array_equal(st["wait_hist"], hist)
        self.check_match(st)

    def check_match(self, st):
        if self.match is None:
            for f in ("n_lobbies", "n_matched", "max_match_wait", "match_wait_hist"):
                assert not st[f].any(), f
            return
        cut, ts, now, nlob = self.match
        cnt, mx, hist = r_section(cut, ts, now, self.n_cut)
        assert np.array_equal(st["n_matched"], cnt)
        assert np.array_equal(st["n_lobbies"], nlob)
        assert np.array_equal(st["max_match_wait"], mx)
        assert np.array_equal(st["match_wait_hist"], hist)


# ---- CPU: buckets, layout, the worker ------------------------------------------------------------------------------
def test_bucket_known_answers():
    assert [eng_mod.wait_bucket(w) for w in range(8)] == list(range(8))
    assert eng_mod.wait_bucket(8) == 8 and eng_mod.wait_bucket(15) == 11 and eng_mod.wait_bucket(16) == 12
    assert eng_mod.wait_bucket(2 ** 31 - 1) == 119
    w = np.concatenate([np.arange(5000), 2 ** np.arange(31), 2 ** np.arange(1, 32) - 1,
                        np.random.default_rng(1).integers(0, 2 ** 31, 100_000)])
    assert np.array_equal(eng_mod.wait_bucket(w), r_bucket(w))


def test_wait_wraps_and_clamps():
    assert eng_mod.wait_of(5, 10) == 0                      # stamped "in the future"
    assert eng_mod.wait_of(100, 100) == 0
    assert eng_mod.wait_of(3, 2 ** 32 - 2) == 5             # across the 2^32 wrap
    assert eng_mod.wait_of(2 ** 32 + 7, 2) == 5             # now is taken modulo 2^32
    assert eng_mod.wait_of(2 ** 31 - 1, 0) == 2 ** 31 - 1
    assert eng_mod.wait_of(2 ** 31, 0) == 0                 # 2^31 reads as negative
    ts = np.random.default_rng(2).integers(0, 2 ** 32, 10_000).astype(np.uint32)
    assert np.array_equal(eng_mod.wait_of(123456, ts), r_wait(123456, ts))


def test_bucket_bounds_cover_the_range():
    lo, hi = eng_mod.wait_bucket_bounds()
    assert len(lo) == len(hi) == abi.MM_WAIT_BUCKETS == NB
    assert lo[0] == 0 and hi[-1] == 2 ** 31 and np.array_equal(lo[1:], hi[:-1]) and (hi > lo).all()
    assert ((hi - lo) * 4 <= np.maximum(lo, 4)).all()  # at most 25 % relative width
    for b in range(NB):  # both ends of every bucket map to it
        assert eng_mod.wait_bucket(lo[b]) == b and eng_mod.wait_bucket(hi[b] - 1) == b


def test_quantiles():
    h = np.zeros(NB, np.uint32)
    assert eng_mod.wait_quantile(h, 0.5) == 0
    h[3], h[12], h[119] = 60, 39, 1
    assert eng_mod.wait_quantile(h, 0.5) == 3
    assert eng_mod.wait_quantile(h, 0.6) == 3
    assert eng_mod.wait_quantile(h, 0.61) == 19
    assert eng_mod.wait_quantile(h, 0.99) == 19
    assert eng_mod.wait_quantile(h, 1.0) == 2 ** 31 - 1


def test_record_layout_matches_header():
    Q = abi.QueueStat
    assert C.sizeof(Q) == 988 == eng_mod.QUEUE_STAT_DTYPE.itemsize
    want = {"mode": 0, "group": 1, "reserved": 2, "n_waiting": 4, "n_removed": 8, "max_wait": 12, "wait_hist": 16,
            "n_lobbies": 496, "n_matched": 500, "max_match_wait": 504, "match_wait_hist": 508}
    for f, off in want.items():
        assert getattr(Q, f).offset == off, f
        assert eng_mod.QUEUE_STAT_DTYPE.fields[f][1] == off, f


class StatsEngine(OracleEngine):
    """The CPU fake with canned queue_stats records: queue (mode m, group g) has 10 m + g + 1 waiting players."""

    def __init__(self, cfg):
        super().__init__(cfg)
        self.calls, self.enq_ts, self.ticks = [], [], []

    def enqueue(self, ids, rating, mode, enq_ts=None):
        self.enq_ts.append(None if enq_ts is None else np.array(enq_ts))
        return super().enqueue(ids, rating, mode, enq_ts)

    def tick(self, now=0):
        self.ticks.append(now)
        return super().tick(now)

    def queue_stats(self, now=0):
        self.calls.append(now)
        G = self.cfg.n_groups
        st = np.zeros(self.cfg.n_modes * G, eng_mod.QUEUE_STAT_DTYPE)
        for c in range(len(st)):
            m, g = divmod(c, G)
            st[c]["mode"], st[c]["group"] = m, g
            st[c]["n_waiting"] = 10 * m + g + 1
            st[c]["max_wait"] = 1000 * m + g
            st[c]["wait_hist"][g] = 50                  # p50 = g
            st[c]["wait_hist"][20 + m] = 50             # p99 in bucket 20 + m
            st[c]["n_matched"] = 2 * (g + 1)
            st[c]["match_wait_hist"][5] = 2 * (g + 1)   # p99 = 5
        return st


def boot(pkg, engine_cls, clock):
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=ARRIVAL, capacity=1000)
    eng, broker = engine_cls(cfg), FakeBroker()
    pool = sw.SearchPool(eng, ["1v1", "5v5"], pkg.synth.REFERENCE_GROUP_NAMES, flush_every_s=3600, clock=clock)
    workers = {}
    for g in pkg.synth.REFERENCE_GROUP_NAMES:
        ok, workers[g] = sw.SearchWorker.start_link(broker, pool, {"group_name": g, "channel_name": f"search.{g}"})
    broker.bind(sw.EXCHANGE_FORWARD, sw.QUEUE_FORWARD, sw.QUEUE_FORWARD)
    return cfg, eng, broker, pool, workers


def publish(pkg, broker, cfg, pid, rating, mode):
    from oracle import oracle as orc
    name = pkg.synth.REFERENCE_GROUP_NAMES[orc.find_rating_group(cfg, rating)]
    broker.publish(sw.generate_exchange_name(name), sw.generate_queue_name(name),
                   json.dumps({"id": pid, "rating": rating, "game-mode": mode}))


def test_worker_status_reports_its_own_group(pkg):
    now = [50.0]
    cfg, eng, broker, pool, workers = boot(pkg, StatsEngine, lambda: now[0])
    now[0] += 1.5
    ok, st = workers["gold"].status()  # gold = group 2
    assert ok == "ok" and eng.calls == [1500]
    lo, hi = eng_mod.wait_bucket_bounds()
    assert st["waiting"] == {
        "1v1": {"waiting": 3, "oldest_wait_ms": 2, "p50_wait_ms": 2, "p99_wait_ms": int(hi[20] - 1),
                "last_tick_matched": 6, "last_tick_p99_match_wait_ms": 5},
        "5v5": {"waiting": 13, "oldest_wait_ms": 1002, "p50_wait_ms": 2, "p99_wait_ms": int(hi[21] - 1),
                "last_tick_matched": 6, "last_tick_p99_match_wait_ms": 5},
    }
    assert st["queue"] == "matchmaking.queues.gold" and st["pool"] == eng.status()
    ok, st = workers["grandmaster"].status()
    assert st["waiting"]["1v1"]["waiting"] == 7 and st["waiting"]["5v5"]["oldest_wait_ms"] == 1006


def test_pool_stamps_batches_and_ticks_with_its_clock(pkg):
    now = [7.0]
    cfg, eng, broker, pool, workers = boot(pkg, StatsEngine, lambda: now[0])
    publish(pkg, broker, cfg, "a", 100, "1v1")
    publish(pkg, broker, cfg, "b", 110, "1v1")
    broker.deliver_all()
    now[0] += 0.25
    assert pool.tick() == 1
    assert np.array_equal(eng.enq_ts[-1], np.array([250, 250], np.uint32)) and eng.enq_ts[-1].dtype == np.uint32
    assert eng.ticks == [250]
    now[0] += 2 ** 32 / 1000 + 0.001  # the millisecond clock wraps modulo 2^32
    pool.tick()
    assert eng.ticks[-1] == 251


def test_status_without_queue_stats_is_unchanged(pkg):
    cfg, eng, broker, pool, workers = boot(pkg, OracleEngine, lambda: 0.0)
    ok, st = workers["gold"].status()
    assert ok == "ok" and set(st) == {"queue", "message_count", "consumer_count", "pool"}
    assert st["pool"] == {"message_count": 0, "active_count": 0}


# ---- GPU: both sections against the restatement --------------------------------------------------------------------
VARIANTS = {
    "reference": dict(flags=0),
    "wide_partitions": dict(flags=abi.MM_F_WIDE_PARTITIONS),
    "dense_ids": dict(flags=abi.MM_F_DENSE_IDS),
}


def make_players(pkg, rng, n, first, now, dense):
    ids, rating, _, _ = pkg.synth.gen_pool(5, n, first=first, bell=True)
    if dense:
        ids = (np.arange(first, first + n) * 7919 % (1 << 20)).astype(np.uint64)  # distinct handles < 2^20
    rating = rating.copy()
    k = n // 50
    rating[rng.integers(0, n, k)] = rng.integers(-300, 5300, k)  # out of every range: the default group
    mode = rng.integers(0, 2, n).astype(np.uint8)
    wait = rng.integers(-200, 2 ** 31 - 1, n)                    # out of order; some stamped in the future
    small = rng.random(n) < 0.3
    wait[small] = rng.integers(-3, 40, int(small.sum()))         # the exact buckets
    ts = ((int(now) - wait) % 2 ** 32).astype(np.uint32)
    return ids, rating, mode, ts


@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("order,spread", [(ARRIVAL, None), (RATING, None), (RATING, 25)])
@pytest.mark.parametrize("tick_impl", [0, 1])
def test_sections_equal_restatement(pkg, variant, order, spread, tick_impl):
    rng = np.random.default_rng(17 + 3 * tick_impl + (spread or 0))
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=order, capacity=60_000,
                                active_capacity=1 << 20 if variant == "dense_ids" else 0, **VARIANTS[variant])
    dense = variant == "dense_ids"
    m = Model(cfg)
    with pkg.Engine(cfg) as eng:
        eng.set_option("tick_impl", tick_impl)
        if spread is not None:
            eng.set_option("max_spread", spread)
        now = 1000                                    # most stamps lie "before 0": waits cross the 2^32 wrap
        m.check(eng.queue_stats(now), now)                 # empty engine: every record zero
        ids, rating, mode, ts = make_players(pkg, rng, 20_000, 0, now, dense)
        m.enqueue(ids, rating, mode, ts, eng.enqueue(ids, rating, mode, ts))
        gone = ids[rng.random(len(ids)) < 0.05]
        eng.remove(gone); m.remove(gone)
        taken = ids[rng.random(len(ids)) < 0.03]
        eng.take(taken); m.remove(taken)
        m.check(eng.queue_stats(now + 5), now + 5)         # no tick yet: the match section is zero
        t1 = now + 12_345
        lob, mem, _seq, st = eng.tick(t1)
        assert st.n_matched > 0
        m.tick(lob, mem, t1)
        m.check(eng.queue_stats(t1), t1)
        # between two ticks: more players, leavers among the matched and the queued, taken queued players
        ids2, rating2, mode2, ts2 = make_players(pkg, rng, 7_000, 20_000, t1, dense)
        m.enqueue(ids2, rating2, mode2, ts2, eng.enqueue(ids2, rating2, mode2, ts2))
        left = np.concatenate([rng.choice(mem, 50, replace=False), rng.choice(ids2, 100, replace=False)])
        eng.remove(left); m.remove(left)
        queued = m.id[m.state == Model.QUEUED]
        taken2 = rng.choice(queued, 200, replace=False)
        eng.take(taken2); m.remove(taken2)
        m.check(eng.queue_stats(t1 + 99), t1 + 99)         # match section unchanged, waiting section updated
        m.check(eng.queue_stats(t1 + 99), t1 + 99)         # a second call changes nothing
        t2 = t1 + 777 + 2 ** 32                       # `now` counts modulo 2^32
        lob, mem, _seq, st = eng.tick(t2)
        m.tick(lob, mem, t2)
        m.check(eng.queue_stats(t2 + 1), t2 + 1)          # the section describes the second tick


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["tick", "tick_packed", "tick_device"])
def test_every_tick_entry_records_now_and_restore_zeroes(pkg, entry):
    rng = np.random.default_rng(3)
    cfg = pkg.synth.make_config(n_groups=8, order=RATING, capacity=30_000, active_capacity=1 << 20,
                                flags=abi.MM_F_DENSE_IDS)
    ids, rating, mode, ts = make_players(pkg, rng, 20_000, 0, 5000, True)
    m = Model(cfg)
    with pkg.Engine(cfg) as eng, pkg.Engine(cfg) as twin:
        m.enqueue(ids, rating, mode, ts, eng.enqueue(ids, rating, mode, ts))
        assert (twin.enqueue(ids, rating, mode, ts) == 1).all()
        m.check(eng.queue_stats(5000), 5000)
        eng.snapshot()
        lob, mem, _s, _st = twin.tick(1)  # the same tick's results (mm_tick_device leaves them on the device)
        if entry == "tick":
            eng.tick(6000)
        elif entry == "tick_packed":
            eng.tick_packed(6000)
        else:
            eng.tick_device(6000)
        m.tick(lob, mem, 6000)
        m.check(eng.queue_stats(6100), 6100)
        eng.restore()
        m = Model(cfg)
        m.enqueue(ids, rating, mode, ts, np.ones(len(ids), np.uint8))
        m.check(eng.queue_stats(6200), 6200)  # the restored pool; the match section is zero


@pytest.mark.gpu
def test_rejected_tick_leaves_pool_and_zeroes_section(pkg):
    rng = np.random.default_rng(4)
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=RATING, capacity=40_000)
    m = Model(cfg)
    with pkg.Engine(cfg) as eng:
        eng.set_option("tick_impl", 0)
        ids, rating, mode, ts = make_players(pkg, rng, 15_000, 0, 100, False)
        m.enqueue(ids, rating, mode, ts, eng.enqueue(ids, rating, mode, ts))
        lob, mem, _s, _st = eng.tick(200)
        m.tick(lob, mem, 200)
        ids2, rating2, mode2, ts2 = make_players(pkg, rng, 15_000, 15_000, 300, False)
        m.enqueue(ids2, rating2, mode2, ts2, eng.enqueue(ids2, rating2, mode2, ts2))
        gone = ids2[:100]
        eng.remove(gone); m.remove(gone)
        m.check(eng.queue_stats(300), 300)
        before = eng.pool_read()
        lob_buf = np.empty(1, eng_mod.LOBBY_DTYPE)
        mem_buf = np.empty(len(ids) + len(ids2), np.uint64)
        st = abi.TickStats()
        rc = eng.lib.mm_tick(eng.h, 400, lob_buf.ctypes.data, 1, mem_buf.ctypes.data, len(mem_buf), None, C.byref(st))
        assert rc == abi.MM_E_CAP
        after = eng.pool_read()
        assert all(np.array_equal(before[k], after[k]) for k in before)
        m.match = None
        m.check(eng.queue_stats(500), 500)  # waiting section as before the call, match section zero
        lob, mem, _s, _st = eng.tick(600)
        m.tick(lob, mem, 600)
        m.check(eng.queue_stats(700), 700)


@pytest.mark.gpu
@pytest.mark.parametrize("tick_impl", [0, 1])
def test_queue_stats_leaves_ticks_unchanged(pkg, tick_impl):
    rng = np.random.default_rng(5)
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=ARRIVAL, capacity=100_000)
    with pkg.Engine(cfg) as a, pkg.Engine(cfg) as b:
        for e in (a, b):
            e.set_option("tick_impl", tick_impl)
        for step in range(3):
            ids, rating, mode, ts = make_players(pkg, rng, 25_000, 25_000 * step, 1000 * step, False)
            assert np.array_equal(a.enqueue(ids, rating, mode, ts), b.enqueue(ids, rating, mode, ts))
            gone = ids[rng.random(len(ids)) < 0.02]
            a.queue_stats(1000 * step)
            assert a.remove(gone) == b.remove(gone)
            a.queue_stats(1000 * step + 1)
            ra, rb = a.tick(1000 * step + 2), b.tick(1000 * step + 2)
            for x, y in zip(ra[:3], rb[:3]):
                assert np.array_equal(x, y)
            assert np.array_equal(a.pool_read()["id"], b.pool_read()["id"])
            a.queue_stats(1000 * step + 3)


@pytest.mark.gpu
def test_cap_and_bad_arguments(pkg):
    cfg = pkg.synth.make_config(n_groups=5, order=ARRIVAL, capacity=100)  # 2 modes x 5 groups
    with pkg.Engine(cfg) as eng:
        out = (abi.QueueStat * 10)()
        n = C.c_uint32(0)
        assert eng.lib.mm_queue_stats(eng.h, 0, out, 9, C.byref(n)) == abi.MM_E_CAP and n.value == 10
        assert eng.lib.mm_queue_stats(eng.h, 0, out, 0, C.byref(n)) == abi.MM_E_CAP and n.value == 10
        assert eng.lib.mm_queue_stats(eng.h, 0, out, 10, C.byref(n)) == abi.MM_OK and n.value == 10
        assert eng.lib.mm_queue_stats(None, 0, out, 10, C.byref(n)) == abi.MM_E_ARG
        assert eng.lib.mm_queue_stats(eng.h, 0, None, 10, C.byref(n)) == abi.MM_E_ARG
        assert eng.lib.mm_queue_stats(eng.h, 0, out, 10, None) == abi.MM_E_ARG
        assert [(r.mode, r.group) for r in out] == [(c // 5, c % 5) for c in range(10)]


@pytest.mark.gpu
def test_config3_ten_million(pkg):
    """BASELINE configs[2]: 10 M players, 32 groups, 5v5, rating order."""
    cfg, mode_idx = pkg.synth.workload_config("config3_10m_g32_5v5", RATING, 10_000_000 + 65536)
    ids, rating, mode, ts = pkg.synth.gen_pool(1, 10_000_000, mode=mode_idx)
    with pkg.Engine(cfg) as eng:
        assert eng.enqueue(ids, rating, mode, ts).all()
        now = 12_000_000
        got = eng.queue_stats(now)
        pr = eng.pool_read()
        cut = pr["mode"].astype(np.int64) * cfg.n_groups + r_group(cfg, pr["rating"])
        cnt, mx, hist = r_section(cut, pr["enq_ts"], now, len(got))
        assert np.array_equal(got["n_waiting"], cnt) and cnt.sum() == 10_000_000
        assert np.array_equal(got["max_wait"], mx) and np.array_equal(got["wait_hist"], hist)
        assert not got["n_removed"].any() and not got["n_matched"].any()
        lob, mem, _s, st = eng.tick(now + 5)
        order = np.argsort(ids)
        idx = order[np.searchsorted(ids, mem, sorter=order)]
        assert np.array_equal(ids[idx], mem)
        mcut = mode[idx].astype(np.int64) * cfg.n_groups + r_group(cfg, rating[idx])
        cnt, mx, hist = r_section(mcut, ts[idx], now + 5, len(got))
        got = eng.queue_stats(now + 9)
        assert np.array_equal(got["n_matched"], cnt) and cnt.sum() == st.n_matched
        assert np.array_equal(got["max_match_wait"], mx) and np.array_equal(got["match_wait_hist"], hist)
        assert np.array_equal(got["n_lobbies"], np.bincount(lob["mode"].astype(np.int64) * cfg.n_groups + lob["group"],
                                                            minlength=len(got)))
        pr = eng.pool_read()
        cut = pr["mode"].astype(np.int64) * cfg.n_groups + r_group(cfg, pr["rating"])
        cnt, mx, hist = r_section(cut, pr["enq_ts"], now + 9, len(got))
        assert np.array_equal(got["n_waiting"], cnt) and np.array_equal(got["wait_hist"], hist)
