"""Match quality (mm_match_quality / Engine.match_quality / SearchPool.match_quality): the rating spread and team
imbalance of the last tick's lobbies, per lobby and per (mode, group) queue, computed on the device.

The restatement below starts from the test's own inputs (id -> rating) and the tick's own outputs (headers, members)
and computes every per-lobby field and every per-queue record; the engine must equal it exactly.
CPU: the ABI mirror, the bucket of values at and above 2^31, SearchPool.match_quality and SearchWorker.status() on an
engine double that reports restated records.
GPU: both orders, S0 and S1, budgets, wide / split / overlapping groups, clamped ratings, 1-team and 1-player-team
modes, both id kinds and no dedupe, removed / taken / requeued / merged players, every tick form, multi-tick
schedules; the report unchanged by every other call; the void states; the refusals; twin engines (no side effects);
config3 at 10 M players.
"""
import ctypes as C
import importlib

import numpy as np
import pytest

from .fakes import FakeBroker, OracleEngine

sw = importlib.import_module("microservice-matchmaking_b200.search_worker")
eng_mod = importlib.import_module("microservice-matchmaking_b200.engine")
abi = importlib.import_module("microservice-matchmaking_b200.abi")

RATING, ARRIVAL = 1, 0
DENSE, WIDE, NO_DEDUPE = 2, 4, 1
NB = abi.MM_WAIT_BUCKETS
# (name, teams, team size): 1v1, 5v5, a one-team mode, one-player teams, an odd shape
MODES = (("1v1", 2, 1), ("5v5", 2, 5), ("coop4", 1, 4), ("ffa6", 6, 1), ("3x3", 3, 3))


# ================================================================================ restatement
class Ratings:
    """id -> rating of every player the test enqueued (the test's own input)."""

    def __init__(self):
        self.ids, self.r = np.zeros(0, np.uint64), np.zeros(0, np.int64)

    def add(self, ids, rating):
        ids = np.asarray(ids, np.uint64)
        ids, first = np.unique(ids, return_index=True)
        keep = ~np.isin(ids, self.ids)
        self.ids = np.concatenate([self.ids, ids[keep]])
        self.r = np.concatenate([self.r, np.asarray(rating, np.int64)[first][keep]])
        o = np.argsort(self.ids)
        self.ids, self.r = self.ids[o], self.r[o]

    def __call__(self, ids):
        ids = np.asarray(ids, np.uint64)
        k = np.searchsorted(self.ids, ids)
        assert (k < len(self.ids)).all() and np.array_equal(self.ids[np.minimum(k, len(self.ids) - 1)], ids)
        return self.r[k]


def clamp_bounds(cfg):
    return (min(cfg.group_lo[g] for g in range(cfg.n_groups)) - 1, max(cfg.group_hi[g] for g in range(cfg.n_groups)) + 1)


def restate(cfg, lob, mem, rating_of):
    """-> (QUALITY_DTYPE[n_modes * n_groups], LOBBY_QUALITY_DTYPE[len(lob)]) of one tick's headers and members."""
    lo, hi = clamp_bounds(cfg)
    G = cfg.n_groups
    n = len(lob)
    pl = np.zeros(n, eng_mod.LOBBY_QUALITY_DTYPE)
    mode = lob["mode"].astype(np.int64)
    for m in np.unique(mode):
        T, S = cfg.modes[m].teams, cfg.modes[m].team_size
        L = T * S
        sel = np.flatnonzero(mode == m)
        assert (lob["n_members"][sel] == L).all()
        idx = lob["first_member"][sel].astype(np.int64)[:, None] + np.arange(L)[None, :]
        r = np.clip(rating_of(np.asarray(mem)[idx.ravel()]).reshape(len(sel), L), lo, hi)
        pl["min_rating"][sel] = r.min(1)
        pl["max_rating"][sel] = r.max(1)
        pl["rating_sum"][sel] = r.sum(1)
        ts = r.reshape(len(sel), T, S).sum(2)
        pl["imbalance"][sel] = np.minimum(ts.max(1) - ts.min(1), 0xFFFFFFFF)
    q = mode * G + lob["group"].astype(np.int64)
    n_cut = cfg.n_modes * G
    pq = np.zeros(n_cut, eng_mod.QUALITY_DTYPE)
    pq["mode"], pq["group"] = np.arange(n_cut) // G, np.arange(n_cut) % G
    spread = pl["max_rating"].astype(np.int64) - pl["min_rating"]
    imb = pl["imbalance"].astype(np.int64)
    pq["n_lobbies"] = np.bincount(q, minlength=n_cut)
    np.maximum.at(pq["max_spread"], q, spread.astype(np.uint32))
    np.maximum.at(pq["max_imbalance"], q, imb.astype(np.uint32))
    np.add.at(pq["sum_spread"], q, spread.astype(np.uint64))
    np.add.at(pq["sum_imbalance"], q, imb.astype(np.uint64))
    np.add.at(pq["spread_hist"], (q, eng_mod.quality_bucket(spread)), 1)
    np.add.at(pq["imbalance_hist"], (q, eng_mod.quality_bucket(imb)), 1)
    return pq, pl


# ================================================================================ CPU
def test_abi_mirror():
    assert C.sizeof(abi.LobbyQuality) == 24 and C.sizeof(abi.QueueQuality) == 992
    for cls, dt in ((abi.LobbyQuality, eng_mod.LOBBY_QUALITY_DTYPE), (abi.QueueQuality, eng_mod.QUALITY_DTYPE)):
        assert dt.itemsize == C.sizeof(cls)
        for f, *_ in cls._fields_:
            assert getattr(cls, f).offset == dt.fields[f][1], f
    want = {"n_lobbies": 4, "max_spread": 8, "max_imbalance": 12, "sum_spread": 16, "sum_imbalance": 24,
            "spread_hist": 32, "imbalance_hist": 512}
    for f, off in want.items():
        assert eng_mod.QUALITY_DTYPE.fields[f][1] == off, f
    assert eng_mod.LOBBY_QUALITY_DTYPE.fields["rating_sum"][1] == 8
    assert eng_mod.LOBBY_QUALITY_DTYPE.fields["imbalance"][1] == 16
    assert "mm_match_quality" in abi.PROTOTYPES


def test_bucket_at_and_above_two_to_the_31():
    v = np.array([0, 7, 8, 9, 10, 1 << 20, (1 << 31) - 1], np.int64)
    assert np.array_equal(eng_mod.quality_bucket(v), eng_mod.wait_bucket(v))
    assert eng_mod.quality_bucket((1 << 31) - 1) == NB - 1
    for x in (1 << 31, (1 << 31) + 1, 3 << 30, (1 << 32) - 1):
        assert eng_mod.quality_bucket(x) == NB - 1
    lo, hi = eng_mod.wait_bucket_bounds()
    assert hi[-1] == 1 << 31  # bucket 119 holds [7 * 2^28, 2^31) and everything above


def test_restatement_by_hand(pkg):
    cfg = pkg.synth.make_config(groups=[(0, 99), (100, 199)], modes=(("2v2", 2, 2), ("solo3", 1, 3)), order=RATING,
                                capacity=100, default_group=-1)
    rt = Ratings()
    rt.add(np.arange(1, 11, dtype=np.uint64), [10, 20, 30, 80, 150, 150, 199, 120, 120, 120])
    lob = np.zeros(3, eng_mod.LOBBY_DTYPE)
    lob[0] = (0, 4, 0, 0)   # 10 20 | 30 80: teams 30 and 110, spread 70
    lob[1] = (4, 4, 0, 1)   # 150 150 | 199 120: teams 300 and 319
    lob[2] = (8, 3, 1, 1)   # 120 120 120: one team
    mem = np.array([1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 8], np.uint64)
    pq, pl = restate(cfg, lob, mem, rt)
    assert pl.tolist() == [(10, 80, 140, 80, 0), (120, 199, 619, 19, 0), (120, 120, 360, 0, 0)]
    assert pq["n_lobbies"].tolist() == [1, 1, 0, 1]
    assert pq["max_spread"].tolist() == [70, 79, 0, 0] and pq["max_imbalance"].tolist() == [80, 19, 0, 0]
    assert pq[3]["spread_hist"][0] == 1 and pq[0]["spread_hist"][eng_mod.wait_bucket(70)] == 1


class QualityEngine(OracleEngine):
    """The CPU engine double whose match_quality() reports the restated records of its last tick."""

    def __init__(self, cfg):
        super().__init__(cfg)
        self.rt = Ratings()
        self.report = None

    def enqueue(self, ids, rating, mode, enq_ts=None):
        acc = super().enqueue(ids, rating, mode, enq_ts)
        self.rt.add(np.asarray(ids, np.uint64)[acc == 1], np.asarray(rating)[acc == 1])
        return acc

    def tick(self, now=0):
        lob, mem, seq, st = super().tick(now)
        self.report = restate(self.cfg, np.asarray(lob, eng_mod.LOBBY_DTYPE), mem, self.rt)
        return lob, mem, seq, st

    def match_quality(self, want_lobbies=False):
        if self.report is None:
            return np.zeros(0, eng_mod.QUALITY_DTYPE), (np.zeros(0, eng_mod.LOBBY_QUALITY_DTYPE) if want_lobbies else None)
        return self.report[0], (self.report[1] if want_lobbies else None)


def test_search_pool_and_worker_status(pkg):
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=ARRIVAL, capacity=1000)
    eng = QualityEngine(cfg)
    pool = sw.SearchPool(eng, ["1v1", "5v5"], pkg.synth.REFERENCE_GROUP_NAMES, flush_every_s=3600, clock=lambda: 5.0)
    broker = FakeBroker()
    ok, w = sw.SearchWorker.start_link(broker, pool, {"group_name": "gold", "channel_name": "search.gold"})
    assert ok == "ok"
    assert pool.match_quality("gold") == {}  # void before the first tick
    assert pool.match_quality("nowhere") == {}
    rng = np.random.default_rng(3)
    n = 400
    ids = np.arange(1, n + 1, dtype=np.uint64)
    rating = rng.integers(2000, 2500, n).astype(np.int32)  # gold
    mode = (np.arange(n) % 3 == 0).astype(np.uint8)
    eng.enqueue(ids, rating, mode)
    eng.tick()
    q = eng.report[0]
    got = pool.match_quality("gold")
    assert set(got) == {"1v1", "5v5"}
    for m, name in enumerate(("1v1", "5v5")):
        r = q[m * cfg.n_groups + 2]
        k = int(r["n_lobbies"])
        assert k > 0
        assert got[name] == {
            "lobbies": k,
            "mean_spread": int(r["sum_spread"]) / k,
            "p50_spread": eng_mod.wait_quantile(r["spread_hist"], 0.5),
            "p99_spread": eng_mod.wait_quantile(r["spread_hist"], 0.99),
            "max_spread": int(r["max_spread"]),
            "mean_imbalance": int(r["sum_imbalance"]) / k,
            "p99_imbalance": eng_mod.wait_quantile(r["imbalance_hist"], 0.99),
            "max_imbalance": int(r["max_imbalance"]),
        }
        assert got[name]["max_spread"] >= got[name]["p99_spread"] * 0.8
    assert pool.match_quality("bronze")["1v1"]["lobbies"] == 0
    ok, st = w.status()
    assert ok == "ok" and st["quality"] == got
    # an engine without match_quality (the plain CPU double): status() has no "quality"
    pool2 = sw.SearchPool(OracleEngine(cfg), ["1v1", "5v5"], pkg.synth.REFERENCE_GROUP_NAMES, flush_every_s=3600)
    ok, w2 = sw.SearchWorker.start_link(FakeBroker(), pool2, {"group_name": "gold", "channel_name": "search.gold"})
    assert "quality" not in w2.status()[1]


# ================================================================================ GPU
def gpu_config(pkg, order, layout, flags=0, modes=MODES, capacity=300_000):
    groups = {"split": pkg.synth.REFERENCE_GROUPS, "wide": pkg.synth.REFERENCE_GROUPS,
              "overlap": [(0, 2000), (1000, 3000), (2500, 5000), (100, 200)], "one": [(0, 5000)]}[layout]
    if layout == "wide":
        flags |= WIDE
    return pkg.synth.make_config(groups=groups, modes=modes, order=order, capacity=capacity,
                                 active_capacity=2 * capacity, default_group=1 if layout == "overlap" else -1,
                                 flags=flags)


class Driver:
    """One engine, its id -> rating book and a supply of fresh players."""

    def __init__(self, pkg, cfg, seed, spread=-1):
        self.pkg, self.cfg = pkg, cfg
        self.dense = bool(cfg.flags & DENSE)
        self.eng = pkg.Engine(cfg)
        if spread >= 0:
            self.eng.set_option("max_spread", spread)
        self.rng = np.random.default_rng(seed)
        self.rt = Ratings()
        self.next = 0
        self.now = 1000

    def fresh(self, n, lo=-400, hi=5400):
        x = np.arange(self.next, self.next + n, dtype=np.uint64)
        self.next += n
        ids = x if self.dense else self.pkg.synth.mix64(x + np.uint64(11 << 40))
        r = self.rng.integers(lo, hi, n).astype(np.int32)
        m = self.rng.integers(0, self.cfg.n_modes, n).astype(np.uint8)
        ts = (self.now - self.rng.integers(0, 60, n)).astype(np.uint32)
        return ids, r, m, ts

    def enqueue(self, n, **kw):
        ids, r, m, ts = self.fresh(n, **kw)
        acc = self.eng.enqueue(ids, r, m, ts)
        self.rt.add(ids[acc == 1], r[acc == 1])
        return ids[acc == 1]

    def close(self):
        self.eng.close()


def check(cfg, eng, res, rt, spread=-1):
    """The engine's report of the tick `res` equals the restatement; -> the report."""
    lob, mem = res[0], res[1]
    want_q, want_l = restate(cfg, lob, mem, rt)
    got_q, got_l = eng.match_quality(want_lobbies=True)
    assert len(got_l) == res[3].n_lobbies == len(lob)
    assert np.array_equal(got_l, want_l)
    assert np.array_equal(got_q, want_q)
    if spread >= 0:
        assert (got_q["max_spread"] <= spread).all()
    q2, none = eng.match_quality()
    assert none is None and np.array_equal(q2, got_q)
    return got_q, got_l


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
@pytest.mark.parametrize("layout", ["split", "wide", "overlap"])
@pytest.mark.parametrize("kind", ["hashed", "dense", "no_dedupe"])
def test_report_equals_restatement(pkg, order, layout, kind):
    from .test_tick_forms_and_schedules import tick_form
    flags = {"hashed": 0, "dense": DENSE, "no_dedupe": NO_DEDUPE}[kind]
    cfg = gpu_config(pkg, order, layout, flags)
    nq = cfg.n_modes * cfg.n_groups
    spreads = [-1, 0, 5, 40, 300] if order == RATING else [-1]
    forms = ["tick_emit", "tick", "packed_emit", "packed", "device"] if kind == "dense" else ["tick_emit", "tick",
                                                                                            "device"]
    rng = np.random.default_rng(order * 5 + len(layout) + len(kind))
    k = 0
    for spread in spreads:
        for budgets in ((None, None), (rng.integers(0, 30, nq), None), (None, np.array([0, 90, 3, 1000, 7])),
                        (rng.integers(0, 3, nq), np.array([5, 0, 1000, 2, 40]))):
            for impl in (1, 0):
                d = Driver(pkg, cfg, seed=k, spread=spread)
                try:
                    d.eng.set_option("tick_impl", impl)
                    d.eng.set_lobby_budget(*budgets)
                    for step in range(3):  # a multi-tick schedule: the leftovers of each tick feed the next
                        ids = d.enqueue(25_000 if step == 0 else 8_000)
                        if kind != "no_dedupe" and step == 1:
                            d.eng.remove(ids[::7])
                            d.eng.take(ids[3::11])
                        form = forms[(k + step) % len(forms)]
                        res = tick_form(pkg, d.eng, form, d.now + step)
                        check(cfg, d.eng, res, d.rt, spread)
                finally:
                    d.close()
                k += 1


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
def test_async_results_and_one_group(pkg, order):
    for layout in ("one", "split"):
        cfg = gpu_config(pkg, order, layout, DENSE)
        d = Driver(pkg, cfg, seed=9)
        try:
            d.eng.set_option("async_results", 1)
            for step in range(4):
                d.enqueue(30_000)
                res = d.eng.tick(d.now + step, want_emit_seq=step % 2 == 0)
                d.eng.results_wait()
                check(cfg, d.eng, res, d.rt)
                lob, mem, _seq, st = d.eng.tick_packed(d.now + step, want_emit_seq=False)
                q, l = d.eng.match_quality(want_lobbies=True)  # read before the packed copies are waited for
                d.eng.results_wait()
                want_q, want_l = restate(cfg, lob, mem.astype(np.uint64), d.rt)
                assert np.array_equal(q, want_q) and np.array_equal(l, want_l)
        finally:
            d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
def test_requeued_and_merged_players(pkg, order):
    cfg = gpu_config(pkg, order, "split")
    d = Driver(pkg, cfg, seed=21, spread=30 if order == RATING else -1)
    other = pkg.Engine(cfg)
    try:
        d.enqueue(40_000)
        lob, mem, _s, st = d.eng.tick(d.now)
        check(cfg, d.eng, (lob, mem, None, st), d.rt, 30 if order == RATING else -1)
        # requeue the members of every third lobby
        back = np.concatenate([mem[h["first_member"]:h["first_member"] + h["n_members"]] for h in lob[::3]])
        pr = d.eng.locate(back)  # matched: still active
        assert (pr["state"] == 2).all()
        r = d.rt(back).astype(np.int32)
        m = np.concatenate([np.full(h["n_members"], h["mode"], np.uint8) for h in lob[::3]])
        ts = np.full(len(back), d.now - 5, np.uint32)
        seq = np.arange(len(back), dtype=np.uint32)  # any strict age order inside a queue
        codes = d.eng.requeue(back, r, m, ts, seq)
        assert (codes == 1).all()
        # merge a queue moved from another engine
        ids, rr, mm, tt = d.fresh(20_000)
        mm[:] = 1
        rr[:] = d.rng.integers(2000, 2500, len(rr))
        assert other.enqueue(ids, rr, mm, tt).all()
        sel = np.zeros(cfg.n_modes * cfg.n_groups, np.uint8)
        sel[1 * cfg.n_groups + 2] = 1
        img = other.export_queues(sel)
        d.eng.export_queues(sel)  # a queue is merged into an engine where it holds no live player
        d.eng.merge_queues(img)
        d.rt.add(ids, rr)
        res = d.eng.tick(d.now + 1)
        check(cfg, d.eng, res, d.rt)
    finally:
        other.close()
        d.close()


def snapshot_of(eng):
    q, l = eng.match_quality(want_lobbies=True)
    return q.copy(), l.copy()


def same(a, b):
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
def test_report_stable_under_every_other_call(pkg, order):
    cfg = gpu_config(pkg, order, "split", DENSE)
    d = Driver(pkg, cfg, seed=5)
    other = pkg.Engine(cfg)
    try:
        d.enqueue(60_000)
        res = d.eng.tick(d.now)
        rep = check(cfg, d.eng, res, d.rt)
        lob, mem = res[0], res[1]
        base = snapshot_of(d.eng)
        assert len(base[1]) == len(lob)

        def fresh(n=3000):
            ids, r, m, ts = d.fresh(n, lo=0, hi=5001)
            d.rt.add(ids, r)
            return ids, r, m, ts

        def packed():
            ids, r, m, ts = fresh()
            return d.eng.enqueue_packed(ids.astype(np.uint32), d.eng.pack_key(r, m), ts)

        def packed_begin_end():
            ids, r, m, ts = fresh()
            d.eng.enqueue_packed_begin(ids.astype(np.uint32), d.eng.pack_key(r, m), ts)
            return d.eng.enqueue_packed_end()

        def device():
            import torch
            ids, r, m, ts = fresh()
            cols = [torch.from_numpy(x.view(np.int64) if x.dtype == np.uint64 else x).cuda() for x in (ids, r, m, ts)]
            acc = torch.zeros(len(ids), dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            return d.eng.enqueue_device(len(ids), *(c.data_ptr() for c in cols), acc.data_ptr())

        ids, r, m, ts = fresh()
        back = mem[lob[0]["first_member"]:lob[0]["first_member"] + lob[0]["n_members"]]
        sel = np.zeros(cfg.n_modes * cfg.n_groups, np.uint8)
        sel[cfg.n_groups + 3] = 1
        ids2, r2, m2, ts2 = d.fresh(2000)
        m2[:], r2[:] = 0, 2200
        d.rt.add(ids2, r2)
        other2 = pkg.Engine(cfg)
        assert other2.enqueue(ids2, r2, m2, ts2).all()
        sel2 = np.zeros_like(sel)
        sel2[2] = 1
        steps = [
            lambda: d.eng.enqueue(*fresh()), packed, packed_begin_end, device,
            lambda: d.eng.enqueue(ids, r, m, ts),
            lambda: d.eng.remove(ids[:100]),
            lambda: d.eng.take(ids[100:200]),
            lambda: d.eng.expire(d.now + 10 ** 6, 10 ** 9),
            lambda: d.eng.requeue(back, d.rt(back).astype(np.int32), np.full(len(back), lob[0]["mode"], np.uint8),
                                  np.full(len(back), d.now, np.uint32), np.arange(len(back), dtype=np.uint32)),
            lambda: d.eng.backfill(1, 2, 2200, 3, 100 if order == RATING else None),
            lambda: d.eng.locate(ids[:50]),
            lambda: d.eng.queue_stats(d.now),
            lambda: d.eng.lobby_candidates(),
            lambda: d.eng.set_lobby_budget(np.zeros(cfg.n_modes * cfg.n_groups, np.uint32)),
            lambda: d.eng.set_option("tick_impl", 0),
            lambda: d.eng.export_state(),
            lambda: other.merge_queues(d.eng.export_queues(sel)),
            lambda: (d.eng.export_queues(sel2), d.eng.merge_queues(other2.export_queues(sel2))),
            lambda: d.eng.snapshot(),
        ]
        if order == RATING:
            steps.append(lambda: d.eng.band_match(20, 1, 2))
        for k, step in enumerate(steps):
            step()
            same(snapshot_of(d.eng), base)
        other2.close()
        assert rep[0]["n_lobbies"].sum() == len(lob)
    finally:
        other.close()
        d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
def test_void_states_and_refusals(pkg, order):
    cfg = gpu_config(pkg, order, "split", capacity=50_000)
    n_cut = cfg.n_modes * cfg.n_groups
    d = Driver(pkg, cfg, seed=2)
    lib = d.eng.lib
    try:
        def void():
            q, l = d.eng.match_quality(want_lobbies=True)
            return len(q) == 0 and len(l) == 0

        assert void()  # before the first tick
        d.enqueue(20_000)
        lob, mem, _s, st = d.eng.tick(d.now)
        assert not void() and st.n_lobbies > 0
        # refusals: nothing written, the counts returned
        outq = np.full(n_cut, 0, eng_mod.QUALITY_DTYPE)
        outq.view(np.uint8)[:] = 0xAB
        outl = np.zeros(st.n_lobbies, eng_mod.LOBBY_QUALITY_DTYPE)
        outl.view(np.uint8)[:] = 0xCD
        n, nl = C.c_uint32(7), C.c_uint32(7)
        p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        rc = lib.mm_match_quality(d.eng.h, p(outq), n_cut - 1, C.byref(n), p(outl), st.n_lobbies, C.byref(nl))
        assert rc == abi.MM_E_CAP and n.value == n_cut and nl.value == st.n_lobbies
        rc = lib.mm_match_quality(d.eng.h, p(outq), n_cut, C.byref(n), p(outl), st.n_lobbies - 1, C.byref(nl))
        assert rc == abi.MM_E_CAP and n.value == n_cut and nl.value == st.n_lobbies
        assert (outq.view(np.uint8) == 0xAB).all() and (outl.view(np.uint8) == 0xCD).all()
        for args in ((None, n_cut, C.byref(n), None, 0, C.byref(nl)), (p(outq), n_cut, None, None, 0, C.byref(nl)),
                     (p(outq), n_cut, C.byref(n), None, 0, None)):
            assert lib.mm_match_quality(d.eng.h, *args) == abi.MM_E_ARG
        assert lib.mm_match_quality(None, p(outq), n_cut, C.byref(n), None, 0, C.byref(nl)) == abi.MM_E_ARG
        # per_lobby NULL skips the lobby check
        assert lib.mm_match_quality(d.eng.h, p(outq), n_cut, C.byref(n), None, 0, C.byref(nl)) == abi.MM_OK
        assert n.value == n_cut and nl.value == st.n_lobbies
        # void after a tick that failed with MM_E_CAP
        d.enqueue(10_000)
        lob_buf, mem_buf, st1 = np.empty(1, eng_mod.LOBBY_DTYPE), np.empty(200_000, np.uint64), abi.TickStats()
        rc = lib.mm_tick(d.eng.h, d.now + 1, p(lob_buf), 1, p(mem_buf), len(mem_buf), None, C.byref(st1))
        assert rc == abi.MM_E_CAP
        assert void()
        res = d.eng.tick(d.now + 2)
        check(cfg, d.eng, res, d.rt)
        # void after mm_restore
        d.eng.snapshot()
        d.enqueue(10_000)
        check(cfg, d.eng, d.eng.tick(d.now + 3), d.rt)
        d.eng.restore()
        assert void()
        check(cfg, d.eng, d.eng.tick(d.now + 4), d.rt)
        # void after mm_import and mm_import_regroup
        img = d.eng.export_state()
        for load in ("import_state", "import_regroup"):
            e2 = pkg.Engine(cfg)
            try:
                if load == "import_state":
                    e2.import_state(img)
                else:
                    e2.import_regroup(img)
                q, l = e2.match_quality(want_lobbies=True)
                assert len(q) == 0 and len(l) == 0
            finally:
                e2.close()
    finally:
        d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
def test_twin_engines_no_side_effects(pkg, order):
    cfg = gpu_config(pkg, order, "overlap", DENSE)
    a, b = Driver(pkg, cfg, seed=4), Driver(pkg, cfg, seed=4)
    try:
        def both(fn):
            ra = fn(a)
            a.eng.match_quality(want_lobbies=True)
            rb = fn(b)
            return ra, rb

        def eq(x, y):
            if isinstance(x, tuple):
                for u, v in zip(x, y):
                    eq(u, v)
            elif isinstance(x, np.ndarray):
                assert np.array_equal(x, y)
            elif isinstance(x, dict):
                assert x.keys() == y.keys()
                for k in x:
                    eq(x[k], y[k])
            elif isinstance(x, abi.TickStats):
                for f, *_ in x._fields_:
                    if not f.endswith("_us"):
                        assert getattr(x, f) == getattr(y, f), f
            else:
                assert x == y

        for step in range(5):
            eq(*both(lambda d: d.enqueue(20_000)))
            eq(*both(lambda d: d.eng.remove(np.arange(step * 1000, step * 1000 + 300, dtype=np.uint64))))
            eq(*both(lambda d: d.eng.queue_stats(d.now)))
            eq(*both(lambda d: d.eng.tick(d.now + step)))
            eq(*both(lambda d: d.eng.locate(np.arange(0, 5000, 7, dtype=np.uint64), d.now)))
            eq(*both(lambda d: d.eng.pool_read()))
        # the export's active section is unordered: compare it as a set
        (ha, sa), (hb, sb) = (eng_mod.read_image(np.array(d.eng.export_state(), np.uint8, copy=True)) for d in (a, b))
        assert (ha.n_players, ha.n_active, ha.seq_next) == (hb.n_players, hb.n_active, hb.seq_next)
        sa["active"], sb["active"] = np.sort(sa["active"]), np.sort(sb["active"])
        eq(sa, sb)
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
def test_config3_ten_million(pkg, order):
    from .test_tile_geometry import config3_pool
    n = 10_000_000
    cfg, _ = pkg.synth.workload_config("config3_10m_g32_5v5", order, n)
    ids, rating, mode, ts = config3_pool(pkg, n)
    rt = Ratings()
    rt.add(ids, rating)
    with pkg.Engine(cfg) as e:
        assert e.enqueue(ids, rating, mode, ts).all()
        res = e.tick(10 ** 6)
        q, _l = check(cfg, e, res, rt)
        assert q["n_lobbies"].sum() == res[3].n_lobbies > 900_000
