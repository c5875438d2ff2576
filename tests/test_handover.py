"""Pool hand-over: mm_export writes the queued players and the active set to a host image, mm_import loads it into a
fresh engine, and the imported engine goes on exactly as the source would have.

GPU: hand-overs inside the long mixed schedules of tests/test_tick_forms_and_schedules.py (the restatement drops its
dead entries, its reject list and its match section at that step; everything after must stay bit-exact); twin engines
driven by the same calls; the re-export of an imported engine; every refusal, each leaving the target fresh; config3
at 10 M players.  CPU: SearchPool.checkpoint / SearchPool.resume over the in-memory broker, with an engine double.
"""
import ctypes as C
import json
import pickle

import numpy as np
import pytest

from .fakes import FakeBroker
from .test_expire import ExpiringEngine, publish, responses
from .test_ingest import hashed_slots
from .test_tick_forms_and_schedules import SCHEDULES, Model, Schedule, check_state, check_tick
from .test_tile_geometry import DENSE, MODES8, WIDE

ARRIVAL, RATING = 0, 1
NO_DEDUPE = 1


def copy_config(cfg, **changes):
    c = type(cfg).from_buffer_copy(cfg)
    for k, v in changes.items():
        setattr(c, k, v)
    return c


def sections(pkg, img):
    return pkg.engine.read_image(np.array(img, np.uint8, copy=True))


# ================================================================================ GPU: hand-over inside the schedules
class HandoverModel(Model):
    def handover(self, cfg):
        """What an imported engine holds: the live queued entries, the active set and the sequence counter."""
        self.q = {k: v[self.q["alive"]] for k, v in self.q.items()}
        self.codes = np.zeros(0, np.uint8)  # the reject list is not carried
        self.match = None                   # nor the last tick's match section
        self.snap = None                    # nor the snapshot
        self.cfg = cfg
        self.hcap = hashed_slots(cfg)


class HandoverSchedule(Schedule):
    def __init__(self, pkg, oracle, cfg, rng, dense):
        super().__init__(pkg, oracle, cfg, rng, dense)
        self.m = HandoverModel(cfg, oracle, pkg.abi)
        self.base_cfg = cfg
        self.handovers = 0

    def handover(self):
        """Export, import into a fresh engine (every other time with twice the capacity), close the old engine."""
        old = self.eng
        img = old.export_state()  # with async_results on, the last tick's host copies may still be in flight
        self.handovers += 1
        cfg = copy_config(self.base_cfg, capacity=self.base_cfg.capacity * (2 if self.handovers % 2 else 1))
        new = self.pkg.Engine(cfg)
        new.import_state(img)
        if self.at is not None:
            self.at.wait()  # the old engine's pending results are complete and correct
        old.close()
        self.eng, self.cfg = new, cfg
        self.m.handover(cfg)
        new.set_option("tick_impl", self.tick_impl)  # options are not in the image
        if self.m.spread >= 0:
            new.set_option("max_spread", self.m.spread)
        if self.async_on:
            new.set_option("async_results", 1)
            self.at = type(self.at)(self.pkg, new, cfg.capacity)
        check_state(new, self.m, self.now, self.sample()[:2000])


@pytest.mark.gpu
@pytest.mark.parametrize("dense,order,wide", SCHEDULES, ids=lambda v: str(v))
def test_handover_inside_long_mixed_schedule(pkg, oracle, dense, order, wide):
    rng = np.random.default_rng(300 + 4 * dense + 2 * order + wide)
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[:3], order=order, capacity=300_000,
                                active_capacity=4_000_000, default_group=-1, flags=(DENSE if dense else 0) | WIDE * wide)
    s = HandoverSchedule(pkg, oracle, cfg, rng, dense)
    ops = []
    try:
        s.enqueue(200_000)
        for k in range(32):
            if k % 6 == 5:
                s.handover()
                ops.append("handover")
            elif k % 6 == 2:  # every hand-over cycle holds at least one tick
                s.now += 1000
                s.tick()
                check_state(s.eng, s.m, s.now, s.sample()[:2000])
                ops.append("tick")
            else:
                ops.append(s.step())
        s.tick()
        s.finish()
        check_state(s.eng, s.m, s.now, s.sample())
    finally:
        s.close()
    assert s.handovers == 5 and ops.count("tick") >= 6, ops


# ================================================================================ GPU: twin engines
def tick_both(a, b, now, packed=False):
    ra = a.tick_packed(now) if packed else a.tick(now)
    rb = b.tick_packed(now) if packed else b.tick(now)
    for x, y in zip(ra[:3], rb[:3]):
        assert np.array_equal(x, y)
    sa, sb = ra[3], rb[3]
    assert (sa.n_lobbies, sa.n_matched, sa.n_residual) == (sb.n_lobbies, sb.n_matched, sb.n_residual)
    return sa


def same_state(a, b, now, sample, dedupe=True):
    pa, pb = a.pool_read(), b.pool_read()
    for k in pa:
        assert np.array_equal(pa[k], pb[k]), k
    if dedupe:
        assert a.active_size() == b.active_size()
        assert np.array_equal(a.in_queue(sample), b.in_queue(sample))
    qa, qb = a.queue_stats(now), b.queue_stats(now)
    for f in ("mode", "group", "n_waiting", "max_wait", "wait_hist"):
        assert np.array_equal(qa[f], qb[f]), f


def twin_config(pkg, kind, order):
    flags = {"hashed": 0, "dense": DENSE, "no_dedupe": NO_DEDUPE}[kind]
    return pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[:3], order=order, capacity=100_000,
                                 active_capacity=400_000, default_group=-1, flags=flags)


def twin_ids(pkg, kind, k0, k1):
    x = np.arange(k0, k1, dtype=np.uint64)
    return x if kind == "dense" else pkg.synth.mix64(x + np.uint64(9 << 40))


def fill_source(pkg, eng, kind, rng, when):
    """A source engine with queued, matched (active, not queued), removed, taken and expired players, some ids offered
    twice; `when` picks where the image is taken."""
    def enq(ids, now):
        r = rng.integers(0, 5001, len(ids)).astype(np.int32)
        mo = rng.integers(0, 3, len(ids)).astype(np.uint8)
        return eng.enqueue(ids, r, mo, np.full(len(ids), now, np.uint32) - rng.integers(0, 50, len(ids)).astype(np.uint32))

    if when == "empty":
        return
    a = twin_ids(pkg, kind, 0, 40_000)
    enq(np.concatenate([a, a[:500]]) if kind == "no_dedupe" else a, 100)
    eng.tick(150)
    enq(twin_ids(pkg, kind, 40_000, 70_000), 200)
    if kind != "no_dedupe":
        q = eng.pool_read()["id"]
        eng.remove(q[:700])
        eng.take(q[700:1200])
    eng.expire(300, 240)
    if when == "restore":
        eng.snapshot()
        enq(twin_ids(pkg, kind, 70_000, 75_000), 310)
        eng.restore()
    if when == "async":  # the image is taken while this tick's host copies may be in flight
        eng.set_option("async_results", 1)
        n = max(eng.pool_size(), 1)
        bufs = (np.empty(n, pkg.engine.LOBBY_DTYPE), np.empty(n, np.uint64))
        eng.tick_raw(bufs[0].ctypes.data, n, bufs[1].ctypes.data, n, now=320)
        return bufs


TWINS = [("hashed", RATING, "plain"), ("dense", ARRIVAL, "plain"), ("hashed", ARRIVAL, "async"),
         ("dense", RATING, "restore"), ("no_dedupe", RATING, "plain"), ("hashed", RATING, "empty"),
         ("dense", ARRIVAL, "empty")]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,order,when", TWINS)
def test_twin_engines_give_the_same_results(pkg, kind, order, when):
    rng = np.random.default_rng(len(kind) + order)
    cfg = twin_config(pkg, kind, order)
    dedupe = kind != "no_dedupe"
    with pkg.Engine(cfg) as a:
        pending = fill_source(pkg, a, kind, rng, when)  # noqa: F841 (async: host arrays of the tick in flight)
        img = a.export_state()
        with pkg.Engine(copy_config(cfg, capacity=150_000)) as b:
            b.import_state(img)
            if when == "async":
                a.results_wait()
                a.set_option("async_results", 0)
            # re-export: the pool sections byte for byte, the active section as a set
            h1, s1 = sections(pkg, img)
            h2, s2 = sections(pkg, b.export_state())
            assert (h1.n_players, h1.n_active, h1.seq_next) == (h2.n_players, h2.n_active, h2.seq_next)
            for k in ("part_count", "id", "rating", "enq_ts", "seq", "mode"):
                assert np.array_equal(s1[k], s2[k]), k
            assert np.array_equal(np.sort(s1["active"]), np.sort(s2["active"]))
            if when == "empty":
                assert h1.n_players == 0 and h1.n_active == 0
            queued = a.pool_read()["id"]
            if dedupe:
                assert len(s1["active"]) == a.active_size() - len(queued)
            else:
                assert len(s1["active"]) == 0
            matched = s1["active"].astype(np.uint64)
            sample = np.concatenate([queued[::50], matched[::20], twin_ids(pkg, kind, 90_000, 90_100)])
            same_state(a, b, 400, sample, dedupe)
            # the same calls on both
            r = np.random.default_rng(5)
            for rnd in range(3):
                now = 500 + 100 * rnd
                ids = np.concatenate([twin_ids(pkg, kind, 80_000 + 5000 * rnd, 85_000 + 5000 * rnd),
                                      queued[:300], matched[:300], queued[:10]])
                rt = r.integers(0, 5200, len(ids)).astype(np.int32)
                mo = r.integers(0, 3, len(ids)).astype(np.uint8)
                ts = np.full(len(ids), now, np.uint32)
                assert np.array_equal(a.enqueue(ids, rt, mo, ts), b.enqueue(ids, rt, mo, ts))
                if dedupe:
                    cur = a.pool_read()["id"]
                    took = cur[1000:1400]
                    assert a.take(took) == b.take(took)
                    assert np.array_equal(a.in_queue(took), b.in_queue(took))
                    gone = np.concatenate([cur[:400], matched[300:500], took[:100]])
                    assert a.remove(gone) == b.remove(gone)
                ea, eb = a.expire(now, 520 - 40 * rnd), b.expire(now, 520 - 40 * rnd)
                oa, ob = np.argsort(ea[1]), np.argsort(eb[1])
                assert np.array_equal(ea[0][oa], eb[0][ob]) and np.array_equal(ea[1][oa], eb[1][ob])
                same_state(a, b, now, sample, dedupe)
                for impl in (1, 0):
                    a.set_option("tick_impl", impl); b.set_option("tick_impl", impl)
                    tick_both(a, b, now + impl, packed=kind == "dense" and impl == 0)
                    same_state(a, b, now + 5, sample, dedupe)
                matched = np.concatenate([matched, queued[:50]])


# ================================================================================ GPU: refusals
def refusal_source(pkg, dense):
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[:2], order=RATING, capacity=20_000,
                                active_capacity=50_000, default_group=-1, flags=DENSE if dense else 0)
    rng = np.random.default_rng(1)
    eng = pkg.Engine(cfg)
    ids = twin_ids(pkg, "dense" if dense else "hashed", 0, 12_000)
    eng.enqueue(ids, rng.integers(0, 5001, len(ids)).astype(np.int32), rng.integers(0, 2, len(ids)).astype(np.uint8),
                rng.integers(0, 100, len(ids)).astype(np.uint32))
    eng.tick(100)
    more = twin_ids(pkg, "dense" if dense else "hashed", 12_000, 18_000)
    eng.enqueue(more, rng.integers(0, 5001, len(more)).astype(np.int32), rng.integers(0, 2, len(more)).astype(np.uint8),
                rng.integers(100, 200, len(more)).astype(np.uint32))
    return cfg, eng


def assert_fresh_and_working(pkg, oracle, eng, cfg):
    """The target after a refusal: empty, and an enqueue + tick equal the oracle."""
    assert eng.pool_size() == 0 and eng.active_size() == 0 and len(eng.pool_read()["id"]) == 0
    rng = np.random.default_rng(2)
    n = 3000
    ids = np.arange(n, dtype=np.uint64) if cfg.flags & DENSE else pkg.synth.mix64(np.arange(n, dtype=np.uint64))
    rating, mode = rng.integers(0, 5001, n).astype(np.int32), rng.integers(0, cfg.n_modes, n).astype(np.uint8)
    assert (eng.enqueue(ids, rating, mode) == 1).all()
    ref = oracle.run_closed_form(cfg, ids, rating, mode)
    check_tick(ref, np.arange(n, dtype=np.uint32), *eng.tick())


def corrupt(pkg, img, what, cfg):
    """A copy of the image with one defect."""
    x = np.array(img, np.uint8, copy=True)
    h, s = pkg.engine.read_image(x)
    hv = x[:C.sizeof(pkg.abi.ImageHeader)].view(np.uint32)
    part = s["part_count"].astype(np.int64)
    first = int(np.nonzero(part)[0][0])  # a partition with players; its players are s[...][0 : part[first]]
    if what == "truncated":
        return x[:-8]
    if what == "magic":
        hv[0] ^= 1
    elif what == "version":
        hv[1] = 99
    elif what == "part_over_capacity":
        s["part_count"][first] += np.uint32(cfg.capacity + 1)
    elif what == "mode":
        s["mode"][3] = cfg.n_modes
    elif what == "rating":
        other = 4500 if s["rating"][0] < 3000 else 100  # another group, so another partition
        s["rating"][0] = other
    elif what == "handle":
        s["id"][5] = cfg.active_capacity
    elif what == "dup_within":
        s["id"][7] = s["id"][2]
    elif what == "dup_across":
        s["active"][0] = s["id"][4]
    elif what == "seq_order":
        s["seq"][[0, 1]] = s["seq"][[1, 0]]
    elif what == "seq_next":
        s["seq"][0] = h.seq_next
    else:
        raise AssertionError(what)
    return x


CORRUPT = ["truncated", "magic", "version", "part_over_capacity", "mode", "rating", "handle", "dup_within",
           "dup_across", "seq_order", "seq_next"]


@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True])
def test_refusals_leave_the_target_fresh(pkg, oracle, dense):
    abi = pkg.abi
    cfg, src = refusal_source(pkg, dense)
    with src:
        img = src.export_state()
        h, s = sections(pkg, img)
        assert h.n_players > 5000 and h.n_active > 5000
        # export: cap too small -> MM_E_CAP and the size; a staged packed batch -> MM_E_STATE
        n = C.c_uint64(0)
        small = np.empty(100, np.uint8)
        assert src.lib.mm_export(src.h, small.ctypes.data_as(C.c_void_p), 100, C.byref(n)) == abi.MM_E_CAP
        assert n.value == len(img)
        if dense:
            src.enqueue_packed_begin(np.arange(5, dtype=np.uint32), src.pack_key(np.full(5, 100), np.zeros(5)))
            with pytest.raises(pkg.EngineError) as ei:
                src.export_state()
            assert ei.value.status == abi.MM_E_STATE
            src.enqueue_packed_end()
            img = src.export_state()
            h, s = sections(pkg, img)
        # corrupted images
        for what in CORRUPT:
            if what == "handle" and not dense:
                continue
            with pkg.Engine(cfg) as t:
                with pytest.raises(pkg.EngineError) as ei:
                    t.import_state(corrupt(pkg, img, what, cfg))
                assert ei.value.status == abi.MM_E_ARG, what
                if what in ("mode", "dup_across", "seq_order"):
                    assert_fresh_and_working(pkg, oracle, t, cfg)
                else:
                    assert t.pool_size() == 0 and t.active_size() == 0
                    t.import_state(img)  # still fresh: the good image loads
                    assert t.pool_size() == h.n_players and t.active_size() == h.n_players + h.n_active
        # config fields
        G = cfg.n_groups
        changes = {"n_groups": dict(n_groups=G - 1), "group_lo": None, "group_hi": None,
                   "default_group": dict(default_group=2), "n_modes": dict(n_modes=1), "modes": None,
                   "order_mode": dict(order_mode=ARRIVAL), "flags": dict(flags=cfg.flags ^ WIDE)}
        for field, ch in changes.items():
            c = copy_config(cfg, **(ch or {}))
            if field == "group_lo":
                c.group_lo[3] += 1
            elif field == "group_hi":
                c.group_hi[3] -= 1
            elif field == "modes":
                c.modes[1].team_size += 1
            with pkg.Engine(c) as t:
                with pytest.raises(pkg.EngineError) as ei:
                    t.import_state(img)
                assert ei.value.status == abi.MM_E_ARG, field
                assert t.pool_size() == 0
        # capacity too small; a target that is not fresh
        with pkg.Engine(copy_config(cfg, capacity=h.n_players - 1)) as t:
            with pytest.raises(pkg.EngineError) as ei:
                t.import_state(img)
            assert ei.value.status == abi.MM_E_CAP
            assert_fresh_and_working(pkg, oracle, t, copy_config(cfg, capacity=h.n_players - 1))
        for how in ("enqueue", "restore", "import"):
            with pkg.Engine(cfg) as t:
                if how == "enqueue":
                    t.enqueue(np.array([1], np.uint64), np.array([100], np.int32), np.array([0], np.uint8))
                elif how == "restore":
                    t.snapshot(); t.restore()
                else:
                    t.import_state(img)
                with pytest.raises(pkg.EngineError) as ei:
                    t.import_state(img)
                assert ei.value.status == abi.MM_E_STATE, how


# ================================================================================ GPU: config3 at 10 M players
@pytest.mark.gpu
@pytest.mark.parametrize("target", ["same_device", "second_device"])
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
def test_config3_ten_million(pkg, order, target):
    import torch
    if target == "second_device" and torch.cuda.device_count() < 2:
        pytest.skip("one CUDA device visible: the import onto a second device is not exercised")
    n = 10_000_000
    cfg = pkg.synth.make_config(n_groups=32, modes=MODES8[3:4], order=order, capacity=n + 65536, active_capacity=2 * n,
                                flags=DENSE)
    _, rating, _, _ = pkg.synth.gen_pool(1, n)
    key = pkg.Engine.pack_key(rating, np.zeros(n, np.uint8))
    with pkg.Engine(cfg) as a:
        assert (a.enqueue_packed(np.arange(n, dtype=np.uint32), key, (np.arange(n) % 977).astype(np.uint32)) == 1).all()
        a.tick_packed(1000)  # about 1 M lobbies: their members stay in the active set
        second = np.arange(n, 2 * n, dtype=np.uint32)
        assert (a.enqueue_packed(second, key, (np.arange(n) % 991).astype(np.uint32)) == 1).all()
        a.remove_packed(second[::997])
        a.take(second[5::1009].astype(np.uint64))
        img = a.export_state()
        h, _ = sections(pkg, img)
        assert h.n_players > 9_900_000 and h.n_active > 9_900_000
        with pkg.Engine(copy_config(cfg, device=1 if target == "second_device" else 0)) as b:
            b.import_state(img)
            assert b.active_size() == a.active_size()
            again = np.arange(0, 20_000, dtype=np.uint32)  # matched ids: "already in the queue"
            assert np.array_equal(a.enqueue_packed(again, key[:20_000]), b.enqueue_packed(again, key[:20_000]))
            tick_both(a, b, 2000, packed=True)
            qa, qb = a.queue_stats(2001), b.queue_stats(2001)
            assert np.array_equal(qa["wait_hist"], qb["wait_hist"])


# ================================================================================ CPU: SearchPool hand-over
class ImagingEngine(ExpiringEngine):
    """The CPU engine double with an image of its own (any format: SearchPool treats it as opaque)."""

    def export_state(self):
        return pickle.dumps((self.q, self.alive, self.active, self.ts, self.dead_pending))

    def import_state(self, buf):
        assert not self.active and not len(self.q[0]), "import into a fresh engine"
        self.q, self.alive, self.active, self.ts, self.dead_pending = pickle.loads(bytes(buf))


def boot(pkg, make_engine, clock, wall, timeout_ms=None, blob=None):
    import importlib
    sw = importlib.import_module("microservice-matchmaking_b200.search_worker")
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=ARRIVAL, capacity=1000, active_capacity=4000)
    eng = make_engine(cfg)
    opts = dict(flush_every_s=3600, clock=clock, wall_clock=wall, timeout_ms=timeout_ms)
    names = (["1v1", "5v5"], list(pkg.synth.REFERENCE_GROUP_NAMES))
    pool = sw.SearchPool(eng, *names, **opts) if blob is None else sw.SearchPool.resume(eng, blob, *names, **opts)
    return sw, cfg, eng, pool


def start_workers(sw, broker, pool, pkg):
    broker.consumers.clear()  # the old pool's consumers are gone
    for g in pkg.synth.REFERENCE_GROUP_NAMES:
        sw.SearchWorker.start_link(broker, pool, {"group_name": g, "channel_name": f"search.{g}"})
    broker.bind(sw.EXCHANGE_FORWARD, sw.QUEUE_FORWARD, sw.QUEUE_FORWARD)
    for k, queues in broker.bindings.items():  # declaring a binding again is idempotent on a real broker
        broker.bindings[k] = list(dict.fromkeys(queues))


def traffic(pkg, make_engine, stop_at=None):
    """Four rounds of players, a tick each; with stop_at the pool is checkpointed in that round — after the round's
    deliveries were consumed but before they were ingested — and resumed in a new pool on a new engine."""
    now, wall = [0.0], [1_700_000_000.0]
    sw, cfg, eng, pool = boot(pkg, make_engine, lambda: now[0], lambda: wall[0])
    broker = FakeBroker()
    start_workers(sw, broker, pool, pkg)
    for step in range(4):
        for i in range(9):
            publish(pkg, broker, cfg, f"p{step}_{i}", 100 + 600 * i, "1v1" if i % 3 else "5v5")
        broker.deliver_all()
        if step == stop_at:
            staged = len(pool._staged)
            assert staged > 0
            blob = pool.checkpoint()
            assert not pool._staged and all(not ch.unacked for ch, _ in sum(broker.consumers.values(), []))
            eng.close()
            sw, cfg, eng, pool = boot(pkg, make_engine, lambda: now[0], lambda: wall[0], blob=blob)
            start_workers(sw, broker, pool, pkg)
        now[0] += 30.0
        wall[0] += 30.0
        pool.tick()
    assert pool.in_queue("p1_0") == (pool.handles.lookup("p1_0") is not None)
    pool.remove_user("p0_1")
    pool.tick()
    return broker, pool


@pytest.mark.parametrize("stop_at", [0, 2])
def test_resumed_pool_publishes_what_an_unstopped_pool_does(pkg, stop_at):
    ref_broker, ref_pool = traffic(pkg, ImagingEngine)
    broker, pool = traffic(pkg, ImagingEngine, stop_at)
    assert {q: list(v) for q, v in broker.queues.items()} == {q: list(v) for q, v in ref_broker.queues.items()}
    assert sorted(broker.acked) == sorted(ref_broker.acked) and broker.nacked == ref_broker.nacked
    assert pool.players == ref_pool.players and pool.handles.handle_of == ref_pool.handles.handle_of


@pytest.mark.gpu
def test_resumed_pool_on_the_gpu_engine(pkg):
    ref_broker, ref_pool = traffic(pkg, pkg.Engine)
    broker, pool = traffic(pkg, pkg.Engine, 2)
    assert {q: list(v) for q, v in broker.queues.items()} == {q: list(v) for q, v in ref_broker.queues.items()}
    assert sorted(broker.acked) == sorted(ref_broker.acked)
    assert pool.engine.active_size() == ref_pool.engine.active_size()
    assert np.array_equal(pool.engine.pool_read()["id"], ref_pool.engine.pool_read()["id"])


def test_duplicates_and_remove_after_resume(pkg):
    now, wall = [0.0], [1000.0]
    sw, cfg, eng, pool = boot(pkg, ImagingEngine, lambda: now[0], lambda: wall[0])
    broker = FakeBroker()
    start_workers(sw, broker, pool, pkg)
    publish(pkg, broker, cfg, "solo", 4500)
    publish(pkg, broker, cfg, "a", 2100, "5v5")
    broker.deliver_all()
    blob = pool.checkpoint()
    sw, cfg, eng, pool = boot(pkg, ImagingEngine, lambda: now[0], lambda: wall[0], blob=blob)
    start_workers(sw, broker, pool, pkg)
    assert pool.in_queue("solo") and pool.in_queue("a")
    publish(pkg, broker, cfg, "solo", 4500)  # "You are already in the queue."
    broker.deliver_all()
    pool.flush()
    assert pool.stats["duplicates"] == 1 and eng.pool_size() == 2
    assert pool.remove_user("a") == ("ok", "removed") and not pool.in_queue("a") and eng.pool_size() == 1
    publish(pkg, broker, cfg, "a", 2100, "5v5")  # queues again
    broker.deliver_all()
    pool.flush()
    assert pool.in_queue("a") and pool.stats["enqueued"] == 1


def test_waits_count_the_time_before_the_checkpoint(pkg):
    mono, wall = [50.0], [1000.0]
    sw, cfg, eng, pool = boot(pkg, ImagingEngine, lambda: mono[0], lambda: wall[0], timeout_ms=2000)
    broker = FakeBroker()
    start_workers(sw, broker, pool, pkg)
    publish(pkg, broker, cfg, "gm", 4500)
    broker.deliver_all()
    assert pool.tick() == 0
    mono[0] += 1.2
    wall[0] += 1.2
    blob = pool.checkpoint()                 # waited 1.2 s
    mono[0] = 7.0                            # another process: another monotonic clock
    wall[0] += 0.5                           # down for 0.5 s
    sw, cfg, eng, pool = boot(pkg, ImagingEngine, lambda: mono[0], lambda: wall[0], timeout_ms=2000, blob=blob)
    start_workers(sw, broker, pool, pkg)
    assert pool.now_ms() == 1700
    mono[0] += 0.299
    assert pool.tick() == 0 and pool.stats["timed_out"] == 0 and pool.in_queue("gm")
    mono[0] += 0.001                         # 1.2 + 0.5 + 0.3 s: the limit
    assert pool.tick() == 0 and pool.stats["timed_out"] == 1 and not pool.in_queue("gm")
    (doc, _), = responses(broker, "gm")
    assert doc["error"]["type"] == "MatchmakingError"


def test_window_schedule_keeps_enqueue_ages(pkg):
    import importlib
    sw = importlib.import_module("microservice-matchmaking_b200.search_worker")
    mono, wall = [10.0], [500.0]
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=RATING, capacity=1000)
    opts = dict(flush_every_s=3600, clock=lambda: mono[0], wall_clock=lambda: wall[0],
                window=sw.WindowSchedule(0, 100.0, 1000))
    names = (["1v1", "5v5"], list(pkg.synth.REFERENCE_GROUP_NAMES))
    pool = sw.SearchPool(ImagingEngine(cfg), *names, **opts)
    broker = FakeBroker()
    start_workers(sw, broker, pool, pkg)
    publish(pkg, broker, cfg, "x", 100)
    publish(pkg, broker, cfg, "y", 1400)
    broker.deliver_all()
    pool.tick()
    assert pool.last_spread == 0
    mono[0] += 3.0; wall[0] += 3.0
    blob = pool.checkpoint()
    mono[0] = 99.0; wall[0] += 2.0
    pool2 = sw.SearchPool.resume(ImagingEngine(cfg), blob, *names, **opts)
    start_workers(sw, broker, pool2, pkg)
    pool2.tick()
    assert pool2.last_spread == 500  # 5 s of wait, the downtime included
    state = json.loads(blob[16:16 + int.from_bytes(blob[8:16], "little")])
    assert state["enqueued_at"][0][1] == pytest.approx(3.0)
