"""Queue move: mm_export_queues releases whole (mode, group) queues into an image, mm_merge loads it into a running
engine, shard.move_queues moves rating groups between ranks, and SearchPool.move_out / move_in carries the host state.

GPU: a source and a target driven by one schedule routed by queue give, queue by queue, what an engine that never
moved anything gives (lobbies in emission order, in_queue, pool_read, the waiting section of queue_stats, expire); the
source equals a twin that removed the moved ids; round trips; every refusal changes nothing; rejected ids; sharded
runs with balanced_owners + move_queues; config3 at 10 M players.  CPU: balanced_owners against a brute force, the
move_queues protocol over LocalComm threads with an engine double, and SearchPool.move_out / move_in.
"""
import ctypes as C
import importlib
import itertools
import threading

import numpy as np
import pytest

from .fakes import FakeBroker
from .test_expire import ExpiringEngine, publish
from .test_tile_geometry import DENSE, MODES8, WIDE

ARRIVAL, RATING = 0, 1
NO_DEDUPE = 1


def shard_mod():
    return importlib.import_module("microservice-matchmaking_b200.shard")


def queue_of(pkg, cfg, rating, mode):
    g = shard_mod().group_of_rating(cfg, rating)
    return np.asarray(mode, np.int64) * cfg.n_groups + g


# ================================================================================ GPU helpers
def move_config(pkg, kind, order, wide=False, capacity=200_000):
    flags = {"hashed": 0, "dense": DENSE, "no_dedupe": NO_DEDUPE}[kind] | (WIDE if wide else 0)
    return pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[:3], order=order, capacity=capacity,
                                 active_capacity=1_000_000, default_group=-1, flags=flags)


class Players:
    """Fresh players: ids unique over the test (dense handles or mixed 64-bit ids), uniform ratings, three modes."""

    def __init__(self, pkg, kind, rng):
        self.pkg, self.kind, self.rng, self.next = pkg, kind, rng, 0

    def batch(self, n, now):
        x = np.arange(self.next, self.next + n, dtype=np.uint64)
        self.next += n
        ids = x if self.kind == "dense" else self.pkg.synth.mix64(x + np.uint64(5 << 40))
        r = self.rng.integers(0, 5001, n).astype(np.int32)
        m = self.rng.integers(0, 3, n).astype(np.uint8)
        ts = (np.full(n, now, np.int64) - self.rng.integers(0, 80, n)).astype(np.uint32)
        return ids, r, m, ts


def per_queue_lobbies(pkg, cfg, res):
    """-> {queue: [member tuple, ...] in emission order (emit_seq ascending)}."""
    lob, mem, seq, _ = res
    out = {}
    order = np.argsort(seq, kind="stable")
    for k in order.tolist():
        h = lob[k]
        q = int(h["mode"]) * cfg.n_groups + int(h["group"])
        a = int(h["first_member"])
        out.setdefault(q, []).append(tuple(mem[a:a + int(h["n_members"])].tolist()))
    return out


def split(d, moved):
    return ({q: v for q, v in d.items() if q in moved}, {q: v for q, v in d.items() if q not in moved})


def pool_by_queue(pkg, cfg, eng, queues=None):
    """pool_read of these queues, queue by queue (enqueue order inside a queue: the order a move keeps)."""
    p = eng.pool_read()
    q = queue_of(pkg, cfg, p["rating"], p["mode"])
    sel = np.ones(len(q), bool) if queues is None else np.isin(q, list(queues))
    order = np.flatnonzero(sel)[np.argsort(q[sel], kind="stable")]
    return {k: v[order] for k, v in p.items()}


def same_pool(a, b):
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def waiting(eng, now, queues):
    qs = eng.queue_stats(now)
    return {q: (int(qs[q]["n_waiting"]), int(qs[q]["max_wait"]), qs[q]["wait_hist"].tolist()) for q in queues}


class Run:
    """A (source), B (target) and U (never moved): one schedule, routed by queue between A and B.  R is the twin of
    A that removes the moved ids instead of exporting them."""

    def __init__(self, pkg, kind, order, wide, spread, tick_impl, seed):
        self.pkg, self.kind = pkg, kind
        self.cfg = move_config(pkg, kind, order, wide)
        self.rng = np.random.default_rng(seed)
        self.P = Players(pkg, kind, self.rng)
        self.A, self.B, self.U, self.R = (pkg.Engine(self.cfg) for _ in range(4))
        for e in self.all():
            e.set_option("tick_impl", tick_impl)
            if spread >= 0:
                e.set_option("max_spread", spread)
        self.moved = set()
        self.now = 1000
        self.dedupe = kind != "no_dedupe"

    def all(self):
        return (self.A, self.B, self.U, self.R)

    def close(self):
        for e in self.all():
            e.close()

    def enqueue(self, n):
        ids, r, m, ts = self.P.batch(n, self.now)
        q = queue_of(self.pkg, self.cfg, r, m)
        to_b = np.isin(q, list(self.moved))
        for e, sel in ((self.A, ~to_b), (self.R, ~to_b), (self.B, to_b), (self.U, np.ones(n, bool))):
            if sel.any():
                e.enqueue(ids[sel], r[sel], m[sel], ts[sel])
        return ids

    def remove(self, ids):
        if self.dedupe:
            for e in self.all():
                e.remove(ids)

    def tick(self):
        self.now += 500
        res = {k: e.tick(self.now) for k, e in zip("ABUR", self.all())}
        la, lb, lu, lr = (per_queue_lobbies(self.pkg, self.cfg, res[k]) for k in "ABUR")
        mu, uu = split(lu, self.moved)
        assert split(lb, self.moved)[0] == mu and not split(lb, self.moved)[1]
        assert split(la, self.moved)[1] == uu and not split(la, self.moved)[0]
        if self.dedupe:  # the remove twin: the same calls, bit for bit
            assert lr == la
            for x, y in zip(res["A"][:3], res["R"][:3]):
                assert np.array_equal(x, y)
        assert res["A"][3].n_matched + res["B"][3].n_matched == res["U"][3].n_matched

    def take(self, ids):
        if self.dedupe:
            got = [e.take(ids) for e in self.all()]
            assert got[0] + got[1] == got[2] and got[0] == got[3]

    def expire(self, max_wait):
        if not self.dedupe:
            return
        got = {k: set(e.expire(self.now, max_wait)[0].tolist()) for k, e in zip("ABUR", self.all())}
        assert got["A"] | got["B"] == got["U"] and not got["A"] & got["B"] and got["A"] == got["R"]

    def check(self, sample):
        queues = set(range(self.cfg.n_modes * self.cfg.n_groups))
        stay = queues - self.moved
        same_pool(pool_by_queue(self.pkg, self.cfg, self.B, self.moved), pool_by_queue(self.pkg, self.cfg, self.U, self.moved))
        same_pool(pool_by_queue(self.pkg, self.cfg, self.A, stay), pool_by_queue(self.pkg, self.cfg, self.U, stay))
        if self.dedupe:
            same_pool(self.A.pool_read(), self.R.pool_read())
        assert waiting(self.B, self.now, self.moved) == waiting(self.U, self.now, self.moved)
        assert waiting(self.A, self.now, stay) == waiting(self.U, self.now, stay)
        if self.dedupe:
            qa, qr = self.A.queue_stats(self.now), self.R.queue_stats(self.now)
            for f in ("n_waiting", "n_removed", "max_wait", "wait_hist"):
                assert np.array_equal(qa[f], qr[f]), f
            assert np.array_equal(self.A.in_queue(sample) | self.B.in_queue(sample), self.U.in_queue(sample))
            assert not (self.A.in_queue(sample) & self.B.in_queue(sample) & ~self.U.in_queue(sample)).any()
            assert self.A.active_size() == self.R.active_size()

    def move(self, mask):
        img = self.A.export_queues(mask)
        h, cols = self.pkg.engine.read_image(img)
        assert h.magic == self.pkg.abi.MM_QUEUE_IMAGE_MAGIC and h.n_active == 0
        sel = set(np.flatnonzero(np.asarray(mask).reshape(-1)).tolist())
        assert set(queue_of(self.pkg, self.cfg, cols["rating"], cols["mode"]).tolist()) <= sel
        if self.dedupe:
            assert self.R.remove(cols["id"]) == h.n_players
            assert not self.A.in_queue(cols["id"]).any()
        rej = self.B.merge_queues(img)
        assert len(rej) == 0
        self.moved |= sel
        return img


MATRIX = [  # kind, order, wide, spread, tick_impl
    ("hashed", RATING, False, -1, 1), ("dense", RATING, False, 3, 0), ("hashed", RATING, True, 3, 1),
    ("dense", ARRIVAL, False, -1, 1), ("hashed", ARRIVAL, False, -1, 0), ("dense", RATING, True, -1, 0),
    ("no_dedupe", RATING, False, 3, 1), ("no_dedupe", ARRIVAL, True, -1, 0),
]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,order,wide,spread,tick_impl", MATRIX)
def test_moved_queues_behave_as_if_never_moved(pkg, kind, order, wide, spread, tick_impl):
    s = Run(pkg, kind, order, wide, spread, tick_impl, seed=11 + len(MATRIX) * order + tick_impl + 3 * wide)
    try:
        ids0 = s.enqueue(30_000)
        s.tick()
        ids1 = s.enqueue(20_000)
        # the target holds dead slots in queues it is about to receive
        G, M = s.cfg.n_groups, s.cfg.n_modes
        mask = s.rng.random((M, G)) < 0.4
        mask[0, 0], mask[0, 1] = True, False
        ids, r, m, ts = s.P.batch(4000, s.now)
        q = queue_of(pkg, s.cfg, r, m)
        inb = np.isin(q, np.flatnonzero(mask.reshape(-1)))
        s.B.enqueue(ids[inb], r[inb], m[inb], ts[inb])
        if s.dedupe:
            s.B.remove(ids[inb])
        else:
            s.B.tick(s.now)  # drops nothing without removals: start the target empty in the moved queues instead
            s.B.close()
            s.B = pkg.Engine(s.cfg)
            s.B.set_option("tick_impl", tick_impl)
            if spread >= 0:
                s.B.set_option("max_spread", spread)
        s.move(mask)
        s.check(np.concatenate([ids0[:3000], ids1[:3000]]))
        for k in range(5):
            new = s.enqueue(8000)
            if k % 2 == 0:
                s.remove(np.concatenate([ids1[k * 500:(k + 1) * 500], new[:200]]))
            else:
                s.take(np.concatenate([ids1[10_000 + k * 300:10_000 + (k + 1) * 300], new[300:400]]))
            s.tick()
            s.check(np.concatenate([ids1[:2000], new[:2000]]))
            if k == 3:
                s.expire(1500)
        s.tick()
    finally:
        s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense", "no_dedupe"])
@pytest.mark.parametrize("what", ["some", "none", "all"])
def test_round_trip_restores_the_source(pkg, kind, what):
    cfg = move_config(pkg, kind, RATING, False)
    rng = np.random.default_rng(len(kind) + len(what))
    P = Players(pkg, kind, rng)
    with pkg.Engine(cfg) as a, pkg.Engine(cfg) as u:
        for e in (a, u):
            e.set_option("max_spread", 2)
        for k in range(2):
            batch = P.batch(40_000, 100 * k)
            a.enqueue(*batch); u.enqueue(*batch)
            assert per_queue_lobbies(pkg, cfg, a.tick(100 * k + 50)) == per_queue_lobbies(pkg, cfg, u.tick(100 * k + 50))
        mask = {"some": rng.random((cfg.n_modes, cfg.n_groups)) < 0.5, "none": np.zeros((cfg.n_modes, cfg.n_groups)),
                "all": np.ones((cfg.n_modes, cfg.n_groups))}[what]
        img = a.export_queues(mask)
        h, _ = pkg.engine.read_image(img)
        assert (h.n_players == 0) == (what == "none")
        if what == "all":
            assert len(a.pool_read()["id"]) == 0
        assert len(a.merge_queues(img)) == 0
        same_pool(pool_by_queue(pkg, cfg, a), pool_by_queue(pkg, cfg, u))
        if kind != "no_dedupe":
            assert a.active_size() == u.active_size()
        for k in range(2, 5):
            batch = P.batch(20_000, 100 * k)
            a.enqueue(*batch); u.enqueue(*batch)
            assert per_queue_lobbies(pkg, cfg, a.tick(100 * k + 50)) == per_queue_lobbies(pkg, cfg, u.tick(100 * k + 50))
            same_pool(pool_by_queue(pkg, cfg, a), pool_by_queue(pkg, cfg, u))
            qa, qu = a.queue_stats(100 * k + 60), u.queue_stats(100 * k + 60)
            for f in ("n_waiting", "max_wait", "wait_hist"):
                assert np.array_equal(qa[f], qu[f]), f


def state_of(pkg, eng, kind):
    st = (eng.pool_size(), eng.active_size() if kind != "no_dedupe" else 0)
    idx, code = eng.enqueue_rejects()
    return st + (tuple(sorted(zip(idx.tolist(), code.tolist()))),)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
def test_refusals_change_nothing(pkg, kind):
    cfg = move_config(pkg, kind, RATING, False, capacity=60_000)
    rng = np.random.default_rng(5)
    P = Players(pkg, kind, rng)
    MM_E_ARG, MM_E_CAP, MM_E_STATE = pkg.abi.MM_E_ARG, pkg.abi.MM_E_CAP, pkg.abi.MM_E_STATE
    with pkg.Engine(cfg) as a, pkg.Engine(cfg) as b, pkg.Engine(cfg) as twin:
        batch = P.batch(30_000, 10)
        a.enqueue(*batch)
        tb = P.batch(5000, 10)
        tb[0][:3] = tb[0][0]  # a reject list on the target's last batch
        for e in (b, twin):
            e.enqueue(*tb)
        mask = np.zeros((cfg.n_modes, cfg.n_groups), bool)
        mask[:, 2] = True
        b_q = queue_of(pkg, cfg, tb[1], tb[2])
        live_on_b = np.isin(np.flatnonzero(mask.reshape(-1)), b_q).any()
        before = state_of(pkg, b, kind)

        def refused(buf, status):
            with pytest.raises(pkg.EngineError) as ei:
                b.merge_queues(buf)
            assert ei.value.status == status, str(ei.value)
            assert state_of(pkg, b, kind) == before

        # the target holds live players in group 2 of some mode: a move of group 2 is refused
        img = a.export_queues(mask)
        assert live_on_b
        refused(img, MM_E_STATE)
        # a full image, a truncated one, a corrupted header
        refused(a.export_state(), MM_E_ARG)
        refused(img[:-8], MM_E_ARG)
        with pkg.Engine(cfg) as fresh:
            with pytest.raises(pkg.EngineError) as ei:
                fresh.import_state(img)
            assert ei.value.status == MM_E_ARG
        other = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[:2], order=RATING,
                                      capacity=60_000, active_capacity=1_000_000, default_group=-1,
                                      flags=DENSE if kind == "dense" else 0)
        with pkg.Engine(other) as o:
            with pytest.raises(pkg.EngineError) as ei:
                o.merge_queues(img)
            assert ei.value.status == MM_E_ARG
        # a fresh target for the player checks (nothing live in the moved queues)
        with pkg.Engine(cfg) as c:
            cids = P.batch(10, 10)[0]
            c.enqueue(cids, np.full(10, 4500, np.int32), np.zeros(10, np.uint8))  # group 6: not moved
            cb = state_of(pkg, c, kind)
            for col, val in (("mode", 7), ("rating", 999_999), ("id", 2 ** 64 - 1 if kind == "hashed" else 10 ** 7)):
                bad = img.copy()
                h, cols = pkg.engine.read_image(bad)
                if h.n_players == 0:
                    continue
                cols[col][h.n_players // 2] = val
                with pytest.raises(pkg.EngineError) as ei:
                    c.merge_queues(bad)
                assert ei.value.status == MM_E_ARG, col
                assert state_of(pkg, c, kind) == cb
        # capacity: the pool, and the reject list's size
        small = move_config(pkg, kind, RATING, False, capacity=100)
        with pkg.Engine(small) as s:
            sb = state_of(pkg, s, kind)
            with pytest.raises(pkg.EngineError) as ei:
                s.merge_queues(img)
            assert ei.value.status == MM_E_CAP
            assert state_of(pkg, s, kind) == sb
        # export with a cap too small changes nothing; so does a staged packed batch
        n = C.c_uint64(0)
        m8 = np.ascontiguousarray(np.ones(cfg.n_modes * cfg.n_groups, np.uint8))
        buf = np.empty(1024, np.uint8)
        size0 = a.pool_size(), a.active_size()
        live0 = a.pool_read()["id"]
        rc = a.lib.mm_export_queues(a.h, m8.ctypes.data_as(C.c_void_p), buf.ctypes.data_as(C.c_void_p), 1024, C.byref(n))
        assert rc == MM_E_CAP and n.value > 1024
        rc = a.lib.mm_export_queues(a.h, m8.ctypes.data_as(C.c_void_p), None, 0, C.byref(n))
        assert rc == 0 and (a.pool_size(), a.active_size()) == size0
        assert np.array_equal(a.pool_read()["id"], live0)
        if kind == "dense":
            with pkg.Engine(cfg) as d:
                d.enqueue_packed_begin(np.arange(10, dtype=np.uint32) + 900_000, d.pack_key(np.full(10, 100), np.zeros(10)))
                with pytest.raises(pkg.EngineError) as ei:
                    d.export_queues(np.ones((cfg.n_modes, cfg.n_groups)))
                assert ei.value.status == MM_E_STATE
                with pytest.raises(pkg.EngineError) as ei:
                    d.merge_queues(img)
                assert ei.value.status == MM_E_STATE
                d.enqueue_packed_end()
        if kind == "hashed":  # the 3/4 load of a hashed active set
            tiny = type(cfg).from_buffer_copy(cfg)
            tiny.active_capacity = 1000  # 2048 slots: 1536 entries, fewer than the image's about 3000 players
            assert pkg.engine.read_image(img)[0].n_players > 1536
            with pkg.Engine(tiny) as t:
                t.enqueue(P.batch(5, 10)[0], np.full(5, 4500, np.int32), np.zeros(5, np.uint8))  # group 6: not moved
                tb0 = state_of(pkg, t, kind)
                with pytest.raises(pkg.EngineError) as ei:
                    t.merge_queues(img)
                assert ei.value.status == MM_E_CAP and "active set" in str(ei.value)
                assert state_of(pkg, t, kind) == tb0
        # the twin target was never touched by a refused call: the next batch and tick give the same results on both,
        # emit_seq numbers (the next enqueue's sequence numbers) included
        nb = P.batch(3000, 400)
        assert np.array_equal(b.enqueue(*nb), twin.enqueue(*nb))
        rb, rt = b.tick(500), twin.tick(500)
        for x, y in zip(rb[:3], rt[:3]):
            assert np.array_equal(x, y)


@pytest.mark.gpu
def test_rejected_ids_come_back_as_image_indices(pkg):
    cfg = move_config(pkg, "hashed", ARRIVAL, False)
    rng = np.random.default_rng(9)
    P = Players(pkg, "hashed", rng)
    with pkg.Engine(cfg) as a, pkg.Engine(cfg) as b:
        ids, r, m, ts = P.batch(20_000, 10)
        a.enqueue(ids, r, m, ts)
        mask = np.zeros((cfg.n_modes, cfg.n_groups), bool)
        mask[:, :3] = True
        img = a.export_queues(mask)
        h, cols = pkg.engine.read_image(img)
        # some moved ids are already active on the target, in a queue that is not moved
        dup = cols["id"][::97].copy()
        b.enqueue(dup, np.full(len(dup), 4500, np.int32), np.zeros(len(dup), np.uint8))
        b.enqueue(P.batch(7, 10)[0], np.full(7, 4600, np.int32), np.zeros(7, np.uint8))
        last = b.enqueue_rejects()
        # and the image repeats an id inside one partition
        img2 = img.copy()
        h2, c2 = pkg.engine.read_image(img2)
        p0 = int(np.flatnonzero(c2["part_count"] > 2)[0])
        first = int(c2["part_count"][:p0].sum())
        c2["id"][first + 2] = c2["id"][first]
        expect = set(range(0, h.n_players, 97)) | {first + 2}  # active here; the later copy of a repeated id
        rej = b.merge_queues(img2)
        assert list(rej) == sorted(rej) and set(rej.tolist()) == expect
        assert all(np.array_equal(x, y) for x, y in zip(b.enqueue_rejects(), last))
        got = b.pool_read()
        merged = np.setdiff1d(np.arange(h.n_players), rej)
        assert np.isin(c2["id"][merged], got["id"]).all()
        # the exact reject count decides the capacity check: the players that are not rejected fill the pool exactly
        exact = type(cfg).from_buffer_copy(cfg)
        exact.capacity = h.n_players
        with pkg.Engine(exact) as c:
            c.enqueue(dup, np.full(len(dup), 4500, np.int32), np.zeros(len(dup), np.uint8))
            assert c.pool_size() + h.n_players > exact.capacity
            rej = c.merge_queues(img)
            assert set(rej.tolist()) == set(range(0, h.n_players, 97))
            assert c.pool_size() == exact.capacity
            c.enqueue(P.batch(1, 10)[0], [4500], [0])
            assert c.enqueue_rejects()[1].tolist() == [3]  # full


# ================================================================================ GPU: shards
def sharded_run(pkg, K, move, seed=3, cap_of=None):
    """K engines in one process, rank 0 owning all groups but the last; a bell-shaped S1 pool leaves many players queued.
    move: after round 1, balanced_owners over the queue depths and move_queues on K threads."""
    shard = pkg.shard
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[:2], order=RATING, capacity=400_000,
                                active_capacity=1_000_000, default_group=-1)
    G = cfg.n_groups
    engines = []
    for r in range(K):
        c = type(cfg).from_buffer_copy(cfg)
        if cap_of is not None:
            c.capacity = cap_of(r)
        e = pkg.Engine(c)
        e.set_option("max_spread", 1)
        engines.append(e)
    owners = np.zeros(G, np.int64)  # a lopsided start: rank 0 holds all groups but the last
    owners[-1] = K - 1
    start = owners.copy()
    out, info = [], None
    try:
        for rnd in range(4):
            ids, r, _m, ts = pkg.synth.gen_pool(seed + rnd, 30_000, first=rnd * 30_000, bell=True)
            m = (np.arange(len(ids)) % 2).astype(np.uint8)
            own = shard.route(cfg, r, K, owners=owners)
            for k, e in enumerate(engines):
                sel = own == k
                e.enqueue(ids[sel], r[sel], m[sel], ts[sel])
            res = {}
            for e in engines:
                for q, v in per_queue_lobbies(pkg, cfg, e.tick(1000 * (rnd + 1))).items():
                    assert q not in res
                    res[q] = v
            out.append(res)
            if move and rnd == 1:
                load = sum(e.queue_stats(0)["n_waiting"].reshape(cfg.n_modes, G).sum(0) for e in engines)
                new = shard.balanced_owners(load, K)
                comm = shard.LocalComm()
                info = [None] * K

                def run(k):
                    info[k] = shard.move_queues(pkg, cfg, owners, new, k, engines[k], comm)
                th = [threading.Thread(target=run, args=(k,)) for k in range(K)]
                for t in th:
                    t.start()
                for t in th:
                    t.join(timeout=300)
                owners = new.copy()
                for k in range(K):
                    for g in info[k]["failed"]:
                        owners[g] = start[g]
    finally:
        for e in engines:
            e.close()
    return out, info, owners


@pytest.mark.gpu
@pytest.mark.parametrize("K", [2, 4])
def test_sharded_rebalance_gives_the_unmoved_results(pkg, K):
    ref, _, _ = sharded_run(pkg, K, move=False)
    got, info, owners = sharded_run(pkg, K, move=True)
    assert got == ref
    moved = sorted(set(sum((i["moved"] for i in info), [])))
    assert moved and not any(i["failed"] for i in info)
    start = np.zeros(7, np.int64)
    start[-1] = K - 1
    assert not np.array_equal(owners, start) and len(set(owners.tolist())) > 2 - (K == 2)


@pytest.mark.gpu
@pytest.mark.parametrize("source_full", [False, True])
def test_refused_move_rolls_back(pkg, source_full):
    """The target is too small for the group: both ranks report it failed, and the source gives what a twin that never
    tried gives — also when the source's pool is full, so that an image it had released could not come back."""
    shard = shard_mod()
    cfg = move_config(pkg, "hashed", RATING, False, capacity=50_000 if source_full else 200_000)
    small = type(cfg).from_buffer_copy(cfg)
    small.capacity = 1000
    P = Players(pkg, "hashed", np.random.default_rng(4))
    batch = P.batch(50_000, 10)
    with pkg.Engine(cfg) as a, pkg.Engine(small) as b, pkg.Engine(cfg) as u:
        for e in (a, u):
            e.set_option("max_spread", 2)
            e.enqueue(*batch)
        old = np.zeros(cfg.n_groups, np.int64)
        new = old.copy()
        new[3] = 1
        comm, info = shard.LocalComm(), [None, None]
        th = [threading.Thread(target=lambda k=k, e=e: info.__setitem__(k, shard.move_queues(pkg, cfg, old, new, k, e, comm)))
              for k, e in enumerate((a, b))]
        for t in th:
            t.start()
        for t in th:
            t.join(timeout=300)
        assert info[0] == info[1] == {"moved": [], "failed": [3], "stranded": {}}
        assert b.pool_size() == 0 and a.pool_size() == u.pool_size()  # nothing was released: no dead slots
        if source_full:
            assert a.pool_size() == cfg.capacity
        same_pool(pool_by_queue(pkg, cfg, a), pool_by_queue(pkg, cfg, u))
        assert a.active_size() == u.active_size()
        assert per_queue_lobbies(pkg, cfg, a.tick(100)) == per_queue_lobbies(pkg, cfg, u.tick(100))


# ================================================================================ GPU: scale
@pytest.mark.gpu
def test_config3_ten_million_move_an_eighth(pkg):
    from .test_tile_geometry import config3_pool
    n = 10_000_000
    cfg = pkg.synth.make_config(n_groups=32, modes=(("5v5", 2, 5),), order=RATING, capacity=n,
                                active_capacity=n + 1024, flags=DENSE)
    ids, rating, mode, ts = config3_pool(pkg, n)
    with pkg.Engine(cfg) as a, pkg.Engine(cfg) as u:
        cfg_b = type(cfg).from_buffer_copy(cfg)
        cfg_b.capacity = n // 4
        with pkg.Engine(cfg_b) as b:
            for e in (a, u):
                e.set_option("max_spread", 0)
                e.enqueue(ids, rating, mode, ts)
            b.set_option("max_spread", 0)
            mask = np.zeros((1, 32), bool)
            mask[0, 12:16] = True
            img = a.export_queues(mask)
            assert len(b.merge_queues(img)) == 0
            moved = set(range(12, 16))
            la, lb, lu = (per_queue_lobbies(pkg, cfg, e.tick(10)) for e in (a, b, u))
            assert lb == split(lu, moved)[0] and la == split(lu, moved)[1]
            assert a.pool_size() + b.pool_size() == u.pool_size()


# ================================================================================ CPU: balanced_owners, route
def brute_owners(load, P):
    G = len(load)
    best = None
    for cuts in itertools.combinations_with_replacement(range(G + 1), P - 1):
        bounds = (0,) + cuts + (G,)
        own = np.empty(G, np.int64)
        loads = []
        for r in range(P):
            own[bounds[r]:bounds[r + 1]] = r
            loads.append(float(np.sum(load[bounds[r]:bounds[r + 1]])))
        key = (max(loads), tuple(own.tolist()))
        best = key if best is None or key < best else best
    return best


@pytest.mark.parametrize("G,P", [(1, 1), (3, 2), (5, 3), (7, 2), (7, 4), (8, 5)])
def test_balanced_owners_equals_brute_force(G, P):
    shard = shard_mod()
    rng = np.random.default_rng(G * 10 + P)
    for trial in range(40):
        load = rng.integers(0, 20, G) if trial % 3 else np.exp(-((np.arange(G) - G / 2) ** 2) / 3) * 1000 // 1
        load = np.asarray(load, np.float64)
        own = shard.balanced_owners(load, P)
        assert (np.diff(own) >= 0).all() and own.min() >= 0 and own.max() < P
        peak = max(float(load[own == r].sum()) for r in range(P))
        best = brute_owners(load, P)
        assert peak == best[0] and tuple(own.tolist()) == best[1]
        assert np.array_equal(shard.balanced_owners(load, P), own)  # deterministic


def test_route_without_owners_is_unchanged(pkg):
    shard = shard_mod()
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, default_group=-1)
    r = np.arange(-100, 5200, 7)
    for P in (1, 2, 3, 4):
        own = shard.owner_of_group(np.arange(cfg.n_groups), cfg.n_groups, P)
        assert np.array_equal(shard.route(cfg, r, P), shard.route(cfg, r, P, owners=own))
        grp = shard.group_of_rating(cfg, r)
        assert np.array_equal(shard.route(cfg, r, P), np.where(grp < 0, -1, own[np.maximum(grp, 0)]))
        for k in range(P):
            assert np.array_equal(shard.groups_of_rank(k, cfg.n_groups, P),
                                  shard.groups_of_rank(k, cfg.n_groups, P, owners=own))
    own = np.array([0, 0, 1, 1, 1, 1, 1])
    assert np.array_equal(shard.groups_of_rank(1, 7, 2, owners=own), [2, 3, 4, 5, 6])


# ================================================================================ CPU: engine double with queue images
def build_image(pkg, cfg, cols_by_queue):
    """A queue image with one partition per queue (the double's layout), 8-byte ids."""
    abi = pkg.abi
    n_parts = cfg.n_modes * cfg.n_groups
    cnt = np.array([len(cols_by_queue.get(q, ((),))[0]) for q in range(n_parts)], np.uint32)
    n = int(cnt.sum())
    off = abi.image_offsets(n_parts, n, 0, 8)
    buf = np.zeros(off[-1], np.uint8)
    h = abi.ImageHeader()
    h.magic, h.version, h.abi_version, h.id_bytes = abi.MM_QUEUE_IMAGE_MAGIC, abi.MM_IMAGE_VERSION, abi.MM_ABI_VERSION, 8
    h.total_bytes, h.n_parts, h.n_players, h.n_active, h.seq_next = off[-1], n_parts, n, 0, n + 1
    h.config = cfg
    buf[:C.sizeof(h)] = np.frombuffer(bytes(h), np.uint8)
    buf[off[0]:off[0] + 4 * n_parts] = cnt.view(np.uint8)
    cat = [np.concatenate([cols_by_queue[q][k] for q in range(n_parts) if q in cols_by_queue] or [np.zeros(0)])
           for k in range(4)]
    for k, (col, dt) in enumerate(zip(cat, (np.uint64, np.int32, np.uint32, np.uint8))):
        a = np.asarray(col, dt)
        sec = (1, 2, 3, 5)[k]
        buf[off[sec]:off[sec] + a.nbytes] = a.view(np.uint8)
    seq = np.arange(1, n + 1, dtype=np.uint32)
    buf[off[4]:off[4] + 4 * n] = seq.view(np.uint8)
    return buf


class MovingEngine(ExpiringEngine):
    """The CPU engine double with queue images (one partition per queue): export releases, merge appends."""

    def export_queues(self, mask):
        mask = np.asarray(mask, bool).reshape(-1)
        live = self.alive.astype(bool)
        grp = shard_mod().group_of_rating(self.cfg, self.q[1])
        q = self.q[2].astype(np.int64) * self.cfg.n_groups + grp
        sel = live & mask[np.maximum(q, 0)] & (grp >= 0)
        by_q = {}
        for k in np.unique(q[sel]).tolist():
            s = sel & (q == k)
            ids = self.q[0][s]
            by_q[k] = (ids, self.q[1][s], np.array([self.ts[p] for p in ids.tolist()], np.uint32), self.q[2][s])
        img = build_image(self.pkg, self.cfg, by_q)
        self.remove(np.concatenate([v[0] for v in by_q.values()]) if by_q else np.zeros(0, np.uint64))
        return img

    def queue_stats(self, now=0):
        out = np.zeros(self.cfg.n_modes * self.cfg.n_groups, [("n_waiting", "<u4")])
        live = self.alive.astype(bool)
        grp = shard_mod().group_of_rating(self.cfg, self.q[1][live])
        np.add.at(out["n_waiting"], self.q[2][live].astype(np.int64) * self.cfg.n_groups + grp, 1)
        return out

    def active_size(self):
        return len(self.active)

    def merge_queues(self, buf):
        h, cols = self.pkg.engine.read_image(np.array(buf, np.uint8))
        if self.refuse == "merge":  # refused after the room check passed (e.g. a CUDA error)
            raise self.pkg.EngineError(self.pkg.abi.MM_E_CUDA, "mm_merge")
        rej = []
        for i in range(h.n_players):
            acc = self.enqueue(cols["id"][i:i + 1], cols["rating"][i:i + 1], cols["mode"][i:i + 1], cols["enq_ts"][i:i + 1])
            if acc[0] != 1:
                rej.append(i)
        self.merged.append(h.n_players)
        return np.array(rej, np.uint32)


def moving_engine(pkg, refuse=None):
    def make(cfg):
        e = MovingEngine(cfg)
        e.pkg, e.refuse, e.merged = pkg, refuse, []
        return e
    return make


def protocol_setup(pkg, K, how):
    """K engine doubles, every group but the last moving up one rank; rank K - 1 refuses: at the room check ("room":
    its pool is full), at the merge ("merge"), or at the merge with a source that cannot take its image back either
    ("stranded": every engine refuses merges)."""
    shard = shard_mod()
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=ARRIVAL, capacity=10_000, default_group=-1)
    G = cfg.n_groups
    old = shard.owner_of_group(np.arange(G), G, K)
    new = (old + 1) % K
    new[-1] = old[-1]
    refuse_rank = K - 1
    engines = []
    for k in range(K):
        refuse = {"merge": "merge" if k == refuse_rank else None, "room": None, "stranded": "merge"}[how]
        engines.append(moving_engine(pkg, refuse=refuse)(cfg))
    rng = np.random.default_rng(K)
    ids = np.arange(1, 3001, dtype=np.uint64)
    r = rng.integers(0, 5001, 3000).astype(np.int32)
    m = rng.integers(0, 2, 3000).astype(np.uint8)
    own = shard.route(cfg, r, K, owners=old)
    for k, e in enumerate(engines):
        e.enqueue(ids[own == k], r[own == k], m[own == k], np.full((own == k).sum(), 5, np.uint32))
    if how == "room":
        e = engines[refuse_rank]
        e.cfg = type(cfg).from_buffer_copy(cfg)
        e.cfg.capacity = e.pool_size()
    return cfg, old, new, refuse_rank, engines, ids, r


def check_protocol(pkg, cfg, old, new, refuse_rank, engines, ids, r, info, before, how):
    shard = shard_mod()
    grp = shard.group_of_rating(cfg, r)
    for g in range(cfg.n_groups):
        src, dst = int(old[g]), int(new[g])
        if src == dst:
            continue
        if dst != refuse_rank and how != "stranded":
            key = "moved"
        else:
            key = "failed"
        assert g in info[src][key] and g in info[dst][key]
        gids = set(ids[grp == g].tolist())
        if how == "stranded" and key == "failed":  # in neither engine, but kept by the source: nothing is lost
            img = info[src]["stranded"][g]
            assert set(pkg.engine.read_image(img)[1]["id"].tolist()) == gids
            assert not any(gids & set(e.pool_read()["id"].tolist()) for e in engines)
            continue
        home = dst if key == "moved" else src
        for k, e in enumerate(engines):
            assert (gids <= set(e.pool_read()["id"].tolist())) == (k == home)
    if how != "stranded":
        assert set().union(*before) == set().union(*(set(e.pool_read()["id"].tolist()) for e in engines))
        assert not any(i["stranded"] for i in info)
    for k in range(len(engines)):  # ascending group order on every rank
        assert info[k]["moved"] == sorted(info[k]["moved"]) and info[k]["failed"] == sorted(info[k]["failed"])


@pytest.mark.parametrize("K", [2, 4])
@pytest.mark.parametrize("how", ["room", "merge", "stranded"])
def test_move_queues_protocol_over_threads(pkg, K, how):
    shard = shard_mod()
    cfg, old, new, refuse_rank, engines, ids, r = protocol_setup(pkg, K, how)
    before = [set(e.pool_read()["id"].tolist()) for e in engines]
    comm = shard.LocalComm()
    info = [None] * K
    th = [threading.Thread(target=lambda k=k: info.__setitem__(k, shard.move_queues(pkg, cfg, old, new, k, engines[k],
                                                                                      comm))) for k in range(K)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=60)
    assert all(i is not None for i in info), "deadlock"
    check_protocol(pkg, cfg, old, new, refuse_rank, engines, ids, r, info, before, how)


class FailingExport(MovingEngine):
    """A source whose export is refused (as mm_export_queues is while a packed batch is staged)."""

    def export_queues(self, mask):
        raise self.pkg.EngineError(self.pkg.abi.MM_E_STATE, "mm_export_queues")


def test_move_queues_refused_export_answers_the_target(pkg):
    shard = shard_mod()
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=ARRIVAL, capacity=1000, default_group=-1)
    a, b = FailingExport(cfg), MovingEngine(cfg)
    for e in (a, b):
        e.pkg, e.refuse, e.merged = pkg, None, []
    a.enqueue([1, 2, 3], [100, 110, 2100], [0, 0, 0], [5, 5, 5])
    old, new = np.zeros(cfg.n_groups, np.int64), np.zeros(cfg.n_groups, np.int64)
    new[0] = 1
    comm, info = shard.LocalComm(), [None, None]
    th = [threading.Thread(target=lambda k=k, e=e: info.__setitem__(k, shard.move_queues(pkg, cfg, old, new, k, e, comm)))
          for k, e in enumerate((a, b))]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=60)
    assert info[0]["failed"] == info[1]["failed"] == [0] and not info[0]["stranded"]
    assert sorted(a.pool_read()["id"].tolist()) == [1, 2, 3] and b.pool_size() == 0


def _gloo_move_worker(rank, world, port, how, q):
    import os
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    pkg = importlib.import_module("microservice-matchmaking_b200")
    shard = shard_mod()
    cfg, old, new, refuse_rank, engines, ids, r = protocol_setup(pkg, world, how)
    before = set(engines[rank].pool_read()["id"].tolist())
    info = shard.move_queues(pkg, cfg, old, new, rank, engines[rank], shard.DistComm())
    info = dict(info, stranded={g: np.asarray(v) for g, v in info["stranded"].items()})
    q.put((rank, info, before, engines[rank].pool_read()["id"]))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("how", ["room", "merge"])
def test_move_queues_over_a_gloo_process_group(pkg, world, how):
    import socket
    import torch.multiprocessing as mp
    sck = socket.socket()
    sck.bind(("127.0.0.1", 0))
    port = sck.getsockname()[1]
    sck.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_move_worker, args=(k, world, port, how, q)) for k in range(world)]
    for p in procs:
        p.start()
    got = dict((x[0], x[1:]) for x in (q.get(timeout=120) for _ in range(world)))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    cfg, old, new, refuse_rank, _engines, ids, r = protocol_setup(pkg, world, how)
    info = [got[k][0] for k in range(world)]
    pools = [set(np.asarray(got[k][2]).tolist()) for k in range(world)]
    grp = shard_mod().group_of_rating(cfg, r)
    for g in range(cfg.n_groups):
        src, dst = int(old[g]), int(new[g])
        if src == dst:
            continue
        key = "failed" if dst == refuse_rank else "moved"
        assert g in info[src][key] and g in info[dst][key]
        home = dst if key == "moved" else src
        gids = set(ids[grp == g].tolist())
        assert all((gids <= pools[k]) == (k == home) for k in range(world))
    assert set().union(*(got[k][1] for k in range(world))) == set().union(*pools)


# ================================================================================ CPU: SearchPool move
def boot_pool(pkg, eng, now, wall, **opts):
    sw = importlib.import_module("microservice-matchmaking_b200.search_worker")
    pool = sw.SearchPool(eng, ["1v1", "5v5"], list(pkg.synth.REFERENCE_GROUP_NAMES), flush_every_s=3600,
                         clock=lambda: now[0], wall_clock=lambda: wall[0], **opts)
    broker = FakeBroker()
    for g in pkg.synth.REFERENCE_GROUP_NAMES:
        sw.SearchWorker.start_link(broker, pool, {"group_name": g, "channel_name": f"search.{g}"})
    broker.bind(sw.EXCHANGE_FORWARD, sw.QUEUE_FORWARD, sw.QUEUE_FORWARD)
    return sw, pool, broker


def test_search_pool_move_out_and_in(pkg):
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=ARRIVAL, capacity=1000, default_group=-1)
    make = moving_engine(pkg)
    now_a, now_b, wall = [50.0], [900.0], [1_700_000_000.0]
    wall_a = wall_b = wall
    ea, eb = make(cfg), make(cfg)
    sw, pa, ba = boot_pool(pkg, ea, now_a, wall_a, timeout_ms=60_000)
    _, pb, bb = boot_pool(pkg, eb, now_b, wall_b, timeout_ms=60_000)
    for i in range(5):  # gold (2000..2499): moved; bronze stays
        publish(pkg, ba, cfg, f"g{i}", 2100 + i)
        publish(pkg, ba, cfg, f"b{i}", 100 + i)
    publish(pkg, ba, cfg, "g5", 2150, "5v5")  # alone in its queue: times out, counting its wait in the old pool
    publish(pkg, bb, cfg, "x0", 3100)
    publish(pkg, bb, cfg, "g4", 4200)  # already queued on the target: its moved copy is rejected
    bb.deliver_all()
    pb.flush()
    ba.deliver_all()
    pa.flush()
    now_a[0] += 20.0; wall[0] += 20.0
    blob = pa.move_out(["gold"])
    assert not pa._staged and all(pa.handles.lookup(f"g{i}") is None for i in range(5))
    assert all(pa.in_queue(f"b{i}") for i in range(5))
    now_b[0] += 5.0; wall[0] += 5.0
    with pytest.raises(ValueError):
        bad = bytearray(blob)
        bad[:8] = b"XXXXXXXX"
        pb.move_in(bytes(bad))
    assert pb.move_in(blob) == 5
    assert all(pb.in_queue(f"g{i}") for i in (0, 1, 2, 3, 5)) and pb.handles.lookup("g4") is not None
    assert pb.players[pb.handles.lookup("g4")]["rating"] == 4200  # the resident copy kept its document
    # handles were remapped: the engine holds this pool's handles, with stamps in this pool's clock
    for i in (0, 1, 2, 3, 5):
        h = pb.handles.lookup(f"g{i}")
        assert pb.players[h]["id"] == f"g{i}"
        wait = (pb.now_ms() - eb.ts[h]) & 0xFFFFFFFF
        assert 25_000 <= wait <= 25_000 + 10, wait  # 20 s in the old pool, 5 s in transit
    # a duplicate of a moved player is still answered
    publish(pkg, bb, cfg, "g0", 2100)
    bb.deliver_all()
    pb.flush()
    assert pb.stats["duplicates"] == 1
    # lobbies come out of the new pool with the same JSON a pool that never moved publishes
    pb.tick()
    got = [p for p, _ in bb.queues[sw.QUEUE_FORWARD]]
    assert len(got) == 2
    teams = [sorted(m["id"] for t in __import__("json").loads(p)["teams"].values() for m in t) for p in got]
    assert sorted(teams) == [["g0", "g1"], ["g2", "g3"]]
    # the timeout counts the time in the old pool: g5 has waited 25 s more than x0
    now_b[0] += 40.0
    pb.tick()
    assert pb.stats["timed_out"] == 1 and pb.handles.lookup("g5") is None and pb.handles.lookup("x0") is not None
    with pytest.raises(ValueError):
        other = sw.SearchPool(make(cfg), ["1v1"], list(pkg.synth.REFERENCE_GROUP_NAMES))
        other.move_in(blob)
