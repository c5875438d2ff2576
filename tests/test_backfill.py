"""Backfill (mm_backfill / Engine.backfill / SearchPool.backfill): the open slots of running lobbies filled from their
queues, nearest rating first (oldest first on an arrival-order engine), requests served one at a time in index order.

CPU: a plain serialized restatement of the definition in include/mm_engine.h on hand-built cases, a vectorised numpy
restatement held equal to it on random cases, the ABI mirror, and SearchPool.backfill with an engine double.
GPU: twin engines (mm_backfill against mm_take of the restatement's ids) over both orders, both id kinds, wide groups
with and without MM_F_WIDE_PARTITIONS and overlapping groups with a default group; requeue of backfilled players; every
refusal; four engines routed by shard.owner_of_group against one; config3 at 10 M players.
"""
import ctypes as C

import numpy as np
import pytest

from .test_requeue import Src, export_sections, requeue_engine, cpu_pool, lobbies, members
from .test_tile_geometry import DENSE, MODES8, WIDE

RATING, ARRIVAL = 1, 0


# ================================================================================ restatements
def group_of(cfg, r):
    for g in range(cfg.n_groups):
        if cfg.group_lo[g] <= r <= cfg.group_hi[g]:
            return g
    return cfg.default_group


def clamp_bounds(cfg):
    return (min(cfg.group_lo[g] for g in range(cfg.n_groups)) - 1, max(cfg.group_hi[g] for g in range(cfg.n_groups)) + 1)


def restate_plain(cfg, ids, rating, mode, reqs):
    """The definition, one request and one candidate at a time.  ids / rating / mode: the live queued players in
    enqueue order; reqs: (mode, group, target, count, window) tuples.  -> (n_taken, [ids of request j])"""
    lo, hi = clamp_bounds(cfg)
    c = lambda x: min(max(int(x), lo), hi)  # noqa: E731
    taken, n_taken, out = set(), [], []
    queue = [(int(mode[i]), group_of(cfg, int(rating[i]))) for i in range(len(ids))]
    for (m, g, t, k, w) in reqs:
        cand = [i for i in range(len(ids)) if queue[i] == (m, g) and i not in taken]
        if cfg.order_mode == RATING:
            cand = [i for i in cand if w < 0 or abs(c(rating[i]) - c(t)) <= w]
            cand.sort(key=lambda i: (abs(c(rating[i]) - c(t)), c(rating[i]), i))
        got = cand[:k]
        taken.update(got)
        n_taken.append(len(got))
        out.append(np.array([ids[i] for i in got], np.uint64))
    return np.array(n_taken, np.uint32), out


def restate(cfg, ids, rating, mode, reqs):
    """The same definition on per-(queue, clamped rating) bins, as numpy arrays: every request consumes bins in
    (distance, rating) order; a bin gives its oldest untaken players.  reqs: arrays mode, group, target, count, window."""
    ids, rating, mode = np.asarray(ids, np.uint64), np.asarray(rating, np.int64), np.asarray(mode, np.int64)
    lo, hi = clamp_bounds(cfg)
    G = cfg.n_groups
    grp_lo = np.array([cfg.group_lo[g] for g in range(G)], np.int64)
    grp_hi = np.array([cfg.group_hi[g] for g in range(G)], np.int64)
    inside = (rating[:, None] >= grp_lo[None, :]) & (rating[:, None] <= grp_hi[None, :]) if G else None
    grp = np.where(inside.any(1), inside.argmax(1), cfg.default_group)
    key = np.clip(rating, lo, hi) if cfg.order_mode == RATING else np.zeros(len(ids), np.int64)
    queue = mode * G + grp
    order = np.lexsort((np.arange(len(ids)), key, queue))  # (queue, key, enqueue order)
    sq, sk, sid = queue[order], key[order], ids[order]
    starts = np.flatnonzero(np.r_[True, (sq[1:] != sq[:-1]) | (sk[1:] != sk[:-1])]) if len(ids) else np.zeros(0, int)
    ends = np.r_[starts[1:], len(ids)].astype(np.int64)
    bq, bk = sq[starts], sk[starts]
    used = np.zeros(len(starts), np.int64)
    qs = {q: np.flatnonzero(bq == q) for q in np.unique(bq)}
    m, g, t, k, w = (np.asarray(x, np.int64) for x in reqs)
    n_taken, out = np.zeros(len(m), np.uint32), []
    for j in range(len(m)):
        b = qs.get(int(m[j] * G + g[j]), np.zeros(0, np.int64))
        if cfg.order_mode == RATING:
            d = np.abs(bk[b] - min(max(int(t[j]), lo), hi))
            sel = np.lexsort((bk[b], d))
            b, d = b[sel], d[sel]
            if w[j] >= 0:
                b = b[d <= w[j]]
        rem = ends[b] - starts[b] - used[b]
        before = np.concatenate([[0], np.cumsum(rem)[:-1]]) if len(b) else rem
        take = np.clip(int(k[j]) - before, 0, rem)
        parts = [sid[starts[x] + used[x]:starts[x] + used[x] + n] for x, n in zip(b[take > 0], take[take > 0])]
        used[b] += take
        n_taken[j] = int(take.sum())
        out.append(np.concatenate(parts).astype(np.uint64) if parts else np.zeros(0, np.uint64))
    return n_taken, out


def cfg_of(pkg, order, groups=None, default_group=-1, flags=0, modes=2, capacity=200_000):
    return pkg.synth.make_config(groups=groups or pkg.synth.REFERENCE_GROUPS, modes=MODES8[:modes], order=order,
                                 capacity=capacity, active_capacity=1_000_000, default_group=default_group, flags=flags)


def as_arrays(reqs):
    return [np.array(c, np.int64) for c in zip(*reqs)]


def both(cfg, ids, rating, mode, reqs):
    a = restate_plain(cfg, ids, rating, mode, reqs)
    b = restate(cfg, ids, rating, mode, as_arrays(reqs))
    assert np.array_equal(a[0], b[0])
    for x, y in zip(a[1], b[1]):
        assert np.array_equal(x, y)
    return a


# ================================================================================ CPU: the definition, hand-built
def test_ties_go_to_the_lower_rating_then_the_older_player(pkg):
    cfg = cfg_of(pkg, RATING, groups=[(0, 1000)])
    ids = np.arange(10, 16, dtype=np.uint64)
    rating = [110, 90, 100, 90, 110, 100]
    n, out = both(cfg, ids, rating, [0] * 6, [(0, 0, 100, 6, -1)])
    assert out[0].tolist() == [12, 15, 11, 13, 10, 14]  # 100 x2, then distance 10: 90 (older first), then 110


def test_window_edge_is_inclusive(pkg):
    cfg = cfg_of(pkg, RATING, groups=[(0, 1000)])
    ids = np.arange(4, dtype=np.uint64)
    n, out = both(cfg, ids, [95, 105, 106, 94], [0] * 4, [(0, 0, 100, 10, 5)])
    assert n.tolist() == [2] and out[0].tolist() == [0, 1]
    n, out = both(cfg, ids, [95, 105, 106, 94], [0] * 4, [(0, 0, 100, 10, 0)])
    assert n.tolist() == [0]


def test_count_larger_than_the_queue_and_zero_count_and_empty_queue(pkg):
    cfg = cfg_of(pkg, RATING, groups=[(0, 999), (1000, 2000)])
    ids = np.arange(3, dtype=np.uint64)
    n, out = both(cfg, ids, [10, 20, 30], [0] * 3, [(0, 0, 0, 0, -1), (0, 0, 0, 100, -1), (0, 1, 1500, 3, -1),
                                                    (1, 0, 0, 3, -1)])
    assert n.tolist() == [0, 3, 0, 0] and out[1].tolist() == [0, 1, 2]


def test_requests_on_one_queue_consume_in_order(pkg):
    cfg = cfg_of(pkg, RATING, groups=[(0, 1000)])
    ids = np.arange(6, dtype=np.uint64)
    n, out = both(cfg, ids, [100, 100, 101, 99, 300, 100], [0] * 6, [(0, 0, 100, 2, -1), (0, 0, 100, 2, -1),
                                                                     (0, 0, 100, 5, 1)])
    assert [o.tolist() for o in out] == [[0, 1], [5, 3], [2]]


def test_default_group_players_at_clamped_keys(pkg):
    cfg = cfg_of(pkg, RATING, groups=[(0, 99), (100, 199)], default_group=1)
    ids = np.arange(5, dtype=np.uint64)
    # -50 and -7 clamp to -1 and sit in the default group; 5000 and 250 clamp to 200
    n, out = both(cfg, ids, [-50, 150, 5000, -7, 250], [0] * 5, [(0, 1, 10_000, 3, -1), (0, 1, -1000, 5, 0)])
    assert out[0].tolist() == [2, 4, 1] and out[1].tolist() == [0, 3]


def test_overlapping_groups_use_rating_distances(pkg):
    cfg = cfg_of(pkg, RATING, groups=[(0, 1000), (400, 600), (0, 2000)], default_group=-1)
    ids = np.arange(5, dtype=np.uint64)
    # group 2 holds 1001..2000 only (first match): 1001 is nearer to 300 than 1500, whatever the key index says
    n, out = both(cfg, ids, [300, 500, 1001, 1500, 1002], [0] * 5, [(0, 2, 300, 2, -1), (0, 0, 450, 9, 200)])
    assert out[0].tolist() == [2, 4] and out[1].tolist() == [1, 0]  # 500 is group 0's (first match)


def test_arrival_order_takes_the_oldest(pkg):
    cfg = cfg_of(pkg, ARRIVAL, groups=[(0, 1000)])
    ids = np.arange(5, dtype=np.uint64)
    n, out = both(cfg, ids, [900, 10, 500, 10, 10], [0, 0, 1, 0, 0], [(0, 0, 10, 2, -1), (0, 0, 0, 5, -1)])
    assert [o.tolist() for o in out] == [[0, 1], [3, 4]]


@pytest.mark.parametrize("seed", range(6))
def test_numpy_restatement_equals_the_plain_one(pkg, seed):
    rng = np.random.default_rng(seed)
    order = RATING if seed % 3 else ARRIVAL
    groups = [[(0, 99), (100, 299)], [(0, 200), (50, 120), (0, 400)], [(10, 60)]][seed % 3]
    cfg = cfg_of(pkg, order, groups=groups, default_group=len(groups) - 1 if seed % 2 else -1)
    n = 300
    rating = rng.integers(-30, 450, n)
    mode = rng.integers(0, 2, n)
    keep = np.array([group_of(cfg, int(r)) >= 0 for r in rating])
    ids = np.arange(n, dtype=np.uint64)[keep]
    rating, mode = rating[keep], mode[keep]
    reqs = [(int(rng.integers(0, 2)), int(rng.integers(0, len(groups))), int(rng.integers(-50, 500)),
             int(rng.integers(0, 12)), -1 if order == ARRIVAL or rng.random() < 0.4 else int(rng.integers(0, 40)))
            for _ in range(40)]
    both(cfg, ids, rating, mode, reqs)


def test_abi_mirror(pkg):
    abi = pkg.abi
    assert C.sizeof(abi.BackfillReq) == 16
    res, args = abi.PROTOTYPES["mm_backfill"]
    assert res is C.c_int and len(args) == 7


# ================================================================================ CPU: SearchPool.backfill
def backfill_engine(pkg):
    class BackfillEngine(requeue_engine(pkg)):
        """The engine double with backfill(): pool_read, the restatement, take."""

        def backfill(self, mode, group, target, count, window):
            p = self.pool_read()
            n, out = restate(self.cfg, p["id"], p["rating"], p["mode"], (mode, group, target, count, window))
            self.take(np.concatenate(out) if out else np.zeros(0, np.uint64))
            return n, out

    return BackfillEngine


def test_search_pool_backfill_flow(pkg):
    from .test_expire import publish
    now = [0.0]
    sw, cfg, eng, pool, broker = cpu_pool(pkg, lambda: now[0], engine=backfill_engine(pkg))
    for i, r in enumerate([100, 120, 130, 700, 900]):  # bronze 1v1, arrival order
        publish(pkg, broker, cfg, f"b{i}", r)
    broker.deliver_all()
    assert len(pool._staged) == 5
    out = pool.backfill([("1v1", "bronze", 0, 2), ("1v1", "bronze", 0, 1), ("5v5", "bronze", 0, 3)])
    assert not pool._staged  # staged deliveries flushed first
    assert [[d["id"] for d in docs] for docs in out] == [["b0", "b1"], ["b2"], []]
    assert pool.stats["backfilled"] == 3
    assert all(eng.in_queue([pool.handles.lookup(f"b{i}")])[0] for i in range(3))  # matched players stay active
    assert eng.pool_size() == 2
    # a backfilled player whose lobby did not start goes back; the other leaves
    assert pool.requeue(out[0]) == ["requeued", "requeued"]
    pool.remove_user("b2")
    assert not pool.in_queue("b2") and pool.requeue(out[1]) == ["gone"]
    now[0] += 1
    pool.tick()
    assert [members(lob) for lob in lobbies(broker, sw)] == [["b0", "b1"], ["b3", "b4"]]


# ================================================================================ GPU: twin engines
def gpu_config(pkg, order, kind, layout, capacity=200_000):
    flags = DENSE if kind == "dense" else 0
    if layout == "wide":
        return cfg_of(pkg, order, flags=flags | WIDE, modes=3, capacity=capacity)
    if layout == "split":
        return cfg_of(pkg, order, flags=flags, modes=3, capacity=capacity)
    return cfg_of(pkg, order, groups=[(0, 2000), (1000, 3000), (2500, 5000), (100, 200)], default_group=1,
                  flags=flags, modes=3, capacity=capacity)


def random_requests(rng, cfg, n, count_hi=6):
    m = rng.integers(0, cfg.n_modes, n)
    g = rng.integers(0, cfg.n_groups, n)
    t = rng.integers(-200, 5300, n)
    k = rng.integers(0, count_hi, n)
    w = np.where(rng.random(n) < 0.5, -1, rng.integers(0, 60, n)) if cfg.order_mode == RATING else np.full(n, -1)
    return m, g, t, k, w


def twin_backfill(pkg, src, reqs, sample):
    """Backfill on src.eng; a twin imported from the state before gets mm_take of the restatement's ids.  Both must
    agree everywhere after.  -> (the twin, the taken ids)"""
    a = src.eng
    b = pkg.Engine(src.cfg)
    b.import_state(a.export_state())
    p = a.pool_read()
    want_n, want = restate(src.cfg, p["id"], p["rating"], p["mode"], reqs)
    n, got = a.backfill(*reqs)
    assert np.array_equal(n, want_n)
    for x, y in zip(got, want):
        assert np.array_equal(x, y)
    ids = np.concatenate(want) if want else np.zeros(0, np.uint64)
    assert b.take(ids) == len(ids)
    same(a, b, src.now, np.concatenate([sample, ids]))
    return b, ids


def same(a, b, now, sample):
    pa, pb = a.pool_read(), b.pool_read()
    for k in pa:
        assert np.array_equal(pa[k], pb[k]), k
    assert a.active_size() == b.active_size()
    assert np.array_equal(a.in_queue(sample), b.in_queue(sample))
    qa, qb = a.queue_stats(now), b.queue_stats(now)
    for f in ("mode", "group", "n_waiting", "max_wait", "wait_hist"):
        assert np.array_equal(qa[f], qb[f]), f


def tick_same(a, b, now):
    ra, rb = a.tick(now), b.tick(now)
    for x, y in zip(ra[:3], rb[:3]):
        assert np.array_equal(x, y)


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
@pytest.mark.parametrize("kind", ["hashed", "dense"])
@pytest.mark.parametrize("layout", ["split", "wide", "overlap"])
def test_twin_engines(pkg, order, kind, layout):
    cfg = gpu_config(pkg, order, kind, layout)
    src = Src(pkg, cfg, kind, seed=7 + order)
    rng = np.random.default_rng(3)
    try:
        lo = -300 if layout == "overlap" else 0
        hi = 5400 if layout == "overlap" else 5001
        src.enqueue(*src.fresh(40_000, lo, hi))
        sample = src.eng.pool_read()["id"][::97]
        # a fresh, unticked pool
        b, ids = twin_backfill(pkg, src, random_requests(rng, cfg, 300), sample)
        tick_same(src.eng, b, src.now)
        b.close()
        # after ticks, with removed and taken players, then after a requeue (held chunks)
        mem = src.eng.tick(src.now)[1]
        src.enqueue(*src.fresh(30_000, lo, hi))
        live = src.eng.pool_read()["id"]
        src.eng.remove(live[::13])
        src.eng.take(live[5::17])
        b, ids = twin_backfill(pkg, src, random_requests(rng, cfg, 500, count_hi=40), sample)
        tick_same(src.eng, b, src.now)
        b.close()
        src.enqueue(*src.fresh(20_000, lo, hi))
        assert (src.requeue(mem[:3000]) == 1).all()
        b, ids = twin_backfill(pkg, src, random_requests(rng, cfg, 200, count_hi=500), sample)
        tick_same(src.eng, b, src.now)
        b.close()
    finally:
        src.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
def test_long_mixed_schedule(pkg, kind):
    cfg = gpu_config(pkg, RATING, kind, "split")
    src = Src(pkg, cfg, kind, seed=11, spread=3)
    rng = np.random.default_rng(5)
    b = pkg.Engine(cfg)
    b.set_option("max_spread", 3)
    try:
        matched = []
        for step in range(30):
            op = step % 5
            if op == 0:
                src.enqueue(*src.fresh(8000), engines=(b,))
            elif op == 1:
                ra, rb = src.eng.tick(src.now), b.tick(src.now)
                for x, y in zip(ra[:3], rb[:3]):
                    assert np.array_equal(x, y)
                matched.append(ra[1])
                src.now += 5
            elif op == 2:
                p = src.eng.pool_read()
                reqs = random_requests(rng, cfg, 100, count_hi=20)
                want_n, want = restate(cfg, p["id"], p["rating"], p["mode"], reqs)
                n, got = src.eng.backfill(*reqs)
                assert np.array_equal(n, want_n) and all(np.array_equal(x, y) for x, y in zip(got, want))
                ids = np.concatenate(want)
                assert b.take(ids) == len(ids)
                matched.append(ids)
            elif op == 3 and matched:
                back = matched[-1][::2]
                assert np.array_equal(src.requeue(back), src.requeue(back, eng=b))
            elif op == 4:
                live = src.eng.pool_read()["id"]
                gone = np.concatenate([live[::31]] + ([matched[0][::3]] if matched else []))
                assert src.eng.remove(gone) == b.remove(gone)
            same(src.eng, b, src.now, src.eng.pool_read()["id"][::50])
    finally:
        b.close()
        src.close()


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
def test_backfilled_players_requeue_to_the_same_export(pkg, order):
    cfg = gpu_config(pkg, order, "hashed", "split")
    src = Src(pkg, cfg, "hashed", seed=19)
    try:
        src.enqueue(*src.fresh(30_000))
        src.eng.tick(src.now)
        src.enqueue(*src.fresh(30_000))
        before = export_sections(pkg, src.eng)
        n, got = src.eng.backfill(*random_requests(np.random.default_rng(2), cfg, 400, count_hi=30))
        ids = np.concatenate(got)
        assert len(ids) == n.sum() > 0 and src.eng.in_queue(ids).all()
        assert (src.requeue(ids) == 1).all()
        after = export_sections(pkg, src.eng)
        assert before[0] == after[0] and np.array_equal(before[2], after[2])
        for k in before[1]:
            assert np.array_equal(before[1][k], after[1][k]), k
    finally:
        src.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense", "no_dedupe"])
def test_refusals_change_nothing(pkg, kind):
    abi = pkg.abi
    flags = {"hashed": 0, "dense": DENSE, "no_dedupe": 1}[kind]
    for order in (RATING, ARRIVAL):
        cfg = cfg_of(pkg, order, flags=flags, modes=3, capacity=50_000)
        with pkg.Engine(cfg) as e:
            ids = np.arange(20_000, dtype=np.uint64) if kind == "dense" else pkg.synth.mix64(np.arange(20_000, dtype=np.uint64))
            rng = np.random.default_rng(1)
            e.enqueue(ids, rng.integers(0, 5001, 20_000).astype(np.int32), rng.integers(0, 3, 20_000).astype(np.uint8))
            e.tick(0)
            before = export_sections(pkg, e)  # the active section is written unordered: compared sorted

            def call(reqs, cap=1 << 16):
                req = np.zeros(len(reqs), np.dtype([("mode", "u1"), ("group", "u1"), ("reserved", "<u2"),
                                                    ("count", "<u4"), ("target", "<i4"), ("window", "<i4")]))
                for i, r in enumerate(reqs):
                    req[i] = r
                n_taken = np.full(max(len(reqs), 1), 77, np.uint32)
                mem = np.empty(max(cap, 1), np.uint64)
                total = C.c_uint32(99)
                rc = e.lib.mm_backfill(e.h, len(reqs), req.ctypes.data_as(C.c_void_p),
                                       n_taken.ctypes.data_as(C.c_void_p), mem.ctypes.data_as(C.c_void_p), cap,
                                       C.byref(total))
                return rc, n_taken, total.value, e.lib.mm_last_error(e.h).decode()

            ok = (0, 0, 0, 3, 2500, -1)
            if kind == "no_dedupe":
                rc, _, total, msg = call([ok])
                assert rc == abi.MM_E_STATE and total == 0 and "NO_DEDUPE" in msg
            else:
                for bad, idx, text in (((3, 0, 0, 1, 0, -1), 1, "mode"), ((0, 7, 0, 1, 0, -1), 2, "group"),
                                       ((0, 0, 1, 1, 0, -1), 0, "reserved")):
                    rc, _, total, msg = call([ok] * idx + [bad])
                    assert rc == abi.MM_E_ARG and total == 0 and f"request {idx}" in msg and text in msg, msg
                rc, _, _, msg = call([ok, (0, 0, 0, 1, 0, 5)])
                assert (rc == abi.MM_E_ARG and "request 1" in msg) if order == ARRIVAL else rc == 0
                if order == RATING:
                    before = export_sections(pkg, e)
                # a dry run: member_cap = 0 answers the counts and takes nothing
                reqs = [(m, g, 0, 5, 2500 + 100 * g, -1) for m in range(3) for g in range(7)]
                rc, n_taken, total, msg = call(reqs, cap=0)
                assert rc == abi.MM_E_CAP and total == n_taken[:len(reqs)].sum() > 0 and "member_cap" in msg
                rc2, n2, total2, _ = call(reqs, cap=total - 1)
                assert rc2 == abi.MM_E_CAP and total2 == total and np.array_equal(n2, n_taken)
                rc, _, total, _ = call([])
                assert rc == 0 and total == 0
            after = export_sections(pkg, e)
            assert after[0] == before[0] and np.array_equal(after[2], before[2])
            for k in before[1]:
                assert np.array_equal(after[1][k], before[1][k]), k


@pytest.mark.gpu
def test_staged_packed_batch_is_refused(pkg):
    abi = pkg.abi
    cfg = cfg_of(pkg, RATING, flags=DENSE, modes=1, capacity=10_000)
    with pkg.Engine(cfg) as e:
        e.enqueue(np.arange(100, dtype=np.uint64), np.arange(100, dtype=np.int32) * 40, np.zeros(100, np.uint8))
        h = np.arange(100, 110, dtype=np.uint32)
        k = np.zeros(10, np.uint16)
        assert e.lib.mm_enqueue_packed_begin(e.h, 10, h.ctypes.data_as(C.c_void_p), k.ctypes.data_as(C.c_void_p),
                                             None) == 0
        req = np.zeros(1, np.dtype([("mode", "u1"), ("group", "u1"), ("reserved", "<u2"), ("count", "<u4"),
                                    ("target", "<i4"), ("window", "<i4")]))
        req["count"] = 3
        n_taken, mem, total = np.zeros(1, np.uint32), np.empty(8, np.uint64), C.c_uint32(0)
        rc = e.lib.mm_backfill(e.h, 1, req.ctypes.data_as(C.c_void_p), n_taken.ctypes.data_as(C.c_void_p),
                               mem.ctypes.data_as(C.c_void_p), 8, C.byref(total))
        assert rc == abi.MM_E_STATE and "staged" in e.lib.mm_last_error(e.h).decode()
        assert e.lib.mm_enqueue_packed_end(e.h, None, None) == 0
        assert e.backfill(0, 0, 0, 3)[0].tolist() == [3]


@pytest.mark.gpu
def test_four_engines_routed_by_owner_of_group_equal_one(pkg):
    from importlib import import_module
    shard = import_module("microservice-matchmaking_b200.shard")
    cfg = gpu_config(pkg, RATING, "hashed", "split")
    src = Src(pkg, cfg, "hashed", seed=23)
    ranks = [pkg.Engine(cfg) for _ in range(4)]
    try:
        ids, r, m, ts = src.fresh(60_000)
        src.enqueue(ids, r, m, ts)
        owner = shard.owner_of_group(np.array([group_of(cfg, int(x)) for x in r]), cfg.n_groups, 4)
        for k, e in enumerate(ranks):
            sel = owner == k
            assert e.enqueue(ids[sel], r[sel], m[sel], ts[sel]).all()
        reqs = random_requests(np.random.default_rng(8), cfg, 400, count_hi=25)
        n, got = src.eng.backfill(*reqs)
        dest = shard.owner_of_group(reqs[1], cfg.n_groups, 4)
        for k, e in enumerate(ranks):
            sel = np.flatnonzero(dest == k)
            nk, gk = e.backfill(*(x[sel] for x in reqs))
            assert np.array_equal(nk, n[sel])
            for j, x in zip(sel, gk):
                assert np.array_equal(x, got[j])
    finally:
        for e in ranks:
            e.close()
        src.close()


@pytest.mark.gpu
def test_config3_ten_million(pkg):
    from .test_tile_geometry import config3_pool
    n = 10_000_000
    cfg, mode_idx = pkg.synth.workload_config("config3_10m_g32_5v5", RATING, n)
    ids, rating, mode, ts = config3_pool(pkg, n)
    rng = np.random.default_rng(4)
    with pkg.Engine(cfg) as e:
        assert e.enqueue(ids, rating, mode, ts).all()
        for reqs in ((np.zeros(1000, np.int64), rng.integers(0, 32, 1000), rng.integers(0, 5001, 1000),
                      rng.integers(1, 6, 1000), np.where(rng.random(1000) < 0.5, -1, rng.integers(0, 20, 1000))),
                     (np.zeros(10_000, np.int64), np.full(10_000, 17), rng.integers(0, 5001, 10_000),
                      rng.integers(1, 6, 10_000), np.full(10_000, -1))):
            p = e.pool_read()
            want_n, want = restate(cfg, p["id"], p["rating"], p["mode"], reqs)
            got_n, got = e.backfill(*reqs)
            assert np.array_equal(got_n, want_n)
            assert np.array_equal(np.concatenate(got), np.concatenate(want))
        assert e.in_queue(np.concatenate(got)).all()  # matched players stay in the active set
