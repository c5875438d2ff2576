"""Search status (mm_locate / Engine.locate / SearchPool.search_status): one player's state, queue, wait, position
and the lobby the next tick gives it, answered on the device without reading the pool.

CPU: a numpy restatement of ahead / depth / the S0 prediction under a lobby budget, held equal to a plain
one-player-at-a-time restatement on random cases; the ABI mirror; SearchPool.search_status with an engine double,
every state included.
GPU: ahead / depth / columns against the live players of mm_export; the prediction against the real next tick over
both orders, S0 and S1, per-queue and per-mode budgets, both id kinds, wide groups with and without
MM_F_WIDE_PARTITIONS, overlapping groups with a default group, the tile-geometry configs, both tick forms, and after
every call that changes the pool; the states; no side effects (twin engines, async results); every refusal; config3 at
10 M players.
"""
import ctypes as C
from importlib import import_module

import numpy as np
import pytest

from .test_backfill import backfill_engine, clamp_bounds, group_of
from .test_requeue import Src, cpu_pool, export_sections
from .test_tile_geometry import DENSE, MODES8, WIDE, fallback_groups, many_partitions_pool, uniform_pool

RATING, ARRIVAL = 1, 0
STAYS = 0xFFFFFFFF
U32 = np.uint32


# ================================================================================ restatements
def apportion(budget, cand):
    """mm_set_lobby_budget's largest-remainder rule (shard.apportion), restated for the CPU tests."""
    c = np.asarray(cand, np.int64)
    total = int(c.sum())
    if total <= budget:
        return c.copy()
    prod = c * int(budget)
    a, rem = prod // total, prod % total
    a[np.lexsort((np.arange(len(c)), -rem))[:int(budget) - int(a.sum())]] += 1
    return a


def restate_plain(cfg, ids, rating, mode, seq, seq_next, bud_queue=None, bud_mode=None):
    """The definition, one player at a time (S0).  ids ... seq: the live queued players in any order.
    -> {id: (queue, ahead, depth, lobby, member)}"""
    lo, hi = clamp_bounds(cfg)
    G = cfg.n_groups
    c = lambda x: min(max(int(x), lo), hi)  # noqa: E731
    age = lambda i: (int(seq[i]) - int(seq_next)) & 0xFFFFFFFF  # noqa: E731
    key = (lambda i: (c(rating[i]), age(i))) if cfg.order_mode == RATING else (lambda i: (age(i),))
    queue = [int(mode[i]) * G + group_of(cfg, int(rating[i])) for i in range(len(ids))]
    lobbies = {}
    for q in set(queue):
        L = cfg.modes[q // G].teams * cfg.modes[q // G].team_size
        lobbies[q] = sum(1 for x in queue if x == q) // L
        if bud_queue is not None:
            lobbies[q] = min(lobbies[q], int(bud_queue[q]))
    if bud_mode is not None:
        for m in range(cfg.n_modes):
            got = apportion(int(bud_mode[m]), [lobbies.get(m * G + g, 0) for g in range(G)])
            for g in range(G):
                if m * G + g in lobbies:
                    lobbies[m * G + g] = int(got[g])
    out = {}
    for i in range(len(ids)):
        q = queue[i]
        mates = [j for j in range(len(ids)) if queue[j] == q]
        ahead = sum(1 for j in mates if key(j) < key(i))
        L = cfg.modes[q // G].teams * cfg.modes[q // G].team_size
        lob, mem = (ahead // L, ahead % L) if ahead < lobbies[q] * L else (STAYS, 0xFFFF)
        out[int(ids[i])] = (q, ahead, len(mates), lob, mem)
    return out


def restate(cfg, ids, rating, mode, seq, seq_next, bud_queue=None, bud_mode=None):
    """The same as columns: -> (queue, ahead, depth, lobby, member) int64 arrays in input order.  With both budgets
    None it covers S0; `lobby` / `member` are what the next S0 tick gives."""
    lo, hi = clamp_bounds(cfg)
    G = cfg.n_groups
    rating, mode = np.asarray(rating, np.int64), np.asarray(mode, np.int64)
    grp = import_module("microservice-matchmaking_b200.shard").group_of_rating(cfg, rating).astype(np.int64)
    queue = mode * G + grp
    age = (np.asarray(seq, np.uint32) - U32(seq_next)).astype(np.uint32).astype(np.int64)
    keys = (age, np.clip(rating, lo, hi), queue) if cfg.order_mode == RATING else (age, queue)
    order = np.lexsort(keys)
    nq = cfg.n_modes * G
    depth_q = np.bincount(queue, minlength=nq)
    first = np.concatenate([[0], np.cumsum(depth_q)[:-1]])
    ahead = np.empty(len(queue), np.int64)
    ahead[order] = np.arange(len(queue)) - first[queue[order]]
    L = np.array([cfg.modes[m].teams * cfg.modes[m].team_size for m in range(cfg.n_modes)], np.int64)
    Lq = np.repeat(L, G)
    lob_q = depth_q // Lq
    if bud_queue is not None:
        lob_q = np.minimum(lob_q, np.asarray(bud_queue, np.int64))
    if bud_mode is not None:
        for m in range(cfg.n_modes):
            lob_q[m * G:(m + 1) * G] = apportion(int(bud_mode[m]), lob_q[m * G:(m + 1) * G])
    Lp = Lq[queue]
    matched = ahead < lob_q[queue] * Lp
    lobby = np.where(matched, ahead // Lp, STAYS)
    member = np.where(matched, ahead % Lp, 0xFFFF)
    return queue, ahead, depth_q[queue], lobby, member


def cfg_of(pkg, order, groups=None, default_group=-1, flags=0, modes=3, capacity=200_000):
    return pkg.synth.make_config(groups=groups or pkg.synth.REFERENCE_GROUPS, modes=MODES8[:modes], order=order,
                                 capacity=capacity, active_capacity=1_000_000, default_group=default_group, flags=flags)


# ================================================================================ CPU
@pytest.mark.parametrize("seed", range(8))
def test_numpy_restatement_equals_the_plain_one(pkg, seed):
    rng = np.random.default_rng(seed)
    order = RATING if seed % 3 else ARRIVAL
    groups = [[(0, 99), (100, 299)], [(0, 200), (50, 120), (0, 400)], [(10, 60)]][seed % 3]
    cfg = cfg_of(pkg, order, groups=groups, default_group=len(groups) - 1 if seed % 2 else -1)
    n = 400
    rating = rng.integers(-30, 450, n)
    mode = rng.integers(0, 3, n)
    keep = np.array([group_of(cfg, int(r)) >= 0 for r in rating])
    ids = np.arange(n, dtype=np.uint64)[keep]
    rating, mode = rating[keep], mode[keep]
    seq_next = int(rng.integers(0, 2 ** 32))
    seq = ((seq_next - 1 - rng.permutation(4 * n)[:len(ids)]) & 0xFFFFFFFF).astype(np.uint32)  # distinct, across the wrap
    nq = cfg.n_modes * cfg.n_groups
    budgets = [(None, None), (rng.integers(0, 6, nq), None), (None, rng.integers(0, 9, cfg.n_modes)),
               (rng.integers(0, 8, nq), rng.integers(0, 12, cfg.n_modes))][seed % 4]
    got = restate(cfg, ids, rating, mode, seq, seq_next, *budgets)
    want = restate_plain(cfg, ids, rating, mode, seq, seq_next, *budgets)
    for i, x in enumerate(ids.tolist()):
        assert tuple(int(col[i]) for col in got) == want[x], x


def test_s0_reduction_without_budget(pkg):
    cfg = cfg_of(pkg, RATING, groups=[(0, 1000)], modes=4)  # mode 3: 5v5
    rating = np.array([500] * 23)
    q, ahead, depth, lobby, member = restate(cfg, np.arange(23), rating, np.full(23, 3), np.arange(23), 23)
    assert depth.tolist() == [23] * 23 and ahead.tolist() == list(range(23))
    assert lobby.tolist() == [a // 10 if a < 20 else STAYS for a in range(23)]


def test_abi_mirror(pkg):
    abi = pkg.abi
    assert C.sizeof(abi.PlayerStatus) == 36 == pkg.engine.PLAYER_STATUS_DTYPE.itemsize
    for f in pkg.engine.PLAYER_STATUS_DTYPE.names:
        assert getattr(abi.PlayerStatus, f).offset == pkg.engine.PLAYER_STATUS_DTYPE.fields[f][1], f
    res, args = abi.PROTOTYPES["mm_locate"]
    assert res is C.c_int and len(args) == 5 and abi.MM_LOCATE_STAYS == STAYS


def locating_engine(pkg):
    class LocatingEngine(backfill_engine(pkg)):
        """The engine double with locate(): the restatement over pool_read and its own sequence numbers."""

        def locate(self, ids, now=0):
            out = np.zeros(len(ids), pkg.engine.PLAYER_STATUS_DTYPE)
            out["lobby"], out["member"] = STAYS, 0xFFFF
            live = self.alive.astype(bool)
            qid, qr, qm = (a[live] for a in self.q)
            seq = np.array([self.seq_of[int(x)] for x in qid], np.uint32)
            cols = restate(self.cfg, qid, qr, qm, seq, self.ctr)
            at = {int(x): i for i, x in enumerate(qid)}
            for k, x in enumerate(np.asarray(ids, np.uint64).tolist()):
                if x in at:
                    i = at[x]
                    ts = int(self.ts[x])
                    w = (int(now) - ts) & 0xFFFFFFFF
                    out[k] = (1, qm[i], cols[0][i] % self.cfg.n_groups, 0, qr[i], ts, seq[i], w if w < 2 ** 31 else 0,
                              cols[1][i], cols[2][i], cols[3][i], cols[4][i], 0)
                elif x in self.active:
                    out[k]["state"] = 2
            return out

    return LocatingEngine


def test_search_pool_search_status(pkg):
    from .test_expire import publish
    now = [0.0]
    sw, cfg, eng, pool, broker = cpu_pool(pkg, lambda: now[0], engine=locating_engine(pkg))
    for i, r in enumerate([100, 120, 130, 700, 1600]):  # bronze x4, silver x1; 1v1, arrival order
        publish(pkg, broker, cfg, f"p{i}", r)
    broker.deliver_all()
    st = pool.search_status(["p0", "p4", "nobody"])
    assert len(pool._staged) == 5  # answered from the staging list, not flushed
    assert st[0] == dict(state="staged", game_mode="1v1", group="bronze", wait_ms=None, position=None,
                         queue_size=None, next_tick=None)
    assert st[1]["state"] == "staged" and st[1]["group"] == "silver"
    assert st[2]["state"] == "unknown" and st[2]["group"] is None
    pool.flush()
    now[0] += 0.25
    st = pool.search_status(["p0", "p1", "p2", "p3", "p4"])
    assert [s["state"] for s in st] == ["searching"] * 5
    assert [s["position"] for s in st] == [0, 1, 2, 3, 0] and [s["queue_size"] for s in st] == [4, 4, 4, 4, 1]
    assert all(s["wait_ms"] == 250 and s["game_mode"] == "1v1" for s in st)
    assert [s["next_tick"] for s in st] == [{"lobby": 0, "team": 0}, {"lobby": 0, "team": 1},
                                            {"lobby": 1, "team": 0}, {"lobby": 1, "team": 1}, None]
    pool.backfill([("1v1", "bronze", 0, 1)])  # p0 taken: matched until removed
    st = pool.search_status(["p0", "p1"])
    assert st[0]["state"] == "matched" and st[0]["next_tick"] is None and st[0]["position"] is None
    assert st[1]["position"] == 0
    pool.remove_user("p0")
    assert pool.search_status(["p0"])[0]["state"] == "unknown"
    pool.tick()
    st = pool.search_status(["p1", "p2", "p3", "p4"])
    assert [s["state"] for s in st] == ["matched", "matched", "searching", "searching"]


# ================================================================================ GPU
def live_players(pkg, eng):
    """The live queued players with their sequence numbers, from mm_export."""
    (n, _na, seq_next), s, _act = export_sections(pkg, eng)
    return s, seq_next


def check_locate(pkg, eng, cfg, now, spread=-1, budgets=(None, None), extra=()):
    """Locate every live player (and `extra` ids), check the restated columns, then tick and check the prediction.
    -> the tick's result."""
    s, seq_next = live_players(pkg, eng)
    ids = s["id"].astype(np.uint64)
    rec = eng.locate(np.concatenate([ids, np.asarray(extra, np.uint64)]), now)
    r, x = rec[:len(ids)], rec[len(ids):]
    q, ahead, depth, lobby, member = restate(cfg, ids, s["rating"], s["mode"], s["seq"], seq_next, *budgets)
    assert (r["state"] == 1).all()
    assert np.array_equal(r["mode"], s["mode"]) and np.array_equal(r["group"], q % cfg.n_groups)
    assert np.array_equal(r["rating"], s["rating"]) and np.array_equal(r["enq_ts"], s["enq_ts"])
    assert np.array_equal(r["seq"], s["seq"])
    w = (np.uint32(now & 0xFFFFFFFF) - s["enq_ts"].astype(np.uint32)).astype(np.int32)
    assert np.array_equal(r["wait"], np.maximum(w, 0).astype(np.uint32))
    assert np.array_equal(r["ahead"], ahead) and np.array_equal(r["depth"], depth)
    assert (r["reserved"] == 0).all() and (r["reserved2"] == 0).all()
    qs = eng.queue_stats(now)
    assert np.array_equal(r["depth"], qs["n_waiting"][q])
    if spread < 0:  # S0 (with or without a budget): the closed form
        assert np.array_equal(r["lobby"], lobby) and np.array_equal(r["member"], member)
    for y in x:  # the extra ids: not queued
        assert y["state"] != 1 and y["lobby"] == STAYS and y["member"] == 0xFFFF and y["ahead"] == y["depth"] == 0
    res = eng.tick(now)
    check_prediction(cfg, ids, r, res, eng)
    return res


def check_prediction(cfg, ids, rec, res, eng):
    lob, mem = res[0], res[1]
    G = cfg.n_groups
    got = {}
    count = {}
    for h in lob:
        q = int(h["mode"]) * G + int(h["group"])
        k = count.get(q, 0)
        count[q] = k + 1
        first, n = int(h["first_member"]), int(h["n_members"])
        for j, x in enumerate(mem[first:first + n].tolist()):
            got[x] = (k, j)
    want = {int(x): (int(a), int(b)) for x, a, b in zip(ids.tolist(), rec["lobby"], rec["member"]) if a != STAYS}
    assert want == got
    stays = {int(x) for x, a in zip(ids.tolist(), rec["lobby"]) if a == STAYS}
    assert {int(x) for x in eng.pool_read()["id"].tolist()} == stays


def gpu_config(pkg, order, kind, layout, capacity=200_000):
    flags = DENSE if kind == "dense" else 0
    if layout == "wide":
        return cfg_of(pkg, order, flags=flags | WIDE, capacity=capacity)
    if layout == "split":
        return cfg_of(pkg, order, flags=flags, capacity=capacity)
    return cfg_of(pkg, order, groups=[(0, 2000), (1000, 3000), (2500, 5000), (100, 200)], default_group=1,
                  flags=flags, capacity=capacity)


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
@pytest.mark.parametrize("kind", ["hashed", "dense"])
@pytest.mark.parametrize("layout", ["split", "wide", "overlap"])
def test_prediction_is_the_next_tick(pkg, order, kind, layout):
    cfg = gpu_config(pkg, order, kind, layout)
    lo, hi = (-300, 5400) if layout == "overlap" else (0, 5001)
    spreads = [-1, 0, 7, 60] if order == RATING else [-1]
    nq = cfg.n_modes * cfg.n_groups
    rng = np.random.default_rng(order * 7 + len(layout))
    for spread in spreads:
        for budgets in ((None, None), (rng.integers(0, 40, nq), None), (None, np.array([0, 150, 9])),
                        (rng.integers(0, 3, nq), np.array([5, 0, 1000]))):
            for impl in (1, 0):
                src = Src(pkg, cfg, kind, seed=3 + spread, spread=spread)
                try:
                    src.eng.set_option("tick_impl", impl)
                    src.eng.set_lobby_budget(*budgets)
                    src.enqueue(*src.fresh(30_000, lo, hi))
                    check_locate(pkg, src.eng, cfg, src.now, spread, budgets)
                    src.enqueue(*src.fresh(20_000, lo, hi))
                    check_locate(pkg, src.eng, cfg, src.now + 5, spread, budgets)
                finally:
                    src.close()
            if order == ARRIVAL or impl == 0 and spread > 0:
                break


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
@pytest.mark.parametrize("kind", ["hashed", "dense"])
def test_after_every_state_change(pkg, order, kind):
    cfg = gpu_config(pkg, order, kind, "split")
    spread = 20 if order == RATING else -1
    src = Src(pkg, cfg, kind, seed=31, spread=spread)
    rng = np.random.default_rng(9)
    try:
        def check(extra=()):
            return check_locate(pkg, src.eng, cfg, src.now, spread, extra=extra)

        src.enqueue(*src.fresh(40_000))
        res = check()
        matched = res[1]
        for _ in range(3):  # several ticks: compaction and generation bumps
            src.enqueue(*src.fresh(15_000))
            res = check()
        # removes and takes (dead slots); the removed ids are state 0, the taken ones state 2
        src.enqueue(*src.fresh(25_000))
        live = src.eng.pool_read()["id"]
        src.eng.remove(live[::13])
        taken = np.setdiff1d(live[5::17], live[::13])
        src.eng.take(taken)
        st = src.eng.locate(np.concatenate([live[::13], taken, matched[:100]]))
        assert (st["state"][:len(live[::13])] == 0).all() and (st["state"][len(live[::13]):] == 2).all()
        res = check(extra=live[::13])
        # requeue (rewritten partitions): matched players come back as state 1
        src.enqueue(*src.fresh(10_000))
        back = res[1][:3000]
        assert (src.eng.locate(back)["state"] == 2).all()
        assert (src.requeue(back) == 1).all()
        assert (src.eng.locate(back)["state"] == 1).all()
        check()
        # expire
        src.enqueue(*src.fresh(20_000))
        src.now += 40
        gone, _ = src.eng.expire(src.now, 70)
        assert len(gone) and (src.eng.locate(gone)["state"] == 0).all()
        check(extra=gone)
        # backfill and band match: taken players are state 2
        src.enqueue(*src.fresh(20_000))
        reqs = (rng.integers(0, 3, 200), rng.integers(0, 7, 200), rng.integers(0, 5000, 200), rng.integers(0, 9, 200),
                np.full(200, -1))
        _n, got = src.eng.backfill(*reqs)
        taken = np.concatenate(got)
        assert len(taken) and (src.eng.locate(taken)["state"] == 2).all()
        if order == RATING:
            _lob, bm, _t, _st = src.eng.band_match(40, 0, cfg.n_groups - 2)
            assert (src.eng.locate(bm)["state"] == 2).all()
        check()
        # export_queues moves queues out (state 0); merge brings them into another engine
        src.enqueue(*src.fresh(20_000))
        mask = np.zeros((cfg.n_modes, cfg.n_groups), bool)
        mask[1, 2] = mask[0, 5] = True
        img = src.eng.export_queues(mask)
        moved = pkg.engine.read_image(np.asarray(img, np.uint8))[1]["id"].astype(np.uint64)
        assert len(moved) and (src.eng.locate(moved)["state"] == 0).all()
        with pkg.Engine(cfg) as other:
            other.set_option("max_spread", spread)
            other.merge_queues(img)
            check_locate(pkg, other, cfg, src.now, spread)
        check(extra=moved)
        # import and import_regroup into fresh engines
        src.enqueue(*src.fresh(20_000))
        image = src.eng.export_state()
        with pkg.Engine(cfg) as imp:
            imp.set_option("max_spread", spread)
            imp.import_state(image)
            check_locate(pkg, imp, cfg, src.now, spread)
        cfg2 = cfg_of(pkg, order, groups=[(0, 999), (1000, 2999), (3000, 5000)], flags=cfg.flags)
        with pkg.Engine(cfg2) as rg:
            rg.set_option("max_spread", spread)
            rg.import_regroup(image)
            check_locate(pkg, rg, cfg2, src.now, spread)
        # never queued / out-of-range handles
        never = np.array([2 ** 40 + 5, 3, 999_999, 10 ** 7] if kind == "dense" else [12345, 2 ** 63 + 1], np.uint64)
        never = never[~src.eng.in_queue(never)]
        assert (src.eng.locate(never)["state"] == 0).all()
        check(extra=never)
    finally:
        src.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["long_rows", "many_partitions", "huge_domain", "huge_domain_split", "fallback",
                                  "many_chunks"])
def test_tile_geometry_configs(pkg, case):
    syn = pkg.synth
    spreads = (-1, 12)
    if case == "long_rows":  # one partition over every row
        cfg = syn.make_config(groups=[(0, 200)], modes=MODES8[3:4], order=RATING, capacity=1_200_000, default_group=0)
        pool = uniform_pool(pkg, 1, 1_000_000, 0, 200)
    elif case == "many_partitions":
        cfg = syn.make_config(groups=[(250 * g, 250 * g + 249) for g in range(20)], modes=MODES8, order=RATING,
                              capacity=2_200_000, default_group=-1)
        pool = many_partitions_pool(pkg)
    elif case in ("huge_domain", "huge_domain_split"):  # the tail parks its counts in global memory
        cfg = syn.make_config(groups=[(0, 20000)], modes=MODES8[3:4], order=RATING, capacity=300_000, default_group=0,
                              flags=WIDE if case == "huge_domain" else 0)
        pool = uniform_pool(pkg, 2, 250_000, -100, 20100)
    elif case == "fallback":  # more than 512 split partitions: whole segments, no chunk histograms
        cfg = syn.make_config(groups=fallback_groups(), modes=MODES8, order=RATING, capacity=300_000, default_group=-1)
        pool = uniform_pool(pkg, 3, 250_000, 0, 4999, n_modes=8)
    else:  # partitions of many chunks
        cfg = syn.make_config(n_groups=2, modes=MODES8[:1], order=RATING, capacity=700_000, default_group=-1)
        pool = uniform_pool(pkg, 4, 600_000, 0, 5000)
    for spread in spreads:
        with pkg.Engine(cfg) as e:
            e.set_option("max_spread", spread)
            ids, rating, mode, ts = pool
            assert e.enqueue(ids, rating, mode, ts).all()
            check_locate(pkg, e, cfg, 10, spread)
            e.remove(ids[::7])
            check_locate(pkg, e, cfg, 10, spread)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
def test_no_side_effects(pkg, kind):
    cfg = gpu_config(pkg, RATING, kind, "split")
    src = Src(pkg, cfg, kind, seed=41, spread=15)
    b = pkg.Engine(cfg)
    b.set_option("max_spread", 15)
    budget = np.full(cfg.n_modes * cfg.n_groups, 30, np.uint32)
    src.eng.set_lobby_budget(budget)
    b.set_lobby_budget(budget)
    rng = np.random.default_rng(2)
    probe = []

    def look():
        p = np.concatenate([src.eng.pool_read()["id"][::11]] + probe[-2:] + [np.array([7, 2 ** 50], np.uint64)])
        src.eng.locate(p, src.now)

    def compare():
        ea, eb = export_sections(pkg, src.eng), export_sections(pkg, b)
        assert ea[0] == eb[0] and np.array_equal(ea[2], eb[2])
        for k in ea[1]:
            assert np.array_equal(ea[1][k], eb[1][k]), k
        qa, qb = src.eng.queue_stats(src.now), b.queue_stats(src.now)
        assert qa.tobytes() == qb.tobytes()
        assert all(np.array_equal(x, y) for x, y in zip(src.eng.lobby_budget_report(), b.lobby_budget_report()))
        assert src.eng.pool_size() == b.pool_size() and src.eng.active_size() == b.active_size()
        ra, rb = src.eng.enqueue_rejects(), b.enqueue_rejects()  # (index, code), unordered
        assert sorted(zip(*(x.tolist() for x in ra))) == sorted(zip(*(x.tolist() for x in rb)))

    try:
        for step in range(16):
            op = step % 4
            if op == 0:
                ids, r, m, ts = src.fresh(12_000)
                ids[:50] = ids[50:100]  # repeats: a reject list
                assert np.array_equal(src.enqueue(ids, r, m, ts), b.enqueue(ids, r, m, ts))
            elif op == 1:
                look()
                ra, rb = src.eng.tick(src.now), b.tick(src.now)
                assert all(np.array_equal(x, y) for x, y in zip(ra[:3], rb[:3]))
                probe.append(ra[1][:500])
                src.now += 7
            elif op == 2:
                live = src.eng.pool_read()["id"]
                assert src.eng.remove(live[::29]) == b.remove(live[::29])
                assert src.eng.take(live[3::31]) == b.take(live[3::31])
            else:
                back = probe[-1][::3]
                assert np.array_equal(src.requeue(back), src.requeue(back, eng=b))
            look()
            compare()
        # between an async tick and its results_wait, and around a snapshot
        for e in (src.eng, b):
            e.set_option("async_results", 1)
            e.snapshot()
        n = src.eng.pool_size()
        out = []
        for e in (src.eng, b):
            lob = np.empty(n, pkg.engine.LOBBY_DTYPE)
            mem = np.empty(max(n, 1), np.uint64)
            st = pkg.abi.TickStats()
            assert e.lib.mm_tick(e.h, src.now, lob.ctypes.data_as(C.c_void_p), n, mem.ctypes.data_as(C.c_void_p), n,
                                 None, C.byref(st)) == 0
            if e is src.eng:
                look()
            e.results_wait()
            out.append((lob[:st.n_lobbies].copy(), mem[:st.n_matched].copy()))
        assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])
        compare()
        for e in (src.eng, b):
            e.restore()
        look()
        compare()
    finally:
        b.close()
        src.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense", "no_dedupe"])
def test_refusals(pkg, kind):
    abi = pkg.abi
    flags = {"hashed": 0, "dense": DENSE, "no_dedupe": 1}[kind]
    cfg = cfg_of(pkg, RATING, flags=flags, capacity=20_000)
    with pkg.Engine(cfg) as e:
        ids = np.arange(5000, dtype=np.uint64)
        e.enqueue(ids, (ids * 7 % 5000).astype(np.int32), (ids % 3).astype(np.uint8))
        out = np.zeros(4, pkg.engine.PLAYER_STATUS_DTYPE)
        q = ids[:4].copy()

        def call(n, p_ids, p_out):
            rc = e.lib.mm_locate(e.h, 0, n, p_ids, p_out)
            return rc, e.lib.mm_last_error(e.h).decode()

        vp = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        assert call(4, None, vp(out))[0] == abi.MM_E_ARG
        rc, msg = call(4, vp(q), None)
        assert rc == abi.MM_E_ARG and "null" in msg
        if kind == "no_dedupe":
            rc, msg = call(4, vp(q), vp(out))
            assert rc == abi.MM_E_STATE and "NO_DEDUPE" in msg
            return
        assert call(0, None, None)[0] == 0
        if kind == "dense":
            h = np.arange(6000, 6010, dtype=np.uint32)
            k = np.zeros(10, np.uint16)
            assert e.lib.mm_enqueue_packed_begin(e.h, 10, vp(h), vp(k), None) == 0
            rc, msg = call(4, vp(q), vp(out))
            assert rc == abi.MM_E_STATE and "staged" in msg and (out["state"] == 0).all()
            assert e.lib.mm_enqueue_packed_end(e.h, None, None) == 0
        assert call(4, vp(q), vp(out))[0] == 0 and (out["state"] == 1).all()
        assert e.lib.mm_locate(None, 0, 4, vp(q), vp(out)) == abi.MM_E_ARG


@pytest.mark.gpu
def test_repeated_ids_get_the_same_record(pkg):
    cfg = cfg_of(pkg, RATING, capacity=20_000)
    with pkg.Engine(cfg) as e:
        ids = pkg.synth.mix64(np.arange(8000, dtype=np.uint64))
        e.enqueue(ids, (np.arange(8000) % 5001).astype(np.int32), (np.arange(8000) % 3).astype(np.uint8))
        q = np.concatenate([ids[::5], ids[::5], ids[::5][:3]])
        r = e.locate(q, 3)
        k = len(ids[::5])
        assert r[:k].tobytes() == r[k:2 * k].tobytes() and r[:3].tobytes() == r[2 * k:].tobytes()


@pytest.mark.gpu
def test_config3_ten_million(pkg):
    from .test_tile_geometry import config3_pool
    n = 10_000_000
    cfg, _ = pkg.synth.workload_config("config3_10m_g32_5v5", RATING, n)
    ids, rating, mode, ts = config3_pool(pkg, n)
    with pkg.Engine(cfg) as e:
        assert e.enqueue(ids, rating, mode, ts).all()
        e.remove(ids[::101])
        check_locate(pkg, e, cfg, 10 ** 6)
