"""Widening search (mm_widen / Engine.widen / SearchPool(widen=...)): lobbies formed around the live queued players who
have waited at least their queue's min_wait, oldest first, each in a rating window that grows with its anchor's wait.

CPU: a plain restatement of the definition in include/mm_engine.h (one anchor and one candidate at a time), a numpy
restatement on per-(queue, rating) bins held equal to it on random pools, hand-built cases, the ABI mirror, and the
SearchPool flow with an engine double.
GPU: the engine against the restatement over both id kinds, split / wide / overlapping layouts, monotone and shuffled
stamps and several rule sets; a twin given mm_take of the returned ids; requeue of the members; a long mixed schedule;
every refusal; no side effects on the last tick's report; config3 at 10 M players.
"""
import ctypes as C

import numpy as np
import pytest

from .test_backfill import clamp_bounds, cfg_of, gpu_config, group_of, same, tick_same
from .test_requeue import Src, export_sections

RATING, ARRIVAL = 1, 0
OFF = 0xFFFFFFFF


# ================================================================================ restatements
def wait_of(now, ts):
    w = ((int(now) - int(ts)) & 0xFFFFFFFF)
    return 0 if w >= 1 << 31 else w


def window(rule, wait):
    min_wait, w0, step, inc, w_max = rule
    return min(w_max, w0 + (wait - min_wait) // step * inc)


def lobby_size(cfg, m):
    return cfg.modes[m].teams * cfg.modes[m].team_size


def restate_plain(cfg, ids, rating, mode, ts, now, rules):
    """The definition, one anchor and one candidate at a time.  ids / rating / mode / ts: the live queued players in age
    order; rules: {(mode, group): (min_wait, w0, step, inc, w_max)}.
    -> [(mode, group, [member ids])] in output order"""
    lo, hi = clamp_bounds(cfg)
    c = lambda x: min(max(int(x), lo), hi)  # noqa: E731
    queue = [(int(mode[i]), group_of(cfg, int(rating[i]))) for i in range(len(ids))]
    out = []
    for (m, g) in sorted(rules):
        L = lobby_size(cfg, m)
        U = [i for i in range(len(ids)) if queue[i] == (m, g)]
        live = set(U)
        A = [i for i in U if wait_of(now, ts[i]) >= rules[(m, g)][0]]
        for a in A:
            if a not in live:
                continue
            w = window(rules[(m, g)], wait_of(now, ts[a]))
            cand = [x for x in U if x in live and abs(c(rating[x]) - c(rating[a])) <= w]
            if len(cand) < L:
                continue
            cand.sort(key=lambda x: (abs(c(rating[x]) - c(rating[a])), c(rating[x]), x))
            lob = sorted(cand[:L], key=lambda x: (c(rating[x]), x))
            live.difference_update(lob)
            out.append((m, g, [int(ids[x]) for x in lob]))
    return out


def restate(cfg, ids, rating, mode, ts, now, rules):
    """The same definition on per-(queue, clamped rating) bins: a lobby takes the oldest untaken players of each bin it
    reaches, so a bin's taken players are a prefix of it and an anchor is absorbed when its rank in its bin lies in it.
    -> (lobbies as (mode, group, n_members, first_member), member ids u64, n_anchors, n_absorbed)"""
    ids, rating, mode = np.asarray(ids, np.uint64), np.asarray(rating, np.int64), np.asarray(mode, np.int64)
    ts = np.asarray(ts, np.int64)
    lo, hi = clamp_bounds(cfg)
    G = cfg.n_groups
    grp = np.array([group_of(cfg, int(r)) for r in rating], np.int64) if len(ids) else np.zeros(0, np.int64)
    key = np.clip(rating, lo, hi)
    w = (np.int64(now) - ts) & 0xFFFFFFFF
    wait = np.where(w >= 1 << 31, 0, w)
    lobbies, members, n_anc, n_abs = [], [], 0, 0
    for (m, g) in sorted(rules):
        rule = rules[(m, g)]
        L = lobby_size(cfg, m)
        sel = np.flatnonzero((mode == m) & (grp == g))  # age order
        if not len(sel):
            continue
        bk, inv = np.unique(key[sel], return_inverse=True)
        rank = np.zeros(len(sel), np.int64)
        for b in range(len(bk)):
            rank[inv == b] = np.arange(int((inv == b).sum()))
        bins = [sel[inv == b] for b in range(len(bk))]
        size = np.array([len(x) for x in bins], np.int64)
        used = np.zeros(len(bk), np.int64)
        for j in np.flatnonzero(wait[sel] >= rule[0]):
            n_anc += 1
            b = inv[j]
            if rank[j] < used[b]:
                n_abs += 1
                continue
            d = np.abs(bk - bk[b])
            order = np.lexsort((bk, d))
            order = order[d[order] <= window(rule, int(wait[sel[j]]))]
            rem = size[order] - used[order]
            if rem.sum() < L:
                continue
            before = np.concatenate([[0], np.cumsum(rem)[:-1]])
            take = np.clip(L - before, 0, rem)
            lob = []
            for x in np.sort(order[take > 0]):  # member order: rating, then age
                t = int(take[order == x][0])
                lob.append(ids[bins[x][used[x]:used[x] + t]])
                used[x] += t
            lobbies.append((m, g, L, sum(len(x) for x in members)))
            members.append(np.concatenate(lob))
    mem = np.concatenate(members).astype(np.uint64) if members else np.zeros(0, np.uint64)
    return lobbies, mem, n_anc, n_abs


def both(cfg, ids, rating, mode, ts, now, rules):
    a = restate_plain(cfg, ids, rating, mode, ts, now, rules)
    lob, mem, _, _ = restate(cfg, ids, rating, mode, ts, now, rules)
    assert [(m, g) for m, g, _ in a] == [(m, g) for m, g, _, _ in lob]
    flat = [x for _, _, ms in a for x in ms]
    assert flat == mem.tolist()
    return [ms for _, _, ms in a]


# ================================================================================ CPU: the definition, hand-built
def one_group(pkg, teams=1, team_size=2, groups=((0, 1000),), default_group=-1):
    cfg = cfg_of(pkg, RATING, groups=list(groups), default_group=default_group, modes=1)
    cfg.modes[0].teams, cfg.modes[0].team_size = teams, team_size
    return cfg


def test_window_edge_is_inclusive(pkg):
    cfg = one_group(pkg)
    ids = np.arange(3, dtype=np.uint64)
    # anchor 0 (rating 100) waits 10: window 5; 105 is inside, 106 not
    assert both(cfg, ids, [100, 106, 105], [0] * 3, [0, 10, 10], 10, {(0, 0): (10, 5, 1, 0, 5)}) == [[0, 2]]
    assert both(cfg, ids, [100, 106, 107], [0] * 3, [0, 10, 10], 10, {(0, 0): (10, 5, 1, 0, 5)}) == []


def test_ties_go_to_the_lower_rating_then_the_older_player(pkg):
    cfg = one_group(pkg, team_size=3)
    ids = np.arange(5, dtype=np.uint64)
    # anchor 100; candidates at distance 10: 110 (older), 90, 90 — the two 90s win, the older of them first
    out = both(cfg, ids, [100, 110, 90, 90, 110], [0] * 5, [0, 5, 5, 5, 5], 10, {(0, 0): (10, 10, 1, 0, 10)})
    assert out == [[2, 3, 0]]


def test_absorbed_anchor(pkg):
    cfg = one_group(pkg)
    ids = np.arange(4, dtype=np.uint64)
    lob, mem, n_anc, n_abs = restate(cfg, ids, [100, 101, 300, 301], [0] * 4, [0, 0, 0, 0], 50,
                                     {(0, 0): (0, 5, 1, 0, 5)})
    assert mem.tolist() == [0, 1, 2, 3] and n_anc == 4 and n_abs == 2
    both(cfg, ids, [100, 101, 300, 301], [0] * 4, [0, 0, 0, 0], 50, {(0, 0): (0, 5, 1, 0, 5)})


def test_all_or_nothing(pkg):
    cfg = one_group(pkg, teams=2, team_size=2)
    ids = np.arange(4, dtype=np.uint64)
    assert both(cfg, ids[:3], [100, 101, 102], [0] * 3, [0] * 3, 10, {(0, 0): (0, 50, 1, 0, 50)}) == []
    assert both(cfg, ids, [100, 101, 102, 103], [0] * 4, [0] * 4, 10, {(0, 0): (0, 50, 1, 0, 50)}) == [[0, 1, 2, 3]]


def test_floor_steps_and_the_cap(pkg):
    assert window((100, 5, 30, 7, 1000), 100) == 5
    assert window((100, 5, 30, 7, 1000), 129) == 5
    assert window((100, 5, 30, 7, 1000), 130) == 12
    assert window((100, 5, 30, 7, 20), 1000) == 20
    cfg = one_group(pkg)
    ids = np.arange(2, dtype=np.uint64)
    rule = {(0, 0): (100, 5, 30, 7, 20)}
    assert both(cfg, ids, [100, 112], [0, 0], [0, 1000], 129, rule) == []  # window 5
    assert both(cfg, ids, [100, 112], [0, 0], [0, 1000], 130, rule) == [[0, 1]]  # window 12
    assert both(cfg, ids, [100, 121], [0, 0], [0, 1000], 10_000, rule) == []  # capped at 20


def test_disabled_queues_are_not_touched(pkg):
    cfg = one_group(pkg, groups=((0, 99), (100, 199)))
    ids = np.arange(4, dtype=np.uint64)
    r = [10, 11, 150, 151]
    assert both(cfg, ids, r, [0] * 4, [0] * 4, 10, {(0, 1): (0, 5, 1, 0, 5)}) == [[2, 3]]
    assert both(cfg, ids, r, [0] * 4, [0] * 4, 10, {}) == []


def test_default_group_players_at_clamped_ratings(pkg):
    cfg = one_group(pkg, groups=((0, 99), (100, 199)), default_group=1)
    ids = np.arange(3, dtype=np.uint64)
    # 5000 and 250 both clamp to 200 and sit in the default group: distance 0 from each other
    assert both(cfg, ids, [5000, 150, 250], [0] * 3, [0, 0, 0], 10, {(0, 1): (0, 0, 1, 0, 0)}) == [[0, 2]]


def test_overlapping_groups_use_rating_distances(pkg):
    cfg = one_group(pkg, groups=((0, 1000), (400, 600), (0, 2000)))
    ids = np.arange(3, dtype=np.uint64)
    # group 2 holds 1001..2000 only: 1001 and 1300 are 299 apart whatever the key index says
    r = [1001, 500, 1300]
    assert both(cfg, ids, r, [0] * 3, [0] * 3, 10, {(0, 2): (0, 298, 1, 0, 298)}) == []
    assert both(cfg, ids, r, [0] * 3, [0] * 3, 10, {(0, 2): (0, 299, 1, 0, 299)}) == [[0, 2]]


def test_non_monotone_stamps_leave_the_anchor_out(pkg):
    cfg = one_group(pkg)
    ids = np.arange(3, dtype=np.uint64)
    # players 0 and 1 are older but were stamped later: only 2 is an anchor; its bin's two oldest form the lobby
    assert both(cfg, ids, [100, 100, 100], [0] * 3, [90, 90, 0], 50, {(0, 0): (50, 0, 1, 0, 0)}) == [[0, 1]]


@pytest.mark.parametrize("seed", range(6))
def test_numpy_restatement_equals_the_plain_one(pkg, seed):
    rng = np.random.default_rng(seed)
    groups = [[(0, 99), (100, 299)], [(0, 200), (50, 120), (0, 400)], [(10, 60)]][seed % 3]
    cfg = cfg_of(pkg, RATING, groups=groups, default_group=len(groups) - 1 if seed % 2 else -1)
    n = 300
    rating = rng.integers(-30, 450, n)
    mode = rng.integers(0, 2, n)
    keep = np.array([group_of(cfg, int(r)) >= 0 for r in rating])
    ids = np.arange(n, dtype=np.uint64)[keep]
    rating, mode = rating[keep], mode[keep]
    ts = rng.integers(0, 100, len(ids)) if seed % 2 else np.sort(rng.integers(0, 100, len(ids)))
    rules = {(m, g): (int(rng.integers(0, 60)), int(rng.integers(0, 5)), int(rng.integers(1, 20)),
                      int(rng.integers(0, 4)), 40) for m in range(2) for g in range(len(groups)) if rng.random() < 0.7}
    both(cfg, ids, rating, mode, ts, 100, rules)


def test_abi_mirror(pkg):
    abi = pkg.abi
    assert C.sizeof(abi.WidenRule) == 24 and C.sizeof(abi.WidenStats) == 32
    assert abi.WidenStats.device_us.offset == 16 and abi.WidenRule.w_max.offset == 16
    assert pkg.Engine.WIDEN_RULE_DTYPE.itemsize == 24
    res, args = abi.PROTOTYPES["mm_widen"]
    assert res is C.c_int and len(args) == 8


def test_symbol_exported(pkg):
    lib = pkg.engine.load_library()
    assert hasattr(lib, "mm_widen")


# ================================================================================ CPU: SearchPool(widen=...)
def widen_engine(pkg, calls):
    from .test_requeue import requeue_engine

    class WidenEngine(requeue_engine(pkg)):
        """The engine double with widen(): pool_read, the restatement, take.  Its tick emits nothing, so every lobby
        the pool publishes is a widen lobby; calls records the order of tick, widen and expire."""

        def tick(self, now=0, *a, **k):
            calls.append("tick")
            return np.zeros(0, pkg.engine.LOBBY_DTYPE), np.zeros(0, np.uint64), None, None

        def widen(self, now, rules):
            calls.append("widen")
            p = self.pool_read()
            ts = [self.ts[int(x)] for x in p["id"]]
            lob, mem, n_anc, n_abs = restate(self.cfg, p["id"], p["rating"], p["mode"], ts, now, rules)
            self.take(mem)
            out = np.zeros(len(lob), pkg.engine.LOBBY_DTYPE)
            for i, (m, g, n, first) in enumerate(lob):
                out[i] = (first, n, m, g)
            return out, mem, pkg.abi.WidenStats(n_anc, len(lob), len(mem), n_abs)

        def expire(self, now, max_wait, want_seq=True):
            calls.append("expire")
            return super().expire(now, max_wait, want_seq)

    return WidenEngine


def test_search_pool_widen_flow(pkg):
    import importlib
    from .fakes import FakeBroker
    from .test_expire import publish
    from .test_handover import start_workers
    from .test_requeue import lobbies, members
    sw = importlib.import_module("microservice-matchmaking_b200.search_worker")
    now, calls = [0.0], []
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=RATING, capacity=1000, active_capacity=4000)
    eng = widen_engine(pkg, calls)(cfg)
    # 1v1: an anchor after 1 s with a window of 10, growing by 10 every 0.5 s; the timeout drops players at 3 s
    pool = sw.SearchPool(eng, ["1v1", "5v5"], list(pkg.synth.REFERENCE_GROUP_NAMES), flush_every_s=3600,
                         clock=lambda: now[0], timeout_ms=3000, window=sw.WindowSchedule(0, 0, 0),
                         widen={"1v1": (1000, 10, 500, 10, 1000)})
    broker = FakeBroker()
    start_workers(sw, broker, pool, pkg)
    for i, r in enumerate([100, 125, 104, 700]):  # bronze 1v1
        publish(pkg, broker, cfg, f"p{i}", r)
    broker.deliver_all()
    assert pool.tick() == 0 and pool.stats["widened"] == 0  # nobody has waited 1 s
    now[0] = 1.2
    assert pool.tick() == 1  # p0 anchors: window 10 holds p2 (104), not p1 (125)
    assert [members(lob) for lob in lobbies(broker, sw)] == [["p0", "p2"]]
    assert pool.stats["widened"] == 1 and pool.stats["lobbies"] == 0
    h = [pool.handles.lookup(f"p{i}") for i in range(4)]
    assert h[0] in pool.matched_at and h[2] in pool.matched_at and h[1] in pool.enqueued_at  # window bookkeeping
    now[0] = 2.6  # p1 waited 2.6 s: its window of 10 + 3 x 10 = 40 holds no one left in its queue
    assert pool.tick() == 0
    assert calls == ["tick", "widen", "expire"] * 3  # widen runs after the tick's lobbies, before the timeout
    assert pool.requeue([d for d in members_docs(lobbies(broker, sw)[0])]) == ["requeued", "requeued"]


def test_search_pool_refuses_widen_on_an_arrival_order_engine(pkg):
    import importlib
    sw = importlib.import_module("microservice-matchmaking_b200.search_worker")
    names = (["1v1", "5v5"], list(pkg.synth.REFERENCE_GROUP_NAMES))
    for order, ok in ((ARRIVAL, False), (RATING, True)):
        cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=order, capacity=1000, active_capacity=4000)
        eng = widen_engine(pkg, [])(cfg)
        sw.SearchPool(eng, *names)  # without widen: any order
        if ok:
            sw.SearchPool(eng, *names, widen={"1v1": (1000, 10, 500, 10, 1000)})
        else:
            with pytest.raises(ValueError, match="MM_ORDER_RATING"):
                sw.SearchPool(eng, *names, widen={"1v1": (1000, 10, 500, 10, 1000)})


def members_docs(lobby):
    return [p for team in lobby["teams"].values() for p in team]


# ================================================================================ GPU
def rules_of(cfg, rules):
    out = np.zeros(cfg.n_modes * cfg.n_groups, [("min_wait", "<u4"), ("step", "<u4"), ("w0", "<i4"), ("inc", "<i4"),
                                                ("w_max", "<i4"), ("reserved", "<u4")])
    out["min_wait"], out["step"] = OFF, 1
    for (m, g), (min_wait, w0, step, inc, w_max) in rules.items():
        out[m * cfg.n_groups + g] = (min_wait, step, w0, inc, w_max, 0)
    return out


def rule_sets(cfg):
    G = cfg.n_groups
    return [
        {(m, g): (40, 0, 5, 2, 60) for m in range(cfg.n_modes) for g in range(G)},
        {(m, g): (20, 3, 1, 1, 500) for m in range(cfg.n_modes) for g in range(0, G, 2)},
        {(1, g): (55, 100, 10, 50, 100_000) for g in range(G)},
    ]


def check_widen(src, rules, now=None):
    """mm_widen on src.eng against the restatement of its pool -> the member ids"""
    now = src.now if now is None else now
    p = src.eng.pool_read()
    want_lob, want_mem, n_anc, n_abs = restate(src.cfg, p["id"], p["rating"], p["mode"], p["enq_ts"], now, rules)
    lob, mem, st = src.eng.widen(now, rules_of(src.cfg, rules))
    assert (st.n_anchors, st.n_absorbed, st.n_lobbies, st.n_matched) == (n_anc, n_abs, len(want_lob), len(want_mem))
    assert [tuple(int(x) for x in (h["mode"], h["group"], h["n_members"], h["first_member"])) for h in lob] == want_lob
    assert np.array_equal(mem, want_mem)
    return mem


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
@pytest.mark.parametrize("layout", ["split", "wide", "overlap"])
@pytest.mark.parametrize("stamps", ["monotone", "shuffled"])
def test_engine_equals_the_restatement_and_a_twin_take(pkg, kind, layout, stamps):
    cfg = gpu_config(pkg, RATING, kind, layout)
    src = Src(pkg, cfg, kind, seed=31)
    lo, hi = (-300, 5400) if layout == "overlap" else (0, 5001)

    def feed(n):
        ids, r, m, ts = src.fresh(n, lo, hi)
        if stamps == "monotone":
            ts = np.sort(ts)  # older entries never carry later stamps
        src.enqueue(ids, r, m, ts)

    total = 0
    try:
        feed(40_000)
        for k, rules in enumerate(rule_sets(cfg)):
            if k == 1:
                mem = src.eng.tick(src.now)[1]
                feed(20_000)
                live = src.eng.pool_read()["id"]
                src.eng.remove(live[::13])
                src.eng.take(live[5::17])
                assert (src.requeue(mem[:2000]) == 1).all()
            b = pkg.Engine(cfg)
            b.import_state(src.eng.export_state())
            sample = src.eng.pool_read()["id"][::97]
            ids = check_widen(src, rules)
            total += len(ids)
            assert b.take(ids) == len(ids)
            same(src.eng, b, src.now, np.concatenate([sample, ids]))
            loc_a, loc_b = src.eng.locate(np.concatenate([sample, ids]), src.now), b.locate(
                np.concatenate([sample, ids]), src.now)
            assert np.array_equal(loc_a, loc_b)
            tick_same(src.eng, b, src.now)
            assert np.array_equal(export_sections(pkg, src.eng)[1]["id"], export_sections(pkg, b)[1]["id"])
            b.close()
            src.now += 7
        assert total > 0
    finally:
        src.close()


@pytest.mark.gpu
def test_requeue_of_the_members_restores_the_export(pkg):
    cfg = gpu_config(pkg, RATING, "hashed", "split")
    src = Src(pkg, cfg, "hashed", seed=19)
    try:
        src.enqueue(*src.fresh(30_000))
        src.eng.tick(src.now)
        src.enqueue(*src.fresh(30_000))
        before = export_sections(pkg, src.eng)
        ids = check_widen(src, rule_sets(cfg)[0])
        assert len(ids) > 0 and src.eng.in_queue(ids).all()
        assert (src.eng.locate(ids, src.now)["state"] == 2).all()
        assert (src.requeue(ids) == 1).all()
        after = export_sections(pkg, src.eng)
        assert before[0] == after[0] and np.array_equal(before[2], after[2])
        for k in before[1]:
            assert np.array_equal(before[1][k], after[1][k]), k
    finally:
        src.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
def test_long_mixed_schedule(pkg, kind):
    cfg = gpu_config(pkg, RATING, kind, "split")
    src = Src(pkg, cfg, kind, seed=11, spread=3)
    b = pkg.Engine(cfg)
    b.set_option("max_spread", 3)
    rules = rule_sets(cfg)
    try:
        matched = []
        for step in range(36):
            op = step % 6
            if op == 0:
                src.enqueue(*src.fresh(8000), engines=(b,))
            elif op == 1:
                tick_same(src.eng, b, src.now)
                src.now += 5
            elif op == 2:
                ids = check_widen(src, rules[step % 3])
                assert b.take(ids) == len(ids)
                matched.append(ids)
            elif op == 3 and matched:
                back = matched[-1][::2]
                assert np.array_equal(src.requeue(back), src.requeue(back, eng=b))
            elif op == 4:
                live = src.eng.pool_read()["id"]
                gone = np.concatenate([live[::31]] + ([matched[0][::3]] if matched else []))
                assert src.eng.remove(gone) == b.remove(gone)
            elif op == 5:
                assert np.array_equal(np.sort(src.eng.expire(src.now, 58)[0]), np.sort(b.expire(src.now, 58)[0]))
            same(src.eng, b, src.now, src.eng.pool_read()["id"][::50])
    finally:
        b.close()
        src.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense", "no_dedupe"])
def test_refusals_change_nothing(pkg, kind):
    """Every refusal is checked against a twin engine that was given the same players and no widen call."""
    abi = pkg.abi
    flags = {"hashed": 0, "dense": 2, "no_dedupe": 1}[kind]

    def twins_agree(a, b, ids):
        pa, pb = a.pool_read(), b.pool_read()
        for k in pa:
            assert np.array_equal(pa[k], pb[k]), k
        assert a.active_size() == b.active_size()
        if kind != "no_dedupe":
            assert np.array_equal(a.in_queue(ids), b.in_queue(ids))
            assert np.array_equal(a.locate(ids, 100), b.locate(ids, 100))
        qa, qb = a.queue_stats(100), b.queue_stats(100)
        for f in qa.dtype.names:
            assert np.array_equal(qa[f], qb[f]), f

    for order in (RATING, ARRIVAL):
        cfg = cfg_of(pkg, order, flags=flags, modes=3, capacity=50_000)
        with pkg.Engine(cfg) as e, pkg.Engine(cfg) as b:
            ids = np.arange(20_000, dtype=np.uint64)
            if kind != "dense":
                ids = pkg.synth.mix64(ids)
            rng = np.random.default_rng(1)
            cols = (ids, rng.integers(0, 5001, 20_000).astype(np.int32), rng.integers(0, 3, 20_000).astype(np.uint8),
                    rng.integers(0, 100, 20_000).astype(np.uint32))
            for x in (e, b):
                x.enqueue(*cols)
                if kind != "no_dedupe":  # an MM_F_NO_DEDUPE engine has no active set to remove from
                    x.remove(ids[::29])
            good = rules_of(cfg, {(m, g): (30, 50, 1, 1, 200) for m in range(3) for g in range(cfg.n_groups)})

            def call(rules, lcap=1 << 14, mcap=1 << 16):
                lob = np.empty(max(lcap, 1), pkg.engine.LOBBY_DTYPE)
                mem = np.empty(max(mcap, 1), np.uint64)
                st = abi.WidenStats()
                rc = e.lib.mm_widen(e.h, 100, rules.ctypes.data_as(C.c_void_p), lob.ctypes.data_as(C.c_void_p), lcap,
                                    mem.ctypes.data_as(C.c_void_p), mcap, C.byref(st))
                return rc, st, e.lib.mm_last_error(e.h).decode()

            rc, _, msg = call(good, 0, 0)
            if order == ARRIVAL:
                assert rc == abi.MM_E_ARG and "MM_ORDER_RATING" in msg
            elif kind == "no_dedupe":
                assert rc == abi.MM_E_STATE and "NO_DEDUPE" in msg
            else:
                for field, value in (("step", 0), ("w0", -1), ("inc", -1), ("w_max", 40), ("reserved", 1)):
                    bad = good.copy()
                    bad[4][field] = value
                    rc, _, msg = call(bad)
                    assert rc == abi.MM_E_ARG and "rule 4" in msg, msg
                off = good.copy()
                off[4]["min_wait"], off[4]["step"] = OFF, 0  # a queue that is off is not checked
                off["min_wait"][5:] = OFF
                rc, st, msg = call(off, 0, 0)
                assert rc == abi.MM_E_CAP and st.n_lobbies > 0 and st.n_matched > 0 and "lobby_cap" in msg
                rc2, st2, _ = call(off, st.n_lobbies, st.n_matched - 1)
                assert rc2 == abi.MM_E_CAP and (st2.n_lobbies, st2.n_matched) == (st.n_lobbies, st.n_matched)
                rc3, st3, _ = call(off, st.n_lobbies - 1, st.n_matched)
                assert rc3 == abi.MM_E_CAP
            st = abi.WidenStats()
            assert e.lib.mm_widen(e.h, 100, None, None, 0, None, 0, C.byref(st)) == abi.MM_E_ARG
            assert e.lib.mm_widen(e.h, 100, good.ctypes.data_as(C.c_void_p), None, 0, None, 0, None) == abi.MM_E_ARG
            twins_agree(e, b, ids)
            if order == RATING and kind != "no_dedupe":
                ra, rb = e.widen(100, off), b.widen(100, off)  # the exact counts of the dry run, on both twins
                assert (ra[2].n_lobbies, ra[2].n_matched) == (st3.n_lobbies, st3.n_matched) == (rb[2].n_lobbies,
                                                                                              rb[2].n_matched)
                assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1])
                twins_agree(e, b, ids)
            tick_same(e, b, 100)
            twins_agree(e, b, ids)


@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True])
def test_between_async_tick_and_results_wait(pkg, packed):
    """A widen call between an async_results tick and mm_results_wait leaves the pending copies alone."""
    cfg = gpu_config(pkg, RATING, "dense", "split")
    src = Src(pkg, cfg, "dense", seed=12 + packed)
    try:
        with pkg.Engine(cfg) as b:
            src.enqueue(*src.fresh(30_000), engines=(b,))
            a = src.eng
            for x in (a, b):
                x.set_option("async_results", 1)
            ref = b.tick_packed(src.now) if packed else b.tick(src.now)
            n = a.pool_size()
            lob = np.empty(n, pkg.engine.LOBBY_DTYPE)
            mem = np.empty(n, np.uint32 if packed else np.uint64)
            seq = np.empty(n, np.uint32)
            st = a.tick_raw(lob.ctypes.data, n, mem.ctypes.data, n, seq.ctypes.data, now=src.now, packed=packed)
            src.enqueue(*src.fresh(20_000))  # the tick left too few players for a lobby: new ones arrive
            q0 = a.queue_stats(src.now + 50)
            got = check_widen(src, rule_sets(cfg)[0], now=src.now + 50)
            assert len(got) > 0
            q1 = a.queue_stats(src.now + 50)
            for f in ("n_lobbies", "n_matched", "max_match_wait", "match_wait_hist"):
                assert np.array_equal(q0[f], q1[f]), f
            a.results_wait()
            assert np.array_equal(lob[:st.n_lobbies], ref[0]) and np.array_equal(mem[:st.n_matched], ref[1])
            assert np.array_equal(seq[:st.n_lobbies], ref[2])
    finally:
        src.close()


@pytest.mark.gpu
def test_staged_packed_batch_is_refused(pkg):
    abi = pkg.abi
    cfg = cfg_of(pkg, RATING, flags=2, modes=1, capacity=10_000)
    with pkg.Engine(cfg) as e:
        e.enqueue(np.arange(100, dtype=np.uint64), np.arange(100, dtype=np.int32) * 40, np.zeros(100, np.uint8))
        h = np.arange(100, 110, dtype=np.uint32)
        k = np.zeros(10, np.uint16)
        assert e.lib.mm_enqueue_packed_begin(e.h, 10, h.ctypes.data_as(C.c_void_p), k.ctypes.data_as(C.c_void_p),
                                             None) == 0
        rules = rules_of(cfg, {(0, g): (0, 5000, 1, 0, 5000) for g in range(cfg.n_groups)})
        st = abi.WidenStats()
        rc = e.lib.mm_widen(e.h, 0, rules.ctypes.data_as(C.c_void_p), None, 0, None, 0, C.byref(st))
        assert rc == abi.MM_E_STATE and "staged" in e.lib.mm_last_error(e.h).decode()
        assert e.lib.mm_enqueue_packed_end(e.h, None, None) == 0
        assert e.widen(0, rules)[2].n_lobbies > 0


@pytest.mark.gpu
def test_no_side_effects_on_the_last_tick(pkg):
    cfg = gpu_config(pkg, RATING, "hashed", "split")
    src = Src(pkg, cfg, "hashed", seed=5, spread=2)
    try:
        src.eng.set_lobby_budget(per_queue=[3] * (cfg.n_modes * cfg.n_groups))
        src.enqueue(*src.fresh(40_000))
        src.eng.tick(src.now)
        q0, mq0, rep0 = src.eng.queue_stats(src.now), src.eng.match_quality(True), src.eng.lobby_budget_report()
        check_widen(src, rule_sets(cfg)[0])
        q1, mq1, rep1 = src.eng.queue_stats(src.now), src.eng.match_quality(True), src.eng.lobby_budget_report()
        for f in ("n_lobbies", "n_matched", "max_match_wait", "match_wait_hist"):
            assert np.array_equal(q0[f], q1[f]), f
        for x, y in zip(mq0, mq1):
            assert np.array_equal(x, y)
        for x, y in zip(rep0, rep1):
            assert np.array_equal(x, y)
    finally:
        src.close()


@pytest.mark.gpu
def test_config3_ten_million(pkg):
    from .test_tile_geometry import config3_pool
    n = 10_000_000
    cfg, _ = pkg.synth.workload_config("config3_10m_g32_5v5", RATING, n)
    ids, rating, mode, ts = config3_pool(pkg, n)
    with pkg.Engine(cfg) as e:
        assert e.enqueue(ids, rating, mode, ts).all()
        e.set_option("max_spread", 2)
        now = int(ts.max()) + 1
        e.set_lobby_budget(per_queue=[1000] * cfg.n_groups)  # the S1 tick leaves most of the pool queued
        e.tick(now)
        p = e.pool_read()
        wait = (now - p["enq_ts"].astype(np.int64))
        min_wait = int(np.quantile(wait, 0.97))  # a few percent of the pool are anchors
        rules = {(0, g): (min_wait, 3, 50, 5, 400) for g in range(cfg.n_groups)}
        lob, mem, st = e.widen(now, e.widen_rules(rules))
        assert st.n_anchors == (wait >= min_wait).sum() and st.n_lobbies > 0
        assert (lob["n_members"] == 10).all() and len(np.unique(mem)) == len(mem)
        assert e.in_queue(mem).all() and not np.isin(mem, e.pool_read()["id"]).any()
        assert (lob["group"][1:] >= lob["group"][:-1]).all()
        # the restatement on sampled queues: every queue's lobbies depend on that queue alone
        for g in (0, 13, 31):
            grp = np.searchsorted([cfg.group_lo[k] for k in range(cfg.n_groups)], p["rating"], side="right") - 1
            keep = grp == g
            want_lob, want_mem, _, _ = restate(cfg, p["id"][keep], p["rating"][keep], p["mode"][keep],
                                               p["enq_ts"][keep], now, {(0, g): rules[(0, g)]})
            h = lob[lob["group"] == g]
            got = np.concatenate([mem[x["first_member"]:x["first_member"] + x["n_members"]] for x in h] +
                                 [np.zeros(0, np.uint64)])
            assert len(h) == len(want_lob) and np.array_equal(got, want_mem)
