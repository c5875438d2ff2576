"""Lobby budget (mm_set_lobby_budget / mm_lobby_budget_report / mm_lobby_candidates, include/mm_engine.h).

The budget is flow control: a tick emits the FIRST a_q lobbies of every (mode, group) queue in its emission order and
keeps everyone else queued.  So the reference result of a budgeted tick is the oracle's unbudgeted result with every
queue's lobby list cut after a_q entries (`clip`), the allowances a_q coming from a pure-Python restatement of the
apportionment rule (`apportion_py`).  The serialized loops with a budget (a queue that has emitted a_q lobbies requeues
every further request) are restated here too and checked against that cut on the CPU.
"""
import ctypes as C
import importlib
import os
import socket
import threading

import numpy as np
import pytest

from .fakes import FakeBroker, OracleEngine

UNL = 0xFFFFFFFF


# ---- reference: apportionment, allowances, the cut -------------------------------------------------------------------
def apportion_py(budget, cand):
    """The rule of include/mm_engine.h with Python integers: no numpy, no fixed width."""
    cand = [int(c) for c in cand]
    total = sum(cand)
    if total <= budget:
        return cand
    a = [budget * c // total for c in cand]
    rem = [budget * c % total for c in cand]
    extra = budget - sum(a)
    for g in sorted(range(len(cand)), key=lambda g: (-rem[g], g))[:extra]:
        a[g] += 1
    return a


def allowances(cfg, cand, per_queue=None, per_mode=None):
    G = cfg.n_groups
    out = []
    for m in range(cfg.n_modes):
        c = [int(x) for x in cand[m * G:(m + 1) * G]]
        if per_queue is not None:
            c = [min(x, int(b)) for x, b in zip(c, per_queue[m * G:(m + 1) * G])]
        out += apportion_py(UNL if per_mode is None else int(per_mode[m]), c)
    return np.array(out, np.int64)


def unbudgeted(oracle, cfg, ids, rating, mode, W=-1):
    return oracle.run_windowed(cfg, W, ids, rating, mode) if W >= 0 else oracle.run_literal(cfg, ids, rating, mode)


def queue_counts(cfg, lobbies):
    return np.bincount(lobbies["mode"].astype(np.int64) * cfg.n_groups + lobbies["group"],
                       minlength=cfg.n_modes * cfg.n_groups)


def clip(cfg, ref, ids, allot):
    """The oracle's result with every queue's lobbies cut after allot[q]: -> dict(lob, mem, seq, resid, cand)."""
    lob = ref.lobbies
    q = lob["mode"].astype(np.int64) * cfg.n_groups + lob["group"]
    assert (np.diff(q) >= 0).all()  # canonical order: a queue's lobbies are contiguous, in emission order
    rank = np.arange(len(q)) - np.searchsorted(q, q, "left")
    keep = rank < np.asarray(allot)[q]
    L = lob["n_members"].astype(np.int64)
    out = lob[keep].copy()
    out["first_member"] = np.cumsum(L[keep]) - L[keep]
    mem = ref.member_ids[np.repeat(keep, L)]
    ids = np.asarray(ids, np.uint64)
    return dict(lob=out, mem=mem, seq=ref.emit_seq[keep], resid=ids[~np.isin(ids, mem)], cand=queue_counts(cfg, lob))


def reference(oracle, cfg, ids, rating, mode, W=-1, per_queue=None, per_mode=None):
    ref = unbudgeted(oracle, cfg, ids, rating, mode, W)
    cand = queue_counts(cfg, ref.lobbies)
    allot = allowances(cfg, cand, per_queue, per_mode)
    out = clip(cfg, ref, ids, allot)
    out["allot"] = allot
    return out


def group_of(cfg, r):
    for g in range(cfg.n_groups):
        if cfg.group_lo[g] <= r <= cfg.group_hi[g]:
            return g
    return cfg.default_group


def literal_budgeted(cfg, ids, rating, mode, allot, order, W=-1):
    """The serialized loop with per-queue allowances, in plain Python.  S0 (W < 0): one request at a time in feed
    order, the queue's partial lobby fills and is emitted; once the queue has emitted allot[q] lobbies every further
    request is requeued (it stays queued).  S1: the greedy windowed walk over the queue's rating-sorted players, which
    stops seeding when the allowance is used up.  -> (lobbies as (queue, [ids]) in (queue, emission) order, queued ids
    in enqueue order)."""
    n, G = len(ids), cfg.n_groups
    rmin = min(cfg.group_lo[g] for g in range(G)) - 1
    rmax = max(cfg.group_hi[g] for g in range(G)) + 1
    feed = list(range(n))
    if order == 1:
        feed.sort(key=lambda i: (int(mode[i]), min(max(int(rating[i]), rmin), rmax), i))
    queue = {i: int(mode[i]) * G + group_of(cfg, int(rating[i])) for i in range(n)}
    lobbies, matched = [], set()
    if W < 0:
        partial, emitted = {}, {}
        for i in feed:
            q = queue[i]
            if emitted.get(q, 0) >= allot[q]:
                continue  # requeued
            partial.setdefault(q, []).append(i)
            L = cfg.modes[q // G].teams * cfg.modes[q // G].team_size
            if len(partial[q]) == L:
                lobbies.append((q, partial.pop(q)))
                emitted[q] = emitted.get(q, 0) + 1
    else:
        for q in sorted(set(queue.values())):
            mine = [i for i in feed if queue[i] == q]
            L = cfg.modes[q // G].teams * cfg.modes[q // G].team_size
            k = done = 0
            while k + L <= len(mine) and done < allot[q]:
                if int(rating[mine[k + L - 1]]) - int(rating[mine[k]]) <= W:
                    lobbies.append((q, mine[k:k + L]))
                    k += L
                    done += 1
                else:
                    k += 1
    lobbies.sort(key=lambda t: t[0])  # stable: emission order inside a queue
    for _q, members in lobbies:
        matched.update(members)
    return ([(q, [int(ids[i]) for i in mem]) for q, mem in lobbies], [int(ids[i]) for i in range(n) if i not in matched])


def small_pool(pkg, seed, n, n_modes=2):
    rng = np.random.default_rng(seed)
    ids, rating, _, ts = pkg.synth.gen_pool(seed, n, bell=True)
    mode = rng.integers(0, n_modes, n).astype(np.uint8)
    return ids, rating, mode, ts


# ---- CPU -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order,W", [(0, -1), (1, -1), (1, 0), (1, 3), (1, 60)])
def test_budgeted_literal_loop_equals_the_cut(pkg, oracle, order, W):
    for seed in range(4):
        cfg = pkg.synth.make_config(n_groups=5, order=order, capacity=4096)
        ids, rating, mode, _ = small_pool(pkg, 100 + seed, 700)
        rng = np.random.default_rng(seed)
        pq = rng.integers(0, 12, cfg.n_modes * cfg.n_groups)
        pq[rng.integers(0, len(pq), 2)] = UNL
        pm = [int(rng.integers(0, 40)), UNL if seed % 2 else 25]
        want = reference(oracle, cfg, ids, rating, mode, W, pq, pm)
        lobs, queued = literal_budgeted(cfg, ids, rating, mode, want["allot"], order, W)
        assert [q for q, _ in lobs] == (want["lob"]["mode"].astype(int) * cfg.n_groups + want["lob"]["group"]).tolist()
        assert [x for _, mem in lobs for x in mem] == want["mem"].tolist()
        assert queued == want["resid"].tolist()
        assert (want["allot"] <= want["cand"]).all()


def test_apportion_properties(pkg):
    shard = importlib.import_module("microservice-matchmaking_b200.shard")
    rng = np.random.default_rng(1)
    for trial in range(300):
        G = int(rng.integers(1, 65))
        cand = rng.integers(0, [3, 50, 10 ** 6, 2 ** 31 // 64][trial % 4], G)
        total = int(cand.sum())
        budget = int(rng.integers(0, total + 2))
        a = shard.apportion(budget, cand)
        assert a.tolist() == apportion_py(budget, cand)
        assert (a <= cand).all() and (a >= 0).all() and int(a.sum()) == min(budget, total)
        if budget < total:  # within one lobby of the exact share (largest remainder is not monotone per queue in B)
            assert all(abs(int(x) * total - budget * int(c)) < total for x, c in zip(a, cand))
    assert shard.apportion(1, [5, 5, 5]).tolist() == [1, 0, 0]  # ties go to the lower group
    assert shard.apportion(2, [5, 5, 5]).tolist() == [1, 1, 0]
    assert shard.apportion(4, [1, 0, 7]).tolist() == [1, 0, 3]  # remainders 4 and 4: the lower group gets the extra
    big = [2 ** 31 - 5, 2 ** 31 - 9]  # products beyond 2^62
    assert shard.apportion(2 ** 32 - 20, big).tolist() == apportion_py(2 ** 32 - 20, big)
    assert shard.apportion(UNL, [3, 4]).tolist() == [3, 4]


class BudgetOracleEngine(OracleEngine):
    """OracleEngine with the lobby-budget calls, by the cut."""

    def __init__(self, cfg):
        super().__init__(cfg)
        self.pq = self.pm = None
        self.report = (np.zeros(cfg.n_modes * cfg.n_groups, np.int64),) * 2
        self.budget_calls = []

    def set_lobby_budget(self, per_queue=None, per_mode=None):
        self.pq, self.pm = per_queue, per_mode
        self.budget_calls.append((None if per_queue is None else np.array(per_queue).tolist(),
                                  None if per_mode is None else np.array(per_mode).tolist()))

    def lobby_candidates(self):
        keep = self.alive.astype(bool)
        return queue_counts(self.cfg, unbudgeted(self.oracle, self.cfg, *[a[keep] for a in self.q], self.max_spread).lobbies)

    def lobby_budget_report(self):
        return self.report

    def tick(self, now=0):
        keep = self.alive.astype(bool)
        ids = self.q[0][keep]
        r = reference(self.oracle, self.cfg, ids, self.q[1][keep], self.q[2][keep], self.max_spread, self.pq, self.pm)
        stay = np.isin(self.q[0], r["resid"])
        self.q = [a[stay] for a in self.q]
        self.alive = np.ones(len(self.q[0]), np.uint8)
        self.report = (r["cand"], r["allot"])
        st = self.abi.TickStats()
        st.n_lobbies, st.n_matched, st.n_residual = len(r["lob"]), len(r["mem"]), len(r["resid"])
        return r["lob"], r["mem"], r["seq"], st


def test_search_pool_budget_pause_and_status(pkg, oracle):
    import json
    sw = importlib.import_module("microservice-matchmaking_b200.search_worker")
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=0, capacity=4096)
    names = list(pkg.synth.REFERENCE_GROUP_NAMES)
    eng = BudgetOracleEngine(cfg)
    slots = {"1v1": 3}
    asked = []

    def free_slots():
        asked.append(dict(slots))
        return dict(slots)

    broker = FakeBroker()
    pool = sw.SearchPool(eng, ["1v1", "5v5"], names, lobby_budget=free_slots)
    workers = {g: sw.SearchWorker.start_link(broker, pool, {"group_name": g})[1] for g in names}
    for i in range(40):  # 20 bronze and 20 gold 1v1 players: 10 candidate lobbies each
        g, r = ("bronze", 100) if i % 2 == 0 else ("gold", 2100)
        broker.publish(sw.generate_exchange_name(g), sw.generate_queue_name(g),
                       json.dumps({"id": f"p{i}", "rating": r, "game-mode": "1v1"}))
    broker.deliver_all()
    assert pool.tick() == 3 and len(asked) == 1
    assert eng.budget_calls[-1][1] == [3, UNL]
    # 10 : 10 candidates under a budget of 3: bronze 2 (tie to the lower group), gold 1
    assert workers["bronze"].status()[1]["held_back"] == {"1v1": 8, "5v5": 0}
    assert workers["gold"].status()[1]["held_back"] == {"1v1": 9, "5v5": 0}
    pool.pause(["bronze"])
    slots["1v1"] = 100
    assert pool.tick() == 9 and len(asked) == 2  # gold's nine; bronze is paused
    assert eng.budget_calls[-1][0][names.index("bronze")] == 0 and eng.budget_calls[-1][0][len(names)] == 0
    assert workers["bronze"].status()[1]["held_back"]["1v1"] == 8
    pool.resume_queues(["bronze"], ["1v1"])
    assert pool.paused == {len(names) + names.index("bronze")}  # the 5v5 queue of bronze is still paused
    assert pool.tick() == 8 and pool.engine.pool_size() == 0
    plain = sw.SearchPool(BudgetOracleEngine(cfg), ["1v1", "5v5"], names)
    plain.pause(["gold"], ["5v5"])  # without a callable the pause is set at once
    assert plain.engine.budget_calls[-1][1] is None
    assert plain.engine.budget_calls[-1][0].count(0) == 1


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _gloo_worker(rank, world, port, n, per_mode, out_q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    pkg = importlib.import_module("microservice-matchmaking_b200")
    shard = importlib.import_module("microservice-matchmaking_b200.shard")
    cfg = pkg.synth.make_config(n_groups=8, order=1, capacity=n)
    ids, rating, mode, _ = small_pool(pkg, 5, n)
    mine = shard.route(cfg, rating, world) == rank
    eng = BudgetOracleEngine(cfg)
    eng.enqueue(ids[mine], rating[mine], mode[mine])
    shard.set_mode_budget(eng, per_mode, comm=shard.DistComm(), rank=rank, world=world)
    lob, mem, seq, _st = eng.tick()
    gathered = [None] * world
    dist.all_gather_object(gathered, (lob, mem, seq, eng.pool_read()["id"]))
    if rank == 0:
        mlob, mmem, _ = shard.merge_results(cfg, [(g[0], g[1], g[2]) for g in gathered])
        out_q.put((mlob, mmem, np.concatenate([g[3] for g in gathered])))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
def test_set_mode_budget_over_gloo(pkg, oracle, world):
    import torch.multiprocessing as mp
    n, per_mode = 6000, [37, 11]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, port, n, per_mode, q)) for r in range(world)]
    for p in procs:
        p.start()
    mlob, mmem, mres = q.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    cfg = pkg.synth.make_config(n_groups=8, order=1, capacity=n)
    ids, rating, mode, _ = small_pool(pkg, 5, n)
    want = reference(oracle, cfg, ids, rating, mode, per_mode=per_mode)
    assert len(want["lob"]) == 48 and (want["allot"] < want["cand"]).any()
    assert np.array_equal(mlob, want["lob"]) and np.array_equal(mmem, want["mem"])
    assert np.array_equal(np.sort(mres), np.sort(want["resid"]))


# ---- GPU -------------------------------------------------------------------------------------------------------------
gpu = pytest.mark.gpu


def make_engine(pkg, cfg, opts=None, W=-1):
    eng = pkg.Engine(cfg)
    for k, v in (opts or {}).items():
        eng.set_option(k, v)
    if W >= 0:
        eng.set_option("max_spread", W)
    return eng


def check_tick(eng, want, now=0, emit_seq=True):
    lob, mem, seq, st = eng.tick(now)
    assert np.array_equal(lob, want["lob"])
    assert np.array_equal(mem, want["mem"])
    if emit_seq:
        assert np.array_equal(seq, want["seq"])
    assert (st.n_lobbies, st.n_matched, st.n_residual) == (len(want["lob"]), len(want["mem"]), len(want["resid"]))
    assert np.array_equal(eng.pool_read()["id"], want["resid"])
    cand, emitted = eng.lobby_budget_report()
    assert np.array_equal(cand, want["cand"]) and np.array_equal(emitted, want["allot"])
    return lob, mem, seq, st


def budgets_for(kind, cfg, cand, rng):
    nq = cfg.n_modes * cfg.n_groups
    G = cfg.n_groups
    pq = pm = None
    if kind in ("queue", "both"):
        pq = np.full(nq, UNL, np.int64)
        some = rng.permutation(nq)[:max(2, nq // 2)]  # binds in some queues only
        pq[some] = [int(rng.integers(0, int(cand[q]) + 2)) for q in some]
        pq[some[0]] = 0
        pq[some[1]] = cand[some[1]]  # lands exactly on c_q
    if kind in ("mode", "both"):
        per = cand.reshape(cfg.n_modes, G).sum(axis=1)
        pm = [int(per[0] * 0.37), UNL] + [int(per[m] // 3) for m in range(2, cfg.n_modes)]
        pm = pm[:cfg.n_modes]
    if kind == "mode0":
        pm = [UNL] * cfg.n_modes
        pm[-1] = 0
    if kind == "zero":
        pq, pm = np.zeros(nq, np.int64), None
    return pq, pm


CASES = [  # order, W, flags, engine options
    (0, -1, 0, {}), (1, -1, 0, {}), (1, 0, 0, {}), (1, 3, 0, {}), (1, 40, 0, {}),
    (1, -1, 4, {}), (1, 5, 4, {}),                       # MM_F_WIDE_PARTITIONS: list-ranked wide groups
    (0, -1, 0, {"tick_impl": 0}), (1, 7, 0, {"tick_impl": 0}), (1, -1, 0, {"rank_impl": 2}), (1, 7, 4, {"rank_impl": 2}),
]


@gpu
@pytest.mark.parametrize("kind", ["queue", "mode", "both", "mode0", "zero"])
@pytest.mark.parametrize("order,W,flags,opts", CASES)
def test_budgeted_tick_equals_oracle(pkg, oracle, order, W, flags, opts, kind):
    n = 60_000
    cfg = pkg.synth.make_config(n_groups=6, order=order, capacity=n, flags=flags)  # groups 834 ratings wide
    ids, rating, mode, ts = small_pool(pkg, 11, n)
    rng = np.random.default_rng(len(kind) + order + W)
    cand = queue_counts(cfg, unbudgeted(oracle, cfg, ids, rating, mode, W).lobbies)
    pq, pm = budgets_for(kind, cfg, cand, rng)
    want = reference(oracle, cfg, ids, rating, mode, W, pq, pm)
    assert (want["allot"] < want["cand"]).any()
    with make_engine(pkg, cfg, opts, W) as eng:
        assert eng.enqueue(ids, rating, mode, ts).all()
        assert np.array_equal(eng.lobby_candidates(), cand)
        eng.set_lobby_budget(pq, pm)
        check_tick(eng, want)
        qs = eng.queue_stats(0)
        assert np.array_equal(qs["n_lobbies"], want["allot"])
        # the held players are ordinary queued players: the next tick without a budget matches them
        eng.set_lobby_budget()
        keep = np.isin(ids, want["resid"])
        check_tick(eng, reference(oracle, cfg, ids[keep], rating[keep], mode[keep], W), emit_seq=False)


@gpu
@pytest.mark.parametrize("order,W", [(0, -1), (1, -1), (1, 4)])
def test_unlimited_budget_is_no_budget(pkg, oracle, order, W):
    n = 50_000
    cfg = pkg.synth.make_config(n_groups=8, order=order, capacity=n)
    ids, rating, mode, ts = small_pool(pkg, 3, n)
    out = []
    for explicit in (False, True):
        with make_engine(pkg, cfg, W=W) as eng:
            if explicit:
                eng.set_lobby_budget(np.full(cfg.n_modes * cfg.n_groups, UNL), [UNL] * cfg.n_modes)
            res = []
            for step in range(3):
                sl = slice(step * n // 3, (step + 1) * n // 3)
                eng.enqueue(ids[sl], rating[sl], mode[sl], ts[sl])
                eng.remove(ids[sl][::17])
                lob, mem, seq, st = eng.tick(1000 * step)
                res.append((lob, mem, seq, (st.n_lobbies, st.n_matched, st.n_residual, st.n_dead), eng.pool_read()["id"],
                            eng.queue_stats(1000 * step).tobytes(), eng.lobby_budget_report()))
            out.append(res)
    for a, b in zip(*out):
        for x, y in zip(a[:3], b[:3]):
            assert np.array_equal(x, y)
        assert a[3] == b[3] and np.array_equal(a[4], b[4]) and a[5] == b[5]
        assert np.array_equal(a[6][0], b[6][0]) and np.array_equal(a[6][0], a[6][1])  # nothing held back


@gpu
@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_budget_at_chunk_edges_and_partition_boundaries(pkg, oracle, delta):
    """One queue of 2 048 k + delta players (pool chunks hold 2 048), budgets that leave exactly a chunk, one player
    more and one less queued; and a wide group (several partitions of <= 255 ratings) cut exactly where a partition
    ends."""
    n = 2048 * 3 + delta
    cfg = pkg.synth.make_config(groups=[(0, 99), (100, 5000)], modes=(("1v1", 2, 1),), order=1, capacity=3 * n)
    rng = np.random.default_rng(7)
    rating = np.concatenate([rng.integers(0, 100, n), np.sort(rng.integers(100, 5001, n))]).astype(np.int32)
    ids = np.arange(1, 2 * n + 1, dtype=np.uint64)
    mode = np.zeros(2 * n, np.uint8)
    # wide group: ratings 100..4 999 split into partitions; cut after the players of the first partitions
    lo_part = int((rating[n:] < 100 + 245).sum())  # 4 901 keys in 20 partitions of 246 keys
    for a0, a1 in [((n - 2048) // 2, lo_part // 2), ((n - 2048) // 2 + 1, lo_part // 2 + 1), (n // 2, 0), (1, n // 2)]:
        want = reference(oracle, cfg, ids, rating, mode, per_queue=[a0, a1])
        with make_engine(pkg, cfg) as eng:
            assert eng.enqueue(ids, rating, mode).all()
            eng.set_lobby_budget(per_queue=[a0, a1])
            check_tick(eng, want)


@gpu
def test_dense_handles_and_packed_tick(pkg, oracle):
    n = 40_000
    cfg = pkg.synth.make_config(n_groups=8, order=1, capacity=n, active_capacity=n, flags=2)  # MM_F_DENSE_IDS
    _ids, rating, mode, ts = small_pool(pkg, 21, n)
    handles = np.random.default_rng(2).permutation(n).astype(np.uint32)
    want = reference(oracle, cfg, handles.astype(np.uint64), rating, mode, per_mode=[500, 77])
    with make_engine(pkg, cfg) as eng:
        assert eng.enqueue_packed(handles, pkg.Engine.pack_key(rating, mode), ts).all()
        eng.set_lobby_budget(per_mode=[500, 77])
        lob, mem, seq, st = eng.tick_packed()
        assert np.array_equal(lob, want["lob"]) and np.array_equal(mem, want["mem"].astype(np.uint32))
        assert np.array_equal(seq, want["seq"]) and st.n_lobbies == 577
        assert np.array_equal(eng.pool_read()["id"], want["resid"])


@gpu
@pytest.mark.parametrize("order,W", [(0, -1), (1, -1), (1, 6)])
def test_budget_equals_tick_and_requeue_of_the_surplus(pkg, oracle, order, W):
    """A twin ticks WITHOUT a budget and hands the members of every lobby beyond the first a_q of its queue back with
    mm_requeue: both engines then hold the same queue state and go on identically."""
    n = 30_000
    # room for the chunks a requeue leaves behind: until the next tick they count as slots in use (mm_requeue)
    cfg = pkg.synth.make_config(n_groups=6, order=order, capacity=4 * n)
    ids, rating, mode, ts = small_pool(pkg, 31, n)
    more = small_pool(pkg, 32, 5000)
    pm = [700, 90]
    pq = np.full(12, UNL, np.int64)
    pq[[1, 8]] = [3, 0]
    with make_engine(pkg, cfg, W=W) as a, make_engine(pkg, cfg, W=W) as b:
        for e in (a, b):
            assert e.enqueue(ids, rating, mode, ts).all()
        a.set_lobby_budget(pq, pm)
        la, ma, sa, _ = a.tick(50)
        lb, mb, sb, _ = b.tick(50)
        cand, emitted = a.lobby_budget_report()
        assert np.array_equal(cand, queue_counts(cfg, lb)) and (emitted < cand).any()
        q = lb["mode"].astype(np.int64) * cfg.n_groups + lb["group"]
        surplus = np.arange(len(q)) - np.searchsorted(q, q, "left") >= emitted[q]
        back = mb[np.repeat(surplus, lb["n_members"].astype(np.int64))]
        assert np.array_equal(ma, mb[np.repeat(~surplus, lb["n_members"].astype(np.int64))])
        assert np.array_equal(sa, sb[~surplus])
        idx = np.searchsorted(np.sort(ids), back)
        src = np.argsort(ids)[idx]  # seq of a player = its index in the one enqueue batch
        codes = b.requeue(back, rating[src], mode[src], ts[src], src.astype(np.uint32))
        assert (codes == 1).all()
        a.set_lobby_budget()
        pa, pb = a.pool_read(), b.pool_read()
        for k in ("id", "rating", "mode", "enq_ts"):
            assert np.array_equal(pa[k], pb[k])
        assert np.array_equal(a.in_queue(ids), b.in_queue(ids))
        wa, wb = a.queue_stats(60), b.queue_stats(60)
        for k in ("n_waiting", "max_wait", "wait_hist"):
            assert np.array_equal(wa[k], wb[k])
        for step in range(2):
            for e in (a, b):
                if step == 0:
                    assert e.enqueue(*more[:3], more[3]).all()
            ra, rb = a.tick(100 + step), b.tick(100 + step)
            for x, y in zip(ra[:3], rb[:3]):
                assert np.array_equal(x, y)
            assert (ra[3].n_lobbies, ra[3].n_matched, ra[3].n_residual) == (rb[3].n_lobbies, rb[3].n_matched, rb[3].n_residual)


@gpu
@pytest.mark.parametrize("order,W", [(0, -1), (1, 5)])
def test_long_schedule_with_changing_budgets(pkg, oracle, order, W):
    cfg = pkg.synth.make_config(n_groups=5, order=order, capacity=60_000)
    rng = np.random.default_rng(order + 40)
    q_ids, q_rating, q_mode, q_ts = (np.zeros(0, t) for t in (np.uint64, np.int32, np.uint8, np.uint32))
    nq = cfg.n_modes * cfg.n_groups
    with make_engine(pkg, cfg, W=W) as eng:
        for step in range(14):
            now = 100 * step
            ids, rating, mode, _ = small_pool(pkg, 500 + step, int(rng.integers(500, 4000)))
            ts = np.full(len(ids), now, np.uint32)
            assert eng.enqueue(ids, rating, mode, ts).all()
            q_ids, q_rating, q_mode, q_ts = (np.concatenate(p) for p in
                                             ((q_ids, ids), (q_rating, rating), (q_mode, mode), (q_ts, ts)))
            gone = q_ids[rng.random(len(q_ids)) < 0.03]
            eng.remove(gone)
            if step % 4 == 3:
                expired, _ = eng.expire(now, 250)
                assert np.array_equal(np.sort(expired), np.sort(q_ids[(now - q_ts.astype(np.int64) >= 250) & ~np.isin(q_ids, gone)]))
                gone = np.concatenate([gone, expired])
            keep = ~np.isin(q_ids, gone)
            q_ids, q_rating, q_mode, q_ts = q_ids[keep], q_rating[keep], q_mode[keep], q_ts[keep]
            cand = queue_counts(cfg, unbudgeted(oracle, cfg, q_ids, q_rating, q_mode, W).lobbies)
            pq, pm = budgets_for(["queue", "mode", "both", "zero", "none"][step % 5], cfg, cand, rng)
            eng.set_lobby_budget(pq, pm)
            want = reference(oracle, cfg, q_ids, q_rating, q_mode, W, pq, pm)
            check_tick(eng, want, now, emit_seq=False)
            keep = np.isin(q_ids, want["resid"])
            q_ids, q_rating, q_mode, q_ts = q_ids[keep], q_rating[keep], q_mode[keep], q_ts[keep]


@gpu
def test_held_players_keep_their_stamps(pkg, oracle):
    cfg = pkg.synth.make_config(n_groups=4, order=0, capacity=10_000)
    ids, rating, mode, _ = small_pool(pkg, 9, 8000)
    with make_engine(pkg, cfg) as eng:
        eng.enqueue(ids, rating, mode, np.full(len(ids), 10, np.uint32))
        eng.set_lobby_budget(per_mode=[0, 0])
        _, _, _, st = eng.tick(100)
        assert (st.n_lobbies, st.n_residual) == (0, 8000)
        assert eng.queue_stats(100)["n_matched"].sum() == 0
        eng.set_lobby_budget()
        _, _, _, st = eng.tick(500)
        qs = eng.queue_stats(500)
        assert st.n_matched > 7900 and (qs["max_match_wait"][qs["n_matched"] > 0] == 490).all()


@gpu
@pytest.mark.parametrize("W", [-1, 4])
def test_lobby_candidates_is_a_dry_run(pkg, oracle, W):
    n = 40_000
    cfg = pkg.synth.make_config(n_groups=8, order=1, capacity=2 * n)
    ids, rating, mode, ts = small_pool(pkg, 13, n)
    more = small_pool(pkg, 14, 9000)
    with make_engine(pkg, cfg, W=W) as eng:
        assert (eng.lobby_candidates() == 0).all() and (np.concatenate(eng.lobby_budget_report()) == 0).all()
        eng.enqueue(ids, rating, mode, ts)
        eng.set_lobby_budget(per_mode=[100, 100])
        eng.tick(7)
        eng.enqueue(*more[:3], more[3])
        eng.remove(ids[::5])
        def image():  # the active section of an image is unordered: compared sorted
            h, cols = read_image(eng.export_state())
            return bytes(h), [np.sort(c) if k == "active" else c for k, c in cols.items()]

        read_image = importlib.import_module("microservice-matchmaking_b200.engine").read_image
        before = (eng.queue_stats(9).tobytes(), image(), eng.lobby_budget_report())
        cand = eng.lobby_candidates()  # budgets ignored
        after = (eng.queue_stats(9).tobytes(), image(), eng.lobby_budget_report())
        assert before[0] == after[0] and before[1][0] == after[1][0]
        assert all(np.array_equal(x, y) for x, y in zip(before[1][1], after[1][1]))
        assert all(np.array_equal(x, y) for x, y in zip(before[2], after[2]))
        eng.set_lobby_budget()
        lob, _, _, _ = eng.tick(10)
        assert np.array_equal(cand, queue_counts(cfg, lob)) and cand.sum() > 1000


@gpu
@pytest.mark.parametrize("K,W", [(2, -1), (4, -1), (4, 5)])
def test_sharded_engines_under_one_mode_budget(pkg, oracle, K, W):
    shard = importlib.import_module("microservice-matchmaking_b200.shard")
    n = 40_000
    cfg = pkg.synth.make_config(n_groups=8, order=1, capacity=n)
    ids, rating, mode, ts = small_pool(pkg, 17, n)
    per_mode = [1234, 321]
    owner = shard.route(cfg, rating, K)
    engines = [make_engine(pkg, cfg, W=W) for _ in range(K)]
    try:
        for r, e in enumerate(engines):
            e.enqueue(ids[owner == r], rating[owner == r], mode[owner == r], ts[owner == r])
        # one thread per rank over the in-process exchange, as the ranks of a job would call it
        comm = shard.LocalComm()
        threads = [threading.Thread(target=shard.set_mode_budget, args=(e, per_mode, comm, r, K))
                   for r, e in enumerate(engines)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        res = [e.tick() for e in engines]
        mlob, mmem, _ = shard.merge_results(cfg, [r[:3] for r in res])
        with make_engine(pkg, cfg, W=W) as single:
            single.enqueue(ids, rating, mode, ts)
            single.set_lobby_budget(per_mode=per_mode)
            lob, mem, _, st = single.tick()
            assert st.n_lobbies == sum(per_mode)
            assert np.array_equal(mlob, lob) and np.array_equal(mmem, mem)
            assert np.array_equal(np.sort(np.concatenate([e.pool_read()["id"] for e in engines])),
                                  np.sort(single.pool_read()["id"]))
            # all engines in one process, no exchange: the budgets the single engine's candidates give
            assert np.array_equal(shard.set_mode_budget(engines, per_mode),
                                  shard.queue_budgets(cfg, per_mode, single.lobby_candidates()))
    finally:
        for e in engines:
            e.close()


@gpu
def test_config3_size_budget_and_pause_everything(pkg, oracle):
    """10 M players, 32 groups, 5v5, rating order: a binding mode budget, then budget 0 (every player a leftover of its
    row), then the unbudgeted tick of the untouched pool."""
    n = 10_000_000
    cfg, m = pkg.synth.workload_config("config3_10m_g32_5v5", 1, n)
    ids, rating, _, ts = pkg.synth.gen_pool(42, n, bell=True)
    mode = np.full(n, m, np.uint8)
    lm, lg, members, resid = oracle.closed_form_numpy(cfg, ids, rating, mode)
    cand = np.bincount(lg, minlength=32)
    B = int(cand.sum()) // 2
    allot = np.array(apportion_py(B, cand))
    with pkg.Engine(cfg) as eng:
        assert eng.enqueue(ids, rating, mode, ts).all()
        eng.snapshot()
        assert np.array_equal(eng.lobby_candidates(), cand)
        eng.set_lobby_budget(per_mode=[B])
        lob, mem, _, st = eng.tick()
        assert (st.n_lobbies, st.n_matched, st.n_residual) == (B, 10 * B, n - 10 * B)
        assert np.array_equal(np.bincount(lob["group"], minlength=32), allot)
        first = np.cumsum(cand) - cand  # the queue's first a_q lobbies of the closed form, members in order
        want = np.concatenate([members[10 * first[g]:10 * (first[g] + allot[g])] for g in range(32)])
        assert np.array_equal(mem, want)
        left = eng.pool_read()["id"]
        assert np.array_equal(left, ids[~np.isin(ids, mem)])  # the survivors, in enqueue order
        eng.restore()
        eng.set_lobby_budget(per_mode=[0])
        _, _, _, st = eng.tick()
        assert (st.n_lobbies, st.n_matched, st.n_residual) == (0, 0, n)
        assert np.array_equal(eng.lobby_budget_report()[0], cand)
        assert np.array_equal(eng.pool_read()["id"], ids)
        eng.set_lobby_budget()
        lob, mem, _, st = eng.tick()
        assert np.array_equal(mem, members) and np.array_equal(lob["group"], lg)
        assert np.array_equal(eng.pool_read()["id"], resid)


@gpu
def test_refusals_and_messages(pkg):
    abi = pkg.abi
    cfg = pkg.synth.make_config(n_groups=4, order=1, capacity=1000, active_capacity=1000, flags=2)
    with pkg.Engine(cfg) as eng:
        lib, h = eng.lib, eng.h
        buf, buf2, k = np.zeros(8, np.uint32), np.zeros(8, np.uint32), C.c_uint32(0)
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        assert lib.mm_lobby_candidates(h, p(buf), 7, C.byref(k)) == abi.MM_E_CAP
        assert (lib.mm_last_error(h).decode(), k.value) == ("need cap >= 8", 8)
        assert lib.mm_lobby_budget_report(h, p(buf), p(buf2), 3, C.byref(k)) == abi.MM_E_CAP
        assert (lib.mm_last_error(h).decode(), k.value) == ("need cap >= 8", 8)
        assert lib.mm_lobby_candidates(h, None, 8, C.byref(k)) == abi.MM_E_ARG
        assert lib.mm_set_lobby_budget(None, None, None) == abi.MM_E_ARG
        eng.enqueue_packed_begin(np.arange(10, dtype=np.uint32), np.full(10, 100, np.uint16))
        for rc in (lib.mm_lobby_candidates(h, p(buf), 8, C.byref(k)), lib.mm_lobby_budget_report(h, p(buf), p(buf2), 8, C.byref(k))):
            assert rc == abi.MM_E_STATE
            assert lib.mm_last_error(h).decode() == "a packed batch is staged: call mm_enqueue_packed_end first"
        eng.set_lobby_budget(per_mode=[1, 1])  # setting a budget needs no device work: allowed with a staged batch
        eng.enqueue_packed_end()
        _, _, _, st = eng.tick_packed()
        assert st.n_lobbies == 1 + 0  # ten 1v1 players of one rating: five candidate lobbies, one allowed
        assert eng.lobby_budget_report()[0].sum() == 5
