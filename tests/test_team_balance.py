"""Balanced teams (mm_set_option("team_balance"), SearchPool(balance_teams=...)): every lobby of a masked two-team mode
is split into the two teams with the least rating difference.

Two independent restatements of the rule (include/mm_engine.h): `split_plain` enumerates the team-1 sets with
itertools, `split_numpy` scores every lobby against a precomputed table of all masks at once.
CPU: the known answers, the two restatements agree (every S <= 8, ties, equal ratings), the balanced imbalance is
never above the unbalanced one, SearchPool's mask.
GPU: twin engines run the same schedule with and without the mask — headers, emit_seq, pool_read, in_queue,
queue_stats and the next tick are identical, each lobby holds the same players, and the masked engine's member order
is the restatement applied to the unmasked one's; mm_widen; mm_match_quality; mm_locate; the refusals; config3 at 10 M
players in both orders.
"""
import importlib
import itertools

import numpy as np
import pytest

from .fakes import OracleEngine

sw = importlib.import_module("microservice-matchmaking_b200.search_worker")
eng_mod = importlib.import_module("microservice-matchmaking_b200.engine")
abi = importlib.import_module("microservice-matchmaking_b200.abi")

RATING, ARRIVAL = 1, 0
DENSE, WIDE = 2, 4


# ================================================================================ restatements
def split_plain(c, S):
    """c: the L = 2S values in today's member order -> (new member order as old indices, imbalance)."""
    L = len(c)
    c = [int(x) for x in c]
    total = sum(c)
    best = None
    for rest in itertools.combinations(range(1, L), S - 1):
        a = (0,) + rest
        d = abs(2 * sum(c[i] for i in a) - total)
        m = sum(1 << i for i in rest)
        if best is None or (d, m) < best[:2]:
            best = (d, m, a)
    d, _m, a = best
    return list(a) + [i for i in range(L) if i not in a], d


_TABLES = {}


def mask_table(S):
    """-> bool[n, 2S]: every team-1 set holding member 0, in ascending mask order."""
    if S not in _TABLES:
        L = 2 * S
        rows = [m | 1 for m in range(0, 1 << L, 2) if bin(m).count("1") == S - 1]
        _TABLES[S] = (np.array(rows, np.int64)[:, None] >> np.arange(L)) & 1 == 1
    return _TABLES[S]


def split_numpy(c, S):
    """c: int[n, 2S] -> (perm int[n, 2S] of old indices, imbalance int64[n]), vectorised over lobbies."""
    c = np.asarray(c, np.int64)
    t = mask_table(S)
    d = np.abs(2 * (c @ t.T.astype(np.int64)) - c.sum(1, keepdims=True))
    k = d.argmin(1)  # the first minimum = the smallest mask (the table is in ascending mask order)
    inA = t[k]
    idx = np.broadcast_to(np.arange(2 * S), c.shape)
    perm = np.concatenate([idx[inA].reshape(len(c), S), idx[~inA].reshape(len(c), S)], 1)
    return perm, d[np.arange(len(c)), k]


def imbalance_of(c, S):
    c = np.asarray(c, np.int64)
    return np.abs(c[..., :S].sum(-1) - c[..., S:].sum(-1))


# ================================================================================ CPU
def test_known_answers():
    c = list(range(1, 11))
    perm, d = split_plain(c, 5)
    assert [c[i] for i in perm] == [1, 5, 6, 7, 8, 2, 3, 4, 9, 10] and d == 1
    assert imbalance_of(c, 5) == 25
    r = [1500, 1500, 1501, 1503, 1510, 1512, 1512, 1520, 1530, 1540]
    perm, d = split_plain(r, 5)
    assert [r[i] for i in perm] == [1500, 1510, 1512, 1512, 1530, 1500, 1501, 1503, 1520, 1540] and d == 0
    assert imbalance_of(r, 5) == 100
    assert split_plain([7, 7, 7, 7], 2) == ([0, 1, 2, 3], 0)
    for v, S in ((c, 5), (r, 5), ([7, 7, 7, 7], 2)):
        perm, d = split_numpy([v], S)
        assert (perm[0].tolist(), d[0]) == split_plain(v, S)


@pytest.mark.parametrize("S", range(1, 9))
def test_restatements_agree(S):
    rng = np.random.default_rng(S)
    L = 2 * S
    n = 300 if S <= 6 else 40
    lobbies = [rng.integers(0, 5000, (n, L)), rng.integers(0, 4, (n, L)),  # many ties
               np.full((5, L), 1234), np.sort(rng.integers(1400, 1600, (n, L)), 1)]
    for c in lobbies:
        perm, d = split_numpy(c, S)
        for i in range(len(c)):
            q, e = split_plain(c[i], S)
            assert perm[i].tolist() == q and d[i] == e
        assert np.array_equal(imbalance_of(np.take_along_axis(c, perm, 1), S), d)
        assert (d <= imbalance_of(c, S)).all()  # never worse than today's order


def test_rating_order_is_strictly_improved_when_ratings_are_distinct():
    rng = np.random.default_rng(7)
    for S in range(2, 9):
        c = np.array([np.sort(rng.choice(5000, 2 * S, replace=False)) for _ in range(100)])
        _p, d = split_numpy(c, S)
        assert (d < imbalance_of(c, S)).all()
    # with ties the rating-order split can already be the best one: 0 0 | 0 1 has no better split
    assert split_plain([0, 0, 0, 1], 2) == ([0, 1, 2, 3], 1)


class OptionEngine(OracleEngine):
    def __init__(self, cfg):
        super().__init__(cfg)
        self.options = {}

    def set_option(self, name, value):
        self.options[name] = value


def test_search_pool_sets_the_mask(pkg):
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=(("1v1", 2, 1), ("5v5", 2, 5), ("3v3", 2, 3)),
                                order=ARRIVAL, capacity=1000)
    names = pkg.synth.REFERENCE_GROUP_NAMES
    eng = OptionEngine(cfg)
    sw.SearchPool(eng, ["1v1", "5v5", "3v3"], names, balance_teams=["5v5", "3v3"])
    assert eng.options == {"team_balance": 0b110}
    eng = OptionEngine(cfg)
    sw.SearchPool(eng, ["1v1", "5v5", "3v3"], names)
    assert "team_balance" not in eng.options  # only set when asked for
    with pytest.raises(ValueError):
        sw.SearchPool(OptionEngine(cfg), ["1v1", "5v5", "3v3"], names, balance_teams=["7v7"])


# ================================================================================ GPU
MODES = (("1v1", 2, 1), ("5v5", 2, 5), ("4v4", 2, 4), ("coop4", 1, 4), ("8v8", 2, 8))
MASK = 0b10111  # 1v1 (accepted, no change), 5v5, 4v4, 8v8; coop4 (one team) cannot be masked


def gpu_config(pkg, order, layout="split", flags=0, modes=MODES, capacity=200_000):
    groups = {"split": pkg.synth.REFERENCE_GROUPS, "wide": pkg.synth.REFERENCE_GROUPS,
              "overlap": [(0, 2000), (1000, 3000), (2500, 5000), (100, 200)]}[layout]
    if layout == "wide":
        flags |= WIDE
    return pkg.synth.make_config(groups=groups, modes=modes, order=order, capacity=capacity,
                                 active_capacity=2 * capacity, default_group=1 if layout == "overlap" else -1,
                                 flags=flags)


def clamp_bounds(cfg):
    return (min(cfg.group_lo[g] for g in range(cfg.n_groups)) - 1, max(cfg.group_hi[g] for g in range(cfg.n_groups)) + 1)


class Book:
    """id -> rating of every player the test enqueued."""

    def __init__(self):
        self.d = {}

    def add(self, ids, r):
        for i, x in zip(ids.tolist(), r.tolist()):
            self.d.setdefault(i, x)

    def c(self, cfg, ids):
        lo, hi = clamp_bounds(cfg)
        return np.clip(np.array([self.d[i] for i in np.asarray(ids).tolist()], np.int64), lo, hi)


def expect_balanced(cfg, mask, lob, mem, book):
    """The restatement applied to unbalanced results -> the member array the masked engine must emit."""
    want = np.array(mem, copy=True)
    for m in range(cfg.n_modes):
        S = cfg.modes[m].team_size
        sel = np.flatnonzero(lob["mode"] == m)
        if not (mask >> m) & 1 or S < 2 or not len(sel):
            continue
        L = 2 * S
        idx = lob["first_member"][sel].astype(np.int64)[:, None] + np.arange(L)
        ids = np.asarray(mem)[idx]
        perm, _d = split_numpy(book.c(cfg, ids.ravel()).reshape(ids.shape), S)
        want[idx] = np.take_along_axis(ids, perm, 1)
    return want


def teams_imbalance(cfg, lob, mem, book):
    out = np.zeros(len(lob), np.int64)
    for h in range(len(lob)):
        m = int(lob["mode"][h])
        T, S = cfg.modes[m].teams, cfg.modes[m].team_size
        f = int(lob["first_member"][h])
        t = book.c(cfg, mem[f:f + T * S]).reshape(T, S).sum(1)
        out[h] = t.max() - t.min()
    return out


def fresh(pkg, rng, base, n, n_modes, dense, lo=-300, hi=5300):
    x = np.arange(base, base + n, dtype=np.uint64)
    ids = x if dense else pkg.synth.mix64(x + np.uint64(5 << 40))
    return ids, rng.integers(lo, hi, n).astype(np.int32), rng.integers(0, n_modes, n).astype(np.uint8), \
        (1000 - rng.integers(0, 60, n)).astype(np.uint32)


def tick(pkg, eng, form, now):
    from .test_tick_forms_and_schedules import tick_form
    return tick_form(pkg, eng, "tick" if form == "async" else ("packed" if form == "async_packed" else form), now)


def same_state(a, b, ids, now):
    pa, pb = a.pool_read(), b.pool_read()
    for k in pa:
        assert np.array_equal(pa[k], pb[k]), k
    assert np.array_equal(a.in_queue(ids), b.in_queue(ids))
    assert np.array_equal(a.queue_stats(now), b.queue_stats(now))


def run_twins(pkg, cfg, seed, mask=MASK, spread=-1, budget=(None, None), impl=1, rank_impl=3, forms=("tick",),
              steps=3, n0=20_000, n1=6_000, check_locate=True):
    rng = np.random.default_rng(seed)
    dense = bool(cfg.flags & DENSE)
    a, b = pkg.Engine(cfg), pkg.Engine(cfg)
    book = Book()
    all_ids = []
    try:
        for e in (a, b):
            e.set_option("tick_impl", impl)
            e.set_option("rank_impl", rank_impl)
            if spread >= 0:
                e.set_option("max_spread", spread)
            e.set_lobby_budget(*budget)
            if "async" in forms[0]:
                e.set_option("async_results", 1)
        b.set_option("team_balance", mask)
        base = 0
        for step in range(steps):
            ids, r, m, ts = fresh(pkg, rng, base, n0 if step == 0 else n1, cfg.n_modes, dense)
            base += len(ids)
            acc = a.enqueue(ids, r, m, ts)
            assert np.array_equal(acc, b.enqueue(ids, r, m, ts))
            book.add(ids[acc == 1], r[acc == 1])
            all_ids.append(ids)
            if step == 1:
                a.remove(ids[::9]); b.remove(ids[::9])
            now = 2000 + step
            probe = np.concatenate(all_ids)[::37] if check_locate else None
            loc = b.locate(probe, now) if check_locate else None
            form = forms[step % len(forms)]
            ra, rb = tick(pkg, a, form, now), tick(pkg, b, form, now)
            assert np.array_equal(ra[0], rb[0])  # headers
            assert (ra[2] is None) == (rb[2] is None) and (ra[2] is None or np.array_equal(ra[2], rb[2]))
            assert ra[3].n_lobbies == rb[3].n_lobbies and ra[3].n_matched == rb[3].n_matched
            lob, mem_a, mem_b = ra[0], np.asarray(ra[1]), np.asarray(rb[1])
            if len(lob):
                starts = lob["first_member"].astype(np.int64)
                ends = starts + lob["n_members"]
                for s, e_ in zip(starts[::97], ends[::97]):  # same players per lobby (spot check; all by the order below)
                    assert set(mem_a[s:e_].tolist()) == set(mem_b[s:e_].tolist())
            want = expect_balanced(cfg, mask, lob, mem_a, book)
            assert np.array_equal(mem_b, want)
            same_state(a, b, np.concatenate(all_ids), now)
            # match quality: the emitted teams' imbalance; everything else as the unbalanced twin's
            qa, la = a.match_quality(want_lobbies=True)
            qb, lb = b.match_quality(want_lobbies=True)
            assert np.array_equal(lb["imbalance"], np.minimum(teams_imbalance(cfg, lob, mem_b, book), 0xFFFFFFFF))
            for f in ("min_rating", "max_rating", "rating_sum"):
                assert np.array_equal(la[f], lb[f])
            assert (lb["imbalance"] <= la["imbalance"]).all()
            for f in ("n_lobbies", "max_spread", "sum_spread", "spread_hist"):
                assert np.array_equal(qa[f], qb[f])
            # locate before the tick: the member index the balanced tick gave each located player
            if check_locate and len(lob):
                pos = {}
                for h in range(len(lob)):
                    f, n = int(lob["first_member"][h]), int(lob["n_members"][h])
                    for k, pid in enumerate(mem_b[f:f + n].tolist()):
                        pos[pid] = k
                for pid, st in zip(probe.tolist(), loc):
                    if st["state"] == 1 and st["lobby"] != abi.MM_LOCATE_STAYS:
                        assert pos[pid] == st["member"], (pid, st)
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
@pytest.mark.parametrize("impl", [1, 0])
def test_twins_s0_forms(pkg, order, impl):
    cfg = gpu_config(pkg, order, flags=DENSE)
    run_twins(pkg, cfg, seed=order * 2 + impl, impl=impl, forms=("tick", "tick_emit", "packed", "device"), steps=4)


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
@pytest.mark.parametrize("form", ["async", "async_packed"])
def test_twins_async_results(pkg, order, form):
    run_twins(pkg, gpu_config(pkg, order, flags=DENSE), seed=5 + order, forms=(form,))


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
@pytest.mark.parametrize("layout", ["wide", "overlap"])
@pytest.mark.parametrize("rank_impl", [2, 3])
def test_twins_layouts_and_rankings(pkg, order, layout, rank_impl):
    run_twins(pkg, gpu_config(pkg, order, layout), seed=11 + rank_impl + order, rank_impl=rank_impl,
              forms=("tick_emit", "device"))


@pytest.mark.gpu
@pytest.mark.parametrize("spread", [0, 6, 40, 400])
def test_twins_max_spread(pkg, spread):
    run_twins(pkg, gpu_config(pkg, RATING), seed=20 + spread, spread=spread, forms=("tick", "device"))


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
def test_twins_lobby_budget(pkg, order):
    cfg = gpu_config(pkg, order)
    nq = cfg.n_modes * cfg.n_groups
    rng = np.random.default_rng(3)
    run_twins(pkg, cfg, seed=30 + order, budget=(rng.integers(0, 20, nq), np.array([5, 0, 40, 9, 1000])),
              forms=("tick_emit", "device"))


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
def test_one_mode_masked_others_untouched(pkg, order):
    run_twins(pkg, gpu_config(pkg, order), seed=40 + order, mask=0b00100, forms=("tick", "device"))


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
def test_option_on_then_off(pkg, order):
    """One engine balances a tick, then the mask is set to 0: its next tick equals the never-balanced twin's."""
    cfg = gpu_config(pkg, order, flags=DENSE)
    rng = np.random.default_rng(50 + order)
    book = Book()
    with pkg.Engine(cfg) as a, pkg.Engine(cfg) as b:
        base = 0
        for step, mask in enumerate((MASK, 0)):
            b.set_option("team_balance", mask)
            ids, r, m, ts = fresh(pkg, rng, base, 20_000, cfg.n_modes, True)
            base += len(ids)
            acc = a.enqueue(ids, r, m, ts)
            assert np.array_equal(acc, b.enqueue(ids, r, m, ts))
            book.add(ids[acc == 1], r[acc == 1])
            ra, rb = a.tick(3000 + step), b.tick(3000 + step)
            assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[2], rb[2])
            want = expect_balanced(cfg, mask, ra[0], ra[1], book)
            assert np.array_equal(rb[1], want)
            assert np.array_equal(rb[1], ra[1]) == (mask == 0)
            la, lb = a.match_quality(want_lobbies=True)[1], b.match_quality(want_lobbies=True)[1]
            assert np.array_equal(la, lb) == (mask == 0)


@pytest.mark.gpu
def test_refusals(pkg):
    modes = (("1v1", 2, 1), ("3x3", 3, 3), ("9v9", 2, 9), ("8v8", 2, 8), ("coop2", 1, 2))
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=modes, order=RATING, capacity=10_000)
    with pkg.Engine(cfg) as e:
        for bad in (1 << 5, 1 << 7, 0b10, 0b100, 0b10000, -1, 1 << 40):
            with pytest.raises(eng_mod.EngineError):
                e.set_option("team_balance", bad)
        e.set_option("team_balance", 0b1001)  # 1v1 and 8v8
        e.set_option("team_balance", 0)


@pytest.mark.gpu
def test_widen_lobbies_are_the_unmasked_twins_permuted(pkg):
    cfg = gpu_config(pkg, RATING, capacity=100_000)
    rng = np.random.default_rng(60)
    book = Book()
    with pkg.Engine(cfg) as a, pkg.Engine(cfg) as b:
        b.set_option("team_balance", MASK)
        ids, r, m, ts = fresh(pkg, rng, 0, 30_000, cfg.n_modes, False)
        ts = (rng.integers(0, 100_000, len(ids))).astype(np.uint32)
        for e in (a, b):
            assert e.enqueue(ids, r, m, ts).all()
        book.add(ids, r)
        rules = {(mm, g): (20_000, 10, 5_000, 15, 400) for mm in range(cfg.n_modes) for g in range(cfg.n_groups)}
        la, ma, sa = a.widen(200_000, rules)
        lb, mb, sb = b.widen(200_000, rules)
        assert sa.n_lobbies == sb.n_lobbies > 0 and np.array_equal(la, lb)
        assert np.array_equal(mb, expect_balanced(cfg, MASK, la, ma, book))
        assert not np.array_equal(ma, mb)
        same_state(a, b, ids, 200_000)


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
@pytest.mark.parametrize("form", ["tick", "device"])
def test_config3_ten_million(pkg, order, form):
    """At 10 M players the pass takes about a millisecond: mm_tick_device must return only once it is done, so the
    members mm_results_device hands out, read on another stream, are the balanced ones."""
    from .test_tile_geometry import config3_pool
    n = 10_000_000
    cfg, _ = pkg.synth.workload_config("config3_10m_g32_5v5", order, n)
    ids, rating, mode, ts = config3_pool(pkg, n)
    lo, hi = clamp_bounds(cfg)
    with pkg.Engine(cfg) as a, pkg.Engine(cfg) as b:
        b.set_option("team_balance", 1)
        for e in (a, b):
            assert e.enqueue(ids, rating, mode, ts).all()
        ra, rb = tick(pkg, a, form, 10 ** 6), tick(pkg, b, form, 10 ** 6)
        assert np.array_equal(ra[0], rb[0]) and ra[3].n_lobbies > 900_000
        assert (ra[2] is None and rb[2] is None) or np.array_equal(ra[2], rb[2])
        lob = ra[0]
        assert (lob["mode"] == 0).all() and (lob["n_members"] == 10).all()
        c = np.clip(rating.astype(np.int64), lo, hi)  # dense ids: id = index
        idx = lob["first_member"].astype(np.int64)[:, None] + np.arange(10)
        ma, mb = ra[1][idx], rb[1][idx]
        perm, d = split_numpy(c[ma.astype(np.int64)], 5)
        assert np.array_equal(mb, np.take_along_axis(ma, perm, 1))
        qa, _ = a.match_quality()
        qb, lqb = b.match_quality(want_lobbies=True)
        assert np.array_equal(lqb["imbalance"], d)
        assert qb["sum_imbalance"].sum() == d.sum() < qa["sum_imbalance"].sum()
        assert np.array_equal(a.pool_read()["id"], b.pool_read()["id"])
