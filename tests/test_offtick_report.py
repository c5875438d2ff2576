"""Off-tick match report (mm_offtick_report / Engine.offtick_report / SearchPool.offtick_status): the waits and the
rating quality of the lobbies the last mm_party_match and the last mm_widen call formed, captured on the device.

The restatement starts from each call's own headers and members and from the test's own maps: solo id -> (rating,
stamp), party member id -> (own rating, party stamp).  The quality half is test_match_quality.restate; the engine must
equal the restatement exactly.
CPU: the ABI mirror, the buckets at and above 2^31, SearchPool.offtick_status / SearchWorker.status() on an engine
double.
GPU: split, wide and overlapping layouts with a default group, clamped ratings and party members whose own ratings lie
outside every group; 1-team, 1-player-team, 2- and 3-team modes; hashed ids and dense handles; team_balance and
party_balance; future stamps, waits across the 2^32 wrap of `now` and the largest wait; the void and empty states,
independence of the sources and of every other call; every refusal; twin engines; the model schedule; config3 at 10 M.
"""
import ctypes as C
import importlib

import numpy as np
import pytest

from .fakes import OracleEngine
from .test_engine_model import EngineSchedule
from .test_match_quality import MODES, gpu_config, restate
from .test_widen import rules_of

sw = importlib.import_module("microservice-matchmaking_b200.search_worker")
eng_mod = importlib.import_module("microservice-matchmaking_b200.engine")
abi = importlib.import_module("microservice-matchmaking_b200.abi")

RATING, ARRIVAL = 1, 0
DENSE, WIDE, NO_DEDUPE = 2, 4, 1
NB = abi.MM_WAIT_BUCKETS
PM, WD = abi.MM_OFFTICK_PARTY_MATCH, abi.MM_OFFTICK_WIDEN
U32 = 1 << 32


# ================================================================================ restatement
class Book:
    """id -> (rating, stamp) of every player a call can put into a lobby: a solo's pool rating and own stamp, a party
    member's own rating and its party's stamp (the test's own inputs).  A later entry for an id replaces the earlier."""

    def __init__(self):
        self.ids, self.r, self.ts = np.zeros(0, np.uint64), np.zeros(0, np.int64), np.zeros(0, np.int64)

    def add(self, ids, rating, ts):
        ids = np.concatenate([np.asarray(ids, np.uint64), self.ids])
        r = np.concatenate([np.asarray(rating, np.int64), self.r])
        ts = np.concatenate([np.asarray(ts, np.int64) & (U32 - 1), self.ts])
        self.ids, first = np.unique(ids, return_index=True)  # the first occurrence: the newest entry
        self.r, self.ts = r[first], ts[first]

    def _at(self, ids):
        ids = np.asarray(ids, np.uint64)
        k = np.searchsorted(self.ids, ids)
        assert (k < len(self.ids)).all() and np.array_equal(self.ids[np.minimum(k, len(self.ids) - 1)], ids)
        return k

    def rating(self, ids):
        return self.r[self._at(ids)]

    def stamp(self, ids):
        return self.ts[self._at(ids)]


def member_slots(lob):
    """The member slots of every lobby, in header order."""
    n = lob["n_members"].astype(np.int64)
    start = np.repeat(lob["first_member"].astype(np.int64), n)
    return start + np.arange(int(n.sum())) - np.repeat(np.cumsum(n) - n, n)


def restate_offtick(cfg, lob, mem, now, book):
    """-> (WAITS_DTYPE, QUALITY_DTYPE, LOBBY_QUALITY_DTYPE) of one call's headers and members at its `now`."""
    lob = np.asarray(lob, eng_mod.LOBBY_DTYPE)
    mem = np.asarray(mem, np.uint64)
    pq, pl = restate(cfg, lob, mem, book.rating)
    G = cfg.n_groups
    n_cut = cfg.n_modes * G
    w = np.zeros(n_cut, eng_mod.WAITS_DTYPE)
    w["mode"], w["group"] = np.arange(n_cut) // G, np.arange(n_cut) % G
    if len(lob):
        q = lob["mode"].astype(np.int64) * G + lob["group"]
        qm = np.repeat(q, lob["n_members"].astype(np.int64))
        wait = eng_mod.wait_of(now, book.stamp(mem[member_slots(lob)]).astype(np.uint64))
        w["n_lobbies"] = np.bincount(q, minlength=n_cut)
        w["n_matched"] = np.bincount(qm, minlength=n_cut)
        np.maximum.at(w["max_match_wait"], qm, wait.astype(np.uint32))
        np.add.at(w["match_wait_hist"], (qm, eng_mod.wait_bucket(wait)), 1)
    return w, pq, pl


def check_report(eng, src, want):
    """The engine's report of `src` equals `want` ((waits, quality, lobbies), or None: void)."""
    w, q, lob = eng.offtick_report(src, want_lobbies=True)
    w2, q2, none = eng.offtick_report(src)
    assert none is None
    if want is None:
        assert len(w) == len(q) == len(lob) == len(w2) == len(q2) == 0
        return
    assert np.array_equal(lob, want[2])
    assert np.array_equal(w, want[0]) and np.array_equal(w2, want[0])
    assert np.array_equal(q, want[1]) and np.array_equal(q2, want[1])


# ================================================================================ CPU
def test_abi_mirror():
    assert C.sizeof(abi.MatchWaits) == 496 == eng_mod.WAITS_DTYPE.itemsize
    for f, *_ in abi.MatchWaits._fields_:
        assert getattr(abi.MatchWaits, f).offset == eng_mod.WAITS_DTYPE.fields[f][1], f
    want = {"n_lobbies": 4, "n_matched": 8, "max_match_wait": 12, "match_wait_hist": 16}
    for f, off in want.items():
        assert eng_mod.WAITS_DTYPE.fields[f][1] == off, f
    # the waits record is the match section of mm_queue_stat, field for field
    base = eng_mod.QUEUE_STAT_DTYPE.fields["n_lobbies"][1] - 4
    for f in ("n_lobbies", "n_matched", "max_match_wait", "match_wait_hist"):
        assert eng_mod.QUEUE_STAT_DTYPE.fields[f][1] - base == eng_mod.WAITS_DTYPE.fields[f][1], f
    assert (abi.MM_OFFTICK_PARTY_MATCH, abi.MM_OFFTICK_WIDEN) == (0, 1)
    assert "mm_offtick_report" in abi.PROTOTYPES


def test_bucket_at_and_above_two_to_the_31():
    # the largest wait: (now - enq_ts) mod 2^32 = 2^31 - 1 -> bucket 119; a difference of 2^31 or more reads as a
    # stamp in the future, wait 0
    assert eng_mod.wait_bucket((1 << 31) - 1) == NB - 1
    assert eng_mod.wait_of((1 << 31) - 1 + 5, 5) == (1 << 31) - 1
    assert eng_mod.wait_of((1 << 31) + 5, 5) == 0 and eng_mod.wait_of(U32 + 3, 5) == 0
    assert eng_mod.wait_of(U32 + 3, U32 - 7) == 10  # across the wrap of now
    for x in (1 << 31, (1 << 31) + 1, 3 << 30, U32 - 1):  # spreads and imbalances of 2^31 or more
        assert eng_mod.quality_bucket(x) == NB - 1


def test_restatement_by_hand(pkg):
    cfg = pkg.synth.make_config(groups=[(0, 99), (100, 199)], modes=(("2v2", 2, 2),), order=RATING, capacity=100,
                                default_group=-1)
    book = Book()
    book.add(np.arange(1, 9, dtype=np.uint64), [10, 20, 30, 80, 150, 150, 199, 120], [990, 900, 1005, 0, 1000, 1000,
                                                                                         1000 - 20, 1000 - 9])
    lob = np.zeros(2, eng_mod.LOBBY_DTYPE)
    lob[0] = (0, 4, 0, 0)
    lob[1] = (4, 4, 0, 1)
    w, q, pl = restate_offtick(cfg, lob, np.arange(1, 9, dtype=np.uint64), 1000, book)
    assert w["n_lobbies"].tolist() == [1, 1] and w["n_matched"].tolist() == [4, 4]
    assert w["max_match_wait"].tolist() == [1000, 20]  # 10, 100, 0 (future), 1000; 0, 0, 20, 9
    assert w[0]["match_wait_hist"][0] == 1 and w[1]["match_wait_hist"][0] == 2
    assert pl["imbalance"].tolist() == [80, 19] and q["n_lobbies"].tolist() == [1, 1]


class WidenEngine(OracleEngine):
    """A CPU engine double with a widening call: each enabled queue's players, oldest first, L at a time; its
    offtick_report restates the lobbies it returned.  Its tick matches nobody."""

    def __init__(self, cfg):
        super().__init__(cfg)
        self.book = Book()
        self.report = None

    def enqueue(self, ids, rating, mode, enq_ts=None):
        acc = super().enqueue(ids, rating, mode, enq_ts)
        k = acc == 1
        self.book.add(np.asarray(ids, np.uint64)[k], np.asarray(rating)[k], np.asarray(enq_ts)[k])
        return acc

    def tick(self, now=0):
        st = self.abi.TickStats()
        return np.zeros(0, eng_mod.LOBBY_DTYPE), np.zeros(0, np.uint64), np.zeros(0, np.uint32), st

    def widen(self, now, rules):
        p = self.pool_read()
        grp = np.array([self.oracle.find_rating_group(self.cfg, int(r)) for r in p["rating"]], np.int64)
        lob, mem = [], []
        for (m, g), _rule in sorted(rules.items()):
            L = self.cfg.modes[m].teams * self.cfg.modes[m].team_size
            x = p["id"][(p["mode"] == m) & (grp == g)]
            x = x[np.argsort(self.book.stamp(x), kind="stable")][:len(x) // L * L]
            for k in range(len(x) // L):
                lob.append((len(mem) + k * L, L, m, g))
            mem.extend(x.tolist())
        lob = np.array(lob, eng_mod.LOBBY_DTYPE)
        mem = np.array(mem, np.uint64)
        self.take(mem)
        self.report = restate_offtick(self.cfg, lob, mem, now, self.book)
        st = self.abi.WidenStats()
        st.n_lobbies, st.n_matched = len(lob), len(mem)
        return lob, mem, st

    def offtick_report(self, source, want_lobbies=False):
        if source != WD or self.report is None:
            return (np.zeros(0, eng_mod.WAITS_DTYPE), np.zeros(0, eng_mod.QUALITY_DTYPE),
                    np.zeros(0, eng_mod.LOBBY_QUALITY_DTYPE) if want_lobbies else None)
        return self.report[0], self.report[1], (self.report[2] if want_lobbies else None)


def test_search_pool_and_worker_status(pkg):
    from .fakes import FakeBroker
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=RATING, capacity=2000)
    eng = WidenEngine(cfg)
    pool = sw.SearchPool(eng, ["1v1", "5v5"], pkg.synth.REFERENCE_GROUP_NAMES, flush_every_s=3600, clock=lambda: 5.0,
                         widen={"1v1": (100, 10, 50, 5, 200), "5v5": (100, 10, 50, 5, 200)})
    ok, w = sw.SearchWorker.start_link(FakeBroker(), pool, {"group_name": "gold", "channel_name": "search.gold"})
    assert ok == "ok"
    assert pool.offtick_status("gold") == {} and w.status()[1]["offtick"] == {}  # void before the first call
    assert pool.offtick_status("nowhere") == {}
    rng = np.random.default_rng(5)
    n, now = 600, 50_000
    ids = np.arange(1, n + 1, dtype=np.uint64)
    rating = rng.integers(2000, 2500, n).astype(np.int32)  # gold
    mode = (np.arange(n) % 3 == 0).astype(np.uint8)
    ts = (now - rng.integers(0, 40_000, n)).astype(np.uint32)
    eng.enqueue(ids, rating, mode, ts)
    lob, mem, _ = eng.widen(now, {(m, 2): None for m in range(2)})
    got = pool.offtick_status("gold")
    assert set(got) == {"1v1", "5v5"} and all(set(v) == {"widen"} for v in got.values())
    for m, name in enumerate(("1v1", "5v5")):
        sel = lob[lob["mode"] == m]
        assert len(sel) > 0
        wait = eng_mod.wait_of(now, eng.book.stamp(mem[member_slots(sel)]))
        hist = np.bincount(eng_mod.wait_bucket(wait), minlength=NB)
        L = int(sel["n_members"][0])
        c = np.clip(eng.book.rating(mem[member_slots(sel)]).reshape(len(sel), L), -1, 5001)
        spread = c.max(1) - c.min(1)
        teams = c.reshape(len(sel), 2, L // 2).sum(2)
        imb = teams.max(1) - teams.min(1)
        q = lambda v, p: eng_mod.wait_quantile(np.bincount(eng_mod.quality_bucket(v), minlength=NB), p)  # noqa: E731
        assert got[name]["widen"] == {
            "lobbies": len(sel), "matched": len(wait),
            "p50_match_wait_ms": eng_mod.wait_quantile(hist, 0.5),
            "p99_match_wait_ms": eng_mod.wait_quantile(hist, 0.99),
            "max_match_wait_ms": int(wait.max()),
            "mean_spread": spread.sum() / len(sel), "p99_spread": q(spread, 0.99), "max_spread": int(spread.max()),
            "mean_imbalance": imb.sum() / len(sel), "p99_imbalance": q(imb, 0.99), "max_imbalance": int(imb.max()),
        }
    ok, st = w.status()
    assert ok == "ok" and st["offtick"] == got
    assert "waiting" not in st or isinstance(st["waiting"], dict)
    # a pool that runs neither parties nor widen, or an engine without offtick_report: no "offtick"
    pool2 = sw.SearchPool(WidenEngine(cfg), ["1v1", "5v5"], pkg.synth.REFERENCE_GROUP_NAMES, flush_every_s=3600)
    ok, w2 = sw.SearchWorker.start_link(FakeBroker(), pool2, {"group_name": "gold", "channel_name": "search.gold"})
    assert "offtick" not in w2.status()[1]
    pool3 = sw.SearchPool(OracleEngine(cfg), ["1v1", "5v5"], pkg.synth.REFERENCE_GROUP_NAMES, flush_every_s=3600,
                          widen={"1v1": (100, 10, 50, 5, 200)})
    ok, w3 = sw.SearchWorker.start_link(FakeBroker(), pool3, {"group_name": "gold", "channel_name": "search.gold"})
    assert "offtick" not in w3.status()[1]


# ================================================================================ GPU
PARTY_MODES = [k for k, (_, T, S) in enumerate(MODES) if S >= 2]  # 5v5, coop4, 3x3


class Driver:
    """One engine with party capacity, its Book and a supply of fresh players and parties."""

    def __init__(self, pkg, cfg, seed, pcap=60_000):
        self.pkg, self.cfg = pkg, cfg
        self.dense = bool(cfg.flags & DENSE)
        self.eng = pkg.Engine(cfg)
        if pcap:
            self.eng.set_option("party_capacity", pcap)
        self.rng = np.random.default_rng(seed)
        self.book = Book()
        self.next = 0
        self.now = 10_000

    def fresh_ids(self, n):
        x = np.arange(self.next, self.next + n, dtype=np.uint64)
        self.next += n
        return x if self.dense else self.pkg.synth.mix64(x + np.uint64(13 << 40))

    def stamps(self, n, spread=3000):
        """Waits up to `spread`; 3 % in the future; a few of the largest wait 2^31 - 1."""
        rng = self.rng
        w = rng.integers(0, spread, n).astype(np.int64)
        w[rng.random(n) < 0.03] = -rng.integers(1, 1000)
        w[rng.random(n) < 0.002] = (1 << 31) - 1
        return ((self.now - w) % U32).astype(np.uint32)

    def solos(self, n, lo=-400, hi=5400):
        rng = self.rng
        ids = self.fresh_ids(n)
        r = rng.integers(lo, hi, n).astype(np.int32)
        m = rng.integers(0, self.cfg.n_modes, n).astype(np.uint8)
        ts = self.stamps(n)
        acc = self.eng.enqueue(ids, r, m, ts)
        self.book.add(ids[acc == 1], r[acc == 1], ts[acc == 1])
        return ids[acc == 1]

    def parties(self, n, modes=PARTY_MODES, spread=700):
        """n parties of 2 .. S members; the members' own ratings spread +-spread around R, so some lie outside every
        group."""
        rng, cfg = self.rng, self.cfg
        mode = rng.choice(modes, n).astype(np.uint8)
        size = np.array([rng.integers(2, cfg.modes[k].team_size + 1) for k in mode], np.uint8)
        ids = self.fresh_ids(int(size.sum()))
        r = (np.repeat(rng.integers(100, 4900, n), size) + rng.integers(-spread, spread + 1, len(ids))).astype(np.int32)
        ts = self.stamps(n)
        code = self.eng.enqueue_party(size, ids, r, mode, ts)
        k = np.repeat(code == 1, size)
        self.book.add(ids[k], r[k], np.repeat(ts, size)[k])
        return code

    def party_match(self, rules):
        lob, mem, st = self.eng.party_match(self.now, rules_of(self.cfg, rules), lobby_cap=1 << 16, member_cap=1 << 20)
        return lob, mem, st, restate_offtick(self.cfg, lob, mem, self.now, self.book)

    def widen(self, rules):
        lob, mem, st = self.eng.widen(self.now, rules_of(self.cfg, rules), lobby_cap=1 << 16, member_cap=1 << 20)
        return lob, mem, st, restate_offtick(self.cfg, lob, mem, self.now, self.book)

    def close(self):
        self.eng.close()


def all_queues(cfg, rule):
    return {(m, g): rule for m in range(cfg.n_modes) for g in range(cfg.n_groups)}


def masked_sum(cfg, quality, mask):
    return sum(int(r["sum_imbalance"]) for r in quality if (mask >> int(r["mode"])) & 1)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["split", "wide", "overlap"])
@pytest.mark.parametrize("kind", ["hashed", "dense"])
def test_report_equals_restatement(pkg, layout, kind):
    cfg = gpu_config(pkg, RATING, layout, DENSE if kind == "dense" else 0)
    d = Driver(pkg, cfg, seed=len(layout) * 3 + len(kind))
    seen = {"bucket119": 0, "bucket0": 0, "pm_modes": set(), "wd_modes": set(), "balanced_pm": 0}
    try:
        # the third step's `now` lies past 2^32: its waits cross the wrap
        for step, now in enumerate((10_000, U32 - 1500, U32 + 1200, 2 * U32 + 7)):
            d.now = now
            tb = 0b11 if step % 2 else 0  # team_balance: 1v1 and 5v5 (the two-team modes)
            pb = 0b10 if step % 2 else 0  # party_balance: 5v5 (3x3 has three teams, coop4 one)
            d.eng.set_option("team_balance", tb)
            d.eng.set_option("party_balance", pb)
            d.solos(40_000)
            d.parties(1500)
            lob, mem, st, want_pm = d.party_match(all_queues(cfg, (0, 40, 100, 20, 500)))
            assert st.n_lobbies > 0
            check_report(d.eng, PM, want_pm)
            if pb:
                assert masked_sum(cfg, want_pm[1], pb) == st.sum_imbalance
                seen["balanced_pm"] += st.sum_imbalance > 0
            seen["pm_modes"] |= set(lob["mode"].tolist())
            d.eng.tick(now)  # the tick leaves both reports alone
            check_report(d.eng, PM, want_pm)
            d.solos(20_000)
            lob, mem, st, want_wd = d.widen(all_queues(cfg, (1500, 30, 200, 40, 800)))
            assert st.n_lobbies > 0
            check_report(d.eng, WD, want_wd)
            check_report(d.eng, PM, want_pm)
            seen["wd_modes"] |= set(lob["mode"].tolist())
            seen["bucket119"] += int(want_wd[0]["match_wait_hist"][:, NB - 1].sum() + want_pm[0]["match_wait_hist"][:, NB - 1].sum())
            seen["bucket0"] += int(want_wd[0]["match_wait_hist"][:, 0].sum() + want_pm[0]["match_wait_hist"][:, 0].sum())
        assert seen["bucket119"] > 0 and seen["bucket0"] > 0, seen
        assert {1, 2, 4} <= seen["pm_modes"], seen  # party modes of 2, 1 and 3 teams
        assert {2, 3} <= seen["wd_modes"], seen     # coop4 (T = 1) and ffa6 (S = 1)
        assert seen["balanced_pm"] > 0, seen
    finally:
        d.close()


def raw_report(eng, src, cap, lobby_cap, waits=True, quality=True, lobbies=True):
    """mm_offtick_report with poisoned buffers -> (status, n_out, n_lobbies, waits, quality, per_lobby)."""
    wb = np.full(max(cap, 1) * eng_mod.WAITS_DTYPE.itemsize, 0xAB, np.uint8)
    qb = np.full(max(cap, 1) * eng_mod.QUALITY_DTYPE.itemsize, 0xAB, np.uint8)
    lb = np.full(max(lobby_cap, 1) * eng_mod.LOBBY_QUALITY_DTYPE.itemsize, 0xAB, np.uint8)
    n, nl = C.c_uint32(0xDEAD), C.c_uint32(0xDEAD)
    p = lambda a, on: a.ctypes.data_as(C.c_void_p) if on else None  # noqa: E731
    rc = eng.lib.mm_offtick_report(eng.h, src, p(wb, waits), p(qb, quality), cap, C.byref(n), p(lb, lobbies), lobby_cap,
                                   C.byref(nl))
    return rc, n.value, nl.value, wb, qb, lb


def untouched(*bufs):
    return all((b == 0xAB).all() for b in bufs)


@pytest.mark.gpu
def test_void_empty_independent_and_refusals(pkg):
    cfg = gpu_config(pkg, RATING, "split")
    n_cut = cfg.n_modes * cfg.n_groups
    d = Driver(pkg, cfg, seed=77, pcap=0)
    e = d.eng
    try:
        check_report(e, PM, None)
        check_report(e, WD, None)
        # refused calls leave the reports void: no party capacity; a bad rule; null rules
        with pytest.raises(pkg.EngineError) as ei:
            e.party_match(d.now, rules_of(cfg, all_queues(cfg, (0, 10, 10, 1, 50))))
        assert ei.value.status == abi.MM_E_STATE
        check_report(e, PM, None)
        e.set_option("party_capacity", 50_000)
        d.solos(30_000)
        # valid and empty: no queue served; no live party; no anchor filled a lobby
        zero_w = np.zeros(n_cut, eng_mod.WAITS_DTYPE)
        zero_w["mode"], zero_w["group"] = np.arange(n_cut) // cfg.n_groups, np.arange(n_cut) % cfg.n_groups
        zero_q = np.zeros(n_cut, eng_mod.QUALITY_DTYPE)
        zero_q["mode"], zero_q["group"] = zero_w["mode"], zero_w["group"]
        empty = (zero_w, zero_q, np.zeros(0, eng_mod.LOBBY_QUALITY_DTYPE))
        lob, _, _ = e.widen(d.now, rules_of(cfg, {}))
        assert len(lob) == 0
        check_report(e, WD, empty)
        lob, _, _ = e.party_match(d.now, rules_of(cfg, all_queues(cfg, (0, 10, 10, 1, 50))))
        assert len(lob) == 0
        check_report(e, PM, empty)
        lob, _, st = e.widen(d.now, rules_of(cfg, all_queues(cfg, (1 << 31, 0, 1, 0, 0))))  # above every wait
        assert len(lob) == 0
        check_report(e, WD, empty)
        lob, mem, st = e.widen(d.now, rules_of(cfg, {(0, 2): (0, 0, 1, 0, 0), (1, 2): (2500, 0, 1, 0, 0)}))
        check_report(e, WD, restate_offtick(cfg, lob, mem, d.now, d.book))

        def refuse(status, call):
            with pytest.raises(pkg.EngineError) as ei:
                call()
            assert ei.value.status == status

        def raw_call(fn, rules, lobby_cap=0, member_cap=0):
            st = abi.WidenStats() if fn == "mm_widen" else abi.PartyStats()
            return getattr(e.lib, fn)(e.h, d.now, None if rules is None else rules.ctypes.data_as(C.c_void_p), None,
                                      lobby_cap, None, member_cap, C.byref(st))

        wrules = rules_of(cfg, all_queues(cfg, (1500, 30, 200, 40, 800)))
        prules = rules_of(cfg, all_queues(cfg, (0, 40, 100, 20, 500)))
        bad = wrules.copy()
        bad["step"][3] = 0
        for fn, src, rules, drv in (("mm_widen", WD, wrules, d.widen), ("mm_party_match", PM, prules, d.party_match)):
            for refusal in ("bad_rule", "null", "dry_run"):
                d.parties(800)
                d.solos(10_000)
                want = drv(all_queues(cfg, (1500, 30, 200, 40, 800)) if src == WD else
                           all_queues(cfg, (0, 40, 100, 20, 500)))[3]
                assert want[0]["n_lobbies"].sum() > 0
                check_report(e, src, want)
                d.parties(800)
                d.solos(10_000)
                rc = {"bad_rule": lambda: raw_call(fn, bad), "null": lambda: raw_call(fn, None),
                      "dry_run": lambda: raw_call(fn, rules)}[refusal]()
                assert rc == (abi.MM_E_CAP if refusal == "dry_run" else abi.MM_E_ARG), (fn, refusal, rc)
                check_report(e, src, None)
        # the sources are independent: a widen report survives party calls and the other way round
        want_wd = d.widen(all_queues(cfg, (1500, 30, 200, 40, 800)))[3]
        d.parties(800)
        want_pm = d.party_match(all_queues(cfg, (0, 40, 100, 20, 500)))[3]
        assert want_pm[0]["n_lobbies"].sum() > 0 and want_wd[0]["n_lobbies"].sum() > 0
        check_report(e, WD, want_wd)
        assert raw_call("mm_party_match", None) == abi.MM_E_ARG
        check_report(e, WD, want_wd)
        check_report(e, PM, None)
        want_pm = d.party_match(all_queues(cfg, (0, 40, 100, 20, 500)))[3]
        check_report(e, PM, want_pm)

        # nothing else changes a report
        def same():
            check_report(e, WD, want_wd)
            check_report(e, PM, want_pm)

        d.parties(300)
        ids = d.solos(5000)
        same()
        e.tick(d.now)
        same()
        e.remove(ids[:50])
        same()
        e.expire(d.now, 2900)
        same()
        d.solos(2000)
        pool = e.pool_read()
        k = min(40, len(pool["id"]))
        assert k > 0
        taken = pool["id"][:k]
        e.take(taken)
        same()
        e.requeue(taken, pool["rating"][:k], pool["mode"][:k], pool["enq_ts"][:k], np.arange(1, k + 1, dtype=np.uint32))
        same()
        e.backfill(1, 2, 2200, 5, 100)
        same()
        e.band_candidates(20, 3)
        same()
        e.band_match(20, 1, 2)
        same()
        e.set_option("team_balance", 1)
        e.set_option("party_balance", 2)
        e.set_option("max_spread", 30)
        e.set_lobby_budget(per_queue=np.full(n_cut, 3, np.uint32))
        same()
        e.set_lobby_budget()
        pr = e.party_read()
        assert len(pr["size"])
        mids, mrat = pr["members"][0]
        e.requeue_party(pr["size"][:1], mids, mrat, pr["mode"][:1], pr["enq_ts"][:1], pr["seq"][:1])
        same()
        pimg = e.export_parties()  # the image calls need the parties released
        same()
        e.snapshot()
        same()
        e.restore()
        same()
        mask = np.zeros(n_cut, bool)
        mask[2::cfg.n_groups] = True
        e.merge_queues(e.export_queues(mask))
        same()
        e.merge_parties(pimg)
        same()
        e.tick(d.now + 5)
        same()
        # an imported engine starts void
        pimg = e.export_parties()
        img = e.export_state()
        with pkg.Engine(cfg) as f:
            f.import_state(img)
            check_report(f, WD, None)
            check_report(f, PM, None)
        e.merge_parties(pimg)
        same()

        # refusals of the report itself: decided before anything is written
        assert e.lib.mm_offtick_report(None, WD, None, None, 0, C.byref(C.c_uint32()), None, 0,
                                       C.byref(C.c_uint32())) == abi.MM_E_ARG
        assert e.lib.mm_offtick_report(e.h, WD, None, None, 0, None, None, 0, C.byref(C.c_uint32())) == abi.MM_E_ARG
        assert e.lib.mm_offtick_report(e.h, WD, None, None, 0, C.byref(C.c_uint32()), None, 0, None) == abi.MM_E_ARG
        rc, n, nl, wb, qb, lb = raw_report(e, 2, n_cut, 1 << 12)
        assert rc == abi.MM_E_ARG and untouched(wb, qb, lb)
        nlob = len(want_wd[2])
        for waits, quality in ((True, False), (False, True), (True, True)):
            rc, n, nl, wb, qb, lb = raw_report(e, WD, n_cut - 1, nlob, waits, quality)
            assert rc == abi.MM_E_CAP and n == n_cut and nl == nlob and untouched(wb, qb, lb)
        rc, n, nl, wb, qb, lb = raw_report(e, WD, 0, 0, False, False, False)  # counts only
        assert rc == abi.MM_OK and n == n_cut and nl == nlob
        rc, n, nl, wb, qb, lb = raw_report(e, WD, n_cut, nlob - 1)
        assert rc == abi.MM_E_CAP and nl == nlob and untouched(wb, qb, lb)
        rc, n, nl, wb, qb, lb = raw_report(e, WD, n_cut, 0, True, True, False)
        assert rc == abi.MM_OK and n == n_cut and nl == nlob and untouched(lb)
        assert np.array_equal(wb.view(eng_mod.WAITS_DTYPE), want_wd[0])
        same()
    finally:
        d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("order,flags", [(ARRIVAL, 0), (RATING, NO_DEDUPE)])
def test_engines_that_refuse_both_calls_stay_void(pkg, order, flags):
    cfg = gpu_config(pkg, order, "split", flags)
    d = Driver(pkg, cfg, seed=9, pcap=0)
    try:
        d.solos(20_000)
        for call in (d.widen, d.party_match):
            with pytest.raises(pkg.EngineError):
                call(all_queues(cfg, (0, 10, 10, 1, 50)))
        d.eng.tick(d.now)
        check_report(d.eng, PM, None)
        check_report(d.eng, WD, None)
    finally:
        d.close()


def outputs_equal(a, b):
    if isinstance(a, tuple):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            outputs_equal(x, y)
    elif isinstance(a, np.ndarray):
        assert np.array_equal(a, b)
    elif isinstance(a, C.Structure):
        for f, *_ in a._fields_:
            if not f.endswith("_us"):  # timings
                x, y = getattr(a, f), getattr(b, f)
                assert (list(x) == list(y)) if hasattr(x, "__len__") else x == y, f
    else:
        assert a == b


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
def test_twin_engines_over_a_mixed_schedule(pkg, kind):
    """Twin A reads both reports after every step, twin B never: every output of every call is equal on both."""
    cfg = gpu_config(pkg, RATING, "overlap", DENSE if kind == "dense" else 0)
    a, b = Driver(pkg, cfg, seed=31), Driver(pkg, cfg, seed=31)
    rng = np.random.default_rng(32)
    try:
        wants = {PM: None, WD: None}
        for step in range(40):
            op = str(rng.choice(["solos", "parties", "party_match", "tick", "widen", "expire", "option"]))
            for d in (a, b):
                d.now += 150
            if op == "solos":
                outputs_equal(a.solos(8000), b.solos(8000))
            elif op == "parties":
                outputs_equal(a.parties(400), b.parties(400))
            elif op == "party_match":
                rule = all_queues(cfg, (int(rng.integers(0, 2000)), 40, 100, 20, 500))
                ra, rb = a.party_match(rule), b.party_match(rule)
                outputs_equal(ra[:3], rb[:3])
                wants[PM] = ra[3]
            elif op == "widen":
                rule = all_queues(cfg, (int(rng.integers(500, 2500)), 30, 200, 40, 800))
                ra, rb = a.widen(rule), b.widen(rule)
                outputs_equal(ra[:3], rb[:3])
                wants[WD] = ra[3]
            elif op == "tick":
                outputs_equal(a.eng.tick(a.now), b.eng.tick(b.now))
            elif op == "expire":  # the expired players come in no set order
                (ia, sa), (ib, sb) = a.eng.expire(a.now, 2800), b.eng.expire(b.now, 2800)
                oa, ob = np.lexsort((sa, ia)), np.lexsort((sb, ib))
                outputs_equal((ia[oa], sa[oa]), (ib[ob], sb[ob]))
            else:
                v = int(rng.integers(0, 4))
                for d in (a, b):
                    d.eng.set_option("team_balance", v)
                    d.eng.set_option("party_balance", v & 2)
            for src in (PM, WD):
                check_report(a.eng, src, wants[src])
        pa, pb = a.eng.pool_read(), b.eng.pool_read()
        for k in pa:
            assert np.array_equal(pa[k], pb[k]), k
        for src in (PM, WD):
            check_report(b.eng, src, wants[src])
    finally:
        a.close()
        b.close()


class OtSchedule(EngineSchedule):
    """EngineSchedule that restates both off-tick reports at every party_match and widen step and checks them after
    every step; a checkpoint loads a fresh engine, whose reports are void."""

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        self.want = {PM: None, WD: None}

    def _book(self, parties):
        m = self.m
        b = Book()
        a = m.q["alive"]
        b.add(m.q["id"][a], m.q["rating"][a], m.q["ts"][a])
        if parties:
            for p in m.parties:
                b.add(p[0], p[1], np.full(len(p[0]), p[3], np.int64))
        return b

    def party_match(self, rules=None):
        book = self._book(True)
        lob, mem = super().party_match(rules)
        self.want[PM] = restate_offtick(self.cfg, lob, mem, self.now, book)
        self.count("offtick_pm" if len(lob) else "offtick_pm_empty")
        return lob, mem

    def widen(self, rules=None):
        book = self._book(False)
        lob, mem = super().widen(rules)
        self.want[WD] = restate_offtick(self.cfg, lob, mem, self.now, book)
        self.count("offtick_wd" if len(lob) else "offtick_wd_empty")
        return lob, mem

    def checkpoint(self):
        super().checkpoint()
        self.want = {PM: None, WD: None}

    def check(self):
        super().check()
        for src in (PM, WD):
            check_report(self.eng, src, self.want[src])


@pytest.mark.gpu
@pytest.mark.parametrize("dense,wide", [(False, False), (True, True)], ids=lambda v: str(v))
def test_model_schedule(pkg, oracle, dense, wide):
    from .test_tile_geometry import MODES8
    rng = np.random.default_rng(900 + 2 * dense + wide)
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[:4], order=RATING, capacity=300_000,
                                active_capacity=4_000_000, default_group=-1, flags=(DENSE if dense else 0) | WIDE * wide)
    s = OtSchedule(pkg, oracle, cfg, rng, dense)
    try:
        s.players(60_000, old=0.02)
        s.party_batch(1500)
        s.check()
        for _ in range(110):
            s.step()
        s.check()
        for what in ("offtick_pm", "offtick_wd", "checkpoint", "queue_move", "requeue", "expire"):
            assert s.counts.get(what, 0) >= 1, (what, s.counts)
    finally:
        s.close()


@pytest.mark.gpu
def test_config3_ten_million(pkg):
    """config3 (32 groups, 5v5) at 10 M solos with 1 % of the players in parties, then a widen call at 10 M whose
    min_wait is about the 99th percentile of the waits."""
    name = "config3_10m_g32_5v5"
    n = pkg.synth.WORKLOADS[name]["n"]
    cfg, mode_idx = pkg.synth.workload_config(name, RATING, n)
    ids, rating, mode, ts = pkg.synth.gen_pool(1, n, mode=mode_idx)
    rng = np.random.default_rng(2)
    now = int(ts.max()) + 1
    dense = bool(cfg.flags & DENSE)
    book = Book()
    book.add(ids, rating, ts)
    with pkg.Engine(cfg) as e:
        assert e.enqueue(ids, rating, mode, ts).all()
        e.set_option("party_capacity", n // 20)
        k = int(n * 0.01 / 0.99 / 3)
        sizes = rng.integers(2, 5, k).astype(np.uint8)
        m = int(sizes.sum())
        x = np.arange(n, n + m, dtype=np.uint64)
        pid = x if dense else pkg.synth.mix64(x + np.uint64(9 << 40))
        prat = np.clip(np.repeat(rng.integers(0, 5001, k), sizes) + rng.integers(-20, 21, m), 0, 5000).astype(np.int32)
        pts = (now - rng.integers(0, 60, k)).astype(np.uint32)
        assert (e.enqueue_party(sizes, pid, prat, np.full(k, mode_idx, np.uint8), pts) == 1).all()
        book.add(pid, prat, np.repeat(pts, sizes))
        rules = {(mode_idx, g): (0, 10, 50, 5, 200) for g in range(cfg.n_groups)}
        lob, mem, st = e.party_match(now, rules_of(cfg, rules), lobby_cap=1 << 21, member_cap=1 << 24)
        assert st.n_lobbies > 10_000
        check_report(e, PM, restate_offtick(cfg, lob, mem, now, book))
        wait = eng_mod.wait_of(now, e.pool_read()["enq_ts"])
        min_wait = int(np.quantile(wait, 0.99))
        rules = {(mode_idx, g): (min_wait, 3, 50, 5, 400) for g in range(cfg.n_groups)}
        lob, mem, st = e.widen(now, rules_of(cfg, rules), lobby_cap=1 << 20, member_cap=1 << 23)
        assert st.n_lobbies > 1000
        check_report(e, WD, restate_offtick(cfg, lob, mem, now, book))
