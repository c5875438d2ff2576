"""Off-tick budget (mm_set_offtick_budget / mm_offtick_budget_report, include/mm_engine.h).

mm_party_match and mm_widen serve every queue on its own and in order, so a budgeted call is the unbudgeted call with
every queue's lobbies cut after its allowance a_q — the tick's apportionment of the budget over the queues' lobby
counts c_q.  The reference result of a budgeted call is therefore the existing restatement of the call (test_widen's
`restate`, test_parties' `restate_plain`) with each queue's lobby list cut, and the allowances come from the
pure-Python restatement of the apportionment in test_lobby_budget.
"""
import ctypes as C
import importlib
import json

import numpy as np
import pytest

from .fakes import FakeBroker
from .test_backfill import gpu_config, same, tick_same
from .test_lobby_budget import UNL, allowances, apportion_py
from .test_parties import PartySrc, party_rules, party_state, restate_plain as party_restate
from .test_party_backfill import strip_images
from .test_requeue import Src
from .test_widen import RATING, restate as widen_restate, rule_sets, rules_of

PARTY, WIDEN = 0, 1


# ---- reference: per-queue counts and the cut --------------------------------------------------------------------------
def queue_counts(cfg, queues):
    return np.bincount(np.asarray(queues, np.int64), minlength=cfg.n_modes * cfg.n_groups)


def clip_lists(cfg, lobbies, allot):
    """lobbies: [(queue, [member ids])] in header order -> the first allot[q] of every queue, in the same order."""
    seen = {}
    out = []
    for q, ms in lobbies:
        seen[q] = seen.get(q, 0) + 1
        if seen[q] <= allot[q]:
            out.append((q, ms))
    return out


def headers_of(cfg, lobbies):
    """[(queue, members)] -> [(mode, group, n_members, first_member)] as the engine writes them."""
    out, at = [], 0
    for q, ms in lobbies:
        out.append((q // cfg.n_groups, q % cfg.n_groups, len(ms), at))
        at += len(ms)
    return out


def engine_lists(cfg, lob, mem):
    return [(int(h["mode"]) * cfg.n_groups + int(h["group"]),
             [int(x) for x in mem[int(h["first_member"]):int(h["first_member"]) + int(h["n_members"])]]) for h in lob]


def widen_lists(cfg, pool, now, rules):
    lob, mem, n_anc, n_abs = widen_restate(cfg, pool["id"], pool["rating"], pool["mode"], pool["enq_ts"], now, rules)
    return [(m * cfg.n_groups + g, [int(x) for x in mem[f:f + n]]) for m, g, n, f in lob], n_anc, n_abs


def party_lists(cfg, pool, parties, now, rules):
    want, n_anc, n_abs, _ = party_restate(cfg, (pool["id"], pool["rating"], pool["mode"], pool["enq_ts"]), parties, now,
                                          rules)
    return [(m * cfg.n_groups + g, [int(x) for x in ms]) for m, g, ms in want], n_anc, n_abs


def budget_cases(cfg, cand, rng):
    """(name, per_queue, per_mode) cases over the unbudgeted counts `cand`."""
    G, M = cfg.n_groups, cfg.n_modes
    by_mode = [int(cand[m * G:(m + 1) * G].sum()) for m in range(M)]
    pq = np.array([int(rng.integers(0, c + 1)) if c else 0 for c in cand], np.int64)
    pq[rng.integers(0, len(pq), 3)] = UNL
    return [
        ("queue", pq, None),
        ("mode_binding", None, [max(0, b // 2 - 1) for b in by_mode]),
        ("mode_loose", None, [b + 3 for b in by_mode]),
        ("mode_zero", None, [0] + [UNL] * (M - 1)),
        ("both", pq, [max(0, b // 3) for b in by_mode]),
        ("unlimited", [UNL] * (M * G), [UNL] * M),
    ]


# ================================================================================ CPU
def test_allowance_restatement_equals_shard_apportion(pkg):
    shard = importlib.import_module("microservice-matchmaking_b200.shard")
    cfg = pkg.synth.make_config(n_groups=7, order=RATING, capacity=4096)
    rng = np.random.default_rng(3)
    G = cfg.n_groups
    for trial in range(200):
        cand = rng.integers(0, [2, 20, 5000][trial % 3], cfg.n_modes * G)
        pq = np.where(rng.random(len(cand)) < 0.3, UNL, rng.integers(0, 30, len(cand)))
        pm = [int(rng.integers(0, int(cand[m * G:(m + 1) * G].sum()) + 2)) for m in range(cfg.n_modes)]
        want = allowances(cfg, cand, pq, pm)
        got = np.concatenate([shard.apportion(pm[m], np.minimum(cand[m * G:(m + 1) * G], pq[m * G:(m + 1) * G]))
                              for m in range(cfg.n_modes)])
        assert got.tolist() == want.tolist()
        assert apportion_py(UNL, cand.tolist()) == cand.tolist()


def test_clip_keeps_each_queues_first_lobbies(pkg):
    cfg = pkg.synth.make_config(n_groups=3, order=RATING, capacity=4096)
    lobs = [(0, [1, 2]), (0, [3, 4]), (2, [5, 6]), (4, [7, 8]), (4, [9, 10]), (4, [11, 12])]
    allot = np.zeros(cfg.n_modes * 3, np.int64)
    allot[[0, 2, 4]] = [1, 0, 2]
    assert clip_lists(cfg, lobs, allot) == [(0, [1, 2]), (4, [7, 8]), (4, [9, 10])]
    assert headers_of(cfg, clip_lists(cfg, lobs, allot)) == [(0, 0, 2, 0), (1, 1, 2, 2), (1, 1, 2, 4)]


class StepEngine:
    """Engine double for one SearchPool step: party_match, the tick and widen could each form cand[source][q] lobbies
    of two queued players from the front of queue q; each emits the allowances of the budget it runs under and records
    that budget."""

    def __init__(self, cfg, cand):
        self.cfg, self.cand = cfg, {k: np.asarray(v, np.int64) for k, v in cand.items()}
        self.abi = importlib.import_module("microservice-matchmaking_b200.abi")
        self.queues = {}      # queue -> handles in enqueue order
        self.budget = {"tick": (None, None), "party_match": (None, None), "widen": (None, None)}
        self.report = {k: (np.zeros(len(v), np.int64),) * 2 for k, v in self.cand.items()}
        self.calls = []       # (source, per_queue, per_mode) each lobby-forming call ran under
        self.budget_sets = []

    def set_option(self, name, value):
        pass

    def enqueue(self, ids, rating, mode, enq_ts=None):
        oracle = importlib.import_module("oracle.oracle")
        for h, r, m in zip(np.asarray(ids).tolist(), np.asarray(rating).tolist(), np.asarray(mode).tolist()):
            g = oracle.find_rating_group(self.cfg, r)
            self.queues.setdefault(m * self.cfg.n_groups + g, []).append(h)
        return np.ones(len(ids), np.uint8)

    def set_lobby_budget(self, per_queue=None, per_mode=None):
        self._set("tick", per_queue, per_mode)

    def set_offtick_budget(self, source, per_queue=None, per_mode=None):
        self._set("party_match" if source == self.abi.MM_OFFTICK_PARTY_MATCH else "widen", per_queue, per_mode)

    def _set(self, name, per_queue, per_mode):
        b = (None if per_queue is None else [int(x) for x in per_queue],
             None if per_mode is None else [int(x) for x in per_mode])
        self.budget[name] = b
        self.budget_sets.append((name,) + b)

    def _form(self, name):
        pq, pm = self.budget[name]
        self.calls.append((name, pq, pm))
        cand = self.cand[name]
        allot = allowances(self.cfg, cand, pq, pm)
        self.report[name] = (cand, allot)
        lob, mem = [], []
        for q in range(len(cand)):
            for _ in range(int(allot[q])):
                take, self.queues[q] = self.queues[q][:2], self.queues[q][2:]
                lob.append((len(mem), 2, q // self.cfg.n_groups, q % self.cfg.n_groups))
                mem += take
        return np.array(lob, pkg_lobby_dtype()), np.array(mem, np.uint64)

    def party_match(self, now, rules):
        return self._form("party_match") + (None,)

    def tick(self, now=0):
        lob, mem = self._form("tick")
        return lob, mem, None, None

    def widen(self, now, rules):
        return self._form("widen") + (None,)

    def lobby_budget_report(self):
        return self.report["tick"]

    def offtick_budget_report(self, source):
        return self.report["party_match" if source == self.abi.MM_OFFTICK_PARTY_MATCH else "widen"]

    def pool_size(self):
        return sum(len(v) for v in self.queues.values())


def pkg_lobby_dtype():
    return importlib.import_module("microservice-matchmaking_b200.engine").LOBBY_DTYPE


def step_pool(pkg, budget_offtick, slots, cand):
    sw = importlib.import_module("microservice-matchmaking_b200.search_worker")
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=[("1v1", 2, 1), ("5v5", 2, 5)], order=RATING,
                                capacity=4096)
    names = list(pkg.synth.REFERENCE_GROUP_NAMES)
    eng = StepEngine(cfg, cand)
    broker = FakeBroker()
    pool = sw.SearchPool(eng, ["1v1", "5v5"], names, lobby_budget=(lambda: dict(slots)) if slots is not None else None,
                         widen={"1v1": (0, 10, 1, 1, 100)}, parties={"1v1": (0, 10, 1, 1, 100)},
                         budget_offtick=budget_offtick)
    workers = {g: sw.SearchWorker.start_link(broker, pool, {"group_name": g})[1] for g in names}
    for i in range(120):  # 60 bronze and 60 gold 1v1 players
        g, r = ("bronze", 100) if i % 2 == 0 else ("gold", 2100)
        broker.publish(sw.generate_exchange_name(g), sw.generate_queue_name(g),
                       json.dumps({"id": f"p{i}", "rating": r, "game-mode": "1v1"}))
    broker.deliver_all()
    return pool, eng, workers, broker, cfg, names


def cand_of(cfg, names, per):
    """{source: {group name: lobbies}} -> {source: u[n_cut]} for the 1v1 mode."""
    out = {}
    for src, d in per.items():
        c = np.zeros(cfg.n_modes * cfg.n_groups, np.int64)
        for g, n in d.items():
            c[names.index(g)] = n
        out[src] = c
    return out


def test_search_pool_step_shares_one_budget(pkg):
    names = list(pkg.synth.REFERENCE_GROUP_NAMES)
    per = {"party_match": {"bronze": 2, "gold": 2}, "tick": {"bronze": 4, "gold": 4}, "widen": {"bronze": 3, "gold": 3}}
    cfg0 = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=RATING, capacity=16)
    cand = cand_of(cfg0, names, per)
    pool, eng, workers, broker, cfg, names = step_pool(pkg, True, {"1v1": 9}, cand)
    assert pool.tick() == 9
    # F = 9: party_match under 9 (emits 4), the tick under 9 - 4 = 5, widen under 5 - 5 = 0
    assert [(c[0], c[2]) for c in eng.calls] == [("party_match", [9, UNL]), ("tick", [5, UNL]), ("widen", [0, UNL])]
    assert all(c[1] == [UNL] * (cfg.n_modes * cfg.n_groups) for c in eng.calls)
    hb = workers["bronze"].status()[1]["held_back"]
    assert hb["1v1"] == {"tick": 1, "party_match": 0, "widen": 3}  # tick: 5 over 4 : 4 gives bronze 3, gold 2
    assert workers["gold"].status()[1]["held_back"]["1v1"] == {"tick": 2, "party_match": 0, "widen": 3}
    assert pool.held_back("nowhere") == {}
    # a paused group publishes no party or widen lobby either
    pool.pause(["bronze"])
    assert pool.tick() == 9  # gold only: party 2, tick 4, widen 3 of F = 9
    b = names.index("bronze")
    for src, pq, pm in eng.calls[-3:]:
        assert pq[b] == 0 and pq[len(names) + b] == 0, src
    assert [c[2][0] for c in eng.calls[-3:]] == [9, 7, 3]
    assert workers["bronze"].status()[1]["held_back"]["1v1"] == {"tick": 4, "party_match": 2, "widen": 3}


def test_search_pool_pause_without_a_callable_sets_every_budget(pkg):
    names = list(pkg.synth.REFERENCE_GROUP_NAMES)
    cfg0 = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=RATING, capacity=16)
    cand = cand_of(cfg0, names, {s: {"bronze": 2, "gold": 2} for s in ("party_match", "tick", "widen")})
    pool, eng, workers, broker, cfg, names = step_pool(pkg, True, None, cand)
    pool.pause(["gold"], ["1v1"])
    assert sorted(s[0] for s in eng.budget_sets) == ["party_match", "tick", "widen"]  # at once, all three
    assert all(s[1][names.index("gold")] == 0 and s[2] is None for s in eng.budget_sets)
    assert pool.tick() == 6  # bronze's two of each source
    assert all(pq[names.index("gold")] == 0 for _s, pq, _pm in eng.calls)
    assert workers["gold"].status()[1]["held_back"]["1v1"] == {"tick": 2, "party_match": 2, "widen": 2}


def test_search_pool_without_the_flag_is_unchanged(pkg):
    names = list(pkg.synth.REFERENCE_GROUP_NAMES)
    cfg0 = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=RATING, capacity=16)
    cand = cand_of(cfg0, names, {"party_match": {"bronze": 2, "gold": 2}, "tick": {"bronze": 4, "gold": 4},
                                 "widen": {"bronze": 3, "gold": 3}})
    pool, eng, workers, broker, cfg, names = step_pool(pkg, False, {"1v1": 5}, cand)
    assert pool.tick() == 4 + 5 + 6  # only the tick is budgeted
    assert [(c[0], c[2]) for c in eng.calls] == [("party_match", None), ("tick", [5, UNL]), ("widen", None)]
    assert [s[0] for s in eng.budget_sets] == ["tick"]
    assert workers["bronze"].status()[1]["held_back"] == {"1v1": 1, "5v5": 0}
    pool.pause(["bronze"])
    assert [s[0] for s in eng.budget_sets] == ["tick"]  # the callable sets the tick's at the next step


def test_abi_mirror(pkg):
    abi = pkg.abi
    assert abi.MM_OFFTICK_PARTY_MATCH == PARTY and abi.MM_OFFTICK_WIDEN == WIDEN
    vp, u32 = C.c_void_p, C.c_uint32
    assert abi.PROTOTYPES["mm_set_offtick_budget"] == (C.c_int, [vp, u32, vp, vp])
    restype, args = abi.PROTOTYPES["mm_offtick_budget_report"]
    assert restype == C.c_int and args[:5] == [vp, u32, vp, vp, u32] and len(args) == 6


# ================================================================================ GPU
def raw_call(eng, source, now, rules, lobby_cap=0, member_cap=0):
    """The ABI call with explicit capacities -> (rc, stats)."""
    lob = np.zeros(max(lobby_cap, 1), pkg_lobby_dtype())
    mem = np.zeros(max(member_cap, 1), np.uint64)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    abi = importlib.import_module("microservice-matchmaking_b200.abi")
    if source == WIDEN:
        st = abi.WidenStats()
        rc = eng.lib.mm_widen(eng.h, int(now), p(rules), p(lob), lobby_cap, p(mem), member_cap, C.byref(st))
    else:
        st = abi.PartyStats()
        rc = eng.lib.mm_party_match(eng.h, int(now), p(rules), p(lob), lobby_cap, p(mem), member_cap, C.byref(st))
    return rc, st


def report(eng, source):
    cand, emitted = eng.offtick_budget_report(source)
    return cand.astype(np.int64), emitted.astype(np.int64)


def check_report_and_offtick(eng, cfg, source, cand, allot, lists):
    c, e = report(eng, source)
    assert c.tolist() == list(cand) and e.tolist() == list(allot)
    waits, quality, per_lobby = eng.offtick_report(source, want_lobbies=True)
    assert waits["n_lobbies"].astype(np.int64).tolist() == list(allot)
    assert len(per_lobby) == len(lists)
    assert quality["n_lobbies"].astype(np.int64).tolist() == list(allot)


def balance_mask(cfg):
    return sum(1 << m for m in range(cfg.n_modes) if cfg.modes[m].teams == 2 and cfg.modes[m].team_size <= 8)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
@pytest.mark.parametrize("layout", ["split", "wide", "overlap"])
@pytest.mark.parametrize("balance", [False, True], ids=["plain", "team_balance"])
def test_widen_budget_is_the_clipped_call(pkg, kind, layout, balance):
    cfg = gpu_config(pkg, RATING, kind, layout)
    src = Src(pkg, cfg, kind, seed=41)
    lo, hi = (-300, 5400) if layout == "overlap" else (0, 5001)
    rng = np.random.default_rng(7)
    engines = []

    def fresh_twin(img):
        t = pkg.Engine(cfg)
        engines.append(t)
        t.import_state(img)
        if balance:
            t.set_option("team_balance", balance_mask(cfg))
        return t

    try:
        src.enqueue(*src.fresh(40_000, lo, hi))
        src.eng.tick(src.now)
        src.enqueue(*src.fresh(30_000, lo, hi))
        img = src.eng.export_state()
        pool = src.eng.pool_read()
        for k, rules in enumerate(rule_sets(cfg)):
            now = src.now + 20 * k
            want, n_anc, n_abs = widen_lists(cfg, pool, now, rules)
            cand = queue_counts(cfg, [q for q, _ in want])
            free = fresh_twin(img)  # the unbudgeted twin
            lob0, mem0, st0 = free.widen(now, rules_of(cfg, rules))
            free_lists = engine_lists(cfg, lob0, mem0)
            if not balance:
                assert free_lists == want
            assert report(free, WIDEN)[0].tolist() == cand.tolist() == report(free, WIDEN)[1].tolist()
            for name, pq, pm in budget_cases(cfg, cand, rng) + [("cleared", None, None)]:
                eng = fresh_twin(img)
                if name == "cleared":
                    eng.set_offtick_budget(WIDEN, per_queue=[0] * len(cand), per_mode=[0] * cfg.n_modes)
                eng.set_offtick_budget(WIDEN, per_queue=pq, per_mode=pm)
                allot = allowances(cfg, cand, pq, pm)
                lob, mem, st = eng.widen(now, rules_of(cfg, rules))
                got = engine_lists(cfg, lob, mem)
                assert got == clip_lists(cfg, free_lists, allot), name
                if not balance:
                    assert got == clip_lists(cfg, want, allot), name
                assert [tuple(int(x) for x in (h["mode"], h["group"], h["n_members"], h["first_member"]))
                        for h in lob] == headers_of(cfg, got)
                assert (st.n_anchors, st.n_absorbed) == (n_anc, n_abs) == (st0.n_anchors, st0.n_absorbed)
                assert (st.n_lobbies, st.n_matched) == (len(got), sum(len(m) for _, m in got))
                if name in ("unlimited", "cleared", "mode_loose"):
                    assert np.array_equal(lob, lob0) and np.array_equal(mem, mem0), name
                check_report_and_offtick(eng, cfg, WIDEN, cand, allot, got)
                # EQUIVALENCE: mm_take of the returned ids
                twin = fresh_twin(img)
                assert twin.take(mem) == len(mem)
                sample = np.concatenate([pool["id"][::211], mem[::3]])
                same(eng, twin, now, sample)
                assert np.array_equal(eng.locate(sample, now), twin.locate(sample, now))
                eng.set_offtick_budget(WIDEN)
                nxt = {(m, g): (0, 30, 1, 3, 400) for m in range(cfg.n_modes) for g in range(cfg.n_groups)}
                ra, rb = eng.widen(now + 5, rules_of(cfg, nxt)), twin.widen(now + 5, rules_of(cfg, nxt))
                assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1])
                tick_same(eng, twin, now + 5)
                for e in (eng, twin):
                    engines.remove(e)
                    e.close()
            engines.remove(free)
            free.close()
    finally:
        for e in engines:
            e.close()
        src.close()


def party_twin(pkg, cfg, pimg, img, placed, solos, cap):
    pimg2, img2 = strip_images(pkg, pimg, img, placed)
    twin = pkg.Engine(cfg)
    twin.import_state(img2)
    twin.set_option("party_capacity", cap)
    assert (twin.merge_parties(pimg2, keep_seq=True) == 1).all()
    assert twin.take(solos) == len(solos)
    return twin


def same_parties(a, b):
    pa, pb = a.party_read(), b.party_read()
    for k in ("size", "seq", "enq_ts", "mode", "group", "rating"):
        assert np.array_equal(pa[k], pb[k]), k
    assert all(np.array_equal(x[0], y[0]) for x, y in zip(pa["members"], pb["members"]))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
@pytest.mark.parametrize("layout", ["split", "wide", "overlap"])
@pytest.mark.parametrize("balance", [False, True], ids=["plain", "party_balance"])
def test_party_match_budget_is_the_clipped_call(pkg, kind, layout, balance):
    cfg = gpu_config(pkg, RATING, kind, layout)
    lo, hi = (-300, 5400) if layout == "overlap" else (0, 5001)
    cap = 200_000
    src = PartySrc(pkg, cfg, kind, seed=23, cap=cap)
    rng = np.random.default_rng(9)
    engines = []
    try:
        src.enqueue(*src.fresh(30_000, lo, hi))
        sizes, ids, rat, mode, ts = src.fresh_parties(3000, lo, hi)
        assert (src.eng.enqueue_party(sizes, ids, rat, mode, ts) == 1).all()
        pimg = src.eng.export_parties()
        img = src.eng.export_state()
        in_party = set(int(x) for x in ids.tolist())

        def load():
            t = pkg.Engine(cfg)
            engines.append(t)
            t.import_state(img)
            t.set_option("party_capacity", cap)
            assert (t.merge_parties(pimg, keep_seq=True) == 1).all()
            if balance:
                t.set_option("party_balance", balance_mask(cfg))
            return t

        base = load()
        pool, parties = base.pool_read(), party_state(base)
        for k, rules in enumerate(party_rules(cfg)):
            now = src.now + 30 * k
            want, n_anc, n_abs = party_lists(cfg, pool, parties, now, rules)
            cand = queue_counts(cfg, [q for q, _ in want])
            free = load()
            lob0, mem0, st0 = free.party_match(now, rules_of(cfg, rules))
            free_lists = engine_lists(cfg, lob0, mem0)
            if not balance:
                assert free_lists == want
            for name, pq, pm in budget_cases(cfg, cand, rng) + [("cleared", None, None)]:
                eng = load()
                if name == "cleared":
                    eng.set_offtick_budget(PARTY, per_queue=[0] * len(cand), per_mode=[0] * cfg.n_modes)
                eng.set_offtick_budget(PARTY, per_queue=pq, per_mode=pm)
                allot = allowances(cfg, cand, pq, pm)
                lob, mem, st = eng.party_match(now, rules_of(cfg, rules))
                got = engine_lists(cfg, lob, mem)
                assert got == clip_lists(cfg, free_lists, allot), name
                if not balance:
                    assert got == clip_lists(cfg, want, allot), name
                assert [tuple(int(x) for x in (h["mode"], h["group"], h["n_members"], h["first_member"]))
                        for h in lob] == headers_of(cfg, got)
                flat = [x for _, ms in got for x in ms]
                placed = np.array([x for x in flat if x in in_party], np.uint64)
                solos = np.array([x for x in flat if x not in in_party], np.uint64)
                placed_set = set(placed.tolist())
                n_parties = sum(1 for p in parties if int(p[0][0]) in placed_set)
                assert (st.n_anchors, st.n_absorbed) == (n_anc, n_abs) == (st0.n_anchors, st0.n_absorbed)
                assert (st.n_lobbies, st.n_matched, st.n_parties) == (len(got), len(flat), n_parties)
                if name in ("unlimited", "cleared", "mode_loose"):
                    assert np.array_equal(lob, lob0) and np.array_equal(mem, mem0), name
                    assert st.sum_imbalance == st0.sum_imbalance
                check_report_and_offtick(eng, cfg, PARTY, cand, allot, got)
                # EQUIVALENCE: the party construction with only the emitted lobbies
                twin = party_twin(pkg, cfg, pimg, img, placed, solos, cap)
                engines.append(twin)
                if balance:
                    twin.set_option("party_balance", balance_mask(cfg))
                sample = np.concatenate([pool["id"][::173], np.array(flat[::3], np.uint64), ids[::11]])
                same(eng, twin, now, sample)
                same_parties(eng, twin)
                assert eng.seq_next() == twin.seq_next()
                eng.set_offtick_budget(PARTY)
                nxt = {(m, g): (0, 40, 1, 5, 600) for m in range(cfg.n_modes) for g in range(cfg.n_groups)}
                ra, rb = eng.party_match(now + 5, rules_of(cfg, nxt)), twin.party_match(now + 5, rules_of(cfg, nxt))
                assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1])
                wa, wb = eng.widen(now + 5, rules_of(cfg, nxt)), twin.widen(now + 5, rules_of(cfg, nxt))
                assert np.array_equal(wa[0], wb[0]) and np.array_equal(wa[1], wb[1])
                tick_same(eng, twin, now + 5)
                for e in (eng, twin):
                    engines.remove(e)
                    e.close()
            engines.remove(free)
            free.close()
    finally:
        for e in engines:
            e.close()
        src.close()


@pytest.mark.gpu
@pytest.mark.parametrize("source", [PARTY, WIDEN], ids=["party_match", "widen"])
def test_report_dry_run_refusals_and_independence(pkg, source):
    cfg = gpu_config(pkg, RATING, "hashed", "split")
    src = PartySrc(pkg, cfg, "hashed", seed=61)
    eng = src.eng
    try:
        n_cut = cfg.n_modes * cfg.n_groups
        assert report(eng, source)[0].tolist() == [0] * n_cut  # before the first call
        src.enqueue(*src.fresh(30_000))
        if source == PARTY:
            assert (eng.enqueue_party(*src.fresh_parties(2000)) == 1).all()
            rules = party_rules(cfg)[0]
        else:
            rules = rule_sets(cfg)[0]
        r = rules_of(cfg, rules)
        before = (eng.pool_read(), eng.active_size())
        eng.set_offtick_budget(source, per_mode=[1] * cfg.n_modes)
        rc, st = raw_call(eng, source, src.now, r)  # a dry run: c_q and a_q, nothing changes
        assert rc == pkg.abi.MM_E_CAP
        cand, emitted = report(eng, source)
        assert cand.sum() > emitted.sum() and emitted.tolist() == allowances(cfg, cand, None, [1] * cfg.n_modes).tolist()
        assert st.n_lobbies == emitted.sum()
        after = (eng.pool_read(), eng.active_size())
        assert all(np.array_equal(before[0][k], after[0][k]) for k in before[0]) and before[1] == after[1]
        waits, _q, _l = eng.offtick_report(source)
        assert len(waits) == 0  # mm_offtick_report is void after MM_E_CAP
        # a refusal: zeros
        bad = r.copy()
        bad["step"][0], bad["min_wait"][0] = 0, 0
        assert raw_call(eng, source, src.now, bad)[0] == pkg.abi.MM_E_ARG
        assert report(eng, source)[0].tolist() == [0] * n_cut and report(eng, source)[1].tolist() == [0] * n_cut
        # the tick's budget and the other source's leave this one alone, and the reverse
        other = WIDEN if source == PARTY else PARTY
        eng.set_lobby_budget(per_mode=[0] * cfg.n_modes)
        eng.set_offtick_budget(other, per_mode=[0] * cfg.n_modes)
        lob, mem, st = (eng.party_match if source == PARTY else eng.widen)(src.now, r)
        cand, emitted = report(eng, source)
        assert emitted.tolist() == allowances(cfg, cand, None, [1] * cfg.n_modes).tolist()
        assert len(lob) == emitted.sum() > 0 and cand.sum() > len(lob)
        t = eng.tick(src.now)
        assert len(t[0]) == 0  # the tick keeps its own budget
        tc, te = eng.lobby_budget_report()
        assert te.sum() == 0 and tc.sum() > 0
        assert report(eng, source)[1].tolist() == emitted.tolist()  # the tick leaves the source's report alone
        # refusals of the two calls
        n = C.c_uint32(0)
        buf = np.zeros(n_cut, np.uint32)
        p = buf.ctypes.data_as(C.c_void_p)
        lib = eng.lib
        assert lib.mm_set_offtick_budget(None, source, None, None) == pkg.abi.MM_E_ARG
        assert lib.mm_set_offtick_budget(eng.h, 2, None, None) == pkg.abi.MM_E_ARG
        assert lib.mm_offtick_budget_report(None, source, p, p, n_cut, C.byref(n)) == pkg.abi.MM_E_ARG
        assert lib.mm_offtick_budget_report(eng.h, source, p, p, n_cut, None) == pkg.abi.MM_E_ARG
        assert lib.mm_offtick_budget_report(eng.h, 2, p, p, n_cut, C.byref(n)) == pkg.abi.MM_E_ARG
        assert lib.mm_offtick_budget_report(eng.h, source, None, None, n_cut, C.byref(n)) == pkg.abi.MM_E_ARG
        assert lib.mm_offtick_budget_report(eng.h, source, p, p, n_cut - 1, C.byref(n)) == pkg.abi.MM_E_CAP
        assert n.value == n_cut
        assert lib.mm_offtick_budget_report(eng.h, source, None, None, 0, C.byref(n)) == pkg.abi.MM_E_CAP
    finally:
        src.close()
    # a staged packed batch (an MM_F_DENSE_IDS engine)
    cfg = gpu_config(pkg, RATING, "dense", "split")
    with pkg.Engine(cfg) as e:
        h = np.arange(100, 110, dtype=np.uint32)
        k = np.zeros(10, np.uint16)
        assert e.lib.mm_enqueue_packed_begin(e.h, 10, h.ctypes.data_as(C.c_void_p), k.ctypes.data_as(C.c_void_p),
                                             None) == 0
        n = C.c_uint32(0)
        buf = np.zeros(cfg.n_modes * cfg.n_groups, np.uint32)
        p = buf.ctypes.data_as(C.c_void_p)
        assert e.lib.mm_offtick_budget_report(e.h, source, p, p, len(buf), C.byref(n)) == pkg.abi.MM_E_STATE
        assert "staged" in e.lib.mm_last_error(e.h).decode()
        assert e.lib.mm_enqueue_packed_end(e.h, None, None) == 0
        assert e.lib.mm_offtick_budget_report(e.h, source, p, p, len(buf), C.byref(n)) == 0


@pytest.mark.gpu
def test_widen_budget_survives_snapshot_and_is_absent_after_import(pkg):
    cfg = gpu_config(pkg, RATING, "hashed", "split")
    src = Src(pkg, cfg, "hashed", seed=71)
    other = None
    try:
        src.enqueue(*src.fresh(40_000))
        rules = rules_of(cfg, rule_sets(cfg)[0])
        src.eng.set_offtick_budget(WIDEN, per_mode=[2] * cfg.n_modes)
        src.eng.snapshot()
        src.eng.restore()
        lob, mem, st = src.eng.widen(src.now, rules)
        cand, emitted = report(src.eng, WIDEN)
        assert emitted.sum() == len(lob) == 2 * cfg.n_modes and cand.sum() > len(lob)
        other = pkg.Engine(cfg)
        other.import_state(src.eng.export_state())
        lob, mem, st = other.widen(src.now, rules)
        cand, emitted = report(other, WIDEN)
        assert cand.tolist() == emitted.tolist() and len(lob) == emitted.sum() > 2 * cfg.n_modes
    finally:
        if other is not None:
            other.close()
        src.close()


@pytest.mark.gpu
def test_config3_ten_million_with_parties_binding_mode_budgets(pkg):
    cfg = pkg.synth.make_config(n_groups=32, modes=[("5v5", 2, 5)], order=RATING, capacity=10_500_000,
                                active_capacity=12_000_000)
    rng = np.random.default_rng(4)
    n = 10_000_000
    ids = np.arange(n, dtype=np.uint64) + np.uint64(1 << 40)
    rating = rng.integers(0, 5001, n).astype(np.int32)
    ts = (100_000 - rng.integers(0, 60_000, n)).astype(np.uint32)
    k = 100_000
    sizes = rng.integers(2, 5, k).astype(np.uint8)
    m = int(sizes.sum())
    pid = np.arange(m, dtype=np.uint64) + np.uint64(1 << 41)
    prat = np.clip(np.repeat(rng.integers(0, 5001, k), sizes) + rng.integers(-30, 31, m), 0, 5000).astype(np.int32)
    pts = (100_000 - rng.integers(0, 60_000, k)).astype(np.uint32)
    rules = {"party_match": {(0, g): (0, 30, 100, 5, 300) for g in range(cfg.n_groups)},
             "widen": {(0, g): (59_000, 20, 100, 5, 400) for g in range(cfg.n_groups)}}

    def build():
        e = pkg.Engine(cfg)
        e.set_option("party_capacity", 1_000_000)
        assert e.enqueue(ids, rating, np.zeros(n, np.uint8), ts).all()
        assert (e.enqueue_party(sizes, pid, prat, np.zeros(k, np.uint8), pts) == 1).all()
        return e

    for source, call in ((PARTY, "party_match"), (WIDEN, "widen")):
        with build() as b:  # the unbudgeted twin
            lob0, mem0, _ = getattr(b, call)(100_000, rules_of(cfg, rules[call]))
        free = engine_lists(cfg, lob0, mem0)
        cand = queue_counts(cfg, [q for q, _ in free])
        B = int(cand.sum()) // 3
        allot = allowances(cfg, cand, None, [B])
        with build() as a:
            a.set_offtick_budget(source, per_mode=[B])
            lob, mem, st = getattr(a, call)(100_000, rules_of(cfg, rules[call]))
            assert engine_lists(cfg, lob, mem) == clip_lists(cfg, free, allot)
            assert len(lob) == B > 0 and (allot < cand).any()
            assert report(a, source)[0].tolist() == cand.tolist() and report(a, source)[1].tolist() == allot.tolist()
