"""Party search status (mm_party_queue_stats / mm_party_locate / Engine.party_queue_stats / Engine.party_locate /
SearchPool.party_search_status / party_queue_status): the waiting section of mm_queue_stats for queued parties, and one
party member's place and the lobby the next mm_party_match gives it, answered on the device.

CPU: a plain restatement of the per-queue records and of every member's status (one party at a time, on test_parties'
plain restatement of mm_party_match) held equal to a numpy one (on the binned restatement) on random tables, with the
off-tick budget (test_lobby_budget's allowances) and party_balance (test_party_balance's split); the ABI mirror;
SearchPool.party_search_status, party_queue_status, party_status and SearchWorker.status()["party_waiting"] with an
engine double.
GPU: the records against the restatement of party_read through a schedule with dead rows, requeues, a KEEP_SEQ merge
behind released rows, a default-group fallback, stamps in the future and across the 2^32 wrap and parties of 16;
every prediction against the real next party_match (absorbed anchors, all-or-nothing failures, MM_WIDEN_OFF queues,
modes of 3, 40 and 256 teams, party_balance, binding and loose budgets per queue and per mode, both id kinds and wide
partitions); no side effects (twin engines); every refusal; config3 with 200 k parties.
"""
import ctypes as C
import importlib

import numpy as np
import pytest

from .test_backfill import clamp_bounds, gpu_config, group_of
from .test_expire import r_wait
from .test_lobby_budget import UNL, allowances
from .test_parties import PartySrc, party_engine, party_rating, party_state, restate_bins, restate_plain
from .test_party_balance import balance_parties
from .test_widen import RATING, ARRIVAL, rules_of, wait_of, window

STAYS = 0xFFFFFFFF
OFF = 0xFFFFFFFF
PARTY = 0  # MM_OFFTICK_PARTY_MATCH


# ================================================================================ restatements
def bucket_plain(w):
    if w < 8:
        return w
    e = w.bit_length() - 1
    return 8 + 4 * (e - 3) + ((w >> (e - 2)) & 3)


def stats_plain(cfg, parties, now):
    """The records, one party at a time.  parties: [(ids, ratings, mode, ts)] of the queued parties (party_state).
    -> {queue: (n_parties, n_members, max_wait, wait_hist list, size_hist list)} for every queue"""
    nq = cfg.n_modes * cfg.n_groups
    out = {q: [0, 0, 0, [0] * 120, [0] * 16] for q in range(nq)}
    for ids, rat, m, ts in parties:
        q = int(m) * cfg.n_groups + group_of(cfg, party_rating(rat))
        w = wait_of(now, ts)
        r = out[q]
        r[0] += 1
        r[1] += len(ids)
        r[2] = max(r[2], w)
        r[3][bucket_plain(w)] += 1
        r[4][min(len(ids), 15)] += 1
    return {q: (a, b, c, list(d), list(e)) for q, (a, b, c, d, e) in out.items()}


def stats_numpy(pkg, cfg, size, mode, group, ts, now):
    """The same from party_read's columns -> PARTY_QUEUE_STAT_DTYPE[n_modes * n_groups]"""
    nq = cfg.n_modes * cfg.n_groups
    q = np.asarray(mode, np.int64) * cfg.n_groups + np.asarray(group, np.int64)
    w = r_wait(now, np.asarray(ts, np.uint32))
    s = np.asarray(size, np.int64)
    out = np.zeros(nq, pkg.engine.PARTY_QUEUE_STAT_DTYPE)
    out["mode"], out["group"] = np.arange(nq) // cfg.n_groups, np.arange(nq) % cfg.n_groups
    out["n_parties"] = np.bincount(q, minlength=nq)
    out["n_members"] = np.bincount(q, s, minlength=nq).astype(np.int64)
    mx = np.zeros(nq, np.int64)
    np.maximum.at(mx, q, w)
    out["max_wait"] = mx
    np.add.at(out["wait_hist"], (q, pkg.engine.wait_bucket(w) if len(w) else np.zeros(0, np.int64)), 1)
    np.add.at(out["size_hist"], (q, np.minimum(s, 15)), 1)
    return out


def as_records(pkg, cfg, plain):
    nq = cfg.n_modes * cfg.n_groups
    out = np.zeros(nq, pkg.engine.PARTY_QUEUE_STAT_DTYPE)
    for q, (n, m, mx, wh, sh) in plain.items():
        out[q] = (q // cfg.n_groups, q % cfg.n_groups, 0, n, m, mx, wh, sh)
    return out


def locate_restate(cfg, solos, parties, now, rules, restate, per_queue=None, per_mode=None, mask=0):
    """Every queued member's status from a restatement of the next party_match (restate_plain or restate_bins).
    solos: (ids, rating, mode, ts) as restate takes them; parties: party_state's list in age order; rules: the dict.
    -> {member id: (queue, index, size, ahead, depth, anchor, window, lobby, member)}"""
    G = cfg.n_groups
    want = restate(cfg, solos, parties, now, rules)[0]
    lists = [(m * G + g, [int(x) for x in ms]) for m, g, ms in want]
    if mask:  # party_balance: each lobby of a masked mode split as the option splits it
        lob = np.zeros(len(lists), [("first_member", "<u4"), ("n_members", "<u2"), ("mode", "u1"), ("group", "u1")])
        at = 0
        for k, (q, ms) in enumerate(lists):
            lob[k] = (at, len(ms), q // G, q % G)
            at += len(ms)
        own = {int(x): int(r) for ps in parties for x, r in zip(ps[0], ps[1])}
        own.update({int(x): int(r) for x, r in zip(solos[0], solos[1])})
        key = {int(x): j for j, ps in enumerate(parties) for x in ps[0]}
        mem, _ = balance_parties(cfg, mask, lob, [x for _, ms in lists for x in ms], own.__getitem__, key.get)
        lists = [(q, [int(x) for x in mem[int(h["first_member"]):int(h["first_member"]) + len(ms)]])
                 for h, (q, ms) in zip(lob, lists)]
    cand = np.bincount([q for q, _ in lists], minlength=cfg.n_modes * G)
    allot = allowances(cfg, cand, per_queue, per_mode) if per_queue is not None or per_mode is not None else cand
    placed, seen = {}, {}
    for q, ms in lists:
        k = seen.get(q, 0)
        seen[q] = k + 1
        if k < allot[q]:
            placed.update((x, (k, i)) for i, x in enumerate(ms))
    out, count = {}, {}
    qs = [int(p[2]) * G + group_of(cfg, party_rating(p[1])) for p in parties]
    depth = np.bincount(qs, minlength=cfg.n_modes * G)
    for (ids, _rat, _m, ts), q in zip(parties, qs):
        ahead = count.get(q, 0)
        count[q] = ahead + 1
        rule = rules.get((q // G, q % G))
        w = wait_of(now, ts)
        anchor = rule is not None and w >= rule[0]
        win = window(rule, w) if anchor else -1
        for i, x in enumerate(ids):
            lobby, member = placed.get(int(x), (STAYS, 0xFFFF))
            out[int(x)] = (q, i, len(ids), ahead, int(depth[q]), int(anchor), win, lobby, member)
    return out


def random_table(rng, cfg, n_parties, n_solos, now):
    """Random solos and parties (age order) -> (solos tuple, parties list)"""
    lo, hi = clamp_bounds(cfg)
    sid = np.arange(10_000, 10_000 + n_solos, dtype=np.uint64)
    srat = rng.integers(lo - 20, hi + 20, n_solos)
    smode = rng.integers(0, cfg.n_modes, n_solos)
    keep = np.array([group_of(cfg, int(r)) >= 0 for r in srat], bool)
    solos = (sid[keep], srat[keep], smode[keep], np.full(int(keep.sum()), now - 5))
    parties, nxt = [], 0
    while len(parties) < n_parties:
        m = int(rng.integers(0, cfg.n_modes))
        S = cfg.modes[m].team_size
        if S < 2:
            continue
        s = int(rng.integers(2, S + 1))
        base = int(rng.integers(lo, hi))
        rat = [base + int(d) for d in rng.integers(-15, 16, s)]
        if group_of(cfg, party_rating(rat)) < 0:
            continue
        parties.append((list(range(nxt, nxt + s)), rat, m, int(now - rng.integers(0, 60))))
        nxt += s
    return solos, parties


# ================================================================================ CPU
@pytest.mark.parametrize("seed", range(6))
def test_stats_restatements_agree(pkg, seed):
    rng = np.random.default_rng(seed)
    groups = [[(0, 99), (100, 299)], [(0, 200), (50, 120), (0, 400)], [(10, 60)]][seed % 3]
    modes = [("a", 2, 16), ("b", 3, 2), ("c", 2, 5)]
    cfg = pkg.synth.make_config(groups=groups, modes=modes, order=RATING, capacity=4096,
                                default_group=len(groups) - 1 if seed % 2 else -1)
    now = [1000, 5, (1 << 32) - 3][seed % 3]
    _solos, parties = random_table(rng, cfg, 300, 0, now)
    parties = [(ids, rat, m, (ts + int(rng.integers(-3, 3))) & 0xFFFFFFFF) for ids, rat, m, ts in parties]
    plain = as_records(pkg, cfg, stats_plain(cfg, parties, now))
    R = [party_rating(p[1]) for p in parties]
    got = stats_numpy(pkg, cfg, [len(p[0]) for p in parties], [p[2] for p in parties],
                      [group_of(cfg, r) for r in R], [p[3] for p in parties], now)
    assert plain.tobytes() == got.tobytes()
    assert got["size_hist"][:, :2].sum() == 0 and got["n_parties"].sum() == len(parties)
    assert got["size_hist"][:, 15].sum() == sum(len(p[0]) >= 15 for p in parties)


@pytest.mark.parametrize("seed", range(6))
def test_locate_restatements_agree(pkg, seed):
    rng = np.random.default_rng(100 + seed)
    modes = [("5v5", 2, 5), ("duo3", 3, 2), ("4v4", 2, 4)]
    cfg = pkg.synth.make_config(groups=[(0, 300), (301, 600)], modes=modes, order=RATING, capacity=4096,
                                default_group=-1)
    now = 1000
    solos, parties = random_table(rng, cfg, 60, 250, now)
    G = cfg.n_groups
    rules = {(m, g): (int(rng.integers(0, 40)), int(rng.integers(0, 30)), int(rng.integers(1, 9)),
                      int(rng.integers(0, 6)), 60) for m in range(cfg.n_modes) for g in range(G) if (m + g + seed) % 4}
    per_queue = per_mode = None
    if seed % 3 == 1:
        per_queue = rng.integers(0, 3, cfg.n_modes * G)
    elif seed % 3 == 2:
        per_mode = [1, UNL, 2]
    mask = 0b101 if seed % 2 else 0
    a = locate_restate(cfg, solos, parties, now, rules, restate_plain, per_queue, per_mode, mask)
    b = locate_restate(cfg, solos, parties, now, rules, restate_bins, per_queue, per_mode, mask)
    assert a == b
    assert len(a) == sum(len(p[0]) for p in parties)
    placed = [v for v in a.values() if v[7] != STAYS]
    if seed == 0:
        assert placed and len(placed) < len(a)
    for x, v in a.items():  # a party is placed whole, in one lobby
        mates = [a[y] for p in parties if x in p[0] for y in p[0]]
        assert len({(m[7]) for m in mates}) == 1


def test_abi_mirror(pkg):
    abi, eng = pkg.abi, pkg.engine
    assert C.sizeof(abi.PartyQueueStat) == 560 and C.sizeof(abi.PartyMemberStatus) == 48
    for dt, st in ((eng.PARTY_QUEUE_STAT_DTYPE, abi.PartyQueueStat), (eng.PARTY_MEMBER_STATUS_DTYPE,
                                                                       abi.PartyMemberStatus)):
        for name, *_ in st._fields_:
            assert dt.fields[name][1] == getattr(st, name).offset, name
    assert abi.PartyMemberStatus.window.offset == 28 and abi.PartyQueueStat.size_hist.offset == 496
    for name in ("mm_party_queue_stats", "mm_party_locate"):
        assert name in abi.PROTOTYPES


def status_engine(pkg, calls):
    class StatusEngine(party_engine(pkg, calls)):
        """party_engine's double with the two status calls, answered by the restatements."""

        def queue_stats(self, now=0):  # SearchWorker.status() reads it beside the party records
            return np.zeros(0, pkg.engine.QUEUE_STAT_DTYPE)

        def party_queue_stats(self, now=0):
            return as_records(pkg, self.cfg, stats_plain(self.cfg, self.parties, now))

        def party_locate(self, ids, now, rules):
            calls.append("party_locate")
            p = self.pool_read()
            ts = [self.ts[int(x)] for x in p["id"]]
            st = locate_restate(self.cfg, (p["id"], p["rating"], p["mode"], ts), self.parties, now, rules,
                                restate_plain)
            out = np.zeros(len(ids), pkg.engine.PARTY_MEMBER_STATUS_DTYPE)
            out["window"], out["lobby"], out["member"] = -1, STAYS, 0xFFFF
            solo = set(p["id"].tolist())
            for k, x in enumerate(np.asarray(ids).tolist()):
                if x in st:
                    q, i, s, ahead, depth, anchor, win, lobby, member = st[x]
                    out[k]["state"], out[k]["mode"], out[k]["group"], out[k]["size"], out[k]["index"] = \
                        3, q // self.cfg.n_groups, q % self.cfg.n_groups, s, i
                    ts_ = next(pp[3] for pp in self.parties if x in pp[0])
                    out[k]["anchor"], out[k]["window"], out[k]["ahead"], out[k]["depth"] = anchor, win, ahead, depth
                    out[k]["wait"], out[k]["lobby"], out[k]["member"] = wait_of(now, ts_), lobby, member
                elif x in self.active:
                    out[k]["state"] = 1 if x in solo else 2
            return out

    return StatusEngine


def test_search_pool_party_status_calls(pkg):
    sw = importlib.import_module("microservice-matchmaking_b200.search_worker")
    from .fakes import FakeBroker
    from .test_expire import publish
    from .test_handover import start_workers
    from .test_parties import publish_party
    calls = []
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=RATING, capacity=1000, active_capacity=4000)
    eng = status_engine(pkg, calls)(cfg)
    clock = [0.0]
    pool = sw.SearchPool(eng, ["1v1", "5v5"], list(pkg.synth.REFERENCE_GROUP_NAMES), flush_every_s=3600,
                         clock=lambda: clock[0], parties={"5v5": (0, 50, 1000, 0, 50)}, party_capacity=100)
    broker = FakeBroker()
    start_workers(sw, broker, pool, pkg)
    for i in range(6):
        publish(pkg, broker, cfg, f"s{i}", 100 + i, mode="5v5")
    publish_party(pkg, broker, sw, "bronze", [(f"a{i}", 100 + i) for i in range(3)], "5v5")
    publish_party(pkg, broker, sw, "bronze", [(f"b{i}", 110 - i) for i in range(2)], "5v5")
    publish_party(pkg, broker, sw, "bronze", [("c0", 4000), ("c1", 4010)], "5v5")
    broker.deliver_all()
    st = pool.party_search_status(["a1", "zz"])
    assert st[0]["state"] == "staged" and st[0]["game_mode"] == "5v5" and st[0]["group"] == "bronze"
    assert st[0]["party_size"] == 3 and st[1]["state"] == "unknown" and st[1]["next_match"] is None
    pool.flush()
    clock[0] = 0.25
    st = pool.party_search_status(["a1", "b0", "c1", "s0", "zz"])
    assert calls[-1] == "party_locate"
    a1, b0, c1, s0, zz = st
    assert a1["state"] == "searching" and a1["game_mode"] == "5v5" and a1["group"] == "bronze"
    assert (a1["party_size"], a1["position"], a1["queue_size"], a1["wait_ms"]) == (3, 0, 2, 250)
    assert a1["anchor"] is True and a1["window"] == 50
    assert a1["next_match"] == {"lobby": 0, "team": 0} and b0["next_match"] == {"lobby": 0, "team": 0}
    assert b0["position"] == 1 and c1["group"] != "bronze" and c1["next_match"] is None and c1["position"] == 0
    assert s0["state"] == "unknown" and zz["state"] == "unknown"  # a queued solo: search_status answers it
    want = {"5v5": {"parties": 2, "players": 5}}
    assert pool.party_status("bronze") == want
    eng_read_only = pool.engine.party_queue_stats
    del type(eng).party_queue_stats  # the same dict from party_read
    try:
        assert not hasattr(pool.engine, "party_queue_stats") and pool.party_status("bronze") == want
    finally:
        type(eng).party_queue_stats = eng_read_only.__func__
    q = pool.party_queue_status("bronze")
    assert q["5v5"]["parties"] == 2 and q["5v5"]["players"] == 5 and q["5v5"]["sizes"] == {2: 1, 3: 1}
    assert q["5v5"]["oldest_wait_ms"] == 250 and q["5v5"]["p99_wait_ms"] >= 250 and q["1v1"]["parties"] == 0
    assert pool.party_queue_status("nope") == {}
    status = pool.workers["bronze"].status()[1]
    assert status["party_waiting"] == q and status["parties"] == want
    pool.tick()
    st = pool.party_search_status(["a1", "c1"])
    assert st[0]["state"] == "matched" and st[1]["state"] == "searching"


# ================================================================================ GPU
def member_cols(parties):
    return np.array([x for p in parties for x in p[0]], np.uint64)


def actual_places(cfg, lob, mem):
    """party_match's output -> {member id: (queue, ordinal inside the queue, index inside the lobby)}"""
    out, seen = {}, {}
    for h in lob:
        q = int(h["mode"]) * cfg.n_groups + int(h["group"])
        k = seen.get(q, 0)
        seen[q] = k + 1
        f = int(h["first_member"])
        for i, x in enumerate(mem[f:f + int(h["n_members"])].tolist()):
            out[int(x)] = (q, k, i)
    return out


def check_stats(pkg, eng, cfg, now):
    pr = eng.party_read()
    want = stats_numpy(pkg, cfg, pr["size"], pr["mode"], pr["group"], pr["enq_ts"], now)
    got = eng.party_queue_stats(now)
    assert got.tobytes() == want.tobytes()
    assert got.tobytes() == as_records(pkg, cfg, stats_plain(cfg, party_state(eng), now)).tobytes()
    return got


def check_prediction(pkg, eng, cfg, now, rules, extra_ids=()):
    """party_locate of every queued member (and extra ids), then the real party_match: every prediction holds.
    -> (records, the party_match result)"""
    parties = party_state(eng)
    ids = np.concatenate([member_cols(parties), np.asarray(extra_ids, np.uint64)])
    rec = eng.party_locate(ids, now, rules)
    want = locate_restate(cfg, (np.zeros(0, np.uint64),) * 4, parties, now, rules, restate_plain)
    G = cfg.n_groups
    for x, r in zip(ids[:len(ids) - len(extra_ids)].tolist(), rec):
        q, i, s, ahead, depth, anchor, win, _lob, _mem = want[x]
        assert int(r["state"]) == 3
        assert (int(r["mode"]) * G + int(r["group"]), int(r["index"]), int(r["size"]), int(r["ahead"]),
                int(r["depth"]), int(r["anchor"]), int(r["window"])) == (q, i, s, ahead, depth, anchor, win), x
    pr = eng.party_read()
    res = eng.party_match(now, rules, lobby_cap=1 << 16, member_cap=1 << 22)
    got = actual_places(cfg, res[0], res[1])
    n_placed = 0
    for x, r in zip(ids[:len(ids) - len(extra_ids)].tolist(), rec):
        if int(r["lobby"]) == STAYS:
            assert x not in got and int(r["member"]) == 0xFFFF, x
        else:
            n_placed += 1
            assert got[x] == (int(r["mode"]) * G + int(r["group"]), int(r["lobby"]), int(r["member"])), x
    assert n_placed == sum(1 for x in got if x in set(member_cols(parties).tolist()))
    assert len(pr["size"]) == len(parties)
    return rec, res


def status_config(pkg, kind, layout, modes=None, capacity=200_000):
    cfg = gpu_config(pkg, RATING, kind, layout, capacity=capacity)
    if modes:
        cfg.n_modes = len(modes)
        for m, (_n, t, s) in enumerate(modes):
            cfg.modes[m].teams, cfg.modes[m].team_size = t, s
    return cfg


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
@pytest.mark.parametrize("layout", ["split", "wide", "overlap"])
def test_stats_equal_the_restatement_over_a_schedule(pkg, kind, layout):
    cfg = status_config(pkg, kind, layout, modes=[("16a", 2, 16), ("duo3", 3, 2), ("5v5", 2, 5)])
    src = PartySrc(pkg, cfg, kind, seed=11)
    eng = src.eng
    rules = {(m, g): (0, 10, 5, 5, 80) for m in range(cfg.n_modes) for g in range(cfg.n_groups)}
    try:
        for step in range(10):
            now = src.now
            sizes, ids, rat, mode, ts = src.fresh_parties(400)
            big = sizes.copy()
            big[::7] = np.where(mode[::7] == 0, 16, sizes[::7])  # parties of 16 in the 16-a-side mode
            if (big != sizes).any():
                ids2, rat2, off = [], [], 0
                for s0, s1 in zip(sizes.tolist(), big.tolist()):
                    x, r, _m, _t = src.fresh(s1)
                    ids2.append(x); rat2.append(np.full(s1, int(rat[off]), np.int32))
                    off += s0
                sizes, ids, rat = big.astype(np.uint8), np.concatenate(ids2), np.concatenate(rat2)
            ts = ts.copy()
            ts[::5] = (now + 7) & 0xFFFFFFFF  # in the future
            assert (eng.enqueue_party(sizes, ids, rat, mode, ts) == 1).all()
            src.enqueue(*src.fresh(3000))
            check_stats(pkg, eng, cfg, now)
            pr = eng.party_read()
            op = step % 5
            if op == 0:  # removed and expired parties leave dead rows
                eng.remove(np.array([m[0][0] for m in pr["members"][::6]], np.uint64))
                eng.expire(now, 55)
            elif op == 1:  # matched parties: dead rows, then requeued ones back at their age
                lob, mem, _st = eng.party_match(now, rules, lobby_cap=1 << 14, member_cap=1 << 20)
                check_stats(pkg, eng, cfg, now)
                pset = {int(x): k for k, ms in enumerate(pr["members"]) for x in ms[0]}
                back = sorted({pset[int(x)] for x in mem if int(x) in pset})[::3]
                if back:
                    eng.requeue_party(pr["size"][back], np.concatenate([pr["members"][k][0] for k in back]),
                                      np.concatenate([pr["members"][k][1] for k in back]), pr["mode"][back],
                                      pr["enq_ts"][back], pr["seq"][back])
            elif op == 2:  # exported parties, merged back with their numbers behind the released rows
                img = eng.export_parties()
                check_stats(pkg, eng, cfg, now)
                assert (eng.merge_parties(img, keep_seq=True) == 1).all()
            elif op == 3:  # the clock across the 2^32 wrap
                src.now = (1 << 32) - 20
            else:
                src.now = (src.now + 30) & 0xFFFFFFFF
            got = check_stats(pkg, eng, cfg, src.now)
            assert got["n_parties"].sum() == len(eng.party_read()["size"])
        assert got["size_hist"][:, 15].sum() > 0
    finally:
        src.close()


def budget_of(cfg, rng, kind):
    G, M = cfg.n_groups, cfg.n_modes
    if kind == "queue":
        return rng.integers(0, 3, M * G).tolist(), None
    if kind == "mode":
        return None, [1] + [2] * (M - 1)
    if kind == "loose":
        return [UNL - 1] * (M * G), [10 ** 6] * M
    return None, None


@pytest.mark.gpu
@pytest.mark.parametrize("kind,layout", [("hashed", "split"), ("dense", "wide"), ("hashed", "overlap")])
@pytest.mark.parametrize("budget", ["none", "queue", "mode", "loose"])
@pytest.mark.parametrize("balance", [0, 1])
def test_prediction_is_the_next_party_match(pkg, kind, layout, budget, balance):
    cfg = status_config(pkg, kind, layout, modes=[("5v5", 2, 5), ("trio", 3, 3), ("duo40", 40, 2)])
    src = PartySrc(pkg, cfg, kind, seed=21)
    eng = src.eng
    rng = np.random.default_rng(7)
    G = cfg.n_groups
    if balance:
        eng.set_option("party_balance", 0b001)
    pq, pm = budget_of(cfg, rng, budget)
    if pq is not None or pm is not None:
        eng.set_offtick_budget(PARTY, pq, pm)
    rule_sets = [
        {(m, g): (0, 10, 5, 5, 80) for m in range(cfg.n_modes) for g in range(G)},
        {(m, g): (20, 0, 1, 2, 300) for m in range(cfg.n_modes) for g in range(0, G, 2)},  # the rest MM_WIDEN_OFF
        {(m, g): (5, 0, 10, 1, 4) for m in range(cfg.n_modes) for g in range(G)},  # narrow: all-or-nothing fails
    ]
    try:
        solo_ids = []
        for step in range(6):
            ids, r, m, ts = src.fresh(2500 if step % 2 == 0 else 300)
            src.enqueue(ids, r, m, ts)
            solo_ids.append(ids[:3])
            assert (eng.enqueue_party(*src.fresh_parties(300)) == 1).all()
            rules = rule_sets[step % 3]
            before = eng.party_read()
            rec, (lob, mem, st) = check_prediction(pkg, eng, cfg, src.now, rules)
            if step % 3 == 0:
                assert st.n_absorbed > 0 and st.n_lobbies > 0
            assert (rec["lobby"] == STAYS).any()
            # states 0 / 1 / 2 and repeated ids, after the call
            gone = before["members"][-1][0][:1]
            eng.remove(gone)
            matched = mem[:2]
            extra = np.concatenate([solo_ids[-1][:2], matched, np.array([2 ** 40 + 5], np.uint64), gone, gone])
            r2 = eng.party_locate(extra, src.now, rules)
            loc = eng.locate(extra, src.now)
            assert r2["state"].tolist() == loc["state"].tolist()
            assert (r2["lobby"][r2["state"] != 3] == STAYS).all() and (r2["window"][r2["state"] != 3] == -1).all()
            assert (r2["member"][r2["state"] != 3] == 0xFFFF).all() and r2[-1].tobytes() == r2[-2].tobytes()
            src.now += 7
    finally:
        src.close()


@pytest.mark.gpu
@pytest.mark.parametrize("teams", [3, 40, 256])
def test_prediction_at_many_teams(pkg, teams):
    cfg = pkg.synth.make_config(groups=[(0, 1000), (1001, 2000)], modes=[("t", teams, 2)], order=RATING,
                                capacity=200_000, active_capacity=1_000_000, default_group=-1)
    src = PartySrc(pkg, cfg, "hashed", seed=teams)
    eng = src.eng
    try:
        for step in range(3):
            src.enqueue(*src.fresh(4 * teams * 2 + 200, 0, 2001, modes=1))
            assert (eng.enqueue_party(*src.fresh_parties(teams + 20, 0, 2001)) == 1).all()
            rules = {(0, g): (0, 40, 5, 20, 3000) for g in range(2)}
            rec, (lob, _mem, _st) = check_prediction(pkg, eng, cfg, src.now, rules)
            assert len(lob) > 0 or step > 0
            src.now += 11
    finally:
        src.close()


def observe(eng, cfg, now):
    """Every output the calls must leave alone, as bytes."""
    out = [eng.pool_read(), eng.party_read(), eng.in_queue(np.arange(0, 5000, dtype=np.uint64)), eng.active_size(),
           eng.seq_next(), eng.queue_stats(now), eng.match_quality(True), eng.lobby_budget_report()]
    for src in (0, 1):
        out += [eng.offtick_report(src, True), eng.offtick_budget_report(src)]
    return out


def same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    if isinstance(a, C.Structure):
        return bytes(a) == bytes(b)
    return a == b


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
def test_no_side_effects_on_a_twin(pkg, kind):
    cfg = status_config(pkg, kind, "split", modes=[("5v5", 2, 5), ("trio", 3, 3)])
    a, b = PartySrc(pkg, cfg, kind, seed=31), PartySrc(pkg, cfg, kind, seed=31)
    rules = {(m, g): (0, 10, 5, 5, 80) for m in range(cfg.n_modes) for g in range(cfg.n_groups)}
    try:
        for e in (a.eng, b.eng):
            e.set_option("party_balance", 1)
            e.set_offtick_budget(PARTY, None, [3, UNL])
        for step in range(8):
            solos, parties = a.fresh(2000), a.fresh_parties(200)
            b.fresh(2000), b.fresh_parties(200)
            ids = np.concatenate([solos[0][:50], parties[1][:50]])
            for s in (a, b):
                if step % 4 != 3:
                    s.enqueue(*solos)
                    s.eng.enqueue_party(*parties)
            a.eng.party_queue_stats(a.now)
            a.eng.party_locate(ids, a.now, rules)
            op = step % 4
            if op == 0:
                ra, rb = a.eng.party_match(a.now, rules), b.eng.party_match(b.now, rules)
            elif op == 1:
                ra, rb = a.eng.tick(a.now)[:2], b.eng.tick(b.now)[:2]
            elif op == 2:
                ra, rb = a.eng.widen(a.now, {(0, 0): (5, 5, 1, 1, 50)}), b.eng.widen(b.now, {(0, 0): (5, 5, 1, 1, 50)})
            else:
                ra, rb = a.eng.remove(ids[::3]), b.eng.remove(ids[::3])
            if op in (0, 2):  # the stats hold a device time
                ra, rb = ra[:2], rb[:2]
            assert same(ra, rb)
            a.eng.party_locate(ids, a.now, rules)
            a.eng.party_queue_stats(a.now)
            assert same(observe(a.eng, cfg, a.now), observe(b.eng, cfg, b.now))
            a.now += 9
            b.now += 9
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
def test_refusals_change_nothing(pkg):
    abi = pkg.abi
    cfg = status_config(pkg, "hashed", "split")
    rules = {(0, 0): (0, 10, 5, 5, 80)}
    src = PartySrc(pkg, cfg, "hashed", seed=41)
    eng = src.eng
    try:
        src.enqueue(*src.fresh(500))
        assert (eng.enqueue_party(*src.fresh_parties(50)) == 1).all()
        before = observe(eng, cfg, src.now)
        ids = member_cols(party_state(eng))
        n = C.c_uint32(0)
        out = np.zeros(cfg.n_modes * cfg.n_groups, pkg.engine.PARTY_QUEUE_STAT_DTYPE)
        assert eng.lib.mm_party_queue_stats(eng.h, 0, out.ctypes.data, 1, C.byref(n)) == abi.MM_E_CAP
        assert n.value == cfg.n_modes * cfg.n_groups
        assert eng.lib.mm_party_queue_stats(eng.h, 0, None, 1, C.byref(n)) == abi.MM_E_ARG
        r = rules_of(cfg, rules)
        rec = np.zeros(len(ids), pkg.engine.PARTY_MEMBER_STATUS_DTYPE)
        assert eng.lib.mm_party_locate(eng.h, 0, None, len(ids), ids.ctypes.data, rec.ctypes.data) == abi.MM_E_ARG
        assert eng.lib.mm_party_locate(eng.h, 0, r.ctypes.data, len(ids), None, rec.ctypes.data) == abi.MM_E_ARG
        bad = r.copy()
        bad["step"][0] = 0
        bad["min_wait"][0] = 0
        assert eng.lib.mm_party_locate(eng.h, 0, bad.ctypes.data, len(ids), ids.ctypes.data, rec.ctypes.data) == \
            abi.MM_E_ARG
        assert b"step" in eng.lib.mm_last_error(eng.h)
        assert eng.lib.mm_party_locate(eng.h, 0, r.ctypes.data, 0, None, None) == abi.MM_OK
        assert same(observe(eng, cfg, src.now), before)
        with pytest.raises(pkg.EngineError):
            eng.party_locate(ids, 0, {(0, 0): (0, 0, 0, 0, 0)})
        assert same(observe(eng, cfg, src.now), before)
    finally:
        src.close()
    # 257 teams, no party capacity, arrival order, no dedupe: refused before anything runs
    big = pkg.synth.make_config(groups=[(0, 1000)], modes=[("t", 257, 2)], order=RATING, capacity=4096,
                                active_capacity=8192, default_group=-1)
    with pkg.Engine(big) as e:
        e.set_option("party_capacity", 1000)
        with pytest.raises(pkg.EngineError) as ex:
            e.party_locate([1], 0, {(0, 0): (0, 1, 1, 1, 1)})
        assert ex.value.status == abi.MM_E_ARG and b"257" in e.lib.mm_last_error(e.h)
    for order, flags, cap, status in ((RATING, 0, 0, abi.MM_E_STATE), (ARRIVAL, 0, 1000, abi.MM_E_ARG),
                                      (RATING, abi.MM_F_NO_DEDUPE, 1000, abi.MM_E_STATE)):
        c = pkg.synth.make_config(groups=[(0, 1000)], modes=[("5v5", 2, 5)], order=order, capacity=4096,
                                  active_capacity=8192, default_group=-1, flags=flags)
        with pkg.Engine(c) as e:
            if cap:
                try:
                    e.set_option("party_capacity", cap)
                except pkg.EngineError:
                    pass
            for call in (lambda: e.party_queue_stats(0), lambda: e.party_locate([1], 0, {(0, 0): (0, 1, 1, 1, 1)})):
                with pytest.raises(pkg.EngineError) as ex:
                    call()
                assert ex.value.status == status


@pytest.mark.gpu
def test_config3_two_hundred_thousand_parties(pkg):
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=[("5v5", 2, 5)], order=RATING,
                                capacity=10_500_000, active_capacity=12_000_000)
    eng = pkg.Engine(cfg)
    rng = np.random.default_rng(1)
    try:
        eng.set_option("party_capacity", 1_000_000)
        n = 10_000_000
        ids = np.arange(n, dtype=np.uint64) + np.uint64(1 << 40)
        eng.enqueue(ids, rng.integers(0, 3000, n).astype(np.int32), np.zeros(n, np.uint8),
                    rng.integers(0, 100, n).astype(np.uint32))
        k = 200_000
        sizes = rng.integers(2, 5, k).astype(np.uint8)
        m = int(sizes.sum())
        pid = np.arange(m, dtype=np.uint64) + np.uint64(1 << 41)
        prat = np.clip(np.repeat(rng.integers(0, 3000, k), sizes) + rng.integers(-30, 31, m), 0, 2999).astype(np.int32)
        assert (eng.enqueue_party(sizes, pid, prat, np.zeros(k, np.uint8), rng.integers(0, 100, k).astype(np.uint32))
                == 1).all()
        check_stats(pkg, eng, cfg, 100)
        rules = {(0, g): (30, 10, 5, 5, 100) for g in range(cfg.n_groups)}
        sel = pid[rng.choice(m, 10_000, replace=False)]
        rec = eng.party_locate(sel, 100, rules)
        assert (rec["state"] == 3).all()
        lob, mem, st = eng.party_match(100, rules, lobby_cap=1 << 20, member_cap=1 << 24)
        got = actual_places(cfg, lob, mem)
        placed = rec["lobby"] != STAYS
        assert placed.sum() > 1000 and (~placed).sum() > 10
        for x, r in zip(sel.tolist(), rec):
            if int(r["lobby"]) == STAYS:
                assert x not in got
            else:
                assert got[x] == (int(r["group"]), int(r["lobby"]), int(r["member"]))
    finally:
        eng.close()
