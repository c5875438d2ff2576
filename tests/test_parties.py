"""Parties (mm_enqueue_party / mm_party_match / mm_party_read / Engine.enqueue_party / Engine.party_match): players who
queue together are matched into one lobby and one team, around the parties that waited longest.

CPU: a plain restatement of the definition in include/mm_engine.h (one anchor, one party and one solo at a time), a
second one on per-bin lists (the shape of the device plan) held equal to it on random pools, hand-built cases, the
serialized enqueue codes, and the ABI mirror.
GPU: the engine against the restatement over both id kinds and split / wide layouts through a mixed schedule; the
enqueue codes against their serialized restatement; a twin given mm_take of the returned solos; the tick of an engine
holding parties against one holding only its solos; remove, expire, locate and requeue of party members; every
refusal; config3 at 10 M solos and 200 k parties.
"""
import ctypes as C

import numpy as np
import pytest

from .test_backfill import clamp_bounds, cfg_of, gpu_config, group_of
from .test_requeue import Src
from .test_widen import RATING, ARRIVAL, rules_of, wait_of, window


# ================================================================================ restatements
def party_rating(ratings):
    s = sum(int(r) for r in ratings)
    return s // len(ratings)  # Python's // floors toward minus infinity


def restate_plain(cfg, solos, parties, now, rules):
    """The definition, one anchor, one party and one solo at a time.
    solos: (ids, rating, mode, ts) of the live queued solos, age order inside every bin (mm_pool_read);
    parties: [(ids, ratings, mode, ts)] of the queued parties in age order (mm_party_read);
    rules: {(mode, group): (min_wait, w0, step, inc, w_max)}.
    -> ([(mode, group, [member ids])] in output order, n_anchors, n_absorbed, n_parties placed)"""
    lo, hi = clamp_bounds(cfg)
    c = lambda x: min(max(int(x), lo), hi)  # noqa: E731
    sid, srat, smode, _ = solos
    squeue = [(int(smode[i]), group_of(cfg, int(srat[i]))) for i in range(len(sid))]
    R = [party_rating(p[1]) for p in parties]
    pqueue = [(int(p[2]), group_of(cfg, R[j])) for j, p in enumerate(parties)]
    out, n_anc, n_abs, n_placed = [], 0, 0, 0
    for (m, g) in sorted(rules):
        rule = rules[(m, g)]
        T, S = cfg.modes[m].teams, cfg.modes[m].team_size
        U = [i for i in range(len(sid)) if squeue[i] == (m, g)]
        P = [j for j in range(len(parties)) if pqueue[j] == (m, g)]
        live, placed = set(U), set()
        for a in [j for j in P if wait_of(now, parties[j][3]) >= rule[0]]:
            n_anc += 1
            if a in placed:
                n_abs += 1
                continue
            w = window(rule, wait_of(now, parties[a][3]))
            room = [S] * T
            room[0] -= len(parties[a][0])
            team = {a: 0}
            Q = [b for b in P if b != a and b not in placed and abs(c(R[b]) - c(R[a])) <= w]
            Q.sort(key=lambda b: (abs(c(R[b]) - c(R[a])), c(R[b]), b))
            for b in Q:
                s = len(parties[b][0])
                t = next((t for t in range(T) if room[t] >= s), None)
                if t is not None:
                    room[t] -= s
                    team[b] = t
            n_open = sum(room)
            cand = [x for x in U if x in live and abs(c(srat[x]) - c(R[a])) <= w]
            if len(cand) < n_open:
                continue
            cand.sort(key=lambda x: (abs(c(srat[x]) - c(R[a])), c(srat[x]), x))
            teams = [[] for _ in range(T)]
            for b, t in team.items():  # placement order (dicts keep insertion order)
                teams[t] += [int(x) for x in parties[b][0]]
            k = 0
            for t in range(T):
                need = S - len(teams[t])
                teams[t] += [int(sid[x]) for x in cand[k:k + need]]
                k += need
            placed.update(team)
            n_placed += len(team)
            live.difference_update(cand[:n_open])
            out.append((m, g, [x for tm in teams for x in tm]))
    return out, n_anc, n_abs, n_placed


def restate_bins(cfg, solos, parties, now, rules):
    """The same definition on per-(queue, clamped rating) bins, as the device plans it: parties sorted by (bin, age),
    solos counted per bin (a lobby takes a bin's oldest untaken solos), both walked outward from the anchor's bin in
    (distance, rating) order.  -> the same as restate_plain"""
    lo, hi = clamp_bounds(cfg)
    sid, srat, smode, _ = solos
    srat = np.asarray(srat, np.int64)
    skey = np.clip(srat, lo, hi)
    sgrp = np.array([group_of(cfg, int(r)) for r in srat], np.int64)
    R = np.array([party_rating(p[1]) for p in parties], np.int64)
    pkey = np.clip(R, lo, hi)
    pgrp = np.array([group_of(cfg, int(r)) for r in R], np.int64)
    pmode = np.array([p[2] for p in parties], np.int64)
    psize = np.array([len(p[0]) for p in parties], np.int64)
    out, n_anc, n_abs, n_placed = [], 0, 0, 0
    for (m, g) in sorted(rules):
        rule = rules[(m, g)]
        T, S = cfg.modes[m].teams, cfg.modes[m].team_size
        ssel = np.flatnonzero((np.asarray(smode) == m) & (sgrp == g))
        psel = np.flatnonzero((pmode == m) & (pgrp == g))
        keys = np.unique(np.concatenate([skey[ssel], pkey[psel]]))
        sbin, pbin = {int(k): [] for k in keys}, {int(k): [] for k in keys}
        o = ssel[np.argsort(skey[ssel], kind="stable")]  # solos of a bin, age order
        cut = np.flatnonzero(np.diff(skey[o])) + 1
        for run in np.split(o, cut) if len(o) else []:
            sbin[int(skey[run[0]])] = run.tolist()
        for j in psel:  # parties of a bin, age order
            pbin[int(pkey[j])].append(int(j))
        used = {int(k): 0 for k in keys}
        lob = np.full(len(parties), -1)
        for a in psel[[wait_of(now, parties[j][3]) >= rule[0] for j in psel]] if len(psel) else []:
            n_anc += 1
            if lob[a] >= 0:
                n_abs += 1
                continue
            w = window(rule, wait_of(now, parties[a][3]))
            ka = int(pkey[a])
            d = np.abs(keys - ka)
            walk = [int(k) for k in keys[np.lexsort((keys, d))][np.sort(d)[:] <= w]]
            room = [S] * T
            room[0] -= int(psize[a])
            team = {int(a): 0}
            for k in walk:
                for b in pbin[k]:
                    if b == a or lob[b] >= 0 or sum(room) < 2:
                        continue
                    t = next((t for t in range(T) if room[t] >= psize[b]), None)
                    if t is not None:
                        room[t] -= int(psize[b])
                        team[int(b)] = t
            n_open = sum(room)
            if sum(len(sbin[k]) - used[k] for k in walk) < n_open:
                continue
            take, need = [], n_open
            for k in walk:
                t = min(need, len(sbin[k]) - used[k])
                take += sbin[k][used[k]:used[k] + t]
                used[k] += t
                need -= t
            teams = [[] for _ in range(T)]
            for b, t in team.items():
                teams[t] += [int(x) for x in parties[b][0]]
                lob[b] = len(out)
            k = 0
            for t in range(T):
                n = S - len(teams[t])
                teams[t] += [int(sid[x]) for x in take[k:k + n]]
                k += n
            n_placed += len(team)
            out.append((m, g, [x for tm in teams for x in tm]))
    return out, n_anc, n_abs, n_placed


def both(cfg, solos, parties, now, rules):
    a = restate_plain(cfg, solos, parties, now, rules)
    b = restate_bins(cfg, solos, parties, now, rules)
    assert a == b
    return [ms for _, _, ms in a[0]]


def enqueue_codes(cfg, active, sizes, ids, rating, mode, room, id_limit):
    """mm_enqueue_party's codes, one party at a time: active = the ids in the active set before the call, room = the
    members the table still holds."""
    codes, seen, used, off = [], set(), 0, 0
    for s, md in zip(sizes, mode):
        mem = [int(x) for x in ids[off:off + s]]
        rat = rating[off:off + s]
        off += s
        bad = md >= cfg.n_modes or s < 2 or s > cfg.modes[md].team_size if md < cfg.n_modes else True
        bad = bad or any(x >= id_limit for x in mem) or len(set(mem)) < s
        bad = bad or (s > 0 and group_of(cfg, min(max(party_rating(rat), -(1 << 31)), (1 << 31) - 1)) < 0)
        taken = any(x in active or x in seen for x in mem)
        seen.update(x for x in mem if x < id_limit)
        if bad:
            codes.append(2)
        elif taken:
            codes.append(0)
        else:
            used += s
            codes.append(3 if used > room else 1)
    return np.array(codes, np.uint8)


# ================================================================================ CPU: the definition, hand-built
def one_queue(pkg, teams=2, team_size=5, groups=((0, 3000),), default_group=-1):
    cfg = cfg_of(pkg, RATING, groups=list(groups), default_group=default_group, modes=1)
    cfg.modes[0].teams, cfg.modes[0].team_size = teams, team_size
    return cfg


def solos_of(ratings, first=100, ts=0):
    n = len(ratings)
    return (np.arange(first, first + n, dtype=np.uint64), np.asarray(ratings, np.int64), np.zeros(n, np.int64),
            np.full(n, ts, np.int64))


def party(first, ratings, ts=0, mode=0):
    return (list(range(first, first + len(ratings))), list(ratings), mode, ts)


RULE = {(0, 0): (0, 50, 1, 0, 50)}


def test_five_v_five_example(pkg):
    cfg = one_queue(pkg)
    parties = [party(0, [1500] * 3), party(10, [1500] * 4), party(20, [1490] * 2), party(30, [1510] * 3)]
    solos = solos_of([1400, 1501, 1620])
    out = both(cfg, solos, parties, 10, RULE)
    # team 0 = the anchor's 3 and the 2 at 1490; team 1 = the 4 and the solo nearest 1500; the 3 at 1510 is skipped
    assert out == [[0, 1, 2, 20, 21, 10, 11, 12, 13, 101]]


def test_window_edge_is_inclusive(pkg):
    cfg = one_queue(pkg, teams=1, team_size=4)
    rule = {(0, 0): (0, 5, 1, 0, 5)}
    assert both(cfg, solos_of([105, 95]), [party(0, [100, 100])], 10, rule) == [[0, 1, 101, 100]]
    assert both(cfg, solos_of([106, 95]), [party(0, [100, 100])], 10, rule) == []
    assert both(cfg, solos_of([]), [party(0, [100, 100]), party(5, [105, 105])], 10, rule) == [[0, 1, 5, 6]]


def test_ties_go_to_the_lower_rating_then_the_older_party(pkg):
    cfg = one_queue(pkg, teams=2, team_size=2)
    # co-parties at distance 10: 110 (oldest), 90, 90 — the older 90 wins team 1
    ps = [party(0, [100, 100]), party(10, [110, 110]), party(20, [90, 90]), party(30, [90, 90])]
    assert both(cfg, solos_of([]), ps, 10, RULE) == [[0, 1, 20, 21], [10, 11, 30, 31]]  # 110 then anchors the rest
    # solos at distance 10: the lower rating first, then the older
    cfg = one_queue(pkg, teams=1, team_size=4)
    assert both(cfg, solos_of([110, 90, 90]), [party(0, [100, 100])], 10, RULE) == [[0, 1, 101, 102]]


def test_absorbed_anchor(pkg):
    cfg = one_queue(pkg, teams=2, team_size=2)
    ps = [party(0, [100, 100]), party(10, [101, 101]), party(20, [300, 300]), party(30, [301, 301])]
    a = restate_plain(cfg, solos_of([]), ps, 10, RULE)
    assert [x[2] for x in a[0]] == [[0, 1, 10, 11], [20, 21, 30, 31]] and a[1:] == (4, 2, 4)
    assert restate_bins(cfg, solos_of([]), ps, 10, RULE) == a


def test_all_or_nothing(pkg):
    cfg = one_queue(pkg, teams=2, team_size=3)
    ps = [party(0, [100, 100]), party(10, [100, 100, 100])]
    assert both(cfg, solos_of([]), ps, 10, RULE) == []  # one open slot and no solo: nothing is placed
    assert both(cfg, solos_of([100, 100]), ps, 10, RULE) == [[0, 1, 100, 10, 11, 12]]
    assert both(cfg, solos_of([100]), [party(0, [100, 100])], 10, RULE) == []  # 4 open slots, 1 solo


def test_floor_steps_and_the_cap(pkg):
    cfg = one_queue(pkg, teams=1, team_size=3)
    rule = {(0, 0): (100, 5, 30, 7, 20)}
    ps = [party(0, [100, 100], ts=0)]
    assert both(cfg, solos_of([112]), ps, 129, rule) == []  # window 5
    assert both(cfg, solos_of([112]), ps, 130, rule) == [[0, 1, 100]]  # window 12
    assert both(cfg, solos_of([121]), ps, 10_000, rule) == []  # capped at 20
    assert both(cfg, solos_of([100]), ps, 99, rule) == []  # not an anchor yet


def test_disabled_queues_are_not_touched(pkg):
    cfg = one_queue(pkg, teams=1, team_size=2, groups=((0, 99), (100, 199)))
    ps = [party(0, [10, 11]), party(10, [150, 151])]
    assert both(cfg, solos_of([]), ps, 10, {(0, 1): (0, 5, 1, 0, 5)}) == [[10, 11]]
    assert both(cfg, solos_of([]), ps, 10, {}) == []


def test_default_group_clamps_the_party_rating(pkg):
    cfg = one_queue(pkg, teams=1, team_size=3, groups=((0, 99), (100, 199)), default_group=1)
    # R = 5000 clamps to 200 in the default group, as the solo at 250 does: distance 0
    assert both(cfg, solos_of([150, 250]), [party(0, [4000, 6000])], 10, {(0, 1): (0, 0, 1, 0, 0)}) == [[0, 1, 101]]
    cfg = one_queue(pkg, teams=1, team_size=4, groups=((0, 99), (100, 199)), default_group=1)
    out = both(cfg, solos_of([250, 900]), [party(0, [4000, 6000])], 10, {(0, 1): (0, 0, 1, 0, 0)})
    assert out == [[0, 1, 100, 101]]


def test_party_rating_floors_negative_sums(pkg):
    assert party_rating([-3, 0]) == -2 and party_rating([-1, -1, 1]) == -1 and party_rating([3, 4]) == 3
    cfg = one_queue(pkg, teams=1, team_size=3, groups=((-10, 10),))
    # R = floor(-3 / 2) = -2: the solo at -2 is at distance 0, the one at -1 is not (window 0)
    assert both(cfg, solos_of([-1, -2]), [party(0, [-3, 0])], 10, {(0, 0): (0, 0, 1, 0, 0)}) == [[0, 1, 101]]


@pytest.mark.parametrize("seed", range(6))
def test_bin_restatement_equals_the_plain_one(pkg, seed):
    rng = np.random.default_rng(seed)
    groups = [[(0, 99), (100, 299)], [(0, 200), (50, 120), (0, 400)], [(10, 60)]][seed % 3]
    cfg = cfg_of(pkg, RATING, groups=groups, default_group=len(groups) - 1 if seed % 2 else -1, modes=3)
    n = 200
    rating = rng.integers(-30, 450, n)
    keep = np.array([group_of(cfg, int(r)) >= 0 for r in rating])
    rating = rating[keep]
    solos = (np.arange(len(rating), dtype=np.uint64) + 1000, rating, rng.integers(1, 3, len(rating)),
             rng.integers(0, 40, len(rating)))
    parties, nxt = [], 0
    for _ in range(60):
        m = int(rng.integers(1, 3))  # 2v2, 3v3
        s = int(rng.integers(2, cfg.modes[m].team_size + 1))
        base = int(rng.integers(-30, 450))
        r = [base + int(x) for x in rng.integers(-5, 6, s)]
        if group_of(cfg, party_rating(r)) < 0:
            continue
        parties.append(party(nxt, r, ts=int(rng.integers(0, 40)), mode=m))
        nxt += s
    rules = {(m, g): (int(rng.integers(0, 30)), int(rng.integers(0, 20)), int(rng.integers(1, 5)),
                      int(rng.integers(0, 10)), 60) for m in (1, 2) for g in range(len(groups)) if rng.random() < .8}
    both(cfg, solos, parties, 40, rules)


def test_enqueue_codes_restatement(pkg):
    cfg = one_queue(pkg, teams=2, team_size=3, groups=((0, 99),))
    sizes = [2, 2, 4, 2, 3, 2, 2, 1]
    ids = [1, 2, 2, 3, 4, 5, 6, 7, 8, 8, 9, 10, 11, 12, 13, 14, 15, 16]
    rating = [10] * len(ids)
    codes = enqueue_codes(cfg, {16}, sizes, ids, rating, [0] * 8, room=7, id_limit=1 << 40)
    # 2 clashes with party 0; 4 members > team size 3; 8 twice; 9..11 and 12, 13 fill the 7; 14, 15 do not fit; a
    # party of one is invalid even though 16 was queued
    assert codes.tolist() == [1, 0, 2, 2, 1, 1, 3, 2]


def test_abi_mirror_and_symbols(pkg):
    abi = pkg.abi
    assert C.sizeof(abi.PartyStats) == 32
    for name, nargs in (("mm_enqueue_party", 8), ("mm_party_match", 8), ("mm_party_read", 13)):
        res, args = abi.PROTOTYPES[name]
        assert res is C.c_int and len(args) == nargs
    import os
    so = os.path.join(os.path.dirname(pkg.__file__), "csrc", "libmm_engine.so")
    if os.path.exists(so):
        lib = C.CDLL(so)
        for name in ("mm_enqueue_party", "mm_party_match", "mm_party_read"):
            assert hasattr(lib, name)


# ================================================================================ GPU
def party_state(eng):
    pr = eng.party_read()
    return [(ids, rat, int(m), int(ts)) for (ids, rat), m, ts in zip(pr["members"], pr["mode"], pr["enq_ts"])]


def check_party(eng, cfg, now, rules):
    """mm_party_match on eng against the restatement of its pool and table -> (member ids, solo ids)"""
    p = eng.pool_read()
    parties = party_state(eng)
    want, n_anc, n_abs, n_pl = restate_plain(cfg, (p["id"], p["rating"], p["mode"], p["enq_ts"]), parties, now, rules)
    lob, mem, st = eng.party_match(now, rules_of(cfg, rules))
    assert (st.n_anchors, st.n_absorbed, st.n_parties, st.n_lobbies) == (n_anc, n_abs, n_pl, len(want))
    off = np.concatenate([[0], np.cumsum([len(x[2]) for x in want])]).astype(np.int64)
    assert [tuple(int(x) for x in (h["mode"], h["group"], h["n_members"], h["first_member"])) for h in lob] == \
        [(m, g, len(ms), int(off[k])) for k, (m, g, ms) in enumerate(want)]
    flat = np.array([x for _, _, ms in want for x in ms], np.uint64)
    assert np.array_equal(mem, flat)
    in_party = set(int(x) for ps in parties for x in ps[0])
    solo = np.array([x for x in flat if int(x) not in in_party], np.uint64)
    return mem, solo


class PartySrc(Src):
    """Src with parties: fresh parties of 2 .. team_size members near one rating."""

    def __init__(self, pkg, cfg, kind, seed, cap=200_000):
        super().__init__(pkg, cfg, kind, seed)
        self.eng.set_option("party_capacity", cap)

    def fresh_parties(self, n, lo=0, hi=5001):
        sizes, ids, rat, mode, ts = [], [], [], [], []
        for _ in range(n):
            m = int(self.rng.integers(0, self.cfg.n_modes))
            S = self.cfg.modes[m].team_size
            if S < 2:
                m = next(k for k in range(self.cfg.n_modes) if self.cfg.modes[k].team_size >= 2)
                S = self.cfg.modes[m].team_size
            s = int(self.rng.integers(2, min(S, 4) + 1))
            x, r, _, t = self.fresh(s, lo, hi)
            r = np.clip(r[:1] + self.rng.integers(-20, 21, s), lo, hi - 1).astype(np.int32)
            sizes.append(s); ids.append(x); rat.append(r); mode.append(m); ts.append(int(t[0]))
        return (np.array(sizes, np.uint8), np.concatenate(ids), np.concatenate(rat), np.array(mode, np.uint8),
                np.array(ts, np.uint32))


def party_rules(cfg):
    G = cfg.n_groups
    return [
        {(m, g): (0, 10, 5, 5, 80) for m in range(cfg.n_modes) for g in range(G)},
        {(m, g): (20, 0, 1, 2, 300) for m in range(cfg.n_modes) for g in range(0, G, 2)},
    ]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
@pytest.mark.parametrize("layout", ["split", "wide"])
def test_engine_equals_the_restatement_over_a_mixed_schedule(pkg, kind, layout):
    cfg = gpu_config(pkg, RATING, kind, layout)
    src = PartySrc(pkg, cfg, kind, seed=5)
    b = pkg.Engine(cfg)  # the twin: the same solos, mm_take of the returned solos, no parties
    rules = party_rules(cfg)
    total = 0
    try:
        for step in range(14):
            op = step % 7
            if op == 0:
                src.enqueue(*src.fresh(6000), engines=(b,))
                assert (src.eng.enqueue_party(*src.fresh_parties(600)) == 1).all()
            elif op == 1:
                mem, solo = check_party(src.eng, cfg, src.now, rules[step % 2])
                total += len(mem)
                assert b.take(solo) == len(solo)
                assert src.eng.in_queue(mem).all()
                assert (src.eng.locate(mem, src.now)["state"] == 2).all()
            elif op == 2:
                ra, rb = src.eng.tick(src.now), b.tick(src.now)
                for x, y in zip(ra[:2], rb[:2]):
                    assert np.array_equal(x, y)
                src.now += 5
            elif op == 3:
                wa, wb = src.eng.widen(src.now, {(0, 0): (10, 5, 1, 1, 50)}), b.widen(src.now, {(0, 0): (10, 5, 1, 1, 50)})
                assert np.array_equal(wa[1], wb[1])
            elif op == 4:
                live = src.eng.pool_read()["id"]
                pr = src.eng.party_read()
                gone = np.concatenate([live[::41]] + [pr["members"][k][0][:1] for k in range(0, len(pr["size"]), 9)])
                n_party = sum(int(pr["size"][k]) for k in range(0, len(pr["size"]), 9))
                assert src.eng.remove(gone) == b.remove(live[::41]) + n_party
            elif op == 5:
                ea, eb = src.eng.expire(src.now, 58), b.expire(src.now, 58)
                na = len(ea[0])
                assert na >= len(eb[0]) and np.array_equal(np.sort(ea[0][:len(eb[0])]), np.sort(eb[0]))
            elif op == 6:
                fa, fb = src.eng.backfill(1, 0, 1000, 3, 40), b.backfill(1, 0, 1000, 3, 40)
                assert np.array_equal(fa[0], fb[0]) and all(np.array_equal(x, y) for x, y in zip(fa[1], fb[1]))
            pa, pb = src.eng.pool_read(), b.pool_read()
            for k in pa:
                assert np.array_equal(pa[k], pb[k]), k
            qa, qb = src.eng.queue_stats(src.now), b.queue_stats(src.now)
            for f in ("mode", "group", "n_waiting", "max_wait", "wait_hist"):
                assert np.array_equal(qa[f], qb[f]), f
            la, lb = src.eng.locate(pa["id"][::61], src.now), b.locate(pa["id"][::61], src.now)
            for f in la.dtype.names:  # seq: the parties took numbers on one engine only
                assert f == "seq" or np.array_equal(la[f], lb[f]), f
        assert total > 0
    finally:
        b.close()
        src.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
def test_enqueue_codes_equal_the_serialized_restatement(pkg, kind):
    cfg = gpu_config(pkg, RATING, kind, "split")
    src = PartySrc(pkg, cfg, kind, seed=9, cap=150)
    try:
        ids, r, m, ts = src.fresh(50)
        src.enqueue(ids, r, m, ts)
        sizes, pid, prat, pmode, pts = src.fresh_parties(120)
        pid = pid.copy()
        rng = np.random.default_rng(3)
        # collisions with solos, with earlier parties of the batch and inside one party; invalid modes and sizes
        k = rng.choice(len(pid), 40, replace=False)
        pid[k[:10]] = ids[:10]
        pid[k[10:30]] = pid[rng.integers(0, len(pid), 20)]
        pmode[::17] = cfg.n_modes
        limit = cfg.active_capacity if kind == "dense" else (1 << 64) - 2
        if kind == "dense":
            pid[k[30:32]] = limit + 5
        active = set(int(x) for x in ids)
        want = enqueue_codes(cfg, active, sizes.tolist(), pid, prat, pmode.tolist(), room=150, id_limit=limit)
        got = src.eng.enqueue_party(sizes, pid, prat, pmode, pts)
        assert np.array_equal(got, want)
        assert (got == 3).any() and (got == 0).any() and (got == 2).any() and (got == 1).any()
        pr = src.eng.party_read()
        assert np.array_equal(pr["size"], sizes[got == 1])
        assert src.eng.active_size() == 50 + int(sizes[got == 1].sum())
        acc = np.concatenate([pid[int(o):int(o) + int(s)] for o, s, c in
                              zip(np.concatenate([[0], np.cumsum(sizes)[:-1]]), sizes, got) if c == 1])
        assert src.eng.in_queue(acc).all()
        lost = np.setdiff1d(pid[pid < limit], np.concatenate([acc, ids]))
        assert not src.eng.in_queue(lost).any()
        assert src.eng.pool_size() == 50
    finally:
        src.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
def test_tick_is_untouched_by_parties_and_seq_is_shared(pkg, kind):
    cfg = gpu_config(pkg, RATING, kind, "split")
    src = PartySrc(pkg, cfg, kind, seed=13)
    b = pkg.Engine(cfg)
    try:
        for _ in range(3):
            src.enqueue(*src.fresh(5000), engines=(b,))
            n = src.eng.seq_next()
            party = src.fresh_parties(300)
            assert (src.eng.enqueue_party(*party) == 1).all()
            assert src.eng.seq_next() == n + 300
            # 300 entries without a mode consume the same 300 numbers on the twin (code 2)
            assert (b.enqueue(*src.fresh(300)[:2], np.full(300, 200, np.uint8)) == 2).all()
        ra, rb = src.eng.tick(src.now), b.tick(src.now)
        assert len(ra[0]) > 0
        assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[2], rb[2])
    finally:
        b.close()
        src.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
def test_lifecycle_of_party_members(pkg, kind):
    cfg = gpu_config(pkg, RATING, kind, "split")
    src = PartySrc(pkg, cfg, kind, seed=17)
    try:
        src.enqueue(*src.fresh(2000))
        sizes, ids, rat, mode, ts = src.fresh_parties(30)
        ts[:10] = src.now - 500
        assert (src.eng.enqueue_party(sizes, ids, rat, mode, ts) == 1).all()
        n0 = src.eng.active_size()
        off = np.concatenate([[0], np.cumsum(sizes.astype(np.int64))])
        # locate: state 3 with the member's own rating and the party's queue
        loc = src.eng.locate(ids, src.now)
        assert (loc["state"] == 3).all() and np.array_equal(loc["rating"], rat)
        assert (loc["lobby"] == pkg.abi.MM_LOCATE_STAYS).all() and (loc["depth"] == 0).all()
        assert np.array_equal(loc["seq"], np.repeat(src.eng.party_read()["seq"], sizes))
        # requeue of a queued member: code 0
        first = off[:3]  # members of three parties: three sequence numbers
        assert (src.eng.requeue(ids[first], rat[first], mode[:3], None, loc["seq"][first]) == 0).all()
        # remove of one member dissolves the party
        j, sizes = 12, sizes.astype(np.int64)
        assert src.eng.remove(ids[off[j]:off[j] + 1]) == sizes[j]
        assert not src.eng.in_queue(ids[off[j]:off[j + 1]]).any()
        assert src.eng.active_size() == n0 - sizes[j]
        # expire: the 10 old parties, every member with the party's seq
        seqs = src.eng.party_read()["seq"]
        got, got_seq = src.eng.expire(src.now, 400)
        assert np.array_equal(np.sort(got), np.sort(ids[:off[10]]))
        assert set(got_seq.tolist()) == set(seqs[:10].tolist())
        assert len(src.eng.party_read()["size"]) == 19
        assert src.eng.active_size() == n0 - sizes[j] - off[10]
        assert src.eng.pool_size() == 2000
    finally:
        src.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense", "no_dedupe"])
def test_refusals_change_nothing(pkg, kind):
    abi = pkg.abi
    flags = {"hashed": 0, "dense": 2, "no_dedupe": 1}[kind]
    cfg = cfg_of(pkg, RATING, flags=flags, modes=3)
    eng = pkg.Engine(cfg)
    try:
        one = (np.array([2], np.uint8), np.array([1, 2], np.uint64), np.array([100, 100], np.int32),
               np.array([1], np.uint8))
        rules = rules_of(cfg, {(1, 0): (0, 5, 1, 0, 5)})
        with pytest.raises(pkg.EngineError) as ex:  # no party capacity
            eng.enqueue_party(*one)
        assert ex.value.status == abi.MM_E_STATE
        with pytest.raises(pkg.EngineError) as ex:
            eng.party_match(0, rules)
        assert ex.value.status == (abi.MM_E_STATE)
        eng.set_option("party_capacity", 100)
        if kind == "no_dedupe":
            with pytest.raises(pkg.EngineError) as ex:
                eng.enqueue_party(*one)
            assert ex.value.status == abi.MM_E_STATE
            return
        eng.enqueue(np.arange(10, 20, dtype=np.uint64), np.full(10, 100, np.int32), np.ones(10, np.uint8))
        assert (eng.enqueue_party(*one) == 1).all()
        with pytest.raises(pkg.EngineError) as ex:
            eng.set_option("party_capacity", 1)
        assert ex.value.status == abi.MM_E_ARG
        bad = rules.copy()
        bad[1 * cfg.n_groups]["step"] = 0
        for r in (bad,):
            with pytest.raises(pkg.EngineError) as ex:
                eng.party_match(0, r)
            assert ex.value.status == abi.MM_E_ARG
        def state():
            pr = eng.party_read()
            return (eng.pool_read()["id"].tolist(), eng.active_size(), eng.in_queue([1, 2, 10]).tolist(),
                    pr["size"].tolist(), pr["seq"].tolist(), eng.seq_next())

        before = state()
        st = abi.PartyStats()
        rc = eng.lib.mm_party_match(eng.h, 0, rules.ctypes.data, None, 0, None, 0, C.byref(st))
        assert rc == abi.MM_E_CAP and st.n_lobbies == 1 and st.n_matched == 4  # 2v2: a dry run
        lob, mem = np.empty(4, pkg.engine.LOBBY_DTYPE), np.empty(4, np.uint64)
        rc = eng.lib.mm_party_match(eng.h, 0, rules.ctypes.data, lob.ctypes.data, 4, mem.ctypes.data, 3, C.byref(st))
        assert rc == abi.MM_E_CAP and st.n_matched == 4  # member_cap one short
        assert state() == before
        other = pkg.Engine(cfg)
        other.enqueue(np.array([900], np.uint64), np.array([100], np.int32), np.array([1], np.uint8))
        img = other.export_queues(np.ones(cfg.n_modes * cfg.n_groups, bool))
        other.close()
        for call in (lambda: eng.export_state(), lambda: eng.snapshot(), lambda: eng.merge_queues(img),
                     lambda: eng.export_queues(np.ones(cfg.n_modes * cfg.n_groups, bool))):
            with pytest.raises(pkg.EngineError) as ex:
                call()
            assert ex.value.status == abi.MM_E_STATE
        if kind == "dense":  # a staged packed batch refuses both party calls
            eng.enqueue_packed_begin(np.array([50], np.uint32), eng.pack_key([100], [1]))
            for call in (lambda: eng.enqueue_party(*one), lambda: eng.party_match(0, rules)):
                with pytest.raises(pkg.EngineError) as ex:
                    call()
                assert ex.value.status == abi.MM_E_STATE
            eng.enqueue_packed_end()
            eng.remove([50])
            before = state()
        assert state() == before
        n_pool = 11 if kind == "dense" else 10  # the removed staged player's slot counts until the next tick
        assert eng.pool_size() == n_pool and eng.in_queue([1, 2]).all() and len(eng.party_read()["size"]) == 1
        lob, mem, st = eng.party_match(0, rules)
        assert mem[:2].tolist() == [1, 2] and len(mem) == 4 and eng.pool_size() == n_pool
        eng.snapshot()  # nothing queued in a party any more
    finally:
        eng.close()
    arr = pkg.Engine(cfg_of(pkg, ARRIVAL, modes=3))
    try:
        arr.set_option("party_capacity", 100)
        for call in (lambda: arr.enqueue_party(*one), lambda: arr.party_match(0, rules)):
            with pytest.raises(pkg.EngineError) as ex:
                call()
            assert ex.value.status == abi.MM_E_ARG
        assert arr.active_size() == 0 and arr.seq_next() == 0
    finally:
        arr.close()


@pytest.mark.gpu
def test_config3_ten_million_solos_and_200k_parties(pkg):
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=[("5v5", 2, 5)], order=RATING,
                                capacity=10_500_000, active_capacity=12_000_000)
    eng = pkg.Engine(cfg)
    rng = np.random.default_rng(1)
    try:
        eng.set_option("party_capacity", 1_000_000)
        n = 10_000_000
        ids = np.arange(n, dtype=np.uint64) + np.uint64(1 << 40)
        r = rng.integers(0, 3000, n).astype(np.int32)
        eng.enqueue(ids, r, np.zeros(n, np.uint8), rng.integers(0, 100, n).astype(np.uint32))
        k = 200_000
        sizes = rng.integers(2, 5, k).astype(np.uint8)
        m = int(sizes.sum())
        pid = np.arange(m, dtype=np.uint64) + np.uint64(1 << 41)
        base = np.repeat(rng.integers(0, 3000, k), sizes)
        prat = np.clip(base + rng.integers(-30, 31, m), 0, 2999).astype(np.int32)
        assert (eng.enqueue_party(sizes, pid, prat, np.zeros(k, np.uint8),
                                  rng.integers(0, 100, k).astype(np.uint32)) == 1).all()
        parties = party_state(eng)
        rules = {(0, g): (30, 10, 5, 5, 100) for g in range(cfg.n_groups)}
        p = eng.pool_read()
        lob, mem, st = eng.party_match(100, rules_of(cfg, rules), lobby_cap=1 << 20, member_cap=1 << 24)
        assert st.n_lobbies > 1000
        pset = {int(x): j for j, ps in enumerate(parties) for x in ps[0]}
        R = np.array([party_rating(ps[1]) for ps in parties])
        lo, hi = clamp_bounds(cfg)
        rating_of = dict(zip(p["id"].tolist(), p["rating"].tolist()))
        for h in lob[::97]:
            ms = mem[h["first_member"]:h["first_member"] + h["n_members"]].tolist()
            assert len(set(ms)) == 10
            js = [pset[x] for x in ms if x in pset]
            anchor = js[0]
            w = window(rules[(0, int(h["group"]))], wait_of(100, parties[anchor][3]))
            ca = min(max(int(R[anchor]), lo), hi)
            for t in range(2):  # every party contiguous on one team
                team = ms[5 * t:5 * t + 5]
                for j in set(pset[x] for x in team if x in pset):
                    assert all(x in team for x in parties[j][0])
            for x in ms:
                rx = int(R[pset[x]]) if x in pset else rating_of[x]
                assert abs(min(max(rx, lo), hi) - ca) <= w
        # the first queue of one group equals the restatement exactly
        g = 0
        sel = np.array([group_of(cfg, int(x)) == g for x in p["rating"]])
        psel = [ps for ps, rr in zip(parties, R) if group_of(cfg, int(rr)) == g]
        want = restate_bins(cfg, (p["id"][sel], p["rating"][sel], p["mode"][sel], p["enq_ts"][sel]), psel, 100,
                            {(0, g): rules[(0, g)]})[0]
        got = [mem[h["first_member"]:h["first_member"] + h["n_members"]].tolist() for h in lob if h["group"] == g]
        assert got == [ms for _, _, ms in want]
    finally:
        eng.close()


# ================================================================================ CPU: SearchPool(parties=...)
def party_engine(pkg, calls):
    from .test_requeue import requeue_engine

    class PartyEngine(requeue_engine(pkg)):
        """The engine double with parties: enqueue_party by the serialized codes, party_match by the restatement over
        its pool and table, then take of the solos.  Its tick emits nothing; calls records the order of the calls."""

        def __init__(self, cfg):
            super().__init__(cfg)
            self.parties = []  # (ids, ratings, mode, ts) in age order
            self.options = {}

        def set_option(self, name, value):
            self.options[name] = value

        def enqueue_party(self, sizes, ids, rating, mode, enq_ts):
            codes = enqueue_codes(self.cfg, self.active, sizes.tolist(), ids, rating, mode.tolist(),
                                  room=self.options.get("party_capacity", 0), id_limit=2 ** 64 - 2)
            off = 0
            for s, c, m, t in zip(sizes.tolist(), codes.tolist(), mode.tolist(), enq_ts.tolist()):
                if c == 1:
                    self.parties.append(([int(x) for x in ids[off:off + s]], list(rating[off:off + s]), m, t))
                    self.active.update(int(x) for x in ids[off:off + s])
                off += s
            self.ctr = (self.ctr + len(sizes)) & 0xFFFFFFFF
            return codes

        def party_read(self):
            R = [party_rating(p[1]) for p in self.parties]
            return dict(size=np.array([len(p[0]) for p in self.parties], np.uint8),
                        mode=np.array([p[2] for p in self.parties], np.uint8),
                        group=np.array([group_of(self.cfg, r) for r in R], np.uint8))

        def party_match(self, now, rules):
            calls.append("party_match")
            p = self.pool_read()
            ts = [self.ts[int(x)] for x in p["id"]]
            out = restate_plain(self.cfg, (p["id"], p["rating"], p["mode"], ts), self.parties, now, rules)[0]
            placed = {x for _, _, ms in out for x in ms}
            self.parties = [q for q in self.parties if q[0][0] not in placed]
            mem = np.array([x for _, _, ms in out for x in ms], np.uint64)
            self.take(mem)
            lob = np.zeros(len(out), pkg.engine.LOBBY_DTYPE)
            first = 0
            for i, (m, g, ms) in enumerate(out):
                lob[i] = (first, len(ms), m, g)
                first += len(ms)
            return lob, mem, pkg.abi.PartyStats()

        def tick(self, now=0, *a, **k):
            calls.append("tick")
            return np.zeros(0, pkg.engine.LOBBY_DTYPE), np.zeros(0, np.uint64), None, None

    return PartyEngine


def publish_party(pkg, broker, sw, group, players, mode):
    import json
    broker.publish(sw.generate_exchange_name(group), sw.generate_queue_name(group),
                   json.dumps({"party": [{"id": pid, "rating": r} for pid, r in players], "game-mode": mode}))


def test_search_pool_party_flow(pkg):
    import importlib
    from .fakes import FakeBroker
    from .test_expire import publish
    from .test_handover import start_workers
    from .test_requeue import lobbies
    sw = importlib.import_module("microservice-matchmaking_b200.search_worker")
    calls = []
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=RATING, capacity=1000, active_capacity=4000)
    eng = party_engine(pkg, calls)(cfg)
    pool = sw.SearchPool(eng, ["1v1", "5v5"], list(pkg.synth.REFERENCE_GROUP_NAMES), flush_every_s=3600,
                         clock=lambda: 0.0, parties={"5v5": (0, 50, 1000, 0, 50)}, party_capacity=100)
    assert eng.options["party_capacity"] == 100
    broker = FakeBroker()
    start_workers(sw, broker, pool, pkg)
    publish(pkg, broker, cfg, "s0", 100, mode="5v5")  # a solo of bronze 5v5
    publish_party(pkg, broker, sw, "bronze", [(f"a{i}", 100 + i) for i in range(5)], "5v5")  # tag 2
    publish_party(pkg, broker, sw, "bronze", [(f"b{i}", 110 - i) for i in range(5)], "5v5")  # tag 3
    publish_party(pkg, broker, sw, "bronze", [("c0", 100), ("c1", 100)], "1v1")  # tag 4: larger than a 1v1 team
    publish_party(pkg, broker, sw, "bronze", [("s0", 100), ("d1", 100)], "5v5")  # tag 5: s0 is already queued
    broker.deliver_all()
    assert not broker.acked and len(pool._staged_parties) == 4  # staged until the next flush
    assert pool.party_status("bronze") == {}
    pool.flush()
    assert sorted(broker.acked) == [1, 2, 3, 5] and broker.nacked == [4]  # by party
    assert pool.in_queue("a0") and pool.in_queue("b4") and not pool.in_queue("d1") and not pool.in_queue("c0")
    assert pool.party_status("bronze") == {"5v5": {"parties": 2, "players": 10}}  # SearchWorker.status()["parties"]
    assert pool.tick() == 1 and calls == ["party_match", "tick"]  # the parties' match runs before the tick
    lob = lobbies(broker, sw)
    assert len(lob) == 1 and lob[0]["game-mode"] == "5v5"
    assert [[p["id"] for p in team] for team in lob[0]["teams"].values()] == [[f"a{i}" for i in range(5)],
                                                                             [f"b{i}" for i in range(5)]]
    assert pool.stats["party_lobbies"] == 1 and pool.stats["lobbies"] == 0
    assert pool.in_queue("s0") and eng.pool_size() == 1  # the solo stays queued: every slot went to a party


def test_search_pool_remove_takes_the_whole_party_out(pkg):
    import importlib
    from .fakes import FakeBroker
    from .test_handover import start_workers
    sw = importlib.import_module("microservice-matchmaking_b200.search_worker")
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=RATING, capacity=1000, active_capacity=4000)
    eng = party_engine(pkg, [])(cfg)
    pool = sw.SearchPool(eng, ["1v1", "5v5"], list(pkg.synth.REFERENCE_GROUP_NAMES), flush_every_s=3600,
                         clock=lambda: 0.0, parties={"5v5": (0, 50, 1000, 0, 50)}, party_capacity=100)
    broker = FakeBroker()
    start_workers(sw, broker, pool, pkg)
    publish_party(pkg, broker, sw, "bronze", [("a0", 100), ("a1", 100)], "5v5")
    broker.deliver_all()
    pool.flush()
    h1 = pool.handles.lookup("a1")
    eng.remove = lambda ids: sum(len(p[0]) for p in eng.parties)  # the engine dissolves the party
    assert pool.remove_user("a0") == ("ok", "removed")
    assert pool.handles.lookup("a0") is None and pool.handles.lookup("a1") is None and h1 not in pool.players
    with pytest.raises(ValueError, match="MM_ORDER_RATING"):
        sw.SearchPool(eng.__class__(pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=ARRIVAL,
                                                           capacity=10, active_capacity=40)),
                      ["1v1", "5v5"], list(pkg.synth.REFERENCE_GROUP_NAMES), parties={"5v5": (0, 1, 1, 0, 1)})
