"""Party backfill (mm_backfill_party / Engine.backfill_party / SearchPool.backfill_teams): the open team slots of
running lobbies filled with whole queued parties of their queues first, then with the nearest solos, requests served
one at a time in index order.

CPU: a plain serialized restatement of the definition in include/mm_engine.h on hand-built cases, a binned restatement
(the shape of the device plan) held equal to it on random cases, the ABI mirror, and SearchPool.backfill_teams with an
engine double, its matched-party book and requeue().
GPU: the engine against the restatement of what mm_pool_read and mm_party_read report, on both id kinds, both
rating-order layouts and overlapping groups with a default group, and on a party table of more than three scatter tiles
with one crowded bin; long mixed schedules of every call with backfill_party among them (`EngineSchedule` with the
call added to its model); the twin engine of the header's EQUIVALENCE; party-free queues against mm_backfill; a round
trip through mm_requeue_party and mm_requeue; every refusal; config3 at 10 M solos and 200 k parties.
"""
import ctypes as C

import numpy as np
import pytest

from .test_backfill import cfg_of, clamp_bounds, gpu_config, group_of
from .test_backfill import restate as bf_restate
from .test_engine_model import U32
from .test_parties import PartySrc, party_rating, party_state
from .test_party_requeue import RequeueModel, RequeueSchedule, party_requeue_engine, requeue_pool
from .test_requeue import export_sections
from .test_tile_geometry import DENSE, MODES8, WIDE

RATING, ARRIVAL = 1, 0


# ================================================================================ restatements
def restate_plain(cfg, solos, parties, reqs):
    """The definition, one request, one party and one solo at a time.
    solos: (ids, rating, mode) of the live queued solos in age order (mm_pool_read); parties: [(ids, ratings, mode)] of
    the queued parties in age order (mm_party_read); reqs: [(mode, group, target, [room per team], window)].
    -> (filled: per request the members per team, members: per request one id list per team)"""
    lo, hi = clamp_bounds(cfg)
    c = lambda x: min(max(int(x), lo), hi)  # noqa: E731
    sid, srat, smode = solos
    squeue = [(int(smode[i]), group_of(cfg, int(srat[i]))) for i in range(len(sid))]
    R = [party_rating(p[1]) for p in parties]
    pqueue = [(int(p[2]), group_of(cfg, R[b])) for b, p in enumerate(parties)]
    taken, placed, filled, members = set(), set(), [], []
    for (m, g, t, room, w) in reqs:
        room, ct = [int(x) for x in room], c(t)
        inside = lambda x: w < 0 or abs(c(x) - ct) <= w  # noqa: E731
        teams = [[] for _ in room]
        Q = [b for b in range(len(parties)) if pqueue[b] == (m, g) and b not in placed and inside(R[b])]
        Q.sort(key=lambda b: (abs(c(R[b]) - ct), c(R[b]), b))
        for b in Q:
            s = len(parties[b][0])
            k = next((k for k in range(len(room)) if room[k] >= s), None)
            if k is None:
                continue
            room[k] -= s
            teams[k] += [int(x) for x in parties[b][0]]
            placed.add(b)
        cand = [x for x in range(len(sid)) if squeue[x] == (m, g) and x not in taken and inside(srat[x])]
        cand.sort(key=lambda x: (abs(c(srat[x]) - ct), c(srat[x]), x))
        at = 0
        for k in range(len(room)):
            got = cand[at:at + room[k]]
            at += len(got)
            taken.update(got)
            teams[k] += [int(sid[x]) for x in got]
        filled.append([len(x) for x in teams])
        members.append(teams)
    return filled, members


def restate_bins(cfg, solos, parties, reqs):
    """The same definition on per-(queue, clamped rating) bins, as the device plans it: parties by (bin, age), solos
    counted per bin (a walk takes a bin's oldest untaken solos), both walked outward from the target in (distance,
    rating) order; the solos once per team, each walk going on where the last one stopped.  -> as restate_plain"""
    lo, hi = clamp_bounds(cfg)
    sid, srat, smode = solos
    srat = np.asarray(srat, np.int64)
    skey = np.clip(srat, lo, hi)
    squeue = np.asarray(smode, np.int64) * cfg.n_groups + np.array([group_of(cfg, int(r)) for r in srat], np.int64)
    R = np.array([party_rating(p[1]) for p in parties], np.int64)
    pkey = np.clip(R, lo, hi)
    pqueue = np.array([int(p[2]) * cfg.n_groups + group_of(cfg, int(r)) for p, r in zip(parties, R)], np.int64)
    sbin, pbin, used = {}, {}, {}
    for x in range(len(sid)):
        sbin.setdefault((int(squeue[x]), int(skey[x])), []).append(x)
    for b in range(len(parties)):
        pbin.setdefault((int(pqueue[b]), int(pkey[b])), []).append(b)
    qkeys = {}
    for (q, k) in list(sbin) + list(pbin):
        qkeys.setdefault(q, set()).add(k)
    qkeys = {q: np.array(sorted(ks), np.int64) for q, ks in qkeys.items()}
    placed = np.zeros(len(parties), bool)
    filled, members = [], []
    for (m, g, t, room, w) in reqs:
        q, ct = int(m) * cfg.n_groups + int(g), min(max(int(t), lo), hi)
        keys = qkeys.get(q, np.zeros(0, np.int64))
        d = np.abs(keys - ct)
        o = np.lexsort((keys, d))
        walk = [int(k) for k in keys[o][(d[o] <= w) if w >= 0 else slice(None)]]
        room = [int(x) for x in room]
        teams = [[] for _ in room]
        for k in walk:
            for b in pbin.get((q, k), []):
                if placed[b]:
                    continue
                s = len(parties[b][0])
                j = next((j for j in range(len(room)) if room[j] >= s), None)
                if j is not None:
                    room[j] -= s
                    teams[j] += [int(x) for x in parties[b][0]]
                    placed[b] = True
        for j in range(len(room)):
            need = room[j]
            for k in walk:
                if not need:
                    break
                run = sbin.get((q, k), [])
                u = used.get((q, k), 0)
                n = min(need, len(run) - u)
                teams[j] += [int(sid[x]) for x in run[u:u + n]]
                used[(q, k)] = u + n
                need -= n
        filled.append([len(x) for x in teams])
        members.append(teams)
    return filled, members


def both(cfg, solos, parties, reqs):
    a = restate_plain(cfg, solos, parties, reqs)
    b = restate_bins(cfg, solos, parties, reqs)
    assert a == b
    return a


def one_mode(pkg, teams=2, team_size=5, groups=((0, 3000),), default_group=-1):
    cfg = cfg_of(pkg, RATING, groups=list(groups), default_group=default_group, modes=1)
    cfg.modes[0].teams, cfg.modes[0].team_size = teams, team_size
    return cfg


def solos_of(ratings, first=100):
    n = len(ratings)
    return np.arange(first, first + n, dtype=np.uint64), np.asarray(ratings, np.int64), np.zeros(n, np.int64)


def pty(first, ratings, mode=0):
    return (list(range(first, first + len(ratings))), list(ratings), mode)


# ================================================================================ CPU: the definition, hand-built
def test_parties_first_then_solos_team_by_team(pkg):
    cfg = one_mode(pkg)
    parties = [pty(0, [1500] * 3), pty(10, [1500] * 2), pty(20, [1490] * 4)]
    solos = solos_of([1500, 1520, 1480, 1400])
    filled, mem = both(cfg, solos, parties, [(0, 0, 1500, [4, 5], -1)])
    # 1500 x3 -> team 0 (room 4), 1500 x2 -> team 1, 1490 x4 fits nowhere (1 and 3 left); then the solos by distance,
    # 1480 before 1520: team 0 takes one, team 1 the next three
    assert mem[0] == [[0, 1, 2, 100], [10, 11, 102, 101, 103]] and filled == [[4, 5]]


def test_ties_go_to_the_lower_rating_then_the_older_party(pkg):
    cfg = one_mode(pkg, teams=4, team_size=2)
    parties = [pty(0, [110, 110]), pty(10, [90, 90]), pty(20, [100, 100]), pty(30, [90, 90]), pty(40, [100, 100])]
    solos = solos_of([110, 90, 100, 90])
    filled, mem = both(cfg, solos, parties, [(0, 0, 100, [2, 2, 2, 2], -1)])
    assert mem[0] == [[20, 21], [40, 41], [10, 11], [30, 31]]  # 100 older first, then 90 before 110
    filled, mem = both(cfg, solos, [], [(0, 0, 100, [1, 1, 1, 1], -1)])
    assert mem[0] == [[102], [101], [103], [100]]


def test_window_edge_is_inclusive(pkg):
    cfg = one_mode(pkg)
    parties = [pty(0, [105, 105]), pty(10, [94, 94])]
    solos = solos_of([95, 106])
    filled, mem = both(cfg, solos, parties, [(0, 0, 100, [5, 5], 5)])
    assert mem[0] == [[0, 1, 100], []] and filled == [[3, 0]]
    filled, mem = both(cfg, solos, parties, [(0, 0, 100, [5, 5], 0)])
    assert filled == [[0, 0]]


def test_a_party_that_fits_no_team_is_skipped_and_a_later_one_fits(pkg):
    cfg = one_mode(pkg, teams=2, team_size=5)
    parties = [pty(0, [100] * 4), pty(10, [100] * 2)]
    filled, mem = both(cfg, solos_of([100] * 3), parties, [(0, 0, 100, [2, 3], -1)])
    assert mem[0] == [[10, 11], [100, 101, 102]]  # the 4 fits neither team; the 2 takes team 0
    assert both(cfg, solos_of([]), parties, [(0, 0, 100, [0, 1], -1)]) == ([[0, 0]], [[[], []]])


def test_a_queue_without_parties_is_plain_backfill(pkg):
    cfg = one_mode(pkg, groups=((0, 99), (100, 200)))
    parties = [pty(0, [150, 150])]  # group 1
    solos = solos_of([10, 50, 20, 30, 40])
    reqs = [(0, 0, 25, [2, 1], -1), (0, 0, 25, [1, 2], 15)]
    filled, mem = both(cfg, solos, parties, reqs)
    n, want = bf_restate(cfg, solos[0], solos[1], solos[2], [np.array(x) for x in zip(*[(m, g, t, sum(r), w)
                                                                                         for m, g, t, r, w in reqs])])
    assert [sum(f) for f in filled] == n.tolist()
    assert [[x for tm in r for x in tm] for r in mem] == [w.tolist() for w in want]


def test_requests_on_one_queue_consume_in_order(pkg):
    cfg = one_mode(pkg, teams=2, team_size=3)
    parties = [pty(0, [100, 100]), pty(10, [101, 101, 101]), pty(20, [99, 99])]
    solos = solos_of([100, 100, 102])
    filled, mem = both(cfg, solos, parties, [(0, 0, 100, [3, 0], -1), (0, 0, 100, [2, 3], -1),
                                             (0, 0, 100, [3, 3], -1)])
    assert mem == [[[0, 1, 100], []], [[20, 21], [10, 11, 12]], [[101, 102], []]]
    assert filled == [[3, 0], [2, 3], [2, 0]]


def test_default_group_clamps_the_party_rating(pkg):
    cfg = one_mode(pkg, groups=((0, 99), (100, 199)), default_group=1)
    # a party of mean -30 and one of mean 5000 sit in the default group at the clamped ratings -1 and 200
    parties = [pty(0, [-40, -20]), pty(10, [5000, 5000]), pty(20, [150, 150])]
    solos = solos_of([-7, 250, 160])
    filled, mem = both(cfg, solos, parties, [(0, 1, 10_000, [5, 0], -1), (0, 1, -1000, [2, 1], 0)])
    assert mem[0] == [[10, 11, 20, 21, 101], []]  # 200, then 150; the party at -1 fits no more
    assert mem[1] == [[0, 1], [100]] and filled == [[5, 0], [2, 1]]


def test_overlapping_groups_use_rating_distances(pkg):
    cfg = one_mode(pkg, groups=((0, 1000), (400, 600), (0, 2000)))
    # group 2 holds 1001..2000 (first match): its parties at 1001 and 1500, nearer by rating than by key index
    parties = [pty(0, [1500, 1500]), pty(10, [1001, 1001]), pty(20, [500, 500])]
    filled, mem = both(cfg, solos_of([1002, 300]), parties, [(0, 2, 300, [2, 1], -1), (0, 0, 450, [4, 1], 200)])
    assert mem == [[[10, 11], [100]], [[20, 21, 101], []]]


@pytest.mark.parametrize("teams", [3, 256])
def test_modes_of_many_teams(pkg, teams):
    cfg = one_mode(pkg, teams=teams, team_size=3)
    parties = [pty(10 * k, [100 + k] * (2 + k % 2)) for k in range(teams + 2)]
    solos = solos_of([100] * (teams + 5), first=100_000)
    room = [3] * teams
    filled, mem = both(cfg, solos, parties, [(0, 0, 100, room, -1)])
    assert all(f == 3 for f in filled[0])
    assert mem[0][0][:2] == [0, 1] and len(set(x for tm in mem[0] for x in tm)) == 3 * teams


@pytest.mark.parametrize("seed", range(6))
def test_binned_restatement_equals_the_plain_one(pkg, seed):
    rng = np.random.default_rng(seed)
    groups = [[(0, 99), (100, 299)], [(0, 200), (50, 120), (0, 400)], [(10, 60)]][seed % 3]
    cfg = cfg_of(pkg, RATING, groups=groups, default_group=len(groups) - 1 if seed % 2 else -1, modes=3)
    n = 300
    rating = rng.integers(-30, 450, n)
    mode = rng.integers(0, cfg.n_modes, n)
    keep = np.array([group_of(cfg, int(r)) >= 0 for r in rating])
    solos = (np.arange(n, dtype=np.uint64)[keep], rating[keep], mode[keep])
    parties = []
    for k in range(80):
        m = int(rng.integers(0, cfg.n_modes))
        S = cfg.modes[m].team_size
        if S < 2:
            continue
        s = int(rng.integers(2, S + 1))
        r = int(rng.integers(-30, 450)) + rng.integers(-10, 11, s)
        if group_of(cfg, party_rating(r)) >= 0:
            parties.append((list(range(1000 + 10 * k, 1000 + 10 * k + s)), r.tolist(), m))
    reqs = []
    for _ in range(50):
        m = int(rng.integers(0, cfg.n_modes))
        md = cfg.modes[m]
        reqs.append((m, int(rng.integers(0, len(groups))), int(rng.integers(-50, 500)),
                     rng.integers(0, md.team_size + 1, md.teams).tolist(),
                     -1 if rng.random() < 0.4 else int(rng.integers(0, 40))))
    both(cfg, solos, parties, reqs)


def test_abi_mirror(pkg):
    res, args = pkg.abi.PROTOTYPES["mm_backfill_party"]
    assert res is C.c_int and len(args) == 9


# ================================================================================ CPU: SearchPool.backfill_teams
def backfill_engine(pkg, calls):
    class Eng(party_requeue_engine(pkg, calls)):
        """The party engine double with backfill_party by the plain restatement over its pool and table."""

        def backfill_party(self, mode, group, target, room, window):
            calls.append("backfill_party")
            p = self.pool_read()
            parties = [(q[0], q[1], q[2]) for q in self.parties]
            self.seq_of.update((int(x), q[4]) for q in self.parties for x in q[0])
            reqs = list(zip(np.asarray(mode).tolist(), np.asarray(group).tolist(), np.asarray(target).tolist(), room,
                            np.asarray(window).tolist()))
            filled, mem = restate_plain(self.cfg, (p["id"], p["rating"], p["mode"]), parties, reqs)
            placed = {x for r in mem for tm in r for x in tm}
            solos = np.array([x for x in placed if x not in {y for q in self.parties for y in q[0]}], np.uint64)
            self.parties = [q for q in self.parties if q[0][0] not in placed]
            self.take(solos)
            return filled, [[np.array(tm, np.uint64) for tm in r] for r in mem]

    return Eng


def test_search_pool_backfill_teams_flow(pkg):
    from .test_expire import publish
    from .test_parties import publish_party
    calls = []
    sw, eng, pool, broker, calls = requeue_pool(pkg, calls=calls, engine=backfill_engine(pkg, calls)(
        pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=RATING, capacity=1000, active_capacity=4000)))
    cfg = eng.cfg
    for i, r in enumerate([100, 120, 130]):
        publish(pkg, broker, cfg, f"s{i}", r, mode="5v5")
    publish_party(pkg, broker, sw, "bronze", [(f"a{i}", 100) for i in range(3)], "5v5")
    publish_party(pkg, broker, sw, "bronze", [(f"b{i}", 110) for i in range(2)], "5v5")
    broker.deliver_all()
    assert len(pool._staged) == 3 and len(pool._staged_parties) == 2
    out = pool.backfill_teams([("5v5", "bronze", 100, [3, 4]), ("5v5", "bronze", 100, [1, 0], 5)])
    assert not pool._staged and not pool._staged_parties  # staged deliveries flushed first
    assert [[[d["id"] for d in tm] for tm in r] for r in out] == [[["a0", "a1", "a2"], ["b0", "b1", "s0", "s1"]],
                                                                  [[], []]]
    assert calls[-1] == "backfill_party" and pool.stats["backfilled_teams"] == 7
    h = pool.handles.lookup
    assert all(h(f"a{i}") in pool.matched_parties for i in range(3)) and h("a0") not in pool.party_of
    assert not pool.party_book and eng.pool_size() == 1 and pool.in_queue("s2")
    assert all(eng.in_queue([h(x)])[0] for x in ("a0", "b1", "s0"))  # matched players stay active
    # the lobby did not start: party a goes back whole, party b and the solos too
    assert pool.requeue(out[0][0] + out[0][1]) == ["requeued"] * 7
    assert ("requeue_party", [3, 2]) in calls
    assert [q[0] for q in eng.parties] == [[h(f"a{i}") for i in range(3)], [h(f"b{i}") for i in range(2)]]
    assert pool.backfill_teams([]) == []


# ================================================================================ GPU: against the restatement
def pbf_requests(rng, cfg, n, lo=-200, hi=5300, full=0.5):
    """n random requests: (mode, group, target, room list, window) tuples"""
    out = []
    for _ in range(n):
        m = int(rng.integers(0, cfg.n_modes))
        md = cfg.modes[m]
        room = np.where(rng.random(md.teams) < full, md.team_size, rng.integers(0, md.team_size + 1, md.teams))
        out.append((m, int(rng.integers(0, cfg.n_groups)), int(rng.integers(lo, hi)), room.tolist(),
                    -1 if rng.random() < 0.4 else int(rng.integers(0, 80))))
    return out


def call(eng, reqs):
    cols = [np.array([r[k] for r in reqs], np.int64) for k in (0, 1, 2, 4)]
    return eng.backfill_party(cols[0], cols[1], cols[2], [r[3] for r in reqs], cols[3])


def check_call(eng, cfg, reqs):
    """mm_backfill_party against the restatement of mm_pool_read / mm_party_read; the pool and the table after it lose
    exactly what it took.  -> (the solos taken, the party members taken)"""
    p = eng.pool_read()
    parties = party_state(eng)
    want_f, want_m = restate_bins(cfg, (p["id"], p["rating"], p["mode"]), [q[:3] for q in parties], reqs)
    got_f, got_m = call(eng, reqs)
    assert got_f == want_f
    for g, w in zip(got_m, want_m):
        assert [t.tolist() for t in g] == w
    flat = np.array([x for r in want_m for tm in r for x in tm], np.uint64)
    pm = set(int(x) for q in parties for x in q[0])
    solo = np.array([x for x in flat.tolist() if x not in pm], np.uint64)
    pmem = np.array([x for x in flat.tolist() if x in pm], np.uint64)
    after = eng.pool_read()
    keep = ~np.isin(p["id"], solo)
    for k in p:
        assert np.array_equal(after[k], p[k][keep]), k
    left = [q for q in parties if not np.isin(q[0], pmem).any()]
    now = party_state(eng)
    assert len(now) == len(left) and all(np.array_equal(a[0], b[0]) for a, b in zip(now, left))
    if len(flat):
        assert eng.in_queue(flat).all()
        assert (eng.locate(flat, 0)["state"] == 2).all()
    return solo, pmem


def party_pool(pkg, cfg, kind, seed, n_solos, n_parties, lo=0, hi=5001, cap=200_000):
    src = PartySrc(pkg, cfg, kind, seed, cap=cap)
    src.enqueue(*src.fresh(n_solos, lo, hi))
    if n_parties:
        sizes, ids, rat, mode, ts = src.fresh_parties(n_parties, lo, hi)
        assert (src.eng.enqueue_party(sizes, ids, rat, mode, ts) == 1).all()
    return src


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
@pytest.mark.parametrize("layout", ["split", "wide", "overlap"])
def test_engine_equals_the_restatement(pkg, kind, layout):
    cfg = gpu_config(pkg, RATING, kind, layout)
    lo, hi = (-300, 5400) if layout == "overlap" else (0, 5001)
    src = party_pool(pkg, cfg, kind, 31, 40_000, 3000, lo, hi)
    rng = np.random.default_rng(4)
    try:
        check_call(src.eng, cfg, pbf_requests(rng, cfg, 300))
        src.eng.tick(src.now)  # after a tick, with dead rows from the call and more parties
        sizes, ids, rat, mode, ts = src.fresh_parties(1000, lo, hi)
        assert (src.eng.enqueue_party(sizes, ids, rat, mode, ts) == 1).all()
        check_call(src.eng, cfg, pbf_requests(rng, cfg, 500, full=0.9))
        check_call(src.eng, cfg, pbf_requests(rng, cfg, 50, full=1.0) * 4)  # repeated requests drain their queues
    finally:
        src.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True], ids=["hashed", "dense"])
def test_party_table_of_many_tiles_with_a_crowded_bin(pkg, dense):
    cfg = pkg.synth.make_config(groups=[(0, 999), (1000, 1999)], modes=[("2v2", 2, 2), ("5v5", 2, 5)], order=RATING,
                                capacity=100_000, active_capacity=400_000, default_group=-1,
                                flags=DENSE if dense else 0)
    src = PartySrc(pkg, cfg, "dense" if dense else "hashed", 3, cap=60_000)
    rng = np.random.default_rng(8)
    try:
        src.enqueue(*src.fresh(20_000, 0, 2000))
        k = 4000  # more than three tiles of 1024 rows; half of them on one rating
        sizes = rng.integers(2, 6, k).astype(np.uint8)
        mode = np.where(sizes > 2, 1, rng.integers(0, 2, k)).astype(np.uint8)
        ids = src.fresh(int(sizes.sum()), 0, 2000)[0]
        base = np.where(rng.random(k) < 0.5, 700, rng.integers(0, 2000, k))
        rat = np.repeat(base, sizes).astype(np.int32)
        assert (src.eng.enqueue_party(sizes, ids, rat, mode, np.zeros(k, np.uint32)) == 1).all()
        reqs = [(1, 0, 700, [5, 5], -1)] * 200 + [(0, 0, 700, [2, 2], 0)] * 100 + pbf_requests(rng, cfg, 300, 0, 2000)
        check_call(src.eng, cfg, reqs)
    finally:
        src.close()


# ================================================================================ GPU: mixed schedules
class PbfModel(RequeueModel):
    """RequeueModel with mm_backfill_party."""

    def backfill_party(self, reqs):
        p = self.pool()
        parties = [(q[0], q[1], q[2]) for q in self.parties]
        filled, mem = restate_bins(self.cfg, (p["id"], p["rating"], p["mode"]), parties, reqs)
        flat = set(x for r in mem for tm in r for x in tm)
        placed = [bool(len(q[0])) and int(q[0][0]) in flat for q in self.parties]
        pm = [q for q, k in zip(self.parties, placed) if k]
        self.matched_parties += pm
        self.party_matched = np.concatenate([self.party_matched] + [q[0] for q in pm])
        self.parties = [q for q, k in zip(self.parties, placed) if not k]
        inp = set(int(x) for q in pm for x in q[0])
        self.take(np.array([x for x in flat if x not in inp], np.uint64))
        return filled, mem


class PbfSchedule(RequeueSchedule):
    """RequeueSchedule on the PbfModel, with a backfill_party step."""

    def __init__(self, pkg, oracle, cfg, rng, dense, **k):
        super().__init__(pkg, oracle, cfg, rng, dense, **k)
        self.m = PbfModel(cfg, oracle, pkg.abi)
        self.setup(self.eng)

    def backfill_party(self, reqs=None):
        reqs = pbf_requests(self.rng, self.cfg, int(self.rng.integers(1, 400)), self.lo - 200, self.hi + 200) \
            if reqs is None else reqs
        want_f, want_m = self.m.backfill_party(reqs)
        got_f, got_m = call(self.eng, reqs)
        assert got_f == want_f
        for g, w in zip(got_m, want_m):
            assert [t.tolist() for t in g] == w
        self.count("backfill_party")
        return got_f, got_m

    OPS = RequeueSchedule.OPS + ["backfill_party", "backfill_party"]


@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True], ids=["hashed", "dense"])
@pytest.mark.parametrize("wide", [False, True], ids=["split", "wide"])
def test_mixed_schedule_with_party_backfill(pkg, oracle, dense, wide):
    rng = np.random.default_rng(900 + 2 * dense + wide)
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[:3], order=RATING, capacity=300_000,
                                active_capacity=4_000_000, default_group=-1,
                                flags=(DENSE if dense else 0) | (WIDE if wide else 0))
    s = PbfSchedule(pkg, oracle, cfg, rng, dense)
    try:
        s.players(60_000, old=0.02)
        s.party_batch(800)
        s.check()
        for _ in range(2 * len(s.OPS)):
            s.step()
        s.tick()
        s.finish()
        s.check()
    finally:
        s.close()
    c = s.counts
    for what in ("backfill_party", "requeue_party", "party_match", "checkpoint"):
        assert c.get(what, 0) >= 2, (what, c)


# ================================================================================ GPU: the EQUIVALENCE
@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True], ids=["hashed", "dense"])
def test_twin_engine_of_the_equivalence(pkg, oracle, dense):
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[:3], order=RATING, capacity=200_000,
                                active_capacity=1_000_000, default_group=-1, flags=DENSE if dense else 0)
    s = PbfSchedule(pkg, oracle, cfg, np.random.default_rng(17 + dense), dense, pcap=50_000)
    twin = None
    try:
        s.players(40_000)
        s.party_batch(1500)
        s.tick()
        s.check()
        pimg = s.eng.export_parties()
        img = s.eng.export_state()
        assert (s.eng.merge_parties(pimg, keep_seq=True) == 1).all()
        pm_before = set(s.m.party_members().tolist())
        _f, mem = s.backfill_party(pbf_requests(s.rng, cfg, 300, full=0.9))
        s.check()
        flat = np.array([x for r in mem for tm in r for x in tm.tolist()], np.uint64)
        placed = np.array([x for x in flat.tolist() if x in pm_before], np.uint64)
        solos = np.array([x for x in flat.tolist() if x not in pm_before], np.uint64)
        assert len(placed) and len(solos)
        pimg2, img2 = strip_images(pkg, pimg, img, placed)
        twin = pkg.Engine(cfg)
        twin.import_state(img2)
        twin.set_option("party_capacity", s.pcap)
        assert (twin.merge_parties(pimg2, keep_seq=True) == 1).all()
        assert twin.take(solos) == len(solos)
        a, b = s.eng, twin
        probe = np.concatenate([flat[::5], s.m.party_members()[::7], s.m.active[::101]])
        rules = {(m, g): (0, 20, 5, 5, 200) for m in range(cfg.n_modes) for g in range(cfg.n_groups)}
        from .test_widen import rules_of
        rng = np.random.default_rng(5)
        for step in range(5):
            now = s.now + 40 * step
            pa, pb = a.party_read(), b.party_read()
            for k in ("size", "seq", "enq_ts", "mode", "group", "rating"):
                assert np.array_equal(pa[k], pb[k]), k
            assert all(np.array_equal(x[0], y[0]) for x, y in zip(pa["members"], pb["members"]))
            assert a.seq_next() == b.seq_next() and a.active_size() == b.active_size()
            assert np.array_equal(a.locate(probe, now), b.locate(probe, now))
            assert np.array_equal(a.in_queue(probe), b.in_queue(probe))
            reqs = pbf_requests(rng, cfg, 100)
            fa, ma = call(a, reqs)
            fb, mb = call(b, reqs)
            assert fa == fb and all(np.array_equal(x, y) for r, q in zip(ma, mb) for x, y in zip(r, q))
            ra, rb = a.party_match(now, rules_of(cfg, rules)), b.party_match(now, rules_of(cfg, rules))
            assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1])
            ta, tb = a.tick(now), b.tick(now)
            for x, y in zip(ta[:3], tb[:3]):
                assert np.array_equal(x, y)
            back = solos[step::5]
            assert np.array_equal(a.requeue(*requeue_cols(s, back)), b.requeue(*requeue_cols(s, back)))
            pa, pb = a.pool_read(), b.pool_read()
            for k in pa:
                assert np.array_equal(pa[k], pb[k]), k
    finally:
        if twin is not None:
            twin.close()
        s.close()


def requeue_cols(s, ids):
    r, md, ts, seq = np.array([s.m.book[int(x)] for x in ids.tolist()], np.int64).reshape(-1, 4).T
    return ids, r.astype(np.int32), md.astype(np.uint8), ts.astype(np.uint32), seq.astype(np.uint32)


def strip_images(pkg, pimg, img, placed):
    """The placed parties out of the party image; their members into section 7 of the engine image (the taken solos
    follow by mm_take, mm_backfill's EQUIVALENCE).  -> (party image, engine image)"""
    ab = pkg.abi
    ph, pc = pkg.engine.read_party_image(pimg)
    cut = np.cumsum(pc["size"].astype(np.int64))[:-1]
    ids = np.split(pc["id"], cut)
    rats = np.split(pc["rating"], cut)
    keep = [j for j, a in enumerate(ids) if not np.isin(a.astype(np.uint64), placed).any()]
    P, M = len(keep), int(sum(len(ids[j]) for j in keep))
    off = ab.party_image_offsets(P, M, ph.id_bytes)
    out = np.zeros(off[-1], np.uint8)
    h2 = ab.ImageHeader.from_buffer_copy(ph)
    h2.n_parts, h2.n_players, h2.total_bytes = P, M, off[-1]
    out[:C.sizeof(h2)] = np.frombuffer(bytes(h2), np.uint8)
    secs = [pc["size"][keep], pc["seq"][keep], pc["enq_ts"][keep], pc["mode"][keep],
            np.concatenate([ids[j] for j in keep]) if keep else np.zeros(0, pc["id"].dtype),
            np.concatenate([rats[j] for j in keep]) if keep else np.zeros(0, np.int32)]
    for k, a in enumerate(secs):
        b = np.ascontiguousarray(a).view(np.uint8)
        out[off[k]:off[k] + len(b)] = b
    img = np.array(img, np.uint8, copy=True)
    h, cols = pkg.engine.read_image(img)
    active = np.concatenate([cols["active"], np.asarray(placed).astype(cols["active"].dtype)])
    o = ab.image_offsets(h.n_parts, h.n_players, len(active), h.id_bytes)
    e = np.zeros(o[-1], np.uint8)
    e[:o[-2]] = img[:o[-2]]
    h3 = ab.ImageHeader.from_buffer_copy(h)
    h3.n_active, h3.total_bytes = len(active), o[-1]
    e[:C.sizeof(h3)] = np.frombuffer(bytes(h3), np.uint8)
    b = np.ascontiguousarray(active).view(np.uint8)
    e[o[-2]:o[-2] + len(b)] = b
    return out, e


# ================================================================================ GPU: party-free queues, round trip
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
def test_party_free_queues_equal_backfill(pkg, kind):
    cfg = gpu_config(pkg, RATING, kind, "split")
    src = party_pool(pkg, cfg, kind, 41, 30_000, 0)
    b = pkg.Engine(cfg)
    rng = np.random.default_rng(6)
    try:
        b.import_state(src.eng.export_state())
        reqs = pbf_requests(rng, cfg, 400)
        filled, mem = call(src.eng, reqs)
        n, got = b.backfill(*(np.array(c, np.int64) for c in zip(*[(r[0], r[1], r[2], sum(r[3]), r[4])
                                                                   for r in reqs])))
        assert [sum(f) for f in filled] == n.tolist()
        for r, g in zip(mem, got):
            assert np.array_equal(np.concatenate(r), g)
        for now in (10, 20):
            ta, tb = src.eng.tick(now), b.tick(now)
            for x, y in zip(ta[:3], tb[:3]):
                assert np.array_equal(x, y)
        pa, pb = src.eng.pool_read(), b.pool_read()
        for k in pa:
            assert np.array_equal(pa[k], pb[k]), k
        assert src.eng.active_size() == b.active_size()
    finally:
        b.close()
        src.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True], ids=["hashed", "dense"])
def test_round_trip_through_requeue_party_and_requeue(pkg, oracle, dense):
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[:3], order=RATING, capacity=200_000,
                                active_capacity=1_000_000, default_group=-1, flags=DENSE if dense else 0)
    s = PbfSchedule(pkg, oracle, cfg, np.random.default_rng(23 + dense), dense, pcap=50_000)
    try:
        s.players(30_000)
        s.party_batch(1200)
        s.tick()
        s.check()
        pimg = s.eng.export_parties()
        before = export_sections(pkg, s.eng)
        assert (s.eng.merge_parties(pimg, keep_seq=True) == 1).all()
        pm = {int(x): q for q in s.m.parties for x in q[0]}
        _f, mem = s.backfill_party(pbf_requests(s.rng, cfg, 300, full=0.9))
        flat = [x for r in mem for tm in r for x in tm.tolist()]
        parties = list({id(pm[x]): pm[x] for x in flat if x in pm}.values())
        solos = np.array([x for x in flat if x not in pm], np.uint64)
        assert parties and len(solos)
        parties.sort(key=lambda q: (q[4] - s.m.seq_next) & U32)
        s.requeue_party([tuple(q) for q in parties], expect=[1] * len(parties))
        assert (s.eng.requeue(*requeue_cols(s, solos)) == 1).all()
        pimg2 = s.eng.export_parties()
        after = export_sections(pkg, s.eng)
        assert np.array_equal(np.frombuffer(pimg, np.uint8), np.frombuffer(pimg2, np.uint8))
        assert before[0] == after[0] and np.array_equal(before[2], after[2])
        for k in before[1]:
            assert np.array_equal(before[1][k], after[1][k]), k
    finally:
        s.close()


# ================================================================================ GPU: refusals
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
def test_refusals_change_nothing(pkg, kind):
    ab = pkg.abi
    cfg = pkg.synth.make_config(groups=[(0, 999), (1000, 1999)], modes=[("2v2", 2, 2), ("5v5", 2, 5), ("300", 300, 1)],
                                order=RATING, capacity=50_000, active_capacity=200_000, default_group=-1,
                                flags=DENSE if kind == "dense" else 0)
    src = party_pool(pkg, cfg, kind, 5, 5000, 400, 0, 2000, cap=5000)
    e = src.eng
    probe = np.concatenate([e.pool_read()["id"][::50], np.concatenate([q[0] for q in party_state(e)])[::7]])
    try:
        def state():
            pr = e.party_read()
            return (e.pool_read()["id"].tolist(), e.active_size(), e.in_queue(probe).tolist(), pr["seq"].tolist(),
                    [x[0].tolist() for x in pr["members"]], e.seq_next(), e.locate(probe, 0).tolist())

        def raw(reqs, room, cap=1 << 16, null=None):
            req = np.zeros(len(reqs), np.dtype([("mode", "u1"), ("group", "u1"), ("reserved", "<u2"),
                                                ("count", "<u4"), ("target", "<i4"), ("window", "<i4")]))
            for i, r in enumerate(reqs):
                req[i] = r
            room = np.asarray(room + [0], np.uint16)
            filled = np.full(len(room), 77, np.uint16)
            n_taken = np.full(max(len(reqs), 1), 77, np.uint32)
            mem = np.empty(max(cap, 1), np.uint64)
            total = C.c_uint32(99)
            args = [req.ctypes.data, room.ctypes.data, filled.ctypes.data, n_taken.ctypes.data]
            if null is not None:
                args[null] = None
            rc = e.lib.mm_backfill_party(e.h, len(reqs), *args, mem.ctypes.data, cap, C.byref(total))
            return rc, filled[:-1], n_taken[:len(reqs)], total.value, e.lib.mm_last_error(e.h).decode()

        before = state()
        ok, okr = (1, 0, 0, 10, 500, -1), [5, 5]
        for bad, room, text in (((3, 0, 0, 1, 0, -1), [1], "mode"), ((0, 7, 0, 2, 0, -1), [1, 1], "group"),
                                ((0, 0, 1, 2, 0, -1), [1, 1], "reserved"), ((0, 0, 0, 3, 0, -1), [3, 0], "team_size"),
                                ((1, 0, 0, 9, 0, -1), [5, 5], "sum"), ((2, 0, 0, 0, 0, -1), [0] * 300, "teams")):
            rc, _f, _n, total, msg = raw([ok, bad], okr + room)
            assert rc == ab.MM_E_ARG and total == 0 and "request 1" in msg and text in msg, msg
            assert state() == before
        for k in range(4):
            rc, *_ = raw([ok], okr, null=k)
            assert rc == ab.MM_E_ARG and state() == before
        # a dry run answers the counts and takes nothing; one less than the total is refused too
        reqs = [(m, g, 0, 4 if m == 0 else 10, 500 + 1000 * g, -1) for m in range(2) for g in range(2)] * 3
        room = [x for r in reqs for x in ([2, 2] if r[0] == 0 else [5, 5])]
        rc, filled, n_taken, total, msg = raw(reqs, room, cap=0)
        assert rc == ab.MM_E_CAP and total == n_taken.sum() > 0 and "member_cap" in msg
        assert n_taken.tolist() == filled.reshape(-1, 2).sum(1).tolist()
        assert state() == before
        rc2, f2, n2, total2, _ = raw(reqs, room, cap=total - 1)
        assert rc2 == ab.MM_E_CAP and total2 == total and np.array_equal(n2, n_taken) and np.array_equal(f2, filled)
        assert state() == before
        assert raw([], [])[0] == 0 and state() == before
        if kind == "dense":  # a staged packed batch (MM_E_STATE)
            e.enqueue_packed_begin(np.array([src.fresh(1)[0][0]], np.uint32), e.pack_key([100], [1]))
            rc, *_, msg = raw([ok], okr)
            assert rc == ab.MM_E_STATE and "staged" in msg
            e.enqueue_packed_end()
    finally:
        src.close()
    # no party capacity, MM_F_NO_DEDUPE (MM_E_STATE); arrival order (MM_E_ARG)
    for flags, order, cap, status in ((0, RATING, 0, ab.MM_E_STATE), (1, RATING, 100, ab.MM_E_STATE),
                                      (0, ARRIVAL, 100, ab.MM_E_ARG)):
        c = pkg.synth.make_config(groups=[(0, 999)], modes=[("2v2", 2, 2)], order=order, capacity=1000,
                                  active_capacity=4000, default_group=-1, flags=flags)
        with pkg.Engine(c) as eng:
            if cap:
                eng.set_option("party_capacity", cap)
            with pytest.raises(pkg.EngineError) as ei:
                eng.backfill_party(0, 0, 0, [1, 1])
            assert ei.value.status == status


# ================================================================================ GPU: scale
@pytest.mark.gpu
def test_config3_ten_million_solos_and_200k_parties(pkg):
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=[("5v5", 2, 5)], order=RATING,
                                capacity=10_500_000, active_capacity=12_000_000)
    rng = np.random.default_rng(2)
    with pkg.Engine(cfg) as eng:
        eng.set_option("party_capacity", 1_000_000)
        n = 10_000_000
        ids = np.arange(n, dtype=np.uint64) + np.uint64(1 << 40)
        eng.enqueue(ids, rng.integers(0, 3000, n).astype(np.int32), np.zeros(n, np.uint8))
        k = 200_000
        sizes = rng.integers(2, 5, k).astype(np.uint8)
        m = int(sizes.sum())
        pid = np.arange(m, dtype=np.uint64) + np.uint64(1 << 41)
        prat = np.clip(np.repeat(rng.integers(0, 3000, k), sizes) + rng.integers(-30, 31, m), 0, 2999).astype(np.int32)
        assert (eng.enqueue_party(sizes, pid, prat, np.zeros(k, np.uint8), np.zeros(k, np.uint32)) == 1).all()
        for nr in (1000, 4000):
            p = eng.pool_read()
            parties = party_state(eng)
            reqs = pbf_requests(rng, cfg, nr, 0, 3000)
            filled, mem = call(eng, reqs)
            for g in (0, 3):  # a sample of queues against the restatement
                sel = [j for j, r in enumerate(reqs) if r[1] == g]
                ssel = np.array([group_of(cfg, int(x)) == g for x in p["rating"]])
                psel = [q[:3] for q in parties if group_of(cfg, party_rating(q[1])) == g]
                wf, wm = restate_bins(cfg, (p["id"][ssel], p["rating"][ssel], p["mode"][ssel]), psel,
                                      [reqs[j] for j in sel])
                assert [filled[j] for j in sel] == wf
                assert [[t.tolist() for t in mem[j]] for j in sel] == wm
