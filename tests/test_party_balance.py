"""Balanced party lobbies (mm_set_option("party_balance"), SearchPool(balance_parties=...)): every mm_party_match lobby
of a masked two-team mode is split into its most even teams, every party kept whole.

Two independent restatements of the rule (include/mm_engine.h): `psplit_plain` enumerates the team-1 sets with
itertools and skips the ones that cut a party, `psplit_numpy` scores every lobby against test_team_balance's table of
all masks and filters it by the continuation test.
CPU: the restatements agree on every S from 2 to 8 and every way a lobby splits into parties and solos; the result is
never worse than the lobby as formed, never cuts a party, and is split_plain's answer whenever that one keeps every
party whole; the known answers; SearchPool's mask.
GPU: twin engines with and without the mask through one schedule of party enqueues, solos, party match, ticks,
removes, expires and party requeues (hashed and dense ids; split, wide and overlapping groups; member ratings clamped
at both key ends); one masked mode among unmasked ones and a three-team mode; party_balance beside team_balance; the
option on, then off; the dry run and the MM_E_CAP refusal; every refusal of the option; a party table of more than
3 x 1024 rows; EngineModel with the restatement over a long mixed schedule; SearchPool end to end.
"""
import ctypes as C
import importlib
import itertools

import numpy as np
import pytest

from .test_backfill import clamp_bounds, gpu_config
from .test_engine_model import EngineModel, EngineSchedule, hdr, party_batch_of
from .test_parties import party_rules, publish_party
from .test_team_balance import OptionEngine, imbalance_of, mask_table, split_numpy, split_plain
from .test_tile_geometry import DENSE, MODES8, WIDE
from .test_widen import RATING, rules_of

sw = importlib.import_module("microservice-matchmaking_b200.search_worker")
eng_mod = importlib.import_module("microservice-matchmaking_b200.engine")
abi = importlib.import_module("microservice-matchmaking_b200.abi")


# ================================================================================ restatements
def cont_of(parts):
    """parts: the lobby's member runs in order, a party of s members as s, a solo as 1 -> the continuation word"""
    cont, i = 0, 0
    for s in parts:
        for j in range(1, s):
            cont |= 1 << (i + j)
        i += s
    return cont


def psplit_plain(c, S, cont):
    """c: the L = 2S values in the lobby's formed order -> (new member order as old indices, imbalance); only sets
    that hold every party whole or not at all."""
    L = len(c)
    c = [int(x) for x in c]
    total = sum(c)
    best = None
    for rest in itertools.combinations(range(1, L), S - 1):
        a = (0,) + rest
        if any(((cont >> i) & 1) and ((i in a) != (i - 1 in a)) for i in range(1, L)):
            continue
        d = abs(2 * sum(c[i] for i in a) - total)
        m = sum(1 << i for i in rest)
        if best is None or (d, m) < best[:2]:
            best = (d, m, a)
    d, _m, a = best
    return list(a) + [i for i in range(L) if i not in a], d


_MASKS = {}


def psplit_numpy(c, S, cont):
    """c: int[n, 2S], cont: int[n] -> (perm int[n, 2S] of old indices, imbalance int64[n]), vectorised over lobbies."""
    c = np.asarray(c, np.int64)
    cont = np.asarray(cont, np.int64)
    t = mask_table(S)
    if S not in _MASKS:
        _MASKS[S] = (t.astype(np.int64) << np.arange(2 * S)).sum(1)
    m = _MASKS[S]
    d = np.abs(2 * (c @ t.T.astype(np.int64)) - c.sum(1, keepdims=True))
    ok = ((m ^ (m << 1))[None, :] & cont[:, None]) == 0
    d = np.where(ok, d, np.iinfo(np.int64).max)
    k = d.argmin(1)  # the first minimum = the smallest mask
    inA = t[k]
    idx = np.broadcast_to(np.arange(2 * S), c.shape)
    perm = np.concatenate([idx[inA].reshape(len(c), S), idx[~inA].reshape(len(c), S)], 1)
    return perm, d[np.arange(len(c)), k]


def balance_parties(cfg, mask, lob, mem, rating, party, plain=False):
    """The option applied to party_match's lobbies as formed.  rating(id): the member's own rating (a party member's,
    or the solo's pool rating); party(id): its party's key, None for a solo.  -> (member ids, summed imbalance)"""
    lo, hi = clamp_bounds(cfg)
    mem = np.array(mem, np.uint64, copy=True)
    total = 0
    for md in range(cfg.n_modes):
        S = cfg.modes[md].team_size
        sel = np.flatnonzero(lob["mode"] == md)
        if not (mask >> md) & 1 or S < 2 or not len(sel):
            continue
        idx = lob["first_member"][sel].astype(np.int64)[:, None] + np.arange(2 * S)[None, :]
        ids = mem[idx].tolist()
        c = np.clip(np.array([[rating(x) for x in row] for row in ids], np.int64), lo, hi)
        cont = np.zeros(len(sel), np.int64)
        for k, row in enumerate(ids):
            p = [party(x) for x in row]
            cont[k] = sum(1 << i for i in range(1, 2 * S) if p[i] is not None and p[i] == p[i - 1])
        if plain:
            res = [psplit_plain(x, S, int(w)) for x, w in zip(c, cont)]
            perm, d = np.array([r[0] for r in res]), np.array([r[1] for r in res])
        else:
            perm, d = psplit_numpy(c, S, cont)
        mem[idx] = mem[np.take_along_axis(idx, perm, 1)]
        total += int(d.sum())
    return mem, total


def parties_whole(perm, S, cont):
    side = [int(i >= S) for i in np.argsort(perm)]  # old member -> its new team
    return all(side[i] == side[i - 1] for i in range(1, 2 * S) if (cont >> i) & 1)


# ================================================================================ CPU
def compositions(n):
    """every way to write n as an ordered sum of positive parts"""
    for cuts in itertools.product([0, 1], repeat=n - 1):
        parts, run = [], 1
        for k in cuts:
            if k:
                parts.append(run)
                run = 1
            else:
                run += 1
        yield parts + [run]


def lobby_shapes(S, rng, n):
    """(parts) of formed lobbies: every team a composition of S (1 = a solo), each party inside one team; all of them
    for S <= 4, else n random ones with the all-party, no-co-party and whole-team shapes."""
    comps = list(compositions(S))
    if S <= 4:
        return [a + b for a in comps for b in comps]
    out = [[S, S], [2] + [1] * (2 * S - 2), [1] * (2 * S), [S] + [1] * S, [2] * (S // 2) + [1] * (S % 2) + [S]]
    for _ in range(n):
        out.append(comps[rng.integers(len(comps))] + comps[rng.integers(len(comps))])
    return out


@pytest.mark.parametrize("S", range(2, 9))
def test_restatements_agree(S):
    rng = np.random.default_rng(40 + S)
    L = 2 * S
    shapes = lobby_shapes(S, rng, 60 if S <= 6 else 12)
    per = 3 if S <= 6 else 1
    for kind in range(4):
        rows, conts = [], []
        for parts in shapes:
            for _ in range(per):
                if kind == 0:
                    c = rng.integers(0, 5000, L)
                elif kind == 1:
                    c = rng.integers(0, 4, L)  # heavy ties
                elif kind == 2:
                    c = np.full(L, 1234)  # equal ratings
                else:
                    c = np.concatenate([np.repeat(rng.integers(1300, 1700, len(parts)), parts)])
                    c = c + rng.integers(-30, 31, L)
                rows.append(c)
                conts.append(cont_of(parts))
        c, cont = np.array(rows, np.int64), np.array(conts, np.int64)
        perm, d = psplit_numpy(c, S, cont)
        for i in range(len(c)):
            q, e = psplit_plain(c[i], S, int(cont[i]))
            assert perm[i].tolist() == q and d[i] == e
            assert parties_whole(perm[i], S, int(cont[i]))  # no party is ever split
            assert perm[i][0] == 0
            free, fd = split_plain(c[i], S)
            if parties_whole(free, S, int(cont[i])):  # the constraint does not bind: the same answer
                assert (q, e) == (free, fd)
            else:
                assert e >= fd  # an equal admissible set with a larger mask may exist
        assert np.array_equal(imbalance_of(np.take_along_axis(c, perm, 1), S), d)
        assert (d <= imbalance_of(c, S)).all()  # never worse than the lobby as formed
        # cont 0 is team_balance's rule
        p0, d0 = psplit_numpy(c, S, np.zeros(len(c), np.int64))
        q0, e0 = split_numpy(c, S)
        assert np.array_equal(p0, q0) and np.array_equal(d0, e0)


def test_known_answers():
    # 5v5: an anchor 2-stack, a 3-stack of its window on team 0, five solos on team 1 (window 50 around R = 1500)
    c = [1900, 1100, 1550, 1550, 1550, 1500, 1495, 1505, 1490, 1510]
    cont = cont_of([2, 3, 1, 1, 1, 1, 1])
    assert imbalance_of(c, 5) == 150
    perm, d = psplit_plain(c, 5, cont)
    assert [c[i] for i in perm] == [1900, 1100, 1500, 1505, 1510, 1550, 1550, 1550, 1495, 1490] and d == 120
    free, fd = split_plain(c, 5)
    assert fd == 20 and not parties_whole(free, 5, cont)
    assert 0 < len({i for i in (2, 3, 4) if i in free[:5]}) < 3  # team_balance's answer cuts the 3-stack
    # a 5-stack anchor: only the lobby as formed is admissible
    c5 = [1000, 1000, 1000, 1000, 1000, 3000, 3001, 2999, 1500, 4000]
    assert psplit_plain(c5, 5, cont_of([5, 1, 1, 1, 1, 1])) == (list(range(10)), imbalance_of(c5, 5))
    # 3v3 where the constraint does not bind
    c3 = [1400, 1600, 1500, 1490, 1510, 1520]
    cont3 = cont_of([2, 1, 1, 1, 1])
    assert imbalance_of(c3, 3) == 20
    perm, d = psplit_plain(c3, 3, cont3)
    assert [c3[i] for i in perm] == [1400, 1600, 1510, 1500, 1490, 1520] and d == 0
    assert (perm, d) == split_plain(c3, 3)
    for v, S, w in ((c, 5, cont), (c5, 5, cont_of([5, 1, 1, 1, 1, 1])), (c3, 3, cont3)):
        p, e = psplit_numpy([v], S, [w])
        assert (p[0].tolist(), e[0]) == psplit_plain(v, S, w)


def test_search_pool_sets_the_mask(pkg):
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=(("1v1", 2, 1), ("5v5", 2, 5), ("3v3", 2, 3)),
                                order=RATING, capacity=1000)
    names = pkg.synth.REFERENCE_GROUP_NAMES
    eng = OptionEngine(cfg)
    sw.SearchPool(eng, ["1v1", "5v5", "3v3"], names, balance_parties=["5v5", "1v1"])
    assert eng.options == {"party_balance": 0b011}
    eng = OptionEngine(cfg)
    sw.SearchPool(eng, ["1v1", "5v5", "3v3"], names, balance_parties=["3v3"], balance_teams=["5v5"])
    assert eng.options == {"party_balance": 0b100, "team_balance": 0b010}
    eng = OptionEngine(cfg)
    sw.SearchPool(eng, ["1v1", "5v5", "3v3"], names)
    assert "party_balance" not in eng.options  # only set when asked for
    with pytest.raises(ValueError):
        sw.SearchPool(OptionEngine(cfg), ["1v1", "5v5", "3v3"], names, balance_parties=["7v7"])


# ================================================================================ GPU
class Book:
    """What the caller keeps: every member's own rating, and each queued or matched party's record."""

    def __init__(self):
        self.rating = {}
        self.party = {}  # id -> seq of its party
        self.rec = {}    # seq -> (ids, ratings, mode, ts)

    def solos(self, ids, r):
        self.rating.update(zip(np.asarray(ids).tolist(), np.asarray(r).tolist()))

    def parties(self, seq0, codes, sizes, ids, r, mode, ts):
        off = np.concatenate([[0], np.cumsum(np.asarray(sizes, np.int64))])
        for j in np.flatnonzero(np.asarray(codes) == 1):
            x, y = np.asarray(ids[off[j]:off[j + 1]], np.uint64), np.asarray(r[off[j]:off[j + 1]], np.int32)
            seq = (seq0 + int(j)) & 0xFFFFFFFF
            self.rec[seq] = (x, y, int(mode[j]), int(ts[j]))
            self.party.update((k, seq) for k in x.tolist())
            self.rating.update(zip(x.tolist(), y.tolist()))

    def balance(self, cfg, mask, lob, mem):
        return balance_parties(cfg, mask, lob, mem, self.rating.__getitem__, self.party.get)


class Twins:
    """Engine a with party_balance `mask`, engine b without it; every call goes to both."""

    def __init__(self, pkg, cfg, kind, seed, mask, cap=200_000, lo=0, hi=5001):
        self.pkg, self.cfg, self.kind, self.mask = pkg, cfg, kind, mask
        self.rng = np.random.default_rng(seed)
        self.a, self.b = pkg.Engine(cfg), pkg.Engine(cfg)
        for e in (self.a, self.b):
            e.set_option("party_capacity", cap)
        self.a.set_option("party_balance", mask)
        self.book = Book()
        self.next, self.now, self.lo, self.hi = 0, 1000, lo, hi
        self.matched = []  # seqs of the parties party_match placed
        self.same_ticks = True  # False while only a has team_balance: mm_locate's member index then differs

    def close(self):
        self.a.close()
        self.b.close()

    def ids(self, n):
        x = np.arange(self.next, self.next + n, dtype=np.uint64)
        self.next += n
        return x if self.kind == "dense" else self.pkg.synth.mix64(x + np.uint64(9 << 40))

    def solos(self, n):
        ids, rng = self.ids(n), self.rng
        r = rng.integers(self.lo, self.hi, n).astype(np.int32)
        m = rng.integers(0, self.cfg.n_modes, n).astype(np.uint8)
        ts = (self.now - rng.integers(0, 60, n)).astype(np.uint32)
        ca = self.a.enqueue(ids, r, m, ts)
        assert np.array_equal(ca, self.b.enqueue(ids, r, m, ts))
        self.book.solos(ids[ca == 1], r[ca == 1])

    def parties(self, n, modes=None, extreme=0.15):
        """n parties of 2 .. S members near one rating; a share `extreme` has a member far below the key domain and one
        far above it (R stays inside: clamped at both ends, the low one without a group of its own)."""
        rng, cfg = self.rng, self.cfg
        ok = modes if modes is not None else [k for k in range(cfg.n_modes) if cfg.modes[k].team_size >= 2]
        mode = rng.choice(ok, n).astype(np.uint8)
        size = np.array([rng.integers(2, cfg.modes[k].team_size + 1) for k in mode], np.uint8)
        base = rng.integers(self.lo + 200, self.hi - 200, n)
        r = np.repeat(base, size) + rng.integers(-20, 21, int(size.sum()))
        off = np.concatenate([[0], np.cumsum(size.astype(np.int64))])
        for j in np.flatnonzero(rng.random(n) < extreme):
            r[off[j]], r[off[j] + 1] = self.lo - 2000, 2 * base[j] - (self.lo - 2000)
            r[off[j] + 2:off[j + 1]] = base[j]
        r = r.astype(np.int32)
        ts = (self.now - rng.integers(0, 60, n)).astype(np.uint32)
        ids = self.ids(int(size.sum()))
        s0 = self.a.seq_next()
        ca = self.a.enqueue_party(size, ids, r, mode, ts)
        assert np.array_equal(ca, self.b.enqueue_party(size, ids, r, mode, ts)) and (ca == 1).all()
        self.book.parties(s0, ca, size, ids, r, mode, ts)

    def party_match(self, rules):
        la, ma, sa = self.a.party_match(self.now, rules_of(self.cfg, rules))
        lb, mb, sb = self.b.party_match(self.now, rules_of(self.cfg, rules))
        assert np.array_equal(la, lb)  # headers and their order
        for f in ("n_anchors", "n_lobbies", "n_matched", "n_parties", "n_absorbed"):
            assert getattr(sa, f) == getattr(sb, f), f
        want, total = self.book.balance(self.cfg, self.mask, lb, mb)
        assert np.array_equal(ma, want)
        for h in lb:  # every lobby holds the same players
            k = slice(int(h["first_member"]), int(h["first_member"]) + int(h["n_members"]))
            assert np.array_equal(np.sort(ma[k]), np.sort(mb[k]))
        assert sa.sum_imbalance == total and sb.sum_imbalance == 0
        self.matched += sorted({self.book.party[x] for x in mb.tolist() if x in self.book.party})
        return lb, mb, total

    def tick(self):
        ra, rb = self.a.tick(self.now), self.b.tick(self.now)
        for x, y in zip(ra[:3], rb[:3]):
            assert np.array_equal(x, y)
        self.now += 5
        return len(ra[0])

    def requeue_parties(self, k):
        """k of the matched parties back whole, on both engines"""
        seqs, self.matched = self.matched[:k], self.matched[k:]
        if not seqs:
            return 0
        recs = [self.book.rec[s] for s in seqs]
        args = ([len(r[0]) for r in recs], np.concatenate([r[0] for r in recs]), np.concatenate([r[1] for r in recs]),
                [r[2] for r in recs], [r[3] for r in recs], seqs)
        ca, cb = self.a.requeue_party(*args), self.b.requeue_party(*args)
        assert np.array_equal(ca, cb) and (ca == 1).all()
        return len(seqs)

    def remove(self):
        live = self.a.pool_read()["id"]
        pr = self.a.party_read()
        gone = np.concatenate([live[::37]] + [pr["members"][k][0][1:2] for k in range(0, len(pr["size"]), 7)])
        assert self.a.remove(gone) == self.b.remove(gone)

    def expire(self, max_wait):
        (ia, sa), (ib, sb) = self.a.expire(self.now, max_wait), self.b.expire(self.now, max_wait)
        oa, ob = np.lexsort((sa, ia)), np.lexsort((sb, ib))  # the listing order is not part of the contract
        assert np.array_equal(ia[oa], ib[ob]) and np.array_equal(sa[oa], sb[ob])

    def check(self):
        pa, pb = self.a.pool_read(), self.b.pool_read()
        for k in pa:
            assert np.array_equal(pa[k], pb[k]), k
        ra, rb = self.a.party_read(), self.b.party_read()
        for k in ("size", "seq", "enq_ts", "mode", "group", "rating"):
            assert np.array_equal(ra[k], rb[k]), k
        assert all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1])
                   for x, y in zip(ra["members"], rb["members"]))
        assert self.a.seq_next() == self.b.seq_next()
        ids = np.array(list(self.book.rating)[::53], np.uint64)
        assert np.array_equal(self.a.in_queue(ids), self.b.in_queue(ids))
        la, lb = self.a.locate(ids, self.now), self.b.locate(ids, self.now)
        for f in la.dtype.names:
            assert (f == "member" and not self.same_ticks) or np.array_equal(la[f], lb[f]), f


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
@pytest.mark.parametrize("layout", ["split", "wide", "overlap"])
def test_twin_engines_over_a_mixed_schedule(pkg, kind, layout):
    cfg = gpu_config(pkg, RATING, kind, layout)
    t = Twins(pkg, cfg, kind, seed=21, mask=0b111)  # 1v1 (accepted, nothing to split), 2v2, 3v3
    rules = party_rules(cfg)
    total = requeued = 0
    try:
        for step in range(18):
            op = step % 6
            if op == 0:
                t.solos(6000)
                t.parties(700)
            elif op == 1:
                _lob, _mem, s = t.party_match(rules[(step // 6) % 2])
                total += s
            elif op == 2:
                requeued += t.requeue_parties(40)
            elif op == 3:
                t.tick()
            elif op == 4:
                t.remove()
            else:
                t.expire(58)
            t.check()
        assert total > 0 and requeued > 0
    finally:
        t.close()


def team_balanced(cfg, mask, lob, mem, rating):
    """team_balance's rule on tick / widen lobbies (test_team_balance's restatement)"""
    lo, hi = clamp_bounds(cfg)
    mem = np.array(mem, np.uint64, copy=True)
    for m in range(cfg.n_modes):
        sel = np.flatnonzero(lob["mode"] == m)
        S = cfg.modes[m].team_size
        if not (mask >> m) & 1 or S < 2 or not len(sel):
            continue
        idx = lob["first_member"][sel].astype(np.int64)[:, None] + np.arange(2 * S)[None, :]
        c = np.clip(np.array([rating[x] for x in mem[idx.ravel()].tolist()], np.int64), lo, hi).reshape(len(sel), -1)
        mem[idx] = mem[np.take_along_axis(idx, split_numpy(c, S)[0], 1)]
    return mem


def dry_party_match(eng, now, rules, lobby_cap, member_cap):
    """mm_party_match with the given capacities, no retry -> (status, PartyStats)"""
    rules = np.ascontiguousarray(rules, eng.WIDEN_RULE_DTYPE)
    lob = np.empty(max(lobby_cap, 1), eng_mod.LOBBY_DTYPE)
    mem = np.empty(max(member_cap, 1), np.uint64)
    st = abi.PartyStats()
    rc = eng.lib.mm_party_match(eng.h, int(now), eng_mod._p(rules), eng_mod._p(lob), lobby_cap, eng_mod._p(mem),
                                member_cap, C.byref(st))
    return rc, st


MASK_MODES = [("1v1", 2, 1), ("2v2", 2, 2), ("3v3", 2, 3), ("5v5", 2, 5), ("duo3", 3, 2), ("9v9", 2, 9)]


@pytest.mark.gpu
def test_masks_team_balance_beside_it_refusals_and_the_option_off(pkg):
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MASK_MODES, order=RATING, capacity=200_000,
                                active_capacity=1_000_000, default_group=-1)
    t = Twins(pkg, cfg, "hashed", seed=33, mask=1 << 3)  # 5v5 only
    G = cfg.n_groups
    try:
        # the refusals: nothing changes, the mask in force stays
        for bad in (1 << 6, -1, 1 << 4, 1 << 5, (1 << 3) | (1 << 4), 1 << 40):
            with pytest.raises(pkg.EngineError) as ei:
                t.a.set_option("party_balance", bad)
            assert ei.value.status == abi.MM_E_ARG
        t.a.set_option("party_balance", 1)  # a 1v1 mode is accepted and changes nothing
        t.a.set_option("party_balance", 1 << 3)
        tb = (1 << 2) | (1 << 3)
        t.a.set_option("team_balance", tb)  # b has neither option
        t.same_ticks = False
        t.solos(40_000)
        t.parties(3000, modes=[1, 2, 3, 4, 5])
        t.check()
        rules = {(m, g): (0, 10, 5, 5, 120) for m in range(cfg.n_modes) for g in range(G)}
        # the dry run and the MM_E_CAP refusal change nothing and run no balance pass
        for caps in ((0, 0), (1, 1 << 20)):
            rc, st = dry_party_match(t.a, t.now, rules_of(cfg, rules), *caps)
            assert rc == abi.MM_E_CAP and st.n_lobbies > 1 and st.sum_imbalance == 0
        t.check()
        # party lobbies follow party_balance only: 5v5 balanced, 2v2 / 3v3 (team_balance), duo3 and 9v9 as formed
        lob, _mem, total = t.party_match(rules)
        assert total > 0 and set(lob["mode"].tolist()) >= {1, 2, 3, 4, 5}
        t.check()
        # tick and widen lobbies follow team_balance only
        t.solos(40_000)
        rating = dict(t.book.rating)
        wa = t.a.widen(t.now, rules_of(cfg, rules))
        wb = t.b.widen(t.now, rules_of(cfg, rules))
        assert np.array_equal(wa[0], wb[0]) and len(wa[0]) > 0
        assert np.array_equal(wa[1], team_balanced(cfg, tb, wb[0], wb[1], rating))
        t.check()
        t.solos(40_000)
        rating = dict(t.book.rating)
        ta, tbk = t.a.tick(t.now), t.b.tick(t.now)
        assert np.array_equal(ta[0], tbk[0]) and len(ta[0]) > 0
        assert np.array_equal(ta[1], team_balanced(cfg, tb, tbk[0], tbk[1], rating))
        t.check()
        # the option off: a is b again
        t.solos(40_000)
        t.parties(3000, modes=[1, 2, 3, 4, 5])
        t.now += 100
        t.a.set_option("party_balance", 0)
        t.mask = 0
        lob, _mem, total = t.party_match(rules)
        assert len(lob) > 0 and total == 0
        t.check()
    finally:
        t.close()


# ================================================================================ GPU: the model
class PbModel(EngineModel):
    """EngineModel whose party_match applies the party_balance restatement to the lobbies it forms."""

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        self.pbal = 0
        self.pb_sum = 0

    def party_match(self, now, rules):
        prat = {x: r for p in self.parties for x, r in zip(p[0].tolist(), p[1].tolist())}
        pid = {x: int(p[4]) for p in self.parties for x in p[0].tolist()}
        a = self.q["alive"]
        srat = dict(zip(self.q["id"][a].tolist(), self.q["rating"][a].tolist()))
        lob, mem, st = super().party_match(now, rules)
        mem, self.pb_sum = balance_parties(self.cfg, self.pbal, lob, mem,
                                           lambda x: prat[x] if x in prat else srat[x], pid.get, self.plain)
        return lob, mem, st


class PbSchedule(EngineSchedule):
    """EngineSchedule on PbModel: party_balance is set on every engine of the schedule and toggled by option steps."""

    def __init__(self, pkg, oracle, cfg, rng, dense, pbal, **kw):
        super().__init__(pkg, oracle, cfg, rng, dense, **kw)
        m = PbModel(cfg, oracle, pkg.abi)
        m.pcap, m.pbal = self.m.pcap, pbal
        self.m, self.full = m, pbal
        self.eng.set_option("party_balance", pbal)

    def setup(self, eng):
        super().setup(eng)
        eng.set_option("party_balance", getattr(self.m, "pbal", 0))

    def party_match(self, rules=None):
        rules = rules if rules is not None else party_rules(self.cfg)[int(self.rng.integers(0, 2))]
        lob, mem, (n_anc, n_abs, n_pl) = self.m.party_match(self.now, rules)
        glob, gmem, st = self.eng.party_match(self.now, rules_of(self.cfg, rules))
        assert (st.n_anchors, st.n_absorbed, st.n_parties, st.n_lobbies, st.n_matched) == \
            (n_anc, n_abs, n_pl, len(lob), len(mem))
        assert hdr(glob) == hdr(lob) and np.array_equal(gmem, mem)
        assert st.sum_imbalance == self.m.pb_sum
        self.count("party_match")
        if self.m.pbal and self.m.pb_sum:
            self.count("balanced_party_match")
        return lob, mem

    def option(self):
        if self.rng.random() < 0.3:
            self.m.pbal = 0 if self.m.pbal else self.full
            self.eng.set_option("party_balance", self.m.pbal)
            self.count("party_balance")
            return
        super().option()


@pytest.mark.gpu
@pytest.mark.parametrize("dense,wide", [(False, False), (True, True)], ids=lambda v: str(v))
def test_model_schedule_with_the_mask(pkg, oracle, dense, wide):
    rng = np.random.default_rng(700 + 2 * dense + wide)
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[:4], order=RATING, capacity=300_000,
                                active_capacity=4_000_000, default_group=-1,
                                flags=(DENSE if dense else 0) | WIDE * wide)
    s = PbSchedule(pkg, oracle, cfg, rng, dense, 0b1111)
    try:
        s.players(60_000, old=0.02)
        s.party_batch(1500)
        s.check()
        for _ in range(110):
            s.step()
        s.tick()
        s.finish()
        s.check()
        for what in ("party_match", "party_balance", "requeue", "expire", "checkpoint", "queue_move", "enqueue_party"):
            assert s.counts.get(what, 0) >= 2, (what, s.counts)
        assert s.counts.get("balanced_party_match", 0) >= 1, s.counts
    finally:
        s.close()


@pytest.mark.gpu
def test_party_table_of_many_tiles(pkg, oracle):
    """More than 3 x 1024 parties, 2 000 of them at one rating: the balance pass meets lobbies written by many CTAs."""
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[2:4] + MODES8[6:7], order=RATING,
                                capacity=400_000, active_capacity=2_000_000, default_group=-1)
    s = PbSchedule(pkg, oracle, cfg, np.random.default_rng(17), False, 0b111, lo=0, hi=5001, pcap=200_000)
    try:
        s.players(150_000)
        s.party_batch(2000)
        s.party_batch(2000, sizes=None, crowd=2500)
        party_batch_of(s, [6] * 200 + [2, 3, 4, 5] * 100, 2)
        assert len(s.m.parties) > 3 * 1024
        s.check()
        for k in range(3):
            s.now += 50
            s.party_match({(m, g): (0, 5 + 20 * k, 5, 5, 100) for m in range(3) for g in range(cfg.n_groups)})
            s.check()
        assert s.counts.get("balanced_party_match", 0) >= 1
    finally:
        s.close()


# ================================================================================ GPU: SearchPool
@pytest.mark.gpu
def test_search_pool_publishes_balanced_party_lobbies_and_requeues_them_whole(pkg):
    from .fakes import FakeBroker
    from .test_expire import publish
    from .test_handover import start_workers
    from .test_requeue import lobbies
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=[("1v1", 2, 1), ("5v5", 2, 5)],
                                order=RATING, capacity=10_000, active_capacity=40_000)
    eng = pkg.Engine(cfg)
    t = [0.0]
    try:
        pool = sw.SearchPool(eng, ["1v1", "5v5"], list(pkg.synth.REFERENCE_GROUP_NAMES), flush_every_s=3600,
                             clock=lambda: t[0], parties={"5v5": (0, 50, 1000, 0, 50)}, party_capacity=1000,
                             requeue_parties=True, balance_parties=["5v5"])
        broker = FakeBroker()
        start_workers(sw, broker, pool, pkg)
        # the 5v5 example, 200 points up so every rating of the lobby is in one group: R = 1700 (silver)
        publish_party(pkg, broker, sw, "silver", [("a0", 2100), ("a1", 1300)], "5v5")
        publish_party(pkg, broker, sw, "silver", [(f"b{i}", 1750) for i in range(3)], "5v5")
        for i, r in enumerate([1700, 1695, 1705, 1690, 1710]):
            publish(pkg, broker, cfg, f"s{i}", r, "5v5")
        broker.deliver_all()
        pool.flush()
        t[0] += 1
        assert pool.tick() == 1
        first = lobbies(broker, sw)[0]
        teams = [[(p["id"], p["rating"]) for p in first["teams"][k]] for k in ("team 1", "team 2")]
        assert teams == [[("a0", 2100), ("a1", 1300), ("s0", 1700), ("s2", 1705), ("s4", 1710)],
                         [("b0", 1750), ("b1", 1750), ("b2", 1750), ("s1", 1695), ("s3", 1690)]]
        docs = [p for team in first["teams"].values() for p in team]
        assert pool.requeue(docs) == ["requeued"] * 10  # a member declined the ready check
        assert eng.party_read()["size"].tolist() == [2, 3]  # both parties back whole, in age order
        t[0] += 1
        assert pool.tick() == 1
        assert lobbies(broker, sw)[1]["teams"] == first["teams"]
    finally:
        eng.close()
