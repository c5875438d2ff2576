"""The off-tick calls together, against one restatement of everything the engine holds.

`EngineModel` extends the tick schedule's model (tests/test_tick_forms_and_schedules.py: ingest codes, S0 / S1 ticks
through the C oracle, mm_queue_stats, snapshot / restore) with the party table and every call that takes players or
reports on them: mm_enqueue_party, mm_party_match, mm_widen, mm_backfill, mm_requeue, mm_expire, the lobby budget and
team_balance of the tick, mm_match_quality, mm_locate, and the checkpoint hand-over (mm_export_parties, mm_export,
mm_import, mm_merge_parties with MM_PARTY_KEEP_SEQ).  Each restatement is the one its feature's test file holds,
imported from there; its input is the model's own pool, party table and book, never what the engine reports.  So a
fault in a primitive the off-tick calls share (the pool walk, the bin keys, the band pipeline, the output scan) cannot
hide behind a twin engine that runs the same code.

CPU: the model driven twice through random schedules, once on the plain restatements and once on the binned / numpy
ones, agreeing at every step.
GPU: long mixed schedules of every call on both id kinds and both rating-order layouts, and an arrival-order run; the
off-tick calls at the tile geometries only the tick had met (huge key domains, the key-domain edge, many partitions,
the whole-segment fallback, overlapping groups clamped at both key ends); party modes of 3, 40, 256 and 257 teams; a
party table of more than three scatter tiles with one crowded bin; balanced 8v8 at clamped ratings; and requeue of
the members of a matched party, who share one enqueue sequence number.
"""
import importlib
from types import SimpleNamespace

import numpy as np
import pytest

from .test_backfill import clamp_bounds, restate as bf_restate, restate_plain as bf_plain
from .test_expire import r_wait
from .test_lobby_budget import allowances, clip, queue_counts
from .test_locate import restate as loc_restate, restate_plain as loc_plain
from .test_match_quality import restate as mq_restate
from .test_parties import enqueue_codes, party_rating, party_rules, restate_bins as pt_bins, restate_plain as pt_plain
from .test_team_balance import split_numpy, split_plain
from .test_tick_forms_and_schedules import (HOST_FORMS, AsyncTicks, Model, Schedule, check_state, check_tick, poison,
                                            tick_form)
from .test_tile_geometry import DENSE, MODES8, WIDE, Layout, edge_config, fallback_groups, key_domain_edge
from .test_widen import restate as wd_restate, restate_plain as wd_plain, rule_sets, rules_of

eng_mod = importlib.import_module("microservice-matchmaking_b200.engine")
abi = importlib.import_module("microservice-matchmaking_b200.abi")

ARRIVAL, RATING = 0, 1
U32 = 0xFFFFFFFF
STAYS = abi.MM_LOCATE_STAYS
LOBBY = eng_mod.LOBBY_DTYPE
OVERLAP = [(0, 2000), (1000, 3000), (2500, 5000), (100, 200)]


class ArgRefused(Exception):
    """The restated call is refused with MM_E_ARG: nothing changes."""


def lobbies_of(groups):
    """[(mode, group, [member ids])] -> (LOBBY headers, member ids u64)"""
    lob = np.zeros(len(groups), LOBBY)
    off = 0
    for k, (m, g, ms) in enumerate(groups):
        lob[k] = (off, len(ms), m, g)
        off += len(ms)
    mem = np.array([x for _, _, ms in groups for x in ms], np.uint64)
    return lob, mem


def hdr(lob):
    return [tuple(int(x) for x in (h["mode"], h["group"], h["n_members"], h["first_member"])) for h in lob]


# ================================================================================ the restatement
class EngineModel(Model):
    """Everything one engine holds, restated.  plain: the one-at-a-time restatements (the CPU cross-check); otherwise
    the binned / numpy ones, which the GPU tests use for speed."""

    def __init__(self, cfg, oracle, abi, spread=-1, plain=False):
        super().__init__(cfg, oracle, abi, spread)
        self.plain = plain
        self.parties = []   # [ids u64, ratings i64, mode, ts, seq] of the queued parties, in age order
        self.pcap = 0       # party_capacity: members the table holds
        self.party_matched = np.zeros(0, np.uint64)  # members of the parties mm_party_match placed
        self.book = {}      # id -> (rating, mode, ts, seq) at its latest queueing: what the caller keeps for mm_requeue
        self.balance = 0    # team_balance mask
        self.budget = (None, None)
        self.last = None    # (lobbies, members, id -> rating) of the last tick: mm_match_quality's input (None: void)
        self.lay = Layout(cfg)
        self.lo, self.hi = clamp_bounds(cfg)

    # ---- what the caller keeps --------------------------------------------------------------------------------------
    def rating_of(self, ids):
        """The ratings the pool holds for live queued ids.  The book may be newer: a restore brings back older
        entries."""
        a = self.q["alive"]
        r = dict(zip(self.q["id"][a].tolist(), self.q["rating"][a].tolist()))
        return np.array([r[x] for x in np.asarray(ids, np.uint64).tolist()], np.int64)

    def party_members(self):
        return np.concatenate([p[0] for p in self.parties]) if self.parties else np.zeros(0, np.uint64)

    # ---- enqueue ----------------------------------------------------------------------------------------------------
    def enqueue(self, ids, rating, mode, ts=None, scalar=False):
        s0 = self.seq_next
        code = super().enqueue(ids, rating, mode, ts, scalar)
        k = np.flatnonzero(code == 1)
        ts = np.zeros(len(code), np.uint32) if ts is None else np.asarray(ts, np.uint32)
        cols = (np.asarray(rating, np.int64)[k], np.asarray(mode, np.int64)[k], ts[k].astype(np.int64), (s0 + k) & U32)
        self.book.update(zip(np.asarray(ids, np.uint64)[k].tolist(), zip(*(c.tolist() for c in cols))))
        return code

    def enqueue_party(self, sizes, ids, rating, mode, ts):
        room = self.pcap - sum(len(p[0]) for p in self.parties)
        code = enqueue_codes(self.cfg, set(self.active.tolist()), [int(s) for s in sizes], ids, rating,
                             [int(m) for m in mode], room, self.id_limit)
        off = np.concatenate([[0], np.cumsum(np.asarray(sizes, np.int64))])
        for j in np.flatnonzero(code == 1):
            mid = np.asarray(ids[off[j]:off[j + 1]], np.uint64)
            rat = np.asarray(rating[off[j]:off[j + 1]], np.int64)
            seq = (self.seq_next + int(j)) & U32
            self.parties.append([mid, rat, int(mode[j]), int(ts[j]), seq])
            self.active = np.concatenate([self.active, mid])
            self.book.update((int(x), (int(r), int(mode[j]), int(ts[j]), seq)) for x, r in zip(mid, rat))
        self.seq_next = (self.seq_next + len(code)) & U32
        return code

    # ---- calls that drop players -------------------------------------------------------------------------------------
    def remove(self, ids):
        """mm_remove: a member of a queued party takes the whole party out."""
        ids = np.asarray(ids, np.uint64)
        hit = [np.isin(p[0], ids).any() for p in self.parties]
        gone = [p[0] for p, h in zip(self.parties, hit) if h]
        self.parties = [p for p, h in zip(self.parties, hit) if not h]
        return super().remove(np.concatenate([ids] + gone))

    def expire(self, now, max_wait):
        """-> ((solo ids, seq), (party member ids, party seq)); solos turn dead, parties leave whole."""
        q = self.q
        k = q["alive"] & (r_wait(now, q["ts"]) >= max_wait)
        solo = (q["id"][k], q["seq"][k])
        old = [r_wait(now, [p[3]])[0] >= max_wait for p in self.parties]
        ps = [p for p, o in zip(self.parties, old) if o]
        self.parties = [p for p, o in zip(self.parties, old) if not o]
        party = (np.concatenate([p[0] for p in ps]) if ps else np.zeros(0, np.uint64),
                 np.array([p[4] for p in ps for _ in p[0]], np.uint32))
        q["alive"] &= ~k
        self.active = self.active[~np.isin(self.active, np.concatenate([solo[0], party[0]]))]
        return solo, party

    # ---- the tick: the oracle, then the lobby budget, then team_balance ----------------------------------------------
    def balanced(self, lob, mem, rating):
        """rating: of every member, in member order."""
        mem = np.array(mem, np.uint64, copy=True)
        rating = np.asarray(rating, np.int64)
        for m in range(self.cfg.n_modes):
            sel = np.flatnonzero(lob["mode"] == m)
            if not (self.balance >> m) & 1 or not len(sel):
                continue
            S = self.cfg.modes[m].team_size
            idx = lob["first_member"][sel].astype(np.int64)[:, None] + np.arange(2 * S)[None, :]
            c = np.clip(rating[idx.ravel()], self.lo, self.hi).reshape(len(sel), 2 * S)
            perm = np.array([split_plain(x, S)[0] for x in c]) if self.plain else split_numpy(c, S)[0]
            mem[idx] = mem[np.take_along_axis(idx, perm, 1)]
        return mem

    def next_tick(self):
        """What the next tick gives: the oracle's lobbies (S0 or S1), cut by the lobby budget, teams balanced."""
        ref, seq_of = self.tick_ref()
        lob, mem, eseq = ref.lobbies, np.asarray(ref.member_ids, np.uint64), np.asarray(ref.emit_seq)
        if self.budgeted():
            c = clip(self.cfg, ref, self.q["id"][self.q["alive"]],
                     allowances(self.cfg, queue_counts(self.cfg, lob), *self.budget))
            lob, mem, eseq = c["lob"], c["mem"], c["seq"]
        mem = self.balanced(lob, mem, self.rating_of(mem))
        alive = int(self.q["alive"].sum())
        return SimpleNamespace(lobbies=lob, member_ids=mem, emit_seq=eseq, n_lobbies=len(lob), n_matched=len(mem),
                               n_residual=alive - len(mem), n_dead=self.slots() - alive), seq_of

    def apply_tick(self, ref, now):
        q, G = self.q, self.cfg.n_groups
        hit = q["alive"] & np.isin(q["id"], ref.member_ids)
        assert hit.sum() == ref.n_matched
        cut = ref.lobbies["mode"].astype(np.int64) * G + ref.lobbies["group"]
        self.match = (q["mode"][hit].astype(np.int64) * G + self.groups(q["rating"][hit]), q["ts"][hit].copy(), now,
                      np.bincount(cut, minlength=self.cfg.n_modes * G))
        # the report reads the ratings the pool held at the tick; a matched id may queue again with another rating
        self.last = (ref.lobbies, ref.member_ids, dict(zip(q["id"][hit].tolist(), q["rating"][hit].tolist())))
        self.q = {k: v[q["alive"] & ~hit] for k, v in q.items()}

    def quality(self):
        """mm_match_quality of the last tick -> (per queue, per lobby), or None when the report is void."""
        if self.match is None or self.last is None:
            return None
        lob, mem, r = self.last
        return mq_restate(self.cfg, lob, mem, lambda ids: np.array([r[x] for x in np.asarray(ids).tolist()], np.int64))

    def budgeted(self):
        return any(b is not None for b in self.budget)

    # ---- calls that take players -------------------------------------------------------------------------------------
    def widen(self, now, rules):
        """-> (headers, member ids, n_anchors, n_absorbed); the members are taken, balanced like a tick's."""
        p = self.pool()
        if self.plain:
            lob, mem = lobbies_of(wd_plain(self.cfg, p["id"], p["rating"], p["mode"], p["enq_ts"], now, rules))
            n_anc = n_abs = None
        else:
            want, mem, n_anc, n_abs = wd_restate(self.cfg, p["id"], p["rating"], p["mode"], p["enq_ts"], now, rules)
            lob = np.zeros(len(want), LOBBY)
            for k, f in enumerate(("mode", "group", "n_members", "first_member")):
                lob[f] = [w[k] for w in want]
        rating = self.rating_of(mem)
        self.take(mem)
        return lob, self.balanced(lob, mem, rating), n_anc, n_abs

    def party_match(self, now, rules):
        """-> (headers, member ids, (n_anchors, n_absorbed, n_parties)); placed parties leave the table, their members
        stay active as matched players; the solos are taken."""
        p = self.pool()
        parties = [(x[0], x[1], x[2], x[3]) for x in self.parties]
        out, n_anc, n_abs, n_pl = (pt_plain if self.plain else pt_bins)(
            self.cfg, (p["id"], p["rating"], p["mode"], p["enq_ts"]), parties, now, rules)
        lob, mem = lobbies_of(out)
        placed = [np.isin(x[0], mem).any() for x in self.parties]
        self.party_matched = np.concatenate([self.party_matched] + [x[0] for x, k in zip(self.parties, placed) if k])
        self.parties = [x for x, k in zip(self.parties, placed) if not k]
        self.take(mem)
        return lob, mem, (n_anc, n_abs, n_pl)

    def backfill(self, reqs):
        p = self.pool()
        if self.plain:
            n, out = bf_plain(self.cfg, p["id"], p["rating"], p["mode"], list(zip(*(np.asarray(x).tolist()
                                                                                   for x in reqs))))
        else:
            n, out = bf_restate(self.cfg, p["id"], p["rating"], p["mode"], reqs)
        self.take(np.concatenate(out) if out else np.zeros(0, np.uint64))
        return n, out

    # ---- requeue ----------------------------------------------------------------------------------------------------
    def requeue(self, ids):
        """mm_requeue of `ids` with the columns the caller kept -> codes; ArgRefused where the engine refuses.  A code-1
        entry goes back at its age position; every partition that receives one drops its dead slots."""
        ids = np.asarray(ids, np.uint64)
        assert len(np.unique(ids)) == len(ids)
        col = np.array([self.book[int(x)] for x in ids.tolist()], np.int64).reshape(-1, 4)
        r, m, ts, seq = col.T
        q = self.q
        live = np.isin(ids, q["id"][q["alive"]]) | np.isin(ids, self.party_members())
        code = np.where(live, 0, np.where(np.isin(ids, self.active), 1, 4)).astype(np.uint8)
        if (m >= self.cfg.n_modes).any() or (self.groups(r) < 0).any():
            raise ArgRefused("a rating without a group")  # a party member's own rating need not have one
        if len(np.unique(seq)) < len(seq) or (seq == self.seq_next).any():
            raise ArgRefused("entries not in strict age order")  # co-members of a party share one seq
        one = code == 1
        part = self.lay.partition_of(r[one], m[one])
        qpart = self.lay.partition_of(q["rating"], q["mode"])
        taken = qpart[q["alive"]] * (1 << 32) + q["seq"][q["alive"]].astype(np.int64)
        if np.isin(part * (1 << 32) + seq[one], taken).any():
            raise ArgRefused("a seq equal to a live player's in its partition")
        keep = q["alive"] | ~np.isin(qpart, part)
        add = dict(id=ids[one], rating=r[one].astype(np.int32), mode=m[one].astype(np.uint8),
                   ts=ts[one].astype(np.uint32), seq=seq[one].astype(np.uint32), alive=np.ones(int(one.sum()), bool))
        q = {k: np.concatenate([v[keep], add[k]]) for k, v in q.items()}
        o = np.argsort((q["seq"].astype(np.int64) - self.seq_next) & U32, kind="stable")
        self.q = {k: v[o] for k, v in q.items()}
        return code

    # ---- locate -----------------------------------------------------------------------------------------------------
    def locate(self, ids, now):
        """-> dict of expected columns per id: state, and for queued solos queue, ahead, depth, lobby, member, rating,
        ts, seq, wait; for queued party members rating and seq."""
        ids = np.asarray(ids, np.uint64)
        q = self.q
        a = q["alive"]
        lid, lr, lm, ls = q["id"][a], q["rating"][a], q["mode"][a], q["seq"][a]
        if self.plain:
            d = loc_plain(self.cfg, lid, lr, lm, ls, self.seq_next)
            queue, ahead, depth = (np.array([d[int(x)][k] for x in lid.tolist()], np.int64) for k in range(3))
        else:
            queue, ahead, depth, _, _ = loc_restate(self.cfg, lid, lr, lm, ls, self.seq_next)
        ref, _ = self.next_tick()
        G = self.cfg.n_groups
        pred, count = {}, {}
        for h in ref.lobbies:
            qq = int(h["mode"]) * G + int(h["group"])
            k = count.get(qq, 0)
            count[qq] = k + 1
            f = int(h["first_member"])
            for j, x in enumerate(ref.member_ids[f:f + int(h["n_members"])].tolist()):
                pred[x] = (k, j)
        pos = {x: i for i, x in enumerate(lid.tolist())}
        pm = {int(x): (int(r), p[4]) for p in self.parties for x, r in zip(p[0], p[1])}
        act = set(self.active.tolist())
        out = []
        for x in ids.tolist():
            if x in pos:
                i = pos[x]
                lob, mem = pred.get(x, (STAYS, 0xFFFF))
                out.append((1, int(queue[i]), int(ahead[i]), int(depth[i]), lob, mem, int(lr[i]),
                            int(q["ts"][a][i]), int(ls[i])))
            elif x in pm:
                out.append((3, -1, 0, 0, STAYS, 0xFFFF, pm[x][0], -1, pm[x][1]))
            else:
                out.append((2 if x in act else 0, -1, 0, 0, STAYS, 0xFFFF, 0, -1, 0))
        cols = np.array(out, np.int64).reshape(-1, 9).T
        return dict(zip(("state", "queue", "ahead", "depth", "lobby", "member", "rating", "ts", "seq"), cols))

    # ---- snapshot and hand-over -------------------------------------------------------------------------------------
    def restore(self):
        super().restore()
        self.parties = []  # mm_restore empties the party table
        self.last = None

    def queue_move(self, mask):
        """The queues of `mask` out to another engine and back (mm_export_queues / mm_merge, with their parties in
        party images), with every other party stepping aside around the image calls.  The moved players leave dead
        slots and come back with this engine's next numbers, queue by queue in their old order; then the other parties
        and then the moved ones are merged back, each taking the next number in age order."""
        q, G = self.q, self.cfg.n_groups
        cut = q["mode"].astype(np.int64) * G + self.groups(q["rating"])
        out = q["alive"] & np.asarray(mask, bool)[cut]
        o = np.flatnonzero(out)
        o = o[np.lexsort((o, cut[o]))]  # queue by queue, age order inside a queue
        back = {k: v[o].copy() for k, v in q.items()}
        q["alive"] &= ~out
        back["seq"] = ((self.seq_next + np.arange(len(o))) & U32).astype(np.uint32)
        self.seq_next = (self.seq_next + len(o)) & U32
        self.q = {k: np.concatenate([q[k], back[k]]) for k in q}
        moved = [bool(mask[p[2] * G + self.group(party_rating(p[1]))]) for p in self.parties]
        self.parties = [p for p, mv in zip(self.parties, moved) if not mv] + \
            [p for p, mv in zip(self.parties, moved) if mv]
        for p in self.parties:
            p[4] = self.seq_next
            self.seq_next = (self.seq_next + 1) & U32
        for x, r, md, ts, sq in zip(*(back[k].tolist() for k in ("id", "rating", "mode", "ts", "seq"))):
            self.book[x] = (r, md, ts, sq)
        for p in self.parties:
            self.book.update((int(x), (int(r), p[2], p[3], p[4])) for x, r in zip(p[0], p[1]))
        return int(out.sum())

    def checkpoint(self):
        """A fresh engine that imported mm_export and merged the party image back with its numbers: the live entries,
        the active set, seq_next and the party table; no reject list, match section, snapshot or last tick."""
        self.q = {k: v[self.q["alive"]] for k, v in self.q.items()}
        self.codes = np.zeros(0, np.uint8)
        self.match = self.snap = self.last = None


# ================================================================================ the engine against the model
def check_engine(eng, m, now, sample=(), stats=True):
    """check_state (pool, active set, in_queue, reject list, queue_stats), plus seq_next, the party table and
    mm_match_quality."""
    check_state(eng, m, now, sample, stats)
    assert eng.seq_next() == m.seq_next
    pr = eng.party_read()
    assert len(pr["size"]) == len(m.parties)
    if m.parties:
        R = np.array([party_rating(p[1]) for p in m.parties], np.int64)
        assert np.array_equal(pr["size"], [len(p[0]) for p in m.parties])
        assert np.array_equal(pr["seq"], [p[4] for p in m.parties])
        assert np.array_equal(pr["enq_ts"], [p[3] for p in m.parties])
        assert np.array_equal(pr["mode"], [p[2] for p in m.parties])
        assert np.array_equal(pr["rating"], R) and np.array_equal(pr["group"], m.groups(R))
        for (gi, gr), p in zip(pr["members"], m.parties):
            assert np.array_equal(gi, p[0]) and np.array_equal(gr, p[1])
    want = m.quality()
    got = eng.match_quality(want_lobbies=True)
    if want is None:
        assert len(got[0]) == 0 and len(got[1]) == 0
    else:
        for w, g in zip(want, got):
            for f in w.dtype.names:
                assert np.array_equal(g[f], w[f]), f


def check_locate(eng, m, ids, now):
    want = m.locate(ids, now)
    rec = eng.locate(ids, now)
    assert np.array_equal(rec["state"], want["state"])
    assert np.array_equal(rec["lobby"], want["lobby"]) and np.array_equal(rec["member"], want["member"])
    s = want["state"] == 1
    G = m.cfg.n_groups
    assert np.array_equal(rec["mode"][s], want["queue"][s] // G)
    assert np.array_equal(rec["group"][s], want["queue"][s] % G)
    assert np.array_equal(rec["ahead"][s], want["ahead"][s]) and np.array_equal(rec["depth"][s], want["depth"][s])
    assert np.array_equal(rec["enq_ts"][s], want["ts"][s])
    assert np.array_equal(rec["wait"][s], r_wait(now, want["ts"][s]))
    p = want["state"] >= 1
    p &= want["state"] != 2
    assert np.array_equal(rec["rating"][p], want["rating"][p]) and np.array_equal(rec["seq"][p], want["seq"][p])
    assert (rec["depth"][want["state"] == 3] == 0).all()
    return rec


PCAP = 60_000


class EngineSchedule(Schedule):
    """One engine and the EngineModel, driven by every call; everything is compared after every step."""

    def __init__(self, pkg, oracle, cfg, rng, dense, parties=True, lo=0, hi=5200, pcap=PCAP):
        super().__init__(pkg, oracle, cfg, rng, dense)
        self.m = EngineModel(cfg, oracle, pkg.abi)
        self.abi = pkg.abi
        self.lo, self.hi = lo, hi
        self.parties = parties and cfg.order_mode == RATING
        self.round = []
        self.rank_impl = None  # the engine's default until an option step sets it
        self.pcap = pcap if self.parties else 0
        self.setup(self.eng)

    def setup(self, eng):
        """The options an engine does not carry through an image."""
        if self.pcap:
            eng.set_option("party_capacity", self.pcap)
            self.m.pcap = self.pcap
        eng.set_option("tick_impl", self.tick_impl)
        if self.rank_impl is not None:
            eng.set_option("rank_impl", self.rank_impl)
        if self.m.spread >= 0:
            eng.set_option("max_spread", self.m.spread)
        eng.set_option("team_balance", self.m.balance)
        eng.set_lobby_budget(*self.m.budget)

    def count(self, what):
        self.counts[what] = self.counts.get(what, 0) + 1

    def refused(self, status, call):
        with pytest.raises(self.pkg.EngineError) as ei:
            call()
        assert ei.value.status == status

    def check(self):
        check_engine(self.eng, self.m, self.now, self.sample()[:2000])

    # ---- players ------------------------------------------------------------------------------------------------
    def players(self, n, old=0.0):
        """n valid fresh players in [lo, hi) of every mode; a fraction `old` has waited 1000 more."""
        rng, cfg = self.rng, self.cfg
        ids = self.fresh(n)
        r = rng.integers(self.lo, self.hi, n).astype(np.int32)
        md = rng.integers(0, cfg.n_modes, n).astype(np.uint8)
        ts = (self.now - rng.integers(0, 60, n) - 1000 * (rng.random(n) < old)).astype(np.uint32)
        assert np.array_equal(self.eng.enqueue(ids, r, md, ts), self.m.enqueue(ids, r, md, ts))

    def party_batch(self, n, sizes=None, crowd=None):
        """n fresh parties of the modes that hold them, sizes 2 .. S (or `sizes`), ratings near one value (`crowd`:
        every party at that rating); a few invalid ones and a few with a member already active."""
        rng, cfg = self.rng, self.cfg
        ok = [k for k in range(cfg.n_modes) if 2 <= cfg.modes[k].team_size]
        mode = rng.choice(ok, n).astype(np.uint8)
        size = np.array([rng.integers(2, cfg.modes[k].team_size + 1) for k in mode] if sizes is None else sizes,
                        np.uint8)
        ids = self.fresh(int(size.sum()))
        base = np.repeat(rng.integers(self.lo, self.hi, n) if crowd is None else np.full(n, crowd), size)
        r = (base + (rng.integers(-20, 21, len(ids)) if crowd is None else 0)).astype(np.int32)
        ts = (self.now - rng.integers(0, 60, n)).astype(np.uint32)
        if crowd is None and n > 20:
            mode[rng.integers(0, n, 2)] = cfg.n_modes  # invalid
            if len(self.m.active):  # a member already active
                ids[rng.integers(0, len(ids), 3)] = rng.choice(self.m.active, 3)
        want = self.m.enqueue_party(size, ids, r, mode, ts)
        assert np.array_equal(self.eng.enqueue_party(size, ids, r, mode, ts), want)
        self.count("enqueue_party")
        return want

    # ---- calls ----------------------------------------------------------------------------------------------------
    def tick(self):
        rng, m = self.rng, self.m
        ref, seq_of = m.next_tick()
        forms = list(HOST_FORMS if self.dense else ("tick_emit", "tick", "device"))
        if self.async_on:
            forms = ["async_tick"] + (["async_packed"] if self.dense else [])
        form = str(rng.choice(forms))
        self.count(form)
        if m.budgeted():
            self.count("budgeted_tick")
        if m.balance:
            self.count("balanced_tick")
        if form.startswith("async"):
            self.at.tick(form == "async_packed", self.now, (ref, seq_of))
        else:
            if not self.async_on:
                poison(self.eng, ref.n_lobbies + 16, ref.n_matched + 16)
            lob, mem, seq, st = tick_form(self.pkg, self.eng, form, self.now)
            check_tick(ref, seq_of, lob, mem, seq, st)
        m.apply_tick(ref, self.now)

    def party_match(self, rules=None):
        rules = rules if rules is not None else party_rules(self.cfg)[int(self.rng.integers(0, 2))]
        lob, mem, (n_anc, n_abs, n_pl) = self.m.party_match(self.now, rules)
        glob, gmem, st = self.eng.party_match(self.now, rules_of(self.cfg, rules))
        assert (st.n_anchors, st.n_absorbed, st.n_parties, st.n_lobbies, st.n_matched) == \
            (n_anc, n_abs, n_pl, len(lob), len(mem))
        assert hdr(glob) == hdr(lob) and np.array_equal(gmem, mem)
        self.count("party_match")
        return lob, mem

    def widen(self, rules=None):
        if rules is None:
            G = self.cfg.n_groups
            rules = {k: v for k, v in rule_sets(self.cfg)[int(self.rng.integers(0, 3))].items()
                     if (k[0] * G + k[1]) % 5 == self.counts.get("widen", 0) % 5}
        lob, mem, n_anc, n_abs = self.m.widen(self.now, rules)
        glob, gmem, st = self.eng.widen(self.now, rules_of(self.cfg, rules))
        assert (st.n_anchors, st.n_absorbed, st.n_lobbies, st.n_matched) == (n_anc, n_abs, len(lob), len(mem))
        assert hdr(glob) == hdr(lob) and np.array_equal(gmem, mem)
        self.count("widen")
        return lob, mem

    def backfill(self, n=300):
        rng, cfg = self.rng, self.cfg
        reqs = (rng.integers(0, cfg.n_modes, n), rng.integers(0, cfg.n_groups, n), rng.integers(self.lo - 200,
                self.hi + 200, n), rng.integers(0, 9, n),
                np.where(rng.random(n) < 0.5, -1, rng.integers(0, 60, n)) if cfg.order_mode == RATING
                else np.full(n, -1))
        want_n, want = self.m.backfill(reqs)
        got_n, got = self.eng.backfill(*reqs)
        assert np.array_equal(got_n, want_n)
        for x, y in zip(got, want):
            assert np.array_equal(x, y)
        self.count("backfill")

    def expire(self, max_wait=None):
        max_wait = int(self.rng.integers(200, 3000)) if max_wait is None else max_wait
        (si, ss), (pi, ps) = self.m.expire(self.now, max_wait)
        ids, seq = self.eng.expire(self.now, max_wait)
        n = len(si)
        assert len(ids) == n + len(pi)
        for (gi, gs), (wi, ws) in (((ids[:n], seq[:n]), (si, ss)), ((ids[n:], seq[n:]), (pi, ps))):
            o, p = np.lexsort((gs, gi)), np.lexsort((ws, wi))
            assert np.array_equal(gi[o], wi[p]) and np.array_equal(gs[o], ws[p])
        self.count("expire")
        return n, len(pi)

    def requeue(self):
        """Matched and taken players back, with queued, removed and matched party members among them."""
        rng, m = self.rng, self.m
        q = m.q
        out = np.setdiff1d(m.active, np.concatenate([q["id"][q["alive"]], m.party_members()]))
        if rng.random() < 0.7:
            out = np.setdiff1d(out, m.party_matched)
        one_each = np.array([p[0][0] for p in m.parties[:6]], np.uint64)  # one queued member of each of 6 parties
        parts = [rng.choice(out, min(len(out), int(rng.integers(1, 3000))), replace=False) if len(out) else out,
                 q["id"][q["alive"]][:20], q["id"][~q["alive"]][:20], one_each]
        ids = np.unique(np.concatenate(parts))
        ids = ids[[int(x) in m.book for x in ids.tolist()]]
        rng.shuffle(ids)
        r, md, ts, seq = np.array([m.book[int(x)] for x in ids.tolist()], np.int64).reshape(-1, 4).T
        try:
            want = m.requeue(ids)
        except ArgRefused:
            self.refused(self.abi.MM_E_ARG, lambda: self.eng.requeue(ids, r, md, ts, seq))
            self.count("requeue_refused")
            return
        assert np.array_equal(self.eng.requeue(ids, r, md, ts, seq), want)
        self.count("requeue")

    def locate(self):
        check_locate(self.eng, self.m, self.sample()[:3000], self.now)
        self.count("locate")

    def option(self):
        rng, eng, m = self.rng, self.eng, self.m
        what = str(rng.choice(["tick_impl", "rank_impl", "max_spread", "async_results", "team_balance", "budget"]))
        if what == "max_spread" and self.cfg.order_mode != RATING:
            what = "tick_impl"
        if what == "tick_impl":
            self.tick_impl ^= 1
            eng.set_option("tick_impl", self.tick_impl)
        elif what == "rank_impl":
            self.rank_impl = int(rng.choice([2, 3]))
            eng.set_option("rank_impl", self.rank_impl)
        elif what == "max_spread":
            m.spread = int(rng.choice([-1, 0, 2, 60]))
            eng.set_option("max_spread", m.spread)
        elif what == "async_results":
            self.async_on = not self.async_on
            if self.at is not None:
                self.at.wait()
            eng.set_option("async_results", int(self.async_on))
            self.at = AsyncTicks(self.pkg, eng, self.cfg.capacity) if self.async_on else None
        elif what == "team_balance":
            m.balance = int(rng.integers(0, 1 << self.cfg.n_modes)) if not m.balance else 0
            m.balance &= sum(1 << k for k in range(self.cfg.n_modes)
                             if self.cfg.modes[k].teams == 2 and self.cfg.modes[k].team_size <= 8)
            eng.set_option("team_balance", m.balance)
        else:
            nq = self.cfg.n_modes * self.cfg.n_groups
            k = int(rng.integers(0, 4))
            m.budget = (rng.integers(0, 30, nq) if k & 1 else None, rng.integers(0, 200, self.cfg.n_modes) if k & 2
                        else None)
            eng.set_lobby_budget(*m.budget)
        self.count(what)

    def snapshot_or_restore(self):
        if self.m.parties and (self.m.snap is None or self.rng.random() < 0.4):
            self.refused(self.abi.MM_E_STATE, self.eng.snapshot)  # a queued party refuses the snapshot
            self.count("snapshot_refused")
            return
        super().snapshot_or_restore()

    def checkpoint(self):
        """export_parties, export_state, import into a fresh engine, merge_parties(keep_seq); the schedule goes on
        with the new engine."""
        if self.at is not None:
            self.at.wait()
        old = self.eng
        pimg = old.export_parties() if self.pcap else None
        img = old.export_state()
        new = self.pkg.Engine(self.cfg)
        try:
            new.import_state(img)
            self.setup(new)
            if pimg is not None:
                assert (new.merge_parties(pimg, keep_seq=True) == 1).all()
        except BaseException:
            new.close()
            raise
        old.close()
        self.eng = new
        if self.async_on:
            new.set_option("async_results", 1)
            self.at = AsyncTicks(self.pkg, new, self.cfg.capacity)
        self.m.checkpoint()
        self.count("checkpoint")

    def queue_move(self):
        """One rating group's queues (every mode) and their parties out to a second engine and back; every other
        party steps aside around the image calls, as SearchPool.move_out / move_in do."""
        if self.at is not None:
            self.at.wait()
        G, a = self.cfg.n_groups, self.eng
        mask = np.zeros((self.cfg.n_modes, G), bool)
        mask[:, int(self.rng.integers(0, G))] = True
        mask = mask.reshape(-1)
        pimg = a.export_parties(mask) if self.pcap else None
        rest = a.export_parties() if self.pcap else None
        qimg = a.export_queues(mask)
        b = self.pkg.Engine(self.cfg)
        try:
            b.merge_queues(qimg)
            if self.pcap:
                b.set_option("party_capacity", self.pcap)
                assert (b.merge_parties(pimg) == 1).all()
                pimg = b.export_parties()
            qimg = b.export_queues(mask)
        finally:
            b.close()
        a.merge_queues(qimg)
        if self.pcap:
            assert (a.merge_parties(rest) == 1).all() and (a.merge_parties(pimg) == 1).all()
        if self.m.queue_move(mask):
            self.count("queue_move")

    OPS = ["enq", "enq", "party", "remove", "take", "tick", "tick", "tick", "option", "option", "snap", "party_match",
           "widen", "backfill", "requeue", "requeue", "expire", "locate", "checkpoint", "queue_move"]

    def step(self):
        rng = self.rng
        self.now += int(rng.integers(1, 400))
        if not self.round:  # every operation once per round, in a random order
            self.round = [o for o in self.OPS if self.parties or o not in ("party", "party_match", "widen")]
            rng.shuffle(self.round)
        op = self.round.pop()
        if op == "enq":
            self.enqueue(min(int(rng.integers(1, 30_000)), max(self.cfg.capacity // 2 - self.m.slots(), 1)))
        elif op == "party":
            self.party_batch(int(rng.integers(50, 600)))
        elif op == "remove":
            self.remove()
        elif op == "take":
            self.take()
        elif op == "tick":
            self.tick()
        elif op == "option":
            self.option()
        elif op == "snap":
            self.snapshot_or_restore()
        else:
            getattr(self, op)()
        self.check()
        return op


# ================================================================================ CPU: the composed model, two ways
def cpu_drive(pkg, oracle, plain, seed, order):
    """A short random schedule on the model alone -> what every step reported."""
    rng = np.random.default_rng(seed)
    cfg = pkg.synth.make_config(groups=[(0, 299), (300, 599), (200, 400)], modes=MODES8[:3], order=order,
                                capacity=4000, active_capacity=100_000, default_group=1)
    m = EngineModel(cfg, oracle, pkg.abi, plain=plain)
    m.pcap = 400 if order == RATING else 0
    nxt, now, log = 0, 1000, []

    def fresh(n):
        nonlocal nxt
        nxt += n
        return pkg.synth.mix64(np.arange(nxt - n, nxt, dtype=np.uint64))

    for step in range(60):
        now += int(rng.integers(1, 40))
        ops = ["enq", "enq", "party", "tick", "party_match", "widen", "backfill", "requeue", "expire", "locate",
               "remove", "take", "option", "move"]
        op = ops[step % len(ops) if step < 2 * len(ops) else int(rng.integers(0, len(ops)))]
        if order == ARRIVAL and op in ("party", "party_match", "widen"):
            op = "tick"
        if op == "enq":
            n = int(rng.integers(50, 400))
            r = rng.integers(-50, 650, n)
            log.append(m.enqueue(fresh(n), r, rng.integers(0, 3, n), (now - rng.integers(0, 80, n)).astype(np.uint32)))
        elif op == "party":
            k = int(rng.integers(5, 40))
            md = rng.integers(1, 3, k).astype(np.uint8)
            size = np.array([rng.integers(2, cfg.modes[x].team_size + 1) for x in md], np.uint8)
            r = np.repeat(rng.integers(-50, 650, k), size) + rng.integers(-5, 6, int(size.sum()))
            log.append(m.enqueue_party(size, fresh(int(size.sum())), r, md, (now - rng.integers(0, 80, k))))
        elif op == "tick":
            ref, seq_of = m.next_tick()
            log.append((hdr(ref.lobbies), ref.member_ids.tolist(), seq_of[ref.emit_seq].tolist()))
            m.apply_tick(ref, now)
            log.append(m.quality())
        elif op == "party_match":
            rules = {(mo, g): (0, 10, 5, 5, 80) for mo in (1, 2) for g in range(3)}
            lob, mem, st = m.party_match(now, rules)
            log.append((hdr(lob), mem.tolist(), st))
        elif op == "widen":
            lob, mem, _, _ = m.widen(now, {(mo, g): (40, 0, 5, 2, 60) for mo in range(3) for g in range(3)})
            log.append((hdr(lob), mem.tolist()))
        elif op == "backfill":
            k = 20
            reqs = (rng.integers(0, 3, k), rng.integers(0, 3, k), rng.integers(-50, 650, k), rng.integers(0, 6, k),
                    np.where(rng.random(k) < 0.5, -1, rng.integers(0, 30, k)) if order == RATING else np.full(k, -1))
            n, out = m.backfill(reqs)
            log.append((n.tolist(), [x.tolist() for x in out]))
        elif op == "requeue":
            q = m.q
            out = np.setdiff1d(m.active, np.concatenate([q["id"][q["alive"]], m.party_members()]))
            ids = np.unique(np.concatenate([out[:200], q["id"][:5]]))
            try:
                log.append(m.requeue(ids))
            except ArgRefused as e:
                log.append(str(e))
        elif op == "expire":
            log.append([x.tolist() for pair in m.expire(now, 60) for x in pair])
        elif op == "locate":
            ids = np.concatenate([m.q["id"][:300], m.party_members()[:20], m.active[:50]])
            log.append({k: v.tolist() for k, v in m.locate(ids, now).items()})
        elif op == "remove":
            log.append(m.remove(np.concatenate([m.q["id"][::7], m.party_members()[::5]])))
        elif op == "take":
            log.append(m.take(m.q["id"][3::11]))
        elif op == "move":
            mask = np.zeros((cfg.n_modes, cfg.n_groups), bool)
            mask[:, step % cfg.n_groups] = True
            log.append(m.queue_move(mask.reshape(-1)))
        else:
            m.balance = int(rng.integers(0, 8))
            nq = cfg.n_modes * cfg.n_groups
            m.budget = (rng.integers(0, 5, nq), None) if rng.random() < 0.5 else (None, None)
            m.spread = int(rng.choice([-1, 0, 7])) if order == RATING else -1
        log.append((op, m.pool()["id"].tolist(), sorted(m.active.tolist()), m.seq_next,
                    [(p[0].tolist(), p[4]) for p in m.parties]))
    return log


def same(a, b):
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        return np.array_equal(a, b)
    if isinstance(a, (list, tuple)):
        return type(a) is type(b) and len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    return a == b


@pytest.mark.parametrize("order", [RATING, ARRIVAL])
@pytest.mark.parametrize("seed", range(3))
def test_model_on_plain_and_binned_restatements_agree(pkg, oracle, order, seed):
    """The composed model, once on the one-at-a-time restatements and once on the binned / numpy ones: every result
    of every step and the state after it agree.  (The plain widen gives no anchor counts: those two are skipped.)"""
    a = cpu_drive(pkg, oracle, True, seed, order)
    b = cpu_drive(pkg, oracle, False, seed, order)
    assert len(a) == len(b)
    for k, (x, y) in enumerate(zip(a, b)):
        assert same(x, y), k
    ops = [x[0] for x in a if isinstance(x, tuple) and len(x) == 5 and isinstance(x[0], str)]
    for op in ("tick", "backfill", "requeue", "expire", "locate", "move") + (("party_match", "widen") if order == RATING
                                                                        else ()):
        assert op in ops, op


def test_model_requeue_of_a_matched_party(pkg, oracle):
    """Members of a matched party share the party's seq: two of them in one call are refused, one at a time the
    second is refused when the first is live in its partition, and not when it went to another partition."""
    cfg = pkg.synth.make_config(groups=[(0, 99), (100, 199)], modes=MODES8[1:2], order=RATING, capacity=1000,
                                active_capacity=10_000, default_group=-1)
    m = EngineModel(cfg, oracle, pkg.abi)
    m.pcap = 100
    ids = np.arange(1, 11, dtype=np.uint64) + np.uint64(1 << 40)
    m.enqueue(ids[4:], [50, 50, 150, 150, 50, 50], np.zeros(6, np.uint8))
    assert (m.enqueue_party([2, 2], ids[:4], [50, 50, 50, 150], [0, 0], [0, 0]) == 1).all()
    lob, mem, _ = m.party_match(10, {(0, 0): (0, 10, 1, 0, 10)})
    assert mem[:2].tolist() == ids[:2].tolist()
    with pytest.raises(ArgRefused):
        m.requeue(ids[:2])
    assert m.requeue(ids[:1]).tolist() == [1]
    with pytest.raises(ArgRefused):
        m.requeue(ids[1:2])


# ================================================================================ GPU: long mixed schedules
SCHEDULES = [(dense, wide) for dense in (False, True) for wide in (0, 1)]


def run_schedule(pkg, oracle, cfg, rng, dense, steps, parties=True):
    s = EngineSchedule(pkg, oracle, cfg, rng, dense, parties=parties)
    ops = []
    try:
        s.m.balance = sum(1 << k for k in range(cfg.n_modes))  # two-team modes of at most 8 a side; options toggle it
        s.eng.set_option("team_balance", s.m.balance)
        s.m.budget = (rng.integers(0, 30, cfg.n_modes * cfg.n_groups), None)  # until an option step changes it
        s.eng.set_lobby_budget(*s.m.budget)
        s.players(60_000, old=0.02)
        if s.parties:
            s.party_batch(800)
        s.check()
        for _ in range(steps):
            ops.append(s.step())
        s.tick()
        s.finish()
        s.check()
    finally:
        s.close()
    return s, ops


@pytest.mark.gpu
@pytest.mark.parametrize("dense,wide", SCHEDULES, ids=lambda v: str(v))
def test_every_call_against_the_model(pkg, oracle, dense, wide):
    rng = np.random.default_rng(500 + 2 * dense + wide)
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[:3], order=RATING, capacity=300_000,
                                active_capacity=4_000_000, default_group=-1,
                                flags=(DENSE if dense else 0) | WIDE * wide)
    s, ops = run_schedule(pkg, oracle, cfg, rng, dense, 150)
    c = s.counts
    for what in ("party_match", "widen", "backfill", "requeue", "expire", "locate", "checkpoint", "queue_move",
                 "budgeted_tick", "balanced_tick", "enqueue_party"):
        assert c.get(what, 0) >= 3, (what, c)
    assert ops.count("tick") >= 10, ops


@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True])
def test_arrival_order_against_the_model(pkg, oracle, dense):
    """No parties and no widen (both refuse arrival order): oldest-first backfill and the arrival path of
    team_balance."""
    rng = np.random.default_rng(600 + dense)
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[:3], order=ARRIVAL, capacity=300_000,
                                active_capacity=4_000_000, default_group=-1, flags=DENSE if dense else 0)
    s, ops = run_schedule(pkg, oracle, cfg, rng, dense, 100, parties=False)
    for what in ("backfill", "requeue", "expire", "locate", "checkpoint", "queue_move", "balanced_tick"):
        assert s.counts.get(what, 0) >= 3, (what, s.counts)


# ================================================================================ GPU: the tile geometries
def geometry_config(pkg, case):
    """-> (cfg, rating lo, rating hi) of a config only the tick had met."""
    syn = pkg.synth
    if case in ("huge_domain", "huge_domain_split"):
        return syn.make_config(groups=[(0, 20000)], modes=MODES8[3:4], order=RATING, capacity=400_000,
                               active_capacity=2_000_000, default_group=0,
                               flags=WIDE if case == "huge_domain" else 0), -100, 20100
    if case == "key_domain_edge":
        span = key_domain_edge(pkg, lambda c: Layout(c).ok)
        return edge_config(pkg, span, capacity=400_000), -3, span + 3
    if case == "many_partitions":
        return syn.make_config(groups=[(250 * g, 250 * g + 249) for g in range(20)], modes=MODES8, order=RATING,
                               capacity=400_000, active_capacity=2_000_000, default_group=-1), 0, 5000
    if case == "fallback":
        return syn.make_config(groups=fallback_groups(), modes=MODES8, order=RATING, capacity=400_000,
                               active_capacity=2_000_000, default_group=-1), 0, 5000
    assert case == "overlap"
    return syn.make_config(groups=OVERLAP, modes=MODES8, order=RATING, capacity=400_000, active_capacity=2_000_000,
                           default_group=1), -300, 5400


GEOMETRIES = ["huge_domain", "huge_domain_split", "key_domain_edge", "many_partitions", "fallback", "overlap"]


def off_tick_round(s, n_players, n_parties):
    """Every off-tick call once against the model, then a balanced tick and its report."""
    s.players(n_players, old=0.003)
    # parties of every size 2 .. S of every mode that holds them
    ok = [k for k in range(s.cfg.n_modes) if s.cfg.modes[k].team_size >= 2]
    s.party_batch(n_parties)
    for k in ok:
        sizes = np.tile(np.arange(2, s.cfg.modes[k].team_size + 1), 40)
        assert (party_batch_of(s, sizes.tolist(), k) == 1).all()
    s.check()
    s.now += 100
    G = s.cfg.n_groups
    s.party_match({(m, g): (0, 30, 5, 5, 200) for m in ok for g in range(G)})
    s.check()
    s.widen({(m, g): (900, 5, 10, 5, 400) for m in range(s.cfg.n_modes) for g in range(G)})
    s.check()
    s.backfill(2000)
    s.check()
    n_solo, n_party = s.expire(1030)
    assert n_solo > 0
    s.check()
    s.m.balance = sum(1 << k for k in range(s.cfg.n_modes) if s.cfg.modes[k].teams == 2 and
                      s.cfg.modes[k].team_size <= 8)
    s.eng.set_option("team_balance", s.m.balance)
    s.locate()
    s.tick()
    s.check()


def party_batch_of(s, sizes, mode):
    """Parties of the given sizes in one mode, each near its own rating."""
    n = len(sizes)
    ids = s.fresh(int(sum(sizes)))
    r = (np.repeat(s.rng.integers(s.lo, s.hi, n), sizes) + s.rng.integers(-20, 21, len(ids))).astype(np.int32)
    md = np.full(n, mode, np.uint8)
    ts = (s.now - s.rng.integers(0, 60, n)).astype(np.uint32)
    want = s.m.enqueue_party(np.array(sizes, np.uint8), ids, r, md, ts)
    assert np.array_equal(s.eng.enqueue_party(np.array(sizes, np.uint8), ids, r, md, ts), want)
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("case", GEOMETRIES)
def test_off_tick_calls_at_tile_geometries(pkg, oracle, case):
    cfg, lo, hi = geometry_config(pkg, case)
    s = EngineSchedule(pkg, oracle, cfg, np.random.default_rng(GEOMETRIES.index(case)), False, lo=lo, hi=hi,
                       pcap=100_000)
    try:
        off_tick_round(s, 200_000, 3000)
    finally:
        s.close()
    assert s.counts["party_match"] == s.counts["widen"] == s.counts["backfill"] == 1


@pytest.mark.gpu
@pytest.mark.parametrize("teams", [3, 40, 256])
def test_party_modes_of_many_teams(pkg, oracle, teams):
    """Teams of two: duo3, a mode past the warp-stride room loops, and kPtMaxTeams itself."""
    cfg = pkg.synth.make_config(groups=[(0, 999), (1000, 1999)], modes=[("duo", teams, 2), ("5v5", 2, 5)],
                                order=RATING, capacity=400_000, active_capacity=2_000_000, default_group=-1)
    s = EngineSchedule(pkg, oracle, cfg, np.random.default_rng(teams), False, lo=0, hi=2000)
    try:
        s.players(150_000)
        party_batch_of(s, [2] * 3000, 0)
        party_batch_of(s, [2, 3, 4, 5] * 300, 1)
        s.check()
        s.now += 100
        lob, mem = s.party_match({(m, g): (0, 40, 5, 10, 400) for m in range(2) for g in range(2)})
        assert (lob["mode"] == 0).sum() > 0
        s.check()
    finally:
        s.close()


@pytest.mark.gpu
def test_party_mode_of_257_teams_is_refused(pkg, oracle):
    cfg = pkg.synth.make_config(groups=[(0, 999)], modes=[("t257", 257, 2), ("2v2", 2, 2)], order=RATING,
                                capacity=100_000, active_capacity=400_000, default_group=-1)
    s = EngineSchedule(pkg, oracle, cfg, np.random.default_rng(7), False, lo=0, hi=1000)
    try:
        s.players(20_000)
        party_batch_of(s, [2] * 200, 0)
        party_batch_of(s, [2] * 200, 1)
        s.check()
        rules = {(0, 0): (0, 40, 5, 10, 400), (1, 0): (0, 40, 5, 10, 400)}
        s.refused(pkg.abi.MM_E_ARG, lambda: s.eng.party_match(s.now, rules_of(cfg, rules)))
        s.check()
        s.party_match({(1, 0): (0, 40, 5, 10, 400)})  # the mode with the rule off is not served: accepted
        s.check()
    finally:
        s.close()


@pytest.mark.gpu
def test_party_table_of_many_tiles_with_a_crowded_bin(pkg, oracle):
    """More than 3 x 1024 parties, 2 000 of them at one rating: that bin's rows straddle warps and scatter tiles."""
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[2:4] + MODES8[6:7], order=RATING,
                                capacity=400_000, active_capacity=2_000_000, default_group=-1)
    s = EngineSchedule(pkg, oracle, cfg, np.random.default_rng(11), False, lo=0, hi=5001, pcap=200_000)
    try:
        s.players(150_000)
        s.party_batch(2000)
        s.party_batch(2000, sizes=None, crowd=2500)
        party_batch_of(s, [6] * 200 + [2, 3, 4, 5] * 100, 2)  # whole-team parties in 6v6
        assert len(s.m.parties) > 3 * 1024
        s.check()
        for k in range(3):
            s.now += 50
            s.party_match({(m, g): (0, 5 + 20 * k, 5, 5, 100) for m in range(3) for g in range(cfg.n_groups)})
            s.check()
    finally:
        s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
def test_balanced_eight_a_side_at_clamped_ratings(pkg, oracle, order):
    cfg = pkg.synth.make_config(groups=OVERLAP, modes=[("8v8", 2, 8), ("5v5", 2, 5)], order=order, capacity=300_000,
                                active_capacity=2_000_000, default_group=1)
    s = EngineSchedule(pkg, oracle, cfg, np.random.default_rng(13 + order), False, parties=False, lo=-3000, hi=8000)
    try:
        s.m.balance = 3
        s.eng.set_option("team_balance", 3)
        for _ in range(3):
            s.players(60_000, old=0.01)
            s.check()
            s.tick()
            s.check()
            if order == RATING:
                s.widen({(m, g): (900, 50, 10, 50, 4000) for m in range(2) for g in range(cfg.n_groups)})
                s.check()
    finally:
        s.close()


# ================================================================================ GPU: matched players of an image
@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True])
@pytest.mark.parametrize("parties", [False, True])
def test_imported_matched_players_stay_matched(pkg, oracle, dense, parties):
    """mm_import puts the matched and taken players of an image in the active set as matched players, not as
    members of party row 0: with a party in that row, and on an engine without a party table, mm_locate reports them
    in state 2, mm_remove of one removes that one player only and mm_requeue gives the others code 1."""
    cfg = pkg.synth.make_config(groups=[(0, 99), (100, 199)], modes=MODES8[1:2], order=RATING, capacity=10_000,
                                active_capacity=10_000, default_group=-1, flags=DENSE if dense else 0)
    s = EngineSchedule(pkg, oracle, cfg, np.random.default_rng(5), dense, parties=parties, lo=0, hi=200, pcap=100)
    try:
        s.players(401)
        s.tick()  # matched players, and one left queued
        matched = np.setdiff1d(s.m.active, s.m.q["id"])[:2]
        taken = s.m.q["id"][:1]
        assert len(matched) == 2 and s.eng.take(taken) == s.m.take(taken) == 1
        s.checkpoint()  # export, import into a fresh engine
        if parties:  # row 0 of the new engine's party table
            ids, r = s.fresh(2), np.array([50, 60], np.int32)
            want = s.m.enqueue_party([2], ids, r, [0], [s.now])
            assert want[0] == 1 and np.array_equal(s.eng.enqueue_party([2], ids, r, [0], [s.now]), want)
            assert len(s.m.parties) == 1
        s.check()
        out = np.concatenate([matched, taken])
        assert (check_locate(s.eng, s.m, out, s.now)["state"] == 2).all()
        assert s.eng.remove(out[:1]) == s.m.remove(out[:1]) == 1
        s.check()
        cols = np.array([s.m.book[int(x)] for x in out[1:].tolist()], np.int64).T
        want = s.m.requeue(out[1:])
        assert (want == 1).all() and np.array_equal(s.eng.requeue(out[1:], *cols), want)
        s.check()
        s.tick()
        s.check()
    finally:
        s.close()


# ================================================================================ GPU: requeue of a matched party
@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True])
def test_requeue_of_matched_party_members(pkg, oracle, dense):
    """Members of a party share its enqueue sequence number, and mm_requeue puts a member back as a solo with it.  So
    two members in one call are refused (MM_E_ARG: not in strict age order); one at a time, a member whose partition
    already holds a requeued co-member is refused (MM_E_ARG: the seq of a live player there), and one that goes to
    another partition is requeued.  Nothing changes on a refusal."""
    cfg = pkg.synth.make_config(groups=[(0, 99), (100, 199)], modes=MODES8[2:3], order=RATING, capacity=10_000,
                                active_capacity=10_000, default_group=-1, flags=DENSE if dense else 0)
    s = EngineSchedule(pkg, oracle, cfg, np.random.default_rng(3), dense, pcap=100, lo=0, hi=200)
    try:
        ids = s.fresh(3)
        r = np.array([50, 50, 150], np.int32)  # R = 83: group 0; the third member's own rating maps to group 1
        want = s.m.enqueue_party([3], ids, r, [0], [s.now])
        assert np.array_equal(s.eng.enqueue_party([3], ids, r, [0], [s.now]), want) and want[0] == 1
        sol = s.fresh(3)
        sr, sm, st = np.array([80, 80, 80], np.int32), np.zeros(3, np.uint8), np.full(3, s.now, np.uint32)
        assert np.array_equal(s.eng.enqueue(sol, sr, sm, st), s.m.enqueue(sol, sr, sm, st))
        lob, mem = s.party_match({(0, 0): (0, 50, 1, 0, 50)})
        assert sorted(mem[:3].tolist()) == sorted(ids.tolist()) and len(mem) == 6
        s.check()
        seq = s.m.book[int(ids[0])][3]
        assert all(s.m.book[int(x)][3] == seq for x in ids.tolist())
        cols = lambda k: tuple(np.array([s.m.book[int(x)][j] for x in ids[k].tolist()]) for j in range(4))  # noqa
        for k in ([0, 1], [0, 2], [0, 1, 2]):  # several members in one call
            with pytest.raises(ArgRefused):
                s.m.requeue(ids[k])
            s.refused(pkg.abi.MM_E_ARG, lambda: s.eng.requeue(ids[k], *cols(k)))
            s.check()
        assert np.array_equal(s.eng.requeue(ids[:1], *cols([0])), s.m.requeue(ids[:1]))
        s.check()
        with pytest.raises(ArgRefused):
            s.m.requeue(ids[1:2])  # same partition as member 0, which is live there with the party's seq
        s.refused(pkg.abi.MM_E_ARG, lambda: s.eng.requeue(ids[1:2], *cols([1])))
        s.check()
        got = s.eng.requeue(ids[2:3], *cols([2]))
        assert np.array_equal(got, s.m.requeue(ids[2:3])) and got.tolist() == [1]  # another partition
        s.check()
        s.tick()
        s.check()
    finally:
        s.close()
