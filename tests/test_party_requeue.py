"""Party requeue (mm_requeue_party / Engine.requeue_party / SearchPool(requeue_parties=True)): the parties of a lobby
that did not start go back into the party table as parties, at the position their enqueue sequence numbers give them.

The restatement extends `EngineModel` (tests/test_engine_model.py) with the call: codes 0 / 4 / 1 in that order, every
refusal, and the merge of the requeued parties into the model's age-ordered party table.  Everything else the model
restates (pool, active set, seq_next, party table, locate, the next mm_party_match through restate_bins) is compared
after every step by check_engine.

CPU: SearchPool routing of a lobby's players (whole parties, several members of a party, a lone member, solos beside
them, a refused party call, a second lone member of a party, the option off), remove_user and checkpoint / resume of
the matched-party book, on an engine double.
GPU, on hashed and dense ids: where a party lands (an empty table, before the first row, after the last and between
every pair of live rows, among dead rows left by mm_party_match, mm_remove, mm_expire and mm_export_parties, and after
mm_export_parties + mm_merge_parties(MM_PARTY_KEEP_SEQ) on the same engine, whose released rows sit before the live
rows of older numbers); a table
of more than 3 x 1024 rows with a crowded bin, parties of every size, modes of 3 and 40 teams; codes 0 and 4 and their
order, after a checkpoint and after a queue move; the twin engine of the header's EQUIVALENCE; every refusal and the
exact room boundary; mixed schedules of every call with requeue_party among them; and a SearchPool end to end.
"""
import ctypes as C
import importlib

import numpy as np
import pytest

from .test_engine_model import (ArgRefused, EngineModel, EngineSchedule, U32, check_locate,
                                party_batch_of)
from .test_expire import r_wait
from .test_parties import party_rating, party_engine, publish_party
from .test_tile_geometry import DENSE, MODES8
from .test_widen import rules_of

RATING = 1


class CapRefused(Exception):
    """The restated call is refused with MM_E_CAP: nothing changes."""


# ================================================================================ the restatement
class RequeueModel(EngineModel):
    """EngineModel with the matched parties remembered (what a caller keeps) and mm_requeue_party."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.matched_parties = []  # [ids, ratings, mode, ts, seq] of the parties mm_party_match placed

    def party_match(self, now, rules):
        before = list(self.parties)
        out = super().party_match(now, rules)
        kept = {id(p) for p in self.parties}
        self.matched_parties += [p for p in before if id(p) not in kept]
        return out

    def requeue_party(self, parties):
        """parties: [(ids, ratings, mode, ts, seq)] in the caller's order -> codes; ArgRefused / CapRefused where the
        engine refuses."""
        cfg = self.cfg
        ages = [(int(p[4]) - self.seq_next) & U32 for p in parties]
        order = sorted(range(len(parties)), key=lambda j: ages[j])  # Engine.requeue_party sorts by age
        flat = [int(x) for p in parties for x in p[0]]
        for p in parties:
            s, md = len(p[0]), int(p[2])
            if md >= cfg.n_modes or s < 2 or s > cfg.modes[md].team_size:
                raise ArgRefused("mode or size")
            if self.groups(np.array([party_rating(p[1])], np.int64))[0] < 0:
                raise ArgRefused("an R without a group")
        if any(x >= self.id_limit for x in flat) or len(set(flat)) < len(flat):
            raise ArgRefused("an id out of range or twice")
        srt = [ages[j] for j in order]
        if any(a == 0 for a in srt) or any(b <= a for a, b in zip(srt, srt[1:])):
            raise ArgRefused("not in strict age order, or seq_next")
        q = self.q
        queued = set(q["id"][q["alive"]].tolist()) | set(self.party_members().tolist())
        active = set(self.active.tolist())
        codes = []
        for p in parties:
            ids = [int(x) for x in p[0]]
            codes.append(0 if any(x in queued for x in ids) else (4 if any(x not in active for x in ids) else 1))
        one = [p for p, c in zip(parties, codes) if c == 1]
        live_seq = {int(p[4]) for p in self.parties}
        if any(int(p[4]) in live_seq for p in one):
            raise ArgRefused("the seq of a queued party")
        if sum(len(p[0]) for p in one) > self.pcap - len(self.party_members()):
            raise CapRefused()
        back = set()
        for p in one:
            self.parties.append([np.asarray(p[0], np.uint64), np.asarray(p[1], np.int64), int(p[2]), int(p[3]),
                                 int(p[4])])
            back.update(int(x) for x in p[0])
        self.parties.sort(key=lambda p: (p[4] - self.seq_next) & U32)
        self.party_matched = self.party_matched[~np.isin(self.party_matched, list(back))]
        self.matched_parties = [p for p in self.matched_parties if int(p[0][0]) not in back]
        return np.array(codes, np.uint8)


def columns(parties):
    """[(ids, ratings, mode, ts, seq)] -> the arguments of Engine.requeue_party"""
    sizes = np.array([len(p[0]) for p in parties], np.uint8)
    cat = lambda k, dt: (np.concatenate([np.asarray(p[k], dt) for p in parties]) if parties  # noqa: E731
                         else np.zeros(0, dt))
    return (sizes, cat(0, np.uint64), cat(1, np.int32), np.array([p[2] for p in parties], np.uint8),
            np.array([p[3] for p in parties], np.uint32), np.array([p[4] for p in parties], np.uint32))


class RequeueSchedule(EngineSchedule):
    """EngineSchedule on the RequeueModel, with a requeue_party step."""

    def __init__(self, pkg, oracle, cfg, rng, dense, **k):
        super().__init__(pkg, oracle, cfg, rng, dense, **k)
        self.m = RequeueModel(cfg, oracle, pkg.abi)
        self.setup(self.eng)

    def requeue_party(self, parties=None, expect=None):
        """Requeue `parties` (default: a random choice of the matched parties, a few cut to their first members, a
        queued party, a party with a removed member) on both; -> codes."""
        m, rng = self.m, self.rng
        if parties is None:
            if not m.matched_parties:
                self.party_match()
            mp = list({p[4]: p for p in m.matched_parties}.values())  # one record per seq
            k = min(len(mp), int(rng.integers(1, 400)))
            parties = [mp[j] for j in rng.choice(len(mp), k, replace=False)] if k else []
            parties = [p if len(p[0]) < 3 or rng.random() < 0.8 else (p[0][:2], p[1][:2], p[2], p[3], p[4])
                       for p in parties]
            if m.parties and rng.random() < 0.5:
                parties.append(m.parties[int(rng.integers(0, len(m.parties)))])
            rng.shuffle(parties)
        try:
            want = m.requeue_party(parties)
        except ArgRefused:
            self.refused(self.abi.MM_E_ARG, lambda: self.eng.requeue_party(*columns(parties)))
            self.count("requeue_party_refused")
            return None
        except CapRefused:
            self.refused(self.abi.MM_E_CAP, lambda: self.eng.requeue_party(*columns(parties)))
            self.count("requeue_party_refused")
            return None
        got = self.eng.requeue_party(*columns(parties))
        assert np.array_equal(got, want)
        if expect is not None:
            assert got.tolist() == expect
        self.count("requeue_party")
        self.count(f"requeue_party_{sorted(set(got.tolist()))}")
        return got

    OPS = EngineSchedule.OPS + ["requeue_party", "requeue_party", "party_match"]


def requeued_locate(s, parties, model=True):
    """mm_locate of every member of the given (requeued) parties: state 3, the party's seq, the wait from its stamp.
    model: also against the model's locate (which predicts the next tick through the C oracle)."""
    ids = np.concatenate([np.asarray(p[0], np.uint64) for p in parties])
    rec = check_locate(s.eng, s.m, ids, s.now) if model else s.eng.locate(ids, s.now)
    assert (rec["state"] == 3).all()
    assert np.array_equal(rec["seq"], np.concatenate([np.full(len(p[0]), p[4], np.uint32) for p in parties]))
    ts = np.concatenate([np.full(len(p[0]), p[3], np.uint32) for p in parties])
    assert np.array_equal(rec["wait"], r_wait(s.now, ts))
    assert s.eng.in_queue(ids).all()


def small_config(pkg, dense, modes=(("2v2", 2, 2), ("5v5", 2, 5)), groups=((0, 999), (1000, 1999))):
    return pkg.synth.make_config(groups=list(groups), modes=list(modes), order=RATING, capacity=100_000,
                                 active_capacity=400_000, default_group=-1, flags=DENSE if dense else 0)


KINDS = [False, True]
kind_id = lambda d: "dense" if d else "hashed"  # noqa: E731


# ================================================================================ CPU: the restatement, hand-built
def test_restatement_codes_order_and_placement(pkg, oracle):
    cfg = small_config(pkg, False)
    m = RequeueModel(cfg, oracle, pkg.abi)
    m.pcap = 100
    ids = np.arange(1, 13, dtype=np.uint64)
    assert (m.enqueue_party([2, 2, 2, 2], ids[:8], [500] * 8, [0, 1, 0, 1], [0] * 4) == 1).all()
    lob, mem, _ = m.party_match(10, {(0, 0): (0, 10, 1, 0, 10)})  # the two 2v2 parties (seq 0 and 2)
    assert sorted(mem.tolist()) == [1, 2, 5, 6] and [p[4] for p in m.matched_parties] == [0, 2]
    a, b = m.matched_parties
    # before the first live row and between the two: the table is in age order again
    assert m.requeue_party([b, a]).tolist() == [1, 1]
    assert [p[4] for p in m.parties] == [0, 1, 2, 3]
    # code 0 before code 4: a queued member and a gone one in one party
    m.remove(ids[2:3])  # dissolves the party of seq 1
    assert m.requeue_party([(np.array([1, 3], np.uint64), [500, 500], 0, 0, 7)]).tolist() == [0]
    assert m.requeue_party([(np.array([3, 9], np.uint64), [500, 500], 0, 0, 7)]).tolist() == [4]


# ================================================================================ GPU: where a party lands
@pytest.mark.gpu
@pytest.mark.parametrize("dense", KINDS, ids=kind_id)
def test_where_the_party_lands(pkg, oracle, dense):
    """2v2 parties (served) between 5v5 parties (not served): after the 2v2 ones are matched, the 5v5 rows are the
    live rows and requeue puts the 2v2 parties before the first, between every pair and after the last.  Dead rows of
    mm_party_match, mm_remove, mm_expire and mm_export_parties are still in the table when the call merges."""
    cfg = small_config(pkg, dense)
    s = RequeueSchedule(pkg, oracle, cfg, np.random.default_rng(1), dense, pcap=10_000, lo=0, hi=2000)
    try:
        s.now += 10_000
        s.players(3000)
        n = 40
        sizes = [2 if j % 2 == 0 else 2 + j % 4 for j in range(2 * n)]
        mode = np.array([j % 2 for j in range(2 * n)], np.uint8)
        ids = s.fresh(sum(sizes))
        base = np.where(mode == 0, 500, np.where(np.arange(2 * n) < n, 300, 1500))  # 5v5 in both groups
        r = np.repeat(base, sizes).astype(np.int32)
        ts = np.full(2 * n, s.now, np.uint32)
        ts[1:12:2] = s.now - 5000  # old 5v5 parties: mm_expire takes them
        want = s.m.enqueue_party(np.array(sizes, np.uint8), ids, r, mode, ts)
        assert (want == 1).all() and np.array_equal(s.eng.enqueue_party(np.array(sizes, np.uint8), ids, r, mode, ts),
                                                    want)
        s.check()
        lob, mem = s.party_match({(0, 0): (0, 10, 1, 0, 10)})
        assert len(lob) == n // 2 and len(s.m.matched_parties) == n
        first = s.m.parties[2][0][:1]  # a 5v5 member: mm_remove dissolves its party
        assert s.eng.remove(first) == s.m.remove(first)
        s.expire(4000)
        mask = np.zeros((cfg.n_modes, cfg.n_groups), bool)
        mask[1, 1] = True
        img = s.eng.export_parties(mask.reshape(-1))
        _h, pc = pkg.engine.read_party_image(img)
        out = np.split(pc["id"].astype(np.uint64), np.cumsum(pc["size"].astype(np.int64))[:-1])
        assert len(out) > 3
        s.m.remove(np.array([x[0] for x in out], np.uint64))  # what the export leaves (header EQUIVALENCE)
        s.check()
        live = [p[4] for p in s.m.parties]
        back = list(s.m.matched_parties)
        ages = [(p[4] - s.m.seq_next) & U32 for p in back]
        lages = [(x - s.m.seq_next) & U32 for x in live]
        assert min(ages) < min(lages) and max(ages) > max(lages)  # before the first and after the last live row
        between = {sum(a > b for b in lages) for a in ages}
        assert between == set(range(len(lages) + 1))  # and in every gap between two live rows
        s.requeue_party(back, expect=[1] * len(back))
        s.check()
        requeued_locate(s, back)
        # the next match: the requeued parties are the oldest, the first anchors first
        s.now += 5
        lob, mem = s.party_match({(0, 0): (0, 10, 1, 0, 10)})
        assert mem[:2].tolist() == back[0][0].tolist()
        s.check()
        # an empty table: a fresh engine of the checkpoint, the matched parties in the image's active section
        s.checkpoint()
        assert s.eng.party_read()["size"].size == len(s.m.parties)
        s.eng.export_parties()  # every queued party out: the table is empty (no rows at all after the merge below)
        s.m.remove(np.array([p[0][0] for p in s.m.parties], np.uint64))
        s.checkpoint()
        assert len(s.m.parties) == 0
        back = list(s.m.matched_parties)
        s.requeue_party(back[:1], expect=[1])
        s.check()
        s.requeue_party(back[1:], expect=[1] * (len(back) - 1))
        s.check()
        requeued_locate(s, back)
        s.tick()
        s.check()
    finally:
        s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dense", KINDS, ids=kind_id)
def test_many_rows_crowded_bin_every_size_and_many_teams(pkg, oracle, dense):
    """More than 3 x 1024 rows, most of them at one rating; parties of every size 2 .. S; modes of 3 and 40 teams."""
    cfg = pkg.synth.make_config(groups=[(0, 999), (1000, 1999)], modes=[("duo3", 3, 2), ("duo40", 40, 2),
                                                                        ("6v6", 2, 6)],
                                order=RATING, capacity=400_000, active_capacity=2_000_000, default_group=-1,
                                flags=DENSE if dense else 0)
    s = RequeueSchedule(pkg, oracle, cfg, np.random.default_rng(3 + dense), dense, pcap=200_000, lo=0, hi=2000)
    try:
        s.players(100_000)
        party_batch_of(s, [2] * 1500, 0)
        party_batch_of(s, [2] * 1500, 1)
        party_batch_of(s, [2, 3, 4, 5, 6] * 200, 2)
        s.party_batch(1200, crowd=700)
        assert len(s.m.parties) > 3 * 1024
        s.check()
        rules = {(m, g): (0, 30, 5, 10, 300) for m in range(3) for g in range(2)}
        for k in range(2):
            s.now += 50
            lob, mem = s.party_match(rules)
            assert len(lob) > 0
            s.check()
            back = list(s.m.matched_parties)
            assert {len(p[0]) for p in back} >= {2, 3, 4, 5, 6} and {p[2] for p in back} == {0, 1, 2}
            s.requeue_party(back, expect=[1] * len(back))
            s.check()
            requeued_locate(s, back[::37], model=False)  # the oracle's tick takes no 40-team mode
        s.now += 50
        s.party_match(rules)
        s.check()
    finally:
        s.close()


# ================================================================================ GPU: after a hand-over in place
@pytest.mark.gpu
@pytest.mark.parametrize("dense", KINDS, ids=kind_id)
def test_requeue_after_export_and_merge_back_on_the_same_engine(pkg, oracle, dense):
    """SearchPool.checkpoint and move_out release every queued party and merge it back with its number on the same
    engine: the released rows stay in the table, before the merged live rows of the same (and younger) numbers, until
    a compaction.  Matched parties interleaved with those live rows then go back between them, and a party with the
    seq of a live row is refused."""
    cfg = small_config(pkg, dense)
    s = RequeueSchedule(pkg, oracle, cfg, np.random.default_rng(21 + dense), dense, pcap=10_000, lo=0, hi=2000)
    try:
        s.players(2000)
        n = 30
        sizes = [2 if j % 2 == 0 else 2 + j % 4 for j in range(2 * n)]
        mode = np.array([j % 2 for j in range(2 * n)], np.uint8)
        ids = s.fresh(sum(sizes))
        r = np.repeat(np.where(mode == 0, 500, 300), sizes).astype(np.int32)
        ts = np.full(2 * n, s.now, np.uint32)
        want = s.m.enqueue_party(np.array(sizes, np.uint8), ids, r, mode, ts)
        assert (want == 1).all() and np.array_equal(s.eng.enqueue_party(np.array(sizes, np.uint8), ids, r, mode, ts),
                                                    want)
        s.party_match({(0, 0): (0, 10, 1, 0, 10)})  # every 2v2 party; the 5v5 ones stay, one between each two
        back = sorted(s.m.matched_parties, key=lambda p: (p[4] - s.m.seq_next) & U32)
        assert len(back) == n and len(s.m.parties) == n

        def in_place():  # the checkpoint's hand-over on the running engine
            img = s.eng.export_parties()
            assert (s.eng.merge_parties(img, keep_seq=True) == 1).all()
            s.check()

        in_place()
        live = s.m.parties[n // 2]
        s.requeue_party([(back[0][0], back[0][1], 0, back[0][3], live[4])])  # the seq of a queued party: refused
        assert s.counts.get("requeue_party_refused") == 1
        s.check()
        s.requeue_party(back[1::2], expect=[1] * len(back[1::2]))
        s.check()
        requeued_locate(s, back[1::2])
        in_place()  # the table again: released rows, then the live ones
        s.requeue_party(back[0::2], expect=[1] * len(back[0::2]))
        s.check()
        requeued_locate(s, back)
        s.now += 5
        lob, mem = s.party_match({(0, 0): (0, 10, 1, 0, 10)})
        assert mem[:2].tolist() == back[0][0].tolist()  # the oldest anchors first
        s.check()
    finally:
        s.close()


# ================================================================================ GPU: codes
@pytest.mark.gpu
@pytest.mark.parametrize("dense", KINDS, ids=kind_id)
def test_codes_and_their_order(pkg, oracle, dense):
    """A member requeued earlier as a solo gives 0, a removed member 4, both 0; after a checkpoint (matched players
    from an image load) and after a queue move."""
    cfg = small_config(pkg, dense)
    s = RequeueSchedule(pkg, oracle, cfg, np.random.default_rng(5), dense, pcap=1000, lo=0, hi=2000)
    try:
        s.players(500)
        sizes = [5] * 12  # two whole-team parties make a lobby
        ids = s.fresh(60)
        r = np.repeat([300, 300, 300, 1200, 1200, 1200] * 2, 5).astype(np.int32)
        md = np.ones(12, np.uint8)
        want = s.m.enqueue_party(np.array(sizes, np.uint8), ids, r, md, np.full(12, s.now, np.uint32))
        assert np.array_equal(s.eng.enqueue_party(np.array(sizes, np.uint8), ids, r, md,
                                                  np.full(12, s.now, np.uint32)), want)
        s.party_match({(1, g): (0, 10, 1, 0, 10) for g in range(2)})
        s.check()
        mp = sorted(s.m.matched_parties, key=lambda p: (p[4] - s.m.seq_next) & U32)
        assert len(mp) >= 8
        # one member of party 0 back as a solo (mm_requeue), one of party 1 removed, both in party 2
        cols = lambda x: tuple(np.array([s.m.book[int(y)][j] for y in x]) for j in range(4))  # noqa: E731
        solo = [int(mp[0][0][1]), int(mp[2][0][0])]
        for x in solo:
            assert np.array_equal(s.eng.requeue([x], *cols([x])), s.m.requeue(np.array([x], np.uint64)))
        gone = [int(mp[1][0][2]), int(mp[2][0][3])]
        assert s.eng.remove(gone) == s.m.remove(np.array(gone, np.uint64))
        s.check()
        s.requeue_party(mp[:4], expect=[0, 4, 0, 1])
        s.check()
        s.checkpoint()  # the matched parties' values now come from the image load
        s.check()
        s.requeue_party(mp[4:6], expect=[1, 1])
        s.check()
        requeued_locate(s, mp[3:6])
        s.queue_move()  # one group's queues out to a second engine and back (the moved parties get new numbers)
        s.check()
        s.requeue_party(mp[6:], expect=[1] * (len(mp) - 6))
        s.check()
        requeued_locate(s, mp[6:])
        s.requeue_party(mp[3:4], expect=[0])  # queued now
        s.check()
    finally:
        s.close()


# ================================================================================ GPU: the twin of the EQUIVALENCE
def twin_images(pkg, cfg, pimg, img, parties, codes):
    """The header's EQUIVALENCE: the code-1 parties into the party image at their seq position, their member ids out of
    section 7 of the engine image."""
    ab = pkg.abi
    ph, pc = pkg.engine.read_party_image(pimg)
    one = [p for p, c in zip(parties, codes) if c == 1]
    idt = pc["id"].dtype
    cut = np.cumsum(pc["size"].astype(np.int64))[:-1]
    rows = [(int(pc["seq"][j]), int(pc["enq_ts"][j]), int(pc["mode"][j]), a, b)
            for j, (a, b) in enumerate(zip(np.split(pc["id"], cut), np.split(pc["rating"], cut)))]
    rows += [(int(p[4]), int(p[3]), int(p[2]), np.asarray(p[0]).astype(idt), np.asarray(p[1], np.int32)) for p in one]
    rows.sort(key=lambda x: (x[0] - ph.seq_next) & U32)
    P, M = len(rows), sum(len(x[3]) for x in rows)
    off = ab.party_image_offsets(P, M, ph.id_bytes)
    out = np.zeros(off[-1], np.uint8)
    h2 = ab.ImageHeader.from_buffer_copy(ph)
    h2.n_parts, h2.n_players, h2.total_bytes = P, M, off[-1]
    out[:C.sizeof(h2)] = np.frombuffer(bytes(h2), np.uint8)
    secs = [np.array([len(x[3]) for x in rows], np.uint8), np.array([x[0] for x in rows], np.uint32),
            np.array([x[1] for x in rows], np.uint32), np.array([x[2] for x in rows], np.uint8),
            np.concatenate([x[3] for x in rows]) if rows else np.zeros(0, idt),
            np.concatenate([x[4] for x in rows]) if rows else np.zeros(0, np.int32)]
    for k, a in enumerate(secs):
        b = np.ascontiguousarray(a).view(np.uint8)
        out[off[k]:off[k] + len(b)] = b
    # the engine image without the requeued members in its active section
    img = np.array(img, np.uint8, copy=True)
    h, cols = pkg.engine.read_image(img)
    gone = np.concatenate([np.asarray(p[0]) for p in one]).astype(cols["active"].dtype)
    active = cols["active"][~np.isin(cols["active"], gone)]
    o = ab.image_offsets(h.n_parts, h.n_players, len(active), h.id_bytes)
    e = np.zeros(o[-1], np.uint8)
    e[:o[-2]] = img[:o[-2]]
    h3 = ab.ImageHeader.from_buffer_copy(h)
    h3.n_active, h3.total_bytes = len(active), o[-1]
    e[:C.sizeof(h3)] = np.frombuffer(bytes(h3), np.uint8)
    b = np.ascontiguousarray(active).view(np.uint8)
    e[o[-2]:o[-2] + len(b)] = b
    return out, e


@pytest.mark.gpu
@pytest.mark.parametrize("dense", KINDS, ids=kind_id)
def test_twin_engine_of_the_equivalence(pkg, oracle, dense):
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[:3], order=RATING, capacity=200_000,
                                active_capacity=1_000_000, default_group=-1, flags=DENSE if dense else 0)
    s = RequeueSchedule(pkg, oracle, cfg, np.random.default_rng(7 + dense), dense, pcap=50_000)
    twin = None
    try:
        s.players(40_000)
        s.party_batch(1500)
        s.now += 60
        rules = {(m, g): (0, 20, 5, 5, 200) for m in range(cfg.n_modes) for g in range(cfg.n_groups)}
        s.party_match(rules)
        s.tick()
        s.check()
        s.party_batch(60)
        mp = list({p[4]: p for p in s.m.matched_parties}.values())
        parties = mp[::2] + s.m.parties[:3]  # code 1 and code 0
        s.m.remove(np.array([mp[2][0][0]], np.uint64))
        s.eng.remove([mp[2][0][0]])  # code 4
        pimg = s.eng.export_parties()
        img = s.eng.export_state()
        assert (s.eng.merge_parties(pimg, keep_seq=True) == 1).all()
        s.check()
        codes = s.requeue_party(parties)
        assert set(codes.tolist()) == {0, 1, 4}
        s.check()
        pimg2, img2 = twin_images(pkg, cfg, pimg, img, parties, codes)
        twin = pkg.Engine(cfg)
        twin.import_state(img2)
        twin.set_option("party_capacity", s.pcap)
        assert (twin.merge_parties(pimg2, keep_seq=True) == 1).all()
        a, b = s.eng, twin
        probe = np.concatenate([s.m.party_members()[::7], s.m.active[::101]])
        for step in range(6):
            now = s.now + 40 * step
            pa, pb = a.party_read(), b.party_read()
            for k in ("size", "seq", "enq_ts", "mode", "group", "rating"):
                assert np.array_equal(pa[k], pb[k]), k
            assert all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1])
                       for x, y in zip(pa["members"], pb["members"]))
            assert a.seq_next() == b.seq_next() and a.active_size() == b.active_size()
            la, lb = a.locate(probe, now), b.locate(probe, now)
            assert np.array_equal(la, lb)
            qa, qb = a.queue_stats(now), b.queue_stats(now)
            for f in ("mode", "group", "n_waiting", "max_wait", "wait_hist"):
                assert np.array_equal(qa[f], qb[f]), f
            ra, rb = a.party_match(now, rules_of(cfg, rules)), b.party_match(now, rules_of(cfg, rules))
            assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1])
            ta, tb = a.tick(now), b.tick(now)
            for x, y in zip(ta[:3], tb[:3]):
                assert np.array_equal(x, y)
            pa, pb = a.pool_read(), b.pool_read()
            for k in pa:
                assert np.array_equal(pa[k], pb[k]), k
    finally:
        if twin is not None:
            twin.close()
        s.close()


# ================================================================================ GPU: refusals
@pytest.mark.gpu
@pytest.mark.parametrize("dense", KINDS, ids=kind_id)
def test_refusals_change_nothing(pkg, oracle, dense):
    ab = pkg.abi
    cfg = small_config(pkg, dense)
    s = RequeueSchedule(pkg, oracle, cfg, np.random.default_rng(9), dense, pcap=1000, lo=0, hi=2000)
    try:
        s.players(200)
        ids = s.fresh(12)
        r = np.full(12, 500, np.int32)
        sz = np.array([2, 2, 4, 4], np.uint8)
        md = np.array([0, 0, 1, 1], np.uint8)
        assert np.array_equal(s.eng.enqueue_party(sz, ids, r, md, np.full(4, s.now, np.uint32)),
                              s.m.enqueue_party(sz, ids, r, md, np.full(4, s.now, np.uint32)))
        s.party_match({(0, 0): (0, 10, 1, 0, 10)})
        a, b = s.m.matched_parties
        live = s.m.parties[0]
        s.check()

        def state():
            pr = s.eng.party_read()
            return (s.eng.pool_read()["id"].tolist(), s.eng.active_size(), s.eng.in_queue(ids).tolist(),
                    pr["size"].tolist(), pr["seq"].tolist(), [x[0].tolist() for x in pr["members"]],
                    s.eng.seq_next(), s.eng.locate(ids, s.now).tolist())

        before = state()
        limit = cfg.active_capacity if dense else (1 << 64) - 2
        cases = {
            "mode": [(a[0], a[1], cfg.n_modes, a[3], a[4])],
            "size 1": [(a[0][:1], a[1][:1], 0, a[3], a[4])],
            "size above team_size": [(np.concatenate([a[0], b[0]]), np.concatenate([a[1], b[1]]), 0, a[3], a[4])],
            "id out of range": [(np.array([a[0][0], limit], np.uint64), a[1], 0, a[3], a[4])],
            "id twice in a party": [(np.array([a[0][0], a[0][0]], np.uint64), a[1], 0, a[3], a[4])],
            "id twice in the call": [a, (np.array([b[0][0], a[0][0]], np.uint64), b[1], 0, b[3], b[4])],
            "R without a group": [(a[0], np.array([5000, 5000]), 0, a[3], a[4])],
            "seq_next": [(a[0], a[1], 0, a[3], s.m.seq_next)],
            "same seq": [a, (b[0], b[1], 0, b[3], a[4])],
            "seq of a queued party": [(a[0], a[1], 0, a[3], live[4])],
        }
        for what, parties in cases.items():
            with pytest.raises(ArgRefused):
                s.m.requeue_party(parties)
            s.refused(ab.MM_E_ARG, lambda: s.eng.requeue_party(*columns(parties)))
            assert state() == before, what
        # entries not in strict age order, through the C call (Engine.requeue_party sorts them)
        cols = columns([b, a])
        k = C.c_uint32(7)
        rc = s.eng.lib.mm_requeue_party(s.eng.h, 2, *(c.ctypes.data for c in cols[:4]), cols[4].ctypes.data,
                                        cols[5].ctypes.data, None, C.byref(k))
        assert rc == ab.MM_E_ARG and k.value == 0 and state() == before
        assert "age order" in s.eng.lib.mm_last_error(s.eng.h).decode()
        rc = s.eng.lib.mm_requeue_party(s.eng.h, 1, None, *(c.ctypes.data for c in cols[1:4]), None,
                                        cols[5].ctypes.data, None, C.byref(k))
        assert rc == ab.MM_E_ARG and state() == before
        assert s.eng.lib.mm_requeue_party(s.eng.h, 0, None, None, None, None, None, None, None, C.byref(k)) == ab.MM_OK
        # the exact room: the queued members plus the party, then one less
        queued = len(s.m.party_members())
        s.eng.set_option("party_capacity", queued + 3)
        s.m.pcap = queued + 3
        with pytest.raises(CapRefused):
            s.m.requeue_party([a, b])
        s.refused(ab.MM_E_CAP, lambda: s.eng.requeue_party(*columns([a, b])))
        assert state() == before
        s.eng.set_option("party_capacity", queued + 4)
        s.m.pcap = queued + 4
        s.requeue_party([a, b], expect=[1, 1])
        s.check()
        # a staged packed batch refuses (MM_E_STATE)
        if dense:
            eng = s.eng
            eng.enqueue_packed_begin(np.array([s.fresh(1)[0]], np.uint32), eng.pack_key([100], [1]))
            s.refused(ab.MM_E_STATE, lambda: eng.requeue_party(*columns([a])))
            eng.enqueue_packed_end()
    finally:
        s.close()
    # no party capacity, MM_F_NO_DEDUPE (MM_E_STATE); arrival order (MM_E_ARG)
    one = columns([(np.array([1, 2], np.uint64), np.array([5, 5]), 0, 0, 5)])
    for flags, order, cap, status in ((DENSE if dense else 0, RATING, 0, ab.MM_E_STATE),
                                      (1, RATING, 100, ab.MM_E_STATE),
                                      (DENSE if dense else 0, 0, 100, ab.MM_E_ARG)):
        c = pkg.synth.make_config(groups=[(0, 999)], modes=[("2v2", 2, 2)], order=order, capacity=1000,
                                  active_capacity=4000, default_group=-1, flags=flags)
        eng = pkg.Engine(c)
        try:
            if cap:
                eng.set_option("party_capacity", cap)
            with pytest.raises(pkg.EngineError) as ei:
                eng.requeue_party(*one)
            assert ei.value.status == status
        finally:
            eng.close()


# ================================================================================ GPU: mixed schedules
@pytest.mark.gpu
@pytest.mark.parametrize("dense", KINDS, ids=kind_id)
def test_mixed_schedule_with_party_requeue(pkg, oracle, dense):
    rng = np.random.default_rng(700 + dense)
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[:3], order=RATING, capacity=300_000,
                                active_capacity=4_000_000, default_group=-1, flags=DENSE if dense else 0)
    s = RequeueSchedule(pkg, oracle, cfg, rng, dense)
    try:
        s.players(60_000, old=0.02)
        s.party_batch(800)
        s.check()
        for _ in range(3 * len(s.OPS)):
            s.step()
        s.tick()
        s.finish()
        s.check()
    finally:
        s.close()
    c = s.counts
    assert c.get("requeue_party", 0) >= 3 and c.get("requeue_party_[1]", 0) + c.get("requeue_party_[0, 1]", 0) + \
        c.get("requeue_party_[0, 1, 4]", 0) + c.get("requeue_party_[1, 4]", 0) >= 3, c
    for what in ("party_match", "requeue", "checkpoint", "queue_move", "expire", "locate"):
        assert c.get(what, 0) >= 3, (what, c)


# ================================================================================ CPU: SearchPool(requeue_parties=...)
def party_requeue_engine(pkg, calls):
    class Eng(party_engine(pkg, calls)):
        """The party engine double with requeue_party by the codes of the definition: the parties go back into the
        table in age order."""

        def party_match(self, now, rules):
            self.seq_of.update((int(x), p[4]) for p in self.parties for x in p[0])
            return super().party_match(now, rules)

        def enqueue_party(self, sizes, ids, rating, mode, enq_ts):
            s0 = self.ctr
            n0 = len(self.parties)
            codes = super().enqueue_party(sizes, ids, rating, mode, enq_ts)
            seqs = [(s0 + int(j)) & U32 for j in np.flatnonzero(codes == 1)]  # party j of the batch: s0 + j
            self.parties[n0:] = [tuple(p) + (q,) for p, q in zip(self.parties[n0:], seqs)]
            return codes

        def requeue_party(self, sizes, ids, rating, mode, enq_ts, seq):
            calls.append(("requeue_party", sizes.tolist()))
            queued = set(self.q[0].tolist()) | {x for p in self.parties for x in p[0]}
            codes, off = [], 0
            for s, md, t, q in zip(sizes.tolist(), mode.tolist(), enq_ts.tolist(), seq.tolist()):
                mem = [int(x) for x in ids[off:off + s]]
                rat = [int(x) for x in rating[off:off + s]]
                off += s
                c = 0 if any(x in queued for x in mem) else 4 if any(x not in self.active for x in mem) else 1
                if c == 1:
                    self.parties.append((mem, rat, md, t, q))
                codes.append(c)
            self.parties.sort(key=lambda p: (p[4] - self.ctr) & U32)
            return np.array(codes, np.uint8)

        def requeue(self, ids, rating, mode, enq_ts, seq):
            calls.append(("requeue", sorted(int(x) for x in ids)))
            return super().requeue(ids, rating, mode, enq_ts, seq)

    return Eng


def requeue_pool(pkg, requeue_parties=True, calls=None, engine=None, blob=None):
    from .fakes import FakeBroker
    from .test_handover import start_workers
    sw = importlib.import_module("microservice-matchmaking_b200.search_worker")
    calls = [] if calls is None else calls
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=RATING, capacity=1000, active_capacity=4000)
    eng = engine or party_requeue_engine(pkg, calls)(cfg)
    opts = dict(flush_every_s=3600, clock=lambda: 0.0, wall_clock=lambda: 1_700_000_000.0,
                parties={"5v5": (0, 50, 1000, 0, 50)}, party_capacity=100, requeue_parties=requeue_parties)
    if blob is None:
        pool = sw.SearchPool(eng, ["1v1", "5v5"], list(pkg.synth.REFERENCE_GROUP_NAMES), **opts)
    else:
        pool = sw.SearchPool.resume(eng, blob, ["1v1", "5v5"], list(pkg.synth.REFERENCE_GROUP_NAMES), **opts)
    broker = FakeBroker()
    start_workers(sw, broker, pool, pkg)
    return sw, eng, pool, broker, calls


def matched_lobby(pkg, requeue_parties=True, solos=0):
    """Parties a (3), b (2) and c (5) of bronze 5v5 and `solos` solos, matched into one party lobby."""
    from .test_expire import publish
    from .test_requeue import lobbies
    sw, eng, pool, broker, calls = requeue_pool(pkg, requeue_parties)
    cfg = eng.cfg
    for i in range(solos):
        publish(pkg, broker, cfg, f"s{i}", 100, mode="5v5")
    publish_party(pkg, broker, sw, "bronze", [(f"a{i}", 100) for i in range(3)], "5v5")
    publish_party(pkg, broker, sw, "bronze", [(f"b{i}", 100) for i in range(2)], "5v5")
    if solos < 5:
        publish_party(pkg, broker, sw, "bronze", [(f"c{i}", 100) for i in range(5)], "5v5")
    broker.deliver_all()
    pool.flush()
    assert pool.tick() == 1
    lob = lobbies(broker, sw)[0]
    docs = [p for team in lob["teams"].values() for p in team]
    calls.clear()
    return sw, eng, pool, broker, calls, docs


def test_requeue_of_whole_parties(pkg):
    sw, eng, pool, broker, calls, docs = matched_lobby(pkg)
    assert pool.requeue(docs) == ["requeued"] * 10
    assert sorted(calls) == [("requeue_party", [3, 2, 5])]
    assert [p[0] for p in eng.parties] == [[pool.handles.lookup(f"a{i}") for i in range(3)],
                                          [pool.handles.lookup(f"b{i}") for i in range(2)],
                                          [pool.handles.lookup(f"c{i}") for i in range(5)]]
    assert [p[4] for p in eng.parties] == [0, 1, 2]  # the numbers the batch gave them
    assert pool.tick() == 1  # and they are matched again
    assert pool.requeue(docs[:1]) == ["requeued"]  # the book followed them to the new lobby


def test_requeue_of_some_members_and_a_lone_member(pkg):
    sw, eng, pool, broker, calls, docs = matched_lobby(pkg)
    ids = [d["id"] for d in docs]
    pick = [docs[ids.index(x)] for x in ("a0", "a2", "b1", "c0", "c1", "c2", "c3", "c4")]
    assert pool.requeue(pick) == ["requeued"] * 8
    h = pool.handles.lookup
    assert ("requeue", [h("b1")]) in calls and ("requeue_party", [2, 5]) in calls
    assert [p[0] for p in eng.parties] == [[h("a0"), h("a2")], [h("c0"), h("c1"), h("c2"), h("c3"), h("c4")]]
    assert eng.seq_of[h("b1")] == 1  # the lone member goes back as a solo with its party's number
    assert pool.requeue([docs[ids.index("a1")], docs[ids.index("a0")]]) == ["requeued", "queued"]
    assert ("requeue", [h("a1")]) in calls  # a1 is the only matched member left of party a


def test_requeue_of_a_lobby_with_solos(pkg):
    sw, eng, pool, broker, calls, docs = matched_lobby(pkg, solos=5)
    assert len(docs) == 10 and sum(d["id"].startswith("s") for d in docs) == 5
    assert pool.requeue(docs) == ["requeued"] * 10
    h = pool.handles.lookup
    assert ("requeue_party", [3, 2]) in calls and ("requeue", sorted(h(f"s{i}") for i in range(5))) in calls
    assert all(pool.in_queue(d["id"]) for d in docs)


def test_a_refused_party_call_answers_its_parties_gone_and_the_solos_go_on(pkg):
    sw, eng, pool, broker, calls, docs = matched_lobby(pkg, solos=5)

    def full(*a):
        calls.append(("requeue_party", a[0].tolist()))
        raise pkg.EngineError(pkg.abi.MM_E_CAP, "mm_requeue_party")

    eng.requeue_party = full
    out = pool.requeue(docs)
    solo = [d["id"].startswith("s") for d in docs]
    assert [o for o, x in zip(out, solo) if x] == ["requeued"] * 5 and [o for o, x in zip(out, solo) if not x] == \
        ["gone"] * 5
    assert [c[0] for c in calls] == ["requeue_party", "requeue"]  # the party call first: nothing changed when refused
    h = pool.handles.lookup
    assert all(h(d["id"]) in pool.players for d, x in zip(docs, solo) if x)
    assert not any(h(d["id"]) in pool.players for d, x in zip(docs, solo) if not x)
    assert all(h(d["id"]) in pool.matched_parties for d, x in zip(docs, solo) if not x)  # remove_user clears them


def test_a_second_lone_member_in_the_same_queue_answers_gone(pkg):
    sw, eng, pool, broker, calls, docs = matched_lobby(pkg)
    ids = [d["id"] for d in docs]
    h = pool.handles.lookup
    assert pool.requeue([docs[ids.index("b0")]]) == ["requeued"]  # a solo with party b's number
    calls.clear()
    assert pool.requeue([docs[ids.index("b1")]]) == ["gone"] and calls == []
    assert h("b1") in pool.matched_parties and h("b1") not in pool.players


def test_requeue_of_party_members_with_the_option_off(pkg):
    sw, eng, pool, broker, calls, docs = matched_lobby(pkg, requeue_parties=False, solos=5)
    out = pool.requeue(docs)
    assert [o for d, o in zip(docs, out) if d["id"].startswith("s")] == ["requeued"] * 5
    assert [o for d, o in zip(docs, out) if not d["id"].startswith("s")] == ["gone"] * 5
    assert not any(c[0] == "requeue_party" for c in calls)
    assert not hasattr(pool, "matched_parties") or not pool.matched_parties


def test_requeue_of_a_queued_party_member_answers_queued(pkg):
    sw, eng, pool, broker, calls, docs = matched_lobby(pkg)
    ids = [d["id"] for d in docs]
    a = [docs[ids.index(f"a{i}")] for i in range(3)]
    assert pool.requeue(a) == ["requeued"] * 3
    calls.clear()
    assert pool.requeue(a[:2]) == ["queued", "queued"] and calls == []


def test_remove_user_drops_the_book_entry(pkg):
    sw, eng, pool, broker, calls, docs = matched_lobby(pkg)
    h = pool.handles.lookup
    a = [h(f"a{i}") for i in range(3)]
    assert all(x in pool.matched_parties for x in a)
    pool.remove_user("a0")
    assert a[0] not in pool.matched_parties and a[1] in pool.matched_parties
    ids = [d["id"] for d in docs]
    out = pool.requeue([docs[ids.index(x)] for x in ("a0", "a1", "a2")])
    assert out == ["gone", "requeued", "requeued"] and ("requeue_party", [2]) in calls
    assert [p[0] for p in eng.parties] == [a[1:]]


def test_checkpoint_and_resume_carry_the_book(pkg):
    import json
    sw, eng, pool, broker, calls, docs = matched_lobby(pkg)
    book = pool._book_records(pool.matched_parties)
    assert len(book) == 3 and pool.party_book == {}
    for e in (eng,):  # no queued party: the party image is empty
        e.export_parties = lambda mask=None: np.zeros(0, np.uint8)
        e.merge_parties = lambda buf, keep_seq=False: np.zeros(0, np.uint8)
    blob = pool.checkpoint()
    calls2 = []
    eng2 = party_requeue_engine(pkg, calls2)(eng.cfg)
    _sw, eng2, pool2, _b, _c = requeue_pool(pkg, engine=eng2, blob=blob, calls=calls2)
    assert pool2._book_records(pool2.matched_parties) == json.loads(json.dumps(book))
    assert pool2.requeue(docs) == ["requeued"] * 10
    assert [len(p[0]) for p in eng2.parties] == [3, 2, 5] and [p[4] for p in eng2.parties] == [0, 1, 2]
    # a pool without the option writes no book
    _sw, eng3, pool3, _b, _c = requeue_pool(pkg, requeue_parties=False)
    eng3.export_parties, eng3.merge_parties = eng.export_parties, eng.merge_parties
    assert b"party_book" not in pool3.checkpoint()


# ================================================================================ GPU: SearchPool end to end
@pytest.mark.gpu
def test_search_pool_requeues_a_declined_party_lobby(pkg):
    """A declined 5v5 party lobby goes back whole; the next tick gives the same parties their lobby again."""
    from .fakes import FakeBroker
    from .test_handover import start_workers
    from .test_requeue import lobbies
    sw = importlib.import_module("microservice-matchmaking_b200.search_worker")
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=[("1v1", 2, 1), ("5v5", 2, 5)],
                                order=RATING, capacity=10_000, active_capacity=40_000)
    eng = pkg.Engine(cfg)
    t = [0.0]
    try:
        pool = sw.SearchPool(eng, ["1v1", "5v5"], list(pkg.synth.REFERENCE_GROUP_NAMES), flush_every_s=3600,
                             clock=lambda: t[0], parties={"5v5": (0, 50, 1000, 0, 50)}, party_capacity=1000,
                             requeue_parties=True)
        broker = FakeBroker()
        start_workers(sw, broker, pool, pkg)
        publish_party(pkg, broker, sw, "bronze", [(f"a{i}", 100 + i) for i in range(5)], "5v5")
        publish_party(pkg, broker, sw, "bronze", [(f"b{i}", 104 - i) for i in range(3)], "5v5")
        publish_party(pkg, broker, sw, "bronze", [(f"c{i}", 102) for i in range(2)], "5v5")
        broker.deliver_all()
        pool.flush()
        t[0] += 1
        assert pool.tick() == 1
        first = lobbies(broker, sw)[0]
        docs = [p for team in first["teams"].values() for p in team]
        assert pool.requeue(docs) == ["requeued"] * 10  # a member declined the ready check
        assert all(pool.in_queue(d["id"]) for d in docs)
        st = pool.search_status([d["id"] for d in docs])
        pr = eng.party_read()
        assert len(pr["size"]) == 3 and pr["size"].tolist() == [5, 3, 2]
        t[0] += 1
        assert pool.tick() == 1
        again = lobbies(broker, sw)[1]
        assert again["teams"] == first["teams"]
        assert len(st) == 10
    finally:
        eng.close()
