"""Requeue (mm_requeue): players of a lobby that did not start go back into their queue at their enqueue position.

GPU: the engine after a requeue against a fresh engine that imported the restated image (the export before the call,
with the requeued players inserted at their sequence position and their ids out of the active section), driven through
the same mixed steps; placement cases; codes; every refusal; async results, snapshot / restore and export / import
around a requeue; config3 at 10 M players.  CPU: SearchPool.requeue with an engine double (the ready-check flow,
timeouts, checkpoint / resume, move_in, a moved-out group).
"""
import ctypes as C
import zlib

import numpy as np
import pytest

from .test_handover import same_state, tick_both
from .test_tile_geometry import DENSE, MODES8, WIDE

ARRIVAL, RATING = 0, 1
NO_DEDUPE = 1
U32 = np.uint32


# ================================================================================ the restatement
def layout_parts(cfg, rating, mode):
    """Layout partition of each (rating, mode), as the engine lays its pool out (one partition per (mode, group)
    queue, or several of <= 255 sort keys for a wide group without MM_F_WIDE_PARTITIONS)."""
    G = cfg.n_groups
    lo = [cfg.group_lo[g] for g in range(G)]
    hi = [cfg.group_hi[g] for g in range(G)]
    key_lo = min(lo) - 1
    KR = max(hi) - min(lo) + 3
    r = np.arange(KR, dtype=np.int64) + key_lo
    grp = np.full(KR, cfg.default_group if cfg.default_group >= 0 else 255, np.int64)
    for g in reversed(range(G)):  # the first matching group wins
        grp[(r >= lo[g]) & (r <= hi[g])] = g
    first = [0] * (G + 1)
    lut = np.zeros(KR, np.int64)
    if cfg.order_mode == RATING:
        nxt = 0
        for g in range(G):
            first[g] = nxt
            ks = np.flatnonzero(grp == g)
            lut[ks] = nxt + np.arange(len(ks))
            nxt += len(ks)
        first[G] = nxt
        stride = max(nxt, 1)
    else:
        lut = np.where(grp == 255, 0, grp)
        first = list(range(G + 1))
        stride = G
    split = not (cfg.flags & WIDE)
    for _ in range(2):
        seg_lo = []
        for m in range(cfg.n_modes):
            for g in range(G):
                b0, nk = m * stride + first[g], first[g + 1] - first[g]
                nsub = max(1, -(-nk // 255)) if split else 1
                per = -(-nk // nsub)
                seg_lo += [b0 + min(nk, j * per) for j in range(nsub)]
        if len(seg_lo) <= 512:
            break
        split = False
    rr = np.clip(np.asarray(rating, np.int64), key_lo, key_lo + KR - 1)
    b = np.asarray(mode, np.int64) * stride + lut[rr - key_lo]
    return np.searchsorted(np.asarray(seg_lo), b, side="right") - 1


def restate(pkg, cfg, img, ids, rating, mode, ts, seq):
    """The image of the Equivalence: `img` (mm_export just before the call) with these players (the code-1 entries)
    inserted in their partition at their sequence position and their ids taken out of the active section."""
    img = np.array(img, np.uint8, copy=True)
    h, s = pkg.engine.read_image(img)
    part = np.concatenate([np.repeat(np.arange(h.n_parts), s["part_count"]), layout_parts(cfg, rating, mode)])
    u = (np.concatenate([s["seq"], np.asarray(seq, U32)]) - U32(h.seq_next)).astype(U32)
    o = np.lexsort((u, part))
    idt = s["id"].dtype
    cols = [np.concatenate([s["id"], np.asarray(ids).astype(idt)])[o],
            np.concatenate([s["rating"], np.asarray(rating, np.int32)])[o],
            np.concatenate([s["enq_ts"], np.asarray(ts, U32)])[o],
            np.concatenate([s["seq"], np.asarray(seq, U32)])[o],
            np.concatenate([s["mode"], np.asarray(mode, np.uint8)])[o]]
    counts = np.bincount(part, minlength=h.n_parts).astype(U32)
    active = s["active"][~np.isin(s["active"], np.asarray(ids).astype(idt))]
    n, m = len(cols[0]), len(active)
    off = pkg.abi.image_offsets(h.n_parts, n, m, h.id_bytes)
    out = np.zeros(off[-1], np.uint8)
    h2 = pkg.abi.ImageHeader.from_buffer_copy(h)
    h2.n_players, h2.n_active, h2.total_bytes = n, m, off[-1]
    out[:C.sizeof(h2)] = np.frombuffer(bytes(h2), np.uint8)
    for k, a in enumerate([counts] + cols + [active]):
        b = np.ascontiguousarray(a).view(np.uint8)
        out[off[k]:off[k] + len(b)] = b
    return out


# ================================================================================ GPU helpers
class Book:
    """What the caller keeps per queued player: rating, mode, stamp and sequence number at its enqueue."""

    def __init__(self):
        self.cols = {k: [] for k in ("id", "rating", "mode", "ts", "seq")}

    def add(self, seq0, ids, r, m, ts, codes):
        ok = np.asarray(codes) == 1
        for k, v in zip(self.cols, (ids, r, m, ts, (U32(seq0) + np.arange(len(ids), dtype=U32)).astype(U32))):
            self.cols[k].append(np.asarray(v)[ok])

    def of(self, ids):
        """-> (rating, mode, ts, seq) of each id at its latest enqueue."""
        c = {k: np.concatenate(v) for k, v in self.cols.items()}
        uniq, first = np.unique(c["id"][::-1], return_index=True)
        last = len(c["id"]) - 1 - first
        idx = last[np.searchsorted(uniq, np.asarray(ids, np.uint64))]
        assert np.array_equal(c["id"][idx], ids)
        return c["rating"][idx], c["mode"][idx], c["ts"][idx], c["seq"][idx]


def config(pkg, kind, order, wide=False, capacity=200_000, groups=None):
    flags = {"hashed": 0, "dense": DENSE, "no_dedupe": NO_DEDUPE}[kind] | (WIDE if wide else 0)
    return pkg.synth.make_config(groups=groups or pkg.synth.REFERENCE_GROUPS, modes=MODES8[:3], order=order,
                                 capacity=capacity, active_capacity=1_000_000, default_group=-1, flags=flags)


class Src:
    """One engine, its book and a supply of fresh players."""

    def __init__(self, pkg, cfg, kind, seed, spread=-1):
        self.pkg, self.cfg, self.kind = pkg, cfg, kind
        self.eng = pkg.Engine(cfg)
        if spread >= 0:
            self.eng.set_option("max_spread", spread)
        self.rng = np.random.default_rng(seed)
        self.book = Book()
        self.next = 0
        self.now = 1000

    def fresh(self, n, lo=0, hi=5001, modes=3):
        x = np.arange(self.next, self.next + n, dtype=np.uint64)
        self.next += n
        ids = x if self.kind == "dense" else self.pkg.synth.mix64(x + np.uint64(7 << 40))
        r = self.rng.integers(lo, hi, n).astype(np.int32)
        m = self.rng.integers(0, modes, n).astype(np.uint8)
        ts = (self.now - self.rng.integers(0, 60, n)).astype(U32)
        return ids, r, m, ts

    def enqueue(self, ids, r, m, ts, engines=()):
        s0 = self.eng.seq_next()
        codes = self.eng.enqueue(ids, r, m, ts)
        for e in engines:
            assert np.array_equal(e.enqueue(ids, r, m, ts), codes)
        self.book.add(s0, ids, r, m, ts, codes)
        return codes

    def requeue(self, ids, eng=None):
        r, m, ts, seq = self.book.of(ids)
        return (eng or self.eng).requeue(ids, r, m, ts, seq)

    def close(self):
        self.eng.close()


def twin_after_requeue(pkg, src, ids):
    """Requeue `ids` on src.eng; -> (codes, a fresh engine that imported the restated image)."""
    img = src.eng.export_state()
    codes = src.requeue(ids)
    sel = codes == 1
    r, m, ts, seq = src.book.of(ids[sel])
    twin = pkg.Engine(src.cfg)
    twin.import_state(restate(pkg, src.cfg, img, ids[sel], r, m, ts, seq))
    return codes, twin


def export_sections(pkg, eng):
    h, s = pkg.engine.read_image(np.array(eng.export_state(), np.uint8, copy=True))
    return (h.n_players, h.n_active, h.seq_next), {k: s[k] for k in ("part_count", "id", "rating", "enq_ts", "seq",
                                                                      "mode")}, np.sort(s["active"])


def same_export(pkg, a, b):
    ha, sa, aa = export_sections(pkg, a)
    hb, sb, ab = export_sections(pkg, b)
    assert ha == hb
    for k in sa:
        assert np.array_equal(sa[k], sb[k]), k
    assert np.array_equal(aa, ab)


def lobby_members(res):
    lob, mem, _, _ = res
    return [mem[int(h["first_member"]):int(h["first_member"]) + int(h["n_members"])] for h in lob]


def drive(pkg, src, twin, steps, rng):
    """The same mixed calls on src.eng and twin; everything but the dead-slot fields must agree."""
    import torch
    a, b = src.eng, twin
    dense = src.kind == "dense"
    matched = []
    for k in range(steps):
        op = k % 10
        src.now += 37
        if op in (0, 4):  # mm_enqueue, with ids already queued / matched
            ids, r, m, ts = src.fresh(int(rng.integers(200, 3000)))
            old = a.pool_read()["id"][:50]
            ids = np.concatenate([ids, old] + ([matched[-1][:20]] if matched else []))
            extra = len(ids) - len(r)
            r = np.concatenate([r, rng.integers(0, 5001, extra).astype(np.int32)])
            m = np.concatenate([m, rng.integers(0, 3, extra).astype(np.uint8)])
            ts = np.concatenate([ts, np.full(extra, src.now, U32)])
            src.enqueue(ids, r, m, ts, engines=(b,))
        elif op == 1:  # packed forms (dense) / device pointers
            ids, r, m, ts = src.fresh(int(rng.integers(200, 2000)))
            s0 = a.seq_next()
            if dense:
                key = pkg.Engine.pack_key(r, m)
                ca = a.enqueue_packed(ids.astype(U32), key, ts)
                assert np.array_equal(ca, b.enqueue_packed(ids.astype(U32), key, ts))
                src.book.add(s0, ids, r, m, ts, ca)
                ids, r, m, ts = src.fresh(500)
                s0 = a.seq_next()
                key = pkg.Engine.pack_key(r, m)
                for e in (a, b):
                    e.enqueue_packed_begin(ids.astype(U32), key, ts)
                got = [e.enqueue_packed_end()[0] for e in (a, b)]
                assert np.array_equal(got[0], got[1])
                src.book.add(s0, ids, r, m, ts, got[0])
            else:
                t = [torch.from_numpy(x).cuda() for x in (ids.view(np.int64), r, m, ts.view(np.int32))]
                acc = [torch.empty(len(ids), dtype=torch.uint8, device="cuda") for _ in range(2)]
                for e, ac in zip((a, b), acc):
                    e.enqueue_device(len(ids), *(x.data_ptr() for x in t), ac.data_ptr())
                ca = acc[0].cpu().numpy()
                assert np.array_equal(ca, acc[1].cpu().numpy())
                src.book.add(s0, ids, r, m, ts, ca)
        elif op == 2:  # a tick, every result form
            form = (k // 10) % 3
            if form == 2:
                sa, sb = a.tick_device(src.now), b.tick_device(src.now)
                assert (sa.n_lobbies, sa.n_matched, sa.n_residual) == (sb.n_lobbies, sb.n_matched, sb.n_residual)
                for e in (a, b):
                    e.tick(src.now)  # the next tick, to host
            res = [e.tick_packed(src.now) if (dense and form == 1) else e.tick(src.now) for e in (a, b)]
            for x, y in zip(res[0][:3], res[1][:3]):
                assert np.array_equal(x, y)
            mem = res[0][1].astype(np.uint64)
            if len(mem):
                matched.append(mem)
        elif op == 3 and matched:  # requeue on both: lobbies of the last ticks, some members removed first
            lobs = matched[-1]
            gone = lobs[: len(lobs) // 7]
            assert a.remove(gone) == b.remove(gone)
            back = np.concatenate([lobs[len(lobs) // 7:], a.pool_read()["id"][:5]])
            ca, cb = src.requeue(back), src.requeue(back, eng=b)
            assert np.array_equal(ca, cb)
            assert (ca[: len(back) - 5] == 1).all() and (ca[len(back) - 5:] == 0).all()
        elif op == 5:  # remove / take
            cur = a.pool_read()["id"]
            assert a.remove(cur[:100]) == b.remove(cur[:100])
            assert a.take(cur[100:200]) == b.take(cur[100:200])
            matched.append(cur[100:200])
        elif op == 6:  # expire
            ea, eb = a.expire(src.now, 400), b.expire(src.now, 400)
            oa, ob = np.argsort(ea[1]), np.argsort(eb[1])
            assert np.array_equal(ea[0][oa], eb[0][ob]) and np.array_equal(ea[1][oa], eb[1][ob])
        elif op == 7:
            same_export(pkg, a, b)
        sample = np.concatenate([a.pool_read()["id"][::40]] + [x[::5] for x in matched[-3:]])
        same_state(a, b, src.now, sample)
        assert a.seq_next() == b.seq_next()


TWINS = [  # kind, order, spread, wide, groups
    ("hashed", RATING, -1, False, None), ("dense", RATING, 3, False, None), ("hashed", ARRIVAL, -1, False, None),
    ("dense", ARRIVAL, -1, False, None), ("hashed", RATING, 2, True, None), ("dense", RATING, -1, True, None),
    ("hashed", RATING, 4, False, ((0, 1999), (2000, 4999), (5000, 5000))),
]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,order,spread,wide,groups", TWINS)
def test_twin_import_gives_the_same_results(pkg, kind, order, spread, wide, groups):
    cfg = config(pkg, kind, order, wide, groups=groups)
    src = Src(pkg, cfg, kind, seed=zlib.crc32(repr((kind, order, spread, wide)).encode()), spread=spread)
    try:
        src.enqueue(*src.fresh(60_000))
        res = src.eng.tick(src.now)
        mem = lobby_members(res)
        back = np.concatenate(mem[::3])
        codes, twin = twin_after_requeue(pkg, src, back)
        assert (codes == 1).all()
        if spread >= 0:
            twin.set_option("max_spread", spread)
        try:
            sample = np.concatenate([back, src.eng.pool_read()["id"][::30]])
            same_state(src.eng, twin, src.now, sample)
            assert src.eng.in_queue(back).all()
            same_export(pkg, src.eng, twin)
            drive(pkg, src, twin, 34, np.random.default_rng(3))
        finally:
            twin.close()
    finally:
        src.close()


# ================================================================================ GPU: placement
def pool_seq_order(pkg, src):
    """pool_read ids with their book seq: must be ascending in age."""
    ids = src.eng.pool_read()["id"]
    seq = src.book.of(ids)[3]
    u = (seq - U32(src.eng.seq_next())).astype(U32)
    assert (np.diff(u.astype(np.int64)) > 0).all()
    return ids


def check_against_twin(pkg, src, ids):
    """Requeue `ids`, compare with the import twin, tick both. -> (codes, pool ids right after the requeue)"""
    codes, twin = twin_after_requeue(pkg, src, ids)
    try:
        same_state(src.eng, twin, src.now, ids)
        same_export(pkg, src.eng, twin)
        pool = pool_seq_order(pkg, src)
        tick_both(src.eng, twin, src.now + 1)
        same_state(src.eng, twin, src.now + 2, ids)
    finally:
        twin.close()
    return codes, pool


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
def test_placement_cases(pkg, kind):
    cfg = config(pkg, kind, RATING, groups=((0, 99), (100, 199)))
    src = Src(pkg, cfg, kind, seed=5)
    try:
        e = src.eng
        # older than every live player: a full lobby of 1v1 (mode 0) matched, then later arrivals stay
        ids, r, m, ts = src.fresh(2, 10, 11, 1)
        src.enqueue(ids, r, m, ts)
        e.tick(src.now)
        later = src.fresh(1, 10, 11, 1)
        src.enqueue(*later)
        codes, pool = check_against_twin(pkg, src, ids)
        assert codes.tolist() == [1, 1] and pool.tolist() == [ids[0], ids[1], later[0][0]]
        # the tick matched the two requeued players first (they are older): the later arrival is left over
        assert e.pool_read()["id"].tolist() == [later[0][0]]
        # newer than every live player, and interleaved, in a queue with dead slots (removed, taken)
        a = src.fresh(8, 20, 25, 2)
        src.enqueue(*a)
        e.take(a[0][:2])                   # taken: dead slots, still active
        b = src.fresh(6, 20, 25, 2)
        src.enqueue(*b)
        e.remove(b[0][:1])
        codes, pool = check_against_twin(pkg, src, a[0][:2])
        assert codes.tolist() == [1, 1] and pool.tolist() == [later[0][0]] + a[0].tolist() + b[0][1:].tolist()
        # into an empty queue (group 1 never had a player), matched several ticks ago
        c = src.fresh(4, 150, 151, 1)
        src.enqueue(*c)
        res = e.tick(src.now)
        for _ in range(3):
            e.tick(src.now)
        assert e.queue_stats(src.now)[1]["n_waiting"] == 0  # (mode 0, group 1) is empty
        codes, pool = check_against_twin(pkg, src, c[0])
        cs = set(c[0].tolist())
        assert codes.tolist() == [1] * 4 and [x for x in pool.tolist() if x in cs] == c[0].tolist()
        # interleaved with live players of the same queue, codes 0 / 1 / 4 mixed
        d = src.fresh(40, 30, 60, 3)
        src.enqueue(*d)
        res = e.tick(src.now)
        mem = res[1].astype(np.uint64)
        e2 = src.fresh(10, 30, 60, 3)
        src.enqueue(*e2)
        live = e.pool_read()["id"]
        e.remove(mem[:1])
        codes, pool = check_against_twin(pkg, src, np.concatenate([mem, live[:3]]))
        assert codes[0] == 4 and (codes[1:len(mem)] == 1).all() and (codes[len(mem):] == 0).all()
        assert len(pool) == len(live) + len(mem) - 1
    finally:
        src.close()


@pytest.mark.gpu
def test_band_match_taken_players_are_requeued(pkg):
    cfg = config(pkg, "hashed", RATING, groups=((0, 99), (100, 199)))
    src = Src(pkg, cfg, "hashed", seed=9)
    try:
        e = src.eng
        src.enqueue(*src.fresh(1, 98, 99, 1))
        src.enqueue(*src.fresh(1, 101, 102, 1))
        lob, mem, taken, st = e.band_match(5, 0, 0)
        assert st.n_matched == 2 and e.pool_read()["id"].size == 0
        codes, pool = check_against_twin(pkg, src, mem.astype(np.uint64))
        assert codes.tolist() == [1, 1] and len(pool) == 2
    finally:
        src.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
def test_sequence_numbers_across_the_wrap(pkg, kind):
    cfg = config(pkg, kind, ARRIVAL)
    src = Src(pkg, cfg, kind, seed=13)
    try:
        # an empty image with seq_next just below 2^32, imported: the next batch's numbers wrap
        img = np.array(src.eng.export_state(), np.uint8, copy=True)
        h = pkg.abi.ImageHeader.from_buffer_copy(img[:C.sizeof(pkg.abi.ImageHeader)].tobytes())
        h.seq_next = 0xFFFFFFFF - 700
        img[:C.sizeof(h)] = np.frombuffer(bytes(h), np.uint8)
        src.eng.close()
        src.eng = pkg.Engine(cfg)
        src.eng.import_state(img)
        back = []
        for _ in range(3):
            src.enqueue(*src.fresh(600))
            back.append(src.eng.tick(src.now)[1].astype(np.uint64))
        back = np.concatenate(back)
        seqs = src.book.of(back)[3]
        assert seqs.min() < 1000 and seqs.max() > 0xFFFFF000  # matched players from both sides of the wrap
        assert (check_against_twin(pkg, src, back)[0] == 1).all()
    finally:
        src.close()


# ================================================================================ GPU: codes and refusals
@pytest.mark.gpu
def test_codes_after_remove_expire_and_export_queues(pkg):
    cfg = config(pkg, "hashed", RATING)
    src = Src(pkg, cfg, "hashed", seed=17)
    try:
        e = src.eng
        src.enqueue(*src.fresh(5000))
        mem = e.tick(src.now)[1].astype(np.uint64)
        removed = mem[:10]
        e.remove(removed)
        ids, r, m, ts = src.fresh(100, 0, 5001)
        ts[:] = 0
        src.enqueue(ids, r, m, ts)
        expired = set(e.expire(src.now, 500)[0].tolist())
        assert expired == set(ids.tolist())
        src.enqueue(*src.fresh(600))
        live = e.pool_read()["id"]
        mask = np.zeros((3, 7), bool)
        mask[0, 3] = True
        q = (e.pool_read()["mode"] == 0) & np.isin(e.pool_read()["rating"], np.arange(cfg.group_lo[3], cfg.group_hi[3] + 1))
        moved = live[q]
        assert len(moved) >= 5
        e.export_queues(mask)
        stay = live[~q][:20]
        back = np.concatenate([removed, mem[10:40], ids[:5], moved[:5], stay])
        codes = check_against_twin(pkg, src, back)[0]
        assert (codes[:10] == 4).all() and (codes[10:40] == 1).all() and (codes[40:50] == 4).all()
        assert (codes[50:] == 0).all()
        assert e.in_queue(mem[10:40]).all() and not e.in_queue(removed).any()
    finally:
        src.close()


def state_bytes(pkg, eng, sample):
    """The export (its active section, which the engine writes unordered, as a sorted list), pool_read, in_queue,
    active_size and seq_next."""
    h, s, act = export_sections(pkg, eng)
    return (h, {k: v.tobytes() for k, v in s.items()}, act.tobytes(), {k: v.tobytes() for k, v in eng.pool_read().items()},
            eng.in_queue(sample).tobytes(), eng.active_size(), eng.seq_next())


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
def test_refusals_change_nothing(pkg, kind):
    cfg = config(pkg, kind, RATING, capacity=40_000)
    src = Src(pkg, cfg, kind, seed=21)
    try:
        e = src.eng
        src.enqueue(*src.fresh(20_000))
        mem = e.tick(src.now)[1].astype(np.uint64)
        src.enqueue(*src.fresh(3000))
        live = e.pool_read()["id"]
        r, m, ts, seq = src.book.of(mem[:50])
        o = np.argsort((seq - U32(e.seq_next())).astype(U32))
        ids, r, m, ts, seq = mem[:50][o], r[o], m[o], ts[o], seq[o]
        sample = np.concatenate([mem[:100], live[::50]])
        before = state_bytes(pkg, e, sample)

        def refused(status, text, ids=ids, r=r, m=m, ts=ts, seq=seq, check=True):
            codes = np.empty(len(ids), np.uint8)
            k = C.c_uint32(7)
            cols = [np.ascontiguousarray(x, dt) for x, dt in ((ids, np.uint64), (r, np.int32), (m, np.uint8),
                                                              (ts, U32), (seq, U32))]
            rc = e.lib.mm_requeue(e.h, len(ids), *(c.ctypes.data_as(C.c_void_p) for c in cols[:4]),
                                  cols[4].ctypes.data_as(C.c_void_p), codes.ctypes.data_as(C.c_void_p), C.byref(k))
            assert rc == status and k.value == 0
            assert e.lib.mm_last_error(e.h).decode() == text
            if check:  # (an export refuses too while a packed batch is staged)
                assert state_bytes(pkg, e, sample) == before

        A = pkg.abi
        refused(A.MM_E_ARG, "requeue refused: mode out of range", m=np.where(np.arange(50) == 3, 3, m))
        refused(A.MM_E_ARG, "requeue refused: rating without a group", r=np.where(np.arange(50) == 3, -5, r))
        bad = np.uint64(1_000_000 if kind == "dense" else 0xFFFFFFFFFFFFFFFF)
        refused(A.MM_E_ARG, "requeue refused: id out of range", ids=np.where(np.arange(50) == 3, bad, ids))
        refused(A.MM_E_ARG, "requeue refused: entries not in age order", ids=ids[::-1], r=r[::-1], m=m[::-1],
                ts=ts[::-1], seq=seq[::-1])
        s2 = seq.copy()
        s2[0] = e.seq_next()
        refused(A.MM_E_ARG, "requeue refused: sequence number equal to seq_next", seq=s2)
        i2 = ids.copy()
        i2[5] = i2[4]
        refused(A.MM_E_ARG, "requeue refused: duplicate id", ids=i2)
        # a matched player given the rating, mode and sequence number of a live player
        lr, lm, lts, lseq = src.book.of(live[:1])
        refused(A.MM_E_ARG, "requeue refused: sequence number of a live player of the partition", ids=mem[:1], r=lr,
                m=lm, ts=lts, seq=lseq)
        # capacity: the touched partitions' old chunks count until the next tick
        big = mem[:15000]
        rb, mb, tb, sb = src.book.of(big)
        ob = np.argsort((sb - U32(e.seq_next())).astype(U32))
        codes = np.empty(len(big), np.uint8)
        k = C.c_uint32(0)
        cols = [np.ascontiguousarray(x, dt) for x, dt in ((big[ob], np.uint64), (rb[ob], np.int32), (mb[ob], np.uint8),
                                                          (tb[ob], U32), (sb[ob], U32))]
        rc = e.lib.mm_requeue(e.h, len(big), *(c.ctypes.data_as(C.c_void_p) for c in cols), codes.ctypes.data_as(C.c_void_p),
                              C.byref(k))
        assert rc == A.MM_E_CAP, rc
        need_msg = e.lib.mm_last_error(e.h).decode()
        assert need_msg.startswith("requeue needs ") and need_msg.endswith("capacity 40000")
        assert state_bytes(pkg, e, sample) == before
        # a staged packed batch (dense) ; then the call goes through
        if kind == "dense":
            x = src.fresh(10)
            e.enqueue_packed_begin(x[0].astype(U32), pkg.Engine.pack_key(x[1], x[2]), x[3])
            pool = e.pool_read()
            refused(A.MM_E_STATE, "a packed batch is staged: call mm_enqueue_packed_end first", check=False)
            for k, v in e.pool_read().items():
                assert np.array_equal(v, pool[k]), k
            e.enqueue_packed_end()
        assert (e.requeue(ids[:2], r[:2], m[:2], ts[:2], seq[:2]) == 1).all()
        assert e.requeue(ids[:0], r[:0], m[:0], ts[:0], seq[:0]).size == 0
    finally:
        src.close()


@pytest.mark.gpu
def test_no_dedupe_engine_is_refused(pkg):
    with pkg.Engine(config(pkg, "no_dedupe", RATING)) as e:
        with pytest.raises(pkg.EngineError) as ei:
            e.requeue(np.arange(3, dtype=np.uint64), np.full(3, 10), np.zeros(3), None, np.arange(1, 4))
        assert ei.value.status == pkg.abi.MM_E_STATE
        assert "MM_F_NO_DEDUPE" in e.lib.mm_last_error(e.h).decode()


# ================================================================================ GPU: interactions
@pytest.mark.gpu
def test_async_results_snapshot_and_export_around_a_requeue(pkg):
    cfg = config(pkg, "dense", RATING)
    src = Src(pkg, cfg, "dense", seed=23)
    try:
        e = src.eng
        src.enqueue(*src.fresh(30_000))
        mem = e.tick(src.now)[1].astype(np.uint64)
        src.enqueue(*src.fresh(20_000))
        with pkg.Engine(cfg) as ref:  # the same engine without async results
            ref.import_state(e.export_state())
            e.set_option("async_results", 1)
            n = e.pool_size()
            bufs = (np.empty(n, pkg.engine.LOBBY_DTYPE), np.empty(n, np.uint64), np.empty(n, U32))
            st = e.tick_raw(bufs[0].ctypes.data, n, bufs[1].ctypes.data, n, bufs[2].ctypes.data, now=src.now)
            codes = src.requeue(mem[:3000])  # between the async tick and its results
            e.results_wait()
            rl, rm, rs, rst = ref.tick(src.now)
            assert st.n_lobbies == rst.n_lobbies
            assert np.array_equal(bufs[0][:st.n_lobbies], rl) and np.array_equal(bufs[1][:st.n_matched], rm)
            assert np.array_equal(bufs[2][:st.n_lobbies], rs)
            assert (codes == 1).all()
            e.set_option("async_results", 0)
        # snapshot / restore around a requeue
        e.snapshot()
        before = e.pool_read()
        back = bufs[1][:st.n_matched][:2000].astype(np.uint64)
        assert (src.requeue(back) == 1).all() and e.in_queue(back).all()
        after = state_bytes(pkg, e, back)
        e.restore()
        for k, v in e.pool_read().items():
            assert np.array_equal(v, before[k]), k
        assert (src.requeue(back) == 1).all()
        assert state_bytes(pkg, e, back) == after
        # export / import after a requeue: the imported engine ticks as the source
        with pkg.Engine(cfg) as b:
            b.import_state(e.export_state())
            tick_both(e, b, src.now + 10)
            same_state(e, b, src.now + 10, back)
    finally:
        src.close()


# ================================================================================ GPU: scale
@pytest.mark.gpu
def test_config3_ten_million_requeue_hundred_thousand_lobbies(pkg, oracle):
    from .test_tile_geometry import config3_pool
    n = 10_000_000
    cfg = pkg.synth.make_config(n_groups=32, modes=(("5v5", 2, 5),), order=RATING, capacity=n + n // 2,
                                active_capacity=n + 1024, flags=DENSE)
    ids, rating, mode, ts = config3_pool(pkg, n)
    with pkg.Engine(cfg) as e:
        e.set_option("max_spread", 2)
        e.enqueue(ids, rating, mode, ts)
        lob, mem, _, st = e.tick(10)
        assert st.n_lobbies >= 100_000
        pick = np.random.default_rng(1).choice(st.n_lobbies, 100_000, replace=False)
        back = np.concatenate([mem[int(lob[k]["first_member"]):int(lob[k]["first_member"]) + 10] for k in pick])
        back = back.astype(np.uint64)
        img = e.export_state()
        # config3_pool: id = enqueue index = stamp = sequence number
        codes = e.requeue(back, rating[back], mode[back], ts[back], back.astype(U32))
        assert (codes == 1).all()
        with pkg.Engine(cfg) as twin:
            twin.set_option("max_spread", 2)
            twin.import_state(restate(pkg, cfg, img, back, rating[back], mode[back], ts[back], back.astype(U32)))
            pa, pt = e.pool_read(), twin.pool_read()
            for k in pa:
                assert np.array_equal(pa[k], pt[k]), k
            ref = oracle.run_windowed(cfg, 2, pa["id"], pa["rating"], pa["mode"])
            lob2, mem2, _, st2 = e.tick(20)
            assert st2.n_matched == ref.n_matched and np.array_equal(mem2, ref.member_ids)
            assert np.array_equal(lob2, ref.lobbies)
            assert np.array_equal(e.pool_read()["id"], ref.residual_ids)


# ================================================================================ CPU: SearchPool.requeue
def requeue_engine(pkg):
    from .test_handover import ImagingEngine
    from .test_queue_move import MovingEngine

    class RequeueEngine(MovingEngine, ImagingEngine):
        """The CPU engine double with enqueue sequence numbers and requeue(): a requeued player goes back into the
        queue list at the position its number gives."""

        def __init__(self, cfg):
            super().__init__(cfg)
            self.pkg, self.refuse, self.merged = pkg, None, []
            self.seq_of, self.ctr = {}, 0

        def seq_next(self):
            return self.ctr

        def enqueue(self, ids, rating, mode, enq_ts=None):
            acc = super().enqueue(ids, rating, mode, enq_ts)
            for i, (p, c) in enumerate(zip(np.asarray(ids, np.uint64).tolist(), acc.tolist())):
                if c == 1:
                    self.seq_of[p] = (self.ctr + i) & 0xFFFFFFFF
            self.ctr = (self.ctr + len(acc)) & 0xFFFFFFFF
            return acc

        def requeue(self, ids, rating, mode, enq_ts, seq):
            codes = np.zeros(len(ids), np.uint8)
            for i, p in enumerate(np.asarray(ids, np.uint64).tolist()):
                if p not in self.active:
                    codes[i] = 4
                elif p in set(self.q[0].tolist()):
                    codes[i] = 0
                else:
                    codes[i] = 1
                    u = [(self.seq_of[x] - self.ctr) & 0xFFFFFFFF for x in self.q[0].tolist()]
                    k = int(np.searchsorted(u, (int(seq[i]) - self.ctr) & 0xFFFFFFFF))
                    for j, v in enumerate((p, rating[i], mode[i])):
                        self.q[j] = np.insert(self.q[j], k, v)
                    self.alive = np.insert(self.alive, k, 1)
                    self.seq_of[p], self.ts[p] = int(seq[i]), int(enq_ts[i])
            return codes

        def export_state(self):
            import pickle
            return pickle.dumps((super().export_state(), self.seq_of, self.ctr))

        def import_state(self, buf):
            import pickle
            base, self.seq_of, self.ctr = pickle.loads(bytes(buf))
            super().import_state(base)

    return RequeueEngine


def cpu_pool(pkg, clock, wall=None, timeout_ms=None, blob=None, engine=None):
    from .test_handover import boot
    from .fakes import FakeBroker
    sw, cfg, eng, pool = boot(pkg, engine or requeue_engine(pkg), clock, wall or (lambda: 1_700_000_000.0),
                              timeout_ms=timeout_ms, blob=blob)
    broker = FakeBroker()
    from .test_handover import start_workers
    start_workers(sw, broker, pool, pkg)
    return sw, cfg, eng, pool, broker


def lobbies(broker, sw):
    import json
    return [json.loads(p) for p, _props in broker.queues[sw.QUEUE_FORWARD]]


def members(lobby):
    return [p["id"] for team in lobby["teams"].values() for p in team]


def test_ready_check_flow(pkg):
    from .test_expire import publish
    now = [0.0]
    sw, cfg, eng, pool, broker = cpu_pool(pkg, lambda: now[0])
    for i in range(4):  # one 1v1 queue (rating 100): p0..p3 make two lobbies
        publish(pkg, broker, cfg, f"p{i}", 100)
    broker.deliver_all()
    now[0] += 1
    assert pool.tick() == 2
    first = lobbies(broker, sw)[0]
    docs = [p for team in first["teams"].values() for p in team]
    assert members(first) == ["p0", "p1"]
    publish(pkg, broker, cfg, "late", 100)  # arrives after the lobby was emitted
    broker.deliver_all()
    # the ready check: p1 declines (removed), p0 goes back ahead of the later arrival
    pool.remove_user("p1")
    out = pool.requeue(docs)
    assert out == ["requeued", "gone"] and pool.stats["requeued"] == 1
    assert pool.in_queue("p0") and not pool.in_queue("p1")
    publish(pkg, broker, cfg, "later", 100)
    broker.deliver_all()
    now[0] += 1
    pool.tick()
    third = lobbies(broker, sw)[2]
    assert members(third) == ["p0", "late"]  # p0 is older than both arrivals
    assert pool.requeue(docs[:1]) == ["requeued"] and pool.requeue(docs[:1]) == ["queued"]


def test_timeout_counts_from_the_first_stamp(pkg):
    from .test_expire import publish
    now = [0.0]
    sw, cfg, eng, pool, broker = cpu_pool(pkg, lambda: now[0], timeout_ms=5000)
    for i in range(2):
        publish(pkg, broker, cfg, f"t{i}", 100)
    broker.deliver_all()
    pool.flush()  # stamped at 0 s
    now[0] = 3.0
    pool.tick()
    docs = [p for team in lobbies(broker, sw)[0]["teams"].values() for p in team]
    pool.remove_user("t1")
    assert pool.requeue(docs) == ["requeued", "gone"]
    now[0] = 4.0
    pool.tick()
    assert pool.in_queue("t0")  # waited 4 s since the first stamp
    now[0] = 5.5
    pool.tick()
    assert not pool.in_queue("t0") and pool.stats["timed_out"] == 1  # 5.5 s since the first stamp, not since requeue


def test_requeue_after_checkpoint_resume_and_move(pkg):
    from .test_expire import publish
    now, wall = [0.0], [1_700_000_000.0]
    sw, cfg, eng, pool, broker = cpu_pool(pkg, lambda: now[0], lambda: wall[0])
    for i in range(6):
        publish(pkg, broker, cfg, f"c{i}", 100)
    broker.deliver_all()
    now[0] += 1
    pool.tick()
    docs = [[p for team in lob["teams"].values() for p in team] for lob in lobbies(broker, sw)]
    publish(pkg, broker, cfg, "fresh", 100)
    broker.deliver_all()
    blob = pool.checkpoint()
    wall[0] += 10
    sw2, _cfg, eng2, pool2, broker2 = cpu_pool(pkg, lambda: now[0], lambda: wall[0], blob=blob)
    assert pool2.requeue(docs[0]) == ["requeued", "requeued"]
    now[0] += 1
    pool2.tick()
    assert members(lobbies(broker2, sw2)[0]) == ["c0", "c1"]  # older than "fresh"
    # a moved-out group: its matched players are not requeued on the source; after move_in they are on the target
    out_blob = pool2.move_out(["bronze"]) if 100 <= cfg.group_hi[0] else None
    assert out_blob is not None
    assert pool2.requeue(docs[1]) == ["gone", "gone"]
    sw3, _c, eng3, pool3, broker3 = cpu_pool(pkg, lambda: now[0], lambda: wall[0])
    pool3.move_in(out_blob)
    assert set(pool3.queued) == {pool3.handles.lookup("fresh")}
    assert pool3.queued[pool3.handles.lookup("fresh")][3] == 0  # the target's numbering
    lob_docs = [{"id": "fresh"}]
    assert pool3.requeue(lob_docs) == ["queued"]
    publish(pkg, broker3, cfg, "x", 100)
    broker3.deliver_all()
    now[0] += 1
    pool3.tick()
    d3 = [p for team in lobbies(broker3, sw3)[0]["teams"].values() for p in team]
    assert members(lobbies(broker3, sw3)[0]) == ["fresh", "x"]
    publish(pkg, broker3, cfg, "y", 100)
    broker3.deliver_all()
    assert pool3.requeue(d3) == ["requeued", "requeued"]
    now[0] += 1
    pool3.tick()
    assert members(lobbies(broker3, sw3)[1]) == ["fresh", "x"]  # both older than "y"


def test_window_gets_the_first_resident_time_back(pkg):
    """With a window policy, a requeued player is again the oldest entry the window reads, at the clock value of its
    first enqueue, also after the pool's 32-bit millisecond clock has wrapped."""
    import importlib
    from .fakes import FakeBroker
    from .test_expire import publish
    from .test_handover import start_workers
    sw = importlib.import_module("microservice-matchmaking_b200.search_worker")
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=RATING, capacity=1000, active_capacity=4000)
    now = [1000.0]
    pool = sw.SearchPool(requeue_engine(pkg)(cfg), ["1v1", "5v5"], list(pkg.synth.REFERENCE_GROUP_NAMES),
                         flush_every_s=3600, clock=lambda: now[0], window=sw.WindowSchedule(0, 100.0, 1000))
    broker = FakeBroker()
    start_workers(sw, broker, pool, pkg)
    now[0] += 50 * 86400.0  # the stamps below are taken after the millisecond clock has passed 2^32
    for i in range(2):
        publish(pkg, broker, cfg, f"a{i}", 100)
    broker.deliver_all()
    pool.flush()
    first = dict(pool.enqueued_at)
    now[0] += 1.0
    publish(pkg, broker, cfg, "b", 100)
    broker.deliver_all()
    pool.tick()
    lob = lobbies(broker, sw)[0]
    assert members(lob) == ["a0", "a1"] and list(pool.enqueued_at) == [pool.handles.lookup("b")]
    docs = [p for team in lob["teams"].values() for p in team]
    assert pool.requeue(docs) == ["requeued", "requeued"]
    assert list(pool.enqueued_at.items())[:2] == list(first.items())
    assert list(pool.enqueued_at)[2] == pool.handles.lookup("b")
