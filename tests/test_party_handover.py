"""Parties in hand-over (mm_export_parties / mm_merge_parties, Engine.export_parties / merge_parties, SearchPool
checkpoint / resume / move_out / move_in and shard.move_queues with parties queued).

CPU: read_party_image on a hand-built image; the ABI mirror.
GPU: export = party_read + remove of one member per party; merge = one enqueue_party batch; the checkpoint sequence
into a fresh engine against the engine that never stopped; regroup; queue moves at the engine, SearchPool and shard
levels; every refusal against a state snapshot; config3 at 10 M solos and 200 k parties.
"""
import ctypes as C
import importlib
import json
import os

import numpy as np
import pytest

from .test_backfill import cfg_of, gpu_config, group_of
from .test_parties import PartySrc, check_party, party_rating, party_state, restate_plain  # noqa: F401
from .test_widen import RATING, ARRIVAL, rules_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def hand_image(pkg, sizes, seq, ts, mode, ids, rating, seq_next, id_bytes=8):
    abi = pkg.abi
    P, M = len(sizes), len(ids)
    off = abi.party_image_offsets(P, M, id_bytes)
    buf = np.zeros(off[-1], np.uint8)
    h = abi.ImageHeader()
    h.magic, h.version, h.abi_version, h.id_bytes = abi.MM_PARTY_IMAGE_MAGIC, abi.MM_IMAGE_VERSION, abi.MM_ABI_VERSION, id_bytes
    h.total_bytes, h.n_parts, h.n_players, h.n_active, h.seq_next = off[-1], P, M, 0, seq_next
    buf[:C.sizeof(h)] = np.frombuffer(bytes(h), np.uint8)
    idt = np.uint64 if id_bytes == 8 else np.uint32
    for k, (a, dt) in enumerate(((sizes, np.uint8), (seq, np.uint32), (ts, np.uint32), (mode, np.uint8), (ids, idt),
                                 (rating, np.int32))):
        b = np.asarray(a, dt).view(np.uint8)
        buf[off[k]:off[k] + len(b)] = b
    return buf


# ================================================================================ CPU
@pytest.mark.parametrize("id_bytes", [8, 4])
def test_read_party_image_round_trips(pkg, id_bytes):
    sizes, seq, ts, mode = [2, 3, 2], [7, 9, 12], [100, 90, 80], [1, 0, 2]
    ids, rating = list(range(40, 47)), [10, -20, 30, 40, 50, 60, 70]
    buf = hand_image(pkg, sizes, seq, ts, mode, ids, rating, 13, id_bytes)
    assert len(buf) % 8 == 0
    h, c = pkg.engine.read_party_image(buf.tobytes())
    assert (h.magic, h.n_parts, h.n_players, h.n_active, h.seq_next, h.id_bytes) == \
        (pkg.abi.MM_PARTY_IMAGE_MAGIC, 3, 7, 0, 13, id_bytes)
    for k, v in (("size", sizes), ("seq", seq), ("enq_ts", ts), ("mode", mode), ("id", ids), ("rating", rating)):
        assert c[k].tolist() == v, k
    assert c["id"].dtype == (np.uint64 if id_bytes == 8 else np.uint32)
    with pytest.raises(ValueError):
        pkg.engine.read_party_image(buf[:-8])
    assert bytes(pkg.abi.MM_PARTY_IMAGE_MAGIC.to_bytes(4, "little")) == b"MPTY"


def test_abi_mirror_lists_the_party_image_calls(pkg):
    abi = pkg.abi
    hdr = open(os.path.join(ROOT, "include", "mm_engine.h")).read()
    for name, nargs in (("mm_export_parties", 5), ("mm_merge_parties", 6)):
        res, args = abi.PROTOTYPES[name]
        assert res is C.c_int and len(args) == nargs
        assert f"int {name}(" in hdr
    assert "#define MM_PARTY_IMAGE_MAGIC 0x5954504Du" in hdr and "#define MM_PARTY_KEEP_SEQ 1u" in hdr
    assert abi.MM_PARTY_KEEP_SEQ == 1
    so = os.path.join(os.path.dirname(pkg.__file__), "csrc", "libmm_engine.so")
    if os.path.exists(so):
        lib = C.CDLL(so)
        assert hasattr(lib, "mm_export_parties") and hasattr(lib, "mm_merge_parties")


# ================================================================================ GPU helpers
RULES = lambda cfg: {(m, g): (0, 10, 5, 5, 80) for m in range(cfg.n_modes) for g in range(cfg.n_groups)}  # noqa: E731


def build(src, rounds=2, solos=4000, parties=500):
    """Solos, queued parties, matched party members, a removed party and expired parties on src.eng."""
    for _ in range(rounds):
        src.enqueue(*src.fresh(solos))
        sz, ids, r, m, ts = src.fresh_parties(parties)
        ts[::7] = src.now - 900
        assert (src.eng.enqueue_party(sz, ids, r, m, ts) == 1).all()
        src.eng.party_match(src.now, rules_of(src.cfg, {(1, 0): (0, 10, 5, 5, 80), (2, 3): (0, 10, 5, 5, 80)}))
        pr = src.eng.party_read()
        src.eng.remove(pr["members"][3][0][:1])
        src.eng.expire(src.now, 800)
        src.now += 7


def snapshot(eng, ids):
    pr = eng.party_read()
    return dict(parties={k: v.tolist() for k, v in pr.items() if k != "members"},
                members=[(a.tolist(), b.tolist()) for a, b in pr["members"]], in_queue=eng.in_queue(ids).tolist(),
                active=eng.active_size(), seq_next=eng.seq_next(), pool={k: v.tolist() for k, v in eng.pool_read().items()})


def same_locate(a, b, ids, now, skip=()):
    la, lb = a.locate(ids, now), b.locate(ids, now)
    for f in la.dtype.names:
        if f not in skip:
            assert np.array_equal(la[f], lb[f]), f


def same_next(cfg, a, b, now):
    ra = a.party_match(now, rules_of(cfg, RULES(cfg)))
    rb = b.party_match(now, rules_of(cfg, RULES(cfg)))
    assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1])
    ta, tb = a.tick(now), b.tick(now)
    assert np.array_equal(ta[0], tb[0]) and np.array_equal(ta[1], tb[1])
    return ra, ta


KINDS = ["hashed", "dense"]


# ================================================================================ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("layout", ["split", "wide"])
def test_export_equals_read_plus_remove(pkg, kind, layout):
    cfg = gpu_config(pkg, RATING, kind, layout)
    a, b = PartySrc(pkg, cfg, kind, seed=3), PartySrc(pkg, cfg, kind, seed=3)
    try:
        build(a)
        build(b)
        G = cfg.n_groups
        mask = np.zeros(cfg.n_modes * G, bool)
        mask[1::3] = True
        pr = a.eng.party_read()
        sel = mask[pr["mode"].astype(np.int64) * G + pr["group"]]
        img = a.eng.export_parties(mask)
        h, c = pkg.engine.read_party_image(img)
        assert (h.n_parts, h.n_players, h.seq_next) == (int(sel.sum()), int(pr["size"][sel].sum()), b.eng.seq_next())
        for k in ("size", "seq", "enq_ts", "mode"):
            assert np.array_equal(c[k], pr[k][sel]), k
        mem = [pr["members"][j] for j in np.flatnonzero(sel)]
        assert np.array_equal(c["id"], np.concatenate([x[0] for x in mem]).astype(c["id"].dtype))
        assert np.array_equal(c["rating"], np.concatenate([x[1] for x in mem]))
        b.eng.remove(np.array([x[0][0] for x in mem], np.uint64))
        ids = np.concatenate([x[0] for x in pr["members"]] + [a.eng.pool_read()["id"][::17]])
        assert snapshot(a.eng, ids) == snapshot(b.eng, ids)
        assert not a.eng.in_queue(c["id"].astype(np.uint64)).any()
        same_locate(a.eng, b.eng, ids, a.now)
        same_next(cfg, a.eng, b.eng, a.now)
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_merge_equals_one_enqueue_party_batch(pkg, kind):
    cfg = gpu_config(pkg, RATING, kind, "split")
    s = PartySrc(pkg, cfg, kind, seed=4)
    x, y = PartySrc(pkg, cfg, kind, seed=5), PartySrc(pkg, cfg, kind, seed=5)
    try:
        build(s, rounds=1)
        for t in (x, y):
            t.next = 300_000  # other ids than the source's (below the dense handle range)
            t.enqueue(*t.fresh(3000))
            assert (t.eng.enqueue_party(*t.fresh_parties(200)) == 1).all()
        img = np.array(s.eng.export_parties(), copy=True)
        h, c = pkg.engine.read_party_image(img)
        # collisions: members active on the target, and a member repeated in a later party of the image
        c["id"][5] = x.eng.pool_read()["id"][0]
        c["id"][int(c["size"][:10].sum())] = c["id"][0]
        c["id"][int(c["size"][:20].sum())] = x.eng.party_read()["members"][2][0][0]
        codes = x.eng.merge_parties(img)
        want = y.eng.enqueue_party(c["size"], c["id"].astype(np.uint64), c["rating"], c["mode"], c["enq_ts"])
        assert np.array_equal(codes, want) and (codes == 0).sum() >= 3 and (codes == 1).any()
        ids = np.concatenate([c["id"].astype(np.uint64), x.eng.pool_read()["id"][::11]])
        assert snapshot(x.eng, ids) == snapshot(y.eng, ids)
        same_locate(x.eng, y.eng, ids, x.now)
        same_next(cfg, x.eng, y.eng, x.now)
    finally:
        for t in (s, x, y):
            t.close()


def checkpoint_into(pkg, src_eng, cfg, regroup=False, cap=200_000):
    """The checkpoint sequence on src_eng (release, export_state, merge back with keep_seq); -> (fresh engine loaded
    from it, codes of the party merge)"""
    pimg = np.array(src_eng.export_parties(), copy=True)
    try:
        img = src_eng.export_state()
    finally:
        assert (src_eng.merge_parties(pimg, keep_seq=True) == 1).all()
    b = pkg.Engine(cfg)
    b.set_option("party_capacity", cap)
    (b.import_regroup if regroup else b.import_state)(img)
    return b, b.merge_parties(pimg, keep_seq=True), pimg


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("layout", ["split", "wide"])
def test_checkpoint_equals_the_engine_that_never_stopped(pkg, kind, layout):
    cfg = gpu_config(pkg, RATING, kind, layout)
    a, a0 = PartySrc(pkg, cfg, kind, seed=7), PartySrc(pkg, cfg, kind, seed=7)
    b = None
    try:
        build(a)
        build(a0)
        b, codes, _ = checkpoint_into(pkg, a.eng, cfg)
        assert (codes == 1).all()
        engs = (a.eng, a0.eng, b)
        everyone = np.concatenate([x[0] for x in a.eng.party_read()["members"]] + [a.eng.pool_read()["id"]])
        matched = []
        for step in range(12):
            op, now = step % 6, a.now
            if op == 0:
                outs = [e.party_match(now, rules_of(cfg, RULES(cfg))) for e in engs]
                for o in outs[1:]:
                    assert np.array_equal(outs[0][0], o[0]) and np.array_equal(outs[0][1], o[1])
                matched = outs[0][1]
            elif op == 1:
                outs = [e.tick(now) for e in engs]
                for o in outs[1:]:
                    assert all(np.array_equal(p, q) for p, q in zip(outs[0][:3], o[:3]))
                solo = np.setdiff1d(outs[0][1], matched)[:50]
                codes = [a.requeue(solo, eng=e) for e in engs]
                assert all(np.array_equal(codes[0], k) for k in codes[1:])
                a.now += 9
            elif op == 2:
                outs = [e.widen(now, {(0, 0): (10, 5, 1, 1, 50), (1, 2): (0, 20, 1, 1, 90)}) for e in engs]
                assert all(np.array_equal(outs[0][1], o[1]) for o in outs[1:])
            elif op == 3:
                outs = [e.expire(now, 700) for e in engs]
                assert all(np.array_equal(np.sort(outs[0][0]), np.sort(o[0])) for o in outs[1:])
                assert all(sorted(zip(outs[0][0], outs[0][1])) == sorted(zip(o[0], o[1])) for o in outs[1:])
            elif op == 4:
                pr = a.eng.party_read()
                gone = np.array([pr["members"][j][0][-1] for j in range(0, len(pr["size"]), 5)], np.uint64)
                assert len({e.remove(gone) for e in engs}) == 1
            elif op == 5:
                sz, ids, r, m, ts = a.fresh_parties(200)
                ids[::13] = everyone[:len(ids[::13])]  # collisions with queued or matched players
                outs = [e.enqueue_party(sz, ids, r, m, ts) for e in engs]
                assert all(np.array_equal(outs[0], o) for o in outs[1:]) and (outs[0] == 0).any()
                everyone = np.concatenate([everyone, ids])
            ids = everyone[::7]
            sa = snapshot(a.eng, ids)
            for e in engs[1:]:
                se = snapshot(e, ids)
                se["pool"], sa2 = None, dict(sa, pool=None)
                assert se == sa2
                same_locate(a.eng, e, ids, a.now)
            assert np.array_equal(a.eng.pool_read()["id"], b.pool_read()["id"])
            qa, qb = a.eng.queue_stats(a.now), b.queue_stats(a.now)
            for f in ("n_waiting", "max_wait", "wait_hist"):
                assert np.array_equal(qa[f], qb[f]), f
    finally:
        for e in (a, a0):
            e.close()
        if b is not None:
            b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_regroup_files_parties_under_the_new_table(pkg, kind):
    cfg = gpu_config(pkg, RATING, kind, "split")
    a = PartySrc(pkg, cfg, kind, seed=11)
    new = cfg_of(pkg, RATING, groups=[(0, 2000), (2500, 5000)], default_group=-1, flags=2 if kind == "dense" else 0,
                 modes=3)  # a party rated 2001 .. 2499 has no queue here
    b = None
    try:
        build(a, rounds=1)
        b, codes, pimg = checkpoint_into(pkg, a.eng, new, regroup=True)
        _h, c = pkg.engine.read_party_image(pimg)
        mem = np.split(c["id"].astype(np.uint64), np.cumsum(c["size"].astype(np.int64))[:-1])
        rat = np.split(c["rating"], np.cumsum(c["size"].astype(np.int64))[:-1])
        R = [party_rating(r) for r in rat]
        want = np.array([1 if group_of(new, R[j]) >= 0 else 2 for j in range(len(R))], np.uint8)
        assert np.array_equal(codes, want) and (want == 2).any()
        pr = b.party_read()
        keep = want == 1
        assert np.array_equal(pr["seq"], c["seq"][keep]) and np.array_equal(pr["size"], c["size"][keep])
        assert pr["group"].tolist() == [group_of(new, R[j]) for j in np.flatnonzero(keep)]
        assert not b.in_queue(np.concatenate([mem[j] for j in np.flatnonzero(~keep)])).any()
        assert b.seq_next() == a.eng.seq_next()
        check_party(b, new, a.now, RULES(new))
    finally:
        a.close()
        if b is not None:
            b.close()


def lobbies_of(res, queues, G):
    lob, mem = res[0], res[1]
    return [mem[h["first_member"]:h["first_member"] + h["n_members"]].tolist() for h in lob
            if int(h["mode"]) * G + int(h["group"]) in queues]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_queue_move_equals_the_engine_without_a_move(pkg, kind):
    cfg = gpu_config(pkg, RATING, kind, "split")
    s, u = PartySrc(pkg, cfg, kind, seed=21), PartySrc(pkg, cfg, kind, seed=21)
    t = pkg.Engine(cfg)
    try:
        build(s, rounds=1)
        build(u, rounds=1)
        t.set_option("party_capacity", 200_000)
        G = cfg.n_groups
        mask = np.zeros(cfg.n_modes * G, bool)
        mask[[G + 1, G + 2, 2 * G + 3, 2 * G + 4]] = True
        moved, other = set(np.flatnonzero(mask).tolist()), set(np.flatnonzero(~mask).tolist())
        pimg = s.eng.export_parties(mask)
        rest = s.eng.export_parties(~mask)
        qimg = s.eng.export_queues(mask)
        assert (s.eng.merge_parties(rest, keep_seq=True) == 1).all()
        t.merge_queues(qimg)
        assert (t.merge_parties(pimg) == 1).all()
        rules = rules_of(cfg, RULES(cfg))
        for k in range(2):
            rs, rt, ru = (e.party_match(s.now, rules) for e in (s.eng, t, u.eng))
            assert lobbies_of(rt, moved, G) == lobbies_of(ru, moved, G) and (k or len(lobbies_of(ru, moved, G)))
            assert lobbies_of(rs, other, G) == lobbies_of(ru, other, G)
            ts, tt, tu = (e.tick(s.now) for e in (s.eng, t, u.eng))
            assert lobbies_of(tt, moved, G) == lobbies_of(tu, moved, G)
            assert lobbies_of(ts, other, G) == lobbies_of(tu, other, G)
            s.now += 40
        # a refused merge changes nothing: the table is full
        small = pkg.Engine(cfg)
        small.set_option("party_capacity", 4)
        before = snapshot(small, np.zeros(1, np.uint64))
        with pytest.raises(pkg.EngineError) as ex:
            small.merge_parties(pimg)
        assert ex.value.status == pkg.abi.MM_E_CAP and snapshot(small, np.zeros(1, np.uint64)) == before
        small.close()
    finally:
        s.close()
        u.close()
        t.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_refusals_change_nothing(pkg, kind):
    abi = pkg.abi
    FLAGS = abi.ImageHeader.config.offset + abi.Config.flags.offset  # config.flags in the header
    cfg = gpu_config(pkg, RATING, kind, "split")
    a = PartySrc(pkg, cfg, kind, seed=31, cap=600)
    try:
        build(a, rounds=1, parties=100)
        ids = np.concatenate([x[0] for x in a.eng.party_read()["members"]] + [a.eng.pool_read()["id"][::5]])
        before = snapshot(a.eng, ids)
        good = np.array(a.eng.export_parties(), copy=True)  # release, then back with the numbers
        assert (a.eng.merge_parties(good, keep_seq=True) == 1).all()
        assert snapshot(a.eng, ids) == before

        def refused(status, call):
            with pytest.raises(pkg.EngineError) as ex:
                call()
            assert ex.value.status == status, ex.value
            assert snapshot(a.eng, ids) == before

        # the dry run and a short buffer
        n = C.c_uint64(0)
        assert a.eng.lib.mm_export_parties(a.eng.h, None, None, 0, C.byref(n)) == abi.MM_OK and n.value == len(good)
        buf = np.zeros(len(good), np.uint8)
        assert a.eng.lib.mm_export_parties(a.eng.h, None, buf.ctypes.data, len(good) - 8, C.byref(n)) == abi.MM_E_CAP
        assert snapshot(a.eng, ids) == before
        # keep_seq with queued parties; unknown flags; keep_seq on an empty table whose seq_next is not the image's
        refused(abi.MM_E_STATE, lambda: a.eng.merge_parties(good, keep_seq=True))
        k0 = C.c_uint32(0)
        assert a.eng.lib.mm_merge_parties(a.eng.h, good.ctypes.data, len(good), 2, None, C.byref(k0)) == abi.MM_E_ARG
        assert snapshot(a.eng, ids) == before
        shifted = np.array(good, copy=True)
        shifted[36:40] = np.array([pkg.engine.read_party_image(good)[0].seq_next + 5], np.uint32).view(np.uint8)
        empty = np.array(a.eng.export_parties(), copy=True)
        released = snapshot(a.eng, ids)
        with pytest.raises(pkg.EngineError) as ex:
            a.eng.merge_parties(shifted, keep_seq=True)
        assert ex.value.status == abi.MM_E_STATE and snapshot(a.eng, ids) == released
        assert (a.eng.merge_parties(empty, keep_seq=True) == 1).all() and snapshot(a.eng, ids) == before
        # hostile images
        h, c = pkg.engine.read_party_image(good)

        def mutate(f):
            x = np.array(good, copy=True)
            f(x, pkg.engine.read_party_image(x)[1])
            return x
        hostile = [
            good[:-8], good[:100],
            mutate(lambda x, c: x.__setitem__(slice(0, 4), 0)),  # magic
            mutate(lambda x, c: x.__setitem__(4, 9)),  # version
            mutate(lambda x, c: c["size"].__setitem__(0, 1)),  # size below 2
            mutate(lambda x, c: c["size"].__setitem__(0, int(c["size"][0]) + 1)),  # sizes do not add up
            mutate(lambda x, c: c["seq"].__setitem__(1, c["seq"][0])),  # seq not increasing
            mutate(lambda x, c: c["seq"].__setitem__(len(c["seq"]) - 1, h.seq_next)),  # seq == seq_next
            mutate(lambda x, c: c["id"].__setitem__(3, c["id"].dtype.type(cfg.active_capacity if kind == "dense"
                                                                           else (1 << 64) - 1))),  # id out of range
            mutate(lambda x, c: x.__setitem__(slice(FLAGS, FLAGS + 4), np.array(  # written by an MM_F_NO_DEDUPE engine
                [int(x[FLAGS:FLAGS + 4].view(np.uint32)[0]) | 1], np.uint32).view(np.uint8))),
        ]
        other_width = PartySrc(pkg, gpu_config(pkg, RATING, "hashed" if kind == "dense" else "dense", "split"),
                               "hashed" if kind == "dense" else "dense", seed=1)
        other_width.eng.enqueue_party(*other_width.fresh_parties(3))
        hostile.append(np.array(other_width.eng.export_parties(), copy=True))
        other_width.close()
        for x in hostile:
            refused(abi.MM_E_ARG, lambda: a.eng.merge_parties(x))
            refused(abi.MM_E_ARG, lambda: a.eng.merge_parties(x, keep_seq=True))
        # exact MM_E_CAP: 600 members of room, the image holds more than the room left
        pimg = np.array(a.eng.export_parties(), copy=True)
        big = PartySrc(pkg, cfg, kind, seed=2)
        big.next = 600_000
        big.eng.enqueue_party(*big.fresh_parties(300))
        bimg = np.array(big.eng.export_parties(), copy=True)
        big.close()
        assert (a.eng.merge_parties(pimg, keep_seq=True) == 1).all()
        refused(abi.MM_E_CAP, lambda: a.eng.merge_parties(bimg))
        # exact: a merge that fits only because its code-0 parties take no room is accepted
        hb, cb = pkg.engine.read_party_image(bimg)
        room = 600 - sum(len(m[0]) for m in a.eng.party_read()["members"])
        k = int(np.searchsorted(np.cumsum(cb["size"].astype(np.int64)), room, side="right"))
        assert 0 < k < len(cb["size"])
        fit = np.array(bimg, copy=True)
        cf = pkg.engine.read_party_image(fit)[1]
        off = np.concatenate([[0], np.cumsum(cf["size"].astype(np.int64))])
        for j in range(k, len(cf["size"])):  # every later party collides with an active id: code 0
            cf["id"][off[j]] = cf["id"].dtype.type(ids[j % len(ids)])
        codes = a.eng.merge_parties(fit)
        assert (codes[:k] == 1).all() and (codes[k:] == 0).all()
        # a refusal for room gives every claim back: the refused ids then queue as solos
        big = PartySrc(pkg, cfg, kind, seed=6)
        big.next = 700_000
        big.eng.enqueue_party(*big.fresh_parties(300))
        rimg = np.array(big.eng.export_parties(), copy=True)
        big.close()
        now = snapshot(a.eng, ids)
        refused_ids = pkg.engine.read_party_image(rimg)[1]["id"].astype(np.uint64)
        with pytest.raises(pkg.EngineError) as ex:
            a.eng.merge_parties(rimg)
        assert ex.value.status == abi.MM_E_CAP and snapshot(a.eng, ids) == now
        assert not a.eng.in_queue(refused_ids).any() and (a.eng.locate(refused_ids, a.now)["state"] == 0).all()
        n0 = a.eng.active_size()
        r = pkg.engine.read_party_image(rimg)[1]["rating"]
        assert (a.eng.enqueue(refused_ids, r, np.zeros(len(r), np.uint8)) == 1).all()
        assert a.eng.active_size() == n0 + len(refused_ids)
    finally:
        a.close()
    # no capacity, a staged batch, an arrival-order engine
    for c2, cap in ((cfg, 0), (gpu_config(pkg, ARRIVAL, kind, "split"), 100)):
        e = pkg.Engine(c2)
        try:
            if cap:
                e.set_option("party_capacity", cap)
            st = (e.active_size(), e.seq_next())
            for call in (lambda: e.export_parties(), lambda: e.merge_parties(good)):
                with pytest.raises(pkg.EngineError) as ex:
                    call()
                assert ex.value.status == (abi.MM_E_STATE if not cap else abi.MM_E_ARG)
            assert (e.active_size(), e.seq_next()) == st
            if kind == "dense" and not cap:
                e.set_option("party_capacity", 100)
                e.enqueue_packed_begin(np.array([50], np.uint32), e.pack_key([100], [1]))
                for call in (lambda: e.export_parties(), lambda: e.merge_parties(good)):
                    with pytest.raises(pkg.EngineError) as ex:
                        call()
                    assert ex.value.status == abi.MM_E_STATE
                e.enqueue_packed_end()
        finally:
            e.close()


# ================================================================================ SearchPool and shard
@pytest.mark.gpu
def test_search_pool_checkpoint_resume_and_moves_with_parties(pkg):
    sw = importlib.import_module(pkg.__name__ + ".search_worker")
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=[("1v1", 2, 1), ("5v5", 2, 5)], order=RATING,
                                capacity=100_000, active_capacity=200_000)
    t = [100.0]
    clock = lambda: t[0]  # noqa: E731
    opts = dict(parties={"5v5": (1500, 30, 5, 5, 200)}, party_capacity=10_000)  # parties match from the second tick
    rng = np.random.default_rng(5)

    def fill(pool, first):
        w = _Pub()
        for k in range(300):
            r = int(rng.integers(0, 3000))
            pool.stage(w, k, {"id": f"s{first + k}", "rating": r}, "5v5" if k % 2 else "1v1", r)
        for k in range(40):
            r = int(rng.integers(0, 3000))
            pool.stage_party(w, 1000 + k, [{"id": f"p{first + k}-{j}", "rating": r + j} for j in range(2 + k % 3)],
                             "5v5")
        pool.flush()
    names = ["1v1", "5v5"], [str(g) for g in range(cfg.n_groups)]
    pools = []
    try:
        for _ in range(2):
            e = pkg.Engine(cfg)
            p = sw.SearchPool(e, *names, clock=clock, wall_clock=clock, **opts)
            pools.append(p)
        for p in pools:
            p.workers = {g: _Pub() for g in names[1]}
        for p in pools:
            rng = np.random.default_rng(5)
            fill(p, 0)
        blob = pools[0].checkpoint()
        e2 = pkg.Engine(cfg)
        resumed = sw.SearchPool.resume(e2, blob, *names, clock=clock, wall_clock=clock, **opts)
        pools.append(resumed)
        for p in pools[1:]:
            p.workers = {g: _Pub() for g in names[1]}
        pools[0].workers = {g: _Pub() for g in names[1]}
        t[0] += 1.0
        outs = []
        for p in (pools[0], pools[1], resumed):
            p.tick()
            outs.append([x for w in p.workers.values() for x in w.sent])
        assert outs[0] == outs[1] == outs[2] and len(outs[0]) > 0
        assert resumed.party_of == pools[1].party_of
        # move_out / move_in of two groups into a fresh pool, against the pool that kept them
        e3 = pkg.Engine(cfg)
        target = sw.SearchPool(e3, *names, clock=clock, wall_clock=clock, **opts)
        target.workers = {g: _Pub() for g in names[1]}
        moved = target.move_in(resumed.move_out(["2", "3"]))
        assert moved > 0 and any(h in target.party_of for h in target.players)
        t[0] += 1.0
        for p in (pools[1], resumed, target):
            for w in p.workers.values():
                w.sent.clear()
            p.tick()
        keep = [x for w in pools[1].workers.values() for x in w.sent]
        got = [x for w in resumed.workers.values() for x in w.sent] + [x for w in target.workers.values() for x in w.sent]
        assert sorted(keep) == sorted(got)
        e3.close()
        # a pool without party capacity writes the parent's blob layout
        e4 = pkg.Engine(cfg)
        plain = sw.SearchPool(e4, *names, clock=clock, wall_clock=clock)
        b = plain.checkpoint()
        n = int.from_bytes(b[8:16], "little")
        assert set(json.loads(b[16:16 + n])) == {"mode_names", "group_names", "id_of", "free", "players", "enqueued_at",
                                                  "matched_at", "queued", "moved_out", "now_ms", "wall"}
        assert b[16 + n:16 + n + 4] == pkg.abi.MM_IMAGE_MAGIC.to_bytes(4, "little")
        e4.close()
    finally:
        for p in pools:
            p.engine.close()


def pool_state(pool):
    e = pool.engine
    pr = e.party_read()
    return dict(pool=e.pool_read()["id"].tolist(), active=e.active_size(), seq=e.seq_next(),
                parties=[x[0].tolist() for x in pr["members"]], pseq=pr["seq"].tolist(), players=dict(pool.players),
                party_of=dict(pool.party_of), queued=dict(pool.queued), id_of=list(pool.handles.id_of),
                free=list(pool.handles.free), moved_out=set(pool.moved_out))


@pytest.mark.gpu
def test_search_pool_refused_move_in_changes_nothing(pkg):
    sw = importlib.import_module(pkg.__name__ + ".search_worker")
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=[("1v1", 2, 1), ("5v5", 2, 5)], order=RATING,
                                capacity=100_000, active_capacity=200_000)
    names = ["1v1", "5v5"], [str(g) for g in range(cfg.n_groups)]
    clock = lambda: 100.0  # noqa: E731
    opts = dict(parties={"5v5": (10_000, 30, 5, 5, 200)})
    src = sw.SearchPool(pkg.Engine(cfg), *names, clock=clock, wall_clock=clock, party_capacity=10_000, **opts)
    small = sw.SearchPool(pkg.Engine(cfg), *names, clock=clock, wall_clock=clock, party_capacity=3, **opts)
    try:
        w = _Pub()
        for k in range(200):
            src.stage(w, k, {"id": f"s{k}", "rating": 100 + k}, "5v5", 100 + k)
            small.stage(w, k, {"id": f"t{k}", "rating": 2100 + k}, "5v5", 2100 + k)
        for k in range(20):
            src.stage_party(w, 1000 + k, [{"id": f"p{k}-{j}", "rating": 200 + k} for j in range(2)], "5v5")
        small.stage_party(w, 2000, [{"id": "q-0", "rating": 2200}, {"id": "q-1", "rating": 2201}], "5v5")
        src.flush()
        small.flush()
        blob = src.move_out(["0"])
        n = int.from_bytes(blob[8:16], "little")
        assert len(json.loads(blob[16:16 + n])["party_players"]) == 40
        before = pool_state(small)
        with pytest.raises(ValueError):  # 1 party of 2 queued, 40 members moved, room for 3
            small.move_in(blob)
        assert pool_state(small) == before
        assert src.move_in(blob) == 200  # the refused move goes back where it came from
        assert len(src.party_of) == 40 and len(src.engine.party_read()["size"]) == 20
    finally:
        src.engine.close()
        small.engine.close()


class _Pub:
    channel_name = "c"

    def __init__(self):
        self.sent = []

    def prepare_game_lobby(self, channel, exchange, queue, payload):
        self.sent.append(payload)

    def ack(self, *a):
        pass

    def nack(self, *a):
        pass

    def send_response(self, *a):
        pass


@pytest.mark.gpu
@pytest.mark.parametrize("K", [2, 4])
def test_shard_move_queues_carries_parties(pkg, K):
    import threading
    cfg = gpu_config(pkg, RATING, "hashed", "split")
    G = cfg.n_groups
    old = np.arange(G) % K
    new = (old + 1) % K
    srcs = [PartySrc(pkg, cfg, "hashed", seed=40 + r) for r in range(K)]
    twins = [PartySrc(pkg, cfg, "hashed", seed=40 + r) for r in range(K)]
    try:
        for r in range(K):
            for x in (srcs[r], twins[r]):
                x.next = r * 200_000
                build(x, rounds=1, solos=2000, parties=200)
                own = old == r  # every rank starts with the groups it owns only
                p = x.eng.pool_read()
                x.eng.remove(p["id"][~own[[group_of(cfg, int(v)) for v in p["rating"]]]])
                pr = x.eng.party_read()
                x.eng.remove(np.array([ms[0][0] for ms, g in zip(pr["members"], pr["group"]) if not own[g]], np.uint64))
        shard = importlib.import_module("microservice-matchmaking_b200.shard")
        comm = shard.LocalComm()
        outs = [None] * K

        def run(r):
            outs[r] = shard.move_queues(pkg, cfg, old, new, r, srcs[r].eng, comm)
        th = [threading.Thread(target=run, args=(r,)) for r in range(K)]
        for x in th:
            x.start()
        for x in th:
            x.join()
        for r, o in enumerate(outs):
            assert sorted(o["moved"]) == sorted(g for g in range(G) if r in (old[g], new[g])), (r, o)
        rules = rules_of(cfg, RULES(cfg))
        now = srcs[0].now
        res_s = [s.eng.party_match(now, rules) for s in srcs]
        res_t = [s.eng.party_match(now, rules) for s in twins]
        for g in range(G):  # rank new[g] now serves group g as rank old[g] would have
            qs = {m * G + g for m in range(cfg.n_modes)}
            assert lobbies_of(res_s[new[g]], qs, G) == lobbies_of(res_t[old[g]], qs, G)
        assert sum(len(r[0]) for r in res_s) > 0
    finally:
        for x in srcs + twins:
            x.close()


@pytest.mark.gpu
def test_config3_checkpoint_with_200k_parties(pkg):
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=[("5v5", 2, 5)], order=RATING,
                                capacity=10_500_000, active_capacity=12_000_000)
    a = pkg.Engine(cfg)
    b = None
    rng = np.random.default_rng(1)
    try:
        a.set_option("party_capacity", 1_000_000)
        n = 10_000_000
        a.enqueue(np.arange(n, dtype=np.uint64) + np.uint64(1 << 40), rng.integers(0, 3000, n).astype(np.int32),
                  np.zeros(n, np.uint8), rng.integers(0, 100, n).astype(np.uint32))
        k = 200_000
        sizes = rng.integers(2, 5, k).astype(np.uint8)
        m = int(sizes.sum())
        prat = np.clip(np.repeat(rng.integers(0, 3000, k), sizes) + rng.integers(-30, 31, m), 0, 2999).astype(np.int32)
        assert (a.enqueue_party(sizes, np.arange(m, dtype=np.uint64) + np.uint64(1 << 41), prat, np.zeros(k, np.uint8),
                                rng.integers(0, 100, k).astype(np.uint32)) == 1).all()
        b, codes, _ = checkpoint_into(pkg, a, cfg, cap=1_000_000)
        assert (codes == 1).all() and len(codes) == k
        rules = rules_of(cfg, {(0, g): (30, 10, 5, 5, 100) for g in range(cfg.n_groups)})
        ra = a.party_match(100, rules, lobby_cap=1 << 20, member_cap=1 << 24)
        rb = b.party_match(100, rules, lobby_cap=1 << 20, member_cap=1 << 24)
        assert ra[2].n_lobbies > 1000 and np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1])
        ta, tb = a.tick(100), b.tick(100)
        assert np.array_equal(ta[0], tb[0]) and np.array_equal(ta[1], tb[1]) and np.array_equal(ta[2], tb[2])
    finally:
        a.close()
        if b is not None:
            b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("why", ["party_room", "staged_batch"])
def test_shard_refused_moves_change_nothing(pkg, why):
    """Rank 1 cannot take rank 0's groups: its party table is full, or a packed batch is staged on it (every engine
    call there is refused).  Every message is still answered, and both ranks keep every player and party."""
    import threading
    cfg = gpu_config(pkg, RATING, "dense", "split")
    G, K = cfg.n_groups, 2
    old = np.arange(G) % K
    new = (old + 1) % K
    srcs = [PartySrc(pkg, cfg, "dense", seed=60 + r) for r in range(K)]
    try:
        for r in range(K):
            x = srcs[r]
            x.next = r * 200_000
            build(x, rounds=1, solos=2000, parties=200)
            own = old == r
            p = x.eng.pool_read()
            x.eng.remove(p["id"][~own[[group_of(cfg, int(v)) for v in p["rating"]]]])
            pr = x.eng.party_read()
            x.eng.remove(np.array([ms[0][0] for ms, g in zip(pr["members"], pr["group"]) if not own[g]], np.uint64))
        if why == "party_room":
            srcs[1].eng.set_option("party_capacity", int(srcs[1].eng.party_read()["size"].sum()) + 1)
        else:
            srcs[1].eng.enqueue_packed_begin(np.array([900_000], np.uint32), srcs[1].eng.pack_key([100], [1]))

        def held(e):
            return (sorted(e.pool_read()["id"].tolist()), sorted(tuple(m[0].tolist()) for m in e.party_read()["members"]))
        def by_group(e, g):
            p, pr = e.pool_read(), e.party_read()
            return (sorted(i for i, r in zip(p["id"].tolist(), p["rating"].tolist()) if group_of(cfg, r) == g),
                    sorted(tuple(m[0].tolist()) for m, q in zip(pr["members"], pr["group"]) if q == g))
        before = [held(srcs[0].eng)]
        groups0 = {g: by_group(srcs[0].eng, g) for g in range(G)}
        shard = importlib.import_module("microservice-matchmaking_b200.shard")
        comm = shard.LocalComm()
        outs = [None] * K

        def run(r):
            outs[r] = shard.move_queues(pkg, cfg, old, new, r, srcs[r].eng, comm)
        th = [threading.Thread(target=run, args=(r,)) for r in range(K)]
        for x in th:
            x.start()
        for x in th:
            x.join()
        assert all(o is not None for o in outs)  # no rank was left waiting
        if why == "party_room":  # a refused group of rank 0 keeps its players and parties there
            failed = [g for g in outs[0]["failed"] if old[g] == 0]
            assert failed and not outs[0]["stranded"] and not outs[1]["stranded"]
            for g in failed:
                assert by_group(srcs[0].eng, g) == groups0[g]
        else:
            assert sorted(outs[0]["failed"] + outs[1]["failed"]) == sorted(list(range(G)) * 2)
            assert not outs[0]["stranded"] and not outs[1]["stranded"]
            assert held(srcs[0].eng) == before[0]  # the refused groups went back (their solos and parties)
            srcs[1].eng.enqueue_packed_end()
    finally:
        for x in srcs:
            x.close()
