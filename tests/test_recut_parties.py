"""Re-cut with parties queued (mm_import_regroup_many_parties, Engine.import_regroup_many_parties, shard.recut).

CPU: the numpy restatement restate_many_parties(images, party_images, cfg, keep, active) -> (R, RP, solo rejects,
party rejects, (solos elsewhere, parties elsewhere)) on hand-built images: one image keeps every number, two images
interleave solos and parties by stamp, a falling party stamp run is keyed by its running maximum, equal stamps go to
the lower image, a party whose R changes group lands in its new group's queue, reject versus skip, and without party
images it is test_recut's restatement.  The ABI mirror.  shard.recut over LocalComm threads with an engine double that
holds parties: a swap everywhere, or a rollback everywhere that merges every rank's party image back with keep_seq.
GPU: the engine after the call against a fresh engine that mm_import'ed R and merged RP with MM_PARTY_KEEP_SEQ; no
party images against mm_import_regroup_many (sections 1-6 byte for byte, the active ids as a set: their order is the
hash table's); one image against import_regroup + merge_parties; every refusal; shard.recut on four ranks of one GPU
against one engine loaded with (R, RP); its rollback; config3 with 10 M solos and 200 k parties.
"""
import ctypes as C
import os
import zlib

import numpy as np
import pytest

from .test_party_handover import hand_image
from .test_recut import PAIRS_MANY, image, pair_configs, restate_many, sharded_sources
from .test_requeue import layout_parts
from .test_regroup import ARRIVAL, NO_DEDUPE, REF, SPLIT, TWO, cfg_of, groups_of, make_image, same_as_image
from .test_tile_geometry import WIDE

U32 = np.uint32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ================================================================================ the restatement
def party_rating(rating, sizes):
    """R = floor(sum / size) of each party's member ratings."""
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    s = np.array([int(np.asarray(rating[off[j]:off[j + 1]], np.int64).sum()) for j in range(len(sizes))], np.int64)
    return np.floor_divide(s, np.asarray(sizes, np.int64))


def restate_many_parties(pkg, images, party_images, cfg, keep=None, active=None):
    """-> (R, RP, rejected [n, 2], party_rejected [n, 2], (n_elsewhere, party_elsewhere)): the header's restated images."""
    K = len(images)
    R0, rej, n_else = restate_many(pkg, images, cfg, keep, active)
    parsed = [pkg.engine.read_image(np.array(img, np.uint8, copy=True)) for img in images]
    sel = np.ones(cfg.n_modes * cfg.n_groups, bool) if keep is None else np.asarray(keep, bool).reshape(-1)
    tsz = np.array([cfg.modes[m].team_size for m in range(cfg.n_modes)])
    prej, p_else, parties = [], 0, []  # parties: (rm, image, age, seq, ts, mode, ids, ratings)
    for k, pimg in enumerate(party_images):
        if pimg is None or len(pimg) == 0:
            continue
        h, c = pkg.engine.read_party_image(np.asarray(pimg, np.uint8).tobytes())
        assert h.seq_next == parsed[k][0].seq_next
        sizes = c["size"].astype(np.int64)
        off = np.concatenate([[0], np.cumsum(sizes)])
        Rp = party_rating(c["rating"], sizes)
        mode = c["mode"].astype(np.int64)
        g = np.full(len(sizes), -1, np.int64)
        ok = mode < cfg.n_modes
        g[ok] = groups_of(cfg, np.clip(Rp[ok], -2**31, 2**31 - 1))
        ok &= g >= 0
        ok[ok] &= sizes[ok] <= tsz[mode[ok]]
        prej += [(k, int(j)) for j in np.flatnonzero(~ok)]
        q = np.where(ok, mode * cfg.n_groups + np.maximum(g, 0), -1)
        kept = ok & sel[np.maximum(q, 0)]
        p_else += int((ok & ~kept).sum())
        rm = c["enq_ts"].astype(np.int64).copy()
        for qq in np.unique(q[kept]):  # image k's run of one queue, in age (= index) order
            sl = np.flatnonzero(kept & (q == qq))
            rm[sl] = np.maximum.accumulate(rm[sl])
        for j in np.flatnonzero(kept):
            age = (int(c["seq"][j]) - int(h.seq_next)) % (1 << 32)
            parties.append((int(rm[j]), k, age, int(c["seq"][j]), int(c["enq_ts"][j]), int(mode[j]),
                            c["id"][off[j]:off[j + 1]].astype(np.uint64), c["rating"][off[j]:off[j + 1]]))
    if K == 1:
        seq_next = parsed[0][0].seq_next
        R = R0
        order = sorted(range(len(parties)), key=lambda i: parties[i][2])
        pseq = [parties[i][3] for i in order]
    else:
        # the solos' keys (rm, image, age) as restate_many computes them, the parties' beside them: one total order
        sk = {x: [] for x in ("rm", "img", "age", "id", "rating", "mode", "ts")}
        for k, (h, s) in enumerate(parsed):
            mode = s["mode"].astype(np.int64)
            g = np.full(len(mode), -1, np.int64)
            has = mode < cfg.n_modes
            g[has] = groups_of(cfg, s["rating"][has])
            ok = g >= 0
            idx = np.flatnonzero(ok & sel[np.where(ok, mode * cfg.n_groups + g, 0)])
            part = layout_parts(cfg, s["rating"][idx], s["mode"][idx]) if len(idx) else np.zeros(0, np.int64)
            age = (s["seq"][idx] - U32(h.seq_next)).astype(U32).astype(np.int64)
            o = np.lexsort((age, part))
            idx, part, age = idx[o], part[o], age[o]
            rm = s["enq_ts"][idx].astype(np.int64)
            for p_ in np.unique(part):
                sl = part == p_
                rm[sl] = np.maximum.accumulate(rm[sl])
            for x, v in (("rm", rm), ("img", np.full(len(idx), k)), ("age", age), ("id", s["id"][idx].astype(np.uint64)),
                         ("rating", s["rating"][idx]), ("mode", s["mode"][idx]), ("ts", s["enq_ts"][idx])):
                sk[x].append(v)
        sk = {x: np.concatenate(v) for x, v in sk.items()}
        ns = len(sk["id"])
        prm = np.array([p[0] for p in parties], np.int64)
        pim = np.array([p[1] for p in parties], np.int64)
        pag = np.array([p[2] for p in parties], np.int64)
        g_order = np.lexsort((np.r_[sk["age"], pag], np.r_[sk["img"], pim], np.r_[sk["rm"], prm]))
        seq_all = np.empty(len(g_order), np.int64)
        seq_all[g_order] = np.arange(len(g_order))
        sseq = seq_all[:ns]
        order = [int(i) - ns for i in g_order if i >= ns]
        pseq = [int(seq_all[ns + i]) for i in order]
        seq_next = len(g_order)
        act = parsed[active][1]["active"].astype(np.uint64) if active is not None else np.zeros(0, np.uint64)
        R = make_image(pkg, cfg, sk["id"], sk["rating"].astype(np.int32), sk["mode"].astype(np.uint8),
                       sk["ts"].astype(U32), sseq.astype(U32), act, seq_next, parsed[0][0].id_bytes)
    ps = [parties[i] for i in order]
    idb = parsed[0][0].id_bytes
    RP = hand_image(pkg, [len(p[6]) for p in ps], pseq, [p[4] for p in ps], [p[5] for p in ps],
                    np.concatenate([p[6] for p in ps]) if ps else [], np.concatenate([p[7] for p in ps]) if ps else [],
                    seq_next, idb)
    h = pkg.abi.ImageHeader.from_buffer_copy(RP[:C.sizeof(pkg.abi.ImageHeader)].tobytes())
    h.config = cfg
    RP[:C.sizeof(h)] = np.frombuffer(bytes(h), np.uint8)
    return R, RP, rej, np.array(prej, np.int64).reshape(-1, 2), (n_else, p_else)


def pparse(pkg, RP):
    _h, c = pkg.engine.read_party_image(np.asarray(RP, np.uint8).tobytes())
    return c


# ================================================================================ CPU: hand-built KATs
def test_one_image_keeps_every_number(pkg):
    cfg = cfg_of(pkg, TWO)
    img = image(pkg, cfg, [1, 2, 3], [100, 1200, 300], [0, 0, 1], [5, 6, 7], [101, 103, 106])
    pimg = hand_image(pkg, [2, 2], [102, 105], [5, 7], [1, 1], [10, 11, 12, 13], [900, 1100, 100, 200], 100)
    R, RP, rej, prej, (ne, pe) = restate_many_parties(pkg, [img], [pimg], cfg)
    assert np.array_equal(R, restate_many(pkg, [img], cfg)[0])
    c = pparse(pkg, RP)
    assert c["seq"].tolist() == [102, 105] and len(prej) == 0 and pe == 0
    assert pkg.engine.read_party_image(RP.tobytes())[0].seq_next == 100


def test_two_images_interleave_solos_and_parties_by_stamp(pkg):
    cfg = cfg_of(pkg, TWO)
    a = image(pkg, cfg, [1, 2], [100, 200], [0, 0], [10, 30], [1, 3], seq_next=0)
    b = image(pkg, cfg, [3], [150], [0], [20], [1], seq_next=0)
    pa = hand_image(pkg, [2], [2], [25], [1], [10, 11], [100, 120], 0)
    pb = hand_image(pkg, [2], [2], [5], [1], [20, 21], [300, 310], 0)
    R, RP, *_ = restate_many_parties(pkg, [a, b], [pa, pb], cfg)
    _h, s = pkg.engine.read_image(np.array(R, copy=True))
    seq = dict(zip(s["id"].tolist(), s["seq"].tolist()))
    c = pparse(pkg, RP)
    # stamps: party b 5, solo 1 10, solo 3 20, party a 25, solo 2 30
    assert c["seq"].tolist() == [0, 3] and c["id"].tolist() == [20, 21, 10, 11]
    assert (seq[1], seq[3], seq[2]) == (1, 2, 4)
    assert pkg.engine.read_party_image(RP.tobytes())[0].seq_next == 5


def test_falling_party_run_takes_its_running_maximum_and_ties_go_to_the_lower_image(pkg):
    cfg = cfg_of(pkg, TWO)
    a = image(pkg, cfg, [], [], [], [], [], seq_next=0)
    b = image(pkg, cfg, [], [], [], [], [], seq_next=0)
    pa = hand_image(pkg, [2, 2], [1, 2], [50, 10], [1, 1], [1, 2, 3, 4], [100, 100, 100, 100], 0)  # run max 50, 50
    pb = hand_image(pkg, [2], [1], [50], [1], [5, 6], [200, 200], 0)
    _R, RP, *_ = restate_many_parties(pkg, [a, b], [pa, pb], cfg)
    assert pparse(pkg, RP)["id"].tolist() == [1, 2, 3, 4, 5, 6]


def test_a_party_whose_rating_moves_lands_in_its_new_queue_and_reject_versus_skip(pkg):
    old = cfg_of(pkg, TWO, modes=3)
    new = cfg_of(pkg, ((0, 499), (500, 1999)), modes=2)
    img = image(pkg, old, [], [], [], [], [], seq_next=0)
    tsz = new.modes[1].team_size
    pimg = hand_image(pkg, [2, 2, 2, tsz + 1], [1, 2, 3, 4], [1, 2, 3, 4], [1, 2, 1, 1],
                      list(range(10, 16 + tsz + 1)), [600, 800, 10, 20, 100, 200] + [700] * (tsz + 1), 0)
    # R 700 was group 0 of the old table (0 .. 999) and is group 1 (500 .. 1999) here: it lands in queue (1, 1), which
    # this rank keeps; R 150 stays in group 0, whose queue (1, 0) another rank keeps
    assert groups_of(old, [700]).tolist() == [0] and groups_of(new, [700]).tolist() == [1]
    keep = np.zeros((new.n_modes, new.n_groups), bool)
    keep[1, 1] = True
    R, RP, rej, prej, (ne, pe) = restate_many_parties(pkg, [img], [pimg], new, keep)
    assert prej.tolist() == [[0, 1], [0, 3]]  # mode 2 dropped; a size above team_size
    c = pparse(pkg, RP)
    assert pe == 1 and c["id"].tolist() == [10, 11] and c["mode"].tolist() == [1] and c["seq"].tolist() == [1]
    keep[1, 1], keep[1, 0] = False, True  # the other share: only the party that stayed in group 0
    _R, RP, _rej, _prej, (_ne, pe) = restate_many_parties(pkg, [img], [pimg], new, keep)
    assert pe == 1 and pparse(pkg, RP)["id"].tolist() == [14, 15]


def test_no_party_images_is_restate_many(pkg):
    cfg = cfg_of(pkg, TWO, flags=WIDE)
    a = image(pkg, cfg, [1, 2, 3], [100, 1200, 300], [0, 0, 1], [5, 6, 7], [101, 103, 106])
    b = image(pkg, cfg, [4, 5], [1300, 10], [1, 0], [1, 9], [102, 104])
    for imgs in ([a], [a, b]):
        R, RP, rej, prej, (ne, pe) = restate_many_parties(pkg, imgs, [None] * len(imgs), cfg, active=0)
        R0, rej0, ne0 = restate_many(pkg, imgs, cfg, active_image=0)
        assert np.array_equal(R, R0) and np.array_equal(rej, rej0) and ne == ne0 and len(prej) == 0


def test_abi_mirror(pkg):
    abi = pkg.abi
    res, args = abi.PROTOTYPES["mm_import_regroup_many_parties"]
    assert res is C.c_int and len(args) == 12
    assert C.sizeof(abi.RecutParties) == 56
    hdr = open(os.path.join(ROOT, "include", "mm_engine.h")).read()
    assert "int mm_import_regroup_many_parties(" in hdr and "typedef struct mm_recut_parties" in hdr


# ================================================================================ GPU
def with_parties(pkg, cfg, engines, fresh, seed, n=400, owners=None):
    """Queue n parties of 2 .. team_size members on every engine (ratings drawn so that some have no group); with
    owners (per group of cfg), only the parties whose group the engine's rank owns, as routing would deliver them."""
    rng = np.random.default_rng(seed)
    tsz = np.array([cfg.modes[m].team_size for m in range(cfg.n_modes)])
    for k, e in enumerate(engines):
        e.set_option("party_capacity", 50_000)
        mode = rng.integers(0, cfg.n_modes, n).astype(np.uint8)
        mode = mode[tsz[mode] >= 2]
        sizes = np.array([rng.integers(2, tsz[m] + 1) for m in mode], np.uint8)
        ids, r, _m, _ts = fresh(int(sizes.sum()))
        ts = np.sort(rng.integers(0, 200, len(sizes))).astype(U32)
        if owners is not None:
            g = groups_of(cfg, party_rating(r, sizes))
            mine = (g >= 0) & (np.asarray(owners)[np.maximum(g, 0)] == k)
            moff = np.concatenate([[0], np.cumsum(sizes.astype(np.int64))])
            take = np.concatenate([np.zeros(0, np.int64)] + [np.arange(moff[j], moff[j + 1]) for j in np.flatnonzero(mine)])
            sizes, mode, ts, ids, r = sizes[mine], mode[mine], ts[mine], ids[take], r[take]
        e.enqueue_party(sizes, ids, r, mode, ts)


def export_all(engines):
    pimgs = [e.export_parties() for e in engines]  # released first, then the engine image: the same stop
    imgs = [e.export_state() for e in engines]
    for e in engines:
        e.close()
    return imgs, pimgs


def twin(pkg, cfg, imgs, pimgs, keep=None, act=None, cap=200_000):
    R, RP, want_rej, want_prej, (ne, pe) = restate_many_parties(pkg, imgs, pimgs, cfg, keep, act)
    a, b = pkg.Engine(cfg), pkg.Engine(cfg)
    a.set_option("party_capacity", cap)
    b.set_option("party_capacity", cap)
    rej, n_else, prej, p_else = a.import_regroup_many_parties(imgs, pimgs, keep=keep, active_image=act)
    assert np.array_equal(rej, want_rej) and n_else == ne
    assert np.array_equal(prej, want_prej) and p_else == pe
    b.import_state(R)
    b.merge_parties(RP, keep_seq=True)
    return a, b


def same_engines(pkg, a, b, cfg, now=300):
    from .test_party_handover import same_locate, same_next, snapshot
    ids = np.concatenate([a.pool_read()["id"][::37]] + [m[0] for m in a.party_read()["members"][::5]])
    assert snapshot(a, ids) == snapshot(b, ids)
    same_locate(a, b, ids, now)
    same_next(cfg, a, b, now)
    pr = a.party_read()
    if len(pr["members"]):
        gone = pr["members"][0][0][:1]
        assert a.remove(gone) == b.remove(gone)
    ea, eb = a.expire(now + 50, 250), b.expire(now + 50, 250)
    assert sorted(ea[0].tolist()) == sorted(eb[0].tolist())
    same_next(cfg, a, b, now + 60)
    assert np.array_equal(a.export_parties(), b.export_parties())
    same_as_image(pkg, a, b.export_state())  # sections 1-6 byte for byte, the active ids as a set


RATING_PAIRS = [n for n, v in PAIRS_MANY.items() if v[1][2] == v[2][2] == 1 and v[0] != "no_dedupe"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", RATING_PAIRS)
def test_twin_equivalence(pkg, name):
    kind, old, new, K = pair_configs(pkg, name)
    seed = zlib.crc32(name.encode())
    engines, fresh = sharded_sources(pkg, old, K, kind, seed)
    with_parties(pkg, old, engines, fresh, seed)
    imgs, pimgs = export_all(engines)
    keeps = [None, np.tile(np.arange(new.n_groups) % 2 == 0, (new.n_modes, 1))]
    for keep in keeps:
        a, b = twin(pkg, new, imgs, pimgs, keep, K // 2)
        with a, b:
            same_engines(pkg, a, b, new)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 2, 4])
def test_no_party_images_is_regroup_many_byte_for_byte(pkg, K):
    old, new = cfg_of(pkg, REF, modes=3), cfg_of(pkg, SPLIT, modes=3)
    engines, _fresh = sharded_sources(pkg, old, K, "hashed", 7 + K)
    imgs = [e.export_state() for e in engines]
    for e in engines:
        e.close()
    with pkg.Engine(new) as a, pkg.Engine(new) as b:
        a.set_option("party_capacity", 1000)
        ra = a.import_regroup_many_parties(imgs, [None] * K, active_image=0)
        rb = b.import_regroup_many(imgs, active_image=0)
        assert np.array_equal(ra[0], rb[0]) and ra[1] == rb[1] and len(ra[2]) == 0
        same_as_image(pkg, a, b.export_state())


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
def test_one_image_is_regroup_plus_keep_seq_merge(pkg, kind):
    from .test_regroup import FLAG
    old, new = cfg_of(pkg, REF, modes=3, flags=FLAG[kind]), cfg_of(pkg, SPLIT, modes=2, flags=FLAG[kind])
    engines, fresh = sharded_sources(pkg, old, 1, kind, 31)
    with_parties(pkg, old, engines, fresh, 31)
    imgs, pimgs = export_all(engines)
    with pkg.Engine(new) as a, pkg.Engine(new) as b:
        a.set_option("party_capacity", 50_000)
        b.set_option("party_capacity", 50_000)
        _r, _e, prej, _pe = a.import_regroup_many_parties(imgs, pimgs, active_image=0)
        b.import_regroup(imgs[0])
        code = b.merge_parties(pimgs[0], keep_seq=True)
        assert np.flatnonzero(code == 2).tolist() == prej[:, 1].tolist()
        same_engines(pkg, a, b, new)


@pytest.mark.gpu
def test_refusals_leave_the_engine_fresh(pkg):
    abi = pkg.abi
    old, new = cfg_of(pkg, REF, modes=3), cfg_of(pkg, SPLIT, modes=2)  # mode 2's parties are rejected
    engines, fresh = sharded_sources(pkg, old, 2, "hashed", 41)
    with_parties(pkg, old, engines, fresh, 41)
    stale = engines[0].export_parties()  # a party image from an earlier stop
    engines[0].enqueue_party(np.array([2], np.uint8), fresh(2)[0], np.array([100, 120], np.int32),
                             np.array([0], np.uint8), np.array([5], U32))
    imgs, pimgs = export_all(engines)
    _R, _RP, _rej, prej, _n = restate_many_parties(pkg, imgs, pimgs, new)
    assert len(prej) > 0
    members = sum(len(m) for m in (pkg.engine.read_party_image(p.tobytes())[1]["id"] for p in pimgs))
    kept_m = members - sum(
        int(pkg.engine.read_party_image(pimgs[k].tobytes())[1]["size"][j]) for k, j in prej.tolist())

    def refused(code, pimgs_, cap=200_000, cfg=new, still_fresh=True, **kw):
        with pkg.Engine(cfg) as t:
            if cap:
                t.set_option("party_capacity", cap)
            with pytest.raises(pkg.EngineError) as ei:
                t.import_regroup_many_parties(imgs, pimgs_, **kw)
            assert ei.value.status == code, (ei.value, code)
            assert t.pool_size() == 0 and t.active_size() == 0
            if cap:
                assert len(t.party_read()["size"]) == 0
            if still_fresh:
                rej, _ne = t.import_regroup_many(imgs)
                assert t.pool_size() > 0

    refused(abi.MM_E_ARG, [stale, pimgs[1]])  # not written at the same stop
    h, c = pkg.engine.read_party_image(pimgs[1].tobytes())
    solo = pkg.engine.read_image(np.array(imgs[0], copy=True))[1]["id"][0]
    ids = c["id"].copy()
    ids[0] = solo  # a member id colliding with a solo of another image
    bad = hand_image(pkg, c["size"], c["seq"], c["enq_ts"], c["mode"], ids, c["rating"], h.seq_next)
    bh = pkg.abi.ImageHeader.from_buffer_copy(pimgs[1][:C.sizeof(h)].tobytes())
    bad[:C.sizeof(h)] = np.frombuffer(bytes(bh), np.uint8)
    refused(abi.MM_E_ARG, [pimgs[0], bad])
    refused(abi.MM_E_ARG, pimgs, cfg=cfg_of(pkg, SPLIT, modes=3, order=ARRIVAL))  # an arrival-order target
    refused(abi.MM_E_STATE, pimgs, cap=0)  # no party capacity
    refused(abi.MM_E_CAP, pimgs, cap=kept_m - 1)  # one member short
    with pkg.Engine(new) as t:  # exactly enough room loads
        t.set_option("party_capacity", kept_m)
        t.import_regroup_many_parties(imgs, pimgs)
        assert sum(t.party_read()["size"].astype(int)) == kept_m
    # malformed party images
    def edited(k, **cols):
        h, c = pkg.engine.read_party_image(pimgs[k].tobytes())
        c = {**c, **cols}
        out = hand_image(pkg, c["size"], c["seq"], c["enq_ts"], c["mode"], c["id"], c["rating"], h.seq_next)
        bh = pkg.abi.ImageHeader.from_buffer_copy(pimgs[k][:C.sizeof(h)].tobytes())
        bh.total_bytes, bh.n_parts, bh.n_players = len(out), len(c["size"]), len(c["id"])
        out[:C.sizeof(bh)] = np.frombuffer(bytes(bh), np.uint8)
        return out
    magic = pimgs[1].copy()
    magic[0] ^= 1
    refused(abi.MM_E_ARG, [pimgs[0], magic])
    version = pimgs[1].copy()
    version[4] ^= 1
    refused(abi.MM_E_ARG, [pimgs[0], version])
    refused(abi.MM_E_ARG, [pimgs[0], pimgs[1][:-8]])  # a length that does not match the header
    sz = c["size"].copy()
    sz[0] = 1  # a party of one member
    refused(abi.MM_E_ARG, [pimgs[0], edited(1, size=sz)])
    sz = c["size"].copy()
    sz[0] += 1  # sizes that add up to more than the member count
    refused(abi.MM_E_ARG, [pimgs[0], edited(1, size=sz)])
    sq = c["seq"].copy()
    sq[0], sq[1] = sq[1], sq[0]  # numbers not increasing in age order
    refused(abi.MM_E_ARG, [pimgs[0], edited(1, seq=sq)])
    solo_seq = pkg.engine.read_image(np.array(imgs[1], copy=True))[1]["seq"]
    sq = c["seq"].copy()
    sq[0] = solo_seq[np.argmin((solo_seq - U32(h.seq_next)).astype(U32))]  # the oldest solo's: still in age order
    refused(abi.MM_E_ARG, [pimgs[0], edited(1, seq=sq)])
    refused(abi.MM_E_ARG, pimgs, cfg=cfg_of(pkg, SPLIT, modes=2, flags=NO_DEDUPE), still_fresh=False)  # no dedupe
    # the reject-cap dry run counts (the fixture always has rejected parties: mode 2 is dropped)
    with pkg.Engine(new) as t:
        t.set_option("party_capacity", 200_000)
        rp = abi.RecutParties()
        pptrs = (C.c_void_p * 2)(*[p.ctypes.data for p in pimgs])
        plens = (C.c_uint64 * 2)(*[len(p) for p in pimgs])
        rp.bufs, rp.n_bytes = C.cast(pptrs, C.c_void_p), C.cast(plens, C.c_void_p)
        ptrs = (C.c_void_p * 2)(*[b.ctypes.data for b in imgs])
        lens = (C.c_uint64 * 2)(*[len(b) for b in imgs])
        k, e = C.c_uint32(0), C.c_uint32(0)
        n = sum(pkg.engine.read_image(np.array(b, copy=True))[0].n_players for b in imgs)
        ri, rx = np.empty(n + 1, U32), np.empty(n + 1, U32)
        rc = t.lib.mm_import_regroup_many_parties(t.h, 2, ptrs, lens, None, 0xFFFFFFFF, n, ri.ctypes.data,
                                                  rx.ctypes.data, C.byref(k), C.byref(e), C.byref(rp))
        assert rc == abi.MM_E_CAP and rp.n_rejected == len(prej)
        assert t.pool_size() == 0 and len(t.party_read()["size"]) == 0


# ================================================================================ shard.recut with parties
def recut_party_engine(pkg, log):
    """Engine double with parties: holds an engine image and a party image; import_regroup_many_parties re-files with
    the restatement (MM_E_CAP past either capacity); merge_parties logs its keep_seq and takes the image back."""
    class RecutPartyEngine:
        def __init__(self, cfg, img=None, pimg=None):
            self.cfg, self.closed, self.party_capacity = cfg, False, 0
            self.img = make_image(pkg, cfg, [], [], [], [], [], [], 0) if img is None else img
            self.pimg = pimg

        def set_option(self, name, value):
            if name == "party_capacity":
                self.party_capacity = int(value)

        def export_parties(self):
            out, self.pimg = self.pimg, None
            return out.copy()

        def export_state(self):
            if self.pimg is not None and len(pparse(pkg, self.pimg)["size"]):
                raise pkg.EngineError(pkg.abi.MM_E_STATE, "mm_export")
            return self.img.copy()

        def merge_parties(self, buf, keep_seq=False):
            log.append(("merge", keep_seq))
            self.pimg = np.array(buf, np.uint8, copy=True)

        def import_regroup_many_parties(self, images, party_images, keep=None, active_image=None):
            log.append(("load", len(images)))
            R, RP, rej, prej, (ne, pe) = restate_many_parties(pkg, images, party_images, self.cfg, keep, active_image)
            if pkg.engine.read_image(R.copy())[0].n_players > self.cfg.capacity or \
                    len(pparse(pkg, RP)["id"]) > self.party_capacity:
                raise pkg.EngineError(pkg.abi.MM_E_CAP, "mm_import_regroup_many_parties")
            self.img, self.pimg = R, RP
            return rej, ne, prej, pe

        def close(self):
            self.closed = True

    return RecutPartyEngine


def cpu_party_shards(pkg, old, imgs):
    """A party image beside every engine image of cpu_shards: two-member parties of mode 1 in the groups the rank
    owns, numbered below the solos (older); rank 2's second party (rating 4800) has no group under MOVED."""
    out = []
    for r, img in enumerate(imgs):
        h = pkg.engine.read_image(np.array(img, copy=True))[0]
        base = 20_000 + 100 * r
        ratings = ([300, 320, 1200, 1210, 1900, 1990], [2100, 2120, 3000, 3010, 2600, 2700],
                   [3600, 3620, 4800, 4800, 4000, 4100])[r]  # in the groups the rank owns
        p = hand_image(pkg, [2, 2, 2], [40, 41, 42], [r, 3 + r, 9], [1, 1, 1], list(range(base, base + 6)), ratings,
                       h.seq_next)
        hh = pkg.abi.ImageHeader.from_buffer_copy(p[:C.sizeof(h)].tobytes())
        hh.config = old
        p[:C.sizeof(hh)] = np.frombuffer(bytes(hh), np.uint8)
        out.append(p)
    return out


@pytest.mark.parametrize("fail", [False, True])
def test_shard_recut_with_parties_swaps_or_rolls_back_everywhere(pkg, fail):
    import threading
    from .test_handover import copy_config
    from .test_recut import MOVED, cpu_shards, run_ranks, shard
    old, new = cfg_of(pkg, REF, modes=2), cfg_of(pkg, MOVED, modes=2)
    o_own, n_own = [0, 0, 1, 1, 1, 2, 2], [2, 2, 0, 1, 1]
    imgs = cpu_shards(pkg, old, o_own, 3)
    pimgs = cpu_party_shards(pkg, old, imgs)
    log = []
    Eng = recut_party_engine(pkg, log)
    olds = [Eng(old, im, p) for im, p in zip(imgs, pimgs)]
    for e in olds:
        e.party_capacity = 100
    comm = shard.LocalComm()
    pcap = {0: 100, 1: 1 if fail else 100, 2: 100}

    def rank_fn(r):
        threading.current_thread().rank = r
        return shard.recut(pkg, old, new, o_own, n_own, r, olds[r], comm, lambda c: Eng(copy_config(c)),
                           party_capacity=pcap[r])
    res = run_ranks(rank_fn, 3)
    if fail:
        for r in range(3):
            assert not res[r]["ok"] and res[r]["engine"] is olds[r] and not olds[r].closed
            assert np.array_equal(olds[r].img, imgs[r]) and np.array_equal(olds[r].pimg, pimgs[r])
            assert res[r]["stranded"] is None
        assert sorted(x for x in log if x[0] == "merge") == [("merge", True)] * 3
        return
    assert not any(x[0] == "merge" for x in log)
    _R, RP_all, _rej, prej_all, _n = restate_many_parties(pkg, imgs, pimgs, new)
    want_drop = []
    for k, j in prej_all.tolist():
        c = pparse(pkg, pimgs[k])
        off = np.concatenate([[0], np.cumsum(c["size"].astype(np.int64))])
        want_drop += c["id"][off[j]:off[j + 1]].tolist()
    assert sorted(np.concatenate([x["dropped_parties"] for x in res]).tolist()) == sorted(want_drop) and want_drop
    kept = []
    for r in range(3):
        assert res[r]["ok"] and olds[r].closed
        c = pparse(pkg, res[r]["engine"].pimg)
        kept += c["id"].tolist()
        off = np.concatenate([[0], np.cumsum(c["size"].astype(np.int64))])
        for j in range(len(c["size"])):  # every party loaded on the rank that owns its queue under MOVED
            R_ = int(np.floor_divide(int(c["rating"][off[j]:off[j + 1]].astype(np.int64).sum()), int(c["size"][j])))
            assert n_own[groups_of(new, [R_])[0]] == r
    assert sorted(kept) == sorted(pparse(pkg, RP_all)["id"].tolist())


def same_stop(engines):
    """Both images of every engine at one stop (the parties released, then the engine), the parties merged back."""
    imgs, pimgs = [], []
    for e in engines:
        pimgs.append(np.array(e.export_parties(), copy=True))
        imgs.append(np.array(e.export_state(), copy=True))
        e.merge_parties(pimgs[-1], keep_seq=True)
    return imgs, pimgs


def party_members(pkg, pimgs, which):
    out = []
    for k, j in np.asarray(which).reshape(-1, 2).tolist():
        c = pparse(pkg, pimgs[k])
        off = np.concatenate([[0], np.cumsum(c["size"].astype(np.int64))])
        out += c["id"][off[j]:off[j + 1]].tolist()
    return sorted(out)


@pytest.mark.gpu
def test_shard_recut_with_parties_ranks_match_one_engine(pkg):
    from .test_party_handover import RULES
    from .test_recut import MOVED, recut_on_one_gpu, shard
    from .test_widen import rules_of
    old = cfg_of(pkg, REF, modes=3, capacity=400_000)
    new = cfg_of(pkg, MOVED, modes=3, capacity=400_000)
    o_own = [0, 0, 1, 1, 2, 3, 3]
    engines, fresh = sharded_sources(pkg, old, 4, "hashed", 5, owners=o_own)
    with_parties(pkg, old, engines, fresh, 5, n=800, owners=o_own)
    imgs, pimgs = same_stop(engines)
    n_own = shard.balanced_owners(np.ones(new.n_groups), 4)
    res = recut_on_one_gpu(pkg, old, new, o_own, n_own, engines, pkg.Engine)
    assert all(x["ok"] for x in res)
    R, RP, rej, prej, _n = restate_many_parties(pkg, imgs, pimgs, new, None, 0)
    assert len(prej) > 0
    assert sorted(np.concatenate([x["dropped_parties"] for x in res]).tolist()) == party_members(pkg, pimgs, prej)
    with pkg.Engine(new) as one:
        one.set_option("party_capacity", 50_000)
        one.import_state(R)
        one.merge_parties(RP, keep_seq=True)
        assert sum(len(x["engine"].party_read()["size"]) for x in res) == len(one.party_read()["size"])
        now = 400
        for t in range(2):
            rules = rules_of(new, RULES(new))
            per = [x["engine"].party_match(now + t, rules) for x in res]
            ref = one.party_match(now + t, rules)
            assert sum(len(p[0]) for p in per) == len(ref[0])
            assert sorted(np.concatenate([p[1] for p in per]).tolist()) == sorted(ref[1].tolist())
            ticks = [x["engine"].tick(now + t) for x in res]
            lob1, mem1, _s, _st = one.tick(now + t)
            lob, mem = shard.merge_results(new, [(a[0], a[1]) for a in ticks])
            assert np.array_equal(mem, mem1) and np.array_equal(lob, lob1), t
    for x in res:
        x["engine"].close()


@pytest.mark.gpu
def test_shard_recut_with_parties_rolls_back_when_one_rank_has_no_room(pkg):
    import threading
    from .test_party_handover import snapshot
    from .test_recut import run_ranks, shard
    old, new = cfg_of(pkg, REF, modes=3), cfg_of(pkg, SPLIT, modes=3)
    o_own = [0, 0, 1, 1, 1, 2, 2]
    engines, fresh = sharded_sources(pkg, old, 3, "hashed", 9, owners=o_own)
    with_parties(pkg, old, engines, fresh, 9, owners=o_own)
    ids = [np.concatenate([e.pool_read()["id"]] + [m[0] for m in e.party_read()["members"]]) for e in engines]
    before = [snapshot(e, i) for e, i in zip(engines, ids)]
    n_own = [0, 0, 0, 1, 1, 1, 2, 2]
    comm = shard.LocalComm()

    def rank_fn(r):  # rank 1's new engine has room for two party members
        return shard.recut(pkg, old, new, o_own, n_own, r, engines[r], comm, party_capacity=2 if r == 1 else None)
    res = run_ranks(rank_fn, 3)
    for r in range(3):
        assert not res[r]["ok"] and res[r]["engine"] is engines[r] and res[r]["stranded"] is None
        assert snapshot(engines[r], ids[r]) == before[r]
        engines[r].close()
    del threading


@pytest.mark.gpu
def test_config3_ten_million_and_200k_parties_into_quantile_groups(pkg):
    from .test_recut import recut_on_one_gpu, shard
    from .test_tile_geometry import DENSE, MODES8
    n, K, P = 10_000_000, 4, 200_000
    old = pkg.synth.make_config(n_groups=32, modes=MODES8[3:4], order=1, capacity=n // 2, active_capacity=2 * n,
                                flags=DENSE)
    _, rating, _, _ = pkg.synth.gen_pool(1, n, bell=True)
    g = groups_of(old, rating)
    o_own = shard.balanced_owners(np.bincount(g, minlength=32), K)
    q = np.quantile(rating, np.linspace(0, 1, 33)[1:-1]).astype(np.int64)
    cuts = np.unique(np.clip(q, 1, 4999))
    groups = tuple(zip(np.r_[0, cuts[:-1] + 1].tolist(), cuts.tolist())) + ((int(cuts[-1]) + 1, 5000),)
    new = pkg.synth.make_config(groups=groups, modes=MODES8[3:4], order=1, capacity=n // 2, active_capacity=2 * n,
                                flags=DENSE)
    rng = np.random.default_rng(12)
    sizes = rng.integers(2, 6, P).astype(np.uint8)
    M = int(sizes.sum())
    pids = np.arange(n, n + M, dtype=np.uint64)
    prat = rng.integers(0, 5001, M).astype(np.int32)
    pto = o_own[groups_of(old, party_rating(prat, sizes))]
    moff = np.concatenate([[0], np.cumsum(sizes.astype(np.int64))])
    ids = np.arange(n, dtype=U32)
    to = o_own[g]
    engines = [pkg.Engine(old) for _ in range(K)]
    for k, e in enumerate(engines):
        s = to == k
        key = pkg.Engine.pack_key(rating[s], np.zeros(int(s.sum()), np.uint8))
        assert (e.enqueue_packed(ids[s], key, (np.flatnonzero(s) % 977).astype(U32)) == 1).all()
        e.tick_packed(1000)
        e.set_option("party_capacity", 1_000_000)
        mine = np.flatnonzero(pto == k)
        take = np.concatenate([np.arange(moff[j], moff[j + 1]) for j in mine])
        code = e.enqueue_party(sizes[mine], pids[take], prat[take], np.zeros(len(mine), np.uint8),
                               (mine % 977).astype(U32))
        assert (code == 1).all()
    imgs, pimgs = same_stop(engines)
    n_own = shard.balanced_owners(np.bincount(groups_of(new, rating), minlength=new.n_groups), K)
    res = recut_on_one_gpu(pkg, old, new, o_own, n_own, engines, pkg.Engine)
    assert all(x["ok"] for x in res)
    assert sum(len(x["engine"].party_read()["size"]) for x in res) == P
    send = shard.recut_sends(old, new, o_own, n_own, K)
    for r in (0, K - 1):  # two ranks against the restatement of what they loaded
        mine = [k for k in range(K) if k == r or send[k, r]]
        keep = np.broadcast_to(n_own == r, (new.n_modes, new.n_groups))
        R, RP, _rej, _prej, _n = restate_many_parties(pkg, [imgs[k] for k in mine], [pimgs[k] for k in mine], new,
                                                      keep, mine.index(r))
        e = res[r]["engine"]
        assert np.array_equal(e.export_parties(), RP)
        same_as_image(pkg, e, R)
    for x in res:
        x["engine"].close()
