"""Re-cut of a sharded deployment (mm_import_regroup_many, shard.recut): the images of K old ranks re-filed under a new
rating-group table into a fresh engine that keeps the queues it owns.

CPU: the numpy restatement restate_many(images, cfg, keep, active_image) -> (R, rejected, n_elsewhere) on hand-built
images (K = 1 equals test_regroup's restatement, interleaving by stamp, a falling stamp run where the running maximum
decides, equal stamps, the renumbering, skip versus reject, the active section, every refusal), and shard.recut over
LocalComm threads with an engine double that writes real images (the send matrix, a swap, a rollback).
GPU: the engine after mm_import_regroup_many against a fresh engine that mm_import'ed R, through mixed steps; K = 1
against mm_import_regroup; shard.recut over K engines on one GPU against one engine, tick by tick, and its rollback;
every refusal; config3 at 10 M players.
"""
import ctypes as C
import importlib
import threading
import zlib

import numpy as np
import pytest

from .test_handover import copy_config, same_state
from .test_regroup import (ARRIVAL, FLAG, MERGED, MOVED, NO_DEDUPE, RATING, REF, SPLIT, TWO, cfg_of, groups_of,
                           kat_image, make_image, mixed_steps, r_ids, regroup, same_as_image)
from .test_requeue import layout_parts
from .test_tick_forms_and_schedules import check_tick
from .test_tile_geometry import DENSE, MODES8, WIDE

U32 = np.uint32
shard = importlib.import_module("microservice-matchmaking_b200.shard")


# ================================================================================ the restatement
def restate_many(pkg, images, cfg, keep=None, active_image=None):
    """-> (R, rejected int64 [n, 2] (image, index) ascending, n_elsewhere): the header's restated image.  Raises
    ValueError for what the call refuses with MM_E_ARG on well-formed images."""
    K = len(images)
    if not 1 <= K <= 64:
        raise ValueError("n_images")
    if active_image is not None and not 0 <= active_image < K:
        raise ValueError("active_image")
    parsed = [pkg.engine.read_image(np.array(img, np.uint8, copy=True)) for img in images]
    c0 = parsed[0][0].config
    for h, _s in parsed[1:]:
        same = (h.config.n_groups, h.config.default_group, h.config.n_modes, h.config.order_mode, h.config.flags) == \
            (c0.n_groups, c0.default_group, c0.n_modes, c0.order_mode, c0.flags)
        same = same and all((h.config.group_lo[g], h.config.group_hi[g]) == (c0.group_lo[g], c0.group_hi[g])
                            for g in range(c0.n_groups))
        same = same and all((h.config.modes[m].teams, h.config.modes[m].team_size) ==
                            (c0.modes[m].teams, c0.modes[m].team_size) for m in range(c0.n_modes))
        if not same:
            raise ValueError("configs differ")
    sel = np.ones(cfg.n_modes * cfg.n_groups, bool) if keep is None else np.asarray(keep, bool).reshape(-1)
    cols = {k: [] for k in ("part", "rm", "img", "age", "id", "rating", "mode", "ts", "seq")}
    rej, n_else = [], 0
    for k, (h, s) in enumerate(parsed):
        mode = s["mode"].astype(np.int64)
        g = np.full(len(mode), -1, np.int64)
        has = mode < cfg.n_modes
        g[has] = groups_of(cfg, s["rating"][has])
        ok = g >= 0
        rej += [(k, int(i)) for i in np.flatnonzero(~ok)]
        kept = ok & sel[np.where(ok, mode * cfg.n_groups + g, 0)]
        n_else += int((ok & ~kept).sum())
        idx = np.flatnonzero(kept)
        part = layout_parts(cfg, s["rating"][idx], s["mode"][idx]) if len(idx) else np.zeros(0, np.int64)
        age = (s["seq"][idx] - U32(h.seq_next)).astype(U32).astype(np.int64)
        o = np.lexsort((age, part))
        idx, part, age = idx[o], part[o], age[o]
        ts = s["enq_ts"][idx].astype(np.int64)
        rm = ts.copy()
        for p in np.unique(part):
            sl = part == p
            rm[sl] = np.maximum.accumulate(ts[sl])
        for name, v in (("part", part), ("rm", rm), ("img", np.full(len(idx), k)), ("age", age),
                        ("id", s["id"][idx].astype(np.uint64)), ("rating", s["rating"][idx]),
                        ("mode", s["mode"][idx]), ("ts", s["enq_ts"][idx]), ("seq", s["seq"][idx])):
            cols[name].append(v)
    c = {k: np.concatenate(v) for k, v in cols.items()}
    ids = c["id"]
    act = parsed[active_image][1]["active"].astype(np.uint64) if active_image is not None else np.zeros(0, np.uint64)
    dedupe = not (cfg.flags & NO_DEDUPE)
    if dedupe:
        every = np.concatenate([np.concatenate([s["id"].astype(np.uint64) for _h, s in parsed]), act])
        if len(np.unique(every)) != len(every):
            raise ValueError("repeated id")
    if K == 1:
        seq, seq_next = c["seq"], parsed[0][0].seq_next
    else:
        g_order = np.lexsort((c["part"], c["age"], c["img"], c["rm"]))
        seq = np.empty(len(ids), np.int64)
        seq[g_order] = np.arange(len(ids))
        seq_next = len(ids)
    # inside a partition: (running max, image, age); make_image files by partition and then by age under seq_next,
    # so the numbers of K > 1 must follow that order, and those of K = 1 already do
    o = np.lexsort((c["age"], c["img"], c["rm"], c["part"]))
    R = make_image(pkg, cfg, ids[o], c["rating"][o], c["mode"][o], c["ts"][o], np.asarray(seq)[o], act, seq_next,
                   parsed[0][0].id_bytes)
    if K > 1:  # the numbering must agree with the merged order inside every partition
        _h, sr = pkg.engine.read_image(R.copy())
        assert np.array_equal(sr["id"], ids[o][np.lexsort((np.asarray(seq)[o], c["part"][o]))])
    return R, np.array(rej, np.int64).reshape(-1, 2), n_else


def image(pkg, cfg, ids, rating, mode, ts, seq, seq_next=100, active=()):
    return make_image(pkg, cfg, np.asarray(ids, np.uint64), np.asarray(rating, np.int32), np.asarray(mode, np.uint8),
                      np.asarray(ts, U32), np.asarray(seq, U32), list(active), seq_next)


def queue_ids(pkg, R):
    return r_ids(pkg, R)[2]


# ================================================================================ CPU: hand-built KATs
def test_one_image_equals_the_regroup_restatement(pkg):
    old = cfg_of(pkg, TWO, flags=WIDE)
    for new in (cfg_of(pkg, ((0, 499), (500, 999), (1000, 1999)), order=ARRIVAL), cfg_of(pkg, ((0, 1999),), flags=WIDE),
                cfg_of(pkg, ((0, 999),), modes=1)):
        img = kat_image(pkg, old, seq_next=5)  # non-monotone stamps (1000 + seq % 97) across the sequence wrap
        R1, rej1 = regroup(pkg, img, new)
        R, rej, n_else = restate_many(pkg, [img], new, active_image=0)
        assert np.array_equal(R, R1) and n_else == 0
        assert rej[:, 0].tolist() == [0] * len(rej1) and rej[:, 1].tolist() == rej1.tolist()


def test_two_images_interleave_by_stamp(pkg):
    cfg = cfg_of(pkg, TWO, flags=WIDE)
    a = image(pkg, cfg, [1, 2, 3], [100, 200, 300], [0, 0, 0], [10, 20, 30], [90, 91, 92], 100, active=[50])
    b = image(pkg, cfg, [11, 12, 13], [150, 250, 350], [0, 0, 0], [15, 16, 40], [7, 8, 9], 10, active=[60])
    R, rej, _ = restate_many(pkg, [a, b], cfg, active_image=1)
    h, s, parts = r_ids(pkg, R)
    assert len(rej) == 0 and parts[0] == [1, 11, 12, 2, 3, 13]
    assert s["seq"][:6].tolist() == [0, 1, 2, 3, 4, 5] and h.seq_next == 6
    assert s["active"].tolist() == [60]


def test_a_falling_stamp_run_is_keyed_by_its_running_maximum(pkg):
    cfg = cfg_of(pkg, TWO, flags=WIDE)
    # image 0 in age order has stamps 50, 10, 60: keys 50, 50, 60; image 1's stamp 30 goes before all three
    a = image(pkg, cfg, [1, 2, 3], [100, 200, 300], [0, 0, 0], [50, 10, 60], [1, 2, 3], 4)
    b = image(pkg, cfg, [11, 12], [150, 250], [0, 0], [30, 55], [1, 2], 3)
    assert queue_ids(pkg, restate_many(pkg, [a, b], cfg)[0])[0] == [11, 1, 2, 12, 3]


def test_equal_stamps_go_to_the_lower_image(pkg):
    cfg = cfg_of(pkg, TWO, flags=WIDE)
    a = image(pkg, cfg, [1, 2], [100, 200], [0, 0], [7, 7], [1, 2], 3)
    b = image(pkg, cfg, [11, 12], [150, 250], [0, 0], [7, 7], [1, 2], 3)
    assert queue_ids(pkg, restate_many(pkg, [b, a], cfg)[0])[0] == [11, 12, 1, 2]
    assert queue_ids(pkg, restate_many(pkg, [a, b], cfg)[0])[0] == [1, 2, 11, 12]


def test_renumbering_is_one_order_across_partitions(pkg):
    cfg = cfg_of(pkg, TWO, flags=WIDE)
    a = image(pkg, cfg, [1, 2, 3], [100, 1100, 200], [0, 0, 1], [5, 1, 9], [1, 2, 3], 4)
    b = image(pkg, cfg, [11, 12], [1500, 300], [0, 1], [3, 9], [1, 2], 3)
    h, s, parts = r_ids(pkg, restate_many(pkg, [a, b], cfg)[0])
    # keys (running max, image, age): 1 (5,0,1) 2 (1,0,2) 3 (9,0,3) 11 (3,1,1) 12 (9,1,2)
    num = dict(zip(s["id"].tolist(), s["seq"].tolist()))
    assert num == {2: 0, 11: 1, 1: 2, 3: 3, 12: 4} and h.seq_next == 5
    assert parts == [[1], [2, 11], [3, 12], []]


def test_skip_versus_reject(pkg):
    old = cfg_of(pkg, TWO, flags=WIDE)
    new = cfg_of(pkg, ((0, 499), (500, 1499)), flags=WIDE)  # 1500 .. 1999: no queue
    img = kat_image(pkg, old)
    keep = np.array([[True, False], [False, True]])  # mode 0: group 0; mode 1: group 1
    R, rej, n_else = restate_many(pkg, [img], new, keep=keep)
    _h, s0 = pkg.engine.read_image(img.copy())
    assert rej[:, 1].tolist() == np.flatnonzero(s0["rating"] >= 1500).tolist()
    g = groups_of(new, s0["rating"])
    skipped = (g >= 0) & ~keep[s0["mode"], np.maximum(g, 0)]
    assert n_else == int(skipped.sum()) > 0
    h, s, parts = r_ids(pkg, R)
    assert sorted(s["id"].tolist()) == sorted(s0["id"][(g >= 0) & ~skipped].tolist()) and h.n_active == 0


def test_the_active_section_is_the_chosen_images(pkg):
    cfg = cfg_of(pkg, TWO, flags=WIDE)
    a = image(pkg, cfg, [1], [100], [0], [1], [1], 2, active=[50, 51])
    b = image(pkg, cfg, [2], [100], [0], [1], [1], 2, active=[60])
    for act, want in ((0, [50, 51]), (1, [60]), (None, [])):
        assert sorted(r_ids(pkg, restate_many(pkg, [a, b], cfg, active_image=act)[0])[1]["active"].tolist()) == want


def test_restatement_refusals(pkg):
    cfg = cfg_of(pkg, TWO, flags=WIDE)
    a = image(pkg, cfg, [1], [100], [0], [1], [1], 2, active=[50])
    for images, kw in (([], {}), ([a] * 65, {}), ([a], {"active_image": 1}),
                       ([a, image(pkg, cfg_of(pkg, MERGED), [2], [100], [0], [1], [1], 2)], {}),
                       ([a, image(pkg, cfg, [1], [100], [0], [1], [1], 2)], {}),
                       ([a, image(pkg, cfg, [50], [100], [0], [1], [1], 2)], {"active_image": 0})):
        with pytest.raises(ValueError):
            restate_many(pkg, images, cfg, **kw)
    # the active section of an image that is not taken is not part of the load
    restate_many(pkg, [a, image(pkg, cfg, [50], [100], [0], [1], [1], 2)], cfg, active_image=1)


# ================================================================================ CPU: shard.recut over LocalComm
def recut_engine(pkg, log):
    """Engine double: holds an image; import_regroup_many re-files with the restatement, MM_E_CAP past capacity."""
    class RecutEngine:
        def __init__(self, cfg, img=None):
            self.cfg, self.img, self.closed = cfg, img, False
            if img is None:
                self.img = make_image(pkg, cfg, [], [], [], [], [], [], 0)

        def export_state(self):
            return self.img.copy()

        def import_regroup_many(self, images, keep=None, active_image=None):
            log.append(len(images))
            R, rej, n_else = restate_many(pkg, images, self.cfg, keep, active_image)
            if pkg.engine.read_image(R.copy())[0].n_players > self.cfg.capacity:
                raise pkg.EngineError(pkg.abi.MM_E_CAP, "mm_import_regroup_many")
            self.img = R
            return rej, n_else

        def close(self):
            self.closed = True

    return RecutEngine


def run_ranks(fn, world):
    out, errs = [None] * world, []

    def one(r):
        try:
            out[r] = fn(r)
        except Exception as e:  # noqa: BLE001
            errs.append(e)
    th = [threading.Thread(target=one, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join(300)
    assert not errs, errs
    return out


def cpu_shards(pkg, old, owners, world, n=400, seed=3):
    """world images under `old`: the players of the groups each rank owns, disjoint ids, rising stamps."""
    rng = np.random.default_rng(seed)
    rating = rng.integers(0, 5001, n).astype(np.int32)
    mode = rng.integers(0, old.n_modes, n).astype(np.uint8)
    g = groups_of(old, rating)
    rank = np.asarray(owners)[np.maximum(g, 0)]
    imgs = []
    for r in range(world):
        s = np.flatnonzero((rank == r) & (g >= 0))
        imgs.append(make_image(pkg, old, 1000 + s, rating[s], mode[s], s // 3, 50 + np.arange(len(s)), [900 + r],
                               50 + len(s)))
    return imgs


def test_send_matrix(pkg):
    old, new = cfg_of(pkg, REF, modes=2), cfg_of(pkg, MOVED, modes=2)
    # old: REF groups 0-1 on rank 0, 2-4 on rank 1, 5-6 on rank 2; new: MOVED groups 0-1 rank 2, 2 rank 0, 3-4 rank 1
    send = shard.recut_sends(old, new, [0, 0, 1, 1, 1, 2, 2], [2, 2, 0, 1, 1], 3)
    # rank 0 holds 0 .. 1999: new groups 0, 1 -> rank 2; rank 1 holds 2000 .. 3499: new 2 (rank 0), 3 (rank 1);
    # rank 2 holds 3500 .. 5000: new 4 (rank 1), 4500 .. 5000 dropped
    assert send.tolist() == [[False, False, True], [True, False, False], [False, True, False]]


@pytest.mark.parametrize("fail", [False, True])
def test_recut_swaps_or_rolls_back_everywhere(pkg, fail):
    old, new = cfg_of(pkg, REF, modes=2), cfg_of(pkg, MOVED, modes=2)
    o_own, n_own = [0, 0, 1, 1, 1, 2, 2], [2, 2, 0, 1, 1]
    imgs = cpu_shards(pkg, old, o_own, 3)
    log = []
    Eng = recut_engine(pkg, log)
    olds = [Eng(old, im) for im in imgs]
    comm = shard.LocalComm()
    cap = {0: 10**6, 1: 10**6, 2: 10**6}
    if fail:
        cap[1] = 1
    make = lambda c: Eng(copy_config(c, capacity=cap[threading.current_thread().rank]))  # noqa: E731

    def rank_fn(r):
        threading.current_thread().rank = r
        return shard.recut(pkg, old, new, o_own, n_own, r, olds[r], comm, make)
    res = run_ranks(rank_fn, 3)
    assert sorted(log) == [2, 2, 2]  # every rank loads its own image and the one old rank that feeds it
    if fail:
        for r in range(3):
            assert not res[r]["ok"] and res[r]["engine"] is olds[r] and not olds[r].closed
            assert np.array_equal(olds[r].img, imgs[r])
        return
    R_all, rej_all, _ = restate_many(pkg, imgs, new)
    whole = {p: ids for p, ids in enumerate(queue_ids(pkg, R_all))}
    for r in range(3):
        assert res[r]["ok"] and olds[r].closed and res[r]["engine"] is not olds[r]
        h, s, parts = r_ids(pkg, res[r]["engine"].img)
        assert s["active"].tolist() == [900 + r]
        mine = n_own
        want_drop = pkg.engine.read_image(imgs[r].copy())[1]["id"][rej_all[rej_all[:, 0] == r, 1]]
        assert np.array_equal(np.sort(res[r]["dropped"]), np.sort(want_drop))
        qp = layout_parts(new, s["rating"], s["mode"]) if h.n_players else []
        for p in np.unique(qp):  # each kept queue holds what one engine holding everything holds, in the same order
            assert parts[p] == whole[p]
        assert all(mine[g] == r for g in groups_of(new, s["rating"]))
        assert res[r]["bytes_sent"] > 0
    assert sum(r_ids(pkg, x["engine"].img)[0].n_players for x in res) == sum(len(v) for v in whole.values())


# ================================================================================ GPU helpers
def sharded_sources(pkg, cfg, K, kind, seed, owners=None):
    """K engines under cfg, each holding the groups `owners` gives it (default contiguous), after a mixed schedule:
    enqueue, tick, enqueue, remove, take, expire.  Ids are disjoint across the engines."""
    rng = np.random.default_rng(seed)
    owners = shard.owner_of_group(np.arange(cfg.n_groups), cfg.n_groups, K) if owners is None else owners
    engines = [pkg.Engine(cfg) for _ in range(K)]
    nxt = [0]

    def fresh(n):
        x = np.arange(nxt[0], nxt[0] + n, dtype=np.uint64)
        nxt[0] += n
        ids = x if kind == "dense" else pkg.synth.mix64(x + np.uint64(5 << 40))
        return (ids, rng.integers(0, 5001, n).astype(np.int32), rng.integers(0, cfg.n_modes, n).astype(np.uint8),
                rng.integers(0, 90, n).astype(U32))

    def deliver(ids, r, m, ts):
        g = groups_of(cfg, r)
        to = np.asarray(owners)[np.maximum(g, 0)]
        for k, e in enumerate(engines):
            s = (to == k) & (g >= 0)
            e.enqueue(ids[s], r[s], m[s], ts[s])

    deliver(*fresh(12_000 * K))
    for e in engines:
        e.tick(100)
    ids, r, m, ts = fresh(8_000 * K)
    deliver(ids, r, m, ts + 100)
    for e in engines:
        if kind != "no_dedupe":
            q = e.pool_read()["id"]
            e.remove(q[:150])
            e.take(q[150:280])
        e.expire(150, 120)
    return engines, fresh


PAIRS_MANY = {  # name: (kind, (old groups, modes, order, flags), (new groups, modes, order, flags), K)
    "split": ("hashed", (REF, 3, RATING, 0), (SPLIT, 3, RATING, 0), 2),
    "merge_across_ranks": ("dense", (REF, 3, RATING, WIDE), (MERGED, 3, RATING, WIDE), 4),
    "moved_dropped": ("dense", (REF, 3, RATING, 0), (MOVED, 3, RATING, 0), 8),
    "mode_added": ("no_dedupe", (REF, 3, ARRIVAL, 0), (REF, 4, ARRIVAL, 0), 2),
    "mode_dropped": ("hashed", (REF, 3, RATING, 0), (SPLIT, 2, RATING, 0), 4),
    "arrival_to_rating": ("hashed", (REF, 3, ARRIVAL, 0), (MERGED, 3, RATING, 0), 4),
    "rating_to_arrival": ("dense", (REF, 3, RATING, 0), (MOVED, 3, ARRIVAL, 0), 2),
    "wide_on": ("hashed", (REF, 3, RATING, 0), (MOVED, 3, RATING, WIDE), 8),
    "wide_off": ("dense", (REF, 3, RATING, WIDE), (SPLIT, 3, RATING, 0), 4),
}


def pair_configs(pkg, name, capacity=400_000):
    kind, old, new, K = PAIRS_MANY[name]
    mk = lambda g, m, o, f: cfg_of(pkg, g, modes=m, order=o, flags=f | FLAG[kind], capacity=capacity)  # noqa: E731
    return kind, mk(*old), mk(*new), K


# ================================================================================ GPU: twin equivalence
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PAIRS_MANY))
def test_regroup_many_equals_import_of_the_restated_image(pkg, oracle, name):
    kind, old, new, K = pair_configs(pkg, name)
    engines, fresh = sharded_sources(pkg, old, K, kind, zlib.crc32(name.encode()))
    images = [e.export_state() for e in engines]
    for e in engines:
        e.close()
    act = K // 2
    keeps = [None]
    if name in ("split", "moved_dropped"):  # a rank's share: every other group
        keeps.append(np.tile(np.arange(new.n_groups) % 2 == 0, (new.n_modes, 1)))
    for keep in keeps:
        R, want_rej, want_else = restate_many(pkg, images, new, keep, act)
        with pkg.Engine(new) as a, pkg.Engine(new) as b:
            rej, n_else = a.import_regroup_many(images, keep=keep, active_image=act)
            assert np.array_equal(rej, want_rej) and n_else == want_else
            b.import_state(R)
            same_as_image(pkg, a, R)
            dedupe = kind != "no_dedupe"
            sample = np.concatenate([a.pool_read()["id"][::41],
                                     pkg.engine.read_image(np.array(images[act], copy=True))[1]["active"][::7]
                                     .astype(np.uint64)])
            same_state(a, b, 200, sample, dedupe)
            if keep is None:
                pr = a.pool_read()
                if name in ("split", "arrival_to_rating", "rating_to_arrival"):
                    with pkg.Engine(new) as c:
                        c.import_regroup_many(images, active_image=act)
                        sr = pkg.engine.read_image(np.array(R, copy=True))[1]
                        seq_of = dict(zip(sr["id"].tolist(), sr["seq"].tolist()))
                        ref = oracle.run_literal(new, pr["id"], pr["rating"], pr["mode"])
                        check_tick(ref, np.array([seq_of[p] for p in pr["id"].tolist()], U32), *c.tick(10))
            mixed_steps(pkg, a, b, fresh, kind, new.order_mode, np.random.default_rng(4), steps=2)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
def test_one_image_is_mm_import_regroup(pkg, kind):
    old = cfg_of(pkg, REF, modes=3, flags=FLAG[kind])
    new = cfg_of(pkg, MOVED, modes=2, order=ARRIVAL, flags=FLAG[kind])
    engines, _fresh = sharded_sources(pkg, old, 1, kind, 21)
    img = engines[0].export_state()
    engines[0].close()
    with pkg.Engine(new) as a, pkg.Engine(new) as b:
        rej, n_else = a.import_regroup_many([img], active_image=0)
        want = b.import_regroup(img)
        assert np.array_equal(rej[:, 1], want) and (rej[:, 0] == 0).all() and n_else == 0
        same_as_image(pkg, a, b.export_state())


# ================================================================================ GPU: shard.recut on one GPU
def recut_on_one_gpu(pkg, old, new, o_own, n_own, engines, make):
    comm = shard.LocalComm()
    return run_ranks(lambda r: shard.recut(pkg, old, new, o_own, n_own, r, engines[r], comm, make), len(engines))


@pytest.mark.gpu
def test_recut_ranks_tick_as_one_engine(pkg):
    kind = "hashed"
    old = cfg_of(pkg, REF, modes=3, capacity=400_000)
    new = cfg_of(pkg, MOVED, modes=3, capacity=400_000)
    o_own = [0, 0, 1, 1, 2, 3, 3]
    engines, fresh = sharded_sources(pkg, old, 4, kind, 5, owners=o_own)
    images = [e.export_state() for e in engines]
    n_own = shard.balanced_owners(np.ones(new.n_groups), 4)
    res = recut_on_one_gpu(pkg, old, new, o_own, n_own, engines, pkg.Engine)
    assert all(x["ok"] for x in res)
    R, rej, _ = restate_many(pkg, images, new, None, 0)
    _h, s_img = pkg.engine.read_image(np.array(images[0], copy=True))
    with pkg.Engine(new) as one:
        one.import_state(R)
        drop_all = np.concatenate([pkg.engine.read_image(np.array(images[k], copy=True))[1]["id"][rej[rej[:, 0] == k, 1]]
                                   for k in range(4)])
        assert np.array_equal(np.sort(np.concatenate([x["dropped"] for x in res])), np.sort(drop_all))
        for t in range(3):
            ids, r, m, ts = fresh(6000)
            to = shard.route(new, r, 4, owners=n_own)
            acc_one = one.enqueue(ids, r, m, ts + 200)
            for k, x in enumerate(res):
                s = to == k
                assert np.array_equal(x["engine"].enqueue(ids[s], r[s], m[s], ts[s] + 200), acc_one[s])
            per = []
            for x in res:
                lob, mem, _seq, _st = x["engine"].tick(300 + t)
                per.append((lob, mem))
            lob1, mem1, _seq1, _st1 = one.tick(300 + t)
            lob, mem = shard.merge_results(new, per)
            assert np.array_equal(mem, mem1) and np.array_equal(lob, lob1), t
    for x in res:
        x["engine"].close()


@pytest.mark.gpu
def test_recut_rolls_back_when_one_rank_is_too_small(pkg):
    old = cfg_of(pkg, REF, modes=2, capacity=400_000)
    new = cfg_of(pkg, SPLIT, modes=2, capacity=400_000)
    o_own = [0, 0, 1, 1, 1, 2, 2]
    engines, _fresh = sharded_sources(pkg, old, 3, "hashed", 9, owners=o_own)
    before = [np.array(e.export_state(), copy=True) for e in engines]
    n_own = [0, 0, 0, 1, 1, 1, 2, 2]

    def make(c):
        small = threading.current_thread().name.endswith("1)")
        return pkg.Engine(copy_config(c, capacity=1000) if small else c)
    comm = shard.LocalComm()

    def rank_fn(r):
        threading.current_thread().name = f"rank({r})"
        return shard.recut(pkg, old, new, o_own, n_own, r, engines[r], comm, make)
    res = run_ranks(rank_fn, 3)
    for r in range(3):
        assert not res[r]["ok"] and res[r]["engine"] is engines[r]
        same_as_image(pkg, engines[r], before[r])  # the active section is a set: its order is not fixed
        engines[r].close()


# ================================================================================ GPU: refusals
@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True])
def test_refusals_leave_the_engine_fresh(pkg, dense):
    abi = pkg.abi
    kind = "dense" if dense else "hashed"
    old = cfg_of(pkg, REF, modes=2, flags=FLAG[kind], capacity=60_000)
    new = cfg_of(pkg, MOVED, modes=2, order=ARRIVAL, flags=FLAG[kind], capacity=60_000)
    engines, _fresh = sharded_sources(pkg, old, 2, kind, 13)
    images = [e.export_state() for e in engines]
    qimg = engines[0].export_queues(np.ones(old.n_modes * old.n_groups, bool))
    for e in engines:
        e.close()
    R, want, _ = restate_many(pkg, images, new, None, 0)
    kept = pkg.engine.read_image(np.array(R, copy=True))[0].n_players
    assert len(want) > 100

    def refused(cfg, imgs, status, prep=None, **kw):
        with pkg.Engine(cfg) as t:
            if prep:
                prep(t)
            with pytest.raises(pkg.EngineError) as ei:
                t.import_regroup_many(imgs, **kw)
            assert ei.value.status == status, (status, ei.value)
            if prep is None:  # still fresh: the good images load
                assert t.pool_size() == 0 and t.active_size() == 0
                rej, _n = t.import_regroup_many(images, active_image=0)
                assert np.array_equal(rej, want)
                same_as_image(pkg, t, R)

    ids = np.arange(1, dtype=np.uint64) + np.uint64(10**6)
    refused(new, images, abi.MM_E_STATE, prep=lambda t: t.enqueue(ids, np.array([100], np.int32), np.zeros(1, np.uint8)))
    refused(new, images, abi.MM_E_STATE, prep=lambda t: t.import_regroup_many(images))
    refused(new, [], abi.MM_E_ARG)
    refused(new, [images[0]] * 65, abi.MM_E_ARG)
    refused(new, images, abi.MM_E_ARG, active_image=2)
    refused(new, [images[0], qimg], abi.MM_E_ARG)
    other = cfg_of(pkg, MERGED, modes=2, flags=FLAG[kind], capacity=60_000)
    with pkg.Engine(other) as o:
        o.enqueue(np.arange(5, dtype=np.uint64) + np.uint64(2 * 10**6), np.full(5, 100, np.int32), np.zeros(5, np.uint8))
        oimg = o.export_state()
    refused(new, [images[0], oimg], abi.MM_E_ARG)
    refused(new, [images[0], images[0]], abi.MM_E_ARG)  # every id twice
    # an id of image 1's players that is in image 0's active section: refused only when that section is taken
    h0, s0 = pkg.engine.read_image(np.array(images[0], copy=True))
    x = np.array(images[1], np.uint8, copy=True)
    _hx, sx = pkg.engine.read_image(x)
    sx["id"][0] = s0["active"][0]
    refused(new, [images[0], x], abi.MM_E_ARG, active_image=0)
    with pkg.Engine(new) as t:
        t.import_regroup_many([images[0], x], active_image=1)
    # capacities and the reject cap
    with pkg.Engine(copy_config(new, capacity=kept - 1)) as t:
        with pytest.raises(pkg.EngineError) as ei:
            t.import_regroup_many(images, active_image=0)
        assert ei.value.status == abi.MM_E_CAP and t.pool_size() == 0 and t.active_size() == 0
    with pkg.Engine(new) as t:
        ptrs = (C.c_void_p * 2)(*[np.ascontiguousarray(i).ctypes.data for i in images])
        lens = (C.c_uint64 * 2)(*[len(i) for i in images])
        k, e = C.c_uint32(0), C.c_uint32(0)
        rc = t.lib.mm_import_regroup_many(t.h, 2, ptrs, lens, None, 0, 0, None, None, C.byref(k), C.byref(e))
        assert rc == abi.MM_E_CAP and k.value == len(want) and t.pool_size() == 0
        rej, _n = t.import_regroup_many(images, active_image=0)
        assert np.array_equal(rej, want)
        same_as_image(pkg, t, R)


# ================================================================================ GPU: config3 at 10 M players
@pytest.mark.gpu
def test_config3_ten_million_into_quantile_groups(pkg):
    n, K = 10_000_000, 4
    old = pkg.synth.make_config(n_groups=32, modes=MODES8[3:4], order=RATING, capacity=n // 2, active_capacity=2 * n,
                                flags=DENSE)
    _, rating, _, _ = pkg.synth.gen_pool(1, n, bell=True)
    g = groups_of(old, rating)
    o_own = shard.balanced_owners(np.bincount(g, minlength=32), K)
    q = np.quantile(rating, np.linspace(0, 1, 25)[1:-1]).astype(np.int64)
    cuts = np.unique(np.clip(q, 1, 4999))
    groups = tuple(zip(np.r_[0, cuts[:-1] + 1].tolist(), cuts.tolist())) + ((int(cuts[-1]) + 1, 5000),)
    new = pkg.synth.make_config(groups=groups, modes=MODES8[3:4], order=RATING, capacity=n // 2, active_capacity=2 * n,
                                flags=DENSE)
    ids = np.arange(n, dtype=U32)
    to = o_own[g]
    engines = [pkg.Engine(old) for _ in range(K)]
    for k, e in enumerate(engines):
        s = to == k
        key = pkg.Engine.pack_key(rating[s], np.zeros(int(s.sum()), np.uint8))
        assert (e.enqueue_packed(ids[s], key, (np.flatnonzero(s) % 977).astype(U32)) == 1).all()
        e.tick_packed(1000)
    images = [e.export_state() for e in engines]
    n_load = np.array([pkg.engine.read_image(np.array(i, copy=True))[0].n_players for i in images])
    n_own = shard.balanced_owners(np.bincount(groups_of(new, rating), minlength=new.n_groups), K)
    res = recut_on_one_gpu(pkg, old, new, o_own, n_own, engines, pkg.Engine)
    assert all(x["ok"] for x in res)
    sizes = [x["engine"].pool_size() for x in res]
    assert sum(sizes) == n_load.sum()
    for r in (0, K - 1):  # two ranks against the restatement of what they loaded
        send = shard.recut_sends(old, new, o_own, n_own, K)
        mine = [k for k in range(K) if k == r or send[k, r]]
        keep = np.broadcast_to(n_own == r, (new.n_modes, new.n_groups))
        R, _rej, _ = restate_many(pkg, [images[k] for k in mine], new, keep, mine.index(r))
        same_as_image(pkg, res[r]["engine"], R)
    for x in res:
        x["engine"].close()
