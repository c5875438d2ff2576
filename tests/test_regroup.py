"""Regroup on import (mm_import_regroup): an mm_export image written under another config re-filed into a fresh
engine, every player keeping its id, rating, mode, stamp and sequence number.

CPU: the numpy restatement regroup(img, cfg) -> (R, rejected) on hand-built images (identity, a split, a merge across
the sequence wrap, a moved boundary, a dropped range, a mode added and dropped, ARRIVAL <-> RATING, wide partitions on
and off), and SearchPool.resume(regroup=True) with an engine double that writes real images.
GPU: the engine after mm_import_regroup(img) against a fresh engine that mm_import'ed R, through mixed steps; identity;
a round trip; the first tick against the oracle; every refusal; config3 at 10 M players.
"""
import ctypes as C
import zlib

import numpy as np
import pytest

from .test_handover import CORRUPT, copy_config, corrupt, same_state, tick_both
from .test_requeue import layout_parts, lobbies, requeue_engine
from .test_tick_forms_and_schedules import check_tick
from .test_tile_geometry import DENSE, MODES8, WIDE, Layout

ARRIVAL, RATING = 0, 1
NO_DEDUPE = 1
U32 = np.uint32


# ================================================================================ the restatement
def groups_of(cfg, rating):
    """Group of each rating under cfg, as the engine's table has it (first match, else default_group; -1: none)."""
    y = Layout(cfg)
    r = np.clip(np.asarray(rating, np.int64), y.key_lo, y.key_lo + y.KR - 1)
    return y.grp[r - y.key_lo]


def make_image(pkg, cfg, ids, rating, mode, ts, seq, active, seq_next, id_bytes=8):
    """An mm_export image of these queued players under cfg: filed by layout partition, in age order inside one."""
    abi = pkg.abi
    rating, mode = np.asarray(rating, np.int32), np.asarray(mode, np.uint8)
    part = layout_parts(cfg, rating, mode) if len(rating) else np.zeros(0, np.int64)
    age = (np.asarray(seq, U32) - U32(seq_next)).astype(U32)
    o = np.lexsort((age, part))
    n_parts = Layout(cfg).n_segs
    idt = np.uint64 if id_bytes == 8 else np.uint32
    active = np.asarray(active).astype(idt)
    cols = [np.bincount(part, minlength=n_parts).astype(U32), np.asarray(ids).astype(idt)[o], rating[o],
            np.asarray(ts, U32)[o], np.asarray(seq, U32)[o], mode[o], active]
    off = abi.image_offsets(n_parts, len(o), len(active), id_bytes)
    h = abi.ImageHeader()
    h.magic, h.version, h.abi_version, h.id_bytes = abi.MM_IMAGE_MAGIC, abi.MM_IMAGE_VERSION, abi.MM_ABI_VERSION, id_bytes
    h.total_bytes, h.n_parts, h.n_players, h.n_active, h.seq_next = off[-1], n_parts, len(o), len(active), seq_next
    h.config = cfg
    out = np.zeros(off[-1], np.uint8)
    out[:C.sizeof(h)] = np.frombuffer(bytes(h), np.uint8)
    for k, a in enumerate(cols):
        b = np.ascontiguousarray(a).view(np.uint8)
        out[off[k]:off[k] + len(b)] = b
    return out


def regroup(pkg, img, cfg):
    """-> (R, rejected): the image re-filed under cfg (the header's Equivalence), and the image indices of the players
    cfg has no queue for, ascending."""
    h, s = pkg.engine.read_image(np.frombuffer(bytes(img), np.uint8).copy())
    keep = s["mode"] < cfg.n_modes
    keep[keep] = groups_of(cfg, s["rating"][keep]) >= 0
    R = make_image(pkg, cfg, s["id"][keep], s["rating"][keep], s["mode"][keep], s["enq_ts"][keep], s["seq"][keep],
                   s["active"], h.seq_next, h.id_bytes)
    return R, np.flatnonzero(~keep).astype(U32)


def cfg_of(pkg, groups, modes=2, order=RATING, flags=0, default=-1, capacity=200_000):
    return pkg.synth.make_config(groups=groups, modes=MODES8[:modes], order=order, capacity=capacity,
                                 active_capacity=1_000_000, default_group=default, flags=flags)


# ================================================================================ CPU: hand-built KATs
TWO = ((0, 999), (1000, 1999))


def kat_image(pkg, cfg, seq_next=100):
    """Eight players: ids 1..8, ratings across both groups, both modes, ages interleaved (seq = seq_next - 20 + k)."""
    rating = np.array([10, 1500, 600, 1200, 300, 1900, 800, 1000], np.int32)
    mode = np.array([0, 0, 0, 0, 1, 1, 0, 0], np.uint8)
    seq = (np.int64(seq_next) - 20 + np.array([3, 1, 7, 2, 5, 4, 0, 6])) % 2 ** 32
    ids = np.arange(1, 9, dtype=np.uint64)
    return make_image(pkg, cfg, ids, rating, mode, 1000 + seq % 97, seq, [50, 51], seq_next)


def r_ids(pkg, R):
    h, s = pkg.engine.read_image(R)
    return h, s, [s["id"][a:b].tolist() for a, b in zip(np.r_[0, np.cumsum(s["part_count"])[:-1]],
                                                         np.cumsum(s["part_count"]))]


def nonempty(parts):
    return [p for p in parts if p]


def test_identity_is_the_image(pkg):
    for cfg in (cfg_of(pkg, TWO), cfg_of(pkg, TWO, order=ARRIVAL), cfg_of(pkg, pkg.synth.REFERENCE_GROUPS, flags=WIDE)):
        img = kat_image(pkg, cfg)
        R, rej = regroup(pkg, img, cfg)
        assert np.array_equal(R, img) and len(rej) == 0


def test_group_split_in_two(pkg):
    old, new = cfg_of(pkg, TWO, order=ARRIVAL), cfg_of(pkg, ((0, 499), (500, 999), (1000, 1999)), order=ARRIVAL)
    R, rej = regroup(pkg, kat_image(pkg, old), new)
    h, s, parts = r_ids(pkg, R)
    assert len(rej) == 0 and h.n_parts == 6 and h.seq_next == 100
    # mode 0: [0, 499] = {1 (age 3)}, [500, 999] = {7 (0), 3 (7)}, [1000, 1999] = {4 (2), 2 (1), 8 (6)} by age
    assert parts == [[1], [7, 3], [2, 4, 8], [5], [], [6]]
    assert sorted(s["active"].tolist()) == [50, 51]


def test_two_groups_merged_across_the_sequence_wrap(pkg):
    old, new = cfg_of(pkg, TWO, flags=WIDE), cfg_of(pkg, ((0, 1999),), flags=WIDE)
    img = kat_image(pkg, old, seq_next=5)  # seq = 2^32 - 15 + k: every number lies before the wrap, seq_next after it
    h0, s0 = pkg.engine.read_image(img.copy())
    assert (s0["seq"] > 2 ** 31).all()
    R, rej = regroup(pkg, img, new)
    h, s, parts = r_ids(pkg, R)
    assert len(rej) == 0
    # ages 7 0 2 4 | 1 3 5 6 for ids 7 1 4 6 | 2 ... : mode 0 = ids 7 (0), 2 (1), 4 (2), 1 (3), 8 (6), 3 (7)
    assert nonempty(parts) == [[7, 2, 4, 1, 8, 3], [6, 5]]
    u = (s["seq"] - U32(h.seq_next)).astype(U32)
    assert (np.diff(u[:6].astype(np.int64)) > 0).all()


def test_boundary_moved(pkg):
    old, new = cfg_of(pkg, TWO, flags=WIDE), cfg_of(pkg, ((0, 1199), (1200, 1999)), flags=WIDE)
    _h, _s, parts = r_ids(pkg, regroup(pkg, kat_image(pkg, old), new)[0])
    assert nonempty(parts) == [[7, 1, 8, 3], [2, 4], [5], [6]]  # 1000 joins the lower group, between 1 and 3 by age


def test_dropped_range_is_rejected_in_image_order(pkg):
    old, new = cfg_of(pkg, TWO, flags=WIDE), cfg_of(pkg, ((0, 999),), default=-1, flags=WIDE)
    img = kat_image(pkg, old)
    R, rej = regroup(pkg, img, new)
    _h, s0 = pkg.engine.read_image(img.copy())
    assert rej.tolist() == np.flatnonzero(s0["rating"] >= 1000).tolist()
    assert (np.diff(rej.astype(np.int64)) > 0).all()
    h, s, parts = r_ids(pkg, R)
    assert nonempty(parts) == [[7, 1, 3], [5]] and h.n_active == 2
    # with a default group, the range is kept there instead
    R2, rej2 = regroup(pkg, img, cfg_of(pkg, ((0, 499), (500, 999)), default=0, flags=WIDE))
    _h2, _s2, parts2 = r_ids(pkg, R2)
    assert len(rej2) == 0 and parts2[0] == [2, 4, 1, 8] and parts2[1] == [7, 3]


def test_mode_added_and_dropped(pkg):
    old = cfg_of(pkg, TWO, modes=2)
    img = kat_image(pkg, old)
    R, rej = regroup(pkg, img, cfg_of(pkg, TWO, modes=3))
    h, _s, parts = r_ids(pkg, R)
    assert len(rej) == 0 and h.n_parts == Layout(cfg_of(pkg, TWO, modes=3)).n_segs and h.config.n_modes == 3
    R, rej = regroup(pkg, img, cfg_of(pkg, TWO, modes=1))
    _h0, s0 = pkg.engine.read_image(img.copy())
    assert rej.tolist() == np.flatnonzero(s0["mode"] == 1).tolist() and len(rej) == 2
    assert sorted(sum(r_ids(pkg, R)[2], [])) == [1, 2, 3, 4, 7, 8]


@pytest.mark.parametrize("src,dst", [(ARRIVAL, RATING), (RATING, ARRIVAL)])
def test_order_switched(pkg, src, dst):
    img = kat_image(pkg, cfg_of(pkg, TWO, order=src, flags=WIDE))
    R, rej = regroup(pkg, img, cfg_of(pkg, TWO, order=dst, flags=WIDE))
    h, _s, parts = r_ids(pkg, R)
    assert len(rej) == 0 and h.config.order_mode == dst and h.n_parts == 4
    assert nonempty(parts) == [[7, 1, 3], [2, 4, 8], [5], [6]]
    # without MM_F_WIDE_PARTITIONS, rating order stores each 1000-rating group as 4 partitions of 250 keys
    R, _rej = regroup(pkg, img, cfg_of(pkg, TWO, order=dst))
    assert nonempty(r_ids(pkg, R)[2]) == ([[1], [3], [7], [4, 8], [2], [5], [6]] if dst == RATING else
                                          [[7, 1, 3], [2, 4, 8], [5], [6]])


@pytest.mark.parametrize("src,dst", [(0, WIDE), (WIDE, 0)])
def test_wide_partitions_switched(pkg, src, dst):
    """A 1000-rating group is 4 partitions of <= 255 keys without MM_F_WIDE_PARTITIONS, one with it."""
    img = kat_image(pkg, cfg_of(pkg, TWO, flags=src))
    R, rej = regroup(pkg, img, cfg_of(pkg, TWO, flags=dst))
    h, s, parts = r_ids(pkg, R)
    assert h.n_parts == (4 if dst == WIDE else 16) and len(rej) == 0
    want = layout_parts(cfg_of(pkg, TWO, flags=dst), s["rating"], s["mode"])
    assert np.array_equal(np.repeat(np.arange(h.n_parts), s["part_count"]), want)
    u = (s["seq"] - U32(h.seq_next)).astype(np.int64)
    for p in range(h.n_parts):
        assert (np.diff(u[want == p]) > 0).all()


# ================================================================================ CPU: SearchPool.resume(regroup=True)
def regroup_engine(pkg):
    """The CPU requeue double with real mm_export images: export_state writes one, import_regroup re-files it with the
    restatement."""
    class RegroupEngine(requeue_engine(pkg)):
        def export_state(self):
            live = self.alive.astype(bool)
            ids, rating, mode = (a[live] for a in self.q)
            queued = set(ids.tolist())
            return make_image(pkg, self.cfg, ids, rating, mode, [self.ts[p] for p in ids.tolist()],
                              [self.seq_of[p] for p in ids.tolist()],
                              sorted(p for p in self.active if p not in queued), self.ctr)

        def import_state(self, buf):
            assert not self.active and not len(self.q[0]), "import into a fresh engine"
            h, s = pkg.engine.read_image(np.frombuffer(bytes(buf), np.uint8).copy())
            o = np.argsort((s["seq"] - U32(h.seq_next)).astype(U32), kind="stable")  # enqueue order
            self.q = [s["id"].astype(np.uint64)[o], s["rating"][o], s["mode"][o]]
            self.alive = np.ones(len(o), np.uint8)
            self.active = set(self.q[0].tolist()) | set(s["active"].astype(np.uint64).tolist())
            self.ts = dict(zip(s["id"].tolist(), s["enq_ts"].tolist()))
            self.seq_of = dict(zip(s["id"].tolist(), s["seq"].tolist()))
            self.ctr = h.seq_next

        def import_regroup(self, buf):
            R, rej = regroup(pkg, buf, self.cfg)
            self.import_state(R)
            return rej

    return RegroupEngine


def checkpointed_pool(pkg):
    """A pool with bronze, gold and grandmaster players in 1v1 and 5v5 and one matched 1v1 bronze lobby."""
    from .test_expire import publish
    from .test_requeue import cpu_pool
    now, wall = [0.0], [1_700_000_000.0]
    sw, cfg, eng, pool, broker = cpu_pool(pkg, lambda: now[0], lambda: wall[0], engine=regroup_engine(pkg))
    for pid, rating in (("b0", 100), ("b1", 120)):
        publish(pkg, broker, cfg, pid, rating)
    broker.deliver_all()
    now[0] += 1
    assert pool.tick() == 1
    lob = [p for team in lobbies(broker, sw)[0]["teams"].values() for p in team]
    for pid, rating, mode in (("b2", 200, "1v1"), ("g0", 2100, "1v1"), ("g1", 2200, "5v5"), ("m0", 4500, "1v1"),
                              ("b3", 300, "5v5")):
        publish(pkg, broker, cfg, pid, rating, mode)
    broker.deliver_all()
    pool.flush()
    return sw, cfg, pool, lob, now, wall


def test_resume_with_regroup_remaps_names_and_returns_the_dropped(pkg):
    sw, cfg, pool, lob, now, wall = checkpointed_pool(pkg)
    blob = pool.checkpoint()
    new = cfg_of(pkg, ((1500, 2999), (3000, 5000)), modes=1, order=ARRIVAL, capacity=1000)
    eng2 = regroup_engine(pkg)(new)
    p2 = sw.SearchPool.resume(eng2, blob, ["1v1"], ["low", "high"], regroup=True, flush_every_s=3600,
                              clock=lambda: now[0], wall_clock=lambda: wall[0])
    assert sorted(d["id"] for d in p2.regroup_dropped) == ["b2", "b3", "g1"]  # bronze has no group, 5v5 no mode
    for pid in ("b2", "b3", "g1"):
        assert p2.handles.lookup(pid) is None and not p2.in_queue(pid)
    assert p2.in_queue("g0") and p2.in_queue("m0") and sorted(p2.players) == sorted(
        p2.handles.lookup(x) for x in ("g0", "m0"))
    assert set(p2.queued) == {p2.handles.lookup(x) for x in ("g0", "m0", "b0", "b1")}
    # a matched bronze player whose rating lost its group reads "gone" instead of refusing the call
    assert p2.requeue(lob + [{"id": "g0"}]) == ["gone", "gone", "queued"]
    # names: the plain resume still refuses other names, and regroup refuses modes that change index
    with pytest.raises(ValueError):
        sw.SearchPool.resume(regroup_engine(pkg)(new), blob, ["1v1"], ["low", "high"])
    with pytest.raises(ValueError):
        sw.SearchPool.resume(regroup_engine(pkg)(new), blob, ["5v5"], ["low", "high"], regroup=True)


def test_resume_with_regroup_refuses_a_pool_with_moved_out_queues(pkg):
    sw, cfg, pool, _lob, now, wall = checkpointed_pool(pkg)
    pool.move_out(["gold"])
    blob = pool.checkpoint()
    with pytest.raises(ValueError, match="moved out"):
        sw.SearchPool.resume(regroup_engine(pkg)(cfg), blob, ["1v1", "5v5"], ["a", "b", "c", "d", "e", "f", "g"],
                             regroup=True, clock=lambda: now[0], wall_clock=lambda: wall[0])


def test_requeue_with_an_unchanged_config_is_unchanged(pkg):
    """Same config and names through regroup=True: nothing dropped, and a requeue reads what it read before."""
    sw, cfg, pool, lob, now, wall = checkpointed_pool(pkg)
    blob = pool.checkpoint()
    p2 = sw.SearchPool.resume(regroup_engine(pkg)(cfg), blob, ["1v1", "5v5"], list(pkg.synth.REFERENCE_GROUP_NAMES),
                              regroup=True, flush_every_s=3600, clock=lambda: now[0], wall_clock=lambda: wall[0])
    assert p2.regroup_dropped == [] and len(p2.players) == 5
    assert p2.requeue(lob) == ["requeued", "requeued"]


# ================================================================================ GPU helpers
def source_engine(pkg, cfg, kind, seed, bell=False, wrap=False):
    """An engine under cfg with queued, matched, removed, taken and expired players.  wrap: it starts from an imported
    image whose sequence numbers are just below 2^32, so the later ones wrap past it."""
    rng = np.random.default_rng(seed)
    eng = pkg.Engine(cfg)
    nxt = [0]

    def fresh(n):
        x = np.arange(nxt[0], nxt[0] + n, dtype=np.uint64)
        nxt[0] += n
        ids = x if kind == "dense" else pkg.synth.mix64(x + np.uint64(3 << 40))
        if bell:
            r = np.clip(rng.normal(2500, 700, n), 0, 5000).astype(np.int32)
        else:
            r = rng.integers(0, 5001, n).astype(np.int32)
        return ids, r, rng.integers(0, cfg.n_modes, n).astype(np.uint8), rng.integers(0, 90, n).astype(U32)

    if wrap:
        ids, r, m, ts = fresh(20_000)
        s0 = 2 ** 32 - 12_000
        seq = (s0 + np.arange(20_000, dtype=np.int64)) % 2 ** 32
        keep = groups_of(cfg, r) >= 0
        eng.import_state(make_image(pkg, cfg, ids[keep], r[keep], m[keep], ts[keep], seq[keep], [],
                                    (s0 + 20_000) % 2 ** 32, 4 if kind == "dense" else 8))
    eng.enqueue(*fresh(40_000))
    eng.tick(100)
    eng.enqueue(*fresh(25_000))
    if kind != "no_dedupe":
        q = eng.pool_read()["id"]
        eng.remove(q[:600])
        eng.take(q[600:1100])
    eng.expire(150, 120)
    return eng, fresh


def mixed_steps(pkg, a, b, fresh, kind, order, rng, steps=3):
    """The same calls on both engines; every result must agree."""
    dedupe = kind != "no_dedupe"
    for rnd in range(steps):
        now = 300 + 100 * rnd
        ids, r, m, ts = fresh(4000)
        old = a.pool_read()["id"][:200]
        ids, r = np.concatenate([ids, old]), np.concatenate([r, r[:len(old)]])
        m, ts = np.concatenate([m, m[:len(old)]]), np.concatenate([ts, ts[:len(old)]])
        assert np.array_equal(a.enqueue(ids, r, m, ts), b.enqueue(ids, r, m, ts))
        if dedupe:
            cur = a.pool_read()["id"]
            assert a.take(cur[500:700]) == b.take(cur[500:700])
            assert a.remove(cur[:300]) == b.remove(cur[:300])
        ea, eb = a.expire(now, 400 - 50 * rnd), b.expire(now, 400 - 50 * rnd)
        oa, ob = np.argsort(ea[1]), np.argsort(eb[1])
        assert np.array_equal(ea[0][oa], eb[0][ob]) and np.array_equal(ea[1][oa], eb[1][ob])
        sample = a.pool_read()["id"][::31]
        same_state(a, b, now, sample, dedupe)
        if order == RATING and rnd == 1:
            for e in (a, b):
                e.set_option("max_spread", 40)
        for impl in (1, 0):
            for e in (a, b):
                e.set_option("tick_impl", impl)
            tick_both(a, b, now + impl, packed=kind == "dense" and impl == 0)
            same_state(a, b, now + 5, sample, dedupe)


def export_sections(pkg, eng):
    h, s = pkg.engine.read_image(np.array(eng.export_state(), np.uint8, copy=True))
    return h, s


def same_as_image(pkg, eng, img):
    """The engine's export holds the image's players (sections 1-6 byte for byte) and active ids (as a set)."""
    h1, s1 = pkg.engine.read_image(np.array(img, np.uint8, copy=True))
    h2, s2 = export_sections(pkg, eng)
    assert (h1.n_parts, h1.n_players, h1.n_active, h1.seq_next) == (h2.n_parts, h2.n_players, h2.n_active, h2.seq_next)
    for k in ("part_count", "id", "rating", "enq_ts", "seq", "mode"):
        assert np.array_equal(s1[k], s2[k]), k
    assert np.array_equal(np.sort(s1["active"]), np.sort(s2["active"]))


REF = ((0, 1499), (1500, 1999), (2000, 2499), (2500, 2999), (3000, 3499), (3500, 3999), (4000, 5000))
SPLIT = ((0, 749), (750, 1499)) + REF[1:]
MERGED = ((0, 1999), (2000, 2999), (3000, 3999), (4000, 5000))
MOVED = ((0, 1299), (1300, 1999), (2000, 2599), (2600, 3499), (3500, 4499))  # 4500 .. 5000: no group
PAIRS = {  # name: (kind, (old groups, modes, order, flags), (new groups, modes, order, flags), bell, wrap)
    "identity": ("hashed", (REF, 3, RATING, 0), (REF, 3, RATING, 0), False, False),
    "split": ("hashed", (REF, 3, RATING, 0), (SPLIT, 3, RATING, 0), True, False),
    "merge_wrap": ("dense", (REF, 3, ARRIVAL, 0), (MERGED, 3, ARRIVAL, 0), False, True),
    "merge_rating": ("hashed", (REF, 3, RATING, WIDE), (MERGED, 3, RATING, WIDE), True, False),
    "moved_dropped": ("dense", (REF, 3, RATING, 0), (MOVED, 3, RATING, 0), False, False),
    "mode_added": ("no_dedupe", (REF, 3, RATING, 0), (REF, 4, RATING, 0), False, False),
    "mode_dropped": ("dense", (REF, 3, RATING, 0), (SPLIT, 2, RATING, 0), True, False),
    "arrival_to_rating": ("hashed", (REF, 3, ARRIVAL, 0), (MERGED, 3, RATING, 0), False, False),
    "rating_to_arrival": ("dense", (REF, 3, RATING, 0), (REF, 3, ARRIVAL, 0), True, False),
    "wide_on": ("hashed", (REF, 3, RATING, 0), (REF, 3, RATING, WIDE), False, False),
    "wide_off": ("dense", (REF, 3, RATING, WIDE), (MOVED, 3, RATING, 0), False, False),
}
FLAG = {"hashed": 0, "dense": DENSE, "no_dedupe": NO_DEDUPE}


def pair_configs(pkg, name, capacity=200_000):
    kind, old, new, _bell, _wrap = PAIRS[name]
    mk = lambda g, m, o, f: cfg_of(pkg, g, modes=m, order=o, flags=f | FLAG[kind], capacity=capacity)  # noqa: E731
    return kind, mk(*old), mk(*new)


# ================================================================================ GPU: twin equivalence
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PAIRS))
def test_regroup_equals_import_of_the_restated_image(pkg, name):
    kind, old, new = pair_configs(pkg, name)
    _k, _o, _n, bell, wrap = PAIRS[name]
    src, fresh = source_engine(pkg, old, kind, zlib.crc32(name.encode()), bell, wrap)
    with src:
        img = src.export_state()
    R, want_rej = regroup(pkg, img, new)
    if name == "identity":
        assert np.array_equal(R, img)
    if name in ("moved_dropped", "mode_dropped"):
        assert len(want_rej) > 1000
    with pkg.Engine(new) as a, pkg.Engine(new) as b:
        rej = a.import_regroup(img)
        assert np.array_equal(rej, want_rej)
        b.import_state(R)
        same_as_image(pkg, a, R)
        dedupe = kind != "no_dedupe"
        _h, s = pkg.engine.read_image(np.array(img, np.uint8, copy=True))
        gone = s["id"][want_rej].astype(np.uint64)
        sample = np.concatenate([a.pool_read()["id"][::41], s["active"][::7].astype(np.uint64), gone[:300]])
        same_state(a, b, 200, sample, dedupe)
        if dedupe:
            assert not a.in_queue(gone).any()
        mixed_steps(pkg, a, b, fresh, kind, new.order_mode, np.random.default_rng(4))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hashed", "dense"])
def test_round_trip_gives_the_original_sections(pkg, kind):
    old = cfg_of(pkg, REF, modes=3, flags=FLAG[kind])
    new = cfg_of(pkg, SPLIT + ((5001, 6000),), modes=4, order=ARRIVAL, flags=FLAG[kind] | WIDE)
    src, _fresh = source_engine(pkg, old, kind, 11)
    with src:
        img = src.export_state()
    with pkg.Engine(new) as b:
        assert len(b.import_regroup(img)) == 0
        mid = b.export_state()
    with pkg.Engine(old) as a:
        assert len(a.import_regroup(mid)) == 0
        same_as_image(pkg, a, img)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["split", "merge_rating", "arrival_to_rating", "moved_dropped"])
def test_first_tick_after_regroup_equals_the_oracle(pkg, oracle, name):
    kind, old, new = pair_configs(pkg, name)
    rng = np.random.default_rng(7)
    n = 3000
    ids = np.arange(n, dtype=np.uint64) if kind == "dense" else pkg.synth.mix64(np.arange(n, dtype=np.uint64))
    with pkg.Engine(old) as src:
        src.enqueue(ids, rng.integers(0, 5001, n).astype(np.int32), rng.integers(0, 3, n).astype(np.uint8),
                    rng.integers(0, 50, n).astype(U32))
        img = src.export_state()
    _h, s = pkg.engine.read_image(np.array(img, np.uint8, copy=True))
    seq_of = dict(zip(s["id"].tolist(), s["seq"].tolist()))
    with pkg.Engine(new) as a:
        a.import_regroup(img)
        pr = a.pool_read()
        ref = oracle.run_literal(new, pr["id"], pr["rating"], pr["mode"])
        check_tick(ref, np.array([seq_of[p] for p in pr["id"].tolist()], U32), *a.tick(10))


# ================================================================================ GPU: refusals
def raw_regroup(pkg, eng, img, cap, with_buf=True):
    rej = np.zeros(max(cap, 1), U32)
    k = C.c_uint32(0)
    buf = np.ascontiguousarray(img, np.uint8)
    rc = eng.lib.mm_import_regroup(eng.h, buf.ctypes.data_as(C.c_void_p), len(buf), cap,
                                   rej.ctypes.data_as(C.c_void_p) if with_buf else None, C.byref(k))
    return rc, k.value, rej


@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True])
def test_refusals_leave_the_engine_fresh(pkg, dense):
    abi = pkg.abi
    kind = "dense" if dense else "hashed"
    old = cfg_of(pkg, REF, modes=2, flags=FLAG[kind], capacity=20_000)
    new = cfg_of(pkg, MOVED, modes=2, order=ARRIVAL, flags=FLAG[kind], capacity=20_000)
    rng = np.random.default_rng(1)
    with pkg.Engine(old) as src:
        ids = np.arange(12_000, dtype=np.uint64) if dense else pkg.synth.mix64(np.arange(12_000, dtype=np.uint64))
        src.enqueue(ids, rng.integers(0, 5001, len(ids)).astype(np.int32), rng.integers(0, 2, len(ids)).astype(np.uint8))
        src.tick(10)
        more = ids + np.uint64(20_000)
        src.enqueue(more, rng.integers(0, 5001, len(ids)).astype(np.int32), rng.integers(0, 2, len(ids)).astype(np.uint8))
        img = src.export_state()
        qimg = src.export_queues(np.ones(old.n_modes * old.n_groups, bool))
    R, want = regroup(pkg, img, new)
    h, s = pkg.engine.read_image(np.array(img, np.uint8, copy=True))
    kept = h.n_players - len(want)
    assert len(want) > 100 and h.n_active > 1000

    def refused(cfg, image, status, prep=None, **kw):
        with pkg.Engine(cfg) as t:
            if prep:
                prep(t)
            with pytest.raises(pkg.EngineError) as ei:
                t.import_regroup(image)
            assert ei.value.status == status, status
            if prep is None:  # still fresh: the good image loads
                assert t.pool_size() == 0 and t.active_size() == 0
                assert np.array_equal(t.import_regroup(img), want)
                same_as_image(pkg, t, R)

    # state
    refused(new, img, abi.MM_E_STATE, prep=lambda t: t.enqueue(ids[:1], np.array([100], np.int32), np.zeros(1, np.uint8)))
    refused(new, img, abi.MM_E_STATE, prep=lambda t: (t.snapshot(), t.restore()))
    refused(new, img, abi.MM_E_STATE, prep=lambda t: t.import_regroup(img))
    if dense:
        refused(new, img, abi.MM_E_STATE, prep=lambda t: t.enqueue_packed_begin(np.arange(5, dtype=U32),
                                                                                 t.pack_key(np.full(5, 100), np.zeros(5))))
    # image kind, id width, MM_F_NO_DEDUPE
    refused(new, qimg, abi.MM_E_ARG)
    with pkg.Engine(copy_config(new, flags=new.flags ^ DENSE)) as t:
        with pytest.raises(pkg.EngineError) as ei:
            t.import_regroup(img)
        assert ei.value.status == abi.MM_E_ARG and t.pool_size() == 0
    with pkg.Engine(copy_config(new, flags=(new.flags & ~DENSE) | NO_DEDUPE)) as t:
        with pytest.raises(pkg.EngineError) as ei:
            t.import_regroup(img)
        assert ei.value.status == abi.MM_E_ARG and t.pool_size() == 0
    # every corruption mm_import refuses, judged against the image's own config
    for what in CORRUPT:
        if what == "handle" and not dense:
            continue
        refused(new, corrupt(pkg, img, what, old), abi.MM_E_ARG)
    # a repeated id among players the new config rejects; a repeated seq the merge puts into one partition
    x = np.array(img, np.uint8, copy=True)
    hx, sx = pkg.engine.read_image(x)
    r0, r1 = int(want[0]), int(want[1])
    sx["id"][r1] = sx["id"][r0]
    refused(new, x, abi.MM_E_ARG)
    merged = cfg_of(pkg, ((0, 5000),), modes=2, flags=FLAG[kind] | WIDE, capacity=40_000)
    x = np.array(img, np.uint8, copy=True)
    hx, sx = pkg.engine.read_image(x)
    # a player of image partition 1 takes the seq of one of partition 0 that fits its neighbours' ages: both
    # partitions stay in order (mm_import under the image's config accepts it), and the merge puts the two together
    u = (sx["seq"] - U32(hx.seq_next)).astype(np.int64)
    a1, a2 = int(sx["part_count"][0]), int(sx["part_count"][0] + sx["part_count"][1])
    assert sx["mode"][0] == sx["mode"][a1] == 0
    for j in range(a1 + 1, a2 - 1):
        cand = np.flatnonzero((u[:a1] > u[j - 1]) & (u[:a1] < u[j + 1]))
        if len(cand):
            break
    sx["seq"][j] = sx["seq"][cand[0]]
    with pkg.Engine(old) as t:
        t.import_state(x)
    with pkg.Engine(merged) as t:
        assert t.import_regroup(np.array(img, np.uint8)).size == 0
    with pkg.Engine(merged) as t:
        with pytest.raises(pkg.EngineError) as ei:
            t.import_regroup(x)
        assert ei.value.status == abi.MM_E_ARG and t.pool_size() == 0 and t.active_size() == 0
    # capacities: players, hashed active-set load
    with pkg.Engine(copy_config(new, capacity=kept - 1)) as t:
        with pytest.raises(pkg.EngineError) as ei:
            t.import_regroup(img)
        assert ei.value.status == abi.MM_E_CAP and t.pool_size() == 0
    with pkg.Engine(copy_config(new, capacity=kept)) as t:
        assert np.array_equal(t.import_regroup(img), want)
    if not dense:
        with pkg.Engine(copy_config(new, active_capacity=(kept + h.n_active) // 3)) as t:
            with pytest.raises(pkg.EngineError) as ei:
                t.import_regroup(img)
            assert ei.value.status == abi.MM_E_CAP and t.pool_size() == 0 and t.active_size() == 0
    # more rejects than cap: the exact count, nothing loaded; the dry run
    with pkg.Engine(new) as t:
        rc, k, _ = raw_regroup(pkg, t, img, len(want) - 1)
        assert rc == abi.MM_E_CAP and k == len(want) and t.pool_size() == 0
        rc, k, _ = raw_regroup(pkg, t, img, 0, with_buf=False)
        assert rc == abi.MM_E_CAP and k == len(want) and t.pool_size() == 0
        rc, k, rej = raw_regroup(pkg, t, img, len(want))
        assert rc == abi.MM_OK and k == len(want) and np.array_equal(rej[:k], want)
        same_as_image(pkg, t, R)


# ================================================================================ GPU: config3 at 10 M players
def config3_targets(pkg, rating, n):
    """(a) 24 equal-width groups, (b) 32 groups cut at the population's quantiles, (c) the 32 groups and a mode more."""
    q = np.quantile(rating, np.linspace(0, 1, 33)[1:-1]).astype(np.int64)
    cuts = np.unique(np.clip(q, 1, 4999))
    balanced = tuple(zip(np.r_[0, cuts[:-1] + 1].tolist(), cuts.tolist())) + ((int(cuts[-1]) + 1, 5000),)
    mk = lambda **kw: pkg.synth.make_config(modes=MODES8[3:4], order=RATING, capacity=n + 65536,  # noqa: E731
                                           active_capacity=2 * n, flags=DENSE, **kw)
    c = pkg.synth.make_config(n_groups=32, modes=MODES8[3:5], order=RATING, capacity=n + 65536, active_capacity=2 * n,
                              flags=DENSE)
    return {"a": mk(n_groups=24), "b": mk(groups=balanced), "c": c}


@pytest.mark.gpu
def test_config3_ten_million(pkg):
    n = 10_000_000
    old = pkg.synth.make_config(n_groups=32, modes=MODES8[3:4], order=RATING, capacity=n + 65536, active_capacity=2 * n,
                                flags=DENSE)
    _, rating, _, _ = pkg.synth.gen_pool(1, n, bell=True)
    key = pkg.Engine.pack_key(rating, np.zeros(n, np.uint8))
    with pkg.Engine(old) as src:
        assert (src.enqueue_packed(np.arange(n, dtype=U32), key, (np.arange(n) % 977).astype(U32)) == 1).all()
        src.tick_packed(1000)  # about 1 M lobbies: their members stay in the active set
        second = np.arange(n, 2 * n, dtype=U32)
        assert (src.enqueue_packed(second, key, (np.arange(n) % 991).astype(U32)) == 1).all()
        img = src.export_state()
    h, _s = pkg.engine.read_image(np.array(img, np.uint8, copy=True))
    assert h.n_players > 9_900_000 and h.n_active > 9_900_000
    for name, new in config3_targets(pkg, rating, n).items():
        R, want = regroup(pkg, img, new)
        with pkg.Engine(new) as a:
            assert np.array_equal(a.import_regroup(img), want), name
            same_as_image(pkg, a, R)
