"""Every refusal of the engine's host entry points: the status and the exact mm_last_error text.

GPU only.  Each case builds the smallest state that reaches one check: mm_import (not fresh, each header check, the
capacities, the device checks of the players), mm_merge (a staged packed batch, live players in a receiving queue, the
reject list, the pool and the active set, the header and device checks), mm_export / mm_export_queues (a staged
packed batch, a short buffer), mm_expire (cap), the ingest (active set full) and the packed staging slots.
"""
import ctypes as C

import numpy as np
import pytest

from .test_ingest import hashed_slots

ARRIVAL = 0
NO_DEDUPE, DENSE = 1, 2
G = 4  # rating groups; arrival order keeps one partition per (mode, group) queue
STAGED = "a packed batch is staged: call mm_enqueue_packed_end first"

pytestmark = pytest.mark.gpu


def config(pkg, **kw):
    kw.setdefault("capacity", 4000)
    return pkg.synth.make_config(n_groups=G, order=ARRIVAL, **kw)


def players(pkg, k0, k1, dense=False, mode=None):
    """ids k0..k1 (handles when dense), ratings over every group, modes 0 / 1 (or `mode`), enqueue stamps 0..99"""
    rng = np.random.default_rng(k0)
    n = k1 - k0
    ids = np.arange(k0, k1, dtype=np.uint64)
    if not dense:
        ids = pkg.synth.mix64(ids + np.uint64(5 << 40))
    modes = rng.integers(0, 2, n) if mode is None else np.full(n, mode)
    return ids, rng.integers(0, 5001, n).astype(np.int32), modes.astype(np.uint8), rng.integers(0, 100, n).astype(np.uint32)


def refused(pkg, eng, call, *args):
    """-> (status, mm_last_error) of an engine call that must fail"""
    with pytest.raises(pkg.EngineError) as ei:
        call(*args)
    return ei.value.status, eng.lib.mm_last_error(eng.h).decode()


def with_header(pkg, img, **fields):
    """a copy of the image with header fields changed"""
    x = np.array(img, np.uint8, copy=True)
    hs = C.sizeof(pkg.abi.ImageHeader)
    h = pkg.abi.ImageHeader.from_buffer_copy(x[:hs].tobytes())
    for k, v in fields.items():
        setattr(h, k, v)
    x[:hs] = np.frombuffer(bytes(h), np.uint8)
    return x


def with_active_section(pkg, img):
    """an image without active section, with one zero id appended as its active section (counts and length agree)"""
    h, _ = pkg.engine.read_image(img)
    off = pkg.abi.image_offsets(h.n_parts, h.n_players, 1, h.id_bytes)
    x = np.zeros(off[-1], np.uint8)
    x[:len(img)] = img
    return with_header(pkg, x, n_active=1, total_bytes=off[-1])


def with_players(pkg, img, *edits):
    """a copy of the image with player columns edited: (column, index, value), or "swap_seq" (players 0 and 1)"""
    x = np.array(img, np.uint8, copy=True)
    _, s = pkg.engine.read_image(x)
    for ed in edits:
        if ed == "swap_seq":
            s["seq"][[0, 1]] = s["seq"][[1, 0]]
        else:
            col, i, v = ed
            s[col][i] = v
    return x


def other_group(rating):
    return (int(rating) + 2500) % 5000  # groups are 1250 wide: another group, so another partition


def source_image(pkg, cfg, dense=False, queues=None):
    """an image of an engine with queued players and matched ids not yet removed (queues: a queue image of them)"""
    with pkg.Engine(cfg) as src:
        src.enqueue(*players(pkg, 0, 1000, dense))
        src.tick(100)
        src.enqueue(*players(pkg, 1000, 1500, dense))
        return src.export_state() if queues is None else src.export_queues(queues)


@pytest.mark.parametrize("dedupe", [True, False])
def test_import_refusals(pkg, dedupe):
    abi = pkg.abi
    cfg = config(pkg, flags=0 if dedupe else NO_DEDUPE)
    img = source_image(pkg, cfg)
    h, s = pkg.engine.read_image(img)
    assert h.n_players > 2 and (h.n_active > 0) == dedupe and s["part_count"][s["part_count"] > 0][0] >= 2
    pre = "image rejected: "
    arg = [
        (img[:100], "shorter than its header"),
        (with_header(pkg, img, magic=abi.MM_QUEUE_IMAGE_MAGIC), "bad magic"),
        (with_header(pkg, img, version=99), "unknown version"),
        (with_header(pkg, img, id_bytes=4), "id width differs from the engine's"),
        (with_header(pkg, img, n_parts=h.n_parts + 1), "partition count differs from the engine's layout"),
        (img[:-8], "length does not match the header's section counts"),
        (with_players(pkg, img, ("part_count", int(np.nonzero(s["part_count"])[0][0]), s["part_count"].max() + 1)),
         "partition counts do not add up to the player count"),
        (with_players(pkg, img, ("mode", 3, cfg.n_modes)), "mode out of range"),
        (with_players(pkg, img, ("rating", 0, other_group(s["rating"][0]))), "rating outside its partition"),
        (with_players(pkg, img, "swap_seq"), "sequence numbers out of order"),
        (with_players(pkg, img, ("mode", 3, cfg.n_modes), "swap_seq"), "mode out of range sequence numbers out of order"),
    ]
    if dedupe:
        arg += [(with_players(pkg, img, ("id", 7, s["id"][2])), "duplicate id"),
                (with_players(pkg, img, ("active", 0, s["id"][4])), "duplicate id")]
    else:
        arg += [(with_active_section(pkg, img), "active section in an image of an engine without an active set")]
    for buf, msg in arg:
        with pkg.Engine(cfg) as t:
            assert refused(pkg, t, t.import_state, buf) == (abi.MM_E_ARG, pre + msg), msg
    with pkg.Engine(config(pkg, default_group=-1, flags=cfg.flags)) as t:
        assert refused(pkg, t, t.import_state, img) == (
            abi.MM_E_ARG, pre + "config differs from the engine's (groups, default_group, modes, order_mode or flags)")
    small = config(pkg, capacity=h.n_players - 1, flags=cfg.flags)
    with pkg.Engine(small) as t:
        assert refused(pkg, t, t.import_state, img) == (
            abi.MM_E_CAP, f"{h.n_players} players, capacity {h.n_players - 1}")
    if dedupe:
        few = config(pkg, active_capacity=100)
        assert (h.n_players + h.n_active) * 4 > hashed_slots(few) * 3
        with pkg.Engine(few) as t:
            assert refused(pkg, t, t.import_state, img) == (
                abi.MM_E_CAP, f"{h.n_players + h.n_active} active ids, active set holds {hashed_slots(few) * 3 // 4}")
    with pkg.Engine(cfg) as t:
        t.enqueue(*players(pkg, 5000, 5001))
        assert refused(pkg, t, t.import_state, img) == (
            abi.MM_E_STATE, "mm_import needs a fresh engine (nothing enqueued, imported or restored)")


def test_merge_refusals(pkg):
    abi = pkg.abi
    cfg = config(pkg)
    mode0 = np.zeros((cfg.n_modes, G), bool)
    mode0[0] = True
    qimg = source_image(pkg, cfg, queues=mode0)  # every mode-0 queue
    h, s = pkg.engine.read_image(qimg)
    n = h.n_players
    assert n > 100 and (s["mode"] == 0).all() and s["part_count"][s["part_count"] > 0][0] >= 2
    pre = "queue image rejected: "
    arg = [
        (source_image(pkg, cfg), "bad magic (not an mm_export_queues image)"),
        (with_active_section(pkg, qimg), "a queue image has no active section"),
        (with_players(pkg, qimg, ("mode", 3, cfg.n_modes)), "mode out of range"),
        (with_players(pkg, qimg, ("rating", 0, other_group(s["rating"][0]))), "rating outside its partition"),
        (with_players(pkg, qimg, "swap_seq"), "sequence numbers out of order"),
    ]
    for buf, msg in arg:
        with pkg.Engine(cfg) as t:
            assert refused(pkg, t, t.merge_queues, buf) == (abi.MM_E_ARG, pre + msg), msg
    # live players in a receiving queue: three in (mode 0, group 1)
    with pkg.Engine(cfg) as t:
        ids, _, _, ts = players(pkg, 9000, 9003)
        t.enqueue(ids, np.array([1300, 1301, 1302], np.int32), np.zeros(3, np.uint8), ts)
        assert refused(pkg, t, t.merge_queues, qimg) == (abi.MM_E_STATE, "queue (mode 0, group 1) holds 3 live players here")
    # five image ids already active here (queued in mode 1): a reject list of 0 is too short
    with pkg.Engine(cfg) as t:
        t.enqueue(s["id"][:5].copy(), np.full(5, 100, np.int32), np.ones(5, np.uint8))
        k = C.c_uint32(0)
        assert t.lib.mm_merge(t.h, qimg.ctypes.data_as(C.c_void_p), len(qimg), 0, None, C.byref(k)) == abi.MM_E_CAP
        assert (t.lib.mm_last_error(t.h).decode(), k.value) == ("5 rejected players, cap 0", 5)
    # the pool: 20 players of mode 1 in use
    with pkg.Engine(config(pkg, capacity=n + 10)) as t:
        t.enqueue(*players(pkg, 8000, 8020, mode=1))
        assert refused(pkg, t, t.merge_queues, qimg) == (
            abi.MM_E_CAP, f"{n} players merged into 20 slots in use, capacity {n + 10}")
    # the active set: 700 ids resident, 768 at most
    few = config(pkg, active_capacity=100)
    assert (700 + n) * 4 > hashed_slots(few) * 3
    with pkg.Engine(few) as t:
        t.enqueue(*players(pkg, 8000, 8700, mode=1))
        assert refused(pkg, t, t.merge_queues, qimg) == (
            abi.MM_E_CAP, f"active set full: 700 ids resident, {n} merged, capacity {hashed_slots(few) * 3 // 4}")


def test_dense_refusals(pkg):
    """Handles out of range, staged packed batches, the staging slots"""
    abi = pkg.abi
    cfg = config(pkg, active_capacity=10_000, flags=DENSE)
    img = source_image(pkg, cfg, dense=True)
    qimg = source_image(pkg, cfg, dense=True, queues=np.ones(cfg.n_modes * G, bool))
    with pkg.Engine(cfg) as t:
        assert refused(pkg, t, t.import_state, with_players(pkg, img, ("id", 5, cfg.active_capacity))) == (
            abi.MM_E_ARG, "image rejected: id out of range")
    with pkg.Engine(cfg) as t:
        assert refused(pkg, t, t.merge_queues, with_players(pkg, qimg, ("id", 5, cfg.active_capacity))) == (
            abi.MM_E_ARG, "queue image rejected: id out of range")
    with pkg.Engine(cfg) as eng:
        eng.enqueue(*players(pkg, 2000, 3000, dense=True))
        k = C.c_uint32(0)
        assert eng.lib.mm_enqueue_packed_end(eng.h, None, C.byref(k)) == abi.MM_E_STATE
        assert eng.lib.mm_last_error(eng.h).decode() == "no staged batch: call mm_enqueue_packed_begin first"
        keys = eng.pack_key(np.full(4, 100), np.zeros(4))
        eng.enqueue_packed_begin(np.arange(5000, 5004, dtype=np.uint32), keys)
        assert refused(pkg, eng, eng.export_state) == (abi.MM_E_STATE, STAGED)
        assert refused(pkg, eng, eng.export_queues, np.ones(cfg.n_modes * G, bool)) == (abi.MM_E_STATE, STAGED)
        assert refused(pkg, eng, eng.merge_queues, qimg) == (abi.MM_E_STATE, STAGED)
        eng.enqueue_packed_begin(np.arange(5004, 5008, dtype=np.uint32), keys)
        assert refused(pkg, eng, eng.enqueue_packed_begin, np.arange(5008, 5012, dtype=np.uint32), keys) == (
            abi.MM_E_STATE, "both staging slots hold a batch: call mm_enqueue_packed_end first")
        assert eng.enqueue_packed_end()[1] == 4 and eng.enqueue_packed_end()[1] == 4


def test_capacity_refusals(pkg):
    """mm_export with a short buffer, mm_expire with a short cap, an ingest batch the active set cannot hold"""
    abi = pkg.abi
    cfg = config(pkg)
    with pkg.Engine(cfg) as eng:
        ids, rating, mode, _ = players(pkg, 0, 100)
        eng.enqueue(ids, rating, mode, np.arange(100, dtype=np.uint32))
        size = len(eng.export_state())
        n = C.c_uint64(0)
        buf = np.empty(100, np.uint8)
        assert eng.lib.mm_export(eng.h, buf.ctypes.data_as(C.c_void_p), 100, C.byref(n)) == abi.MM_E_CAP
        assert (eng.lib.mm_last_error(eng.h).decode(), n.value) == (f"need cap >= {size}", size)
        k = C.c_uint32(0)
        out = np.empty(1, np.uint64)
        assert eng.lib.mm_expire(eng.h, 1000, 10, out.ctypes.data_as(C.c_void_p), None, 1, C.byref(k)) == abi.MM_E_CAP
        assert (eng.lib.mm_last_error(eng.h).decode(), k.value) == ("need cap >= 100", 100)
        assert eng.pool_size() == 100  # a refused expire changes nothing
    few = config(pkg, active_capacity=100)
    with pkg.Engine(few) as eng:
        assert refused(pkg, eng, eng.enqueue, *players(pkg, 0, 800)[:3]) == (
            abi.MM_E_CAP, f"active set full: 0 ids resident, batch of 800, capacity {hashed_slots(few) * 3 // 4}")
