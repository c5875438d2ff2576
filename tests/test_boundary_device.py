"""EXTENSION (DESIGN.md §6): the boundary pass on the device — mm_band_candidates / mm_band_match and
shard.boundary_pass_device — against the host path shard.boundary_pass on the same engine state.

Every comparison runs both paths from one mm_snapshot per rank: the host path first, then mm_restore and the device
path.  Equal means the pass's dict (hdr in order and every field, member_ids in order, the four counts) and, after
it, every rank's pool_read, in_queue, active_size, the waiting section of queue_stats and the next tick's results."""
import ctypes as C
import importlib
import threading

import numpy as np
import pytest

from .test_boundary import make_cfg, make_players

shard = importlib.import_module("microservice-matchmaking_b200.shard")
LOBBY_DTYPE = importlib.import_module("microservice-matchmaking_b200.engine").LOBBY_DTYPE
RATING = 1
NOW = 1_000


# ---- CPU: the ABI mirror -----------------------------------------------------------------------------------------
def test_band_prototypes_and_stats_layout(pkg):
    abi = pkg.abi
    assert C.sizeof(abi.BandStats) == 32
    assert len(abi.PROTOTYPES["mm_band_candidates"][1]) == 8
    assert len(abi.PROTOTYPES["mm_band_match"][1]) == 15
    assert abi.PROTOTYPES["mm_band_match"][1][-1] == C.POINTER(abi.BandStats)


# ---- helpers ---------------------------------------------------------------------------------------------------------
def rank_config(pkg, cfg, capacity, flags=0, order=RATING):
    c = type(cfg).from_buffer_copy(cfg)
    c.capacity = max(int(capacity), 1)
    c.flags = flags
    c.order_mode = order
    if flags & pkg.abi.MM_F_DENSE_IDS:
        c.active_capacity = c.capacity
    return c


def load_ranks(pkg, cfg, W, K, ids, rating, mode, flags=0, tick=True, between=None):
    """K engines holding the players routed to them, ticked at NOW (unless tick=False) -> [(engine, ids of the rank)]"""
    owner = shard.route(cfg, rating, K)
    ranks = []
    for r in range(K):
        mine = owner == r
        eng = pkg.Engine(rank_config(pkg, cfg, mine.sum() + 16, flags))
        eng.set_option("max_spread", W)
        ts = np.arange(mine.sum(), dtype=np.uint32) % 600
        assert (eng.enqueue(ids[mine], rating[mine], mode[mine], ts) == 1).all()
        if tick:
            eng.tick(now=NOW)
        if between is not None:
            between(r, eng, ids[mine])
        ranks.append((eng, ids[mine]))
    return ranks


def run_ranks(K, fn):
    """fn(rank, comm) on K threads sharing one LocalComm -> per-rank results"""
    comm = shard.LocalComm()
    out, errs = [None] * K, []

    def work(r):
        try:
            out[r] = fn(r, comm)
        except BaseException as ex:  # noqa: BLE001 — surfaced below
            errs.append(ex)

    th = [threading.Thread(target=work, args=(r,)) for r in range(K)]
    [t.start() for t in th]
    [t.join(600) for t in th]
    if errs:
        raise errs[0]
    assert all(o is not None for o in out), "a rank did not finish"
    return out


def state_of(eng, ids):
    pr = eng.pool_read()
    qs = eng.queue_stats(NOW + 10)
    lob, mem, seq, st = eng.tick(now=NOW + 20)
    return dict(pool=[pr[k].copy() for k in ("id", "rating", "mode", "enq_ts")], inq=eng.in_queue(ids),
                active=eng.active_size(), wait=[qs[k].copy() for k in ("n_waiting", "n_removed", "max_wait", "wait_hist")],
                tick=(lob.copy(), mem.copy(), seq.copy(), st.n_lobbies, st.n_matched, st.n_residual, st.n_dead))


def same(a, b):
    if a is None or b is None:
        return a is None and b is None
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return a.dtype == b.dtype and np.array_equal(a, b)
    return a == b


def compare_paths(pkg, cfg, W, K, ids, rating, mode, flags=0, tick=True, between=None, full_state=True):
    """Host pass, then (after mm_restore) device pass, from the same state on every rank -> (host dicts, device dicts)"""
    ranks = load_ranks(pkg, cfg, W, K, ids, rating, mode, flags, tick, between)
    try:
        for eng, _ in ranks:
            eng.snapshot()
        host = run_ranks(K, lambda r, comm: shard.boundary_pass(pkg, cfg, W, K, r, ranks[r][0], comm))
        host_state = [state_of(eng, own) for eng, own in ranks] if full_state else None
        for eng, _ in ranks:
            eng.restore()
        dev = run_ranks(K, lambda r, comm: shard.boundary_pass_device(pkg, cfg, W, K, r, ranks[r][0], comm))
        dev_state = [state_of(eng, own) for eng, own in ranks] if full_state else None
    finally:
        for eng, _ in ranks:
            eng.close()
    for r in range(K):
        assert same(host[r], dev[r]), f"rank {r}: the device pass differs from the host pass"
        if full_state:
            assert same(host_state[r], dev_state[r]), f"rank {r}: the state after the pass differs"
    return host, dev


def max_w(cfg):
    return min((cfg.group_hi[g] - cfg.group_lo[g] + 1) // 2 for g in range(cfg.n_groups))


def uniform_players(seed, n, lo, hi, n_modes=2):
    rng = np.random.default_rng(seed)
    ids = rng.permutation(np.arange(1, n + 1, dtype=np.uint64) * np.uint64(7919) + np.uint64(10 ** 9))
    return ids, rng.integers(lo, hi + 1, n).astype(np.int32), rng.integers(0, n_modes, n).astype(np.uint8)


# ---- equivalence -----------------------------------------------------------------------------------------------------
G16 = 16


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 2, 4, 8])
@pytest.mark.parametrize("W", [0, 1, 2, 5, "max"])
def test_device_pass_equals_host_pass(pkg, K, W):
    n = 4_000
    cfg = make_cfg(pkg, G16, n + 1000)
    W = max_w(cfg) if W == "max" else W
    ids, rating, mode = make_players(pkg, n, 7, G16)
    host, dev = compare_paths(pkg, cfg, W, K, ids, rating, mode)
    matched = sum(d["matched"] for d in dev)
    if 1 <= W <= 5:  # (at the largest W the local tick's window already spans most of a group and leaves no band)
        assert matched > 0
    if K > 1 and 1 <= W <= 5:
        assert sum(d["sent"] for d in dev) == sum(d["received"] for d in dev) > 0
    if W == 0:
        assert matched == 0 and all(d["hdr"] is None for d in dev)


# ---- layouts ---------------------------------------------------------------------------------------------------------
WIDE_700 = [(0, 699), (700, 1399), (1400, 2099), (2100, 2799)]  # 3 partitions of <= 234 keys per group


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [0, 4], ids=["split", "wide_partitions"])
@pytest.mark.parametrize("groups,W", [("reference", 2), ("reference", 250), (WIDE_700, 300), (WIDE_700, 117)])
def test_wide_groups_bands_across_partitions(pkg, flags, groups, W):
    """The reference's 500 - 1 500-rating groups and 700-wide groups: a side of a band covers one or two of a group's
    <= 255-key partitions (W = 300: keys 400..699 of a 700-key group = two partitions), or lies in one partition with
    MM_F_WIDE_PARTITIONS.  No tick first: the bands are full."""
    n = 6_000
    grp = pkg.synth.REFERENCE_GROUPS if groups == "reference" else groups
    cfg = pkg.synth.make_config(groups=grp, modes=(("1v1", 2, 1), ("2v2", 2, 2)), order=RATING, capacity=n,
                                default_group=-1)
    lo, hi = grp[0][0], grp[-1][1]
    ids, rating, mode = uniform_players(3, n, lo, hi)
    for K in (1, 2):
        host, dev = compare_paths(pkg, cfg, W, K, ids, rating, mode, flags=flags, tick=False)
        assert sum(d["matched"] for d in dev) > 0


@pytest.mark.gpu
def test_dense_ids_engine(pkg):
    n = 4_000
    cfg = make_cfg(pkg, G16, n)
    _, rating, mode = make_players(pkg, n, 5, G16)
    ids = np.random.default_rng(1).permutation(len(rating)).astype(np.uint64)  # handles 0 .. n-1
    host, dev = compare_paths(pkg, cfg, 2, 1, ids, rating, mode, flags=pkg.abi.MM_F_DENSE_IDS)
    assert dev[0]["matched"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 2])
def test_removed_and_taken_players_are_not_candidates(pkg, K):
    n, W = 4_000, 3
    cfg = make_cfg(pkg, G16, n)
    ids, rating, mode = make_players(pkg, n, 9, G16)
    gone = []

    def between(r, eng, own):
        left = eng.pool_read()
        near = np.zeros(len(left["id"]), bool)
        for g in range(G16 - 1):
            near |= np.abs(left["rating"].astype(np.int64) - cfg.group_hi[g]) <= W
        cand = left["id"][near]
        eng.remove(cand[0::3])
        assert eng.take(cand[1::3]) == len(cand[1::3])
        gone.extend(cand[0::3].tolist() + cand[1::3].tolist())

    host, dev = compare_paths(pkg, cfg, W, K, ids, rating, mode, between=between)
    assert gone
    members = np.concatenate([d["member_ids"] for d in dev])
    assert not np.isin(members, np.array(gone, np.uint64)).any()


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 4])
def test_pass_on_a_pool_that_was_not_ticked(pkg, K):
    n = 6_000
    cfg = make_cfg(pkg, G16, n + 1000)
    ids, rating, mode = make_players(pkg, n, 13, G16)
    host, dev = compare_paths(pkg, cfg, 4, K, ids, rating, mode, tick=False)
    assert sum(d["matched"] for d in dev) > 0


# ---- ordering, out-of-range ratings, refusals ------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("W", [1, 5, 156])
def test_candidates_are_the_sorted_numpy_selection(pkg, W):
    n = 5_000
    cfg = make_cfg(pkg, G16, n)
    ids, rating, mode = make_players(pkg, n, 21, G16)
    with pkg.Engine(rank_config(pkg, cfg, n + 100)) as eng:
        eng.enqueue(ids, rating, mode)
        eng.remove(ids[::17])
        pr = eng.pool_read()
        grp = shard.group_of_rating(cfg, pr["rating"])
        for g in range(1, G16):
            sel = (grp == g) & (pr["rating"] > cfg.group_hi[g - 1]) & (pr["rating"] <= cfg.group_hi[g - 1] + W)
            i = np.nonzero(sel)[0]
            i = i[np.lexsort((pr["rating"][i], pr["mode"][i]))]  # stable: enqueue order inside a (mode, rating)
            got = eng.band_candidates(W, g)
            assert np.array_equal(got[0], pr["id"][i]) and np.array_equal(got[1], pr["rating"][i])
            assert np.array_equal(got[2], pr["mode"][i])
        assert eng.pool_size() == len(ids) and len(eng.pool_read()["id"]) == len(pr["id"])  # a query only reads


@pytest.mark.gpu
def test_out_of_range_ratings_are_never_candidates(pkg):
    """Ratings outside every group fall back to the default group; their clamped sort key lies outside every band."""
    G, n, W = 8, 3_000, 40
    cfg = pkg.synth.make_config(n_groups=G, modes=(("1v1", 2, 1),), order=RATING, capacity=n + 100)
    d = cfg.default_group
    assert d >= 1
    ids, rating, mode = uniform_players(4, n, 0, 5000, n_modes=1)
    odd_ids = np.arange(1, 41, dtype=np.uint64)
    odd_rating = np.where(np.arange(40) % 2 == 0, -5, 6000).astype(np.int32)  # below / above every group
    with pkg.Engine(rank_config(pkg, cfg, n + 100)) as eng:
        eng.set_option("max_spread", W)
        assert (eng.enqueue(odd_ids, odd_rating, np.zeros(40, np.uint8)) == 1).all()
        eng.enqueue(ids, rating, mode)
        for g in (d, d + 1):
            if g < G:
                assert not np.isin(odd_ids, eng.band_candidates(W, g)[0]).any()
        lob, mem, taken, st = eng.band_match(W, 0, G - 2)
        assert st.n_matched > 0 and st.n_taken == st.n_matched
        assert not np.isin(odd_ids, mem).any()
        assert eng.in_queue(odd_ids).all() and np.isin(odd_ids, eng.pool_read()["id"]).all()


def refusal(pkg, fn, status, text):
    with pytest.raises(pkg.EngineError) as ex:
        fn()
    assert ex.value.status == status
    assert str(ex.value).endswith(" " + text), str(ex.value)


def twin_state(eng, ids):
    pr = eng.pool_read()
    qs = eng.queue_stats(NOW)
    return dict(pool=[pr[k].copy() for k in ("id", "rating", "mode", "enq_ts")], inq=eng.in_queue(ids),
                active=eng.active_size(), size=eng.pool_size(),
                wait=[qs[k].copy() for k in ("n_waiting", "n_removed", "max_wait", "wait_hist")])


@pytest.mark.gpu
def test_refusals_change_nothing(pkg):
    abi = pkg.abi
    n, W = 3_000, 2
    cfg = make_cfg(pkg, G16, n)
    ids, rating, mode = make_players(pkg, n, 17, G16)
    E_ARG, E_STATE, E_CAP = abi.MM_E_ARG, abi.MM_E_STATE, abi.MM_E_CAP
    engines = [pkg.Engine(rank_config(pkg, cfg, n + 100)) for _ in range(2)]
    try:
        for e in engines:
            e.set_option("max_spread", W)
            e.enqueue(ids, rating, mode)
        eng, twin = engines
        hi = [cfg.group_hi[g] for g in range(G16)]
        B = 6  # boundary 6|7: three upper candidates over both modes (make_players)
        cand = eng.band_candidates(W, B + 1)
        assert len(cand[0]) > 0
        refusal(pkg, lambda: eng.band_candidates(-1, 3), E_ARG, "W must be >= 0")
        refusal(pkg, lambda: eng.band_match(-1, 0, 3), E_ARG, "W must be >= 0")
        refusal(pkg, lambda: eng.band_match(200, 0, 3), E_ARG,
                "rating group 0 is narrower than 2 x W: boundary bands would overlap")
        refusal(pkg, lambda: eng.band_candidates(W, 0), E_ARG,
                f"group 0 has no low boundary: need 1 <= group < n_groups = {G16}")
        refusal(pkg, lambda: eng.band_candidates(W, G16), E_ARG,
                f"group {G16} has no low boundary: need 1 <= group < n_groups = {G16}")
        refusal(pkg, lambda: eng.band_match(W, 5, 4), E_ARG,
                f"boundaries 5..4: need g_first <= g_last < n_groups - 1 = {G16 - 1}")
        refusal(pkg, lambda: eng.band_match(W, 0, G16 - 1), E_ARG,
                f"boundaries 0..{G16 - 1}: need g_first <= g_last < n_groups - 1 = {G16 - 1}")
        # malformed upper columns (another rank's band): order, rating range, mode — checked on the device
        up = eng.band_candidates(W, B + 1)
        bad_order = (up[0][::-1].copy(), up[1][::-1].copy(), up[2][::-1].copy())
        assert len(up[0]) > 1 and not (np.array_equal(bad_order[1], up[1]) and np.array_equal(bad_order[2], up[2]))
        refusal(pkg, lambda: eng.band_match(W, 0, B, bad_order), E_ARG,
                "the upper candidates are not sorted by (mode, rating)")
        for r in (hi[B], hi[B] + W + 1):
            bad = (up[0].copy(), up[1].copy(), up[2].copy())
            bad[1][-1] = r
            refusal(pkg, lambda: eng.band_match(W, 0, B, bad), E_ARG,
                    f"an upper candidate's rating is outside ({hi[B]}, {hi[B] + W}]")
        bad = (up[0].copy(), up[1].copy(), up[2].copy())
        bad[2][-1] = 2
        refusal(pkg, lambda: eng.band_match(W, 0, B, bad), E_ARG, "an upper candidate's mode is >= n_modes")
        # upper columns without upper_remote (raw call)
        lob = np.empty(4, LOBBY_DTYPE)
        mem = np.empty(4, np.uint64)
        tk = np.empty(len(up[0]), np.uint8)
        st = abi.BandStats()
        P = lambda a: a.ctypes.data_as(C.c_void_p)
        rc = eng.lib.mm_band_match(eng.h, W, 0, B, 0, P(up[0]), P(up[1]), P(up[2]), len(up[0]), P(lob), 4, P(mem), 4,
                                   P(tk), C.byref(st))
        assert rc == E_ARG and eng.lib.mm_last_error(eng.h) == b"upper candidates given without upper_remote"
        # a short cap is a dry run: counts, nothing taken
        n_need = C.c_uint32(0)
        rc = eng.lib.mm_band_candidates(eng.h, W, B + 1, None, None, None, 0, C.byref(n_need))
        assert rc == E_CAP and n_need.value == len(cand[0])
        assert eng.lib.mm_last_error(eng.h) == f"need cap >= {len(cand[0])}".encode()
        rc = eng.lib.mm_band_match(eng.h, W, 0, G16 - 2, 0, None, None, None, 0, None, 0, None, 0, None, C.byref(st))
        assert rc == E_CAP and st.n_matched > 0 and st.n_taken == st.n_matched and st.n_upper_taken == 0
        assert eng.lib.mm_last_error(eng.h) == f"need lobby_cap >= {st.n_lobbies} and member_cap >= {st.n_matched}".encode()
        dry = (st.n_lobbies, st.n_matched)
        assert same(twin_state(eng, ids), twin_state(twin, ids))
        # the real call matches what the dry run counted; its twin does the same through the host path
        lobs, mems, _, st2 = eng.band_match(W, 0, G16 - 2)
        assert (st2.n_lobbies, st2.n_matched) == dry and st2.n_taken == st2.n_matched
        ref = shard.boundary_pass(pkg, cfg, W, 1, 0, twin, shard.LocalComm())
        assert np.array_equal(ref["hdr"], lobs) and np.array_equal(ref["member_ids"], mems)
        assert same(twin_state(eng, ids), twin_state(twin, ids))
    finally:
        for e in engines:
            e.close()


@pytest.mark.gpu
def test_refusals_of_engine_state(pkg):
    abi = pkg.abi
    n, W = 2_000, 2
    cfg = make_cfg(pkg, G16, n)
    _, rating, mode = make_players(pkg, n, 19, G16)
    m = len(rating)
    handles = np.arange(m, dtype=np.uint64)
    # arrival order, non-contiguous groups
    with pkg.Engine(rank_config(pkg, cfg, m, order=abi.MM_ORDER_ARRIVAL)) as eng:
        refusal(pkg, lambda: eng.band_candidates(W, 3), abi.MM_E_ARG, "the boundary pass needs MM_ORDER_RATING")
    gap = pkg.synth.make_config(groups=[(0, 99), (200, 299)], order=RATING, capacity=100, default_group=-1)
    with pkg.Engine(gap) as eng:
        refusal(pkg, lambda: eng.band_match(W, 0, 0), abi.MM_E_ARG,
                "the boundary pass needs contiguous ascending rating groups")
    # upper columns on a dense-handle engine; a staged packed batch
    engines = [pkg.Engine(rank_config(pkg, cfg, m, flags=abi.MM_F_DENSE_IDS)) for _ in range(2)]
    try:
        for e in engines:
            e.set_option("max_spread", W)
            e.enqueue(handles, rating, mode)
        eng, twin = engines
        up = eng.band_candidates(W, 5)
        refusal(pkg, lambda: eng.band_match(W, 0, 4, up), abi.MM_E_ARG,
                "upper candidates on an MM_F_DENSE_IDS engine: another engine's handles are not ids here")
        keys = pkg.Engine.pack_key(np.array([cfg.group_hi[3]], np.int32), np.array([0], np.uint8))
        for e in engines:
            e.enqueue_packed_begin(np.array([m + 1], np.uint32), keys)
        staged = "a packed batch is staged: call mm_enqueue_packed_end first"
        refusal(pkg, lambda: eng.band_candidates(W, 5), abi.MM_E_STATE, staged)
        refusal(pkg, lambda: eng.band_match(W, 0, 4), abi.MM_E_STATE, staged)
        for e in engines:
            e.enqueue_packed_end()
        assert same(twin_state(eng, handles), twin_state(twin, handles))
    finally:
        for e in engines:
            e.close()
    # no-dedupe engine: mm_take cannot run there, neither can the pass
    with pkg.Engine(rank_config(pkg, cfg, m, flags=abi.MM_F_NO_DEDUPE)) as eng:
        eng.set_option("max_spread", W)
        eng.enqueue(handles + 5, rating, mode)
        text = "an MM_F_NO_DEDUPE engine cannot take matched players"
        refusal(pkg, lambda: eng.band_candidates(W, 5), abi.MM_E_STATE, text)
        refusal(pkg, lambda: eng.band_match(W, 0, 4), abi.MM_E_STATE, text)
        assert eng.pool_size() == m


# ---- size --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 4])
def test_config3_size_pass_without_a_tick(pkg, K):
    """10 M players, 32 groups, 5v5, W = 2, no tick before the pass: about 2W/157 of the pool are candidates."""
    n, W = 10_000_000, 2
    cfg = pkg.synth.make_config(n_groups=32, modes=(("5v5", 2, 5),), order=RATING, capacity=n)
    ids, rating, mode, _ = pkg.synth.gen_pool(3, n)
    host, dev = compare_paths(pkg, cfg, W, K, ids, rating, mode, tick=False, full_state=False)
    assert sum(d["matched"] for d in dev) > 100_000
