"""Pool compaction by the rows themselves (compact_row, mm_epilogue.cuh).

After placing its tiles a row moves the players it leaves queued into the compacted pool.  The leftovers of
partition p in the rows before row r are a closed form of the placement's slot arithmetic:
    left_before(r, p) = sum over the bins b of p of  min(pre_b, max(0, outbase[b] + pre_b - binlim[b]))
with pre_b the players of bin b in rows before r.  The CPU half restates the tick geometry, the tail's outbase /
binlim and that sum in numpy, and holds the rank every leftover would get against the rank of the same player among
its partition's residual players in the C oracle's output (enqueue order).  The GPU half runs pools whose leftovers
sit in most rows, with rows holding the leftovers of several partitions, and checks the compacted pool, a second
tick on it and the match section of mm_queue_stats bit-exact.
"""
import numpy as np
import pytest

from .test_queue_stats import Model
from .test_tile_geometry import DENSE, MODES8, RATING, ARRIVAL, TILE, WIDE, Device, Geometry, Layout, check, uniform_pool


# ---- numpy restatement ---------------------------------------------------------------------------------------------
def tick_geometry(lay, rating, mode):
    """Geometry of a fresh pool, and every player's partition, bin and row (virtual position = T0[p] * kTile + its
    enqueue index inside the partition; removed players keep their position)."""
    p = lay.partition_of(rating, mode)
    assert (p >= 0).all()
    fills = np.bincount(p, minlength=lay.n_segs)
    g = Geometry(lay, fills)
    T0 = np.concatenate([[0], np.cumsum((fills + TILE - 1) // TILE)])
    order = np.argsort(p, kind="stable")
    start = np.concatenate([[0], np.cumsum(fills)])
    j = np.empty(len(p), np.int64)
    j[order] = np.arange(len(p)) - start[p[order]]
    row = (T0[p] * TILE + j) // TILE // g.tpr
    k = np.clip(np.asarray(rating, np.int64), lay.key_lo, lay.key_lo + lay.KR - 1) - lay.key_lo
    b = np.asarray(mode, np.int64) * lay.stride + lay.lut[k]
    return g, p, b, row


def tail_bounds(lay, cfg, b, alive, matched=None):
    """outbase / binlim of every bin.  S0 (matched None): each (mode, group) cut segment matches the first
    (n // L) * L of its players in sorted order (the shift by earlier partitions' leftovers cancels in left_before).
    S1: a bin's matched players are given (counted from the oracle's lobbies)."""
    tot = np.bincount(b[alive], minlength=lay.K)
    if matched is not None:
        ob = np.concatenate([[0], np.cumsum(matched)[:-1]])
        return ob, ob + matched
    sbb = np.concatenate([[0], np.cumsum(tot)])
    ob, lim = np.zeros(lay.K, np.int64), np.zeros(lay.K, np.int64)
    for c in np.unique(lay.part_cut):
        ps = np.nonzero(lay.part_cut == c)[0]
        b0, b1 = lay.seg_lo[ps[0]], lay.seg_lo[ps[-1] + 1]
        m = c // cfg.n_groups
        L = cfg.modes[m].teams * cfg.modes[m].team_size
        cs, ce = sbb[b0], sbb[b1]
        mend = cs + (ce - cs) // L * L
        ob[b0:b1] = np.minimum(sbb[b0:b1], mend)
        lim[b0:b1] = np.minimum(sbb[b0 + 1:b1 + 1], mend)
    return ob, lim


def left_before(lay, g, b, row, alive, ob, lim):
    """[rows + 1, partitions]: leftovers of partition p in the rows before r (row `rows`: all of them)."""
    M = np.zeros((g.rows, lay.K), np.int64)
    np.add.at(M, (row[alive], b[alive]), 1)
    pre = np.vstack([np.zeros((1, lay.K), np.int64), np.cumsum(M, 0)])
    per_bin = np.minimum(pre, np.maximum(0, ob + pre - lim))
    return np.add.reduceat(per_bin, lay.seg_lo[:-1], axis=1)


def compacted_ranks(lay, g, p, b, row, alive, ob, lim, resid):
    """Rank of every leftover in its partition's part of the compacted pool, as compact_row computes it: left_before
    of its row + its rank among the row's leftovers of the partition (virtual-position order)."""
    lb = left_before(lay, g, b, row, alive, ob, lim)
    idx = np.nonzero(resid)[0]  # input order = virtual-position order inside a partition
    key = p[idx] * (g.rows + 1) + row[idx]
    o = np.argsort(key, kind="stable")
    ks = key[o]
    first = np.searchsorted(ks, ks, side="left")
    k = np.empty(len(idx), np.int64)
    k[o] = np.arange(len(idx)) - first
    return idx, lb[row[idx], p[idx]] + k, lb


def oracle_ranks(p, idx):
    """Rank of each residual player among its partition's residual players in enqueue order."""
    o = np.argsort(p[idx], kind="stable")
    ps = p[idx][o]
    r = np.empty(len(idx), np.int64)
    r[o] = np.arange(len(idx)) - np.searchsorted(ps, ps, side="left")
    return r


def matched_per_bin(lay, b, alive, ids, ref):
    """S1: matched players per bin from the oracle's lobbies; they must be a prefix of the bin in enqueue order."""
    hit = np.isin(ids, ref.member_ids) & alive
    m = np.bincount(b[hit], minlength=lay.K)
    idx = np.nonzero(alive)[0]
    o = np.argsort(b[idx], kind="stable")
    bs = b[idx][o]
    rank = np.arange(len(idx)) - np.searchsorted(bs, bs, side="left")
    assert (hit[idx][o] == (rank < m[bs])).all(), "a bin's matched players are not a prefix in enqueue order"
    return m


def restate(pkg, oracle, cfg, pool, alive, spread):
    ids, rating, mode, _ = pool
    lay = Layout(cfg)
    assert lay.ok
    g, p, b, row = tick_geometry(lay, rating, mode)
    alive = np.asarray(alive, bool)
    a8 = alive.astype(np.uint8)
    ref = oracle.run_windowed(cfg, spread, ids, rating, mode, a8) if spread >= 0 else \
        oracle.run_closed_form(cfg, ids, rating, mode, a8)
    m = matched_per_bin(lay, b, alive, ids, ref) if spread >= 0 else None
    ob, lim = tail_bounds(lay, cfg, b, alive, m)
    resid = np.isin(ids, ref.residual_ids) & alive
    assert resid.sum() == ref.n_residual
    idx, got, lb = compacted_ranks(lay, g, p, b, row, alive, ob, lim, resid)
    assert np.array_equal(got, oracle_ranks(p, idx))
    assert np.array_equal(lb[g.rows], np.bincount(p[idx], minlength=lay.n_segs))  # = n_left of every partition
    rows_with = np.unique(row[idx])
    parts_per_row = np.array([len(np.unique(p[idx][row[idx] == r])) for r in rows_with])
    return g, lay, len(rows_with), int(parts_per_row.max(initial=0))


def eight_by_twenty(pkg, n_big, n_small, seed, dense=False, width=50):
    """8 modes x 20 groups of `width` ratings: mode 0 holds n_big players per group, the other modes n_small (every
    fifth group empty), so rows of a few tiles span several partitions."""
    rng = np.random.default_rng(seed)
    r, m = [], []
    for mo in range(8):
        for gr in range(20):
            k = n_big if mo == 0 else (0 if (3 * mo + gr) % 5 == 2 else n_small)
            r.append(rng.integers(width * gr, width * gr + width, k))
            m.append(np.full(k, mo))
    rating, mode = np.concatenate(r), np.concatenate(m)
    o = rng.permutation(len(rating))
    n = len(rating)
    ids = np.arange(n, dtype=np.uint64) if dense else pkg.synth.mix64(np.arange(n, dtype=np.uint64) + np.uint64(seed << 40))
    return ids, rating[o].astype(np.int32), mode[o].astype(np.uint8), np.arange(n, dtype=np.uint32)


def eight_by_twenty_config(pkg, n, order=RATING, flags=0, width=50):
    return pkg.synth.make_config(groups=[(width * g, width * g + width - 1) for g in range(20)], modes=MODES8,
                                 order=order, capacity=n, active_capacity=2 * n if flags & DENSE else 0, flags=flags)


# ================================================================================ CPU
@pytest.mark.parametrize("order,spread", [(RATING, -1), (ARRIVAL, -1), (RATING, 1)])  # S1: rating order only
def test_left_before_rows_spanning_several_partitions(pkg, oracle, order, spread):
    pool = eight_by_twenty(pkg, 6_000, 700, 3)
    cfg = eight_by_twenty_config(pkg, len(pool[0]), order)
    alive = np.random.default_rng(5).random(len(pool[0])) > 0.03
    g, lay, n_rows, parts = restate(pkg, oracle, cfg, pool, alive, spread)
    assert g.max_parts >= 2 and parts >= 2, g.summary()
    assert n_rows >= g.rows // 2 if spread >= 0 else n_rows >= 20


@pytest.mark.parametrize("spread", [-1, 3])
def test_left_before_partitions_over_many_rows(pkg, oracle, spread):
    """One rating group over the whole pool: partitions span more than 24 rows, the column scan's P holds pre_b."""
    n = 2_000_003
    cfg = pkg.synth.make_config(groups=[(0, 200)], modes=MODES8[3:4], order=RATING, default_group=0, capacity=n)
    pool = uniform_pool(pkg, 8, n, -2, 202)
    alive = np.random.default_rng(6).random(n) > 0.01
    g, lay, n_rows, _ = restate(pkg, oracle, cfg, pool, alive, spread)
    assert g.colscan and g.max_rows > 24, g.summary()
    assert n_rows >= 1


@pytest.mark.parametrize("spread", [-1, 2])
def test_left_before_wide_partitions(pkg, oracle, spread):
    """MM_F_WIDE_PARTITIONS: partitions of more than 255 keys (list ranking)."""
    n = 300_007
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=RATING, capacity=n, flags=WIDE)
    pool = uniform_pool(pkg, 9, n, -20, 5020, n_modes=2)
    alive = np.random.default_rng(7).random(n) > 0.02
    g, lay, n_rows, _ = restate(pkg, oracle, cfg, pool, alive, spread)
    assert lay.max_nb > 255 and not g.halves, g.summary()
    assert n_rows >= 1


# ================================================================================ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True])
@pytest.mark.parametrize("tick_impl,rank_impl", [(1, 3), (0, 3), (1, 2), (0, 2)])
def test_leftovers_in_most_rows(pkg, oracle, tick_impl, rank_impl, dense):
    """Policy S1 with W = 0 on 8 modes x 20 groups: most rows hold leftovers, many of them of several partitions.
    The compacted pool, the match section of mm_queue_stats and a second tick on the compacted pool after removes,
    takes and new arrivals are bit-exact to the oracle."""
    spread = 0
    pool = eight_by_twenty(pkg, 3_000, 600, 11, dense)
    ids, rating, mode, ts = pool
    n = len(ids)
    cfg = eight_by_twenty_config(pkg, n + 100_000, flags=DENSE if dense else 0)
    lay = Layout(cfg, Device.current())
    g, lay, n_rows, parts = restate(pkg, oracle, cfg, pool, np.ones(n, bool), spread)
    assert lay.fused and n_rows >= 0.6 * g.rows and parts >= 2, (n_rows, parts, g.summary())
    ref = oracle.run_windowed(cfg, spread, ids, rating, mode)
    keep = np.isin(ids, ref.residual_ids)
    q_ids, q_r, q_m, q_seq = ids[keep], rating[keep], mode[keep], np.nonzero(keep)[0].astype(np.uint32)
    rng = np.random.default_rng(12)
    gone = rng.random(len(q_ids)) < 0.1
    taken = ~gone & (rng.random(len(q_ids)) < 0.1)
    a_ids, a_r, a_m, a_ts = uniform_pool(pkg, 93, 60_000, 0, 999, n_modes=8, dense=dense)
    a_ids = a_ids + np.uint64(n if dense else 0)
    a_ts = a_ts + np.uint32(n)
    q2 = [np.concatenate([q_ids, a_ids]), np.concatenate([q_r, a_r]), np.concatenate([q_m, a_m])]
    alive2 = np.concatenate([~(gone | taken), np.ones(len(a_ids), bool)]).astype(np.uint8)
    seq2 = np.concatenate([q_seq, n + np.arange(len(a_ids), dtype=np.uint32)])
    ref2 = oracle.run_windowed(cfg, spread, *q2, alive2)
    with pkg.Engine(cfg) as eng:
        eng.set_option("tick_impl", tick_impl)
        eng.set_option("rank_impl", rank_impl)
        eng.set_option("max_spread", spread)
        qm = Model(cfg)
        qm.enqueue(ids, rating, mode, ts, eng.enqueue(ids, rating, mode, ts))
        t1 = 500_000
        lob, mem, seq, st = eng.tick(t1)
        assert st.n_launches == (1 if tick_impl == 1 else 4)
        check(eng, ref, lob, mem, seq, st)
        qm.tick(lob, mem, t1)
        qm.check(eng.queue_stats(t1), t1)
        assert eng.remove(q_ids[gone]) == int(gone.sum())
        assert eng.take(q_ids[taken]) == int(taken.sum())
        qm.remove(q_ids[gone | taken])
        qm.enqueue(a_ids, a_r, a_m, a_ts, eng.enqueue(a_ids, a_r, a_m, a_ts))
        t2 = t1 + 4321
        lob, mem, seq, st = eng.tick(t2)
        check(eng, ref2, lob, mem, seq, st, seq_of=seq2)
        qm.tick(lob, mem, t2)
        qm.check(eng.queue_stats(t2), t2)
