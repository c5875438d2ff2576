"""Every form the tick's results take, and long mixed schedules, against the oracle and a serialized restatement.

A fused tick asked for emission order meets at grid barrier 2 and writes the lobby headers in `epilogue_body`;
without it (mm_tick / mm_tick_packed with emit_seq NULL, mm_tick_device) the rows write them after compacting their
leftovers, in 8 192-lobby chunks claimed from `TickCtr::hdr_next` (`headers_claimed`).  The split tick writes them
in `k_epilogue`.  Each pool here is ticked through every entry point on both tick implementations, and each result is
held bit-exact to the oracle, with the result buffers poisoned before the tick so that a header or member the tick
does not write shows.  The pools reach the edges of the chunk claim: one row (no helper CTA), a few rows, the full
grid, lobby totals at 8 192 +- 1 and up to about 1 M, empty partitions between and after non-empty ones, and lobbies
that start in one partition of a wide group and end in the next.

`Model` extends the ingest restatement (tests/test_ingest.py) with policy S1 ticks (the oracle's windowed run), the
match section of mm_queue_stats (checked by the restatement of tests/test_queue_stats.py) and mm_snapshot /
mm_restore.  The schedules draw one operation per step, switch tick_impl, rank_impl, max_spread and async_results
between ticks of one engine, mix every tick and enqueue entry point, and compare everything the engine reports after
every step.  A restore brings back the active set as it was at the snapshot, not only the pool.
"""
import numpy as np
import pytest

from .test_ingest import Model as IngestModel, Refused
from .test_queue_stats import Model as StatsModel
from .test_tile_geometry import DENSE, MODES8, WIDE, Device, Geometry, Layout, NumpyTick

ARRIVAL, RATING = 0, 1
HDR_CHUNK = 8192  # kHdrChunk (mm_epilogue.cuh)


# ---- the restatement ------------------------------------------------------------------------------------------------
class Model(IngestModel):
    """The ingest restatement, plus: policy S1 ticks (spread >= 0: the oracle's windowed run; the entries left queued
    are the oracle's residual players), the last tick's matched players for mm_queue_stats, and a snapshot (queued
    entries, active set, sequence counter)."""

    def __init__(self, cfg, oracle, abi, spread=-1):
        super().__init__(cfg, oracle, abi)
        self.spread = spread
        self.match = None
        self.snap = None

    def tick_ref(self, literal_max=100_000):
        q = self.q
        alive = q["alive"].astype(np.uint8)
        if self.spread >= 0:
            return self.oracle.run_windowed(self.cfg, self.spread, q["id"], q["rating"], q["mode"], alive), q["seq"].copy()
        if self.slots() > 2_000_000:  # the C oracle's closed form is slow at config3's size; NumpyTick restates it
            return NumpyTick(self.cfg, q["id"], q["rating"], q["mode"], alive), q["seq"].copy()
        return super().tick_ref(literal_max)

    def after_tick(self, ref, now=0):
        q, G = self.q, self.cfg.n_groups
        keep = self.residual_mask() if self.spread < 0 else q["alive"] & np.isin(q["id"], ref.residual_ids)
        assert np.array_equal(q["id"][keep], ref.residual_ids)
        hit = q["alive"] & ~keep
        assert hit.sum() == ref.n_matched
        lob_cut = ref.lobbies["mode"].astype(np.int64) * G + ref.lobbies["group"]
        self.match = (q["mode"][hit].astype(np.int64) * G + self.groups(q["rating"][hit]), q["ts"][hit].copy(), now,
                      np.bincount(lob_cut, minlength=self.cfg.n_modes * G))
        self.q = {k: v[keep] for k, v in q.items()}

    def snapshot(self):
        self.snap = ({k: v.copy() for k, v in self.q.items()}, self.active.copy(), self.seq_next)

    def restore(self):
        q, active, self.seq_next = self.snap
        self.q = {k: v.copy() for k, v in q.items()}
        self.active = active.copy()
        self.match = None  # mm_restore voids the last tick's match section

    def check_queue_stats(self, st, now):
        """Both sections of mm_queue_stats, by the restatement of tests/test_queue_stats.py."""
        q = self.q
        sm = StatsModel(self.cfg)
        sm.id = q["id"]
        sm.cut = q["mode"].astype(np.int64) * self.cfg.n_groups + self.groups(q["rating"])
        sm.ts = q["ts"]
        sm.state = np.where(q["alive"], sm.QUEUED, sm.DEAD).astype(np.uint8)
        sm.match = self.match
        sm.check(st, now)


def check_state(eng, m, now, sample=(), stats=True):
    """Everything the engine reports between ticks, against the model (mm_queue_stats's counts only unless stats)."""
    ridx, rcode = m.rejects()
    idx, code = eng.enqueue_rejects(cap=max(len(ridx), 1))
    o = np.argsort(idx)
    assert np.array_equal(idx[o], ridx) and np.array_equal(code[o], rcode)
    assert eng.pool_size() == m.slots()
    assert eng.active_size() == len(m.active)
    sample = np.asarray(sample, np.uint64)
    if m.dedupe and len(sample):
        assert np.array_equal(eng.in_queue(sample), m.in_queue(sample))
    got, want = eng.pool_read(), m.pool()
    for k in want:
        assert np.array_equal(got[k], want[k]), k
    qs = eng.queue_stats(now)
    if stats:
        m.check_queue_stats(qs, now)
    else:
        n_wait, n_rem = m.queue_counts()
        assert np.array_equal(qs["n_waiting"], n_wait) and np.array_equal(qs["n_removed"], n_rem)


def check_tick(ref, seq_of, lob, mem, seq, st, fused=None):
    assert (st.n_lobbies, st.n_matched, st.n_residual, st.n_dead) == \
        (ref.n_lobbies, ref.n_matched, ref.n_residual, ref.n_dead)
    if fused is not None:
        assert st.n_launches == (1 if fused else 4)
    bad = np.nonzero(lob != ref.lobbies)[0]
    assert not len(bad), f"{len(bad)} lobby headers differ, first at {bad[:5]}: {lob[bad[:3]]} != {ref.lobbies[bad[:3]]}"
    assert np.array_equal(np.asarray(mem, np.uint64), ref.member_ids)
    if seq is not None:
        assert np.array_equal(seq, seq_of[ref.emit_seq])


# ---- device buffers ---------------------------------------------------------------------------------------------------
def device_view(ptr, n, typestr):
    """torch view of n elements at a device address (the engine's result buffers)."""
    import torch

    class _View:
        __cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "strides": None,
                                    "version": 2}
    return torch.as_tensor(_View(), device="cuda")


def device_results(eng, st, pkg):
    """mm_results_device: the last tick's headers and members, read from HBM."""
    p_lob, p_mem = eng.results_device()
    lob = device_view(p_lob, st.n_lobbies, "<i8").cpu().numpy().view(pkg.engine.LOBBY_DTYPE) if st.n_lobbies else \
        np.zeros(0, pkg.engine.LOBBY_DTYPE)
    mem = device_view(p_mem, st.n_matched, "<i8").cpu().numpy().view(np.uint64) if st.n_matched else \
        np.zeros(0, np.uint64)
    return lob, mem


def poison(eng, n_lob, n_mem):
    """All ones over the first n_lob headers and n_mem members of the result buffers the next tick writes (no host
    copy of an earlier tick may be pending).  The engine holds capacity / min L + 1 headers and capacity + 64 members."""
    import torch
    cfg = eng.cfg
    min_l = min(cfg.modes[k].teams * cfg.modes[k].team_size for k in range(cfg.n_modes))
    n_lob, n_mem = min(n_lob, cfg.capacity // min_l + 1), min(n_mem, cfg.capacity + 64)
    p_lob, p_mem = eng.results_device()
    if n_lob:
        device_view(p_lob, n_lob, "<i8").fill_(-1)
    if n_mem:
        device_view(p_mem, n_mem, "<i8").fill_(-1)
    torch.cuda.synchronize()  # the engine's stream does not wait for torch's


# ---- tick forms -----------------------------------------------------------------------------------------------------
HOST_FORMS = ("tick_emit", "tick", "packed_emit", "packed", "device")


def tick_form(pkg, eng, form, now):
    """One tick through `form` -> (lobbies, member ids u64, emit_seq or None, stats)."""
    if form in ("tick_emit", "tick"):
        return eng.tick(now, want_emit_seq=form == "tick_emit")
    if form in ("packed_emit", "packed"):
        lob, mem, seq, st = eng.tick_packed(now, want_emit_seq=form == "packed_emit")
        return lob, mem.astype(np.uint64), seq, st
    assert form == "device"
    st = eng.tick_device(now)
    lob, mem = device_results(eng, st, pkg)
    return lob, mem, None, st


class AsyncTicks:
    """async_results: mm_tick / mm_tick_packed into pinned host arrays that alternate between ticks; tick k's arrays
    are read once tick k + 1 has returned (or after mm_results_wait)."""

    def __init__(self, pkg, eng, n_slots):
        import torch
        self.pkg, self.eng = pkg, eng
        self.lob_cap, self.mem_cap = max(n_slots // 2, 1), max(n_slots, 1)
        self.lob = [torch.empty(self.lob_cap, dtype=torch.int64).pin_memory() for _ in range(2)]
        self.mem = [torch.empty(self.mem_cap, dtype=torch.int64).pin_memory() for _ in range(2)]
        self.k = 0
        self.pending = None  # (k, packed, expected...) of the tick whose host arrays are not yet complete

    def tick(self, packed, now, want):
        """Run a tick; `want` = (ref, seq_of) it must equal.  Returns its stats; the previous tick's arrays are checked."""
        k = self.k & 1
        self.lob[k].fill_(-1); self.mem[k].fill_(-1)
        st = self.eng.tick_raw(self.lob[k].data_ptr(), self.lob_cap, self.mem[k].data_ptr(), self.mem_cap, now=now,
                               packed=packed)
        self.check_pending()
        self.pending = (k, packed, st, want)
        self.k += 1
        return st

    def check_pending(self):
        if self.pending is None:
            return
        k, packed, st, (ref, seq_of) = self.pending
        lob = self.lob[k].numpy()[:st.n_lobbies].view(self.pkg.engine.LOBBY_DTYPE)
        mem = self.mem[k].numpy().view(np.uint32 if packed else np.uint64)[:st.n_matched]
        check_tick(ref, seq_of, lob, mem, None, st)
        self.pending = None

    def wait(self):
        self.eng.results_wait()
        self.check_pending()


# ---- pools at the edges of the header chunk claim ---------------------------------------------------------------------
def counts_pool(rng, counts, lo_hi, mode_of, first_id=0):
    """Players of given counts per (mode, rating range), shuffled into one arrival order."""
    r, m = [], []
    for (mo, (lo, hi)), k in zip([(mode_of[i], lo_hi[i]) for i in range(len(counts))], counts):
        r.append(rng.integers(lo, hi + 1, k))
        m.append(np.full(k, mo))
    rating, mode = np.concatenate(r).astype(np.int32), np.concatenate(m).astype(np.uint8)
    o = rng.permutation(len(rating))
    n = len(rating)
    return (np.arange(first_id, first_id + n, dtype=np.uint64), rating[o], mode[o],
            rng.integers(0, 1000, n).astype(np.uint32))


def lobbies_shape(total, rng):
    """1v1 over six groups of 100 ratings: the lobbies of groups 0, 2 and 3 add up to `total`; groups 1, 4 and 5 hold
    one player each (empty partitions between and after non-empty ones)."""
    a = total // 3
    lob = [a, 0, a, total - 2 * a, 0, 0]
    counts = [2 * x + (1 if x == 0 else int(rng.integers(0, 2))) for x in lob]
    groups = [(100 * g, 100 * g + 99) for g in range(6)]
    return groups, counts


LOBBY_TOTALS = {"lob8191": 8191, "lob8192": 8192, "lob8193": 8193, "lob5chunks": 5 * HDR_CHUNK + 17}


def make_shape(pkg, name, order, seed):
    """-> (cfg, pool, alive, regime check(geometry, layout, ref)) of a named pool shape."""
    rng = np.random.default_rng(seed)
    syn = pkg.synth
    if name in LOBBY_TOTALS:
        total = LOBBY_TOTALS[name]
        groups, counts = lobbies_shape(total, rng)
        pool = counts_pool(rng, counts, groups, [0] * 6)
        cfg = syn.make_config(groups=groups, modes=MODES8[:1], order=order, capacity=len(pool[0]),
                              default_group=-1)
        alive = np.ones(len(pool[0]), bool)

        def regime(g, lay, ref):
            lob = np.bincount(ref.lobbies["group"], minlength=6)
            assert ref.n_lobbies == total and (lob[[1, 4, 5]] == 0).all() and (lob[[0, 2, 3]] > 0).all()
        return cfg, pool, alive, regime
    if name == "one_row":
        groups = [(0, 200)]
        pool = counts_pool(rng, [1999], groups, [0])
        cfg = syn.make_config(groups=groups, modes=MODES8[:1], order=order, capacity=4000, default_group=-1)

        def regime(g, lay, ref):
            assert g.rows == 1 and lay.n_segs == 1 and ref.n_lobbies > 900
    elif name == "few_rows":
        groups = [(250 * g, 250 * g + 249) for g in range(8)]
        counts = [int(x) for x in rng.integers(3000, 12000, 16)]
        counts[5] = 0
        pool = counts_pool(rng, counts, groups * 2, [0] * 8 + [1] * 8)
        cfg = syn.make_config(groups=groups, modes=(MODES8[0], MODES8[3]), order=order, capacity=len(pool[0]),
                              default_group=-1)

        def regime(g, lay, ref):
            assert 2 <= g.rows < 64 and ref.n_lobbies > HDR_CHUNK
    elif name == "full_grid":
        groups = [(160 * g, 160 * g + 159) for g in range(31)]
        n = 1_200_000
        pool = counts_pool(rng, [n // 31] * 31, groups, [0] * 31)
        cfg = syn.make_config(groups=groups, modes=MODES8[:1], order=order, capacity=n, default_group=-1)

        def regime(g, lay, ref):
            assert g.rows == lay.tick_rows(10 ** 9) and g.rows >= 64 and ref.n_lobbies > 60 * HDR_CHUNK
    elif name == "wide_group":
        # one 1 000-rating group of 5v5 stored as 4 partitions: lobbies start in one partition and end in the next
        groups = [(0, 999), (1000, 1099)]
        pool = counts_pool(rng, [200_003, 4], groups, [0, 0])
        cfg = syn.make_config(groups=groups, modes=MODES8[3:4], order=order, capacity=len(pool[0]), default_group=-1)

        def regime(g, lay, ref):
            assert ref.n_lobbies > 2 * HDR_CHUNK and ref.lobbies["group"][-1] == 0
            if order == RATING:  # group 0's partitions do not end on lobby boundaries: lobbies straddle them
                fills = lay.fills(pool[1], pool[2])
                assert lay.n_segs == 5 and lay.max_nb <= 255 and (np.cumsum(fills[:3]) % 10 != 0).any()
    else:
        assert name == "no_lobbies"
        groups = [(100 * g, 100 * g + 99) for g in range(40)]
        pool = counts_pool(rng, [int(x) for x in rng.integers(0, 10, 40)], groups, [0] * 40)
        cfg = syn.make_config(groups=groups, modes=MODES8[3:4], order=order, capacity=1000, default_group=-1)

        def regime(g, lay, ref):
            assert ref.n_lobbies == 0 and ref.n_residual > 100
    alive = np.ones(len(pool[0]), bool)
    return cfg, pool, alive, regime


def dense_config(pkg, cfg, active):
    c = pkg.synth.make_config(groups=[(cfg.group_lo[g], cfg.group_hi[g]) for g in range(cfg.n_groups)],
                              modes=[("m", cfg.modes[m].teams, cfg.modes[m].team_size) for m in range(cfg.n_modes)],
                              order=cfg.order_mode, capacity=cfg.capacity, active_capacity=active,
                              default_group=cfg.default_group, flags=cfg.flags | DENSE)
    return c


def run_forms(pkg, oracle, cfg, pool, alive, spread, regime=None, dense=True, impls=(1, 0)):
    """One pool, ticked through every form on both tick implementations from one snapshot; each tick bit-exact to
    the model (oracle), and everything the engine reports after it too."""
    ids, rating, mode, ts = pool
    m = Model(cfg, oracle, pkg.abi, spread)
    now = 1_000_000
    big = len(ids) > 2_000_000  # config3: the queue-stats restatement of 10 M players runs once per implementation
    with pkg.Engine(cfg) as eng:
        if spread >= 0:
            eng.set_option("max_spread", spread)
        if dense:
            acc = eng.enqueue_packed(ids.astype(np.uint32), eng.pack_key(rating, mode), ts)
        else:
            acc = eng.enqueue(ids, rating, mode, ts)
        assert np.array_equal(acc, m.enqueue(ids, rating, mode, ts))
        gone = ids[~alive]
        assert eng.remove(gone) == m.remove(gone)
        eng.snapshot()
        m.snapshot()
        ref, seq_of = m.tick_ref()
        lay = Layout(cfg, Device.current())
        g = Geometry(lay, lay.fills(rating, mode), n=m.slots())
        if regime is not None:
            regime(g, lay, ref)
        m.after_tick(ref, now)  # the state after the tick, the same for every form
        ticked = (m.q, m.match)
        sample = np.concatenate([ids[:200], ids[-200:], gone[:50]])

        def after_tick():
            m.q, m.match = {k: v.copy() for k, v in ticked[0].items()}, ticked[1]

        forms = HOST_FORMS if dense else ("tick_emit", "tick", "device")
        for impl in impls:
            eng.set_option("tick_impl", impl)
            fused = impl == 1 and lay.fused
            for i, form in enumerate(forms):
                eng.restore(); m.restore()
                if i == 0:
                    check_state(eng, m, now, sample)
                poison(eng, ref.n_lobbies + 64, ref.n_matched + 64)
                lob, mem, seq, st = tick_form(pkg, eng, form, now)
                check_tick(ref, seq_of, lob, mem, seq, st, fused)
                after_tick()
                check_state(eng, m, now + 5, sample, stats=i == 0 or not big)
            # async_results: two ticks of the same pool into alternating host arrays; the first one's arrays are read
            # after the second has returned (packed: its kernels ran while the first one's copies were in flight)
            for packed in ((False, True) if dense else (False,)):
                eng.set_option("async_results", 1)
                at = AsyncTicks(pkg, eng, cfg.capacity)
                for _ in range(2):
                    eng.restore(); m.restore()
                    st = at.tick(packed, now, (ref, seq_of))
                    assert st.n_launches == (1 if fused else 4)
                    after_tick()
                    check_state(eng, m, now + 5, sample, stats=not big)
                at.wait()
                eng.set_option("async_results", 0)
    return ref


# ================================================================================ CPU: the model against the oracle
def small_pool(pkg, rng, n, n_modes=3, first=0):
    ids = pkg.synth.mix64(np.arange(first, first + n, dtype=np.uint64) + np.uint64(77 << 40))
    return ids, rng.integers(0, 5200, n).astype(np.int32), rng.integers(0, n_modes, n).astype(np.uint8), \
        rng.integers(0, 1000, n).astype(np.uint32)


@pytest.mark.parametrize("spread", [0, 2, 40])
def test_model_s1_ticks_equal_the_oracle(pkg, oracle, spread):
    """S1 in the model: the residual entries are the oracle's, in enqueue order, over ticks with removes, takes and
    repeats of matched and removed ids in between; every lobby spans at most `spread` ratings."""
    rng = np.random.default_rng(spread)
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[:3], order=RATING, capacity=30_000,
                                default_group=-1)
    m = Model(cfg, oracle, pkg.abi, spread)
    ids, rating, mode, ts = small_pool(pkg, rng, 40_000)
    m.enqueue(ids[:20_000], rating[:20_000], mode[:20_000], ts[:20_000])
    for step in range(4):
        q = m.q["id"][m.q["alive"]]
        m.remove(q[rng.choice(len(q), 300)])
        m.take(q[rng.choice(len(q), 200)])
        ref, seq_of = m.tick_ref()
        rq = m.q["rating"][m.q["alive"]].astype(np.int64)
        by_id = dict(zip(m.q["id"][m.q["alive"]].tolist(), rq.tolist()))
        r = np.array([by_id[int(x)] for x in ref.member_ids], np.int64)
        for h in ref.lobbies[:2000]:
            seg = r[h["first_member"]:h["first_member"] + h["n_members"]]
            assert seg.max() - seg.min() <= spread
        before = m.slots()
        m.after_tick(ref, step)
        assert m.slots() == ref.n_residual and before - m.slots() == ref.n_matched + ref.n_dead
        assert m.match[0].size == ref.n_matched and m.match[3].sum() == ref.n_lobbies
        k = 5000 * step
        again = np.concatenate([ids[20_000 + k:25_000 + k], ref.member_ids[:100], q[:100]])
        m.enqueue(again, rng.integers(0, 5200, len(again)), rng.integers(0, 3, len(again)))


def test_model_s0_tick_equals_numpy_tick_and_oracle(pkg, oracle):
    """The model's two S0 references (the C oracle, NumpyTick for the largest pools) agree on a pool with dead
    entries, and the entries left queued are the oracle's residual players."""
    rng = np.random.default_rng(4)
    for order in (ARRIVAL, RATING):
        cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[:3], order=order, capacity=50_000,
                                    default_group=-1)
        m = Model(cfg, oracle, pkg.abi)
        ids, rating, mode, ts = small_pool(pkg, rng, 50_000)
        m.enqueue(ids, rating, mode, ts)
        m.remove(ids[::13])
        ref, seq_of = m.tick_ref()
        q = m.q
        nt = NumpyTick(cfg, q["id"], q["rating"], q["mode"], q["alive"])
        for f in ("lobbies", "member_ids", "emit_seq", "residual_ids"):
            assert np.array_equal(getattr(nt, f), getattr(ref, f)), f
        m.after_tick(ref)


def test_model_snapshot_restores_everything(pkg, oracle):
    """Snapshot / restore in the model: the queued entries, the active set and the sequence counter come back after
    enqueues, removes, takes and ticks, and twice from one snapshot; the reject list and the match section do not."""
    rng = np.random.default_rng(8)
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=RATING, capacity=5000, default_group=-1)
    m = Model(cfg, oracle, pkg.abi)
    ids, rating, mode, ts = small_pool(pkg, rng, 9000, n_modes=2)
    m.enqueue(ids[:3000], rating[:3000], mode[:3000], ts[:3000])
    m.after_tick(m.tick_ref()[0])
    m.snapshot()
    state = ({k: v.copy() for k, v in m.q.items()}, np.sort(m.active), m.seq_next)
    for _ in range(2):
        code = m.enqueue(ids[3000:6000], rating[3000:6000], mode[3000:6000])
        m.remove(ids[:1000]); m.take(ids[1000:1500])
        m.after_tick(m.tick_ref()[0], 9)
        codes = m.codes.copy()
        m.restore()
        for k in state[0]:
            assert np.array_equal(m.q[k], state[0][k])
        assert np.array_equal(np.sort(m.active), state[1]) and m.seq_next == state[2] and m.match is None
        assert np.array_equal(m.codes, codes)
        assert np.array_equal(m.enqueue(ids[3000:6000], rating[3000:6000], mode[3000:6000]), code)
        m.restore()


def test_shapes_reach_their_regimes_on_h100(pkg, oracle):
    """The CPU half of the form tests' regime checks, on the H100 SXM geometry (132 SMs)."""
    for name in ("one_row", "few_rows", "lob8191", "lob8193", "wide_group", "no_lobbies"):
        for order in (RATING, ARRIVAL):
            cfg, pool, alive, regime = make_shape(pkg, name, order, 3)
            m = Model(cfg, oracle, pkg.abi)
            assert (m.enqueue(*pool) == 1).all()
            lay = Layout(cfg)
            regime(Geometry(lay, lay.fills(pool[1], pool[2])), lay, m.tick_ref()[0])


# ================================================================================ GPU: every result form
@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
@pytest.mark.parametrize("name", ["one_row", "few_rows", "full_grid", "lob8191", "lob8192", "lob8193", "lob5chunks",
                                  "wide_group", "no_lobbies"])
def test_result_forms_equal_the_oracle(pkg, oracle, name, order):
    cfg, pool, alive, regime = make_shape(pkg, name, order, 11)
    alive = alive & (np.random.default_rng(2).random(len(alive)) > 0.01) if name in ("few_rows", "full_grid") else alive
    n = len(pool[0])
    run_forms(pkg, oracle, dense_config(pkg, cfg, n + 64), pool, alive, -1, regime)
    if name in ("few_rows", "lob8193", "wide_group"):  # hashed active set: the compaction re-stamps through the table
        run_forms(pkg, oracle, cfg, (pkg.synth.mix64(pool[0]),) + pool[1:], alive, -1, regime, dense=False)


@pytest.mark.gpu
@pytest.mark.parametrize("name,spread", [("few_rows", 0), ("few_rows", 7), ("wide_group", 3), ("lob8193", 1)])
def test_result_forms_s1_equal_the_oracle(pkg, oracle, name, spread):
    cfg, pool, alive, _ = make_shape(pkg, name, RATING, 12)
    ref = run_forms(pkg, oracle, dense_config(pkg, cfg, len(pool[0]) + 64), pool, alive, spread)
    assert ref.n_lobbies > 0 and ref.n_residual > 0


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
def test_result_forms_config3_ten_million(pkg, oracle, order):
    """BASELINE config3 (10 M players, 5v5, 32 groups): about 1 M lobbies, 122 header chunks, the full grid."""
    n = 10_000_000
    cfg = pkg.synth.make_config(n_groups=32, modes=MODES8[3:4], order=order, capacity=n, active_capacity=n,
                                flags=DENSE)
    _, rating, _, _ = pkg.synth.gen_pool(1, n)
    pool = (np.arange(n, dtype=np.uint64), rating, np.zeros(n, np.uint8), (np.arange(n) % 977).astype(np.uint32))

    def regime(g, lay, ref):
        assert g.rows >= 64 and ref.n_lobbies > 120 * HDR_CHUNK

    run_forms(pkg, oracle, cfg, pool, np.ones(n, bool), -1, regime)


# ================================================================================ GPU: restore restores the active set
def restore_engine(pkg, dense, cap=20_000, active=200_000):
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=RATING, capacity=cap, active_capacity=active,
                                default_group=-1, flags=DENSE if dense else 0)
    return cfg


RESTORE_AFTER = ("enqueue_remove", "take", "ticks", "twice", "async")


def ids_of(pkg, dense, k0, k1):
    x = np.arange(k0, k1, dtype=np.uint64)
    return x if dense else pkg.synth.mix64(x + np.uint64(5 << 40))


@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True])
@pytest.mark.parametrize("what", RESTORE_AFTER)
def test_restore_brings_back_the_active_set(pkg, oracle, dense, what):
    """After mm_restore, an id enqueued since the snapshot is accepted again (code 1), an id removed since is queued
    again and mm_remove drops it, and active_size is its value at the snapshot."""
    rng = np.random.default_rng(RESTORE_AFTER.index(what) + 10 * dense)
    cfg = restore_engine(pkg, dense)
    m = Model(cfg, oracle, pkg.abi)
    with pkg.Engine(cfg) as eng:
        def enq(ids, now=0):
            r = rng.integers(0, 5001, len(ids)).astype(np.int32)
            mo = rng.integers(0, 2, len(ids)).astype(np.uint8)
            ts = np.full(len(ids), now, np.uint32)
            assert np.array_equal(eng.enqueue(ids, r, mo, ts), m.enqueue(ids, r, mo, ts))

        def tick(now):
            ref, seq_of = m.tick_ref()
            check_tick(ref, seq_of, *eng.tick(now))
            m.after_tick(ref, now)

        first = ids_of(pkg, dense, 0, 12_000)
        enq(first)
        tick(10)
        enq(ids_of(pkg, dense, 12_000, 15_000), 11)
        if what == "async":
            eng.set_option("async_results", 1)
            at = AsyncTicks(pkg, eng, cfg.capacity)
            ref, seq_of = m.tick_ref()
            at.tick(dense, 14, (ref, seq_of))
            m.after_tick(ref, 14)
            enq(ids_of(pkg, dense, 15_000, 18_000), 14)  # the next batch and the snapshot while the tick's host
            eng.snapshot(); m.snapshot()                 # copies are in flight
            at.wait()
            eng.set_option("async_results", 0)
        else:
            eng.snapshot(); m.snapshot()
        snap_active = eng.active_size()
        assert snap_active == len(m.active)
        queued = m.q["id"][m.q["alive"]].copy()
        matched = np.setdiff1d(m.active, queued)
        new = ids_of(pkg, dense, 20_000, 21_500)
        gone = np.concatenate([queued[:300], matched[:200]])
        rounds = 2 if what == "twice" else 1
        for rnd in range(rounds):
            enq(new, 20)
            assert eng.remove(gone) == m.remove(gone)
            if what == "take":
                took = m.q["id"][m.q["alive"]][:400]
                assert eng.take(took) == m.take(took)
            if what in ("ticks", "twice"):
                for k in range(3):
                    tick(30 + k)
                    enq(ids_of(pkg, dense, 22_000 + 500 * k, 22_500 + 500 * k), 31 + k)
            eng.restore(); m.restore()
            assert eng.active_size() == snap_active
            check_state(eng, m, 40, np.concatenate([new[:200], gone]))
            assert eng.in_queue(gone).all() and not eng.in_queue(new).any()
        # the ids enqueued since the snapshot are accepted again; the removed ones are queued and removable
        r = rng.integers(0, 5001, len(new)).astype(np.int32)
        mo = np.zeros(len(new), np.uint8)
        code = eng.enqueue(new, r, mo)
        assert np.array_equal(code, m.enqueue(new, r, mo)) and (code == 1).all()
        assert eng.remove(queued[:300]) == m.remove(queued[:300]) == 300
        check_state(eng, m, 41, np.concatenate([new[:200], gone]))
        tick(50)
        check_state(eng, m, 50, gone)


@pytest.mark.gpu
def test_restore_after_a_rehash_forced_by_tombstones(pkg, oracle):
    """A rehash between snapshot and restore switches the current hashed table: the restore writes the table that is
    current, and the refusal rule counts the snapshot's ids and tombstones again."""
    from .test_ingest import hashed_slots
    rng = np.random.default_rng(6)
    cfg = pkg.synth.make_config(n_groups=8, default_group=-1, order=ARRIVAL, capacity=200_000, active_capacity=300_000)
    limit = hashed_slots(cfg) * 3 // 4
    m = Model(cfg, oracle, pkg.abi)
    with pkg.Engine(cfg) as eng:
        def enq(ids):
            r = rng.integers(0, 5001, len(ids)).astype(np.int32)
            mo = rng.integers(0, 2, len(ids)).astype(np.uint8)
            try:
                want = m.enqueue(ids, r, mo)
            except Refused:
                with pytest.raises(pkg.EngineError):
                    eng.enqueue(ids, r, mo)
                return None
            assert np.array_equal(eng.enqueue(ids, r, mo), want)
            return want

        a = ids_of(pkg, False, 0, 150_000)
        enq(a)
        eng.snapshot(); m.snapshot()
        assert eng.remove(a[:140_000]) == m.remove(a[:140_000])  # tombstones
        ref, _ = m.tick_ref(); eng.tick(); m.after_tick(ref)
        b = ids_of(pkg, False, 1_000_000, 1_000_000 + limit - len(m.active) - 1000)
        assert len(m.active) + 140_000 + len(b) > limit  # this batch rehashes first
        enq(b)
        eng.restore(); m.restore()
        assert eng.active_size() == 150_000
        check_state(eng, m, 0, np.concatenate([a[::100], b[::1000]]))
        assert enq(b[:limit - 150_000 + 1]) is None  # refused: the restored ids count again
        enq(b[:limit - 150_000 - 10])
        assert eng.remove(a[:10]) == 10 == m.remove(a[:10])
        check_state(eng, m, 0, np.concatenate([a[::100], b[::1000]]))
        ref, seq_of = m.tick_ref()
        check_tick(ref, seq_of, *eng.tick())


# ================================================================================ GPU: long mixed schedules
class Schedule:
    """One engine and the model, driven by a random schedule; every step is compared in full."""

    def __init__(self, pkg, oracle, cfg, rng, dense):
        self.pkg, self.cfg, self.rng, self.dense = pkg, cfg, rng, dense
        self.eng = pkg.Engine(cfg)
        self.m = Model(cfg, oracle, pkg.abi)
        self.async_on, self.at = False, None
        self.tick_impl = 1
        self.now = 1000
        self.next_id = 0
        self.id_space = cfg.active_capacity if dense else 1 << 40
        self.seen = np.zeros(0, np.uint64)
        self.counts = {}

    def close(self):
        self.eng.close()

    def fresh(self, n):
        x = np.arange(self.next_id, self.next_id + n, dtype=np.uint64)
        self.next_id += n
        assert self.next_id < self.id_space
        return x if self.dense else self.pkg.synth.mix64(x)

    def pick(self, n):
        """Ids of every kind: fresh, queued, matched (active, not queued), removed, unknown, repeated."""
        rng, m = self.rng, self.m
        k = n // 4 if len(self.seen) else 0
        parts = [self.fresh(n - k)]
        if k:
            parts.append(rng.choice(self.seen, k))
        ids = np.concatenate(parts)
        rep = rng.random(len(ids)) < 0.01
        ids[rep] = ids[rng.integers(0, len(ids), int(rep.sum()))]
        rng.shuffle(ids)
        self.seen = np.concatenate([self.seen, ids[:2000]])[-50_000:]
        return ids

    def sample(self):
        q = self.m.q["id"]
        parts = [self.seen[-300:], q[:: max(1, len(q) // 300)], self.m.active[:: max(1, len(self.m.active) // 300)]]
        return np.concatenate(parts)

    # ---- operations -------------------------------------------------------------------------------------------------
    def enqueue(self, n):
        rng, cfg = self.rng, self.cfg
        ids = self.pick(n)
        rating = rng.integers(0, 5200, n).astype(np.int32)  # 5001 .. 5199: no group, no default group
        mode = rng.integers(0, cfg.n_modes, n).astype(np.uint8)
        mode[rng.random(n) < 0.005] = cfg.n_modes  # not configured: invalid
        ts = (self.now - rng.integers(0, 500, n)).astype(np.uint32)
        if self.dense:
            ids[rng.random(n) < 0.002] = np.uint64(cfg.active_capacity + 5)  # past the handle range: invalid
            form = rng.choice(["host", "device", "packed", "staged"])
        else:
            ids[rng.random(n) < 0.002] = np.uint64(2 ** 64 - 1)
            form = rng.choice(["host", "device"])
        self.counts[f"enq_{form}"] = self.counts.get(f"enq_{form}", 0) + 1
        try:
            want = self.m.enqueue(ids, rating, mode, ts)
        except Refused:
            with pytest.raises(self.pkg.EngineError) as ei:
                self.engine_enqueue(form, ids, rating, mode, ts)
            assert ei.value.status == self.pkg.abi.MM_E_CAP
            return
        acc = self.engine_enqueue(form, ids, rating, mode, ts)
        if acc is not None:
            bad = np.nonzero(acc != want)[0]
            assert not len(bad), (form, bad[:8], acc[bad[:8]], want[bad[:8]])

    def engine_enqueue(self, form, ids, rating, mode, ts):
        eng = self.eng
        if form == "host":
            return eng.enqueue(ids, rating, mode, ts)
        if form == "device":
            import torch
            cols = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in
                    (ids.view(np.int64), rating, mode, ts.view(np.int32))]
            acc = torch.full((len(ids),), 0xEE, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            eng.enqueue_device(len(ids), *[c.data_ptr() for c in cols], acc.data_ptr())
            return acc.cpu().numpy()
        h, key = ids.astype(np.uint32), eng.pack_key(rating, mode)
        if form == "packed":
            return eng.enqueue_packed(h, key, ts)
        eng.enqueue_packed_begin(h, key, ts)
        return eng.enqueue_packed_end()[0]

    def remove(self):
        ids = self.ids_to_hit()
        if self.dense and self.rng.random() < 0.5:
            assert self.eng.remove_packed(ids.astype(np.uint32)) == self.m.remove(ids)
        else:
            assert self.eng.remove(ids) == self.m.remove(ids)

    def take(self):
        ids = self.ids_to_hit()
        assert self.eng.take(ids) == self.m.take(ids)

    def ids_to_hit(self):
        rng, m = self.rng, self.m
        q = m.q["id"]
        k = int(rng.integers(1, 3000))
        parts = [rng.choice(q, min(k, len(q))) if len(q) else q, rng.choice(m.active, min(k // 4, len(m.active)))
                 if len(m.active) else m.active, self.fresh(20)]
        return np.concatenate(parts)

    def tick(self):
        rng, m = self.rng, self.m
        ref, seq_of = m.tick_ref()
        forms = list(HOST_FORMS if self.dense else ("tick_emit", "tick", "device"))
        if self.async_on:
            forms = ["async_tick"] + (["async_packed"] if self.dense else [])
        form = str(rng.choice(forms))
        self.counts[form] = self.counts.get(form, 0) + 1
        if form.startswith("async"):
            self.at.tick(form == "async_packed", self.now, (ref, seq_of))
        else:
            if not self.async_on:
                poison(self.eng, ref.n_lobbies + 16, ref.n_matched + 16)
            lob, mem, seq, st = tick_form(self.pkg, self.eng, form, self.now)
            check_tick(ref, seq_of, lob, mem, seq, st)
        m.after_tick(ref, self.now)

    def option(self):
        rng, eng = self.rng, self.eng
        what = str(rng.choice(["tick_impl", "rank_impl", "max_spread", "async_results"]))
        if what == "max_spread" and self.cfg.order_mode != RATING:
            what = "tick_impl"
        if what == "tick_impl":
            self.tick_impl ^= 1
            eng.set_option("tick_impl", self.tick_impl)
        elif what == "rank_impl":
            eng.set_option("rank_impl", int(rng.choice([2, 3])))
        elif what == "max_spread":
            self.m.spread = int(rng.choice([-1, 0, 2, 60]))
            eng.set_option("max_spread", self.m.spread)
        else:
            self.async_on = not self.async_on
            if self.at is not None:
                self.at.wait()
            eng.set_option("async_results", int(self.async_on))
            self.at = AsyncTicks(self.pkg, eng, self.cfg.capacity) if self.async_on else None
        self.counts[what] = self.counts.get(what, 0) + 1

    def snapshot_or_restore(self):
        if self.m.snap is None or self.rng.random() < 0.4:
            self.eng.snapshot(); self.m.snapshot()
            self.counts["snapshot"] = self.counts.get("snapshot", 0) + 1
        else:
            self.eng.restore(); self.m.restore()
            self.counts["restore"] = self.counts.get("restore", 0) + 1

    def step(self):
        rng = self.rng
        self.now += int(rng.integers(1, 3000))
        op = str(rng.choice(["enq", "enq", "enq", "remove", "take", "in_queue", "tick", "tick", "tick", "option",
                             "stats", "snap"]))
        if op == "enq":
            big = rng.random() < 0.04
            self.enqueue(int(rng.integers(1_048_577, 1_300_000)) if big else int(rng.integers(1, 40_000)))
        elif op == "remove":
            self.remove()
        elif op == "take":
            self.take()
        elif op == "in_queue":
            s = self.sample()
            assert np.array_equal(self.eng.in_queue(s), self.m.in_queue(s))
        elif op == "tick":
            self.tick()
        elif op == "option":
            self.option()
        elif op == "snap":
            self.snapshot_or_restore()
        check_state(self.eng, self.m, self.now, self.sample()[:2000])
        return op

    def finish(self):
        if self.at is not None:
            self.at.wait()


SCHEDULES = [(dense, order, wide) for dense in (False, True) for order in (ARRIVAL, RATING) for wide in (0, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("dense,order,wide", SCHEDULES, ids=lambda v: str(v))
def test_long_mixed_schedule(pkg, oracle, dense, order, wide):
    rng = np.random.default_rng(100 + 4 * dense + 2 * order + wide)
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[:3], order=order, capacity=300_000,
                                active_capacity=4_000_000, default_group=-1, flags=(DENSE if dense else 0) | WIDE * wide)
    s = Schedule(pkg, oracle, cfg, rng, dense)
    ops = []
    try:
        s.enqueue(200_000)
        for _ in range(40):
            ops.append(s.step())
        s.tick()
        s.finish()
        check_state(s.eng, s.m, s.now, s.sample())
    finally:
        s.close()
    assert ops.count("tick") >= 5 and ops.count("enq") >= 3, ops


@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True])
def test_pool_near_capacity_under_s1_w0(pkg, oracle, dense):
    """Policy S1 with W = 0 leaves many players queued; every batch overflows the pool, which has been compacted by
    every tick before it, so ingest takes its capacity cut on a pool whose chunks were handed out many times."""
    rng = np.random.default_rng(7 + dense)
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, modes=MODES8[:3], order=RATING, capacity=60_000,
                                active_capacity=4_000_000, default_group=-1, flags=DENSE if dense else 0)
    s = Schedule(pkg, oracle, cfg, rng, dense)
    try:
        s.m.spread = 0
        s.eng.set_option("max_spread", 0)
        for k in range(24):
            s.now += 1000
            s.enqueue(2 * (cfg.capacity - s.m.slots()) + int(rng.integers(20_000, 40_000)))  # a quarter repeats
            assert (s.m.codes == 3).any() and s.m.slots() == cfg.capacity
            check_state(s.eng, s.m, s.now, s.sample()[:2000])
            if k % 5 == 4:
                s.tick_impl ^= 1
                s.eng.set_option("tick_impl", s.tick_impl)
            if k % 3 == 2:
                s.remove()
                s.take()
            s.tick()
            check_state(s.eng, s.m, s.now, s.sample()[:2000])
        assert s.m.slots() > cfg.capacity // 4
    finally:
        s.close()


@pytest.mark.gpu
@pytest.mark.parametrize("order", [ARRIVAL, RATING])
def test_remove_after_take_marks_the_slot_dead_once(pkg, oracle, order):
    """mm_take, then mm_remove of the same players before the next tick: the slot's bin total and chunk histogram are
    updated once.  (Counting them twice corrupted the histogram of another chunk, and the next tick failed with
    MM_E_STATE.)"""
    rng = np.random.default_rng(3)
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=order, capacity=100_000, default_group=-1)
    m = Model(cfg, oracle, pkg.abi)
    n = 90_000
    ids = pkg.synth.mix64(np.arange(n, dtype=np.uint64))
    rating, mode = rng.integers(0, 5001, n).astype(np.int32), rng.integers(0, 2, n).astype(np.uint8)
    with pkg.Engine(cfg) as eng:
        assert np.array_equal(eng.enqueue(ids, rating, mode), m.enqueue(ids, rating, mode))
        both = ids[rng.choice(n, 5000, replace=False)]
        assert eng.take(both) == m.take(both) == 5000
        assert eng.remove(both) == m.remove(both) == 5000
        check_state(eng, m, 0, both[:500])
        ref, seq_of = m.tick_ref()
        check_tick(ref, seq_of, *eng.tick())
        m.after_tick(ref)
        check_state(eng, m, 0, both[:500])
