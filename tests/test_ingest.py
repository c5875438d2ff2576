"""Ingest (claim -> count/scan/cut -> route -> alloc -> append, remove, take, lookup) against a serialized
restatement: every enqueue entry point, at the chunk, block and capacity edges, held exactly to a per-entry loop.

`Model` states what the engine holds between calls: the active set, the queued entries in enqueue order (a removed or
taken entry keeps its slot until the next tick), the enqueue sequence counter and the codes of the last batch.  It has
two enqueue rules that must agree: a plain per-entry loop (`scalar=True`) and a numpy twin for batches of millions."""
import numpy as np
import pytest

ARRIVAL, RATING = 0, 1
U32 = 0xFFFFFFFF


class Refused(Exception):
    """The batch is refused as a whole (MM_E_CAP): nothing changes, no sequence number is consumed."""


def hashed_slots(cfg):
    """Slots of a hashed active set, sized as mm_create sizes it (load factor <= 0.75 at active_capacity)."""
    want = cfg.active_capacity or 2 * cfg.capacity
    h = 1024
    while h * 3 < want * 4 + 64:
        h <<= 1
    return h


class Model:
    COLS = (("id", np.uint64), ("rating", np.int32), ("mode", np.uint8), ("ts", np.uint32), ("seq", np.uint32),
            ("alive", bool))

    def __init__(self, cfg, oracle, abi):
        self.cfg, self.oracle = cfg, oracle
        self.dedupe = not cfg.flags & abi.MM_F_NO_DEDUPE
        self.dense = self.dedupe and bool(cfg.flags & abi.MM_F_DENSE_IDS)
        self.id_limit = (cfg.active_capacity or 2 * cfg.capacity) if self.dense else 2 ** 64 - 2
        self.hcap = hashed_slots(cfg)
        self.active = np.zeros(0, np.uint64)
        self.q = {k: np.zeros(0, t) for k, t in self.COLS}
        self.seq_next = 0
        self.codes = np.zeros(0, np.uint8)
        self._grp = {}
        self.L = np.array([cfg.modes[m].teams * cfg.modes[m].team_size for m in range(cfg.n_modes)], np.int64)
        self.tsize = np.array([cfg.modes[m].team_size for m in range(cfg.n_modes)], np.uint8)

    # ---- rating groups (first {lo, hi} in list order, else the default group, else -1) -------------------------
    def group(self, r):
        g = self._grp.get(r)
        if g is None:
            g = self._grp[r] = self.oracle.find_rating_group(self.cfg, r)
        return g

    def groups(self, rating):
        u, inv = np.unique(np.asarray(rating, np.int64), return_inverse=True)
        return np.array([self.group(int(r)) for r in u], np.int64)[inv.reshape(-1)]

    def slots(self):
        return len(self.q["id"])

    # ---- enqueue --------------------------------------------------------------------------------------------
    def enqueue(self, ids, rating, mode, ts=None, scalar=False):
        ids = np.asarray(ids, np.uint64); rating = np.asarray(rating, np.int32); mode = np.asarray(mode, np.uint8)
        n = len(ids)
        ts = np.zeros(n, np.uint32) if ts is None else np.asarray(ts, np.uint32)
        if self.dedupe and not self.dense and (len(self.active) + n) * 4 > self.hcap * 3:
            raise Refused()
        code = self._codes_scalar(ids, rating, mode) if scalar else self._codes_vec(ids, rating, mode)
        k = code == 1
        seq = ((self.seq_next + np.arange(n, dtype=np.int64)) & U32).astype(np.uint32)
        for key, col in (("id", ids), ("rating", rating), ("mode", mode), ("ts", ts), ("seq", seq)):
            self.q[key] = np.concatenate([self.q[key], col[k]])
        self.q["alive"] = np.concatenate([self.q["alive"], np.ones(int(k.sum()), bool)])
        if self.dedupe:
            self.active = np.concatenate([self.active, ids[k]])
        self.seq_next = (self.seq_next + n) & U32
        self.codes = code
        return code

    def _codes_scalar(self, ids, rating, mode):
        active = set(self.active.tolist())
        room = self.cfg.capacity - self.slots()
        accepted = 0
        code = np.zeros(len(ids), np.uint8)
        for i, (p, r, m) in enumerate(zip(ids.tolist(), rating.tolist(), mode.tolist())):
            if m >= self.cfg.n_modes or p >= self.id_limit or self.group(r) < 0:
                code[i] = 2
            elif p in active:
                code[i] = 0  # queued earlier, accepted earlier in this batch, or matched and not yet removed
            elif accepted >= room:
                code[i] = 3
            else:
                code[i] = 1
                accepted += 1
                if self.dedupe:
                    active.add(p)
        return code

    def _codes_vec(self, ids, rating, mode):
        n = len(ids)
        valid = (mode < self.cfg.n_modes) & (ids < np.uint64(self.id_limit)) & (self.groups(rating) >= 0)
        vi = np.nonzero(valid)[0]
        if self.dedupe:
            _, first, inv = np.unique(ids[vi], return_index=True, return_inverse=True)
            head = vi[first][inv.reshape(-1)]  # batch index of the entry's first valid occurrence
            fresh = ~np.isin(ids[vi], self.active)
        else:
            head = vi
            fresh = np.ones(len(vi), bool)
        cand = (head == vi) & fresh
        rank = np.cumsum(cand) - 1
        room = max(self.cfg.capacity - self.slots(), 0)
        code = np.full(n, 2, np.uint8)
        cv = np.zeros(len(vi), np.uint8)
        cv[cand] = np.where(rank[cand] < room, 1, 3)
        code[vi] = cv
        rep = (head != vi) & fresh  # a repeat inside the batch follows its first occurrence
        code[vi[rep]] = np.where(code[head[rep]] == 3, 3, 0)
        return code

    # ---- remove / take / in_queue ----------------------------------------------------------------------------
    def remove(self, ids):
        hit = np.isin(self.active, np.asarray(ids, np.uint64))
        gone = self.active[hit]
        self.active = self.active[~hit]
        self.q["alive"] &= ~np.isin(self.q["id"], gone)  # the slot stays in use until the next tick
        return int(hit.sum())

    def take(self, ids):
        hit = self.q["alive"] & np.isin(self.q["id"], np.asarray(ids, np.uint64))
        self.q["alive"] &= ~hit
        return int(hit.sum())

    def in_queue(self, ids):
        return np.isin(np.asarray(ids, np.uint64), self.active)

    # ---- tick -------------------------------------------------------------------------------------------------
    def residual_mask(self):
        """Queued entries the next tick leaves queued (per (mode, group) partition, in the configured order, the
        first whole lobbies are matched); positional, so it holds with repeated ids too."""
        q, cfg = self.q, self.cfg
        n, G = len(q["id"]), cfg.n_groups
        keep = np.zeros(n, bool)
        idx = np.nonzero(q["alive"])[0]
        if not len(idx):
            return keep
        rating = q["rating"].astype(np.int64)
        if cfg.order_mode == RATING:
            lo = min(cfg.group_lo[g] for g in range(G)) - 1
            hi = max(cfg.group_hi[g] for g in range(G)) + 1
            feed = idx[np.lexsort((idx, np.clip(rating[idx], lo, hi), q["mode"][idx]))]
        else:
            feed = idx
        seg = q["mode"][feed].astype(np.int64) * G + self.groups(rating[feed])
        o = np.argsort(seg, kind="stable")
        part, seg_s = feed[o], seg[o]
        bounds = np.searchsorted(seg_s, np.arange(cfg.n_modes * G + 1))
        pos = np.arange(len(part)) - bounds[seg_s]
        cnt = bounds[seg_s + 1] - bounds[seg_s]
        L = self.L[seg_s // G]
        keep[part[pos >= cnt // L * L]] = True
        return keep

    def tick_ref(self, literal_max=100_000):
        """-> (oracle result of the next tick, sequence number of every oracle input).  The literal loop keeps the
        reference's id-keyed active set, so a removed entry whose id was offered again before the tick (or any repeated
        id under MM_F_NO_DEDUPE) would pass its in_queue? check; the engine drops removed entries by slot, which is
        what the closed form states."""
        q = self.q
        unique = len(np.unique(q["id"])) == self.slots()
        fn = self.oracle.run_literal if unique and self.slots() <= literal_max else self.oracle.run_closed_form
        return fn(self.cfg, q["id"], q["rating"], q["mode"], alive=q["alive"].astype(np.uint8)), q["seq"].copy()

    def after_tick(self, ref=None):
        keep = self.residual_mask()
        if ref is not None:
            assert np.array_equal(self.q["id"][keep], ref.residual_ids)
        self.q = {k: v[keep] for k, v in self.q.items()}

    # ---- what the engine reports -------------------------------------------------------------------------------
    def pool(self):
        q = self.q
        a = q["alive"]
        return dict(id=q["id"][a], rating=q["rating"][a], mode=q["mode"][a], team_size=self.tsize[q["mode"][a]],
                    enq_ts=q["ts"][a])

    def queue_counts(self):
        q, n_cut = self.q, self.cfg.n_modes * self.cfg.n_groups
        cut = q["mode"].astype(np.int64) * self.cfg.n_groups + self.groups(q["rating"])
        return (np.bincount(cut[q["alive"]], minlength=n_cut), np.bincount(cut[~q["alive"]], minlength=n_cut))

    def rejects(self):
        idx = np.nonzero(self.codes != 1)[0]
        return idx, self.codes[idx]


@pytest.fixture
def model(oracle, pkg):
    return lambda cfg: Model(cfg, oracle, pkg.abi)


# =====================================================================================================================
# CPU: the restatement against itself and against the host test double
# =====================================================================================================================
def random_schedule(rng, abi):
    """A small random config and a schedule of enqueue / remove / take / tick steps over a small id domain, so that
    repeats, pool-full cuts and stale (removed, unticked) slots are common."""
    flags = [0, 0, abi.MM_F_NO_DEDUPE, abi.MM_F_DENSE_IDS][rng.integers(0, 4)]
    groups = [((0, 1499), (1500, 5000)), ((0, 1499), (1500, 1999), (2000, 2499), (2500, 5000))][rng.integers(0, 2)]
    default = int(rng.integers(-1, len(groups)))
    cap = int(rng.integers(1, 60))
    steps = []
    for _ in range(int(rng.integers(3, 12))):
        kind = rng.choice(["enq", "enq", "enq", "remove", "take", "tick"])
        if kind == "enq":
            n = int(rng.integers(0, 40))
            ids = rng.integers(0, 100, n).astype(np.uint64)
            odd = rng.random(n) < 0.05
            ids[odd] = rng.choice(np.array([2 ** 64 - 1, 2 ** 64 - 2, 2 ** 64 - 3], np.uint64), int(odd.sum()))
            steps.append(("enq", ids, rng.integers(-100, 6000, n).astype(np.int32),
                          rng.integers(0, 3, n).astype(np.uint8), rng.integers(0, 1000, n).astype(np.uint32)))
        elif kind in ("remove", "take"):
            steps.append((kind, rng.integers(0, 100, int(rng.integers(0, 20))).astype(np.uint64)))
        else:
            steps.append(("tick",))
    return dict(groups=groups, default=default, cap=cap, flags=flags, active=int(rng.integers(0, 120))), steps


def test_scalar_and_vectorized_restatements_agree(pkg, model):
    rng = np.random.default_rng(2024)
    n_cut = n_two = n_zero = 0
    for trial in range(300):
        c, steps = random_schedule(rng, pkg.abi)
        cfg = pkg.synth.make_config(groups=c["groups"], order=[ARRIVAL, RATING][trial % 2], capacity=c["cap"],
                                    active_capacity=c["active"], default_group=c["default"], flags=c["flags"])
        a, b = model(cfg), model(cfg)
        for st in steps:
            if st[0] == "enq":
                try:
                    ca = a.enqueue(*st[1:], scalar=True)
                except Refused:
                    with pytest.raises(Refused):
                        b.enqueue(*st[1:])
                    continue
                cb = b.enqueue(*st[1:])
                assert np.array_equal(ca, cb), (trial, st)
                n_cut += int((ca == 3).sum()); n_two += int((ca == 2).sum()); n_zero += int((ca == 0).sum())
            elif not a.dedupe:
                continue  # mm_remove / mm_take answer MM_E_STATE without an active set
            elif st[0] == "remove":
                assert a.remove(st[1]) == b.remove(st[1])
            elif st[0] == "take":
                assert a.take(st[1]) == b.take(st[1])
            else:
                ref, _ = a.tick_ref()
                a.after_tick(ref); b.after_tick(ref)
            for k in a.q:
                assert np.array_equal(a.q[k], b.q[k])
            assert np.array_equal(np.sort(a.active), np.sort(b.active)) and a.seq_next == b.seq_next
    assert n_cut > 100 and n_two > 100 and n_zero > 100  # the schedules reach every code


def test_scalar_restatement_equals_the_oracle_engine_double(pkg, model):
    """fakes.OracleEngine frees a removed or taken player's slot at once, the engine (and the restatement) at the next
    tick: the schedules here tick between a remove / take and the next enqueue, where the two agree."""
    from tests.fakes import OracleEngine
    rng = np.random.default_rng(77)
    for trial in range(120):
        cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS[:int(rng.integers(2, 8))],
                                    order=[ARRIVAL, RATING][trial % 2], capacity=int(rng.integers(1, 50)),
                                    default_group=int(rng.integers(-1, 2)))
        m, f = model(cfg), OracleEngine(cfg)
        for _ in range(6):
            n = int(rng.integers(0, 40))
            ids = rng.integers(0, 80, n).astype(np.uint64)
            rating, mode = rng.integers(-100, 6000, n).astype(np.int32), rng.integers(0, 3, n).astype(np.uint8)
            assert np.array_equal(m.enqueue(ids, rating, mode, scalar=True), f.enqueue(ids, rating, mode)), trial
            probe = rng.integers(0, 80, 30).astype(np.uint64)
            assert np.array_equal(m.in_queue(probe), f.in_queue(probe))
            assert np.array_equal(m.pool()["id"], f.pool_read()["id"])
            gone, took = rng.integers(0, 80, 8).astype(np.uint64), rng.integers(0, 80, 8).astype(np.uint64)
            assert m.remove(gone) == f.remove(gone)
            assert m.take(took) == f.take(took)
            ref, _ = m.tick_ref()
            m.after_tick(ref)
            lob, mem, _, _ = f.tick()
            assert np.array_equal(mem, ref.member_ids) and m.slots() == f.pool_size()


def test_restatement_codes_by_hand(pkg, model):
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=ARRIVAL, capacity=5)
    m = model(cfg)
    # 6 and 7 are cut; their repeats are cut too; 2 repeated is "already in the queue"; mode 7 is invalid
    code = m.enqueue([1, 2, 3, 4, 5, 6, 7, 6, 2, 7], [100] * 10, [0, 0, 0, 0, 0, 0, 0, 0, 0, 7], scalar=True)
    assert list(code) == [1, 1, 1, 1, 1, 3, 3, 3, 0, 2] and m.seq_next == 10
    assert m.remove([1]) == 1 and m.slots() == 5  # a removed player holds its slot until the next tick
    assert list(m.enqueue([8], [100], [0])) == [3]
    m.after_tick()
    assert list(m.enqueue([8, 9], [100, 100], [0, 0])) == [1, 1] and m.seq_next == 13


# =====================================================================================================================
# GPU: four entry points held to the restatement
# =====================================================================================================================
class HostHashed:
    """mm_enqueue on a hashed active set (1 M-entry chunks, columns over PCIe)."""
    dense = False

    def __init__(self, pkg, cfg):
        self.eng = pkg.Engine(cfg)

    def enqueue(self, ids, rating, mode, ts):
        acc = self.eng.enqueue(ids, rating, mode, ts)
        return acc, int((acc == 1).sum())

    def tick(self):
        lob, mem, seq, st = self.eng.tick()
        return lob, mem, seq, st


class DeviceHashed(HostHashed):
    """mm_enqueue_device on a hashed active set (4 M-entry chunks, columns in HBM, device `accepted` buffer)."""

    def enqueue(self, ids, rating, mode, ts):
        import torch
        n = len(ids)
        cols = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in
                (np.asarray(ids, np.uint64).view(np.int64), np.asarray(rating, np.int32), np.asarray(mode, np.uint8),
                 np.asarray(ts, np.uint32).view(np.int32))]
        acc = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()  # the engine's stream does not wait for torch's
        na = self.eng.enqueue_device(n, *[c.data_ptr() for c in cols], acc.data_ptr())
        return acc.cpu().numpy(), na


class PackedDense(HostHashed):
    """mm_enqueue_packed on a dense active set (u32 handle + u16 mode << 13 | rating)."""
    dense = True

    def enqueue(self, ids, rating, mode, ts):
        acc = self.eng.enqueue_packed(np.asarray(ids).astype(np.uint32), self.eng.pack_key(rating, mode), ts)
        return acc, int((acc == 1).sum())

    def tick(self):
        lob, mem, seq, st = self.eng.tick_packed()
        return lob, mem.astype(np.uint64), seq, st


class StagedDense(PackedDense):
    """mm_enqueue_packed_begin / _end on a dense active set (4 M-entry chunks)."""

    def enqueue(self, ids, rating, mode, ts):
        self.eng.enqueue_packed_begin(np.asarray(ids).astype(np.uint32), self.eng.pack_key(rating, mode), ts)
        return self.eng.enqueue_packed_end()


ALL_FOUR = (HostHashed, DeviceHashed, PackedDense, StagedDense)


def engines(pkg, cfg, kinds=ALL_FOUR):
    out = []
    for k in kinds:
        c = pkg.synth.make_config(groups=[(cfg.group_lo[g], cfg.group_hi[g]) for g in range(cfg.n_groups)],
                                  modes=[("m", cfg.modes[m].teams, cfg.modes[m].team_size) for m in range(cfg.n_modes)],
                                  order=cfg.order_mode, capacity=cfg.capacity, active_capacity=cfg.active_capacity,
                                  default_group=cfg.default_group, flags=cfg.flags)
        if k.dense:
            c.flags |= pkg.abi.MM_F_DENSE_IDS
        out.append(k(pkg, c))
    return out


class Run:
    """One schedule through several engines and the restatement; every step is compared in full."""

    def __init__(self, pkg, model, cfg, kinds=ALL_FOUR):
        self.pkg = pkg
        self.m = model(cfg)
        self.engs = engines(pkg, cfg, kinds)

    def close(self):
        for e in self.engs:
            e.eng.close()

    def enqueue(self, ids, rating, mode, ts=None, sample=()):
        ts = np.arange(len(ids), dtype=np.uint32) * 7 + 3 if ts is None else ts
        try:
            want = self.m.enqueue(ids, rating, mode, ts)
        except Refused:
            for e in self.engs:
                if e.dense:  # a direct-mapped set never refuses: this run is for the hashed entry points only
                    raise AssertionError("a refusal schedule must not include dense engines")
                with pytest.raises(self.pkg.EngineError) as ei:
                    e.enqueue(ids, rating, mode, ts)
                assert ei.value.status == self.pkg.abi.MM_E_CAP
            self.check(sample)
            return None
        for e in self.engs:
            acc, na = e.enqueue(ids, rating, mode, ts)
            bad = np.nonzero(acc != want)[0]
            assert not len(bad), f"{type(e).__name__}: {len(bad)} codes differ, first at {bad[:8]}: " \
                                 f"got {acc[bad[:8]]}, want {want[bad[:8]]}"
            assert na == int((want == 1).sum())
        self.check(sample)
        return want

    def remove(self, ids):
        want = self.m.remove(ids)
        for e in self.engs:
            assert e.eng.remove(ids) == want
        self.check(ids[:64])

    def take(self, ids):
        want = self.m.take(ids)
        for e in self.engs:
            assert e.eng.take(ids) == want
        self.check(ids[:64])

    def check(self, sample=()):
        m = self.m
        ridx, rcode = m.rejects()
        pool = m.pool()
        n_wait, n_rem = m.queue_counts()
        sample = np.asarray(sample, np.uint64)
        for e in self.engs:
            name = type(e).__name__
            idx, code = e.eng.enqueue_rejects(cap=max(len(ridx), 1))
            o = np.argsort(idx)
            assert np.array_equal(idx[o], ridx) and np.array_equal(code[o], rcode), name
            assert e.eng.pool_size() == m.slots(), name
            assert e.eng.active_size() == len(m.active), name
            if m.dedupe and len(sample):
                assert np.array_equal(e.eng.in_queue(sample), m.in_queue(sample)), name
            got = e.eng.pool_read()
            for k in pool:
                assert np.array_equal(got[k], pool[k]), (name, k)
            qs = e.eng.queue_stats()
            assert np.array_equal(qs["n_waiting"], n_wait) and np.array_equal(qs["n_removed"], n_rem), name

    def tick(self):
        ref, seq_of = self.m.tick_ref()
        for e in self.engs:
            name = type(e).__name__
            lob, mem, seq, st = e.tick()
            assert (st.n_lobbies, st.n_matched, st.n_residual, st.n_dead) == \
                   (ref.n_lobbies, ref.n_matched, ref.n_residual, ref.n_dead), name
            assert np.array_equal(lob, ref.lobbies) and np.array_equal(mem, ref.member_ids), name
            assert np.array_equal(seq, seq_of[ref.emit_seq]), name
        self.m.after_tick(ref)
        self.check()
        return ref


class Ids:
    """Fresh ids below the dense handle range, in a shuffled order (so hashed probes and dense handles scatter)."""

    def __init__(self, rng, limit):
        self.perm = rng.permutation(limit).astype(np.uint64)
        self.next = 0

    def take(self, n):
        out = self.perm[self.next:self.next + n]
        assert len(out) == n
        self.next += n
        return out.copy()


def plant(ids, mode, rating, src, dst, bad_mode=None):
    """Entry dst repeats entry src's id; with bad_mode, the copy is offered with an invalid mode instead."""
    if 0 <= src < len(ids) and 0 <= dst < len(ids) and src != dst:
        ids[dst] = ids[src]
        if bad_mode is not None:
            mode[dst] = bad_mode


SPREAD = (1, 33, 256, 300, 1 << 20, (1 << 20) + 256, 1 << 22, (1 << 22) + 1)  # same warp, next block, chunk, 4 M chunk


def edge_batch(rng, fresh, n, n_modes, queued, cut_at, bad_mode, max_rating=5000):
    """A batch of n mostly fresh players with repeats of accepted ids, of ids around the capacity cut `cut_at` and of
    ids queued before the batch, each placed in the same warp, the next block, the next 1 M and the next 4 M chunk,
    plus copies of valid ids with an invalid mode placed before their valid first occurrence."""
    ids = fresh.take(n)
    rating = rng.integers(0, max_rating + 1, n).astype(np.int32)
    mode = rng.integers(0, n_modes, n).astype(np.uint8)
    srcs = [0, 5, n // 3, n - 300]
    if cut_at is not None:
        srcs += [cut_at - 3, cut_at - 1, cut_at, cut_at + 1, cut_at + 40]
        rating[cut_at] = min(rating[cut_at], 5000)  # a valid fresh player: the cut can land on it
    used = {cut_at}  # the cut lands on a fresh player
    for s in srcs:
        if 0 <= s < n:
            used.add(s)
            for d in SPREAD:
                if s + d < n and s + d not in used:
                    plant(ids, mode, rating, s, s + d)
                    used.add(s + d)
    for s in srcs:  # an invalid-mode copy just before the valid first occurrence
        if bad_mode is not None and 1 <= s < n and s - 1 not in used:
            plant(ids, mode, rating, s, s - 1, bad_mode)
            used.add(s - 1)
    if len(queued):  # ids queued before the batch, again at every distance
        for k, d in enumerate((2, 64, 700, (1 << 20) + 3, (1 << 22) + 5, n - 2)):
            if d < n and d not in used:
                ids[d] = queued[k % len(queued)]
                used.add(d)
    return ids, rating, mode


def first_winner_at_or_after(m, ids, rating, mode, i):
    """Batch index of the first entry at or after i that would take a slot (were the pool unbounded)."""
    cap = m.cfg.capacity
    m.cfg.capacity = 1 << 31
    try:
        code = m._codes_vec(np.asarray(ids, np.uint64), rating, mode)
    finally:
        m.cfg.capacity = cap
    win = np.nonzero(code == 1)[0]
    return win, int(win[np.searchsorted(win, i)])


def winners_before(m, ids, rating, mode, i):
    win, _ = first_winner_at_or_after(m, ids, rating, mode, 0)
    return int(np.searchsorted(win, i))


# (batch size, groups, modes, order, flags, where the capacity cut lands)
EDGE_CASES = [
    (1023, "reference", 2, ARRIVAL, 0, "block3"),
    (1024, "reference", 2, RATING, 0, None),
    (1025, "reference", 2, ARRIVAL, 0, "room0"),
    ((1 << 20) - 1, 32, 2, RATING, 0, None),
    (1 << 20, "reference", 2, ARRIVAL, "wide", "block3"),
    ((1 << 20) + 1, 32, 2, ARRIVAL, 0, "chunk1"),
    ((1 << 22) + (1 << 20) + 3, 64, 8, ARRIVAL, 0, "chunk1"),
    ((1 << 22) + (1 << 20) + 3, 16, 2, ARRIVAL, 0, "dev_chunk1"),
]


def edge_config(pkg, n, groups, n_modes, order, flags, cap):
    modes = [("1v1", 2, 1), ("5v5", 2, 5), ("2v2", 2, 2), ("3v3", 2, 3), ("ffa4", 4, 1), ("4v4", 2, 4),
             ("1v1b", 2, 1), ("ffa3", 3, 1)][:n_modes]
    fl = pkg.abi.MM_F_WIDE_PARTITIONS if flags == "wide" else 0
    kw = dict(modes=modes, order=order, capacity=cap, active_capacity=2 * n + 100_000, flags=fl)
    if groups == "reference":
        return pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, **kw)
    # equal-width groups, no default group: ratings 5001 .. 8191 (still packable) are invalid
    return pkg.synth.make_config(n_groups=groups, default_group=-1, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("case", EDGE_CASES, ids=lambda c: f"{c[0]}-g{c[1]}-m{c[2]}-o{c[3]}-{c[4]}-{c[5]}")
def test_four_entry_points_at_chunk_block_and_capacity_edges(pkg, model, case):
    n, groups, n_modes, order, flags, where = case
    rng = np.random.default_rng(n + n_modes)
    probe = edge_config(pkg, n, groups, n_modes, order, flags, 1 << 31)
    fresh = Ids(rng, probe.active_capacity)
    bad_mode = 7 if n_modes < 8 else None  # mode 8 does not fit the packed key
    max_rating = 5000 if groups == "reference" else 5100
    q0 = 3000
    first = fresh.take(q0), rng.integers(0, 5001, q0).astype(np.int32), rng.integers(0, n_modes, q0).astype(np.uint8)
    gone, took = first[0][10:50], first[0][100:130]
    # where the cut lands decides the capacity: count the winners before it with an unbounded pool
    m0 = model(probe)
    m0.enqueue(*first)
    m0.remove(gone); m0.take(took)
    # room 0 / inside block 3 of chunk 0 / exactly on the first winner of the second 1 M chunk / inside the second
    # 4 M chunk
    cut_at = {"block3": 3 * 256 + 77, "chunk1": 1 << 20, "dev_chunk1": (1 << 22) + 12_345, "room0": 0, None: None}[where]
    ids, rating, mode = edge_batch(rng, fresh, n, n_modes, first[0][::97], cut_at, bad_mode, max_rating)
    if cut_at is not None:
        _, cut_at = first_winner_at_or_after(m0, ids, rating, mode, cut_at)
    cap = q0 + (winners_before(m0, ids, rating, mode, cut_at) if cut_at is not None else n)
    cfg = edge_config(pkg, n, groups, n_modes, order, flags, cap)
    run = Run(pkg, model, cfg)
    try:
        run.enqueue(*first, sample=first[0][:100])
        run.remove(gone)
        run.take(took)
        sample = np.concatenate([ids[:50], ids[max(cut_at or 0, 0):][:200], ids[-50:], gone, took]) \
            if n > 0 else gone
        want = run.enqueue(ids, rating, mode, sample=sample)
        if cut_at is not None:
            assert want[cut_at] == 3 and (want == 3).sum() > 0  # the cut lands where it was put
            assert ((want == 1).nonzero()[0] < cut_at).all()
        assert (want == 0).any() and (want == 2).any()
        run.tick()  # the removed and taken players' slots are free after it
        # repeats of cut players, of removed ones and of matched ones, then fresh players: they fit now
        again = np.concatenate([ids[want == 3][:500], gone[:20], first[0][200:260], fresh.take(400)])
        r2 = rng.integers(0, 5001, len(again)).astype(np.int32)
        m2 = rng.integers(0, n_modes, len(again)).astype(np.uint8)
        run.enqueue(again, r2, m2, sample=again[::7])
        run.tick()
    finally:
        run.close()


@pytest.mark.gpu
@pytest.mark.parametrize("order", [ARRIVAL, RATING])
@pytest.mark.parametrize("wide", [0, 1])
def test_reference_groups_cut_and_repeats(pkg, model, order, wide):
    """The reference groups (a 1 500-rating group, ratings above 5000 in the default group), with and without
    MM_F_WIDE_PARTITIONS: several batches, each cut by the pool capacity, with repeats and leavers between them."""
    rng = np.random.default_rng(31 + 2 * order + wide)
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=order, capacity=50_000,
                                active_capacity=400_000, flags=pkg.abi.MM_F_WIDE_PARTITIONS * wide)
    fresh = Ids(rng, 400_000)
    run = Run(pkg, model, cfg)
    try:
        prev = np.zeros(0, np.uint64)
        for step in range(4):
            n = int(rng.integers(20_000, 70_001))
            ids = fresh.take(n)
            k = min(len(prev), n // 10)
            if k:
                ids[rng.choice(n, k, replace=False)] = rng.choice(prev, k)
            ids[rng.choice(n, n // 20, replace=False)] = ids[rng.choice(n, n // 20)]
            rating = rng.integers(0, 8192, n).astype(np.int32)
            mode = rng.integers(0, 3, n).astype(np.uint8)  # mode 2 is not configured
            run.enqueue(ids, rating, mode, sample=ids[::97])
            prev = np.concatenate([prev, ids])
            run.remove(prev[rng.choice(len(prev), 500)])
            run.take(prev[rng.choice(len(prev), 300)])
            if step % 2:
                run.tick()
        run.tick()
    finally:
        run.close()


@pytest.mark.gpu
def test_repeat_of_a_cut_player_is_cut_in_every_entry_point(pkg, model):
    """A repeat inside a batch follows its first occurrence: when that did not fit, neither does the repeat (code 3,
    not "already in the queue"), whichever chunk of the batch the two fall into."""
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=ARRIVAL, capacity=5, active_capacity=100)
    run = Run(pkg, model, cfg)
    try:
        want = run.enqueue(np.array([1, 2, 3, 4, 5, 6, 7, 6, 2, 7], np.uint64), [100] * 10, [0] * 9 + [7],
                           sample=np.arange(10, dtype=np.uint64))
        assert list(want) == [1, 1, 1, 1, 1, 3, 3, 3, 0, 2]
        assert not run.engs[0].eng.in_queue([6])[0]
    finally:
        run.close()


@pytest.mark.gpu
def test_removed_and_taken_players_hold_their_slots_until_the_tick(pkg, model):
    rng = np.random.default_rng(5)
    cfg = pkg.synth.make_config(n_groups=8, default_group=-1, order=ARRIVAL, capacity=2000, active_capacity=10_000)
    fresh = Ids(rng, 10_000)
    run = Run(pkg, model, cfg)
    try:
        ids = fresh.take(2000)
        run.enqueue(ids, rng.integers(0, 5001, 2000), rng.integers(0, 2, 2000))
        run.remove(ids[:37])
        run.take(ids[500:561])
        more = fresh.take(300)
        want = run.enqueue(more, rng.integers(0, 5001, 300), rng.integers(0, 2, 300), sample=more)
        assert (want == 3).all()  # room = 0: the stale slots still count
        run.tick()
        want = run.enqueue(more, rng.integers(0, 5001, 300), rng.integers(0, 2, 300), sample=more)
        assert (want == 1).sum() > 0
    finally:
        run.close()


@pytest.mark.gpu
def test_no_dedupe_queues_every_repeat(pkg, model):
    """MM_F_NO_DEDUPE: no active set.  Repeated ids are all queued (up to the capacity) and the tick equals the closed
    form over the whole feed; remove / take / in_queue answer MM_E_STATE."""
    rng = np.random.default_rng(12)
    n = (1 << 20) + 4097
    cfg = pkg.synth.make_config(n_groups=16, default_group=-1, order=RATING, capacity=n // 2,
                                flags=pkg.abi.MM_F_NO_DEDUPE)
    ids = rng.integers(0, n // 4, n).astype(np.uint64)  # about four copies of every id
    rating = rng.integers(0, 5200, n).astype(np.int32)
    mode = rng.integers(0, 3, n).astype(np.uint8)
    run = Run(pkg, model, cfg, kinds=(HostHashed, DeviceHashed))
    try:
        want = run.enqueue(ids, rating, mode)
        assert (want == 3).sum() > 0 and not (want == 0).any()
        for e in run.engs:
            for call in (e.eng.remove, e.eng.take, e.eng.in_queue):
                with pytest.raises(pkg.EngineError) as ei:
                    call(ids[:3])
                assert ei.value.status == pkg.abi.MM_E_STATE
        run.tick()
        run.enqueue(ids[:5000], rating[:5000], mode[:5000])
        run.tick()
    finally:
        run.close()


@pytest.mark.gpu
def test_hashed_refusal_threshold_and_what_a_refusal_leaves(pkg, model):
    """A batch is refused as a whole when (ids resident + batch) * 4 > slots * 3: the pool, the active set, the
    sequence numbers and the previous batch's reject list are unchanged.  The refused batch is the longest so far."""
    rng = np.random.default_rng(3)
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=ARRIVAL, capacity=1000, active_capacity=3000)
    limit = hashed_slots(cfg) * 3 // 4
    fresh = Ids(rng, 1 << 20)
    run = Run(pkg, model, cfg, kinds=(HostHashed, DeviceHashed))
    try:
        ids = fresh.take(1200)
        ids[900:910] = ids[:10]
        ids[1150:1160] = ids[1100:1110]
        want = run.enqueue(ids, rng.integers(0, 5001, 1200), np.where(np.arange(1200) % 50 == 7, 7, 0))
        assert {0, 1, 2, 3} <= set(want.tolist())
        run.tick()  # frees most slots; matched players stay in the active set
        n_act = len(run.m.active)
        over = fresh.take(limit - n_act + 1)
        assert len(over) > len(ids)
        seq = run.m.seq_next
        assert run.enqueue(over, np.full(len(over), 100), np.zeros(len(over)), sample=ids[::10]) is None  # refused
        assert run.m.seq_next == seq
        under = over[:-1]  # exactly at the limit (rehashes the cut players' tombstones away first)
        run.enqueue(under, np.full(len(under), 100), np.zeros(len(under)), sample=under[::50])
        run.tick()  # emit_seq of players offered after the refusal: it consumed no sequence number
    finally:
        run.close()


@pytest.mark.gpu
def test_tombstones_force_a_rehash_before_a_multi_chunk_batch(pkg, model):
    rng = np.random.default_rng(21)
    cfg = pkg.synth.make_config(n_groups=8, default_group=-1, order=ARRIVAL, capacity=600_000,
                                active_capacity=1_500_000)
    limit = hashed_slots(cfg) * 3 // 4
    fresh = Ids(rng, 1 << 24)
    run = Run(pkg, model, cfg, kinds=(HostHashed, DeviceHashed))
    try:
        a = fresh.take(1_000_000)
        run.enqueue(a, rng.integers(0, 5001, len(a)), rng.integers(0, 2, len(a)))  # 400 000 cut: tombstones
        queued = run.m.q["id"]
        run.remove(queued[rng.choice(len(queued), 300_000, replace=False)])  # 300 000 more
        run.tick()
        n = (1 << 20) + 5
        tombs = 400_000 + 300_000
        assert (len(run.m.active) + tombs + n) > limit >= len(run.m.active) + n  # this batch rehashes first
        b = fresh.take(n)
        b[::5] = a[rng.choice(len(a), len(b[::5]))]  # cut ids, removed ids, matched and queued ones
        run.enqueue(b, rng.integers(0, 5001, n), rng.integers(0, 2, n), sample=b[::1001])
        run.tick()
    finally:
        run.close()


@pytest.mark.gpu
def test_reject_list_survives_lookup_remove_and_take(pkg, model):
    """mm_enqueue_rejects reports the last batch whatever ran since: mm_in_queue, mm_remove and mm_take with lists
    longer than any batch before them."""
    rng = np.random.default_rng(9)
    cfg = pkg.synth.make_config(groups=pkg.synth.REFERENCE_GROUPS, order=ARRIVAL, capacity=4000,
                                active_capacity=100_000)
    fresh = Ids(rng, 100_000)
    run = Run(pkg, model, cfg, kinds=(HostHashed, PackedDense))
    try:
        ids = fresh.take(5000)
        ids[4500:4600] = ids[100:200]  # repeats of queued players
        want = run.enqueue(ids, rng.integers(0, 5001, 5000), np.where(np.arange(5000) % 97 == 0, 7, 0))
        assert {0, 1, 2, 3} <= set(want.tolist())
        for e in run.engs:
            e.eng.in_queue(fresh.perm[:20_000])
            e.eng.remove(fresh.perm[-30_000:])
            e.eng.take(ids[:10])
            idx, code = e.eng.enqueue_rejects()
            o = np.argsort(idx)
            ridx, rcode = run.m.rejects()
            assert np.array_equal(idx[o], ridx) and np.array_equal(code[o], rcode), type(e).__name__
    finally:
        run.close()


@pytest.mark.gpu
def test_sequence_numbers_wrap(pkg, model):
    """About 2^32 invalid-mode entries through mm_enqueue_device between two groups of queued players of one
    partition: pool_read keeps enqueue order across the wrap, and so does the ARRIVAL tick's emit_seq."""
    import torch
    # a hashed set refuses a batch longer than 3/4 of its slots, invalid entries included: room for one 2^22 batch
    cfg = pkg.synth.make_config(n_groups=1, modes=(("1v1", 2, 1),), order=ARRIVAL, capacity=64, active_capacity=1 << 22)
    run = Run(pkg, model, cfg, kinds=(DeviceHashed,))
    eng = run.engs[0].eng
    chunk = 1 << 22
    d_id = torch.zeros(chunk, dtype=torch.int64, device="cuda")
    d_r = torch.full((chunk,), 100, dtype=torch.int32, device="cuda")
    d_m = torch.full((chunk,), 7, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def offer_invalid(total):
        while total:
            k = min(chunk, total)
            assert eng.enqueue_device(k, d_id.data_ptr(), d_r.data_ptr(), d_m.data_ptr()) == 0
            run.m.seq_next = (run.m.seq_next + k) & U32
            run.m.codes = np.full(k, 2, np.uint8)
            total -= k

    try:
        offer_invalid((1 << 32) - 8)
        run.enqueue(np.arange(1, 4, dtype=np.uint64), [100] * 3, [0] * 3)  # sequence numbers 2^32 - 8 .. 2^32 - 6
        # three more invalid entries, then four players across the wrap: 2^32 - 2, 2^32 - 1, 0, 1
        run.enqueue(np.array([0, 0, 0, 10, 11, 12, 13], np.uint64), [100] * 7, [7, 7, 7, 0, 0, 0, 0])
        assert list(run.m.q["seq"]) == [U32 - 7, U32 - 6, U32 - 5, U32 - 1, U32, 0, 1]
        ref = run.tick()  # lobbies (1, 2), (3, 10), (11, 12); 13 stays
        assert ref.n_lobbies == 3 and list(ref.residual_ids) == [13]
    finally:
        run.close()
