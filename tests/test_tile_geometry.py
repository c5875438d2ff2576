"""Tick geometry: which placement paths a pool reaches, and GPU parity at the geometries the other tests miss.

The CPU half restates, in numpy, how the engine lays a pool out for a tick:
  * partitions (mm_engine.cu build_tables): key -> group / bin LUTs, (mode, group) segments split into partitions of
    at most 255 keys, and the fallback to whole segments when the split would need more than 512 partitions;
  * mm_create's choice of placement stages and rows per SM (place_smem_bytes, colscan_smem), and tick_rows;
  * the virtual tile sequence of geo_build (NT, tiles per row, most rows a partition spans, column-scan condition);
  * the slot-counter window rule of place_halves / place_body (place_cnt_cap), tile by tile.
It reports, per row, the tiles, the partitions, the window reloads after the row's first tile (and which tile
pipeline did each on the two-pipeline path), LIST / FAST tile transitions and the tiles past the 64-entry
descriptor cache.

Every GPU test first asserts that its pool reaches the regime it is about, with margin, so a change of the geometry
that moves a test off its path fails the test instead of leaving the path unchecked.  Each one is then held bit-exact
to the oracle (lobbies, members, emission order, counts, leftovers), and runs a second tick on the compacted pool after
removes, takes and new arrivals: that tick ranks on chunk histograms rebuilt by the first tick and updated by ingest,
remove and take, and fails with MM_E_STATE if any tile's histogram disagrees with its keys.
"""
import ctypes as C

import numpy as np
import pytest

ARRIVAL, RATING = 0, 1

# ---- constants of the tick (mm_common.cuh, mm_place.cuh, mm_hist.cuh, mm_scan.cuh, mm_engine.cu) ----------------
TILE = 2048           # kTile
DESC_CAP = 64         # kDescCap
FAST_BINS = 255       # kFastBins
MAX_SEGS = 64 * 8     # kMaxSegs = MM_MAX_GROUPS * MM_MAX_MODES
MAX_ROWS = 2048       # kMaxRows
MAX_STAGES = 4        # kMaxStages
TILE_BYTES = TILE * 10
CHUNK_HIST = 256
HALVES_HDR = 288
HALF_BYTES = 8 * 256 * 4 + 8 * 256 * 2 + 256 * 4 + TILE * 4
PLACE_UNION = 16 * 256 * 4 + 16 * 256 * 2 + 1024 + TILE * 4
DESC_BYTES = 2 * DESC_CAP * 4
STATIC_SMEM = (MAX_SEGS + 1) * 4 + 16 + 512  # sizeof(Geo) + 512: mm_create's allowance for static shared memory
TAIL_FIXED = 64 + 4 + 9 * MAX_SEGS + 12      # kTailScratchWords
COL_SCRATCH = (512 // 32) * 33               # kColScratchWords
INLINE_PREFIX_ROWS = 24
HIST_STAGES = 8                              # kHistStages
EPI_SCRATCH = (MAX_ROWS + 1) + 64 + (MAX_SEGS + 1) + 4 * MAX_SEGS + 2048  # kEpiScratchWords
K_TICK_STATIC = 2304                         # static shared memory of k_tick<512> (ptxas -v)
WIDE = 4                                     # MM_F_WIDE_PARTITIONS
DENSE = 2                                    # MM_F_DENSE_IDS


class Device:
    """What the geometry depends on: SM count and shared memory (sm_90: 228 KB per SM, 227 KB per block)."""

    def __init__(self, n_sms=132, smem_sm=233472, smem_optin=232448):
        self.n_sms, self.smem_sm, self.smem_optin = n_sms, smem_sm, smem_optin

    @classmethod
    def current(cls):
        import torch
        p = torch.cuda.get_device_properties(0)
        return cls(p.multi_processor_count, getattr(p, "shared_memory_per_multiprocessor", 233472),
                   getattr(p, "shared_memory_per_block_optin", 232448))


H100_SXM = Device()


def place_cnt_cap(max_nb):
    return max(max_nb, 1024)


def place_smem_bytes(max_nb, stages):
    cnt = ((place_cnt_cap(max_nb) + 3) & ~3) * 4
    whole = stages * TILE_BYTES + 128 + cnt + PLACE_UNION + DESC_BYTES + 16
    halves = stages * (TILE_BYTES + CHUNK_HIST * 4) + HALVES_HDR + cnt + 2 * HALF_BYTES + DESC_BYTES + 16
    return halves if max_nb <= FAST_BINS and halves > whole else whole


def colscan_smem(Kp, dev):
    def words(layout):
        return TAIL_FIXED + (Kp + 2) + ((Kp + 2) if layout & 1 else 0) + ((Kp + 3) // 2 if layout & 2 else 0)
    if words(3) * 4 <= 100 * 1024:
        layout = 3
    elif words(1) * 4 + 1024 <= dev.smem_optin:
        layout = 1
    else:
        layout = 0
    return max(COL_SCRATCH, words(layout)) * 4


class Layout:
    """build_tables + mm_create's shared-memory plan for a config.  .ok is False where mm_create gives MM_E_ARG."""

    def __init__(self, cfg, dev=H100_SXM):
        self.cfg, self.dev, self.ok = cfg, dev, False
        G, nm = cfg.n_groups, cfg.n_modes
        lo = np.array([cfg.group_lo[g] for g in range(G)], np.int64)
        hi = np.array([cfg.group_hi[g] for g in range(G)], np.int64)
        self.key_lo = int(lo.min()) - 1
        self.KR = int(hi.max()) - int(lo.min()) + 3
        if self.KR > 65535:
            return
        keys = self.key_lo + np.arange(self.KR)
        grp = np.full(self.KR, -1, np.int64)
        for g in range(G):
            grp[(grp < 0) & (keys >= lo[g]) & (keys <= hi[g])] = g
        grp[grp < 0] = cfg.default_group
        self.grp = grp
        lut = np.zeros(self.KR, np.int64)
        if cfg.order_mode == RATING:
            first = [0]
            for g in range(G):
                k = np.nonzero(grp == g)[0]
                lut[k] = first[-1] + np.arange(len(k))
                first.append(first[-1] + len(k))
            self.stride = max(first[-1], 1)
        else:
            lut = np.where(grp < 0, 0, grp)
            first = list(range(G + 1))
            self.stride = G
        self.lut, self.first = lut, first
        self.K = nm * self.stride
        self.Kp = self.K + 1
        if self.Kp > 65535:
            return
        split = not (cfg.flags & WIDE)
        for _ in range(2):
            seg_lo, part_cut = [], []
            for m in range(nm):
                for g in range(G):
                    b0, nk = m * self.stride + first[g], first[g + 1] - first[g]
                    nsub = max(1, -(-nk // FAST_BINS)) if split else 1
                    per = -(-nk // nsub)
                    for j in range(nsub):
                        seg_lo.append(b0 + min(nk, j * per))
                        part_cut.append(m * G + g)
            if len(seg_lo) <= MAX_SEGS:
                break
            split = False
        self.split = split
        self.n_segs = len(seg_lo)
        if self.n_segs > MAX_SEGS:
            return
        self.seg_lo = np.array(seg_lo + [self.K], np.int64)
        self.part_cut = np.array(part_cut, np.int64)
        self.nb = np.diff(self.seg_lo)
        self.max_nb = max(1, int(self.nb.max()))
        self.min_L = min(cfg.modes[m].teams * cfg.modes[m].team_size for m in range(nm))
        self.chist = self.max_nb <= FAST_BINS
        # mm_create: two CTAs per SM with 2 stages if they fit, else one CTA with the deepest ring that fits
        self.stages = 0
        if 2 * (place_smem_bytes(self.max_nb, 2) + STATIC_SMEM + 1024) <= dev.smem_sm:
            self.stages, self.rows_per_sm = 2, 2
        else:
            for st in range(MAX_STAGES, 0, -1):
                if place_smem_bytes(self.max_nb, st) + STATIC_SMEM + 1024 <= dev.smem_optin:
                    self.stages, self.rows_per_sm = st, 1
                    break
        if not self.stages or colscan_smem(self.Kp, dev) + STATIC_SMEM + 1024 > dev.smem_optin:
            return
        total = min(dev.n_sms * self.rows_per_sm, MAX_ROWS)
        self.helpers = 4 if total >= 64 else (1 if total > 1 else 0)
        self.R = total - self.helpers
        # the fused cooperative tick needs every CTA resident: its dynamic shared memory is the largest phase's
        hist = HIST_STAGES * TILE * 2 + 256 + ((self.max_nb + 4) & ~3) * 4 + DESC_BYTES + 16
        sz = max(hist, place_smem_bytes(self.max_nb, self.stages), EPI_SCRATCH * 4, colscan_smem(self.Kp, dev))
        per_sm = min(2, dev.smem_sm // (sz + K_TICK_STATIC + 1024))  # 64 registers x 512 threads: 2 CTAs at most
        self.fused = per_sm * dev.n_sms >= total
        self.ok = True

    def partition_of(self, rating, mode):
        """layout partition of every player (-1: rejected at ingest)."""
        k = np.clip(np.asarray(rating, np.int64), self.key_lo, self.key_lo + self.KR - 1) - self.key_lo
        mode = np.asarray(mode, np.int64)
        g = self.grp[k]
        b = mode * self.stride + self.lut[k]
        p = np.searchsorted(self.seg_lo[:-1], b, side="right") - 1
        return np.where((g < 0) | (mode >= self.cfg.n_modes), -1, p)

    def fills(self, rating, mode):
        p = self.partition_of(rating, mode)
        return np.bincount(p[p >= 0], minlength=self.n_segs)

    def tick_rows(self, n):
        tiles = n // TILE + self.n_segs
        total = self.R + self.helpers
        want = min(32, max(self.helpers, (total * 14 // 100 + self.min_L - 1) // self.min_L))
        return min(total - want, max(1, (tiles + 1) // 2))

    def heavy(self, rating, mode, alive=None):
        """TickCtr::heavy: some partition of > 255 keys has a bin expected at > 8 players per tile."""
        k = np.clip(np.asarray(rating, np.int64), self.key_lo, self.key_lo + self.KR - 1) - self.key_lo
        b = np.asarray(mode, np.int64) * self.stride + self.lut[k]
        keep = np.ones(len(b), bool) if alive is None else np.asarray(alive, bool)
        tot = np.bincount(b[keep], minlength=self.K)
        fill = self.fills(rating, mode)
        for p in np.nonzero(self.nb > FAST_BINS)[0]:
            if fill[p] and int(tot[self.seg_lo[p]:self.seg_lo[p + 1]].max()) * TILE > 8 * int(fill[p]):
                return True
        return False


class Geometry:
    """geo_build + the window rule of the placement pass, for one tick of a pool with these partition fills."""

    def __init__(self, lay, fills, rank_impl=3, n=None):
        self.lay = lay
        fills = np.asarray(fills, np.int64)
        n = int(fills.sum()) if n is None else n
        self.rows = lay.tick_rows(n)
        T = (fills + TILE - 1) // TILE
        T0 = np.concatenate([[0], np.cumsum(T)])
        self.NT = int(T0[-1])
        self.tpr = -(-self.NT // self.rows) if self.NT else 1
        spans = [(int(T0[p + 1]) - 1) // self.tpr - int(T0[p]) // self.tpr + 1 for p in range(lay.n_segs) if T[p]]
        self.max_rows = max(spans, default=0)
        self.colscan = self.NT > self.tpr * INLINE_PREFIX_ROWS and self.max_rows > INLINE_PREFIX_ROWS
        self.halves = lay.chist and rank_impl == 3  # place_halves: two tile pipelines per CTA
        self.hist = "rowsum" if lay.chist else "hist"
        seg_of_tile = np.repeat(np.arange(lay.n_segs), T)
        cap = place_cnt_cap(lay.max_nb)
        seg_lo, nb = lay.seg_lo, lay.nb
        self.row = []
        for r in range(self.rows):
            s0 = min(r * self.tpr, self.NT)
            s1 = min(s0 + self.tpr, self.NT)
            segs = seg_of_tile[s0:s1]
            rep = dict(tiles=len(segs), parts=len(np.unique(segs)), reloads=[0, 0], prefixed=0, transitions=0,
                       mixed=False, past_cache=max(0, len(segs) - DESC_CAP))
            if len(segs):
                p_last = int(segs[-1])
                wb = we = 0
                kinds = []
                for t, p in enumerate(segs.tolist()):
                    b0, b1 = int(seg_lo[p]), int(seg_lo[p + 1])
                    if b0 < wb or b1 > we:
                        wb, we = b0, b1
                        for q in range(p + 1, p_last + 1):
                            e = int(seg_lo[q + 1])
                            if e - wb > cap:
                                break
                            we = e
                        if t:
                            rep["reloads"][t % 2 if self.halves else 0] += 1
                            # rows before this one hold tiles of a partition of the new window: its M / P row
                            # prefix is not zero (a reload only happens on entering a partition, so never)
                            rep["prefixed"] += int((T0[p:p_last + 1][seg_lo[p + 1:p_last + 2] <= we] < s0).any())
                    kinds.append(rank_impl == 3 and nb[p] <= FAST_BINS)
                rep["transitions"] = int(np.count_nonzero(np.diff(np.array(kinds, np.int8))))
                rep["mixed"] = len(set(kinds)) == 2
            self.row.append(rep)
        self.max_tiles = max((x["tiles"] for x in self.row), default=0)
        self.max_parts = max((x["parts"] for x in self.row), default=0)
        self.reloads = [sum(x["reloads"][h] for x in self.row) for h in (0, 1)]
        self.prefixed = sum(x["prefixed"] for x in self.row)
        self.mixed_rows = sum(x["mixed"] for x in self.row)
        self.transitions = sum(x["transitions"] for x in self.row)
        self.rows_past_cache = sum(x["past_cache"] > 0 for x in self.row)

    def summary(self):
        return dict(rows=self.rows, NT=self.NT, tpr=self.tpr, max_tiles=self.max_tiles, max_parts=self.max_parts,
                    reloads=tuple(self.reloads), mixed_rows=self.mixed_rows, transitions=self.transitions,
                    rows_past_cache=self.rows_past_cache, rows_per_sm=self.lay.rows_per_sm, stages=self.lay.stages,
                    halves=self.halves, colscan=self.colscan, hist=self.hist, n_segs=self.lay.n_segs,
                    max_nb=self.lay.max_nb)


# ---- the pools of each regime -------------------------------------------------------------------------------------
MODES8 = (("1v1", 2, 1), ("2v2", 2, 2), ("3v3", 2, 3), ("5v5", 2, 5), ("solo4", 4, 1), ("duo3", 3, 2), ("6v6", 2, 6),
          ("solo3", 3, 1))
ALT_GROUPS = ((0, 99), (100, 1299), (1300, 1399), (1400, 2999), (3000, 3200), (3201, 5000))


def fallback_groups():
    """64 groups over 0..4999: 60 of 66 ratings and 4 of 260, so 8 modes need more than 512 split partitions."""
    w = [260 if g in (10, 25, 40, 55) else 66 for g in range(64)]
    lo = np.concatenate([[0], np.cumsum(w)[:-1]])
    return [(int(a), int(a + b - 1)) for a, b in zip(lo, w)]


def many_partitions_pool(pkg, seed=1):
    """8 modes x 20 groups of 250 ratings: mode 0 holds 2 M players (100 000 per group), the other seven 300 per
    group, with every fifth group empty so that the rows' window reloads fall on both tile pipelines."""
    rng = np.random.default_rng(seed)
    parts_r, parts_m = [], []
    for m in range(8):
        for g in range(20):
            k = 100_000 if m == 0 else (0 if (3 * m + g) % 5 == 2 else 300)
            parts_r.append(rng.integers(250 * g, 250 * g + 250, k))
            parts_m.append(np.full(k, m))
    rating = np.concatenate(parts_r)
    mode = np.concatenate(parts_m)
    o = rng.permutation(len(rating))  # arrival order mixes the modes
    n = len(rating)
    ids = pkg.synth.mix64(np.arange(n, dtype=np.uint64) + np.uint64(seed << 40))
    return ids, rating[o].astype(np.int32), mode[o].astype(np.uint8), np.arange(n, dtype=np.uint32)


def uniform_pool(pkg, seed, n, lo, hi, n_modes=1, dense=False):
    rng = np.random.default_rng(seed)
    ids = np.arange(n, dtype=np.uint64) if dense else pkg.synth.mix64(np.arange(n, dtype=np.uint64) + np.uint64(seed << 40))
    rating = rng.integers(lo, hi + 1, n).astype(np.int32)
    mode = rng.integers(0, n_modes, n).astype(np.uint8)
    return ids, rating, mode, np.arange(n, dtype=np.uint32)


def config3_pool(pkg, n):
    """BASELINE config3's shape (5v5 only, 32 groups) at n players with dense ids."""
    _, rating, _, _ = pkg.synth.gen_pool(1, n)
    return np.arange(n, dtype=np.uint64), rating, np.zeros(n, np.uint8), np.arange(n, dtype=np.uint32)


# ---- numpy closed form with emission order -----------------------------------------------------------------------
class NumpyTick:
    """oracle.closed_form_numpy plus lobby headers and emit_seq (input index of each lobby's last member in feed
    order), for pools too large for the C oracle in a test.  Policy S0 only."""

    def __init__(self, cfg, ids, rating, mode, alive=None):
        G = cfg.n_groups
        rating = np.asarray(rating, np.int64)
        mode = np.asarray(mode, np.int64)
        n = len(ids)
        grp = np.full(n, cfg.default_group, np.int64)
        unset = np.ones(n, bool)
        for g in range(G):
            hit = unset & (rating >= cfg.group_lo[g]) & (rating <= cfg.group_hi[g])
            grp[hit] = g
            unset &= ~hit
        keep = np.ones(n, bool) if alive is None else np.asarray(alive, bool)
        idx = np.nonzero(keep)[0]
        if cfg.order_mode == RATING:
            rmin = min(cfg.group_lo[g] for g in range(G))
            rmax = max(cfg.group_hi[g] for g in range(G))
            ck = np.clip(rating[idx], rmin - 1, rmax + 1)
            feed = idx[np.lexsort((idx, ck, mode[idx]))]
        else:
            feed = idx
        seg = mode[feed] * G + grp[feed]
        part = feed[np.argsort(seg, kind="stable")]
        bounds = np.searchsorted(np.sort(seg, kind="stable"), np.arange(cfg.n_modes * G + 1))
        take, hdr, last, resid = [], [], [], []
        off = 0
        for s in range(cfg.n_modes * G):
            a, b = bounds[s], bounds[s + 1]
            m = s // G
            L = cfg.modes[m].teams * cfg.modes[m].team_size
            nl = (b - a) // L
            take.append(part[a:a + nl * L])
            hdr.append(np.stack([off + L * np.arange(nl), np.full(nl, L), np.full(nl, m), np.full(nl, s % G)], 1))
            last.append(part[a + L - 1:a + nl * L:L])
            resid.append(part[a + nl * L:b])
            off += nl * L
        h = np.concatenate(hdr)
        self.lobbies = np.zeros(len(h), np.dtype([("first_member", "<u4"), ("n_members", "<u2"), ("mode", "u1"),
                                                  ("group", "u1")]))
        for i, f in enumerate(("first_member", "n_members", "mode", "group")):
            self.lobbies[f] = h[:, i]
        self.member_ids = np.asarray(ids, np.uint64)[np.concatenate(take)]
        self.emit_seq = np.concatenate(last).astype(np.uint32)
        self.residual_ids = np.asarray(ids, np.uint64)[np.sort(np.concatenate(resid))]
        self.n_lobbies, self.n_matched = len(self.lobbies), len(self.member_ids)
        self.n_residual, self.n_dead = len(self.residual_ids), int(n - keep.sum())


# ================================================================================ CPU: the model on known shapes
def test_numpy_tick_equals_the_c_oracle(pkg, oracle):
    """NumpyTick (used for the largest pools) against the C oracle's closed form, emission order included."""
    for order in (RATING, ARRIVAL):
        cfg = pkg.synth.make_config(groups=fallback_groups()[:20] + [(1600, 5000)], modes=MODES8[:3], order=order,
                                    capacity=60_000)
        ids, rating, mode, _ = uniform_pool(pkg, 5, 60_000, -30, 5030, n_modes=3)
        alive = (np.random.default_rng(2).random(60_000) > 0.05).astype(np.uint8)
        ref = oracle.run_closed_form(cfg, ids, rating, mode, alive)
        got = NumpyTick(cfg, ids, rating, mode, alive)
        assert np.array_equal(got.lobbies, ref.lobbies) and np.array_equal(got.member_ids, ref.member_ids)
        assert np.array_equal(got.emit_seq, ref.emit_seq) and np.array_equal(got.residual_ids, ref.residual_ids)
        assert (got.n_dead, got.n_residual) == (ref.n_dead, ref.n_residual)


def test_layout_partitions_and_fallback(pkg):
    syn = pkg.synth
    ref = Layout(syn.make_config(groups=syn.REFERENCE_GROUPS, order=RATING))
    # 1 500 + 2 clamp keys in the default group ("diamond" is 500 wide): 1 500 / 255 -> 6 partitions of 250
    assert ref.ok and ref.split and ref.max_nb <= FAST_BINS and ref.chist
    assert ref.n_segs == 2 * (6 + 2 + 2 + 2 + 2 + 2 + 4)
    wide = Layout(syn.make_config(groups=syn.REFERENCE_GROUPS, order=RATING, flags=WIDE))
    assert wide.n_segs == 14 and wide.max_nb == 1500 and not wide.chist
    fb = Layout(syn.make_config(groups=fallback_groups(), modes=MODES8, order=RATING))
    assert fb.ok and not fb.split and fb.n_segs == 512 and fb.max_nb == 260
    assert (fb.rows_per_sm, fb.stages) == (2, 2)
    # the partition of a player is the one whose bins hold it: every partition's bin range is its keys'
    cfg = syn.make_config(n_groups=8, order=RATING)
    lay = Layout(cfg)
    ids, rating, mode, _ = uniform_pool(pkg, 3, 20_000, -50, 5050, n_modes=2)
    p = lay.partition_of(rating, mode)
    k = np.clip(rating, lay.key_lo, lay.key_lo + lay.KR - 1) - lay.key_lo
    b = mode.astype(np.int64) * lay.stride + lay.lut[k]
    assert ((lay.seg_lo[p] <= b) & (b < lay.seg_lo[p + 1])).all()
    grp = np.where((rating < 0) | (rating > 5000), cfg.default_group,
                   np.searchsorted(syn.equal_width_groups(8)[1], np.clip(rating, 0, 5000)))
    assert (lay.part_cut[p] == mode * 8 + grp).all()


def test_stage_choice_and_key_domain_edge(pkg):
    syn = pkg.synth
    huge = Layout(syn.make_config(groups=[(0, 20000)], modes=MODES8[3:4], order=RATING, default_group=0, flags=WIDE))
    assert huge.ok and huge.max_nb == 20003 and (huge.rows_per_sm, huge.stages) == (1, 4) and huge.R == 128
    split = Layout(syn.make_config(groups=[(0, 20000)], modes=MODES8[3:4], order=RATING, default_group=0))
    assert split.ok and split.n_segs == 79 and split.chist and (split.rows_per_sm, split.stages) == (2, 2)
    # rows_per_sm = 1 from about 9 400 keys per partition
    assert Layout(syn.make_config(groups=[(0, 9420)], order=RATING, flags=WIDE)).rows_per_sm == 2
    assert Layout(syn.make_config(groups=[(0, 9440)], order=RATING, flags=WIDE)).rows_per_sm == 1
    # largest rating span accepted with 2 modes: the scan tail's shared memory bounds it
    span = key_domain_edge(pkg, lambda cfg: Layout(cfg).ok)
    assert span == 26257
    for flags in (0, WIDE):
        assert Layout(edge_config(pkg, span, flags)).ok and not Layout(edge_config(pkg, span + 1, flags)).ok


def test_config3_geometry_stays_inside_the_descriptor_cache(pkg):
    """config3 (10 M, 5v5, 32 groups): 20 tiles per row with the 1v1 mode configured too (test_engine_gpu), 19 with
    5v5 alone (bench.py); 65 only from about 34.1 M players."""
    _, rating, _, _ = pkg.synth.gen_pool(1, 10_000_000)
    two = Layout(pkg.synth.make_config(n_groups=32, order=RATING))
    g = Geometry(two, two.fills(rating, np.ones(len(rating), np.int64)))
    assert (g.rows, g.max_tiles, g.rows_past_cache, g.reloads) == (246, 20, 0, [0, 0])
    assert g.halves and g.max_parts <= 3
    assert two.fused
    lay = Layout(pkg.synth.make_config(n_groups=32, modes=MODES8[3:4], order=RATING))
    g = Geometry(lay, lay.fills(rating, np.zeros(len(rating), np.int64)))
    assert (g.rows, g.max_tiles, g.rows_past_cache, g.reloads) == (260, 19, 0, [0, 0])
    per = np.full(lay.n_segs, 34_100_000 // lay.n_segs)
    assert Geometry(lay, per).max_tiles == 65
    assert Geometry(lay, np.full(lay.n_segs, 33_000_000 // lay.n_segs)).max_tiles < 65


def test_existing_shapes_reload_no_window_mid_row(pkg):
    """The pools of test_engine_gpu / test_rating_window (a sample of their shapes): no row reloads its slot-counter
    window after its first tile on the two-pipeline path, and no row passes the descriptor cache."""
    syn = pkg.synth
    shapes = [
        (syn.make_config(n_groups=8, order=RATING), 1_000_003, 2),
        (syn.make_config(groups=syn.REFERENCE_GROUPS, order=RATING), 70_001, 2),
        (syn.make_config(groups=syn.REFERENCE_GROUPS, order=RATING), 600_011, 2),
        (syn.make_config(n_groups=64, modes=MODES8[:4], order=RATING), 400_009, 4),
        (syn.make_config(n_groups=32, order=RATING), 400_003, 2),
    ]
    for cfg, n, nm in shapes:
        lay = Layout(cfg)
        _, rating, mode, _ = uniform_pool(pkg, n, n, -20, 5020, n_modes=nm)
        g = Geometry(lay, lay.fills(rating, mode))
        assert g.halves and g.reloads == [0, 0] and g.max_parts <= 4 and g.rows_past_cache == 0, g.summary()


def test_regime_models(pkg):
    """The geometry each GPU test below relies on, reproduced on the host for a 132-SM H100."""
    syn = pkg.synth
    # many partitions per row
    lay = Layout(syn.make_config(groups=[(250 * g, 250 * g + 249) for g in range(20)], modes=MODES8, order=RATING))
    _, rating, mode, _ = many_partitions_pool(pkg)
    g = Geometry(lay, lay.fills(rating, mode))
    assert lay.n_segs == 160 and g.tpr == 5 and g.halves
    assert not lay.fused  # 8 x 5 002 keys: the scan tail's shared memory leaves one CTA per SM
    assert g.reloads[0] >= 8 and g.reloads[1] >= 8, g.summary()
    # a window loaded after the row's first tile starts at a partition whose first tile is in this row: its row
    # prefix (outbase + P or the sum of earlier rows' M) is zero, so only the row's first window carries one
    assert g.prefixed == 0
    # 512-partition fallback: mixed LIST / FAST rows
    lay = Layout(syn.make_config(groups=fallback_groups(), modes=MODES8, order=RATING))
    _, rating, mode, _ = uniform_pool(pkg, 12, 1_000_000, 0, 4999, n_modes=8)
    g = Geometry(lay, lay.fills(rating, mode))
    assert not g.halves and g.mixed_rows >= 20 and g.hist == "hist", g.summary()
    assert Geometry(lay, lay.fills(rating, mode), rank_impl=2).mixed_rows == 0


# ================================================================================ GPU
def key_domain_edge(pkg, accepts):
    """Largest rating span S (one group 0..S, 2 modes) that `accepts`; binary search."""
    lo, hi = 1, 40_000
    assert accepts(edge_config(pkg, lo)) and not accepts(edge_config(pkg, hi))
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if accepts(edge_config(pkg, mid)) else (lo, mid)
    return lo


def edge_config(pkg, span, flags=0, capacity=4096):
    return pkg.synth.make_config(groups=[(0, span)], modes=MODES8[:2], order=RATING, default_group=0,
                                 capacity=capacity, flags=flags)


def check(eng, ref, lob, mem, seq, st, seq_of=None):
    assert (st.n_lobbies, st.n_matched, st.n_residual, st.n_dead) == (ref.n_lobbies, ref.n_matched, ref.n_residual,
                                                                        ref.n_dead)
    assert np.array_equal(lob, ref.lobbies)
    assert np.array_equal(mem, ref.member_ids)
    assert np.array_equal(seq, ref.emit_seq if seq_of is None else np.asarray(seq_of, np.uint32)[ref.emit_seq])
    assert np.array_equal(eng.pool_read()["id"], ref.residual_ids)


def run_regime(pkg, oracle, cfg, pool, variants, fused, alive=None, spread=-1, big=False, new_arrivals=None):
    """Tick the pool on a fresh engine per (tick_impl, rank_impl) variant against the oracle; then remove and take
    some of the leftovers, add new arrivals and tick the compacted pool again.  fused: tick_impl 1 runs the single
    cooperative launch (Layout.fused: False where a phase's shared memory leaves fewer CTAs per SM than rows)."""
    ids, rating, mode, ts = pool
    n = len(ids)
    if spread >= 0:
        ref = oracle.run_windowed(cfg, spread, ids, rating, mode, alive)
    elif big:
        ref = NumpyTick(cfg, ids, rating, mode, alive)
    else:
        ref = oracle.run_closed_form(cfg, ids, rating, mode, alive)
    keep = np.isin(ids, ref.residual_ids)
    q_ids, q_r, q_m, q_seq = ids[keep], rating[keep], mode[keep], np.nonzero(keep)[0].astype(np.uint32)
    rng = np.random.default_rng(len(q_ids))
    gone = rng.random(len(q_ids)) < 0.1
    taken = ~gone & (rng.random(len(q_ids)) < 0.1)
    a_ids, a_r, a_m, a_ts = new_arrivals
    a_ids = a_ids + (np.uint64(n) if cfg.flags & DENSE else np.uint64(0))
    # removed and taken players both leave the pool at the next tick and count as dead there
    q2 = [np.concatenate([q_ids, a_ids]), np.concatenate([q_r, a_r]), np.concatenate([q_m, a_m])]
    alive2 = np.concatenate([~(gone | taken), np.ones(len(a_ids), bool)]).astype(np.uint8)
    seq2 = np.concatenate([q_seq, n + np.arange(len(a_ids), dtype=np.uint32)])
    ref2 = (oracle.run_windowed(cfg, spread, *q2, alive2) if spread >= 0 else
            oracle.run_closed_form(cfg, *q2, alive2))
    for tick_impl, rank_impl in variants:
        with pkg.Engine(cfg) as eng:
            eng.set_option("tick_impl", tick_impl)
            eng.set_option("rank_impl", rank_impl)
            eng.set_option("max_spread", spread)
            assert (eng.enqueue(ids, rating, mode, ts) == 1).all()
            if alive is not None:
                assert eng.remove(ids[alive == 0]) == int((alive == 0).sum())
            lob, mem, seq, st = eng.tick()
            assert st.n_launches == (1 if tick_impl == 1 and fused else 4)
            check(eng, ref, lob, mem, seq, st)
            assert eng.remove(q_ids[gone]) == int(gone.sum())
            assert eng.take(q_ids[taken]) == int(taken.sum())
            assert (eng.enqueue(a_ids, a_r, a_m, a_ts) == 1).all()
            lob, mem, seq, st = eng.tick()
            check(eng, ref2, lob, mem, seq, st, seq_of=seq2)
            del lob, mem, seq


def assert_regime(g, **want):
    s = g.summary()
    for k, v in want.items():
        assert s[k] == v, (k, s)


BOTH_RANKINGS = ((1, 3), (0, 3), (1, 2))
LIST_ONLY = ((1, 3), (0, 3))


@pytest.mark.gpu
@pytest.mark.parametrize("removed", [0.0, 0.02])
def test_many_partitions_per_row(pkg, oracle, removed):
    """160 partitions, 4 to a slot-counter window: rows of 5 single-tile partitions reload their window mid-row, on
    both tile pipelines."""
    cfg = pkg.synth.make_config(groups=[(250 * g, 250 * g + 249) for g in range(20)], modes=MODES8, order=RATING,
                                capacity=2_200_000)
    pool = many_partitions_pool(pkg)
    n = len(pool[0])
    lay = Layout(cfg, Device.current())
    g = Geometry(lay, lay.fills(pool[1], pool[2]))
    assert lay.n_segs == 160 and g.halves and g.max_parts >= 5, g.summary()
    assert g.reloads[0] >= 8 and g.reloads[1] >= 8, g.summary()
    alive = (np.random.default_rng(3).random(n) >= removed).astype(np.uint8) if removed else None
    arrivals = uniform_pool(pkg, 99, 100_000, 0, 4999, n_modes=8)
    run_regime(pkg, oracle, cfg, pool, BOTH_RANKINGS, lay.fused, alive=alive, new_arrivals=arrivals)


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
def test_rows_longer_than_the_descriptor_cache(pkg, oracle, order):
    """config3's shape at 40 M players: rows of more than 64 tiles, so placement and the histogram row sums read the
    descriptors past the cache from the tile geometry."""
    n = 40_000_000
    cfg = pkg.synth.make_config(n_groups=32, modes=MODES8[3:4], order=order, capacity=n + 200_000,
                                active_capacity=n + 200_000, flags=DENSE)
    pool = config3_pool(pkg, n)
    lay = Layout(cfg, Device.current())
    g = Geometry(lay, lay.fills(pool[1], pool[2]))
    assert g.halves and g.max_tiles >= 70 and g.rows_past_cache >= g.rows // 2, g.summary()
    arrivals = uniform_pool(pkg, 98, 150_000, -10, 5010, dense=True)
    run_regime(pkg, oracle, cfg, pool, BOTH_RANKINGS, lay.fused, big=True, new_arrivals=arrivals)


@pytest.mark.gpu
@pytest.mark.parametrize("order", [RATING, ARRIVAL])
def test_partition_fallback_mixes_list_and_fast_tiles(pkg, oracle, order):
    """8 modes x 64 groups with four groups wider than 255 keys: the split would need more than 512 partitions, so
    every segment stays whole; rows hold LIST tiles (260 keys) next to FAST ones."""
    cfg = pkg.synth.make_config(groups=fallback_groups(), modes=MODES8, order=order, capacity=1_000_000)
    pool = uniform_pool(pkg, 12, 1_000_000, 0, 4999, n_modes=8)
    lay = Layout(cfg, Device.current())
    g = Geometry(lay, lay.fills(pool[1], pool[2]))
    if order == RATING:
        assert lay.n_segs == 512 and lay.max_nb == 260 and not g.halves and g.mixed_rows >= 20, g.summary()
    alive = (np.random.default_rng(4).random(len(pool[0])) > 0.02).astype(np.uint8)
    arrivals = uniform_pool(pkg, 97, 100_000, 0, 4999, n_modes=8)
    run_regime(pkg, oracle, cfg, pool, BOTH_RANKINGS if order == RATING else LIST_ONLY, lay.fused, alive=alive,
               new_arrivals=arrivals)


@pytest.mark.gpu
@pytest.mark.parametrize("heavy", [False, True])
def test_wide_partitions_alternating_with_narrow(pkg, oracle, heavy):
    """MM_F_WIDE_PARTITIONS, narrow and wide groups alternating: rows switch between LIST and FAST tiles; with every
    player of a wide group at one rating the LIST ranking aggregates per warp (heavy)."""
    n = 1_000_000
    cfg = pkg.synth.make_config(groups=ALT_GROUPS, modes=MODES8[:2], order=RATING, capacity=n, flags=WIDE)
    ids, rating, mode, ts = uniform_pool(pkg, 21, n, 0, 5000, n_modes=2)
    if heavy:
        rating[(rating >= 1400) & (rating <= 2999)] = 2000
    lay = Layout(cfg, Device.current())
    g = Geometry(lay, lay.fills(rating, mode))
    assert lay.max_nb == 1800 and not g.halves and g.mixed_rows >= 6 and g.transitions >= 6, g.summary()
    assert lay.heavy(rating, mode) == heavy
    arrivals = uniform_pool(pkg, 96, 100_000, 0, 5000, n_modes=2)
    run_regime(pkg, oracle, cfg, (ids, rating, mode, ts), BOTH_RANKINGS, lay.fused, new_arrivals=arrivals)


@pytest.mark.gpu
@pytest.mark.parametrize("spread", [-1, 0])
@pytest.mark.parametrize("wide", [1, 0])
def test_huge_key_domain(pkg, oracle, wide, spread):
    """One group over ratings 0..20 000.  Whole (MM_F_WIDE_PARTITIONS): 20 003 keys in one partition, one CTA per SM
    with a 4-stage ring, LIST ranking on the streamed histogram, rows past the descriptor cache.  Split: 79
    partitions per mode on the chunk-histogram path."""
    n = 20_000_000
    cfg = pkg.synth.make_config(groups=[(0, 20000)], modes=MODES8[3:4], order=RATING, default_group=0,
                                capacity=n + 200_000, active_capacity=n + 200_000, flags=DENSE | (WIDE * wide))
    pool = uniform_pool(pkg, 31, n, -5, 20005, dense=True)
    lay = Layout(cfg, Device.current())
    g = Geometry(lay, lay.fills(pool[1], pool[2]))
    if wide:
        assert (lay.max_nb, lay.rows_per_sm, lay.stages, g.hist, g.halves) == (20003, 1, 4, "hist", False), g.summary()
        assert g.max_tiles >= 70 and g.rows_past_cache >= g.rows // 2 and g.colscan, g.summary()
    else:
        assert (lay.n_segs, lay.rows_per_sm, g.hist, g.halves) == (79, 2, "rowsum", True), g.summary()
    arrivals = uniform_pool(pkg, 95, 150_000, -5, 20005, dense=True)
    run_regime(pkg, oracle, cfg, pool, LIST_ONLY if wide else BOTH_RANKINGS, lay.fused, spread=spread, big=spread < 0,
               new_arrivals=arrivals)


@pytest.mark.gpu
def test_key_domain_edge(pkg, oracle):
    """The largest rating span mm_create accepts with 2 modes is the model's; one more gives MM_E_ARG (not a CUDA
    error), and a tick at the edge matches the oracle under S0 and S1."""
    lib = pkg.load_library()

    def create(cfg):
        h = C.c_void_p()
        rc = lib.mm_create(C.byref(cfg), C.byref(h))
        if rc == pkg.abi.MM_OK:
            lib.mm_destroy(h)
        assert rc in (pkg.abi.MM_OK, pkg.abi.MM_E_ARG), rc
        return rc == pkg.abi.MM_OK

    dev = Device.current()
    span = key_domain_edge(pkg, create)
    assert span == key_domain_edge(pkg, lambda cfg: Layout(cfg, dev).ok)
    for flags in (0, WIDE):
        assert create(edge_config(pkg, span, flags)) and not create(edge_config(pkg, span + 1, flags))
    n = 600_000
    cfg = edge_config(pkg, span, capacity=n)
    pool = uniform_pool(pkg, 41, n, -3, span + 3, n_modes=2)
    arrivals = uniform_pool(pkg, 94, 50_000, -3, span + 3, n_modes=2)
    for spread in (-1, 2):
        run_regime(pkg, oracle, cfg, pool, BOTH_RANKINGS, Layout(cfg, dev).fused, spread=spread, new_arrivals=arrivals)
