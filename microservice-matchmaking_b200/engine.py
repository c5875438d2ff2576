"""Python host binding of libmm_engine.so (ctypes over include/mm_engine.h).

Mirrors the Elixir-side module SURVEY §8(b) sketches (`Matchmaking.Search.Engine`:
new / enqueue / remove / in_queue? / tick / status) — columns cross the boundary as
flat numpy buffers, never per-player objects.  No compute happens in Python and
there is no CPU fallback: a missing library raises at load time.
"""
import ctypes as C
import os

import numpy as np

from . import abi

_CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc")
_lib = None


class EngineError(RuntimeError):
    def __init__(self, status, what, detail=""):
        self.status = status
        super().__init__(f"{what}: status {status}{(' — ' + detail) if detail else ''}")


def library_path():
    return os.path.join(_CSRC, "libmm_engine.so")


def load_library():
    """dlopen csrc/libmm_engine.so and bind every symbol of mm_engine.h."""
    global _lib
    if _lib is None:
        path = library_path()
        if not os.path.exists(path):
            raise ImportError(
                f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a).  There is no CPU fallback for the search tick.")
        _lib = abi.bind(C.CDLL(path))
        if _lib.mm_abi_version() != abi.MM_ABI_VERSION:
            raise ImportError("libmm_engine.so ABI version mismatch")
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


LOBBY_DTYPE = np.dtype([("first_member", "<u4"), ("n_members", "<u2"), ("mode", "u1"), ("group", "u1")])

# mm_player_status (include/mm_engine.h) as a numpy record
PLAYER_STATUS_DTYPE = np.dtype([
    ("state", "u1"), ("mode", "u1"), ("group", "u1"), ("reserved", "u1"), ("rating", "<i4"), ("enq_ts", "<u4"),
    ("seq", "<u4"), ("wait", "<u4"), ("ahead", "<u4"), ("depth", "<u4"), ("lobby", "<u4"), ("member", "<u2"),
    ("reserved2", "<u2")])
assert PLAYER_STATUS_DTYPE.itemsize == C.sizeof(abi.PlayerStatus)

# mm_queue_stat (include/mm_engine.h) as a numpy record
QUEUE_STAT_DTYPE = np.dtype([
    ("mode", "u1"), ("group", "u1"), ("reserved", "<u2"),
    ("n_waiting", "<u4"), ("n_removed", "<u4"), ("max_wait", "<u4"), ("wait_hist", "<u4", (abi.MM_WAIT_BUCKETS,)),
    ("n_lobbies", "<u4"), ("n_matched", "<u4"), ("max_match_wait", "<u4"),
    ("match_wait_hist", "<u4", (abi.MM_WAIT_BUCKETS,)),
])

# mm_party_queue_stat / mm_party_member_status (include/mm_engine.h) as numpy records
PARTY_QUEUE_STAT_DTYPE = np.dtype([
    ("mode", "u1"), ("group", "u1"), ("reserved", "<u2"), ("n_parties", "<u4"), ("n_members", "<u4"),
    ("max_wait", "<u4"), ("wait_hist", "<u4", (abi.MM_WAIT_BUCKETS,)), ("size_hist", "<u4", (abi.MM_PARTY_SIZE_BUCKETS,)),
])
assert PARTY_QUEUE_STAT_DTYPE.itemsize == C.sizeof(abi.PartyQueueStat)
PARTY_MEMBER_STATUS_DTYPE = np.dtype([
    ("state", "u1"), ("mode", "u1"), ("group", "u1"), ("size", "u1"), ("index", "u1"), ("anchor", "u1"),
    ("reserved", "<u2"), ("rating", "<i4"), ("party_rating", "<i4"), ("enq_ts", "<u4"), ("seq", "<u4"), ("wait", "<u4"),
    ("window", "<i4"), ("ahead", "<u4"), ("depth", "<u4"), ("lobby", "<u4"), ("member", "<u2"), ("reserved2", "<u2")])
assert PARTY_MEMBER_STATUS_DTYPE.itemsize == C.sizeof(abi.PartyMemberStatus)

# mm_lobby_quality / mm_queue_quality (include/mm_engine.h) as numpy records
LOBBY_QUALITY_DTYPE = np.dtype([("min_rating", "<i4"), ("max_rating", "<i4"), ("rating_sum", "<i8"),
                                ("imbalance", "<u4"), ("reserved", "<u4")])
assert LOBBY_QUALITY_DTYPE.itemsize == C.sizeof(abi.LobbyQuality)
QUALITY_DTYPE = np.dtype([
    ("mode", "u1"), ("group", "u1"), ("reserved", "<u2"),
    ("n_lobbies", "<u4"), ("max_spread", "<u4"), ("max_imbalance", "<u4"), ("sum_spread", "<u8"),
    ("sum_imbalance", "<u8"), ("spread_hist", "<u4", (abi.MM_WAIT_BUCKETS,)),
    ("imbalance_hist", "<u4", (abi.MM_WAIT_BUCKETS,)),
])
assert QUALITY_DTYPE.itemsize == C.sizeof(abi.QueueQuality)

# mm_match_waits (include/mm_engine.h) as a numpy record: the match section of QUEUE_STAT_DTYPE
WAITS_DTYPE = np.dtype([
    ("mode", "u1"), ("group", "u1"), ("reserved", "<u2"), ("n_lobbies", "<u4"), ("n_matched", "<u4"),
    ("max_match_wait", "<u4"), ("match_wait_hist", "<u4", (abi.MM_WAIT_BUCKETS,)),
])
assert WAITS_DTYPE.itemsize == C.sizeof(abi.MatchWaits)


def wait_of(now, enq_ts):
    """Wait of a player as mm_queue_stats counts it: (now - enq_ts) mod 2^32 read as a signed 32-bit value, negative
    ("in the future") clamped to 0."""
    d = (np.asarray(now, np.uint64) - np.asarray(enq_ts, np.uint64)) & np.uint64(0xFFFFFFFF)
    w = d.astype(np.uint32).view(np.int32) if d.ndim else np.uint32(d).view(np.int32)
    return np.maximum(w, 0).astype(np.int64)


def wait_bucket(w):
    """Histogram bucket of a wait w in [0, 2^31): w below 8, else 8 + 4 (e - 3) + ((w >> (e - 2)) & 3) with
    e = floor(log2 w) — four sub-buckets per octave, 120 in all."""
    w = np.asarray(w, np.int64)
    e = np.maximum(np.frexp(w.astype(np.float64))[1] - 1, 3)  # floor(log2 w), exact for integers below 2^53
    b = np.where(w < 8, w, 8 + 4 * (e - 3) + ((w >> (e - 2)) & 3))
    return b if b.ndim else int(b)


def quality_bucket(v):
    """Histogram bucket of a spread or imbalance in rating points (mm_match_quality): wait_bucket's, with every value
    of 2^31 or more in the last bucket."""
    v = np.asarray(v, np.int64)
    b = np.where(v >= 1 << 31, abi.MM_WAIT_BUCKETS - 1, wait_bucket(np.minimum(v, (1 << 31) - 1)))
    return b if b.ndim else int(b)


def wait_bucket_bounds():
    """-> (lo, hi) int64[MM_WAIT_BUCKETS]: bucket b holds the waits [lo[b], hi[b]); together [0, 2^31) without gaps."""
    b = np.arange(abi.MM_WAIT_BUCKETS, dtype=np.int64)
    e = 3 + (b - 8) // 4
    s = (b - 8) % 4
    lo = np.where(b < 8, b, (4 + s) << np.maximum(e - 2, 0))
    hi = np.where(b < 8, b + 1, (5 + s) << np.maximum(e - 2, 0))
    return lo, hi


def wait_quantile(hist, q):
    """Upper bound (the largest wait it holds) of the bucket that holds the q-quantile of a wait histogram; 0 for an
    empty one.  Exact for waits below 8, at most 25 % high above."""
    hist = np.asarray(hist, np.int64)
    total = int(hist.sum())
    if total == 0:
        return 0
    rank = min(total, max(1, int(np.ceil(q * total))))
    b = int(np.searchsorted(np.cumsum(hist), rank))
    return int(wait_bucket_bounds()[1][b] - 1)


def read_image(buf):
    """Parse an mm_export image without a GPU -> (abi.ImageHeader, dict of numpy views: part_count, id, rating,
    enq_ts, seq, mode, active).  Raises ValueError when the buffer is shorter than its header says."""
    buf = np.frombuffer(buf, np.uint8) if isinstance(buf, (bytes, bytearray, memoryview)) else np.asarray(buf, np.uint8)
    if len(buf) < C.sizeof(abi.ImageHeader):
        raise ValueError("image shorter than its header")
    h = abi.ImageHeader.from_buffer_copy(buf[:C.sizeof(abi.ImageHeader)].tobytes())
    off = abi.image_offsets(h.n_parts, h.n_players, h.n_active, h.id_bytes)
    if len(buf) < off[-1]:
        raise ValueError("image shorter than its sections")
    idt = np.uint64 if h.id_bytes == 8 else np.uint32
    n, m = h.n_players, h.n_active
    cols = {}
    for k, (name, dt, cnt) in enumerate((("part_count", np.uint32, h.n_parts), ("id", idt, n), ("rating", np.int32, n),
                                         ("enq_ts", np.uint32, n), ("seq", np.uint32, n), ("mode", np.uint8, n),
                                         ("active", idt, m))):
        cols[name] = buf[off[k]:off[k] + cnt * np.dtype(dt).itemsize].view(dt)
    return h, cols


def active_set_limit(cfg):
    """Ids a hashed active set holds at its 3/4 load (the table size mm_create picks for cfg); None for an engine
    without one (MM_F_NO_DEDUPE) or with a direct-mapped handle table (MM_F_DENSE_IDS)."""
    if int(cfg.flags) & 3:
        return None
    want = cfg.active_capacity or 2 * cfg.capacity
    h = 1024
    while h * 3 < want * 4 + 64:
        h <<= 1
    return h * 3 // 4


def read_party_image(buf):
    """Parse an mm_export_parties image without a GPU -> (abi.ImageHeader, dict of numpy views: size, seq, enq_ts, mode
    per party, id and rating per member).  Raises ValueError when the buffer is shorter than its header says."""
    buf = np.frombuffer(buf, np.uint8) if isinstance(buf, (bytes, bytearray, memoryview)) else np.asarray(buf, np.uint8)
    if len(buf) < C.sizeof(abi.ImageHeader):
        raise ValueError("party image shorter than its header")
    h = abi.ImageHeader.from_buffer_copy(buf[:C.sizeof(abi.ImageHeader)].tobytes())
    off = abi.party_image_offsets(h.n_parts, h.n_players, h.id_bytes)
    if len(buf) < off[-1]:
        raise ValueError("party image shorter than its sections")
    idt = np.uint64 if h.id_bytes == 8 else np.uint32
    p, m = h.n_parts, h.n_players
    cols = {}
    for k, (name, dt, cnt) in enumerate((("size", np.uint8, p), ("seq", np.uint32, p), ("enq_ts", np.uint32, p),
                                         ("mode", np.uint8, p), ("id", idt, m), ("rating", np.int32, m))):
        cols[name] = buf[off[k]:off[k] + cnt * np.dtype(dt).itemsize].view(dt)
    return h, cols


class Engine:
    """One GPU-resident player pool + active set + search tick (single writer)."""

    def __init__(self, cfg):
        self.lib = load_library()
        self.cfg = cfg
        h = C.c_void_p()
        rc = self.lib.mm_create(C.byref(cfg), C.byref(h))
        if rc != abi.MM_OK:
            raise EngineError(rc, "mm_create", self.lib.mm_strerror(rc).decode())
        self.h = h
        self._staged = []  # host arrays of staged packed batches (kept alive until their _end)

    # -- lifecycle ---------------------------------------------------------------
    def close(self):
        if getattr(self, "h", None):
            self.lib.mm_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _check(self, rc, what):
        if rc != abi.MM_OK:
            raise EngineError(rc, what, self.lib.mm_strerror(rc).decode() + " " + self.lib.mm_last_error(self.h).decode())

    # -- active set + ingest -----------------------------------------------------
    def enqueue(self, ids, rating, mode, enq_ts=None):
        """-> accepted u8[n]: 1 queued, 0 already in the queue, 2 invalid, 3 full."""
        ids = np.ascontiguousarray(ids, np.uint64)
        rating = np.ascontiguousarray(rating, np.int32)
        mode = np.ascontiguousarray(mode, np.uint8)
        n = len(ids)
        assert len(rating) == n and len(mode) == n
        if enq_ts is not None:
            enq_ts = np.ascontiguousarray(enq_ts, np.uint32)
        acc = np.empty(n, np.uint8)
        self._check(self.lib.mm_enqueue(self.h, n, _p(ids), _p(rating), _p(mode), _p(enq_ts), _p(acc)), "mm_enqueue")
        return acc

    def enqueue_raw(self, n, p_ids, p_rating, p_mode, p_ts=0, p_accepted=0):
        """mm_enqueue on raw HOST addresses (e.g. pinned torch tensors' data_ptr())."""
        self._check(self.lib.mm_enqueue(self.h, n, p_ids, p_rating, p_mode, p_ts or None, p_accepted or None),
                    "mm_enqueue")

    def tick_raw(self, p_lobbies, lobby_cap, p_members, member_cap, p_emit_seq=0, now=0, packed=False):
        """mm_tick (u64 ids) / mm_tick_packed (u32 handles) on raw HOST addresses. -> TickStats"""
        st = abi.TickStats()
        fn = self.lib.mm_tick_packed if packed else self.lib.mm_tick
        self._check(fn(self.h, now, p_lobbies, lobby_cap, p_members, member_cap, p_emit_seq or None, C.byref(st)),
                    "mm_tick_packed" if packed else "mm_tick")
        return st

    # -- packed host formats (MM_F_DENSE_IDS engines): u32 handle + u16 (mode << 13 | rating) --------------
    @staticmethod
    def pack_key(rating, mode):
        rating = np.asarray(rating)
        assert rating.min(initial=0) >= 0 and rating.max(initial=0) <= 8191, "packed keys carry ratings 0..8191"
        return (np.asarray(mode, np.uint16) << 13 | rating.astype(np.uint16)).astype(np.uint16)

    def enqueue_packed(self, handles, keys, enq_ts=None):
        """-> accepted u8[n] (codes as enqueue)."""
        handles = np.ascontiguousarray(handles, np.uint32)
        keys = np.ascontiguousarray(keys, np.uint16)
        n = len(handles)
        assert len(keys) == n
        if enq_ts is not None:
            enq_ts = np.ascontiguousarray(enq_ts, np.uint32)
        acc = np.empty(n, np.uint8)
        self._check(self.lib.mm_enqueue_packed(self.h, n, _p(handles), _p(keys), _p(enq_ts), _p(acc)), "mm_enqueue_packed")
        return acc

    def enqueue_packed_raw(self, n, p_handles, p_keys, p_ts=0, p_accepted=0):
        self._check(self.lib.mm_enqueue_packed(self.h, n, p_handles, p_keys, p_ts or None, p_accepted or None),
                    "mm_enqueue_packed")

    def enqueue_packed_begin(self, handles, keys, enq_ts=None):
        """Start the upload of a packed batch (mm_enqueue_packed_begin); the arrays are kept alive until the matching
        enqueue_packed_end()."""
        handles = np.ascontiguousarray(handles, np.uint32)
        keys = np.ascontiguousarray(keys, np.uint16)
        assert len(keys) == len(handles)
        if enq_ts is not None:
            enq_ts = np.ascontiguousarray(enq_ts, np.uint32)
        self._check(self.lib.mm_enqueue_packed_begin(self.h, len(handles), _p(handles), _p(keys), _p(enq_ts)),
                    "mm_enqueue_packed_begin")
        self._staged.append((handles, keys, enq_ts))

    def enqueue_packed_end(self, want_codes=True):
        """Ingest the oldest staged batch -> (accepted u8[n] or None, n_accepted)."""
        acc = None
        if want_codes and self._staged:
            acc = np.empty(len(self._staged[0][0]), np.uint8)
        n_acc = C.c_uint32(0)
        rc = self.lib.mm_enqueue_packed_end(self.h, _p(acc), C.byref(n_acc))
        if self._staged:
            self._staged.pop(0)
        self._check(rc, "mm_enqueue_packed_end")
        return acc, n_acc.value

    def enqueue_packed_begin_raw(self, n, p_handles, p_keys, p_ts=0):
        self._check(self.lib.mm_enqueue_packed_begin(self.h, n, p_handles, p_keys, p_ts or None), "mm_enqueue_packed_begin")

    def enqueue_packed_end_raw(self):
        n_acc = C.c_uint32(0)
        self._check(self.lib.mm_enqueue_packed_end(self.h, None, C.byref(n_acc)), "mm_enqueue_packed_end")
        return n_acc.value

    def enqueue_rejects(self, cap=4096):
        """(batch index, code) of the entries of the last enqueue batch that were not queued (unordered)."""
        while True:
            idx = np.empty(cap, np.uint32)
            code = np.empty(cap, np.uint8)
            n = C.c_uint32(0)
            rc = self.lib.mm_enqueue_rejects(self.h, cap, _p(idx), _p(code), C.byref(n))
            if rc == abi.MM_E_CAP:
                cap = n.value
                continue
            self._check(rc, "mm_enqueue_rejects")
            return idx[:n.value], code[:n.value]

    def remove_packed(self, handles):
        handles = np.ascontiguousarray(handles, np.uint32)
        nr = C.c_uint32(0)
        self._check(self.lib.mm_remove_packed(self.h, len(handles), _p(handles), C.byref(nr)), "mm_remove_packed")
        return nr.value

    def tick_packed(self, now=0, lobby_cap=None, member_cap=None, want_emit_seq=True):
        """Host-buffer tick, members as u32 handles -> (lobbies, member_handles u32, emit_seq|None, TickStats)."""
        n = self.pool_size()
        member_cap = max(n, 1) if member_cap is None else member_cap
        lobby_cap = max(n // 2, 1) if lobby_cap is None else lobby_cap
        lob = np.empty(lobby_cap, LOBBY_DTYPE)
        mem = np.empty(member_cap, np.uint32)
        seq = np.empty(lobby_cap, np.uint32) if want_emit_seq else None
        st = abi.TickStats()
        self._check(self.lib.mm_tick_packed(self.h, now, _p(lob), lobby_cap, _p(mem), member_cap, _p(seq), C.byref(st)),
                    "mm_tick_packed")
        self.results_wait()
        return lob[:st.n_lobbies], mem[:st.n_matched], (seq[:st.n_lobbies] if seq is not None else None), st

    def enqueue_device(self, n, d_ids, d_rating, d_mode, d_ts=0, d_accepted=0):
        """Device-pointer ingest (ints = raw device addresses). -> n_accepted"""
        na = C.c_uint32(0)
        self._check(self.lib.mm_enqueue_device(self.h, n, d_ids, d_rating, d_mode, d_ts or None, d_accepted or None,
                                               C.byref(na)), "mm_enqueue_device")
        return na.value

    def remove(self, ids):
        ids = np.ascontiguousarray(ids, np.uint64)
        nr = C.c_uint32(0)
        self._check(self.lib.mm_remove(self.h, len(ids), _p(ids), C.byref(nr)), "mm_remove")
        return nr.value

    def take(self, ids):
        """Queued players matched outside this engine's tick leave the pool but stay active (mm_take). -> count"""
        ids = np.ascontiguousarray(ids, np.uint64)
        nt = C.c_uint32(0)
        self._check(self.lib.mm_take(self.h, len(ids), _p(ids), C.byref(nt)), "mm_take")
        return nt.value

    def seq_next(self):
        """The enqueue sequence number the next offered player will get (mm_seq_next)."""
        v = C.c_uint32(0)
        self._check(self.lib.mm_seq_next(self.h, C.byref(v)), "mm_seq_next")
        return v.value

    def requeue(self, ids, rating, mode, enq_ts, seq):
        """Put players of a lobby that did not start back into their queue at their enqueue position (mm_requeue).
        The columns are what each player had when it was queued (enq_ts may be None).  The entries may come in any
        order: they are sorted by age here.  -> codes u8[n] in the caller's order: 1 requeued, 0 still queued,
        4 not in the active set (the player left).  The members of a matched party share the party's seq: at most one
        of them per call, not one whose partition already holds a co-member requeued earlier, and not one whose own
        rating has no group (each MM_E_ARG)."""
        ids = np.ascontiguousarray(ids, np.uint64)
        n = len(ids)
        seq = np.ascontiguousarray(seq, np.uint32)
        assert len(rating) == n and len(mode) == n and len(seq) == n
        order = np.argsort((seq - np.uint32(self.seq_next())).astype(np.uint32))  # a tie is refused: no order to keep
        cols = [np.ascontiguousarray(np.asarray(a)[order], dt) for a, dt in
                ((ids, np.uint64), (rating, np.int32), (mode, np.uint8), (seq, np.uint32))]
        ts = None if enq_ts is None else np.ascontiguousarray(np.asarray(enq_ts)[order], np.uint32)
        codes = np.empty(n, np.uint8)
        k = C.c_uint32(0)
        self._check(self.lib.mm_requeue(self.h, n, _p(cols[0]), _p(cols[1]), _p(cols[2]), _p(ts), _p(cols[3]),
                                        _p(codes), C.byref(k)), "mm_requeue")
        out = np.empty(n, np.uint8)
        out[order] = codes
        return out

    # -- boundary pass on the device (mm_band_candidates / mm_band_match) ----------------------------------------
    def band_candidates(self, W, group):
        """The upper side of the boundary group-1 | group: live queued players of `group` with rating in
        (hi_{group-1}, hi_{group-1} + W], sorted by (mode, rating, enqueue order) -> (ids u64, rating i32, mode u8)."""
        cap = 1 << 14
        while True:
            ids, rating, mode = np.empty(cap, np.uint64), np.empty(cap, np.int32), np.empty(cap, np.uint8)
            n = C.c_uint32(0)
            rc = self.lib.mm_band_candidates(self.h, int(W), int(group), _p(ids), _p(rating), _p(mode), cap, C.byref(n))
            if rc == abi.MM_E_CAP and n.value > cap:
                cap = n.value
                continue
            self._check(rc, "mm_band_candidates")
            k = n.value
            return ids[:k], rating[:k], mode[:k]

    def band_match(self, W, g_first, g_last, upper=None):
        """Match the bands of the boundaries g|g+1, g_first <= g <= g_last, and take the local matched players.
        upper: (ids, rating, mode) of the upper side of boundary g_last|g_last+1 from another engine
        (band_candidates), or None to read it from this engine.
        -> (lobbies[LOBBY_DTYPE], member_ids u64, upper_taken bool[len(upper ids)], BandStats)"""
        remote = upper is not None
        if remote:
            up = (np.ascontiguousarray(upper[0], np.uint64), np.ascontiguousarray(upper[1], np.int32),
                  np.ascontiguousarray(upper[2], np.uint8))
        else:
            up = (np.zeros(0, np.uint64), np.zeros(0, np.int32), np.zeros(0, np.uint8))
        n_up = len(up[0])
        taken = np.zeros(max(n_up, 1), np.uint8)
        lobby_cap, member_cap = 1 << 10, 1 << 12  # resized from the counts of an MM_E_CAP refusal
        while True:
            lob = np.empty(lobby_cap, LOBBY_DTYPE)
            mem = np.empty(member_cap, np.uint64)
            st = abi.BandStats()
            rc = self.lib.mm_band_match(self.h, int(W), int(g_first), int(g_last), int(remote), _p(up[0]), _p(up[1]),
                                        _p(up[2]), n_up, _p(lob), lobby_cap, _p(mem), member_cap, _p(taken), C.byref(st))
            if rc == abi.MM_E_CAP and (st.n_lobbies > lobby_cap or st.n_matched > member_cap):
                lobby_cap, member_cap = max(lobby_cap, st.n_lobbies), max(member_cap, st.n_matched)
                continue
            self._check(rc, "mm_band_match")
            return lob[:st.n_lobbies], mem[:st.n_matched], taken[:n_up].astype(bool), st

    # -- backfill (mm_backfill) ------------------------------------------------------------------------------------
    def backfill(self, mode, group, target, count, window=None):
        """Fill the open slots of running lobbies from their queues: request j takes up to count[j] live queued players
        of queue (mode[j], group[j]), nearest to target[j] first within `window` (None or < 0: no limit) on a
        rating-order engine, the oldest first on an arrival-order one (target ignored, window must be None or < 0).
        Arguments are scalars or arrays of one length.  -> (n_taken u32[n], [member ids u64 of request j, ...])"""
        cols = np.broadcast_arrays(*(np.asarray(x, np.int64) for x in
                                     (mode, group, target, count, -1 if window is None else window)))
        n = cols[0].size
        req = np.zeros(n, np.dtype([("mode", "u1"), ("group", "u1"), ("reserved", "<u2"), ("count", "<u4"),
                                    ("target", "<i4"), ("window", "<i4")]))
        for name, col in zip(("mode", "group", "target", "count", "window"), cols):
            req[name] = col.ravel()
        n_taken = np.zeros(max(n, 1), np.uint32)
        cap = 1 << 12  # resized from the total of an MM_E_CAP refusal
        while True:
            mem = np.empty(cap, np.uint64)
            total = C.c_uint32(0)
            rc = self.lib.mm_backfill(self.h, n, _p(req), _p(n_taken), _p(mem), cap, C.byref(total))
            if rc == abi.MM_E_CAP and total.value > cap:
                cap = total.value
                continue
            self._check(rc, "mm_backfill")
            n_taken = n_taken[:n].copy()
            if n == 0:
                return n_taken, []
            return n_taken, np.split(mem[:total.value], np.cumsum(n_taken.astype(np.int64))[:-1])

    # -- party backfill (mm_backfill_party) ---------------------------------------------------------------------------
    def backfill_party(self, mode, group, target, room, window=None):
        """Fill the open team slots of running lobbies with whole queued parties of their queues, then with the nearest
        solos (rating-order engines with party_capacity set).  mode, group, target and window are scalars or arrays of
        the n requests' length (window None or < 0: no limit); room holds one list of open slots per team for each
        request (one list for a single request given as scalars).  -> (filled, members): per request, the members each
        team received and one u64 id array per team (its parties first, then its solos)."""
        cols = np.broadcast_arrays(*(np.asarray(x, np.int64) for x in (mode, group, target,
                                                                        -1 if window is None else window)))
        n = cols[0].size
        if n == 1 and len(room) and np.ndim(room[0]) == 0:
            room = [room]
        room = [np.asarray(r, np.int64).ravel() for r in room]
        if len(room) != n:
            raise ValueError(f"{len(room)} room lists for {n} requests")
        for j, (m, r) in enumerate(zip(cols[0].ravel().tolist(), room)):  # the engine reads `teams` entries per request
            if 0 <= m < self.cfg.n_modes and r.size != self.cfg.modes[m].teams:
                raise ValueError(f"request {j}: {r.size} room entries for a mode of {self.cfg.modes[m].teams} teams")
        req = np.zeros(n, np.dtype([("mode", "u1"), ("group", "u1"), ("reserved", "<u2"), ("count", "<u4"),
                                    ("target", "<i4"), ("window", "<i4")]))
        for name, col in zip(("mode", "group", "target", "window"), cols):
            req[name] = col.ravel()
        req["count"] = [int(r.sum()) for r in room]
        flat = np.concatenate(room + [np.zeros(1, np.int64)]).astype(np.uint16)
        filled = np.zeros(flat.size, np.uint16)
        n_taken = np.zeros(max(n, 1), np.uint32)
        cap = 1 << 12  # resized from the total of an MM_E_CAP refusal
        while True:
            mem = np.empty(cap, np.uint64)
            total = C.c_uint32(0)
            rc = self.lib.mm_backfill_party(self.h, n, _p(req), _p(flat), _p(filled), _p(n_taken), _p(mem), cap,
                                            C.byref(total))
            if rc == abi.MM_E_CAP and total.value > cap:
                cap = total.value
                continue
            self._check(rc, "mm_backfill_party")
            break
        out_filled, out_members, e, m = [], [], 0, 0
        for r in room:
            f = filled[e:e + r.size].astype(np.int64)
            out_filled.append(f.tolist())
            out_members.append([mem[m + a:m + b].copy() for a, b in zip(np.cumsum(f) - f, np.cumsum(f))])
            e += r.size
            m += int(f.sum())
        return out_filled, out_members

    # -- widening search (mm_widen) --------------------------------------------------------------------------------
    WIDEN_RULE_DTYPE = np.dtype([("min_wait", "<u4"), ("step", "<u4"), ("w0", "<i4"), ("inc", "<i4"),
                                 ("w_max", "<i4"), ("reserved", "<u4")])

    def widen_rules(self, rules=None):
        """A rule array for widen(): every queue off, then rules[(mode, group)] = (min_wait, w0, step, inc, w_max)."""
        out = np.zeros(self.cfg.n_modes * self.cfg.n_groups, self.WIDEN_RULE_DTYPE)
        out["min_wait"] = abi.MM_WIDEN_OFF
        out["step"] = 1
        for (m, g), (min_wait, w0, step, inc, w_max) in (rules or {}).items():
            out[m * self.cfg.n_groups + g] = (min_wait, step, w0, inc, w_max, 0)
        return out

    def widen(self, now, rules, lobby_cap=1 << 10, member_cap=1 << 12):
        """Form lobbies around the live queued players who have waited at least their queue's min_wait, each in a
        rating window that grows with its wait (mm_widen).  rules: WIDEN_RULE_DTYPE[n_modes * n_groups], or the dict
        widen_rules() takes.  -> (lobbies[LOBBY_DTYPE], member_ids u64, WidenStats).  An MM_E_CAP refusal is retried
        once with its counts."""
        if isinstance(rules, dict):
            rules = self.widen_rules(rules)
        rules = np.ascontiguousarray(rules, self.WIDEN_RULE_DTYPE)
        for attempt in range(2):
            lob = np.empty(max(lobby_cap, 1), LOBBY_DTYPE)
            mem = np.empty(max(member_cap, 1), np.uint64)
            st = abi.WidenStats()
            rc = self.lib.mm_widen(self.h, int(now), _p(rules), _p(lob), lobby_cap, _p(mem), member_cap, C.byref(st))
            if rc == abi.MM_E_CAP and attempt == 0:
                lobby_cap, member_cap = max(lobby_cap, st.n_lobbies), max(member_cap, st.n_matched)
                continue
            self._check(rc, "mm_widen")
            return lob[:st.n_lobbies], mem[:st.n_matched], st

    # -- parties (mm_enqueue_party / mm_party_match / mm_party_read) ---------------------------------------------
    def enqueue_party(self, sizes, ids, rating, mode, enq_ts=None):
        """Queue parties: party j's members are the next sizes[j] entries of ids / rating.  -> codes u8[n_parties]:
        1 queued, 0 a member already queued (or in an earlier party of the batch), 2 invalid, 3 the table is full."""
        sizes = np.ascontiguousarray(sizes, np.uint8)
        ids = np.ascontiguousarray(ids, np.uint64)
        rating = np.ascontiguousarray(rating, np.int32)
        mode = np.ascontiguousarray(mode, np.uint8)
        n = len(sizes)
        assert len(mode) == n and len(ids) == len(rating) == int(sizes.sum(dtype=np.int64))
        if enq_ts is not None:
            enq_ts = np.ascontiguousarray(enq_ts, np.uint32)
            assert len(enq_ts) == n
        acc = np.empty(max(n, 1), np.uint8)
        self._check(self.lib.mm_enqueue_party(self.h, n, _p(sizes), _p(ids), _p(rating), _p(mode), _p(enq_ts), _p(acc)),
                    "mm_enqueue_party")
        return acc[:n]

    def party_match(self, now, rules, lobby_cap=1 << 10, member_cap=1 << 12):
        """Form lobbies around the queued parties that waited at least their queue's min_wait (mm_party_match).
        rules as widen() takes them.  -> (lobbies[LOBBY_DTYPE], member_ids u64, PartyStats).  An MM_E_CAP refusal is
        retried once with its counts."""
        if isinstance(rules, dict):
            rules = self.widen_rules(rules)
        rules = np.ascontiguousarray(rules, self.WIDEN_RULE_DTYPE)
        for attempt in range(2):
            lob = np.empty(max(lobby_cap, 1), LOBBY_DTYPE)
            mem = np.empty(max(member_cap, 1), np.uint64)
            st = abi.PartyStats()
            rc = self.lib.mm_party_match(self.h, int(now), _p(rules), _p(lob), lobby_cap, _p(mem), member_cap,
                                         C.byref(st))
            if rc == abi.MM_E_CAP and attempt == 0:
                lobby_cap, member_cap = max(lobby_cap, st.n_lobbies), max(member_cap, st.n_matched)
                continue
            self._check(rc, "mm_party_match")
            return lob[:st.n_lobbies], mem[:st.n_matched], st

    def party_read(self):
        """The queued parties in age order (mm_party_read) -> dict of per-party columns size, seq, enq_ts, mode, group,
        rating (R) and `members`, a list of (ids u64, ratings i32) per party."""
        pc, mc = 1 << 10, 1 << 12
        while True:
            cols = dict(size=np.empty(pc, np.uint8), seq=np.empty(pc, np.uint32), enq_ts=np.empty(pc, np.uint32),
                        mode=np.empty(pc, np.uint8), group=np.empty(pc, np.uint8), rating=np.empty(pc, np.int32))
            mid, mrt = np.empty(mc, np.uint64), np.empty(mc, np.int32)
            np_, nm = C.c_uint32(0), C.c_uint32(0)
            rc = self.lib.mm_party_read(self.h, pc, mc, *(_p(cols[k]) for k in ("size", "seq", "enq_ts", "mode", "group",
                                                                                 "rating")),
                                        _p(mid), _p(mrt), C.byref(np_), C.byref(nm))
            if rc == abi.MM_E_CAP and (np_.value > pc or nm.value > mc):
                pc, mc = max(pc, np_.value), max(mc, nm.value)
                continue
            self._check(rc, "mm_party_read")
            out = {k: v[:np_.value] for k, v in cols.items()}
            cut = np.cumsum(out["size"].astype(np.int64))[:-1]
            out["members"] = list(zip(np.split(mid[:nm.value], cut), np.split(mrt[:nm.value], cut))) if np_.value else []
            return out

    def party_queue_stats(self, now=0):
        """The queued parties per (mode, group) queue (mm_party_queue_stats) -> PARTY_QUEUE_STAT_DTYPE[n_modes * n_groups],
        record mode * n_groups + group: parties, members, the longest wait at `now`, the wait histogram (one count per
        party, queue_stats' buckets) and the size histogram."""
        cap = self.cfg.n_modes * self.cfg.n_groups
        out = np.zeros(cap, PARTY_QUEUE_STAT_DTYPE)
        n = C.c_uint32(0)
        self._check(self.lib.mm_party_queue_stats(self.h, int(now) & 0xFFFFFFFFFFFFFFFF, _p(out), cap, C.byref(n)),
                    "mm_party_queue_stats")
        return out[:n.value]

    def party_locate(self, ids, now, rules):
        """Search status of each id as a party member (mm_party_locate) -> PARTY_MEMBER_STATUS_DTYPE[len(ids)]: state
        (mm_locate's; 3 = queued in a party), its party's queue, size, its index in the party, the party's rating,
        stamp, seq and wait at `now`, anchor / window under `rules`, the parties of its queue ahead of it and the
        queue's parties, and the lobby ordinal / member index the next party_match(now, rules) gives it (lobby =
        abi.MM_LOCATE_STAYS: its party stays queued).  rules as party_match takes them."""
        if isinstance(rules, dict):
            rules = self.widen_rules(rules)
        rules = np.ascontiguousarray(rules, self.WIDEN_RULE_DTYPE)
        ids = np.ascontiguousarray(ids, np.uint64)
        out = np.zeros(len(ids), PARTY_MEMBER_STATUS_DTYPE)
        self._check(self.lib.mm_party_locate(self.h, int(now) & 0xFFFFFFFFFFFFFFFF, _p(rules), len(ids), _p(ids),
                                             _p(out)), "mm_party_locate")
        return out

    def export_parties(self, mask=None):
        """Release the queued parties of the selected (mode, group) queues into a party image (mm_export_parties) ->
        uint8 array (read_party_image).  mask: bool per queue as export_queues takes it, or None for every queue.  The
        exported parties leave this engine as if remove() had been called with one member of each."""
        sel = None
        if mask is not None:
            sel = np.ascontiguousarray(np.asarray(mask, bool).reshape(-1), np.uint8)
            assert len(sel) == self.cfg.n_modes * self.cfg.n_groups
        n = C.c_uint64(0)
        self._check(self.lib.mm_export_parties(self.h, _p(sel), None, 0, C.byref(n)), "mm_export_parties")
        for attempt in range(2):  # the size query and the export are two calls: a party enqueued between them is retried
            buf = np.empty(n.value, np.uint8)
            rc = self.lib.mm_export_parties(self.h, _p(sel), _p(buf), n.value, C.byref(n))
            if rc == abi.MM_E_CAP and attempt == 0:
                continue
            self._check(rc, "mm_export_parties")
            return buf[:n.value]

    def merge_parties(self, buf, keep_seq=False):
        """Merge a party image (export_parties) into this engine (mm_merge_parties): one enqueue_party batch of its
        columns, all or nothing on room.  keep_seq: every party keeps its number (after import_state / import_regroup
        of the image taken at the same stop).  -> codes u8[n_parties] as enqueue_party gives them (never 3)."""
        buf = np.ascontiguousarray(np.frombuffer(buf, np.uint8) if isinstance(buf, (bytes, bytearray, memoryview))
                                   else buf, np.uint8)
        hs = C.sizeof(abi.ImageHeader)
        n = abi.ImageHeader.from_buffer_copy(buf[:hs].tobytes()).n_parts if len(buf) >= hs else 0
        code = np.zeros(max(min(n, len(buf)), 1), np.uint8)  # a party takes more than a byte: a corrupt count is capped
        k = C.c_uint32(0)
        self._check(self.lib.mm_merge_parties(self.h, _p(buf), len(buf), abi.MM_PARTY_KEEP_SEQ if keep_seq else 0,
                                              _p(code), C.byref(k)), "mm_merge_parties")
        return code[:n]

    def requeue_party(self, sizes, ids, rating, mode, enq_ts, seq):
        """Put the parties of a lobby that did not start back into the party table as parties, at their age position
        (mm_requeue_party).  Party j's members are the next sizes[j] entries of ids / rating; mode, enq_ts (may be
        None) and seq are per party, what it had when it was queued.  The parties may come in any order: they are
        sorted by age here.  -> codes u8[n] in the caller's order: 1 requeued, 0 a member still queued, 4 a member not
        in the active set (the party was not requeued)."""
        sizes = np.ascontiguousarray(sizes, np.uint8)
        ids = np.ascontiguousarray(ids, np.uint64)
        rating = np.ascontiguousarray(rating, np.int32)
        seq = np.ascontiguousarray(seq, np.uint32)
        n = len(sizes)
        assert len(mode) == n and len(seq) == n and len(ids) == len(rating) == int(sizes.sum(dtype=np.int64))
        order = np.argsort((seq - np.uint32(self.seq_next())).astype(np.uint32), kind="stable")  # a tie is refused
        start = np.concatenate([[0], np.cumsum(sizes.astype(np.int64))])
        so = sizes[order].astype(np.int64)  # the members of party order[k] follow those of order[k - 1]
        take = np.repeat(start[order], so) + np.arange(len(ids)) - np.repeat(np.cumsum(so) - so, so)
        cols = [np.ascontiguousarray(a, dt) for a, dt in ((sizes[order], np.uint8), (ids[take], np.uint64),
                                                          (rating[take], np.int32), (np.asarray(mode)[order], np.uint8),
                                                          (seq[order], np.uint32))]
        ts = None if enq_ts is None else np.ascontiguousarray(np.asarray(enq_ts)[order], np.uint32)
        codes = np.empty(max(n, 1), np.uint8)
        k = C.c_uint32(0)
        self._check(self.lib.mm_requeue_party(self.h, n, _p(cols[0]), _p(cols[1]), _p(cols[2]), _p(cols[3]), _p(ts),
                                              _p(cols[4]), _p(codes), C.byref(k)), "mm_requeue_party")
        out = np.empty(n, np.uint8)
        out[order] = codes[:n]
        return out

    def in_queue(self, ids):
        ids = np.ascontiguousarray(ids, np.uint64)
        out = np.empty(len(ids), np.uint8)
        self._check(self.lib.mm_in_queue(self.h, len(ids), _p(ids), _p(out)), "mm_in_queue")
        return out.astype(bool)

    def locate(self, ids, now=0):
        """Search status of each id (mm_locate) -> PLAYER_STATUS_DTYPE[len(ids)]: state (0 gone, 1 queued, 2 matched or
        taken and not yet removed), its queue, rating, stamp, seq, wait at `now`, players ahead of it in its queue's feed
        order and the queue's depth, and the lobby ordinal / member index the next tick gives it (lobby =
        abi.MM_LOCATE_STAYS: it stays queued)."""
        ids = np.ascontiguousarray(ids, np.uint64)
        out = np.zeros(len(ids), PLAYER_STATUS_DTYPE)
        self._check(self.lib.mm_locate(self.h, int(now) & 0xFFFFFFFFFFFFFFFF, len(ids), _p(ids), _p(out)), "mm_locate")
        return out

    def pool_size(self):
        v = C.c_uint32(0)
        self._check(self.lib.mm_pool_size(self.h, C.byref(v)), "mm_pool_size")
        return v.value

    def active_size(self):
        v = C.c_uint32(0)
        self._check(self.lib.mm_active_size(self.h, C.byref(v)), "mm_active_size")
        return v.value

    def pool_read(self):
        n = self.pool_size()
        ids = np.empty(n, np.uint64)
        rating = np.empty(n, np.int32)
        mode = np.empty(n, np.uint8)
        tsz = np.empty(n, np.uint8)
        ts = np.empty(n, np.uint32)
        k = C.c_uint32(0)
        self._check(self.lib.mm_pool_read(self.h, n, _p(ids), _p(rating), _p(mode), _p(tsz), _p(ts), C.byref(k)),
                    "mm_pool_read")
        k = k.value
        return dict(id=ids[:k], rating=rating[:k], mode=mode[:k], team_size=tsz[:k], enq_ts=ts[:k])

    # -- the tick ------------------------------------------------------------------
    def tick(self, now=0, lobby_cap=None, member_cap=None, want_emit_seq=True):
        """Host-buffer tick -> (lobbies[LOBBY_DTYPE], member_ids u64, emit_seq u32|None, TickStats)."""
        n = self.pool_size()
        if member_cap is None:
            member_cap = max(n, 1)
        if lobby_cap is None:
            lobby_cap = max(n // 2, 1)  # L >= 2 for every sensible mode; resized on MM_E_CAP
        while True:
            lob = np.empty(lobby_cap, LOBBY_DTYPE)
            mem = np.empty(member_cap, np.uint64)
            seq = np.empty(lobby_cap, np.uint32) if want_emit_seq else None
            st = abi.TickStats()
            rc = self.lib.mm_tick(self.h, now, _p(lob), lobby_cap, _p(mem), member_cap, _p(seq), C.byref(st))
            if rc == abi.MM_E_CAP and lobby_cap < max(n, 1):
                lobby_cap = max(n, 1)
                continue
            self._check(rc, "mm_tick")
            break
        self.results_wait()  # no-op unless the "async_results" option is on
        nl, nm = st.n_lobbies, st.n_matched
        return lob[:nl], mem[:nm], (seq[:nl] if seq is not None else None), st

    def results_wait(self):
        """Block until the host buffers of the last mm_tick are filled ("async_results" mode)."""
        self._check(self.lib.mm_results_wait(self.h), "mm_results_wait")

    def tick_device(self, now=0):
        st = abi.TickStats()
        self._check(self.lib.mm_tick_device(self.h, now, C.byref(st)), "mm_tick_device")
        return st

    def results_device(self):
        a, b = C.c_void_p(), C.c_void_p()
        self._check(self.lib.mm_results_device(self.h, C.byref(a), C.byref(b)), "mm_results_device")
        return a.value, b.value

    def queue_stats(self, now=0):
        """Per-(mode, group) queue status (mm_queue_stats) -> QUEUE_STAT_DTYPE[n_modes * n_groups], record
        mode * n_groups + group: the pool at `now` and the players the last tick matched at that tick's `now`."""
        cap = self.cfg.n_modes * self.cfg.n_groups
        out = np.zeros(cap, QUEUE_STAT_DTYPE)
        n = C.c_uint32(0)
        self._check(self.lib.mm_queue_stats(self.h, int(now) & 0xFFFFFFFFFFFFFFFF, _p(out), cap, C.byref(n)),
                    "mm_queue_stats")
        return out[:n.value]

    def match_quality(self, want_lobbies=False):
        """Rating spread and team imbalance of the last tick's lobbies (mm_match_quality) -> (QUALITY_DTYPE[n_modes *
        n_groups] in queue_stats() record order, LOBBY_QUALITY_DTYPE[n_lobbies] in the tick's lobby order, or None
        without want_lobbies).  Both are empty when the report is void (no tick yet, a failed tick, a pool loaded
        since)."""
        cap = self.cfg.n_modes * self.cfg.n_groups
        lobby_cap = 1 << 12 if want_lobbies else 0  # resized from the count of an MM_E_CAP refusal
        n, nl = C.c_uint32(0), C.c_uint32(0)
        while True:
            out = np.zeros(cap, QUALITY_DTYPE)
            lob = np.zeros(lobby_cap, LOBBY_QUALITY_DTYPE) if want_lobbies else None
            rc = self.lib.mm_match_quality(self.h, _p(out), cap, C.byref(n), _p(lob), lobby_cap, C.byref(nl))
            if rc == abi.MM_E_CAP and (n.value > cap or (want_lobbies and nl.value > lobby_cap)):
                cap, lobby_cap = max(cap, n.value), max(lobby_cap, nl.value)
                continue
            self._check(rc, "mm_match_quality")
            return out[:n.value], (lob[:nl.value] if want_lobbies else None)

    def offtick_report(self, source, want_lobbies=False):
        """Waits and rating quality of the lobbies the last call of `source` formed (mm_offtick_report; source
        abi.MM_OFFTICK_PARTY_MATCH or abi.MM_OFFTICK_WIDEN) -> (WAITS_DTYPE[n_modes * n_groups], QUALITY_DTYPE[n_modes *
        n_groups], both in queue_stats() record order, LOBBY_QUALITY_DTYPE[n_lobbies] in that call's lobby order, or None
        without want_lobbies).  All are empty when the report is void (no such call yet, or its last one failed)."""
        cap = self.cfg.n_modes * self.cfg.n_groups
        lobby_cap = 1 << 12 if want_lobbies else 0  # resized from the count of an MM_E_CAP refusal
        n, nl = C.c_uint32(0), C.c_uint32(0)
        while True:
            waits = np.zeros(cap, WAITS_DTYPE)
            quality = np.zeros(cap, QUALITY_DTYPE)
            lob = np.zeros(lobby_cap, LOBBY_QUALITY_DTYPE) if want_lobbies else None
            rc = self.lib.mm_offtick_report(self.h, source, _p(waits), _p(quality), cap, C.byref(n), _p(lob), lobby_cap,
                                            C.byref(nl))
            if rc == abi.MM_E_CAP and (n.value > cap or (want_lobbies and nl.value > lobby_cap)):
                cap, lobby_cap = max(cap, n.value), max(lobby_cap, nl.value)
                continue
            self._check(rc, "mm_offtick_report")
            return waits[:n.value], quality[:n.value], (lob[:nl.value] if want_lobbies else None)

    # -- lobby budget ----------------------------------------------------------------
    def set_lobby_budget(self, per_queue=None, per_mode=None):
        """Lobbies every (mode, group) queue / every mode may emit per tick, from the next tick until set again
        (mm_set_lobby_budget).  per_queue: n_modes * n_groups values in queue_stats() record order (or
        [n_modes][n_groups]); per_mode: n_modes values; None, or abi.MM_BUDGET_UNLIMITED in an entry = no limit."""
        q, m = self._budget_arrays(per_queue, per_mode)
        self._check(self.lib.mm_set_lobby_budget(self.h, _p(q), _p(m)), "mm_set_lobby_budget")

    def _budget_arrays(self, per_queue, per_mode):
        def arr(a, n):
            if a is None:
                return None
            a = np.ascontiguousarray(np.asarray(a, np.int64).reshape(-1).clip(0, abi.MM_BUDGET_UNLIMITED), np.uint32)
            assert len(a) == n
            return a
        return arr(per_queue, self.cfg.n_modes * self.cfg.n_groups), arr(per_mode, self.cfg.n_modes)

    def lobby_budget_report(self):
        """-> (candidates u32[n_modes * n_groups], emitted u32[...]) of the last completed tick: the lobbies every queue
        had, budgets ignored, and the lobbies it emitted (mm_lobby_budget_report)."""
        cap = self.cfg.n_modes * self.cfg.n_groups
        cand, emitted = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
        n = C.c_uint32(0)
        self._check(self.lib.mm_lobby_budget_report(self.h, _p(cand), _p(emitted), cap, C.byref(n)),
                    "mm_lobby_budget_report")
        return cand[:n.value], emitted[:n.value]

    def set_offtick_budget(self, source, per_queue=None, per_mode=None):
        """Lobbies every (mode, group) queue / every mode may emit per call of `source` (abi.MM_OFFTICK_PARTY_MATCH:
        party_match, abi.MM_OFFTICK_WIDEN: widen), from the next such call until set again (mm_set_offtick_budget).
        Arrays as in set_lobby_budget; each source's budget is separate from the other's and from the tick's."""
        q, m = self._budget_arrays(per_queue, per_mode)
        self._check(self.lib.mm_set_offtick_budget(self.h, source, _p(q), _p(m)), "mm_set_offtick_budget")

    def offtick_budget_report(self, source):
        """-> (candidates u32[n_modes * n_groups], emitted u32[...]) of the last call of `source` that returned MM_OK
        or was an MM_E_CAP dry run: the lobbies every queue had, budgets ignored, and the lobbies it emitted (or would
        have) (mm_offtick_budget_report).  All zeros before such a call."""
        cap = self.cfg.n_modes * self.cfg.n_groups
        cand, emitted = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
        n = C.c_uint32(0)
        self._check(self.lib.mm_offtick_budget_report(self.h, source, _p(cand), _p(emitted), cap, C.byref(n)),
                    "mm_offtick_budget_report")
        return cand[:n.value], emitted[:n.value]

    def lobby_candidates(self):
        """-> u32[n_modes * n_groups]: the lobbies a tick without a budget would emit from every queue of the pool as it
        is now; nothing changes (mm_lobby_candidates)."""
        cap = self.cfg.n_modes * self.cfg.n_groups
        cand = np.zeros(cap, np.uint32)
        n = C.c_uint32(0)
        self._check(self.lib.mm_lobby_candidates(self.h, _p(cand), cap, C.byref(n)), "mm_lobby_candidates")
        return cand[:n.value]

    def expire(self, now, max_wait, want_seq=True):
        """Search timeout (mm_expire): every queued player whose wait at `now` (as queue_stats counts it) is >=
        max_wait leaves the pool and the active set, like remove(). -> (ids u64, enqueue seq u32 | None), unordered."""
        return self._expire(self.lib.mm_expire, np.uint64, now, max_wait, want_seq, "mm_expire")

    def expire_packed(self, now, max_wait, want_seq=True):
        """expire() on an MM_F_DENSE_IDS engine, ids as u32 handles (mm_expire_packed)."""
        return self._expire(self.lib.mm_expire_packed, np.uint32, now, max_wait, want_seq, "mm_expire_packed")

    def _expire(self, fn, dtype, now, max_wait, want_seq, what):
        cap = self.pool_size()  # every resident player fits: the engine makes a single pass
        max_wait = max(0, min(int(max_wait), 0xFFFFFFFF))
        for attempt in range(2):  # queued party members may not fit: a refusal counts them and changes nothing
            ids = np.empty(max(cap, 1), dtype)
            seq = np.empty(max(cap, 1), np.uint32) if want_seq else None
            n = C.c_uint32(0)
            rc = fn(self.h, int(now) & 0xFFFFFFFFFFFFFFFF, max_wait, _p(ids), _p(seq), cap, C.byref(n))
            if rc == abi.MM_E_CAP and attempt == 0:
                cap = n.value
                continue
            self._check(rc, what)
            return ids[:n.value], (seq[:n.value] if seq is not None else None)

    def export_state(self):
        """Host image of the queue state (mm_export) -> uint8 array; the engine is not changed.  Layout:
        include/mm_engine.h, or read_image()."""
        # one call: a buffer of the layout's size at its upper bound (every slot in use live, every active id outside
        # the pool, the most partitions, 8-byte ids) always holds the image
        bound = abi.image_offsets(abi.MM_MAX_GROUPS * abi.MM_MAX_MODES, self.pool_size(), self.active_size(), 8)[-1]
        buf = np.empty(bound, np.uint8)
        n = C.c_uint64(0)
        self._check(self.lib.mm_export(self.h, _p(buf), bound, C.byref(n)), "mm_export")
        return buf[:n.value]

    def import_state(self, buf):
        """Load an image written by export_state() into this engine, which must be fresh (mm_import)."""
        buf = np.ascontiguousarray(np.frombuffer(buf, np.uint8) if isinstance(buf, (bytes, bytearray, memoryview))
                                   else buf, np.uint8)
        self._check(self.lib.mm_import(self.h, _p(buf), len(buf)), "mm_import")

    def import_regroup(self, buf):
        """Load an image written by export_state() under ANOTHER config (rating groups, default group, modes, order,
        MM_F_WIDE_PARTITIONS) into this fresh engine (mm_import_regroup): every player keeps its id, rating, mode,
        stamp and sequence number and goes to the queue its rating and mode map to here.  -> image indices (u32,
        ascending) of the players this config has no queue for: they are not queued, and the caller answers them."""
        buf = np.ascontiguousarray(np.frombuffer(buf, np.uint8) if isinstance(buf, (bytes, bytearray, memoryview))
                                   else buf, np.uint8)
        hs = C.sizeof(abi.ImageHeader)
        n = abi.ImageHeader.from_buffer_copy(buf[:hs].tobytes()).n_players if len(buf) >= hs else 0
        n = min(n, len(buf))  # a player takes more than a byte: a corrupt count must not size the reject list
        rej = np.empty(max(n, 1), np.uint32)
        k = C.c_uint32(0)
        self._check(self.lib.mm_import_regroup(self.h, _p(buf), len(buf), n, _p(rej), C.byref(k)), "mm_import_regroup")
        return rej[:k.value]

    def import_regroup_many(self, images, keep=None, active_image=None):
        """Load several export_state() images written under ONE config (the old ranks of a sharded deployment) into
        this fresh engine, re-filed under its config (mm_import_regroup_many).  keep: bool per (mode, group) queue of
        this config ([n_modes, n_groups] or flat in mm_queue_stats order; None = all): players of an unselected queue
        are skipped.  active_image: the image whose active section this engine takes (None = none).  Inside a queue the
        images interleave by running-max stamp (ties to the lower image); with more than one image the kept players
        are renumbered 0 .. n_kept-1 (include/mm_engine.h).  -> (rejected, n_elsewhere): rejected = int64 [n, 2]
        (image, index) pairs, ascending, of the players this config has no queue for; n_elsewhere = players skipped."""
        bufs = [np.ascontiguousarray(np.frombuffer(b, np.uint8) if isinstance(b, (bytes, bytearray, memoryview))
                                     else b, np.uint8) for b in images]
        K = len(bufs)
        ptrs = (C.c_void_p * max(K, 1))(*[b.ctypes.data for b in bufs])
        lens = (C.c_uint64 * max(K, 1))(*[len(b) for b in bufs])
        hs = C.sizeof(abi.ImageHeader)
        n = sum(min(abi.ImageHeader.from_buffer_copy(b[:hs].tobytes()).n_players, len(b)) if len(b) >= hs else 0
                for b in bufs)  # a player takes more than a byte: a corrupt count must not size the reject list
        n = min(n, 0xFFFFFFFF)
        sel = None
        if keep is not None:
            sel = np.ascontiguousarray(np.asarray(keep, bool).reshape(-1), np.uint8)
            if len(sel) != self.cfg.n_modes * self.cfg.n_groups:
                raise ValueError("keep needs n_modes * n_groups entries")
        rimg, ridx = np.empty(max(n, 1), np.uint32), np.empty(max(n, 1), np.uint32)
        k, e = C.c_uint32(0), C.c_uint32(0)
        self._check(self.lib.mm_import_regroup_many(self.h, K, ptrs, lens, _p(sel),
                                                    0xFFFFFFFF if active_image is None else int(active_image), n,
                                                    _p(rimg), _p(ridx), C.byref(k), C.byref(e)),
                    "mm_import_regroup_many")
        return np.stack([rimg[:k.value], ridx[:k.value]], 1).astype(np.int64), int(e.value)

    def import_regroup_many_parties(self, images, party_images, keep=None, active_image=None):
        """import_regroup_many() with the queued parties: party_images[k] is what export_parties() gave on the rank
        that wrote images[k], taken just before it (None or empty = no parties).  Parties are classified under this
        config as solos are, and numbered with the solos in one order (mm_import_regroup_many_parties).  -> (rejected,
        n_elsewhere, party_rejected, party_elsewhere): party_rejected = int64 [n, 2] (image, party index) pairs,
        ascending, of the parties this config has no queue for; party_elsewhere = parties skipped."""
        def arr(b):
            return np.ascontiguousarray(np.frombuffer(b, np.uint8) if isinstance(b, (bytes, bytearray, memoryview))
                                        else b, np.uint8)
        bufs = [arr(b) for b in images]
        pbufs = [None if b is None else arr(b) for b in party_images]
        K = len(bufs)
        if len(pbufs) != K:
            raise ValueError("one party image (or None) per image")
        ptrs = (C.c_void_p * max(K, 1))(*[b.ctypes.data for b in bufs])
        lens = (C.c_uint64 * max(K, 1))(*[len(b) for b in bufs])
        pptrs = (C.c_void_p * max(K, 1))(*[b.ctypes.data if b is not None and len(b) else None for b in pbufs])
        plens = (C.c_uint64 * max(K, 1))(*[len(b) if b is not None else 0 for b in pbufs])
        hs = C.sizeof(abi.ImageHeader)
        n = sum(min(abi.ImageHeader.from_buffer_copy(b[:hs].tobytes()).n_players, len(b)) if len(b) >= hs else 0
                for b in bufs)  # a player takes more than a byte: a corrupt count must not size the reject list
        n = min(n, 0xFFFFFFFF)
        np_ = sum(min(abi.ImageHeader.from_buffer_copy(b[:hs].tobytes()).n_parts, len(b))
                  for b in pbufs if b is not None and len(b) >= hs)
        np_ = min(np_, 0xFFFFFFFF)
        sel = None
        if keep is not None:
            sel = np.ascontiguousarray(np.asarray(keep, bool).reshape(-1), np.uint8)
            if len(sel) != self.cfg.n_modes * self.cfg.n_groups:
                raise ValueError("keep needs n_modes * n_groups entries")
        rimg, ridx = np.empty(max(n, 1), np.uint32), np.empty(max(n, 1), np.uint32)
        pimg, pidx = np.empty(max(np_, 1), np.uint32), np.empty(max(np_, 1), np.uint32)
        rp = abi.RecutParties()
        rp.bufs = C.cast(pptrs, C.c_void_p)
        rp.n_bytes = C.cast(plens, C.c_void_p)
        rp.cap = np_
        rp.rej_image, rp.rej_index = pimg.ctypes.data, pidx.ctypes.data
        k, e = C.c_uint32(0), C.c_uint32(0)
        self._check(self.lib.mm_import_regroup_many_parties(self.h, K, ptrs, lens, _p(sel),
                                                            0xFFFFFFFF if active_image is None else int(active_image),
                                                            n, _p(rimg), _p(ridx), C.byref(k), C.byref(e),
                                                            C.byref(rp)),
                    "mm_import_regroup_many_parties")
        return (np.stack([rimg[:k.value], ridx[:k.value]], 1).astype(np.int64), int(e.value),
                np.stack([pimg[:rp.n_rejected], pidx[:rp.n_rejected]], 1).astype(np.int64), int(rp.n_elsewhere))

    def export_queues(self, mask):
        """Release whole (mode, group) queues into a queue image (mm_export_queues) -> uint8 array.  mask: bool per
        queue in queue_stats() record order (mode * n_groups + group), or [n_modes][n_groups].  The exported players
        leave this engine as if remove() had been called with their ids; matched-not-removed ids stay here."""
        mask = np.ascontiguousarray(np.asarray(mask, bool).reshape(-1), np.uint8)
        assert len(mask) == self.cfg.n_modes * self.cfg.n_groups
        bound = abi.image_offsets(abi.MM_MAX_GROUPS * abi.MM_MAX_MODES, self.pool_size(), 0, 8)[-1]
        buf = np.empty(bound, np.uint8)
        n = C.c_uint64(0)
        self._check(self.lib.mm_export_queues(self.h, _p(mask), _p(buf), bound, C.byref(n)), "mm_export_queues")
        return buf[:n.value]

    def merge_queues(self, buf):
        """Load a queue image (export_queues) into this running engine (mm_merge) -> image indices (u32, ascending)
        of the players that were not queued: ids already active here, and later copies of an id."""
        buf = np.ascontiguousarray(np.frombuffer(buf, np.uint8) if isinstance(buf, (bytes, bytearray, memoryview))
                                   else buf, np.uint8)
        hs = C.sizeof(abi.ImageHeader)
        n = abi.ImageHeader.from_buffer_copy(buf[:hs].tobytes()).n_players if len(buf) >= hs else 0
        n = min(n, len(buf))  # a player takes more than a byte: a corrupt count must not size the reject list
        rej = np.empty(max(n, 1), np.uint32)
        k = C.c_uint32(0)
        self._check(self.lib.mm_merge(self.h, _p(buf), len(buf), n, _p(rej), C.byref(k)), "mm_merge")
        return rej[:k.value]

    def snapshot(self):
        self._check(self.lib.mm_snapshot(self.h), "mm_snapshot")

    def restore(self):
        self._check(self.lib.mm_restore(self.h), "mm_restore")

    def set_stream(self, cuda_stream):
        self._check(self.lib.mm_set_stream(self.h, C.c_void_p(cuda_stream)), "mm_set_stream")

    party_capacity = 0  # the option "party_capacity" as last set

    def set_option(self, name, value):
        self._check(self.lib.mm_set_option(self.h, name.encode(), int(value)), "mm_set_option")
        if name == "party_capacity":
            self.party_capacity = int(value)

    def status(self):
        """Search.Worker.status/0 analogue (search/worker.ex:115-117,326-334): queue depth."""
        return {"message_count": self.pool_size(), "active_count": self.active_size()}
