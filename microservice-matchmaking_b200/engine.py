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

# mm_queue_stat (include/mm_engine.h) as a numpy record
QUEUE_STAT_DTYPE = np.dtype([
    ("mode", "u1"), ("group", "u1"), ("reserved", "<u2"),
    ("n_waiting", "<u4"), ("n_removed", "<u4"), ("max_wait", "<u4"), ("wait_hist", "<u4", (abi.MM_WAIT_BUCKETS,)),
    ("n_lobbies", "<u4"), ("n_matched", "<u4"), ("max_match_wait", "<u4"),
    ("match_wait_hist", "<u4", (abi.MM_WAIT_BUCKETS,)),
])


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

    def in_queue(self, ids):
        ids = np.ascontiguousarray(ids, np.uint64)
        out = np.empty(len(ids), np.uint8)
        self._check(self.lib.mm_in_queue(self.h, len(ids), _p(ids), _p(out)), "mm_in_queue")
        return out.astype(bool)

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

    def snapshot(self):
        self._check(self.lib.mm_snapshot(self.h), "mm_snapshot")

    def restore(self):
        self._check(self.lib.mm_restore(self.h), "mm_restore")

    def set_stream(self, cuda_stream):
        self._check(self.lib.mm_set_stream(self.h, C.c_void_p(cuda_stream)), "mm_set_stream")

    def set_option(self, name, value):
        self._check(self.lib.mm_set_option(self.h, name.encode(), int(value)), "mm_set_option")

    def status(self):
        """Search.Worker.status/0 analogue (search/worker.ex:115-117,326-334): queue depth."""
        return {"message_count": self.pool_size(), "active_count": self.active_size()}
