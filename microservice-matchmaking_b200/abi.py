"""ctypes mirror of include/mm_engine.h (the C ABI of libmm_engine.so).

Only PODs and prototypes live here; no compute.  The same structs are reused by
the test-side oracle wrapper (oracle/oracle.py), which shares `mm_config`.
"""
import ctypes as C

MM_ABI_VERSION = 2
MM_MAX_GROUPS = 64
MM_MAX_MODES = 8
MM_MODE_DEAD = 0xFF

MM_OK = 0
MM_E_ARG = -1
MM_E_CUDA = -2
MM_E_CAP = -3
MM_E_NCCL = -4
MM_E_STATE = -5

MM_ORDER_ARRIVAL = 0
MM_ORDER_RATING = 1

MM_F_NO_DEDUPE = 1
MM_F_DENSE_IDS = 2
MM_F_WIDE_PARTITIONS = 4


class ModeDesc(C.Structure):
    _fields_ = [("teams", C.c_uint16), ("team_size", C.c_uint16)]


class Config(C.Structure):
    _fields_ = [
        ("abi_version", C.c_uint32),
        ("n_groups", C.c_uint32),
        ("group_lo", C.c_int32 * MM_MAX_GROUPS),
        ("group_hi", C.c_int32 * MM_MAX_GROUPS),
        ("default_group", C.c_int32),
        ("n_modes", C.c_uint32),
        ("modes", ModeDesc * MM_MAX_MODES),
        ("order_mode", C.c_uint32),
        ("capacity", C.c_uint32),
        ("active_capacity", C.c_uint32),
        ("device", C.c_int32),
        ("flags", C.c_uint32),
    ]


class LobbyHdr(C.Structure):
    _fields_ = [
        ("first_member", C.c_uint32),
        ("n_members", C.c_uint16),
        ("mode", C.c_uint8),
        ("group", C.c_uint8),
    ]


class TickStats(C.Structure):
    _fields_ = [
        ("pool_before", C.c_uint32),
        ("n_lobbies", C.c_uint32),
        ("n_matched", C.c_uint32),
        ("n_residual", C.c_uint32),
        ("n_dead", C.c_uint32),
        ("n_launches", C.c_uint32),
        ("device_us", C.c_float),
        ("place_us", C.c_float),
        ("hist_us", C.c_float),
        ("scan_us", C.c_float),
        ("epilogue_us", C.c_float),
        ("reserved", C.c_uint32),
    ]


MM_WAIT_BUCKETS = 120


class QueueStat(C.Structure):
    """One (mode, group) queue: the resident pool at `now` and the players the last tick matched (988 bytes)."""
    _fields_ = [
        ("mode", C.c_uint8),
        ("group", C.c_uint8),
        ("reserved", C.c_uint16),
        ("n_waiting", C.c_uint32),
        ("n_removed", C.c_uint32),
        ("max_wait", C.c_uint32),
        ("wait_hist", C.c_uint32 * MM_WAIT_BUCKETS),
        ("n_lobbies", C.c_uint32),
        ("n_matched", C.c_uint32),
        ("max_match_wait", C.c_uint32),
        ("match_wait_hist", C.c_uint32 * MM_WAIT_BUCKETS),
    ]


# every symbol include/mm_engine.h declares: name -> (restype, argtypes)
_P = C.POINTER
_vp = C.c_void_p
PROTOTYPES = {
    "mm_create": (C.c_int, [_P(Config), _P(_vp)]),
    "mm_destroy": (C.c_int, [_vp]),
    "mm_config_default": (None, [_P(Config)]),
    "mm_group_of": (C.c_int, [_P(Config), C.c_int32]),
    "mm_enqueue": (C.c_int, [_vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp]),
    "mm_enqueue_device": (C.c_int, [_vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp, _P(C.c_uint32)]),
    "mm_enqueue_packed": (C.c_int, [_vp, C.c_uint32, _vp, _vp, _vp, _vp]),
    "mm_enqueue_packed_begin": (C.c_int, [_vp, C.c_uint32, _vp, _vp, _vp]),
    "mm_enqueue_packed_end": (C.c_int, [_vp, _vp, _vp]),
    "mm_enqueue_rejects": (C.c_int, [_vp, C.c_uint32, _vp, _vp, _P(C.c_uint32)]),
    "mm_remove": (C.c_int, [_vp, C.c_uint32, _vp, _P(C.c_uint32)]),
    "mm_remove_packed": (C.c_int, [_vp, C.c_uint32, _vp, _P(C.c_uint32)]),
    "mm_take": (C.c_int, [_vp, C.c_uint32, _vp, _P(C.c_uint32)]),
    "mm_in_queue": (C.c_int, [_vp, C.c_uint32, _vp, _vp]),
    "mm_pool_size": (C.c_int, [_vp, _P(C.c_uint32)]),
    "mm_active_size": (C.c_int, [_vp, _P(C.c_uint32)]),
    "mm_tick": (C.c_int, [_vp, C.c_uint64, _vp, C.c_uint32, _vp, C.c_uint64, _vp, _P(TickStats)]),
    "mm_tick_packed": (C.c_int, [_vp, C.c_uint64, _vp, C.c_uint32, _vp, C.c_uint64, _vp, _P(TickStats)]),
    "mm_results_wait": (C.c_int, [_vp]),
    "mm_tick_device": (C.c_int, [_vp, C.c_uint64, _P(TickStats)]),
    "mm_results_device": (C.c_int, [_vp, _P(_vp), _P(_vp)]),
    "mm_pool_read": (C.c_int, [_vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp, _P(C.c_uint32)]),
    "mm_queue_stats": (C.c_int, [_vp, C.c_uint64, _vp, C.c_uint32, _P(C.c_uint32)]),
    "mm_snapshot": (C.c_int, [_vp]),
    "mm_restore": (C.c_int, [_vp]),
    "mm_set_stream": (C.c_int, [_vp, _vp]),
    "mm_set_option": (C.c_int, [_vp, C.c_char_p, C.c_int64]),
    "mm_strerror": (C.c_char_p, [C.c_int]),
    "mm_last_error": (C.c_char_p, [_vp]),
    "mm_abi_version": (C.c_uint32, []),
}


def bind(lib):
    """Attach restype/argtypes for every declared symbol; raises if one is missing."""
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export it
        fn.restype = res
        fn.argtypes = args
    return lib
