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

MM_BUDGET_UNLIMITED = 0xFFFFFFFF


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


class BandStats(C.Structure):
    """mm_band_stats: counts of one mm_band_match call (32 bytes)."""
    _fields_ = [
        ("n_lobbies", C.c_uint32),
        ("n_matched", C.c_uint32),
        ("n_taken", C.c_uint32),
        ("n_upper_taken", C.c_uint32),
        ("device_us", C.c_float),
        ("reserved", C.c_uint32 * 3),
    ]


MM_WAIT_BUCKETS = 120


class BackfillReq(C.Structure):
    """mm_backfill_req: one backfill request (16 bytes)."""
    _fields_ = [
        ("mode", C.c_uint8),
        ("group", C.c_uint8),
        ("reserved", C.c_uint16),
        ("count", C.c_uint32),
        ("target", C.c_int32),
        ("window", C.c_int32),
    ]


MM_WIDEN_OFF = 0xFFFFFFFF


class WidenRule(C.Structure):
    """mm_widen_rule: the widening window of one (mode, group) queue (24 bytes)."""
    _fields_ = [
        ("min_wait", C.c_uint32),
        ("step", C.c_uint32),
        ("w0", C.c_int32),
        ("inc", C.c_int32),
        ("w_max", C.c_int32),
        ("reserved", C.c_uint32),
    ]


class WidenStats(C.Structure):
    """mm_widen_stats: counts of one mm_widen call (32 bytes)."""
    _fields_ = [
        ("n_anchors", C.c_uint32),
        ("n_lobbies", C.c_uint32),
        ("n_matched", C.c_uint32),
        ("n_absorbed", C.c_uint32),
        ("device_us", C.c_float),
        ("reserved", C.c_uint32 * 3),
    ]


class PartyStats(C.Structure):
    """mm_party_stats: counts of one mm_party_match call (32 bytes)."""
    _fields_ = [
        ("n_anchors", C.c_uint32),
        ("n_lobbies", C.c_uint32),
        ("n_matched", C.c_uint32),
        ("n_parties", C.c_uint32),
        ("n_absorbed", C.c_uint32),
        ("device_us", C.c_float),
        ("sum_imbalance", C.c_uint64),  # party_balance: summed imbalance of the emitted lobbies of masked modes
    ]


assert C.sizeof(WidenRule) == 24 and C.sizeof(WidenStats) == 32 and C.sizeof(PartyStats) == 32

MM_LOCATE_STAYS = 0xFFFFFFFF


class PlayerStatus(C.Structure):
    """mm_player_status: one player's search status (36 bytes)."""
    _fields_ = [
        ("state", C.c_uint8),
        ("mode", C.c_uint8),
        ("group", C.c_uint8),
        ("reserved", C.c_uint8),
        ("rating", C.c_int32),
        ("enq_ts", C.c_uint32),
        ("seq", C.c_uint32),
        ("wait", C.c_uint32),
        ("ahead", C.c_uint32),
        ("depth", C.c_uint32),
        ("lobby", C.c_uint32),
        ("member", C.c_uint16),
        ("reserved2", C.c_uint16),
    ]


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


class LobbyQuality(C.Structure):
    """mm_lobby_quality: rating spread, sum and team imbalance of one lobby of the last tick (24 bytes)."""
    _fields_ = [
        ("min_rating", C.c_int32),
        ("max_rating", C.c_int32),
        ("rating_sum", C.c_int64),
        ("imbalance", C.c_uint32),
        ("reserved", C.c_uint32),
    ]


class QueueQuality(C.Structure):
    """mm_queue_quality: spread and imbalance of one (mode, group) queue's lobbies of the last tick (992 bytes)."""
    _fields_ = [
        ("mode", C.c_uint8),
        ("group", C.c_uint8),
        ("reserved", C.c_uint16),
        ("n_lobbies", C.c_uint32),
        ("max_spread", C.c_uint32),
        ("max_imbalance", C.c_uint32),
        ("sum_spread", C.c_uint64),
        ("sum_imbalance", C.c_uint64),
        ("spread_hist", C.c_uint32 * MM_WAIT_BUCKETS),
        ("imbalance_hist", C.c_uint32 * MM_WAIT_BUCKETS),
    ]


MM_PARTY_SIZE_BUCKETS = 16


class PartyQueueStat(C.Structure):
    """mm_party_queue_stat: the queued parties of one (mode, group) queue (560 bytes)."""
    _fields_ = [
        ("mode", C.c_uint8),
        ("group", C.c_uint8),
        ("reserved", C.c_uint16),
        ("n_parties", C.c_uint32),
        ("n_members", C.c_uint32),
        ("max_wait", C.c_uint32),
        ("wait_hist", C.c_uint32 * MM_WAIT_BUCKETS),
        ("size_hist", C.c_uint32 * MM_PARTY_SIZE_BUCKETS),
    ]


class PartyMemberStatus(C.Structure):
    """mm_party_member_status: one party member's search status and next mm_party_match lobby (48 bytes)."""
    _fields_ = [
        ("state", C.c_uint8),
        ("mode", C.c_uint8),
        ("group", C.c_uint8),
        ("size", C.c_uint8),
        ("index", C.c_uint8),
        ("anchor", C.c_uint8),
        ("reserved", C.c_uint16),
        ("rating", C.c_int32),
        ("party_rating", C.c_int32),
        ("enq_ts", C.c_uint32),
        ("seq", C.c_uint32),
        ("wait", C.c_uint32),
        ("window", C.c_int32),
        ("ahead", C.c_uint32),
        ("depth", C.c_uint32),
        ("lobby", C.c_uint32),
        ("member", C.c_uint16),
        ("reserved2", C.c_uint16),
    ]


assert C.sizeof(PartyQueueStat) == 560 and C.sizeof(PartyMemberStatus) == 48

MM_OFFTICK_PARTY_MATCH = 0  # mm_offtick_report / mm_set_offtick_budget sources
MM_OFFTICK_WIDEN = 1


class MatchWaits(C.Structure):
    """mm_match_waits: the match section of mm_queue_stat for one off-tick call's lobbies of a queue (496 bytes)."""
    _fields_ = [
        ("mode", C.c_uint8),
        ("group", C.c_uint8),
        ("reserved", C.c_uint16),
        ("n_lobbies", C.c_uint32),
        ("n_matched", C.c_uint32),
        ("max_match_wait", C.c_uint32),
        ("match_wait_hist", C.c_uint32 * MM_WAIT_BUCKETS),
    ]


MM_IMAGE_MAGIC = 0x474D494D
MM_QUEUE_IMAGE_MAGIC = 0x5155514D  # mm_export_queues: same header and sections, no active section
MM_IMAGE_VERSION = 1
MM_PARTY_IMAGE_MAGIC = 0x5954504D  # mm_export_parties: the mm_image_header, then the party sections
MM_PARTY_KEEP_SEQ = 1  # mm_merge_parties: every party keeps its image seq (resume)


class ImageHeader(C.Structure):
    """mm_image_header: the first 624 bytes of an mm_export image."""
    _fields_ = [
        ("magic", C.c_uint32),
        ("version", C.c_uint32),
        ("abi_version", C.c_uint32),
        ("id_bytes", C.c_uint32),
        ("total_bytes", C.c_uint64),
        ("n_parts", C.c_uint32),
        ("n_players", C.c_uint32),
        ("n_active", C.c_uint32),
        ("seq_next", C.c_uint32),
        ("config", Config),
        ("reserved", C.c_uint32),
    ]


class RecutParties(C.Structure):
    """mm_recut_parties: the party images of mm_import_regroup_many_parties and what the call reports about them."""
    _fields_ = [
        ("bufs", C.c_void_p),
        ("n_bytes", C.c_void_p),
        ("cap", C.c_uint32),
        ("rej_image", C.c_void_p),
        ("rej_index", C.c_void_p),
        ("n_rejected", C.c_uint32),
        ("n_elsewhere", C.c_uint32),
        ("n_loaded", C.c_uint32),
        ("reserved", C.c_uint32),
    ]


def image_offsets(n_parts, n_players, n_active, id_bytes):
    """Section offsets of an image (include/mm_engine.h): part_count, id, rating, enq_ts, seq, mode, active, and the
    total length.  Every section starts at the next multiple of 8 after the one before it."""
    sizes = (4 * n_parts, id_bytes * n_players, 4 * n_players, 4 * n_players, 4 * n_players, n_players,
             id_bytes * n_active)
    off = [C.sizeof(ImageHeader)]
    for s in sizes:
        off.append((off[-1] + s + 7) & ~7)
    return off


def party_image_offsets(n_parties, n_members, id_bytes):
    """Section offsets of a party image (include/mm_engine.h): size, seq, enq_ts, mode, id, rating, and the total
    length.  Every section starts at the next multiple of 8 after the one before it."""
    sizes = (n_parties, 4 * n_parties, 4 * n_parties, n_parties, id_bytes * n_members, 4 * n_members)
    off = [C.sizeof(ImageHeader)]
    for s in sizes:
        off.append((off[-1] + s + 7) & ~7)
    return off


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
    "mm_requeue": (C.c_int, [_vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp, _vp, _P(C.c_uint32)]),
    "mm_seq_next": (C.c_int, [_vp, _P(C.c_uint32)]),
    "mm_band_candidates": (C.c_int, [_vp, C.c_int32, C.c_uint32, _vp, _vp, _vp, C.c_uint32, _P(C.c_uint32)]),
    "mm_band_match": (C.c_int, [_vp, C.c_int32, C.c_uint32, C.c_uint32, C.c_uint32, _vp, _vp, _vp, C.c_uint32,
                                _vp, C.c_uint32, _vp, C.c_uint64, _vp, _P(BandStats)]),
    "mm_backfill": (C.c_int, [_vp, C.c_uint32, _vp, _vp, _vp, C.c_uint64, _P(C.c_uint32)]),
    "mm_backfill_party": (C.c_int, [_vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp, C.c_uint64, _P(C.c_uint32)]),
    "mm_widen": (C.c_int, [_vp, C.c_uint64, _vp, _vp, C.c_uint32, _vp, C.c_uint64, _P(WidenStats)]),
    "mm_enqueue_party": (C.c_int, [_vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mm_party_match": (C.c_int, [_vp, C.c_uint64, _vp, _vp, C.c_uint32, _vp, C.c_uint64, _P(PartyStats)]),
    "mm_party_read": (C.c_int, [_vp, C.c_uint32, C.c_uint32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _P(C.c_uint32),
                                _P(C.c_uint32)]),
    "mm_export_parties": (C.c_int, [_vp, _vp, _vp, C.c_uint64, _P(C.c_uint64)]),
    "mm_merge_parties": (C.c_int, [_vp, _vp, C.c_uint64, C.c_uint32, _vp, _P(C.c_uint32)]),
    "mm_requeue_party": (C.c_int, [_vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _P(C.c_uint32)]),
    "mm_in_queue": (C.c_int, [_vp, C.c_uint32, _vp, _vp]),
    "mm_locate": (C.c_int, [_vp, C.c_uint64, C.c_uint32, _vp, _vp]),
    "mm_pool_size": (C.c_int, [_vp, _P(C.c_uint32)]),
    "mm_active_size": (C.c_int, [_vp, _P(C.c_uint32)]),
    "mm_tick": (C.c_int, [_vp, C.c_uint64, _vp, C.c_uint32, _vp, C.c_uint64, _vp, _P(TickStats)]),
    "mm_tick_packed": (C.c_int, [_vp, C.c_uint64, _vp, C.c_uint32, _vp, C.c_uint64, _vp, _P(TickStats)]),
    "mm_results_wait": (C.c_int, [_vp]),
    "mm_tick_device": (C.c_int, [_vp, C.c_uint64, _P(TickStats)]),
    "mm_results_device": (C.c_int, [_vp, _P(_vp), _P(_vp)]),
    "mm_pool_read": (C.c_int, [_vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp, _P(C.c_uint32)]),
    "mm_queue_stats": (C.c_int, [_vp, C.c_uint64, _vp, C.c_uint32, _P(C.c_uint32)]),
    "mm_party_queue_stats": (C.c_int, [_vp, C.c_uint64, _vp, C.c_uint32, _P(C.c_uint32)]),
    "mm_party_locate": (C.c_int, [_vp, C.c_uint64, _vp, C.c_uint32, _vp, _vp]),
    "mm_match_quality": (C.c_int, [_vp, _vp, C.c_uint32, _P(C.c_uint32), _vp, C.c_uint32, _P(C.c_uint32)]),
    "mm_offtick_report": (C.c_int, [_vp, C.c_uint32, _vp, _vp, C.c_uint32, _P(C.c_uint32), _vp, C.c_uint32,
                                    _P(C.c_uint32)]),
    "mm_set_lobby_budget": (C.c_int, [_vp, _vp, _vp]),
    "mm_lobby_budget_report": (C.c_int, [_vp, _vp, _vp, C.c_uint32, _P(C.c_uint32)]),
    "mm_lobby_candidates": (C.c_int, [_vp, _vp, C.c_uint32, _P(C.c_uint32)]),
    "mm_set_offtick_budget": (C.c_int, [_vp, C.c_uint32, _vp, _vp]),
    "mm_offtick_budget_report": (C.c_int, [_vp, C.c_uint32, _vp, _vp, C.c_uint32, _P(C.c_uint32)]),
    "mm_expire": (C.c_int, [_vp, C.c_uint64, C.c_uint32, _vp, _vp, C.c_uint32, _P(C.c_uint32)]),
    "mm_expire_packed": (C.c_int, [_vp, C.c_uint64, C.c_uint32, _vp, _vp, C.c_uint32, _P(C.c_uint32)]),
    "mm_export": (C.c_int, [_vp, _vp, C.c_uint64, _P(C.c_uint64)]),
    "mm_import": (C.c_int, [_vp, _vp, C.c_uint64]),
    "mm_export_queues": (C.c_int, [_vp, _vp, _vp, C.c_uint64, _P(C.c_uint64)]),
    "mm_merge": (C.c_int, [_vp, _vp, C.c_uint64, C.c_uint32, _vp, _P(C.c_uint32)]),
    "mm_import_regroup": (C.c_int, [_vp, _vp, C.c_uint64, C.c_uint32, _vp, _P(C.c_uint32)]),
    "mm_import_regroup_many": (C.c_int, [_vp, C.c_uint32, _vp, _vp, _vp, C.c_uint32, C.c_uint32, _vp, _vp,
                                         _P(C.c_uint32), _P(C.c_uint32)]),
    "mm_import_regroup_many_parties": (C.c_int, [_vp, C.c_uint32, _vp, _vp, _vp, C.c_uint32, C.c_uint32, _vp, _vp,
                                                 _P(C.c_uint32), _P(C.c_uint32), _P(RecutParties)]),
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
