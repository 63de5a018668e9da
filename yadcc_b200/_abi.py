"""ctypes declarations for include/ydsched.h (one-to-one, same order)."""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import numpy as np

ABI_VERSION = 1

STATUS_ENVIRONMENT_NOT_FOUND = 0  # WaitStatus::EnvironmentNotFound, task_dispatcher.h:42
STATUS_TIMEOUT = 1  # WaitStatus::Timeout, task_dispatcher.h:43
STATUS_GRANTED = 2

PRIORITY_UNKNOWN = 0  # scheduler.proto:38-48
PRIORITY_DEDICATED = 1
PRIORITY_USER = 2

REQ_FLAG_PREFETCH = 1
NO_SERVANT = 0xFFFFFFFF

# struct yd_task_req (24 B) / yd_grant (16 B) / yd_servant_state (32 B)
REQ_DTYPE = np.dtype(
    [
        ("env_id", "<u4"),
        ("min_version", "<u4"),
        ("requestor_ip", "<u4"),
        ("flags", "<u4"),
        ("expires_in_ns", "<i8"),
    ]
)
GRANT_DTYPE = np.dtype([("task_id", "<u8"), ("servant_index", "<u4"), ("status", "<u4")])
SERVANT_STATE_DTYPE = np.dtype(
    [
        ("running_tasks", "<u8"),
        ("ever_assigned_tasks", "<u8"),
        ("capacity_available", "<u8"),
        ("expires_at_ns", "<i8"),
    ]
)
# struct yd_rpc_wait (32 B) / yd_rpc_wait_result (16 B)
RPC_WAIT_DTYPE = np.dtype(
    [
        ("env_id", "<u4"),
        ("min_version", "<u4"),
        ("requestor_ip", "<u4"),
        ("immediate_reqs", "<u4"),
        ("prefetch_reqs", "<u4"),
        ("milliseconds_to_wait", "<u4"),
        ("next_keep_alive_ns", "<i8"),
    ]
)
RUNNING_HIT_DTYPE = np.dtype([("servant_task_id", "<u8"), ("snapshot_index", "<u4"), ("found", "<u4")])
RPC_RESULT_DTYPE = np.dtype([("status", "<u4"), ("n_grants", "<u4"), ("first_grant", "<u4"), ("reserved", "<u4")])
RPC_OK, RPC_NO_QUOTA_AVAILABLE, RPC_INVALID_ARGUMENT, RPC_ENVIRONMENT_NOT_AVAILABLE = 0, 1001, 1004, 1006
# struct yd_task_req16 (16 B) / yd_grant8 (8 B) / yd_packed_ids: the packed interface
REQ16_DTYPE = np.dtype([("env_id", "<u4"), ("min_version", "<u4"), ("requestor_ip", "<u4"), ("lease", "<u4")])
GRANT8_DTYPE = np.dtype([("servant_index", "<u4"), ("status_ordinal", "<u4")])
PACKED_IDS_DTYPE = np.dtype([("first_task_id", "<u8"), ("stride", "<u8")])
LEASE_PREFETCH = 0x80000000
assert REQ_DTYPE.itemsize == 24 and GRANT_DTYPE.itemsize == 16 and RPC_WAIT_DTYPE.itemsize == 32
assert REQ16_DTYPE.itemsize == 16 and GRANT8_DTYPE.itemsize == 8


class yd_prefilter(C.Structure):
    _fields_ = [("cache_keys", C.c_void_p), ("cache_key_len", C.c_size_t), ("cache_key_stride", C.c_size_t),
                ("task_digests", C.c_void_p), ("task_digest_len", C.c_size_t), ("task_digest_stride", C.c_size_t)]


class yd_prefilter_packed(C.Structure):
    """The pre-filters over 32-byte binary digests: n contiguous records each, or NULL to skip the stage."""
    _fields_ = [("cache_digests", C.c_void_p), ("task_digests", C.c_void_p)]


FILTER_OFFERED, FILTER_CACHE_HIT, FILTER_JOINED = 0, 1, 2


class yd_task_sources(C.Structure):
    _fields_ = [("args", C.c_void_p), ("args_offsets", C.c_void_p), ("n_args", C.c_size_t), ("args_index", C.c_void_p),
                ("source_digests", C.c_void_p), ("source_digest_len", C.c_size_t), ("source_digest_stride", C.c_size_t)]


KEYS_OK, KEYS_BAD_SOURCES, KEYS_UNKNOWN_ENV, KEYS_BAD_ARGS_INDEX, KEYS_TOO_LONG = 0, 1, 2, 3, 4
KEYS_CACHE_KEY_LEN, KEYS_TASK_DIGEST_LEN = 81, 64
KEYS_MAX_ARGS_LEN, KEYS_MAX_DIGEST_LEN = 256 << 10, 64 << 10
STAGE_CACHE, STAGE_DEDUPE = 1, 2


class yd_config(C.Structure):
    _fields_ = [
        ("abi_version", C.c_uint32),
        ("device", C.c_int32),
        ("servant_min_memory_for_accepting_new_task", C.c_char_p),
        ("solver", C.c_uint32),
        ("reserved", C.c_uint32),
        ("id_stride", C.c_uint32),
        ("id_offset", C.c_uint32),
    ]


class yd_servant(C.Structure):
    _fields_ = [
        ("version", C.c_int32),
        ("priority", C.c_int32),
        ("not_accepting_task_reason", C.c_int32),
        ("num_envs", C.c_uint32),
        ("observed_location", C.c_char_p),
        ("reported_location", C.c_char_p),
        ("env_digests", C.POINTER(C.c_char_p)),
        ("num_processors", C.c_uint32),
        ("current_load", C.c_uint32),
        ("max_tasks", C.c_uint32),
        ("reserved", C.c_uint32),
        ("total_memory_in_bytes", C.c_uint64),
        ("memory_available_in_bytes", C.c_uint64),
    ]


class yd_running_task(C.Structure):
    _fields_ = [
        ("servant_task_id", C.c_uint64),
        ("task_grant_id", C.c_uint64),
        ("servant_location", C.c_char_p),
        ("task_digest", C.c_char_p),
    ]


class yd_heartbeat_item(C.Structure):
    _fields_ = [
        ("servant_location", C.c_char_p),
        ("tasks", C.POINTER(yd_running_task)),
        ("n_tasks", C.c_size_t),
    ]


class yd_service_config(C.Structure):
    _fields_ = [
        ("acceptable_user_tokens", C.c_char_p),
        ("acceptable_servant_tokens", C.c_char_p),
        ("min_daemon_version", C.c_int32),
        ("serving_daemon_token_rollout_interval_s", C.c_int32),
        ("token_seed", C.c_uint64),
    ]


class yd_heartbeat_request(C.Structure):
    _fields_ = [
        ("token", C.c_char_p),
        ("location", C.c_char_p),
        ("remote_ip", C.c_char_p),
        ("remote_is_ipv6", C.c_uint32),
        ("next_heartbeat_in_ms", C.c_uint32),
        ("version", C.c_uint32),
        ("num_processors", C.c_uint32),
        ("current_load", C.c_uint32),
        ("servant_priority", C.c_uint32),
        ("not_accepting_task_reason", C.c_uint32),
        ("capacity", C.c_uint32),
        ("n_env_digests", C.c_uint32),
        ("total_memory_in_bytes", C.c_uint64),
        ("memory_available_in_bytes", C.c_uint64),
        ("env_digests", C.POINTER(C.c_char_p)),
        ("running_tasks", C.POINTER(yd_running_task)),
        ("n_running_tasks", C.c_size_t),
    ]


class yd_heartbeat_response(C.Structure):
    _fields_ = [
        ("acceptable_tokens", C.c_char_p * 3),
        ("expired_tasks", C.POINTER(C.c_uint64)),
        ("n_expired_tasks", C.c_size_t),
    ]


class yd_keep_task_alive_request(C.Structure):
    _fields_ = [
        ("token", C.c_char_p),
        ("next_keep_alive_in_ms", C.c_uint32),
        ("task_grant_ids", C.c_void_p),
        ("n", C.c_size_t),
        ("statuses", C.c_void_p),
    ]


class yd_free_task_request(C.Structure):
    _fields_ = [("token", C.c_char_p), ("task_grant_ids", C.c_void_p), ("n", C.c_size_t)]


class yd_wire_in(C.Structure):
    _fields_ = [("data", C.c_void_p), ("len", C.c_size_t), ("remote_ip", C.c_char_p), ("remote_is_ipv6", C.c_uint32),
                ("reserved", C.c_uint32)]


class yd_wire_out(C.Structure):
    _fields_ = [("consumed", C.c_size_t), ("offset", C.c_size_t), ("len", C.c_size_t), ("verdict", C.c_int32),
                ("status", C.c_int32)]


class yd_solve_stats(C.Structure):
    _fields_ = [
        ("total_ms", C.c_double),
        ("solve_ms", C.c_double),
        ("prep_ms", C.c_double),
        ("final_ms", C.c_double),
        ("decisions", C.c_uint64),
        ("granted", C.c_uint64),
        ("kernel_launches", C.c_uint32),
        ("solver", C.c_uint32),
        ("h2d_bytes", C.c_uint64),
        ("d2h_bytes", C.c_uint64),
    ]


# Every symbol include/ydsched.h declares: (name, restype, argtypes).
_P = C.c_void_p
PROTOTYPES = [
    ("yd_create", _P, [C.POINTER(yd_config)]),
    ("yd_destroy", None, [_P]),
    ("yd_backend_name", C.c_char_p, []),
    ("yd_parse_size", C.c_int, [C.c_char_p, C.POINTER(C.c_uint64)]),
    ("yd_intern_env", C.c_uint32, [_P, C.c_char_p, C.c_size_t]),
    ("yd_intern_ip", C.c_uint32, [_P, C.c_char_p, C.c_size_t]),
    ("yd_keep_servant_alive", None, [_P, C.c_int64, C.POINTER(yd_servant), C.c_int64]),
    (
        "yd_notify_servant_running_tasks",
        C.c_size_t,
        [_P, C.c_char_p, C.POINTER(yd_running_task), C.c_size_t, C.POINTER(C.c_uint64)],
    ),
    ("yd_get_running_tasks", C.c_size_t, [_P, C.POINTER(yd_running_task), C.c_size_t]),
    ("yd_on_expiration_timer", None, [_P, C.c_int64]),
    ("yd_wait_for_starting_new_tasks", None, [_P, C.c_int64, _P, C.c_size_t, _P]),
    ("yd_wait_for_starting_new_tasks_packed", None, [_P, C.c_int64, _P, C.c_size_t, _P, _P]),
    ("yd_stage_requests", None, [_P, _P, C.c_size_t]),
    ("yd_wait_for_staged_tasks", None, [_P, C.c_int64, C.c_size_t, _P]),
    ("yd_keep_task_alive", None, [_P, C.c_int64, _P, C.c_size_t, C.c_int64, _P]),
    ("yd_free_tasks", None, [_P, _P, C.c_size_t]),
    ("yd_wait_for_starting_task_rpcs", C.c_size_t, [_P, C.c_int64, _P, C.c_size_t, _P, _P, C.c_size_t]),
    ("yd_grant_capacity_bound", C.c_uint64, [_P]),
    ("yd_keep_servants_alive", None, [_P, C.c_int64, C.POINTER(yd_servant), C.POINTER(C.c_int64), C.c_size_t]),
    ("yd_notify_servants_running_tasks", C.c_size_t,
     [_P, C.POINTER(yd_heartbeat_item), C.c_size_t, C.POINTER(C.c_uint64), C.POINTER(C.c_size_t)]),
    ("yd_rpc_expanded_requests", C.c_size_t, [_P, _P, C.c_size_t]),
    ("yd_filter_and_wait_for_starting_new_tasks", C.c_size_t, [_P, C.c_int64, _P, C.c_size_t, _P, _P, _P, _P]),
    ("yd_bloom_reset", C.c_int, [_P, C.c_uint64, C.c_uint32]),
    ("yd_bloom_load", C.c_int, [_P, _P, C.c_size_t, C.c_uint32]),
    ("yd_bloom_add", None, [_P, _P, C.c_size_t, C.c_size_t, C.c_size_t]),
    ("yd_bloom_possibly_contains", None, [_P, _P, C.c_size_t, C.c_size_t, C.c_size_t, _P]),
    ("yd_bloom_get_bytes", C.c_size_t, [_P, _P, C.c_size_t]),
    ("yd_get_servant_personality", C.c_int, [_P, C.c_uint32, C.POINTER(yd_servant)]),
    ("yd_running_index_refresh", C.c_size_t, [_P]),
    ("yd_running_index_size", C.c_size_t, [_P]),
    ("yd_running_index_find", None, [_P, _P, C.c_size_t, C.c_size_t, C.c_size_t, _P]),
    ("yd_running_index_entry", C.c_int, [_P, C.c_uint32, _P]),
    ("yd_num_servants", C.c_size_t, [_P]),
    ("yd_servant_location", C.c_char_p, [_P, C.c_uint32]),
    ("yd_get_servant_state", C.c_size_t, [_P, _P, C.c_size_t]),
    ("yd_next_task_id", C.c_uint64, [_P]),
    ("yd_num_tasks", C.c_uint64, [_P]),
    ("yd_dump_internals_json", C.c_size_t, [_P, C.c_char_p, C.c_size_t]),
    ("yd_last_solve_stats", C.c_int, [_P, C.POINTER(yd_solve_stats)]),
    ("yd_alloc_host", _P, [C.c_size_t]),
    ("yd_free_host", None, [_P]),
]


def cuda_library_path() -> Path:
    """In-tree location of the product library (built by `make` / build())."""
    env = os.environ.get("YDSCHED_LIBRARY")
    return Path(env) if env else Path(__file__).resolve().parent / "libydsched.so"


def load_library(path: os.PathLike | str | None = None) -> C.CDLL:
    """dlopen a library exporting the ydsched C ABI and attach prototypes.

    With no argument this loads the CUDA product library and fails loudly if it
    has not been built -- there is no CPU fallback on the product path.
    """
    p = Path(path) if path is not None else cuda_library_path()
    if not p.exists():
        raise FileNotFoundError(
            f"{p} not found: build it first (`make -C {Path(__file__).resolve().parent.parent}` "
            "or `python -c 'import __graft_entry__ as g; g.build()'`). "
            "yadcc_b200 has no CPU fallback."
        )
    lib = C.CDLL(str(p), mode=C.RTLD_LOCAL)
    for name, restype, argtypes in PROTOTYPES + SERVICE_PROTOTYPES + WIRE_PROTOTYPES:
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.restype = restype
        fn.argtypes = argtypes
    # include/ydstate.h: the CUDA library and the port's state build (checkers/) export and import state; the task keys
    # are exported by the CUDA library and the checkers' key builds
    for name, restype, argtypes in STATE_PROTOTYPES + KEYS_PROTOTYPES:
        fn = getattr(lib, name, None)
        if fn is not None:
            fn.restype = restype
            fn.argtypes = argtypes
    # include/ydshard.h: only the CUDA library has the range-sharded multi-GPU path; include/ydfilter_packed.h,
    # include/ydrpcs_packed.h and include/ydruns.h: the CPU checkers export them from builds of their own (the product
    # library must export all)
    for name, restype, argtypes in SHARD_PROTOTYPES + FILTER_PACKED_PROTOTYPES + RPCS_PACKED_PROTOTYPES + RUNS_PROTOTYPES:
        fn = getattr(lib, name) if path is None else getattr(lib, name, None)
        if fn is not None:
            fn.restype = restype
            fn.argtypes = argtypes
    lib._yd_path = str(p)
    return lib


class yd_shard_stats(C.Structure):
    _fields_ = [
        ("total_ms", C.c_float),
        ("exchange_ms", C.c_float * 4),
        ("exchange_bytes", C.c_uint64 * 4),
        ("decisions_local", C.c_uint64),
        ("granted_local", C.c_uint64),
        ("granted_total", C.c_uint64),
        ("merge_rounds", C.c_uint32),
        ("kernel_launches", C.c_uint32),
    ]


SHARD_UNIQUE_ID_BYTES = 128
# Every symbol include/ydshard.h declares.
SHARD_PROTOTYPES = [
    ("yd_shard_unique_id", C.c_int, [_P]),
    ("yd_shard_init", C.c_int, [_P, C.c_int, C.c_int, _P]),
    ("yd_shard_finalize", None, [_P]),
    ("yd_shard_wait_for_starting_new_tasks", C.c_int, [_P, C.c_int64, _P, C.c_size_t, _P]),
    ("yd_shard_wait_for_starting_new_tasks_packed", C.c_int, [_P, C.c_int64, _P, C.c_size_t, _P, _P]),
    ("yd_shard_free_tasks", C.c_int, [_P, _P, C.c_size_t]),
    ("yd_shard_last_stats", C.c_int, [_P, C.POINTER(yd_shard_stats)]),
    ("yd_shard_export_state", C.c_size_t, [_P, C.c_int64, _P, C.c_size_t]),
    ("yd_shard_import_state", C.c_int, [_P, C.c_int64, _P, C.c_size_t]),
    ("yd_shard_keep_task_alive", C.c_int, [_P, C.c_int64, _P, C.c_size_t, C.c_int64, _P]),
    ("yd_shard_keep_tasks_alive", C.c_int, [_P, C.c_int64, _P, _P, C.c_size_t, _P]),
    ("yd_shard_notify_servants_running_tasks", C.c_size_t,
     [_P, C.POINTER(yd_heartbeat_item), C.c_size_t, C.POINTER(C.c_uint64), C.POINTER(C.c_size_t)]),
    ("yd_shard_get_running_tasks", C.c_size_t, [_P, C.POINTER(yd_running_task), C.c_size_t]),
    ("yd_shard_running_index_refresh", C.c_size_t, [_P]),
    ("yd_shard_wait_for_starting_task_rpcs", C.c_size_t, [_P, C.c_int64, _P, C.c_size_t, _P, _P, C.c_size_t]),
    ("yd_shard_service_create", _P, [_P, C.c_int64, C.POINTER(yd_service_config)]),
    ("yd_shard_filter_and_wait_for_starting_new_tasks", C.c_size_t, [_P, C.c_int64, _P, C.c_size_t, _P, _P, _P, _P]),
    ("yd_shard_derive_filter_and_wait_for_starting_new_tasks", C.c_size_t,
     [_P, C.c_int64, _P, C.c_size_t, _P, C.c_uint32, _P, _P, _P]),
    ("yd_shard_filter_and_wait_for_starting_new_tasks_packed", C.c_size_t,
     [_P, C.c_int64, _P, C.c_size_t, _P, _P, _P, _P, _P]),
    ("yd_shard_wait_for_starting_task_rpcs_packed", C.c_size_t, [_P, C.c_int64, _P, C.c_size_t, _P, _P, C.c_size_t, _P]),
]

# Every symbol include/ydstate.h declares, and its status codes.
# include/ydfilter_packed.h: the pre-filtered solve over binary digests and packed records.
FILTER_PACKED_PROTOTYPES = [
    ("yd_filter_and_wait_for_starting_new_tasks_packed", C.c_size_t,
     [_P, C.c_int64, _P, C.c_size_t, _P, _P, _P, _P, _P]),
]

# include/ydrpcs_packed.h: a window of WaitForStartingTask RPCs with 8-byte grants.
RPCS_PACKED_PROTOTYPES = [
    ("yd_wait_for_starting_task_rpcs_packed", C.c_size_t, [_P, C.c_int64, _P, C.c_size_t, _P, _P, C.c_size_t, _P]),
]

# include/ydkeys.h: the task keys, exported by the CUDA library and by the checkers' builds that have them
KEYS_PROTOTYPES = [
    ("yd_derive_task_keys", C.c_int, [_P, _P, C.c_size_t, _P, _P, _P]),
    ("yd_derive_filter_and_wait_for_starting_new_tasks", C.c_size_t,
     [_P, C.c_int64, _P, C.c_size_t, _P, C.c_uint32, _P, _P, _P]),
]

STATE_PROTOTYPES = [
    ("yd_export_state", C.c_size_t, [_P, C.c_int64, _P, C.c_size_t]),
    ("yd_import_state", C.c_int, [_P, C.c_int64, _P, C.c_size_t]),
]
STATE_OK, STATE_BAD_BLOB, STATE_NOT_FRESH, STATE_CONFIG_MISMATCH, STATE_UNSUPPORTED, STATE_NO_MEMORY = 0, 1, 2, 3, 4, 5

# Every symbol include/ydservice.h declares.
SERVICE_PROTOTYPES = [
    ("yd_service_create", _P, [_P, C.c_int64, C.POINTER(yd_service_config)]),
    ("yd_service_destroy", None, [_P]),
    ("yd_service_heartbeat", C.c_int, [_P, C.c_int64, C.POINTER(yd_heartbeat_request), C.POINTER(yd_heartbeat_response)]),
    ("yd_service_get_config", C.c_int, [_P, C.c_int64, C.c_char_p, C.POINTER(C.c_char_p)]),
    ("yd_service_wait_for_starting_tasks", C.c_size_t,
     [_P, C.c_int64, C.POINTER(C.c_char_p), _P, C.c_size_t, _P, _P, C.c_size_t]),
    ("yd_service_keep_task_alive", C.c_int, [_P, C.c_int64, C.c_char_p, C.c_uint32, _P, C.c_size_t, _P]),
    ("yd_service_free_task", C.c_int, [_P, C.c_char_p, _P, C.c_size_t]),
    ("yd_service_get_running_tasks", C.c_size_t, [_P, C.POINTER(yd_running_task), C.c_size_t]),
]

# include/ydruns.h: runs of Heartbeat, KeepTaskAlive and FreeTask RPCs as one batch each, and KeepTaskAlive with a lease
# length per id.
RUNS_PROTOTYPES = [
    ("yd_keep_tasks_alive", None, [_P, C.c_int64, _P, _P, C.c_size_t, _P]),
    ("yd_service_heartbeats", None,
     [_P, C.c_int64, C.POINTER(yd_heartbeat_request), C.c_size_t, C.POINTER(yd_heartbeat_response), C.POINTER(C.c_int)]),
    ("yd_service_keep_tasks_alive", None, [_P, C.c_int64, C.POINTER(yd_keep_task_alive_request), C.c_size_t, C.POINTER(C.c_int)]),
    ("yd_service_free_tasks", None, [_P, C.POINTER(yd_free_task_request), C.c_size_t, C.POINTER(C.c_int)]),
]

# Every symbol include/ydwire.h declares.
WIRE_PROTOTYPES = [
    ("yd_wire_handle_frames", C.c_size_t,
     [_P, C.c_int64, C.POINTER(yd_wire_in), C.c_size_t, _P, C.c_size_t, C.POINTER(yd_wire_out)]),
    ("yd_wire_call", C.c_int,
     [_P, C.c_int64, C.c_char_p, C.c_char_p, C.c_uint32, _P, C.c_size_t, _P, C.c_size_t, C.POINTER(C.c_size_t),
      C.POINTER(C.c_char_p)]),
]
