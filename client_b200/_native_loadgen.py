"""ctypes declarations for include/tb200_loadgen.h (loaded by _native.load())."""

import ctypes

from ._native import CheckJob, CopyJob, FillJob

c_vp, c_u64, c_int = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_int


class LoadgenConfig(ctypes.Structure):
    """tb200_loadgen_config."""

    _fields_ = [
        ("host", ctypes.c_char_p), ("port", c_int), ("concurrency", c_int),
        ("requests", ctypes.POINTER(c_vp)), ("request_sizes", ctypes.POINTER(c_u64)),
        ("tails", ctypes.POINTER(c_vp)), ("tail_sizes", ctypes.POINTER(c_u64)),
        ("ctx", c_vp), ("fill_jobs", ctypes.POINTER(FillJob)), ("fill_jobs_per_slot", c_int),
        ("seed", c_u64), ("regenerate", c_int),
        ("check_jobs", ctypes.POINTER(CheckJob)), ("check_jobs_per_slot", c_int), ("results", c_vp),
        ("device_window_us", ctypes.c_uint32), ("protocol", ctypes.c_uint32), ("grpc_path", ctypes.c_char_p),
        ("lookahead", ctypes.c_uint32), ("tail_stride", c_u64), ("requests_per_slot", ctypes.c_uint32),
        ("pipeline_depth", ctypes.c_uint32),
        ("replay_entries", c_u64), ("copy_jobs", ctypes.POINTER(CopyJob)), ("copy_jobs_per_slot", c_int),
        ("copy_src_stride", ctypes.POINTER(c_u64)), ("check_b_stride", ctypes.POINTER(c_u64)),
    ]


class LoadgenStats(ctypes.Structure):
    """tb200_loadgen_stats."""

    _fields_ = [
        ("completed_request_count", c_u64), ("failed_request_count", c_u64),
        ("cumulative_total_request_time_ns", c_u64), ("cumulative_send_time_ns", c_u64),
        ("cumulative_receive_time_ns", c_u64),
        ("p50_ns", c_u64), ("p90_ns", c_u64), ("p95_ns", c_u64), ("p99_ns", c_u64), ("min_ns", c_u64), ("max_ns", c_u64),
        ("window_seconds", ctypes.c_double),
        ("device_batches", c_u64), ("device_slots", c_u64), ("nonfinite_outputs", c_u64), ("check_mismatches", c_u64),
        ("response_count", c_u64), ("first_response_p50_ns", c_u64), ("first_response_p99_ns", c_u64),
    ]


LOADGEN_SIGNATURES = {
    "tb200_loadgen_create": (c_int, [ctypes.POINTER(LoadgenConfig), ctypes.POINTER(c_vp)]),
    "tb200_loadgen_start": (c_int, [c_vp]),
    "tb200_loadgen_window": (c_int, [c_vp, ctypes.c_double, ctypes.POINTER(LoadgenStats)]),
    "tb200_loadgen_wait_count": (c_int, [c_vp, c_u64, ctypes.c_double, ctypes.POINTER(c_u64)]),
    "tb200_loadgen_stop": (c_int, [c_vp]),
    "tb200_loadgen_destroy": (c_int, [c_vp]),
    "tb200_loadgen_replay_entry": (c_u64, [c_u64, c_u64, ctypes.c_uint32, c_int, c_u64]),
    "tb200_stub_server_start": (c_int, [ctypes.c_char_p, ctypes.POINTER(c_int), ctypes.c_char_p, ctypes.POINTER(c_vp)]),
    "tb200_stub_server_stop": (c_int, [c_vp]),
    "tb200_grpc_stub_server_start": (c_int, [ctypes.c_char_p, ctypes.POINTER(c_int), c_vp, c_u64, ctypes.POINTER(c_vp)]),
    "tb200_grpc_stub_server_start_streaming": (c_int, [ctypes.c_char_p, ctypes.POINTER(c_int), c_vp, c_u64, c_vp, c_u64, c_int, ctypes.POINTER(c_vp)]),
    "tb200_grpc_stub_server_stop": (c_int, [c_vp]),
    "tb200_grpc_echo_server_start": (c_int, [ctypes.c_char_p, ctypes.POINTER(c_int), ctypes.POINTER(c_vp)]),
    "tb200_grpc_echo_server_stop": (c_int, [c_vp]),
    "tb200_mock_server_start": (c_int, [ctypes.c_char_p, ctypes.POINTER(c_int), c_int, ctypes.POINTER(c_vp)]),
    "tb200_mock_server_start2": (c_int, [ctypes.c_char_p, ctypes.POINTER(c_int), ctypes.POINTER(c_int), c_int, ctypes.POINTER(c_vp)]),
    "tb200_mock_server_requests": (ctypes.c_uint64, [c_vp]),
    "tb200_mock_server_batches": (ctypes.c_uint64, [c_vp]),
    "tb200_mock_server_stop": (c_int, [c_vp]),
}


def declare(lib):
    for name, (restype, argtypes) in LOADGEN_SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = restype
        fn.argtypes = argtypes
