"""ctypes binding of libtb200.so (C ABI: include/tb200.h).

This is the only place that loads the native library.  Loading is lazy and
loud: if the library is missing or a symbol is absent the import of the first
CUDA-backed feature raises -- there is no Python/numpy fallback for device work.
"""

import ctypes
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libtb200.so")

c_u8p = ctypes.POINTER(ctypes.c_uint8)
c_vp = ctypes.c_void_p
c_u64 = ctypes.c_uint64
c_u32 = ctypes.c_uint32
c_i64 = ctypes.c_int64
c_int = ctypes.c_int

# tb200_dtype ---------------------------------------------------------------
DTYPE_CODES = {
    "BOOL": 1, "UINT8": 2, "UINT16": 3, "UINT32": 4, "UINT64": 5,
    "INT8": 6, "INT16": 7, "INT32": 8, "INT64": 9,
    "FP16": 10, "FP32": 11, "FP64": 12, "BYTES": 13, "BF16": 14,
}
DTYPE_NAMES = {v: k for k, v in DTYPE_CODES.items()}
DTYPE_SIZES = {
    "BOOL": 1, "UINT8": 1, "INT8": 1, "UINT16": 2, "INT16": 2, "FP16": 2, "BF16": 2,
    "UINT32": 4, "INT32": 4, "FP32": 4, "UINT64": 8, "INT64": 8, "FP64": 8,
}

FILL_RANDOM, FILL_ZERO, FILL_BYTE = 0, 1, 2
SCALE_NONE, SCALE_INCEPTION, SCALE_VGG = 0, 1, 2
SCALING_CODES = {"NONE": 0, "INCEPTION": 1, "VGG": 2}
NCHW, NHWC = 0, 1
CHECK_SUM, CHECK_EQUAL, CHECK_ADDSUB, CHECK_TOP1 = 0, 1, 2, 3
IPC_HANDLE_BYTES = 64
MAX_DIMS = 8


class FillJob(ctypes.Structure):
    """tb200_fill_job (64 bytes)."""

    _fields_ = [
        ("dst", c_u64), ("nbytes", c_u64), ("stream", c_u64),
        ("dtype", c_u32), ("mode", c_u32),
        ("lo", ctypes.c_double), ("span", ctypes.c_double),
        ("ilo", c_i64), ("irange", c_u64),
    ]


class CopyJob(ctypes.Structure):
    """tb200_copy_job."""

    _fields_ = [("dst", c_u64), ("src", c_u64), ("nbytes", c_u64)]


class CheckJob(ctypes.Structure):
    """tb200_check_job (48 bytes)."""

    _fields_ = [
        ("a", c_u64), ("b", c_u64), ("c", c_u64), ("d", c_u64),
        ("nbytes", c_u64), ("kind", c_u32), ("pad", c_u32),
    ]


class CheckResult(ctypes.Structure):
    """tb200_check_result (32 bytes)."""

    _fields_ = [
        ("mismatches", c_u64), ("sum", c_u64), ("xor32", c_u32),
        ("argmax", c_u32), ("max_value", ctypes.c_float), ("pad", c_u32),
    ]


class TopkJob(ctypes.Structure):
    """tb200_topk_job (24 bytes)."""

    _fields_ = [("src", c_u64), ("count", c_u64), ("dtype", c_u32), ("pad", c_u32)]


class TopkEntry(ctypes.Structure):
    """tb200_topk_entry."""

    _fields_ = [("value", ctypes.c_float), ("index", c_u32)]


assert ctypes.sizeof(TopkJob) == 24 and ctypes.sizeof(TopkEntry) == 8
assert ctypes.sizeof(FillJob) == 64
assert ctypes.sizeof(CopyJob) == 24
assert ctypes.sizeof(CheckJob) == 48
assert ctypes.sizeof(CheckResult) == 32

# name -> (restype, argtypes); every symbol include/tb200.h declares
SIGNATURES = {
    "tb200_dtype_size": (c_u32, [c_u32]),
    "tb200_dtype_from_name": (c_u32, [ctypes.c_char_p]),
    "tb200_dtype_name": (ctypes.c_char_p, [c_u32]),
    "tb200_abi_version": (c_int, []),
    "tb200_last_error": (ctypes.c_char_p, []),
    "tb200_device_count": (c_int, [ctypes.POINTER(c_int)]),
    "tb200_ctx_create": (c_int, [c_int, ctypes.POINTER(c_vp)]),
    "tb200_ctx_destroy": (c_int, [c_vp]),
    "tb200_ctx_set_stream": (c_int, [c_vp, c_vp]),
    "tb200_ctx_stream": (c_vp, [c_vp]),
    "tb200_ctx_device": (c_int, [c_vp]),
    "tb200_ctx_sync": (c_int, [c_vp]),
    "tb200_ctx_fork": (c_int, [c_vp]),
    "tb200_ctx_join": (c_int, [c_vp]),
    "tb200_ctx_select": (c_int, [c_vp, c_int]),
    "tb200_ctx_launch_count": (c_u64, [c_vp]),
    "tb200_ctx_sm_count": (c_int, [c_vp]),
    "tb200_timer_create": (c_int, [c_vp, ctypes.POINTER(c_vp)]),
    "tb200_timer_start": (c_int, [c_vp]),
    "tb200_timer_stop": (c_int, [c_vp]),
    "tb200_timer_elapsed_ms": (c_int, [c_vp, ctypes.POINTER(ctypes.c_float)]),
    "tb200_timer_destroy": (c_int, [c_vp]),
    "tb200_region_create": (c_int, [ctypes.c_char_p, c_u64, c_int, ctypes.POINTER(c_vp)]),
    "tb200_region_open": (c_int, [c_u8p, c_u64, c_int, ctypes.POINTER(c_vp)]),
    "tb200_region_destroy": (c_int, [c_vp]),
    "tb200_region_ipc_handle": (c_int, [c_vp, c_u8p]),
    "tb200_region_base": (c_u64, [c_vp]),
    "tb200_region_size": (c_u64, [c_vp]),
    "tb200_region_device": (c_int, [c_vp]),
    "tb200_region_name": (ctypes.c_char_p, [c_vp]),
    "tb200_region_write_host": (c_int, [c_vp, c_vp, c_u64, c_vp, c_u64]),
    "tb200_region_write_host_gather": (c_int, [c_vp, c_vp, c_u64, c_int, ctypes.POINTER(c_vp), ctypes.POINTER(c_u64)]),
    "tb200_region_read_host": (c_int, [c_vp, c_vp, c_u64, c_vp, c_u64]),
    "tb200_region_write_ptr": (c_int, [c_vp, c_vp, c_u64, c_vp, c_u64]),
    "tb200_host_alloc": (c_int, [c_u64, ctypes.POINTER(c_vp), ctypes.POINTER(c_vp)]),
    "tb200_host_free": (c_int, [c_vp]),
    "tb200_device_alloc": (c_int, [c_int, c_u64, ctypes.POINTER(c_vp)]),
    "tb200_device_free": (c_int, [c_int, c_vp]),
    "tb200_memcpy_h2d_async": (c_int, [c_vp, c_vp, c_vp, c_u64]),
    "tb200_memcpy_d2h_async": (c_int, [c_vp, c_vp, c_vp, c_u64]),
    "tb200_fill_async": (c_int, [c_vp, ctypes.POINTER(FillJob), c_int, c_u64, c_u64]),
    "tb200_fill_epoch_async": (c_int, [c_vp, ctypes.POINTER(FillJob), c_int, c_u64, c_u64]),
    "tb200_pack_image_async": (c_int, [c_vp, c_vp, c_u32, c_u32, c_vp, c_int, c_int, c_int, c_int, c_u32]),
    "tb200_resize_pack_image_async": (c_int, [c_vp, c_vp, c_u32, c_u32, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_u32]),
    "tb200_cast_async": (c_int, [c_vp, c_vp, c_u32, c_vp, c_u32, c_u64]),
    "tb200_pack_strided_async": (c_int, [c_vp, c_vp, c_vp, c_u32, c_int, ctypes.POINTER(c_i64), ctypes.POINTER(c_i64)]),
    "tb200_concat_async": (c_int, [c_vp, ctypes.POINTER(CopyJob), c_int]),
    "tb200_check_async": (c_int, [c_vp, ctypes.POINTER(CheckJob), c_int, c_vp]),
    "tb200_deflate_bound": (c_u64, [c_u64]),
    "tb200_deflate_async": (c_int, [c_vp, c_vp, c_u64, c_vp, c_u64, c_u32, c_vp]),
    "tb200_topk_async": (c_int, [c_vp, ctypes.POINTER(TopkJob), c_int, c_int, c_vp]),
    "tb200_bytes_decode_async": (c_int, [c_vp, c_vp, c_u64, c_u64, c_vp, c_vp, c_u64, c_vp]),
    "tb200_graph_begin": (c_int, [c_vp]),
    "tb200_graph_end": (c_int, [c_vp, ctypes.POINTER(c_vp)]),
    "tb200_graph_launch": (c_int, [c_vp, c_vp]),
    "tb200_graph_destroy": (c_int, [c_vp]),
    "tb200_ctx_epoch_set": (c_int, [c_vp, c_u64]),
    "tb200_ctx_epoch_bump_async": (c_int, [c_vp, c_u64]),
    "tb200_l2_flush_async": (c_int, [c_vp]),
    "tb200_tune": (c_int, [ctypes.c_char_p, c_int]),
    "tb200_step_sync": (c_int, [c_vp, ctypes.POINTER(FillJob), c_int, c_u64, c_u64, ctypes.POINTER(CheckJob), c_int, c_vp]),
    "tb200_step_submit": (c_int, [c_vp, ctypes.POINTER(FillJob), c_int, c_u64, c_u64, ctypes.POINTER(CheckJob), c_int, c_vp, ctypes.POINTER(c_u64)]),
    "tb200_step_wait": (c_int, [c_vp, c_u64]),
}

_lib = None
_lock = threading.Lock()


class NativeError(RuntimeError):
    """A libtb200 call failed; ``code`` is the tb200_status, message from
    tb200_last_error()."""

    def __init__(self, code, message):
        super().__init__("[tb200 %d] %s" % (code, message))
        self.code = code
        self.message = message


def load():
    """Load libtb200.so once and type every entry point."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "libtb200.so not found at %s -- build it with "
                "`python -m client_b200.build` (nvcc, sm_90a). client_b200 has no "
                "host fallback for its CUDA path." % LIB_PATH
            )
        lib = ctypes.CDLL(LIB_PATH)
        for name, (restype, argtypes) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the symbol is missing
            fn.restype = restype
            fn.argtypes = argtypes
        from . import _native_loadgen

        _native_loadgen.declare(lib)
        if lib.tb200_abi_version() != 1:
            raise RuntimeError("libtb200 ABI version mismatch")
        _lib = lib
    return _lib


def last_error():
    msg = load().tb200_last_error()
    return msg.decode("utf-8", "replace") if msg else ""


def check(rc):
    """Raise NativeError for a negative status."""
    if rc != 0:
        raise NativeError(rc, last_error())
    return rc


class Context:
    """tb200_ctx: one device, one stream, scratch. Not thread safe (like the
    reference's per-device global stream, cuda_shared_memory/__init__.py:57-70)."""

    def __init__(self, device_id=0):
        self._lib = load()
        h = c_vp()
        check(self._lib.tb200_ctx_create(int(device_id), ctypes.byref(h)))
        self._h = h
        self.device_id = int(device_id)

    @property
    def handle(self):
        return self._h

    def close(self):
        if getattr(self, "_h", None):
            self._lib.tb200_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sync(self):
        check(self._lib.tb200_ctx_sync(self._h))

    def set_stream(self, cuda_stream_ptr):
        check(self._lib.tb200_ctx_set_stream(self._h, c_vp(cuda_stream_ptr)))

    @property
    def launch_count(self):
        return int(self._lib.tb200_ctx_launch_count(self._h))

    @property
    def sm_count(self):
        return int(self._lib.tb200_ctx_sm_count(self._h))


class Timer:
    """CUDA-event stopwatch on a context's stream."""

    def __init__(self, ctx):
        self._lib = load()
        self._ctx = ctx
        h = c_vp()
        check(self._lib.tb200_timer_create(ctx.handle, ctypes.byref(h)))
        self._h = h

    def start(self):
        check(self._lib.tb200_timer_start(self._h))

    def stop(self):
        check(self._lib.tb200_timer_stop(self._h))

    def elapsed_ms(self):
        ms = ctypes.c_float()
        check(self._lib.tb200_timer_elapsed_ms(self._h, ctypes.byref(ms)))
        return float(ms.value)

    def close(self):
        if getattr(self, "_h", None):
            self._lib.tb200_timer_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_contexts = threading.local()


def default_context(device_id):
    """Per-thread context per device (the analogue of the reference's ``_dlpack_stream``
    dict, made thread-local so that the module-level shared memory functions can be
    called from several threads)."""
    table = getattr(_contexts, "table", None)
    if table is None:
        table = _contexts.table = {}
    ctx = table.get(device_id)
    if ctx is None:
        ctx = Context(device_id)
        table[device_id] = ctx
    return ctx
