"""The C-ABI library loads and exports every symbol include/*.h declares; the
ctypes mirrors of the job structs have the documented sizes.  No compute calls
(those are the -m gpu tests)."""

import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared(header):
    text = open(os.path.join(ROOT, "include", header)).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(tb200_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    from client_b200 import _native

    lib = _native.load()
    names = _declared("tb200.h")
    assert len(names) >= 45
    for n in names:
        assert hasattr(lib, n), "libtb200.so does not export %s" % n
        assert n in _native.SIGNATURES, "no ctypes signature for %s" % n
    if os.path.exists(os.path.join(ROOT, "include", "tb200_loadgen.h")):
        for n in _declared("tb200_loadgen.h"):
            assert hasattr(lib, n), "libtb200.so does not export %s" % n
    assert lib.tb200_abi_version() == 1


def test_struct_sizes_and_dtype_table():
    from client_b200 import _native

    lib = _native.load()
    assert ctypes.sizeof(_native.FillJob) == 64 and ctypes.sizeof(_native.CheckJob) == 48
    assert ctypes.sizeof(_native.CheckResult) == 32 and ctypes.sizeof(_native.CopyJob) == 24
    for name, code in _native.DTYPE_CODES.items():
        assert lib.tb200_dtype_from_name(name.encode()) == code
        assert lib.tb200_dtype_name(code).decode() == name
        assert lib.tb200_dtype_size(code) == _native.DTYPE_SIZES.get(name, 0)
    assert lib.tb200_dtype_from_name(b"FP8") == 0


def test_no_gpu_means_loud_failure_not_fallback():
    """Without a CUDA device every device entry point fails with an error message."""
    from client_b200 import _native

    lib = _native.load()
    n = ctypes.c_int(-1)
    rc = lib.tb200_device_count(ctypes.byref(n))
    if rc == 0 and n.value > 0:
        pytest.skip("a GPU is present")
    h = ctypes.c_void_p()
    assert lib.tb200_ctx_create(0, ctypes.byref(h)) < 0 and _native.last_error()
    with pytest.raises(Exception):
        import client_b200.utils.cuda_shared_memory as cudashm

        cudashm.create_shared_memory_region("x", 64, 0)


def test_sass_has_tma_bulk_copy_and_wide_stores():
    """Evidence the kernels are what DESIGN.md says: UBLKCP (cp.async.bulk), 128-bit
    global stores, IMAD.WIDE Philox rounds."""
    from client_b200 import _native

    try:
        sass = subprocess.run(["cuobjdump", "-sass", _native.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    except (FileNotFoundError, subprocess.TimeoutExpired):
        pytest.skip("cuobjdump not available")
    assert "UBLKCP" in sass and "STG.E.EF.128" in sass and "IMAD.WIDE.U32" in sass
    assert "sm_90a" in subprocess.run(["cuobjdump", "-lelf", _native.LIB_PATH], capture_output=True, text=True).stdout


def test_device_compression_has_no_host_fallback():
    """http.set_device_compression(True) on a machine without a GPU: the compressed request
    raises instead of silently using zlib."""
    import numpy as np
    import pytest

    import client_b200.http as httpclient
    from client_b200 import _native

    try:
        _native.default_context(0)
        pytest.skip("a CUDA device is present")
    except _native.NativeError:
        pass
    httpclient.set_device_compression(True)
    try:
        client = httpclient.InferenceServerClient("127.0.0.1:1")
        inp = httpclient.InferInput("X", [4], "INT32").set_data_from_numpy(np.arange(4, dtype=np.int32))
        with pytest.raises(_native.NativeError):
            client.infer("m", [inp], request_compression_algorithm="gzip")
    finally:
        httpclient.set_device_compression(False)
