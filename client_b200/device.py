"""Python face of the libtb200 kernels: job builders and thin launch wrappers.

Everything here is plumbing over the C ABI (include/tb200.h): argument
marshalling into the job structs, buffer lifetimes, error translation.  No
tensor arithmetic happens in Python.
"""

import ctypes

import numpy as np

from . import _native
from ._native import CheckJob, CheckResult, CopyJob, FillJob

_FLOAT_TYPES = ("FP16", "FP32", "FP64", "BF16")
_KINDS = {"sum": _native.CHECK_SUM, "equal": _native.CHECK_EQUAL,
          "addsub": _native.CHECK_ADDSUB, "top1": _native.CHECK_TOP1}


def make_fill_job(dst, nbytes, datatype, stream_id=0, mode="random", low=0.0, high=None, string_length=None):
    """Build a tb200_fill_job.

    Floats: uniform in [low, high); ``high=None`` -> the unit interval (``low``
    must be 0).  Integers: uniform in [low, high); ``high=None`` -> raw bits.
    ``mode`` "zero" writes zeros, "byte" writes ``low`` as a repeated byte.
    BYTES: ``string_length`` random alphanumeric characters per element in the
    serialised ``<u32 length><chars>`` form; nbytes = count * (4 + string_length).
    """
    code = _native.DTYPE_CODES.get(datatype)
    if code is None or (datatype == "BYTES" and (string_length is None or mode != "random")):
        raise ValueError("datatype '%s' cannot be generated" % datatype)
    job = FillJob()
    job.dst = int(dst)
    job.nbytes = int(nbytes)
    job.stream = int(stream_id) & 0xFFFFFFFFFFFFFFFF
    job.dtype = code
    if datatype == "BYTES":
        if int(nbytes) % (4 + int(string_length)) != 0:
            raise ValueError("nbytes must be count * (4 + string_length)")
        job.mode = _native.FILL_RANDOM
        job.irange = int(string_length)
        return job
    if mode == "zero":
        job.mode = _native.FILL_ZERO
        return job
    if mode == "byte":
        job.mode = _native.FILL_BYTE
        job.ilo = int(low)
        return job
    if mode != "random":
        raise ValueError("unknown fill mode '%s'" % mode)
    job.mode = _native.FILL_RANDOM
    if datatype in _FLOAT_TYPES:
        if high is None:
            if float(low) != 0.0:
                raise ValueError("low must be 0 for the unit interval; pass high as well")
            job.lo, job.span = 0.0, 0.0
        else:
            span = float(high) - float(low)
            if not span > 0.0:
                raise ValueError("high must be greater than low")
            job.lo, job.span = float(low), span
    elif datatype != "BOOL":
        if high is None:
            job.ilo, job.irange = 0, 0
        else:
            rng = int(high) - int(low)
            if rng <= 0:
                raise ValueError("high must be greater than low")
            job.ilo, job.irange = int(low), rng
    return job


class HostBuffer:
    """Pinned, device-mapped host memory (tb200_host_alloc): where the kernels
    emit HTTP binary bodies / gRPC raw_input_contents and small results."""

    def __init__(self, nbytes):
        self._lib = _native.load()
        hp, dp = ctypes.c_void_p(), ctypes.c_void_p()
        _native.check(self._lib.tb200_host_alloc(int(nbytes), ctypes.byref(hp), ctypes.byref(dp)))
        self.nbytes = int(nbytes)
        self.host_ptr = hp.value
        self.device_ptr = dp.value
        self._ctype = (ctypes.c_uint8 * max(self.nbytes, 1)).from_address(self.host_ptr)

    def array(self, dtype=np.uint8, count=None, offset=0):
        """numpy view (no copy) over the pinned bytes."""
        dt = np.dtype(dtype)
        n = (self.nbytes - offset) // dt.itemsize if count is None else count
        return np.frombuffer(self._ctype, dtype=dt, count=n, offset=offset)

    def view(self, offset=0, nbytes=None):
        end = self.nbytes if nbytes is None else offset + nbytes
        return memoryview(self._ctype).cast("B")[offset:end]

    def close(self):
        if getattr(self, "host_ptr", None):
            self._ctype = None
            self._lib.tb200_host_free(ctypes.c_void_p(self.host_ptr))
            self.host_ptr = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DeviceBuffer:
    """Plain device memory owned by the caller (tb200_device_alloc)."""

    def __init__(self, device_id, nbytes):
        self._lib = _native.load()
        p = ctypes.c_void_p()
        _native.check(self._lib.tb200_device_alloc(int(device_id), int(nbytes), ctypes.byref(p)))
        self.ptr = p.value
        self.nbytes = int(nbytes)
        self.device_id = int(device_id)

    def close(self):
        if getattr(self, "ptr", None):
            self._lib.tb200_device_free(self.device_id, ctypes.c_void_p(self.ptr))
            self.ptr = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Graph:
    """A captured sequence of libtb200 launches (tb200_graph)."""

    def __init__(self, ops, handle):
        self._ops = ops
        self._h = handle

    def launch(self):
        _native.check(self._ops._lib.tb200_graph_launch(self._ops._ctx.handle, self._h))

    def close(self):
        if getattr(self, "_h", None):
            self._ops._lib.tb200_graph_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DeviceOps:
    """Launch wrappers bound to one context (device + stream)."""

    def __init__(self, ctx=None, device_id=0):
        self._lib = _native.load()
        self._ctx = ctx if ctx is not None else _native.default_context(device_id)
        self._ticket = ctypes.c_uint64(0)
        self._ticket_ref = ctypes.byref(self._ticket)

    @property
    def ctx(self):
        return self._ctx

    @property
    def device_id(self):
        return self._ctx.device_id

    def sync(self):
        self._ctx.sync()

    # -- raw copies -------------------------------------------------------------
    def h2d(self, dst_ptr, src_host_ptr, nbytes):
        _native.check(self._lib.tb200_memcpy_h2d_async(self._ctx.handle, dst_ptr, src_host_ptr, int(nbytes)))

    def d2h(self, dst_host_ptr, src_ptr, nbytes):
        _native.check(self._lib.tb200_memcpy_d2h_async(self._ctx.handle, dst_host_ptr, src_ptr, int(nbytes)))

    def upload(self, array):
        """Blocking convenience: numpy array -> new DeviceBuffer."""
        arr = np.ascontiguousarray(array)
        buf = DeviceBuffer(self.device_id, max(arr.nbytes, 16))
        if arr.nbytes:
            self.h2d(buf.ptr, arr.ctypes.data, arr.nbytes)
            self.sync()
        return buf

    def download(self, ptr, nbytes, dtype=np.uint8):
        """Blocking convenience: device bytes -> numpy array."""
        out = np.empty(int(nbytes), dtype=np.uint8)
        if nbytes:
            self.d2h(out.ctypes.data, ptr, nbytes)
            self.sync()
        return out.view(dtype)

    # -- kernels ------------------------------------------------------------------
    @staticmethod
    def job_array(jobs, ctype):
        if isinstance(jobs, ctypes.Array):
            return jobs, len(jobs)
        arr = (ctype * max(len(jobs), 1))(*jobs)
        return arr, len(jobs)

    def fill(self, jobs, seed=0, epoch=0):
        arr, n = self.job_array(jobs, FillJob)
        _native.check(self._lib.tb200_fill_async(self._ctx.handle, arr, n, int(seed), int(epoch)))

    def fill_epoch(self, jobs, seed=0, bump=0):
        """Fill with the device epoch added to every stream id; ``bump`` advances the
        epoch inside the same kernel (graph replays then never repeat data)."""
        arr, n = self.job_array(jobs, FillJob)
        _native.check(self._lib.tb200_fill_epoch_async(self._ctx.handle, arr, n, int(seed), int(bump)))

    def fork(self):
        """Later launches run on a side stream, concurrently with the main stream."""
        _native.check(self._lib.tb200_ctx_fork(self._ctx.handle))

    def select(self, side):
        """While forked: route the following launches to the main (False) or side (True) stream."""
        _native.check(self._lib.tb200_ctx_select(self._ctx.handle, 1 if side else 0))

    def join(self):
        _native.check(self._lib.tb200_ctx_join(self._ctx.handle))

    def epoch_set(self, value):
        _native.check(self._lib.tb200_ctx_epoch_set(self._ctx.handle, int(value)))

    def epoch_bump(self, delta=1):
        _native.check(self._lib.tb200_ctx_epoch_bump_async(self._ctx.handle, int(delta)))

    def pack_image(self, dst_ptr, datatype, layout, src_ptr, n, h, w, c, scaling="NONE"):
        _native.check(
            self._lib.tb200_pack_image_async(
                self._ctx.handle, dst_ptr, _native.DTYPE_CODES[datatype],
                _native.NCHW if layout == "NCHW" else _native.NHWC,
                src_ptr, int(n), int(h), int(w), int(c), _native.SCALING_CODES[scaling],
            )
        )

    def pack_image_from_host(self, dst_ptr, datatype, layout, images_u8_nhwc, scaling="NONE"):
        """Stage uint8 NHWC host images on the device, then pack into dst."""
        arr = np.ascontiguousarray(images_u8_nhwc, dtype=np.uint8)
        n, h, w, c = arr.shape
        staging = self._scratch(arr.nbytes)
        self.h2d(staging.ptr, arr.ctypes.data, arr.nbytes)
        self.pack_image(dst_ptr, datatype, layout, staging.ptr, n, h, w, c, scaling)
        self.sync()  # arr must stay alive until the H2D completed

    def resize_pack_image(self, dst_ptr, datatype, layout, src_ptr, n, src_h, src_w, c, dst_h, dst_w, scaling="NONE"):
        """Image.resize((dst_w, dst_h), BILINEAR) + astype + scaling + layout in one launch."""
        _native.check(
            self._lib.tb200_resize_pack_image_async(
                self._ctx.handle, dst_ptr, _native.DTYPE_CODES[datatype],
                _native.NCHW if layout == "NCHW" else _native.NHWC,
                src_ptr, int(n), int(src_h), int(src_w), int(c), int(dst_h), int(dst_w), _native.SCALING_CODES[scaling],
            )
        )

    def resize_pack_image_from_host(self, dst_ptr, datatype, layout, images_u8_nhwc, dst_h, dst_w, scaling="NONE"):
        arr = np.ascontiguousarray(images_u8_nhwc, dtype=np.uint8)
        n, h, w, c = arr.shape
        staging = self._scratch(arr.nbytes)
        self.h2d(staging.ptr, arr.ctypes.data, arr.nbytes)
        self.resize_pack_image(dst_ptr, datatype, layout, staging.ptr, n, h, w, c, dst_h, dst_w, scaling)
        self.sync()  # arr must stay alive until the H2D completed

    def _scratch(self, nbytes):
        cur = getattr(self, "_scratch_buf", None)
        if cur is None or cur.nbytes < nbytes:
            self.sync()
            self._scratch_buf = DeviceBuffer(self.device_id, max(int(nbytes), 1 << 20))
        return self._scratch_buf

    def cast(self, dst_ptr, dst_type, src_ptr, src_type, nelem):
        _native.check(
            self._lib.tb200_cast_async(
                self._ctx.handle, dst_ptr, _native.DTYPE_CODES[dst_type], src_ptr,
                _native.DTYPE_CODES[src_type], int(nelem),
            )
        )

    def pack_strided(self, dst_ptr, src_ptr, elem_size, shape, strides_bytes):
        nd = len(shape)
        c_shape = (ctypes.c_int64 * max(nd, 1))(*[int(s) for s in shape])
        c_strides = (ctypes.c_int64 * max(nd, 1))(*[int(s) for s in strides_bytes])
        _native.check(
            self._lib.tb200_pack_strided_async(
                self._ctx.handle, dst_ptr, src_ptr, int(elem_size), nd, c_shape, c_strides
            )
        )

    def concat(self, jobs):
        arr, n = self.job_array(jobs, CopyJob)
        _native.check(self._lib.tb200_concat_async(self._ctx.handle, arr, n))

    def check(self, jobs, results_ptr):
        arr, n = self.job_array(jobs, CheckJob)
        _native.check(self._lib.tb200_check_async(self._ctx.handle, arr, n, results_ptr))

    def check_one(self, kind, a, nbytes, b=0, c=0, d=0):
        """Blocking convenience: run one check job, return its result as a dict."""
        job = CheckJob(a=int(a), b=int(b), c=int(c), d=int(d), nbytes=int(nbytes), kind=_KINDS[kind], pad=0)
        res = self._result_buf()
        self.check([job], res.device_ptr)
        self.sync()
        return result_dict(res.array(np.uint8, ctypes.sizeof(CheckResult)).tobytes())

    def check_one_deferred(self, kind, a, nbytes, b=0, c=0, d=0):
        """Launch one check job and return a callable that waits for the stream and decodes the result --
        whatever else was queued on the stream in between (the next request's fill) shares that one wait.
        One deferred check at a time per DeviceOps (they share the pinned result slot)."""
        job = CheckJob(a=int(a), b=int(b), c=int(c), d=int(d), nbytes=int(nbytes), kind=_KINDS[kind], pad=0)
        res = self._result_buf()
        self.check([job], res.device_ptr)

        def result():
            self.sync()
            return result_dict(res.array(np.uint8, ctypes.sizeof(CheckResult)).tobytes())

        return result

    def bytes_decode(self, src_ptr, src_bytes, count):
        """Blocking on-device decode of a serialised BYTES tensor (tb200_bytes_decode_async):
        ``count`` elements of ``<u32 length><payload>`` starting at device address ``src_ptr``.
        Returns (offsets uint32[count + 1], packed payload bytes, consumed source bytes); only the
        offsets and the payloads cross PCIe.  Raises on a truncated or inconsistent stream."""
        count, src_bytes = int(count), int(src_bytes)
        need = 64 + (count + 1) * 4 + src_bytes  # status | offsets | packed (payloads <= source bytes)
        buf = getattr(self, "_bytes_buf", None)
        if buf is None or buf.nbytes < need:
            buf = self._bytes_buf = HostBuffer(max(need, 1 << 16))
        off_at = 64
        packed_at = (off_at + (count + 1) * 4 + 15) & ~15
        if buf.nbytes < packed_at + src_bytes:
            buf = self._bytes_buf = HostBuffer(packed_at + src_bytes)
        _native.check(self._lib.tb200_bytes_decode_async(self._ctx.handle, int(src_ptr), src_bytes, count, buf.device_ptr + off_at,
                                                        buf.device_ptr + packed_at, src_bytes, buf.device_ptr))
        self.sync()
        status = buf.array(np.uint64, 4)
        if int(status[3]) != 0:
            raise ValueError("serialised BYTES tensor is %s after %d of %d elements" % (
                {1: "truncated", 2: "inconsistent (a length runs past the buffer)", 3: "larger than 4 GiB"}.get(int(status[3]), "invalid"), int(status[0]), count))
        offsets = buf.array(np.uint32, count + 1, offset=off_at).copy()
        packed = buf.array(np.uint8, int(status[2]), offset=packed_at).tobytes()
        return offsets, packed, int(status[1])

    def topk(self, vectors, k):
        """Blocking top-k of device vectors (tb200_topk_async).

        vectors: [(device_address, element_count, "FP32" | "FP16" | "BF16"), ...];
        returns (values float32 [n, k], indices uint32 [n, k]); slots past a vector's
        length carry index 0xFFFFFFFF.  Only 8*k bytes per vector leave the device."""
        from ._native import TopkJob

        jobs = [TopkJob(src=int(a), count=int(n), dtype=_native.DTYPE_CODES[dt], pad=0) for a, n, dt in vectors]
        arr, n = self.job_array(jobs, TopkJob)
        k = int(k)
        need = max(1, n * k * 8)
        buf = getattr(self, "_topk_buf", None)
        if buf is None or buf.nbytes < need:
            buf = self._topk_buf = HostBuffer(max(need, 1 << 16))
        _native.check(self._lib.tb200_topk_async(self._ctx.handle, arr, n, k, buf.device_ptr))
        self.sync()
        ent = buf.array(np.dtype([("value", "<f4"), ("index", "<u4")]), n * k).reshape(n, k)
        return ent["value"].copy(), ent["index"].copy()

    def deflate_async(self, dst_ptr, dst_capacity, src_ptr, nbytes, out_size_ptr, algorithm="gzip"):
        """Compress device bytes into a zlib ("deflate") or gzip stream on the device
        (tb200_deflate_async); the stream length lands in ``*out_size_ptr`` (uint64)."""
        fmt = {"deflate": 0, "zlib": 0, "gzip": 1}[algorithm]
        _native.check(self._lib.tb200_deflate_async(self._ctx.handle, dst_ptr, int(dst_capacity), src_ptr, int(nbytes), fmt, out_size_ptr))

    def deflate(self, src_ptr, nbytes, algorithm="gzip"):
        """Blocking convenience: the compressed stream as ``bytes`` — what
        ``gzip.compress`` / ``zlib.compress`` produce for a request body
        (reference http/_client.py:1440-1460), decodable by the same decoders."""
        cap = int(self._lib.tb200_deflate_bound(int(nbytes)))
        dst = self._scratch2(cap)
        size = self._result_buf()
        self.deflate_async(dst.ptr, cap, src_ptr, nbytes, size.device_ptr + 2048, algorithm)
        self.sync()
        n = int(size.array(np.uint64, 1, offset=2048)[0])
        return self.download(dst.ptr, n).tobytes()

    def _scratch2(self, nbytes):
        cur = getattr(self, "_scratch2_buf", None)
        if cur is None or cur.nbytes < nbytes:
            self.sync()
            self._scratch2_buf = DeviceBuffer(self.device_id, max(int(nbytes), 1 << 20))
        return self._scratch2_buf

    def _result_buf(self):
        cur = getattr(self, "_res_buf", None)
        if cur is None:
            self._res_buf = HostBuffer(4096)
        return self._res_buf

    def step(self, fill_jobs, check_jobs, results_ptr, seed=0, epoch=0):
        """One closed-loop step (tb200_step_sync): generate inputs || validate outputs, wait."""
        fa, nf = self.job_array(fill_jobs, FillJob)
        ca, nc = self.job_array(check_jobs, CheckJob)
        _native.check(self._lib.tb200_step_sync(self._ctx.handle, fa, nf, int(seed), int(epoch), ca, nc, results_ptr))

    def step_submit(self, fill_jobs, check_jobs, results_ptr, seed=0, epoch=0):
        """The same step without the wait (tb200_step_submit): returns a ticket for step_wait().
        Up to 8 steps may be in flight; they must not share slots or result entries."""
        fa, nf = self.job_array(fill_jobs, FillJob)
        ca, nc = self.job_array(check_jobs, CheckJob)
        ticket = self._ticket  # one reusable out-parameter: this object is used by one thread (like the context)
        _native.check(self._lib.tb200_step_submit(self._ctx.handle, fa, nf, seed, epoch, ca, nc, results_ptr, self._ticket_ref))
        return ticket.value

    def step_submit_copy(self, copy_jobs, check_jobs, results_ptr):
        """step_submit with the inputs copied (tb200_step_submit_copy): the copy jobs run as one
        concat launch on the main stream, the checks on the side stream.  Returns a ticket for step_wait()."""
        ca, nc = self.job_array(copy_jobs, CopyJob)
        ka, nk = self.job_array(check_jobs, CheckJob)
        _native.check(self._lib.tb200_step_submit_copy(self._ctx.handle, ca, nc, ka, nk, results_ptr, self._ticket_ref))
        return self._ticket.value

    def step_wait(self, ticket):
        """Returns when the step's inputs are generated and its results are visible."""
        _native.check(self._lib.tb200_step_wait(self._ctx.handle, ticket))

    def l2_flush(self):
        _native.check(self._lib.tb200_l2_flush_async(self._ctx.handle))

    # -- graphs ---------------------------------------------------------------------
    def graph_begin(self):
        _native.check(self._lib.tb200_graph_begin(self._ctx.handle))

    def graph_end(self):
        h = ctypes.c_void_p()
        _native.check(self._lib.tb200_graph_end(self._ctx.handle, ctypes.byref(h)))
        return Graph(self, h)


def result_dict(raw):
    """Decode one tb200_check_result (32 bytes)."""
    r = CheckResult.from_buffer_copy(raw)
    return {
        "mismatches": int(r.mismatches),
        "sum": int(r.sum),
        "xor32": int(r.xor32),
        "argmax": int(r.argmax),
        "max_value": float(r.max_value),
    }


def results_array(host_buffer, count):
    """Structured numpy view over an array of tb200_check_result in pinned memory."""
    dt = np.dtype(
        [("mismatches", "<u8"), ("sum", "<u8"), ("xor32", "<u4"), ("argmax", "<u4"),
         ("max_value", "<f4"), ("pad", "<u4")]
    )
    return host_buffer.array(dt, count)
