"""Driver of the native load generator (include/tb200_loadgen.h): builds the per-slot
requests with the drop-in request model (HTTP/1.1 text, or ModelInferRequest bytes for the
gRPC-over-HTTP/2 transport), hands them plus the device job tables to libtb200 and reads back
windowed statistics.  Synchronous closed loop."""

import ctypes

from .. import _native
from .._native_loadgen import LoadgenConfig, LoadgenStats
from ..http import InferenceServerClient, InferInput, InferRequestedOutput


def frame_http_request(host, port, uri, body, json_size, head_only_bytes=None):
    """A complete HTTP/1.1 POST.  ``head_only_bytes``: when given, ``body`` holds only the
    JSON header and that many tensor bytes follow from the pinned tail."""
    total = len(body) + (head_only_bytes or 0)
    lines = ["POST /%s HTTP/1.1" % uri.lstrip("/"), "Host: %s:%d" % (host, port), "Content-Length: %d" % total]
    if json_size is not None:
        lines.append("Inference-Header-Content-Length: %d" % json_size)
        lines.append("Content-Type: application/octet-stream")
    else:
        lines.append("Content-Type: application/json")
    return ("\r\n".join(lines) + "\r\n\r\n").encode("ascii") + body


def _varint(n):
    out = bytearray()
    while n >= 0x80:
        out.append((n & 0x7F) | 0x80)
        n >>= 7
    out.append(n)
    return bytes(out)


def grpc_wire_prefixes(inputs):
    """What precedes each tensor inside a serialised ModelInferRequest: the tag of
    ``raw_input_contents`` (field 7, length-delimited: 0x3A) and the byte length.  Passed to
    SlotSet(wire_prefixes=...) so that a slot's staging image is the tail of the message."""
    return [b"\x3a" + _varint(t.nbytes) for t in inputs]


class NativeLoadGenerator:
    """One tb200_loadgen instance over a SlotSet (cuda shm or wire mode)."""

    def __init__(self, url, model_name, model_version, slotset, concurrency, regenerate=True, validate=True,
                 device_window_us=0, protocol="http", request_parameters=None, pipeline_depth=3):
        """``protocol``: "http" (HTTP/1.1), "grpc" (unary ModelInfer) or "grpc-stream" (one
        ModelStreamInfer stream per connection; windows then report ``ttft_p50_us`` and
        ``responses``).  ``pipeline_depth``: device passes in flight (1 = one at a time)."""
        self._lib = _native.load()
        self.protocol = protocol
        self.request_parameters = request_parameters
        host, _, port = url.partition(":")
        self.host, self.port = host, int(port or 80)
        ss = slotset
        self.slotset = ss
        uri = InferenceServerClient._model_uri(model_name, model_version, "/infer")
        self._keep = []
        reqs, tails = [], []
        grpc_like = protocol in ("grpc", "grpc-stream")
        if grpc_like:
            reqs, tails = self._grpc_requests(model_name, model_version, ss, concurrency, request_parameters)
        # requests that name shared-memory offsets exist once per staging image of a slot
        self._rps = ss.lookahead if ss.shared_memory == "cuda" else 1
        for slot, gen in ((s, g) for s in range(0 if grpc_like else concurrency) for g in range(self._rps)):
            inputs, outputs = [], []
            for i, t in enumerate(ss.inputs):
                inp = InferInput(t.name, t.shape, t.datatype)
                if ss.shared_memory in ("cuda", "system"):
                    inp.set_shared_memory(ss.prefix + "_in", t.nbytes, offset=ss.input_offset(slot, i, gen))
                else:
                    inp._parameters["binary_data_size"] = t.nbytes  # bytes follow from the pinned tail
                    inp._raw_data = b""
                inputs.append(inp)
            for i, t in enumerate(ss.outputs):
                out = InferRequestedOutput(t.name)
                if ss.shared_memory in ("cuda", "system"):
                    out.set_shared_memory(ss.prefix + "_out", t.nbytes, offset=ss.output_offset(slot, i, gen))
                outputs.append(out)
            body, json_size = InferenceServerClient.generate_request_body(inputs, outputs=outputs, parameters=request_parameters)
            if ss.shared_memory == "none":
                json_size = len(body)
                reqs.append(frame_http_request(self.host, self.port, uri, body, json_size, head_only_bytes=ss.in_bytes))
                tails.append((ss._wire.host_ptr + slot * ss.lookahead * ss.wire_stride, ss.wire_stride))
            else:
                reqs.append(frame_http_request(self.host, self.port, uri, body, json_size))
        n = concurrency
        bufs = [ctypes.create_string_buffer(r, len(r)) for r in reqs]
        self._keep.append(bufs)
        cfg = LoadgenConfig()
        cfg.host = self.host.encode("ascii")
        cfg.port = self.port
        cfg.concurrency = n
        cfg.requests_per_slot = self._rps
        assert len(reqs) == n * self._rps
        cfg.requests = (ctypes.c_void_p * len(reqs))(*[ctypes.addressof(b) for b in bufs])
        cfg.request_sizes = (ctypes.c_uint64 * len(reqs))(*[len(r) for r in reqs])
        if tails:
            cfg.tails = (ctypes.c_void_p * n)(*[p for p, _ in tails])
            cfg.tail_sizes = (ctypes.c_uint64 * n)(*[s for _, s in tails])
        if ss._ops is not None:
            cfg.ctx = ss._ops.ctx.handle
            per = len(ss.inputs) * ss.lookahead
            if ss.replay is not None:
                # replayed entries: templates at entry 0, the device thread adds entry * tensor size
                copies = ss._copy_jobs(list(range(n)), at_entry=0)
                cfg.replay_entries = ss.replay.entries
                cfg.copy_jobs = (_native.CopyJob * len(copies))(*copies)
                cfg.copy_jobs_per_slot = per
                cfg.copy_src_stride = (ctypes.c_uint64 * per)(*[t.nbytes for _ in range(ss.lookahead) for t in ss.inputs])
            else:
                fills = ss._fill_jobs(list(range(n)))
                cfg.fill_jobs = (_native.FillJob * len(fills))(*fills)
                cfg.fill_jobs_per_slot = per
            cfg.seed = ss.seed
            cfg.regenerate = 1 if regenerate else 0
            if validate and ss.shared_memory == "cuda" and ss.outputs:
                from ..device import HostBuffer

                checks = ss._check_jobs(list(range(n)), at_entry=0)
                self._results = HostBuffer(len(checks) * 32)
                cfg.check_jobs = (_native.CheckJob * len(checks))(*checks)
                cfg.check_jobs_per_slot = len(ss.outputs) * ss.lookahead
                cfg.results = self._results.device_ptr
                if ss.replay is not None:
                    strides = [t.nbytes if t.name in ss.replay.expected else 0 for _ in range(ss.lookahead) for t in ss.outputs]
                    cfg.check_b_stride = (ctypes.c_uint64 * len(strides))(*strides)
        cfg.device_window_us = int(device_window_us)
        cfg.lookahead = ss.lookahead
        cfg.tail_stride = ss.wire_stride
        cfg.protocol = {"http": 0, "grpc": 1, "grpc-stream": 2}[protocol]
        cfg.pipeline_depth = int(pipeline_depth)
        self._keep.append(cfg)
        h = ctypes.c_void_p()
        _native.check(self._lib.tb200_loadgen_create(ctypes.byref(cfg), ctypes.byref(h)))
        self._h = h

    @staticmethod
    def _grpc_requests(model_name, model_version, ss, concurrency, request_parameters=None):
        """Per slot: ModelInferRequest bytes up to (not including) raw_input_contents; in wire
        mode the rest of the message is the slot's staging image (tag + length + tensor per
        input), which must have been laid out with grpc_wire_prefixes()."""
        from .. import grpc as grpcclient
        from ..grpc._utils import _get_inference_request

        reqs, tails = [], []
        rps = ss.lookahead if ss.shared_memory == "cuda" else 1
        for slot, gen in ((s, g) for s in range(concurrency) for g in range(rps)):
            inputs, outputs = [], []
            for i, t in enumerate(ss.inputs):
                inp = grpcclient.InferInput(t.name, t.shape, t.datatype)
                if ss.shared_memory in ("cuda", "system"):
                    inp.set_shared_memory(ss.prefix + "_in", t.nbytes, offset=ss.input_offset(slot, i, gen))
                inputs.append(inp)
            for i, t in enumerate(ss.outputs):
                out = grpcclient.InferRequestedOutput(t.name)
                if ss.shared_memory in ("cuda", "system"):
                    out.set_shared_memory(ss.prefix + "_out", t.nbytes, offset=ss.output_offset(slot, i, gen))
                outputs.append(out)
            request = _get_inference_request(model_name=model_name, inputs=inputs, model_version=model_version, request_id="",
                                             outputs=outputs, sequence_id=0, sequence_start=False, sequence_end=False,
                                             priority=0, timeout=None, parameters=request_parameters)
            reqs.append(request.SerializeToString())
            if ss.shared_memory == "none":
                if ss.wire_stride == ss.in_bytes and ss.in_bytes:
                    raise ValueError("the SlotSet of a gRPC wire-mode run needs wire_prefixes=grpc_wire_prefixes(inputs)")
                tails.append((ss._wire.host_ptr + slot * ss.lookahead * ss.wire_stride, ss.wire_stride))
        return reqs, tails

    def start(self):
        _native.check(self._lib.tb200_loadgen_start(self._h))

    def window(self, seconds):
        st = LoadgenStats()
        _native.check(self._lib.tb200_loadgen_window(self._h, float(seconds), ctypes.byref(st)))
        n = st.completed_request_count
        return {
            "count": int(n), "failed": int(st.failed_request_count), "seconds": st.window_seconds,
            "throughput": n / st.window_seconds if st.window_seconds > 0 else 0.0,
            "avg_us": st.cumulative_total_request_time_ns / n / 1e3 if n else 0.0,
            "send_us": st.cumulative_send_time_ns / n / 1e3 if n else 0.0,
            "recv_us": st.cumulative_receive_time_ns / n / 1e3 if n else 0.0,
            "p50_us": st.p50_ns / 1e3, "p90_us": st.p90_ns / 1e3, "p95_us": st.p95_ns / 1e3, "p99_us": st.p99_ns / 1e3,
            "min_us": st.min_ns / 1e3, "max_us": st.max_ns / 1e3,
            "device_batches": int(st.device_batches), "device_slots": int(st.device_slots),
            "nonfinite": int(st.nonfinite_outputs), "mismatches": int(st.check_mismatches),
            **({"responses": int(st.response_count), "responses_per_s": st.response_count / st.window_seconds if st.window_seconds > 0 else 0.0,
                "ttft_p50_us": st.first_response_p50_ns / 1e3, "ttft_p99_us": st.first_response_p99_ns / 1e3}
               if self.protocol == "grpc-stream" else {}),
        }

    def wait_count(self, count, timeout=60.0):
        """Block until ``count`` requests finished since the last window() (count windows)."""
        got = ctypes.c_uint64(0)
        _native.check(self._lib.tb200_loadgen_wait_count(self._h, int(count), float(timeout), ctypes.byref(got)))
        return int(got.value)

    def stop(self):
        if getattr(self, "_h", None):
            self._lib.tb200_loadgen_stop(self._h)
            self._lib.tb200_loadgen_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.stop()
        except Exception:
            pass


class GrpcStubServer:
    """tb200_grpc_stub_server: every unary call answered with one canned message; with
    ``final_response`` given (stream mode, ModelStreamInfer) every request MESSAGE on a stream is
    answered with ``responses_per_request - 1`` x ``response`` and one ``final_response``."""

    def __init__(self, response=b"", host="127.0.0.1", port=0, final_response=None, responses_per_request=1):
        self._lib = _native.load()
        p = ctypes.c_int(port)
        h = ctypes.c_void_p()
        buf = ctypes.create_string_buffer(response, max(len(response), 1))
        if final_response is not None:
            fin = ctypes.create_string_buffer(final_response, max(len(final_response), 1))
            _native.check(self._lib.tb200_grpc_stub_server_start_streaming(host.encode(), ctypes.byref(p), buf, len(response), fin,
                                                                           len(final_response), int(responses_per_request), ctypes.byref(h)))
        else:
            _native.check(self._lib.tb200_grpc_stub_server_start(host.encode(), ctypes.byref(p), buf, len(response), ctypes.byref(h)))
        self._h, self.host, self.port = h, host, p.value

    @property
    def url(self):
        return "%s:%d" % (self.host, self.port)

    def stop(self):
        if getattr(self, "_h", None):
            self._lib.tb200_grpc_stub_server_stop(self._h)
            self._h = None


class GrpcEchoServer:
    """tb200_grpc_echo_server (csrc/grpc_server.h): answers every call with its own request."""

    def __init__(self, host="127.0.0.1", port=0):
        self._lib = _native.load()
        p = ctypes.c_int(port)
        h = ctypes.c_void_p()
        _native.check(self._lib.tb200_grpc_echo_server_start(host.encode(), ctypes.byref(p), ctypes.byref(h)))
        self._h, self.host, self.port = h, host, p.value

    @property
    def url(self):
        return "%s:%d" % (self.host, self.port)

    def stop(self):
        if getattr(self, "_h", None):
            self._lib.tb200_grpc_echo_server_stop(self._h)
            self._h = None


def stream_token_responses(output_name="token", token=7):
    """(response, final_response) for GrpcStubServer's stream mode: ModelStreamInferResponse
    messages carrying one INT32[1,1] token, the last one flagged triton_final_response."""
    import numpy as np

    from ..grpc import service_pb2

    out = []
    for final in (False, True):
        m = service_pb2.ModelStreamInferResponse()
        r = m.infer_response
        r.model_name = "stub"
        r.parameters["triton_final_response"].bool_param = final
        o = r.outputs.add()
        o.name, o.datatype = output_name, "INT32"
        o.shape.extend([1, 1])
        r.raw_output_contents.append(np.array([[token]], np.int32).tobytes())
        out.append(m.SerializeToString())
    return tuple(out)


class StubServer:
    """tb200_stub_server: canned 200 responses, for measuring the generator itself."""

    def __init__(self, body='{"model_name":"stub","outputs":[]}', host="127.0.0.1", port=0):
        self._lib = _native.load()
        p = ctypes.c_int(port)
        h = ctypes.c_void_p()
        _native.check(self._lib.tb200_stub_server_start(host.encode(), ctypes.byref(p), body.encode(), ctypes.byref(h)))
        self._h, self.host, self.port = h, host, p.value

    @property
    def url(self):
        return "%s:%d" % (self.host, self.port)

    def stop(self):
        if getattr(self, "_h", None):
            self._lib.tb200_stub_server_stop(self._h)
            self._h = None
