"""Closed-loop load generation with device-side request data.

perf_analyzer's ConcurrencyManager / ConcurrencyWorker / data loader are NOT part of
the reference (SURVEY.md F1, row P); what is restated here is their publicly
documented behaviour: keep N requests in flight, synthetic (random / zero) inputs,
optional system / CUDA shared memory, measurement windows with a stability
criterion, percentile latency.  Parity with perf_analyzer itself is unpinned.

GPU-native part: every concurrency slot owns an input and an output region (CUDA
IPC, registered with the server).  A single device thread serves all slots: the
slots whose responses came back since the last pass are validated (``check_kernel``)
and regenerated (``fill_kernel``) with ONE launch each, then handed back to the
transport workers -- no numpy serialise and no host->device tensor copy sits on the
request path.  The per-request timestamps follow the reference's C++ RequestTimers
(src/c++/library/common.h:568-648).
"""

import queue
import threading
import time

import numpy as np

from .. import _native
from ..utils import InferenceServerException, deserialize_bytes_tensor, triton_to_np_dtype
from .input_data import InputDataError, replay_entry


class TensorSpec:
    """One model input / output.  BYTES tensors carry fixed-length strings
    (perf_analyzer's --string-length): 4 + string_length serialised bytes per element."""

    def __init__(self, name, datatype, shape, string_length=128):
        self.name, self.datatype, self.shape = name, datatype, [int(d) for d in shape]
        self.string_length = int(string_length) if datatype == "BYTES" else None
        es = 4 + self.string_length if datatype == "BYTES" else _native.DTYPE_SIZES.get(datatype)
        if es is None:
            raise ValueError("tensor '%s': datatype %s is not supported by the load generator" % (name, datatype))
        self.nbytes = int(np.prod(self.shape)) * es if self.shape else es


class RequestRecord:
    """REQUEST_START / SEND_START / SEND_END / RECV_START / RECV_END / REQUEST_END of
    the reference's RequestTimers, reduced to what a Python transport can observe."""

    __slots__ = ("start_ns", "end_ns", "first_response_ns", "ok")

    def __init__(self, start_ns, end_ns, first_response_ns=None, ok=True):
        self.start_ns, self.end_ns, self.first_response_ns, self.ok = start_ns, end_ns, first_response_ns, ok


class InferStat:
    """Cumulative client-side statistics (reference InferStat, common.h:93-114)."""

    def __init__(self):
        self.completed_request_count = 0
        self.cumulative_total_request_time_ns = 0
        self.failed_request_count = 0

    def add(self, rec):
        if rec.ok:
            self.completed_request_count += 1
            self.cumulative_total_request_time_ns += rec.end_ns - rec.start_ns
        else:
            self.failed_request_count += 1


class SlotSet:
    """Per-slot input/output buffers and their device job tables.

    ``replay``: an ``input_data.InputData`` (``--input-data FILE|DIR``).  The slots' inputs are
    then copied from its device pool instead of generated, and outputs named in its
    ``validation_data`` are compared bytewise with the expected entry (cuda shm only)."""

    def __init__(self, inputs, outputs, slots, shared_memory, device_id, input_data, seed, token_range=None,
                 name_prefix="tb200", staging=None, wire_prefixes=None, lookahead=1, replay=None):
        self.inputs, self.outputs, self.slots = inputs, outputs, slots
        self.replay = replay
        if replay is not None and replay.expected and shared_memory != "cuda":
            raise InputDataError("validation_data is checked on the device, which holds the outputs only with --shared-memory cuda")
        self._gen = [-1] * slots  # replay: the generation each slot's inputs hold (-1: not written yet)
        self.validation_mismatches = 0  # bytes that differ from validation_data, over all validate() calls
        # wire mode + native engine: every slot owns `lookahead` staging images that one device
        # pass generates together; the transport sends them one after the other and returns the
        # slot to the device thread only when all are used (every request still carries fresh
        # data, the device is visited once per `lookahead` requests)
        self.lookahead = max(1, int(lookahead))
        if self.lookahead > 1 and shared_memory == "system":
            raise ValueError("lookahead applies to --shared-memory none / cuda")
        self.shared_memory, self.device_id = shared_memory, device_id
        self.input_data, self.seed = input_data, seed
        self.in_bytes = sum(t.nbytes for t in inputs)
        # wire mode only: constant bytes in front of every tensor inside the staging image of a
        # slot (gRPC: the raw_input_contents tag + length), written once; the kernels fill
        # the tensor bytes between them
        self._prefixes = [bytes(b) for b in wire_prefixes] if wire_prefixes else [b""] * len(inputs)
        if any(self._prefixes) and shared_memory != "none":
            raise ValueError("wire prefixes only apply to --shared-memory none")
        self.wire_stride = self.in_bytes + sum(len(b) for b in self._prefixes)
        self.out_bytes = sum(t.nbytes for t in outputs)
        self.prefix = name_prefix
        self.epoch = 0
        self._ops = None
        self._staging = None
        self.token_range = token_range or {}
        if shared_memory == "cuda":
            from ..device import DeviceOps
            from ..utils import cuda_shared_memory as cudashm

            self._cudashm = cudashm
            self._ops = DeviceOps(_native.Context(device_id))
            self.in_region = cudashm.create_shared_memory_region(self.prefix + "_in", max(slots * self.lookahead * self.in_bytes, 16), device_id)
            self.out_region = cudashm.create_shared_memory_region(self.prefix + "_out", max(slots * self.lookahead * self.out_bytes, 16), device_id)
            self.in_base, self.out_base = self.in_region._base_addr, self.out_region._base_addr
        elif shared_memory == "system":
            from ..utils import shared_memory as sysshm

            self._sysshm = sysshm
            self.in_region = sysshm.create_shared_memory_region(self.prefix + "_in", "/" + self.prefix + "_in", max(slots * self.in_bytes, 16))
            self.out_region = sysshm.create_shared_memory_region(self.prefix + "_out", "/" + self.prefix + "_out", max(slots * self.out_bytes, 16))
            self._wire = None
        if shared_memory != "cuda":
            # wire / system-shm mode: the kernels emit into pinned, device-mapped host
            # memory.  No host fallback: without libtb200 / a GPU this raises.  (Tests on
            # CPU-only machines inject their own ``staging`` object.)
            if staging is not None:
                self._staging = staging
                staging.allocate(max(slots * self.lookahead * self.wire_stride, 16))
            else:
                from ..device import DeviceOps, HostBuffer

                self._ops = DeviceOps(_native.Context(device_id))
                self._wire = HostBuffer(max(slots * self.lookahead * self.wire_stride, 16))
                self.in_base = self._wire.device_ptr
            if any(self._prefixes):
                for s, g in ((s, g) for s in range(slots) for g in range(self.lookahead)):
                    for i, b in enumerate(self._prefixes):
                        off = self.input_offset(s, i, g) - len(b)
                        view = self._staging.view(off, len(b)) if self._staging is not None else self._wire.view(off, len(b))
                        view[:] = b
        self._results = None
        self._result_view = None
        if replay is not None and self._staging is None:
            replay.upload(self._ops)

    # -- layout ------------------------------------------------------------------------
    def input_offset(self, slot, index, generation=0):
        if self.shared_memory == "none":
            before = sum(len(self._prefixes[k]) + self.inputs[k].nbytes for k in range(index))
            return (slot * self.lookahead + generation) * self.wire_stride + before + len(self._prefixes[index])
        return (slot * self.lookahead + generation) * self.in_bytes + sum(t.nbytes for t in self.inputs[:index])

    def output_offset(self, slot, index, generation=0):
        return (slot * self.lookahead + generation) * self.out_bytes + sum(t.nbytes for t in self.outputs[:index])

    def input_bytes(self, slot, index):
        """Host view of a generated input (wire / system-shm modes)."""
        off, n = self.input_offset(slot, index), self.inputs[index].nbytes
        if self._staging is not None:
            return self._staging.view(off, n)
        return self._wire.view(off, n)

    # -- device work -----------------------------------------------------------------------
    def _fill_jobs(self, slot_ids):
        from ..device import make_fill_job

        jobs = []
        for s, g in ((s, g) for s in slot_ids for g in range(self.lookahead)):
            image = s * self.lookahead + g  # == s without lookahead: stream ids as before
            for i, t in enumerate(self.inputs):
                mode = "zero" if self.input_data == "zero" else "random"
                lo, hi = 0.0, None
                if t.datatype.startswith(("INT", "UINT")) and mode == "random":
                    rng = self.token_range.get(t.name)
                    lo, hi = (rng if rng else (0, None))
                if t.datatype == "BYTES":
                    # zero data for strings = empty-content strings is not expressible at a
                    # fixed byte size; perf_analyzer sends random strings in both modes
                    jobs.append(make_fill_job(self.in_base + self.input_offset(s, i, g), t.nbytes, "BYTES",
                                              stream_id=(image << 8) | i, string_length=t.string_length))
                    continue
                jobs.append(make_fill_job(self.in_base + self.input_offset(s, i, g), t.nbytes, t.datatype,
                                          stream_id=(image << 8) | i, mode=mode, low=lo, high=hi))
        return jobs

    def entry(self, slot, image=0):
        """The replayed entry that image ``image`` of the slot's current generation carries."""
        return replay_entry(slot, self._gen[slot] * self.lookahead + image, self.lookahead, False, self.replay.entries)

    def _copy_jobs(self, slot_ids, at_entry=None):
        """Copies of replayed entries into the inputs of the given slots (slot, image, input order,
        like _fill_jobs): each image's own entry, or entry ``at_entry`` everywhere."""
        from .._native import CopyJob

        jobs = []
        for s, g in ((s, g) for s in slot_ids for g in range(self.lookahead)):
            e = self.entry(s, g) if at_entry is None else at_entry
            for i, t in enumerate(self.inputs):
                jobs.append(CopyJob(dst=self.in_base + self.input_offset(s, i, g), src=self.replay.input_ptr(t.name) + e * t.nbytes, nbytes=t.nbytes))
        return jobs

    def _check_jobs(self, slot_ids, at_entry=None):
        """Validation of the outputs of the given slots (slot, image, output order): EQUAL against the
        replayed entry for outputs named in validation_data, else TOP1 (FP32) / SUM."""
        from .._native import CheckJob

        expected = self.replay.expected if self.replay is not None else {}
        jobs = []
        for s, g in ((s, g) for s in slot_ids for g in range(self.lookahead)):
            for i, t in enumerate(self.outputs):
                a = self.out_base + self.output_offset(s, i, g)
                if t.name in expected:
                    e = self.entry(s, g) if at_entry is None else at_entry
                    jobs.append(CheckJob(a=a, b=self.replay.expected_ptr(t.name) + e * t.nbytes, nbytes=t.nbytes, kind=_native.CHECK_EQUAL))
                else:
                    jobs.append(CheckJob(a=a, nbytes=t.nbytes, kind=_native.CHECK_TOP1 if t.datatype == "FP32" else _native.CHECK_SUM))
        return jobs

    def generate(self, slot_ids):
        """(Re)generate the inputs of the given slots: one launch, returns when visible.  With
        replayed data every slot moves on to its next generation's entries."""
        if not slot_ids:
            return
        if self.replay is not None:
            for s in slot_ids:
                self._gen[s] += 1
            if self._staging is not None:
                for s, g in ((s, g) for s in slot_ids for g in range(self.lookahead)):
                    for i, t in enumerate(self.inputs):
                        self._staging.view(self.input_offset(s, i, g), t.nbytes)[:] = self.replay.inputs[t.name][self.entry(s, g)]
            else:
                self._ops.concat(self._copy_jobs(slot_ids))
                self._ops.sync()
        elif self._staging is not None:
            self._staging.fill([(self.input_offset(s, i, g), t) for s in slot_ids for g in range(self.lookahead) for i, t in enumerate(self.inputs)],
                               self.input_data, self.seed + self.epoch)
        else:
            self._ops.fill(self._fill_jobs(slot_ids), seed=self.seed, epoch=self.epoch)
            self._ops.sync()
        self.epoch += 1 << 20
        if self.shared_memory == "system":
            # POSIX shm is host memory: copy the generated slot from the pinned staging
            buf = self.in_region._mpsm_handle.buf
            for s in slot_ids:
                off = s * self.in_bytes
                buf[off:off + self.in_bytes] = self._slot_view(off)

    def _slot_view(self, off):
        if self._staging is not None:
            return self._staging.view(off, self.in_bytes)
        return self._wire.view(off, self.in_bytes)

    def validate(self, slot_ids):
        """Device-side checksum / top-1 of the outputs of the given slots (cuda shm), and the
        bytewise comparison with validation_data (added to ``validation_mismatches``); returns the
        number of non-finite values seen (0 expected)."""
        if self.shared_memory != "cuda" or not slot_ids or not self.outputs:
            return 0
        from ..device import HostBuffer, results_array

        if self._results is None:
            n = self.slots * self.lookahead * len(self.outputs)
            self._results = HostBuffer(n * 32)
            self._result_view = results_array(self._results, n)
        jobs = self._check_jobs(slot_ids)
        self._ops.check(jobs, self._results.device_ptr)
        self._ops.sync()
        bad = 0
        for k, job in enumerate(jobs):
            if job.kind == _native.CHECK_TOP1:
                bad += int(self._result_view["mismatches"][k])
            elif job.kind == _native.CHECK_EQUAL:
                self.validation_mismatches += int(self._result_view["mismatches"][k])
        return bad

    # -- server registration --------------------------------------------------------------------
    def register(self, client):
        if self.shared_memory == "cuda":
            client.register_cuda_shared_memory(self.prefix + "_in", self._cudashm.get_raw_handle(self.in_region), self.device_id, max(self.slots * self.lookahead * self.in_bytes, 16))
            client.register_cuda_shared_memory(self.prefix + "_out", self._cudashm.get_raw_handle(self.out_region), self.device_id, max(self.slots * self.lookahead * self.out_bytes, 16))
        elif self.shared_memory == "system":
            client.register_system_shared_memory(self.prefix + "_in", "/" + self.prefix + "_in", max(self.slots * self.in_bytes, 16))
            client.register_system_shared_memory(self.prefix + "_out", "/" + self.prefix + "_out", max(self.slots * self.out_bytes, 16))

    def unregister(self, client):
        try:
            if self.shared_memory == "cuda":
                client.unregister_cuda_shared_memory(self.prefix + "_in")
                client.unregister_cuda_shared_memory(self.prefix + "_out")
            elif self.shared_memory == "system":
                client.unregister_system_shared_memory(self.prefix + "_in")
                client.unregister_system_shared_memory(self.prefix + "_out")
        except InferenceServerException:
            pass

    def close(self):
        if self.shared_memory == "cuda":
            self._cudashm.destroy_shared_memory_region(self.in_region)
            self._cudashm.destroy_shared_memory_region(self.out_region)
        elif self.shared_memory == "system":
            self._sysshm.destroy_shared_memory_region(self.in_region)
            self._sysshm.destroy_shared_memory_region(self.out_region)


class ConcurrencyManager:
    """Keeps ``concurrency`` requests in flight: one transport worker per in-flight
    request plus one device thread that regenerates / validates slots in batches."""

    def __init__(self, make_client, protocol, model_name, model_version, slotset, concurrency,
                 per_request_data=True, validate=True, streaming=False, request_parameters=None):
        self.make_client, self.protocol = make_client, protocol
        self.model_name, self.model_version = model_name, model_version
        self.slotset, self.concurrency = slotset, concurrency
        self.per_request_data, self.validate = per_request_data, validate
        self.streaming = streaming
        self.request_parameters = request_parameters
        self.records = []
        self._records_lock = threading.Lock()
        self._ready = queue.Queue()
        self._returned = queue.Queue()
        self._stop = threading.Event()
        self._threads = []
        self.stat = InferStat()
        self.device_batches = []
        self.nonfinite = 0
        self.errors = []

    # -- request construction ---------------------------------------------------------------
    def _build(self, mod, slot):
        ss = self.slotset
        inputs, outputs = [], []
        for i, t in enumerate(ss.inputs):
            inp = mod.InferInput(t.name, t.shape, t.datatype)
            if ss.shared_memory in ("cuda", "system"):
                inp.set_shared_memory(ss.prefix + "_in", t.nbytes, offset=ss.input_offset(slot, i))
            inputs.append(inp)
        for i, t in enumerate(ss.outputs):
            out = mod.InferRequestedOutput(t.name)
            if ss.shared_memory in ("cuda", "system"):
                out.set_shared_memory(ss.prefix + "_out", t.nbytes, offset=ss.output_offset(slot, i))
            outputs.append(out)
        return inputs, outputs

    def _attach_wire_data(self, inputs, slot):
        ss = self.slotset
        for i, t in enumerate(ss.inputs):
            if t.datatype == "BYTES":  # the staging holds the serialised elements
                arr = deserialize_bytes_tensor(bytes(ss.input_bytes(slot, i))).reshape(t.shape)
            else:
                arr = np.frombuffer(ss.input_bytes(slot, i), dtype=triton_to_np_dtype(t.datatype)).reshape(t.shape)
            inputs[i].set_data_from_numpy(arr)

    # -- threads --------------------------------------------------------------------------------
    def _worker(self):
        if self.protocol == "grpc":
            from .. import grpc as mod
        else:
            from .. import http as mod
        client = self.make_client()
        built = {}
        first_response = {}
        stream_done = queue.Queue()
        if self.streaming:
            def on_response(result, error):
                now = time.perf_counter_ns()
                if error is not None:
                    stream_done.put((now, error))
                    return
                params = result.get_response().parameters
                final = params["triton_final_response"].bool_param if "triton_final_response" in params else True
                if "first" not in first_response:
                    first_response["first"] = now
                if final:
                    stream_done.put((now, None))

            client.start_stream(callback=on_response)
        try:
            while not self._stop.is_set():
                try:
                    slot = self._ready.get(timeout=0.05)
                except queue.Empty:
                    continue
                if slot not in built:
                    built[slot] = self._build(mod, slot)
                inputs, outputs = built[slot]
                if self.slotset.shared_memory == "none":
                    self._attach_wire_data(inputs, slot)
                ok, first = True, None
                t0 = time.perf_counter_ns()
                try:
                    if self.streaming:
                        first_response.clear()
                        client.async_stream_infer(self.model_name, inputs, model_version=self.model_version,
                                                  outputs=outputs, parameters=self.request_parameters)
                        t1, err = stream_done.get(timeout=120)
                        first = first_response.get("first")
                        ok = err is None
                    else:
                        client.infer(self.model_name, inputs, model_version=self.model_version, outputs=outputs,
                                     parameters=self.request_parameters)
                        t1 = time.perf_counter_ns()
                except Exception as ex:  # noqa: BLE001
                    t1 = time.perf_counter_ns()
                    ok = False
                    if len(self.errors) < 5:
                        self.errors.append(repr(ex))
                rec = RequestRecord(t0, t1, first, ok)
                with self._records_lock:
                    self.records.append(rec)
                    self.stat.add(rec)
                self._returned.put(slot)
        finally:
            if self.streaming:
                client.stop_stream()
            client.close()

    def _device_thread(self):
        ss = self.slotset
        while not self._stop.is_set():
            try:
                batch = [self._returned.get(timeout=0.05)]
            except queue.Empty:
                continue
            while True:  # everything that came back meanwhile joins the same launches
                try:
                    batch.append(self._returned.get_nowait())
                except queue.Empty:
                    break
            if self.validate:
                self.nonfinite += ss.validate(batch)
            if self.per_request_data:
                ss.generate(batch)
            self.device_batches.append(len(batch))
            for s in batch:
                self._ready.put(s)

    def start(self):
        self.slotset.generate(list(range(self.concurrency)))
        for s in range(self.concurrency):
            self._ready.put(s)
        t = threading.Thread(target=self._device_thread, daemon=True)
        t.start()
        self._threads.append(t)
        for _ in range(self.concurrency):
            t = threading.Thread(target=self._worker, daemon=True)
            t.start()
            self._threads.append(t)

    def stop(self):
        self._stop.set()
        for t in self._threads:
            t.join(timeout=30)

    def swap_records(self):
        with self._records_lock:
            recs, self.records = self.records, []
        return recs


def summarize(records, window_s, percentile=None):
    ok = [r for r in records if r.ok]
    lat = np.array([(r.end_ns - r.start_ns) / 1e3 for r in ok], dtype=np.float64)
    out = {"count": len(ok), "failed": len(records) - len(ok), "throughput": len(ok) / window_s if window_s > 0 else 0.0}
    if lat.size:
        out.update(avg_us=float(lat.mean()), p50_us=float(np.percentile(lat, 50)), p90_us=float(np.percentile(lat, 90)),
                   p95_us=float(np.percentile(lat, 95)), p99_us=float(np.percentile(lat, 99)),
                   min_us=float(lat.min()), max_us=float(lat.max()))
        out["latency_us"] = float(np.percentile(lat, percentile)) if percentile else out["avg_us"]
    ttft = np.array([(r.first_response_ns - r.start_ns) / 1e3 for r in ok if r.first_response_ns], dtype=np.float64)
    if ttft.size:
        out.update(ttft_p50_us=float(np.percentile(ttft, 50)), ttft_p99_us=float(np.percentile(ttft, 99)))
    return out


def measure(manager, interval_ms=1000, stability_pct=10.0, max_trials=10, percentile=None, min_windows=3):
    """time_windows measurement: windows of ``interval_ms`` until the last three agree
    within ``stability_pct`` in throughput and latency, or ``max_trials`` windows."""
    manager.swap_records()
    windows = []
    seen = manager.slotset.validation_mismatches
    for _ in range(max_trials):
        t0 = time.perf_counter()
        time.sleep(interval_ms / 1e3)
        recs = manager.swap_records()
        windows.append(summarize(recs, time.perf_counter() - t0, percentile))
        now = manager.slotset.validation_mismatches
        windows[-1]["validation_mismatches"], seen = now - seen, now
        if len(windows) >= min_windows:
            last = windows[-min_windows:]
            thr = [w["throughput"] for w in last]
            lat = [w.get("latency_us", 0.0) for w in last]
            if min(thr) > 0 and (max(thr) - min(thr)) / max(thr) <= stability_pct / 100.0 and \
                    (max(lat) == 0 or (max(lat) - min(lat)) / max(lat) <= stability_pct / 100.0):
                break
    last = windows[-min_windows:] if len(windows) >= min_windows else windows
    total = sum(w["count"] for w in last)
    merged = dict(last[-1])
    merged["throughput"] = float(np.mean([w["throughput"] for w in last]))
    merged["windows"] = len(windows)
    merged["stable"] = len(windows) < max_trials or len(windows) == min_windows
    merged["count"] = total
    merged["validation_mismatches"] = sum(w["validation_mismatches"] for w in last)
    return merged
