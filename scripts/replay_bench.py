"""Replayed inputs (--input-data FILE|DIR) on the device: what one tb200_step_submit_copy pass costs for
config C2, and the loopback throughput with replayed against generated inputs.
   python scripts/replay_bench.py   (GPU box)

Pass: 64 slots x FP32[3,224,224] (602,112 B) copied from a pool of 64 entries (slot s takes entry
(s + pass) mod 64), optionally with 64 EQUAL checks of 4,000 B outputs against expected entries.
Algorithmic bytes per pass: read + write of every copied byte (2 x 64 x 602,112), plus both operands
of every check (2 x 64 x 4,000); reported over CUDA-event time and as a fraction of the H100 SXM data
sheet's 3.35 TB/s."""
import base64
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from client_b200 import _native  # noqa: E402
from client_b200._native import CheckJob, CopyJob  # noqa: E402
from client_b200.device import DeviceBuffer, DeviceOps, HostBuffer  # noqa: E402

SLOTS, ENTRIES, IN_BYTES, OUT_BYTES = 64, 64, 602112, 4000
PEAK = 3.35e12
WARMUP, PASSES = 200, 2000


def pass_bench():
    ctx = _native.Context(0)
    ops = DeviceOps(ctx)
    rng = np.random.default_rng(0)
    pool = ops.upload(rng.integers(0, 256, (ENTRIES, IN_BYTES), dtype=np.uint8))
    expected = ops.upload(rng.integers(0, 256, (ENTRIES, OUT_BYTES), dtype=np.uint8))
    inputs, outputs = DeviceBuffer(0, SLOTS * IN_BYTES), DeviceBuffer(0, SLOTS * OUT_BYTES)
    ring = 8  # result blocks: one per step the ticket ring can hold in flight
    res = HostBuffer(ring * SLOTS * 32)
    # job tables of every rotation, built before timing so that the loop times the device, not Python
    copies = [(CopyJob * SLOTS)(*[CopyJob(dst=inputs.ptr + s * IN_BYTES, src=pool.ptr + ((s + p) % ENTRIES) * IN_BYTES, nbytes=IN_BYTES)
                                  for s in range(SLOTS)]) for p in range(ENTRIES)]
    checks = [(CheckJob * SLOTS)(*[CheckJob(a=outputs.ptr + s * OUT_BYTES, b=expected.ptr + ((s + p) % ENTRIES) * OUT_BYTES, nbytes=OUT_BYTES,
                                            kind=_native.CHECK_EQUAL) for s in range(SLOTS)]) for p in range(ENTRIES)]
    timer = _native.Timer(ctx)
    out = {}
    for name, with_checks in (("copies", False), ("copies+checks", True)):
        def run(n, first):
            tickets = []
            for i in range(n):
                p = (first + i) % ENTRIES
                tickets.append(ops.step_submit_copy(copies[p], checks[p] if with_checks else [], res.device_ptr + (i % ring) * SLOTS * 32))
            for t in tickets[-ring:]:
                ops.step_wait(t)

        run(WARMUP, 0)
        ops.sync()
        timer.start()
        run(PASSES, WARMUP)
        timer.stop()  # recorded after every step's events completed: covers the side-stream checks too
        ms = timer.elapsed_ms()
        nbytes = 2 * SLOTS * IN_BYTES + (2 * SLOTS * OUT_BYTES if with_checks else 0)
        rate = nbytes * PASSES / (ms * 1e-3)
        out[name] = (ms * 1e3 / PASSES, rate)
        print("%-14s %8.1f us/pass  %7.1f GB/s  %.3f of 3.35 TB/s  (%d passes, %d B per pass)" % (
            name, ms * 1e3 / PASSES, rate / 1e9, rate / PEAK, PASSES, nbytes), flush=True)
    for b in (pool, expected, inputs, outputs):
        b.close()
    return out


def loopback():
    """densenet_onnx, native engine, cuda shm, concurrency 64: --input-data random against a JSON of 64 entries."""
    from client_b200.perf import cli

    tmp = tempfile.mkdtemp(prefix="replay_bench_")
    proc = subprocess.Popen([sys.executable, "-m", "client_b200.testing.native_server", "--port", "0"], cwd=ROOT,
                            stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        line = proc.stdout.readline()
        assert "listening" in line, line
        url = line.split()[5]
        rng = np.random.default_rng(1)
        entries = [{"data_0": {"b64": base64.b64encode(rng.random(IN_BYTES // 4, dtype=np.float32).tobytes()).decode()}} for _ in range(ENTRIES)]
        path = os.path.join(tmp, "densenet_64.json")
        with open(path, "w") as fh:
            json.dump({"data": entries}, fh)
        common = ["-m", "densenet_onnx", "-u", url, "--shared-memory", "cuda", "--engine", "native", "--concurrency-range", "64",
                  "-p", "1000", "-r", "6", "--json"]
        rows = {}
        for name, data in (("random", "random"), ("json64", path)):
            r = cli.main(common + ["--input-data", data])[0]
            rows[name] = r
            print("loopback densenet_onnx c64 --input-data %-7s %9.0f infer/s  p50 %6.0f us  failed %d  nonfinite %d  entries %d" % (
                name, r["throughput"], r["p50_us"], r["failed"], r["nonfinite"], r["input_data_entries"]), flush=True)
        return rows
    finally:
        proc.terminate()
        proc.wait(10)
        shutil.rmtree(tmp, ignore_errors=True)


def main():
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv"], capture_output=True, text=True).stdout.strip()
    print(card, flush=True)
    pass_bench()
    loopback()


if __name__ == "__main__":
    main()
