"""--input-data FILE|DIR on the GPU: replayed entries reach the server byte for byte, in the order
the entry rule gives; validation_data is checked on the device by both engines; directory mode;
and tb200_step_submit_copy itself against numpy."""

import base64
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from client_b200.perf import cli
from client_b200.perf import input_data as idata

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def server():
    """The native stand-in server (own process: it opens the client's CUDA IPC handles)."""
    proc = subprocess.Popen([sys.executable, "-m", "client_b200.testing.native_server", "--port", "0", "--grpc-port", "0"],
                            cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    line = proc.stdout.readline()
    assert "listening" in line and "grpc=" in line, line + proc.stdout.read()
    yield {"http": line.split()[5], "grpc": line.split("grpc=")[1].strip()}
    proc.terminate()
    proc.wait(10)


def _bert_entries(n):
    return [{"input_ids": (1000 * e + np.arange(384)).tolist(), "attention_mask": [e % 2] * 384} for e in range(n)]


@pytest.mark.parametrize("depth,lookahead,once", [(1, 1, False), (1, 4, False), (3, 1, False), (3, 4, False), (3, 1, True), (3, 4, True)])
def test_replayed_wire_bytes_reach_the_server(depth, lookahead, once):
    """Every request a grpcio server receives carries both tensors of exactly one entry; per-request
    data cycles through every entry, data written once only the entries (s + g) mod N of its images."""
    from concurrent import futures

    import grpc

    from client_b200.grpc import service_pb2, service_pb2_grpc
    from client_b200.perf.loadgen import SlotSet, TensorSpec
    from client_b200.perf.native import NativeLoadGenerator, grpc_wire_prefixes

    received = []

    class Capture(service_pb2_grpc.GRPCInferenceServiceServicer):
        def ModelInfer(self, request, context):
            received.append([bytes(b) for b in request.raw_input_contents])
            return service_pb2.ModelInferResponse(model_name=request.model_name)

    srv = grpc.server(futures.ThreadPoolExecutor(max_workers=8))
    service_pb2_grpc.add_GRPCInferenceServiceServicer_to_server(Capture(), srv)
    port = srv.add_insecure_port("127.0.0.1:0")
    srv.start()
    n = 5
    slots = 1 if once else 8
    ins = [TensorSpec("input_ids", "INT64", [1, 384]), TensorSpec("attention_mask", "INT64", [1, 384])]
    data = idata.parse_json({"data": _bert_entries(n)}, ins, [])
    entry_bytes = [(data.inputs["input_ids"][e].tobytes(), data.inputs["attention_mask"][e].tobytes()) for e in range(n)]
    try:
        ss = SlotSet(ins, [], slots, "none", 0, "random", 5, name_prefix="replaywire", wire_prefixes=grpc_wire_prefixes(ins),
                     lookahead=lookahead, replay=data)
        gen = NativeLoadGenerator("127.0.0.1:%d" % port, "bert_large", "", ss, slots, regenerate=not once, validate=False,
                                  protocol="grpc", pipeline_depth=depth)
        gen.start()
        w = gen.window(0.6)
        gen.stop()
        ss.close()
        assert w["failed"] == 0 and w["count"] >= 4 * lookahead * slots, w
        seen = set()
        for tensors in received:
            matches = [e for e in range(n) if tuple(tensors) == entry_bytes[e]]
            assert len(matches) == 1, "a request carried bytes of no entry, or a mix of entries"
            seen.add(matches[0])
        allowed = {(s + g) % n for s in range(slots) for g in range(lookahead)} if once else set(range(n))
        assert seen == allowed
    finally:
        data.close()
        srv.stop(0)


def _simple_file(tmp_path, n=4, flip=False):
    data, valid = [], []
    for e in range(n):
        a = (np.arange(16) * (e + 1)).astype(np.int32)
        b = np.full(16, 3 - e, np.int32)
        out0 = (a + b).astype(np.int32).view(np.uint8).copy()
        if flip:
            out0[0] ^= 0xFF
        data.append({"INPUT0": {"content": a.tolist(), "shape": [1, 16]}, "INPUT1": b.reshape(1, 16).tolist()})
        valid.append({"OUTPUT0": {"b64": base64.b64encode(out0.tobytes()).decode()}, "OUTPUT1": (a - b).tolist()})
    path = tmp_path / ("simple_flipped.json" if flip else "simple.json")
    path.write_text(json.dumps({"data": data, "validation_data": valid}))
    return str(path)


@pytest.mark.parametrize("protocol", ["http", "grpc"])
@pytest.mark.parametrize("depth,lookahead", [(1, 1), (1, 2), (3, 1), (3, 2)])
def test_native_engine_validates_on_the_device(server, tmp_path, protocol, depth, lookahead):
    common = ["-m", "simple", "-u", server[protocol], "-i", protocol, "--shared-memory", "cuda", "--engine", "native",
              "--device-pipeline", str(depth), "--lookahead", str(lookahead), "--concurrency-range", "4", "-p", "300", "-r", "3", "--json"]
    rows = cli.main(common + ["--input-data", _simple_file(tmp_path)])
    r = rows[0]
    assert r["count"] > 0 and r["failed"] == 0 and r["input_data_entries"] == 4 and r["validation_mismatches"] == 0, r
    assert cli.exit_status(rows) == 0

    # first byte of every expected OUTPUT0 flipped: one differing byte per returned image
    from client_b200.perf.loadgen import SlotSet, TensorSpec
    from client_b200.perf.native import NativeLoadGenerator

    ins = [TensorSpec("INPUT0", "INT32", [1, 16]), TensorSpec("INPUT1", "INT32", [1, 16])]
    outs = [TensorSpec("OUTPUT0", "INT32", [1, 16]), TensorSpec("OUTPUT1", "INT32", [1, 16])]
    data = idata.load(_simple_file(tmp_path, flip=True), ins, outs)
    if protocol == "grpc":
        import client_b200.grpc as client_mod
    else:
        import client_b200.http as client_mod
    client = client_mod.InferenceServerClient(server[protocol])
    ss = SlotSet(ins, outs, 4, "cuda", 0, "random", 0, name_prefix="flip_%s_%d_%d" % (protocol, depth, lookahead), lookahead=lookahead, replay=data)
    ss.register(client)
    try:
        gen = NativeLoadGenerator(server[protocol], "simple", "", ss, 4, protocol=protocol, pipeline_depth=depth)
        gen.start()
        gen.window(0.1)
        w = gen.window(0.4)
        gen.stop()
        assert w["failed"] == 0 and w["device_slots"] > 0, w
        assert w["mismatches"] == w["device_slots"] * lookahead, w
    finally:
        ss.unregister(client)
        ss.close()
        data.close()
        client.close()


def test_cli_exits_1_on_a_mismatch(server, tmp_path):
    r = subprocess.run([sys.executable, "-m", "client_b200.perf", "-m", "simple", "-u", server["http"], "--shared-memory", "cuda",
                        "--engine", "native", "--concurrency-range", "2", "-p", "200", "-r", "3", "--json",
                        "--input-data", _simple_file(tmp_path, flip=True)], cwd=ROOT, capture_output=True, text=True, timeout=300)
    assert r.returncode == 1, r.stdout[-800:] + r.stderr[-800:]
    row = json.loads(r.stdout.strip().splitlines()[-1])
    assert row["validation_mismatches"] > 0 and row["input_data_entries"] == 4


def test_python_engine_validates_on_the_device(server, tmp_path):
    common = ["-m", "simple", "-u", server["http"], "--shared-memory", "cuda", "--concurrency-range", "2", "-p", "300", "-r", "3", "--json"]
    rows = cli.main(common + ["--input-data", _simple_file(tmp_path)])
    assert rows[0]["count"] > 0 and rows[0]["failed"] == 0 and rows[0]["validation_mismatches"] == 0, rows
    assert rows[0]["input_data_entries"] == 4
    rows = cli.main(common + ["--input-data", _simple_file(tmp_path, flip=True)])
    assert rows[0]["count"] > 0 and rows[0]["validation_mismatches"] > 0 and cli.exit_status(rows) == 1, rows


def test_directory_mode_once_densenet(server, tmp_path):
    """One entry from raw files, written once: after the run every slot's input region holds the file."""
    import client_b200.http as httpclient
    import client_b200.utils.cuda_shared_memory as cudashm
    from client_b200.perf.loadgen import SlotSet, TensorSpec
    from client_b200.perf.native import NativeLoadGenerator

    raw = np.random.default_rng(3).random(3 * 224 * 224, dtype=np.float32).tobytes()
    (tmp_path / "data_0").write_bytes(raw)
    ins, outs = [TensorSpec("data_0", "FP32", [3, 224, 224])], [TensorSpec("fc6_1", "FP32", [1000])]
    data = idata.load(str(tmp_path), ins, outs)
    slots = 4
    client = httpclient.InferenceServerClient(server["http"])
    ss = SlotSet(ins, outs, slots, "cuda", 0, "random", 0, name_prefix="replaydir", replay=data)
    ss.register(client)
    try:
        gen = NativeLoadGenerator(server["http"], "densenet_onnx", "", ss, slots, regenerate=False)
        gen.start()
        w = gen.window(0.4)
        gen.stop()
        assert w["count"] > slots and w["failed"] == 0 and w["nonfinite"] == 0, w
        region = cudashm.get_contents_as_numpy(ss.in_region, np.uint8, [slots * ss.in_bytes])
        for s in range(slots):
            assert region[s * ss.in_bytes:(s + 1) * ss.in_bytes].tobytes() == raw, "slot %d" % s
    finally:
        ss.unregister(client)
        ss.close()
        data.close()
        client.close()
    rows = cli.main(["-m", "densenet_onnx", "-u", server["http"], "--shared-memory", "cuda", "--engine", "native", "--input-data-mode", "once",
                     "--input-data", str(tmp_path), "--concurrency-range", "4", "-p", "300", "-r", "3", "--json"])
    assert rows[0]["count"] > 0 and rows[0]["failed"] == 0 and rows[0]["input_data_entries"] == 1, rows


def test_step_submit_copy_against_numpy(gpu_ops):
    """Copies + EQUAL checks of several steps in flight: every copy lands, every mismatch count is numpy's."""
    from client_b200._native import CheckJob, CopyJob
    from client_b200.device import DeviceBuffer, HostBuffer, results_array

    rng = np.random.default_rng(11)
    entries, nbytes, jobs, steps = 8, 4096 * 3 + 5, 6, 4
    pool = rng.integers(0, 256, (entries, nbytes), dtype=np.uint8)
    outs = np.repeat(pool[None], steps, axis=0).reshape(steps * entries, nbytes).copy()
    flips = rng.integers(0, 40, steps * entries)
    for k, f in enumerate(flips):
        outs[k, rng.choice(nbytes, size=int(f), replace=False)] ^= 0x5A
    dpool, douts = gpu_ops.upload(pool), gpu_ops.upload(outs)
    dst = DeviceBuffer(0, steps * jobs * nbytes)
    res = HostBuffer(steps * jobs * 32)
    view = results_array(res, steps * jobs)
    tickets, want_dst, want_mism = [], [], []
    for st in range(steps):
        copies, checks = [], []
        for j in range(jobs):
            e = (st + 3 * j) % entries
            copies.append(CopyJob(dst=dst.ptr + (st * jobs + j) * nbytes, src=dpool.ptr + e * nbytes, nbytes=nbytes))
            want_dst.append(pool[e])
            k = st * entries + e
            checks.append(CheckJob(a=douts.ptr + k * nbytes, b=dpool.ptr + e * nbytes, nbytes=nbytes, kind=1))
            want_mism.append(int(np.count_nonzero(outs[k] != pool[e])))
        tickets.append(gpu_ops.step_submit_copy(copies, checks, res.device_ptr + st * jobs * 32))
    assert len(set(tickets)) == steps
    for t in tickets:
        gpu_ops.step_wait(t)
    got = gpu_ops.download(dst.ptr, steps * jobs * nbytes).reshape(steps * jobs, nbytes)
    assert np.array_equal(got, np.stack(want_dst))
    assert view["mismatches"].tolist() == want_mism and sum(want_mism) > 0
    for b in (dpool, douts, dst):
        b.close()
    res.close()
