"""Host logic of bench.py that needs no GPU: which device ordinal and environment the processes of GPU d
get, and how the client processes of a box are spawned."""

import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402


def test_processes_see_every_gpu(monkeypatch):
    monkeypatch.delenv("CUDA_VISIBLE_DEVICES", raising=False)
    box = bench.LoopbackBox([0, 3])
    assert box.ordinal == {0: 0, 3: 3}
    assert "CUDA_VISIBLE_DEVICES" not in box.envs[3] and "TB200_PIN_GPU" not in box.envs[3]


def _env_probe(impl, url, device, tag, seconds, data_mode, ready, go, q):
    """stands in for bench._host_loop_worker: `url` is a directory here; leave what this child sees in it"""
    import json

    with open(os.path.join(url, tag + ".json"), "w") as fh:
        json.dump([device, os.environ.get("CUDA_VISIBLE_DEVICES"), os.environ.get("TB200_PIN_GPU")], fh)
    ready.wait()
    go.wait()
    q.put((1, [1000.0], None))


def test_host_loop_children_inherit_their_gpus_environment(monkeypatch, tmp_path):
    """host_loops spawns the clients of GPU d with d's environment and ordinal, and leaves this process's environment alone"""
    import json

    class Box:
        devices = [0, 1]
        urls = {0: str(tmp_path), 1: str(tmp_path)}
        ordinal = {0: 0, 1: 0}
        envs = {0: {"CUDA_VISIBLE_DEVICES": "4", "TB200_PIN_GPU": "4"},
                1: {"CUDA_VISIBLE_DEVICES": "6", "TB200_PIN_GPU": "6"}}

    monkeypatch.setenv("CUDA_VISIBLE_DEVICES", "4,6")
    monkeypatch.delenv("TB200_PIN_GPU", raising=False)
    monkeypatch.setattr(bench, "_host_loop_worker", _env_probe)
    synced = []
    out = bench.host_loops(Box, "b200", 4, 0.01, "once", sync=lambda: synced.append(1))
    assert out["count"] == 4 and out["processes"] == 4 and out["failed_workers"] == 0 and synced == [1]
    seen = sorted(tuple(json.load(open(os.path.join(str(tmp_path), f)))) for f in os.listdir(str(tmp_path)))
    assert seen == sorted([(0, "4", "4"), (0, "6", "6")] * 2)
    assert os.environ["CUDA_VISIBLE_DEVICES"] == "4,6" and "TB200_PIN_GPU" not in os.environ


FAKE_CHILD = """#!%s
import json, os, sys, time
args = sys.argv[1:]
sync_dir = args[args.index("--sync-dir") + 1] if "--sync-dir" in args else None
if "--fail" in args:
    sys.exit("child broke before it was warm")
if sync_dir:
    open(os.path.join(sync_dir, "ready"), "w").close()
    t0 = time.time()
    while not os.path.exists(os.path.join(sync_dir, "go")):
        time.sleep(0.001)
        assert time.time() - t0 < 20
print(json.dumps({"infer_per_s": 123.0, "device": int(args[args.index("--device") + 1]), "synced": bool(sync_dir),
                  "pin": os.environ.get("TB200_PIN_GPU")}))
"""


def test_generator_child_is_released_by_the_rendezvous(monkeypatch, tmp_path):
    """LoopbackBox.generator: the child reports ready, the caller's sync runs exactly once (also when the child
    dies first), then the child is told to go; the child gets its GPU's environment and ordinal"""
    fake = tmp_path / "fake_python"
    fake.write_text(FAKE_CHILD % sys.executable)
    fake.chmod(0o755)
    import shutil

    monkeypatch.setattr(shutil, "which", lambda name: None)
    box = bench.LoopbackBox([2])
    box.urls[2] = "127.0.0.1:9"
    box.envs[2] = dict(os.environ, TB200_PIN_GPU="5")
    box.ordinal[2] = 0
    monkeypatch.setattr(sys, "executable", str(fake))
    order = []
    g = box.generator(2, 20, 5, sync=lambda: order.append("sync"))
    assert g == {"infer_per_s": 123.0, "device": 0, "synced": True, "pin": "5"} and order == ["sync"]
    assert box.generator(2, 20, 5)["synced"] is False  # no rendezvous asked for: plain run
    import pytest

    with pytest.raises(RuntimeError, match="generator child failed"):
        box.generator(2, 20, 5, extra=("--fail",), sync=lambda: order.append("sync"))
    assert order == ["sync", "sync"]  # the failing rank still met the others
