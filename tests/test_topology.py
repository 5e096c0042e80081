"""perf/topology.py: the per-GPU core plan (no GPU needed: the sysfs facts are passed in)."""

import os

from client_b200.perf import topology


def _gpus():
    # an 8-GPU box with two NUMA nodes: GPU0-3 -> 0-31,64-95; GPU4-7 -> 32-63,96-127
    a, b = topology.parse_cpulist("0-31,64-95"), topology.parse_cpulist("32-63,96-127")
    return [{"index": i, "bus_id": "x", "numa_node": 0 if i < 4 else 1, "ranges": a if i < 4 else b} for i in range(8)]


def test_parse_cpulist():
    assert topology.parse_cpulist("0-3,8,10-11\n") == [[0, 1, 2, 3], [8], [10, 11]]


def test_plan_slices_are_disjoint_and_numa_local():
    plan = topology.plan(_gpus(), allowed=set(range(128)))
    seen = set()
    for i in range(8):
        p = plan[i]
        assert len(p["all"]) == 16 and not (set(p["all"]) & seen)
        seen |= set(p["all"])
        node_cpus = set(range(0, 32)) | set(range(64, 96)) if i < 4 else set(range(32, 64)) | set(range(96, 128))
        assert set(p["all"]) <= node_cpus
        assert len(p["server"]) == 8 and len(p["generator"]) == 8 and not set(p["server"]) & set(p["generator"])
        assert set(p["server"]) | set(p["generator"]) == set(p["all"])
        # a core and its hyperthread sibling (cpu + 64) stay in the same slice
        assert {c + 64 for c in p["server"] if c < 64} == {c for c in p["server"] if c >= 64}
    assert plan[0]["all"][:8] == list(range(0, 8)) and plan[3]["all"][:8] == list(range(24, 32))
    assert seen == set(range(128))


def test_plan_respects_the_allowed_mask_and_small_boxes():
    plan = topology.plan(_gpus()[:1], allowed={0, 1, 2, 3, 64, 65, 66, 67})
    assert plan[0]["all"] == [0, 1, 2, 3, 64, 65, 66, 67]
    assert plan[0]["server"] == [0, 1, 64, 65] and plan[0]["generator"] == [2, 3, 66, 67]
    tiny = topology.plan([{"index": 0, "bus_id": "x", "numa_node": -1, "ranges": [[5]]}], allowed={5})
    assert tiny[0]["server"] == tiny[0]["generator"] == [5]


def test_pin_changes_and_restores_the_affinity_mask():
    before = sorted(os.sched_getaffinity(0))
    try:
        assert topology.pin(before[:1]) == before[:1]
        assert topology.pin([]) == []
    finally:
        os.sched_setaffinity(0, set(before))


def test_physical_index_follows_cuda_visible_devices(monkeypatch):
    from client_b200.perf import topology

    monkeypatch.delenv("CUDA_VISIBLE_DEVICES", raising=False)
    monkeypatch.delenv("TB200_PIN_GPU", raising=False)
    assert topology.physical_index(3) == 3
    monkeypatch.setenv("CUDA_VISIBLE_DEVICES", "5")
    assert topology.physical_index(0) == 5
    monkeypatch.setenv("CUDA_VISIBLE_DEVICES", "2, 6,7")
    assert [topology.physical_index(i) for i in range(3)] == [2, 6, 7]
    assert topology.physical_index(4) == 4  # out of range: left alone
    monkeypatch.setenv("CUDA_VISIBLE_DEVICES", "GPU-8f6c1e2a")
    assert topology.physical_index(0) == 0
    monkeypatch.setenv("CUDA_VISIBLE_DEVICES", "0")  # a container that exposes board 6 as its only device
    monkeypatch.setenv("TB200_PIN_GPU", "6")
    assert topology.physical_index(0) == 6


def test_loopback_rendezvous_waits_for_go(tmp_path):
    """client_b200/perf/loopback.py: an instance reports `ready` and starts timing only when `go` appears"""
    import threading
    import time

    from client_b200.perf import loopback

    def release():
        while not (tmp_path / "ready").exists():
            time.sleep(0.001)
        time.sleep(0.05)
        (tmp_path / "go").write_text("")

    th = threading.Thread(target=release)
    th.start()
    t0 = time.perf_counter()
    loopback.rendezvous(str(tmp_path), timeout=5.0)
    assert time.perf_counter() - t0 >= 0.05 and (tmp_path / "ready").exists()
    th.join()
    t0 = time.perf_counter()
    loopback.rendezvous(str(tmp_path / "missing_parent") if False else str(tmp_path), timeout=0.2)  # go already there: returns at once
    assert time.perf_counter() - t0 < 0.1
