"""Which host cores belong to which GPU, and pinning a process to them.

The north star's deployment is one load-generation instance per GPU ("pinned per GPU across the
8xB200 box"); the reference offers the per-device hook only
(``create_shared_memory_region(..., device_id)``,
src/python/library/tritonclient/utils/cuda_shared_memory/__init__.py:107,131) and leaves placement
to the user.  An instance here is a few epoll threads + one device thread (generator) or the same
on the serving side, all host-bound on socket work -- so each instance gets its own slice of the
cores of the NUMA node its GPU hangs off, and the slices of different GPUs never overlap.

Source of truth: ``/sys/bus/pci/devices/<gpu bus id>/local_cpulist`` (what ``nvidia-smi topo -m``
prints as CPU affinity).  GPUs that share a CPU list split it evenly, in GPU index order; within
a GPU's slice the first half goes to the server process, the second to the generator.
"""

import os
import subprocess


def parse_cpulist(text):
    """'0-31,64-95' -> [[0..31], [64..95]] (one list per range, order kept)."""
    ranges = []
    for part in text.strip().split(","):
        part = part.strip()
        if not part:
            continue
        lo, _, hi = part.partition("-")
        ranges.append(list(range(int(lo), int(hi or lo) + 1)))
    return ranges


def gpu_cpulists():
    """[{'index': i, 'bus_id': '0000:1b:00.0', 'numa_node': n, 'ranges': [[...], ...]}, ...]
    for every visible GPU; ranges is empty when sysfs has nothing to say."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=index,pci.bus_id", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout
    except Exception:
        return []
    gpus = []
    for line in out.strip().splitlines():
        idx, _, bus = line.partition(",")
        bus = bus.strip().lower()
        if bus.count(":") == 2 and len(bus.split(":")[0]) == 8:  # nvidia-smi prints an 8-digit domain
            bus = bus[4:]
        base = "/sys/bus/pci/devices/%s" % bus
        ranges, node = [], -1
        try:
            with open(base + "/local_cpulist") as fh:
                ranges = parse_cpulist(fh.read())
            with open(base + "/numa_node") as fh:
                node = int(fh.read().strip())
        except (OSError, ValueError):
            pass
        gpus.append({"index": int(idx), "bus_id": bus, "numa_node": node, "ranges": ranges})
    return gpus


def split_ranges(ranges, parts, which):
    """Slice `which` of `parts` equal slices of every range (hyperthread siblings sit in the second
    range at the same offset, so a slice keeps cores and their siblings together)."""
    out = []
    for r in ranges:
        n = len(r) // parts
        if n == 0:
            continue
        out.extend(r[which * n:(which + 1) * n])
    return out


def plan(gpus=None, allowed=None):
    """{gpu index: {'all': [...], 'server': [...], 'generator': [...], 'numa_node': n}}.

    GPUs with the same CPU list share it in index order.  ``allowed``: the CPUs this process may
    use at all (default: its current affinity mask) -- a container's cgroup mask wins."""
    gpus = gpu_cpulists() if gpus is None else gpus
    if allowed is None:
        allowed = set(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else None
    groups = {}
    for g in gpus:
        groups.setdefault(tuple(tuple(r) for r in g["ranges"]), []).append(g)
    out = {}
    for key, members in groups.items():
        members.sort(key=lambda g: g["index"])
        for pos, g in enumerate(members):
            ranges = [[c for c in r if allowed is None or c in allowed] for r in g["ranges"]]
            ranges = [r for r in ranges if r]
            mine = split_ranges(ranges, len(members), pos) if ranges else []
            mine_ranges = [[c for c in r if c in set(mine)] for r in ranges]
            mine_ranges = [r for r in mine_ranges if r]
            out[g["index"]] = {"all": sorted(mine), "server": sorted(split_ranges(mine_ranges, 2, 0)),
                               "generator": sorted(split_ranges(mine_ranges, 2, 1)), "numa_node": g["numa_node"]}
            if not out[g["index"]]["server"] or not out[g["index"]]["generator"]:  # too few cores to split
                out[g["index"]]["server"] = out[g["index"]]["generator"] = out[g["index"]]["all"]
    return out


def pin(cpus):
    """Restrict this process (and every thread it starts afterwards) to ``cpus``; returns the
    mask in effect, [] when pinning is not possible (no cores given, platform without it)."""
    if not cpus or not hasattr(os, "sched_setaffinity"):
        return []
    try:
        os.sched_setaffinity(0, set(cpus))
        return sorted(os.sched_getaffinity(0))
    except OSError:
        return []


def physical_index(device_id):
    """The nvidia-smi index behind CUDA ordinal ``device_id``: CUDA_VISIBLE_DEVICES renumbers the devices a
    process sees, sysfs and nvidia-smi do not.  (UUID entries cannot be mapped here and leave the ordinal.)"""
    forced = os.environ.get("TB200_PIN_GPU", "").strip()  # set by whoever remapped the devices in a way this cannot see
    if forced.isdigit():                                   # (e.g. a container that exposes one board as ordinal 0)
        return int(forced)
    parts = [x.strip() for x in os.environ.get("CUDA_VISIBLE_DEVICES", "").split(",") if x.strip()]
    if parts and all(x.isdigit() for x in parts) and 0 <= int(device_id) < len(parts):
        return int(parts[int(device_id)])
    return int(device_id)


def pin_for(device_id, role):
    """Pin to the cores planned for (GPU ``device_id``, role 'server' | 'generator' | 'all')."""
    p = plan().get(physical_index(device_id))
    return pin(p[role]) if p else []
