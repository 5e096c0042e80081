"""Sustained inferences/sec against a local CUDA-shared-memory server -- the north-star metric --
as one measurement a benchmark can call: this process is ONE load-generation instance (the native
generator, include/tb200_loadgen.h) for ONE GPU, pinned to that GPU's share of the host cores.

    python -m client_b200.perf.loopback -u 127.0.0.1:8000 --device 0 --concurrency 64 \\
        --steps 2000 --warmup 20 --input-data-mode per-request --json

A *step* is one closed-loop round of the concurrency slots: ``concurrency`` completed requests.
After ``warmup`` steps the timed region is exactly ``steps`` steps (a count window,
tb200_loadgen_wait_count); it is repeated until at least ``--min-seconds`` have been timed and the
median repetition is reported, so a caller that asks for 20 steps still gets a number that is not
ramp-up noise.  ``--min-seconds 0`` times exactly ``--repetitions`` repetitions of ``steps`` steps,
however long they take, and reports the median repetition: the work timed depends on the arguments
alone, and one stall of the host or of the GPU's time slicing moves at most one repetition.
``--input-data-mode per-request``: every request's input tensor is regenerated
on the device and every response validated on the device (no tensor byte crosses PCIe); ``once``:
regions are filled once and requests only name them (what perf_analyzer does, SURVEY.md section 10).

It runs as its own process so that (a) its threads can be pinned, (b) a benchmark process that
already owns a CUDA context does not matter.  bench.py spawns one per GPU.
"""

import argparse
import json
import sys
import time


def rendezvous(sync_dir, timeout=180.0):
    """Tell the parent this instance is warm (``ready``) and keep the loop running until it says ``go``:
    with one instance per GPU the timed regions then start together, after every instance's start-up
    (context creation and region registration of one process stall CUDA calls of the others)."""
    import os

    with open(os.path.join(sync_dir, "ready"), "w"):
        pass
    t_end = time.perf_counter() + timeout
    while not os.path.exists(os.path.join(sync_dir, "go")) and time.perf_counter() < t_end:
        time.sleep(0.001)


def timed_repetition(gen, count, stall_seconds=30.0):
    """One count window of at least `count` finished requests, however long it takes; raises when the
    generator finishes nothing for `stall_seconds` (a window is never closed short)."""
    gen.window(0.0)  # reset: the count window starts here
    last = -1
    while True:
        got = gen.wait_count(count, timeout=stall_seconds)
        if got >= count:
            break
        if got == last:
            raise RuntimeError("the generator finished no request for %.0f s (%d of %d in the window)" % (stall_seconds, got, count))
        last = got
    w = gen.window(0.0)
    if w["count"] < count:
        raise RuntimeError("count window closed at %d of %d requests" % (w["count"], count))
    return w


def measure(gen, concurrency, steps, warmup, min_seconds, max_seconds=20.0, sync_dir=None, repetitions=1):
    """[per-repetition dicts]; a repetition = exactly `steps` x `concurrency` finished requests.
    min_seconds <= 0: exactly `repetitions` repetitions, whatever their time; otherwise repetitions
    until `min_seconds` are timed (and 3 repetitions or 1 s), no new one after `max_seconds`."""
    per_rep = steps * concurrency
    gen.window(0.0)
    if warmup > 0:
        gen.wait_count(warmup * concurrency, timeout=30.0)
    if sync_dir:
        rendezvous(sync_dir)
    if min_seconds <= 0:
        return [timed_repetition(gen, per_rep) for _ in range(max(1, repetitions))]
    reps, timed, t_start = [], 0.0, time.perf_counter()
    while True:
        w = timed_repetition(gen, per_rep)
        reps.append(w)
        timed += w["seconds"]
        if (timed >= min_seconds and (len(reps) >= 3 or timed >= 1.0)) or time.perf_counter() - t_start > max_seconds:
            break
    return reps


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("-u", "--url", required=True)
    ap.add_argument("-m", "--model-name", default="densenet_onnx")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--concurrency", type=int, default=64)
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--min-seconds", type=float, default=0.1)
    ap.add_argument("--repetitions", type=int, default=1, help="with --min-seconds 0: timed repetitions of --steps steps (median reported)")
    ap.add_argument("--input-data-mode", default="per-request", choices=["per-request", "once"])
    ap.add_argument("--device-pipeline", type=int, default=3)
    ap.add_argument("--device-window-us", type=int, default=0)
    ap.add_argument("--lookahead", type=int, default=1)
    ap.add_argument("--seed", type=int, default=20260921)
    ap.add_argument("--pin-cpus", action="store_true")
    ap.add_argument("--sync-dir", default=None, help="after the warm-up create <dir>/ready and start timing when <dir>/go appears")
    ap.add_argument("--no-validate", action="store_true")
    ap.add_argument("--json", action="store_true")
    args = ap.parse_args(argv)

    pinned = []
    if args.pin_cpus:
        from .topology import pin_for

        pinned = pin_for(args.device, "generator")

    from .. import http as httpclient
    from .loadgen import SlotSet, TensorSpec
    from .native import NativeLoadGenerator

    control = httpclient.InferenceServerClient(args.url)
    md = control.get_model_metadata(args.model_name)
    inputs = [TensorSpec(t["name"], t["datatype"], [int(d) for d in t["shape"]]) for t in md["inputs"]]
    outputs = [TensorSpec(t["name"], t["datatype"], [int(d) for d in t["shape"]]) for t in md["outputs"]]
    ss = SlotSet(inputs, outputs, args.concurrency, "cuda", args.device, "random", args.seed + 1000003 * args.device,
                 name_prefix="lb_d%d_c%d" % (args.device, args.concurrency), lookahead=args.lookahead)
    ss.register(control)
    per_request = args.input_data_mode == "per-request"
    gen = NativeLoadGenerator(args.url, args.model_name, "", ss, args.concurrency, regenerate=per_request,
                              validate=per_request and not args.no_validate, device_window_us=args.device_window_us,
                              pipeline_depth=args.device_pipeline)
    gen.start()
    try:
        reps = measure(gen, args.concurrency, args.steps, args.warmup, args.min_seconds, sync_dir=args.sync_dir, repetitions=args.repetitions)
    finally:
        gen.stop()
        ss.unregister(control)
        ss.close()
        control.close()
    reps.sort(key=lambda w: w["throughput"])
    mid = reps[len(reps) // 2]
    out = {
        "device": args.device, "concurrency": args.concurrency, "steps": args.steps, "warmup": args.warmup,
        "input_data_mode": args.input_data_mode, "infer_per_s": mid["throughput"], "count": mid["count"], "seconds": mid["seconds"],
        "repetitions": len(reps), "infer_per_s_min": reps[0]["throughput"], "infer_per_s_max": reps[-1]["throughput"],
        "p50_us": mid["p50_us"], "p99_us": mid["p99_us"], "failed": sum(w["failed"] for w in reps),
        "nonfinite": sum(w["nonfinite"] for w in reps), "mismatches": sum(w["mismatches"] for w in reps),
        "device_passes": mid["device_batches"], "slots_per_device_pass": mid["device_slots"] / max(1, mid["device_batches"]),
        "gpu_launches": (2 if per_request and not args.no_validate else (1 if per_request else 0)) * mid["device_batches"],
        "pipeline_depth": args.device_pipeline, "request_input_bytes": ss.in_bytes, "cpus": len(pinned),
    }
    print(json.dumps(out) if args.json else out, flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
