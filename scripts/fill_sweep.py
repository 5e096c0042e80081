"""Time the fill kernel variants (tb200_tune fill_variant) on one GPU.

Usage:  python scripts/fill_sweep.py > fill_sweep.txt
For each variant: FP32 C2 step (64 x 602,112 B), FP16 C3 tensor (38,535,168 B), the C4
wire shape (512 x 3,072 B INT64) and a 256-slot launch (154 MB), all timed with CUDA
events around back-to-back launches inside one CUDA graph, rotating over > L2 of memory.
"""

import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from client_b200 import _native  # noqa: E402
from client_b200.device import DeviceBuffer, DeviceOps, make_fill_job  # noqa: E402
from oracle import cref  # noqa: E402

# negative keys: knobs of the default policy rather than a general-kernel variant
VARIANTS = {0: "default: fill_uniform_kernel + overlapped launches (PDL)", -1: "fill_uniform_kernel, launches serialised (fill_pdl=0)",
            -2: "general kernels only (fill_uniform=0): range u3 / stride", 20: "stride 256t u1 cap8", 21: "stride 256t u2 cap6",
            22: "stride 256t u2 cap16", 24: "stride 256t u4 cap4",
            101: "range 256t u2", 102: "range 256t u4", 106: "range 512t u2", 111: "range 256t u3",
            28: "stride 1 round (NOT the contract)", 110: "range 1 round (NOT the contract)", 109: "range 7 rounds (NOT the contract)"}
NOT_CONTRACT = (28, 109, 110)


def timed(ops, ctx, build, nbytes, sets=4, reps=4, iters=30):
    ops.graph_begin()
    for _ in range(reps):
        for s in range(sets):
            build(s)
    g = ops.graph_end()
    for _ in range(3):
        g.launch()
    ops.sync()
    t = _native.Timer(ctx)
    t.start()
    for _ in range(iters):
        g.launch()
    t.stop()
    ops.sync()
    ms = t.elapsed_ms() / (iters * reps * sets)
    g.close()
    return ms, nbytes / ms / 1e6


def main():
    lib = _native.load()
    ctx = _native.Context(0)
    ops = DeviceOps(ctx)
    slot = 602112
    big = DeviceBuffer(0, 4 * 64 * slot)
    c2 = [[make_fill_job(big.ptr + (s * 64 + k) * slot, slot, "FP32", stream_id=k) for k in range(64)] for s in range(4)]
    c3 = [[make_fill_job(big.ptr + s * 64 * slot, 64 * slot, "FP16", stream_id=s)] for s in range(4)]
    c4 = [[make_fill_job(big.ptr + s * 64 * slot + k * 3072, 3072, "INT64", stream_id=k, low=0, high=30522) for k in range(512)] for s in range(4)]
    all256 = [make_fill_job(big.ptr + k * slot, slot, "FP32", stream_id=k) for k in range(256)]
    print("%-52s %12s %12s %12s %12s" % ("variant", "C2 64xFP32", "C3 1xFP16", "C4 512xI64", "256xFP32"))
    for v, name in VARIANTS.items():
        _native.check(lib.tb200_tune(b"fill_variant", max(v, 0)))
        _native.check(lib.tb200_tune(b"fill_pdl", 0 if v == -1 else 1))
        if v == -2:
            _native.check(lib.tb200_tune(b"fill_uniform", 0))
        if v not in NOT_CONTRACT:  # correctness spot check
            ops.fill(c2[0][:2], seed=5)
            got = ops.download(big.ptr + slot, slot)
            assert np.array_equal(got, cref.fill(slot, "FP32", seed=5, stream=1)), name
        r = []
        r.append(timed(ops, ctx, lambda s: ops.fill_epoch(c2[s], seed=1), 64 * slot))
        r.append(timed(ops, ctx, lambda s: ops.fill_epoch(c3[s], seed=1), 64 * slot))
        r.append(timed(ops, ctx, lambda s: ops.fill_epoch(c4[s], seed=1), 512 * 3072, iters=50))
        r.append(timed(ops, ctx, lambda s: ops.fill_epoch(all256, seed=1), 256 * slot, sets=1, reps=4, iters=20))
        print("%-52s " % name + " ".join("%6.2fus%6.0f" % (ms * 1e3, gbs) for ms, gbs in r), flush=True)
    _native.check(lib.tb200_tune(b"fill_variant", 0))
    # write-only reference: cudaMemsetAsync of 256 MB (the L2-flush helper)
    t = _native.Timer(ctx)
    ops.l2_flush()
    ops.sync()
    t.start()
    for _ in range(10):
        ops.l2_flush()
    t.stop()
    ops.sync()
    print("cudaMemsetAsync 256 MiB: %.2f us  %.0f GB/s" % (t.elapsed_ms() * 100, (256 << 20) / (t.elapsed_ms() / 10) / 1e6))
    # zero-fill mode of the same kernel (no Philox at all)
    zero = [make_fill_job(big.ptr + k * slot, slot, "FP32", stream_id=k, mode="zero") for k in range(256)]
    print("zero-fill 64 slots / 256 slots: %s / %s" % (
        "%.2fus %.0f GB/s" % tuple(x * (1e3 if i == 0 else 1) for i, x in enumerate(timed(ops, ctx, lambda s: ops.fill_epoch(zero[s * 64:(s + 1) * 64]), 64 * slot))),
        "%.2fus %.0f GB/s" % tuple(x * (1e3 if i == 0 else 1) for i, x in enumerate(timed(ops, ctx, lambda s: ops.fill_epoch(zero), 256 * slot, sets=1, reps=4, iters=20)))))


if __name__ == "__main__":
    main()
