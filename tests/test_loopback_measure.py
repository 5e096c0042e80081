"""client_b200.perf.loopback.measure on the CPU: a repetition is exactly `steps` x `concurrency`
finished requests however slowly they come, and a generator that stops finishing requests fails
the measurement instead of closing a short window."""

import pytest

from client_b200.perf import loopback


class SlowGenerator:
    """Stands in for NativeLoadGenerator: every wait_count call lets `per_wait` more requests finish
    (and reports a timeout while the count is not reached), as a generator far slower than the
    wait's deadline would."""

    def __init__(self, per_wait):
        self.per_wait, self.done, self.waits = per_wait, 0, 0

    def wait_count(self, count, timeout=60.0):
        self.waits += 1
        self.done += self.per_wait
        return self.done

    def window(self, seconds):
        n, self.done = self.done, 0
        return {"count": n, "seconds": 1.0, "throughput": float(n), "failed": 0, "nonfinite": 0, "mismatches": 0}


@pytest.mark.parametrize("min_seconds,repetitions", [(0, 5), (0, 1), (0.5, 1)])
def test_every_repetition_is_the_full_count(min_seconds, repetitions):
    gen = SlowGenerator(per_wait=7)
    reps = loopback.measure(gen, concurrency=64, steps=20, warmup=0, min_seconds=min_seconds, repetitions=repetitions)
    assert len(reps) == repetitions  # with min_seconds=0.5: one 1 s window is enough
    assert all(w["count"] >= 20 * 64 for w in reps)
    assert gen.waits >= len(reps) * (20 * 64 // 7)  # many deadlines passed, no window was closed early


def test_a_stalled_generator_fails_the_measurement():
    with pytest.raises(RuntimeError, match="finished no request"):
        loopback.measure(SlowGenerator(per_wait=0), concurrency=64, steps=20, warmup=0, min_seconds=0, repetitions=5)
