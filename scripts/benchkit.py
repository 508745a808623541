"""The measurement helpers of the scripts/bench_*.py: the card a number was taken on, and device time from CUDA events.

Importing it puts the repository root and scripts/ on sys.path, so a bench script imports the package, the oracles and its sibling
scripts from wherever it is started."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (os.path.join(ROOT, "scripts"), ROOT):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402


def card() -> str:
    """Name, power limit and maximum SM clock of GPU 0, read from nvidia-smi: a time means something only next to the card and the power
    limit it was taken at.  A failed query does not stop the benchmark: the result is then torch's device name and the reason."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30, check=True)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:
        return f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable: {e})"


def _events(stream):
    """Two timing events and the torch stream to record them on.  stream is the one the measured call runs on: a torch stream, or a raw
    cudaStream_t as a facade's .stream holds it (0 is the legacy default stream, torch's default stream)."""
    if not isinstance(stream, torch.cuda.Stream):
        handle = getattr(stream, "value", stream)
        stream = torch.cuda.ExternalStream(handle) if handle else torch.cuda.default_stream()
    return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True), stream


def window_ms(fn, reps: int, warmup: int, stream) -> float:
    """Device ms per call of fn: warmup calls, then reps calls back to back between two events on stream."""
    e0, e1, s = _events(stream)
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0.record(s)
    for _ in range(reps):
        fn()
    e1.record(s)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def calls_ms(fn, reps: int, warmup: int, stream) -> list:
    """Device ms of each of reps calls of fn after warmup calls: events around every call on stream, a synchronise after each."""
    e0, e1, s = _events(stream)
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        e0.record(s)
        fn()
        e1.record(s)
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1))
    return out
