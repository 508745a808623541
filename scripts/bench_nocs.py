#!/usr/bin/env python3
"""Device time of one bt_nocs_metrics call for 10^4 and 10^5 NOCS records (CUDA events around the call, median of 3 after a warm-up),
next to the numpy oracle's host time for the same records.  Prints one JSON line per size with the card's name and power limit.

    python scripts/bench_nocs.py [--sizes 10000 100000]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _records(n: int, seed: int = 0):
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.normal(size=(n, 3, 3)))
    Q *= np.sign(np.linalg.det(Q))[:, None, None]
    G = np.tile(np.eye(4), (n, 1, 1))
    G[:, :3, :3] = Q * rng.uniform(0.1, 0.4, (n, 1, 1))
    G[:, :3, 3] = rng.uniform(-200, 200, (n, 3)) + [0, 0, 800]
    D, _ = np.linalg.qr(np.eye(3) + rng.normal(size=(n, 3, 3)) * 0.05)
    D *= np.sign(np.linalg.det(D))[:, None, None]
    P = np.tile(np.eye(4), (n, 1, 1))
    P[:, :3, :3] = D @ Q
    P[:, :3, 3] = G[:, :3, 3] + rng.normal(size=(n, 3)) * 30
    e = rng.uniform(40, 160, (n, 1, 3))
    C = np.array([[sx, sy, sz] for sx in (1, -1) for sy in (1, -1) for sz in (1, -1)], np.float64)[None] * e
    sym = rng.integers(1, 7, n)
    return P, G, C, np.isin(sym, (1, 2, 4)).astype(np.int32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[10000, 100000])
    a = ap.parse_args()
    import ctypes
    import torch
    from bundletrack_b200 import _lib, metrics
    from oracle import nocs_oracle
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        card = q.stdout.strip().splitlines()[0]
    except Exception:
        card = torch.cuda.get_device_name(0)
    m = metrics.NocsMetrics(max(a.sizes))
    lib = _lib.load()
    for n in a.sizes:
        P, G, C, S = _records(n)
        out = torch.empty((3, n), dtype=torch.float64, device="cuda")
        p = lambda x: x.ctypes.data_as(ctypes.c_void_p)
        Cf = np.ascontiguousarray(C.reshape(-1))

        def call():
            _lib.check(lib.bt_nocs_metrics(m.ctx, p(P), p(G), p(Cf), p(S), ctypes.c_int(n), ctypes.c_void_p(out[0].data_ptr()),
                                           ctypes.c_void_p(out[1].data_ptr()), ctypes.c_void_p(out[2].data_ptr()), None), "bt_nocs_metrics")
        call()
        torch.cuda.synchronize()
        dev_ms = []
        for _ in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            h0 = time.perf_counter()
            e0.record()
            call()
            e1.record()
            torch.cuda.synchronize()
            dev_ms.append((e0.elapsed_time(e1), (time.perf_counter() - h0) * 1e3))
        nocs_oracle.record_metrics(P[:100], G[:100], C[:100], S[:100])
        host_ms = []
        for _ in range(3):
            h0 = time.perf_counter()
            nocs_oracle.record_metrics(P, G, C, S)
            host_ms.append((time.perf_counter() - h0) * 1e3)
        print(json.dumps({"records": n, "card": card, "device_call_ms_median": float(np.median([d[0] for d in dev_ms])),
                          "host_wall_ms_median": float(np.median([d[1] for d in dev_ms])), "oracle_numpy_ms_median": float(np.median(host_ms))}))
    m.close()


if __name__ == "__main__":
    main()
