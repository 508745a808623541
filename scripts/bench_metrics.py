#!/usr/bin/env python3
"""Per-frame time of bt_pose_metrics (ADD + ADD-S, exact nearest neighbour on the device) against the reference's way, a scipy cKDTree per
frame queried on all host cores, for model sizes of a YCB points.xyz (2 600) up to 100 000 points.  Prints one JSON line (--out also writes it).

    python scripts/bench_metrics.py [--frames 1000] [--sizes 2600,30000,100000] [--kdtree_frames 50] [--reps 3]
"""
from __future__ import annotations

import argparse
import json
import os
import time

import numpy as np

import benchkit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--sizes", default="2600,30000,100000")
    ap.add_argument("--kdtree_frames", type=int, default=50, help="frames timed for the cKDTree baseline (per-frame time is the mean)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from scipy.spatial import cKDTree
    from bundletrack_b200 import synth
    from bundletrack_b200.metrics import PoseMetrics
    assert torch.cuda.is_available(), "bench_metrics measures the device call: it needs cuda:0"
    sizes = [int(s) for s in a.sizes.split(",")]
    rng = np.random.default_rng(0)
    F = a.frames
    gt, pred = np.zeros((F, 4, 4)), np.zeros((F, 4, 4))
    for f in range(F):
        Q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        gt[f] = synth.se3(Q * np.sign(np.linalg.det(Q)), np.array([0, 0, 0.7]) + rng.normal(0, 0.05, 3))
        pred[f] = synth.se3(synth.so3_exp(rng.normal(size=3) * np.deg2rad(3.0)), rng.normal(0, 0.01, 3)) @ gt[f]
    pm = PoseMetrics(max(sizes), F)
    res = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": benchkit.card(), "frames": F, "sizes": {}}
    for n in sizes:
        d = rng.normal(size=(n, 3))
        P = d / np.linalg.norm(d, axis=1, keepdims=True) * np.array([0.05, 0.08, 0.03])
        Pd = torch.from_numpy(P).cuda()
        pm(Pd, pred[:8], gt[:8])                                          # warm-up
        times = []
        for _ in range(a.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            add, adds = pm(Pd, pred, gt)                                  # ends in a stream synchronise
            times.append(time.perf_counter() - t0)
        kf = min(a.kdtree_frames, F)
        t0 = time.perf_counter()
        ref = np.zeros(kf)
        for f in range(kf):
            pp, gp = P @ pred[f, :3, :3].T + pred[f, :3, 3], P @ gt[f, :3, :3].T + gt[f, :3, 3]
            ref[f] = cKDTree(pp).query(gp, k=1, workers=-1)[0].mean()
        t_kd = (time.perf_counter() - t0) / kf
        dev_ms = 1e3 * float(np.median(times)) / F
        res["sizes"][str(n)] = {"device_ms_per_frame": round(dev_ms, 5), "device_call_s": round(float(np.median(times)), 4),
                                "kdtree_ms_per_frame": round(1e3 * t_kd, 4), "speedup": round(1e3 * t_kd / dev_ms, 1),
                                "pairs_per_s": float(n) * n * F / float(np.median(times)), "max_abs_diff_vs_kdtree": float(np.abs(adds[:kf] - ref).max())}
    pm.close()
    res["host_cores"] = os.cpu_count()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
