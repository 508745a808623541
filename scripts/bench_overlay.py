#!/usr/bin/env python3
"""Cost of the LOG frames (bundletrack_b200.overlay):

    device      bt_pose_overlay's device time per frame (CUDA events on its stream) for models of 1 k, 10 k and 100 k points drawn as given,
                one frame per call and 100 frames per call, 640 x 480 frames
    host        the same work per frame through the numpy oracle (oracle/overlay_oracle.py: transform, 1 cm voxel grid, projection, dimming)
                plus cv2.circle per centroid, on the host's cores.  PCL is not available, so this stands in for the reference's pattern
                (pcl::transformPointCloudWithNormals + pcl::VoxelGrid + the host loop)
    sequence    run_sequence's per-frame wall time with log off and on, on scripts/bench_run_sequence.py's synthetic scene (640 x 480, 2000
                features), the two alternated twice

Prints the card's name and power limit with the numbers, then one JSON line.

    python scripts/bench_overlay.py [--frames 300] [--out_json path]
"""
from __future__ import annotations

import argparse
import json
import os
import tempfile
import time

import numpy as np

import benchkit


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--feats", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out_json", default=None)
    a = ap.parse_args()
    import torch
    from bench_run_sequence import stats
    from bundletrack_b200 import sequence, synth
    from bundletrack_b200.overlay import Overlay
    from oracle import overlay_oracle as oo
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    dev = torch.device("cuda", 0)
    H, W, K = 480, 640, (590.0, 590.0, 322.5, 244.1)
    rng = np.random.default_rng(0)
    F = 100
    colour = [torch.from_numpy(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).to(dev) for _ in range(F)]
    fg = [torch.from_numpy((rng.random((H, W)) < 0.3).astype(np.uint8)).to(dev) for _ in range(F)]
    viz = [torch.empty((H, W, 3), dtype=torch.uint8, device=dev) for _ in range(F)]
    raw = [torch.empty_like(v) for v in viz]
    poses = []
    for _ in range(F):
        ob_in_cam = synth.se3(synth.so3_exp(rng.normal(size=3)), np.array([rng.uniform(-0.1, 0.1), rng.uniform(-0.1, 0.1), rng.uniform(0.5, 0.9)]))
        poses.append(np.linalg.inv(ob_in_cam).astype(np.float32))
    poses = np.stack(poses)
    out = {"card": benchkit.card(), "torch_device": torch.cuda.get_device_name(0), "H": H, "W": W, "device": {}, "host": {}}
    stream = torch.cuda.Stream(dev)
    for n in (1000, 10000, 100000):
        model = synth.make_ellipsoid_model(n, n, radii=(0.12, 0.09, 0.07))
        ov = Overlay(model, K, H, W, max_frames=F, stream=stream.cuda_stream, leaf=None)
        try:
            for per_call in (1, F):
                ms = benchkit.window_ms(lambda: ov.render(poses[:per_call], colour[:per_call], fg[:per_call], viz[:per_call], raw[:per_call]),
                                        a.reps, 3, stream)
                out["device"][f"{n}_pts_{per_call}_per_call_ms_per_frame"] = ms / per_call
        finally:
            ov.close()
        try:
            import cv2
        except ImportError:
            cv2 = None
        if cv2 is not None:
            c0, f0 = colour[0].cpu().numpy(), fg[0].cpu().numpy()
            t = []
            for r in range(5):
                t0 = time.perf_counter()
                img = oo.dim(c0, f0)
                for u, v in oo.project(oo.voxel_grid(oo.transform(model, oo.inverse4(poses[r])), 0.01), K, H, W):
                    cv2.circle(img, (int(u), int(v)), 1, (0, 255, 255), -1)
                t.append(time.perf_counter() - t0)
            out["host"][f"{n}_pts_ms_per_frame"] = float(np.median(t) * 1000)
        else:
            out["host"][f"{n}_pts_ms_per_frame"] = "not measured: no cv2"

    # run_sequence with log off and on
    N = a.frames
    seq = synth.make_sequence(7, N, H=H, W=W, n_feats=a.feats)
    features = synth.recorded_features(seq)
    with tempfile.TemporaryDirectory() as tmp:
        nocs, masks = synth.write_nocs_scene(seq, tmp, obj_points=synth.make_ellipsoid_model(1, 20000, radii=seq.radii))
        loader = sequence.NocsScene(nocs, 1, "camera_bench_norm", masks)
        sequence.run_sequence(loader, None, features, f"{tmp}/warm", max_feats=a.feats, log=1)
        runs = {0: [], 1: []}
        for rep in range(2):
            for log in (0, 1):
                res = sequence.run_sequence(loader, None, features, f"{tmp}/log{log}_{rep}", max_feats=a.feats, log=log)
                runs[log] += [r[2] for r in res]
    out["sequence"] = {"frames": N, "feats": a.feats, "model_pts_obj": 20000, "log0": stats(runs[0]), "log1": stats(runs[1])}
    print(f"card: {out['card']}")
    for k, v in out["device"].items():
        print(f"device {k:40s} {v:8.4f} ms")
    for k, v in out["host"].items():
        print(f"host   {k:40s} {v if isinstance(v, str) else f'{v:8.3f} ms'}")
    for k in ("log0", "log1"):
        s = out["sequence"][k]
        print(f"run_sequence {k}: median {s['median_ms']:.3f} ms  p90 {s['p90_ms']:.3f} ms")
    line = json.dumps(out)
    print(line)
    if a.out_json:
        os.makedirs(os.path.dirname(os.path.abspath(a.out_json)), exist_ok=True)
        with open(a.out_json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
