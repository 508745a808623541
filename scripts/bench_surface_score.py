#!/usr/bin/env python3
"""Cost of scoring an object model against a reference mesh (bundletrack_b200.metrics.SurfaceScore, DESIGN.md §3.15):

    sample      bt_mesh_sample of N points on a mesh of about 80 000 faces (an ellipsoid with 0.06 / 0.045 / 0.035 m semi-axes), per call;
                the call's one read-back (the face check and the CDF's total) is inside
    distances   bt_surface_distances of N x N points both ways: the model's samples against those of the same ellipsoid grown by 2 mm
    rate        distance tests per second: 2 N^2 over the distances time (every pair passes the fp32 filter; the float64 reranks are extra)

at N = 10^5 and 10^6, each timed with CUDA events on the facade's stream after a warm-up call.  Prints the card's name and power limit with
the numbers, then one JSON line.

    python scripts/bench_surface_score.py [--sizes 100000 1000000] [--reps 5] [--out_json path]
"""
from __future__ import annotations

import argparse
import json

import numpy as np

import benchkit


def ellipsoid(radii, n_lat: int = 200, n_lon: int = 200):
    """A closed triangulated ellipsoid: poles plus n_lat - 1 rings of n_lon vertices."""
    th = np.pi * np.arange(1, n_lat) / n_lat
    ph = 2 * np.pi * np.arange(n_lon) / n_lon
    ring = np.stack([np.sin(th)[:, None] * np.cos(ph), np.sin(th)[:, None] * np.sin(ph), np.repeat(np.cos(th)[:, None], n_lon, 1)], -1).reshape(-1, 3)
    v = np.concatenate([[[0, 0, 1]], ring, [[0, 0, -1]]]) * np.asarray(radii)
    idx = lambda i, j: 1 + i * n_lon + (j % n_lon)
    f = [(0, idx(0, j), idx(0, j + 1)) for j in range(n_lon)]
    for i in range(n_lat - 2):
        for j in range(n_lon):
            f += [(idx(i, j), idx(i + 1, j), idx(i + 1, j + 1)), (idx(i, j), idx(i + 1, j + 1), idx(i, j + 1))]
    f += [(len(v) - 1, idx(n_lat - 2, j + 1), idx(n_lat - 2, j)) for j in range(n_lon)]
    return v, np.asarray(f, np.int32)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out_json", default=None)
    a = ap.parse_args()
    import torch
    from bundletrack_b200.metrics import SurfaceScore
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    radii = np.array([0.06, 0.045, 0.035])
    mv, mf = ellipsoid(radii)
    rv, rf = ellipsoid(radii + 0.002)
    ss = SurfaceScore(len(mf), max(a.sizes))

    def timed(fn):
        t = [ms * 1e-3 for ms in benchkit.calls_ms(fn, a.reps, 1, ss.stream)]
        return float(np.median(t)), t

    name = benchkit.card()
    res = {"card": name, "faces": len(mf), "sizes": {}}
    print(f"card: {name}; meshes of {len(mf)} faces")
    for n in a.sizes:
        pa = ss.sample(mv, mf, n, 0)
        pb = ss.sample(rv, rf, n, 0)
        t_sample, _ = timed(lambda: ss.sample(mv, mf, n, 0))
        d_ab = torch.empty(n, dtype=torch.float64, device=pa.device)
        d_ba = torch.empty(n, dtype=torch.float64, device=pa.device)
        lib = ss.lib

        def dist():
            rc = lib.bt_surface_distances(ss.ctx, pa.data_ptr(), n, pb.data_ptr(), n, d_ab.data_ptr(), d_ba.data_ptr(), ss.stream)
            assert rc == 0, rc

        t_dist, all_t = timed(dist)
        rate = 2.0 * n * n / t_dist
        acc = float(d_ab.mean().item())
        res["sizes"][str(n)] = {"sample_s": t_sample, "distances_s": t_dist, "distances_all_s": all_t, "tests_per_s": rate, "accuracy_m": acc}
        print(f"N = {n}: sample {t_sample * 1e3:.3f} ms, distances (both ways) {t_dist * 1e3:.2f} ms, {rate:.3e} distance tests/s, "
              f"mean model->ref {acc * 1e3:.4f} mm")
    ss.close()
    line = json.dumps(res)
    print(line)
    if a.out_json:
        with open(a.out_json, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
