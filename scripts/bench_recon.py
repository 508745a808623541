#!/usr/bin/env python3
"""Cost of the object model (bundletrack_b200.recon):

    device      bt_tsdf_fuse and bt_tsdf_mesh per call (CUDA events on their stream, so fuse's bounds read-back and mesh's count read-back are
                inside), 640 x 480 depth maps of an ellipsoid with 0.12 / 0.09 / 0.07 m semi-axes seen from 30, 100 and 200 views spread over a
                sphere 0.5 m around it, at 2 mm and 1 mm voxels (trunc four voxels)
    sequence    run_sequence's wall time per frame without and with model_out (the whole run over its frames, so the fuse and mesh after
                the last frame count), on a synthetic 640 x 480 sequence, the two alternated twice

Prints the card's name and power limit with the numbers, then one JSON line.

    python scripts/bench_recon.py [--frames 100] [--out_json path]
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import tempfile
import time

import numpy as np

import benchkit


def sphere_views(n: int, dist: float):
    """ob_in_cam [n,4,4]: cameras on a Fibonacci sphere of radius dist, each looking at the origin."""
    out = []
    for k in range(n):
        z = 1 - 2 * (k + 0.5) / n
        phi = k * np.pi * (3 - np.sqrt(5))
        d = np.array([np.sqrt(1 - z * z) * np.cos(phi), np.sqrt(1 - z * z) * np.sin(phi), z])
        c = dist * d
        zc = -d
        up = np.array([0.0, 0.0, 1.0]) if abs(zc[2]) < 0.9 else np.array([0.0, 1.0, 0.0])
        x = np.cross(up, zc)
        x /= np.linalg.norm(x)
        R = np.stack([x, np.cross(zc, x), zc])
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = R, -R @ c
        out.append(T)
    return np.stack(out)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--frames", type=int, default=100, help="frames of the run_sequence leg")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out_json", default=None)
    a = ap.parse_args()
    import torch
    from bundletrack_b200 import _lib, recon, sequence, synth
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    dev = torch.device("cuda", 0)
    H, W, K = 480, 640, (590.0, 590.0, 319.5, 239.5)
    radii = (0.12, 0.09, 0.07)
    out = {"card": benchkit.card(), "torch_device": torch.cuda.get_device_name(0), "H": H, "W": W, "radii": radii, "device": {}}
    stream = torch.cuda.Stream(dev)
    T = sphere_views(200, 0.5)
    rng = np.random.default_rng(0)
    depths = [torch.from_numpy(synth.render_ellipsoid(radii, T[k], K, H, W, rng)[0]).to(dev) for k in range(len(T))]
    cim = np.stack([np.linalg.inv(t) for t in T]).astype(np.float32)
    torch.cuda.synchronize()
    tsdf = recon.Tsdf(200, H, W, max_voxels=1 << 25, max_vertices=1 << 22, max_faces=1 << 23, stream=stream.cuda_stream)
    lib = tsdf.lib
    try:
        for n in (30, 100, 200):
            sel = np.linspace(0, 199, n).round().astype(int)       # spread over the sphere
            d = [depths[k] for k in sel]
            for voxel in (0.002, 0.001):
                nv, nf = ctypes.c_int(0), ctypes.c_int(0)
                tf = benchkit.calls_ms(lambda: tsdf.fuse(d, cim[sel], K, voxel, 4 * voxel), a.reps, 2, stream)
                tm = benchkit.calls_ms(lambda: _lib.check(lib.bt_tsdf_mesh(tsdf.ctx, _lib.ptr(tsdf.verts), _lib.ptr(tsdf.faces), ctypes.byref(nv),
                                                                           ctypes.byref(nf), tsdf.stream)), a.reps, 2, stream)
                dims = tsdf.grid()["dims"]
                out["device"][f"{n}_frames_{voxel * 1000:g}mm"] = {"fuse_ms": float(np.median(tf)), "mesh_ms": float(np.median(tm)), "dims": dims,
                                                                   "samples": int(np.prod(dims)), "verts": nv.value, "faces": nf.value}
    finally:
        tsdf.close()

    N = a.frames
    seq = synth.make_sequence(9, N, H=H, W=W, n_feats=1000, rot_deg=(3.0, 6.0))
    features = synth.recorded_features(seq)
    with tempfile.TemporaryDirectory() as tmp:
        synth.write_ycbineoat_video(seq, f"{tmp}/video")
        loader = sequence.YcbineoatVideo(f"{tmp}/video")
        sequence.run_sequence(loader, None, features, f"{tmp}/warm", max_feats=1000, model_out=f"{tmp}/warm.ply")
        runs = {"without": [], "with": []}
        for rep in range(2):
            for key in ("without", "with"):
                t0 = time.perf_counter()
                sequence.run_sequence(loader, None, features, f"{tmp}/{key}{rep}", max_feats=1000,
                                      model_out=f"{tmp}/{key}{rep}.ply" if key == "with" else None)
                runs[key].append((time.perf_counter() - t0) / N * 1000)
    out["sequence"] = {"frames": N, "feats": 1000, "without_ms_per_frame": runs["without"], "with_ms_per_frame": runs["with"]}
    print(f"card: {out['card']}")
    for k, v in out["device"].items():
        print(f"{k:18s} dims {str(v['dims']):18s} fuse {v['fuse_ms']:8.3f} ms  mesh {v['mesh_ms']:8.3f} ms  ({v['verts']} verts, {v['faces']} faces)")
    print(f"run_sequence per frame without model_out {runs['without']} ms, with {runs['with']} ms")
    line = json.dumps(out)
    print(line)
    if a.out_json:
        os.makedirs(os.path.dirname(os.path.abspath(a.out_json)), exist_ok=True)
        with open(a.out_json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
