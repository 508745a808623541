#!/usr/bin/env python3
"""Accuracy of an object model (run_nocs.py / run_ycbineoat.py --save_model) against a reference mesh, e.g. the object's YCB CAD model:

    accuracy      mean distance from the model's surface samples to the reference's surface samples
    completeness  mean distance from the reference's samples to the model's
    chamfer       (accuracy + completeness) / 2
    per threshold tau: precision (model samples within tau), recall (reference samples within tau) and their F-score

Both meshes are sampled uniformly by area on the device with the same seed, and every distance is the exact nearest one (DESIGN.md §3.15).
The meshes are compared in the frame they are given in, with no alignment: a run writes its model in the object's frame, and aligning it
would hide the tracking error this is meant to show.  This script only reads files.

    python scripts/eval_model.py --model /tmp/run/model.ply --reference YCB_Video_Dataset/models/006_mustard_bottle/textured.obj
"""
from __future__ import annotations

import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def evaluate(model: str, reference: str, samples: int = 100_000, taus=(0.002, 0.005, 0.01), seed: int = 0, device: int = 0, out=print) -> dict:
    """Returns metrics.SurfaceScore.score's dict (metres) plus the two paths; prints one line per threshold (millimetres)."""
    from bundletrack_b200.metrics import SurfaceScore
    from bundletrack_b200.recon import read_mesh
    mv, mf = read_mesh(model)
    rv, rf = read_mesh(reference)
    if len(mf) == 0 or len(rf) == 0:
        raise ValueError(f"{model if len(mf) == 0 else reference}: the mesh has no face")
    ss = SurfaceScore(max(len(mf), len(rf)), samples, device=device)
    try:
        res = ss.score(mv, mf, rv, rf, n_samples=samples, taus=taus, seed=seed)
    finally:
        ss.close()
    res.update(model=model, reference=reference)
    out(f"{os.path.basename(model)} vs {os.path.basename(reference)}, {samples} samples each: accuracy {res['accuracy'] * 1e3:.3f} mm, "
        f"completeness {res['completeness'] * 1e3:.3f} mm, chamfer {res['chamfer'] * 1e3:.3f} mm")
    for t, p, r, f in zip(res["taus"], res["precision"], res["recall"], res["fscore"]):
        out(f"tau {t * 1e3:g} mm: precision {p * 100:.2f} %, recall {r * 100:.2f} %, F {f * 100:.2f}")
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--model", required=True, help="the model mesh (.ply as --save_model writes it, or .obj)")
    ap.add_argument("--reference", required=True, help="the reference mesh (.obj or binary .ply), in the model's frame and in metres")
    ap.add_argument("--samples", type=int, default=100_000, help="surface samples per mesh")
    ap.add_argument("--tau", type=float, nargs="+", default=[0.002, 0.005, 0.01], help="F-score thresholds, metres")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    return evaluate(a.model, a.reference, a.samples, tuple(a.tau), a.seed, a.device)


if __name__ == "__main__":
    main()
