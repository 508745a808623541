#!/usr/bin/env python3
"""Records tests/golden/ref_mask_score.npz: mask pairs with their DAVIS counts, J and F, and per-sequence statistics, the boundaries dilated
by OpenCV (cv2.dilate with the disk dx^2 + dy^2 <= r^2 as its kernel, as the DAVIS toolkit does) instead of the oracle's row intervals.
The device's results are held against it where OpenCV is not installed.

    python scripts/make_golden_mask_score.py [--out tests/golden/ref_mask_score.npz]
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def cv2_counts(P, G, bound_th):
    import cv2
    from oracle import mask_oracle as mo
    r = mo.radius(*P.shape, bound_th)
    y, x = np.mgrid[-r:r + 1, -r:r + 1]
    disk = (x * x + y * y <= r * r).astype(np.uint8)
    bp, bg = mo.boundary(P), mo.boundary(G)
    dp, dg = cv2.dilate(bp.astype(np.uint8), disk) > 0, cv2.dilate(bg.astype(np.uint8), disk) > 0
    P, G = P != 0, G != 0
    return [(P & G).sum(), (P | G).sum(), bp.sum(), bg.sum(), (bp & dg).sum(), (bg & dp).sum()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "ref_mask_score.npz"))
    a = ap.parse_args()
    from bundletrack_b200 import synth
    from oracle import mask_oracle as mo
    rng = np.random.default_rng(17)
    noise = [((rng.random((5, 37, 53)) < p) * 255).astype(np.uint8) for p in (0.03, 0.04)]
    cases = {"ellipses": synth.ragged_ellipse_masks(6, 480, 640, seed=3) + (0.008,), "noise": (noise[0], noise[1], 0.02)}
    out = {}
    for name, (pred, gt, th) in cases.items():
        counts = np.array([cv2_counts(p, g, th) for p, g in zip(pred, gt)], np.int64)
        jf = np.array([mo.j_and_f(c) for c in counts], np.float64)
        out.update({f"{name}_pred": pred, f"{name}_gt": gt, f"{name}_bound_th": np.float64(th), f"{name}_counts": counts,
                    f"{name}_j": jf[:, 0], f"{name}_f": jf[:, 1], f"{name}_score": np.array(list(mo.score(jf[:, 0], jf[:, 1]).values()))})
    np.savez_compressed(a.out, **out)
    print(f"{a.out}: {os.path.getsize(a.out)} bytes")


if __name__ == "__main__":
    main()
