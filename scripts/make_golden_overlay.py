#!/usr/bin/env python3
"""Writes tests/golden/ref_overlay.npz: a few synthetic LOG frames drawn by OpenCV itself, so the GPU tests need neither cv2 nor the reference.

Per frame: a BGR colour image of channel ramps, an elliptic object mask, an ellipsoid model of 8000 points (voxel-gridded at 1.5 cm as the loaders do) and a pose that puts the model near a border
or corner of the 120 x 160 image (one frame has points just behind the camera plane).  The image is built as Bundler::saveNewframeResult
builds it (Bundler.cpp:379-399): the dimming loop (uchar)(c * 0.2) where fg == 0, then cv2.circle(img, (u, v), 1, (0, 255, 255), -1) at
every centre the numpy oracle projects (oracle/overlay_oracle.py), then cv2.putText(id, (5, 30), FONT_HERSHEY_PLAIN, 2, (255, 0, 0), 1, 8).
label_mask marks the pixels the label can touch (where putText draws on a black image).

    python scripts/make_golden_overlay.py
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, W = 120, 160
K = np.array([150.0, 150.0, 80.0, 60.0], np.float32)
# object centre in the camera frame per frame: left-top corner, right border, bottom-right corner, straddling z = 0
CENTRES = [(-0.26, -0.19, 0.5), (0.32, 0.0, 0.5), (0.26, 0.19, 0.5), (0.0, 0.0, 0.02)]


def make_frames(seed: int = 0):
    from bundletrack_b200 import synth
    rng = np.random.default_rng(seed)
    F = len(CENTRES)
    vv, uu = np.mgrid[0:H, 0:W]
    colour = np.stack([np.stack([(uu * (3 + k) + vv * (5 - k) + 40 * f) % 256 for k in range(3)], -1) for f in range(F)]).astype(np.uint8)
    fg = np.zeros((F, H, W), np.uint8)
    poses = np.zeros((F, 4, 4), np.float32)
    for f, c in enumerate(CENTRES):
        fg[f] = ((((uu - 30 - 30 * f) / 40.0) ** 2 + ((vv - 60) / 30.0) ** 2) <= 1).astype(np.uint8) * 255
        R = synth.so3_exp(rng.normal(size=3) * 0.5)
        ob_in_cam = synth.se3(R, np.asarray(c, np.float64))
        poses[f] = np.linalg.inv(ob_in_cam).astype(np.float32)
    model = synth.make_ellipsoid_model(seed, 8000, radii=(0.12, 0.1, 0.08))
    ids = [f"{k:04d}" for k in range(F)]
    return colour, fg, model, poses, ids


def draw(colour, fg, model, pose, id_str):
    """(viz with label, label_mask, raw) drawn by OpenCV."""
    import cv2
    from oracle import overlay_oracle as oo
    img = colour.copy()
    for h in range(H):                         # the reference's dimming loop, pixel by pixel
        for w in range(W):
            if fg[h, w] == 0:
                img[h, w] = [int(float(c) * 0.2) for c in img[h, w]]
    for u, v in oo.project(oo.centroids(oo.voxel_grid(model, 0.015), pose), K, H, W):
        cv2.circle(img, (int(u), int(v)), 1, (0, 255, 255), -1)
    cv2.putText(img, id_str, (5, 30), cv2.FONT_HERSHEY_PLAIN, 2, (255, 0, 0), 1, 8, False)
    blank = np.zeros_like(img)
    cv2.putText(blank, id_str, (5, 30), cv2.FONT_HERSHEY_PLAIN, 2, (255, 0, 0), 1, 8, False)
    raw = np.where((fg != 0)[..., None], colour, 0).astype(np.uint8)
    return img, blank.any(-1), raw


def main():
    colour, fg, model, poses, ids = make_frames()
    out = [draw(colour[f], fg[f], model, poses[f], ids[f]) for f in range(len(ids))]
    path = os.path.join(ROOT, "tests", "golden", "ref_overlay.npz")
    np.savez_compressed(path, colour=colour, fg=fg, model=model, cur_in_model=poses, K=K, ids=np.array(ids),
                        viz=np.stack([o[0] for o in out]), label_mask=np.stack([o[1] for o in out]), raw=np.stack([o[2] for o in out]))
    print(f"wrote {path}: {len(ids)} frames of {W} x {H}, {len(model)} model points")


if __name__ == "__main__":
    main()
