"""Record tests/golden/ref_matchviz.npz: the reference's match images (SiftManager::vizCorresBetween) as OpenCV draws them, through cv2
(cv2.resize with fx = fy = scale, cv2.drawMatches with random colours and NOT_DRAW_SINGLE_POINTS, the RNG seeded with cv2.setRNGSeed).

Each case is two ROIs of the closed-form test colour (oracle.segment_oracle.test_colour), a (uA, vA, uB, vB) list and the seed; images of
the chain continue the RNG from the previous image instead of reseeding.  Images up to 128 KB are stored whole (the narrow-crop cases,
so a mismatch there shows its pixels), larger ones as the SHA-256 of their bytes.

    python scripts/make_golden_matchviz.py            # writes tests/golden/ref_matchviz.npz
"""
from __future__ import annotations

import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import matchviz_oracle as mv  # noqa: E402
from oracle.segment_oracle import test_colour  # noqa: E402

H, W = 480, 640
WHOLE_MAX = 128 * 1024


def cv_image(cv2, colour, roi_a, roi_b, uv, seed=None):
    """vizCorresBetween's picture through cv2; seed None continues theRNG."""
    ca, cb = mv.crop(colour, roi_a), mv.crop(colour, roi_b)
    s = mv.viz_scale(ca.shape[0], cb.shape[0])
    ra, rb = cv2.resize(ca, (0, 0), fx=s, fy=s), cv2.resize(cb, (0, 0), fx=s, fy=s)
    kp = mv.keypoints(uv, roi_a, roi_b, s)
    ka = [cv2.KeyPoint(float(x), float(y), 1) for x, y in kp[:, :2]]
    kb = [cv2.KeyPoint(float(x), float(y), 1) for x, y in kp[:, 2:]]
    m = [cv2.DMatch(i, i, 0) for i in range(len(kp))]
    if seed is not None:
        cv2.setRNGSeed(seed)
    return cv2.drawMatches(ra, ka, rb, kb, m, None, matchColor=(-1, -1, -1, -1), singlePointColor=(-1, -1, -1, -1),
                           flags=cv2.DrawMatchesFlags_NOT_DRAW_SINGLE_POINTS)


def cases():
    """(name, roi_a, roi_b, uv float32 [n, 4], seed) per image; a seed of 0 continues the previous image's RNG."""
    rs = np.random.default_rng(11)
    out = []
    # lines in every octant, horizontal, vertical and zero length (uv outside the ROI reach the clipping too), scale 22
    ra, rb = (100, 140, 50, 90), (300, 340, 200, 240)
    c = np.array([120.0, 70.0], np.float32)
    uv = []
    for ang in range(0, 360, 15):
        d = np.array([np.cos(np.deg2rad(ang)), np.sin(np.deg2rad(ang))]) * 15
        uv.append([c[0], c[1], rb[0] + (c[0] - ra[0]) - 40 + d[0], rb[2] + (c[1] - ra[2]) + d[1]])
    uv += [[110.25, 60.5, 300 + 10.25 - 40, 200 + 10.5],        # zero length: kp2 lands on kp1
           [130.0, 55.0, 300 + 30.0 - 40, 200 + 30.0],          # vertical
           [105.0, 80.0, 330.0, 200 + 30.0]]                    # horizontal
    out.append(("octants", ra, rb, np.array(uv, np.float32), 12345))
    # keypoints on and next to the seam, the cols - 1 clamp, circles cut by their half
    ra, rb = (10, 60, 100, 130), (200, 230, 100, 130)
    uv = [[59.9, 110.0, 200.0, 110.0], [59.5, 129.9, 200.1, 100.0], [10.0, 100.0, 229.99, 129.99], [58.0, 115.0, 229.5, 115.0],
          [59.999, 100.0, 229.999, 100.0], [35.0, 129.5, 215.0, 129.5]]
    out.append(("seam", ra, rb, np.array(uv, np.float32), 7))
    # unequal heights (zero padding under the shorter crop), scale 3
    ra, rb = (0, 80, 0, 300), (400, 520, 380, 420)
    n = 40
    uv = np.stack([rs.uniform(0, 80, n), rs.uniform(0, 300, n), rs.uniform(400, 520, n), rs.uniform(380, 420, n)], 1)
    out.append(("unequal", ra, rb, uv.astype(np.float32), 99))
    # scale 1 (over 450 rows) with one match, and with none
    ra, rb = (20, 140, 10, 470), (300, 420, 0, 455)
    out.append(("scale1_one", ra, rb, np.array([[80.5, 200.25, 350.75, 300.125]], np.float32), 1))
    out.append(("scale1_none", ra, rb, np.zeros((0, 4), np.float32), 1))
    # about 3000 overlapping matches in a small ROI pair: the drawing order decides every pixel
    ra, rb = (200, 260, 200, 250), (210, 270, 205, 255)
    n = 3000
    uv = np.stack([rs.uniform(200, 260, n), rs.uniform(200, 250, n), rs.uniform(210, 270, n), rs.uniform(205, 255, n)], 1)
    out.append(("dense3000", ra, rb, uv.astype(np.float32), 4242))
    # the RNG carried across three consecutive images (the later ones are not reseeded)
    for k in range(3):
        ra, rb = (50 + 10 * k, 110 + 10 * k, 60, 100 + 5 * k), (250, 330, 70, 130)
        n = 5 + 7 * k
        uv = np.stack([rs.uniform(ra[0], ra[1], n), rs.uniform(ra[2], ra[3], n), rs.uniform(rb[0], rb[1], n), rs.uniform(rb[2], rb[3], n)], 1)
        out.append((f"chain{k}", ra, rb, uv.astype(np.float32), 31337 if k == 0 else 0))
    # small enough to store whole: narrow crops at scale 1 (460 x 40 pixels) and at scale 3 (900 x 36 pixels), a few matches each
    ra, rb = (100, 120, 10, 470), (300, 320, 0, 455)
    uv = [[101.0, 20.0, 301.0, 30.0], [119.5, 460.0, 300.0, 454.5], [110.25, 240.75, 310.5, 100.25], [115.0, 300.0, 305.0, 300.0],
          [100.0, 469.0, 319.0, 0.0]]
    out.append(("small_scale1", ra, rb, np.array(uv, np.float32), 555))
    ra, rb = (200, 206, 100, 400), (400, 406, 150, 450)
    uv = [[200.0, 100.0, 405.9, 449.9], [203.5, 250.0, 402.5, 250.0], [205.99, 399.5, 400.0, 150.0]]
    out.append(("small_scale3", ra, rb, np.array(uv, np.float32), 777))
    return out


def main():
    import cv2
    colour = test_colour(H, W)
    rec = {"cv2_version": np.array(cv2.__version__), "H": np.array(H), "W": np.array(W)}
    names = []
    for name, ra, rb, uv, seed in cases():
        img = cv_image(cv2, colour, ra, rb, uv, seed if seed else None)
        names.append(name)
        rec[f"{name}/roi_a"] = np.array(ra, np.int32)
        rec[f"{name}/roi_b"] = np.array(rb, np.int32)
        rec[f"{name}/uv"] = uv
        rec[f"{name}/seed"] = np.array(seed, np.int64)
        rec[f"{name}/shape"] = np.array(img.shape, np.int64)
        if img.nbytes <= WHOLE_MAX:
            rec[f"{name}/image"] = img
        else:
            rec[f"{name}/sha256"] = np.array(hashlib.sha256(np.ascontiguousarray(img).tobytes()).hexdigest())
    rec["names"] = np.array(names)
    path = os.path.join(ROOT, "tests", "golden", "ref_matchviz.npz")
    np.savez_compressed(path, **rec)
    print(f"wrote {path}: {len(names)} images, cv2 {cv2.__version__}")


if __name__ == "__main__":
    main()
