"""Records tests/golden/ref_segment.npz: the reference's object-mask segmentation and LF-Net request computed with OpenCV itself
(cv2, CPU), statement by statement as src/Frame.cpp:267-374 and src/FeatureManager.cpp:813-873 run it, for masks from
synth.make_object_mask in both modes at 480 x 640 and at odd sizes.  The colour image is oracle.segment_oracle.test_colour (closed
form), so only the masks and the outputs are stored.  Each 400 x 400 x 3 request is stored as the SHA-256 digest of its bytes:
the tests compare the digest of what they compute, which is still a byte-for-byte check, at 32 bytes instead of 480 KB per case.
The reference picks the largest component by iterating an unordered_map, so a tie would be unpinned: every recorded case asserts
that its largest component is unique.

    python scripts/make_golden_segment.py        (needs cv2; writes tests/golden/ref_segment.npz)
"""
import hashlib
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bundletrack_b200 import synth  # noqa: E402
from oracle import segment_oracle as so  # noqa: E402

# (seed, H, W, mode, mask variant): "bin" = 0/255, "grey" = the PNG's own values vary per pixel (as-is mode keeps them in fg)
CASES = [
    (0, 480, 640, 1, "bin"), (1, 480, 640, 1, "bin"), (2, 480, 640, 1, "bin"), (3, 480, 640, 1, "bin"),
    (4, 480, 640, 0, "bin"), (5, 480, 640, 0, "grey"), (6, 480, 640, 0, "bin"), (7, 480, 640, 1, "grey"),
    (8, 97, 131, 1, "bin"), (9, 97, 131, 0, "bin"), (10, 131, 97, 1, "bin"), (11, 131, 97, 0, "grey"),
    (12, 33, 257, 1, "bin"), (13, 257, 33, 0, "bin"), (14, 480, 640, 1, "empty"), (15, 61, 47, 1, "bin"),
]


def make_mask(seed, H, W, variant):
    if variant == "empty":
        return np.zeros((H, W), np.uint8)
    m = synth.make_object_mask(seed, H, W)
    if variant == "grey":
        y, x = np.mgrid[0:H, 0:W]
        m = np.where(m != 0, (x * 7 + y * 3) % 250 + 1, 0).astype(np.uint8)
    return m


def reference(mask, mode, colour):
    H, W = mask.shape
    m = mask.copy()
    if mode == so.MASK_LARGEST_HULL:
        _, label = cv2.connectedComponents(m, connectivity=8)
        hist = np.bincount(label[m != 0].ravel())
        if hist.size and hist.max() > 0:
            best = int(hist.argmax())
            assert (hist == hist[best]).sum() == 1, "two largest components: the reference's choice would be unpinned"
            ys, xs = np.nonzero((label == best) & (m != 0))
            hull = cv2.convexHull(np.stack([xs, ys], 1).astype(np.int32))
            m = np.zeros((H, W), np.uint8)
            cv2.fillConvexPoly(m, hull, 1)
        else:
            m = np.zeros((H, W), np.uint8)
    fg = cv2.dilate(m, cv2.getStructuringElement(cv2.MORPH_RECT, (5, 5)))
    ys, xs = np.nonzero(fg)
    roi = np.array([xs.min(), xs.max(), ys.min(), ys.max()] if len(xs) else [9999, 0, 9999, 0], np.int32)
    req = None
    if not (roi[1] - roi[0] < 10 or roi[3] - roi[2] < 10):
        umin, umax, vmin, vmax = (int(v) for v in roi)
        Wr, Hr = umax - umin, vmax - vmin
        side = max(Wr, Hr)
        col = colour.copy()
        col[fg == 0] = 0
        img = np.zeros((side, side, 3), np.uint8)
        img[:Hr, :Wr] = col[vmin:vmin + Hr, umin:umin + Wr]
        req = cv2.resize(img, (400, 400))
    return fg, roi, req


def main():
    out = {"n_cases": np.int32(len(CASES)), "cv2_version": np.array(cv2.__version__)}
    for i, (seed, H, W, mode, variant) in enumerate(CASES):
        mask = make_mask(seed, H, W, variant)
        fg, roi, req = reference(mask, mode, so.test_colour(H, W))
        out[f"mask_{i}"], out[f"mode_{i}"], out[f"fg_{i}"], out[f"roi_{i}"] = mask, np.int32(mode), fg, roi
        if req is not None:
            out[f"req_sha256_{i}"] = np.frombuffer(hashlib.sha256(np.ascontiguousarray(req, np.uint8).tobytes()).digest(), np.uint8)
        print(i, (H, W), "hull" if mode else "as-is", variant, roi.tolist(), "request" if req is not None else "gate fails")
    path = os.path.join(ROOT, "tests", "golden", "ref_segment.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
