"""CPU checks of oracle/segment_oracle.py: byte for byte against the OpenCV recordings in tests/golden/ref_segment.npz (made by
scripts/make_golden_segment.py) and, where cv2 is installed, against OpenCV itself on a few hundred seeded masks."""
import hashlib
import os

import numpy as np
import pytest

from bundletrack_b200 import synth
from oracle import segment_oracle as so

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ref_segment.npz")


def test_oracle_equals_golden():
    g = np.load(GOLDEN)
    for i in range(int(g["n_cases"])):
        mask = g[f"mask_{i}"]
        fg, roi = so.segment(mask, int(g[f"mode_{i}"]))
        assert np.array_equal(fg, g[f"fg_{i}"]), i
        assert np.array_equal(roi, g[f"roi_{i}"]), i
        req = so.lfnet_request(so.test_colour(*mask.shape), fg, roi)
        if f"req_sha256_{i}" in g:
            assert req is not None and request_digest(req) == g[f"req_sha256_{i}"].tobytes(), i
        else:
            assert req is None, i


def request_digest(req):
    """SHA-256 of the request's bytes: how ref_segment.npz records OpenCV's 400 x 400 x 3 request images."""
    return hashlib.sha256(np.ascontiguousarray(req, np.uint8).tobytes()).digest()


def test_tie_rule_and_degenerate_hulls():
    m = np.zeros((20, 30), np.uint8)
    m[2:5, 20:24] = 1          # 12 pixels, first pixel (2, 20)
    m[10:13, 3:7] = 1          # 12 pixels, first pixel (10, 3)
    lab, best = so.largest_component(m)
    assert lab[2, 20] == best
    assert so.convex_hull([(3, 3), (4, 4), (5, 5), (6, 6)]) == [(3, 3), (6, 6)]     # collinear points are dropped
    one = np.zeros((9, 9), np.uint8); one[4, 4] = 7
    assert np.array_equal(so.hull_mask(one), (one != 0).astype(np.uint8))
    fg, roi = so.segment(np.zeros((9, 9), np.uint8), so.MASK_LARGEST_HULL)
    assert not fg.any() and tuple(roi) == so.ROI_EMPTY


def _cv_reference(cv2, mask, mode):
    m = mask.copy()
    if mode == so.MASK_LARGEST_HULL:
        _, label = cv2.connectedComponents(m, connectivity=8)
        hist = np.bincount(label[m != 0].ravel())
        if hist.size and hist.max() > 0:
            best = int(hist.argmax())
            if (hist == hist[best]).sum() > 1:
                return None                 # OpenCV's numbering would decide; the reference leaves this unpinned
            ys, xs = np.nonzero((label == best) & (m != 0))
            m = np.zeros_like(m)
            cv2.fillConvexPoly(m, cv2.convexHull(np.stack([xs, ys], 1).astype(np.int32)), 1)
        else:
            m = np.zeros_like(m)
    return cv2.dilate(m, cv2.getStructuringElement(cv2.MORPH_RECT, (5, 5)))


@pytest.mark.parametrize("chunk", range(4))
def test_oracle_equals_opencv(chunk):
    cv2 = pytest.importorskip("cv2")
    sizes = [(480, 640), (97, 131), (240, 320), (61, 700), (300, 45)]
    for seed in range(chunk * 50, chunk * 50 + 50):
        H, W = sizes[seed % len(sizes)]
        mask = synth.make_object_mask(seed, H, W, n_distractors=seed % 5, speckle_frac=0.0005 * (seed % 4), n_holes=seed % 6)
        mode = seed % 2 if seed % 7 else so.MASK_LARGEST_HULL
        ref = _cv_reference(cv2, mask, mode)
        if ref is None:
            continue
        fg, roi = so.segment(mask, mode)
        assert np.array_equal(fg, ref), (seed, mode)
        ys, xs = np.nonzero(ref)
        assert np.array_equal(roi, [xs.min(), xs.max(), ys.min(), ys.max()] if len(xs) else so.ROI_EMPTY), seed


def test_resize_equals_opencv():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(0)
    for side in list(range(10, 30)) + [57, 199, 200, 333, 399, 400, 401, 479, 600, 639, 800, 801, 1000]:
        img = rng.integers(0, 256, (side, side, 3), dtype=np.uint8)
        assert np.array_equal(so.resize_linear_u8(img), cv2.resize(img, (400, 400))), side


def test_request_crop_equals_the_reference_loop():
    colour = so.test_colour(50, 70)
    fg = np.zeros((50, 70), np.uint8); fg[5:40, 10:30] = 1; fg[20, 15] = 0
    roi = so.roi_of(fg)
    img = so.crop_square(colour, fg, roi)
    assert img.shape == (34, 34, 3)                                   # side = max(umax - umin, vmax - vmin): the last row / column dropped
    ref = np.zeros_like(img)
    for h in range(roi[3] - roi[2]):
        for w in range(roi[1] - roi[0]):
            y, x = h + roi[2], w + roi[0]
            ref[h, w] = colour[y, x] if fg[y, x] else 0
    assert np.array_equal(img, ref)
    assert so.lfnet_request(colour, np.zeros_like(fg), so.roi_of(np.zeros_like(fg))) is None
