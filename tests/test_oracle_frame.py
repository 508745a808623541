"""CPU tests of the frame front-end oracle (oracle/frame_oracle.py): pinned against the golden vectors of the reference's own
kernels (tests/golden/ref_frame_*.npz, made by scripts/make_golden_frame.py) and checked for the properties the
reference's front end has by construction."""
import glob
import os

import numpy as np
import pytest

from bundletrack_b200 import synth
from oracle import frame_oracle as fo

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "ref_frame_*.npz")))


@pytest.mark.skipif(not GOLDEN, reason="no golden vectors")
@pytest.mark.parametrize("path", GOLDEN)
def test_oracle_matches_reference_kernels(path):
    g = np.load(path)
    dp = {k: float(g[k]) for k in fo.DEFAULTS}
    d, xyz, n = fo.preprocess(g["raw"], tuple(g["K"]), dp)
    bad_d = np.abs(d - g["depth"]) > 2e-6          # fast-math exp/division in the reference build: a few float ulps at ~1 m
    assert bad_d.mean() <= 2e-3, f"{bad_d.mean():.2e} of the pixels differ (max {np.abs(d - g['depth']).max():.2e})"
    ok = ~bad_d
    assert np.abs(xyz[..., :3] - g["xyz"])[ok].max() <= 3e-6
    bad_n = np.abs(n[..., :3] - g["normal"]).max(-1) > 1e-3
    assert bad_n.mean() <= 4e-3, f"{bad_n.mean():.2e} of the normals differ"


def test_front_end_properties():
    raw, K = synth.make_raw_depth(9, 120, 160)
    d, xyz, n = fo.preprocess(raw, K)
    valid = d >= 0.1
    assert valid.sum() > 0.05 * d.size
    # normals are unit or zero, face the camera, and vanish on the image border and wherever the point is invalid
    ln = np.linalg.norm(n[..., :3], axis=-1)
    assert np.all((np.abs(ln - 1) < 1e-5) | (ln == 0))
    assert np.all(np.sum(n[..., :3] * -xyz[..., :3], -1)[ln > 0] >= 0)
    assert not n[0].any() and not n[-1].any() and not n[:, 0].any() and not n[:, -1].any()
    assert not n[~valid].any()
    # the point map is the pinhole back-projection of the filtered depth
    fx, fy, cx, cy = K
    ys, xs = np.nonzero(valid)
    assert np.allclose(xyz[ys, xs, 0], (xs - cx) / fx * d[ys, xs], atol=2e-6)
    assert np.allclose(xyz[ys, xs, 1], (ys - cy) / fy * d[ys, xs], atol=2e-6)
    assert np.array_equal(xyz[..., 2], np.where(valid, d, 0)) and np.array_equal(xyz[..., 3], valid.astype(np.float32))
    # flying pixels (1 % of a fronto-parallel plane, 2-6 cm off it) do not survive erosion + filtering, bar the rare one with a like neighbour
    rng = np.random.default_rng(3)
    plane = (0.6 + rng.normal(0, 0.0002, (120, 160))).astype(np.float32)
    fly = rng.random(plane.shape) < 0.01
    noisy = plane + fly * rng.uniform(0.02, 0.06, plane.shape).astype(np.float32)
    dp_, _, _ = fo.preprocess(noisy, K)
    inner = np.zeros(plane.shape, bool); inner[3:-3, 3:-3] = True
    assert np.mean(np.abs(dp_ - 0.6)[inner] > 0.002) < 5e-4 and fly.sum() > 100
    # zero in, zero out
    z = fo.preprocess(np.zeros((40, 50), np.float32), K)
    assert not z[0].any() and not z[1].any() and not z[2].any()


def test_erode_and_filter_follow_the_reference_rules():
    d = np.full((9, 9), 0.5, np.float32)
    d[4, 4] = 0.56                               # every neighbour differs by > 1 mm -> 8/9 >= 0.8 -> removed
    e = fo.erode(d, 1, 0.001, 0.8)
    assert e[4, 4] == 0 and np.all(e[d == 0.5] == 0.5)
    d2 = d.copy(); d2[4, 4] = 0.5; d2[0, 0] = 0  # corner: only in-image neighbours are counted, the divisor stays 9
    assert fo.erode(d2, 1, 0.001, 0.8)[0, 1] == 0.5
    g = fo.gauss(e, 2, 2.0, 1e5)
    assert abs(g[4, 4] - 0.5) < 1e-6             # the hole is refilled from its neighbours (invalid centre pixels are filtered too)
    far = np.full((9, 9), 0.5, np.float32); far[:, 5:] = 0.7
    gf = fo.gauss(far, 2, 2.0, 1e5)              # |d - mean| >= 1 cm on both sides of the step near the edge -> weight sum 0 -> 0
    assert gf[4, 4] == 0 and abs(gf[4, 0] - 0.5) < 1e-6 and abs(gf[4, 8] - 0.7) < 1e-6
