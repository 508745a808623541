"""Mask accuracy on the host (DESIGN.md §3.16): the numpy restatement in oracle/mask_oracle.py against OpenCV and scipy, bt_mask_score bit
for bit against numpy's db_statistics, and eval_masks.py's file pairing."""
import math
import os
import sys

import numpy as np
import pytest

from bundletrack_b200 import _lib, metrics
from oracle import mask_oracle as mo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import eval_masks  # noqa: E402


def _disk(r):
    y, x = np.mgrid[-r:r + 1, -r:r + 1]
    return x * x + y * y <= r * r


def _random_boundaries(seed):
    rng = np.random.default_rng(seed)
    for _ in range(40):
        h, w = (int(v) for v in rng.integers(1, 70, 2))
        yield rng.random((h, w)) < rng.choice([0.005, 0.05, 0.3]), int(rng.integers(1, 12))


def test_oracle_dilation_equals_cv2_disk():
    cv2 = pytest.importorskip("cv2")
    for b, r in _random_boundaries(1):
        want = cv2.dilate(b.astype(np.uint8), _disk(r).astype(np.uint8)) > 0
        assert (mo.dilate(b, r) == want).all(), (b.shape, r)


def test_oracle_dilation_equals_scipy():
    from scipy import ndimage
    for b, r in _random_boundaries(2):
        assert (mo.dilate(b, r) == ndimage.binary_dilation(b, structure=_disk(r))).all(), (b.shape, r)


def test_radius_and_boundary_edge_rules():
    assert [mo.radius(*s) for s in [(480, 640), (480, 854), (720, 1280), (1080, 1920)]] == [7, 8, 12, 18]
    assert not mo.boundary(np.ones((5, 7), np.uint8)).any()               # a full frame has no boundary
    m = np.zeros((6, 8), np.uint8)
    m[:3, :4] = 1                                                         # foreground along the top and left edges
    b = mo.boundary(m)
    assert not b[0, :3].any() and not b[:2, 0].any() and b[2, :4].all() and b[:3, 3].all()
    one = np.zeros((4, 4), np.uint8)
    one[3, 3] = 1
    b = mo.boundary(one)
    assert not b[3, 3] and b[2:, 2:].sum() == 3 and b.sum() == 3          # the corner is never a boundary; its neighbours see it


def _score(j, f):
    return np.array(list(metrics.mask_score(j, f).values()))


@pytest.mark.parametrize("n", list(range(1, 13)) + [100, 255, 256, 257, 1000, 4099])
def test_mask_score_equals_numpy(n):
    rng = np.random.default_rng(n)
    for values in (rng.random(n), rng.choice([0.0, 0.25, 0.5, 0.5000000000000001, 0.75, 1.0], n), np.full(n, 0.5)):
        j, f = values, rng.permutation(values)
        got = _score(j, f)
        want = np.array(list(mo.score(j, f).values()))
        assert got.tobytes() == want.tobytes(), (n, got, want)
    assert _score(np.full(n, 0.5), np.full(n, 0.5))[[2, 5]].tolist() == [0.0, 0.0]      # the recall is strictly above 0.5


def test_mask_score_refuses():
    lib = _lib.load()
    out = np.zeros(7)
    x = np.ones(3)
    assert lib.bt_mask_score(_lib.ptr(x), _lib.ptr(x), 0, _lib.ptr(out)) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_mask_score(None, _lib.ptr(x), 3, _lib.ptr(out)) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_mask_score(_lib.ptr(x), _lib.ptr(x), 3, None) == _lib.BT_ERR_INVALID_ARG
    with pytest.raises(ValueError):
        metrics.mask_score([1.0, 0.5], [1.0])


def test_known_answers_of_the_oracle():
    rng = np.random.default_rng(3)
    g = (rng.random((30, 41)) < 0.4).astype(np.uint8)
    assert mo.j_and_f(mo.frame_counts(g, g)) == (1.0, 1.0)
    z = np.zeros_like(g)
    assert mo.j_and_f(mo.frame_counts(z, z)) == (1.0, 1.0)
    assert mo.j_and_f(mo.frame_counts(z, g)) == (0.0, 0.0)
    assert mo.j_and_f(mo.frame_counts(np.ones_like(g), g))[1] == 0.0


def _touch(d, names):
    os.makedirs(d, exist_ok=True)
    for n in names:
        open(os.path.join(d, n), "wb").close()


def test_eval_masks_pairs_files(tmp_path):
    gt, pred = str(tmp_path / "gt_mask"), str(tmp_path / "masks_vos")
    _touch(gt, ["0002.png", "0000.png", "0001.png", "notes.txt"])
    _touch(pred, ["0000.png", "0001.png", "0002.png", "0003.png"])
    pairs = eval_masks.pair_files(gt, pred)
    assert [i for i, _, _ in pairs] == ["0000", "0001", "0002"]
    assert pairs[1] == ("0001", os.path.join(gt, "0001.png"), os.path.join(pred, "0001.png"))
    assert [i for i, _, _ in eval_masks.protocol_frames(pairs)] == ["0001"]
    assert eval_masks.protocol_frames(pairs, keep_ends=True) == pairs
    with pytest.raises(ValueError, match="keep_ends"):
        eval_masks.protocol_frames(pairs[:2])
    os.remove(os.path.join(pred, "0001.png"))
    with pytest.raises(FileNotFoundError, match=r"masks_vos.0001\.png"):
        eval_masks.pair_files(gt, pred)
    _touch(str(tmp_path / "vid_b" / "gt_mask"), ["0000.png"])
    _touch(str(tmp_path / "vid_a" / "gt_mask"), ["0000.png"])
    assert [v for v, _, _ in eval_masks.ycbineoat_sequences(str(tmp_path), "masks_vos")] == ["vid_a", "vid_b"]


def test_eval_masks_refuses_a_mask_that_is_not_8_bit_grey(tmp_path):
    from bundletrack_b200 import synth
    synth.write_png(str(tmp_path / "rgb.png"), np.zeros((4, 5, 3), np.uint8))
    with pytest.raises(ValueError, match="8-bit grey"):
        eval_masks._read([str(tmp_path / "rgb.png")])
