"""Per-object mask scores with void pixels on the host (DESIGN.md §3.17): oracle/mask_objects_oracle.py against an independent restatement
of the DAVIS toolkit's db_eval_iou / f_measure with void_pixels, the palette PNG reader and writer, and eval_masks.py's DAVIS protocol."""
import os
import sys

import numpy as np
import pytest

from bundletrack_b200 import synth, vos
from oracle import mask_objects_oracle as moo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import eval_masks  # noqa: E402


def _seg2bmap(seg):
    seg = np.asarray(seg, bool)
    e, s, se = np.zeros_like(seg), np.zeros_like(seg), np.zeros_like(seg)
    e[:, :-1] = seg[:, 1:]
    s[:-1, :] = seg[1:, :]
    se[:-1, :-1] = seg[1:, 1:]
    b = seg ^ e | seg ^ s | seg ^ se
    b[-1, :] = seg[-1, :] ^ e[-1, :]
    b[:, -1] = seg[:, -1] ^ s[:, -1]
    b[-1, -1] = 0
    return b


def _toolkit(fg, gt, void, bound_th=0.008):
    """(J, F) of one object as the toolkit's db_eval_iou and f_measure compute them with void_pixels, dilating with cv2 and the disk."""
    import cv2
    keep = ~void
    inter, union = np.sum(fg & gt & keep), np.sum((fg | gt) & keep)
    j = 1.0 if union == 0 else inter / union
    r = int(np.ceil(bound_th * np.linalg.norm(fg.shape)))
    yy, xx = np.mgrid[-r:r + 1, -r:r + 1]
    disk = (xx * xx + yy * yy <= r * r).astype(np.uint8)
    fb, gb = _seg2bmap(fg & keep), _seg2bmap(gt & keep)
    fd, gd = cv2.dilate(fb.astype(np.uint8), disk), cv2.dilate(gb.astype(np.uint8), disk)
    n_fg, n_gt = np.sum(fb), np.sum(gb)
    if n_fg == 0 and n_gt > 0:
        p, rc = 1, 0
    elif n_fg > 0 and n_gt == 0:
        p, rc = 0, 1
    elif n_fg == 0 and n_gt == 0:
        p, rc = 1, 1
    else:
        p, rc = np.sum(fb * gd) / float(n_fg), np.sum(gb * fd) / float(n_gt)
    f = 0 if p + rc == 0 else 2 * p * rc / (p + rc)
    return float(j), float(f)


@pytest.mark.parametrize("h,w,n,void_value", [(60, 90, 3, 255), (41, 33, 5, 0), (48, 64, 2, -1), (1, 17, 2, 255), (23, 1, 1, 200)])
def test_object_metrics_equal_the_toolkit_restatement(h, w, n, void_value):
    pred, gt = synth.ragged_label_maps(4, h, w, n, void_from=1, seed=h + w)
    if void_value not in (-1, 255):
        gt[gt == 255] = void_value
    pred[1][pred[1] == 2] = 0                    # object 2 absent from one prediction
    pred[2][pred[2] == n] = 0                    # and the last from one frame of both masks
    gt[2][gt[2] == n] = 0
    pred[3][:, : w // 3] = 255 if void_value != 255 else 0
    j, f, c = moo.object_metrics(pred, gt, n, void_value)
    assert j.shape == f.shape == (4, n) and c.shape == (4, n, 6)
    for i in range(4):
        void = np.zeros((h, w), bool) if void_value < 0 else gt[i] == void_value
        for k in range(1, n + 1):
            wj, wf = _toolkit(pred[i] == k, gt[i] == k, void)
            assert (j[i, k - 1], f[i, k - 1]) == (wj, wf), (i, k)
    assert (j[2, n - 1], f[2, n - 1]) == (1.0, 1.0)         # absent from both masks


def test_void_is_removed_from_both_masks():
    gt = np.zeros((20, 20), np.uint8)
    gt[5:15, 5:15] = 1
    gt[5:15, 12:15] = 255
    pred = np.zeros_like(gt)
    pred[5:15, 5:15] = 1                          # covers the void columns too: they count for neither mask
    j, f, c = moo.object_metrics(pred[None], gt[None], 1, 255)
    assert j[0, 0] == 1.0 and f[0, 0] == 1.0 and c[0, 0, 0] == c[0, 0, 1] == 70
    j, _, _ = moo.object_metrics(pred[None], gt[None], 1, -1)
    assert j[0, 0] == 70 / 100


def test_palette_masks_round_trip(tmp_path):
    rng = np.random.default_rng(2)
    labels = rng.integers(0, 6, (13, 29)).astype(np.uint8)
    labels[0, :3] = 255
    palette = rng.integers(0, 256, (256, 3)).astype(np.uint8)
    path = str(tmp_path / "a.png")
    vos.write_palette_mask(path, labels, palette)
    from PIL import Image
    with Image.open(path) as im:
        assert im.mode == "P"
    got, pal = vos.read_palette_mask(path)
    assert np.array_equal(got, labels) and np.array_equal(pal, palette)
    # a DAVIS-style palette of a few colours, and a grey PNG read as its samples
    vos.write_palette_mask(path, labels % 3, palette[:3])
    got, pal = vos.read_palette_mask(path)
    assert np.array_equal(got, labels % 3) and np.array_equal(pal[:3], palette[:3])
    Image.fromarray(labels).save(str(tmp_path / "grey.png"))
    got, pal = vos.read_palette_mask(str(tmp_path / "grey.png"))
    assert np.array_equal(got, labels) and pal is None


def test_palette_reader_refuses_other_modes(tmp_path):
    from PIL import Image
    Image.fromarray(np.zeros((4, 5, 3), np.uint8)).save(str(tmp_path / "rgb.png"))
    with pytest.raises(ValueError, match=r"rgb\.png: a mode 'RGB' image"):
        vos.read_palette_mask(str(tmp_path / "rgb.png"))
    Image.fromarray(np.zeros((4, 5), np.uint16)).save(str(tmp_path / "deep.png"))
    with pytest.raises(ValueError, match=r"deep\.png: a mode 'I;16"):
        vos.read_palette_mask(str(tmp_path / "deep.png"))


def test_read_init_mask_on_a_palette_png_gives_the_blue_channel(tmp_path):
    """Why the DAVIS path reads indices: cv2 decodes a palette PNG to colours, and DAVIS object 1 (red) has blue 0."""
    pal = np.array([[0, 0, 0], [128, 0, 0], [0, 128, 0]], np.uint8)
    labels = np.array([[0, 1, 2]], np.uint8)
    vos.write_palette_mask(str(tmp_path / "a.png"), labels, pal)
    assert vos.read_init_mask(str(tmp_path / "a.png")).tolist() == [[0, 0, 0]]
    assert vos.read_palette_mask(str(tmp_path / "a.png"))[0].tolist() == [[0, 1, 2]]


def _write_sequence(d, masks, pal):
    os.makedirs(d, exist_ok=True)
    for k, m in enumerate(masks):
        vos.write_palette_mask(os.path.join(d, f"{k:05d}.png"), m, pal)


PAL = np.array([[0, 0, 0], [128, 0, 0], [0, 128, 0], [128, 128, 0]] + [[i, i, i] for i in range(4, 256)], np.uint8)


def test_davis_object_count_and_frames(tmp_path):
    g0 = np.zeros((6, 7), np.uint8)
    g0[0, 0], g0[1, 1], g0[2, 2] = 2, 1, 255
    assert eval_masks.davis_object_count(g0) == 2                      # void is not an object
    assert eval_masks.davis_object_count(np.full((2, 2), 255, np.uint8)) == 0
    gt = np.zeros((5, 6, 7), np.uint8)
    gt[0] = g0
    gt[3, 0, :] = 3                                                   # a later id above the count is the toolkit's to ignore too
    _write_sequence(str(tmp_path / "gt"), gt, PAL)
    _write_sequence(str(tmp_path / "pred"), np.ones((5, 6, 7), np.uint8), PAL)
    ids, g, p, n = eval_masks.davis_read_sequence(str(tmp_path / "gt"), str(tmp_path / "pred"))
    assert ids == ["00001", "00002", "00003"] and n == 2
    assert np.array_equal(g, gt[1:-1]) and np.array_equal(p, np.ones((3, 6, 7), np.uint8))
    # the first and the last predictions are not read
    os.remove(tmp_path / "pred" / "00000.png")
    os.remove(tmp_path / "pred" / "00004.png")
    assert eval_masks.davis_read_sequence(str(tmp_path / "gt"), str(tmp_path / "pred"))[0] == ids
    os.remove(tmp_path / "pred" / "00002.png")
    with pytest.raises(FileNotFoundError, match=r"00002\.png: no prediction"):
        eval_masks.davis_read_sequence(str(tmp_path / "gt"), str(tmp_path / "pred"))


def test_davis_sequence_too_short_to_score(tmp_path):
    gt = np.ones((2, 5, 6), np.uint8)
    _write_sequence(str(tmp_path / "gt"), gt, PAL)
    with pytest.raises(ValueError, match="2 frames leave none to score once the first and last are left out$"):
        eval_masks.davis_read_sequence(str(tmp_path / "gt"), str(tmp_path / "pred"))


def test_davis_refuses_an_id_above_the_object_count(tmp_path):
    gt = np.zeros((4, 5, 6), np.uint8)
    gt[:, 1, 1], gt[:, 2, 2] = 1, 2
    pred = gt.copy()
    pred[2, 3, 3] = 3
    _write_sequence(str(tmp_path / "gt"), gt, PAL)
    _write_sequence(str(tmp_path / "pred"), pred, PAL)
    with pytest.raises(ValueError, match=r"00002\.png: object id 3 in the prediction, the sequence has 2 objects"):
        eval_masks.davis_read_sequence(str(tmp_path / "gt"), str(tmp_path / "pred"))
    with pytest.raises(ValueError, match="object id 255"):
        eval_masks.davis_check_ids(np.full((2, 2), 255, np.uint8), 2, "x.png")


def test_davis_object_missing_from_the_predictions_is_an_empty_mask(tmp_path):
    pred, gt = synth.ragged_label_maps(5, 40, 50, 3, void_from=2, seed=4)
    pred[pred == 2] = 0
    _write_sequence(str(tmp_path / "gt"), gt, PAL)
    _write_sequence(str(tmp_path / "pred"), pred, PAL)
    _, g, p, n = eval_masks.davis_read_sequence(str(tmp_path / "gt"), str(tmp_path / "pred"))
    assert n == 3 and not (p == 2).any()
    j, f, c = moo.object_metrics(p, g, n)
    empty = moo.object_metrics(np.zeros_like(g), g, n)
    assert np.array_equal(j[:, 1], empty[0][:, 1]) and np.array_equal(f[:, 1], empty[1][:, 1])
    assert (c[:, 1, 0] == 0).all() and (c[:, 1, 2] == 0).all()


def test_davis_csv_columns(tmp_path):
    from bundletrack_b200.metrics import MASK_SCORE_KEYS
    per = {"bike_1": dict(zip(MASK_SCORE_KEYS, np.linspace(0.1, 0.7, 7))), "bike_2": dict(zip(MASK_SCORE_KEYS, np.linspace(0.2, 0.8, 7)))}
    mean = dict(zip(MASK_SCORE_KEYS, np.linspace(0.15, 0.75, 7)))
    g, s = eval_masks.write_davis_csvs(str(tmp_path), "val", per, mean)
    assert os.path.basename(g) == "global_results-val.csv" and os.path.basename(s) == "per-sequence_results-val.csv"
    assert open(g).read().splitlines() == ["J&F-Mean,J-Mean,J-Recall,J-Decay,F-Mean,F-Recall,F-Decay",
                                           "0.150,0.250,0.350,0.450,0.550,0.650,0.750"]
    assert open(s).read().splitlines() == ["Sequence,J-Mean,F-Mean", "bike_1,0.200,0.500", "bike_2,0.300,0.600"]


def test_davis_sequence_names(tmp_path):
    os.makedirs(tmp_path / "ImageSets" / "2017")
    (tmp_path / "ImageSets" / "2017" / "val.txt").write_text("bike\ncows\n\n")
    assert eval_masks.davis_sequence_names(str(tmp_path), "val") == ["bike", "cows"]
    assert eval_masks.davis_sequence_names(str(tmp_path), "val", "a, b") == ["a", "b"]
