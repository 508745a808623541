"""Mask accuracy on the device (bt_mask_metrics, metrics.MaskScore, DESIGN.md §3.16): counts equal to oracle/mask_oracle.py's integers and
J / F equal bit for bit over widths and heights around the word and band sizes, the disk's edge, known answers, batching, the OpenCV
fixture, refusals and eval_masks.py end to end."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest

from bundletrack_b200 import _lib, metrics, synth
from oracle import mask_oracle as mo

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIDTHS = [1, 2, 31, 32, 33, 63, 65, 640, 854, 1920]
HEIGHTS = [1, 2, 3, 17, 480, 1080]


def _live():
    d, p, h = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_int()
    assert _lib.load().bt_debug_live_resources(ctypes.byref(d), ctypes.byref(p), ctypes.byref(h)) == 0
    return d.value, p.value, h.value


@pytest.fixture(scope="module")
def ms(cuda_device):
    s = metrics.MaskScore(64, 1080, 1920)
    yield s
    s.close()


def _th_for(r, h, w):
    """A bound_th whose radius at h x w is r."""
    th = (r - 0.5) / math.hypot(h, w)
    assert mo.radius(h, w, th) == r
    return th


def _frames(rng, h, w):
    """Noise against noise, sparse specks against sparse specks, and ragged ellipses, with assorted foreground values."""
    p_e, g_e = synth.ragged_ellipse_masks(1, h, w, seed=h * 7919 + w)
    pred = [rng.random((h, w)) < 0.5, rng.random((h, w)) < 0.02, p_e[0]]
    gt = [rng.random((h, w)) < 0.5, rng.random((h, w)) < 0.03, g_e[0]]
    return (np.stack([(m != 0) * v for m, v in zip(pred, (1, 255, 255))]).astype(np.uint8),
            np.stack([(m != 0) * v for m, v in zip(gt, (7, 255, 1))]).astype(np.uint8))


def _check(ms, pred, gt, th):
    j, f, c = ms(pred, gt, th, counts=True)
    wj, wf, wc = mo.metrics(pred, gt, th)
    assert (c == wc).all(), (pred.shape, th, c, wc)
    assert j.tobytes() == wj.tobytes() and f.tobytes() == wf.tobytes(), (pred.shape, th)
    return j, f, c


@pytest.mark.parametrize("h", HEIGHTS)
def test_counts_and_scores_equal_the_oracle(ms, h):
    rng = np.random.default_rng(h)
    for w in WIDTHS:
        pred, gt = _frames(rng, h, w)
        _check(ms, pred, gt, 0.008)
        diag = math.hypot(h, w)
        if h * w <= 480 * 854 and diag > 20:                     # a wide radius too, up to the limit of 64 (the oracle's time grows with r)
            _check(ms, pred, gt, _th_for(min(64, int(0.3 * diag)), h, w))


def test_unaligned_inputs(ms, cuda_device):
    import torch
    rng = np.random.default_rng(5)
    for h, w, off in [(17, 33, 3), (480, 641, 7), (61, 65, 15), (3, 1, 1)]:
        pred, gt = _frames(rng, h, w)
        n = pred.size
        bp = torch.full((n + 32,), 9, dtype=torch.uint8, device=cuda_device)       # non-zero bytes on either side of the masks
        bg = torch.full((n + 32,), 9, dtype=torch.uint8, device=cuda_device)
        bp[off:off + n] = torch.from_numpy(pred.ravel()).to(cuda_device)
        bg[off + 5:off + 5 + n] = torch.from_numpy(gt.ravel()).to(cuda_device)
        j, f, c = ms(bp[off:off + n].view(pred.shape), bg[off + 5:off + 5 + n].view(gt.shape), 0.05, counts=True)
        wj, wf, wc = mo.metrics(pred, gt, 0.05)
        assert (c == wc).all() and j.tobytes() == wj.tobytes() and f.tobytes() == wf.tobytes(), (h, w, off)


def test_disk_edge_across_bands(ms):
    """One-pixel masks: a pixel's boundary is the 2 x 2 block ending at it, so two blocks (a + 1, b + 1) apart are a, b apart at their
    nearest pixels.  a^2 + b^2 = r^2 matches exactly one pixel each way; r^2 + 1 matches none.  The pairs sit across the band edges."""
    h, w = 200, 300
    cases = [(5, 3, 4, True), (5, 1, 5, False), (13, 5, 12, True), (13, 12, 5, True), (13, 7, 11, False), (25, 7, 24, True),
             (25, 24, 7, True), (25, 1, 25, False), (64, 0, 64, True), (64, 64, 0, True), (64, 1, 64, False)]
    for r, a, b, match in cases:
        th = _th_for(r, h, w)
        preds, gts = [], []
        for y in (62, 63, 64, 65, 66, 127, 128, 129):
            for sy, sx in ((1, 1), (-1, 1), (1, -1), (-1, -1)):
                yp, xp = y + sy * (a + 1), 150 + sx * (b + 1)
                if not (1 <= yp < h - 1 and 1 <= y < h - 1 and 1 <= xp < w - 1):
                    continue
                p, g = np.zeros((h, w), np.uint8), np.zeros((h, w), np.uint8)
                p[yp, xp], g[y, 150] = 255, 255
                preds.append(p)
                gts.append(g)
        _, _, c = _check(ms, np.stack(preds), np.stack(gts), th)
        assert (c[:, 2:4] == 4).all() and (c[:, 4:] == (1 if match else 0)).all(), (r, a, b, c)


def test_known_answers(ms):
    rng = np.random.default_rng(2)
    for h, w in [(480, 640), (33, 65), (1, 1)]:
        g = synth.ragged_ellipse_masks(1, h, w, seed=1)[1][0]
        z, full = np.zeros_like(g), np.full_like(g, 255)
        j, f = ms(np.stack([g, z]), np.stack([g, z]))
        assert j.tolist() == [1.0, 1.0] and f.tolist() == [1.0, 1.0]
        if g.any() and h > 1:
            j, f = ms(z[None], g[None])
            assert j.tolist() == [0.0] and f.tolist() == [0.0]
            _, f = ms(full[None], g[None])
            assert f.tolist() == [0.0]
    noise = (rng.random((3, 50, 70)) < 0.3).astype(np.uint8)
    j, f = ms(noise, noise)
    assert (j == 1.0).all() and (f == 1.0).all()


def test_batching_and_input_kinds(ms, cuda_device):
    import torch
    pred, gt = synth.ragged_ellipse_masks(150, 120, 161, seed=4)
    j, f, c = ms(pred, gt, 0.02, counts=True)
    small = metrics.MaskScore(7, 120, 161)
    j7, f7, c7 = small(pred, gt, 0.02, counts=True)
    small.close()
    assert j7.tobytes() == j.tobytes() and f7.tobytes() == f.tobytes() and (c7 == c).all()
    jt, ft = ms(torch.from_numpy(pred).to(cuda_device), torch.from_numpy(gt).to(cuda_device), 0.02)
    jb, fb = ms(pred != 0, torch.from_numpy(gt != 0).to(cuda_device), 0.02)
    assert jt.tobytes() == j.tobytes() and ft.tobytes() == f.tobytes() and jb.tobytes() == j.tobytes() and fb.tobytes() == f.tobytes()
    wj, wf, wc = mo.metrics(pred[::10], gt[::10], 0.02)
    assert (c[::10] == wc).all() and j[::10].tobytes() == wj.tobytes() and f[::10].tobytes() == wf.tobytes()


def test_golden_opencv_fixture(ms):
    g = np.load(os.path.join(ROOT, "tests", "golden", "ref_mask_score.npz"))
    for name in ("ellipses", "noise"):
        j, f, c = ms(g[f"{name}_pred"], g[f"{name}_gt"], float(g[f"{name}_bound_th"]), counts=True)
        assert (c == g[f"{name}_counts"]).all(), name
        assert j.tobytes() == g[f"{name}_j"].tobytes() and f.tobytes() == g[f"{name}_f"].tobytes(), name
        assert np.array(list(metrics.mask_score(j, f).values())).tobytes() == g[f"{name}_score"].tobytes(), name


def test_refusals_leave_outputs_untouched(cuda_device):
    import torch
    lib = _lib.load()
    before = _live()
    s = metrics.MaskScore(4, 100, 200)
    pm = torch.zeros((5, 100, 200), dtype=torch.uint8, device=cuda_device)
    out = torch.full((3, 5), 7.0, dtype=torch.float64, device=cuda_device)
    cnt = torch.full((5, 6), 7, dtype=torch.int64, device=cuda_device)
    p = _lib.ptr

    def call(n=2, h=100, w=200, th=0.008, pred=pm, gt=pm, j=out[0], f=out[1], ctx=None):
        return lib.bt_mask_metrics(ctx or s.ctx, p(pred), p(gt), n, h, w, th, p(j), p(f), p(cnt), s.stream if ctx is None else None)

    def untouched():
        torch.cuda.synchronize()
        return bool((out == 7.0).all()) and bool((cnt == 7).all())

    invalid = [dict(pred=None), dict(gt=None), dict(j=None), dict(f=None), dict(n=0), dict(h=0), dict(w=-1), dict(th=0.0), dict(th=1.0),
               dict(th=float("nan")), dict(th=-0.1), dict(th=0.3)]          # 0.3 x |(100, 200)| gives r = 68 > 64
    for kw in invalid:
        assert call(**kw) == _lib.BT_ERR_INVALID_ARG, kw
        assert untouched(), kw
    assert call(th=0.3) == _lib.BT_ERR_INVALID_ARG and b"radius 68" in lib.bt_last_error()
    for kw in [dict(n=5), dict(h=101), dict(w=201)]:
        assert call(**kw) == _lib.BT_ERR_CAPACITY, kw
        assert untouched(), kw
    other = _lib.Context(0)
    assert call(ctx=other) == _lib.BT_ERR_INVALID_ARG and b"bt_mask_reserve" in lib.bt_last_error()
    assert untouched()
    other.close()
    # a reserve whose band cannot fit in shared memory is refused and leaves the module as it was
    assert lib.bt_mask_reserve(s.ctx, 4, 1000, 100_000) == _lib.BT_ERR_INVALID_ARG and b"shared memory" in lib.bt_last_error()
    assert lib.bt_mask_reserve(s.ctx, 0, 100, 200) == _lib.BT_ERR_INVALID_ARG
    rng = np.random.default_rng(0)
    pred, gt = (rng.random((2, 2, 100, 200)) < 0.2).astype(np.uint8)
    want = s(pred, gt)
    # a reserve that fails partway refuses every call until one succeeds, then serves as before
    for n in range(1, 10):
        assert lib.bt_debug_fail_alloc(n) == 0
        rc = lib.bt_mask_reserve(s.ctx, 64, 400, 500)
        assert lib.bt_debug_fail_alloc(0) == 0
        if rc == _lib.BT_OK:
            break
        assert call() == _lib.BT_ERR_INVALID_ARG and b"bt_mask_reserve" in lib.bt_last_error()
        assert untouched()
    assert n > 1
    got = s(pred, gt)
    assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes()
    s.close()
    del pm, out, cnt
    torch.cuda.synchronize()
    assert _live() == before


def test_eval_masks_script(tmp_path, cuda_device):
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import eval_masks
    rows = []
    for v, (n, h, w) in enumerate([(9, 120, 160), (5, 61, 97)]):
        pred, gt = synth.ragged_ellipse_masks(n, h, w, seed=v)
        for sub, masks in (("gt_mask", gt), ("masks_vos", pred)):
            os.makedirs(tmp_path / f"video{v}" / sub)
            for k, m in enumerate(masks):
                synth.write_png(str(tmp_path / f"video{v}" / sub / f"{k:07d}.png"), m)
        rows.append((pred, gt))
    lines = []
    res = eval_masks.evaluate(eval_masks.ycbineoat_sequences(str(tmp_path), "masks_vos"), out=lines.append)
    assert len(lines) == 3
    for v, (pred, gt) in enumerate(rows):
        wj, wf, _ = mo.metrics(pred[1:-1], gt[1:-1])
        r = res["sequences"][f"video{v}"]
        assert r["frames"] == [f"{k:07d}" for k in range(1, len(pred) - 1)]
        assert np.array(r["j"]).tobytes() == wj.tobytes() and np.array(r["f"]).tobytes() == wf.tobytes()
        want = mo.score(wj, wf)
        assert all(r[k] == want[k] for k in metrics.MASK_SCORE_KEYS)
    assert res["mean"]["J-Mean"] == np.mean([res["sequences"][s]["J-Mean"] for s in ("video0", "video1")])
    kept = eval_masks.evaluate([("v0", str(tmp_path / "video0" / "gt_mask"), str(tmp_path / "video0" / "masks_vos"))], keep_ends=True,
                               out=lines.append)
    assert len(kept["sequences"]["v0"]["frames"]) == 9
