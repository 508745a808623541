"""DAVIS 2017 on the device (DESIGN.md §3.17): bt_mask_metrics_objects against oracle/mask_objects_oracle.py (integer counts, J and F bit
for bit) over sizes, object counts, void and alignment, against bt_mask_metrics for one binary object, refusals; bt_vos_labels against the
mask and the float64 restatement; run_vos.py --davis and eval_masks.py --davis end to end on a synthetic DAVIS tree."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from bundletrack_b200 import _lib, metrics, synth, vos
from oracle import mask_objects_oracle as moo
from oracle import vos_oracle as vo

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))


@pytest.fixture(scope="module")
def ms(cuda_device):
    s = metrics.MaskScore(64, 1080, 1920)
    yield s
    s.close()


def _check(ms, pred, gt, n, void_value, th=0.008):
    j, f, c = ms.objects(pred, gt, n, void_value, th, counts=True)
    wj, wf, wc = moo.object_metrics(pred, gt, n, void_value, th)
    assert (c == wc).all(), (pred.shape, n, void_value)
    assert j.tobytes() == wj.tobytes() and f.tobytes() == wf.tobytes(), (pred.shape, n, void_value)
    return j, f, c


@pytest.mark.parametrize("h,w", [(1, 1), (1, 1920), (1080, 1), (2, 65), (17, 33), (65, 127), (480, 854), (1080, 1920)])
def test_counts_and_scores_equal_the_oracle(ms, h, w):
    frames = 2 if h * w > 100_000 else 4
    for n in ((1, 8) if h * w > 500_000 else range(1, 9)):
        pred, gt = synth.ragged_label_maps(frames, h, w, n, void_from=1, seed=h * 31 + w + n)
        pred[-1][pred[-1] == 1] = 0                               # an object absent from one prediction
        if n > 1:
            gt[0][gt[0] == n] = 0                                 # and one absent from both masks of a frame
            pred[0][pred[0] == n] = 0
        if w > 2:
            pred[1][:, : w // 4] = 255                            # predictions over the void value and outside the objects
        _check(ms, pred, gt, n, 255)
        _check(ms, pred, gt, n, -1)
        gt0 = np.where(gt == 255, 0, gt)
        _check(ms, pred, gt0, n, 0)                               # void 0: only the objects' pixels are scored


def test_wide_radius(ms):
    pred, gt = synth.ragged_label_maps(3, 300, 400, 4, void_from=0, seed=11)
    _check(ms, pred, gt, 4, 255, th=60.5 / 500.0)                 # r = 61


def test_unaligned_inputs(ms, cuda_device):
    for h, w, op, og in [(17, 33, 3, 8), (480, 641, 7, 0), (61, 65, 15, 1), (3, 1, 1, 14), (40, 200, 0, 9), (33, 97, 9, 9)]:
        pred, gt = synth.ragged_label_maps(3, h, w, 3, void_from=0, seed=h + w)
        n = pred.size
        bp = torch.full((n + 32,), 255, dtype=torch.uint8, device=cuda_device)      # void and object bytes on either side of the maps
        bg = torch.full((n + 32,), 2, dtype=torch.uint8, device=cuda_device)
        bp[op:op + n] = torch.from_numpy(pred.ravel()).to(cuda_device)
        bg[og:og + n] = torch.from_numpy(gt.ravel()).to(cuda_device)
        P, G = bp[op:op + n].view(pred.shape), bg[og:og + n].view(gt.shape)
        for void_value in (255, -1):
            j, f, c = ms.objects(P, G, 3, void_value, 0.05, counts=True)
            wj, wf, wc = moo.object_metrics(pred, gt, 3, void_value, 0.05)
            assert (c == wc).all() and j.tobytes() == wj.tobytes() and f.tobytes() == wf.tobytes(), (h, w, op, og, void_value)


def test_one_binary_object_equals_bt_mask_metrics(ms):
    for h, w in [(1, 1), (37, 1000), (480, 854)]:
        p, g = synth.ragged_ellipse_masks(5, h, w, seed=w)
        p, g = (p > 0).astype(np.uint8), (g > 0).astype(np.uint8)
        j1, f1, c1 = ms(p, g, counts=True)
        j, f, c = ms.objects(p, g, 1, -1, counts=True)
        assert (c[:, 0] == c1).all() and j[:, 0].tobytes() == j1.tobytes() and f[:, 0].tobytes() == f1.tobytes()


def test_batching_over_the_reserved_rows(cuda_device):
    """64 rows hold 21 frames of 3 objects: 50 frames take three calls and give what one frame at a time gives."""
    s = metrics.MaskScore(64, 100, 120)
    pred, gt = synth.ragged_label_maps(50, 100, 120, 3, void_from=10, seed=5)
    j, f = s.objects(pred, gt, 3)
    wj, wf, _ = moo.object_metrics(pred, gt, 3)
    assert j.tobytes() == wj.tobytes() and f.tobytes() == wf.tobytes()
    with pytest.raises(ValueError, match="65 reserved rows"):
        s.objects(pred, gt, 65, -1)
    s.close()


def test_refusals_leave_outputs_untouched(cuda_device):
    lib = _lib.load()
    s = metrics.MaskScore(8, 100, 200)
    pm = torch.zeros((9, 100, 200), dtype=torch.uint8, device=cuda_device)
    out = torch.full((2, 16), 7.0, dtype=torch.float64, device=cuda_device)
    cnt = torch.full((16, 6), 7, dtype=torch.int64, device=cuda_device)
    p = _lib.ptr

    def call(n=2, h=100, w=200, k=3, void=255, th=0.008, pred=pm, gt=pm, j=out[0], f=out[1], ctx=None):
        return lib.bt_mask_metrics_objects(ctx or s.ctx, p(pred), p(gt), n, h, w, k, void, th, p(j), p(f), p(cnt), s.stream if ctx is None else None)

    def untouched():
        torch.cuda.synchronize()
        return bool((out == 7.0).all()) and bool((cnt == 7).all())

    invalid = [dict(pred=None), dict(gt=None), dict(j=None), dict(f=None), dict(n=0), dict(h=0), dict(w=-1), dict(k=0), dict(k=256),
               dict(void=1), dict(void=3), dict(void=256), dict(void=-2), dict(th=0.0), dict(th=1.0), dict(th=0.3)]
    for kw in invalid:
        assert call(**kw) == _lib.BT_ERR_INVALID_ARG, kw
        assert untouched(), kw
    assert call(void=3) == _lib.BT_ERR_INVALID_ARG and b"void_value 3" in lib.bt_last_error()
    for kw in [dict(n=3), dict(n=9, k=1), dict(k=9, n=1), dict(h=101), dict(w=201)]:     # 3 x 3 = 9 rows > 8
        assert call(**kw) == _lib.BT_ERR_CAPACITY, kw
        assert untouched(), kw
    assert call(n=3) == _lib.BT_ERR_CAPACITY and b"9 rows" in lib.bt_last_error()
    other = _lib.Context(0)
    assert call(ctx=other) == _lib.BT_ERR_INVALID_ARG and b"bt_mask_reserve" in lib.bt_last_error()
    assert untouched()
    other.close()
    for n in range(1, 10):                                      # after a failed reserve: refused, naming it, until one succeeds
        assert lib.bt_debug_fail_alloc(n) == 0
        rc = lib.bt_mask_reserve(s.ctx, 64, 400, 500)
        assert lib.bt_debug_fail_alloc(0) == 0
        if rc == _lib.BT_OK:
            break
        assert call() == _lib.BT_ERR_INVALID_ARG and b"bt_mask_reserve" in lib.bt_last_error()
        assert untouched()
    assert n > 1
    assert call(n=2, k=8, void=-1) == _lib.BT_OK
    torch.cuda.synchronize()
    assert (out == 1.0).all()                                   # empty maps: every object J = F = 1
    s.close()


# ---- labels from the VOS network -------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sd():
    import test_vos_gpu as tv
    s = vo.random_state_dict(7, calibrate=tv.video(1, 96, 128, seed=9)[0][0])
    return {k[len("module."):]: v.double().numpy() for k, v in s.items() if not k.endswith("num_batches_tracked")}


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("H,W,n", [(48, 64, 30), (97, 131, 12)])
def test_vos_labels(cuda_device, sd, H, W, n):
    import test_vos_gpu as tv
    frames, m0 = tv.video(n, H, W)
    P = dict(vos.DEFAULTS)
    v = vos.VosDevice(sd, P, H, W)
    with pytest.raises(_lib.BtError, match="bt_vos_labels: no sequence begun"):
        v.labels()
    v.begin(_dev(frames[0]), _dev(m0))
    assert np.array_equal(v.labels().cpu().numpy(), m0)
    R = v.debug(0)["slots"]
    values = np.array([0, 3, 7])
    listed = []
    for k in range(1, n):
        mask = v.next(_dev(frames[k])).cpu().numpy()
        lab = v.labels().cpu().numpy()
        assert np.array_equal((lab != 0) * 255, mask), k
        assert set(np.unique(lab)) <= {0, 3, 7}, k
        dbg = v.debug(k % R)
        hist = [v.debug(i % R) for i in vo.schedule(k, P["ref_num"], P["range"])]
        pred = vo.predict([h["feat"] for h in hist], [h["label"][..., :3] for h in hist], dbg["feat"], k, P["sigma1"], P["sigma2"],
                          P["temperature"])
        up = vo.upsample(pred, dbg["Hd"], dbg["Wd"], H, W)
        for y, x in np.argwhere(lab != values[np.argmax(up, 0)]):
            assert vo.margin(up[:, y, x:x + 1])[0] < tv.MARGIN, (k, y, x)
            listed.append((k, int(y), int(x)))
    print(f"label pixels inside the margin that differ: {listed}")
    assert len(listed) <= 0.001 * H * W * (n - 1)
    # a refused begin (too many values) leaves the last sequence's labels
    before = v.labels().cpu().numpy()
    many = (np.arange(H * W) % 9).reshape(H, W).astype(np.uint8) * 10 + 1
    with pytest.raises(_lib.BtError, match="9 distinct values"):
        v.begin(_dev(frames[0]), _dev(many))
    assert np.array_equal(v.labels().cpu().numpy(), before)
    v.close()


def test_vos_labels_leave_the_masks_unchanged(cuda_device, sd):
    import test_vos_gpu as tv
    H, W = 97, 131
    frames, m0 = tv.video(10, H, W)
    v = vos.VosDevice(sd, {}, H, W)
    a = tv._run(v, frames, m0)
    b = [v.begin(_dev(frames[0]), _dev(m0)).cpu().numpy()]
    v.labels()
    for f in frames[1:]:
        b.append(v.next(_dev(f)).cpu().numpy())
        v.labels()
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    v.close()


# ---- DAVIS folders end to end ----------------------------------------------------------------------------------------------------
DAVIS_PAL = np.array([[0, 0, 0], [128, 0, 0], [0, 128, 0], [128, 128, 0], [0, 0, 128]] + [[224, 224, 192]] * 251, np.uint8)


def _davis_tree(root, seqs):
    """A DAVIS 2017 layout: JPEGImages/480p/<seq>/*.jpg, Annotations/480p/<seq>/*.png (palette), ImageSets/2017/val.txt."""
    import cv2
    import test_vos_gpu as tv
    for name, (n, H, W, seed) in seqs.items():
        frames, _ = tv.video(n, H, W, seed=seed)
        _, gt = synth.ragged_label_maps(n, H, W, 3, void_from=2, seed=seed)
        for d in ("JPEGImages", "Annotations"):
            os.makedirs(os.path.join(root, d, "480p", name))
        for k in range(n):
            cv2.imwrite(os.path.join(root, "JPEGImages", "480p", name, f"{k:05d}.jpg"), frames[k])
            vos.write_palette_mask(os.path.join(root, "Annotations", "480p", name, f"{k:05d}.png"), gt[k], DAVIS_PAL)
    os.makedirs(os.path.join(root, "ImageSets", "2017"))
    with open(os.path.join(root, "ImageSets", "2017", "val.txt"), "w") as f:
        f.write("".join(f"{s}\n" for s in seqs))


def test_davis_scripts_end_to_end(tmp_path, cuda_device, sd):
    import cv2
    from PIL import Image
    import eval_masks
    import test_mask_objects as tmo
    root, res = str(tmp_path / "DAVIS"), str(tmp_path / "results")
    seqs = {"alpha": (8, 64, 80, 1), "beta": (6, 48, 72, 2)}
    _davis_tree(root, seqs)
    ck = tmp_path / "ck.pth.tar"
    torch.save({"epoch": 1, "state_dict": {"module." + k: torch.from_numpy(x).float() for k, x in sd.items()}, "optimizer": {},
                "scheduler": {}}, ck)
    subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "run_vos.py"), "--davis", root, "--results", res, "--resume", str(ck)],
                   check=True)
    for name, (n, H, W, _) in seqs.items():
        m0, pal = vos.read_palette_mask(os.path.join(root, "Annotations", "480p", name, "00000.png"))
        v = vos.load_vos(str(ck), H=H, W=W)
        for k in range(n):
            path = os.path.join(res, name, f"{k:05d}.png")
            with Image.open(path) as im:
                assert im.mode == "P"
            got, got_pal = vos.read_palette_mask(path)
            assert np.array_equal(got_pal, pal)
            c = torch.from_numpy(cv2.imread(os.path.join(root, "JPEGImages", "480p", name, f"{k:05d}.jpg"), cv2.IMREAD_COLOR)).cuda()
            if k == 0:
                v.begin(c, _dev(m0))
            else:
                v.next(c)
            assert np.array_equal(got, v.labels().cpu().numpy()), (name, k)
        assert np.array_equal(vos.read_palette_mask(os.path.join(res, name, "00000.png"))[0], m0)
        v.close()

    out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "eval_masks.py"), "--davis", root, "--results", res],
                         check=True, capture_output=True, text=True).stdout
    print(out)
    lines = []
    got = eval_masks.evaluate_davis(root, res, out=lines.append)
    assert out.splitlines() == lines
    want_rows = {}
    for name, (n, H, W, _) in seqs.items():
        gt = np.stack([vos.read_palette_mask(os.path.join(root, "Annotations", "480p", name, f"{k:05d}.png"))[0] for k in range(1, n - 1)])
        pred = np.stack([vos.read_palette_mask(os.path.join(res, name, f"{k:05d}.png"))[0] for k in range(1, n - 1)])
        assert (gt == 255).any()
        # the toolkit's semi-supervised path: void is background of the ground truth, and no void mask reaches db_eval_iou / f_measure
        wj, wf, _ = moo.object_metrics(pred, gt, 3, -1)
        gt0 = np.where(gt == 255, 0, gt)
        none = np.zeros(gt.shape[1:], bool)
        assert [[list(tmo._toolkit(p == k, g == k, none)) for k in (1, 2, 3)] for p, g in zip(pred, gt0)] == np.stack([wj, wf], -1).tolist()
        removed = moo.object_metrics(pred, gt, 3, 255)
        assert (pred[gt == 255] != 0).any() and not np.array_equal(np.stack([wj, wf]), np.stack(removed[:2]))
        for k in range(3):
            r = got["objects"][f"{name}_{k + 1}"]
            assert np.array(r["j"]).tobytes() == wj[:, k].tobytes() and np.array(r["f"]).tobytes() == wf[:, k].tobytes(), (name, k)
            assert [r[key] for key in metrics.MASK_SCORE_KEYS] == list(metrics.mask_score(wj[:, k], wf[:, k]).values())
            want_rows[f"{name}_{k + 1}"] = r
    assert list(got["objects"]) == ["alpha_1", "alpha_2", "alpha_3", "beta_1", "beta_2", "beta_3"]
    rows = open(os.path.join(res, "per-sequence_results-val.csv")).read().splitlines()
    assert rows == ["Sequence,J-Mean,F-Mean"] + [f"{s},{r['J-Mean']:.3f},{r['F-Mean']:.3f}" for s, r in want_rows.items()]
    mean = {k: float(np.mean([r[k] for r in want_rows.values()])) for k in metrics.MASK_SCORE_KEYS}
    mean["J&F-Mean"] = (mean["J-Mean"] + mean["F-Mean"]) / 2
    assert got["mean"] == mean
    g = open(os.path.join(res, "global_results-val.csv")).read().splitlines()
    assert g == [",".join(metrics.MASK_SCORE_KEYS), ",".join(f"{mean[k]:.3f}" for k in metrics.MASK_SCORE_KEYS)]


def test_run_vos_davis_skips_a_sequence_with_too_many_objects(tmp_path, cuda_device, sd):
    root, res = str(tmp_path / "DAVIS"), str(tmp_path / "results")
    _davis_tree(root, {"many": (3, 40, 56, 3), "few": (3, 40, 56, 4)})
    many = (np.arange(40 * 56) % 9).reshape(40, 56).astype(np.uint8)          # ids 0..8: 9 label channels
    vos.write_palette_mask(os.path.join(root, "Annotations", "480p", "many", "00000.png"), many, DAVIS_PAL)
    ck = tmp_path / "ck.pth.tar"
    torch.save({"state_dict": {k: torch.from_numpy(x).float() for k, x in sd.items()}}, ck)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "run_vos.py"), "--davis", root, "--results", res, "--resume", str(ck)],
                         check=True, capture_output=True, text=True).stdout
    assert "many: skipped" in out and "9 distinct values" in out and out.rstrip().endswith("skipped 1 sequences: many")
    assert sorted(os.listdir(res)) == ["few"] and len(os.listdir(os.path.join(res, "few"))) == 3
