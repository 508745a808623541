"""GPU tests of object-mask propagation (bt_vos_*) against the float64 restatement of run_video.py (oracle/vos_oracle.py): backbone
features at 480 x 640 and at a size that is no multiple of 8; every step of a 70-frame sequence recomputed from the device's own history
(bt_vos_debug), so one flipped label cannot make the runs diverge; repeat determinism; refusals."""
import os

import numpy as np
import pytest
import torch

from bundletrack_b200 import _lib, vos
from oracle import vos_oracle as vo

pytestmark = pytest.mark.gpu

FEAT_TOL = 1e-4          # of each feature map's largest magnitude
PRED_TOL = 1e-5          # of each prediction map's largest value
MARGIN = 1e-4            # labels and mask pixels may differ where the oracle's top two channels are closer than this
LABEL0_TOL = 1e-5        # frame 0's label: float32 bilinear weights against float64


@pytest.fixture(scope="module")
def sd():
    s = vo.random_state_dict(7, calibrate=video(1, 96, 128, seed=9)[0][0])
    return {k[len("module."):]: v.double().numpy() for k, v in s.items() if not k.endswith("num_batches_tracked")}


def video(n, H, W, seed=3):
    """BGR frames of two discs moving over a textured background, and frame 0's mask (values 0, 3 and 7)."""
    rng = np.random.default_rng(seed)
    bg = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    yy, xx = np.mgrid[:H, :W]
    frames, masks = [], []
    for k in range(n):
        f = bg.copy()
        m = np.zeros((H, W), np.uint8)
        for val, col, (cy, cx, r, vy, vx) in ((3, (40, 200, 60), (0.3, 0.3, 0.18, 0.004, 0.006)), (7, (220, 60, 90), (0.65, 0.7, 0.14, -0.003, -0.005))):
            inside = (yy - (cy + vy * k) * H) ** 2 + (xx - (cx + vx * k) * W) ** 2 < (r * min(H, W)) ** 2
            f[inside] = col
            m[inside] = val
        frames.append(f)
        masks.append(m)
    return frames, masks[0]


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("H,W", [(480, 640), (97, 131)])
def test_backbone_matches_float64(cuda_device, sd, H, W):
    frames, m0 = video(1, H, W)
    v = vos.VosDevice(sd, {}, H, W)
    v.begin(_dev(frames[0]), _dev(m0))
    got = v.debug(0)
    want = vo.features(frames[0], sd).numpy()
    assert got["feat"].shape == want.shape == (-(-H // 8), -(-W // 8), 256)
    err = np.abs(got["feat"] - want).max() / np.abs(want).max()
    f32 = np.abs(vo.features(frames[0], sd, torch.float32).numpy() - want).max() / np.abs(want).max()
    print(f"features {H}x{W}: max |err| / max |f| = {err:.3e} (torch float32 on the CPU: {f32:.3e}), max |f| = {np.abs(want).max():.3g}")
    assert err <= FEAT_TOL
    v.close()


def _run(v, frames, m0):
    return [v.begin(_dev(frames[0]), _dev(m0)).cpu().numpy()] + [v.next(_dev(f)).cpu().numpy() for f in frames[1:]]


@pytest.mark.parametrize("H,W,n", [(48, 64, 70), (97, 131, 20)])
def test_every_step_matches_float64_on_the_device_history(cuda_device, sd, H, W, n):
    """With the defaults: at 48 x 64 for 70 frames, k <= 9, 10..15, > 15 and the ring's wrap (45 slots) all run in one 64-pixel target
    tile; at 97 x 131 (221 grid pixels) 20 frames run over four target tiles, the last one partial."""
    frames, m0 = video(n, H, W)
    P = dict(vos.DEFAULTS)
    v = vos.VosDevice(sd, P, H, W)
    assert np.array_equal(v.begin(_dev(frames[0]), _dev(m0)).cpu().numpy(), np.where(m0 > 0, 255, 0))
    R = v.debug(0)["slots"]
    assert R == 45
    d = vo.compress_labels(m0)[1]
    worst, listed = 0.0, []
    for k in range(1, n):
        mask = v.next(_dev(frames[k])).cpu().numpy()
        dbg = v.debug(k % R)
        Hd, Wd = dbg["Hd"], dbg["Wd"]
        assert dbg["frame"] == k and dbg["n_labels"] == d == 3
        hist = [v.debug(i % R) for i in vo.schedule(k, P["ref_num"], P["range"])]
        pred = vo.predict([h["feat"] for h in hist], [h["label"][..., :d] for h in hist], dbg["feat"], k, P["sigma1"], P["sigma2"],
                          P["temperature"])
        assert not dbg["pred"][d:].any()
        err = np.abs(dbg["pred"][:d] - pred).max() / np.abs(pred).max()
        worst = max(worst, err)
        print(f"frame {k}: prediction err {err:.2e}")
        assert err <= PRED_TOL, (k, err)
        # the new history label: the one-hot of the low-resolution argmax
        lab = dbg["label"].reshape(-1, 8)
        assert np.array_equal(lab, np.eye(8, dtype=np.float32)[np.argmax(lab, 1)])
        bad = np.flatnonzero((np.argmax(lab, 1) != np.argmax(pred, 0)) & (vo.margin(pred) >= MARGIN))
        assert bad.size == 0, (k, bad)
        up = vo.upsample(pred, Hd, Wd, H, W)
        for y, x in np.argwhere(mask != np.where(np.argmax(up, 0) > 0, 255, 0)):
            assert vo.margin(up[:, y, x:x + 1])[0] < MARGIN, (k, y, x)
            listed.append((k, int(y), int(x)))
    print(f"prediction: worst max |err| / max |pred| = {worst:.3e}; mask pixels inside the margin that differ: {listed}")
    assert len(listed) <= 0.001 * H * W * (n - 1)
    v.close()


def test_frame0_label_is_the_resized_one_hot(cuda_device, sd):
    H, W = 97, 131
    frames, m0 = video(1, H, W)
    v = vos.VosDevice(sd, {}, H, W)
    v.begin(_dev(frames[0]), _dev(m0))
    comp, d = vo.compress_labels(m0)
    got = v.debug(0)["label"]
    np.testing.assert_allclose(got[..., :d], vo.init_label(comp, d), atol=LABEL0_TOL)
    assert not got[..., d:].any()
    v.close()


def test_repeat_gives_identical_masks(cuda_device, sd):
    H, W = 97, 131
    frames, m0 = video(24, H, W)
    v = vos.VosDevice(sd, {}, H, W)
    a = _run(v, frames, m0)
    b = _run(v, frames, m0)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    assert any((x == 255).any() for x in a[1:])
    v.close()


def test_refusals(cuda_device, sd):
    H, W = 40, 56
    frames, m0 = video(2, H, W)
    v = vos.VosDevice(sd, {}, H, W)
    with pytest.raises(_lib.BtError, match="bt_vos_begin"):
        v.next(_dev(frames[1]))
    with pytest.raises(ValueError, match="reserved size"):
        v.begin(_dev(frames[0][:-1]), _dev(m0[:-1]))
    many = (np.arange(H * W) % 9).reshape(H, W).astype(np.uint8) * 10 + 1       # 9 values, none of them 0: 10 channels
    with pytest.raises(_lib.BtError, match="9 distinct values"):
        v.begin(_dev(frames[0]), _dev(many))
    eight = (np.arange(H * W) % 8).reshape(H, W).astype(np.uint8)               # 0..7: 8 channels, accepted
    v.begin(_dev(frames[0]), _dev(eight))
    v.next(_dev(frames[1]))
    assert v.debug(0)["n_labels"] == 8
    v.close()


def test_run_vos_script_writes_the_device_masks(tmp_path, cuda_device, sd):
    """scripts/run_vos.py on a checkpoint saved as main.py saves it: frame 0's PNG is the initial mask with > 0 -> 255, the others are
    VosDevice's masks."""
    import cv2
    import subprocess
    import sys
    H, W = 64, 80
    frames, m0 = video(12, H, W)
    (tmp_path / "rgb").mkdir()
    for k, f in enumerate(frames):
        cv2.imwrite(str(tmp_path / "rgb" / f"{k:04d}.png"), f)
    cv2.imwrite(str(tmp_path / "init.png"), m0)
    ck = tmp_path / "ck.pth.tar"
    torch.save({"epoch": 1, "state_dict": {"module." + k: torch.from_numpy(x).float() for k, x in sd.items()}, "optimizer": {},
                "scheduler": {}}, ck)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.run([sys.executable, os.path.join(root, "scripts", "run_vos.py"), "--img_dir", str(tmp_path / "rgb"), "--init_mask_file",
                    str(tmp_path / "init.png"), "--mask_save_dir", str(tmp_path / "out"), "--resume", str(ck)], check=True)
    v = vos.load_vos(str(ck), H=H, W=W)
    want = _run(v, frames, m0)
    v.close()
    for k in range(len(frames)):
        got = cv2.imread(str(tmp_path / "out" / f"{k:04d}.png"), cv2.IMREAD_UNCHANGED)
        assert np.array_equal(got, want[k]), k
    assert np.array_equal(want[0], np.where(m0 > 0, 255, 0))


def test_run_sequence_with_the_vos_source_equals_reading_its_pngs(tmp_path, cuda_device, sd):
    """run_sequence with masks=VosSource on a synthetic YCBInEOAT-layout scene writes pose files byte-identical to a run that reads the
    PNGs the source wrote (mask_save_dir) in place of the scene's masks; frame 0's PNG is the initial mask with > 0 -> 255."""
    import shutil
    import test_sequence_gpu as tsg
    from bundletrack_b200 import sequence, synth
    H, W, FEATS, N = 240, 320, 400, 12
    seq = synth.make_sequence(52, N, H=H, W=W, n_feats=FEATS, detect_fail=(6,))
    video = tmp_path / "synthvideo"
    tsg._write_frames(seq, lambda k: f"{video}/rgb/{k:07d}.png", lambda k: f"{video}/depth/{k:07d}.png", lambda k: f"{video}/masks/{k:07d}.png")
    K = np.array([[seq.K[0], 0, seq.K[2]], [0, seq.K[1], seq.K[3]], [0, 0, 1]])
    (video / "cam_K.txt").write_text("".join(" ".join(f"{v:.9g}" for v in row) + "\n" for row in K))
    (video / "annotated_poses").mkdir()
    for k in range(N):
        G = np.linalg.inv(np.asarray(seq.poses_gt[k], np.float64))
        (video / "annotated_poses" / f"{k:07d}.txt").write_text("".join(" ".join(f"{v:.9g}" for v in row) + "\n" for row in G))
    ck = tmp_path / "ck.pth.tar"
    torch.save({"epoch": 1, "state_dict": {"module." + k: torch.from_numpy(x).float() for k, x in sd.items()}}, ck)
    init = str(tmp_path / "init.png")
    shutil.copy(f"{video}/masks/{0:07d}.png", init)
    shutil.rmtree(video / "masks")                       # the VOS run must not need the scene's masks
    before = tsg._live()
    src = vos.load_source(str(ck), init, H, W, mask_save_dir=str(tmp_path / "vos_masks"))
    res_vos = sequence.run_sequence(sequence.YcbineoatVideo(str(video)), None, tsg._features(seq), str(tmp_path / "run_vos"),
                                    max_feats=FEATS, masks=src)
    src.close()
    assert tsg._live() == before
    written = sorted(os.listdir(tmp_path / "vos_masks"))
    assert written == [f"{k:07d}.png" for k in range(N)]
    assert np.array_equal(sequence.read_image(str(tmp_path / "vos_masks" / written[0]), "mask"), np.where(seq.mask[0] > 0, 255, 0))
    shutil.copytree(tmp_path / "vos_masks", video / "masks")
    res_png = sequence.run_sequence(sequence.YcbineoatVideo(str(video)), None, tsg._features(seq), str(tmp_path / "run_png"), max_feats=FEATS)
    assert tsg._files(str(tmp_path / "run_vos" / "poses")) == tsg._files(str(tmp_path / "run_png" / "poses"))
    assert [r[:2] for r in res_vos] == [r[:2] for r in res_png]
    assert len(res_vos) == N
    print("vos source run:", sequence.summary(res_vos))
