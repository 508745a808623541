"""The tracking overlay on the device against the numpy oracle (oracle/overlay_oracle.py): bt_voxel_downsample bit for bit (count, order,
centroids), bt_pose_overlay byte for byte (viz and raw) and against the OpenCV-drawn golden frames, batches against single calls, a logging
run of run_sequence on a synthetic NOCS tree, and no resource left behind."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest

from bundletrack_b200 import _lib, sequence, synth
from bundletrack_b200.overlay import TILE, Overlay, VoxelGrid
from oracle import overlay_oracle as oo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
K640 = (590.0, 590.0, 322.5, 244.1)


def _live():
    lib = _lib.load()
    d, p, h = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_int()
    assert lib.bt_debug_live_resources(ctypes.byref(d), ctypes.byref(p), ctypes.byref(h)) == 0
    return d.value, p.value, h.value


def same(a, b):
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def _cloud(seed, n, spread=0.3):
    rng = np.random.default_rng(seed)
    p = (rng.normal(size=(n, 3)) * spread + rng.normal(size=3)).astype(F32)
    if n > 10:
        p[rng.random(n) < 0.01, rng.integers(0, 3)] = np.nan
    return p


SIZES = [1, 2, TILE - 1, TILE, TILE + 1, 2 * TILE - 1, 2 * TILE + 1, 200_000]


@pytest.mark.gpu
def test_voxel_downsample_equals_oracle(cuda_device):
    vg = VoxelGrid(200_000, 16)
    try:
        for n in SIZES:
            p = _cloud(n, n)
            for leaf in (0.01, 0.05):
                got = vg([p], leaf)[0]
                assert same(got, oo.voxel_grid(p, leaf)), (n, leaf)
        # every point in one voxel, at the tile sizes and large
        for n in (TILE - 1, TILE + 1, 100_000):
            rng = np.random.default_rng(n)
            p = (F32(-0.2995) + rng.random((n, 3)).astype(F32) * F32(0.009)).astype(F32)
            got = vg([p], 0.01)[0]
            assert got.shape == (1, 3) and same(got, oo.voxel_grid(p, 0.01)), n
        # the overflow rule: leaf 1e-6 over a 10 m cloud returns the input, non-finite points included
        p = (np.random.default_rng(5).random((3000, 3)) * 10).astype(F32)
        p[11] = np.nan
        got = vg([p], 1e-6)[0]
        assert same(got, p)
        # only non-finite points: nothing
        assert vg([np.full((5, 3), np.nan, F32)], 0.01)[0].shape == (0, 3)
    finally:
        vg.close()


@pytest.mark.gpu
def test_voxel_downsample_batch_equals_single_calls(cuda_device):
    rng = np.random.default_rng(7)
    sizes = [1, 2, 17, TILE - 1, TILE, TILE + 1, 5000, 1, 30000, 3, TILE * 3 + 5, 999, 2, 12345, 60, 4097]
    clouds = [_cloud(100 + k, n, spread=float(rng.uniform(0.01, 1.0))) for k, n in enumerate(sizes)]
    clouds[5] = (np.random.default_rng(9).random((TILE, 3)) * 10).astype(F32)        # overflows at 1e-6, inside a batch
    vg = VoxelGrid(max(sizes), 16)
    try:
        for leaf in (0.01, 1e-6):
            batch = vg(clouds, leaf)
            for k, c in enumerate(clouds):
                single = vg([c], leaf)[0]
                assert same(batch[k], single), (k, leaf)
                if leaf == 0.01:
                    assert same(single, oo.voxel_grid(c, leaf)), k
    finally:
        vg.close()


def _frames(seed, F, H=480, W=640):
    rng = np.random.default_rng(seed)
    colour = rng.integers(0, 256, (F, H, W, 3), dtype=np.uint8)
    vv, uu = np.mgrid[0:H, 0:W]
    fg = np.stack([((((uu - rng.uniform(0, W)) / 150) ** 2 + ((vv - rng.uniform(0, H)) / 100) ** 2) <= 1) for _ in range(F)]).astype(np.uint8)
    return colour, fg


def _border_poses(seed, F, K, H=480, W=640):
    """Poses whose model centre projects at or just past every border and corner, a few near z = 0 (points behind the camera)."""
    rng = np.random.default_rng(seed)
    fx, fy, cx, cy = K
    targets = [(0, 0), (W - 1, 0), (0, H - 1), (W - 1, H - 1), (-3, H / 2), (W + 2, H / 3), (W / 2, -2), (W / 3, H + 1), (W / 2, H / 2)]
    poses = []
    for f in range(F):
        u, v = targets[f % len(targets)]
        z = 0.015 if f % len(targets) == len(targets) - 1 else float(rng.uniform(0.4, 1.2))
        t = np.array([(u - cx) * z / fx, (v - cy) * z / fy, z])
        ob_in_cam = synth.se3(synth.so3_exp(rng.normal(size=3)), t)
        poses.append(np.linalg.inv(ob_in_cam).astype(F32))
    return np.stack(poses)


@pytest.mark.gpu
@pytest.mark.parametrize("n_model", [500, 5000, 50000])
def test_pose_overlay_equals_oracle(cuda_device, n_model):
    model = synth.make_ellipsoid_model(n_model, n_model, radii=(0.08, 0.06, 0.05))
    F = 9
    colour, fg = _frames(n_model, F)
    poses = _border_poses(n_model, F, K640)
    ov = Overlay(model, K640, 480, 640, max_frames=F)
    try:
        assert same(ov.model, oo.voxel_grid(model, 0.015))
        viz, raw = ov.render_host(poses, colour, fg)
        for f in range(F):
            want_viz, want_raw = oo.render(colour[f], fg[f], ov.model, poses[f], K640)
            assert same(viz[f], want_viz), (n_model, f, int((viz[f] != want_viz).any(-1).sum()))
            assert same(raw[f], want_raw), (n_model, f)
        stamped = (viz == np.array([0, 255, 255], np.uint8)).all(-1)
        assert stamped[:, 0, :].any() and stamped[:, -1, :].any() and stamped[:, :, 0].any() and stamped[:, :, -1].any()
    finally:
        ov.close()


@pytest.mark.gpu
def test_pose_overlay_batch_equals_single_calls(cuda_device):
    model = synth.make_ellipsoid_model(3, 20000, radii=(0.1, 0.07, 0.05))
    F = 32
    colour, fg = _frames(11, F)
    poses = _border_poses(12, F, K640)
    ov = Overlay(model, K640, 480, 640, max_frames=F)
    try:
        viz, raw = ov.render_host(poses, colour, fg)
        for f in range(F):
            v1, r1 = ov.render_host(poses[f:f + 1], colour[f:f + 1], fg[f:f + 1])
            assert same(v1[0], viz[f]) and same(r1[0], raw[f]), f
    finally:
        ov.close()


@pytest.mark.gpu
def test_pose_overlay_equals_golden_frames(cuda_device):
    g = np.load(os.path.join(ROOT, "tests", "golden", "ref_overlay.npz"))
    F, H, W = g["colour"].shape[:3]
    ov = Overlay(g["model"], g["K"], H, W, max_frames=F)
    try:
        assert same(ov.model, oo.voxel_grid(g["model"], 0.015))
        viz, raw = ov.render_host(g["cur_in_model"], g["colour"], g["fg"])
        for f in range(F):
            keep = ~g["label_mask"][f]
            assert np.array_equal(viz[f][keep], g["viz"][f][keep]), f
            assert same(raw[f], g["raw"][f]), f
    finally:
        ov.close()


@pytest.mark.gpu
def test_overlay_context_frees_everything(cuda_device):
    before = _live()
    ov = Overlay(synth.make_ellipsoid_model(1, 1000), K640, 480, 640, max_frames=4)
    ov.render_host(_border_poses(1, 4, K640), *_frames(1, 4))
    ov.close()
    assert _live() == before


# ---- a logging run ------------------------------------------------------------------------------------------------------------------------

def _seq_gpu():
    spec = importlib.util.spec_from_file_location("seq_gpu_helpers", os.path.join(ROOT, "tests", "test_sequence_gpu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.gpu
def test_run_sequence_log_writes_every_frame(tmp_path, cuda_device):
    cv2 = pytest.importorskip("cv2")
    import torch
    from bundletrack_b200.overlay import label, load_obj_points
    sg = _seq_gpu()          # the synthetic NOCS tree test_sequence_gpu.py builds, rebuilt here
    H, W, FEATS, N = 240, 320, 400, 14
    seq = synth.make_sequence(31, N, H=H, W=W, n_feats=FEATS, roi_fail=(5,), detect_fail=(9,))
    nocs_dir, mask_dir = sg._nocs_scene(str(tmp_path), seq)
    model = synth.make_ellipsoid_model(2, 4000, radii=seq.radii)
    os.makedirs(f"{nocs_dir}/obj_models/real_test", exist_ok=True)
    with open(f"{nocs_dir}/obj_models/real_test/camera_tracked_norm.obj", "w") as f:
        f.write("".join(f"v {x:.9g} {y:.9g} {z:.9g}\n" for x, y, z in model.astype(np.float64)))
    loader = sequence.NocsScene(nocs_dir, 4, "camera_tracked_norm", mask_dir)
    before = _live()
    outs = {}
    for log in (0, 1):
        out = str(tmp_path / f"log{log}")
        outs[log] = (out, sequence.run_sequence(loader, None, sg._features(seq), out, max_feats=FEATS, device=0, log=log))
        assert _live() == before
    assert sg._files(f"{outs[0][0]}/poses") == sg._files(f"{outs[1][0]}/poses")
    assert sorted(os.listdir(outs[0][0])) == ["poses"]
    st = {i: s for i, s, _ in outs[1][1]}
    assert st["0005"] == _lib.BT_FRAME_FAIL and st["0009"] == _lib.BT_FRAME_FAIL
    # the tracker's fg per frame, from a hand loop over the same frames
    from bundletrack_b200.tracker import Tracker
    trk = Tracker(None, H, W, loader.K, FEATS, 2 + 4, mode=loader.mask_mode, max_keyframes=-(-N // 2))
    rq = torch.zeros((400, 400, 3), dtype=torch.uint8, device=cuda_device)
    fgs = {}
    try:
        for i, ff in enumerate(loader.frames):
            d, m, c = sequence.read_frame(ff)
            s, roi, _, pose = trk.begin_frame_mm(sg._dev(d, cuda_device), sg._dev(m, cuda_device), sg._dev(c, cuda_device), rq, loader_id=i,
                                                 first_pose=loader.initial_pose(i))
            torch.cuda.synchronize()
            fg = np.empty((H, W), np.uint8)
            _lib.check(_lib.load().bt_memcpy_d2h(fg.ctypes.data_as(ctypes.c_void_p), ctypes.c_void_p(trk.last_fg()), ctypes.c_size_t(H * W), None))
            fgs[ff.id_str] = fg
            if s == _lib.BT_FRAME_OTHER:
                f = seq.feats[i]
                if f is None:
                    trk.drop_frame()
                else:
                    trk.end_frame(f["kpts"], torch.from_numpy(f["desc"]).to(cuda_device))
    finally:
        trk.close()
    mdl = oo.voxel_grid(load_obj_points(loader.model_path), 0.015)
    out = outs[1][0]
    n_stamped = 0
    for ff in loader.frames:
        i = ff.id_str
        paths = [f"{out}/{i}/color_viz.jpg", f"{out}/color_viz/{i}_color_viz.jpg", f"{out}/color_raw/{i}_color_raw.png"]
        assert all(os.path.exists(p) for p in paths), i
        colour = sequence.read_image(ff.colour, "colour")
        raw = cv2.imread(paths[2], cv2.IMREAD_UNCHANGED)
        assert same(raw, np.where((fgs[i] != 0)[..., None], colour, 0).astype(np.uint8)), i
        pose = np.loadtxt(f"{out}/poses/{i}.txt").astype(F32)
        cur_in_model = np.linalg.inv(pose.astype(np.float64)).astype(F32)
        viz, _ = oo.render(colour, fgs[i], mdl, cur_in_model, loader.K[[0, 1, 0, 1], [0, 1, 2, 2]])
        want = label(viz, i).astype(np.int16)
        got = cv2.imread(paths[0], cv2.IMREAD_COLOR).astype(np.int16)
        assert open(paths[0], "rb").read() == open(paths[1], "rb").read()
        err = np.abs(got - want)
        assert err.mean() < 3.0 and np.percentile(err, 99) < 40, (i, err.mean(), np.percentile(err, 99))
        n_stamped += int((viz == np.array([0, 255, 255], np.uint8)).all(-1).sum())
    assert n_stamped > 0
