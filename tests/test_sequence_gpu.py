"""16-bit depth into the front end and the tracker (bt_frames_preprocess_masked_u16, bt_tracker_begin_frame_u16) against the float entry
points on the host's readDepthImage conversion, and whole runs of bundletrack_b200.sequence.run_sequence on synthetic NOCS and YCBInEOAT
trees: one pose file per frame, identical to a hand loop and across prefetch depths, scored by the evaluation scripts, no resource left."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest

from bundletrack_b200 import _lib, policy, sequence, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _script(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "scripts", f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def read_depth_image(mm: np.ndarray) -> np.ndarray:
    """Utils::readDepthImage (Utils.cpp:57-66) in numpy float64: (float)s * 0.001 in double, rounded to float, 0 below 0.1 m."""
    d = (mm.astype(np.float64) * 0.001).astype(np.float32)
    d[d.astype(np.float64) < 0.1] = 0
    return d


def _dev(a, dev):
    import torch
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint16:
        return torch.from_numpy(a.view(np.int16)).to(dev).view(torch.uint16)
    return torch.from_numpy(a).to(dev)


def _live():
    lib = _lib.load()
    d, p, h = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_int()
    assert lib.bt_debug_live_resources(ctypes.byref(d), ctypes.byref(p), ctypes.byref(h)) == 0
    return d.value, p.value, h.value


def test_read_depth_image_gate():
    d = read_depth_image(np.arange(65536, dtype=np.uint16))
    assert d[99] == 0 and d[100] == np.float32(0.1) and d[100] > 0
    assert (d[:100] == 0).all() and (d[100:] > 0).all()


OTHER_PARAMS = {"depth_processing": {"erode": {"radius": 2, "diff": 0.003, "ratio": 0.6},
                                     "bilateral_filter": {"radius": 1, "sigma_D": 3, "sigma_R": 0.05}}}


@pytest.mark.gpu
@pytest.mark.parametrize("params", ["shipped", "other"])
@pytest.mark.parametrize("mode", [_lib.BT_MASK_AS_IS, _lib.BT_MASK_LARGEST_HULL])
def test_u16_front_end_equals_float_on_converted_depth(cuda_device, params, mode):
    import torch
    from bundletrack_b200.config import NOCS_DEFAULTS
    from bundletrack_b200.frontend import FrameFrontEnd
    yml = None if params == "shipped" else dict(NOCS_DEFAULTS, **OTHER_PARAMS)
    every = np.arange(65536, dtype=np.uint32).reshape(256, 256)
    every = np.ascontiguousarray(every.T if mode == _lib.BT_MASK_AS_IS else every).astype(np.uint16)   # every sample value, two layouts
    cases = [(every, synth.make_object_mask(1, 256, 256), synth.NOCS_K)]
    for seed, (H, W) in ((2, (240, 320)), (3, (480, 640)), (4, (97, 131))):
        raw, K = synth.make_raw_depth(seed, H, W)
        cases.append((synth.depth_mm(raw), synth.make_object_mask(seed, H, W), K))
    fe = FrameFrontEnd(yml)
    try:
        for mm, mask, K in cases:
            H, W = mm.shape
            outs = {}
            for kind, depth in (("u16", _dev(mm, cuda_device)), ("f32", _dev(read_depth_image(mm), cuda_device))):
                d = torch.full((H, W), -1.0, device=cuda_device)
                x, n = torch.full((H, W, 4), -1.0, device=cuda_device), torch.full((H, W, 4), -1.0, device=cuda_device)
                fg = torch.full((H, W), 7, dtype=torch.uint8, device=cuda_device)
                roi = fe.process_masked([depth], [_dev(mask, cuda_device)], H, W, K, [d], [n], [fg], xyz_out=[x], mode=mode)
                torch.cuda.synchronize()
                outs[kind] = [t.cpu().numpy() for t in (d, x, n, fg)] + [roi]
            for name, a, b in zip(("depth", "xyz", "normal", "fg", "roi"), outs["u16"], outs["f32"]):
                assert a.tobytes() == b.tobytes(), (name, mm.shape)
            if mm is not every:                  # (the every-value image steps 1 mm one way and 256 mm the other: it may erode to nothing)
                assert (outs["u16"][0] > 0).any()
    finally:
        fe.close()


@pytest.mark.gpu
def test_front_end_refuses_mixed_depth_types(cuda_device):
    import torch
    from bundletrack_b200.frontend import FrameFrontEnd
    fe = FrameFrontEnd()
    try:
        H, W = 16, 16
        z = lambda dt: torch.empty((H, W), dtype=dt, device=cuda_device)
        with pytest.raises(_lib.BtError, match="float32 or all uint16"):
            fe.process_masked([z(torch.float32), z(torch.uint16)], [z(torch.uint8)] * 2, H, W, synth.NOCS_K, [z(torch.float32)] * 2,
                              [torch.empty((H, W, 4), device=cuda_device)] * 2, [z(torch.uint8)] * 2)
    finally:
        fe.close()


@pytest.mark.gpu
def test_begin_frame_u16_equals_begin_frame(cuda_device):
    """Two trackers, one fed the depth PNG's millimetres and one the host's readDepthImage floats, over a sequence with a ROI failure of the
    first frame, a later ROI failure and a dropped detection: the same statuses, poses and request images, and begin_frame_u16's id and pose
    are the reference's (loader id and first pose with no frame alive, else the newest frame's id + 1 and pose)."""
    import torch
    from bundletrack_b200.tracker import Tracker
    H, W, FEATS, N = 240, 320, 400, 16
    seq = synth.make_sequence(41, N, H=H, W=W, n_feats=FEATS, roi_fail=(0, 7), detect_fail=(4, 11))
    a, b = Tracker(None, H, W, seq.K, FEATS, 8, max_keyframes=N), Tracker(None, H, W, seq.K, FEATS, 8, max_keyframes=N)
    rqa = torch.zeros((400, 400, 3), dtype=torch.uint8, device=cuda_device)
    rqb = torch.zeros_like(rqa)
    first = np.asarray(seq.poses_gt[0], np.float32) @ synth.se3(synth.so3_exp(np.array([0.01, -0.02, 0.01])), np.array([0.003, 0.0, -0.002])).astype(np.float32)
    statuses = []
    try:
        for k in range(N):
            mm = synth.depth_mm(seq.depth_raw[k])
            m, c = _dev(seq.mask[k], cuda_device), _dev(seq.colour[k], cuda_device)
            fp = first if k == 0 else np.eye(4, dtype=np.float32)
            ids, poses, _ = a.state()
            exp_id, exp_pose = (k, fp) if len(ids) == 0 else (int(ids.max()) + 1, poses[np.argmax(ids)])
            sa, roia, fid, pose0 = a.begin_frame_mm(_dev(mm, cuda_device), m, c, rqa, loader_id=k, first_pose=fp)
            sb, roib = b.begin_frame(_dev(read_depth_image(mm), cuda_device), m, c, rqb, loader_id=k, first_pose=fp)
            assert (sa, roia.tolist()) == (sb, roib.tolist()), k
            assert fid == exp_id and np.array_equal(pose0, exp_pose), (k, fid, exp_id)
            if sa == _lib.BT_FRAME_FAIL:
                statuses.append(("roi", k))
                continue
            assert torch.equal(rqa, rqb), k
            if seq.feats[k] is None:
                pa, pb = a.drop_frame(), b.drop_frame()
                assert np.array_equal(pa, pb) and np.array_equal(pa, pose0)
                statuses.append(("drop", k))
                continue
            desc = torch.from_numpy(seq.feats[k]["desc"]).to(cuda_device)
            pa, sa = a.end_frame(seq.feats[k]["kpts"], desc)
            pb, sb = b.end_frame(seq.feats[k]["kpts"], desc)
            assert sa == sb and np.array_equal(pa, pb), k
            statuses.append((sa, k))
    finally:
        a.close()
        b.close()
    assert ("roi", 0) in statuses and ("roi", 7) in statuses and ("drop", 4) in statuses and ("drop", 11) in statuses
    assert sum(s in (_lib.BT_FRAME_OTHER, _lib.BT_FRAME_NO_BA) for s, _ in statuses) >= N - 5, statuses


# ---- whole runs ---------------------------------------------------------------------------------------------------------------------------

def _features(seq):
    def source(id_str, request, roi):
        f = seq.feats[int(id_str)]
        if f is None:
            raise sequence.DetectionFailed(f"frame {id_str}: no features")
        return f["kpts"], f["desc"]
    return source


def _write_frames(seq, colour_path, depth_path, mask_path):
    for k in range(seq.n_frames):
        for path, img in ((colour_path(k), seq.colour[k]), (depth_path(k), synth.depth_mm(seq.depth_raw[k])), (mask_path(k), seq.mask[k])):
            os.makedirs(os.path.dirname(path), exist_ok=True)
            synth.write_png(path, img)


def _nocs_scene(tmp, seq, model="camera_tracked_norm", scene=4):
    """make_golden_nocs's synthetic tree plus one tracked (model, scene) with images, masks, the text ground truth and the benchmark's inputs."""
    import pickle
    mk = _script("make_golden_nocs")
    nocs_dir, _ = mk.write_tree(tmp, mk.make_tree(3, n_frames=6, anomalies=False))
    N = seq.n_frames
    data = f"{nocs_dir}/real_test/scene_{scene}"
    mask_dir = f"{tmp}/masks/scene_{scene}_model_{model}"
    _write_frames(seq, lambda k: f"{data}/{k:04d}_color.png", lambda k: f"{data}/{k:04d}_depth.png", lambda k: f"{mask_dir}/{k:04d}.png")
    gt_txt = f"{nocs_dir}/gts/real_test_text/scene_{scene}/model_{model}"
    os.makedirs(gt_txt)
    for k in range(N):
        G = np.linalg.inv(np.asarray(seq.poses_gt[k], np.float64))          # ob_in_cam: the model frame is camera frame 0
        with open(f"{gt_txt}/{k:04d}.txt", "w") as f:
            f.write("".join(" ".join(f"{v:.9g}" for v in row) + "\n" for row in G))
        with open(f"{data}/{k:04d}_meta.txt", "w") as f:
            f.write(f"1 3 {model}\n")
        with open(f"{nocs_dir}/gts/real_test/results_real_test_scene_{scene}_{k:04d}.pkl", "wb") as f:
            pickle.dump({"gt_RTs": np.asarray([G])}, f)
    r = np.asarray(seq.radii) * 1000
    corners = np.array([[sx * r[0], sy * r[1], sz * r[2]] for sx in (1, -1) for sy in (1, -1) for sz in (1, -1)])
    with open(f"{nocs_dir}/NOCS-REAL275-additional/model_scales/{model}.txt", "w") as f:
        f.write("".join(f"{x:.6f} {y:.6f} {z:.6f}\n" for x, y, z in corners))
    os.makedirs(f"{nocs_dir}/NOCS-REAL275-additional/data_list/real_val/3/{model}")
    with open(f"{nocs_dir}/NOCS-REAL275-additional/data_list/real_val/3/{model}/list.txt", "w") as f:
        f.write("".join(f"real_val/scene_{scene}/{k:04d}\n" for k in range(N)))
    return nocs_dir, mask_dir


def _hand_loop(loader, features, out_dir, max_feats, dev):
    """run_sequence's rules written out over the same decoded arrays, without the reader."""
    import torch
    from bundletrack_b200.tracker import Tracker
    W, H = sequence.png_layout(loader.frames[0].colour)[:2]
    trk = Tracker(None, H, W, loader.K, max_feats, 2 + 4, mode=loader.mask_mode, max_keyframes=-(-len(loader) // 2))
    os.makedirs(f"{out_dir}/poses", exist_ok=True)
    rq = torch.zeros((400, 400, 3), dtype=torch.uint8, device=dev)
    try:
        for i, ff in enumerate(loader.frames):
            d, m, c = sequence.read_frame(ff)
            st, roi, _, pose = trk.begin_frame_mm(_dev(d, dev), _dev(m, dev), _dev(c, dev), rq, loader_id=i, first_pose=loader.initial_pose(i))
            if st == _lib.BT_FRAME_OTHER:
                try:
                    kp, de = features(ff.id_str, rq.cpu().numpy(), roi)
                except sequence.DetectionFailed:
                    pose = trk.drop_frame()
                else:
                    pose, st = trk.end_frame(kp, torch.from_numpy(de).to(dev))
            policy.save_pose_txt(f"{out_dir}/poses/{ff.id_str}.txt", pose)
    finally:
        trk.close()


def _files(d):
    return {f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d))}


@pytest.mark.gpu
def test_run_sequence_on_a_nocs_tree(tmp_path, cuda_device):
    try:
        import PIL  # noqa: F401
        have_pil = True
    except ImportError:
        have_pil = False
    if not (sequence._have_cv2() or have_pil):
        pytest.skip("needs cv2 or PIL")
    H, W, FEATS, N = 240, 320, 400, 20
    seq = synth.make_sequence(31, N, H=H, W=W, n_feats=FEATS, roi_fail=(5,), detect_fail=(9,))
    nocs_dir, mask_dir = _nocs_scene(str(tmp_path), seq)
    loader = sequence.NocsScene(nocs_dir, 4, "camera_tracked_norm", mask_dir)
    assert [f.id_str for f in loader.frames] == [f"{k:04d}" for k in range(N)]
    before = _live()
    res = {}
    for pf in (2, 0):
        out = str(tmp_path / f"results_p{pf}" / "camera_tracked_norm_4")
        res[pf] = sequence.run_sequence(loader, None, _features(seq), out, max_feats=FEATS, device=0, prefetch=pf)
        assert _live() == before
    hand = str(tmp_path / "results_hand" / "camera_tracked_norm_4")
    _hand_loop(loader, _features(seq), hand, FEATS, cuda_device)
    files = {k: _files(str(tmp_path / f"results_{k}" / "camera_tracked_norm_4" / "poses")) for k in ("p2", "p0", "hand")}
    assert sorted(files["p2"]) == [f"{k:04d}.txt" for k in range(N)]
    assert files["p2"] == files["hand"] and files["p0"] == files["hand"]
    st = dict((i, s) for i, s, _ in res[2])
    assert st["0005"] == _lib.BT_FRAME_FAIL and st["0009"] == _lib.BT_FRAME_FAIL
    assert [r[:2] for r in res[2]] == [r[:2] for r in res[0]]
    assert sum(s != _lib.BT_FRAME_FAIL for s in st.values()) >= N - 4
    ev = _script("eval_nocs")
    for noise in (None, (0.02, 0.0)):
        r_run = ev.evaluate(nocs_dir, str(tmp_path / "results_p2"), noise, out=lambda *a: None)
        r_hand = ev.evaluate(nocs_dir, str(tmp_path / "results_hand"), noise, out=lambda *a: None)
        for key in ("5cm5deg", "iou25", "rot_err", "tran_err", "n", "n_scored"):
            assert np.array_equal(r_run[key], r_hand[key], equal_nan=True), key
        for key in ("theta", "shift", "iou"):
            assert np.array_equal(r_run["records"][key], r_hand["records"][key], equal_nan=True), key
        assert r_run["n_scored"] >= N
    print("nocs run:", sequence.summary(res[2]))


@pytest.mark.gpu
def test_run_sequence_ycbineoat_layout_scored(tmp_path, cuda_device):
    H, W, FEATS, N = 240, 320, 400, 12
    seq = synth.make_sequence(52, N, H=H, W=W, n_feats=FEATS, detect_fail=(6,))
    video = tmp_path / "data" / "synthvideo"
    _write_frames(seq, lambda k: f"{video}/rgb/{k:07d}.png", lambda k: f"{video}/depth/{k:07d}.png", lambda k: f"{video}/masks/{k:07d}.png")
    K = np.array([[seq.K[0], 0, seq.K[2]], [0, seq.K[1], seq.K[3]], [0, 0, 1]])
    (video / "cam_K.txt").write_text("".join(" ".join(f"{v:.9g}" for v in row) + "\n" for row in K))
    (video / "annotated_poses").mkdir()
    for k in range(N):
        G = np.linalg.inv(np.asarray(seq.poses_gt[k], np.float64))
        (video / "annotated_poses" / f"{k:07d}.txt").write_text("".join(" ".join(f"{v:.9g}" for v in row) + "\n" for row in G))
    rng = np.random.default_rng(0)
    u = rng.normal(size=(500, 3))
    pts = u / np.linalg.norm(u, axis=1, keepdims=True) * np.asarray(seq.radii)
    (tmp_path / "models" / "synth_object").mkdir(parents=True)
    np.savetxt(tmp_path / "models" / "synth_object" / "points.xyz", pts)
    loader = sequence.YcbineoatVideo(str(video))
    before = _live()
    res = sequence.run_sequence(loader, None, _features(seq), str(tmp_path / "results" / "synthvideo"), max_feats=FEATS, device=0)
    assert _live() == before
    assert len(res) == N and res[6][1] == _lib.BT_FRAME_FAIL
    lines = []
    r = _script("eval_poses").evaluate(str(tmp_path / "data"), str(tmp_path / "models"), str(tmp_path / "results"), {"synthvideo": "synth_object"},
                                       out=lines.append)
    assert r["n"] == N and f"synthvideo: #rgb_files={N}, #pred_files={N}, #gt_files={N}" in lines
    print("ycbineoat run:", sequence.summary(res), "ADD-S AUC", r["adds_auc"])


@pytest.mark.gpu
def test_capacity_stops_the_run_and_frees_everything(tmp_path, cuda_device):
    H, W, FEATS, N = 240, 320, 400, 6
    seq = synth.make_sequence(63, N, H=H, W=W, n_feats=FEATS)
    nocs_dir, mask_dir = _nocs_scene(str(tmp_path), seq)
    loader = sequence.NocsScene(nocs_dir, 4, "camera_tracked_norm", mask_dir)
    before = _live()
    with pytest.raises(_lib.BtError, match="max_keyframes") as e:
        sequence.run_sequence(loader, None, _features(seq), str(tmp_path / "out"), max_feats=FEATS, max_keyframes=1, device=0)
    assert e.value.rc == _lib.BT_ERR_CAPACITY
    assert _live() == before
    assert os.listdir(tmp_path / "out" / "poses") == ["0000.txt"]
