"""bt_pose_metrics on the device against a float64 numpy / scipy cKDTree restatement of the reference's Utils.add / Utils.adi, on synthetic
models and poses, on the tracker's own output, and through scripts/eval_poses.py against a restatement of eval_ycbineoat.py."""
import os
import sys

import numpy as np
import pytest
from scipy.spatial import cKDTree

from bundletrack_b200 import metrics, policy, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-9     # metres


def transform(T, P):
    return P @ T[:3, :3].T + T[:3, 3]


def add_ref(pred, gt, P):
    return np.array([np.linalg.norm(transform(p, P) - transform(g, P), axis=1).mean() for p, g in zip(pred, gt)])


def adi_ref(pred, gt, P):
    return np.array([cKDTree(transform(p, P)).query(transform(g, P), k=1)[0].mean() for p, g in zip(pred, gt)])


def vocap_ref(rec, max_err=0.1):
    """eval_ycbineoat.py's VOCap."""
    rec = np.sort(np.array(rec, np.float64))
    n = len(rec)
    if n == 0:
        return 0
    prec = np.arange(1, n + 1) / float(n)
    index = np.where(rec < max_err)[0]
    if len(index) == 0:
        return 0
    rec, prec = sorted(rec[index]), sorted(prec[index])
    mrec = np.array([0, *rec, max_err])
    mpre = [0, *prec, prec[-1]]
    for i in range(1, len(mpre)):
        mpre[i] = max(mpre[i], mpre[i - 1])
    mpre = np.array(mpre)
    i = np.where(mrec[1:] != mrec[:-1])[0] + 1
    return np.sum((mrec[i] - mrec[i - 1]) * mpre[i]) * 10


def rand_rot(rng):
    Q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    return Q * np.sign(np.linalg.det(Q))


def model(rng, n):
    """An object-sized cloud: points on a box surface with a few centimetres of extent, off the origin like a YCB model's frame."""
    p = rng.uniform(-1, 1, (n, 3))
    ax = rng.integers(0, 3, n)
    p[np.arange(n), ax] = np.sign(p[np.arange(n), ax] + 1e-9)
    return p * np.array([0.05, 0.08, 0.03]) + np.array([0.01, -0.02, 0.005])


def tracked(rng, F, rot_deg=3.0, trans=0.01):
    """F ground-truth ob_in_cam in front of a camera, and predictions a few degrees / millimetres off."""
    gt, pred = np.zeros((F, 4, 4)), np.zeros((F, 4, 4))
    for f in range(F):
        gt[f] = synth.se3(rand_rot(rng), np.array([0, 0, 0.7]) + rng.normal(0, 0.05, 3))
        d = synth.se3(synth.so3_exp(rng.normal(size=3) * np.deg2rad(rot_deg) / np.sqrt(3)), rng.normal(0, trans, 3))
        pred[f] = d @ gt[f]
    return pred, gt


def check(P, pred, gt, add, adds):
    ra, rs = add_ref(pred, gt, P), adi_ref(pred, gt, P)
    assert np.abs(add - ra).max() <= TOL, np.abs(add - ra).max()
    assert np.abs(adds - rs).max() <= TOL, np.abs(adds - rs).max()
    return ra, rs


@pytest.fixture(scope="module")
def pm(cuda_device):
    m = metrics.PoseMetrics(60000, 2000)
    yield m
    m.close()


SIZES = [(1, 7), (2, 7), (2600, 1), (2600, 7), (3073, 7), (50000, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,F", SIZES)
def test_add_adds_equal_the_kdtree_restatement(pm, n, F):
    rng = np.random.default_rng(100 + n + F)
    P = model(rng, n)
    pred, gt = tracked(rng, F)
    add, adds = pm(P, pred, gt)
    check(P, pred, gt, add, adds)
    assert (adds <= add + 1e-15).all()


@pytest.mark.gpu
def test_two_thousand_frames_in_one_call(pm):
    rng = np.random.default_rng(5)
    P = model(rng, 2600)
    pred, gt = tracked(rng, 2000, rot_deg=8.0, trans=0.02)
    add, adds = pm(P, pred, gt)
    check(P, pred, gt, add, adds)
    # one call of F frames == F calls of one frame == a second run, bit for bit
    add2, adds2 = pm(P, pred, gt)
    assert add.tobytes() == add2.tobytes() and adds.tobytes() == adds2.tobytes()
    for f in (0, 1, 999, 1999):
        a1, s1 = pm(P, pred[f:f + 1], gt[f:f + 1])
        assert a1[0] == add[f] and s1[0] == adds[f], f


@pytest.mark.gpu
def test_identity_poses_give_zero(pm):
    rng = np.random.default_rng(7)
    P = model(rng, 3000)
    T = np.stack([synth.se3(rand_rot(rng), rng.normal(0, 1, 3)) for _ in range(5)])
    add, adds = pm(P, T, T)
    assert (add == 0).all() and (adds == 0).all()


@pytest.mark.gpu
def test_coincident_and_duplicate_points(pm):
    rng = np.random.default_rng(8)
    base = model(rng, 400)
    P = np.concatenate([base, base[:150], np.repeat(base[7:8], 50, 0), np.zeros((20, 3))])
    pred, gt = tracked(rng, 7)
    add, adds = pm(P, pred, gt)
    check(P, pred, gt, add, adds)
    one = np.repeat(base[3:4], 64, 0)                    # every point the same: ADD-S == ADD
    add, adds = pm(one, pred, gt)
    check(one, pred, gt, add, adds)
    assert np.allclose(add, adds, rtol=0, atol=1e-15)


@pytest.mark.gpu
def test_poses_metres_apart(pm):
    rng = np.random.default_rng(9)
    P = model(rng, 2000)
    gt = np.stack([synth.se3(rand_rot(rng), rng.normal(0, 3, 3)) for _ in range(7)])
    pred = np.stack([synth.se3(rand_rot(rng), rng.normal(0, 3, 3)) for _ in range(7)])
    add, adds = pm(P, pred, gt)
    ra, _ = check(P, pred, gt, add, adds)
    assert ra.min() > 0.5


@pytest.mark.gpu
def test_symmetric_model_adds_much_smaller_than_add(pm):
    rng = np.random.default_rng(10)
    d = rng.normal(size=(4000, 3))
    P = 0.05 * d / np.linalg.norm(d, axis=1, keepdims=True) + np.array([0.02, 0.0, -0.01])      # a sphere off the model origin
    c = np.array([0.02, 0.0, -0.01])
    gt = np.stack([synth.se3(rand_rot(rng), np.array([0, 0, 0.8])) for _ in range(7)])
    pred = np.zeros_like(gt)
    for f in range(7):
        R = synth.so3_exp(rng.normal(size=3) / np.sqrt(3) * np.deg2rad(60))          # a large turn about the sphere's centre
        S = synth.se3(R, c - R @ c)
        pred[f] = gt[f] @ S
    add, adds = pm(P, pred, gt)
    check(P, pred, gt, add, adds)
    assert (adds < 0.1 * add).all(), (add, adds)


@pytest.mark.gpu
def test_float32_poses_read_back_from_text(pm, tmp_path):
    """Poses as the tracker writes them (float32, 10 significant digits): their rotations are orthonormal only to ~1e-7."""
    rng = np.random.default_rng(12)
    P = model(rng, 2600)
    pred, gt = tracked(rng, 7, rot_deg=10.0, trans=0.03)
    back = []
    for f in range(7):
        path = str(tmp_path / f"{f}.txt")
        policy.save_pose_txt(path, np.linalg.inv(pred[f]).astype(np.float32))
        back.append(np.loadtxt(path))
    back = np.stack(back)
    add, adds = pm(P, back, gt)
    check(P, back, gt, add, adds)


def ellipsoid_points(seq, n, seed=0):
    """Points on the sequence's ellipsoid, in the model frame (camera frame 0)."""
    d = np.random.default_rng(seed).normal(size=(n, 3))
    x = d / np.linalg.norm(d, axis=1, keepdims=True) * seq.radii
    return transform(seq.ob_in_cam0, x)


@pytest.mark.gpu
def test_tracker_sequence_scored_on_the_device(pm, cuda_device):
    import torch
    from bundletrack_b200 import _lib
    from bundletrack_b200.tracker import Tracker
    H, W, FEATS, N = 240, 320, 400, 30
    seq = synth.make_sequence(31, N, H=H, W=W, n_feats=FEATS)
    trk = Tracker(None, H, W, seq.K, FEATS, 40)
    poses, ks = [], []
    for k in range(N):
        d, m, c = (torch.from_numpy(np.ascontiguousarray(a[k])).to(cuda_device) for a in (seq.depth_raw, seq.mask, seq.colour))
        rq = torch.zeros((400, 400, 3), dtype=torch.uint8, device=cuda_device)
        st, _ = trk.begin_frame(d, m, c, rq, loader_id=0, first_pose=seq.poses_gt[k])
        if st != _lib.BT_FRAME_OTHER:
            continue
        pose, st = trk.end_frame(seq.feats[k]["kpts"], torch.from_numpy(seq.feats[k]["desc"]).to(cuda_device))
        if st in (_lib.BT_FRAME_OTHER, _lib.BT_FRAME_NO_BA):
            poses.append(pose)
            ks.append(k)
    trk.close()
    assert len(ks) >= N - 2
    P = ellipsoid_points(seq, 2600)
    pred = metrics.ob_in_cam(np.stack(poses))
    gt = np.linalg.inv(seq.poses_gt[ks])
    add, adds = pm(P, pred, gt)
    ra, rs = check(P, pred, gt, add, adds)
    auc_adds, auc_add = metrics.vocap(adds) * 100, metrics.vocap(add) * 100
    assert abs(auc_adds - vocap_ref(rs) * 100) <= 1e-10 and abs(auc_add - vocap_ref(ra) * 100) <= 1e-10
    print(f"tracker over {len(ks)} frames: ADD-S AUC {auc_adds:.2f}, ADD AUC {auc_add:.2f}; mean ADD-S {adds.mean() * 1e3:.2f} mm, ADD {add.mean() * 1e3:.2f} mm")


def loadtxt_or_eye(path):
    try:
        return np.loadtxt(path)
    except Exception:
        return np.eye(4)


@pytest.mark.gpu
def test_eval_poses_script_equals_the_reference_evaluation(tmp_path, cuda_device):
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import eval_poses
    rng = np.random.default_rng(13)
    v2o = {"vid_a": "obj_1", "vid_b": "obj_1", "vid_c": "obj_2"}
    ds, res, mdl = tmp_path / "ds", tmp_path / "res", tmp_path / "models"
    models = {"obj_1": model(rng, 900), "obj_2": model(rng, 1700) * 1.5}
    for obj, P in models.items():
        os.makedirs(mdl / obj)
        np.savetxt(mdl / obj / "points.xyz", P)
    expect = {o: {"add": [], "add-s": []} for o in models}
    for v, F in (("vid_a", 40), ("vid_b", 25), ("vid_c", 33)):
        pred, gt = tracked(rng, F, rot_deg=12.0, trans=0.05)
        for sub in ("rgb", "annotated_poses"):
            os.makedirs(ds / v / sub)
        os.makedirs(res / v / "poses")
        for f in range(F):
            (ds / v / "rgb" / f"{f:06d}.png").write_bytes(b"")
            np.savetxt(ds / v / "annotated_poses" / f"{f:06d}.txt", gt[f])
            policy.save_pose_txt(str(res / v / "poses" / f"{f:06d}.txt"), np.linalg.inv(pred[f]).astype(np.float32))
        if v == "vid_b":
            (res / v / "poses" / "000003.txt").write_text("not a pose\n")      # an unreadable prediction counts as the identity
        P = models[v2o[v]]
        pr = np.stack([loadtxt_or_eye(p) for p in sorted((res / v / "poses").glob("*.txt"))])
        gt_back = np.stack([np.loadtxt(p) for p in sorted((ds / v / "annotated_poses").glob("*.txt"))])
        expect[v2o[v]]["add"] += add_ref(pr, gt_back, P).tolist()
        expect[v2o[v]]["add-s"] += adi_ref(pr, gt_back, P).tolist()
    lines = []
    got = eval_poses.evaluate(str(ds), str(mdl), str(res), v2o, out=lines.append)
    for o in models:
        assert abs(got["objects"][o]["adds_auc"] - vocap_ref(expect[o]["add-s"]) * 100) <= 1e-9
        assert abs(got["objects"][o]["add_auc"] - vocap_ref(expect[o]["add"]) * 100) <= 1e-9
        assert np.abs(np.array(got["objects"][o]["add-s"]) - expect[o]["add-s"]).max() <= TOL
    all_adds = expect["obj_1"]["add-s"] + expect["obj_2"]["add-s"]
    all_add = expect["obj_1"]["add"] + expect["obj_2"]["add"]
    assert abs(got["adds_auc"] - vocap_ref(all_adds) * 100) <= 1e-9 and abs(got["add_auc"] - vocap_ref(all_add) * 100) <= 1e-9
    assert got["n"] == 98 and any(l.startswith("ERROR pose file not readable") for l in lines)
    assert lines[-1].startswith("\nOverall, adi=") and "vid_a: #rgb_files=40, #pred_files=40, #gt_files=40" in lines
    assert 0 < got["adds_auc"] < 100
