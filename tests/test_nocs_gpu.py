"""bt_nocs_metrics on the device against the reference's own 6-PACK benchmark (tests/golden/ref_nocs.npz) and the numpy oracle, per record
and through scripts/eval_nocs.py; call structure, context resources, and a tracked sequence scored end to end."""
import ctypes
import importlib.util
import json
import os

import numpy as np
import pytest

from bundletrack_b200 import _lib, metrics, policy, synth
from oracle import nocs_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_nocs.npz")
SETS = ("main_noise", "main_plain", "far_plain", "adv")
ENDPOINT_ULP = 64          # arccos arguments this close to +-1 are marginal: NaN or not may differ
MARGIN = 1e-9              # threshold distances below this (relative) are marginal


def _script(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "scripts", f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def z():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def nm(cuda_device):
    m = metrics.NocsMetrics(20000)
    yield m
    m.close()


def _set(z, name):
    cls = z[f"{name}_cls"]
    if name != "adv":
        cls = cls[z[f"{name}_scored"] == 1]
    return z[f"{name}_pred"], z[f"{name}_gt"], z[f"{name}_corners"], cls, z[f"{name}_theta"], z[f"{name}_shift"], z[f"{name}_iou"]


def _decisions(t, s, u):
    with np.errstate(invalid="ignore"):
        return np.stack([(t < 5) & (s < 50), u > 0.25, (u > 0.25) & (t < 360)])


@pytest.mark.gpu
@pytest.mark.parametrize("name", SETS)
def test_records_equal_the_reference(z, nm, name):
    P, G, C, cls, theta, shift, iou = _set(z, name)
    t, s, u = nm(P, G, C, np.isin(cls, nocs_oracle.SYMMETRIC))
    o = nocs_oracle.record_metrics(P, G, C, np.isin(cls, nocs_oracle.SYMMETRIC))
    far = np.abs(o["margins"]["arg_ulp"]) > ENDPOINT_ULP
    fin = ~np.isnan(iou)
    assert np.array_equal(np.isnan(u), ~fin)
    assert np.abs(u[fin] - iou[fin]).max() <= 1e-14, np.abs(u[fin] - iou[fin]).max()
    assert (np.abs(s - shift) <= 1e-15 * np.abs(shift)).all() or (np.abs(s - shift) / np.maximum(shift, 1e-300)).max() <= 1e-15
    assert np.array_equal(np.isnan(t[far]), np.isnan(theta[far]))
    ok = far & ~np.isnan(theta)
    assert np.abs(t[ok] - theta[ok]).max(initial=0) <= 1e-6, np.abs(t[ok] - theta[ok]).max()
    # against the oracle, which pins the same operation order: IoU and shift bit for bit, theta to CUDA's cbrt / acos
    assert np.array_equal(u, o["iou"], equal_nan=True) and np.array_equal(s, o["shift"])
    assert np.abs(t[ok] - o["theta"][ok]).max(initial=0) <= 1e-6
    # decisions: equal on every record without a margin below MARGIN; the marginal ones are listed
    marginal = ~far | (nocs_oracle.min_margin(o["margins"]) < MARGIN)
    d_gpu, d_ref = _decisions(t, s, u), _decisions(theta, shift, iou)
    assert np.array_equal(d_gpu[:, ~marginal], d_ref[:, ~marginal])
    diff = np.nonzero((d_gpu != d_ref).any(0) | (np.isnan(t) != np.isnan(theta)))[0]
    print(f"{name}: {len(t)} records, {marginal.sum()} marginal, differing decisions or NaN at {diff.tolist()}; "
          f"max |dtheta| {np.abs(t[ok] - theta[ok]).max(initial=0):.3g} deg, max |dIoU| {np.abs(u[fin] - iou[fin]).max():.3g}")
    assert set(diff.tolist()) <= set(np.nonzero(marginal)[0].tolist())


@pytest.mark.gpu
def test_adversarial_kinds(z, nm):
    P, G, C, cls, theta, shift, iou = _set(z, "adv")
    t, s, u = nm(P, G, C, np.isin(cls, nocs_oracle.SYMMETRIC))
    kind = np.array(json.loads(str(z["adv_kind"])))
    assert (t[kind == "gt_bottom_row"] == 10000).all() and (s[kind == "gt_bottom_row"] == 10000).all()
    # an improper rotation divided by its negative cube root flips sign: R1 R2^T is -I and the arccos argument sits at -1, where
    # NaN or 180 is decided by the last bits (marginal, as in the reference)
    neg = kind == "negative_det"
    assert (np.isnan(t[neg]) | (np.abs(t[neg] - 180) < 1e-4)).all() and np.isfinite(u[neg]).all()
    flip = (kind == "flip180")
    assert (np.isnan(t[flip]) | (np.abs(t[flip] - 180) < 1e-5)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 5, 37, 1001])
def test_one_call_equals_single_record_calls(z, nm, n):
    P, G, C, cls, _, _, _ = _set(z, "main_noise")
    A, B = _set(z, "adv")[:2]
    P, G = np.concatenate([P, A])[:n], np.concatenate([G, B])[:n]
    C = np.concatenate([C, _set(z, "adv")[2]])[:n]
    sym = np.concatenate([cls, _set(z, "adv")[3]])[:n]
    sym = np.isin(sym, nocs_oracle.SYMMETRIC)
    t, s, u = nm(P, G, C, sym)
    for i in range(0, n, max(1, n // 40)):
        ti, si, ui = nm(P[i:i + 1], G[i:i + 1], C[i:i + 1], sym[i:i + 1])
        assert np.array_equal(ti, t[i:i + 1], equal_nan=True) and np.array_equal(si, s[i:i + 1]) and np.array_equal(ui, u[i:i + 1], equal_nan=True), i
    t2, s2, u2 = nm(P, G, C, sym)
    assert np.array_equal(t, t2, equal_nan=True) and np.array_equal(s, s2) and np.array_equal(u, u2, equal_nan=True)


@pytest.mark.gpu
def test_capacity_and_reserve(cuda_device):
    m = metrics.NocsMetrics(3)
    try:
        with pytest.raises(_lib.BtError, match="status -2"):
            m(np.tile(np.eye(4), (4, 1, 1)), np.tile(np.eye(4), (4, 1, 1)), np.ones((8, 3)), np.zeros(4))
        t, s, u = m(np.tile(np.eye(4), (3, 1, 1)), np.tile(np.eye(4), (3, 1, 1)), np.ones((8, 3)), np.zeros(3))
        assert t.shape == (3,)
    finally:
        m.close()


@pytest.mark.gpu
def test_context_resources_return(z, cuda_device):
    lib = _lib.load()

    def live():
        d, p, h = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_int()
        assert lib.bt_debug_live_resources(ctypes.byref(d), ctypes.byref(p), ctypes.byref(h)) == 0
        return d.value, p.value, h.value

    before = live()
    P, G, C, cls, _, _, _ = _set(z, "main_plain")
    m = metrics.NocsMetrics(100)
    m(P[:50], G[:50], C[:50], np.isin(cls[:50], nocs_oracle.SYMMETRIC))
    lib.bt_nocs_reserve(m.ctx, 5000)
    m(P, G, C, np.isin(cls, nocs_oracle.SYMMETRIC))
    assert live() != before
    m.close()
    assert live() == before


@pytest.mark.gpu
@pytest.mark.parametrize("run,noise", [("main_noise", (0.02, 0.0)), ("main_plain", None), ("far_plain", None)])
def test_eval_nocs_script_equals_the_reference(z, tmp_path, cuda_device, run, noise):
    mk, ev = _script("make_golden_nocs"), _script("eval_nocs")
    nocs_dir, results_dir = mk.write_tree(str(tmp_path), mk.tree_from_arrays(z, run.split("_")[0]))
    lines = []
    res = ev.evaluate(nocs_dir, results_dir, noise, out=lambda *a: lines.append(" ".join(map(str, a))))
    ref = z[f"{run}_printed"]
    got = [[v["5cm5deg"], v["iou25"], v["rot_err"], v["tran_err"]] for v in res["classes"].values()]
    got = np.array(got + [[res["5cm5deg"], res["iou25"], res["rot_err"], res["tran_err"]]] * 2)
    assert np.array_equal(got[:, :2], ref[:, :2]), (got, ref)
    assert np.array_equal(np.isnan(got[:, 2:]), np.isnan(ref[:, 2:]))
    fin = ~np.isnan(ref[:, 2:])
    assert (np.abs(got[:, 2:][fin] - ref[:, 2:][fin]) <= 1e-12 * np.abs(ref[:, 2:][fin])).all(), (got, ref)
    assert res["n"] == len(z[f"{run}_cls"]) and lines[-1] == "*" * 56
    print(run, "printed", got[6].tolist(), "reference", ref[6].tolist())


@pytest.mark.gpu
def test_tracked_sequence_scored_like_the_oracle(tmp_path, cuda_device):
    """A synthetic sequence tracked with the NOCS defaults, written with bt_pose_write_txt as class 'camera' of a NOCS tree, then scored by
    the script; the oracle scores the same files."""
    import torch
    from bundletrack_b200.tracker import Tracker
    mk, ev = _script("make_golden_nocs"), _script("eval_nocs")
    tree = mk.make_tree(3, n_frames=6, anomalies=False)
    H, W, FEATS, N = 240, 320, 400, 24
    seq = synth.make_sequence(31, N, H=H, W=W, n_feats=FEATS)
    trk = Tracker(None, H, W, seq.K, FEATS, 40)
    model = "camera_tracked_norm"
    nocs_dir, results_dir = mk.write_tree(str(tmp_path), tree)
    os.makedirs(f"{results_dir}/{model}_4/poses")
    ks = []
    for k in range(N):
        d, m, c = (torch.from_numpy(np.ascontiguousarray(a[k])).to(cuda_device) for a in (seq.depth_raw, seq.mask, seq.colour))
        rq = torch.zeros((400, 400, 3), dtype=torch.uint8, device=cuda_device)
        st, _ = trk.begin_frame(d, m, c, rq, loader_id=0, first_pose=seq.poses_gt[k])
        if st != _lib.BT_FRAME_OTHER:
            continue
        pose, st = trk.end_frame(seq.feats[k]["kpts"], torch.from_numpy(seq.feats[k]["desc"]).to(cuda_device))
        if st in (_lib.BT_FRAME_OTHER, _lib.BT_FRAME_NO_BA):
            policy.save_pose_txt(f"{results_dir}/{model}_4/poses/{k:04d}.txt", pose)
            ks.append(k)
    trk.close()
    assert len(ks) >= N - 2
    r = np.asarray(seq.radii) * 1000
    corners = np.array([[sx * r[0], sy * r[1], sz * r[2]] for sx in (1, -1) for sy in (1, -1) for sz in (1, -1)])
    with open(f"{nocs_dir}/NOCS-REAL275-additional/model_scales/{model}.txt", "w") as f:
        f.write("".join(f"{x:.6f} {y:.6f} {zz:.6f}\n" for x, y, zz in corners))
    os.makedirs(f"{nocs_dir}/NOCS-REAL275-additional/data_list/real_val/3/{model}")
    with open(f"{nocs_dir}/NOCS-REAL275-additional/data_list/real_val/3/{model}/list.txt", "w") as f:
        f.write("".join(f"real_val/scene_4/{k:04d}\n" for k in range(N)))
    import pickle
    os.makedirs(f"{nocs_dir}/real_test/scene_4", exist_ok=True)
    for k in range(N):
        with open(f"{nocs_dir}/real_test/scene_4/{k:04d}_meta.txt", "w") as f:
            f.write(f"1 3 {model}\n")
        G = np.linalg.inv(np.asarray(seq.poses_gt[k], np.float64))          # ob_in_cam, metres
        with open(f"{nocs_dir}/gts/real_test/results_real_test_scene_4_{k:04d}.pkl", "wb") as f:
            pickle.dump({"gt_RTs": np.asarray([G])}, f)
    for noise in (None, (0.02, 0.0)):
        res = ev.evaluate(nocs_dir, results_dir, noise, out=lambda *a: None)
        rec = res["records"]
        sc = np.array(rec["scored"]) == 1
        cls = np.array(rec["cls"])
        o = nocs_oracle.record_metrics(rec["pred"], rec["gt"], rec["corners"], np.isin(cls[sc], nocs_oracle.SYMMETRIC))
        marginal = (np.abs(o["margins"]["arg_ulp"]) <= ENDPOINT_ULP) | (nocs_oracle.min_margin(o["margins"]) < MARGIN)
        t, s, u = rec["theta"], rec["shift"], rec["iou"]
        # per record: the device against the oracle on the same files, decisions equal away from the margins
        ok = ~marginal & ~np.isnan(o["theta"])
        assert np.array_equal(np.isnan(t[sc][~marginal]), np.isnan(o["theta"][~marginal]))
        assert np.abs(t[sc][ok] - o["theta"][ok]).max(initial=0) <= 1e-6
        assert np.array_equal(s[sc], o["shift"]) and np.array_equal(u[sc], o["iou"], equal_nan=True)
        assert np.array_equal(_decisions(t[sc], s[sc], u[sc])[:, ~marginal], _decisions(o["theta"], o["shift"], o["iou"])[:, ~marginal])
        # the printed numbers: the benchmark's aggregation of these records, bit for bit
        per, ov = nocs_oracle.score(cls, rec["scored"], t, s, u)
        cam = res["classes"]["camera"]
        print(f"tracked {len(ks)} frames, noise {noise}: camera 5cm5deg {cam['5cm5deg']:.2f} IoU25 {cam['iou25']:.2f} rot {cam['rot_err']:.4f} "
              f"tran {cam['tran_err']:.4f}; {marginal.sum()} marginal records")
        assert cam["5cm5deg"] == per[2, 0] * 100 and cam["iou25"] == per[2, 1] * 100
        assert np.array_equal([cam["rot_err"], cam["tran_err"]], [per[2, 2], per[2, 3] / 10], equal_nan=True)
        assert np.array_equal([res["5cm5deg"], res["rot_err"]], [ov[0] * 100, ov[2]], equal_nan=True)
        assert res["n_scored"] >= len(ks)
