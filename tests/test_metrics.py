"""Pose metrics without a GPU: the exports, bt_pose_metrics' argument checks, bt_vocap against a numpy restatement of the reference's VOCap
(scripts/eval_ycbineoat.py), BT_ERR_NO_DEVICE and the ob_in_cam helper."""
import ctypes

import numpy as np
import pytest

from bundletrack_b200 import _lib, metrics

NEW = ("bt_metrics_reserve", "bt_pose_metrics", "bt_vocap")


def vocap_ref(rec, max_err=0.1):
    """VOCap as eval_ycbineoat.py states it, with its 0.1 m as max_err."""
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
    return np.sum((mrec[i] - mrec[i - 1]) * mpre[i]) * (1.0 / max_err)


def test_metrics_symbols_are_exported():
    lib = _lib.load()
    for name in NEW:
        assert name in _lib.EXPORTS and hasattr(lib, name), name


@pytest.mark.parametrize("case", ["random", "empty", "all_above", "all_zero", "duplicates", "one", "nan", "wide"])
def test_vocap_equals_the_reference(case):
    rng = np.random.default_rng(11)
    err, max_err = {
        "random": (rng.exponential(0.03, 500), 0.1),
        "empty": (np.zeros(0), 0.1),
        "all_above": (0.1 + rng.uniform(0, 1, 40), 0.1),
        "all_zero": (np.zeros(25), 0.1),
        "duplicates": (np.repeat(rng.uniform(0, 0.12, 30), 3), 0.1),
        "one": (np.array([0.02]), 0.1),
        "nan": (np.array([0.01, np.nan, 0.05, 0.3]), 0.1),
        "wide": (rng.uniform(0, 0.5, 300), 0.25),
    }[case]
    got = metrics.vocap(err, max_err)
    assert abs(got - vocap_ref(err, max_err)) <= 1e-12, (got, vocap_ref(err, max_err))
    assert 0.0 <= got <= 1.0


def test_vocap_argument_checks():
    lib = _lib.load()
    out = ctypes.c_double(-1)
    e = np.array([0.01, 0.02])
    p = e.ctypes.data_as(ctypes.c_void_p)
    assert lib.bt_vocap(p, 2, ctypes.c_double(0.1), None) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_vocap(None, 2, ctypes.c_double(0.1), ctypes.byref(out)) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_vocap(p, -1, ctypes.c_double(0.1), ctypes.byref(out)) == _lib.BT_ERR_INVALID_ARG
    for bad in (0.0, -0.1, float("inf"), float("nan")):
        assert lib.bt_vocap(p, 2, ctypes.c_double(bad), ctypes.byref(out)) == _lib.BT_ERR_INVALID_ARG, bad
    assert lib.bt_vocap(None, 0, ctypes.c_double(0.1), ctypes.byref(out)) == _lib.BT_OK and out.value == 0.0


def test_pose_metrics_argument_checks():
    """The arguments are checked before the context is looked at, so every refusal shows here without a GPU."""
    lib = _lib.load()
    F = 3
    P = np.tile(np.eye(4), (F, 1, 1))
    G = P.copy()
    pts = ctypes.c_void_p(0x1000)          # never dereferenced on the host: the call is refused first
    out = ctypes.c_void_p(0x2000)
    ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p)

    def call(ctx=None, model=pts, n=10, pred=P, gt=G, f=F, add=out, adds=out):
        return lib.bt_pose_metrics(ctx, model, ctypes.c_int(n), None if pred is None else ptr(pred), None if gt is None else ptr(gt), ctypes.c_int(f), add, adds, None)

    for kw, msg in ((dict(n=0), b"n_pts"), (dict(f=0), b"n_frames"), (dict(model=None), b"NULL"), (dict(pred=None), b"NULL"), (dict(gt=None), b"NULL"),
                    (dict(add=None), b"NULL"), (dict(adds=None), b"NULL"), (dict(), b"ctx is NULL")):
        assert call(**kw) == _lib.BT_ERR_INVALID_ARG, kw
        assert msg in lib.bt_last_error(), (kw, lib.bt_last_error())
    for bad in (np.nan, np.inf, -np.inf):
        for which in ("pred", "gt"):
            A = P.copy()
            A[2, 1, 3] = bad
            assert call(**{which: A}) == _lib.BT_ERR_INVALID_ARG
            assert b"frame 2 has a non-finite" in lib.bt_last_error()
    assert lib.bt_metrics_reserve(None, 10, 10) == _lib.BT_ERR_INVALID_ARG


def test_pose_metrics_without_gpu_is_no_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_lib.BtError, match="status -4"):
        metrics.pose_metrics(np.zeros((5, 3)), np.eye(4)[None], np.eye(4)[None])
    with pytest.raises(_lib.BtError, match="status -4"):
        metrics.PoseMetrics(100, 10)


def test_ob_in_cam_inverts_the_tracker_pose():
    rng = np.random.default_rng(2)
    from bundletrack_b200 import synth
    R, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    cam_in_model = synth.se3(R * np.sign(np.linalg.det(R)), rng.normal(size=3)).astype(np.float32)
    O = metrics.ob_in_cam(np.stack([cam_in_model, cam_in_model]))
    assert O.dtype == np.float64 and O.shape == (2, 4, 4)
    assert np.allclose(O[0] @ cam_in_model.astype(np.float64), np.eye(4), atol=1e-12)
