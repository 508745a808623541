"""NOCS-REAL275 scoring without a GPU: the exports and argument checks of bt_nocs_reserve / bt_nocs_metrics / bt_nocs_score,
BT_ERR_NO_DEVICE, bt_nocs_score against every number the reference's 6-PACK benchmark printed (tests/golden/ref_nocs.npz, bit for bit),
the numpy oracle against the benchmark's per-record values, and scripts/eval_nocs.py's conversion, noise and pairing against the records
the benchmark visited."""
import ctypes
import importlib.util
import json
import os
import sys

import numpy as np
import pytest

from bundletrack_b200 import _lib, metrics
from oracle import nocs_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_nocs.npz")
RUNS = ("main_noise", "main_plain", "far_plain")
NEW = ("bt_nocs_reserve", "bt_nocs_metrics", "bt_nocs_score")


def _script(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "scripts", f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def z():
    return np.load(GOLDEN)


def _full(z, run):
    """Per-record theta / shift / IoU over all records (NaN where not scored)."""
    sc = z[f"{run}_scored"] == 1
    out = []
    for k in ("theta", "shift", "iou"):
        a = np.full(len(sc), np.nan)
        a[sc] = z[f"{run}_{k}"]
        out.append(a)
    return out


def _printed(per, ov):
    rows = [[p[0] * 100, p[1] * 100, p[2], p[3] / 10] for p in list(per) + [ov, ov]]
    return np.array([[float(v) for v in r] for r in rows])


def test_nocs_symbols_are_exported():
    lib = _lib.load()
    for name in NEW:
        assert name in _lib.EXPORTS and hasattr(lib, name), name


def test_nocs_metrics_argument_checks():
    """The arguments are checked before the context is looked at, so every refusal shows here without a GPU."""
    lib = _lib.load()
    n = 3
    P = np.tile(np.eye(4), (n, 1, 1))
    G = P.copy()
    C = np.ones((n, 8, 3))
    S = np.zeros(n, np.int32)
    out = ctypes.c_void_p(0x2000)          # never dereferenced on the host: the call is refused first
    ptr = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)

    def call(ctx=None, pred=P, gt=G, corners=C, sym=S, k=n, t=out, s=out, u=out):
        return lib.bt_nocs_metrics(ctx, ptr(pred), ptr(gt), ptr(corners), ptr(sym), ctypes.c_int(k), t, s, u, None)

    for kw, msg in ((dict(k=0), b"n 0"), (dict(k=-1), b"n -1"), (dict(pred=None), b"NULL"), (dict(gt=None), b"NULL"), (dict(corners=None), b"NULL"),
                    (dict(sym=None), b"NULL"), (dict(t=None), b"NULL"), (dict(s=None), b"NULL"), (dict(u=None), b"NULL"), (dict(), b"ctx is NULL")):
        assert call(**kw) == _lib.BT_ERR_INVALID_ARG, kw
        assert msg in lib.bt_last_error(), (kw, lib.bt_last_error())
    for bad in (np.nan, np.inf, -np.inf):
        for which in ("pred", "gt"):
            A = P.copy()
            A[2, 3, 1] = bad
            assert call(**{which: A}) == _lib.BT_ERR_INVALID_ARG
            assert b"record 2 has a non-finite pose" in lib.bt_last_error()
        B = C.copy()
        B[1, 7, 2] = bad
        assert call(corners=B) == _lib.BT_ERR_INVALID_ARG
        assert b"record 1 has a non-finite corner" in lib.bt_last_error()
    assert lib.bt_nocs_reserve(None, 10) == _lib.BT_ERR_INVALID_ARG


def test_nocs_score_argument_checks():
    lib = _lib.load()
    cls = np.arange(1, 7, dtype=np.int32)
    sc = np.ones(6, np.int32)
    v = np.ones(6)
    per, ov = np.zeros(24), np.zeros(4)
    ptr = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)

    def call(c=cls, s=sc, t=v, d=v, u=v, n=6, p=per, o=ov):
        return lib.bt_nocs_score(ptr(c), ptr(s), ptr(t), ptr(d), ptr(u), ctypes.c_int(n), ptr(p), ptr(o))

    assert call() == _lib.BT_OK
    for kw in (dict(c=None), dict(s=None), dict(t=None), dict(d=None), dict(u=None), dict(p=None), dict(o=None), dict(n=0)):
        assert call(**kw) == _lib.BT_ERR_INVALID_ARG, kw
    for bad in (0, 7, -1):
        c = cls.copy()
        c[3] = bad
        assert call(c=c) == _lib.BT_ERR_INVALID_ARG
        assert b"outside 1..6" in lib.bt_last_error()
    c = cls.copy()
    c[4] = 1                                # class 5 has no record: the benchmark divides by zero there
    assert call(c=c) == _lib.BT_ERR_INVALID_ARG
    assert b"class 5 has no record" in lib.bt_last_error()


def test_nocs_metrics_without_gpu_is_no_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_lib.BtError, match="status -4"):
        metrics.NocsMetrics(10)
    with pytest.raises(_lib.BtError, match="status -4"):
        metrics.nocs_metrics(np.eye(4)[None], np.eye(4)[None], np.ones((8, 3)), [0])


@pytest.mark.parametrize("run", RUNS)
def test_nocs_score_equals_the_reference_printout_bit_for_bit(z, run):
    t, s, u = _full(z, run)
    per, ov = metrics.nocs_score(z[f"{run}_cls"], z[f"{run}_scored"], t, s, u)
    got = _printed(per, ov)
    ref = z[f"{run}_printed"]
    assert np.array_equal(got, ref, equal_nan=True), (got, ref)
    # the numpy restatement of main's aggregation agrees too
    per2, ov2 = nocs_oracle.score(z[f"{run}_cls"], z[f"{run}_scored"], t, s, u)
    assert np.array_equal(_printed(per2, ov2), ref, equal_nan=True)
    if run == "far_plain":
        assert np.isnan(ref[4, 2:]).all() and np.isnan(ref[6, 2:]).all()     # laptop: no record above IoU 0.25, and the NaN reaches overall


def _check_oracle(pred, gt, corners, cls, theta, shift, iou):
    r = nocs_oracle.record_metrics(pred, gt, corners, np.isin(cls, nocs_oracle.SYMMETRIC))
    far = np.abs(r["margins"]["arg_ulp"]) > 64
    # NaN where the benchmark has NaN, away from the endpoints
    assert np.array_equal(np.isnan(r["theta"][far]), np.isnan(theta[far]))
    rel = lambda a, b: np.abs(a - b) / np.maximum(np.abs(b), 1e-300)
    ok = far & ~np.isnan(theta)
    # theta = arccos(arg) amplifies the argument's rounding by 1 / sin(theta): the difference, taken back to the argument, is a few ulp
    # (the benchmark's dot / trace go through BLAS); this bound is 16 ulp, and 1e-12 relative where arccos does not amplify
    arg_err = np.abs(np.deg2rad(r["theta"][ok] - theta[ok])) * np.sin(np.deg2rad(theta[ok])) / 2.0 ** -53
    assert np.all((arg_err <= 16) | (rel(r["theta"][ok], theta[ok]) <= 1e-12)), arg_err.max()
    assert np.all((rel(r["shift"], shift) <= 1e-12) | (np.abs(r["shift"] - shift) <= 1e-12))
    assert np.array_equal(np.isnan(r["iou"]), np.isnan(iou))
    fin = ~np.isnan(iou)
    assert np.all(np.abs(r["iou"][fin] - iou[fin]) <= 1e-12), np.abs(r["iou"][fin] - iou[fin]).max()
    return r


@pytest.mark.parametrize("run", RUNS)
def test_oracle_equals_the_reference_records(z, run):
    sc = z[f"{run}_scored"] == 1
    _check_oracle(z[f"{run}_pred"], z[f"{run}_gt"], z[f"{run}_corners"], z[f"{run}_cls"][sc], z[f"{run}_theta"], z[f"{run}_shift"], z[f"{run}_iou"])


def test_oracle_equals_the_reference_adversarial_records(z):
    r = _check_oracle(z["adv_pred"], z["adv_gt"], z["adv_corners"], z["adv_cls"], z["adv_theta"], z["adv_shift"], z["adv_iou"])
    kind = np.array(json.loads(str(z["adv_kind"])))
    assert np.all(z["adv_theta"][kind == "gt_bottom_row"] == 10000) and np.all(r["theta"][kind == "gt_bottom_row"] == 10000)
    # the reference's NaN branch is real: identical poses give NaN theta for some records, and the oracle sees them at the endpoint
    eq = kind == "equal"
    assert np.isnan(z["adv_theta"][eq]).any()
    assert np.all(np.abs(r["margins"]["arg_ulp"][eq]) <= 64)


def test_eval_nocs_conversion_and_pairing_equal_the_reference(z, tmp_path):
    mk, ev = _script("make_golden_nocs"), _script("eval_nocs")
    for tname, runs in (("main", (("main_noise", (0.02, 0.0)), ("main_plain", None))), ("far", (("far_plain", None),))):
        nocs_dir, results_dir = mk.write_tree(str(tmp_path / tname), mk.tree_from_arrays(z, tname))
        for run, noise in runs:
            rec = ev.collect(nocs_dir, results_dir, noise, out=lambda *a: None)
            for k in ("cls", "scored", "frame"):
                assert np.array_equal(np.array(rec[k]), z[f"{run}_{k}"]), (run, k)
            for k in ("model", "scene"):
                assert rec[k] == json.loads(str(z[f"{run}_{k}"])), (run, k)
            for k in ("pred", "gt", "corners"):
                assert np.array_equal(rec[k], z[f"{run}_{k}"]), (run, k, np.abs(rec[k] - z[f"{run}_{k}"]).max())
