"""NOCS-REAL275 scoring restated in numpy: the reference's 6-PACK benchmark (scripts/benchmark.py) compute_RT_degree_cm_symmetry,
compute_3d_iou_new and main's aggregation.  Test infrastructure only.

Per record the arithmetic follows the benchmark statement by statement in float64, vectorised over records, in the operation order the
device kernel pins (DESIGN.md §3.8): sums of products left to right, det by the first row's cofactors, corner products in corner order.
Elementwise numpy does not fuse multiply-adds, so this equals k_nocs_metrics up to cbrt and arccos (1-2 ulp each on the device).

Each record also reports its margins: how far the arccos argument is from +-1 (units of 2^-53, the float64 spacing just below 1; negative
beyond), and the relative distances of theta, shift and IoU from the thresholds the benchmark compares them with."""
from __future__ import annotations

import math

import numpy as np

SYMMETRIC = (1, 2, 4)          # bottle, bowl, can: benchmark.py's y-axis rule (mugs never, handle_visibility is always 1)
ROT_CS = np.array([[math.cos(2 * math.pi * i / float(20)), math.sin(2 * math.pi * i / float(20))] for i in range(20)])


def _normalize(M):
    M = M.copy()
    for c in range(3):
        n = np.sqrt(((M[:, 0, c] * M[:, 0, c] + M[:, 1, c] * M[:, 1, c]) + M[:, 2, c] * M[:, 2, c]) + M[:, 3, c] * M[:, 3, c])
        M[:, :, c] = M[:, :, c] / n[:, None]
    return M


def _det3(M):
    a = M[:, 0, 0] * (M[:, 1, 1] * M[:, 2, 2] - M[:, 1, 2] * M[:, 2, 1])
    b = M[:, 0, 1] * (M[:, 1, 0] * M[:, 2, 2] - M[:, 1, 2] * M[:, 2, 0])
    c = M[:, 0, 2] * (M[:, 1, 0] * M[:, 2, 1] - M[:, 1, 1] * M[:, 2, 0])
    return (a - b) + c


def _dot3(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _extent(M, C):
    """transform_coordinates_3d of every corner, then per corner the max / min over x, y, z (NaN propagates as in np.amax)."""
    x, y, z = C[:, :, 0], C[:, :, 1], C[:, :, 2]
    w = [((M[:, r, 0, None] * x + M[:, r, 1, None] * y) + M[:, r, 2, None] * z) + M[:, r, 3, None] for r in range(4)]
    u = np.stack([w[0] / w[3], w[1] / w[3], w[2] / w[3]])
    return np.maximum(np.maximum(u[0], u[1]), u[2]), np.minimum(np.minimum(u[0], u[1]), u[2])


def _iou(G, P, C):
    hi1, lo1 = _extent(G, C)
    hi2, lo2 = _extent(P, C)
    d = np.minimum(hi1, hi2) - np.maximum(lo1, lo2)
    inter, v1, v2, dmin = d[:, 0], hi1[:, 0] - lo1[:, 0], hi2[:, 0] - lo2[:, 0], d[:, 0]
    for c in range(1, 8):
        inter = inter * d[:, c]
        v1 = v1 * (hi1[:, c] - lo1[:, c])
        v2 = v2 * (hi2[:, c] - lo2[:, c])
        dmin = np.minimum(dmin, d[:, c])
    inter = np.where(dmin < 0, 0.0, inter)
    return inter / ((v1 + v2) - inter)


def record_metrics(pred, gt, corners, symmetric):
    """pred, gt [N,4,4] (mm), corners [N,8,3], symmetric [N] -> dict of theta (deg), shift, iou, arg (the arccos argument) and margins."""
    P0 = np.asarray(pred, np.float64).reshape(-1, 4, 4)
    G0 = np.asarray(gt, np.float64).reshape(-1, 4, 4)
    N = len(P0)
    C = np.broadcast_to(np.asarray(corners, np.float64), (N, 8, 3)) if np.shape(corners) == (8, 3) else np.asarray(corners, np.float64).reshape(N, 8, 3)
    sym = np.asarray(symmetric).reshape(-1) != 0
    P, G = _normalize(P0), _normalize(G0)
    with np.errstate(all="ignore"):
        unit = np.array([0.0, 0.0, 0.0, 1.0])
        bottom = np.all(P[:, 3, :] == unit, axis=1) & np.all(G[:, 3, :] == unit, axis=1)
        R1 = P[:, :3, :3] / np.cbrt(_det3(P))[:, None, None]
        R2 = G[:, :3, :3] / np.cbrt(_det3(G))[:, None, None]
        y1, y2 = R1[:, :, 1], R2[:, :, 1]
        arg_sym = _dot3(y1, y2) / (np.sqrt(_dot3(y1, y1)) * np.sqrt(_dot3(y2, y2)))
        tr = (_dot3(R1[:, 0], R2[:, 0]) + _dot3(R1[:, 1], R2[:, 1])) + _dot3(R1[:, 2], R2[:, 2])
        arg = np.where(sym, arg_sym, (tr - 1.0) / 2.0)
        theta = np.arccos(arg) * (180 / np.pi)
        dT = P[:, :3, 3] - G[:, :3, 3]
        shift = np.sqrt(_dot3(dT, dT))
        theta = np.where(bottom, theta, 10000.0)
        shift = np.where(bottom, shift, 10000.0)
        arg = np.where(bottom, arg, np.nan)
        iou = _iou(G, P, C)
        best = np.zeros(N)
        for c, s in ROT_CS:
            Gr = G.copy()
            Gr[:, :, 0] = G[:, :, 0] * c + G[:, :, 2] * (-s)
            Gr[:, :, 2] = G[:, :, 0] * s + G[:, :, 2] * c
            v = _iou(Gr, P, C)
            best = np.where(v > best, v, best)          # max(max_iou, v) from 0: NaN never enters
        iou = np.where(sym, best, iou)
        m = {
            "arg_ulp": np.where(bottom, (1.0 - np.abs(arg)) / 2.0 ** -53, np.inf),
            "theta5": np.abs(theta - 5.0) / 5.0,
            "theta360": np.abs(theta - 360.0) / 360.0,
            "shift50": np.abs(shift - 50.0) / 50.0,
            "iou25": np.abs(iou - 0.25) / 0.25,
        }
    return {"theta": theta, "shift": shift, "iou": iou, "arg": arg, "margins": m}


def min_margin(m: dict) -> np.ndarray:
    """The smallest relative threshold margin of each record (the arccos margin is separate: it is in ulp)."""
    return np.nanmin(np.stack([m["theta5"], m["theta360"], m["shift50"], m["iou25"]]), axis=0)


def score(cls, scored, theta, shift, iou):
    """benchmark.py main's aggregation, statement by statement: per class [5 deg 5 cm, IoU25, mean theta, mean shift] and overall x += v / 6."""
    per = np.zeros((6, 4))
    overall = [0, 0, 0, 0]
    cls = np.asarray(cls).reshape(-1)
    for c in range(1, 7):
        idx = np.nonzero(cls == c)[0]
        cls_num, in55, iou25, rot, trans = len(idx), 0, 0, [], []
        for i in idx:
            if not scored[i]:
                continue
            if iou[i] > 0.25 and theta[i] < 360:
                rot.append(theta[i])
            if iou[i] > 0.25:
                trans.append(shift[i])
                iou25 += 1
            if theta[i] < 5 and shift[i] < 50:
                in55 += 1
        with np.errstate(all="ignore"):
            import warnings
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                v = [in55 / cls_num, iou25 / cls_num, np.mean(rot), np.mean(trans)]
        per[c - 1] = v
        overall = [overall[k] + v[k] / 6 for k in range(4)]
    return per, np.array(overall, np.float64)
