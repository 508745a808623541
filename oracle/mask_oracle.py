"""numpy restatement of the DAVIS mask scores as bundletrack_b200/csrc/metrics.cu computes them (DESIGN.md §3.16, include/bundletrack_b200.h):

- J = |P & G| / |P | G| in float64, 1 for an empty union;
- the boundary map b(S) with _seg2bmap's edge rules: (S ^ e) | (S ^ s) | (S ^ se) inside, S ^ e on the last row, S ^ s on the last column,
  0 at the corner, e / s / se the east, south and south-east neighbours (0 outside the image);
- r = ceil(bound_th sqrt(H^2 + W^2)) and the disk dx^2 + dy^2 <= r^2, applied here as explicit row intervals (row y + dy within x +- isqrt(r^2
  - dy^2)), not with OpenCV, so that the tests can hold it against cv2.dilate and scipy as an independent implementation;
- m_P, m_G, n_P, n_G, precision, recall and F with the toolkit's rules for empty boundaries;
- db_statistics: mean, recall mean(X > 0.5) and decay over four bins of round(linspace(1, n, 5) + 1e-10) - 1.

Test infrastructure only: bundletrack_b200/ never imports it."""
from __future__ import annotations

import math

import numpy as np

COUNT_KEYS = ("inter", "union", "n_pred", "n_gt", "m_pred", "m_gt")
SCORE_KEYS = ("J&F-Mean", "J-Mean", "J-Recall", "J-Decay", "F-Mean", "F-Recall", "F-Decay")


def radius(h: int, w: int, bound_th: float = 0.008) -> int:
    """ceil(bound_th * |(h, w)|), the toolkit's tolerance in pixels."""
    return int(np.ceil(bound_th * np.sqrt(float(h) * h + float(w) * w)))


def boundary(seg) -> np.ndarray:
    """_seg2bmap: bool [H, W] boundary map of a mask (foreground = value != 0)."""
    S = np.asarray(seg) != 0
    e, s, se = np.zeros_like(S), np.zeros_like(S), np.zeros_like(S)
    e[:, :-1] = S[:, 1:]
    s[:-1, :] = S[1:, :]
    se[:-1, :-1] = S[1:, 1:]
    b = (S ^ e) | (S ^ s) | (S ^ se)
    b[-1, :] = S[-1, :] ^ e[-1, :]
    b[:, -1] = S[:, -1] ^ s[:, -1]
    b[-1, -1] = False
    return b


def dilate(b, r: int) -> np.ndarray:
    """b dilated by the disk dx^2 + dy^2 <= r^2, nothing dilating in from outside the image: out(y, x) is set when some b(y + dy, x') is,
    with |x' - x| <= isqrt(r^2 - dy^2).  Each row's intervals come from a prefix count."""
    b = np.asarray(b, bool)
    H, W = b.shape
    cs = np.zeros((H, W + 1), np.int64)
    np.cumsum(b, axis=1, out=cs[:, 1:])
    x = np.arange(W)
    out = np.zeros_like(b)
    for dy in range(-min(r, H - 1), min(r, H - 1) + 1):
        hw = math.isqrt(r * r - dy * dy)
        lo, hi = np.maximum(x - hw, 0), np.minimum(x + hw + 1, W)
        row_any = (cs[:, hi] - cs[:, lo]) > 0                   # row y' has a set pixel within hw columns of x
        if dy >= 0:
            out[:H - dy] |= row_any[dy:]
        else:
            out[-dy:] |= row_any[:H + dy]
    return out


def frame_counts(pred, gt, bound_th: float = 0.008) -> np.ndarray:
    """int64 [6]: |P & G|, |P | G|, n_P, n_G, m_P, m_G of one frame pair."""
    P, G = np.asarray(pred) != 0, np.asarray(gt) != 0
    if P.shape != G.shape or P.ndim != 2:
        raise ValueError(f"pred {P.shape} and gt {G.shape} must be one H x W shape")
    r = radius(*P.shape, bound_th)
    bp, bg = boundary(P), boundary(G)
    return np.array([(P & G).sum(), (P | G).sum(), bp.sum(), bg.sum(), (bp & dilate(bg, r)).sum(), (bg & dilate(bp, r)).sum()], np.int64)


def j_and_f(c) -> tuple:
    """(J, F) in float64 from one frame's six counts."""
    inter, union, n_p, n_g, m_p, m_g = (int(v) for v in c)
    j = 1.0 if union == 0 else inter / union
    if n_p == 0 and n_g > 0:
        precision, recall = 1.0, 0.0
    elif n_p > 0 and n_g == 0:
        precision, recall = 0.0, 1.0
    elif n_p == 0 and n_g == 0:
        precision, recall = 1.0, 1.0
    else:
        precision, recall = m_p / float(n_p), m_g / float(n_g)
    f = 0.0 if precision + recall == 0 else 2 * precision * recall / (precision + recall)
    return j, f


def metrics(pred, gt, bound_th: float = 0.008):
    """(j, f, counts) of [F, H, W] sequences: float64 [F], float64 [F], int64 [F, 6]."""
    pred, gt = np.asarray(pred), np.asarray(gt)
    counts = np.stack([frame_counts(p, g, bound_th) for p, g in zip(pred, gt)])
    jf = np.array([j_and_f(c) for c in counts], np.float64).reshape(-1, 2)
    return jf[:, 0], jf[:, 1], counts


def db_statistics(x) -> tuple:
    """(mean, recall, decay) of one sequence's per-frame values."""
    x = np.asarray(x, np.float64)
    m = np.mean(x)
    o = np.mean(x > 0.5)
    ids = (np.round(np.linspace(1, len(x), 5) + 1e-10) - 1).astype(np.int64)
    bins = [x[ids[i]:ids[i + 1] + 1] for i in range(4)]
    return m, o, np.mean(bins[0]) - np.mean(bins[3])


def score(j, f) -> dict:
    """The seven statistics of a sequence, in the toolkit's CSV order."""
    jm, jr, jd = db_statistics(j)
    fm, fr, fd = db_statistics(f)
    return dict(zip(SCORE_KEYS, [(jm + fm) / 2.0, jm, jr, jd, fm, fr, fd]))
