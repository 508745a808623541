"""numpy restatement of the per-object mask scores with void pixels as bundletrack_b200/csrc/metrics.cu's bt_mask_metrics_objects computes
them (DESIGN.md §3.17, include/bundletrack_b200.h): for object k of a frame pair of label maps, V = (gt == void_value) (empty for -1),
P = (pred == k) & ~V and G = (gt == k) & ~V, then mask_oracle's counts, J and F of P and G.

Test infrastructure only: bundletrack_b200/ never imports it."""
from __future__ import annotations

import numpy as np

from . import mask_oracle


def object_masks(pred, gt, k: int, void_value: int = 255) -> tuple:
    """(P, G), bool [H, W]: object k of one frame pair with the void pixels removed from both."""
    pred, gt = np.asarray(pred), np.asarray(gt)
    keep = np.ones(gt.shape, bool) if void_value < 0 else gt != void_value
    return (pred == k) & keep, (gt == k) & keep


def object_counts(pred, gt, n_objects: int, void_value: int = 255, bound_th: float = 0.008) -> np.ndarray:
    """int64 [n_objects, 6]: |P & G|, |P | G|, n_P, n_G, m_P, m_G of objects 1..n_objects of one frame pair."""
    return np.stack([mask_oracle.frame_counts(*object_masks(pred, gt, k, void_value), bound_th) for k in range(1, n_objects + 1)])


def object_metrics(pred, gt, n_objects: int, void_value: int = 255, bound_th: float = 0.008):
    """(j, f, counts) of [F, H, W] label-map sequences: float64 [F, n_objects], float64 [F, n_objects], int64 [F, n_objects, 6]."""
    counts = np.stack([object_counts(p, g, n_objects, void_value, bound_th) for p, g in zip(np.asarray(pred), np.asarray(gt))])
    jf = np.array([[mask_oracle.j_and_f(c) for c in row] for row in counts], np.float64).reshape(counts.shape[0], n_objects, 2)
    return jf[..., 0], jf[..., 1], counts
