#!/usr/bin/env python3
"""DAVIS scores of predicted object masks (e.g. run_vos.py's masks_vos/) against ground-truth masks, per sequence:

    J   region similarity, |P & G| / |P | G| per frame
    F   boundary accuracy, the F-score of the two masks' boundary pixels matched within ceil(0.008 * image diagonal) pixels
    J&F-Mean, J-Mean, J-Recall, J-Decay, F-Mean, F-Recall, F-Decay   the DAVIS toolkit's per-sequence statistics, in its CSV order

Scored on the device (bundletrack_b200.metrics.MaskScore, DESIGN.md §3.16).  The frames are the ids of the ground-truth directory's PNGs
(the file name up to its first dot), sorted; each needs <pred_dir>/<id>.png, and a missing one is an error that names it.  As the DAVIS
semi-supervised protocol does, the first and last frames are left out (the first is the mask the segmentation starts from); --keep_ends
keeps them.  Masks are read as the tracker reads them (sequence.read_image, "mask"): 8-bit grey PNGs only, anything else is refused by
name.  This script only reads files.

    python scripts/eval_masks.py --gt video/gt_mask --pred video/masks_vos
    python scripts/eval_masks.py --ycbineoat YCBInEOAT --pred_name masks_vos
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CHUNK = 256          # frames read and scored per device call


def pair_files(gt_dir: str, pred_dir: str) -> list:
    """[(id, gt path, pred path)] for every PNG of gt_dir, sorted by id.  Raises FileNotFoundError naming the first missing prediction."""
    ids = sorted(name.split(".")[0] for name in os.listdir(gt_dir) if name.lower().endswith(".png"))
    if not ids:
        raise FileNotFoundError(f"{gt_dir}: no PNG ground-truth masks")
    out = []
    for i in ids:
        pred = os.path.join(pred_dir, f"{i}.png")
        if not os.path.isfile(pred):
            raise FileNotFoundError(f"{pred}: no prediction for ground-truth frame {i}")
        out.append((i, os.path.join(gt_dir, f"{i}.png"), pred))
    return out


def protocol_frames(pairs: list, keep_ends: bool = False) -> list:
    """The frames scored: all of them with keep_ends, otherwise all but the first and the last."""
    kept = pairs if keep_ends else pairs[1:-1]
    if not kept:
        raise ValueError(f"{len(pairs)} frames leave none to score once the first and last are left out (--keep_ends keeps them)")
    return kept


def _read(paths: list) -> np.ndarray:
    from bundletrack_b200.sequence import read_image
    masks = [read_image(p, "mask") for p in paths]
    for p, m in zip(paths, masks):
        if m.shape != masks[0].shape:
            raise ValueError(f"{p}: {m.shape[0]} x {m.shape[1]}, the sequence's masks are {masks[0].shape[0]} x {masks[0].shape[1]}")
    return np.stack(masks)


def score_sequence(gt_dir: str, pred_dir: str, keep_ends: bool = False, bound_th: float = 0.008, device: int = 0) -> dict:
    """metrics.mask_score of one sequence plus "frames" (the ids scored), "j" and "f" (per frame)."""
    from bundletrack_b200.metrics import MaskScore, mask_score
    pairs = protocol_frames(pair_files(gt_dir, pred_dir), keep_ends)
    j, f, ms = [], [], None
    try:
        for s in range(0, len(pairs), CHUNK):
            part = pairs[s:s + CHUNK]
            gt, pred = _read([g for _, g, _ in part]), _read([p for _, _, p in part])
            if gt.shape[1:] != pred.shape[1:]:
                raise ValueError(f"{pred_dir}: predictions of {pred.shape[1]} x {pred.shape[2]}, ground truth of {gt.shape[1]} x {gt.shape[2]}")
            if ms is None:
                ms = MaskScore(CHUNK, gt.shape[1], gt.shape[2], device=device)
            jj, ff = ms(pred, gt, bound_th)
            j.append(jj)
            f.append(ff)
    finally:
        if ms is not None:
            ms.close()
    j, f = np.concatenate(j), np.concatenate(f)
    res = mask_score(j, f)
    res.update(frames=[i for i, _, _ in pairs], j=j.tolist(), f=f.tolist())
    return res


def evaluate(sequences: list, keep_ends: bool = False, bound_th: float = 0.008, device: int = 0, out=print) -> dict:
    """sequences: [(name, gt dir, pred dir)].  Prints one line per sequence and the mean over sequences of each statistic; returns
    {"sequences": {name: score_sequence's dict}, "mean": {statistic: mean over sequences}}."""
    from bundletrack_b200.metrics import MASK_SCORE_KEYS
    per = {}
    for name, gt_dir, pred_dir in sequences:
        r = score_sequence(gt_dir, pred_dir, keep_ends, bound_th, device)
        per[name] = r
        out(f"{name}: {len(r['frames'])} frames, " + ", ".join(f"{k} {r[k]:.4f}" for k in MASK_SCORE_KEYS))
    mean = {k: float(np.mean([r[k] for r in per.values()])) for k in MASK_SCORE_KEYS}
    out(f"mean over {len(per)} sequences: " + ", ".join(f"{k} {mean[k]:.4f}" for k in MASK_SCORE_KEYS))
    return {"sequences": per, "mean": mean}


def ycbineoat_sequences(root: str, pred_name: str) -> list:
    """[(video, ROOT/<video>/gt_mask, ROOT/<video>/<pred_name>)] of every video directory that has a gt_mask/, sorted."""
    seqs = [(v, os.path.join(root, v, "gt_mask"), os.path.join(root, v, pred_name)) for v in sorted(os.listdir(root))
            if os.path.isdir(os.path.join(root, v, "gt_mask"))]
    if not seqs:
        raise FileNotFoundError(f"{root}: no <video>/gt_mask directory")
    return seqs


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--gt", help="one sequence: the ground-truth mask directory")
    ap.add_argument("--pred", help="one sequence: the predicted mask directory")
    ap.add_argument("--ycbineoat", help="a YCBInEOAT root: every <video>/gt_mask against <video>/<pred_name>")
    ap.add_argument("--pred_name", default="masks_vos", help="the prediction directory's name inside each video (with --ycbineoat)")
    ap.add_argument("--keep_ends", action="store_true", help="score the first and last frames too")
    ap.add_argument("--bound_th", type=float, default=0.008, help="boundary tolerance, a fraction of the image diagonal")
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    if a.ycbineoat and (a.gt or a.pred):
        ap.error("give either --ycbineoat or --gt and --pred")
    if a.ycbineoat:
        seqs = ycbineoat_sequences(a.ycbineoat, a.pred_name)
    elif a.gt and a.pred:
        seqs = [(os.path.basename(os.path.normpath(a.pred)), a.gt, a.pred)]
    else:
        ap.error("give --gt and --pred, or --ycbineoat")
    return evaluate(seqs, a.keep_ends, a.bound_th, a.device)


if __name__ == "__main__":
    main()
