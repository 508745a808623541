#!/usr/bin/env python3
"""DAVIS scores of predicted object masks (e.g. run_vos.py's masks_vos/) against ground-truth masks, per sequence:

    J   region similarity, |P & G| / |P | G| per frame
    F   boundary accuracy, the F-score of the two masks' boundary pixels matched within ceil(0.008 * image diagonal) pixels
    J&F-Mean, J-Mean, J-Recall, J-Decay, F-Mean, F-Recall, F-Decay   the DAVIS toolkit's per-sequence statistics, in its CSV order

Scored on the device (bundletrack_b200.metrics.MaskScore, DESIGN.md §3.16).  The frames are the ids of the ground-truth directory's PNGs
(the file name up to its first dot), sorted; each needs <pred_dir>/<id>.png, and a missing one is an error that names it.  As the DAVIS
semi-supervised protocol does, the first and last frames are left out (the first is the mask the segmentation starts from); --keep_ends
keeps them.  Masks are read as the tracker reads them (sequence.read_image, "mask"): 8-bit grey PNGs only, anything else is refused by
name.

--davis scores multi-object label maps (e.g. run_vos.py --davis's results) by the DAVIS 2017 semi-supervised protocol, per object
(bundletrack_b200.metrics.MaskScore.objects, DESIGN.md §3.17): the sequences of ImageSets/2017/<set>.txt, the ground truth
Annotations/<resolution>/<seq>/*.png and the predictions <results>/<seq>/<id>.png, both read as palette indices.  Ground-truth 255 is void:
it is no object, and, as in the toolkit's semi-supervised evaluation, it is background of the ground truth, so a prediction's object
pixels on it count against the prediction (the toolkit passes no void masks on that path); the object count is the first ground-truth
frame's largest id once void is removed; the first and last frames are left out; a prediction id above the object count is refused,
naming the file; an object absent from the predictions scores as an empty mask.  Each object is a row <seq>_<k> with the seven statistics, and the global row is the mean of each over all objects,
J&F being the mean of the two means.  It writes global_results-<set>.csv and per-sequence_results-<set>.csv under <results>, with the
toolkit's columns.  The other modes only read files.

    python scripts/eval_masks.py --gt video/gt_mask --pred video/masks_vos
    python scripts/eval_masks.py --ycbineoat YCBInEOAT --pred_name masks_vos
    python scripts/eval_masks.py --davis DAVIS --results results/davis --set val
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


DAVIS_VOID = 255
DAVIS_SEQUENCE_COLUMNS = ("Sequence", "J-Mean", "F-Mean")


def davis_sequence_names(root: str, set_name: str = "val", sequences: str | None = None) -> list:
    """The sequences of ImageSets/2017/<set_name>.txt, in its order, or the comma-separated `sequences` when given."""
    if sequences:
        return [n for n in (x.strip() for x in sequences.split(",")) if n]
    path = os.path.join(root, "ImageSets", "2017", f"{set_name}.txt")
    with open(path) as f:
        names = [line.strip() for line in f if line.strip()]
    if not names:
        raise ValueError(f"{path}: no sequences")
    return names


def davis_object_count(gt0) -> int:
    """The objects of a sequence: its first ground-truth frame's largest id once the void value is removed (0 for none)."""
    g = np.asarray(gt0)
    ids = g[g != DAVIS_VOID]
    return int(ids.max()) if ids.size else 0


def davis_check_ids(pred, n_objects: int, path: str) -> None:
    """Refuses a prediction holding an id above the sequence's object count, naming the file and the id."""
    top = int(np.asarray(pred).max())
    if top > n_objects:
        raise ValueError(f"{path}: object id {top} in the prediction, the sequence has {n_objects} objects")


def davis_read_sequence(gt_dir: str, pred_dir: str) -> tuple:
    """(frame ids, gt [F, H, W], pred [F, H, W], object count) of one sequence by the semi-supervised protocol: the object count from the
    first ground-truth frame, then every frame but the first and the last.  Predictions are read as indices and checked."""
    from bundletrack_b200.vos import read_palette_mask
    ids = sorted(name.split(".")[0] for name in os.listdir(gt_dir) if name.lower().endswith(".png"))
    if not ids:
        raise FileNotFoundError(f"{gt_dir}: no PNG ground-truth masks")
    n_objects = davis_object_count(read_palette_mask(os.path.join(gt_dir, f"{ids[0]}.png"))[0])
    if n_objects < 1:
        raise ValueError(f"{gt_dir}: the first ground-truth frame holds no object")
    kept = ids[1:-1]
    if not kept:
        raise ValueError(f"{gt_dir}: {len(ids)} frames leave none to score once the first and last are left out")
    gt, pred = [], []
    for i in kept:
        g = read_palette_mask(os.path.join(gt_dir, f"{i}.png"))[0]
        path = os.path.join(pred_dir, f"{i}.png")
        if not os.path.isfile(path):
            raise FileNotFoundError(f"{path}: no prediction for ground-truth frame {i}")
        p = read_palette_mask(path)[0]
        if gt and g.shape != gt[0].shape:
            raise ValueError(f"{gt_dir}/{i}.png: {g.shape[0]} x {g.shape[1]}, the sequence's masks are {gt[0].shape[0]} x {gt[0].shape[1]}")
        if p.shape != g.shape:
            raise ValueError(f"{path}: {p.shape[0]} x {p.shape[1]}, the ground truth is {g.shape[0]} x {g.shape[1]}")
        davis_check_ids(p, n_objects, path)
        gt.append(g)
        pred.append(p)
    return kept, np.stack(gt), np.stack(pred), n_objects


def write_davis_csvs(results: str, set_name: str, per_object: dict, mean: dict) -> tuple:
    """global_results-<set>.csv (MASK_SCORE_KEYS, one row) and per-sequence_results-<set>.csv (Sequence, J-Mean, F-Mean, a row per
    object) under `results`, three decimals, as the toolkit writes them.  Returns the two paths."""
    from bundletrack_b200.metrics import MASK_SCORE_KEYS
    g = os.path.join(results, f"global_results-{set_name}.csv")
    s = os.path.join(results, f"per-sequence_results-{set_name}.csv")
    with open(g, "w") as f:
        f.write(",".join(MASK_SCORE_KEYS) + "\n" + ",".join(f"{mean[k]:.3f}" for k in MASK_SCORE_KEYS) + "\n")
    with open(s, "w") as f:
        f.write(",".join(DAVIS_SEQUENCE_COLUMNS) + "\n")
        for name, r in per_object.items():
            f.write(f"{name},{r['J-Mean']:.3f},{r['F-Mean']:.3f}\n")
    return g, s


def evaluate_davis(root: str, results: str, set_name: str = "val", sequences: str | None = None, resolution: str = "480p",
                   bound_th: float = 0.008, device: int = 0, out=print) -> dict:
    """Scores every sequence's objects and writes the two CSVs.  Returns {"objects": {<seq>_<k>: mask_score's dict plus "frames", "j",
    "f"}, "mean": {statistic: mean over objects, J&F the mean of the two means}, "csv": (global path, per-sequence path)}."""
    from bundletrack_b200.metrics import MASK_SCORE_KEYS, MaskScore, mask_score
    per = {}
    for seq in davis_sequence_names(root, set_name, sequences):
        ids, gt, pred, n = davis_read_sequence(os.path.join(root, "Annotations", resolution, seq), os.path.join(results, seq))
        ms = MaskScore(CHUNK, gt.shape[1], gt.shape[2], device=device)
        try:
            # void_value -1: the toolkit's semi-supervised path scores G = (gt == k) with void as background and no void mask
            j, f = ms.objects(pred, gt, n, -1, bound_th)
        finally:
            ms.close()
        for k in range(n):
            r = mask_score(j[:, k], f[:, k])
            r.update(frames=ids, j=j[:, k].tolist(), f=f[:, k].tolist())
            per[f"{seq}_{k + 1}"] = r
            out(f"{seq}_{k + 1}: {len(ids)} frames, " + ", ".join(f"{key} {r[key]:.4f}" for key in MASK_SCORE_KEYS))
    mean = {k: float(np.mean([r[k] for r in per.values()])) for k in MASK_SCORE_KEYS}
    mean["J&F-Mean"] = (mean["J-Mean"] + mean["F-Mean"]) / 2.0
    out(f"global, {len(per)} objects: " + ", ".join(f"{k} {mean[k]:.4f}" for k in MASK_SCORE_KEYS))
    return {"objects": per, "mean": mean, "csv": write_davis_csvs(results, set_name, per, mean)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--gt", help="one sequence: the ground-truth mask directory")
    ap.add_argument("--pred", help="one sequence: the predicted mask directory")
    ap.add_argument("--ycbineoat", help="a YCBInEOAT root: every <video>/gt_mask against <video>/<pred_name>")
    ap.add_argument("--pred_name", default="masks_vos", help="the prediction directory's name inside each video (with --ycbineoat)")
    ap.add_argument("--davis", help="a DAVIS root: every sequence of --set, per object, against <results>/<seq>")
    ap.add_argument("--results", help="with --davis: the predictions' directory, where the CSVs are written")
    ap.add_argument("--set", default="val", help="with --davis: the ImageSets/2017 list")
    ap.add_argument("--sequences", help="with --davis: comma-separated sequences in place of --set's")
    ap.add_argument("--resolution", default="480p", help="with --davis: the Annotations resolution")
    ap.add_argument("--keep_ends", action="store_true", help="score the first and last frames too")
    ap.add_argument("--bound_th", type=float, default=0.008, help="boundary tolerance, a fraction of the image diagonal")
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    if a.davis:
        if a.ycbineoat or a.gt or a.pred or a.keep_ends:
            ap.error("--davis takes --results, --set, --sequences and --resolution, not --gt, --pred, --ycbineoat or --keep_ends")
        if not a.results:
            ap.error("--davis needs --results")
        return evaluate_davis(a.davis, a.results, a.set, a.sequences, a.resolution, a.bound_th, a.device)
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
