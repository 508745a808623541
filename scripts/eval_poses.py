#!/usr/bin/env python3
"""ADD / ADD-S AUC of tracked sequences, with the reference's evaluation (scripts/eval_ycbineoat.py) and its directory layout:

    <dataset_dir>/<video>/rgb/*.png                 one per frame (counted only)
    <dataset_dir>/<video>/annotated_poses/*.txt     ground-truth ob_in_cam, 4 x 4 text
    <results_dir>/<video>/poses/*.txt               tracked ob_in_cam (bt_pose_write_txt / Bundler::saveNewframeResult)
    <model_dir>/<object>/points.xyz                 the model points, one "x y z" row each

Files are paired by sorted name; the three counts of a video must agree.  A pose file that cannot be read counts as the identity, as in the
reference.  ADD and ADD-S come from one device call per video (bt_pose_metrics); AUC is VOCap at 0.1 m, printed x 100 per object and overall
in the reference's format.  This script only reads files.

    python scripts/eval_poses.py --dataset_dir YCBInEOAT --model_dir YCB_Video_Dataset/models --results_dir /tmp/BundleTrack/ycbineoat
"""
from __future__ import annotations

import argparse
import glob
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# YCBInEOAT's videos and the YCB-Video object each one shows
YCBINEOAT_OBJECTS = {
    "bleach0": "021_bleach_cleanser",
    "bleach_hard_00_03_chaitanya": "021_bleach_cleanser",
    "cracker_box_reorient": "003_cracker_box",
    "cracker_box_yalehand0": "003_cracker_box",
    "mustard0": "006_mustard_bottle",
    "mustard_easy_00_02": "006_mustard_bottle",
    "sugar_box1": "004_sugar_box",
    "sugar_box_yalehand0": "004_sugar_box",
    "tomato_soup_can_yalehand0": "005_tomato_soup_can",
}


def load_pose(path: str, out=print) -> np.ndarray:
    try:
        P = np.loadtxt(path)
        if P.shape != (4, 4):
            raise ValueError(f"shape {P.shape}")
        return P
    except Exception:
        out(f"ERROR pose file not readable {path}")
        return np.eye(4)


def evaluate(dataset_dir: str, model_dir: str, results_dir: str, video_to_object: dict = None, device: int = 0, max_err: float = 0.1, out=print) -> dict:
    """Returns {"objects": {object: {"add": [...], "add-s": [...], "add_auc": x, "adds_auc": y}}, "add_auc": x, "adds_auc": y, "n": frames};
    AUCs x 100 as printed."""
    from bundletrack_b200.metrics import PoseMetrics, vocap
    v2o = dict(YCBINEOAT_OBJECTS if video_to_object is None else video_to_object)
    res = {obj: {"add": [], "add-s": []} for obj in v2o.values()}
    jobs = []
    for folder in sorted(glob.glob(os.path.join(dataset_dir, "*"))):
        if ".tar.gz" in folder or not os.path.isdir(folder):
            continue
        video = os.path.basename(folder)
        rgb = sorted(glob.glob(os.path.join(folder, "rgb", "*.png")))
        pred = sorted(glob.glob(os.path.join(results_dir, video, "poses", "*.txt")))
        gt = sorted(glob.glob(os.path.join(folder, "annotated_poses", "*.txt")))
        out(f"{video}: #rgb_files={len(rgb)}, #pred_files={len(pred)}, #gt_files={len(gt)}")
        if len(rgb) != len(pred) or len(pred) != len(gt):
            raise RuntimeError(f"ERROR files not match {folder}")
        if video not in v2o:
            raise RuntimeError(f"no object is known for video {video}")
        if not rgb:
            continue
        jobs.append((v2o[video], np.stack([load_pose(p, out) for p in pred]), np.stack([load_pose(p, out) for p in gt])))
    models = {obj: np.loadtxt(os.path.join(model_dir, obj, "points.xyz"), ndmin=2)[:, :3] for obj in {j[0] for j in jobs}}
    if jobs:
        pm = PoseMetrics(max(len(m) for m in models.values()), max(len(j[1]) for j in jobs), device=device)
        try:
            for obj, P, G in jobs:
                add, adds = pm(models[obj], P, G)
                res[obj]["add"] += add.tolist()
                res[obj]["add-s"] += adds.tolist()
        finally:
            pm.close()
    out("----------------------------------")
    all_add, all_adds = [], []
    for obj, r in res.items():
        all_add += r["add"]
        all_adds += r["add-s"]
        r["adds_auc"], r["add_auc"] = vocap(r["add-s"], max_err) * 100, vocap(r["add"], max_err) * 100
        out(f"{obj} #pred={len(r['add-s'])}: adi={r['adds_auc']} add={r['add_auc']}")
    adds_auc, add_auc = vocap(all_adds, max_err) * 100, vocap(all_add, max_err) * 100
    out(f"Total pose: {len(all_adds)}")
    out(f"\nOverall, adi={adds_auc} add={add_auc}")
    return {"objects": res, "add_auc": add_auc, "adds_auc": adds_auc, "n": len(all_adds)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--dataset_dir", required=True)
    ap.add_argument("--model_dir", required=True)
    ap.add_argument("--results_dir", required=True)
    ap.add_argument("--objects", default=None, help="JSON file {video: object}; default: the YCBInEOAT videos")
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    v2o = None
    if a.objects:
        with open(a.objects) as f:
            v2o = json.load(f)
    evaluate(a.dataset_dir, a.model_dir, a.results_dir, v2o, a.device)


if __name__ == "__main__":
    main()
