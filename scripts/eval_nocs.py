#!/usr/bin/env python3
"""NOCS-REAL275 scores of tracked sequences (5 deg 5 cm, IoU25, rotation and translation error), as the reference's scripts/eval_nocs.py
converts the tracker's poses and its scripts/benchmark.py (the 6-PACK benchmark) scores them, with the reference's directory layout:

    <nocs_dir>/NOCS-REAL275-additional/data_list/real_val/<cls>/<model>/list.txt   lines "real_val/scene_<k>/<frame>"
    <nocs_dir>/real_test/scene_<k>/<frame>_meta.txt                                 "<instance> <class> ... <model>" per line
    <nocs_dir>/gts/real_test/results_real_test_scene_<k>_<frame>.pkl                {"gt_RTs": [...]} (metres)
    <nocs_dir>/NOCS-REAL275-additional/model_scales/<model>.txt                     8 corner rows "x y z"
    <results_dir>/<model>_<k>/poses/<frame:04d>.txt                                 tracked ob_in_cam (run_nocs.py, bt_pose_write_txt)

The conversion happens in memory and the script writes nothing.  Kept from the reference, because they move its numbers (DESIGN.md §3.8):
  - a pose file that cannot be read as 4 x 4 is the identity (printed as ERROR);
  - the initial-pose noise of eval_nocs.py's __main__ (--noise 0.02 0: metres, degrees; --no-noise turns it off), draw for draw from
    np.random.seed(0) over the list files in sorted order: per scene 3 translation uniforms, the rotation magnitude and random_direction's
    two, then Rodrigues and inv(init_pose @ inv(pred)) @ init_pose_new for the scene's later frames;
  - the benchmark numbers its prediction files by the count of records with a ground-truth pickle, the conversion by line index, so after a
    missing pickle a model's later records read the prediction of the line before them (or none, counted but not scored, across a scene
    change); a record whose meta file does not name the instance is counted but not scored;
  - the benchmark's theta, shift and IoU (bt_nocs_metrics, one device call for all records) and its aggregation (bt_nocs_score).
Models within a class are taken in sorted order (the reference's glob order is not pinned).  Prints in the benchmark's format.

    python scripts/eval_nocs.py --nocs_dir NOCS --results_dir /tmp/BundleTrack/nocs
"""
from __future__ import annotations

import argparse
import glob
import math
import os
import pickle
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SYNSET_NAMES = ["BG", "bottle", "bowl", "camera", "can", "laptop", "mug"]
SYMMETRIC = ("bottle", "bowl", "can")
STARS = "*" * 56


def load_pose(path: str, out=print) -> np.ndarray:
    try:
        P = np.loadtxt(path)
        if P.shape != (4, 4):
            raise ValueError(f"shape {P.shape}")
        return P
    except Exception as e:
        out("ERROR", e)
        return np.eye(4)


def rodrigues(v) -> np.ndarray:
    """The rotation matrix of the axis-angle vector v (OpenCV's Rodrigues formula; a zero vector is the identity)."""
    v = np.asarray(v, np.float64).reshape(3)
    th = math.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])
    if th < np.finfo(np.float64).eps:
        return np.eye(3)
    c, s = math.cos(th), math.sin(th)
    r = v * (1.0 / th)
    rx = np.array([[0.0, -r[2], r[1]], [r[2], 0.0, -r[0]], [-r[1], r[0], 0.0]])
    return c * np.eye(3) + (1.0 - c) * np.outer(r, r) + s * rx


def _random_direction(rng) -> np.ndarray:
    theta = rng.uniform(0, 1) * np.pi * 2
    phi = np.arccos((2 * (rng.uniform(0, 1))) - 1)
    return np.array([1 * math.sin(phi) * math.cos(theta), 1 * math.sin(phi) * math.sin(theta), 1 * math.cos(phi)])


def convert(nocs_dir: str, results_dir: str, noise=(0.02, 0.0), out=print) -> dict:
    """eval_nocs.py's conversion in memory: {(class id, "<model>_scene_<k>_<line>"): 4 x 4 pose as the benchmark reads it back (the rotation
    and the translation in mm, bottom row [0,0,0,1])}.  noise = (metres, degrees), or None for no noise."""
    rng = np.random.RandomState(0)
    files = {}
    for list_file in sorted(glob.glob(f"{nocs_dir}/NOCS-REAL275-additional/data_list/real_val/*/*/list.txt")):
        with open(list_file) as ff:
            lines = ff.readlines()
        ob_name = list_file.split("/")[-2]
        class_id = next((k for k, name in enumerate(SYNSET_NAMES) if name in ob_name), None)
        last_scene_id, init_pose, init_pose_new = None, None, None
        for i in range(len(lines)):
            line = lines[i].rstrip().split("/")
            scene_id, frame_id = int(line[1][-1]), int(line[2])
            pred = load_pose(f"{results_dir}/{ob_name}_{scene_id}/poses/{frame_id:04d}.txt", out)
            if last_scene_id is None or last_scene_id != scene_id:
                init_pose = pred.copy()
                if noise is not None:
                    trans_noise, rot_noise = noise[0], noise[1] / 180.0 * np.pi
                    pred[:3, 3] += np.array([rng.uniform(-trans_noise, trans_noise) for _ in range(3)])
                    mag_R = rng.uniform(-rot_noise, rot_noise)
                    pred[:3, :3] = pred[:3, :3] @ rodrigues(_random_direction(rng) * mag_R)
                    init_pose_new = pred.copy()
            elif noise is not None:
                cam_in_firstcam = init_pose @ np.linalg.inv(pred)
                pred = np.linalg.inv(cam_in_firstcam) @ init_pose_new
            P = np.eye(4)
            P[:3, :3] = pred[:3, :3]
            P[:3, 3] = pred[:3, 3] * 1000          # the z-180 flips of the conversion and the benchmark cancel exactly
            files[(class_id, f"{ob_name}_scene_{scene_id}_{i}")] = P
            last_scene_id = scene_id
    return files


def collect(nocs_dir: str, results_dir: str, noise=(0.02, 0.0), out=print) -> dict:
    """The benchmark's records in its visiting order: class, model, scene, frame, scored flag, and for scored ones pred / gt (mm) and the
    model's corners."""
    files = convert(nocs_dir, results_dir, noise, out)
    rec = {"cls": [], "model": [], "scene": [], "frame": [], "scored": [], "pred": [], "gt": [], "corners": []}
    for cls_idx in range(1, 7):
        cls_path = os.path.join(nocs_dir, "NOCS-REAL275-additional", "data_list/real_val", str(cls_idx))
        models = sorted(glob.glob(os.path.join(cls_path, "*")))
        if not models:
            raise RuntimeError(f"no model listed under {cls_path}")
        for model_path in models:
            model_name = model_path.split("/")[-1]
            model_num = 0
            corners = None
            with open(os.path.join(model_path, "list.txt")) as list_file:
                for img_path in list_file:
                    img_path = os.path.join(nocs_dir, img_path.replace("real_val", "real_test")).replace("\n", "")
                    scene = img_path.split("/")[-2]
                    frame_id = int(os.path.basename(img_path))
                    gt_path = os.path.join(nocs_dir, "gts", "real_test", "results_real_test_" + scene + "_%04d.pkl" % frame_id)
                    if not os.path.exists(gt_path):
                        out("ERROR nocs_gt_path not found:", gt_path)
                        continue
                    key = (cls_idx, f"{model_name}_{scene}_{model_num}")
                    model_num += 1
                    for k, v in (("cls", cls_idx), ("model", model_name), ("scene", scene), ("frame", frame_id), ("scored", 0)):
                        rec[k].append(v)
                    if key not in files:
                        out(f"ERROR prediction {key[1]} not found")
                        continue
                    num_idx, found = 0, False
                    with open(img_path + "_meta.txt") as obj_f:
                        for ln in obj_f:
                            if int(ln.split(" ")[1]) == cls_idx and ln.split(" ")[-1].replace("\n", "") == model_name:
                                found = True
                                break
                            num_idx += 1
                    if not found:
                        continue
                    with open(gt_path, "rb") as f:
                        result = pickle.load(f)
                    try:
                        gt = np.array(result["gt_RTs"][num_idx])
                    except Exception as e:
                        out(f"ERROR loading gt from {gt_path}:", e)
                        gt = np.eye(4)
                    gt[:3, 3] = gt[:3, 3] * 1000
                    if corners is None:
                        corners = np.loadtxt(os.path.join(nocs_dir, "NOCS-REAL275-additional", "model_scales", model_name + ".txt"), ndmin=2)
                    rec["scored"][-1] = 1
                    rec["pred"].append(files[key])
                    rec["gt"].append(gt.astype(np.float64))
                    rec["corners"].append(np.asarray(corners, np.float64).reshape(8, 3))
    rec["pred"] = np.array(rec["pred"]).reshape(-1, 4, 4)
    rec["gt"] = np.array(rec["gt"]).reshape(-1, 4, 4)
    rec["corners"] = np.array(rec["corners"]).reshape(-1, 8, 3)
    return rec


def evaluate(nocs_dir: str, results_dir: str, noise=(0.02, 0.0), device: int = 0, out=print) -> dict:
    """Returns {"classes": {name: {"5cm5deg", "iou25", "rot_err", "tran_err"}}, and the same four overall, "n", "n_scored", "records"},
    with the numbers as printed: fractions x 100, the rotation error in degrees and the translation error in cm."""
    from bundletrack_b200.metrics import NocsMetrics, nocs_score
    rec = collect(nocs_dir, results_dir, noise, out)
    scored = np.array(rec["scored"], np.int32)
    cls = np.array(rec["cls"], np.int32)
    theta, shift, iou = (np.full(len(cls), np.nan) for _ in range(3))
    n_scored = int(scored.sum())
    if n_scored:
        nm = NocsMetrics(n_scored, device=device)
        try:
            t, s, u = nm(rec["pred"], rec["gt"], rec["corners"], np.isin(cls[scored == 1], [SYNSET_NAMES.index(c) for c in SYMMETRIC]))
        finally:
            nm.close()
        theta[scored == 1], shift[scored == 1], iou[scored == 1] = t, s, u
    per, ov = nocs_score(cls, scored, theta, shift, iou)
    res = {"classes": {}, "n": len(cls), "n_scored": n_scored, "records": dict(rec, theta=theta, shift=shift, iou=iou)}
    for c in range(6):
        v = {"5cm5deg": float(per[c, 0]) * 100, "iou25": float(per[c, 1]) * 100, "rot_err": float(per[c, 2]), "tran_err": float(per[c, 3]) / 10}
        res["classes"][SYNSET_NAMES[c + 1]] = v
        out(STARS)
        out(f"class={SYNSET_NAMES[c + 1]}")
        out("5cm 5degree:", v["5cm5deg"])
        out("IoU 25:     ", v["iou25"])
        out("rot error:  ", v["rot_err"])
        out("tran error: ", v["tran_err"])
    res.update({"5cm5deg": float(ov[0]) * 100, "iou25": float(ov[1]) * 100, "rot_err": float(ov[2]), "tran_err": float(ov[3]) / 10})
    out(STARS)
    out("5cm 5degree:", res["5cm5deg"])
    out("IoU 25:     ", res["iou25"])
    out("rot error:  ", res["rot_err"])
    out("tran error: ", res["tran_err"])
    out(STARS)
    out("Mean 5cm 5degree:", res["5cm5deg"])
    out("Mean IoU 25:     ", res["iou25"])
    out("Mean rot error:  ", res["rot_err"])
    out("Mean tran error: ", res["tran_err"])
    out(STARS)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--nocs_dir", required=True)
    ap.add_argument("--results_dir", required=True)
    ap.add_argument("--noise", type=float, nargs=2, default=[0.02, 0.0], metavar=("TRANS_M", "ROT_DEG"),
                    help="initial-pose noise of the reference's protocol (default 0.02 0)")
    ap.add_argument("--no-noise", action="store_true", help="score the tracked poses as they are")
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    evaluate(a.nocs_dir, a.results_dir, None if a.no_noise else tuple(a.noise), a.device)


if __name__ == "__main__":
    main()
