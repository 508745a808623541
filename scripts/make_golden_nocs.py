#!/usr/bin/env python3
"""tests/golden/ref_nocs.npz: NOCS-REAL275 scores from the reference's OWN 6-PACK benchmark (scripts/benchmark.py) and conversion
(scripts/eval_nocs.py), imported from a reference checkout at generation time.  The tests read only the .npz.

A synthetic NOCS tree (all six classes, two bottle models, three scenes, 40 frames per model and scene; pose errors around 5 deg, 50 mm and
IoU 0.25; a missing ground-truth pickle mid-list and a meta file without one instance) is written to a temporary directory and scored by
eval_nocs.eval_all_ours with and without noise.  A second, small tree has a class with no record above IoU 0.25 (NaN means).  The reference's
modules that eval_nocs imports but never calls (matplotlib, open3d, transformations) are stubbed, and its hard-coded output directory is
pointed at a temporary one.  Recorded: the trees (every text file and the pickles' gt_RTs), the records in the order the benchmark visited
them with their inputs and theta / shift / IoU, and every printed number.  An adversarial record set is scored through the benchmark's
functions directly: pred == gt bit for bit, 180 deg flips, a float32 + 10-digit text round trip, negative determinants and ground-truth
bottom rows other than [0,0,0,1].

    python scripts/make_golden_nocs.py --reference <reference checkout> [--out tests/golden/ref_nocs.npz]
"""
from __future__ import annotations

import argparse
import contextlib
import importlib.util
import io
import json
import os
import pickle
import sys
import tempfile
import types

import numpy as np

SYNSET = ["BG", "bottle", "bowl", "camera", "can", "laptop", "mug"]
MODELS = {1: ["bottle_blue_norm", "bottle_red_norm"], 2: ["bowl_white_norm"], 3: ["camera_black_norm"], 4: ["can_tea_norm"],
          5: ["laptop_air_norm"], 6: ["mug_brown_norm"]}
N_FRAMES = 40


def _rot(axis, deg):
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    t = np.deg2rad(deg)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(t) * K + (1 - np.cos(t)) * K @ K


def _fmt(P) -> str:
    return "".join(" ".join(f"{v:.10g}" for v in row) + "\n" for row in P)


def make_tree(seed: int = 0, far_class: int | None = None, n_frames: int = N_FRAMES, anomalies: bool = True) -> dict:
    """{"files": {relative path: text}, "pickles": {relative path: gt_RTs [k,4,4]}} of a synthetic NOCS tree.  Paths are relative to the
    tree's root, which holds nocs/ (the dataset) and results/ (the tracker's poses)."""
    rng = np.random.default_rng(seed)
    files, pickles = {}, {}
    scenes = {1: [(1, 0), (1, 1), (2, 0), (3, 0), (4, 0), (5, 0), (6, 0)],          # scene -> (class, model index)
              2: [(1, 0), (2, 0), (3, 0), (4, 0), (5, 0), (6, 0)],
              3: [(1, 1), (2, 0), (4, 0), (6, 0)]}
    scales = {}
    for c, names in MODELS.items():
        for m in names:
            ext = rng.uniform(40, 160, 3)          # half extents, mm
            corners = np.array([[sx * ext[0], sy * ext[1], sz * ext[2]] for sx in (1, -1) for sy in (1, -1) for sz in (1, -1)])
            scales[m] = corners
            files[f"nocs/NOCS-REAL275-additional/model_scales/{m}.txt"] = "".join(f"{x:.6f} {y:.6f} {z:.6f}\n" for x, y, z in corners)
    lists = {}
    for k, objs in scenes.items():
        gts = {}
        for c, mi in objs:
            m = MODELS[c][mi]
            s = rng.uniform(0.15, 0.4)
            R0 = _rot(rng.normal(size=3), rng.uniform(0, 180))
            t0 = np.array([rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2), rng.uniform(0.6, 1.2)])
            w, v = rng.normal(size=3), rng.normal(size=3) * 0.004
            for f in range(n_frames):
                R = _rot(w, 0.8 * f) @ R0
                t = t0 + v * f
                G = np.eye(4)
                G[:3, :3], G[:3, 3] = s * R, t
                gts.setdefault(f, []).append((c, m, G))
                # tracked pose: the ground truth with an error that straddles 5 deg, 50 mm and IoU 0.25
                if f == 0:
                    ang, dt = 2.0 + rng.uniform(0, 1), rng.normal(size=3) * 0.004        # non-marginal first-frame rotation error
                else:
                    ang = rng.choice([rng.uniform(0, 4), rng.uniform(3, 7), rng.uniform(6, 20)])
                    dt = rng.normal(size=3) * rng.choice([0.01, 0.035, 0.08, 0.2])
                if far_class == c:
                    dt = np.array([0.0, 0.0, 1.5]) + rng.normal(size=3) * 0.1
                P = np.eye(4)
                P[:3, :3] = _rot(rng.normal(size=3), ang) @ R
                P[:3, 3] = t + dt
                files[f"results/{m}_{k}/poses/{f:04d}.txt"] = _fmt(P.astype(np.float32).astype(np.float64))
                lists.setdefault((c, m), []).append(f"real_val/scene_{k}/{f:04d}")
        for f, inst in gts.items():
            if anomalies and k == 2 and f == 17:
                continue                                  # no ground-truth pickle: the benchmark's pairing shifts from here on
            keep = [x for x in inst if not (anomalies and k == 1 and f == 9 and x[1] == "can_tea_norm")]     # meta without this instance
            files[f"nocs/real_test/scene_{k}/{f:04d}_meta.txt"] = "".join(f"{j + 1} {c} {m}\n" for j, (c, m, _) in enumerate(keep))
            pickles[f"nocs/gts/real_test/results_real_test_scene_{k}_{f:04d}.pkl"] = np.stack([G for _, _, G in keep])
    for (c, m), lines in lists.items():
        files[f"nocs/NOCS-REAL275-additional/data_list/real_val/{c}/{m}/list.txt"] = "".join(ln + "\n" for ln in lines)
    return {"files": files, "pickles": pickles}


def write_tree(root: str, tree: dict) -> tuple:
    """Writes a make_tree() tree under root; returns (nocs_dir, results_dir)."""
    for rel, text in tree["files"].items():
        p = os.path.join(root, rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "w") as f:
            f.write(text)
    for rel, gt in tree["pickles"].items():
        p = os.path.join(root, rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "wb") as f:
            pickle.dump({"gt_RTs": np.asarray(gt, np.float64)}, f)
    return os.path.join(root, "nocs"), os.path.join(root, "results")


def tree_to_arrays(tree: dict, prefix: str) -> dict:
    keys = sorted(tree["pickles"])
    return {f"{prefix}_files": np.array(json.dumps(tree["files"], sort_keys=True)), f"{prefix}_pkl_keys": np.array(json.dumps(keys)),
            f"{prefix}_pkl_n": np.array([len(tree["pickles"][k]) for k in keys], np.int64),
            f"{prefix}_pkl_rts": np.concatenate([tree["pickles"][k] for k in keys]).astype(np.float64)}


def tree_from_arrays(z, prefix: str) -> dict:
    keys = json.loads(str(z[f"{prefix}_pkl_keys"]))
    off = np.concatenate([[0], np.cumsum(z[f"{prefix}_pkl_n"])])
    rts = z[f"{prefix}_pkl_rts"]
    return {"files": json.loads(str(z[f"{prefix}_files"])), "pickles": {k: rts[off[i]:off[i + 1]] for i, k in enumerate(keys)}}


# ---- running the reference -------------------------------------------------------------------------------------------------------------

def _load(name: str, path: str, src: str | None = None):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    if src is None:
        spec.loader.exec_module(mod)
    else:
        exec(compile(src, path, "exec"), mod.__dict__)
    return mod


def _stubs():
    for name in ("matplotlib", "matplotlib.pyplot", "open3d", "transformations"):
        if name not in sys.modules:
            sys.modules[name] = types.ModuleType(name)
    sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]


def run_reference(ref_scripts: str, nocs_dir: str, results_dir: str, add_noise: bool, out_dir: str) -> dict:
    """eval_nocs.eval_all_ours on a fresh import (np.random.seed(0) as at the reference's start), traced record by record."""
    _stubs()
    sys.path.insert(0, ref_scripts)
    bench = _load("benchmark", os.path.join(ref_scripts, "benchmark.py"))
    _load("Utils", os.path.join(ref_scripts, "Utils.py"))
    src = open(os.path.join(ref_scripts, "eval_nocs.py")).read()
    assert src.count("'/tmp/nocs_res_ours'") == 1
    ev = _load("eval_nocs_ref", os.path.join(ref_scripts, "eval_nocs.py"), src.replace("'/tmp/nocs_res_ours'", repr(out_dir)))
    ev.nocs_dir, ev.results_dir, ev.args = nocs_dir, results_dir, argparse.Namespace(nocs_dir=nocs_dir)

    recs, cur, pending = [], {}, []

    def t_open(path, *a, **k):
        if str(path).endswith("list.txt"):
            parts = str(path).split("/")
            cur.update(cls=int(parts[-3]), model=parts[-2])
        return open(path, *a, **k)

    class PathProxy:
        def __getattr__(self, k):
            return getattr(os.path, k)

        @staticmethod
        def exists(p):
            r = os.path.exists(p)
            if r and str(p).endswith(".pkl") and "results_real_test_" in str(p):
                stem = os.path.basename(p)[len("results_real_test_"):-4]
                recs.append(dict(cls=cur["cls"], model=cur["model"], scene=stem.rsplit("_", 1)[0], frame=int(stem.rsplit("_", 1)[1]), scored=0))
            return r

    class OsProxy:
        path = PathProxy()

        def __getattr__(self, k):
            return getattr(os, k)

    norm0, rt0, iou0 = bench.normalizeRotation, bench.compute_RT_degree_cm_symmetry, bench.compute_3d_iou_new

    def t_norm(pose):
        pending.append(np.array(pose, np.float64, copy=True))
        return norm0(pose)

    def t_rt(RT_1, RT_2, class_id, hv, names):
        r = rt0(RT_1, RT_2, class_id, hv, names)
        recs[-1].update(scored=1, pred=pending[-2], gt=pending[-1], theta=float(r[0]), shift=float(r[1]))
        pending.clear()
        return r

    def t_iou(RT_1, RT_2, c1, c2, hv, n1, n2):
        v = iou0(RT_1, RT_2, c1, c2, hv, n1, n2)
        recs[-1].update(iou=float(v), corners=np.asarray(c1, np.float64).T.copy())
        return v

    bench.open, bench.os = t_open, OsProxy()
    bench.normalizeRotation, bench.compute_RT_degree_cm_symmetry, bench.compute_3d_iou_new = t_norm, t_rt, t_iou
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        ev.eval_all_ours(use_6pack_eval_code=True, verbose=True, add_noise=add_noise, noise_pair=[0.02, 0])
    sys.path.remove(ref_scripts)
    text = buf.getvalue()
    printed = _parse_printed(text)
    return {"records": recs, "printed": printed, "text": text}


def _parse_printed(text: str) -> np.ndarray:
    """[8, 4]: the six classes, the overall lines and the Mean lines: 5cm 5degree, IoU 25, rot error, tran error as printed."""
    keys = ("5cm 5degree:", "IoU 25:", "rot error:", "tran error:")
    rows, row = [], []
    for ln in text.splitlines():
        s = ln.strip()
        if s.startswith("Mean "):
            s = s[5:]
        for k in keys:
            if s.startswith(k):
                row.append(float(s[len(k):].strip()))
                if len(row) == 4:
                    rows.append(row)
                    row = []
    assert len(rows) == 8, rows
    return np.array(rows, np.float64)


def _records_to_arrays(recs: list, prefix: str) -> dict:
    sc = [r for r in recs if r["scored"]]
    return {f"{prefix}_cls": np.array([r["cls"] for r in recs], np.int32), f"{prefix}_scored": np.array([r["scored"] for r in recs], np.int32),
            f"{prefix}_model": np.array(json.dumps([r["model"] for r in recs])), f"{prefix}_scene": np.array(json.dumps([r["scene"] for r in recs])),
            f"{prefix}_frame": np.array([r["frame"] for r in recs], np.int32),
            f"{prefix}_pred": np.array([r["pred"] for r in sc]).reshape(-1, 4, 4), f"{prefix}_gt": np.array([r["gt"] for r in sc]).reshape(-1, 4, 4),
            f"{prefix}_corners": np.array([r["corners"] for r in sc]).reshape(-1, 8, 3),
            f"{prefix}_theta": np.array([r["theta"] for r in sc]), f"{prefix}_shift": np.array([r["shift"] for r in sc]),
            f"{prefix}_iou": np.array([r["iou"] for r in sc])}


def adversarial(bench, seed: int = 5) -> dict:
    """Records scored by the benchmark's functions directly, each pose pair as main() hands it over (normalised first)."""
    rng = np.random.default_rng(seed)
    P, G, C, cls, kind = [], [], [], [], []

    def pose(s=1.0):
        M = np.eye(4)
        M[:3, :3] = s * _rot(rng.normal(size=3), rng.uniform(0, 180))
        M[:3, 3] = rng.uniform(-200, 200, 3) + [0, 0, 800]
        return M

    def box():
        e = rng.uniform(40, 160, 3)
        return np.array([[sx * e[0], sy * e[1], sz * e[2]] for sx in (1, -1) for sy in (1, -1) for sz in (1, -1)])

    def add(p, g, c, k):
        P.append(p); G.append(g); C.append(box()); cls.append(c); kind.append(k)

    for c in (1, 2, 4, 3, 5, 6):
        for _ in range(40):
            g = pose(rng.uniform(0.1, 0.4))
            add(g.copy(), g.copy(), c, "equal")
            p = g.copy()
            p[:3, :3] = g[:3, :3] @ _rot([1, 0, 0] if c in (1, 2, 4) else rng.normal(size=3), 180.0)
            add(p, g, c, "flip180")
            q = np.array([[float(f"{v:.10g}") for v in row] for row in g.astype(np.float32)])
            q[3] = [0, 0, 0, 1]
            add(q, g, c, "text_roundtrip")
        for _ in range(6):
            g = pose()
            p = g.copy()
            p[:3, :3] = p[:3, :3] @ np.diag([1.0, 1.0, -1.0])
            add(p, g, c, "negative_det")
            g2 = g.copy()
            g2[3] = [0, 0, 0, 2] if _ % 2 else [1e-3, 0, 0, 1]
            add(pose(), g2, c, "gt_bottom_row")
    thetas, shifts, ious = [], [], []
    for p, g, c, bb in zip(P, G, cls, C):
        pn, gn = bench.normalizeRotation(p.copy()), bench.normalizeRotation(g.copy())
        r = bench.compute_RT_degree_cm_symmetry(pn, gn, c, 1, SYNSET)
        v = bench.compute_3d_iou_new(gn, pn, bb.T, bb.T, 1, SYNSET[c], SYNSET[c])
        thetas.append(float(r[0])); shifts.append(float(r[1])); ious.append(float(v))
    return {"adv_pred": np.array(P), "adv_gt": np.array(G), "adv_corners": np.array(C), "adv_cls": np.array(cls, np.int32),
            "adv_kind": np.array(json.dumps(kind)), "adv_theta": np.array(thetas), "adv_shift": np.array(shifts), "adv_iou": np.array(ious)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reference", required=True, help="a checkout of the reference (its scripts/ are imported)")
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ref_nocs.npz"))
    a = ap.parse_args()
    ref_scripts = os.path.join(a.reference, "scripts")
    out = {}
    import warnings
    warnings.simplefilter("ignore")
    with tempfile.TemporaryDirectory() as tmp:
        trees = {"main": make_tree(0), "far": make_tree(1, far_class=5, n_frames=12, anomalies=False)}
        runs = (("main_noise", "main", True), ("main_plain", "main", False), ("far_plain", "far", False))
        for name, tree in trees.items():
            out.update(tree_to_arrays(tree, name))
        for run, tname, noise in runs:
            root = os.path.join(tmp, tname)
            if not os.path.isdir(root):
                write_tree(root, trees[tname])
            nocs_dir, results_dir = os.path.join(root, "nocs"), os.path.join(root, "results")
            r = run_reference(ref_scripts, nocs_dir, results_dir, noise, os.path.join(tmp, "out_" + run))
            out.update(_records_to_arrays(r["records"], run))
            out[f"{run}_printed"] = r["printed"]
            print(run, len(r["records"]), "records,", sum(x["scored"] for x in r["records"]), "scored; printed:\n", r["printed"])
        out.update(adversarial(_load("benchmark_adv", os.path.join(ref_scripts, "benchmark.py"))))
    np.savez_compressed(a.out, **out)
    print("wrote", a.out, os.path.getsize(a.out), "bytes")


if __name__ == "__main__":
    main()
