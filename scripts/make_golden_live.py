"""Records, on an H100 with oracle/_ref built, what the reference's own kernels return for the inputs of the GPU tests that compare
with the reference, so that those tests run from stored data wherever the reference is not available:

  ref_live_solver.npz   optimizeFrames on the windows of test_solver_gpu.py (two windows, the 30-keyframe pool, the 200-window
                        sweep): poses (3x4 rows; the sweep's as rotation vector + translation), the reference's pair directions,
                        and for the sweep its run-to-run difference
  ref_live_frame.npz    the Frame front end on synth.make_raw_depth(7, 480, 640), every pixel, stored as the difference from
                        oracle/frame_oracle.py's outputs in small int8 steps (see frame_encode in tests/test_frontend_gpu.py)
  ref_live_ransac.npz   ransacMultiPairGPU on the point sets of test_ransac_matches_reference_live, inlier sets as bit masks
  ref_live_fused.npz    optimizeFrames (twice) on the EntryJ list the fused matcher chain builds in
                        test_fused_pipeline_matches_oracle_and_feeds_solver, with that list

    python scripts/make_golden_live.py OUT_DIR [solver] [frame] [ransac] [fused]      (default: all; then copy
    OUT_DIR/ref_live_*.npz to tests/golden/)
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from scipy.spatial.transform import Rotation

import oracle
from bundletrack_b200 import synth

out_dir = sys.argv[1]
parts = set(sys.argv[2:]) or {"solver", "frame", "ransac", "fused"}
os.makedirs(out_dir, exist_ok=True)
dev = torch.device("cuda:0")
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))


def upload(w):
    return [torch.from_numpy(w.depth[k]).to(dev) for k in range(w.n_frames)], [torch.from_numpy(w.normal[k]).to(dev) for k in range(w.n_frames)]


def ref_solve(w, depth, normal, corr=None):
    return oracle.ref_optimize_frames([d.data_ptr() for d in depth], [n.data_ptr() for n in normal], w.H, w.W, w.K, w.corr if corr is None else corr, w.poses_init)


# ---- solver windows
if "solver" in parts:
    save = {}
    for name, (seed, N, C, occ) in {"w0": (0, 10, 2000, False), "w40": (40, 6, 1200, False), "cfg3": (63, 30, 3000, True)}.items():
        w = synth.make_window(seed, n_frames=N, n_corr=C, occlusion=occ)
        d, n = upload(w)
        ref, pairs, _, _ = ref_solve(w, d, n)
        save[f"{name}_poses"] = ref[:, :3, :].astype(np.float32)
        save[f"{name}_pairs"] = pairs.astype(np.uint32)
    sweep_poses, sweep_pairs, sweep_np, jitter = [], [], [], []
    for seed in range(200):
        N = 3 + seed % 6
        w = synth.make_window(5000 + seed, n_frames=N, n_corr=200 * N)
        d, n = upload(w)
        ref, pairs, _, _ = ref_solve(w, d, n)
        ref2 = ref_solve(w, d, n)[0]
        sweep_poses.append(ref[:, :3, :]); sweep_pairs.append(pairs); sweep_np.append(len(pairs))
        jitter.append(max(synth.pose_errors(ref2, ref)))
    sweep_poses = np.concatenate(sweep_poses).astype(np.float64)      # the sweep's rotations as rotation vectors: half the bytes, ~1e-7 rad
    save.update(sweep_rotvec=Rotation.from_matrix(sweep_poses[:, :3, :3]).as_rotvec().astype(np.float32), sweep_t=sweep_poses[:, :3, 3].astype(np.float32), sweep_pairs=np.concatenate(sweep_pairs).astype(np.uint32),
                sweep_n_pairs=np.asarray(sweep_np, np.int32), sweep_jitter=np.asarray(jitter, np.float32))
    np.savez_compressed(os.path.join(out_dir, "ref_live_solver.npz"), **save)
    print("solver: sweep run-to-run max", max(jitter))

# ---- frame front end
if "frame" in parts:
    from test_frontend_gpu import frame_encode
    raw, K = synth.make_raw_depth(7, 480, 640)
    rd, rx, rn, _ = oracle.ref_frame_preprocess(raw, K)
    np.savez_compressed(os.path.join(out_dir, "ref_live_frame.npz"), **frame_encode(raw, K, rd, rx, rn))

# ---- RANSAC
if "ransac" in parts:
    masks, sizes = [], []
    groups = [((8, 0.005), [synth.make_ransac_case(7000 + 10 * 8 + k, 8, 0.5 + 0.1 * k) for k in range(3)])]
    for n, thresh in ((60, 0.005), (300, 0.01), (1000, 0.005), (3000, 0.005)):
        groups.append(((n, thresh), [synth.make_ransac_case(7000 + 10 * n + k, n, 0.5 + 0.1 * k) for k in range(3)]))
    rng = np.random.default_rng(5)
    groups.append(((None, 0.005), [synth.make_ransac_case(8000 + p, int(rng.integers(300, 1600)), float(rng.uniform(0.3, 0.9))) for p in range(45)]))
    for (_, thresh), cases in groups:
        ref, _ = oracle.ref_ransac_pairs([c[0] for c in cases], [c[1] for c in cases], 2000, thresh)
        for c, ids in zip(cases, ref):
            m = np.zeros(len(c[0]), bool); m[ids] = True
            masks.append(m); sizes.append(len(m))
    np.savez_compressed(os.path.join(out_dir, "ref_live_ransac.npz"), bits=np.packbits(np.concatenate(masks)), sizes=np.asarray(sizes, np.int32))

# ---- the fused matcher chain's EntryJ list, handed to the reference's solver
if "fused" in parts:
    from test_matcher_gpu import FUSED_YML, _feature_window  # noqa: E402
    from bundletrack_b200.matcher import MatchPipeline  # noqa: E402
    w, host, devf = _feature_window(5, 4, 500, dev)
    mp = MatchPipeline(FUSED_YML, max_pairs=8, max_feats=512)
    ent, n_ent, off = mp.match_pairs([(devf[a], devf[b]) for a, b in [(j, i) for i in range(4) for j in range(i + 1, 4)]], w.H, w.W, w.K)
    mp.close()
    depth = [f["depth"] for f in devf]; normal = [f["normal"] for f in devf]
    ref_same, pairs, _, _ = ref_solve(w, depth, normal, corr=ent)
    ref_again = ref_solve(w, depth, normal, corr=ent)[0]
    np.savez_compressed(os.path.join(out_dir, "ref_live_fused.npz"), ent=np.ascontiguousarray(ent).view(np.uint8).reshape(-1, 32), poses=ref_same.astype(np.float32),
                        pairs=pairs.astype(np.uint32), poses_again=ref_again.astype(np.float32))
    print("wrote", sorted((f, os.path.getsize(os.path.join(out_dir, f))) for f in os.listdir(out_dir) if f.startswith("ref_live_")))
