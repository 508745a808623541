"""Per-frame cost of the whole tracking step (bt_tracker_*): begin_frame and end_frame wall time (median, p90) over a 640x480 sequence with
2000 features per frame in both mask modes, the same sequence through the Python composition of the public pieces (tests/test_tracker_gpu.py;
results must be identical), kernel time by kernel and the synchronising runtime calls per frame from torch.profiler in a separate run.

    python scripts/bench_tracker.py [--frames 100] [--feats 2000] [--out results.json]

Needs an sm_90 GPU; there is no CPU path.  Prints one JSON line, and writes it to --out when that is given."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

import benchkit

sys.path.insert(0, os.path.join(benchkit.ROOT, "tests"))

SYNC_CALLS = ("cudaStreamSynchronize", "cudaEventSynchronize", "cudaDeviceSynchronize", "cudaMemcpy")


def upload(seq, dev):
    import torch
    fr = []
    for k in range(seq.n_frames):
        d, m, c = (torch.from_numpy(np.ascontiguousarray(a[k])).to(dev) for a in (seq.depth_raw, seq.mask, seq.colour))
        f = seq.feats[k]
        fr.append((d, m, c, None if f is None else f["kpts"], None if f is None else torch.from_numpy(f["desc"]).to(dev)))
    torch.cuda.synchronize()
    return fr


def run(obj, frames, seq, timed=True):
    """Feeds a sequence to a Tracker or a Composition; returns (statuses, poses, begin times, end times) with the wall time of each call
    up to the end of its device work."""
    import torch
    from bundletrack_b200 import _lib
    dev = torch.device("cuda", 0)
    rq = torch.zeros((400, 400, 3), dtype=torch.uint8, device=dev)
    is_trk = hasattr(obj, "begin_frame")
    st_all, poses, tb, te = [], [], [], []
    for k, (d, m, c, kp, desc) in enumerate(frames):
        t0 = time.perf_counter()
        r = obj.begin_frame(d, m, c, rq, first_pose=seq.poses_gt[k]) if is_trk else obj.begin(d, m, c, rq, first_pose=seq.poses_gt[k])
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        st, pose = r[0], None
        if st == _lib.BT_FRAME_OTHER:
            pose, st = obj.end_frame(kp, desc) if is_trk else obj.end(kp, desc)
            torch.cuda.synchronize()
            te.append(time.perf_counter() - t1)
        tb.append(t1 - t0)
        st_all.append(st)
        poses.append(pose)
    return st_all, poses, tb, te


def stats_ms(v):
    v = np.asarray(v) * 1e3
    return {"median": round(float(np.median(v)), 3), "p90": round(float(np.percentile(v, 90)), 3), "n": len(v)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--feats", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=15)
    ap.add_argument("--profile-frames", type=int, default=30)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from bundletrack_b200 import _lib, synth
    from bundletrack_b200.config import load_yml
    from bundletrack_b200.tracker import Tracker
    from test_tracker_gpu import Composition
    assert torch.cuda.is_available(), "bench_tracker needs an sm_90 GPU"
    dev = torch.device("cuda", 0)
    H, W, F = 480, 640, 64
    res = {"gpu": benchkit.card(), "H": H, "W": W, "feats": a.feats, "frames": a.frames}
    seq = synth.make_sequence(11, a.frames, H=H, W=W, n_feats=a.feats)
    frames = upload(seq, dev)
    warm = synth.make_sequence(12, a.warmup, H=H, W=W, n_feats=a.feats)
    warm_frames = upload(warm, dev)
    y = load_yml(None)
    for mode, name in ((_lib.BT_MASK_LARGEST_HULL, "largest_hull"), (_lib.BT_MASK_AS_IS, "as_is")):
        t = Tracker(y, H, W, seq.K, a.feats, F, mode=mode)
        run(t, warm_frames, warm)
        t.close()
        t = Tracker(y, H, W, seq.K, a.feats, F, mode=mode)
        st_t, p_t, tb, te = run(t, frames, seq)
        n_kf = int(t.state()[2].sum())
        t.close()
        comp = Composition(y, seq.K, a.feats, F, mode, H=H, W=W)
        run(comp, warm_frames[:3], warm)
        comp.close()
        comp = Composition(y, seq.K, a.feats, F, mode, H=H, W=W)
        st_c, p_c, cb, ce = run(comp, frames, seq)
        n_nb = comp.n_neighbour
        comp.close()
        same = st_t == st_c and all((x is None and z is None) or (x is not None and z is not None and x.tobytes() == z.tobytes()) for x, z in zip(p_t, p_c))
        rot = [np.degrees(synth.rot_geodesic(p[:3, :3], seq.poses_gt[k][:3, :3])) for k, p in enumerate(p_t) if p is not None]
        trn = [float(np.linalg.norm(p[:3, 3] - seq.poses_gt[k][:3, 3])) for k, p in enumerate(p_t) if p is not None]
        res[name] = {"tracker_begin_ms": stats_ms(tb), "tracker_end_ms": stats_ms(te), "composition_begin_ms": stats_ms(cb), "composition_end_ms": stats_ms(ce),
                     "identical": bool(same), "statuses": {s: st_t.count(s) for s in (0, 1, 2)}, "keyframes": n_kf,
                     "neighbour_entries_median": int(np.median(n_nb)) if n_nb else 0,
                     "rot_err_deg": {"mean": round(float(np.mean(rot)), 3), "max": round(float(np.max(rot)), 3)},
                     "trans_err_mm": {"mean": round(float(np.mean(trn)) * 1e3, 3), "max": round(float(np.max(trn)) * 1e3, 3)}}
    # kernel time and synchronising calls, in a run of its own (largest-hull mode, the first frames of the sequence after a warm-up)
    t = Tracker(y, H, W, seq.K, a.feats, F, mode=_lib.BT_MASK_LARGEST_HULL)
    run(t, warm_frames, warm)
    t.close()
    t = Tracker(y, H, W, seq.K, a.feats, F, mode=_lib.BT_MASK_LARGEST_HULL)
    n = min(a.profile_frames, a.frames)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        run(t, frames[:n], seq)
    t.close()
    kern, calls = {}, {}
    for e in prof.key_averages():
        dt = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if e.key.startswith("k_") or "::k_" in e.key or ("void" in e.key and dt > 0):
            kern[e.key] = {"calls": e.count, "total_us": round(dt, 1), "avg_us": round(dt / max(e.count, 1), 2)}
        if e.key in SYNC_CALLS:
            calls[e.key] = round(e.count / n, 2)
    # torch.cuda.synchronize() in the timing harness adds one cudaDeviceSynchronize per call; they are not the tracker's
    res["profile"] = {"frames": n, "sync_calls_per_frame": calls, "harness_device_syncs_per_frame": 2,
                      "kernels": dict(sorted(kern.items(), key=lambda kv: -kv[1]["total_us"]))}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
