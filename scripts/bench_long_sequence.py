"""A whole sequence through the tracker with a keyframe pool (bt_tracker_params::max_keyframes): 640x480, 2000 features per frame, NOCS config in
largest-hull mode, max_frames_alive = 8 and max_keyframes = 256 by default.  Reports

  - begin_frame / end_frame wall time (median, p90) per 100-frame bucket next to the keyframes alive, so a step cost that grows with the pool shows;
  - the device memory bt_tracker_create reserved (cudaMemGetInfo before and after);
  - at the end the map points alive, the cached pairs and the entries they hold (bt_tracker_usage);
  - the frame at which the tracker without a pool (max_frames_alive = 64, max_keyframes = 0) returns BT_ERR_CAPACITY;
  - the host loops that grow with the keyframes, at the end's keyframe count: the keyframe-pose array, bt_select_keyframes and
    bt_match_cache_forget_frame's scan over the cached pairs;
  - kernel time per frame for the last frames of the sequence from torch.profiler, in a run of its own.

    python scripts/bench_long_sequence.py [--frames 600] [--feats 2000] [--keyframes 256] [--out results.json]

Needs an sm_90 GPU; there is no CPU path.  Prints one JSON line, and writes it to --out when that is given."""
from __future__ import annotations

import argparse
import ctypes
import itertools
import json
import os
import time

import numpy as np

import benchkit
from bench_tracker import stats_ms, upload


def feed(trk, frames, seq, lo, hi, tb=None, te=None):
    """Frames [lo, hi) through a Tracker, each call timed up to the end of its device work: tb gets begin_frame's time per frame, te
    (frame, end_frame's time, keyframes after it) per frame that reached end_frame.  Returns the frame of a BT_ERR_CAPACITY, or None."""
    import torch
    from bundletrack_b200 import _lib
    rq = torch.zeros((400, 400, 3), dtype=torch.uint8, device="cuda")
    for k in range(lo, hi):
        d, m, c, kp, desc = frames[k]
        t0 = time.perf_counter()
        st, _ = trk.begin_frame(d, m, c, rq, first_pose=seq.poses_gt[k])
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        if tb is not None:
            tb.append(t1 - t0)
        if st != _lib.BT_FRAME_OTHER:
            continue
        if kp is None:
            trk.drop_frame()
            continue
        try:
            trk.end_frame(kp, desc)
        except _lib.BtError as e:
            if "status -2:" in str(e):
                return k
            raise
        torch.cuda.synchronize()
        if te is not None:
            te.append((k, time.perf_counter() - t1, int(trk.state()[2].sum())))
    return None


def host_loops(n_kf, n_pairs, max_ba, reps=200):
    """Microseconds per call of the host work that grows with the keyframes, at n_kf keyframes and n_pairs cached pairs."""
    from bundletrack_b200 import _lib, synth
    lib = _lib.load()
    rng = np.random.default_rng(0)
    poses = np.stack([synth.se3(synth.so3_exp(rng.normal(size=3)), rng.normal(size=3) * 0.01) for _ in range(n_kf)]).astype(np.float32)
    pose_of = {k: poses[k].reshape(16).copy() for k in range(n_kf)}
    t0 = time.perf_counter()
    for _ in range(reps):
        kp = np.empty((n_kf, 16), np.float32)
        for k in range(n_kf):
            kp[k] = pose_of[k]
    t_arr = (time.perf_counter() - t0) / reps * 1e6
    chosen, n_chosen = np.zeros(n_kf, np.int32), ctypes.c_int(0)
    new = poses[-1].copy()
    t0 = time.perf_counter()
    for _ in range(reps):
        _lib.check(lib.bt_select_keyframes(new.ctypes.data_as(ctypes.c_void_p), poses.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(n_kf), ctypes.c_int(max_ba),
                                           chosen.ctypes.data_as(ctypes.c_void_p), ctypes.byref(n_chosen)), "bt_select_keyframes")
    t_sel = (time.perf_counter() - t0) / reps * 1e6
    ctx = ctypes.c_void_p()
    _lib.check(lib.bt_ctx_create(ctypes.byref(ctx), 0), "bt_ctx_create")
    _lib.check(lib.bt_match_cache_reserve_entries(ctx, ctypes.c_int(max(n_pairs, 1)), ctypes.c_longlong(1)), "bt_match_cache_reserve_entries")
    ids = list(itertools.islice(((a, b) for a in range(1, 1 << 20) for b in range(max(0, a - 14), a)), n_pairs))
    for a, b in ids:                                # empty blocks: only the host record matters for the scan
        z = np.zeros(1, np.int32)
        _lib.check(lib.bt_match_cache_put(ctx, 1, (ctypes.c_int32 * 1)(a), (ctypes.c_int32 * 1)(b), None, z.ctypes.data_as(ctypes.c_void_p),
                                          z.ctypes.data_as(ctypes.c_void_p), None, None), "bt_match_cache_put")
    t0 = time.perf_counter()
    for _ in range(reps):
        _lib.check(lib.bt_match_cache_forget_frame(ctx, ctypes.c_int(-5)), "bt_match_cache_forget_frame")     # a frame with no pair: a full scan
    t_fgt = (time.perf_counter() - t0) / reps * 1e6
    lib.bt_ctx_destroy(ctx)
    return {"keyframes": n_kf, "cached_pairs": n_pairs, "keyframe_pose_array_us": round(t_arr, 2), "select_keyframes_us": round(t_sel, 2),
            "match_cache_forget_scan_us": round(t_fgt, 2), "note": "the pose array is timed as a Python loop; the library builds it in C++"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=600)
    ap.add_argument("--feats", type=int, default=2000)
    ap.add_argument("--alive", type=int, default=8)
    ap.add_argument("--keyframes", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--profile-frames", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from bundletrack_b200 import _lib, synth
    from bundletrack_b200.config import load_yml
    from bundletrack_b200.tracker import Tracker
    assert torch.cuda.is_available(), "bench_long_sequence needs an sm_90 GPU"
    H, W = 480, 640
    mode = _lib.BT_MASK_LARGEST_HULL
    y = load_yml(None)
    res = {"gpu": benchkit.card(), "H": H, "W": W, "feats": a.feats, "frames": a.frames, "max_frames_alive": a.alive, "max_keyframes": a.keyframes}
    t0 = time.perf_counter()
    seq = synth.make_sequence(11, a.frames, H=H, W=W, n_feats=a.feats)
    res["generate_s"] = round(time.perf_counter() - t0, 1)
    frames = upload(seq, torch.device("cuda", 0))
    warm = synth.make_sequence(12, a.warmup, H=H, W=W, n_feats=a.feats)
    warm_frames = upload(warm, torch.device("cuda", 0))
    t = Tracker(y, H, W, seq.K, a.feats, a.alive, mode=mode, max_keyframes=a.keyframes)
    feed(t, warm_frames, warm, 0, a.warmup)
    t.close()
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    t = Tracker(y, H, W, seq.K, a.feats, a.alive, mode=mode, max_keyframes=a.keyframes)
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    res["create_reserved_gb"] = round((free0 - free1) / 1e9, 3)
    tb, te = [], []
    cap = feed(t, frames, seq, 0, a.frames, tb, te)
    assert cap is None, f"the pool tracker returned BT_ERR_CAPACITY at frame {cap}"
    ids, _, is_kf = t.state()
    pts, pairs, ents = t.usage()
    t.close()
    res["end"] = {"keyframes": int(is_kf.sum()), "frames_alive": len(ids), "points_alive": pts, "cached_pairs": pairs, "cached_entries": ents,
                  "cached_entries_per_pair": round(ents / max(pairs, 1), 1),
                  "cache_budget_entries": (a.alive + a.keyframes) * int(y["bundle"]["max_BA_frames"]) * 3 * a.feats // 2}
    # per 100-frame bucket of processed frames (end_frame was reached); begin_frame over every frame of the bucket
    buckets = []
    for lo in range(0, a.frames, 100):
        sel = [r for r in te if lo <= r[0] < lo + 100]
        buckets.append({"frames": f"{lo}-{min(lo + 100, a.frames) - 1}", "begin_ms": stats_ms(tb[lo:lo + 100]),
                        "end_ms": stats_ms([r[1] for r in sel]) if sel else None, "keyframes_at_end": sel[-1][2] if sel else None})
    res["buckets"] = buckets
    # the tracker without a keyframe pool on the same sequence
    t = Tracker(y, H, W, seq.K, a.feats, 64, mode=mode)
    res["no_pool_capacity_at_frame"] = feed(t, frames, seq, 0, a.frames)
    t.close()
    res["host_loops"] = host_loops(int(is_kf.sum()), pairs, int(y["bundle"]["max_BA_frames"]))
    # kernel time over the last frames, in a run of its own
    t = Tracker(y, H, W, seq.K, a.feats, a.alive, mode=mode, max_keyframes=a.keyframes)
    n = min(a.profile_frames, a.frames)
    feed(t, frames, seq, 0, a.frames - n)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        feed(t, frames, seq, a.frames - n, a.frames)
    t.close()
    kern = {}
    for e in prof.key_averages():
        dt = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if dt > 0 and ("k_" in e.key or "void" in e.key):
            kern[e.key[:80]] = {"calls": e.count, "us_per_frame": round(dt / n, 1)}
    res["profile"] = {"frames": f"{a.frames - n}-{a.frames - 1}", "kernel_us_per_frame": round(sum(v["us_per_frame"] for v in kern.values()), 1),
                      "kernels": dict(sorted(kern.items(), key=lambda kv: -kv[1]["us_per_frame"])[:15])}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
