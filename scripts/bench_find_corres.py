"""Per-frame cost of SiftManager::findCorres for a new frame against a 10- and a 15-frame window (2000 features per frame, descriptors in
the pool), two ways:
  (a) pair by pair, as a caller had to do with the host map-point table: per pair bt_tracks_propagate on the host -> bt_match_pairs_ex
      (n_pairs = 1) -> read back counts and the emitted (uA, vA, uB, vB) -> bt_tracks_update_pair on the host;
  (b) one bt_find_corres_pairs call on the device table, then one read-back of the counts.
Reports the wall time per new frame up to the final read-back (median over repeated frames after warm-up), the kernel time per frame from
a separate torch.profiler run, and the card's name and power limit.  Both paths must produce the same entries.

    python scripts/bench_find_corres.py [--reps 30] [--warmup 5] [--out result.json]
"""
import argparse
import ctypes
import json
import os
import statistics
import time

import numpy as np

import benchkit
from bundletrack_b200 import _lib, synth
from bundletrack_b200.matcher import MatchPipeline, DeviceTracks
from bundletrack_b200.policy import Tracks

NF = 2000
YML = {"feature_corres": {"max_dist_no_neighbor": 0.02, "max_normal_no_neighbor": 45, "max_dist_neighbor": 10000, "max_normal_neighbor": 180},
       "ransac": {"max_iter": 2000, "inlier_dist": 0.01}}


class Setup:
    def __init__(self, window, dev):
        import torch
        self.N = window + 1
        self.w = synth.make_window(11, n_frames=self.N, n_corr=10)
        fr = synth.make_feature_frames(self.w, NF, seed=11)
        self.f = [{"kpts": torch.from_numpy(fr[k]["kpts"]).to(dev), "depth": torch.from_numpy(self.w.depth[k]).to(dev),
                   "normal": torch.from_numpy(self.w.normal[k]).to(dev), "pose": self.w.poses_init[k], "id": k, "window_index": k} for k in range(self.N)]
        self.mp = MatchPipeline(YML, max_pairs=16, max_feats=2048)
        self.mp.pool_reserve(self.N)
        for k in range(self.N):
            self.mp.pool_store(k, torch.from_numpy(fr[k]["desc"]).to(dev))
        self.dt = DeviceTracks(ctx=self.mp.ctx, max_frames=self.N + 2, max_keys_per_frame=2048)
        self.ht = Tracks()
        self.dev = dev

    @staticmethod
    def pairs(f):
        return [(f, f - 1)] + [(f, j) for j in range(0, f - 1)]      # neighbour first, then the older frames oldest first (Bundler.cpp:298-305)

    def tail(self):
        mp, w = self.mp, self.w
        return (ctypes.c_int(w.H), ctypes.c_int(w.W), ctypes.c_float(w.K[0]), ctypes.c_float(w.K[1]), ctypes.c_float(w.K[2]), ctypes.c_float(w.K[3]),
                ctypes.byref(mp.prune), ctypes.c_int(mp.ransac_trials), ctypes.c_float(mp.ransac_inlier_dist), ctypes.c_uint64(0))

    def path_a(self, f):
        """One bt_match_pairs_ex call per pair with the host table; returns the entries of the frame's pairs."""
        import torch
        lib, mp, out = self.mp.lib, self.mp, []
        for a, b in self.pairs(f):
            A, B, _, _ = mp._views([(self.f[a], self.f[b])])
            extra = (_lib.MatchExtra * 1)()
            prop = np.zeros((0, 4), np.float32)
            if a - b != 1:
                prop = np.ascontiguousarray(self.ht.propagate(a, b, prop), np.float32)
                extra[0].uv, extra[0].n = (prop.ctypes.data if len(prop) else None), len(prop)
            cap = 2 * NF + len(prop)
            ent = torch.empty((cap, 8), dtype=torch.int32, device=self.dev); uvo = torch.empty((cap, 4), dtype=torch.float32, device=self.dev)
            meta = torch.empty((3, 1), dtype=torch.int32, device=self.dev); tot = torch.empty(4, dtype=torch.int32, device=self.dev)
            _lib.check(lib.bt_match_pairs_ex(mp.ctx, ctypes.c_int(1), A, B, None, None, (ctypes.c_int32 * 1)(a), (ctypes.c_int32 * 1)(b), *self.tail(), extra,
                                             ctypes.c_void_p(ent.data_ptr()), ctypes.c_int(cap), ctypes.c_void_p(meta[0].data_ptr()), ctypes.c_void_p(meta[1].data_ptr()),
                                             ctypes.c_void_p(tot.data_ptr()), ctypes.c_void_p(meta[2].data_ptr()), ctypes.c_void_p(uvo.data_ptr()), mp.stream), "bt_match_pairs_ex")
            n = int(meta[0, 0].item())
            if n:
                self.ht.update_pair(a, b, uvo[:n].cpu().numpy())
            out.append(ent[:n])
        return out

    def path_b(self, f):
        import torch
        lib, mp = self.mp.lib, self.mp
        prs = self.pairs(f)
        n = len(prs)
        A, B, _, _ = mp._views([(self.f[a], self.f[b]) for a, b in prs])
        cap = n * (2 * NF + mp.max_feats)
        ent = torch.empty((cap, 8), dtype=torch.int32, device=self.dev)
        meta = torch.empty((3, n), dtype=torch.int32, device=self.dev); tot = torch.empty(4, dtype=torch.int32, device=self.dev)
        _lib.check(lib.bt_find_corres_pairs(mp.ctx, ctypes.c_int(n), A, B, None, None, (ctypes.c_int32 * n)(*[a for a, _ in prs]), (ctypes.c_int32 * n)(*[b for _, b in prs]),
                                            *self.tail(), ctypes.c_void_p(ent.data_ptr()), ctypes.c_int(cap), ctypes.c_void_p(meta[0].data_ptr()),
                                            ctypes.c_void_p(meta[1].data_ptr()), ctypes.c_void_p(tot.data_ptr()), ctypes.c_void_p(meta[2].data_ptr()), None, mp.stream),
                   "bt_find_corres_pairs")
        m = meta.cpu().numpy()             # the one read-back
        return [ent[int(m[1, p]):int(m[1, p]) + int(m[0, p])] for p in range(n)]

    def forget(self, f, which):
        (self.ht if which == "a" else self.dt).forget_frame(f)


def run(window, reps, warmup, dev):
    import torch
    from torch.profiler import profile, ProfilerActivity
    s = Setup(window, dev)
    new = s.N - 1
    for f in range(1, new):         # the window's history: both tables hold the same map points
        s.path_a(f); s.path_b(f)
    ea, eb = s.path_a(new), s.path_b(new)
    same = len(ea) == len(eb) and all(torch.equal(x, y) for x, y in zip(ea, eb))
    n_entries = int(sum(x.shape[0] for x in eb))
    s.forget(new, "a"); s.forget(new, "b")
    res = {}
    for which, fn in (("a", s.path_a), ("b", s.path_b)):
        t = []
        for r in range(warmup + reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn(new)                       # ends with its read-back
            t1 = time.perf_counter()
            s.forget(new, which)          # (not timed) drops the new frame's map and observations, but the points its pairs created stay in
                                          # the older frames' maps: the table is not restored.  It grows mostly in the first repetition (later
                                          # ones find most of those keys), the same way for both paths
            if r >= warmup:
                t.append((t1 - t0) * 1e3)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                fn(new); s.forget(new, which)
            torch.cuda.synchronize()
        kern = [e for e in prof.key_averages() if e.device_type is not None and str(e.device_type).endswith("CUDA") and e.count > 0]
        dev_us = sum(getattr(e, "self_device_time_total", getattr(e, "self_cuda_time_total", 0.0)) for e in kern) / 5.0
        top = sorted(kern, key=lambda e: -getattr(e, "self_device_time_total", getattr(e, "self_cuda_time_total", 0.0)))[:6]
        res[which] = {"wall_ms_median": statistics.median(t), "wall_ms_min": min(t), "wall_ms_max": max(t), "device_ms_per_frame": dev_us / 1e3,
                      "top_kernels_us_per_frame": {e.key: getattr(e, "self_device_time_total", getattr(e, "self_cuda_time_total", 0.0)) / 5.0 for e in top}}
    return {"window": window, "pairs": window, "features_per_frame": NF, "entries": n_entries, "identical_entries": bool(same),
            "a_pair_by_pair_host_table": res["a"], "b_one_call_device_table": res["b"],
            "speedup_wall": res["a"]["wall_ms_median"] / res["b"]["wall_ms_median"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--windows", type=int, nargs="+", default=[10, 15])
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_find_corres needs a GPU"
    dev = torch.device("cuda:0")
    out = {"card": benchkit.card(), "rows": [run(w, a.reps, a.warmup, dev) for w in a.windows]}
    txt = json.dumps(out, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(txt)


if __name__ == "__main__":
    main()
