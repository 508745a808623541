#!/usr/bin/env python
"""Where one flagship step's device time goes: bench.py's `value` loop (32 windows x 10 keyframes x 2000 correspondences; per step one
new frame per window is stored into the frame cache, then pose prep + k_solve) under torch.profiler with CUDA activities, in a run of
its own.  Prints, for each steady-state step, its kernels and copies in stream order with their durations and the gap to the previous
one (negative: the two overlapped), the step's device time outside k_solve, and the summary over the steps.

The tail phase (last dense tile's end -> k_solve's end: only the windows' last-iteration tails run) comes from the solver's phase
records (bt_solve_enable_profile) of one extra step.  Their stamps are only comparable across SMs in a build with -DBT_PROF_GLOBALTIMER
(scripts/build_variant.sh gtimer bundletrack_b200/csrc/solver.cu -DBT_PROF_GLOBALTIMER, then BT_B200_LIB=... --globaltimer); without it
the script reports the longest last-iteration tail, each measured on its own SM, in SM cycles.

    python scripts/bench_step_timeline.py [--steps 20] [--warmup 10] [--timing 1] [--globaltimer] [--json OUT.json]
"""
from __future__ import annotations

import argparse
import json
import os
import tempfile

import numpy as np

import benchkit


def short(name: str) -> str:
    if name.startswith("Memcpy") or name.startswith("Memset"):
        return name.split(" (")[0]
    n = name.split("(")[0].replace("void ", "")
    return n.split("::")[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--timing", type=int, default=1, help="bt_solve_enable_timing as bench.py runs the value loop (1) or off (0)")
    ap.add_argument("--globaltimer", action="store_true", help="the loaded library was built with -DBT_PROF_GLOBALTIMER")
    ap.add_argument("--json", default=None, help="also write the per-step table and the summary here")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    from bundletrack_b200.optimizer import OptimizerGpu, SolveWindow

    assert torch.cuda.is_available(), "bench_step_timeline.py needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    bargs = argparse.Namespace(windows=32, frames=10, corr=2000, scenes=4)
    wins, _ = bench.make_batch(bargs, 0, dev)
    N = bargs.frames
    stream = torch.cuda.current_stream().cuda_stream
    opt = OptimizerGpu(None, device=0, max_windows=len(wins), max_frames=N, max_corr=bargs.corr, stream=stream)
    opt.enable_timing(bool(args.timing))
    nF = len(wins) * N
    opt.reserve_frame_cache(nF, wins[0].H, wins[0].W)
    slots = list(range(nF))
    opt.store_frames(slots, [d for w in wins for d in w.depths], [n_ for w in wins for n_ in w.normals], wins[0].H, wins[0].W, wins[0].K)
    cwins = [SolveWindow(w.corr, w.H, w.W, None, None, w.poses, w.K, cache_slots=slots[i * N:(i + 1) * N], corr_block_n=w.corr_block_n) for i, w in enumerate(wins)]
    new_slots = [i * N + (N - 1) for i in range(len(wins))]
    store_args = opt.prepare_store(new_slots, [w.depths[N - 1] for w in wins], [w.normals[N - 1] for w in wins], wins[0].H, wins[0].W, wins[0].K)
    opt.stage(cwins)

    def step():
        opt.store_prepared(store_args)
        opt.run()

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps + 1):
            step()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    ops = sorted(({"name": short(e["name"]), "ts": float(e["ts"]), "dur": float(e.get("dur", 0.0))} for e in trace["traceEvents"]
                  if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")), key=lambda o: o["ts"])
    solves = [k for k, o in enumerate(ops) if o["name"].startswith("k_solve")]
    if len(solves) < 2:
        raise SystemExit(f"expected {args.steps + 1} k_solve launches in the trace, found {len(solves)}")
    rows, outside, period, solve_dur = [], [], [], []
    for s in range(1, len(solves)):      # step s: everything after k_solve s-1 up to and including k_solve s
        prev = ops[solves[s - 1]]
        t0 = prev["ts"] + prev["dur"]
        end_prev = t0
        print(f"step {s}:  (t = 0 at the previous k_solve's end)")
        print(f"  {'op':28s} {'start us':>9s} {'dur us':>9s} {'gap us':>9s}")
        step_rows = []
        for o in ops[solves[s - 1] + 1:solves[s] + 1]:
            gap = o["ts"] - end_prev
            print(f"  {o['name']:28s} {o['ts'] - t0:9.2f} {o['dur']:9.2f} {gap:9.2f}")
            step_rows.append({"op": o["name"], "start_us": o["ts"] - t0, "dur_us": o["dur"], "gap_us": gap})
            end_prev = max(end_prev, o["ts"] + o["dur"])
        cur = ops[solves[s]]
        p = cur["ts"] + cur["dur"] - t0
        period.append(p); solve_dur.append(cur["dur"]); outside.append(p - cur["dur"])
        print(f"  step {p:.2f} us, k_solve {cur['dur']:.2f} us, outside k_solve {p - cur['dur']:.2f} us")
        rows.append(step_rows)
    names = [r["op"] for r in rows[-1]]
    summ = {"steps": len(period), "timing": bool(args.timing), "step_us_median": float(np.median(period)), "k_solve_us_median": float(np.median(solve_dur)),
            "outside_k_solve_us_median": float(np.median(outside)), "outside_k_solve_us_min_max": [float(np.min(outside)), float(np.max(outside))],
            "per_op_median": {}}
    for j, n in enumerate(names):
        col = [r[j] for r in rows if len(r) == len(names) and r[j]["op"] == n]
        summ["per_op_median"][f"{j}:{n}"] = {"dur_us": float(np.median([c["dur_us"] for c in col])), "gap_us": float(np.median([c["gap_us"] for c in col]))}

    # ---- tail phase of one more step, from the solver's phase records
    opt.enable_profile(400000)
    step()
    torch.cuda.synchronize()
    rec = opt.get_profile()
    kind = rec[:, 0] >> 32
    tiles, tails = rec[kind == 0], rec[kind == 1]
    last_it = int((tails[:, 1] >> 32).max())
    lt = tails[(tails[:, 1] >> 32) == last_it]
    if args.globaltimer:
        tail = {"unit": "us", "last_tile_end_to_last_tail_end": float(tails[:, 10].max() - tiles[:, 6].max()) / 1e3,
                "last_iteration_tail_max": float((lt[:, 10] - lt[:, 2]).max()) / 1e3, "last_iteration_tail_median": float(np.median(lt[:, 10] - lt[:, 2])) / 1e3}
    else:
        tail = {"unit": "SM cycles", "last_iteration_tail_max": int((lt[:, 10] - lt[:, 2]).max()), "last_iteration_tail_median": float(np.median(lt[:, 10] - lt[:, 2]))}
    tail["last_iteration_windows"] = int(len(lt))
    summ["tail"] = tail
    opt.close()
    summ["device"] = torch.cuda.get_device_name(dev)
    summ["card"] = benchkit.card()
    print(json.dumps(summ, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"summary": summ, "steps": rows}, f, indent=1)


if __name__ == "__main__":
    main()
