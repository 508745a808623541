"""Times the object-mask front end on the GPU (CUDA events and torch.profiler kernel times) and, as a host baseline, the reference's
OpenCV pipeline on the same masks on this machine's CPU.  Prints one JSON object (and writes it to --out if given).

    python scripts/bench_segment.py [--H 480 --W 640 --batches 1 32 --iters 50 --out FILE]

Rows, per frame: unmasked front end (bt_frames_preprocess), masked front end in as-is and largest-hull mode
(bt_frames_preprocess_masked), bt_lfnet_request; kernel times per name from torch.profiler; the CPU pipeline (components, hull, fill,
dilate, invalidate loop, ROI loop, crop and resize) when cv2 is importable, "not measured" otherwise.
"""
import argparse
import json
import os
import statistics
import time

import numpy as np

import benchkit


def cpu_pipeline(cv2, mask, mode, depth, normal, colour):
    m = mask.copy()
    if mode == 1:
        _, label = cv2.connectedComponents(m, connectivity=8)
        hist = np.bincount(label[m != 0].ravel())
        best = int(hist.argmax()) if hist.size else 0
        m = np.zeros_like(m)
        if hist.size and hist[best] > 0:
            ys, xs = np.nonzero(label == best)
            cv2.fillConvexPoly(m, cv2.convexHull(np.stack([xs, ys], 1).astype(np.int32)), 1)
    fg = cv2.dilate(m, cv2.getStructuringElement(cv2.MORPH_RECT, (5, 5)))
    bg = fg == 0
    depth[bg] = 0; normal[bg] = 0; colour[bg] = 0
    ys, xs = np.nonzero(fg)
    if len(xs) == 0:
        return
    umin, umax, vmin, vmax = xs.min(), xs.max(), ys.min(), ys.max()
    Wr, Hr = umax - umin, vmax - vmin
    if Wr < 10 or Hr < 10:
        return
    side = max(Wr, Hr)
    img = np.zeros((side, side, 3), np.uint8)
    img[:Hr, :Wr] = colour[vmin:vmin + Hr, umin:umin + Wr]
    cv2.resize(img, (400, 400))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--H", type=int, default=480)
    ap.add_argument("--W", type=int, default=640)
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 32])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from bundletrack_b200 import _lib, synth
    from bundletrack_b200.frontend import FrameFrontEnd
    from oracle import segment_oracle as so
    assert torch.cuda.is_available(), "bench_segment needs a GPU"
    dev = torch.device("cuda:0")
    H, W = args.H, args.W
    res = {"card": benchkit.card(), "H": H, "W": W, "rows": {}}
    fe = FrameFrontEnd()

    def time_events(fn):
        """ms per call: the median of three windows, the first after five warm-up calls."""
        return statistics.median(benchkit.window_ms(fn, args.iters, warmup, fe.stream) for warmup in (5, 0, 0))

    for B in args.batches:
        raws = [torch.from_numpy(synth.make_raw_depth(s % 8, H, W)[0]).to(dev) for s in range(B)]
        masks = [torch.from_numpy(synth.make_object_mask(s, H, W)).to(dev) for s in range(B)]
        cols = [torch.from_numpy(so.test_colour(H, W)).to(dev) for _ in range(B)]
        d = [torch.empty((H, W), device=dev) for _ in range(B)]
        nn = [torch.empty((H, W, 4), device=dev) for _ in range(B)]
        fg = [torch.empty((H, W), dtype=torch.uint8, device=dev) for _ in range(B)]
        req = [torch.empty((400, 400, 3), dtype=torch.uint8, device=dev) for _ in range(B)]
        K = synth.NOCS_K
        fns = {
            "frontend_unmasked": lambda: fe.process(raws, H, W, K, d, nn),
            "frontend_masked_as_is": lambda: fe.process_masked(raws, masks, H, W, K, d, nn, fg, mode=_lib.BT_MASK_AS_IS, fetch_roi=False),
            "frontend_masked_hull": lambda: fe.process_masked(raws, masks, H, W, K, d, nn, fg, mode=_lib.BT_MASK_LARGEST_HULL, fetch_roi=False),
        }
        row = {}
        for name, fn in fns.items():
            row[name + "_ms_per_frame"] = time_events(fn) / B
        fe.process_masked(raws, masks, H, W, K, d, nn, fg, mode=_lib.BT_MASK_LARGEST_HULL)
        row["lfnet_request_ms_per_frame"] = time_events(lambda: fe.lfnet_request(cols, fg, H, W, req)) / B
        # kernel times per name, from a profiled run of its own
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(10):
                for fn in fns.values():
                    fn()
                fe.lfnet_request(cols, fg, H, W, req)
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if ev.key.startswith(("bt::k_", "void bt::k_", "k_")) or "bt::" in ev.key:
                t = getattr(ev, "device_time_total", None)
                if t is None:
                    t = ev.cuda_time_total
                kern[ev.key.split("(")[0].replace("void ", "")] = t / 1000.0 / max(ev.count, 1) / B
        row["kernel_ms_per_frame"] = kern
        res["rows"][f"batch_{B}"] = row
        print(f"batch {B}: " + ", ".join(f"{k} {v:.4f}" for k, v in row.items() if not isinstance(v, dict)), flush=True)
        print("  kernels/frame (ms): " + ", ".join(f"{k} {v:.4f}" for k, v in sorted(kern.items())), flush=True)
    fe.close()
    try:
        import cv2
        cpu = {}
        depth = synth.make_raw_depth(0, H, W)[0]
        normal = np.zeros((H, W, 4), np.float32)
        colour = so.test_colour(H, W)
        for mode, name in ((0, "as_is"), (1, "hull")):
            ts = []
            for s in range(20):
                m = synth.make_object_mask(s, H, W)
                dd, nq, cc = depth.copy(), normal.copy(), colour.copy()
                t0 = time.perf_counter()
                cpu_pipeline(cv2, m, mode, dd, nq, cc)
                ts.append(time.perf_counter() - t0)
            cpu[f"cpu_opencv_{name}_ms_per_frame"] = float(np.median(ts) * 1e3)
        cpu["cv2_version"] = cv2.__version__
        cpu["cpu"] = os.cpu_count()
    except ImportError:
        cpu = {"cpu_opencv": "not measured (cv2 is not installed here)"}
    res["host_baseline"] = cpu
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
