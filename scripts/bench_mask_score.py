#!/usr/bin/env python3
"""Cost of scoring object masks against ground truth (bundletrack_b200.metrics.MaskScore, DESIGN.md §3.16): bt_mask_metrics of synthetic
sequences of moving ragged ellipses (synth.ragged_ellipse_masks), already on the device, at the default bound_th 0.008:

    480 x 640      1000 frames (r = 7), the YCBInEOAT and NOCS frame size
    1080 x 1920     300 frames (r = 18)

and bt_mask_metrics_objects (MaskScore.objects, DESIGN.md §3.17) of DAVIS-style label maps (synth.ragged_label_maps, a void band in
every ground-truth frame):

    480 x 854       90 frames (r = 8) of 1, 3 and 7 objects, DAVIS's 480p size, with void_value -1 (eval_masks.py --davis: no void
                    mask, as the toolkit's semi-supervised path) and with void_value 255 (void removed from both masks)

Each sequence is scored in one call, timed with CUDA events on the facade's stream over --reps calls after a warm-up call.  Prints device
ms per frame and the input read rate (both masks' bytes over the call's time) as a fraction of the H100 SXM data sheet's 3.35 TB/s, with
the card's name and power limit, then one JSON line.  A label-map call packs each frame's two maps once per object, and with a void value
it also reads the ground truth a second time per object to take void out of the prediction (the arrays here are equally aligned, so one
ground-truth block per prediction block): 2 or 3 map bytes per pixel and object.

    python scripts/bench_mask_score.py [--reps 10] [--out_json path]
"""
from __future__ import annotations

import argparse
import json

import numpy as np

import benchkit

HBM_BYTES_PER_S = 3.35e12
SEQUENCES = [(1000, 480, 640), (300, 1080, 1920)]
OBJECT_SEQUENCES = [(90, 480, 854, k, void) for void in (-1, 255) for k in (1, 3, 7)]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out_json", default=None)
    a = ap.parse_args()
    import torch
    from bundletrack_b200 import synth
    from bundletrack_b200.metrics import MaskScore, mask_score
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    name = benchkit.card()
    print(f"card: {name}")
    res = {"card": name, "bound_th": 0.008, "sequences": {}}
    for n, h, w in SEQUENCES:
        pred, gt = synth.ragged_ellipse_masks(n, h, w, seed=0)
        dev = torch.device("cuda", 0)
        p, g = torch.from_numpy(pred).to(dev), torch.from_numpy(gt).to(dev)
        ms = MaskScore(n, h, w)
        j = torch.empty(n, dtype=torch.float64, device=dev)
        f = torch.empty(n, dtype=torch.float64, device=dev)

        def call():
            rc = ms.lib.bt_mask_metrics(ms.ctx, p.data_ptr(), g.data_ptr(), n, h, w, 0.008, j.data_ptr(), f.data_ptr(), None, ms.stream)
            assert rc == 0, rc

        t = [ms_ * 1e-3 for ms_ in benchkit.calls_ms(call, a.reps, 1, ms.stream)]
        t_med = float(np.median(t))
        rate = 2.0 * n * h * w / t_med
        score = mask_score(j.cpu().numpy(), f.cpu().numpy())
        ms.close()
        key = f"{h}x{w}"
        res["sequences"][key] = {"frames": n, "call_s": t_med, "call_all_s": t, "ms_per_frame": t_med * 1e3 / n, "input_bytes_per_s": rate,
                                 "fraction_of_3.35TBps": rate / HBM_BYTES_PER_S, "J-Mean": score["J-Mean"], "F-Mean": score["F-Mean"]}
        print(f"{n} frames of {h} x {w}: {t_med * 1e3:.3f} ms per call, {t_med * 1e3 / n:.4f} ms per frame, input {rate / 1e12:.3f} TB/s "
              f"({100 * rate / HBM_BYTES_PER_S:.1f} % of 3.35 TB/s); J-Mean {score['J-Mean']:.4f}, F-Mean {score['F-Mean']:.4f}")
    res["objects"] = {}
    maps = {}
    for n, h, w, k, void in OBJECT_SEQUENCES:
        if (n, h, w, k) not in maps:
            maps[(n, h, w, k)] = synth.ragged_label_maps(n, h, w, k, void_from=0, seed=k)
        pred, gt = maps[(n, h, w, k)]
        dev = torch.device("cuda", 0)
        p, g = torch.from_numpy(pred).to(dev), torch.from_numpy(gt).to(dev)
        ms = MaskScore(n * k, h, w)
        j = torch.empty((n, k), dtype=torch.float64, device=dev)
        f = torch.empty((n, k), dtype=torch.float64, device=dev)

        def call():
            rc = ms.lib.bt_mask_metrics_objects(ms.ctx, p.data_ptr(), g.data_ptr(), n, h, w, k, void, 0.008, j.data_ptr(), f.data_ptr(), None,
                                                ms.stream)
            assert rc == 0, rc

        t = [ms_ * 1e-3 for ms_ in benchkit.calls_ms(call, a.reps, 1, ms.stream)]
        t_med = float(np.median(t))
        rate = (2.0 if void < 0 else 3.0) * n * k * h * w / t_med
        jm, fm = float(j.mean().item()), float(f.mean().item())
        ms.close()
        key = f"{h}x{w}x{k}_void{void}"
        res["objects"][key] = {"frames": n, "objects": k, "void_value": void, "call_s": t_med, "call_all_s": t, "ms_per_frame": t_med * 1e3 / n,
                               "ms_per_frame_object": t_med * 1e3 / (n * k), "input_bytes_per_s": rate,
                               "fraction_of_3.35TBps": rate / HBM_BYTES_PER_S, "J-Mean": jm, "F-Mean": fm}
        print(f"{n} frames of {h} x {w}, {k} objects, void_value {void}: {t_med * 1e3:.3f} ms per call, {t_med * 1e3 / n:.4f} ms per frame, "
              f"{t_med * 1e3 / (n * k):.4f} ms per frame and object, input {rate / 1e12:.3f} TB/s ({100 * rate / HBM_BYTES_PER_S:.1f} % of "
              f"3.35 TB/s); mean J {jm:.4f}, mean F {fm:.4f}")
    line = json.dumps(res)
    print(line)
    if a.out_json:
        with open(a.out_json, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
