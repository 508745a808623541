#!/usr/bin/env python3
"""Per-frame wall time of bundletrack_b200.sequence.run_sequence on a synthetic NOCS scene (synth.make_sequence written as PNGs: 640 x 480,
2000 features per frame, the NOCS defaults, largest-hull masks, an in-process feature source), for three cases:

    prefetch 2      a worker thread decodes and uploads frames ahead of the tracker
    prefetch 0      decode and upload in line
    on device       the tracker alone over uint16 depth, masks and colour already on the device (begin_frame_mm / end_frame)

and, per frame, the host's PNG decode time and the front end on uint16 depth (bt_frames_preprocess_masked_u16) against the float front end
fed by the host's readDepthImage conversion and a float upload.  Prints the card's name and power limit with the numbers, then one JSON line.

    python scripts/bench_run_sequence.py [--frames 300] [--out_json path]
"""
from __future__ import annotations

import argparse
import json
import os
import tempfile
import time

import numpy as np

import benchkit


def stats(t):
    t = np.asarray(t) * 1000
    return {"median_ms": float(np.median(t)), "p90_ms": float(np.percentile(t, 90)), "mean_ms": float(np.mean(t))}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--feats", type=int, default=2000)
    ap.add_argument("--out_json", default=None)
    a = ap.parse_args()
    import torch
    from bundletrack_b200 import _lib, sequence, synth
    from bundletrack_b200.frontend import FrameFrontEnd
    from bundletrack_b200.tracker import Tracker
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    dev = torch.device("cuda", 0)
    H, W, N = 480, 640, a.frames
    t0 = time.perf_counter()
    seq = synth.make_sequence(7, N, H=H, W=W, n_feats=a.feats)
    print(f"sequence of {N} frames generated in {time.perf_counter() - t0:.1f} s", flush=True)

    features = synth.recorded_features(seq)
    mm = [synth.depth_mm(d) for d in seq.depth_raw]
    with tempfile.TemporaryDirectory() as tmp:
        nocs, masks = synth.write_nocs_scene(seq, tmp)
        loader = sequence.NocsScene(nocs, 1, "camera_bench_norm", masks)

        # host decode per frame
        dec = []
        for ff in loader.frames:
            t0 = time.perf_counter()
            sequence.read_frame(ff)
            dec.append(time.perf_counter() - t0)

        # warm-up run (module load, allocator), then the two reader depths alternated twice
        sequence.run_sequence(loader, None, features, f"{tmp}/warm", max_feats=a.feats, prefetch=2)
        runs = {2: [], 0: []}
        for rep in range(2):
            for pf in (2, 0):
                res = sequence.run_sequence(loader, None, features, f"{tmp}/p{pf}_{rep}", max_feats=a.feats, prefetch=pf)
                runs[pf] += [r[2] for r in res]
                statuses = [r[1] for r in res]

        # the tracker over arrays already on the device
        dd = [torch.from_numpy(m.view(np.int16)).to(dev) for m in mm]
        md = [torch.from_numpy(np.ascontiguousarray(seq.mask[k])).to(dev) for k in range(N)]
        cd = [torch.from_numpy(np.ascontiguousarray(seq.colour[k])).to(dev) for k in range(N)]
        rq = torch.empty((400, 400, 3), dtype=torch.uint8, device=dev)
        on_dev = []
        trk = Tracker(None, H, W, seq.K, a.feats, 2 + 4, max_keyframes=min(1024, -(-N // 2)))
        try:
            for k in range(N):
                t0 = time.perf_counter()
                st, roi, _, pose = trk.begin_frame_mm(dd[k], md[k], cd[k], rq, loader_id=k, first_pose=loader.initial_pose(k))
                if st == _lib.BT_FRAME_OTHER:
                    rq.cpu()
                    kp, de = features(f"{k:04d}", None, roi)
                    trk.end_frame(kp, torch.from_numpy(de).to(dev))
                torch.cuda.synchronize()
                on_dev.append(time.perf_counter() - t0)
        finally:
            trk.close()

        # front end: uint16 on the device vs host conversion + float upload + float front end
        fe = FrameFrontEnd()
        d_out, n_out = torch.empty((H, W), device=dev), torch.empty((H, W, 4), device=dev)
        fg = torch.empty((H, W), dtype=torch.uint8, device=dev)
        fe_u16, fe_f32 = [], []
        try:
            for rep in range(3):
                for k in range(min(N, 100)):
                    t0 = time.perf_counter()
                    dm = torch.from_numpy(mm[k].view(np.int16)).to(dev).view(torch.uint16)
                    fe.process_masked([dm], [md[k]], H, W, seq.K, [d_out], [n_out], [fg], fetch_roi=False)
                    torch.cuda.synchronize()
                    t1 = time.perf_counter()
                    f = (mm[k].astype(np.float64) * 0.001).astype(np.float32)
                    f[f.astype(np.float64) < 0.1] = 0
                    fe.process_masked([torch.from_numpy(f).to(dev)], [md[k]], H, W, seq.K, [d_out], [n_out], [fg], fetch_roi=False)
                    torch.cuda.synchronize()
                    t2 = time.perf_counter()
                    if rep:
                        fe_u16.append(t1 - t0)
                        fe_f32.append(t2 - t1)
        finally:
            fe.close()

    out = {"card": benchkit.card(), "torch_device": torch.cuda.get_device_name(0), "frames": N, "H": H, "W": W, "feats": a.feats,
           "statuses": {str(s): statuses.count(s) for s in sorted(set(statuses))},
           "prefetch2": stats(runs[2]), "prefetch0": stats(runs[0]), "on_device": stats(on_dev), "decode": stats(dec),
           "frontend_u16_upload": stats(fe_u16), "frontend_host_convert_f32_upload": stats(fe_f32)}
    print(f"card: {out['card']}")
    for k in ("prefetch2", "prefetch0", "on_device", "decode", "frontend_u16_upload", "frontend_host_convert_f32_upload"):
        print(f"{k:34s} median {out[k]['median_ms']:8.3f} ms   p90 {out[k]['p90_ms']:8.3f} ms")
    line = json.dumps(out)
    print(line)
    if a.out_json:
        os.makedirs(os.path.dirname(os.path.abspath(a.out_json)), exist_ok=True)
        with open(a.out_json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
