"""Match images on the device against cv2.drawMatches on the host, at the tracker's sizes (640 x 480 frames, ROIs of 120-300 rows).

Device time per image (one image per call) and per batch of a step's images (max_BA_frames = 15: 105 BA images plus the 3 images of each
pair computed in the step), from CUDA events; host time of the same images through cv2 (crop, resize, drawMatches).  Prints one JSON line
with the card's name and power limit.

    python scripts/bench_matchviz.py [--matches 300] [--reps 20]
"""
from __future__ import annotations

import argparse
import json
import time

import numpy as np

import benchkit


def main():
    import torch
    from bundletrack_b200.overlay import MatchViz, match_image_shape
    from oracle import matchviz_oracle as mv
    from oracle.segment_oracle import test_colour

    ap = argparse.ArgumentParser()
    ap.add_argument("--matches", type=int, default=300)
    ap.add_argument("--images", type=int, default=105 + 3 * 14)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    rs = np.random.default_rng(0)
    colour = torch.from_numpy(test_colour(480, 640)).to(dev)
    jobs = []
    for _ in range(a.images):
        rois = []
        for _ in range(2):
            h, w = int(rs.integers(120, 300)), int(rs.integers(120, 300))
            u0, v0 = int(rs.integers(0, 640 - w)), int(rs.integers(0, 480 - h))
            rois.append((u0, u0 + w, v0, v0 + h))
        ra, rb = rois
        n = a.matches
        uv = np.stack([rs.uniform(ra[0], ra[1], n), rs.uniform(ra[2], ra[3], n), rs.uniform(rb[0], rb[1], n), rs.uniform(rb[2], rb[3], n)], 1)
        jobs.append((colour, ra, colour, rb, torch.from_numpy(uv.astype(np.float32)).to(dev), mv.RNG_DEFAULT))
    outs = [torch.empty((*match_image_shape(j[1], j[3]), 3), dtype=torch.uint8, device=dev) for j in jobs]
    mz = MatchViz(max_images=len(jobs), max_matches=a.matches * len(jobs), stream=torch.cuda.current_stream(dev).cuda_stream)
    single = benchkit.window_ms(lambda: mz.draw(jobs[:1], outs[:1]), a.reps, 1, mz.stream)
    batch = benchkit.window_ms(lambda: mz.draw(jobs, outs), a.reps, 1, mz.stream)
    import cv2
    host_col = colour.cpu().numpy()
    t0 = time.perf_counter()
    for ca, ra, cb, rb, uv, st in jobs[:20]:
        A, B = mv.crop(host_col, ra), mv.crop(host_col, rb)
        s = mv.viz_scale(A.shape[0], B.shape[0])
        A, B = cv2.resize(A, (0, 0), fx=s, fy=s), cv2.resize(B, (0, 0), fx=s, fy=s)
        kp = mv.keypoints(uv.cpu().numpy(), ra, rb, s)
        ka = [cv2.KeyPoint(float(x), float(y), 1) for x, y in kp[:, :2]]
        kb = [cv2.KeyPoint(float(x), float(y), 1) for x, y in kp[:, 2:]]
        cv2.drawMatches(A, ka, B, kb, [cv2.DMatch(i, i, 0) for i in range(len(kp))], None, flags=cv2.DrawMatchesFlags_NOT_DRAW_SINGLE_POINTS)
    host = (time.perf_counter() - t0) * 1e3 / 20
    px = sum(o.numel() // 3 for o in outs) / len(outs)
    print(json.dumps({"card": benchkit.card(), "matches_per_image": a.matches, "images_per_batch": len(jobs), "mean_pixels_per_image": round(px),
                      "device_ms_one_image": round(single, 4), "device_ms_batch": round(batch, 4),
                      "device_ms_per_image_in_batch": round(batch / len(jobs), 4), "host_cv2_ms_per_image": round(host, 3)}))
    mz.close()


if __name__ == "__main__":
    main()
