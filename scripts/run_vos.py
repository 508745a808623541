#!/usr/bin/env python3
"""Propagates a first-frame object mask through a video on the device, as transductive-vos.pytorch's run_video.py does, and writes one
<name>.png per frame (0 / 255) to --mask_save_dir, <name> being the colour file's name up to its first dot.  The frames are the files of
--img_dir in sorted order; the first one's mask is --init_mask_file (channel 0 when it has three).  The network is resnet50 only.

    python scripts/run_vos.py --img_dir video/rgb --init_mask_file video/masks/0000.png --mask_save_dir video/masks_vos \\
        --resume davis_trainval.pth.tar
"""
from __future__ import annotations

import argparse
import glob
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref_num", "-n", type=int, default=9)
    ap.add_argument("--resume", "-r", type=str, required=True, help="the checkpoint run_video.py --resume takes")
    ap.add_argument("--model", type=str, default="resnet50", help="resnet50 only")
    ap.add_argument("--sigma1", type=float, default=8.0)
    ap.add_argument("--sigma2", type=float, default=21.0)
    ap.add_argument("--range", type=int, default=40)
    ap.add_argument("--temperature", "-t", type=float, default=1.0)
    ap.add_argument("--img_dir", type=str, required=True)
    ap.add_argument("--init_mask_file", type=str, required=True)
    ap.add_argument("--mask_save_dir", type=str, required=True)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    if a.model != "resnet50":
        ap.error(f"--model {a.model}: only resnet50 is implemented")
    import cv2
    import torch
    from bundletrack_b200.vos import load_vos, read_init_mask

    files = sorted(glob.glob(os.path.join(a.img_dir, "*")))
    if not files:
        ap.error(f"no frames in {a.img_dir}")
    try:
        mask0 = read_init_mask(a.init_mask_file)
    except ValueError as e:
        ap.error(str(e))
    first = cv2.imread(files[0], cv2.IMREAD_COLOR)
    H, W = first.shape[:2]
    if mask0.shape != (H, W):
        ap.error(f"the initial mask is {mask0.shape}, the frames {H} x {W}")
    dev = torch.device("cuda", a.device)
    params = dict(ref_num=a.ref_num, range=a.range, sigma1=a.sigma1, sigma2=a.sigma2, temperature=a.temperature)
    v = load_vos(a.resume, params, H=H, W=W, device=a.device)
    os.makedirs(a.mask_save_dir, exist_ok=True)
    for k, path in enumerate(files):
        colour = first if k == 0 else cv2.imread(path, cv2.IMREAD_COLOR)
        if colour is None or colour.shape != (H, W, 3):
            raise SystemExit(f"{path}: not an {H} x {W} colour image")
        c = torch.from_numpy(colour).to(dev)
        m = v.begin(c, torch.from_numpy(mask0).to(dev)) if k == 0 else v.next(c)
        name = os.path.basename(path).split(".")[0]
        cv2.imwrite(os.path.join(a.mask_save_dir, f"{name}.png"), m.cpu().numpy())
    v.close()
    print(f"{len(files)} masks written to {a.mask_save_dir}")


if __name__ == "__main__":
    main()
