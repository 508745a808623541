#!/usr/bin/env python3
"""Propagates a first-frame object mask through a video on the device, as transductive-vos.pytorch's run_video.py does, and writes one
<name>.png per frame (0 / 255) to --mask_save_dir, <name> being the colour file's name up to its first dot.  The frames are the files of
--img_dir in sorted order; the first one's mask is --init_mask_file (channel 0 when it has three).  The network is resnet50 only.

    python scripts/run_vos.py --img_dir video/rgb --init_mask_file video/masks/0000.png --mask_save_dir video/masks_vos \\
        --resume davis_trainval.pth.tar

--davis ROOT runs a DAVIS 2017 folder instead, as lib/predict.py does: for each sequence of ImageSets/2017/<set>.txt (or --sequences a,b),
the frames JPEGImages/<resolution>/<seq>/*.jpg in sorted order, decoded with cv2 as above, and the first frame's annotation
Annotations/<resolution>/<seq>/<first>.png read as palette indices (not cv2's channel 0, which is a palette colour's blue value).  Each
frame's label map (VosDevice.labels) is written to <results>/<seq>/<name>.png as a palette PNG with the annotation's palette, as
lib/utils.py's save_prediction does; frame 0's is the annotation's indices.  A sequence whose annotation has more label values than the
network carries is skipped with bt_vos_begin's message, and the skipped ones are listed at the end; any other error stops the run.

    python scripts/run_vos.py --davis DAVIS --results results/davis --set val --resume davis_trainval.pth.tar
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
    ap.add_argument("--img_dir", type=str)
    ap.add_argument("--init_mask_file", type=str)
    ap.add_argument("--mask_save_dir", type=str)
    ap.add_argument("--davis", type=str, help="a DAVIS 2017 root, in place of --img_dir, --init_mask_file and --mask_save_dir")
    ap.add_argument("--results", type=str, help="with --davis: where <seq>/<name>.png are written")
    ap.add_argument("--set", type=str, default="val", help="with --davis: the ImageSets/2017 list")
    ap.add_argument("--sequences", type=str, help="with --davis: comma-separated sequences in place of --set's")
    ap.add_argument("--resolution", type=str, default="480p", help="with --davis: the JPEGImages / Annotations resolution")
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    if a.model != "resnet50":
        ap.error(f"--model {a.model}: only resnet50 is implemented")
    params = dict(ref_num=a.ref_num, range=a.range, sigma1=a.sigma1, sigma2=a.sigma2, temperature=a.temperature)
    if a.davis:
        if a.img_dir or a.init_mask_file or a.mask_save_dir:
            ap.error("--davis takes --results, not --img_dir, --init_mask_file or --mask_save_dir")
        if not a.results:
            ap.error("--davis needs --results")
        return run_davis(a.davis, a.results, a.set, a.sequences, a.resolution, a.resume, params, a.device)
    if not (a.img_dir and a.init_mask_file and a.mask_save_dir):
        ap.error("give --img_dir, --init_mask_file and --mask_save_dir, or --davis and --results")
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


def run_davis(root: str, results: str, set_name: str, sequences: str | None, resolution: str, checkpoint: str, params: dict,
              device: int = 0) -> list:
    """Writes every sequence's label maps; returns the sequences skipped because bt_vos_begin refused their annotation."""
    import cv2
    import torch
    from bundletrack_b200 import _lib
    from bundletrack_b200.vos import VosDevice, read_checkpoint, read_palette_mask, write_palette_mask
    from eval_masks import davis_sequence_names

    sd = read_checkpoint(checkpoint)
    dev = torch.device("cuda", device)
    nets = {}                        # (H, W) -> VosDevice: each frame size gets its own reservation
    skipped = []
    try:
        for seq in davis_sequence_names(root, set_name, sequences):
            files = sorted(glob.glob(os.path.join(root, "JPEGImages", resolution, seq, "*.jpg")))
            if not files:
                raise SystemExit(f"{os.path.join(root, 'JPEGImages', resolution, seq)}: no .jpg frames")
            names = [os.path.basename(p).split(".")[0] for p in files]
            mask0, palette = read_palette_mask(os.path.join(root, "Annotations", resolution, seq, f"{names[0]}.png"))
            if palette is None:      # an 8-bit grey annotation: its values are the indices
                palette = [v for i in range(256) for v in (i, i, i)]
            first = cv2.imread(files[0], cv2.IMREAD_COLOR)
            H, W = first.shape[:2]
            if mask0.shape != (H, W):
                raise SystemExit(f"{seq}: the annotation is {mask0.shape[0]} x {mask0.shape[1]}, the frames {H} x {W}")
            if (H, W) not in nets:
                nets[(H, W)] = VosDevice(sd, params, H, W, device=device)
            v = nets[(H, W)]
            labels = torch.empty((H, W), dtype=torch.uint8, device=dev)
            try:
                v.begin(torch.from_numpy(first).to(dev), torch.from_numpy(mask0).to(dev))
            except _lib.BtError as e:
                if e.rc != _lib.BT_ERR_INVALID_ARG or "distinct values" not in str(e):      # only the channel-count refusal skips
                    raise
                print(f"{seq}: skipped: {e}")
                skipped.append(seq)
                continue
            out_dir = os.path.join(results, seq)
            os.makedirs(out_dir, exist_ok=True)
            for k, (path, name) in enumerate(zip(files, names)):
                if k > 0:
                    colour = cv2.imread(path, cv2.IMREAD_COLOR)
                    if colour is None or colour.shape != (H, W, 3):
                        raise SystemExit(f"{path}: not an {H} x {W} colour image")
                    v.next(torch.from_numpy(colour).to(dev))
                write_palette_mask(os.path.join(out_dir, f"{name}.png"), v.labels(labels).cpu().numpy(), palette)
            print(f"{seq}: {len(files)} label maps written to {out_dir}")
    finally:
        for v in nets.values():
            v.close()
    if skipped:
        print(f"skipped {len(skipped)} sequences: {', '.join(skipped)}")
    return skipped


if __name__ == "__main__":
    main()
