#!/usr/bin/env python3
"""Tracks one model in one NOCS-REAL275 scene, as the reference's scripts/run_nocs.py + bundle_track_nocs do, and writes one pose file per
frame to <out_dir>/<model>_<scene>/poses/<id>.txt, the layout scripts/eval_nocs.py reads.  Features come from a running LF-Net server
(lf-net-release/run_server.py) at tcp://127.0.0.1:<port>.  Frames follow the 6-PACK data list (bundletrack_b200.sequence.NocsScene); the
masks are <mask_dir>/<id>.png.  With --log 1 the
reference's LOG images are written next to the poses (bundletrack_b200.overlay).  Nothing under out_dir is removed.

    python scripts/run_nocs.py --nocs_dir NOCS --scene_id 1 --model_name can_arizona_tea_norm --mask_dir masks/scene_1_model_can_arizona_tea_norm \\
        --out_dir results --port 5555
    python scripts/eval_nocs.py --nocs_dir NOCS --results_dir results
"""
from __future__ import annotations

import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    from bundletrack_b200.sequence import LfnetClient, NocsScene, run_sequence, summary
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--nocs_dir", required=True)
    ap.add_argument("--scene_id", type=int, default=1)
    ap.add_argument("--model_name", default="can_arizona_tea_norm")
    ap.add_argument("--port", type=int, default=5555, help="the LF-Net server's port")
    ap.add_argument("--lfnet_model", default=None, help="instead of the server: a released LF-Net model directory (config.pkl and "
                                                        "weights.npz from scripts/lfnet_export_weights.py), run on the device")
    ap.add_argument("--mask_dir", required=True, help="the scene's and model's masks, <id>.png")
    ap.add_argument("--out_dir", required=True)
    ap.add_argument("--vos_model", default=None, help="instead of the mask files: a transductive-vos checkpoint (run_video.py --resume) "
                                                      "that propagates --init_mask through the video on the device")
    ap.add_argument("--init_mask", default=None, help="with --vos_model: the first frame's mask (label values, 8-bit)")
    ap.add_argument("--mask_save_dir", default=None, help="with --vos_model: also write each frame's mask there as <id>.png, 0 / 255")
    ap.add_argument("--config", default=None, help="a config_nocs.yml (default: its values, bundletrack_b200.config.NOCS_DEFAULTS)")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--log", type=int, default=0, help="the config's LOG: > 0 also writes every frame's overlay images under the output "
                                                       "directory (<id>/color_viz.jpg, color_viz/, color_raw/); needs cv2")
    a = ap.parse_args()
    loader = NocsScene(a.nocs_dir, a.scene_id, a.model_name, a.mask_dir)
    if (a.init_mask or a.mask_save_dir) and not a.vos_model:
        raise SystemExit("--init_mask and --mask_save_dir go with --vos_model")
    masks = None
    if a.vos_model:
        if not a.init_mask:
            raise SystemExit("--vos_model needs --init_mask, the first frame's mask")
        from bundletrack_b200.sequence import png_layout
        from bundletrack_b200.vos import load_source
        W, H = png_layout(loader.frames[0].colour)[:2]
        masks = load_source(a.vos_model, a.init_mask, H, W, a.mask_save_dir, device=a.device)
    if a.lfnet_model:
        from bundletrack_b200.lfnet import load_lfnet
        client = load_lfnet(a.lfnet_model, device=a.device)
    else:
        client = LfnetClient(f"tcp://127.0.0.1:{a.port}")
    try:
        res = run_sequence(loader, a.config, client, os.path.join(a.out_dir, f"{a.model_name}_{a.scene_id}"), device=a.device, log=a.log, masks=masks)
    finally:
        client.close()
        if masks is not None:
            masks.close()
    print(summary(res))


if __name__ == "__main__":
    main()
