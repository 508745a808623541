#!/usr/bin/env python3
"""Write an LF-Net model directory (config.pkl + weights.npz, as load_lfnet reads it) as one weights file that bt_lfnet_load_file, the C++
LfnetGpu and scripts/lfnet_server.py --weights_file load: the bt_lfnet_params of the config at --top_k, then the float32 blob with BN folded
(layout: include/bundletrack_b200.h).  No GPU is needed.

    python scripts/lfnet_export_blob.py --model lf-net-release/release/models/indoor --out indoor.btlfnet
"""
from __future__ import annotations

import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--model", required=True, help="the model directory: config.pkl and weights.npz (scripts/lfnet_export_weights.py)")
    ap.add_argument("--out", default=None, help="default: <model>/lfnet.btlfnet")
    ap.add_argument("--top_k", type=int, default=500, help="run_server.py's --top_k, which the file fixes")
    a = ap.parse_args()
    from bundletrack_b200 import lfnet
    out = a.out or os.path.join(a.model, "lfnet.btlfnet")
    lfnet.write_weights_file(a.model, out, a.top_k)
    hp, n = lfnet.file_info(out)
    print(f"top_k {hp['top_k']}, desc_dim {hp['desc_dim']}, {n} floats -> {out}")


if __name__ == "__main__":
    main()
