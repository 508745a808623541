#!/usr/bin/env python3
"""The LF-Net feature server on the device, with lf-net-release/run_server.py's protocol: unmodified clients (the reference's Lfnet class,
sequence.LfnetClient) connect to tcp://<host>:<port> as they would to the TensorFlow server.  Concurrent clients are batched into one
bt_lfnet_detect of at most --max_batch requests.  Runs in the foreground until interrupted (Ctrl-C), then closes the socket and the context.

    python scripts/lfnet_server.py --lfnet_model lf-net-release/release/models/indoor --port 5555
    python scripts/lfnet_server.py --weights_file indoor.btlfnet --port 5555 --max_batch 8
"""
from __future__ import annotations

import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--lfnet_model", help="a model directory: config.pkl and weights.npz")
    src.add_argument("--weights_file", help="a weights file (scripts/lfnet_export_blob.py); it fixes top_k")
    ap.add_argument("--port", type=int, default=5555)
    ap.add_argument("--top_k", type=int, default=None, help="run_server.py's --top_k (default 500); with --lfnet_model only")
    ap.add_argument("--max_batch", type=int, default=8, help="most requests run in one call")
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    if a.weights_file and a.top_k is not None:
        ap.error("--top_k applies to --lfnet_model: a weights file holds its own top_k (scripts/lfnet_export_blob.py --top_k)")
    if a.max_batch < 1:
        ap.error("--max_batch must be at least 1")
    from bundletrack_b200 import lfnet
    from bundletrack_b200.lfnet_server import LfnetServer
    if a.weights_file:
        net = lfnet.LfnetDevice.from_file(a.weights_file, max_images=a.max_batch, device=a.device)
    else:
        net = lfnet.load_lfnet(a.lfnet_model, top_k=500 if a.top_k is None else a.top_k, max_images=a.max_batch, device=a.device)
    server = LfnetServer(net, f"tcp://*:{a.port}", max_batch=a.max_batch)
    print(f"LF-Net on cuda:{a.device} listening on tcp://*:{a.port} (top_k {net.hp['top_k']}, up to {a.max_batch} requests per call)", flush=True)
    try:
        server.serve_forever()
    except KeyboardInterrupt:
        pass
    finally:
        server.close()


if __name__ == "__main__":
    main()
