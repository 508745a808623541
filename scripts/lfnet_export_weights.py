"""Turn a released LF-Net TF checkpoint into the weights.npz bundletrack_b200.lfnet.load_lfnet reads: every variable of the checkpoint
under its TF name (ConvOnlyResNet/..., SimpleDesc/..., without ':0'), as float32.  The model directory's config.pkl is read as it is.

    python scripts/lfnet_export_weights.py --model lf-net-release/release/models/indoor

Needs TensorFlow 1.x (CPU is enough), which this package does not install or test; run it once where the reference's server runs and
copy weights.npz next to config.pkl.  load_lfnet checks the names and shapes against the network and names any that differ."""
import argparse
import os

import numpy as np


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--model", required=True, help="the model directory (checkpoint + config.pkl) or a checkpoint prefix")
    ap.add_argument("--out", default=None, help="default: <model directory>/weights.npz")
    a = ap.parse_args()
    import tensorflow as tf
    ckpt = tf.train.latest_checkpoint(a.model) if os.path.isdir(a.model) else a.model
    if ckpt is None:
        raise SystemExit(f"no checkpoint under {a.model}")
    reader = tf.train.NewCheckpointReader(ckpt)
    names = sorted(n for n in reader.get_variable_to_shape_map() if n.startswith(("ConvOnlyResNet/", "SimpleDesc/")))
    out = a.out or os.path.join(a.model if os.path.isdir(a.model) else os.path.dirname(a.model), "weights.npz")
    np.savez(out, **{n: np.asarray(reader.get_tensor(n), np.float32) for n in names})
    print(f"{len(names)} variables -> {out}")


if __name__ == "__main__":
    main()
