"""Device time of bt_lfnet_detect (LF-Net on the device) for 1 and 8 requests, split by stage, and run_sequence's per-frame wall time with
the device source against a host callable that returns the same features (request downloaded, descriptors uploaded).  Seeded random
weights under the TF variable names; requests from synthetic scenes.  Prints one JSON object; --out also writes it to a file.

    python scripts/bench_lfnet.py [--iters 50] [--out results.json]

There is no TF1 figure on the H100 to compare with: the reference's server is not run here (not measured)."""
import argparse
import ctypes
import json
import os
import tempfile

import numpy as np

import benchkit

STAGES = ("trunk", "score_maps", "detection", "keypoints_patches", "descriptor")


def requests(dev, n):
    import torch
    from bundletrack_b200 import _lib, synth
    from bundletrack_b200.frontend import FrameFrontEnd
    H, W = 480, 640
    seq = synth.make_sequence(3, n, H=H, W=W)
    fe = FrameFrontEnd()
    out = []
    for k in range(n):
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        d, nrm, fg = torch.empty((H, W), device=dev), torch.empty((H, W, 4), device=dev), torch.empty((H, W), dtype=torch.uint8, device=dev)
        req = torch.zeros((400, 400, 3), dtype=torch.uint8, device=dev)
        fe.process_masked([t(seq.depth_raw[k])], [t(seq.mask[k])], H, W, seq.K, [d], [nrm], [fg], mode=_lib.BT_MASK_AS_IS)
        fe.lfnet_request([t(seq.colour[k])], [fg], H, W, [req])
        out.append(req)
    torch.cuda.synchronize()
    fe.close()
    return out


def time_detect(net, reqs, iters):
    from bundletrack_b200 import _lib
    total = benchkit.window_ms(lambda: net.detect(reqs), iters, 3, net.stream)
    _lib.check(net.lib.bt_lfnet_enable_timing(net.ctx, 1))
    ms = (ctypes.c_float * 5)()
    acc = np.zeros(5)
    for _ in range(iters):
        net.detect(reqs)
        _lib.check(net.lib.bt_lfnet_get_timing(net.ctx, ms))
        acc += np.array(ms[:])
    _lib.check(net.lib.bt_lfnet_enable_timing(net.ctx, 0))
    return {"ms_per_call": round(total, 4), "ms_per_request": round(total / len(reqs), 4),
            "stages_ms": {k: round(v / iters, 4) for k, v in zip(STAGES, acc)}}


def sequence_runs(net, dev, n_frames):
    import torch
    from bundletrack_b200 import policy, sequence, synth
    H, W = 480, 640
    seq = synth.make_sequence(9, n_frames, H=H, W=W)
    tmp = tempfile.mkdtemp()
    video = os.path.join(tmp, "synthvideo")
    synth.write_ycbineoat_video(seq, video)
    loader = sequence.YcbineoatVideo(video)

    def host(id_str, request, roi):
        kp, de, nk = net.detect([torch.from_numpy(request).to(dev)])
        n = int(nk[0])
        if n == 0:
            raise sequence.DetectionFailed(id_str)
        return policy.lfnet_reply_keypoints(n, net.hp["desc_dim"], kp[0, :n].cpu().numpy(), roi), de[0, :n].cpu().numpy()
    out = {}
    for rep in range(2):                 # the second pass of each is reported: the first loads modules and warms caches
        for name, src in (("device_source", net), ("host_callable", host)):
            res = sequence.run_sequence(loader, None, src, os.path.join(tmp, f"{name}{rep}"), max_feats=net.hp["top_k"], device=0)
            t = np.array([r[2] for r in res[1:]]) * 1000
            out[name] = {"frames": len(res), "median_ms_per_frame": round(float(np.median(t)), 3), "summary": sequence.summary(res)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from bundletrack_b200 import lfnet
    from oracle import lfnet_oracle as lo
    dev = torch.device("cuda:0")
    hp = dict(lfnet.DEFAULTS)
    net = lfnet.LfnetDevice(lo.random_weights(lfnet.weight_shapes(hp), 11), hp, max_images=8)
    reqs = requests(dev, 8)
    res = {"card": benchkit.card(), "torch": torch.__version__,
           "detect_1": time_detect(net, reqs[:1], a.iters), "detect_8": time_detect(net, reqs, a.iters),
           "run_sequence": sequence_runs(net, dev, a.frames), "tf1_server_on_h100": "not measured"}
    net.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
