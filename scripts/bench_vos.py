"""Object-mask propagation on one GPU: device time per stage and per frame of bt_vos_next at 640 x 480 with run_video.py's defaults, the
achieved rate from the work computed from the shapes, and, in the same run, the reference's graph as PyTorch runs it in float32 on the same
GPU (cuDNN convolutions with TF32 allowed, an FP32 mm: torch's defaults) with its time and its mask disagreement with the library.

    python scripts/bench_vos.py [--frames 60] [--warmup 10] [--H 480 --W 640]

The per-frame window is also run with each frame's label map written after it (bt_vos_labels after every bt_vos_next, DESIGN.md §3.17),
and bt_vos_labels is timed alone; python scripts/bench_vos.py --H 480 --W 854 measures them at DAVIS's 480p size.

It also times run_sequence over a synthetic YCBInEOAT-layout scene (bundletrack_b200.synth, host feature callable) at the same size: the
median wall time per frame reading the mask files, and with masks=VosSource propagating them on the device.  Weights are seeded (oracle.vos_oracle.random_state_dict, BN statistics calibrated on a frame); speed does not depend on them."""
import argparse
import json
import os

import numpy as np

import benchkit


def backbone_macs(H, W):
    """Multiply-adds of the network for one H x W frame, from the layer shapes."""
    from bundletrack_b200 import vos

    def out(n, ks, s):
        return (n + 2 * (ks // 2) - ks) // s + 1
    h, w = out(H, 7, 2), out(W, 7, 2)
    total = h * w * 64 * 7 * 7 * 3
    h, w = out(h, 3, 2), out(w, 3, 2)
    inp = 64
    for n, planes, stride in vos.LAYERS:
        for b in range(n):
            s = stride if b == 0 else 1
            h2, w2 = out(h, 3, s), out(w, 3, s)
            total += h * w * inp * planes + h2 * w2 * planes * planes * 9 + h2 * w2 * planes * 4 * planes
            if b == 0 and (s != 1 or inp != 4 * planes):
                total += h2 * w2 * inp * 4 * planes
            h, w, inp = h2, w2, 4 * planes
    return total + h * w * 1024 * 256


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--H", type=int, default=480)
    ap.add_argument("--W", type=int, default=640)
    a = ap.parse_args()
    import torch
    import torch.nn.functional as F
    from bundletrack_b200 import vos
    from oracle import vos_oracle as vo
    assert torch.cuda.is_available(), "bench_vos.py measures on a GPU"
    dev = torch.device("cuda:0")
    name = torch.cuda.get_device_name(0)
    H, W, n = a.H, a.W, a.warmup + a.frames
    P = dict(vos.DEFAULTS)
    rng = np.random.default_rng(1)
    yy, xx = np.mgrid[:H, :W]
    bg = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    frames = []
    for k in range(n):
        f = bg.copy()
        f[(yy - H * (0.4 + 0.002 * k)) ** 2 + (xx - W * (0.4 + 0.003 * k)) ** 2 < (0.15 * H) ** 2] = (30, 200, 80)
        frames.append(torch.from_numpy(f).to(dev))
    m0 = np.zeros((H, W), np.uint8)
    m0[(yy - 0.4 * H) ** 2 + (xx - 0.4 * W) ** 2 < (0.15 * H) ** 2] = 1
    state = vo.random_state_dict(7, calibrate=frames[0][::4, ::4].cpu().numpy())
    sd = {k[len("module."):]: v.double().numpy() for k, v in state.items() if not k.endswith("num_batches_tracked")}
    v = vos.VosDevice(sd, P, H, W)
    stream = torch.cuda.current_stream().cuda_stream

    # per-stage device time (each call timed by the library's events)
    v.begin(frames[0], torch.from_numpy(m0).to(dev), stream=stream)
    v.enable_timing(True)
    stages = []
    for k in range(1, n):
        v.next(frames[k], stream=stream)
        if k > a.warmup:
            stages.append(v.timing())
    v.enable_timing(False)
    med = {s: float(np.median([t[s] for t in stages])) for s in ("backbone", "propagation", "mask")}
    # per-frame device time with no timing events inside: events around the whole run
    outs = [torch.empty((H, W), dtype=torch.uint8, device=dev) for _ in range(n)]
    v.begin(frames[0], torch.from_numpy(m0).to(dev), out=outs[0], stream=stream)
    ks = iter(range(1, n))

    def next_frame():
        k = next(ks)
        v.next(frames[k], out=outs[k], stream=stream)
    per_frame = benchkit.window_ms(next_frame, n - a.warmup - 1, a.warmup, stream)
    # the same window writing each frame's label map too, then bt_vos_labels alone on the last frame
    lab = torch.empty((H, W), dtype=torch.uint8, device=dev)
    v.begin(frames[0], torch.from_numpy(m0).to(dev), out=outs[0], stream=stream)
    ks = iter(range(1, n))

    def next_frame_and_labels():
        k = next(ks)
        v.next(frames[k], out=outs[k], stream=stream)
        v.labels(lab, stream=stream)
    per_frame_labels = benchkit.window_ms(next_frame_and_labels, n - a.warmup - 1, a.warmup, stream)
    labels_ms = float(np.median(benchkit.calls_ms(lambda: v.labels(lab, stream=stream), 50, 5, stream)))
    Hd, Wd = -(-H // 8), -(-W // 8)
    HW = Hd * Wd
    bb = backbone_macs(H, W)
    prop = P["ref_num"] * HW * HW * 256
    # the reference's graph in float32 on the GPU, torch's defaults (cuDNN may use TF32 for convolutions; mm stays FP32)
    torch.backends.cudnn.benchmark = False
    sdt = {k: torch.from_numpy(x).float().to(dev) for k, x in sd.items()}
    wd = torch.from_numpy(vo.spatial_weight(Hd, Wd, P["sigma1"])).float().to(dev)
    ws = torch.from_numpy(vo.spatial_weight(Hd, Wd, P["sigma2"])).float().to(dev)
    comp, d = vo.compress_labels(m0)
    feats = [vo.features(frames[0].cpu().numpy(), sdt, torch.float32, dev).reshape(HW, 256)]
    labels = [torch.from_numpy(vo.init_label(comp, d)).float().to(dev).reshape(HW, d)]
    ups = []
    ks = iter(range(1, n))

    def ref_frame():
        k = next(ks)
        f = vo.features(frames[k].cpu().numpy(), sdt, torch.float32, dev).reshape(HW, 256)
        idx = vo.schedule(k, P["ref_num"], P["range"])
        R = torch.cat([feats[i] for i in idx])
        S = (R @ f.T * P["temperature"]).softmax(0).view(len(idx), HW, HW)
        if k > 15:
            S = torch.cat([S[:-4] * ws, S[-4:] * wd])
        else:
            S = S * wd
        pred = torch.cat([labels[i] for i in idx]).T @ S.reshape(-1, HW)
        lab = F.one_hot(pred.argmax(0), d).float()
        ups.append(F.interpolate(pred.view(1, d, Hd, Wd), size=(H, W), mode="bilinear", align_corners=False)[0].argmax(0))
        feats.append(f)
        labels.append(lab)
    t_ref = benchkit.calls_ms(ref_frame, n - a.warmup - 1, a.warmup, stream)
    ref_masks = [torch.where(up > 0, 255, 0).to(torch.uint8) for up in ups]
    disagree = float(np.mean([(r != o).float().mean().item() for r, o in zip(ref_masks, outs[1:])]))
    res = dict(gpu=name, power_limit=benchkit.card(), H=H, W=W, frames=a.frames, params=P,
               stage_ms_median=med, per_frame_ms=per_frame, per_frame_with_labels_ms=per_frame_labels, labels_ms_median=labels_ms,
               backbone_gmac=bb / 1e9, propagation_gmac=prop / 1e9,
               backbone_tflops_3xtf32_counted_once=2 * bb / med["backbone"] / 1e9,
               propagation_tflops_counted_once=2 * prop / med["propagation"] / 1e9,
               torch_fp32_graph_per_frame_ms_median=float(np.median(t_ref)),
               mask_disagreement_with_torch_fp32=disagree)
    v.close()
    res.update(run_sequence_times(H, W, a.frames + a.warmup, sd))
    print(json.dumps(res))


def run_sequence_times(H, W, n, sd):
    """Median per-frame wall time of run_sequence on a synthetic YCBInEOAT scene written to a temporary directory, with the scene's mask
    files and with the VOS source (the first frame's mask propagated); the first 10 frames are left out of each median."""
    import tempfile
    import torch
    from bundletrack_b200 import sequence, synth, vos
    seq = synth.make_sequence(52, n, H=H, W=W, n_feats=400)
    features = synth.recorded_features(seq)
    with tempfile.TemporaryDirectory() as tmp:
        video = os.path.join(tmp, "synthvideo")
        synth.write_ycbineoat_video(seq, video)
        out = {}
        for name in ("mask_files", "vos_source"):
            masks = None
            if name == "vos_source":
                masks = vos.VosSource(vos.VosDevice(sd, {}, H, W), seq.mask[0].astype(np.uint8))
            res = sequence.run_sequence(sequence.YcbineoatVideo(video), None, features, os.path.join(tmp, name), max_feats=400, masks=masks)
            if masks is not None:
                masks.close()
            torch.cuda.synchronize()
            out[f"run_sequence_ms_per_frame_median_{name}"] = float(np.median([r[2] for r in res[10:]]) * 1000)
    return out


if __name__ == "__main__":
    main()
