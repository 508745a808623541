"""Float64 restatement of transductive-vos.pytorch's run_video.py (resnet50), written from its description in DESIGN.md §3.13 with
torch.nn.functional on the CPU: the feature network, frame 0's labels, the reference-frame schedule, the prediction and the output mask.

random_state_dict(seed) builds a VOSNet-shaped state dict (module. prefix, as main.py saves it) initialised as resnet.py does: conv
weights normal with std sqrt(2 / n), n = k * k * out_channels, and randomised BN statistics.  Given a calibration image, each BN's
statistics are that image's per-channel mean and variance, perturbed at random, so activations stay near unit scale through the 16
residual blocks as in a trained network (uncalibrated, the features of a 640 x 480 frame reach 1e4 and the softmax is one-hot)."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
BN_EPS = 1e-5
LAYERS = ((3, 64, 1), (4, 128, 2), (6, 256, 1), (3, 256, 1))     # blocks, planes, stride of layer1..layer4


def state_shapes() -> dict:
    """name -> shape of every tensor of VOSNet('resnet50')'s state dict (without num_batches_tracked and the module. prefix)."""
    s = {}

    def bn(name, c):
        for v in ("weight", "bias", "running_mean", "running_var"):
            s[f"{name}.{v}"] = (c,)
    s["backbone.0.weight"] = (64, 3, 7, 7)
    bn("backbone.1", 64)
    inp = 64
    for li, (n, planes, stride) in enumerate(LAYERS):
        for b in range(n):
            p = f"backbone.{4 + li}.{b}"
            s[f"{p}.conv1.weight"] = (planes, inp, 1, 1); bn(f"{p}.bn1", planes)
            s[f"{p}.conv2.weight"] = (planes, planes, 3, 3); bn(f"{p}.bn2", planes)
            s[f"{p}.conv3.weight"] = (4 * planes, planes, 1, 1); bn(f"{p}.bn3", 4 * planes)
            if b == 0 and (stride != 1 or inp != 4 * planes):
                s[f"{p}.downsample.0.weight"] = (4 * planes, inp, 1, 1); bn(f"{p}.downsample.1", 4 * planes)
            inp = 4 * planes
    s["adjust_dim.weight"] = (256, 1024, 1, 1)
    bn("bn256", 256)
    return s


def random_state_dict(seed: int, prefix: str = "module.", calibrate: np.ndarray | None = None) -> dict:
    g = torch.Generator().manual_seed(seed)
    out = {}
    for name, shp in state_shapes().items():
        if name.endswith(".weight") and len(shp) == 4:
            n = shp[2] * shp[3] * shp[0]
            t = torch.randn(shp, generator=g, dtype=torch.float64) * np.sqrt(2.0 / n)
        elif name.endswith("running_var"):
            t = 0.5 + torch.rand(shp, generator=g, dtype=torch.float64)
        elif name.endswith("running_mean") or name.endswith(".bias"):
            t = 0.2 * torch.randn(shp, generator=g, dtype=torch.float64)
        else:                                                    # BN weight
            t = 0.5 + torch.rand(shp, generator=g, dtype=torch.float64)
        out[prefix + name] = t.float()
        if name.endswith("running_var"):
            out[prefix + name[: -len("running_var")] + "num_batches_tracked"] = torch.tensor(0, dtype=torch.long)
    if calibrate is not None:
        stats = {}
        features(calibrate, out, stats=(stats, g))
        for k, t in stats.items():
            out[prefix + k] = t.float()
    return out


def _bn(x, sd, name, stats=None):
    if stats is not None:        # calibration: this BN's statistics from x, perturbed, written back before it is applied
        out, g = stats
        mean, var = x.mean((0, 2, 3)), x.var((0, 2, 3))
        c = mean.numel()
        sd[f"{name}.running_mean"] = mean + 0.1 * var.sqrt() * torch.randn(c, generator=g, dtype=x.dtype)
        sd[f"{name}.running_var"] = var * (0.8 + 0.4 * torch.rand(c, generator=g, dtype=x.dtype)) + 1e-3
        out[f"{name}.running_mean"], out[f"{name}.running_var"] = sd[f"{name}.running_mean"], sd[f"{name}.running_var"]
    w, b, m, v = (sd[f"{name}.{k}"].to(x) for k in ("weight", "bias", "running_mean", "running_var"))
    return F.batch_norm(x, m, v, w, b, training=False, eps=BN_EPS)


def normalise(bgr: np.ndarray) -> torch.Tensor:
    """cv2 BGR uint8 H x W x 3 -> 1 x 3 x H x W: RGB, / 255, (x - mean) / std, each step rounded to float32 as ToTensor and Normalize do."""
    x = torch.from_numpy(np.ascontiguousarray(bgr[..., ::-1])).permute(2, 0, 1).float().div(255)
    x = (x - torch.tensor(MEAN).view(3, 1, 1)) / torch.tensor(STD).view(3, 1, 1)
    return x.unsqueeze(0).double()


def features(bgr: np.ndarray, sd: dict, dtype=torch.float64, device="cpu", stats=None) -> torch.Tensor:
    """The network's output for one frame: ceil(H / 8) x ceil(W / 8) x 256, in float64 on the CPU unless asked otherwise.  stats
    (random_state_dict's calibration): ({} to fill, generator)."""
    sd = {(k[len("module."):] if k.startswith("module.") else k): torch.as_tensor(v).to(device, dtype) for k, v in sd.items()}
    with torch.no_grad():
        x = normalise(bgr).to(device, dtype)
        x = F.relu(_bn(F.conv2d(x, sd["backbone.0.weight"], stride=2, padding=3), sd, "backbone.1", stats))
        x = F.max_pool2d(x, 3, 2, 1)
        for li, (n, planes, stride) in enumerate(LAYERS):
            for b in range(n):
                p = f"backbone.{4 + li}.{b}"
                s = stride if b == 0 else 1
                t = F.relu(_bn(F.conv2d(x, sd[f"{p}.conv1.weight"]), sd, f"{p}.bn1", stats))
                t = F.relu(_bn(F.conv2d(t, sd[f"{p}.conv2.weight"], stride=s, padding=1), sd, f"{p}.bn2", stats))
                t = _bn(F.conv2d(t, sd[f"{p}.conv3.weight"]), sd, f"{p}.bn3", stats)
                r = x
                if f"{p}.downsample.0.weight" in sd:
                    r = _bn(F.conv2d(x, sd[f"{p}.downsample.0.weight"], stride=s), sd, f"{p}.downsample.1", stats)
                x = F.relu(t + r)
        x = _bn(F.conv2d(x, sd["adjust_dim.weight"]), sd, "bn256", stats)
    return x[0].permute(1, 2, 0)


def compress_labels(mask: np.ndarray) -> tuple[np.ndarray, int]:
    """The initial mask's values as consecutive channels: 0 -> 0 (kept when absent), the other present values in increasing order."""
    vals = [v for v in np.unique(mask) if v != 0]
    chan = np.zeros(256, np.int64)
    for i, v in enumerate(vals):
        chan[v] = i + 1
    return chan[mask], len(vals) + 1


def init_label(mask: np.ndarray, d: int) -> np.ndarray:
    """Frame 0's history label: the one-hot of the (compressed) mask bilinearly resized to (ceil(H / 8), ceil(W / 8)), align_corners =
    False; Hd x Wd x d."""
    H, W = mask.shape
    oh = F.one_hot(torch.from_numpy(mask.astype(np.int64)), d).permute(2, 0, 1).unsqueeze(0).double()
    return F.interpolate(oh, size=(-(-H // 8), -(-W // 8)), mode="bilinear", align_corners=False)[0].permute(1, 2, 0).numpy()


def schedule(k: int, ref_num: int, rng: int) -> list:
    if k <= ref_num:
        return list(range(k))
    end = k - 4
    start = max(end - rng, 0)
    return np.linspace(start, end, ref_num - 3).astype(int).tolist() + [k - 3, k - 2, k - 1]


def spatial_weight(Hd: int, Wd: int, sigma: float) -> np.ndarray:
    yy, xx = np.divmod(np.arange(Hd * Wd), Wd)
    d2 = (yy[:, None] - yy[None, :]) ** 2 + (xx[:, None] - xx[None, :]) ** 2
    return np.exp(-d2 / sigma ** 2)


def predict(ref_feats: list, ref_labels: list, target: np.ndarray, k: int, sigma1=8.0, sigma2=21.0, temperature=1.0) -> np.ndarray:
    """lib/predict.py's prediction for frame k from the selected references (in schedule order): d x HW, float64."""
    Hd, Wd, C = target.shape
    N = len(ref_feats)
    R = np.concatenate([f.reshape(-1, C) for f in ref_feats]).astype(np.float64)
    S = R @ target.reshape(-1, C).astype(np.float64).T * temperature
    S = np.exp(S - S.max(0, keepdims=True))
    S /= S.sum(0, keepdims=True)
    S = S.reshape(N, Hd * Wd, Hd * Wd)
    wd, ws = spatial_weight(Hd, Wd, sigma1), spatial_weight(Hd, Wd, sigma2)
    for j in range(N):
        S[j] *= ws if (k > 15 and j < N - 4) else wd
    L = np.concatenate([lab.reshape(Hd * Wd, -1) for lab in ref_labels]).astype(np.float64)
    return L.T @ S.reshape(N * Hd * Wd, Hd * Wd)


def upsample(pred: np.ndarray, Hd: int, Wd: int, H: int, W: int) -> np.ndarray:
    """The prediction bilinearly upsampled to H x W (align_corners = False): d x H x W."""
    p = torch.from_numpy(pred.reshape(1, -1, Hd, Wd))
    return F.interpolate(p, size=(H, W), mode="bilinear", align_corners=False)[0].numpy()


def margin(p: np.ndarray) -> np.ndarray:
    """Per pixel of a d x ... prediction, the gap between its two largest channels (inf with one channel)."""
    if p.shape[0] < 2:
        return np.full(p.shape[1:], np.inf)
    s = np.sort(p, axis=0)
    return s[-1] - s[-2]
