"""LF-Net inference in float64 numpy: the graph lf-net-release/run_server.py builds (build_networks with mso_resnet_detector, simple_desc,
desc_inputs = photos and use_nms3d), stated stage by stage from the reference's Python, with every intermediate exposed.

`weights` maps TF variable names (ConvOnlyResNet/..., SimpleDesc/...) to arrays; `cfg` holds the hyper-parameters under the reference's
config keys.  BN is applied as tf.layers.batch_normalization does at inference (moving statistics, epsilon 1e-5), unfolded."""
from __future__ import annotations

import numpy as np

SIDE = 400
BN_EPS = 1e-5          # tf_layer_utils.py:185
IN_EPS = 1e-3          # det_tools.py:793


# ---- layers -----------------------------------------------------------------------------------------------------------------------------

def grey(request: np.ndarray) -> np.ndarray:
    """run_server.py:155-157: cv2.cvtColor(photo, COLOR_RGB2GRAY) on the request's BGR bytes (byte 0 is weighted as red), OpenCV's
    uint8 fixed point of OpenCV 4 (R 9798, G 19235, B 3735 over 2^15, rounded), as uint8."""
    r = request.astype(np.int64)
    return ((r[..., 0] * 9798 + r[..., 1] * 19235 + r[..., 2] * 3735 + (1 << 14)) >> 15).astype(np.uint8)


def photo(request: np.ndarray) -> np.ndarray:
    """The network input [H, W, 1]: the grey image / 255 as the server computes it (float32), widened to float64."""
    return (grey(request).astype(np.float32) / np.float32(255.0)).astype(np.float64)[..., None]


def leaky_relu(x, alpha):
    return np.where(x > 0, x, x * alpha)


def same_pads(size: int, k: int, stride: int):
    """TF 'SAME': out = ceil(size / stride), pad_total = max((out - 1) stride + k - size, 0), the smaller half before."""
    out = -(-size // stride)
    total = max((out - 1) * stride + k - size, 0)
    return out, total // 2, total - total // 2


def conv2d(x: np.ndarray, W: np.ndarray, b=None, stride: int = 1) -> np.ndarray:
    """tf.nn.conv2d(padding='SAME') (+ bias) on [..., H, W, Cin] with W [k, k, Cin, Cout].  conv2d_fixed_padding at stride 1 is this
    (tf_layer_utils.py:326-329)."""
    k = W.shape[0]
    H, Wd = x.shape[-3], x.shape[-2]
    oh, pt, pb = same_pads(H, k, stride)
    ow, pl, pr = same_pads(Wd, k, stride)
    pad = [(0, 0)] * (x.ndim - 3) + [(pt, pb), (pl, pr), (0, 0)]
    xp = np.pad(x, pad)
    out = np.zeros(x.shape[:-3] + (oh, ow, W.shape[3]))
    for ky in range(k):
        for kx in range(k):
            sl = xp[..., ky:ky + (oh - 1) * stride + 1:stride, kx:kx + (ow - 1) * stride + 1:stride, :]
            out += sl @ W[ky, kx]
    return out if b is None else out + b


def batch_norm(x, w: dict, name: str):
    g, be, m, v = (w[f"{name}/{k}"] for k in ("gamma", "beta", "moving_mean", "moving_variance"))
    return (x - m) / np.sqrt(v + BN_EPS) * g + be


def resize_bilinear(x: np.ndarray, oh: int, ow: int) -> np.ndarray:
    """TF1 tf.image.resize_images (bilinear, align_corners=False, half_pixel_centers=False) on [H, W, C]: src = dst * in / out, lower =
    floor, upper = min(ceil, in - 1), top and bottom lerped in x, then y."""
    H, W = x.shape[:2]

    def axis(o, n):
        src = np.arange(o) * (n / o)
        lo = np.floor(src).astype(np.int64)
        hi = np.minimum(np.ceil(src).astype(np.int64), n - 1)
        return lo, hi, src - lo
    y0, y1, fy = axis(oh, H)
    x0, x1, fx = axis(ow, W)
    fx = fx[None, :, None]
    top = x[y0][:, x0] + (x[y0][:, x1] - x[y0][:, x0]) * fx
    bot = x[y1][:, x0] + (x[y1][:, x1] - x[y1][:, x0]) * fx
    return top + (bot - top) * fy[:, None, None]


def instance_norm(x: np.ndarray) -> np.ndarray:
    """det_tools.py:789-803 on one [H, W, C] map: moments over H, W; epsilon 1e-3."""
    m = x.mean(axis=(0, 1), keepdims=True)
    v = ((x - m) ** 2).mean(axis=(0, 1), keepdims=True)
    return (x - m) / np.sqrt(v + IN_EPS)


def box(x: np.ndarray, r: int, op) -> np.ndarray:
    """op (np.max or np.sum) over the (2r+1)^2 window of each pixel of [H, W], clipped at the border: SAME max pooling ignores the
    padding, a SAME sum convolution pads zeros.  Taken as a pass along x, then one along y (the same window)."""
    fill = -np.inf if op is np.max else 0.0
    for axis in (1, 0):
        n = x.shape[axis]
        pad = [(0, 0), (0, 0)]
        pad[axis] = (r, r)
        xp = np.pad(x, pad, constant_values=fill)
        x = op(np.stack([np.take(xp, np.arange(d, d + n), axis=axis) for d in range(2 * r + 1)]), axis=0)
    return x


def random_weights(shapes: dict, seed: int) -> dict:
    """Seeded weights for the TF variables `shapes` (name -> shape): Glorot-scaled normal kernels, small biases, and BN statistics
    away from the identity (gamma in [0.5, 1.5], beta and moving_mean N(0, 0.1), moving_variance in [0.5, 2])."""
    rng = np.random.default_rng(seed)
    out = {}
    for name, shp in shapes.items():
        leaf = name.rsplit("/", 1)[1]
        if leaf == "weights":
            fan_in, fan_out = int(np.prod(shp[:-1])), int(np.prod(shp[:-2]) * shp[-1]) if len(shp) == 4 else shp[-1]
            v = rng.normal(0.0, np.sqrt(2.0 / (fan_in + fan_out)), shp)
        elif leaf == "biases":
            v = rng.normal(0.0, 0.05, shp)
        elif leaf == "gamma":
            v = rng.uniform(0.5, 1.5, shp)
        elif leaf == "moving_variance":
            v = rng.uniform(0.5, 2.0, shp)
        else:
            v = rng.normal(0.0, 0.1, shp)
        out[name] = v.astype(np.float32)
    return out


def soft_nms_3d(scale_logits: np.ndarray, ksize: int, com: float) -> np.ndarray:
    """det_tools.py:772-787 on [H, W, S]: the 3-D max pool and box sum span all scales (depth kernel = stride = S), so both are 2-D
    windows of ksize over the scale-wise max / sum; the + 1e-6 stays."""
    r = ksize // 2
    max_maps = box(scale_logits.max(axis=-1), r, np.max)[..., None]
    exp_maps = np.exp(com * (scale_logits - max_maps))
    sum_ex = box(exp_maps.sum(axis=-1), r, np.sum)[..., None]
    return exp_maps / (sum_ex + 1e-6)


def soft_max_and_argmax_1d(x: np.ndarray, index: np.ndarray, c1: float, c2: float):
    """det_tools.py:1707-1725 over the last axis."""
    m = x.max(axis=-1, keepdims=True)
    e1 = np.exp(c1 * (x - m))
    s1 = e1 / (e1.sum(axis=-1, keepdims=True) + 1e-8)
    e2 = np.exp(c2 * (x - m))
    s2 = e2 / (e2.sum(axis=-1, keepdims=True) + 1e-8)
    return (x * s1).sum(axis=-1), (index * s2).sum(axis=-1)


def eof_mask(H: int, W: int, radius: int) -> np.ndarray:
    m = np.zeros((H, W))
    m[radius:H - radius, radius:W - radius] = 1.0
    return m


def non_max_suppression(x: np.ndarray, thresh: float, ksize: int) -> np.ndarray:
    """det_tools.py:806-834 on [H, W]: values below thresh become 0, zero padding, the centre strictly greater than all other ksize^2 - 1."""
    hk = ksize // 2
    works = np.where(x < thresh, 0.0, x)
    H, W = x.shape
    wp = np.pad(works, hk)
    peak = np.ones((H, W), bool)
    for dy in range(ksize):
        for dx in range(ksize):
            if dy == hk and dx == hk:
                continue
            peak &= works > wp[dy:dy + H, dx:dx + W]
    return peak.astype(np.float64)


def top_k_map(scores: np.ndarray, k: int) -> np.ndarray:
    """make_top_k_sparse_tensor (det_tools.py:848-861): 1 at the k largest scores.  Ties at the k-th value (the zero fill included) go
    to the lower flat index: TF's own order among equal values is not specified."""
    flat = scores.reshape(-1)
    idx = np.argsort(-flat, kind="stable")[:k]
    out = np.zeros(flat.shape)
    out[idx] = 1.0
    return out.reshape(scores.shape)


def linspace_grid(n: int):
    t = np.linspace(-1.0, 1.0, n)
    return np.meshgrid(t, t)          # x varies along columns, y along rows (spatial_transformer.py:11-14)


def transformer_crop(img: np.ndarray, out: int, kpts: np.ndarray, scale: np.ndarray, ori=None) -> np.ndarray:
    """spatial_transformer.py:23-139 for one image [H, W, C]: per keypoint the out x out grid on [-1, 1]^2, through theta = scale
    (R(cos, sin) when ori is given), times out / 2, plus the keypoint; bilinear with floor / +1 corners clipped to the image and the
    weights taken from the clipped corners."""
    H, W = img.shape[:2]
    xt, yt = linspace_grid(out)
    s = scale[:, None, None]
    if ori is None:
        c, sn = np.ones_like(s), np.zeros_like(s)
    else:
        c, sn = ori[:, 0][:, None, None], ori[:, 1][:, None, None]
    x = (s * c * xt + s * -sn * yt) * out / 2.0 + kpts[:, 0][:, None, None]
    y = (s * sn * xt + s * c * yt) * out / 2.0 + kpts[:, 1][:, None, None]
    x0 = np.floor(x).astype(np.int64)
    y0 = np.floor(y).astype(np.int64)
    x1, y1 = np.clip(x0 + 1, 0, W - 1), np.clip(y0 + 1, 0, H - 1)
    x0, y0 = np.clip(x0, 0, W - 1), np.clip(y0, 0, H - 1)
    wa = ((x1 - x) * (y1 - y))[..., None]
    wb = ((x1 - x) * (y - y0))[..., None]
    wc = ((x - x0) * (y1 - y))[..., None]
    wd = ((x - x0) * (y - y0))[..., None]
    return wa * img[y0, x0] + wb * img[y1, x0] + wc * img[y0, x1] + wd * img[y1, x1]


def soft_argmax_2d(patches: np.ndarray, com: float) -> np.ndarray:
    """det_tools.py:1727-1750 with do_softmax: [N, n, n] -> [N, 2] (dx, dy) on the patch's [-1, 1] grid."""
    n = patches.shape[1]
    xt, yt = linspace_grid(n)
    e = np.exp(com * (patches - patches.max(axis=(1, 2), keepdims=True)))
    sm = e / (e.sum(axis=(1, 2), keepdims=True) + 1e-8)
    return np.stack([(xt * sm).sum(axis=(1, 2)), (yt * sm).sum(axis=(1, 2))], axis=1)


def l2_normalize(x: np.ndarray, axis: int = -1) -> np.ndarray:
    """tf.nn.l2_normalize: x / sqrt(max(sum x^2, 1e-12))."""
    return x / np.sqrt(np.maximum((x * x).sum(axis=axis, keepdims=True), 1e-12))


# ---- the network ------------------------------------------------------------------------------------------------------------------------

def scale_factors(cfg) -> np.ndarray:
    n = cfg["net_num_scales"]
    if n == 1:
        return np.array([1.0])
    return np.exp(np.linspace(np.log(cfg["net_max_scale"]), np.log(cfg["net_min_scale"]), n))     # mso_resnet_detector.py:106-110


def scale_sizes(cfg, side: int = SIDE) -> list:
    """int(base * inv_s + 0.5) with base and inv_s as float32 (mso_resnet_detector.py:126-132)."""
    return [int(np.float32(side) * np.float32(1.0 / s) + np.float32(0.5)) for s in scale_factors(cfg)]


def trunk(x: np.ndarray, w: dict, cfg) -> np.ndarray:
    """mso_resnet_detector.get_model up to feat_maps (lines 81-104): init conv, pre-activation residual blocks, fin-bn + activation."""
    a = cfg["leaky_alpha"]
    p = "ConvOnlyResNet"
    cur = conv2d(x, w[f"{p}/init_conv/weights"], w[f"{p}/init_conv/biases"])
    for i in range(1, cfg["net_block"] + 1):
        b = f"{p}/block-{i}"
        t = leaky_relu(batch_norm(cur, w, f"{b}/pre-bn"), a)
        t = conv2d(t, w[f"{b}/conv1/weights"], w[f"{b}/conv1/biases"])
        t = leaky_relu(batch_norm(t, w, f"{b}/mid-bn"), a)
        cur = conv2d(t, w[f"{b}/conv2/weights"], w[f"{b}/conv2/biases"]) + cur
    return leaky_relu(batch_norm(cur, w, f"{p}/fin-bn"), a)


def descriptor(patches: np.ndarray, w: dict, cfg) -> np.ndarray:
    """simple_desc.get_model (lines 28-56): stride-2 SAME convs + BN + ReLU, flatten (HWC), fc1 + BN + ReLU, fc2, l2norm."""
    cur = patches
    for i in range(1, cfg["desc_net_depth"] + 1):
        cur = conv2d(cur, w[f"SimpleDesc/conv{i}/weights"], w[f"SimpleDesc/conv{i}/biases"], stride=2)
        cur = np.maximum(batch_norm(cur, w, f"SimpleDesc/bn{i}"), 0.0)
    cur = cur.reshape(len(cur), -1)
    cur = cur @ w["SimpleDesc/fc1/weights"] + w["SimpleDesc/fc1/biases"]
    cur = np.maximum(batch_norm(cur, w, "SimpleDesc/fc-bn1"), 0.0)
    raw = cur @ w["SimpleDesc/fc2/weights"] + w["SimpleDesc/fc2/biases"]
    return l2_normalize(raw, axis=1)


def detect(request: np.ndarray, w: dict, cfg) -> dict:
    """The whole graph on one 400 x 400 x 3 request.  Returns every intermediate: photo, feat (trunk features), logits (per scale, before
    the instance norm), scale_logits, max_heatmaps, max_scales, nms_maps, nms_scores, kpts_int, kpts_scale, ori, kpts (refined), patches,
    desc."""
    o = {}
    x = photo(request)
    o["photo"] = x[..., 0]
    H, W = x.shape[:2]
    # input_inst_norm's photos1 is computed and never used (run_server.py:33-37): nothing to do
    feat = trunk(x, w, cfg)
    o["feat"] = feat
    sf = scale_factors(cfg)
    k = cfg["conv_ksize"]
    logits, up = [], []
    for i, S in enumerate(scale_sizes(cfg, H)):
        lg = conv2d(resize_bilinear(feat, S, S), w[f"ConvOnlyResNet/score_conv_{i}/weights"], w[f"ConvOnlyResNet/score_conv_{i}/biases"])
        logits.append(lg[..., 0])
        up.append(resize_bilinear(instance_norm(lg), H, W)[..., 0])     # inference.py:176-180
    o["logits"] = logits
    scale_logits = np.stack(up, axis=-1)
    o["scale_logits"] = scale_logits
    heat = soft_nms_3d(scale_logits, cfg["sm_ksize"], cfg["com_strength"])
    mh, ms = soft_max_and_argmax_1d(heat, sf.astype(np.float32).astype(np.float64), cfg["score_com_strength"], cfg["scale_com_strength"])
    # pad_size = num_conv * (ksize // 2): the init conv, two per block and the score conv (mso_resnet_detector.py:85,96,139,171)
    pad = (2 + 2 * cfg["net_block"]) * (k // 2)
    mh = mh * eof_mask(H, W, pad)
    o["max_heatmaps"], o["max_scales"] = mh, ms
    nms = non_max_suppression(mh, cfg["nms_thresh"], cfg["nms_ksize"])
    scores = mh * nms * eof_mask(H, W, cfg["crop_radius"])
    o["nms_maps"], o["nms_scores"] = nms, scores
    top = top_k_map(scores, cfg["top_k"]) * nms                           # inference.py:208-209
    ys, xs = np.nonzero(top > 0)                                          # tf.where: row-major
    kint = np.stack([xs, ys], axis=1)
    o["kpts_int"] = kint
    ks = ms[ys, xs]
    o["kpts_scale"] = ks
    # ori_conv (mso_resnet_detector.py:144-148) only where it is gathered
    Wo, bo = w["ConvOnlyResNet/ori_conv/weights"], w["ConvOnlyResNet/ori_conv/biases"]
    r = Wo.shape[0] // 2
    fp = np.pad(feat, ((r, r), (r, r), (0, 0)))
    ori = np.stack([np.einsum("ijc,ijco->o", fp[y:y + 2 * r + 1, x:x + 2 * r + 1], Wo) + bo for x, y in kint]) if len(kint) else np.zeros((0, 2))
    ori = l2_normalize(ori, axis=1)
    o["ori"] = ori
    loc = cfg["kp_loc_size"]
    crops = transformer_crop(mh[..., None], loc, kint.astype(np.float64), ks)[..., 0]
    dxdy = soft_argmax_2d(crops, cfg["kp_com_strength"])
    kpts = kint + dxdy * ks[:, None] * loc / 2                            # inference.py:230
    o["kpts"] = kpts
    patches = transformer_crop(x, cfg["patch_size"], kpts, ks, ori)
    o["patches"] = patches[..., 0]
    o["desc"] = descriptor(patches, w, cfg) if len(kpts) else np.zeros((0, cfg["desc_dim"]))
    return o
