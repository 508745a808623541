"""LF-Net on the device: the feature server of Lfnet::detectFeature (lf-net-release/run_server.py) as a library call, no TensorFlow.

load_lfnet(model_dir) reads a released model's config.pkl and weights.npz (scripts/lfnet_export_weights.py makes the latter from a TF
checkpoint) and returns an LfnetDevice, a feature source run_sequence drives on the device: the request image never leaves the GPU and
the descriptors go straight to the tracker.  write_weights_file turns the same directory into one weights file that bt_lfnet_load_file
(LfnetDevice.from_file, the C++ LfnetGpu, scripts/lfnet_server.py) loads without Python.  DESIGN.md §3.12."""
from __future__ import annotations

import ctypes
import io
import os
import pickle

import numpy as np

from . import _lib

SIDE = 400
FC_HIDDEN = 512          # simple_desc.py:44
BN_EPS = 1e-5            # tf.layers.batch_normalization as tf_layer_utils.py:185 calls it

# train_lfnet.py:1051-1189 at its defaults, and run_server.py's --top_k: the numeric hyper-parameters bt_lfnet_params carries
DEFAULTS = dict(top_k=500, net_channel=16, net_block=3, conv_ksize=5, net_num_scales=5, net_min_scale=1.0 / np.sqrt(2), net_max_scale=np.sqrt(2),
                leaky_alpha=0.2, sm_ksize=15, com_strength=3.0, score_com_strength=100.0, scale_com_strength=100.0, kp_loc_size=9,
                kp_com_strength=1.0, nms_ksize=5, nms_thresh=0.0, crop_radius=16, patch_size=32, desc_net_channel=64, desc_net_depth=3,
                desc_conv_ksize=3, desc_dim=256)
# the network the kernels implement: any other value of these keys is refused by name
REQUIRED = dict(detector="mso_resnet_detector", descriptor="simple_desc", desc_inputs="photos", desc_norm="l2norm", activ_fn="leaky_relu",
                desc_activ_fn="relu", perform_bn=True, desc_perform_bn=True, use_nms3d=True, soft_scale=True, soft_kpts=True,
                do_softmax_kp_refine=True, use_bias=True, bn_affine=True)


class _ConfigUnpickler(pickle.Unpickler):
    """config.pkl holds an argparse.Namespace of plain values.  train_lfnet.py's scale defaults are numpy floats (np.sqrt(2),
    train_lfnet.py:1133-1136), which pickle as numpy scalars, so those are allowed too; any other class is refused."""
    ALLOWED = {("argparse", "Namespace"), ("numpy", "dtype"), ("numpy.core.multiarray", "scalar"), ("numpy._core.multiarray", "scalar")}

    def find_class(self, module, name):
        if (module, name) not in self.ALLOWED:
            raise pickle.UnpicklingError(f"config.pkl names {module}.{name}: only argparse.Namespace and plain values are read")
        return super().find_class(module, name)


def read_config(path: str) -> dict:
    with open(path, "rb") as f:
        ns = _ConfigUnpickler(io.BytesIO(f.read())).load()
    if not hasattr(ns, "__dict__"):
        raise ValueError(f"{path}: not an argparse.Namespace")
    return dict(vars(ns))


def check_config(cfg: dict, top_k: int = 500) -> dict:
    """The hyper-parameters of cfg (config.pkl's keys) as a dict of DEFAULTS' keys.  top_k is run_server.py's --top_k, which replaces the
    training value (run_server.py:99-106).  A key the network depends on that is missing, or a REQUIRED key with another value, raises
    ValueError naming the key."""
    for k, want in REQUIRED.items():
        if k not in cfg:
            if k in ("use_bias", "bn_affine"):          # read with getattr defaults True (mso_resnet_detector.py:184-187)
                continue
            raise ValueError(f"config key {k!r} is missing; the network here needs {k} = {want!r}")
        got = cfg[k]
        ok = (isinstance(got, (bool, np.bool_)) and bool(got) == want) if isinstance(want, bool) else got == want
        if not ok:
            raise ValueError(f"config key {k!r} = {got!r} is not supported: only {want!r} is implemented")
    out = {}
    for k, dflt in DEFAULTS.items():
        if k == "top_k":
            out[k] = int(top_k)
            continue
        if k not in cfg:
            raise ValueError(f"config key {k!r} is missing")
        v = cfg[k]
        if isinstance(dflt, int):
            if int(v) != v:
                raise ValueError(f"config key {k!r} = {v!r} is not an integer")
            v = int(v)
        else:
            v = float(v)
        out[k] = v
    return out


def params_struct(hp: dict) -> "_lib.LfnetParams":
    p = _lib.LfnetParams()
    for k, v in hp.items():
        setattr(p, k, v)
    return p


def weight_shapes(hp: dict) -> dict:
    """Every TF variable the network reads (name -> shape), as build_networks creates them."""
    k, C = hp["conv_ksize"], hp["net_channel"]
    s = {"ConvOnlyResNet/init_conv/weights": (k, k, 1, C), "ConvOnlyResNet/init_conv/biases": (C,)}
    bn = ("gamma", "beta", "moving_mean", "moving_variance")

    def add_bn(name, n):
        for v in bn:
            s[f"{name}/{v}"] = (n,)
    for i in range(1, hp["net_block"] + 1):
        b = f"ConvOnlyResNet/block-{i}"
        add_bn(f"{b}/pre-bn", C)
        s[f"{b}/conv1/weights"], s[f"{b}/conv1/biases"] = (k, k, C, C), (C,)
        add_bn(f"{b}/mid-bn", C)
        s[f"{b}/conv2/weights"], s[f"{b}/conv2/biases"] = (k, k, C, C), (C,)
    add_bn("ConvOnlyResNet/fin-bn", C)
    for i in range(hp["net_num_scales"]):
        s[f"ConvOnlyResNet/score_conv_{i}/weights"], s[f"ConvOnlyResNet/score_conv_{i}/biases"] = (k, k, C, 1), (1,)
    s["ConvOnlyResNet/ori_conv/weights"], s["ConvOnlyResNet/ori_conv/biases"] = (k, k, C, 2), (2,)
    h, cin, kd = hp["patch_size"], 1, hp["desc_conv_ksize"]
    for i in range(1, hp["desc_net_depth"] + 1):
        cout = hp["desc_net_channel"] * 2 ** (i - 1)
        s[f"SimpleDesc/conv{i}/weights"], s[f"SimpleDesc/conv{i}/biases"] = (kd, kd, cin, cout), (cout,)
        add_bn(f"SimpleDesc/bn{i}", cout)
        h, cin = -(-h // 2), cout
    s["SimpleDesc/fc1/weights"], s["SimpleDesc/fc1/biases"] = (h * h * cin, FC_HIDDEN), (FC_HIDDEN,)
    add_bn("SimpleDesc/fc-bn1", FC_HIDDEN)
    s["SimpleDesc/fc2/weights"], s["SimpleDesc/fc2/biases"] = (FC_HIDDEN, hp["desc_dim"]), (hp["desc_dim"],)
    return s


def make_blob(weights: dict, hp: dict) -> np.ndarray:
    """The float32 blob bt_lfnet_load_weights takes (layout: include/bundletrack_b200.h) from the TF variables.  Every variable must be
    present with its shape (a missing key or a wrong shape raises ValueError naming it); BN is folded in float64 and rounded once."""
    shapes = weight_shapes(hp)
    w = {}
    for name, shp in shapes.items():
        if name not in weights:
            raise ValueError(f"weight {name!r} is missing")
        a = np.asarray(weights[name], np.float64)
        if a.shape != shp:
            raise ValueError(f"weight {name!r} has shape {a.shape}, the network needs {shp}")
        if not np.isfinite(a).all():
            raise ValueError(f"weight {name!r} has non-finite values")
        w[name] = a

    def bn(name, bias=None):
        s = w[f"{name}/gamma"] / np.sqrt(w[f"{name}/moving_variance"] + BN_EPS)
        t = w[f"{name}/beta"] - w[f"{name}/moving_mean"] * s
        return [s, t if bias is None else t + bias * s]
    parts = [w["ConvOnlyResNet/init_conv/weights"], w["ConvOnlyResNet/init_conv/biases"]]
    for i in range(1, hp["net_block"] + 1):
        b = f"ConvOnlyResNet/block-{i}"
        parts += bn(f"{b}/pre-bn") + [w[f"{b}/conv1/weights"], w[f"{b}/conv1/biases"]]
        parts += bn(f"{b}/mid-bn") + [w[f"{b}/conv2/weights"], w[f"{b}/conv2/biases"]]
    parts += bn("ConvOnlyResNet/fin-bn")
    for i in range(hp["net_num_scales"]):
        parts += [w[f"ConvOnlyResNet/score_conv_{i}/weights"], w[f"ConvOnlyResNet/score_conv_{i}/biases"]]
    parts += [w["ConvOnlyResNet/ori_conv/weights"], w["ConvOnlyResNet/ori_conv/biases"]]
    for i in range(1, hp["desc_net_depth"] + 1):
        parts += [w[f"SimpleDesc/conv{i}/weights"]] + bn(f"SimpleDesc/bn{i}", w[f"SimpleDesc/conv{i}/biases"])
    parts += [w["SimpleDesc/fc1/weights"]] + bn("SimpleDesc/fc-bn1", w["SimpleDesc/fc1/biases"])
    parts += [w["SimpleDesc/fc2/weights"], w["SimpleDesc/fc2/biases"]]
    blob = np.concatenate([p.reshape(-1) for p in parts]).astype(np.float32)
    n = ctypes.c_size_t(0)
    _lib.check(_lib.load().bt_lfnet_weights_size(ctypes.byref(params_struct(hp)), ctypes.byref(n)), "bt_lfnet_weights_size")
    assert blob.size == n.value, (blob.size, n.value)
    return blob


def read_weights(path: str) -> dict:
    with np.load(path, allow_pickle=False) as z:
        return {k: z[k] for k in z.files}


FILE_MAGIC = b"BTLFNETW"
FILE_VERSION = 1


def weights_file_bytes(blob: np.ndarray, hp: dict) -> bytes:
    """The weights file bt_lfnet_load_file reads (layout: include/bundletrack_b200.h): magic, version, sizeof(bt_lfnet_params), the params
    struct and the float count, then the blob."""
    p = params_struct(hp)
    blob = np.ascontiguousarray(blob, np.float32)
    return (FILE_MAGIC + np.array([FILE_VERSION, ctypes.sizeof(p)], "<u4").tobytes() + bytes(p) + np.array([blob.size], "<u8").tobytes()
            + blob.astype("<f4").tobytes())


def write_weights_file(model_dir: str, out_path: str, top_k: int = 500) -> dict:
    """A released model directory (config.pkl + weights.npz, as load_lfnet reads it) as one weights file any host can load with
    bt_lfnet_load_file, BN folded as make_blob folds it.  Returns the hyper-parameters written."""
    hp = check_config(read_config(os.path.join(model_dir, "config.pkl")), top_k)
    data = weights_file_bytes(make_blob(read_weights(os.path.join(model_dir, "weights.npz")), hp), hp)
    with open(out_path, "wb") as f:
        f.write(data)
    return hp


def file_info(path: str) -> tuple:
    """(hyper-parameters, float count) of a weights file, checked as bt_lfnet_load_file checks it (no GPU)."""
    p, n = _lib.LfnetParams(), ctypes.c_size_t(0)
    _lib.check(_lib.load().bt_lfnet_file_info(os.fsencode(path), ctypes.byref(p), ctypes.byref(n)), "bt_lfnet_file_info")
    return {f: getattr(p, f) for f, _ in p._fields_}, n.value


class LfnetDevice(_lib.Facade):
    """The LF-Net server's network on the device.  detect() runs a batch of request images (bt_lfnet_request's output) in one call;
    as a run_sequence feature source (on_device) it hands the tracker host keypoints in image pixels and the device descriptors.
    LfnetDevice.from_file loads a weights file instead of TF variables."""
    on_device = True

    def __init__(self, weights: dict, hp: dict, max_images: int = 1, device: int = 0, stream: int = 0, ctx=None, _file: str = None):
        super().__init__(ctx, device, stream)
        if _file is None:
            self.hp = dict(hp)
            self.params = params_struct(self.hp)
            blob = make_blob(weights, self.hp)
            _lib.check(self.lib.bt_lfnet_reserve(self.ctx, ctypes.byref(self.params), max_images), "bt_lfnet_reserve")
            _lib.check(self.lib.bt_lfnet_load_weights(self.ctx, _lib.ptr(blob), blob.size), "bt_lfnet_load_weights")
        else:
            self.params = _lib.LfnetParams()
            _lib.check(self.lib.bt_lfnet_load_file(self.ctx, os.fsencode(_file), max_images, ctypes.byref(self.params)), "bt_lfnet_load_file")
            self.hp = {f: getattr(self.params, f) for f, _ in self.params._fields_}
        import torch
        self.max_images = max_images
        dev = torch.device("cuda", device)
        K, D = self.hp["top_k"], self.hp["desc_dim"]
        self.kpts = torch.empty((max_images, K, 2), dtype=torch.float32, device=dev)
        self.desc = torch.empty((max_images, K, D), dtype=torch.float32, device=dev)
        self.n = torch.empty((max_images,), dtype=torch.int32, device=dev)
        self._host = torch.empty((K * 2 + 1,), dtype=torch.float32, pin_memory=True)

    @classmethod
    def from_file(cls, path: str, max_images: int = 1, device: int = 0, stream: int = 0, ctx=None) -> "LfnetDevice":
        """The network of a weights file (write_weights_file), loaded by bt_lfnet_load_file: the same device state as the constructor
        makes from the TF variables the file was written from."""
        return cls(None, None, max_images, device, stream, ctx, _file=path)

    def detect(self, requests, stream=None):
        """requests: device uint8 [400, 400, 3] tensors.  Enqueues one bt_lfnet_detect on `stream` (default: the facade's) and returns
        views (kpts [n, top_k, 2], desc [n, top_k, desc_dim], n_kpts [n]) of this object's output buffers, valid until the next call."""
        n = len(requests)
        st = self.stream if stream is None else ctypes.c_void_p(stream)
        for r in requests:
            if tuple(r.shape) != (SIDE, SIDE, 3) or not r.is_cuda or not r.is_contiguous():
                raise ValueError(f"a request must be a contiguous CUDA uint8 tensor of shape ({SIDE}, {SIDE}, 3), got {tuple(r.shape)}")
        _lib.check(self.lib.bt_lfnet_detect(self.ctx, n, _lib.ptrs(requests), _lib.ptr(self.kpts), _lib.ptr(self.desc), _lib.ptr(self.n), st),
                   "bt_lfnet_detect")
        return self.kpts[:n], self.desc[:n], self.n[:n]

    def features_on_device(self, id_str: str, request, roi, stream: int):
        """run_sequence's device feature source: one request on `stream`.  Returns (kpts [n, 2] float32 host, image pixels through
        policy.lfnet_reply_keypoints, desc [n, desc_dim] device view); zero keypoints raise DetectionFailed."""
        import torch
        from . import policy
        from .sequence import DetectionFailed
        kp, de, nk = self.detect([request], stream)
        K = self.hp["top_k"]
        with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
            self._host[:2 * K].copy_(kp[0].reshape(-1), non_blocking=True)
            self._host[2 * K:].view(torch.int32).copy_(nk, non_blocking=True)
        _lib.check(self.lib.bt_stream_sync(ctypes.c_void_p(stream)), "bt_stream_sync")
        n = int(self._host[2 * K:].view(torch.int32).item())
        if n == 0:
            raise DetectionFailed(f"frame {id_str}: LF-Net found no keypoints")
        xy = self._host[:2 * n].numpy()
        kpts = policy.lfnet_reply_keypoints(n, self.hp["desc_dim"], xy, roi)
        return kpts, de[0, :n]


def load_lfnet(model_dir: str, top_k: int = 500, max_images: int = 1, device: int = 0, stream: int = 0) -> LfnetDevice:
    """A released model directory (config.pkl + weights.npz) as an LfnetDevice.  The config must describe the network run_server.py
    builds at train_lfnet.py's defaults (check_config); weights.npz holds the TF variables by name (scripts/lfnet_export_weights.py)."""
    hp = check_config(read_config(os.path.join(model_dir, "config.pkl")), top_k)
    return LfnetDevice(read_weights(os.path.join(model_dir, "weights.npz")), hp, max_images=max_images, device=device, stream=stream)
