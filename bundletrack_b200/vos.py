"""Object masks on the device: transductive-vos.pytorch's run_video.py (resnet50) as library calls, no PyTorch network.

load_vos(path, params) reads the checkpoint run_video.py --resume takes and returns a VosDevice: begin() takes frame 0 and its mask,
next() propagates that mask to each later frame, and both write uint8 0 / 255 masks on the device; labels() gives the last frame's label
map, the initial mask's values per pixel.  DESIGN.md §3.13, §3.17."""
from __future__ import annotations

import ctypes
import os
import queue
import threading

import numpy as np

from . import _lib

BN_EPS = 1e-5
LAYERS = ((3, 64, 1), (4, 128, 2), (6, 256, 1), (3, 256, 1))     # blocks, planes, stride of layer1..layer4 (layer3, layer4 at stride 1)
DEFAULTS = dict(ref_num=9, range=40, sigma1=8.0, sigma2=21.0, temperature=1.0)
MAX_LABELS = 8


def params_struct(p: dict) -> "_lib.VosParams":
    return _lib.VosParams(int(p["ref_num"]), int(p["range"]), float(p["sigma1"]), float(p["sigma2"]), float(p["temperature"]))


def conv_order() -> list:
    """(conv weight name, BN prefix) of every conv in the blob's order (include/bundletrack_b200.h)."""
    out = [("backbone.0.weight", "backbone.1")]
    inp = 64
    for li, (n, planes, stride) in enumerate(LAYERS):
        for b in range(n):
            p = f"backbone.{4 + li}.{b}"
            out += [(f"{p}.conv1.weight", f"{p}.bn1"), (f"{p}.conv2.weight", f"{p}.bn2"), (f"{p}.conv3.weight", f"{p}.bn3")]
            if b == 0 and (stride != 1 or inp != 4 * planes):
                out.append((f"{p}.downsample.0.weight", f"{p}.downsample.1"))
            inp = 4 * planes
    out.append(("adjust_dim.weight", "bn256"))
    return out


def state_shapes() -> dict:
    """name -> shape of every tensor the network reads from VOSNet('resnet50')'s state dict."""
    s = {}
    inp = 64
    shapes = {"backbone.0.weight": (64, 3, 7, 7)}
    for li, (n, planes, stride) in enumerate(LAYERS):
        for b in range(n):
            p = f"backbone.{4 + li}.{b}"
            shapes[f"{p}.conv1.weight"] = (planes, inp, 1, 1)
            shapes[f"{p}.conv2.weight"] = (planes, planes, 3, 3)
            shapes[f"{p}.conv3.weight"] = (4 * planes, planes, 1, 1)
            if b == 0 and (stride != 1 or inp != 4 * planes):
                shapes[f"{p}.downsample.0.weight"] = (4 * planes, inp, 1, 1)
            inp = 4 * planes
    shapes["adjust_dim.weight"] = (256, 1024, 1, 1)
    for w, bn in conv_order():
        s[w] = shapes[w]
        for v in ("weight", "bias", "running_mean", "running_var"):
            s[f"{bn}.{v}"] = (shapes[w][0],)
    return s


def _variant(keys) -> str | None:
    """The resnet a state dict's keys come from when it is not resnet50: BasicBlock layers (resnet18 / 34) have no conv3, resnet101 has a
    23-block layer3."""
    if any(k.startswith("backbone.4.0.conv2.") for k in keys) and not any(k.startswith("backbone.4.0.conv3.") for k in keys):
        return "resnet18 or resnet34 (BasicBlock)"
    if any(k.startswith("backbone.6.6.") for k in keys):
        return "resnet101"
    return None


def read_checkpoint(path: str) -> dict:
    """The state dict of a run_video.py --resume checkpoint (main.py saves {'epoch', 'state_dict', 'optimizer', 'scheduler'}; a bare state
    dict is taken too), as float64 numpy arrays by name without DataParallel's module. prefix.  Read with weights_only=True.  A missing
    key, an unexpected key or a wrong shape raises ValueError naming it; another resnet is refused by name."""
    import torch
    ck = torch.load(path, map_location="cpu", weights_only=True)
    sd = ck["state_dict"] if isinstance(ck, dict) and "state_dict" in ck else ck
    if not isinstance(sd, dict):
        raise ValueError(f"{path}: no state_dict")
    sd = {(k[len("module."):] if k.startswith("module.") else k): v for k, v in sd.items() if not k.endswith("num_batches_tracked")}
    v = _variant(sd)
    if v is not None:
        raise ValueError(f"{path}: a {v} checkpoint; only --model resnet50 is implemented")
    shapes = state_shapes()
    for k in sorted(shapes):
        if k not in sd:
            raise ValueError(f"{path}: key {k!r} is missing")
        if tuple(sd[k].shape) != shapes[k]:
            raise ValueError(f"{path}: key {k!r} has shape {tuple(sd[k].shape)}, resnet50's VOSNet has {shapes[k]}")
    extra = sorted(set(sd) - set(shapes))
    if extra:
        raise ValueError(f"{path}: unexpected key {extra[0]!r}" + (f" and {len(extra) - 1} more" if len(extra) > 1 else ""))
    return {k: sd[k].double().numpy() for k in shapes}


def make_blob(sd: dict) -> np.ndarray:
    """The float32 blob bt_vos_load_weights takes from read_checkpoint's arrays: per conv W[co][ky][kx][ci], then BN scale and shift
    folded in float64 and rounded once."""
    parts = []
    for w, bn in conv_order():
        scale = sd[f"{bn}.weight"] / np.sqrt(sd[f"{bn}.running_var"] + BN_EPS)
        shift = sd[f"{bn}.bias"] - sd[f"{bn}.running_mean"] * scale
        parts += [np.transpose(sd[w], (0, 2, 3, 1)), scale, shift]
    blob = np.concatenate([p.reshape(-1) for p in parts]).astype(np.float32)
    n = ctypes.c_size_t(0)
    _lib.check(_lib.load().bt_vos_weights_size(ctypes.byref(params_struct(DEFAULTS)), ctypes.byref(n)), "bt_vos_weights_size")
    assert blob.size == n.value, (blob.size, n.value)
    if not np.isfinite(blob).all():
        raise ValueError("the checkpoint has non-finite weights")
    return blob


def schedule(k: int, ref_num: int, rng: int) -> list:
    """The history frames frame k reads (bt_vos_schedule)."""
    buf = (ctypes.c_int32 * max(ref_num, k))()
    n = ctypes.c_int(0)
    _lib.check(_lib.load().bt_vos_schedule(k, ref_num, rng, buf, ctypes.byref(n)), "bt_vos_schedule")
    return list(buf[:n.value])


class VosDevice(_lib.Facade):
    """The segmentation network and propagation on the device for H x W frames.  begin(colour, init_mask) starts a sequence, next(colour)
    gives each later frame's mask; colour is a CUDA uint8 H x W x 3 BGR tensor (cv2.imread's order), masks are CUDA uint8 H x W 0 / 255."""

    def __init__(self, sd: dict, params: dict, H: int, W: int, device: int = 0, stream: int = 0, ctx=None):
        super().__init__(ctx, device, stream)
        import torch
        self.params = dict(DEFAULTS, **params)
        self.H, self.W = H, W
        blob = make_blob(sd)
        _lib.check(self.lib.bt_vos_reserve(self.ctx, ctypes.byref(params_struct(self.params)), H, W), "bt_vos_reserve")
        _lib.check(self.lib.bt_vos_load_weights(self.ctx, _lib.ptr(blob), blob.size), "bt_vos_load_weights")
        self.device = torch.device("cuda", device)

    def _check(self, t, shape, what):
        import torch
        if tuple(t.shape) != shape or not t.is_cuda or t.dtype != torch.uint8 or not t.is_contiguous():
            raise ValueError(f"{what} must be a contiguous CUDA uint8 tensor of shape {shape} (the reserved size), got {tuple(t.shape)}")

    def _out(self, out):
        import torch
        if out is None:
            out = torch.empty((self.H, self.W), dtype=torch.uint8, device=self.device)
        self._check(out, (self.H, self.W), "the output mask")
        return out

    def begin(self, colour, init_mask, out=None, stream=None):
        """Frame 0: init_mask holds label values (H x W, or H x W x 3 whose channel 0 is taken); returns the mask with > 0 -> 255."""
        if init_mask.dim() == 3:
            init_mask = init_mask[..., 0].contiguous()
        self._check(colour, (self.H, self.W, 3), "colour")
        self._check(init_mask, (self.H, self.W), "init_mask")
        out = self._out(out)
        st = self.stream if stream is None else ctypes.c_void_p(stream)
        _lib.check(self.lib.bt_vos_begin(self.ctx, _lib.ptr(colour), _lib.ptr(init_mask), _lib.ptr(out), st), "bt_vos_begin")
        return out

    def next(self, colour, out=None, stream=None):
        """The next frame's mask, enqueued on `stream` (default: the facade's)."""
        self._check(colour, (self.H, self.W, 3), "colour")
        out = self._out(out)
        st = self.stream if stream is None else ctypes.c_void_p(stream)
        _lib.check(self.lib.bt_vos_next(self.ctx, _lib.ptr(colour), _lib.ptr(out), st), "bt_vos_next")
        return out

    def labels(self, out=None, stream=None):
        """The label map (CUDA uint8 H x W) of the last frame begin() or next() processed, enqueued on `stream`: the initial mask's value of
        each pixel's label channel, non-zero exactly where that frame's mask is 255; after begin(), the initial mask itself.  Call it before
        the next next() in stream order, which overwrites what it reads (bt_vos_labels)."""
        out = self._out(out)
        st = self.stream if stream is None else ctypes.c_void_p(stream)
        _lib.check(self.lib.bt_vos_labels(self.ctx, _lib.ptr(out), st), "bt_vos_labels")
        return out

    def enable_timing(self, on: bool = True) -> None:
        _lib.check(self.lib.bt_vos_enable_timing(self.ctx, int(on)), "bt_vos_enable_timing")

    def timing(self) -> dict:
        ms = (ctypes.c_float * 3)()
        _lib.check(self.lib.bt_vos_get_timing(self.ctx, ms), "bt_vos_get_timing")
        return dict(backbone=ms[0], propagation=ms[1], mask=ms[2])

    def debug(self, slot: int, stream=None) -> dict:
        """Ring slot `slot`'s features and label, the last next()'s low-resolution prediction, and the state (bt_vos_debug)."""
        info = (ctypes.c_int32 * 5)()
        _lib.check(self.lib.bt_vos_debug(self.ctx, 0, None, None, None, info, self.stream), "bt_vos_debug")
        Hd, Wd = info[3], info[4]
        feat = np.empty((Hd, Wd, 256), np.float32)
        label = np.empty((Hd, Wd, MAX_LABELS), np.float32)
        pred = np.empty((MAX_LABELS, Hd * Wd), np.float32)
        st = self.stream if stream is None else ctypes.c_void_p(stream)
        _lib.check(self.lib.bt_vos_debug(self.ctx, slot, _lib.ptr(feat), _lib.ptr(label), _lib.ptr(pred), info, st), "bt_vos_debug")
        return dict(feat=feat, label=label, pred=pred, frame=info[0], n_labels=info[1], slots=info[2], Hd=Hd, Wd=Wd)


def load_vos(path: str, params: dict | None = None, H: int = 480, W: int = 640, device: int = 0, stream: int = 0) -> VosDevice:
    """A run_video.py checkpoint (--resume) as a VosDevice for H x W frames; params: run_video.py's ref_num, range, sigma1, sigma2 and
    temperature (DEFAULTS for the ones not given)."""
    return VosDevice(read_checkpoint(path), params or {}, H, W, device=device, stream=stream)


def read_init_mask(path: str) -> np.ndarray:
    """run_video.py's --init_mask_file: cv2.imread(path, -1), channel 0 when it has three.  Label values are 8-bit: a 16-bit or float
    image is refused rather than wrapped."""
    import cv2
    m = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if m is None:
        raise ValueError(f"{path}: not an image")
    if m.ndim == 3:
        m = m[..., 0]
    if m.dtype != np.uint8:
        raise ValueError(f"{path}: {m.dtype} samples; the initial mask's label values must be 8-bit (uint8)")
    return np.ascontiguousarray(m)


def read_palette_mask(path: str) -> tuple:
    """(indices, palette) of a DAVIS annotation as lib/predict.py's prepare_first_frame reads it: PIL's palette indices (uint8 H x W) and the
    palette (uint8 [n, 3], None for an 8-bit grey PNG, whose samples are taken as indices).  Any other PNG mode is refused by name."""
    from PIL import Image
    with Image.open(path) as im:
        if im.mode not in ("P", "L"):
            raise ValueError(f"{path}: a mode {im.mode!r} image; object annotations must be palette (P) or 8-bit grey (L) PNGs")
        a = np.array(im, dtype=np.uint8)
        pal = im.getpalette() if im.mode == "P" else None
    if pal is not None:
        pal = np.asarray(pal, np.uint8).reshape(-1, 3)
    return np.ascontiguousarray(a), pal


def write_palette_mask(path: str, labels, palette) -> None:
    """lib/utils.py's save_prediction: labels (uint8 H x W) as a mode P PNG with `palette` (uint8 [n, 3] or a flat list of RGB bytes)."""
    from PIL import Image
    a = np.asarray(labels)
    if a.dtype != np.uint8 or a.ndim != 2:
        raise ValueError(f"{path}: labels must be uint8 H x W, got {a.dtype} {a.shape}")
    im = Image.fromarray(np.ascontiguousarray(a)).convert("L")
    im.putpalette(np.asarray(palette, np.uint8).reshape(-1).tolist())      # an L image with a palette becomes mode P, indices kept
    im.convert("P").save(path)


class MaskWriter:
    """Writes device masks as <dir>/<id>.png (8-bit grey) on a thread: submit() copies the mask into one of `slots` pinned buffers on the
    caller's stream, and the thread waits for that copy and writes the file, as sequence.LogWriter does for the LOG images."""

    def __init__(self, out_dir: str, H: int, W: int, slots: int = 3):
        import torch
        self.torch, self.out_dir = torch, out_dir
        os.makedirs(out_dir, exist_ok=True)
        self.slots = [(torch.empty((H, W), dtype=torch.uint8, pin_memory=True), torch.cuda.Event()) for _ in range(slots)]
        self._free, self._q, self._err = queue.Queue(), queue.Queue(), None
        for k in range(slots):
            self._free.put(k)
        self._thread = threading.Thread(target=self._run, daemon=True)
        self._thread.start()

    def _raise(self):
        if self._err is not None:
            e, self._err = self._err, None
            raise RuntimeError(f"writing a mask failed: {e}") from e

    def _run(self):
        import cv2
        while True:
            item = self._q.get()
            if item is None:
                return
            k, id_str = item
            h, ev = self.slots[k]
            try:
                if self._err is None:
                    ev.synchronize()
                    if not cv2.imwrite(os.path.join(self.out_dir, f"{id_str}.png"), h.numpy()):
                        raise OSError(f"cv2 could not write {id_str}.png under {self.out_dir}")
            except BaseException as e:      # handed to the submitting thread
                self._err = e
            finally:
                self._free.put(k)

    def submit(self, id_str: str, mask_dev, stream: int) -> None:
        self._raise()
        k = self._free.get()
        h, ev = self.slots[k]
        st = self.torch.cuda.ExternalStream(stream)
        with self.torch.cuda.stream(st):
            h.copy_(mask_dev, non_blocking=True)
            ev.record(st)
        self._q.put((k, id_str))

    def close(self) -> None:
        """Waits for every mask submitted, then raises the writer's error if there was one."""
        if self._thread is not None:
            self._q.put(None)
            self._thread.join()
            self._thread = None
        self._raise()


class VosSource:
    """run_sequence's mask source (masks=): frame 0's mask is init_mask (label values, H x W uint8), every later frame's is propagated by
    `vos` from the frames before it, on the tracker's stream.  mask_save_dir: also write each mask as <id>.png, 0 / 255, on a thread."""

    def __init__(self, vos: VosDevice, init_mask: np.ndarray, mask_save_dir: str | None = None):
        import torch
        init_mask = np.asarray(init_mask)
        if init_mask.dtype != np.uint8 or init_mask.shape != (vos.H, vos.W):
            raise ValueError(f"init_mask must be uint8 {vos.H} x {vos.W}, got {init_mask.dtype} {init_mask.shape}")
        self.vos = vos
        self.init = torch.from_numpy(np.ascontiguousarray(init_mask)).to(vos.device)
        self.out = torch.empty((vos.H, vos.W), dtype=torch.uint8, device=vos.device)
        self.writer = MaskWriter(mask_save_dir, vos.H, vos.W) if mask_save_dir else None

    def mask(self, i: int, id_str: str, colour, stream: int):
        """Frame i's mask (the buffer is rewritten by the next call, in stream order)."""
        m = self.vos.begin(colour, self.init, self.out, stream) if i == 0 else self.vos.next(colour, self.out, stream)
        if self.writer is not None:
            self.writer.submit(id_str, m, stream)
        return m

    def flush(self) -> None:
        if self.writer is not None:
            self.writer.close()
            self.writer = None

    def close(self) -> None:
        self.flush()
        self.vos.close()


def load_source(model_path: str, init_mask_path: str, H: int, W: int, mask_save_dir: str | None = None, params: dict | None = None,
                device: int = 0) -> VosSource:
    """The run scripts' --vos_model / --init_mask / --mask_save_dir as a VosSource for H x W frames."""
    m = read_init_mask(init_mask_path)
    if m.shape != (H, W):
        raise ValueError(f"{init_mask_path}: {m.shape[0]} x {m.shape[1]}, the frames are {H} x {W}")
    return VosSource(load_vos(model_path, params, H=H, W=W, device=device), m, mask_save_dir)
