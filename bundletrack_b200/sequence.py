"""Tracking a dataset scene end to end: the reference's applications (src/app/bundle_track_nocs.cpp, bundle_track_ycbineoat.cpp) on the
library.  The pieces:

- loaders that restate DataLoaderNOCS / DataLoaderYcbineoat (src/DataLoader.cpp) and the mask-file rule of the Frame constructor
  (Frame.cpp:251-258), quirks included;
- image reading with the reference's cv::imread flags (cv2 when it is importable, PIL otherwise; both give the same arrays), refusing any
  file layout the reference would misread;
- a prefetching frame reader: a worker thread decodes frames ahead into pinned host buffers and uploads them on a copy stream, and the
  16-bit depth goes to the device as it is (bt_tracker_begin_frame_u16 converts it in the front-end kernel);
- the LF-Net client (Lfnet::detectFeature's ZMQ round trip, FeatureManager.cpp:861-908);
- run_sequence: Bundler::processNewFrame + saveNewframeResult for every frame, one pose file per frame and, with log > 0, the LOG frame's
  images (overlay.py), encoded on a writer thread.

Deliberate difference: the reference finds the ground-truth directory and decides the mask mode by searching data_dir for "NOCS" (DataLoader.cpp:
68-72, Frame.cpp:251,267).  Here the loader's type decides both, so the dataset root may have any name."""
from __future__ import annotations

import math
import os
import queue
import threading
import time
from dataclasses import dataclass

import numpy as np

from . import _lib, policy
from .config import load_yml

SYNSET_NAMES = ["BG", "bottle", "bowl", "camera", "can", "laptop", "mug"]
# DataLoader.cpp:75-77
NOCS_K = np.array([[591.0125, 0, 322.525], [0, 590.16775, 244.11084], [0, 0, 1]], np.float32)
LFNET_SIDE = 400            # the request image is 400 x 400 x 3 (FeatureManager.cpp:848-849)
DESC_DIM = 256


class DetectionFailed(Exception):
    """A feature source found no usable features for the frame: the tracker drops it (Bundler.cpp:103-117)."""


@dataclass
class FrameFiles:
    id_str: str
    colour: str
    depth: str
    mask: str


def _listdir(d: str) -> list:
    """Utils::readDirectory (Utils.cpp:113-130): every entry but . and .., byte-wise sorted."""
    return sorted(os.listdir(d))


def _read_matrix(path: str, r: int, c: int) -> np.ndarray:
    """Utils::parseMatrixTxt into a float matrix: the first r x c numbers of the file, row by row."""
    with open(path) as f:
        v = f.read().split()
    if len(v) < r * c:
        raise ValueError(f"{path}: {len(v)} numbers, a {r} x {c} matrix needs {r * c}")
    return np.array([float(x) for x in v[:r * c]], np.float64).astype(np.float32).reshape(r, c)


def initial_pose(ob_in_cam0) -> np.ndarray:
    """Frame 0's pose: ob_in_cam0.inverse() (DataLoader.cpp:206-210, 371-375) with its rotation columns normalised as the Frame constructor
    does (Frame.cpp:59, Utils::normalizeRotationMatrix): per column n = (x*x + y*y) + z*z and the column divided by sqrt(n), in float32.
    Eigen's 4 x 4 float inverse has no pinned rounding (its operation order depends on the SIMD path it was built with), so the inverse is
    taken in float64 from the float32 matrix and rounded once."""
    P = np.linalg.inv(np.asarray(ob_in_cam0, np.float32).astype(np.float64)).astype(np.float32)
    for c in range(3):
        x, y, z = P[0, c], P[1, c], P[2, c]
        n = np.float32(np.float32(x * x + y * y) + z * z)
        if n > 0:
            P[:3, c] = P[:3, c] / np.float32(np.sqrt(n))
    return P


class _Loader:
    """Shared by both loaders: frames (FrameFiles, in the reference's order), K (3 x 3 float32), ob_in_cam0 (4 x 4 float32), mask_mode, and
    model_path, the object's OBJ file the LOG frames draw (None: not known)."""
    frames: list
    K: np.ndarray
    ob_in_cam0: np.ndarray
    mask_mode: int
    model_path: str = None

    def __len__(self) -> int:
        return len(self.frames)

    def initial_pose(self, i: int) -> np.ndarray:
        """The pose the loader gives frame i: ob_in_cam0^-1 for the first frame, the identity for every later one (DataLoader.cpp:206-210,
        371-375).  So after a first frame that fails its ROI gate the next frame starts from the identity, as in the reference."""
        return initial_pose(self.ob_in_cam0) if i == 0 else np.eye(4, dtype=np.float32)


class NocsScene(_Loader):
    """DataLoaderNOCS (DataLoader.cpp:61-215) for one (scene, model) of NOCS-REAL275 under nocs_dir, masks from mask_dir/<id>.png."""

    def __init__(self, nocs_dir: str, scene_id: int, model_name: str, mask_dir: str, use_6pack_datalist: bool = True):
        from ._lib import BT_MASK_LARGEST_HULL
        # the reference takes the scene id as the one digit after data_dir's first "scene_" (DataLoader.cpp:65); NOCS-REAL275's scenes are 1-6,
        # where that digit is the scene id given here
        data_dir = f"{nocs_dir}/real_test/scene_{scene_id}/"
        self.data_dir, self.scene_id, self.model_name, self.mask_dir = data_dir, int(scene_id), model_name, mask_dir
        self.K = NOCS_K.copy()
        self.model_path = f"{nocs_dir}/obj_models/real_test/{model_name}.obj"    # DataLoader.cpp:68-70
        gt_dir = f"{nocs_dir}/gts/real_test_text/scene_{scene_id}/model_{model_name}/"
        gts = _listdir(gt_dir)
        if not gts:
            raise FileNotFoundError(f"no ground-truth pose under {gt_dir}")
        self.ob_in_cam0 = _read_matrix(gt_dir + gts[0], 4, 4)              # DataLoader.cpp:80-85: the first sorted file
        self.mask_mode = BT_MASK_LARGEST_HULL                             # Frame.cpp:267: NOCS keeps the largest component's hull
        if use_6pack_datalist:
            # DataLoader.cpp:118-145: the class is the first synset name (from index 1) found in the model name (0 if none); the frames are the
            # list's lines that contain "scene_<k>" anywhere (so scene_1 also takes scene_1x lines), in file order, named by their last token
            cls = next((i for i in range(1, len(SYNSET_NAMES)) if SYNSET_NAMES[i] in model_name), 0)
            list_file = f"{data_dir}/../../NOCS-REAL275-additional/data_list/real_val/{cls}/{model_name}/list.txt"
            with open(list_file) as f:
                lines = f.read().split("\n")
            colour = [f"{data_dir}/../../real_test/scene_{scene_id}/{ln.split('/')[-1]}_color.png" for ln in lines if f"scene_{scene_id}" in ln]
        else:
            # DataLoader.cpp:104-115: every sorted entry of data_dir whose name contains "color.png"
            colour = [data_dir + f for f in _listdir(data_dir) if "color.png" in f]
        self.frames = []
        for path in colour:
            # DataLoader.cpp:163: four characters from five before the FIRST "color" anywhere in the path (a directory named "color..." wins)
            k = path.find("color")
            if k < 5:
                raise ValueError(f"{path}: no frame id before 'color'")
            id_str = path[k - 5:k - 1]
            # DataLoader.cpp:166 (depth) and Frame.cpp:253-255 (mask)
            self.frames.append(FrameFiles(id_str, path, data_dir + id_str + "_depth.png", f"{mask_dir}/{id_str}.png"))


class YcbineoatVideo(_Loader):
    """DataLoaderYcbineoat (DataLoader.cpp:303-380) for one video directory.  model_dir: the object's OBJ file (the yml's model_dir key,
    DataLoader.cpp:292), needed only for LOG frames."""

    def __init__(self, data_dir: str, model_dir: str = None):
        from ._lib import BT_MASK_AS_IS
        self.data_dir = data_dir
        self.model_path = model_dir
        self.K = _read_matrix(f"{data_dir}/cam_K.txt", 3, 3)                 # DataLoader.cpp:310
        gt_dir = f"{data_dir}/annotated_poses/"
        gts = _listdir(gt_dir)
        if not gts:
            raise FileNotFoundError(f"no ground-truth pose under {gt_dir}")
        self.ob_in_cam0 = _read_matrix(gt_dir + gts[0], 4, 4)              # DataLoader.cpp:314-318: the first sorted file
        self.mask_mode = BT_MASK_AS_IS                                    # Frame.cpp:267: other datasets use the mask as it is
        self.frames = []
        for f in _listdir(f"{data_dir}/rgb/"):
            # DataLoader.cpp:359-364: the id is the file name up to its FIRST "."; depth/<id>.png.  Frame.cpp:258: the mask is
            # <data_dir>/masks/<id>.png whatever the config's mask_dir says
            id_str = f.split(".")[0]
            self.frames.append(FrameFiles(id_str, f"{data_dir}/rgb/{f}", f"{data_dir}/depth/{id_str}.png", f"{data_dir}/masks/{id_str}.png"))


# ---- image reading --------------------------------------------------------------------------------------------------------------------------

# (bit depth, PNG colour type) each kind accepts.  colour: 8-bit RGB or RGBA (cv::IMREAD_COLOR drops alpha); depth: 16-bit grey, read as
# cv::imread(path, CV_16UC1 = IMREAD_ANYDEPTH) (Utils.cpp:52); mask: 8-bit grey, read with IMREAD_UNCHANGED (Frame.cpp:257).  Anything else
# the reference would read as another type through at<uchar> / at<unsigned short>.
_LAYOUTS = {"colour": {(8, 2), (8, 6)}, "depth": {(16, 0)}, "mask": {(8, 0)}}
_PNG_TYPES = {0: "grey", 2: "RGB", 3: "palette", 4: "grey + alpha", 6: "RGBA"}


def png_layout(path: str):
    """(width, height, bit depth, colour type) from the PNG's IHDR chunk."""
    with open(path, "rb") as f:
        h = f.read(29)
    if len(h) < 29 or h[:8] != b"\x89PNG\r\n\x1a\n" or h[12:16] != b"IHDR":
        raise ValueError(f"{path}: not a PNG file")
    return int.from_bytes(h[16:20], "big"), int.from_bytes(h[20:24], "big"), h[24], h[25]


def _check_layout(path: str, kind: str):
    W, H, depth, ctype = png_layout(path)
    if (depth, ctype) not in _LAYOUTS[kind]:
        want = " or ".join(f"{d}-bit {_PNG_TYPES[c]}" for d, c in sorted(_LAYOUTS[kind]))
        raise ValueError(f"{path}: {depth}-bit {_PNG_TYPES.get(ctype, ctype)} PNG; a {kind} image must be {want}")
    return W, H


def _have_cv2() -> bool:
    try:
        import cv2  # noqa: F401
        return True
    except ImportError:
        return False


def read_image(path: str, kind: str, reader: str = None) -> np.ndarray:
    """kind "colour" -> uint8 [H,W,3] BGR, "depth" -> uint16 [H,W] (the PNG's samples, millimetres), "mask" -> uint8 [H,W].  reader: "cv2",
    "pil" or None (cv2 when it is importable)."""
    _check_layout(path, kind)
    reader = reader or ("cv2" if _have_cv2() else "pil")
    if reader == "cv2":
        import cv2
        flag = {"colour": cv2.IMREAD_COLOR, "depth": cv2.IMREAD_ANYDEPTH, "mask": cv2.IMREAD_UNCHANGED}[kind]
        a = cv2.imread(path, flag)
        if a is None:
            raise ValueError(f"{path}: cv2 could not decode it")
    else:
        from PIL import Image
        with Image.open(path) as im:
            if kind == "colour":
                a = np.asarray(im.convert("RGB"))[..., ::-1]
            else:
                a = np.asarray(im)
        if kind == "depth":
            a = a.astype(np.uint16)           # Pillow opens 16-bit grey as "I;16" or, in older versions, as int32 "I"
    dtype, ndim = {"colour": (np.uint8, 3), "depth": (np.uint16, 2), "mask": (np.uint8, 2)}[kind]
    if a.dtype != dtype or a.ndim != ndim:
        raise ValueError(f"{path}: decoded as {a.dtype} {a.shape}, expected {np.dtype(dtype)} with {ndim} dimensions")
    return np.ascontiguousarray(a)


def read_frame(ff: FrameFiles, reader: str = None, with_mask: bool = True):
    """(depth uint16 [H,W], mask uint8 [H,W], colour uint8 [H,W,3] BGR) of one frame; the three must have one size.  with_mask=False
    leaves the mask file unread and gives zeros in its place (the masks come from elsewhere)."""
    d, c = read_image(ff.depth, "depth", reader), read_image(ff.colour, "colour", reader)
    m = read_image(ff.mask, "mask", reader) if with_mask else np.zeros(d.shape, np.uint8)
    if d.shape != m.shape or d.shape != c.shape[:2]:
        raise ValueError(f"frame {ff.id_str}: depth {d.shape}, mask {m.shape} and colour {c.shape[:2]} differ in size")
    return d, m, c


# ---- prefetching frame reader ---------------------------------------------------------------------------------------------------------------

class FrameReader:
    """Frames of a loader on the device, in order.  A worker thread decodes up to `prefetch` frames ahead into a ring of pinned host buffers
    (uint16 depth, mask, BGR colour) and uploads each on a copy stream; get(i) makes `stream` wait for frame i's upload and returns its
    device tensors.  release(i) records an event on `stream` behind the work that reads frame i; the copy stream waits for that event before
    it rewrites the slot, so work enqueued before release (bt_lfnet_request reads the colour after begin_frame's ROI synchronisation) is
    covered.  prefetch=0 decodes and uploads in get(), in the calling thread.  with_mask=False reads no mask files (get's mask is then
    left as it was: the caller supplies the masks)."""

    def __init__(self, loader, H: int, W: int, device: int, stream, prefetch: int = 2, with_mask: bool = True):
        import torch
        self.torch, self.loader, self.stream, self.prefetch = torch, loader, stream, int(prefetch)
        self.with_mask = with_mask
        self.dev = torch.device("cuda", device)
        self.copy = torch.cuda.Stream(self.dev)
        R = self.prefetch + 1
        shapes = ((H, W), (H, W), (H, W, 3))
        dtypes = (torch.int16, torch.uint8, torch.uint8)     # the depth buffers hold the uint16 samples' bytes (the library reads them as uint16)
        self.host = [[torch.empty(s, dtype=t, pin_memory=True) for s, t in zip(shapes, dtypes)] for _ in range(R)]
        self.devbuf = [[torch.empty(s, dtype=t, device=self.dev) for s, t in zip(shapes, dtypes)] for _ in range(R)]
        self.uploaded = [torch.cuda.Event() for _ in range(R)]
        self.consumed = [torch.cuda.Event() for _ in range(R)]
        self.decode_s = [0.0] * len(loader)
        self.R = R
        self._stop = threading.Event()
        self._q = queue.Queue()
        self._free = threading.Semaphore(R)
        self._thread = None
        if self.prefetch > 0:
            self._thread = threading.Thread(target=self._worker, daemon=True)
            self._thread.start()

    def _fill(self, i: int) -> None:
        torch = self.torch
        s = i % self.R
        t0 = time.perf_counter()
        arrays = read_frame(self.loader.frames[i], with_mask=self.with_mask)
        self.decode_s[i] = time.perf_counter() - t0
        self.uploaded[s].synchronize()                  # the slot's previous upload has read the pinned buffers
        for h, a in zip(self.host[s], arrays):
            if tuple(h.shape) != a.shape:
                raise ValueError(f"frame {self.loader.frames[i].id_str}: {a.shape[1]} x {a.shape[0]} images, the sequence is {h.shape[1]} x {h.shape[0]}")
            h.numpy()[...] = a.view(np.int16) if a.dtype == np.uint16 else a
        with torch.cuda.device(self.dev), torch.cuda.stream(self.copy):
            self.copy.wait_event(self.consumed[s])         # the tracker's reads of the slot's previous frame are done
            for d, h in zip(self.devbuf[s], self.host[s]):
                d.copy_(h, non_blocking=True)
            self.uploaded[s].record(self.copy)

    def _worker(self):
        try:
            for i in range(len(self.loader)):
                while not self._free.acquire(timeout=0.1):
                    if self._stop.is_set():
                        return
                if self._stop.is_set():
                    return
                self._fill(i)
                self._q.put(i)
        except BaseException as e:      # handed to the consumer, which raises it
            self._q.put(e)

    def get(self, i: int):
        """(depth_mm, mask, colour) device tensors of frame i, ready on `stream`.  Frames are taken in order, each released before the next."""
        if self._thread is None:
            self._fill(i)
        else:
            j = self._q.get()
            if isinstance(j, BaseException):
                raise j
            assert j == i, (j, i)
        s = i % self.R
        self.stream.wait_event(self.uploaded[s])
        return self.devbuf[s]

    def release(self, i: int) -> None:
        self.consumed[i % self.R].record(self.stream)
        self._free.release()

    def close(self):
        self._stop.set()
        if self._thread is not None:
            self._thread.join()
            self._thread = None
        self.copy.synchronize()


# ---- feature sources ------------------------------------------------------------------------------------------------------------------------

class LfnetClient:
    """Lfnet::detectFeature's round trip (FeatureManager.cpp:861-908) with pyzmq: a REQ socket connected to the LF-Net server's endpoint.
    The request is [int32 W, H] and the 400 x 400 x 3 request bytes; the reply [int32 n, dim], the keypoints and the descriptors
    (lf-net-release/run_server.py:142-177), mapped back to image pixels by policy.lfnet_parse_reply.  A reply that does not parse, or whose
    descriptors are not 256-dimensional, raises DetectionFailed (the reference's catch, Bundler.cpp:103-117).  No reply within timeout_s
    raises RuntimeError naming the endpoint: the run cannot go on without the server.  context: a zmq.Context to use (an inproc:// endpoint
    needs the server's), else the client makes its own."""

    def __init__(self, endpoint: str, timeout_s: float = 60.0, context=None):
        import zmq
        self.zmq, self.endpoint, self.timeout_ms = zmq, endpoint, int(timeout_s * 1000)
        self._own_ctx = context is None
        self.ctx = zmq.Context() if context is None else context
        self.sock = self.ctx.socket(zmq.REQ)
        self.sock.setsockopt(zmq.LINGER, 0)
        self.sock.connect(endpoint)

    def __call__(self, id_str: str, request: np.ndarray, roi):
        req = np.ascontiguousarray(request, np.uint8)
        if req.shape != (LFNET_SIDE, LFNET_SIDE, 3):
            raise ValueError(f"request image of shape {req.shape}, expected ({LFNET_SIDE}, {LFNET_SIDE}, 3)")
        self.sock.send_multipart([np.array([req.shape[1], req.shape[0]], np.int32).tobytes(), req.tobytes()])
        if not self.sock.poll(self.timeout_ms, self.zmq.POLLIN):
            raise RuntimeError(f"LF-Net server at {self.endpoint}: no reply for frame {id_str} within {self.timeout_ms / 1000:g} s")
        parts = self.sock.recv_multipart()
        if len(parts) != 3:
            raise DetectionFailed(f"frame {id_str}: the reply has {len(parts)} parts, not 3")
        try:
            kpts, desc = policy.lfnet_parse_reply(parts, roi)
        except _lib.BtError as e:
            raise DetectionFailed(f"frame {id_str}: {e}") from e
        if desc.shape[1] != DESC_DIM:
            raise DetectionFailed(f"frame {id_str}: {desc.shape[1]}-dimensional descriptors, the tracker takes {DESC_DIM}")
        return kpts, desc

    def close(self):
        if self.sock is not None:
            self.sock.close(0)
            if self._own_ctx:
                self.ctx.term()
            self.sock = None


# ---- LOG frames -----------------------------------------------------------------------------------------------------------------------------

class LogWriter:
    """Writes LOG frames (overlay.write_log_frame) on a thread of its own, so the JPEG and PNG encodes stay off the tracking thread.
    submit() copies the device images into one of `depth` pinned slots behind the work already on `stream` and returns; it blocks only while
    every slot is still being written.  An error on the writer thread is raised by the next submit() or by close()."""

    def __init__(self, debug_dir: str, H: int, W: int, depth: int = 4):
        import torch
        from .overlay import _cv2
        _cv2()                                           # no OpenCV: fail before the run starts
        self.torch, self.debug_dir = torch, debug_dir
        self.slots = [(torch.empty((H, W, 3), dtype=torch.uint8, pin_memory=True), torch.empty((H, W, 3), dtype=torch.uint8, pin_memory=True),
                       torch.cuda.Event()) for _ in range(depth)]
        self._free = queue.Queue()
        for k in range(depth):
            self._free.put(k)
        self._q = queue.Queue()
        self._err = None
        self._thread = threading.Thread(target=self._run, daemon=True)
        self._thread.start()

    def _raise(self):
        if self._err is not None:
            e, self._err = self._err, None
            raise RuntimeError(f"writing a LOG frame failed: {e}") from e

    def _run(self):
        from .overlay import write_log_frame
        while True:
            item = self._q.get()
            if item is None:
                return
            k, id_str = item
            hv, hr, ev = self.slots[k]
            try:
                if self._err is None:
                    ev.synchronize()
                    write_log_frame(self.debug_dir, id_str, hv.numpy(), hr.numpy())
            except BaseException as e:      # handed to the tracking thread
                self._err = e
            finally:
                self._free.put(k)

    def submit(self, id_str: str, viz_dev, raw_dev, stream) -> None:
        self._raise()
        k = self._free.get()
        hv, hr, ev = self.slots[k]
        with self.torch.cuda.stream(stream):
            hv.copy_(viz_dev, non_blocking=True)
            hr.copy_(raw_dev, non_blocking=True)
            ev.record(stream)
        self._q.put((k, id_str))

    def close(self) -> None:
        """Waits for every frame submitted, then raises the writer's error if there was one."""
        if self._thread is not None:
            self._q.put(None)
            self._thread.join()
            self._thread = None
        self._raise()


# ---- the run --------------------------------------------------------------------------------------------------------------------------------

def run_sequence(loader, yml, features, out_dir: str, max_feats: int = 2000, max_keyframes: int = None, device: int = 0, prefetch: int = 2,
                 log: int = 0, masks=None, model_out: str = None):
    """Tracks every frame the loader yields (Bundler::processNewFrame) and writes <out_dir>/poses/<id_str>.txt for each one with
    policy.save_pose_txt (Bundler::saveNewframeResult runs after every frame): the initial pose of a frame that fails the ROI gate, the
    pose drop_frame reports when detection fails, otherwise end_frame's.  features(id_str, request uint8 [400,400,3] host, roi) returns
    (kpts [n,2] image pixels, desc [n,256] float32) or raises DetectionFailed; a reply with more than max_feats rows or descriptors that are
    not 256-dimensional is dropped too.  A source marked on_device (lfnet.LfnetDevice) is called as features.features_on_device(id_str,
    request uint8 [400,400,3] on the device, roi, stream) instead and returns the keypoints on the host and the descriptors on the device, so
    neither the request nor the descriptors cross the bus.  Sizing as INTEGRATION.md §7: max_frames_alive = bundle.window_size + 4, max_keyframes defaults to
    min(1024, ceil(n_frames / 2)).  Nothing under out_dir is removed.  Returns [(id_str, status, wall seconds)] per frame.
    log > 0 (the yml's LOG): every frame's LOG images under out_dir (the reference's debug_dir), drawn on the device with the pose its pose
    file holds (overlay.Overlay over loader.model_path) and written by a LogWriter thread; needs cv2.  log = 0 runs none of it.
    masks (vos.VosSource): each frame's object mask is propagated on the device from the first frame's, on the tracker's stream, over the
    frames the loader yields in order; the loader's mask files are not read.
    model_out (a path): after the last frame, the keyframes' depth maps are fused with their final poses into a TSDF on the tracker's stream
    (recon.fuse_keyframes at recon.VOXEL / TRUNC) and its zero surface is written there as a binary PLY, in the model
    frame (the object's frame when the loader's first pose is its ob_in_cam0).  None runs none of it; tracking is the same either way."""
    import torch
    from .tracker import Tracker
    n = len(loader)
    if n == 0:
        return []
    y = load_yml(yml)
    W, H = png_layout(loader.frames[0].colour)[:2]
    if max_keyframes is None:
        max_keyframes = min(1024, math.ceil(n / 2))
    os.makedirs(os.path.join(out_dir, "poses"), exist_ok=True)
    dev = torch.device("cuda", device)
    stream = torch.cuda.Stream(dev)
    trk = Tracker(y, H, W, loader.K, max_feats, int(y["bundle"]["window_size"]) + 4, device=device, stream=stream.cuda_stream,
                  mode=loader.mask_mode, max_keyframes=max_keyframes)
    reader = ovl = writer = None
    on_device = getattr(features, "on_device", False)
    out = []
    try:
        if log > 0:
            from .overlay import Overlay, load_obj_points
            if not loader.model_path:
                raise ValueError("log > 0 draws the object model: the loader has no model path (YcbineoatVideo needs model_dir)")
            writer = LogWriter(out_dir, H, W)
            ovl = Overlay(load_obj_points(loader.model_path), loader.K, H, W, device=device, stream=stream.cuda_stream)
            with torch.cuda.device(dev):
                viz, raw = (torch.empty((H, W, 3), dtype=torch.uint8, device=dev) for _ in range(2))
        reader = FrameReader(loader, H, W, device, stream, prefetch, with_mask=masks is None)
        with torch.cuda.device(dev):
            request = torch.empty((LFNET_SIDE, LFNET_SIDE, 3), dtype=torch.uint8, device=dev)
        for i, ff in enumerate(loader.frames):
            t0 = time.perf_counter()
            depth, mask, colour = reader.get(i)
            if masks is not None:
                mask = masks.mask(i, ff.id_str, colour, stream.cuda_stream)
            st, roi, _, pose = trk.begin_frame_mm(depth, mask, colour, request, loader_id=i, first_pose=loader.initial_pose(i))
            if ovl is None:
                reader.release(i)
            if st == _lib.BT_FRAME_OTHER:
                try:
                    if on_device:
                        kpts, desc = features.features_on_device(ff.id_str, request, roi, stream.cuda_stream)
                    else:
                        with torch.cuda.device(dev), torch.cuda.stream(stream):
                            req = request.cpu()
                        kpts, desc = features(ff.id_str, req.numpy(), roi)
                        kpts = np.ascontiguousarray(kpts, np.float32).reshape(-1, 2)
                        desc = np.ascontiguousarray(desc, np.float32)
                    if desc.ndim != 2 or desc.shape[1] != DESC_DIM or len(desc) != len(kpts) or len(kpts) > max_feats:
                        raise DetectionFailed(f"frame {ff.id_str}: {len(kpts)} keypoints with descriptors {tuple(desc.shape)}; the tracker takes at "
                                              f"most {max_feats} rows of {DESC_DIM}")
                except DetectionFailed:
                    pose, st = trk.drop_frame(), _lib.BT_FRAME_FAIL
                else:
                    if on_device:
                        desc_dev = desc
                    else:
                        with torch.cuda.device(dev), torch.cuda.stream(stream):
                            desc_dev = torch.from_numpy(desc).to(dev)
                    try:
                        pose, st = trk.end_frame(kpts, desc_dev)
                    except _lib.BtError as e:
                        if e.rc != _lib.BT_ERR_CAPACITY:
                            raise
                        trk.drop_frame()
                        raise _lib.BtError(f"frame {ff.id_str}: the tracker is full ({e}); raise max_keyframes (now {max_keyframes})",
                                           _lib.BT_ERR_CAPACITY) from e
            policy.save_pose_txt(os.path.join(out_dir, "poses", f"{ff.id_str}.txt"), pose)
            if ovl is not None:
                # the frame's colour slot and the tracker's fg map are read on `stream` before the slot is released and the next begin_frame
                ovl.render(pose, [colour], [trk.last_fg()], [viz], [raw])
                reader.release(i)
                writer.submit(ff.id_str, viz, raw, stream)
            out.append((ff.id_str, st, time.perf_counter() - t0))
        if writer is not None:
            writer.close()
        if masks is not None:
            masks.flush()
        if model_out is not None:
            _write_model(trk, loader.K, H, W, device, stream, model_out)
    finally:
        if reader is not None:
            reader.close()
        stream.synchronize()
        if writer is not None:
            try:
                writer.close()
            except Exception:
                pass                # (the run is already failing: its own error is the one raised)
        if ovl is not None:
            ovl.close()
        trk.close()
    return out


def _write_model(trk, K, H: int, W: int, device: int, stream, path: str) -> None:
    """The keyframes fused and meshed on the tracker's stream, the mesh written to path (recon.py)."""
    from . import recon
    tsdf = recon.Tsdf(max(1, int(trk.state()[2].sum())), H, W, device=device, stream=stream.cuda_stream)
    try:
        recon.fuse_keyframes(trk, tsdf, K)
        verts, faces = tsdf.mesh()
    finally:
        tsdf.close()
    recon.write_ply(path, verts, faces)


def summary(result) -> str:
    """One line on a run_sequence result: frames, statuses and the per-frame wall time."""
    if not result:
        return "0 frames"
    st = np.array([r[1] for r in result])
    t = np.array([r[2] for r in result]) * 1000
    return (f"{len(result)} frames: {int((st == _lib.BT_FRAME_OTHER).sum())} OK, {int((st == _lib.BT_FRAME_NO_BA).sum())} NO_BA, "
            f"{int((st == _lib.BT_FRAME_FAIL).sum())} FAIL; wall per frame median {np.median(t):.2f} ms, p90 {np.percentile(t, 90):.2f} ms")
