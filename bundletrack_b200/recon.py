"""Object model from a tracking run: depth maps fused into a TSDF in the model frame on the device and its zero surface meshed by marching
tetrahedra.  A thin ctypes mirror of bt_recon_reserve / bt_tsdf_fuse / bt_tsdf_mesh (include/bundletrack_b200.h, DESIGN.md §3.14):

- Tsdf: fuse(depths, poses, K, voxel, trunc) and mesh() on a context;
- fuse_keyframes: a tracker's keyframes, with their current poses and their processed depth, fused on the tracker's stream;
- write_ply: the mesh as binary little-endian PLY; read_mesh: that PLY, or a Wavefront OBJ (a reference mesh to score the model
  against, bundletrack_b200.metrics.SurfaceScore)."""
from __future__ import annotations

import ctypes
import os

import numpy as np

from . import _lib

VOXEL = 0.002               # metres: the default sample spacing
TRUNC = 4 * VOXEL           # metres: the default truncation, four samples


class Tsdf(_lib.Facade):
    """A TSDF grid of up to max_voxels samples fused from up to max_frames depth maps of H x W, and mesh outputs of up to max_vertices /
    max_faces.  Device work runs on `stream`; fuse() and mesh() each synchronise it once (the grid's size, the mesh's counts)."""

    def __init__(self, max_frames: int, H: int, W: int, max_voxels: int = 1 << 24, max_vertices: int = 1 << 21, max_faces: int = 1 << 22,
                 device: int = 0, stream: int = 0, ctx=None):
        import torch
        super().__init__(ctx, device, stream)
        self.device, self.H, self.W = device, int(H), int(W)
        _lib.check(self.lib.bt_recon_reserve(self.ctx, max_frames, self.H, self.W, max_voxels, max_vertices, max_faces), "bt_recon_reserve")
        dev = torch.device("cuda", device)
        self.verts = torch.empty((max_vertices, 3), dtype=torch.float32, device=dev)
        self.faces = torch.empty((max_faces, 3), dtype=torch.int32, device=dev)

    def fuse(self, depths, poses, K, voxel: float = VOXEL, trunc: float = TRUNC) -> None:
        """depths: contiguous float32 [H,W] CUDA tensors on this device (metres, 0 = none) or raw device addresses; poses: [F,4,4] cam->model;
        K: 3 x 3 or (fx, fy, cx, cy).  Replaces the grid.  Reads the depths on the stream: they must be ready there."""
        import torch
        P = np.ascontiguousarray(np.asarray(poses, np.float32).reshape(-1, 16))
        if len(P) != len(depths):
            raise ValueError(f"{len(P)} poses and {len(depths)} depth maps")
        for k, d in enumerate(depths):
            if isinstance(d, int):
                continue
            if not isinstance(d, torch.Tensor) or not d.is_cuda or d.device.index != self.device:
                raise ValueError(f"depth {k} must be a CUDA tensor on device {self.device} (or a device address)")
            if d.dtype != torch.float32 or not d.is_contiguous() or tuple(d.shape) != (self.H, self.W):
                raise ValueError(f"depth {k} must be a contiguous float32 [{self.H}, {self.W}] tensor, not {d.dtype} {list(d.shape)}")
        p = _lib.TsdfParams(voxel, trunc)
        _lib.check(self.lib.bt_tsdf_fuse(self.ctx, len(P), _lib.ptrs(depths), _lib.ptr(P), *_lib.intrinsics(K), self.H, self.W, ctypes.byref(p),
                                         self.stream), "bt_tsdf_fuse")

    def mesh(self):
        """(verts float32 [n,3], faces int32 [m,3]) numpy of the grid's zero surface, faces wound towards free space."""
        nv, nf = ctypes.c_int(0), ctypes.c_int(0)
        _lib.check(self.lib.bt_tsdf_mesh(self.ctx, _lib.ptr(self.verts), _lib.ptr(self.faces), ctypes.byref(nv), ctypes.byref(nf), self.stream), "bt_tsdf_mesh")
        _lib.check(self.lib.bt_stream_sync(self.stream), "bt_stream_sync")
        return self.verts[:nv.value].cpu().numpy(), self.faces[:nf.value].cpu().numpy()

    def grid(self):
        """The last fused grid on the host: dict of dims (nx, ny, nz), origin [3], lo / hi [3] (the valid pixels' bounds), sum float32 and
        count int32 [nz, ny, nx].  Synchronises the stream."""
        dims = (ctypes.c_int * 3)()
        origin, bounds = (ctypes.c_float * 3)(), (ctypes.c_float * 6)()
        s_dev, c_dev = ctypes.c_void_p(), ctypes.c_void_p()
        _lib.check(self.lib.bt_tsdf_grid(self.ctx, dims, origin, bounds, ctypes.byref(s_dev), ctypes.byref(c_dev)), "bt_tsdf_grid")
        _lib.check(self.lib.bt_stream_sync(self.stream), "bt_stream_sync")
        n = tuple(dims)
        s = np.empty((n[2], n[1], n[0]), np.float32)
        c = np.empty((n[2], n[1], n[0]), np.int32)
        for host, dev in ((s, s_dev), (c, c_dev)):
            _lib.check(self.lib.bt_memcpy_d2h(_lib.ptr(host), dev, host.nbytes, self.stream), "bt_memcpy_d2h")
        b = np.frombuffer(bounds, np.float32)
        return {"dims": n, "origin": np.frombuffer(origin, np.float32).copy(), "lo": b[:3].copy(), "hi": b[3:].copy(), "sum": s, "count": c}


def keyframe_depths(tracker):
    """(ids int32 [k], poses float32 [k,4,4] cam->model, device addresses of the processed depth) of the tracker's keyframes, oldest first."""
    ids, poses, kf = tracker.state()
    addr = []
    for i in ids[kf]:
        p = ctypes.c_void_p()
        _lib.check(tracker.lib.bt_tracker_frame_depth(tracker.t, int(i), ctypes.byref(p)), "bt_tracker_frame_depth")
        addr.append(int(p.value))
    return ids[kf], poses[kf], addr


def fuse_keyframes(tracker, tsdf: Tsdf, K, voxel: float = VOXEL, trunc: float = TRUNC) -> int:
    """Fuses the tracker's keyframes (is_keyframe in state()) with their current poses into tsdf, whose stream must be the tracker's (so the
    depth maps are read behind the tracking work) and whose context is on the tracker's device.  Returns the number of keyframes fused;
    raises ValueError when there is none."""
    ids, poses, addr = keyframe_depths(tracker)
    if len(ids) == 0:
        raise ValueError("the tracker holds no keyframe")
    tsdf.fuse(addr, poses, K, voxel, trunc)
    return len(ids)


def write_ply(path: str, verts, faces) -> None:
    """Binary little-endian PLY: `element vertex` with float x y z, `element face` with list uchar int vertex_indices."""
    v = np.ascontiguousarray(verts, "<f4").reshape(-1, 3)
    f = np.ascontiguousarray(faces, "<i4").reshape(-1, 3)
    if len(f) and (f.min() < 0 or f.max() >= len(v)):
        raise ValueError(f"face indices must lie in [0, {len(v)})")
    head = ("ply\nformat binary_little_endian 1.0\n"
            f"element vertex {len(v)}\nproperty float x\nproperty float y\nproperty float z\n"
            f"element face {len(f)}\nproperty list uchar int vertex_indices\nend_header\n")
    rows = np.empty(len(f), [("n", "u1"), ("i", "<i4", (3,))])
    rows["n"], rows["i"] = 3, f
    with open(path, "wb") as out:
        out.write(head.encode("ascii"))
        out.write(v.tobytes())
        out.write(rows.tobytes())


def _read_obj(path: str):
    verts, faces = [], []
    with open(path, "r", errors="replace") as fh:
        for ln, line in enumerate(fh, 1):
            tok = line.split()
            if not tok:
                continue
            if tok[0] == "v":
                verts.append([float(x) for x in tok[1:4]])
            elif tok[0] == "f":
                # a / b / c forms keep the vertex index; a negative index counts back from the last vertex so far; polygons are fanned
                raw = [int(t.split("/")[0]) for t in tok[1:]]
                idx = [i - 1 if i > 0 else len(verts) + i for i in raw]
                if len(idx) < 3 or 0 in raw or min(idx) < 0 or max(idx) >= len(verts):
                    raise ValueError(f"{path}:{ln}: bad face {line.strip()!r} ({len(verts)} vertices so far)")
                faces += [(idx[0], idx[k], idx[k + 1]) for k in range(1, len(idx) - 1)]
    return np.asarray(verts, np.float64).reshape(-1, 3), np.asarray(faces, np.int32).reshape(-1, 3)


_PLY_TYPES = {"char": "i1", "uchar": "u1", "short": "<i2", "ushort": "<u2", "int": "<i4", "uint": "<u4", "float": "<f4", "double": "<f8",
              "int8": "i1", "uint8": "u1", "int16": "<i2", "uint16": "<u2", "int32": "<i4", "uint32": "<u4", "float32": "<f4", "float64": "<f8"}


def _read_ply(path: str):
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.find(b"end_header\n")
    if not data.startswith(b"ply\n") or end < 0:
        raise ValueError(f"{path}: not a PLY file")
    lines = data[:end].decode("ascii", "replace").splitlines()
    if "format binary_little_endian 1.0" not in lines:
        fmt = next((l for l in lines if l.startswith("format")), "format ?")
        raise ValueError(f"{path}: PLY '{fmt}' is not read, only binary_little_endian (what write_ply writes)")
    elems = []                                   # (name, count, [(property, type or (count type, index type))])
    for l in lines:
        t = l.split()
        if t and t[0] == "element":
            elems.append((t[1], int(t[2]), []))
        elif t and t[0] == "property":
            elems[-1][2].append((t[-1], (t[2], t[3]) if t[1] == "list" else t[1]))
    names = [e[0] for e in elems]
    if names != ["vertex", "face"]:
        raise ValueError(f"{path}: PLY elements {names} are not read, only vertex then face")
    (_, nv, vprops), (_, nf, fprops) = elems
    vdt = np.dtype([(n, _PLY_TYPES[t]) for n, t in vprops])
    if len(fprops) != 1 or not isinstance(fprops[0][1], tuple) or fprops[0][1][0] not in ("uchar", "uint8"):
        raise ValueError(f"{path}: the face element must be one 'list uchar <int type>' property")
    fdt = np.dtype([("n", "u1"), ("i", _PLY_TYPES[fprops[0][1][1]], (3,))])
    off = end + len(b"end_header\n")
    v = np.frombuffer(data, vdt, nv, off)
    rows = np.frombuffer(data, fdt, nf, off + vdt.itemsize * nv)
    if nf and (rows["n"] != 3).any():
        raise ValueError(f"{path}: only triangles are read from PLY")
    f = rows["i"].astype(np.int64)
    if nf and (f.min() < 0 or f.max() >= nv):
        raise ValueError(f"{path}: face indices must lie in [0, {nv})")
    return np.stack([v["x"], v["y"], v["z"]], 1).astype(np.float64), f.astype(np.int32).reshape(-1, 3)


def read_mesh(path: str):
    """(verts float64 [n,3], faces int32 [m,3]) of a Wavefront OBJ (`v` and `f` lines; `f a/b/c` forms, negative indices, polygons split
    into fans from their first vertex) or of a binary little-endian PLY of triangles as write_ply writes it.  Other files are refused."""
    ext = os.path.splitext(path)[1].lower()
    if ext == ".obj":
        return _read_obj(path)
    if ext == ".ply":
        return _read_ply(path)
    raise ValueError(f"{path}: '{ext or path}' meshes are not read, only .obj and binary .ply")
