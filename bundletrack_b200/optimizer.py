"""Host-side mirror of the reference's optimizer facade, on top of the C-ABI.

`OptimizerGpu.optimizeFrames` keeps the reference's name, argument order and in-place pose semantics
(/root/reference/src/cuda/LossGPU.h:50, LossGPU.cu:53-139): poses are cam->model 4x4, every frame of the window is
overwritten with its optimised pose, frame 0 is the gauge.  `optimizeWindows` is the batched form (many independent
windows in one persistent launch) that the reference does not have.  All arithmetic happens in
lib/libbundletrack_b200.so on the GPU; this file only marshals pointers.
"""
from __future__ import annotations

import ctypes
from typing import List, Optional, Sequence

import numpy as np

from . import _lib
from .config import solver_params
from .synth import ENTRYJ_DTYPE


class SolveWindow:
    """One window's inputs: device frame maps + host correspondences/poses (the reference's argument list)."""

    def __init__(self, corr: np.ndarray, H: int, W: int, depths_gpu: Sequence, normals_gpu: Sequence, poses: np.ndarray, K,
                 dense_pairs: Optional[np.ndarray] = None, compat_flip: bool = True, cache_slots: Optional[Sequence[int]] = None,
                 corr_dev=None, blocks=None, corr_block_n=None):
        self.corr = np.ascontiguousarray(corr if corr is not None else np.zeros(0, ENTRYJ_DTYPE), dtype=ENTRYJ_DTYPE)
        # device-resident correspondences (bt_match_pairs output): corr_dev = device EntryJ buffer, blocks = (off, n, i, j) host arrays
        self.corr_dev = corr_dev
        self.blocks = None if blocks is None else tuple(np.ascontiguousarray(b, t) for b, t in zip(blocks, (np.int32, np.int32, np.uint32, np.uint32)))
        # host correspondences: optional per-pair counts (Bundler::optimizeGPU's n_match_per_pair): the library then skips its grouping pass
        self.corr_block_n = None if corr_block_n is None else np.ascontiguousarray(corr_block_n, np.int32)
        self.H, self.W = int(H), int(W)
        self.depths = [_lib.ptr(d) for d in (depths_gpu or [])]
        self.normals = [_lib.ptr(n) for n in (normals_gpu or [])]
        self.poses = np.ascontiguousarray(poses, np.float32).reshape(-1, 4, 4)
        self.K = _lib.intrinsics(K)
        self.dense_pairs = None if dense_pairs is None else np.ascontiguousarray(dense_pairs, np.uint32).reshape(-1, 2)
        self.compat_flip = bool(compat_flip)
        self.cache_slots = None if cache_slots is None else np.ascontiguousarray(cache_slots, np.int32)
        self._keep = (depths_gpu, normals_gpu)

    @staticmethod
    def block_counts(corr: np.ndarray) -> np.ndarray:
        """Run lengths of (imgIdx_i, imgIdx_j) in an EntryJ array that is already grouped pair by pair (what n_match_per_pair holds)."""
        if len(corr) == 0:
            return np.zeros(0, np.int32)
        key = corr["imgIdx_i"].astype(np.int64) << 32 | corr["imgIdx_j"].astype(np.int64)
        cut = np.flatnonzero(np.diff(key) != 0) + 1
        return np.diff(np.concatenate([[0], cut, [len(corr)]])).astype(np.int32)

    _MARSHALLED = frozenset(("corr_block_n", "corr", "H", "W", "depths", "normals", "poses", "K", "dense_pairs", "compat_flip", "cache_slots", "corr_dev", "blocks"))

    def __setattr__(self, name, value):
        if name in SolveWindow._MARSHALLED:
            self.__dict__.pop("_cwin", None)        # the cached bt_window is rebuilt on the next call
        object.__setattr__(self, name, value)

    def c_window(self) -> "_lib.Window":
        """The bt_window of this object (built once: per-call ctypes field stores cost more than the GPU work)."""
        cw = self.__dict__.get("_cwin")
        if cw is None:
            N = self.n_frames
            dp = (ctypes.c_void_p * N)(*self.depths) if self.depths else None
            nq = (ctypes.c_void_p * N)(*self.normals) if self.normals else None
            cw = _lib.Window()
            cw.n_frames, cw.H, cw.W, cw.n_corr = N, self.H, self.W, len(self.corr)
            cw.corr = self.corr.ctypes.data if len(self.corr) else None
            if dp is not None:
                cw.depth_dev = ctypes.cast(dp, ctypes.POINTER(ctypes.c_void_p))
                cw.normal_dev = ctypes.cast(nq, ctypes.POINTER(ctypes.c_void_p))
            if self.cache_slots is not None:
                if len(self.cache_slots) != N:
                    raise ValueError("cache_slots needs one slot per frame")
                cw.cache_slots = self.cache_slots.ctypes.data
            if self.corr_dev is not None:
                off, nb, bi, bj = self.blocks
                cw.corr_dev = _lib.ptr(self.corr_dev)
                cw.n_blocks = len(off)
                cw.block_off, cw.block_n, cw.block_i, cw.block_j = off.ctypes.data, nb.ctypes.data, bi.ctypes.data, bj.ctypes.data
            elif self.corr_block_n is not None and len(self.corr_block_n):
                cw.n_blocks = len(self.corr_block_n)
                cw.block_n = self.corr_block_n.ctypes.data
            cw.fx, cw.fy, cw.cx, cw.cy = self.K
            zero = None
            if self.dense_pairs is not None:
                zero = ctypes.c_uint32(0)
                cw.dense_pairs = self.dense_pairs.ctypes.data if len(self.dense_pairs) else ctypes.addressof(zero)
                cw.n_dense_pairs = len(self.dense_pairs)
            else:
                cw.dense_pairs, cw.n_dense_pairs = None, 0
            cw.compat_flip = 1 if self.compat_flip else 0
            self.__dict__["_cwin"] = cw
            self.__dict__["_cwin_keep"] = (dp, nq, zero, self.corr, self.dense_pairs, self.cache_slots, self.corr_dev, self.blocks, self.corr_block_n)
        return cw

    @property
    def n_frames(self) -> int:
        return self.poses.shape[0]


class _PreparedBatch:
    """bt_window array + pose block of a batch (OptimizerGpu.prepare_batch)."""
    __slots__ = ("arr", "poses", "keep", "off")

    def __init__(self, arr, poses, keep, off):
        self.arr, self.poses, self.keep, self.off = arr, poses, keep, off


class OptimizerGpu(_lib.Facade):
    def __init__(self, yml=None, device: int = 0, max_windows: int = 1, max_frames: int = 15, max_corr: int = 65536,
                 H: int = 480, W: int = 640, stream: int = 0, ctx=None):
        super().__init__(ctx, device, stream)
        self.params = solver_params(yml)
        self.reserve(max_windows, max_frames, max_corr, H, W)
        self._staged = None

    def reserve(self, max_windows: int, max_frames: int, max_corr: int, H: int, W: int):
        """Size the context's solver: windows per call, frames per window, correspondences per window and the largest frame."""
        self.limits = _lib.SolverLimits(max_windows, max_frames, max_corr, H, W, self.params.image_downscale)
        _lib.check(self.lib.bt_solver_reserve(self.ctx, self.limits), "bt_solver_reserve")

    # ---- frame cache: quarter-res maps built once per keyframe instead of once per call (CUDACache.cpp:76-88) ----------
    def reserve_frame_cache(self, capacity: int, H: int = None, W: int = None):
        _lib.check(self.lib.bt_frame_cache_reserve(self.ctx, capacity, H or self.limits.H, W or self.limits.W, self.params.image_downscale),
                   "bt_frame_cache_reserve")

    def store_frames(self, slots: Sequence[int], depths_gpu: Sequence, normals_gpu: Sequence, H: int, W: int, K):
        self.store_prepared(self.prepare_store(slots, depths_gpu, normals_gpu, H, W, K))

    def prepare_store(self, slots: Sequence[int], depths_gpu: Sequence, normals_gpu: Sequence, H: int, W: int, K):
        """The argument block of one bt_frame_cache_store call, marshalled ONCE (a C / C++ caller hands the library plain arrays; from Python
        the per-frame pointer extraction costs more than the library call itself).  Pass the result to store_prepared()."""
        args = _lib.prepared(self.lib.bt_frame_cache_store, self.ctx, len(slots), _lib.i32s(slots), _lib.ptrs(depths_gpu), _lib.ptrs(normals_gpu), H, W,
                             *_lib.intrinsics(K), self.params.depth_min, self.params.depth_max, self.stream)
        return args, (depths_gpu, normals_gpu)      # (the tensors are kept alive with the block)

    def store_prepared(self, prepared):
        _lib.check(self.lib.bt_frame_cache_store(*prepared[0]), "bt_frame_cache_store")

    def prepare_batch(self, windows: List[SolveWindow]):
        """The bt_window array + the flat pose block of a batch, marshalled once; begin_prepared() / solve_prepared() then cost one library
        call.  `batch.poses` ([sum n_frames, 16] float32) is the input pose block: rewrite it in place between calls if the poses change."""
        arr, poses, keep = self._marshal(windows)
        off = np.cumsum([0] + [w.n_frames for w in windows])
        return _PreparedBatch(arr, np.ascontiguousarray(poses, np.float32), keep, off)

    def begin_prepared(self, batch):
        _lib.check(self.lib.bt_solve_windows_begin(self.ctx, len(batch.keep), batch.arr, self.params, _lib.ptr(batch.poses), self.stream),
                   "bt_solve_windows_begin")

    def end_prepared(self, batch, out: np.ndarray = None) -> np.ndarray:
        """Poses of the oldest batch in flight as one [sum n_frames, 4, 4] array (batch.off gives the windows' first frames)."""
        if out is None:
            out = np.empty((batch.poses.shape[0], 4, 4), np.float32)
        _lib.check(self.lib.bt_solve_windows_end(self.ctx, _lib.ptr(out)), "bt_solve_windows_end")
        return out

    def solve_prepared(self, batch, out: np.ndarray = None) -> np.ndarray:
        if out is None:
            out = np.empty((batch.poses.shape[0], 4, 4), np.float32)
        np.copyto(out.reshape(-1, 16), batch.poses)
        _lib.check(self.lib.bt_solve_windows(self.ctx, len(batch.keep), batch.arr, self.params, _lib.ptr(out), self.stream), "bt_solve_windows")
        return out

    # ---- reference-shaped single-window call (LossGPU.h:50) -------------------------------------------------
    def optimizeFrames(self, global_corres, n_match_per_pair, n_frames, H, W, depths_gpu, colors_gpu, normals_gpu, poses, K,
                       dense_pairs=None, compat_flip=True):
        """poses: [n_frames,4,4] float32, modified in place (the reference's in-out std::vector<Eigen::Matrix4f>).
        n_match_per_pair and colors_gpu are accepted and ignored, as in the reference (LossGPU.cu:53, SBA.cpp:28-32)."""
        poses_arr = np.asarray(poses)
        win = SolveWindow(global_corres, H, W, depths_gpu[:n_frames], normals_gpu[:n_frames], poses_arr[:n_frames], K, dense_pairs, compat_flip)
        out = self.optimizeWindows([win])[0]
        poses_arr[:n_frames] = out
        return poses_arr

    # ---- batched form ---------------------------------------------------------------------------------------------
    def _marshal(self, windows: List[SolveWindow]):
        n = len(windows)
        arr = (_lib.Window * n)()
        sz = ctypes.sizeof(_lib.Window)
        base = ctypes.addressof(arr)
        for i, w in enumerate(windows):
            ctypes.memmove(base + i * sz, ctypes.addressof(w.c_window()), sz)
        poses = np.concatenate([w.poses.reshape(-1, 16) for w in windows], 0)
        return arr, poses, windows

    def optimizeWindows(self, windows: List[SolveWindow]) -> List[np.ndarray]:
        arr, poses, keep = self._marshal(windows)
        _lib.check(self.lib.bt_solve_windows(self.ctx, len(windows), arr, self.params, _lib.ptr(poses), self.stream), "bt_solve_windows")
        del keep
        return self._split(windows, poses)

    # ---- streaming form: up to two batches in flight, the host side of batch k+1 overlaps the GPU side of batch k ----------------
    def begin(self, windows: List[SolveWindow]):
        arr, poses, keep = self._marshal(windows)
        _lib.check(self.lib.bt_solve_windows_begin(self.ctx, len(windows), arr, self.params, _lib.ptr(poses), self.stream), "bt_solve_windows_begin")
        if not hasattr(self, "_inflight"):
            self._inflight = []
        self._inflight.append((windows, poses, keep, arr))

    def end(self) -> List[np.ndarray]:
        if not getattr(self, "_inflight", None):      # nothing begun: let the library say so
            _lib.check(self.lib.bt_solve_windows_end(self.ctx, None), "bt_solve_windows_end")
        windows, poses, _, _ = self._inflight.pop(0)
        out = np.empty_like(poses)
        _lib.check(self.lib.bt_solve_windows_end(self.ctx, _lib.ptr(out)), "bt_solve_windows_end")
        return self._split(windows, out)

    @staticmethod
    def _split(windows, poses):
        out, o = [], 0
        p4 = poses.reshape(-1, 4, 4)          # `poses` is a fresh array owned by this call: per-window views, no copies
        for w in windows:
            out.append(p4[o:o + w.n_frames])
            o += w.n_frames
        return out

    # split API used by bench.py to time the resident-input kernel path separately from staging
    def stage(self, windows: List[SolveWindow]):
        arr, poses, keep = self._marshal(windows)
        _lib.check(self.lib.bt_solve_stage(self.ctx, len(windows), arr, self.params, _lib.ptr(poses), self.stream), "bt_solve_stage")
        self._staged = (windows, poses, keep, arr)

    def run(self):
        _lib.check(self.lib.bt_solve_run(self.ctx, self.stream), "bt_solve_run")

    def fetch(self) -> List[np.ndarray]:
        windows, poses, _, _ = self._staged
        out = np.empty_like(poses)
        _lib.check(self.lib.bt_solve_fetch(self.ctx, _lib.ptr(out), self.stream), "bt_solve_fetch")
        return self._split(windows, out)

    def stats(self) -> dict:
        st = _lib.SolveStats()
        _lib.check(self.lib.bt_solve_get_stats(self.ctx, st), "bt_solve_get_stats")
        return {"n_windows": st.n_windows, "n_tiles_total": st.n_tiles_total, "n_kernel_launches": st.n_kernel_launches,
                "n_src_pixels": int(st.n_src_pixels)}

    def enable_timing(self, on=True):
        _lib.check(self.lib.bt_solve_enable_timing(self.ctx, 1 if on else 0), "bt_solve_enable_timing")

    def timing_ms(self):
        ms = (ctypes.c_float * 3)()
        _lib.check(self.lib.bt_solve_get_timing(self.ctx, ms), "bt_solve_get_timing")
        return {"prep": ms[0], "plan": ms[1], "solve": ms[2]}

    def host_timing_us(self):
        us = (ctypes.c_double * 6)()
        _lib.check(self.lib.bt_solve_get_host_timing(self.ctx, us), "bt_solve_get_host_timing")
        return {"tables_upload": us[0], "prep_launch": us[1], "scan_stage_upload": us[2], "solve_launch": us[3], "fetch_wait": us[4], "total": us[5]}

    def enable_profile(self, max_records=200000):
        _lib.check(self.lib.bt_solve_enable_profile(self.ctx, max_records), "bt_solve_enable_profile")
        self._prof_cap = max_records

    def get_profile(self):
        out = np.zeros((self._prof_cap, 12), np.int64)
        n = self.lib.bt_solve_get_profile(self.ctx, _lib.ptr(out), self._prof_cap)
        if n < 0:
            _lib.check(n, "bt_solve_get_profile")
        return out[:n]

    def enable_debug(self, on=True):
        _lib.check(self.lib.bt_solve_enable_debug(self.ctx, 1 if on else 0), "bt_solve_enable_debug")

    def debug_counts(self, w: int, n_pairs: int):
        c = np.zeros(n_pairs, np.float32)
        _lib.check(self.lib.bt_solve_debug_counts(self.ctx, w, n_pairs, _lib.ptr(c)), "bt_solve_debug_counts")
        return c

    def debug_dense(self, w: int, n_frames: int):
        dim = 6 * n_frames
        J = np.zeros((dim, dim), np.float32)
        r = np.zeros(dim, np.float32)
        _lib.check(self.lib.bt_solve_debug_dense(self.ctx, w, _lib.ptr(J), _lib.ptr(r)), "bt_solve_debug_dense")
        return J, r

    def debug_system(self, w: int, n_frames: int):
        """(A, rhs, minv, delta) the PCG of the last GN iteration of window w solved: unknowns of frames 1..N-1, trans 0-2 / rot 3-5."""
        dim = 6 * (n_frames - 1)
        A = np.zeros((dim, dim), np.float32)
        rhs, minv, delta = (np.zeros(dim, np.float32) for _ in range(3))
        _lib.check(self.lib.bt_solve_debug_system(self.ctx, w, n_frames, *(_lib.ptr(v) for v in (A, rhs, minv, delta))), "bt_solve_debug_system")
        return A, rhs, minv, delta
