"""Host-side mirror of the reference's per-frame depth front end (`Frame::processDepth` + `Frame::depthToCloudAndNormals`,
/root/reference/src/Frame.cpp:152-233) on top of the C-ABI `bt_frames_preprocess`, with the object mask
(`Frame::segmentationByMaskFile` + `invalidatePixelsByMask`, Frame.cpp:236-374) through `bt_frames_preprocess_masked` and the
LF-Net request image (FeatureManager.cpp:813-873) through `bt_lfnet_request`.  All arithmetic runs in
lib/libbundletrack_b200.so on the GPU; this file only marshals device pointers."""
from __future__ import annotations

import ctypes
from typing import Sequence

from . import _lib
from .config import depth_params, mask_mode


def _ptr(x) -> int:
    return int(x.data_ptr()) if hasattr(x, "data_ptr") else int(x)


class FrameFrontEnd:
    def __init__(self, yml=None, device: int = 0, stream: int = 0, ctx=None):
        self.lib = _lib.load()
        self.params = depth_params(yml)
        self.mask_mode = mask_mode(yml)
        self.stream = ctypes.c_void_p(stream)
        self._roi_dev, self._roi_cap, self._last_roi = ctypes.c_void_p(), 0, None
        self._own = ctx is None
        self.ctx = ctypes.c_void_p() if ctx is None else ctx
        if self._own:
            _lib.check(self.lib.bt_ctx_create(ctypes.byref(self.ctx), ctypes.c_int(device)), "bt_ctx_create")

    def close(self):
        if getattr(self, "_roi_dev", None):
            self.lib.bt_dev_free(self._roi_dev)
            self._roi_dev, self._roi_cap, self._last_roi = ctypes.c_void_p(), 0, None
        if self._own and self.ctx:
            self.lib.bt_ctx_destroy(self.ctx)
            self.ctx = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def process(self, depth_raw: Sequence, H: int, W: int, K, depth_out: Sequence, normal_out: Sequence, xyz_out: Sequence = None):
        """depth_raw/depth_out: per-frame device float32 [H,W]; normal_out/xyz_out: device float32 [H,W,4].
        K = (fx, fy, cx, cy) or a 3x3 matrix.  Outputs are written in place; returns None."""
        import numpy as np
        Kn = np.asarray(K, np.float64)
        fx, fy, cx, cy = (Kn[0, 0], Kn[1, 1], Kn[0, 2], Kn[1, 2]) if Kn.ndim == 2 else Kn
        n = len(depth_raw)
        arr = lambda seq: (ctypes.c_void_p * n)(*[_ptr(t) for t in seq])
        a_in, a_out, a_n = arr(depth_raw), arr(depth_out), arr(normal_out)
        a_x = arr(xyz_out) if xyz_out is not None else None
        _lib.check(self.lib.bt_frames_preprocess(self.ctx, ctypes.c_int(n), a_in, ctypes.c_int(H), ctypes.c_int(W),
                                                 ctypes.c_float(fx), ctypes.c_float(fy), ctypes.c_float(cx), ctypes.c_float(cy),
                                                 ctypes.byref(self.params), a_out, a_x, a_n, self.stream), "bt_frames_preprocess")

    def process_masked(self, depth_raw: Sequence, mask: Sequence, H: int, W: int, K, depth_out: Sequence, normal_out: Sequence,
                       fg_out: Sequence, xyz_out: Sequence = None, mode: int = None, roi_out=None, fetch_roi: bool = True):
        """`process` plus the object mask (Frame::segmentationByMaskFile + invalidatePixelsByMask): depth_raw is per-frame device float32
        metres, or uint16 millimetres as the depth PNG holds them (bt_frames_preprocess_masked_u16 converts them as Utils::readDepthImage does;
        every frame of a call has the same dtype); mask/fg_out are per-frame device
        uint8 [H,W] (fg_out = Frame::_fg_mask, not the mask's own buffer); the maps are zeroed where fg == 0.  mode: _lib.BT_MASK_*
        (default: config.mask_mode of this object's yml).  roi_out: device int32 [n,4] (default: a buffer this object keeps, which
        `lfnet_request` reads by default).  Returns the ROI (umin, umax, vmin, vmax) per frame as numpy int32 [n,4], read back with
        one small copy that waits for the stream, or None with fetch_roi=False."""
        import numpy as np
        Kn = np.asarray(K, np.float64)
        fx, fy, cx, cy = (Kn[0, 0], Kn[1, 1], Kn[0, 2], Kn[1, 2]) if Kn.ndim == 2 else Kn
        n = len(depth_raw)
        arr = lambda seq: (ctypes.c_void_p * n)(*[_ptr(t) for t in seq])
        dtypes = {str(getattr(t, "dtype", "float32")).replace("torch.", "") for t in depth_raw}
        if len(dtypes) != 1 or not dtypes <= {"float32", "uint16"}:
            raise _lib.BtError(f"process_masked: depth frames must all be float32 or all uint16, got {sorted(dtypes)}")
        u16 = dtypes == {"uint16"}
        fn = self.lib.bt_frames_preprocess_masked_u16 if u16 else self.lib.bt_frames_preprocess_masked
        roi = _ptr(roi_out) if roi_out is not None else self._roi_buffer(n)
        self._last_roi = roi
        _lib.check(fn(
            self.ctx, ctypes.c_int(n), arr(depth_raw), arr(mask), ctypes.c_int(self.mask_mode if mode is None else mode), ctypes.c_int(H), ctypes.c_int(W),
            ctypes.c_float(fx), ctypes.c_float(fy), ctypes.c_float(cx), ctypes.c_float(cy), ctypes.byref(self.params), arr(depth_out),
            arr(xyz_out) if xyz_out is not None else None, arr(normal_out), arr(fg_out), ctypes.c_void_p(roi), self.stream), "bt_frames_preprocess_masked" + ("_u16" if u16 else ""))
        if not fetch_roi:
            return None
        out = np.empty((n, 4), np.int32)
        _lib.check(self.lib.bt_memcpy_d2h(out.ctypes.data_as(ctypes.c_void_p), ctypes.c_void_p(roi), ctypes.c_size_t(out.nbytes), self.stream), "bt_memcpy_d2h")
        return out

    def lfnet_request(self, colour: Sequence, fg: Sequence, H: int, W: int, request_out: Sequence, roi=None):
        """Lfnet::detectFeature's request image: colour = per-frame device uint8 [H,W,3] BGR, fg = process_masked's fg_out,
        request_out = per-frame device uint8 [400,400,3].  roi: device int32 [n,4] (default: the last process_masked call's).
        Frames whose ROI fails the tracker's 10-pixel gate keep request_out as it was.  Asynchronous; returns None."""
        n = len(colour)
        if roi is None and getattr(self, "_last_roi", None) is None:
            raise _lib.BtError("lfnet_request: no ROI (call process_masked first or pass roi)")
        arr = lambda seq: (ctypes.c_void_p * n)(*[_ptr(t) for t in seq])
        r = _ptr(roi) if roi is not None else self._last_roi
        _lib.check(self.lib.bt_lfnet_request(self.ctx, ctypes.c_int(n), arr(colour), arr(fg), ctypes.c_void_p(r), ctypes.c_int(H), ctypes.c_int(W),
                                             arr(request_out), self.stream), "bt_lfnet_request")

    def _roi_buffer(self, n: int) -> int:
        if self._roi_cap < n:
            if self._roi_dev:
                self.lib.bt_dev_free(self._roi_dev)
                self._roi_dev, self._roi_cap = ctypes.c_void_p(), 0
            _lib.check(self.lib.bt_dev_alloc(ctypes.byref(self._roi_dev), ctypes.c_size_t(16 * n)), "bt_dev_alloc")
            self._roi_cap = n
        return int(self._roi_dev.value)
