"""Host-side mirror of the reference's per-frame depth front end (`Frame::processDepth` + `Frame::depthToCloudAndNormals`,
/root/reference/src/Frame.cpp:152-233) on top of the C-ABI `bt_frames_preprocess`, with the object mask
(`Frame::segmentationByMaskFile` + `invalidatePixelsByMask`, Frame.cpp:236-374) through `bt_frames_preprocess_masked` and the
LF-Net request image (FeatureManager.cpp:813-873) through `bt_lfnet_request`.  All arithmetic runs in
lib/libbundletrack_b200.so on the GPU; this file only marshals device pointers."""
from __future__ import annotations

from typing import Sequence

from . import _lib
from .config import depth_params, mask_mode


class FrameFrontEnd(_lib.Facade):
    def __init__(self, yml=None, device: int = 0, stream: int = 0, ctx=None):
        super().__init__(ctx, device, stream)
        self.params = depth_params(yml)
        self.mask_mode = mask_mode(yml)
        self._roi, self._roi_cap, self._last_roi = None, 0, None

    def close(self):
        if self._roi is not None:
            self._roi.close()
        self._roi, self._roi_cap, self._last_roi = None, 0, None
        super().close()

    def process(self, depth_raw: Sequence, H: int, W: int, K, depth_out: Sequence, normal_out: Sequence, xyz_out: Sequence = None):
        """depth_raw/depth_out: per-frame device float32 [H,W]; normal_out/xyz_out: device float32 [H,W,4].
        K = (fx, fy, cx, cy) or a 3x3 matrix.  Outputs are written in place; returns None."""
        _lib.check(self.lib.bt_frames_preprocess(self.ctx, len(depth_raw), _lib.ptrs(depth_raw), H, W, *_lib.intrinsics(K), self.params,
                                                 _lib.ptrs(depth_out), None if xyz_out is None else _lib.ptrs(xyz_out), _lib.ptrs(normal_out), self.stream),
                   "bt_frames_preprocess")

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
        n = len(depth_raw)
        dtypes = {str(getattr(t, "dtype", "float32")).replace("torch.", "") for t in depth_raw}
        if len(dtypes) != 1 or not dtypes <= {"float32", "uint16"}:
            raise _lib.BtError(f"process_masked: depth frames must all be float32 or all uint16, got {sorted(dtypes)}")
        what = "bt_frames_preprocess_masked" + ("_u16" if dtypes == {"uint16"} else "")
        roi = _lib.ptr(roi_out) if roi_out is not None else self._roi_buffer(n)
        self._last_roi = roi
        _lib.check(getattr(self.lib, what)(
            self.ctx, n, _lib.ptrs(depth_raw), _lib.ptrs(mask), self.mask_mode if mode is None else mode, H, W, *_lib.intrinsics(K), self.params,
            _lib.ptrs(depth_out), None if xyz_out is None else _lib.ptrs(xyz_out), _lib.ptrs(normal_out), _lib.ptrs(fg_out), roi, self.stream), what)
        if not fetch_roi:
            return None
        out = np.empty((n, 4), np.int32)
        _lib.check(self.lib.bt_memcpy_d2h(_lib.ptr(out), roi, out.nbytes, self.stream), "bt_memcpy_d2h")
        return out

    def lfnet_request(self, colour: Sequence, fg: Sequence, H: int, W: int, request_out: Sequence, roi=None):
        """Lfnet::detectFeature's request image: colour = per-frame device uint8 [H,W,3] BGR, fg = process_masked's fg_out,
        request_out = per-frame device uint8 [400,400,3].  roi: device int32 [n,4] (default: the last process_masked call's).
        Frames whose ROI fails the tracker's 10-pixel gate keep request_out as it was.  Asynchronous; returns None."""
        if roi is None and self._last_roi is None:
            raise _lib.BtError("lfnet_request: no ROI (call process_masked first or pass roi)")
        r = _lib.ptr(roi) if roi is not None else self._last_roi
        _lib.check(self.lib.bt_lfnet_request(self.ctx, len(colour), _lib.ptrs(colour), _lib.ptrs(fg), r, H, W, _lib.ptrs(request_out), self.stream),
                   "bt_lfnet_request")

    def _roi_buffer(self, n: int) -> "_lib.Handle":
        if self._roi_cap < n:
            if self._roi is not None:
                self._roi.close()
            self._roi, self._roi_cap = None, 0
            self._roi = _lib.Handle("bt_dev_alloc", "bt_dev_free", 16 * n)
            self._roi_cap = n
        return self._roi
