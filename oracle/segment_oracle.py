"""TEST INFRASTRUCTURE ONLY — CPU restatement (numpy / scipy, integer arithmetic) of the reference's object-mask segmentation
and of the LF-Net request image.

Only tests/ and scripts/ may import this; nothing under bundletrack_b200/ does.

Follows, statement by statement:
  Frame::segmentationByMaskFile   reference src/Frame.cpp:267-317   (largest 8-connected component -> convex hull -> fillConvexPoly,
                                                                     then a 5x5 rectangular dilation)
  Frame::invalidatePixelsByMask   src/Frame.cpp:342-374             (ROI of the dilated mask)
  Lfnet::detectFeature            src/FeatureManager.cpp:813-873    (crop to the ROI, pad to a square, resize to 400 x 400; rot_deg = 0)
OpenCV's parts are restated from its public algorithms: cv::convexHull drops collinear points, cv::fillConvexPoly (shift 0, LINE_8)
draws the Bresenham outline of every edge and fills the 16.16 fixed-point scanline spans between the two edge chains, and the 8-bit
INTER_LINEAR resize uses 11-bit coefficients with the vector path's rounding in the vertical pass.  tests/golden/ref_segment.npz
(scripts/make_golden_segment.py, recorded with OpenCV) pins all of it.
"""
import numpy as np
from scipy import ndimage

MASK_AS_IS, MASK_LARGEST_HULL = 0, 1
ROI_EMPTY = (9999, 0, 9999, 0)
REQ_SIDE = 400


def largest_component(mask):
    """(label map, winning label or 0) of the 8-connected components of mask != 0.  Ties in size go to the component whose first
    pixel in row-major order comes first."""
    lab, n = ndimage.label(np.asarray(mask) != 0, structure=np.ones((3, 3), int))
    if n == 0:
        return lab, 0
    flat = lab.ravel()
    counts = np.bincount(flat, minlength=n + 1)[1:]
    first = np.full(n, flat.size, np.int64)
    nz = np.flatnonzero(flat)
    np.minimum.at(first, flat[nz] - 1, nz)
    best = max(range(n), key=lambda i: (counts[i], -first[i]))
    return lab, best + 1


def convex_hull(pts):
    """Integer monotone chain without collinear points; pts: iterable of (x, y).  Counter-clockwise in (x, y) order."""
    p = sorted(set((int(x), int(y)) for x, y in pts))
    if len(p) <= 2:
        return p

    def cross(o, a, b):
        return (a[0] - o[0]) * (b[1] - o[1]) - (a[1] - o[1]) * (b[0] - o[0])

    lower, upper = [], []
    for q in p:
        while len(lower) >= 2 and cross(lower[-2], lower[-1], q) <= 0:
            lower.pop()
        lower.append(q)
    for q in reversed(p):
        while len(upper) >= 2 and cross(upper[-2], upper[-1], q) <= 0:
            upper.pop()
        upper.append(q)
    return lower[:-1] + upper[:-1]


def _line8(img, p0, p1):
    """cv::line with LINE_8 between integer points inside the image (the LineIterator is run left to right)."""
    (x0, y0), (x1, y1) = p0, p1
    if x1 < x0:
        x0, y0, x1, y1 = x1, y1, x0, y0
    dx, dy = x1 - x0, y1 - y0
    sy = -1 if dy < 0 else 1
    dy = abs(dy)
    vert = dy > dx
    major, minor = (dy, dx) if vert else (dx, dy)
    err = major - 2 * minor
    x, y = x0, y0
    for _ in range(major + 1):
        img[y, x] = 1
        step_minor = err < 0
        err += -2 * minor + (2 * major if step_minor else 0)
        if vert:
            y += sy
            x += 1 if step_minor else 0
        else:
            x += 1
            y += sy if step_minor else 0


def _tdiv(a, b):
    """C integer division (truncates towards zero), b > 0."""
    return a // b if a >= 0 else -((-a) // b)


def fill_convex_poly(H, W, v):
    """cv::fillConvexPoly(zeros(H, W), v, 1, LINE_8, shift 0); v: hull vertices (x, y) inside the image."""
    img = np.zeros((H, W), np.uint8)
    n = len(v)
    if n == 0:
        return img
    p0 = v[-1]
    for p in v:
        _line8(img, p0, p)
        p0 = p
    if n < 3:
        return img
    ys = [p[1] for p in v]
    ymin, ymax = min(ys), min(max(ys), H - 1)
    imin = ys.index(min(ys))
    SH, HALF = 16, 1 << 15
    edge = [dict(idx=imin, di=1, x=-(1 << SH), dx=0, ye=ymin), dict(idx=imin, di=n - 1, x=-(1 << SH), dx=0, ye=ymin)]
    edges, y = n, ymin
    while True:
        for e in edge:
            if y >= e["ye"]:
                idx0, di = e["idx"], e["di"]
                idx = (idx0 + di) % n
                while True:
                    more = edges > 0
                    edges -= 1
                    if not more:
                        break
                    ty = v[idx][1]
                    if ty > y:
                        xs, xe = v[idx0][0] << SH, v[idx][0] << SH
                        e.update(ye=ty, dx=_tdiv((xe - xs) * 2 + (ty - y), 2 * (ty - y)), x=xs, idx=idx)
                        break
                    idx0, idx = idx, (idx + di) % n
        if edges < 0:
            break
        left, right = (1, 0) if edge[0]["x"] > edge[1]["x"] else (0, 1)
        x1, x2 = (edge[left]["x"] + HALF) >> SH, (edge[right]["x"] + HALF) >> SH
        if x2 >= 0 and x1 < W:
            img[y, max(x1, 0):min(x2, W - 1) + 1] = 1
        edge[0]["x"] += edge[0]["dx"]
        edge[1]["x"] += edge[1]["dx"]
        y += 1
        if y > ymax:
            break
    return img


def hull_mask(mask):
    """The reference's NOCS branch before the dilation: fillConvexPoly of the convex hull of the largest component (0/1), or all
    zero without foreground.  The hull is built from each row's extreme columns, which have the same hull as all the pixels."""
    H, W = mask.shape
    lab, best = largest_component(mask)
    if best == 0:
        return np.zeros((H, W), np.uint8)
    sel = lab == best
    rows = np.flatnonzero(sel.any(1))
    pts = []
    for y in rows:
        xs = np.flatnonzero(sel[y])
        pts += [(xs[0], y), (xs[-1], y)]
    return fill_convex_poly(H, W, convex_hull(pts))


def dilate5(m):
    """cv::dilate with a 5 x 5 rectangle: the maximum over the in-image window."""
    return ndimage.maximum_filter(np.asarray(m, np.uint8), size=5, mode="constant", cval=0)


def roi_of(fg):
    """Frame::_roi = (umin, umax, vmin, vmax) of fg != 0, (9999, 0, 9999, 0) when empty."""
    ys, xs = np.nonzero(fg)
    if len(xs) == 0:
        return np.array(ROI_EMPTY, np.int32)
    return np.array([xs.min(), xs.max(), ys.min(), ys.max()], np.int32)


def segment(mask, mode):
    """-> (fg = Frame::_fg_mask, roi).  mode: MASK_AS_IS or MASK_LARGEST_HULL."""
    m = hull_mask(mask) if mode == MASK_LARGEST_HULL else np.asarray(mask, np.uint8)
    fg = dilate5(m)
    return fg, roi_of(fg)


def gate_ok(roi):
    """The tracker's gate (Bundler.cpp:88-93): a frame whose ROI is under 10 pixels in either direction fails."""
    return not (int(roi[1]) - int(roi[0]) < 10 or int(roi[3]) - int(roi[2]) < 10)


def _coeffs(dst, src, clamp_weights):
    """OpenCV's INTER_LINEAR source indices and 11-bit weights per destination index.  Both directions clamp the source indices to
    the image; only the horizontal one also moves the weight onto the edge sample (the vertical pass keeps the fractional weights
    and reads the edge row twice, which rounds differently in its two truncating products)."""
    scale = 1.0 / (float(dst) / float(src))
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if clamp_weights:
        lo = s < 0
        f[lo], s[lo] = 0, 0
        hi = s >= src - 1
        f[hi], s[hi] = 0, src - 1
    w0 = np.rint((np.float32(1) - f) * np.float32(2048)).astype(np.int64)
    w1 = np.rint(f * np.float32(2048)).astype(np.int64)
    return np.clip(s, 0, src - 1), np.clip(s + 1, 0, src - 1), w0, w1


def resize_linear_u8(img, side_out=REQ_SIDE):
    """cv::resize(img, {side_out, side_out}) with INTER_LINEAR on 8-bit channels (a copy when the size is already right)."""
    img = np.asarray(img, np.uint8)
    Hs, Ws = img.shape[:2]
    if Hs == side_out and Ws == side_out:
        return img.copy()
    sx0, sx1, a0, a1 = _coeffs(side_out, Ws, True)
    sy0, sy1, b0, b1 = _coeffs(side_out, Hs, False)
    I = img.astype(np.int64)
    hr = I[:, sx0] * a0[None, :, None] + I[:, sx1] * a1[None, :, None]          # horizontal pass, exact
    t0 = (b0[:, None, None] * (hr[sy0] >> 4)) >> 16                             # the vector path's 16-bit products, then (t + 2) >> 2
    t1 = (b1[:, None, None] * (hr[sy1] >> 4)) >> 16
    return np.clip((t0 + t1 + 2) >> 2, 0, 255).astype(np.uint8)


def crop_square(colour, fg, roi):
    """The side x side BGR image the reference builds before its resize: the colour, zeroed where fg == 0, cropped to
    [vmin, vmax) x [umin, umax) (the last row and column are dropped, as in the reference) and padded with zeros."""
    umin, umax, vmin, vmax = (int(v) for v in roi)
    Wr, Hr = umax - umin, vmax - vmin
    side = max(Wr, Hr)
    img = np.zeros((side, side, 3), np.uint8)
    c = np.where((np.asarray(fg) != 0)[..., None], colour, 0).astype(np.uint8)
    img[:Hr, :Wr] = c[vmin:vmin + Hr, umin:umin + Wr]
    return img


def lfnet_request(colour, fg, roi):
    """400 x 400 x 3 BGR bytes of the LF-Net request, or None when the ROI fails the tracker's gate."""
    if not gate_ok(roi):
        return None
    return resize_linear_u8(crop_square(colour, fg, roi))


def test_colour(H, W):
    """The closed-form BGR image the fixtures and tests use (no RNG, so nothing of it needs storing)."""
    y, x = np.mgrid[0:H, 0:W].astype(np.int64)
    c = np.stack([(7 * x + 3 * y + (x * y) % 29), (5 * x + 11 * y + (x ^ y) % 17), (13 * x + 2 * y + ((x + 2 * y) * (x + 1)) % 37)], -1)
    return (c & 255).astype(np.uint8)
