"""numpy restatement of the reference's match images (SiftManager::vizCorresBetween, src/FeatureManager.cpp:760-796), which end in
cv::drawMatches(..., NOT_DRAW_SINGLE_POINTS) of OpenCV 4.x (DESIGN.md §3.11):

- crop: the masked colour cut to the ROI [roi2, roi3) x [roi0, roi1);
- scale = min(900 / rowsA, 900 / rowsB) in integer division; each crop resized by it with 8-bit INTER_LINEAR (a copy at scale 1);
- keypoints ((u - roi0) scale, (v - roi2) scale) in float32, in list order;
- the canvas: zeros, max(rowsA, rowsB) x (colsA + colsB), A at the left, B to its right;
- per match: a colour from cv::RNG (multiply-with-carry, coefficient 4164903690), a circle (radius 3, thickness 1, LINE_AA, shift 4) at
  kp1 clipped to the A half and one at kp2 clipped to the B half, then a LINE_AA line (shift 4) on the whole canvas from kp1 to
  (min(kp2.x + colsA, cols - 1), kp2.y);
- the circle is EllipseEx -> ellipse2Poly (a 30 degree step for a 3-pixel radius) -> an open PolyLine of LineAA segments;
- LineAA: clipLine, then 16.16 fixed-point steps along the major axis, three pixels across, each with an alpha from FilterTable scaled by
  the slope and end-point corrections; each channel is blended twice, v += ((c - v) a + 127) >> 8.

Every primitive becomes a list of fragments (x, y, alpha) whose pixels are distinct within the list (a LineAA call never visits a pixel
twice), so an image is the fold of its fragments in drawing order.  The device draws the same fragments (csrc/matchviz.cu)."""
from __future__ import annotations

import numpy as np

from oracle.segment_oracle import _coeffs

XY_SHIFT = 16
XY_ONE = 1 << XY_SHIFT
DRAW_SHIFT = 4
RNG_COEFF = 4164903690
RNG_DEFAULT = 0xFFFFFFFF

SLOPE_CORR = (181, 181, 181, 182, 182, 183, 184, 185, 187, 188, 190, 192, 194, 196, 198, 201,
              203, 206, 209, 211, 214, 218, 221, 224, 227, 231, 235, 238, 242, 246, 250, 254)
FILTER = np.array([168, 177, 185, 194, 202, 210, 218, 224, 231, 236, 241, 246, 249, 252, 254, 254,
                   254, 254, 252, 249, 246, 241, 236, 231, 224, 218, 210, 202, 194, 185, 177, 168,
                   158, 149, 140, 131, 122, 114, 105, 97, 89, 82, 75, 68, 62, 56, 50, 45,
                   40, 36, 32, 28, 25, 22, 19, 16, 14, 12, 11, 9, 8, 7, 5, 5], np.int64)


# ---- cv::RNG and the colour of a match

def rng_next(state: int) -> int:
    """cv::RNG::next: the new 64-bit state (its low 32 bits are the value drawn)."""
    return ((state & 0xFFFFFFFF) * RNG_COEFF + (state >> 32)) & 0xFFFFFFFFFFFFFFFF


def rng_seed(seed: int) -> int:
    """cv::RNG(seed) / cv2.setRNGSeed: a zero seed means the default state."""
    return seed & 0xFFFFFFFFFFFFFFFF or RNG_DEFAULT


def match_colour(state: int):
    """((B, G, R), state after): Scalar(rng(256), rng(256), rng(256)) with its arguments evaluated right to left, as the OpenCV build
    of the reference and of cv2 does it: the first draw is R, the last is B."""
    d = []
    for _ in range(3):
        state = rng_next(state)
        d.append((state & 0xFFFFFFFF) % 256)
    return (d[2], d[1], d[0]), state


def rng_advance(state: int, n_matches: int) -> int:
    """The state after drawing n_matches images' worth of colours (three draws per match)."""
    for _ in range(3 * n_matches):
        state = rng_next(state)
    return state


# ---- crop and resize

def crop(colour, roi):
    """The ROI of the (masked) colour, rows [roi2, roi3), columns [roi0, roi1)."""
    u0, u1, v0, v1 = (int(x) for x in roi)
    return np.ascontiguousarray(np.asarray(colour, np.uint8)[v0:v1, u0:u1])


def viz_scale(rows_a: int, rows_b: int) -> int:
    return min(900 // rows_a, 900 // rows_b)


def resize_int(img, s: int):
    """cv::resize(img, {0, 0}, s, s) with INTER_LINEAR on 8-bit channels: a copy at s = 1."""
    img = np.asarray(img, np.uint8)
    if s == 1:
        return img.copy()
    Hs, Ws = img.shape[:2]
    sx0, sx1, a0, a1 = _coeffs(Ws * s, Ws, True)
    sy0, sy1, b0, b1 = _coeffs(Hs * s, Hs, False)
    I = img.astype(np.int64)
    hr = I[:, sx0] * a0[None, :, None] + I[:, sx1] * a1[None, :, None]
    t0 = (b0[:, None, None] * (hr[sy0] >> 4)) >> 16
    t1 = (b1[:, None, None] * (hr[sy1] >> 4)) >> 16
    return np.clip((t0 + t1 + 2) >> 2, 0, 255).astype(np.uint8)


def keypoints(uv, roi_a, roi_b, s: int):
    """float32 [n, 4] (xA, yA, xB, yB): ((u - roi0) scale, (v - roi2) scale), each operation rounded to float32."""
    uv = np.asarray(uv, np.float32).reshape(-1, 4)
    f = np.float32
    off = np.array([roi_a[0], roi_a[2], roi_b[0], roi_b[2]], np.float32)
    return ((uv - off).astype(f) * f(s)).astype(f)


# ---- LineAA and the circle polygon

def _tdiv(a: int, b: int) -> int:
    """C integer division (towards zero)."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def clip_line(w: int, h: int, p1, p2):
    """cv::clipLine on a w x h rectangle (16.16 sizes already shifted): (inside, p1, p2)."""
    if w <= 0 or h <= 0:
        return False, p1, p2
    right, bottom = w - 1, h - 1
    x1, y1 = p1
    x2, y2 = p2
    c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8
    c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8
    if (c1 & c2) == 0 and (c1 | c2) != 0:
        if c1 & 12:
            a = 0 if c1 < 8 else bottom
            x1 += int(float(a - y1) * (x2 - x1) / (y2 - y1))
            y1 = a
            c1 = (x1 < 0) + (x1 > right) * 2
        if c2 & 12:
            a = 0 if c2 < 8 else bottom
            x2 += int(float(a - y2) * (x2 - x1) / (y2 - y1))
            y2 = a
            c2 = (x2 < 0) + (x2 > right) * 2
        if (c1 & c2) == 0 and (c1 | c2) != 0:
            if c1:
                a = 0 if c1 == 1 else right
                y1 += int(float(a - x1) * (y2 - y1) / (x2 - x1))
                x1 = a
                c1 = 0
            if c2:
                a = 0 if c2 == 1 else right
                y2 += int(float(a - x2) * (y2 - y1) / (x2 - x1))
                x2 = a
                c2 = 0
    return (c1 | c2) == 0, (x1, y1), (x2, y2)


def line_aa(w: int, h: int, p1, p2):
    """Fragments (x, y, alpha) int64 arrays of cv::LineAA from p1 to p2 (16.16) on a w x h image, pixels distinct."""
    e = np.zeros(0, np.int64)
    ok, (x1, y1), (x2, y2) = clip_line(w << XY_SHIFT, h << XY_SHIFT, p1, p2)
    if not ok:
        return e, e, e
    dx, dy = x2 - x1, y2 - y1
    ax, ay = abs(dx), abs(dy)
    xmajor = ax > ay
    if xmajor:
        if dx < 0:
            dy = -dy
            x1, x2, y1, y2 = x2, x1, y2, y1
        step = _tdiv(dy << XY_SHIFT, ax | 1)
        x2 += XY_ONE
        ecount = (x2 >> XY_SHIFT) - (x1 >> XY_SHIFT)
        j = -(x1 & (XY_ONE - 1))
        y1 += ((step * j) >> XY_SHIFT) + (XY_ONE >> 1)
        i, j = (x1 >> (XY_SHIFT - 7)) & 0x78, (x2 >> (XY_SHIFT - 7)) & 0x78
        major0, minor0 = x1 >> XY_SHIFT, y1
        n_major, n_minor = w, h
    else:
        if dy < 0:
            dx = -dx
            x1, x2, y1, y2 = x2, x1, y2, y1
        step = _tdiv(dx << XY_SHIFT, ay | 1)
        y2 += XY_ONE
        ecount = (y2 >> XY_SHIFT) - (y1 >> XY_SHIFT)
        j = -(y1 & (XY_ONE - 1))
        x1 += ((step * j) >> XY_SHIFT) + (XY_ONE >> 1)
        i, j = (y1 >> (XY_SHIFT - 7)) & 0x78, (y2 >> (XY_SHIFT - 7)) & 0x78
        major0, minor0 = y1 >> XY_SHIFT, x1
        n_major, n_minor = h, w
    slope = (step >> (XY_SHIFT - 5)) & 0x3F
    slope ^= 0x3F if step < 0 else 0
    slope = 0x100 if slope & 0x20 else SLOPE_CORR[slope]
    t0, t1, t2 = slope << 7, ((0x78 - i) | 4) * slope, (j | 4) * slope
    ep = [0] * 9
    ep[8] = slope
    ep[1] = ep[3] = ((((j - i) & 0x78) | 4) * slope >> 8) & 0x1FF
    ep[2] = (t1 >> 8) & 0x1FF
    ep[4] = ((((j - i) + 0x80) | 4) * slope >> 8) & 0x1FF
    ep[5] = ((t1 + t0) >> 8) & 0x1FF
    ep[6] = (t2 >> 8) & 0x1FF
    ep[7] = ((t2 + t0) >> 8) & 0x1FF
    ep = np.array(ep, np.int64)
    k = np.arange(ecount + 1, dtype=np.int64)
    sc, ec = k, ecount - k
    major = major0 + k
    minor = minor0 + k * step
    keep = (major >= 0) & (major < n_major)
    sc, ec, major, minor = sc[keep], ec[keep], major[keep], minor[keep]
    corr = ep[(((sc >= 2) + 1) & (sc | 2)) * 3 + (((ec >= 2) + 1) & (ec | 2))]
    dist = (minor >> (XY_SHIFT - 5)) & 31
    m0 = (minor >> XY_SHIFT) - 1
    mj, mn, al = [], [], []
    for o, idx in ((0, dist + 32), (1, dist), (2, 63 - dist)):
        a = (corr * FILTER[idx] >> 8) & 0xFF
        q = m0 + o
        ok = (q >= 0) & (q < n_minor)
        mj.append(major[ok]); mn.append(q[ok]); al.append(a[ok])
    mj, mn, al = np.concatenate(mj), np.concatenate(mn), np.concatenate(al)
    return (mj, mn, al) if xmajor else (mn, mj, al)


_SIN = np.round(np.sin(np.deg2rad(np.arange(451))), 7).astype(np.float32)      # OpenCV's SinTable: 7-digit float literals


def circle_poly(cx16: int, cy16: int, r16: int):
    """EllipseEx's polygon (16.16) of cv::circle(center, radius, thickness 1, LINE_AA, shift 4), centre and radius in 1/16 pixels."""
    shift = XY_SHIFT - DRAW_SHIFT
    cx, cy, r = cx16 << shift, cy16 << shift, r16 << shift
    d = (r + (XY_ONE >> 1)) >> XY_SHIFT
    delta = 90 if d < 3 else 30 if d < 10 else 18 if d < 15 else 5
    v = []
    prev = None
    for ang in range(0, 360 + delta, delta):
        ang = min(ang, 360)
        x = float(r) * float(_SIN[450 - ang])
        y = float(r) * float(_SIN[ang])
        px = float(cx) + x * 1.0 - y * 0.0
        py = float(cy) + x * 0.0 + y * 1.0
        qx = int(np.rint(px / XY_ONE)) << XY_SHIFT
        qy = int(np.rint(py / XY_ONE)) << XY_SHIFT
        qx += int(np.rint(px - qx))
        qy += int(np.rint(py - qy))
        if (qx, qy) != prev:
            v.append((qx, qy))
            prev = (qx, qy)
    if len(v) == 1:
        v = [(cx, cy), (cx, cy)]
    return v


def circle_aa(w: int, h: int, cx16: int, cy16: int, r16: int = 3 << DRAW_SHIFT):
    """Fragment lists, one per polygon segment in drawing order."""
    v = circle_poly(cx16, cy16, r16)
    return [line_aa(w, h, v[k - 1], v[k]) for k in range(1, len(v))]


# ---- one image

def blend(img, x, y, a, colour):
    """ICV_PUT_POINT on a 3-channel image for fragments at distinct pixels: each channel blended twice."""
    if len(x) == 0:
        return
    v = img[y, x].astype(np.int64)
    c = np.asarray(colour, np.int64)[None, :]
    aa = a[:, None]
    v = v + (((c - v) * aa + 127) >> 8)
    v = v + (((c - v) * aa + 127) >> 8)
    img[y, x] = v.astype(np.uint8)


def draw_matches(img_a, img_b, kp, state: int = RNG_DEFAULT):
    """cv::drawMatches(img_a, kpA, img_b, kpB, matches i <-> i, random colours, NOT_DRAW_SINGLE_POINTS): (image, RNG state after).
    kp: float32 [n, 4] (xA, yA, xB, yB)."""
    ha, wa = img_a.shape[:2]
    hb, wb = img_b.shape[:2]
    H, W = max(ha, hb), wa + wb
    out = np.zeros((H, W, 3), np.uint8)
    out[:ha, :wa] = img_a
    out[:hb, wa:] = img_b
    kp = np.asarray(kp, np.float32).reshape(-1, 4)
    r16 = lambda t: int(np.rint(np.float32(t) * np.float32(1 << DRAW_SHIFT)))
    for xa, ya, xb, yb in kp:
        col, state = match_colour(state)
        for (x, y, a) in circle_aa(wa, ha, r16(xa), r16(ya)):
            blend(out, x, y, a, col)
        for (x, y, a) in circle_aa(wb, hb, r16(xb), r16(yb)):
            blend(out, x + wa, y, a, col)
        x2 = min(np.float32(xb + np.float32(wa)), np.float32(W - 1))
        sh = XY_SHIFT - DRAW_SHIFT
        x, y, a = line_aa(W, H, (r16(xa) << sh, r16(ya) << sh), (r16(x2) << sh, r16(yb) << sh))
        blend(out, x, y, a, col)
    return out, state


def match_image(colour_a, roi_a, colour_b, roi_b, uv, state: int = RNG_DEFAULT):
    """vizCorresBetween's picture before imwrite: (image, RNG state after).  uv: [n, 4] (uA, vA, uB, vB) in full-image pixels."""
    ca, cb = crop(colour_a, roi_a), crop(colour_b, roi_b)
    s = viz_scale(ca.shape[0], cb.shape[0])
    return draw_matches(resize_int(ca, s), resize_int(cb, s), keypoints(uv, roi_a, roi_b, s), state)


def image_shape(roi_a, roi_b):
    """(rows, cols) of the match image of two ROIs."""
    ha, wa = int(roi_a[3]) - int(roi_a[2]), int(roi_a[1]) - int(roi_a[0])
    hb, wb = int(roi_b[3]) - int(roi_b[2]), int(roi_b[1]) - int(roi_b[0])
    s = viz_scale(ha, hb)
    return max(ha, hb) * s, (wa + wb) * s
