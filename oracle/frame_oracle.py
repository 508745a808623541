"""TEST INFRASTRUCTURE ONLY — CPU restatement (numpy, float32) of the reference's per-frame depth front end.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this; nothing under bundletrack_b200/ does.

Follows, statement by statement (same neighbour order in the float accumulations, same float/double comparisons):
  erodeDepthMapDevice                          /root/reference/src/cuda/CUDAImageUtil.cu:676-718
  gaussFilterDepthMapDevice                    /root/reference/src/cuda/CUDAImageUtil.cu:735-796
  convertDepthFloatToCameraSpaceFloat4_Kernel  /root/reference/src/cuda/CUDAImageUtil.cu:310-326
  computeNormals_Kernel                        /root/reference/src/cuda/CUDAImageUtil.cu:342-413
in the order Frame::processDepth / Frame::depthToCloudAndNormals call them (/root/reference/src/Frame.cpp:152-233).
Pinned against the reference's own kernels (oracle/_ref, compiled with the reference's -use_fast_math) through
tests/golden/ref_frame_*.npz (made by scripts/make_golden_frame.py): the only differences are the fast-math exp and
division of the reference build, i.e. ~1e-7 relative on the filtered depth and a handful of threshold flips per image.
"""
import numpy as np

DEFAULTS = dict(erode_radius=1, erode_diff=0.001, erode_ratio=0.8, bf_radius=2, sigma_D=2.0, sigma_R=100000.0)   # config_nocs.yml:12-20
F = np.float32


def _shift(a, dy, dx, fill=0.0):
    """out[y,x] = a[y+dy, x+dx] where inside the image, `fill` elsewhere; also returns the inside mask."""
    H, W = a.shape
    out = np.full_like(a, fill)
    inside = np.zeros((H, W), bool)
    ys, ye = max(0, -dy), min(H, H - dy)
    xs, xe = max(0, -dx), min(W, W - dx)
    if ys < ye and xs < xe:
        out[ys:ye, xs:xe] = a[ys + dy:ye + dy, xs + dx:xe + dx]
        inside[ys:ye, xs:xe] = True
    return out, inside


def erode(d, radius, diff, ratio):
    d = d.astype(F)
    count = np.zeros(d.shape, np.uint32)
    for i in range(-radius, radius + 1):
        for j in range(-radius, radius + 1):
            nb, inside = _shift(d, i, j)
            bad = (nb == F(-np.inf)) | (nb < F(0.1)) | (np.abs(nb - d) > F(diff))
            count += (inside & bad).astype(np.uint32)
    total = F((2 * radius + 1) ** 2)
    frac = count.astype(F) / total
    out = np.where(frac >= F(ratio), F(0), d)
    return np.where(d <= F(0.1), F(0), out).astype(F)


def gauss(d, radius, sigma_D, sigma_R):
    d = d.astype(F)
    H, W = d.shape
    mean = np.zeros((H, W), F)
    nv = np.zeros((H, W), np.int32)
    offs = [(m, n) for m in range(-radius, radius + 1) for n in range(-radius, radius + 1)]    # x offset outer, y offset inner
    for m, n in offs:
        nb, inside = _shift(d, n, m)
        ok = inside & (nb >= F(0.1))
        nv += ok
        mean = np.where(ok, mean + nb, mean).astype(F)
    with np.errstate(divide="ignore", invalid="ignore"):
        mean = (mean / nv.astype(F)).astype(F)
    s = np.zeros((H, W), F)
    sw = np.zeros((H, W), F)
    two_sd = F(2.0) * F(sigma_D) * F(sigma_D)
    two_sr = F(2) * F(sigma_R) * F(sigma_R)
    for m, n in offs:
        nb, inside = _shift(d, n, m)
        with np.errstate(invalid="ignore"):
            ok = inside & (nb >= F(0.1)) & (np.abs(nb - mean).astype(np.float64) < 0.01)
        arg = (-F(m * m + n * n) / two_sd - (d - nb) * (d - nb) / two_sr).astype(F)
        w = np.exp(arg).astype(F)
        sw = np.where(ok, sw + w, sw).astype(F)
        s = np.where(ok, s + w * nb, s).astype(F)
    with np.errstate(divide="ignore", invalid="ignore"):
        out = np.where((nv > 0) & (sw > 0), s / sw, F(0))
    return out.astype(F)


def inverse_intrinsics(K):
    """Eigen::Matrix3f::inverse() of [[fx,0,cx],[0,fy,cy],[0,0,1]] (Frame.cpp:189): cofactors times 1/det, in float."""
    fx, fy, cx, cy = (F(v) for v in K)
    invdet = F(1.0) / (fx * fy)
    return fy * invdet, fx * invdet, (F(0) * cy - cx * fy) * invdet, -(fx * cy - cx * F(0)) * invdet


def to_camera(d, K):
    d = d.astype(F)
    H, W = d.shape
    k00, k11, k02, k12 = inverse_intrinsics(K)
    x = np.arange(W, dtype=F)[None, :] * np.ones((H, 1), F)
    y = np.arange(H, dtype=F)[:, None] * np.ones((1, W), F)
    xd, yd = (x * d).astype(F), (y * d).astype(F)
    out = np.zeros((H, W, 4), F)
    ok = d.astype(np.float64) >= 0.1
    out[..., 0] = np.where(ok, ((k00 * xd + F(0) * yd).astype(F) + k02 * d).astype(F) + F(0) * d, 0)
    out[..., 1] = np.where(ok, ((F(0) * xd + k11 * yd).astype(F) + k12 * d).astype(F) + F(0) * d, 0)
    out[..., 2] = np.where(ok, d, 0)
    out[..., 3] = np.where(ok, F(1), 0)
    return out


def normals(xyz):
    H, W, _ = xyz.shape
    P = xyz[..., :3].astype(F)
    z = P[..., 2]
    out = np.zeros((H, W, 4), F)

    def sh(a, dy, dx):
        o = np.zeros_like(a)
        ys, ye = max(0, -dy), min(H, H - dy)
        xs, xe = max(0, -dx), min(W, W - dx)
        o[ys:ye, xs:xe] = a[ys + dy:ye + dy, xs + dx:xe + dx]
        return o
    PC, MC, CP, CM = sh(P, 1, 0), sh(P, -1, 0), sh(P, 0, 1), sh(P, 0, -1)
    zt = F(0.02)
    def near(Q):
        return (Q[..., 2].astype(np.float64) >= 0.1) & (np.abs(Q[..., 2] - z) <= zt)
    pc, mc, cp, cm = near(PC), near(MC), near(CP), near(CM)
    a = np.where((pc & mc)[..., None], PC - MC, np.where(pc[..., None], PC - P, MC - P)).astype(F)
    b = np.where((cp & cm)[..., None], CP - CM, np.where(cp[..., None], CP - P, CM - P)).astype(F)
    n = np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                  a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1).astype(F)
    l = np.sqrt((n[..., 0] * n[..., 0] + n[..., 1] * n[..., 1]).astype(F) + n[..., 2] * n[..., 2]).astype(F)
    with np.errstate(divide="ignore", invalid="ignore"):
        n = (n / l[..., None]).astype(F)
        flip = ((n[..., 0] * -P[..., 0] + n[..., 1] * -P[..., 1]).astype(F) + n[..., 2] * -P[..., 2]) < 0
    n = np.where(flip[..., None], -n, n)
    interior = np.zeros((H, W), bool)
    interior[1:H - 1, 1:W - 1] = True
    ok = interior & ~(z.astype(np.float64) < 0.1) & (pc | mc) & (cp | cm) & (l > 0)
    out[..., :3] = np.where(ok[..., None], n, 0)
    return out


def preprocess(depth_raw, K, dp=None):
    """Frame::processDepth + depthToCloudAndNormals.  Returns (depth [H,W], xyz [H,W,4], normal [H,W,4])."""
    dp = dict(DEFAULTS, **(dp or {}))
    d = erode(np.asarray(depth_raw, F), int(dp["erode_radius"]), dp["erode_diff"], dp["erode_ratio"])
    d = gauss(d, int(dp["bf_radius"]), dp["sigma_D"], dp["sigma_R"])
    d = gauss(d, int(dp["bf_radius"]), dp["sigma_D"], dp["sigma_R"])
    xyz = to_camera(d, K)
    return d, xyz, normals(xyz)
