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


# ------------------------------------------------------------------------------------------------------------ float64 statement
TH_VALID = float(F(0.1))        # d >= 0.1f: the smallest float above 0.1, so (double)d >= 0.1 <=> d >= 0.1f for float d
TH_MEAN = 0.01                  # the filter keeps |d - mean| < 0.01 (double); for float x, x < 0.01 <=> x <= 0.01f
TH_NORMAL = float(F(0.02))      # the normals' neighbour gate |dz| <= 0.02f
U = 2.0 ** -24                  # unit roundoff of float32
ARG_NORMAL = float(np.log(2.0 ** -126))     # expf of a larger argument is a normal float
ARG_TINY = -110.0                           # expf of a smaller argument is 0 however it rounds (exp(-110) < 2^-158)
A_SUB = 2.0 ** -148                         # expf's 2 ulp where the result is subnormal (ulp 2^-149): an absolute error


def hulp(x):
    """Half a float32 ulp at |x| (the largest error of one correctly rounded float32 result near x), taken 2^-12 above |x| so that a
    value within that relative distance of the next binade is charged that binade's half ulp.  2^-150 in the subnormal range."""
    e = np.frexp(np.abs(np.asarray(x, np.float64)) * (1 + 2.0 ** -12))[1]          # |x| in [2^(e-1), 2^e): float32 ulp 2^(e-24)
    return np.ldexp(1.0, np.maximum(e - 25, -150))


def is_f32(x):
    with np.errstate(over="ignore"):
        return np.asarray(x, np.float64).astype(F).astype(np.float64) == x


class Frame64:
    """preprocess64's result: float64 depth [H,W], xyz [H,W,4], normal [H,W,4]; per-pixel bounds on the float32 device result's
    distance from them (depth_err, xyz_err [H,W] per coordinate, normal_err [H,W] per component) wherever the pixel is not tainted;
    taint [H,W] (a float32 gate decision could go the other way), and the taint of each stage (filter1, filter2: the depth after that
    pass; normal: the normal stencil's own gates); subnormal [H,W]: pixels whose depth, point or normal depends on a filter window that
    kept a weight below float32's normal range, where float32 itself loses accuracy and only the derived bounds hold."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def _filter64(d, e, t, br, sig_d, sig_r):
    """One pass of the depth filter in float64 on inputs d with error bounds e (0 = the device's input equals d bit for bit) and
    taint t.  Returns (out, err, taint, sub): sub marks the outputs whose window kept a weight below float32's normal range.

    Bounds (u = 2^-24, h(x) = half a float32 ulp at x; a sum's h is charged at each partial sum the device rounds):
      * mean: the device adds the valid taps in order and divides by nv, so |mean_f - mean| <= sum_k h(S_k) / nv + h(mean) + max e_i,
        and 0 when every partial sum and the quotient are float32 numbers and the inputs are exact.
      * mean gate: the device keeps a tap when x_f = fl(d_i - mean_f) < 0.01 and |x_f - x| <= e_i + e_mean + h(x) (0 when exact), so
        the decision is the float64 one unless | |x| - 0.01 | is within that bound: then the pixel is tainted.
      * validity (pass 2 only, where the input is itself filtered): |d_i - 0.1f| <= e_i taints.
      * weight w_i = exp(a_i - q_i): expf is within 2 ulp (2^-22 relative); a_i, q_i = (c - d_i)^2 / (2 sigma_R^2) and a_i - q_i are
        each rounded (2^-22 |a|, 2^-22 q, 2^-24 |a - q|), and the inputs move q by 2 |c - d_i| (e_c + e_i) / (2 sigma_R^2).  The
        kernel is built without flush-to-zero, so float32 keeps subnormal weights; where the weight is below 2^-126 (ARG_TINY < a - q <
        ln 2^-126) expf's 2 ulp are an absolute 2^-148 (A_SUB) on top of the relative bound.  Below ARG_TINY the statement's weight is
        0, and so is expf's.  So |w_f - w| <= eps_i w + A_SUB [subnormal].
      * sw > 0: the device's sw_f >= sw_lo = sw - max eps_i sw - n_sub A_SUB - sum_k h(sw_k).  A pixel with sw > 0 but sw_lo <= 0 may
        be zeroed on the device: it is tainted.  One kept weight in float32's normal range (>= 2^-126) rules this out, so only
        windows whose every kept weight is subnormal can be tainted here.
      * output s / sw, a weighted mean of the kept taps: the inputs' errors add at most max e_i, the weights' errors at most
        (sum w_i eps_i + n_sub A_SUB) / sw_lo * (max - min of the kept taps), and the sums' rounding (sum_k h(s_k) + sum_i h(w_i d_i) +
        out * sum_k h(sw_k)) / sw_lo, plus h(out) for the quotient.  h is at least 2^-150, the rounding of a subnormal result.
    br = 0 is exact: the only tap is the centre, with weight expf(-0) = 1 and s / sw = d / 1."""
    H, W = d.shape
    if br == 0:
        ok = d >= TH_VALID
        marg = (e > 0) & (np.abs(d - TH_VALID) <= e)
        return np.where(ok, d, 0.0), np.where(ok, e, 0.0), t | marg, np.zeros((H, W), bool)
    offs = [(m, n) for m in range(-br, br + 1) for n in range(-br, br + 1)]     # x offset outer, y offset inner
    taps = []
    for m, n in offs:
        nb, inside = _shift(d, n, m)
        taps.append((m, n, nb, _shift(e, n, m)[0], _shift(t, n, m, False)[0], inside & (nb >= TH_VALID), inside))
    S = np.zeros((H, W)); nv = np.zeros((H, W), np.int64); acc = np.zeros((H, W)); exact = np.ones((H, W), bool)
    emax = np.zeros((H, W)); tin = t.copy(); marg = np.zeros((H, W), bool)
    for m, n, nb, en, tn, ok, inside in taps:
        tin |= tn
        marg |= inside & (en > 0) & (np.abs(nb - TH_VALID) <= en)
        S_new = S + np.where(ok, nb, 0.0)
        step = ok & (nv > 0)
        acc += np.where(step, hulp(S_new), 0.0)
        exact &= ~step | is_f32(S_new)
        S, nv = S_new, nv + ok
        emax = np.maximum(emax, np.where(ok, en, 0.0))
    with np.errstate(divide="ignore", invalid="ignore"):
        mean = np.where(nv > 0, S / np.maximum(nv, 1), 0.0)
    e_mean = np.where(exact & is_f32(mean) & (emax == 0), 0.0, acc / np.maximum(nv, 1) + hulp(mean) + emax)
    two_sd, two_sr = 2.0 * float(F(sig_d)) ** 2, 2.0 * float(F(sig_r)) ** 2
    s = np.zeros((H, W)); sw = np.zeros((H, W)); cnt = np.zeros((H, W), np.int64)
    acc_s = np.zeros((H, W)); acc_sw = np.zeros((H, W)); wepsum = np.zeros((H, W)); ein = np.zeros((H, W))
    kmax = np.full((H, W), -np.inf); kmin = np.full((H, W), np.inf); nsub = np.zeros((H, W)); epsmax = np.zeros((H, W))
    for m, n, nb, en, tn, ok, inside in taps:
        x = nb - mean
        err_x = en + e_mean + np.where((en + e_mean == 0) & is_f32(x), 0.0, hulp(x))
        marg |= ok & (np.abs(np.abs(x) - TH_MEAN) <= err_x)
        keep = ok & (np.abs(x) < TH_MEAN)
        a = -(m * m + n * n) / two_sd
        q = (d - nb) ** 2 / two_sr
        arg = a - q
        with np.errstate(under="ignore"):
            w = np.where(keep & (arg > ARG_TINY), np.exp(arg), 0.0)
        nsub += keep & (arg > ARG_TINY) & (arg < ARG_NORMAL)
        eps = 2.0 ** -22 * (1 + abs(a) + q) + U * np.abs(a - q) + 2 * np.abs(d - nb) * (e + en) / two_sr
        epsmax = np.maximum(epsmax, np.where(keep, eps, 0.0))
        s_new, sw_new = s + w * nb, sw + w
        step = keep & (cnt > 0)
        acc_s += np.where(step, hulp(s_new), 0.0) + np.where(keep, hulp(w * nb), 0.0)
        acc_sw += np.where(step, hulp(sw_new), 0.0)
        s, sw, cnt = s_new, sw_new, cnt + keep
        wepsum += w * eps
        ein = np.maximum(ein, np.where(keep, en, 0.0))
        kmax = np.where(keep, np.maximum(kmax, nb), kmax)
        kmin = np.where(keep, np.minimum(kmin, nb), kmin)
    good = (nv > 0) & (sw > 0)
    sw_lo = sw - epsmax * sw - nsub * A_SUB - acc_sw
    zero_marg = good & (sw_lo <= 0)
    good_lo = good & ~zero_marg
    with np.errstate(divide="ignore", invalid="ignore"):
        out = np.where(good, s / np.where(good, sw, 1.0), 0.0)
        err = ((acc_s + out * acc_sw + (wepsum + nsub * A_SUB) * (kmax - kmin)) / np.where(good_lo, sw_lo, 1.0) * (1 + 2.0 ** -10)
               + ein + hulp(out))
    return out, np.where(good, err, 0.0), tin | marg | zero_marg, good & (nsub > 0)


def preprocess64(depth_raw, K, dp=None):
    """The front end stated in float64, with a taint mask and error bounds for the float32 device kernel (frontend.cu).  Returns a Frame64.

    * Erode: every gate is one correctly rounded float32 operation on float32 inputs (d <= 0.1f, d == -inf, d < 0.1f,
      fl(|d - old|) > erode_diff, fl(count / sum) >= erode_ratio), evaluated here exactly as float32 does: exact, never tainted.
      Its output is the raw value or 0, so it is exact too.
    * Filter, twice: _filter64 (the mean gate, pass 2's validity, the weights and the output bound).  Taint spreads: a tainted
      input of a pass taints that pass's output across its (2 br + 1)^2 window.
    * Points: K^-1 is the float inverse the device forms (inverse_intrinsics); X = k00 x d + k02 d, Y = k11 y d + k12 d, Z = d.
      The device rounds x d, the product and the sum (contracted or not), so |X_f - X| <= (|k00 x| + |k02|) (e_d + 3 u d).
      Validity d >= 0.1f is marginal when |d - 0.1f| <= e_d (never when e_d = 0).
    * Normals: the gates |dz| <= 0.02f on filtered depth (a float32 subtraction, exact when both depths are exact and so is dz,
      otherwise within e_P + e_C + h(dz)) and the neighbours' validity are marginal within those bounds.  The stencil vectors a, b
      carry |da| <= |e_a| + h (per component, e_a the sum of the two points' bounds); the cross product n = a x b then moves by at
      most |da||b| + |a||db| + |da||db| + 2 u |(|a_y b_z| + |a_z b_y|, ...)| (two products and a subtraction per component), the unit normal by twice that
      over l = |n| plus 8 u for the norm and quotient: e_n = 2 dn / l + 8 u, which grows as the stencil's conditioning
      |a||b| / l.  (The device's differences are exact when the points are and the float64 difference is a float32 number, and a
      product of zeros is exact, so dn = 0 when every term is.)  l > 0 is marginal when dn > 0 and l <= 2 dn, the orientation when |n . C| <= e_n |C| + |e_C| + 4 u |C|.  A tainted depth
      taints the normals of its four stencil neighbours and its own.
    The taint mask is the union of every stage's."""
    dp = dict(DEFAULTS, **(dp or {}))
    er, br = int(dp["erode_radius"]), int(dp["bf_radius"])
    raw = np.asarray(depth_raw, F)
    H, W = raw.shape
    # erode: float32 gates, exact
    count = np.zeros((H, W), np.int64)
    for i in range(-er, er + 1):
        for j in range(-er, er + 1):
            nb, inside = _shift(raw, i, j)
            with np.errstate(invalid="ignore"):
                bad = (nb == F(-np.inf)) | (nb < F(0.1)) | (np.abs(nb - raw) > F(dp["erode_diff"]))
            count += inside & bad
    eroded = (count.astype(F) / F((2 * er + 1) ** 2)) >= F(dp["erode_ratio"])
    d = np.where((raw <= F(0.1)) | eroded, 0.0, raw.astype(np.float64))
    e = np.zeros((H, W))
    d1, e1, t1, s1 = _filter64(d, e, np.zeros((H, W), bool), br, dp["sigma_D"], dp["sigma_R"])
    d2, e2, t2, s2 = _filter64(d1, e1, t1, br, dp["sigma_D"], dp["sigma_R"])
    for i in range(-br, br + 1):
        for j in range(-br, br + 1):
            s2 |= (d2 > 0) & _shift(s1, i, j, False)[0]
    # points
    k00, k11, k02, k12 = (float(v) for v in inverse_intrinsics(K))
    xs = np.arange(W, dtype=np.float64)[None, :] * np.ones((H, 1))
    ys = np.arange(H, dtype=np.float64)[:, None] * np.ones((1, W))
    valid = d2 >= TH_VALID
    vmarg = (e2 > 0) & (np.abs(d2 - TH_VALID) <= e2)
    xyz = np.zeros((H, W, 4))
    xyz[..., 0] = np.where(valid, k00 * xs * d2 + k02 * d2, 0.0)
    xyz[..., 1] = np.where(valid, k11 * ys * d2 + k12 * d2, 0.0)
    xyz[..., 2] = np.where(valid, d2, 0.0)
    xyz[..., 3] = valid
    exyz = np.zeros((H, W, 3))
    exyz[..., 0] = np.where(valid, (np.abs(k00 * xs) + abs(k02)) * (e2 + 3 * U * d2) * (1 + 2.0 ** -10), 0.0)
    exyz[..., 1] = np.where(valid, (np.abs(k11 * ys) + abs(k12)) * (e2 + 3 * U * d2) * (1 + 2.0 ** -10), 0.0)
    exyz[..., 2] = np.where(valid, e2, 0.0)
    # normals
    P, z = xyz[..., :3], xyz[..., 2]

    def sh(a, dy, dx, fill=0.0):
        return _shift(a, dy, dx, fill)[0] if a.ndim == 2 else np.stack([_shift(a[..., c], dy, dx, fill)[0] for c in range(a.shape[-1])], -1)
    nbs = [(sh(P, dy, dx), sh(exyz, dy, dx), sh(e2, dy, dx), sh(vmarg, dy, dx, False)) for dy, dx in ((1, 0), (-1, 0), (0, 1), (0, -1))]
    near, nmarg = [], np.zeros((H, W), bool)
    for Q, eQ, ez, vm in nbs:
        dz = Q[..., 2] - z
        ok = Q[..., 2] >= TH_VALID
        err = ez + e2 + np.where((ez + e2 == 0) & is_f32(dz), 0.0, hulp(dz))
        near.append(ok & (np.abs(dz) <= TH_NORMAL))
        nmarg |= vm | (ok & (np.abs(np.abs(dz) - TH_NORMAL) <= err))
    (PC, ePC), (MC, eMC), (CP, eCP), (CM, eCM) = ((q[0], q[1]) for q in nbs)
    pc, mc, cp, cm = near
    both_a, both_b = (pc & mc)[..., None], (cp & cm)[..., None]
    A = np.where(both_a, PC - MC, np.where(pc[..., None], PC - P, MC - P))
    eA = np.where(both_a, ePC + eMC, np.where(pc[..., None], ePC + exyz, eMC + exyz))
    eA += np.where((eA == 0) & is_f32(A), 0.0, hulp(A))
    B = np.where(both_b, CP - CM, np.where(cp[..., None], CP - P, CM - P))
    eB = np.where(both_b, eCP + eCM, np.where(cp[..., None], eCP + exyz, eCM + exyz))
    eB += np.where((eB == 0) & is_f32(B), 0.0, hulp(B))
    N = np.cross(A, B)
    l = np.linalg.norm(N, axis=-1)
    la, lb, lea, leb = (np.linalg.norm(v, axis=-1) for v in (A, B, eA, eB))
    rnd = np.stack([np.abs(A[..., 1] * B[..., 2]) + np.abs(A[..., 2] * B[..., 1]), np.abs(A[..., 2] * B[..., 0]) + np.abs(A[..., 0] * B[..., 2]),
                    np.abs(A[..., 0] * B[..., 1]) + np.abs(A[..., 1] * B[..., 0])], -1)
    dn = (lea * lb + la * leb + lea * leb + 2 * U * np.linalg.norm(rnd, axis=-1)) * (1 + 2.0 ** -10)
    with np.errstate(divide="ignore", invalid="ignore"):
        en = np.where(l > 0, 2 * dn / l + 8 * U, np.inf)
        nrm = N / l[..., None]
    dot = np.sum(nrm * -P, -1)
    lc, lec = np.linalg.norm(P, axis=-1), np.linalg.norm(exyz, axis=-1)
    nrm = np.where((dot < 0)[..., None], -nrm, nrm)
    interior = np.zeros((H, W), bool)
    interior[1:H - 1, 1:W - 1] = True
    gated = interior & valid & (pc | mc) & (cp | cm)
    ok = gated & (l > 0)
    normal = np.zeros((H, W, 4))
    normal[..., :3] = np.where(ok[..., None], nrm, 0.0)
    tn = interior & ((valid & nmarg) | vmarg)
    tn |= gated & (((dn > 0) & (l <= 2 * dn)) | (ok & (np.abs(dot) <= np.where(ok, en, 0.0) * lc + lec + 4 * U * lc)))
    t2n = t2.copy()
    for dy, dx in ((1, 0), (-1, 0), (0, 1), (0, -1)):
        t2n |= interior & _shift(t2, dy, dx, False)[0]
    taint = t2n | tn | vmarg
    sub = s2.copy()
    for dy, dx in ((1, 0), (-1, 0), (0, 1), (0, -1)):
        sub |= interior & _shift(s2, dy, dx, False)[0]
    return Frame64(depth=d2, xyz=xyz, normal=normal, taint=taint, filter1=t1, filter2=t2, normal_taint=tn, subnormal=sub,
                   depth_err=e2, xyz_err=exyz, normal_err=np.where(ok, en, 0.0))


DEPTH_CAP, XYZ_CAP, NORMAL_CAP = 2e-6, 3e-6, 1e-3   # never looser than these: depth 2e-6 at 1 m (relative), xyz 3e-6 m, normals 1e-3


def device_report(d, xyz, n, r, f32=None):
    """Holds one frame of float32 device maps (depth [H,W], xyz [H,W,4] or None, normal [H,W,4]) to a Frame64 `r`, pixel by pixel with
    no fraction allowance.  Outside r.taint: depth within min(depth_err, 2e-6 d), xyz within min(xyz_err, 3e-6), normals within
    min(normal_err, 1e-3) per component, and +0.0 bit for bit wherever the float64 result is zero (depth, point, normal vector).
    On r.subnormal pixels float32 itself can be further than those caps from float64, so the derived bounds alone apply there, and
    when f32 = (depth, xyz, normal) of the float32 restatement is given those pixels must also lie within 2e-6 / 3e-6 / 1e-3 of it.
    Everywhere: xyz.w == (d >= 0.1f) of the device's own depth and normal.w is +0.0.  Returns a dict: failures (list of strings),
    tainted and subnormal (counts), flipped (untainted pixels whose kept-or-zeroed depth differs), and the worst error as a fraction
    of each bound."""
    fails = []
    ok = ~r.taint
    sub = r.subnormal
    bits = lambda a: np.asarray(a, np.float32).view(np.uint32)
    bd = np.where(sub, r.depth_err, np.minimum(r.depth_err, DEPTH_CAP * r.depth))
    ed = np.abs(d.astype(np.float64) - r.depth)
    zero = r.depth == 0
    flipped = ok & ((d > 0) != (r.depth > 0))
    if flipped.any():
        fails.append(f"depth kept-or-zeroed differs at {np.argwhere(flipped)[:5].tolist()}")
    bad = ok & ~zero & (ed > bd)
    if bad.any():
        fails.append(f"depth beyond bound at {np.argwhere(bad)[:5].tolist()} (worst {(ed / np.where(bd > 0, bd, 1))[bad].max():.3g} x bound)")
    if (ok & zero & (bits(d) != 0)).any():
        fails.append(f"depth not +0.0 at {np.argwhere(ok & zero & (bits(d) != 0))[:5].tolist()}")
    rep = {"tainted": int(r.taint.sum()), "subnormal": int((sub & ok & ~zero).sum()), "flipped": int(flipped.sum()), "valid": int((r.depth > 0).sum()),
           "depth_frac": float((ed / np.where(bd > 0, bd, 1))[ok & ~zero].max(initial=0.0))}
    if xyz is not None:
        if not np.array_equal(xyz[..., 3], (d >= np.float32(0.1)).astype(np.float32)):
            fails.append("xyz.w differs from d >= 0.1f")
        bx = np.where(sub[..., None], r.xyz_err, np.minimum(r.xyz_err, XYZ_CAP))
        ex = np.abs(xyz[..., :3].astype(np.float64) - r.xyz[..., :3])
        valid = r.xyz[..., 3] > 0
        badx = ok[..., None] & valid[..., None] & (ex > bx)
        if badx.any():
            fails.append(f"xyz beyond bound at {np.argwhere(badx.any(-1))[:5].tolist()}")
        zx = ok & ~valid & (bits(xyz) != 0).any(-1)
        if zx.any():
            fails.append(f"xyz not +0.0 at {np.argwhere(zx)[:5].tolist()}")
        rep["xyz_frac"] = float((ex / np.where(bx > 0, bx, 1))[ok & valid].max(initial=0.0))
    has = r.normal_err > 0
    bn = np.where(sub, r.normal_err, np.minimum(r.normal_err, NORMAL_CAP))
    en = np.abs(n[..., :3].astype(np.float64) - r.normal[..., :3]).max(-1)
    badn = ok & has & (en > bn)
    if badn.any():
        fails.append(f"normal beyond bound at {np.argwhere(badn)[:5].tolist()} (worst {(en / np.where(bn > 0, bn, 1))[badn].max():.3g} x bound)")
    zn = ok & ~has & (bits(n[..., :3]) != 0).any(-1)
    if zn.any():
        fails.append(f"normal not +0.0 at {np.argwhere(zn)[:5].tolist()}")
    if (bits(n[..., 3]) != 0).any():
        fails.append("normal.w is not +0.0")
    if f32 is not None and (sub & ok).any():
        d32, x32, n32 = f32
        m = sub & ok
        far = m & ((np.abs(d - d32) > DEPTH_CAP) | (np.abs(n[..., :3] - n32[..., :3]).max(-1) > NORMAL_CAP))
        if xyz is not None:
            far |= m & (np.abs(xyz[..., :3] - x32[..., :3]).max(-1) > XYZ_CAP)
        if far.any():
            fails.append(f"subnormal-weight pixels beyond 2e-6 / 3e-6 / 1e-3 of the float32 restatement at {np.argwhere(far)[:5].tolist()}")
    rep["normal_frac"] = float((en / np.where(bn > 0, bn, 1))[ok & has].max(initial=0.0))
    rep["failures"] = fails
    return rep
