"""Raw depth frames and front-end parameters built to sit on the edges of the fused frame front end (frontend.cu): tile seams and image
borders, every radius pair the halo admits, and the gate equalities of erode, the filter and the normals.  Shared by the oracle's CPU
test and the GPU test of the kernel.

A family is a dict:
  name, frames [list of float32 H x W raw depth], K (fx, fy, cx, cy), dp (front-end parameters),
  claims: [(kind, frame index, y, x, value)], cells whose gate value the CPU test recomputes in exact arithmetic
          ("erode_diff": |d - old| of the neighbour at (y, x) against the centre in value, "ratio": count at centre (y, x),
           "centre": the raw centre, "mean_dist": |d - mean| of the tap at (y, x) in its centre's window, which is value,
           "normal_dz": the raw |dz| of the normal stencil neighbour at (y, x)),
  taint: the number of pixels preprocess64 taints in each frame: 0, except in filter_marginal, built so that the kernel's float32 mean
         gate decides some taps the other way from float64 (its count is preprocess64's; its claims name the windows).
filter_subnormal holds hole-filled centres whose every filter weight is a float32 subnormal.

The seam and radius frames are piecewise constant, with steps of 29.3, 37.1 and 363.7 mm and flying pixels 49.3 mm off, so that no
window's |d - mean| (a step times a fraction k / nv) lands within rounding of 0.01 by accident; the gate families use planes with
dyadic slopes.  Gate cells that must be exact use br = 0, where the filter is the identity on valid depth and the
output shows erode's decision, or er = 0, where erode only removes depth <= 0.1f."""
import numpy as np

F32 = np.float32
K = (512.0, 512.0, 40.0, 30.0)
SHIPPED = dict(erode_radius=1, erode_diff=0.001, erode_ratio=0.8, bf_radius=2, sigma_D=2.0, sigma_R=100000.0)
WIDTHS = (1, 2, 3, 63, 64, 65, 127, 129, 640)
HEIGHTS = (1, 2, 3, 31, 32, 33, 65, 480)
MAX_HALO = 12
RADII = [(er, br) for br in range(6) for er in range(12) if er + 2 * br + 1 <= MAX_HALO]
LARGEST = [(er, br) for er, br in RADII if er + 2 * br + 1 == MAX_HALO]
MINF = F32(-np.inf)


def up(x, k=1):
    x = F32(x)
    for _ in range(k):
        x = np.nextafter(x, F32(np.inf))
    return x


def down(x, k=1):
    x = F32(x)
    for _ in range(k):
        x = np.nextafter(x, F32(-np.inf))
    return x


def plane(H, W, base=0.6):
    """base + x / 4096 + y / 8192: neighbours differ by far less than every gate."""
    y, x = np.mgrid[0:H, 0:W]
    return (base + x / 4096.0 + y / 8192.0).astype(F32)


def edge_lines(n, period):
    """Image rows (or columns) 0, 1, n-2, n-1 and every tile seam pair (k period - 1, k period)."""
    s = {0, 1, n - 2, n - 1}
    for k in range(period, n + 1, period):
        s |= {k - 1, k}
    return sorted(v for v in s if 0 <= v < n)


def seam_frame(H, W):
    """A plane at 0.6 m with a 37.1 mm step at the first column seam and a 29.3 mm step at the first row seam, and on every crossing of an edge row and
    an edge column one of: a hole, a flying pixel 49.3 mm in front, a -inf sample."""
    y, x = np.mgrid[0:H, 0:W]
    d = (F32(0.6) + F32(0.0371) * (x >= 64) + F32(0.0293) * (y >= 32)).astype(F32)
    rows, cols = edge_lines(H, 32), edge_lines(W, 64)
    for i, r in enumerate(rows):
        for j, c in enumerate(cols):
            k = (i + j) % 4
            if k == 0:
                d[r, c] = 0.0
            elif k == 1:
                d[r, c] = d[r, c] - F32(0.0493)
            elif k == 2:
                d[r, c] = MINF
    return d


def seams():
    sizes = [(33, w) for w in WIDTHS] + [(h, 65) for h in HEIGHTS if h != 33] + [(480, 640)]
    out = []
    for er, br in ((1, 2), LARGEST[0], LARGEST[-1]):
        dp = dict(SHIPPED, erode_radius=er, bf_radius=br)
        for H, W in sizes:
            out.append({"name": f"seams_{H}x{W}_er{er}_br{br}", "frames": [seam_frame(H, W)], "K": K, "dp": dp, "claims": [], "taint": [0]})
    return out


def object_frame(H, W, seed=0):
    """A disc at 0.5 m crossing the tile seams, on a background at 0.8637 m, with holes and flying pixels."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W]
    disc = (x - W * 0.55) ** 2 + (y - H * 0.45) ** 2 <= (0.35 * min(H, W)) ** 2
    d = np.where(disc, F32(0.5), F32(0.8637)).astype(F32)
    cells = rng.integers(0, H * W, 40)
    d.flat[cells[:20]] = 0.0
    d.flat[cells[20:]] = d.flat[cells[20:]] + F32(0.0493)
    return d


def radii():
    out = []
    for er, br in RADII:
        out.append({"name": f"radii_97x131_er{er}_br{br}", "frames": [object_frame(97, 131)], "K": K,
                    "dp": dict(SHIPPED, erode_radius=er, bf_radius=br), "claims": [], "taint": [0]})
    for er, br in LARGEST:
        out.append({"name": f"radii_480x640_er{er}_br{br}", "frames": [object_frame(480, 640, 1)], "K": K,
                    "dp": dict(SHIPPED, erode_radius=er, bf_radius=br), "claims": [], "taint": [0]})
    return out


# ------------------------------------------------------------------------------------------------------------------ erode gates
EH, EW = 33, 65                     # two tiles each way


def _cells(H, W, step=6):
    """Centres far enough apart that their 3 x 3 neighbourhoods do not touch, away from the border."""
    return [(y, x) for y in range(3, H - 3, step) for x in range(3, W - 3, step)]


def erode_diff_family():
    """erode_diff = 2^-10; around centre 0.5 one neighbour at |d - old| = erode_diff and one float32 step either side, above and below
    the centre.  One bad neighbour erodes (ratio 1/9)."""
    diff = 2.0 ** -10
    dp = dict(SHIPPED, erode_radius=1, bf_radius=0, erode_diff=diff, erode_ratio=float(F32(1) / F32(9)))
    d = np.full((EH, EW), F32(0.5))
    claims = []
    vals = [F32(0.5 + diff), up(0.5 + diff), down(0.5 + diff), F32(0.5 - diff), up(0.5 - diff), down(0.5 - diff)]
    for (y, x), v in zip(_cells(EH, EW), vals * 4):
        d[y, x + 1] = v
        claims.append(("erode_diff", 0, y, x + 1, (y, x)))
    return {"name": "erode_diff", "frames": [d], "K": K, "dp": dp, "claims": claims, "taint": [0]}


def erode_validity_family():
    """erode_diff = 1 so that only validity decides: centres at 0.1f, the float below and the float above; neighbours at 0.1f, the float
    below it and -inf, at interior cells and on the image border."""
    dp = dict(SHIPPED, erode_radius=1, bf_radius=0, erode_diff=1.0, erode_ratio=float(F32(1) / F32(9)))
    d = np.full((EH, EW), F32(0.2))
    claims = []
    cells = _cells(EH, EW)
    for (y, x), v in zip(cells[:6], [F32(0.1), down(0.1), up(0.1)] * 2):
        d[y, x] = v
        claims.append(("centre", 0, y, x, v))
    for (y, x), v in zip(cells[6:15], [F32(0.1), down(0.1), MINF] * 3):
        d[y + 1, x - 1] = v
        claims.append(("centre", 0, y + 1, x - 1, v))
    for (y, x), v in zip([(0, 10), (EH - 1, 20), (12, 0), (20, EW - 1), (0, 0), (EH - 1, EW - 1)], [F32(0.1), down(0.1), MINF] * 2):
        d[y, x] = v
        claims.append(("centre", 0, y, x, v))
    return {"name": "erode_validity", "frames": [d], "K": K, "dp": dp, "claims": claims, "taint": [0]}


def erode_ratio_families():
    """erode_ratio = fl(3/9) and one float32 step either side, with centres that have 2, 3 and 4 bad neighbours (a neighbour 10 mm off),
    inside the image and on every border and corner, where out-of-image neighbours are not counted but the divisor stays 9; and
    erode_ratio = 0, where every pixel is eroded."""
    r = F32(3) / F32(9)
    out = []
    for name, ratio in (("erode_ratio_eq", r), ("erode_ratio_up", up(r)), ("erode_ratio_down", down(r)), ("erode_ratio_zero", F32(0))):
        dp = dict(SHIPPED, erode_radius=1, bf_radius=0, erode_diff=0.001, erode_ratio=float(ratio))
        d = np.full((EH, EW), F32(0.5))
        claims = []
        centres = _cells(EH, EW)[:9] + [(0, 10), (0, 20), (EH - 1, 30), (EH - 1, 40), (12, 0), (20, 0), (10, EW - 1), (24, EW - 1),
                                         (0, 0), (0, EW - 1), (EH - 1, 0), (EH - 1, EW - 1)]
        for k, (y, x) in enumerate(centres):
            nbad = 2 + k % 3
            nbs = [(y + i, x + j) for i in (-1, 0, 1) for j in (-1, 0, 1) if (i, j) != (0, 0) and 0 <= y + i < EH and 0 <= x + j < EW]
            for yy, xx in nbs[:nbad]:
                d[yy, xx] = F32(0.51)
            claims.append(("ratio", 0, y, x, min(nbad, len(nbs))))
        out.append({"name": name, "frames": [d], "K": K, "dp": dp, "claims": claims, "taint": [0]})
    return out


# ----------------------------------------------------------------------------------------------------------------- filter gates
def filter_gates_family():
    """er = 0, br = 1.  Windows of nine taps on 0.75 + j 2^-21, so that the float32 running sum and the mean are exact, in which the
    tap left of the centre is the nearest float32 distance below 0.01 on that grid, or the nearest above, from the window's mean.  0.01f
    itself is not reachable: depths >= 0.1 differ by multiples of 2^-27 or more, and 0.01f is an odd multiple of 2^-29.  Also windows
    with no valid tap, invalid centres that are hole-filled, and, in a second family, sigma_R small enough that every weight of a
    hole-filled centre underflows, so sw == 0 and the output is 0."""
    dp = dict(SHIPPED, erode_radius=0, bf_radius=1, erode_ratio=0.8)
    rng = np.random.default_rng(11)
    d = np.zeros((EH, EW), F32)
    claims = []
    g = 2.0 ** -21
    for n, (y, x) in enumerate(_cells(EH, EW, 8)[:12]):
        k = 20971 + n % 2                                          # k g: the grid's nearest distances below and above 0.01
        j = rng.integers(-64, 64, 8)
        j[0] += (-k - int(j.sum())) % 8                            # 9 k + sum j = 0 (mod 8): the tap below lands on the grid
        rest = 8 * 0.75 + int(j.sum()) * g
        v = (rest + 9 * k * g) / 8                                 # v - (rest + v) / 9 = k g
        taps = list(0.75 + j * g)
        taps.insert(1, v)                                          # x offset outer, y offset inner: tap 1 is (dx, dy) = (-1, 0)
        win = np.asarray(taps, F32).reshape(3, 3).T                # win[dy + 1, dx + 1]
        d[y - 1:y + 2, x - 1:x + 2] = win
        claims.append(("mean_dist", 0, y, x - 1, k * g))
    # the rest of the frame is 0: windows with no valid tap
    hole = plane(EH, EW)
    hole[10, 50] = 0.0
    hole[20, 55] = 0.0
    d2 = plane(EH, EW)
    d2[::5, ::7] = 0.0                                              # hole-filled centres; with sigma_R = 1e-3 their weights underflow
    f = {"name": "filter_gates", "frames": [d, hole], "K": K, "dp": dp, "claims": claims, "taint": [0, 0]}
    g = {"name": "filter_underflow", "frames": [d2], "K": K, "dp": dict(dp, sigma_R=1e-3), "claims": [], "taint": [0]}
    return [f, g]


# ----------------------------------------------------------------------------------------------------------------- normal gates
def normal_gates_family():
    """(er, br) = (0, 0): the filtered depth is the raw depth bit for bit.  0.02f is not a reachable |dz| (an odd multiple of 2^-28,
    while depths >= 0.1 differ by multiples of 2^-27 or more), so neighbours of centres at 0.5 sit at the nearest differences either side
    of it on that depth's 2^-24 grid; centres at 0.1f, the float below and the float above.  A second frame uses intrinsics whose float determinant overflows:
    K^-1 is then 0, every point lies on the optical axis, neighbours are collinear and l = 0."""
    dp = dict(SHIPPED, erode_radius=0, bf_radius=0, erode_ratio=0.8)
    d = np.full((EH, EW), F32(0.5))
    claims = []
    lo, hi = 335544 * 2.0 ** -24, 335545 * 2.0 ** -24              # around 0.02f at depths in [0.5, 1), a 2^-24 grid
    cells = _cells(EH, EW, 6)
    for k, (y, x) in enumerate(cells[:16]):
        dz = lo if k % 2 == 0 else hi
        dy, dx = ((1, 0), (-1, 0), (0, 1), (0, -1))[(k // 2) % 4]
        d[y + dy, x + dx] = F32(0.5 + dz)
        claims.append(("normal_dz", 0, y + dy, x + dx, dz))
    for (y, x), v in zip(cells[16:22], [F32(0.1), down(0.1), up(0.1)] * 2):
        d[y, x] = v
        claims.append(("centre", 0, y, x, v))
    axis = {"name": "normal_collinear", "frames": [plane(EH, EW)], "K": (1e20, 1e20, 40.0, 30.0), "dp": dp, "claims": [], "taint": [0]}
    return [{"name": "normal_gates", "frames": [d], "K": K, "dp": dp, "claims": claims, "taint": [0]}, axis]


def _f32_mean_gate(taps, t):
    """The kernel's float32 mean gate on tap t of a window (taps in the kernel's order): fl(d_t - fl(sum / nv)) <= 0.01f."""
    s = F32(0)
    for v in taps:
        s = F32(s + v)
    m = F32(s / F32(len(taps)))
    return bool(abs(F32(taps[t] - m)) <= F32(0.01))


def filter_marginal_family():
    """Built to be marginal: er = 0, br = 1, windows of nine taps near 0.75 m on a 2^-24 grid (so the float32 running sum rounds) in
    which the tap left of the centre lies within rounding of |d - mean| = 0.01, and the kernel's float32 gate decides it the other way
    from the float64 one.  preprocess64 must taint these windows' centres; the claimed taint count is the pixels that taint reaches."""
    dp = dict(SHIPPED, erode_radius=0, bf_radius=1, erode_ratio=0.8)
    rng = np.random.default_rng(5)
    d = np.zeros((EH, EW), F32)
    claims = []
    for y, x in _cells(EH, EW, 8)[:6]:
        while True:
            taps = [F32(0.75 + int(j) * 2.0 ** -24 * 37) for j in rng.integers(-3000, 3000, 9)]
            rest = sum(float(v) for i, v in enumerate(taps) if i != 1)
            v0 = F32((rest + 9 * 0.01) / 8)                         # |v - mean| = 0.01 in exact arithmetic
            hit = None
            for k in range(-6, 7):
                taps[1] = F32(float(v0) + k * 2.0 ** -24)
                mean64 = (rest + float(taps[1])) / 9
                if (float(taps[1]) - mean64 < 0.01) != _f32_mean_gate(taps, 1):
                    hit = taps[1]
                    break
            if hit is not None:
                break
        win = np.asarray(taps, F32).reshape(3, 3).T                # win[dy + 1, dx + 1], taps in x-outer, y-inner order
        d[y - 1:y + 2, x - 1:x + 2] = win
        claims.append(("mean_flip", 0, y, x - 1, (y, x)))
    return {"name": "filter_marginal", "frames": [d], "K": K, "dp": dp, "claims": claims, "taint": [None]}


def subnormal_family():
    """Hole-filled centres whose every kept weight is subnormal in float32 (er = 0, br = 1, sigma_R chosen so that (c - d)^2 / (2
    sigma_R^2) is about 88 for a hole in a 0.75 m plane, so every weight lies just below 2^-126): the kernel, built without
    flush-to-zero, keeps those weights, and the output is a weighted mean of subnormals.  preprocess64 bounds it with the absolute
    rounding of subnormal results; nothing here is tainted.  (Deeper in the subnormal range, near 2^-149, a product w d keeps only a
    few bits: the bound grows to millimetres and the windows the second pass and the normals read from those pixels are tainted.)"""
    dp = dict(SHIPPED, erode_radius=0, bf_radius=1, erode_ratio=0.8, sigma_R=float(np.sqrt(0.75 ** 2 / 176)))
    d = plane(EH, EW, 0.75)
    d[2::5, 3::7] = 0.0
    return {"name": "filter_subnormal", "frames": [d], "K": K, "dp": dp, "claims": [], "taint": [0]}


def _with_counted_taint(fam):
    """Fills in the taint count of a family built to be marginal from preprocess64 (its claims say which cells must be among them)."""
    from oracle import frame_oracle as fo
    fam["taint"] = [int(fo.preprocess64(fr, fam["K"], fam["dp"]).taint.sum()) for fr in fam["frames"]]
    return fam


def families():
    return (seams() + radii() + [erode_diff_family(), erode_validity_family()] + erode_ratio_families() + filter_gates_family()
            + [_with_counted_taint(filter_marginal_family()), subnormal_family()] + normal_gates_family())
