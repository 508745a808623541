"""CPU tests of the front end's float64 statement (oracle.frame_oracle.preprocess64) and of the frames built on the kernel's edges
(oracle/frame_families.py): the families land where they claim, the float64 statement agrees with the float32 restatement within its
per-pixel bounds outside its taint mask, and the kernel's float rewrites of the reference's comparisons and its weight-table shortcut
are exact."""
from collections import Counter
from fractions import Fraction as Q

import numpy as np
import pytest

from bundletrack_b200 import synth
from oracle import frame_families as ff
from oracle import frame_oracle as fo

FAMILIES = {f["name"]: f for f in ff.families()}
F32 = np.float32


def test_families_cover_the_issue_space():
    assert len(ff.RADII) == 42 and set(ff.LARGEST) == {(11, 0), (9, 1), (7, 2), (5, 3), (3, 4), (1, 5)}
    sizes = {f["frames"][0].shape for n, f in FAMILIES.items() if n.startswith("seams")}
    assert {w for _, w in sizes} == set(ff.WIDTHS) and {h for h, _ in sizes} == set(ff.HEIGHTS)
    for n, f in FAMILIES.items():
        dp = f["dp"]
        assert dp["erode_radius"] + 2 * dp["bf_radius"] + 1 <= ff.MAX_HALO, n
        assert len({fr.shape for fr in f["frames"]}) == 1 and len(f["taint"]) == len(f["frames"]), n


def test_seam_features_sit_on_seams_and_borders():
    d = FAMILIES["seams_480x640_er1_br2"]["frames"][0]
    feats = (d == 0) | np.isinf(d) | np.isin(d, [F32(F32(v) - F32(0.0493)) for v in (0.6, 0.6 + 0.0371, 0.6 + 0.0293)])
    rows, cols = np.nonzero(feats)
    assert set(rows) <= set(ff.edge_lines(480, 32)) and set(cols) <= set(ff.edge_lines(640, 64))
    assert {0, 1, 31, 32, 478, 479} <= set(rows) and {0, 1, 63, 64, 638, 639} <= set(cols)


def _exact_erode_count(raw, y, x, diff):
    H, W = raw.shape
    old, c = raw[y, x], 0
    for i in (-1, 0, 1):
        for j in (-1, 0, 1):
            if 0 <= y + i < H and 0 <= x + j < W:
                v = raw[y + i, x + j]
                c += bool(np.isinf(v) or v < F32(0.1) or F32(abs(Q(float(v)) - Q(float(old)))) > F32(diff))
    return c


def test_gate_families_land_where_they_claim():
    # erode_diff: above and below a 0.5 centre, |d - old| exactly erode_diff and one float32 step either side, four cells each
    diff = Q(float(F32(2.0 ** -10)))
    got = Counter()
    for kind, i, y, x, (cy, cx) in FAMILIES["erode_diff"]["claims"]:
        raw = FAMILIES["erode_diff"]["frames"][i]
        assert raw[cy, cx] == F32(0.5) and (cy, cx) == (y, x - 1)
        got[(1 if raw[y, x] > 0.5 else -1, abs(Q(float(raw[y, x])) - Q(1, 2)))] += 1
    up, dn = Q(2) ** -24, Q(2) ** -25               # float32 steps above and below 0.5
    assert got == Counter({(1, diff): 4, (1, diff + up): 4, (1, diff - up): 4, (-1, diff): 4, (-1, diff - dn): 4, (-1, diff + dn): 4})
    # erode_validity: the exact multiset of centres and neighbours, and each claimed cell holds its value
    f = FAMILIES["erode_validity"]
    for _, i, y, x, v in f["claims"]:
        assert f["frames"][i][y, x].tobytes() == F32(v).tobytes()
    got = Counter(F32(v).tobytes() for *_, v in f["claims"])
    assert got == Counter({F32(0.1).tobytes(): 7, ff.down(0.1).tobytes(): 7, ff.up(0.1).tobytes(): 2, F32(-np.inf).tobytes(): 5})
    r = F32(3) / F32(9)
    assert Q(float(FAMILIES["erode_ratio_eq"]["dp"]["erode_ratio"])) == Q(float(r))
    assert FAMILIES["erode_ratio_up"]["dp"]["erode_ratio"] == float(ff.up(r)) and FAMILIES["erode_ratio_down"]["dp"]["erode_ratio"] == float(ff.down(r))
    for name in ("erode_ratio_eq", "erode_ratio_up", "erode_ratio_down"):
        f = FAMILIES[name]
        counts = [_exact_erode_count(f["frames"][0], y, x, f["dp"]["erode_diff"]) for _, _, y, x, _ in f["claims"]]
        assert counts == [c for *_, c in f["claims"]]
        assert {2, 3, 4} <= set(counts)
        border = [(y, x) for _, _, y, x, _ in f["claims"] if y in (0, ff.EH - 1) or x in (0, ff.EW - 1)]
        assert len(border) == 12
    # the filter's windows: the float32 running sum is exact, so is the mean, and the tap sits at the claimed distance from it
    f = FAMILIES["filter_gates"]
    for _, i, y, x, dist in f["claims"]:
        cy, cx = y, x + 1
        win = f["frames"][i][cy - 1:cy + 2, cx - 1:cx + 2]
        taps = [win[dy + 1, dx + 1] for dx in (-1, 0, 1) for dy in (-1, 0, 1)]
        s = F32(0)
        for t in taps:
            assert Q(float(s + t)) == Q(float(s)) + Q(float(t))
            s = s + t
        mean = s / F32(9)
        assert Q(float(mean)) == Q(float(s)) / 9
        got = abs(Q(float(f["frames"][i][y, x])) - Q(float(mean)))
        assert got == Q(dist) and (got < Q(1, 100)) == (dist < 0.01)
        assert abs(got - Q(1, 100)) < Q(2) ** -21
    assert {d < 0.01 for *_, d in f["claims"]} == {True, False}
    # the normals' neighbours: exactly the claimed |dz| from a 0.5 m centre, the nearest on the grid either side of 0.02f
    f = FAMILIES["normal_gates"]
    for kind, i, y, x, dz in f["claims"]:
        if kind == "normal_dz":
            assert Q(float(f["frames"][i][y, x])) - Q(1, 2) == Q(dz)
            assert abs(Q(dz) - Q(float(F32(0.02)))) < Q(2) ** -24
    assert {d < float(F32(0.02)) for k, *_, d in f["claims"] if k == "normal_dz"} == {True, False}


def test_only_the_marginal_family_is_tainted_and_it_flips():
    """Every family but filter_marginal claims no tainted pixel.  filter_marginal's windows put a tap within rounding of the mean gate
    where the kernel's float32 gate really decides the other way (checked exactly); preprocess64 taints each such centre, and its taint
    reaches no further than the two filter windows and the normal stencil from a claimed cell."""
    for n, f in FAMILIES.items():
        if n == "filter_marginal":
            assert f["taint"][0] > 0
        else:
            assert f["taint"] == [0] * len(f["frames"]), n
    f = FAMILIES["filter_marginal"]
    raw = f["frames"][0]
    r = fo.preprocess64(raw, f["K"], f["dp"])
    d32 = fo.preprocess(raw, f["K"], f["dp"])[0]
    for _, _, y, x, (cy, cx) in f["claims"]:
        win = raw[cy - 1:cy + 2, cx - 1:cx + 2]
        taps = [win[dy + 1, dx + 1] for dx in (-1, 0, 1) for dy in (-1, 0, 1)]
        assert taps[1] == raw[y, x]
        exact = Q(float(taps[1])) - sum(Q(float(v)) for v in taps) / 9
        assert abs(exact - Q(1, 100)) < Q(2) ** -20
        assert (exact < Q(1, 100)) != ff._f32_mean_gate(taps, 1)
        assert r.filter1[cy, cx] and r.taint[cy, cx]
        assert abs(float(d32[cy, cx]) - r.depth[cy, cx]) > r.depth_err[cy, cx]       # the flip moves the float32 result off the bound
    reach = np.zeros(raw.shape, bool)
    for *_, (cy, cx) in f["claims"]:
        reach[max(cy - 3, 0):cy + 4, max(cx - 3, 0):cx + 4] = True
    assert not (r.taint & ~reach).any()


@pytest.mark.parametrize("name", [n for n in FAMILIES if "480" not in n])
def test_preprocess64_agrees_with_float32_restatement(name):
    """On every family: the float32 restatement lies within preprocess64's per-pixel bounds outside the taint mask, the taint count is
    the family's, and with (er, br) = (0, 0) the filtered depth is the raw depth bit for bit."""
    f = FAMILIES[name]
    for i, raw in enumerate(f["frames"]):
        r = fo.preprocess64(raw, f["K"], f["dp"])
        d, x, n = fo.preprocess(raw, f["K"], f["dp"])
        rep = fo.device_report(d, x, n, r, (d, x, n))
        assert not rep["failures"], rep["failures"]
        assert rep["tainted"] == f["taint"][i]
        if f["dp"]["erode_radius"] == 0 and f["dp"]["bf_radius"] == 0:
            keep = raw > F32(0.1)
            assert np.array_equal(d, np.where(keep, raw, 0).astype(F32)) and np.array_equal(r.depth, np.where(keep, raw, 0))
            assert not r.depth_err.any()


@pytest.mark.parametrize("name", [n for n in FAMILIES if "480" in n][:3])
def test_preprocess64_agrees_at_full_size(name):
    test_preprocess64_agrees_with_float32_restatement(name)


@pytest.mark.parametrize("seed,H,W", [(0, 120, 160), (1, 97, 131), (2, 480, 640)])
def test_preprocess64_bounds_on_synthetic_frames(seed, H, W):
    """The bounds hold the float32 restatement with room, and stay within today's tolerances at the shipped parameters."""
    raw, K = synth.make_raw_depth(seed, H, W)
    r = fo.preprocess64(raw, K)
    f32 = fo.preprocess(raw, K)
    rep = fo.device_report(*f32, r, f32)
    assert not rep["failures"]
    assert rep["depth_frac"] < 0.5 and rep["normal_frac"] < 0.5
    assert rep["tainted"] < 1e-2 * rep["valid"]


def test_comparison_rewrites():
    """(double)x < 0.01 <=> x <= 0.01f and (double)d >= 0.1 <=> d >= 0.1f on the floats around each threshold."""
    for th, fth, op64, op32 in ((0.01, F32(0.01), lambda a: a < 0.01, lambda a: a <= F32(0.01)),
                                (0.1, F32(0.1), lambda a: a >= 0.1, lambda a: a >= F32(0.1))):
        x = fth
        for _ in range(64):
            x = np.nextafter(x, F32(-np.inf))
        for _ in range(128):
            assert op64(float(x)) == bool(op32(x)), x
            x = np.nextafter(x, F32(np.inf))
    assert float(F32(0.01)) < 0.01 < float(ff.up(0.01)) and float(ff.down(0.1)) < 0.1 < float(F32(0.1))


@pytest.mark.parametrize("sigma_d", [1.5, 2.0, 3.0])
@pytest.mark.parametrize("sigma_r", [1e5, 1.0, 0.05, 1e-3])
def test_weight_table_shortcut_is_exact(sigma_d, sigma_r):
    """Where (centre - d)^2 < t_q the kernel uses expf(a_tap) for expf(a_tap - dd / inv2sr); that is exact when
    fl(a - fl(dd / inv2sr)) == a for every float dd below t_q (a != 0), and for the centre tap (a = 0) when the argument stays within
    2^-26 of 0, where exp rounds to 1.  Checked with the device's own float32 operations, for every tap of every
    radius 0..5, on dd from 0 up to t_q (a geometric sweep plus the floats next to t_q)."""
    inv2sd = F32(2.0) * F32(sigma_d) * F32(sigma_d)
    inv2sr = F32(2) * F32(sigma_r) * F32(sigma_r)
    for br in range(6):
        side = 2 * br + 1
        for t in range(side * side):
            mm, nn = t // side - br, t % side - br
            a = -F32(mm * mm + nn * nn) / inv2sd
            tq = inv2sr * abs(a) * F32(1.4901161e-8) if a != 0 else inv2sr * F32(1.4901161e-8)
            below = np.concatenate([[F32(0)], (tq * np.geomspace(1e-12, 1, 200, dtype=np.float64)).astype(F32)])
            near = [ff.down(tq, k) for k in range(1, 9)]
            dd = np.array([v for v in list(below) + near if v < tq], F32)
            with np.errstate(under="ignore"):
                arg = a - dd / inv2sr
                if a != 0:
                    assert np.all(arg == a), (br, t, sigma_d, sigma_r)
                else:       # the centre tap: |arg| < 2^-26, and exp(arg) > 1 - 2^-25 rounds to expf(0) = 1
                    assert np.all(-arg <= F32(2.0 ** -26)) and np.all(np.exp(arg.astype(np.float64)) > 1 - 2.0 ** -25)
                    assert np.all(np.exp(arg) == F32(1))
            # and t_q is within a factor 8 of where the argument starts to move, so the shortcut is taken wherever it matters
            if a != 0:
                assert (a - (tq * F32(8)) / inv2sr) != a
