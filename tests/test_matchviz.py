"""The match images' numpy oracle (oracle/matchviz_oracle.py) against OpenCV: byte for byte on every recorded golden case
(tests/golden/ref_matchviz.npz, from scripts/make_golden_matchviz.py) and, where cv2 is importable, on a few hundred seeded cases drawn live;
the colour rule (the first RNG draw is red); the output shape and file names; and what the writer does past JPEG's size limit."""
import hashlib
import os

import numpy as np
import pytest

from oracle import matchviz_oracle as mv
from oracle import segment_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "ref_matchviz.npz"))
NAMES = [str(n) for n in GOLDEN["names"]]


def golden_images():
    """(name, oracle image, recorded image or None, recorded sha256 or None), the RNG carried across unseeded cases."""
    colour = segment_oracle.test_colour(int(GOLDEN["H"]), int(GOLDEN["W"]))
    state = mv.RNG_DEFAULT
    out = []
    for name in NAMES:
        seed = int(GOLDEN[f"{name}/seed"])
        if seed:
            state = mv.rng_seed(seed)
        img, state = mv.match_image(colour, GOLDEN[f"{name}/roi_a"], colour, GOLDEN[f"{name}/roi_b"], GOLDEN[f"{name}/uv"], state)
        whole = GOLDEN[f"{name}/image"] if f"{name}/image" in GOLDEN.files else None
        sha = str(GOLDEN[f"{name}/sha256"]) if f"{name}/sha256" in GOLDEN.files else None
        out.append((name, img, whole, sha))
    return out


def test_golden_cases_cover_the_quirks():
    shapes = {n: tuple(GOLDEN[f"{n}/shape"]) for n in NAMES}
    scales = {mv.viz_scale(int(GOLDEN[f"{n}/roi_a"][3] - GOLDEN[f"{n}/roi_a"][2]), int(GOLDEN[f"{n}/roi_b"][3] - GOLDEN[f"{n}/roi_b"][2])) for n in NAMES}
    assert 1 in scales and max(scales) >= 2
    counts = {len(GOLDEN[f"{n}/uv"]) for n in NAMES}
    assert {0, 1}.issubset(counts) and max(counts) >= 3000
    assert any(int(GOLDEN[f"{n}/seed"]) == 0 for n in NAMES)                    # an image that continues the RNG
    assert any(f"{n}/image" in GOLDEN.files for n in NAMES)                        # a case stored whole, to diff pixels against
    for n in NAMES:
        assert shapes[n] == (*mv.image_shape(GOLDEN[f"{n}/roi_a"], GOLDEN[f"{n}/roi_b"]), 3)


def test_oracle_equals_the_golden_images():
    for name, img, whole, sha in golden_images():
        assert img.shape == tuple(GOLDEN[f"{name}/shape"]), name
        if whole is not None:
            assert img.tobytes() == whole.tobytes(), name
        else:
            assert hashlib.sha256(img.tobytes()).hexdigest() == sha, name


def _random_case(rs):
    ha, wa, hb, wb = (int(v) for v in rs.integers(3, 70, 4))
    a = rs.integers(0, 256, (ha, wa, 3), dtype=np.uint8)
    b = rs.integers(0, 256, (hb, wb, 3), dtype=np.uint8)
    n = int(rs.integers(0, 25))
    # keypoints mostly inside their crops, some outside (clipping), some on the seam and the borders
    kp = np.stack([rs.uniform(-3, wa + 3, n), rs.uniform(-3, ha + 3, n), rs.uniform(-3, wb + 3, n), rs.uniform(-3, hb + 3, n)], 1)
    edge = rs.random((n, 4)) < 0.2
    kp[edge] = np.round(kp[edge])
    return a, b, kp.astype(np.float32), int(rs.integers(1, 2 ** 31))


def _cv_draw(cv2, a, b, kp):
    ka = [cv2.KeyPoint(float(x), float(y), 1) for x, y in kp[:, :2]]
    kb = [cv2.KeyPoint(float(x), float(y), 1) for x, y in kp[:, 2:]]
    m = [cv2.DMatch(i, i, 0) for i in range(len(kp))]
    return cv2.drawMatches(a, ka, b, kb, m, None, matchColor=(-1, -1, -1, -1), singlePointColor=(-1, -1, -1, -1),
                           flags=cv2.DrawMatchesFlags_NOT_DRAW_SINGLE_POINTS)


def test_oracle_equals_cv2_live():
    cv2 = pytest.importorskip("cv2")
    rs = np.random.default_rng(2024)
    for t in range(300):
        a, b, kp, seed = _random_case(rs)
        cv2.setRNGSeed(seed)
        ref = _cv_draw(cv2, a, b, kp)
        got, state = mv.draw_matches(a, b, kp, mv.rng_seed(seed))
        assert ref.tobytes() == got.tobytes(), t
        # the state after the image is where cv2 continues
        cv2.setRNGSeed(seed)
        _cv_draw(cv2, a, b, kp)
        nxt = _cv_draw(cv2, b, a, kp[:, [2, 3, 0, 1]])
        assert nxt.tobytes() == mv.draw_matches(b, a, kp[:, [2, 3, 0, 1]], state)[0].tobytes(), t


def test_resize_equals_cv2_live():
    cv2 = pytest.importorskip("cv2")
    rs = np.random.default_rng(5)
    for s in (1, 2, 3, 5, 9, 22, 90):
        img = rs.integers(0, 256, (int(rs.integers(1, 40)), int(rs.integers(1, 40)), 3), dtype=np.uint8)
        assert mv.resize_int(img, s).tobytes() == cv2.resize(img, (0, 0), fx=s, fy=s).tobytes(), s


def test_colour_rule_first_draw_is_red():
    """Scalar(rng(256), rng(256), rng(256)): the recorded images pin the right-to-left evaluation; the other orders must disagree."""
    state = mv.rng_seed(12345)
    (b, g, r), after = mv.match_colour(state)
    d = []
    s = state
    for _ in range(3):
        s = mv.rng_next(s)
        d.append((s & 0xFFFFFFFF) % 256)
    assert (r, g, b) == tuple(d) and after == s
    name = "octants"
    colour = segment_oracle.test_colour(int(GOLDEN["H"]), int(GOLDEN["W"]))
    orig = mv.match_colour
    try:
        mv.match_colour = lambda st: ((lambda c: ((c[0][2], c[0][1], c[0][0]), c[1]))(orig(st)))      # left to right instead
        img, _ = mv.match_image(colour, GOLDEN[f"{name}/roi_a"], colour, GOLDEN[f"{name}/roi_b"], GOLDEN[f"{name}/uv"],
                                mv.rng_seed(int(GOLDEN[f"{name}/seed"])))
    finally:
        mv.match_colour = orig
    ref = GOLDEN[f"{name}/image"] if f"{name}/image" in GOLDEN.files else None
    if ref is not None:
        assert img.tobytes() != ref.tobytes()
    else:
        assert hashlib.sha256(img.tobytes()).hexdigest() != str(GOLDEN[f"{name}/sha256"])


def test_rng_matches_opencv_default_and_zero_seed():
    assert mv.rng_seed(0) == mv.RNG_DEFAULT == 0xFFFFFFFF
    s = mv.rng_advance(mv.RNG_DEFAULT, 2)
    t = mv.RNG_DEFAULT
    for _ in range(6):
        t = mv.rng_next(t)
    assert s == t


def test_shape_and_scale():
    assert mv.image_shape((0, 10, 0, 10), (0, 20, 0, 30)) == (900, 900)                 # min(90, 30) = 30
    assert mv.image_shape((0, 640, 0, 451), (0, 640, 0, 10)) == (451, 1280)            # scale 1
    assert mv.image_shape((0, 640, 0, 10), (0, 640, 0, 10)) == (900, 2 * 640 * 90)     # past JPEG's width limit


def test_match_image_path_and_jpeg_limit(tmp_path):
    from bundletrack_b200 import overlay
    assert overlay.match_image_path("d", "0007", "0007", "0003", "before_ransac") == os.path.join("d", "0007", "0007_match_0003_before_ransac.jpg")
    assert overlay.rng_after(mv.RNG_DEFAULT, 5) == mv.rng_advance(mv.RNG_DEFAULT, 5)
    pytest.importorskip("cv2")
    wide = np.zeros((10, overlay.JPEG_MAX_SIDE + 1, 3), np.uint8)
    p = str(tmp_path / "a" / "wide.jpg")
    assert overlay.write_match_image(p, wide) is False and not os.path.exists(p)
    ok = str(tmp_path / "a" / "ok.jpg")
    assert overlay.write_match_image(ok, np.zeros((10, 20, 3), np.uint8)) is True and os.path.getsize(ok) > 0
