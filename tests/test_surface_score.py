"""Object model accuracy on the host (DESIGN.md §3.15): the sampling restatement in oracle/surface_oracle.py is uniform by area, lies on its
faces, never picks a zero-area face and is reproducible; bt_surface_score equals a numpy restatement; recon.read_mesh reads OBJ and PLY."""
import numpy as np
import pytest

from bundletrack_b200 import metrics, recon
from oracle import surface_oracle as so

# a unit square split into a sliver (area 1e-3 of the square) and the rest
SQUARE_V = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [0.002, 1, 0]], np.float64)
SQUARE_F = np.array([[0, 1, 4], [1, 2, 4], [0, 4, 3]], np.int32)


def test_sampling_is_uniform_by_area():
    n = 200_000
    _, face = so.sample(SQUARE_V, SQUARE_F, n, seed=3, return_faces=True)
    area = 0.5 * so.face_weights(SQUARE_V, SQUARE_F)
    p = area / area.sum()
    counts = np.bincount(face, minlength=3)
    for c, q in zip(counts, p):
        assert abs(c - n * q) <= 5 * np.sqrt(n * q * (1 - q)) + 1, (counts, n * p)
    assert counts[2] > 0                                     # the sliver (1e-3 of the area) is sampled


def test_samples_lie_on_their_faces():
    rng = np.random.default_rng(1)
    V = rng.normal(size=(60, 3))
    F = rng.integers(0, 60, size=(200, 3)).astype(np.int32)
    F = F[(F[:, 0] != F[:, 1]) & (F[:, 1] != F[:, 2]) & (F[:, 0] != F[:, 2])]
    p, face = so.sample(V, F, 5000, seed=9, return_faces=True)
    A, B, C = V[F[face, 0]], V[F[face, 1]], V[F[face, 2]]
    # barycentric coordinates by least squares in the face's plane: all >= 0, summing to 1, and no distance off the plane
    M = np.stack([B - A, C - A], -1)
    uv, *_ = zip(*[np.linalg.lstsq(M[i], p[i] - A[i], rcond=None) for i in range(len(p))])
    uv = np.asarray(uv)
    assert (uv >= -1e-9).all() and (uv.sum(1) <= 1 + 1e-9).all()
    off = p - (A + np.einsum("nij,nj->ni", M, uv))
    assert np.abs(off).max() <= 1e-12


def test_degenerate_faces_are_never_chosen():
    V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 2, 2], [3, 3, 3], [4, 4, 4], [0.5, 1e-12, 0]], np.float64)
    # a zero-area face (collinear), a repeated vertex, the real triangle, and an area below 2^-32 of it
    F = np.array([[3, 4, 5], [0, 0, 1], [0, 1, 2], [0, 1, 6]], np.int32)
    _, face = so.sample(V, F, 20_000, seed=0, return_faces=True)
    assert set(face.tolist()) == {2}
    with pytest.raises(ValueError, match="no area"):
        so.sample(V, F[:2], 10)


def test_the_same_seed_gives_the_same_bytes():
    v, f = so.uv_sphere(0.05, 12, 20)
    a, b = so.sample(v, f, 3000, seed=7), so.sample(v, f, 3000, seed=7)
    assert a.tobytes() == b.tobytes()
    assert a.tobytes() != so.sample(v, f, 3000, seed=8).tobytes()
    assert np.abs(np.linalg.norm(a, axis=1) - 0.05).max() < 0.05 * (1 - np.cos(np.pi / 12))


def test_splitmix64_known_values():
    # the published splitmix64 stream from state 0
    assert so.splitmix64(0, np.arange(3, dtype=np.uint64)).tolist() == [0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4, 0x06C45D188009454F]


@pytest.mark.parametrize("case", ["random", "ties", "zero"])
def test_surface_score_equals_numpy(case):
    rng = np.random.default_rng(4)
    taus = [0.002, 0.005, 0.01]
    if case == "random":
        a, b = rng.exponential(0.004, 1001), rng.exponential(0.006, 37)
    elif case == "ties":                                     # d == tau is not counted; repeated values at the quantiles
        a = np.array([0.002, 0.005, 0.01, 0.001, 0.002, 0.0])
        b = np.array([0.01, 0.01, 0.0049999, 0.005])
    else:                                                    # nothing within any tau: P + R = 0 gives F = 0
        a, b = np.full(5, 0.5), np.full(3, 0.25)
    got = metrics.surface_score(a, b, taus)
    want = so.score(a, b, taus)
    for k in metrics.SCORE_KEYS:
        assert got[k] == want[k], k
    for k in ("precision", "recall", "fscore"):
        assert got[k] == want[k], k
    assert got["taus"] == taus
    assert got["median_model_to_ref"] == pytest.approx(np.percentile(a, 50), rel=1e-14, abs=1e-18)
    assert got["p95_ref_to_model"] == pytest.approx(np.percentile(b, 95), rel=1e-14, abs=1e-18)
    if case == "ties":
        assert got["precision"] == [2 / 6, 4 / 6, 5 / 6] and got["recall"] == [0.0, 1 / 4, 2 / 4]
    if case == "zero":
        assert got["fscore"] == [0.0, 0.0, 0.0]


def test_surface_score_refusals():
    ok = np.ones(3)
    for a, b, t in ((ok, ok, [0.0]), (ok, ok, [np.inf]), (np.array([1.0, np.nan]), ok, [0.1]), (ok, -ok, [0.1]), (ok[:0], ok, [0.1])):
        with pytest.raises(Exception):
            metrics.surface_score(a, b, t)
    assert metrics.surface_score(ok, ok, [])["taus"] == []


def test_read_mesh_obj(tmp_path):
    p = tmp_path / "m.obj"
    p.write_text("# a quad with texture and normal indices, then a triangle by negative indices\n"
                 "v 0 0 0\nv 1 0 0\nv 1 1 0\nv 0 1 0\nvt 0 0\nvn 0 0 1\n"
                 "f 1/1/1 2/1/1 3/1/1 4/1/1\n"
                 "v 0 0 1\n"
                 "f -1 -4//1 -3\n"
                 "f 1//1 5 2/1\n")
    v, f = recon.read_mesh(str(p))
    assert v.dtype == np.float64 and v.shape == (5, 3) and v[4].tolist() == [0, 0, 1]
    assert f.dtype == np.int32 and f.tolist() == [[0, 1, 2], [0, 2, 3], [4, 1, 2], [0, 4, 1]]
    (tmp_path / "bad.obj").write_text("v 0 0 0\nf 1 2 3\n")
    with pytest.raises(ValueError, match="bad face"):
        recon.read_mesh(str(tmp_path / "bad.obj"))


def test_read_mesh_round_trips_write_ply(tmp_path):
    rng = np.random.default_rng(2)
    v = rng.normal(size=(50, 3)).astype(np.float32)
    f = rng.integers(0, 50, size=(80, 3)).astype(np.int32)
    p = str(tmp_path / "m.ply")
    recon.write_ply(p, v, f)
    rv, rf = recon.read_mesh(p)
    assert rv.dtype == np.float64 and np.array_equal(rv, v.astype(np.float64)) and np.array_equal(rf, f)
    q = str(tmp_path / "m2.ply")
    recon.write_ply(q, rv, rf)
    assert open(p, "rb").read() == open(q, "rb").read()


def test_read_mesh_refuses_other_files(tmp_path):
    (tmp_path / "m.stl").write_bytes(b"solid x\n")
    with pytest.raises(ValueError, match="'.stl'"):
        recon.read_mesh(str(tmp_path / "m.stl"))
    (tmp_path / "a.ply").write_bytes(b"ply\nformat ascii 1.0\nelement vertex 0\nend_header\n")
    with pytest.raises(ValueError, match="ascii"):
        recon.read_mesh(str(tmp_path / "a.ply"))
