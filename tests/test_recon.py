"""The object-model oracle (oracle/recon_oracle.py) on depth maps of an analytic sphere and ellipsoid seen from 26 views around them: the
marching-tetrahedra mesh is closed and consistently wound, a sphere (Euler characteristic 2), encloses the right volume and lies on the
true surface; the tet tables are positively oriented; write_ply's bytes parse back to the same arrays."""
import numpy as np
import pytest

from bundletrack_b200 import recon, synth
from oracle import recon_oracle as ro

K = (600.0, 600.0, 319.5, 239.5)
H, W = 480, 640


def _views(radii):
    T = ro.views_around(0.35)
    depths = [synth.render_ellipsoid(radii, T[k], K, H, W, None)[0] for k in range(len(T))]
    return depths, np.stack([np.linalg.inv(t) for t in T]).astype(np.float32)


def test_tets_tile_the_cube_with_positive_orientation():
    corner = lambda c: np.array([c & 1, (c >> 1) & 1, (c >> 2) & 1], np.float64)
    vol = 0.0
    for code in ro.TETS:
        p = [corner(c) for c in code]
        det = np.linalg.det(np.stack([p[1] - p[0], p[2] - p[0], p[3] - p[0]]))
        assert det > 0
        vol += det / 6
    assert vol == pytest.approx(1.0)


@pytest.mark.parametrize("inside", range(1, 15))
def test_every_case_faces_the_outside(inside):
    """Each triangle's normal points from the inside corners of its tet to the outside ones."""
    corner = lambda c: np.array([c & 1, (c >> 1) & 1, (c >> 2) & 1], np.float64)
    for t, code in enumerate(ro.TETS):
        ins = [corner(code[k]) for k in range(4) if inside >> k & 1]
        out = [corner(code[k]) for k in range(4) if not inside >> k & 1]
        for tri in ro.tet_triangles(t, inside):
            p = [0.5 * (corner(a) + corner(b)) for a, b in tri]
            n = np.cross(p[1] - p[0], p[2] - p[0])
            assert np.dot(n, np.mean(out, 0) - np.mean(ins, 0)) > 0, (t, inside, tri)


@pytest.mark.parametrize("radii", [(0.05, 0.05, 0.05), (0.06, 0.045, 0.035)], ids=["sphere", "ellipsoid"])
def test_oracle_mesh_of_a_rendered_object(radii):
    voxel = 0.004
    depths, cim = _views(radii)
    g = ro.fuse(depths, cim, K, voxel, 3 * voxel)
    v, f = ro.mesh(g, voxel)
    assert len(f) > 1000
    assert ro.edge_check(f)
    assert ro.euler(v, f) == 2
    assert len(np.unique(f)) == len(v)                        # every vertex is used
    vol = ro.signed_volume(v, f)
    assert vol > 0 and abs(vol / (4 / 3 * np.pi * np.prod(radii)) - 1) < 0.03
    assert ro.ellipsoid_distance(v, radii).max() < 0.5 * voxel
    # the grid holds the object: the valid pixels' bounds are the box the object's silhouettes span
    assert np.all(g["lo"] > -np.asarray(radii) - voxel) and np.all(g["hi"] < np.asarray(radii) + voxel)


def test_grid_rules():
    lo, hi = np.array([0.0, -0.1, 0.2], np.float32), np.array([0.1, -0.05, 0.2], np.float32)
    n, origin = ro.grid(lo, hi, 0.01, 0.025)
    m = 4                                                     # ceil(2.5) + 1
    assert n == (int(np.ceil(np.float32(0.1) / np.float32(0.01))) + 1 + 2 * m, 5 + 1 + 2 * m, 1 + 2 * m)
    assert np.array_equal(origin, (lo - np.float32(m) * np.float32(0.01)).astype(np.float32))
    assert ro.bounds([np.zeros((4, 4), np.float32)], np.eye(4)[None], (1, 1, 2, 2)) is None


def test_unobserved_tets_make_no_faces():
    """A field with count 0 at one corner of a crossing: the tets that touch it contribute nothing, and no vertex is left unused."""
    n = (3, 3, 3)
    s = np.ones((3, 3, 3), np.float32)
    s[1, 1, 1] = -1
    c = np.ones((3, 3, 3), np.int32)
    g = {"dims": n, "origin": np.zeros(3, np.float32), "sum": s, "count": c}
    v, f = ro.mesh(g, 1.0)
    assert ro.edge_check(f) and ro.euler(v, f) == 2 and ro.signed_volume(v, f) > 0
    c[0, 0, 0] = 0
    v2, f2 = ro.mesh(g, 1.0)
    assert 0 < len(f2) < len(f) and len(np.unique(f2)) == len(v2)


def _read_ply(path):
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode("ascii").split("\n")
    assert head[:2] == ["ply", "format binary_little_endian 1.0"]
    nv = int(next(l for l in head if l.startswith("element vertex")).split()[2])
    nf = int(next(l for l in head if l.startswith("element face")).split()[2])
    assert "property list uchar int vertex_indices" in head and [l for l in head if l.startswith("property float")] == [
        "property float x", "property float y", "property float z"]
    v = np.frombuffer(data, "<f4", 3 * nv, end).reshape(nv, 3)
    rows = np.frombuffer(data, [("n", "u1"), ("i", "<i4", (3,))], nf, end + 12 * nv)
    assert (rows["n"] == 3).all() and len(data) == end + 12 * nv + 13 * nf
    return v, rows["i"]


def test_write_ply_round_trip(tmp_path):
    g = {"dims": (3, 3, 3), "origin": np.array([0.1, 0.2, 0.3], np.float32), "sum": np.ones((3, 3, 3), np.float32),
         "count": np.ones((3, 3, 3), np.int32)}
    g["sum"][1, 1, 1] = -0.5
    v, f = ro.mesh(g, 0.01)
    path = str(tmp_path / "m.ply")
    recon.write_ply(path, v, f)
    v2, f2 = _read_ply(path)
    assert np.array_equal(v2, v) and np.array_equal(f2, f)
    recon.write_ply(path, np.zeros((0, 3)), np.zeros((0, 3)))
    v3, f3 = _read_ply(path)
    assert v3.shape == (0, 3) and f3.shape == (0, 3)
    with pytest.raises(ValueError):
        recon.write_ply(path, v, f + len(v))
