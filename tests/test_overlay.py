"""The tracking overlay's definition on the CPU: the numpy oracle's VoxelGrid (oracle/overlay_oracle.py) on hand cases and against an
independent dictionary-of-voxels restatement, its drawing against OpenCV and the golden frames, load_obj_points and write_log_frame."""
import os

import numpy as np
import pytest

from oracle import overlay_oracle as oo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def dict_voxel_grid(p, leaf):
    """VoxelGrid restated over a dict of voxels: bounds from the finite points, (i, j, k) per point, sums in input order."""
    p = np.asarray(p, F32).reshape(-1, 3)
    inv = F32(1) / F32(leaf)
    fin = [i for i in range(len(p)) if np.isfinite(p[i]).all()]
    if not fin:
        return np.zeros((0, 3), F32)
    mn = [min(p[i][a] for i in fin) for a in range(3)]
    mx = [max(p[i][a] for i in fin) for a in range(3)]
    if np.prod([int((mx[a] - mn[a]) * inv) + 1 for a in range(3)], dtype=object) > 2 ** 31 - 1:
        return p.copy()
    lo = [int(np.floor(mn[a] * inv)) for a in range(3)]
    div = [int(np.floor(mx[a] * inv)) - lo[a] + 1 for a in range(3)]
    vox = {}
    for i in fin:
        ijk = [int(np.floor(p[i][a] * inv) - F32(lo[a])) for a in range(3)]
        key = ijk[0] + ijk[1] * div[0] + ijk[2] * div[0] * div[1]
        s, n = vox.get(key, ([F32(0)] * 3, 0))
        vox[key] = ([F32(s[a] + p[i][a]) for a in range(3)], n + 1)
    return np.array([[s[a] / F32(n) for a in range(3)] for _, (s, n) in sorted(vox.items())], F32).reshape(-1, 3)


def same(a, b):
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def test_voxel_boundaries_and_negative_coordinates():
    # points exactly on voxel faces (0, 0.5, 1 at leaf 0.5) and negative ones: floorf puts -0.25 in voxel -1, 0.5 in voxel 1
    p = np.array([[0, 0, 0], [0.5, 0, 0], [-0.25, 0, 0], [1.0, 0, 0], [-0.5, 0, 0], [0.25, 0, 0], [-0.75, 0, 0]], F32)
    got = oo.voxel_grid(p, 0.5)
    want = np.array([[-0.75, 0, 0], [-0.375, 0, 0], [0.125, 0, 0], [0.5, 0, 0], [1.0, 0, 0]], F32)
    assert same(got, want)
    assert same(got, dict_voxel_grid(p, 0.5))


def test_single_point_and_one_voxel():
    p = np.array([[0.1234, -5.5, 3.25]], F32)
    assert same(oo.voxel_grid(p, 0.01), p)
    rng = np.random.default_rng(1)
    q = (F32(0.2) + rng.random((1000, 3)).astype(F32) * F32(0.009)).astype(F32)     # all inside one 1 cm voxel
    got = oo.voxel_grid(q, 0.01)
    assert got.shape == (1, 3)
    s = np.zeros(3, F32)
    for row in q:
        s = (s + row).astype(F32)
    assert same(got, (s / F32(1000)).reshape(1, 3))


def test_non_finite_points_are_skipped():
    p = np.array([[0, 0, 0], [np.nan, 0, 0], [0.001, 0.002, 0.003], [np.inf, 1, 1], [5, -np.inf, 0], [1, 1, 1]], F32)
    got = oo.voxel_grid(p, 0.1)
    assert same(got, dict_voxel_grid(p, 0.1))
    assert got.shape == (2, 3) and np.isfinite(got).all()
    assert oo.voxel_grid(np.full((3, 3), np.nan, F32), 0.1).shape == (0, 3)


def test_overflow_returns_the_input():
    rng = np.random.default_rng(2)
    p = (rng.random((500, 3)) * 10).astype(F32)
    p[7] = np.nan
    got = oo.voxel_grid(p, 1e-6)
    assert got.shape == p.shape and np.array_equal(np.isnan(got), np.isnan(p)) and np.array_equal(got[~np.isnan(p)], p[~np.isnan(p)])


@pytest.mark.parametrize("seed", range(4))
def test_random_clouds_equal_dictionary_of_voxels(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 3000))
    p = (rng.normal(size=(n, 3)) * rng.random(3) * 0.2 + rng.normal(size=3)).astype(F32)
    p[rng.random(n) < 0.02, rng.integers(0, 3)] = np.nan
    for leaf in (0.01, 0.015, 0.05):
        assert same(oo.voxel_grid(p, leaf), dict_voxel_grid(p, leaf)), (seed, leaf)


def test_roundf_and_projection_rules():
    v = np.array([0.5, 1.5, -0.5, -1.5, 0.49999997, -0.49999997, 2.5], F32)
    assert oo._roundf(v).tolist() == [1, 2, -1, -2, 0, -0.0, 3]
    # (u, v) rounding to -0 is column 0; NaN (z = 0 with x = 0), infinite and behind-camera-but-inside points follow the rules
    c = np.array([[-0.005, 0, 1], [0, 0, 0], [1, 0, 0], [0.2, 0.1, -1], [1e30, 0, 1e-30]], F32)
    uv = oo.project(c, (100, 100, 0.2, 0.5), 10, 10)
    assert uv.tolist() == [[0, 1]]
    uv = oo.project(np.array([[-0.05, -0.04, -1]], F32), (100, 100, 0, 0), 10, 10)
    assert uv.tolist() == [[5, 4]]


def test_inverse4_matches_float64_inverse_closely():
    from bundletrack_b200 import synth
    P = synth.se3(synth.so3_exp(np.array([0.3, -0.2, 0.5])), np.array([0.1, -0.2, 0.7])).astype(F32)
    assert np.abs(oo.inverse4(P) - np.linalg.inv(P.astype(np.float64))).max() < 1e-6


def _cv2():
    return pytest.importorskip("cv2")


def test_stamp_and_dimming_equal_opencv_at_every_border():
    cv2 = _cv2()
    H, W = 7, 9
    rng = np.random.default_rng(3)
    colour = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    fg = (rng.random((H, W)) < 0.5).astype(np.uint8)
    ref = colour.copy()
    for h in range(H):
        for w in range(W):
            if fg[h, w] == 0:
                ref[h, w] = [int(float(c) * 0.2) for c in ref[h, w]]
    assert same(oo.dim(colour, fg), ref)
    centres = [(u, v) for u in (0, 1, W // 2, W - 2, W - 1) for v in (0, 1, H // 2, H - 2, H - 1)]
    for u, v in centres:
        a = np.zeros((H, W, 3), np.uint8)
        b = a.copy()
        cv2.circle(a, (u, v), 1, (0, 255, 255), -1)
        oo.stamp(b, np.array([[u, v]]))
        assert same(a, b), (u, v)
    a, b = ref.copy(), ref.copy()
    for u, v in centres:
        cv2.circle(a, (u, v), 1, (0, 255, 255), -1)
    oo.stamp(b, np.array(centres))
    assert same(a, b)


def test_oracle_equals_golden_frames():
    g = np.load(os.path.join(ROOT, "tests", "golden", "ref_overlay.npz"))
    model = oo.voxel_grid(g["model"], 0.015)
    for f in range(len(g["ids"])):
        viz, raw = oo.render(g["colour"][f], g["fg"][f], model, g["cur_in_model"][f], g["K"])
        keep = ~g["label_mask"][f]
        assert np.array_equal(viz[keep], g["viz"][f][keep]), f
        assert same(raw, g["raw"][f]), f
    if _have_cv2():
        from bundletrack_b200.overlay import label
        for f in range(len(g["ids"])):
            viz, _ = oo.render(g["colour"][f], g["fg"][f], model, g["cur_in_model"][f], g["K"])
            assert same(label(viz, str(g["ids"][f])), g["viz"][f]), f


def _have_cv2():
    try:
        import cv2  # noqa: F401
        return True
    except ImportError:
        return False


OBJ = """# a model with vertex colours, normals, texture coordinates and faces
mtllib model.mtl
v 0.1 0.2 0.3 1.0 0.5 0.25
vn 0 0 1
v -1e-3 2.5e-2 -0.75
vt 0.5 0.5
  v 4 5 6
o part
f 1/1/1 2/1/1 3/1/1
v 7 8 9 0.1
"""


def test_load_obj_points(tmp_path):
    from bundletrack_b200.overlay import load_obj_points
    p = tmp_path / "model.obj"
    p.write_text(OBJ)
    got = load_obj_points(str(p))
    want = np.array([[0.1, 0.2, 0.3], [-1e-3, 2.5e-2, -0.75], [4, 5, 6], [7, 8, 9]], np.float64).astype(F32)
    assert same(got, want)
    assert same(oo.load_obj_vertices(str(p)), want)


def test_write_log_frame_writes_the_reference_files(tmp_path):
    cv2 = _cv2()
    from bundletrack_b200.overlay import write_log_frame
    rng = np.random.default_rng(4)
    viz = rng.integers(0, 256, (48, 64, 3), dtype=np.uint8)
    raw = rng.integers(0, 256, (48, 64, 3), dtype=np.uint8)
    write_log_frame(str(tmp_path), "0042", viz, raw)
    paths = [tmp_path / "0042" / "color_viz.jpg", tmp_path / "color_viz" / "0042_color_viz.jpg", tmp_path / "color_raw" / "0042_color_raw.png"]
    assert all(p.exists() for p in paths)
    img = viz.copy()
    cv2.putText(img, "0042", (5, 30), cv2.FONT_HERSHEY_PLAIN, 2, (255, 0, 0), 1, 8, False)
    ok, jpg = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 80])
    assert ok
    want = tmp_path / "want.jpg"
    cv2.imwrite(str(want), img, [cv2.IMWRITE_JPEG_QUALITY, 80])
    assert paths[0].read_bytes() == want.read_bytes() == paths[1].read_bytes() == jpg.tobytes()
    assert same(cv2.imread(str(paths[2]), cv2.IMREAD_UNCHANGED), raw)


def test_write_log_frame_without_cv2_says_so(monkeypatch):
    import sys
    from bundletrack_b200 import overlay
    monkeypatch.setitem(sys.modules, "cv2", None)
    with pytest.raises(RuntimeError, match="cv2"):
        overlay.write_log_frame("/nonexistent", "0000", np.zeros((4, 4, 3), np.uint8), np.zeros((4, 4, 3), np.uint8))


def test_loaders_find_the_model(tmp_path):
    from bundletrack_b200 import sequence
    v = tmp_path / "video"
    (v / "annotated_poses").mkdir(parents=True)
    (v / "rgb").mkdir()
    (v / "cam_K.txt").write_text("1 0 2\n0 3 4\n0 0 1\n")
    (v / "annotated_poses" / "0000000.txt").write_text(" ".join(str(x) for x in np.eye(4).reshape(-1)))
    assert sequence.YcbineoatVideo(str(v)).model_path is None
    assert sequence.YcbineoatVideo(str(v), "/models/obj/textured.obj").model_path == "/models/obj/textured.obj"


def test_cpp_overlay_shims_compile(tmp_path):
    """downsamplePointClouds / drawProjectPoints instantiate against the header with any operator()(row, col) matrix type, and link."""
    import shutil
    import subprocess
    import textwrap
    if not shutil.which("g++"):
        pytest.skip("no g++")
    src = tmp_path / "overlay_shim.cpp"
    src.write_text(textwrap.dedent(r'''
        #include "bundletrack_b200/hostcpp/bt_optimizer.hpp"
        struct M { float v[16]; float operator()(int r, int c) const { return v[4 * r + c]; } };
        int main(int argc, char**) {
            if (argc > 5) {          // never run: linking is the check
                bt_ctx* ctx = nullptr;
                std::vector<const float*> in(1, nullptr); std::vector<float*> out(1, nullptr); std::vector<int> n(1, 1);
                downsamplePointClouds(ctx, in, n, 0.015f, out, nullptr);
                M P{}, K{};
                drawProjectPoints(ctx, nullptr, 1, P, K, nullptr, nullptr, 480, 640, nullptr);
            }
            return 0;
        }
    '''))
    lib_dir = os.path.join(ROOT, "bundletrack_b200", "lib")
    exe = tmp_path / "overlay_shim"
    subprocess.check_call(["g++", "-std=c++17", "-I", ROOT, str(src), "-o", str(exe), "-L", lib_dir, "-lbundletrack_b200", f"-Wl,-rpath,{lib_dir}"])
    subprocess.check_call([str(exe)])
