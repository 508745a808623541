"""The application layer without a GPU (bundletrack_b200/sequence.py): the dataset loaders on synthetic trees, the image layouts the readers
accept and refuse, the LF-Net client's wire format over inproc://, frame 0's initial pose, and the C++ shim's uint16 overloads."""
import os
import subprocess
import struct
import textwrap
import threading
import zlib

import numpy as np
import pytest

from bundletrack_b200 import _lib, policy, sequence, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _pose_text(P):
    return "".join(" ".join(f"{v:.9g}" for v in row) + "\n" for row in P)


def _rigid(seed, scale=1.0):
    rng = np.random.default_rng(seed)
    P = np.eye(4)
    P[:3, :3] = synth.so3_exp(rng.normal(size=3)) * scale
    P[:3, 3] = rng.uniform(-0.3, 0.3, 3) + [0, 0, 0.8]
    return P


def _nocs_tree(root, scene=2, model="mug_brown_norm", ids=(3, 0, 7), other_scene_ids=(1,)):
    """A NOCS tree: data list lines for `ids` in this order (plus lines of other scenes), two ground-truth files, colour files for listdir mode."""
    nocs = os.path.join(root, "NOCS")
    data = f"{nocs}/real_test/scene_{scene}"
    os.makedirs(data)
    gt = f"{nocs}/gts/real_test_text/scene_{scene}/model_{model}"
    os.makedirs(gt)
    with open(f"{gt}/0001.txt", "w") as f:
        f.write(_pose_text(_rigid(2)))
    with open(f"{gt}/0000.txt", "w") as f:             # the first sorted file
        f.write(_pose_text(_rigid(1, 0.3)))
    lst = f"{nocs}/NOCS-REAL275-additional/data_list/real_val/6/{model}"
    os.makedirs(lst)
    lines = [f"real_val/scene_{s}/{k:04d}" for s in other_scene_ids for k in (5,)] + [f"real_val/scene_{scene}/{k:04d}" for k in ids]
    with open(f"{lst}/list.txt", "w") as f:
        f.write("\n".join(lines) + "\n")
    for k in (9, 4, 1):
        for suffix in ("color.png", "depth.png", "meta.txt"):
            open(f"{data}/{k:04d}_{suffix}", "w").close()
    return nocs


def test_nocs_loader_data_list(tmp_path):
    nocs = _nocs_tree(str(tmp_path))
    ld = sequence.NocsScene(nocs, 2, "mug_brown_norm", "/masks/x")
    assert [f.id_str for f in ld.frames] == ["0003", "0000", "0007"]           # list order, other scenes' lines skipped
    data = f"{nocs}/real_test/scene_2/"
    assert ld.frames[1].colour == f"{data}/../../real_test/scene_2/0000_color.png"
    assert ld.frames[1].depth == data + "0000_depth.png" and ld.frames[1].mask == "/masks/x/0000.png"
    assert np.array_equal(ld.K, np.array([[591.0125, 0, 322.525], [0, 590.16775, 244.11084], [0, 0, 1]], np.float32))
    assert np.array_equal(ld.ob_in_cam0, np.loadtxt(f"{nocs}/gts/real_test_text/scene_2/model_mug_brown_norm/0000.txt").astype(np.float32))
    assert ld.mask_mode == _lib.BT_MASK_LARGEST_HULL
    assert np.array_equal(ld.initial_pose(0), sequence.initial_pose(ld.ob_in_cam0))
    for i in (1, 2):
        assert np.array_equal(ld.initial_pose(i), np.eye(4, dtype=np.float32))


def test_nocs_loader_scene_prefix_and_listdir(tmp_path):
    # "scene_1" is a substring of "scene_12": the reference takes those lines too
    nocs = _nocs_tree(str(tmp_path), scene=1, ids=(2,), other_scene_ids=(12,))
    assert [f.id_str for f in sequence.NocsScene(nocs, 1, "mug_brown_norm", "m").frames] == ["0005", "0002"]
    ld = sequence.NocsScene(nocs, 1, "mug_brown_norm", "m", use_6pack_datalist=False)
    assert [f.id_str for f in ld.frames] == ["0001", "0004", "0009"]           # sorted *color.png
    assert ld.frames[0].colour == f"{nocs}/real_test/scene_1/0001_color.png"


def test_nocs_id_from_the_first_color_in_the_path(tmp_path):
    # a directory whose name contains "color" earlier in the path decides the id, as DataLoader.cpp:163 does
    root = tmp_path / "my_colorful_data"
    nocs = _nocs_tree(str(root), ids=(3,))
    path = f"{nocs}/real_test/scene_2//../../real_test/scene_2/0003_color.png"
    k = path.find("color")
    ld = sequence.NocsScene(nocs, 2, "mug_brown_norm", "m")
    assert k < path.find("0003_color") and ld.frames[0].id_str == path[k - 5:k - 1] != "0003"
    assert ld.frames[0].depth == f"{nocs}/real_test/scene_2/{path[k - 5:k - 1]}_depth.png"


def test_ycbineoat_loader(tmp_path):
    d = tmp_path / "bleach0"
    for sub in ("rgb", "depth", "masks", "annotated_poses"):
        (d / sub).mkdir(parents=True)
    for name in ("0002.png", "0000.png", "0001.tar.png"):
        (d / "rgb" / name).touch()
    K = np.array([[319.58, 0, 320.22], [0, 417.11, 244.35], [0, 0, 1]])
    (d / "cam_K.txt").write_text(_pose_text(K))
    (d / "annotated_poses" / "0000000.txt").write_text(_pose_text(_rigid(4)))
    (d / "annotated_poses" / "0000001.txt").write_text(_pose_text(_rigid(5)))
    ld = sequence.YcbineoatVideo(str(d))
    assert [f.id_str for f in ld.frames] == ["0000", "0001", "0002"]             # the name up to its first "."
    assert ld.frames[1].depth == f"{d}/depth/0001.png" and ld.frames[1].mask == f"{d}/masks/0001.png"
    assert np.array_equal(ld.K, K.astype(np.float32))
    assert np.array_equal(ld.ob_in_cam0, _rigid(4).astype(np.float32)) and ld.mask_mode == _lib.BT_MASK_AS_IS
    assert np.array_equal(ld.initial_pose(2), np.eye(4, dtype=np.float32))


@pytest.mark.parametrize("seed,scale", [(0, 1.0), (1, 0.25), (2, 3.0), (3, 1.0)])
def test_initial_pose_within_4_ulp(seed, scale):
    G = _rigid(seed, scale).astype(np.float32)
    P = sequence.initial_pose(G)
    R = np.linalg.inv(G.astype(np.float64))
    R[:3, :3] /= np.linalg.norm(R[:3, :3], axis=0)
    ulp = np.spacing(np.abs(R).astype(np.float32))
    assert P.dtype == np.float32 and (np.abs(P - R) <= 4 * ulp).all(), np.abs(P - R) / ulp


# ---- image layouts ------------------------------------------------------------------------------------------------------------------------

def _png_raw(path, W, H, depth, ctype, rows: bytes, extra=b""):
    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)
    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, depth, ctype, 0, 0, 0)) + extra
                + chunk(b"IDAT", zlib.compress(rows)) + chunk(b"IEND", b""))


def _readers():
    out = []
    for name, mod in (("cv2", "cv2"), ("pil", "PIL")):
        try:
            __import__(mod)
            out.append(name)
        except ImportError:
            pass
    return out


@pytest.fixture
def images(tmp_path):
    rng = np.random.default_rng(3)
    H, W = 37, 53
    d = rng.integers(0, 65536, (H, W), dtype=np.uint16)
    d[0, :4] = [0, 99, 100, 65535]
    m = rng.integers(0, 256, (H, W), dtype=np.uint8)
    c = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    paths = {k: str(tmp_path / f"{k}.png") for k in ("depth", "mask", "colour")}
    synth.write_png(paths["depth"], d)
    synth.write_png(paths["mask"], m)
    synth.write_png(paths["colour"], c)
    rgba = np.concatenate([c[..., ::-1], np.full((H, W, 1), 7, np.uint8)], 2)
    paths["rgba"] = str(tmp_path / "rgba.png")
    _png_raw(paths["rgba"], W, H, 8, 6, b"".join(b"\0" + rgba[y].tobytes() for y in range(H)))
    return paths, d, m, c


@pytest.mark.parametrize("reader", _readers())
def test_accepted_layouts_read_as_written(images, reader):
    paths, d, m, c = images
    assert np.array_equal(sequence.read_image(paths["depth"], "depth", reader), d)
    assert np.array_equal(sequence.read_image(paths["mask"], "mask", reader), m)
    assert np.array_equal(sequence.read_image(paths["colour"], "colour", reader), c)
    assert np.array_equal(sequence.read_image(paths["rgba"], "colour", reader), c)       # IMREAD_COLOR drops alpha
    got = sequence.read_image(paths["depth"], "depth", reader)
    assert got.dtype == np.uint16 and got.flags.c_contiguous


@pytest.mark.skipif(len(_readers()) < 2, reason="needs both cv2 and PIL")
def test_cv2_and_pil_give_identical_arrays(images):
    paths = images[0]
    for kind, p in (("depth", paths["depth"]), ("mask", paths["mask"]), ("colour", paths["colour"]), ("colour", paths["rgba"])):
        a, b = sequence.read_image(p, kind, "cv2"), sequence.read_image(p, kind, "pil")
        assert a.dtype == b.dtype and np.array_equal(a, b), (kind, p)


def test_refused_layouts_name_the_file(tmp_path):
    H, W = 8, 9
    u8, u16, rgb = np.zeros((H, W), np.uint8), np.zeros((H, W), np.uint16), np.zeros((H, W, 3), np.uint8)
    cases = []
    p = str(tmp_path / "depth8.png"); synth.write_png(p, u8); cases.append((p, "depth"))           # 8-bit depth
    p = str(tmp_path / "mask16.png"); synth.write_png(p, u16); cases.append((p, "mask"))           # 16-bit mask
    p = str(tmp_path / "mask3.png"); synth.write_png(p, rgb); cases.append((p, "mask"))            # 3-channel mask
    p = str(tmp_path / "colour16.png"); synth.write_png(p, u16); cases.append((p, "colour"))       # 16-bit grey colour
    p = str(tmp_path / "pal.png")                                                                  # palette mask
    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)
    _png_raw(p, W, H, 8, 3, b"".join(b"\0" + bytes(W) for _ in range(H)), chunk(b"PLTE", bytes(range(6))))
    cases.append((p, "mask"))
    p = str(tmp_path / "depth_ga.png")                                                             # 16-bit grey + alpha depth
    _png_raw(p, W, H, 16, 4, b"".join(b"\0" + bytes(4 * W) for _ in range(H)))
    cases.append((p, "depth"))
    p = str(tmp_path / "not_a.png"); open(p, "wb").write(b"JFIF" * 10); cases.append((p, "colour"))
    for p, kind in cases:
        for reader in _readers() or [None]:
            with pytest.raises(ValueError, match=os.path.basename(p)):
                sequence.read_image(p, kind, reader)


# ---- the LF-Net client ----------------------------------------------------------------------------------------------------------------------

def _serve(ctx, endpoint, replies, got):
    import zmq as z
    s = ctx.socket(z.REP)
    s.bind(endpoint)
    try:
        for rep in replies:
            got.append(s.recv_multipart())
            s.send_multipart(rep)
    finally:
        s.close(0)


def _reply(n, dim, seed=0):
    rng = np.random.default_rng(seed)
    k = rng.uniform(0, 400, (n, 2)).astype(np.float32)
    d = rng.normal(size=(n, dim)).astype(np.float32)
    return [np.array([n, dim], np.int32).tobytes(), k.tobytes(), d.tobytes()], k, d


def test_lfnet_client_wire_format_and_drop_path():
    z = pytest.importorskip("zmq")
    ctx = z.Context()
    ep = "inproc://lfnet-test"
    good, k, d = _reply(37, 256)
    replies = [good, _reply(5, 128)[0], [b"\x01\x00", b"", b""], [good[0], good[1]], _reply(0, 256)[0]]
    got = []
    th = threading.Thread(target=_serve, args=(ctx, ep, replies, got))
    th.start()
    cl = sequence.LfnetClient(ep, timeout_s=20, context=ctx)
    try:
        req = np.random.default_rng(1).integers(0, 256, (400, 400, 3), dtype=np.uint8)
        roi = (100, 260, 80, 300)
        kp, de = cl("0000", req, roi)
        ek, ed = policy.lfnet_parse_reply(good, roi)
        assert np.array_equal(kp, ek) and np.array_equal(de, ed) and np.array_equal(de, d)
        assert got[0][0] == np.array([400, 400], np.int32).tobytes() and got[0][1] == req.tobytes() and len(got[0]) == 2
        for i in range(3):                                       # dim 128, a header that does not parse, two parts: dropped
            with pytest.raises(sequence.DetectionFailed):
                cl(f"{i + 1:04d}", req, roi)
        kp, de = cl("0004", req, roi)
        assert kp.shape == (0, 2) and de.shape == (0, 256)
    finally:
        th.join()
        cl.close()
        ctx.term()


def test_lfnet_client_timeout_names_the_endpoint():
    z = pytest.importorskip("zmq")
    ctx = z.Context()
    ep = "inproc://lfnet-silent"
    s = ctx.socket(z.REP)
    s.bind(ep)
    cl = sequence.LfnetClient(ep, timeout_s=0.2, context=ctx)
    try:
        with pytest.raises(RuntimeError, match="inproc://lfnet-silent"):
            cl("0000", np.zeros((400, 400, 3), np.uint8), (0, 20, 0, 20))
    finally:
        cl.close()
        s.close(0)
        ctx.term()


def test_cpp_shim_uint16_overloads_compile(tmp_path):
    src = tmp_path / "shim_u16.cpp"
    src.write_text(textwrap.dedent(r'''
        #include "bundletrack_b200/hostcpp/bt_optimizer.hpp"
        #include <cstdio>
        struct Mat4 { float m[16]; float& operator()(int r, int c) { return m[c * 4 + r]; } float operator()(int r, int c) const { return m[c * 4 + r]; } };
        struct Mat3 { float m[9]; float operator()(int r, int c) const { return m[c * 3 + r]; } };
        struct Vec4 { float v[4]; float& operator()(int i) { return v[i]; } };
        struct float4_ { float x, y, z, w; };
        int main() {
            try {
                Mat3 K{}; Vec4 roi{};
                processDepthNormalsAndMask(nullptr, (const uint16_t*)nullptr, (const uint8_t*)nullptr, BT_MASK_LARGEST_HULL, (float*)nullptr,
                                           (float4_*)nullptr, (float4_*)nullptr, (uint8_t*)nullptr, (int32_t*)nullptr, 480, 640, K, BtDepthConfig(), roi);
            } catch (const std::exception& e) { std::printf("caught: %s\n", e.what()); }
            try {
                bt_tracker_params p{};
                BundlerGpu b(p);
                Mat4 pose{}; int id = -1;
                b.beginFrame<Mat4>(0, nullptr, (const uint16_t*)nullptr, nullptr, nullptr, nullptr, id, pose);
            } catch (const std::exception& e) { std::printf("caught: %s\n", e.what()); }
            return 0;
        }
    '''))
    exe = tmp_path / "shim_u16"
    lib_dir = os.path.join(ROOT, "bundletrack_b200", "lib")
    subprocess.check_call(["g++", "-std=c++17", "-I", ROOT, str(src), "-o", str(exe), "-L", lib_dir, "-lbundletrack_b200", f"-Wl,-rpath,{lib_dir}"])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0, out.stderr
    assert out.stdout.count("caught:") == 2, out.stdout
