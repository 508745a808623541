"""GPU tests of the LF-Net weights file: a network loaded by bt_lfnet_load_file equals one loaded from the TF variables, bit for bit; the
loader's refusals pass bt_lfnet_reserve's and bt_lfnet_load_weights' through; and the C++ loop of INTEGRATION.md §7 (BundlerGpu + LfnetGpu,
tests/cpp/lfnet_main.cpp) tracks a sequence exactly as run_sequence does with the LfnetDevice source, detection failures included."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest

from bundletrack_b200 import _lib, lfnet, sequence, synth
from oracle import lfnet_oracle as lo

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HP = dict(lfnet.DEFAULTS)
# no pixel is an NMS peak when every value counts as 0 (k_nms): the network of this threshold finds no keypoints on any request
HP_EMPTY = dict(HP, nms_thresh=1e30)


@pytest.fixture(scope="module")
def weights():
    return lo.random_weights(lfnet.weight_shapes(HP), 11)


@pytest.fixture(scope="module")
def files(weights, tmp_path_factory):
    d = tmp_path_factory.mktemp("lfnet_files")
    blob = lfnet.make_blob(weights, HP)
    out = {}
    for name, hp in (("net", HP), ("empty", HP_EMPTY)):
        out[name] = str(d / f"{name}.btlfnet")
        with open(out[name], "wb") as f:
            f.write(lfnet.weights_file_bytes(blob, hp))
    return out


@pytest.fixture(scope="module")
def requests(cuda_device):
    """Requests made by bt_lfnet_request from a synthetic scene in both mask modes, and a random image."""
    import torch
    from bundletrack_b200.frontend import FrameFrontEnd
    H, W = 240, 320
    seq = synth.make_sequence(23, 2, H=H, W=W)
    fe = FrameFrontEnd()
    out = []
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda_device)
    for k, mode in ((0, _lib.BT_MASK_LARGEST_HULL), (1, _lib.BT_MASK_AS_IS)):
        d, nrm, fg = torch.empty((H, W), device=cuda_device), torch.empty((H, W, 4), device=cuda_device), torch.empty((H, W), dtype=torch.uint8, device=cuda_device)
        req = torch.zeros((400, 400, 3), dtype=torch.uint8, device=cuda_device)
        fe.process_masked([dev(seq.depth_raw[k])], [dev(seq.mask[k])], H, W, seq.K, [d], [nrm], [fg], mode=mode)
        fe.lfnet_request([dev(seq.colour[k])], [fg], H, W, [req])
        out.append(req)
    torch.cuda.synchronize()
    fe.close()
    out.append(dev(np.random.default_rng(7).integers(0, 256, (400, 400, 3), dtype=np.uint8)))
    return out


def _bits(net, reqs):
    import torch
    kp, de, nk = net.detect(reqs)
    torch.cuda.synchronize()
    return nk.cpu().numpy().tobytes(), kp.cpu().numpy().tobytes(), de.cpu().numpy().tobytes()


def test_load_file_equals_tf_variables_bit_for_bit(weights, files, requests):
    a = lfnet.LfnetDevice(weights, HP, max_images=3)
    b = lfnet.LfnetDevice.from_file(files["net"], max_images=3)
    try:
        want = lfnet.params_struct(HP)
        assert all(getattr(want, f) == b.hp[f] for f, _ in want._fields_)
        for reqs in ([requests[0]], [requests[1]], [requests[2]], requests):
            ga, gb = _bits(a, reqs), _bits(b, reqs)
            assert ga == gb, len(reqs)
            assert np.frombuffer(ga[0], np.int32).min() > 0
    finally:
        a.close()
        b.close()


def test_load_file_passes_reserve_and_load_refusals_through(weights, tmp_path, cuda_device):
    lib = _lib.load()
    ctx = _lib.Context(0)
    try:
        blob = lfnet.make_blob(weights, HP)
        # a params block bt_lfnet_weights_size takes but bt_lfnet_reserve refuses
        p = tmp_path / "c32.btlfnet"
        hp32 = dict(HP, net_channel=32)
        n = ctypes.c_size_t(0)
        _lib.check(lib.bt_lfnet_weights_size(ctypes.byref(lfnet.params_struct(hp32)), ctypes.byref(n)))
        p.write_bytes(lfnet.weights_file_bytes(np.zeros(n.value, np.float32), hp32))
        assert lib.bt_lfnet_load_file(ctx, os.fsencode(str(p)), 1, None) == _lib.BT_ERR_INVALID_ARG
        assert lib.bt_last_error().startswith(b"bt_lfnet_reserve: net_channel = 32")
        # max_images out of range
        good = tmp_path / "good.btlfnet"
        good.write_bytes(lfnet.weights_file_bytes(blob, HP))
        assert lib.bt_lfnet_load_file(ctx, os.fsencode(str(good)), 0, None) == _lib.BT_ERR_INVALID_ARG
        assert lib.bt_last_error().startswith(b"bt_lfnet_reserve: max_images 0")
        # a non-finite float
        bad = blob.copy()
        bad[1234] = np.inf
        nf = tmp_path / "inf.btlfnet"
        nf.write_bytes(lfnet.weights_file_bytes(bad, HP))
        assert lib.bt_lfnet_load_file(ctx, os.fsencode(str(nf)), 1, None) == _lib.BT_ERR_INVALID_ARG
        assert lib.bt_last_error() == b"bt_lfnet_load_weights: float 1234 is not finite"
        # a header refusal names the entry point called
        assert lib.bt_lfnet_load_file(ctx, os.fsencode(str(tmp_path / "none")), 1, None) == _lib.BT_ERR_INVALID_ARG
        assert lib.bt_last_error().startswith(b"bt_lfnet_load_file: ")
        # and the context still loads a good file afterwards, reporting its parameters
        got = _lib.LfnetParams()
        _lib.check(lib.bt_lfnet_load_file(ctx, os.fsencode(str(good)), 2, ctypes.byref(got)), "bt_lfnet_load_file")
        assert bytes(got) == bytes(lfnet.params_struct(HP))
    finally:
        ctx.close()


class _Switch:
    """A run_sequence device source that sends the frames in `empty` to a second network."""
    on_device = True

    def __init__(self, net, other, empty):
        self.net, self.other, self.empty = net, other, set(empty)

    def features_on_device(self, id_str, request, roi, stream):
        return (self.other if id_str in self.empty else self.net).features_on_device(id_str, request, roi, stream)


def test_cpp_bundler_with_lfnet_gpu_equals_run_sequence(tmp_path, weights, files, cuda_device):
    """tests/cpp/lfnet_main.cpp: beginFrame -> LfnetGpu::detectFeature -> endFrame over a synthetic video, with a frame that fails the ROI
    gate and two whose detection finds no keypoints (dropFrame).  Statuses and pose files equal run_sequence with LfnetDevice, byte for byte."""
    H, W, N = 240, 320, 10
    seq = synth.make_sequence(31, N, H=H, W=W, roi_fail=(3,))
    video = tmp_path / "video"
    synth.write_ycbineoat_video(seq, str(video))
    loader = sequence.YcbineoatVideo(str(video))
    empty = {f"{k:07d}" for k in (5, 6)}
    net, other = lfnet.LfnetDevice(weights, HP), lfnet.LfnetDevice(weights, HP_EMPTY)
    try:
        res = sequence.run_sequence(loader, None, _Switch(net, other, empty), str(tmp_path / "py"), max_feats=HP["top_k"], device=0)
    finally:
        net.close()
        other.close()
    from bundletrack_b200.tracker import tracker_params
    from bundletrack_b200.config import load_yml
    prm = tracker_params(None, H, W, loader.K, HP["top_k"], int(load_yml(None)["bundle"]["window_size"]) + 4, mode=loader.mask_mode,
                         max_keyframes=min(1024, math.ceil(N / 2)))
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        f.write(np.array([N, H, W, ctypes.sizeof(prm)], np.int32).tobytes() + bytes(prm))
        for i, ff in enumerate(loader.frames):
            d, m, c = sequence.read_frame(ff)
            ident = ff.id_str.encode()
            f.write(np.array([len(ident)], np.int32).tobytes() + ident + np.array([ff.id_str in empty], np.int32).tobytes())
            f.write(np.ascontiguousarray(loader.initial_pose(i), np.float32).tobytes() + d.tobytes() + m.tobytes() + c.tobytes())
    exe = tmp_path / "lfnet_main"
    lib_dir = os.path.join(ROOT, "bundletrack_b200", "lib")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", ROOT, os.path.join(ROOT, "tests", "cpp", "lfnet_main.cpp"), "-o", str(exe),
                           "-L", lib_dir, "-lbundletrack_b200", f"-Wl,-rpath,{lib_dir}"])
    out = tmp_path / "cpp"
    (out / "poses").mkdir(parents=True)
    run = subprocess.run([str(exe), str(inp), str(out), files["net"], files["empty"]], capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stderr
    print(run.stderr)
    statuses = np.fromfile(out / "status.bin", np.int32).tolist()
    assert statuses == [r[1] for r in res]
    want = sorted(os.listdir(tmp_path / "py" / "poses"))
    assert sorted(os.listdir(out / "poses")) == want and len(want) == N
    for name in want:
        assert (out / "poses" / name).read_bytes() == (tmp_path / "py" / "poses" / name).read_bytes(), name
    st = dict((r[0], r[1]) for r in res)
    assert st["0000003"] == _lib.BT_FRAME_FAIL and all(st[e] == _lib.BT_FRAME_FAIL for e in empty)
    assert sum(s == _lib.BT_FRAME_OTHER for s in statuses) >= 4
    print(sequence.summary(res))
