"""CPU tests of LF-Net on the device: the oracle's grey conversion against OpenCV, its resize and padding against hand-worked cases, the
loader's refusals, the weight blob's size and the C-ABI of bt_lfnet_params."""
import argparse
import ctypes
import os
import pickle
import subprocess

import numpy as np
import pytest

from bundletrack_b200 import _lib, lfnet
from oracle import lfnet_oracle as lo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _requests():
    rng = np.random.default_rng(5)
    rnd = rng.integers(0, 256, (400, 400, 3), dtype=np.uint8)
    masked = rnd.copy()
    yy, xx = np.mgrid[0:400, 0:400]
    masked[(xx - 180) ** 2 + (yy - 220) ** 2 > 120 ** 2] = 0
    extremes = np.array([[[0, 0, 0], [255, 255, 255], [255, 0, 0], [0, 255, 0], [0, 0, 255], [1, 2, 3]]], np.uint8)
    return [rnd, masked, extremes]


def test_grey_equals_opencv_rgb2gray():
    """run_server.py converts the BGR request with COLOR_RGB2GRAY: the oracle's fixed point equals OpenCV byte for byte."""
    cv2 = pytest.importorskip("cv2")
    for req in _requests():
        assert np.array_equal(lo.grey(req), cv2.cvtColor(req, cv2.COLOR_RGB2GRAY))


def test_resize_hand_worked():
    """TF1 bilinear without half-pixel centres: src = dst * in / out, the upper neighbour clipped to the last row."""
    x = np.array([[0.0, 10.0], [20.0, 30.0]])[..., None]
    up = lo.resize_bilinear(x, 4, 4)[..., 0]
    # src = 0, 0.5, 1, 1.5 -> rows and columns 0, 0|1 halfway, 1, 1 (clipped)
    assert np.allclose(up, [[0, 5, 10, 10], [10, 15, 20, 20], [20, 25, 30, 30], [20, 25, 30, 30]])
    down = lo.resize_bilinear(np.arange(25.0).reshape(5, 5, 1), 2, 2)[..., 0]
    # src = 0, 2.5: rows 0 and halfway between rows 2 and 3
    assert np.allclose(down, [[0, 2.5], [12.5, 15.0]])
    assert lo.scale_sizes(lfnet.DEFAULTS) == [283, 336, 400, 476, 566]


def test_same_padding_hand_worked():
    """simple_desc's stride-2 SAME convs: a 32-wide input pads 0 before and 1 after (3 x 3), so output (0, 0) sees input rows 0..2."""
    assert lo.same_pads(32, 3, 2) == (16, 0, 1)
    assert lo.same_pads(16, 3, 2) == (8, 0, 1)
    assert lo.same_pads(400, 5, 1) == (400, 2, 2)
    x = np.arange(16.0).reshape(1, 4, 4, 1)
    W = np.ones((3, 3, 1, 1))
    y = lo.conv2d(x, W, stride=2)[0, ..., 0]
    assert np.allclose(y, [[x[0, 0:3, 0:3].sum(), x[0, 0:3, 2:4].sum()], [x[0, 2:4, 0:3].sum(), x[0, 2:4, 2:4].sum()]])


def _cfg(**kw):
    c = dict(lfnet.DEFAULTS)
    c.pop("top_k")
    c.update(lfnet.REQUIRED)
    c.update(kw)
    return c


def _model_dir(tmp_path, cfg, weights):
    with open(tmp_path / "config.pkl", "wb") as f:
        pickle.dump(argparse.Namespace(**cfg), f)
    np.savez(tmp_path / "weights.npz", **weights)
    return str(tmp_path)


def test_config_defaults_pass_and_top_k_comes_from_the_server():
    hp = lfnet.check_config(_cfg(top_k=512), top_k=500)
    assert hp == dict(lfnet.DEFAULTS)
    # train_lfnet.py's scale defaults are numpy floats: they survive the restricted unpickler
    cfg = _cfg(net_min_scale=np.float64(1 / np.sqrt(2)), net_max_scale=np.sqrt(2))
    blob = pickle.dumps(argparse.Namespace(**cfg))
    import io
    assert lfnet._ConfigUnpickler(io.BytesIO(blob)).load().net_max_scale == np.sqrt(2)


@pytest.mark.parametrize("key,value", [("detector", "resnet_detector"), ("descriptor", "other_desc"), ("desc_inputs", "det_feats"),
                                       ("desc_norm", "rootsift"), ("use_nms3d", False), ("soft_kpts", False), ("perform_bn", False),
                                       ("activ_fn", "relu")])
def test_config_refusals_name_the_key(key, value):
    with pytest.raises(ValueError, match=repr(key)):
        lfnet.check_config(_cfg(**{key: value}))


def test_config_missing_key_is_named():
    c = _cfg()
    del c["sm_ksize"]
    with pytest.raises(ValueError, match="'sm_ksize'"):
        lfnet.check_config(c)


def test_weight_refusals_name_the_variable():
    hp = dict(lfnet.DEFAULTS)
    w = lo.random_weights(lfnet.weight_shapes(hp), 0)
    assert lfnet.make_blob(w, hp).dtype == np.float32
    missing = dict(w)
    del missing["SimpleDesc/bn2/moving_mean"]
    with pytest.raises(ValueError, match="SimpleDesc/bn2/moving_mean"):
        lfnet.make_blob(missing, hp)
    bad = dict(w)
    bad["ConvOnlyResNet/ori_conv/weights"] = np.zeros((3, 3, 16, 2), np.float32)
    with pytest.raises(ValueError, match="ConvOnlyResNet/ori_conv/weights"):
        lfnet.make_blob(bad, hp)


def test_restricted_unpickler_refuses_other_classes(tmp_path):
    import collections
    with open(tmp_path / "config.pkl", "wb") as f:
        pickle.dump(argparse.Namespace(detector=collections.OrderedDict(a=1)), f)
    with pytest.raises(pickle.UnpicklingError, match="collections.OrderedDict"):
        lfnet.read_config(str(tmp_path / "config.pkl"))


def test_load_lfnet_refuses_before_touching_the_device(tmp_path):
    """A wrong config is refused by load_lfnet itself, naming the key; no GPU is needed to get there."""
    d = _model_dir(tmp_path, _cfg(desc_inputs="concat"), {})
    with pytest.raises(ValueError, match="'desc_inputs'"):
        lfnet.load_lfnet(d)


def test_blob_size_matches_the_library():
    """bt_lfnet_weights_size (host code) and the Python layout agree, at the defaults and at other numeric parameters."""
    lib = _lib.load()
    for kw in ({}, dict(net_block=2, net_num_scales=3, desc_net_channel=32, desc_net_depth=2, desc_dim=128, patch_size=24)):
        hp = dict(lfnet.DEFAULTS, **kw)
        n = ctypes.c_size_t(0)
        _lib.check(lib.bt_lfnet_weights_size(ctypes.byref(lfnet.params_struct(hp)), ctypes.byref(n)))
        assert n.value == lfnet.make_blob(lo.random_weights(lfnet.weight_shapes(hp), 1), hp).size
    assert lib.bt_lfnet_weights_size(None, None) == _lib.BT_ERR_INVALID_ARG


def test_params_struct_matches_the_c_header(tmp_path):
    cls = _lib.LfnetParams
    exprs = ["sizeof(bt_lfnet_params)"] + [f"offsetof(bt_lfnet_params, {f})" for f, _ in cls._fields_]
    want = [ctypes.sizeof(cls)] + [getattr(cls, f).offset for f, _ in cls._fields_]
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "bundletrack_b200.h"\nint main(){\n'
                   + "".join(f'printf("%zu\\n", (size_t){e});\n' for e in exprs) + "return 0;}\n")
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == want
