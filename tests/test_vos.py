"""CPU tests of the object-mask propagation's host side: the reference-frame schedule, the checkpoint reader and its refusals, the blob
size, the params struct, and the label compression argument of oracle/vos_oracle.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from bundletrack_b200 import _lib, vos
from oracle import vos_oracle as vo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _numpy_schedule(k, ref_num, rng):
    if k <= ref_num:
        return list(range(k))
    end = k - 4
    return np.linspace(max(end - rng, 0), end, ref_num - 3).astype(int).tolist() + [k - 3, k - 2, k - 1]


@pytest.mark.parametrize("ref_num,rng", [(9, 40), (5, 40), (9, 3), (9, 0), (12, 7), (20, 100), (64, 5)])
def test_schedule_equals_numpy_linspace(ref_num, rng):
    lib = _lib.load()
    buf = (ctypes.c_int32 * 3001)()
    n = ctypes.c_int(0)
    dup = False
    for k in range(1, 3001):
        _lib.check(lib.bt_vos_schedule(k, ref_num, rng, buf, ctypes.byref(n)))
        want = _numpy_schedule(k, ref_num, rng)
        assert list(buf[:n.value]) == want, k
        dup |= len(set(want)) < len(want)
    if rng < ref_num - 4:
        assert dup            # the small ranges do produce duplicates, and they are kept
    assert vos.schedule(100, 9, 40) == _numpy_schedule(100, 9, 40)


def test_schedule_refusals():
    lib = _lib.load()
    buf = (ctypes.c_int32 * 100)()
    n = ctypes.c_int(0)
    assert lib.bt_vos_schedule(0, 9, 40, buf, ctypes.byref(n)) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_vos_schedule(5, 4, 40, buf, ctypes.byref(n)) == _lib.BT_ERR_INVALID_ARG


def _save(tmp_path, sd, name="ck.pth.tar"):
    """As main.py saves a checkpoint."""
    p = tmp_path / name
    torch.save({"epoch": 3, "state_dict": sd, "optimizer": {"state": {}, "param_groups": []}, "scheduler": {"last_epoch": 3}}, p)
    return str(p)


@pytest.fixture(scope="module")
def state():
    return vo.random_state_dict(5)


def test_read_checkpoint_maps_every_tensor(tmp_path, state):
    sd = vos.read_checkpoint(_save(tmp_path, state))
    assert set(sd) == set(vos.state_shapes())
    for k, v in sd.items():
        np.testing.assert_array_equal(v, state["module." + k].double().numpy())
    # without the DataParallel prefix too
    sd2 = vos.read_checkpoint(_save(tmp_path, {k[len("module."):]: v for k, v in state.items()}, "bare.pth.tar"))
    assert all(np.array_equal(sd[k], sd2[k]) for k in sd)


def test_read_checkpoint_refusals_name_the_key(tmp_path, state):
    miss = dict(state)
    del miss["module.backbone.5.2.bn2.running_var"]
    with pytest.raises(ValueError, match=r"backbone\.5\.2\.bn2\.running_var.*missing"):
        vos.read_checkpoint(_save(tmp_path, miss, "a"))
    extra = dict(state)
    extra["module.classifier.weight"] = torch.zeros(3)
    with pytest.raises(ValueError, match=r"unexpected key 'classifier\.weight'"):
        vos.read_checkpoint(_save(tmp_path, extra, "b"))
    shape = dict(state)
    shape["module.adjust_dim.weight"] = torch.zeros(128, 1024, 1, 1)
    with pytest.raises(ValueError, match=r"adjust_dim\.weight.*\(128, 1024, 1, 1\)"):
        vos.read_checkpoint(_save(tmp_path, shape, "c"))


def test_read_checkpoint_refuses_other_resnets_by_name(tmp_path, state):
    r18 = {k: v for k, v in state.items() if not k.startswith("module.backbone.")}
    g = torch.Generator().manual_seed(1)
    r18["module.backbone.0.weight"] = state["module.backbone.0.weight"]
    for L, planes in enumerate((64, 128, 256, 256)):
        for b in range(2):
            r18[f"module.backbone.{4 + L}.{b}.conv1.weight"] = torch.randn(planes, planes, 3, 3, generator=g)
            r18[f"module.backbone.{4 + L}.{b}.conv2.weight"] = torch.randn(planes, planes, 3, 3, generator=g)
    with pytest.raises(ValueError, match="resnet18"):
        vos.read_checkpoint(_save(tmp_path, r18, "r18"))
    r101 = dict(state)
    r101["module.backbone.6.6.conv1.weight"] = torch.zeros(256, 1024, 1, 1)
    with pytest.raises(ValueError, match="resnet101"):
        vos.read_checkpoint(_save(tmp_path, r101, "r101"))


def test_blob_size_matches_the_library(state):
    sd = {k[len("module."):]: v.double().numpy() for k, v in state.items() if not k.endswith("num_batches_tracked")}
    blob = vos.make_blob(sd)
    n = ctypes.c_size_t(0)
    _lib.check(_lib.load().bt_vos_weights_size(ctypes.byref(vos.params_struct(vos.DEFAULTS)), ctypes.byref(n)))
    assert blob.size == n.value == sum(int(np.prod(s)) for k, s in vos.state_shapes().items()
                                       if k.endswith(".weight") and len(s) == 4) + 2 * sum(s[0] for k, s in vos.state_shapes().items()
                                                                                          if k.endswith(".weight") and len(s) == 4)
    # the first conv in [co][ky][kx][ci], then its folded BN
    w = sd["backbone.0.weight"]
    np.testing.assert_array_equal(blob[:w.size], np.transpose(w, (0, 2, 3, 1)).reshape(-1).astype(np.float32))
    s = sd["backbone.1.weight"] / np.sqrt(sd["backbone.1.running_var"] + 1e-5)
    np.testing.assert_array_equal(blob[w.size:w.size + 64], s.astype(np.float32))


def test_params_struct_matches_the_c_header(tmp_path):
    cls = _lib.VosParams
    exprs = ["sizeof(bt_vos_params)"] + [f"offsetof(bt_vos_params, {f})" for f, _ in cls._fields_]
    want = [ctypes.sizeof(cls)] + [getattr(cls, f).offset for f, _ in cls._fields_]
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "bundletrack_b200.h"\nint main(){\n'
                   + "".join(f'printf("%zu\\n", (size_t){e});\n' for e in exprs) + "return 0;}\n")
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == want


@pytest.mark.parametrize("values", [(0, 3, 7), (5, 9), (0,), (2, 200, 17, 4), (0, 255)])
def test_label_compression_changes_no_argmax(values):
    """Predictions built from one-hot labels in the reference's d = max + 1 channels and in the compressed channels give the same
    argmax, once mapped back: empty channels predict exactly 0, present channels keep their order, and an all-zero pixel resolves to
    channel 0 either way."""
    rng = np.random.default_rng(len(values))
    mask = rng.choice(np.array(values, np.uint8), size=(6, 7))
    comp, d = vo.compress_labels(mask)
    full = int(mask.max()) + 1
    order = sorted(set(int(v) for v in np.unique(mask)) - {0})
    assert d == len(order) + 1
    for trial in range(20):
        w = rng.random((mask.size, mask.size)) * (rng.random((mask.size, mask.size)) < 0.5)   # some target pixels see no weight
        w[:, trial] = 0
        p_full = np.eye(full)[mask.reshape(-1)].T @ w
        p_comp = np.eye(d)[comp.reshape(-1)].T @ w
        back = np.array([0] + order)[np.argmax(p_comp, 0)]
        assert np.array_equal(np.argmax(p_full, 0), back)
        assert (np.argmax(p_full, 0)[trial] == 0) and (back[trial] == 0)
