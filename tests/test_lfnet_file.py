"""CPU tests of the LF-Net weights file (lfnet.write_weights_file, bt_lfnet_file_info), of the C++ LfnetGpu building against the library,
and of the feature server's request validation and reply layout."""
import argparse
import ctypes
import os
import pickle
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from bundletrack_b200 import _lib, lfnet, lfnet_server
from oracle import lfnet_oracle as lo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HP = dict(lfnet.DEFAULTS)
HEAD = 8 + 4 + 4 + ctypes.sizeof(_lib.LfnetParams) + 8


def _model_dir(path, hp, seed):
    """A model directory as load_lfnet reads it, with seeded weights."""
    cfg = {k: v for k, v in hp.items() if k != "top_k"}
    cfg.update(lfnet.REQUIRED)
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "config.pkl"), "wb") as f:
        pickle.dump(argparse.Namespace(**cfg), f)
    w = lo.random_weights(lfnet.weight_shapes(hp), seed)
    np.savez(os.path.join(path, "weights.npz"), **w)
    return str(path), w


@pytest.fixture(scope="module")
def written(tmp_path_factory):
    d = tmp_path_factory.mktemp("lfnet")
    model, w = _model_dir(d / "model", HP, 11)
    out = str(d / "net.btlfnet")
    hp = lfnet.write_weights_file(model, out, top_k=HP["top_k"])
    return out, hp, lfnet.make_blob(w, HP)


def _size(hp):
    n = ctypes.c_size_t(0)
    _lib.check(_lib.load().bt_lfnet_weights_size(ctypes.byref(lfnet.params_struct(hp)), ctypes.byref(n)))
    return n.value


def test_file_holds_params_and_blob_byte_for_byte(written):
    path, hp, blob = written
    assert hp == HP
    data = open(path, "rb").read()
    P = ctypes.sizeof(_lib.LfnetParams)
    assert data[:8] == b"BTLFNETW"
    assert np.frombuffer(data[8:16], "<u4").tolist() == [1, P]
    assert data[16:16 + P] == bytes(lfnet.params_struct(HP))
    assert int(np.frombuffer(data[16 + P:HEAD], "<u8")[0]) == blob.size == _size(HP)
    assert data[HEAD:] == blob.tobytes()
    assert len(data) == HEAD + 4 * _size(HP)


def test_file_info_reads_params_and_count_back(written, tmp_path):
    path, _, blob = written
    hp, n = lfnet.file_info(path)
    assert n == blob.size
    want = lfnet.params_struct(HP)
    assert all(getattr(want, f) == hp[f] for f, _ in want._fields_)
    # other numeric parameters: another blob size, read back the same way
    hp2 = dict(HP, top_k=64, net_block=2, net_num_scales=3, desc_dim=128)
    model, _ = _model_dir(tmp_path / "m2", hp2, 3)
    lfnet.write_weights_file(model, str(tmp_path / "m2.btlfnet"), top_k=64)
    got, n2 = lfnet.file_info(str(tmp_path / "m2.btlfnet"))
    assert n2 == _size(hp2) != n and got["top_k"] == 64 and got["desc_dim"] == 128 and got["net_block"] == 2
    # the outputs are optional
    assert _lib.load().bt_lfnet_file_info(os.fsencode(path), None, None) == _lib.BT_OK


def _corrupt(data: bytes, kind: str) -> bytes:
    P = ctypes.sizeof(_lib.LfnetParams)
    b = bytearray(data)
    if kind == "magic":
        b[0:8] = b"BTLFNETX"
    elif kind == "version":
        b[8:12] = np.array([2], "<u4").tobytes()
    elif kind == "struct size":
        b[12:16] = np.array([P - 8], "<u4").tobytes()
    elif kind == "truncated blob":
        del b[-4:]
    elif kind == "truncated header":
        del b[20:]
    elif kind == "count":
        b[16 + P:HEAD] = np.array([12345], "<u8").tobytes()
    elif kind == "trailing":
        b += b"\0\0\0\0"
    elif kind == "params":
        p = lfnet.params_struct(dict(HP, net_block=99))
        b[16:16 + P] = bytes(p)
    return bytes(b)


@pytest.mark.parametrize("kind,message", [("magic", "bad magic"), ("version", "format version 2"), ("struct size", "struct size of"),
                                          ("truncated blob", "truncated"), ("truncated header", "truncated"), ("count", "float count of 12345"),
                                          ("trailing", "4 more than"), ("params", "out of range")])
def test_file_info_refuses_each_corruption_naming_it(written, tmp_path, kind, message):
    bad = tmp_path / "bad.btlfnet"
    bad.write_bytes(_corrupt(open(written[0], "rb").read(), kind))
    lib = _lib.load()
    assert lib.bt_lfnet_file_info(os.fsencode(str(bad)), None, None) == _lib.BT_ERR_INVALID_ARG
    msg = lib.bt_last_error().decode()
    assert message in msg and str(bad) in msg and msg.startswith("bt_lfnet_file_info: "), msg
    with pytest.raises(_lib.BtError, match=message):
        lfnet.file_info(str(bad))


def test_file_info_refuses_missing_file_and_null_path(tmp_path):
    lib = _lib.load()
    assert lib.bt_lfnet_file_info(os.fsencode(str(tmp_path / "none")), None, None) == _lib.BT_ERR_INVALID_ARG
    assert b"cannot open" in lib.bt_last_error()
    assert lib.bt_lfnet_file_info(None, None, None) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_lfnet_load_file(None, os.fsencode(str(tmp_path / "none")), 1, None) == _lib.BT_ERR_INVALID_ARG
    assert b"ctx is NULL" in lib.bt_last_error()


def test_export_script_writes_the_same_file(written, tmp_path):
    model, _ = _model_dir(tmp_path / "model", HP, 11)
    out = tmp_path / "script.btlfnet"
    run = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "lfnet_export_blob.py"), "--model", model, "--out", str(out)],
                         capture_output=True, text=True, timeout=300)
    assert run.returncode == 0, run.stderr
    assert out.read_bytes() == open(written[0], "rb").read()


def test_cpp_lfnet_gpu_compiles_and_links(tmp_path):
    src = tmp_path / "lfnet_shim.cpp"
    src.write_text(textwrap.dedent(r'''
        #include "bundletrack_b200/hostcpp/bt_optimizer.hpp"
        #include <cstdio>
        struct KeyPoint { struct { float x, y; } pt; float size; };
        int main(int argc, char** argv) {
            try {
                LfnetGpu net(argv[1], 2);              // throws without a GPU: the product has no CPU fallback
                std::vector<KeyPoint> k; bt_desc_view d{}; const int32_t roi[4] = {0, 100, 0, 100};
                net.detectFeature((const uint8_t*)nullptr, roi, k, d);
                std::vector<std::vector<KeyPoint>> ks; std::vector<bt_desc_view> ds; const uint8_t* rq[2] = {nullptr, nullptr}; const int32_t* rr[2] = {roi, roi};
                net.detectFeatures(2, rq, rr, ks, ds);
            } catch (const std::exception& e) { std::printf("caught: %s\n", e.what()); return 0; }
            return 0;
        }
    '''))
    exe = tmp_path / "lfnet_shim"
    lib_dir = os.path.join(ROOT, "bundletrack_b200", "lib")
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-I", ROOT, str(src), "-o", str(exe), "-L", lib_dir, "-lbundletrack_b200", f"-Wl,-rpath,{lib_dir}"])
    out = subprocess.run([str(exe), str(tmp_path / "missing.btlfnet")], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and "caught:" in out.stdout, out.stderr


# ---- the server's request validation --------------------------------------------------------------------------------------------------

def _wh(w, h):
    return np.array([w, h], np.int32).tobytes()


GOOD_IMAGE = np.random.default_rng(2).integers(0, 256, (400, 400, 3), dtype=np.uint8)


@pytest.mark.parametrize("body", [
    [],                                                             # no parts
    [_wh(400, 400)],                                                # one part
    [_wh(400, 400), GOOD_IMAGE.tobytes(), b"x"],                    # three parts
    [_wh(320, 240), np.zeros(320 * 240 * 3, np.uint8).tobytes()],   # another size, consistent payload
    [_wh(400, 401), GOOD_IMAGE.tobytes()],                          # wrong H
    [_wh(401, 400), GOOD_IMAGE.tobytes()],                          # wrong W
    [_wh(400, 400), GOOD_IMAGE.tobytes()[:-1]],                     # short payload
    [_wh(400, 400), GOOD_IMAGE.tobytes() + b"\0"],                  # long payload
    [_wh(400, 400)[:4], GOOD_IMAGE.tobytes()],                      # short size part
    [_wh(400, 400) + b"\0\0\0\0", GOOD_IMAGE.tobytes()],            # long size part
    [_wh(400, 400), GOOD_IMAGE[..., 0].tobytes()],                  # one channel
])
def test_malformed_requests_get_an_empty_reply(body):
    assert lfnet_server.request_image(body) is None
    info, kp, de = lfnet_server.empty_reply(256)
    assert np.frombuffer(info, np.int32).tolist() == [0, 256] and kp == b"" and de == b""


def test_good_request_and_reply_layout():
    img = lfnet_server.request_image([_wh(400, 400), GOOD_IMAGE.tobytes()])
    assert img.shape == (400, 400, 3) and img.dtype == np.uint8 and np.array_equal(img, GOOD_IMAGE)
    rng = np.random.default_rng(4)
    k, d = rng.uniform(0, 400, (37, 2)).astype(np.float32), rng.normal(size=(37, 256)).astype(np.float32)
    parts = lfnet_server.reply_parts(k, d)
    # run_server.py:170-177: int32 (n, dim), float32 n x 2, float32 n x dim
    assert parts == [np.array([37, 256], np.int32).tobytes(), k.tobytes(), d.tobytes()]
    from bundletrack_b200 import policy
    kp, de = policy.lfnet_parse_reply(parts, (100, 260, 80, 300))
    assert kp.shape == (37, 2) and np.array_equal(de, d)


def test_envelope_split():
    assert lfnet_server.split_envelope([b"id", b"", b"a", b"b"]) == ([b"id", b""], [b"a", b"b"])
    assert lfnet_server.split_envelope([b"id", b"p1", b"", b"a"]) == ([b"id", b"p1", b""], [b"a"])
    assert lfnet_server.split_envelope([b"id", b"a", b"b"]) == ([b"id"], [b"a", b"b"])
