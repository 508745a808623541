"""C-ABI surface: the in-tree .so loads (no GPU needed for that) and exports exactly what include/*.h declares."""
import ctypes
import os
import re

import pytest

from bundletrack_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    hdr = open(os.path.join(ROOT, "include", "bundletrack_b200.h")).read()
    return sorted(set(re.findall(r"^BT_API\s+[\w\s\*]+?\b(bt_\w+)\s*\(", hdr, flags=re.M)))


def test_header_and_binding_agree():
    assert _declared() == sorted(_lib.EXPORTS)


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    for name in _declared():
        assert hasattr(lib, name), name


def test_struct_layouts_match_reference_types():
    # EntryJ is 32 bytes (/root/reference/src/cuda/SIFTImageManager.h:44-59); params are 10 x 4 bytes
    from bundletrack_b200.synth import ENTRYJ_DTYPE
    assert ENTRYJ_DTYPE.itemsize == 32
    assert ctypes.sizeof(_lib.SolverParams) == 40
    assert ENTRYJ_DTYPE.fields["pos_i"][1] == 8 and ENTRYJ_DTYPE.fields["pos_j"][1] == 20


def test_ctypes_structs_match_the_c_header(tmp_path):
    """sizeof of every struct the Python mirror passes by pointer, measured by compiling the C header with gcc."""
    import os, subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include "bundletrack_b200.h"\nint main(){printf("%zu %zu %zu %zu %zu\\n", sizeof(bt_window), sizeof(bt_depth_params), '
                   'sizeof(bt_solver_params), sizeof(bt_solver_limits), sizeof(bt_entryj));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [ctypes.sizeof(_lib.Window), ctypes.sizeof(_lib.DepthParams), ctypes.sizeof(_lib.SolverParams), ctypes.sizeof(_lib.SolverLimits), 32]


def test_no_gpu_fails_loudly():
    """Without a CUDA device the library must refuse (BT_ERR_NO_DEVICE), never fall back to a CPU path."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = _lib.load()
    ctx = ctypes.c_void_p()
    rc = lib.bt_ctx_create(ctypes.byref(ctx), 0)
    assert rc == -4
    assert b"no CPU fallback" in lib.bt_last_error()
    from bundletrack_b200.optimizer import OptimizerGpu
    with pytest.raises(_lib.BtError):
        OptimizerGpu(None)


def test_live_resource_counts_need_no_device():
    """bt_debug_live_resources reads counters the handle types keep: it answers without a GPU and refuses NULL outputs."""
    lib = _lib.load()
    d, p, h = ctypes.c_longlong(-1), ctypes.c_longlong(-1), ctypes.c_int(-1)
    assert lib.bt_debug_live_resources(ctypes.byref(d), ctypes.byref(p), ctypes.byref(h)) == 0
    assert d.value >= 0 and p.value >= 0 and h.value >= 0
    assert lib.bt_debug_live_resources(None, ctypes.byref(p), ctypes.byref(h)) == -1


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "bundletrack_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp", ".hpp")):
                txt = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(import|from)\s+oracle\b", txt, flags=re.M), f
                assert "liboracle" not in txt and "libbt_ref" not in txt, f
