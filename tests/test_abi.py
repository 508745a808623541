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


# the header's structs the binding mirrors, and the ctypes Structure that mirrors each
MIRRORED = {"bt_solver_params": _lib.SolverParams, "bt_window": _lib.Window, "bt_solver_limits": _lib.SolverLimits, "bt_solve_stats": _lib.SolveStats,
            "bt_desc_view": _lib.DescView, "bt_match_frame": _lib.MatchFrame, "bt_prune_params": _lib.PruneParams, "bt_match_extra": _lib.MatchExtra,
            "bt_depth_params": _lib.DepthParams, "bt_tracker_params": _lib.TrackerParams, "bt_match_viz_desc": _lib.MatchVizDesc}
SCALARS = {"int": ctypes.c_int, "int32_t": ctypes.c_int, "float": ctypes.c_float, "double": ctypes.c_double, "long long": ctypes.c_longlong,
           "size_t": ctypes.c_size_t, "uint64_t": ctypes.c_uint64}


def _c_type(decl: str, result: bool = False):
    """The ctypes type a C parameter or return type maps to: scalars by SCALARS, a pointer to a mirrored struct as POINTER(<Structure>),
    any other pointer or handle as c_void_p (a returned string as c_char_p)."""
    words = re.sub(r"\bconst\b", " ", decl).replace("*", " * ").split()
    stars, base = words.count("*"), " ".join(w for w in words if w != "*")
    if stars == 0:
        return None if base == "void" else SCALARS[base]
    if result and stars == 1 and base == "char":
        return ctypes.c_char_p
    return ctypes.POINTER(MIRRORED[base]) if stars == 1 and base in MIRRORED else ctypes.c_void_p


def _prototypes():
    """{name: (return type, [(parameter type, parameter name)])} of every BT_API prototype in the header."""
    hdr = re.sub(r"/\*.*?\*/", " ", open(os.path.join(ROOT, "include", "bundletrack_b200.h")).read(), flags=re.S)
    out = {}
    for ret, name, params in re.findall(r"^BT_API\s+([\w\s\*]+?)\b(bt_\w+)\s*\(([^)]*)\)\s*;", hdr, flags=re.M):
        ps = [p.strip() for p in params.split(",")]
        ps = [] if ps == ["void"] else ps
        out[name] = (ret, [(p[:len(p) - len(re.search(r"\w+$", p).group())], re.search(r"\w+$", p).group()) for p in ps])
    return out


def test_prototype_table_matches_the_header():
    """Every entry point's restype and argtypes, arity included, as the header declares it: a call site can pass plain Python values."""
    want = {name: (_c_type(ret, result=True), [_c_type(t) for t, _ in params]) for name, (ret, params) in _prototypes().items()}
    got = {name: (restype, list(argtypes)) for name, (restype, argtypes) in _lib.PROTOTYPES.items()}
    assert sorted(got) == sorted(want)
    for name in want:
        assert got[name] == want[name], name
    lib = _lib.load()
    for name, (restype, argtypes) in _lib.PROTOTYPES.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and list(fn.argtypes) == list(argtypes), name


def test_ctypes_structs_match_the_c_header(tmp_path):
    """sizeof and every field's offsetof of each struct the binding mirrors, measured by compiling the C header with gcc."""
    import subprocess
    exprs, want = ["sizeof(bt_entryj)"], [32]
    for cname, cls in MIRRORED.items():
        exprs.append(f"sizeof({cname})")
        want.append(ctypes.sizeof(cls))
        for field, _ in cls._fields_:
            exprs.append(f"offsetof({cname}, {field})")
            want.append(getattr(cls, field).offset)
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "bundletrack_b200.h"\nint main(){\n'
                   + "".join(f'printf("%zu\\n", (size_t){e});\n' for e in exprs) + "return 0;}\n")
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert dict(zip(exprs, got)) == dict(zip(exprs, want))


def test_null_handles_are_refused():
    """Every entry point on a bt_ctx, bt_tracker or bt_tracks refuses a NULL handle with BT_ERR_INVALID_ARG (zeros and NULL for the other
    arguments); destroying NULL does nothing.  A Handle a holder closed is NULL for every holder, so this is what a late call meets."""
    lib = _lib.load()
    seen = set()
    for name, (ret, params) in _prototypes().items():
        first = re.sub(r"\bconst\b", "", params[0][0]).replace(" ", "") if params else ""
        if first not in ("bt_ctx*", "bt_tracker*", "bt_tracks*"):
            continue
        args = [0 if t in SCALARS.values() else None for t in _lib.PROTOTYPES[name][1]]
        rc = getattr(lib, name)(*args)
        if name.endswith("_destroy"):
            assert rc is None, name
        else:
            assert rc == _lib.BT_ERR_INVALID_ARG, (name, rc, lib.bt_last_error())
        seen.add(first)
    assert seen == {"bt_ctx*", "bt_tracker*", "bt_tracks*"}


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
