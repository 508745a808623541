"""oracle/ — TEST INFRASTRUCTURE ONLY (CPU restatement of the reference hot path + the recipe that compiles the
reference's own CUDA kernels into oracle/_ref).  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
`--impl reference` legs may import this package.  bundletrack_b200/ never does.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))


class OracleParams(ctypes.Structure):
    _fields_ = [
        ("num_iter_outer", ctypes.c_int),
        ("num_iter_inner", ctypes.c_int),
        ("robust_delta", ctypes.c_float),
        ("image_downscale", ctypes.c_float),
        ("dense_dist_thresh", ctypes.c_float),
        ("dense_cos_normal_thresh", ctypes.c_float),
        ("depth_min", ctypes.c_float),
        ("depth_max", ctypes.c_float),
        ("w_sparse", ctypes.c_float),
        ("w_dense", ctypes.c_float),
    ]


def default_params(**kw) -> OracleParams:
    """Values of config_nocs.yml (bundle.*, p2p.*) + the constants hard-wired in CUDASolverBundling.cpp:92-99."""
    p = OracleParams(7, 5, 0.005, 4.0, 0.02, float(np.cos(np.deg2rad(45.0))), 0.1, 9999.0, 1.0, 1.0)
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def build(force: bool = False) -> None:
    """Compile the C restatement (gcc) — building the checker is not using it."""
    src = os.path.join(_HERE, "solver_oracle.c")
    for name, extra in (("liboracle_f32.so", []), ("liboracle_f64.so", ["-DORACLE_REAL=double"])):
        out = os.path.join(_HERE, name)
        if force or not os.path.exists(out) or os.path.getmtime(out) < os.path.getmtime(src):
            subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", *extra, "-o", out, src, "-lm"])
    src = os.path.join(_HERE, "matcher_oracle.c")
    if os.path.exists(src):
        out = os.path.join(_HERE, "liboracle_match.so")
        if force or not os.path.exists(out) or os.path.getmtime(out) < os.path.getmtime(src):
            subprocess.check_call(["gcc", "-O3", "-march=native", "-fopenmp", "-fPIC", "-shared", "-ffp-contract=off", "-o", out, src, "-lm"])


_libs = {}


def _lib(precision: str):
    if precision not in _libs:
        build()
        lib = ctypes.CDLL(os.path.join(_HERE, f"liboracle_{precision}.so"))
        lib.oracle_solve_window.restype = ctypes.c_int
        lib.oracle_dense_system.restype = ctypes.c_int
        lib.oracle_build_cache.restype = ctypes.c_int
        _libs[precision] = lib
    return _libs[precision]


def _fp(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def default_pairs(n_frames: int) -> np.ndarray:
    """(target, source) list with target = the larger index: what FindImageImageCorr_Kernel yields when the
    CUDACachedFrame::d_num_valid_points allocations have ascending addresses (SURVEY.md Q1)."""
    return np.array([(i, j) for i in range(n_frames) for j in range(i)], dtype=np.uint32).reshape(-1, 2)


def solve_window(depth, normal, K, corr, poses, pairs=None, params=None, precision="f32", want_debug=False):
    """Run Oracle A on one window.  Returns new poses [N,4,4] float32 (and the iter-0 dense system if asked)."""
    lib = _lib(precision)
    depth = np.ascontiguousarray(depth, np.float32)
    normal = np.ascontiguousarray(normal, np.float32)
    N, H, W = depth.shape
    corr = np.ascontiguousarray(corr)
    poses = np.ascontiguousarray(poses, np.float32).copy()
    if pairs is None:
        pairs = default_pairs(N)
    pairs = np.ascontiguousarray(pairs, np.uint32)
    params = params or default_params()
    dim = 6 * N
    JtJ = np.zeros((dim, dim), np.float64)
    Jtr = np.zeros(dim, np.float64)
    rc = lib.oracle_solve_window(
        ctypes.c_int(N), ctypes.c_int(H), ctypes.c_int(W), _fp(depth), _fp(normal),
        ctypes.c_float(K[0]), ctypes.c_float(K[1]), ctypes.c_float(K[2]), ctypes.c_float(K[3]),
        ctypes.c_int(len(corr)), _fp(corr), _fp(pairs), ctypes.c_int(len(pairs)),
        ctypes.byref(params), _fp(poses), _fp(JtJ) if want_debug else None, _fp(Jtr) if want_debug else None)
    if rc != 0:
        raise RuntimeError(f"oracle_solve_window rc={rc}")
    return (poses, JtJ, Jtr) if want_debug else poses


def dense_system(depth, normal, K, poses, pairs=None, params=None, precision="f32"):
    lib = _lib(precision)
    depth = np.ascontiguousarray(depth, np.float32)
    normal = np.ascontiguousarray(normal, np.float32)
    N, H, W = depth.shape
    poses = np.ascontiguousarray(poses, np.float32)
    if pairs is None:
        pairs = default_pairs(N)
    pairs = np.ascontiguousarray(pairs, np.uint32)
    params = params or default_params()
    dim = 6 * N
    JtJ = np.zeros((dim, dim), np.float64)
    Jtr = np.zeros(dim, np.float64)
    nfound = np.zeros(len(pairs), np.int32)
    rc = lib.oracle_dense_system(
        ctypes.c_int(N), ctypes.c_int(H), ctypes.c_int(W), _fp(depth), _fp(normal),
        ctypes.c_float(K[0]), ctypes.c_float(K[1]), ctypes.c_float(K[2]), ctypes.c_float(K[3]),
        _fp(pairs), ctypes.c_int(len(pairs)), ctypes.byref(params), _fp(poses), _fp(JtJ), _fp(Jtr), _fp(nfound))
    if rc != 0:
        raise RuntimeError(f"oracle_dense_system rc={rc}")
    return JtJ, Jtr, nfound


# A gate decision counts as MARGINAL when the pixel's gate quantity lies within this relative distance of the boundary (see
# `dense_extra` in solver_oracle.c for what each distance is divided by).  A float32 implementation evaluates the transform chain
# (pose round trip, 3x4 transform, projection, bilinear blend, distance and cosine) in roughly 30 dependent operations, each rounded
# to 2^-24 relative to the magnitude the distance is scaled by; 64 * 2^-24 = 3.8e-6 covers twice that chain, so a pixel with a larger
# margin is decided the same way by any correctly rounded float32 evaluation and by this float64 one.
MARGIN_EPS = 64.0 * 2.0 ** -24


def dense_system_ex(depth, normal, K, poses, pairs=None, params=None, precision="f64", flip=True):
    """oracle_dense_system with everything a per-entry comparison needs.  Returns a dict: JtJ, Jtr (FlipJtJ applied when flip, else
    the raw addToLocalSystem sums), JtJ_abs / Jtr_abs (the same sums over |term|), n_found [P], and per (pair, quarter-res source
    pixel) margin / accepted / contrib ([P, h*w]; see dense_extra in solver_oracle.c)."""
    lib = _lib(precision)
    depth = np.ascontiguousarray(depth, np.float32)
    normal = np.ascontiguousarray(normal, np.float32)
    N, H, W = depth.shape
    poses = np.ascontiguousarray(poses, np.float32)
    pairs = np.ascontiguousarray(default_pairs(N) if pairs is None else pairs, np.uint32).reshape(-1, 2)
    params = params or default_params()
    dim, P = 6 * N, len(pairs)
    npix = int(W / params.image_downscale) * int(H / params.image_downscale)
    out = dict(JtJ=np.zeros((dim, dim)), Jtr=np.zeros(dim), n_found=np.zeros(P, np.int32), JtJ_abs=np.zeros((dim, dim)), Jtr_abs=np.zeros(dim),
               margin=np.zeros((P, npix), np.float32), accepted=np.zeros((P, npix), np.uint8), contrib=np.zeros((P, npix), np.float32))
    rc = lib.oracle_dense_system_ex(
        ctypes.c_int(N), ctypes.c_int(H), ctypes.c_int(W), _fp(depth), _fp(normal),
        ctypes.c_float(K[0]), ctypes.c_float(K[1]), ctypes.c_float(K[2]), ctypes.c_float(K[3]),
        _fp(pairs) if P else None, ctypes.c_int(P), ctypes.byref(params), _fp(poses), ctypes.c_int(1 if flip else 0),
        *(_fp(out[k]) for k in ("JtJ", "Jtr", "n_found", "JtJ_abs", "Jtr_abs", "margin", "accepted", "contrib")))
    if rc != 0:
        raise RuntimeError(f"oracle_dense_system_ex rc={rc}")
    return out


def sparse_system(corr, poses, params=None, precision="f64"):
    """Explicit matrix of the reference's matrix-free sparse operator at `poses`, its right-hand side -wS J^T F, the Jacobi
    preconditioner and the gradient's |term| sums: (A [6(N-1)]^2, rhs, minv, rhs_abs), unknowns of frames 1..N-1, trans 0-2 / rot 3-5."""
    lib = _lib(precision)
    corr = np.ascontiguousarray(corr)
    poses = np.ascontiguousarray(poses, np.float32)
    N = poses.shape[0]
    d = 6 * (N - 1)
    A, rhs, minv, ra = np.zeros((d, d)), np.zeros(d), np.zeros(d), np.zeros(d)
    rc = lib.oracle_sparse_system(ctypes.c_int(N), ctypes.c_int(len(corr)), _fp(corr), ctypes.byref(params or default_params()), _fp(poses),
                                  _fp(A), _fp(rhs), _fp(minv), _fp(ra))
    if rc != 0:
        raise RuntimeError(f"oracle_sparse_system rc={rc}")
    return A, rhs, minv, ra


def sparse_apply(corr, poses, x, params=None, precision="f64"):
    """The matrix-free operator applyJT(applyJ(x)) itself, x in the layout of sparse_system."""
    lib = _lib(precision)
    corr = np.ascontiguousarray(corr)
    poses = np.ascontiguousarray(poses, np.float32)
    x = np.ascontiguousarray(x, np.float64)
    y = np.zeros_like(x)
    rc = lib.oracle_sparse_apply(ctypes.c_int(poses.shape[0]), ctypes.c_int(len(corr)), _fp(corr), ctypes.byref(params or default_params()), _fp(poses), _fp(x), _fp(y))
    if rc != 0:
        raise RuntimeError(f"oracle_sparse_apply rc={rc}")
    return y


def build_cache(depth, normal, K, downscale=4.0, precision="f32"):
    lib = _lib(precision)
    depth = np.ascontiguousarray(depth, np.float32)
    normal = np.ascontiguousarray(normal, np.float32)
    N, H, W = depth.shape
    w, h = int(W / downscale), int(H / downscale)
    campos = np.zeros((N, h, w, 4), np.float32)
    nrm = np.zeros((N, h, w, 4), np.float32)
    intr = np.zeros(4, np.float32)
    lib.oracle_build_cache(ctypes.c_int(N), ctypes.c_int(H), ctypes.c_int(W), _fp(depth), _fp(normal),
                           ctypes.c_float(K[0]), ctypes.c_float(K[1]), ctypes.c_float(K[2]), ctypes.c_float(K[3]),
                           ctypes.c_float(downscale), _fp(campos), _fp(nrm), _fp(intr))
    return campos, nrm, intr


def matrix_to_pose(T):
    lib = _lib("f32")
    T = np.ascontiguousarray(T, np.float32)
    r = np.zeros(3, np.float32)
    t = np.zeros(3, np.float32)
    lib.oracle_matrix_to_pose(_fp(T), _fp(r), _fp(t))
    return r, t


def pose_to_matrix(r, t):
    lib = _lib("f32")
    r = np.ascontiguousarray(r, np.float32)
    t = np.ascontiguousarray(t, np.float32)
    T = np.zeros((4, 4), np.float32)
    lib.oracle_pose_to_matrix(_fp(r), _fp(t), _fp(T))
    return T


# ---------------------------------------------------------------------------------------------------------------------
# Oracle B: the reference's own CUDA kernels, compiled verbatim by oracle/Makefile (`make ref`) into oracle/_ref.
# Needs a GPU; used by the `-m gpu` parity tests and by `bench.py --impl reference`.
class RefParams(ctypes.Structure):
    _fields_ = OracleParams._fields_


_ref = None


def build_ref(force: bool = False) -> bool:
    """(Re)build oracle/_ref/libbt_ref.so from /root/reference when it is present (this container only)."""
    out = os.path.join(_HERE, "_ref", "libbt_ref.so")
    if os.path.isdir("/root/reference/src/cuda") and (force or not os.path.exists(out)):
        subprocess.check_call(["make", "-C", _HERE, "ref", "-j4"], stdout=subprocess.DEVNULL)
    return os.path.exists(out)


def ref_lib():
    global _ref
    if _ref is None:
        path = os.path.join(_HERE, "_ref", "libbt_ref.so")
        if not os.path.exists(path):
            raise RuntimeError("oracle/_ref/libbt_ref.so missing: run `make -C oracle ref` where /root/reference exists")
        _ref = ctypes.CDLL(path)
        _ref.ref_optimize_frames.restype = ctypes.c_int
        _ref.ref_ransac_pairs.restype = ctypes.c_int
        _ref.ref_frame_preprocess.restype = ctypes.c_int
    return _ref


def ref_optimize_frames(depth_ptrs, normal_ptrs, H, W, K, corr, poses, params=None):
    """Run the reference's optimizeFrames-equivalent on the current CUDA device.
    depth_ptrs/normal_ptrs: lists of device addresses.  Returns (poses [N,4,4], pairs [(tgt,src)], t_outer_ms, t_solve_ms)."""
    lib = ref_lib()
    N = len(depth_ptrs)
    params = params or default_params()
    rp = RefParams(*[getattr(params, f[0]) for f in OracleParams._fields_])
    dp = (ctypes.c_void_p * N)(*[int(p) for p in depth_ptrs])
    nq = (ctypes.c_void_p * N)(*[int(p) for p in normal_ptrs])
    corr = np.ascontiguousarray(corr)
    poses = np.ascontiguousarray(poses, np.float32).copy()
    pairs = np.zeros((N * (N - 1) // 2 + 1, 2), np.uint32)
    npairs = ctypes.c_int(0)
    t_outer = ctypes.c_double(0)
    t_solve = ctypes.c_double(0)
    rc = lib.ref_optimize_frames(ctypes.c_int(N), ctypes.c_int(H), ctypes.c_int(W), dp, nq,
                                 ctypes.c_float(K[0]), ctypes.c_float(K[1]), ctypes.c_float(K[2]), ctypes.c_float(K[3]),
                                 ctypes.c_int(len(corr)), _fp(corr), _fp(poses), ctypes.byref(rp),
                                 _fp(pairs), ctypes.byref(npairs), ctypes.byref(t_outer), ctypes.byref(t_solve))
    if rc != 0:
        raise RuntimeError(f"ref_optimize_frames rc={rc}")
    return poses, pairs[: npairs.value].copy(), t_outer.value, t_solve.value


def ref_frame_preprocess(depth_raw, K, dp=None):
    """The reference's Frame front end (its own kernels, oracle/_ref) on the current CUDA device.
    depth_raw [H,W] float32, K=(fx,fy,cx,cy), dp = dict(erode_radius, erode_diff, erode_ratio, bf_radius, sigma_D, sigma_R).
    Returns (depth [H,W], xyz [H,W,4], normal [H,W,4], t_ms)."""
    from . import frame_oracle
    lib = ref_lib()
    dp = dict(frame_oracle.DEFAULTS, **(dp or {}))
    d = np.ascontiguousarray(depth_raw, np.float32)
    H, W = d.shape
    dout = np.zeros((H, W), np.float32); xyz = np.zeros((H, W, 4), np.float32); nrm = np.zeros((H, W, 4), np.float32)
    t = ctypes.c_double(0)
    rc = lib.ref_frame_preprocess(ctypes.c_int(H), ctypes.c_int(W), _fp(d), ctypes.c_float(K[0]), ctypes.c_float(K[1]), ctypes.c_float(K[2]), ctypes.c_float(K[3]),
                                  ctypes.c_int(int(dp["erode_radius"])), ctypes.c_float(dp["erode_diff"]), ctypes.c_float(dp["erode_ratio"]),
                                  ctypes.c_int(int(dp["bf_radius"])), ctypes.c_float(dp["sigma_D"]), ctypes.c_float(dp["sigma_R"]),
                                  _fp(dout), _fp(xyz), _fp(nrm), ctypes.byref(t))
    if rc != 0:
        raise RuntimeError(f"ref_frame_preprocess failed: {rc}")
    return dout, xyz, nrm, t.value


def ref_ransac_pairs(ptsA, ptsB, n_trials=2000, dist_thresh=0.005):
    """The reference's ransacMultiPairGPU (/root/reference/src/cuda/cuda_ransac.cu:1228-1323, its own kernels in oracle/_ref) on the
    current CUDA device, behind the upload SiftManager::runRansacMultiPairGPU does (FeatureManager.cpp:701-717).
    ptsA[p], ptsB[p]: [n_p, 4] float32 model-frame points (w = 1).  Returns (list of int32 inlier-id arrays, t_ms)."""
    lib = ref_lib()
    n = len(ptsA)
    A = [np.ascontiguousarray(a, np.float32) for a in ptsA]
    B = [np.ascontiguousarray(b, np.float32) for b in ptsB]
    cnt = (ctypes.c_int * n)(*[a.shape[0] for a in A])
    pa = (ctypes.c_void_p * n)(*[a.ctypes.data for a in A])
    pb = (ctypes.c_void_p * n)(*[b.ctypes.data for b in B])
    total = sum(a.shape[0] for a in A)
    ids = np.zeros(max(total, 1), np.int32)
    nin = np.zeros(n, np.int32)
    t = ctypes.c_double(0)
    rc = lib.ref_ransac_pairs(ctypes.c_int(n), pa, pb, cnt, ctypes.c_int(n_trials), ctypes.c_float(dist_thresh), _fp(ids), _fp(nin), ctypes.byref(t))
    if rc != 0:
        raise RuntimeError(f"ref_ransac_pairs rc={rc}")
    out, o = [], 0
    for p in range(n):
        out.append(ids[o:o + int(nin[p])].copy())
        o += int(nin[p])
    return out, t.value
