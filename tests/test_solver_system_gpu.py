"""The per-iteration system of k_solve against oracle A (float64), entry by entry.

Every case solves ONE Gauss-Newton iteration (num_iter_outer = 1), so the system the library assembles is evaluated at the input
poses exactly and no earlier gate flip can spread into it.  Against the float64 build of oracle/solver_oracle.c:
  * per-pair gate counts: |library - oracle| <= the pair's marginal pixels (MARGIN_EPS);
  * the dense blocks (bt_solve_debug_dense): per entry c * sum|terms| of that entry;
  * the assembled PCG matrix and right-hand side (bt_solve_debug_system): oracle sparse (the explicit matrix of the reference's
    matrix-free operator) + oracle dense, after the FlipJtJ rule;
  * the PCG result: the reference's recurrences in float64 on the library's own A, rhs and Jacobi diagonal; the pose update against
    exp(delta) exp(x) in float64.
Pairs with a marginal pixel are left out of the entry-wise dense check (their counts are still checked); most windows have none.
test_tolerance_is_below_one_pixel (CPU only) shows the dense tolerance is smaller than what one median pixel of a pair adds."""
import dataclasses

import numpy as np
import pytest

import oracle
from bundletrack_b200 import synth

C_DENSE = 1e-4       # per-entry tolerance factor on sum|terms| (float32 sums of a few thousand terms, model-frame Jacobians)
C_JTR = 5e-4         # the same for Jtr: its terms carry the residual, a float32 difference of two ~1 m points (relative error ~1e-4)
C_MIX = 64 * 2.0 ** -24   # plus C_MIX * sqrt(D_aa D_bb): the library rotates each pair's 6x6 sums into the model frame, which mixes an
                          # entry's rounding with that of the larger entries of its rows and columns (bounded by the diagonals)
C_SPARSE = 2e-5      # sparse blocks: relative to the largest entry of the 6x6 block (moment sums vs matrix-free products)


def _yml(downscale=4, robust_delta=0.005, max_dist=0.02, angle=45.0, inner=5):
    return {"bundle": {"num_iter_outter": 1, "num_iter_inner": inner, "robust_delta": robust_delta, "image_downscale": downscale},
            "p2p": {"max_dist": max_dist, "max_normal_angle": angle}}


def _oparams(o):
    return oracle.OracleParams(*[getattr(o.params, f) for f, _ in oracle.OracleParams._fields_])


def _scaled_K(H, W):
    fx, fy, cx, cy = synth.NOCS_K
    return (fx * W / 640.0, fy * H / 480.0, cx * (W - 1) / 639.0, cy * (H - 1) / 479.0)


def _window(seed, N=5, C=800, H=480, W=640, **kw):
    return synth.make_window(seed, n_frames=N, n_corr=C, H=H, W=W, K=_scaled_K(H, W), **kw)


def _upload(w, dev):
    import torch
    return ([torch.from_numpy(np.ascontiguousarray(w.depth[k])).to(dev) for k in range(w.n_frames)],
            [torch.from_numpy(np.ascontiguousarray(w.normal[k])).to(dev) for k in range(w.n_frames)])


def _opt(yml, max_windows=1, max_frames=8, max_corr=4096, H=480, W=640, debug=True):
    from bundletrack_b200.optimizer import OptimizerGpu
    o = OptimizerGpu(yml, max_windows=max_windows, max_frames=max_frames, max_corr=max_corr, H=H, W=W)
    if debug:
        o.enable_debug(True)
    return o


def _sw(w, dev, corr=None, pairs=None, compat_flip=True, cache_slots=None, maps=None):
    from bundletrack_b200.optimizer import SolveWindow
    d, n = (None, None) if cache_slots is not None else (maps or _upload(w, dev))
    return SolveWindow(w.corr if corr is None else corr, w.H, w.W, d, n, w.poses_init, w.K, dense_pairs=pairs, compat_flip=compat_flip,
                       cache_slots=cache_slots)


def _sym(J):
    """Raw addToLocalSystem sums -> the full symmetric system (every cross block kept: compat_flip = False)."""
    return J + J.T - np.diag(np.diag(J))


def _flip(J):
    """FlipJtJ: upper := lower (compat_flip = True)."""
    L = np.tril(J)
    return L + np.tril(J, -1).T


def _se3_exp(d):
    """poseToMatrix in float64; d = (trans 0-2, rot 3-5)."""
    t, w = np.asarray(d[:3], np.float64), np.asarray(d[3:], np.float64)
    th2 = w @ w
    th = np.sqrt(th2)
    if th2 < 1e-12:
        A, B, C = 1.0, 0.5, 1.0 / 6.0
    else:
        A, B, C = np.sin(th) / th, (1 - np.cos(th)) / th2, (1 - np.sin(th) / th) / th2
    Wx = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    T = np.eye(4)
    T[:3, :3] = np.eye(3) + A * Wx + B * Wx @ Wx
    T[:3, 3] = t + B * np.cross(w, t) + C * np.cross(w, np.cross(w, t))
    return T


def _pcg64(A, b, minv, n_iter):
    """The reference's PCG recurrences (SolverBundling.cu PCGInit / PCGStep, 1e-6 guards) in float64."""
    A, b, minv = (np.asarray(v, np.float64) for v in (A, b, minv))
    r = b.copy(); p = minv * r; rz = r @ p; x = np.zeros_like(b)
    for _ in range(n_iter):
        Ap = A @ p
        pAp = p @ Ap
        alpha = rz / pAp if pAp > 1e-6 else 0.0
        x += alpha * p; r -= alpha * Ap
        z = minv * r
        rz_new = z @ r
        beta = rz_new / rz if rz > 1e-6 else 0.0
        rz = rz_new
        p = z + beta * p
    return x


def _pcg32_spread(A, b, minv, n_iter):
    """How far float32 rounding of the same recurrences moves delta on THIS system: numpy float32 against float64."""
    A32, b32, m32 = (np.asarray(v, np.float32) for v in (A, b, minv))
    r = b32.copy(); p = m32 * r; rz = np.float32(r @ p); x = np.zeros_like(b32)
    for _ in range(n_iter):
        Ap = A32 @ p
        pAp = np.float32(p @ Ap)
        alpha = np.float32(rz / pAp) if pAp > 1e-6 else np.float32(0)
        x += alpha * p; r -= alpha * Ap
        z = m32 * r
        rz_new = np.float32(z @ r)
        beta = np.float32(rz_new / rz) if rz > 1e-6 else np.float32(0)
        rz = rz_new
        p = z + beta * p
    return np.abs(x - _pcg64(A, b, minv, n_iter)).max()


def _reference(w, o, pairs, corr=None, compat_flip=True):
    """Oracle A (float64) for one window at its input poses.  The dense term is evaluated ONE PAIR AT A TIME (raw addToLocalSystem sums,
    no FlipJtJ), so every pair's own blocks, gate count, marginal pixels and per-pixel contributions are known; the window's system is
    their sum after the FlipJtJ rule (compat_flip) or with every cross block mirrored (not compat_flip).
    A marginal pixel (closer than MARGIN_EPS to a gate boundary) may be decided either way by a float32 evaluation.  Its possible
    contribution is added to the tolerance of the entries of its pair's blocks: per JtJ entry |J_a J_b w| <= w (|J_i|^2 + |J_j|^2), taken
    as twice the largest contribution of an accepted pixel of the pair; per Jtr entry |J_a r w| <= sqrt(w (|J_i|^2 + |J_j|^2)) |r| with
    |r| <= max_dist (w <= 1)."""
    prm = _oparams(o)
    N = w.n_frames
    pairs = oracle.default_pairs(N) if pairs is None else np.asarray(pairs, np.uint32).reshape(-1, 2)
    dim = 6 * N
    d = dict(JtJ=np.zeros((dim, dim)), JtJ_abs=np.zeros((dim, dim)), Jtr=np.zeros(dim), Jtr_abs=np.zeros(dim),
             marg_J=np.zeros((dim, dim)), marg_r=np.zeros(dim), n_found=np.zeros(len(pairs), np.int64), n_marg=np.zeros(len(pairs), np.int64))
    cmax = np.zeros(len(pairs))
    for p in range(len(pairs)):
        e = oracle.dense_system_ex(w.depth, w.normal, w.K, w.poses_init, pairs=pairs[p:p + 1], params=prm, flip=False)
        for k in ("JtJ", "JtJ_abs", "Jtr", "Jtr_abs"):
            d[k] += e[k]
        d["n_found"][p] = e["n_found"][0]
        d["n_marg"][p] = ((e["margin"][0] < oracle.MARGIN_EPS) & (e["margin"][0] < 1)).sum()
        acc = e["accepted"][0] > 0
        cmax[p] = float(e["contrib"][0][acc].max()) if acc.any() else 0.0
    for p, (t, s_) in enumerate(pairs):
        m = d["n_marg"][p]
        if not m:
            continue
        c = 2.0 * (cmax[p] or cmax.max())
        idx = np.array([6 * f + a for f in (int(t), int(s_)) if f > 0 for a in range(6)], int)
        d["marg_J"][np.ix_(idx, idx)] += m * c
        d["marg_r"][idx] += m * np.sqrt(c) * prm.dense_dist_thresh
    glue = _flip if compat_flip else _sym
    d["D"], d["D_abs"] = glue(d["JtJ"]), glue(d["JtJ_abs"])
    d["pairs"] = pairs
    d["S"], d["rhs_s"], d["minv"], d["rhs_s_abs"] = oracle.sparse_system(w.corr if corr is None else corr, w.poses_init, params=prm)
    return d


def _check_system(o, k, w, ref, compat_flip=True, pose_out=None, c_dense=C_DENSE):
    """Window k of the last call of `o` against `ref` (from _reference), every entry.  Returns the number of marginal pixels."""
    N = w.n_frames
    pairs, n_marg = ref["pairs"], ref["n_marg"]
    P = len(pairs)
    cnt = o.debug_counts(k, P) if P else np.zeros(0)
    assert (np.abs(cnt - ref["n_found"]) <= n_marg).all(), (cnt, ref["n_found"], n_marg)
    # dense blocks, cross blocks included (with compat_flip = False every pair's -S is there)
    J, r = o.debug_dense(k, N)
    dg = np.sqrt(np.diag(ref["D_abs"]))
    tolJ = c_dense * ref["D_abs"] + C_MIX * np.outer(dg, dg) + ref["marg_J"] + 1e-9
    bad = np.abs(J - ref["D"]) > tolJ
    assert not bad.any(), (np.argwhere(bad)[:5], np.abs(J - ref["D"])[bad][:5], tolJ[bad][:5])
    tolr = C_JTR * ref["Jtr_abs"] + ref["marg_r"] + 1e-9
    assert (np.abs(r - ref["Jtr"]) <= tolr).all(), np.abs(r - ref["Jtr"]).max()
    # assembled system: sparse (explicit matrix of the matrix-free operator) + dense, frames 1..N-1
    A, rhs, minv, delta = o.debug_system(k, N)
    Ao = ref["S"] + ref["D"][6:, 6:]
    blk = np.abs(ref["S"]).reshape(N - 1, 6, N - 1, 6).max(axis=(1, 3))
    tolA = C_SPARSE * np.kron(blk, np.ones((6, 6))) + tolJ[6:, 6:]
    badA = np.abs(A - Ao) > tolA
    assert not badA.any(), (np.argwhere(badA)[:5], np.abs(A - Ao)[badA][:5], tolA[badA][:5])
    rhs_o = ref["rhs_s"] - ref["Jtr"][6:]
    tol_rhs = C_SPARSE * ref["rhs_s_abs"] + tolr[6:]
    assert (np.abs(rhs - rhs_o) <= tol_rhs).all(), np.abs(rhs - rhs_o).max()
    assert np.allclose(minv, ref["minv"], rtol=1e-5, atol=0)
    # PCG in isolation on the library's own system: within a few times what float32 rounding of the same recurrences does on it
    d64 = _pcg64(A, rhs, minv, o.params.num_iter_inner)
    spread = _pcg32_spread(A, rhs, minv, o.params.num_iter_inner)
    assert np.abs(delta - d64).max() <= 8 * spread + 64 * 2.0 ** -24 * np.abs(d64).max(), (np.abs(delta - d64).max(), spread, np.abs(d64).max())
    if pose_out is not None:      # x <- log(exp(delta) exp(x)): the output pose is exp(delta) * (input pose after its se(3) round trip)
        for f in range(1, N):
            r_, t_ = oracle.matrix_to_pose(w.poses_init[f])
            want = _se3_exp(delta[(f - 1) * 6:f * 6].astype(np.float64)) @ _se3_exp(np.concatenate([t_, r_]).astype(np.float64))
            assert np.abs(pose_out[f] - want).max() <= 2e-6, (f, np.abs(pose_out[f] - want).max())
    return int(n_marg.sum())


def _run_and_check(dev, ws, yml=None, pairs=None, max_frames=None, H=480, W=640, max_corr=4096, c_dense=C_DENSE):
    """Every window solved with compat_flip = False (each pair's cross block visible) and with compat_flip = True (the FlipJtJ rule),
    each checked entry by entry; debug on and off give the same bits."""
    o = _opt(yml or _yml(), max_windows=len(ws), max_frames=max_frames or max(w.n_frames for w in ws), H=H, W=W, max_corr=max_corr)
    marg = []
    for compat_flip in (False, True):
        sws = [_sw(w, dev, pairs=pairs, compat_flip=compat_flip) for w in ws]
        o.enable_debug(True)
        out = o.optimizeWindows(sws)
        m = [_check_system(o, k, w, _reference(w, o, pairs, compat_flip=compat_flip), compat_flip, out[k], c_dense) for k, w in enumerate(ws)]
        marg = marg or m
        o.enable_debug(False)
        plain = o.optimizeWindows(sws)
        for a, b in zip(out, plain):
            assert a.tobytes() == b.tobytes()      # the debug dump does not change a bit
    o.close()
    return marg


@pytest.mark.gpu
@pytest.mark.parametrize("N", [2, 3, 11, 12, 16, 32])
def test_frames(cuda_device, N):
    """One-warp PCG (N <= 11) to multi-warp PCG (N >= 12); at 32 frames the groups' moment sums stay in global memory."""
    H, W = (240, 320) if N >= 16 else (480, 640)
    w = _window(100 + N, N=N, C=100 * N, H=H, W=W)
    pairs = None if N < 32 else np.array([(i, j) for i in range(1, N) for j in (i - 1, i - 2) if j >= 0], np.uint32)   # all 496 pairs do not fit the tail
    _run_and_check(cuda_device, [w], pairs=pairs, max_frames=N, H=H, W=W)


@pytest.mark.gpu
@pytest.mark.parametrize("HW", [(97, 131), (121, 163), (483, 641), (8, 8)])
def test_image_sizes(cuda_device, HW):
    H, W = HW
    w = _window(200 + H, N=4, C=400, H=H, W=W)
    _run_and_check(cuda_device, [w], H=H, W=W)


def _cropped(seed):
    """A 640 x 480 window cut off at the object's centre column and row: the object runs into the right and bottom image borders, so
    projected pixels land next to the last column and row (the bilinear taps' validity edge)."""
    w = _window(seed, N=4, C=400)
    ys, xs = np.nonzero(w.depth[0] > 0)
    Hc, Wc = int(ys.mean()), int(xs.mean())
    return dataclasses.replace(w, depth=w.depth[:, :Hc, :Wc].copy(), normal=w.normal[:, :Hc, :Wc].copy())


@pytest.mark.gpu
def test_object_cut_by_the_image_border(cuda_device):
    w = _cropped(250)
    _run_and_check(cuda_device, [w], H=w.H, W=w.W)


@pytest.mark.gpu
def test_mixed_image_sizes_in_one_batch(cuda_device):
    ws = [_window(210 + k, N=3 + k, C=300, H=H, W=W) for k, (H, W) in enumerate([(97, 131), (480, 640), (121, 163), (483, 641), (8, 8)])]
    marg = _run_and_check(cuda_device, ws, H=483, W=641)
    assert sum(m == 0 for m in marg) >= 3      # most windows have no marginal pixel: the count check is an equality there


@pytest.mark.gpu
@pytest.mark.parametrize("downscale", [2, 3, 4, 2.5])
def test_downscale(cuda_device, downscale):
    w = _window(300, N=4, C=400, H=240, W=320)
    _run_and_check(cuda_device, [w], yml=_yml(downscale=downscale), H=240, W=320)


def _masked_to(w, f, n_valid, downscale=4.0):
    """Copy of w whose frame f keeps exactly n_valid quarter-res valid pixels (the first ones in raster order)."""
    w2 = dataclasses.replace(w, depth=w.depth.copy(), normal=w.normal.copy())
    N, H, W = w.depth.shape
    cam, _, _ = oracle.build_cache(w.depth[f:f + 1], w.normal[f:f + 1], w.K, downscale)
    h, wq = cam.shape[1:3]
    valid = np.flatnonzero(cam[0, :, :, 2].reshape(-1) >= 0.1)
    assert len(valid) >= n_valid
    keep = valid[:n_valid]
    sW, sH = np.float32(np.float32(W - 1) / np.float32(wq - 1)), np.float32(np.float32(H - 1) / np.float32(h - 1))
    xi = ((keep % wq).astype(np.float32) * sW + np.float32(0.5)).astype(np.int64)
    yi = ((keep // wq).astype(np.float32) * sH + np.float32(0.5)).astype(np.int64)
    m = np.zeros((H, W), bool)
    m[yi, xi] = True
    w2.depth[f][~m] = 0
    w2.normal[f][~m] = 0
    return w2


def _chunks_for(n, chunk):
    if n <= 0:
        return 0
    nch = -(-n // chunk)
    per = ((-(-n // nch)) + 31) & ~31
    return -(-n // per)


@pytest.mark.gpu
@pytest.mark.parametrize("n_src", [1, 2, 31, 33, 255, 257, 511, 513])
def test_chunk_tails(cuda_device, monkeypatch, n_src):
    """Source frame 0 of the pair (1, 0) masked to an exact number of valid pixels, chunk forced to 256: the last chunk holds 1 to 31
    pixels or an odd count (the odd tail of the two-pixels-in-flight loop)."""
    monkeypatch.setenv("BT_SOLVE_CHUNK", "256")
    w = _masked_to(_window(400, N=2, C=200), 0, n_src, downscale=2.0)
    o = _opt(_yml(downscale=2), max_frames=2)
    out = o.optimizeWindows([_sw(w, cuda_device, compat_flip=False)])
    assert o.stats()["n_src_pixels"] == n_src + 0      # pair (1, 0): the source is frame 0
    assert o.stats()["n_tiles_total"] == _chunks_for(n_src, 256) + 2
    _check_system(o, 0, w, _reference(w, o, None, compat_flip=False), False, out[0])
    o.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["huber_all", "huber_none", "gates"])
def test_gates_and_huber(cuda_device, case):
    yml = {"huber_all": _yml(robust_delta=1e-5), "huber_none": _yml(robust_delta=10.0), "gates": _yml(max_dist=0.0113, angle=31.0)}[case]
    w = _window(500, N=5, C=600)
    # On the Huber branch a pixel's weight is delta / |r|: the float32 rounding of the residual (~1e-7 m of two ~1 m points) enters every
    # term relative to |r|, which is not a rounding of the term itself.  With every pixel there the dense entries hold to 5e-2 sum|terms|.
    _run_and_check(cuda_device, [w], yml=yml, c_dense=5e-2 if case == "huber_all" else C_DENSE)


@pytest.mark.gpu
def test_non_unique_blocks_are_exact_and_reproducible(cuda_device):
    """Correspondence groups (i,j) and (j,i) together, and a dense list naming both directions with compat_flip = False: the cross
    blocks are then summed with shared-memory atomics.  Checked against the oracle, and solved 20 more times for the same bits."""
    w = _window(600, N=5, C=800)
    c = w.corr.copy()
    sw = c[(c["imgIdx_i"] == 1) & (c["imgIdx_j"] == 3)].copy()
    sw["imgIdx_i"], sw["imgIdx_j"] = 3, 1
    sw["pos_i"], sw["pos_j"] = sw["pos_j"].copy(), sw["pos_i"].copy()
    corr = np.concatenate([c, sw])
    pairs = np.array([(1, 0), (2, 1), (1, 2), (3, 1), (1, 3), (4, 2), (3, 4), (4, 3)], np.uint32)
    o = _opt(_yml())
    win = _sw(w, cuda_device, corr=corr, pairs=pairs, compat_flip=False)
    out = o.optimizeWindows([win])[0]
    _check_system(o, 0, w, _reference(w, o, pairs, corr=corr, compat_flip=False), False, out)
    A1 = o.debug_system(0, 5)[0]
    for _ in range(20):
        again = o.optimizeWindows([win])[0]
        assert again.tobytes() == out.tobytes() and o.debug_system(0, 5)[0].tobytes() == A1.tobytes()
    o.close()


@pytest.mark.gpu
def test_gauge_and_degenerate_inputs(cuda_device):
    from bundletrack_b200 import _lib
    w = _window(700, N=4, C=600)
    o = _opt(_yml())
    # groups that touch only frame 0 (and frame 1 through them)
    c0 = w.corr[(w.corr["imgIdx_i"] == 0)]
    out = o.optimizeWindows([_sw(w, cuda_device, corr=c0, compat_flip=False)])[0]
    _check_system(o, 0, w, _reference(w, o, None, corr=c0, compat_flip=False), False, out)
    # one correspondence
    c1 = w.corr[5:6]
    out = o.optimizeWindows([_sw(w, cuda_device, corr=c1, compat_flip=False)])[0]
    _check_system(o, 0, w, _reference(w, o, None, corr=c1, compat_flip=False), False, out)
    # a source frame without a valid pixel next to full ones
    wz = dataclasses.replace(w, depth=w.depth.copy(), normal=w.normal.copy())
    wz.depth[2] = 0
    wz.normal[2] = 0
    out = o.optimizeWindows([_sw(wz, cuda_device, compat_flip=False)])[0]
    _check_system(o, 0, wz, _reference(wz, o, None, compat_flip=False), False, out)
    # a correspondence whose two frames are the same is refused
    cs = w.corr.copy()
    cs["imgIdx_j"][:3] = cs["imgIdx_i"][:3]
    with pytest.raises(_lib.BtError):
        o.optimizeWindows([_sw(w, cuda_device, corr=cs)])
    o.close()


@pytest.mark.gpu
def test_invariance_of_counts_and_poses(cuda_device, monkeypatch):
    """Per-pair gate counts do not depend on the chunk size, the batch composition or where the maps come from; cached frames give
    the poses of the per-call rebuild bit for bit."""
    ws = [_window(800 + k, N=4 + k, C=500) for k in range(3)]
    maps = [_upload(w, cuda_device) for w in ws]
    counts = {}
    for chunk in ("256", "16384"):
        monkeypatch.setenv("BT_SOLVE_CHUNK", chunk)
        o = _opt(_yml(), max_windows=3, max_frames=6)
        o.optimizeWindows([_sw(w, cuda_device, maps=m) for w, m in zip(ws, maps)])
        counts[chunk] = [o.debug_counts(k, w.n_frames * (w.n_frames - 1) // 2).copy() for k, w in enumerate(ws)]
        o.optimizeWindows([_sw(ws[1], cuda_device, maps=maps[1])])
        assert np.array_equal(o.debug_counts(0, 10), counts[chunk][1])
        if chunk == "16384":
            plain = o.optimizeWindows([_sw(w, cuda_device, maps=m) for w, m in zip(ws, maps)])
            o.reserve_frame_cache(16)
            slots, f0 = [], 0
            for w, (d, n) in zip(ws, maps):
                slots.append(list(range(f0, f0 + w.n_frames)))
                o.store_frames(slots[-1], d, n, w.H, w.W, w.K)
                f0 += w.n_frames
            cached = o.optimizeWindows([_sw(w, cuda_device, cache_slots=s) for w, s in zip(ws, slots)])
            for k, w in enumerate(ws):
                assert cached[k].tobytes() == plain[k].tobytes()
                assert np.array_equal(o.debug_counts(k, w.n_frames * (w.n_frames - 1) // 2), counts[chunk][k])
        o.close()
    for a, b in zip(counts["256"], counts["16384"]):
        assert np.array_equal(a, b)


@pytest.mark.gpu
def test_large_batch_beyond_1024_windows_and_pairs(cuda_device):
    """1100 two-frame windows on small images: the tile plan's `base` loop and its one_each = false branch.  Every window equals its
    solve alone and oracle A's counts and system."""
    from bundletrack_b200.optimizer import OptimizerGpu
    H, W = 40, 48
    scenes = [_window(900 + k, N=2, C=60, H=H, W=W) for k in range(4)]
    maps = [_upload(w, cuda_device) for w in scenes]
    o = _opt(_yml(), max_windows=1100, max_frames=2, max_corr=64, H=H, W=W)
    wins = [_sw(scenes[k % 4], cuda_device, maps=maps[k % 4]) for k in range(1100)]
    batch = o.optimizeWindows(wins)
    refs = [_reference(w, o, None) for w in scenes]
    for k in (0, 1, 2, 3, 517, 1023, 1024, 1025, 1099):
        _check_system(o, k, scenes[k % 4], refs[k % 4], True, batch[k])
    # 120 quarter-res pixels per frame: one tile per pair whatever the chunk, so a window's sums do not depend on the batch
    alone = [o.optimizeWindows([wins[k]])[0] for k in range(4)]
    for k in range(1100):
        assert batch[k].tobytes() == alone[k % 4].tobytes(), k
    o.close()


def _self_check_cases():
    """(window, oracle params, dense pairs) of every case above that is checked with C_DENSE."""
    def prm(**kw):
        y = _yml(**kw)
        b, p2p = y["bundle"], y["p2p"]
        return oracle.default_params(num_iter_outer=1, robust_delta=b["robust_delta"], image_downscale=float(b["image_downscale"]),
                                     dense_dist_thresh=p2p["max_dist"], dense_cos_normal_thresh=float(np.cos(np.deg2rad(p2p["max_normal_angle"]))))
    for N in (2, 3, 11, 12, 16, 32):
        H, W = (240, 320) if N >= 16 else (480, 640)
        pairs = None if N < 32 else np.array([(i, j) for i in range(1, N) for j in (i - 1, i - 2) if j >= 0], np.uint32)
        yield _window(100 + N, N=N, C=100 * N, H=H, W=W), prm(), pairs
    for H, W in ((97, 131), (121, 163), (483, 641), (8, 8)):
        yield _window(200 + H, N=4, C=400, H=H, W=W), prm(), None
    for k, (H, W) in enumerate([(97, 131), (480, 640), (121, 163), (483, 641), (8, 8)]):
        yield _window(210 + k, N=3 + k, C=300, H=H, W=W), prm(), None
    yield _cropped(250), prm(), None
    for ds in (2, 3, 4, 2.5):
        yield _window(300, N=4, C=400, H=240, W=320), prm(downscale=ds), None
    for n_src in (1, 2, 31, 33, 255, 257, 511, 513):
        yield _masked_to(_window(400, N=2, C=200), 0, n_src, downscale=2.0), prm(downscale=2), None
    yield _window(500, N=5, C=600), prm(robust_delta=10.0), None
    yield _window(500, N=5, C=600), prm(max_dist=0.0113, angle=31.0), None
    yield _window(600, N=5, C=800), prm(), np.array([(1, 0), (2, 1), (1, 2), (3, 1), (1, 3), (4, 2), (3, 4), (4, 3)], np.uint32)
    yield _window(700, N=4, C=600), prm(), None
    for k in range(3):
        yield _window(800 + k, N=4 + k, C=500), prm(), None
    for k in range(4):
        yield _window(900 + k, N=2, C=60, H=40, W=48), prm(), None


def test_tolerance_is_below_one_pixel():
    """CPU only: for every window above that is held to C_DENSE, the dense tolerance on the trace of a pair's diagonal blocks
    (C_DENSE * sum|terms| over the frames other than the gauge, plus C_MIX times the window's diagonal there) is smaller than what the pair's median accepted pixel adds to that trace
    (`contrib` is zero for the gauge frame: its Jacobian is never formed).  A dropped, doubled or mis-weighted pixel cannot hide in it;
    a dropped or doubled one also moves the pair's gate count, which is checked exactly wherever the pair has no marginal pixel."""
    n_checked = 0
    for w, prm, pairs in _self_check_cases():
        pairs = oracle.default_pairs(w.n_frames) if pairs is None else pairs
        full = np.diag(oracle.dense_system_ex(w.depth, w.normal, w.K, w.poses_init, pairs=pairs, params=prm, flip=False)["JtJ_abs"])
        for p, (t, s) in enumerate(pairs):
            d = oracle.dense_system_ex(w.depth, w.normal, w.K, w.poses_init, pairs=pairs[p:p + 1], params=prm, flip=False)
            acc = d["accepted"][0] > 0
            idx = [6 * int(f) + a for f in (t, s) if f > 0 for a in range(6)]
            if acc.sum() == 0 or not idx:
                continue
            trace_tol = C_DENSE * d["JtJ_abs"][idx, idx].sum() + C_MIX * full[idx].sum()
            assert trace_tol < np.median(d["contrib"][0][acc]), (w.n_frames, p, trace_tol, np.median(d["contrib"][0][acc]))
            n_checked += 1
    assert n_checked > 400
