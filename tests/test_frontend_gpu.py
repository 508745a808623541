"""GPU parity tests of the fused frame front end (bt_frames_preprocess through the C-ABI) against the CPU restatement
(oracle/frame_oracle.py) and the committed golden vectors of the reference's kernels (ref_frame_*.npz, and ref_live_frame.npz:
the reference's outputs for a whole 640x480 frame, recorded on an H100 by scripts/make_golden_live.py and stored to within a
small fraction of the tolerances below).  Against the oracle, every pixel outside the float64 statement's taint mask is held to its
own bound (frame_oracle.device_report, no fraction allowance).  Against the reference's recordings: filtered depth 2e-6 m (a few
float ulps at ~1 m; the reference build uses fast-math exp/division), normals 1e-3, on every pixel: the pixels beyond those are
counted and printed, and there are none (measured on an H100: 0 in each of the three recordings)."""
import glob
import os
import zlib

import numpy as np
import pytest

from bundletrack_b200 import synth
from oracle import frame_oracle

pytestmark = pytest.mark.gpu
GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "ref_frame_*.npz")))


@pytest.fixture(scope="module")
def fe(cuda_device):
    from bundletrack_b200.frontend import FrameFrontEnd
    f = FrameFrontEnd()
    yield f
    f.close()


def _run(fe, raws, K, dev, dp=None, want_xyz=True):
    import torch
    from bundletrack_b200 import _lib
    if dp:
        full = dict(frame_oracle.DEFAULTS, **dp)
        fe.params = _lib.DepthParams(int(full["erode_radius"]), full["erode_diff"], full["erode_ratio"], int(full["bf_radius"]), full["sigma_D"], full["sigma_R"])
    else:
        from bundletrack_b200.config import depth_params
        fe.params = depth_params(None)
    H, W = raws[0].shape
    tin = [torch.from_numpy(np.ascontiguousarray(r)).to(dev) for r in raws]
    dout = [torch.full((H, W), -7.0, device=dev) for _ in raws]
    nout = [torch.full((H, W, 4), -7.0, device=dev) for _ in raws]
    xout = [torch.full((H, W, 4), -7.0, device=dev) for _ in raws] if want_xyz else None
    fe.process(tin, H, W, K, dout, nout, xout)
    torch.cuda.synchronize()
    return [d.cpu().numpy() for d in dout], [n.cpu().numpy() for n in nout], ([x.cpu().numpy() for x in xout] if want_xyz else None)


def _check64(d, n, x, raw, K, dp=None):
    """Per pixel against preprocess64 (and, where subnormal filter weights feed a pixel, against the float32 restatement at 2e-6 / 3e-6
    / 1e-3).  Tainted pixels are exempt, so their number is printed and held below 1 % of the valid pixels."""
    rep = frame_oracle.device_report(d, x, n, frame_oracle.preprocess64(raw, K, dp), frame_oracle.preprocess(raw, K, dp))
    print(f"tainted {rep['tainted']}, subnormal-weight {rep['subnormal']}, of {rep['valid']} valid; "
          f"worst error / bound: depth {rep['depth_frac']:.3f} normal {rep['normal_frac']:.3f}")
    assert not rep["failures"], "; ".join(rep["failures"])
    assert rep["tainted"] <= 0.01 * rep["valid"]


def _check_recorded(d, n, x, rd, rn, rx, raw, K, dp=None):
    """Against the reference's recorded maps: no pixel beyond 2e-6 (depth), 3e-6 (points) or 1e-3 (normals).  Differing pixels are
    printed with whether preprocess64 taints them, i.e. whether a float32 gate decision there may go either way."""
    bad_d = np.abs(d - rd) > 2e-6
    bad_n = np.abs(n[..., :3] - rn[..., :3]).max(-1) > 1e-3
    taint = frame_oracle.preprocess64(raw, K, dp).taint
    print(f"pixels differing from the reference: depth {int(bad_d.sum())}, normals {int(bad_n.sum())} (tainted in float64: {int(taint.sum())})")
    bad = bad_d | bad_n
    assert not bad.any(), [(p, bool(taint[tuple(p)])) for p in np.argwhere(bad)[:10].tolist()]
    if x is not None:
        assert np.abs(x[..., :3] - rx[..., :3]).max() <= 3e-6
        assert np.array_equal(x[..., 3], (rd >= 0.1).astype(np.float32))
    assert np.all(n[..., 3] == 0)


@pytest.mark.parametrize("seed,H,W", [(0, 120, 160), (1, 97, 131), (2, 480, 640)])
def test_matches_oracle(fe, cuda_device, seed, H, W):
    raw, K = synth.make_raw_depth(seed, H, W)
    d, n, x = _run(fe, [raw], K, cuda_device)
    _check64(d[0], n[0], x[0], raw, K)
    assert (d[0] > 0).sum() > 0.02 * H * W          # the filter fills small holes and keeps the object


def test_other_parameters_and_batch(fe, cuda_device):
    dp = {"erode_radius": 2, "erode_diff": 0.004, "erode_ratio": 0.5, "bf_radius": 1, "sigma_D": 1.5, "sigma_R": 0.05}
    raws, K = [], None
    for s in (3, 4, 5):
        r, K = synth.make_raw_depth(s, 100, 140)
        raws.append(r)
    d, n, x = _run(fe, raws, K, cuda_device, dp)
    for i, r in enumerate(raws):
        _check64(d[i], n[i], x[i], r, K, dp)
    # a batch equals the same frames one at a time, bit for bit; xyz is optional
    d1, n1, _ = _run(fe, [raws[1]], K, cuda_device, dp, want_xyz=False)
    assert np.array_equal(d1[0], d[1]) and np.array_equal(n1[0], n[1])


def test_edge_cases(fe, cuda_device):
    import torch
    from bundletrack_b200 import _lib
    K = synth.NOCS_K
    zero = np.zeros((70, 90), np.float32)
    d, n, x = _run(fe, [zero], K, cuda_device)
    assert not d[0].any() and not n[0].any() and not x[0].any()
    # constant plane: interior depth unchanged to rounding, normals point at the camera; the image border has no normal
    plane = np.full((64, 80), 0.75, np.float32)
    d, n, x = _run(fe, [plane], K, cuda_device)
    assert np.abs(d[0] - 0.75).max() < 1e-6
    assert np.allclose(n[0][1:-1, 1:-1, :3], [0, 0, -1], atol=1e-3)     # (x - cx) / fx * d differences cancel to ~1e-4 relative
    assert not n[0][0].any() and not n[0][-1].any() and not n[0][:, 0].any() and not n[0][:, -1].any()
    # an isolated flying pixel is eroded away and refilled from its neighbours by the filter
    spike = plane.copy(); spike[30, 40] = 0.80
    d, _, _ = _run(fe, [spike], K, cuda_device)
    assert abs(d[0][30, 40] - 0.75) < 1e-6
    # errors are reported, not fatal
    t = torch.zeros((64, 80), device=cuda_device)
    nn = torch.zeros((64, 80, 4), device=cuda_device)
    with pytest.raises(_lib.BtError):
        fe.process([t], 64, 80, K, [t], [nn])                       # in place
    fe.params = _lib.DepthParams(5, 0.001, 0.8, 4, 2.0, 1e5)         # halo 14 > supported
    with pytest.raises(_lib.BtError):
        fe.process([t], 64, 80, K, [torch.zeros_like(t)], [nn])


@pytest.mark.skipif(not GOLDEN, reason="no golden vectors")
@pytest.mark.parametrize("path", GOLDEN)
def test_golden_reference_kernels(fe, cuda_device, path):
    g = np.load(path)
    dp = {k: float(g[k]) for k in frame_oracle.DEFAULTS}
    d, n, x = _run(fe, [g["raw"]], tuple(g["K"]), cuda_device, dp)
    rn = np.concatenate([g["normal"], np.zeros(g["normal"].shape[:2] + (1,), np.float32)], -1)
    rx = np.concatenate([g["xyz"], (g["depth"] >= 0.1).astype(np.float32)[..., None]], -1)
    _check_recorded(d[0], n[0], x[0], g["depth"], rn, rx, g["raw"], tuple(g["K"]), dp)


# (name, quantisation step): at most half a step from the reference, i.e. <= 6 % of the depth / point tolerance and < 1 % of the normal one
_FRAME_OUT = (("depth", 2.0 ** -22), ("xyz", 2.0 ** -22), ("normal", 2.0 ** -16))


def frame_encode(raw, K, *ref):
    """The reference's front-end outputs (depth, xyz, normal) of a whole frame, stored as their difference from what
    oracle/frame_oracle.py computes for the same raw frame, in int8 multiples of a step far below the test tolerances (zero almost
    everywhere: a few tens of KB), plus a CRC of the decoded arrays that catches a restatement which no longer decodes them."""
    out = {}
    for (name, step), r, o in zip(_FRAME_OUT, ref, frame_oracle.preprocess(raw, K)):
        assert np.isfinite(r).all() and np.isfinite(o).all(), name
        q = np.rint((np.asarray(r, np.float64) - np.asarray(o, np.float64)) / step)
        assert np.abs(q).max() <= 127, f"{name}: the reference differs from the restatement by more than int8 steps hold"
        out[name] = q.astype(np.int8)
        out[name + "_crc"] = np.uint32(zlib.crc32(_decode(o, out[name], step).tobytes()))
    return out


def _decode(o, q, step):
    return (np.asarray(o, np.float64) + q.astype(np.float64) * step).astype(np.float32)


def frame_decode(raw, K, g):
    ref = []
    for (name, step), o in zip(_FRAME_OUT, frame_oracle.preprocess(raw, K)):
        r = _decode(o, g[name], step)
        assert zlib.crc32(r.tobytes()) == int(g[name + "_crc"]), f"{name}: oracle/frame_oracle.py changed; re-record tests/golden/ref_live_frame.npz"
        ref.append(r)
    return ref


def test_matches_reference_kernels_live(fe, cuda_device):
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "ref_live_frame.npz"))
    raw, K = synth.make_raw_depth(7, 480, 640)
    rd, rx, rn = frame_decode(raw, K, g)
    d, n, x = _run(fe, [raw], K, cuda_device)
    _check_recorded(d[0], n[0], x[0], rd, rn, rx, raw, K)


def test_feeds_the_solver(fe, cuda_device):
    """Front-end outputs are exactly the maps bt_solve_windows consumes: solving on GPU-filtered maps equals the oracle solving
    on oracle-filtered maps (1e-4 rad / 1e-4 m, north_star's gate)."""
    import torch
    import oracle
    from bundletrack_b200.optimizer import OptimizerGpu, SolveWindow
    w = synth.make_window(11, n_frames=3, n_corr=400, H=240, W=320, K=tuple(v * 0.5 for v in synth.NOCS_K))
    rng = np.random.default_rng(5)
    raws = [(w.depth[k] + (w.depth[k] > 0) * rng.normal(0, 0.0003, w.depth[k].shape)).astype(np.float32) for k in range(3)]
    d, n, _ = _run(fe, raws, w.K, cuda_device, want_xyz=False)
    td = [torch.from_numpy(v).to(cuda_device) for v in d]
    tn = [torch.from_numpy(v).to(cuda_device) for v in n]
    opt = OptimizerGpu(None, max_windows=1, max_frames=3, max_corr=400, H=240, W=320)
    got = opt.optimizeWindows([SolveWindow(w.corr, 240, 320, td, tn, w.poses_init, w.K)])[0]
    opt.close()
    od = np.stack([frame_oracle.preprocess(r, w.K)[0] for r in raws])
    on = np.stack([frame_oracle.preprocess(r, w.K)[2] for r in raws])
    ref = oracle.solve_window(od, on, w.K, w.corr, w.poses_init)
    r, t = synth.pose_errors(got, ref)
    assert r <= 1e-4 and t <= 1e-4
