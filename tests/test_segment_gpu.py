"""GPU tests of the object-mask front end (bt_frames_preprocess_masked) and the LF-Net request (bt_lfnet_request): byte for byte
against OpenCV's recordings (tests/golden/ref_segment.npz) and the CPU restatement (oracle/segment_oracle.py), the masked maps
bit for bit against bt_frames_preprocess's with the mask applied afterwards, and the solver fed from them."""
import hashlib
import os

import numpy as np
import pytest

from bundletrack_b200 import _lib, synth
from oracle import segment_oracle as so

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ref_segment.npz")
HULL, AS_IS = _lib.BT_MASK_LARGEST_HULL, _lib.BT_MASK_AS_IS


@pytest.fixture(scope="module")
def fe(cuda_device):
    from bundletrack_b200.frontend import FrameFrontEnd
    f = FrameFrontEnd()
    yield f
    f.close()


def _raw(seed, H, W):
    if H >= 32 and W >= 32:
        return synth.make_raw_depth(seed, H, W)[0]
    return np.full((H, W), 0.7, np.float32)


def _masked(fe, raws, masks, mode, dev, K=synth.NOCS_K, want_xyz=True):
    import torch
    H, W = raws[0].shape
    n = len(raws)
    tin = [torch.from_numpy(np.ascontiguousarray(r)).to(dev) for r in raws]
    tm = [torch.from_numpy(np.ascontiguousarray(m)).to(dev) for m in masks]
    d = [torch.full((H, W), -7.0, device=dev) for _ in range(n)]
    nn = [torch.full((H, W, 4), -7.0, device=dev) for _ in range(n)]
    x = [torch.full((H, W, 4), -7.0, device=dev) for _ in range(n)] if want_xyz else None
    fg = [torch.full((H, W), 77, dtype=torch.uint8, device=dev) for _ in range(n)]
    roi = fe.process_masked(tin, tm, H, W, K, d, nn, fg, xyz_out=x, mode=mode)
    torch.cuda.synchronize()
    c = lambda ts: [t.cpu().numpy() for t in ts]
    return c(d), c(nn), (c(x) if want_xyz else None), c(fg), roi, fg


def _unmasked(fe, raws, dev, K=synth.NOCS_K):
    import torch
    H, W = raws[0].shape
    tin = [torch.from_numpy(np.ascontiguousarray(r)).to(dev) for r in raws]
    d = [torch.empty((H, W), device=dev) for _ in raws]
    nn = [torch.empty((H, W, 4), device=dev) for _ in raws]
    x = [torch.empty((H, W, 4), device=dev) for _ in raws]
    fe.process(tin, H, W, K, d, nn, x)
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in d], [t.cpu().numpy() for t in nn], [t.cpu().numpy() for t in x]


def _request(fe, colours, fg_dev, dev, roi=None, fill=123):
    import torch
    tc = [torch.from_numpy(np.ascontiguousarray(c)).to(dev) for c in colours]
    out = [torch.full((400, 400, 3), fill, dtype=torch.uint8, device=dev) for _ in colours]
    H, W = colours[0].shape[:2]
    fe.lfnet_request(tc, fg_dev, H, W, out, roi=roi)
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in out]


def _check_frame(raw, mask, mode, d, n, x, fg, roi, ud, un, ux):
    """fg / roi equal the oracle; every map equals the unmasked one where fg != 0 and is exactly +0.0 elsewhere."""
    rf, rr = so.segment(mask, mode)
    assert np.array_equal(fg, rf)
    assert np.array_equal(roi, rr)
    keep = fg != 0
    for got, ref in ((d, ud), (n, un), (x, ux)):
        exp = np.where(keep if ref.ndim == 2 else keep[..., None], ref, np.float32(0))
        assert np.array_equal(got.view(np.uint32), exp.astype(np.float32).view(np.uint32))


def test_equals_golden(fe, cuda_device):
    g = np.load(GOLDEN)
    for i in range(int(g["n_cases"])):
        mask = g[f"mask_{i}"]
        H, W = mask.shape
        raw = _raw(i, H, W)
        d, n, x, fg, roi, fg_dev = _masked(fe, [raw], [mask], int(g[f"mode_{i}"]), cuda_device)
        assert np.array_equal(fg[0], g[f"fg_{i}"]), i
        assert np.array_equal(roi[0], g[f"roi_{i}"]), i
        req = _request(fe, [so.test_colour(H, W)], fg_dev, cuda_device)[0]
        if f"req_sha256_{i}" in g:                      # OpenCV's request, recorded as the SHA-256 of its bytes
            if hashlib.sha256(np.ascontiguousarray(req).tobytes()).digest() != g[f"req_sha256_{i}"].tobytes():
                ref = so.lfnet_request(so.test_colour(H, W), g[f"fg_{i}"], g[f"roi_{i}"])
                pytest.fail(f"case {i}: request differs from OpenCV's; {int((req != ref).sum())} bytes differ from the oracle's")
        else:
            assert (req == 123).all(), i


@pytest.mark.parametrize("mode", [HULL, AS_IS])
@pytest.mark.parametrize("seed,H,W", [(0, 480, 640), (1, 97, 131), (2, 3, 5)])
def test_matches_oracle(fe, cuda_device, seed, H, W, mode):
    raw = _raw(seed, H, W)
    mask = synth.make_object_mask(seed, H, W) if H > 8 else np.array([[0, 0, 9, 0, 0], [0, 9, 0, 0, 0], [0, 0, 0, 0, 3]], np.uint8)
    d, n, x, fg, roi, fg_dev = _masked(fe, [raw], [mask], mode, cuda_device)
    ud, un, ux = _unmasked(fe, [raw], cuda_device)
    _check_frame(raw, mask, mode, d[0], n[0], x[0], fg[0], roi[0], ud[0], un[0], ux[0])
    req = _request(fe, [so.test_colour(H, W)], fg_dev, cuda_device)[0]
    ref = so.lfnet_request(so.test_colour(H, W), fg[0], roi[0])
    assert (req == 123).all() if ref is None else np.array_equal(req, ref)


@pytest.mark.parametrize("mode", [HULL, AS_IS])
def test_batch_of_mixed_frames(fe, cuda_device, mode):
    H, W = 120, 160
    masks = [synth.make_object_mask(s, H, W, n_distractors=s % 4, speckle_frac=0.001 * (s % 3)) for s in range(6)]
    masks += [np.zeros((H, W), np.uint8), np.full((H, W), 200, np.uint8)]
    masks[3][masks[3] != 0] = 17
    raws = [_raw(20 + s, H, W) for s in range(8)]
    d, n, x, fg, roi, fg_dev = _masked(fe, raws, masks, mode, cuda_device)
    ud, un, ux = _unmasked(fe, raws, cuda_device)
    for k in range(8):
        _check_frame(raws[k], masks[k], mode, d[k], n[k], x[k], fg[k], roi[k], ud[k], un[k], ux[k])
    cols = [np.roll(so.test_colour(H, W), 7 * k, axis=1) for k in range(8)]
    reqs = _request(fe, cols, fg_dev, cuda_device)
    for k in range(8):
        ref = so.lfnet_request(cols[k], fg[k], roi[k])
        assert (reqs[k] == 123).all() if ref is None else np.array_equal(reqs[k], ref), k
    # the same frames one at a time give the same bytes
    d1, _, _, fg1, roi1, _ = _masked(fe, [raws[2]], [masks[2]], mode, cuda_device)
    assert np.array_equal(d1[0], d[2]) and np.array_equal(fg1[0], fg[2]) and np.array_equal(roi1[0], roi[2])


def _spiral(H, W):
    """A 1-pixel-wide rectangular spiral with 1-pixel gaps between its turns: one component that crosses every tile border."""
    m = np.zeros((H, W), np.uint8)
    top, left, bottom, right = 1, 1, H - 2, W - 2
    while top + 2 <= bottom and left + 2 <= right:
        m[top, left:right + 1] = 1
        m[top:bottom + 1, right] = 1
        m[bottom, left:right + 1] = 1
        m[top + 2:bottom + 1, left] = 1
        m[top + 2, left:left + 2] = 1          # the step into the next turn
        top, left, bottom, right = top + 2, left + 2, bottom - 2, right - 2
    return m


def _adversarial(H, W):
    y, x = np.mgrid[0:H, 0:W]
    cases = {"checkerboard": ((x + y) % 2 == 0), "spiral": _spiral(H, W) != 0}
    comb = np.zeros((H, W), bool); comb[0, :] = True; comb[:, ::3] = True; comb[H // 2, 1::3] = False
    cases["comb"] = comb
    cases["staircase"] = (x == y) | (x == y + 40) | (x + y == W - 1)                 # diagonal-only connections
    tie = np.zeros((H, W), bool); tie[300:340, 400:430] = True; tie[100:130, 50:90] = True   # 1200 pixels each; (100, 50) first
    cases["tie"] = tie
    border = np.zeros((H, W), bool); border[0, :] = True; border[:, 0] = True; border[H - 1, :] = True; border[:, W - 1] = True
    border[200:260, 300:500] = True; border[230, 0:300] = True
    cases["border"] = border
    cases["empty"] = np.zeros((H, W), bool)
    cases["full"] = np.ones((H, W), bool)
    return cases


@pytest.mark.parametrize("name", ["checkerboard", "spiral", "comb", "staircase", "tie", "border", "empty", "full"])
def test_adversarial_masks(fe, cuda_device, name):
    H, W = 480, 640
    mask = (_adversarial(H, W)[name] * 255).astype(np.uint8)
    raw = _raw(3, H, W)
    ud, un, ux = _unmasked(fe, [raw], cuda_device)
    for mode in (HULL, AS_IS):
        d, n, x, fg, roi, _ = _masked(fe, [raw], [mask], mode, cuda_device)
        _check_frame(raw, mask, mode, d[0], n[0], x[0], fg[0], roi[0], ud[0], un[0], ux[0])
        if name == "empty":
            assert tuple(roi[0]) == so.ROI_EMPTY and not d[0].any() and not n[0].any() and not x[0].any() and not fg[0].any()
    if name == "tie":
        lab, best = so.largest_component(mask)
        assert lab[100, 50] == best


def test_all_255_as_is_equals_unmasked(fe, cuda_device):
    raw = _raw(4, 480, 640)
    d, n, x, fg, roi, _ = _masked(fe, [raw], [np.full((480, 640), 255, np.uint8)], AS_IS, cuda_device)
    ud, un, ux = _unmasked(fe, [raw], cuda_device)
    assert d[0].tobytes() == ud[0].tobytes() and n[0].tobytes() == un[0].tobytes() and x[0].tobytes() == ux[0].tobytes()
    assert (fg[0] == 255).all() and tuple(roi[0]) == (0, 639, 0, 479)


def test_feeds_the_solver(fe, cuda_device):
    """Masked maps -> bt_frame_cache_store -> solve gives byte-identical poses to the same solve on unmasked maps masked by torch."""
    import torch
    from bundletrack_b200.optimizer import OptimizerGpu, SolveWindow
    H, W = 240, 320
    w = synth.make_window(11, n_frames=3, n_corr=400, H=H, W=W, K=tuple(v * 0.5 for v in synth.NOCS_K))
    rng = np.random.default_rng(5)
    raws = [(w.depth[k] + (w.depth[k] > 0) * rng.normal(0, 0.0003, w.depth[k].shape)).astype(np.float32) for k in range(3)]
    masks = []
    for k in range(3):
        m = ((w.depth[k] > 0) * 255).astype(np.uint8)
        m[:, : W // 2 - 10 + 5 * k] = 0                          # cut away part of the object so the mask changes the solve
        m[5:9, 5:9] = 255                                         # a distractor the hull mode drops
        masks.append(m)
    tin = [torch.from_numpy(r).to(cuda_device) for r in raws]
    tm = [torch.from_numpy(m).to(cuda_device) for m in masks]
    md = [torch.empty((H, W), device=cuda_device) for _ in range(3)]
    mn = [torch.empty((H, W, 4), device=cuda_device) for _ in range(3)]
    fg = [torch.empty((H, W), dtype=torch.uint8, device=cuda_device) for _ in range(3)]
    fe.process_masked(tin, tm, H, W, w.K, md, mn, fg, mode=HULL)
    ud = [torch.empty((H, W), device=cuda_device) for _ in range(3)]
    un = [torch.empty((H, W, 4), device=cuda_device) for _ in range(3)]
    fe.process(tin, H, W, w.K, ud, un)
    td = [torch.where(f != 0, d, torch.zeros_like(d)) for f, d in zip(fg, ud)]
    tn = [torch.where((f != 0)[..., None], v, torch.zeros_like(v)) for f, v in zip(fg, un)]
    torch.cuda.synchronize()
    assert any((f == 0).any().item() for f in fg) and all((f != 0).any().item() for f in fg)
    opt = OptimizerGpu(None, max_windows=1, max_frames=3, max_corr=400, H=H, W=W)
    opt.reserve_frame_cache(6, H, W)
    opt.store_frames([0, 1, 2], md, mn, H, W, w.K)
    opt.store_frames([3, 4, 5], td, tn, H, W, w.K)
    a = opt.optimizeWindows([SolveWindow(w.corr, H, W, md, mn, w.poses_init, w.K, cache_slots=[0, 1, 2])])[0]
    b = opt.optimizeWindows([SolveWindow(w.corr, H, W, td, tn, w.poses_init, w.K, cache_slots=[3, 4, 5])])[0]
    opt.close()
    assert np.isfinite(a).all() and a.tobytes() == b.tobytes()


def test_request_cases(fe, cuda_device):
    import torch
    H, W = 480, 640
    colour = so.test_colour(H, W)
    cases = {
        "small": (100, 180, 200, 260),        # side 80 < 400
        "tall": (10, 60, 0, 470),             # side 470 > 400
        "exact": (100, 500, 40, 300),         # side 400: a copy
        "borders": (0, 639, 0, 479),          # touches every border
        "gate": (100, 109, 50, 300),          # 9 columns: fails the gate, buffer untouched
        "empty": so.ROI_EMPTY,
    }
    fg = np.zeros((H, W), np.uint8)
    fg[::3, ::2] = 1
    fg[100:300, 150:400] = 255
    fg_dev = [torch.from_numpy(fg).to(cuda_device)]
    for name, roi in cases.items():
        r = torch.tensor([roi], dtype=torch.int32, device=cuda_device)
        got = _request(fe, [colour], fg_dev, cuda_device, roi=r, fill=201)[0]
        ref = so.lfnet_request(colour, fg, np.array(roi))
        if ref is None:
            assert (got == 201).all(), name
        else:
            assert np.array_equal(got, ref), name
    # a batch with one failing frame leaves only that frame's buffer as it was
    rois = torch.tensor([cases["small"], cases["gate"], cases["tall"]], dtype=torch.int32, device=cuda_device)
    got = _request(fe, [colour] * 3, fg_dev * 3, cuda_device, roi=rois, fill=9)
    assert np.array_equal(got[0], so.lfnet_request(colour, fg, np.array(cases["small"]))) and (got[1] == 9).all()
    assert np.array_equal(got[2], so.lfnet_request(colour, fg, np.array(cases["tall"])))


def test_argument_errors_and_repeatability(fe, cuda_device):
    import ctypes
    import torch
    lib = _lib.load()
    H, W = 64, 80
    raw = torch.full((H, W), 0.7, device=cuda_device)
    mask = torch.zeros((H, W), dtype=torch.uint8, device=cuda_device); mask[10:40, 20:60] = 255
    d, nn, fg = torch.empty_like(raw), torch.empty((H, W, 4), device=cuda_device), torch.empty_like(mask)
    roi = torch.empty((1, 4), dtype=torch.int32, device=cuda_device)
    P = lambda *ts: (ctypes.c_void_p * len(ts))(*[t.data_ptr() if t is not None else None for t in ts])
    K = synth.NOCS_K

    def call(mask_a, mode, fg_a, d_a=None, roi_p=None):
        return lib.bt_frames_preprocess_masked(fe.ctx, 1, P(raw), mask_a, mode, H, W, *[ctypes.c_float(v) for v in K], ctypes.byref(fe.params),
                                               d_a if d_a is not None else P(d), None, P(nn), fg_a, ctypes.c_void_p(roi.data_ptr()) if roi_p is None else roi_p, None)
    assert call(P(mask), HULL, P(fg)) == 0
    assert call(None, HULL, P(fg)) == _lib.BT_ERR_INVALID_ARG                      # NULL mask array
    assert call(P(mask), HULL, None) == _lib.BT_ERR_INVALID_ARG                    # NULL fg array
    assert call(P(mask), HULL, P(fg), roi_p=ctypes.c_void_p()) == _lib.BT_ERR_INVALID_ARG
    assert call(P(mask), HULL, (ctypes.c_void_p * 1)(None)) == _lib.BT_ERR_INVALID_ARG   # NULL fg map
    assert call(P(mask), HULL, P(fg), d_a=(ctypes.c_void_p * 1)(None)) == _lib.BT_ERR_INVALID_ARG
    assert call(P(mask), 7, P(fg)) == _lib.BT_ERR_INVALID_ARG                      # unknown mode
    assert call(P(mask), AS_IS, P(mask)) == _lib.BT_ERR_INVALID_ARG                # fg_out aliases the mask
    assert lib.bt_lfnet_request(fe.ctx, 1, None, P(fg), ctypes.c_void_p(roi.data_ptr()), H, W, P(fg), None) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_lfnet_request(fe.ctx, 1, P(fg), P(fg), ctypes.c_void_p(), H, W, P(fg), None) == _lib.BT_ERR_INVALID_ARG
    torch.cuda.synchronize()
    # two identical calls give identical bytes
    raws = [_raw(6, 480, 640)]
    masks = [synth.make_object_mask(6, 480, 640)]
    for mode in (HULL, AS_IS):
        a = _masked(fe, raws, masks, mode, cuda_device)
        b = _masked(fe, raws, masks, mode, cuda_device)
        for u, v in zip(a[:4], b[:4]):
            assert all(p.tobytes() == q.tobytes() for p, q in zip(u, v))
        assert np.array_equal(a[4], b[4])
