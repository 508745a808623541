"""Destroying a context or a tracker frees everything it made: every device buffer, pinned block, event and stream, counted exactly by
bt_debug_live_resources (what the library's handle types hold, across the process).  Each case uses every module once, so each state's
lazily made events (upload guards, timing, the streaming pipe, the staging copy stream) exist when the context goes."""
import ctypes
import gc

import numpy as np
import pytest

from bundletrack_b200 import _lib, synth
from bundletrack_b200.optimizer import OptimizerGpu, SolveWindow

pytestmark = pytest.mark.gpu

YML = {"feature_corres": {"max_dist_no_neighbor": 0.02, "max_normal_no_neighbor": 45, "max_dist_neighbor": 10000, "max_normal_neighbor": 180},
       "ransac": {"max_iter": 200, "inlier_dist": 0.01}}


def _live():
    d, p, h = ctypes.c_longlong(-1), ctypes.c_longlong(-1), ctypes.c_int(-1)
    _lib.check(_lib.load().bt_debug_live_resources(ctypes.byref(d), ctypes.byref(p), ctypes.byref(h)), "bt_debug_live_resources")
    return d.value, p.value, h.value


@pytest.fixture
def before(cuda_device):
    """The counts with nothing of this case alive; no earlier test's __del__ may run (and free its context) while the case runs."""
    gc.collect()
    gc.disable()
    try:
        yield _live()
    finally:
        gc.enable()


def _grew(now, base):
    return all(n > b for n, b in zip(now, base))


def _feature_frames(dev, n=3, n_feats=300):
    import torch
    w = synth.make_window(31, n_frames=n, n_corr=10)
    fr = synth.make_feature_frames(w, n_feats, seed=31)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return w, [{"kpts": t(fr[k]["kpts"]), "desc": t(fr[k]["desc"]), "depth": t(w.depth[k]), "normal": t(w.normal[k]), "pose": w.poses_init[k],
                "id": k, "window_index": k} for k in range(n)]


def _masked_front_end(fe, dev, H, W):
    import torch
    raw, K = synth.make_raw_depth(5, H, W)
    mask = np.zeros((H, W), np.uint8)
    mask[H // 4:3 * H // 4, W // 4:3 * W // 4] = 255
    mask[2:6, 2:6] = 255                                     # a second, smaller blob: largest-hull mode drops it
    d, n = torch.empty((H, W), device=dev), torch.empty((H, W, 4), device=dev)
    fg = torch.empty((H, W), dtype=torch.uint8, device=dev)
    fe.process_masked([torch.from_numpy(raw).to(dev)], [torch.from_numpy(mask).to(dev)], H, W, K, [d], [n], [fg], mode=_lib.BT_MASK_LARGEST_HULL)
    colour = torch.full((H, W, 3), 90, dtype=torch.uint8, device=dev)
    req = torch.zeros((400, 400, 3), dtype=torch.uint8, device=dev)
    fe.lfnet_request([colour], [fg], H, W, [req])


@pytest.mark.parametrize("grow", [False, True], ids=["reserved_once", "reserved_twice"])
def test_context_destroy_frees_every_module(before, cuda_device, grow):
    import torch
    from bundletrack_b200.frontend import FrameFrontEnd
    from bundletrack_b200.matcher import FindCorres, MatchPipeline, Ransac
    from bundletrack_b200.metrics import PoseMetrics
    dev = cuda_device
    mp = MatchPipeline(YML, max_pairs=4, max_feats=512)          # owns the context every module below shares
    lib, ctx = mp.lib, mp.ctx
    # solver + frame cache: one fused call and one begin / end pair, timing and the profile on
    sw = synth.make_window(7, n_frames=4, n_corr=400)
    depth = [torch.from_numpy(sw.depth[k]).to(dev) for k in range(4)]
    normal = [torch.from_numpy(sw.normal[k]).to(dev) for k in range(4)]
    opt = OptimizerGpu(ctx=ctx, max_windows=1, max_frames=8, max_corr=4096, H=sw.H, W=sw.W)
    opt.enable_timing()
    opt.enable_profile(1000)
    opt.reserve_frame_cache(4)
    opt.store_frames([0, 1, 2, 3], depth, normal, sw.H, sw.W, sw.K)
    win = SolveWindow(sw.corr, sw.H, sw.W, depth, normal, sw.poses_init, sw.K)
    assert np.isfinite(opt.optimizeWindows([win])[0]).all()
    opt.timing_ms()
    opt.begin([win])
    assert np.isfinite(opt.end()[0]).all()
    # pipeline + descriptor pool + match cache + device map-point table: one findCorres call and its cache put, kNN timing on
    w, frames = _feature_frames(dev)
    mp.pool_reserve(3)
    for k, f in enumerate(frames):
        mp.pool_store(k, f["desc"])
    fc = FindCorres(mp, max_pairs_cached=16, max_frames=8)
    _lib.check(lib.bt_knn_enable_timing(ctx, 1), "bt_knn_enable_timing")
    fc.find_corres([(frames[1], frames[0]), (frames[2], frames[1]), (frames[2], frames[0])], [(1, 0), (2, 1), (2, 0)], w.H, w.W, w.K)
    fc.window_entries(frames, dev)
    # RANSAC on host-listed pairs
    rng = np.random.default_rng(3)
    a = rng.normal(size=(200, 4)).astype(np.float32)
    r = Ransac(ctx=ctx, max_pairs=2, max_pts=256, max_trials=100)
    r.ransac_pairs([torch.from_numpy(a).to(dev)], [torch.from_numpy(a + 0.001).to(dev)], n_trials=100, dist_thresh=0.01)
    # masked front end in largest-hull mode (grows the segmentation scratch) + the LF-Net request
    fe = FrameFrontEnd(ctx=ctx)
    _masked_front_end(fe, dev, 120, 160)
    # pose metrics
    pm = PoseMetrics(500, 4, ctx=ctx)
    pm(rng.normal(size=(500, 3)), np.tile(np.eye(4), (4, 1, 1)), np.tile(np.eye(4), (4, 1, 1)))
    torch.cuda.synchronize()
    alive = _live()
    assert _grew(alive, before), (alive, before)
    grown = alive
    if grow:
        opt.reserve(2, 10, 8192, sw.H, sw.W)
        opt.reserve_frame_cache(8)
        _lib.check(lib.bt_pipeline_reserve(ctx, 8, 1024, 256, 300), "bt_pipeline_reserve")
        mp.pool_reserve(8)
        _lib.check(lib.bt_tracks_dev_reserve_ex(ctx, 16, 1024, 32768), "bt_tracks_dev_reserve_ex")
        _lib.check(lib.bt_match_cache_reserve(ctx, 64, 3 * 1024), "bt_match_cache_reserve")
        _lib.check(lib.bt_ransac_reserve(ctx, 16, 4096, 400), "bt_ransac_reserve")
        _lib.check(lib.bt_metrics_reserve(ctx, 5000, 16), "bt_metrics_reserve")
        _masked_front_end(fe, dev, 240, 320)                 # the front end grows on demand
        torch.cuda.synchronize()
        grown = _live()
        assert grown[0] > alive[0] and grown[1] > alive[1], (grown, alive)
    for o in (pm, fe, r, opt):
        o.close()                                            # (borrowed context: none of these frees it)
    assert _live() == grown
    mp.close()
    assert _live() == before


def _front_end_run(fe, dev):
    """One bt_frames_preprocess call through fe; returns its depth and normal maps."""
    import torch
    raw, K = synth.make_raw_depth(5, 120, 160)
    d, n = torch.empty((120, 160), device=dev), torch.empty((120, 160, 4), device=dev)
    fe.process([torch.from_numpy(raw).to(dev)], 120, 160, K, [d], [n])
    torch.cuda.synchronize()
    return d.cpu().numpy(), n.cpu().numpy()


def test_borrower_after_owner_close_is_refused(before, cuda_device):
    """bench.py's sharing: a front end on the optimizer's context.  Once the owner closes the context, the borrower's call passes NULL and
    the library refuses it; no call reaches the destroyed context."""
    from bundletrack_b200.frontend import FrameFrontEnd
    opt = OptimizerGpu(max_windows=1, max_frames=4, max_corr=1024, H=120, W=160)
    fe = FrameFrontEnd(ctx=opt.ctx)
    _front_end_run(fe, cuda_device)
    opt.close()
    assert _live() == before
    with pytest.raises(_lib.BtError) as e:
        _front_end_run(fe, cuda_device)
    assert e.value.rc == _lib.BT_ERR_INVALID_ARG
    fe.close()


def test_borrower_outlives_its_owner(before, cuda_device):
    """Deleting the owner leaves the shared context to the borrower, which keeps working; the context goes with the last holder."""
    from bundletrack_b200.frontend import FrameFrontEnd
    opt = OptimizerGpu(max_windows=1, max_frames=4, max_corr=1024, H=120, W=160)
    fe = FrameFrontEnd(ctx=opt.ctx)
    want = _front_end_run(fe, cuda_device)
    del opt
    assert _grew(_live()[:1], before[:1])
    got = _front_end_run(fe, cuda_device)
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    del fe
    assert _live() == before


def test_tracker_destroy_frees_everything(before, cuda_device):
    import torch
    from bundletrack_b200.tracker import Tracker
    H, W, feats = 240, 320, 400
    seq = synth.make_sequence(11, 5, H=H, W=W, n_feats=feats)
    dev = cuda_device
    trk = Tracker(None, H, W, seq.K, feats, 8)
    assert _grew(_live()[:2], before[:2])                   # (events and the copy stream are made on first use)
    for k in range(seq.n_frames):
        d, m, c = (torch.from_numpy(np.ascontiguousarray(a[k])).to(dev) for a in (seq.depth_raw, seq.mask, seq.colour))
        rq = torch.zeros((400, 400, 3), dtype=torch.uint8, device=dev)
        st, _ = trk.begin_frame(d, m, c, rq, loader_id=0, first_pose=seq.poses_gt[k])
        if st == _lib.BT_FRAME_OTHER:
            trk.end_frame(seq.feats[k]["kpts"], torch.from_numpy(seq.feats[k]["desc"]).to(dev))
    torch.cuda.synchronize()
    assert len(trk.state()[0]) >= 2 and _grew(_live(), before)
    trk.close()
    assert _live() == before


def test_refused_tracker_create_leaves_nothing(before, cuda_device):
    from bundletrack_b200.tracker import tracker_params
    lib = _lib.load()
    p = tracker_params(None, 240, 320, synth.NOCS_K, 400, 1)       # max_frames_alive 1: refused before anything is made
    t = ctypes.c_void_p()
    assert lib.bt_tracker_create(ctypes.byref(t), 0, ctypes.byref(p)) == _lib.BT_ERR_INVALID_ARG
    assert not t.value
    assert _live() == before
