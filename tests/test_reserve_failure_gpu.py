"""A reserve that fails partway (an allocation refused by bt_debug_fail_alloc, or a real out-of-memory) leaves its module refusing every
call with BT_ERR_INVALID_ARG and a text that names the reserve, without launching anything or allocating, until a reserve succeeds; then
the module serves again and gives what it gave before.  A reserve refused for bad arguments leaves the previous reservation serving."""
import ctypes

import numpy as np
import pytest

from bundletrack_b200 import _lib, synth

pytestmark = pytest.mark.gpu

BT_ERR_CUDA, BT_ERR_UNSUPPORTED = -3, -5          # (include/bundletrack_b200.h)
YML = {"feature_corres": {"max_dist_no_neighbor": 0.02, "max_normal_no_neighbor": 45, "max_dist_neighbor": 10000, "max_normal_neighbor": 180},
       "ransac": {"max_iter": 200, "inlier_dist": 0.01}}

# An argument block for refused calls: each 8-byte word holds the block's own address, so every pointer argument, and every pointer an
# array argument holds, is non-NULL, and every number read from it is finite.  A refused call reads no further than its argument checks.
_WORDS = np.zeros(1 << 16, np.uint64)
_WORDS[:] = _WORDS.ctypes.data


def _args(name):
    out = []
    for t in _lib.PROTOTYPES[name][1][1:]:
        if t in (ctypes.c_float, ctypes.c_double):
            out.append(1.0)
        elif t in (ctypes.c_int, ctypes.c_longlong, ctypes.c_size_t, ctypes.c_uint64):
            out.append(1)
        elif t is ctypes.c_void_p:
            out.append(_WORDS.ctypes.data)
        else:
            out.append(ctypes.cast(_WORDS.ctypes.data, t))
    return out


def _rc(f):
    try:
        f()
        return _lib.BT_OK
    except _lib.BtError as e:
        return e.rc


def _live():
    d, p, h = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_int()
    _lib.check(_lib.load().bt_debug_live_resources(ctypes.byref(d), ctypes.byref(p), ctypes.byref(h)), "bt_debug_live_resources")
    return d.value, p.value, h.value


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(y), equal_nan=True)


def _cases(dev):
    """The context first, then per module: (name, the reserve its refusals name, its entry points, a good call returning host arrays, a
    larger reserve returning its rc)."""
    import torch
    from bundletrack_b200 import lfnet, vos
    from bundletrack_b200.matcher import DeviceTracks, FindCorres, KnnMatcher, MatchPipeline, Ransac
    from bundletrack_b200.metrics import NocsMetrics, PoseMetrics
    from bundletrack_b200.optimizer import OptimizerGpu, SolveWindow
    from bundletrack_b200.overlay import VoxelGrid
    from oracle import lfnet_oracle as lo
    from oracle import vos_oracle as vo
    mp = MatchPipeline(YML, max_pairs=2, max_feats=512)
    lib, ctx = mp.lib, mp.ctx
    yield ctx
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    host = lambda xs: [x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x) for x in xs]
    # solver and frame cache
    sw = synth.make_window(7, n_frames=4, n_corr=400)
    depth, normal = [t(d) for d in sw.depth], [t(n) for n in sw.normal]
    opt = OptimizerGpu(ctx=ctx, max_windows=1, max_frames=4, max_corr=1024, H=sw.H, W=sw.W)
    opt.reserve_frame_cache(2)
    win = SolveWindow(sw.corr, sw.H, sw.W, depth, normal, sw.poses_init, sw.K)
    solver_calls = ["bt_solve_enable_debug", "bt_solve_enable_timing", "bt_solve_get_timing", "bt_solve_stage", "bt_solve_run", "bt_solve_fetch",
                    "bt_solve_windows", "bt_solve_windows_begin", "bt_solve_windows_end", "bt_solve_get_host_timing", "bt_frame_cache_reserve",
                    "bt_frame_cache_store", "bt_solve_get_stats", "bt_solve_enable_profile", "bt_solve_get_profile", "bt_solve_debug_counts",
                    "bt_solve_debug_dense", "bt_solve_debug_system"]
    yield ("solver", "bt_solver_reserve", solver_calls, lambda: [opt.optimizeWindows([win])[0]],
           lambda: _rc(lambda: opt.reserve(2, 8, 4096, sw.H, sw.W)))
    yield ("frame cache", "bt_frame_cache_reserve", ["bt_frame_cache_store"],
           lambda: (opt.store_frames([0, 1], depth[:2], normal[:2], sw.H, sw.W, sw.K), [opt.optimizeWindows([win])[0]])[1],
           lambda: _rc(lambda: opt.reserve_frame_cache(8)))
    # matcher, descriptor pool, RANSAC
    a, b, _, _ = synth.make_descriptors(3, 300, 420)
    km = KnnMatcher(max_pairs=2, max_feats=512, ctx=ctx)
    km.pool_reserve(2)
    knn_calls = ["bt_knn_match_pairs", "bt_knn_match_slots", "bt_desc_pool_reserve", "bt_desc_pool_store", "bt_knn_debug_force_fallback",
                 "bt_knn_enable_timing", "bt_knn_get_timing"]
    knn_good = lambda: host(km.knn_match_pairs([(t(a), t(b))], k=5)[0]) + host(km.knn_match_pairs([(t(b), t(a))], k=3)[1])
    yield ("matcher", "bt_matcher_reserve", knn_calls, knn_good, lambda: lib.bt_matcher_reserve(ctx, 4, 1024, a.shape[1]))
    # (re-allocating the pool moves the matcher's own slots too: a failed pool reserve leaves the matcher to bt_matcher_reserve)
    yield ("descriptor pool", "bt_matcher_reserve", knn_calls,
           lambda: (km.pool_store(0, t(a)), km.pool_store(1, t(b)), host(km.knn_match_slots([(0, 1)], [(300, 420)])[0]))[2],
           lambda: lib.bt_matcher_reserve(ctx, 2, 512, a.shape[1]) or lib.bt_desc_pool_reserve(ctx, 8))
    rng = np.random.default_rng(3)
    pa = rng.normal(size=(200, 4)).astype(np.float32)
    r = Ransac(ctx=ctx, max_pairs=2, max_pts=256, max_trials=100)
    yield ("ransac", "bt_ransac_reserve", ["bt_ransac_pairs", "bt_ransac_debug", "bt_ransac_debug_trials"],
           lambda: host(r.ransac_pairs([t(pa)], [t(pa + 0.001)], n_trials=100, dist_thresh=0.01)), lambda: lib.bt_ransac_reserve(ctx, 4, 1024, 200))
    # pipeline, match cache, map-point table: one findCorres call on fresh state
    w = synth.make_window(31, n_frames=3, n_corr=10)
    fr = synth.make_feature_frames(w, 300, seed=31)
    frames = [{"kpts": t(fr[k]["kpts"]), "desc": t(fr[k]["desc"]), "depth": t(w.depth[k]), "normal": t(w.normal[k]), "pose": w.poses_init[k],
               "id": k, "window_index": k} for k in range(3)]
    fc = FindCorres(mp, max_pairs_cached=16, max_frames=8)

    def find_corres():
        _lib.check(lib.bt_pipeline_reserve(ctx, 4, 512, 256, 200), "bt_pipeline_reserve")
        mp.pool_reserve(3)
        for k, f in enumerate(frames):
            mp.pool_store(k, f["desc"])
        _lib.check(lib.bt_match_cache_reserve(ctx, 16, 3 * 512), "bt_match_cache_reserve")               # (empties the cache)
        _lib.check(lib.bt_tracks_dev_reserve_ex(ctx, 8, 512, 4096), "bt_tracks_dev_reserve_ex")           # (empties the table)
        fc.find_corres([(frames[1], frames[0]), (frames[2], frames[1]), (frames[2], frames[0])], [(1, 0), (2, 1), (2, 0)], w.H, w.W, w.K)
        entries, (off, cnt, _, _) = fc.window_entries(frames, dev)
        return host([entries[:int(off[-1] + cnt[-1])], off, cnt])

    yield ("pipeline", "bt_pipeline_reserve", ["bt_prune_mutual_pairs", "bt_match_pairs", "bt_match_pairs_pool", "bt_match_pairs_ex",
                                               "bt_find_corres_pairs"], find_corres, lambda: lib.bt_pipeline_reserve(ctx, 8, 512, 256, 300))
    yield ("match cache", "bt_match_cache_reserve", ["bt_match_cache_put", "bt_match_cache_has", "bt_match_cache_status", "bt_match_cache_usage",
                                                     "bt_match_cache_gather", "bt_match_cache_forget_frame"],
           lambda: (find_corres(), [fc.has(1, 0), fc.has(2, 0)])[1], lambda: lib.bt_match_cache_reserve(ctx, 64, 3 * 1024))
    tr = DeviceTracks(ctx=ctx, max_frames=8, max_keys_per_frame=256, max_points=2048)

    def tracks_good():
        _lib.check(lib.bt_tracks_dev_reserve_ex(ctx, 8, 256, 2048), "bt_tracks_dev_reserve_ex")
        uv = np.random.default_rng(9).integers(0, 100, size=(50, 4)).astype(np.float32)
        tr.update_pair(1, 0, uv)
        tr.update_pair(2, 1, uv[::-1])
        return [tr.propagate(2, 0, uv[:10]), np.array(tr.stats())]

    yield ("map-point table", "bt_tracks_dev_reserve", ["bt_tracks_dev_update_pair", "bt_tracks_dev_propagate", "bt_tracks_dev_forget_frame",
                                                        "bt_tracks_dev_stats", "bt_find_corres_pairs"],
           tracks_good, lambda: lib.bt_tracks_dev_reserve_ex(ctx, 16, 1024, 32768))
    # metrics, NOCS, overlay
    pm = PoseMetrics(500, 4, ctx=ctx)
    pts, P = rng.normal(size=(500, 3)), np.tile(np.eye(4), (4, 1, 1))
    G = P.copy()
    G[:, :3, 3] = rng.normal(size=(4, 3)) * 0.01
    yield ("metrics", "bt_metrics_reserve", ["bt_pose_metrics"], lambda: list(pm(pts, P, G)), lambda: lib.bt_metrics_reserve(ctx, 5000, 16))
    nm = NocsMetrics(8, ctx=ctx)
    corners = np.array([[x, y, z] for x in (-50, 50) for y in (-40, 40) for z in (-30, 30)], np.float64)
    Pn = np.tile(np.eye(4), (3, 1, 1))
    Pn[:, :3, 3] = [[0, 0, 500], [5, 0, 500], [0, 9, 510]]
    yield ("nocs", "bt_nocs_reserve", ["bt_nocs_metrics"], lambda: list(nm(Pn, Pn[::-1].copy(), corners, [0, 1, 0])),
           lambda: lib.bt_nocs_reserve(ctx, 64))
    vg = VoxelGrid(2000, 2, ctx=ctx)
    cloud = rng.uniform(-0.1, 0.1, size=(1500, 3)).astype(np.float32)
    yield ("overlay", "bt_overlay_reserve", ["bt_voxel_downsample", "bt_pose_overlay"], lambda: vg([cloud, cloud[:700]], 0.01),
           lambda: lib.bt_overlay_reserve(ctx, 20000, 8))
    _lib.check(lib.bt_match_viz_reserve(ctx, 2, 16), "bt_match_viz_reserve")
    yield ("match images", "bt_match_viz_reserve", ["bt_match_viz"], lambda: [_match_viz(lib, ctx, dev)], lambda: lib.bt_match_viz_reserve(ctx, 8, 4096))
    # LF-Net and VOS (their weights stay loaded through a reserve of the same network; VOS grows its frame ring, which two frames do not
    # reach, so the outputs stay those of the first reservation)
    hp = dict(lfnet.DEFAULTS)
    net = lfnet.LfnetDevice(lo.random_weights(lfnet.weight_shapes(hp), 11), hp, max_images=1, ctx=ctx)
    req = t(rng.integers(0, 256, size=(400, 400, 3), dtype=np.uint8))
    yield ("lfnet", "bt_lfnet_reserve", ["bt_lfnet_load_weights", "bt_lfnet_detect", "bt_lfnet_enable_timing", "bt_lfnet_get_timing",
                                         "bt_lfnet_debug_maps"], lambda: host(net.detect([req])), lambda: lib.bt_lfnet_reserve(ctx, ctypes.byref(net.params), 2))
    sd = vo.random_state_dict(7)
    sd = {k[len("module."):]: v.double().numpy() for k, v in sd.items() if not k.endswith("num_batches_tracked")}
    v = vos.VosDevice(sd, {}, 40, 56, ctx=ctx)
    colour = [t(rng.integers(0, 256, size=(40, 56, 3), dtype=np.uint8)) for _ in range(2)]
    m0 = np.zeros((40, 56), np.uint8)
    m0[10:30, 12:40] = 3
    yield ("vos", "bt_vos_reserve", ["bt_vos_load_weights", "bt_vos_begin", "bt_vos_next", "bt_vos_enable_timing", "bt_vos_get_timing",
                                     "bt_vos_debug"], lambda: host([v.begin(colour[0], t(m0)), v.next(colour[1])]),
           lambda: lib.bt_vos_reserve(ctx, ctypes.byref(vos.params_struct(dict(v.params, range=v.params["range"] + 64))), 40, 56))
    for o in (v, net, vg, nm, pm, tr, r, km, opt):
        o.close()
    mp.close()


def _match_viz(lib, ctx, dev):
    import torch
    img = torch.full((60, 80, 3), 100, dtype=torch.uint8, device=dev)
    uv = torch.tensor([[10.0, 10.0, 20.0, 30.0], [40.0, 50.0, 5.0, 5.0]], device=dev)
    d = _lib.MatchVizDesc()
    d.colour_a = d.colour_b = _lib.ptr(img)
    d.H_a = d.H_b = 60
    d.W_a = d.W_b = 80
    for k, v in enumerate((0, 80, 0, 60)):
        d.roi_a[k] = d.roi_b[k] = v
    d.uv, d.n = _lib.ptr(uv), 2
    rows, cols = ctypes.c_int(), ctypes.c_int()
    _lib.check(lib.bt_match_viz_shape(ctypes.addressof(d.roi_a), ctypes.addressof(d.roi_b), ctypes.byref(rows), ctypes.byref(cols)), "bt_match_viz_shape")
    out = torch.empty((rows.value, cols.value, 3), dtype=torch.uint8, device=dev)
    _lib.check(lib.bt_match_viz(ctx, 1, ctypes.byref(d), _lib.ptrs([out]), None), "bt_match_viz")
    return out.cpu().numpy()


def test_failed_reserve_refuses_until_a_reserve_succeeds(cuda_device):
    import torch
    lib = _lib.load()
    cases = _cases(cuda_device)
    ctx = next(cases)
    for name, reserve, calls, good, grow in cases:
        want = good()
        torch.cuda.synchronize()
        for n in range(1, 1000):
            _lib.check(lib.bt_debug_fail_alloc(n), "bt_debug_fail_alloc")
            rc = grow()
            _lib.check(lib.bt_debug_fail_alloc(0), "bt_debug_fail_alloc")
            if rc == _lib.BT_OK:
                break
            assert rc == BT_ERR_CUDA and b"bt_debug_fail_alloc" in lib.bt_last_error(), (name, n, rc, lib.bt_last_error())
            torch.cuda.synchronize()
            live = _live()
            for call in calls:
                assert getattr(lib, call)(ctx, *_args(call)) == _lib.BT_ERR_INVALID_ARG, (name, n, call, lib.bt_last_error())
                assert reserve.encode() in lib.bt_last_error(), (name, n, call, lib.bt_last_error())
            torch.cuda.synchronize()
            assert _live() == live, (name, n)
        else:
            pytest.fail(f"{name}: the reserve never succeeded")
        assert n > 1, name                                   # (at least one allocation failed)
        _same(good(), want)
        torch.cuda.synchronize()


def test_refused_arguments_keep_the_reservation(cuda_device):
    import torch
    from bundletrack_b200.matcher import Ransac
    r = Ransac(max_pairs=2, max_pts=256, max_trials=100)
    pa = np.random.default_rng(5).normal(size=(200, 4)).astype(np.float32)
    run = lambda: [x.cpu().numpy() for x in r.ransac_pairs([torch.from_numpy(pa).cuda()], [torch.from_numpy(pa + 0.001).cuda()], n_trials=100, dist_thresh=0.01)]
    want = run()
    lib = r.lib
    assert lib.bt_ransac_reserve(r.ctx, 4, 1024, 0) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_pipeline_reserve(r.ctx, 4, 512, 256, 0) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_pipeline_reserve(r.ctx, 4, 512, 128, 200) == BT_ERR_UNSUPPORTED
    assert lib.bt_metrics_reserve(r.ctx, 0, 4) == _lib.BT_ERR_INVALID_ARG
    _same(run(), want)
    r.close()


def test_out_of_memory_solver_reserve_leaves_no_stale_error(cuda_device):
    """The first staging block of this reserve asks for tens of terabytes (2^16 windows of 2^24 correspondences) while the sizes before it
    stay far from int overflow: the reserve fails in cudaMalloc, and that error must not come back from the next, unrelated call."""
    from bundletrack_b200.optimizer import OptimizerGpu, SolveWindow
    w = synth.make_window(7, n_frames=2, n_corr=100, H=64, W=64)
    opt = OptimizerGpu(max_windows=1, max_frames=2, max_corr=1024, H=64, W=64)
    with pytest.raises(_lib.BtError) as e:
        opt.reserve(1 << 16, 2, 1 << 24, 64, 64)
    assert e.value.rc == BT_ERR_CUDA
    opt.reserve(1, 2, 1024, 64, 64)
    import torch
    depth = [torch.from_numpy(d).cuda() for d in w.depth]
    normal = [torch.from_numpy(n).cuda() for n in w.normal]
    assert np.isfinite(opt.optimizeWindows([SolveWindow(w.corr, w.H, w.W, depth, normal, w.poses_init, w.K)])[0]).all()
    opt.close()
