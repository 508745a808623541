"""The object model on the device (bt_tsdf_fuse / bt_tsdf_mesh, bundletrack_b200.recon) against oracle/recon_oracle.py bit for bit, its
refusals, the tracker's frame-depth accessor, and run_sequence's model_out: the pose files do not change, the mesh lies on the object."""
import ctypes
import os

import numpy as np
import pytest

from bundletrack_b200 import _lib, recon, sequence, synth
from oracle import recon_oracle as ro

K = (300.0, 300.0, 159.5, 119.5)
H, W = 240, 320
RADII = (0.06, 0.045, 0.035)


def _live():
    d, p, h = ctypes.c_longlong(), ctypes.c_longlong(), ctypes.c_int()
    assert _lib.load().bt_debug_live_resources(ctypes.byref(d), ctypes.byref(p), ctypes.byref(h)) == 0
    return d.value, p.value, h.value


def _views(dist=0.35, seed=3):
    rng = np.random.default_rng(seed)
    T = ro.views_around(dist)
    depths = [synth.render_ellipsoid(RADII, T[k], K, H, W, rng)[0] for k in range(len(T))]
    return depths, np.stack([np.linalg.inv(t) for t in T]).astype(np.float32)


def _assert_same(dev_grid, want, v, f, want_v, want_f):
    assert dev_grid["dims"] == want["dims"]
    for k in ("lo", "hi", "origin", "sum", "count"):
        assert np.array_equal(dev_grid[k], want[k]), k
    assert v.shape == want_v.shape and f.shape == want_f.shape
    assert v.tobytes() == want_v.tobytes() and np.array_equal(f, want_f)


def _fuse_both(tsdf, depths, cim, voxel, trunc, dev):
    import torch
    d = [torch.from_numpy(x).to(dev) for x in depths]
    torch.cuda.synchronize()
    tsdf.fuse(d, cim, K, voxel, trunc)
    v, f = tsdf.mesh()
    g = tsdf.grid()
    want = ro.fuse(depths, cim, K, voxel, trunc)
    return g, v, f, want


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["v4", "v3.5", "v3", "empty_frame", "single_frame", "border"])
def test_device_equals_oracle(case, cuda_device):
    depths, cim = _views(0.12 if case == "border" else 0.35)
    voxel = {"v3.5": 0.0035, "v3": 0.003}.get(case, 0.004)
    if case == "empty_frame":
        depths[5] = np.zeros_like(depths[5])
    if case == "single_frame":
        depths, cim = depths[:1], cim[:1]
    if case == "border":
        assert any((d[0] > 0).any() or (d[:, -1] > 0).any() for d in depths)
    tsdf = recon.Tsdf(len(depths), H, W, max_voxels=1 << 22, max_vertices=1 << 18, max_faces=1 << 19)
    try:
        g, v, f, want = _fuse_both(tsdf, depths, cim, voxel, 4 * voxel, cuda_device)
        want_v, want_f = ro.mesh(want, voxel)
        print(case, "dims", g["dims"], "samples", np.prod(g["dims"]), "verts", len(v), "faces", len(f))
        assert np.prod(g["dims"]) % 256 != 0 or case == "border"
        assert len(f) > 0
        _assert_same(g, want, v, f, want_v, want_f)
        v2, f2 = tsdf.mesh()                                   # same bytes again
        assert v2.tobytes() == v.tobytes() and f2.tobytes() == f.tobytes()
    finally:
        tsdf.close()


@pytest.mark.gpu
def test_refusals_leave_outputs_untouched(cuda_device):
    import torch
    lib = _lib.load()
    before = _live()
    depths, cim = _views()
    d = [torch.from_numpy(x).to(cuda_device) for x in depths]
    torch.cuda.synchronize()
    # calls before a reserve
    ctx = _lib.Context(0)
    nv, nf = ctypes.c_int(-7), ctypes.c_int(-7)
    p = _lib.TsdfParams(0.004, 0.016)
    assert lib.bt_tsdf_fuse(ctx, len(d), _lib.ptrs(d), _lib.ptr(cim), *K, H, W, ctypes.byref(p), None) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_tsdf_mesh(ctx, 1, 1, ctypes.byref(nv), ctypes.byref(nf), None) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_tsdf_grid(ctx, None, None, None, None, None) == _lib.BT_ERR_INVALID_ARG
    ctx.close()
    tsdf = recon.Tsdf(len(d), H, W, max_voxels=60000, max_vertices=1000, max_faces=100000)
    try:
        # a mesh before any fuse
        with pytest.raises(_lib.BtError) as e:
            tsdf.mesh()
        assert e.value.rc == _lib.BT_ERR_INVALID_ARG
        tsdf.fuse(d, cim, K, 0.004, 0.016)
        g0 = tsdf.grid()
        # too many samples: named dims, the grid as it was
        with pytest.raises(_lib.BtError, match=r"\d+ x \d+ x \d+ samples") as e:
            tsdf.fuse(d, cim, K, 0.002, 0.008)
        assert e.value.rc == _lib.BT_ERR_CAPACITY
        g1 = tsdf.grid()
        for k in ("dims", "origin", "lo", "hi", "sum", "count"):
            assert np.array_equal(g0[k], g1[k]), k
        # non-finite pose, n_frames < 1, wrong tensors
        bad = cim.copy()
        bad[2, 0, 3] = np.nan
        with pytest.raises(_lib.BtError, match="non-finite") as e:
            tsdf.fuse(d, bad, K, 0.004, 0.016)
        assert e.value.rc == _lib.BT_ERR_INVALID_ARG
        assert lib.bt_tsdf_fuse(tsdf.ctx, 0, _lib.ptrs(d), _lib.ptr(cim), *K, H, W, ctypes.byref(p), None) == _lib.BT_ERR_INVALID_ARG
        with pytest.raises(ValueError):
            tsdf.fuse([x.cpu() for x in d], cim, K)
        with pytest.raises(ValueError):
            tsdf.fuse([x.double() for x in d], cim, K)
        with pytest.raises(ValueError):
            tsdf.fuse([x[:-1] for x in d], cim, K)
        with pytest.raises(ValueError):
            tsdf.fuse(d[:-1], cim, K)
        # too many vertices (and, on a second context, faces): the counts reported, the outputs untouched
        tsdf.verts.fill_(-3.0)
        tsdf.faces.fill_(-3)
        nv, nf = ctypes.c_int(0), ctypes.c_int(0)
        rc = lib.bt_tsdf_mesh(tsdf.ctx, _lib.ptr(tsdf.verts), _lib.ptr(tsdf.faces), ctypes.byref(nv), ctypes.byref(nf), None)
        assert rc == _lib.BT_ERR_CAPACITY and nv.value > 1000 and nf.value > 1000
        torch.cuda.synchronize()
        assert bool((tsdf.verts == -3.0).all()) and bool((tsdf.faces == -3).all())
        want_v, want_f = ro.mesh(ro.fuse(depths, cim, K, 0.004, 0.016), 0.004)
        assert (nv.value, nf.value) == (len(want_v), len(want_f))
    finally:
        tsdf.close()
    small = recon.Tsdf(len(d), H, W, max_voxels=60000, max_vertices=1 << 16, max_faces=100)
    try:
        small.fuse(d, cim, K, 0.004, 0.016)
        small.faces.fill_(-3)
        with pytest.raises(_lib.BtError, match="faces") as e:
            small.mesh()
        assert e.value.rc == _lib.BT_ERR_CAPACITY
        assert bool((small.faces == -3).all())
    finally:
        small.close()
    # the reserve's limits
    ctx = _lib.Context(0)
    for args in ((0, H, W, 1000, 1, 1), (1, H, W, 4, 1, 1), (1, H, W, (1 << 27) + 1, 1, 1), (70000, H, W, 1000, 1, 1)):
        assert lib.bt_recon_reserve(ctx, *args) == _lib.BT_ERR_INVALID_ARG, args
    ctx.close()
    assert _live() == before


def _track(seq, dev, n_frames=None):
    """A Tracker over the sequence's frames (float depth), as run_sequence drives it; returns the open tracker."""
    import torch
    from bundletrack_b200.tracker import Tracker
    N = seq.n_frames if n_frames is None else n_frames
    Hs, Ws = seq.depth_raw.shape[1:]
    trk = Tracker(None, Hs, Ws, seq.K, 400, 6, mode=_lib.BT_MASK_LARGEST_HULL, max_keyframes=N)
    rq = torch.zeros((400, 400, 3), dtype=torch.uint8, device=dev)
    for i in range(N):
        d, m, c = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (seq.depth_raw[i], seq.mask[i], seq.colour[i]))
        st, _ = trk.begin_frame(d, m, c, rq, loader_id=i, first_pose=np.eye(4, dtype=np.float32) if i == 0 else None)
        if st == _lib.BT_FRAME_OTHER:
            f = seq.feats[i]
            trk.end_frame(f["kpts"], torch.from_numpy(f["desc"]).to(dev))
    return trk


@pytest.mark.gpu
def test_tracker_frame_depth_and_fuse_keyframes(cuda_device):
    import torch
    seq = synth.make_sequence(71, 14, H=H, W=W, n_feats=400)
    trk = _track(seq, cuda_device)
    lib = trk.lib
    try:
        ids, poses, kf = trk.state()
        assert kf.sum() >= 2
        p = ctypes.c_void_p()
        for bad in (-1, int(ids.max()) + 1):
            assert lib.bt_tracker_frame_depth(trk.t, bad, ctypes.byref(p)) == _lib.BT_ERR_INVALID_ARG
        assert lib.bt_tracker_frame_depth(trk.t, int(ids[0]), None) == _lib.BT_ERR_INVALID_ARG
        kid, kpose, addr = recon.keyframe_depths(trk)
        assert len(set(addr)) == len(addr)
        torch.cuda.synchronize()
        host = []
        for a in addr:
            h = np.empty((H, W), np.float32)
            _lib.check(lib.bt_memcpy_d2h(_lib.ptr(h), a, h.nbytes, None), "bt_memcpy_d2h")
            host.append(h)
        assert all((h > 0).sum() > 1000 for h in host)
        tsdf = recon.Tsdf(len(kid), H, W, device=0, stream=0)
        try:
            assert recon.fuse_keyframes(trk, tsdf, seq.K, 0.004, 0.016) == len(kid)
            v, f = tsdf.mesh()
            want = ro.fuse(host, kpose, seq.K, 0.004, 0.016)
            want_v, want_f = ro.mesh(want, 0.004)
            _assert_same(tsdf.grid(), want, v, f, want_v, want_f)
        finally:
            tsdf.close()
    finally:
        trk.close()


@pytest.mark.gpu
def test_run_sequence_model_out(tmp_path, cuda_device):
    """Pose files byte-identical with and without model_out; the mesh, moved into the object's frame, lies on the true ellipsoid."""
    N = 40
    seq = synth.make_sequence(81, N, H=480, W=640, n_feats=400, rot_deg=(4.0, 8.0))
    video = str(tmp_path / "data" / "synthvideo")
    synth.write_ycbineoat_video(seq, video)
    loader = sequence.YcbineoatVideo(video)

    def features(id_str, request, roi):
        f = seq.feats[int(id_str)]
        return f["kpts"], f["desc"]

    before = _live()
    out_a, out_b = str(tmp_path / "a"), str(tmp_path / "b")
    model = str(tmp_path / "model.ply")
    ra = sequence.run_sequence(loader, None, features, out_a, max_feats=400, device=0)
    rb = sequence.run_sequence(loader, None, features, out_b, max_feats=400, device=0, model_out=model)
    assert _live() == before
    assert [r[:2] for r in ra] == [r[:2] for r in rb]
    files = sorted(os.listdir(os.path.join(out_a, "poses")))
    assert len(files) == N and files == sorted(os.listdir(os.path.join(out_b, "poses")))
    for fn in files:
        assert open(os.path.join(out_a, "poses", fn), "rb").read() == open(os.path.join(out_b, "poses", fn), "rb").read(), fn
    with open(model, "rb") as fh:
        data = fh.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode()
    nv = int(head.split("element vertex ")[1].split()[0])
    nf = int(head.split("element face ")[1].split()[0])
    assert nv > 1000 and nf > 1000 and len(data) == end + 12 * nv + 13 * nf
    v = np.frombuffer(data, "<f4", 3 * nv, end).reshape(nv, 3).astype(np.float64)
    # the model frame is camera 0's (the video's first annotated pose is the identity); the object frame is ob_in_cam0^-1 of it
    G = np.linalg.inv(seq.ob_in_cam0)
    obj = v @ G[:3, :3].T + G[:3, 3]
    d = ro.ellipsoid_distance(obj, seq.radii) * 1000
    med, p95 = float(np.median(d)), float(np.percentile(d, 95))
    print(f"model_out: {nv} vertices, {nf} faces; distance to the true ellipsoid median {med:.3f} mm, p95 {p95:.3f} mm; "
          f"wall per frame {np.mean([r[2] for r in ra]) * 1e3:.1f} / {np.mean([r[2] for r in rb]) * 1e3:.1f} ms")
    assert med < 3.0 and p95 < 7.5                            # measured on an H100: 2.33 mm and 5.53 mm
