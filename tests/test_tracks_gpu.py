"""The device map-point table (bt_tracks_dev_*) against the host table (bt_tracks), and the ordered multi-pair findCorres call
(bt_find_corres_pairs) against the pair-by-pair composition of bt_match_pairs_ex with the host table."""
import ctypes

import numpy as np
import pytest

from bundletrack_b200 import _lib, synth

pytestmark = pytest.mark.gpu

BT_ERR_CAPACITY = -2


def _bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


# ------------------------------------------------------------------------------------------------ 1. table parity
def _key_pool(rng, n):
    """Coordinates that collide on purpose: +0 and -0, values one ulp apart, a few repeats."""
    base = rng.uniform(0.0, 640.0, n).astype(np.float32)
    base[:4] = [0.0, -0.0, 1.0, np.nextafter(np.float32(1.0), np.float32(2.0))]
    base[4] = np.nextafter(base[5], np.float32(1e9))
    base[6] = np.nextafter(base[7], np.float32(-1e9))
    return base


def _run_parity(seed, n_ops, max_keys, max_list, pool_u, pool_v, n_frames=10):
    """Seeded random updates / propagations / forgets through the host and the device table; every propagation byte-identical.
    The keys of a frame are the kA and kB of every entry that named it since it was last forgotten (an entry is either skipped because
    both keys are in, or puts them in); the pools keep that below max_keys, so the device never runs out of room where the host does not."""
    from bundletrack_b200.matcher import DeviceTracks
    from bundletrack_b200.policy import Tracks
    rng = np.random.default_rng(seed)
    assert len(pool_u) * len(pool_v) <= max_keys
    host, dev = Tracks(), DeviceTracks(max_frames=16, max_keys_per_frame=max_keys, max_points=64 * max_keys)
    keys = {f: set() for f in range(n_frames)}       # normalised keys per frame
    anchors = set()                                   # frames some point is anchored at
    c = dict(ops=0, prop=0, nonempty=0, forgot_anchor=0, long_list=0, max_keys_propagated=0)

    def draw(n):
        uv = np.stack([pool_u[rng.integers(0, len(pool_u), n)], pool_v[rng.integers(0, len(pool_v), n)],
                       pool_u[rng.integers(0, len(pool_u), n)], pool_v[rng.integers(0, len(pool_v), n)]], 1).astype(np.float32)
        if n > 3:   # repeated kA and repeated kB within the list
            uv[rng.integers(0, n)][:2] = uv[0][:2]
            uv[rng.integers(0, n)][2:] = uv[1][2:]
        return np.ascontiguousarray(uv)

    for _ in range(n_ops):
        r = rng.random()
        alive = [f for f in range(n_frames) if keys[f]]
        if r < 0.5 or len(alive) < 2:
            a, b = (int(x) for x in sorted(rng.choice(n_frames, 2, replace=False))[::-1])
            n = 0 if rng.random() < 0.1 else int(rng.integers(1, max_list + 1))
            uv = draw(n)
            inl = (rng.random(n) < 0.8).astype(np.uint8) if rng.random() < 0.3 else None
            host.update_pair(a, b, uv, inl)
            dev.update_pair(a, b, uv, inl)
            kept = uv if inl is None else uv[inl.astype(bool)]
            keys[a] |= {(float(u) + 0.0, float(v) + 0.0) for u, v in kept[:, :2]}
            keys[b] |= {(float(u) + 0.0, float(v) + 0.0) for u, v in kept[:, 2:]}
            anchors |= {b} if len(kept) else set()
            c["long_list"] += len(kept) > 1024
        elif r < 0.9:
            a, b = (int(x) for x in sorted(rng.choice(n_frames, 2, replace=False))[::-1])
            ex = draw(int(rng.integers(0, 6))) if rng.random() < 0.3 else np.zeros((0, 4), np.float32)
            want = host.propagate(a, b, ex)
            got = dev.propagate(a, b, ex)
            assert got.shape == want.shape and np.array_equal(_bits(got), _bits(want)), (a, b)
            c["prop"] += 1
            c["nonempty"] += len(want) > 0
            if len(want):
                c["max_keys_propagated"] = max(c["max_keys_propagated"], len(keys[a]))
        else:
            f = int(rng.choice(alive))
            c["forgot_anchor"] += f in anchors
            host.forget_frame(f)
            dev.forget_frame(f)           # the id comes back in later updates: the slot is reused
            keys[f] = set()
            anchors.discard(f)
        c["ops"] += 1
    assert host.stats() == dev.stats()
    dev.close()
    return c


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_device_table_equals_host_table(cuda_device, seed):
    """Short lists over a small key pool: many collisions, repeated keys, +-0, keys one ulp apart."""
    rng = np.random.default_rng(100 + seed)
    pool = _key_pool(rng, 24)
    c = _run_parity(seed, 360, 1024, 40, pool, pool)
    assert c["ops"] >= 300 and c["prop"] >= 80 and c["nonempty"] >= 20 and c["forgot_anchor"] >= 5, c


def test_device_table_long_lists_and_full_frames(cuda_device):
    """Lists longer than one CTA (the update's multi-chunk scans), frames with more keys than one CTA and more than half of a
    max_keys_per_frame that is not a power of two (propagate's sort runs over the next power of two)."""
    rng = np.random.default_rng(7)
    pool_u, pool_v = _key_pool(rng, 50), _key_pool(rng, 40)        # 2000 distinct keys at most
    c = _run_parity(4, 60, 2000, 1800, pool_u, pool_v, n_frames=6)
    assert c["long_list"] >= 5 and c["max_keys_propagated"] > 1024 and c["nonempty"] >= 5 and c["forgot_anchor"] >= 1, c


def test_device_table_signed_zero_and_key_bits(cuda_device):
    """-0 and +0 are one key; the key keeps the bits it was inserted with, the observation the bits last assigned."""
    from bundletrack_b200.matcher import DeviceTracks
    from bundletrack_b200.policy import Tracks
    host, dev = Tracks(), DeviceTracks(max_frames=4, max_keys_per_frame=16, max_points=64)
    one_up = np.nextafter(np.float32(3.0), np.float32(4.0))
    lists = [(2, 1, [[-0.0, 5.0, 0.0, 1.0], [3.0, 1.0, 7.0, -0.0]]),
             (2, 1, [[0.0, 5.0, -0.0, 1.0], [one_up, 1.0, 7.0, 0.0]]),
             (3, 1, [[0.0, -0.0, 7.0, 0.0], [9.0, 9.0, -0.0, 1.0]]),
             (3, 2, [])]
    for a, b, uv in lists:
        uv = np.array(uv, np.float32).reshape(-1, 4)
        host.update_pair(a, b, uv)
        dev.update_pair(a, b, uv)
    for a, b in [(2, 1), (3, 1), (3, 2)]:
        want, got = host.propagate(a, b, np.zeros((0, 4), np.float32)), dev.propagate(a, b, np.zeros((0, 4), np.float32))
        assert np.array_equal(_bits(got), _bits(want)), (a, b, got, want)
    host.forget_frame(1); dev.forget_frame(1)            # the frame both points are anchored at
    assert host.stats() == dev.stats()
    assert len(dev.propagate(3, 2, np.zeros((0, 4), np.float32))) == len(host.propagate(3, 2, np.zeros((0, 4), np.float32)))
    dev.close()


# ------------------------------------------------------------------------------------------------ 2. ordered call = composition
YML = {"feature_corres": {"max_dist_no_neighbor": 0.02, "max_normal_no_neighbor": 45, "max_dist_neighbor": 10000, "max_normal_neighbor": 180},
       "ransac": {"max_iter": 2000, "inlier_dist": 0.01}}


def _frames(seed, N, n_feats, dev):
    import torch
    w = synth.make_window(seed, n_frames=N, n_corr=10)
    fr = synth.make_feature_frames(w, n_feats, seed=seed)
    host, devf = [], []
    for k in range(N):
        host.append({"kpts": fr[k]["kpts"], "desc": fr[k]["desc"], "depth": w.depth[k], "normal": w.normal[k], "pose": w.poses_init[k], "id": k})
        devf.append({"kpts": torch.from_numpy(fr[k]["kpts"]).to(dev), "desc": torch.from_numpy(fr[k]["desc"]).to(dev),
                     "depth": torch.from_numpy(w.depth[k]).to(dev), "normal": torch.from_numpy(w.normal[k]).to(dev),
                     "pose": w.poses_init[k], "id": k, "window_index": k})
    return w, host, devf


def _tail(mp, w, seed=0):
    return (ctypes.c_int(w.H), ctypes.c_int(w.W), ctypes.c_float(w.K[0]), ctypes.c_float(w.K[1]), ctypes.c_float(w.K[2]), ctypes.c_float(w.K[3]),
            ctypes.byref(mp.prune), ctypes.c_int(mp.ransac_trials), ctypes.c_float(mp.ransac_inlier_dist), ctypes.c_uint64(seed))


def _outputs(cap, n, dev):
    import torch
    return (torch.zeros((max(cap, 1), 8), dtype=torch.int32, device=dev), torch.zeros((4, n), dtype=torch.int32, device=dev),
            torch.zeros(4, dtype=torch.int32, device=dev), torch.zeros((max(cap, 1), 4), dtype=torch.float32, device=dev))


def test_ordered_call_equals_pair_by_pair_composition(cuda_device):
    """An 8-frame sequence: each new frame against its neighbour, then the older frames oldest first, in ONE bt_find_corres_pairs call;
    the same pairs one bt_match_pairs_ex call at a time, fed from and feeding the host table.  Byte-identical outputs."""
    from bundletrack_b200.matcher import MatchPipeline, DeviceTracks
    from bundletrack_b200.policy import Tracks
    from oracle import matcher_oracle as mo
    N, NF = 8, 500
    w, host, devf = _frames(31, N, NF, cuda_device)
    mp_seq, mp_one = MatchPipeline(YML, max_pairs=8, max_feats=512), MatchPipeline(YML, max_pairs=8, max_feats=512)
    for mp in (mp_seq, mp_one):
        mp.pool_reserve(N)
        for f in range(N):
            mp.pool_store(f, devf[f]["desc"])
    DeviceTracks(ctx=mp_one.ctx, max_frames=16, max_keys_per_frame=512)       # the table of mp_one's context
    tracks, lagged = Tracks(), Tracks()       # lagged: updated only after a whole frame, i.e. without the earlier pairs of the same call
    lib = mp_one.lib
    prm = (mp_seq.prune.max_dist_no_neighbor, mp_seq.prune.cos_max_normal_no_neighbor, mp_seq.prune.max_dist_neighbor, mp_seq.prune.cos_max_normal_neighbor)
    n_prop_emitted = n_order_matters = 0
    for f in range(1, N):
        prs = [(f, f - 1)] + [(f, j) for j in range(0, f - 1)]
        n = len(prs)
        # (a) pair by pair
        want_ent, want_meta, want_uv, done = [], [], [], []
        for a, b in prs:
            A, B, _, _ = mp_seq._views([(devf[a], devf[b])])
            extra = (_lib.MatchExtra * 1)()
            prop = np.zeros((0, 4), np.float32)
            if a - b != 1:
                prop = np.ascontiguousarray(tracks.propagate(a, b, np.zeros((0, 4), np.float32)), np.float32)
                extra[0].uv, extra[0].n = (prop.ctypes.data if len(prop) else None), len(prop)
                if not np.array_equal(_bits(prop), _bits(lagged.propagate(a, b, np.zeros((0, 4), np.float32)))):
                    n_order_matters += 1
            cap = NF * 2 + len(prop)
            ent, meta, tot, uvo = _outputs(cap, 1, cuda_device)
            _lib.check(lib.bt_match_pairs_ex(mp_seq.ctx, ctypes.c_int(1), A, B, None, None, (ctypes.c_int32 * 1)(a), (ctypes.c_int32 * 1)(b), *_tail(mp_seq, w),
                                             extra, ctypes.c_void_p(ent.data_ptr()), ctypes.c_int(cap), ctypes.c_void_p(meta[0].data_ptr()),
                                             ctypes.c_void_p(meta[1].data_ptr()), ctypes.c_void_p(tot.data_ptr()), ctypes.c_void_p(meta[2].data_ptr()),
                                             ctypes.c_void_p(uvo.data_ptr()), mp_seq.stream), "bt_match_pairs_ex")
            m = meta.cpu().numpy()
            k = int(m[0][0])
            uv = uvo[:k].cpu().numpy()
            want_ent.append(ent[:k].cpu().numpy()); want_meta.append((k, int(m[2][0]))); want_uv.append(uv)
            if k:
                tracks.update_pair(a, b, uv)
                done.append((a, b, uv))
            if a - b != 1 and k and len(prop):
                ia, ib = mo.knn(host[a]["desc"], host[b]["desc"])[0], mo.knn(host[b]["desc"], host[a]["desc"])[0]
                md, cm = prm[0], prm[1]
                mut = mo.collect_mutual(host[a], host[b], mo.prune_matches(host[a], host[b], ia, w.K, md, cm), mo.prune_matches(host[b], host[a], ib, w.K, md, cm))[:, :4]
                pset = {tuple(r) for r in _bits(prop).tolist()}
                ka, kb = {tuple(r) for r in _bits(mut[:, :2]).tolist()}, {tuple(r) for r in _bits(mut[:, 2:4]).tolist()}
                for r in _bits(uv).tolist():
                    n_prop_emitted += tuple(r) in pset and tuple(r[:2]) not in ka and tuple(r[2:]) not in kb
        for a, b, uv in done:
            lagged.update_pair(a, b, uv)
        # (b) one ordered call
        A, B, _, _ = mp_one._views([(devf[a], devf[b]) for a, b in prs])
        cap = n * (2 * NF + 512)
        ent, meta, tot, uvo = _outputs(cap, n, cuda_device)
        _lib.check(lib.bt_find_corres_pairs(mp_one.ctx, ctypes.c_int(n), A, B, None, None, (ctypes.c_int32 * n)(*[a for a, _ in prs]),
                                            (ctypes.c_int32 * n)(*[b for _, b in prs]), *_tail(mp_one, w), ctypes.c_void_p(ent.data_ptr()), ctypes.c_int(cap),
                                            ctypes.c_void_p(meta[0].data_ptr()), ctypes.c_void_p(meta[1].data_ptr()), ctypes.c_void_p(tot.data_ptr()),
                                            ctypes.c_void_p(meta[2].data_ptr()), ctypes.c_void_p(uvo.data_ptr()), mp_one.stream), "bt_find_corres_pairs")
        m = meta.cpu().numpy()
        counts = np.array([k for k, _ in want_meta], np.int32)
        assert np.array_equal(m[0], counts), (f, m[0], counts)
        assert np.array_equal(m[1], np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int32)), f
        assert np.array_equal(m[2], np.array([s for _, s in want_meta], np.int32)), f
        assert int(tot[0]) == counts.sum()
        total = int(counts.sum())
        assert np.array_equal(ent[:total].cpu().numpy(), np.concatenate(want_ent).reshape(-1, 8)), f
        assert np.array_equal(_bits(uvo[:total].cpu().numpy()), _bits(np.concatenate(want_uv).reshape(-1, 4))), f
    pts, obs = ctypes.c_int(), ctypes.c_int()
    _lib.check(lib.bt_tracks_dev_stats(mp_one.ctx, ctypes.byref(pts), ctypes.byref(obs), mp_one.stream), "bt_tracks_dev_stats")
    assert (pts.value, obs.value) == tracks.stats()
    assert n_prop_emitted >= 3, n_prop_emitted          # propagated matches went through RANSAC into the EntryJ list
    assert n_order_matters >= 1, n_order_matters        # a pair saw map points an earlier pair of the same call made
    mp_seq.close(); mp_one.close()


# ------------------------------------------------------------------------------------------------ 4. errors
def test_capacity_and_argument_errors(cuda_device):
    import torch
    from bundletrack_b200.matcher import DeviceTracks
    from bundletrack_b200.policy import Tracks
    dev = DeviceTracks(max_frames=2, max_keys_per_frame=4, max_points=3)
    host = Tracks()
    lib, ctx = dev.lib, dev.ctx
    ok = np.array([[1, 1, 2, 2], [3, 3, 4, 4]], np.float32)
    dev.update_pair(1, 0, ok); host.update_pair(1, 0, ok)
    big = np.array([[10 + k, 0, 20 + k, 0] for k in range(5)], np.float32)        # 5 new keys per frame > 4
    dev.update_pair(1, 0, big)
    with pytest.raises(_lib.BtError, match="status -2"):
        dev.stats()
    assert dev.stats() == host.stats()                 # the overflowing update changed nothing; the flag was reported once
    z = np.zeros((0, 4), np.float32)
    assert np.array_equal(_bits(dev.propagate(1, 0, z)), _bits(host.propagate(1, 0, z)))
    pts = np.array([[5, 5, 6, 6]], np.float32)        # a 2nd new point fits (3 points), a 3rd frame does not
    dev.update_pair(1, 0, pts); host.update_pair(1, 0, pts)
    assert dev.stats() == host.stats()
    with pytest.raises(_lib.BtError, match="status -2"):
        dev.update_pair(2, 0, ok)
    more = np.array([[7, 7, 8, 8], [9, 9, 10, 10]], np.float32)       # two more points > 3 points
    dev.update_pair(1, 0, more)
    with pytest.raises(_lib.BtError, match="status -2"):
        dev.stats()
    wide = DeviceTracks(ctx=ctx, max_frames=2, max_keys_per_frame=4, max_points=3)   # re-reserving empties the table
    assert wide.stats() == (0, 0)
    small = np.array([[1, 1, 2, 2]], np.float32)
    dev.update_pair(1, 0, small)
    assert dev.propagate(1, 0, z).shape == (1, 4)
    # propagation longer than the caller's capacity
    dev.update_pair(1, 0, np.array([[5, 5, 6, 6]], np.float32))
    with pytest.raises(_lib.BtError, match="status -2"):
        dev.propagate(1, 0, z, capacity=1)
    # bad arguments
    d_n = torch.zeros(1, dtype=torch.int32, device=cuda_device)
    assert lib.bt_tracks_dev_update_pair(ctx, 0, 1, None, ctypes.c_void_p(d_n.data_ptr()), 0, None) == _lib.BT_ERR_INVALID_ARG     # A not newer
    assert lib.bt_tracks_dev_update_pair(ctx, 1, 0, None, None, 0, None) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_tracks_dev_propagate(ctx, 1, 0, None, 3, None, 0, ctypes.c_void_p(d_n.data_ptr()), None) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_tracks_dev_reserve(ctx, 65, 4, 3) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_tracks_dev_reserve(ctx, 2, 0, 3) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_tracks_dev_stats(None, None, None, None) == _lib.BT_ERR_INVALID_ARG
    bare = ctypes.c_void_p()
    _lib.check(lib.bt_ctx_create(ctypes.byref(bare), 0), "bt_ctx_create")
    assert lib.bt_tracks_dev_forget_frame(bare, 0, None) == _lib.BT_ERR_INVALID_ARG        # no table reserved
    frame = (_lib.MatchFrame * 1)()
    assert lib.bt_find_corres_pairs(bare, 1, frame, frame, None, None, (ctypes.c_int32 * 1)(0), (ctypes.c_int32 * 1)(0), 1, 1, ctypes.c_float(1), ctypes.c_float(1),
                                    ctypes.c_float(0), ctypes.c_float(0), None, 1, ctypes.c_float(0.01), ctypes.c_uint64(0), None, 0, None, None, None, None, None,
                                    None) == _lib.BT_ERR_INVALID_ARG
    lib.bt_ctx_destroy(bare)
    dev.close()
