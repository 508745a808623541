"""Host-side mirror of the matcher boundary (SiftManager::findCorresbyNN's two knnMatch calls,
/root/reference/src/FeatureManager.cpp:271-273), batched over frame pairs, on top of the C-ABI."""
from __future__ import annotations

import ctypes
from typing import List, Sequence, Tuple

from . import _lib


class _DescPool(_lib.Facade):
    """The context's persistent descriptor pool: a frame's descriptors are converted once (Lfnet::detectFeature, FeatureManager.cpp:907)."""

    def pool_reserve(self, n_slots: int):
        _lib.check(self.lib.bt_desc_pool_reserve(self.ctx, n_slots), "bt_desc_pool_reserve")

    def pool_store(self, slot: int, desc: "torch.Tensor"):
        _lib.check(self.lib.bt_desc_pool_store(self.ctx, slot, _lib.desc_view(desc), self.stream), "bt_desc_pool_store")


class KnnMatcher(_DescPool):
    """knnMatch(query, train, k) for many (A, B) pairs at once; ONE tensor-core contraction per pair serves both directions."""

    def __init__(self, device: int = 0, max_pairs: int = 64, max_feats: int = 4096, dim: int = 256, stream: int = 0, ctx=None):
        super().__init__(ctx, device, stream)
        _lib.check(self.lib.bt_matcher_reserve(self.ctx, max_pairs, max_feats, dim), "bt_matcher_reserve")
        self.dim = dim

    def knn_match_pairs(self, pairs: Sequence[Tuple["torch.Tensor", "torch.Tensor"]], k: int = 5):
        """pairs: list of (A [nA,dim] fp32 cuda, B [nB,dim] fp32 cuda); rows may be pitched (stride(0) >= dim).
        Returns (idxAB, distAB, idxBA, distBA): lists (one entry per pair) of [n,k] int32 / float32 cuda tensors.
        distance = sqrt(sum (a-b)^2) ascending, ties -> lower train index (cv::DMatch semantics)."""
        import torch
        for t in (t for p in pairs for t in p):
            assert t.is_cuda and t.dtype == torch.float32 and t.dim() == 2 and t.stride(1) == 1
        n = len(pairs)
        A = (_lib.DescView * n)(*[_lib.desc_view(a) for a, _ in pairs])
        B = (_lib.DescView * n)(*[_lib.desc_view(b) for _, b in pairs])
        return self._knn(self.lib.bt_knn_match_pairs, "bt_knn_match_pairs", A, B, [(a.shape[0], b.shape[0]) for a, b in pairs], k, pairs[0][0].device)

    def knn_match_slots(self, slot_pairs: Sequence[Tuple[int, int]], sizes: Sequence[Tuple[int, int]], k: int = 5, device=None):
        """slot_pairs: (slotA, slotB) per pair; sizes: (nA, nB) per pair (what was stored).  Same outputs as knn_match_pairs."""
        import torch
        sa, sb = _lib.i32s([a for a, _ in slot_pairs]), _lib.i32s([b for _, b in slot_pairs])
        return self._knn(self.lib.bt_knn_match_slots, "bt_knn_match_slots", sa, sb, sizes, k, device or torch.device("cuda", torch.cuda.current_device()))

    def _knn(self, fn, what, A, B, sizes, k, dev):
        import torch
        na, nb = sum(a for a, _ in sizes), sum(b for _, b in sizes)
        idxAB = torch.empty((max(na, 1), k), dtype=torch.int32, device=dev)
        distAB = torch.empty((max(na, 1), k), dtype=torch.float32, device=dev)
        idxBA = torch.empty((max(nb, 1), k), dtype=torch.int32, device=dev)
        distBA = torch.empty((max(nb, 1), k), dtype=torch.float32, device=dev)
        _lib.check(fn(self.ctx, len(sizes), A, B, k, *(_lib.ptr(t) for t in (idxAB, distAB, idxBA, distBA)), self.stream), what)
        oAB, oBA, ia, ib = [], [], 0, 0
        for a, b in sizes:
            oAB.append((idxAB[ia:ia + a], distAB[ia:ia + a]))
            oBA.append((idxBA[ib:ib + b], distBA[ib:ib + b]))
            ia += a
            ib += b
        return [x[0] for x in oAB], [x[1] for x in oAB], [x[0] for x in oBA], [x[1] for x in oBA]

    def force_fallback(self, every_nth: int):
        """Test knob: every n-th query row goes through the exact brute-force kernel (0 = off)."""
        _lib.check(self.lib.bt_knn_debug_force_fallback(self.ctx, every_nth), "bt_knn_debug_force_fallback")

    def enable_timing(self, on=True):
        _lib.check(self.lib.bt_knn_enable_timing(self.ctx, 1 if on else 0), "bt_knn_enable_timing")

    def timing(self):
        ms = (ctypes.c_float * 4)()
        info = (ctypes.c_int * 3)()
        _lib.check(self.lib.bt_knn_get_timing(self.ctx, ms, info), "bt_knn_get_timing")
        return {"prep_ms": ms[0], "tc_ms": ms[1], "rerank_ms": ms[2], "fallback_ms": ms[3], "units": info[0], "rows": info[1], "fallback_rows": info[2]}


class Ransac(_lib.Facade):
    """ransacMultiPairGPU (/root/reference/src/cuda/cuda_ransac.h:50) for a batch of pairs."""

    def __init__(self, device: int = 0, max_pairs: int = 64, max_pts: int = 8192, max_trials: int = 2000, stream: int = 0, ctx=None):
        super().__init__(ctx, device, stream)
        _lib.check(self.lib.bt_ransac_reserve(self.ctx, max_pairs, max_pts, max_trials), "bt_ransac_reserve")
        self.max_trials = max_trials

    def ransac_pairs(self, ptsA: List["torch.Tensor"], ptsB: List["torch.Tensor"], n_trials: int, dist_thresh: float, seed: int = 0):
        """ptsA[p], ptsB[p]: [n_p,4] float32 cuda (w ignored).  Returns list of int32 cuda tensors of inlier ids (ascending)."""
        import torch
        n = len(ptsA)
        total = sum(t.shape[0] for t in ptsA)
        dev = ptsA[0].device
        ids = torch.empty(max(total, 1), dtype=torch.int32, device=dev)
        nin = torch.empty(n, dtype=torch.int32, device=dev)
        _lib.check(self.lib.bt_ransac_pairs(self.ctx, n, _lib.ptrs(ptsA), _lib.ptrs(ptsB), _lib.i32s([t.shape[0] for t in ptsA]), n_trials, dist_thresh, seed,
                                            _lib.ptr(ids), _lib.ptr(nin), self.stream), "bt_ransac_pairs")
        nin_h = nin.cpu().numpy()
        out, o = [], 0
        for p in range(n):
            out.append(ids[o:o + int(nin_h[p])])
            o += ptsA[p].shape[0]
        return out

    def debug(self, n_trials: int, n_pairs: int):
        import numpy as np
        u3 = np.zeros((n_trials, 3), np.float32)
        bt = np.zeros(n_pairs, np.int32)
        _lib.check(self.lib.bt_ransac_debug(self.ctx, _lib.ptr(u3), n_trials, _lib.ptr(bt), n_pairs), "bt_ransac_debug")
        return u3, bt

    def debug_trials(self, pair: int, n_trials: int):
        """Pair `pair` of the last call: (poses [n_trials, 3, 4] float32 [R | t], good [n_trials] int32, the winner's inlier count or -1)."""
        return ransac_debug_trials(self.lib, self.ctx, pair, n_trials)


def ransac_debug_trials(lib, ctx, pair: int, n_trials: int):
    """bt_ransac_debug_trials on any context that ran RANSAC (a Ransac facade or the matcher chain of a MatchPipeline)."""
    import numpy as np
    poses = np.zeros((n_trials, 3, 4), np.float32)
    good = np.zeros(n_trials, np.int32)
    cnt = ctypes.c_int32(0)
    _lib.check(lib.bt_ransac_debug_trials(ctx, pair, n_trials, _lib.ptr(poses), _lib.ptr(good), ctypes.byref(cnt)), "bt_ransac_debug_trials")
    return poses, good, cnt.value


class MatchPipeline(_DescPool):
    """The matcher half of the hot path, device-resident: SiftManager::findCorres for a batch of frame pairs
    (kNN both directions -> pruneMatches -> collectMutualMatches -> runRansacBetween) ending in the EntryJ records
    Bundler::optimizeGPU would build (/root/reference/src/FeatureManager.cpp:173-368,561-741; src/Bundler.cpp:298-324)."""

    def __init__(self, yml=None, device: int = 0, max_pairs: int = 64, max_feats: int = 4096, dim: int = 256, stream: int = 0, ctx=None):
        from .config import load_yml, prune_params
        super().__init__(ctx, device, stream)
        y = load_yml(yml)
        rs = y["ransac"]
        self.prune = prune_params(y)
        self.ransac_trials = int(rs["max_iter"])
        self.ransac_inlier_dist = float(rs["inlier_dist"])
        _lib.check(self.lib.bt_pipeline_reserve(self.ctx, max_pairs, max_feats, dim, max(self.ransac_trials, 1)), "bt_pipeline_reserve")
        self.max_pairs, self.max_feats = max_pairs, max_feats

    @staticmethod
    def _frame(fr) -> "_lib.MatchFrame":
        """fr: dict with kpts [n,2] cuda f32, depth [H,W] cuda f32, normal [H,W,4] cuda f32, pose [4,4] numpy, id, window_index."""
        import numpy as np
        m = _lib.MatchFrame()
        m.kpts_dev, m.n = fr["kpts"].data_ptr(), fr["kpts"].shape[0]
        m.depth_dev, m.normal_dev = fr["depth"].data_ptr(), fr["normal"].data_ptr()
        P = np.ascontiguousarray(fr["pose"], np.float32).reshape(16)
        for k in range(16):
            m.pose[k] = float(P[k])
        m.frame_id, m.window_index = int(fr["id"]), int(fr.get("window_index", fr["id"]))
        return m

    def _views(self, pairs):
        n = len(pairs)
        A = (_lib.MatchFrame * n)(*[self._frame(fa) for fa, _ in pairs])
        B = (_lib.MatchFrame * n)(*[self._frame(fb) for _, fb in pairs])
        # (frames whose descriptors live in the pool need no view)
        dA = (_lib.DescView * n)(*[_lib.desc_view(fa["desc"]) if fa.get("desc") is not None else _lib.DescView() for fa, _ in pairs])
        dB = (_lib.DescView * n)(*[_lib.desc_view(fb["desc"]) if fb.get("desc") is not None else _lib.DescView() for _, fb in pairs])
        return A, B, dA, dB

    def prune_mutual(self, pairs, idxAB, idxBA, H, W, K, k=5):
        """pairs: list of (frameA newer, frameB older) dicts; idxAB/idxBA: concatenated [sum n, k] int32 cuda kNN indices.
        Returns list of [m,10] float32 cuda tensors (uA,vA,uB,vB,ptA_cam,ptB_cam)."""
        import torch
        A, B, _, _ = self._views(pairs)
        n = len(pairs)
        cap = sum(fa["kpts"].shape[0] + fb["kpts"].shape[0] for fa, fb in pairs)
        dev = pairs[0][0]["kpts"].device
        corr = torch.empty((max(cap, 1), 10), dtype=torch.float32, device=dev)
        cnt = torch.empty(n, dtype=torch.int32, device=dev)
        _lib.check(self.lib.bt_prune_mutual_pairs(self.ctx, n, A, B, H, W, *_lib.intrinsics(K), _lib.ptr(idxAB), _lib.ptr(idxBA), k, self.prune,
                                                  _lib.ptr(corr), _lib.ptr(cnt), self.stream), "bt_prune_mutual_pairs")
        ch = cnt.cpu().numpy()
        out, o = [], 0
        for p, (fa, fb) in enumerate(pairs):
            out.append(corr[o:o + int(ch[p])])
            o += fa["kpts"].shape[0] + fb["kpts"].shape[0]
        return out

    def match_pairs(self, pairs, H, W, K, seed: int = 0, capacity: int = 0, keep_on_device: bool = False, slots=None):
        """Fused pipeline.  slots: optional list of (slotA, slotB) naming descriptor sets stored with pool_store (the frames' "desc" entries
        are then not read).  Returns (entries [total] EntryJ structured numpy array, n_entry [n_pairs], entry_off [n_pairs]).
        keep_on_device=True: the entries stay on the GPU - returns (device int32 tensor [cap, 8], n_entry, entry_off) and only the
        two small count arrays are read back; hand them to SolveWindow(corr_dev=..., blocks=...) (see `solver_blocks`)."""
        import numpy as np
        import torch
        from .synth import ENTRYJ_DTYPE
        A, B, dA, dB = self._views(pairs)
        n = len(pairs)
        cap = capacity or sum(fa["kpts"].shape[0] + fb["kpts"].shape[0] for fa, fb in pairs)
        dev = pairs[0][0]["kpts"].device
        ent = torch.empty((max(cap, 1), 8), dtype=torch.int32, device=dev)     # 32-byte EntryJ records
        n_ent = torch.empty(n, dtype=torch.int32, device=dev)
        off = torch.empty(n, dtype=torch.int32, device=dev)
        tot = torch.zeros(4, dtype=torch.int32, device=dev)
        tail = (H, W, *_lib.intrinsics(K), self.prune, self.ransac_trials, self.ransac_inlier_dist, seed,
                _lib.ptr(ent), cap, _lib.ptr(n_ent), _lib.ptr(off), _lib.ptr(tot), self.stream)
        if slots is None:
            _lib.check(self.lib.bt_match_pairs(self.ctx, n, A, B, dA, dB, *tail), "bt_match_pairs")
        else:
            _lib.check(self.lib.bt_match_pairs_pool(self.ctx, n, A, B, _lib.i32s([a for a, _ in slots]), _lib.i32s([b for _, b in slots]), *tail),
                       "bt_match_pairs_pool")
        self.last = (ent, n_ent, off, tot)
        if keep_on_device:
            cnt = torch.stack([n_ent, off]).cpu().numpy()      # one small D2H (2 x n_pairs ints), no entry leaves the device
            return ent, cnt[0], cnt[1]
        total = int(tot[0].item())
        host = ent[:total].cpu().numpy().view(np.uint8).reshape(-1).view(ENTRYJ_DTYPE)
        return host, n_ent.cpu().numpy(), off.cpu().numpy()

    @staticmethod
    def solver_blocks(pairs, n_entry, entry_off):
        """blocks=(off, n, i, j) for SolveWindow from match_pairs(keep_on_device=True): block p carries (imgIdx_i, imgIdx_j) =
        (older frame B's window index, newer frame A's), exactly what k_emit_entryj writes into the entries."""
        import numpy as np
        bi = np.array([fb["window_index"] for _, fb in pairs], np.uint32)
        bj = np.array([fa["window_index"] for fa, _ in pairs], np.uint32)
        return np.asarray(entry_off, np.int32), np.asarray(n_entry, np.int32), bi, bj


class DeviceTracks(_lib.Facade):
    """The map-point table on the device (bt_tracks_dev_*), owned by a context: the methods of policy.Tracks with the same results,
    host arrays in and out.  FindCorres keeps one; bt_find_corres_pairs reads and updates it without leaving the device.
    Capacities: frames alive (<= 64 + 1024, bt_tracks_dev_reserve_ex), keys per frame (<= 8192), map points alive (default
    16 x max_keys_per_frame x ceil(max_frames / 64)).  The table takes max_points x max_frames x 8 B for the observations plus
    max_frames x max_keys_per_frame x 48 B for the frame maps: 34 MB and 13 MB at the defaults, 0.34 GB and 25 MB at 264 frames of 2000 keys.
    All work, including the uploads and read-backs of the methods below, runs on `stream`."""

    def __init__(self, ctx=None, device: int = 0, max_frames: int = 64, max_keys_per_frame: int = 4096, max_points: int = 0, stream: int = 0):
        super().__init__(ctx, device, stream)
        self.device = device
        max_points = max_points or 16 * max_keys_per_frame * -(-max_frames // 64)
        _lib.check(self.lib.bt_tracks_dev_reserve_ex(self.ctx, max_frames, max_keys_per_frame, max_points), "bt_tracks_dev_reserve_ex")

    def _on_stream(self):
        """torch work (allocation, upload, read-back) on the table's stream: the kernels then see the uploads complete, the read-backs
        see the kernels complete, and the caching allocator hands a freed buffer only to later work on the same stream."""
        import contextlib
        import torch
        if not self.stream.value:
            return contextlib.nullcontext()       # the legacy default stream orders against every other stream already
        return torch.cuda.stream(torch.cuda.ExternalStream(self.stream.value, device=torch.device("cuda", self.device)))

    def update_pair(self, frame_a: int, frame_b: int, uv, is_inlier=None):
        import numpy as np
        import torch
        uv = np.ascontiguousarray(uv, np.float32).reshape(-1, 4)
        if is_inlier is not None:
            uv = np.ascontiguousarray(uv[np.asarray(is_inlier).astype(bool)])
        dev = torch.device("cuda", self.device)
        with self._on_stream():
            d_uv = torch.from_numpy(uv).to(dev) if len(uv) else torch.zeros((1, 4), dtype=torch.float32, device=dev)
            d_n = torch.tensor([len(uv)], dtype=torch.int32, device=dev)
            _lib.check(self.lib.bt_tracks_dev_update_pair(self.ctx, frame_a, frame_b, _lib.ptr(d_uv), _lib.ptr(d_n), len(uv), self.stream),
                       "bt_tracks_dev_update_pair")

    def propagate(self, frame_a: int, frame_b: int, existing_uv, capacity: int = 65536):
        import numpy as np
        import torch
        ex = np.ascontiguousarray(existing_uv, np.float32).reshape(-1, 4)
        dev = torch.device("cuda", self.device)
        with self._on_stream():
            d_ex = torch.from_numpy(ex).to(dev) if len(ex) else None
            out = torch.empty((max(capacity, 1), 4), dtype=torch.float32, device=dev)
            n = torch.zeros(1, dtype=torch.int32, device=dev)
            _lib.check(self.lib.bt_tracks_dev_propagate(self.ctx, frame_a, frame_b, _lib.ptr(d_ex), len(ex), _lib.ptr(out), capacity, _lib.ptr(n), self.stream),
                       "bt_tracks_dev_propagate")
            self.stats()                # synchronises the stream; a propagation longer than `capacity` is an error, as on the host
            k = int(n.item())
            return out[:k].cpu().numpy()

    def forget_frame(self, frame: int):
        _lib.check(self.lib.bt_tracks_dev_forget_frame(self.ctx, frame, self.stream), "bt_tracks_dev_forget_frame")

    def stats(self):
        a, b = ctypes.c_int(0), ctypes.c_int(0)
        _lib.check(self.lib.bt_tracks_dev_stats(self.ctx, ctypes.byref(a), ctypes.byref(b), self.stream), "bt_tracks_dev_stats")
        return a.value, b.value


class FindCorres:
    """`SiftManager::findCorres` (/root/reference/src/FeatureManager.cpp:173-242) on the device-resident chain: per pair (A newer)
    kNN both ways -> prune -> mutual union -> [non-neighbour: map-point propagation] -> RANSAC -> EntryJ, with the `_matches` cache
    (a pair is matched once), the map-point table on the device (`tracks`, a DeviceTracks: max_frames alive, max_points map points,
    default 16 x the pipeline's max_feats x ceil(max_frames / 64); see DeviceTracks for its memory) and the Frame::FAIL outcome.  Descriptors
    live in the pool.  The cache's arena holds max_entries_total entries of 32 B (None: max_pairs_cached x max_entries_per_pair, each pair
    at most max_entries_per_pair; bt_match_cache_reserve / _reserve_entries)."""

    def __init__(self, pipeline: "MatchPipeline", max_pairs_cached: int = 512, max_entries_per_pair: int = 0, max_frames: int = 64, max_points: int = 0,
                 max_entries_total: int = None):
        self.mp = pipeline
        self.lib = pipeline.lib
        self.ctx = pipeline.ctx
        self.tracks = DeviceTracks(ctx=pipeline.ctx, max_frames=max_frames, max_keys_per_frame=pipeline.max_feats, max_points=max_points, stream=pipeline.stream.value or 0)
        self.slot_entries = max_entries_per_pair or 3 * pipeline.max_feats
        if max_entries_total is None:
            _lib.check(self.lib.bt_match_cache_reserve(self.ctx, max_pairs_cached, self.slot_entries), "bt_match_cache_reserve")
        else:
            _lib.check(self.lib.bt_match_cache_reserve_entries(self.ctx, max_pairs_cached, max_entries_total), "bt_match_cache_reserve_entries")
        self.failed = set()          # ids of frames the reference would mark Frame::FAIL

    def has(self, id_a: int, id_b: int) -> bool:
        rc = self.lib.bt_match_cache_has(self.ctx, id_a, id_b)
        if rc < 0:
            _lib.check(rc, "bt_match_cache_has")
        return bool(rc)

    def find_corres(self, pairs, slots, H, W, K, seed: int = 0):
        """pairs: list of (frameA newer, frameB older) dicts as for MatchPipeline.match_pairs; slots: their descriptor-pool slots.
        Pairs already in the cache are skipped (FeatureManager.cpp:176).  The others are matched IN THE GIVEN ORDER in one asynchronous
        call (bt_find_corres_pairs): a pair's propagated map-point matches see what the earlier pairs of the same call added to the table,
        exactly as the reference's pair-by-pair loop does (Bundler.cpp:298-305) - hand a new frame's neighbour pair first, then its older
        frames oldest first.  One small read-back (counts, offsets, status) at the end feeds the cache.
        Returns {(idA, idB): (n_entries, status)} of the pairs processed in this call."""
        import numpy as np
        import torch
        todo = [(k, p) for k, p in enumerate(pairs) if not self.has(p[0]["id"], p[1]["id"])]
        if not todo:
            return {}
        prs = [p for _, p in todo]
        sl = [slots[k] for k, _ in todo]
        n = len(prs)
        A, B, _, _ = self.mp._views(prs)      # (descriptor views unused: the pool is named by slot)
        cap = sum(a["kpts"].shape[0] + b["kpts"].shape[0] for a, b in prs) + n * self.mp.max_feats      # never truncates: room for every propagated match
        dev = prs[0][0]["kpts"].device
        ent = torch.empty((max(cap, 1), 8), dtype=torch.int32, device=dev)
        meta = torch.zeros((3, n), dtype=torch.int32, device=dev)              # n_entry, entry_off, status
        tot = torch.zeros(4, dtype=torch.int32, device=dev)
        mp = self.mp
        _lib.check(self.lib.bt_find_corres_pairs(self.ctx, n, A, B, None, None, _lib.i32s([a for a, _ in sl]), _lib.i32s([b for _, b in sl]), H, W,
                                                 *_lib.intrinsics(K), mp.prune, mp.ransac_trials, mp.ransac_inlier_dist, seed, _lib.ptr(ent), cap,
                                                 _lib.ptr(meta[0]), _lib.ptr(meta[1]), _lib.ptr(tot), _lib.ptr(meta[2]), None, mp.stream), "bt_find_corres_pairs")
        m = meta.cpu().numpy()                                                  # 3 x n ints: the call's only read-back
        self.tracks.stats()                                                     # (the stream is idle: raises if the table ran out of room)
        n_h = np.ascontiguousarray(m[0]); off_h = np.ascontiguousarray(m[1]); st_h = np.ascontiguousarray(m[2])
        _lib.check(self.lib.bt_match_cache_put(self.ctx, n, _lib.i32s([a["id"] for a, _ in prs]), _lib.i32s([b["id"] for _, b in prs]), _lib.ptr(ent),
                                               _lib.ptr(n_h), _lib.ptr(off_h), _lib.ptr(st_h), mp.stream), "bt_match_cache_put")
        out = {}
        for i, (a, b) in enumerate(prs):
            if st_h[i] == 2:
                self.failed.add(a["id"])
            out[(a["id"], b["id"])] = (int(n_h[i]), int(st_h[i]))
        self._keep = ent
        return out

    def window_entries(self, frames, device):
        """The EntryJ list Bundler::optimizeGPU builds for the window `frames` (oldest first; window index = position), straight from
        the cache: returns (device EntryJ tensor, blocks) for SolveWindow(corr_dev=..., blocks=...)."""
        import numpy as np
        import torch
        prs = [(frames[j]["id"], frames[i]["id"], i, j) for i in range(len(frames)) for j in range(i + 1, len(frames))]
        n = len(prs)
        wi = np.array([p[2] for p in prs], np.uint32); wj = np.array([p[3] for p in prs], np.uint32)
        cap = n * self.slot_entries
        dst = torch.empty((max(min(cap, 1 << 22), 1), 8), dtype=torch.int32, device=device)
        off = np.zeros(n, np.int32); cnt = np.zeros(n, np.int32)
        _lib.check(self.lib.bt_match_cache_gather(self.ctx, n, _lib.i32s([p[0] for p in prs]), _lib.i32s([p[1] for p in prs]), _lib.ptr(wi), _lib.ptr(wj),
                                                  _lib.ptr(dst), dst.shape[0], _lib.ptr(off), _lib.ptr(cnt), self.mp.stream), "bt_match_cache_gather")
        return dst, (off, cnt, wi, wj)

    def forget_frame(self, frame_id: int):
        _lib.check(self.lib.bt_match_cache_forget_frame(self.ctx, frame_id), "bt_match_cache_forget_frame")
        self.tracks.forget_frame(frame_id)
