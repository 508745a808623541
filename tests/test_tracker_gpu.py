"""The tracker (bt_tracker_*, bundletrack_b200.tracker.Tracker) against an independent composition of the existing public pieces that follows
Bundler::processNewFrame (the reference's src/Bundler.cpp:56-183) line for line, byte for byte over whole sequences; the device initial pose
(bt_pose_init) against bt_rigid_transform; argument and capacity errors; accuracy against the sequences' ground truth; the C++ BundlerGpu."""
import collections
import ctypes
import os
import subprocess

import numpy as np
import pytest

from bundletrack_b200 import _lib, policy, synth
from bundletrack_b200.config import load_yml
from bundletrack_b200.synth import ENTRYJ_DTYPE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, W = 240, 320
FEATS = 400


def xform(P, p):
    """pcl::transformPointWithNormal's point part in float32, ((m0 x + m1 y) + m2 z) + m3: one rounding per operation (numpy does not fuse)."""
    P = np.asarray(P, np.float32)
    return np.stack([((P[r, 0] * p[:, 0] + P[r, 1] * p[:, 1]) + P[r, 2] * p[:, 2]) + P[r, 3] for r in range(3)], 1)


def compose(O, P):
    """offset * pose, each element ((o0 p0 + o1 p1) + o2 p2) + o3 p3 in float32."""
    O, P = np.asarray(O, np.float32), np.asarray(P, np.float32)
    out = np.zeros((4, 4), np.float32)
    for i in range(4):
        for j in range(4):
            out[i, j] = ((O[i, 0] * P[0, j] + O[i, 1] * P[1, j]) + O[i, 2] * P[2, j]) + O[i, 3] * P[3, j]
    return out


class Composition:
    """Bundler::processNewFrame from FrameFrontEnd, MatchPipeline's pool, FindCorres, policy.* and OptimizerGpu with the frame cache.
    Holds its own frame deque and keyframe list; `ev` counts the events a sequence went through."""

    def __init__(self, yml, K, max_feats, max_frames_alive, mode, H=H, W=W):
        import torch
        from bundletrack_b200.frontend import FrameFrontEnd
        from bundletrack_b200.matcher import FindCorres, MatchPipeline
        from bundletrack_b200.optimizer import OptimizerGpu
        self.y, self.K, self.mode, self.dev = load_yml(yml), K, mode, torch.device("cuda", 0)
        self.H, self.W = H, W
        self.n_neighbour = []                 # entries of each neighbour pair that went to the initial pose
        b, kf = self.y["bundle"], self.y["keyframe"]
        self.ws, self.max_ba, self.min_edges = int(b["window_size"]), int(b["max_BA_frames"]), int(b["min_fm_edges_newframe"])
        self.min_feat, self.min_rot = int(kf["min_feat_num"]), float(kf["min_rot"])
        F = max_frames_alive
        max_pairs = self.max_ba * (self.max_ba - 1) // 2
        self.fe = FrameFrontEnd(self.y)
        self.mp = MatchPipeline(self.y, max_pairs=max_pairs, max_feats=max_feats)
        self.mp.pool_reserve(F + 1)
        self.fc = FindCorres(self.mp, max_pairs_cached=F * (F - 1) // 2, max_entries_per_pair=3 * max_feats, max_frames=F)
        self.opt = OptimizerGpu(self.y, max_windows=1, max_frames=self.max_ba, max_corr=max_pairs * 3 * max_feats, H=H, W=W)
        self.opt.reserve_frame_cache(F, H, W)
        self.frames, self.keyframes = [], []
        self.free_slots, self.free_cslots = list(range(F + 1)), list(range(F))
        self.pend = None
        self.ev = collections.Counter()

    def close(self):
        for o in (self.fe, self.mp, self.opt):
            o.close()

    def begin(self, depth_raw, mask, colour, request_out, loader_id=0, first_pose=None):
        import torch
        if self.frames:                                                       # Bundler.cpp:74-81
            fid, pose = self.frames[-1]["id"] + 1, self.frames[-1]["pose"].copy()
        else:
            fid, pose = loader_id, (np.eye(4, dtype=np.float32) if first_pose is None else np.asarray(first_pose, np.float32).copy())
        f = {"id": fid, "pose": pose, "depth": torch.zeros((self.H, self.W), device=self.dev), "normal": torch.zeros((self.H, self.W, 4), device=self.dev),
             "fg": torch.zeros((self.H, self.W), dtype=torch.uint8, device=self.dev), "keyframe": False, "cslot": -1}
        roi = self.fe.process_masked([depth_raw], [mask], self.H, self.W, self.K, [f["depth"]], [f["normal"]], [f["fg"]], mode=self.mode)[0]
        if roi[1] - roi[0] < 10 or roi[3] - roi[2] < 10:                     # Bundler.cpp:88-93
            self.ev["roi_fail"] += 1
            return _lib.BT_FRAME_FAIL, roi, fid
        self.fe.lfnet_request([colour], [f["fg"]], self.H, self.W, [request_out])
        f["slot"] = self.free_slots.pop()
        self.pend = f
        return _lib.BT_FRAME_OTHER, roi, fid

    def _forget(self, f):
        self.fc.forget_frame(f["id"])

    def _release(self, f):
        self.free_slots.append(f["slot"])
        if f["cslot"] >= 0:
            self.free_cslots.append(f["cslot"])

    def _cache(self, f):
        if f["cslot"] < 0:
            f["cslot"] = self.free_cslots.pop()
            self.opt.store_frames([f["cslot"]], [f["depth"]], [f["normal"]], self.H, self.W, self.K)

    def drop(self):
        f, self.pend = self.pend, None
        self._forget(f)
        self._release(f)
        self.ev["drop"] += 1
        return f["pose"]

    def end(self, kpts, desc):
        import torch
        f, self.pend = self.pend, None
        f["kpts"] = torch.from_numpy(np.ascontiguousarray(kpts, np.float32)).to(self.dev)
        f["n"] = len(kpts)
        self.mp.pool_store(f["slot"], desc)
        status = _lib.BT_FRAME_OTHER
        if self.frames:                                                       # Bundler.cpp:119-138
            last = self.frames[-1]
            n, st = self.fc.find_corres([(f, last)], [(f["slot"], last["slot"])], self.H, self.W, self.K)[(f["id"], last["id"])]
            if st == _lib.BT_PAIR_FAIL:
                self.ev["neighbour_fail"] += 1
                self._forget(f)
                self._release(f)
                return f["pose"], _lib.BT_FRAME_FAIL
            ent, (_, cnt, _, _) = self.fc.window_entries([last, f], self.dev)
            self.n_neighbour.append(int(cnt[0]))
            e = ent[:int(cnt[0])].cpu().numpy().view(np.uint8).reshape(-1).view(ENTRYJ_DTYPE)
            offset = policy.rigid_transform(xform(f["pose"], e["pos_j"]), xform(last["pose"], e["pos_i"])) if st == _lib.BT_PAIR_OK else np.eye(4, dtype=np.float32)
            f["pose"] = compose(offset, f["pose"])
        if len(self.frames) >= self.ws + 3:                                   # Bundler.cpp:149-157
            o = self.frames.pop(0)
            if not o["keyframe"]:
                self.ev["forgotten_on_pop"] += 1
                self._forget(o)
                self._release(o)
        self.frames.append(f)
        if f["id"] != 0:                                                      # selectKeyFramesForBA + optimizeGPU
            if len(self.keyframes) + 1 > self.max_ba:
                self.ev["greedy_selection"] += 1
            chosen = policy.select_keyframes(f["pose"], [k["pose"] for k in self.keyframes] or np.zeros((0, 4, 4), np.float32), self.max_ba)
            win = [self.keyframes[i] for i in chosen] + [f]
            N = len(win)
            pairs = [(win[j], win[i]) for i in range(N) for j in range(i + 1, N)]
            done = self.fc.find_corres(pairs, [(a["slot"], b["slot"]) for a, b in pairs], self.H, self.W, self.K) if pairs else {}
            if len(done) < len(pairs):
                self.ev["cached_pair_skipped"] += 1
            if any(st == _lib.BT_PAIR_FAIL and ida == f["id"] for (ida, _), (_, st) in done.items()):
                status = _lib.BT_FRAME_FAIL
            n_edges, ent, blocks = 0, None, None
            if N >= 2:
                ent, blocks = self.fc.window_entries(win, self.dev)
                n_edges = int(sum(c for c, j in zip(blocks[1], blocks[3]) if j == N - 1))
            if status != _lib.BT_FRAME_FAIL:
                if not policy.ba_gate(n_edges, self.min_edges):
                    status = _lib.BT_FRAME_NO_BA
                    self.ev["no_ba"] += 1
                elif N >= 2:
                    from bundletrack_b200.optimizer import SolveWindow
                    self._cache(f)
                    sw = SolveWindow(None, self.H, self.W, [w["depth"] for w in win], [w["normal"] for w in win], np.stack([w["pose"] for w in win]), self.K,
                                     cache_slots=[w["cslot"] for w in win], corr_dev=ent, blocks=blocks)
                    out = self.opt.optimizeWindows([sw])[0]
                    for k, w in enumerate(win):
                        w["pose"] = out[k].copy()
        if status == _lib.BT_FRAME_FAIL:                                      # Bundler.cpp:173-179
            self._forget(f)
            self.frames.pop()
            self._release(f)
            return f["pose"], status
        if status == _lib.BT_FRAME_OTHER and policy.keyframe_check(f["pose"], f["id"], f["n"], [k["pose"] for k in self.keyframes] or np.zeros((0, 4, 4), np.float32),
                                                                  self.min_feat, self.min_rot):
            self._cache(f)
            f["keyframe"] = True
            self.keyframes.append(f)
        else:
            if status == _lib.BT_FRAME_OTHER:
                self.ev["keyframe_rejected"] += 1
            if f["cslot"] >= 0:
                self.free_cslots.append(f["cslot"])
                f["cslot"] = -1
        return f["pose"], status

    def state(self):
        alive = {f["id"]: f for f in self.frames}
        alive.update({f["id"]: f for f in self.keyframes})
        ids = sorted(alive)
        return (np.array(ids, np.int32), np.stack([alive[i]["pose"] for i in ids]) if ids else np.zeros((0, 4, 4), np.float32),
                np.array([alive[i]["keyframe"] for i in ids], bool))


def _yml(**bundle):
    y = load_yml(None)
    y["bundle"].update(bundle)
    return y


# (name, yml, mask mode, frames, events): NOCS config in largest-hull mode; as-is mode with max_BA_frames = 5 (greedy selection); a
# min_fm_edges_newframe no window reaches (every frame NO_BA)
CASES = {
    "nocs_hull": (_yml(), _lib.BT_MASK_LARGEST_HULL, 60, dict(roi_fail=(0, 23), neighbour_fail=(11, 40), detect_fail=(31,))),
    "asis_ba5": (_yml(max_BA_frames=5), _lib.BT_MASK_AS_IS, 30, dict(roi_fail=(9,), neighbour_fail=(17,), detect_fail=(5,))),
    "no_ba": (_yml(min_fm_edges_newframe=10 ** 9), _lib.BT_MASK_AS_IS, 16, dict(neighbour_fail=(6,))),
}
MAX_ALIVE = 40


def _run(name):
    """Runs the Tracker and the composition side by side over a case's sequence; returns everything both produced."""
    import torch
    from bundletrack_b200.tracker import Tracker
    yml, mode, n, events = CASES[name]
    seq = synth.make_sequence(7 + len(name), n, H=H, W=W, n_feats=FEATS, **events)
    dev = torch.device("cuda", 0)
    trk = Tracker(yml, H, W, seq.K, FEATS, MAX_ALIVE, mode=mode)
    comp = Composition(yml, seq.K, FEATS, MAX_ALIVE, mode)
    rec = []
    for k in range(n):
        d, m, c = (torch.from_numpy(np.ascontiguousarray(a[k])).to(dev) for a in (seq.depth_raw, seq.mask, seq.colour))
        rq_t, rq_c = torch.zeros((400, 400, 3), dtype=torch.uint8, device=dev), torch.ones((400, 400, 3), dtype=torch.uint8, device=dev)
        st_t, roi_t = trk.begin_frame(d, m, c, rq_t, loader_id=0, first_pose=seq.poses_gt[k])
        st_c, roi_c, fid = comp.begin(d, m, c, rq_c, loader_id=0, first_pose=seq.poses_gt[k])
        r = {"k": k, "id": fid, "begin": (st_t, st_c), "roi": (roi_t, roi_c)}
        if st_t == _lib.BT_FRAME_OTHER:
            r["request"] = torch.equal(rq_t, rq_c)
            if seq.feats[k] is None:
                r["pose"] = (trk.drop_frame(), comp.drop())
                r["status"] = (_lib.BT_FRAME_FAIL, _lib.BT_FRAME_FAIL)
            else:
                desc = torch.from_numpy(seq.feats[k]["desc"]).to(dev)
                p_t, s_t = trk.end_frame(seq.feats[k]["kpts"], desc)
                p_c, s_c = comp.end(seq.feats[k]["kpts"], desc)
                r["pose"], r["status"] = (p_t, p_c), (s_t, s_c)
        r["state"] = (trk.state(), comp.state())
        rec.append(r)
    torch.cuda.synchronize()
    trk.close()
    ev = comp.ev
    comp.close()
    return seq, rec, ev


@pytest.fixture(scope="module")
def runs(cuda_device):
    return {name: _run(name) for name in CASES}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_sequence_matches_composition_byte_for_byte(runs, name):
    seq, rec, _ = runs[name]
    for r in rec:
        assert r["begin"][0] == r["begin"][1] and np.array_equal(*r["roi"]), r["k"]
        if "request" in r:
            assert r["request"], r["k"]
        if "pose" in r:
            assert r["status"][0] == r["status"][1], (r["k"], r["status"])
            assert r["pose"][0].tobytes() == r["pose"][1].tobytes(), r["k"]
        (ids_t, poses_t, kf_t), (ids_c, poses_c, kf_c) = r["state"]
        assert np.array_equal(ids_t, ids_c) and np.array_equal(kf_t, kf_c), (r["k"], ids_t, ids_c)
        assert poses_t.tobytes() == poses_c.tobytes(), r["k"]
        if r.get("status", (None,))[0] in (_lib.BT_FRAME_OTHER, _lib.BT_FRAME_NO_BA):
            assert ids_t[-1] == r["id"]          # the new frame is the newest frame alive


@pytest.mark.gpu
def test_sequences_cover_every_event(runs):
    ev = collections.Counter()
    for _, _, e in runs.values():
        ev.update(e)
    for name in ("roi_fail", "neighbour_fail", "drop", "no_ba", "keyframe_rejected", "forgotten_on_pop", "greedy_selection", "cached_pair_skipped"):
        assert ev[name] >= 1, (name, dict(ev))
    # the first frame of nocs_hull fails the ROI gate: the next frame takes its id (loader_id 0); a neighbour FAIL frees its id the same way
    _, rec, _ = runs["nocs_hull"]
    assert rec[0]["begin"][0] == _lib.BT_FRAME_FAIL and rec[1]["id"] == 0 == rec[0]["id"]
    for name, (_, _, _, events) in CASES.items():
        _, rec, _ = runs[name]
        for k in events.get("neighbour_fail", ()):
            assert rec[k]["status"][0] == _lib.BT_FRAME_FAIL and rec[k + 1]["id"] == rec[k]["id"], (name, k)
    assert all(r.get("status", (None,))[0] != _lib.BT_FRAME_OTHER for r in runs["no_ba"][1][1:])


# Tracked poses against the ground truth (the first frame gets its ground-truth pose).  Measured on an H100 80GB HBM3 (400 W power limit):
# worst case over the three sequences 9.6 degrees and 108 mm (DESIGN.md §9.4); the bounds are 1.5x that.  The error is drift: even a fit on
# the ground-truth matches of these sequences is off by 0.3-1.3 degrees per frame (few shared features per pair, depth read at the rounded
# keypoint as the reference does), and the translation error is mostly that rotation error times the 0.6-0.8 m to the object.
ACC_ROT_DEG, ACC_TRANS_M = 14.5, 0.165


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_accuracy_against_ground_truth(runs, name):
    seq, rec, _ = runs[name]
    rot, trans = [], []
    for r in rec:
        if r.get("status", (None,))[0] in (_lib.BT_FRAME_OTHER, _lib.BT_FRAME_NO_BA):
            gt = seq.poses_gt[r["k"]]
            rot.append(np.degrees(synth.rot_geodesic(r["pose"][0][:3, :3], gt[:3, :3])))
            trans.append(float(np.linalg.norm(r["pose"][0][:3, 3] - gt[:3, 3])))
    print(f"{name}: {len(rot)} frames, rotation error mean {np.mean(rot):.3f} max {np.max(rot):.3f} deg, translation mean {np.mean(trans) * 1e3:.2f} "
          f"max {np.max(trans) * 1e3:.2f} mm")
    assert np.max(rot) <= ACC_ROT_DEG and np.max(trans) <= ACC_TRANS_M


@pytest.mark.gpu
def test_pose_init_equals_rigid_transform(cuda_device):
    """bt_pose_init on the neighbour pairs of a sequence == bt_rigid_transform on the same float points, composed in the pinned order; a pair
    whose status is not OK gives the identity offset."""
    import torch
    from bundletrack_b200.frontend import FrameFrontEnd
    from bundletrack_b200.matcher import FindCorres, MatchPipeline
    seq = synth.make_sequence(3, 8, H=H, W=W, n_feats=FEATS)
    fe, mp = FrameFrontEnd(None), MatchPipeline(None, max_pairs=1, max_feats=FEATS)
    mp.pool_reserve(8)
    fc = FindCorres(mp, max_frames=8)
    lib, dev = _lib.load(), cuda_device
    frames, n_ok = [], 0
    for k in range(seq.n_frames):
        f = {"id": k, "depth": torch.zeros((H, W), device=dev), "normal": torch.zeros((H, W, 4), device=dev), "pose": seq.poses_gt[k].astype(np.float32),
             "kpts": torch.from_numpy(seq.feats[k]["kpts"]).to(dev)}
        fg = torch.zeros((H, W), dtype=torch.uint8, device=dev)
        fe.process_masked([torch.from_numpy(seq.depth_raw[k]).to(dev)], [torch.from_numpy(seq.mask[k]).to(dev)], H, W, seq.K, [f["depth"]], [f["normal"]], [fg])
        mp.pool_store(k, torch.from_numpy(seq.feats[k]["desc"]).to(dev))
        frames.append(f)
        if k == 0:
            continue
        a, b = f, frames[k - 1]
        n, st = fc.find_corres([(a, b)], [(k, k - 1)], H, W, seq.K)[(k, k - 1)]
        ent, (_, cnt, _, _) = fc.window_entries([b, a], dev)
        e = ent[:int(cnt[0])].cpu().numpy().view(np.uint8).reshape(-1).view(ENTRYJ_DTYPE)
        # poses that differ from each other, so both transforms matter
        pa = compose(synth.se3(synth.so3_exp([0.1 * k, -0.05, 0.02]), [0.01, -0.02, 0.03 * k]).astype(np.float32), a["pose"])
        pb = b["pose"]
        for status in (st, _lib.BT_PAIR_EMPTY, _lib.BT_PAIR_FAIL):
            nd = torch.tensor([n], dtype=torch.int32, device=dev)
            sd = torch.tensor([status], dtype=torch.int32, device=dev)
            out = torch.zeros(16, dtype=torch.float32, device=dev)
            _lib.check(lib.bt_pose_init(mp.ctx, ctypes.c_void_p(ent.data_ptr()), ctypes.c_void_p(nd.data_ptr()), ctypes.c_void_p(sd.data_ptr()),
                                        pa.ctypes.data_as(ctypes.c_void_p), pb.ctypes.data_as(ctypes.c_void_p), ctypes.c_void_p(out.data_ptr()), None), "bt_pose_init")
            got = out.cpu().numpy().reshape(4, 4)
            off = policy.rigid_transform(xform(pa, e["pos_j"]), xform(pb, e["pos_i"])) if status == _lib.BT_PAIR_OK else np.eye(4, dtype=np.float32)
            assert got.tobytes() == compose(off, pa).tobytes(), (k, status)
            n_ok += status == _lib.BT_PAIR_OK and not np.array_equal(off, np.eye(4, dtype=np.float32))
    assert n_ok >= 5
    for o in (fe, mp):
        o.close()


def _raises(status, fn, *a):
    with pytest.raises(_lib.BtError, match=f"status {status}:"):
        fn(*a)


@pytest.mark.gpu
def test_errors_leave_the_tracker_unchanged(cuda_device):
    import torch
    from bundletrack_b200.tracker import Tracker
    dev = cuda_device
    y = load_yml(None)
    y["keyframe"]["min_rot"] = 0          # every frame that passes becomes a keyframe: they fill max_frames_alive = 4
    seq = synth.make_sequence(5, 7, H=H, W=W, n_feats=FEATS, roi_fail=(1,))
    trk = Tracker(y, H, W, seq.K, FEATS, 4)
    lib = trk.lib
    rq = torch.zeros((400, 400, 3), dtype=torch.uint8, device=dev)
    ins = [[torch.from_numpy(np.ascontiguousarray(a[k])).to(dev) for a in (seq.depth_raw, seq.mask, seq.colour)] for k in range(seq.n_frames)]
    desc = [torch.from_numpy(f["desc"]).to(dev) for f in seq.feats]

    def same(a, b):
        return all(np.array_equal(x, z) for x, z in zip(a, b))

    s0 = trk.state()
    _raises(-1, trk.end_frame, seq.feats[0]["kpts"], desc[0])                 # end without begin
    _raises(-1, trk.drop_frame)
    assert trk.begin_frame(*ins[0], rq, loader_id=0)[0] == _lib.BT_FRAME_OTHER
    _raises(-1, trk.begin_frame, *ins[0], rq)                                 # begin twice
    big = np.zeros((FEATS + 1, 2), np.float32)
    _raises(-1, trk.end_frame, big, torch.zeros((FEATS + 1, 256), device=dev))   # n_kpts > max_feats
    st = ctypes.c_int(0)
    pose = np.zeros(16, np.float32)
    kp = seq.feats[0]["kpts"]
    for args in ((None, pose.ctypes.data_as(ctypes.c_void_p), ctypes.byref(st)), (ctypes.c_void_p(1), None, ctypes.byref(st)), (ctypes.c_void_p(1), pose.ctypes.data_as(ctypes.c_void_p), None)):
        view = None if args[0] is None else ctypes.byref(_lib.DescView(desc[0].data_ptr(), len(kp), 256, 1024))
        assert lib.bt_tracker_end_frame(trk.t, kp.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(len(kp)), view, args[1], args[2], None) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_tracker_begin_frame(trk.t, 0, None, None, None, None, None, None, ctypes.byref(st), None) == _lib.BT_ERR_INVALID_ARG
    assert same(trk.state(), s0)
    p, s = trk.end_frame(seq.feats[0]["kpts"], desc[0])                       # the pending frame goes on normally
    ids, _, kf = trk.state()
    assert s == _lib.BT_FRAME_OTHER and list(ids) == [0] and list(kf) == [True] and np.array_equal(p, np.eye(4, dtype=np.float32))
    # a frame that failed the ROI gate is done: end_frame refuses it
    assert trk.begin_frame(*ins[1], rq)[0] == _lib.BT_FRAME_FAIL
    _raises(-1, trk.end_frame, seq.feats[1]["kpts"], desc[1])
    # fill max_frames_alive with keyframes, then BT_ERR_CAPACITY before anything changes
    k, kept = 2, []
    while True:
        assert trk.begin_frame(*ins[k], rq)[0] == _lib.BT_FRAME_OTHER
        before = trk.state()
        try:
            trk.end_frame(seq.feats[k]["kpts"], desc[k])
        except _lib.BtError as e:
            assert "status -2:" in str(e) and len(before[0]) == 4
            break
        k += 1
        assert k < seq.n_frames
    assert same(trk.state(), before)
    _raises(-2, trk.end_frame, seq.feats[k]["kpts"], desc[k])                 # still pending, still refused
    trk.drop_frame()
    assert same(trk.state(), before)
    trk.close()
    # an empty tracker takes the loader's id and the first pose; a first frame whose id is not 0 has a one-frame window: NO_BA, and it does
    # not become a keyframe (Bundler.cpp:161-171,192)
    trk = Tracker(y, H, W, seq.K, FEATS, 4)
    P = compose(synth.se3(synth.so3_exp([0.3, -0.2, 0.1]), [0.01, 0.02, -0.03]).astype(np.float32), np.eye(4, dtype=np.float32))
    assert trk.begin_frame(*ins[0], rq, loader_id=7, first_pose=P)[0] == _lib.BT_FRAME_OTHER
    p, s = trk.end_frame(seq.feats[0]["kpts"], desc[0])
    ids, poses, kf = trk.state()
    assert s == _lib.BT_FRAME_NO_BA and list(ids) == [7] and list(kf) == [False] and p.tobytes() == P.tobytes() == poses[0].tobytes()
    trk.close()


@pytest.mark.gpu
def test_cpp_bundler_gpu_equals_python_tracker(tmp_path, cuda_device):
    """tests/cpp/tracker_main.cpp drives BundlerGpu (hostcpp/bt_optimizer.hpp) with a column-major Mat4 over a short sequence with every event;
    statuses, poses and request images are the Python Tracker's, byte for byte."""
    import torch
    from bundletrack_b200.tracker import Tracker
    seq = synth.make_sequence(21, 12, H=H, W=W, n_feats=FEATS, roi_fail=(3,), neighbour_fail=(6,), detect_fail=(8,))
    inp = tmp_path / "seq.bin"
    with open(inp, "wb") as f:
        np.array([seq.n_frames, H, W, FEATS], np.int32).tofile(f)
        np.asarray(seq.K, np.float32).tofile(f)
        for k in range(seq.n_frames):
            seq.depth_raw[k].tofile(f); seq.mask[k].tofile(f); seq.colour[k].tofile(f)
            ft = seq.feats[k]
            np.array([-1 if ft is None else len(ft["kpts"])], np.int32).tofile(f)
            if ft is not None:
                ft["kpts"].tofile(f); ft["desc"].tofile(f)
    exe = tmp_path / "tracker_main"
    lib_dir = os.path.join(ROOT, "bundletrack_b200", "lib")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", ROOT, os.path.join(ROOT, "tests", "cpp", "tracker_main.cpp"), "-o", str(exe),
                           "-L", lib_dir, "-lbundletrack_b200", f"-Wl,-rpath,{lib_dir}"])
    outp = tmp_path / "out.bin"
    run = subprocess.run([str(exe), str(inp), str(outp)], capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stderr
    got = np.fromfile(outp, np.uint8)
    dev = cuda_device
    trk = Tracker(None, H, W, seq.K, FEATS, 24)
    want = bytearray()
    for k in range(seq.n_frames):
        d, m, c = (torch.from_numpy(np.ascontiguousarray(a[k])).to(dev) for a in (seq.depth_raw, seq.mask, seq.colour))
        rq = torch.zeros((400, 400, 3), dtype=torch.uint8, device=dev)
        st, _ = trk.begin_frame(d, m, c, rq)
        pose = np.eye(4, dtype=np.float32)
        if st == _lib.BT_FRAME_OTHER:
            if seq.feats[k] is None:
                pose, st = trk.drop_frame(), _lib.BT_FRAME_FAIL
            else:
                pose, st = trk.end_frame(seq.feats[k]["kpts"], torch.from_numpy(seq.feats[k]["desc"]).to(dev))
        want += np.array([st], np.int32).tobytes() + pose.tobytes() + rq.cpu().numpy().tobytes()
    trk.close()
    assert got.tobytes() == bytes(want)
