"""The tracker with a keyframe pool (bt_tracker_params::max_keyframes) over a sequence that admits more than 64 keyframes, byte for byte against
the composition of tests/test_tracker_gpu.py sized for the same frames; the same results whatever the slot assignment; a full pool."""
import numpy as np
import pytest

from bundletrack_b200 import _lib, synth
from bundletrack_b200.config import load_yml
from test_tracker_gpu import CASES, FEATS, H, W, Composition

pytestmark = pytest.mark.gpu


def _inputs(seq, k, dev):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(a[k])).to(dev) for a in (seq.depth_raw, seq.mask, seq.colour)]


def _same_state(a, b):
    return all(np.asarray(x).tobytes() == np.asarray(z).tobytes() for x, z in zip(a, b))


def _feed(trk, seq, k, ins, desc, rq):
    """One frame through a Tracker: (begin status, roi, end status or None, pose or None)."""
    st, roi = trk.begin_frame(*ins, rq, loader_id=0, first_pose=seq.poses_gt[k])
    if st != _lib.BT_FRAME_OTHER:
        return st, roi, None, None
    if seq.feats[k] is None:
        return st, roi, _lib.BT_FRAME_FAIL, trk.drop_frame()
    pose, s = trk.end_frame(seq.feats[k]["kpts"], desc)
    return st, roi, s, pose


def test_long_sequence_matches_composition(cuda_device):
    """300 frames (NOCS config, largest-hull mode): Tracker(max_frames_alive=8, max_keyframes=128) against Composition(max_frames_alive=136),
    statuses, poses, request images and every step's frames alive byte for byte; more than 64 keyframes at the end, which the tracker
    without a pool (max_frames_alive = 64) refuses with BT_ERR_CAPACITY."""
    import torch
    from bundletrack_b200.tracker import Tracker
    dev = cuda_device
    n = 300
    seq = synth.make_sequence(11, n, H=H, W=W, n_feats=FEATS)
    y, mode = load_yml(None), _lib.BT_MASK_LARGEST_HULL
    trk = Tracker(y, H, W, seq.K, FEATS, 8, mode=mode, max_keyframes=128)
    comp = Composition(y, seq.K, FEATS, 8 + 128, mode)
    legacy = Tracker(y, H, W, seq.K, FEATS, 64, mode=mode)
    legacy_capacity_at = None
    n_other = 0
    for k in range(n):
        ins = _inputs(seq, k, dev)
        desc = None if seq.feats[k] is None else torch.from_numpy(seq.feats[k]["desc"]).to(dev)
        rq_t, rq_c = torch.zeros((400, 400, 3), dtype=torch.uint8, device=dev), torch.ones((400, 400, 3), dtype=torch.uint8, device=dev)
        st_t, roi_t, s_t, p_t = _feed(trk, seq, k, ins, desc, rq_t)
        st_c, roi_c, _ = comp.begin(*ins, rq_c, loader_id=0, first_pose=seq.poses_gt[k])
        assert st_t == st_c and np.array_equal(roi_t, roi_c), k
        if st_c == _lib.BT_FRAME_OTHER:
            assert torch.equal(rq_t, rq_c), k
            if seq.feats[k] is None:
                p_c, s_c = comp.drop(), _lib.BT_FRAME_FAIL
            else:
                p_c, s_c = comp.end(seq.feats[k]["kpts"], desc)
            assert s_t == s_c and p_t.tobytes() == p_c.tobytes(), (k, s_t, s_c)
            n_other += s_t == _lib.BT_FRAME_OTHER
        assert _same_state(trk.state(), comp.state()), k
        if legacy is not None:
            rq_l = torch.zeros((400, 400, 3), dtype=torch.uint8, device=dev)
            try:
                _feed(legacy, seq, k, ins, desc, rq_l)
            except _lib.BtError as e:
                assert "status -2:" in str(e), e
                legacy_capacity_at = k
                legacy.close()
                legacy = None
    torch.cuda.synchronize()
    ids, _, kf = trk.state()
    pts, pairs, ents = trk.usage()
    print(f"{n} frames: {int(kf.sum())} keyframes, {len(ids)} frames alive, {pts} map points alive, {pairs} cached pairs holding {ents} entries; "
          f"the tracker without a pool stopped at frame {legacy_capacity_at}")
    assert int(kf.sum()) > 64 and n_other >= n // 2
    assert legacy_capacity_at is not None and legacy_capacity_at < n - 1
    assert pairs > 0 and ents > 0 and pts > 0
    trk.close()
    comp.close()


def test_slot_assignment_does_not_leak_into_results(cuda_device):
    """The 60-frame NOCS sequence of tests/test_tracker_gpu.py through max_keyframes = 0 with max_frames_alive = 32 and through
    max_keyframes = 32 with max_frames_alive = 8: identical statuses, poses and frames alive."""
    import torch
    from bundletrack_b200.tracker import Tracker
    dev = cuda_device
    yml, mode, n, events = CASES["nocs_hull"]
    seq = synth.make_sequence(7 + len("nocs_hull"), n, H=H, W=W, n_feats=FEATS, **events)
    a = Tracker(yml, H, W, seq.K, FEATS, 32, mode=mode)
    b = Tracker(yml, H, W, seq.K, FEATS, 8, mode=mode, max_keyframes=32)
    n_kf = 0
    for k in range(n):
        ins = _inputs(seq, k, dev)
        desc = None if seq.feats[k] is None else torch.from_numpy(seq.feats[k]["desc"]).to(dev)
        ra = _feed(a, seq, k, ins, desc, torch.zeros((400, 400, 3), dtype=torch.uint8, device=dev))
        rb = _feed(b, seq, k, ins, desc, torch.zeros((400, 400, 3), dtype=torch.uint8, device=dev))
        assert ra[0] == rb[0] and ra[2] == rb[2] and np.array_equal(ra[1], rb[1]), k
        assert (ra[3] is None and rb[3] is None) or ra[3].tobytes() == rb[3].tobytes(), k
        sa = a.state()
        assert _same_state(sa, b.state()), k
        n_kf = int(sa[2].sum())
    assert n_kf >= 10, n_kf
    a.close()
    b.close()


def test_full_keyframe_pool_is_capacity(cuda_device):
    """max_keyframes = 3 and min_rot = 0 (every frame that passes becomes a keyframe): the end_frame that could admit a fourth returns
    BT_ERR_CAPACITY and changes nothing, again on a retry; drop_frame still finishes the frame."""
    import torch
    from bundletrack_b200.tracker import Tracker
    dev = cuda_device
    y = load_yml(None)
    y["keyframe"]["min_rot"] = 0
    seq = synth.make_sequence(5, 8, H=H, W=W, n_feats=FEATS)
    trk = Tracker(y, H, W, seq.K, FEATS, 8, max_keyframes=3)
    assert trk.state()[0].shape == (0,)
    rq = torch.zeros((400, 400, 3), dtype=torch.uint8, device=dev)
    k = 0
    while True:
        ins = _inputs(seq, k, dev)
        desc = torch.from_numpy(seq.feats[k]["desc"]).to(dev)
        assert trk.begin_frame(*ins, rq, loader_id=0)[0] == _lib.BT_FRAME_OTHER
        before = trk.state()
        try:
            trk.end_frame(seq.feats[k]["kpts"], desc)
        except _lib.BtError as e:
            assert "status -2:" in str(e) and "keyframe pool" in str(e), e
            break
        k += 1
        assert k < seq.n_frames
    ids, _, kf = before
    assert int(kf.sum()) == 3 and len(ids) - 3 + 1 <= 8          # the pool, not max_frames_alive, refused the frame
    assert _same_state(trk.state(), before)
    with pytest.raises(_lib.BtError, match="status -2:"):
        trk.end_frame(seq.feats[k]["kpts"], desc)
    assert _same_state(trk.state(), before)
    trk.drop_frame()
    assert _same_state(trk.state(), before)
    trk.close()
