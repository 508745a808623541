"""The tracker's surface without a GPU: exported symbols, the ctypes layout of bt_tracker_params, BT_ERR_NO_DEVICE, and the synthetic
sequence generator (deterministic, events where the knobs put them)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from bundletrack_b200 import _lib, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("bt_pose_init", "bt_tracker_create", "bt_tracker_destroy", "bt_tracker_begin_frame", "bt_tracker_end_frame", "bt_tracker_drop_frame", "bt_tracker_state")


def test_tracker_symbols_are_exported():
    lib = _lib.load()
    for name in NEW:
        assert name in _lib.EXPORTS and hasattr(lib, name), name


def test_tracker_params_layout_matches_the_header(tmp_path):
    fields = [f for f, _ in _lib.TrackerParams._fields_]
    src = tmp_path / "tp.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "bundletrack_b200.h"\nint main(){printf("%zu' + " %zu" * len(fields) + '\\n", sizeof(bt_tracker_params)'
                   + "".join(f", offsetof(bt_tracker_params, {f})" for f in fields) + ");return 0;}\n")
    exe = tmp_path / "tp"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [ctypes.sizeof(_lib.TrackerParams)] + [getattr(_lib.TrackerParams, f).offset for f in fields]


def test_tracker_params_from_yml():
    from bundletrack_b200.tracker import tracker_params
    y = {"bundle": {"num_iter_outter": 7, "num_iter_inner": 5, "window_size": 3, "max_BA_frames": 9, "robust_delta": 0.005, "min_fm_edges_newframe": 15,
                    "image_downscale": 4},
         "keyframe": {"min_interval": 1, "min_feat_num": 20, "min_rot": 7.5},
         "feature_corres": {"max_dist_no_neighbor": 0.02, "max_normal_no_neighbor": 45, "max_dist_neighbor": 10000, "max_normal_neighbor": 180},
         "ransac": {"max_iter": 1000, "inlier_dist": 0.004}, "p2p": {"max_dist": 0.02, "max_normal_angle": 45}, "data_dir": "/data/YCBInEOAT/x"}
    p = tracker_params(y, 480, 640, synth.NOCS_K, 2000, 32)
    assert (p.window_size, p.max_BA_frames, p.min_fm_edges_newframe, p.min_feat_num, p.ransac_trials) == (3, 9, 15, 20, 1000)
    assert p.min_rot_deg == np.float32(7.5) and p.ransac_inlier_dist == np.float32(0.004) and p.mask_mode == _lib.BT_MASK_AS_IS
    assert (p.H, p.W, p.max_feats, p.max_frames_alive) == (480, 640, 2000, 32) and p.fx == np.float32(synth.NOCS_K[0])


def test_tracker_create_without_gpu_is_no_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from bundletrack_b200.tracker import Tracker, tracker_params
    lib = _lib.load()
    t = ctypes.c_void_p()
    p = tracker_params(None, 480, 640, synth.NOCS_K, 2000, 32)
    assert lib.bt_tracker_create(ctypes.byref(t), 0, ctypes.byref(p)) == _lib.BT_ERR_NO_DEVICE and not t
    p.max_frames_alive = 65                                  # out-of-range parameters are refused before the device is looked at
    assert lib.bt_tracker_create(ctypes.byref(t), 0, ctypes.byref(p)) == _lib.BT_ERR_INVALID_ARG
    with pytest.raises(_lib.BtError):
        Tracker(None, 480, 640, synth.NOCS_K, 2000, 32)


def test_make_sequence_is_deterministic_and_places_events():
    kw = dict(H=96, W=128, n_feats=120, roi_fail=(1,), neighbour_fail=(2,), detect_fail=(4,))
    a, b = synth.make_sequence(4, 6, **kw), synth.make_sequence(4, 6, **kw)
    for x, y in ((a.depth_raw, b.depth_raw), (a.mask, b.mask), (a.colour, b.colour), (a.poses_gt, b.poses_gt)):
        assert np.array_equal(x, y)
    for fa, fb in zip(a.feats, b.feats):
        assert (fa is None) == (fb is None)
        if fa is not None:
            assert np.array_equal(fa["kpts"], fb["kpts"]) and np.array_equal(fa["desc"], fb["desc"])
    assert a.mask.shape == (6, 96, 128) and a.colour.shape == (6, 96, 128, 3) and a.mask.dtype == np.uint8 and a.colour.dtype == np.uint8
    for k in range(6):
        assert (a.mask[k].max() == 0) == (k == 1)                      # the ROI event: an empty mask
        assert (a.feats[k] is None) == (k == 4)                        # the detection event
    u, v = np.rint(a.feats[2]["kpts"]).astype(int).T                  # the neighbour event: every keypoint on a pixel without depth
    assert len(u) == 120 and (a.depth_raw[2][v, u] == 0).all()
    u, v = np.rint(a.feats[3]["kpts"]).astype(int).T
    assert (a.depth_raw[3][np.clip(v, 0, 95), np.clip(u, 0, 127)] > 0).mean() > 0.5
    # the mask has the silhouette and a separate distractor blob; the motion is 2-6 degrees per frame
    assert (a.mask[0] > 0).sum() > (a.depth_raw[0] > 0).sum()
    for k in range(1, 6):
        ang = np.degrees(synth.rot_geodesic(a.poses_gt[k - 1][:3, :3], a.poses_gt[k][:3, :3]))
        assert 1.9 <= ang <= 6.1
    c = synth.make_sequence(5, 6, **kw)
    assert not np.array_equal(a.depth_raw, c.depth_raw)
