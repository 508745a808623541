"""The keyframe pool's surface without a GPU: the new symbols, bt_tracker_params::max_keyframes from Python, and the ranges that are
checked before the device is looked at."""
import ctypes

from bundletrack_b200 import _lib, synth

NEW = ("bt_tracks_dev_reserve_ex", "bt_match_cache_reserve_entries", "bt_match_cache_usage", "bt_tracker_usage")


def test_keyframe_pool_symbols_are_exported():
    lib = _lib.load()
    for name in NEW:
        assert name in _lib.EXPORTS and hasattr(lib, name), name
    assert lib.bt_version() == 101


def test_max_keyframes_is_the_last_field():
    """(tests/test_tracker.py compares every field's offset with the header.)"""
    from bundletrack_b200.tracker import tracker_params
    assert _lib.TrackerParams._fields_[-1] == ("max_keyframes", ctypes.c_int)
    assert tracker_params(None, 480, 640, synth.NOCS_K, 2000, 8).max_keyframes == 0
    assert tracker_params(None, 480, 640, synth.NOCS_K, 2000, 8, max_keyframes=256).max_keyframes == 256


def test_out_of_range_sizes_are_refused_before_the_device():
    from bundletrack_b200.tracker import tracker_params
    lib = _lib.load()
    t = ctypes.c_void_p()
    for F, K in ((8, -1), (8, 1025), (65, 0), (65, 16), (1, 16)):
        p = tracker_params(None, 480, 640, synth.NOCS_K, 2000, F, max_keyframes=K)
        assert lib.bt_tracker_create(ctypes.byref(t), 0, ctypes.byref(p)) == _lib.BT_ERR_INVALID_ARG and not t, (F, K)
    assert lib.bt_tracks_dev_reserve_ex(None, 8, 4, 3) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_match_cache_reserve_entries(None, 8, ctypes.c_longlong(100)) == _lib.BT_ERR_INVALID_ARG
    assert lib.bt_tracker_usage(None, None, None, None, None) == _lib.BT_ERR_INVALID_ARG
