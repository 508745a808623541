"""kNN oracle (exact brute force) vs OpenCV's CPU BFMatcher — the reference's own NO_OPENCV_CUDA path
(/root/reference/src/FeatureManager.cpp:266-269) — and its edge cases."""
import numpy as np
import pytest

from bundletrack_b200 import synth
from oracle import matcher_oracle as mo
from oracle.knn_families import PLACEMENTS, cluster_case


def test_knn_matches_opencv_bfmatcher():
    cv2 = pytest.importorskip("cv2")
    a, b, _, _ = synth.make_descriptors(1, 700, 900)
    i1, d1 = mo.knn(a, b)
    i2, d2 = mo.knn_cv2(a, b)
    assert np.array_equal(i1, i2)
    assert np.abs(d1 - d2).max() < 1e-6


def test_knn_planted_matches_are_nearest():
    a, b, ia, ib = synth.make_descriptors(2, 400, 500, match_frac=0.5, noise=0.02)
    idx, dist = mo.knn(b[ib], a, k=1)
    assert (idx[:, 0] == ia).mean() > 0.99
    assert (np.diff(mo.knn(a, b)[1], axis=1) >= 0).all()       # ascending


def test_knn_ties_go_to_lower_index_and_padding():
    a = np.zeros((3, 256), np.float32); a[:, 0] = 1
    b = np.zeros((4, 256), np.float32); b[:, 0] = [1, 1, 0.5, 1]   # rows 0,1,3 identical
    idx, dist = mo.knn(a, b, k=5)
    assert idx[0].tolist() == [0, 1, 3, 2, -1]
    assert np.isinf(dist[0, 4]) and dist[0, 0] == 0
    e_i, e_d = mo.knn(a[:0], b)
    assert e_i.shape == (0, 5)
    z_i, z_d = mo.knn(a, b[:0])
    assert (z_i == -1).all() and np.isinf(z_d).all()


@pytest.mark.parametrize("C", [1.0, 1e2, 1e3, 1e4])
def test_knn_equals_direct_brute_force_under_common_offset(C):
    """Descriptors sharing a large offset, C c + N(0, 1e-3) with c ~ N(0, 1): the expansion |q|^2 + |t|^2 - 2 q.t cancels, so knn() may only use it to
    preselect (at C = 1e4 a fixed short list taken from it picks the wrong rows for most queries)."""
    rng = np.random.default_rng(int(C))
    c = rng.normal(size=256)
    a = (C * c + rng.normal(0, 1e-3, (300, 256))).astype(np.float32)
    b = (C * c + rng.normal(0, 1e-3, (400, 256))).astype(np.float32)
    for q, t in ((a, b), (b, a)):
        i1, d1 = mo.knn(q, t, 5)
        i2, d2 = mo.knn_direct(q, t, 5)
        assert np.array_equal(i1, i2)
        assert np.array_equal(d1, d2)


@pytest.mark.parametrize("family,placement", [("tie", "g17"), ("tie", "one_group"), ("near", "spread12"), ("near", "g5")])
def test_knn_equals_direct_brute_force_on_ties_and_near_ties(family, placement):
    """The adversarial families of the GPU tests (exact ties, near-ties 2^-20 apart in reverse index order), k = 1..8."""
    qs, ts = cluster_case(family, PLACEMENTS[placement], seed=3)
    for k in (1, 4, 8):
        for q, t in ((qs, ts), (ts, qs)):
            i1, d1 = mo.knn(q, t, k)
            i2, d2 = mo.knn_direct(q, t, k)
            assert np.array_equal(i1, i2) and np.array_equal(d1, d2)
    rows = sorted(PLACEMENTS[placement], reverse=not family == "tie")     # near-ties: nearest member at the highest row; ties: lowest first
    m = min(8, len(rows))
    assert mo.knn(qs, ts, 8)[0][37, :m].tolist() == rows[:m]


def test_knn_direct_pads_and_breaks_ties_by_index():
    a = np.zeros((2, 256), np.float32)
    b = np.zeros((3, 256), np.float32); b[:, 0] = [1, 1, 0.5]
    idx, dist = mo.knn_direct(a, b, 5)
    assert idx[0].tolist() == [2, 0, 1, -1, -1] and np.isinf(dist[0, 3:]).all()
    assert (mo.knn_direct(a, b[:0], 3)[0] == -1).all() and mo.knn_direct(a[:0], b, 3)[0].shape == (0, 3)


def test_ransac_oracle_against_reference_golden():
    """Pins mo.ransac_pair (float64 Kabsch fit, deterministic arg-max) to the reference's own ransacMultiPairGPU: on the committed
    inputs its winner has at least the reference's inlier count up to borderline points, and the two sets describe the same motion."""
    import os
    gold = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    path = os.path.join(gold, "ref_ransac.npz")
    if not os.path.exists(path):
        pytest.skip("tests/golden/ref_ransac.npz not generated yet")
    g = np.load(path)
    u3 = np.load(os.path.join(gold, "curand_xorwow_seed0.npy"))[: int(g["n_trials"])]
    same = 0
    for k in range(int(g["n_cases"])):
        A, B, ref, thr = g[f"A{k}"], g[f"B{k}"], g[f"ref{k}"], float(g["thresh"][k])
        ids, best, counts = mo.ransac_pair(A, B, u3, thr)
        assert len(ids) >= len(ref) - max(2, len(ref) // 100), (k, len(ids), len(ref))
        assert len(np.intersect1d(ids, ref)) >= min(len(ids), len(ref)) - max(2, len(ref) // 100)
        same += int(np.array_equal(ids, ref))
    assert same >= 1
