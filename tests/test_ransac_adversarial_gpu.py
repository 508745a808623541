"""Batched RANSAC (ransac.cu) against its float64 restatement on the pairs of oracle/ransac_families.py: exact count ties between models,
winners in the last check step of the last chunk behind an early decoy, tying trials racing to publish over 512 pairs, the threshold at
d2_max and one float32 either side, thresholds 0, -1, NaN and +inf with an odd tail, degenerate or non-finite samples, probes on the
boundary between the kernel's contraction and the uncontracted ones, and a tie and a chunk layout through the matcher chain.

Given the device's own float32 poses (bt_ransac_debug_trials) the result is deterministic, so nothing is allowed slack:
  * good flags: n >= 3, three distinct ids and six finite sample points;
  * every trial's count restated from its pose (matcher_oracle.counts_from_poses); the winner is (max count, lowest trial), the readout's
    count is that count and n_inliers equals it; the inlier ids are exactly the winner's restated set, ascending, at the pair's offset;
  * the fit of every good trial: R^T R = I to 1e-5, det R > 0, its residual sum of squares on its own samples at most the float64 Kabsch
    minimum plus 64 u times the samples' scatter plus 3 (16 u M)^2 (M the largest coordinate), and on well-conditioned samples every entry of
    R within 2e-5 and of t within 2e-5 (1 + M) of Kabsch.  These bounds hold for a float32 emulation of k_ransac_model
    (test_oracle_ransac_families.py); the worst observed ratio is printed."""
import numpy as np
import pytest

from oracle import matcher_oracle as mo
from oracle import ransac_families as rf

pytestmark = pytest.mark.gpu
U3 = rf.table()
CALLS = {c["name"]: c for c in rf.all_calls()}
FIT_WORST = {"rss": 0.0, "pose": 0.0}


@pytest.fixture(scope="module")
def ransac(cuda_device):
    from bundletrack_b200.matcher import Ransac
    r = Ransac(max_pairs=rf.PUB_PAIRS, max_pts=rf.MAX_PTS, max_trials=rf.MAX_TRIALS)
    yield r
    print(f"fit: worst rss excess / tolerance {FIT_WORST['rss']:.3g}, worst pose error / tolerance {FIT_WORST['pose']:.3g}")
    r.close()


def _run(r, call, dev):
    import torch
    A = [torch.from_numpy(a).to(dev) for a, _ in call["pairs"]]
    B = [torch.from_numpy(b).to(dev) for _, b in call["pairs"]]
    ids = r.ransac_pairs(A, B, call["n_trials"], call["thresh"])
    _, best = r.debug(call["n_trials"], len(A))
    return [i.cpu().numpy() for i in ids], best


def _check_fits(A, B, sids, poses, good, well=()):
    for t in np.nonzero(good)[0]:
        s, d = A[sids[t], :3].astype(np.float64), B[sids[t], :3].astype(np.float64)
        P = poses[t].astype(np.float64)
        R = P[:, :3]
        assert np.abs(R.T @ R - np.eye(3)).max() <= 1e-5 and np.linalg.det(R) > 0, (t, P)
        Rk, tk, rss = mo.kabsch64(s, d)
        rss_tol, r_tol, t_tol = rf.fit_tolerances(s, d)
        got = ((d - (s @ R.T + P[:, 3])) ** 2).sum()
        assert got <= rss + rss_tol, (t, got, rss, rss_tol)
        FIT_WORST["rss"] = max(FIT_WORST["rss"], (got - rss) / rss_tol)
        if t in well:
            err = max(np.abs(R - Rk).max() / r_tol, np.abs(P[:, 3] - tk).max() / t_tol)      # in units of the tolerance
            assert err <= 1.0, (t, err, P, Rk, tk)
            FIT_WORST["pose"] = max(FIT_WORST["pose"], err)


def _check_pair(r, p, A, B, call, got_ids, best_trial, exp, well=(), fits=True):
    """One pair against the restatement over its device poses; returns (winner, count)."""
    T, th = call["n_trials"], call["thresh"]
    poses, good, best_count = r.debug_trials(p, T)
    n = len(A)
    sids = mo.ransac_sample_ids(U3[:T], n)
    assert np.array_equal(good != 0, mo.ransac_expected_good(A, B, sids, n)), (call["name"], p)
    assert np.isfinite(poses[good != 0]).all()
    counts, marg = mo.counts_from_poses(A, B, poses, good, th)
    assert marg.sum() == 0, (call["name"], p, np.nonzero(marg)[0][:5])
    W, C = mo.ransac_winner(counts, good)
    assert (int(best_trial), best_count) == (W, C), (call["name"], p, n, int(best_trial), best_count, W, C)
    want = np.nonzero(mo.ransac_classify(poses[W], A, B, th)[0])[0] if W >= 0 else np.zeros(0, np.int64)
    assert len(got_ids) == max(C, 0) and np.array_equal(got_ids, want), (call["name"], p, len(got_ids), C)
    if exp is not None:
        assert (W, C) == exp, (call["name"], p, (W, C), exp)
    if np.isfinite(th):
        bad = ~(np.isfinite(A[:, :3]).all(1) & np.isfinite(B[:, :3]).all(1))
        assert not np.isin(np.nonzero(bad)[0], got_ids).any()
    if fits:
        _check_fits(A, B, sids, poses, good != 0, well)
    return W, C, poses, good


@pytest.mark.parametrize("name", [n for n in CALLS if n != "publication"])
def test_family(ransac, cuda_device, name):
    call = CALLS[name]
    ids, best = _run(ransac, call, cuda_device)
    well = [t for t, c in call.get("trials", {}).items() if c in rf.WELL]
    for p, ((A, B), exp) in enumerate(zip(call["pairs"], call["expect"])):
        _check_pair(ransac, p, A, B, call, ids[p], best[p], exp, well)
    if name == "degenerate":
        bad = call["nonfinite"]
        assert not np.isin(bad, ids[0]).any()


def test_publication_order(ransac, cuda_device):
    """The tying pair repeated over 512 pairs: every pair gives pair 0's good flags and poses, winner and inlier ids, and pair 0 is the restatement's."""
    call = CALLS["publication"]
    ids, best = _run(ransac, call, cuda_device)
    A, B = call["pairs"][0]
    W, C, poses0, good0 = _check_pair(ransac, 0, A, B, call, ids[0], best[0], call["expect"][0])
    lost = []
    for p in range(1, len(call["pairs"])):
        poses, good, cnt = ransac.debug_trials(p, call["n_trials"])
        assert np.array_equal(good, good0) and np.array_equal(poses[good0 != 0].view(np.uint32), poses0[good0 != 0].view(np.uint32)), p
        if (int(best[p]), cnt) != (W, C) or not np.array_equal(ids[p], ids[0]):
            lost.append((p, int(best[p]), cnt, len(ids[p])))
    assert not lost, lost[:8]


def test_seed_table_across_calls(ransac, cuda_device):
    """Seed 0, then 1, then 0 in one context with n_trials growing 1 -> 257 -> MAX_TRIALS: the seed-0 table comes back each time."""
    import torch
    A, B = CALLS["tie_0"]["pairs"][0]
    a, b = torch.from_numpy(A).to(cuda_device), torch.from_numpy(B).to(cuda_device)
    for seed, T in ((0, 1), (1, 257), (0, rf.MAX_TRIALS)):
        ransac.ransac_pairs([a], [b], T, rf.THRESH, seed=seed)
        u3, _ = ransac.debug(T, 1)
        if seed == 0:
            assert np.array_equal(u3, U3[:T]), (seed, T)
        else:
            assert not np.array_equal(u3, U3[:T])


def test_operation_order(cuda_device):
    """k_ransac_eval chooses the winner with the documented contraction (mul y, fma x, fma z, add t; mul dy, fma dx, fma dz) and
    k_ransac_inliers reports its set: the two must agree point for point.  Run once, read the winner's device pose, move never-sampled
    probes onto the boundary between that order and each uncontracted one (matcher_oracle.RANSAC_ORDERS: squares, model point, both),
    half accepted and half rejected by the documented order; run again.  Every good trial's pose stays bit-equal, the winner stays, its count and
    n_inliers grow by the accepted probes, and the ids are exactly the documented order's set."""
    from bundletrack_b200.matcher import Ransac
    call, probe_ids = rf.op_order()
    T, th = call["n_trials"], call["thresh"]
    r = Ransac(max_pairs=1, max_pts=rf.OP_N, max_trials=T)
    try:
        A, B = call["pairs"][0]
        ids1, best1 = _run(r, call, cuda_device)
        W, C, poses1, good1 = _check_pair(r, 0, A, B, call, ids1[0], best1[0], call["expect"][0])
        probes = rf.op_order_probes(poses1[W], probe_ids, th, np.random.default_rng(11))
        A2, B2 = A.copy(), B.copy()
        for i, (a, b, _) in probes.items():
            A2[i, :3], B2[i, :3] = a, b
        n_in = sum(k for _, _, k in probes.values())
        assert 0 < n_in < len(probes)
        ids2, best2 = _run(r, dict(call, pairs=[(A2, B2)]), cuda_device)
        poses2, good2, cnt2 = r.debug_trials(0, T)
        assert np.array_equal(good2, good1) and np.array_equal(poses2[good1 != 0].view(np.uint32), poses1[good1 != 0].view(np.uint32))
        counts, marg = mo.counts_from_poses(A2, B2, poses2, good2, th)
        assert marg[W] == len(probes) and marg.sum() == marg[W], (marg[W], marg.sum())
        assert mo.ransac_winner(counts, good2) == (W, C + n_in) == (int(best2[0]), cnt2), (int(best2[0]), cnt2, W, C, n_in)
        dec, _ = mo.ransac_classify(poses2[W], A2, B2, th)
        assert np.array_equal(ids2[0], np.nonzero(dec)[0])
        assert all((i in set(ids2[0].tolist())) == k for i, (_, _, k) in probes.items())
    finally:
        r.close()


def _ransac_readout(lib, ctx, pair, n_trials, n_pairs):
    import ctypes
    from bundletrack_b200 import _lib
    from bundletrack_b200.matcher import ransac_debug_trials
    best = np.zeros(n_pairs, np.int32)
    _lib.check(lib.bt_ransac_debug(ctx, None, 0, _lib.ptr(best), n_pairs), "bt_ransac_debug")
    return (int(best[pair]),) + ransac_debug_trials(lib, ctx, pair, n_trials)


def test_fused_chain(cuda_device):
    """A tie pair (two clusters of 24 under different motions) and a chunk pair (1100 points, the winner's other members in the last 128,
    a decoy one smaller below 1024) through bt_match_pairs_ex with prune thresholds every row passes.  The chain's RANSAC points are the
    rows in order; the readout after the chain gives the restated winner over its own poses, the emitted entries are exactly the restated
    inlier rows, and the standalone call on the same points gives the same good flags and poses, winner and ids."""
    import copy
    import torch
    import test_find_corres_adversarial_gpu as fca
    from bundletrack_b200.config import load_yml
    from bundletrack_b200.matcher import MatchPipeline, Ransac
    from oracle import corres_families as cf
    T, th = rf.MAX_TRIALS, rf.CHAIN_THRESH
    built = rf.chain_frames()
    frames = [(A, B) for A, B, _ in built]
    yml = copy.deepcopy(load_yml(None))
    yml["ransac"]["max_iter"], yml["ransac"]["inlier_dist"] = T, th
    mp = MatchPipeline(yml, max_pairs=2, max_feats=max(len(A["kpts"]) for A, _ in frames))
    r = Ransac(max_pairs=1, max_pts=1100, max_trials=T)
    try:
        cap = sum(len(A["kpts"]) + len(B["kpts"]) for A, B in frames)
        got = fca._match_ex(mp, fca._on_device(frames, cuda_device), None, fca.WIDE, T, th, cap, cuda_device)
        chain, want_rows = [], []
        for p, (A, B, clusters) in enumerate(built):
            cand, _ = mo.find_corres(A, B, cf.K, fca.WIDE, U3[:1], th)
            assert len(cand) == len(B["kpts"])
            PA, PB = np.zeros((len(cand), 4), np.float32), np.zeros((len(cand), 4), np.float32)
            PA[:, :3], PB[:, :3] = cand[:, 4:7], cand[:, 7:10]          # identity frame poses: the model points are the camera points
            best, poses, good, cnt = _ransac_readout(mp.lib, mp.ctx, p, T, 2)
            counts, marg = mo.counts_from_poses(PA, PB, poses, good, th)
            assert marg.sum() == 0
            W, C = mo.ransac_winner(counts, good)
            assert (best, cnt) == (W, C) == (clusters[0][0], len(clusters[0][1])), (p, best, cnt, W, C, clusters[0][0])
            want_rows.append(cand[np.nonzero(mo.ransac_classify(poses[W], PA, PB, th)[0])[0]])
            chain.append((PA, PB, poses, good, W, C))
        fca._check_emitted(got, frames, want_rows, cap)
        for PA, PB, poses, good, W, C in chain:           # the same points through bt_ransac_pairs
            ids = r.ransac_pairs([torch.from_numpy(PA).to(cuda_device)], [torch.from_numpy(PB).to(cuda_device)], T, th)[0].cpu().numpy()
            _, best = r.debug(T, 1)
            p2, g2, c2 = r.debug_trials(0, T)
            assert (int(best[0]), c2) == (W, C) and np.array_equal(g2, good)
            assert np.array_equal(p2[good != 0].view(np.uint32), poses[good != 0].view(np.uint32))      # (other rows are never written)
            assert np.array_equal(ids, np.nonzero(mo.ransac_classify(poses[W], PA, PB, th)[0])[0])
    finally:
        r.close()
        mp.close()
