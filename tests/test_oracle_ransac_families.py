"""The RANSAC families (oracle/ransac_families.py) land where they claim, checked on the CPU: the intended trial is the lowest pure one and
wins with the intended count under float64 Kabsch fits rounded to float32 (the exact [I | 0] of the float32 fit emulation for the
identity-motion family), no point lies within float32 reach of the threshold, the equality probes compute exactly to d2_max and the floats
next to it in every contraction order, and the fit tolerances of the GPU test hold for the float32 emulation of the 3-point fit."""
import numpy as np
import pytest

from oracle import matcher_oracle as mo
from oracle import ransac_families as rf

CALLS = {c["name"]: c for c in rf.all_calls()}
U3 = rf.table()


def kabsch_poses(A, B, ids, good):
    """[T, 3, 4] float32: the float64 Kabsch fit of every good trial's samples, rounded; NaN for the others."""
    out = np.full((len(ids), 3, 4), np.nan, np.float32)
    for t in np.nonzero(good)[0]:
        R, tt, _ = mo.kabsch64(A[ids[t], :3], B[ids[t], :3])
        out[t, :, :3], out[t, :, 3] = R, tt
    return out


def identity_poses(A, B, ids, good):
    """[T, 3, 4] float32 from the float32 fit emulation; every good trial of an identity-motion pair must come out exactly [I | 0]."""
    out = np.full((len(ids), 3, 4), np.nan, np.float32)
    eye = np.concatenate([np.eye(3), np.zeros((3, 1))], 1).astype(np.float32)
    for t in np.nonzero(good)[0]:
        P = mo.ransac_model_f32(A[ids[t], :3], B[ids[t], :3])
        assert P is not None and np.array_equal(P, eye), (t, P)
        out[t] = P
    return out


@pytest.mark.parametrize("name", list(CALLS))
def test_family_winner_and_count(name):
    call = CALLS[name]
    T = call["n_trials"]
    pairs = call["pairs"][:1] if name == "publication" else call["pairs"]     # (the same pair repeated)
    for p, ((A, B), exp) in enumerate(zip(pairs, call["expect"])):
        n = len(A)
        ids = mo.ransac_sample_ids(U3[:T], n)
        good = mo.ransac_expected_good(A, B, ids, n)
        if n < 3:
            assert not good.any() and exp is None
            continue
        if exp is None:
            continue
        poses = (identity_poses if name.startswith("eq_") else kabsch_poses)(A, B, ids, good)
        counts, marg = mo.counts_from_poses(A, B, poses, good, call["thresh"])
        assert marg.sum() == 0, (name, p, np.nonzero(marg)[0][:5])
        assert mo.ransac_winner(counts, good) == exp, (name, p, n, mo.ransac_winner(counts, good), exp)
        if exp[1] > 0 and np.isfinite(call["thresh"]) and call["thresh"] > 0 and not name.startswith("eq_"):
            pure = counts == exp[1]
            assert rf.lowest_pure(ids[:T], np.nonzero(mo.ransac_classify(poses[exp[0]], A, B, call["thresh"])[0])[0]) == exp[0]
            if name.startswith("tie_") and name != "tie_last":     # an exact tie between two models: a higher trial of another cluster
                others = np.nonzero(pure)[0]
                R0 = poses[exp[0], :, :3]
                assert any(np.abs(poses[t, :, :3] - R0).max() > 0.1 for t in others), name


def test_equality_probes_sit_on_d2_max():
    eye = np.concatenate([np.eye(3), np.zeros((3, 1))], 1).astype(np.float32)
    seen = 0
    for name, call in CALLS.items():
        for (A, B), probes in zip(call["pairs"], call.get("probes", [])):
            d2m = mo.sqrt_le_max(call["thresh"] if name != "eq_0" and np.isfinite(call["thresh"]) and call["thresh"] > 0 else 0.005)
            want = {"eq": d2m, "above": np.nextafter(d2m, np.float32(np.inf)), "below": np.nextafter(d2m, np.float32(0))}
            for i, kind in probes.items():
                for order in ("kernel", "plain"):
                    assert mo.ransac_d2_exact(eye, A[i], B[i], order) == float(want[kind]), (name, i, kind, order)
                seen += 1
    assert seen == 3 * 7


def test_equality_triples_are_not_collinear():
    """A collinear triple would tie Horn's largest eigenvalue and the fit would no longer be exactly [I | 0]."""
    for name, call in CALLS.items():
        if not name.startswith("eq_"):
            continue
        A, B = call["pairs"][0]
        ids = mo.ransac_sample_ids(U3[:call["n_trials"]], len(A))
        for t in np.nonzero(mo.ransac_expected_good(A, B, ids, len(A)))[0]:
            s = A[ids[t], :3].astype(np.float64)
            ev = np.linalg.eigvalsh((s - s.mean(0)).T @ (s - s.mean(0)))
            assert ev[1] >= 1e-3 * ev[2], (name, t, ev)


def test_layouts():
    pub = CALLS["publication"]
    H = pub["n_trials"] - 1
    L = pub["expect"][0][0]
    n = len(pub["pairs"][0][0])
    ids = mo.ransac_sample_ids(U3[:H + 1], n)
    assert H >= 256 and H % 256 < 32 and L < 256 and len(pub["pairs"]) >= 256
    assert (ids[H] < 1024).all() and (ids[L] >= n - 1024).all()
    ch = CALLS["chunks"]
    ns = sorted(len(A) for A, _ in ch["pairs"])
    assert ns == sorted(rf.CHUNK_NS + [0, 0, 2])
    for (A, B), exp in zip(ch["pairs"], ch["expect"]):
        n = len(A)
        if exp is None or n <= 5:
            continue
        ids = mo.ransac_sample_ids(U3[:ch["n_trials"]], n)
        assert (ids[exp[0]] >= max(0, n - 1024)).all(), (n, exp)


def test_degenerate_fits_within_stated_tolerances():
    """The float32 emulation of k_ransac_model meets the GPU test's tolerances on every degenerate sample, and with 2 Jacobi sweeps
    instead of 8 it misses the pose tolerance on some well-conditioned one (the tolerance can see an unconverged eigenvector)."""
    call = CALLS["degenerate"]
    A, B = call["pairs"][0]
    ids = mo.ransac_sample_ids(U3[:call["n_trials"]], len(A))
    good = mo.ransac_expected_good(A, B, ids, len(A))
    worst, missed = 0.0, []
    for t, cfg in call["trials"].items():
        s, d = A[ids[t], :3], B[ids[t], :3]
        if not good[t]:
            assert "nan" in cfg or "inf" in cfg, cfg
            continue
        R, tt, rss = mo.kabsch64(s, d)
        rss_tol, r_tol, t_tol = rf.fit_tolerances(s, d)
        for sweeps in (8, 2):
            P = mo.ransac_model_f32(s, d, sweeps).astype(np.float64)
            got = ((d - (s @ P[:, :3].T + P[:, 3])) ** 2).sum()
            err = max(np.abs(P[:, :3] - R).max() / r_tol, np.abs(P[:, 3] - tt).max() / t_tol)      # in units of the tolerance
            if sweeps == 8:
                assert np.abs(P[:, :3].T @ P[:, :3] - np.eye(3)).max() <= 1e-5 and np.linalg.det(P[:, :3]) > 0, cfg
                assert got <= rss + rss_tol, (cfg, got, rss, rss_tol)
                if cfg in rf.WELL:
                    assert err <= 1.0, (cfg, err)
                    worst = max(worst, err)
            elif cfg in rf.WELL and err > 1.0:
                missed.append(cfg)
    assert missed, "2 Jacobi sweeps stay within the pose tolerance"
    print(f"worst emulated pose error / tolerance {worst:.3f}; 2 sweeps miss on {missed}")


def test_op_order_family():
    """The operation-order pair: its one cluster's only pure trial wins with OP_K, and probes moved onto the contraction boundary of that
    trial's (Kabsch) pose are all marginal, half of them accepted by the kernel order, a third of them against the uncontracted squares."""
    call, probe_ids = rf.op_order()
    A, B = call["pairs"][0]
    T, th = call["n_trials"], call["thresh"]
    ids = mo.ransac_sample_ids(U3[:T], len(A))
    good = mo.ransac_expected_good(A, B, ids, len(A))
    poses = kabsch_poses(A, B, ids, good)
    counts, marg = mo.counts_from_poses(A, B, poses, good, th)
    assert marg.sum() == 0 and mo.ransac_winner(counts, good) == call["expect"][0]
    W = call["expect"][0][0]
    assert (counts[good] == call["expect"][0][1]).sum() == 1
    assert not set(probe_ids) & set(int(i) for i in ids.ravel())
    probes = rf.op_order_probes(poses[W], probe_ids, th, np.random.default_rng(11))
    A2, B2 = A.copy(), B.copy()
    for i, (a, b, _) in probes.items():
        A2[i, :3], B2[i, :3] = a, b
    dec, st = mo.ransac_classify(poses[W], A2, B2, th)
    assert all(st[i] == mo.MARGINAL and dec[i] == k for i, (_, _, k) in probes.items())
    assert sum(k for _, _, k in probes.values()) == len(probes) // 2
    d2m = float(mo.sqrt_le_max(th))
    squares = [i for j, i in enumerate(probe_ids) if mo.RANSAC_ORDERS[1 + j % 3] == "plain_squares"]
    for i in squares:
        a, b, k = probes[i]
        assert (mo.ransac_d2_exact(poses[W], a, b, "plain_squares") <= d2m) != k


def test_chain_rows():
    """The rows of the fused-chain test survive pruneMatches and collectMutualMatches in order, and cluster 0's trial wins on them."""
    from oracle import corres_families as cf
    for p, (A, B, clusters) in enumerate(rf.chain_frames()):
        cand, _ = mo.find_corres(A, B, cf.K, (4.0, -1.0, 4.0, -1.0), U3[:1], rf.CHAIN_THRESH)
        n = len(B["kpts"])
        assert len(cand) == n
        PA, PB = cand[:, 4:7], cand[:, 7:10]
        ids = mo.ransac_sample_ids(U3[:rf.MAX_TRIALS], n)
        good = mo.ransac_expected_good(PA, PB, ids, n)
        counts, marg = mo.counts_from_poses(PA, PB, kabsch_poses(PA, PB, ids, good), good, rf.CHAIN_THRESH)
        assert marg.sum() == 0
        assert mo.ransac_winner(counts, good) == (clusters[0][0], len(clusters[0][1]))
        if p == 0:          # an exact tie with the other cluster's later trial
            assert (counts == len(clusters[1][1])).sum() > (counts == len(clusters[1][1]))[:clusters[0][0] + 1].sum()
