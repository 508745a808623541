"""findCorres after the kNN (prune.cu) against its float64 restatement on pairs built to sit on its edges (oracle/corres_families.py):
the pruneMatches gates at equality and one ulp off, pixel rounding and depth validity, candidate lists, 512-row chunks, propagated
matches, the five-match rules around RANSAC, the capacity cut and batches of more than 1024 pairs.

Rows and counts must equal the restatement's exactly and in order.  A query takes the first candidate the float64 gate does not reject;
a candidate inside the gate's float32 bound may go either way and is printed.  Cloud points are bit-equal on dyadic families and within
2 float32 ulps otherwise."""
import copy
import ctypes
import os

import numpy as np
import pytest

from bundletrack_b200 import _lib, synth
from oracle import corres_families as cf
from oracle import matcher_oracle as mo

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
U3 = np.load(os.path.join(GOLD, "curand_xorwow_seed0.npy"))
CALLS = {c["name"]: c for c in cf.prune_calls()}
WIDE = (4.0, -1.0, 4.0, -1.0)          # prune thresholds every built row passes: the count rules decide alone


def _dev(fr, dev, window_index=None):
    import torch
    d = {"kpts": torch.from_numpy(fr["kpts"]).to(dev), "depth": torch.from_numpy(fr["depth"]).to(dev),
         "normal": torch.from_numpy(fr["normal"]).to(dev), "pose": fr["pose"], "id": fr["id"],
         "window_index": fr["id"] if window_index is None else window_index}
    if "desc" in fr:
        d["desc"] = torch.from_numpy(fr["desc"]).to(dev)
    return d


@pytest.fixture(scope="module")
def pipe(cuda_device):
    from bundletrack_b200.matcher import MatchPipeline
    mp = MatchPipeline(None, max_pairs=16, max_feats=cf.SIZES_MAX_FEATS)
    yield mp
    mp.close()


# ------------------------------------------------------------------------------------------------ gates, candidate lists, sizes
@pytest.mark.parametrize("name", list(CALLS))
def test_prune_family(pipe, cuda_device, name):
    import torch
    call = CALLS[name]
    cases = call["cases"]
    pairs = [(_dev(A, cuda_device), _dev(B, cuda_device)) for A, B, _, _ in cases]
    iab = torch.from_numpy(np.ascontiguousarray(np.concatenate([c[2] for c in cases]))).to(cuda_device)
    iba = torch.from_numpy(np.ascontiguousarray(np.concatenate([c[3] for c in cases]))).to(cuda_device)
    saved = pipe.prune
    pipe.prune = _lib.PruneParams(*call["prm"])
    try:
        got = pipe.prune_mutual(pairs, iab, iba, cf.H, cf.W, cf.K, k=call["k"])
    finally:
        pipe.prune = saved
    md_o, c_o, md_n, c_n = call["prm"]
    ulps = 0 if call["dyadic"] else 2
    marginals, total = [], 0
    for p, (A, B, idxAB, idxBA) in enumerate(cases):
        nb = abs(A["id"] - B["id"]) == 1
        md, cm = (md_n, c_n) if nb else (md_o, c_o)
        oab, mab = mo.prune_options(A, B, idxAB, cf.K, md, cm)
        oba, mba = mo.prune_options(B, A, idxBA, cf.K, md, cm)
        marginals += [(p, "AB") + m[:2] for m in mab] + [(p, "BA") + m[:2] for m in mba]
        g = got[p].cpu().numpy()
        want, _ = mo.mutual_rows_resolved(A, B, oab, oba, got=g, ulps=ulps)
        assert g.shape == want.shape, (name, p, len(A["kpts"]), len(B["kpts"]), g.shape, want.shape)
        if not mo.rows_match(g, want, ulps):
            bad = np.nonzero([not mo.rows_match(g[i], want[i], ulps) for i in range(len(g))])[0]
            raise AssertionError(f"{name} pair {p}: {len(bad)} rows differ, first at {bad[0]}: got {g[bad[0]]} want {want[bad[0]]}")
        total += len(want)
    print(f"{name}: {total} rows; marginal candidates (pair, direction, query, train): {marginals}")
    assert call["marginal_ok"] or not marginals, marginals


# ------------------------------------------------------------------------------------------------ the fused chain, bt_match_pairs_ex
def _match_ex(mp, pairs, extras, prm, trials, inlier_dist, capacity, dev):
    """One bt_match_pairs_ex call over device frame pairs (descriptor views).  Returns (entries, n_entry, entry_off, total, status, uv)."""
    import torch
    A, B, dA, dB = mp._views(pairs)
    n = len(pairs)
    ex = (_lib.MatchExtra * n)()
    keep = []
    for p, e in enumerate(extras or []):
        if e is not None and len(e):
            arr = np.ascontiguousarray(e, np.float32)
            keep.append(arr)
            ex[p].uv, ex[p].n = arr.ctypes.data, len(arr)
    ent = torch.zeros((max(capacity, 1), 8), dtype=torch.int32, device=dev)
    meta = torch.full((3, n), -7, dtype=torch.int32, device=dev)
    tot = torch.zeros(4, dtype=torch.int32, device=dev)
    uvo = torch.zeros((max(capacity, 1), 4), dtype=torch.float32, device=dev)
    fx, fy, cx, cy = cf.K
    P = _lib.PruneParams(*prm)
    _lib.check(mp.lib.bt_match_pairs_ex(mp.ctx, ctypes.c_int(n), A, B, dA, dB, None, None, ctypes.c_int(cf.H), ctypes.c_int(cf.W), ctypes.c_float(fx),
                                        ctypes.c_float(fy), ctypes.c_float(cx), ctypes.c_float(cy), ctypes.byref(P), ctypes.c_int(trials),
                                        ctypes.c_float(inlier_dist), ctypes.c_uint64(0), ex, ctypes.c_void_p(ent.data_ptr()), ctypes.c_int(capacity),
                                        ctypes.c_void_p(meta[0].data_ptr()), ctypes.c_void_p(meta[1].data_ptr()), ctypes.c_void_p(tot.data_ptr()),
                                        ctypes.c_void_p(meta[2].data_ptr()), ctypes.c_void_p(uvo.data_ptr()), mp.stream), "bt_match_pairs_ex")
    m = meta.cpu().numpy()
    e = ent.cpu().numpy().view(np.uint8).reshape(-1).view(synth.ENTRYJ_DTYPE)
    return e, m[0], m[1], int(tot[0].item()), m[2], uvo.cpu().numpy()


def _on_device(frames, dev):
    return [(_dev(A, dev), _dev(B, dev)) for A, B in frames]


def _restate(frames, extras, prm, trials, inlier_dist):
    """Per pair: the emitted rows find_corres gives (rows[inlier ids], empty when the pair is cleared)."""
    out = []
    for (A, B), e in zip(frames, extras):
        rows, ids = mo.find_corres(A, B, cf.K, prm, U3[:trials], inlier_dist, propagated=e)
        out.append(np.zeros((0, 10), np.float32) if ids is None else rows[ids])
    return out


def _check_emitted(got, frames, want_rows, capacity, ulps=0):
    """Counts, offsets, total, statuses, entries and uv_out against emit_plan over the restated rows."""
    ent, n_entry, off, total, status, uv = got
    nb = [abs(A["id"] - B["id"]) == 1 for A, B in frames]
    w_n, w_off, w_total, w_status = mo.emit_plan([len(r) for r in want_rows], nb, capacity)
    assert np.array_equal(n_entry, w_n), (n_entry.tolist(), w_n.tolist())
    assert np.array_equal(off, w_off), (off.tolist(), w_off.tolist())
    assert total == w_total and np.array_equal(status, w_status), (total, w_total, status.tolist(), w_status.tolist())
    assert ((off >= 0) & (off + n_entry <= capacity)).all()
    full = np.concatenate(want_rows + [np.zeros((0, 10), np.float32)], 0)[:total]
    assert np.array_equal(uv[:total].view(np.uint32), full[:, :4].view(np.uint32))
    got_rows = np.concatenate([uv[:total], ent[:total]["pos_j"], ent[:total]["pos_i"]], 1)
    assert mo.rows_match(got_rows, full, ulps)
    wi = np.concatenate([np.full(n, fr[1]["id"], np.uint32) for n, fr in zip(w_n, frames)] + [np.zeros(0, np.uint32)])
    wj = np.concatenate([np.full(n, fr[0]["id"], np.uint32) for n, fr in zip(w_n, frames)] + [np.zeros(0, np.uint32)])
    assert np.array_equal(ent[:total]["imgIdx_i"], wi) and np.array_equal(ent[:total]["imgIdx_j"], wj)


def test_propagated_matches(pipe, cuda_device):
    """findCorresByMapPoints through bt_match_pairs_ex's host extras, in order, against find_corres(propagated=...): duplicates on
    (uA, vA), on (uB, vB), on both and on neither, -0.0 against +0.0, extras outside the image and on invalid depth, more than 256 of
    them; a pair whose extras meet no mutual match; a neighbour pair, whose extras are ignored.  An infinite RANSAC threshold keeps
    every candidate, so the emitted list is the candidate list."""
    rng = np.random.default_rng(41)
    rows, ex = cf.propagated_case(rng)
    A0, B0 = cf.desc_pair(rng, rows, 6, 2)
    px = cf.free_pixels(rng, 8)
    dead = [("sym", (u, v, 0.0), (u, v, 0.75)) for u, v in px[:4]]
    A1, B1 = cf.desc_pair(rng, dead, 7, 2)
    B1["depth"][px[5][1], px[5][0]] = 0.5
    A1["depth"][px[4][1], px[4][0]] = 0.625
    ex1 = np.asarray([(px[4][0], px[4][1], px[5][0], px[5][1])] * 3 + [(u, v, u, v) for u, v in px[:4]] + [(1.0, 1.0, 2.0, 2.0)], np.float32)
    A2, B2 = cf.desc_pair(rng, rows, 3, 2)
    frames, extras = [(A0, B0), (A1, B1), (A2, B2)], [ex, ex1, ex[:20]]
    want = _restate(frames, extras, WIDE, 200, float("inf"))
    assert 256 < len(want[0]) - 16 <= len(ex) - 4 and len(want[1]) == len(ex1) and len(want[2]) == 16, [len(w) for w in want]
    cap = sum(len(A["kpts"]) + len(B["kpts"]) for A, B in frames) + len(ex) + len(ex1)
    got = _match_ex(pipe, _on_device(frames, cuda_device), extras, WIDE, 200, float("inf"), cap, cuda_device)
    _check_emitted(got, frames, want, cap)


def _count_rule_frames(rng):
    frames, names = [], []
    for rule in cf.COUNT_RULES:
        for ida, idb in ((9, 8), (9, 6)):
            frames.append(cf.desc_pair(rng, cf.count_rule_rows(rng, rule), ida, idb))
            names.append((rule, ida - idb == 1))
    return frames, names


def test_count_rules(pipe, cuda_device):
    """Exactly 5 and 6 candidates before RANSAC (<= 5 clears the pair), exactly 4 and 5 inliers after it (< 5 clears), on neighbour and
    non-neighbour pairs: n_entry and OK / EMPTY / FAIL as the reference's rules give them."""
    rng = np.random.default_rng(42)
    frames, names = _count_rule_frames(rng)
    want = _restate(frames, [None] * len(frames), WIDE, 500, 0.01)
    expect = {"c5": 0, "c6": 6, "i4": 0, "i5": 5, "i5o1": 5}
    assert [len(w) for w in want] == [expect[r] for r, _ in names], [len(w) for w in want]
    cap = sum(len(A["kpts"]) + len(B["kpts"]) for A, B in frames)
    got = _match_ex(pipe, _on_device(frames, cuda_device), None, WIDE, 500, 0.01, cap, cuda_device)
    _check_emitted(got, frames, want, cap)


@pytest.mark.parametrize("cut", ["uncut", "zero", "mid_pair", "total", "total_minus_one", "pair_boundary"])
def test_capacity_cut(pipe, cuda_device, cut):
    """entry_capacity 0, inside a pair, exactly the total, one below it and on a pair boundary: (entry_off, n_entry) stay inside the
    buffer, *total = min(sum, capacity), the entries are the uncut list's prefix, uv_out follows them, and every pair keeps the status of
    its match outcome.  One pair has 300 entries (more than k_emit_fill's 256 threads)."""
    rng = np.random.default_rng(43)
    frames = [cf.desc_pair(rng, rows, 5 + p, 4 + (p % 2)) for p, rows in enumerate(cf.emission_templates(rng))]
    want = _restate(frames, [None] * len(frames), WIDE, 500, 0.01)
    sizes = [len(w) for w in want]
    assert sizes == [6, 0, 300, 5, 0, 12], sizes
    total = sum(sizes)
    cap = {"uncut": sum(len(A["kpts"]) + len(B["kpts"]) for A, B in frames), "zero": 0, "mid_pair": 6 + 123, "total": total,
           "total_minus_one": total - 1, "pair_boundary": 6 + 300}[cut]
    got = _match_ex(pipe, _on_device(frames, cuda_device), None, WIDE, 500, 0.01, cap, cuda_device)
    _check_emitted(got, frames, want, cap)


def test_more_than_1024_pairs(cuda_device):
    """One bt_match_pairs_ex call over 2100 small pairs (k_emit_entryj scans 1024 pairs at a time and carries the sum across): counts,
    offsets and statuses equal a host prefix sum over the restated pairs, with non-empty and cleared pairs on both sides of pair 1024
    and pair 2048."""
    from bundletrack_b200.matcher import MatchPipeline
    n_pairs, trials = 2100, 64
    rng = np.random.default_rng(44)
    templates = [cf.desc_pair(rng, rows, 20, 10) for rows in cf.many_pair_templates(rng)]
    per_t = _restate(templates, [None] * len(templates), WIDE, trials, 0.01)
    assert [len(w) for w in per_t] == [0, 0, 6, 0, 16, 5, 10], [len(w) for w in per_t]
    from bundletrack_b200.config import load_yml
    yml = copy.deepcopy(load_yml(None))
    yml["ransac"]["max_iter"] = trials          # the per-pair RANSAC model buffer stays small
    mp = MatchPipeline(yml, max_pairs=n_pairs, max_feats=48)
    try:
        pick = [(p * 5 + p // 7) % len(templates) for p in range(n_pairs)]
        neighbour = [p % 3 == 0 for p in range(n_pairs)]
        frames, want = [], []
        for p in range(n_pairs):
            A, B = templates[pick[p]]
            A = dict(A, id=11 if neighbour[p] else 12)
            frames.append((A, B))
            want.append(per_t[pick[p]])
        for lo, hi in ((1000, 1024), (1024, 1048), (2024, 2048), (2048, 2072)):
            assert any(len(want[p]) for p in range(lo, hi)) and not all(len(want[p]) for p in range(lo, hi))
        # each template's frames go to the device once, so the call names few descriptor sets
        dev_t = _on_device(templates, cuda_device)
        pairs = [(dict(dev_t[t][0], id=A["id"], window_index=A["id"]), dev_t[t][1]) for (A, _), t in zip(frames, pick)]
        cap = sum(len(A["kpts"]) + len(B["kpts"]) for A, B in frames)
        got = _match_ex(mp, pairs, None, WIDE, trials, 0.01, cap, cuda_device)
        _check_emitted(got, frames, want, cap)
    finally:
        mp.close()

