"""The kNN matcher (knn.cu) against exact brute force on descriptors built to stress the bound of k_knn_select: exact ties, near-ties
far below the resolution of the stored fp16 keys, clusters placed against the 4-row group and 128 / 256-row tile layout, scale
extremes (fp16 clamp and flush, large common offsets), every tile edge and k = 1..8.

Comparison rule, both directions of every pair: indices equal the reference exactly (padding -1 / inf), distances within one float32
ulp of float32(sqrt(d2)) with d2 the float64 direct-difference sum; bit-equal on dyadic data, where every d2 is exact in float64.
The reference is oracle/matcher_oracle.py::knn, itself checked against a plain brute force (tests/test_oracle_matcher.py).

Each case also reads the call's fallback row count (bt_knn_get_timing): families built to stay within the selection's 16 groups /
16 candidates must not reach k_knn_exact (else the soundness checks would only have tested the brute force), the overflowing ones
must send their constructed query to it."""
import numpy as np
import pytest

from bundletrack_b200 import synth
from oracle import matcher_oracle as mo
from oracle.knn_families import (D, FAST, N_SET, OVERFLOW, PLACEMENTS, Q_ROW, cluster_case, flush_case, grid_rows, group_rows, knn_unpos,
                                 offset_ladder_case, offset_set)

MAX_FEATS = 5120
FALLBACKS = {}      # family -> fallback rows per call, printed at the end of the module


def test_knn_unpos_is_a_permutation_of_each_block():
    for blk in range(3):
        rows = [knn_unpos(128 * blk + p) for p in range(128)]
        assert sorted(rows) == list(range(128 * blk, 128 * blk + 128))
    # a group's rows are {r, r + 8, r + 64, r + 72}: rows one thread of the tensor pass holds
    for g in range(32):
        r = group_rows(g)
        assert r == [r[0], r[0] + 8, r[0] + 64, r[0] + 72]


def f32(x):
    return np.ascontiguousarray(x, np.float32)


# ------------------------------------------------------------------------------------------------------------ comparison
def _ulps(got, want):
    return np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))


def check_direction(q, t, idx, dist, k, dyadic, what):
    want_i, want_d = mo.knn(q, t, k)
    got_i, got_d = idx.cpu().numpy(), dist.cpu().numpy()
    assert got_i.shape == want_i.shape, what
    bad = np.nonzero((got_i != want_i).any(1))[0]
    assert len(bad) == 0, (what, bad[:5], got_i[bad[:3]], want_i[bad[:3]])
    fin = want_i >= 0
    assert np.isinf(got_d[~fin]).all() and (got_d[~fin] > 0).all(), what
    if dyadic:
        assert np.array_equal(got_d[fin].view(np.int32), want_d[fin].view(np.int32)), what
    elif fin.any():
        assert _ulps(got_d[fin], want_d[fin]).max() <= 1, (what, _ulps(got_d[fin], want_d[fin]).max())


def to_dev(x, dev):
    import torch
    return torch.from_numpy(f32(x)).to(dev) if len(x) else torch.zeros((0, D), device=dev)


def run_and_check(matcher, dev, pairs, k, dyadic=False, family=None):
    """One bt_knn_match_pairs call on the float64 pairs (exact in float32); every pair both ways against the reference.  Returns the
    call's fallback row count and the outputs."""
    ts = [(to_dev(a, dev), to_dev(b, dev)) for a, b in pairs]
    out = matcher.knn_match_pairs(ts, k=k)
    fb = matcher.timing()["fallback_rows"]
    for p, (a, b) in enumerate(pairs):
        check_direction(f32(a), f32(b), out[0][p], out[1][p], k, dyadic, f"pair {p} A->B")
        check_direction(f32(b), f32(a), out[2][p], out[3][p], k, dyadic, f"pair {p} B->A")
    if family is not None:
        FALLBACKS.setdefault(family, []).append(fb)
    return fb, out


@pytest.fixture(scope="module")
def matcher(cuda_device):
    from bundletrack_b200.matcher import KnnMatcher
    m = KnnMatcher(max_pairs=64, max_feats=MAX_FEATS)
    m.enable_timing(True)
    yield m
    m.close()
    for fam in sorted(FALLBACKS):
        v = FALLBACKS[fam]
        print(f"fallback rows per call  {fam:28s} calls {len(v):4d}  min {min(v):5d}  max {max(v):5d}")


KS = list(range(1, 9))


# ------------------------------------------------------------------------------------------------------------ 1-3: ties and placement
@pytest.mark.gpu
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("side", ["B", "A"])
@pytest.mark.parametrize("placement", sorted(PLACEMENTS))
@pytest.mark.parametrize("family", ["tie", "near"])
def test_cluster_placement(matcher, cuda_device, family, placement, side, k):
    """A cluster of exact ties or sub-fp16 near-ties around one query, placed against the group / tile layout, in B (clusters of
    train rows) or in A (the same rows clustered on the query side of the B->A matrix)."""
    qs, ts = cluster_case(family, PLACEMENTS[placement], seed=100 * sorted(PLACEMENTS).index(placement) + 10 * k + (family == "near"))
    pair = (qs, ts) if side == "B" else (ts, qs)
    run_and_check(matcher, cuda_device, [pair], k, dyadic=True, family=f"{family}/{placement}, {N_SET}-row sets")
    # The constructed query alone on its side: the 4-row group minimum over the query's group is then its own key, so the fallback count
    # is the query's alone (among 1024 background rows, k = 4..8, a few dozen background queries overflow on group mates' keys).
    q1 = qs[Q_ROW:Q_ROW + 1]
    fb, _ = run_and_check(matcher, cuda_device, [(q1, ts) if side == "B" else (ts, q1)], k, dyadic=True, family=f"{family}/{placement}, query alone")
    if family == "near" and placement in FAST:
        assert fb == 0, (family, placement, side, k, fb)
    if placement in OVERFLOW:
        assert fb >= 1, (family, placement, side, k, fb)      # every member is inside the threshold: the query cannot stay on the fast path


@pytest.mark.gpu
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("side", ["B", "A"])
@pytest.mark.parametrize("extra", ["k-1", "k", "k+1", "15", "16", "17", "64", "65"])
def test_exact_tie_counts(matcher, cuda_device, extra, side, k):
    """m train rows at exactly the same distance from one query, m = k - 1 .. 65, contiguous and centred on the 127 / 128 row edge: the
    lowest indices win."""
    m = {"k-1": k - 1, "k": k, "k+1": k + 1}[extra] if extra.startswith("k") else int(extra)
    qs, ts = cluster_case("tie", list(range(128 - m // 2, 128 - m // 2 + m)), seed=1000 + 10 * m + k)
    pair = (qs, ts) if side == "B" else (ts, qs)
    run_and_check(matcher, cuda_device, [pair], k, dyadic=True, family=f"tie/m={extra}, {N_SET}-row sets")
    q1 = qs[Q_ROW:Q_ROW + 1]
    fb, _ = run_and_check(matcher, cuda_device, [(q1, ts) if side == "B" else (ts, q1)], k, dyadic=True, family=f"tie/m={extra}, query alone")
    if m >= 17:
        assert fb >= 1, (m, side, k, fb)


# ------------------------------------------------------------------------------------------------------------ terms of the bound
@pytest.mark.gpu
@pytest.mark.parametrize("side", ["B", "A"])
@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_rounding_error_decides_the_nearest_row(matcher, cuda_device, sign, side):
    """fp16 flushing moves the true nearest row away from the query and the decoy onto it (flush_case): only the full 2 e of the bound
    (the query's and the train row's rounding error, once in T and once in R) keeps the true row among the candidates."""
    q, t, want = flush_case(sign)
    pair = (q, t) if side == "B" else (t, q)
    _, out = run_and_check(matcher, cuda_device, [pair], 1, family="flush decides")
    got = (out[0] if side == "B" else out[2])[0].cpu().numpy()
    assert got[0, 0] == want


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 5, 8])
@pytest.mark.parametrize("side", ["B", "A"])
def test_fp16_exact_rows_on_common_offset(matcher, cuda_device, side, k):
    """fp16-exact rows (e = 0) on a common offset: the fp32 accumulation error of the tensor pass is the bound's only real term."""
    qs, ts = offset_ladder_case(200 + k)
    run_and_check(matcher, cuda_device, [(qs, ts) if side == "B" else (ts, qs)], k, dyadic=True, family="offset ladder")


# ------------------------------------------------------------------------------------------------------------ 4: scales
def scale_pairs(seed):
    """(name, A, B, fast): sets of very different scale side by side in one call.  'xS' sets have N(0, S^2) components."""
    rng = np.random.default_rng(seed)
    g = lambda n, s: rng.normal(0.0, s, (n, D))
    # about 5 % of the components of an 'x1e-3' set lie below fp16's normal range (6.1e-5) and flush: the measured error then widens the bound so
    # far that queries at k = 8 overflow.  The fast-path set keeps every component at 1e-4 or more; flushing has its own sets below.
    unflushed = lambda x: np.sign(x) * np.maximum(np.abs(x), 1e-4)
    c = rng.normal(size=D)
    unit_a, unit_b, _, _ = synth.make_descriptors(seed, N_SET, N_SET + 76)
    mixed = g(240, 1.0)
    mixed[::7] *= 1e5            # clamped rows: emax is large while the unit rows set m2
    mixed[3::7] *= 1e-6          # flushed rows
    out = [("unit-norm", unit_a, unit_b, True),      # (fast-path sets at N_SET rows, see cluster_case)
           ("x1e-3", unflushed(g(N_SET, 1e-3)), unflushed(g(N_SET + 50, 1e-3)), True),
           ("x1", g(N_SET, 1.0), g(N_SET + 50, 1.0), True),
           ("x1e3", g(N_SET, 1e3), g(N_SET + 50, 1e3), True),
           ("clamped ~1e5", g(120, 1e5), g(140, 1e5), False),
           ("flushed ~1e-6 (m2 = 0)", g(120, 1e-6), g(130, 1e-6), False),      # every row flushes: s = 1
           ("flushed vs unit", g(90, 1e-6), g(110, 1.0), False),
           ("mixed clamped/flushed/unit", mixed, g(200, 1.0), False)]
    for C in (10.0, 100.0, 1000.0):
        for sigma in (1e-3, 1e-1):
            out.append((f"offset C={C:g} sigma={sigma:g}", offset_set(rng, 130, C, sigma, c), offset_set(rng, 150, C, sigma, c), False))
    return [(n, f32(a).astype(np.float64), f32(b).astype(np.float64), fast) for n, a, b, fast in out]


# The scale exponent of k_knn_pairconst is clamped to +-100, which no input reaches: the fp16 conversion clamps at 65504 and flushes
# below 2^-14, so a set's largest rounded norm m2 is 0 (s = 1) or within [2^-28, 256 * 65504^2 < 2^41].
@pytest.mark.gpu
@pytest.mark.parametrize("k", KS)
def test_scale_extremes_mixed_in_one_call(matcher, cuda_device, k):
    sp = scale_pairs(50 + k)
    run_and_check(matcher, cuda_device, [(a, b) for _, a, b, _ in sp], k, family="scales mixed call")
    # fast-path proof on 8 query rows per set: rows 0..7 lie in eight different groups whose other rows are padding, so each group
    # minimum on the query side is the row's own key (with all 1024 rows, some queries overflow on their group mates' keys)
    fast = [(a[:8], b) for _, a, b, f in sp if f] + [(b[:8], a) for _, a, b, f in sp if f]
    fb, _ = run_and_check(matcher, cuda_device, fast, k, family="scales x1e-3..x1e3, 8 queries")
    assert fb == 0, (k, fb)


# ------------------------------------------------------------------------------------------------------------ 5: shapes
SIZES = [0, 1, 3, 4, 5, 127, 128, 129, 255, 256, 257, 383, 384, 385]
SHAPE_PAIRS = [(SIZES[i], SIZES[(5 * i + 3) % len(SIZES)]) for i in range(len(SIZES))]     # every size on both sides


def shape_pairs(seed):
    out = []
    for na, nb in SHAPE_PAIRS:
        a, b, _, _ = synth.make_descriptors(seed + na * 7 + nb, max(na, 1), max(nb, 1))
        out.append((a[:na].astype(np.float64), b[:nb].astype(np.float64)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("k", KS)
def test_tile_edge_shapes(matcher, cuda_device, k):
    run_and_check(matcher, cuda_device, shape_pairs(k), k, family="shapes")


@pytest.mark.gpu
def test_max_feats_both_sides(matcher, cuda_device):
    a, b, _, _ = synth.make_descriptors(77, MAX_FEATS, MAX_FEATS)
    run_and_check(matcher, cuda_device, [(a.astype(np.float64), b.astype(np.float64))], 8, family="max_feats")


@pytest.mark.gpu
def test_k8_fewer_train_rows_than_k(matcher, cuda_device):
    pairs = []
    for nt in range(1, 8):
        a, b, _, _ = synth.make_descriptors(90 + nt, 50, nt)
        pairs += [(a.astype(np.float64), b.astype(np.float64)), (b.astype(np.float64), a.astype(np.float64))]
    run_and_check(matcher, cuda_device, pairs, 8, family="k=8, nt < 8")


@pytest.mark.gpu
def test_64_pairs_mixed_sizes_and_empty_sets(matcher, cuda_device):
    """The fixture's max_pairs in one call, empty sets among them and more tensor-pass units than SMs."""
    rng = np.random.default_rng(64)
    sizes = rng.integers(0, 700, size=(64, 2))
    sizes[::9, 0] = 0
    sizes[4::11, 1] = 0
    pairs = []
    for p, (na, nb) in enumerate(sizes):
        a, b, _, _ = synth.make_descriptors(400 + p, max(na, 1), max(nb, 1))
        pairs.append((a[:na].astype(np.float64), b[:nb].astype(np.float64)))
    import torch
    run_and_check(matcher, cuda_device, pairs, 5, family="64 pairs")
    assert matcher.timing()["units"] > torch.cuda.get_device_properties(cuda_device).multi_processor_count


# ------------------------------------------------------------------------------------------------------------ 6: exact fallback
@pytest.mark.gpu
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("na,nb", [(100, 120), (300, 400)])      # <= 256 fallback rows: split over segments; more: one CTA per row
def test_forced_fallback_every_k(matcher, cuda_device, na, nb, k):
    rng = np.random.default_rng(na + k)
    a, b = grid_rows(rng, na), grid_rows(rng, nb)
    b[5] = b[6] = b[110] = a[3]                                  # ties across the fallback's segments
    _, fast = run_and_check(matcher, cuda_device, [(a, b)], k, dyadic=True)
    matcher.force_fallback(1)
    try:
        fb, slow = run_and_check(matcher, cuda_device, [(a, b)], k, dyadic=True)
    finally:
        matcher.force_fallback(0)
    assert fb == na + nb
    assert _bits(fast) == _bits(slow)


# ------------------------------------------------------------------------------------------------------------ 7: equivalences
def _bits(out):
    return [t.cpu().numpy().tobytes() for four in out for t in four]


@pytest.mark.gpu
def test_batch_equals_single_calls_and_repeats(matcher, cuda_device):
    pairs = shape_pairs(3) + [(a, b) for _, a, b, _ in scale_pairs(4)]
    ts = [(to_dev(a, cuda_device), to_dev(b, cuda_device)) for a, b in pairs]
    batch = matcher.knn_match_pairs(ts, k=7)
    again = matcher.knn_match_pairs(ts, k=7)
    assert _bits(batch) == _bits(again)
    for p, tp in enumerate(ts):
        one = matcher.knn_match_pairs([tp], k=7)
        assert _bits([[x[p]] for x in batch]) == _bits([[x[0]] for x in one]), p


@pytest.mark.gpu
def test_slots_equal_pairs_on_near_ties_and_scales(matcher, cuda_device):
    sets = []
    for placement in ("spread12", "g17", "edge255"):
        sets += list(cluster_case("near", PLACEMENTS[placement], seed=5))
    for _, a, b, _ in scale_pairs(6):
        sets += [a, b]
    dev = [to_dev(s, cuda_device) for s in sets]
    matcher.pool_reserve(len(sets))
    for i, d in enumerate(dev):
        matcher.pool_store(i, d)
    idx = [(i, i + 1) for i in range(0, len(sets), 2)]
    sizes = [(len(sets[a]), len(sets[b])) for a, b in idx]
    for k in (1, 5, 8):
        want = matcher.knn_match_pairs([(dev[a], dev[b]) for a, b in idx], k=k)
        got = matcher.knn_match_slots(idx, sizes, k=k, device=cuda_device)
        assert _bits(want) == _bits(got), k


@pytest.mark.gpu
def test_slot_overwritten_with_smaller_then_larger_norms(matcher, cuda_device):
    """A slot's per-set maxima (m2, emax) follow what the slot holds now, not what it held before."""
    import torch
    rng = np.random.default_rng(11)
    base = rng.normal(size=(300, D))
    other = f32(rng.normal(size=(260, D)))
    matcher.pool_reserve(2)
    matcher.pool_store(1, torch.from_numpy(other).to(cuda_device))
    for scale in (1.0, 1e-3, 1e3):
        s = f32(base * scale)
        o = f32(other * scale)
        matcher.pool_store(0, torch.from_numpy(s).to(cuda_device))
        matcher.pool_store(1, torch.from_numpy(o).to(cuda_device))
        iAB, dAB, iBA, dBA = matcher.knn_match_slots([(0, 1)], [(len(s), len(o))], k=6, device=cuda_device)
        check_direction(s, o, iAB[0], dAB[0], 6, False, f"scale {scale} A->B")
        check_direction(o, s, iBA[0], dBA[0], 6, False, f"scale {scale} B->A")
        if scale != 1.0:      # slot 1 keeps the unit set while slot 0 moves: the pair's constants mix both slots' maxima
            matcher.pool_store(1, torch.from_numpy(other).to(cuda_device))
            iAB, dAB, iBA, dBA = matcher.knn_match_slots([(0, 1)], [(len(s), len(other))], k=6, device=cuda_device)
            check_direction(s, other, iAB[0], dAB[0], 6, False, f"scale {scale} vs unit A->B")
            check_direction(other, s, iBA[0], dBA[0], 6, False, f"scale {scale} vs unit B->A")
