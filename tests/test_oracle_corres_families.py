"""The findCorres families (oracle/corres_families.py) land where they claim, and the float64 gate and emission rules of matcher_oracle
decide them as the reference's rules do: equalities are equal in float32, one-ulp cases are one ulp off, exact families have no
marginal candidate.  No GPU needed."""
import os

import numpy as np
import pytest

from oracle import corres_families as cf
from oracle import matcher_oracle as mo

F32 = np.float32


def _outcomes(call):
    """Per case: (rows, marginals) of prune_options over both directions."""
    md_o, c_o, md_n, c_n = call["prm"]
    out = []
    for A, B, iab, iba in call["cases"]:
        nb = abs(A["id"] - B["id"]) == 1
        md, cm = (md_n, c_n) if nb else (md_o, c_o)
        oab, mab = mo.prune_options(A, B, iab, cf.K, md, cm)
        oba, mba = mo.prune_options(B, A, iba, cf.K, md, cm)
        rows, _ = mo.mutual_rows_resolved(A, B, oab, oba)
        out.append((rows, mab + mba, oab, oba))
    return out


@pytest.mark.parametrize("call", [c for c in cf.prune_calls() if c["name"] != "sizes"], ids=lambda c: c["name"])
def test_no_marginal_outside_the_near_family(call):
    for rows, marg, _, _ in _outcomes(call):
        assert call["marginal_ok"] == bool(marg), (call["name"], marg)


def test_sizes_family_chunks_and_no_marginal():
    (call,) = cf.sizes()
    res = _outcomes(call)
    assert not any(m for _, m, _, _ in res)
    sizes = {(len(A["kpts"]), len(B["kpts"])) for A, B, _, _ in call["cases"]}
    for s in (0, 1, 511, 512, 513, 1024, 1025, cf.SIZES_MAX_FEATS):
        assert any(s in pair for pair in sizes), s
    # survivors past the first 512-row chunk in one direction, and a pair whose B->A lists are empty but A->B survives
    assert any(sum(o[-1][0] is not None for o in oab) > 512 for _, _, oab, _ in res)
    A, B, iab, iba = call["cases"][-1]
    assert (iba == -1).all() and len(res[-1][0]) > 0


def test_rounding_is_half_away_from_zero_and_in_image():
    assert F32(cf._below(2.5)) == np.nextafter(F32(2.5), F32(0)) and F32(cf._above(-0.5)) == F32(-0.49999997)
    assert [mo._round_half_away(x) for x in (2.5, 3.5, cf._below(2.5), -0.5, cf._above(-0.5), cf.W - 0.5)] == [3, 4, 2, -1, 0, cf.W]
    (call,) = cf.rounding()
    res = _outcomes(call)
    n = len(cf.ROUND_X) + len(cf.ROUND_Y)
    inside = [0 <= mo._round_half_away(x) < cf.W for x in cf.ROUND_X] + [0 <= mo._round_half_away(y) < cf.H for y in cf.ROUND_Y]
    for rows, _, oab, _ in res:
        assert [o[-1][0] is not None for o in oab] == inside
        assert len(rows) == 2 * sum(inside) and n == len(oab)


def test_depth_validity_keeps_only_0_1():
    (call,) = cf.depth_validity()
    res = _outcomes(call)
    kept = [len(rows) > 0 for rows, _, _, _ in res]
    assert kept == [d == F32(0.1) for d in cf.DEPTHS for _ in (0, 1)]
    assert mo._cloud_point(np.full((1, 1), np.nan, F32), cf.K, 0, 0).tolist() == [0.0, 0.0, 0.0]


def test_distance_family_is_exact_at_and_one_ulp_off_the_threshold():
    calls = {c["name"]: c for c in cf.distance()}
    A, B, _, _ = calls["dist_eq"]["cases"][0]
    v, p, q, d = mo.prune_gate64(A, B, 0, 0, cf.K, 5 * cf.C_NEIGHBOR, -1.0)
    assert v == mo.GATE_PASS and d["exact"] and d["dist"] == 5 * cf.C_NEIGHBOR
    assert F32(calls["dist_below"]["prm"][2]) == np.nextafter(F32(5 * cf.C_NEIGHBOR), F32(0))
    assert F32(calls["dist_above"]["prm"][0]) == np.nextafter(F32(5 * cf.C_OTHER), F32(1))
    for name, c in calls.items():
        for (A, B, _, _), (rows, marg, _, _) in zip(c["cases"], _outcomes(c)):
            nb = abs(A["id"] - B["id"]) == 1
            dist = 5 * (cf.C_NEIGHBOR if B["pose"][0, 3] == 3 * cf.C_NEIGHBOR else cf.C_OTHER)
            thr = c["prm"][2] if nb else c["prm"][0]
            assert not marg and (len(rows) == 2) == (dist <= thr), (name, A["id"], B["id"], dist, thr)


def test_normal_family_exact_dots():
    assert cf.COS_90 > 0 and cf.COS_90 == F32(6.123234e-17)
    for c in cf.normal_gate() + cf.zero_normal():
        for (A, B, _, _), (rows, marg, oab, _) in zip(c["cases"], _outcomes(c)):
            assert not marg
            for q in range(len(A["kpts"])):
                _, _, _, d = mo.prune_gate64(A, B, q, q, cf.K, 64.0, -1.0)
                assert d["zero_normal"] or d["dot"] in (-1.0, 0.0, 1.0)
    c = cf.zero_normal()[0]
    assert all(len(rows) == 6 for rows, _, _, _ in _outcomes(c))       # kept under ZERO_NORMAL_KEEPS, even at cos_max = 1


def test_candidate_lists_cover_skips_first_wins_and_all_fail():
    for c in cf.candidates():
        k = c["k"]
        seen = dict(skip_neg=0, skip_big=0, all_fail=0, first_not_closest=0)
        md_o, _, md_n, _ = c["prm"]
        for (A, B, iab, _), (_, marg, oab, _) in zip(c["cases"], _outcomes(c)):
            md = md_n if abs(A["id"] - B["id"]) == 1 else md_o
            assert not marg
            seen["skip_neg"] += int((iab == -1).sum())
            seen["skip_big"] += int((iab >= len(B["kpts"])).sum())
            for q, o in enumerate(oab):
                if o[-1][0] is None:
                    seen["all_fail"] += 1
                    continue
                passing = [(mo.prune_gate64(A, B, q, int(t), cf.K, md, -1.0)[3].get("dist", np.inf), i) for i, t in enumerate(iab[q])
                           if 0 <= t < len(B["kpts"]) and mo.prune_gate64(A, B, q, int(t), cf.K, md, -1.0)[0] == mo.GATE_PASS]
                if len(passing) > 1 and min(passing)[1] != passing[0][1]:
                    seen["first_not_closest"] += 1
        assert seen["skip_neg"] and seen["skip_big"] and seen["all_fail"], (k, seen)
        assert k == 1 or seen["first_not_closest"], (k, seen)


def test_descriptor_pairs_end_on_the_count_rules():
    """The one-way rows give one candidate each, the sym rows two; consistent rows are RANSAC inliers and outliers are not, so find_corres
    ends exactly on the five-match rules."""
    u3 = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "curand_xorwow_seed0.npy"))[:500]
    rng = np.random.default_rng(3)
    want = {"c5": (5, 0), "c6": (6, 6), "i4": (6, 0), "i5": (7, 5), "i5o1": (6, 5)}
    for rule, (n_cand, n_out) in want.items():
        A, B = cf.desc_pair(rng, cf.count_rule_rows(rng, rule), 9, 6)
        rows, ids = mo.find_corres(A, B, cf.K, (4.0, -1.0, 4.0, -1.0), u3, 0.01)
        assert len(rows) == n_cand and (0 if ids is None else len(ids)) == n_out, rule


def test_emit_plan_cuts_and_keeps_the_status():
    n, off, total, st = mo.emit_plan([6, 3, 300, 5], [True, True, False, False], 100)
    assert n.tolist() == [6, 0, 94, 0] and off.tolist() == [0, 6, 6, 100] and total == 100 and st.tolist() == [0, 2, 0, 0]
    n, off, total, st = mo.emit_plan([6, 0], [True, False], 0)
    assert n.tolist() == [0, 0] and off.tolist() == [0, 0] and total == 0 and st.tolist() == [0, 1]


def test_ulp_distance_and_row_match():
    a = np.zeros((1, 10), F32)
    b = a.copy()
    b[0, 5] = np.nextafter(F32(0), F32(1))
    assert mo.rows_match(a, b, 1) and not mo.rows_match(a, b, 0)
    b = a.copy()
    b[0, 0] = -0.0
    assert not mo.rows_match(a, b, 2)                      # uv are compared bit for bit
    assert mo.ulp_distance(np.array([1.0], F32), np.array([np.nextafter(F32(1), F32(2))], F32))[0] == 1
