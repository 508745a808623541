"""Frame pairs built against findCorres after the kNN (prune.cu): candidates on the gates of pruneMatches, on the 512-row chunks of
k_prune_mutual, propagated matches against the mutual ones, and pairs that end exactly on the five-match rules.  Shared by the oracle's
CPU tests and the GPU tests of prune.cu.

Geometry is dyadic wherever a decision has to be exact: fx = fy = 512, (cx, cy) = (32, 24), identity or signed-permutation rotations,
translations and depths that are multiples of a power of two.  Every float32 operation of the gate is then exact (the float64 gate,
matcher_oracle.prune_gate64, checks that step by step), Pythagorean offsets put the distance exactly on its threshold and axis-aligned
normals give dot products of exactly -1, 0 or 1.

A prune call is a dict: name, cases [(A, B, idxAB [nA, k], idxBA [nB, k])], prm (max_dist_no_neighbor, cos_no_neighbor,
max_dist_neighbor, cos_neighbor), k, dyadic (cloud points bit-equal) and marginal_ok (the only family built to sit inside the bound).
A frame is the dict matcher_oracle uses: kpts [n, 2], depth [H, W], normal [H, W, 4], pose [4, 4] (float32), id."""
import numpy as np

H, W = 48, 64
K = (512.0, 512.0, 32.0, 24.0)
CENTRE = (32, 24)                       # (cx, cy): x = y = 0 at any depth
F32 = np.float32
EZ, EX = (0.0, 0.0, 1.0), (1.0, 0.0, 0.0)


def frame(fid, kpts, depth, normal=None, pose=None):
    if normal is None:
        normal = np.zeros((H, W, 4), F32)
        normal[..., 2] = 1.0
    return {"kpts": np.ascontiguousarray(np.asarray(kpts, F32).reshape(-1, 2)), "depth": np.ascontiguousarray(depth, F32),
            "normal": np.ascontiguousarray(normal, F32), "pose": np.ascontiguousarray(np.eye(4) if pose is None else pose, F32), "id": int(fid)}


def _idx(rows, k):
    """[n, k] int32 candidate lists, each row padded with -1."""
    out = np.full((len(rows), k), -1, np.int32)
    for i, r in enumerate(rows):
        out[i, :len(r)] = r
    return out


def _pose(R=np.eye(3), t=(0.0, 0.0, 0.0)):
    P = np.eye(4)
    P[:3, :3] = R
    P[:3, 3] = t
    return P.astype(F32)


def _dyadic_depth():
    """0.5 + u / 64 + v / 1024: a different dyadic depth at every pixel."""
    v, u = np.mgrid[0:H, 0:W]
    return (0.5 + u / 64.0 + v / 1024.0).astype(F32)


def _below(x):
    return float(np.nextafter(F32(x), F32(-np.inf)))


def _above(x):
    return float(np.nextafter(F32(x), F32(np.inf)))


# ---------------------------------------------------------------------------------------------------------------- 1. pixel rounding
ROUND_X = [2.5, 3.5, _below(2.5), _below(3.5), 0.0, -0.0, -0.5, _above(-0.5), W - 0.5, _below(W - 0.5), W - 1.0]
ROUND_Y = [10.5, 11.5, _below(10.5), -0.5, _above(-0.5), H - 0.5, _below(H - 0.5)]


def _rounded(c, lim):
    """std::round of c, or lim - 1 when that lies outside [0, lim) (the integer partner of an out-of-image coordinate)."""
    r = int(np.floor(abs(c) + 0.5) * (1 if c >= 0 else -1))
    return r if 0 <= r < lim else lim - 1


def rounding():
    """Keypoints at k + 0.5, one float32 below it, -0.5, just above -0.5, W - 0.5 and H - 0.5 (and just below), against integer
    keypoints at std::round of them on the other frame.  Depth differs at every pixel and max_dist is 2^-12, so only a candidate whose
    two keypoints round to the same pixel passes; rintf (half to even) or a shifted in-image test changes rows."""
    D = _dyadic_depth()
    tricky = [(x, 20.0) for x in ROUND_X] + [(30.0, y) for y in ROUND_Y]
    plain = [(_rounded(x, W), _rounded(y, H)) for x, y in tricky]
    n = len(tricky)
    ident = _idx([[i] for i in range(n)], 1)
    cases = []
    for ida, idb, ka, kb in ((3, 1, tricky, plain), (3, 1, plain, tricky), (2, 1, tricky, plain), (2, 1, plain, tricky)):
        cases.append((frame(ida, ka, D), frame(idb, kb, D), ident, ident))
    return [dict(name="rounding", cases=cases, prm=(2.0 ** -12, -1.0, 2.0 ** -12, -1.0), k=1, dyadic=True, marginal_ok=False)]


# ---------------------------------------------------------------------------------------------------------------- 2. depth validity
DEPTHS = [0.1, _below(0.1), 0.0, -1.0, -np.inf, np.nan]


def depth_validity():
    """One feature per pair at pixel (10, 12): depth 0.1f, one float32 below, 0, negative, -inf and NaN on one side, 0.1f on the other.
    The organised cloud holds zeros wherever !(d >= 0.1), so only 0.1f itself passes."""
    cases = []
    one = _idx([[0]], 1)
    for d in DEPTHS:
        for side in (0, 1):
            da, db = np.full((H, W), 0.1, F32), np.full((H, W), 0.1, F32)
            (da if side == 0 else db)[12, 10] = d
            cases.append((frame(5, [(10.0, 12.0)], da), frame(3, [(10.0, 12.0)], db), one, one))
    return [dict(name="depth", cases=cases, prm=(2.0 ** -4, -1.0, 2.0 ** -4, -1.0), k=1, dyadic=False, marginal_ok=False)]


# ---------------------------------------------------------------------------------------------------------------- 3. distance gate
C_NEIGHBOR, C_OTHER = 2.0 ** -4, 2.0 ** -6           # offsets (3c, 0, 4c): distance exactly 5c, 0.3125 and 0.078125


def distance():
    """Three calls whose thresholds are 5c exactly, one float32 below and one above (c per neighbour class), over neighbour pairs (ids
    5, 4 and 4, 5) and non-neighbour pairs (7, 4 and 4, 7) whose one feature each lies at distance 5c of either class: B's point is
    (0, 0, 1 + 4c) at the principal point, moved by (3c, 0, 0) by B's pose.  Equality is kept (the reference tests dist > max_dist)."""
    calls = []
    for name, shift in (("dist_eq", lambda x: x), ("dist_below", _below), ("dist_above", _above)):
        cases = []
        for ida, idb in ((5, 4), (4, 5), (7, 4), (4, 7)):
            for c in (C_NEIGHBOR, C_OTHER):
                db = np.ones((H, W), F32)
                db[CENTRE[1], CENTRE[0]] = 1.0 + 4.0 * c
                one = _idx([[0]], 1)
                cases.append((frame(ida, [CENTRE], np.ones((H, W), F32)), frame(idb, [CENTRE], db, pose=_pose(t=(3.0 * c, 0.0, 0.0))), one, one))
        prm = (shift(5.0 * C_OTHER), -1.0, shift(5.0 * C_NEIGHBOR), -1.0)
        calls.append(dict(name=name, cases=cases, prm=prm, k=1, dyadic=True, marginal_ok=False))
    return calls


# ---------------------------------------------------------------------------------------------------------------- 4. normal gate
COS_90 = float(F32(np.cos(np.pi / 2)))                 # 6.1e-17, not 0: a dot of exactly 0 is rejected at 90 degrees
R_PERM = np.array([[0.0, -1.0, 0.0], [0.0, 0.0, 1.0], [-1.0, 0.0, 0.0]])       # a signed permutation (det +1)


def normal_gate():
    """Exact dot products 1, 0 and -1 of model-frame normals (B's pose is a signed permutation, its camera normals rotated back) against
    cos_max of 1, 0, cos(90 deg) and -1, neighbour pair (2, 1) and non-neighbour pair (3, 1) in each call."""
    calls = []
    pixels = [(8, 8), (16, 8), (24, 8)]
    for ci, (c_other, c_nb) in enumerate(((1.0, 0.0), (COS_90, -1.0), (-1.0, 1.0), (0.0, COS_90))):
        cases = []
        for ida in (2, 3):
            na = np.zeros((H, W, 4), F32)
            nb = np.zeros((H, W, 4), F32)
            for (u, v), m in zip(pixels, (EZ, EX, (0.0, 0.0, -1.0))):
                na[v, u, :3] = EZ
                nb[v, u, :3] = R_PERM.T @ np.asarray(m)      # model normal R n = m
            ident = _idx([[0], [1], [2]], 1)
            cases.append((frame(ida, pixels, np.ones((H, W), F32), na), frame(1, pixels, np.ones((H, W), F32), nb, _pose(R_PERM)), ident, ident))
        calls.append(dict(name=f"normal_{ci}", cases=cases, prm=(64.0, c_other, 64.0, c_nb), k=1, dyadic=True, marginal_ok=False))
    return calls


def zero_normal():
    """THE zero-normal case: a zero normal on A, on B and on both, at cos_max = 1.  A zero normal normalises to NaN and the NaN dot does
    not reject (matcher_oracle.ZERO_NORMAL_KEEPS; Eigen 3.3 would give 0 and reject: DESIGN.md §3.2)."""
    pixels = [(8, 30), (16, 30), (24, 30)]
    cases = []
    for ida in (2, 3):
        na = np.zeros((H, W, 4), F32)
        nb = np.zeros((H, W, 4), F32)
        for j, (u, v) in enumerate(pixels):
            na[v, u, :3] = (0.0, 0.0, 0.0) if j != 1 else EZ
            nb[v, u, :3] = (0.0, 0.0, 0.0) if j != 0 else EZ
        ident = _idx([[0], [1], [2]], 1)
        cases.append((frame(ida, pixels, np.ones((H, W), F32), na), frame(1, pixels, np.ones((H, W), F32), nb), ident, ident))
    return [dict(name="zero_normal", cases=cases, prm=(64.0, 1.0, 64.0, 1.0), k=1, dyadic=True, marginal_ok=False)]


NEAR_S = 2.0 ** -6


def normal_near():
    """Dots next to cos_max, inside the float32 bound: B's normal (s, 0, 1) against A's (0, 0, 1), dot 1 / sqrt(1 + s^2), with cos_max
    the float32 nearest to it and a few ulps either side.  Either decision is allowed; the test prints them."""
    dot = 1.0 / np.sqrt(1.0 + NEAR_S ** 2)
    calls = []
    for j, c in enumerate((float(F32(dot)), _below(dot), _above(dot), float(F32(dot) + F32(4 * 2.0 ** -24)))):
        na = np.zeros((H, W, 4), F32)
        nb = np.zeros((H, W, 4), F32)
        na[8, 8, :3] = EZ
        nb[8, 8, :3] = (NEAR_S, 0.0, 1.0)
        one = _idx([[0]], 1)
        cases = [(frame(3, [(8, 8)], np.ones((H, W), F32), na), frame(1, [(8, 8)], np.ones((H, W), F32), nb), one, one)]
        calls.append(dict(name=f"normal_near_{j}", cases=cases, prm=(64.0, c, 64.0, c), k=1, dyadic=True, marginal_ok=True))
    return calls


# ---------------------------------------------------------------------------------------------------------------- 5/6. candidate lists, sizes
MAX_DIST_SCENE = 0.04


def _scene_depth(rng):
    """Dyadic depths (multiples of 1/64 in [0.5, 1.5)), about one pixel in seven invalid (0)."""
    d = (32 + rng.integers(0, 64, size=(H, W))) / 64.0
    d[rng.random((H, W)) < 0.15] = 0.0
    return d.astype(F32)


def scene_pair(rng, nA, nB, k, idA, idB, one_way=False):
    """Random integer keypoints on one dyadic depth map shared by both frames (identity poses): a candidate passes when its two points
    are within MAX_DIST_SCENE, e.g. the same pixel.  B's first min(nA, nB) keypoints are A's, shuffled, so most A queries have a
    same-pixel partner; each list holds k entries drawn from: the partner, a keypoint next to it, random rows, -1, nT and larger
    indices.  one_way: B's lists are all -1 (only the A->B direction can survive)."""
    D = _scene_depth(rng)
    ka = np.stack([rng.integers(0, W, nA), rng.integers(0, H, nA)], 1).astype(F32)
    kb = np.stack([rng.integers(0, W, nB), rng.integers(0, H, nB)], 1).astype(F32)
    m = min(nA, nB)
    perm = rng.permutation(nB)[:m] if nB else np.zeros(0, np.int64)
    kb[perm] = ka[:m]
    near = kb[perm] + rng.integers(-1, 2, size=(m, 2))
    near = np.clip(near, [0, 0], [W - 1, H - 1])

    def lists(nq, nt, partner):
        out = np.empty((nq, k), np.int32)
        for q in range(nq):
            pool = []
            for _ in range(k):
                r = rng.random()
                if r < 0.1:
                    pool.append(-1)
                elif r < 0.15:
                    pool.append(nt + int(rng.integers(0, 3)) * 1000)
                else:
                    pool.append(int(rng.integers(0, nt)) if nt else -1)
            if partner is not None and q < len(partner) and rng.random() < 0.85:
                pool[int(rng.integers(0, k))] = int(partner[q])
            out[q] = pool
        return out

    inv = np.full(nB, -1, np.int64)
    inv[perm] = np.arange(m)
    idxAB = lists(nA, nB, perm)
    idxBA = np.full((nB, k), -1, np.int32) if one_way else lists(nB, nA, np.where(inv >= 0, inv, rng.integers(0, max(nA, 1), nB)) if nA else None)
    B = frame(idB, kb, D)
    if m:      # some partners moved to a neighbouring pixel in B: those candidates pass or fail on distance
        moved = rng.random(m) < 0.2
        B["kpts"][perm[moved]] = near[moved]
    return frame(idA, ka, D), B, idxAB, idxBA


def candidates(seed=11):
    """k = 1, 5 and 8: lists with -1, indices >= Tn.n, failing candidates (invalid depth, too far), and passing candidates behind a
    passing one (the first wins, not the closest); neighbour and non-neighbour pairs."""
    calls = []
    for k in (1, 5, 8):
        rng = np.random.default_rng(seed + k)
        cases = [scene_pair(rng, 96, 80, k, 1, 0), scene_pair(rng, 80, 96, k, 6, 2)]
        calls.append(dict(name=f"candidates_k{k}", cases=cases, prm=(MAX_DIST_SCENE, -1.0, MAX_DIST_SCENE / 2, -1.0), k=k, dyadic=True, marginal_ok=False))
    return calls


SIZES_MAX_FEATS = 1100
SIZES = [(0, 1), (1, 0), (1, 1), (511, 512), (512, 513), (513, 1024), (1024, 1025), (1025, SIZES_MAX_FEATS), (SIZES_MAX_FEATS, 511)]


def sizes(seed=5):
    """nA, nB across 0, 1, 511, 512, 513, 1024, 1025 and max_feats in one batch (k_prune_mutual's 512-row chunks and its running
    base), plus a pair where only A->B can survive."""
    rng = np.random.default_rng(seed)
    cases = [scene_pair(rng, nA, nB, 5, 4 + (p % 2), 3) for p, (nA, nB) in enumerate(SIZES)]
    cases.append(scene_pair(rng, 700, 600, 5, 9, 3, one_way=True))
    return [dict(name="sizes", cases=cases, prm=(MAX_DIST_SCENE, -1.0, MAX_DIST_SCENE, -1.0), k=5, dyadic=True, marginal_ok=False)]


def prune_calls():
    return rounding() + depth_validity() + distance() + normal_gate() + zero_normal() + normal_near() + candidates() + sizes()


# ---------------------------------------------------------------------------------------------------------------- descriptor-driven pairs
D = 256
N_DECOY = 5            # = the k of findCorres: a B feature whose 5 nearest A rows are decoys never reaches its real partner
DEAD = (0, 0)          # A's decoy pixel, depth 0


def _desc_rows(rng, n):
    return (rng.integers(-256, 257, size=(n, D)) / 64.0).astype(F32)


def desc_pair(rng, rows, idA, idB, pixels=None):
    """A frame pair for bt_match_pairs_ex built from match rows.  A row is (kind, (uA, vA, dA), (uB, vB, dB)):
      "sym"  A and B features with one descriptor: matched A->B and B->A, two candidate rows;
      "one"  A's descriptor is B's plus 0.25 on one component, and N_DECOY A features at the dead pixel carry B's exactly: B's five
             nearest A rows all fail the depth test, so only the A->B candidate exists.
    Rows are matched in order (A->B block in A's feature order, which is the rows' order; then B->A).  Identity poses, normals e_z;
    each pixel carries its row's depth.  Returns (A, B) with "desc" [n, 256] float32 added."""
    da, db = np.zeros((H, W), F32), np.zeros((H, W), F32)
    ka, kb, desc_a, desc_b, decoys = [], [], [], [], []
    base = _desc_rows(rng, len(rows))
    for i, (kind, (ua, va, dA), (ub, vb, dB)) in enumerate(rows):
        da[va, ua], db[vb, ub] = dA, dB
        ka.append((ua, va)); kb.append((ub, vb)); desc_b.append(base[i])
        if kind == "sym":
            desc_a.append(base[i])
        else:
            bumped = base[i].copy()
            bumped[i % D] += 0.25
            desc_a.append(bumped)
            decoys += [base[i]] * N_DECOY
    ka += [DEAD] * len(decoys)
    desc_a += decoys
    da[DEAD[1], DEAD[0]] = 0.0
    A = frame(idA, ka, da)
    B = frame(idB, kb, db)
    A["desc"] = np.asarray(desc_a, F32).reshape(-1, D)
    B["desc"] = np.asarray(desc_b, F32).reshape(-1, D)
    return A, B


def free_pixels(rng, n):
    """n distinct pixels away from the dead pixel and from column 0."""
    flat = rng.choice(np.arange(W + 1, H * W), size=n, replace=False)
    return [(int(f % W), int(f // W)) for f in flat]


def _depth(rng):
    return float((40 + rng.integers(0, 48)) / 64.0)


def consistent_rows(rng, kind, n, pixels):
    """n rows whose two endpoints are the same 3-D point (same pixel, same depth): exact RANSAC inliers."""
    out = []
    for j in range(n):
        u, v = pixels.pop()
        d = _depth(rng)
        out.append((kind, (u, v, d), (u, v, d)))
    return out


def outlier_rows(rng, kind, n, pixels):
    """n rows whose B endpoint lies 0.5 m or more behind the A endpoint: far outside any inlier threshold below 0.1."""
    out = []
    for j in range(n):
        u, v = pixels.pop()
        d = _depth(rng)
        out.append((kind, (u, v, d), (u, v, d + 0.5 + 0.25 * (j % 3))))
    return out


def count_rule_rows(rng, name):
    """Pairs that end exactly on the five-match rules: c5 / c6 candidates before RANSAC (<= 5 clears the pair), i4 / i5 inliers after it
    (< 5 clears), all one-way rows."""
    px = free_pixels(rng, 32)
    return {"c5": consistent_rows(rng, "one", 5, px),
            "c6": consistent_rows(rng, "one", 6, px),
            "i4": consistent_rows(rng, "one", 4, px) + outlier_rows(rng, "one", 2, px),
            "i5": consistent_rows(rng, "one", 5, px) + outlier_rows(rng, "one", 2, px),
            "i5o1": consistent_rows(rng, "one", 5, px) + outlier_rows(rng, "one", 1, px)}[name]


COUNT_RULES = ["c5", "c6", "i4", "i5", "i5o1"]


def emission_templates(rng):
    """Pairs for the capacity cut: 6 and 7 entries (one-way), a cleared pair, 300 entries (150 sym rows: k_emit_fill's 256-thread loop),
    12 entries (6 sym rows)."""
    px = free_pixels(rng, 600)
    return [consistent_rows(rng, "one", 6, px), consistent_rows(rng, "sym", 2, px), consistent_rows(rng, "sym", 150, px),
            consistent_rows(rng, "one", 5, px) + outlier_rows(rng, "one", 2, px), consistent_rows(rng, "one", 4, px),
            consistent_rows(rng, "sym", 6, px)]


def many_pair_templates(rng):
    """Small pairs for a batch of thousands: cleared before RANSAC (4 and 5 candidates), cleared after it (4 inliers), and 6 to 16
    entries."""
    px = lambda: free_pixels(rng, 16)
    return [consistent_rows(rng, "sym", 2, px()), consistent_rows(rng, "one", 5, px()), consistent_rows(rng, "sym", 3, px()),
            consistent_rows(rng, "one", 4, px()) + outlier_rows(rng, "one", 2, px()), consistent_rows(rng, "sym", 8, px()),
            consistent_rows(rng, "one", 5, px()) + outlier_rows(rng, "one", 1, px()), consistent_rows(rng, "sym", 5, px())]


def propagated_case(rng, n_fresh=300):
    """A non-neighbour pair's mutual rows (8 sym rows, one at column 0) and the propagated matches of findCorresByMapPoints against them:
    duplicates on (uA, vA) only, on (uB, vB) only, on both, on neither; -0.0 against a mutual row's +0.0; outside the image; on invalid
    depth; and n_fresh more (over k_append_propagated's 256-thread CTA).  Returns (rows, extras [m, 4] float32)."""
    px = free_pixels(rng, 24)
    rows = consistent_rows(rng, "sym", 7, px) + [("sym", (0, 7, 0.75), (0, 9, 0.75))]
    a0, a1, a2 = rows[0][1], rows[1][1], rows[2][1]
    b1, b2 = rows[1][2], rows[2][2]
    f = px[:8]
    ex = [(a0[0], a0[1], f[0][0], f[0][1]),          # (uA, vA) taken
          (f[1][0], f[1][1], b1[0], b1[1]),          # (uB, vB) taken
          (a2[0], a2[1], b2[0], b2[1]),              # both
          (f[2][0], f[2][1], f[3][0], f[3][1]),      # neither
          (-0.0, 7.0, f[4][0], f[4][1]),             # -0.0 == the mutual row's +0.0
          (f[5][0], f[5][1], 0.0, 9.0 + 0.25),       # uB +0.0 but vB differs: kept
          (-3.0, 5.0, f[6][0], f[6][1]),             # outside the image: zero A point
          (f[7][0], f[7][1], W + 2.0, 4.0),          # outside the image: zero B point
          (0.0, 0.0, 0.0, 0.0),                      # invalid depth on A (the dead pixel)
          (f[2][0] + 0.5, f[2][1], f[3][0], f[3][1] + 0.4999)]
    fresh = np.stack([rng.integers(1, W, n_fresh) + rng.choice([0.0, 0.25, 0.5], n_fresh), rng.integers(1, H, n_fresh),
                      rng.integers(1, W, n_fresh), rng.integers(1, H, n_fresh) + rng.choice([0.0, 0.5], n_fresh)], 1)
    return rows, np.concatenate([np.asarray(ex, F32), fresh.astype(F32)], 0)
