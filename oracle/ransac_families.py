"""Point pairs built against batched RANSAC (ransac.cu) from the sampling table alone: which three ids every trial draws is fixed by
tests/golden/curand_xorwow_seed0.npy for any n, so a pair can be laid out to make a chosen trial the winner.  Shared by the oracle's CPU
tests and the GPU tests of ransac.cu.

Words used below: a cluster is a set of ids whose B points are one rigid motion of their A points; a trial is pure for a cluster when its
three ids are distinct members of it.  A pure trial fits its cluster to ~1e-7 m, so it counts every member; every point outside the
clusters lies at least 1 m from every cluster's motion, and a trial mixing clusters and outliers fits neither.  The winner is the lowest
pure trial of the largest cluster.

A call is a dict: name, pairs [(A [n, 4] float32, B [n, 4] float32)], n_trials, thresh, expect [per pair (trial, count) or None: the winner
and its count] and, for the threshold family, probes [per pair: {id: "eq" | "above" | "below"}]."""
import os

import numpy as np

from . import matcher_oracle as mo

F32 = np.float32
GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "curand_xorwow_seed0.npy")
THRESH = 0.01
MAX_PTS = 4200            # the reserve of the chunk family: 4 full 1024-point chunks and a 104-point tail
MAX_TRIALS = 2000


def table():
    return np.load(GOLD)


def sample_ids(n, n_trials):
    return mo.ransac_sample_ids(table()[:n_trials], n)


def _rotation(rng, angle=None, axis=None):
    axis = rng.normal(size=3) if axis is None else np.asarray(axis, np.float64)
    axis = axis / np.linalg.norm(axis)
    a = rng.uniform(0.2, 3.0) if angle is None else angle
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K


def _distinct(tri):
    return len(set(int(i) for i in tri)) == 3


def lowest_pure(ids, members, n_trials=None):
    """The lowest trial whose three distinct ids all lie in `members`, or -1."""
    m = np.zeros(int(ids.max()) + 1 if len(ids) else 1, bool)
    m[[i for i in members if i < len(m)]] = True
    T = len(ids) if n_trials is None else n_trials
    for t in range(T):
        if _distinct(ids[t]) and m[ids[t]].all():
            return t
    return -1


def grow_cluster(ids, T, k, pool, taken, rng):
    """k ids holding trial T's three whose lowest pure trial is T: members are drawn from `pool` (minus `taken`) and skipped when they
    would complete the triple of an earlier trial.  Returns the member list, or None when T's ids are not distinct or already taken."""
    tri = [int(i) for i in ids[T]]
    if not _distinct(tri) or any(i in taken for i in tri):
        return None
    members = set(tri)
    if lowest_pure(ids[:T], members) >= 0:
        return None
    by_id = {}
    for t in range(T):
        if _distinct(ids[t]):
            for i in set(int(v) for v in ids[t]):
                by_id.setdefault(i, []).append(t)
    for c in rng.permutation(np.asarray(sorted(set(pool) - taken - members), np.int64)):
        if len(members) >= k:
            break
        c = int(c)
        if any(all(int(v) in members or int(v) == c for v in ids[t]) for t in by_id.get(c, [])):
            continue
        members.add(c)
    return sorted(members) if len(members) == k else None


def build_pair(n, clusters, rng, motions=None):
    """A [n, 4] and B [n, 4] float32: cluster c's B is its own motion of A (identity rotation for no motion given: translations 3 m apart),
    every other point an outlier ten metres away.  A lies in the cube [-0.5, 0.5]^3."""
    A = rng.uniform(-0.5, 0.5, size=(n, 3))
    B = A + np.array([0.0, 0.0, 10.0]) + rng.uniform(-1.0, 1.0, size=(n, 3))
    for c, mem in enumerate(clusters):
        R = _rotation(rng) if motions is None else motions[c]
        t = np.array([3.0 * c - 3.0, 0.5, -0.25])
        mem = np.asarray(mem, np.int64)
        B[mem] = A[mem] @ R.T + t
    return _pack(A), _pack(B)


def _pack(P):
    out = np.zeros((len(P), 4), F32)
    out[:, :3] = P
    return out


# ---------------------------------------------------------------------------------------------------------------- 1. ties
K_TIE = 24


def _tie_case(rng, n, n_trials, specs):
    """specs: [(trial, size)] in build order; each later cluster's trial is searched from its given trial upwards until its ids are free.
    Returns (A, B, [(trial, members)])."""
    ids = sample_ids(n, n_trials)
    taken, got = set(), []
    for T, k in specs:
        while True:
            mem = grow_cluster(ids, T, k, range(n), taken, rng)
            if mem is not None or T >= n_trials - 1:
                break
            T += 1
        assert mem is not None, (n, specs)
        taken |= set(mem)
        got.append((T, mem))
    A, B = build_pair(n, [m for _, m in got], rng)
    return A, B, got


def ties(seed=1):
    """Two (or three) equal clusters under different motions whose lowest pure trials are T and a later one: T = 0, 255, 256 and 1023
    win with K_TIE.  tie_last: n_trials = 1800 and the winner is trial 1799, the last of a part-filled block, against an earlier cluster
    one point smaller.  near_tie: a cluster of K_TIE - 1 whose pure trial comes first loses to a cluster of K_TIE whose trial is >= 1000."""
    rng = np.random.default_rng(seed)
    calls = []
    n = 1500
    for T in (0, 255, 256, 1023):
        specs = [(T, K_TIE), (T + 1 + 37 * (T % 5), K_TIE)] + ([(T + 200, K_TIE)] if T == 256 else [])
        A, B, got = _tie_case(rng, n, MAX_TRIALS, specs)
        assert got[0][0] == T
        calls.append(dict(name=f"tie_{T}", pairs=[(A, B)], n_trials=MAX_TRIALS, thresh=THRESH, expect=[(T, K_TIE)]))
    A, B, got = _tie_case(rng, n, 1800, [(1799, K_TIE), (3, K_TIE - 1)])
    assert got[0][0] == 1799
    calls.append(dict(name="tie_last", pairs=[(A, B)], n_trials=1800, thresh=THRESH, expect=[(1799, K_TIE)]))
    A, B, got = _tie_case(rng, n, MAX_TRIALS, [(1000, K_TIE), (2, K_TIE - 1)])
    calls.append(dict(name="near_tie", pairs=[(A, B)], n_trials=MAX_TRIALS, thresh=THRESH, expect=[(got[0][0], K_TIE)]))
    return calls


# ---------------------------------------------------------------------------------------------------------------- 2. chunks and tails
CHUNK_NS = [3, 4, 5, 1023, 1024, 1025, 2047, 2048, 2049, 3073, MAX_PTS]
K_WIN, K_DECOY = 40, 39


def _first_in(ids, lo, hi, taken=(), start=0):
    for t in range(start, len(ids)):
        tri = [int(i) for i in ids[t]]
        if _distinct(tri) and all(lo <= i < hi and i not in taken for i in tri):
            return t
    return -1


def chunks(seed=2):
    """One batch: n in CHUNK_NS plus pairs of 0 and 2 points.  For n >= 1023 the winner's three samples lie in the last 1024 points and
    its other members in the final 128 (the last check step, or the two last when the tail chunk is shorter), and a decoy cluster one
    point smaller, sampled earlier, sits in the first chunk: its count is published while the winner has seen few of its points.  For
    n = 3, 4, 5 the winner is the first good trial and its three points the only cluster.
    Only the winner's other members are confined to the final 128 points, not its three samples: a trial whose three ids all fall in the
    last 128 of n points has probability (128 / n)^3, about 1 in 35000 at n = 4200, so 2000 trials rarely hold one.  The winner has then
    counted at most 3 points at the check before the final step, with k - 3 still ahead."""
    rng = np.random.default_rng(seed)
    pairs, expect = [], []
    for n in CHUNK_NS:
        ids = sample_ids(n, MAX_TRIALS)
        if n <= 5:
            T = next(t for t in range(MAX_TRIALS) if _distinct(ids[t]))
            A, B = build_pair(n, [sorted(int(i) for i in ids[T])], rng)
            pairs.append((A, B))
            expect.append((T, 3))
            continue
        win_lo, tail_lo = max(0, n - 1024), n - 128
        dec_hi = min(1024, tail_lo)
        start = 0
        while True:
            W = _first_in(ids, win_lo, n, start=start)
            assert W >= 0, n
            win = grow_cluster(ids, W, K_WIN, range(tail_lo, n), set(), rng)
            if win is not None and lowest_pure(ids, win) == W:
                break
            start = W + 1
        D = _first_in(ids, 0, dec_hi, taken=set(win))
        dec = grow_cluster(ids, D, K_DECOY, range(0, dec_hi), set(win), rng)
        assert dec is not None, n
        A, B = build_pair(n, [win, dec], rng)
        pairs.append((A, B))
        expect.append((W, K_WIN))
    for n in (0, 2, 0):
        A, B = build_pair(n, [], rng)
        pairs.append((A, B))
        expect.append(None)
    order = rng.permutation(len(pairs))           # sizes differ from pair to pair, small and empty pairs between large ones
    return [dict(name="chunks", pairs=[pairs[i] for i in order], n_trials=MAX_TRIALS, thresh=THRESH, expect=[expect[i] for i in order])]


# ---------------------------------------------------------------------------------------------------------------- 3. publication order
PUB_PAIRS, PUB_N, PUB_K = 512, 4096, 64


def publication(seed=3):
    """Two tying clusters of PUB_K, repeated over PUB_PAIRS pairs (more than one wave of eval blocks).  The lower trial L sits in block 0
    and samples the last chunk; the higher, H, is the last trial (n_trials = H + 1), one of at most 32 in the last block, and samples the
    first chunk.  L wins; a tying trial that finishes first must not stop it."""
    rng = np.random.default_rng(seed)
    ids = sample_ids(PUB_N, MAX_TRIALS)
    n = PUB_N
    for H in range(256, MAX_TRIALS):
        if H % 256 >= 32 or not (_distinct(ids[H]) and (ids[H] < 1024).all()):
            continue
        L = _first_in(ids[:256], n - 1024, n)
        cl = grow_cluster(ids, L, PUB_K, range(n - 1024, n), set(), rng)
        ch = grow_cluster(ids, H, PUB_K, range(0, 1024), set(cl), rng)
        if ch and lowest_pure(ids[:H + 1], cl) == L and lowest_pure(ids[:H + 1], ch) == H:
            break
    else:
        raise AssertionError("no layout found")
    A, B = build_pair(n, [cl, ch], rng)
    return [dict(name="publication", pairs=[(A, B)] * PUB_PAIRS, n_trials=H + 1, thresh=THRESH, expect=[(L, PUB_K)] * PUB_PAIRS)]


# ---------------------------------------------------------------------------------------------------------------- 4. threshold equality
EQ_N, EQ_TRIALS = 600, 200
EQ_THRESH = [0.005, 0.01, 2.0 ** -7, 2.0 ** -50]


def probe_offset(target):
    """(dx, dy) float32 with fl(dx^2 + fl(dy^2)) == target exactly, dx^2 exact in float32 (12 significant bits): with a = 0, b = (dx, dy,
    0) and the pose [I | 0], the kernel's d2 is that in every contraction order."""
    from fractions import Fraction
    target = float(F32(target))
    m, e = np.frexp(np.sqrt(target) * (1.0 - 2.0 ** -9))
    dx = float(np.ldexp(np.floor(m * 2 ** 12) / 2 ** 12, e))
    r = target - dx * dx
    dy0 = float(F32(np.sqrt(r)))
    for k in range(64):
        for dy in (dy0, float(np.nextafter(F32(dy0), F32(np.inf))), float(np.nextafter(F32(dy0), F32(0)))):
            dy2 = mo.f32_round(Fraction(dy) * Fraction(dy))
            if mo.f32_round(Fraction(dx) * Fraction(dx) + Fraction(dy2)) == target:
                return dx, dy
        dy0 = float(np.nextafter(F32(dy0), F32(np.inf if mo.f32_round(Fraction(dx) ** 2 + Fraction(dy0) ** 2) < target else 0)))
    raise AssertionError(target)


def equality_pair(n, thresh, rng, probes=True):
    """Identity-motion pair (B = A bit for bit): every pure trial's fit is exactly [I | 0].  Every sampled id is a cluster point; three
    never-sampled ids carry probes at a = 0 whose d2 is exactly d2_max, one float above and one below.  Returns (A, B, {id: kind})."""
    ids = sample_ids(n, EQ_TRIALS)
    A = rng.uniform(0.1, 0.6, size=(n, 3))
    while True:          # no sampled triple near collinear: the second scatter eigenvalue at least 1e-2 of the largest
        bad = []
        for tri in ids:
            if _distinct(tri):
                s = A[tri] - A[tri].mean(0)
                ev = np.linalg.eigvalsh(s.T @ s)
                if ev[1] < 1e-2 * ev[2]:
                    bad += [int(i) for i in tri]
        if not bad:
            break
        A[bad] = rng.uniform(0.1, 0.6, size=(len(bad), 3))
    A = A.astype(F32).astype(np.float64)
    B = A.copy()
    kinds = {}
    if probes:
        free = sorted(set(range(n)) - set(int(i) for i in ids.ravel()))
        d2m = mo.sqrt_le_max(thresh)
        for kind, target, i in (("eq", d2m, free[0]), ("above", np.nextafter(d2m, F32(np.inf)), free[len(free) // 2]),
                                ("below", np.nextafter(d2m, F32(0)), free[-1])):
            dx, dy = probe_offset(target)
            A[i] = 0.0
            B[i] = (dx, dy, 0.0)
            kinds[i] = kind
    return _pack(A), _pack(B), kinds


def equality(seed=4):
    """Probes at exactly d2_max, one float32 above and one below for thresholds 0.005, 0.01, 2^-7 and 2^-50; the same pair at 0 (only
    distance 0 passes), -1 and NaN (nothing passes); and every point of an odd-sized pair at +inf (the padding point of the odd tail
    never counts).  All trials are pure, so the winner is the first good trial."""
    rng = np.random.default_rng(seed)
    calls = []
    for th in EQ_THRESH:
        A, B, kinds = equality_pair(EQ_N, th, rng)
        T = lowest_pure(sample_ids(EQ_N, EQ_TRIALS), range(EQ_N))
        calls.append(dict(name=f"eq_{th:g}", pairs=[(A, B)], n_trials=EQ_TRIALS, thresh=th, expect=[(T, EQ_N - 1)], probes=[kinds]))
    A, B, kinds = equality_pair(EQ_N, 0.005, rng)
    T = lowest_pure(sample_ids(EQ_N, EQ_TRIALS), range(EQ_N))
    for th, cnt in ((0.0, EQ_N - 3), (-1.0, 0), (float("nan"), 0)):
        calls.append(dict(name=f"eq_{th:g}", pairs=[(A, B)], n_trials=EQ_TRIALS, thresh=th, expect=[(T, cnt)], probes=[kinds]))
    A, B, _ = equality_pair(EQ_N + 1, float("inf"), rng, probes=False)
    T = lowest_pure(sample_ids(EQ_N + 1, EQ_TRIALS), range(EQ_N + 1))
    calls.append(dict(name="eq_inf_odd", pairs=[(A, B)], n_trials=EQ_TRIALS, thresh=float("inf"), expect=[(T, EQ_N + 1)]))
    return calls


# ---------------------------------------------------------------------------------------------------------------- 5. degenerate samples
DEG_N = 2000
WELL = {"generic", "generic_noisy", "mirror", "rot180_x", "rot180_y", "rot180_z", "rot179.9_x", "rot179.9_y", "rot179.9_z", "near_col_1e-1"}


def _configs(rng):
    """(name, s [3, 3], d [3, 3]) per degenerate sample."""
    out = []
    R, t = _rotation(rng), np.array([0.3, -0.2, 0.5])
    s = rng.uniform(-0.5, 0.5, size=(3, 3))
    out.append(("generic", s, s @ R.T + t))
    out.append(("generic_noisy", s, s @ R.T + t + rng.normal(scale=0.05, size=(3, 3))))
    c2 = s.copy()
    c2[1] = c2[0]
    out.append(("coincident_2", c2, c2 @ R.T + t))
    c3 = np.repeat(s[:1], 3, 0)
    out.append(("coincident_3", c3, c3 @ R.T + t))
    line = np.array([[0.0, 0.0, 0.0], [0.25, 0.5, 0.125], [0.75, 1.5, 0.375]])
    out.append(("collinear", line, line + np.array([0.5, 0.25, -0.5])))
    for eps in (1e-1, 1e-2, 1e-3, 1e-4, 1e-5, 1e-6):
        nc = np.array([[0.0, 0.0, 0.0], [0.5, 0.0, 0.0], [0.25, eps, 0.0]])
        out.append((f"near_col_{eps:g}", nc, nc @ R.T + t))
    m = s * np.array([1.0, 1.0, -1.0])
    out.append(("mirror", s, m + t))
    for ang in (np.pi, np.radians(179.9)):
        for ax, v in zip("xyz", np.eye(3)):
            Rx = _rotation(rng, ang, v)
            out.append((f"rot{np.degrees(ang):.4g}_{ax}", s, s @ Rx.T + t))
    far = 100.0 + rng.uniform(-5e-4, 5e-4, size=(3, 3))
    out.append(("far_1mm", far, far @ R.T + t))
    nan_s = s.copy()
    nan_s[0, 1] = np.nan
    out.append(("nan_sample", nan_s, s @ R.T + t))
    inf_d = s @ R.T + t
    inf_d[2, 0] = np.inf
    out.append(("inf_sample", s, inf_d))
    return out


def degenerate(seed=5):
    """One pair of DEG_N points, a generic cluster under one motion plus outliers, where each degenerate sample is given to its own trial
    (the trials chosen in order with ids disjoint from the earlier ones): generic, noisy, two and three coincident points at distinct ids,
    exactly collinear, near-collinear with the offset swept from 1e-1 to 1e-6, a mirror image, 180 and 179.9 degree turns about each axis,
    a 1 mm spread 100 m from the origin, NaN and inf in a sample; and NaN and inf points at ids no trial samples.  Returns the call with
    `trials` {trial: config name}."""
    rng = np.random.default_rng(seed)
    ids = sample_ids(DEG_N, MAX_TRIALS)
    base = sorted(rng.choice(DEG_N, DEG_N // 2, replace=False).tolist())
    A, B = build_pair(DEG_N, [base], rng)
    used, trials, t = set(), {}, 0
    for name, s, d in _configs(rng):
        while not (_distinct(ids[t]) and not (set(int(i) for i in ids[t]) & used)):
            t += 1
        tri = [int(i) for i in ids[t]]
        used |= set(tri)
        with np.errstate(invalid="ignore"):
            A[tri, :3] = s
            B[tri, :3] = d
        trials[t] = name
        t += 1
    free = sorted(set(range(DEG_N)) - set(int(i) for i in ids.ravel()))
    A[free[0], :3] = np.nan
    B[free[1], :3] = (np.inf, 0.0, 0.0)
    A[free[2], :3] = (-np.inf, 1.0, 1.0)
    B[free[3], :3] = np.nan
    return [dict(name="degenerate", pairs=[(A, B)], n_trials=MAX_TRIALS, thresh=0.05, expect=[None], trials=trials,
                 nonfinite=free[:4])]


def all_calls():
    return ties() + chunks() + publication() + equality() + degenerate()


# ---------------------------------------------------------------------------------------------------------------- the 3-point fit
_U = 2.0 ** -24


def fit_tolerances(s, d):
    """(rss_tol, r_tol, t_tol) for one trial's float32 fit of samples s -> d, against the float64 Kabsch fit.
    rss: the device's residual sum of squares on its own samples may exceed Kabsch's minimum by 64 u times the samples' scatter (an error
    e in the quaternion costs at most e times the profile matrix's scale) plus the translation's rounding, 3 (16 u M)^2 with M the largest
    coordinate magnitude.  pose (well-conditioned samples only): every entry of R within 2e-5 and of t within 2e-5 (1 + M)."""
    s = np.asarray(s, np.float64)
    d = np.asarray(d, np.float64)
    scatter = ((s - s.mean(0)) ** 2).sum() + ((d - d.mean(0)) ** 2).sum()
    M = max(np.abs(s).max(), np.abs(d).max())
    return 64.0 * _U * scatter + 3.0 * (16.0 * _U * M) ** 2, 2e-5, 2e-5 * (1.0 + M)


# ---------------------------------------------------------------------------------------------------------------- 6. operation order
OP_N, OP_TRIALS, OP_K, OP_PROBES = 8000, 300, 40, 24


def op_order(seed=6):
    """A pair of OP_N points of which the OP_TRIALS trials sample few: one cluster of OP_K under a generic motion whose only pure trial W
    is the first that can hold it (its other members are never sampled), outliers elsewhere, and OP_PROBES never-sampled ids kept free
    (outliers in this layout) for op_order_probes.  Returns (call, probe ids)."""
    rng = np.random.default_rng(seed)
    ids = sample_ids(OP_N, OP_TRIALS)
    sampled = set(int(i) for i in ids.ravel())
    free = [i for i in range(OP_N) if i not in sampled]
    probes = [int(i) for i in rng.choice(free, OP_PROBES, replace=False)]
    pool = sorted(set(free) - set(probes))
    W = next(t for t in range(OP_TRIALS) if _distinct(ids[t]))
    mem = grow_cluster(ids, W, OP_K, pool, set(probes), rng)
    A, B = build_pair(OP_N, [mem], rng)
    return dict(name="op_order", pairs=[(A, B)], n_trials=OP_TRIALS, thresh=THRESH, expect=[(W, OP_K)]), probes


def _d2_grid(m, bx, by, bz, fused_sq):
    """d2 of every b in the grid for the float32 model point m, in float32 arithmetic (numpy's float32 subtraction and products are
    correctly rounded; a fused multiply-add is the exact float64 product plus the addend, rounded twice, so hits are confirmed exactly)."""
    f = np.float32
    dx, dy, dz = (np.asarray(bx, f) - f(m[0])), (np.asarray(by, f) - f(m[1])), (np.asarray(bz, f) - f(m[2]))
    d64 = [v.astype(np.float64) for v in (dx, dy, dz)]
    if fused_sq:
        inner = (d64[0] * d64[0] + (dy * dy).astype(np.float64)).astype(f)
        return (d64[2] * d64[2] + inner.astype(np.float64)).astype(f)
    return ((dx * dx) + (dy * dy)) + (dz * dz)


def op_order_probes(P, probe_ids, thresh, rng, span=120):
    """Moves the probe points onto the contraction boundary of the float32 pose P [3, 4]: each probe (a, b) has b about thresh from
    P a, and b is searched over a grid of (2 span + 1)^2 float32 steps in two coordinates for a point where the kernel order and one other
    order of matcher_oracle.RANSAC_ORDERS decide differently, confirmed exactly (ransac_d2_exact).  The probes cycle through the three
    other orders and alternate between the kernel accepting and rejecting.  Returns {id: (a [3], b [3], the kernel's decision)}."""
    d2_max = F32(mo.sqrt_le_max(thresh))
    P64 = np.asarray(P, np.float32).astype(np.float64)
    Pl = [[float(v) for v in row] for row in np.asarray(P, np.float32)]
    out = {}
    for j, i in enumerate(probe_ids):
        other = mo.RANSAC_ORDERS[1 + j % 3]
        want_in = j % 2 == 0
        found = None
        while found is None:
            a = rng.uniform(-0.5, 0.5, size=3).astype(F32)
            al = [float(v) for v in a]
            u = rng.normal(size=3)
            u /= np.linalg.norm(u)
            b0 = (P64[:, :3] @ a.astype(np.float64) + P64[:, 3] + u * thresh).astype(F32)
            ms = {}
            for fused_m in (True, False):
                ms[fused_m] = [mo.f32_add(mo.f32_fma(r[2], al[2], mo.f32_fma(r[0], al[0], mo.f32_mul(r[1], al[1]))), r[3]) if fused_m else
                               mo.f32_add(mo.f32_add(mo.f32_add(mo.f32_mul(r[0], al[0]), mo.f32_mul(r[1], al[1])), mo.f32_mul(r[2], al[2])), r[3])
                               for r in Pl]
            ax0, ax1 = rng.choice(3, 2, replace=False)
            k = np.arange(-span, span + 1, dtype=np.float32)
            g0, g1 = np.meshgrid(b0[ax0] + k * np.spacing(b0[ax0]), b0[ax1] + k * np.spacing(b0[ax1]), indexing="ij")
            bb = [np.full(g0.shape, b0[c], F32) for c in range(3)]
            bb[ax0], bb[ax1] = g0.astype(F32), g1.astype(F32)
            kin = _d2_grid(ms[True], *bb, True) <= d2_max
            fm, fs = other in ("plain_squares",), other in ("plain_model",)
            oin = _d2_grid(ms[fm], *bb, fs) <= d2_max
            for c in np.argwhere((kin == want_in) & (oin != want_in))[:8]:
                b = np.array([bb[0][tuple(c)], bb[1][tuple(c)], bb[2][tuple(c)]], F32)
                ke = mo.ransac_d2_exact(P, a, b, "kernel") <= float(d2_max)
                if ke == want_in and (mo.ransac_d2_exact(P, a, b, other) <= float(d2_max)) != ke:
                    found = (a, b, ke)
                    break
        out[i] = found
    return out


# ---------------------------------------------------------------------------------------------------------------- 7. through the matcher chain
CHAIN_SHIFT = 32          # cluster 1's B pixel is its A pixel moved by 32 columns: at depth 0.75 and fx = 512 a translation of 0.046875 m
CHAIN_THRESH = 0.002      # the scene spans ~10 cm: a tighter threshold than THRESH keeps a model mixing both clusters from fitting either


def chain_rows(rng, n, specs, n_trials, tail=False):
    """Rows for corres_families.desc_pair (one-way rows, so RANSAC point i is row i) laid out like ties() or chunks(): specs [(trial, size)]
    as in _tie_case, cluster 0 under the identity (same pixel, same depth on both frames) and cluster 1 under a translation (B pixel
    CHAIN_SHIFT columns right of A's, both at depth 0.75; image rows 0-15, columns 0-31 for A).  Other rows are outliers, B between 0.5
    and 2 m behind A at random (multiples of 1/64, so every cloud point is exact on the device and in the oracle), so no three of them
    agree on a motion.
    tail=True: cluster 0's other members are drawn from the last 128 rows and cluster 1's from rows below 1024, as in chunks().
    Returns (rows, [(trial, members)])."""
    from . import corres_families as cf
    ids = sample_ids(n, n_trials)
    taken, got = set(), []
    for c, (T, k) in enumerate(specs):
        pool = (range(n - 128, n) if c == 0 else range(0, min(1024, n - 128))) if tail else range(n)
        while True:
            mem = grow_cluster(ids, T, k, pool, taken, rng)
            if mem is not None:
                break
            T += 1
            assert T < n_trials, (n, specs)
        taken |= set(mem)
        got.append((T, mem))
    member = {i: c for c, (_, mem) in enumerate(got) for i in mem}
    low = [(u, v) for v in range(16) for u in range(CHAIN_SHIFT) if (u, v) != cf.DEAD]
    high = [(u, v) for v in range(16, cf.H) for u in range(cf.W)]
    rng.shuffle(low)
    rng.shuffle(high)
    rows = []
    for i in range(n):
        c = member.get(i)
        if c == 1:
            u, v = low.pop()
            rows.append(("one", (u, v, 0.75), (u + CHAIN_SHIFT, v, 0.75)))
        else:
            u, v = high.pop()
            d = float((40 + rng.integers(0, 48)) / 64.0)
            rows.append(("one", (u, v, d), (u, v, d if c == 0 else d + 0.5 + float(rng.integers(0, 97)) / 64.0)))
    return rows, got


def chain_frames(seed=12):
    """The fused chain's two frame pairs: a tie (two clusters of 24, cluster 0's trial first) on 300 rows, non-neighbour ids 7 and 5, and a
    chunk layout (winner 40 with its other members in the last 128 rows, decoy 39 below row 1024) on 1100 rows, neighbour ids 7 and 6.
    Returns [(A, B, clusters)] with clusters as chain_rows gives them."""
    from . import corres_families as cf
    rng = np.random.default_rng(seed)
    out = []
    for p, (n, specs, tail) in enumerate(((300, [(0, 24), (5, 24)], False), (1100, [(0, 40), (0, 39)], True))):
        rows, clusters = chain_rows(rng, n, specs, MAX_TRIALS, tail)
        A, B = cf.desc_pair(rng, rows, 7, 5 + p)
        out.append((A, B, clusters))
    return out
