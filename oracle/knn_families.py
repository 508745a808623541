"""Descriptor sets built against the kNN matcher's bound (knn.cu, k_knn_select): exact ties, near-ties below the fp16 key's resolution,
clusters placed against the 4-row group layout, fp16 flushing that makes the rows' rounding error the deciding term of the bound, and
fp16-exact rows on a large common offset.  Shared by the oracle's CPU tests and the matcher's GPU tests."""
import numpy as np

D = 256
GRID = 2.0 ** -6


def knn_unpos(p):
    """knn.cu's position -> row map: position p of a 128-row block belongs to group (p / 4) % 32; a group's four rows are one thread's."""
    return (p & ~127) + 16 * ((p >> 5) & 3) + ((p >> 2) & 7) + 8 * (p & 1) + 64 * ((p >> 1) & 1)


def group_rows(g):
    """The four rows of group g (groups counted from row 0, 32 per 128-row block)."""
    return [knn_unpos(4 * g + j) for j in range(4)]


def grid_rows(rng, n, lim=4.0):
    """Rows of multiples of 2^-6 in [-lim, lim]: exact in fp16, float32 and float64, and so is every d2 between them."""
    return rng.integers(-int(lim * 64), int(lim * 64) + 1, size=(n, D)) * GRID


def exact_ties(rng, q, m):
    """m rows at distance exactly 1 from q: q +- e_i over distinct i (q within [-3, 3] keeps them on the grid in [-4, 4])."""
    dims = rng.permutation(D)[:m]
    t = np.repeat(q[None, :], m, 0)
    t[np.arange(m), dims] += rng.choice([-1.0, 1.0], m)
    return t


def near_ties(rng, q, m):
    """t_j = q +- 2^-1 (1 + j 2^-20) e_{i_j}, j = 0..m-1 (ascending distance).  Neighbouring d2 differ by about 2^-19 relative, far
    below the 2^-11 resolution of a stored fp16 key and far above float64 noise.  With |q_i| <= 2 every component is a multiple of
    2^-21 below 4: exact in float32 (asserted by assert_dyadic)."""
    dims = rng.permutation(D)[:m]
    t = np.repeat(q[None, :], m, 0)
    t[np.arange(m), dims] += 0.5 * (1.0 + np.arange(m) * 2.0 ** -20) * rng.choice([-1.0, 1.0], m)
    return t


def assert_dyadic(a, b, frac_bits):
    """Every component is a float32 multiple of 2^-frac_bits and every d2 between the sets stays below 2^(53 - 2 frac_bits): then d2 is
    an integer multiple of 2^(-2 frac_bits) below 2^53 units, and so is every partial sum, so float64 gets it exactly in any order."""
    for x in (a, b):
        assert np.array_equal(x.astype(np.float32).astype(np.float64), x)
        assert np.array_equal(np.round(x * 2.0 ** frac_bits), x * 2.0 ** frac_bits)
    na = np.sqrt((a * a).sum(1)).max(initial=0.0)
    nb = np.sqrt((b * b).sum(1)).max(initial=0.0)
    assert (na + nb) ** 2 < 2.0 ** (53 - 2 * frac_bits)


def offset_set(rng, n, C, sigma, c):
    """C c + N(0, sigma): descriptors sharing a large common offset (c ~ N(0, 1): components of about C)."""
    return C * c[None, :] + rng.normal(0.0, sigma, (n, D))


# cluster placements against the group layout: the train rows that receive the m cluster members
PLACEMENTS = {
    "one_group": group_rows(5),                                        # 4 members, one group
    "spread12": [group_rows(3 * g)[g % 4] for g in range(12)],         # 12 members in 12 groups (fast path)
    "g16": [group_rows(2 * g)[g % 4] for g in range(16)],              # 16 members in 16 groups: both limits met exactly
    "g17": [group_rows(2 * g)[g % 4] for g in range(17)],              # 17 groups: the group list overflows
    "g5": sum((group_rows(g) for g in (3, 10, 17, 24)), []) + group_rows(40)[:1],   # 17 members in 5 groups: the candidate list overflows
    "edge127": list(range(124, 132)),                                  # across the 128-row A tile edge
    "edge255": list(range(252, 260)),                                  # across the 256-row B tile edge
}
FAST = {"one_group", "spread12", "edge127", "edge255", "g16"}           # within 16 groups and 16 candidates
OVERFLOW = {"g17", "g5"}
# Background sets of 1024 rows put every query, the constructed one among them, next to 1023 others in the tensor pass and the group
# minima; the fast-path and overflow assertions then run the constructed query alone on its side (see test_cluster_placement).
N_SET, Q_ROW = 1024, 37


def cluster_case(family, rows, seed):
    """(query set, train set): query row Q_ROW of a grid background, and its cluster of len(rows) exact ties (distance 1, grid in [-4, 4],
    dyadic with 6 fractional bits) or near-ties (grid in [-2, 2], 21 fractional bits) at train rows `rows`, nearest member at the
    HIGHEST row: distances ascend with falling index, so an index tie-break cannot pass by accident."""
    rng = np.random.default_rng(seed)
    lim = 2.0 if family == "near" else 4.0
    qs = grid_rows(rng, N_SET, lim)
    qs[Q_ROW] = grid_rows(rng, 1, min(lim, 3.0))[0]
    ts = grid_rows(rng, N_SET, lim)
    if len(rows):
        cl = (near_ties if family == "near" else exact_ties)(rng, qs[Q_ROW], len(rows))
        ts[sorted(rows, reverse=True)] = cl
    assert_dyadic(qs, ts, 21 if family == "near" else 6)
    return qs, ts


# fp16 flushes |x| < 2^-14 (6.1035e-5) to zero.  FLUSHED lies just below that, KEPT just above, 6.4 % apart.
FLUSHED, KEPT = 6.09e-5, 6.5e-5


def flush_case(sign=1.0):
    """(query set [1 row], train set [2 rows], index of the true nearest row): the rows' fp16 rounding error decides the answer.
    The query (every component FLUSHED) and the decoy (zeros) both round to the zero row, so the decoy's key is exactly 0.  The true
    nearest row (every component KEPT) is 16 (KEPT - FLUSHED) = 6.6e-5 from the query but 16 KEPT = 1.04e-3 from it after rounding.
    The query's rounding error e = 16 FLUSHED = 9.7e-4 is far larger than delta (the set norms are about 1e-3) and than the fp16 key
    rounding, so the threshold is T + e = sqrt(D2hi) + 2e ~ 1.96e-3: the true row is inside; with a single e (~9.9e-4) it would not be."""
    q = np.full((1, D), sign * FLUSHED)
    t = np.stack([np.full(D, sign * KEPT), np.zeros(D)])      # true nearest at row 0, decoy at row 1
    return q, t, 0


def offset_ladder_case(seed, n_rungs=24):
    """(query set, train set): fp16-exact rows on a common offset of 64 (components in [64, 71), multiples of 2^-4), where the fp32
    accumulation of the tensor pass works on norms of about 1.1e6 while the query's neighbours are 1 .. 6.25 away in d2.  Rungs
    t_j = q + (1 + j / 16) e_{i_j}, nearest at the highest row, then background rows about 700 away."""
    rng = np.random.default_rng(seed)
    base = lambda n: 64.0 + rng.integers(0, 64, size=(n, D)) / 16.0
    qs = base(64)
    ts = base(256)
    q = qs[Q_ROW]
    dims = rng.permutation(D)[:n_rungs]
    rungs = np.repeat(q[None, :], n_rungs, 0)
    rungs[np.arange(n_rungs), dims] += 1.0 + np.arange(n_rungs) / 16.0
    ts[np.arange(100, 100 + n_rungs)[::-1]] = rungs
    assert_dyadic(qs, ts, 4)
    return qs, ts
