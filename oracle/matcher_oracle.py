"""oracle/matcher_oracle.py — TEST INFRASTRUCTURE ONLY.

CPU restatement of the matcher half of the hot path (SURVEY.md §8a a15-a18):
  * knn()            what the two cv::cuda::DescriptorMatcher::knnMatch(…, k=5) calls in SiftManager::findCorresbyNN
                     (/root/reference/src/FeatureManager.cpp:271-273) return: for every query row the k train rows of
                     smallest L2 distance, ascending, DMatch.distance = sqrt(sum (a-b)^2).  The arithmetic lives in
                     OpenCV's cudafeatures2d brute-force matcher, which is NOT under /root/reference and whose version the
                     reference never pins (CMakeLists.txt:23 `find_package(OpenCV REQUIRED)`); there are no reference
                     tests at that boundary => parity unpinned by the reference.  We define it as EXACT brute force:
                     distances accumulated in float64 from the float32 inputs, ties -> lower train index, and cross-check
                     against OpenCV's CPU BFMatcher (the reference's own NO_OPENCV_CUDA path, FeatureManager.cpp:266-269).
  * prune_matches()  SiftManager::pruneMatches (FeatureManager.cpp:290-336)
  * collect_mutual() SiftManager::collectMutualMatches (:338-368) — a UNION, duplicates kept (SURVEY.md D1)
"""
from __future__ import annotations

import numpy as np


def _d2_direct(qrow: np.ndarray, t: np.ndarray) -> np.ndarray:
    """float64 sum of (q - t)^2 over the last axis: the distance both knn() and knn_direct() order by, computed alike."""
    diff = qrow[None, :] - t
    return (diff * diff).sum(1)


def _top_k(c: np.ndarray, dd: np.ndarray, kk: int, idx_row: np.ndarray, dist_row: np.ndarray):
    order = np.lexsort((c, dd))[:kk]
    idx_row[:kk] = c[order]
    dist_row[:kk] = np.sqrt(dd[order]).astype(np.float32)


def knn(query: np.ndarray, train: np.ndarray, k: int = 5, block: int = 512):
    """Exact kNN.  Returns (idx [nq,k] int32, dist [nq,k] float32); rows with fewer than k candidates pad with -1/inf.

    The float64 expansion |q|^2 + |t|^2 - 2 q.t only preselects: it cancels when descriptors share a large offset (|q|, |t| >> |q - t|).
    Whatever the summation order, its error is below (dim + 2) 2^-53 (|q| + |t|)^2 (norms and dot product each to dim 2^-53 of their
    magnitude, plus the two additions); `margin` is four times that for the row's largest train norm.  The k rows of smallest expanded d2
    have exact d2 <= kth + margin, so every row whose exact d2 is at most that has expanded d2 <= kth + 2 margin: those rows are
    recomputed by direct differences and ordered by (d2, index), as knn_direct() orders all of them."""
    q = np.asarray(query, np.float32)
    t = np.asarray(train, np.float32).astype(np.float64)
    nq, nt = q.shape[0], t.shape[0]
    idx = np.full((nq, k), -1, np.int32)
    dist = np.full((nq, k), np.inf, np.float32)
    if nq == 0 or nt == 0:
        return idx, dist
    tn = (t * t).sum(1)
    tmax = np.sqrt(tn.max())
    kk = min(k, nt)
    for s in range(0, nq, block):
        qb = q[s:s + block].astype(np.float64)
        qn = (qb * qb).sum(1)
        d2 = qn[:, None] + tn[None, :] - 2.0 * (qb @ t.T)
        kth = np.partition(d2, kk - 1, axis=1)[:, kk - 1]
        margin = 4.0 * 2.0 ** -53 * (q.shape[1] + 2) * (np.sqrt(qn) + tmax) ** 2
        keep = d2 <= (kth + 2.0 * margin)[:, None]
        for r in range(qb.shape[0]):
            c = np.nonzero(keep[r])[0]
            _top_k(c, _d2_direct(qb[r], t[c]), kk, idx[s + r], dist[s + r])
    return idx, dist


def knn_direct(query: np.ndarray, train: np.ndarray, k: int = 5):
    """Plain brute force: direct-difference float64 d2 to every train row, top k by (d2, index).  Slow; the check on knn()."""
    q = np.asarray(query, np.float32).astype(np.float64)
    t = np.asarray(train, np.float32).astype(np.float64)
    nq, nt = q.shape[0], t.shape[0]
    idx = np.full((nq, k), -1, np.int32)
    dist = np.full((nq, k), np.inf, np.float32)
    all_rows = np.arange(nt)
    for r in range(nq if nt else 0):
        _top_k(all_rows, _d2_direct(q[r], t), min(k, nt), idx[r], dist[r])
    return idx, dist


def knn_cv2(query, train, k=5):
    """OpenCV CPU brute force (the reference's NO_OPENCV_CUDA=1 path) — used as a cross-check and as the timed CPU baseline."""
    import cv2
    m = cv2.BFMatcher(cv2.NORM_L2).knnMatch(np.ascontiguousarray(query, np.float32), np.ascontiguousarray(train, np.float32), k=k)
    idx = np.full((len(m), k), -1, np.int32)
    dist = np.full((len(m), k), np.inf, np.float32)
    for r, row in enumerate(m):
        for c, dm in enumerate(row):
            idx[r, c] = dm.trainIdx
            dist[r, c] = dm.distance
    return idx, dist


# ---------------------------------------------------------------------------------------------------------------------
def ransac_pair(A, B, u3, dist_thresh):
    """Restatement of ransacMultiPairGPU for ONE pair (/root/reference/src/cuda/cuda_ransac.cu:1145-1217,1293-1302).
    A, B: [n,3] model-frame points; u3: [n_trials,3] the uniforms curand_uniform() yields after curand_init(0, trial, 0)
    (XORWOW; taken from tests/golden/curand_xorwow_seed0.npy, generated with the same curand call).
    Rigid fit = least-squares rotation (Kabsch, float64 SVD) — the reference uses an approximate fp32 SVD of the same
    3x3 matrix.  Winner = max inlier count, ties -> lowest trial id (the reference's arg-max is racy, SURVEY.md Q8).
    Returns (inlier ids ascending, best trial id, per-trial counts)."""
    A = np.asarray(A, np.float64)[:, :3]
    B = np.asarray(B, np.float64)[:, :3]
    n = A.shape[0]
    T = u3.shape[0]
    counts = np.zeros(T, np.int64)
    poses = [None] * T
    if n >= 3:
        # round half away from zero like CUDA roundf
        ids = np.floor(np.asarray(u3, np.float32) * np.float32(n - 1) + np.float32(0.5)).astype(np.int64)
        for t in range(T):
            i0, i1, i2 = ids[t]
            if i0 == i1 or i1 == i2 or i0 == i2:
                continue
            s, d = A[[i0, i1, i2]], B[[i0, i1, i2]]
            sm, dm = s.mean(0), d.mean(0)
            S = (s - sm).T @ (d - dm)                      # S[a][b] = sum src_a dst_b
            U, _, Vt = np.linalg.svd(S)
            R = Vt.T @ U.T
            if np.linalg.det(R) < 0:
                Vt[2] *= -1
                R = Vt.T @ U.T
            tt = dm - R @ sm
            poses[t] = (R, tt)
            dist = np.linalg.norm(B - (A @ R.T + tt), axis=1)
            counts[t] = int((dist <= dist_thresh).sum())
    best = int(np.argmax(counts)) if counts.max() > 0 else -1      # argmax returns the first (lowest) index on ties
    if best < 0:
        return np.zeros(0, np.int32), -1, counts
    R, tt = poses[best]
    dist = np.linalg.norm(B - (A @ R.T + tt), axis=1)
    return np.nonzero(dist <= dist_thresh)[0].astype(np.int32), best, counts


# ---------------------------------------------------------------------------------------------------------------------
def _cloud_point(depth, K, u, v):
    """Frame::depthToCloudAndNormals (/root/reference/src/Frame.cpp:199-233): K^-1 (u d, v d, d), zeros when d < 0.1."""
    fx, fy, cx, cy = [np.float32(x) for x in K]
    d = np.float32(depth[v, u])
    if d < np.float32(0.1):
        return np.zeros(3, np.float32)
    ifx, ify, icx, icy = np.float32(1) / fx, np.float32(1) / fy, -cx / fx, -cy / fy
    return np.array([ifx * (np.float32(u) * d) + icx * d, ify * (np.float32(v) * d) + icy * d, d], np.float32)


def _round_half_away(x):
    return int(np.floor(abs(float(x)) + 0.5) * (1 if x >= 0 else -1))


def prune_matches(Q, T, knn_idx, K, max_dist, cos_max):
    """SiftManager::pruneMatches (/root/reference/src/FeatureManager.cpp:290-336) for one direction.
    Q, T: dicts with kpts [n,2], depth [H,W], normal [H,W,4], pose [4,4].  Returns list of (q, t, ptQ_cam, ptT_cam)."""
    H, W = Q["depth"].shape
    out = []
    Rq, tq = Q["pose"][:3, :3].astype(np.float32), Q["pose"][:3, 3].astype(np.float32)
    Rt, tt = T["pose"][:3, :3].astype(np.float32), T["pose"][:3, 3].astype(np.float32)
    for q in range(len(Q["kpts"])):
        for t in knn_idx[q]:
            if t < 0:
                continue
            uq, vq = _round_half_away(Q["kpts"][q, 0]), _round_half_away(Q["kpts"][q, 1])
            ut, vt = _round_half_away(T["kpts"][t, 0]), _round_half_away(T["kpts"][t, 1])
            if not (0 <= uq < W and 0 <= vq < H and 0 <= ut < W and 0 <= vt < H):
                continue
            pq, pt = _cloud_point(Q["depth"], K, uq, vq), _cloud_point(T["depth"], K, ut, vt)
            if pq[2] < 0.1 or pt[2] < 0.1:
                continue
            mq, mt = Rq @ pq + tq, Rt @ pt + tt
            nq, nt = Rq @ Q["normal"][vq, uq, :3], Rt @ T["normal"][vt, ut, :3]
            dist = np.float32(np.linalg.norm((mq - mt).astype(np.float32)))
            with np.errstate(invalid="ignore", divide="ignore"):
                dotn = np.float32(np.dot(nq / np.float32(np.linalg.norm(nq)), nt / np.float32(np.linalg.norm(nt))))
            if dist > max_dist or dotn < cos_max:      # NaN dot (zero normal) does NOT reject (FeatureManager.cpp:326)
                continue
            out.append((q, int(t), pq, pt))
            break
    return out


def collect_mutual(A, B, mAB, mBA):
    """SiftManager::collectMutualMatches (:338-368): A->B survivors then B->A survivors, duplicates kept.
    Rows: [uA, vA, uB, vB, ptA_cam(3), ptB_cam(3)]."""
    rows = []
    for (q, t, pq, pt) in mAB:
        rows.append(np.concatenate([A["kpts"][q], B["kpts"][t], pq, pt]))
    for (q, t, pq, pt) in mBA:
        rows.append(np.concatenate([A["kpts"][t], B["kpts"][q], pt, pq]))
    return np.asarray(rows, np.float32).reshape(-1, 10)


def find_corres(A, B, K, prune, u3, ransac_inlier_dist, k=5, propagated=None):
    """findCorresbyNN [+ findCorresByMapPoints for a non-neighbour pair] + runRansacBetween for one pair (A newer).
    prune = (max_dist_nn, cos_nn, max_dist_n, cos_n).  propagated: [m,4] (uA,vA,uB,vB) of the map points both frames observe, in
    the order SiftManager::findCorresByMapPoints walks them (/root/reference/src/FeatureManager.cpp:489-520): appended unless an
    existing match has the same (uA,vA) or (uB,vB), with the organised-cloud points at round(u), round(v).
    Returns (mutual rows incl. the appended ones, inlier row ids or None if the pair was dropped)."""
    iAB, _ = knn(A["desc"], B["desc"], k)
    iBA, _ = knn(B["desc"], A["desc"], k)
    neighbor = abs(A["id"] - B["id"]) == 1
    max_dist, cos_max = (prune[2], prune[3]) if neighbor else (prune[0], prune[1])
    rows = collect_mutual(A, B, prune_matches(A, B, iAB, K, max_dist, cos_max), prune_matches(B, A, iBA, K, max_dist, cos_max))
    if propagated is not None and not neighbor and len(propagated):
        H, W = A["depth"].shape
        extra = []
        for uA, vA, uB, vB in np.asarray(propagated, np.float32):
            if len(rows) and (((rows[:, 0] == uA) & (rows[:, 1] == vA)) | ((rows[:, 2] == uB) & (rows[:, 3] == vB))).any():
                continue
            ua, va, ub, vb = _round_half_away(uA), _round_half_away(vA), _round_half_away(uB), _round_half_away(vB)
            pa = _cloud_point(A["depth"], K, ua, va) if (0 <= ua < W and 0 <= va < H) else np.zeros(3, np.float32)
            pb = _cloud_point(B["depth"], K, ub, vb) if (0 <= ub < W and 0 <= vb < H) else np.zeros(3, np.float32)
            extra.append(np.concatenate([[uA, vA, uB, vB], pa, pb]).astype(np.float32))
        if extra:
            rows = np.concatenate([rows.reshape(-1, 10), np.asarray(extra, np.float32)], 0)
    if len(rows) <= 5:
        return rows, None
    PA = rows[:, 4:7] @ A["pose"][:3, :3].T.astype(np.float32) + A["pose"][:3, 3].astype(np.float32)
    PB = rows[:, 7:10] @ B["pose"][:3, :3].T.astype(np.float32) + B["pose"][:3, 3].astype(np.float32)
    ids, best, counts = ransac_pair(PA, PB, u3, ransac_inlier_dist)
    if len(ids) < 5:
        return rows, None
    return rows, ids
