"""NumPy restatement of model::SparsifiedGP::_sparsify (model/sparsified_gp.hpp:121-183).  TEST INFRASTRUCTURE ONLY.

While more than max_points points remain, remove the densest one: the point whose k = D nearest remaining neighbours have the
smallest sum of Euclidean distances, found by a strict < from DBL_MAX over the points in index order (lowest index on equal sums);
stop early when no sum is below DBL_MAX.  Distances round as the reference's squaredNorm()/norm() (s = 0; s += t*t per
dimension, then sqrt), and a sum adds the k smallest distances in ascending order from 0.0.

The reference re-sorts every row of an N x N matrix per removal (O(N^3)); here every point keeps its k nearest remaining
neighbours as (s, j) pairs in lexicographic order (s = squared distance).  Removing p only changes the lists that hold p: their
other k - 1 entries stay, and the smallest remaining pair above the old k-th pair completes them.  This is the algorithm of
limbo_b200/csrc/sparsify.cu, so N = 16384 -> 4096 takes about a minute instead of hours."""
from __future__ import annotations

import numpy as np

DBL_MAX = np.finfo(np.float64).max


def _dist2(X: np.ndarray, rows: np.ndarray) -> np.ndarray:
    """squared distances (len(rows) x N), summed over the dimensions in order from 0.0 with every operation rounded"""
    s = np.zeros((len(rows), X.shape[0]))
    for d in range(X.shape[1]):
        t = X[rows, d][:, None] - X[None, :, d]
        s = s + t * t
    return s


def _scores(nbr_s: np.ndarray) -> np.ndarray:
    sc = np.zeros(nbr_s.shape[0])
    for i in range(nbr_s.shape[1]):
        sc = sc + np.sqrt(nbr_s[:, i])
    return sc


def sparsify(X, max_points: int):
    """Returns (kept, removed, removed_score): the kept indices (ascending), the removal order and the sum each removed point had
    when it was chosen."""
    X = np.ascontiguousarray(X, dtype=np.float64)
    if X.ndim == 1:
        X = X[:, None]
    N, D = X.shape
    k = D
    if N <= max_points:
        return np.arange(N), np.zeros(0, dtype=np.int64), np.zeros(0)
    assert max_points >= k and np.isfinite(X).all()
    idx = np.arange(N)
    nbr_s = np.empty((N, k))
    nbr_j = np.empty((N, k), dtype=np.int64)
    for r0 in range(0, N, 512):
        rows = idx[r0:r0 + 512]
        s = _dist2(X, rows)
        s[np.arange(len(rows)), rows] = np.inf
        order = np.lexsort((np.broadcast_to(idx, s.shape), s), axis=1)[:, :k] if N <= 4096 else None
        if order is None:  # k smallest by (s, j): everything below the k-th value, then the lowest indices at the k-th value
            kth = np.partition(s, k - 1, axis=1)[:, k - 1]
            order = np.empty((len(rows), k), dtype=np.int64)
            for a in range(len(rows)):
                c = np.flatnonzero(s[a] <= kth[a])
                c = c[np.lexsort((c, s[a, c]))][:k]
                order[a] = c
        nbr_j[rows] = order
        nbr_s[rows] = np.take_along_axis(s, order, axis=1)
    score = _scores(nbr_s)
    alive = np.ones(N, dtype=bool)
    removed, removed_score = [], []
    n = N
    while n > max_points:
        cand = np.where(alive, score, np.inf)
        p = int(np.argmin(cand))  # first index of the minimum
        if not cand[p] < DBL_MAX:
            break
        removed.append(p)
        removed_score.append(float(score[p]))
        alive[p] = False
        n -= 1
        rows = np.flatnonzero(alive & (nbr_j == p).any(axis=1))
        if len(rows):
            s = _dist2(X, rows)
            thr_s, thr_j = nbr_s[rows, k - 1][:, None], nbr_j[rows, k - 1][:, None]
            ok = alive[None, :] & (idx[None, :] != rows[:, None]) & ((s > thr_s) | ((s == thr_s) & (idx[None, :] > thr_j)))
            s = np.where(ok, s, np.inf)
            for a, r in enumerate(rows):
                keep = nbr_j[r] != p
                if ok[a].any():
                    m = s[a].min()
                    j = int(np.flatnonzero(ok[a] & (s[a] == m))[0])
                    new_s, new_j = m, j
                else:
                    new_s, new_j = np.inf, -1
                nbr_s[r] = np.append(nbr_s[r][keep], new_s)
                nbr_j[r] = np.append(nbr_j[r][keep], new_j)
            score[rows] = _scores(nbr_s[rows])
    return np.flatnonzero(alive), np.array(removed, dtype=np.int64), np.array(removed_score)
