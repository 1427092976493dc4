"""Chunked numpy emulator of the k-nearest reference search behind trust scores (TEST INFRASTRUCTURE, no GPU): what
``csrc/knn.cuh`` computes, at the sizes of the full training split.

* the space is the MMD test's: ``mmd_walk.embed`` with the trust reference's constants, and ``mmd_walk.dists`` for the squared
  distances (bit-identical to the kernels'); a NaN distance counts as +inf;
* per class, the reference rows of that class in their original order; per query row the k smallest (d, index) pairs in
  lexicographic order, so a tie goes to the lower index;
* the answer is the correctly rounded sqrt of d and the original row index, laid out (n, 2, k) as ``b2f_knn``'s.
"""

from __future__ import annotations

import numpy as np

import mmd_walk


def embedding(rows_ref: np.ndarray, n_cat: int, n_num: int, impute):
    """-> (mean, scale, embed): the trust reference's z-score constants and a function embedding encoded rows with them."""
    from databricks_kubernetes_mlops_poc_b200 import mmd

    mean, scale = mmd.standardization(mmd.numerics(rows_ref, n_cat, n_num, impute))
    return mean, scale, lambda rows: mmd_walk.embed(rows, n_cat, n_num, impute, mean, scale)


def topk(d: np.ndarray, k: int) -> np.ndarray:
    """(m, n) distances -> (m, k) column indices of the k smallest (d, column) pairs per row, in that order."""
    kth = np.partition(d, k - 1, axis=1)[:, k - 1]
    out = np.empty((len(d), k), dtype=np.int64)
    for r in range(len(d)):
        cand = np.nonzero(d[r] <= kth[r])[0]  # ascending columns: a stable sort keeps ties in index order
        out[r] = cand[np.argsort(d[r, cand], kind="stable")[:k]]
    return out


def neighbours(zq, cq, zr, cr, cls, k: int, chunk: int = 1024):
    """Query embedding (zq, cq), reference embedding (zr, cr) with classes ``cls`` -> (float64 (n, 2, k) distances, int64
    (n, 2, k) reference row indices)."""
    n = len(zq)
    dist = np.empty((n, 2, k), dtype=np.float64)
    index = np.empty((n, 2, k), dtype=np.int64)
    for c in (0, 1):
        ref = np.nonzero(np.asarray(cls) == c)[0]
        for i0 in range(0, n, chunk):
            d = mmd_walk.dists(zq[i0:i0 + chunk], cq[i0:i0 + chunk], zr[ref], cr[ref])
            d[np.isnan(d)] = np.inf
            top = topk(d, k)
            dist[i0:i0 + chunk, c] = np.sqrt(np.take_along_axis(d, top, axis=1))
            index[i0:i0 + chunk, c] = ref[top]
    return dist, index
