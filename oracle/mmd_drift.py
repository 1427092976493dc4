"""CPU oracle for the MMD drift test (TEST INFRASTRUCTURE): alibi-detect 0.12's ``MMDDrift`` (PyTorch backend) restated on an
explicit kernel matrix.  Small sizes only: it holds the (n_ref + m)^2 matrix.

What alibi-detect 0.12 does, restated from the published source (the package is not installed here, so parity is pinned to
this restatement and stated as unpinned against alibi-detect itself in DESIGN.md):

* ``GaussianRBF``: k(a, b) = exp(-d(a, b) / (2 sigma^2)), d the squared Euclidean distance.  alibi computes d as
  |a|^2 + |b|^2 - 2 a.b clamped at 1e-30; this restatement takes direct differences (the two differ in the last bits).
* ``sigma_median(x, y, dist)``: with x = y = x_ref (n rows) the n x n matrix ``dist`` is flattened, sorted, and
  sigma = sqrt(0.5 * sorted[n + (n^2 - n) // 2 - 1]).  The n diagonal zeros sort first and every pair appears twice, so the
  entry at n + 2q and n + 2q + 1 is the q-th smallest (0-based) of the P = n (n - 1) / 2 pair distances, and index
  n + P - 1 is pair q = floor((P - 1) / 2) (``median_pair_index``).
* ``score``: the kernel matrix of [x_ref; x] with a zeroed diagonal; ``mmd2_from_kernel_matrix``:
  mmd^2 = K_xx.sum() / (n (n - 1)) + K_yy.sum() / (m (m - 1)) - 2 K_xy.mean(), Y the last m rows of the (permuted) pool;
  p_val = mean(mmd^2 <= mmd^2_permuted); distance_threshold = the permuted statistics sorted descending at index
  int(p_val * B) (clamped to B - 1 here: alibi raises at p_val = 1).  alibi's permutations are ``torch.randperm`` of the
  pool and its permuted statistics float32; here they are given subsets (``subsets``) and float64.
"""

from __future__ import annotations

import numpy as np


def pairwise_sq(x: np.ndarray, y: np.ndarray, chunk: int = 256) -> np.ndarray:
    """float64 (len(x), len(y)) squared Euclidean distances by direct differences."""
    out = np.empty((len(x), len(y)), dtype=np.float64)
    for i in range(0, len(x), chunk):
        out[i:i + chunk] = ((x[i:i + chunk, None, :] - y[None, :, :]) ** 2).sum(axis=-1)
    return out


def median_pair_index(n: int) -> int:
    """The 0-based rank among the n (n - 1) / 2 pair distances of the entry ``sigma_median`` selects."""
    pairs = n * (n - 1) // 2
    return (pairs - 1) // 2


def sigma_median(x_ref: np.ndarray) -> float:
    """alibi's ``sigma_median(x_ref, x_ref, dist)`` on the flattened, sorted n x n distance matrix."""
    n = len(x_ref)
    dist = pairwise_sq(x_ref, x_ref)
    np.fill_diagonal(dist, 0.0)
    n_median = n + (n * n - n) // 2 - 1
    return float(np.sqrt(0.5 * np.sort(dist.ravel())[n_median]))


def kernel_matrix(pool: np.ndarray, sigma: float) -> np.ndarray:
    """The pool's kernel matrix with a zeroed diagonal."""
    k = np.exp(-pairwise_sq(pool, pool) / (2.0 * sigma * sigma))
    np.fill_diagonal(k, 0.0)
    return k


def mmd2_from_kernel_matrix(k: np.ndarray, y: np.ndarray) -> float:
    """``mmd2_from_kernel_matrix`` for the split whose batch side Y is the boolean mask ``y`` over the pool."""
    x = ~y
    n, m = int(x.sum()), int(y.sum())
    xf, yf = x.astype(np.float64), y.astype(np.float64)
    ky = k @ yf
    k_xx = xf @ (k @ xf)
    k_yy = yf @ ky
    k_xy = xf @ ky
    return k_xx / (n * (n - 1)) + k_yy / (m * (m - 1)) - 2.0 * k_xy / (n * m)


def mmd_drift(x_ref: np.ndarray, x: np.ndarray, subsets: np.ndarray, sigma: float | None = None, p_val: float = 0.05) -> dict:
    """``MMDDrift(x_ref, p_val=p_val, sigma=sigma).predict(x)["data"]`` with the permutations given as subsets of the pool
    [x_ref; x]: each the batch side of its split when len(x) <= len(x_ref), else the reference side.  Plus ``sigma`` and
    ``distance_permuted``."""
    n, m = len(x_ref), len(x)
    sigma = sigma_median(x_ref) if sigma is None else float(sigma)
    k = kernel_matrix(np.concatenate([x_ref, x]), sigma)
    y = np.zeros(n + m, dtype=bool)
    y[n:] = True
    mmd2 = mmd2_from_kernel_matrix(k, y)
    perm = np.empty(len(subsets), dtype=np.float64)
    for b, u in enumerate(subsets):
        side = np.zeros(n + m, dtype=bool)
        side[np.asarray(u)] = True
        perm[b] = mmd2_from_kernel_matrix(k, side if m <= n else ~side)
    pv = float(np.mean(mmd2 <= perm))
    idx = min(int(p_val * len(perm)), len(perm) - 1)
    return {"is_drift": int(pv < p_val), "distance": float(mmd2), "p_val": pv, "threshold": p_val,
            "distance_threshold": float(np.sort(perm)[::-1][idx]), "sigma": sigma, "distance_permuted": perm}
