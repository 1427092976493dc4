"""Chunked numpy emulator of the MMD drift test's algebraic form (TEST INFRASTRUCTURE, no GPU): what
``csrc/mmd_drift.cuh`` computes, at sizes up to the full curated table, without an explicit kernel matrix.

* ``embed``: encoded rows -> (z float64 (N, n_num), codes int32 (N, n_cat)), as ``k_mmd_embed``.
* ``dists``: the squared distances with the device's arithmetic (numerics in field order as d + x * x, the integer
  categorical cost last), so they are bit-identical to the kernels'.
* ``rank_counts``: how many reference pairs lie below a distance, and those near it, by chunked counting (the full table
  has 4.5e8 pairs: no np.partition).
* ``calibration_frames``: the curated-table split of the calibration (a quiet held-out slice and its joint shift).
* ``statistics``: pool row sums r, T, and per subset the pair sum inside it -> the same mmd^2 algebra as ``k_mmd_finish``,
  with the magnitude of its three terms (mmd^2 is a difference of near-equal terms).
"""

from __future__ import annotations

import numpy as np

from databricks_kubernetes_mlops_poc_b200 import mmd


def embed(rows: np.ndarray, n_cat: int, n_num: int, impute, mean, scale):
    z = (mmd.numerics(rows, n_cat, n_num, impute) - np.asarray(mean, dtype=np.float64)) / np.asarray(scale, dtype=np.float64)
    return z, rows[:, :n_cat].view(np.int32).copy()


def dists(za, ca, zb, cb) -> np.ndarray:
    d = np.zeros((len(za), len(zb)), dtype=np.float64)
    for f in range(za.shape[1]):
        x = za[:, None, f] - zb[None, :, f]
        d = d + x * x
    cost = np.zeros(d.shape, dtype=np.int64)
    for f in range(ca.shape[1]):
        a, b = ca[:, None, f], cb[None, :, f]
        cost += np.where(a == b, 0, np.where((a < 0) | (b < 0), 1, 2))
    return d + cost


def rank_counts(z, c, lo: float, hi: float, chunk: int = 1024) -> tuple[int, np.ndarray]:
    """Over the pairs i < j of the rows: (how many distances lie below lo, the sorted distances in [lo, hi])."""
    below, near = 0, []
    n = len(z)
    for i0 in range(0, n, chunk):
        i1 = min(n, i0 + chunk)
        d = dists(z[i0:i1], c[i0:i1], z[i0:], c[i0:])
        keep = np.arange(i0, i1)[:, None] < np.arange(i0, n)[None, :]
        below += int(((d < lo) & keep).sum())
        near.append(d[keep & (d >= lo) & (d <= hi)])
    return below, np.sort(np.concatenate(near))


def median_pair(z, c) -> float:
    """The floor((P - 1) / 2)-th smallest pair distance (small n: the pairs are materialised)."""
    d = dists(z, c, z, c)
    pairs = d[np.triu_indices(len(z), 1)]
    k = (len(pairs) - 1) // 2
    return float(np.partition(pairs, k)[k])


def sigma(z, c) -> float:
    return float(np.sqrt(0.5 * median_pair(z, c)))


def row_sums(za, ca, zb, cb, coef: float, same: bool, chunk: int = 512) -> np.ndarray:
    """r[a] = sum over b of k(a, b), b != a when ``same`` (A and B are the same rows)."""
    r = np.empty(len(za), dtype=np.float64)
    for i0 in range(0, len(za), chunk):
        k = np.exp(-dists(za[i0:i0 + chunk], ca[i0:i0 + chunk], zb, cb) * coef)
        if same:
            idx = np.arange(i0, min(len(za), i0 + chunk))
            k[idx - i0, idx] = 0.0
        r[i0:i0 + chunk] = k.sum(axis=1)
    return r


def statistics(zr, cr, zb, cb, subsets: np.ndarray, sigma_: float):
    """-> (mmd2 (1 + B,), terms (1 + B,)): entry 0 the observed split, then one per subset; terms = |S_xx| / (n (n - 1)) +
    |S_yy| / (m (m - 1)) + 2 |S_xy| / (n m)."""
    n, m = len(zr), len(zb)
    coef = 1.0 / (2.0 * sigma_ * sigma_)
    z, c = np.concatenate([zr, zb]), np.concatenate([cr, cb])
    r = row_sums(z, c, z, c, coef, True)
    total = r.sum()
    u_is_batch = m <= n
    obs = np.arange(n, n + m) if u_is_batch else np.arange(n)
    mmd2, terms = [], []
    for u in [obs, *subsets]:
        u = np.asarray(u)
        k = np.exp(-dists(z[u], c[u], z[u], c[u]) * coef)
        np.fill_diagonal(k, 0.0)
        s_uu = k.sum()
        s_uv = r[u].sum() - s_uu
        s_vv = total - s_uu - 2.0 * s_uv
        s_xx, s_yy = (s_vv, s_uu) if u_is_batch else (s_uu, s_vv)
        a, b, x = s_xx / (n * (n - 1)), s_yy / (m * (m - 1)), 2.0 * s_uv / (n * m)
        mmd2.append(a + b - x)
        terms.append(abs(a) + abs(b) + abs(x))
    return np.array(mmd2), np.array(terms)


def calibration_frames(curated):
    """(reference 5 000 rows, held-out 500 rows, the held-out rows with each column shuffled on its own) of the curated table,
    a random split on which K3's per-field tests see no drift: the shuffle keeps every marginal and destroys the joint."""
    from oracle import reference_pipeline as rp

    order = np.random.default_rng(3).permutation(len(curated))
    ref = curated[rp.FEATURES].iloc[order[:5000]].reset_index(drop=True)
    held = curated[rp.FEATURES].iloc[order[5000:5500]].reset_index(drop=True)
    rng = np.random.default_rng(1)
    shuffled = held.copy()
    for c in shuffled.columns:
        shuffled[c] = shuffled[c].to_numpy()[rng.permutation(len(shuffled))]
    return ref, held, shuffled
