"""Numpy emulator of the online MMD detector's device decomposition (TEST INFRASTRUCTURE, no GPU): what
``csrc/mmd_online.cuh`` computes, without a reference kernel matrix.

* reference row sums r (``mmd_walk.row_sums``) and T = sum r;
* a bootstrap y: q_s = the kernel sum of y_s over the rest of y, c_s = r_{y_s} - q_s, K_RR = T - 2 sum r_y + sum q;
* band prefixes P[L][s] = sum_{d = 1 .. L} k(x_s, x_{s-d}) (transposed, as on the device);
* a window starting at w: S_RW = sum c, S_WW = 2 sum_s P[s - w][s], stat = K_RR / (rw (rw - 1)) + S_WW / (W (W - 1)) -
  2 S_RW / (rw W);
* the stream: c of a row from its kernel sum against the sub-reference, the window state the last W - 1 rows.

``Emulator.configure`` runs the host's own draws, threshold loop and split loop (``mmd_online.py``) on it.
"""

from __future__ import annotations

import numpy as np

import mmd_walk
from databricks_kubernetes_mlops_poc_b200 import mmd_online


def pair_dists(za, ca, zb, cb) -> np.ndarray:
    """d(a_i, b_i) row by row, with mmd_walk.dists' arithmetic."""
    d = np.zeros(len(za), dtype=np.float64)
    for f in range(za.shape[1]):
        x = za[:, f] - zb[:, f]
        d = d + x * x
    cost = np.zeros(len(za), dtype=np.int64)
    for f in range(ca.shape[1]):
        a, b = ca[:, f], cb[:, f]
        cost += np.where(a == b, 0, np.where((a < 0) | (b < 0), 1, 2))
    return d + cost


def band(z, c, coef: float, W: int) -> np.ndarray:
    """float64 (W, n): P[L][s] for L <= min(s, W - 1), 0 elsewhere."""
    n = len(z)
    P = np.zeros((W, n), dtype=np.float64)
    for L in range(1, min(W, n)):
        k = np.exp(-pair_dists(z[L:], c[L:], z[:-L], c[:-L]) * coef)
        P[L, L:] = P[L - 1, L:] + k
    return P


def windows(cv, P, W: int, starts, k_rr: float, rw: int) -> np.ndarray:
    out = np.empty(len(starts), dtype=np.float64)
    for i, w in enumerate(starts):
        s_rw = cv[w:w + W].sum()
        s_ww = 2.0 * P[np.arange(W), w + np.arange(W)].sum()
        out[i] = k_rr / (rw * (rw - 1.0)) + s_ww / (W * (W - 1.0)) - 2.0 * s_rw / (rw * W)
    return out


class Emulator:
    def __init__(self, z, c, sigma: float):
        self.z, self.c = z, c
        self.n = len(z)
        self.coef = 1.0 / (2.0 * sigma * sigma)
        self.r = mmd_walk.row_sums(z, c, z, c, self.coef, True)
        self.total = self.r.sum()

    def bootstrap(self, etw: np.ndarray, W: int):
        """-> (stats (n_boot, W), K_RR (n_boot,)), as b2f_mmd_online_bootstrap."""
        etw = np.asarray(etw)
        rw = self.n - (2 * W - 1)
        stats = np.empty((len(etw), W))
        k_rr = np.empty(len(etw))
        for b, y in enumerate(etw):
            zy, cy = self.z[y], self.c[y]
            k = np.exp(-mmd_walk.dists(zy, cy, zy, cy) * self.coef)
            np.fill_diagonal(k, 0.0)
            q = k.sum(axis=1)
            cv = self.r[y] - q
            k_rr[b] = self.total - 2.0 * self.r[y].sum() + q.sum()
            stats[b] = windows(cv, band(zy, cy, self.coef, W), W, range(W), k_rr[b], rw)
        return stats, k_rr

    def configure(self, ert, window_size, n_bootstraps, random_state):
        """The host's configure on this emulator -> (thresholds, perm, attempts, bootstrap stats)."""
        ert, W, n_boot, random_state = mmd_online.check_config(self.n, ert, window_size, n_bootstraps, random_state)
        rng = np.random.default_rng(random_state)
        etw = mmd_online.draw_bootstraps(rng, self.n, W, n_boot)
        stats, _ = self.bootstrap(etw, W)
        thr = mmd_online.thresholds(stats, ert)
        perm, attempts = mmd_online.split(rng, self.n, W, thr, lambda y: self.bootstrap(y[None], W)[0][0, W - 1])
        self.set_split(perm, W)
        return thr, perm, attempts, stats

    def set_split(self, perm, W: int):
        """As b2f_mmd_online_configure."""
        self.W = W
        self.rw = self.n - (2 * W - 1)
        self.R = np.asarray(perm[:self.rw])
        self.k_rr = float(self.bootstrap(np.asarray(perm[self.rw:])[None], W)[1][0])
        init = np.asarray(perm[self.n - (W - 1):])
        self.init = (self.z[init], self.c[init], self.col(self.z[init], self.c[init]))
        self.reset()

    def col(self, z, c) -> np.ndarray:
        return mmd_walk.row_sums(z, c, self.z[self.R], self.c[self.R], self.coef, False)

    def reset(self):
        self.state = tuple(a.copy() for a in self.init)
        self.t = 0

    def push(self, z, c) -> np.ndarray:
        """-> the statistic of each pushed row's window, as b2f_mmd_online_push."""
        W = self.W
        cz, cc, ccv = self.state
        sz, sc = np.concatenate([cz, z]), np.concatenate([cc, c])
        scv = np.concatenate([ccv, self.col(z, c)])
        out = windows(scv, band(sz, sc, self.coef, W), W, range(len(z)), self.k_rr, self.rw)
        self.state = (sz[len(z):], sc[len(z):], scv[len(z):])
        self.t += len(z)
        return out
