"""Oracle of the online MMD drift detector (TEST INFRASTRUCTURE, no GPU): alibi-detect 0.12's ``MMDDriftOnline`` (PyTorch
backend: ``_configure_thresholds``, ``_configure_ref_subset``, ``score``, ``get_threshold``) restated literally in numpy on
an explicit reference kernel matrix, with numpy's draws in place of torch's (``mmd_online.py``).

The space is the MMD test's: ``kernel(za, ca, zb, cb)`` = exp(-d / (2 sigma^2)) on K9's embedding (``mmd_walk.embed``).
alibi-detect is not installed here, so this is pinned to the restatement, not to alibi-detect itself.
"""

from __future__ import annotations

import numpy as np

import mmd_walk


def zero_diag(k: np.ndarray) -> np.ndarray:
    return k - np.diag(np.diag(k))


def quantile(sample: np.ndarray, p: float) -> float:
    """alibi's ``quantile(sample, p, type=7)``: the linear interpolation of the sorted sample at (n - 1) p."""
    s = np.sort(np.asarray(sample, dtype=np.float64))
    h = (len(s) - 1) * p
    lo = int(np.floor(h))
    hi = min(lo + 1, len(s) - 1)
    return float(s[lo] + (h - lo) * (s[hi] - s[lo]))


class OnlineOracle:
    def __init__(self, z, c, sigma: float, ert: float, window_size: int, n_bootstraps: int, random_state: int):
        self.z, self.c = z, c
        self.coef = 1.0 / (2.0 * sigma * sigma)
        self.n = len(z)
        self.ert, self.window_size, self.n_bootstraps = ert, window_size, n_bootstraps
        self.rng = np.random.default_rng(random_state)
        self.k_xx = self.kernel(z, c, z, c)
        self._configure_thresholds()
        self._configure_ref_subset()

    def kernel(self, za, ca, zb, cb) -> np.ndarray:
        return np.exp(-mmd_walk.dists(za, ca, zb, cb) * self.coef)

    def _configure_thresholds(self):
        W = self.window_size
        etw_size = 2 * W - 1
        rw_size = self.n - etw_size
        perms = [self.rng.permutation(self.n) for _ in range(self.n_bootstraps)]
        p_inds_all = [perm[:-etw_size] for perm in perms]
        q_inds_all = [perm[-etw_size:] for perm in perms]
        k_xy_col_sums_all = [self.k_xx[p_inds][:, q_inds].sum(0) for p_inds, q_inds in zip(p_inds_all, q_inds_all)]
        k_full_sum = zero_diag(self.k_xx).sum()
        k_xx_sums_all = [(k_full_sum - zero_diag(self.k_xx[q_inds][:, q_inds]).sum() - 2 * k_xy_col_sums.sum()) / (rw_size * (rw_size - 1))
                         for q_inds, k_xy_col_sums in zip(q_inds_all, k_xy_col_sums_all)]
        k_xy_col_sums_all = [k_xy_col_sums / (rw_size * W) for k_xy_col_sums in k_xy_col_sums_all]
        mmd_s_all = np.empty((W, self.n_bootstraps))
        for b, (q_inds, k_xx_sum, col) in enumerate(zip(q_inds_all, k_xx_sums_all, k_xy_col_sums_all)):
            k_yy = self.k_xx[q_inds][:, q_inds]
            for w in range(W):
                k_yy_sum = zero_diag(k_yy[w:w + W, w:w + W]).sum() / (W * (W - 1))
                mmd_s_all[w, b] = k_xx_sum + k_yy_sum - 2 * col[w:w + W].sum()
        self.bootstrap_stats = mmd_s_all.T.copy()  # (n_bootstraps, W), as the device gives them
        self.bootstrap_q = np.array(q_inds_all)
        bootstrap_stats = mmd_s_all
        thresholds = []
        p = 1 / self.ert
        for w in range(W):
            if bootstrap_stats.shape[1] == 0:
                raise ValueError(f"no bootstrap stream is left at window position {w}")
            thresholds.append(quantile(bootstrap_stats[w], 1 - p))
            bootstrap_stats = bootstrap_stats[:, bootstrap_stats[w] < thresholds[-1]]
        self.thresholds = np.array(thresholds)

    def _configure_ref_subset(self, max_attempts: int = 100):
        W = self.window_size
        etw_size = 2 * W - 1
        rw_size = self.n - etw_size
        mmd_init = None
        self.split_attempts = 0
        while mmd_init is None or mmd_init >= self.get_threshold(0):
            if self.split_attempts == max_attempts:
                raise ValueError(f"{max_attempts} splits all start in detection")
            self.split_attempts += 1
            perm = self.rng.permutation(self.n)
            self.perm = perm
            self.ref_inds, self.init_test_inds = perm[:rw_size], perm[-W:]
            self.k_xx_sub = self.k_xx[self.ref_inds][:, self.ref_inds]
            self.k_xx_sub_sum = zero_diag(self.k_xx_sub).sum() / (rw_size * (rw_size - 1))
            self.k_xy_col_sums = self.k_xx[self.ref_inds][:, self.init_test_inds].sum(0)
            k_yy = self.k_xx[self.init_test_inds][:, self.init_test_inds]
            mmd_init = (self.k_xx_sub_sum + zero_diag(k_yy).sum() / (W * (W - 1)) - 2 * self.k_xy_col_sums.sum() / (W * rw_size))
        self.initial_stat = mmd_init
        self.reset_state()

    def reset_state(self):
        self.t = 0
        self.test_z = self.z[self.init_test_inds]
        self.test_c = self.c[self.init_test_inds]
        self.k_xy = self.k_xx[self.ref_inds][:, self.init_test_inds]

    def get_threshold(self, t: int) -> float:
        return self.thresholds[t] if t < self.window_size else self.thresholds[-1]

    def score(self, z_t, c_t) -> float:
        """One row: alibi's _update_state, then its score."""
        W = self.window_size
        self.t += 1
        kernel_col = self.kernel(self.z[self.ref_inds], self.c[self.ref_inds], z_t[None], c_t[None])
        self.test_z = np.concatenate([self.test_z[1 - W:], z_t[None]], 0)
        self.test_c = np.concatenate([self.test_c[1 - W:], c_t[None]], 0)
        self.k_xy = np.concatenate([self.k_xy[:, 1 - W:], kernel_col], 1)
        k_yy = self.kernel(self.test_z, self.test_c, self.test_z, self.test_c)
        return float(self.k_xx_sub_sum + zero_diag(k_yy).sum() / (W * (W - 1)) - 2 * self.k_xy.mean())

    def predict(self, z_t, c_t) -> dict:
        stat = self.score(z_t, c_t)
        threshold = self.get_threshold(self.t)
        return {"is_drift": int(stat > threshold), "time": self.t, "test_stat": stat, "threshold": threshold}
