"""CPU oracle for the batch drift scores (TEST INFRASTRUCTURE; SURVEY.md section 8a row a7, 8f rank 2).

Reference path: ``self.drift.predict(df[self.all_features].values)`` (``databricks/src/02-register-model.ipynb:338``)
on a detector built as ``TabularDrift(x_ref, p_val=0.05, categories_per_feature={0..8: None})`` (``:224-229``); the
response carries ``(1 - p_val).tolist()`` (``:345-349``).

The arithmetic lives in two un-vendored packages (SURVEY 8c): alibi-detect==0.12.0 (``app/requirements.txt:6``;
NOT installed, NOT in the reference checkout) and scipy (installed; it holds the numerics).  What alibi-detect
0.12.0's ``TabularDrift.feature_score`` does, restated from the published source:

* categorical feature f: the category set is the UNION of the values seen in the reference column and in the
  batch column; ``chi2_contingency`` on the 2 x K table of (reference counts, batch counts) over that set;
* numeric feature f: ``scipy.stats.ks_2samp(x_ref[:, f], x[:, f], alternative="two-sided", method="exact")``;
* p-values are stored in a float32 array.

``tabular_drift_p_values`` below is that restatement on top of the real scipy calls: it is the oracle the GPU path
(K3, ``csrc/drift_stats.cuh``) is checked against.  Parity status: pinned against scipy itself (every number here
comes out of the installed scipy), UNPINNED against alibi-detect (absent) -- stated in DESIGN.md.

The second half restates scipy's own exact two-sample K-S computation (``scipy/stats/_stats_py.py`` ``ks_2samp`` /
``_attempt_exact_2kssamp`` and the pythran kernel ``_compute_outer_prob_inside_method``, Hodges 1958 / Viehmann 2021)
in plain Python / numpy, in the integer form the GPU uses; tests pin it against the compiled scipy functions.
"""

from __future__ import annotations

import math

import numpy as np
import pandas as pd
from scipy import stats


# ----------------------------------------------------------------------------- the oracle proper (real scipy calls)
def tabular_drift_p_values(x_ref: pd.DataFrame, batch: pd.DataFrame, cat_features) -> np.ndarray:
    """float32 p-value per column of ``x_ref`` (alibi-detect 0.12.0 ``TabularDrift.feature_score``)."""
    cats = set(cat_features)
    p = np.zeros(len(x_ref.columns), dtype=np.float32)
    for i, name in enumerate(x_ref.columns):
        if name in cats:
            ref = x_ref[name].astype(str).to_numpy()
            x = batch[name].astype(str).to_numpy()
            union = sorted(set(ref.tolist()) | set(x.tolist()))
            table = np.array([[np.sum(ref == v) for v in union], [np.sum(x == v) for v in union]])
            p[i] = stats.chi2_contingency(table)[1]
        else:
            p[i] = stats.ks_2samp(x_ref[name].to_numpy(dtype=float), batch[name].to_numpy(dtype=float),
                                  alternative="two-sided", method="exact")[1]
    return p


def drift_scores(x_ref: pd.DataFrame, batch: pd.DataFrame, cat_features) -> list:
    """``(1 - p_val).tolist()`` in float32, as the response carries it (02-register-model.ipynb:345-349)."""
    return (np.float32(1) - tabular_drift_p_values(x_ref, batch, cat_features)).tolist()


# ----------------------------------------------------------------------------- restatement of scipy's exact K-S
def ks_numerator(ref_sorted: np.ndarray, x: np.ndarray) -> int:
    """max_t |n * #{ref <= t} - m * #{x <= t}| over the pooled sample points (m = len(ref), n = len(x)).

    ``D = numerator / (m * n)``.  scipy evaluates both right-continuous ECDFs at every pooled point
    (``ks_2samp``: ``cddiffs = cdf1 - cdf2``, ``d = max(maxS, clip(-minS, 0, 1))``)."""
    m, n = len(ref_sorted), len(x)
    pts = np.concatenate((ref_sorted, x))
    c1 = np.searchsorted(ref_sorted, pts, side="right").astype(np.int64)
    c2 = np.searchsorted(np.sort(x), pts, side="right").astype(np.int64)
    return int(np.abs(c1 * n - c2 * m).max())


def outer_prob_inside_method(m: int, n: int, g: int, h: int) -> float:
    """Proportion of lattice paths (0,0)->(m,n) that do NOT stay strictly inside |x/m - y/n| < h/lcm(m,n).

    Restates ``_compute_outer_prob_inside_method`` cell by cell in the form the GPU wavefront uses:
        P(i, j) = 1                              if |ng*i - mg*j| >= h          (outside the band)
                = 0                              if i == 0                      (inside, first column)
                = (P(i-1, j)*i + P(i, j-1)*j) / (i + j)     otherwise           (j == 0: the second term vanishes)
    with m >= n, mg = m/g, ng = n/g; the answer is P(m, n)."""
    if m < n:
        m, n = n, m
    mg, ng = m // g, n // g
    prev = np.ones(n + 1)
    for i in range(0, m + 1):
        cur = np.ones(n + 1)
        lo = max(0, (ng * i - h) // mg + 1)
        hi = min(n + 1, -((-(ng * i + h)) // mg))  # ceil
        left = 1.0
        for j in range(lo, hi):
            if i == 0:
                v = 0.0
            else:
                v = (prev[j] * i + (left * j if j > 0 else 0.0)) / (i + j)
            cur[j] = v
            left = v
        prev = cur
    return float(min(max(prev[n], 0.0), 1.0))


def ks_2samp_exact(ref_sorted: np.ndarray, x: np.ndarray):
    """(D, p) of the two-sided exact test, or (D, None) where scipy switches to the asymptotic formula."""
    m, n = len(ref_sorted), len(x)
    num = ks_numerator(ref_sorted, x)
    g = math.gcd(m, n)
    d = num / (m * n)
    if (m // g) >= np.iinfo(np.int32).max / (n // g):
        return d, None
    h = num // g  # == round(d * lcm): numerator / g with lcm = m*n/g
    if h == 0:
        return d, 1.0
    return d, outer_prob_inside_method(m, n, g, h)


def chi2_pvalue(ref_counts: np.ndarray, x_counts: np.ndarray):
    """(statistic, p) of ``scipy.stats.chi2_contingency`` on the 2 x K table, written out (Pearson, Yates when dof == 1)."""
    obs = np.vstack((ref_counts, x_counts)).astype(np.float64)
    k = obs.shape[1]
    if k < 2:
        return 0.0, 1.0
    row, col, tot = obs.sum(1), obs.sum(0), obs.sum()
    exp = np.outer(row, col) / tot
    if k - 1 == 1:
        diff = exp - obs
        obs = obs + np.minimum(0.5, np.abs(diff)) * np.sign(diff)
    stat = float(((obs - exp) ** 2 / exp).sum())
    return stat, float(stats.chi2.sf(stat, k - 1))
