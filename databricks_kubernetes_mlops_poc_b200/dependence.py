"""Partial dependence and ICE curves (``B200Model.partial_dependence``): grids, their encoding, and the per-feature split of
the kernel's output (``csrc/partial_dependence.cuh``).

The grid rule is scikit-learn's ``sklearn.inspection._partial_dependence._grid_from_X``: a categorical field, or one with
fewer unique values than ``grid_resolution``, is probed at its sorted unique values; any other at ``grid_resolution``
evenly spaced points between two ``mquantiles`` (alphap = betap = 0.4, scipy's default plotting positions, reimplemented
here in numpy).  One difference: missing values (NaN numerics, None / NaN categories) are left out of a default grid,
where scikit-learn would fail (a category column with None) or put NaN on the grid.  Explicit ``custom_values`` may hold
None / NaN: such a point means "missing" and is imputed exactly as the pipeline imputes a missing request value.
"""

from __future__ import annotations

import numpy as np
import pandas as pd

MAX_POINTS = 256  # grid points per feature (B2F_PD_MAX_POINTS)
MAX_FEATURES = 23  # features per call (B2F_PD_MAX_PROBES)
KINDS = ("average", "individual", "both")
DEFAULT_RESOLUTION = 100
DEFAULT_PERCENTILES = (0.05, 0.95)


def mquantiles(x: np.ndarray, prob, alphap: float = 0.4, betap: float = 0.4) -> np.ndarray:
    """``scipy.stats.mstats.mquantiles(x, prob, alphap, betap)`` of a 1-D array without missing values, with scipy's
    operations in scipy's order."""
    x = np.sort(np.asarray(x, dtype=np.float64))
    n = len(x)
    p = np.atleast_1d(np.asarray(prob, dtype=np.float64))
    if n == 1:
        return np.resize(x, p.shape)
    m = alphap + p * (1.0 - alphap - betap)
    aleph = n * p + m
    k = np.floor(aleph.clip(1, n - 1)).astype(int)
    gamma = (aleph - k).clip(0, 1)
    return (1.0 - gamma) * x[(k - 1).tolist()] + gamma * x[k.tolist()]


def _present(values, is_categorical: bool) -> np.ndarray:
    """The column without its missing values: strings for a categorical field, float64 otherwise."""
    if is_categorical:
        v = np.asarray(values, dtype=object)
        return np.array([s for s in v if isinstance(s, str)], dtype=object)
    v = pd.to_numeric(pd.Series(values), errors="raise").to_numpy(dtype=np.float64, na_value=np.nan)
    return v[~np.isnan(v)]


def grid_from_column(values, is_categorical: bool, grid_resolution: int = 100, percentiles=(0.05, 0.95)) -> np.ndarray:
    """The default grid of one field from a column of raw values (sklearn's ``_grid_from_X`` rule, missing values left
    out).  ValueError when the column has no present value, or the percentiles coincide."""
    if len(percentiles) != 2 or not all(0 <= q <= 1 for q in percentiles) or percentiles[0] >= percentiles[1]:
        raise ValueError("'percentiles' must be two increasing values in [0, 1]")
    if grid_resolution <= 1:
        raise ValueError("'grid_resolution' must be strictly greater than 1.")
    x = _present(values, is_categorical)
    if len(x) == 0:
        raise ValueError("the column has no present value to build a grid from")
    uniques = np.unique(x)
    if is_categorical or uniques.shape[0] < grid_resolution:
        return uniques
    q = mquantiles(x, prob=percentiles)
    if np.allclose(q[0], q[1]):
        raise ValueError("percentiles are too close to each other, unable to build the grid. Please choose percentiles that are "
                         "further apart.")
    return np.linspace(q[0], q[1], num=grid_resolution, endpoint=True)


def encode_grid(encoder, feature: str, values) -> np.ndarray:
    """A feature's grid values -> its row word per point (uint32), encoded by ``encoder`` as a G-row request frame is, so
    float64 -> float32 rounding, NaN, overflow (ValueError) and category codes follow the request path."""
    values = list(values)
    g = len(values)
    frame = {name: [None] * g for name in encoder.cat_features}
    frame.update({name: np.full(g, np.nan) for name in encoder.num_features})
    col = np.empty(g, dtype=object)
    col[:] = values
    frame[feature] = col if feature in encoder.cat_features else pd.to_numeric(pd.Series(col), errors="raise").to_numpy(dtype=np.float64)
    rows = encoder.encode_frame(pd.DataFrame(frame))
    return rows[:, word_of(encoder, feature)].copy()


def word_of(encoder, feature: str) -> int:
    """The row word of a request field: categoricals first, then numerics."""
    if feature in encoder.cat_features:
        return encoder.cat_features.index(feature)
    return encoder.n_cat + encoder.num_features.index(feature)


def check_request(features, all_features, kind: str) -> list:
    """Validate the feature list and kind -> the list of names (ValueError on a bad one)."""
    features = [features] if isinstance(features, str) else list(features)
    if not features:
        raise ValueError("at least one feature is needed")
    if len(features) > MAX_FEATURES:
        raise ValueError(f"{len(features)} features: at most {MAX_FEATURES} per call")
    unknown = [f for f in features if f not in all_features]
    if unknown:
        raise ValueError(f"unknown feature(s) {unknown}; expected names from {list(all_features)}")
    if kind not in KINDS:
        raise ValueError(f"kind={kind!r}: expected one of {KINDS}")
    return features


def split_output(out: np.ndarray, counts, kind: str) -> dict:
    """The kernel's (n, sum G) curves -> ``{"average": [...], "individual": [...]}`` per ``kind``; the average is numpy's
    mean over the rows, as scikit-learn takes it."""
    res = {}
    individual, lo = [], 0
    for g in counts:
        individual.append(out[:, lo:lo + g])
        lo += g
    if kind in ("average", "both"):
        res["average"] = [c.mean(axis=0) for c in individual]
    if kind in ("individual", "both"):
        res["individual"] = [np.ascontiguousarray(c) for c in individual]
    return res
