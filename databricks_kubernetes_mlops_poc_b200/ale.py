"""Accumulated local effects (``B200Model.accumulated_local_effects``): the request checks, the edge rule, the float32
edges, and the host arithmetic around K12 (``csrc/ale.cuh``).

ALE (Apley & Zhu, JRSS-B 2020) answers what partial dependence answers -- how P(class 1) moves with one numeric field --
without scoring applicants at values they do not have.  For a field with float32 edges z_0 < ... < z_K, a row with a
present value x lies in bin k = clamp(#{j : z_j < x}, 1, K) (``searchsorted(z, x, "left")`` clamped at both ends) and is
scored only at z_{k-1} and z_k.  The device returns per bin the sum of f(z_k) - f(z_{k-1}) over its n_k rows and n_k; the
host takes

    d_k = sum / n_k (0 when n_k = 0),   A_0 = 0, A_k = d_1 + ... + d_k,
    ale0 = sum_k n_k (A_{k-1} + A_k) / 2 / sum_k n_k,   ale_values = A - ale0   (alibi's centring),

in float64 numpy, in that order.  The default edges follow alibi's approach: a quantile grid whose bins each hold at least
``min_bin_points`` rows (the largest K from ``bins`` down that does), and every distinct value when there are at most
``bins + 1`` of them.
"""

from __future__ import annotations

import numpy as np

from . import dependence

MAX_BINS = 256  # B2F_ALE_MAX_BINS
DEFAULT_BINS = 20
DEFAULT_MIN_BIN_POINTS = 4


def check_features(features, numeric_features, categorical_features) -> list:
    """The probed fields: None = every numeric field in field order; ValueError for an unknown, categorical or repeated one."""
    features = list(numeric_features) if features is None else ([features] if isinstance(features, str) else list(features))
    if not features:
        raise ValueError("at least one feature is needed")
    cats = [f for f in features if f in categorical_features]
    if cats:
        raise ValueError(f"categorical feature(s) {cats} have no order, so accumulated local effects do not apply; "
                         "use partial_dependence for them")
    unknown = [f for f in features if f not in numeric_features]
    if unknown:
        raise ValueError(f"unknown feature(s) {unknown}; expected names from {list(numeric_features)}")
    if len(set(features)) != len(features):
        raise ValueError(f"repeated feature(s) {sorted({f for f in features if features.count(f) > 1})}")
    return features


def check_params(bins, min_bin_points) -> tuple:
    """-> (bins, min_bin_points) as ints; ValueError for bins outside 1..256 or min_bin_points < 1."""
    if isinstance(bins, bool) or not isinstance(bins, (int, np.integer)) or not 1 <= int(bins) <= MAX_BINS:
        raise ValueError(f"bins={bins!r}: expected an integer in 1..{MAX_BINS}")
    if isinstance(min_bin_points, bool) or not isinstance(min_bin_points, (int, np.integer)) or int(min_bin_points) < 1:
        raise ValueError(f"min_bin_points={min_bin_points!r}: expected an integer >= 1")
    return int(bins), int(min_bin_points)


def present_float32(encoder, feature: str, values) -> np.ndarray:
    """A column of raw values -> its present values as the float32 the encoder produces (overflow: ValueError)."""
    x = dependence.encode_grid(encoder, feature, list(values)).view(np.float32)
    return x[~np.isnan(x)]


def check_custom_edges(feature: str, edges) -> np.ndarray:
    """Caller edges -> float32; ValueError unless 2..257 finite numbers, strictly increasing after rounding to float32."""
    try:
        z64 = np.asarray([float(v) for v in edges], dtype=np.float64)
    except (TypeError, ValueError):
        raise ValueError(f"custom edges of {feature!r} must be numbers") from None
    if not 2 <= len(z64) <= MAX_BINS + 1:
        raise ValueError(f"feature {feature!r}: {len(z64)} custom edges, expected 2..{MAX_BINS + 1}")
    with np.errstate(over="ignore"):
        z = z64.astype(np.float32)
    if not np.isfinite(z).all():
        raise ValueError(f"custom edges of {feature!r} must be finite float32 numbers")
    if not (z[1:] > z[:-1]).all():
        raise ValueError(f"custom edges of {feature!r} must be strictly increasing after rounding to float32")
    return z


def sorted_quantiles(xs: np.ndarray, q: np.ndarray) -> np.ndarray:
    """``np.quantile(x, q)`` (method "linear") of an ascending float64 column, with numpy's operations in numpy's order."""
    n = len(xs)
    q = np.asarray(q, dtype=np.float64)
    vi = (n - 1) * q
    prev = np.floor(vi)
    gamma = vi - prev
    lo = prev.astype(np.intp)
    lo[vi >= n - 1] = n - 1
    hi = np.minimum(lo + 1, n - 1)
    a, b = xs[lo], xs[hi]
    diff = b - a
    out = a + diff * gamma
    up = gamma >= 0.5
    out[up] = (b - diff * (1 - gamma))[up]
    return out


def bin_counts(x32: np.ndarray, z: np.ndarray) -> np.ndarray:
    """Rows per bin: bin k = clamp(searchsorted(z, x, "left"), 1, K), as the kernel bins them -> int64 (K,)."""
    K = len(z) - 1
    k = np.clip(np.searchsorted(z, x32, side="left"), 1, K)
    return np.bincount(k - 1, minlength=K).astype(np.int64)


def default_edges(x32: np.ndarray, bins: int, min_bin_points: int) -> np.ndarray:
    """The edge rule over a field's present float32 values -> float32 edges (one edge when there is one distinct value).
    ValueError when there is no present value."""
    x32 = np.asarray(x32, dtype=np.float32)
    if len(x32) == 0:
        raise ValueError("the column has no present value to build edges from")
    u = np.unique(x32)
    if len(u) <= bins + 1:
        return u
    xs = np.sort(x32).astype(np.float64)
    for K in range(bins, 0, -1):
        z = np.unique(sorted_quantiles(xs, np.linspace(0, 1, K + 1)).astype(np.float32))
        if len(z) >= 2 and bin_counts(x32, z).min() >= min_bin_points:
            return z
    return u[[0, -1]]


def effects(sums: np.ndarray, counts: np.ndarray) -> dict:
    """A field's per-bin delta sums and row counts -> bin_effects, the centred ale_values (K + 1) and ale0."""
    n = np.asarray(counts, dtype=np.int64)
    s = np.asarray(sums, dtype=np.float64)
    d = np.zeros(len(n), dtype=np.float64)
    nz = n > 0
    d[nz] = s[nz] / n[nz]
    A = np.concatenate([[0.0], np.cumsum(d)])
    total = int(n.sum())
    ale0 = float(np.sum(n * (A[:-1] + A[1:]) / 2) / total) if total else 0.0
    return {"bin_effects": d, "bin_rows": n, "ale_values": A - ale0, "ale0": ale0}


def probe_plan(words, edges) -> tuple:
    """Row words and float32 edges per field -> (probes [(word, edge offset, bins)], the concatenated edges, the index of
    each probed field): fields with one edge (no bin) are left out."""
    probes, parts, which, off = [], [], [], 0
    for i, (w, z) in enumerate(zip(words, edges)):
        if len(z) >= 2:
            probes.append((int(w), off, len(z) - 1))
            parts.append(np.asarray(z, dtype=np.float32))
            which.append(i)
            off += len(z)
    return probes, (np.concatenate(parts) if parts else np.zeros(0, np.float32)), which


def result(features, edges, sums, counts, probes, which) -> dict:
    """The device's per-bin sums and counts (probe order) -> the answer of ``accumulated_local_effects`` (without
    ``constant_value`` and ``rows``)."""
    res = {"feature_names": list(features), "output": "probability", "feature_values": [], "ale_values": [], "bin_effects": [],
           "bin_rows": [], "ale0": []}
    at = {i: p for i, p in zip(which, probes)}
    boff = 0
    for i, z in enumerate(edges):
        res["feature_values"].append(np.asarray(z, dtype=np.float32).astype(np.float64))
        if i in at:
            K = at[i][2]
            e = effects(sums[boff:boff + K], counts[boff:boff + K])
            boff += K
        else:
            e = {"bin_effects": np.zeros(0), "bin_rows": np.zeros(0, np.int64), "ale_values": np.zeros(1), "ale0": 0.0}
        for k in ("ale_values", "bin_effects", "bin_rows", "ale0"):
            res[k].append(e[k])
    return res
