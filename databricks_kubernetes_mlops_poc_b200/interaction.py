"""How pairs of request fields act together (``B200Model.pair_dependence`` and ``B200Model.interaction_strength``): the
checks, point tables and host arithmetic around K10 (``csrc/pair_dependence.cuh``).

Two-way partial dependence is scikit-learn's ``partial_dependence(pipe, X, [a, b], method="brute")``: each field's grid
comes from ``dependence.grid_from_column``, and the points are their Cartesian product, the first field slowest (sklearn's
``cartesian`` order).

Friedman's H-statistic (Friedman & Popescu 2008, *Predictive learning via rule ensembles*, eq. 44) over a sample S of the
rows, with f = P(class 1):
    F_jk(i) = mean over l in S of f(x_l with j <- x_ij, k <- x_ik),   F_j(i) = mean over l in S of f(x_l with j <- x_ij),
each centred over S (F~ = F - mean over S of F), and
    H^2_jk = sum_i (F~_jk - F~_j - F~_k)^2 / sum_i F~_jk^2      (NaN where the denominator is 0).
F_jk(i) is the two-way partial dependence at the point (x_ij, x_ik), so rows of S that share those two words share it: the
device scores each distinct point once, as a mean over S, and the host maps the means back to the rows.
"""

from __future__ import annotations

import itertools

import numpy as np

from . import dependence

MAX_AXIS_POINTS = dependence.MAX_POINTS  # grid points per field of a pair
MAX_SAMPLE = 10000  # rows of the H-statistic's sample
DEFAULT_SAMPLE = 1000
MAX_INDIVIDUAL_VALUES = 1 << 24  # curves one HTTP answer may hold


def check_pairs(pairs, all_features) -> list:
    """A pair ``(a, b)`` or a list of them -> list of 2-tuples; ValueError for an unknown field or a pair of one field."""
    if isinstance(pairs, tuple) and len(pairs) == 2 and all(isinstance(f, str) for f in pairs):
        pairs = [pairs]
    pairs = [tuple(p) for p in pairs]
    if not pairs:
        raise ValueError("at least one pair of features is needed")
    for p in pairs:
        if len(p) != 2:
            raise ValueError(f"{p!r}: a pair is two feature names")
        unknown = [f for f in p if f not in all_features]
        if unknown:
            raise ValueError(f"unknown feature(s) {unknown}; expected names from {list(all_features)}")
        if p[0] == p[1]:
            raise ValueError(f"pair {p!r}: the two features must differ")
    return pairs


def cartesian(words_a: np.ndarray, words_b: np.ndarray) -> np.ndarray:
    """Two axes' row words -> (g_a * g_b, 2) uint32 point words, the first axis slowest."""
    wa = np.asarray(words_a, dtype=np.uint32)
    wb = np.asarray(words_b, dtype=np.uint32)
    return np.stack([np.repeat(wa, len(wb)), np.tile(wb, len(wa))], axis=1)


def check_features(features, all_features) -> list:
    """The fields of ``interaction_strength``: None = all; ValueError for an unknown or repeated one, or fewer than two."""
    features = list(all_features) if features is None else ([features] if isinstance(features, str) else list(features))
    unknown = [f for f in features if f not in all_features]
    if unknown:
        raise ValueError(f"unknown feature(s) {unknown}; expected names from {list(all_features)}")
    if len(set(features)) != len(features):
        raise ValueError(f"repeated feature(s) {sorted({f for f in features if features.count(f) > 1})}")
    if len(features) < 2:
        raise ValueError("interaction strength needs at least two features")
    return features


def check_sample(sample, random_state) -> tuple:
    """-> (sample, random_state) as ints; ValueError for a sample outside 2..MAX_SAMPLE or a seed outside [0, 2**32)."""
    if isinstance(sample, bool) or not isinstance(sample, (int, np.integer)) or not 2 <= int(sample) <= MAX_SAMPLE:
        raise ValueError(f"sample={sample!r}: expected an integer in 2..{MAX_SAMPLE}")
    if isinstance(random_state, bool) or not isinstance(random_state, (int, np.integer)) or not 0 <= int(random_state) < 2**32:
        raise ValueError(f"random_state={random_state!r}: expected an integer in [0, 2**32 - 1]")
    return int(sample), int(random_state)


def sample_rows(n: int, sample: int, random_state: int) -> np.ndarray:
    """The sample S: every row when n <= sample, else ``RandomState(random_state).choice(n, sample, replace=False)``.
    ValueError when fewer than two rows remain."""
    if n < 2:
        raise ValueError(f"interaction strength needs at least 2 rows, got {n}")
    if n <= sample:
        return np.arange(n)
    return np.random.RandomState(random_state).choice(n, sample, replace=False)


def impute(rows: np.ndarray, n_cat: int, n_num: int, medians) -> np.ndarray:
    """Encoded (n, 24) rows with NaN numerics replaced by the float32 training medians, as the kernels score them."""
    w = np.array(rows, dtype=np.uint32, copy=True)
    f = w[:, n_cat:n_cat + n_num].view(np.float32)
    med = np.asarray(medians, dtype=np.float32)[n_cat:n_cat + n_num]
    nan = np.isnan(f)
    f[nan] = np.broadcast_to(med, f.shape)[nan]
    return w


def _order_key(words: np.ndarray, categorical: bool) -> np.ndarray:
    """A column of row words -> float64 keys in value order (codes for a categorical word, values for a numeric one)."""
    w = np.asarray(words, dtype=np.uint32)
    return w.view(np.int32).astype(np.float64) if categorical else w.view(np.float32).astype(np.float64)


def distinct_points(cols, categorical) -> tuple:
    """One or two columns of (imputed) row words of the rows -> (points (m, len(cols)) uint32, inverse (n,)): the distinct
    word tuples, sorted by value (first column slowest) so a 32-point segment holds neighbouring values and forks less,
    and for each row the index of its tuple."""
    cols = [np.asarray(c, dtype=np.uint32) for c in cols]
    key = cols[0].astype(np.uint64)
    if len(cols) == 2:
        key = (key << np.uint64(32)) | cols[1].astype(np.uint64)
    uniq, inverse = np.unique(key, return_inverse=True)
    parts = [(uniq >> np.uint64(32)).astype(np.uint32), (uniq & np.uint64(0xFFFFFFFF)).astype(np.uint32)] if len(cols) == 2 else [uniq.astype(np.uint32)]
    order = np.lexsort([_order_key(p, c) for p, c in zip(parts, categorical)][::-1])
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    return np.stack([p[order] for p in parts], axis=1), rank[inverse.reshape(-1)]


def centred(F: np.ndarray) -> np.ndarray:
    return F - F.mean()


def h_squared(F_jk: np.ndarray, F_j: np.ndarray, F_k: np.ndarray) -> tuple:
    """Per-row partial dependences over S -> (H^2, numerator, denominator); H^2 is NaN where the denominator is 0."""
    c_jk, c_j, c_k = centred(F_jk), centred(F_j), centred(F_k)
    num = float(np.sum((c_jk - c_j - c_k) ** 2))
    den = float(np.sum(c_jk ** 2))
    return (num / den if den > 0 else float("nan")), num, den


def strength_plan(words: np.ndarray, fields, categorical) -> tuple:
    """The imputed row words (|S|, 24) of the sample, the probed row words and whether each is categorical -> (probes,
    point words (P, 2), maps): one one-way probe per field (its distinct words), then one probe per pair in
    ``itertools.combinations`` order (its distinct word pairs); maps[p] = (first point of probe p, each row's point)."""
    probes, parts, maps, off = [], [], [], 0
    for w, c in zip(fields, categorical):
        pts, inv = distinct_points([words[:, w]], [c])
        probes.append((w, -1, off, len(pts)))
        parts.append(np.stack([pts[:, 0], np.zeros(len(pts), dtype=np.uint32)], axis=1))
        maps.append((off, inv))
        off += len(pts)
    for (wj, cj), (wk, ck) in itertools.combinations(list(zip(fields, categorical)), 2):
        pts, inv = distinct_points([words[:, wj], words[:, wk]], [cj, ck])
        probes.append((wj, wk, off, len(pts)))
        parts.append(pts)
        maps.append((off, inv))
        off += len(pts)
    return probes, np.concatenate(parts), maps


def strength_result(means: np.ndarray, maps, features) -> dict:
    """The device means of ``strength_plan``'s points -> the answer of ``interaction_strength`` (without ``rows``)."""
    F = len(features)
    single = [means[o + inv] for o, inv in maps[:F]]
    pairs, h2, num, den = [], [], [], []
    matrix = np.full((F, F), np.nan)
    for p, (j, k) in enumerate(itertools.combinations(range(F), 2)):
        o, inv = maps[F + p]
        h, a, b = h_squared(means[o + inv], single[j], single[k])
        pairs.append((features[j], features[k]))
        h2.append(h), num.append(a), den.append(b)
        matrix[j, k] = matrix[k, j] = h
    return {"pairs": pairs, "h_squared": np.array(h2), "numerator": np.array(num), "denominator": np.array(den), "matrix": matrix,
            "feature_names": list(features)}
