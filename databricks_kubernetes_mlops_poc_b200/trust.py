"""Trust scores (``B200Model.trust_score``): alibi's ``TrustScore`` (Jiang et al., *To Trust or Not to Trust a Classifier*,
NeurIPS 2018) against a labelled reference table, with the exact nearest-neighbour search on the GPU (``csrc/knn.cuh``) and
everything else here: argument checks, the distance filter's percentile rule, the map back to frame positions and the score.

Space: the MMD test's embedding (``mmd.py``): one-hot categoricals (an unknown or missing code is the all-zero block) and the
numerics as scored, z-scored in float64 with the trust reference's own mean and population std, computed over the whole
reference before any filtering.  Distances are Euclidean on that embedding.

Fit: per class c the fitted set is the reference rows of class c.  ``filter_type="distance_knn"`` is alibi's
``filter_by_distance_knn`` per class: each row's ``k_filter + 1`` nearest rows of its own class (itself included) give a radius
r, the last of those distances ("point") or the mean of all but the first ("mean"), and the rows with
``r <= np.percentile(r, (1 - alpha) * 100)`` are kept.

Score: per row and class, D_c is the k-th nearest distance to the class's fitted set ("point") or the mean of the k nearest
("mean"); ``trust_score = D_other / (D_pred + 1e-12)``, with the predicted class the classifier's and the other class the
closest class that is not predicted (the model is binary).
"""

from __future__ import annotations

import numpy as np

from .mmd import MAX_REFERENCE

MAX_K = 64  # B2F_KNN_MAX_K
MAX_K_FILTER = MAX_K - 1
FILTER_TYPES = (None, "distance_knn")
DIST_TYPES = ("point", "mean")
EPS = 1e-12  # alibi's TrustScore.eps


def _is_int(v) -> bool:
    return isinstance(v, (int, np.integer)) and not isinstance(v, bool)


def check_fit(n: int, k_filter, alpha, filter_type, dist_filter_type) -> tuple[int, float, str | None, str]:
    """-> (k_filter, alpha, filter_type, dist_filter_type); ValueError for a reference outside 2..MAX_REFERENCE rows, k_filter
    outside 1..MAX_K_FILTER, alpha outside [0, 1), an unknown filter or distance type."""
    if not 2 <= n <= MAX_REFERENCE:
        raise ValueError(f"a trust reference needs 2..{MAX_REFERENCE} rows, not {n}")
    if not _is_int(k_filter) or not 1 <= k_filter <= MAX_K_FILTER:
        raise ValueError(f"k_filter must be an integer in 1..{MAX_K_FILTER}, not {k_filter!r}")
    a = float(alpha)
    if not 0.0 <= a < 1.0:
        raise ValueError(f"alpha must be in [0, 1), not {alpha!r}")
    if filter_type == "probability_knn":
        raise ValueError("filter_type='probability_knn' is not supported: use None or 'distance_knn'")
    if filter_type not in FILTER_TYPES:
        raise ValueError(f"filter_type must be one of {FILTER_TYPES}, not {filter_type!r}")
    if dist_filter_type not in DIST_TYPES:
        raise ValueError(f"dist_filter_type must be one of {DIST_TYPES}, not {dist_filter_type!r}")
    return int(k_filter), a, filter_type, dist_filter_type


def class_indices(labels, classes) -> np.ndarray:
    """Labels (the model's class values) -> int32 class indices 0 / 1; ValueError for another value or a length mismatch."""
    y = np.asarray(labels)
    classes = np.asarray(classes)
    if y.ndim != 1:
        raise ValueError(f"labels must be one-dimensional, not {y.shape}")
    out = np.full(len(y), -1, dtype=np.int32)
    for c, v in enumerate(classes):
        out[y == v] = c
    if (out < 0).any():
        bad = y[out < 0][0]
        raise ValueError(f"label {bad!r} is not one of the model's classes {classes.tolist()}")
    return out


def check_class_rows(cls: np.ndarray, filter_type, k_filter: int) -> None:
    """Each class needs a row, and k_filter + 1 rows when the distance filter runs."""
    need = k_filter + 1 if filter_type == "distance_knn" else 1
    for c in (0, 1):
        n_c = int((cls == c).sum())
        if n_c < need:
            raise ValueError(f"class {c} has {n_c} reference rows; " + (f"the distance filter with k_filter={k_filter} needs {need}"
                                                                          if need > 1 else "each class needs at least one"))


def filter_radius(dist: np.ndarray, dist_filter_type: str) -> np.ndarray:
    """(m, k_filter + 1) sorted distances of each row to its own class, itself included -> the radius of each row."""
    return dist[:, -1] if dist_filter_type == "point" else np.mean(dist[:, 1:], axis=1)


def filter_keep(r: np.ndarray, alpha: float) -> np.ndarray:
    """The rows alibi's ``filter_by_distance_knn`` keeps: radius at most the (1 - alpha) percentile."""
    return r <= np.percentile(r, (1.0 - alpha) * 100.0)


def check_score(k, dist_type, reference_rows) -> tuple[int, str]:
    """-> (k, dist_type); ValueError for k outside 1..MAX_K or above the rows kept in either class, or an unknown dist_type."""
    if not _is_int(k) or not 1 <= k <= MAX_K:
        raise ValueError(f"k must be an integer in 1..{MAX_K}, not {k!r}")
    if k > min(reference_rows):
        raise ValueError(f"k={k} is more than the {min(reference_rows)} reference rows kept in the smaller class")
    if dist_type not in DIST_TYPES:
        raise ValueError(f"dist_type must be one of {DIST_TYPES}, not {dist_type!r}")
    return int(k), dist_type


def class_distance(dist: np.ndarray, dist_type: str) -> np.ndarray:
    """(n, k) sorted distances to one class -> D_c per row."""
    return dist[:, -1] if dist_type == "point" else np.mean(dist, axis=1)


def result(dist: np.ndarray, index: np.ndarray, proba: np.ndarray, pred: np.ndarray, classes, positions: np.ndarray, k: int,
           dist_type: str, reference_rows) -> dict:
    """The answer from b2f_knn's (n, 2, k) distances and reference indices, the classifier's P(class 1) and predicted class index
    per row; ``positions`` maps an attached reference row to its position in the frame the reference was fitted on."""
    n = len(pred)
    d = np.stack([class_distance(dist[:, c, :], dist_type) for c in (0, 1)], axis=1) if n else np.empty((0, 2))
    rows = np.arange(n)
    d_pred, d_other = d[rows, pred], d[rows, 1 - pred]
    classes = np.asarray(classes)
    return {"trust_score": d_other / (d_pred + EPS), "closest_not_pred": classes[1 - pred], "predictions": np.asarray(proba, dtype=np.float64),
            "labels": classes[pred], "distance_to_pred": d_pred, "distance_to_other": d_other, "k": int(k), "dist_type": dist_type,
            "reference_rows": [int(r) for r in reference_rows],
            "neighbours": [{"class": classes[c].item(), "index": positions[index[:, c, :]], "distance": dist[:, c, :].copy()} for c in (0, 1)]}
