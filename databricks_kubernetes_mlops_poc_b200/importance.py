"""Permutation importance (``B200Model.permutation_importance``): the permutations scikit-learn draws, and the scorer
formulas that turn the kernel's records (``csrc/permutation_importance.cuh``) into scikit-learn's numbers.

``sklearn.inspection.permutation_importance(estimator, X, y, scoring=..., n_repeats=R, random_state=rs)`` draws one seed,
``check_random_state(rs).randint(2**31)``, and replays the same ``RandomState(seed)`` for every column: ``idx = arange(n)``,
then per repeat ``shuffle(idx)`` and ``X[:, c] = X[idx, c]`` on the already permuted column.  So repeat r reads row
``sigma_r(i)`` with ``sigma_r = sigma_{r-1}[idx_r]``, the same for every column, whatever the column order.

This module is the one place that knows the scorer names.
"""

from __future__ import annotations

import math

import numpy as np
from sklearn.utils import check_random_state

MAX_REPEATS = 256  # B2F_PERM_MAX_REPEATS
# name -> greater is better, as sklearn's scorers (the neg_* ones are negated losses)
SCORERS = ("accuracy", "precision", "recall", "f1", "roc_auc", "neg_log_loss", "neg_brier_score")
DEFAULT_SCORER = "accuracy"  # estimator.score of a classifier


def permutations(n: int, n_repeats: int, random_state=None) -> np.ndarray:
    """The row permutations scikit-learn's ``permutation_importance`` applies: int32 (n_repeats, n), row r = sigma_r."""
    seed = check_random_state(random_state).randint(np.iinfo(np.int32).max + 1)
    rs = np.random.RandomState(seed)
    idx = np.arange(n)
    out = np.empty((n_repeats, n), dtype=np.int32)
    sigma = np.arange(n)
    for r in range(n_repeats):
        rs.shuffle(idx)
        sigma = sigma[idx]
        out[r] = sigma
    return out


def check_scoring(scoring) -> tuple[list[str], bool]:
    """``scoring`` (None, one name or a list of names) -> (names, whether the answer is a dict keyed by name)."""
    if scoring is None:
        return [DEFAULT_SCORER], False
    if isinstance(scoring, str):
        names, multi = [scoring], False
    else:
        names, multi = list(scoring), True
        if not names:
            raise ValueError("scoring: an empty list of scorers")
        if len(set(names)) != len(names):
            raise ValueError(f"scoring: repeated scorer(s) {sorted({s for s in names if names.count(s) > 1})}")
    unknown = [s for s in names if s not in SCORERS]
    if unknown:
        raise ValueError(f"unsupported scorer(s) {unknown}; expected names from {list(SCORERS)}")
    return names, multi


def check_labels(y, n: int) -> np.ndarray:
    """-> int32 (n,) of 0/1 labels (ValueError otherwise)."""
    a = np.asarray(y)
    if a.ndim != 1 or a.shape[0] != n:
        raise ValueError(f"y must hold one label per row: got shape {a.shape} for {n} rows")
    if a.dtype.kind == "f":
        if not np.all((a == 0) | (a == 1)):
            raise ValueError("y must hold 0/1 labels")
    elif a.dtype.kind == "b":
        pass
    elif a.dtype.kind not in "iu":
        raise ValueError(f"y must hold 0/1 labels, not {a.dtype}")
    elif not np.all((a == 0) | (a == 1)):
        raise ValueError("y must hold 0/1 labels")
    return a.astype(np.int32)


def check_n_repeats(n_repeats) -> int:
    if isinstance(n_repeats, bool) or not isinstance(n_repeats, (int, np.integer)) or not 1 <= int(n_repeats) <= MAX_REPEATS:
        raise ValueError(f"n_repeats={n_repeats!r}: expected an integer in 1..{MAX_REPEATS}")
    return int(n_repeats)


def check_single_class(names, labels: np.ndarray) -> None:
    """sklearn's log_loss refuses labels of one class."""
    if "neg_log_loss" in names and len(np.unique(labels)) < 2:
        raise ValueError(f"y_true contains only one label ({int(labels[0])}). Please provide the list of all expected class labels "
                         "explicitly through the labels argument.")


def _ratio(a, b):
    return np.where(b > 0, a / np.where(b > 0, b, 1), 0.0)


def score(name: str, rec) -> np.ndarray:
    """Records (any shape, ``PERM_SCORE_DTYPE``) -> sklearn's score ``name`` of each, float64."""
    tp, fp, tn, fn = (rec[k].astype(np.float64) for k in ("tp", "fp", "tn", "fn"))
    n = tp + fp + tn + fn
    if name == "accuracy":
        return (tp + tn) / n
    if name == "precision":
        return _ratio(tp, tp + fp)
    if name == "recall":
        return _ratio(tp, tp + fn)
    if name == "f1":
        return _ratio(2 * tp, 2 * tp + fp + fn)
    if name == "roc_auc":
        pos, neg = tp + fn, fp + tn
        u2 = rec["auc_u2"].astype(np.float64)
        with np.errstate(invalid="ignore", divide="ignore"):
            return np.where((pos > 0) & (neg > 0), u2 / (2.0 * pos * neg), np.nan)
    if name == "neg_log_loss":
        return -(rec["log_loss_sum"] / n)
    if name == "neg_brier_score":
        return -(rec["brier_sum"] / n)
    raise ValueError(f"unsupported scorer {name!r}")


def result(name: str, records, baseline, feature_names, n_repeats: int, rows: int) -> dict:
    """One scorer's answer from the kernel's records (F, R) and baseline record, as sklearn's Bunch holds it."""
    base = float(score(name, baseline))
    imp = base - score(name, records)
    return {"importances": imp, "importances_mean": np.mean(imp, axis=1), "importances_std": np.std(imp, axis=1),
            "baseline_score": base, "feature_names": list(feature_names), "n_repeats": n_repeats, "rows": rows}


def json_number(v):
    """A float for JSON: NaN -> null."""
    v = float(v)
    return None if math.isnan(v) else v
