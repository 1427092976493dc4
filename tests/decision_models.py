"""Models whose rows land on a decision boundary, and an order-independent reference for the decision.

Small reference pipelines are fitted, then their leaves are overwritten through ``tree_.value`` (sklearn >= 1.4 keeps
the writes and ``predict_proba`` / ``predict`` read them back):

* ``rf_exact_ties``: every leaf holds a dyadic class-1 fraction (0, 1/4, 1/2, 3/4, 1), so every summation order is
  exact and a known share of rows has ``p1 == 0.5`` exactly -- sklearn's argmax gives them class 0;
* ``rf_near_ties``: every leaf holds ``[1 - b, b]`` or ``[b, 1 - b]`` with ``b`` one of the doubles 0.6, 0.7, 0.8, 0.9
  (``1 - b`` is exact, so each leaf's fractions add to exactly 1): rows whose decimal sum is ``T / 2`` have an exact
  margin of a few units of 2^-54 or exactly zero, and the sign of a float64 sum of them depends on the order;
* ``gbdt_zero_raw``: ``init='zero'``, learning rate 1/2 and leaves of +-1/8, +-1/4, so many rows reach ``raw == 0``
  exactly; tree 0 also holds leaves of 2^-56, which give rows with ``0 < raw <= 5.6e-17`` (expit rounds to 0.5).

The reference decision is the exact sign of ``sum_t p1_t - sum_t p0_t`` (RF) or of ``init + sum_t lr * v_t`` (GBDT),
taken with ``math.fsum`` over sklearn's own per-tree leaf values at the leaves sklearn's ``apply`` reaches: a correctly
rounded sum has the sign of the exact one, whatever order the terms come in."""

from __future__ import annotations

import math

import numpy as np

EPS = float(np.finfo(np.float64).eps)
TINY = 2.0**-56
NEAR_B = (0.6, 0.7, 0.8, 0.9)


def fit_rf(curated, n_trees: int, depth: int = 6, rows: int = 3000):
    from oracle import reference_pipeline as rp

    tr = curated.iloc[:rows]
    pipe = rp.make_classifier_pipeline(dict(n_estimators=n_trees, max_depth=depth, random_state=n_trees))
    pipe.fit(tr[rp.FEATURES], tr[rp.TARGET].to_numpy())
    return pipe


def _leaves(tree):
    return np.nonzero(tree.children_left == -1)[0]


def rf_exact_ties(curated, n_trees: int):
    """Leaves of dyadic class-1 fractions: exact in every order."""
    pipe = fit_rf(curated, n_trees)
    rng = np.random.default_rng(100 + n_trees)
    for est in pipe.named_steps["classifier"].estimators_:
        v = est.tree_.value
        lv = _leaves(est.tree_)
        q = rng.choice([0.0, 0.25, 0.5, 0.75, 1.0], size=lv.size, p=[0.1, 0.25, 0.3, 0.25, 0.1])
        v[lv, 0, 0] = 1.0 - q
        v[lv, 0, 1] = q
    return pipe


def rf_near_ties(curated, n_trees: int):
    """Leaves ``[1 - b, b]`` / ``[b, 1 - b]``: sums of T / 2 in decimal, a few ulps off it in binary."""
    pipe = fit_rf(curated, n_trees)
    rng = np.random.default_rng(200 + n_trees)
    for est in pipe.named_steps["classifier"].estimators_:
        v = est.tree_.value
        lv = _leaves(est.tree_)
        b = rng.choice(NEAR_B, size=lv.size)
        hi = rng.random(lv.size) < 0.5
        v[lv, 0, 1] = np.where(hi, b, 1.0 - b)
        v[lv, 0, 0] = np.where(hi, 1.0 - b, b)
    return pipe


def gbdt_zero_raw(curated, n_trees: int = 24):
    """``init='zero'``, lr = 1/2, leaves +-1/8 and +-1/4 (tree 0: some leaves 2^-56 instead)."""
    from oracle import reference_pipeline as rp

    tr = curated.iloc[:3000]
    pipe = rp.fit_gbdt_pipeline(tr, tr[rp.TARGET].to_numpy(),
                                dict(n_estimators=n_trees, max_depth=3, learning_rate=0.5, init="zero", random_state=0))
    rng = np.random.default_rng(300)
    for t, est in enumerate(pipe.named_steps["classifier"].estimators_[:, 0]):
        v = est.tree_.value
        lv = _leaves(est.tree_)
        vals = rng.choice([-0.5, -0.25, 0.25, 0.5], size=lv.size)  # x lr = +-1/4, +-1/8
        if t == 0:
            vals[::2] = 2.0 * TINY  # x lr = 2^-56
        v[lv, 0, 0] = vals
    return pipe


def leaf_terms(pipe, df):
    """-> (n, T) per-tree terms at the leaves sklearn reaches: RF (p0, p1) normalised as ``predict_proba`` does,
    GBDT ``lr * value`` (p0 is None)."""
    from oracle import reference_pipeline as rp

    X = pipe.named_steps["preprocessor"].transform(df[rp.FEATURES])
    X = np.asarray(X.toarray() if hasattr(X, "toarray") else X, dtype=np.float32)
    clf = pipe.named_steps["classifier"]
    if type(clf).__name__ == "RandomForestClassifier":
        leaves = clf.apply(X)
        p0 = np.empty(leaves.shape)
        p1 = np.empty(leaves.shape)
        for t, est in enumerate(clf.estimators_):
            v = est.tree_.value[leaves[:, t], 0, :]
            s = v.sum(axis=1)
            p0[:, t] = v[:, 0] / s
            p1[:, t] = v[:, 1] / s
        return p0, p1
    leaves = clf.apply(X)[:, :, 0].astype(np.int64)
    terms = np.empty(leaves.shape)
    for t, est in enumerate(clf.estimators_[:, 0]):
        terms[:, t] = clf.learning_rate * est.tree_.value[leaves[:, t], 0, 0]
    return None, terms


def exact_margin(p0, p1) -> np.ndarray:
    """Correctly rounded ``sum p1 - sum p0`` (RF) or ``sum terms`` (GBDT, ``p0`` None; init is zero): its sign is exact."""
    if p0 is None:
        return np.array([math.fsum(r) for r in p1])
    return np.array([math.fsum(np.concatenate([a, -b])) for a, b in zip(p1, p0)])


def exact_labels(p0, p1) -> np.ndarray:
    """RF: class 1 iff the margin is positive (a tie is class 0).  GBDT: class 1 iff raw >= 0."""
    m = exact_margin(p0, p1)
    return (m >= 0.0 if p0 is None else m > 0.0).astype(np.int32)


def shared_outlier_score(score: np.ndarray) -> float:
    """The outlier score (``-decision_function``) the most rows share: a threshold that many rows sit on."""
    vals, counts = np.unique(score, return_counts=True)
    return float(vals[np.argmax(counts)])


def band(n_trees: int) -> float:
    """Half-width of the rounding band of an RF margin: a float64 sum of T payloads in [0, 1] is within T^2 eps of the
    exact one in any order, and the label is the sign of 2 s - T."""
    return 4.0 * n_trees * EPS * n_trees
