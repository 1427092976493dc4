"""CPU oracle for trust scores (TEST INFRASTRUCTURE): alibi's ``alibi.confidence.TrustScore`` restated with
``sklearn.neighbors.KDTree``, the structure alibi uses, on dense vectors.

What alibi does, restated from its published source (alibi is not installed here, so parity is pinned to this restatement
and stated as unpinned against alibi itself in DESIGN.md):

* ``fit(X, Y)``: per class c, X_fit = X[Y == c] (``filter_type=None``) or ``filter_by_distance_knn(X[Y == c])``, and a KDTree
  over it.  ``filter_by_distance_knn``: ``knn_r = KDTree(X).query(X, k=k_filter + 1)[0]``; "point": ``knn_r[:, -1]``,
  "mean": ``np.mean(knn_r[:, 1:], axis=1)``; keep ``knn_r <= np.percentile(knn_r, (1 - alpha) * 100)``.
* ``score(X, Y, k, dist_type)``: ``d[:, c]`` = the k-th distance ("point") or the mean of the k distances ("mean") of
  ``kdtrees[c].query(X, k=k)``; the distance to the closest class that is not the predicted one, and
  ``trust_score = d_to_closest_not_pred / (d_to_pred + 1e-12)``.  With two classes the closest other class is the other one.
"""

from __future__ import annotations

import numpy as np
from sklearn.neighbors import KDTree

EPS = 1e-12


class TrustScore:
    def __init__(self, k_filter: int = 10, alpha: float = 0.0, filter_type=None, leaf_size: int = 40, dist_filter_type: str = "point"):
        self.k_filter, self.alpha, self.filter, self.leaf_size, self.dist_filter_type = k_filter, alpha, filter_type, leaf_size, dist_filter_type

    def filter_by_distance_knn(self, X: np.ndarray) -> np.ndarray:
        """-> the kept row indices of X (alibi returns the rows themselves)."""
        knn_r = KDTree(X, leaf_size=self.leaf_size).query(X, k=self.k_filter + 1)[0]
        r = knn_r[:, -1] if self.dist_filter_type == "point" else np.mean(knn_r[:, 1:], axis=1)
        return np.where(r <= np.percentile(r, (1 - self.alpha) * 100))[0]

    def fit(self, X: np.ndarray, Y: np.ndarray, classes: int = 2) -> "TrustScore":
        self.classes = classes
        self.kept = []  # per class: the kept row indices of X
        self.kdtrees = []
        for c in range(classes):
            rows = np.where(Y == c)[0]
            if self.filter == "distance_knn":
                rows = rows[self.filter_by_distance_knn(X[rows])]
            self.kept.append(rows)
            self.kdtrees.append(KDTree(X[rows], leaf_size=self.leaf_size))
        return self

    def distances(self, X: np.ndarray, k: int = 2, dist_type: str = "point") -> np.ndarray:
        """(n, classes) D_c."""
        d = np.empty((len(X), self.classes))
        for c in range(self.classes):
            dk = self.kdtrees[c].query(X, k=k)[0]
            d[:, c] = dk[:, -1] if dist_type == "point" else np.mean(dk, axis=1)
        return d

    def score(self, X: np.ndarray, Y: np.ndarray, k: int = 2, dist_type: str = "point"):
        """-> (trust_score, closest_not_pred) for predicted classes Y."""
        d = self.distances(X, k, dist_type)
        sorted_d = np.sort(d, axis=1)
        d_to_pred = d[range(d.shape[0]), Y]
        d_to_closest_not_pred = np.where(sorted_d[:, 0] != d_to_pred, sorted_d[:, 0], sorted_d[:, 1])
        return d_to_closest_not_pred / (d_to_pred + EPS), 1 - Y


def dense(pipe, df, mean=None, scale=None, n_num: int = 14):
    """The classifier's input vectors of ``df`` (sklearn's transform, float32, as scored) with the last ``n_num`` columns
    z-scored by (mean, scale); None: the columns' own mean and population std (scale 1 where it is 0).  -> (X, mean, scale)."""
    X = pipe.named_steps["preprocessor"].transform(df)
    X = (X.toarray() if hasattr(X, "toarray") else np.asarray(X)).astype(np.float32).astype(np.float64)
    if mean is None:
        mean = X[:, -n_num:].mean(axis=0)
        std = X[:, -n_num:].std(axis=0)
        scale = np.where(std > 0.0, std, 1.0)
    X[:, -n_num:] = (X[:, -n_num:] - mean) / scale
    return X, mean, scale
