"""Independent CPU restatement of path-dependent TreeSHAP (TEST INFRASTRUCTURE).

Lundberg et al., "Consistent Individualized Feature Attribution for Tree Ensembles" (arXiv:1802.03888): Algorithm 1
(the conditional expectation ``v(S)`` of one tree) and Algorithm 2 (polynomial-time exact Shapley values of that game,
with EXTEND / UNWIND of the unique path and the unwinding of a feature met twice on one path).  Written from the paper,
on the arrays of ``treewalk.dump_pipeline`` plus each node's cover (``tree_.weighted_n_node_samples``).

Players are REQUEST FIELDS, not the columns the trees see: every one-hot column of a categorical field maps to that
field, so ``v(S)`` follows the row's branch at every node of a field in ``S`` and averages over both children (weighted by
cover) at every other node.  Rows enter as the dense float32 matrix ``treewalk.transform_dense`` builds, so NaN
imputation and unknown categories are exactly what the forest sees.

Both algorithms are vectorised over rows: every node is visited for every row and only the one-fractions (which branch
the row takes) differ per row, so the recursion runs once per tree on ``(path length, n)`` arrays.
"""

from __future__ import annotations

import itertools
import math

import numpy as np

from . import treewalk as tw


def dump_covers(pipeline) -> np.ndarray:
    """Per node cover (``tree_.weighted_n_node_samples``), concatenated in ``dump_pipeline``'s node order."""
    clf = pipeline.named_steps["classifier"]
    if clf.__class__.__name__ == "RandomForestClassifier":
        trees = [e.tree_ for e in clf.estimators_]
    else:
        trees = [e.tree_ for e in clf.estimators_[:, 0]]
    return np.concatenate([t.weighted_n_node_samples.astype(np.float64) for t in trees])


def column_fields(dump: dict) -> np.ndarray:
    """Dense column -> request field (categorical fields first, in ``all_features`` order, then the numerics)."""
    offs = dump["cat_offsets"]
    n_ohe = int(offs[-1])
    n_cat = len(offs) - 1
    n_num = len(dump["medians"])
    f = np.empty(n_ohe + n_num, dtype=np.int64)
    f[:n_ohe] = np.searchsorted(offs, np.arange(n_ohe), side="right") - 1
    f[n_ohe:] = n_cat + np.arange(n_num)
    return f


def _leaf_payload(dump: dict, t: int) -> np.ndarray:
    lo, hi = int(dump["tree_off"][t]), int(dump["tree_off"][t + 1])
    v = dump["value"][lo:hi]
    return v if dump["kind"] == tw.RF_MEAN else dump["scale"] * v


def _tree(dump, covers, t):
    lo, hi = int(dump["tree_off"][t]), int(dump["tree_off"][t + 1])
    return (dump["left"][lo:hi], dump["right"][lo:hi], dump["feature"][lo:hi], dump["threshold"][lo:hi], covers[lo:hi],
            _leaf_payload(dump, t))


def _extend(path, pz, po, pi):
    """EXTEND: path = (fields list, zero list, one list of (n,) arrays, weight list of (n,) arrays); returns a new path."""
    d, z, o, w = list(path[0]), list(path[1]), list(path[2]), [x.copy() for x in path[3]]
    l = len(d)
    d.append(pi)
    z.append(pz)
    o.append(po)
    w.append(np.ones_like(po) if l == 0 else np.zeros_like(po))
    for i in range(l - 1, -1, -1):
        w[i + 1] = w[i + 1] + po * w[i] * (i + 1) / (l + 1)
        w[i] = pz * w[i] * (l - i) / (l + 1)
    return d, z, o, w


def _unwind(path, i):
    """UNWIND element i out of the path (vectorised over rows: its one-fraction is 0 or 1 per row)."""
    d, z, o, w = list(path[0]), list(path[1]), list(path[2]), [x.copy() for x in path[3]]
    l = len(d) - 1
    oi, zi = o[i], z[i]
    one = oi != 0
    nxt = w[l].copy()
    for j in range(l - 1, -1, -1):
        with np.errstate(divide="ignore", invalid="ignore"):
            t = w[j]
            w_one = nxt * (l + 1) / ((j + 1) * np.where(one, oi, 1.0))
            nxt = np.where(one, t - w_one * zi * (l - j) / (l + 1), nxt)
            w_zero = (t * (l + 1)) / (zi * (l - j))
        w[j] = np.where(one, w_one, w_zero)
    for j in range(i, l):
        d[j], z[j], o[j] = d[j + 1], z[j + 1], o[j + 1]
    return d[:l], z[:l], o[:l], w[:l]


def tree_shap(dump: dict, covers: np.ndarray, X32: np.ndarray):
    """Algorithm 2 over every tree -> (phi float64 (n, n_fields), base_value) in the model's output space: probability
    for a RandomForest (mean over trees), log-odds for a GBDT (init + sum over trees of lr * leaf)."""
    fields = column_fields(dump)
    n_fields = int(fields.max()) + 1
    n = X32.shape[0]
    phi = np.zeros((n, n_fields), dtype=np.float64)
    base = 0.0
    for t in range(dump["n_trees"]):
        L, R, F, T, C, V = _tree(dump, covers, t)

        def recurse(j, path, pz, po, pi):
            path = _extend(path, pz, po, pi)
            if L[j] == -1:
                for i in range(1, len(path[0])):
                    w = sum(_unwind(path, i)[3])
                    phi[:, path[0][i]] += w * (path[2][i] - path[1][i]) * V[j]
                return
            f = int(fields[F[j]])
            go_left = X32[:, F[j]].astype(np.float64) <= T[j]
            iz, io = 1.0, np.ones(n)
            if f in path[0][1:]:
                k = path[0].index(f, 1)
                iz, io = path[1][k], path[2][k]
                path = _unwind(path, k)
            recurse(L[j], path, iz * C[L[j]] / C[j], io * go_left, f)
            recurse(R[j], path, iz * C[R[j]] / C[j], io * ~go_left, f)

        recurse(0, ([], [], [], []), 1.0, np.ones(n), -1)
        leaves = L == -1
        base += float(np.dot(V[leaves], C[leaves] / C[0]))
    if dump["kind"] == tw.RF_MEAN:
        return phi / dump["n_trees"], base / dump["n_trees"]
    return phi, dump["init_raw"] + base


# ---------------------------------------------------------------------------------------------------------- brute force
def _expvalue(L, R, F, T, C, V, fields, X32, S):
    """Algorithm 1: v(S) of one tree for every row (cover-weighted average over both children off S)."""
    n = X32.shape[0]

    def g(j, w):
        if L[j] == -1:
            return w * V[j]
        if int(fields[F[j]]) in S:
            left = X32[:, F[j]].astype(np.float64) <= T[j]
            return g(L[j], w * left) + g(R[j], w * ~left)
        return g(L[j], w * (C[L[j]] / C[j])) + g(R[j], w * (C[R[j]] / C[j]))

    return g(0, np.ones(n))


def brute_force_shap(dump: dict, covers: np.ndarray, X32: np.ndarray):
    """Shapley values from the definition, summed over every subset of the fields each tree uses (shallow forests only:
    2^|fields of a tree| evaluations of Algorithm 1 per tree)."""
    fields = column_fields(dump)
    n_fields = int(fields.max()) + 1
    n = X32.shape[0]
    phi = np.zeros((n, n_fields), dtype=np.float64)
    base = 0.0
    for t in range(dump["n_trees"]):
        L, R, F, T, C, V = _tree(dump, covers, t)
        used = sorted({int(fields[F[j]]) for j in range(len(L)) if L[j] != -1})
        if len(used) > 12:
            raise ValueError("brute force is for shallow trees")
        U = len(used)
        v = {}
        for k in range(U + 1):
            for S in itertools.combinations(used, k):
                v[frozenset(S)] = _expvalue(L, R, F, T, C, V, fields, X32, set(S))
        base += float(v[frozenset()][0]) if n else 0.0
        for i in used:
            others = [f for f in used if f != i]
            for k in range(U):
                wgt = math.factorial(k) * math.factorial(U - k - 1) / math.factorial(U)
                for S in itertools.combinations(others, k):
                    s = frozenset(S)
                    phi[:, i] += wgt * (v[s | {i}] - v[s])
    if dump["kind"] == tw.RF_MEAN:
        return phi / dump["n_trees"], base / dump["n_trees"]
    return phi, dump["init_raw"] + base
