"""Independent CPU restatement of path-dependent TreeSHAP interaction values (TEST INFRASTRUCTURE).

Lundberg et al., "Consistent Individualized Feature Attribution for Tree Ensembles" (arXiv:1802.03888) §4: the SHAP
interaction value of fields i != j is half the Shapley interaction index, and it is computed there by CONDITIONING.  For
each field j, Algorithm 2 runs over the other fields twice: once with j always known (at a node of j only the row's own
branch is taken) and once with j never known (both branches, weighted by cover); j never enters the path.  Then
``Phi_ij = (phi_i(j on) - phi_i(j off)) / 2`` and ``Phi_jj = phi_j - sum_{i != j} Phi_ij``.  This is independent of the
path-table algebra the kernel uses (UNWIND of one element, then the unwound sum of the other) and of the flattener.

Players, game, output space and rows are ``oracle/treeshap.py``'s.  ``brute_force_interactions`` evaluates the index's
definition with Algorithm 1 over every subset of the fields a tree uses (shallow forests only).
"""

from __future__ import annotations

import itertools
import math

import numpy as np

from oracle import treeshap as ts
from oracle import treewalk as tw


def _conditioned_tree(L, R, F, T, C, V, fields, X32, j, on, phi):
    """Algorithm 2 on one tree with field j conditioned on (``on``) or off; adds its phi (n, n_fields) into ``phi``."""
    n = X32.shape[0]

    def recurse(k, path, pz, po, pi, cond):
        if pi != j:
            path = ts._extend(path, pz, po, pi)
        if L[k] == -1:
            for i in range(1, len(path[0])):
                w = sum(ts._unwind(path, i)[3])
                phi[:, path[0][i]] += w * (path[2][i] - path[1][i]) * V[k] * cond
            return
        f = int(fields[F[k]])
        go_left = X32[:, F[k]].astype(np.float64) <= T[k]
        if f == j:
            if on:
                recurse(L[k], path, 1.0, np.ones(n), f, cond * go_left)
                recurse(R[k], path, 1.0, np.ones(n), f, cond * ~go_left)
            else:
                recurse(L[k], path, 1.0, np.ones(n), f, cond * (C[L[k]] / C[k]))
                recurse(R[k], path, 1.0, np.ones(n), f, cond * (C[R[k]] / C[k]))
            return
        iz, io = 1.0, np.ones(n)
        if f in path[0][1:]:
            q = path[0].index(f, 1)
            iz, io = path[1][q], path[2][q]
            path = ts._unwind(path, q)
        recurse(L[k], path, iz * C[L[k]] / C[k], io * go_left, f, cond)
        recurse(R[k], path, iz * C[R[k]] / C[k], io * ~go_left, f, cond)

    recurse(0, ([], [], [], []), 1.0, np.ones(n), -1, np.ones(n))


def tree_shap_interactions(dump: dict, covers: np.ndarray, X32: np.ndarray):
    """-> (phi2 float64 (n, n_fields, n_fields), base_value) in the model's output space (probability for a RandomForest,
    log-odds for a GBDT).  Fields a tree does not test are null players of that tree and skipped there."""
    fields = ts.column_fields(dump)
    n_fields = int(fields.max()) + 1
    n = X32.shape[0]
    phi2 = np.zeros((n, n_fields, n_fields), dtype=np.float64)
    for t in range(dump["n_trees"]):
        L, R, F, T, C, V = ts._tree(dump, covers, t)
        used = sorted({int(fields[F[k]]) for k in range(len(L)) if L[k] != -1})
        for j in used:
            on = np.zeros((n, n_fields))
            off = np.zeros((n, n_fields))
            _conditioned_tree(L, R, F, T, C, V, fields, X32, j, True, on)
            _conditioned_tree(L, R, F, T, C, V, fields, X32, j, False, off)
            phi2[:, :, j] += (on - off) / 2.0
    phi, base = ts.tree_shap(dump, covers, X32)
    scale = 1.0 / dump["n_trees"] if dump["kind"] == tw.RF_MEAN else 1.0
    phi2 *= scale
    idx = np.arange(n_fields)
    phi2[:, idx, idx] = 0.0
    phi2[:, idx, idx] = phi - phi2.sum(axis=2)
    return phi2, base


def brute_force_interactions(dump: dict, covers: np.ndarray, X32: np.ndarray):
    """The Shapley interaction index from its definition (Algorithm 1 over every subset of the fields each tree uses), halved
    off the diagonal; the diagonal from brute-force Shapley values.  Shallow forests only."""
    fields = ts.column_fields(dump)
    n_fields = int(fields.max()) + 1
    n = X32.shape[0]
    phi2 = np.zeros((n, n_fields, n_fields), dtype=np.float64)
    for t in range(dump["n_trees"]):
        L, R, F, T, C, V = ts._tree(dump, covers, t)
        used = sorted({int(fields[F[k]]) for k in range(len(L)) if L[k] != -1})
        if len(used) > 12:
            raise ValueError("brute force is for shallow trees")
        U = len(used)
        v = {}
        for k in range(U + 1):
            for S in itertools.combinations(used, k):
                v[frozenset(S)] = ts._expvalue(L, R, F, T, C, V, fields, X32, set(S))
        for i, j in itertools.combinations(used, 2):
            others = [f for f in used if f != i and f != j]
            acc = np.zeros(n)
            for k in range(U - 1):
                wgt = math.factorial(k) * math.factorial(U - k - 2) / (2.0 * math.factorial(U - 1))
                for S in itertools.combinations(others, k):
                    s = frozenset(S)
                    acc += wgt * (v[s | {i, j}] - v[s | {i}] - v[s | {j}] + v[s])
            phi2[:, i, j] += acc
            phi2[:, j, i] += acc
    phi, base = ts.brute_force_shap(dump, covers, X32)
    if dump["kind"] == tw.RF_MEAN:
        phi2 /= dump["n_trees"]
    idx = np.arange(n_fields)
    phi2[:, idx, idx] = phi - phi2.sum(axis=2)
    return phi2, base
