"""Independent CPU restatement of interventional TreeSHAP against a background set (TEST INFRASTRUCTURE).

Lundberg et al., "From local explanations to global understanding with explainable AI for trees" (Nat. Mach. Intell. 2020,
arXiv:1905.04610): for a row x and a background row z, the Shapley values of v_z(S) = f(x_S, z_rest) come from one recursion
over each tree.  At a node on field f: if f was already given to x's side (A) the walk follows x, if to z's side (B) it
follows z; if x and z take the same child it goes there; otherwise it goes to x's child with f in A and to z's child with f
in B.  A leaf reached with |A| = a, |B| = b gives each field of A +leaf (a-1)! b! / (a+b)! and each field of B
-leaf a! (b-1)! / (a+b)!.  phi(x) is the mean over z.

Written from the paper on the arrays of ``oracle/treewalk.dump_pipeline``, fields as players (every one-hot column of a
categorical field maps to that field, as in ``oracle/treeshap.py``), independently of the path table.  Every node is visited
once per tree with the state of all (x, z) pairs at once: a pair reaches a node in at most one state, since the path to it
fixes, node by node, which side must take each branch; only the pairs that reach a node are carried into it.  ``interventional_bruteforce`` enumerates coalitions instead.
"""

from __future__ import annotations

import itertools
import math

import numpy as np

from oracle import treeshap as ts
from oracle import treewalk as tw


def _w(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """(a-1)! b! / (a+b)! elementwise, 0 where a = 0."""
    out = np.zeros(np.broadcast(a, b).shape)
    for (x, y) in {(int(x), int(y)) for x, y in zip(np.ravel(a), np.ravel(b))}:
        if x:
            out[(a == x) & (b == y)] = math.factorial(x - 1) * math.factorial(y) / math.factorial(x + y)
    return out


def output(dump: dict, X32: np.ndarray) -> np.ndarray:
    """f in the output space: probability (RandomForest) or raw margin (GBDT)."""
    p, _, raw = tw.walk_numpy(dump, X32)
    return p if dump["kind"] == tw.RF_MEAN else raw


def interventional_shap(dump: dict, X: np.ndarray, Z: np.ndarray):
    """-> (phi float64 (n, n_fields), base_value = mean f(Z)) for dense rows X (n, cols) against background Z (m, cols)."""
    fields = ts.column_fields(dump)
    n_fields = int(fields.max()) + 1
    n, m = X.shape[0], Z.shape[0]
    Xp = np.repeat(X, m, axis=0)  # pair i * m + j = (x_i, z_j)
    Zp = np.tile(Z, (n, 1))
    phi = np.zeros((n * m, n_fields))
    for t in range(dump["n_trees"]):
        lo, hi = int(dump["tree_off"][t]), int(dump["tree_off"][t + 1])
        L, R, Fc, T = dump["left"][lo:hi], dump["right"][lo:hi], dump["feature"][lo:hi], dump["threshold"][lo:hi]
        V = dump["value"][lo:hi] if dump["kind"] == tw.RF_MEAN else dump["scale"] * dump["value"][lo:hi]
        # (node, the pairs that reach it, their A and B): a pair reaching no node of a subtree is not carried into it
        stack = [(0, np.arange(n * m), np.zeros((n * m, n_fields), bool), np.zeros((n * m, n_fields), bool))]
        while stack:
            j, idx, A, B = stack.pop()
            if len(idx) == 0:
                continue
            if L[j] == -1:
                a, b = A.sum(axis=1), B.sum(axis=1)
                phi[idx] += V[j] * (A * _w(a, b)[:, None] - B * _w(b, a)[:, None])
                continue
            f = int(fields[Fc[j]])
            xl = Xp[idx, Fc[j]].astype(np.float64) <= T[j]
            zl = Zp[idx, Fc[j]].astype(np.float64) <= T[j]
            for child, xg, zg in ((L[j], xl, zl), (R[j], ~xl, ~zl)):
                x_only, z_only = xg & ~zg, zg & ~xg
                # neither side goes there, or only the side f was not given to: the pair does not reach the child
                ok = (xg | zg) & ~(x_only & B[:, f]) & ~(z_only & A[:, f])
                nA, nB = A[ok], B[ok]
                nA[:, f] |= x_only[ok]
                nB[:, f] |= z_only[ok]
                stack.append((child, idx[ok], nA, nB))
    if dump["kind"] == tw.RF_MEAN:
        phi /= dump["n_trees"]
    return phi.reshape(n, m, n_fields).mean(axis=1), float(output(dump, Z).mean())


def interventional_bruteforce(dump: dict, X: np.ndarray, Z: np.ndarray, max_fields: int = 10):
    """Shapley values from the definition for every pair: v(S) = f(hybrid) with the columns of the fields in S from x and the
    rest from z, over the coalitions of the fields where x and z differ (at most ``max_fields`` of them)."""
    fields = ts.column_fields(dump)
    n_fields = int(fields.max()) + 1
    phi = np.zeros((X.shape[0], n_fields))
    for i, x in enumerate(X):
        for z in Z:
            D = sorted({int(fields[c]) for c in np.nonzero(x.view(np.uint32) != z.view(np.uint32))[0]})
            if len(D) > max_fields:
                raise ValueError(f"the pair differs in {len(D)} fields")
            subsets = [frozenset(S) for k in range(len(D) + 1) for S in itertools.combinations(D, k)]
            H = np.repeat(z[None, :], len(subsets), axis=0)
            for r, S in enumerate(subsets):
                cols = np.isin(fields, list(S))
                H[r, cols] = x[cols]
            v = dict(zip(subsets, output(dump, H)))
            d = len(D)
            for f in D:
                for S in subsets:
                    if f in S:
                        continue
                    k = len(S)
                    phi[i, f] += math.factorial(k) * math.factorial(d - k - 1) / math.factorial(d) * (v[S | {f}] - v[S])
    return phi / Z.shape[0], float(output(dump, Z).mean())
