"""numpy emulation of the TreeSHAP interaction kernel over a path table (TEST INFRASTRUCTURE).

Mirrors ``csrc/tree_shap_interactions.cuh`` on top of ``path_walk`` (row words, one-fractions, the same factor tables):
per path, EXTEND over its merged elements; per element a, UNWIND a (its unwound sum is phi_a's term), then for every
element b of a higher field K5's closed-form unwound sum of b over the unwound polynomial gives the pair term
``leaf (o_a - z_a)(o_b - z_b) / 2 * sum``, stored once for the unordered pair.  The diagonal is ``phi_a - sum_{b != a}
Phi_ab``.  Vectorised over (paths of one length) x rows.  Nothing in the product imports it.
"""

import numpy as np

from databricks_kubernetes_mlops_poc_b200.flatten import parse_explainer
from path_walk import EXT_A, EXT_B, UNW_C, UNW_D, one_fractions, row_words


def _closed_sum(pw, l, o, z, iz):
    """K5's closed-form sum of the polynomial pw[:, 0..l] with one element (one-fraction o, zero-fraction z) unwound."""
    nxt = pw[:, l].copy()
    tot1 = np.zeros_like(nxt)
    tot0 = np.zeros_like(nxt)
    for i in range(l - 1, -1, -1):
        tmp = nxt * UNW_C[l, i]
        tot1 += tmp
        nxt = pw[:, i] - tmp * z * EXT_B[l, i]
        tot0 += pw[:, i] * iz * UNW_D[l, i]
    return np.where(o == 1.0, tot1, tot0)


def explain_interactions_paths(paths: bytes, blob: bytes, rows: np.ndarray):
    """-> (phi2 float64 (n, F, F), base_value), the kernel's algorithm in numpy."""
    h = parse_explainer(paths)
    F = h["n_cat"] + h["n_num"]
    w = row_words(blob, rows)
    n = w.shape[0]
    tri = np.zeros((n, F * F))  # slot a * F + b, a <= b: the kernel's upper triangle (phi_a on the diagonal)
    P, E = h["paths"], h["elems"]
    for L in np.unique(P["len"]):
        sel = P[P["len"] == L]
        d = int(L) - 1
        idx = sel["first"][:, None].astype(np.int64) + np.arange(L)[None, :]
        el = E[idx.reshape(-1)]
        o = one_fractions(el, w).reshape(len(sel), L, n)
        z = el["zero_fraction"].reshape(len(sel), L)
        iz = el["inv_zero_fraction"].reshape(len(sel), L)
        fld = el["field"].reshape(len(sel), L).astype(np.int64)
        pw = np.zeros((len(sel), L, n))
        pw[:, 0] = 1.0
        for l in range(1, L):
            ol, zl = o[:, l], z[:, l][:, None]
            for i in range(l - 1, -1, -1):
                pw[:, i + 1] += ol * pw[:, i] * EXT_A[l, i]
                pw[:, i] = zl * pw[:, i] * EXT_B[l, i]
        leaf = sel["leaf"][:, None]
        for ka in range(1, L):
            oa, za, iza = o[:, ka], z[:, ka][:, None], iz[:, ka][:, None]
            # UNWIND a: wa[:, 0..d-1]
            wa = np.zeros((len(sel), d, n))
            nxt = pw[:, d].copy()
            for i in range(d - 1, -1, -1):
                w1 = nxt * UNW_C[d, i]
                nxt = pw[:, i] - w1 * za * EXT_B[d, i]
                wa[:, i] = np.where(oa == 1.0, w1, pw[:, i] * iza * UNW_D[d, i])
            tot = np.zeros((len(sel), n))
            for i in range(d - 1, -1, -1):
                tot += wa[:, i]
            ga = (oa - za) * leaf
            np.add.at(tri.T, fld[:, ka] * (F + 1), tot * ga)
            for kb in range(1, L):
                if kb == ka:
                    continue
                up = fld[:, kb] > fld[:, ka]
                if not up.any():
                    continue
                ob, zb, izb = o[up, kb], z[up, kb][:, None], iz[up, kb][:, None]
                t = _closed_sum(wa[up], d - 1, ob, zb, izb)
                np.add.at(tri.T, fld[up, ka] * F + fld[up, kb], t * (0.5 * ga[up]) * (ob - zb))
    tri = tri.reshape(n, F, F)
    diag = np.diagonal(tri, axis1=1, axis2=2).copy()
    off = np.triu(tri, 1)
    full = off + np.transpose(off, (0, 2, 1))
    a = np.arange(F)
    full[:, a, a] = diag - full.sum(axis=2)
    return full / h["denom"], h["base_value"]
