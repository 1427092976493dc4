"""numpy emulation of the TreeSHAP kernel's semantics over a path table (TEST INFRASTRUCTURE).

Mirrors ``csrc/tree_shap.cuh``: the one-fraction of each merged path element is the prediction kernels' compare on the
imputed row word (numeric: ``geu(x, lo) and (no upper bound or x < hi)``; categorical: bit ``code + 1`` of the mask, codes
outside ``[-1, 126]`` read bit 0), then EXTEND over the path's elements and the closed-form UNWIND sum per element, with the
``(i+1)/(l+1)``, ``(l-i)/(l+1)``, ``(l+1)/(i+1)`` and ``(l+1)/(l-i)`` factors from the same tables and ``1/zero_fraction`` from
the table.  Vectorised over (paths of one length) x rows, so the flattener is pinned on a CPU-only box.  Nothing in the
product imports it.
"""

import numpy as np

from databricks_kubernetes_mlops_poc_b200.flatten import PE_CAT, PE_HAS_HI, parse_explainer, parse_header

MAXL = 24
_l = np.arange(MAXL)[:, None].astype(np.float64)
_i = np.arange(MAXL)[None, :].astype(np.float64)
with np.errstate(divide="ignore"):
    EXT_A = (_i + 1) / (_l + 1)
    EXT_B = (_l - _i) / (_l + 1)
    UNW_C = (_l + 1) / (_i + 1)
    UNW_D = (_l + 1) / (_l - _i)


def row_words(blob: bytes, rows: np.ndarray) -> np.ndarray:
    """(n, 24) uint32 rows -> imputed row words, as the kernels read them."""
    h = parse_header(blob)
    n_cat, n_num = h["n_cat"], h["n_num"]
    w = np.ascontiguousarray(rows, dtype=np.uint32).copy()
    f = w.view(np.float32)
    nan = np.isnan(f[:, n_cat : n_cat + n_num])
    imp = np.broadcast_to(h["impute"][n_cat : n_cat + n_num], nan.shape)
    f[:, n_cat : n_cat + n_num][nan] = imp[nan]
    return w


def one_fractions(el, w: np.ndarray) -> np.ndarray:
    """(k,) path elements x (n, 24) row words -> (k, n) 0/1 float64."""
    x = w[:, np.minimum(el["field"], 23).astype(np.int64)].T  # (k, n) uint32; bias elements read the padding word, unused
    xf = x.view(np.float32)
    with np.errstate(invalid="ignore"):
        geu = ~(xf < el["lo"][:, None])
        below = (xf < el["hi"][:, None]) | ((el["kind"] & PE_HAS_HI) == 0)[:, None]
    num = geu & below
    code = x.view(np.int32).astype(np.int64)
    bit = np.where((code >= -1) & (code <= 126), code + 1, 0)
    word = np.take_along_axis(el["mask"].astype(np.uint64), bit // 32, axis=1)
    cat = ((word >> (bit % 32).astype(np.uint64)) & 1) == 1
    return np.where(((el["kind"] & PE_CAT) != 0)[:, None], cat, num).astype(np.float64)


def explain_paths(paths: bytes, blob: bytes, rows: np.ndarray):
    """-> (phi float64 (n, n_cat + n_num), base_value), the kernel's algorithm in numpy."""
    h = parse_explainer(paths)
    F = h["n_cat"] + h["n_num"]
    w = row_words(blob, rows)
    n = w.shape[0]
    phi = np.zeros((n, F), dtype=np.float64)
    P, E = h["paths"], h["elems"]
    for L in np.unique(P["len"]):
        sel = P[P["len"] == L]
        d = int(L) - 1
        idx = sel["first"][:, None].astype(np.int64) + np.arange(L)[None, :]  # (p, L)
        el = E[idx.reshape(-1)]
        o = one_fractions(el, w).reshape(len(sel), L, n)
        z = el["zero_fraction"].reshape(len(sel), L)
        iz = el["inv_zero_fraction"].reshape(len(sel), L)
        fld = el["field"].reshape(len(sel), L).astype(np.int64)
        pw = np.zeros((len(sel), L, n))
        pw[:, 0] = 1.0  # the bias element: zero = one = 1
        for l in range(1, L):
            ol, zl = o[:, l], z[:, l][:, None]
            for i in range(l - 1, -1, -1):
                pw[:, i + 1] += ol * pw[:, i] * EXT_A[l, i]
                pw[:, i] = zl * pw[:, i] * EXT_B[l, i]
        leaf = sel["leaf"][:, None]
        for k in range(1, L):
            ok, zk, izk = o[:, k], z[:, k][:, None], iz[:, k][:, None]
            nxt = pw[:, d].copy()
            tot1 = np.zeros((len(sel), n))
            tot0 = np.zeros((len(sel), n))
            for i in range(d - 1, -1, -1):
                tmp = nxt * UNW_C[d, i]
                tot1 += tmp
                nxt = pw[:, i] - tmp * zk * EXT_B[d, i]
                tot0 += pw[:, i] * izk * UNW_D[d, i]
            tot = np.where(ok == 1.0, tot1, tot0)
            contrib = tot * (ok - zk) * leaf
            np.add.at(phi.T, fld[:, k], contrib)
    return phi / h["denom"], h["base_value"]
