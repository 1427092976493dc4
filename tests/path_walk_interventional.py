"""numpy emulation of interventional TreeSHAP over the path table and its background table (TEST INFRASTRUCTURE).

Mirrors ``csrc/tree_shap_interventional.cuh``: per path, the background rows' masks (bit k: the row satisfies element k, the
prediction kernels' test of ``path_walk.one_fractions``; bit 0 the bias, always set) as distinct masks with counts in mask
order for paths of up to 12 field elements, else one entry of count 1 per row in row order; then, per row x with mask Fx,
the entries covering every element x fails, with A = Fx minus the entry and B = the elements x fails, and the weights
W[x][y] = 1 / (x C(x+y, y)) of the kernel's table.  Nothing in the product imports it.
"""

import math

import numpy as np

from databricks_kubernetes_mlops_poc_b200.flatten import parse_explainer
from path_walk import one_fractions, row_words

HIST_LEN = 12
L = 24
W = np.array([[0.0 if x == 0 else 1.0 / (x * math.comb(x + y, y)) for y in range(L)] for x in range(L)])


def _masks(h, w: np.ndarray, p: int) -> np.ndarray:
    """(n,) int64 masks of the rows w (imputed words) on path p."""
    P, E = h["paths"], h["elems"]
    first, ln = int(P["first"][p]), int(P["len"][p])
    o = one_fractions(E[first + 1 : first + ln], w).astype(np.int64)  # (d, n)
    return 1 + (o << np.arange(1, ln, dtype=np.int64)[:, None]).sum(axis=0)


def background_table(paths: bytes, blob: bytes, bg_rows: np.ndarray):
    """-> (offsets int64 (P + 1,), masks uint32, counts uint32, table_bytes, base_value) as b2f_model_attach_background builds them."""
    h = parse_explainer(paths)
    w = row_words(blob, bg_rows)
    n = w.shape[0]
    P = h["paths"]
    offs, masks, counts = [0], [], []
    moved = 0.0
    for p in range(h["n_paths"]):
        ln = int(P["len"][p])
        m = _masks(h, w, p)
        if ln - 1 <= HIST_LEN:
            u, c = np.unique(m, return_counts=True)
        else:
            u, c = m, np.ones(n, np.int64)
        masks.append(u.astype(np.uint32))
        counts.append(c.astype(np.uint32))
        offs.append(offs[-1] + len(u))
        first = int(P["first"][p])
        pz = np.prod(h["elems"]["zero_fraction"][first + 1 : first + ln])
        reach = int((m == (1 << ln) - 1).sum())
        moved += float(P["leaf"][p]) * (reach / n - pz)
    offs = np.asarray(offs, np.int64)
    cat = lambda xs: np.concatenate(xs) if xs else np.zeros(0, np.uint32)  # noqa: E731
    masks, counts = cat(masks), cat(counts)
    return offs, masks, counts, 8 * len(offs) + 8 * len(masks), h["base_value"] + moved / h["denom"]


def explain_interventional(paths: bytes, blob: bytes, rows: np.ndarray, bg_rows: np.ndarray):
    """-> (phi float64 (n, n_cat + n_num), base_value, table_bytes), the kernel's algorithm in numpy."""
    h = parse_explainer(paths)
    F = h["n_cat"] + h["n_num"]
    offs, masks, counts, nbytes, base = background_table(paths, blob, bg_rows)
    w = row_words(blob, rows)
    n = w.shape[0]
    phi = np.zeros((n, F))
    P, E = h["paths"], h["elems"]
    for p in range(h["n_paths"]):
        first, ln, leaf = int(P["first"][p]), int(P["len"][p]), float(P["leaf"][p])
        fx = _masks(h, w, p)  # (n,)
        need = ((1 << ln) - 1) & ~fx
        b = np.array([bin(int(v)).count("1") for v in need])
        m = masks[offs[p] : offs[p + 1]].astype(np.int64)
        c = counts[offs[p] : offs[p + 1]].astype(np.float64)
        valid = (m[None, :] & need[:, None]) == need[:, None]  # (n, e)
        am = fx[:, None] & ~m[None, :]
        a = np.zeros(am.shape, np.int64)
        for k in range(1, ln):
            a += (am >> k) & 1
        sb = np.where(valid, c[None, :] * W[b[:, None], a], 0.0).sum(axis=1)
        wa = np.where(valid, c[None, :] * W[a, b[:, None]], 0.0)
        for k in range(1, ln):
            f = int(E["field"][first + k])
            sa = np.where((am >> k) & 1 == 1, wa, 0.0).sum(axis=1)
            phi[:, f] += np.where((fx >> k) & 1 == 1, sa, -sb) * leaf
    return phi / (h["denom"] * bg_rows.shape[0]), base, nbytes
