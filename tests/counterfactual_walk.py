"""numpy emulation of k_counterfactual / k_counterfactual_finish (csrc/counterfactual.cuh) over a forest blob (TEST
INFRASTRUCTURE).

Split values are read from the blob's node words on their own (not through the library), every piece of a probed word is
scored at its representative by ``dependence_walk.pd_walk`` (K6's walk, one representative per piece), and a plain
reduction picks the nearest flips on each side of the row's own piece.  Nothing in the product imports it.
"""

import numpy as np

from databricks_kubernetes_mlops_poc_b200.flatten import META_CAT, META_FEAT_SHIFT, META_SLOT_MASK, SENTINEL_WORD, parse_header
from dependence_walk import pd_walk


def split_values(blob: bytes, word: int) -> np.ndarray:
    """Sorted distinct float32 split values t' of row word ``word`` over every tree of the blob (-0.0 and +0.0 once)."""
    h = parse_header(blob)
    buf = np.frombuffer(blob, dtype=np.uint8)
    vals = []
    for g in h["groups"]:
        base = h["chunks_off"] + g["chunk_off"]
        N = buf[base:base + g["n_slots"] * 256].view(np.uint32).reshape(g["n_slots"], 32, 2)[:, :g["n_trees"]]
        T, M = N[..., 0], N[..., 1]
        slot = np.arange(g["n_slots"], dtype=np.uint32)[:, None]
        sel = ((M & META_SLOT_MASK) != slot) & ((M & META_CAT) == 0) & ((M >> META_FEAT_SHIFT) == word) & (word != SENTINEL_WORD)
        vals.append(T[sel].view(np.float32))
    v = np.concatenate(vals) if vals else np.empty(0, np.float32)
    return np.unique(v)


def representatives(t: np.ndarray) -> np.ndarray:
    """One float32 per piece: nextdown(t'_0) for piece 0, t'_{k-1} for piece k >= 1; 0 for the one piece of an unsplit word."""
    if len(t) == 0:
        return np.zeros(1, np.float32)
    return np.concatenate([[np.nextafter(t[0], np.float32(-np.inf))], t]).astype(np.float32)


def imputed(blob: bytes, rows: np.ndarray) -> np.ndarray:
    """(n, 24) uint32 rows -> their float32 words as scored (NaN numerics -> the blob's imputation values)."""
    h = parse_header(blob)
    f = np.ascontiguousarray(rows, dtype=np.uint32).copy().view(np.float32)
    lo, hi = h["n_cat"], h["n_cat"] + h["n_num"]
    nan = np.isnan(f[:, lo:hi])
    f[:, lo:hi][nan] = np.broadcast_to(h["impute"][lo:hi], nan.shape)[nan]
    return f


def piece_scores(blob: bytes, rows: np.ndarray, word: int):
    """-> (t', p1 float64 (n, m + 1)): every piece of ``word`` scored at its representative by K6's walk."""
    t = split_values(blob, word)
    reps = representatives(t)
    out, _ = pd_walk(blob, rows, [(word, 0, len(reps))], reps.view(np.uint32))
    return t, out


def reduce(t: np.ndarray, p: np.ndarray, x: np.ndarray, cutoff: float):
    """Piece scores p (n, m + 1) and the rows' values x (n,) -> (p1_j, lower, lower_p1, upper, upper_p1), NaN = none."""
    n, m = len(x), len(t)
    j = np.where(np.isnan(x), m, np.searchsorted(t, x, side="right"))
    pj = p[np.arange(n), j]
    res = np.full((4, n), np.nan)
    for i in range(n):
        flip = (p[i] > cutoff) != (pj[i] > cutoff)
        below, above = np.flatnonzero(flip[:j[i]]), np.flatnonzero(flip[j[i] + 1:]) + j[i] + 1
        if len(below):
            k = below[-1]
            res[0, i], res[1, i] = np.nextafter(t[k], np.float32(-np.inf)), p[i, k]
        if len(above):
            k = above[0]
            res[2, i], res[3, i] = t[k - 1], p[i, k]
    return pj, res[0], res[1], res[2], res[3]


def counterfactual(blob: bytes, rows: np.ndarray, words, cutoff: float = 0.5, cache: dict | None = None):
    """What b2f_counterfactual returns: (proba (n,), records (n, len(words)) with the fields of COUNTERFACTUAL_DTYPE).
    ``cache`` (word -> piece_scores of these rows) lets several cutoffs share one walk per word."""
    from databricks_kubernetes_mlops_poc_b200._cabi import COUNTERFACTUAL_DTYPE

    rows = np.ascontiguousarray(rows, dtype=np.uint32)
    x = imputed(blob, rows)
    out = np.zeros((len(rows), len(words)), dtype=COUNTERFACTUAL_DTYPE)
    proba = None
    for f, w in enumerate(words):
        if cache is None or w not in cache:
            scored = piece_scores(blob, rows, w)
            if cache is not None:
                cache[w] = scored
        t, p = cache[w] if cache is not None else scored
        pj, lo, plo, hi, phi = reduce(t, p, x[:, w], cutoff)
        proba = pj if proba is None else proba
        out["value"][:, f], out["lower"][:, f], out["lower_p1"][:, f] = x[:, w], lo, plo
        out["upper"][:, f], out["upper_p1"][:, f] = hi, phi
    return proba, out
