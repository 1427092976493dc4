"""numpy emulation of b2f_permutation_scores (csrc/permutation_importance.cuh) over a forest blob (TEST INFRASTRUCTURE).

Each (field, repeat) materialises the substituted rows -- word f of row i taken from row perm[r, i] -- and scores them
with K6's arithmetic: a tree-order sum from the GBDT init value, then the aggregate of ``forest_predict.cuh``
(``tree_order_scores``, which a CPU test pins to ``dependence_walk.pd_walk`` row by row).  The records are then counted
from the scores the way the kernels count them: confusion counts of the predicted label, the clipped log-loss and Brier
sums, and twice the Mann-Whitney statistic of the ranking key (P(class 1) for a RandomForest, the raw margin for a GBDT).
Nothing in the product imports it.
"""

import numpy as np

from databricks_kubernetes_mlops_poc_b200.flatten import META_CAT, META_FEAT_SHIFT, META_SLOT_MASK, SENTINEL_BITS, SENTINEL_WORD, parse_header

EPS = np.finfo(np.float64).eps


def tree_order_scores(blob: bytes, rows: np.ndarray):
    """(n, 24) uint32 rows -> (p1, label, key) per row: the tile kernel's tree-order sum, aggregated; key = p1 for a
    RandomForest and the raw margin for a GBDT."""
    h = parse_header(blob)
    n = rows.shape[0]
    n_cat, n_num = h["n_cat"], h["n_num"]
    w = np.ascontiguousarray(rows, dtype=np.uint32).copy()
    f = w.view(np.float32)
    nan = np.isnan(f[:, n_cat:n_cat + n_num])
    f[:, n_cat:n_cat + n_num][nan] = np.broadcast_to(h["impute"][n_cat:n_cat + n_num], nan.shape)[nan]
    w[:, SENTINEL_WORD] = SENTINEL_BITS
    gbdt = h["agg_mode"] == 1
    acc = np.full(n, h["init_raw"] if gbdt else 0.0)
    buf = np.frombuffer(blob, dtype=np.uint8)
    ridx = np.arange(n)
    for g in h["groups"]:
        base = h["chunks_off"] + g["chunk_off"]
        ns, nl = g["n_slots"], g["n_leaf_slots"]
        N = buf[base:base + ns * 256].view(np.uint32).reshape(ns, 32, 2)
        LV = buf[base + ns * 256:base + ns * 256 + nl * 256].view(np.float64).reshape(nl, 32)
        for lane in range(g["n_trees"]):  # tree order
            T, M = N[:, lane, 0], N[:, lane, 1]
            node = np.zeros(n, dtype=np.int64)
            for _ in range(g["depth"] + 1):
                m, t = M[node], T[node]
                first = (m & np.uint32(META_SLOT_MASK)).astype(np.int64)
                leaf = first == node
                x = w[ridx, (m >> META_FEAT_SHIFT).astype(np.int64) % w.shape[1]]
                with np.errstate(invalid="ignore"):
                    geu = ~(x.view(np.float32) < t.view(np.float32))
                second = (x == t) | (geu & ((m & META_CAT) == 0))
                node = np.where(leaf, node, first + second.astype(np.int64))
            acc += LV[T[node].astype(np.int64), lane]
    if gbdt:
        raw = 0.0 + acc
        return 1.0 / (1.0 + np.exp(-raw)), (raw >= 0).astype(np.int32), raw
    p1 = acc / h["denom"]
    return p1, (acc > h["denom"] - acc).astype(np.int32), p1


def record(p1: np.ndarray, label: np.ndarray, key: np.ndarray, y: np.ndarray):
    """One b2f_perm_score (as a PERM_SCORE_DTYPE scalar) from a point's scores and the labels."""
    from databricks_kubernetes_mlops_poc_b200._cabi import PERM_SCORE_DTYPE

    r = np.zeros((), dtype=PERM_SCORE_DTYPE)
    y = np.asarray(y).astype(np.int64)
    r["tp"], r["fp"] = np.sum((label == 1) & (y == 1)), np.sum((label == 1) & (y == 0))
    r["tn"], r["fn"] = np.sum((label == 0) & (y == 0)), np.sum((label == 0) & (y == 1))
    q = np.where(y == 1, p1, 1.0 - p1)
    r["log_loss_sum"] = np.sum(-np.log(np.clip(q, EPS, 1 - EPS)))
    r["brier_sum"] = np.sum((y - p1) ** 2)
    # twice Mann-Whitney: per positive, negatives strictly below plus negatives at or below
    neg = np.sort(key[y == 0])
    pos = key[y == 1]
    r["auc_u2"] = int(np.sum(np.searchsorted(neg, pos, side="left")) + np.sum(np.searchsorted(neg, pos, side="right")))
    return r


def substituted(rows: np.ndarray, word: int, src: np.ndarray) -> np.ndarray:
    """rows with word ``word`` of row i taken from row src[i]."""
    out = np.array(rows, dtype=np.uint32, copy=True)
    out[:, word] = rows[src, word]
    return out


def permutation_scores(blob: bytes, rows: np.ndarray, labels, perm: np.ndarray, words):
    """What b2f_permutation_scores returns: (records (len(words), R), baseline record)."""
    from databricks_kubernetes_mlops_poc_b200._cabi import PERM_SCORE_DTYPE

    rows = np.ascontiguousarray(rows, dtype=np.uint32)
    y = np.asarray(labels)
    base = record(*tree_order_scores(blob, rows), y)
    out = np.zeros((len(words), perm.shape[0]), dtype=PERM_SCORE_DTYPE)
    for f, w in enumerate(words):
        for r in range(perm.shape[0]):
            out[f, r] = record(*tree_order_scores(blob, substituted(rows, w, perm[r])), y)
    return out, base
