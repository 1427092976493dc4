"""numpy emulation of k_ale (csrc/ale.cuh) over a forest blob (TEST INFRASTRUCTURE).

Mirrors the kernel: each row's bin per probed field from its raw word (NaN: no part), then per (row, tree, segment of up
to 16 fields in word order) one depth-first walk with an explicit stack of (node, point mask) over the row's 2 points per
field -- point 2j its lower edge, 2j + 1 its upper edge; at a split on field j's word the other fields' points follow
the row and the field's own two points go by their edges -- leaf payloads to every point of the mask, in tree order
from the GBDT init value, then the aggregate of ``forest_predict.cuh``.  ``ordered_sums`` adds the deltas in the
documented order (128-row CTAs in row order, then the CTA partials in CTA order); ``brute_ale`` is the brute-force
oracle on ``predict_proba``.  It also counts node visits per walk, so a test can check that no walk visits a node twice.  It is not a fallback: nothing in the product imports it.
"""

import numpy as np
import pandas as pd

from dependence_walk import _second
from databricks_kubernetes_mlops_poc_b200.flatten import META_FEAT_SHIFT, META_SLOT_MASK, SENTINEL_BITS, SENTINEL_WORD, parse_header

SEG_PROBES = 16
CTA_ROWS = 128


def row_bins(rows: np.ndarray, word: int, z: np.ndarray) -> tuple:
    """-> (bin index k - 1 per row (int64), present mask) of rows (n, 24) for a field with float32 edges z."""
    x = rows[:, word].view(np.float32)
    present = ~np.isnan(x)
    k = np.clip(np.searchsorted(np.asarray(z, np.float32), np.where(present, x, np.float32(0)), side="left"), 1, len(z) - 1)
    return k - 1, present


def ordered_sums(delta: np.ndarray, b: np.ndarray, present: np.ndarray, K: int) -> tuple:
    """A field's per-row deltas, bins and present mask -> (sums (K,), counts (K,)) added in the kernel's order."""
    sums, counts = [0.0] * K, [0] * K
    n = len(delta)
    for c0 in range(0, n, CTA_ROWS):
        part = [0.0] * K
        for r in range(c0, min(n, c0 + CTA_ROWS)):
            if present[r]:
                part[b[r]] += float(delta[r])
                counts[b[r]] += 1
        for k in range(K):
            sums[k] += part[k]
    return np.array(sums), np.array(counts, dtype=np.int64)


def ale_walk(blob: bytes, rows: np.ndarray, probes, edges: np.ndarray):
    """rows (n, 24) uint32, probes [(word, edge_offset, bins)], edges float32 -> (bin sums, bin counts (probe order, as
    b2f_ale), per probe (delta (n,), bin index (n,), present (n,)), largest number of visits of one node in one walk)."""
    h = parse_header(blob)
    n_cat, n_num = h["n_cat"], h["n_num"]
    w = rows.astype(np.uint32).copy()
    f = w.view(np.float32)
    nan = np.isnan(f[:, n_cat:n_cat + n_num])
    f[:, n_cat:n_cat + n_num][nan] = np.broadcast_to(h["impute"][n_cat:n_cat + n_num], nan.shape)[nan]
    w[:, SENTINEL_WORD] = SENTINEL_BITS
    n = rows.shape[0]
    info = []
    for word, off, K in probes:
        z = np.asarray(edges[off:off + K + 1], dtype=np.float32)
        b, present = row_bins(rows, word, z)
        info.append((int(word), z.view(np.uint32), b, present))
    order = sorted(range(len(probes)), key=lambda i: info[i][0])
    segs = [order[s:s + SEG_PROBES] for s in range(0, len(order), SEG_PROBES)]
    gbdt = h["agg_mode"] == 1
    acc = np.full((n, 2 * len(probes)), h["init_raw"] if gbdt else 0.0)  # column 2i / 2i + 1: probe i's lower / upper
    buf = np.frombuffer(blob, dtype=np.uint8)
    max_visits = 0
    for g in h["groups"]:
        base = h["chunks_off"] + g["chunk_off"]
        ns, nl = g["n_slots"], g["n_leaf_slots"]
        N = buf[base:base + ns * 256].view(np.uint32).reshape(ns, 32, 2)
        LV = buf[base + ns * 256:base + ns * 256 + nl * 256].view(np.float64).reshape(nl, 32)
        for lane in range(g["n_trees"]):  # tree order
            T, M = N[:, lane, 0].tolist(), N[:, lane, 1].tolist()
            for i in range(n):
                wi = w[i].tolist()
                for seg in segs:
                    jof = {info[p][0]: j for j, p in enumerate(seg)}
                    pts, cols, full = [], [], 0
                    for j, p in enumerate(seg):
                        word, zw, b, present = info[p]
                        pts += [int(zw[b[i]]), int(zw[b[i] + 1])]
                        cols += [2 * p, 2 * p + 1]
                        if present[i]:
                            full |= 3 << (2 * j)
                    if not full:
                        continue
                    visits = {}
                    stack = [(0, full)]
                    while stack:
                        node, mask = stack.pop()
                        while True:
                            visits[node] = visits.get(node, 0) + 1
                            t, m = T[node], M[node]
                            first = m & META_SLOT_MASK
                            if first == node:  # leaf
                                v = LV[t, lane]
                                for k in range(len(pts)):
                                    if (mask >> k) & 1:
                                        acc[i, cols[k]] += v
                                break
                            feat = m >> META_FEAT_SHIFT
                            row_sec = _second(wi[feat], t, m)
                            if feat in jof:
                                j = jof[feat]
                                own = 3 << (2 * j)
                                sec = ((0xFFFFFFFF & ~own) if row_sec else 0) | (int(_second(pts[2 * j], t, m)) << (2 * j)) | \
                                      (int(_second(pts[2 * j + 1], t, m)) << (2 * j + 1))
                                m2, m1 = mask & sec, mask & ~sec
                                if m1 and m2:
                                    stack.append((first + 1, m2))
                                    node, mask = first, m1
                                else:
                                    node = first + (1 if m2 else 0)
                            else:
                                node = first + (1 if row_sec else 0)
                    max_visits = max(max_visits, max(visits.values()))
    p1 = acc / h["denom"] if h["agg_mode"] == 0 else 1.0 / (1.0 + np.exp(-acc))
    sums, counts, per = [], [], []
    for i, (word, off, K) in enumerate(probes):
        delta = p1[:, 2 * i + 1] - p1[:, 2 * i]
        _, _, b, present = info[i]
        s, c = ordered_sums(delta, b, present, K)
        sums.append(s), counts.append(c), per.append((delta, b, present))
    return np.concatenate(sums), np.concatenate(counts), per, max_visits


def brute_ale(pipe, X: pd.DataFrame, feature: str, z: np.ndarray, x32: np.ndarray) -> dict:
    """The oracle: ``predict_proba`` on the rows with the field set to each row's lower and upper edge, then the formulas
    of ``ale.py`` written out directly (x32: the rows' values as float32, NaN = missing)."""
    z = np.asarray(z, dtype=np.float32)
    K = len(z) - 1
    present = ~np.isnan(x32)
    k = np.clip(np.searchsorted(z, x32[present], side="left"), 1, K)
    Xp = X[present].reset_index(drop=True)
    lo, hi = Xp.copy(), Xp.copy()
    lo[feature] = z[k - 1].astype(np.float64)
    hi[feature] = z[k].astype(np.float64)
    cols = list(pipe.named_steps["preprocessor"].feature_names_in_)
    delta = pipe.predict_proba(hi[cols])[:, 1] - pipe.predict_proba(lo[cols])[:, 1]
    n = np.array([(k == b).sum() for b in range(1, K + 1)], dtype=np.int64)
    d = np.array([delta[k == b].mean() if n[b - 1] else 0.0 for b in range(1, K + 1)])
    A = np.concatenate([[0.0], np.cumsum(d)])
    ale0 = sum(n[j] * (A[j] + A[j + 1]) / 2 for j in range(K)) / n.sum()
    return {"ale_values": A - ale0, "bin_rows": n}
