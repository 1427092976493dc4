"""numpy emulation of k_pair_dependence (csrc/pair_dependence.cuh) over a forest blob (TEST INFRASTRUCTURE).

Mirrors the kernel's two-word walk: per (row, tree, segment of up to 32 points) one depth-first walk with an explicit stack
of (node, point mask) that splits the mask on the point's first word at splits on word a, on its second word at splits on
word b, and follows the row elsewhere; leaf payloads go to every point of the mask, each point's sum in tree order from
the GBDT init value, then the aggregate of ``forest_predict.cuh``.  A probe with word b = -1 is one-way.  It also reports
the deepest stack a walk used, so a test can check the one-entry-per-level bound.  It is not a fallback: nothing in the
product imports it.
"""

import numpy as np

from dependence_walk import SEG, _second
from databricks_kubernetes_mlops_poc_b200.flatten import META_FEAT_SHIFT, META_SLOT_MASK, SENTINEL_BITS, SENTINEL_WORD, parse_header


def _impute_point(word: int, v: int, n_cat: int, impute) -> int:
    if word >= n_cat and np.isnan(np.array([v], dtype=np.uint32).view(np.float32)[0]):
        return int(np.array([impute[word]], dtype=np.float32).view(np.uint32)[0])
    return int(v)


def pair_walk(blob: bytes, rows: np.ndarray, probes, point_words: np.ndarray):
    """rows (n, 24) uint32, probes [(word_a, word_b or -1, point_offset, count)], point_words (P', 2) uint32 -> (out float64
    (n, sum counts), deepest stack of one walk)."""
    h = parse_header(blob)
    n_cat, n_num = h["n_cat"], h["n_num"]
    w = rows.astype(np.uint32).copy()
    f = w.view(np.float32)
    nan = np.isnan(f[:, n_cat:n_cat + n_num])
    f[:, n_cat:n_cat + n_num][nan] = np.broadcast_to(h["impute"][n_cat:n_cat + n_num], nan.shape)[nan]
    w[:, SENTINEL_WORD] = SENTINEL_BITS
    pw = np.asarray(point_words, dtype=np.uint32).reshape(-1, 2)
    segs, col = [], 0  # (word a, word b, [(u, v)], first output column)
    for wa, wb, off, count in probes:
        pts = [(_impute_point(wa, pw[off + k, 0], n_cat, h["impute"]), _impute_point(wb, pw[off + k, 1], n_cat, h["impute"]) if wb >= 0 else 0)
               for k in range(count)]
        for s in range(0, count, SEG):
            segs.append((int(wa), int(wb), pts[s:s + SEG], col + s))
        col += count
    n = rows.shape[0]
    gbdt = h["agg_mode"] == 1
    acc = np.full((n, col), h["init_raw"] if gbdt else 0.0)
    buf = np.frombuffer(blob, dtype=np.uint8)
    deepest = 0
    for g in h["groups"]:
        base = h["chunks_off"] + g["chunk_off"]
        ns, nl = g["n_slots"], g["n_leaf_slots"]
        N = buf[base:base + ns * 256].view(np.uint32).reshape(ns, 32, 2)
        LV = buf[base + ns * 256:base + ns * 256 + nl * 256].view(np.float64).reshape(nl, 32)
        for lane in range(g["n_trees"]):  # tree order
            T, M = N[:, lane, 0].tolist(), N[:, lane, 1].tolist()
            for i in range(n):
                wi = w[i].tolist()
                for wa, wb, pts, c0 in segs:
                    stack = [(0, (1 << len(pts)) - 1)]
                    while stack:
                        node, mask = stack.pop()
                        while True:
                            t, m = T[node], M[node]
                            first = m & META_SLOT_MASK
                            if first == node:  # leaf
                                v = LV[t, lane]
                                for k in range(len(pts)):
                                    if (mask >> k) & 1:
                                        acc[i, c0 + k] += v
                                break
                            feat = m >> META_FEAT_SHIFT
                            if feat == wa or (wb >= 0 and feat == wb):
                                j = 0 if feat == wa else 1
                                sec = sum(1 << k for k in range(len(pts)) if _second(pts[k][j], t, m))
                                m2, m1 = mask & sec, mask & ~sec
                                if m1 and m2:
                                    stack.append((first + 1, m2))
                                    deepest = max(deepest, len(stack))
                                    node, mask = first, m1
                                else:
                                    node = first + (1 if m2 else 0)
                            else:
                                node = first + (1 if _second(wi[feat], t, m) else 0)
    if h["agg_mode"] == 0:
        return acc / h["denom"], deepest
    return 1.0 / (1.0 + np.exp(-acc)), deepest
