"""numpy emulation of k_partial_dependence (csrc/partial_dependence.cuh) over a forest blob (TEST INFRASTRUCTURE).

Mirrors the kernel's walk: per (row, tree, segment of up to 32 grid points) one depth-first walk with an explicit stack of
(node, point mask) that follows the row at splits on other words and splits the mask at splits on the probed word; leaf
payloads go to every point of the mask, each point's sum in tree order from the GBDT init value, then the aggregate of
``forest_predict.cuh``.  It also counts node visits per walk, so a test can check that no walk visits a node twice.  It is
not a fallback: nothing in the product imports it.
"""

import numpy as np

from databricks_kubernetes_mlops_poc_b200.flatten import META_CAT, META_FEAT_SHIFT, META_SLOT_MASK, SENTINEL_BITS, SENTINEL_WORD, parse_header

SEG = 32


def _second(x: int, t: int, m: int) -> bool:
    """take_second of forest_blob.h: bit equality, or (numeric and (x >= t or unordered))."""
    if x == t:
        return True
    if m & META_CAT:
        return False
    xf, tf = np.array([x, t], dtype=np.uint32).view(np.float32)
    return not bool(xf < tf)


def pd_walk(blob: bytes, rows: np.ndarray, probes, grid_words: np.ndarray):
    """rows (n, 24) uint32, probes [(word, grid_offset, count)], grid_words uint32 -> (out float64 (n, sum counts), largest
    number of visits of one node within one walk)."""
    h = parse_header(blob)
    n_cat, n_num = h["n_cat"], h["n_num"]
    w = rows.astype(np.uint32).copy()
    f = w.view(np.float32)
    nan = np.isnan(f[:, n_cat:n_cat + n_num])
    f[:, n_cat:n_cat + n_num][nan] = np.broadcast_to(h["impute"][n_cat:n_cat + n_num], nan.shape)[nan]
    w[:, SENTINEL_WORD] = SENTINEL_BITS
    # segments: (word, [imputed grid words], first output column)
    segs, col = [], 0
    for word, off, count in probes:
        g = np.asarray(grid_words[off:off + count], dtype=np.uint32).copy()
        if word >= n_cat:
            gf = g.view(np.float32)
            gf[np.isnan(gf)] = h["impute"][word]
        for s in range(0, count, SEG):
            segs.append((int(word), [int(v) for v in g[s:s + SEG]], col + s))
        col += count
    n = rows.shape[0]
    gbdt = h["agg_mode"] == 1
    acc = np.full((n, col), h["init_raw"] if gbdt else 0.0)
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
                for word, gw, c0 in segs:
                    visits = {}
                    stack = [(0, (1 << len(gw)) - 1)]
                    while stack:
                        node, mask = stack.pop()
                        while True:
                            visits[node] = visits.get(node, 0) + 1
                            t, m = T[node], M[node]
                            first = m & META_SLOT_MASK
                            if first == node:  # leaf
                                v = LV[t, lane]
                                for k in range(len(gw)):
                                    if (mask >> k) & 1:
                                        acc[i, c0 + k] += v
                                break
                            feat = m >> META_FEAT_SHIFT
                            if feat == word:
                                sec = sum(1 << k for k in range(len(gw)) if _second(gw[k], t, m))
                                m2, m1 = mask & sec, mask & ~sec
                                if m1 and m2:
                                    stack.append((first + 1, m2))
                                    node, mask = first, m1
                                else:
                                    node = first + (1 if m2 else 0)
                            else:
                                node = first + (1 if _second(wi[feat], t, m) else 0)
                    max_visits = max(max_visits, max(visits.values()))
    if h["agg_mode"] == 0:
        return acc / h["denom"], max_visits
    return 1.0 / (1.0 + np.exp(-acc)), max_visits
