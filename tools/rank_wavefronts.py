"""CPU only: the walk's two throughput floors for k_forest_predict_rank on the benchmark's workload.

Replays the rank-layout walk (tests/rank_walk.py's arithmetic) over the benchmark's model (GBDT 100 x depth 6, bench.py's
fit) and one seeded 65 536-row batch, warp by warp (32 consecutive rows = one tile = one warp's rows), and counts the
shared-memory wavefronts of every warp-level load of the walk:
  node     LDS.32 of each lane's node word from level 2 down: per bank, the number of distinct words (equal words
           broadcast); levels 0 and 1 come from the kernel's parameter block (constant bank) and cost none;
  value    LDS.U16 from the lane's own column of the tile's value block: bank = lane by construction;
  payload  LDS.64 of each lane's leaf payload: per pair of banks, the number of distinct 8-byte words.
Tiles per CTA follow the kernel's split of 2 048 tiles over `--sms` CTAs.  The two floors per CTA:
  wavefronts  sum of the wavefronts of its tiles' walks, at one wavefront per clock per SM;
  issue       `--group-instructions` warp instructions per (tile, group of U = 4 trees), over 4 schedulers per SM.
`--group-instructions` is read off the compiled walk loop (cuobjdump -sass of k_forest_predict_rank<6,4,false,float>:
204 for one 4-tree group in the current build); `--mhz` converts cycles to time (1 965 MHz: the median SM clock the
benchmark records at 400 W).  The walk replayed as "now" covers the ceil(n_trees / 4) groups the resident kernel walks;
"before" is the earlier walk -- every padded tree (a multiple of 8), every level from shared memory, 196 instructions per
group (`--group-instructions-before`) -- for comparison.  Writes $B2F_TOOL_OUT/rank_wavefronts.json.

    python tools/rank_wavefronts.py [--sms 132] [--mhz 1965] [--group-instructions 204] [--group-instructions-before 196]
"""

from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.environ.get("B2F_TOOL_OUT", "tools_out")
U = 4  # trees per group (the resident kernel's default)


def wavefronts(addr: np.ndarray, word: int, banks: int) -> np.ndarray:
    """addr (warps, 32) byte addresses of one warp-level load -> wavefronts per warp: max over bank groups of distinct words."""
    w = np.sort(addr // word, axis=1)
    first = np.ones_like(w, dtype=bool)
    first[:, 1:] = w[:, 1:] != w[:, :-1]  # one entry per distinct word
    counts = np.zeros((w.shape[0], banks), dtype=np.int64)
    rows = np.broadcast_to(np.arange(w.shape[0])[:, None], w.shape)
    np.add.at(counts, (rows[first], (w % banks)[first]), 1)
    return counts.max(axis=1)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sms", type=int, default=132)
    ap.add_argument("--mhz", type=float, default=1965.0)
    ap.add_argument("--group-instructions", type=int, default=204)
    ap.add_argument("--group-instructions-before", type=int, default=196)
    args = ap.parse_args()

    import bench
    from databricks_kubernetes_mlops_poc_b200 import flatten
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from rank_walk import unpack_ranked

    pipe, base = bench.get_pipeline("gbdt100d6", bench.Dist(1, use_cuda=False, solo=True))
    flat = flatten.flatten_pipeline(pipe)
    enc = RowEncoder(flat)
    _, _, _, rows24 = bench.make_batches(base, enc, 1, bench.DATA_SEED)
    info, layout = enc.rank_info(), enc.rank_layout()
    x = unpack_ranked(enc.rank_rows(rows24), info)
    n, D = x.shape[0], info.depth
    slots, stride = 1 << D, (1 << D) * 12
    n_trees_padded = layout.size // stride
    n_walked = -(-int(info.n_trees) // U) * U  # the resident kernel walks ceil(n_trees / U) groups (earlier: all padded trees)
    warps = n // 32
    ridx = np.arange(n)
    wf = {"node": np.zeros(warps), "value": np.zeros(warps), "payload": np.zeros(warps)}
    node_top = np.zeros(warps)  # node loads of levels 0 and 1: the constant bank now, shared memory earlier
    walked = {}  # wavefronts per warp after tree t (t + 1 trees walked)
    leaves_distinct = np.zeros(warps)
    for t in range(n_trees_padded):
        b = t * stride
        nodes = layout[b : b + slots * 4].view(np.uint32)
        i = np.zeros(n, dtype=np.int64)
        for d in range(D):
            nw = nodes[i]
            (node_top if d < 2 else wf["node"])[:] += wavefronts((b + 4 * i).reshape(warps, 32), 4, 32)
            off = (nw & np.uint32(0x1F82)).astype(np.int64)  # byte offset of value[f] in the lane's column
            lane = np.arange(n) % 32
            wf["value"] += wavefronts(((ridx // 32) * 8192 + lane * 4 + off).reshape(warps, 32), 4, 32)
            f = (off >> 7) * 2 + ((off >> 1) & 1)
            v = x[ridx, np.minimum(f, x.shape[1] - 1)]
            i = 2 * i + 1 + (((v << np.uint32(16)) | np.uint32(0xFFFF)) >= nw).astype(np.int64)
        leaf = (i - (slots - 1)).reshape(warps, 32)
        wf["payload"] += wavefronts(b + slots * 4 + 8 * leaf, 8, 16)
        leaves_distinct += np.array([len(np.unique(r)) for r in leaf])
        if t + 1 == n_walked:
            walked["now"] = {k: v.copy() for k, v in wf.items()}
    walked["before"] = {**{k: v.copy() for k, v in wf.items()}, "node": wf["node"] + node_top}
    trees_walked = {"now": n_walked, "before": n_trees_padded}
    per_tree = {w: {k: float(v.mean() / trees_walked[w]) for k, v in walked[w].items()} for w in walked}
    per_tree_per_level = {"node": {"now": per_tree["now"]["node"] / max(D - 2, 1), "before": per_tree["before"]["node"] / D},
                          "value": per_tree["now"]["value"] / D}
    tile_wf = {w: sum(walked[w].values()) for w in walked}  # wavefronts of one tile's whole walk

    n_tiles = warps
    ctas = min(args.sms, n_tiles)
    tq, tr = divmod(n_tiles, ctas)
    cta_tiles = tq + (np.arange(ctas) < tr)
    starts = np.concatenate([[0], np.cumsum(cta_tiles)[:-1]])
    us = lambda cycles: float(cycles / args.mhz)  # noqa: E731
    floors = {}
    for w, gi in (("now", args.group_instructions), ("before", args.group_instructions_before)):
        cta_wf = np.array([tile_wf[w][s : s + k].sum() for s, k in zip(starts, cta_tiles)])
        cta_issue = cta_tiles * (trees_walked[w] // U) * gi / 4.0
        floors[w] = {
            "trees_walked": int(trees_walked[w]), "groups_of_4": int(trees_walked[w] // U),
            "node_loads_from_shared_memory": "levels 2 .. D-1" if w == "now" else "every level",
            "wavefronts_per_warp_per_tree": {**per_tree[w], "total": float(sum(per_tree[w].values()))},
            "wavefront_floor": {"cycles_max_cta": float(cta_wf.max()), "us_max_cta": us(cta_wf.max()), "us_mean_cta": us(cta_wf.mean())},
            "issue_floor": {"instructions_per_group": gi, "cycles_max_cta": float(cta_issue.max()),
                            "us_max_cta": us(cta_issue.max()), "us_mean_cta": us(cta_issue.mean())},
        }
    result = {
        "workload": f"gbdt100d6 (bench.py's fit), {n} ranked rows (seed {bench.DATA_SEED}), {n_tiles} tiles over {ctas} CTAs",
        "depth": D, "trees": int(info.n_trees),
        "tiles_per_cta": {str(k): int((cta_tiles == k).sum()) for k in sorted(set(cta_tiles.tolist()))},
        "now": floors["now"], "before": floors["before"],
        "wavefronts_per_warp_per_level": per_tree_per_level,
        "distinct_leaves_per_warp_per_tree": float(leaves_distinct.mean() / n_trees_padded),
        "mhz": args.mhz,
    }
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "rank_wavefronts.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
