"""Measurement helper: K5b (k_tree_shap_interactions) device time of b2f_explain_interactions by batch size, for rf100d6, the
benchmark's GBDT 100 x d6 and rf500d8, with the float64 operation count taken from each path table and its share of the H100
SXM data-sheet FP64 peak (34 TFLOP/s, non-tensor).  Device time = CUDA events around the whole call (H2D, kernels, D2H of the
n x 23 x 23 doubles), median of 5 after 2 warm-ups; the card's name and power limit are read in the same run.

Operations per (row, path of L elements, d = L - 1), counted once per path as the algorithm needs them (the kernel repeats
EXTEND in every warp that owns a field of the path; that repetition is not counted): EXTEND d(d+1)/2 steps of 4 flops; per
element, UNWIND d steps of 4 flops plus 2 for its phi term; per unordered pair of elements, the unwound sum d - 1 steps of
4 flops plus 4 for its term.  That is 2d(d+1) + d(4d + 2) + 2d^2(d - 1)."""
import json, os, sys

OUT = os.environ.get("B2F_TOOL_OUT", "tools_out")  # where the result file goes
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (its GBDT recipe and the card record)
from databricks_kubernetes_mlops_poc_b200 import training  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer, flatten_pipeline, parse_explainer  # noqa: E402
from oracle import datasets, reference_pipeline as rp  # noqa: E402

FP64_PEAK = 34e12
SIZES = (1, 16, 256, 4096, 65536)


def flops_per_row(table: bytes) -> float:
    d = parse_explainer(table)["paths"]["len"].astype(np.float64) - 1
    return float((2 * d * (d + 1) + d * (4 * d + 2) + 2 * d * d * (d - 1)).sum())


def main():
    base = training.load_base_frame()
    curated = datasets.load_curated()
    kind, params = bench.MODELS["gbdt100d6"]
    models = {
        "rf100d6": rp.fit_reference_pipeline(curated, rp.PINNED_RF["rf100d6"]),
        "gbdt100d6": training.fit_synthetic(kind, base, bench.N_TRAIN, bench.TRAIN_SEED, **params),
        "rf500d8": rp.fit_reference_pipeline(curated, rp.PINNED_RF["rf500d8"]),
    }
    _, codes, nums = training.synth_arrays(base, max(SIZES), bench.DATA_SEED)
    res = {"device": bench.device_record(0), "fp64_peak_tflops": FP64_PEAK / 1e12, "models": {}}
    for name, pipe in models.items():
        flat = flatten_pipeline(pipe)
        table = flatten_explainer(pipe, flat)
        h = parse_explainer(table)
        eng = ForestEngine(flat, 0)
        eng.attach_explainer(table)
        rows = RowEncoder(flat).encode_arrays(codes, nums)
        fpr = flops_per_row(table)
        per = {}
        for n in SIZES:
            for _ in range(2):
                eng.explain_interactions_rows(rows[:n])
            ms = [eng.explain_interactions_rows(rows[:n], device_ms=True)[2] for _ in range(5)]
            k5 = float(np.median([eng.explain_rows(rows[:n], device_ms=True)[2] for _ in range(5)]))
            med = float(np.median(ms))
            per[str(n)] = {"device_ms": med, "min_ms": float(min(ms)), "max_ms": float(max(ms)), "gflop": n * fpr / 1e9,
                           "tflops": n * fpr / (med * 1e-3) / 1e12, "share_of_fp64_peak": n * fpr / (med * 1e-3) / FP64_PEAK,
                           "k5_explain_device_ms": k5}
        eng.close()
        res["models"][name] = {"n_trees": h["n_trees"], "paths": h["n_paths"], "max_len": h["max_len"],
                               "mean_len": float(h["paths"]["len"].mean()), "flop_per_row": fpr, "by_rows": per}
        print(name, json.dumps(res["models"][name]), flush=True)
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "explain_interactions_time.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["device"]))


if __name__ == "__main__":
    main()
