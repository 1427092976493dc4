"""Measurement helper: K5c (k_tree_shap_interventional) device time of b2f_explain_interventional by batch size and background
size, for rf100d6, the benchmark's GBDT 100 x d6 and rf500d8, with the background's attach time and table bytes, and K5
(b2f_explain, path-dependent) from the same run in brackets.  Device time = CUDA events around the whole call (H2D, kernels,
D2H), median of 5 after 2 warm-ups; attach time = host clock around b2f_model_attach_background (it synchronises), median of 3.
Backgrounds are the first B rows of the curated table (30 000 = all of it); requests are the benchmark's synthetic rows."""
import json, os, sys, time

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

SIZES = (1, 16, 256, 4096, 65536)
BACKGROUNDS = (100, 1000, 30000)


def device_ms(fn, rows, warm=2, reps=5):
    for _ in range(warm):
        fn(rows)
    return float(np.median([fn(rows, device_ms=True)[2] for _ in range(reps)]))


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
    res = {"device": bench.device_record(0), "models": {}}
    for name, pipe in models.items():
        flat = flatten_pipeline(pipe)
        table = flatten_explainer(pipe, flat)
        h = parse_explainer(table)
        enc = RowEncoder(flat)
        eng = ForestEngine(flat, 0)
        eng.attach_explainer(table)
        rows = enc.encode_arrays(codes, nums)
        bg_all = enc.encode_frame(curated[rp.FEATURES])
        k5 = {str(n): device_ms(eng.explain_rows, rows[:n]) for n in SIZES}
        per_bg = {}
        for B in BACKGROUNDS:
            ts, nbytes = [], 0
            for _ in range(3):
                t0 = time.perf_counter()
                nbytes = eng.attach_background(bg_all[:B])
                ts.append((time.perf_counter() - t0) * 1e3)
            by_rows = {str(n): {"device_ms": device_ms(eng.explain_interventional_rows, rows[:n]), "k5_device_ms": k5[str(n)]} for n in SIZES}
            per_bg[str(B)] = {"attach_ms": float(np.median(ts)), "table_bytes": int(nbytes),
                              "entries_per_path": (nbytes - 8 * (h["n_paths"] + 1)) / 8 / max(1, h["n_paths"]), "by_rows": by_rows}
            print(name, B, json.dumps(per_bg[str(B)]), flush=True)
        eng.close()
        res["models"][name] = {"n_trees": h["n_trees"], "paths": h["n_paths"], "max_len": h["max_len"], "mean_len": float(h["paths"]["len"].mean()),
                               "by_background": per_bg}
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "explain_interventional_time.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["device"]))


if __name__ == "__main__":
    main()
