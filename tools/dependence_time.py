"""Measurement helper: K6 (k_partial_dependence) at 65 536 rows for rf100d6, the benchmark's GBDT 100 x d6 and rf500d8, on
two workloads: (a) credit_limit x 100 points, (b) all 23 fields with their default grids from the curated table.

Per model and workload:
* kernel_ms: host clock around b2f_partial_dependence_device + b2f_sync on device-resident rows (one kernel launch and the
  spec upload), median of 5 after 2 warm-ups;
* host_call_ms: host clock around b2f_partial_dependence on host rows (H2D, kernels, D2H of n x sum(G) doubles), median of
  5; device_ms: CUDA events from the first H2D to the end of the last D2H of that call; d2h_bytes: the output's bytes;
* expanded_predict_ms: the same curves from the predict path, b2f_predict_f64 on the n x G expanded rows (one call per
  field), host clock, one run;
* sklearn_1000_ms: sklearn's partial_dependence(method="brute") on 1 000 of the rows on the host CPUs (workload (b) for
  rf100d6 only), once.
Requests are the benchmark's synthetic rows, as 24-word rows, or with B2F_TOOL_ROWS=packed as 64-byte packed rows
(ROWS_PACKED64, written to dependence_time_packed.json); the expanded predict path takes the 24-word rows either way."""
import json, os, sys, time

OUT = os.environ.get("B2F_TOOL_OUT", "tools_out")  # where the result file goes
PACKED = os.environ.get("B2F_TOOL_ROWS", "words24") == "packed"  # the row format K6 reads
import numpy as np
import pandas as pd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (its GBDT recipe and the card record)
from databricks_kubernetes_mlops_poc_b200 import dependence, training  # noqa: E402
from databricks_kubernetes_mlops_poc_b200._cabi import ROWS_PACKED64, ROWS_WORDS24  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline  # noqa: E402
from oracle import datasets, reference_pipeline as rp  # noqa: E402

N = 65536


def median_ms(fn, warm=2, reps=5):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def main():
    from sklearn.inspection import partial_dependence

    base = training.load_base_frame()
    curated = datasets.load_curated()
    kind, params = bench.MODELS["gbdt100d6"]
    models = {
        "rf100d6": rp.fit_reference_pipeline(curated, rp.PINNED_RF["rf100d6"]),
        "gbdt100d6": training.fit_synthetic(kind, base, bench.N_TRAIN, bench.TRAIN_SEED, **params),
        "rf500d8": rp.fit_reference_pipeline(curated, rp.PINNED_RF["rf500d8"]),
    }
    vocabs, codes, nums = training.synth_arrays(base, N, bench.DATA_SEED)
    X = {f: np.where(codes[:1000, j] >= 0, vocabs[j][np.maximum(codes[:1000, j], 0)], "unknown") for j, f in enumerate(rp.CATEGORICAL_FEATURES)}
    X.update({f: nums[:1000, k] for k, f in enumerate(rp.NUMERIC_FEATURES)})
    X = pd.DataFrame(X)[rp.FEATURES]  # the same 1 000 rows as raw columns, for sklearn
    grids = {f: dependence.grid_from_column(curated[f], f in rp.CATEGORICAL_FEATURES) for f in rp.FEATURES}
    workloads = {"a_credit_limit_x100": ["credit_limit"], "b_all_23_fields": list(rp.FEATURES)}
    res = {"device": bench.device_record(0), "rows": N, "models": {}}
    if PACKED:
        res["row_format"] = "packed64"
    fmt = ROWS_PACKED64 if PACKED else ROWS_WORDS24
    for name, pipe in models.items():
        flat = flatten_pipeline(pipe)
        enc = RowEncoder(flat)
        eng = ForestEngine(flat, 0)
        words24 = enc.encode_arrays(codes, nums)
        rows = enc.pack_rows(words24) if PACKED else words24
        d_rows = eng.device_alloc(rows.nbytes)
        eng.h2d(d_rows, rows)
        per = {}
        for wl, feats in workloads.items():
            words, probes, off = [], [], 0
            for f in feats:
                words.append(dependence.encode_grid(enc, f, grids[f]))
                probes.append((dependence.word_of(enc, f), off, len(grids[f])))
                off += len(grids[f])
            grid = np.concatenate(words)
            d_out = eng.device_alloc(N * off * 8)

            def kernel():
                eng.partial_dependence_device(d_rows, N, probes, grid, d_out, fmt)
                eng.sync()

            k_ms = median_ms(kernel)
            eng.device_free(d_out)
            host_ms = median_ms(lambda: eng.partial_dependence_rows(rows, probes, grid))
            dev_ms = float(np.median([eng.partial_dependence_rows(rows, probes, grid, device_ms=True)[1] for _ in range(5)]))

            def expanded():
                for (word, _, g), w in zip(probes, words):
                    big = np.repeat(words24, g, axis=0)
                    big[:, word] = np.tile(w, N)
                    eng.predict_rows(big, np.float64)

            exp_ms = median_ms(expanded, warm=0, reps=1)
            rec = {"points": off, "kernel_ms": k_ms, "host_call_ms": host_ms, "device_ms": dev_ms, "d2h_bytes": N * off * 8,
                   "expanded_predict_ms": exp_ms}
            if wl.startswith("a") or name == "rf100d6":
                t0 = time.perf_counter()
                for f in feats:
                    partial_dependence(pipe, X, [f], method="brute", kind="both", categorical_features=rp.CATEGORICAL_FEATURES,
                                       custom_values={f: np.asarray(grids[f], dtype=object if f in rp.CATEGORICAL_FEATURES else np.float64)})
                rec["sklearn_1000_ms"] = (time.perf_counter() - t0) * 1e3
            per[wl] = rec
            print(name, wl, json.dumps(rec), flush=True)
        eng.device_free(d_rows)
        eng.close()
        res["models"][name] = per
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "dependence_time_packed.json" if PACKED else "dependence_time.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["device"]))


if __name__ == "__main__":
    main()
