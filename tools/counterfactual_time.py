"""Measurement helper: K7 (k_counterfactual + k_counterfactual_finish) for rf100d6, the benchmark's GBDT 100 x d6 and
rf500d8, all 14 numeric fields, at n = 1, 64, 1 024 and 65 536 of the benchmark's synthetic rows, cutoff 0.5.

Per model and n:
* kernel_ms: host clock around b2f_counterfactual_device + b2f_sync on device-resident rows, median of 5 after 2 warm-ups
  (of 3 after 1 at 65 536 rows);
* host_call_ms: host clock around b2f_counterfactual on host rows (H2D, kernels, D2H of the records), same repetitions;
  device_ms: CUDA events from the first H2D to the end of the last D2H of that call;
* segments: the call's 32-piece segments (pieces = split values + 1 per field).
At n = 1 024 also expanded_predict_ms: the same piece scores from the predict path, b2f_predict_f64 on the n x P
substituted rows (P = every piece of every field; one call per field), host clock, one run.
Writes counterfactual_time_<W>w.json (W = the power limit read in the same run) under $B2F_TOOL_OUT (default profiles/h100)."""
import json, os, sys, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.environ.get("B2F_TOOL_OUT", os.path.join(ROOT, "profiles", "h100"))
import bench  # noqa: E402  (its GBDT recipe and the card record)
from databricks_kubernetes_mlops_poc_b200 import _cabi, training  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine, blob_split_values  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline  # noqa: E402
from oracle import datasets, reference_pipeline as rp  # noqa: E402

SIZES = (1, 64, 1024, 65536)


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
    base = training.load_base_frame()
    curated = datasets.load_curated()
    kind, params = bench.MODELS["gbdt100d6"]
    models = {
        "rf100d6": rp.fit_reference_pipeline(curated, rp.PINNED_RF["rf100d6"]),
        "gbdt100d6": training.fit_synthetic(kind, base, bench.N_TRAIN, bench.TRAIN_SEED, **params),
        "rf500d8": rp.fit_reference_pipeline(curated, rp.PINNED_RF["rf500d8"]),
    }
    vocabs, codes, nums = training.synth_arrays(base, max(SIZES), bench.DATA_SEED)
    res = {"device": bench.device_record(0), "fields": list(rp.NUMERIC_FEATURES), "cutoff": 0.5, "models": {}}
    for name, pipe in models.items():
        flat = flatten_pipeline(pipe)
        enc = RowEncoder(flat)
        eng = ForestEngine(flat, 0)
        words = list(range(enc.n_cat, enc.n_cat + enc.n_num))
        splits = [blob_split_values(flat.blob, w) for w in words]
        all_rows = enc.encode_arrays(codes, nums)
        per = {"split_values": [len(s) for s in splits], "segments": int(sum((len(s) + 1 + 31) // 32 for s in splits)), "by_rows": {}}
        for n in SIZES:
            rows = np.ascontiguousarray(all_rows[:n])
            warm, reps = (1, 3) if n >= 65536 else (2, 5)
            d_rows, d_p, d_out = eng.device_alloc(rows.nbytes), eng.device_alloc(n * 8), eng.device_alloc(n * len(words) * 32)
            eng.h2d(d_rows, rows)

            def kernel():
                eng.counterfactual_device(d_rows, n, words, 0.5, d_p, d_out)
                eng.sync()

            rec = {"kernel_ms": median_ms(kernel, warm, reps),
                   "host_call_ms": median_ms(lambda: eng.counterfactual_rows(rows, words), warm, reps),
                   "device_ms": float(np.median([eng.counterfactual_rows(rows, words, device_ms=True)[2] for _ in range(reps)]))}
            for d in (d_rows, d_p, d_out):
                eng.device_free(d)
            if n == 1024:
                def expanded():
                    for w, s in zip(words, splits):
                        reps_k = np.concatenate([[np.nextafter(s[0], np.float32(-np.inf))], s]).astype(np.float32) if len(s) else np.zeros(1, np.float32)
                        big = np.repeat(rows, len(reps_k), axis=0)
                        big[:, w] = np.tile(reps_k.view(np.uint32), n)
                        eng.predict_rows(big, np.float64)

                rec["expanded_predict_ms"] = median_ms(expanded, warm=0, reps=1)
                rec["expanded_rows"] = int(n * sum(len(s) + 1 for s in splits))
            per["by_rows"][str(n)] = rec
            print(name, n, json.dumps(rec), flush=True)
        eng.close()
        res["models"][name] = per
    watts = res["device"]["power_limit_w"]
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, f"counterfactual_time_{int(round(watts)) if watts else 0}w.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(path, json.dumps(res["device"]))


if __name__ == "__main__":
    _cabi.load_library()
    main()
