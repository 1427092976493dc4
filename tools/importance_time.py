"""Measurement helper: K8 (b2f_permutation_scores: k_permutation_scores, the metric kernels and the segmented sort) for
rf100d6, the benchmark's GBDT 100 x d6 and rf500d8, all 23 fields, R = 5 repeats, at n = 1 000 (the test split's first
rows), 6 000 (the reference's test split), 30 000 (the curated table) and 262 144 (the benchmark's synthetic rows, random
labels).

Per model and n:
* device_ms: CUDA events around one b2f_permutation_scores call (uploads, kernels, sorts, records back), median of 3 after
  one warm-up;
* host_call_ms: host clock around the same call, including the argument checks, median of the same runs;
* groups: the call's groups of points under B2F_PERM_SCRATCH_BYTES;
* materialised_predict_ms: the n * 23 * 5 substituted rows scored through b2f_predict_f64 (one call, host clock, one run;
  the metrics are not computed) -- what scoring each permuted copy costs without the mask walk.
At n = 6 000 also sklearn_ms: sklearn.inspection.permutation_importance(pipeline, X, y, scoring="roc_auc", n_repeats=5,
random_state=0, n_jobs=1) on this host.
Writes importance_time_<W>w.json (W = the power limit read in the same run) under $B2F_TOOL_OUT (default profiles/h100)."""
import json, os, sys, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.environ.get("B2F_TOOL_OUT", os.path.join(ROOT, "profiles", "h100"))
import bench  # noqa: E402  (its GBDT recipe and the card record)
from databricks_kubernetes_mlops_poc_b200 import _cabi, importance, training  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline  # noqa: E402
from oracle import datasets, reference_pipeline as rp  # noqa: E402

SIZES = (1000, 6000, 30000, 262144)
REPEATS = 5
SCRATCH_BYTES = 256 << 20  # B2F_PERM_SCRATCH_BYTES


def main():
    base = training.load_base_frame()
    curated = datasets.load_curated()
    _, test = rp.reference_split(curated)
    kind, params = bench.MODELS["gbdt100d6"]
    models = {
        "rf100d6": rp.fit_reference_pipeline(curated, rp.PINNED_RF["rf100d6"]),
        "gbdt100d6": training.fit_synthetic(kind, base, bench.N_TRAIN, bench.TRAIN_SEED, **params),
        "rf500d8": rp.fit_reference_pipeline(curated, rp.PINNED_RF["rf500d8"]),
    }
    vocabs, codes, nums = training.synth_arrays(base, SIZES[-1], bench.DATA_SEED)
    synth_y = np.random.default_rng(0).integers(0, 2, SIZES[-1]).astype(np.int32)
    res = {"device": bench.device_record(0), "fields": 23, "n_repeats": REPEATS, "models": {}}
    for name, pipe in models.items():
        flat = flatten_pipeline(pipe)
        enc = RowEncoder(flat)
        eng = ForestEngine(flat, 0)
        words = list(range(enc.n_cat + enc.n_num))
        sources = {1000: (test.iloc[:1000], None), 6000: (test, None), 30000: (curated, None), 262144: (None, synth_y)}
        per = {"by_rows": {}}
        for n in SIZES:
            frame, y = sources[n]
            if frame is not None:
                rows = enc.encode_frame(frame[rp.FEATURES])
                y = frame[rp.TARGET].to_numpy().astype(np.int32)
            else:
                rows = np.ascontiguousarray(enc.encode_arrays(codes, nums)[:n])
            perm = importance.permutations(n, REPEATS, 0)
            eng.permutation_scores(rows, y, perm, words)  # warm-up
            dev, host = [], []
            for _ in range(3):
                t0 = time.perf_counter()
                _, _, ms = eng.permutation_scores(rows, y, perm, words, device_ms=True)
                host.append((time.perf_counter() - t0) * 1e3)
                dev.append(ms)
            points = 1 + len(words) * REPEATS
            gp = max(1, min(points, SCRATCH_BYTES // (18 * n)))
            rec = {"device_ms": float(np.median(dev)), "host_call_ms": float(np.median(host)), "groups": int(-(-points // gp)),
                   "substituted_rows": int(n * len(words) * REPEATS)}
            big = np.empty((n * len(words) * REPEATS, rows.shape[1]), dtype=np.uint32)
            k = 0
            for w in words:
                for r in range(REPEATS):
                    big[k:k + n] = rows
                    big[k:k + n, w] = rows[perm[r], w]
                    k += n
            t0 = time.perf_counter()
            eng.predict_rows(big, np.float64)
            rec["materialised_predict_ms"] = (time.perf_counter() - t0) * 1e3
            del big
            if n == 6000:
                from sklearn.inspection import permutation_importance

                X = test[rp.FEATURES]
                t0 = time.perf_counter()
                permutation_importance(pipe, X, test[rp.TARGET].to_numpy(), scoring="roc_auc", n_repeats=REPEATS, random_state=0, n_jobs=1)
                rec["sklearn_ms"] = (time.perf_counter() - t0) * 1e3
            per["by_rows"][str(n)] = rec
            print(name, n, json.dumps(rec), flush=True)
        eng.close()
        res["models"][name] = per
    watts = res["device"]["power_limit_w"]
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, f"importance_time_{int(round(watts)) if watts else 0}w.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(path, json.dumps(res["device"]))


if __name__ == "__main__":
    _cabi.load_library()
    main()
