"""Measurement helper: K12 (b2f_ale: k_ale and k_ale_finish) over all 14 numeric fields for rf100d6, the benchmark's GBDT
100 x d6 and rf500d8, at 1 000, 65 536 and 1 048 576 rows (the benchmark's synthetic rows; edges by the default rule,
bins = 20, min_bin_points = 4, over the same rows).

Per model and row count:
* device_form_ms: host clock around b2f_ale_device on rows already on the device, through b2f_sync (spec upload, the
  walks, the finishing kernels); median of 5 after a warm-up.
* host_call_ms / device_ms: host clock around b2f_ale (rows up, kernels, sums back), and its CUDA-event time; medians of 5.
* predict_f64_ms: the obvious alternative -- b2f_predict_f64 on the 2 F n substituted rows (each row with one field set to
  its lower or upper edge), one call per field on rows built beforehand (building them and reducing the deltas is not
  counted); median of 3 (1 at 1 048 576 rows).
* sklearn_oracle_ms (6 000 rows, per model): pipeline.predict_proba on the 2 F x 6 000 substituted rows of the brute-force
  oracle, on this host's CPUs.
Writes ale_time_<W>w.json (W = the power limit read in the same run) under $B2F_TOOL_OUT (default profiles/h100), after
every model."""
import json, os, sys, time

import numpy as np
import pandas as pd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.environ.get("B2F_TOOL_OUT", os.path.join(ROOT, "profiles", "h100"))
import bench  # noqa: E402  (its GBDT recipe and the card record)
from databricks_kubernetes_mlops_poc_b200 import _cabi, ale, dependence, training  # noqa: E402
from databricks_kubernetes_mlops_poc_b200._cabi import ptr  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.model import B200Model  # noqa: E402
from oracle import datasets, reference_pipeline as rp  # noqa: E402

SIZES = (1000, 65536, 1 << 20)
ORACLE_ROWS = 6000


def _median_ms(fn, reps):
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def _substituted(rows, probes, edges):
    """Per probe: the rows with the word at each row's lower edge, then at its upper edge (2n rows)."""
    out = []
    for word, off, K in probes:
        z = np.asarray(edges[off:off + K + 1], dtype=np.float32)
        x = rows[:, word].view(np.float32)
        k = np.clip(np.searchsorted(z, np.where(np.isnan(x), np.float32(0), x), side="left"), 1, K)
        sub = np.concatenate([rows, rows])
        sub[:len(rows), word] = z.view(np.uint32)[k - 1]
        sub[len(rows):, word] = z.view(np.uint32)[k]
        out.append(sub)
    return out


def main():
    base = training.load_base_frame()
    curated = datasets.load_curated()
    kind, params = bench.MODELS["gbdt100d6"]
    recipes = {
        "rf100d6": lambda: rp.fit_reference_pipeline(curated, rp.PINNED_RF["rf100d6"]),
        "gbdt100d6": lambda: training.fit_synthetic(kind, base, bench.N_TRAIN, bench.TRAIN_SEED, **params),
        "rf500d8": lambda: rp.fit_reference_pipeline(curated, rp.PINNED_RF["rf500d8"]),
    }
    vocabs, codes, nums = training.synth_arrays(base, max(SIZES), bench.DATA_SEED)
    res = {"device": bench.device_record(0), "fields": rp.NUMERIC_FEATURES, "bins": ale.DEFAULT_BINS,
           "min_bin_points": ale.DEFAULT_MIN_BIN_POINTS, "models": {}}
    watts = res["device"]["power_limit_w"]
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, f"ale_time_{int(round(watts)) if watts else 0}w.json")
    for name, fit in recipes.items():
        pipe = fit()
        m = B200Model.from_pipeline(pipe)
        eng, enc = m.engine, m.encoder
        all_rows = np.ascontiguousarray(enc.encode_arrays(codes, nums)[:max(SIZES)])
        words = [dependence.word_of(enc, f) for f in rp.NUMERIC_FEATURES]
        per = {}
        for n in SIZES:
            rows = all_rows[:n]
            edges = [ale.default_edges(rows[:, w].view(np.float32)[~np.isnan(rows[:, w].view(np.float32))], ale.DEFAULT_BINS,
                                       ale.DEFAULT_MIN_BIN_POINTS) for w in words]
            probes, z, _ = ale.probe_plan(words, edges)
            K = int(sum(p[2] for p in probes))
            eng.ale_rows(rows, probes, z)  # warm-up
            d_rows, d_s, d_c = eng.device_alloc(rows.nbytes), eng.device_alloc(K * 8), eng.device_alloc(K * 8)
            try:
                eng.h2d(d_rows, rows)

                def device_form():
                    eng.ale_device(d_rows, n, probes, z, d_s, d_c)
                    eng.sync()

                device_form()
                dev_ms = _median_ms(device_form, 5)
            finally:
                for d in (d_rows, d_s, d_c):
                    eng.device_free(d)
            host, evs = [], []
            for _ in range(5):
                t0 = time.perf_counter()
                _, _, ms = eng.ale_rows(rows, probes, z, device_ms=True)
                host.append((time.perf_counter() - t0) * 1e3)
                evs.append(ms)
            subs = _substituted(rows, probes, z)
            proba, label = np.empty(2 * n), np.empty(2 * n, dtype=np.int32)
            lib = eng._lib

            def predict_all():
                for s in subs:
                    _cabi.check(lib.b2f_predict_f64(eng.handle, ptr(s), len(s), ptr(proba), ptr(label)), "b2f_predict_f64")

            predict_all()  # warm-up
            pred_ms = _median_ms(predict_all, 3 if n < (1 << 20) else 1)
            del subs
            rec = {"rows": n, "fields": len(probes), "bins": K, "point_scorings": 2 * len(probes) * n, "device_form_ms": dev_ms,
                   "host_call_ms": float(np.median(host)), "device_ms": float(np.median(evs)), "predict_f64_ms": pred_ms}
            rec["predict_over_device_form"] = pred_ms / dev_ms
            per[str(n)] = rec
            print(name, json.dumps(rec), flush=True)
        X = curated[rp.FEATURES].iloc[:ORACLE_ROWS].reset_index(drop=True)
        big = []
        for f in rp.NUMERIC_FEATURES:
            x32 = ale.present_float32(enc, f, X[f])
            zf = ale.default_edges(x32, ale.DEFAULT_BINS, ale.DEFAULT_MIN_BIN_POINTS)
            k = np.clip(np.searchsorted(zf, X[f].to_numpy(dtype=np.float32), side="left"), 1, len(zf) - 1)
            for e in (zf[k - 1], zf[k]):
                Y = X.copy()
                Y[f] = e.astype(np.float64)
                big.append(Y)
        big = pd.concat(big, ignore_index=True)
        t0 = time.perf_counter()
        pipe.predict_proba(big)
        per["sklearn_oracle_ms"] = {"rows": ORACLE_ROWS, "substituted_rows": len(big), "ms": (time.perf_counter() - t0) * 1e3,
                                    "host_cpus": os.cpu_count()}
        t0 = time.perf_counter()
        m.accumulated_local_effects(X)
        per["model_call_6000_ms"] = (time.perf_counter() - t0) * 1e3
        print(name, "sklearn_oracle", json.dumps(per["sklearn_oracle_ms"]), "model_call_6000_ms", per["model_call_6000_ms"], flush=True)
        m.close()
        res["models"][name] = per
        with open(path, "w") as f:
            json.dump(res, f, indent=1)
    print(path, json.dumps(res["device"]))


if __name__ == "__main__":
    _cabi.load_library()
    main()
