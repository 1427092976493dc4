"""Measurement helper: K10 (b2f_pair_dependence: k_pair_dependence and k_pair_dependence_finish) for rf100d6, the
benchmark's GBDT 100 x d6 and rf500d8.

Per model:
* two_way_100x100: the mean over 65 536 rows (the benchmark's synthetic rows) of the 10 000 points of credit_limit x
  bill_amount_1 on 100-point grids.  kernel_ms: host clock around the device form on rows already on the device, through
  its synchronise (spec upload, the walks, the finishing kernel), median of 5 after a warm-up; device_ms: CUDA events of
  the host form (row upload, kernels, means back); host_call_ms: host clock around the host form.  Both medians of 5.
* interaction_strength: B200Model.interaction_strength over all 23 fields of the 30 000-row curated table at sample 1 000
  and 10 000: host clock (sampling, dedupe, the one device call, the H^2 arithmetic), median of 3 after a warm-up (one
  run at 10 000), the points scored and their point scorings (points x rows).
* sklearn_one_pair_ms (rf100d6 only; "not measured" for the others): F_jk of one pair (credit_limit, age) in the brute form
  at n = 1 000 -- pipeline.predict_proba on the 10^6 materialised rows -- on this host's CPUs.
Writes pair_dependence_time_<W>w.json (W = the power limit read in the same run) under $B2F_TOOL_OUT (default
profiles/h100), after every model."""
import json, os, sys, time

import numpy as np
import pandas as pd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.environ.get("B2F_TOOL_OUT", os.path.join(ROOT, "profiles", "h100"))
import bench  # noqa: E402  (its GBDT recipe and the card record)
from databricks_kubernetes_mlops_poc_b200 import _cabi, dependence, interaction, training  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.model import B200Model  # noqa: E402
from oracle import datasets, reference_pipeline as rp  # noqa: E402

ROWS = 65536
PAIR = ("credit_limit", "bill_amount_1")


def _median_ms(fn, reps):
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def main():
    base = training.load_base_frame()
    curated = datasets.load_curated()
    kind, params = bench.MODELS["gbdt100d6"]
    recipes = {
        "rf100d6": lambda: rp.fit_reference_pipeline(curated, rp.PINNED_RF["rf100d6"]),
        "gbdt100d6": lambda: training.fit_synthetic(kind, base, bench.N_TRAIN, bench.TRAIN_SEED, **params),
        "rf500d8": lambda: rp.fit_reference_pipeline(curated, rp.PINNED_RF["rf500d8"]),
    }
    vocabs, codes, nums = training.synth_arrays(base, ROWS, bench.DATA_SEED)
    res = {"device": bench.device_record(0), "rows": ROWS, "pair": list(PAIR), "models": {}}
    watts = res["device"]["power_limit_w"]
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, f"pair_dependence_time_{int(round(watts)) if watts else 0}w.json")
    for name, fit in recipes.items():
        pipe = fit()
        m = B200Model.from_pipeline(pipe)
        eng, enc = m.engine, m.encoder
        rows = np.ascontiguousarray(enc.encode_arrays(codes, nums)[:ROWS])
        ga = dependence.grid_from_column(curated[PAIR[0]], False, 100)
        gb = dependence.grid_from_column(curated[PAIR[1]], False, 100)
        pts = interaction.cartesian(dependence.encode_grid(enc, PAIR[0], ga), dependence.encode_grid(enc, PAIR[1], gb))
        probes = [(dependence.word_of(enc, PAIR[0]), dependence.word_of(enc, PAIR[1]), 0, len(pts))]
        eng.pair_dependence_rows(rows, probes, pts, mean=True)  # warm-up
        d_rows, d_out = eng.device_alloc(rows.nbytes), eng.device_alloc(len(pts) * 8)
        try:
            eng.h2d(d_rows, rows)

            def device_form():
                eng.pair_dependence_device(d_rows, ROWS, probes, pts, d_out, mean=True)
                eng.sync()

            device_form()
            kernel_ms = _median_ms(device_form, 5)
        finally:
            eng.device_free(d_rows)
            eng.device_free(d_out)
        dev, host = [], []
        for _ in range(5):
            t0 = time.perf_counter()
            _, ms = eng.pair_dependence_rows(rows, probes, pts, mean=True, device_ms=True)
            host.append((time.perf_counter() - t0) * 1e3)
            dev.append(ms)
        two_way = {"points": len(pts), "point_scorings": ROWS * len(pts), "kernel_ms": kernel_ms, "device_ms": float(np.median(dev)),
                   "host_call_ms": float(np.median(host))}
        two_way["point_scorings_per_s"] = two_way["point_scorings"] / (kernel_ms / 1e3)
        print(name, "two_way", json.dumps(two_way), flush=True)
        per = {"two_way_100x100": two_way, "interaction_strength": {}}
        X = curated[rp.FEATURES]
        m.interaction_strength(X.iloc[:200])  # warm-up
        for sample, reps in ((1000, 3), (10000, 1)):
            S = interaction.sample_rows(len(X), sample, 0)
            from databricks_kubernetes_mlops_poc_b200.flatten import parse_header

            words = interaction.impute(enc.encode_frame(X.iloc[S]), enc.n_cat, len(enc.num_features), parse_header(m.flat.blob)["impute"])
            probes_s, _, _ = interaction.strength_plan(words, list(range(23)), [w < enc.n_cat for w in range(23)])
            P = int(sum(p[3] for p in probes_s))
            rec = {"rows": sample, "probes": len(probes_s), "points": P, "point_scorings": P * sample,
                   "host_call_ms": _median_ms(lambda: m.interaction_strength(X, sample=sample), reps), "runs": reps}
            rec["point_scorings_per_s"] = rec["point_scorings"] / (rec["host_call_ms"] / 1e3)
            per["interaction_strength"][str(sample)] = rec
            print(name, "interaction_strength", json.dumps(rec), flush=True)
        if name == "rf100d6":
            Xn = X.iloc[:1000].reset_index(drop=True)
            big = pd.concat([Xn] * 1000, ignore_index=True)
            for c in ("credit_limit", "age"):
                big[c] = np.repeat(Xn[c].to_numpy(), 1000)
            t0 = time.perf_counter()
            pipe.predict_proba(big)
            per["sklearn_one_pair_ms"] = (time.perf_counter() - t0) * 1e3
            per["sklearn_host_cpus"] = os.cpu_count()
        else:
            per["sklearn_one_pair_ms"] = "not measured"
        print(name, "sklearn_one_pair_ms", per["sklearn_one_pair_ms"], flush=True)
        m.close()
        res["models"][name] = per
        with open(path, "w") as f:
            json.dump(res, f, indent=1)
    print(path, json.dumps(res["device"]))


if __name__ == "__main__":
    _cabi.load_library()
    main()
