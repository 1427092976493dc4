"""Measurement helper: K9 (the MMD drift test: b2f_model_attach_mmd_reference, b2f_mmd_drift) against the 30 000-row curated
table as the reference.

* attach: CUDA events around one b2f_model_attach_mmd_reference call (upload, embed, the six select passes when sigma is
  not given, the reference x reference row sums), with and without the select, median of 3 after one warm-up;
* per call, B = 100 permutations, batches of m in {2, 100, 1 000, 10 000, 65 536} curated rows (drawn with replacement
  past 30 000): device_ms (CUDA events from the upload to the last copy back) and host_call_ms (host clock around
  B200-level work: the draws, encoding and the call), medians of 3 after one warm-up;
* kernel pair evaluations per call from the shapes: the row sums n_ref * m + m * (n_ref + m) and the subsets'
  (B + 1) * s (s - 1) / 2, s = min(m, n_ref); per attach n_ref (n_ref - 1) (row sums) plus 6 * n_ref (n_ref - 1) / 2 (select);
  and their rate over device_ms;
* oracle_host_ms: oracle/mmd_drift.py (the explicit kernel matrix, numpy, this host's CPU) at m = 1 000 against a 5 000-row
  reference (the full table's 31 000^2 matrix does not fit its memory plan), B = 100.
Writes mmd_time_<W>w.json (W = the power limit read in the same run) under $B2F_TOOL_OUT (default profiles/h100)."""
import json, os, sys, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.environ.get("B2F_TOOL_OUT", os.path.join(ROOT, "profiles", "h100"))
import bench  # noqa: E402  (the card record)
from databricks_kubernetes_mlops_poc_b200 import mmd  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline, parse_header  # noqa: E402
from oracle import datasets, mmd_drift as om, reference_pipeline as rp  # noqa: E402

SIZES = (2, 100, 1000, 10000, 65536)
B = 100


def main():
    curated = datasets.load_curated()
    pipe = rp.fit_reference_pipeline(curated, rp.PINNED_RF["rf100d6"])
    flat = flatten_pipeline(pipe)
    enc = RowEncoder(flat)
    eng = ForestEngine(flat, 0)
    n_cat, n_num = len(flat.cat_features), len(flat.num_features)
    impute = parse_header(flat.blob)["impute"][n_cat:n_cat + n_num]
    ref = curated[rp.FEATURES]
    n_ref = len(ref)
    rows_ref = enc.encode_frame(ref)
    mean, scale = mmd.standardization(mmd.numerics(rows_ref, n_cat, n_num, impute))
    res = {"device": bench.device_record(0), "reference_rows": n_ref, "n_permutations": B, "attach": {}, "calls": {}}

    for label, given in (("median_heuristic", None), ("sigma_given", 3.0)):
        eng.attach_mmd_reference(rows_ref, mean, scale, given)
        ms = [eng.attach_mmd_reference(rows_ref, mean, scale, given, device_ms=True)[1] for _ in range(3)]
        pairs = n_ref * (n_ref - 1) + (6 * n_ref * (n_ref - 1) // 2 if given is None else 0)
        res["attach"][label] = {"device_ms": sorted(ms)[1], "runs_ms": ms, "pair_evaluations": pairs,
                                "pairs_per_s": pairs / (sorted(ms)[1] * 1e-3)}
    sigma = eng.attach_mmd_reference(rows_ref, mean, scale, None)
    res["sigma"] = sigma

    rng = np.random.default_rng(0)
    for m in SIZES:
        idx = rng.choice(n_ref, m, replace=m > n_ref)
        rows = enc.encode_frame(ref.iloc[idx].reset_index(drop=True))
        sub = mmd.draw_subsets(n_ref, m, B, 0)
        eng.mmd_statistics(rows, sub)
        dev, host = [], []
        for _ in range(3):
            t0 = time.perf_counter()
            sub = mmd.draw_subsets(n_ref, m, B, 0)
            _, _, ms = eng.mmd_statistics(rows, sub, device_ms=True)
            host.append((time.perf_counter() - t0) * 1e3)
            dev.append(ms)
        s = min(m, n_ref)
        pairs = n_ref * m + m * (n_ref + m) + (B + 1) * s * (s - 1) // 2
        d = sorted(dev)[1]
        res["calls"][str(m)] = {"device_ms": d, "runs_ms": dev, "host_call_ms": sorted(host)[1], "pair_evaluations": pairs,
                                "pairs_per_s": pairs / (d * 1e-3)}
        print(m, res["calls"][str(m)], flush=True)
    eng.close()

    # the explicit-matrix oracle on the host
    pre = pipe.named_steps["preprocessor"]
    xr = pre.transform(ref.iloc[:5000])
    xr = (xr.toarray() if hasattr(xr, "toarray") else np.asarray(xr)).astype(np.float32).astype(np.float64)
    xb = pre.transform(ref.iloc[10000:11000])
    xb = (xb.toarray() if hasattr(xb, "toarray") else np.asarray(xb)).astype(np.float32).astype(np.float64)
    mu, sc = mmd.standardization(xr[:, -n_num:])
    xr[:, -n_num:] = (xr[:, -n_num:] - mu) / sc
    xb[:, -n_num:] = (xb[:, -n_num:] - mu) / sc
    t0 = time.perf_counter()
    om.mmd_drift(xr, xb, mmd.draw_subsets(5000, 1000, B, 0))
    res["oracle_host_ms"] = {"reference_rows": 5000, "rows": 1000, "n_permutations": B, "ms": (time.perf_counter() - t0) * 1e3}

    watts = res["device"]["power_limit_w"]
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, f"mmd_time_{int(watts) if watts else 'unknown'}w.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
