"""Measurement helper: K11 (the k-nearest reference search of trust scores: b2f_model_attach_knn_reference, b2f_knn) against
the reference's 24 000-row training split of the curated table, rf100d6.

* attach: CUDA-synchronous host time of one b2f_model_attach_knn_reference (class sort, upload, embed), median of 3 after one
  warm-up; and B200Model.attach_trust_reference end to end (encode, constants, attach) without a filter and with
  filter_type="distance_knn" (alpha 0.05, k_filter 10: a second search of the reference against itself and the re-attach);
* per call, k = 2, query batches of m in {1, 1 000, 6 000, 65 536} rows (the 6 000-row test split, drawn with replacement
  past it): device_ms (CUDA events from the upload to the last copy back, median of 5 after one warm-up) and pair distances
  per second, m * 24 000 / device_ms; also at k = 64 for m = 6 000;
* kdtree_host_ms: the KDTree oracle (tests/trust_oracle.py, sklearn, this host's CPUs): fit on the training split and score
  the 6 000 test rows, k = 2.
Writes trust_time_<W>w.json (W = the power limit read in the same run) under $B2F_TOOL_OUT (default profiles/h100)."""
import json, os, sys, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.environ.get("B2F_TOOL_OUT", os.path.join(ROOT, "profiles", "h100"))
import bench  # noqa: E402  (the card record)
import trust_oracle as ot  # noqa: E402
from databricks_kubernetes_mlops_poc_b200 import mmd  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.flatten import parse_header  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.model import B200Model  # noqa: E402
from oracle import datasets, reference_pipeline as rp  # noqa: E402

SIZES = (1, 1000, 6000, 65536)


def main():
    curated = datasets.load_curated()
    pipe = rp.fit_reference_pipeline(curated, rp.PINNED_RF["rf100d6"])
    train, test = rp.reference_split(curated)
    train, test = train.reset_index(drop=True), test.reset_index(drop=True)
    model = B200Model.from_pipeline(pipe, devices=[0])
    eng, enc = model.engine, model.encoder
    n_cat, n_num = len(model.categorical_features), len(model.numeric_features)
    impute = parse_header(model.flat.blob)["impute"][n_cat:n_cat + n_num]
    rows_ref = enc.encode_frame(train[rp.FEATURES])
    cls = train[rp.TARGET].to_numpy().astype(np.int32)
    mean, scale = mmd.standardization(mmd.numerics(rows_ref, n_cat, n_num, impute))
    res = {"device": bench.device_record(0), "reference_rows": len(train), "class_rows": [int((cls == 0).sum()), int((cls == 1).sum())],
           "attach": {}, "calls": {}}

    eng.attach_knn_reference(rows_ref, cls, mean, scale)
    ms = []
    for _ in range(3):
        t0 = time.perf_counter()
        eng.attach_knn_reference(rows_ref, cls, mean, scale)
        ms.append((time.perf_counter() - t0) * 1e3)
    res["attach"]["engine_host_ms"] = {"median": sorted(ms)[1], "runs": ms}
    for label, kw in (("model_no_filter", {}), ("model_distance_knn_point", dict(filter_type="distance_knn", alpha=0.05)),
                      ("model_distance_knn_mean", dict(filter_type="distance_knn", alpha=0.05, dist_filter_type="mean"))):
        model.attach_trust_reference(train, **kw)
        ms = []
        for _ in range(3):
            t0 = time.perf_counter()
            kept = model.attach_trust_reference(train, **kw)
            ms.append((time.perf_counter() - t0) * 1e3)
        res["attach"][label] = {"median_ms": sorted(ms)[1], "runs_ms": ms, "kept": kept}
        print(label, res["attach"][label], flush=True)

    eng.attach_knn_reference(rows_ref, cls, mean, scale)
    rng = np.random.default_rng(0)
    for m, k in [(m, 2) for m in SIZES] + [(6000, 64)]:
        idx = np.arange(m) if m <= len(test) else rng.choice(len(test), m, replace=True)
        rows = enc.encode_frame(test[rp.FEATURES].iloc[idx].reset_index(drop=True))
        eng.knn(rows, k)
        dev, host = [], []
        for _ in range(5):
            t0 = time.perf_counter()
            dev.append(eng.knn(rows, k, device_ms=True)[2])
            host.append((time.perf_counter() - t0) * 1e3)
        d = sorted(dev)[2]
        pairs = m * len(train)
        res["calls"][f"m{m}_k{k}"] = {"rows": m, "k": k, "device_ms": d, "runs_ms": dev, "host_call_ms": sorted(host)[2],
                                      "pair_distances": pairs, "pairs_per_s": pairs / (d * 1e-3)}
        print(m, k, res["calls"][f"m{m}_k{k}"], flush=True)
    model.close()

    xr, mu, sc = ot.dense(pipe, train[rp.FEATURES])
    xq, _, _ = ot.dense(pipe, test[rp.FEATURES], mu, sc)
    pred = pipe.predict(test[rp.FEATURES]).astype(np.int64)
    t0 = time.perf_counter()
    ot.TrustScore().fit(xr, cls).score(xq, pred, k=2)
    res["kdtree_host_ms"] = {"reference_rows": len(train), "rows": len(test), "k": 2, "ms": (time.perf_counter() - t0) * 1e3,
                             "cpus": os.cpu_count()}

    watts = res["device"]["power_limit_w"]
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, f"trust_time_{int(watts) if watts else 'unknown'}w.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
