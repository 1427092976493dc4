"""Measurement helper: K13 (the online MMD drift detector: b2f_mmd_online_bootstrap / _configure / _push) against the
30 000-row curated table as the MMD reference (rf100d6's encoder, sigma by the median heuristic).

* configure at W in {10, 100, 256}, B = 1 000 bootstraps: device_ms of the bootstrap call and of the configure call (CUDA
  events), and host_call_ms (host clock around B200Model.configure_online_drift: draws, bootstrap, threshold loop, split
  loop, configure), medians of 3 after one warm-up; kernel values of the bootstrap, B E (E - 1) / 2 with E = 2W - 1;
* push of m in {1, 100, 1 000, 65 536} curated rows at W = 100: device_ms (events from the upload to the last copy back)
  and host_call_ms (host clock around B200Model.online_drift: encoding, the push, the answer), medians of 5 after one
  warm-up; kernel values m (rw + W) and their rate;
* calibration (tests/test_gpu_mmd_online.py::test_calibration): the first detection times of the 20 no-drift streams and
  of the late-repayment stream, ERT = 100, W = 20, 5 000 bootstraps, a 4 000-row reference.
Writes mmd_online_time_<W>w.json (W = the power limit read in the same run) under $B2F_TOOL_OUT (default profiles/h100)."""
import json, os, sys, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.environ.get("B2F_TOOL_OUT", os.path.join(ROOT, "profiles", "h100"))
import bench  # noqa: E402  (the card record)
from databricks_kubernetes_mlops_poc_b200 import mmd_online  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.model import B200Model  # noqa: E402
from oracle import datasets, reference_pipeline as rp  # noqa: E402

WINDOWS = (10, 100, 256)
PUSHES = (1, 100, 1000, 65536)
B = 1000


def med(v):
    return sorted(v)[len(v) // 2]


def calibration(pipe, feats):
    order = np.random.default_rng(7).permutation(len(feats))
    ref, rest = feats.iloc[order[:4000]], feats.iloc[order[4000:]]
    model = B200Model.from_pipeline(pipe, devices=[0], mmd_reference=ref)
    try:
        model.configure_online_drift(ert=100, window_size=20, n_bootstraps=5000, random_state=0)
        firsts = []
        for k in range(20):
            model.reset_online_drift()
            stream = rest.iloc[np.random.default_rng(100 + k).permutation(len(rest))[:2000]]
            f = model.online_drift(stream)["first_drift"]
            firsts.append(2000 if f is None else f)
        late = rest[~rest["repayment_status_1"].isin(["no_delay", "duly_paid", "delay_1_month"])]
        model.reset_online_drift()
        drifted = model.online_drift(late.iloc[np.random.default_rng(1).permutation(len(late))[:500]])["first_drift"]
    finally:
        model.close()
    return {"ert": 100, "window_size": 20, "n_bootstraps": 5000, "reference_rows": 4000, "censored_at": 2000,
            "no_drift_first_detections": firsts, "no_drift_mean": float(np.mean(firsts)), "late_repayment_first_detection": drifted}


def main():
    curated = datasets.load_curated()
    pipe = rp.fit_reference_pipeline(curated, rp.PINNED_RF["rf100d6"])
    feats = curated[rp.FEATURES]
    n_ref = len(feats)
    model = B200Model.from_pipeline(pipe, devices=[0], mmd_reference=feats)
    eng = model.engine
    res = {"device": bench.device_record(0), "reference_rows": n_ref, "sigma": model.mmd_sigma, "n_bootstraps": B, "configure": {},
           "push": {}}
    for W in WINDOWS:
        E = 2 * W - 1
        rng = np.random.default_rng(0)
        etw = mmd_online.draw_bootstraps(rng, n_ref, W, B)
        perm = rng.permutation(n_ref)
        boot, conf, host = [], [], []
        for i in range(4):
            _, _, ms_b = eng.mmd_online_bootstrap(etw, W, device_ms=True)
            ms_c = eng.mmd_online_configure(perm, W, device_ms=True)
            t0 = time.perf_counter()
            model.configure_online_drift(ert=100, window_size=W, n_bootstraps=B, random_state=0)
            if i:
                boot.append(ms_b), conf.append(ms_c), host.append((time.perf_counter() - t0) * 1e3)
        values = B * E * (E - 1) // 2
        res["configure"][str(W)] = {"bootstrap_device_ms": med(boot), "configure_device_ms": med(conf), "host_call_ms": med(host),
                                    "runs_bootstrap_ms": boot, "runs_configure_ms": conf, "runs_host_ms": host,
                                    "bootstrap_kernel_values": values, "bootstrap_values_per_s": values / (med(boot) * 1e-3)}
        print(W, res["configure"][str(W)], flush=True)

    W = 100
    model.configure_online_drift(ert=100, window_size=W, n_bootstraps=B, random_state=0)
    rw = n_ref - (2 * W - 1)
    rng = np.random.default_rng(1)
    for m in PUSHES:
        df = feats.iloc[rng.choice(n_ref, m, replace=m > n_ref)].reset_index(drop=True)
        rows = model.encoder.encode_frame(df)
        eng.mmd_online_push(rows)
        model.online_drift(df)
        dev, host = [], []
        for _ in range(5):
            dev.append(eng.mmd_online_push(rows, device_ms=True)[2])
            t0 = time.perf_counter()
            model.online_drift(df)
            host.append((time.perf_counter() - t0) * 1e3)
        values = m * (rw + W)
        res["push"][str(m)] = {"window_size": W, "device_ms": med(dev), "host_call_ms": med(host), "runs_ms": dev, "runs_host_ms": host,
                               "kernel_values": values, "values_per_s": values / (med(dev) * 1e-3)}
        print(m, res["push"][str(m)], flush=True)
    model.close()
    res["calibration"] = calibration(pipe, feats)
    print(res["calibration"], flush=True)

    watts = res["device"]["power_limit_w"]
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, f"mmd_online_time_{int(watts) if watts else 'unknown'}w.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
