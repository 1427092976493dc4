"""Measurement helper: K3 device / call time by batch size: row scan in shared memory, row scan through the global scratch (<= 48 rows),
anti-diagonal sweep."""
import json, os, sys, time
OUT = os.environ.get("B2F_TOOL_OUT", "tools_out")  # where the result file goes
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from databricks_kubernetes_mlops_poc_b200 import training
from databricks_kubernetes_mlops_poc_b200.drift import TabularDrift
from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES, CATEGORICAL_FEATURES

base = training.load_base_frame()
ref = base[ALL_FEATURES]
rng = np.random.default_rng(7)
out = {}
for mode in ("rowscan", "rowscan_global", "sweep"):
    os.environ.pop("B2F_DRIFT_ROWSCAN", None)
    os.environ.pop("B2F_DRIFT_ROWSCAN_SMEM", None)
    if mode == "sweep":
        os.environ["B2F_DRIFT_ROWSCAN"] = "0"
    if mode == "rowscan_global":
        os.environ["B2F_DRIFT_ROWSCAN_SMEM"] = "0"
    det = TabularDrift(ref, CATEGORICAL_FEATURES, device=0)
    rows = {}
    for n in (1, 2, 16, 48, 64, 128, 200, 250, 320, 512, 1000, 1025):
        batch = ref.iloc[rng.integers(0, len(ref), n)].reset_index(drop=True)
        det.statistics(batch)
        dev, wall = [], []
        for _ in range(10):
            t0 = time.perf_counter(); det.statistics(batch); wall.append(time.perf_counter() - t0); dev.append(det.last_device_ms)
        rows[str(n)] = {"device_ms": float(np.median(dev)), "call_ms": 1e3 * float(np.median(wall))}
    det.close()
    out[mode] = rows
print(json.dumps(out, indent=1))
os.makedirs(OUT, exist_ok=True)
json.dump(out, open(os.path.join(OUT, "drift_time.json"), "w"), indent=1)
