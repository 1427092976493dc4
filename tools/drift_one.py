"""Measurement helper (also for ncu): one TabularDrift.statistics call on a batch of DRIFT_N rows (default 128) after two warm-up calls."""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from databricks_kubernetes_mlops_poc_b200 import training
from databricks_kubernetes_mlops_poc_b200.drift import TabularDrift
from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES, CATEGORICAL_FEATURES

n = int(os.environ.get("DRIFT_N", "128"))
ref = training.load_base_frame()[ALL_FEATURES]
batch = ref.iloc[np.random.default_rng(7).integers(0, len(ref), n)].reset_index(drop=True)
det = TabularDrift(ref, CATEGORICAL_FEATURES, device=0)
for _ in range(3):
    p, stat, flags = det.statistics(batch)
print(n, det.last_device_ms, p[:4])
det.close()
