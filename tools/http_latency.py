"""POST /predict latency through the HTTP layer (in-process TestClient): this package's server with the classifier,
outlier forest and drift detector on the GPU, next to the reference's handler logic (app/main.py:42-86 restated: list ->
DataFrame -> model.predict -> dict, one request at a time) over the CPU restatement of CustomModel
(oracle/custom_model.py: sklearn pipeline + scipy drift + IsolationForest).  Writes http_latency.json under $B2F_TOOL_OUT (default tools_out/)."""
import json
import os
OUT = os.environ.get("B2F_TOOL_OUT", "tools_out")  # where the result file goes
import sys
import time
from types import SimpleNamespace

import numpy as np
import pandas as pd
from fastapi import FastAPI
from fastapi.testclient import TestClient

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from databricks_kubernetes_mlops_poc_b200.model import B200Model  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES, LoanApplicant, ModelOutput  # noqa: E402
from databricks_kubernetes_mlops_poc_b200.server import create_app  # noqa: E402
from oracle import datasets, reference_pipeline as rp  # noqa: E402
from oracle.custom_model import ReferenceCustomModel  # noqa: E402

cur = datasets.load_curated()
pipe = rp.fit_reference_pipeline(cur, rp.PINNED_RF["rf100d6"])
ref_model = ReferenceCustomModel(pipe, cur)
gpu_model = B200Model.from_pipeline(pipe, reference_frame=cur, outlier=SimpleNamespace(isolationforest=ref_model.iforest, threshold=0.95), devices=[0])

ref_app = FastAPI()


@ref_app.post("/predict", response_model=ModelOutput)
async def predict(data: list[LoanApplicant]):
    input_df = pd.DataFrame([{k: getattr(r, k) for k in ALL_FEATURES} for r in data])
    input_df.to_json(orient="records")  # the reference logs the request as a JSON string
    out = ref_model.predict(None, input_df)
    json.dumps(out)  # ... and the response
    return out


def run(client, body, reps):
    client.post("/predict", json=body)
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = client.post("/predict", json=body)
        ts.append(time.perf_counter() - t0)
        assert r.status_code == 200, r.text[:200]
    return 1e3 * float(np.percentile(ts, 50)), 1e3 * float(np.percentile(ts, 99)), r.json()


out = []
with TestClient(create_app(model=gpu_model)) as gpu_client, TestClient(ref_app) as ref_client:
    for n in (1, 100, 1000):
        body = cur[ALL_FEATURES].iloc[:n].to_dict(orient="records")
        g50, g99, gj = run(gpu_client, body, 30)
        c50, c99, cj = run(ref_client, body, 5 if n >= 1000 else 10)
        dp = float(np.abs(np.asarray(gj["predictions"]) - np.asarray(cj["predictions"])).max())
        dd = float(np.abs(np.asarray(list(gj["feature_drift_batch"].values())) - np.asarray(list(cj["feature_drift_batch"].values()))).max())
        row = dict(rows=n, b200_p50_ms=g50, b200_p99_ms=g99, cpu_reference_p50_ms=c50, cpu_reference_p99_ms=c99, speedup_p50=c50 / g50,
                   max_abs_dp=dp, max_abs_ddrift=dd, outliers_equal=gj["outliers"] == [float(v) for v in cj["outliers"]])
        out.append(row)
        print(row, flush=True)
gpu_model.close()
os.makedirs(OUT, exist_ok=True)
json.dump({"what": __doc__, "cores": os.cpu_count(), "by_request_rows": out}, open(os.path.join(OUT, "http_latency.json"), "w"), indent=1)
