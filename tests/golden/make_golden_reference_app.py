#!/usr/bin/env python
"""Freeze the reference service's HTTP behaviour into ``reference_app.json``.

The reference's ``app/main.py`` is imported unmodified, with this package's ``mlflow`` shim ahead on the path, and serves
``POST /predict`` from a deterministic stub plugin (``StubPlugin`` below: no model, no GPU).  For each request body in
``BODIES`` the status code and, for a 200, the parsed JSON response are stored, together with the request schema the
reference publishes in its OpenAPI document.  ``tests/test_server_cpu.py`` serves the same bodies through this package's
own app with the same stub and compares.

Usage:  python tests/golden/make_golden_reference_app.py --reference <checkout of nfmoore/databricks-kubernetes-mlops-poc>
"""

from __future__ import annotations

import argparse
import importlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES, sample_request  # noqa: E402

BODIES = {
    "sample_request": sample_request(),
    "three_rows_with_defaults": [{"credit_limit": 1250.0}, {}, {"sex": "female", "credit_limit": 9333}],
    "one_empty_row": [{}],
    "coerced_numbers": [{"age": "41", "credit_limit": 5001, "unknown_key": 1}, {"bill_amount_1": 1e3, "education": ""}],
    "wrong_type": [{"sex": 3}],
    "not_a_list": {"sex": "male"},
    "empty_list": [],
}


def stub_outputs(df):
    """-> (predictions, outlier flags, drift scores) of the stub plugin: P = (credit_limit mod 1000) / 1000,
    flag = credit_limit > 5000, drift score of feature i = i / 100."""
    x = df["credit_limit"].to_numpy(dtype=float)
    return ((x % 1000) / 1000.0).tolist(), (x > 5000).astype(int).tolist(), [i / 100.0 for i in range(len(ALL_FEATURES))]


class StubPlugin:
    """The plugin boundary of the reference: ``predict(DataFrame) -> dict`` (its ``CustomModel.predict``)."""

    def predict(self, df):
        if len(df.columns) == 0:
            raise KeyError("no columns")  # the reference's CustomModel fails on the column-less frame of []
        p, o, d = stub_outputs(df)
        return {"predictions": p, "outliers": o, "feature_drift_batch": dict(zip(ALL_FEATURES, d))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", required=True)
    args = ap.parse_args()
    from fastapi.testclient import TestClient

    import databricks_kubernetes_mlops_poc_b200 as pkg

    sys.path.insert(0, os.path.join(args.reference, "app"))
    sys.path.insert(0, os.path.join(os.path.dirname(pkg.__file__), "shim"))
    pkg.load_model = lambda path: StubPlugin()
    main_mod = importlib.import_module("main")
    assert os.path.samefile(os.path.dirname(main_mod.__file__), os.path.join(args.reference, "app"))
    out = {"bodies": BODIES, "responses": {}}
    with TestClient(main_mod.app, raise_server_exceptions=False) as c:
        for name, body in BODIES.items():
            r = c.post("/predict", json=body)
            out["responses"][name] = {"status": r.status_code, "json": r.json() if r.status_code == 200 else None}
        spec = c.get("/openapi.json").json()
    schema = spec["paths"]["/predict"]["post"]["requestBody"]["content"]["application/json"]["schema"]
    if "$ref" in schema.get("items", {}):
        schema = {"type": schema["type"], "items": spec["components"]["schemas"][schema["items"]["$ref"].rsplit("/", 1)[1]]}
    out["request_schema_properties"] = {k: {"type": v.get("type"), "default": v.get("default")} for k, v in schema["items"]["properties"].items()}
    with open(os.path.join(HERE, "reference_app.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
