"""``mlflow.pyfunc.load_model`` -> the H100 model, ``B200Model`` (reference ``app/main.py:26-28``)."""

from __future__ import annotations


def load_model(model_uri: str, *args, **kwargs):
    """Same call shape as ``mlflow.pyfunc.load_model(model_uri)``; returns an object whose
    ``predict(DataFrame) -> {"predictions", "outliers", "feature_drift_batch"}`` has the contract of the
    reference's ``CustomModel.predict`` (``databricks/src/02-register-model.ipynb:330-353``)."""
    from databricks_kubernetes_mlops_poc_b200 import load_model as _load

    return _load(model_uri)
