"""b200-forest-serve: H100-native scoring engine for the credit-default service.

Drop-in for the hot path of nfmoore/databricks-kubernetes-mlops-poc:
``POST /predict`` -> ``model.predict(DataFrame) -> dict`` (reference ``app/main.py:42-86``,
``databricks/src/02-register-model.ipynb:330-353``), with the sklearn pipeline arithmetic replaced by
hand-written sm_90a CUDA kernels behind a C ABI (``include/b2f.h``).  No CPU fallback.
"""

from .flatten import FlatForest, flatten_pipeline  # noqa: F401
from .schema import ALL_FEATURES, CATEGORICAL_FEATURES, NUMERIC_FEATURES  # noqa: F401

__version__ = "0.1.0"


def load_model(path: str, **kw):
    """Drop-in for ``mlflow.pyfunc.load_model(path)`` (reference ``app/main.py:26-28``)."""
    from .model import load_model as _load

    return _load(path, **kw)


def __getattr__(name):
    if name == "B200Model":
        from .model import B200Model

        return B200Model
    if name in ("ForestEngine", "EngineGroup"):
        from . import engine

        return getattr(engine, name)
    raise AttributeError(name)
