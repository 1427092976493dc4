"""Stand-in for the one corner of ``mlflow`` the reference service touches at run time.

The reference's ``app/main.py`` imports ``mlflow`` and makes exactly one call into it:
``mlflow.pyfunc.load_model(MODEL_DIRECTORY)`` in ``lifespan`` (``app/main.py:8,26-28``), then
``.predict(DataFrame)`` on the result (``:72``).  With this directory on ``PYTHONPATH`` ahead of site-packages,

    PYTHONPATH=<repo>/databricks_kubernetes_mlops_poc_b200/shim uvicorn app.main:app --port 5000

runs the reference's UNMODIFIED ``app/main.py`` on the H100 engine (SURVEY.md section 8f rank 4).  It is opt-in by path:
nothing in the package imports it, and a real mlflow installation is shadowed only for that process.
"""

from . import pyfunc  # noqa: F401

__version__ = "0+b200shim"
