"""Shared fixtures.  GPU tests are marked ``gpu``; everything else runs on a CPU-only box."""

import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu on a machine that has one)")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Make sure the CUDA engine and the C oracle are compiled (nvcc cross-compiles without a GPU)."""
    import __graft_entry__ as ge

    ge.build()


@pytest.fixture(scope="session")
def curated():
    from oracle import datasets

    return datasets.load_curated()


@pytest.fixture(scope="session")
def inference():
    from oracle import datasets

    return datasets.load_inference()


def _fit_rf(curated, name):
    from oracle import reference_pipeline as rp

    return rp.fit_reference_pipeline(curated, rp.PINNED_RF[name])


@pytest.fixture(scope="session")
def rf100d6(curated):
    return _fit_rf(curated, "rf100d6")


@pytest.fixture(scope="session")
def rf500d8(curated):
    return _fit_rf(curated, "rf500d8")


@pytest.fixture(scope="session")
def gbdt_small(curated):
    """A small GBDT in the reference preprocessing (BASELINE configs 2-4 stand-in), fast to fit."""
    from oracle import reference_pipeline as rp

    tr, _ = rp.reference_split(curated)
    tr = tr.iloc[:4000]
    return rp.fit_gbdt_pipeline(tr, tr[rp.TARGET].to_numpy(), dict(n_estimators=40, max_depth=5, random_state=0))


@pytest.fixture(scope="session")
def adversarial(curated, rf100d6):
    """Rows built to sit on every edge the reference pipeline has: unknown / missing categories, NaN
    numerics, +-0, huge-but-finite values, and values exactly equal to split thresholds (and one
    float32 ulp either side)."""
    import pandas as pd

    from oracle import reference_pipeline as rp
    from oracle import treewalk as tw

    rng = np.random.default_rng(7)
    base = curated[rp.FEATURES].iloc[rng.integers(0, len(curated), 600)].reset_index(drop=True).copy()
    for name in rp.CATEGORICAL_FEATURES:
        col = base[name].astype(object)
        col[rng.random(len(base)) < 0.10] = "never_seen_category"
        col[rng.random(len(base)) < 0.05] = None
        col[rng.random(len(base)) < 0.03] = "missing"
        base[name] = col
    dump = tw.dump_pipeline(rf100d6)
    n_ohe = int(dump["cat_offsets"][-1])
    num_nodes = np.nonzero((dump["left"] != -1) & (dump["feature"] >= n_ohe))[0]
    pick = rng.choice(num_nodes, size=len(base), replace=True)
    thr32 = dump["threshold"][pick].astype(np.float32)
    for i in range(len(base)):
        col = rp.NUMERIC_FEATURES[int(dump["feature"][pick[i]]) - n_ohe]
        t = thr32[i]
        base.loc[i, col] = float([t, np.nextafter(t, np.float32(np.inf)), np.nextafter(t, np.float32(-np.inf)), dump["threshold"][pick[i]]][i % 4])
    for name in rp.NUMERIC_FEATURES:
        col = base[name].to_numpy(dtype=np.float64).copy()
        r = rng.random(len(base))
        col[r < 0.04] = np.nan
        col[(r >= 0.04) & (r < 0.05)] = 0.0
        col[(r >= 0.05) & (r < 0.06)] = -0.0
        col[(r >= 0.06) & (r < 0.07)] = 3.0e38
        col[(r >= 0.07) & (r < 0.08)] = -3.0e38
        col[(r >= 0.08) & (r < 0.09)] = 1e-45
        base[name] = col
    return pd.DataFrame(base)


@pytest.fixture(scope="session")
def iforest(curated):
    """The reference's outlier detector, minus the alibi-detect wrapper (not installed): ``IForest(threshold=0.95)
    .fit(df[NUMERIC_FEATURES].values)`` (02-register-model.ipynb:232-233) holds a default sklearn IsolationForest."""
    from sklearn.ensemble import IsolationForest

    from oracle import reference_pipeline as rp

    return IsolationForest(n_estimators=100, random_state=0).fit(curated[rp.NUMERIC_FEATURES].to_numpy())


@pytest.fixture(scope="session")
def iforest_edges(curated, iforest):
    """Rows whose numerics sit exactly on isolation-tree thresholds (and one float32 ulp either side); no NaN."""
    from oracle import reference_pipeline as rp

    rng = np.random.default_rng(11)
    base = curated[rp.FEATURES].iloc[rng.integers(0, len(curated), 800)].reset_index(drop=True).copy()
    for i in range(len(base)):
        tree = iforest.estimators_[int(rng.integers(len(iforest.estimators_)))].tree_
        node = int(rng.choice(np.nonzero(tree.children_left != -1)[0]))
        t64 = float(tree.threshold[node])
        t = np.float32(t64)
        v = [t, np.nextafter(t, np.float32(np.inf)), np.nextafter(t, np.float32(-np.inf)), t64][i % 4]
        base.loc[i, rp.NUMERIC_FEATURES[int(tree.feature[node])]] = float(v)
    return base


def has_gpu() -> bool:
    try:
        from databricks_kubernetes_mlops_poc_b200 import _cabi

        return _cabi.load_library().b2f_device_count() > 0
    except Exception:
        return False
