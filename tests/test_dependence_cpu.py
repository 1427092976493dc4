"""Partial dependence on the CPU: the grid rule against scikit-learn's, and the numpy emulator of k_partial_dependence
(tests/dependence_walk.py) against ``sklearn.inspection.partial_dependence(method="brute")`` to 1e-12, on the reference
forests and the schema-zoo schemas; no walk visits a node twice."""

import numpy as np
import pandas as pd
import pytest
from sklearn.inspection import partial_dependence

import schema_zoo as sz
from dependence_walk import pd_walk

TOL = 1e-12


def _emulated(pipe, X, features, categorical, grid_resolution=100, percentiles=(0.05, 0.95), custom_values=None):
    """-> (grid per feature, individual per feature, max visits) from the emulator, grids and words built as
    B200Model.partial_dependence builds them."""
    from databricks_kubernetes_mlops_poc_b200 import dependence
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline

    flat = flatten_pipeline(pipe)
    enc = RowEncoder(flat)
    custom_values = custom_values or {}
    grids, words, probes, off = [], [], [], 0
    for f in features:
        grid = list(custom_values[f]) if f in custom_values else dependence.grid_from_column(X[f], f in categorical, grid_resolution, percentiles).tolist()
        grids.append(grid)
        words.append(dependence.encode_grid(enc, f, grid))
        probes.append((dependence.word_of(enc, f), off, len(grid)))
        off += len(grid)
    out, visits = pd_walk(flat.blob, enc.encode_frame(X), probes, np.concatenate(words))
    parts = dependence.split_output(out, [len(g) for g in grids], "both")
    return grids, parts["individual"], parts["average"], visits


def _agree(pipe, X, features, categorical, **kw):
    grids, ind, avg, visits = _emulated(pipe, X, features, categorical, **kw)
    assert visits == 1
    for k, f in enumerate(features):
        skw = {key: v for key, v in kw.items() if key != "custom_values"}
        if "custom_values" in kw and f in kw["custom_values"]:
            skw["custom_values"] = {f: kw["custom_values"][f]}
        want = partial_dependence(pipe, X, [f], method="brute", kind="both", categorical_features=categorical, **skw)
        assert list(want["grid_values"][0]) == list(grids[k])
        assert np.abs(ind[k] - want["individual"][0]).max() <= TOL, f
        assert np.abs(avg[k] - want["average"][0]).max() <= TOL, f


def test_grid_rule_matches_sklearn(curated):
    """Every field of the curated frame, at the default and a non-default resolution and percentiles: the same grid as
    scikit-learn's own ``partial_dependence`` (a constant classifier keeps its brute-force pass cheap)."""
    from sklearn.dummy import DummyClassifier
    from sklearn.pipeline import Pipeline

    from databricks_kubernetes_mlops_poc_b200 import dependence
    from oracle import reference_pipeline as rp

    X = curated[rp.FEATURES].iloc[:400]
    pipe = Pipeline([("m", DummyClassifier(strategy="prior"))]).fit(X, curated[rp.TARGET].iloc[:400])
    n_more = 0
    for grid_resolution, percentiles in ((100, (0.05, 0.95)), (7, (0.1, 0.8))):
        for f in rp.FEATURES:
            cat = f in rp.CATEGORICAL_FEATURES
            want = partial_dependence(pipe, X, [f], method="brute", kind="average", categorical_features=rp.CATEGORICAL_FEATURES,
                                      grid_resolution=grid_resolution, percentiles=percentiles)["grid_values"][0]
            got = dependence.grid_from_column(X[f], cat, grid_resolution, percentiles)
            assert list(got) == list(want), f
            n_more += (not cat) and len(np.unique(X[f])) >= grid_resolution
    assert n_more > 0  # some numerics took the percentile rule, the rest their unique values


def test_mquantiles_matches_scipy():
    from scipy.stats.mstats import mquantiles

    from databricks_kubernetes_mlops_poc_b200 import dependence

    rng = np.random.default_rng(3)
    for n in (1, 2, 3, 10, 1001):
        x = rng.normal(size=n) * 1e3
        for p in ((0.05, 0.95), (0.0, 1.0), (0.3, 0.31)):
            assert np.array_equal(dependence.mquantiles(x, p), np.asarray(mquantiles(x, prob=p)))


def test_default_grid_leaves_missing_out():
    from databricks_kubernetes_mlops_poc_b200 import dependence

    assert list(dependence.grid_from_column(pd.Series(["b", None, "a", np.nan, "b"], dtype=object), True)) == ["a", "b"]
    assert list(dependence.grid_from_column(pd.Series([2.0, np.nan, 1.0]), False)) == [1.0, 2.0]
    with pytest.raises(ValueError):
        dependence.grid_from_column(pd.Series([np.nan, np.nan]), False)


def test_emulator_rf100d6(rf100d6, curated):
    from oracle import reference_pipeline as rp

    X = curated[rp.FEATURES].iloc[100:112].reset_index(drop=True)
    feats = ["credit_limit", "repayment_status_1", "bill_amount_1", "age", "education"]
    feats = [f for f in feats if f in rp.FEATURES]
    _agree(rf100d6, X, feats, rp.CATEGORICAL_FEATURES)
    _agree(rf100d6, X, feats[:2], rp.CATEGORICAL_FEATURES, grid_resolution=9, percentiles=(0.2, 0.7))


def test_emulator_custom_values(rf100d6, curated):
    from oracle import reference_pipeline as rp

    X = curated[rp.FEATURES].iloc[:10].reset_index(drop=True)
    num = rp.NUMERIC_FEATURES[0]
    cat = rp.CATEGORICAL_FEATURES[0]
    vals = sorted(X[cat].unique().tolist())
    _agree(rf100d6, X, [num, cat], rp.CATEGORICAL_FEATURES,
           custom_values={num: [5e4, -1.0, 0.0, 1e5, 2e3], cat: list(reversed(vals))})


def test_emulator_gbdt_small(gbdt_small, curated):
    from oracle import reference_pipeline as rp

    X = curated[rp.FEATURES].iloc[:10].reset_index(drop=True)
    _agree(gbdt_small, X, rp.FEATURES[:3] + rp.NUMERIC_FEATURES[:3], rp.CATEGORICAL_FEATURES, grid_resolution=20)


@pytest.mark.parametrize("name", ["packed_wide", "tiny", "over16"])
def test_emulator_schema_zoo(name):
    spec, pipe = sz.fitted(name)
    X = sz.make_frame(spec, 8, seed=5, target=False)
    cats = sz.cat_names(spec)
    feats = sz.features(spec)
    if name == "packed_wide":
        feats = [cats[4], cats[8], sz.num_names(spec)[1], sz.num_names(spec)[2]]  # the 126- and 100-category fields
        X = sz.make_frame(spec, 400, seed=5, target=False)  # enough rows to see most categories
        _agree(pipe, X.iloc[:6].reset_index(drop=True), feats, cats,
               custom_values={cats[4]: sorted(X[cats[4]].unique().tolist())})
        return
    _agree(pipe, X, feats[:6], cats, grid_resolution=12)
