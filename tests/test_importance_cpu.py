"""Permutation importance on the CPU: the permutation replay of ``importance.py`` against scikit-learn's own shuffles, the
scorer formulas against ``sklearn.metrics`` on records counted by the numpy emulator (tests/importance_walk.py), the
whole emulated importance against ``sklearn.inspection.permutation_importance`` on the fitted pipelines, and the argument
and route validation of ``POST /explain/importance``."""

import json
import os
import warnings

import numpy as np
import pandas as pd
import pytest
from fastapi.testclient import TestClient

from importance_walk import permutation_scores, record, substituted, tree_order_scores

TOL = 1e-12


def _sklearn_permutations(n: int, n_repeats: int, random_state):
    """The rows sklearn's permutation_importance puts in a column of row numbers, repeat by repeat."""
    from sklearn.dummy import DummyClassifier
    from sklearn.inspection import permutation_importance

    seen = []

    def scorer(est, X, y):
        seen.append(np.asarray(X)[:, 0].astype(np.int64).copy())
        return 0.0

    X = np.arange(n, dtype=np.float64)[:, None]
    y = np.arange(n) % 2
    permutation_importance(DummyClassifier().fit(X, y), X, y, scoring=scorer, n_repeats=n_repeats, random_state=random_state, n_jobs=1)
    return np.array(seen[1:])  # seen[0] is the baseline


@pytest.mark.parametrize("n_repeats", [1, 5, 33])
def test_permutations_replay_sklearn(n_repeats):
    from databricks_kubernetes_mlops_poc_b200 import importance

    for n, rs in ((1, 0), (7, 3), (250, 0), (250, 12345)):
        assert np.array_equal(importance.permutations(n, n_repeats, rs), _sklearn_permutations(n, n_repeats, rs)), (n, rs)
    got = importance.permutations(100, n_repeats, np.random.RandomState(4))
    assert np.array_equal(got, _sklearn_permutations(100, n_repeats, np.random.RandomState(4)))
    p = importance.permutations(64, n_repeats, None)
    assert p.dtype == np.int32 and p.shape == (n_repeats, 64)
    assert all(np.array_equal(np.sort(r), np.arange(64)) for r in p)


def _sk_score(name, y, p1, label, key):
    from sklearn import metrics

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if name == "accuracy":
            return metrics.accuracy_score(y, label)
        if name == "precision":
            return metrics.precision_score(y, label, zero_division=0)
        if name == "recall":
            return metrics.recall_score(y, label, zero_division=0)
        if name == "f1":
            return metrics.f1_score(y, label, zero_division=0)
        if name == "roc_auc":
            return metrics.roc_auc_score(y, key)
        if name == "neg_log_loss":
            return -metrics.log_loss(y, np.stack([1 - p1, p1], axis=1))
        return -metrics.brier_score_loss(y, p1)


def test_scorer_formulas_match_sklearn_metrics():
    from databricks_kubernetes_mlops_poc_b200 import importance

    rng = np.random.default_rng(0)
    cases = []
    for n in (1, 2, 9, 400):
        p1 = rng.integers(0, 11, n) / 10.0  # ties, and exactly 0 and 1
        cases.append((rng.integers(0, 2, n), p1))
        cases.append((np.ones(n, np.int64), p1))  # one class
        cases.append((np.zeros(n, np.int64), p1))
        cases.append((rng.integers(0, 2, n), rng.random(n)))
        cases.append((rng.integers(0, 2, n), np.zeros(n)))  # no positive prediction: zero denominators
    for y, p1 in cases:
        label = (p1 > 0.5).astype(np.int32)
        rec = record(p1, label, p1, y)
        for name in importance.SCORERS:
            if name == "neg_log_loss" and len(np.unique(y)) < 2:
                with pytest.raises(ValueError):
                    _sk_score(name, y, p1, label, p1)
                with pytest.raises(ValueError):
                    importance.check_single_class([name], y)
                continue
            want, got = _sk_score(name, y, p1, label, p1), float(importance.score(name, rec))
            if np.isnan(want):
                assert np.isnan(got), name
            else:
                assert abs(got - want) <= TOL * max(1.0, abs(want)), (name, got, want)


def test_tree_order_scores_equal_the_dependence_walk(rf100d6, gbdt_small, curated):
    from dependence_walk import pd_walk

    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline
    from oracle import reference_pipeline as rp

    for pipe in (rf100d6, gbdt_small):
        flat = flatten_pipeline(pipe)
        rows = RowEncoder(flat).encode_frame(curated[rp.FEATURES].iloc[100:106])
        p1, _, _ = tree_order_scores(flat.blob, rows)
        for i in range(len(rows)):  # one probe at the row's own value: K6's walk of the row as it is
            out, _ = pd_walk(flat.blob, rows[i:i + 1], [(12, 0, 1)], rows[i, 12:13])
            assert out[0, 0] == p1[i]


def _emulated_importance(pipe, X, y, scoring, n_repeats, random_state):
    from databricks_kubernetes_mlops_poc_b200 import importance
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline

    flat = flatten_pipeline(pipe)
    enc = RowEncoder(flat)
    rows = enc.encode_frame(X)
    perm = importance.permutations(len(X), n_repeats, random_state)
    rec, base = permutation_scores(flat.blob, rows, y, perm, list(range(enc.n_cat + enc.n_num)))
    return {s: importance.result(s, rec, base, flat.all_features, n_repeats, len(X)) for s in scoring}


@pytest.mark.parametrize("which", ["rf100d6", "gbdt_small"])
def test_emulated_importance_equals_sklearn(which, request, curated):
    from sklearn.inspection import permutation_importance
    from sklearn.metrics import check_scoring

    from databricks_kubernetes_mlops_poc_b200 import importance
    from oracle import reference_pipeline as rp

    pipe = request.getfixturevalue(which)
    X = curated[rp.FEATURES].iloc[21000:21240].reset_index(drop=True)
    y = curated[rp.TARGET].iloc[21000:21240].to_numpy()
    scoring = list(importance.SCORERS)
    want = permutation_importance(pipe, X, y, scoring=scoring, n_repeats=3, random_state=0, n_jobs=1)
    got = _emulated_importance(pipe, X, y, scoring, 3, 0)
    for s in scoring:
        w, g = want[s], got[s]
        assert g["baseline_score"] == pytest.approx(check_scoring(pipe, scoring=s)(pipe, X, y), rel=TOL, abs=TOL), s
        tol = 0 if s in ("accuracy", "precision", "recall", "f1") else TOL
        assert np.allclose(g["importances"], w["importances"], rtol=tol, atol=tol), s
        assert np.allclose(g["importances_mean"], w["importances_mean"], rtol=tol, atol=tol), s
        assert np.allclose(g["importances_std"], w["importances_std"], rtol=tol, atol=max(tol, 1e-15)), s


def test_column_substitution_is_the_raw_column_permutation(rf100d6, curated):
    """Encoding and imputation work value by value: permuting a row word equals encoding the permuted raw column."""
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline
    from oracle import reference_pipeline as rp

    flat = flatten_pipeline(rf100d6)
    enc = RowEncoder(flat)
    X = curated[rp.FEATURES].iloc[:50].reset_index(drop=True).copy()
    X.loc[3, "age"] = np.nan
    X.loc[5, "education"] = "never_seen"
    rows = enc.encode_frame(X)
    src = np.random.default_rng(1).permutation(50)
    for f, name in enumerate(flat.all_features):
        Xp = X.copy()
        Xp[name] = X[name].to_numpy()[src]
        assert np.array_equal(enc.encode_frame(Xp), substituted(rows, f, src)), name


def test_argument_checks():
    from databricks_kubernetes_mlops_poc_b200 import importance

    assert importance.check_scoring(None) == (["accuracy"], False)
    assert importance.check_scoring("f1") == (["f1"], False)
    assert importance.check_scoring(["f1", "roc_auc"]) == (["f1", "roc_auc"], True)
    for bad in ("r2", ["f1", "balanced_accuracy"], [], ["f1", "f1"]):
        with pytest.raises(ValueError):
            importance.check_scoring(bad)
    for bad in (0, 257, 2.5, True, "5"):
        with pytest.raises(ValueError):
            importance.check_n_repeats(bad)
    assert importance.check_n_repeats(np.int64(256)) == 256
    assert importance.check_labels([0, 1, 1.0], 3).tolist() == [0, 1, 1]
    for bad, n in (([0, 2], 2), ([0.5, 1], 2), ([0, 1], 3), (["a", "b"], 2), ([[0, 1]], 2)):
        with pytest.raises(ValueError):
            importance.check_labels(bad, n)


class StubModel:
    """The model the route calls: records its arguments, answers NaN for roc_auc."""

    drift = None

    def __init__(self):
        self.replicas = [self]
        self.calls = []

    def predict_proba1(self, df):
        return np.zeros(len(df))

    def permutation_importance(self, df, y, *, scoring, n_repeats, random_state):
        from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES

        self.calls.append((df, np.asarray(y), scoring, n_repeats, random_state))
        F = len(ALL_FEATURES)
        out = {}
        for s in scoring:
            imp = np.full((F, n_repeats), np.nan if s == "roc_auc" else 0.25)
            out[s] = {"importances": imp, "importances_mean": imp.mean(axis=1), "importances_std": imp.std(axis=1),
                      "baseline_score": np.nan if s == "roc_auc" else 0.5, "feature_names": list(ALL_FEATURES), "n_repeats": n_repeats,
                      "rows": len(df)}
        return out


def test_route_contract_and_validation():
    from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES, DEFAULTS, TARGET
    from databricks_kubernetes_mlops_poc_b200.server import create_app

    stub = StubModel()
    body = [{TARGET: 1, "age": 30.0}, {TARGET: 0, "sex": "female"}]
    with TestClient(create_app(model=stub), raise_server_exceptions=False) as c:
        r = c.post("/explain/importance", json=body)
        assert r.status_code == 200, r.text
        j = r.json()
        assert j["feature_names"] == ALL_FEATURES and j["rows"] == 2 and j["n_repeats"] == 5 and j["random_state"] == 0
        assert list(j["scores"]) == ["accuracy"] and j["scores"]["accuracy"]["baseline"] == 0.5
        assert len(j["scores"]["accuracy"]["importances"]) == 23 and len(j["scores"]["accuracy"]["importances"][0]) == 5
        df, y, scoring, n_repeats, rs = stub.calls[-1]
        assert y.tolist() == [1, 0] and scoring == ["accuracy"] and n_repeats == 5 and rs == 0
        assert df.loc[0, "age"] == 30.0 and df.loc[1, "sex"] == "female" and df.loc[0, "sex"] == DEFAULTS["sex"]
        assert list(df.columns) == ALL_FEATURES
        r = c.post("/explain/importance?scoring=roc_auc&scoring=f1&n_repeats=2&random_state=7", json=body)
        j = r.json()
        assert r.status_code == 200 and list(j["scores"]) == ["roc_auc", "f1"] and j["random_state"] == 7 and j["n_repeats"] == 2
        assert j["scores"]["roc_auc"]["baseline"] is None and j["scores"]["roc_auc"]["importances_mean"][0] is None  # NaN -> null
        assert stub.calls[-1][2:] == (["roc_auc", "f1"], 2, 7)
        n_calls = len(stub.calls)
        for q in ("scoring=r2", "n_repeats=0", "n_repeats=257", "n_repeats=x", "random_state=-1", "random_state=4294967296",
                  "random_state=a", "scoring=f1&scoring=f1"):
            assert c.post(f"/explain/importance?{q}", json=body).status_code == 422, q
        for bad in ([{"age": 30.0}], [{TARGET: 2}], [{TARGET: "yes"}], [{TARGET: 0.5}], [{TARGET: 1, "sex": 3}]):
            assert c.post("/explain/importance", json=bad).status_code == 422, bad
        one_class = [{TARGET: 1}, {TARGET: 1}]
        r = c.post("/explain/importance?scoring=neg_log_loss", json=one_class)
        assert r.status_code == 422 and "only one label" in r.json()["detail"]
        assert len(stub.calls) == n_calls
        assert c.post("/explain/importance?scoring=roc_auc", json=one_class).status_code == 200
        assert c.post("/explain/importance", json=[]).status_code == 500
        paths = c.get("/openapi.json").json()["paths"]
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    for path, name in (("/predict", "openapi_predict.json"), ("/explain", "openapi_explain.json")):
        with open(os.path.join(golden, name)) as f:
            assert paths[path] == json.load(f)
    entry = paths["/explain/importance"]["post"]
    assert {p["name"] for p in entry["parameters"]} == {"scoring", "n_repeats", "random_state"}
    item = entry["requestBody"]["content"]["application/json"]["schema"]["items"]
    assert TARGET in item["required"] and set(ALL_FEATURES) <= set(item["properties"])
