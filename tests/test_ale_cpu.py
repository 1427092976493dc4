"""Accumulated local effects on the CPU: the edge rule of ``ale.py`` on the curated columns, the numpy emulator of k_ale
(tests/ale_walk.py) against a brute-force oracle on ``predict_proba`` to 1e-12 with identical bin counts (reference
forests, schema-zoo schemas and a schema of 18 numerics that spans two walk segments), the host arithmetic, and the 422s
of POST /explain/ale."""

import numpy as np
import pandas as pd
import pytest
from fastapi.testclient import TestClient

import schema_zoo as sz
from ale_walk import ale_walk, brute_ale

TOL = 1e-12


def _encoder(pipe):
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline

    flat = flatten_pipeline(pipe)
    return flat, RowEncoder(flat)


def _check_emulator(pipe, X, features, bins=10, min_bin_points=3):
    from databricks_kubernetes_mlops_poc_b200 import ale, dependence

    flat, enc = _encoder(pipe)
    rows = enc.encode_frame(X)
    edges = [ale.default_edges(ale.present_float32(enc, f, X[f]), bins, min_bin_points) for f in features]
    probes, z, which = ale.probe_plan([dependence.word_of(enc, f) for f in features], edges)
    sums, counts, _, visits = ale_walk(flat.blob, rows, probes, z)
    assert visits == 1  # no walk visits a node twice
    res = ale.result(features, edges, sums, counts, probes, which)
    for i, f in enumerate(features):
        x32 = rows[:, dependence.word_of(enc, f)].view(np.float32)
        if len(edges[i]) < 2:
            assert res["ale_values"][i].tolist() == [0.0]
            continue
        want = brute_ale(pipe, X, f, edges[i], x32)
        assert np.array_equal(res["bin_rows"][i], want["bin_rows"]), f
        assert np.abs(res["ale_values"][i] - want["ale_values"]).max() <= TOL, f
    return res


def test_emulator_rf100d6(rf100d6, curated, adversarial):
    from oracle import reference_pipeline as rp

    X = pd.concat([curated[rp.FEATURES].iloc[:90], adversarial.iloc[:40]], ignore_index=True)
    _check_emulator(rf100d6, X, rp.NUMERIC_FEATURES)


def test_emulator_gbdt_small(gbdt_small, curated):
    from oracle import reference_pipeline as rp

    X = curated[rp.FEATURES].iloc[9000:9140].reset_index(drop=True)
    X.loc[[3, 7, 11], "bill_amount_1"] = np.nan
    _check_emulator(gbdt_small, X, ["bill_amount_1", "credit_limit", "age", "payment_amount_3"], bins=8, min_bin_points=5)


@pytest.mark.parametrize("name", ["packed_wide_gbdt", "tiny", "over16", "num18"])
def test_emulator_schemas(name):
    if name == "num18":  # 18 numerics: a row's fields span two walk segments
        spec = ([3], 18)
        pipe = sz.fit_pipeline(spec, sz.make_frame(spec, 1500, seed=0), "rf", n_estimators=6, max_depth=5, random_state=0)
    else:
        spec, pipe = sz.fitted(name)
    X = pd.concat([sz.edge_rows(spec, pipe, n=30), sz.make_frame(spec, 50, seed=9, target=False)], ignore_index=True)
    _check_emulator(pipe, X, sz.num_names(spec), bins=6, min_bin_points=2)


def test_edge_rule_on_curated(curated):
    from databricks_kubernetes_mlops_poc_b200 import ale
    from oracle import reference_pipeline as rp

    for f in rp.NUMERIC_FEATURES:
        col = curated[f].to_numpy(dtype=np.float64)
        x32 = col.astype(np.float32)
        for bins, mbp in ((20, 4), (7, 1), (256, 200)):
            z = ale.default_edges(x32, bins, mbp)
            assert z.dtype == np.float32 and (np.diff(z) > 0).all() and len(z) - 1 <= bins, f
            u = np.unique(x32)
            if len(u) <= bins + 1:
                assert np.array_equal(z, u)
                continue
            assert ale.bin_counts(x32, z).min() >= mbp, (f, bins)
            xs = np.sort(x32).astype(np.float64)
            K = len(z) - 1
            # every larger K of the search fails the rule, and this K is the quantile grid
            for K2 in range(bins, 0, -1):
                z2 = np.unique(np.quantile(x32.astype(np.float64), np.linspace(0, 1, K2 + 1)).astype(np.float32))
                if np.array_equal(z2, z):
                    break
                assert len(z2) < 2 or ale.bin_counts(x32, z2).min() < mbp, (f, K2)
            assert K >= 1 and xs[0] == z[0] and xs[-1] == z[-1]


def test_sorted_quantiles_equal_numpy(curated):
    from databricks_kubernetes_mlops_poc_b200 import ale
    from oracle import reference_pipeline as rp

    rng = np.random.default_rng(0)
    cols = [curated[f].to_numpy(dtype=np.float32).astype(np.float64) for f in rp.NUMERIC_FEATURES]
    cols += [rng.normal(size=7), np.array([5.0]), np.array([1.0, 2.0]), rng.integers(0, 3, 1001).astype(np.float64)]
    for x in cols:
        xs = np.sort(x)
        for K in (1, 2, 3, 7, 20, 100, 256):
            q = np.linspace(0, 1, K + 1)
            assert np.array_equal(ale.sorted_quantiles(xs, q), np.quantile(x, q)), (len(x), K)


def test_low_resolution_and_missing():
    from databricks_kubernetes_mlops_poc_b200 import ale

    x = np.array([3, 1, 2, 2, 3, 1, np.nan, 2], dtype=np.float32)
    present = x[~np.isnan(x)]
    assert ale.default_edges(present, 20, 4).tolist() == [1.0, 2.0, 3.0]
    assert ale.default_edges(np.array([7.5, 7.5], np.float32), 20, 4).tolist() == [7.5]
    with pytest.raises(ValueError):
        ale.default_edges(np.zeros(0, np.float32), 20, 4)
    # more distinct values than bins + 1, too few rows for any K: the ends
    assert ale.default_edges(np.arange(6, dtype=np.float32), 2, 10).tolist() == [0.0, 5.0]
    assert ale.bin_counts(np.array([0, 1, 1.5, 2, 9, -4], np.float32), np.array([1, 2, 3], np.float32)).tolist() == [5, 1]


def test_host_arithmetic():
    from databricks_kubernetes_mlops_poc_b200 import ale

    e = ale.effects(np.array([0.3, 0.0, -0.9]), np.array([3, 0, 2]))
    assert e["bin_effects"].tolist() == [0.3 / 3, 0.0, -0.9 / 2]  # the empty bin adds nothing
    A = np.concatenate([[0.0], np.cumsum(e["bin_effects"])])
    assert np.array_equal(e["ale_values"], A - e["ale0"])
    n = e["bin_rows"]
    c = e["ale_values"]
    assert abs(np.sum(n * (c[:-1] + c[1:]) / 2)) <= 1e-15
    res = ale.result(["a", "b"], [np.array([1.0], np.float32), np.array([0, 1, 2], np.float32)], np.array([0.5, 0.25]), np.array([5, 5]),
                     [(10, 1, 2)], [1])
    assert res["ale_values"][0].tolist() == [0.0] and res["bin_rows"][0].size == 0 and res["ale0"][0] == 0.0
    assert res["bin_effects"][1].tolist() == [0.5 / 5, 0.25 / 5]
    for bad in ([1.0], [1.0, 1.0], [2.0, 1.0], [0.0, np.inf], [0.0, 1e39], ["x", 1.0], list(range(258)), [1.0, 1.0 + 1e-9]):
        with pytest.raises(ValueError):
            ale.check_custom_edges("f", bad)
    assert ale.check_custom_edges("f", [-1, 0, 2.5]).tolist() == [-1.0, 0.0, 2.5]
    for b, m in ((0, 4), (257, 4), (True, 4), (2.0, 4), (20, 0), (20, False)):
        with pytest.raises(ValueError):
            ale.check_params(b, m)


def test_feature_checks():
    from databricks_kubernetes_mlops_poc_b200 import ale
    from databricks_kubernetes_mlops_poc_b200.schema import CATEGORICAL_FEATURES, NUMERIC_FEATURES

    assert ale.check_features(None, NUMERIC_FEATURES, CATEGORICAL_FEATURES) == NUMERIC_FEATURES
    assert ale.check_features("age", NUMERIC_FEATURES, CATEGORICAL_FEATURES) == ["age"]
    with pytest.raises(ValueError, match="partial_dependence"):
        ale.check_features(["education"], NUMERIC_FEATURES, CATEGORICAL_FEATURES)
    for bad in ([], ["nope"], ["age", "age"]):
        with pytest.raises(ValueError):
            ale.check_features(bad, NUMERIC_FEATURES, CATEGORICAL_FEATURES)


class StubModel:
    """A model with the one method the route calls, recording what it was asked."""

    def __init__(self):
        self.calls = []

    def accumulated_local_effects(self, df, features, *, bins, min_bin_points, custom_edges=None):
        from databricks_kubernetes_mlops_poc_b200 import ale
        from databricks_kubernetes_mlops_poc_b200.schema import CATEGORICAL_FEATURES, NUMERIC_FEATURES

        self.calls.append((len(df), features, bins, min_bin_points, custom_edges))
        features = ale.check_features(features, NUMERIC_FEATURES, CATEGORICAL_FEATURES)
        if min_bin_points == 99:  # stands for any ValueError of the model, such as a field without a present value
            raise ValueError("feature 'age': the column has no present value to build edges from")
        z = [np.array([0.0, 1.0, 2.0])] * len(features)
        return {"feature_names": features, "output": "probability", "rows": len(df), "constant_value": 0.25, "feature_values": z,
                "ale_values": [np.array([-0.1, 0.0, 0.1])] * len(features), "bin_effects": [np.array([0.1, 0.1])] * len(features),
                "bin_rows": [np.array([2, 1])] * len(features), "ale0": [0.05] * len(features)}


def test_route_contract_and_validation():
    from databricks_kubernetes_mlops_poc_b200.schema import NUMERIC_FEATURES
    from databricks_kubernetes_mlops_poc_b200.server import create_app

    stub = StubModel()
    body = [{"age": 30.0}, {"age": 40.0}, {}]
    with TestClient(create_app(model=stub), raise_server_exceptions=False) as c:
        r = c.post("/explain/ale", json=body)
        assert r.status_code == 200, r.text
        j = r.json()
        assert set(j) == {"feature_names", "output", "rows", "constant_value", "feature_values", "ale_values", "bin_effects", "bin_rows", "ale0"}
        assert j["feature_names"] == NUMERIC_FEATURES and j["bin_rows"][0] == [2, 1] and j["rows"] == 3
        assert stub.calls[-1] == (3, None, 20, 4, None)
        r = c.post("/explain/ale?feature=age&value=20&value=35.5&value=60&bins=5&min_bin_points=2", json=body)
        assert r.status_code == 200 and stub.calls[-1] == (3, ["age"], 5, 2, {"age": [20.0, 35.5, 60.0]})
        n_calls = len(stub.calls)
        for q in ("feature=nope", "feature=education", "feature=age&feature=age", "bins=0", "bins=257", "bins=x", "bins=2.5",
                  "min_bin_points=0", "min_bin_points=x", "feature=age&value=1", "feature=age&value=2&value=1",
                  "feature=age&value=1&value=x", "feature=age&value=1&value=inf", "value=1&value=2",
                  "feature=age&feature=credit_limit&value=1&value=2", "feature=age&value=1&value=1.00000001"):
            r = c.post(f"/explain/ale?{q}", json=body)
            assert r.status_code == 422, (q, r.text)
        assert len(stub.calls) == n_calls
        r = c.post("/explain/ale?feature=age&min_bin_points=99", json=body)  # the model's ValueError
        assert r.status_code == 422 and "no present value" in r.json()["detail"]
        spec = c.get("/openapi.json").json()["paths"]
        assert {p["name"] for p in spec["/explain/ale"]["post"]["parameters"]} == {"feature", "bins", "min_bin_points", "value"}
