"""Interventional TreeSHAP on the CPU: the per-pair recursion (tests/treeshap_interventional.py) against Shapley values from
the definition, the path-table emulator (tests/path_walk_interventional.py) against the recursion, the identities the GPU
tests rely on, the background file of a model directory, and POST /explain/interventional with a stub model."""

import json
import os

import numpy as np
import pandas as pd
import pytest

from test_explain_cpu import _edge_rows, _fit


def _pairs(curated, pipe, n, m, max_fields=10, seed=5):
    """n request rows (curated plus every edge of _edge_rows: unknown / missing categories, NaN, split thresholds), each
    with a background of m rows that differ from it in at most ``max_fields`` fields -> [(x, z)] frames."""
    from oracle import reference_pipeline as rp

    rng = np.random.default_rng(seed)
    pool = _edge_rows(curated, pipe)
    out = []
    for i in rng.choice(len(pool), n, replace=False):
        x = pool.iloc[[i]].reset_index(drop=True)
        z = pd.concat([x] * m, ignore_index=True)
        donors = pool.iloc[rng.integers(0, len(pool), m)].reset_index(drop=True)
        for j in range(m):
            for f in rng.choice(rp.FEATURES, int(rng.integers(0, max_fields + 1)), replace=False):
                z.at[j, f] = donors.at[j, f]
        out.append((x, z))
    return out


def _dense(pipe, df):
    from oracle import treewalk as tw

    dump = tw.dump_pipeline(pipe)
    return dump, tw.transform_dense(dump, *tw.encode_frame(dump, df))


@pytest.mark.parametrize("kind,params", [("rf", dict(n_estimators=8, max_depth=3, random_state=0)),
                                         ("gbdt", dict(n_estimators=10, max_depth=3, random_state=0)),
                                         ("rf", dict(n_estimators=3, max_depth=6, random_state=2))])
def test_recursion_equals_brute_force(kind, params, curated):
    import treeshap_interventional as ti

    pipe = _fit(curated, kind, **params)
    for x, z in _pairs(curated, pipe, 8, 6):
        dump, X = _dense(pipe, x)
        _, Z = _dense(pipe, z)
        phi, base = ti.interventional_shap(dump, X, Z)
        want, wbase = ti.interventional_bruteforce(dump, X, Z)
        assert np.abs(phi - want).max() <= 1e-12 and abs(base - wbase) <= 1e-12
        assert np.abs(base + phi.sum(axis=1) - ti.output(dump, X)).max() <= 1e-12


def _emulate_vs_recursion(pipe, x, z):
    import path_walk_interventional as pwi
    import treeshap_interventional as ti

    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer, flatten_pipeline

    flat = flatten_pipeline(pipe)
    table = flatten_explainer(pipe, flat)
    enc = RowEncoder(flat)
    phi, base, _ = pwi.explain_interventional(table, flat.blob, enc.encode_frame(x), enc.encode_frame(z))
    dump, X = _dense(pipe, x)
    _, Z = _dense(pipe, z)
    want, wbase = ti.interventional_shap(dump, X, Z)
    assert abs(base - wbase) <= 1e-12
    assert np.abs(phi - want).max() <= 1e-12
    assert np.abs(base + phi.sum(axis=1) - ti.output(dump, X)).max() <= 1e-12
    return phi


@pytest.mark.parametrize("which", ["rf100d6", "gbdt_small", "deep"])
def test_emulator_equals_recursion(which, request, curated):
    from oracle import reference_pipeline as rp

    if which == "deep":
        pipe = rp.fit_reference_pipeline(curated.iloc[:6000], dict(n_estimators=5, max_depth=24, criterion="entropy", random_state=1))
        from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer, parse_explainer

        assert parse_explainer(flatten_explainer(pipe))["max_len"] > 13  # paths longer than the histogram's 12 elements
    else:
        pipe = request.getfixturevalue(which)
    rng = np.random.default_rng(11)
    pool = _edge_rows(curated, pipe, n=40)
    x = pool.iloc[rng.choice(len(pool), 24, replace=False)].reset_index(drop=True)
    z = pool.iloc[rng.choice(len(pool), 30, replace=False)].reset_index(drop=True)
    _emulate_vs_recursion(pipe, x, z)


def test_identities(rf100d6, curated):
    """The row as its own background moves nothing; doubling every background row changes nothing."""
    import path_walk_interventional as pwi

    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer, flatten_pipeline
    from oracle import reference_pipeline as rp

    flat = flatten_pipeline(rf100d6)
    table = flatten_explainer(rf100d6, flat)
    enc = RowEncoder(flat)
    rows = enc.encode_frame(curated[rp.FEATURES].iloc[:40])
    for i in range(3):
        phi, _, _ = pwi.explain_interventional(table, flat.blob, rows[i : i + 1], rows[i : i + 1])
        assert (phi == 0.0).all()
    bg = rows[10:30]
    phi, base, nbytes = pwi.explain_interventional(table, flat.blob, rows[:10], bg)
    phi2, base2, nbytes2 = pwi.explain_interventional(table, flat.blob, rows[:10], np.concatenate([bg, bg]))
    assert np.abs(phi - phi2).max() <= 1e-14 and abs(base - base2) <= 1e-14 and nbytes2 == nbytes


def test_background_file_round_trip(tmp_path, rf100d6, curated):
    """explain_background.npz keeps the raw values the encoder sees: strings, None and NaN categories, NaN numerics."""
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline
    from databricks_kubernetes_mlops_poc_b200.model import _load_background, _save_background
    from oracle import reference_pipeline as rp

    flat = flatten_pipeline(rf100d6)
    df = _edge_rows(curated, rf100d6, n=50)
    path = str(tmp_path / "bg.npz")
    _save_background(path, flat, df[list(reversed(rp.FEATURES))])
    back = _load_background(path, flat)
    assert list(back.columns) == list(flat.all_features)
    enc = RowEncoder(flat)
    assert np.array_equal(enc.encode_frame(back), enc.encode_frame(df))
    with np.load(path) as z:
        assert all(z[name].dtype.kind in "Uf" for name in flat.all_features)


def test_background_needs_explain(rf100d6, curated):
    from databricks_kubernetes_mlops_poc_b200.model import B200Model
    from oracle import reference_pipeline as rp

    with pytest.raises(ValueError, match="explain=True"):
        B200Model.from_pipeline(rf100d6, background=curated[rp.FEATURES].iloc[:10])


# --------------------------------------------------------------------------------------------------------- HTTP (stub)
class StubModel:
    drift = None

    def __init__(self, explainer=True, background=True):
        from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES

        self.replicas = [self]
        self.explainer_attached = explainer
        self.background_attached = explainer and background
        self.all_features = list(ALL_FEATURES)

    def predict_proba1(self, df):
        return (df["credit_limit"].to_numpy() % 1000) / 1000.0

    def explain_interventional(self, df):
        if "education" in df and (df["education"] == "boom").any():
            raise RuntimeError("scoring failed")
        n = len(df)
        contrib = np.zeros((n, len(self.all_features)))
        contrib[:, self.all_features.index("credit_limit")] = self.predict_proba1(df) - 0.5
        return {"feature_names": self.all_features, "output": "probability", "base_value": 0.5, "contributions": contrib,
                "predictions": self.predict_proba1(df).tolist(), "background_rows": 100}


def _client(model):
    from fastapi.testclient import TestClient

    from databricks_kubernetes_mlops_poc_b200.server import create_app

    return TestClient(create_app(model=model), raise_server_exceptions=False)


def test_http_explain_interventional_stub():
    from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES

    with _client(StubModel()) as c:
        paths = c.get("/openapi.json").json()["paths"]
        r = c.post("/explain/interventional", json=[{"credit_limit": 1250.0}, {}])
        assert r.status_code == 200
        j = r.json()
        assert set(j) == {"feature_names", "output", "base_value", "predictions", "contributions", "background_rows"}
        assert j["feature_names"] == ALL_FEATURES and j["base_value"] == 0.5 and j["background_rows"] == 100
        assert j["predictions"] == [0.25, 0.0] and len(j["contributions"]) == 2 and all(len(r) == 23 for r in j["contributions"])
        assert c.post("/explain/interventional", json=[{"sex": 3}]).status_code == 422
        assert c.post("/explain/interventional", json=[]).status_code == 500
        assert c.post("/explain/interventional", json=[{"education": "boom"}]).status_code == 500
    for stub in (StubModel(explainer=False), StubModel(background=False)):
        with _client(stub) as c:
            r = c.post("/explain/interventional", json=[{}])
            assert r.status_code == 501 and "no " in r.json()["detail"]
            assert c.post("/predict", json=[{}]).status_code == 200
    # the entries of /predict and /explain are the ones recorded before this route existed
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    for path, name in (("/predict", "openapi_predict.json"), ("/explain", "openapi_explain.json")):
        with open(os.path.join(golden, name)) as f:
            assert paths[path] == json.load(f)
    assert "/explain/interventional" in paths
