"""TreeSHAP interaction values on the CPU: the conditioning oracle (tests/treeshap_interactions.py) against the interaction
index's definition, its sum rules, the path-table emulator (tests/path_walk_interactions.py) against the oracle, exact zeros
for fields that share no path, and POST /explain/interactions with a stub model."""

import json
import os

import numpy as np
import pytest

from test_explain_cpu import _edge_rows

SHALLOW = {
    "rf12d4": ("rf", dict(n_estimators=12, max_depth=4, random_state=0)),
    "gbdt30d3": ("gbdt", dict(n_estimators=30, max_depth=3, random_state=0)),
    "rf33d3": ("rf", dict(n_estimators=33, max_depth=3, random_state=0)),
}


@pytest.fixture(scope="module")
def shallow(curated):
    from oracle import reference_pipeline as rp

    tr = curated.iloc[:3000]
    out = {}
    for name, (kind, params) in SHALLOW.items():
        out[name] = rp.fit_reference_pipeline(tr, params) if kind == "rf" else rp.fit_gbdt_pipeline(tr, tr[rp.TARGET].to_numpy(), params)
    return out


def _dense(pipe, df):
    from oracle import treeshap as ts
    from oracle import treewalk as tw

    dump = tw.dump_pipeline(pipe)
    return dump, ts.dump_covers(pipe), tw.transform_dense(dump, *tw.encode_frame(dump, df))


def _emulate(pipe, df):
    import path_walk_interactions as pwi

    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer, flatten_pipeline

    flat = flatten_pipeline(pipe)
    table = flatten_explainer(pipe, flat)
    return pwi.explain_interactions_paths(table, flat.blob, RowEncoder(flat).encode_frame(df)), table


def test_fixtures_repeat_a_numeric_and_a_categorical_field(shallow):
    """Each shallow forest has a path that tests one numeric field twice and a path that tests one categorical field twice,
    so merging (flattener) and unwinding a repeated field (oracle) are checked against the definition."""
    from oracle import treeshap as ts
    from oracle import treewalk as tw

    for pipe in shallow.values():
        dump = tw.dump_pipeline(pipe)
        fields = ts.column_fields(dump)
        n_cat = len(dump["cat_offsets"]) - 1
        rep_num = rep_cat = False
        for t in range(dump["n_trees"]):
            lo = int(dump["tree_off"][t])
            L, R, F = dump["left"][lo:], dump["right"][lo:], dump["feature"][lo:]
            stack = [(0, ())]
            while stack:
                j, seen = stack.pop()
                if L[j] == -1:
                    continue
                f = int(fields[F[j]])
                rep_cat |= f in seen and f < n_cat
                rep_num |= f in seen and f >= n_cat
                stack += [(L[j], seen + (f,)), (R[j], seen + (f,))]
        assert rep_num and rep_cat


@pytest.mark.parametrize("name", sorted(SHALLOW))
def test_oracle_equals_brute_force(name, shallow, curated):
    import treeshap_interactions as ti

    pipe = shallow[name]
    dump, cov, X = _dense(pipe, _edge_rows(curated, pipe))
    phi2, base = ti.tree_shap_interactions(dump, cov, X)
    want, wbase = ti.brute_force_interactions(dump, cov, X)
    assert phi2.shape == (X.shape[0], 23, 23)
    assert np.abs(phi2 - want).max() <= 1e-13 and abs(base - wbase) <= 1e-13


@pytest.mark.parametrize("name", ["rf12d4", "gbdt30d3", "gbdt_small"])
def test_oracle_sum_rules(name, shallow, gbdt_small, curated):
    """Symmetric; each row sums to tree_shap's phi; each matrix sums to prediction - base."""
    import treeshap_interactions as ti

    from oracle import treeshap as ts
    from oracle import treewalk as tw

    pipe = gbdt_small if name == "gbdt_small" else shallow[name]
    df = _edge_rows(curated, pipe, n=100)
    dump, cov, X = _dense(pipe, df)
    phi2, base = ti.tree_shap_interactions(dump, cov, X)
    phi, pbase = ts.tree_shap(dump, cov, X)
    assert base == pbase
    assert np.abs(phi2 - phi2.transpose(0, 2, 1)).max() <= 1e-13
    assert np.abs(phi2.sum(axis=2) - phi).max() <= 1e-13
    p, _, raw = tw.walk_numpy(dump, X)
    assert np.abs(base + phi2.sum(axis=(1, 2)) - (p if dump["kind"] == tw.RF_MEAN else raw)).max() <= 1e-12


@pytest.mark.parametrize("which", ["rf100d6", "gbdt_small", "deep"])
def test_path_table_emulator_equals_oracle(which, request, curated):
    import treeshap_interactions as ti

    from oracle import reference_pipeline as rp

    if which == "deep":
        # two trees: the conditioning oracle runs Algorithm 2 twice per field a tree uses, slow on 24-deep trees
        pipe = rp.fit_reference_pipeline(curated.iloc[:6000], dict(n_estimators=2, max_depth=24, criterion="entropy", random_state=1))
        df = _edge_rows(curated, pipe, n=20).iloc[::10].reset_index(drop=True)
    else:
        pipe = request.getfixturevalue(which)
        df = _edge_rows(curated, pipe, n=200)
    (phi2, base), table = _emulate(pipe, df)
    from databricks_kubernetes_mlops_poc_b200.flatten import parse_explainer

    assert (parse_explainer(table)["max_len"] > 16) == (which == "deep")
    assert np.array_equal(phi2, phi2.transpose(0, 2, 1))
    dump, cov, X = _dense(pipe, df)
    want, wbase = ti.tree_shap_interactions(dump, cov, X)
    assert abs(base - wbase) <= 1e-12
    assert np.abs(phi2 - want).max() <= 1e-12


def test_fields_sharing_no_path_get_exactly_zero(shallow, curated):
    from databricks_kubernetes_mlops_poc_b200.flatten import parse_explainer

    pipe = shallow["rf33d3"]
    (phi2, _), table = _emulate(pipe, _edge_rows(curated, pipe))
    h = parse_explainer(table)
    together = np.zeros((23, 23), dtype=bool)
    for p in h["paths"]:
        f = h["elems"]["field"][p["first"] + 1 : p["first"] + p["len"]].astype(np.int64)
        together[np.ix_(f, f)] = True
    apart = ~together
    assert apart.sum() >= 100  # many pairs of a depth-3 forest never meet
    assert (phi2[:, apart] == 0.0).all()
    assert np.abs(phi2[:, together & ~np.eye(23, dtype=bool)]).max() > 0.0


# --------------------------------------------------------------------------------------------------------- HTTP (stub)
class StubModel:
    drift = None

    def __init__(self, explainer=True):
        from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES

        self.replicas = [self]
        self.explainer_attached = explainer
        self.all_features = list(ALL_FEATURES)

    def predict_proba1(self, df):
        return (df["credit_limit"].to_numpy() % 1000) / 1000.0

    def explain_interactions(self, df):
        n, F = len(df), len(self.all_features)
        phi2 = np.zeros((n, F, F))
        k = self.all_features.index("credit_limit")
        phi2[:, k, k] = self.predict_proba1(df) - 0.5
        return {"feature_names": self.all_features, "output": "probability", "base_value": 0.5,
                "interactions": phi2, "predictions": self.predict_proba1(df).tolist()}


def _client(model):
    from fastapi.testclient import TestClient

    from databricks_kubernetes_mlops_poc_b200.server import create_app

    return TestClient(create_app(model=model), raise_server_exceptions=False)


def test_http_explain_interactions_stub():
    from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES

    with _client(StubModel()) as c:
        paths = c.get("/openapi.json").json()["paths"]
        r = c.post("/explain/interactions", json=[{"credit_limit": 1250.0}, {}])
        assert r.status_code == 200
        j = r.json()
        assert set(j) == {"feature_names", "output", "base_value", "predictions", "interactions"}
        assert j["feature_names"] == ALL_FEATURES and j["output"] == "probability" and j["base_value"] == 0.5
        assert j["predictions"] == [0.25, 0.0]
        assert len(j["interactions"]) == 2 and all(len(m) == 23 and all(len(r) == 23 for r in m) for m in j["interactions"])
        k = ALL_FEATURES.index("credit_limit")
        assert j["interactions"][0][k][k] == -0.25
        assert c.post("/explain/interactions", json=[{"sex": 3}]).status_code == 422
        assert c.post("/explain/interactions", json=[]).status_code == 500
    with _client(StubModel(explainer=False)) as c:
        assert c.post("/explain/interactions", json=[{}]).status_code == 501
        assert c.post("/predict", json=[{}]).status_code == 200
    # the /predict and /explain entries are the ones the app served before /explain/interactions existed (recorded with
    # json.dump(app.openapi()["paths"][path], indent=1, sort_keys=True))
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    for path, name in (("/predict", "openapi_predict.json"), ("/explain", "openapi_explain.json")):
        with open(os.path.join(golden, name)) as f:
            assert paths[path] == json.load(f)
    assert "/explain/interactions" in paths


def test_explain_interactions_uses_the_first_gpu_only_under_its_lock():
    """On a multi-GPU model explain_interactions() runs on the first GPU's handle only: interaction values from its engine,
    predictions from its scoring replica with the classifier alone, never the group call that drives every GPU.  The first
    replica's lock is held across both calls."""
    import pandas as pd

    from databricks_kubernetes_mlops_poc_b200.model import B200Model
    from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES, sample_request
    from test_explain_cpu import _Replica, _Untouchable

    class Engine:
        def explain_interactions_rows(self, rows):
            return np.zeros((rows.shape[0], 23, 23)), 0.25

    class Encoder:
        def encode_frame(self, df):
            return np.zeros((len(df), 24), dtype=np.uint32)

    class Flat:
        agg_mode = 0

    log = []
    m = object.__new__(B200Model)
    m.explain_blob, m.all_features, m.flat = b"table", list(ALL_FEATURES), Flat()
    m.engine, m.encoder, m.group = Engine(), Encoder(), _Untouchable()
    m.replicas = [_Replica(0, log), _Replica(1, log)]
    df = pd.DataFrame(sample_request() * 3)
    df["credit_limit"] = [1250.0, 2500.0, 100.0]
    out = m.explain_interactions(df)
    assert log == [(0, False, True)] and not m.replicas[0].lock._is_owned()
    assert out["predictions"] == [0.25, 0.5, 0.1] and out["base_value"] == 0.25 and out["interactions"].shape == (3, 23, 23)
    m.explain_blob = None
    with pytest.raises(RuntimeError, match="no explainer"):
        m.explain_interactions(df)
