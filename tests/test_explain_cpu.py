"""TreeSHAP on the CPU: the numpy Algorithm-2 oracle against brute-force Shapley values, the path-table emulator
(tests/path_walk.py) against the oracle, local accuracy, b2f_paths_validate, and POST /explain with a stub model."""

import json
import os
import struct
import threading

import numpy as np
import pandas as pd
import pytest


def _edge_rows(curated, pipe, n=200, seed=3):
    """200 curated rows plus rows on every edge the preprocessing has: unknown, missing (None / NaN) and "missing"
    categories, NaN, +-0, +-3e38, and numerics exactly on a split threshold of ``pipe`` and one float32 ulp either side."""
    from oracle import reference_pipeline as rp
    from oracle import treewalk as tw

    rng = np.random.default_rng(seed)
    base = curated[rp.FEATURES].iloc[rng.integers(0, len(curated), n)].reset_index(drop=True).copy()
    edge = curated[rp.FEATURES].iloc[rng.integers(0, len(curated), 240)].reset_index(drop=True).copy()
    for name in rp.CATEGORICAL_FEATURES:
        col = edge[name].astype(object)
        r = rng.random(len(edge))
        col[r < 0.15] = "never_seen_category"
        col[(r >= 0.15) & (r < 0.25)] = None
        col[(r >= 0.25) & (r < 0.3)] = np.nan
        col[(r >= 0.3) & (r < 0.4)] = "missing"
        edge[name] = col
    dump = tw.dump_pipeline(pipe)
    n_ohe = int(dump["cat_offsets"][-1])
    nodes = np.nonzero((dump["left"] != -1) & (dump["feature"] >= n_ohe))[0]
    for i in range(len(edge)):
        j = nodes[rng.integers(len(nodes))]
        t = np.float32(dump["threshold"][j])
        edge.loc[i, rp.NUMERIC_FEATURES[int(dump["feature"][j]) - n_ohe]] = float(
            [t, np.nextafter(t, np.float32(np.inf)), np.nextafter(t, np.float32(-np.inf)), dump["threshold"][j]][i % 4])
    for name in rp.NUMERIC_FEATURES:
        col = edge[name].to_numpy(dtype=np.float64).copy()
        r = rng.random(len(edge))
        col[r < 0.05] = np.nan
        col[(r >= 0.05) & (r < 0.07)] = 0.0
        col[(r >= 0.07) & (r < 0.09)] = -0.0
        col[(r >= 0.09) & (r < 0.10)] = 3.0e38
        col[(r >= 0.10) & (r < 0.11)] = -3.0e38
        edge[name] = col
    return pd.concat([base, edge], ignore_index=True)


def _fit(curated, kind, **params):
    from oracle import reference_pipeline as rp

    tr = curated.iloc[:3000]
    if kind == "rf":
        return rp.fit_reference_pipeline(tr, params)
    return rp.fit_gbdt_pipeline(tr, tr[rp.TARGET].to_numpy(), params)


SHALLOW = {
    "rf8d3": ("rf", dict(n_estimators=8, max_depth=3, random_state=0)),
    "gbdt10d3": ("gbdt", dict(n_estimators=10, max_depth=3, random_state=0)),
    "stump": ("rf", dict(n_estimators=1, max_depth=1, random_state=0)),
    "rf33d3": ("rf", dict(n_estimators=33, max_depth=3, random_state=0)),
}


@pytest.fixture(scope="module")
def shallow(curated):
    return {k: _fit(curated, kind, **p) for k, (kind, p) in SHALLOW.items()}


def _dense(pipe, df):
    from oracle import treeshap as ts
    from oracle import treewalk as tw

    dump = tw.dump_pipeline(pipe)
    return dump, ts.dump_covers(pipe), tw.transform_dense(dump, *tw.encode_frame(dump, df))


@pytest.mark.parametrize("name", sorted(SHALLOW))
def test_oracle_equals_brute_force(name, shallow, curated):
    from oracle import treeshap as ts
    from oracle import treewalk as tw

    pipe = shallow[name]
    dump, cov, X = _dense(pipe, _edge_rows(curated, pipe))
    phi, base = ts.tree_shap(dump, cov, X)
    bphi, bbase = ts.brute_force_shap(dump, cov, X)
    assert np.abs(phi - bphi).max() <= 1e-13 and abs(base - bbase) <= 1e-13
    p, _, raw = tw.walk_numpy(dump, X)
    assert np.abs(base + phi.sum(axis=1) - (p if dump["kind"] == tw.RF_MEAN else raw)).max() <= 1e-12


def test_fixtures_merge_repeated_fields(shallow):
    """The shallow forests checked against brute force have paths that test one numeric field twice and one categorical
    field twice, so the oracle's unwinding of a repeated field (and the flattener's merging) is checked against the
    definition of the Shapley value."""
    from oracle import treeshap as ts
    from oracle import treewalk as tw

    rep_num = rep_cat = False
    for pipe in shallow.values():
        dump = tw.dump_pipeline(pipe)
        fields = ts.column_fields(dump)
        n_cat = len(dump["cat_offsets"]) - 1
        for t in range(dump["n_trees"]):
            lo, hi = int(dump["tree_off"][t]), int(dump["tree_off"][t + 1])
            L, R, F = dump["left"][lo:hi], dump["right"][lo:hi], dump["feature"][lo:hi]
            stack = [(0, ())]
            while stack:
                j, seen = stack.pop()
                if L[j] == -1:
                    continue
                f = int(fields[F[j]])
                if f in seen:
                    rep_cat |= f < n_cat
                    rep_num |= f >= n_cat
                stack += [(L[j], seen + (f,)), (R[j], seen + (f,))]
    assert rep_num and rep_cat


@pytest.mark.parametrize("which", ["rf100d6", "gbdt_small", "deep"])
def test_path_table_emulator_equals_oracle(which, request, curated):
    import path_walk

    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer, flatten_pipeline, parse_explainer
    from oracle import reference_pipeline as rp
    from oracle import treeshap as ts

    if which == "deep":
        pipe = rp.fit_reference_pipeline(curated.iloc[:6000], dict(n_estimators=37, max_depth=24, criterion="entropy", random_state=1))
    else:
        pipe = request.getfixturevalue(which)
    df = _edge_rows(curated, pipe, n=60 if which == "deep" else 200)
    if which == "deep":
        df = df.iloc[::4].reset_index(drop=True)
    flat = flatten_pipeline(pipe)
    table = flatten_explainer(pipe, flat)
    h = parse_explainer(table)
    assert h["max_len"] <= 24 and h["n_paths"] > 0
    rows = RowEncoder(flat).encode_frame(df)
    phi, base = path_walk.explain_paths(table, flat.blob, rows)
    dump, cov, X = _dense(pipe, df)
    want, wbase = ts.tree_shap(dump, cov, X)
    assert abs(base - wbase) <= 1e-12
    assert np.abs(phi - want).max() <= 1e-12


def test_unused_field_gets_exactly_zero(shallow, curated):
    from oracle import treeshap as ts

    pipe = shallow["stump"]
    dump, cov, X = _dense(pipe, _edge_rows(curated, pipe))
    phi, _ = ts.tree_shap(dump, cov, X)
    used = {int(ts.column_fields(dump)[f]) for f, l in zip(dump["feature"], dump["left"]) if l != -1}
    assert len(used) == 1
    for f in range(phi.shape[1]):
        if f not in used:
            assert (phi[:, f] == 0.0).all()


def _tables(shallow, rf100d6, gbdt_small):
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer

    return [flatten_explainer(p) for p in list(shallow.values()) + [rf100d6, gbdt_small]]


def test_paths_validate(shallow, rf100d6, gbdt_small):
    from databricks_kubernetes_mlops_poc_b200._cabi import B2FError
    from databricks_kubernetes_mlops_poc_b200.engine import validate_paths
    from databricks_kubernetes_mlops_poc_b200.flatten import parse_explainer

    for t in _tables(shallow, rf100d6, gbdt_small):
        validate_paths(t)
    t = _tables(shallow, rf100d6, gbdt_small)[-2]
    h = parse_explainer(t)
    with pytest.raises(B2FError, match="truncated"):
        validate_paths(t[:-48])
    with pytest.raises(B2FError, match="magic"):
        validate_paths(b"X" + t[1:])
    with pytest.raises(B2FError, match="version"):
        validate_paths(t[:8] + struct.pack("<I", 2) + t[12:])
    bad = bytearray(t)  # an element's field out of range
    off = h["elems_off"] + 48 * 1
    bad[off : off + 4] = struct.pack("<I", 23)
    with pytest.raises(B2FError, match="field"):
        validate_paths(bytes(bad))
    bad = bytearray(t)  # a path longer than 24
    bad[h["paths_off"] + 4 : h["paths_off"] + 8] = struct.pack("<I", 25)
    with pytest.raises(B2FError, match="path 0 malformed"):
        validate_paths(bytes(bad))
    bad = bytearray(t)  # max_len over 24
    bad[8 + 4 * 7 : 8 + 4 * 8] = struct.pack("<I", 25)
    with pytest.raises(B2FError, match="max_len"):
        validate_paths(bytes(bad))


def test_flattener_is_path_vectorised_and_fast(rf500d8):
    """rf500d8's 80 490 paths flatten in well under a minute on one CPU core (the time is printed with -s)."""
    import time

    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer, flatten_pipeline, parse_explainer

    flat = flatten_pipeline(rf500d8)
    t0 = time.perf_counter()
    h = parse_explainer(flatten_explainer(rf500d8, flat))
    dt = time.perf_counter() - t0
    print(f"flatten_explainer rf500d8: {h['n_paths']} paths, {h['n_elems']} elements, max length {h['max_len']}, {dt:.2f} s")
    assert h["max_len"] <= 9 and dt < 60


# --------------------------------------------------------------------------------------------------------- HTTP (stub)
class StubModel:
    drift = None
    all_features = None

    def __init__(self, explainer=True):
        from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES

        self.replicas = [self]
        self.explainer_attached = explainer
        self.all_features = list(ALL_FEATURES)

    def predict_proba1(self, df):
        return (df["credit_limit"].to_numpy() % 1000) / 1000.0

    def explain(self, df):
        n = len(df)
        contrib = np.zeros((n, len(self.all_features)))
        contrib[:, self.all_features.index("credit_limit")] = self.predict_proba1(df) - 0.5
        return {"feature_names": self.all_features, "output": "probability", "base_value": 0.5,
                "contributions": contrib, "predictions": self.predict_proba1(df).tolist()}


def _client(model):
    from fastapi.testclient import TestClient

    from databricks_kubernetes_mlops_poc_b200.server import create_app

    return TestClient(create_app(model=model), raise_server_exceptions=False)


def test_http_explain_stub():
    from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES

    with _client(StubModel()) as c:
        predict_entry = c.get("/openapi.json").json()["paths"]["/predict"]
        r = c.post("/explain", json=[{"credit_limit": 1250.0}, {}])
        assert r.status_code == 200
        j = r.json()
        assert set(j) == {"feature_names", "output", "base_value", "predictions", "contributions"}
        assert j["feature_names"] == ALL_FEATURES and j["output"] == "probability" and j["base_value"] == 0.5
        assert j["predictions"] == [0.25, 0.0]
        assert len(j["contributions"]) == 2 and all(len(row) == 23 for row in j["contributions"])
        assert c.post("/explain", json=[{"sex": 3}]).status_code == 422
        assert c.post("/explain", json=[]).status_code == 500

    with _client(StubModel(explainer=False)) as c:
        assert c.post("/explain", json=[{}]).status_code == 501
        assert c.post("/predict", json=[{}]).status_code == 200
    # /predict's whole OpenAPI entry is the one the app served before /explain existed (recorded from that app with
    # json.dump(app.openapi()["paths"]["/predict"], indent=1, sort_keys=True))
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "openapi_predict.json")) as f:
        assert predict_entry == json.load(f)


class _Replica:
    def __init__(self, idx, log):
        self.idx, self.log = idx, log
        self.lock = threading.RLock()

    def score(self, df, want_outliers=True):
        self.log.append((self.idx, want_outliers, self.lock._is_owned()))
        if self.idx:
            raise AssertionError("explain() must not touch another GPU's replica")
        return (df["credit_limit"].to_numpy(dtype=np.float64) % 1000) / 1000.0, None


class _Untouchable:
    def __getattr__(self, name):
        raise AssertionError(f"explain() must not use the multi-GPU group ({name})")


def test_explain_uses_the_first_gpu_only_under_its_lock():
    """On a multi-GPU model explain() runs entirely on the first GPU's handle -- contributions from its engine, predictions
    from its scoring replica (classifier only) -- and never enters the group call that drives every GPU's handle, whose
    replicas the HTTP batcher's other workers are using at the same time.  The first replica's lock is held across both
    calls, so the batcher's first worker cannot score on that handle in between."""
    from databricks_kubernetes_mlops_poc_b200.model import B200Model
    from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES, sample_request

    class Engine:
        def explain_rows(self, rows):
            return np.zeros((rows.shape[0], 23)), 0.25

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
    out = m.explain(df)
    assert log == [(0, False, True)] and not m.replicas[0].lock._is_owned()
    assert out["predictions"] == [0.25, 0.5, 0.1] and out["base_value"] == 0.25 and out["output"] == "probability"
