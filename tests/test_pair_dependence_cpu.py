"""Two-way partial dependence and the H-statistic on the CPU: the numpy emulator of k_pair_dependence (tests/pair_walk.py)
against scikit-learn's two-way ``partial_dependence(method="brute")`` to 1e-12 (numeric x numeric, categorical x numeric,
categorical x categorical) with sklearn's grid values and Cartesian order; the H^2 restatement of ``interaction.py`` on
emulated means against a brute numpy form on ``predict_proba``; the sample draw; dedupe and map-back; the routes' 422s."""

import itertools

import numpy as np
import pandas as pd
import pytest
from fastapi.testclient import TestClient
from sklearn.inspection import partial_dependence

from pair_walk import pair_walk

TOL = 1e-12


def _encoder(pipe):
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline

    flat = flatten_pipeline(pipe)
    return flat, RowEncoder(flat)


def _emulated_pair(pipe, X, a, b, categorical, grid_resolution=100):
    """-> (grid a, grid b, individual (n, g_a, g_b), deepest stack), points built as B200Model.pair_dependence builds them."""
    from databricks_kubernetes_mlops_poc_b200 import dependence, interaction

    flat, enc = _encoder(pipe)
    ga = dependence.grid_from_column(X[a], a in categorical, grid_resolution).tolist()
    gb = dependence.grid_from_column(X[b], b in categorical, grid_resolution).tolist()
    pts = interaction.cartesian(dependence.encode_grid(enc, a, ga), dependence.encode_grid(enc, b, gb))
    out, deepest = pair_walk(flat.blob, enc.encode_frame(X), [(dependence.word_of(enc, a), dependence.word_of(enc, b), 0, len(pts))], pts)
    return ga, gb, out.reshape(len(X), len(ga), len(gb)), deepest


@pytest.mark.parametrize("pair", [("credit_limit", "age"), ("education", "credit_limit"), ("repayment_status_1", "education")])
def test_emulator_matches_sklearn_two_way(rf100d6, curated, pair):
    from oracle import reference_pipeline as rp

    X = curated[rp.FEATURES].iloc[:30].reset_index(drop=True)
    ga, gb, ind, deepest = _emulated_pair(rf100d6, X, *pair, rp.CATEGORICAL_FEATURES, grid_resolution=9)
    want = partial_dependence(rf100d6, X, list(pair), method="brute", kind="both", categorical_features=rp.CATEGORICAL_FEATURES,
                              grid_resolution=9)
    # sklearn's grids, and its Cartesian order (the first field slowest)
    assert [list(g) for g in want["grid_values"]] == [ga, gb]
    assert want["individual"].shape == (1, len(X), len(ga), len(gb))
    assert np.abs(ind - want["individual"][0]).max() <= TOL
    assert np.abs(ind.mean(axis=0) - want["average"][0]).max() <= TOL
    assert deepest <= 6  # one stack entry per level at most


def test_one_way_probe_is_k6(rf100d6, curated):
    """A probe with no second word scores as K6's one-word walk."""
    from dependence_walk import pd_walk

    from databricks_kubernetes_mlops_poc_b200 import dependence
    from oracle import reference_pipeline as rp

    flat, enc = _encoder(rf100d6)
    X = curated[rp.FEATURES].iloc[:12]
    rows = enc.encode_frame(X)
    g = dependence.encode_grid(enc, "credit_limit", np.linspace(1e4, 5e5, 40).tolist())
    w = dependence.word_of(enc, "credit_limit")
    want, _ = pd_walk(flat.blob, rows, [(w, 0, len(g))], g)
    pts = np.stack([g, np.full(len(g), 12345, dtype=np.uint32)], axis=1)
    got, _ = pair_walk(flat.blob, rows, [(w, -1, 0, len(g))], pts)
    assert np.array_equal(got, want)


def test_cartesian_and_check_pairs():
    from databricks_kubernetes_mlops_poc_b200 import interaction
    from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES

    pts = interaction.cartesian(np.array([1, 2, 3], np.uint32), np.array([7, 8], np.uint32))
    assert pts.tolist() == [[1, 7], [1, 8], [2, 7], [2, 8], [3, 7], [3, 8]]
    assert interaction.check_pairs(("age", "sex"), ALL_FEATURES) == [("age", "sex")]
    assert interaction.check_pairs([["age", "sex"], ("sex", "age")], ALL_FEATURES) == [("age", "sex"), ("sex", "age")]
    for bad in ([], [("age", "age")], [("age", "nope")], [("age",)]):
        with pytest.raises(ValueError):
            interaction.check_pairs(bad, ALL_FEATURES)


def _brute_h2(pipe, X, j, k):
    """H^2, numerator, denominator of fields j, k over all rows of X from predict_proba on the materialised n x n rows."""
    n = len(X)

    def F(cols):
        big = pd.concat([X] * n, ignore_index=True)  # block i: every row l with the columns of row i
        for c in cols:
            big[c] = np.repeat(X[c].to_numpy(), n)
        return pipe.predict_proba(big)[:, 1].reshape(n, n).mean(axis=1)

    Fjk, Fj, Fk = F([j, k]), F([j]), F([k])
    c = [v - v.mean() for v in (Fjk, Fj, Fk)]
    num, den = float(np.sum((c[0] - c[1] - c[2]) ** 2)), float(np.sum(c[0] ** 2))
    return num / den, num, den


def test_h_statistic_restatement_against_brute(rf100d6, curated):
    """interaction.py's plan (distinct points per probe, means over S, map-back) on the emulator's means equals the brute
    form on predict_proba."""
    from databricks_kubernetes_mlops_poc_b200 import dependence, interaction
    from databricks_kubernetes_mlops_poc_b200.flatten import parse_header
    from oracle import reference_pipeline as rp

    flat, enc = _encoder(rf100d6)
    X = curated[rp.FEATURES].iloc[100:124].reset_index(drop=True)
    X.loc[3, "age"] = np.nan  # imputed before dedupe: the median's point
    features = ["credit_limit", "age", "education", "repayment_status_1"]
    rows = enc.encode_frame(X)
    words = interaction.impute(rows, enc.n_cat, len(enc.num_features), parse_header(flat.blob)["impute"])
    fields = [dependence.word_of(enc, f) for f in features]
    probes, points, maps = interaction.strength_plan(words, fields, [f in rp.CATEGORICAL_FEATURES for f in features])
    assert len(probes) == 4 + 6 and all(p[1] == -1 for p in probes[:4])
    out, _ = pair_walk(flat.blob, rows, probes, points)
    res = interaction.strength_result(out.mean(axis=0), maps, features)
    assert res["pairs"] == list(itertools.combinations(features, 2))
    for p, (j, k) in enumerate(res["pairs"]):
        h, num, den = _brute_h2(rf100d6, X, j, k)
        assert abs(res["numerator"][p] - num) <= 1e-9 * max(num, 1e-300) + 1e-18
        assert abs(res["denominator"][p] - den) <= 1e-9 * den
        assert abs(res["h_squared"][p] - h) <= 1e-9 * h + 1e-15
    m = res["matrix"]
    assert np.isnan(np.diag(m)).all() and np.array_equal(m, m.T, equal_nan=True)


def test_h_squared_nan_where_flat():
    from databricks_kubernetes_mlops_poc_b200 import interaction

    flat = np.full(5, 0.25)
    h, num, den = interaction.h_squared(flat, flat, flat)
    assert np.isnan(h) and num == 0.0 and den == 0.0


def test_sample_draw():
    from databricks_kubernetes_mlops_poc_b200 import interaction

    assert np.array_equal(interaction.sample_rows(50, 1000, 0), np.arange(50))
    a = interaction.sample_rows(5000, 1000, 7)
    assert np.array_equal(a, np.random.RandomState(7).choice(5000, 1000, replace=False))
    assert np.array_equal(a, interaction.sample_rows(5000, 1000, 7)) and not np.array_equal(a, interaction.sample_rows(5000, 1000, 8))
    assert len(set(a.tolist())) == 1000
    with pytest.raises(ValueError):
        interaction.sample_rows(1, 1000, 0)
    for s, r in ((1, 0), (10001, 0), (True, 0), (2.5, 0), (100, -1), (100, 2**32)):
        with pytest.raises(ValueError):
            interaction.check_sample(s, r)
    assert interaction.check_sample(np.int64(10000), 0) == (10000, 0)


def test_dedupe_and_map_back():
    from databricks_kubernetes_mlops_poc_b200 import interaction

    rng = np.random.default_rng(0)
    num = rng.choice(np.array([3.5, -1.0, 0.0, -0.0, 2e5], dtype=np.float32), 400).view(np.uint32)
    cat = rng.integers(-1, 4, 400).astype(np.int32).view(np.uint32)
    pts, inv = interaction.distinct_points([cat, num], [True, False])
    assert np.array_equal(pts[inv], np.stack([cat, num], axis=1))  # map-back
    assert len({tuple(p) for p in pts.tolist()}) == len(pts) == len({(int(c), int(v)) for c, v in zip(cat, num)})
    keys = [(int(c), float(v)) for c, v in zip(pts[:, 0].view(np.int32), pts[:, 1].view(np.float32))]
    assert keys == sorted(keys)  # value order, the first column slowest (codes -1 first)
    one, inv1 = interaction.distinct_points([num], [False])
    assert np.array_equal(one[inv1, 0], num) and list(one[:, 0].view(np.float32)) == sorted(one[:, 0].view(np.float32))


def test_strength_result_shapes():
    from databricks_kubernetes_mlops_poc_b200 import interaction

    words = np.zeros((6, 24), dtype=np.uint32)
    words[:, 0] = [0, 1, 0, 1, 2, 2]
    words[:, 9] = np.array([1, 2, 3, 1, 2, 3], dtype=np.float32).view(np.uint32)
    words[:, 10] = np.array([5, 5, 5, 5, 5, 5], dtype=np.float32).view(np.uint32)
    probes, points, maps = interaction.strength_plan(words, [0, 9, 10], [True, False, False])
    assert [p[3] for p in probes] == [3, 3, 1, 6, 3, 3]
    assert [p[2] for p in probes] == [0, 3, 6, 7, 13, 16] and points.shape == (19, 2)
    means = np.arange(19, dtype=np.float64)
    res = interaction.strength_result(means, maps, ["a", "b", "c"])
    assert res["pairs"] == [("a", "b"), ("a", "c"), ("b", "c")] and res["matrix"].shape == (3, 3)
    assert np.isnan(res["h_squared"][2]) or res["denominator"][2] > 0


class StubModel:
    """A model with the two methods the routes call, recording what they were asked."""

    categorical_features = ["sex", "education", "marriage"] + [f"repayment_status_{i}" for i in range(1, 7)]

    def __init__(self):
        self.calls = []

    def pair_grids(self, df, pairs, *, grid_resolution=100, custom_values=None, grid_frame=None):
        from databricks_kubernetes_mlops_poc_b200 import interaction

        (a, b), = pairs
        g = lambda f: list(range(300)) if f == "age" and grid_resolution == 99 else list(range(grid_resolution if f != "sex" else 2))
        out = [[g(a), g(b)]]
        for ga in out[0]:
            if len(ga) > interaction.MAX_AXIS_POINTS:
                raise ValueError("too many grid points")
        return out

    def pair_dependence(self, df, pairs, *, kind, custom_values):
        self.calls.append(("pair", len(df), pairs, kind))
        (a, b), = pairs
        ga, gb = custom_values[a], custom_values[b]
        res = {"output": "probability", "grid_values": [[ga, gb]], "feature_names": pairs}
        if kind in ("average", "both"):
            res["average"] = [np.zeros((len(ga), len(gb)))]
        if kind in ("individual", "both"):
            res["individual"] = [np.zeros((len(df), len(ga), len(gb)))]
        return res

    def interaction_strength(self, df, features, *, sample, random_state):
        from databricks_kubernetes_mlops_poc_b200 import interaction
        from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES

        self.calls.append(("strength", len(df), features, sample, random_state))
        features = interaction.check_features(features, ALL_FEATURES)
        F = len(features)
        means = np.linspace(0.1, 0.9, 64)
        res = {"pairs": list(itertools.combinations(features, 2)), "feature_names": features, "rows": min(len(df), sample)}
        P = len(res["pairs"])
        res["h_squared"], res["numerator"], res["denominator"] = np.full(P, np.nan), np.zeros(P), np.zeros(P)
        res["h_squared"][0] = means[0]
        res["matrix"] = np.full((F, F), np.nan)
        return res


def test_routes_contract_and_validation():
    from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES
    from databricks_kubernetes_mlops_poc_b200.server import create_app

    stub = StubModel()
    body = [{"age": 30.0}, {"sex": "female"}, {}]
    with TestClient(create_app(model=stub), raise_server_exceptions=False) as c:
        r = c.post("/explain/dependence/pair?feature=age&feature=sex&grid_resolution=5&kind=both", json=body)
        assert r.status_code == 200, r.text
        j = r.json()
        assert j["feature_names"] == ["age", "sex"] and j["grid_values"] == [list(range(5)), [0, 1]]
        assert np.asarray(j["average"]).shape == (5, 2) and np.asarray(j["individual"]).shape == (3, 5, 2)
        assert stub.calls[-1] == ("pair", 3, [("age", "sex")], "both")
        n_calls = len(stub.calls)
        for q in ("feature=age", "feature=age&feature=sex&feature=education", "feature=age&feature=age", "feature=age&feature=nope",
                  "feature=age&feature=sex&kind=x", "feature=age&feature=sex&grid_resolution=1",
                  "feature=age&feature=sex&grid_resolution=x", "feature=age&feature=sex&grid_resolution=257",
                  "feature=age&feature=sex&grid_resolution=99",  # an axis of 300 points
                  "", "feature=age&feature=credit_limit&grid_resolution=256&kind=individual"):
            big = body if "256" not in q else [{}] * 300  # 300 x 256 x 256 > 2^24 curve values
            r = c.post(f"/explain/dependence/pair?{q}", json=big)
            assert r.status_code == 422, (q, r.text)
        assert len(stub.calls) == n_calls
        # the average alone holds no curves: no 2^24 limit
        r = c.post("/explain/dependence/pair?feature=age&feature=credit_limit&grid_resolution=256", json=[{}] * 300)
        assert r.status_code == 200 and "individual" not in r.json()

        r = c.post("/explain/interaction_strength", json=body)
        assert r.status_code == 200, r.text
        j = r.json()
        assert set(j) == {"feature_names", "rows", "pairs", "h_squared", "numerator", "denominator", "matrix"}
        assert j["feature_names"] == ALL_FEATURES and len(j["pairs"]) == 253 and j["h_squared"][1] is None
        assert stub.calls[-1] == ("strength", 3, None, 1000, 0)
        r = c.post("/explain/interaction_strength?feature=age&feature=sex&sample=50&random_state=3", json=body)
        assert r.status_code == 200 and stub.calls[-1] == ("strength", 3, ["age", "sex"], 50, 3)
        assert r.json()["pairs"] == [["age", "sex"]] and r.json()["matrix"] == [[None, None], [None, None]]
        n_calls = len(stub.calls)
        for q in ("feature=age", "feature=age&feature=age", "feature=nope&feature=age", "sample=1", "sample=10001", "sample=x",
                  "random_state=-1", "random_state=1.5", f"random_state={2**32}"):
            r = c.post(f"/explain/interaction_strength?{q}", json=body)
            assert r.status_code == 422, (q, r.text)
        assert c.post("/explain/interaction_strength", json=body[:1]).status_code == 422
        assert len(stub.calls) == n_calls
        spec = c.get("/openapi.json").json()["paths"]
        assert {p["name"] for p in spec["/explain/dependence/pair"]["post"]["parameters"]} == {"feature", "kind", "grid_resolution"}
        assert {p["name"] for p in spec["/explain/interaction_strength"]["post"]["parameters"]} == {"feature", "sample", "random_state"}
