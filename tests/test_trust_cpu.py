"""Trust scores on the CPU: the chunked emulator of the device search (tests/knn_walk.py) against the KDTree restatement of
alibi's TrustScore (tests/trust_oracle.py), the distance filter's percentile rule, ties on duplicate rows, the argument
checks of ``trust.py``, the route's validation, and the calibration of the score on the reference split."""

import numpy as np
import pytest
from fastapi.testclient import TestClient

import knn_walk
import trust_oracle as ot

REL = 1e-12


def _split(curated):
    from oracle import reference_pipeline as rp

    train, test = rp.reference_split(curated)
    return train.reset_index(drop=True), test.reset_index(drop=True)


class _Space:
    """The encoder and the emulator's embedding of one pipeline, with a reference frame's constants."""

    def __init__(self, pipe, ref):
        from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
        from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline, parse_header

        self.flat = flatten_pipeline(pipe)
        self.enc = RowEncoder(self.flat)
        n_cat, n_num = len(self.flat.cat_features), len(self.flat.num_features)
        impute = parse_header(self.flat.blob)["impute"][n_cat:n_cat + n_num]
        self.rows_ref = self.enc.encode_frame(ref[self.flat.all_features])
        self.mean, self.scale, self._embed = knn_walk.embedding(self.rows_ref, n_cat, n_num, impute)
        self.zr, self.cr = self._embed(self.rows_ref)

    def embed(self, frame):
        return self._embed(self.enc.encode_frame(frame[self.flat.all_features]))

    def neighbours(self, frame, cls, k):
        zq, cq = self.embed(frame)
        return knn_walk.neighbours(zq, cq, self.zr, self.cr, cls, k)


@pytest.mark.parametrize("dist_type", ["point", "mean"])
def test_emulator_scores_equal_the_kdtree_oracle(curated, rf100d6, dist_type):
    from databricks_kubernetes_mlops_poc_b200 import trust
    from oracle import reference_pipeline as rp

    train, test = _split(curated)
    queries = test.iloc[:400]
    y = train[rp.TARGET].to_numpy()
    sp = _Space(rf100d6, train)
    dist, index = sp.neighbours(queries, y, 2)
    proba = rf100d6.predict_proba(queries[rp.FEATURES])[:, 1]
    pred = rf100d6.predict(queries[rp.FEATURES]).astype(np.int64)
    got = trust.result(dist, index, proba, pred, [0, 1], np.arange(len(train)), 2, dist_type, [int((y == 0).sum()), int((y == 1).sum())])

    xr, mean, scale = ot.dense(rf100d6, train[rp.FEATURES])
    xq, _, _ = ot.dense(rf100d6, queries[rp.FEATURES], mean, scale)
    assert np.array_equal(mean, sp.mean) and np.array_equal(scale, sp.scale)
    ts = ot.TrustScore().fit(xr, y)
    want, other = ts.score(xq, pred, k=2, dist_type=dist_type)
    assert np.abs(got["trust_score"] - want).max() <= REL * np.abs(want).max()
    assert np.array_equal(got["closest_not_pred"], other) and np.array_equal(got["labels"], pred)
    d = ts.distances(xq, 2, dist_type)
    assert np.abs(got["distance_to_pred"] - d[np.arange(len(pred)), pred]).max() <= REL * d.max()
    # the neighbours' distances are the distances of the rows they name
    for c in (0, 1):
        nb = got["neighbours"][c]
        assert (y[nb["index"]] == c).all()
        assert np.allclose(nb["distance"], np.linalg.norm(xq[:, None, :] - xr[nb["index"]], axis=2), rtol=1e-13, atol=0)
        assert (np.diff(nb["distance"], axis=1) >= 0).all()


def test_filter_percentile_rule():
    from databricks_kubernetes_mlops_poc_b200 import trust

    r = np.array([1.0, 2.0, 3.0, 4.0, 5.0])
    assert trust.filter_keep(r, 0.2).tolist() == [True, True, True, True, False]  # percentile 80 = 4.2
    assert trust.filter_keep(np.array([1.0, 1.0, 1.0, 2.0]), 0.5).tolist() == [True, True, True, False]  # <= keeps the tie
    assert trust.filter_keep(np.array([3.0, 1.0, 2.0]), 0.0).all()  # alpha 0 keeps every row
    d = np.array([[0.0, 1.0, 4.0], [0.0, 2.0, 2.0]])
    assert trust.filter_radius(d, "point").tolist() == [4.0, 2.0]
    assert trust.filter_radius(d, "mean").tolist() == [2.5, 2.0]  # the first (the row itself) is left out


@pytest.mark.parametrize("dist_filter_type", ["point", "mean"])
def test_emulated_filter_keeps_the_oracles_rows(curated, rf100d6, dist_filter_type):
    from databricks_kubernetes_mlops_poc_b200 import trust
    from oracle import reference_pipeline as rp

    train, _ = _split(curated)
    ref = train.iloc[:3000]
    y = ref[rp.TARGET].to_numpy()
    sp = _Space(rf100d6, ref)
    dist, _ = sp.neighbours(ref, y, 11)
    xr, _, _ = ot.dense(rf100d6, ref[rp.FEATURES])
    for alpha in (0.0, 0.05, 0.3):
        want = ot.TrustScore(k_filter=10, alpha=alpha, filter_type="distance_knn", dist_filter_type=dist_filter_type).fit(xr, y).kept
        for c in (0, 1):
            own = np.nonzero(y == c)[0]
            keep = trust.filter_keep(trust.filter_radius(dist[own, c, :], dist_filter_type), alpha)
            assert np.array_equal(own[keep], want[c]), (alpha, c)
            if alpha == 0.0:
                assert keep.all()


def test_ties_on_duplicate_rows_go_to_the_lower_index(curated, rf100d6):
    from oracle import reference_pipeline as rp

    train, _ = _split(curated)
    y = train[rp.TARGET].to_numpy()
    sp = _Space(rf100d6, train)
    z = np.concatenate([sp.zr, sp.cr.astype(np.float64)], axis=1)
    _, first, inverse, counts = np.unique(z, axis=0, return_index=True, return_inverse=True, return_counts=True)
    assert 20 <= len(train) - len(first) <= 60  # about 34 exact duplicates in the training split
    dup = np.nonzero(counts[inverse.ravel()] > 1)[0]
    dist, index = sp.neighbours(train.iloc[dup], y, 2)
    for row, i in enumerate(dup):
        c = y[i]
        same = np.nonzero((inverse.ravel() == inverse.ravel()[i]) & (y == c))[0]
        assert dist[row, c, 0] == 0.0 and index[row, c, 0] == same[0]
        if len(same) > 1:
            assert dist[row, c, 1] == 0.0 and index[row, c, 1] == same[1]


def test_argument_checks():
    from databricks_kubernetes_mlops_poc_b200 import trust

    assert trust.check_fit(10, 10, 0.0, None, "point") == (10, 0.0, None, "point")
    assert trust.check_fit(2, 63, 0.5, "distance_knn", "mean") == (63, 0.5, "distance_knn", "mean")
    for bad in (dict(n=1), dict(n=131073), dict(k_filter=0), dict(k_filter=64), dict(k_filter=2.0), dict(k_filter=True), dict(alpha=1.0),
                dict(alpha=-0.1), dict(alpha=float("nan")), dict(filter_type="probability_knn"), dict(filter_type="knn"),
                dict(dist_filter_type="max")):
        kw = dict(n=100, k_filter=10, alpha=0.0, filter_type=None, dist_filter_type="point") | bad
        with pytest.raises(ValueError):
            trust.check_fit(**kw)
    assert trust.class_indices(np.array([1, 0, 1]), [0, 1]).tolist() == [1, 0, 1]
    with pytest.raises(ValueError):
        trust.class_indices(np.array([0, 2]), [0, 1])
    trust.check_class_rows(np.array([0, 1]), None, 10)
    with pytest.raises(ValueError):
        trust.check_class_rows(np.array([0, 0]), None, 10)
    with pytest.raises(ValueError, match="k_filter"):
        trust.check_class_rows(np.array([0] * 11 + [1] * 10), "distance_knn", 10)
    trust.check_class_rows(np.array([0] * 11 + [1] * 11), "distance_knn", 10)
    assert trust.check_score(2, "point", [5, 7]) == (2, "point")
    assert trust.check_score(64, "mean", [64, 100]) == (64, "mean")
    for k, dt, kept in ((0, "point", [5, 5]), (65, "point", [100, 100]), (6, "point", [5, 100]), (2.0, "point", [5, 5]), (2, "median", [5, 5])):
        with pytest.raises(ValueError):
            trust.check_score(k, dt, kept)


class StubModel:
    def __init__(self, attached=True):
        self.trust_reference_attached = attached
        self.trust_reference_rows = [30, 20] if attached else None
        self.calls = []

    def trust_score(self, df, *, k, dist_type):
        from databricks_kubernetes_mlops_poc_b200 import trust

        self.calls.append((len(df), k, dist_type))
        n = len(df)
        dist = np.tile(np.arange(1.0, k + 1.0), (n, 2, 1))
        dist[0, 1, :] = np.inf
        index = np.tile(np.arange(k, dtype=np.int32), (n, 2, 1))
        return trust.result(dist, index, np.full(n, 0.25), np.zeros(n, dtype=np.int64), [0, 1], np.arange(50), k, dist_type,
                            self.trust_reference_rows)


def test_route_contract_and_validation():
    from databricks_kubernetes_mlops_poc_b200.server import create_app

    stub = StubModel()
    body = [{"age": 30.0}, {"sex": "female"}, {}]
    with TestClient(create_app(model=stub), raise_server_exceptions=False) as c:
        r = c.post("/explain/trust", json=body)
        assert r.status_code == 200, r.text
        j = r.json()
        assert set(j) == {"trust_score", "closest_not_pred", "predictions", "labels", "distance_to_pred", "distance_to_other", "k",
                          "dist_type", "reference_rows"}
        assert j["k"] == 2 and j["dist_type"] == "point" and j["reference_rows"] == [30, 20] and stub.calls[-1] == (3, 2, "point")
        assert j["trust_score"][0] is None and j["distance_to_other"][0] is None and j["trust_score"][1] == 2.0 / (2.0 + 1e-12)
        assert j["labels"] == [0, 0, 0] and j["closest_not_pred"] == [1, 1, 1]
        r = c.post("/explain/trust?k=3&dist_type=mean&neighbours=true", json=body)
        assert r.status_code == 200 and stub.calls[-1] == (3, 3, "mean")
        nb = r.json()["neighbours"]
        assert [x["class"] for x in nb] == [0, 1] and nb[0]["index"][0] == [0, 1, 2] and nb[1]["distance"][0] == [None] * 3
        n_calls = len(stub.calls)
        for q in ("k=0", "k=65", "k=x", "k=2.5", "k=21", "dist_type=median", "neighbours=yes", "neighbours=1"):
            r = c.post(f"/explain/trust?{q}", json=body)
            assert r.status_code == 422, (q, r.text)
        assert len(stub.calls) == n_calls
        assert "/explain/trust" in c.get("/openapi.json").json()["paths"]
    with TestClient(create_app(model=StubModel(attached=False)), raise_server_exceptions=False) as c:
        assert c.post("/explain/trust", json=body).status_code == 501


def test_calibration_on_the_oracle(curated, rf100d6):
    """Low trust marks the decisions the model gets wrong more often: accuracy on the lowest-trust decile of the test split is
    below the overall accuracy, which is below the highest decile's."""
    from oracle import reference_pipeline as rp

    train, test = _split(curated)
    xr, mean, scale = ot.dense(rf100d6, train[rp.FEATURES])
    xq, _, _ = ot.dense(rf100d6, test[rp.FEATURES], mean, scale)
    pred = rf100d6.predict(test[rp.FEATURES]).astype(np.int64)
    score, _ = ot.TrustScore().fit(xr, train[rp.TARGET].to_numpy()).score(xq, pred, k=2)
    right = pred == test[rp.TARGET].to_numpy()
    order = np.argsort(score, kind="stable")
    tenth = len(order) // 10
    low, high = right[order[:tenth]].mean(), right[order[-tenth:]].mean()
    assert low < right.mean() < high, (low, right.mean(), high)
    assert 0.05 < (score < 1.0).mean() < 0.2
