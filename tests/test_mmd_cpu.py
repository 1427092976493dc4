"""The MMD drift test on the CPU: the explicit-matrix restatement of alibi-detect's MMDDrift (oracle/mmd_drift.py) against
the algebraic form the kernels use (tests/mmd_walk.py), the median heuristic's index, the embedding's distances against
sklearn's dense vectors, the argument checks and draws of ``mmd.py``, a calibration on the curated table, and the route's
validation."""

import numpy as np
import pandas as pd
import pytest
from fastapi.testclient import TestClient

import mmd_walk
import schema_zoo as zoo

TOL = 1e-12


def _embedded(spec, pipe, ref: pd.DataFrame, batch: pd.DataFrame):
    """-> (emulator embeddings of ref and batch, the oracle's dense z-scored vectors of both)."""
    from databricks_kubernetes_mlops_poc_b200 import mmd
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline, parse_header

    flat = flatten_pipeline(pipe)
    enc = RowEncoder(flat)
    n_cat, n_num = len(flat.cat_features), len(flat.num_features)
    impute = parse_header(flat.blob)["impute"][n_cat:n_cat + n_num]
    rr, rb = enc.encode_frame(ref), enc.encode_frame(batch)
    mean, scale = mmd.standardization(mmd.numerics(rr, n_cat, n_num, impute))
    er, eb = mmd_walk.embed(rr, n_cat, n_num, impute, mean, scale), mmd_walk.embed(rb, n_cat, n_num, impute, mean, scale)

    def dense(df):
        x = zoo.dense(pipe, df[flat.all_features]).astype(np.float64)
        x[:, -n_num:] = (x[:, -n_num:] - mean) / scale
        return x

    return er, eb, dense(ref), dense(batch)


@pytest.mark.parametrize("name", ["tiny", "packed_wide", "over16"])
def test_embedding_distances_equal_dense_vectors(name):
    from oracle import mmd_drift as om

    spec, pipe = zoo.fitted(name)
    ref = zoo.make_frame(spec, 200, seed=3, target=False)
    edges = zoo.edge_rows(spec, pipe, n=120, seed=5)
    # +-3e38 squares past float64's range only through the z-scores' scale; keep them out of the distance check
    nums = zoo.num_names(spec)
    big = np.abs(edges[nums].to_numpy(dtype=np.float64)) > 1e30
    edges = edges[~big.any(axis=1)].reset_index(drop=True)
    (zr, cr), (zb, cb), xr, xb = _embedded(spec, pipe, ref, edges)
    got = mmd_walk.dists(zb, cb, zr, cr)
    want = om.pairwise_sq(xb, xr)
    assert np.abs(got - want).max() <= TOL * max(1.0, np.abs(want).max())
    got = mmd_walk.dists(zb, cb, zb, cb)
    want = om.pairwise_sq(xb, xb)
    assert np.abs(got - want).max() <= TOL * max(1.0, np.abs(want).max())


@pytest.mark.parametrize("n", [2, 3, 4, 5, 10, 51, 200])
def test_sigma_median_index_is_the_middle_pair(n):
    from oracle import mmd_drift as om

    rng = np.random.default_rng(n)
    x = rng.normal(size=(n, 4))
    x[n // 3] = x[0]  # a zero pair
    d = om.pairwise_sq(x, x)
    pairs = np.sort(d[np.triu_indices(n, 1)])
    assert len(pairs) == n * (n - 1) // 2
    k = om.median_pair_index(n)
    assert k == (len(pairs) - 1) // 2
    assert om.sigma_median(x) == float(np.sqrt(0.5 * pairs[k]))
    # the same index into alibi's flattened n x n matrix
    flat = np.sort(np.where(np.eye(n, dtype=bool), 0.0, d).ravel())
    assert flat[n + (n * n - n) // 2 - 1] == pairs[k]


@pytest.mark.parametrize("name,n_ref,m", [("tiny", 40, 7), ("tiny", 30, 45), ("packed_wide", 60, 2), ("packed_wide", 25, 25),
                                          ("over16", 50, 31), ("over16", 12, 40)])
def test_explicit_matrix_equals_the_algebraic_form(name, n_ref, m):
    from databricks_kubernetes_mlops_poc_b200 import mmd
    from oracle import mmd_drift as om

    spec, pipe = zoo.fitted(name)
    ref = zoo.make_frame(spec, n_ref, seed=11, target=False)
    batch = zoo.make_frame(spec, m, seed=12, target=False)
    (zr, cr), (zb, cb), xr, xb = _embedded(spec, pipe, ref, batch)
    subsets = mmd.draw_subsets(n_ref, m, 40, 5)
    want = om.mmd_drift(xr, xb, subsets)
    sigma = mmd_walk.sigma(zr, cr)
    assert abs(sigma - want["sigma"]) <= TOL * want["sigma"]
    got, terms = mmd_walk.statistics(zr, cr, zb, cb, subsets, sigma)
    assert abs(got[0] - want["distance"]) <= TOL * terms[0]
    assert (np.abs(got[1:] - want["distance_permuted"]) <= TOL * terms[1:]).all()
    res = mmd.result(got[0], got[1:], 0.05, sigma, n_ref, m)
    assert res["p_val"] == want["p_val"] or np.any(np.abs(got[1:] - got[0]) <= TOL * terms[1:])


def test_draws_and_argument_checks():
    from databricks_kubernetes_mlops_poc_b200 import mmd

    for n_ref, m in ((5, 3), (3, 5), (100, 100), (2, 2)):
        s = min(n_ref, m)
        sub = mmd.draw_subsets(n_ref, m, 50, 9)
        assert sub.dtype == np.int32 and sub.shape == (50, s)
        assert (np.diff(sub, axis=1) > 0).all() and sub.min() >= 0 and sub.max() < n_ref + m
        assert np.array_equal(sub, mmd.draw_subsets(n_ref, m, 50, 9))
        rng = np.random.default_rng(9)
        assert np.array_equal(sub[0], np.sort(rng.choice(n_ref + m, s, replace=False, shuffle=False)))
        assert np.array_equal(sub[1], np.sort(rng.choice(n_ref + m, s, replace=False, shuffle=False)))
    assert not np.array_equal(mmd.draw_subsets(50, 10, 5, 0), mmd.draw_subsets(50, 10, 5, 1))
    # uniform: every pool index is drawn about equally often
    counts = np.bincount(mmd.draw_subsets(6, 3, 6000, 0).ravel(), minlength=9)
    assert np.abs(counts / 6000 - 3 / 9).max() < 0.03

    assert mmd.check_request(2, 10, 100, 0.05, 0) == (100, 0.05, 0)
    for bad in (dict(m=1), dict(n_permutations=0), dict(n_permutations=10001), dict(n_permutations=2.5), dict(n_permutations=True),
                dict(p_val=0.0), dict(p_val=1.5), dict(p_val=float("nan")), dict(random_state=-1), dict(random_state=1.5)):
        kw = dict(m=10, n_ref=10, n_permutations=100, p_val=0.05, random_state=0) | bad
        with pytest.raises(ValueError):
            mmd.check_request(**kw)
    # the pair budget: B * s (s - 1) / 2 <= 2^36
    s = 30000
    ok = mmd.PAIR_BUDGET // (s * (s - 1) // 2)
    mmd.check_request(65536, s, ok, 0.05, 0)
    with pytest.raises(ValueError, match="budget"):
        mmd.check_request(65536, s, ok + 1, 0.05, 0)
    for bad in (0.0, -1.0, float("inf"), float("nan")):
        with pytest.raises(ValueError):
            mmd.check_sigma(bad)
    assert mmd.check_sigma(None) is None and mmd.check_sigma(2) == 2.0
    with pytest.raises(ValueError):
        mmd.check_reference(1)
    with pytest.raises(ValueError):
        mmd.check_reference(mmd.MAX_REFERENCE + 1)

    perm = np.array([0.3, 0.1, 0.2, 0.5])
    r = mmd.result(0.2, perm, 0.5, 1.5, 10, 4)
    assert r["p_val"] == 0.75 and r["is_drift"] == 0 and r["distance_threshold"] == 0.2 and r["threshold"] == 0.5
    assert mmd.result(0.6, perm, 1.0, 1.5, 10, 4)["distance_threshold"] == 0.1  # index clamped to B - 1
    assert mmd.result(0.6, perm, 0.05, 1.5, 10, 4)["is_drift"] == 1


def test_calibration_joint_shift_on_the_oracle(curated, rf100d6):
    from databricks_kubernetes_mlops_poc_b200 import mmd
    from oracle import drift as od
    from oracle import mmd_drift as om
    from oracle import reference_pipeline as rp

    ref, held, shuffled = mmd_walk.calibration_frames(curated)
    # the marginals are kept: every per-field test is quiet on the shuffled rows
    assert od.tabular_drift_p_values(ref, shuffled, rp.CATEGORICAL_FEATURES).min() > 0.05
    n_num = len(rp.NUMERIC_FEATURES)
    pre = rf100d6.named_steps["preprocessor"]

    def dense(df):
        x = pre.transform(df[rp.FEATURES])
        return (x.toarray() if hasattr(x, "toarray") else np.asarray(x)).astype(np.float32).astype(np.float64)

    xr = dense(ref)
    mean, scale = mmd.standardization(xr[:, -n_num:])

    def z(x):
        x = x.copy()
        x[:, -n_num:] = (x[:, -n_num:] - mean) / scale
        return x

    subsets = mmd.draw_subsets(5000, 500, 100, 0)
    sigma = om.sigma_median(z(xr))
    assert om.mmd_drift(z(xr), z(dense(held)), subsets, sigma=sigma)["p_val"] > 0.05
    out = om.mmd_drift(z(xr), z(dense(shuffled)), subsets, sigma=sigma)
    assert out["p_val"] < 0.05 and out["is_drift"] == 1


class StubModel:
    def __init__(self, attached=True):
        self.mmd_reference_attached = attached
        self.mmd_reference_rows = 1000 if attached else 0
        self.calls = []

    def mmd_drift(self, df, *, n_permutations, p_val, random_state):
        from databricks_kubernetes_mlops_poc_b200 import mmd

        self.calls.append((df, n_permutations, p_val, random_state))
        return mmd.result(0.01, np.linspace(0.0, 0.02, n_permutations), p_val, 2.5, self.mmd_reference_rows, len(df))


def test_route_contract_and_validation():
    from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES
    from databricks_kubernetes_mlops_poc_b200.server import create_app

    stub = StubModel()
    body = [{"age": 30.0}, {"sex": "female"}, {}]
    with TestClient(create_app(model=stub), raise_server_exceptions=False) as c:
        r = c.post("/drift/mmd", json=body)
        assert r.status_code == 200, r.text
        j = r.json()
        assert set(j) == {"is_drift", "distance", "p_val", "threshold", "distance_threshold", "sigma", "n_permutations", "reference_rows", "rows"}
        assert j["rows"] == 3 and j["n_permutations"] == 100 and j["threshold"] == 0.05 and j["reference_rows"] == 1000
        df, b, p, rs = stub.calls[-1]
        assert list(df.columns) == ALL_FEATURES and (b, p, rs) == (100, 0.05, 0) and df.loc[0, "age"] == 30.0
        r = c.post("/drift/mmd?n_permutations=7&p_val=0.2&random_state=3", json=body)
        assert r.status_code == 200 and r.json()["n_permutations"] == 7 and stub.calls[-1][1:] == (7, 0.2, 3)
        n_calls = len(stub.calls)
        for q in ("n_permutations=0", "n_permutations=10001", "n_permutations=x", "p_val=0", "p_val=2", "random_state=-1",
                  "random_state=1.5"):
            r = c.post(f"/drift/mmd?{q}", json=body)
            assert r.status_code == 422, (q, r.text)
        assert c.post("/drift/mmd", json=body[:1]).status_code == 422
        assert c.post("/drift/mmd", json=[]).status_code == 422
        # 10 000 permutations of 4 000 rows are 8e10 kernel pairs, above the 2^36 budget
        stub.mmd_reference_rows = 100000
        big = [{}] * 4000
        r = c.post("/drift/mmd?n_permutations=10000", json=big)
        assert r.status_code == 422 and "budget" in r.json()["detail"]
        assert len(stub.calls) == n_calls
    with TestClient(create_app(model=StubModel(attached=False)), raise_server_exceptions=False) as c:
        assert c.post("/drift/mmd", json=body).status_code == 501
