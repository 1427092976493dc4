"""The online MMD drift detector without a GPU: the device decomposition's emulator (tests/mmd_online_walk.py) against
the literal restatement of alibi-detect's MMDDriftOnline (tests/mmd_online_oracle.py) -- bootstrap statistics,
thresholds, split and per-step statistics -- then every argument check, the exhaustion and split-limit errors, and the
``/drift/online`` routes through a stub model."""

import numpy as np
import pytest
from fastapi.testclient import TestClient

import mmd_online_oracle
import mmd_online_walk
import mmd_walk
import schema_zoo as zoo

TOL = 1e-12


def tolerance(emu, W: int) -> float:
    """TOL, times the size of the K_RR term where it exceeds 1: K_RR = T - 2 sum r_y + S_EE cancels down from T, and on a
    reference of 2W + 1 rows (rw = 2) T / (rw (rw - 1)) is of the order of n_ref^2."""
    rw = emu.n - (2 * W - 1)
    return TOL * max(1.0, emu.total / (rw * (rw - 1)))


def _embedded(name: str, n: int, seed: int, extra: int = 0):
    """-> (z, c) of n reference rows and (z, c) of ``extra`` stream rows of a zoo schema, in the MMD embedding."""
    from databricks_kubernetes_mlops_poc_b200 import mmd
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline, parse_header

    spec, pipe = zoo.fitted(name)
    flat = flatten_pipeline(pipe)
    enc = RowEncoder(flat)
    n_cat, n_num = len(flat.cat_features), len(flat.num_features)
    impute = parse_header(flat.blob)["impute"][n_cat:n_cat + n_num]
    rr = enc.encode_frame(zoo.make_frame(spec, n, seed=seed, target=False)[flat.all_features])
    mean, scale = mmd.standardization(mmd.numerics(rr, n_cat, n_num, impute))
    ref = mmd_walk.embed(rr, n_cat, n_num, impute, mean, scale)
    rs = enc.encode_frame(zoo.make_frame(spec, max(extra, 1), seed=seed + 100, target=False)[flat.all_features])
    return ref, mmd_walk.embed(rs, n_cat, n_num, impute, mean, scale)


CASES = [(W, n_ref, seed) for W in (2, 3, 10, 40) for n_ref in (2 * W + 1, 64, 600) for seed in (0, 1) if n_ref >= 2 * W + 1]


@pytest.mark.parametrize("W,n_ref,seed", CASES)
def test_emulator_equals_the_oracle(W, n_ref, seed):
    (z, c), (zs, cs) = _embedded("tiny", n_ref, seed=seed, extra=3 * W + 5)
    sigma = mmd_walk.sigma(z, c)
    ert, n_boot = 50.0, 120
    oracle = mmd_online_oracle.OnlineOracle(z, c, sigma, ert, W, n_boot, seed)
    emu = mmd_online_walk.Emulator(z, c, sigma)
    thr, perm, attempts, stats = emu.configure(ert, W, n_boot, seed)
    tol = tolerance(emu, W)
    assert np.abs(stats - oracle.bootstrap_stats).max() <= tol
    assert np.abs(thr - oracle.thresholds).max() <= tol
    assert attempts == oracle.split_attempts and np.array_equal(perm, oracle.perm)
    # the stream, cut into pieces of 1, 2 and the rest; then reset and replayed whole
    got = np.concatenate([emu.push(zs[:1], cs[:1]), emu.push(zs[1:3], cs[1:3]), emu.push(zs[3:], cs[3:])])
    want = [oracle.predict(zs[i], cs[i]) for i in range(len(zs))]
    assert np.abs(got - np.array([p["test_stat"] for p in want])).max() <= tol
    thr_t = thr[np.minimum(np.arange(1, len(zs) + 1), W - 1)]
    assert np.array_equal((got > thr_t).astype(int), [p["is_drift"] for p in want])
    assert np.abs(thr_t - np.array([p["threshold"] for p in want])).max() <= tol
    emu.reset()
    again = emu.push(zs, cs)
    assert again.tobytes() == got.tobytes()


def test_decomposition_equals_the_explicit_window_mmd():
    """stat_b(w) is the explicit unbiased MMD^2 of window w against the rest of the reference."""
    (z, c), _ = _embedded("packed_wide", 80, seed=4)
    sigma = mmd_walk.sigma(z, c)
    emu = mmd_online_walk.Emulator(z, c, sigma)
    W = 7
    y = np.random.default_rng(2).permutation(len(z))[-(2 * W - 1):]
    stats, _ = emu.bootstrap(y[None], W)
    R = np.setdiff1d(np.arange(len(z)), y)
    k = np.exp(-mmd_walk.dists(z, c, z, c) * emu.coef)
    for w in range(W):
        win = y[w:w + W]
        kxx = mmd_online_oracle.zero_diag(k[np.ix_(R, R)]).sum() / (len(R) * (len(R) - 1))
        kyy = mmd_online_oracle.zero_diag(k[np.ix_(win, win)]).sum() / (W * (W - 1))
        assert abs(stats[0, w] - (kxx + kyy - 2 * k[np.ix_(R, win)].mean())) <= TOL


def test_argument_checks(monkeypatch):
    from databricks_kubernetes_mlops_poc_b200 import mmd_online as mo

    assert mo.check_config(100, 50, 10, 1000, 0) == (50.0, 10, 1000, 0)
    for ert in (1, 0.5, float("inf"), float("nan"), "x", None):
        with pytest.raises(ValueError, match="ert"):
            mo.check_config(100, ert, 10, 1000, 0)
    for W in (1, 257, 2.0, True, "3"):
        with pytest.raises(ValueError, match="window_size"):
            mo.check_config(1000, 50, W, 1000, 0)
    with pytest.raises(ValueError, match="at least 2 \\* window_size \\+ 1 = 21 rows"):
        mo.check_config(20, 50, 10, 1000, 0)
    assert mo.check_config(21, 50, 10, 1, 0)[1] == 10
    for b in (0, 100001, 1.5, True):
        with pytest.raises(ValueError, match="n_bootstraps"):
            mo.check_config(100, 50, 10, b, 0)
    for rs in (-1, 1.5, True, None):
        with pytest.raises(ValueError, match="random_state"):
            mo.check_config(100, 50, 10, 10, rs)
    # 100 000 bootstraps of window 256 are 1.3e10 kernel values: inside the budget; the budget is what it says
    mo.check_config(100000, 50, 256, 100000, 0)
    monkeypatch.setattr(mo, "KERNEL_BUDGET", 10**6)
    with pytest.raises(ValueError, match="budget"):
        mo.check_config(1000, 50, 100, 1000, 0)
    monkeypatch.undo()
    mo.check_push(1, 30000, 10)
    with pytest.raises(ValueError, match="at least one row"):
        mo.check_push(0, 30000, 10)
    with pytest.raises(ValueError, match="budget"):
        mo.check_push(3_000_000, 30000, 10)


def test_draws_are_numpys():
    from databricks_kubernetes_mlops_poc_b200 import mmd_online as mo

    etw = mo.draw_bootstraps(np.random.default_rng(5), 50, 4, 3)
    rng = np.random.default_rng(5)
    assert etw.dtype == np.int32 and etw.shape == (3, 7)
    for b in range(3):
        assert np.array_equal(etw[b], rng.permutation(50)[-7:])


def test_exhaustion_and_split_limit():
    from databricks_kubernetes_mlops_poc_b200 import mmd_online as mo

    # equal statistics at window position 0: the quantile is that value and no bootstrap lies below it
    with pytest.raises(ValueError, match="window position 1.*n_bootstraps"):
        mo.thresholds(np.ones((10, 3)), 100.0)
    thr = mo.thresholds(np.random.default_rng(0).random((1000, 3)), 100.0)
    assert thr.shape == (3,) and abs(thr[0] - np.quantile(np.random.default_rng(0).random((1000, 3))[:, 0], 0.99)) == 0
    calls = []
    with pytest.raises(ValueError, match="100 splits"):
        mo.split(np.random.default_rng(0), 30, 3, np.array([0.0, 0.0, 0.0]), lambda y: calls.append(y) or 1.0)
    assert len(calls) == mo.SPLIT_ATTEMPTS and all(len(y) == 5 for y in calls)
    initial = iter([0.9, 0.7, 0.1])
    perm, attempts = mo.split(np.random.default_rng(0), 30, 3, np.array([0.5]), lambda y: next(initial))
    assert attempts == 3 and sorted(perm) == list(range(30))


def test_result():
    from databricks_kubernetes_mlops_poc_b200 import mmd_online as mo

    out = mo.result(np.array([0.1, 0.5, 0.2, 0.9]), 2, np.array([0.3, 0.4, 0.6]), 20.0, 3)
    assert out["time"].tolist() == [2, 3, 4, 5]
    assert out["threshold"].tolist() == [0.6, 0.6, 0.6, 0.6]
    assert out["is_drift"].tolist() == [0, 0, 0, 1] and out["first_drift"] == 5
    out = mo.result(np.array([0.35, 0.35]), 1, np.array([0.3, 0.4, 0.6]), 20.0, 3)
    assert out["threshold"].tolist() == [0.4, 0.6] and out["is_drift"].tolist() == [0, 0] and out["first_drift"] is None


class StubModel:
    def __init__(self, configured=True):
        self.online_drift_configured = configured
        self.mmd_reference_rows = 1000
        self.calls = []
        self.resets = 0
        self.time = 0

    def online_drift_state(self):
        return {"thresholds": np.array([0.1, 0.2]), "sub_reference_rows": 997, "split_attempts": 1, "ert": 50.0, "window_size": 2,
                "n_bootstraps": 10, "random_state": 0, "time": self.time}

    def online_drift(self, df):
        from databricks_kubernetes_mlops_poc_b200 import mmd_online as mo

        self.calls.append(df)
        out = mo.result(np.linspace(0.0, 0.3, len(df)), self.time + 1, np.array([0.1, 0.2]), 50.0, 2)
        self.time += len(df)
        return out

    def reset_online_drift(self):
        self.resets += 1
        self.time = 0


def test_routes_contract_and_validation():
    from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES
    from databricks_kubernetes_mlops_poc_b200.server import create_app

    stub = StubModel()
    body = [{"age": 30.0}, {"sex": "female"}, {}]
    with TestClient(create_app(model=stub), raise_server_exceptions=False) as c:
        r = c.post("/drift/online", json=body)
        assert r.status_code == 200, r.text
        j = r.json()
        assert set(j) == {"time", "test_stat", "threshold", "is_drift", "first_drift", "ert", "window_size"}
        assert j["time"] == [1, 2, 3] and j["is_drift"] == [0, 0, 1] and j["first_drift"] == 3 and j["threshold"] == [0.2, 0.2, 0.2]
        df = stub.calls[-1]
        assert list(df.columns) == ALL_FEATURES and df.loc[0, "age"] == 30.0
        g = c.get("/drift/online")
        assert g.status_code == 200 and g.json()["time"] == 3 and g.json()["thresholds"] == [0.1, 0.2]
        r = c.post("/drift/online/reset")
        assert r.status_code == 200 and r.json()["time"] == 0 and stub.resets == 1
        n_calls = len(stub.calls)
        assert c.post("/drift/online", json=[]).status_code == 422
        # 1 000 rows against a sub-reference of 1e8 rows are 1e11 kernel values, above the 2^36 budget
        stub.mmd_reference_rows = 10**8
        r = c.post("/drift/online", json=[{}] * 1000)
        assert r.status_code == 422 and "budget" in r.json()["detail"]
        assert len(stub.calls) == n_calls
    with TestClient(create_app(model=StubModel(configured=False)), raise_server_exceptions=False) as c:
        assert c.post("/drift/online", json=body).status_code == 501
        assert c.post("/drift/online/reset").status_code == 501
        assert c.get("/drift/online").status_code == 501
