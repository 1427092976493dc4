"""One scoring replica per GPU: every call on a GPU's handle holds that replica's lock, and each handle gets exactly one
request pipeline (``Scorer``), whichever of ``predict``, the HTTP batcher and the explanations score on it."""

import threading

import numpy as np
import pytest


def _small_pipeline(curated):
    from oracle import reference_pipeline as rp

    return rp.fit_reference_pipeline(curated.iloc[:3000], dict(n_estimators=5, max_depth=2, random_state=0))


def test_first_gpu_calls_hold_its_replica_lock(curated):
    """Every B200Model method that calls the first GPU's engine holds ``replicas[0].lock`` around that call, so it may run
    beside the HTTP batcher's worker and ``predict`` on the same handle."""
    from databricks_kubernetes_mlops_poc_b200._cabi import COUNTERFACTUAL_DTYPE
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline
    from databricks_kubernetes_mlops_poc_b200.model import B200Model
    from oracle import reference_pipeline as rp

    calls = []

    class Replica:
        lock = threading.RLock()

        def score(self, df, want_outliers=True):
            return np.zeros(len(df)), None

    class Engine:
        def _called(self, name):
            assert m.replicas[0].lock._is_owned(), f"engine.{name} called without replicas[0].lock"
            calls.append(name)

        def explain_rows(self, rows):
            self._called("explain_rows")
            return np.zeros((rows.shape[0], 23)), 0.25

        def explain_interactions_rows(self, rows):
            self._called("explain_interactions_rows")
            return np.zeros((rows.shape[0], 23, 23)), 0.25

        def explain_interventional_rows(self, rows):
            self._called("explain_interventional_rows")
            return np.zeros((rows.shape[0], 23)), 0.25

        def partial_dependence_rows(self, rows, probes, words):
            self._called("partial_dependence_rows")
            return np.zeros((rows.shape[0], sum(p[2] for p in probes)))

        def counterfactual_rows(self, rows, words, cutoff):
            self._called("counterfactual_rows")
            return np.zeros(rows.shape[0]), np.zeros((rows.shape[0], len(words)), dtype=COUNTERFACTUAL_DTYPE)

        def attach_background(self, rows):
            self._called("attach_background")
            return 64 * rows.shape[0]

    flat = flatten_pipeline(_small_pipeline(curated))
    m = object.__new__(B200Model)
    m.flat, m.all_features = flat, flat.all_features
    m.categorical_features, m.numeric_features = list(flat.cat_features), list(flat.num_features)
    m.encoder, m.engine, m.group, m.replicas = RowEncoder(flat), Engine(), None, [Replica()]
    m.explain_blob, m.background_rows = b"table", 0
    df = curated[rp.FEATURES].iloc[:40].reset_index(drop=True)

    m.attach_background(df)
    m.explain(df)
    m.explain_interactions(df)
    m.explain_interventional(df)
    m.partial_dependence(df, ["credit_limit", "education"], kind="both")
    m.counterfactuals(df, ["credit_limit", "education"])
    assert calls == ["attach_background", "explain_rows", "explain_interactions_rows", "explain_interventional_rows",
                     "partial_dependence_rows", "counterfactual_rows", "partial_dependence_rows"]
    assert not m.replicas[0].lock._is_owned()


def _counting_scorers(monkeypatch):
    """Wrap ForestEngine.scorer -> the list of (engine, scorer) it has created."""
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine

    made, scorer = [], ForestEngine.scorer

    def counted(self, encoder, threads=0):
        sc = scorer(self, encoder, threads)
        made.append((self, sc))
        return sc

    monkeypatch.setattr(ForestEngine, "scorer", counted)
    return made


@pytest.mark.gpu
def test_one_scorer_per_gpu(rf100d6, curated, monkeypatch):
    """predict, explain, the replica's score, POST /predict and POST /explain on a one-GPU model share one request
    pipeline: one pool of encoder threads polls per GPU."""
    from fastapi.testclient import TestClient

    from databricks_kubernetes_mlops_poc_b200.model import B200Model
    from databricks_kubernetes_mlops_poc_b200.server import create_app
    from oracle import reference_pipeline as rp

    made = _counting_scorers(monkeypatch)
    m = B200Model.from_pipeline(rf100d6, explain=True, devices=[0])
    df = curated[rp.FEATURES].iloc[:300].reset_index(drop=True)
    try:
        want = m.predict(df)["predictions"]
        assert m.predict(df)["predictions"] == want
        out = m.explain(df)
        proba, flags = m.replicas[0].score(df)
        assert proba.tolist() == want and out["predictions"] == want and flags is None
        body = df.iloc[:20].to_dict(orient="records")
        with TestClient(create_app(model=m)) as c:
            r = c.post("/predict", json=body)
            assert r.status_code == 200 and np.abs(np.asarray(r.json()["predictions"]) - want[:20]).max() <= 1e-12
            r = c.post("/explain", json=body)
            assert r.status_code == 200 and np.abs(np.asarray(r.json()["predictions"]) - want[:20]).max() <= 1e-12
        assert [e for e, _ in made] == [m.engine]
        assert m.replicas[0]._scorer is made[0][1]
    finally:
        m.close()


@pytest.mark.gpu
def test_host_threads_reach_the_server_pool(rf100d6, curated):
    """B200Model(host_threads=...) sizes the pool that the HTTP batcher scores through."""
    from fastapi.testclient import TestClient

    from databricks_kubernetes_mlops_poc_b200.model import B200Model
    from databricks_kubernetes_mlops_poc_b200.server import create_app
    from oracle import reference_pipeline as rp

    m = B200Model.from_pipeline(rf100d6, devices=[0], host_threads=3)
    try:
        with TestClient(create_app(model=m)) as c:
            assert c.post("/predict", json=curated[rp.FEATURES].iloc[:5].to_dict(orient="records")).status_code == 200
        assert m.replicas[0]._scorer.threads == 3
    finally:
        m.close()


@pytest.mark.gpu
def test_one_scorer_per_replica_on_several_gpus(rf100d6, curated, monkeypatch):
    """On several GPUs predict is one group call under every replica's lock, and each replica creates its own scorer once.
    A box with one GPU runs two handles on it."""
    from databricks_kubernetes_mlops_poc_b200.engine import device_count
    from databricks_kubernetes_mlops_poc_b200.model import B200Model
    from oracle import reference_pipeline as rp

    made = _counting_scorers(monkeypatch)
    n = device_count()
    m = B200Model.from_pipeline(rf100d6, devices=list(range(n)) if n >= 2 else [0, 0])
    df = curated[rp.FEATURES].iloc[:300].reset_index(drop=True)
    try:
        want = np.asarray(m.predict(df)["predictions"])
        for r in m.replicas + m.replicas:
            proba, _ = r.score(df)
            assert np.abs(proba - want).max() <= 1e-12
        assert not any(r.lock._is_owned() for r in m.replicas)
        assert [e for e, _ in made] == m.group.engines
        assert [r._scorer for r in m.replicas] == [sc for _, sc in made]
    finally:
        m.close()
