"""Trust scores (K11) on the GPU: b2f_knn's distances bit-identical to the emulator (tests/knn_walk.py) and its indices equal
to it on the training split, adversarial rows, reference rows as queries and the schema-zoo schemas; the k bounds and every
error code; both row formats, determinism and pieces; the filter and scores end to end against the KDTree oracle
(tests/trust_oracle.py); and the B200Model, save/load and ``POST /explain/trust`` layers."""

import threading

import numpy as np
import pandas as pd
import pytest

import knn_walk
import schema_zoo as zoo
import trust_oracle as ot

pytestmark = pytest.mark.gpu

REL = 1e-12


def _split(curated):
    from oracle import reference_pipeline as rp

    train, test = rp.reference_split(curated)
    return train.reset_index(drop=True), test.reset_index(drop=True)


class _Setup:
    """One forest's engine and encoder, with a reference attached and the emulator's embedding of it."""

    def __init__(self, pipe):
        from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
        from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine
        from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline, parse_header

        self.flat = flatten_pipeline(pipe)
        self.eng = ForestEngine(self.flat, 0)
        self.enc = RowEncoder(self.flat)
        self.n_cat, self.n_num = len(self.flat.cat_features), len(self.flat.num_features)
        self.impute = parse_header(self.flat.blob)["impute"][self.n_cat:self.n_cat + self.n_num]

    def attach(self, ref: pd.DataFrame, cls):
        self.rows_ref = self.enc.encode_frame(ref[self.flat.all_features])
        self.cls = np.asarray(cls, dtype=np.int32)
        self.mean, self.scale, self.embed = knn_walk.embedding(self.rows_ref, self.n_cat, self.n_num, self.impute)
        self.zr, self.cr = self.embed(self.rows_ref)
        self.eng.attach_knn_reference(self.rows_ref, self.cls, self.mean, self.scale)

    def check(self, batch: pd.DataFrame, k: int):
        """Device neighbours against the emulator's, bit for bit; both row formats and a second call give the same bytes."""
        rows = self.enc.encode_frame(batch[self.flat.all_features])
        dist, index = self.eng.knn(rows, k)
        zq, cq = self.embed(rows)
        with np.errstate(over="ignore", invalid="ignore"):
            want_d, want_i = knn_walk.neighbours(zq, cq, self.zr, self.cr, self.cls, k)
        assert dist.tobytes() == want_d.tobytes(), np.nanmax(np.abs(dist - want_d))
        assert np.array_equal(index, want_i)
        if self.enc.packed_ok:
            d2, i2 = self.eng.knn(self.enc.pack_rows(rows), k)
            assert d2.tobytes() == dist.tobytes() and i2.tobytes() == index.tobytes()
        d3, i3 = self.eng.knn(rows, k)
        assert d3.tobytes() == dist.tobytes() and i3.tobytes() == index.tobytes()
        return dist, index

    def close(self):
        self.eng.close()


@pytest.fixture(scope="module")
def train_setup(rf100d6, curated):
    from oracle import reference_pipeline as rp

    train, _ = _split(curated)
    s = _Setup(rf100d6)
    s.attach(train, train[rp.TARGET].to_numpy())
    yield s
    s.close()


@pytest.mark.parametrize("m", [1, 31, 1000, 6000])
def test_neighbours_equal_the_emulator(train_setup, curated, m):
    _, test = _split(curated)
    train_setup.check(test.iloc[:m], 2)


@pytest.mark.parametrize("k", [1, 64])
@pytest.mark.parametrize("m", [1, 31, 1000])
def test_k_bounds_of_the_search(train_setup, curated, m, k):
    _, test = _split(curated)
    train_setup.check(test.iloc[100:100 + m], k)


def test_adversarial_rows(train_setup, adversarial):
    train_setup.check(adversarial, 2)
    train_setup.check(adversarial.iloc[:40], 64)


def test_reference_rows_as_queries(train_setup, curated):
    from oracle import reference_pipeline as rp

    train, _ = _split(curated)
    dist, index = train_setup.check(train.iloc[:700], 3)
    y = train[rp.TARGET].to_numpy()[:700]
    rows = np.arange(700)
    assert (dist[rows, y, 0] == 0.0).all()
    assert (index[rows, y, 0] <= rows).all()  # itself, or an equal row before it


@pytest.mark.parametrize("name", ["tiny", "over16", "packed_wide"])
def test_schema_zoo_with_edge_rows(name):
    spec, pipe = zoo.fitted(name)
    s = _Setup(pipe)
    try:
        ref = zoo.make_frame(spec, 400, seed=21, target=False)
        ref[zoo.num_names(spec)[0]] = 4.25  # a constant reference column: scale 1
        cls = (np.arange(len(ref)) % 3 == 0).astype(np.int32)
        s.attach(ref, cls)
        edges = zoo.edge_rows(spec, pipe, n=150, seed=9)
        s.check(edges, 2)
        s.check(edges.iloc[:9], 64)
        s.check(ref.iloc[:50], 1)
    finally:
        s.close()


def test_pieces_equal_one_call(train_setup, curated):
    from oracle import reference_pipeline as rp

    rng = np.random.default_rng(5)
    big = curated[rp.FEATURES].iloc[rng.integers(0, len(curated), 70000)].reset_index(drop=True)
    rows = train_setup.enc.encode_frame(big)
    dist, index = train_setup.eng.knn(rows, 4)
    d1, i1 = train_setup.eng.knn(rows[:65536], 4)
    d2, i2 = train_setup.eng.knn(rows[65536:], 4)
    assert dist.tobytes() == np.concatenate([d1, d2]).tobytes() and index.tobytes() == np.concatenate([i1, i2]).tobytes()
    some = rng.integers(0, 70000, 300)
    d3, i3 = train_setup.eng.knn(rows[some], 4)
    assert d3.tobytes() == dist[some].tobytes() and i3.tobytes() == index[some].tobytes()


def test_c_abi_errors(rf100d6, curated):
    from databricks_kubernetes_mlops_poc_b200._cabi import B2FError

    s = _Setup(rf100d6)
    try:
        ref = curated.iloc[:50]
        cls = np.array([0] * 30 + [1] * 20, dtype=np.int32)
        rows = s.enc.encode_frame(curated[s.flat.all_features].iloc[100:110])
        with pytest.raises(B2FError, match=r"rc=-6\)"):  # no reference
            s.eng.knn(rows, 2)
        rows_ref = s.enc.encode_frame(ref[s.flat.all_features])
        mean, scale = np.zeros(s.n_num), np.ones(s.n_num)
        for r, c, m2, s2 in ((rows_ref[:1], cls[:1], mean, scale), (rows_ref, np.where(cls == 1, 2, 0), mean, scale),
                             (rows_ref, np.zeros(50), mean, scale), (rows_ref, cls, np.full(s.n_num, np.nan), scale),
                             (rows_ref, cls, mean, np.zeros(s.n_num)), (rows_ref, cls, mean, -scale)):
            with pytest.raises(B2FError, match=r"rc=-1\)"):
                s.eng.attach_knn_reference(r, c, m2, s2)
        if s.eng.rank_words:
            with pytest.raises(B2FError, match=r"rc=-1\).*ranked"):
                s.eng.attach_knn_reference(s.enc.rank_rows(rows_ref), cls, mean, scale)
        s.attach(ref, cls)
        for k in (0, 21, 65):  # k above the 20 rows of class 1, above B2F_KNN_MAX_K
            with pytest.raises(B2FError, match=r"rc=-1\)"):
                s.eng.knn(rows, k)
        s.check(curated.iloc[100:110], 20)
        with pytest.raises(B2FError, match=r"rc=-1\)"):  # no rows
            s.eng.knn(rows[:0], 2)
        if s.eng.rank_words:
            with pytest.raises(B2FError, match=r"rc=-1\).*ranked"):
                s.eng.knn(s.enc.rank_rows(rows), 2)
        s.eng.knn(rows, 2)  # the reference survived the refusals
        with pytest.raises(B2FError):  # a failed attach leaves no reference
            s.eng.attach_knn_reference(rows_ref[:1], cls[:1], mean, scale)
        with pytest.raises(B2FError, match=r"rc=-6\)"):
            s.eng.knn(rows, 2)
    finally:
        s.close()


_FITS = {}  # the oracle's filtered fits by reference vectors: they depend on the rows, labels and the pipeline's preprocessing


def _filter_oracle(pipe, ref):
    from oracle import reference_pipeline as rp

    xr, mean, scale = ot.dense(pipe, ref[rp.FEATURES])
    key = hash(xr.tobytes())
    if key not in _FITS:
        y = ref[rp.TARGET].to_numpy()
        _FITS[key] = {t: ot.TrustScore(k_filter=10, alpha=0.05, filter_type="distance_knn", dist_filter_type=t).fit(xr, y)
                      for t in ("point", "mean")}
    return mean, scale, _FITS[key]


@pytest.mark.parametrize("pipe_name", ["rf100d6", "rf500d8", "gbdt_small"])
def test_filter_and_scores_against_the_oracle(request, curated, pipe_name):
    from databricks_kubernetes_mlops_poc_b200.model import B200Model
    from oracle import reference_pipeline as rp

    pipe = request.getfixturevalue(pipe_name)
    train, test = _split(curated)
    ref = train.iloc[:8000]
    mean, scale, fits = _filter_oracle(pipe, ref)
    queries = test.iloc[:1000]
    xq, _, _ = ot.dense(pipe, queries[rp.FEATURES], mean, scale)
    pred = pipe.predict(queries[rp.FEATURES]).astype(np.int64)
    model = B200Model.from_pipeline(pipe, devices=[0])
    try:
        for t, ts in fits.items():
            kept = model.attach_trust_reference(ref, filter_type="distance_knn", alpha=0.05, dist_filter_type=t)
            assert kept == [len(ts.kept[0]), len(ts.kept[1])]
            assert np.array_equal(np.sort(model._trust_positions), np.sort(np.concatenate(ts.kept)))
            for dist_type in ("point", "mean"):
                out = model.trust_score(queries, k=2, dist_type=dist_type)
                want, _ = ts.score(xq, pred, k=2, dist_type=dist_type)
                assert np.array_equal(out["labels"], pred)
                assert np.abs(out["trust_score"] - want).max() <= REL * np.abs(want).max()
                for c in (0, 1):
                    assert np.isin(out["neighbours"][c]["index"], ts.kept[c]).all()
    finally:
        model.close()


def test_model_save_load_http_and_inflight_predict(rf100d6, curated, tmp_path):
    from fastapi.testclient import TestClient

    from databricks_kubernetes_mlops_poc_b200.model import B200Model, load_model, save_model_dir
    from databricks_kubernetes_mlops_poc_b200.server import create_app
    from oracle import reference_pipeline as rp

    train, test = _split(curated)
    ref = train.iloc[:3000].copy()
    ref.loc[3, "sex"] = None
    ref.loc[4, "education"] = np.nan
    ref.loc[5, "age"] = np.nan
    batch = test[rp.FEATURES].iloc[:120].copy()
    batch.loc[batch.index[0], "age"] = np.nan  # the classifier alone is scored: NaN numerics are accepted
    opts = {"k_filter": 5, "alpha": 0.1, "filter_type": "distance_knn", "dist_filter_type": "mean"}
    model = B200Model.from_pipeline(rf100d6, devices=[0], trust_reference=ref, trust_options=opts)
    try:
        out = model.trust_score(batch, k=3)
        assert set(out) == {"trust_score", "closest_not_pred", "predictions", "labels", "distance_to_pred", "distance_to_other", "k",
                            "dist_type", "reference_rows", "neighbours"}
        assert out["k"] == 3 and out["dist_type"] == "point" and sum(out["reference_rows"]) < 3000
        assert np.array_equal(out["predictions"], model.predict_proba1(batch))
        with pytest.raises(ValueError):
            model.trust_score(batch, k=65)
        with pytest.raises(ValueError):
            model.trust_score(batch, dist_type="max")

        errors = []

        def scorer():
            try:
                want_p = model.predict_proba1(batch.iloc[1:])
                for _ in range(20):
                    assert np.array_equal(model.predict_proba1(batch.iloc[1:]), want_p)
            except Exception as e:  # noqa: BLE001
                errors.append(e)

        th = threading.Thread(target=scorer)
        th.start()
        for _ in range(5):
            again = model.trust_score(batch, k=3)
            assert again["trust_score"].tobytes() == out["trust_score"].tobytes()
        th.join()
        assert not errors, errors

        with TestClient(create_app(model=model), raise_server_exceptions=False) as c:
            body = batch.iloc[1:51].to_dict(orient="records")  # a request's numerics are numbers: row 0's NaN age stays out
            r = c.post("/explain/trust?k=3&neighbours=true", json=body)
            assert r.status_code == 200, r.text
            j = r.json()
            want = model.trust_score(pd.DataFrame(body), k=3)
            assert j["trust_score"] == want["trust_score"].tolist() and j["labels"] == want["labels"].tolist()
            assert j["neighbours"][1]["index"] == want["neighbours"][1]["index"].tolist()
            assert "neighbours" not in c.post("/explain/trust", json=body).json()
            assert c.post("/explain/trust?k=0", json=body).status_code == 422

        save_model_dir(str(tmp_path / "m"), model.flat, trust_reference=ref, trust_options=opts)
    finally:
        model.close()
    loaded = load_model(str(tmp_path / "m"), devices=[0])
    try:
        back = loaded.trust_score(batch, k=3)
        assert back["reference_rows"] == out["reference_rows"]
        assert back["trust_score"].tobytes() == out["trust_score"].tobytes()
    finally:
        loaded.close()
    bare = B200Model.from_pipeline(rf100d6, devices=[0])
    try:
        with pytest.raises(RuntimeError):
            bare.trust_score(batch)
        with TestClient(create_app(model=bare), raise_server_exceptions=False) as c:
            assert c.post("/explain/trust", json=batch.iloc[1:6].to_dict(orient="records")).status_code == 501
    finally:
        bare.close()
