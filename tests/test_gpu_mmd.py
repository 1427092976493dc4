"""The MMD drift test (K9) on the GPU: sigma against the emulator (tests/mmd_walk.py) and by rank on the full curated table,
the observed and permuted statistics against the emulator on the reference forest and the schema-zoo schemas with edge
rows, p-values and ties, determinism across calls and row formats, the C-ABI errors, the calibration case, and the
B200Model, save/load and ``POST /drift/mmd`` layers."""

import threading

import numpy as np
import pandas as pd
import pytest

import mmd_walk
import schema_zoo as zoo

pytestmark = pytest.mark.gpu

TOL = 1e-12


class _Setup:
    """One forest's engine, encoder and the embedding constants of a reference frame."""

    def __init__(self, pipe):
        from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
        from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine
        from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline, parse_header

        self.flat = flatten_pipeline(pipe)
        self.eng = ForestEngine(self.flat, 0)
        self.enc = RowEncoder(self.flat)
        self.n_cat, self.n_num = len(self.flat.cat_features), len(self.flat.num_features)
        self.impute = parse_header(self.flat.blob)["impute"][self.n_cat:self.n_cat + self.n_num]

    def attach(self, ref: pd.DataFrame, sigma=None):
        from databricks_kubernetes_mlops_poc_b200 import mmd

        self.rows_ref = self.enc.encode_frame(ref[self.flat.all_features])
        self.mean, self.scale = mmd.standardization(mmd.numerics(self.rows_ref, self.n_cat, self.n_num, self.impute))
        self.sigma = self.eng.attach_mmd_reference(self.rows_ref, self.mean, self.scale, sigma)
        return self.sigma

    def embed(self, rows):
        return mmd_walk.embed(rows, self.n_cat, self.n_num, self.impute, self.mean, self.scale)

    def check(self, batch: pd.DataFrame, n_perm=20, seed=0):
        """Device statistics against the emulator's; -> (device observed, device permuted, emulator terms)."""
        from databricks_kubernetes_mlops_poc_b200 import mmd

        rows = self.enc.encode_frame(batch[self.flat.all_features])
        sub = mmd.draw_subsets(len(self.rows_ref), len(rows), n_perm, seed)
        obs, perm = self.eng.mmd_statistics(rows, sub)
        (zr, cr), (zb, cb) = self.embed(self.rows_ref), self.embed(rows)
        want, terms = mmd_walk.statistics(zr, cr, zb, cb, sub, self.sigma)
        assert abs(obs - want[0]) <= TOL * terms[0], (obs, want[0])
        assert (np.abs(perm - want[1:]) <= TOL * terms[1:]).all(), np.abs(perm - want[1:]).max()
        # p-value: equal to the emulator's wherever no permuted statistic is within the tolerance of the observed one
        if not np.any(np.abs(want[1:] - want[0]) <= 2 * TOL * terms[1:]):
            assert np.mean(obs <= perm) == np.mean(want[0] <= want[1:])
        if self.enc.packed_ok:
            o2, p2 = self.eng.mmd_statistics(self.enc.pack_rows(rows), sub)
            assert o2 == obs and p2.tobytes() == perm.tobytes()
        o3, p3 = self.eng.mmd_statistics(rows, sub)
        assert o3 == obs and p3.tobytes() == perm.tobytes()
        return obs, perm, terms

    def close(self):
        self.eng.close()


@pytest.fixture(scope="module")
def ref_setup(rf100d6):
    s = _Setup(rf100d6)
    yield s
    s.close()


def _features(curated):
    from oracle import reference_pipeline as rp

    return curated[rp.FEATURES]


@pytest.mark.parametrize("n_ref", [2, 3, 500, 5000])
def test_sigma_equals_the_emulators_median(ref_setup, curated, n_ref):
    ref = _features(curated).iloc[1000:1000 + n_ref]
    sigma = ref_setup.attach(ref)
    z, c = ref_setup.embed(ref_setup.rows_ref)
    want = mmd_walk.sigma(z, c)
    assert abs(sigma - want) <= 1e-13 * want


def _rank_ok(z, c, sigma, k):
    """Some double v with sqrt(0.5 v) == sigma has count(d < v) <= k < count(d <= v)."""
    v = 2.0 * sigma * sigma
    cands = [v]
    for _ in range(3):
        cands = sorted({np.nextafter(x, np.inf) for x in cands} | {np.nextafter(x, -np.inf) for x in cands} | set(cands))
    cands = [x for x in cands if float(np.sqrt(0.5 * x)) == sigma]
    below_lo, near = mmd_walk.rank_counts(z, c, min(cands), max(cands))
    for x in cands:
        below = below_lo + int(np.searchsorted(near, x, side="left"))
        at = below_lo + int(np.searchsorted(near, x, side="right"))
        if below <= k < at:
            return True
    return False


def test_sigma_by_rank_on_the_full_table(ref_setup, curated):
    ref = _features(curated)
    n = len(ref)
    sigma = ref_setup.attach(ref)
    z, c = ref_setup.embed(ref_setup.rows_ref)
    assert _rank_ok(z, c, sigma, (n * (n - 1) // 2 - 1) // 2)


@pytest.mark.parametrize("m", [2, 3, 31, 1000])
def test_statistics_against_the_emulator(ref_setup, curated, m):
    ref_setup.attach(_features(curated).iloc[:500])
    ref_setup.check(_features(curated).iloc[20000:20000 + m])


def test_statistics_with_a_larger_batch_than_reference(ref_setup, curated):
    ref_setup.attach(_features(curated).iloc[:200])
    ref_setup.check(_features(curated).iloc[5000:5300])  # subsets on the reference side
    ref_setup.attach(_features(curated).iloc[:2])
    ref_setup.check(_features(curated).iloc[5000:5040], n_perm=50)


@pytest.mark.parametrize("name", ["tiny", "over16", "packed_wide"])
def test_schema_zoo_with_edge_rows(name):
    spec, pipe = zoo.fitted(name)
    s = _Setup(pipe)
    try:
        ref = zoo.make_frame(spec, 300, seed=21, target=False)
        ref[zoo.num_names(spec)[0]] = 4.25  # a constant reference column: scale 1
        s.attach(ref)
        edges = zoo.edge_rows(spec, pipe, n=150, seed=9)
        nums = zoo.num_names(spec)
        edges = edges[~(np.abs(edges[nums].to_numpy(dtype=np.float64)) > 1e30).any(axis=1)].reset_index(drop=True)
        s.check(edges)
        s.check(edges.iloc[:7], n_perm=30, seed=4)
        s.attach(ref, sigma=1.75)
        assert s.sigma == 1.75
        s.check(edges.iloc[:40])
    finally:
        s.close()


def test_tiny_pool_p_value_is_exact_with_ties(ref_setup, curated):
    from databricks_kubernetes_mlops_poc_b200 import mmd

    ref_setup.attach(_features(curated).iloc[10:13])
    rows = ref_setup.enc.encode_frame(_features(curated).iloc[40:42])
    sub = mmd.draw_subsets(3, 2, 200, 1)
    obs, perm = ref_setup.eng.mmd_statistics(rows, sub)
    is_batch = (sub == np.array([3, 4])).all(axis=1)
    assert is_batch.sum() > 5
    assert (perm[is_batch] == obs).all()  # the same subset through the same code: the same bits
    (zr, cr), (zb, cb) = ref_setup.embed(ref_setup.rows_ref), ref_setup.embed(rows)
    want, terms = mmd_walk.statistics(zr, cr, zb, cb, sub, ref_setup.sigma)
    assert (np.abs(perm - want[1:]) <= TOL * terms[1:]).all()
    # every other split's statistic is away from the observed one, so the count is exact
    others = ~is_batch
    assert (np.abs(want[1:][others] - want[0]) > 10 * TOL * terms[1:][others]).all()
    assert np.mean(obs <= perm) == np.mean(obs <= np.where(is_batch, obs, want[1:]))


def test_c_abi_errors(rf100d6, curated):
    from databricks_kubernetes_mlops_poc_b200 import mmd
    from databricks_kubernetes_mlops_poc_b200._cabi import B2FError

    s = _Setup(rf100d6)
    try:
        ref = _features(curated).iloc[:50]
        rows = s.enc.encode_frame(_features(curated).iloc[100:110])
        with pytest.raises(B2FError, match=r"rc=-6\)"):  # no reference
            s.eng.mmd_statistics(rows, mmd.draw_subsets(50, 10, 3, 0))
        with pytest.raises(B2FError, match=r"rc=-1\)"):  # one reference row
            s.attach(ref.iloc[:1])
        for bad in (0.0, -2.0, float("inf")):
            with pytest.raises(B2FError, match=r"rc=-1\)"):
                s.attach(ref, sigma=bad)
        rows_ref = s.enc.encode_frame(ref)
        mean, scale = np.zeros(s.n_num), np.ones(s.n_num)
        for m2, s2 in ((np.full(s.n_num, np.nan), scale), (mean, np.zeros(s.n_num)), (mean, -scale), (mean, np.full(s.n_num, np.inf))):
            with pytest.raises(B2FError, match=r"rc=-1\)"):
                s.eng.attach_mmd_reference(rows_ref, m2, s2)
        same = pd.concat([ref.iloc[:1]] * 10, ignore_index=True)  # every pair distance 0: no median heuristic
        with pytest.raises(B2FError, match=r"rc=-1\).*sigma"):
            s.attach(same)
        s.attach(same, sigma=1.0)
        if s.eng.rank_words:
            with pytest.raises(B2FError, match=r"rc=-1\).*ranked"):
                s.eng.attach_mmd_reference(s.enc.rank_rows(rows_ref), s.mean, s.scale)
        s.attach(ref)
        sub = mmd.draw_subsets(50, 10, 4, 0)
        for fix in (lambda u: u.__setitem__((1, 0), 60), lambda u: u.__setitem__((1, 0), -1), lambda u: u.__setitem__((2, slice(None)), u[2][::-1].copy()),
                    lambda u: u.__setitem__((3, 1), u[3, 0])):
            u = sub.copy()
            fix(u)
            with pytest.raises(B2FError, match=r"rc=-1\)"):
                s.eng.mmd_statistics(rows, u)
        with pytest.raises(B2FError, match=r"rc=-1\)"):  # one row
            s.eng.mmd_statistics(rows[:1], mmd.draw_subsets(50, 1, 2, 0))
        with pytest.raises(B2FError, match=r"rc=-1\)"):  # no permutations
            s.eng.mmd_statistics(rows, sub[:0])
        if s.eng.rank_words:
            with pytest.raises(B2FError, match=r"rc=-1\).*ranked"):
                s.eng.mmd_statistics(s.enc.rank_rows(rows), sub)
        s.eng.mmd_statistics(rows, sub)  # the reference survived the refusals
        with pytest.raises(B2FError):  # a failed attach leaves no reference
            s.attach(ref.iloc[:1])
        with pytest.raises(B2FError, match=r"rc=-6\)"):
            s.eng.mmd_statistics(rows, sub)
    finally:
        s.close()


def test_calibration_joint_shift_is_flagged(rf100d6, curated):
    from databricks_kubernetes_mlops_poc_b200.model import B200Model

    ref, held, shuffled = mmd_walk.calibration_frames(curated)
    model = B200Model.from_pipeline(rf100d6, devices=[0], mmd_reference=ref)
    try:
        quiet = model.mmd_drift(held)
        moved = model.mmd_drift(shuffled)
        assert quiet["p_val"] > 0.05 and quiet["is_drift"] == 0
        assert moved["p_val"] < 0.05 and moved["is_drift"] == 1 and moved["distance"] > moved["distance_threshold"]
    finally:
        model.close()


def test_model_save_load_http_and_inflight_predict(rf100d6, curated, tmp_path):
    from fastapi.testclient import TestClient

    from databricks_kubernetes_mlops_poc_b200 import mmd
    from databricks_kubernetes_mlops_poc_b200.model import B200Model, load_model, save_model_dir
    from databricks_kubernetes_mlops_poc_b200.server import create_app

    ref = _features(curated).iloc[:800].copy()
    ref.loc[3, "sex"] = None
    ref.loc[4, "education"] = np.nan
    ref.loc[5, "age"] = np.nan
    batch = _features(curated).iloc[9000:9120]
    model = B200Model.from_pipeline(rf100d6, devices=[0], mmd_reference=ref)
    try:
        out = model.mmd_drift(batch, n_permutations=40, p_val=0.1, random_state=3)
        assert set(out) == {"is_drift", "distance", "p_val", "threshold", "distance_threshold", "sigma", "n_permutations", "reference_rows", "rows"}
        assert out["reference_rows"] == 800 and out["rows"] == 120 and out["n_permutations"] == 40 and out["threshold"] == 0.1
        rows = model.encoder.encode_frame(batch)
        obs, perm = model.engine.mmd_statistics(rows, mmd.draw_subsets(800, 120, 40, 3))
        assert out == mmd.result(obs, perm, 0.1, model.mmd_sigma, 800, 120)
        with pytest.raises(ValueError):
            model.mmd_drift(batch.iloc[:1])
        with pytest.raises(ValueError):
            model.mmd_drift(batch, n_permutations=0)

        # calls interleaved with in-flight predict batches
        want_p = model.predict_proba1(batch)
        errors = []

        def scorer():
            try:
                for _ in range(20):
                    assert np.array_equal(model.predict_proba1(batch), want_p)
            except Exception as e:  # noqa: BLE001
                errors.append(e)

        th = threading.Thread(target=scorer)
        th.start()
        for _ in range(5):
            assert model.mmd_drift(batch, n_permutations=40, p_val=0.1, random_state=3) == out
        th.join()
        assert not errors, errors

        with TestClient(create_app(model=model), raise_server_exceptions=False) as c:
            body = batch.iloc[:50].replace({np.nan: None}).to_dict(orient="records")
            r = c.post("/drift/mmd?n_permutations=30&random_state=2", json=body)
            assert r.status_code == 200, r.text
            assert r.json() == model.mmd_drift(pd.DataFrame(body), n_permutations=30, random_state=2)
            assert c.post("/drift/mmd", json=body[:1]).status_code == 422
            assert c.post("/drift/mmd?p_val=0", json=body).status_code == 422

        save_model_dir(str(tmp_path / "m"), model.flat, mmd_reference=ref)
        save_model_dir(str(tmp_path / "s"), model.flat, mmd_reference=ref, mmd_sigma=2.5)
    finally:
        model.close()
    loaded = load_model(str(tmp_path / "m"), devices=[0])
    try:
        assert loaded.mmd_sigma == out["sigma"]
        assert loaded.mmd_drift(batch, n_permutations=40, p_val=0.1, random_state=3) == out
    finally:
        loaded.close()
    loaded = load_model(str(tmp_path / "s"), devices=[0])
    try:
        assert loaded.mmd_sigma == 2.5
    finally:
        loaded.close()
    bare = B200Model.from_pipeline(rf100d6, devices=[0])
    try:
        with pytest.raises(RuntimeError):
            bare.mmd_drift(batch)
        with TestClient(create_app(model=bare), raise_server_exceptions=False) as c:
            assert c.post("/drift/mmd", json=batch.iloc[:5].to_dict(orient="records")).status_code == 501
    finally:
        bare.close()
