"""The online MMD drift detector (K13) on the GPU: bootstrap statistics, thresholds, split and per-step statistics against
the emulator (tests/mmd_online_walk.py) and the alibi restatement (tests/mmd_online_oracle.py) on curated references and
the schema-zoo schemas with edge rows; byte identity across calls, row formats, cuts of the stream and pieces of a push;
reset; re-attaching the reference; a larger model beside it; the C-ABI errors; the calibration case; and the B200Model,
save/load, ``B200_ONLINE_DRIFT=off`` and ``/drift/online`` layers."""

import numpy as np
import pandas as pd
import pytest

import mmd_online_oracle
import mmd_online_walk
import mmd_walk
import schema_zoo as zoo

pytestmark = pytest.mark.gpu

TOL = 1e-12


def _features(curated):
    from oracle import reference_pipeline as rp

    return curated[rp.FEATURES]


def _emulator(model, ref: pd.DataFrame):
    """The emulator of a model's attached MMD reference, and a function embedding a frame in its space."""
    n_cat, n_num = len(model.categorical_features), len(model.numeric_features)
    from databricks_kubernetes_mlops_poc_b200.flatten import parse_header

    impute = parse_header(model.flat.blob)["impute"][n_cat:n_cat + n_num]
    rows = model.encoder.encode_frame(ref[model.all_features])
    mean, scale = model._embedding_constants(rows)

    def embed(df):
        return mmd_walk.embed(model.encoder.encode_frame(df[model.all_features]), n_cat, n_num, impute, mean, scale)

    z, c = embed(ref)
    return mmd_online_walk.Emulator(z, c, model.mmd_sigma), embed


def _tol(emu, W):
    """TOL, times the K_RR term's size where it exceeds 1 (tests/test_mmd_online_cpu.py)."""
    rw = emu.n - (2 * W - 1)
    return TOL * max(1.0, emu.total / (rw * (rw - 1)))


@pytest.fixture(scope="module")
def ref_model(rf100d6, curated):
    from databricks_kubernetes_mlops_poc_b200.model import B200Model

    model = B200Model.from_pipeline(rf100d6, devices=[0], mmd_reference=_features(curated).iloc[1000:1700])
    yield model
    model.close()


@pytest.mark.parametrize("W,n_boot,ert", [(2, 200, 50.0), (10, 200, 50.0), (100, 300, 1000.0), (256, 600, 1000.0)])
def test_device_against_emulator_and_oracle(ref_model, curated, W, n_boot, ert):
    ref = _features(curated).iloc[1000:1700]
    emu, embed = _emulator(ref_model, ref)
    cfg = ref_model.configure_online_drift(ert=ert, window_size=W, n_bootstraps=n_boot, random_state=W)
    thr, perm, attempts, stats = emu.configure(ert, W, n_boot, W)
    tol = _tol(emu, W)
    rng = np.random.default_rng(W)
    etw = np.asarray([rng.permutation(700)[-(2 * W - 1):] for _ in range(n_boot)], dtype=np.int32)
    got, k_rr = ref_model.engine.mmd_online_bootstrap(etw, W)
    assert np.abs(got - stats).max() <= tol
    again, k_rr2 = ref_model.engine.mmd_online_bootstrap(etw, W)
    assert again.tobytes() == got.tobytes() and k_rr2.tobytes() == k_rr.tobytes()
    assert np.abs(cfg["thresholds"] - thr).max() <= tol
    assert cfg["split_attempts"] == attempts and cfg["sub_reference_rows"] == 700 - (2 * W - 1)
    stream = _features(curated).iloc[20000:20000 + 3 * W + 40]
    zs, cs = embed(stream)
    out = [ref_model.online_drift(stream.iloc[:1]), ref_model.online_drift(stream.iloc[1:W + 3]), ref_model.online_drift(stream.iloc[W + 3:])]
    stat = np.concatenate([o["test_stat"] for o in out])
    assert np.concatenate([o["time"] for o in out]).tolist() == list(range(1, len(stream) + 1))
    want = emu.push(zs, cs)
    assert np.abs(stat - want).max() <= tol
    if W <= 100:
        oracle = mmd_online_oracle.OnlineOracle(emu.z, emu.c, ref_model.mmd_sigma, ert, W, n_boot, W)
        assert np.abs(cfg["thresholds"] - oracle.thresholds).max() <= tol and np.array_equal(oracle.perm, perm)
        o = [oracle.predict(zs[i], cs[i]) for i in range(len(zs))]
        assert np.abs(stat - np.array([p["test_stat"] for p in o])).max() <= tol
        assert np.concatenate([x["is_drift"] for x in out]).tolist() == [p["is_drift"] for p in o]
    ref_model.reset_online_drift()
    assert ref_model.online_drift(stream)["test_stat"].tobytes() == stat.tobytes()


@pytest.mark.parametrize("name", ["tiny", "packed_wide", "over16"])
def test_schema_zoo_with_edge_rows(name):
    from databricks_kubernetes_mlops_poc_b200.model import B200Model

    spec, pipe = zoo.fitted(name)
    ref = zoo.make_frame(spec, 300, seed=3, target=False)
    edges = zoo.edge_rows(spec, pipe, n=120, seed=5)
    nums = zoo.num_names(spec)
    # +-3e38 squares past float64's range only through the z-scores' scale; keep them out, as the MMD tests do
    edges = edges[~(np.abs(edges[nums].to_numpy(dtype=np.float64)) > 1e30).any(axis=1)].reset_index(drop=True)
    model = B200Model.from_pipeline(pipe, devices=[0], mmd_reference=ref)
    try:
        emu, embed = _emulator(model, ref)
        cfg = model.configure_online_drift(ert=50, window_size=10, n_bootstraps=100, random_state=1)
        thr, _, attempts, _ = emu.configure(50.0, 10, 100, 1)
        tol = _tol(emu, 10)
        assert np.abs(cfg["thresholds"] - thr).max() <= tol and cfg["split_attempts"] == attempts
        got = model.online_drift(edges)["test_stat"]
        zs, cs = embed(edges)
        assert np.abs(got - emu.push(zs, cs)).max() <= tol
        if model.encoder.packed_ok:
            model.reset_online_drift()
            rows = model.encoder.encode_frame(edges[model.all_features])
            stat, t0 = model.engine.mmd_online_push(model.encoder.pack_rows(rows))
            assert t0 == 1 and stat.tobytes() == got.tobytes()
    finally:
        model.close()


def test_byte_identity_across_cuts_formats_and_pieces(rf100d6, curated):
    from databricks_kubernetes_mlops_poc_b200.model import B200Model

    feats = _features(curated)
    model = B200Model.from_pipeline(rf100d6, devices=[0], mmd_reference=feats.iloc[:2000])
    try:
        model.configure_online_drift(ert=1000, window_size=256, n_bootstraps=300, random_state=0)
        eng = model.engine
        rows = model.encoder.encode_frame(feats.iloc[2000:][model.all_features])
        small = rows[:1000]
        whole, t0 = eng.mmd_online_push(small)
        assert t0 == 1
        eng.mmd_online_reset()
        cut = [eng.mmd_online_push(small[a:b]) for a, b in ((0, 1), (1, 8), (8, 264), (264, 1000))]
        assert [t for _, t in cut] == [1, 2, 9, 265]
        assert np.concatenate([s for s, _ in cut]).tobytes() == whole.tobytes()
        eng.mmd_online_reset()
        assert eng.mmd_online_push(model.encoder.pack_rows(small))[0].tobytes() == whole.tobytes()
        # 250 000 rows at W = 256 take three pieces of the 256 MiB scratch; cut differently, the same bytes
        big = np.concatenate([rows] * 10)[:250000]
        eng.mmd_online_reset()
        one, _ = eng.mmd_online_push(big)
        assert one[:1000].tobytes() == whole.tobytes()
        eng.mmd_online_reset()
        two = np.concatenate([eng.mmd_online_push(big[:123457])[0], eng.mmd_online_push(big[123457:])[0]])
        assert two.tobytes() == one.tobytes()

        # a larger model beside it: its limits set after this model's, then this model again, the same bits
        spec, pipe = zoo.fitted("over16")
        other = B200Model.from_pipeline(pipe, devices=[0], mmd_reference=zoo.make_frame(spec, 600, seed=2, target=False))
        try:
            other.configure_online_drift(ert=100, window_size=64, n_bootstraps=200)
            other.online_drift(zoo.make_frame(spec, 500, seed=9, target=False))
            eng.mmd_online_reset()
            assert eng.mmd_online_push(small)[0].tobytes() == whole.tobytes()
        finally:
            other.close()
        eng.mmd_online_reset()
        assert eng.mmd_online_push(small)[0].tobytes() == whole.tobytes()
    finally:
        model.close()


def _rc(fn):
    from databricks_kubernetes_mlops_poc_b200._cabi import B2FError

    with pytest.raises(B2FError) as e:
        fn()
    return int(str(e.value).split("rc=")[1].split(")")[0]), str(e.value)


def test_c_abi_errors(rf100d6, curated):
    from databricks_kubernetes_mlops_poc_b200 import mmd
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline, parse_header

    flat = flatten_pipeline(rf100d6)
    eng = ForestEngine(flat, 0)
    enc = RowEncoder(flat)
    try:
        rows = enc.encode_frame(_features(curated).iloc[:40][flat.all_features])
        etw = np.arange(19, dtype=np.int32)[None]
        assert _rc(lambda: eng.mmd_online_bootstrap(etw, 10))[0] == -6
        assert _rc(lambda: eng.mmd_online_push(rows))[0] == -6
        assert _rc(lambda: eng.mmd_online_reset())[0] == -6
        n_cat, n_num = len(flat.cat_features), len(flat.num_features)
        impute = parse_header(flat.blob)["impute"][n_cat:n_cat + n_num]
        mean, scale = mmd.standardization(mmd.numerics(rows, n_cat, n_num, impute))
        eng.attach_mmd_reference(rows, mean, scale)
        assert _rc(lambda: eng.mmd_online_push(rows))[0] == -6
        assert _rc(lambda: eng.mmd_online_reset())[0] == -6
        assert _rc(lambda: eng.mmd_online_bootstrap(np.arange(1, dtype=np.int32)[None], 1))[0] == -1
        assert _rc(lambda: eng.mmd_online_bootstrap(np.zeros((1, 513), dtype=np.int32), 257))[0] == -1
        rc, msg = _rc(lambda: eng.mmd_online_bootstrap(np.arange(39, dtype=np.int32)[None], 20))
        assert rc == -1 and "at least 2W + 1 = 41 rows" in msg
        assert _rc(lambda: eng.mmd_online_bootstrap(np.zeros((0, 19), dtype=np.int32), 10))[0] == -1
        bad = np.arange(19, dtype=np.int32)[None].copy()
        bad[0, 3] = 40
        assert _rc(lambda: eng.mmd_online_bootstrap(bad, 10))[0] == -1
        bad[0, 3] = 7
        assert "twice" in _rc(lambda: eng.mmd_online_bootstrap(bad, 10))[1]
        eng.mmd_online_bootstrap(np.stack([np.arange(19), np.arange(19)]).astype(np.int32), 10)  # repeats across sequences are fine
        eng.mmd_online_configure(np.arange(40), 10)
        stat, t0 = eng.mmd_online_push(rows)
        assert t0 == 1 and np.isfinite(stat).all()
        perm = np.arange(40)
        perm[5] = 6
        assert _rc(lambda: eng.mmd_online_configure(perm, 10))[0] == -1
        assert _rc(lambda: eng.mmd_online_push(rows))[0] == -6  # a failed configure leaves none
        eng.mmd_online_configure(np.arange(40), 10)
        eng.attach_mmd_reference(rows, mean, scale)
        assert _rc(lambda: eng.mmd_online_push(rows))[0] == -6  # re-attaching drops the detector
    finally:
        eng.close()


def test_calibration(rf100d6, curated):
    """ERT = 100, W = 20: the mean first detection of no-drift streams lies within [ERT / 4, 4 ERT], and a stream of
    applicants two or more months late on their last repayment is detected within 5W rows."""
    from databricks_kubernetes_mlops_poc_b200.model import B200Model

    feats = _features(curated)
    order = np.random.default_rng(7).permutation(len(feats))
    ref, rest = feats.iloc[order[:4000]], feats.iloc[order[4000:]]
    model = B200Model.from_pipeline(rf100d6, devices=[0], mmd_reference=ref)
    try:
        model.configure_online_drift(ert=100, window_size=20, n_bootstraps=5000, random_state=0)
        firsts = []
        for k in range(20):
            model.reset_online_drift()
            stream = rest.iloc[np.random.default_rng(100 + k).permutation(len(rest))[:2000]]
            f = model.online_drift(stream)["first_drift"]
            firsts.append(2000 if f is None else f)
        assert 25 <= np.mean(firsts) <= 400, firsts
        late = rest[~rest["repayment_status_1"].isin(["no_delay", "duly_paid", "delay_1_month"])]
        model.reset_online_drift()
        out = model.online_drift(late.iloc[np.random.default_rng(1).permutation(len(late))[:500]])
        assert out["first_drift"] is not None and out["first_drift"] <= 100, out["first_drift"]
    finally:
        model.close()


def test_model_save_load_off_and_routes(rf100d6, curated, tmp_path, monkeypatch):
    from fastapi.testclient import TestClient

    from databricks_kubernetes_mlops_poc_b200.model import B200Model, load_model, save_model_dir
    from databricks_kubernetes_mlops_poc_b200.server import create_app

    feats = _features(curated)
    ref = feats.iloc[:800].copy()
    batch = feats.iloc[9000:9100]
    bare = B200Model.from_pipeline(rf100d6, devices=[0])
    try:
        with pytest.raises(RuntimeError, match="MMD reference"):
            bare.configure_online_drift(ert=50, window_size=10)
        bare.attach_mmd_reference(ref)
        with pytest.raises(RuntimeError, match="not configured"):
            bare.online_drift(batch)
        assert bare.online_drift_state() is None
        with pytest.raises(ValueError, match="window_size"):
            bare.configure_online_drift(ert=50, window_size=1)
    finally:
        bare.close()
    online = dict(ert=50, window_size=10, n_bootstraps=200, random_state=4)
    model = B200Model.from_pipeline(rf100d6, devices=[0], mmd_reference=ref, online_drift=online)
    try:
        st = model.online_drift_state()
        assert st["time"] == 0 and st["ert"] == 50.0 and st["window_size"] == 10 and st["n_bootstraps"] == 200
        first = model.online_drift(batch)
        assert set(first) == {"time", "test_stat", "threshold", "is_drift", "first_drift", "ert", "window_size"}
        assert model.online_drift_state()["time"] == 100
        with pytest.raises(ValueError):
            model.online_drift(batch.iloc[:0])
        with TestClient(create_app(model=model), raise_server_exceptions=False) as c:
            assert c.post("/drift/online/reset").json()["time"] == 0
            body = batch.replace({np.nan: None}).to_dict(orient="records")
            r = c.post("/drift/online", json=body)
            assert r.status_code == 200, r.text
            assert r.json()["test_stat"] == first["test_stat"].tolist() and r.json()["time"] == list(range(1, 101))
            g = c.get("/drift/online").json()
            assert g["time"] == 100 and g["thresholds"] == st["thresholds"].tolist()
            assert c.post("/drift/online", json=[]).status_code == 422
        save_model_dir(str(tmp_path / "m"), model.flat, mmd_reference=ref, online_drift=online)
        with pytest.raises(ValueError, match="mmd_reference"):
            save_model_dir(str(tmp_path / "x"), model.flat, online_drift=online)
        model.attach_mmd_reference(ref)
        assert not model.online_drift_configured
        with pytest.raises(RuntimeError, match="not configured"):
            model.online_drift(batch)
    finally:
        model.close()
    loaded = load_model(str(tmp_path / "m"), devices=[0])
    try:
        assert loaded.online_drift_state()["thresholds"].tobytes() == st["thresholds"].tobytes()
        assert loaded.online_drift(batch)["test_stat"].tobytes() == first["test_stat"].tobytes()
    finally:
        loaded.close()
    monkeypatch.setenv("B200_ONLINE_DRIFT", "off")
    off = load_model(str(tmp_path / "m"), devices=[0])
    try:
        assert off.mmd_reference_attached and not off.online_drift_configured
        with TestClient(create_app(model=off), raise_server_exceptions=False) as c:
            assert c.post("/drift/online", json=[{}]).status_code == 501
            assert c.get("/drift/online").status_code == 501
    finally:
        off.close()
