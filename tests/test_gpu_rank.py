"""GPU parity of the rank kernel (k_forest_predict_rank on B2F_ROWS_RANKED rows) and of the columnar request pipeline
(b2f_scorer behind B200Model.predict for large frames), against the library itself.  float64 outputs <= 1e-12, labels exact."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TOL64 = 1e-12
TOL32 = 2e-7


def _engine(pipe, device=0):
    from databricks_kubernetes_mlops_poc_b200 import flatten
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine

    flat = flatten.flatten_pipeline(pipe)
    return ForestEngine(flat, device), RowEncoder(flat)


@pytest.mark.parametrize("which", ["rf100d6", "gbdt_small"])
def test_rank_kernel_all_reference_rows(curated, inference, adversarial, rf100d6, gbdt_small, which):
    from oracle import reference_pipeline as rp

    pipe = {"rf100d6": rf100d6, "gbdt_small": gbdt_small}[which]
    eng, enc = _engine(pipe)
    try:
        info = eng.info()
        assert info["rank_ok"] and info["rank_row_bytes"] == 32
        l0 = info["launches_rank"]
        for df in (curated, inference, adversarial):
            want_p, want_l = rp.oracle_predict(pipe, df)
            rk = enc.rank_rows(enc.encode_frame(df))
            p64, l64 = eng.predict_rows(rk, np.float64)
            p32, l32 = eng.predict_rows(rk, np.float32)
            assert np.abs(p64 - want_p).max() <= TOL64 and (l64 == want_l).all()
            assert np.abs(p32.astype(np.float64) - want_p).max() <= TOL32 and (l32 == want_l).all()
        assert eng.info()["launches_rank"] > l0, "ranked rows must be scored by the rank kernel"
    finally:
        eng.close()


def test_rank_kernel_batch_size_edges_and_determinism(curated, rf100d6):
    from oracle import reference_pipeline as rp

    eng, enc = _engine(rf100d6)
    try:
        want_p, want_l = rp.oracle_predict(rf100d6, curated)
        rk = enc.rank_rows(enc.encode_frame(curated))
        # 1 .. 33: fewer tree groups than warps; 132*32+1: one tile more than CTAs on an H100 (132 SMs); 90 000 below: a second round per CTA
        for n in (0, 1, 2, 31, 32, 33, 131, 132 * 32 + 1, 147, 4737, 16384, 30000):
            p, l = eng.predict_rows(rk[:n], np.float64)
            assert p.shape == (n,)
            if n:
                assert np.abs(p - want_p[:n]).max() <= TOL64 and (l == want_l[:n]).all()
        big = np.concatenate([rk, rk, rk])  # 90 000 rows: CTAs take more than 16 tiles -> several rounds
        p, l = eng.predict_rows(big, np.float64)
        assert np.abs(p - np.tile(want_p, 3)).max() <= TOL64 and (l == np.tile(want_l, 3)).all()
        p2, l2 = eng.predict_rows(big, np.float64)
        assert (p == p2).all() and (l == l2).all()  # fixed summation order: bit-identical run to run
        perm = np.random.default_rng(3).permutation(len(rk))
        pp, lp = eng.predict_rows(rk[perm], np.float64)
        assert np.abs(pp - p[: len(rk)][perm]).max() <= 1e-15 and (lp == l[: len(rk)][perm]).all()
        # async ring + pairs output on ranked rows
        out = eng.predict_pairs(rk[:20000])
        assert np.abs(out["proba1"].astype(np.float64) - want_p[:20000]).max() <= TOL32 and (out["label"] == want_l[:20000]).all()
    finally:
        eng.close()


def test_rank_unavailable_is_refused(curated):
    """A forest without a rank layout (depth > 8) refuses ranked rows loudly and keeps scoring float32 rows."""
    from oracle import reference_pipeline as rp

    pipe = rp.fit_reference_pipeline(curated.iloc[:3000], dict(n_estimators=9, max_depth=12, random_state=0))
    eng, enc = _engine(pipe)
    try:
        assert not eng.info()["rank_ok"]
        with pytest.raises(ValueError):  # the Python layer does not even know a ranked width for this model
            eng.predict_rows(np.zeros((4, 8), dtype=np.uint32), np.float64)
        from databricks_kubernetes_mlops_poc_b200 import _cabi

        rows, out = np.zeros((4, 8), dtype=np.uint32), np.zeros(4, dtype=np.float64)
        rc = _cabi.load_library().b2f_predict_ex(eng.handle, _cabi.ptr(rows), 4, _cabi.ROWS_RANKED, _cabi.ptr(out), 1, None)
        assert rc == -1 and "not available" in _cabi.last_error()  # the C ABI refuses the format with B2F_EINVAL
        want_p, want_l = rp.oracle_predict(pipe, curated.iloc[3000:3500])
        p, l = eng.predict_rows(enc.encode_frame(curated.iloc[3000:3500]), np.float64)
        assert np.abs(p - want_p).max() <= TOL64 and (l == want_l).all()
    finally:
        eng.close()


@pytest.mark.parametrize("rows", ["packed64", "ranked"])
def test_pipeline_predict_large_frames(curated, inference, adversarial, rf100d6, iforest, rows, monkeypatch):
    """B200Model.predict on frames large enough for the chunked columnar pipeline (b2f_scorer): every row of the reference
    table, other column orders, object-dtype columns (portable path), float32 overflow, and the outlier forest riding along.
    Both row formats the scorer's workers can write: the 64-byte float32 rows (default: cheapest on the host) and the
    32-byte ranked rows (B200_SCORER_ROWS=ranked)."""
    import pandas as pd

    from databricks_kubernetes_mlops_poc_b200 import engine as engine_mod
    from databricks_kubernetes_mlops_poc_b200.model import B200Model
    from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES
    from oracle import reference_pipeline as rp

    monkeypatch.setattr(engine_mod, "_FMT_OVERRIDE", engine_mod.ROWS_RANKED if rows == "ranked" else None)
    model = B200Model.from_pipeline(rf100d6, devices=[0])
    try:
        want_p, _ = rp.oracle_predict(rf100d6, curated)
        df = curated[ALL_FEATURES]
        out = model.predict(df)
        assert model.last_timing is not None and model.last_timing["chunks"] >= 2, "30 000 rows must take the chunked pipeline"
        assert model.last_timing["row_format"] == (2 if rows == "ranked" else 1)
        assert np.abs(np.asarray(out["predictions"]) - want_p).max() <= TOL64
        assert out["outliers"] == [0] * len(df) and len(out["predictions"]) == len(df)
        # the same frame again (staging reuse), reversed column order, a slice with an offset
        assert model.predict(df)["predictions"] == out["predictions"]
        assert model.predict(df[ALL_FEATURES[::-1]])["predictions"] == out["predictions"]
        # another batch size groups the per-warp partial sums differently: equal to the last bit or two, not bitwise
        part = model.predict(df.iloc[1234:9999])
        assert np.abs(np.asarray(part["predictions"]) - np.asarray(out["predictions"][1234:9999])).max() <= 1e-15
        # object-dtype string columns with None / NaN / unknown categories: the general path, same answers
        big_adv = pd.concat([adversarial] * 5, ignore_index=True)
        wa, _ = rp.oracle_predict(rf100d6, big_adv)
        assert np.abs(np.asarray(model.predict(big_adv)["predictions"]) - wa).max() <= TOL64
        # Arrow-backed strings with nulls and unknowns through the pipeline itself
        arrow_adv = big_adv.copy()
        for c in rp.CATEGORICAL_FEATURES:
            arrow_adv[c] = arrow_adv[c].astype("str")
        got = model.predict(arrow_adv)["predictions"]
        # NaN and None become the same Arrow null: compare with the library on the frame it would see
        wa2, _ = rp.oracle_predict(rf100d6, arrow_adv)
        assert np.abs(np.asarray(got) - wa2).max() <= TOL64
        bad = df.iloc[:5000].copy()
        bad.iloc[4321, bad.columns.get_loc("credit_limit")] = 1e39
        with pytest.raises(ValueError):
            model.predict(bad)
        again = model.predict(df.iloc[:5000])["predictions"]  # the scorer survives a refused request
        assert np.abs(np.asarray(again) - np.asarray(out["predictions"][:5000])).max() <= 1e-15
    finally:
        model.close()

    full = B200Model.from_pipeline(rf100d6, outlier=iforest, outlier_threshold=0.0, devices=[0])
    try:
        df = curated[ALL_FEATURES].iloc[:20000]
        out = full.predict(df)
        want_o = (-iforest.decision_function(df[rp.NUMERIC_FEATURES].to_numpy()) > 0.0).astype(int)
        assert full.last_timing["row_format"] == 1  # with the outlier forest attached: float32 (packed) rows, 24-byte records back
        assert np.abs(np.asarray(out["predictions"]) - want_p[:20000]).max() <= TOL64
        assert out["outliers"] == want_o.tolist()
    finally:
        full.close()


def test_scorer_c_abi_directly(curated, rf100d6):
    """b2f_scorer_* through ctypes: explicit chunk size, every row format, float32 outputs, one thread (synchronous)."""
    from databricks_kubernetes_mlops_poc_b200.engine import Scorer
    from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES
    from oracle import reference_pipeline as rp

    eng, enc = _engine(rf100d6)
    try:
        want_p, _ = rp.oracle_predict(rf100d6, curated)
        df = curated[ALL_FEATURES]
        cols = enc.frame_columns(df)
        assert cols is not None
        for threads in (1, 5):
            sc = Scorer(eng, enc, threads)
            assert sc.threads == threads
            for fmt, mode, tol in ((2, 1, TOL64), (1, 1, TOL64), (0, 0, TOL32), (2, 0, TOL32)):
                for chunk in (0, 777, 30000, 100000):
                    n_chunks = sc.start(len(df), cols, out_mode=mode, chunk_rows=chunk, fmt=fmt)
                    # the chunks tile the request
                    assert sc.bounds[0] == 0 and sc.bounds[-1] == len(df) and len(sc.bounds) == n_chunks + 1
                    assert all(a < b for a, b in zip(sc.bounds, sc.bounds[1:]))
                    if chunk:
                        assert sc.bounds[1] == min(chunk, len(df))
                    for c in range(n_chunks):
                        sc.wait(c)
                    got = np.array(sc.results(), dtype=np.float64)
                    assert np.abs(got - want_p).max() <= tol, (threads, fmt, mode, chunk)
            sc.close()
    finally:
        eng.close()


def test_schema_with_fewer_categoricals(curated):
    """A model with 7 categorical and 11 numeric features (round-1 advisor finding: the packed 64-byte row is decoded for
    exactly nine categoricals).  Such a model is never offered packed rows; 96-byte rows, ranked rows and the plugin call on
    more than 128 rows all agree with the library."""
    from sklearn.compose import ColumnTransformer
    from sklearn.ensemble import RandomForestClassifier
    from sklearn.impute import SimpleImputer
    from sklearn.pipeline import Pipeline
    from sklearn.preprocessing import OneHotEncoder

    from databricks_kubernetes_mlops_poc_b200 import _cabi
    from databricks_kubernetes_mlops_poc_b200.model import B200Model
    from oracle import reference_pipeline as rp

    cat, num = rp.CATEGORICAL_FEATURES[:7], rp.NUMERIC_FEATURES[:11]
    catp = Pipeline([("imputer", SimpleImputer(strategy="constant", fill_value="missing")), ("ohe", OneHotEncoder(handle_unknown="ignore"))])
    nump = Pipeline([("imputer", SimpleImputer(strategy="median"))])
    pipe = Pipeline([("preprocessor", ColumnTransformer([("categorical", catp, cat), ("numeric", nump, num)])),
                     ("classifier", RandomForestClassifier(n_estimators=30, max_depth=6, random_state=0, n_jobs=-1))])
    tr = curated.iloc[:4000]
    pipe.fit(tr[cat + num], tr[rp.TARGET].to_numpy())
    df = curated[cat + num].iloc[4000:4700]
    want = pipe.predict_proba(df)[:, 1]
    model = B200Model.from_pipeline(pipe, devices=[0])
    try:
        eng, enc = model.engine, model.encoder
        assert not enc.packed_ok and not eng.info()["packed_ok"] and eng.info()["rank_ok"]
        rows = enc.encode_frame(df)
        p, _ = eng.predict_rows(rows, np.float64)
        assert np.abs(p - want).max() <= TOL64
        p, _ = eng.predict_rows(enc.rank_rows(rows), np.float64)
        assert np.abs(p - want).max() <= TOL64
        bad = np.zeros((4, 16), dtype=np.uint32)
        out = np.zeros(4, dtype=np.float64)
        assert _cabi.load_library().b2f_predict_ex(eng.handle, _cabi.ptr(bad), 4, _cabi.ROWS_PACKED64, _cabi.ptr(out), 1, None) == -1
        got = model.predict(df)["predictions"]  # 700 rows: the columnar pipeline, ranked rows
        assert model.last_timing is not None and np.abs(np.asarray(got) - want).max() <= TOL64
        small = model.predict(df.iloc[:5])["predictions"]
        assert np.abs(np.asarray(small) - want[:5]).max() <= TOL64
    finally:
        model.close()
