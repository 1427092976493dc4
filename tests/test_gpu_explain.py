"""k_tree_shap on the GPU against the numpy TreeSHAP oracle (oracle/treeshap.py), local accuracy against the library's own
predictions, batch edges, determinism, the C-ABI error paths, B200Model / load_model and POST /explain.

Oracle cost on the CPU is noted where it is large: Algorithm 2 in numpy visits every node for every row."""

import os

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu


def _dense(pipe, df):
    from oracle import treeshap as ts
    from oracle import treewalk as tw

    dump = tw.dump_pipeline(pipe)
    X = tw.transform_dense(dump, *tw.encode_frame(dump, df))
    return dump, ts.dump_covers(pipe), X


def _engine(pipe):
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer, flatten_pipeline

    flat = flatten_pipeline(pipe)
    eng = ForestEngine(flat, 0)
    eng.attach_explainer(flatten_explainer(pipe, flat))
    return flat, eng, RowEncoder(flat)


def _check(pipe, frames, oracle_rows=None, tol=1e-12):
    """Both float32 row formats vs the oracle; local accuracy vs the library's float64 predictions."""
    from oracle import treeshap as ts
    from oracle import treewalk as tw

    flat, eng, enc = _engine(pipe)
    try:
        for df in frames:
            rows = enc.encode_frame(df)
            phi, base = eng.explain_rows(rows)
            p, _ = eng.predict_rows(rows, np.float64)
            dump, cov, X = _dense(pipe, df)
            _, _, raw = tw.walk_numpy(dump, X)
            target = p if flat.agg_mode == 0 else raw
            assert np.abs(base + phi.sum(axis=1) - target).max() <= 1e-12
            if enc.packed_ok:
                phi_p, _ = eng.explain_rows(enc.pack_rows(rows))
                assert np.array_equal(phi_p, phi)
            sel = slice(None) if oracle_rows is None else slice(0, oracle_rows)
            want, want_base = ts.tree_shap(dump, cov, X[sel])
            assert abs(want_base - base) <= 1e-12
            assert np.abs(phi[sel] - want).max() <= tol
    finally:
        eng.close()


def test_rf100d6_all_curated_rows(rf100d6, curated, inference, adversarial):
    """30 000 curated rows: the numpy oracle takes about a minute on one CPU core for these."""
    from oracle import reference_pipeline as rp

    inf = inference[list(reversed(rp.FEATURES))]  # another column order
    _check(rf100d6, [curated[rp.FEATURES], inf, adversarial])


def test_rf500d8(rf500d8, curated, adversarial):
    from oracle import reference_pipeline as rp

    _check(rf500d8, [curated[rp.FEATURES].iloc[:2048], adversarial])
    # local accuracy on all rows (no oracle)
    flat, eng, enc = _engine(rf500d8)
    try:
        rows = enc.encode_frame(curated[rp.FEATURES])
        phi, base = eng.explain_rows(rows)
        p, _ = eng.predict_rows(rows, np.float64)
        assert np.abs(base + phi.sum(axis=1) - p).max() <= 1e-12
    finally:
        eng.close()


def test_gbdt_small(gbdt_small, curated, adversarial):
    from oracle import reference_pipeline as rp

    _check(gbdt_small, [curated[rp.FEATURES].iloc[:3000], adversarial])


def test_bench_gbdt100d6_full_batch():
    """The benchmark's GBDT 100 x d6 (its own recipe) on its 65 536-row synthetic batch: local accuracy in log-odds on the whole
    batch against the raw margin, the oracle on a 2 048-row sample."""
    import bench
    from databricks_kubernetes_mlops_poc_b200 import training
    from oracle import treeshap as ts
    from oracle import treewalk as tw

    base = training.load_base_frame()
    kind, params = bench.MODELS["gbdt100d6"]
    pipe = training.fit_synthetic(kind, base, bench.N_TRAIN, bench.TRAIN_SEED, **params)
    flat, eng, enc = _engine(pipe)
    try:
        _, codes, nums = training.synth_arrays(base, bench.BATCH, bench.DATA_SEED)
        rows = enc.encode_arrays(codes, nums)
        phi, b0 = eng.explain_rows(rows)
        dump = tw.dump_pipeline(pipe)
        # the same rows as the oracle's dense matrix: codes as they are, NaN numerics imputed
        X = tw.transform_dense(dump, codes, nums)
        _, _, raw = tw.walk_numpy(dump, X)
        assert np.abs(b0 + phi.sum(axis=1) - raw).max() <= 1e-12
        want, wb = ts.tree_shap(dump, ts.dump_covers(pipe), X[:2048])
        assert abs(wb - b0) <= 1e-12 and np.abs(phi[:2048] - want).max() <= 1e-12
    finally:
        eng.close()


def test_deep_forest_stumps_one_and_33_trees(curated, adversarial):
    from oracle import reference_pipeline as rp

    deep = rp.fit_reference_pipeline(curated.iloc[:6000], dict(n_estimators=37, max_depth=24, criterion="entropy", random_state=1))
    _check(deep, [curated[rp.FEATURES].iloc[6000:6400], adversarial.iloc[:200]])
    for params in (dict(n_estimators=1, max_depth=1, random_state=0), dict(n_estimators=33, max_depth=1, random_state=0),
                   dict(n_estimators=1, max_depth=6, random_state=0), dict(n_estimators=33, max_depth=3, random_state=0)):
        pipe = rp.fit_reference_pipeline(curated.iloc[:3000], params)
        _check(pipe, [curated[rp.FEATURES].iloc[3000:3500], adversarial])


def test_batch_edges_and_determinism(rf100d6, curated):
    from oracle import reference_pipeline as rp

    flat, eng, enc = _engine(rf100d6)
    try:
        rows = enc.encode_frame(curated[rp.FEATURES].iloc[:1024])
        big = np.concatenate([rows] * 64)  # 65 536 rows
        ref, _ = eng.explain_rows(big)
        again, _ = eng.explain_rows(big)
        assert np.array_equal(ref, again)  # bit-identical run to run
        for n in (0, 1, 2, 31, 32, 33, 1000, 4097, 65536):
            phi, _ = eng.explain_rows(big[:n])
            assert phi.shape == (n, 23)
            if n:
                assert np.abs(phi - ref[:n]).max() <= 1e-14
                phi2, _ = eng.explain_rows(big[:n])
                assert np.array_equal(phi, phi2)
    finally:
        eng.close()


def test_errors(rf100d6, gbdt_small, curated):
    from databricks_kubernetes_mlops_poc_b200._cabi import B2FError
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer, flatten_pipeline
    from oracle import reference_pipeline as rp

    flat, eng, enc = _engine(rf100d6)
    plain = ForestEngine(flat, 0)
    try:
        other = flatten_explainer(gbdt_small)
        with pytest.raises(B2FError, match=r"rc=-1\).*(shape|fingerprint)"):
            eng.attach_explainer(other)
        rf_other = rp.fit_reference_pipeline(curated.iloc[:2000], rp.PINNED_RF["rf100d6"])
        with pytest.raises(B2FError, match=r"rc=-1\).*fingerprint"):
            eng.attach_explainer(flatten_explainer(rf_other))
        rows = enc.encode_frame(curated[rp.FEATURES].iloc[:64])
        if eng.rank_words:
            with pytest.raises(B2FError, match=r"rc=-1\).*ranked"):
                eng.explain_rows(enc.rank_rows(rows))
        with pytest.raises(B2FError, match=r"rc=-6\).*no explainer"):
            plain.explain_rows(rows)
        # the failed attaches left the first explainer in place
        phi, _ = eng.explain_rows(rows)
        assert phi.shape == (64, 23)
    finally:
        plain.close()
        eng.close()
    assert flatten_pipeline(rf100d6).blob == flat.blob


def test_model_dir_with_and_without_explainer(tmp_path, rf100d6, curated, adversarial):
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer, flatten_pipeline
    from databricks_kubernetes_mlops_poc_b200.model import EXPLAIN_FILE, load_model, save_model_dir
    from oracle import reference_pipeline as rp

    flat = flatten_pipeline(rf100d6)
    save_model_dir(str(tmp_path / "plain"), flat)
    save_model_dir(str(tmp_path / "expl"), flat, explain_blob=flatten_explainer(rf100d6, flat))
    assert os.path.exists(tmp_path / "expl" / EXPLAIN_FILE)
    df = pd.concat([curated[rp.FEATURES].iloc[:700], adversarial], ignore_index=True)[list(reversed(rp.FEATURES))]
    a, b = load_model(str(tmp_path / "plain")), load_model(str(tmp_path / "expl"))
    try:
        pa, pb = a.predict(df), b.predict(df)
        assert np.asarray(pa["predictions"]).tobytes() == np.asarray(pb["predictions"]).tobytes()
        assert pa["outliers"] == pb["outliers"]
        with pytest.raises(RuntimeError, match="no explainer"):
            a.explain(df)
        out = b.explain(df)
        assert out["feature_names"] == b.all_features and out["output"] == "probability"
        assert out["predictions"] == pb["predictions"]
        phi, base = b.engine.explain_rows(b.encoder.encode_frame(df))
        assert np.array_equal(out["contributions"], phi) and out["base_value"] == base
    finally:
        a.close()
        b.close()
    os.environ["B200_EXPLAIN"] = "off"
    try:
        c = load_model(str(tmp_path / "expl"))
        assert not c.explainer_attached
        c.close()
    finally:
        del os.environ["B200_EXPLAIN"]


def test_http_explain_matches_model_under_concurrent_predict(rf100d6, curated):
    import asyncio

    import httpx

    from databricks_kubernetes_mlops_poc_b200.model import B200Model
    from databricks_kubernetes_mlops_poc_b200.server import create_app
    from oracle import reference_pipeline as rp

    model = B200Model.from_pipeline(rf100d6, explain=True)
    df = curated[rp.FEATURES].iloc[:300].reset_index(drop=True)
    want = model.explain(df)
    want_p = model.predict(df)["predictions"]
    body = df.to_dict(orient="records")
    app = create_app(model=model)

    async def main():
        async with app.router.lifespan_context(app):
            transport = httpx.ASGITransport(app=app)
            async with httpx.AsyncClient(transport=transport, base_url="http://t") as c:
                reqs = []
                for i in range(24):
                    reqs.append(c.post("/explain" if i % 3 == 0 else "/predict", json=body[i * 10:(i + 1) * 10 + 5]))
                return await asyncio.gather(*reqs)

    try:
        rs = asyncio.run(main())
        for i, r in enumerate(rs):
            assert r.status_code == 200
            lo, hi = i * 10, (i + 1) * 10 + 5
            j = r.json()
            if i % 3 == 0:
                assert j["feature_names"] == want["feature_names"] and j["output"] == "probability"
                assert j["base_value"] == want["base_value"]
                # another batch size may group partial sums differently: last bits only
                assert np.abs(np.asarray(j["contributions"]) - want["contributions"][lo:hi]).max() <= 1e-14
                assert np.abs(np.asarray(j["predictions"]) - np.asarray(want["predictions"][lo:hi])).max() <= 1e-12
            else:
                assert np.abs(np.asarray(j["predictions"]) - np.asarray(want_p[lo:hi])).max() <= 1e-12
    finally:
        model.close()


def test_explain_device_matches_host_path(rf100d6, curated):
    """b2f_explain_device (compute stream, its own scratch, the finishing kernel for small batches) equals b2f_explain."""
    from databricks_kubernetes_mlops_poc_b200._cabi import ROWS_PACKED64, ROWS_WORDS24
    from oracle import reference_pipeline as rp

    flat, eng, enc = _engine(rf100d6)
    try:
        rows = enc.encode_frame(curated[rp.FEATURES].iloc[:20000])
        for n in (5, 20000):
            want, _ = eng.explain_rows(rows[:n])
            for fmt, r in ((ROWS_WORDS24, rows[:n]), (ROWS_PACKED64, enc.pack_rows(rows[:n]))):
                r = np.ascontiguousarray(r)
                d_rows, d_phi = eng.device_alloc(r.nbytes), eng.device_alloc(n * 23 * 8)
                try:
                    eng.h2d(d_rows, r)
                    eng.explain_device(d_rows, n, d_phi, fmt)
                    eng.sync()
                    got = np.empty((n, 23), dtype=np.float64)
                    eng.d2h(got, d_phi)
                finally:
                    eng.device_free(d_rows)
                    eng.device_free(d_phi)
                assert np.array_equal(got, want)
    finally:
        eng.close()


def test_explain_with_outlier_forest_accepts_nan(rf100d6, curated, iforest):
    """With an outlier forest attached predict() refuses NaN numerics (the detector does); explain() uses the classifier
    alone, so such rows are explained, and its predictions are predict()'s for rows predict() accepts."""
    from databricks_kubernetes_mlops_poc_b200.model import B200Model
    from oracle import reference_pipeline as rp

    model = B200Model.from_pipeline(rf100d6, explain=True, outlier=iforest, outlier_threshold=0.0)
    try:
        df = curated[rp.FEATURES].iloc[:500].reset_index(drop=True).copy()
        clean = model.explain(df)
        assert clean["predictions"] == model.predict(df)["predictions"]
        df.loc[::7, "credit_limit"] = np.nan
        with pytest.raises(ValueError):
            model.predict(df)
        out = model.explain(df)
        p = model.engine.predict_rows(model.encoder.encode_frame(df), np.float64)[0]
        assert np.abs(np.asarray(out["predictions"]) - p).max() <= 1e-12
        assert np.abs(out["base_value"] + out["contributions"].sum(axis=1) - p).max() <= 1e-12
    finally:
        model.close()


def test_http_explain_multi_gpu(rf100d6, curated):
    """A model on every GPU of the box: /explain runs on the first GPU only, while /predict batches go round-robin over all of
    them; every answer is right."""
    import asyncio

    import httpx

    from databricks_kubernetes_mlops_poc_b200.engine import device_count
    from databricks_kubernetes_mlops_poc_b200.model import B200Model
    from databricks_kubernetes_mlops_poc_b200.server import create_app
    from oracle import reference_pipeline as rp

    ndev = device_count()
    if ndev < 2:
        pytest.skip("one GPU on this machine")
    model = B200Model.from_pipeline(rf100d6, explain=True, devices=list(range(ndev)))
    single = B200Model.from_pipeline(rf100d6, explain=True, devices=[0])
    df = curated[rp.FEATURES].iloc[:400].reset_index(drop=True)
    want = single.explain(df)
    body = df.to_dict(orient="records")
    app = create_app(model=model)

    async def main():
        async with app.router.lifespan_context(app):
            async with httpx.AsyncClient(transport=httpx.ASGITransport(app=app), base_url="http://t") as c:
                return await asyncio.gather(*[c.post("/explain" if i % 2 == 0 else "/predict", json=body[i * 10:(i + 1) * 10 + 5])
                                              for i in range(36)])

    try:
        for i, r in enumerate(asyncio.run(main())):
            assert r.status_code == 200
            lo, hi = i * 10, (i + 1) * 10 + 5
            j = r.json()
            if i % 2 == 0:
                assert np.abs(np.asarray(j["contributions"]) - want["contributions"][lo:hi]).max() <= 1e-14
            assert np.abs(np.asarray(j["predictions"]) - np.asarray(want["predictions"][lo:hi])).max() <= 1e-12
    finally:
        model.close()
        single.close()
