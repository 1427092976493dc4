"""k_tree_shap_interventional on the GPU against the per-pair recursion (tests/treeshap_interventional.py) and the path-table
emulator (tests/path_walk_interventional.py): parity, local accuracy against the library's own predictions, base_value
against the mean prediction over the background, identities, batch edges, determinism, the C-ABI error paths and lifecycle,
B200Model / load_model and POST /explain/interventional.

The recursion visits every node for every (row, background row) pair, so it runs on small row samples."""

import os

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu


def _dense(pipe, df):
    from oracle import treewalk as tw

    dump = tw.dump_pipeline(pipe)
    return dump, tw.transform_dense(dump, *tw.encode_frame(dump, df))


def _engine(pipe):
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer, flatten_pipeline

    flat = flatten_pipeline(pipe)
    table = flatten_explainer(pipe, flat)
    eng = ForestEngine(flat, 0)
    eng.attach_explainer(table)
    return flat, table, eng, RowEncoder(flat)


def _check(pipe, frames, backgrounds, oracle_rows=8, emulate_bytes=False):
    """Per background: both float32 row formats (requests and background) give identical arrays; base_value is the mean of the
    library's outputs over the background; local accuracy on every row; the recursion on the first ``oracle_rows`` rows
    where rows x background rows stay within 40 000 pairs; ``emulate_bytes``: table_bytes equals the emulator's count."""
    import treeshap_interventional as ti

    from oracle import treewalk as tw

    flat, table, eng, enc = _engine(pipe)
    try:
        for bg in backgrounds:
            zr = enc.encode_frame(bg)
            nbytes = eng.attach_background(zr)
            dump, Z = _dense(pipe, bg)
            if flat.agg_mode == 0:
                want_base = eng.predict_rows(zr, np.float64)[0].mean()
            else:
                want_base = tw.walk_numpy(dump, Z)[2].mean()
            for df in frames:
                rows = enc.encode_frame(df)
                phi, base = eng.explain_interventional_rows(rows)
                assert abs(base - want_base) <= 1e-12
                _, X = _dense(pipe, df)
                target = eng.predict_rows(rows, np.float64)[0] if flat.agg_mode == 0 else tw.walk_numpy(dump, X)[2]
                assert np.abs(base + phi.sum(axis=1) - target).max() <= 1e-12
                if enc.packed_ok:
                    assert np.array_equal(eng.explain_interventional_rows(enc.pack_rows(rows))[0], phi)
                if oracle_rows * len(bg) <= 40000:  # the recursion's cost grows with rows x background rows x nodes
                    want, wbase = ti.interventional_shap(dump, X[:oracle_rows], Z)
                    assert abs(wbase - base) <= 1e-12
                    assert np.abs(phi[:oracle_rows] - want).max() <= 1e-12
            if enc.packed_ok:
                assert eng.attach_background(enc.pack_rows(zr)) == nbytes
                assert np.array_equal(eng.explain_interventional_rows(rows)[0], phi)
            if emulate_bytes:
                import path_walk_interventional as pwi

                assert pwi.background_table(table, flat.blob, zr)[3] == nbytes
    finally:
        eng.close()


def test_rf100d6(rf100d6, curated, inference, adversarial):
    from oracle import reference_pipeline as rp

    cur = curated[rp.FEATURES]
    inf = inference[list(reversed(rp.FEATURES))]  # another column order
    _check(rf100d6, [cur.iloc[:4096], inf, adversarial], [cur.iloc[[7]], cur.iloc[100:200], cur.iloc[5000:6000]])
    _check(rf100d6, [cur.iloc[:2048], adversarial], [cur], oracle_rows=1, emulate_bytes=True)


def test_rf500d8(rf500d8, curated, adversarial):
    from oracle import reference_pipeline as rp

    cur = curated[rp.FEATURES]
    _check(rf500d8, [cur.iloc[:2048], adversarial], [cur.iloc[[3]], cur.iloc[200:300], cur], oracle_rows=2)


def test_gbdt_small(gbdt_small, curated, adversarial):
    from oracle import reference_pipeline as rp

    cur = curated[rp.FEATURES]
    _check(gbdt_small, [cur.iloc[:3000], adversarial], [cur.iloc[[11]], cur.iloc[300:400], cur.iloc[8000:9000]])


def test_bench_gbdt100d6_full_batch():
    """The benchmark's GBDT 100 x d6 on its 65 536-row batch against 1 000 of its rows: local accuracy in log-odds on every
    row, the recursion on a sample."""
    import bench
    import treeshap_interventional as ti

    from databricks_kubernetes_mlops_poc_b200 import training
    from oracle import treewalk as tw

    base = training.load_base_frame()
    kind, params = bench.MODELS["gbdt100d6"]
    pipe = training.fit_synthetic(kind, base, bench.N_TRAIN, bench.TRAIN_SEED, **params)
    flat, table, eng, enc = _engine(pipe)
    try:
        _, codes, nums = training.synth_arrays(base, bench.BATCH, bench.DATA_SEED)
        rows = enc.encode_arrays(codes, nums)
        dump = tw.dump_pipeline(pipe)
        X = tw.transform_dense(dump, codes, nums)
        eng.attach_background(rows[-1000:])
        phi, b0 = eng.explain_interventional_rows(rows)
        raw = tw.walk_numpy(dump, X)[2]
        assert abs(b0 - raw[-1000:].mean()) <= 1e-12
        assert np.abs(b0 + phi.sum(axis=1) - raw).max() <= 1e-12
        want, wb = ti.interventional_shap(dump, X[:8], X[-1000:])
        assert abs(wb - b0) <= 1e-12 and np.abs(phi[:8] - want).max() <= 1e-12
    finally:
        eng.close()


def test_deep_forest_stumps_one_and_33_trees(curated, adversarial):
    from oracle import reference_pipeline as rp

    cur = curated[rp.FEATURES]
    deep = rp.fit_reference_pipeline(curated.iloc[:6000], dict(n_estimators=37, max_depth=24, criterion="entropy", random_state=1))
    _check(deep, [cur.iloc[6000:6400], adversarial.iloc[:200]], [cur.iloc[[1]], cur.iloc[:100]], oracle_rows=4)
    for params in (dict(n_estimators=1, max_depth=1, random_state=0), dict(n_estimators=33, max_depth=1, random_state=0),
                   dict(n_estimators=1, max_depth=6, random_state=0), dict(n_estimators=33, max_depth=3, random_state=0)):
        pipe = rp.fit_reference_pipeline(curated.iloc[:3000], params)
        _check(pipe, [cur.iloc[3000:3500], adversarial], [cur.iloc[[2]], cur.iloc[:100]])


def test_identities_batch_edges_and_determinism(rf100d6, curated):
    from oracle import reference_pipeline as rp

    flat, table, eng, enc = _engine(rf100d6)
    try:
        rows = enc.encode_frame(curated[rp.FEATURES].iloc[:1024])
        for i in (0, 5, 77):  # the row itself as the background: nothing moves
            eng.attach_background(rows[i : i + 1])
            phi, base = eng.explain_interventional_rows(rows[i : i + 1])
            assert (phi == 0.0).all()
            assert abs(base - eng.predict_rows(rows[i : i + 1], np.float64)[0][0]) <= 1e-12
        bg = enc.encode_frame(curated[rp.FEATURES].iloc[2000:2500])
        eng.attach_background(np.concatenate([bg, bg]))
        doubled, b2 = eng.explain_interventional_rows(rows)
        eng.attach_background(bg)
        big = np.concatenate([rows] * 64)  # 65 536 rows
        ref, b1 = eng.explain_interventional_rows(big)
        assert np.abs(doubled - ref[:1024]).max() <= 1e-14 and abs(b1 - b2) <= 1e-14
        assert np.array_equal(ref, eng.explain_interventional_rows(big)[0])  # bit-identical run to run
        for n in (0, 1, 31, 32, 33, 1000, 65536):
            phi, _ = eng.explain_interventional_rows(big[:n])
            assert phi.shape == (n, 23)
            if n:
                assert np.abs(phi - ref[:n]).max() <= 1e-14
                assert np.array_equal(phi, eng.explain_interventional_rows(big[:n])[0])
    finally:
        eng.close()


def test_errors_and_lifecycle(rf100d6, curated):
    from databricks_kubernetes_mlops_poc_b200._cabi import B2FError
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine
    from oracle import reference_pipeline as rp

    flat, table, eng, enc = _engine(rf100d6)
    plain = ForestEngine(flat, 0)
    try:
        rows = enc.encode_frame(curated[rp.FEATURES].iloc[:64])
        with pytest.raises(B2FError, match=r"rc=-6\).*no explainer"):
            plain.attach_background(rows)
        with pytest.raises(B2FError, match=r"rc=-6\).*no explainer"):
            plain.explain_interventional_rows(rows)
        with pytest.raises(B2FError, match=r"rc=-6\).*no background"):
            eng.explain_interventional_rows(rows)
        with pytest.raises(B2FError, match=r"rc=-1\).*at least one row"):
            eng.attach_background(rows[:0])
        if eng.rank_words:
            with pytest.raises(B2FError, match=r"rc=-1\).*ranked"):
                eng.attach_background(enc.rank_rows(rows))
        eng.attach_background(rows[:10])
        if eng.rank_words:
            with pytest.raises(B2FError, match=r"rc=-1\).*ranked"):
                eng.explain_interventional_rows(enc.rank_rows(rows))
        first, _ = eng.explain_interventional_rows(rows)
        eng.attach_background(rows[10:40])  # replaces the first background
        second, _ = eng.explain_interventional_rows(rows)
        fresh = ForestEngine(flat, 0)
        try:
            fresh.attach_explainer(table)
            fresh.attach_background(rows[10:40])
            assert np.array_equal(second, fresh.explain_interventional_rows(rows)[0])
        finally:
            fresh.close()
        assert not np.array_equal(first, second)
        eng.attach_explainer(table)  # a new explainer drops the background
        with pytest.raises(B2FError, match=r"rc=-6\).*no background"):
            eng.explain_interventional_rows(rows)
        assert eng.explain_rows(rows)[0].shape == (64, 23)
    finally:
        plain.close()
        eng.close()


def test_device_entry_matches_host_path(rf100d6, curated):
    from databricks_kubernetes_mlops_poc_b200._cabi import ROWS_PACKED64, ROWS_WORDS24
    from oracle import reference_pipeline as rp

    flat, table, eng, enc = _engine(rf100d6)
    try:
        rows = enc.encode_frame(curated[rp.FEATURES].iloc[:20000])
        eng.attach_background(rows[-500:])
        for n in (5, 20000):
            want, _ = eng.explain_interventional_rows(rows[:n])
            for fmt, r in ((ROWS_WORDS24, rows[:n]), (ROWS_PACKED64, enc.pack_rows(rows[:n]))):
                r = np.ascontiguousarray(r)
                d_rows, d_phi = eng.device_alloc(r.nbytes), eng.device_alloc(n * 23 * 8)
                try:
                    eng.h2d(d_rows, r)
                    eng.explain_interventional_device(d_rows, n, d_phi, fmt)
                    eng.sync()
                    got = np.empty((n, 23), dtype=np.float64)
                    eng.d2h(got, d_phi)
                finally:
                    eng.device_free(d_rows)
                    eng.device_free(d_phi)
                assert np.array_equal(got, want)
    finally:
        eng.close()


def test_model_dir_and_http(tmp_path, rf100d6, curated, adversarial):
    import asyncio

    import httpx

    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer, flatten_pipeline
    from databricks_kubernetes_mlops_poc_b200.model import BACKGROUND_FILE, B200Model, load_model, save_model_dir
    from databricks_kubernetes_mlops_poc_b200.server import create_app
    from oracle import reference_pipeline as rp

    bg = pd.concat([curated[rp.FEATURES].iloc[:300], adversarial.iloc[:40]], ignore_index=True)
    df = pd.concat([curated[rp.FEATURES].iloc[1000:1300], adversarial], ignore_index=True)[list(reversed(rp.FEATURES))]
    model = B200Model.from_pipeline(rf100d6, explain=True, background=bg)
    flat = flatten_pipeline(rf100d6)
    save_model_dir(str(tmp_path / "m"), flat, explain_blob=flatten_explainer(rf100d6, flat), explain_background=bg)
    assert os.path.exists(tmp_path / "m" / BACKGROUND_FILE)
    loaded = load_model(str(tmp_path / "m"))
    try:
        assert model.background_attached and loaded.background_attached
        want = model.explain_interventional(df)
        got = loaded.explain_interventional(df)
        assert got["background_rows"] == want["background_rows"] == len(bg)
        assert np.array_equal(got["contributions"], want["contributions"]) and got["base_value"] == want["base_value"]
        assert want["predictions"] == model.predict(df)["predictions"]
        body = df.iloc[:50].to_dict(orient="records")
        app = create_app(model=loaded)

        async def main():
            async with app.router.lifespan_context(app):
                async with httpx.AsyncClient(transport=httpx.ASGITransport(app=app), base_url="http://t") as c:
                    return await c.post("/explain/interventional", json=body)

        j = asyncio.run(main()).json()
        assert j["background_rows"] == len(bg) and j["base_value"] == want["base_value"]
        assert np.abs(np.asarray(j["contributions"]) - want["contributions"][:50]).max() <= 1e-14
    finally:
        model.close()
        loaded.close()
    plain = B200Model.from_pipeline(rf100d6, explain=True)
    try:
        assert not plain.background_attached
        with pytest.raises(RuntimeError, match="no background"):
            plain.explain_interventional(df)
    finally:
        plain.close()
    os.environ["B200_EXPLAIN"] = "off"
    try:
        c = load_model(str(tmp_path / "m"))
        assert not c.explainer_attached and not c.background_attached
        c.close()
    finally:
        del os.environ["B200_EXPLAIN"]
