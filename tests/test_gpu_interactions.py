"""k_tree_shap_interactions on the GPU against the path-table emulator (tests/path_walk_interactions.py) and the conditioning
oracle (tests/treeshap_interactions.py), its sum rules against b2f_explain and the library's predictions, batch edges,
determinism, the device entry point, the C-ABI error paths, interleaving with predict / explain, B200Model and
POST /explain/interactions.

The emulator and the oracle are numpy restatements and slow on the CPU; they see samples, the sum rules see every row."""

import os

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu


def _engine(pipe):
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer, flatten_pipeline

    flat = flatten_pipeline(pipe)
    eng = ForestEngine(flat, 0)
    table = flatten_explainer(pipe, flat)
    eng.attach_explainer(table)
    return flat, eng, RowEncoder(flat), table


def _emulate(table, flat, rows, block=512):
    import path_walk_interactions as pwi

    parts = [pwi.explain_interactions_paths(table, flat.blob, rows[i : i + block])[0] for i in range(0, len(rows), block)]
    return np.concatenate(parts) if parts else np.zeros((0, 23, 23))


def _sum_rules(flat, eng, rows, phi2, base, raw=None):
    """Exactly symmetric; rows sum to b2f_explain's phi; base + total = RF probability / GBDT raw margin."""
    assert np.array_equal(phi2, phi2.transpose(0, 2, 1))
    phi, pbase = eng.explain_rows(rows)
    assert pbase == base
    assert np.abs(phi2.sum(axis=2) - phi).max() <= 1e-12
    target = eng.predict_rows(rows, np.float64)[0] if flat.agg_mode == 0 else raw
    if target is not None:
        assert np.abs(base + phi2.sum(axis=(1, 2)) - target).max() <= 1e-12


def _check(pipe, frames, emu_rows=256, oracle_rows=0):
    """Both float32 row formats; sum rules on every row; the emulator on the first emu_rows of each frame, the oracle on the
    first oracle_rows of the first frame (it visits every node of every tree twice per field the tree tests: minutes for a
    100-tree forest whatever the row count, so the large forests meet it through the emulator, checked against it on the CPU)."""
    import treeshap_interactions as ti

    from oracle import treeshap as ts
    from oracle import treewalk as tw

    flat, eng, enc, table = _engine(pipe)
    try:
        for df in frames:
            rows = enc.encode_frame(df)
            phi2, base = eng.explain_interactions_rows(rows)
            assert phi2.shape == (len(rows), 23, 23)
            dump = tw.dump_pipeline(pipe)
            X = tw.transform_dense(dump, *tw.encode_frame(dump, df))
            _sum_rules(flat, eng, rows, phi2, base, raw=tw.walk_numpy(dump, X)[2])
            if enc.packed_ok:
                assert np.array_equal(eng.explain_interactions_rows(enc.pack_rows(rows))[0], phi2)
            if emu_rows:
                assert np.abs(phi2[:emu_rows] - _emulate(table, flat, rows[:emu_rows])).max() <= 1e-12
            if oracle_rows and df is frames[0]:
                o, ob = ti.tree_shap_interactions(dump, ts.dump_covers(pipe), X[:oracle_rows])
                assert abs(ob - base) <= 1e-12 and np.abs(phi2[:oracle_rows] - o).max() <= 1e-12
    finally:
        eng.close()


def test_rf100d6_curated_inference_adversarial(rf100d6, curated, inference, adversarial):
    """Sum rules on all 30 000 curated rows and every inference and adversarial row; the emulator on 1 024 curated rows and
    256 of each other frame."""
    from oracle import reference_pipeline as rp

    inf = inference[list(reversed(rp.FEATURES))]
    _check(rf100d6, [curated[rp.FEATURES].iloc[:1024], inf, adversarial])
    _check(rf100d6, [curated[rp.FEATURES]], emu_rows=0)


def test_rf500d8(rf500d8, curated, adversarial):
    from oracle import reference_pipeline as rp

    _check(rf500d8, [curated[rp.FEATURES].iloc[:2048], adversarial.iloc[:256]], emu_rows=64)


def test_gbdt_small(gbdt_small, curated, adversarial):
    from oracle import reference_pipeline as rp

    _check(gbdt_small, [curated[rp.FEATURES].iloc[:3000], adversarial], oracle_rows=32)


def test_bench_gbdt100d6_full_batch():
    """The benchmark's GBDT 100 x d6 on its 65 536-row batch: sum rules on the whole batch, the emulator on 1 024 rows."""
    import bench

    from databricks_kubernetes_mlops_poc_b200 import training
    from oracle import treewalk as tw

    base = training.load_base_frame()
    kind, params = bench.MODELS["gbdt100d6"]
    pipe = training.fit_synthetic(kind, base, bench.N_TRAIN, bench.TRAIN_SEED, **params)
    flat, eng, enc, table = _engine(pipe)
    try:
        _, codes, nums = training.synth_arrays(base, bench.BATCH, bench.DATA_SEED)
        rows = enc.encode_arrays(codes, nums)
        phi2, b0 = eng.explain_interactions_rows(rows)
        X = tw.transform_dense(tw.dump_pipeline(pipe), codes, nums)
        _sum_rules(flat, eng, rows, phi2, b0, raw=tw.walk_numpy(tw.dump_pipeline(pipe), X)[2])
        assert np.abs(phi2[:1024] - _emulate(table, flat, rows[:1024])).max() <= 1e-12
    finally:
        eng.close()


def test_deep_forest_stumps_one_and_33_trees(curated, adversarial):
    from databricks_kubernetes_mlops_poc_b200.flatten import parse_explainer
    from oracle import reference_pipeline as rp

    deep = rp.fit_reference_pipeline(curated.iloc[:6000], dict(n_estimators=37, max_depth=24, criterion="entropy", random_state=1))
    _, eng, _, table = _engine(deep)
    eng.close()
    assert parse_explainer(table)["max_len"] > 16  # the 24-element bucket
    _check(deep, [curated[rp.FEATURES].iloc[6000:6400], adversarial.iloc[:200]], emu_rows=64)
    for params in (dict(n_estimators=1, max_depth=1, random_state=0), dict(n_estimators=33, max_depth=1, random_state=0),
                   dict(n_estimators=1, max_depth=6, random_state=0), dict(n_estimators=33, max_depth=3, random_state=0)):
        pipe = rp.fit_reference_pipeline(curated.iloc[:3000], params)
        _check(pipe, [curated[rp.FEATURES].iloc[3000:3500], adversarial], oracle_rows=32)


def test_batch_edges_and_determinism(rf100d6, curated):
    from oracle import reference_pipeline as rp

    flat, eng, enc, _ = _engine(rf100d6)
    try:
        rows = enc.encode_frame(curated[rp.FEATURES].iloc[:1024])
        big = np.concatenate([rows] * 40)  # 40 960 rows: three chunks
        ref, _ = eng.explain_interactions_rows(big)
        again, _ = eng.explain_interactions_rows(big)
        assert np.array_equal(ref, again)
        # 1 .. 12 000 rows: several path ranges and the finishing kernel; 20 000: one range
        for n in (0, 1, 31, 32, 33, 1000, 12000, 20000):
            phi2, _ = eng.explain_interactions_rows(big[:n])
            assert phi2.shape == (n, 23, 23)
            if n:
                assert np.abs(phi2 - ref[:n]).max() <= 1e-14
                assert np.array_equal(phi2, eng.explain_interactions_rows(big[:n])[0])
    finally:
        eng.close()


def test_device_path_matches_host_path(rf100d6, curated):
    from databricks_kubernetes_mlops_poc_b200._cabi import ROWS_PACKED64, ROWS_WORDS24
    from oracle import reference_pipeline as rp

    flat, eng, enc, _ = _engine(rf100d6)
    try:
        rows = enc.encode_frame(curated[rp.FEATURES].iloc[:20000])
        for n in (5, 20000):
            want, _ = eng.explain_interactions_rows(rows[:n])
            for fmt, r in ((ROWS_WORDS24, rows[:n]), (ROWS_PACKED64, enc.pack_rows(rows[:n]))):
                r = np.ascontiguousarray(r)
                d_rows, d_out = eng.device_alloc(r.nbytes), eng.device_alloc(n * 23 * 23 * 8)
                try:
                    eng.h2d(d_rows, r)
                    eng.explain_interactions_device(d_rows, n, d_out, fmt)
                    eng.sync()
                    got = np.empty((n, 23, 23), dtype=np.float64)
                    eng.d2h(got, d_out)
                finally:
                    eng.device_free(d_rows)
                    eng.device_free(d_out)
                assert np.array_equal(got, want)
    finally:
        eng.close()


def test_errors_leave_the_handle_working(rf100d6, curated):
    import ctypes as C

    from databricks_kubernetes_mlops_poc_b200._cabi import ROWS_WORDS24, B2FError
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine
    from oracle import reference_pipeline as rp

    flat, eng, enc, _ = _engine(rf100d6)
    plain = ForestEngine(flat, 0)
    try:
        rows = enc.encode_frame(curated[rp.FEATURES].iloc[:64])
        want_p = eng.predict_rows(rows, np.float64)[0]
        want_phi = eng.explain_rows(rows)[0]
        want2 = eng.explain_interactions_rows(rows)[0]
        with pytest.raises(B2FError, match=r"rc=-6\).*no explainer"):
            plain.explain_interactions_rows(rows)
        lib, h = eng._lib, eng._h
        ptr = rows.ctypes.data_as(C.c_void_p)
        assert lib.b2f_explain_interactions(h, ptr, 64, ROWS_WORDS24, None, None, None) == -1  # NULL output
        assert lib.b2f_explain_interactions(h, ptr, -1, ROWS_WORDS24, None, None, None) == -1  # negative n
        assert lib.b2f_explain_interactions_device(h, None, -1, ROWS_WORDS24, None) == -1
        assert lib.b2f_explain_interactions_device(plain._h, None, 0, ROWS_WORDS24, None) == -6
        if eng.rank_words:
            with pytest.raises(B2FError, match=r"rc=-1\).*ranked"):
                eng.explain_interactions_rows(enc.rank_rows(rows))
        assert np.array_equal(eng.predict_rows(rows, np.float64)[0], want_p)
        assert np.array_equal(eng.explain_rows(rows)[0], want_phi)
        assert np.array_equal(eng.explain_interactions_rows(rows)[0], want2)
    finally:
        plain.close()
        eng.close()


def test_interleaved_calls(rf100d6, curated):
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine
    from oracle import reference_pipeline as rp

    flat, eng, enc, table = _engine(rf100d6)
    probes, grid = [(12, 0, 64)], np.linspace(-5.0, 5e5, 64, dtype=np.float32).view(np.uint32)
    try:
        rows = enc.encode_frame(curated[rp.FEATURES].iloc[:5000])
        alone = (eng.predict_rows(rows, np.float64)[0], eng.explain_rows(rows)[0], eng.explain_interactions_rows(rows)[0])
        pd_alone = eng.partial_dependence_rows(rows, probes, grid)
        for _ in range(2):
            p2 = eng.explain_interactions_rows(rows)[0]
            p = eng.predict_rows(rows, np.float64)[0]
            phi = eng.explain_rows(rows)[0]
            assert np.array_equal(p, alone[0]) and np.array_equal(phi, alone[1]) and np.array_equal(p2, alone[2])
    finally:
        eng.close()
    # every slot stream carries a score batch still in flight when explain, interactions and partial dependence grow the
    # output and scratch buffers those batches share: each buffer is freed only after its stream has finished with it
    eng = ForestEngine(flat, 0)
    try:
        eng.attach_explainer(table)
        n = len(rows)
        staged, proba, label = eng.staging(4 * n)
        proba[:] = -1
        tickets = []
        for k in range(4):
            staged[k * n : (k + 1) * n] = rows
            tickets.append(eng.predict_rows_async(staged[k * n : (k + 1) * n], proba[k * n : (k + 1) * n], label[k * n : (k + 1) * n]))
        got = (eng.explain_rows(rows)[0], eng.explain_interactions_rows(rows)[0], eng.partial_dependence_rows(rows, probes, grid))
        for t in tickets:
            eng.wait(t)
        assert np.array_equal(proba, np.tile(alone[0], 4))
        assert np.array_equal(got[0], alone[1]) and np.array_equal(got[1], alone[2]) and np.array_equal(got[2], pd_alone)
    finally:
        eng.close()


def test_model_dir_and_http_under_concurrent_predict(tmp_path, rf100d6, curated):
    import asyncio

    import httpx

    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer, flatten_pipeline
    from databricks_kubernetes_mlops_poc_b200.model import load_model, save_model_dir
    from databricks_kubernetes_mlops_poc_b200.server import create_app
    from oracle import reference_pipeline as rp

    flat = flatten_pipeline(rf100d6)
    save_model_dir(str(tmp_path / "expl"), flat, explain_blob=flatten_explainer(rf100d6, flat))
    model = load_model(str(tmp_path / "expl"))
    df = curated[rp.FEATURES].iloc[:300].reset_index(drop=True)
    want = model.explain_interactions(df)
    assert want["output"] == "probability" and want["interactions"].shape == (300, 23, 23)
    assert np.abs(want["interactions"].sum(axis=2) - model.explain(df)["contributions"]).max() <= 1e-12
    want_p = model.predict(df)["predictions"]
    body = df.to_dict(orient="records")
    app = create_app(model=model)

    async def main():
        async with app.router.lifespan_context(app):
            async with httpx.AsyncClient(transport=httpx.ASGITransport(app=app), base_url="http://t") as c:
                return await asyncio.gather(*[c.post("/explain/interactions" if i % 3 == 0 else "/predict", json=body[i * 10:(i + 1) * 10 + 5])
                                              for i in range(24)])

    try:
        for i, r in enumerate(asyncio.run(main())):
            assert r.status_code == 200
            lo, hi = i * 10, (i + 1) * 10 + 5
            j = r.json()
            if i % 3 == 0:
                assert j["base_value"] == want["base_value"] and j["feature_names"] == want["feature_names"]
                assert np.abs(np.asarray(j["interactions"]) - want["interactions"][lo:hi]).max() <= 1e-14
            assert np.abs(np.asarray(j["predictions"]) - np.asarray(want_p[lo:hi])).max() <= 1e-12
    finally:
        model.close()
    os.environ["B200_EXPLAIN"] = "off"
    try:
        off = load_model(str(tmp_path / "expl"))
        from fastapi.testclient import TestClient

        with TestClient(create_app(model=off), raise_server_exceptions=False) as c:
            assert c.post("/explain/interactions", json=body[:3]).status_code == 501
        with pytest.raises(RuntimeError, match="no explainer"):
            off.explain_interactions(pd.DataFrame(body[:3]))
        off.close()
    finally:
        del os.environ["B200_EXPLAIN"]
