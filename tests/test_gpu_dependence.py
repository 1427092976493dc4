"""k_partial_dependence on the GPU: scikit-learn's ``partial_dependence(method="brute")`` to 1e-12 on the reference
forests, deep and tiny forests and the schema-zoo schemas; bit-identity with the tile kernel scoring the expanded rows;
grid edges; batch edges, both row formats, the device entry point and determinism; the C-ABI errors; B200Model /
load_model and POST /explain/dependence under concurrent /predict."""

import asyncio
import os

import numpy as np
import pandas as pd
import pytest
from sklearn.inspection import partial_dependence

import schema_zoo as sz

pytestmark = pytest.mark.gpu

TOL = 1e-12


def _model(pipe):
    from databricks_kubernetes_mlops_poc_b200.model import B200Model

    return B200Model.from_pipeline(pipe)


def _sk_agree(pipe, X, out, categorical, rows=None):
    """``out`` of B200Model.partial_dependence(kind="both") against scikit-learn's on the same grids (custom_values), on
    the first ``rows`` rows."""
    Xs = X if rows is None else X.iloc[:rows].reset_index(drop=True)
    for k, f in enumerate(out["feature_names"]):
        want = partial_dependence(pipe, Xs, [f], method="brute", kind="both", categorical_features=categorical,
                                  custom_values={f: np.asarray(out["grid_values"][k], dtype=object if f in categorical else np.float64)})
        ind = out["individual"][k][: len(Xs)]
        assert np.abs(ind - want["individual"][0]).max() <= TOL, f
        if rows is None:
            assert np.abs(out["average"][k] - want["average"][0]).max() <= TOL, f


def _expanded_tile(pipe, X, out):
    """Every curve point scored by a B2F_KERNEL=tile engine on the rows with the field replaced: bit-identical.  False
    when the forest does not fit the tile kernel."""
    from databricks_kubernetes_mlops_poc_b200 import dependence
    from databricks_kubernetes_mlops_poc_b200._cabi import B2FError
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline

    flat = flatten_pipeline(pipe)
    os.environ["B2F_KERNEL"] = "tile"
    try:
        tile = ForestEngine(flat, 0)
    except B2FError as e:
        assert "tile kernel" in str(e)
        return False
    finally:
        del os.environ["B2F_KERNEL"]
    try:
        enc = RowEncoder(flat)
        rows = enc.encode_frame(X)
        for k, f in enumerate(out["feature_names"]):
            words = dependence.encode_grid(enc, f, out["grid_values"][k])
            big = np.repeat(rows, len(words), axis=0)
            big[:, dependence.word_of(enc, f)] = np.tile(words, len(rows))
            p, _ = tile.predict_rows(big, np.float64)
            assert np.array_equal(p.reshape(len(rows), len(words)), out["individual"][k]), f
        return True
    finally:
        tile.close()


def test_rf100d6_all_fields(rf100d6, curated, inference, adversarial):
    from oracle import reference_pipeline as rp

    m = _model(rf100d6)
    try:
        cur = curated[rp.FEATURES].iloc[:80].reset_index(drop=True)
        out = m.partial_dependence(cur, rp.FEATURES, kind="both")
        assert out["output"] == "probability" and len(out["grid_values"]) == 23
        _sk_agree(rf100d6, cur, out, rp.CATEGORICAL_FEATURES)
        assert _expanded_tile(rf100d6, cur, out)
        for X in (inference[list(reversed(rp.FEATURES))].iloc[:200].reset_index(drop=True), adversarial.iloc[:200]):
            out = m.partial_dependence(X, rp.FEATURES, kind="both", grid_frame=curated, grid_resolution=30)
            _sk_agree(rf100d6, X[rp.FEATURES], out, rp.CATEGORICAL_FEATURES, rows=25)
            _expanded_tile(rf100d6, X, out)
            avg = m.partial_dependence(X, rp.FEATURES, kind="average", grid_frame=curated, grid_resolution=30)
            assert "individual" not in avg and all(np.array_equal(a, b) for a, b in zip(avg["average"], out["average"]))
    finally:
        m.close()


@pytest.mark.parametrize("which", ["rf500d8", "gbdt_small", "bench_gbdt", "deep24", "stumps", "one_tree", "trees33"])
def test_other_forests(which, request, curated, adversarial):
    from oracle import reference_pipeline as rp

    if which in ("rf500d8", "gbdt_small"):
        pipe = request.getfixturevalue(which)
    elif which == "bench_gbdt":
        import bench

        from databricks_kubernetes_mlops_poc_b200 import training

        kind, params = bench.MODELS["gbdt100d6"]
        pipe = training.fit_synthetic(kind, training.load_base_frame(), bench.N_TRAIN, bench.TRAIN_SEED, **params)
    else:
        params = {"deep24": dict(n_estimators=37, max_depth=24, criterion="entropy", random_state=1),
                  "stumps": dict(n_estimators=33, max_depth=1, random_state=0), "one_tree": dict(n_estimators=1, max_depth=6, random_state=0),
                  "trees33": dict(n_estimators=33, max_depth=3, random_state=0)}[which]
        pipe = rp.fit_reference_pipeline(curated.iloc[:6000], params)
    m = _model(pipe)
    try:
        X = pd.concat([curated[rp.FEATURES].iloc[7000:7020], adversarial.iloc[:12]], ignore_index=True)
        feats = ["credit_limit", "repayment_status_1", "education"]
        out = m.partial_dependence(X, feats, kind="both", grid_frame=curated)
        _sk_agree(pipe, X, out, rp.CATEGORICAL_FEATURES)
        _expanded_tile(pipe, X, out)
    finally:
        m.close()


@pytest.mark.parametrize("name", ["packed_wide", "packed_wide_gbdt", "tiny", "tiny_gbdt", "over16"])
def test_schema_zoo(name):
    from databricks_kubernetes_mlops_poc_b200.model import B200Model

    spec, pipe = sz.fitted(name)
    X = pd.concat([sz.edge_rows(spec, pipe, n=40), sz.make_frame(spec, 40, seed=9, target=False)], ignore_index=True)
    grid_frame = sz.make_frame(spec, 2000, seed=3, target=False)
    cats = sz.cat_names(spec)
    m = B200Model.from_pipeline(pipe)
    try:
        out = m.partial_dependence(X, sz.features(spec), kind="both", grid_frame=grid_frame, grid_resolution=17)
        _sk_agree(pipe, X, out, cats, rows=20)
        _expanded_tile(pipe, X, out)
    finally:
        m.close()


def test_grid_edges(rf100d6, curated):
    from oracle import reference_pipeline as rp
    from oracle import treewalk as tw

    m = _model(rf100d6)
    try:
        X = curated[rp.FEATURES].iloc[:64].reset_index(drop=True)
        dump = tw.dump_pipeline(rf100d6)
        n_ohe = int(dump["cat_offsets"][-1])
        f = rp.NUMERIC_FEATURES.index("credit_limit")
        thr = np.unique(dump["threshold"][(dump["left"] != -1) & (dump["feature"] == n_ohe + f)])[:40]
        t32 = thr.astype(np.float32)
        pts = np.concatenate([t32, np.nextafter(t32, np.float32(np.inf)), np.nextafter(t32, np.float32(-np.inf)), thr]).astype(np.float64)
        pts = [float(v) for v in pts[:150]] + [np.nan, None, 0.0, -0.0, pts[3], pts[3]]
        out = m.partial_dependence(X, ["credit_limit"], kind="both", custom_values={"credit_limit": pts})
        assert out["grid_values"][0] == pts  # the caller's order, duplicates kept
        ind = out["individual"][0]
        assert np.array_equal(ind[:, -1], ind[:, -2])
        from databricks_kubernetes_mlops_poc_b200.flatten import parse_header

        median = float(parse_header(m.flat.blob)["impute"][len(rp.CATEGORICAL_FEATURES) + f])
        med = m.partial_dependence(X, ["credit_limit"], kind="both", custom_values={"credit_limit": [median]})
        assert np.array_equal(ind[:, 150], med["individual"][0][:, 0]) and np.array_equal(ind[:, 151], ind[:, 150])  # NaN, None: the median
        _sk_agree(rf100d6, X, {**out, "grid_values": [[v for v in pts if v is not None and v == v]],
                               "individual": [np.delete(ind, [150, 151], axis=1)], "feature_names": ["credit_limit"]},
                  rp.CATEGORICAL_FEATURES, rows=64)
        assert _expanded_tile(rf100d6, X, out)
        cat = "education"
        vals = ["never_seen", None, np.nan, "missing"] + sorted(X[cat].unique().tolist(), reverse=True)
        out = m.partial_dependence(X, [cat, cat], kind="both", custom_values={cat: vals})
        assert np.array_equal(out["individual"][0], out["individual"][1])  # duplicate names: independent, identical probes
        assert _expanded_tile(rf100d6, X, out)
        for g in (1, 64, 65, 256):
            grid = np.linspace(1e4, 8e5, g).tolist()
            out = m.partial_dependence(X, ["credit_limit"], kind="both", custom_values={"credit_limit": grid})
            assert out["individual"][0].shape == (64, g)
            _sk_agree(rf100d6, X, out, rp.CATEGORICAL_FEATURES, rows=10 if g > 64 else None)
        proba = m.predict_proba1(X)
        own = m.partial_dependence(X.iloc[:1], rp.FEATURES, kind="individual", custom_values={f: [X[f].iloc[0]] for f in rp.FEATURES})
        assert all(abs(v[0, 0] - proba[0]) <= TOL for v in own["individual"])  # the row's own value: its prediction
    finally:
        m.close()


def test_unused_field_is_flat(curated):
    from oracle import reference_pipeline as rp

    pipe = rp.fit_reference_pipeline(curated.iloc[:3000], dict(n_estimators=5, max_depth=2, random_state=0))
    from oracle import treewalk as tw

    dump = tw.dump_pipeline(pipe)
    n_ohe = int(dump["cat_offsets"][-1])
    used = {rp.NUMERIC_FEATURES[int(v) - n_ohe] for v in dump["feature"][dump["left"] != -1] if v >= n_ohe}
    unused = [f for f in rp.NUMERIC_FEATURES if f not in used][0]
    m = _model(pipe)
    try:
        X = curated[rp.FEATURES].iloc[:100]
        out = m.partial_dependence(X, [unused], kind="individual")
        proba = m.predict_proba1(X)
        ind = out["individual"][0]
        assert (ind == ind[:, :1]).all() and np.abs(ind[:, 0] - proba).max() <= TOL
    finally:
        m.close()


def test_batches_formats_device_and_determinism(rf100d6, curated):
    from databricks_kubernetes_mlops_poc_b200 import dependence
    from databricks_kubernetes_mlops_poc_b200._cabi import ROWS_PACKED64, ROWS_WORDS24
    from oracle import reference_pipeline as rp

    m = _model(rf100d6)
    eng, enc = m.engine, m.encoder
    try:
        cur = curated[rp.FEATURES]
        feats = ["credit_limit", "repayment_status_1", "age"]
        words, probes, off = [], [], 0
        for f in feats:
            g = dependence.grid_from_column(cur[f], f in rp.CATEGORICAL_FEATURES)
            words.append(dependence.encode_grid(enc, f, g))
            probes.append((dependence.word_of(enc, f), off, len(g)))
            off += len(g)
        grid = np.concatenate(words)
        rows = enc.encode_frame(cur.iloc[:2048])
        big = np.concatenate([rows] * 32)  # 65 536 rows
        ref = eng.partial_dependence_rows(big, probes, grid)
        assert ref.shape == (65536, off)
        assert np.array_equal(ref, eng.partial_dependence_rows(big, probes, grid))  # run to run
        assert np.array_equal(ref[:2048], ref[2048:4096])
        chunk = 16384
        for n in (0, 1, 31, 32, 33, chunk - 1, chunk + 1, 3 * chunk + 7):
            got = eng.partial_dependence_rows(big[:n], probes, grid)
            assert got.shape == (n, off) and np.array_equal(got, ref[:n])
        assert np.array_equal(eng.partial_dependence_rows(enc.pack_rows(big), probes, grid), ref)
        # all 23 fields, 256 points each: the fixed chunk is below 16 384 rows
        wide = [(w, 0, 256) for w in range(23)]
        gw = np.zeros(256 * 23, dtype=np.uint32)
        gw.view(np.float32)[:] = np.linspace(-5, 5e5, 256 * 23)
        gw[:256] = np.arange(256) % 2  # word 0 is categorical: codes 0/1
        wide = [(0, 0, 256)] + [(w, 256 * w, 256) for w in range(9, 23)]
        wide_ref = eng.partial_dependence_rows(big[:20000], wide, gw)
        assert np.array_equal(wide_ref[:1500], eng.partial_dependence_rows(big[:1500], wide, gw))
        for fmt, r in ((ROWS_WORDS24, big[:5000]), (ROWS_PACKED64, enc.pack_rows(big[:5000]))):
            r = np.ascontiguousarray(r)
            d_rows, d_out = eng.device_alloc(r.nbytes), eng.device_alloc(5000 * off * 8)
            try:
                eng.h2d(d_rows, r)
                eng.partial_dependence_device(d_rows, 5000, probes, grid, d_out, fmt)
                eng.sync()
                got = np.empty((5000, off), dtype=np.float64)
                eng.d2h(got, d_out)
            finally:
                eng.device_free(d_rows)
                eng.device_free(d_out)
            assert np.array_equal(got, ref[:5000])
        # interleaved with predict and explain-free scoring: unchanged
        p_before, _ = eng.predict_rows(rows, np.float64)
        assert np.array_equal(eng.partial_dependence_rows(rows, probes, grid), ref[:2048])
        assert np.array_equal(eng.predict_rows(rows, np.float64)[0], p_before)
    finally:
        m.close()


def test_errors(rf100d6, curated):
    from databricks_kubernetes_mlops_poc_b200._cabi import B2FError
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer, flatten_pipeline
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from oracle import reference_pipeline as rp

    flat = flatten_pipeline(rf100d6)
    eng, enc = ForestEngine(flat, 0), RowEncoder(flat)
    try:
        rows = enc.encode_frame(curated[rp.FEATURES].iloc[:100])
        g = np.zeros(8, dtype=np.uint32)
        g.view(np.float32)[:] = np.linspace(1e4, 5e5, 8)
        good = [(9, 0, 8)]
        want = eng.partial_dependence_rows(rows, good, g)
        bad = [
            ([(23, 0, 8)], g, -1), ([(-1, 0, 8)], g, -1), ([(9, 0, 0)], g, -1), ([(9, 0, 257)], np.zeros(300, np.uint32), -1),
            ([(9, -1, 8)], g, -1), ([(9, 23 * 256 - 7, 8)], g, -1), ([(9, 0, 8)] * 24, g, -1), ([], g, -1),
            ([(0, 0, 2)], np.array([5, 99], dtype=np.uint32), -1), ([(0, 0, 1)], np.array([0xFFFFFFFE], dtype=np.uint32), -1),
            ([(9, 0, 1)], np.array([0x7F800000], dtype=np.uint32), -7),
        ]
        for probes, grid, rc in bad:
            with pytest.raises(B2FError, match=rf"rc={rc}\)"):
                eng.partial_dependence_rows(rows, probes, grid)
            assert np.array_equal(eng.partial_dependence_rows(rows, good, g), want)  # the handle keeps working
        if eng.rank_words:
            with pytest.raises(B2FError, match=r"rc=-1\).*ranked"):
                eng.partial_dependence_rows(enc.rank_rows(rows), good, g)
        # an explainer attached or not changes nothing; explain calls interleave
        eng.attach_explainer(flatten_explainer(rf100d6, flat))
        phi, _ = eng.explain_rows(rows)
        assert np.array_equal(eng.partial_dependence_rows(rows, good, g), want)
        assert np.array_equal(eng.explain_rows(rows)[0], phi)
    finally:
        eng.close()


def test_model_dir_and_http(tmp_path, rf100d6, curated):
    import httpx

    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer, flatten_pipeline
    from databricks_kubernetes_mlops_poc_b200.model import B200Model, load_model, save_model_dir
    from databricks_kubernetes_mlops_poc_b200.server import create_app
    from oracle import reference_pipeline as rp

    bg = curated[rp.FEATURES].iloc[:3000]
    df = curated[rp.FEATURES].iloc[5000:5040].reset_index(drop=True)
    flat = flatten_pipeline(rf100d6)
    save_model_dir(str(tmp_path / "bg"), flat, explain_blob=flatten_explainer(rf100d6, flat), explain_background=bg)
    save_model_dir(str(tmp_path / "plain"), flat)
    with_bg, plain = load_model(str(tmp_path / "bg")), load_model(str(tmp_path / "plain"))
    try:
        assert with_bg.background_attached and with_bg.dependence_grids is not None and plain.dependence_grids is None
        direct = B200Model.from_pipeline(rf100d6)
        try:
            want = direct.partial_dependence(df, ["credit_limit", "sex"], kind="both", grid_frame=bg)
        finally:
            direct.close()
        got = with_bg.partial_dependence(df, ["credit_limit", "sex"], kind="both", grid_frame=bg)
        assert all(np.array_equal(a, b) for a, b in zip(got["individual"], want["individual"]))
        assert [list(g) for g in want["grid_values"]] == [list(with_bg.dependence_grids[f]) for f in ("credit_limit", "sex")]
        body = df.to_dict(orient="records")

        async def main(model, queries):
            app = create_app(model=model)
            async with app.router.lifespan_context(app):
                async with httpx.AsyncClient(transport=httpx.ASGITransport(app=app), base_url="http://t") as c:
                    preds = [c.post("/predict", json=body) for _ in range(8)]
                    deps = [c.post("/explain/dependence", params=q, json=body) for q in queries]
                    return await asyncio.gather(*deps, *preds)

        queries = [[("feature", "credit_limit"), ("feature", "sex"), ("kind", "both")],
                   [("feature", "age"), ("value", "30"), ("value", "20"), ("value", ""), ("kind", "individual")],
                   [("feature", "nope")], [("feature", "age"), ("kind", "x")], [("feature", "age"), ("grid_resolution", "1")],
                   [("feature", "age"), ("grid_resolution", "300")], [("feature", "age"), ("feature", "sex"), ("value", "1")]]
        res = asyncio.run(main(with_bg, queries))
        j = res[0].json()
        assert res[0].status_code == 200 and j["feature_names"] == ["credit_limit", "sex"]
        assert np.abs(np.asarray(j["individual"][0]) - want["individual"][0]).max() == 0.0
        assert np.abs(np.asarray(j["average"][1]) - want["average"][1]).max() == 0.0
        j = res[1].json()
        assert j["grid_values"] == [[30.0, 20.0, None]] and "average" not in j
        explicit = plain.partial_dependence(df, ["age"], kind="individual", custom_values={"age": [30.0, 20.0, None]})
        assert np.array_equal(np.asarray(j["individual"][0]), explicit["individual"][0])
        assert [r.status_code for r in res[2:7]] == [422] * 5
        assert all(r.status_code == 200 for r in res[7:])
        res = asyncio.run(main(plain, [[("feature", "credit_limit"), ("kind", "both")]]))
        from_rows = plain.partial_dependence(df, ["credit_limit"], kind="both")
        assert res[0].json()["grid_values"][0] == from_rows["grid_values"][0]
    finally:
        with_bg.close()
        plain.close()
