"""k_ale on the GPU: accumulated local effects against the brute-force oracle on ``predict_proba`` to 1e-12 with exact bin
counts (reference, bench, deep and tiny forests, the schema-zoo schemas and a schema of 18 numerics); every bin sum
replayed bit for bit from tile-kernel scores of the substituted rows in the documented order; edge cases; batch edges,
both row formats, the device entry point and determinism; the C-ABI errors; load_model and POST /explain/ale under
concurrent /predict."""

import asyncio
import os

import numpy as np
import pandas as pd
import pytest

import schema_zoo as sz
from ale_walk import brute_ale, ordered_sums, row_bins

pytestmark = pytest.mark.gpu

TOL = 1e-12


def _model(pipe):
    from databricks_kubernetes_mlops_poc_b200.model import B200Model

    return B200Model.from_pipeline(pipe)


def _oracle_agree(pipe, m, X, out):
    """``out`` of accumulated_local_effects against brute_ale field by field."""
    from databricks_kubernetes_mlops_poc_b200 import dependence

    rows = m.encoder.encode_frame(X)
    for i, f in enumerate(out["feature_names"]):
        z = np.asarray(out["feature_values"][i], dtype=np.float32)
        if len(z) < 2:
            assert out["ale_values"][i].tolist() == [0.0]
            continue
        want = brute_ale(pipe, X, f, z, rows[:, dependence.word_of(m.encoder, f)].view(np.float32))
        assert np.array_equal(out["bin_rows"][i], want["bin_rows"]), f
        assert np.abs(out["ale_values"][i] - want["ale_values"]).max() <= TOL, f


def _tile_engine(flat):
    from databricks_kubernetes_mlops_poc_b200._cabi import B2FError
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine

    os.environ["B2F_KERNEL"] = "tile"
    try:
        return ForestEngine(flat, 0)
    except B2FError as e:
        assert "tile kernel" in str(e)
        return None
    finally:
        del os.environ["B2F_KERNEL"]


def _replay(tile, rows, probes, edges):
    """Every substituted row scored by the tile kernel, the deltas added in the documented order -> (sums, counts)."""
    sums, counts = [], []
    for word, off, K in probes:
        z = np.asarray(edges[off:off + K + 1], dtype=np.float32)
        b, present = row_bins(rows, word, z)
        lo, hi = rows.copy(), rows.copy()
        lo[:, word] = z.view(np.uint32)[b]
        hi[:, word] = z.view(np.uint32)[b + 1]
        p_lo, _ = tile.predict_rows(lo, np.float64)
        p_hi, _ = tile.predict_rows(hi, np.float64)
        s, c = ordered_sums(p_hi - p_lo, b, present, K)
        sums.append(s), counts.append(c)
    return np.concatenate(sums), np.concatenate(counts)


def _plan(m, X, features, bins=20, min_bin_points=4):
    from databricks_kubernetes_mlops_poc_b200 import ale, dependence

    edges = [ale.default_edges(ale.present_float32(m.encoder, f, X[f]), bins, min_bin_points) for f in features]
    return ale.probe_plan([dependence.word_of(m.encoder, f) for f in features], edges)


def test_rf100d6_all_numerics(rf100d6, curated):
    from oracle import reference_pipeline as rp

    m = _model(rf100d6)
    try:
        X = curated[rp.FEATURES].iloc[:6000].reset_index(drop=True)
        out = m.accumulated_local_effects(X)
        assert out["feature_names"] == rp.NUMERIC_FEATURES and out["output"] == "probability" and out["rows"] == 6000
        _oracle_agree(rf100d6, m, X, out)
        assert abs(out["constant_value"] - rf100d6.predict_proba(X)[:, 1].mean()) <= TOL
        for i in range(len(rp.NUMERIC_FEATURES)):
            n, A = out["bin_rows"][i], out["ale_values"][i]
            assert n.sum() == 6000 and len(A) == len(out["feature_values"][i]) and abs(np.sum(n * (A[:-1] + A[1:]) / 2)) <= 1e-12
        # bit-exact replay from the tile kernel's scores of every substituted row
        tile = _tile_engine(m.flat)
        assert tile is not None
        try:
            rows = m.encoder.encode_frame(X.iloc[:3000])
            probes, edges, _ = _plan(m, X, rp.NUMERIC_FEATURES)
            sums, counts = m.engine.ale_rows(rows, probes, edges)
            want_s, want_c = _replay(tile, rows, probes, edges)
            assert np.array_equal(counts, want_c) and np.array_equal(sums, want_s)
        finally:
            tile.close()
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
        X = pd.concat([curated[rp.FEATURES].iloc[6000:8000], adversarial.iloc[:200]], ignore_index=True)
        out = m.accumulated_local_effects(X, bins=12)
        _oracle_agree(pipe, m, X, out)
        tile = _tile_engine(m.flat)
        if tile is not None:
            try:
                rows = m.encoder.encode_frame(X)
                probes, edges, _ = _plan(m, X, rp.NUMERIC_FEATURES, bins=12)
                got = m.engine.ale_rows(rows, probes, edges)
                want = _replay(tile, rows, probes, edges)
                assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
            finally:
                tile.close()
    finally:
        m.close()


def test_edge_cases(rf100d6, curated, adversarial):
    from databricks_kubernetes_mlops_poc_b200 import dependence
    from oracle import reference_pipeline as rp
    from oracle import treewalk as tw

    m = _model(rf100d6)
    try:
        X = pd.concat([adversarial, curated[rp.FEATURES].iloc[:300]], ignore_index=True)  # NaN, +-0, +-3e38, 1e-45, thresholds
        out = m.accumulated_local_effects(X)
        _oracle_agree(rf100d6, m, X, out)
        rows = m.encoder.encode_frame(X)
        for i, f in enumerate(out["feature_names"]):  # NaN rows take no part
            assert out["bin_rows"][i].sum() == int((~np.isnan(rows[:, dependence.word_of(m.encoder, f)].view(np.float32))).sum())
        # values on the edges and one ulp either side; custom edges leave rows outside [z_0, z_K]
        dump = tw.dump_pipeline(rf100d6)
        n_ohe = int(dump["cat_offsets"][-1])
        k = rp.NUMERIC_FEATURES.index("credit_limit")
        thr = np.unique(dump["threshold"][(dump["left"] != -1) & (dump["feature"] == n_ohe + k)]).astype(np.float32)
        z = np.unique(thr[:: max(1, len(thr) // 30)])[1:-1]
        Y = curated[rp.FEATURES].iloc[:len(z) * 4].reset_index(drop=True).copy()
        vals = np.concatenate([z, np.nextafter(z, np.float32(np.inf)), np.nextafter(z, np.float32(-np.inf)), z])
        vals[-4:] = [-3.0e38, 3.0e38, 0.0, -0.0]
        Y["credit_limit"] = vals.astype(np.float64)
        out = m.accumulated_local_effects(Y, ["credit_limit", "age"], custom_edges={"credit_limit": z.tolist()})
        assert np.array_equal(out["feature_values"][0], z.astype(np.float64)) and out["bin_rows"][0].sum() == len(Y)
        _oracle_agree(rf100d6, m, Y, out)
        with pytest.raises(ValueError, match="no present value"):
            m.accumulated_local_effects(Y.assign(age=np.nan), ["age"])
        one = m.accumulated_local_effects(Y.assign(age=33.0), ["age", "credit_limit"])
        assert one["ale_values"][0].tolist() == [0.0] and one["feature_values"][0].tolist() == [33.0]
        for bad in (dict(features=["education"]), dict(features=["age", "age"]), dict(features=["nope"]), dict(bins=0), dict(bins=257),
                    dict(min_bin_points=0), dict(features=["age"], custom_edges={"age": [1.0]}),
                    dict(features=["age"], custom_edges={"age": [2.0, 1.0]}), dict(features=["age"], custom_edges={"credit_limit": [1, 2]})):
            with pytest.raises(ValueError):
                m.accumulated_local_effects(Y, **bad)
        with pytest.raises(ValueError):
            m.accumulated_local_effects(Y.iloc[:0])
    finally:
        m.close()


def test_unused_field_is_zero(curated):
    from oracle import reference_pipeline as rp
    from oracle import treewalk as tw

    pipe = rp.fit_reference_pipeline(curated.iloc[:3000], dict(n_estimators=5, max_depth=2, random_state=0))
    dump = tw.dump_pipeline(pipe)
    n_ohe = int(dump["cat_offsets"][-1])
    used = {rp.NUMERIC_FEATURES[int(v) - n_ohe] for v in dump["feature"][dump["left"] != -1] if v >= n_ohe}
    unused = [f for f in rp.NUMERIC_FEATURES if f not in used][0]
    m = _model(pipe)
    try:
        out = m.accumulated_local_effects(curated[rp.FEATURES].iloc[:500], [unused])
        assert (out["ale_values"][0] == 0.0).all() and (out["bin_effects"][0] == 0.0).all() and out["ale0"][0] == 0.0
    finally:
        m.close()


@pytest.mark.parametrize("name", ["packed_wide", "packed_wide_gbdt", "tiny", "tiny_gbdt", "over16", "num18"])
def test_schema_zoo(name):
    if name == "num18":  # 18 numerics: a row's fields span two walk segments
        spec = ([3], 18)
        pipe = sz.fit_pipeline(spec, sz.make_frame(spec, 4000, seed=0), "rf", n_estimators=30, max_depth=7, random_state=0)
    else:
        spec, pipe = sz.fitted(name)
    X = pd.concat([sz.edge_rows(spec, pipe, n=300), sz.make_frame(spec, 1200, seed=9, target=False)], ignore_index=True)
    m = _model(pipe)
    try:
        out = m.accumulated_local_effects(X)
        assert out["feature_names"] == sz.num_names(spec)
        _oracle_agree(pipe, m, X, out)
        tile = _tile_engine(m.flat)
        if tile is not None:
            try:
                rows = m.encoder.encode_frame(X)
                probes, edges, _ = _plan(m, X, sz.num_names(spec))
                got = m.engine.ale_rows(rows, probes, edges)
                want = _replay(tile, rows, probes, edges)
                assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
            finally:
                tile.close()
    finally:
        m.close()


def test_batches_formats_device_and_determinism(rf100d6, curated):
    from oracle import reference_pipeline as rp

    m = _model(rf100d6)
    eng, enc = m.engine, m.encoder
    tile = _tile_engine(m.flat)
    try:
        cur = curated[rp.FEATURES]
        probes, edges, _ = _plan(m, cur, rp.NUMERIC_FEATURES)
        rows = enc.encode_frame(cur)
        big = np.concatenate([rows, rows, rows])[:65537]
        for n in (1, 127, 128, 129, 65537):
            got = eng.ale_rows(big[:n], probes, edges)
            want = _replay(tile, big[:n], probes, edges)
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), n
            again = eng.ale_rows(big[:n], probes, edges)
            assert np.array_equal(again[0], got[0]) and np.array_equal(again[1], got[1])  # run to run
            packed = eng.ale_rows(enc.pack_rows(big[:n]), probes, edges)
            assert np.array_equal(packed[0], got[0]) and np.array_equal(packed[1], got[1])
        ref_s, ref_c = eng.ale_rows(big, probes, edges)
        # a field's result does not depend on the other fields of the call
        off = 0
        for word, eoff, K in probes:
            s, c = eng.ale_rows(big, [(word, 0, K)], edges[eoff:eoff + K + 1])
            assert np.array_equal(s, ref_s[off:off + K]) and np.array_equal(c, ref_c[off:off + K])
            off += K
        s, c = eng.ale_rows(big, probes[::-1], edges)  # the output follows the probe order
        K = [p[2] for p in probes]
        assert np.array_equal(s[len(s) - K[0]:], ref_s[:K[0]]) and np.array_equal(s[:K[-1]], ref_s[len(ref_s) - K[-1]:])
        # the device form equals the host form, in both formats
        for r in (big, enc.pack_rows(big)):
            r = np.ascontiguousarray(r)
            fmt = 0 if r.shape[1] == 24 else 1
            K = len(ref_s)
            d_rows, d_s, d_c = eng.device_alloc(r.nbytes), eng.device_alloc(K * 8), eng.device_alloc(K * 8)
            try:
                eng.h2d(d_rows, r)
                eng.ale_device(d_rows, len(r), probes, edges, d_s, d_c, fmt)
                eng.sync()
                s, c = np.empty(K), np.empty(K, dtype=np.int64)
                eng.d2h(s, d_s)
                eng.d2h(c, d_c)
            finally:
                for d in (d_rows, d_s, d_c):
                    eng.device_free(d)
            assert np.array_equal(s, ref_s) and np.array_equal(c, ref_c)
        p_before, _ = eng.predict_rows(rows, np.float64)
        assert np.array_equal(eng.ale_rows(big, probes, edges)[0], ref_s)
        assert np.array_equal(eng.predict_rows(rows, np.float64)[0], p_before)
    finally:
        tile.close()
        m.close()


def test_errors(rf100d6, curated):
    from databricks_kubernetes_mlops_poc_b200._cabi import B2FError
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline, parse_header
    from oracle import reference_pipeline as rp

    flat = flatten_pipeline(rf100d6)
    eng, enc = ForestEngine(flat, 0), RowEncoder(flat)
    try:
        rows = enc.encode_frame(curated[rp.FEATURES].iloc[:300])
        z = np.linspace(1e4, 5e5, 9).astype(np.float32)
        good = [(9, 0, 8)]
        want = eng.ale_rows(rows, good, z)
        big = np.linspace(0, 1e5, 300).astype(np.float32)
        bad = [
            ([(0, 0, 8)], z, -1), ([(8, 0, 8)], z, -1), ([(23, 0, 8)], z, -1), ([(9, 0, 8), (9, 0, 8)], z, -1), ([(9, 0, 0)], z, -1),
            ([(9, 0, 257)], np.concatenate([big, big]), -1), ([(9, -1, 8)], z, -1), ([(9, 23 * 257 - 8, 8)], z, -1),
            ([(9, 0, 8)] * 15, z, -1), ([], z, -1), ([(9, 0, 8)], z[::-1].copy(), -1), ([(9, 0, 2)], np.array([1, 1, 2], np.float32), -1),
            ([(9, 0, 2)], np.array([1, np.inf, 2], np.float32), -7), ([(9, 0, 1)], np.array([np.nan, 2], np.float32), -7),
        ]
        for probes, edges, rc in bad:
            with pytest.raises(B2FError, match=rf"rc={rc}\)"):
                eng.ale_rows(rows, probes, edges)
            got = eng.ale_rows(rows, good, z)  # the handle keeps working
            assert np.array_equal(got[0], want[0])
        with pytest.raises(B2FError, match=r"rc=-1\)"):
            eng.ale_rows(rows[:0], good, z)
        if eng.rank_words:
            with pytest.raises(B2FError, match=r"rc=-1\).*ranked"):
                eng.ale_rows(enc.rank_rows(rows), good, z)
        lib, pr = eng._lib, np.array([(9, 0, 8)], dtype=np.dtype([("w", np.int32), ("o", np.int32), ("b", np.int32)]))
        from databricks_kubernetes_mlops_poc_b200._cabi import ptr

        out_s, out_c = np.empty(8), np.empty(8, np.int64)
        assert lib.b2f_ale(eng.handle, None, 300, 0, ptr(pr), 1, ptr(z), ptr(out_s), ptr(out_c), None) == -1
        assert lib.b2f_ale(eng.handle, ptr(rows), 300, 0, None, 1, ptr(z), ptr(out_s), ptr(out_c), None) == -1
        assert lib.b2f_ale(eng.handle, ptr(rows), 300, 0, ptr(pr), 1, None, ptr(out_s), ptr(out_c), None) == -1
        assert lib.b2f_ale(eng.handle, ptr(rows), 300, 0, ptr(pr), 1, ptr(z), None, ptr(out_c), None) == -1
        assert lib.b2f_ale_device(eng.handle, None, 300, 0, ptr(pr), 1, ptr(z), None, None) == -1
    finally:
        eng.close()
    # a forest deeper than the walk stack
    pipe = rp.fit_reference_pipeline(curated.iloc[:8000], dict(n_estimators=3, max_depth=None, min_samples_leaf=1, random_state=0))
    flat = flatten_pipeline(pipe)
    if parse_header(flat.blob)["max_depth"] <= 32:
        pytest.skip("this forest fits the walk stack")
    eng = ForestEngine(flat, 0)
    try:
        with pytest.raises(B2FError, match=r"rc=-1\).*depth"):
            eng.ale_rows(RowEncoder(flat).encode_frame(curated[rp.FEATURES].iloc[:10]), [(9, 0, 8)], np.linspace(1e4, 5e5, 9).astype(np.float32))
    finally:
        eng.close()


def test_model_dir_and_http(tmp_path, rf100d6, curated):
    import httpx

    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline
    from databricks_kubernetes_mlops_poc_b200.model import load_model, save_model_dir
    from databricks_kubernetes_mlops_poc_b200.server import create_app
    from oracle import reference_pipeline as rp

    df = curated[rp.FEATURES].iloc[5000:5400].reset_index(drop=True)
    save_model_dir(str(tmp_path / "plain"), flatten_pipeline(rf100d6))
    m = load_model(str(tmp_path / "plain"))
    try:
        want = m.accumulated_local_effects(df)
        body = df.to_dict(orient="records")

        async def main(queries):
            app = create_app(model=m)
            async with app.router.lifespan_context(app):
                async with httpx.AsyncClient(transport=httpx.ASGITransport(app=app), base_url="http://t") as c:
                    preds = [c.post("/predict", json=body) for _ in range(8)]
                    ales = [c.post("/explain/ale", params=q, json=body) for q in queries]
                    return await asyncio.gather(*ales, *preds)

        queries = [[], [("feature", "age"), ("value", "20"), ("value", "35"), ("value", "80"), ("bins", "3")],
                   [("feature", "education")], [("bins", "0")], [("feature", "age"), ("value", "3"), ("value", "1")]]
        res = asyncio.run(main(queries))
        j = res[0].json()
        assert res[0].status_code == 200 and j["feature_names"] == rp.NUMERIC_FEATURES
        for i in range(len(rp.NUMERIC_FEATURES)):
            assert j["ale_values"][i] == want["ale_values"][i].tolist() and j["bin_rows"][i] == want["bin_rows"][i].tolist()
        assert j["constant_value"] == want["constant_value"]
        explicit = m.accumulated_local_effects(df, ["age"], custom_edges={"age": [20, 35, 80]})
        assert res[1].status_code == 200 and res[1].json()["ale_values"][0] == explicit["ale_values"][0].tolist()
        assert [r.status_code for r in res[2:5]] == [422] * 3
        assert all(r.status_code == 200 for r in res[5:])
    finally:
        m.close()


def test_beside_models_of_other_shapes(rf100d6, curated):
    """K12 on one model between calls on models of other schemas in the same process: unchanged results."""
    from oracle import reference_pipeline as rp

    m = _model(rf100d6)
    others = []
    try:
        X = curated[rp.FEATURES].iloc[:2000].reset_index(drop=True)
        ref = m.accumulated_local_effects(X)
        for name in ("tiny", "packed_wide", "over16"):
            spec, pipe = sz.fitted(name)
            o = _model(pipe)
            others.append(o)
            Y = sz.make_frame(spec, 700, seed=4, target=False)
            got = o.accumulated_local_effects(Y)
            _oracle_agree(pipe, o, Y, got)
            again = m.accumulated_local_effects(X)
            assert all(np.array_equal(a, b) for a, b in zip(again["ale_values"], ref["ale_values"]))
    finally:
        for o in others:
            o.close()
        m.close()
