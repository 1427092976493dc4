"""k_pair_dependence on the GPU: scikit-learn's two-way ``partial_dependence(method="brute")`` to 1e-12 on the reference
forests, a GBDT, a deep forest and the schema-zoo schemas; bit-identity with the tile kernel scoring the expanded rows;
the device mean against numpy's; Friedman's H^2 against a brute oracle on ``predict_proba``, and ~0 where the model is
additive; determinism, row formats, the device form and grouping; the C-ABI errors; both HTTP routes under /predict."""

import asyncio
import itertools
import os

import numpy as np
import pandas as pd
import pytest
from sklearn.inspection import partial_dependence

import schema_zoo as sz

pytestmark = pytest.mark.gpu

TOL = 1e-12
PAIRS = [("credit_limit", "age"), ("education", "credit_limit"), ("repayment_status_1", "education")]


def _model(pipe):
    from databricks_kubernetes_mlops_poc_b200.model import B200Model

    return B200Model.from_pipeline(pipe)


def _small_grids(X, pairs, categorical, g=10):
    """custom_values of about g points per axis: a categorical field's values present in X, a numeric field's quantiles."""
    cv = {}
    for f in {f for p in pairs for f in p}:
        if f in categorical:
            cv[f] = sorted(v for v in X[f].unique().tolist() if isinstance(v, str))[:g]
        else:
            cv[f] = np.unique(np.nanquantile(X[f].to_numpy(dtype=np.float64), np.linspace(0.02, 0.98, g))).tolist()
    return cv


def _check(pipe, m, X, pairs, categorical, tile=True):
    """B200Model.pair_dependence(kind="both") against sklearn (1e-12), the tile kernel (bits) and numpy's mean (1e-12)."""
    cv = _small_grids(X, pairs, categorical)
    out = m.pair_dependence(X, pairs, kind="both", custom_values=cv)
    assert out["feature_names"] == [tuple(p) for p in pairs] and out["output"] == "probability"
    for k, (a, b) in enumerate(pairs):
        want = partial_dependence(pipe, X, [a, b], method="brute", kind="both", categorical_features=categorical,
                                  custom_values={f: np.asarray(cv[f], dtype=object if f in categorical else np.float64) for f in (a, b)})
        assert [list(g) for g in want["grid_values"]] == [list(g) for g in out["grid_values"][k]]
        ind, avg = out["individual"][k], out["average"][k]
        assert ind.shape == want["individual"][0].shape and avg.shape == want["average"][0].shape
        assert np.abs(ind - want["individual"][0]).max() <= TOL, (a, b)
        assert np.abs(avg - want["average"][0]).max() <= TOL, (a, b)
        assert np.abs(avg - ind.mean(axis=0)).max() <= TOL, (a, b)
    if tile:
        _expanded_tile(pipe, X, out)
    return out


def _expanded_tile(pipe, X, out):
    """Every curve point scored by a B2F_KERNEL=tile engine on the rows with both fields replaced: bit-identical.  False
    when the forest does not fit the tile kernel."""
    from databricks_kubernetes_mlops_poc_b200 import dependence, interaction
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
        for k, (a, b) in enumerate(out["feature_names"]):
            ga, gb = out["grid_values"][k]
            pts = interaction.cartesian(dependence.encode_grid(enc, a, ga), dependence.encode_grid(enc, b, gb))
            big = np.repeat(rows, len(pts), axis=0)
            big[:, dependence.word_of(enc, a)] = np.tile(pts[:, 0], len(rows))
            big[:, dependence.word_of(enc, b)] = np.tile(pts[:, 1], len(rows))
            p, _ = tile.predict_rows(big, np.float64)
            assert np.array_equal(p.reshape(out["individual"][k].shape), out["individual"][k]), (a, b)
        return True
    finally:
        tile.close()


def test_rf100d6_three_pair_types(rf100d6, curated, adversarial):
    from oracle import reference_pipeline as rp

    m = _model(rf100d6)
    try:
        X = curated[rp.FEATURES].iloc[:40].reset_index(drop=True)
        assert _check(rf100d6, m, X, PAIRS, rp.CATEGORICAL_FEATURES)
        # default grids (sklearn's rule), and edge rows (NaN, unknown categories, threshold values)
        out = m.pair_dependence(X, PAIRS[:1], kind="both", grid_resolution=7)
        want = partial_dependence(rf100d6, X, list(PAIRS[0]), method="brute", kind="both", categorical_features=rp.CATEGORICAL_FEATURES,
                                  grid_resolution=7)
        assert [list(g) for g in want["grid_values"]] == out["grid_values"][0]
        assert np.abs(out["individual"][0] - want["individual"][0]).max() <= TOL
        E = adversarial.iloc[:40].reset_index(drop=True)
        out = m.pair_dependence(E, PAIRS, kind="individual", custom_values=_small_grids(X, PAIRS, rp.CATEGORICAL_FEATURES))
        _expanded_tile(rf100d6, E, out)
        avg = m.pair_dependence(E, PAIRS, kind="average", custom_values=_small_grids(X, PAIRS, rp.CATEGORICAL_FEATURES))
        assert "individual" not in avg
        for a, i in zip(avg["average"], out["individual"]):
            assert np.abs(a - i.mean(axis=0)).max() <= TOL
    finally:
        m.close()


@pytest.mark.parametrize("which", ["rf500d8", "gbdt_small", "deep24"])
def test_other_forests(which, request, curated, adversarial):
    from oracle import reference_pipeline as rp

    if which == "deep24":
        pipe = rp.fit_reference_pipeline(curated.iloc[:6000], dict(n_estimators=37, max_depth=24, criterion="entropy", random_state=1))
    else:
        pipe = request.getfixturevalue(which)
    m = _model(pipe)
    try:
        X = pd.concat([curated[rp.FEATURES].iloc[7000:7028], adversarial.iloc[:12]], ignore_index=True)
        _check(pipe, m, X, PAIRS, rp.CATEGORICAL_FEATURES)
    finally:
        m.close()


@pytest.mark.parametrize("name", ["packed_wide", "packed_wide_gbdt", "tiny", "tiny_gbdt", "over16"])
def test_schema_zoo(name):
    spec, pipe = sz.fitted(name)
    X = pd.concat([sz.edge_rows(spec, pipe, n=20), sz.make_frame(spec, 20, seed=9, target=False)], ignore_index=True)
    cats, feats = sz.cat_names(spec), sz.features(spec)
    nums = [f for f in feats if f not in cats]
    pairs = [(nums[0], nums[-1]), (cats[0], nums[0])] + ([(cats[0], cats[-1])] if len(cats) > 1 else [])
    m = _model(pipe)
    try:
        _check(pipe, m, X, pairs, cats)
    finally:
        m.close()


def _brute_h2(pipe, X, j, k):
    n = len(X)

    def F(cols):
        big = pd.concat([X] * n, ignore_index=True)  # block i: every row l with the columns of row i
        for c in cols:
            big[c] = np.repeat(X[c].to_numpy(), n)
        return pipe.predict_proba(big)[:, 1].reshape(n, n).mean(axis=1)

    c = [v - v.mean() for v in (F([j, k]), F([j]), F([k]))]
    num, den = float(np.sum((c[0] - c[1] - c[2]) ** 2)), float(np.sum(c[0] ** 2))
    return num / den, num, den


@pytest.mark.parametrize("which", ["rf100d6", "gbdt_small"])
def test_h_statistic_brute_oracle(which, request, curated):
    from oracle import reference_pipeline as rp

    pipe = request.getfixturevalue(which)
    m = _model(pipe)
    try:
        X = curated[rp.FEATURES].iloc[2000:2048].reset_index(drop=True)
        X.loc[5, "credit_limit"] = np.nan
        feats = ["credit_limit", "age", "education", "repayment_status_1", "bill_amount_1"]
        res = m.interaction_strength(X, feats)
        assert res["rows"] == 48 and res["pairs"] == list(itertools.combinations(feats, 2))
        for p, (j, k) in enumerate(res["pairs"]):
            h, num, den = _brute_h2(pipe, X, j, k)
            assert abs(res["denominator"][p] - den) <= 1e-9 * den, (j, k)
            assert abs(res["numerator"][p] - num) <= 1e-9 * num + 1e-18, (j, k)
            assert abs(res["h_squared"][p] - h) <= 1e-9 * h + 1e-15, (j, k)
            assert res["matrix"][feats.index(j), feats.index(k)] == res["h_squared"][p]
        again = m.interaction_strength(X, feats)
        assert all(np.array_equal(res[key], again[key], equal_nan=True) for key in ("h_squared", "numerator", "denominator", "matrix"))
    finally:
        m.close()


def test_h_statistic_additive(curated):
    """A field the model never reads, and a forest of stumps (additive in probability): H^2 <= 1e-20."""
    from oracle import reference_pipeline as rp
    from oracle import treewalk as tw

    pipe = rp.fit_reference_pipeline(curated.iloc[:3000], dict(n_estimators=5, max_depth=2, random_state=0))
    dump = tw.dump_pipeline(pipe)
    n_ohe = int(dump["cat_offsets"][-1])
    used = {rp.NUMERIC_FEATURES[int(v) - n_ohe] for v in dump["feature"][dump["left"] != -1] if v >= n_ohe}
    unused = [f for f in rp.NUMERIC_FEATURES if f not in used][:2]
    X = curated[rp.FEATURES].iloc[4000:4300].reset_index(drop=True)
    m = _model(pipe)
    try:
        feats = sorted(used)[:2] + unused
        res = m.interaction_strength(X, feats)
        for p, (j, k) in enumerate(res["pairs"]):
            if (j in unused) != (k in unused):
                assert res["denominator"][p] > 0 and res["h_squared"][p] <= 1e-20, (j, k, res["h_squared"][p])
    finally:
        m.close()
    stumps = rp.fit_reference_pipeline(curated.iloc[:6000], dict(n_estimators=33, max_depth=1, random_state=0))
    m = _model(stumps)
    try:
        res = m.interaction_strength(X, ["credit_limit", "age", "repayment_status_1", "education", "bill_amount_1"])
        live = res["denominator"] > 1e-12
        assert live.any() and (res["h_squared"][live] <= 1e-20).all(), res["h_squared"]
    finally:
        m.close()


def test_determinism_formats_device_and_grouping(rf100d6, curated):
    from databricks_kubernetes_mlops_poc_b200 import dependence, interaction
    from databricks_kubernetes_mlops_poc_b200._cabi import ROWS_PACKED64, ROWS_WORDS24
    from oracle import reference_pipeline as rp

    m = _model(rf100d6)
    eng, enc = m.engine, m.encoder
    try:
        cur = curated[rp.FEATURES]
        probes, pts, off = [], [], 0
        for a, b in PAIRS:
            ga = dependence.grid_from_column(cur[a], a in rp.CATEGORICAL_FEATURES, 40)
            gb = dependence.grid_from_column(cur[b], b in rp.CATEGORICAL_FEATURES, 40)
            p = interaction.cartesian(dependence.encode_grid(enc, a, ga), dependence.encode_grid(enc, b, gb))
            probes.append((dependence.word_of(enc, a), dependence.word_of(enc, b), off, len(p)))
            pts.append(p)
            off += len(p)
        probes.append((dependence.word_of(enc, "age"), -1, off, 40))  # a one-way probe
        pts.append(np.stack([pts[0][:40, 1], np.zeros(40, np.uint32)], axis=1))
        off += 40
        points = np.concatenate(pts)
        rows = enc.encode_frame(cur.iloc[:3000])
        ind = eng.pair_dependence_rows(rows, probes, points)
        assert ind.shape == (3000, off)
        assert np.array_equal(ind, eng.pair_dependence_rows(rows, probes, points))  # run to run
        mean = eng.pair_dependence_rows(rows, probes, points, mean=True)
        assert np.array_equal(mean, eng.pair_dependence_rows(rows, probes, points, mean=True))
        assert np.abs(mean - ind.mean(axis=0)).max() <= TOL
        # the one-way probe is K6's curve
        k6 = eng.partial_dependence_rows(rows, [(probes[-1][0], 0, 40)], pts[-1][:, 0].copy())
        assert np.array_equal(ind[:, off - 40:], k6)
        packed = enc.pack_rows(rows)
        assert np.array_equal(eng.pair_dependence_rows(packed, probes, points), ind)
        assert np.array_equal(eng.pair_dependence_rows(packed, probes, points, mean=True), mean)
        for n in (1, 31, 33, 129):
            assert np.array_equal(eng.pair_dependence_rows(rows[:n], probes, points), ind[:n])
        for fmt, r in ((ROWS_WORDS24, rows), (ROWS_PACKED64, packed)):
            r = np.ascontiguousarray(r)
            d_rows, d_out, d_mean = eng.device_alloc(r.nbytes), eng.device_alloc(ind.nbytes), eng.device_alloc(mean.nbytes)
            try:
                eng.h2d(d_rows, r)
                eng.pair_dependence_device(d_rows, len(r), probes, points, d_out, fmt=fmt)
                eng.pair_dependence_device(d_rows, len(r), probes, points, d_mean, mean=True, fmt=fmt)
                eng.sync()
                got, got_mean = np.empty_like(ind), np.empty_like(mean)
                eng.d2h(got, d_out)
                eng.d2h(got_mean, d_mean)
            finally:
                for d in (d_rows, d_out, d_mean):
                    eng.device_free(d)
            assert np.array_equal(got, ind) and np.array_equal(got_mean, mean)
        # a call whose per-CTA sums need several scratch groups (300 000 rows: 2 344 CTAs, 14 316 points per group) equals
        # one call per probe, and the points do not depend on their neighbours
        big = np.concatenate([rows] * 100)
        p0, p2 = probes[0], probes[2]
        gprobes = [(p0[0], p0[1], 0, 10000), (p2[0], p2[1], 10000, 6000)]
        gpoints = np.concatenate([np.resize(points[:p0[3]], (10000, 2)), np.resize(points[p2[2]:p2[2] + p2[3]], (6000, 2))])
        together = eng.pair_dependence_rows(big, gprobes, gpoints, mean=True)
        alone = np.concatenate([eng.pair_dependence_rows(big, [(p[0], p[1], 0, p[3])], gpoints[p[2]:p[2] + p[3]], mean=True) for p in gprobes])
        assert np.array_equal(together, alone)
        assert np.array_equal(together[:p0[3]], together[p0[3]:2 * p0[3]])  # repeated points: the same bits
        assert np.abs(together[:p0[3]] - mean[:p0[3]]).max() <= TOL  # 100 copies of the rows: the same mean
    finally:
        m.close()


def test_errors(rf100d6, curated):
    from databricks_kubernetes_mlops_poc_b200._cabi import B2FError
    from oracle import reference_pipeline as rp

    m = _model(rf100d6)
    eng, enc = m.engine, m.encoder
    try:
        rows = enc.encode_frame(curated[rp.FEATURES].iloc[:100])
        pts = np.zeros((8, 2), dtype=np.uint32)
        pts[:, 0].view(np.float32)[:] = np.linspace(1e4, 5e5, 8)
        pts[:, 1] = np.arange(8) % 2
        good = [(9, 0, 0, 8)]
        want = eng.pair_dependence_rows(rows, good, pts)
        inf = pts.copy()
        inf[3, 0] = 0x7F800000
        big = np.zeros((40000, 2), dtype=np.uint32)
        bad = [
            ([(9, 9, 0, 8)], pts, False, -1), ([(23, 0, 0, 8)], pts, False, -1), ([(9, 23, 0, 8)], pts, False, -1),
            ([(-1, 0, 0, 8)], pts, False, -1), ([(9, -2, 0, 8)], pts, False, -1), ([(9, 0, 0, 0)], pts, False, -1),
            ([(9, 0, 0, 65537)], np.zeros((65537, 2), np.uint32), True, -1), ([(9, 0, -1, 8)], pts, False, -1),
            ([(9, 0, 0, 8)] * 277, pts, True, -1), ([], pts, False, -1),
            ([(9, 0, 0, 40000), (10, 0, 0, 40000)], big, False, -1),  # curves of more than 65 536 points per row
            ([(0, 9, 0, 8)], np.stack([np.full(8, 99, np.uint32), pts[:, 0]], axis=1), False, -1),  # a code outside the vocabulary
            ([(9, 0, 0, 8)], np.stack([pts[:, 0], np.full(8, 0xFFFFFFFE, np.uint32)], axis=1), True, -1),  # code -2
            ([(9, 0, 0, 8)], inf, False, -7), ([(9, 0, 0, 8)], inf, True, -7),
        ]
        for probes, p, mean, rc in bad:
            with pytest.raises(B2FError, match=rf"rc={rc}\)"):
                eng.pair_dependence_rows(rows, probes, p, mean=mean)
            assert np.array_equal(eng.pair_dependence_rows(rows, good, pts), want)  # the handle keeps working
        # 276 probes and a mean over more than 65 536 points are fine
        assert eng.pair_dependence_rows(rows[:5], [(9, 0, 0, 8)] * 276, pts, mean=True).shape == (276 * 8,)
        assert eng.pair_dependence_rows(rows[:5], [(9, 0, 0, 40000), (10, 0, 0, 40000)], big, mean=True).shape == (80000,)
        with pytest.raises(B2FError, match=r"rc=-1\)"):
            eng.pair_dependence_rows(rows[:0], good, pts, mean=True)  # a mean needs a row
        if eng.rank_words:
            with pytest.raises(B2FError, match=r"rc=-1\).*ranked"):
                eng.pair_dependence_rows(enc.rank_rows(rows), good, pts)
        # NaN point words are the median's
        from databricks_kubernetes_mlops_poc_b200.flatten import parse_header

        nan = pts.copy()
        nan[2, 0] = 0x7FC00000
        med = pts.copy()
        med[2, 0] = np.array([parse_header(m.flat.blob)["impute"][9]], dtype=np.float32).view(np.uint32)[0]
        assert np.array_equal(eng.pair_dependence_rows(rows, good, nan), eng.pair_dependence_rows(rows, good, med))
        for bad_model in ("features", "kind", "same"):
            with pytest.raises(ValueError):
                {"features": lambda: m.pair_dependence(curated.iloc[:5], [("age", "nope")]),
                 "kind": lambda: m.pair_dependence(curated.iloc[:5], [("age", "sex")], kind="x"),
                 "same": lambda: m.pair_dependence(curated.iloc[:5], [("age", "age")])}[bad_model]()
        with pytest.raises(ValueError):
            m.interaction_strength(curated.iloc[:1])
        with pytest.raises(ValueError):
            m.interaction_strength(curated.iloc[:20000], sample=10001)
    finally:
        m.close()


def test_deeper_than_the_walk_stack(curated):
    from databricks_kubernetes_mlops_poc_b200._cabi import B2FError
    from databricks_kubernetes_mlops_poc_b200.flatten import parse_header
    from oracle import reference_pipeline as rp

    pipe = rp.fit_reference_pipeline(curated.iloc[:8000], dict(n_estimators=3, max_depth=None, min_samples_leaf=1, random_state=0))
    m = _model(pipe)
    try:
        if parse_header(m.flat.blob)["max_depth"] <= 32:
            pytest.skip("this forest fits the walk stack")
        rows = m.encoder.encode_frame(curated[rp.FEATURES].iloc[:8])
        with pytest.raises(B2FError, match="depth"):
            m.engine.pair_dependence_rows(rows, [(9, 10, 0, 1)], np.zeros((1, 2), np.uint32))
    finally:
        m.close()


def test_model_dir_and_http(tmp_path, rf100d6, curated):
    import httpx

    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer, flatten_pipeline
    from databricks_kubernetes_mlops_poc_b200.model import load_model, save_model_dir
    from databricks_kubernetes_mlops_poc_b200.server import create_app
    from oracle import reference_pipeline as rp

    bg = curated[rp.FEATURES].iloc[:3000]
    df = curated[rp.FEATURES].iloc[5000:5040].reset_index(drop=True)
    flat = flatten_pipeline(rf100d6)
    save_model_dir(str(tmp_path / "bg"), flat, explain_blob=flatten_explainer(rf100d6, flat), explain_background=bg)
    model = load_model(str(tmp_path / "bg"))
    try:
        grids = {f: model.dependence_grids[f] for f in ("credit_limit", "education")}
        want = model.pair_dependence(df, [("credit_limit", "education")], kind="both", custom_values=grids)
        strength = model.interaction_strength(df, ["credit_limit", "education", "age"])
        body = df.to_dict(orient="records")

        async def main(queries):
            app = create_app(model=model)
            async with app.router.lifespan_context(app):
                async with httpx.AsyncClient(transport=httpx.ASGITransport(app=app), base_url="http://t") as c:
                    preds = [c.post("/predict", json=body) for _ in range(8)]
                    calls = [c.post(path, params=q, json=body) for path, q in queries]
                    return await asyncio.gather(*calls, *preds)

        pair = "/explain/dependence/pair"
        queries = [(pair, [("feature", "credit_limit"), ("feature", "education"), ("kind", "both")]),
                   (pair, [("feature", "credit_limit"), ("feature", "education")]),
                   ("/explain/interaction_strength", [("feature", "credit_limit"), ("feature", "education"), ("feature", "age")]),
                   (pair, [("feature", "age")]), (pair, [("feature", "age"), ("feature", "age")]),
                   ("/explain/interaction_strength", [("feature", "age")])]
        res = asyncio.run(main(queries))
        j = res[0].json()
        assert res[0].status_code == 200 and j["feature_names"] == ["credit_limit", "education"]
        assert j["grid_values"] == [list(grids["credit_limit"]), list(grids["education"])]
        assert np.array_equal(np.asarray(j["individual"]), want["individual"][0])
        assert np.array_equal(np.asarray(j["average"]), want["average"][0])
        assert res[1].status_code == 200 and "individual" not in res[1].json()
        assert np.array_equal(np.asarray(res[1].json()["average"]), want["average"][0])
        j = res[2].json()
        assert res[2].status_code == 200 and j["rows"] == 40 and j["pairs"] == [list(p) for p in strength["pairs"]]
        assert np.array_equal(np.asarray(j["h_squared"], dtype=np.float64), strength["h_squared"], equal_nan=True)
        assert [r.status_code for r in res[3:6]] == [422] * 3
        assert all(r.status_code == 200 for r in res[6:])
    finally:
        model.close()
