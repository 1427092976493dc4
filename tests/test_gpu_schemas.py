"""Every kernel on request schemas other than the credit-default one (tests/schema_zoo.py), against the library and the
oracles: packed field 4 across the word boundary, the rank kernel's 8-byte categorical block and a value block filled
to its 128th pseudo-feature, TreeSHAP masks past code 31 / 63 / 95, three fields for eight warps, 17 categoricals, and
the moments kernel's NC = 0..4 categorical words per vector and its pivot.  The preconditions are asserted in
tests/test_schemas_cpu.py::test_schema_preconditions; the few a test leans on directly are asserted again here.

Bars as in the rest of the suite: float64 outputs 1e-12, float32 outputs 2e-7, labels exact."""

import os

import numpy as np
import pandas as pd
import pytest

import schema_zoo as sz

pytestmark = pytest.mark.gpu

TOL64 = 1e-12
TOL32 = 2e-7
BATCHES = (1, 31, 33, 4096, 65536)


def _with_env(env: dict, make):
    old = {k: os.environ.get(k) for k in env}
    try:
        os.environ.update(env)
        return make()
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _engine(pipe, env=None, explain=False):
    from databricks_kubernetes_mlops_poc_b200 import flatten
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine

    flat = flatten.flatten_pipeline(pipe)
    eng = _with_env(env or {}, lambda: ForestEngine(flat, 0))
    if explain:
        eng.attach_explainer(flatten.flatten_explainer(pipe, flat))
    return flat, eng, RowEncoder(flat)


_FRAMES = {}


def _big_frame(name, n):
    """Edge rows first, then synthetic rows, ``n`` in all; with the library's answers."""
    key = (name, n)
    if key not in _FRAMES:
        spec, pipe = sz.fitted(name)
        edge = sz.edge_rows(spec, pipe)
        df = pd.concat([edge, sz.make_frame(spec, n - len(edge), seed=21, target=False)], ignore_index=True)
        _FRAMES[key] = (df, *sz.predict(pipe, df))
    return _FRAMES[key]


def _agree(eng, rows, want_p, want_l):
    p64, l64 = eng.predict_rows(rows, np.float64)
    p32, l32 = eng.predict_rows(rows, np.float32)
    assert np.abs(p64 - want_p).max() <= TOL64 and (l64 == want_l).all()
    assert np.abs(p32.astype(np.float64) - want_p).max() <= TOL32 and (l32 == want_l).all()


@pytest.mark.parametrize("name", ["packed_wide", "packed_wide_gbdt", "rank_wide", "rank_wide_129", "tiny", "tiny_gbdt", "over16"])
def test_predict_kernels(name):
    """Each float32-row kernel (warp, tile, split, auto) on the 96-byte rows and, where the schema packs, the 64-byte rows;
    the resident rank kernel and its streaming form on ranked rows where the forest has a rank layout."""
    spec, pipe = sz.fitted(name)
    df, want_p, want_l = _big_frame(name, 90000)
    flat, eng, enc = _engine(pipe)
    try:
        rows = enc.encode_frame(df)
        packed = enc.pack_rows(rows) if enc.packed_ok else None
        rank_ok = bool(eng.info()["rank_ok"])
        ranked = enc.rank_rows(rows) if rank_ok else None
        assert rank_ok == (name in ("rank_wide", "tiny", "tiny_gbdt"))
    finally:
        eng.close()
    for kernel in ("warp", "tile", "split", "auto"):
        _, eng, _ = _engine(pipe, {"B2F_KERNEL": kernel})
        try:
            for n in BATCHES:
                _agree(eng, rows[:n], want_p[:n], want_l[:n])
                if packed is not None:
                    _agree(eng, packed[:n], want_p[:n], want_l[:n])
        finally:
            eng.close()
    if ranked is None:
        return
    for env in ({}, {"B2F_RANK_STREAM": "1"}):
        _, eng, _ = _engine(pipe, env)
        try:
            l0 = eng.info()["launches_rank"]
            for n in BATCHES + (90000,):
                _agree(eng, ranked[:n], want_p[:n], want_l[:n])
            assert eng.info()["launches_rank"] > l0
            p1, _ = eng.predict_rows(ranked, np.float64)
            p2, _ = eng.predict_rows(ranked, np.float64)
            assert np.array_equal(p1, p2)
        finally:
            eng.close()


EXPLAIN = ["packed_wide", "packed_wide_gbdt", "packed_wide_shallow", "rank_wide", "tiny", "tiny_gbdt", "over16"]


@pytest.mark.parametrize("name", EXPLAIN)
def test_explainers(name):
    """K5 (path-dependent TreeSHAP), K5b (interactions) and K5c (interventional) against the oracles on row samples, and
    their identities on every row: local accuracy, base values, exact symmetry, row sums equal to K5's phi; packed rows
    give the 96-byte rows' results bit for bit.  Brute-force Shapley values on the shallow forests."""
    import treeshap_interactions as tsi
    import treeshap_interventional as tiv

    from oracle import treeshap as ts
    from oracle import treewalk as tw

    spec, pipe = sz.fitted(name)
    df, want_p, _ = _big_frame(name, 4096)
    bg = sz.make_frame(spec, 24, seed=31, target=False)
    flat, eng, enc = _engine(pipe, explain=True)
    dump, cov = tw.dump_pipeline(pipe), ts.dump_covers(pipe)
    try:
        rows = enc.encode_frame(df)
        X = sz.dense(pipe, df)
        _, _, raw = tw.walk_numpy(dump, X)
        target = want_p if flat.agg_mode == 0 else raw
        F = len(spec[0]) + spec[1]
        phi, base = eng.explain_rows(rows)
        assert phi.shape == (len(df), F)
        assert np.abs(base + phi.sum(axis=1) - target).max() <= TOL64
        s = slice(0, 120)
        want, wbase = ts.tree_shap(dump, cov, X[s])
        assert abs(base - wbase) <= TOL64 and np.abs(phi[s] - want).max() <= TOL64
        if name in ("packed_wide_shallow", "tiny_gbdt"):
            bphi, bbase = ts.brute_force_shap(dump, cov, X[:60])
            assert np.abs(phi[:60] - bphi).max() <= TOL64 and abs(base - bbase) <= TOL64

        n2 = 1024
        phi2, base2 = eng.explain_interactions_rows(rows[:n2])
        assert phi2.shape == (n2, F, F) and abs(base2 - base) <= TOL64
        assert np.array_equal(phi2, phi2.transpose(0, 2, 1))
        assert np.abs(phi2.sum(axis=2) - phi[:n2]).max() <= TOL64
        if name not in ("packed_wide", "over16"):  # the interaction oracle on 60 trees of depth 8 is minutes of numpy
            want2, _ = tsi.tree_shap_interactions(dump, cov, X[:24])
            assert np.abs(phi2[:24] - want2).max() <= TOL64

        eng.attach_background(enc.encode_frame(bg))
        iphi, ibase = eng.explain_interventional_rows(rows)
        assert np.abs(ibase + iphi.sum(axis=1) - target).max() <= TOL64
        Z = sz.dense(pipe, bg)
        want, wbase = tiv.interventional_shap(dump, X[:40], Z)
        assert abs(ibase - wbase) <= TOL64 and np.abs(iphi[:40] - want).max() <= TOL64

        if enc.packed_ok:
            pk = enc.pack_rows(rows)
            assert np.array_equal(eng.explain_rows(pk)[0], phi)
            assert np.array_equal(eng.explain_interactions_rows(pk[:n2])[0], phi2)
            assert np.array_equal(eng.explain_interventional_rows(pk)[0], iphi)
        for n in (1, 31, 33):  # another batch size groups the sums differently: equal to the last bit or two
            assert np.abs(eng.explain_rows(rows[:n])[0] - phi[:n]).max() <= 1e-14
    finally:
        eng.close()


@pytest.mark.parametrize("rows", ["default", "ranked"])
@pytest.mark.parametrize("name", ["packed_wide", "rank_wide", "over16"])
def test_plugin_predict_and_explain(name, rows, monkeypatch):
    """B200Model.from_pipeline(...).predict / .explain on more than 128 rows (the columnar pipeline) against the library,
    with the scorer's default rows and with ranked rows; a 17-categorical schema answers through the portable encoder."""
    from databricks_kubernetes_mlops_poc_b200 import engine as engine_mod
    from databricks_kubernetes_mlops_poc_b200.model import B200Model

    spec, pipe = sz.fitted(name)
    df, want_p, _ = _big_frame(name, 4096)
    df = df.iloc[400:].reset_index(drop=True)  # no object-dtype edge rows: the native path where the schema has one
    want_p = want_p[400:]
    monkeypatch.setattr(engine_mod, "_FMT_OVERRIDE", engine_mod.ROWS_RANKED if rows == "ranked" else None)
    model = B200Model.from_pipeline(pipe, devices=[0], explain=True)
    try:
        for frame, want in ((df, want_p), (df.iloc[:200], want_p[:200]), (df.iloc[:5], want_p[:5])):
            out = model.predict(frame)
            assert np.abs(np.asarray(out["predictions"]) - want).max() <= TOL64
        arrow = df.copy()
        for c in sz.cat_names(spec):
            arrow[c] = arrow[c].astype("string[pyarrow]")
        assert np.abs(np.asarray(model.predict(arrow)["predictions"]) - want_p).max() <= TOL64
        if rows == "ranked" and model.engine.info()["rank_ok"]:
            assert model.last_timing is not None and model.last_timing["row_format"] == 2
        ex = model.explain(df.iloc[:300])
        assert np.abs(ex["base_value"] + np.asarray(ex["contributions"]).sum(axis=1) - want_p[:300]).max() <= TOL64
    finally:
        model.close()


def test_isolation_forest_after_16_categoricals():
    """b2f_predict_full on rank_wide: the detector's words start at n_cat = 16; against sklearn's IsolationForest."""
    from sklearn.ensemble import IsolationForest

    from databricks_kubernetes_mlops_poc_b200 import flatten

    spec, pipe = sz.fitted("rank_wide")
    df, want_p, want_l = _big_frame("rank_wide", 4096)
    nums = sz.num_names(spec)
    train = sz.make_frame(spec, 3000, seed=41, target=False)
    iso = IsolationForest(n_estimators=100, random_state=0).fit(train[nums].to_numpy())
    clean = df.iloc[400:].reset_index(drop=True)  # no NaN or +-3e38: sklearn's detector refuses NaN
    thr = 0.0
    flat, eng, enc = _engine(pipe)
    try:
        eng.attach_outlier_forest(flatten.flatten_isolation_forest(iso, 16, 7, vocab=[len(c) for c in flat.categories], threshold=thr))
        want_s = -iso.decision_function(clean[nums].to_numpy())
        rows = enc.encode_frame(clean)
        for n in (1, 31, 33, len(clean)):
            out = eng.predict_full(rows[:n])
            assert np.abs(out["proba1"] - want_p[400 : 400 + n]).max() <= TOL64 and (out["label"] == want_l[400 : 400 + n]).all()
            assert np.abs(out["outlier_score"].astype(np.float64) - want_s[:n]).max() <= TOL32
            clear = np.abs(want_s[:n] - thr) > TOL32  # flags of scores within float32 rounding of the threshold may differ
            assert (out["is_outlier"][clear] == (want_s[:n] > thr)[clear]).all()
    finally:
        eng.close()


def test_drift_wide_vocabulary():
    """TabularDrift on packed_wide's columns (a 126-category field, a 100-category field) against scipy."""
    from scipy import stats

    from databricks_kubernetes_mlops_poc_b200.drift import TabularDrift

    spec, _ = sz.fitted("packed_wide")
    cats, feats = sz.cat_names(spec), sz.features(spec)
    ref = sz.make_frame(spec, 3000, seed=51, target=False)[feats]
    det = TabularDrift(ref, cats, device=0)
    try:
        moved = sz.make_frame(spec, 700, seed=52, target=False)[feats]
        moved[sz.num_names(spec)[0]] = moved[sz.num_names(spec)[0]] + 0.5
        for batch in (sz.make_frame(spec, 300, seed=53, target=False)[feats], moved, ref.iloc[:7].reset_index(drop=True)):
            p, stat, flags = det.statistics(batch)
            assert (flags == 0).all()
            for i, name in enumerate(feats):
                if name in cats:
                    a, x = ref[name].astype(str).to_numpy(), batch[name].astype(str).to_numpy()
                    union = sorted(set(a.tolist()) | set(x.tolist()))
                    r = stats.chi2_contingency(np.array([[np.sum(a == v) for v in union], [np.sum(x == v) for v in union]]))
                    assert abs(stat[i] - r[0]) <= 1e-10 * max(r[0], 1e-300), name
                    assert abs(p[i] - r[1]) <= 1e-9 * max(r[1], 1e-300), name
                else:
                    r = stats.ks_2samp(ref[name].to_numpy(float), batch[name].to_numpy(float), alternative="two-sided", method="exact")
                    assert abs(stat[i] - r.statistic) <= 4e-16, name
                    assert abs(p[i] - r.pvalue) <= 1e-9 * max(r.pvalue, 1e-300), (name, p[i], r.pvalue)
        assert len(set(ref[cats[4]])) == 126
    finally:
        det.close()


@pytest.mark.parametrize("n_cat", sz.MOMENT_N_CAT)
def test_moments(n_cat):
    """k_feature_moments against np.nanmean / np.nanvar for n_cat categorical words (every compiled NC = 0..4 at some
    vector q > 0 over the set).  Column n_cat is 1e6 + N(0, 1) with row 0 missing, column n_cat + 3 is 5e5 + N(0, 0.5)
    missing in the first half of the rows: the shift must be a value of the column, not 0 (which cancels to ~1e-5
    relative error in m2).  The last column is entirely missing: count 0, mean 0, m2 0."""
    spec = sz.moments_schema(n_cat)
    vocab, n_num = spec
    _, pipe = sz.fitted_small(spec)
    _, eng, enc = _engine(pipe)
    try:
        n = 200_003
        codes, nums = sz.make_codes_nums(spec, n, seed=61 + n_cat)
        rng = np.random.default_rng(n_cat)
        nums[:, 0] = 1e6 + rng.normal(0.0, 1.0, n)
        nums[rng.random(n) < 0.03, 0] = np.nan
        nums[0, 0] = np.nan
        nums[:40, 1] = np.nan  # the first present value beyond the first 32 rows
        nums[rng.random(n) < 0.1, 2 % n_num] = np.nan
        nums[:, 3] = 5e5 + rng.normal(0.0, 0.5, n)
        nums[: n // 2, 3] = np.nan  # a field that appears halfway through the batch: most blocks meet no value of it
        nums[:, n_num - 1] = np.nan
        rows = enc.encode_arrays(codes, nums)
        got = eng.moments(rows)
        f = rows.view(np.float32)[:, n_cat : n_cat + n_num].astype(np.float64)
        cnt = (~np.isnan(f)).sum(axis=0)
        assert (got[n_cat : n_cat + n_num, 0] == cnt).all()
        assert cnt[-1] == 0 and (got[n_cat + n_num - 1] == 0).all()
        live = slice(n_cat, n_cat + n_num - 1)
        with np.errstate(invalid="ignore"):
            mean, var = np.nanmean(f[:, :-1], axis=0), np.nanvar(f[:, :-1], axis=0)
        assert np.allclose(got[live, 1], mean, rtol=1e-9, atol=0)
        assert np.allclose(got[live, 2] / cnt[:-1], var, rtol=1e-9, atol=0), np.nanmax(np.abs(got[live, 2] / cnt[:-1] / var - 1))
        c = codes.astype(np.float64)
        assert (got[:n_cat, 0] == n).all()
        assert np.allclose(got[:n_cat, 1], c.mean(axis=0), rtol=1e-10)
        assert np.allclose(got[:n_cat, 2] / n, c.var(axis=0), rtol=1e-9)
        assert (got[n_cat + n_num :, 0] == n).all() and (got[n_cat + n_num :, 1:] == 0).all()  # zero padding words
        assert np.array_equal(eng.moments(rows), got)  # fixed reduction order: bit-identical run to run
        for m in (1, 31, 33, 4096):  # few rows: one or a few CTAs, pivots from inside the batch
            part = eng.moments(rows[:m])
            fm = f[:m, :-1]
            pres = ~np.isnan(fm)
            assert (part[live, 0] == pres.sum(axis=0)).all()
            ok = pres.sum(axis=0) > 0
            with np.errstate(invalid="ignore"):
                pm, pv = np.nanmean(fm, axis=0), np.nanvar(fm, axis=0)
            assert np.allclose(part[live, 1][ok], pm[ok], rtol=1e-9, atol=1e-12)
            assert np.allclose(part[live, 2][ok] / pres.sum(axis=0)[ok], pv[ok], rtol=1e-9, atol=1e-12)
            assert (part[live, 1][~ok] == 0).all() and (part[live, 2][~ok] == 0).all()
    finally:
        eng.close()
