"""k_permutation_scores on the GPU: every record equal to the numpy emulator (tests/importance_walk.py) on the reference
forests, GBDTs, deep, tiny and 33-tree forests and the schema-zoo schemas, in both float32 row formats; the end-to-end
importances equal to scikit-learn's ``permutation_importance`` of the fitted pipeline; the baseline against the predict
kernels; determinism, independence from the field grouping, the C-ABI errors, calls among in-flight score batches, and the
B200Model and ``POST /explain/importance`` layers."""

import asyncio

import numpy as np
import pandas as pd
import pytest

import schema_zoo as sz
from importance_walk import permutation_scores as emulate

pytestmark = pytest.mark.gpu

INT_FIELDS = ("tp", "fp", "tn", "fn", "auc_u2")
THRESHOLD_SCORERS = ("accuracy", "precision", "recall", "f1")


def _engine(pipe):
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline

    flat = flatten_pipeline(pipe)
    return flat, ForestEngine(flat, 0), RowEncoder(flat)


def _records_equal(got, want):
    """Integer fields exactly, the loss sums to 1e-12 relative (CUDA's log / exp may differ from numpy's in the last bit)."""
    for k in INT_FIELDS:
        assert np.array_equal(got[k], want[k]), k
    for k in ("log_loss_sum", "brier_sum"):
        assert np.allclose(got[k], want[k], rtol=1e-12, atol=1e-300), k


def _check(pipe, X, y, n_repeats=3, words=None, seed=0):
    from databricks_kubernetes_mlops_poc_b200 import importance

    flat, eng, enc = _engine(pipe)
    try:
        rows = enc.encode_frame(X)
        words = list(range(enc.n_cat + enc.n_num)) if words is None else words
        perm = importance.permutations(len(rows), n_repeats, seed)
        want, want_base = emulate(flat.blob, rows, y, perm, words)
        got, base = eng.permutation_scores(rows, y, perm, words)
        _records_equal(got, want)
        _records_equal(base, want_base)
        if enc.packed_ok:
            g2, b2 = eng.permutation_scores(enc.pack_rows(rows), y, perm, words)
            assert g2.tobytes() == got.tobytes() and b2.tobytes() == base.tobytes()
    finally:
        eng.close()


def _frame(curated, adversarial, lo, n, n_adv):
    from oracle import reference_pipeline as rp

    X = pd.concat([curated[rp.FEATURES].iloc[lo:lo + n], adversarial.iloc[:n_adv]], ignore_index=True)
    y = np.concatenate([curated[rp.TARGET].iloc[lo:lo + n].to_numpy(), np.arange(n_adv) % 2]).astype(np.int32)
    return X, y


def test_rf100d6(rf100d6, curated, adversarial):
    X, y = _frame(curated, adversarial, 20000, 150, 50)
    _check(rf100d6, X, y, n_repeats=3)
    _check(rf100d6, X.iloc[:40], y[:40], n_repeats=33, words=[9, 0, 9])  # a segment of 32 and one of 1; a repeated word


@pytest.mark.parametrize("which", ["rf500d8", "gbdt_small", "bench_gbdt", "deep24", "stumps", "trees33"])
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
                  "stumps": dict(n_estimators=33, max_depth=1, random_state=0),
                  "trees33": dict(n_estimators=33, max_depth=3, random_state=0)}[which]
        pipe = rp.fit_reference_pipeline(curated.iloc[:6000], params)
    n = 40 if which in ("rf500d8", "deep24") else 120
    X, y = _frame(curated, adversarial, 7000, n, n // 3)
    _check(pipe, X, y, n_repeats=2, words=[0, 3, 9, 10, 12, 22] if which in ("rf500d8", "deep24") else None)


@pytest.mark.parametrize("name", ["packed_wide", "packed_wide_gbdt", "tiny", "tiny_gbdt", "over16"])
def test_schema_zoo(name):
    spec, pipe = sz.fitted(name)
    X = pd.concat([sz.edge_rows(spec, pipe, n=16), sz.make_frame(spec, 48, seed=9, target=False)], ignore_index=True)
    y = (np.arange(len(X)) * 7 % 3 == 0).astype(np.int32)
    _check(pipe, X, y, n_repeats=2)


def _ordered(frame, inference):
    """The frame's features in the order of the inference table's columns."""
    from oracle import reference_pipeline as rp

    return frame[[c for c in inference.columns if c in rp.FEATURES]]


def _against_sklearn(model, pipe, X, y, n_repeats, scoring):
    from sklearn.inspection import permutation_importance
    from sklearn.metrics import check_scoring

    got = model.permutation_importance(X, y, scoring=scoring, n_repeats=n_repeats, random_state=0)
    want = permutation_importance(pipe, X, y, scoring=scoring, n_repeats=n_repeats, random_state=0, n_jobs=1)
    order = [list(X.columns).index(f) for f in model.all_features]
    for s in scoring:
        g, w = got[s], want[s]
        assert g["feature_names"] == list(model.all_features) and g["rows"] == len(X) and g["n_repeats"] == n_repeats
        tol = 0.0 if s in THRESHOLD_SCORERS else 1e-12
        assert np.allclose(g["baseline_score"], check_scoring(pipe, scoring=s)(pipe, X, y), rtol=tol, atol=tol), s
        for k in ("importances", "importances_mean", "importances_std"):
            assert np.allclose(g[k], w[k][order], rtol=tol, atol=max(tol, 1e-15 if k == "importances_std" else tol)), (s, k)
    return got


def test_end_to_end_equals_sklearn(rf100d6, rf500d8, gbdt_small, curated, inference):
    from databricks_kubernetes_mlops_poc_b200 import importance
    from databricks_kubernetes_mlops_poc_b200.model import B200Model
    from oracle import reference_pipeline as rp

    _, test = rp.reference_split(curated)
    X, y = _ordered(test, inference).reset_index(drop=True), test[rp.TARGET].to_numpy()
    assert len(X) == 6000
    scoring = list(importance.SCORERS)
    for pipe, n in ((rf100d6, 6000), (rf500d8, 1000), (gbdt_small, 1000)):
        m = B200Model.from_pipeline(pipe)
        try:
            got = _against_sklearn(m, pipe, X.iloc[:n], y[:n], 5, scoring)
            if n == 6000:
                # the baseline against the predict kernels on the unpermuted rows
                p1, lab = m.predict_proba1(X), m.predict_label(X)
                rec = emulate_record(p1, lab, y)
                for s in scoring:
                    # integers exactly; p1 may come from another kernel's summation order here, so the rest to 1e-9
                    assert got[s]["baseline_score"] == pytest.approx(float(importance.score(s, rec)), rel=0 if s in THRESHOLD_SCORERS else 1e-9,
                                                                     abs=0 if s in THRESHOLD_SCORERS else 1e-9), s
                # column order does not matter
                again = m.permutation_importance(X[list(m.all_features)], y, scoring=scoring, n_repeats=5, random_state=0)
                for s in scoring:
                    assert np.array_equal(again[s]["importances"], got[s]["importances"], equal_nan=True)
        finally:
            m.close()


def emulate_record(p1, lab, y):
    from importance_walk import record

    return record(np.asarray(p1, np.float64), np.asarray(lab), np.asarray(p1, np.float64), y)


def test_determinism_and_grouping(rf100d6, curated):
    """n = 300 000 rows take several groups of points (B2F_PERM_SCRATCH_BYTES); a call is bit-identical to itself and to
    the same call made one field at a time."""
    from databricks_kubernetes_mlops_poc_b200 import importance
    from oracle import reference_pipeline as rp

    flat, eng, enc = _engine(rf100d6)
    try:
        base_rows = enc.encode_frame(curated[rp.FEATURES])
        idx = np.arange(300_000) % len(base_rows)
        rows = base_rows[idx]
        y = curated[rp.TARGET].to_numpy()[idx].astype(np.int32)
        perm = importance.permutations(len(rows), 5, 3)
        words = list(range(enc.n_cat + enc.n_num))
        assert 18 * len(rows) * (1 + 23 * 5) > (256 << 20)  # more than one group
        a, base_a = eng.permutation_scores(rows, y, perm, words)
        b, base_b = eng.permutation_scores(rows, y, perm, words)
        assert a.tobytes() == b.tobytes() and base_a.tobytes() == base_b.tobytes()
        for w in words:
            one, base_one = eng.permutation_scores(rows, y, perm, [w])
            assert one.tobytes() == a[w:w + 1].tobytes() and base_one.tobytes() == base_a.tobytes(), w
        packed = eng.permutation_scores(enc.pack_rows(rows), y, perm, words)[0]
        assert packed.tobytes() == a.tobytes()
    finally:
        eng.close()


def test_during_inflight_scores(rf100d6, curated):
    """Score batches in flight on every slot stream while a permutation call runs on the compute stream: both give what
    they give alone."""
    from databricks_kubernetes_mlops_poc_b200 import importance
    from oracle import reference_pipeline as rp

    flat, eng, enc = _engine(rf100d6)
    try:
        rows = enc.encode_frame(curated[rp.FEATURES].iloc[:5000])
        y = curated[rp.TARGET].iloc[:5000].to_numpy().astype(np.int32)
        perm = importance.permutations(len(rows), 4, 1)
        p_alone = eng.predict_rows(rows, np.float64)[0]
        alone = eng.permutation_scores(rows, y, perm, [0, 9, 12])
    finally:
        eng.close()
    _, eng, _ = _engine(rf100d6)
    try:
        n = len(rows)
        staged, proba, label = eng.staging(4 * n)
        proba[:] = -1
        tickets = []
        for k in range(4):
            staged[k * n:(k + 1) * n] = rows
            tickets.append(eng.predict_rows_async(staged[k * n:(k + 1) * n], proba[k * n:(k + 1) * n], label[k * n:(k + 1) * n]))
        got = eng.permutation_scores(rows, y, perm, [0, 9, 12])
        for t in tickets:
            eng.wait(t)
        assert np.array_equal(proba, np.tile(p_alone, 4))
        assert got[0].tobytes() == alone[0].tobytes() and got[1].tobytes() == alone[1].tobytes()
    finally:
        eng.close()


def test_errors(rf100d6, curated):
    from databricks_kubernetes_mlops_poc_b200 import _cabi, importance
    from databricks_kubernetes_mlops_poc_b200._cabi import B2FError, ptr
    from oracle import reference_pipeline as rp

    flat, eng, enc = _engine(rf100d6)
    try:
        rows = enc.encode_frame(curated[rp.FEATURES].iloc[:64])
        y = (np.arange(64) % 2).astype(np.int32)
        perm = importance.permutations(64, 2, 0)
        lib, h = eng._lib, eng.handle
        out = np.zeros(46, dtype=_cabi.PERM_SCORE_DTYPE)
        base = np.zeros(1, dtype=_cabi.PERM_SCORE_DTYPE)

        def call(rows_=rows, n=64, fmt=_cabi.ROWS_WORDS24, y_=y, perm_=perm, reps=2, words=np.arange(23, dtype=np.int32), nw=None):
            return lib.b2f_permutation_scores(h, ptr(rows_), n, fmt, ptr(y_), ptr(perm_), reps, ptr(words), len(words) if nw is None else nw,
                                              ptr(out), ptr(base), None)

        assert call() == 0
        cases = {
            "ranked": dict(fmt=_cabi.ROWS_RANKED), "n = 0": dict(n=0), "n < 0": dict(n=-1), "n >= 2^31": dict(n=1 << 31),
            "label 2": dict(y_=np.where(np.arange(64) == 5, 2, y).astype(np.int32)),
            "label -1": dict(y_=np.where(np.arange(64) == 63, -1, y).astype(np.int32)),
            "repeats 0": dict(reps=0), "repeats 257": dict(reps=257),
            "word 23": dict(words=np.array([0, 23], np.int32)), "word -1": dict(words=np.array([-1], np.int32)), "no words": dict(nw=0),
            "perm 64": dict(perm_=np.where(np.arange(128).reshape(2, 64) == 100, 64, perm).astype(np.int32)),
            "perm -1": dict(perm_=np.where(np.arange(128).reshape(2, 64) == 3, -1, perm).astype(np.int32)),
        }
        for what, kw in cases.items():
            assert call(**kw) == -1, what
            assert _cabi.last_error(), what
        assert call(**cases["perm 64"]) == -1 and "not a row index" in _cabi.last_error()
        assert call(**cases["label 2"]) == -1 and "expected 0 or 1" in _cabi.last_error()
        assert lib.b2f_permutation_scores(h, ptr(rows), 64, 0, ptr(y), ptr(perm), 2, None, 1, ptr(out), ptr(base), None) == -1
        with pytest.raises(B2FError):
            eng.permutation_scores(rows, y, perm[:0], [0])
        # rows that cannot fit the 80 GB device: B2F_ENOMEM with the byte count.  The checks read every label and perm
        # entry (zero pages, never written); the rows buffer is the first allocation, so the rows are never read.
        big = 900_000_000
        ybig, pbig = np.zeros(big, np.int32), np.zeros(big, np.int32)
        rc = lib.b2f_permutation_scores(h, ptr(rows), big, 0, ptr(ybig), ptr(pbig), 1, ptr(np.zeros(1, np.int32)), 1, ptr(out), ptr(base), None)
        assert rc == -4 and "86400000000 device bytes" in _cabi.last_error(), _cabi.last_error()
        del ybig, pbig
        assert call() == 0  # the model still works
    finally:
        eng.close()


def test_deeper_than_the_walk_stack(curated):
    from databricks_kubernetes_mlops_poc_b200 import importance
    from databricks_kubernetes_mlops_poc_b200._cabi import B2FError
    from oracle import reference_pipeline as rp

    pipe = rp.fit_reference_pipeline(curated.iloc[:8000], dict(n_estimators=3, max_depth=None, min_samples_leaf=1, random_state=0))
    flat, eng, enc = _engine(pipe)
    try:
        from databricks_kubernetes_mlops_poc_b200.flatten import parse_header

        if parse_header(flat.blob)["max_depth"] <= 32:
            pytest.skip("this forest fits the walk stack")
        rows = enc.encode_frame(curated[rp.FEATURES].iloc[:8])
        with pytest.raises(B2FError, match="depth"):
            eng.permutation_scores(rows, np.zeros(8, np.int32), importance.permutations(8, 1, 0), [0])
    finally:
        eng.close()


def test_model_and_http(tmp_path, rf100d6, curated, iforest):
    import httpx

    from databricks_kubernetes_mlops_poc_b200 import importance
    from databricks_kubernetes_mlops_poc_b200.model import B200Model
    from databricks_kubernetes_mlops_poc_b200.schema import TARGET
    from databricks_kubernetes_mlops_poc_b200.server import create_app
    from oracle import reference_pipeline as rp

    m = B200Model.from_pipeline(rf100d6, outlier=iforest, outlier_threshold=0.0)
    try:
        X = curated[rp.FEATURES].iloc[3000:3400].reset_index(drop=True).copy()
        y = curated[rp.TARGET].iloc[3000:3400].to_numpy()
        X.loc[[1, 7, 30], "age"] = np.nan  # accepted: the classifier alone is scored
        one = m.permutation_importance(X, y, n_repeats=3, random_state=4)
        assert set(one) == {"importances", "importances_mean", "importances_std", "baseline_score", "feature_names", "n_repeats", "rows"}
        assert one["importances"].shape == (23, 3) and one["rows"] == 400
        rows = m.encoder.encode_frame(X)
        rec, base = m.engine.permutation_scores(rows, y, importance.permutations(400, 3, 4), list(range(23)))
        assert np.array_equal(one["importances"], float(importance.score("accuracy", base)) - importance.score("accuracy", rec))
        assert np.array_equal(one["importances_std"], np.std(one["importances"], axis=1))
        multi = m.permutation_importance(X, y, scoring=["roc_auc"], n_repeats=3, random_state=np.random.RandomState(0))
        assert list(multi) == ["roc_auc"]
        assert np.isnan(m.permutation_importance(X, np.ones(400, int), scoring="roc_auc", n_repeats=1)["baseline_score"])
        for kw in (dict(scoring="r2"), dict(n_repeats=0), dict(n_repeats=300), dict(scoring=["f1", "f1"])):
            with pytest.raises(ValueError):
                m.permutation_importance(X, y, **kw)
        with pytest.raises(ValueError):
            m.permutation_importance(X, np.ones(400, int), scoring="neg_log_loss")
        with pytest.raises(ValueError):
            m.permutation_importance(X, np.full(400, 2))
        with pytest.raises(ValueError):
            m.permutation_importance(X, y[:10])
        with pytest.raises(ValueError):
            m.predict(X)  # the outlier forest still refuses NaN on the scoring path

        body = [dict(r, **{TARGET: int(t)}) for r, t in zip(curated[rp.FEATURES].iloc[3000:3300].to_dict(orient="records"), y[:300])]
        pred_body = curated[rp.FEATURES].iloc[:50].to_dict(orient="records")
        direct = m.permutation_importance(pd.DataFrame(body)[rp.FEATURES], y[:300], scoring=["roc_auc", "neg_log_loss"], n_repeats=4,
                                          random_state=0)

        async def main():
            app = create_app(model=m)
            async with app.router.lifespan_context(app):
                async with httpx.AsyncClient(transport=httpx.ASGITransport(app=app), base_url="http://t", timeout=120) as c:
                    preds = [c.post("/predict", json=pred_body) for _ in range(6)]
                    imps = [c.post("/explain/importance", params=[("scoring", "roc_auc"), ("scoring", "neg_log_loss"), ("n_repeats", "4")], json=body),
                            c.post("/explain/importance", json=body), c.post("/explain/importance", params={"scoring": "nope"}, json=body)]
                    return await asyncio.gather(*imps, *preds)

        res = asyncio.run(main())
        j = res[0].json()
        assert res[0].status_code == 200 and j["rows"] == 300 and j["n_repeats"] == 4 and j["random_state"] == 0
        for s in ("roc_auc", "neg_log_loss"):
            assert j["scores"][s]["baseline"] == direct[s]["baseline_score"]
            assert j["scores"][s]["importances"] == direct[s]["importances"].tolist()
            assert j["scores"][s]["importances_mean"] == direct[s]["importances_mean"].tolist()
        again = res[1].json()
        assert res[1].status_code == 200 and list(again["scores"]) == ["accuracy"] and len(again["scores"]["accuracy"]["importances"][0]) == 5
        assert res[2].status_code == 422
        assert all(r.status_code == 200 for r in res[3:])
    finally:
        m.close()
