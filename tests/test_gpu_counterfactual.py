"""k_counterfactual on the GPU: every record equal to the numpy emulator (tests/counterfactual_walk.py) on the reference
forests, deep, tiny and GBDT forests and the schema-zoo schemas, in both float32 row formats; bit-identity of every
returned p1 with the tile kernel scoring the substituted row, and the decision one float32 step toward the row's value;
batch edges, chunking, the device form, determinism, the C-ABI errors and calls among in-flight score batches; categorical
flips against K6's ICE points; B200Model / load_model and POST /explain/counterfactual under concurrent /predict."""

import asyncio
import os

import numpy as np
import pandas as pd
import pytest

import schema_zoo as sz
from counterfactual_walk import counterfactual as emulate

pytestmark = pytest.mark.gpu

FIELDS = ["credit_limit", "age", "bill_amount_1", "payment_amount_1"]


def _engine(pipe):
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline

    flat = flatten_pipeline(pipe)
    return flat, ForestEngine(flat, 0), RowEncoder(flat)


def _same(a, b) -> bool:
    """Equal arrays, NaN equal to NaN."""
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))


def _records_equal(got, want, gbdt=False):
    """Exactly equal records.  GBDT probabilities: the emulator's expit is numpy's exp, which may differ from CUDA's in the
    last bit, so there p1 agrees to 4 ulp (the positions stay exact; the tile-kernel check is bit for bit)."""
    for k in ("value", "lower", "upper", "lower_p1", "upper_p1"):
        if gbdt and k.endswith("p1"):
            assert _same(np.isnan(got[k]), np.isnan(want[k])) and np.allclose(got[k], want[k], rtol=1e-15, atol=0, equal_nan=True), k
        else:
            assert _same(got[k], want[k]), k


def _tile_checks(flat, rows, words, proba, rec, cutoff):
    """Every returned p1 is the tile kernel's score of the row with the word set to the returned value, its decision
    differs from the row's, and one float32 step toward the row's value keeps the row's decision.  False when the forest
    does not fit the tile kernel."""
    from databricks_kubernetes_mlops_poc_b200._cabi import B2FError
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine

    os.environ["B2F_KERNEL"] = "tile"
    try:
        tile = ForestEngine(flat, 0)
    except B2FError as e:
        assert "tile kernel" in str(e)
        return False
    finally:
        del os.environ["B2F_KERNEL"]
    try:
        own = tile.predict_rows(rows, np.float64)[0]
        assert np.array_equal(own, proba)
        d = proba > cutoff
        for f, w in enumerate(words):
            for side, p_key in (("lower", "lower_p1"), ("upper", "upper_p1")):
                v = rec[side][:, f]
                hit = ~np.isnan(v)
                if not hit.any():
                    continue
                sub = rows[hit].copy()
                sub[:, w] = v[hit].view(np.uint32)
                p = tile.predict_rows(sub, np.float64)[0]
                assert np.array_equal(p, rec[p_key][hit, f]), (w, side)
                assert ((p > cutoff) != d[hit]).all()
                toward = np.nextafter(v[hit], np.float32(np.inf) if side == "lower" else np.float32(-np.inf)).astype(np.float32)
                sub[:, w] = toward.view(np.uint32)
                assert ((tile.predict_rows(sub, np.float64)[0] > cutoff) == d[hit]).all(), (w, side)
        return True
    finally:
        tile.close()


def _check(pipe, X, fields, cutoffs=(0.5,), tile=True):
    """Both row formats (packed where the schema fits) against the emulator, exactly; the tile checks.  -> flips seen."""
    from databricks_kubernetes_mlops_poc_b200.flatten import parse_header

    flat, eng, enc = _engine(pipe)
    gbdt = parse_header(flat.blob)["agg_mode"] == 1
    try:
        rows = enc.encode_frame(X)
        words = [enc.n_cat + enc.num_features.index(f) for f in fields]
        flips, cache = 0, {}
        for cutoff in cutoffs:
            want_p, want = emulate(flat.blob, rows, words, cutoff, cache)
            proba, rec = eng.counterfactual_rows(rows, words, cutoff)
            if gbdt:
                assert np.allclose(proba, want_p, rtol=1e-15, atol=0)
            else:
                assert np.array_equal(proba, want_p)
            _records_equal(rec, want, gbdt)
            if enc.packed_ok:
                p2, r2 = eng.counterfactual_rows(enc.pack_rows(rows), words, cutoff)
                assert np.array_equal(p2, proba) and _same(r2["lower"], rec["lower"]) and _same(r2["upper_p1"], rec["upper_p1"])
            if tile:
                _tile_checks(flat, rows, words, proba, rec, cutoff)
            flips += int((~np.isnan(rec["lower"])).sum() + (~np.isnan(rec["upper"])).sum())
        return flips
    finally:
        eng.close()


def test_rf100d6(rf100d6, curated, adversarial):
    from oracle import reference_pipeline as rp

    X = pd.concat([curated[rp.FEATURES].iloc[20000:20016], adversarial.iloc[:24]], ignore_index=True)
    assert _check(rf100d6, X, rp.NUMERIC_FEATURES, cutoffs=(0.0, 0.3, 0.5, 1.0)) > 0


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
    n = 2 if which in ("rf500d8", "deep24") else 8
    X = pd.concat([curated[rp.FEATURES].iloc[7000:7000 + n], adversarial.iloc[:n]], ignore_index=True)
    fields = FIELDS[:2] if which == "rf500d8" else FIELDS
    _check(pipe, X, fields, cutoffs=(0.3, 0.5))


@pytest.mark.parametrize("name", ["packed_wide", "packed_wide_gbdt", "tiny", "tiny_gbdt", "over16"])
def test_schema_zoo(name):
    spec, pipe = sz.fitted(name)
    X = pd.concat([sz.edge_rows(spec, pipe, n=16), sz.make_frame(spec, 16, seed=9, target=False)], ignore_index=True)
    _check(pipe, X, sz.num_names(spec), cutoffs=(0.3, 0.5))


def test_unsplit_field_and_no_flip(curated):
    """A word no node splits on: both sides NaN.  At cutoff 1 nothing is above the cutoff: no row flips anywhere."""
    from oracle import reference_pipeline as rp

    pipe = rp.fit_reference_pipeline(curated.iloc[:3000], dict(n_estimators=5, max_depth=2, random_state=0))
    flat, eng, enc = _engine(pipe)
    try:
        X = curated[rp.FEATURES].iloc[100:164].reset_index(drop=True)
        rows = enc.encode_frame(X)
        words = list(range(enc.n_cat, enc.n_cat + enc.n_num))
        from databricks_kubernetes_mlops_poc_b200.engine import blob_split_values

        unsplit = [w for w in words if len(blob_split_values(flat.blob, w)) == 0]
        assert unsplit
        proba, rec = eng.counterfactual_rows(rows, unsplit)
        assert np.isnan(rec["lower"]).all() and np.isnan(rec["upper"]).all() and np.isnan(rec["upper_p1"]).all()
        assert np.array_equal(rec["value"][:, 0], rows[:, unsplit[0]].view(np.float32))
        _, rec = eng.counterfactual_rows(rows, words, 1.0)
        assert np.isnan(rec["lower"]).all() and np.isnan(rec["upper"]).all()
    finally:
        eng.close()


def test_batches_formats_device_and_determinism(rf100d6, curated):
    from databricks_kubernetes_mlops_poc_b200._cabi import COUNTERFACTUAL_DTYPE, ROWS_PACKED64, ROWS_WORDS24
    from oracle import reference_pipeline as rp

    flat, eng, enc = _engine(rf100d6)
    try:
        cur = curated[rp.FEATURES]
        words = list(range(9, 23))
        rows = enc.encode_frame(cur.iloc[:2048])
        big = np.concatenate([rows] * 20)  # 40 960 rows: three chunks of at most 16 384
        ref_p, ref = eng.counterfactual_rows(big, words)
        p2, r2 = eng.counterfactual_rows(big, words)
        assert np.array_equal(ref_p, p2) and ref.tobytes() == r2.tobytes()  # run to run, bit for bit
        assert ref[:2048].tobytes() == ref[2048:4096].tobytes()  # a row's result does not depend on the batch
        want_p, want = emulate(flat.blob, rows[:6], words)
        assert np.array_equal(ref_p[:6], want_p)
        _records_equal(ref[:6], want)
        for n in (0, 1, 31, 33, 16383, 16385):
            p, r = eng.counterfactual_rows(big[:n], words)
            assert p.shape == (n,) and r.shape == (n, 14) and r.tobytes() == ref[:n].tobytes() and np.array_equal(p, ref_p[:n])
        p, r = eng.counterfactual_rows(enc.pack_rows(big), words)
        assert r.tobytes() == ref.tobytes() and np.array_equal(p, ref_p)
        for fmt, src in ((ROWS_WORDS24, big[:5000]), (ROWS_PACKED64, enc.pack_rows(big[:5000]))):
            src = np.ascontiguousarray(src)
            d_rows, d_p, d_out = eng.device_alloc(src.nbytes), eng.device_alloc(5000 * 8), eng.device_alloc(5000 * 14 * 32)
            try:
                eng.h2d(d_rows, src)
                eng.counterfactual_device(d_rows, 5000, words, 0.5, d_p, d_out, fmt)
                eng.sync()
                got_p, got = np.empty(5000, np.float64), np.empty((5000, 14), COUNTERFACTUAL_DTYPE)
                eng.d2h(got_p, d_p)
                eng.d2h(got, d_out)
                eng.counterfactual_device(d_rows, 5000, words, 0.5, 0, d_out, fmt)  # proba may be NULL
                eng.sync()
            finally:
                for d in (d_rows, d_p, d_out):
                    eng.device_free(d)
            assert np.array_equal(got_p, ref_p[:5000]) and got.tobytes() == ref[:5000].tobytes()
        # interleaved with scoring: unchanged
        p_before, _ = eng.predict_rows(rows, np.float64)
        assert eng.counterfactual_rows(rows, words)[1].tobytes() == ref[:2048].tobytes()
        assert np.array_equal(eng.predict_rows(rows, np.float64)[0], p_before)
    finally:
        eng.close()


def test_during_inflight_scores(rf100d6, curated):
    """Every slot stream carries a score batch still in flight when a counterfactual call grows the slot buffers those
    batches share: both give what they give alone."""
    from oracle import reference_pipeline as rp

    flat, eng, enc = _engine(rf100d6)
    try:
        rows = enc.encode_frame(curated[rp.FEATURES].iloc[:5000])
        p_alone = eng.predict_rows(rows, np.float64)[0]
        cf_alone = eng.counterfactual_rows(rows, [9, 10, 12])
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
        got = eng.counterfactual_rows(rows, [9, 10, 12])
        for t in tickets:
            eng.wait(t)
        assert np.array_equal(proba, np.tile(p_alone, 4))
        assert np.array_equal(got[0], cf_alone[0]) and got[1].tobytes() == cf_alone[1].tobytes()
    finally:
        eng.close()


def test_errors(rf100d6, curated):
    from databricks_kubernetes_mlops_poc_b200 import _cabi
    from databricks_kubernetes_mlops_poc_b200._cabi import B2FError
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine
    from oracle import reference_pipeline as rp

    flat, eng, enc = _engine(rf100d6)
    lib = _cabi.load_library()
    try:
        rows = enc.encode_frame(curated[rp.FEATURES].iloc[:100])
        want = eng.counterfactual_rows(rows, [9])
        bad = [([], 0.5), ([9] * 24, 0.5), ([8], 0.5), ([0], 0.5), ([23], 0.5), ([-1], 0.5), ([9], float("nan")), ([9], -0.1),
               ([9], 1.5), ([9], float("inf"))]
        for words, cutoff in bad:
            with pytest.raises(B2FError, match=r"rc=-1\)"):
                eng.counterfactual_rows(rows, words, cutoff)
            assert eng.counterfactual_rows(rows, [9])[1].tobytes() == want[1].tobytes()  # the handle keeps working
        with pytest.raises(B2FError, match=r"rc=-1\).*b2f_partial_dependence"):
            eng.counterfactual_rows(rows, [3])
        w = np.array([9], np.int32)
        assert lib.b2f_counterfactual(eng._h, _cabi.ptr(rows), -1, 0, _cabi.ptr(w), 1, 0.5, None, None, None) == -1
        assert lib.b2f_counterfactual(eng._h, _cabi.ptr(rows), 5, 0, _cabi.ptr(w), 1, 0.5, None, None, None) == -1  # NULL out
        assert lib.b2f_counterfactual(eng._h, _cabi.ptr(rows), 0, 0, _cabi.ptr(w), 1, 0.5, None, None, None) == 0
        assert lib.b2f_counterfactual_device(eng._h, None, 5, 0, _cabi.ptr(w), 1, 0.5, None, None) == -1
        if eng.rank_words:
            with pytest.raises(B2FError, match=r"rc=-1\).*ranked"):
                eng.counterfactual_rows(enc.rank_rows(rows), [9])
        # 0 / 1 cutoffs are accepted
        for c in (0.0, 1.0):
            eng.counterfactual_rows(rows, [9], c)
    finally:
        eng.close()
    # a forest deeper than the walk stack
    blob = bytearray(flat.blob)
    blob[40:44] = np.uint32(33).tobytes()  # header max_depth
    try:
        deep = ForestEngine(bytes(blob), 0)
    except B2FError:
        return
    try:
        with pytest.raises(B2FError, match=r"rc=-1\).*depth"):
            deep.counterfactual_rows(rows, [9])
    finally:
        deep.close()


def test_categorical_flips_and_model(tmp_path, rf100d6, curated, adversarial):
    import httpx

    from databricks_kubernetes_mlops_poc_b200 import dependence
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline
    from databricks_kubernetes_mlops_poc_b200.model import load_model, save_model_dir
    from databricks_kubernetes_mlops_poc_b200.server import create_app
    from oracle import reference_pipeline as rp

    flat = flatten_pipeline(rf100d6)
    save_model_dir(str(tmp_path / "m"), flat)
    m = load_model(str(tmp_path / "m"))
    try:
        X = pd.concat([curated[rp.FEATURES].iloc[5000:5030], adversarial.iloc[:10]], ignore_index=True)
        out = m.counterfactuals(X, cutoff=0.3)
        assert out["feature_names"] == list(m.all_features) and out["output"] == "probability" and out["cutoff"] == 0.3
        assert np.array_equal(out["decisions"], out["predictions"] > 0.3)
        rows = m.encoder.encode_frame(X)
        words = [dependence.word_of(m.encoder, f) for f in rp.NUMERIC_FEATURES]
        proba, rec = m.engine.counterfactual_rows(rows, words, 0.3)
        assert np.array_equal(out["predictions"], proba)
        for f, cf in zip(out["feature_names"], out["counterfactuals"]):
            if f in rp.CATEGORICAL_FEATURES:
                vocab = list(flat.categories[rp.CATEGORICAL_FEATURES.index(f)])
                w = dependence.word_of(m.encoder, f)
                ice = m.engine.partial_dependence_rows(rows, [(w, 0, len(vocab))], np.arange(len(vocab), dtype=np.uint32))
                want = [[(vocab[c], float(ice[i, c])) for c in range(len(vocab)) if (ice[i, c] > 0.3) != (proba[i] > 0.3)] for i in range(len(X))]
                assert cf["flips"] == want, f
                codes = rows[:, w].view(np.int32)
                assert cf["value"] == [vocab[c] if c >= 0 else None for c in codes]
            else:
                k = rp.NUMERIC_FEATURES.index(f)
                assert _same(cf["lower"], rec["lower"][:, k]) and _same(cf["upper_prediction"], rec["upper_p1"][:, k])
        only_cat = m.counterfactuals(X, ["sex", "education"])
        assert np.array_equal(only_cat["predictions"], m.engine.counterfactual_rows(rows, [9])[0])
        for bad in (["nope"], ["age", "age"], []):
            with pytest.raises(ValueError):
                m.counterfactuals(X, bad)
        for c in (-0.1, 1.1, float("nan"), "0.5"):
            with pytest.raises(ValueError):
                m.counterfactuals(X, ["age"], cutoff=c)
        body = X.iloc[:30].to_dict(orient="records")
        direct = m.counterfactuals(X.iloc[:30], ["age", "sex"])

        async def main(queries):
            app = create_app(model=m)
            async with app.router.lifespan_context(app):
                async with httpx.AsyncClient(transport=httpx.ASGITransport(app=app), base_url="http://t") as c:
                    preds = [c.post("/predict", json=body) for _ in range(8)]
                    cfs = [c.post("/explain/counterfactual", params=q, json=body) for q in queries]
                    return await asyncio.gather(*cfs, *preds)

        queries = [[("feature", "age"), ("feature", "sex")], [], [("feature", "nope")], [("feature", "age"), ("feature", "age")],
                   [("cutoff", "x")], [("cutoff", "1.5")], [("cutoff", "nan")], [("feature", "age"), ("cutoff", "1")]]
        res = asyncio.run(main(queries))
        j = res[0].json()
        assert res[0].status_code == 200 and j["feature_names"] == ["age", "sex"] and j["cutoff"] == 0.5
        assert j["predictions"] == direct["predictions"].tolist() and j["decisions"] == direct["decisions"].tolist()
        age = j["counterfactuals"][0]
        assert age["feature"] == "age" and set(age) == {"feature", "value", "lower", "lower_prediction", "upper", "upper_prediction"}
        for k in ("value", "lower", "upper", "lower_prediction", "upper_prediction"):
            assert _same([np.nan if v is None else v for v in age[k]], direct["counterfactuals"][0][k]), k
        sex = j["counterfactuals"][1]
        assert sex["value"] == direct["counterfactuals"][1]["value"]
        assert sex["flips"] == [[[c, p] for c, p in row] for row in direct["counterfactuals"][1]["flips"]]
        assert res[1].status_code == 200 and len(res[1].json()["counterfactuals"]) == 23
        assert [r.status_code for r in res[2:7]] == [422] * 5
        last = res[7].json()["counterfactuals"][0]
        assert all(v is None for v in last["lower"] + last["upper"])  # nothing is above 1
        assert all(r.status_code == 200 for r in res[8:])
        # a returned boundary sent back as a request value reproduces the flip
        hit = [i for i, v in enumerate(age["upper"]) if v is not None]
        if hit:
            i = hit[0]
            row = dict(body[i], age=age["upper"][i])
            p = m.counterfactuals(pd.DataFrame([row]), ["age"])
            assert p["predictions"][0] == age["upper_prediction"][i] and p["decisions"][0] != j["decisions"][i]
    finally:
        m.close()
