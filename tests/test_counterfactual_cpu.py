"""Counterfactuals on the CPU: ``b2f_blob_split_values`` against the split values of scikit-learn's own trees on every
forest shape (and against the ranker's tables where there is one), and the numpy emulator of K7
(tests/counterfactual_walk.py) against scikit-learn's ``predict_proba`` on every substituted row, with its lower / upper
against a brute-force scan of those scores."""

import numpy as np
import pandas as pd
import pytest

import schema_zoo as sz
from counterfactual_walk import imputed, piece_scores, reduce, representatives, split_values

TOL = 1e-12
CUTOFFS = (0.0, 0.3, 0.5, 1.0)


def _sk_split_values(pipe, n_cat_cols: int, k: int) -> np.ndarray:
    """Sorted distinct nextup(floor32(threshold)) of numeric feature k over the pipeline's trees."""
    from oracle import treewalk as tw

    dump = tw.dump_pipeline(pipe)
    n_ohe = int(dump["cat_offsets"][-1])
    thr = dump["threshold"][(dump["left"] != -1) & (dump["feature"] == n_ohe + k)].astype(np.float64)
    t32 = thr.astype(np.float32)
    over = t32.astype(np.float64) > thr
    t32[over] = np.nextafter(t32[over], np.float32(-np.inf))  # floor32
    return np.unique(np.nextafter(t32, np.float32(np.inf)))


def _ranker_tables(blob: bytes, n_num: int):
    """The ranker's split-value tables (b2f_ranker_thresholds), or None when the forest has no rank layout."""
    import ctypes as C

    from databricks_kubernetes_mlops_poc_b200 import _cabi

    lib = _cabi.load_library()
    buf = np.frombuffer(blob, dtype=np.uint8)
    r = lib.b2f_ranker_create(_cabi.ptr(buf), buf.size)
    try:
        info = _cabi.RankInfo()
        assert lib.b2f_ranker_info(r, C.byref(info)) == 0
        if not info.ok:
            return None
        out = []
        for k in range(n_num):
            cnt = C.c_int32(0)
            p = lib.b2f_ranker_thresholds(r, k, C.byref(cnt))
            out.append(np.ctypeslib.as_array(p, (cnt.value,)).copy() if cnt.value else np.empty(0, np.float32))
        return out
    finally:
        lib.b2f_ranker_destroy(r)


def _check_split_values(pipe) -> bool:
    """b2f_blob_split_values == sklearn's == the emulator's for every numeric word; == the ranker's tables where the forest
    has a rank layout.  -> whether it has one."""
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.engine import blob_split_values
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline

    flat = flatten_pipeline(pipe)
    enc = RowEncoder(flat)
    ranked = _ranker_tables(flat.blob, enc.n_num)
    for k in range(enc.n_num):
        got = blob_split_values(flat.blob, enc.n_cat + k)
        assert np.array_equal(got, _sk_split_values(pipe, enc.n_cat, k)), enc.num_features[k]
        assert np.array_equal(split_values(flat.blob, enc.n_cat + k), got)
        if ranked is not None:
            assert np.array_equal(ranked[k], got)
    return ranked is not None


@pytest.mark.parametrize("which", ["rf100d6", "rf500d8", "gbdt_small", "deep24"])
def test_split_values_match_sklearn(which, request, curated):
    from oracle import reference_pipeline as rp

    if which == "deep24":
        pipe = rp.fit_reference_pipeline(curated.iloc[:6000], dict(n_estimators=37, max_depth=24, criterion="entropy", random_state=1))
    else:
        pipe = request.getfixturevalue(which)
    assert _check_split_values(pipe) == (which != "deep24")


@pytest.mark.parametrize("name", ["packed_wide", "packed_wide_gbdt", "tiny", "tiny_gbdt", "over16"])
def test_split_values_schema_zoo(name):
    _, pipe = sz.fitted(name)
    _check_split_values(pipe)


def test_split_values_errors(rf100d6):
    from databricks_kubernetes_mlops_poc_b200 import _cabi
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline

    lib = _cabi.load_library()
    flat = flatten_pipeline(rf100d6)
    buf = np.frombuffer(flat.blob, dtype=np.uint8)
    n_cat = len(flat.cat_features)
    for word in (-1, 0, n_cat - 1, n_cat + len(flat.num_features), 23):
        assert lib.b2f_blob_split_values(_cabi.ptr(buf), buf.size, word, None, 0) == -1
    assert lib.b2f_blob_split_values(_cabi.ptr(buf), buf.size - 8, n_cat, None, 0) == -1
    total = lib.b2f_blob_split_values(_cabi.ptr(buf), buf.size, n_cat, None, 0)
    part = np.zeros(5, np.float32)
    assert lib.b2f_blob_split_values(_cabi.ptr(buf), buf.size, n_cat, _cabi.ptr(part), 5) == total > 5
    assert np.array_equal(part, _sk_split_values(rf100d6, n_cat, 0)[:5])


def _brute_force(pipe, X: pd.DataFrame, field: str, reps: np.ndarray) -> np.ndarray:
    """sklearn's P(class 1) of every row of X with ``field`` set to each representative: (n, len(reps))."""
    big = X.loc[X.index.repeat(len(reps))].reset_index(drop=True)
    big[field] = np.tile(reps.astype(np.float64), len(X))
    return pipe.predict_proba(big)[:, 1].reshape(len(X), len(reps))


def _scan(p: np.ndarray, j: int, cutoff: float):
    """Nearest pieces below and above j whose decision differs from piece j's, by walking outwards (None = none)."""
    d = p[j] > cutoff
    lo = next((k for k in range(j - 1, -1, -1) if (p[k] > cutoff) != d), None)
    hi = next((k for k in range(j + 1, len(p)) if (p[k] > cutoff) != d), None)
    return lo, hi


def _emulator_agrees(pipe, X: pd.DataFrame, fields, numeric_features):
    """Emulated piece scores equal sklearn's to 1e-12; the reduction's lower / upper equal the brute-force scan wherever no
    sklearn score sits within 1e-12 of the cutoff.  -> number of (row, field, cutoff) cases with a flip."""
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_pipeline

    flat = flatten_pipeline(pipe)
    enc = RowEncoder(flat)
    rows = enc.encode_frame(X)
    flips = 0
    for field in fields:
        w = enc.n_cat + enc.num_features.index(field)
        t, p = piece_scores(flat.blob, rows, w)
        want = _brute_force(pipe, X, field, representatives(t))
        assert np.abs(p - want).max() <= TOL, field
        x = imputed(flat.blob, rows)[:, w]
        j = np.searchsorted(t, x, side="right")
        for cutoff in CUTOFFS:
            pj, lo, plo, hi, phi = reduce(t, p, x, cutoff)
            assert np.array_equal(pj, p[np.arange(len(x)), j])
            for i in range(len(x)):
                if np.abs(want[i] - cutoff).min() <= TOL:
                    continue  # a tie at the cutoff: sklearn's rounding may decide otherwise
                klo, khi = _scan(want[i], j[i], cutoff)
                if klo is None:
                    assert np.isnan(lo[i]) and np.isnan(plo[i])
                else:
                    assert lo[i] == np.nextafter(t[klo], np.float32(-np.inf)) and plo[i] == p[i, klo]
                    assert lo[i] < x[i] and (p[i, klo] > cutoff) != (pj[i] > cutoff)
                if khi is None:
                    assert np.isnan(hi[i]) and np.isnan(phi[i])
                else:
                    assert hi[i] == t[khi - 1] and phi[i] == p[i, khi] and hi[i] > x[i]
                flips += (klo is not None) + (khi is not None)
    return flips


def test_emulator_rf100d6(rf100d6, curated, adversarial):
    from oracle import reference_pipeline as rp

    X = pd.concat([curated[rp.FEATURES].iloc[20000:20016], adversarial.iloc[:24]], ignore_index=True)
    fields = ["credit_limit", "age", "bill_amount_1", "payment_amount_1", "payment_amount_2"]
    assert _emulator_agrees(rf100d6, X, fields, rp.NUMERIC_FEATURES) > 0


def test_emulator_gbdt_and_zoo(gbdt_small, curated, adversarial):
    from oracle import reference_pipeline as rp

    X = pd.concat([curated[rp.FEATURES].iloc[9000:9010], adversarial.iloc[30:40]], ignore_index=True)
    assert _emulator_agrees(gbdt_small, X, rp.NUMERIC_FEATURES[:3], rp.NUMERIC_FEATURES) > 0
    spec, pipe = sz.fitted("tiny")
    X = pd.concat([sz.edge_rows(spec, pipe, n=12), sz.make_frame(spec, 12, seed=9, target=False)], ignore_index=True)
    _emulator_agrees(pipe, X, sz.num_names(spec), sz.num_names(spec))
