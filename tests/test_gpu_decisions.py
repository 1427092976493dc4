"""Every decision boundary on the GPU: class labels at exact and near ties, and outlier flags at their threshold.

Each kernel turns a float64 sum of leaf payloads into a decision in ``aggregate()`` (``csrc/forest_predict.cuh``), and
each adds the payloads in its own order.  The models of ``tests/decision_models.py`` put rows on the boundary; they go
through the warp, tile and split kernels, the rank kernel (resident and streamed), batch sizes 1 to 90 000 with the
boundary rows at several positions, float64 and float32 outputs, ``{proba, label}`` and full records, the stream dealer
and ``B200Model``.  What must hold:

* exact ties (dyadic payloads, every order exact): every label is sklearn's (class 0) and ``p1 == 0.5``;
* near ties: every label is the exact sign of ``sum p1 - sum p0``, so one row gets one label from every path and batch;
* outside the rounding band every label is sklearn's;
* GBDT ``raw == 0`` (and ``0 < raw <= 5.6e-17``): label 1, ``p1 == 0.5``;
* outlier flags equal sklearn's at, one ulp above and one ulp below a score many rows share, float32 as float64."""

import os
from contextlib import contextmanager

import numpy as np
import pytest

import decision_models as dm

pytestmark = pytest.mark.gpu

SIZES = (1, 33, 4096, 65536, 90000)


@contextmanager
def _env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    try:
        for k, v in kv.items():
            os.environ[k] = v
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def base(curated):
    from oracle import reference_pipeline as rp

    return curated[rp.FEATURES].iloc[3000:9000].reset_index(drop=True)


def _placements(boundary: np.ndarray, n_base: int, seed: int):
    """Per batch size, an index array into the base rows: boundary rows first, last and in the middle, the rest permuted."""
    rng = np.random.default_rng(seed)
    out = []
    for n in SIZES:
        if n == 1:
            out.append(boundary[:1])
            continue
        idx = rng.permutation(np.resize(rng.permutation(n_base), n))
        picks = rng.choice(boundary, size=min(8, boundary.size), replace=False)
        for k, pos in enumerate([0, n - 1, n // 2, n // 3, 32 % n, 31 % n, (n // 2) | 31, n - 33]):
            if k < picks.size and 0 <= pos < n:
                idx[pos] = picks[k]
        out.append(idx)
    return out


def _every_path(pipe, base, placements, *, iforest=None):
    """Yield (path name, index array, label, p1) for every scoring path and batch."""
    from databricks_kubernetes_mlops_poc_b200 import flatten
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.engine import EngineGroup, ForestEngine
    from databricks_kubernetes_mlops_poc_b200.model import B200Model

    flat = flatten.flatten_pipeline(pipe)
    enc = RowEncoder(flat)
    rows = enc.encode_frame(base)
    iso_blob = flatten.flatten_isolation_forest(iforest, 9, 14, threshold=0.0) if iforest is not None else None

    for kernel in ("warp", "tile", "split"):
        with _env(B2F_KERNEL=kernel):
            eng = ForestEngine(flat, 0)
        try:
            if iso_blob is not None:
                eng.attach_outlier_forest(iso_blob)
            for idx in placements:
                if kernel == "split" and idx.size > 4096:
                    continue
                r = rows[idx]
                pk = enc.pack_rows(r)
                for name, rr in (("rows96", r), ("packed", pk)):
                    p, lab = eng.predict_rows(rr, np.float64)
                    yield f"{kernel}/{name}/f64", idx, lab, p
                    p32, lab32 = eng.predict_rows(rr, np.float32)
                    yield f"{kernel}/{name}/f32", idx, lab32, p32.astype(np.float64)
                out = eng.predict_pairs(pk)
                yield f"{kernel}/pairs", idx, out["label"], out["proba1"].astype(np.float64)
                if iso_blob is not None:
                    full = eng.predict_full(pk)
                    yield f"{kernel}/full", idx, full["label"], full["proba1"]
            info = eng.info()
            assert info["launches"] > 0 and info["launches_rank"] == 0
            if kernel in ("tile", "split"):
                assert info[f"launches_{kernel}"] > 0
        finally:
            eng.close()

    # ranked rows: resident (up to 288 trees, whose top levels ride in the kernel parameters) and streamed
    for stream in ("0", "1"):
        with _env(B2F_RANK_STREAM=stream):
            eng = ForestEngine(flat, 0)
        try:
            info = eng.info()
            if stream == "0" and flat.n_trees > 288:
                assert not info["rank_ok"]  # resident forced but impossible: no rank kernel
                continue
            assert info["rank_ok"] and info["rank_stream"] == (stream == "1")
            kind = "rank/stream" if info["rank_stream"] else "rank/resident"
            l0 = info["launches_rank"]
            for idx in placements:
                rk = enc.rank_rows(rows[idx])
                p, lab = eng.predict_rows(rk, np.float64)
                yield f"{kind}/f64", idx, lab, p
                p32, lab32 = eng.predict_rows(rk, np.float32)
                yield f"{kind}/f32", idx, lab32, p32.astype(np.float64)
            assert eng.info()["launches_rank"] > l0
        finally:
            eng.close()

    # the stream dealer over two replicas on GPU 0
    grp = EngineGroup(flat, devices=[0, 0])
    try:
        idx = placements[-1]
        pk = enc.pack_rows(rows[idx])
        p = np.full(idx.size, -1, dtype=np.float64)
        lab = np.full(idx.size, -1, dtype=np.int32)
        grp.predict_stream(pk, 4096, p, lab)
        yield "stream", idx, lab, p
    finally:
        grp.close()

    # the plugin: predict_label (staged path) and predict (columnar scorer)
    m = B200Model.from_pipeline(pipe, devices=[0])
    try:
        for idx in placements:
            frame = base.iloc[idx]
            lab = np.asarray(m.predict_label(frame)).astype(np.int32)
            p = np.asarray(m.predict(frame)["predictions"], dtype=np.float64)
            yield "model", idx, lab, p
    finally:
        m.close()


def _check_rf(pipe, base, n_trees, *, iforest=None):
    """Every path and batch: every label is the exact sign (so one row gets one label everywhere), sklearn's outside the
    rounding band; with dyadic payloads every tie scores 0.5 in float64."""
    from oracle import reference_pipeline as rp

    p0, p1 = dm.leaf_terms(pipe, base)
    margin = dm.exact_margin(p0, p1)
    exact = dm.exact_labels(p0, p1)
    near = np.abs(margin) <= dm.band(n_trees)
    dyadic = (p1 * 4 == np.round(p1 * 4)).all()  # every summation order is exact: a tie scores 0.5 everywhere
    dyadic_tie = (margin == 0.0) & dyadic
    want_p, want_l = rp.oracle_predict(pipe, base)
    assert near.any()
    paths = set()
    for name, idx, lab, p in _every_path(pipe, base, _placements(np.nonzero(near)[0], len(base), n_trees), iforest=iforest):
        paths.add("/".join(name.split("/")[:2]) if name.startswith("rank") else name.split("/")[0])
        bad = lab != exact[idx]
        assert not bad.any(), f"{name} n={idx.size}: rows {np.unique(idx[bad])[:6]} differ from the exact sign"
        out = ~near[idx]
        assert (lab[out] == want_l[idx][out]).all(), name
        if not name.endswith("f32") and not name.endswith("pairs"):
            assert np.abs(p - want_p[idx]).max() <= 1e-12, name
            assert (p[dyadic_tie[idx]] == 0.5).all(), name
    want_paths = {"warp", "tile", "split", "rank/stream", "stream", "model"} | ({"rank/resident"} if n_trees <= 288 else set())
    assert want_paths <= paths, want_paths - paths


@pytest.mark.parametrize("n_trees", [2, 4, 100, 290])
def test_rf_exact_ties(curated, base, n_trees):
    """Dyadic payloads: sums are exact in every kernel, ties go to class 0 as in sklearn."""
    pipe = dm.rf_exact_ties(curated, n_trees)
    p0, p1 = dm.leaf_terms(pipe, base)
    tie = dm.exact_margin(p0, p1) == 0.0
    assert tie.sum() >= 50 and (pipe.predict(base)[tie] == 0).all()
    _check_rf(pipe, base, n_trees)


@pytest.mark.parametrize("n_trees", [4, 100, 290])
def test_rf_near_ties(curated, base, iforest, n_trees):
    """Payloads a few ulps off a tie, whose float64 sum depends on the order: every path and batch size gives the exact
    sign, re-decided on the device for rows inside the rounding band."""
    pipe = dm.rf_near_ties(curated, n_trees)
    _check_rf(pipe, base, n_trees, iforest=iforest if n_trees == 100 else None)


def test_rf_outside_band(base, rf100d6, rf500d8):
    """A fitted forest nobody edited: every row is outside the band, every label is sklearn's on every path."""
    from oracle import reference_pipeline as rp

    for pipe, t in ((rf100d6, 100), (rf500d8, 500)):
        want_p, want_l = rp.oracle_predict(pipe, base)
        placements = _placements(np.arange(len(base)), len(base), t)
        for name, idx, lab, p in _every_path(pipe, base, placements):
            assert (lab == want_l[idx]).all(), name
            if not name.endswith("f32") and not name.endswith("pairs"):
                assert np.abs(p - want_p[idx]).max() <= 1e-12, name


def test_gbdt_raw_zero(curated, base):
    """raw == 0 and 0 < raw <= 5.6e-17: label 1 with p1 == 0.5 in every path; the counterfactual decision at cutoff
    0.5 is ``p1 > 0.5`` (False) there, as its docstring says."""
    from databricks_kubernetes_mlops_poc_b200.model import B200Model

    pipe = dm.gbdt_zero_raw(curated)
    _, terms = dm.leaf_terms(pipe, base)
    raw = dm.exact_margin(None, terms)
    edge = (raw == 0.0) | ((raw > 0.0) & (raw <= 5.6e-17))
    assert edge.sum() >= 20
    want = dm.exact_labels(None, terms)
    assert (pipe.predict(base) == want).all()
    placements = _placements(np.nonzero(edge)[0], len(base), 7)
    for name, idx, lab, p in _every_path(pipe, base, placements):
        assert (lab == want[idx]).all(), name
        e = edge[idx]
        assert (lab[e] == 1).all() and (p[e] == 0.5).all(), name

    m = B200Model.from_pipeline(pipe, devices=[0])
    try:
        frame = base.iloc[np.nonzero(edge)[0][:64]]
        cf = m.counterfactuals(frame, features=["credit_limit"], cutoff=0.5)
        pred = np.asarray(cf["predictions"])
        assert (pred == 0.5).all()
        assert (np.asarray(cf["decisions"]) == (pred > 0.5)).all() and not np.asarray(cf["decisions"]).any()
        assert (m.predict_label(frame) == 1).all()  # the label and the counterfactual decision part here, by design
    finally:
        m.close()


def test_trust_labels_are_predict_labels(curated, base):
    """``trust_score``'s labels are ``predict_label``'s, tie rows (class 0) included."""
    from oracle import reference_pipeline as rp

    from databricks_kubernetes_mlops_poc_b200.model import B200Model

    pipe = dm.rf_exact_ties(curated, 100)
    p0, p1 = dm.leaf_terms(pipe, base)
    tie = np.nonzero(dm.exact_margin(p0, p1) == 0.0)[0]
    frame = base.iloc[np.concatenate([tie, np.arange(200)])]
    m = B200Model.from_pipeline(pipe, devices=[0])
    try:
        m.attach_trust_reference(curated[rp.FEATURES + [rp.TARGET]].iloc[:2000])
        got = m.trust_score(frame)
        assert (np.asarray(got["labels"]) == m.predict_label(frame)).all()
        assert (np.asarray(got["labels"])[: tie.size] == 0).all()
    finally:
        m.close()


def _outlier_setup(curated, iforest, rf100d6, split=False):
    """-> (classifier flat, encoder, encoded rows, sklearn's scores of those rows, a score many curated rows share).  The
    split kernel gets the first 4 096 rows plus every row at the shared score."""
    from oracle import reference_pipeline as rp

    from databricks_kubernetes_mlops_poc_b200 import flatten
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder

    score_all = -iforest.decision_function(curated[rp.NUMERIC_FEATURES].to_numpy())
    thr0 = dm.shared_outlier_score(score_all)
    at = np.nonzero(score_all == thr0)[0]
    idx = np.union1d(np.arange(4096), at) if split else np.arange(len(curated))
    flat = flatten.flatten_pipeline(rf100d6)
    enc = RowEncoder(flat)
    return flat, enc, enc.encode_frame(curated[rp.FEATURES].iloc[idx]), score_all[idx], thr0


@pytest.mark.parametrize("kernel", ["warp", "tile", "split"])
def test_outlier_flag_at_threshold(curated, iforest, rf100d6, kernel):
    """Threshold = a score many rows share, and one ulp either side: every flag is sklearn's ``score > thr`` in float64,
    float32 and full records."""
    from databricks_kubernetes_mlops_poc_b200 import flatten
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine

    flat, enc, rows, score, thr0 = _outlier_setup(curated, iforest, rf100d6, split=kernel == "split")
    assert (score == thr0).sum() >= 20
    for thr in (thr0, float(np.nextafter(thr0, np.inf)), float(np.nextafter(thr0, -np.inf))):
        want = score > thr
        blob = flatten.flatten_isolation_forest(iforest, 9, 14, threshold=thr)
        with _env(B2F_KERNEL=kernel):
            eng = ForestEngine(blob, 0)
            cls = ForestEngine(flat, 0)
        try:
            cls.attach_outlier_forest(blob)
            full = cls.predict_full(enc.pack_rows(rows))["is_outlier"]
            assert (full == want).all(), f"thr={thr!r} full: {int((full != want).sum())} flags differ"
            for fmt, r in (("rows96", rows), ("packed", enc.pack_rows(rows))):
                s64, f64 = eng.predict_rows(r, np.float64)
                _, f32 = eng.predict_rows(r, np.float32)
                assert (f64 == want).all(), f"thr={thr!r} {fmt}: {int((f64 != want).sum())} flags differ"
                assert (f32 == want).all()
                assert np.abs(s64 - score).max() <= 1e-12
        finally:
            eng.close()
            cls.close()


def test_model_outlier_flags_at_threshold(curated, iforest, rf100d6):
    """``B200Model.predict`` (columnar scorer) and the per-GPU replica path at the shared-score threshold: sklearn's flag on
    every row, whatever the batch."""
    from oracle import reference_pipeline as rp

    from databricks_kubernetes_mlops_poc_b200.model import B200Model

    df = curated[rp.FEATURES]
    score = -iforest.decision_function(df[rp.NUMERIC_FEATURES].to_numpy())
    thr = dm.shared_outlier_score(score)
    at = np.nonzero(score == thr)[0]
    m = B200Model.from_pipeline(rf100d6, devices=[0], outlier=iforest, outlier_threshold=thr)
    try:
        want = score > thr
        assert (np.asarray(m.predict(df)["outliers"]) == want).all()
        for frame_idx in (at[:1], at, np.concatenate([np.arange(33), at])):
            frame = df.iloc[frame_idx]
            assert (np.asarray(m.predict(frame)["outliers"]) == want[frame_idx]).all()
            _, flags = m.replicas[0].score(frame)
            assert (flags == want[frame_idx]).all()
    finally:
        m.close()


@pytest.mark.parametrize("kernel", ["warp", "tile"])
def test_smaller_forest_later_keeps_earlier_launches_working(curated, rf100d6, kernel):
    """The dynamic shared-memory limit of a kernel is shared by every model of the process: creating an engine for a
    smaller forest must not break the launches of one created before it."""
    from oracle import reference_pipeline as rp

    from databricks_kubernetes_mlops_poc_b200 import flatten
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine

    big = flatten.flatten_pipeline(rf100d6)
    small = flatten.flatten_pipeline(dm.fit_rf(curated, 4, depth=3))
    frame = curated[rp.FEATURES].iloc[:4096]
    rows = RowEncoder(big).encode_frame(frame)
    with _env(B2F_KERNEL=kernel):
        first = ForestEngine(big, 0)
        second = ForestEngine(small, 0)
    try:
        want_p, want_l = rp.oracle_predict(rf100d6, frame)
        p, lab = first.predict_rows(rows, np.float64)
        assert np.abs(p - want_p).max() <= 1e-12 and (lab == want_l).all()
        second.predict_rows(RowEncoder(small).encode_frame(frame), np.float64)
    finally:
        first.close()
        second.close()
