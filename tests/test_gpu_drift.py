"""GPU parity for the batch drift detector (K3, SURVEY a7 / section 8f rank 2) through the C ABI (b2f_drift_*).

Oracle: ``oracle/drift.py`` -- alibi-detect 0.12.0's ``TabularDrift.feature_score`` restated on top of the real scipy
calls (``chi2_contingency``, ``ks_2samp(method="exact")``).  Bar: K-S D identical to the last bit of the integer
numerator, |dp| <= 1e-9 relative on float64 p-values, float32 response scores within 1e-6."""

import numpy as np
import pytest
from scipy import stats

pytestmark = pytest.mark.gpu

RTOL = 1e-9


def _detector(curated):
    from oracle import reference_pipeline as rp

    from databricks_kubernetes_mlops_poc_b200.drift import TabularDrift

    return TabularDrift(curated[rp.FEATURES], rp.CATEGORICAL_FEATURES, device=0)


def _check(det, ref, batch):
    from oracle import drift as od
    from oracle import reference_pipeline as rp

    p, stat, flags = det.statistics(batch)
    assert (flags == 0).all()
    for i, name in enumerate(rp.FEATURES):
        if name in rp.CATEGORICAL_FEATURES:
            a = ref[name].astype(str).to_numpy()
            x = batch[name].astype(str).to_numpy()
            union = sorted(set(a.tolist()) | set(x.tolist()))
            r = stats.chi2_contingency(np.array([[np.sum(a == v) for v in union], [np.sum(x == v) for v in union]]))
            assert abs(stat[i] - r[0]) <= 1e-10 * max(r[0], 1e-300), name
            assert abs(p[i] - r[1]) <= RTOL * max(r[1], 1e-300), name
        else:
            r = stats.ks_2samp(ref[name].to_numpy(float), batch[name].to_numpy(float), alternative="two-sided", method="exact")
            assert abs(stat[i] - r.statistic) <= 4e-16, name
            assert abs(p[i] - r.pvalue) <= RTOL * max(r.pvalue, 1e-300), (name, p[i], r.pvalue)
    want = od.drift_scores(ref, batch, rp.CATEGORICAL_FEATURES)
    got = det.score(batch)
    assert np.abs(np.asarray(got) - np.asarray(want)).max() <= 1e-6
    return p


def test_drift_matches_scipy(curated, inference):
    """Request-sized batches (1 .. 4096 rows) of the reference's own data, shifted data, the inference.csv rows."""
    from oracle import reference_pipeline as rp

    ref = curated[rp.FEATURES]
    det = _detector(curated)
    try:
        rng = np.random.default_rng(5)
        for n in (1, 2, 16, 81, 256, 1000, 4096):
            batch = ref.iloc[rng.integers(0, len(ref), n)].reset_index(drop=True)
            _check(det, ref, batch)
        _check(det, ref, inference[rp.FEATURES])
        shifted = ref.iloc[:500].copy()  # real drift: every numeric scaled, one category over-represented
        for name in rp.NUMERIC_FEATURES:
            shifted[name] = shifted[name] * 1.15 + 3.0
        shifted["sex"] = shifted["sex"].iloc[0]
        p = _check(det, ref, shifted)
        assert (p < 0.05).sum() >= 10
        assert det.launches >= 2 * 9
    finally:
        det.close()


def test_drift_edge_cases(curated):
    """Unseen categories (union columns), values outside the reference range, heavy ties, NaN, equal sample sizes."""
    from oracle import reference_pipeline as rp

    ref = curated[rp.FEATURES]
    det = _detector(curated)
    try:
        batch = ref.iloc[:64].copy().reset_index(drop=True)
        batch.loc[3, "sex"] = "unseen_value"
        batch.loc[4, "sex"] = "another_unseen"
        batch.loc[5, "education"] = "unseen_value"
        batch.loc[0, rp.NUMERIC_FEATURES[0]] = -1e12  # below every reference value
        batch.loc[1, rp.NUMERIC_FEATURES[0]] = 1e12   # above every reference value
        batch[rp.NUMERIC_FEATURES[1]] = float(np.median(ref[rp.NUMERIC_FEATURES[1]]))  # one value, all ties
        _check(det, ref, batch)
        same = ref.iloc[:1].copy()
        _check(det, ref, same)
        nan = ref.iloc[:10].copy().reset_index(drop=True)
        nan.loc[2, rp.NUMERIC_FEATURES[3]] = np.nan
        p, _, flags = det.statistics(nan)
        k = rp.FEATURES.index(rp.NUMERIC_FEATURES[3])
        assert flags[k] == 2 and np.isnan(p[k]) and np.isfinite(np.delete(p, k)).all()
        with pytest.raises(ValueError):
            det.statistics(ref.iloc[:0])
    finally:
        det.close()
    # a small reference: equal sizes (scipy's other closed form), batch larger than the reference, wide bands
    from databricks_kubernetes_mlops_poc_b200.drift import TabularDrift

    small = ref.iloc[:300].reset_index(drop=True)
    det = TabularDrift(small, rp.CATEGORICAL_FEATURES, device=0)
    try:
        for batch in (ref.iloc[300:600], ref.iloc[1000:3500], ref.iloc[5000:5007]):
            _check(det, small, batch.reset_index(drop=True))
        far = ref.iloc[300:900].copy().reset_index(drop=True)
        far[rp.NUMERIC_FEATURES[0]] = far[rp.NUMERIC_FEATURES[0]] + 1e9  # D = 1: the band is the whole lattice
        _check(det, small, far)
    finally:
        det.close()


def test_drift_large_batches(curated):
    """BASELINE's largest batch (65 536 rows, larger than the reference): ~95 000 anti-diagonals, rings of
    hundreds of slots; and a batch size where scipy itself falls back to the asymptotic formula."""
    from oracle import reference_pipeline as rp

    from databricks_kubernetes_mlops_poc_b200 import training

    ref = curated[rp.FEATURES]
    det = _detector(curated)
    try:
        rng = np.random.default_rng(9)
        batch = ref.iloc[rng.integers(0, len(ref), 65536)].reset_index(drop=True)
        _check(det, ref, batch)
        assert det.last_device_ms > 0
        # a band too wide for the shared-memory ring (D * mn/(m+n) > ~2045): the sweep keeps its rings in global memory
        from databricks_kubernetes_mlops_poc_b200.drift import TabularDrift

        one = TabularDrift(ref[[rp.NUMERIC_FEATURES[0]]], [], device=0)
        try:
            col = ref[[rp.NUMERIC_FEATURES[0]]]
            moved = col.iloc[rng.integers(0, len(ref), 40000)].reset_index(drop=True) * 1.5 + 20000.0
            r = stats.ks_2samp(col.iloc[:, 0].to_numpy(float), moved.iloc[:, 0].to_numpy(float), alternative="two-sided", method="exact")
            p1, s1, f1 = one.statistics(moved)
            assert f1[0] == 0 and abs(s1[0] - r.statistic) <= 4e-16 and r.statistic > 0.1
            assert abs(p1[0] - r.pvalue) <= RTOL * max(r.pvalue, 1e-300), (p1[0], r.pvalue)
        finally:
            one.close()
        odd = ref.iloc[rng.integers(0, len(ref), 99991)].reset_index(drop=True)  # 30000 * 99991 / gcd >= 2^31
        p, stat, flags = det.statistics(odd)
        for i, name in enumerate(rp.FEATURES):
            if name in rp.NUMERIC_FEATURES:
                assert flags[i] == 1
                with pytest.warns(RuntimeWarning):
                    r = stats.ks_2samp(ref[name].to_numpy(float), odd[name].to_numpy(float), alternative="two-sided", method="exact")
                assert abs(stat[i] - r.statistic) <= 4e-16 and abs(p[i] - r.pvalue) <= 1e-12 + RTOL * r.pvalue
    finally:
        det.close()


def test_model_predict_drift(curated, inference, rf100d6, tmp_path):
    """Plugin level: ``B200Model.predict`` carries the GPU drift scores; the artefact directory round-trips."""
    from oracle import drift as od
    from oracle import reference_pipeline as rp

    from databricks_kubernetes_mlops_poc_b200 import flatten, load_model
    from databricks_kubernetes_mlops_poc_b200.model import B200Model, save_model_dir

    ref = curated[rp.FEATURES]
    m = B200Model.from_pipeline(rf100d6, reference_frame=curated, devices=[0])
    try:
        for df in (ref.iloc[:64], inference):
            got = m.predict(df)["feature_drift_batch"]
            want = od.drift_scores(ref, df[rp.FEATURES], rp.CATEGORICAL_FEATURES)
            assert list(got) == rp.FEATURES
            assert np.abs(np.asarray(list(got.values())) - np.asarray(want)).max() <= 1e-6
    finally:
        m.close()
    save_model_dir(str(tmp_path), flatten.flatten_pipeline(rf100d6), reference_frame=curated)
    m2 = load_model(str(tmp_path))
    try:
        got = m2.predict(ref.iloc[100:200])["feature_drift_batch"]
        want = od.drift_scores(ref, ref.iloc[100:200], rp.CATEGORICAL_FEATURES)
        assert np.abs(np.asarray(list(got.values())) - np.asarray(want)).max() <= 1e-6
    finally:
        m2.close()


def test_drift_against_frozen_library_outputs(curated, inference):
    """The GPU detector against tests/golden/expected_detectors.npz (scipy outputs frozen by make_golden_detectors.py)."""
    import importlib.util
    import os

    from oracle import datasets
    from oracle import reference_pipeline as rp

    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_golden_detectors.py")
    spec = importlib.util.spec_from_file_location("make_golden_detectors", here)
    mg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mg)
    exp = datasets.load_expected("detectors")
    det = _detector(curated)
    try:
        for key, batch in mg.drift_batches(curated, inference).items():
            p, stat, flags = det.statistics(batch)
            assert (flags == 0).all()
            want_p, want_s = exp[f"drift_p_{key}"], exp[f"drift_stat_{key}"]
            assert (np.abs(stat - want_s) <= 1e-10 * np.abs(want_s) + 4e-16).all(), key
            assert (np.abs(p - want_p) <= RTOL * want_p + 1e-300).all(), key
    finally:
        det.close()


def test_row_scan_and_sweep_agree(curated):
    """Request-sized batches take a row-scan form of the exact p-value -- the row resident in shared memory (2 .. 1024 rows, band
    narrower than the ring), else through the global scratch (2 .. 48 rows) -- larger ones the anti-diagonal sweep; the same
    batches through all three forms give the same p-values, feature by feature, and each run equals scipy's."""
    import os

    from oracle import reference_pipeline as rp

    from databricks_kubernetes_mlops_poc_b200.drift import TabularDrift

    ref = curated[rp.FEATURES]
    rng = np.random.default_rng(11)
    batches = [ref.iloc[rng.integers(0, len(ref), n)].reset_index(drop=True) for n in (2, 3, 16, 17, 48, 64, 127, 128, 250, 600, 1000, 1024)]
    shifted = ref.iloc[:40].copy()
    for c in rp.NUMERIC_FEATURES:
        shifted[c] = shifted[c] * 1.7 + 3.0  # wide bands: some features leave the shared-memory ring
    batches.append(shifted)
    slightly = ref.iloc[1000:1300].copy()
    for c in rp.NUMERIC_FEATURES:
        slightly[c] = slightly[c] * 1.02
    batches.append(slightly)
    det = TabularDrift(ref, rp.CATEGORICAL_FEATURES, device=0)  # shared-memory row scan up to 448 rows, sweep beyond
    try:
        a = [det.statistics(b) for b in batches]
        for b in batches:
            _check(det, ref, b)
    finally:
        det.close()
    for env in ({"B2F_DRIFT_ROWSCAN": "0"}, {"B2F_DRIFT_ROWSCAN_SMEM": "0"}, {"B2F_DRIFT_ROWSCAN_SMEM": "1024"}):
        os.environ.update(env)
        try:
            det = TabularDrift(ref, rp.CATEGORICAL_FEATURES, device=0)
        finally:
            for k in env:
                os.environ.pop(k)
        try:
            for b, (p, stat, flags) in zip(batches, a):
                p2, stat2, flags2 = det.statistics(b)
                assert (flags == flags2).all() and (stat == stat2).all()
                assert (np.abs(p - p2) <= 1e-11 * np.maximum(np.abs(p), 1e-300)).all(), (env, len(b))  # feature by feature
                _check(det, ref, b)
        finally:
            det.close()
