"""Every form of the drift detector's exact K-S p-value, and the chi-squared edges, against scipy -- feature by feature.

``k_drift_finish`` picks one of several forms per numeric feature from (n_ref, n, D): p = 1 at h = 0, the asymptotic
branch (flag 1), the n = 1 closed form, the shared-memory and global-scratch row scans, the anti-diagonal sweep in one warp
(ring 32) or ``sweep_block<1|2|4>``, and ``sweep_wide`` for bands wider than the shared-memory ring.  Synthetic frames are
built per (n_ref, n) so that their columns land in each form that pair can reach (``drift_walk.route`` mirrors the router);
every case runs under the default limits and under ``B2F_DRIFT_ROWSCAN=0`` / ``B2F_DRIFT_ROWSCAN_SMEM=0`` /
``B2F_DRIFT_ROWSCAN_SMEM=1024``, and every feature of every run is compared with ``scipy.stats.ks_2samp(method="exact")``:
D to 4e-16, p to 1e-9 relative, flags exact."""

import functools
import math
import os

import numpy as np
import pandas as pd
import pytest
from scipy import stats

import drift_walk as dw

RTOL = 1e-9
ENVS = ({}, {"B2F_DRIFT_ROWSCAN": "0"}, {"B2F_DRIFT_ROWSCAN_SMEM": "0"}, {"B2F_DRIFT_ROWSCAN_SMEM": "1024"})
NREF = (1, 2, 31, 1023, 1024, 1025, 4096, 30000, 30011, 200000)
NB = (1, 2, 3, 47, 48, 49, 447, 448, 449, 1024, 1025, 4096, 65536, 200000)


def _affordable(r, b):
    """scipy's exact method costs ~ max * band: large unequal pairs only where one size divides the other"""
    lo, hi = min(r, b), max(r, b)
    return hi <= 4096 or lo <= 1025 and hi <= 30011 or r == b or hi % lo == 0 or (r, b) in ((30000, 4096), (30011, 4096), (30000, 65536))


PAIRS = [(r, b) for r in NREF for b in NB if _affordable(r, b)] + [(30000, 30000), (30000, 71581), (30000, 71587)]


def _widths(r, b):
    """target sweep widths 2 D mn/(m+n): ring 32, NS = 1, 2, 4, the wide form -- and D = 0.5, 1 where the lattice is small"""
    eff = r * b / (r + b)
    ds = [w / (2 * eff) for w in (20, 500, 1500, 3000, 5000)]
    if max(r, b) <= 4096:
        ds += [0.5, 1.0]
    if (r, b) == (30000, 30000):
        ds.append(0.1421)  # scipy: 1.6e-264; the kernel once returned 0 here
    if (r, b) == (30000, 65536):
        ds = [d for d in ds if d <= 0.11]  # scipy's cost grows with the band
    return sorted({min(d, 1.0) for d in ds if d <= 1.0})


def _column(rng, r, b, d_target, ties):
    """(reference, batch) of one numeric feature with K-S D close to d_target: the batch is the reference's distribution
    shifted, the shift found by bisection on the exact integer numerator"""
    ref = rng.normal(size=r)
    base = rng.normal(size=b)
    if ties:
        ref, base = np.round(ref * 4) / 4, np.round(base * 4) / 4
    ref = np.sort(ref)
    lo, hi = 0.0, 50.0
    for _ in range(40):
        mid = 0.5 * (lo + hi)
        if dw.ks_numerator(ref, base + mid) / (r * b) < d_target:
            lo = mid
        else:
            hi = mid
    x = base + hi
    if ties:
        x = np.round(x * 4) / 4
    return ref, x


@functools.lru_cache(maxsize=None)
def _case(r, b):
    """-> (reference frame, batch frame): one numeric column per target D (tied values on every other one), one at D ~ 0
    (the batch drawn like the reference), and one categorical column"""
    rng = np.random.default_rng(r * 7919 + b)
    ref_cols, x_cols = {}, {}
    for k, d in enumerate([0.0] + _widths(r, b)):
        rc, xc = _column(rng, r, b, d, ties=bool(k % 2)) if d > 0 else (np.sort(rng.normal(size=r)), rng.normal(size=b))
        ref_cols[f"x{k}"], x_cols[f"x{k}"] = rc, xc
    if r == b:  # the same values in another order: D = 0, h = 0
        ref_cols["same"], x_cols["same"] = ref_cols["x0"], rng.permutation(ref_cols["x0"])
    cats = np.array(["a", "b", "c", "d"])
    ref_cols["cat"] = cats[rng.integers(0, 4, r)]
    x_cols["cat"] = cats[rng.integers(0, 3, b)]
    return pd.DataFrame(ref_cols), pd.DataFrame(x_cols)


@functools.lru_cache(maxsize=None)
def _scipy(r, b):
    """per feature: (D, p, flag) of scipy's exact two-sample K-S, chi-squared (stat, p) for the categorical one"""
    import warnings

    ref, x = _case(r, b)
    out = {}
    for c in ref.columns:
        if c == "cat":
            union = sorted(set(ref[c]) | set(x[c]))
            t = np.array([[np.sum(ref[c] == v) for v in union], [np.sum(x[c] == v) for v in union]])
            out[c] = stats.chi2_contingency(t)[:2] if len(union) > 1 else (0.0, 1.0)
            continue
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            res = stats.ks_2samp(ref[c].to_numpy(), x[c].to_numpy(), alternative="two-sided", method="exact")
        out[c] = (res.statistic, res.pvalue, int(any(issubclass(i.category, RuntimeWarning) for i in w)))
    return out


def _routes(r, b, env):
    ref, x = _case(r, b)
    want = _scipy(r, b)
    forms = {}
    for c in ref.columns:
        if c != "cat":
            num = dw.ks_numerator(ref[c].to_numpy(), x[c].to_numpy())
            forms[c] = dw.route(r, b, num, env, p=want[c][1])
    return forms


def test_parametrization_covers_every_form():
    """The cases below reach every form of k_drift_finish under some environment (router mirrored in drift_walk.route)."""
    hit = {}
    for r, b in PAIRS:
        for env in ENVS:
            for c, f in _routes(r, b, env).items():
                hit.setdefault(f, (r, b, c, env))
    need = {"h0", "asymptotic", "n1", "rows_smem", "rows_global", "ring32", "ns1", "ns2", "ns4", "wide"}
    assert need <= set(hit), sorted(need - set(hit))


def _detector(frame, cats, env):
    from databricks_kubernetes_mlops_poc_b200.drift import TabularDrift

    old = {k: os.environ.get(k) for k in ("B2F_DRIFT_ROWSCAN", "B2F_DRIFT_ROWSCAN_SMEM", "B200_DRIFT_HANDLES")}
    for k in ("B2F_DRIFT_ROWSCAN", "B2F_DRIFT_ROWSCAN_SMEM"):
        os.environ.pop(k, None)
    os.environ.update(env)
    os.environ["B200_DRIFT_HANDLES"] = "1"
    try:
        return TabularDrift(frame, cats, device=0)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.mark.gpu
@pytest.mark.parametrize("r,b", PAIRS, ids=[f"{r}x{b}" for r, b in PAIRS])
def test_every_form_matches_scipy(r, b):
    ref, x = _case(r, b)
    want = _scipy(r, b)
    for env in ENVS:
        det = _detector(ref, ["cat"], env)
        try:
            p, stat, flags = det.statistics(x)
            forms = _routes(r, b, env)
            for i, c in enumerate(det.features):
                if c == "cat":
                    assert flags[i] == 0 and abs(stat[i] - want[c][0]) <= 1e-10 * max(want[c][0], 1e-300), (env, c)
                    assert abs(p[i] - want[c][1]) <= RTOL * max(want[c][1], 1e-300), (env, c, p[i], want[c])
                    continue
                d, pv, fl = want[c]
                what = (env, c, forms[c], stat[i], d, p[i], pv)
                assert flags[i] == fl, what
                assert abs(stat[i] - d) <= 4e-16, what
                tol = 1e-12 + RTOL * pv if fl == 1 else RTOL * max(pv, 1e-300)
                assert abs(p[i] - pv) <= tol, what
            again = det.statistics(x)  # deterministic: bit for bit
            assert all(np.array_equal(u, v, equal_nan=True) for u, v in zip((p, stat, flags), again)), env
        finally:
            det.close()


def _ks_check(det, ref, x, names):
    p, stat, flags = det.statistics(x)
    for i, c in enumerate(det.features):
        if c not in names:
            continue
        a, bb = ref[c].to_numpy(float), x[c].to_numpy(float)
        if np.isnan(bb).any():
            assert flags[i] == 2 and np.isnan(p[i]), c
            continue
        res = stats.ks_2samp(a, bb, alternative="two-sided", method="exact")
        assert flags[i] == 0 and abs(stat[i] - res.statistic) <= 4e-16, (c, stat[i], res.statistic)
        assert abs(p[i] - res.pvalue) <= RTOL * max(res.pvalue, 1e-300), (c, p[i], res.pvalue)
    return p, stat, flags


@pytest.mark.gpu
def test_ks_numerator_edges():
    """Ties straddling batch and reference, +-inf, -0.0 beside +0.0, subnormals, batch values at the reference min and max,
    an all-NaN batch feature (flag 2) -- under every environment."""
    rng = np.random.default_rng(17)
    r, b = 1025, 449
    tiny = np.finfo(float).tiny
    ref = pd.DataFrame({
        "ties": np.round(rng.normal(size=r)),
        "inf": np.concatenate((rng.normal(size=r - 4), [-np.inf, -np.inf, np.inf, 5.0])),
        "zero": np.concatenate((np.full(r // 2, -0.0), np.full(r - r // 2, 0.0))),
        "sub": np.concatenate((rng.integers(-3, 4, r - 5) * tiny * 2.0 ** -30, [5e-324, -5e-324, 0.0, tiny, -tiny])),
        "ends": rng.normal(size=r),
        "nan": rng.normal(size=r),
    })
    x = pd.DataFrame({
        "ties": np.round(rng.normal(0.3, 1, size=b)),
        "inf": np.concatenate((rng.normal(size=b - 5), [np.inf, np.inf, -np.inf, 5.0, 5.0])),
        "zero": np.where(rng.random(b) < 0.3, 0.0, -0.0) + np.where(rng.random(b) < 0.1, 1e-300, 0.0),
        "sub": rng.integers(-2, 3, b) * tiny * 2.0 ** -31,
        "ends": np.where(rng.random(b) < 0.5, ref["ends"].min(), ref["ends"].max()),
        "nan": np.full(b, np.nan),
    })
    x.loc[0, "ends"] = float(np.median(ref["ends"]))
    for env in ENVS:
        det = _detector(ref, [], env)
        try:
            first = _ks_check(det, ref, x, set(ref.columns))
            assert all(np.array_equal(u, v, equal_nan=True) for u, v in zip(first, det.statistics(x)))
        finally:
            det.close()


def _chi2_det(ref_vals, env=None):
    return _detector(pd.DataFrame({"c": np.asarray(ref_vals, dtype=object).astype(str)}), ["c"], env or {})


def _chi2_check(det, ref_vals, x_vals):
    ref_vals, x_vals = np.asarray(ref_vals).astype(str), np.asarray(x_vals).astype(str)
    p, stat, flags = det.statistics(pd.DataFrame({"c": x_vals.astype(object)}))
    union = sorted(set(ref_vals.tolist()) | set(x_vals.tolist()))
    t = np.array([[np.sum(ref_vals == v) for v in union], [np.sum(x_vals == v) for v in union]])
    s, pv = stats.chi2_contingency(t)[:2]
    assert flags[0] == 0 and abs(stat[0] - s) <= 1e-10 * max(s, 1e-300) + 1e-300, (len(union), stat[0], s)
    assert abs(p[0] - pv) <= RTOL * max(pv, 1e-300), (len(union), p[0], pv)
    return p[0], stat[0]


@pytest.mark.gpu
def test_chi2_edges():
    """K = 1 (dof 0: stat 0, p 1), K = 2 with the Yates clip reaching 0, K up to 512 (513 refused), statistics on both
    sides of the series / continued-fraction switch of gamma_q (x ~ a + 1) for a up to 255.5, p-values down to ~1e-230."""
    from databricks_kubernetes_mlops_poc_b200._cabi import B2FError

    det = _chi2_det(["a"] * 40)
    try:
        assert _chi2_check(det, ["a"] * 40, ["a"] * 7) == (1.0, 0.0)
    finally:
        det.close()
    ref = ["a"] * 300 + ["b"]
    det = _chi2_det(ref)
    try:
        assert _chi2_check(det, ref, ["a"] * 5) == (1.0, 0.0)  # [[300, 1], [5, 0]]: |o - e| < 0.5 everywhere
    finally:
        det.close()
    rng = np.random.default_rng(23)
    for K in (3, 40, 200, 512):
        cats = np.array([f"k{i:03d}" for i in range(K)])
        ref = cats[np.concatenate((np.arange(K), rng.integers(0, K, 40 * K)))]  # every category present
        det = _chi2_det(ref)
        try:
            seen = set()
            for trial in range(12):  # stat / 2 on both sides of a + 1 = (K + 1) / 2
                x = cats[rng.integers(0, K, 20 * K)]
                s = _chi2_check(det, ref, x)[1]
                seen.add(0.5 * s < 0.5 * (K - 1) + 1.0)
            assert seen == {True, False} or K >= 200, (K, seen)
            skew = np.concatenate((cats[rng.integers(0, K, 10 * K)], np.repeat(cats[:1], int(8 * K ** 0.5) + 60)))
            pv = _chi2_check(det, ref, skew)[0]  # a strongly over-represented category
            assert pv < 1e-6
            if K == 512:
                with pytest.raises(B2FError):  # 512 reference categories + one new one
                    det.statistics(pd.DataFrame({"c": np.array(["new"] + list(x[1:]), dtype=object)}))
        finally:
            det.close()
    ref = np.array(["a"] * 20000 + ["b"] * 20000 + ["c"] * 20000)
    det = _chi2_det(ref)
    try:
        for k in (300, 1000, 2000, 2600, 3000):  # down to p ~ 1e-230
            pv = _chi2_check(det, ref, np.array(["a"] * (k + 3000) + ["b"] * 3000 + ["c"] * 3000))[0]
        assert 0.0 < pv < 1e-200
    finally:
        det.close()


def test_reference_nan_is_refused():
    """A NaN in a numeric reference column: scipy would answer NaN for that feature on every request; the detector refuses
    the reference, naming the column (also a one-row reference, which no sortedness check can catch)."""
    from databricks_kubernetes_mlops_poc_b200.drift import TabularDrift

    for n in (1, 2, 300):
        ref = pd.DataFrame({"ok": np.arange(n, dtype=float), "bad": np.arange(n, dtype=float)})
        ref.loc[n // 2, "bad"] = np.nan
        with pytest.raises(ValueError, match="'bad'"):
            TabularDrift(ref, [], device=0)
