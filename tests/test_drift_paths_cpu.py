"""The router of k_drift_finish (mirrored in drift_walk.route, constants parsed from csrc/drift_stats.cuh) and the emulators of
the forms it routes to, against scipy's exact two-sample K-S -- on the whole domain each form can receive."""

import math

import pytest

import drift_walk as dw


def _scipy_p(m0, n0, h):
    from scipy.stats import _stats_pythran as sp

    g = math.gcd(m0, n0)
    return min(max(sp._compute_outer_prob_inside_method(max(m0, n0), min(m0, n0), g, h), 0.0), 1.0)


def _h(m0, n0, d):
    g = math.gcd(m0, n0)
    return max(1, round(d * (m0 // g) * n0))


ENVS = ({}, {"B2F_DRIFT_ROWSCAN": "0"}, {"B2F_DRIFT_ROWSCAN_SMEM": "0"}, {"B2F_DRIFT_ROWSCAN_SMEM": "1024"})


def test_router_follows_the_kernel_constants():
    lim = dw.kernel_limits()
    assert lim == {"THREADS": 1024, "RING_MAX": 4096, "ROWSCAN_MAX": 48, "ROWSCAN_SMEM_MAX": 448, "ROWSCAN_SMEM_LIMIT": 1024,
                   "ROWSCAN_CAP": 28672}
    assert dw.host_limits({}) == {"rows": 48, "smem": 448, "cap": 28672, "ring_max": 4096, "threads": 1024}
    assert dw.host_limits({"B2F_DRIFT_ROWSCAN": "0"})["smem"] == 0
    assert dw.host_limits({"B2F_DRIFT_ROWSCAN_SMEM": "5000"})["smem"] == 1024
    g = lambda m, n, d: _h(m, n, d) * math.gcd(m, n)  # noqa: E731  (K-S numerator)
    assert dw.route(30000, 16, 0) == "h0"
    assert dw.route(30000, 1, g(30000, 1, 0.5)) == "n1"
    assert dw.route(30000, 16, g(30000, 16, 0.2)) == "rows_smem"
    assert dw.route(30000, 16, g(30000, 16, 0.2), {"B2F_DRIFT_ROWSCAN_SMEM": "0"}) == "rows_global"
    assert dw.route(30000, 16, g(30000, 16, 0.2), {"B2F_DRIFT_ROWSCAN": "0"}) == "ring32"
    assert dw.route(30000, 449, g(30000, 449, 0.1)) == "ns1"
    assert dw.route(30000, 449, g(30000, 449, 0.1), {"B2F_DRIFT_ROWSCAN_SMEM": "1024"}) == "rows_smem"
    assert dw.route(16, 30000, g(16, 30000, 0.2)) == "ring32"  # the batch is the larger sample: no row scan
    assert dw.route(30000, 30000, g(30000, 30000, 0.1)) == "ns4"
    assert dw.route(30000, 30000, g(30000, 30000, 0.1421)) == "wide"
    assert dw.route(30000, 71587, 12345) == "asymptotic" and dw.route(30000, 71581, 12345) != "asymptotic"


def test_row_scans_are_exact_wherever_the_router_sends_them():
    """The global-scratch form (n <= 48) and the shared-memory form (n <= 1024 with the environment knob, band up to the
    kernel's cap of 28 672 cells) equal scipy wherever the router keeps their result; where it does not, it is the sweep."""
    cap = dw.kernel_limits()["ROWSCAN_CAP"]
    worst, kept = 0.0, 0
    for m in (1024, 4096, 30000, 30011):
        for n in (2, 3, 17, 48):
            for d in (0.03, 0.3, 0.7, 0.97):
                h = _h(m, n, d)
                num = h * math.gcd(m, n)
                want = _scipy_p(m, n, h)
                for env in ENVS:
                    form = dw.route(m, n, num, env, p=want)
                    assert form not in ("rows_smem", "rows_global") or dw.route(m, n, num, env) == form
                got = dw.exact_p_rows(m, n, num)[0]
                if dw.rows_scan_trusted(got, m, n, (2 * h) // (n // math.gcd(m, n)) + 1):
                    worst = max(worst, abs(got - want) / max(want, 1e-300))
                    kept += 1
    # the shared-memory schedule at the kernel's ring size, n up to the knob's limit, bands up to the cap
    for m, n, d in ((1024, 1024, 0.1), (1024, 1024, 0.6), (4096, 448, 0.3), (30000, 448, 0.02), (30000, 1024, 0.01)):
        h = _h(m, n, d)
        num = h * math.gcd(m, n)
        want = _scipy_p(m, n, h)
        assert dw.route(m, n, num, {"B2F_DRIFT_ROWSCAN_SMEM": "1024"}) == "rows_smem"
        got = dw.exact_p_rows_ring(m, n, num, cap=cap)[0]
        if dw.rows_scan_trusted(got, m, n, (2 * h) // (n // math.gcd(m, n)) + 1):
            worst = max(worst, abs(got - want) / max(want, 1e-300))
            kept += 1
        else:  # p ~ 1e-160 at (1024, 1024, 0.6): beyond what the row scale can resolve, the sweep recomputes it
            assert want < 1e-100 and dw.route(m, n, num, {"B2F_DRIFT_ROWSCAN_SMEM": "1024"}, p=want) == "ns1"
    assert kept >= 60 and worst <= 1e-12, (kept, worst)


@pytest.mark.parametrize("m,n,d", [(30000, 1000, 0.5), (30000, 1024, 0.45)])
def test_half_p_cases_stay_outside_the_row_scans(m, n, d):
    """Seeds C(lo - 1 + j, j) far below a row's scale underflow: the row scan returns half of scipy's p here.  The router must
    never keep such a result -- (30000, 1024, 0.45) fits the shared-memory ring under B2F_DRIFT_ROWSCAN_SMEM=1024."""
    g = math.gcd(m, n)
    h = _h(m, n, d)
    want = _scipy_p(m, n, h)
    got = dw.exact_p_rows(m, n, h * g)[0]
    assert 1e-300 < want < 1e-150 and abs(got / want - 0.5) < 1e-6
    assert not dw.rows_scan_trusted(got, m, n, (2 * h) // (n // g) + 1)
    for env in ENVS:
        assert dw.route(m, n, h * g, env, p=want) not in ("rows_smem", "rows_global"), env
    assert dw.route(m, n, h * g, {"B2F_DRIFT_ROWSCAN_SMEM": "1024"}) == ("rows_smem" if n == 1024 else "ns1")


def test_wide_band_sweep_matches_scipy():
    """sweep_wide (rings in global memory, slot cells recomputed per diagonal) emulated with a small shared-memory limit so
    that ordinary lattices take it, against scipy; and where it is the only form: m = n = 30 000 at D = 0.1421."""
    worst, ran = 0.0, 0
    for m, n in ((50, 7), (64, 48), (300, 16), (97, 100), (31, 31), (200, 400), (1025, 47)):
        g = math.gcd(m, n)
        lcm = m // g * n
        for h in sorted({lcm // 10 + 1, lcm // 5 + 1, lcm // 3 + 1, lcm // 2 + 1, lcm}):
            for ring_max in (32, 64):
                res = dw.exact_p_wide(m, n, h * g, ring_max=ring_max)
                if res is None:
                    continue
                want = _scipy_p(m, n, h)
                worst = max(worst, abs(res[0] - want) / max(want, 1e-300))
                ran += 1
                assert res[0] == dw.exact_p(m, n, h * g, force_ring=2 ** math.ceil(math.log2((2 * h) // (m // g + n // g) + 5)))[0] or n == 1
    assert ran >= 15 and worst <= 1e-12, (ran, worst)
    h = _h(30000, 30000, 0.1421)
    assert dw.exact_p_wide(30000, 30000, h * 30000, ring_max=4096 * 1024) is None
    assert dw.route(30000, 30000, h * 30000) == "wide"  # a shared-memory ring of 4096 slots cannot hold this band
    assert dw.exact_p(300, 300, 280 * 300, force_ring=4096) == dw.exact_p_wide(300, 300, 280 * 300, ring_max=128)
