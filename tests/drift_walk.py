"""numpy emulation of the drift kernels' semantics (TEST INFRASTRUCTURE).

Mirrors ``csrc/drift_stats.cuh`` step for step -- the two binary searches and histograms of ``k_drift_count``, the
prefix-sum / tie-flag candidates of the K-S numerator, and the anti-diagonal ring sweep of the exact p-value with its
"designated j per slot" indexing -- so the algorithm can be checked against scipy on a CPU-only box.  Nothing in the
product imports it.
"""

import math

import numpy as np

RING_MAX = 4096


def ks_numerator(ref_sorted: np.ndarray, x: np.ndarray) -> int:
    m0, n0 = len(ref_sorted), len(x)
    a = np.searchsorted(ref_sorted, x, side="left")   # #ref <  x
    b = np.searchsorted(ref_sorted, x, side="right")  # #ref <= x
    ha = np.bincount(a, minlength=m0 + 1).astype(np.int64)
    hb = np.bincount(b, minlength=m0 + 1).astype(np.int64)
    cle = np.cumsum(ha)[:m0]
    clt = np.cumsum(hb)[:m0]
    j = np.arange(m0, dtype=np.int64)
    first = np.ones(m0, dtype=bool)
    first[1:] = ref_sorted[1:] != ref_sorted[:-1]
    last = np.ones(m0, dtype=bool)
    last[:-1] = ref_sorted[1:] != ref_sorted[:-1]
    v_last = np.abs((j + 1) * n0 - cle * m0)[last]
    v_first = np.abs(j * n0 - clt * m0)[first]
    return int(max(v_last.max(initial=0), v_first.max(initial=0)))


def exact_p(m0: int, n0: int, num: int, force_ring: int | None = None, check_bookkeeping: bool = False):
    """-> (p, flag): the ring sweep of k_drift_finish."""
    g = math.gcd(m0, n0)
    m, n = max(m0, n0), min(m0, n0)
    mg, ng = m // g, n // g
    h = num // g
    if (m0 // g) >= 2147483647.0 / (n0 // g):
        return -1.0, 1
    width = (2 * h) // (ng + mg) + 2
    ring = 32
    while ring < width + 3 and ring < RING_MAX:
        ring <<= 1
    if force_ring:
        ring = force_ring
    if h == 0:
        return 1.0, 0
    if width + 3 > ring:  # wider than the shared-memory ring: k_drift_finish runs sweep_wide
        return exact_p_wide(m0, n0, num, ring_max=RING_MAX)
    if n == 1 and not force_ring:  # single-row request: closed form (m + 1 equally likely paths), as in the kernel
        lo, hi = max(m - h + 1, 0), min(h - 1, m)
        inside = hi - lo + 1 if hi >= lo else 0
        return (m + 1 - inside) / (m + 1.0), 0
    mask = ring - 1
    den = ng + mg
    T = m + n
    j_lo = -(h // den) - 1
    while den * j_lo <= -h:
        j_lo += 1
    # slot state kept INCREMENTALLY, as SlotState / slot_advance in the kernel do
    s = np.arange(ring, dtype=np.int64)
    js = j_lo - 1
    edge = -h - den * j_lo
    j = js + ((s - js) & mask)
    i = -j
    dev = -den * j
    v = np.ones(ring)
    for t in range(T + 1):
        if check_bookkeeping:  # the closed forms the increments must reproduce
            jl = (ng * t - h) // den + 1
            assert js == jl - 1
            assert (j == js + ((s - js) & mask)).all() and (i == t - j).all() and (dev == ng * i - mg * j).all()
        left = v[(s - 1) & mask]
        rt = 1.0 / t if t > 0 else 0.0
        with np.errstate(invalid="ignore"):
            val = (left * j + v * i) * rt
        offl = (j < 0) | (j > n) | (i < 0) | (i > m) | (np.abs(dev) >= h)
        v = np.where(offl, 1.0, np.where(i == 0, 0.0, val))
        edge += ng
        adv = edge >= 0
        if adv:
            edge -= den
            js += 1
        i = i + 1
        dev = dev + ng
        if adv:
            jump = j < js
            j = np.where(jump, j + ring, j)
            i = np.where(jump, i - ring, i)
            dev = np.where(jump, dev - den * ring, dev)
    return float(min(max(v[n & mask], 0.0), 1.0)), 0


def gamma_q(a: float, x: float) -> float:
    if not x > 0.0:
        return 1.0
    if x < a + 1.0:
        ap, s = a, 1.0 / a
        d = s
        for _ in range(100000):
            ap += 1.0
            d *= x / ap
            s += d
            if abs(d) < abs(s) * 1e-17:
                break
        return 1.0 - s * math.exp(-x + a * math.log(x) - math.lgamma(a))
    tiny = 1e-300
    b = x + 1.0 - a
    c = 1.0 / tiny
    d = 1.0 / b
    hcf = d
    for it in range(1, 100000):
        an = -it * (it - a)
        b += 2.0
        d = an * d + b
        if abs(d) < tiny:
            d = tiny
        c = b + an / c
        if abs(c) < tiny:
            c = tiny
        d = 1.0 / d
        de = d * c
        hcf *= de
        if abs(de - 1.0) < 1e-16:
            break
    return math.exp(-x + a * math.log(x) - math.lgamma(a)) * hcf


def chi2(ref_counts, batch_counts, new_counts=()):
    o0 = np.concatenate((np.asarray(ref_counts, dtype=np.float64), np.zeros(len(new_counts))))
    o1 = np.concatenate((np.asarray(batch_counts, dtype=np.float64), np.asarray(new_counts, dtype=np.float64)))
    K = len(o0)
    if K < 2:
        return 0.0, 1.0
    row0, row1 = o0.sum(), o1.sum()
    tot = row0 + row1
    col = o0 + o1
    e0, e1 = row0 * col / tot, row1 * col / tot
    d0, d1 = o0 - e0, o1 - e1
    if K == 2:
        d0 = np.where(d0 > 0, d0 - np.minimum(0.5, d0), d0 + np.minimum(0.5, -d0))
        d1 = np.where(d1 > 0, d1 - np.minimum(0.5, d1), d1 + np.minimum(0.5, -d1))
    s = float((d0 * d0 / e0 + d1 * d1 / e1).sum())
    return s, gamma_q(0.5 * (K - 1), 0.5 * s)


# ----------------------------------------------------------------------------- row-scan form of the exact p-value
def _binom_scaled(t: int, k: int, e: int) -> float:
    """C(t, k) * 2**(-e) by the running product prod (t - k + r) / r with exponent tracking (as the kernel does it)."""
    v, ex = 1.0, 0
    for r in range(1, k + 1):
        v = v * float(t - k + r) / float(r)
        if v > 2.0 ** 400:
            v *= 2.0 ** -400
            ex += 400
    return math.ldexp(v, ex - e)


def _binom_exponent(t: int, k: int) -> int:
    v, ex = 1.0, 0
    for r in range(1, k + 1):
        v = v * float(t - k + r) / float(r)
        if v > 2.0 ** 400:
            v *= 2.0 ** -400
            ex += 400
    return ex + math.frexp(v)[1]


def exact_p_rows(m0: int, n0: int, num: int):
    """The ROW-SCAN form of the exact two-sided p-value (k_drift_finish for request-sized batches):
    W(i, j) = number of lattice paths (0,0)->(i,j) that left the band |ng*i - mg*j| < h obeys, inside the band,
    W(i, j) = W(i-1, j) + W(i, j-1) -- the (i+j)-normalised recursion of scipy multiplied through by C(i+j, j) -- and is
    C(i+j, j) outside.  Inside the band a row is therefore ONE prefix sum over i of the previous row (extended by the
    binomials of the cells that were outside one row earlier), seeded with the binomial of the cell left of the band:
    n prefix sums of length <= m instead of m + n dependent anti-diagonal steps.  Every row is scaled by 2**-E_j
    (E_j = exponent of the largest binomial of the row) so nothing overflows.  -> (p, flag)."""
    g = math.gcd(m0, n0)
    m, n = max(m0, n0), min(m0, n0)
    mg, ng = m // g, n // g
    h = num // g
    if (m0 // g) >= 2147483647.0 / (n0 // g):
        return -1.0, 1
    if h == 0:
        return 1.0, 0

    def lo_hi(j):
        lo = (mg * j - h) // ng + 1  # first i with ng*i - mg*j > -h
        hi = -((-(mg * j + h)) // ng) - 1  # last i with ng*i - mg*j < h
        return max(lo, 0), min(hi, m)

    lo_p, hi_p = lo_hi(0)
    prev = np.zeros(m + 1, dtype=np.float64)  # row 0 inside the band: no path has left it yet
    e_prev = _binom_exponent(hi_p + 0, 0)
    for j in range(1, n + 1):
        lo, hi = lo_hi(j)
        e = _binom_exponent(hi + j, j)
        # cells (i, j-1) right of the previous row's band are outside it: every path to them has left the band
        for i in range(hi_p + 1, hi + 1):
            prev[i] = _binom_scaled(i + j - 1, j - 1, e_prev)
        seed = _binom_scaled(lo - 1 + j, j, e) if lo >= 1 else 0.0
        cur = np.zeros(m + 1, dtype=np.float64)
        cur[lo : hi + 1] = seed + np.cumsum(prev[lo : hi + 1] * math.ldexp(1.0, e_prev - e))
        prev, lo_p, hi_p, e_prev = cur, lo, hi, e
    total = _binom_scaled(m + n, n, e_prev)
    return float(min(max(prev[m] / total, 0.0), 1.0)), 0


def exact_p_rows_ring(m0: int, n0: int, num: int, cap: int = 26624, nt: int = 1024):
    """`rows_scan_smem` step by step: the row lives in a ring of `cap` slots (cell i at i mod cap) and is updated in place;
    thread t owns L (odd) consecutive cells from lo_j + t*L; cells the previous row had outside the band are written into the ring
    before the scan.  -> (p, flag), or None when the band is too wide for the ring (the kernel takes another form then)."""
    g = math.gcd(m0, n0)
    m, n = max(m0, n0), min(m0, n0)
    mg, ng = m // g, n // g
    h = num // g
    if (m0 // g) >= 2147483647.0 / (n0 // g):
        return -1.0, 1
    if h == 0:
        return 1.0, 0
    if (2 * h) // ng + 2 > cap:
        return None
    ring = np.full(cap, np.nan)  # NaN: a slot read before it was written poisons the result
    hi_p = min(-((-h) // ng) - 1, m)
    for i in range(hi_p + 1):
        ring[i % cap] = 0.0
    e_p = 1
    for j in range(1, n + 1):
        lo = max((mg * j - h) // ng + 1, 0)
        hi = min(-((-(mg * j + h)) // ng) - 1, m)
        e = _binom_exponent(hi + j, j)
        seed = _binom_scaled(lo - 1 + j, j, e) if lo >= 1 else 0.0
        # cells below lo are not read by this row: writing them (in parallel, on the GPU) could wrap onto slots that are
        written = {}
        for i in range(max(hi_p + 1, lo), hi + 1):
            assert i % cap not in written, "two cells of one extension share a slot"
            written[i % cap] = i
            ring[i % cap] = _binom_scaled(i + j - 1, j - 1, e_p)
        scale = math.ldexp(1.0, e_p - e)
        w = hi - lo + 1
        L = ((max(w, 1) + nt - 1) // nt) | 1
        # pass A: per-thread sums in cell order, exclusive scan in thread order
        run = seed
        for t in range(nt):
            a0 = lo + t * L
            a1 = min(a0 + L, hi + 1)
            for i in range(a0, a1):  # pass B of thread t (its offset is the running total so far)
                run += ring[i % cap] * scale
                ring[i % cap] = run
        hi_p, e_p = hi, e
    total = _binom_scaled(m + n, n, e_p)
    return float(min(max(ring[m % cap] / total, 0.0), 1.0)), 0


# ----------------------------------------------------------------------------- which form k_drift_finish runs
def kernel_limits(path: str | None = None) -> dict:
    """The router's constants, parsed from ``csrc/drift_stats.cuh`` (so a change there reaches the mirror below)."""
    import os
    import re

    if path is None:
        path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "databricks_kubernetes_mlops_poc_b200", "csrc",
                            "drift_stats.cuh")
    src = open(path).read()
    out = {}
    for key in ("THREADS", "RING_MAX", "ROWSCAN_MAX", "ROWSCAN_SMEM_MAX", "ROWSCAN_SMEM_LIMIT", "ROWSCAN_CAP"):
        out[key] = int(re.search(rf"#define\s+B2F_DRIFT_{key}\s+(\d+)", src).group(1))
    return out


def host_limits(env: dict | None = None, limits: dict | None = None) -> dict:
    """What ``drift_init`` makes of the environment: the largest batch of each row-scan form (0 = off)."""
    lim = limits or kernel_limits()
    env = env or {}
    rows = lim["ROWSCAN_MAX"]
    if "B2F_DRIFT_ROWSCAN" in env:
        rows = max(0, min(lim["ROWSCAN_MAX"], int(env["B2F_DRIFT_ROWSCAN"])))
    smem = 0 if ("B2F_DRIFT_ROWSCAN" in env and rows == 0) else lim["ROWSCAN_SMEM_MAX"]
    if "B2F_DRIFT_ROWSCAN_SMEM" in env:
        smem = max(0, min(lim["ROWSCAN_SMEM_LIMIT"], int(env["B2F_DRIFT_ROWSCAN_SMEM"])))
    return {"rows": rows, "smem": smem, "cap": lim["ROWSCAN_CAP"], "ring_max": lim["RING_MAX"], "threads": lim["THREADS"]}


def rows_scan_trusted(p: float, m: int, n: int, w: int) -> bool:
    """Mirror of ``rows_scan_trusted``: the row scans lose what a row holds below 2^-1074 of its scale; their p-value is kept
    only where that loss is below 2^-40 of it."""
    lg = math.log2(n * (w + 2)) + (4.0 - 1074.0 + 40.0) + n * math.log2((m + w + 1) / (m + 1))
    return p >= 2.0 ** lg if lg > -1100 else True


def route(n_ref: int, n0: int, num: int, env: dict | None = None, p: float | None = None, limits: dict | None = None) -> str:
    """-> the form ``k_drift_finish`` takes for a numeric feature with K-S numerator ``num`` (D = num / (n_ref n0)):
    'nan' / 'asymptotic' (flags 2 / 1), 'h0' (p = 1), 'n1' (closed form), 'rows_smem', 'rows_global', 'ring32',
    'ns1' / 'ns2' / 'ns4' (sweep_block<NS>), 'wide' (sweep_wide, rings in global memory).  With ``p`` (the true p-value)
    a row scan whose result would not be trusted reports the sweep form that recomputes it."""
    hl = host_limits(env, limits)
    g = math.gcd(n_ref, n0)
    m, n = max(n_ref, n0), min(n_ref, n0)
    mg, ng = m // g, n // g
    h = num // g
    if (n_ref // g) >= 2147483647.0 / (n0 // g):
        return "asymptotic"
    if h == 0:
        return "h0"
    if n == 1:
        return "n1"
    width = (2 * h) // (ng + mg) + 2
    ring = 32
    while ring < width + 3:
        ring <<= 1
    smem_max = hl["smem"] if 2 <= n0 <= hl["smem"] else 0
    smem_rows = 2 <= n <= smem_max and m == n_ref and m >= 1024 and (2 * h) // ng + 2 <= hl["cap"]
    global_rows = hl["rows"] > 0 and n_ref >= 1024 and 2 <= n <= hl["rows"] and m == n_ref and m >= 1024
    if smem_rows or global_rows:
        if p is None or rows_scan_trusted(p, m, n, (2 * h) // ng + 1):
            return "rows_smem" if smem_rows else "rows_global"
    if ring > hl["ring_max"]:
        return "wide"
    if ring == 32:
        return "ring32"
    return f"ns{ring // min(hl['threads'], ring)}"


def exact_p_wide(m0: int, n0: int, num: int, ring_max: int = RING_MAX):
    """`sweep_wide` step by step: a ring wider than ``ring_max`` in global memory, every slot's cell recomputed each diagonal
    from the lowest covered j (j = js + ((s - js) mod ring), i = t - j) instead of tracked.  -> (p, flag), or None when the band
    fits the shared-memory ring (the kernel takes another form)."""
    g = math.gcd(m0, n0)
    m, n = max(m0, n0), min(m0, n0)
    mg, ng = m // g, n // g
    h = num // g
    if (m0 // g) >= 2147483647.0 / (n0 // g):
        return -1.0, 1
    if h == 0:
        return 1.0, 0
    den = ng + mg
    width = (2 * h) // den + 2
    ring = 32
    while ring < width + 3:
        ring <<= 1
    if ring <= ring_max:
        return None
    mask = ring - 1
    j_lo = -(h // den) - 1
    while den * j_lo <= -h:
        j_lo += 1
    js, edge = j_lo - 1, -h - den * j_lo
    s = np.arange(ring, dtype=np.int64)
    prev = np.ones(ring)
    for t in range(m + n + 1):
        j = js + ((s - js) & mask)
        i = t - j
        dev = ng * i - mg * j
        left = prev[(s - 1) & mask]
        rt = 1.0 / t if t > 0 else 0.0
        off = (j < 0) | (j > n) | (i < 0) | (i > m) | (np.abs(dev) >= h)
        scale = np.where(off | (i == 0), 0.0, rt)
        with np.errstate(invalid="ignore", over="ignore"):
            prev = (left * j + prev * i) * scale + np.where(off, 1.0, 0.0)
        edge += ng
        if edge >= 0:
            edge -= den
            js += 1
    return float(min(max(prev[n & mask], 0.0), 1.0)), 0
