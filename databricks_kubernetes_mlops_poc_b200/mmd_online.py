"""The online MMD drift detector (``B200Model.configure_online_drift`` / ``online_drift``): alibi-detect 0.12's
``MMDDriftOnline`` on the MMD test's space (``mmd.py``: the same embedding, kernel, reference and sigma), with the kernel
sums on the GPU (``csrc/mmd_online.cuh``) and everything else here: argument checks, the draws, the threshold loop, the
split loop and the answer.

W = window_size, E = 2W - 1, rw = n_ref - E, fpr = 1 / ERT.  A window's statistic is the unbiased MMD^2 of its W rows against
a sub-reference R of rw rows.

Thresholds: ``rng = np.random.default_rng(random_state)``; bootstrap b draws y = ``rng.permutation(n_ref)[-E:]`` (R is the
other rows) and the GPU gives the statistic of each of its W windows y_w .. y_{w+W-1}.  For w = 0 .. W-1 in order,
thresholds[w] is the type-7 (numpy ``linear``) quantile at 1 - fpr of the window-w statistics of the bootstraps still alive,
and a bootstrap stays alive only while its statistic is below the threshold.  So, with no drift, the expected run time
between false alarms is about ERT.

Split: on the same rng, ``perm = rng.permutation(n_ref)`` until the initial window perm[n_ref - W:] scores below
thresholds[0] against R = perm[:rw] (at most ``SPLIT_ATTEMPTS`` draws; alibi has no limit).

Stream: t counts the rows pushed since configure or reset, from 1; stat(t) is the statistic of the last W rows of [initial
window; pushed rows], threshold(t) = thresholds[min(t, W - 1)] and is_drift = stat > threshold.  Nothing resets on a
detection.  The draws are numpy's, not torch's: the same distribution, not the same draws.
"""

from __future__ import annotations

import math

import numpy as np

from .mmd import PAIR_BUDGET

MAX_WINDOW = 256  # B2F_MMD_ONLINE_MAX_WINDOW
MAX_BOOTSTRAPS = 100000  # B2F_MMD_ONLINE_MAX_BOOT
SPLIT_ATTEMPTS = 100
# at most this many kernel values per configure (n_bootstraps * E (E - 1) / 2) and per push (m * (rw + W)): the GPU is shared
KERNEL_BUDGET = PAIR_BUDGET


def _is_int(v) -> bool:
    return not isinstance(v, bool) and isinstance(v, (int, np.integer))


def check_config(n_ref: int, ert, window_size, n_bootstraps, random_state) -> tuple[float, int, int, int]:
    """-> (ert, window_size, n_bootstraps, random_state); ValueError for an ERT that is not finite and > 1, a window outside
    2..MAX_WINDOW or above (n_ref - 1) / 2, n_bootstraps outside 1..MAX_BOOTSTRAPS, a random_state that is not an integer
    >= 0, or more kernel values than KERNEL_BUDGET."""
    try:
        e = float(ert)
    except (TypeError, ValueError):
        raise ValueError(f"ert must be a finite number > 1, not {ert!r}") from None
    if not (math.isfinite(e) and e > 1.0):
        raise ValueError(f"ert must be a finite number > 1, not {ert!r}")
    if not _is_int(window_size) or not 2 <= window_size <= MAX_WINDOW:
        raise ValueError(f"window_size must be an integer in 2..{MAX_WINDOW}, not {window_size!r}")
    if n_ref < 2 * window_size + 1:
        raise ValueError(f"window_size {window_size} needs a reference of at least 2 * window_size + 1 = {2 * window_size + 1} rows; "
                         f"the MMD reference has {n_ref}")
    if not _is_int(n_bootstraps) or not 1 <= n_bootstraps <= MAX_BOOTSTRAPS:
        raise ValueError(f"n_bootstraps must be an integer in 1..{MAX_BOOTSTRAPS}, not {n_bootstraps!r}")
    if not _is_int(random_state) or random_state < 0:
        raise ValueError(f"random_state must be an integer >= 0, not {random_state!r}")
    E = 2 * int(window_size) - 1
    values = int(n_bootstraps) * E * (E - 1) // 2
    if values > KERNEL_BUDGET:
        raise ValueError(f"{n_bootstraps} bootstraps of window {window_size} are {values} kernel values, above the budget of "
                         f"{KERNEL_BUDGET}: ask for fewer bootstraps or a smaller window")
    return e, int(window_size), int(n_bootstraps), int(random_state)


def check_push(m: int, n_ref: int, window_size: int) -> None:
    """ValueError for no rows or more kernel values than KERNEL_BUDGET (m * (rw + W))."""
    if m < 1:
        raise ValueError("online drift needs at least one row")
    values = m * (n_ref - 2 * window_size + 1 + window_size)
    if values > KERNEL_BUDGET:
        raise ValueError(f"{m} rows against a sub-reference of {n_ref - 2 * window_size + 1} rows are {values} kernel values, above the "
                         f"budget of {KERNEL_BUDGET}: push fewer rows per call")


def draw_bootstraps(rng: np.random.Generator, n_ref: int, window_size: int, n_bootstraps: int) -> np.ndarray:
    """int32 (n_bootstraps, E): bootstrap b's y = rng.permutation(n_ref)[-E:]."""
    E = 2 * window_size - 1
    out = np.empty((n_bootstraps, E), dtype=np.int32)
    for b in range(n_bootstraps):
        out[b] = rng.permutation(n_ref)[-E:]
    return out


def thresholds(stats: np.ndarray, ert: float) -> np.ndarray:
    """float64 (W,) from the bootstrap statistics (n_bootstraps, W): the quantile-and-filter loop.  ValueError naming the
    window position that no bootstrap survives."""
    stats = np.asarray(stats, dtype=np.float64)
    q = 1.0 - 1.0 / ert
    out = np.empty(stats.shape[1], dtype=np.float64)
    for w in range(stats.shape[1]):
        if stats.shape[0] == 0:
            raise ValueError(f"no bootstrap stream is left at window position {w}: configure with more n_bootstraps (or a smaller ert)")
        out[w] = np.quantile(stats[:, w], q)
        stats = stats[stats[:, w] < out[w]]
    return out


def split(rng: np.random.Generator, n_ref: int, window_size: int, thr: np.ndarray, initial_stat) -> tuple[np.ndarray, int]:
    """-> (perm int32 (n_ref,), attempts): the first ``rng.permutation(n_ref)`` whose initial window scores below thr[0];
    ``initial_stat(y)`` gives the statistic of the window perm[n_ref - W:] for y = perm[rw:].  ValueError after
    SPLIT_ATTEMPTS draws."""
    rw = n_ref - (2 * window_size - 1)
    for attempt in range(1, SPLIT_ATTEMPTS + 1):
        perm = rng.permutation(n_ref).astype(np.int32)
        if initial_stat(perm[rw:]) < thr[0]:
            return perm, attempt
    raise ValueError(f"{SPLIT_ATTEMPTS} splits of the reference all start in detection (initial statistic >= threshold "
                     f"{thr[0]!r}): configure with more n_bootstraps or a larger ert")


def result(stat: np.ndarray, t_first: int, thr: np.ndarray, ert: float, window_size: int) -> dict:
    """The answer of one push: per row ``time``, ``test_stat``, ``threshold`` and ``is_drift`` (0/1), ``first_drift`` (the
    first time of this push with is_drift, else None), ``ert`` and ``window_size``."""
    stat = np.asarray(stat, dtype=np.float64)
    time = int(t_first) + np.arange(len(stat), dtype=np.int64)
    threshold = np.asarray(thr, dtype=np.float64)[np.minimum(time, window_size - 1)]
    is_drift = (stat > threshold).astype(np.int64)
    hit = np.flatnonzero(is_drift)
    return {"time": time, "test_stat": stat, "threshold": threshold, "is_drift": is_drift,
            "first_drift": int(time[hit[0]]) if len(hit) else None, "ert": float(ert), "window_size": int(window_size)}
