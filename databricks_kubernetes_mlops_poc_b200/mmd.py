"""The MMD drift test (``B200Model.mmd_drift``): alibi-detect 0.12's ``MMDDrift`` of a batch against a reference table,
with the kernel sums on the GPU (``csrc/mmd_drift.cuh``) and everything else here: argument checks, the embedding's
constants, the permutation draws and the answer.

Embedding: a row is the classifier's input vector, its one-hot categoricals and its numerics as scored (float32, NaN
imputed with the training median), the numerics z-scored in float64 with the reference's mean and population std (a std
of 0 gives scale 1).  The constants are computed once, here, when the reference is attached.

Permutations: one ``np.random.default_rng(random_state)`` per request; per permutation ``choice(N, s, replace=False,
shuffle=False)`` of the pool [reference; batch] (N = n_ref + m indices, s = min(m, n_ref)), sorted.  The subset is the
batch-sized side of the split when m <= n_ref, else the reference-sized side; a uniform subset's complement is uniform too,
so the split has alibi's ``randperm`` distribution (not its draws).  alibi keeps its permuted statistics in float32; these
are float64.
"""

from __future__ import annotations

import math

import numpy as np

MAX_REFERENCE = 131072  # B2F_MMD_MAX_REF
MAX_PERMUTATIONS = 10000  # B2F_MMD_MAX_PERM
# at most this many kernel evaluations over the subsets of one request, n_permutations * s (s - 1) / 2: the GPU is shared
PAIR_BUDGET = 2**36


def numerics(rows: np.ndarray, n_cat: int, n_num: int, impute) -> np.ndarray:
    """Encoded rows (N, 24) -> float64 (N, n_num): the numerics as the classifier scores them (NaN -> the training median)."""
    v = rows[:, n_cat:n_cat + n_num].view(np.float32).copy()
    nan = np.isnan(v)
    v[nan] = np.broadcast_to(np.asarray(impute, dtype=np.float32), v.shape)[nan]
    return v.astype(np.float64)


def standardization(x: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """The reference's numerics float64 (N, n_num) -> (mean, scale): the mean and population std per column, scale 1 where
    the std is 0."""
    mean = x.mean(axis=0)
    std = x.std(axis=0)
    return mean, np.where(std > 0.0, std, 1.0)


def check_sigma(sigma) -> float | None:
    if sigma is None:
        return None
    s = float(sigma)
    if not (math.isfinite(s) and s > 0.0):
        raise ValueError(f"sigma must be a finite positive number, not {sigma!r}")
    return s


def check_reference(n_ref: int) -> None:
    if not 2 <= n_ref <= MAX_REFERENCE:
        raise ValueError(f"an MMD reference needs 2..{MAX_REFERENCE} rows, not {n_ref}")


def check_request(m: int, n_ref: int, n_permutations, p_val, random_state) -> tuple[int, float, int]:
    """-> (n_permutations, p_val, random_state) as int, float, int; ValueError for fewer than 2 rows, n_permutations outside
    1..MAX_PERMUTATIONS, p_val outside (0, 1], a random_state that is not an integer >= 0, or more pairs than PAIR_BUDGET."""
    if isinstance(n_permutations, bool) or not isinstance(n_permutations, (int, np.integer)) or not 1 <= n_permutations <= MAX_PERMUTATIONS:
        raise ValueError(f"n_permutations must be an integer in 1..{MAX_PERMUTATIONS}, not {n_permutations!r}")
    p = float(p_val)
    if not 0.0 < p <= 1.0:
        raise ValueError(f"p_val must be in (0, 1], not {p_val!r}")
    if isinstance(random_state, bool) or not isinstance(random_state, (int, np.integer)) or random_state < 0:
        raise ValueError(f"random_state must be an integer >= 0, not {random_state!r}")
    if m < 2:
        raise ValueError(f"the MMD test needs at least 2 rows, not {m}")
    s = min(m, n_ref)
    pairs = int(n_permutations) * s * (s - 1) // 2
    if pairs > PAIR_BUDGET:
        raise ValueError(f"{n_permutations} permutations of {s} rows are {pairs} kernel pairs, above the budget of {PAIR_BUDGET}: "
                         "send fewer rows or ask for fewer permutations")
    return int(n_permutations), p, int(random_state)


def draw_subsets(n_ref: int, m: int, n_permutations: int, random_state: int) -> np.ndarray:
    """int32 (n_permutations, min(m, n_ref)): each row a sorted uniform subset of the pool's N = n_ref + m indices."""
    rng = np.random.default_rng(random_state)
    n, s = n_ref + m, min(m, n_ref)
    out = np.empty((n_permutations, s), dtype=np.int32)
    for b in range(n_permutations):
        out[b] = np.sort(rng.choice(n, s, replace=False, shuffle=False))
    return out


def result(mmd2: float, mmd2_perm: np.ndarray, p_val: float, sigma: float, n_ref: int, m: int) -> dict:
    """alibi's ``MMDDrift.predict`` data: is_drift, distance, p_val, threshold, distance_threshold, plus sigma, n_permutations,
    reference_rows and rows."""
    perm = np.asarray(mmd2_perm, dtype=np.float64)
    pv = float(np.mean(mmd2 <= perm))
    idx = min(int(p_val * len(perm)), len(perm) - 1)
    return {"is_drift": int(pv < p_val), "distance": float(mmd2), "p_val": pv, "threshold": float(p_val),
            "distance_threshold": float(np.sort(perm)[::-1][idx]), "sigma": float(sigma), "n_permutations": len(perm),
            "reference_rows": int(n_ref), "rows": int(m)}
