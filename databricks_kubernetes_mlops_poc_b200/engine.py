"""ForestEngine: one flattened forest resident on one H100, driven through the C ABI.

Python-side owner of a ``b2f_model*`` (``include/b2f.h``).  It replaces the object the
reference keeps in ``self.classifier`` (``databricks/src/02-register-model.ipynb:318-322``) for the
purposes of ``predict_proba(...)[:, 1]`` / ``predict`` (``:335-337``).  No CPU fallback.
"""

from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import _cabi
from ._cabi import (
    MOMENT_VALUES, OUT_F32, OUT_F64, OUT_FULL, OUT_PAIRS, PACKED_ROW_WORDS, ROW_WORDS, ROWS_PACKED64, ROWS_RANKED, ROWS_WORDS24, B2FError, Info,
    PinnedBuffer, RankInfo, check, ptr,
)
from .flatten import FlatForest


def device_count() -> int:
    n = _cabi.load_library().b2f_device_count()
    if n < 0:
        raise B2FError(f"no usable CUDA device: {_cabi.last_error()}")
    return n


def validate_paths(blob: bytes) -> None:
    """Structural check of a TreeSHAP path table (no GPU needed); raises B2FError when malformed."""
    buf = np.frombuffer(blob, dtype=np.uint8)
    check(_cabi.load_library().b2f_paths_validate(ptr(buf), buf.size), "b2f_paths_validate")


def validate_blob(blob: bytes) -> None:
    """Structural check of a forest blob (no GPU needed); raises B2FError when malformed."""
    buf = np.frombuffer(blob, dtype=np.uint8)
    check(_cabi.load_library().b2f_blob_validate(ptr(buf), buf.size), "b2f_blob_validate")


class ForestEngine:
    def __init__(self, flat: FlatForest | bytes, device: int = 0):
        """``flat``: a FlatForest (classifier) or raw forest-blob bytes (e.g. an isolation forest on its own)."""
        self._lib = _cabi.load_library()
        self.flat = flat
        self.device = int(device)
        buf = np.frombuffer(flat.blob if isinstance(flat, FlatForest) else flat, dtype=np.uint8)
        self._h = self._lib.b2f_model_create(ptr(buf), buf.size, self.device)
        if not self._h:
            raise B2FError(f"b2f_model_create(device={device}) failed: {_cabi.last_error()}")
        self._pinned: dict[str, PinnedBuffer] = {}
        self.explainer_attached = False
        self.background_rows = 0
        self.mmd_reference_rows = 0
        self.knn_class_rows = (0, 0)  # rows of each class in the attached trust reference
        inf = self.info()
        self.rank_words = inf["rank_row_bytes"] // 4 if inf["rank_ok"] else 0  # width of a ranked row, 0 = not available

    def _fmt(self, rows: np.ndarray) -> int:
        return _row_format(rows, self.rank_words)

    # ------------------------------------------------------------------ lifetime
    def close(self) -> None:
        if getattr(self, "_h", None):
            self._lib.b2f_model_destroy(self._h)
            self._h = None
        for b in self._pinned.values():
            b.close()
        self._pinned = {}

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        return self._h

    def info(self) -> dict:
        inf = Info()
        check(self._lib.b2f_model_info(self._h, C.byref(inf)), "b2f_model_info")
        d = {name: getattr(inf, name) for name, _ in Info._fields_}
        d["walk"] = _cabi.WALK_NAMES.get(d["walk_mode"], "?")
        d["agg"] = _cabi.AGG_NAMES.get(d["agg_mode"], "?")
        return d

    def rank_info(self) -> RankInfo:
        inf = RankInfo()
        check(self._lib.b2f_model_rank_info(self._h, C.byref(inf)), "b2f_model_rank_info")
        return inf

    # ------------------------------------------------------------------ pinned staging
    def pinned(self, tag: str, nbytes: int) -> PinnedBuffer:
        """A reusable page-locked buffer of at least nbytes (grown geometrically)."""
        b = self._pinned.get(tag)
        if b is None or b.nbytes < nbytes:
            if b is not None:
                b.close()
            b = PinnedBuffer(max(int(nbytes * 1.5), 1 << 16), device=self.device)  # pages on the GPU's NUMA node
            self._pinned[tag] = b
        return b

    def staging(self, n: int, packed: bool = False):
        """(rows uint32 (n,24) or packed (n,16), proba f64 (n,), label i32 (n,)) views over pinned memory."""
        words = PACKED_ROW_WORDS if packed else ROW_WORDS
        rows = self.pinned("rows", n * ROW_WORDS * 4).view(np.uint32, (n, words))
        proba = self.pinned("proba", n * 24).view(np.float64, (n,))  # 24 B per row: also holds b2f_scored_full records
        label = self.pinned("label", n * 4).view(np.int32, (n,))
        return rows, proba, label

    def staging_full(self, n: int) -> np.ndarray:
        """SCORED_FULL_DTYPE (n,) view over the pinned result buffer (shares storage with ``staging``'s proba)."""
        return self.pinned("proba", n * 24).view(_cabi.SCORED_FULL_DTYPE, (n,))

    # ------------------------------------------------------------------ scoring (host buffers)
    def predict_rows(self, rows: np.ndarray, proba_dtype=np.float64, want_label: bool = True, out_proba=None, out_label=None):
        """Encoded rows (N, 24) uint32 in host memory -> (proba1, label)."""
        rows = np.ascontiguousarray(rows)
        fmt = self._fmt(rows)
        n = rows.shape[0]
        f64 = np.dtype(proba_dtype) == np.float64
        proba = out_proba if out_proba is not None else np.empty(n, dtype=np.float64 if f64 else np.float32)
        label = out_label if out_label is not None else (np.empty(n, dtype=np.int32) if want_label else None)
        check(self._lib.b2f_predict_ex(self._h, ptr(rows), n, fmt, ptr(proba), int(f64), ptr(label)), "b2f_predict_ex")
        return proba, label

    def predict_pairs(self, rows: np.ndarray, out: np.ndarray | None = None) -> np.ndarray:
        """Encoded rows -> structured array of (proba1 float32, label int32), one D2H copy per chunk."""
        rows = np.ascontiguousarray(rows)
        n = rows.shape[0]
        if out is None:
            out = np.empty(n, dtype=_cabi.SCORED_DTYPE)
        check(self._lib.b2f_predict_pairs(self._h, ptr(rows), n, self._fmt(rows), ptr(out)), "b2f_predict_pairs")
        return out

    # ------------------------------------------------------------------ columnar request pipeline (csrc/scorer.h)
    def scorer(self, encoder, threads: int = 0):
        """A ``Scorer`` bound to this engine and ``encoder`` (created once, reused for every request)."""
        return Scorer(self, encoder, threads)

    # ------------------------------------------------------------------ classifier + outlier detector in one pass
    def attach_outlier_forest(self, blob: bytes) -> None:
        """Attach an isolation-forest blob (``flatten.flatten_isolation_forest``) evaluated on the same rows."""
        buf = np.frombuffer(blob, dtype=np.uint8)
        check(self._lib.b2f_model_attach_outlier_forest(self._h, ptr(buf), buf.size), "b2f_model_attach_outlier_forest")

    def predict_full(self, rows: np.ndarray, out: np.ndarray | None = None) -> np.ndarray:
        """Encoded rows -> structured array (proba1, label, outlier_score, is_outlier): one H2D copy of the rows,
        both forests walked on the GPU, one D2H copy per chunk."""
        rows = np.ascontiguousarray(rows)
        n = rows.shape[0]
        if out is None:
            out = np.empty(n, dtype=_cabi.SCORED_FULL_DTYPE)
        check(self._lib.b2f_predict_full(self._h, ptr(rows), n, self._fmt(rows), ptr(out)), "b2f_predict_full")
        return out

    def predict_rows_async(self, rows: np.ndarray, proba: np.ndarray, label: np.ndarray | None) -> int:
        """Pinned buffers in, ticket out; pair with wait()."""
        t = C.c_uint64(0)
        check(
            self._lib.b2f_predict_async_ex(
                self._h, ptr(rows), rows.shape[0], self._fmt(rows), ptr(proba), int(proba.dtype == np.float64), ptr(label), C.byref(t)
            ),
            "b2f_predict_async_ex",
        )
        return t.value

    def predict_pairs_async(self, rows: np.ndarray, out: np.ndarray) -> int:
        """Asynchronous ``predict_pairs`` on pinned buffers (``out``: SCORED_DTYPE); pair with wait()."""
        t = C.c_uint64(0)
        check(
            self._lib.b2f_predict_async_ex(self._h, ptr(rows), rows.shape[0], self._fmt(rows), ptr(out), OUT_PAIRS, None, C.byref(t)),
            "b2f_predict_async_ex",
        )
        return t.value

    def wait(self, ticket: int) -> None:
        check(self._lib.b2f_wait(self._h, ticket), "b2f_wait")

    # ------------------------------------------------------------------ explanations (TreeSHAP, csrc/tree_shap.cuh)
    def attach_explainer(self, blob: bytes) -> None:
        """Attach a path table (``flatten.flatten_explainer``) built from this engine's forest."""
        buf = np.frombuffer(blob, dtype=np.uint8)
        check(self._lib.b2f_model_attach_explainer(self._h, ptr(buf), buf.size), "b2f_model_attach_explainer")
        self.explainer_attached = True
        self.background_rows = 0  # the background belongs to the explainer it was attached to

    def attach_background(self, rows: np.ndarray) -> int:
        """Attach encoded background rows (N, 24) or packed (N, 16), N >= 1, for ``explain_interventional_rows``; replaces an
        earlier background.  -> the device bytes of its compressed table."""
        rows = np.ascontiguousarray(rows)
        nbytes = C.c_size_t(0)
        check(self._lib.b2f_model_attach_background(self._h, ptr(rows), rows.shape[0], self._fmt(rows), C.byref(nbytes)),
              "b2f_model_attach_background")
        self.background_rows = rows.shape[0]
        return nbytes.value

    def explain_rows(self, rows: np.ndarray, device_ms: bool = False):
        """Encoded rows (N, 24) or packed (N, 16) -> (phi float64 (N, n_cat + n_num), base_value[, device ms]): exact
        path-dependent TreeSHAP per request field, in probability (RandomForest) or log-odds (GBDT) space."""
        return self._explained("b2f_explain", 1, rows, device_ms)

    def explain_device(self, rows_dev: int, n: int, phi_dev: int, fmt: int = ROWS_WORDS24) -> None:
        """Enqueue an explanation of device-resident rows into device phi (n x fields doubles); ``sync`` waits."""
        check(self._lib.b2f_explain_device(self._h, rows_dev, n, fmt, phi_dev), "b2f_explain_device")

    def explain_interactions_rows(self, rows: np.ndarray, device_ms: bool = False):
        """Encoded rows (N, 24) or packed (N, 16) -> (phi2 float64 (N, F, F), base_value[, device ms]) with F = n_cat + n_num:
        exact path-dependent SHAP interaction values per pair of request fields.  Each matrix is symmetric, its rows sum to
        ``explain_rows``' phi and its total to the prediction - base_value."""
        return self._explained("b2f_explain_interactions", 2, rows, device_ms)

    def explain_interactions_device(self, rows_dev: int, n: int, phi2_dev: int, fmt: int = ROWS_WORDS24) -> None:
        """Enqueue interaction values of device-resident rows into device phi2 (n x fields x fields doubles); ``sync`` waits."""
        check(self._lib.b2f_explain_interactions_device(self._h, rows_dev, n, fmt, phi2_dev), "b2f_explain_interactions_device")

    def explain_interventional_rows(self, rows: np.ndarray, device_ms: bool = False):
        """Encoded rows (N, 24) or packed (N, 16) -> (phi float64 (N, n_cat + n_num), base_value[, device ms]): exact
        interventional TreeSHAP against the attached background (``attach_background``), the mean over background rows z of
        the Shapley values of f(x_S, z_rest).  base_value is the mean prediction over the background, in the output space of
        ``explain_rows``, and base_value + phi.sum(1) the prediction."""
        return self._explained("b2f_explain_interventional", 1, rows, device_ms)

    def explain_interventional_device(self, rows_dev: int, n: int, phi_dev: int, fmt: int = ROWS_WORDS24) -> None:
        """Enqueue interventional values of device-resident rows into device phi (n x fields doubles); ``sync`` waits."""
        check(self._lib.b2f_explain_interventional_device(self._h, rows_dev, n, fmt, phi_dev), "b2f_explain_interventional_device")

    def _explained(self, fn: str, field_axes: int, rows: np.ndarray, device_ms: bool):
        """C function ``fn`` (b2f_explain / b2f_explain_interactions / b2f_explain_interventional) on host rows into float64 of shape (N,) + (F,) * field_axes
        with F = n_cat + n_num -> (values, base_value[, device ms])."""
        rows = np.ascontiguousarray(rows)
        fmt = self._fmt(rows)
        n = rows.shape[0]
        inf = self.info()
        out = np.empty((n,) + (inf["n_cat"] + inf["n_num"],) * field_axes, dtype=np.float64)
        base, ms = C.c_double(0.0), C.c_float(0.0)
        check(getattr(self._lib, fn)(self._h, ptr(rows), n, fmt, ptr(out), C.byref(base), C.byref(ms)), fn)
        return (out, base.value, ms.value) if device_ms else (out, base.value)

    # ------------------------------------------------------------------ partial dependence (csrc/partial_dependence.cuh)
    def partial_dependence_rows(self, rows: np.ndarray, probes, grid_words: np.ndarray, device_ms: bool = False):
        """Encoded rows (N, 24) or packed (N, 16), probes [(row word, grid offset, count)] and the grid's row words ->
        float64 (N, sum of counts)[, device ms]: column block p holds, for each row, the model's output with word
        ``probes[p][0]`` replaced by each of its grid words in turn (a row's ICE curves, concatenated in probe order)."""
        rows = np.ascontiguousarray(rows)
        pr = _probe_table(probes)
        grid = np.ascontiguousarray(grid_words, dtype=np.uint32)
        out = np.empty((rows.shape[0], int(pr["count"].sum())), dtype=np.float64)
        ms = C.c_float(0.0)
        check(self._lib.b2f_partial_dependence(self._h, ptr(rows), rows.shape[0], self._fmt(rows), ptr(pr), len(pr), ptr(grid), ptr(out),
                                               C.byref(ms)), "b2f_partial_dependence")
        return (out, ms.value) if device_ms else out

    def partial_dependence_device(self, rows_dev: int, n: int, probes, grid_words: np.ndarray, out_dev: int, fmt: int = ROWS_WORDS24) -> None:
        """Enqueue the curves of device-resident rows into device out (n x sum of counts doubles); probes and grid words are
        host arrays, as for ``partial_dependence_rows``; ``sync`` waits."""
        pr = _probe_table(probes)
        grid = np.ascontiguousarray(grid_words, dtype=np.uint32)
        check(self._lib.b2f_partial_dependence_device(self._h, rows_dev, n, fmt, ptr(pr), len(pr), ptr(grid), out_dev),
              "b2f_partial_dependence_device")

    # ------------------------------------------------------------------ two-way partial dependence (csrc/pair_dependence.cuh)
    def pair_dependence_rows(self, rows: np.ndarray, probes, point_words: np.ndarray, mean: bool = False, device_ms: bool = False):
        """Encoded rows (N, 24) or packed (N, 16), probes [(word a, word b or -1, point offset, count)] and the points' row
        words (P', 2) -> float64 (N, sum of counts), or with ``mean`` (sum of counts,) [, device ms]: each point's score of
        every row with word a set to the point's first word and word b to its second (a probe's points concatenated in
        probe order), or its mean over the rows, taken on the device."""
        rows = np.ascontiguousarray(rows)
        pr = _pair_probe_table(probes)
        words = np.ascontiguousarray(point_words, dtype=np.uint32).reshape(-1, 2)
        P = int(pr["count"].sum())
        out = np.empty(P if mean else (rows.shape[0], P), dtype=np.float64)
        ms = C.c_float(0.0)
        check(self._lib.b2f_pair_dependence(self._h, ptr(rows), rows.shape[0], self._fmt(rows), ptr(pr), len(pr), ptr(words), int(bool(mean)),
                                            ptr(out), C.byref(ms)), "b2f_pair_dependence")
        return (out, ms.value) if device_ms else out

    def pair_dependence_device(self, rows_dev: int, n: int, probes, point_words: np.ndarray, out_dev: int, mean: bool = False,
                               fmt: int = ROWS_WORDS24) -> None:
        """Enqueue the two-way curves (n x sum of counts doubles) or, with ``mean``, their means (sum of counts doubles) of
        device-resident rows into device out; probes and point words are host arrays, as for ``pair_dependence_rows``;
        ``sync`` waits."""
        pr = _pair_probe_table(probes)
        words = np.ascontiguousarray(point_words, dtype=np.uint32).reshape(-1, 2)
        check(self._lib.b2f_pair_dependence_device(self._h, rows_dev, n, fmt, ptr(pr), len(pr), ptr(words), int(bool(mean)), out_dev),
              "b2f_pair_dependence_device")

    # ------------------------------------------------------------------ accumulated local effects (csrc/ale.cuh)
    def ale_rows(self, rows: np.ndarray, probes, edges: np.ndarray, device_ms: bool = False):
        """Encoded rows (N, 24) or packed (N, 16), probes [(numeric row word, edge offset, bins K)] and float32 edges ->
        (float64 bin sums, int64 bin row counts[, device ms]), each (sum of K,) in probe order: per bin of a probe, the sum
        over the rows whose value of the word lies in it of f(upper edge) - f(lower edge), and the number of those rows."""
        rows = np.ascontiguousarray(rows)
        pr = _ale_probe_table(probes)
        z = np.ascontiguousarray(edges, dtype=np.float32)
        K = int(pr["bins"].sum()) if len(pr) else 0
        sums, counts = np.empty(K, dtype=np.float64), np.empty(K, dtype=np.int64)
        ms = C.c_float(0.0)
        check(self._lib.b2f_ale(self._h, ptr(rows), rows.shape[0], self._fmt(rows), ptr(pr), len(pr), ptr(z), ptr(sums), ptr(counts),
                                C.byref(ms)), "b2f_ale")
        return (sums, counts, ms.value) if device_ms else (sums, counts)

    def ale_device(self, rows_dev: int, n: int, probes, edges: np.ndarray, sums_dev: int, counts_dev: int, fmt: int = ROWS_WORDS24) -> None:
        """Enqueue the per-bin sums (doubles) and row counts (int64) of device-resident rows into device buffers; probes and
        edges are host arrays, as for ``ale_rows``; ``sync`` waits."""
        pr = _ale_probe_table(probes)
        z = np.ascontiguousarray(edges, dtype=np.float32)
        check(self._lib.b2f_ale_device(self._h, rows_dev, n, fmt, ptr(pr), len(pr), ptr(z), sums_dev, counts_dev), "b2f_ale_device")

    # ------------------------------------------------------------------ counterfactuals (csrc/counterfactual.cuh)
    def counterfactual_rows(self, rows: np.ndarray, words, cutoff: float = 0.5, device_ms: bool = False):
        """Encoded rows (N, 24) or packed (N, 16) and numeric row words -> (proba float64 (N,), records (N, len(words)) of
        ``COUNTERFACTUAL_DTYPE``[, device ms]): per row and word, the nearest float32 values below and above the row's value
        whose decision ``p1 > cutoff`` differs from the row's, with p1 there (NaN: none on that side)."""
        rows = np.ascontiguousarray(rows)
        w = np.ascontiguousarray(words, dtype=np.int32)
        n = rows.shape[0]
        proba = np.empty(n, dtype=np.float64)
        out = np.empty((n, len(w)), dtype=_cabi.COUNTERFACTUAL_DTYPE)
        ms = C.c_float(0.0)
        check(self._lib.b2f_counterfactual(self._h, ptr(rows), n, self._fmt(rows), ptr(w), len(w), float(cutoff), ptr(proba), ptr(out),
                                           C.byref(ms)), "b2f_counterfactual")
        return (proba, out, ms.value) if device_ms else (proba, out)

    def counterfactual_device(self, rows_dev: int, n: int, words, cutoff: float, proba_dev: int, out_dev: int, fmt: int = ROWS_WORDS24) -> None:
        """Enqueue the counterfactuals of device-resident rows into device proba (n doubles; 0: not written) and out (n x
        len(words) records); ``sync`` waits."""
        w = np.ascontiguousarray(words, dtype=np.int32)
        check(self._lib.b2f_counterfactual_device(self._h, rows_dev, n, fmt, ptr(w), len(w), float(cutoff), proba_dev, out_dev),
              "b2f_counterfactual_device")

    # ------------------------------------------------------------------ permutation importance (csrc/permutation_importance.cuh)
    def permutation_scores(self, rows: np.ndarray, labels, perm: np.ndarray, words, device_ms: bool = False):
        """Encoded rows (N, 24) or packed (N, 16), 0/1 labels (N,), permutations (R, N) of row indices and probed row words
        -> (records (len(words), R) of ``PERM_SCORE_DTYPE``, baseline record[, device ms]): the metric sums of the rows
        scored with each word taken from row ``perm[r, i]``, and of the rows as they are (``importance.py`` turns them into
        scores)."""
        rows = np.ascontiguousarray(rows)
        y = np.ascontiguousarray(labels, dtype=np.int32)
        p = np.ascontiguousarray(perm, dtype=np.int32)
        w = np.ascontiguousarray(words, dtype=np.int32)
        n_repeats = p.shape[0] if p.ndim == 2 else 0
        if y.shape != (rows.shape[0],) or p.ndim != 2 or p.shape[1] != rows.shape[0]:
            raise ValueError(f"labels {y.shape} and perm {p.shape} must be ({rows.shape[0]},) and (n_repeats, {rows.shape[0]})")
        out = np.zeros((len(w), max(n_repeats, 1)), dtype=_cabi.PERM_SCORE_DTYPE)
        base = np.zeros(1, dtype=_cabi.PERM_SCORE_DTYPE)
        ms = C.c_float(0.0)
        check(self._lib.b2f_permutation_scores(self._h, ptr(rows), rows.shape[0], self._fmt(rows), ptr(y), ptr(p), n_repeats, ptr(w), len(w),
                                               ptr(out), ptr(base), C.byref(ms)), "b2f_permutation_scores")
        return (out, base[0], ms.value) if device_ms else (out, base[0])

    # ------------------------------------------------------------------ MMD drift test (csrc/mmd_drift.cuh)
    def attach_mmd_reference(self, rows: np.ndarray, num_mean, num_scale, sigma: float | None = None, device_ms: bool = False):
        """Encoded reference rows (N, 24) or packed (N, 16), 2 <= N <= 131 072, and the per-numeric mean and scale of the
        embedding -> sigma[, device ms]; ``sigma=None``: alibi's median heuristic on the reference.  Replaces an earlier
        reference."""
        rows = np.ascontiguousarray(rows)
        mean = np.ascontiguousarray(num_mean, dtype=np.float64)
        scale = np.ascontiguousarray(num_scale, dtype=np.float64)
        out, ms = C.c_double(0.0), C.c_float(0.0)
        self.mmd_reference_rows = 0  # a failed attach leaves no reference
        check(self._lib.b2f_model_attach_mmd_reference(self._h, ptr(rows), rows.shape[0], self._fmt(rows), ptr(mean), ptr(scale),
                                                       float("nan") if sigma is None else float(sigma), C.byref(out), C.byref(ms)),
              "b2f_model_attach_mmd_reference")
        self.mmd_reference_rows = rows.shape[0]
        return (out.value, ms.value) if device_ms else out.value

    def mmd_statistics(self, rows: np.ndarray, subsets: np.ndarray, device_ms: bool = False):
        """Encoded batch rows (M, 24) or packed (M, 16), M >= 2, and (B, min(M, N_ref)) sorted pool indices -> (observed
        mmd^2, float64 (B,) permuted mmd^2[, device ms]) against the attached reference (``mmd.py`` draws the subsets)."""
        rows = np.ascontiguousarray(rows)
        sub = np.ascontiguousarray(subsets, dtype=np.int32)
        if sub.ndim != 2:
            raise ValueError(f"subsets must be (n_permutations, subset size), not {sub.shape}")
        if self.mmd_reference_rows and sub.shape[1] != min(rows.shape[0], self.mmd_reference_rows):
            raise ValueError(f"subsets hold {sub.shape[1]} indices each; this batch needs min({rows.shape[0]}, {self.mmd_reference_rows})")
        perm = np.empty(sub.shape[0], dtype=np.float64)
        obs, ms = C.c_double(0.0), C.c_float(0.0)
        check(self._lib.b2f_mmd_drift(self._h, ptr(rows), rows.shape[0], self._fmt(rows), ptr(sub), sub.shape[0], C.byref(obs), ptr(perm),
                                      C.byref(ms)), "b2f_mmd_drift")
        return (obs.value, perm, ms.value) if device_ms else (obs.value, perm)

    # ------------------------------------------------------------------ k-nearest reference rows of trust scores (csrc/knn.cuh)
    def attach_knn_reference(self, rows: np.ndarray, classes, num_mean, num_scale) -> None:
        """Encoded reference rows (N, 24) or packed (N, 16), 2 <= N <= 131 072, their classes (0 / 1, each present) and the
        per-numeric mean and scale of the embedding.  Replaces an earlier reference; a failed attach leaves none."""
        rows = np.ascontiguousarray(rows)
        cls = np.ascontiguousarray(classes, dtype=np.int32)
        if cls.shape != (rows.shape[0],):
            raise ValueError(f"classes must be ({rows.shape[0]},), not {cls.shape}")
        mean = np.ascontiguousarray(num_mean, dtype=np.float64)
        scale = np.ascontiguousarray(num_scale, dtype=np.float64)
        self.knn_class_rows = (0, 0)
        check(self._lib.b2f_model_attach_knn_reference(self._h, ptr(rows), rows.shape[0], self._fmt(rows), ptr(cls), ptr(mean), ptr(scale)),
              "b2f_model_attach_knn_reference")
        self.knn_class_rows = (int((cls == 0).sum()), int((cls == 1).sum()))

    def knn(self, rows: np.ndarray, k: int, device_ms: bool = False):
        """Encoded query rows (M, 24) or packed (M, 16), M >= 1 -> (float64 (M, 2, k) distances, int32 (M, 2, k) reference row
        indices[, device ms]): per class the k nearest reference rows, ordered by (distance, index)."""
        rows = np.ascontiguousarray(rows)
        n = rows.shape[0]
        dist = np.empty((n, 2, max(int(k), 0)), dtype=np.float64)
        index = np.empty((n, 2, max(int(k), 0)), dtype=np.int32)
        ms = C.c_float(0.0)
        check(self._lib.b2f_knn(self._h, ptr(rows), n, self._fmt(rows), int(k), ptr(dist), ptr(index), C.byref(ms)), "b2f_knn")
        return (dist, index, ms.value) if device_ms else (dist, index)

    # ------------------------------------------------------------------ device-resident interface
    def device_alloc(self, nbytes: int) -> int:
        p = self._lib.b2f_device_alloc(self._h, nbytes)
        if not p:
            raise B2FError(f"b2f_device_alloc({nbytes}) failed: {_cabi.last_error()}")
        return p

    def device_free(self, dptr: int) -> None:
        self._lib.b2f_device_free(self._h, dptr)

    def h2d(self, dptr: int, a: np.ndarray) -> None:
        a = np.ascontiguousarray(a)
        check(self._lib.b2f_copy_h2d(self._h, dptr, ptr(a), a.nbytes), "b2f_copy_h2d")

    def d2h(self, a: np.ndarray, dptr: int) -> None:
        check(self._lib.b2f_copy_d2h(self._h, ptr(a), dptr, a.nbytes), "b2f_copy_d2h")

    def predict_device(self, rows_dev: int, n: int, proba_dev: int, proba_is_f64: bool, label_dev: int, packed: bool = False, fmt: int | None = None) -> None:
        check(
            self._lib.b2f_predict_device_ex(self._h, rows_dev, n, fmt if fmt is not None else (ROWS_PACKED64 if packed else ROWS_WORDS24), proba_dev, int(proba_is_f64), label_dev),
            "b2f_predict_device_ex",
        )

    def sync(self) -> None:
        check(self._lib.b2f_sync(self._h), "b2f_sync")

    def predict_device_timed(self, rows_dev, n, proba_dev, proba_is_f64, label_dev, iters: int, flush_l2: bool) -> np.ndarray:
        ms = np.zeros(iters, dtype=np.float32)
        check(
            self._lib.b2f_predict_device_timed(
                self._h, rows_dev, n, proba_dev, int(proba_is_f64), label_dev, iters, int(flush_l2), ptr(ms)
            ),
            "b2f_predict_device_timed",
        )
        return ms

    def predict_stream_timed(self, rows_dev, n, pool, proba_dev, proba_is_f64, label_dev, steps: int, packed: bool = False, fmt: int | None = None,
                             per_launch: bool = True):
        """``steps`` launches cycling over ``pool`` device-resident batches -> (ms_each or None, ms_total).
        ``per_launch=False`` records no events between launches (back-to-back launches of the rank kernel then overlap)."""
        ms = np.zeros(steps, dtype=np.float32) if per_launch else None
        tot = C.c_float(0.0)
        if fmt is None:
            fmt = ROWS_PACKED64 if packed else ROWS_WORDS24
        check(
            self._lib.b2f_predict_stream_timed_ex(self._h, rows_dev, n, fmt, pool, proba_dev, int(proba_is_f64), label_dev, steps, ptr(ms), C.byref(tot)),
            "b2f_predict_stream_timed_ex",
        )
        return ms, float(tot.value)

    # ------------------------------------------------------------------ moments
    def moments(self, rows: np.ndarray) -> np.ndarray:
        """Per-word (count, mean, M2) over host rows -> float64 (24, 3)."""
        rows = np.ascontiguousarray(rows)
        out = np.zeros(MOMENT_VALUES, dtype=np.float64)
        check(self._lib.b2f_moments(self._h, ptr(rows), rows.shape[0], ptr(out)), "b2f_moments")
        return out.reshape(ROW_WORDS, 3)

    def moments_device(self, rows_dev: int, n: int) -> np.ndarray:
        out = np.zeros(MOMENT_VALUES, dtype=np.float64)
        check(self._lib.b2f_moments_device(self._h, rows_dev, n, ptr(out)), "b2f_moments_device")
        return out.reshape(ROW_WORDS, 3)

    def moments_device_timed(self, rows_dev: int, n: int, iters: int, flush_l2: bool):
        ms = np.zeros(iters, dtype=np.float32)
        out = np.zeros(MOMENT_VALUES, dtype=np.float64)
        check(self._lib.b2f_moments_device_timed(self._h, rows_dev, n, iters, int(flush_l2), ptr(ms), ptr(out)), "b2f_moments_device_timed")
        return ms, out.reshape(ROW_WORDS, 3)

    # ------------------------------------------------------------------ NCCL (one process per GPU)
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = np.zeros(128, dtype=np.uint8)
        check(_cabi.load_library().b2f_comm_unique_id(ptr(buf)), "b2f_comm_unique_id")
        return buf.tobytes()

    def comm_init_rank(self, nranks: int, rank: int, unique_id: bytes) -> None:
        buf = np.frombuffer(unique_id, dtype=np.uint8)
        check(self._lib.b2f_comm_init_rank(self._h, nranks, rank, ptr(buf)), "b2f_comm_init_rank")

    def moments_allgather(self, local: np.ndarray) -> np.ndarray:
        local = np.ascontiguousarray(local, dtype=np.float64).reshape(-1)
        out = np.zeros(MOMENT_VALUES, dtype=np.float64)
        check(self._lib.b2f_moments_allgather(self._h, ptr(local), ptr(out)), "b2f_moments_allgather")
        return out.reshape(ROW_WORDS, 3)


_FMT_OVERRIDE = {"ranked": ROWS_RANKED}.get(os.environ.get("B200_SCORER_ROWS", ""))
STREAMED_RANK_MIN_ROWS = 16384  # below this a streamed rank layout loses to the float32-row latency kernels


class Scorer:
    """Owner of a ``b2f_scorer*``: DataFrame columns -> encode (worker threads, pinned staging) -> H2D -> kernel -> D2H,
    chunk by chunk (``csrc/scorer.h``).  One job at a time."""

    def __init__(self, engine: "ForestEngine", encoder, threads: int = 0):
        self._lib = engine._lib
        self.engine, self.encoder = engine, encoder
        h_enc = encoder._native_handle()
        if h_enc is None:
            raise B2FError("the native row encoder is not available")
        # Which rows the workers write.  The host is the bound of this path (a container gets a few CPUs; the GPU scores a
        # 65 536-row chunk in far less time than they take to encode it), so the format is chosen by HOST cost: the 32-byte
        # ranked rows need 14 rank lookups per row on top of what the 64-byte float32 rows cost.  Ranked rows are for callers that
        # stream PRE-ENCODED rows through the C ABI, where PCIe bytes are the bound; B200_SCORER_ROWS=ranked selects them here too.
        self.fmt = self.fmt_small = ROWS_PACKED64 if encoder.packed_ok else ROWS_WORDS24
        self.rank_min_rows = 0
        info = engine.info()
        want_ranked = _FMT_OVERRIDE == ROWS_RANKED or not encoder.packed_ok
        if want_ranked and encoder.ranked_ok and info["rank_ok"] and self._lib.b2f_encoder_attach_ranker(h_enc, encoder._ranker) == 0:
            encoder._ranker_attached = True
            self.fmt = ROWS_RANKED
            # a forest whose rank layout STREAMS through shared memory pays a full pass over it per launch: small requests keep
            # the float32 rows and the latency kernels (split / warp-per-row), large ones take the ranked rows
            self.rank_min_rows = STREAMED_RANK_MIN_ROWS if info["rank_stream"] else 0
        self._h = self._lib.b2f_scorer_create(engine.handle, h_enc, int(threads))
        if not self._h:
            raise B2FError(f"b2f_scorer_create failed: {_cabi.last_error()}")
        self.threads = self._lib.b2f_scorer_threads(self._h)

    def close(self) -> None:
        if getattr(self, "_h", None):
            self._lib.b2f_scorer_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def start(self, n: int, columns, out_mode: int = OUT_F64, chunk_rows: int = 0, fmt: int | None = None) -> int:
        """``columns``: what ``RowEncoder.frame_columns`` returned.  -> number of chunks."""
        scol, ptrs, strides, _keep = columns
        if fmt is None:
            fmt = self.fmt if n >= self.rank_min_rows else self.fmt_small
        if fmt == ROWS_RANKED and not getattr(self.encoder, "_ranker_attached", False):
            # an explicit request for ranked rows on a scorer that writes float32 rows by default: hand the encoder the tables now
            # (no job is in flight: one job at a time)
            if not (self.encoder.ranked_ok and self.engine.info()["rank_ok"]
                    and self._lib.b2f_encoder_attach_ranker(self.encoder._native_handle(), self.encoder._ranker) == 0):
                raise ValueError("ranked rows are not available for this model")
            self.encoder._ranker_attached = True
        self.last_fmt = fmt
        rc = self._lib.b2f_scorer_start(self._h, n, scol, ptrs, ptr(strides), fmt, out_mode, chunk_rows)
        if rc == -7:
            raise ValueError("Input X contains infinity or a value too large for dtype('float32').")
        if rc < 0:
            raise B2FError(f"b2f_scorer_start failed (rc={rc}): {_cabi.last_error()}")
        self._n, self._mode = n, out_mode
        self._chunk = self._lib.b2f_scorer_chunk_rows(self._h)
        lo, cnt = C.c_int64(0), C.c_int64(0)
        self.bounds = []  # chunk c = rows [bounds[c], bounds[c + 1])
        for c in range(max(rc, 0)):
            check(self._lib.b2f_scorer_chunk_range(self._h, c, C.byref(lo), C.byref(cnt)), "b2f_scorer_chunk_range")
            self.bounds.append(lo.value)
        self.bounds.append(n)
        return rc

    def wait(self, chunk: int) -> None:
        rc = self._lib.b2f_scorer_wait(self._h, chunk)
        if rc == -7:
            raise ValueError("Input X contains infinity or a value too large for dtype('float32').")
        check(rc, "b2f_scorer_wait")

    def results(self) -> np.ndarray:
        """View over the pinned result buffer of the current job (valid until the next ``start``)."""
        dt = {OUT_F32: np.dtype(np.float32), OUT_F64: np.dtype(np.float64), OUT_FULL: _cabi.SCORED_FULL_DTYPE}[self._mode]
        addr = self._lib.b2f_scorer_results(self._h)
        buf = (C.c_uint8 * (self._n * dt.itemsize)).from_address(addr)
        return np.frombuffer(buf, dtype=dt, count=self._n)

    @property
    def chunk_rows(self) -> int:
        return self._chunk


def _row_format(rows: np.ndarray, rank_words: int = 0) -> int:
    """Row layout from the array shape: (N, 24) words, (N, 16) packed, (N, rank_words) ranked rows (the model's own
    ``rank_row_bytes / 4``: 8 words for the credit-default schema; never 16 or 24)."""
    if rows.dtype == np.uint32 and rows.ndim == 2:
        if rows.shape[1] == ROW_WORDS:
            return ROWS_WORDS24
        if rows.shape[1] == PACKED_ROW_WORDS:
            return ROWS_PACKED64
        if rank_words and rows.shape[1] == rank_words:
            return ROWS_RANKED
    raise ValueError(f"rows must be uint32 (N, {ROW_WORDS}), packed (N, {PACKED_ROW_WORDS})" + (f" or ranked (N, {rank_words})" if rank_words else ""))


def blob_split_values(blob: bytes, word: int) -> np.ndarray:
    """The sorted distinct float32 split values of numeric row word ``word`` over a forest blob (``b2f_blob_split_values``;
    needs no GPU)."""
    lib = _cabi.load_library()
    buf = np.frombuffer(blob, dtype=np.uint8)
    n = lib.b2f_blob_split_values(ptr(buf), buf.size, int(word), None, 0)
    check(min(int(n), 0), "b2f_blob_split_values")
    out = np.empty(int(n), dtype=np.float32)
    check(min(int(lib.b2f_blob_split_values(ptr(buf), buf.size, int(word), ptr(out), out.size)), 0), "b2f_blob_split_values")
    return out


def _probe_table(probes) -> np.ndarray:
    """[(row word, grid offset, count)] -> b2f_pd_probe records."""
    return np.array([tuple(int(v) for v in p) for p in probes], dtype=_cabi.PD_PROBE_DTYPE)


def _pair_probe_table(probes) -> np.ndarray:
    """[(word a, word b or -1, point offset, count)] -> b2f_pair_probe records."""
    return np.array([tuple(int(v) for v in p) for p in probes], dtype=_cabi.PAIR_PROBE_DTYPE)


def _ale_probe_table(probes) -> np.ndarray:
    """[(row word, edge offset, bins)] -> b2f_ale_probe records."""
    return np.array([tuple(int(v) for v in p) for p in probes], dtype=_cabi.ALE_PROBE_DTYPE)


def moments_merge(parts: np.ndarray) -> np.ndarray:
    """Chan merge of k (24, 3) partials (host)."""
    parts = np.ascontiguousarray(parts, dtype=np.float64).reshape(-1, MOMENT_VALUES)
    out = np.zeros(MOMENT_VALUES, dtype=np.float64)
    _cabi.load_library().b2f_moments_merge(ptr(parts), parts.shape[0], ptr(out))
    return out.reshape(ROW_WORDS, 3)


class EngineGroup:
    """The same forest replicated on several GPUs of one box; batches are sliced across them
    by one C call (``b2f_predict_multi``) -- rows are independent, so no collective on this path.
    The reference's analogue is the k8s Service in front of pod replicas (``kubernetes/manifest.yml:23-36``)."""

    def __init__(self, flat: FlatForest, devices=None, nccl: bool = False):
        if devices is None:
            devices = list(range(device_count()))
        self.engines = [ForestEngine(flat, d) for d in devices]
        self._lib = _cabi.load_library()
        self._handles = (C.c_void_p * len(self.engines))(*[e.handle for e in self.engines])
        if nccl and len(self.engines) > 1:
            check(self._lib.b2f_comm_init_all(self._handles, len(self.engines)), "b2f_comm_init_all")

    def close(self) -> None:
        for a in getattr(self, "_striped", []):
            self._lib.b2f_pinned_free_striped(a)
        self._striped = []
        for e in self.engines:
            e.close()

    def predict_rows(self, rows: np.ndarray, proba_dtype=np.float64, out_proba=None, out_label=None):
        rows = np.ascontiguousarray(rows)
        n = rows.shape[0]
        f64 = np.dtype(proba_dtype) == np.float64
        proba = out_proba if out_proba is not None else np.empty(n, dtype=np.float64 if f64 else np.float32)
        label = out_label if out_label is not None else np.empty(n, dtype=np.int32)
        check(
            self._lib.b2f_predict_multi_ex(self._handles, len(self.engines), ptr(rows), n, self.engines[0]._fmt(rows), ptr(proba), int(f64), ptr(label)),
            "b2f_predict_multi_ex",
        )
        return proba, label

    def attach_outlier_forest(self, blob: bytes) -> None:
        for e in self.engines:
            e.attach_outlier_forest(blob)

    def predict_full(self, rows: np.ndarray, out: np.ndarray | None = None) -> np.ndarray:
        rows = np.ascontiguousarray(rows)
        n = rows.shape[0]
        if out is None:
            out = np.empty(n, dtype=_cabi.SCORED_FULL_DTYPE)
        check(
            self._lib.b2f_predict_multi_ex(self._handles, len(self.engines), ptr(rows), n, self.engines[0]._fmt(rows), ptr(out), OUT_FULL, None),
            "b2f_predict_multi_ex",
        )
        return out

    def pinned_striped(self, dtype, shape, stripe_rows: int) -> np.ndarray:
        """A page-locked array whose row stripes (``stripe_rows`` rows each, dealt round-robin) sit on the NUMA node of the GPU
        that will copy them (``b2f_pinned_alloc_striped``).  Kept alive by the group; freed in ``close``."""
        dt = np.dtype(dtype)
        row_bytes = dt.itemsize * int(np.prod(shape[1:])) if len(shape) > 1 else dt.itemsize
        total = row_bytes * int(shape[0])
        addr = self._lib.b2f_pinned_alloc_striped(self._handles, len(self.engines), stripe_rows * row_bytes, total)
        if not addr:
            raise B2FError(f"b2f_pinned_alloc_striped failed: {_cabi.last_error()}")
        self._striped = getattr(self, "_striped", []) + [addr]
        return np.frombuffer((C.c_uint8 * total).from_address(addr), dtype=dt).reshape(shape)

    def predict_stream(self, rows: np.ndarray, batch: int, out_proba: np.ndarray, out_label: np.ndarray | None, inflight: int = 2) -> None:
        """Deal a long stream in ``batch``-row batches round-robin over the GPUs (one host thread per GPU inside
        the C call, ``inflight`` batches in flight per GPU).  Buffers should be pinned."""
        check(
            self._lib.b2f_predict_stream(
                self._handles, len(self.engines), ptr(rows), rows.shape[0], int(batch), self.engines[0]._fmt(rows), ptr(out_proba),
                int(out_proba.dtype == np.float64), ptr(out_label), int(inflight)
            ),
            "b2f_predict_stream",
        )

    def moments(self, rows: np.ndarray) -> np.ndarray:
        rows = np.ascontiguousarray(rows)
        out = np.zeros(MOMENT_VALUES, dtype=np.float64)
        check(self._lib.b2f_moments_multi(self._handles, len(self.engines), ptr(rows), rows.shape[0], ptr(out)), "b2f_moments_multi")
        return out.reshape(ROW_WORDS, 3)
