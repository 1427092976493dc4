"""Batch drift scores on the GPU (K3): the drop-in for the reference's ``TabularDrift`` detector.

The reference builds ``alibi_detect.cd.TabularDrift(x_ref, p_val=0.05, categories_per_feature={0..8: None})``
on the 30 000 x 23 curated table (``databricks/src/02-register-model.ipynb:224-229``), calls
``self.drift.predict(df[all_features].values)`` per request (``:338``) and returns ``1 - p_val`` per
feature (``:345-349``).  alibi-detect (pinned 0.12.0, ``app/requirements.txt:6``) is neither vendored in the
reference nor installed in this image; what its ``feature_score`` computes is restated in ``oracle/drift.py``:

* categorical feature: chi-squared test on the 2 x K table of reference vs batch counts over the UNION of the
  categories seen in either (``scipy.stats.chi2_contingency``);
* numeric feature: two-sided two-sample Kolmogorov-Smirnov test, exact p-value (``scipy.stats.ks_2samp``);
* p-values kept as float32, the response carries ``1 - p_val``.

Here the reference table is uploaded once (numeric columns pre-sorted, category counts pre-computed -- the
reference re-sorts / re-counts its 30 000 rows on every request) and every request is two small host->device
copies and two kernels (``csrc/drift_stats.cuh``): binary-search histograms + prefix sums for the exact integer K-S
numerator, an anti-diagonal sweep of the lattice-path recursion for the exact p-value, and the chi-squared tail.
The host side below only turns strings into category indices.  No CPU fallback: without the CUDA engine, creating
the detector fails.

Parity status: checked against scipy through ``oracle/drift.py`` (|dp| <= 1e-9); unpinned against alibi-detect
itself, which is absent (DESIGN.md).
"""

from __future__ import annotations

import ctypes as C
import json
import threading

import numpy as np
import pandas as pd

from . import _cabi
from ._cabi import B2FError, check, ptr


class TabularDrift:
    def __init__(self, reference: pd.DataFrame, cat_features, device: int | None = 0):
        """``device=None`` only prepares the reference statistics (for ``save``); scoring needs a device."""
        cat_set = set(cat_features)
        self.features = [str(c) for c in reference.columns]
        self.cat_features = [c for c in self.features if c in cat_set]
        self.num_features = [c for c in self.features if c not in cat_set]
        self.n_ref = len(reference)
        self.ref_sorted = {name: np.sort(reference[name].to_numpy(dtype=np.float64)) for name in self.num_features}
        for name, col in self.ref_sorted.items():  # np.sort puts NaN last
            if len(col) and np.isnan(col[-1]):
                # scipy's K-S (and so alibi-detect) would answer NaN for this feature on every request: refuse the reference instead
                raise ValueError(f"drift reference column {name!r} holds {int(np.isnan(col).sum())} NaN value(s); "
                                 "drop or impute them before building the detector")
        self.ref_cats, self.ref_counts = {}, {}
        for name in self.cat_features:
            cats, counts = np.unique(reference[name].astype(str).to_numpy(), return_counts=True)
            self.ref_cats[name] = cats
            self.ref_counts[name] = counts.astype(np.int64)
        self._host_init()
        if device is not None:
            self._open(device)

    # ------------------------------------------------------------------ device state
    def _host_init(self) -> None:
        self._h = None
        self._index = {name: {v: i for i, v in enumerate(self.ref_cats[name].tolist())} for name in self.cat_features}
        # output position of every feature: the C ABI returns categorical features first, then numeric ones
        order = self.cat_features + self.num_features
        self._perm = np.array([order.index(f) for f in self.features], dtype=np.int64)
        self.last_device_ms = 0.0
        self._num_pos, self._cat_pos = {}, {}  # column positions per columns Index (encode.column_positions)

    def _open(self, device: int, handles: int | None = None) -> None:
        """Upload the reference table.  ``handles`` (default ``B200_DRIFT_HANDLES`` or 4) independent device states,
        each with its own stream and scratch, let that many requests be scored concurrently: one request occupies
        one CTA per feature (23 of the 132 SMs), and the server scores every request's drift on its own thread."""
        import os

        self._lib = _cabi.load_library()
        self.device = int(device)
        ref = np.ascontiguousarray(np.stack([self.ref_sorted[n] for n in self.num_features])) if self.num_features else np.zeros((0, self.n_ref))
        sizes = np.array([len(self.ref_cats[n]) for n in self.cat_features], dtype=np.int32)
        counts = np.concatenate([self.ref_counts[n] for n in self.cat_features]).astype(np.int64) if self.cat_features else np.zeros(0, np.int64)
        k = max(1, int(handles if handles is not None else os.environ.get("B200_DRIFT_HANDLES", "4")))
        self._handles, self._locks = [], []
        for _ in range(k):
            h = self._lib.b2f_drift_create(self.device, self.n_ref, len(self.num_features), ptr(ref), len(self.cat_features), ptr(sizes), ptr(counts))
            if not h:
                msg = _cabi.last_error()
                self.close()
                raise B2FError(f"b2f_drift_create(device={device}) failed: {msg}")
            self._handles.append(h)
            self._locks.append(threading.Lock())
        self._h = self._handles[0]
        self._next = 0

    def close(self) -> None:
        for h in getattr(self, "_handles", []):
            self._lib.b2f_drift_destroy(h)
        self._handles = []
        self._h = None
        if getattr(self, "_enc", None) is not None:
            self._enc_lib.b2f_encoder_destroy(self._enc)
            self._enc = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def launches(self) -> int:
        return sum(int(self._lib.b2f_drift_launches(h)) for h in self._handles)

    # ------------------------------------------------------------------ scoring
    def encode_batch(self, batch: pd.DataFrame):
        """Host half of a request (no device needed): -> (x float64 (n_num, n), codes int32 (n_cat, n) with -1 for
        values outside the reference categories, new_off int32 (n_cat + 1), new_counts int64 -- the counts of those
        outside values, one entry per distinct value)."""
        n = len(batch)
        nn, nc = len(self.num_features), len(self.cat_features)
        x = np.empty((nn, n), dtype=np.float64)
        try:  # block-manager access: a Series per column costs more than everything else at request size
            from .encode import column_positions

            pos = column_positions(batch, self.num_features, self._num_pos)
            fetch = batch._mgr.iget_values
            for k, i in enumerate(pos):
                if i < 0:
                    raise KeyError(self.num_features[k])
                x[k] = fetch(int(i))
        except (AttributeError, TypeError, ValueError):
            for k, name in enumerate(self.num_features):
                x[k] = batch[name].to_numpy(dtype=np.float64)
        codes = np.empty((nc, n), dtype=np.int32)
        new_off = np.zeros(nc + 1, dtype=np.int32)
        new_counts = []
        # Arrow-backed string columns: the native encoder's perfect-hash lookup over the buffers (no per-column pandas hashing, no
        # per-row Python); only a column that holds values outside the reference categories still goes through the general path
        native_ok = np.zeros(nc, dtype=bool)
        if nc and self._native_codes(batch, codes):
            native_ok = (codes >= 0).all(axis=1)
        for c, name in enumerate(self.cat_features):
            idx = self._index[name]
            if native_ok[c]:
                new_off[c + 1] = len(new_counts)
                continue
            if n <= 128:  # request-sized batches: a Python loop beats the vectorised machinery
                # missing values (None / NaN) are outside the reference's contract (alibi-detect's np.unique raises on
                # them); both paths here count them as one category "nan"
                vals = [v if type(v) is str else ("nan" if (v is None or v != v) else str(v)) for v in batch[name].tolist()]
                col = np.fromiter((idx.get(v, -1) for v in vals), dtype=np.int32, count=n)
                unseen = {}
                for v, k in zip(vals, col.tolist()):
                    if k < 0:
                        unseen[v] = unseen.get(v, 0) + 1
            else:  # hash the column once, look up only its distinct values
                inv, uniq = pd.factorize(batch[name], use_na_sentinel=False)
                names = [u if type(u) is str else ("nan" if (u is None or u != u) else str(u)) for u in uniq]
                mapped = np.fromiter((idx.get(v, -1) for v in names), dtype=np.int32, count=len(names))
                col = mapped[inv]
                unseen = {}
                if (mapped < 0).any():
                    cnt = np.bincount(inv, minlength=len(names))
                    for v, k, q in zip(names, mapped.tolist(), cnt.tolist()):
                        if k < 0:
                            unseen[v] = unseen.get(v, 0) + q
            codes[c] = col
            # values outside the reference categories: each distinct one is a column of its own in the contingency table
            new_counts.extend(unseen[v] for v in sorted(unseen))
            new_off[c + 1] = len(new_counts)
        return x, codes, new_off, np.asarray(new_counts, dtype=np.int64)

    def _native_codes(self, batch: pd.DataFrame, codes: np.ndarray) -> bool:
        """codes[c, i] = index of batch[cat c][i] among the reference categories (-1: not one of them) through
        b2f_encoder_codes; False when the columns are not Arrow-backed strings (the caller takes the general path)."""
        from .encode import NATIVE_THREADS, arrow_string_columns, column_positions

        got = arrow_string_columns(batch, self.cat_features, column_positions(batch, self.cat_features, self._cat_pos))
        if got is None:
            return False
        if getattr(self, "_enc", None) is None:
            lib = _cabi.load_library()
            blobs = [str(v).encode("utf-8") for name in self.cat_features for v in self.ref_cats[name].tolist()]
            offsets = np.zeros(len(blobs) + 1, dtype=np.int64)
            np.cumsum([len(b) for b in blobs], out=offsets[1:])
            counts = np.array([len(self.ref_cats[name]) for name in self.cat_features], dtype=np.int32)
            nulls = np.array([self._index[name].get("nan", -1) for name in self.cat_features], dtype=np.int32)  # missing counts as "nan"
            h = lib.b2f_encoder_create(len(self.cat_features), 0, ptr(counts), b"".join(blobs), ptr(offsets), ptr(nulls))
            if not h:
                return False
            self._enc, self._enc_lib = h, lib
        scol, _keep = got
        return self._enc_lib.b2f_encoder_codes(self._enc, len(batch), scol, ptr(codes), NATIVE_THREADS) == 0

    def statistics(self, batch: pd.DataFrame):
        """-> (p float64, stat float64, flags int32), each in ``self.features`` order."""
        n = len(batch)
        if n < 1:
            raise ValueError("Data passed to ks_2samp must not be empty")
        if not self._h:
            raise B2FError("drift detector has no device state (created with device=None or closed); there is no CPU fallback")
        nn, nc = len(self.num_features), len(self.cat_features)
        x, codes, new_off, newc = self.encode_batch(batch)
        F = nn + nc
        p, stat, flags = np.empty(F), np.empty(F), np.empty(F, dtype=np.int32)
        ms = C.c_float(0.0)
        k = self._next = (self._next + 1) % len(self._handles)  # round-robin; a benign race only skews the rotation
        with self._locks[k]:
            check(
                self._lib.b2f_drift_score(self._handles[k], n, ptr(x), ptr(codes), ptr(new_off) if len(newc) else None,
                                          ptr(newc) if len(newc) else None, ptr(p), ptr(stat), ptr(flags), C.byref(ms)),
                "b2f_drift_score",
            )
        self.last_device_ms = float(ms.value)
        # flags == 1 (lcm of the sample sizes >= 2^31, batches of >= 71 583 rows against the 30 000-row table): scipy itself
        # leaves the exact method for kstwo.sf(D, round(m n / (m + n))); the library has applied that formula (b2f_kstwo_sf)
        return p[self._perm], stat[self._perm], flags[self._perm]

    def p_values(self, batch: pd.DataFrame) -> np.ndarray:
        """float32 p-value per feature (alibi-detect stores them in a float32 array)."""
        return self.statistics(batch)[0].astype(np.float32)

    def score(self, batch: pd.DataFrame) -> list:
        """``(1 - p_val).tolist()`` as in 02-register-model.ipynb:345-349 (float32 arithmetic)."""
        return (np.float32(1) - self.p_values(batch)).tolist()

    # ------------------------------------------------------------------ persistence
    def save(self, path: str) -> None:
        arrays = {f"sorted__{k}": v for k, v in self.ref_sorted.items()}
        arrays.update({f"cats__{k}": v.astype("U") for k, v in self.ref_cats.items()})
        arrays.update({f"counts__{k}": v for k, v in self.ref_counts.items()})
        arrays["meta"] = np.array(json.dumps(dict(features=self.features, cat_features=self.cat_features, n_ref=self.n_ref)))
        np.savez_compressed(path, **arrays)

    @classmethod
    def load(cls, path: str, device: int = 0) -> "TabularDrift":
        self = cls.__new__(cls)
        with np.load(path) as z:
            meta = json.loads(str(z["meta"]))
            self.features, self.cat_features = meta["features"], meta["cat_features"]
            self.num_features = [f for f in self.features if f not in set(self.cat_features)]
            self.ref_sorted = {k[len("sorted__"):]: z[k] for k in z.files if k.startswith("sorted__")}
            self.ref_cats = {k[len("cats__"):]: z[k] for k in z.files if k.startswith("cats__")}
            self.ref_counts = {k[len("counts__"):]: z[k] for k in z.files if k.startswith("counts__")}
        self.n_ref = int(meta.get("n_ref", len(next(iter(self.ref_sorted.values()))) if self.ref_sorted else 0))
        self._host_init()
        self._open(device)
        return self
