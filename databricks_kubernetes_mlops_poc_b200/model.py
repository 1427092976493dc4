"""B200Model: the drop-in for the object ``mlflow.pyfunc.load_model(dir)`` returns in the reference.

Plugin boundary being mirrored (SURVEY.md section 8b):

* reference ``app/main.py:26-28``  ``ml_models["credit_default"] = mlflow.pyfunc.load_model(MODEL_DIRECTORY)``
* reference ``app/main.py:72``     ``model_output = ml_models["credit_default"].predict(input_df)``
* reference ``CustomModel.predict`` (``databricks/src/02-register-model.ipynb:330-353``): returns
  ``{"predictions": [...], "outliers": [...], "feature_drift_batch": {23 names -> float}}``.

``predictions`` (the accelerated path, SURVEY a6) comes from the CUDA engine -- dictionary-encode on
the host into pinned memory, H2D, fused kernel, D2H -- with no CPU fallback.  ``outliers`` (SURVEY a8)
comes from the same pass when an outlier forest is attached: the isolation forest is a second forest
blob walked by the same kernels over the same rows in HBM (``b2f_predict_full``); without one it is the
constant 0 the reference provably returns (its ``IForest(threshold=0.95)`` compares a score bounded by
0.5 with 0.95; SURVEY section 5).  ``feature_drift_batch`` (SURVEY a7) comes from the GPU drift detector
in ``drift.py`` (K3: the reference table resident in HBM, chi-squared and exact K-S p-values per request),
when a reference table is supplied; without one every score is 0.0.
"""

from __future__ import annotations

import os
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pandas as pd

from ._cabi import OUT_F64, OUT_FULL
from ._pylists import ListBuilder
from .encode import RowEncoder
from .engine import EngineGroup, ForestEngine
from .flatten import AGG_RF_MEAN, FlatForest, flatten_explainer, flatten_isolation_forest, flatten_pipeline

BLOB_FILE = "forest.b2f.npz"
OUTLIER_BLOB_FILE = "outlier.b2f"
DRIFT_FILE = "drift_reference.npz"
EXPLAIN_FILE = "explain.b2f"  # TreeSHAP path table (flatten_explainer); optional
BACKGROUND_FILE = "explain_background.npz"  # background rows of interventional explanations (raw columns); optional
OUTLIER_PICKLE = os.path.join("artifacts", "outlier.pkl")  # joblib.dump(outlier, ".../outlier.pkl"), 02-register-model.ipynb:264,326-328
SKLEARN_PICKLE = os.path.join("artifacts", "classifier", "model", "model.pkl")  # MLflow layout, 02-register-model.ipynb:317-321


class B200Model:
    def __init__(self, flat: FlatForest, devices=None, drift=None, proba_dtype=np.float64, outlier_blob: bytes | None = None, host_threads: int = 0,
                 explain_blob: bytes | None = None, explain_background: pd.DataFrame | None = None):
        self.flat = flat
        self.all_features = flat.all_features
        self.categorical_features = list(flat.cat_features)
        self.numeric_features = list(flat.num_features)
        self.encoder = RowEncoder(flat)
        devices = [0] if devices is None else list(devices)
        if len(devices) == 1:
            self.engine = ForestEngine(flat, devices[0])
            self.group = None
        else:
            self.group = EngineGroup(flat, devices)
            self.engine = self.group.engines[0]
        self.drift = drift
        self.proba_dtype = np.dtype(proba_dtype)
        self.classes = np.asarray(flat.classes)
        self._pool = ThreadPoolExecutor(max_workers=2, thread_name_prefix="b200-drift") if drift is not None else None
        self.outlier_blob = outlier_blob
        if outlier_blob is not None:
            (self.group if self.group is not None else self.engine).attach_outlier_forest(outlier_blob)
        # the explainer (TreeSHAP path table) lives on the first GPU only: explain() runs there
        self.explain_blob = explain_blob
        if explain_blob is not None:
            self.engine.attach_explainer(explain_blob)
        self.background_rows = 0
        if explain_background is not None:
            self.attach_background(explain_background)
        # one scoring replica per GPU for the server's round-robin batcher (each has its own handle,
        # pinned staging and worker thread; the forest is replicated, rows are independent)
        engines = self.group.engines if self.group is not None else [self.engine]
        self.replicas = [_Replica(self.encoder, e, outlier_blob is not None, self.numeric_features) for e in engines]
        # the columnar request pipeline of the first GPU (csrc/scorer.h): created on first use
        self._scorer = None
        self._scorer_lock = threading.Lock()
        self.host_threads = int(os.environ.get("B200_HOST_THREADS", host_threads or 0))  # 0: half the CPUs of the GPU's NUMA node
        self._scorer_failed = os.environ.get("B200_SCORER", "1") == "0"
        self.last_timing = None  # seconds spent in the stages of the last large predict(): columns / first chunk / lists

    # ------------------------------------------------------------------ construction
    @classmethod
    def from_pipeline(cls, pipeline, reference_frame: pd.DataFrame | None = None, outlier=None, explain: bool = False,
                      background: pd.DataFrame | None = None, **kw) -> "B200Model":
        """Fitted sklearn Pipeline (the reference's model.pkl) -> model on the GPU.

        ``outlier``: the reference's fitted outlier detector (an alibi-detect ``IForest`` or a bare sklearn
        ``IsolationForest`` plus ``outlier_threshold=``), flattened into a second forest over the same rows.
        ``explain``: also build the TreeSHAP path table, so that ``explain()`` works.  ``background``: a frame of raw rows
        (e.g. the training table) to attach for ``explain_interventional()``; it needs ``explain``."""
        if background is not None and not explain:
            raise ValueError("a background is for interventional explanations: pass explain=True with it")
        flat = flatten_pipeline(pipeline)
        if background is not None:
            kw["explain_background"] = background
        if explain:
            kw["explain_blob"] = flatten_explainer(pipeline, flat)
        drift = None
        if reference_frame is not None:
            from .drift import TabularDrift

            devices = kw.get("devices")
            drift = TabularDrift(reference_frame[flat.all_features], flat.cat_features, device=devices[0] if devices else 0)
        threshold = kw.pop("outlier_threshold", None)
        blob = None
        if outlier is not None:
            blob = flatten_isolation_forest(outlier, len(flat.cat_features), len(flat.num_features),
                                            vocab=[len(c) for c in flat.categories], threshold=threshold)
        return cls(flat, drift=drift, outlier_blob=blob, **kw)

    def close(self) -> None:
        for r in self.replicas:
            if r._scorer is not None:
                r._scorer.close()
                r._scorer = None
        if self._scorer is not None:
            self._scorer.close()
            self._scorer = None
        if self._pool is not None:
            self._pool.shutdown(wait=True)
        if self.drift is not None:
            self.drift.close()
        if self.group is not None:
            self.group.close()
        else:
            self.engine.close()

    # ------------------------------------------------------------------ scoring
    def _score(self, df: pd.DataFrame, want_outliers: bool = False):
        """-> (proba1, label, is_outlier or None); one H2D copy of the encoded rows whichever outputs are wanted."""
        n = len(df)
        # large requests travel as 64-byte packed rows (one third fewer PCIe bytes), encoded natively in one pass
        packed = self.encoder.packed_ok and n > self.encoder.SMALL_BATCH
        rows, proba, label = self.engine.staging(n, packed=packed)
        if packed:
            self.encoder.encode_frame_packed(df, out=rows)
        else:
            self.encoder.encode_frame(df, out=rows)
        target = self.group if self.group is not None else self.engine
        if want_outliers and self.outlier_blob is not None:
            _reject_nan(df, self.numeric_features)
            rec = target.predict_full(rows, out=self.engine.staging_full(n))
            return rec["proba1"], rec["label"], rec["is_outlier"]
        if self.proba_dtype != np.float64:
            proba = proba.view(np.float32)[:n]
        target.predict_rows(rows, proba_dtype=self.proba_dtype, out_proba=proba, out_label=label)
        return proba, label, None

    def predict_proba1(self, df: pd.DataFrame) -> np.ndarray:
        """``classifier.predict_proba(df[all_features])[:, 1]`` (02-register-model.ipynb:335-337)."""
        return np.array(self._score(df)[0], dtype=np.float64)

    def predict_label(self, df: pd.DataFrame) -> np.ndarray:
        """``pipeline.predict(df)`` (hard labels, 01-train-model.ipynb:290)."""
        return self.classes[np.array(self._score(df)[1])]

    PIPELINE_MIN_ROWS = int(os.environ.get("B200_PIPELINE_MIN_ROWS", "1"))  # from here up a request goes through the columnar pipeline

    def _pipeline(self, df: pd.DataFrame):
        """Large requests on one GPU: the DataFrame's column buffers go to the native scorer in ONE call; chunks come back while
        later chunks are still being encoded / copied / scored, and each chunk's Python floats are built as it lands.
        -> (predictions list, outlier-flag list or None), or None when this request has to take the general path."""
        if self._scorer_failed or self.group is not None or len(df) < self.PIPELINE_MIN_ROWS:
            return None
        import time

        t0 = time.perf_counter()
        if self._scorer is None:
            try:
                self._scorer = self.engine.scorer(self.encoder, self.host_threads)
            except Exception:
                self._scorer_failed = True
                return None
        cols = self.encoder.frame_columns(df)
        if cols is None:
            return None
        sc = self._scorer
        n = len(df)
        full = self.outlier_blob is not None
        with self._scorer_lock:  # one job at a time per scorer: concurrent predict() calls on one model take turns
            return self._pipeline_locked(sc, df, n, full, cols, t0)

    def _pipeline_locked(self, sc, df, n, full, cols, t0):
        import time

        if full:
            _reject_nan(df, self.numeric_features)
        t1 = time.perf_counter()
        # classifier only: the scorer's own choice (64-byte float32 rows: cheapest to encode; ranked rows with B200_SCORER_ROWS=ranked);
        # with the outlier forest on the same rows: float32 rows (ranks are relative to ONE forest's split values)
        n_chunks = sc.start(n, cols, out_mode=OUT_FULL if full else OUT_F64, fmt=(1 if self.encoder.packed_ok else 0) if full else None)
        out = sc.results()
        bounds = sc.bounds
        # Python lists are built chunk by chunk while later chunks are in flight (float objects recycled: _pylists.py); what does
        # not depend on the results -- the empty lists, the all-zero outlier list of a classifier-only model -- is made while
        # the first chunk is on its way
        preds = ListBuilder(n)
        flags = ListBuilder(n) if full else None
        zeros = None if full else [0] * n
        t_first = None
        for c in range(n_chunks):
            sc.wait(c)
            if t_first is None:
                t_first = time.perf_counter()
            lo = bounds[c]
            part = out[lo:bounds[c + 1]]
            if full:
                preds.fill(lo, part["proba1"])
                flags.fill(lo, part["is_outlier"])
            else:
                preds.fill(lo, part)
        preds, flags = preds.items, (flags.items if full else zeros)
        t2 = time.perf_counter()
        self.last_timing = {"columns_s": t1 - t0, "first_chunk_s": (t_first or t2) - t1, "chunks_and_lists_s": t2 - t1, "chunks": n_chunks,
                            "threads": sc.threads, "row_format": sc.last_fmt}
        return preds, flags

    def predict(self, model_input) -> dict:
        """Mirror of ``CustomModel.predict(context, model_input)`` (02-register-model.ipynb:330-353)."""
        df = model_input if isinstance(model_input, pd.DataFrame) else pd.DataFrame(model_input)  # never mutated here
        if len(df.columns) == 0:
            # the reference dies in df[self.all_features] on an empty request (-> HTTP 500)
            raise KeyError(f"None of {self.all_features} are in the [columns]")
        # the drift sweep takes milliseconds of device time on its own stream (2.2 ms for 1 000 rows on an H100): start it
        # first, score the rows meanwhile
        pending = self._pool.submit(self.drift.score, df) if self.drift is not None else None
        try:
            preds, flags = self._predictions(df)
        finally:
            drift_scores = pending.result() if pending is not None else [0.0] * len(self.all_features)
        return {
            "predictions": preds,
            "outliers": flags,
            "feature_drift_batch": dict(zip(self.all_features, drift_scores)),
        }


    def _predictions(self, df: pd.DataFrame):
        """-> (predictions list, outlier-flag list): what ``predict`` returns for these rows, without the drift scores."""
        n = len(df)
        fast = self._pipeline(df)
        if fast is not None:
            preds, flags = fast
            return preds, flags if flags is not None else [0] * n
        proba, _, fl = self._score(df, want_outliers=True)
        return proba.tolist(), fl.tolist() if fl is not None else [0] * n

    # ------------------------------------------------------------------ explanations
    @property
    def explainer_attached(self) -> bool:
        return self.explain_blob is not None

    @property
    def explain_output(self) -> str:
        """The space contributions are in: the probability (RandomForest) or the raw margin (GBDT)."""
        return "probability" if self.flat.agg_mode == AGG_RF_MEAN else "log_odds"

    def explain(self, model_input) -> dict:
        """Exact path-dependent TreeSHAP contributions of every request field to every row's score.

        -> ``{"feature_names": all_features, "output": "probability" | "log_odds", "base_value": float,
        "contributions": float64 (n, n_fields), "predictions": the classifier's P(class 1) for these rows}``, with
        ``base_value + contributions[i].sum()`` equal to row i's probability (RandomForest) or raw margin (GBDT; the
        probability is its logistic).  A categorical field is one player, so its contribution is not the sum of per one-hot
        column values other tools report.  Raises RuntimeError when the model has no explainer.

        Everything runs on the FIRST GPU's handle only (the explainer lives there): the contributions, and the predictions,
        which come from that GPU's scoring replica (``replicas[0].score``, the same call the HTTP batcher's first worker makes)
        with the classifier alone.  So a row with a NaN numeric is explained even when an outlier forest is attached (the
        outlier detector, not the classifier, refuses NaN in ``predict``).  On one GPU the predictions are the numbers
        ``predict`` returns; a multi-GPU ``predict`` slices the batch over all GPUs and may differ from them in the last bits.
        Calls on one handle must not overlap: a caller that also scores on ``replicas[0]`` from other threads serialises the
        two (the HTTP server takes the first batcher worker's lock)."""
        return self._explained(model_input, "explain_rows", "contributions")

    def explain_interactions(self, model_input) -> dict:
        """Exact path-dependent SHAP interaction values of every pair of request fields for every row's score.

        -> ``{"feature_names", "output", "base_value", "interactions": float64 (n, n_fields, n_fields), "predictions"}``, the
        other keys as in ``explain``.  ``interactions[i]`` is symmetric; entry ``[a][b]`` (a != b) is half the Shapley
        interaction index of fields a and b, and the diagonal holds what is left of each field's own contribution, so each
        row of the matrix sums to ``explain``'s contribution of that field and the whole matrix to the prediction -
        base_value.  Any model with an explainer has them; the same rules as ``explain`` apply (first GPU's handle only,
        predictions from ``replicas[0].score`` with the classifier alone, RuntimeError without an explainer)."""
        return self._explained(model_input, "explain_interactions_rows", "interactions")

    @property
    def background_attached(self) -> bool:
        return self.background_rows > 0

    def attach_background(self, frame: pd.DataFrame) -> int:
        """Attach the background set of ``explain_interventional``: raw rows (at least one) encoded as requests are, compressed
        once on the first GPU; replaces an earlier background.  -> the device bytes of its table.  RuntimeError without an
        explainer."""
        if self.explain_blob is None:
            raise RuntimeError("a background needs an explainer: build the model with from_pipeline(..., explain=True)")
        nbytes = self.engine.attach_background(self.encoder.encode_frame(frame))
        self.background_rows = len(frame)
        return nbytes

    def explain_interventional(self, model_input) -> dict:
        """Exact interventional TreeSHAP contributions of every request field against the attached background set (what
        shap's ``TreeExplainer(model, data)`` computes): the mean, over background rows z, of each field's Shapley value in
        the game where the fields in S take the row's values and the others z's.  A field the model never reads gets 0, even
        when it is correlated with one it reads.  With a one-row background this is baseline Shapley against that row.

        -> ``explain``'s keys plus ``"background_rows"``; ``base_value`` is the mean over the background of the probability
        (RandomForest) or raw margin (GBDT), and ``base_value + contributions[i].sum()`` row i's.  The same rules as
        ``explain`` apply (first GPU's handle only, predictions from ``replicas[0].score``); RuntimeError without an explainer
        or a background."""
        if self.explain_blob is not None and not self.background_attached:
            raise RuntimeError("this model has no background set: attach_background(frame), from_pipeline(..., background=frame) or a "
                               f"model directory that holds {BACKGROUND_FILE} (save_model_dir(..., explain_background=frame))")
        out = self._explained(model_input, "explain_interventional_rows", "contributions")
        out["background_rows"] = self.background_rows
        return out

    def _explained(self, model_input, method: str, key: str) -> dict:
        """``engine.<method>`` on the encoded rows, answered as ``key`` beside the keys both explanations share."""
        if self.explain_blob is None:
            raise RuntimeError("this model has no explainer: build it with from_pipeline(..., explain=True) or load a model directory "
                               f"that holds {EXPLAIN_FILE} (save_model_dir(..., explain_blob=flatten_explainer(pipeline)))")
        df = model_input if isinstance(model_input, pd.DataFrame) else pd.DataFrame(model_input)
        if len(df.columns) == 0:
            raise KeyError(f"None of {self.all_features} are in the [columns]")
        values, base = getattr(self.engine, method)(self.encoder.encode_frame(df))
        proba, _ = self.replicas[0].score(df, want_outliers=False)
        return {"feature_names": list(self.all_features), "output": self.explain_output, "base_value": float(base),
                key: values, "predictions": proba.tolist()}


def _reject_nan(df: pd.DataFrame, numeric_features) -> None:
    """The reference's outlier detector refuses NaN inputs: scikit-learn 1.1.1 (``app/requirements.txt:14``)
    validates ``IsolationForest.decision_function``'s input with ``force_all_finite=True`` -> ValueError -> HTTP 500."""
    for name in numeric_features:
        if np.isnan(df[name].to_numpy(dtype=np.float64, copy=False)).any():
            raise ValueError("Input X contains NaN.\nIsolationForest does not accept missing values encoded as NaN natively.")


class _Replica:
    """One GPU's view of the model: encode into that engine's pinned staging and score there."""

    def __init__(self, encoder: RowEncoder, engine: ForestEngine, has_outlier: bool = False, numeric_features=()):
        self.encoder, self.engine, self.has_outlier, self.numeric_features = encoder, engine, has_outlier, list(numeric_features)
        self._scorer, self._scorer_failed = None, os.environ.get("B200_SCORER", "1") == "0"

    def _scorer_for(self):
        if self._scorer is None and not self._scorer_failed:
            try:
                self._scorer = self.engine.scorer(self.encoder, int(os.environ.get("B200_HOST_THREADS", "0")))
            except Exception:
                self._scorer_failed = True
        return self._scorer

    def score(self, df: pd.DataFrame, want_outliers: bool = True):
        """-> (proba1 float64 (n,), is_outlier int32 (n,) or None).  ``want_outliers=False``: the classifier alone (no
        outlier forest, so NaN numerics are accepted), on the same row format and kernels as the full pass."""
        n = len(df)
        full = self.has_outlier and want_outliers
        sc = self._scorer_for() if n else None
        cols = self.encoder.frame_columns(df) if sc is not None else None
        if cols is not None:
            # the columnar request pipeline (csrc/scorer.h): column buffers -> encode threads -> H2D -> kernel(s) -> D2H
            if full:
                _reject_nan(df, self.numeric_features)
            n_chunks = sc.start(n, cols, out_mode=OUT_FULL if full else OUT_F64,
                                fmt=(1 if self.encoder.packed_ok else 0) if self.has_outlier else None)
            for c in range(n_chunks):  # chunks ride different streams: each has its own completion event
                sc.wait(c)
            out = sc.results()
            if full:
                return np.array(out["proba1"], dtype=np.float64), np.array(out["is_outlier"])
            return np.array(out, dtype=np.float64), None
        packed = self.encoder.packed_ok and n > self.encoder.SMALL_BATCH
        rows, proba, _ = self.engine.staging(n, packed=packed)
        if packed:
            self.encoder.encode_frame_packed(df, out=rows)
        else:
            self.encoder.encode_frame(df, out=rows)
        if full:
            _reject_nan(df, self.numeric_features)
            rec = self.engine.predict_full(rows, out=self.engine.staging_full(n))
            return np.array(rec["proba1"], dtype=np.float64), np.array(rec["is_outlier"])
        self.engine.predict_rows(rows, proba_dtype=np.float64, want_label=False, out_proba=proba)
        return np.array(proba, dtype=np.float64), None

    def predict_proba1(self, df: pd.DataFrame) -> np.ndarray:
        return self.score(df)[0]


# ---------------------------------------------------------------------- loading
def save_model_dir(path: str, flat: FlatForest, reference_frame: pd.DataFrame | None = None, outlier_blob: bytes | None = None,
                   explain_blob: bytes | None = None, explain_background: pd.DataFrame | None = None) -> None:
    """Write the GPU-side artefact next to (or instead of) the MLflow pickles.  ``explain_blob``: the TreeSHAP path table
    (``flatten_explainer``), written as ``explain.b2f`` so that ``load_model`` attaches it.  ``explain_background``: raw
    rows written as ``explain_background.npz``, attached by ``load_model`` with the explainer."""
    os.makedirs(path, exist_ok=True)
    flat.save(os.path.join(path, BLOB_FILE))
    if explain_blob is not None:
        with open(os.path.join(path, EXPLAIN_FILE), "wb") as f:
            f.write(explain_blob)
    if explain_background is not None:
        _save_background(os.path.join(path, BACKGROUND_FILE), flat, explain_background)
    if outlier_blob is not None:
        with open(os.path.join(path, OUTLIER_BLOB_FILE), "wb") as f:
            f.write(outlier_blob)
    if reference_frame is not None:
        from .drift import TabularDrift

        TabularDrift(reference_frame[flat.all_features], flat.cat_features, device=None).save(os.path.join(path, DRIFT_FILE))


def _save_background(path: str, flat: FlatForest, frame: pd.DataFrame) -> None:
    """The raw columns of ``flat.all_features``: numerics as float64, categories as ``U`` strings with ``null__<name>`` telling
    a string (0) from None (1) and NaN (2), which the encoder maps differently."""
    arrays = {}
    for name in flat.all_features:
        if name in flat.num_features:
            arrays[name] = frame[name].to_numpy(dtype=np.float64)
            continue
        col = frame[name].to_numpy(dtype=object)
        null = np.array([_null_kind(name, v) for v in col], dtype=np.uint8)
        arrays[name] = np.array([v if isinstance(v, str) else "" for v in col], dtype="U")
        arrays[f"null__{name}"] = null
    np.savez(path, **arrays)


def _null_kind(name: str, v) -> int:
    if isinstance(v, str):
        return 0
    if v is None:
        return 1
    if isinstance(v, float) and v != v:
        return 2
    raise ValueError(f"background column {name!r}: {v!r} is not a string, None or NaN")


def _load_background(path: str, flat: FlatForest) -> pd.DataFrame:
    with np.load(path, allow_pickle=False) as z:
        cols = {}
        for name in flat.all_features:
            if name in flat.num_features:
                cols[name] = z[name]
                continue
            v = z[name].astype(object)
            null = z[f"null__{name}"]
            v[null == 1] = None
            v[null == 2] = np.nan
            cols[name] = v
    return pd.DataFrame(cols)


def _load_outlier_blob(path: str, flat: FlatForest):
    """Cached isolation-forest blob, else the reference's ``outlier.pkl`` (needs alibi-detect to unpickle)."""
    cached = os.path.join(path, OUTLIER_BLOB_FILE)
    if os.path.exists(cached):
        with open(cached, "rb") as f:
            return f.read()
    pkl = os.path.join(path, OUTLIER_PICKLE)
    if not os.path.exists(pkl):
        return None
    import joblib

    try:
        detector = joblib.load(pkl)
    except ImportError:  # alibi-detect absent: `outliers` stays the constant 0 the reference's threshold produces anyway
        return None
    blob = flatten_isolation_forest(detector, len(flat.cat_features), len(flat.num_features), vocab=[len(c) for c in flat.categories])
    try:
        with open(cached, "wb") as f:
            f.write(blob)
    except OSError:
        pass
    return blob


def load_model(path: str, devices=None, **kw) -> B200Model:
    """Drop-in for ``mlflow.pyfunc.load_model(path)`` as used at reference ``app/main.py:26-28``.

    Looks for the cached forest blob first; otherwise for the sklearn pipeline pickle in the MLflow
    artefact layout (only loadable when the pickle's sklearn version matches) and flattens it.
    """
    blob_path = os.path.join(path, BLOB_FILE)
    if os.path.exists(blob_path):
        flat = FlatForest.load(blob_path)
    else:
        pkl = os.path.join(path, SKLEARN_PICKLE)
        if not os.path.exists(pkl):
            raise FileNotFoundError(f"neither {blob_path} nor {pkl} exists")
        import joblib

        flat = flatten_pipeline(joblib.load(pkl))
        try:
            flat.save(blob_path)
        except OSError:
            pass  # read-only image: keep the blob in memory only
    if devices is None:
        env = os.environ.get("B200_DEVICES")
        devices = [int(d) for d in env.split(",")] if env else [0]
    drift = None
    drift_path = os.path.join(path, DRIFT_FILE)
    if os.path.exists(drift_path) and os.environ.get("B200_DRIFT", "gpu") != "off":
        from .drift import TabularDrift

        drift = TabularDrift.load(drift_path, device=devices[0])
    outlier_blob = _load_outlier_blob(path, flat) if os.environ.get("B200_OUTLIERS", "gpu") != "off" else None
    explain_path = os.path.join(path, EXPLAIN_FILE)
    if "explain_blob" not in kw and os.path.exists(explain_path) and os.environ.get("B200_EXPLAIN", "gpu") != "off":
        with open(explain_path, "rb") as f:
            kw["explain_blob"] = f.read()
        background_path = os.path.join(path, BACKGROUND_FILE)
        if "explain_background" not in kw and os.path.exists(background_path):
            kw["explain_background"] = _load_background(background_path, flat)
    return B200Model(flat, devices=devices, drift=drift, outlier_blob=outlier_blob, **kw)
