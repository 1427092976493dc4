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

import contextlib
import math
import os
import threading
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pandas as pd

from . import ale, dependence, importance, interaction, mmd, trust
from ._cabi import OUT_F64, OUT_FULL, ROWS_PACKED64, ROWS_WORDS24, B2FError
from ._pylists import ListBuilder
from .encode import RowEncoder
from .engine import EngineGroup, ForestEngine
from .flatten import AGG_RF_MEAN, FlatForest, flatten_explainer, flatten_isolation_forest, flatten_pipeline, parse_header

BLOB_FILE = "forest.b2f.npz"
OUTLIER_BLOB_FILE = "outlier.b2f"
DRIFT_FILE = "drift_reference.npz"
EXPLAIN_FILE = "explain.b2f"  # TreeSHAP path table (flatten_explainer); optional
BACKGROUND_FILE = "explain_background.npz"  # background rows of interventional explanations (raw columns); optional
MMD_FILE = "mmd_reference.npz"  # reference rows of the MMD drift test (raw columns, and its sigma); optional
TRUST_FILE = "trust_reference.npz"  # labelled reference rows of trust scores (raw columns, labels, fit options); optional
TRUST_TARGET = "default_payment_next_month"  # the label column a trust reference frame carries by default
OUTLIER_PICKLE = os.path.join("artifacts", "outlier.pkl")  # joblib.dump(outlier, ".../outlier.pkl"), 02-register-model.ipynb:264,326-328
SKLEARN_PICKLE = os.path.join("artifacts", "classifier", "model", "model.pkl")  # MLflow layout, 02-register-model.ipynb:317-321


class B200Model:
    def __init__(self, flat: FlatForest, devices=None, drift=None, outlier_blob: bytes | None = None, host_threads: int = 0,
                 explain_blob: bytes | None = None, explain_background: pd.DataFrame | None = None,
                 mmd_reference: pd.DataFrame | None = None, mmd_sigma: float | None = None,
                 trust_reference: pd.DataFrame | None = None, trust_options: dict | None = None):
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
        self.classes = np.asarray(flat.classes)
        self._pool = ThreadPoolExecutor(max_workers=2, thread_name_prefix="b200-drift") if drift is not None else None
        self.outlier_blob = outlier_blob
        if outlier_blob is not None:
            (self.group if self.group is not None else self.engine).attach_outlier_forest(outlier_blob)
        # the explainer (TreeSHAP path table) lives on the first GPU only: explain() runs there
        self.explain_blob = explain_blob
        if explain_blob is not None:
            self.engine.attach_explainer(explain_blob)
        # encoder threads of each GPU's request pipeline (csrc/scorer.h); 0: the library's default for the GPU
        self.host_threads = int(host_threads or os.environ.get("B200_HOST_THREADS", 0))
        # one scoring replica per GPU: the only code that scores on that GPU's handle (predict, the server's round-robin
        # batcher, explain); the forest is replicated, rows are independent
        engines = self.group.engines if self.group is not None else [self.engine]
        self.replicas = [_Replica(self.encoder, e, outlier_blob is not None, self.numeric_features, self.host_threads) for e in engines]
        self.background_rows = 0
        self.background = None  # the attached background frame (raw columns)
        self.dependence_grids = None  # field -> default partial-dependence grid of the background (attach_background)
        if explain_background is not None:
            self.attach_background(explain_background)
        self.mmd_reference_rows = 0
        self.mmd_sigma = None  # the attached MMD reference's kernel width
        if mmd_reference is not None:
            self.attach_mmd_reference(mmd_reference, sigma=mmd_sigma)
        self.trust_reference_rows = None  # rows kept per class of the attached trust reference
        self._trust_positions = None  # attached reference row -> its position in the fitted frame
        if trust_reference is not None:
            self.attach_trust_reference(trust_reference, **(trust_options or {}))

    # ------------------------------------------------------------------ construction
    @classmethod
    def from_pipeline(cls, pipeline, reference_frame: pd.DataFrame | None = None, outlier=None, explain: bool = False,
                      background: pd.DataFrame | None = None, **kw) -> "B200Model":
        """Fitted sklearn Pipeline (the reference's model.pkl) -> model on the GPU.

        ``outlier``: the reference's fitted outlier detector (an alibi-detect ``IForest`` or a bare sklearn
        ``IsolationForest`` plus ``outlier_threshold=``), flattened into a second forest over the same rows.
        ``explain``: also build the TreeSHAP path table, so that ``explain()`` works.  ``background``: a frame of raw rows
        (e.g. the training table) to attach for ``explain_interventional()``; it needs ``explain``.  ``mmd_reference=frame``
        (and ``mmd_sigma=``): the reference table of ``mmd_drift()``.  ``trust_reference=frame`` (and ``trust_options=``, the
        keywords of ``attach_trust_reference``): the labelled reference of ``trust_score()``."""
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
        if self._pool is not None:
            self._pool.shutdown(wait=True)
        if self.drift is not None:
            self.drift.close()
        if self.group is not None:
            self.group.close()
        else:
            self.engine.close()

    # ------------------------------------------------------------------ scoring
    @property
    def last_timing(self) -> dict | None:
        """Seconds spent in the stages of the last job on the first GPU's request pipeline: columns / first chunk / chunks."""
        return self.replicas[0].last_timing

    def _staged(self, df: pd.DataFrame, full: bool = False):
        """The general path, copied out of the first GPU's pinned staging -> (proba1, label, is_outlier or None).  On several
        GPUs it is one group call (``b2f_predict_multi``) that slices the rows over every GPU, so it holds every replica's lock,
        taken in index order: a batcher worker holds one lock and ``explain`` the first, so neither can deadlock against it."""
        with contextlib.ExitStack() as held:
            for r in self.replicas if self.group is not None else self.replicas[:1]:
                held.enter_context(r.lock)
            return tuple(None if a is None else np.array(a) for a in self.replicas[0]._staged(df, full, self.group))

    def predict_proba1(self, df: pd.DataFrame) -> np.ndarray:
        """``classifier.predict_proba(df[all_features])[:, 1]`` (02-register-model.ipynb:335-337)."""
        if self.group is None:
            return self.replicas[0].score(df, want_outliers=False)[0]
        return self._staged(df)[0]

    def predict_label(self, df: pd.DataFrame) -> np.ndarray:
        """``pipeline.predict(df)`` (hard labels, 01-train-model.ipynb:290)."""
        return self.classes[self._staged(df)[1]]

    def predict(self, model_input) -> dict:
        """Mirror of ``CustomModel.predict(context, model_input)`` (02-register-model.ipynb:330-353)."""
        df = self._frame(model_input)
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

    def _frame(self, model_input) -> pd.DataFrame:
        """A request as a frame (never mutated here); KeyError when it has no columns, as the reference raises from
        ``df[self.all_features]`` on an empty request (-> HTTP 500)."""
        df = model_input if isinstance(model_input, pd.DataFrame) else pd.DataFrame(model_input)
        if len(df.columns) == 0:
            raise KeyError(f"None of {self.all_features} are in the [columns]")
        return df

    def _predictions(self, df: pd.DataFrame):
        """-> (predictions list, outlier-flag list): what ``predict`` returns for these rows, without the drift scores."""
        n, full = len(df), self.outlier_blob is not None
        if self.group is not None:
            proba, _, flags = self._staged(df, full)
            return proba.tolist(), flags.tolist() if full else [0] * n
        # one GPU: each chunk's Python floats are built as it lands, while later chunks are still being encoded / copied /
        # scored (float objects recycled: _pylists.py)
        chunks = self.replicas[0]._chunks(df, full)
        next(chunks)
        # the job is in flight: what does not depend on its results -- the empty lists, the all-zero outlier list of a
        # classifier-only model -- is made while the first chunk is on its way
        preds = ListBuilder(n)
        flags = ListBuilder(n) if full else None
        zeros = None if full else [0] * n
        for lo, proba, outlier in chunks:
            preds.fill(lo, proba)
            if full:
                flags.fill(lo, outlier)
        return preds.items, flags.items if full else zeros

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
        It holds ``replicas[0].lock`` across both calls, so it may run beside ``predict`` and the HTTP batcher's workers."""
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
        rows = self.encoder.encode_frame(frame)
        with self.replicas[0].lock:
            nbytes = self.engine.attach_background(rows)
        self.background_rows = len(frame)
        self.background = frame
        self.dependence_grids = self._default_grids(frame, dependence.DEFAULT_RESOLUTION, dependence.DEFAULT_PERCENTILES)
        return nbytes

    def _default_grids(self, frame: pd.DataFrame, grid_resolution: int, percentiles) -> dict:
        """field -> its default grid over ``frame`` (``dependence.grid_from_column``); a field without a grid (no present
        value, coinciding percentiles) is left out."""
        grids = {}
        for name in self.all_features:
            try:
                grids[name] = dependence.grid_from_column(frame[name], name in self.categorical_features, grid_resolution, percentiles)
            except ValueError:
                pass
        return grids

    def partial_dependence(self, model_input, features, *, kind: str = "average", grid_resolution: int = 100, percentiles=(0.05, 0.95),
                           custom_values: dict | None = None, grid_frame: pd.DataFrame | None = None) -> dict:
        """One-way partial dependence and ICE curves of request fields, as scikit-learn's
        ``partial_dependence(pipeline, model_input, features, kind=..., method="brute", categorical_features=...)`` returns
        them, one feature at a time.

        -> ``{"feature_names": features, "output": "probability", "grid_values": [grid per feature], "average": [float64
        (G_f,)], "individual": [float64 (n, G_f)]}``: ``individual[f][i, g]`` is P(class 1) for row i with field f set to
        ``grid_values[f][g]`` (its own value ignored), bit for bit the tile kernel's score of that row; ``average`` (kind
        "average" or "both") is its mean over rows, ``individual`` is there for "individual" and "both".  Duplicate names are
        probed independently.  Grids: ``custom_values[f]`` when given (None / NaN = missing, imputed as in requests; an unknown
        category behaves as any unknown category), else the default rule of ``dependence.grid_from_column`` over the column of
        ``grid_frame``, or of ``model_input`` without one; missing values never enter a default grid.  At most 256 points per
        feature and 23 features per call.  Every model has it, with or without an explainer.  Rows with NaN numerics are
        accepted (the classifier alone is scored).  It runs on the first GPU's handle only, like ``explain``."""
        df = self._frame(model_input)
        features = dependence.check_request(features, self.all_features, kind)
        grid_of = self._grid_rule(custom_values, grid_resolution, percentiles, dependence.MAX_POINTS)
        source = df if grid_frame is None else grid_frame
        grids, words, probes, off = [], [], [], 0
        for name in features:
            grid = grid_of(name, source)
            grids.append(grid)
            words.append(dependence.encode_grid(self.encoder, name, grid))
            probes.append((dependence.word_of(self.encoder, name), off, len(grid)))
            off += len(grid)
        rows = self.encoder.encode_frame(df)
        with self.replicas[0].lock:
            out = self.engine.partial_dependence_rows(rows, probes, np.concatenate(words))
        res = {"feature_names": features, "output": "probability", "grid_values": grids}
        res.update(dependence.split_output(out, [len(g) for g in grids], kind))
        return res

    def pair_grids(self, model_input, pairs, *, grid_resolution: int = 100, percentiles=(0.05, 0.95), custom_values: dict | None = None,
                   grid_frame: pd.DataFrame | None = None) -> list:
        """The two grids of each pair ``pair_dependence`` probes: ``custom_values[f]`` when given, else the default rule of
        ``dependence.grid_from_column`` over ``grid_frame``'s column, or ``model_input``'s.  ValueError for an unknown field,
        a pair of one field, or an axis outside 1..256 points."""
        pairs = interaction.check_pairs(pairs, self.all_features)
        grid_of = self._grid_rule(custom_values, grid_resolution, percentiles, interaction.MAX_AXIS_POINTS)
        source = model_input if grid_frame is None else grid_frame
        source = source if isinstance(source, pd.DataFrame) else pd.DataFrame(source)
        cache, out = {}, []
        for pair in pairs:
            for name in pair:
                if name not in cache:
                    cache[name] = grid_of(name, source)
            out.append([cache[pair[0]], cache[pair[1]]])
        return out

    def _grid_rule(self, custom_values: dict | None, grid_resolution: int, percentiles, max_points: int):
        """-> grid_of(name, source): the grid of a probed field, ``custom_values[name]`` when given, else the default rule of
        ``dependence.grid_from_column`` over ``source[name]``.  ValueError for custom values of an unknown field (here) or a
        grid outside 1..max_points points (from grid_of)."""
        custom_values = dict(custom_values or {})
        unknown = [f for f in custom_values if f not in self.all_features]
        if unknown:
            raise ValueError(f"custom_values for unknown feature(s) {unknown}")

        def grid_of(name: str, source) -> list:
            if name in custom_values:
                grid = list(custom_values[name])
            else:
                grid = dependence.grid_from_column(source[name], name in self.categorical_features, grid_resolution, percentiles).tolist()
            if not 1 <= len(grid) <= max_points:
                raise ValueError(f"feature {name!r}: {len(grid)} grid points, expected 1..{max_points}")
            return grid

        return grid_of

    def pair_dependence(self, model_input, pairs, *, kind: str = "average", grid_resolution: int = 100, percentiles=(0.05, 0.95),
                        custom_values: dict | None = None, grid_frame: pd.DataFrame | None = None) -> dict:
        """Two-way partial dependence of pairs of request fields: per pair ``(a, b)``, what scikit-learn's
        ``partial_dependence(pipeline, model_input, [a, b], kind=..., method="brute", categorical_features=...)`` returns.

        -> ``{"feature_names": pairs, "output": "probability", "grid_values": [[grid a, grid b] per pair], "average": [float64
        (G_a, G_b)], "individual": [float64 (n, G_a, G_b)]}``: ``individual[p][i, u, v]`` is P(class 1) for row i with field
        a set to ``grid_values[p][0][u]`` and b to ``grid_values[p][1][v]``, bit for bit the tile kernel's score of that
        row; ``average`` (kind "average" or "both") is its mean over the rows, taken on the device in a fixed order (never
        copying the curves), ``individual`` is there for "individual" and "both".  Grids follow ``pair_grids``: at most 256
        points per axis.  ``pairs``: one pair or a list of them.  Every model has it; rows with NaN numerics are accepted
        (the classifier alone is scored).  It runs on the first GPU's handle only, under ``replicas[0].lock``."""
        df = self._frame(model_input)
        if kind not in dependence.KINDS:
            raise ValueError(f"kind={kind!r}: expected one of {dependence.KINDS}")
        pairs = interaction.check_pairs(pairs, self.all_features)
        grids = self.pair_grids(df, pairs, grid_resolution=grid_resolution, percentiles=percentiles, custom_values=custom_values,
                                grid_frame=grid_frame)
        if len(df) == 0:
            raise ValueError("pair dependence needs at least one row")
        probes, points, off = [], [], 0
        for (a, b), (ga, gb) in zip(pairs, grids):
            pts = interaction.cartesian(dependence.encode_grid(self.encoder, a, ga), dependence.encode_grid(self.encoder, b, gb))
            probes.append((dependence.word_of(self.encoder, a), dependence.word_of(self.encoder, b), off, len(pts)))
            points.append(pts)
            off += len(pts)
        rows = self.encoder.encode_frame(df)
        res = {"feature_names": pairs, "output": "probability", "grid_values": grids}
        shapes = [(len(ga), len(gb)) for ga, gb in grids]
        with self.replicas[0].lock:
            if kind in ("average", "both"):
                means = self.engine.pair_dependence_rows(rows, probes, np.concatenate(points), mean=True)
                res["average"] = [means[p[2]:p[2] + p[3]].reshape(s) for p, s in zip(probes, shapes)]
            if kind in ("individual", "both"):  # one call per pair: a call's curves hold at most 65 536 points per row
                res["individual"] = [self.engine.pair_dependence_rows(rows, [(p[0], p[1], 0, p[3])], pts).reshape((len(df),) + s)
                                     for p, pts, s in zip(probes, points, shapes)]
        return res

    def interaction_strength(self, model_input, features=None, *, sample: int = interaction.DEFAULT_SAMPLE, random_state: int = 0) -> dict:
        """Which pairs of request fields interact, across the applicants: Friedman's H-statistic H^2 of every pair of
        ``features`` (default: every field, in field order) over a sample S of the rows (every row when there are at most
        ``sample``, else ``RandomState(random_state).choice(n, sample, replace=False)``); the formula is in
        ``interaction.py``, with f = P(class 1) as ``partial_dependence`` scores it.

        -> ``{"pairs": [(a, b)] in itertools.combinations order, "h_squared", "numerator", "denominator": float64 (pairs,),
        "matrix": float64 (F, F) symmetric with a NaN diagonal, "feature_names", "rows": |S|}``; H^2 is NaN where the
        denominator is 0, and unstable where F_jk is nearly flat (hence the numerator and denominator).  One device call
        scores the distinct (x_j, x_k) of S per pair and the distinct x_j per field, each as a mean over S; centring and
        sums are float64 numpy in a fixed order.  ValueError for an unknown or repeated field, fewer than two fields, a
        sample outside 2..10 000, a bad seed or fewer than two rows.  It runs on the first GPU's handle only, under
        ``replicas[0].lock``."""
        df = self._frame(model_input)
        features = interaction.check_features(features, self.all_features)
        sample, random_state = interaction.check_sample(sample, random_state)
        S = interaction.sample_rows(len(df), sample, random_state)
        rows = self.encoder.encode_frame(df.iloc[S].reset_index(drop=True))
        n_cat, n_num = len(self.categorical_features), len(self.numeric_features)
        words = interaction.impute(rows, n_cat, n_num, parse_header(self.flat.blob)["impute"])
        fields = [dependence.word_of(self.encoder, f) for f in features]
        probes, points, maps = interaction.strength_plan(words, fields, [f in self.categorical_features for f in features])
        with self.replicas[0].lock:
            means = self.engine.pair_dependence_rows(rows, probes, points, mean=True)
        res = interaction.strength_result(means, maps, features)
        res["rows"] = len(S)
        return res

    def accumulated_local_effects(self, model_input, features=None, *, bins: int = ale.DEFAULT_BINS, min_bin_points: int = ale.DEFAULT_MIN_BIN_POINTS,
                                  custom_edges: dict | None = None, grid_frame: pd.DataFrame | None = None) -> dict:
        """How P(class 1) moves with each numeric request field where the applicants actually are: accumulated local
        effects (Apley & Zhu), which score each row only at the two edges of the bin its own value lies in, so correlated
        fields are never pushed to combinations no applicant has (partial dependence's weakness).  The formulas and the
        default edge rule are in ``ale.py``; f = P(class 1) as ``partial_dependence`` scores it, each substituted row bit
        for bit the tile kernel's score.

        ``features``: numeric fields (default: every numeric field, in field order).  Edges: ``custom_edges[f]`` (2..257
        finite numbers, strictly increasing as float32; rows outside [z_0, z_K] go to the end bins), else the edge rule over
        the present values of ``grid_frame[f]``, or of ``model_input[f]`` without one.  A row whose field is missing takes
        no part in that field.  -> ``{"feature_names", "output": "probability", "feature_values": [edges (K + 1)],
        "ale_values": [(K + 1)], "bin_effects": [d_k (K)], "bin_rows": [n_k (K)], "ale0": [float], "constant_value": mean
        P(class 1) over the rows, "rows"}``; a field with one distinct value has one edge and ``ale_values == [0.0]``.
        ValueError for an unknown, categorical or repeated field, bins outside 1..256, min_bin_points < 1, bad custom edges,
        zero rows, or a field with no present value to build edges from.  Every model has it.  It runs on the first GPU's
        handle only, under ``replicas[0].lock``."""
        df = self._frame(model_input)
        features = ale.check_features(features, self.numeric_features, self.categorical_features)
        bins, min_bin_points = ale.check_params(bins, min_bin_points)
        custom_edges = dict(custom_edges or {})
        extra = [f for f in custom_edges if f not in features]
        if extra:
            raise ValueError(f"custom_edges for feature(s) {extra} that are not probed")
        if len(df) == 0:
            raise ValueError("accumulated local effects need at least one row")
        source = df if grid_frame is None else grid_frame
        edges = []
        for f in features:
            if f in custom_edges:
                edges.append(ale.check_custom_edges(f, custom_edges[f]))
            else:
                try:
                    edges.append(ale.default_edges(ale.present_float32(self.encoder, f, source[f]), bins, min_bin_points))
                except ValueError as e:
                    raise ValueError(f"feature {f!r}: {e}") from None
        probes, flat_edges, which = ale.probe_plan([dependence.word_of(self.encoder, f) for f in features], edges)
        rows = self.encoder.encode_frame(df)
        with self.replicas[0].lock:
            if probes:
                sums, counts = self.engine.ale_rows(rows, probes, flat_edges)
            else:
                sums, counts = np.zeros(0), np.zeros(0, np.int64)
            proba, _ = self.engine.predict_rows(rows, np.float64)
        res = ale.result(features, edges, sums, counts, probes, which)
        res["constant_value"] = float(np.mean(proba))
        res["rows"] = len(df)
        return res

    def counterfactuals(self, model_input, features=None, *, cutoff: float = 0.5) -> dict:
        """What would change the decision: per applicant and request field, the nearest value of that field alone at which
        the decision ``P(class 1) > cutoff`` differs from the applicant's own.

        -> ``{"feature_names", "output": "probability", "cutoff", "predictions": float64 (n,), "decisions": bool (n,),
        "counterfactuals": [one dict per field, in order]}``.  A numeric field's dict holds float64 (n,) arrays ``value`` (the
        value as scored: a missing value is the training median), ``lower`` / ``upper`` (the largest float32 below / smallest
        above ``value`` whose decision differs; NaN when no value on that side does) and ``lower_prediction`` /
        ``upper_prediction`` (P(class 1) there, bit for bit the tile kernel's score of the row with the field set to that
        value).  These are exact float32 boundaries: sent back as request values they reproduce the flip, and the float32
        one step toward ``value`` keeps the decision.  A categorical field has no order: its dict holds ``value`` (the
        category, None when missing or unknown) and ``flips``, per row the list of ``(category, P(class 1))`` of the
        vocabulary categories, in code order, whose decision differs.  At cutoff 0.5 the decision is the model's label except
        where P(class 1) rounds to exactly 0.5.  ``features=None`` probes every field; unknown or repeated names raise
        ValueError, as does a cutoff outside [0, 1].  Every model has it, with or without an explainer; rows with NaN
        numerics are accepted.  It runs on the first GPU's handle only, like ``partial_dependence``."""
        df = self._frame(model_input)
        features = list(self.all_features) if features is None else ([features] if isinstance(features, str) else list(features))
        if not features:
            raise ValueError("at least one feature is needed")
        unknown = [f for f in features if f not in self.all_features]
        if unknown:
            raise ValueError(f"unknown feature(s) {unknown}; expected names from {list(self.all_features)}")
        if len(set(features)) != len(features):
            raise ValueError(f"repeated feature(s) {sorted({f for f in features if features.count(f) > 1})}")
        if isinstance(cutoff, bool) or not isinstance(cutoff, (int, float, np.integer, np.floating)) or not 0.0 <= float(cutoff) <= 1.0:
            raise ValueError(f"cutoff={cutoff!r}: expected a number in [0, 1]")
        cutoff = float(cutoff)
        rows = self.encoder.encode_frame(df)
        n = rows.shape[0]
        cats = [f for f in features if f in self.categorical_features]
        nums = [f for f in features if f not in self.categorical_features]
        proba, rec = None, None
        if nums:
            with self.replicas[0].lock:
                proba, rec = self.engine.counterfactual_rows(rows, [dependence.word_of(self.encoder, f) for f in nums], cutoff)
        # categoricals: K6 ICE points over the whole vocabulary, at most 256 points per probe; without a numeric field the
        # predictions are the ICE point at each row's own code (-1 added to the first field's grid for unknown categories)
        probes, words, spans = [], [], {}
        for f in cats:
            word, vocab = dependence.word_of(self.encoder, f), len(self.flat.categories[self.categorical_features.index(f)])
            codes = list(range(-1 if (proba is None and not probes) else 0, vocab))
            spans[f] = (len(words), codes)
            for lo in range(0, len(codes), dependence.MAX_POINTS):
                probes.append((word, len(words) + lo, min(dependence.MAX_POINTS, len(codes) - lo)))
            words.extend(codes)
        ice = None
        if probes:
            with self.replicas[0].lock:
                ice = self.engine.partial_dependence_rows(rows, probes, np.asarray(words, dtype=np.int32).view(np.uint32))
        if proba is None:
            f0 = cats[0]
            own = rows[:, dependence.word_of(self.encoder, f0)].view(np.int32).astype(np.int64)
            proba = ice[np.arange(n), spans[f0][0] + own + 1] if n else np.empty(0, dtype=np.float64)
        decisions = proba > cutoff
        out, k = [], 0
        for f in features:
            if f in spans:
                start, codes = spans[f]
                vocab = self.flat.categories[self.categorical_features.index(f)]
                own = rows[:, dependence.word_of(self.encoder, f)].view(np.int32)
                first = start + (1 if codes[0] == -1 else 0)
                curve = ice[:, first:start + len(codes)]
                flips = [[(vocab[c], float(curve[i, c])) for c in np.flatnonzero((curve[i] > cutoff) != decisions[i])] for i in range(n)]
                out.append({"value": [vocab[c] if c >= 0 else None for c in own.tolist()], "flips": flips})
            else:
                r = rec[:, k]
                k += 1
                out.append({"value": r["value"].astype(np.float64), "lower": r["lower"].astype(np.float64), "lower_prediction": r["lower_p1"].copy(),
                            "upper": r["upper"].astype(np.float64), "upper_prediction": r["upper_p1"].copy()})
        return {"feature_names": features, "output": "probability", "cutoff": cutoff, "predictions": proba, "decisions": decisions,
                "counterfactuals": out}

    def permutation_importance(self, df, y, *, scoring=None, n_repeats: int = 5, random_state=None) -> dict:
        """How much the model relies on each request field: scikit-learn's ``permutation_importance(pipeline, df, y,
        scoring=scoring, n_repeats=n_repeats, random_state=random_state)`` of the fitted pipeline, computed on the GPU.

        Every request field is probed, in the model's field order (the frame's column order does not matter: sklearn uses
        one permutation for every column).  ``scoring``: None (accuracy, as ``estimator.score``), one name of
        ``importance.SCORERS`` or a list of them; with a list the answer is a dict keyed by scorer, as sklearn's.  Each
        answer holds ``importances`` float64 (n_fields, n_repeats) (baseline minus permuted score), ``importances_mean``,
        ``importances_std`` (ddof 0), ``baseline_score``, ``feature_names``, ``n_repeats`` and ``rows``.  ``y``: one 0/1
        label per row.  Rows are scored by the classifier alone, as ``explain`` scores them, so NaN numerics are accepted
        even with an outlier forest attached.  ``roc_auc`` is NaN with one class in ``y``; ``neg_log_loss`` raises
        ValueError there, as sklearn does.  It runs on the first GPU's handle only, under ``replicas[0].lock``."""
        names, multi = importance.check_scoring(scoring)
        n_repeats = importance.check_n_repeats(n_repeats)
        df = self._frame(df)
        labels = importance.check_labels(y, len(df))
        if len(df) == 0:
            raise ValueError("permutation importance needs at least one row")
        importance.check_single_class(names, labels)
        perm = importance.permutations(len(df), n_repeats, random_state)
        rows = self.encoder.encode_frame(df)
        words = [dependence.word_of(self.encoder, f) for f in self.all_features]
        with self.replicas[0].lock:
            rec, base = self.engine.permutation_scores(rows, labels, perm, words)
        out = {s: importance.result(s, rec, base, self.all_features, n_repeats, len(df)) for s in names}
        return out if multi else out[names[0]]

    def _embedding_constants(self, rows: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
        """Encoded reference rows -> the z-score (mean, scale) of the embedding MMD drift and trust scores share (``mmd.py``)."""
        n_cat, n_num = len(self.categorical_features), len(self.numeric_features)
        impute = parse_header(self.flat.blob)["impute"][n_cat:n_cat + n_num]
        return mmd.standardization(mmd.numerics(rows, n_cat, n_num, impute))

    @property
    def mmd_reference_attached(self) -> bool:
        return self.mmd_reference_rows > 0

    def attach_mmd_reference(self, frame: pd.DataFrame, *, sigma: float | None = None) -> float:
        """Attach the reference table of ``mmd_drift``: 2..131 072 raw rows, encoded as requests are, embedded once on the
        first GPU with the z-score constants of their numerics; replaces an earlier reference.  ``sigma``: the Gaussian
        kernel's width; None: alibi-detect's median heuristic on the reference (ValueError when the median pair distance is 0).
        -> sigma."""
        sigma = mmd.check_sigma(sigma)
        frame = frame if isinstance(frame, pd.DataFrame) else pd.DataFrame(frame)
        mmd.check_reference(len(frame))
        rows = self.encoder.encode_frame(frame)
        mean, scale = self._embedding_constants(rows)
        self.mmd_reference_rows, self.mmd_sigma = 0, None
        with self.replicas[0].lock:
            try:
                got = self.engine.attach_mmd_reference(rows, mean, scale, sigma)
            except B2FError as e:
                if "median pair distance is 0" in str(e):
                    raise ValueError(f"{e}: attach this reference with an explicit sigma") from e
                raise
        self.mmd_reference_rows, self.mmd_sigma = len(frame), got
        return got

    def mmd_drift(self, model_input, *, n_permutations: int = 100, p_val: float = 0.05, random_state: int = 0) -> dict:
        """Has the joint distribution of the request fields moved?  alibi-detect's ``MMDDrift(x_ref, p_val=p_val,
        n_permutations=n_permutations).predict(x)["data"]`` on the classifier's input vectors (``mmd.py``), with the kernel
        sums on the GPU: the unbiased MMD^2 of the batch against the attached reference and a p-value from permutations of
        the pooled rows.  -> ``{"is_drift": 0/1, "distance": mmd^2, "p_val", "threshold": p_val, "distance_threshold": the
        permuted statistic at the p_val quantile, "sigma", "n_permutations", "reference_rows", "rows"}``.  It runs on the
        first GPU's handle only, under ``replicas[0].lock``.  RuntimeError without a reference; ValueError for fewer than 2
        rows, a bad argument or more kernel pairs than ``mmd.PAIR_BUDGET``."""
        if not self.mmd_reference_attached:
            raise RuntimeError("this model has no MMD reference: attach_mmd_reference(frame), from_pipeline(..., mmd_reference=frame) "
                               f"or a model directory that holds {MMD_FILE} (save_model_dir(..., mmd_reference=frame))")
        df = self._frame(model_input)
        n_ref = self.mmd_reference_rows
        n_permutations, p_val, random_state = mmd.check_request(len(df), n_ref, n_permutations, p_val, random_state)
        rows = self.encoder.encode_frame(df)
        subsets = mmd.draw_subsets(n_ref, len(df), n_permutations, random_state)
        with self.replicas[0].lock:
            obs, perm = self.engine.mmd_statistics(rows, subsets)
        return mmd.result(obs, perm, p_val, self.mmd_sigma, n_ref, len(df))

    @property
    def trust_reference_attached(self) -> bool:
        return self.trust_reference_rows is not None

    def attach_trust_reference(self, frame: pd.DataFrame, labels=None, *, k_filter: int = 10, alpha: float = 0.0, filter_type=None,
                               dist_filter_type: str = "point") -> list:
        """Fit alibi's ``TrustScore(k_filter, alpha, filter_type, dist_filter_type).fit(X, Y)`` on a labelled reference
        (``trust.py``): 2..131 072 raw rows, encoded as requests are and embedded on the first GPU with the z-score constants of
        their numerics, taken over the whole frame.  ``labels``: the model's classes per row (default: the frame's
        ``default_payment_next_month`` column).  ``filter_type="distance_knn"`` drops, per class, the rows whose distance to
        their ``k_filter``-th nearest same-class row ("point") or mean distance to the ``k_filter`` nearest ("mean") lies above
        the ``(1 - alpha)`` percentile; its neighbours come from the same GPU search as the scores.  Replaces an earlier
        reference.  -> the rows kept per class.  ValueError for a bad argument, a label outside the model's classes, or a class
        with too few rows."""
        frame = frame if isinstance(frame, pd.DataFrame) else pd.DataFrame(frame)
        k_filter, alpha, filter_type, dist_filter_type = trust.check_fit(len(frame), k_filter, alpha, filter_type, dist_filter_type)
        if labels is None:
            if TRUST_TARGET not in frame.columns:
                raise ValueError(f"pass labels, or a frame with a {TRUST_TARGET!r} column")
            labels = frame[TRUST_TARGET].to_numpy()
        if len(labels) != len(frame):
            raise ValueError(f"{len(labels)} labels for {len(frame)} reference rows")
        cls = trust.class_indices(labels, self.classes)
        trust.check_class_rows(cls, filter_type, k_filter)
        rows = self.encoder.encode_frame(frame)
        mean, scale = self._embedding_constants(rows)
        positions = np.arange(len(frame))
        self.trust_reference_rows, self._trust_positions = None, None
        with self.replicas[0].lock:
            self.engine.attach_knn_reference(rows, cls, mean, scale)
            if filter_type == "distance_knn":
                dist, _ = self.engine.knn(rows, k_filter + 1)
                keep = np.zeros(len(frame), dtype=bool)
                for c in (0, 1):
                    own = cls == c
                    keep[own] = trust.filter_keep(trust.filter_radius(dist[own, c, :], dist_filter_type), alpha)
                positions = np.nonzero(keep)[0]
                self.engine.attach_knn_reference(rows[positions], cls[positions], mean, scale)
        kept = [int((cls[positions] == c).sum()) for c in (0, 1)]
        self.trust_reference_rows, self._trust_positions = kept, positions
        return kept

    def trust_score(self, model_input, *, k: int = 2, dist_type: str = "point") -> dict:
        """Can this decision be trusted?  alibi's ``TrustScore.score(X, Y, k, dist_type)`` with Y the classifier's own
        predictions: per row, D_c is the k-th nearest distance ("point") or the mean of the k nearest distances ("mean") to
        the attached reference rows of class c, and ``trust_score = D_other / (D_pred + 1e-12)``: below 1 the other class's
        reference rows are nearer than the predicted class's.  -> ``{"trust_score", "closest_not_pred", "predictions": P(class
        1), "labels": the predicted class, "distance_to_pred", "distance_to_other", "k", "dist_type", "reference_rows": rows
        kept per class, "neighbours": per class {"class", "index": (n, k) positions in the fitted frame, "distance": (n, k)}}``,
        neighbours ordered by (distance, position).  The classifier alone is scored, so NaN numerics are accepted.  It runs on
        the first GPU's handle only, under ``replicas[0].lock``.  RuntimeError without a reference; ValueError for a bad k or
        dist_type or no rows."""
        if not self.trust_reference_attached:
            raise RuntimeError("this model has no trust reference: attach_trust_reference(frame), from_pipeline(..., trust_reference=frame) "
                               f"or a model directory that holds {TRUST_FILE} (save_model_dir(..., trust_reference=frame))")
        df = self._frame(model_input)
        k, dist_type = trust.check_score(k, dist_type, self.trust_reference_rows)
        if len(df) == 0:
            raise ValueError("trust scores need at least one row")
        rows = self.encoder.encode_frame(df)
        with self.replicas[0].lock:
            dist, index = self.engine.knn(rows, k)
            proba, _ = self.replicas[0].score(df, want_outliers=False)
            _, label = self.engine.predict_rows(rows)
        return trust.result(dist, index, proba, label.astype(np.int64), self.classes, self._trust_positions, k, dist_type,
                            self.trust_reference_rows)

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
        df = self._frame(model_input)
        rows = self.encoder.encode_frame(df)
        with self.replicas[0].lock:
            values, base = getattr(self.engine, method)(rows)
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
    """One GPU's scoring path, and the only code that scores on its engine's handle: the columnar request pipeline
    (``csrc/scorer.h``, created on first use), else the general path through that engine's pinned staging.

    ``lock`` is held around every call on the handle, whoever makes it (calls on one handle must not overlap:
    ``include/b2f.h``).  It is reentrant because ``B200Model.explain`` holds it across the engine call and ``score``."""

    def __init__(self, encoder: RowEncoder, engine: ForestEngine, has_outlier: bool = False, numeric_features=(), host_threads: int = 0):
        self.encoder, self.engine, self.has_outlier, self.numeric_features = encoder, engine, has_outlier, list(numeric_features)
        self.host_threads = host_threads
        self.lock = threading.RLock()
        self._scorer, self._scorer_failed = None, os.environ.get("B200_SCORER", "1") == "0"
        self.last_timing = None  # seconds spent in the stages of the last request-pipeline job: columns / first chunk / chunks

    def score(self, df: pd.DataFrame, want_outliers: bool = True):
        """-> (proba1 float64 (n,), is_outlier int32 (n,) or None).  ``want_outliers=False``: the classifier alone (no
        outlier forest, so NaN numerics are accepted), on the same row format and kernels as the full pass."""
        n = len(df)
        full = self.has_outlier and want_outliers
        chunks = self._chunks(df, full)
        next(chunks)
        proba, flags = np.empty(n, dtype=np.float64), (np.empty(n, dtype=np.int32) if full else None)
        for lo, p, f in chunks:
            proba[lo:lo + len(p)] = p
            if full:
                flags[lo:lo + len(f)] = f
        return proba, flags

    def _chunks(self, df: pd.DataFrame, full: bool):
        """Score ``df`` on this GPU, holding ``lock`` until the generator is exhausted or closed.  Yields None once the job is
        in flight (what the caller makes meanwhile overlaps the first chunk), then ``(lo, proba1, is_outlier or None)`` for
        rows [lo, lo + len(proba1)) as they land; ``full``: the outlier forest too.  The parts are views over pinned buffers
        that the next job reuses."""
        t0 = time.perf_counter()
        with self.lock:
            n = len(df)
            if self._scorer is None and not self._scorer_failed and n:
                try:
                    self._scorer = self.engine.scorer(self.encoder, self.host_threads)
                except Exception:
                    self._scorer_failed = True
            cols = self.encoder.frame_columns(df) if self._scorer is not None and n else None
            if cols is None:
                yield None
                proba, _, flags = self._staged(df, full)
                yield 0, proba, flags
                return
            # the columnar request pipeline: column buffers -> encode threads -> H2D -> kernel(s) -> D2H, chunk by chunk
            if full:
                _reject_nan(df, self.numeric_features)
            t1 = time.perf_counter()
            sc = self._scorer
            # classifier only: the scorer's own choice of rows (64-byte float32 rows: cheapest to encode; ranked rows with
            # B200_SCORER_ROWS=ranked); with an outlier forest attached float32 rows, even for the classifier alone (ranks are
            # relative to ONE forest's split values)
            fmt = (ROWS_PACKED64 if self.encoder.packed_ok else ROWS_WORDS24) if self.has_outlier else None
            n_chunks = sc.start(n, cols, out_mode=OUT_FULL if full else OUT_F64, fmt=fmt)
            out, bounds, t_first = sc.results(), sc.bounds, None
            yield None
            for c in range(n_chunks):  # chunks ride different streams: each has its own completion event
                sc.wait(c)
                t_first = t_first or time.perf_counter()
                part = out[bounds[c]:bounds[c + 1]]
                yield (bounds[c], part["proba1"], part["is_outlier"]) if full else (bounds[c], part, None)
            t2 = time.perf_counter()
            self.last_timing = {"columns_s": t1 - t0, "first_chunk_s": (t_first or t2) - t1, "chunks_and_lists_s": t2 - t1,
                                "chunks": n_chunks, "threads": sc.threads, "row_format": sc.last_fmt}

    def _staged(self, df: pd.DataFrame, full: bool, target=None):
        """The general path: encode into this engine's pinned staging and score with ONE call of ``target`` (this engine, or the
        group that slices the rows over every GPU) -> views (proba1, label, is_outlier or None) over that staging.  The caller
        holds the lock of every handle ``target`` drives."""
        n = len(df)
        # large requests travel as 64-byte packed rows (one third fewer PCIe bytes), encoded natively in one pass
        packed = self.encoder.packed_ok and n > self.encoder.SMALL_BATCH
        rows, proba, label = self.engine.staging(n, packed=packed)
        if packed:
            self.encoder.encode_frame_packed(df, out=rows)
        else:
            self.encoder.encode_frame(df, out=rows)
        target = self.engine if target is None else target
        if full:
            _reject_nan(df, self.numeric_features)
            rec = target.predict_full(rows, out=self.engine.staging_full(n))
            return rec["proba1"], rec["label"], rec["is_outlier"]
        target.predict_rows(rows, out_proba=proba, out_label=label)
        return proba, label, None


# ---------------------------------------------------------------------- loading
def save_model_dir(path: str, flat: FlatForest, reference_frame: pd.DataFrame | None = None, outlier_blob: bytes | None = None,
                   explain_blob: bytes | None = None, explain_background: pd.DataFrame | None = None,
                   mmd_reference: pd.DataFrame | None = None, mmd_sigma: float | None = None,
                   trust_reference: pd.DataFrame | None = None, trust_options: dict | None = None) -> None:
    """Write the GPU-side artefact next to (or instead of) the MLflow pickles.  ``explain_blob``: the TreeSHAP path table
    (``flatten_explainer``), written as ``explain.b2f`` so that ``load_model`` attaches it.  ``explain_background``: raw
    rows written as ``explain_background.npz``, attached by ``load_model`` with the explainer.  ``mmd_reference``: raw rows
    written as ``mmd_reference.npz`` with ``mmd_sigma`` (None: the median heuristic at load), attached by ``load_model``.
    ``trust_reference``: raw rows written as ``trust_reference.npz`` with their labels (``trust_options["labels"]``, else the
    frame's ``default_payment_next_month``) and the other ``attach_trust_reference`` options, fitted by ``load_model``."""
    os.makedirs(path, exist_ok=True)
    flat.save(os.path.join(path, BLOB_FILE))
    if explain_blob is not None:
        with open(os.path.join(path, EXPLAIN_FILE), "wb") as f:
            f.write(explain_blob)
    if explain_background is not None:
        _save_background(os.path.join(path, BACKGROUND_FILE), flat, explain_background)
    if mmd_reference is not None:
        sigma = mmd.check_sigma(mmd_sigma)
        _save_background(os.path.join(path, MMD_FILE), flat, mmd_reference, mmd_sigma=np.float64(np.nan if sigma is None else sigma))
    if trust_reference is not None:
        opts = dict(trust_options or {})
        labels = opts.pop("labels", None)
        unknown = set(opts) - {"k_filter", "alpha", "filter_type", "dist_filter_type"}
        if unknown:
            raise ValueError(f"unknown trust option(s) {sorted(unknown)}")
        k_filter, alpha, filter_type, dist_filter_type = trust.check_fit(len(trust_reference), opts.get("k_filter", 10), opts.get("alpha", 0.0),
                                                                         opts.get("filter_type"), opts.get("dist_filter_type", "point"))
        labels = np.asarray(trust_reference[TRUST_TARGET] if labels is None else labels)
        trust.class_indices(labels, flat.classes)
        _save_background(os.path.join(path, TRUST_FILE), flat, trust_reference, trust_labels=labels, trust_k_filter=np.int64(k_filter),
                         trust_alpha=np.float64(alpha), trust_filter_type=np.str_(filter_type or ""),
                         trust_dist_filter_type=np.str_(dist_filter_type))
    if outlier_blob is not None:
        with open(os.path.join(path, OUTLIER_BLOB_FILE), "wb") as f:
            f.write(outlier_blob)
    if reference_frame is not None:
        from .drift import TabularDrift

        TabularDrift(reference_frame[flat.all_features], flat.cat_features, device=None).save(os.path.join(path, DRIFT_FILE))


def _save_background(path: str, flat: FlatForest, frame: pd.DataFrame, **extra) -> None:
    """The raw columns of ``flat.all_features``: numerics as float64, categories as ``U`` strings with ``null__<name>`` telling
    a string (0) from None (1) and NaN (2), which the encoder maps differently; ``extra`` arrays beside them."""
    arrays = dict(extra)
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
    mmd_path = os.path.join(path, MMD_FILE)
    if "mmd_reference" not in kw and os.path.exists(mmd_path) and os.environ.get("B200_MMD", "gpu") != "off":
        kw["mmd_reference"] = _load_background(mmd_path, flat)
        with np.load(mmd_path, allow_pickle=False) as z:
            sigma = float(z["mmd_sigma"])
        kw["mmd_sigma"] = None if math.isnan(sigma) else sigma
    trust_path = os.path.join(path, TRUST_FILE)
    if "trust_reference" not in kw and os.path.exists(trust_path) and os.environ.get("B200_TRUST", "gpu") != "off":
        kw["trust_reference"] = _load_background(trust_path, flat)
        with np.load(trust_path, allow_pickle=False) as z:
            kw["trust_options"] = {"labels": z["trust_labels"], "k_filter": int(z["trust_k_filter"]), "alpha": float(z["trust_alpha"]),
                                   "filter_type": str(z["trust_filter_type"]) or None, "dist_filter_type": str(z["trust_dist_filter_type"])}
    return B200Model(flat, devices=devices, drift=drift, outlier_blob=outlier_blob, **kw)
