"""FastAPI serving layer: the reference's ``app/main.py`` with the new request-batching loop.

Same HTTP surface as the reference (``app/main.py:35-43``): ``POST /predict`` takes a JSON list of
``LoanApplicant`` rows and returns ``ModelOutput``; Swagger UI at ``/``; ``MODEL_DIRECTORY`` and
``SERVICE_NAME`` environment variables; the model is loaded once in ``lifespan`` (``:20-31``) and cleared
at shutdown; both log records (``type: InferenceData`` ``:60-69`` and ``type: ModelOutput`` ``:75-84``) keep
their schema because the reference's KQL dashboards query it.  Error behaviour is the reference's too:
type errors are FastAPI's 422, anything raised while scoring is a 500, an empty list is a 500.

What is new sits between the reference's lines 54 and 72:

* a request body of the regular shape goes from bytes to the 23 columns in one pass of the native parser
  (``ingest.py`` / ``csrc/json_rows.h``: float64 arrays + Arrow string buffers, no per-row Python objects); any other
  body is validated by pydantic-core with the same field rules and 422 behaviour as ``list[LoanApplicant]`` (no
  ``pd.DataFrame(list_of_models)`` either way);
* a micro-batcher collects concurrent requests for up to ``B200_BATCH_WINDOW_US`` microseconds (or
  ``B200_MAX_BATCH`` rows), dictionary-encodes them into one pinned staging slot, and scores the whole
  slot with ONE engine call (H2D + classifier kernel + outlier-forest kernel + D2H); batches are dealt round-robin
  to the GPUs listed in ``B200_DEVICES`` -- the reference instead blocks its event loop per request (``async def``
  calling blocking code, ``app/main.py:43,72``), so requests are strictly serialised there;
* the per-request drift scores (GPU, ``drift.py``) run concurrently with that on their own stream and thread;
* the two JSON log lines are produced on a logging thread, off the request's critical path.
"""

from __future__ import annotations

import asyncio
import json
import logging
import os
import queue
import threading
import time
import uuid
from concurrent.futures import ThreadPoolExecutor
from contextlib import asynccontextmanager
from typing import AsyncGenerator

import numpy as np
import pandas as pd
from fastapi import FastAPI, Request, Response

from fastapi.exceptions import RequestValidationError
from pydantic import ValidationError

from . import ale, dependence, importance, interaction, mmd, trust
from .ingest import NativeRequestParser, parse_rows, rows_to_frame  # noqa: F401  (rows_to_frame re-exported)
from .schema import ALL_FEATURES, CATEGORICAL_FEATURES, LABELLED_ROWS, NUMERIC_FEATURES, TARGET, LabelledApplicant, LoanApplicant, ModelOutput

ml_models: dict = {}


def _service_name() -> str:
    return os.environ.get("SERVICE_NAME", "credit-default-api")


parse_request = parse_rows  # the general validator (pydantic-core over the raw bytes); see ingest.py


_REQUEST_SCHEMA = {"required": True, "content": {"application/json": {"schema": {
    "title": "Data", "type": "array", "items": LoanApplicant.model_json_schema()}}}}


class _Pending:
    __slots__ = ("frame", "future", "loop", "n")

    def __init__(self, frame, future, loop):
        self.frame, self.future, self.loop, self.n = frame, future, loop, len(frame)


class MicroBatcher:
    """Cross-request batching in front of a replica's ``score`` (one worker thread per model; ``score`` takes the replica's
    lock, so other callers of the same GPU's handle take turns with the worker).

    ``models`` is a list (one per GPU); consecutive batches go round-robin over it."""

    def __init__(self, models, max_rows: int = 65536, window_us: int = 200):
        self.models = list(models)
        self.max_rows = int(max_rows)
        self.window_s = window_us * 1e-6
        self.q: queue.Queue = queue.Queue()
        self.batches = 0
        self.rows = 0
        self._stop = False
        self._threads = [threading.Thread(target=self._run, args=(i,), daemon=True, name=f"b200-batcher-{i}")
                         for i in range(len(self.models))]
        for t in self._threads:
            t.start()

    async def score(self, frame: pd.DataFrame):
        """-> (proba1 (n,), is_outlier (n,) or None) for this request's rows."""
        loop = asyncio.get_running_loop()
        fut = loop.create_future()
        self.q.put(_Pending(frame, fut, loop))
        return await fut

    def close(self) -> None:
        self._stop = True
        for _ in self._threads:
            self.q.put(None)
        for t in self._threads:
            t.join(timeout=5)

    def _collect(self):
        first = self.q.get()
        if first is None:
            return None
        items, rows = [first], first.n
        deadline = time.perf_counter() + self.window_s
        while rows < self.max_rows:
            left = deadline - time.perf_counter()
            try:
                nxt = self.q.get(timeout=left) if left > 0 else self.q.get_nowait()
            except queue.Empty:
                break
            if nxt is None:
                self.q.put(None)
                break
            items.append(nxt)
            rows += nxt.n
        return items

    def _score_items(self, model, items):
        """One engine call for the whole batch -> per-item (proba, flags) parts."""
        frame = items[0].frame if len(items) == 1 else pd.concat([it.frame for it in items], ignore_index=True)
        # encode -> pinned slot -> H2D -> classifier kernel (+ outlier-forest kernel) -> D2H
        scorer = getattr(model, "score", None)
        proba, flags = scorer(frame) if scorer is not None else (model.predict_proba1(frame), None)
        self.batches += 1
        self.rows += len(frame)
        parts, off = [], 0
        for it in items:
            parts.append((proba[off:off + it.n], None if flags is None else flags[off:off + it.n]))
            off += it.n
        return parts

    def _run(self, idx: int) -> None:
        model = self.models[idx]
        while not self._stop:
            items = self._collect()
            if items is None:
                return
            self._serve(model, items)

    def _serve(self, model, items) -> None:
        try:
            parts = self._score_items(model, items)
            for it, part in zip(items, parts):
                it.loop.call_soon_threadsafe(_resolve, it.future, part, None)
        except BaseException as e:  # surfaces as HTTP 500, like any model exception in the reference
            if len(items) == 1:
                items[0].loop.call_soon_threadsafe(_resolve, items[0].future, None, e)
                return
            # the reference scores requests independently (app/main.py:72): a request the model rejects (a value
            # that overflows float32, NaN with the outlier forest attached ...) must fail ALONE -- re-score the
            # batch one request at a time and route each outcome to its own caller
            for it in items:
                try:
                    part = self._score_items(model, [it])[0]
                    it.loop.call_soon_threadsafe(_resolve, it.future, part, None)
                except BaseException as e1:
                    it.loop.call_soon_threadsafe(_resolve, it.future, None, e1)


def _resolve(fut, value, err):
    if fut.cancelled():
        return
    if err is not None:
        fut.set_exception(err)
    else:
        fut.set_result(value)


class _BoundedLogPool:
    """One logging thread with a BOUNDED backlog: each queued record holds its request's DataFrame, so an unbounded
    queue grows without limit when logging falls behind.  Above the backlog the record is written inline on the
    caller's thread (back-pressure, nothing is dropped: the log schema is an API for the reference's KQL queries)."""

    def __init__(self, backlog: int = 256):
        self._pool = ThreadPoolExecutor(max_workers=1, thread_name_prefix="b200-log")
        self._slots = threading.BoundedSemaphore(max(1, backlog))
        self.inline = 0

    def submit(self, fn, *args):
        if not self._slots.acquire(blocking=False):
            self.inline += 1
            fn(*args)
            return None

        def run():
            try:
                fn(*args)
            finally:
                self._slots.release()

        return self._pool.submit(run)


def _as_list(a: np.ndarray) -> list:
    """ndarray -> list; large float64 / int32 results go through the recycling list builder (``_pylists.py``)."""
    if len(a) >= 256 and a.ndim == 1 and a.dtype in (np.float64, np.int32):
        from ._pylists import ListBuilder

        b = ListBuilder(len(a))
        b.fill(0, a)
        return b.items
    return a.tolist()


_DEPENDENCE_PARAMETERS = [
    {"name": "feature", "in": "query", "required": True, "description": "request field to probe; repeat for several (at most 23)",
     "schema": {"type": "array", "items": {"type": "string"}}, "style": "form", "explode": True},
    {"name": "kind", "in": "query", "required": False, "schema": {"type": "string", "enum": list(dependence.KINDS), "default": "average"}},
    {"name": "grid_resolution", "in": "query", "required": False,
     "schema": {"type": "integer", "minimum": 2, "maximum": dependence.MAX_POINTS, "default": dependence.DEFAULT_RESOLUTION}},
    {"name": "value", "in": "query", "required": False,
     "description": "explicit grid point of the one probed field; repeat for several; empty = missing",
     "schema": {"type": "array", "items": {"type": "string"}}, "style": "form", "explode": True},
]


_PAIR_PARAMETERS = [
    {"name": "feature", "in": "query", "required": True, "description": "the two request fields of the pair, in order: exactly two, distinct",
     "schema": {"type": "array", "items": {"type": "string"}, "minItems": 2, "maxItems": 2}, "style": "form", "explode": True},
    {"name": "kind", "in": "query", "required": False, "schema": {"type": "string", "enum": list(dependence.KINDS), "default": "average"}},
    {"name": "grid_resolution", "in": "query", "required": False,
     "schema": {"type": "integer", "minimum": 2, "maximum": interaction.MAX_AXIS_POINTS, "default": dependence.DEFAULT_RESOLUTION}},
]

_STRENGTH_PARAMETERS = [
    {"name": "feature", "in": "query", "required": False, "description": "request field; repeat for several (at least 2), each at most once; none = every field",
     "schema": {"type": "array", "items": {"type": "string"}}, "style": "form", "explode": True},
    {"name": "sample", "in": "query", "required": False, "description": "rows of the sample the statistic is taken over",
     "schema": {"type": "integer", "minimum": 2, "maximum": interaction.MAX_SAMPLE, "default": interaction.DEFAULT_SAMPLE}},
    {"name": "random_state", "in": "query", "required": False, "description": "seed of the sample (numpy RandomState)",
     "schema": {"type": "integer", "minimum": 0, "maximum": 2**32 - 1, "default": 0}},
]


def _pair_problem(features, kind, grid_resolution) -> str | None:
    """Why a /explain/dependence/pair query is unprocessable, or None."""
    if len(features) != 2:
        return "exactly two feature parameters are needed"
    unknown = [f for f in features if f not in ALL_FEATURES]
    if unknown:
        return f"unknown feature(s) {unknown}"
    if features[0] == features[1]:
        return "the two features must differ"
    if kind not in dependence.KINDS:
        return f"kind must be one of {list(dependence.KINDS)}"
    if grid_resolution < 2:
        return "grid_resolution must be at least 2"
    if grid_resolution > interaction.MAX_AXIS_POINTS:
        return f"at most {interaction.MAX_AXIS_POINTS} grid points per feature"
    return None


def _strength_problem(features, sample: str, random_state: str) -> str | None:
    """Why a /explain/interaction_strength query is unprocessable, or None."""
    try:
        interaction.check_features(features or None, ALL_FEATURES)
    except ValueError as e:
        return str(e)
    try:
        interaction.check_sample(int(sample), int(random_state))
    except ValueError:
        return f"sample must be an integer in 2..{interaction.MAX_SAMPLE} and random_state an integer in [0, 2**32 - 1]"
    return None


def _nullable(a) -> list:
    """A float array for JSON: NaN -> null."""
    return [None if v != v else v for v in np.asarray(a, dtype=np.float64).tolist()]


_COUNTERFACTUAL_PARAMETERS = [
    {"name": "feature", "in": "query", "required": False,
     "description": "request field to probe; repeat for several, each at most once; none = every field",
     "schema": {"type": "array", "items": {"type": "string"}}, "style": "form", "explode": True},
    {"name": "cutoff", "in": "query", "required": False, "description": "the decision is P(class 1) > cutoff",
     "schema": {"type": "number", "minimum": 0, "maximum": 1, "default": 0.5}},
]


def _counterfactual_problem(features, cutoff: str) -> str | None:
    """Why a /explain/counterfactual query is unprocessable, or None."""
    unknown = [f for f in features if f not in ALL_FEATURES]
    if unknown:
        return f"unknown feature(s) {unknown}"
    if len(set(features)) != len(features):
        return f"repeated feature(s) {sorted({f for f in features if features.count(f) > 1})}"
    try:
        c = float(cutoff)
    except ValueError:
        c = float("nan")
    if not 0.0 <= c <= 1.0:
        return "cutoff must be a number in [0, 1]"
    return None


def _counterfactual_json(name: str, cf: dict) -> dict:
    """One field's counterfactuals for JSON: NaN (none) -> null."""
    if "flips" in cf:
        return {"feature": name, "value": cf["value"], "flips": [[[c, p] for c, p in row] for row in cf["flips"]]}
    return {"feature": name, **{k: [None if v != v else v for v in np.asarray(cf[k], dtype=np.float64).tolist()]
                                for k in ("value", "lower", "lower_prediction", "upper", "upper_prediction")}}


_LABELLED_SCHEMA = {"required": True, "content": {"application/json": {"schema": {
    "title": "Data", "type": "array", "items": LabelledApplicant.model_json_schema()}}}}

_IMPORTANCE_PARAMETERS = [
    {"name": "scoring", "in": "query", "required": False, "description": "scorer; repeat for several; none = accuracy",
     "schema": {"type": "array", "items": {"type": "string", "enum": list(importance.SCORERS)}}, "style": "form", "explode": True},
    {"name": "n_repeats", "in": "query", "required": False,
     "schema": {"type": "integer", "minimum": 1, "maximum": importance.MAX_REPEATS, "default": 5}},
    {"name": "random_state", "in": "query", "required": False, "description": "seed of the permutations (numpy RandomState)",
     "schema": {"type": "integer", "minimum": 0, "maximum": 2**32 - 1, "default": 0}},
]


def _importance_problem(scoring, n_repeats: str, random_state: str) -> str | None:
    """Why a /explain/importance query is unprocessable, or None."""
    try:
        importance.check_scoring(scoring or None)
    except ValueError as e:
        return str(e)
    try:
        importance.check_n_repeats(int(n_repeats))
    except ValueError:
        return f"n_repeats must be an integer in 1..{importance.MAX_REPEATS}"
    try:
        seed = int(random_state)
    except ValueError:
        seed = -1
    if not 0 <= seed < 2**32:
        return "random_state must be an integer in [0, 2**32 - 1]"
    return None


def parse_labelled(raw: bytes) -> list:
    """A /explain/importance body -> validated dict rows (pydantic-core, FastAPI's 422 on a bad field or label)."""
    try:
        return LABELLED_ROWS.validate_json(raw)
    except ValidationError as e:
        raise RequestValidationError([{**err, "loc": ("body", *err["loc"])} for err in e.errors(include_url=False, include_context=False)])


def _dependence_problem(features, values, kind, grid_resolution) -> str | None:
    """Why a /explain/dependence query is unprocessable, or None."""
    if not features:
        return "at least one feature parameter is needed"
    if len(features) > dependence.MAX_FEATURES:
        return f"at most {dependence.MAX_FEATURES} features per request"
    unknown = [f for f in features if f not in ALL_FEATURES]
    if unknown:
        return f"unknown feature(s) {unknown}"
    if kind not in dependence.KINDS:
        return f"kind must be one of {list(dependence.KINDS)}"
    if grid_resolution < 2:
        return "grid_resolution must be at least 2"
    if grid_resolution > dependence.MAX_POINTS or len(values) > dependence.MAX_POINTS:
        return f"at most {dependence.MAX_POINTS} grid points per feature"
    if values and len(features) != 1:
        return "explicit values need exactly one feature"
    return None


_ALE_PARAMETERS = [
    {"name": "feature", "in": "query", "required": False,
     "description": "numeric request field; repeat for several, each at most once; none = every numeric field",
     "schema": {"type": "array", "items": {"type": "string", "enum": list(NUMERIC_FEATURES)}}, "style": "form", "explode": True},
    {"name": "bins", "in": "query", "required": False, "description": "most bins per field of the default (quantile) edges",
     "schema": {"type": "integer", "minimum": 1, "maximum": ale.MAX_BINS, "default": ale.DEFAULT_BINS}},
    {"name": "min_bin_points", "in": "query", "required": False, "description": "fewest request rows per bin of the default edges",
     "schema": {"type": "integer", "minimum": 1, "default": ale.DEFAULT_MIN_BIN_POINTS}},
    {"name": "value", "in": "query", "required": False,
     "description": "explicit bin edge of the one probed field; repeat for 2..257 strictly increasing numbers",
     "schema": {"type": "array", "items": {"type": "number"}}, "style": "form", "explode": True},
]


def _ale_problem(features, values, bins: str, min_bin_points: str) -> str | None:
    """Why a /explain/ale query is unprocessable, or None (edges the rows cannot give are the model's ValueError)."""
    try:
        ale.check_features(features or None, NUMERIC_FEATURES, CATEGORICAL_FEATURES)
        ale.check_params(int(bins), int(min_bin_points))
    except ValueError as e:
        return str(e) if "invalid literal" not in str(e) else "bins and min_bin_points must be integers"
    if values:
        if len(features) != 1:
            return "explicit values need exactly one feature"
        try:
            ale.check_custom_edges(features[0], values)
        except ValueError as e:
            return str(e)
    return None


_MMD_PARAMETERS = [
    {"name": "n_permutations", "in": "query", "required": False,
     "schema": {"type": "integer", "minimum": 1, "maximum": mmd.MAX_PERMUTATIONS, "default": 100}},
    {"name": "p_val", "in": "query", "required": False, "description": "drift when the permutation p-value is below it",
     "schema": {"type": "number", "exclusiveMinimum": 0, "maximum": 1, "default": 0.05}},
    {"name": "random_state", "in": "query", "required": False, "description": "seed of the permutations (numpy default_rng)",
     "schema": {"type": "integer", "minimum": 0, "default": 0}},
]


_TRUST_PARAMETERS = [
    {"name": "k", "in": "query", "required": False, "description": "neighbours per class: at most the rows the reference keeps in either class",
     "schema": {"type": "integer", "minimum": 1, "maximum": trust.MAX_K, "default": 2}},
    {"name": "dist_type", "in": "query", "required": False, "description": "D_c: the k-th nearest distance (point) or the mean of the k nearest",
     "schema": {"type": "string", "enum": list(trust.DIST_TYPES), "default": "point"}},
    {"name": "neighbours", "in": "query", "required": False, "description": "also answer each applicant's neighbours per class",
     "schema": {"type": "boolean", "default": False}},
]


def _trust_problem(k: str, dist_type: str, neighbours: str) -> str | None:
    """Why a /explain/trust query is unprocessable, or None (the k bound against the reference is the model's)."""
    try:
        k_ = int(k)
    except ValueError:
        return f"k must be an integer in 1..{trust.MAX_K}"
    if not 1 <= k_ <= trust.MAX_K:
        return f"k must be an integer in 1..{trust.MAX_K}"
    if dist_type not in trust.DIST_TYPES:
        return f"dist_type must be one of {list(trust.DIST_TYPES)}"
    if neighbours not in ("true", "false"):
        return "neighbours must be true or false"
    return None


def _finite_or_null(a) -> list:
    """A float array for JSON: every value that is not a finite number (NaN, or a distance past float64's range) -> null."""
    a = np.asarray(a, dtype=np.float64)
    out = a.astype(object)
    out[~np.isfinite(a)] = None
    return out.tolist()


def _unprocessable(detail: str) -> Response:
    return Response(content=json.dumps({"detail": detail}), status_code=422, media_type="application/json")


def _query_value(v: str, categorical: bool):
    """A `value` query parameter -> a grid value: the string for a categorical field, else a float; empty = missing."""
    if v == "":
        return None
    return v if categorical else float(v)


def _json_value(v):
    """A grid value for JSON: NaN (missing) -> null, numpy scalars -> Python."""
    if isinstance(v, (float, np.floating)) and v != v:
        return None
    return v.item() if isinstance(v, np.generic) else v


def _log_record(kind: str, request_id: str, payload) -> None:
    logging.info(json.dumps({"service_name": _service_name(), "type": kind, "request_id": request_id, "data": payload}))


def create_app(model=None, loader=None) -> FastAPI:
    """Build the app.  ``model``: an already-built B200Model (tests); otherwise ``loader`` (default
    ``databricks_kubernetes_mlops_poc_b200.load_model``) is called in ``lifespan`` on ``MODEL_DIRECTORY``."""
    log_pool = _BoundedLogPool(int(os.environ.get("B200_LOG_BACKLOG", "256")))
    parser = NativeRequestParser()

    @asynccontextmanager
    async def lifespan(app: FastAPI) -> AsyncGenerator[None, None]:
        if model is not None:
            ml_models["credit_default"] = model
        else:
            from . import load_model

            ml_models["credit_default"] = (loader or load_model)(os.getenv("MODEL_DIRECTORY", "./app/model"))
        m = ml_models["credit_default"]
        ml_models["_batcher"] = MicroBatcher(
            getattr(m, "replicas", None) or [m],
            max_rows=int(os.environ.get("B200_MAX_BATCH", "65536")),
            window_us=int(os.environ.get("B200_BATCH_WINDOW_US", "200")),
        )
        yield
        ml_models["_batcher"].close()
        closer = getattr(ml_models.get("credit_default"), "close", None)
        ml_models.clear()
        if closer and model is None:
            closer()

    app = FastAPI(title=_service_name(), docs_url="/", lifespan=lifespan)

    async def answered(request: Request, call) -> Response:
        """What the /explain routes share: parse the body like /predict (an empty list is a 500, as there), then run
        ``call(model, frame)`` on the executor.  It returns the answer: a Response, or a dict sent as compact JSON."""
        input_df = parser.frame(await request.body())
        if len(input_df) == 0:
            raise KeyError(f"None of {ALL_FEATURES} are in the [columns]")
        out = await asyncio.get_running_loop().run_in_executor(None, call, ml_models["credit_default"], input_df)
        if isinstance(out, Response):
            return out
        return Response(content=json.dumps(out, allow_nan=False, separators=(",", ":")).encode("utf-8"), media_type="application/json")

    async def explained(request: Request, method: str, key: str, attached: str = "explainer_attached", missing: str = "explainer",
                        extra: tuple = ()) -> Response:
        """The TreeSHAP routes: 501 unless ``model.<attached>`` (the model has a ``missing``), else ``model.<method>``'s ``key``
        array as nested lists, plus its ``extra`` keys."""

        def call(m, input_df):
            if not getattr(m, attached, False):
                return Response(content=json.dumps({"detail": f"this model has no {missing}"}), status_code=501, media_type="application/json")
            out = getattr(m, method)(input_df)
            body = {"feature_names": list(out["feature_names"]), "output": out["output"], "base_value": float(out["base_value"]),
                    "predictions": list(out["predictions"]), key: np.asarray(out[key], dtype=np.float64).tolist()}
            body.update({k: out[k] for k in extra})
            return body

        return await answered(request, call)

    @app.post("/explain", openapi_extra={"requestBody": _REQUEST_SCHEMA})
    async def explain(request: Request):
        """Explain each applicant's score: exact TreeSHAP contribution of every request field (probability space for a random
        forest, log-odds for a GBDT), the base value they start from, and the predictions themselves.  501 when the model was
        loaded without an explainer."""
        return await explained(request, "explain", "contributions")

    @app.post("/explain/interactions", openapi_extra={"requestBody": _REQUEST_SCHEMA})
    async def explain_interactions(request: Request):
        """Explain each applicant's score by pairs of request fields: exact TreeSHAP interaction values, one symmetric
        fields x fields matrix per applicant whose rows sum to /explain's contributions (same output space, base value and
        predictions).  501 when the model was loaded without an explainer."""
        return await explained(request, "explain_interactions", "interactions")

    @app.post("/explain/interventional", openapi_extra={"requestBody": _REQUEST_SCHEMA})
    async def explain_interventional(request: Request):
        """Explain each applicant's score against the model's background set: exact interventional TreeSHAP, the mean over
        background rows of each request field's Shapley value when the applicant's values replace the background row's (same
        output space as /explain; base_value is the mean prediction over the background, whose size is background_rows).  A
        field the model never reads gets 0.  501 when the model has no explainer or no background."""
        return await explained(request, "explain_interventional", "contributions", "background_attached", "background set",
                               ("background_rows",))

    @app.post("/explain/dependence", openapi_extra={"requestBody": _REQUEST_SCHEMA, "parameters": _DEPENDENCE_PARAMETERS})
    async def explain_dependence(request: Request):
        """What-if curves: each applicant's default probability with one request field set to each point of a grid (ICE
        curves, `individual`) and their mean over the applicants (partial dependence, `average`), one field at a time.  The
        grid is the repeated `value` parameters (one field only), else the default grid of the model's background set when it
        has one, else of the request rows.  422 for an unknown field, a bad kind, grid_resolution < 2 or more than 256
        points."""
        q = request.query_params
        features, values, kind = q.getlist("feature"), q.getlist("value"), q.get("kind", "average")
        try:
            grid_resolution = int(q.get("grid_resolution", dependence.DEFAULT_RESOLUTION))
        except ValueError:
            return _unprocessable("grid_resolution must be an integer")
        problem = _dependence_problem(features, values, kind, grid_resolution)
        if problem:
            return _unprocessable(problem)

        def call(m, input_df):
            kw = {"kind": kind, "grid_resolution": grid_resolution}
            if values:
                name = features[0]
                try:
                    kw["custom_values"] = {name: [_query_value(v, name in m.categorical_features) for v in values]}
                except ValueError:
                    return _unprocessable(f"value parameters of numeric field {name!r} must be numbers")
            elif getattr(m, "background_attached", False):
                grids = m.dependence_grids if grid_resolution == dependence.DEFAULT_RESOLUTION else {}
                kw["custom_values"] = {f: grids[f] for f in features if f in grids}
                kw["grid_frame"] = m.background
            out = m.partial_dependence(input_df, features, **kw)
            body = {"feature_names": out["feature_names"], "output": out["output"],
                    "grid_values": [[_json_value(v) for v in g] for g in out["grid_values"]]}
            for key in ("average", "individual"):
                if key in out:
                    body[key] = [np.asarray(a, dtype=np.float64).tolist() for a in out[key]]
            return body

        return await answered(request, call)

    @app.post("/explain/dependence/pair", openapi_extra={"requestBody": _REQUEST_SCHEMA, "parameters": _PAIR_PARAMETERS})
    async def explain_dependence_pair(request: Request):
        """How the score moves when two fields change together: two-way partial dependence.  For each point (u, v) of the
        two fields' grids (their Cartesian product, the first field slowest), each applicant's default probability with
        the first field set to u and the second to v (`individual`, applicants x u x v) and their mean over the applicants
        (`average`, u x v).  Grids as /explain/dependence: the model's background set when it has one, else the request
        rows.  422 for other than two distinct known fields, a bad kind, grid_resolution < 2, an axis of more than 256
        points, or an `individual` of more than 2^24 values."""
        q = request.query_params
        features, kind = q.getlist("feature"), q.get("kind", "average")
        try:
            grid_resolution = int(q.get("grid_resolution", dependence.DEFAULT_RESOLUTION))
        except ValueError:
            return _unprocessable("grid_resolution must be an integer")
        problem = _pair_problem(features, kind, grid_resolution)
        if problem:
            return _unprocessable(problem)
        pair = (features[0], features[1])

        def call(m, input_df):
            kw = {"grid_resolution": grid_resolution}
            if getattr(m, "background_attached", False):
                grids = m.dependence_grids if grid_resolution == dependence.DEFAULT_RESOLUTION else {}
                kw["custom_values"] = {f: grids[f] for f in pair if f in grids}
                kw["grid_frame"] = m.background
            try:
                (ga, gb), = m.pair_grids(input_df, [pair], **kw)
            except ValueError as e:
                return _unprocessable(str(e))
            if kind != "average" and len(input_df) * len(ga) * len(gb) > interaction.MAX_INDIVIDUAL_VALUES:
                return _unprocessable(f"individual would hold {len(input_df) * len(ga) * len(gb)} values, more than 2^24")
            out = m.pair_dependence(input_df, [pair], kind=kind, custom_values={pair[0]: ga, pair[1]: gb})
            body = {"feature_names": list(pair), "output": out["output"],
                    "grid_values": [[_json_value(v) for v in g] for g in out["grid_values"][0]]}
            for key in ("average", "individual"):
                if key in out:
                    body[key] = np.asarray(out[key][0], dtype=np.float64).tolist()
            return body

        return await answered(request, call)

    @app.post("/explain/interaction_strength", openapi_extra={"requestBody": _REQUEST_SCHEMA, "parameters": _STRENGTH_PARAMETERS})
    async def explain_interaction_strength(request: Request):
        """Which pairs of fields interact across the applicants: Friedman's H-statistic H^2 of every pair of the `feature`
        fields (every field without one), over a sample of at most `sample` applicants (numpy RandomState(random_state)
        when there are more).  H^2 is the share of the pair's two-way partial dependence that the two one-way ones do not
        explain: 0 for fields that act additively.  The answer lists the pairs, `h_squared` with its `numerator` and
        `denominator` (H^2 is unstable where the denominator is small), the symmetric `matrix` and the sample size `rows`;
        null where the denominator is 0.  422 for an unknown or repeated field, fewer than 2 fields, a bad sample or
        random_state, or fewer than 2 applicants."""
        q = request.query_params
        features, sample, random_state = q.getlist("feature"), q.get("sample", str(interaction.DEFAULT_SAMPLE)), q.get("random_state", "0")
        problem = _strength_problem(features, sample, random_state)
        if problem:
            return _unprocessable(problem)

        def call(m, input_df):
            if len(input_df) < 2:
                return _unprocessable(f"interaction strength needs at least 2 rows, got {len(input_df)}")
            out = m.interaction_strength(input_df, features or None, sample=int(sample), random_state=int(random_state))
            return {"feature_names": list(out["feature_names"]), "rows": int(out["rows"]), "pairs": [list(p) for p in out["pairs"]],
                    "h_squared": _nullable(out["h_squared"]), "numerator": _nullable(out["numerator"]),
                    "denominator": _nullable(out["denominator"]), "matrix": [_nullable(r) for r in out["matrix"]]}

        return await answered(request, call)

    @app.post("/explain/ale", openapi_extra={"requestBody": _REQUEST_SCHEMA, "parameters": _ALE_PARAMETERS})
    async def explain_ale(request: Request):
        """How the default probability moves with each numeric field where the applicants actually are: accumulated local
        effects.  Each applicant is scored only at the two edges of the bin its own value lies in; a bin's effect is the
        mean change over its applicants, and `ale_values` (one per edge in `feature_values`) are the effects summed along
        the field and centred on the applicants (`ale0` is what was taken off).  Unlike /explain/dependence, no applicant is
        moved to values far from its own, so correlated fields (the six bill amounts) are not scored at combinations no one
        has.  The edges are the repeated `value` parameters (one field only), else quantiles of the request rows with at
        least `min_bin_points` rows per bin, at most `bins` bins (every distinct value when there are few).  An applicant
        missing the field takes no part in it.  `bin_effects` and `bin_rows` give each bin's effect and size;
        `constant_value` is the mean probability.  422 for an unknown, categorical or repeated field, a bad bins or
        min_bin_points, bad values, or a field no request row has a value for."""
        q = request.query_params
        features, values = q.getlist("feature"), q.getlist("value")
        bins, min_bin_points = q.get("bins", str(ale.DEFAULT_BINS)), q.get("min_bin_points", str(ale.DEFAULT_MIN_BIN_POINTS))
        problem = _ale_problem(features, values, bins, min_bin_points)
        if problem:
            return _unprocessable(problem)

        def call(m, input_df):
            kw = {"bins": int(bins), "min_bin_points": int(min_bin_points)}
            if values:
                kw["custom_edges"] = {features[0]: [float(v) for v in values]}
            try:
                out = m.accumulated_local_effects(input_df, features or None, **kw)
            except ValueError as e:
                return _unprocessable(str(e))
            return {"feature_names": list(out["feature_names"]), "output": out["output"], "rows": int(out["rows"]),
                    "constant_value": float(out["constant_value"]),
                    "feature_values": [np.asarray(v, dtype=np.float64).tolist() for v in out["feature_values"]],
                    "ale_values": [np.asarray(v, dtype=np.float64).tolist() for v in out["ale_values"]],
                    "bin_effects": [np.asarray(v, dtype=np.float64).tolist() for v in out["bin_effects"]],
                    "bin_rows": [np.asarray(v, dtype=np.int64).tolist() for v in out["bin_rows"]],
                    "ale0": [float(v) for v in out["ale0"]]}

        return await answered(request, call)

    @app.post("/explain/counterfactual", openapi_extra={"requestBody": _REQUEST_SCHEMA, "parameters": _COUNTERFACTUAL_PARAMETERS})
    async def explain_counterfactual(request: Request):
        """What would change the decision: for each applicant and probed field (every field without a `feature` parameter),
        the nearest value of that field alone at which the decision P(class 1) > cutoff flips.  A numeric field answers the
        largest value below (`lower`) and the smallest above (`upper`) the applicant's `value` that flip it, exact float32
        boundaries, with the probability there; null when no value on that side flips it.  A categorical field answers the
        categories that flip it (`flips`: [category, probability] pairs).  422 for an unknown or repeated field or a cutoff
        that is not a number in [0, 1]."""
        q = request.query_params
        features, cutoff = q.getlist("feature"), q.get("cutoff", "0.5")
        problem = _counterfactual_problem(features, cutoff)
        if problem:
            return _unprocessable(problem)

        def call(m, input_df):
            out = m.counterfactuals(input_df, features or None, cutoff=float(cutoff))
            return {"feature_names": list(out["feature_names"]), "output": out["output"], "cutoff": out["cutoff"],
                    "predictions": np.asarray(out["predictions"], dtype=np.float64).tolist(), "decisions": np.asarray(out["decisions"]).tolist(),
                    "counterfactuals": [_counterfactual_json(f, cf) for f, cf in zip(out["feature_names"], out["counterfactuals"])]}

        return await answered(request, call)

    @app.post("/explain/importance", openapi_extra={"requestBody": _LABELLED_SCHEMA, "parameters": _IMPORTANCE_PARAMETERS})
    async def explain_importance(request: Request):
        """Which fields the model relies on: permutation importance against labelled applicants (each applicant's fields
        plus its observed `default_payment_next_month`), scikit-learn's `permutation_importance` of the fitted pipeline.
        Every field is shuffled across the applicants `n_repeats` times and the drop of each scorer below its baseline is
        reported per field (`importances_mean`, `importances_std`, and every repeat in `importances`); null where a score is
        undefined (roc_auc with one class).  422 for an unknown scorer, a bad n_repeats or random_state, a missing or
        non-0/1 label, and labels of one class with neg_log_loss."""
        q = request.query_params
        scoring, n_repeats, random_state = q.getlist("scoring"), q.get("n_repeats", "5"), q.get("random_state", "0")
        problem = _importance_problem(scoring, n_repeats, random_state)
        if problem:
            return _unprocessable(problem)
        rows = parse_labelled(await request.body())
        if len(rows) == 0:
            raise KeyError(f"None of {ALL_FEATURES} are in the [columns]")
        labels = np.array([r[TARGET] for r in rows], dtype=np.int32)
        names = scoring or [importance.DEFAULT_SCORER]
        try:
            importance.check_single_class(names, labels)
        except ValueError as e:
            return _unprocessable(str(e))
        frame = rows_to_frame(rows)

        def call():
            out = ml_models["credit_default"].permutation_importance(frame, labels, scoring=names, n_repeats=int(n_repeats),
                                                                    random_state=int(random_state))
            first = out[names[0]]
            return {"feature_names": list(first["feature_names"]), "rows": int(first["rows"]), "n_repeats": int(first["n_repeats"]),
                    "random_state": int(random_state),
                    "scores": {s: {"baseline": importance.json_number(r["baseline_score"]),
                                   "importances_mean": [importance.json_number(v) for v in r["importances_mean"]],
                                   "importances_std": [importance.json_number(v) for v in r["importances_std"]],
                                   "importances": [[importance.json_number(v) for v in row] for row in r["importances"]]}
                               for s, r in out.items()}}

        out = await asyncio.get_running_loop().run_in_executor(None, call)
        return Response(content=json.dumps(out, allow_nan=False, separators=(",", ":")).encode("utf-8"), media_type="application/json")

    @app.post("/explain/trust", openapi_extra={"requestBody": _REQUEST_SCHEMA, "parameters": _TRUST_PARAMETERS})
    async def explain_trust(request: Request):
        """Can each decision be trusted?  alibi's trust score against the model's labelled reference: the distance from the
        applicant to its k-th nearest reference applicant of the other class (`distance_to_other`) over the distance to its
        k-th nearest of the predicted class (`distance_to_pred`), on the classifier's input vectors (one-hot categoricals,
        z-scored numerics).  Below 1, applicants like this one mostly turned out the other way.  `labels` is the predicted
        class, `closest_not_pred` the other one, `predictions` P(class 1).  With `neighbours=true`, per class the reference
        rows found (positions in the reference frame) and their distances, nearest first.  null stands for a value that is
        not a finite number.  501 when the model has no trust reference; 422 for a bad k, dist_type or neighbours."""
        q = request.query_params
        k, dist_type, neighbours = q.get("k", "2"), q.get("dist_type", "point"), q.get("neighbours", "false")
        problem = _trust_problem(k, dist_type, neighbours)
        if problem:
            return _unprocessable(problem)
        m = ml_models["credit_default"]
        if not getattr(m, "trust_reference_attached", False):
            return Response(content=json.dumps({"detail": "this model has no trust reference"}), status_code=501, media_type="application/json")
        try:
            trust.check_score(int(k), dist_type, m.trust_reference_rows)
        except ValueError as e:
            return _unprocessable(str(e))

        def call(m, input_df):
            out = m.trust_score(input_df, k=int(k), dist_type=dist_type)
            body = {"trust_score": _finite_or_null(out["trust_score"]), "closest_not_pred": np.asarray(out["closest_not_pred"]).tolist(),
                    "predictions": np.asarray(out["predictions"], dtype=np.float64).tolist(), "labels": np.asarray(out["labels"]).tolist(),
                    "distance_to_pred": _finite_or_null(out["distance_to_pred"]), "distance_to_other": _finite_or_null(out["distance_to_other"]),
                    "k": out["k"], "dist_type": out["dist_type"], "reference_rows": list(out["reference_rows"])}
            if neighbours == "true":
                body["neighbours"] = [{"class": nb["class"], "index": np.asarray(nb["index"]).tolist(), "distance": _finite_or_null(nb["distance"])}
                                      for nb in out["neighbours"]]
            return body

        return await answered(request, call)

    @app.post("/drift/mmd", openapi_extra={"requestBody": _REQUEST_SCHEMA, "parameters": _MMD_PARAMETERS})
    async def drift_mmd(request: Request):
        """Has the joint distribution of the applicants moved?  The kernel two-sample (MMD) test of the batch against the
        model's reference table, alibi-detect's MMDDrift on the classifier's input vectors: `distance` is the unbiased MMD^2,
        `p_val` its permutation p-value, `is_drift` = p_val < `threshold`, and `distance_threshold` the permuted statistic
        at that quantile.  Per-field tests (/predict's feature_drift_batch) cannot see a change in how fields move together;
        this can.  501 when the model has no reference; 422 for fewer than 2 applicants, a bad parameter, or a request whose
        permutations need more than 2^36 kernel pairs."""
        q = request.query_params
        try:
            n_permutations, p_val, random_state = int(q.get("n_permutations", "100")), float(q.get("p_val", "0.05")), int(q.get("random_state", "0"))
        except ValueError:
            return _unprocessable("n_permutations and random_state must be integers and p_val a number")
        m = ml_models["credit_default"]
        if not getattr(m, "mmd_reference_attached", False):
            return Response(content=json.dumps({"detail": "this model has no MMD reference"}), status_code=501, media_type="application/json")
        input_df = parser.frame(await request.body())
        try:
            mmd.check_request(len(input_df), m.mmd_reference_rows, n_permutations, p_val, random_state)
        except ValueError as e:
            return _unprocessable(str(e))
        out = await asyncio.get_running_loop().run_in_executor(
            None, lambda: m.mmd_drift(input_df, n_permutations=n_permutations, p_val=p_val, random_state=random_state))
        return Response(content=json.dumps(out, allow_nan=False, separators=(",", ":")).encode("utf-8"), media_type="application/json")

    @app.post("/predict", response_model=ModelOutput, openapi_extra={"requestBody": _REQUEST_SCHEMA})
    async def predict(request: Request):
        """Score a list of loan applicants: default probability, outlier flag, per-feature batch drift."""
        # list[LoanApplicant] semantics (422 on a type error, defaults filled): native one-pass parser for bodies of the
        # regular shape, pydantic-core for everything else (ingest.py)
        input_df = parser.frame(await request.body())
        if len(input_df) == 0:
            # the reference's empty DataFrame has no columns and dies in df[self.all_features] -> HTTP 500
            raise KeyError(f"None of {ALL_FEATURES} are in the [columns]")
        m = ml_models["credit_default"]
        request_id = uuid.uuid4().hex
        log_pool.submit(lambda: _log_record("InferenceData", request_id, input_df.to_json(orient="records")))

        # the drift scores depend on this request's rows only (no cross-request batching): start them first, on their
        # own device stream, and let them run while the batcher encodes and scores the rows
        drift = getattr(m, "drift", None)
        pending = asyncio.get_running_loop().run_in_executor(None, drift.score, input_df) if drift is not None else None
        try:
            proba, flags = await ml_models["_batcher"].score(input_df)
        finally:
            drift_scores = (await pending) if pending is not None else [0.0] * len(ALL_FEATURES)
        model_output = {
            "predictions": _as_list(proba),
            "outliers": _as_list(flags) if flags is not None else [0] * len(input_df),
            "feature_drift_batch": dict(zip(ALL_FEATURES, drift_scores)),
        }
        log_pool.submit(_log_record, "ModelOutput", request_id, model_output)
        # Response side (reference app/main.py:42,86: `response_model=ModelOutput` makes FastAPI validate the dict field by
        # field and run it through jsonable_encoder before rendering).  Every value here was produced by this handler with
        # the declared types, so the body is rendered once, exactly as Starlette's JSONResponse would render the validated
        # model (compact separators, allow_nan=False -> a NaN drift score is the same ValueError -> HTTP 500)
        body = json.dumps(model_output, ensure_ascii=False, allow_nan=False, indent=None, separators=(",", ":")).encode("utf-8")
        return Response(content=body, media_type="application/json")

    return app


logging.basicConfig(level=logging.INFO)

if __name__ == "__main__":
    import uvicorn

    uvicorn.run(create_app(), host="0.0.0.0", port=5000)
