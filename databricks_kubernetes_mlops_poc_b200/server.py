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

from . import dependence
from .ingest import NativeRequestParser, parse_rows, rows_to_frame  # noqa: F401  (rows_to_frame re-exported)
from .schema import ALL_FEATURES, LoanApplicant, ModelOutput

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
