"""Request / response schema of the scoring service.

Wire-compatible with the reference's pydantic models (``LoanApplicant`` reference
``app/model.py:8-34``, ``FeatureBatchDrift`` ``:37-61``, ``ModelOutput`` ``:64-70``): same field
names, order, types and defaults, so FastAPI validates and serialises requests identically
(422 on a type error, missing fields take the defaults, ``[{}]`` is a valid request, integer
outlier flags are serialised as floats).  The models are generated from one feature table
instead of being spelled out, and they are plain pydantic models (the reference additionally
makes them dataclasses only so that ``pd.DataFrame(rows)`` works, ``app/main.py:54``; the
batching loop here builds its columns directly and does not need that).
"""

from __future__ import annotations

from typing import Annotated, Required, TypedDict

from pydantic import BaseModel, Field, TypeAdapter, create_model

# (name, default) in the order the model was trained on: categorical block, then numeric block
# (reference 01-train-model.ipynb:126-158; defaults from app/model.py:12-34 -- including the
# reference's own `age` = 18000 default, kept because defaults are part of the API)
_CATEGORICAL = [
    ("sex", "male"),
    ("education", "university"),
    ("marriage", "married"),
    *[(f"repayment_status_{i}", "duly_paid") for i in (1, 2, 3, 4)],
    *[(f"repayment_status_{i}", "no_delay") for i in (5, 6)],
]
_NUMERIC = [
    ("credit_limit", 18000.0),
    ("age", 18000.0),
    *zip([f"bill_amount_{i}" for i in range(1, 7)], [764.95, 2221.95, 1131.85, 5074.85, 18000.0, 1419.95]),
    *zip([f"payment_amount_{i}" for i in range(1, 7)], [2236.5, 1137.55, 5084.55, 111.65, 306.9, 805.65]),
]

CATEGORICAL_FEATURES = [n for n, _ in _CATEGORICAL]
NUMERIC_FEATURES = [n for n, _ in _NUMERIC]
ALL_FEATURES = CATEGORICAL_FEATURES + NUMERIC_FEATURES
DEFAULTS = {**dict(_CATEGORICAL), **dict(_NUMERIC)}

LoanApplicant = create_model(
    "LoanApplicant",
    **{n: (str, d) for n, d in _CATEGORICAL},
    **{n: (float, d) for n, d in _NUMERIC},
)
LoanApplicant.__doc__ = "One applicant: 9 categorical strings then 14 numerics, every field defaulted."

# The same row as a TypedDict: what the server validates request bodies into.  Same fields, types and coercion rules as
# ``LoanApplicant`` (pydantic validates both with the same core schema per field); absent keys stay absent and take
# ``DEFAULTS`` when the columns are built, so no per-row model object is constructed on the request path.
LoanApplicantRow = TypedDict(
    "LoanApplicantRow",
    {**{n: str for n in CATEGORICAL_FEATURES}, **{n: float for n in NUMERIC_FEATURES}},
    total=False,
)
REQUEST_ROWS = TypeAdapter(list[LoanApplicantRow])  # validate_json: JSON parsing + validation in one pass of pydantic-core

# A labelled applicant (``POST /explain/importance``): the same fields plus the reference's target column, required and 0/1
# (reference 01-train-model.ipynb: ``default_payment_next_month``).
TARGET = "default_payment_next_month"
_Label = Annotated[int, Field(ge=0, le=1)]
LabelledApplicant = create_model("LabelledApplicant", __base__=LoanApplicant, **{TARGET: (_Label, ...)})
LabelledApplicant.__doc__ = "One applicant with its observed outcome: LoanApplicant's fields plus the 0/1 target."
LabelledApplicantRow = TypedDict(
    "LabelledApplicantRow",
    {**{n: str for n in CATEGORICAL_FEATURES}, **{n: float for n in NUMERIC_FEATURES}, TARGET: Required[_Label]},
    total=False,
)
LABELLED_ROWS = TypeAdapter(list[LabelledApplicantRow])

FeatureBatchDrift = create_model("FeatureBatchDrift", **{n: (float, ...) for n in ALL_FEATURES})
FeatureBatchDrift.__doc__ = "Per-feature drift score of the request batch (1 - p-value)."


class ModelOutput(BaseModel):
    """Response body: per-row P(default), per-row outlier flag, per-feature batch drift."""

    predictions: list[float]
    outliers: list[float]
    feature_drift_batch: FeatureBatchDrift


def sample_request() -> list[dict]:
    """The one-row body of the reference's CI smoke test (``app/sample-request.json``):
    every field at its schema default."""
    return [dict(DEFAULTS)]
