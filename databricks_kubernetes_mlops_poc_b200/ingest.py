"""Request body -> the 23 named columns.

The reference does this with ``json.loads`` + one ``LoanApplicant`` object per row + ``pd.DataFrame(rows)``
(``app/main.py:42-54``, ``app/model.py:8-34``).  Here a body of the regular shape goes through the native parser
(``csrc/json_rows.h``, C ABI ``b2f_json_parser_*``): one pass over the bytes into float64 arrays and Arrow string
buffers, which become the DataFrame's columns without any per-row Python object.  Bodies outside that narrow grammar
(unknown keys, escapes, numbers in strings, malformed JSON, ...) are handed unchanged to the general validator
(``parse_rows``: pydantic-core over the raw bytes), which applies ``list[LoanApplicant]``'s coercions and produces
FastAPI's 422 responses -- so the observable behaviour is the validator's, the fast path only makes the common case cheap.
The native parser is host code inside ``libb200forest.so``; like the rest of the package it has no pure-Python twin.
"""

from __future__ import annotations

import ctypes as C
import threading

import numpy as np
import pandas as pd
from fastapi.exceptions import RequestValidationError
from pydantic import ValidationError

from . import _cabi
from .schema import ALL_FEATURES, CATEGORICAL_FEATURES, DEFAULTS, NUMERIC_FEATURES, REQUEST_ROWS

try:  # Arrow-backed string columns straight from the parser's buffers
    import pyarrow as pa
except ImportError:  # pragma: no cover - pyarrow ships with the image
    pa = None

EIRREGULAR = -8
# below this body size the 23 pandas / Arrow column objects cost more than the per-row Python work they replace
NATIVE_MIN_BYTES = 48 * 1024


def parse_rows(raw: bytes) -> list:
    """Request body -> validated dict rows, with FastAPI's own 422 behaviour (``RequestValidationError`` ->
    {"detail": [...]}, locations prefixed with "body") -- one pydantic-core pass over the bytes."""
    try:
        return REQUEST_ROWS.validate_json(raw)
    except ValidationError as e:
        # rows are validated as TypedDicts (no per-row model object); the one place that shows through is the error type of
        # a non-object row, which list[LoanApplicant] reports as "model_type" -- rewritten so the 422 body is identical
        raise RequestValidationError([{**err, "type": "model_type" if err["type"] == "dict_type" else err["type"], "loc": ("body", *err["loc"])}
                                      for err in e.errors(include_url=False, include_context=False)])


def rows_to_frame(data) -> pd.DataFrame:
    """Validated request rows -> the 23 named columns, built column-wise.  Rows are dicts (``LoanApplicantRow``: absent
    keys take the schema defaults) or objects with the 23 attributes."""
    cols = {}
    if len(data) and isinstance(data[0], dict):
        for name in CATEGORICAL_FEATURES:
            d = DEFAULTS[name]
            # validated `str` fields: an Arrow-backed string column, which the native row encoder reads in place
            cols[name] = pd.array([r.get(name, d) for r in data], dtype="str")
        for name in NUMERIC_FEATURES:
            d = DEFAULTS[name]
            cols[name] = np.array([r.get(name, d) for r in data], dtype=np.float64)
        return pd.DataFrame(cols, columns=ALL_FEATURES)
    for name in CATEGORICAL_FEATURES:
        cols[name] = pd.array([getattr(r, name) for r in data], dtype="str")
    for name in NUMERIC_FEATURES:
        cols[name] = np.array([getattr(r, name) for r in data], dtype=np.float64)
    return pd.DataFrame(cols, columns=ALL_FEATURES)


class NativeRequestParser:
    """Owner of a ``b2f_json_parser*`` for the service's schema (thread-safe: one parse at a time)."""

    def __init__(self, min_bytes: int = NATIVE_MIN_BYTES):
        self._lib = _cabi.load_library()
        self.min_bytes = int(min_bytes)
        names = "".join(ALL_FEATURES).encode()
        name_off = np.cumsum([0] + [len(n.encode()) for n in ALL_FEATURES]).astype(np.int32)
        dstr = [DEFAULTS[n].encode() for n in CATEGORICAL_FEATURES]
        dstr_off = np.cumsum([0] + [len(b) for b in dstr]).astype(np.int32)
        dnum = np.array([DEFAULTS[n] for n in NUMERIC_FEATURES], dtype=np.float64)
        self._h = self._lib.b2f_json_parser_create(len(CATEGORICAL_FEATURES), len(NUMERIC_FEATURES), names, _cabi.ptr(name_off), b"".join(dstr),
                                                   _cabi.ptr(dstr_off), _cabi.ptr(dnum))
        if not self._h:
            raise _cabi.B2FError("b2f_json_parser_create failed")
        self._lock = threading.Lock()
        self.fast = 0
        self.general = 0

    def close(self) -> None:
        if getattr(self, "_h", None):
            self._lib.b2f_json_parser_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def columns(self, raw: bytes):
        """-> (n_rows, {name: column}) for a body of the regular shape, or None (use the general validator)."""
        with self._lock:
            n = self._lib.b2f_json_parser_parse(self._h, raw, len(raw))
            if n < 0:
                return None
            cols = {}
            for j, name in enumerate(CATEGORICAL_FEATURES):
                nb = C.c_int64(0)
                dptr = self._lib.b2f_json_parser_str_data(self._h, j, C.byref(nb))
                off = np.ctypeslib.as_array(self._lib.b2f_json_parser_str_offsets(self._h, j), shape=(n + 1,)).copy()
                data = bytes(C.string_at(dptr, nb.value)) if nb.value else b""
                cols[name] = (off, data)
            for k, name in enumerate(NUMERIC_FEATURES):
                cols[name] = np.ctypeslib.as_array(self._lib.b2f_json_parser_numeric(self._h, k), shape=(n,)).copy() if n else np.zeros(0)
        return int(n), cols

    def frame(self, raw: bytes) -> pd.DataFrame:
        """Request body -> DataFrame with the 23 columns (0 rows for ``[]``); raises ``RequestValidationError`` (-> 422)
        exactly where ``list[LoanApplicant]`` validation would."""
        got = self.columns(raw) if (pa is not None and len(raw) >= self.min_bytes) else None
        if got is None:
            self.general += 1
            rows = parse_rows(raw)
            return rows_to_frame(rows) if rows else pd.DataFrame(columns=ALL_FEATURES)
        self.fast += 1
        n, cols = got
        out = {}
        for name in CATEGORICAL_FEATURES:
            off, data = cols[name]
            arr = pa.StringArray.from_buffers(n, pa.py_buffer(off), pa.py_buffer(data))
            out[name] = pd.array(arr, dtype="str")
        for name in NUMERIC_FEATURES:
            out[name] = cols[name]
        return pd.DataFrame(out, columns=ALL_FEATURES)
