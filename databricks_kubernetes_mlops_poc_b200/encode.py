"""Host-side row encoder: request columns -> 96-byte encoded rows (layout in ``include/b2f.h``).

This is the host half of the "fused preprocess": everything sklearn's ColumnTransformer does
that needs *strings* happens here, vectorised per column, straight into the (pinned) staging
buffer; everything arithmetic (median imputation, one-hot comparison, float32 compare) happens
in the kernel.

Reference behaviour being matched (``databricks/src/01-train-model.ipynb:195-221``):

* ``SimpleImputer(constant "missing")`` + ``OneHotEncoder(handle_unknown="ignore")``: a category
  string is looked up in the sorted training vocabulary; unknown strings and missing values get
  code -1 (== all-zero one-hot block) unless "missing" itself was a training category;
* numeric columns are cast float64 -> float32 exactly as sklearn's tree predict does; NaN stays
  NaN (the kernel imputes the median); +-inf or a value that overflows float32 raises the same
  ``ValueError`` sklearn raises;
* columns are selected by NAME (``df[self.all_features]``, ``02-register-model.ipynb:335``), so any
  column order works (the reference's ``inference.csv`` puts ``credit_limit`` first).
"""

from __future__ import annotations

import ctypes as C
import os

import numpy as np
import pandas as pd

try:  # Arrow's C++ hash lookup for the categorical columns; pandas fallback if absent
    import pyarrow as pa
    import pyarrow.compute as pc
except ImportError:  # pragma: no cover
    pa = pc = None

from .flatten import ROW_WORDS, FlatForest

PACKED_ROW_WORDS = 16  # B2F_ROWS_PACKED64: 64-byte rows (include/b2f.h)
NATIVE_THREADS = max(1, min(16, (os.cpu_count() or 1)))

_F32_MAX = float(np.finfo(np.float32).max)


def column_positions(df: pd.DataFrame, names, cache: dict):
    """Positions of ``names`` in ``df.columns`` (-1: absent), cached per column Index object (building an Index from a
    list of names costs more than a small request's whole device time)."""
    cols = df.columns
    hit = cache.get(id(cols))
    if hit is None or hit[0] is not cols:
        if len(cache) > 64:
            cache.clear()
        hit = cache[id(cols)] = (cols, [int(i) for i in cols.get_indexer(list(names))])
    return hit[1]


def arrow_string_columns(df: pd.DataFrame, names, positions=None):
    """The Arrow buffers behind the string columns ``names`` of ``df`` as a ``b2f_str_column`` array (what the native
    encoder reads in place) -> (array, keep-alive list), or None when a column is not Arrow-backed (object dtype ...)."""
    from . import _cabi

    if pa is None:
        return None
    scol = (_cabi.StrColumn * max(len(names), 1))()
    keep = []
    try:  # block-manager access: no Series per column
        idx = positions if positions is not None else df.columns.get_indexer(list(names))
        fetch = df._mgr.iget_values
        arrays = [fetch(int(i)) if i >= 0 else None for i in idx]
    except AttributeError:
        arrays = [df[name].array if name in df.columns else None for name in names]
    for j, arr in enumerate(arrays):
        if arr is None:
            raise KeyError(names[j])
        pa_arr = getattr(arr, "_pa_array", None)
        if pa_arr is None:
            return None
        if isinstance(pa_arr, pa.ChunkedArray):
            pa_arr = pa_arr.chunk(0) if pa_arr.num_chunks == 1 else pa_arr.combine_chunks()
        t = pa_arr.type
        large = pa.types.is_large_string(t)
        if not (large or pa.types.is_string(t)):
            return None
        validity, offsets, data = pa_arr.buffers()
        keep.append((arr, pa_arr, validity, offsets, data))
        c = scol[j]
        c.offsets = offsets.address
        c.data = data.address if data is not None else 0
        c.validity = validity.address if (validity is not None and pa_arr.null_count) else 0
        c.offset = pa_arr.offset
        c.data_bytes = data.size if data is not None else 0
        c.offsets_are_64 = 1 if large else 0
    return scol, keep


class RowEncoder:
    def __init__(self, flat: FlatForest):
        self.cat_features = list(flat.cat_features)
        self.num_features = list(flat.num_features)
        self.n_cat = len(self.cat_features)
        self.n_num = len(self.num_features)
        self._index = [pd.Index(list(v), dtype=object) for v in flat.categories]
        self._lut = [{c: i for i, c in enumerate(v)} for v in flat.categories]
        self._colpos = {}  # column-order tuple -> positions of the model's features
        self._colpos_fast = {}  # id(columns Index) -> (Index, positions): the block-manager path of frame_columns
        self._last_columns = None  # ((columns id, n, block ids), buffer descriptions) of the last frame frame_columns described
        self._pa_vocab = [pa.array(list(v), type=pa.string()) for v in flat.categories] if pa is not None else None
        self._missing = list(flat.missing_codes) if flat.missing_codes else [-1] * self.n_cat  # NaN -> imputer constant
        self._none = list(flat.none_codes) if flat.none_codes else [-1] * self.n_cat  # None -> None category, if any
        # packed 64-byte rows: nine 7-bit (code + 1) fields + 14 float32 numerics
        self.packed_ok = self.n_cat == 9 and self.n_num <= 14 and all(len(v) <= 126 for v in flat.categories)
        self._blob = flat.blob
        self._ranker = None  # b2f_ranker*: the forest's split-value tables (ranked rows), created on first use
        self._rank_info = None
        self._native = None  # b2f_encoder*, created on first use (needs libb200forest.so, not a GPU)
        self._native_failed = pa is None
        self._categories = [list(v) for v in flat.categories]

    # ------------------------------------------------------------------ native encoder (csrc/row_encoder.h)
    def _native_handle(self):
        if self._native is None and not self._native_failed:
            try:
                from . import _cabi

                lib = _cabi.load_library()
                blobs = [c.encode("utf-8") for v in self._categories for c in v]
                offsets = np.zeros(len(blobs) + 1, dtype=np.int64)
                np.cumsum([len(b) for b in blobs], out=offsets[1:])
                counts = np.array([len(v) for v in self._categories], dtype=np.int32)
                # a null entry: pandas' Arrow-backed strings cannot tell None from NaN; NaN semantics first
                nulls = np.array([m if m >= 0 else n for m, n in zip(self._missing, self._none)], dtype=np.int32)
                h = lib.b2f_encoder_create(self.n_cat, self.n_num, _cabi.ptr(counts), b"".join(blobs), _cabi.ptr(offsets), _cabi.ptr(nulls))
                if not h:
                    raise RuntimeError("b2f_encoder_create failed")
                self._native, self._lib, self._cabi = h, lib, _cabi
            except Exception:
                self._native_failed = True
        return self._native

    def __del__(self):
        try:
            if self._native:
                self._lib.b2f_encoder_destroy(self._native)
            if self._ranker:
                self._rk_lib.b2f_ranker_destroy(self._ranker)
        except Exception:
            pass

    # ------------------------------------------------------------------ ranked rows (csrc/forest_rank.h)
    def rank_info(self):
        """-> _cabi.RankInfo of this forest (``ok`` = 0 when it has no rank layout).  Needs the library, not a GPU."""
        if self._rank_info is None:
            from . import _cabi

            lib = _cabi.load_library()
            buf = np.frombuffer(self._blob, dtype=np.uint8)
            h = lib.b2f_ranker_create(_cabi.ptr(buf), buf.size)
            if not h:
                raise _cabi.B2FError(f"b2f_ranker_create failed: {_cabi.last_error()}")
            info = _cabi.RankInfo()
            _cabi.check(lib.b2f_ranker_info(h, C.byref(info)), "b2f_ranker_info")
            self._ranker, self._rk_lib, self._rank_info = h, lib, info
        return self._rank_info

    @property
    def ranked_ok(self) -> bool:
        return bool(self.rank_info().ok)

    @property
    def ranked_row_words(self) -> int:
        return self.rank_info().row_bytes // 4

    def rank_thresholds(self, k: int) -> np.ndarray:
        """Sorted distinct float32 split values of numeric feature k."""
        self.rank_info()
        cnt = C.c_int32(0)
        p = self._rk_lib.b2f_ranker_thresholds(self._ranker, k, C.byref(cnt))
        return np.ctypeslib.as_array(p, shape=(cnt.value,)).copy() if cnt.value else np.zeros(0, dtype=np.float32)

    def rank_layout(self) -> np.ndarray:
        """The forest's rank layout (bytes the GPU kernel walks): complete trees of 4-byte nodes + float64 payloads."""
        self.rank_info()
        nb = C.c_int64(0)
        p = self._rk_lib.b2f_ranker_layout(self._ranker, C.byref(nb))
        return np.frombuffer((C.c_uint8 * nb.value).from_address(p), dtype=np.uint8).copy() if nb.value else np.zeros(0, dtype=np.uint8)

    def rank_rows(self, rows: np.ndarray, out: np.ndarray | None = None, threads: int = NATIVE_THREADS) -> np.ndarray:
        """Encoded rows (N, 24) / packed (N, 16) -> ranked rows (N, row_bytes / 4) uint32."""
        from . import _cabi

        info = self.rank_info()
        if not info.ok:
            raise ValueError(f"this forest has no rank layout: {info.why.decode()}")
        rows = np.ascontiguousarray(rows)
        n = rows.shape[0]
        fmt = 1 if rows.shape[1] == PACKED_ROW_WORDS else 0
        if out is None:
            out = np.empty((n, info.row_bytes // 4), dtype=np.uint32)
        _cabi.check(self._rk_lib.b2f_ranker_rank_rows(self._ranker, _cabi.ptr(rows), n, fmt, _cabi.ptr(out), threads), "b2f_ranker_rank_rows")
        return out

    def encode_frame_ranked(self, df: pd.DataFrame, out: np.ndarray | None = None) -> np.ndarray:
        """DataFrame -> ranked rows in one native pass (large frames) or via the 96-byte rows (small / irregular ones)."""
        n = len(df)
        words = self.ranked_row_words
        if out is None:
            out = np.empty((n, words), dtype=np.uint32)
        if n > self.SMALL_BATCH:
            missing = [c for c in self.cat_features + self.num_features if c not in df.columns]
            if missing:
                raise KeyError(f"{missing} not in index")
            if self._encode_native(df, out, fmt=2):
                return out
        return self.rank_rows(self.encode_frame(df), out=out)

    def frame_columns(self, df: pd.DataFrame):
        """The physical buffers behind the model's 23 columns of ``df``, as the native encoder / scorer take them:
        -> (StrColumn array, float64 pointer array, strides, keep-alive list), or None when a column does not have the
        expected physical type (object-dtype strings, non-numeric numerics ...: the portable path handles those).
        Column lookup goes through the block manager (one ``get_indexer`` per distinct column index, then an array fetch per
        column) -- ``df[name]`` builds a Series per column, which for 23 columns costs more than encoding a small request."""
        if self._native_handle() is None:
            return None
        cols = df.columns
        key = id(cols)
        pos = self._colpos_fast.get(key)
        if pos is None or pos[0] is not cols:
            idx = cols.get_indexer(self.cat_features + self.num_features)
            if (idx < 0).any():
                missing = [c for c, i in zip(self.cat_features + self.num_features, idx) if i < 0]
                raise KeyError(f"{missing} not in index")  # what df[self.all_features] raises
            if len(self._colpos_fast) > 64:
                self._colpos_fast.clear()
            pos = self._colpos_fast[key] = (cols, [int(i) for i in idx])
        pos = pos[1]
        try:
            fetch = df._mgr.iget_values
        except AttributeError:  # pandas without this internal: public (slower) access
            def fetch(i, _df=df):
                return _df.iloc[:, i].array
        n = len(df)
        # the same BLOCKS as last time (a service scoring one frame again, a benchmark loop): the buffer descriptions are still
        # valid -- Arrow string arrays are immutable, and a float64 block written in place is read in place.  The block value
        # objects are kept alive with the descriptions, so their ids cannot be recycled for other arrays.
        try:
            blocks = [b.values for b in df._mgr.blocks]
        except AttributeError:
            blocks = None
        ids = (key, n, tuple(map(id, blocks))) if blocks is not None else None
        last = self._last_columns
        if ids is not None and last is not None and last[0] == ids:
            return last[1]
        scol = (self._cabi.StrColumn * max(self.n_cat, 1))()
        keep = [blocks]
        for j in range(self.n_cat):
            arr = fetch(pos[j])
            pa_arr = getattr(arr, "_pa_array", None)
            if pa_arr is None:
                return None  # object-dtype strings (None and NaN are different things there) -> portable path
            if isinstance(pa_arr, pa.ChunkedArray):
                pa_arr = pa_arr.chunk(0) if pa_arr.num_chunks == 1 else pa_arr.combine_chunks()
            t = pa_arr.type
            large = pa.types.is_large_string(t)
            if not (large or pa.types.is_string(t)):
                return None
            validity, offsets, data = pa_arr.buffers()
            keep.append((pa_arr, validity, offsets, data))
            c = scol[j]
            c.offsets = offsets.address
            c.data = data.address if data is not None else 0
            c.validity = validity.address if (validity is not None and pa_arr.null_count) else 0
            c.offset = pa_arr.offset
            c.data_bytes = data.size if data is not None else 0
            c.offsets_are_64 = 1 if large else 0
        ptrs = (C.c_void_p * max(self.n_num, 1))()
        strides = np.ones(max(self.n_num, 1), dtype=np.int64)
        for k in range(self.n_num):
            col = fetch(pos[self.n_cat + k])
            if not isinstance(col, np.ndarray):
                col = np.asarray(col)
            if col.dtype != np.float64:
                if col.dtype.kind not in "iuf":
                    return None
                col = col.astype(np.float64)
            keep.append(col)
            ptrs[k] = col.ctypes.data
            strides[k] = col.strides[0] // 8 if n > 1 else 1
        keep.append(strides)
        self._last_columns = (ids, (scol, ptrs, strides, keep)) if ids is not None else None
        return scol, ptrs, strides, keep

    def _encode_native(self, df: pd.DataFrame, out: np.ndarray, packed: bool = False, fmt: int | None = None) -> bool:
        """Columnar fast path: Arrow string buffers + float64 columns -> rows, in C++ threads.  Returns False when
        a column does not have the expected physical type (the caller then takes the portable path)."""
        h = self._native_handle()
        if h is None:
            return False
        if fmt is None:
            fmt = 1 if packed else 0
        if fmt == 2 and not getattr(self, "_ranker_attached", False):
            if not self.rank_info().ok or self._lib.b2f_encoder_attach_ranker(h, self._ranker) != 0:
                return False
            self._ranker_attached = True
        n = len(df)
        cols = (self._cabi.StrColumn * max(self.n_cat, 1))()
        keep = []  # keep the Arrow arrays alive during the call
        for j, name in enumerate(self.cat_features):
            ser = df[name]
            if ser.dtype == object:
                # object columns can hold None and NaN side by side, which the library treats differently
                # (None is not imputed); Arrow would merge them into one null -> portable path
                return False
            try:
                arr = pa.array(ser, from_pandas=True)
            except (pa.ArrowInvalid, pa.ArrowTypeError, pa.ArrowNotImplementedError):
                return False
            if isinstance(arr, pa.ChunkedArray):
                arr = arr.combine_chunks()
            if pa.types.is_dictionary(arr.type):
                arr = arr.dictionary_decode()
            if not (pa.types.is_string(arr.type) or pa.types.is_large_string(arr.type)):
                return False
            validity, offsets, data = arr.buffers()
            keep.append((arr, validity, offsets, data))
            cols[j].offsets = offsets.address
            cols[j].data = data.address if data is not None else 0
            cols[j].validity = validity.address if (validity is not None and arr.null_count) else 0
            cols[j].offset = arr.offset
            cols[j].data_bytes = data.size if data is not None else 0
            cols[j].offsets_are_64 = 1 if pa.types.is_large_string(arr.type) else 0
        ptrs = (C.c_void_p * max(self.n_num, 1))()
        strides = np.ones(max(self.n_num, 1), dtype=np.int64)
        for k, name in enumerate(self.num_features):
            col = df[name].to_numpy()
            if col.dtype != np.float64:
                if col.dtype.kind not in "iuf":
                    return False
                col = col.astype(np.float64)
            keep.append(col)
            ptrs[k] = col.ctypes.data
            strides[k] = col.strides[0] // 8 if n > 1 else 1
        rc = self._lib.b2f_encoder_encode(h, n, cols, ptrs, self._cabi.ptr(strides), fmt, self._cabi.ptr(out), NATIVE_THREADS)
        if rc == -7:
            raise ValueError("Input X contains infinity or a value too large for dtype('float32').")
        if rc != 0:
            raise RuntimeError(f"b2f_encoder_encode failed (rc={rc})")
        return True

    # ------------------------------------------------------------------ columns
    def encode_categorical(self, j: int, values) -> np.ndarray:
        """One categorical column (any array-like of str / None) -> int32 codes, -1 = unknown.
        Arrow's ``index_in`` does the vocabulary lookup in C++ (zero-copy for pandas' Arrow-backed
        string columns); non-string columns fall back to a pandas hash lookup."""
        if pa is not None:
            try:
                arr = pa.array(values, from_pandas=True)
                if pa.types.is_dictionary(arr.type):
                    arr = arr.dictionary_decode()
                if pa.types.is_string(arr.type) or pa.types.is_large_string(arr.type):
                    idx = pc.index_in(arr, value_set=self._pa_vocab[j].cast(arr.type))
                    codes = idx.fill_null(-1).to_numpy(zero_copy_only=False).astype(np.int32)
                    if arr.null_count and (self._missing[j] >= 0 or self._none[j] >= 0):
                        codes[arr.is_null().to_numpy(zero_copy_only=False)] = self._null_codes(j, values)
                    return codes
            except (pa.ArrowInvalid, pa.ArrowTypeError, pa.ArrowNotImplementedError):
                pass
        arr = values if isinstance(values, (pd.Series, np.ndarray)) else np.asarray(values, dtype=object)
        codes = self._index[j].get_indexer(pd.Index(arr, dtype=object)).astype(np.int32)  # -1 = not in vocabulary
        if self._missing[j] >= 0 or self._none[j] >= 0:
            isna = np.asarray(pd.isna(arr))
            if isna.any():
                codes[isna] = self._null_codes(j, arr)
        return codes

    def _null_codes(self, j: int, values) -> np.ndarray:
        """Codes for the null entries of a column: None -> the None category (if fit saw one), NaN -> the
        imputer's constant category (if fit saw missing values); Arrow-backed columns only have one kind of null."""
        obj = np.asarray(values, dtype=object)
        nulls = obj[np.asarray(pd.isna(obj))]
        is_none = np.fromiter((v is None for v in nulls), dtype=bool, count=len(nulls))
        return np.where(is_none, self._none[j], self._missing[j]).astype(np.int32)

    @staticmethod
    def cast_numeric(block64: np.ndarray) -> np.ndarray:
        """float64 (N, k) -> float32 with sklearn's finiteness rule (NaN allowed: missing)."""
        bad = np.abs(block64) > _F32_MAX  # False for NaN
        if bad.any():
            raise ValueError("Input X contains infinity or a value too large for dtype('float32').")
        return block64.astype(np.float32)

    # ------------------------------------------------------------------ frames
    SMALL_BATCH = 128  # below this, per-column vectorised machinery costs more than a Python loop

    def encode_frame(self, df: pd.DataFrame, out: np.ndarray | None = None) -> np.ndarray:
        """DataFrame with (at least) the 23 named columns -> uint32 (N, 24) encoded rows."""
        n = len(df)
        if out is None:
            out = np.empty((n, ROW_WORDS), dtype=np.uint32)
        else:
            assert out.shape == (n, ROW_WORDS) and out.dtype == np.uint32
        cols = df.columns
        missing = [c for c in self.cat_features + self.num_features if c not in cols]
        if missing:
            raise KeyError(f"{missing} not in index")  # what df[self.all_features] raises
        as_i32 = out.view(np.int32)
        if n <= self.SMALL_BATCH:
            # small request: ONE object-array extraction of the whole frame (pandas column selection alone costs
            # more than the rest of a small request), then dictionary lookups / float() in Python
            key = tuple(cols)
            pos = self._colpos.get(key)
            if pos is None:
                pos = self._colpos[key] = [cols.get_loc(c) for c in self.cat_features + self.num_features]
            recs = df.to_numpy(dtype=object)
            nums = np.empty((n, self.n_num), dtype=np.float64)
            for i in range(n):
                rec = recs[i]
                for j in range(self.n_cat):
                    v = rec[pos[j]]
                    as_i32[i, j] = self._lut[j].get(v, -1) if isinstance(v, str) else (self._none[j] if v is None else (self._missing[j] if v != v else -1))
                for k in range(self.n_num):
                    v = rec[pos[self.n_cat + k]]
                    nums[i, k] = np.nan if v is None else float(v)  # float("abc") raises ValueError, as pd.to_numeric does
            if self.n_num:
                out.view(np.float32)[:, self.n_cat : self.n_cat + self.n_num] = self.cast_numeric(nums)
        elif self._encode_native(df, out, packed=False):
            return out
        else:
            for j, name in enumerate(self.cat_features):
                as_i32[:, j] = self.encode_categorical(j, df[name])
            if self.n_num:
                try:
                    block = df[self.num_features].to_numpy(dtype=np.float64, na_value=np.nan)
                except (ValueError, TypeError):
                    block = np.empty((n, self.n_num), dtype=np.float64)
                    for k, name in enumerate(self.num_features):
                        block[:, k] = pd.to_numeric(df[name], errors="raise").to_numpy(dtype=np.float64, na_value=np.nan)
                out.view(np.float32)[:, self.n_cat : self.n_cat + self.n_num] = self.cast_numeric(block)
        out[:, self.n_cat + self.n_num :] = 0
        return out

    def encode_arrays(self, codes: np.ndarray, nums: np.ndarray, out: np.ndarray | None = None) -> np.ndarray:
        """Already-dictionary-encoded input (int codes (N, n_cat), float nums (N, n_num)) -> rows."""
        n = codes.shape[0]
        if out is None:
            out = np.empty((n, ROW_WORDS), dtype=np.uint32)
        out.view(np.int32)[:, : self.n_cat] = codes
        out.view(np.float32)[:, self.n_cat : self.n_cat + self.n_num] = self.cast_numeric(
            np.asarray(nums, dtype=np.float64)
        )
        out[:, self.n_cat + self.n_num :] = 0
        return out

    # ------------------------------------------------------------------ packed 64-byte rows
    def pack_rows(self, rows24: np.ndarray, out: np.ndarray | None = None) -> np.ndarray:
        """(N, 24) encoded rows -> (N, 16) packed rows (B2F_ROWS_PACKED64): one third fewer bytes over PCIe.
        Lossless: code + 1 in 7 bits (0 = unknown), numerics untouched."""
        if not self.packed_ok:
            raise ValueError("schema does not fit the packed row (exactly 9 categoricals of <= 126 categories, <= 14 numerics)")
        n = rows24.shape[0]
        if out is None:
            out = np.zeros((n, PACKED_ROW_WORDS), dtype=np.uint32)
        fields = (rows24.view(np.int32)[:, : self.n_cat].astype(np.int64) + 1).astype(np.uint64)
        word = np.zeros(n, dtype=np.uint64)
        for j in range(self.n_cat):
            word |= fields[:, j] << np.uint64(7 * j)
        out[:, 0] = (word & np.uint64(0xFFFFFFFF)).astype(np.uint32)
        out[:, 1] = (word >> np.uint64(32)).astype(np.uint32)
        out[:, 2 : 2 + self.n_num] = rows24[:, self.n_cat : self.n_cat + self.n_num]
        out[:, 2 + self.n_num :] = 0
        return out

    def encode_frame_packed(self, df: pd.DataFrame, out: np.ndarray | None = None) -> np.ndarray:
        """DataFrame -> (N, 16) packed rows; large frames go through the native encoder in one pass."""
        n = len(df)
        if n > self.SMALL_BATCH and self.packed_ok:
            missing = [c for c in self.cat_features + self.num_features if c not in df.columns]
            if missing:
                raise KeyError(f"{missing} not in index")
            if out is None:
                out = np.empty((n, PACKED_ROW_WORDS), dtype=np.uint32)
            if self._encode_native(df, out, packed=True):
                return out
        return self.pack_rows(self.encode_frame(df), out=out)

    def encode_arrays_packed(self, codes: np.ndarray, nums: np.ndarray, out: np.ndarray | None = None) -> np.ndarray:
        return self.pack_rows(self.encode_arrays(codes, nums), out=out)
