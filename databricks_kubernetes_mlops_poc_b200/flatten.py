"""Fitted sklearn Pipeline -> forest blob (the layout in ``csrc/forest_blob.h``).

The reference serves ``artifacts/classifier/model/model.pkl`` -- a pickled sklearn
``Pipeline(ColumnTransformer -> RandomForestClassifier)`` (definition: reference
``databricks/src/01-train-model.ipynb:195-231``; loaded at
``02-register-model.ipynb:317-321``).  This module turns such a fitted object into
the flat, versioned binary the GPU engine consumes; it is the only place that knows
sklearn's attribute names.  It does arithmetic-free bookkeeping only:

* one-hot column ``j`` of the ColumnTransformer output is rewritten as
  ``(categorical row word f, category code c)``: the split ``x_j <= 0.5`` becomes
  "second child iff code[f] == c"  (unknown / missing category = code -1 = all-zero
  one-hot block = always first child, which is ``handle_unknown="ignore"``,
  ``01-train-model.ipynb:203-206``);
* float64 thresholds become the float32 ``t' = nextup(floor32(t64))``: for float32 ``x``,
  ``x <= t64  <=>  x <= max{f32 <= t64}  <=>  x < t'`` (sklearn compares float32 X with
  float64 thresholds, ``sklearn/tree/_tree.pyx`` ``_apply_dense``), so the kernel's test is
  "second child iff ``x >= t'``";
* leaf payloads stay float64: RF class-1 fraction, or ``learning_rate * value`` for GBDT
  (the product sklearn's ``predict_stages`` forms before adding);
* nodes are re-numbered breadth-first so siblings are adjacent, leaves become
  self-looping slots, and 32 trees are interleaved per group (see ``forest_blob.h``).
"""

from __future__ import annotations

import json
import struct
from dataclasses import dataclass, field

import numpy as np

ROW_WORDS = 24
SENTINEL_WORD = 23
SENTINEL_BITS = 0xFFFFFFFF
META_CAT = 0x04000000
META_SLOT_MASK = 0x00FFFFFF
META_FEAT_SHIFT = 27
NODE_STRIDE = 256
GROUP_TREES = 32
MAX_TREES = 1024
HEADER_BYTES = 512
AGG_RF_MEAN = 0
AGG_GBDT_LOGISTIC = 1
AGG_IFOREST = 2
BLOB_VERSION = 2

_HEADER_FMT = "<8s" + "I" * 10 + "dd" + "Q" * 4 + "24f" + "24i" + "dd"  # 304 bytes, padded to 512
HEADER_HAS_PATH_BOUND = 1  # header flags bit: ``path_bound`` holds the isolation forest's decision bound
_GROUP_FMT = "<8I"


@dataclass
class FlatForest:
    """A forest blob plus the host-side vocabulary needed to encode rows for it."""

    blob: bytes
    cat_features: list
    num_features: list
    categories: list  # per categorical feature: list[str], sorted as OneHotEncoder.categories_
    classes: list  # class labels in sklearn order, e.g. [0, 1]
    agg_mode: int
    n_trees: int
    max_depth: int
    total_nodes: int
    missing_codes: list = field(default_factory=list)  # per cat feature: code NaN maps to (the imputer's "missing") or -1
    none_codes: list = field(default_factory=list)  # per cat feature: code None maps to (a None category seen at fit) or -1

    @property
    def all_features(self):
        return list(self.cat_features) + list(self.num_features)

    def save(self, path: str) -> None:
        meta = dict(
            cat_features=self.cat_features,
            num_features=self.num_features,
            categories=self.categories,
            classes=self.classes,
            agg_mode=self.agg_mode,
            n_trees=self.n_trees,
            max_depth=self.max_depth,
            total_nodes=self.total_nodes,
            missing_codes=self.missing_codes,
            none_codes=self.none_codes,
        )
        np.savez_compressed(path, blob=np.frombuffer(self.blob, dtype=np.uint8), meta=np.array(json.dumps(meta)))

    @staticmethod
    def load(path: str) -> "FlatForest":
        with np.load(path) as z:
            meta = json.loads(str(z["meta"]))
            return FlatForest(blob=z["blob"].tobytes(), **meta)


def floor_to_f32(t64: np.ndarray) -> np.ndarray:
    """Largest float32 <= t64 (elementwise); +-inf pass through."""
    t64 = np.asarray(t64, dtype=np.float64)
    with np.errstate(over="ignore"):
        t32 = t64.astype(np.float32)
    too_big = t32.astype(np.float64) > t64
    t32[too_big] = np.nextafter(t32[too_big], np.float32(-np.inf))
    return t32


def _bfs_slots(left: np.ndarray, right: np.ndarray):
    """Breadth-first renumbering with adjacent siblings.  Returns (slot_of_node, depth)."""
    n = left.shape[0]
    slot = np.full(n, -1, dtype=np.int64)
    slot[0] = 0
    nxt = 1
    level = np.array([0], dtype=np.int64)
    depth = 0
    while True:
        internal = level[left[level] != -1]
        if internal.size == 0:
            break
        first = nxt + 2 * np.arange(internal.size, dtype=np.int64)
        slot[left[internal]] = first
        slot[right[internal]] = first + 1
        nxt += 2 * internal.size
        level = np.empty(2 * internal.size, dtype=np.int64)
        level[0::2] = left[internal]
        level[1::2] = right[internal]
        depth += 1
    assert nxt == n and (slot >= 0).all(), "tree has unreachable nodes"
    return slot, depth


def strict_upper_f32(t64: np.ndarray) -> np.ndarray:
    """t' = nextup(floor32(t64)): the float32 with  x <= t64  <=>  x < t'  for every finite float32 x."""
    return np.nextafter(floor_to_f32(t64), np.float32(np.inf))


def _flatten_tree(tree, col_word, col_cat_code, col_is_cat, leaf_value):
    """One sklearn ``Tree`` -> (T uint32[n], M uint32[n], LV float64[n_leaves], depth), slot-indexed."""
    left = tree.children_left.astype(np.int64)
    right = tree.children_right.astype(np.int64)
    n = left.shape[0]
    if n >= (1 << 24):
        raise NotImplementedError("tree too large for 24-bit slot offsets")
    slot, depth = _bfs_slots(left, right)
    T = np.zeros(n, dtype=np.uint32)
    M = np.zeros(n, dtype=np.uint32)
    is_leaf = left == -1
    internal = np.nonzero(~is_leaf)[0]
    leaves = np.nonzero(is_leaf)[0]

    # leaves: numbered in slot order; T = row of the leaf's payload in LV, M = self-loop
    leaf_order = leaves[np.argsort(slot[leaves])]
    leaf_id = np.arange(leaf_order.size, dtype=np.uint32)
    ls = slot[leaf_order]
    T[ls] = leaf_id
    M[ls] = ls.astype(np.uint32) | np.uint32(META_CAT) | np.uint32(SENTINEL_WORD << META_FEAT_SHIFT)
    LV = leaf_value[leaf_order].astype(np.float64)

    if internal.size:
        col = tree.feature[internal].astype(np.int64)
        thr = tree.threshold[internal].astype(np.float64)
        s = slot[internal]
        first = slot[left[internal]].astype(np.uint32)
        word = col_word[col].astype(np.uint32) << np.uint32(META_FEAT_SHIFT)
        cat = col_is_cat[col]
        t_words = strict_upper_f32(thr).view(np.uint32).copy()
        m_words = first | word
        if cat.any():
            # one-hot column x in {0, 1}:  x <= thr ?  x=0 -> (0 <= thr), x=1 -> (1 <= thr)
            zero_left = 0.0 <= thr
            one_left = 1.0 <= thr
            normal = cat & zero_left & ~one_left  # the only case sklearn produces (thr = 0.5)
            always_left = cat & zero_left & one_left
            always_right = cat & ~zero_left
            t_words[normal] = col_cat_code[col[normal]].astype(np.uint32)
            m_words[normal] |= np.uint32(META_CAT)
            t_words[always_left] = np.uint32(0x7FFFFFFF)  # never equals a category code
            m_words[always_left] |= np.uint32(META_CAT)
            # always second child: numeric test on the sentinel word (NaN bits): geu(NaN, t) is true
            t_words[always_right] = np.uint32(0)
            m_words[always_right] = first[always_right] | np.uint32(SENTINEL_WORD << META_FEAT_SHIFT)
        T[s] = t_words
        M[s] = m_words
    return T, M, LV, depth


def _assemble_blob(flat, agg, init_raw, denom, n_cat, n_num, impute, vocab, threshold=0.0, path_bound=None):
    """Flattened trees ``[(T, M, LV, depth), ...]`` -> (blob bytes, max depth): groups of 32 interleaved trees."""
    n_trees = len(flat)
    if not (1 <= n_trees <= MAX_TREES):
        raise NotImplementedError(f"n_trees={n_trees} outside [1, {MAX_TREES}]")
    n_groups = (n_trees + GROUP_TREES - 1) // GROUP_TREES
    groups, chunks, off = [], [], 0
    for g in range(n_groups):
        members = flat[g * GROUP_TREES : (g + 1) * GROUP_TREES]
        n_slots = max(len(m[0]) for m in members)
        n_leaf = max(len(m[2]) for m in members)
        depth = max(m[3] for m in members)
        N = np.empty((n_slots, GROUP_TREES, 2), dtype=np.uint32)  # [slot][tree] -> (T, M)
        LV = np.zeros((n_leaf, GROUP_TREES), dtype=np.float64)
        # unused slots / stub trees: self-looping leaf with payload row 0 (value 0.0 for stubs)
        N[:, :, 0] = 0
        N[:, :, 1] = np.arange(n_slots, dtype=np.uint32)[:, None] | np.uint32(META_CAT | (SENTINEL_WORD << META_FEAT_SHIFT))
        for lane, (t, m, lv, _) in enumerate(members):
            N[: len(t), lane, 0] = t
            N[: len(m), lane, 1] = m
            LV[: len(lv), lane] = lv
        chunk = N.tobytes() + LV.tobytes()
        assert len(chunk) == (n_slots + n_leaf) * 256
        groups.append((off, len(chunk), n_slots, n_leaf, depth, len(members), 0, 0))
        chunks.append(chunk)
        off += len(chunk)

    max_depth = max(m[3] for m in flat)
    groups_off = HEADER_BYTES
    chunks_off = (groups_off + 32 * n_groups + 255) // 256 * 256
    total = chunks_off + off
    header = struct.pack(
        _HEADER_FMT,
        b"B2FOREST",
        BLOB_VERSION,
        HEADER_BYTES,
        agg,
        n_trees,
        n_groups,
        ROW_WORDS,
        n_cat,
        n_num,
        max_depth,
        0 if path_bound is None else HEADER_HAS_PATH_BOUND,
        init_raw,
        denom,
        groups_off,
        chunks_off,
        off,
        total,
        *np.asarray(impute, dtype=np.float32).tolist(),
        *np.asarray(vocab, dtype=np.int32).tolist(),
        float(threshold),
        0.0 if path_bound is None else float(path_bound),
    )
    header = header + b"\0" * (HEADER_BYTES - len(header))
    table = b"".join(struct.pack(_GROUP_FMT, *g) for g in groups)
    pad = b"\0" * (chunks_off - groups_off - len(table))
    blob = header + table + pad + b"".join(chunks)
    assert len(blob) == total
    return blob, int(max_depth)


def _average_path_length(n):
    """c(n): average path length of an unsuccessful BST search over n points (Liu et al. 2008, eq. 1), with
    sklearn's conventions c(<=1) = 0, c(2) = 1 (``sklearn/ensemble/_iforest.py`` ``_average_path_length``)."""
    n = np.asarray(n, dtype=np.float64)
    out = np.zeros(n.shape, dtype=np.float64)
    out[n == 2] = 1.0
    big = n > 2
    out[big] = 2.0 * (np.log(n[big] - 1.0) + np.euler_gamma) - 2.0 * (n[big] - 1.0) / n[big]
    return out


def iforest_path_bound(offset: float, denom: float, threshold: float) -> float:
    """The largest path-length sum ``s >= 0`` that sklearn flags: ``-decision_function = -((-(2 ** (-s / denom))) - offset)
    > threshold``, evaluated with numpy exactly as ``IsolationForest`` does.  The score falls as ``s`` grows, so the kernels
    decide ``s <= bound`` on the path-length sum instead of comparing a score rounded by other arithmetic (CUDA's exp2)
    with the threshold.  -inf: no sum is flagged; +inf: every sum is."""

    def flagged(bits: int) -> bool:
        s = np.array([bits], dtype=np.int64).view(np.float64)
        scores = 2 ** (-np.divide(s, denom))
        return bool(-(-scores - offset)[0] > threshold)

    inf_bits = int(np.array([np.inf]).view(np.int64)[0])
    if not flagged(0):
        return -np.inf
    if flagged(inf_bits):
        return np.inf
    lo, hi = 0, inf_bits  # flagged(lo), not flagged(hi): non-negative doubles are ordered as their bit patterns
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if flagged(mid) else (lo, mid)
    return float(np.array([lo], dtype=np.int64).view(np.float64)[0])


def flatten_isolation_forest(detector, n_cat: int, n_num: int, vocab=None, threshold: float | None = None) -> bytes:
    """Fitted outlier detector -> forest blob with ``agg_mode = AGG_IFOREST`` over the classifier's encoded rows.

    ``detector`` is a fitted ``sklearn.ensemble.IsolationForest`` or an object carrying one as
    ``.isolationforest`` plus ``.threshold`` (alibi-detect's ``IForest``; the reference builds
    ``IForest(threshold=0.95).fit(df[NUMERIC_FEATURES].values)``, ``02-register-model.ipynb:232-233``, and calls
    ``.predict(df[numeric_features].values)`` per request, ``:339,344``).  Feature k of the detector is numeric
    feature k of the request, i.e. row word ``n_cat + k``.  What the GPU reproduces:

    * ``score = -decision_function(X) = 2 ** (-sum_t h_t(x) / (n_trees * c(max_samples))) + offset_`` with
      ``h_t(x) = (depth(leaf) + 1) + c(n_node_samples[leaf]) - 1.0``, sklearn's per-tree term to the last bit
      (``_iforest.py`` ``_compute_score_samples``);
    * ``is_outlier = score > threshold``, decided as ``sum_t h_t(x) <= iforest_path_bound(...)``; a row near the bound is
      summed again in tree order, as sklearn sums it (``csrc/forest_decide.cuh``), so the flag is sklearn's.

    Splits compare float32 inputs with float64 thresholds exactly as the classifier's trees do.  NaN inputs are
    outside the contract: the reference's pinned scikit-learn 1.1.1 (``app/requirements.txt:14``) rejects them in
    ``IsolationForest.decision_function`` (ValueError -> HTTP 500) and ``B200Model`` does the same; newer sklearn
    routes them by a per-node random ``missing_go_to_left`` flag that the 8-byte node does not carry (on the GPU a
    NaN takes the second child at every split: the imputation table of this blob holds NaN).
    """
    iso = getattr(detector, "isolationforest", detector)
    if type(iso).__name__ != "IsolationForest":
        raise NotImplementedError(f"unsupported outlier detector {type(iso).__name__}")
    if threshold is None:
        threshold = getattr(detector, "threshold", None)
    if threshold is None:
        raise ValueError("an outlier threshold is required (alibi-detect IForest(threshold=...))")
    if iso.n_features_in_ != n_num:
        raise NotImplementedError(f"detector was fitted on {iso.n_features_in_} features, the request schema has {n_num} numerics")
    if n_cat + n_num > SENTINEL_WORD:
        raise NotImplementedError(f"at most {SENTINEL_WORD} raw features supported")
    flat = []
    for est, feats in zip(iso.estimators_, iso.estimators_features_):
        tree = est.tree_
        feats = np.asarray(feats, dtype=np.int64)
        col_word = n_cat + feats  # the tree's local column j is detector feature feats[j]
        none = np.zeros(col_word.shape[0], dtype=bool)
        # h(leaf) = number of edges from the root + c(training points that ended in the leaf)
        left, right = tree.children_left, tree.children_right
        depth = np.zeros(tree.node_count, dtype=np.float64)
        for i in range(tree.node_count):  # sklearn stores parents before children
            if left[i] != -1:
                depth[left[i]] = depth[right[i]] = depth[i] + 1.0
        payload = (depth.astype(np.int64) + 1) + _average_path_length(tree.n_node_samples) - 1.0
        flat.append(_flatten_tree(tree, col_word, np.zeros_like(col_word), none, payload))
    denom = float(len(flat)) * float(_average_path_length(np.array([iso._max_samples]))[0])
    if not denom > 0.0:
        raise NotImplementedError("isolation forest fitted on a single sample")
    impute = np.zeros(ROW_WORDS, dtype=np.float32)
    impute[n_cat : n_cat + n_num] = np.nan
    v = np.zeros(ROW_WORDS, dtype=np.int32)
    if vocab is not None:
        v[:n_cat] = np.asarray(vocab, dtype=np.int32)[:n_cat]
    bound = iforest_path_bound(float(iso.offset_), denom, float(threshold))
    blob, _ = _assemble_blob(flat, AGG_IFOREST, float(iso.offset_), denom, n_cat, n_num, impute, v, threshold=float(threshold),
                             path_bound=bound)
    return blob


def _describe_preprocessor(pre):
    """ColumnTransformer of the reference shape -> column maps for its output matrix."""
    cat_cols, num_cols, ohe, num_imputer, cat_imputer = None, None, None, None, None
    for name, trans, cols in pre.transformers_:
        if trans == "drop" or (isinstance(trans, str) and trans == "passthrough"):
            continue
        steps = dict(trans.named_steps) if hasattr(trans, "named_steps") else {"only": trans}
        kinds = {type(s).__name__ for s in steps.values()}
        if "OneHotEncoder" in kinds:
            cat_cols = list(cols)
            ohe = next(s for s in steps.values() if type(s).__name__ == "OneHotEncoder")
            cat_imputer = next((s for s in steps.values() if type(s).__name__ == "SimpleImputer"), None)
            cat_name = name
        else:
            num_cols = list(cols)
            num_imputer = next((s for s in steps.values() if type(s).__name__ == "SimpleImputer"), None)
            num_name = name
    if ohe is None or num_cols is None or num_imputer is None:
        raise NotImplementedError("expected ColumnTransformer([categorical: imputer+OneHotEncoder, numeric: imputer])")
    if ohe.handle_unknown != "ignore" or getattr(ohe, "drop", None) is not None:
        raise NotImplementedError("OneHotEncoder must use handle_unknown='ignore' and drop=None")
    if len(cat_cols) + len(num_cols) > SENTINEL_WORD:
        raise NotImplementedError(f"at most {SENTINEL_WORD} raw features supported")
    # a training column that held None / NaN gives OneHotEncoder a non-string category (sorted last); keep its
    # position under a placeholder no request string can equal, and remember it for the encoder
    NONE_TOKEN = "\x00<none>"
    categories = [[c if isinstance(c, str) else NONE_TOKEN for c in cats] for cats in ohe.categories_]
    n_cat, n_num = len(cat_cols), len(num_cols)
    cat_slice = pre.output_indices_[cat_name]
    num_slice = pre.output_indices_[num_name]
    n_out = max(cat_slice.stop, num_slice.stop)
    col_word = np.zeros(n_out, dtype=np.int64)
    col_code = np.zeros(n_out, dtype=np.int64)
    col_is_cat = np.zeros(n_out, dtype=bool)
    j = cat_slice.start
    for f, cats in enumerate(categories):
        for c in range(len(cats)):
            col_word[j], col_code[j], col_is_cat[j] = f, c, True
            j += 1
    assert j == cat_slice.stop
    for k in range(n_num):
        col_word[num_slice.start + k] = n_cat + k
    medians = np.asarray(num_imputer.statistics_, dtype=np.float64)
    fill = getattr(cat_imputer, "fill_value", None) if cat_imputer is not None else None
    # NaN is imputed to the constant `fill` ("missing") before encoding; None is left alone by SimpleImputer and
    # only matches a None category seen at fit time
    missing_codes = [cats.index(fill) if (fill is not None and fill in cats) else -1 for cats in categories]
    none_codes = [cats.index(NONE_TOKEN) if NONE_TOKEN in cats else -1 for cats in categories]
    return cat_cols, num_cols, categories, medians, col_word, col_code, col_is_cat, missing_codes, none_codes


def flatten_pipeline(pipeline) -> FlatForest:
    """Fitted reference-style Pipeline -> FlatForest."""
    pre = pipeline.named_steps["preprocessor"]
    clf = pipeline.named_steps["classifier"]
    cat_cols, num_cols, categories, medians, col_word, col_code, col_is_cat, missing_codes, none_codes = _describe_preprocessor(pre)
    n_cat, n_num = len(cat_cols), len(num_cols)

    kind = type(clf).__name__
    if kind == "RandomForestClassifier":
        if len(clf.classes_) != 2 or clf.n_outputs_ != 1:
            raise NotImplementedError("binary single-output RandomForestClassifier only")
        agg = AGG_RF_MEAN
        trees = [e.tree_ for e in clf.estimators_]
        init_raw, denom = 0.0, float(len(trees))

        def leaf_values(t):
            v = t.value[:, 0, :]
            s = v.sum(axis=1)
            s = np.where(s == 0.0, 1.0, s)
            return v[:, 1] / s  # class-1 fraction (normalised for sklearn < 1.4 weighted counts)

    elif kind == "GradientBoostingClassifier":
        if len(clf.classes_) != 2:
            raise NotImplementedError("binary GradientBoostingClassifier only")
        agg = AGG_GBDT_LOGISTIC
        trees = [e.tree_ for e in clf.estimators_[:, 0]]
        if isinstance(clf.init_, str) and clf.init_ == "zero":
            init_raw = 0.0
        elif type(clf.init_).__name__ == "DummyClassifier":
            eps = np.finfo(np.float64).eps
            p1 = float(np.clip(clf.init_.class_prior_[1], eps, 1 - eps))
            init_raw = float(np.log(p1 / (1 - p1)))
        else:
            raise NotImplementedError("GBDT init estimator must be the default prior or 'zero'")
        denom = 1.0
        lr = np.float64(clf.learning_rate)

        def leaf_values(t):
            return lr * t.value[:, 0, 0].astype(np.float64)

    else:
        raise NotImplementedError(f"unsupported classifier {kind}")

    flat = [_flatten_tree(t, col_word, col_code, col_is_cat, leaf_values(t)) for t in trees]
    impute = np.zeros(ROW_WORDS, dtype=np.float32)
    with np.errstate(over="ignore"):
        impute[n_cat : n_cat + n_num] = medians.astype(np.float32)
    vocab = np.zeros(ROW_WORDS, dtype=np.int32)
    vocab[:n_cat] = [len(c) for c in categories]
    blob, max_depth = _assemble_blob(flat, agg, init_raw, denom, n_cat, n_num, impute, vocab)
    n_trees = len(trees)
    return FlatForest(
        blob=blob,
        cat_features=[str(c) for c in cat_cols],
        num_features=[str(c) for c in num_cols],
        categories=categories,
        classes=[c.item() if hasattr(c, "item") else c for c in clf.classes_],
        agg_mode=agg,
        n_trees=n_trees,
        max_depth=int(max_depth),
        total_nodes=int(sum(len(m[0]) for m in flat)),
        missing_codes=missing_codes,
        none_codes=none_codes,
    )


def parse_header(blob: bytes) -> dict:
    """Decode the fixed header + group table (host-side mirror of ``forest_blob.h``)."""
    f = struct.unpack_from(_HEADER_FMT, blob, 0)
    keys = ["magic", "version", "header_bytes", "agg_mode", "n_trees", "n_groups", "row_words", "n_cat", "n_num",
            "max_depth", "flags", "init_raw", "denom", "groups_off", "chunks_off", "chunks_bytes", "total_bytes"]
    h = dict(zip(keys, f[:17]))
    h["impute"] = np.array(f[17:41], dtype=np.float32)
    h["vocab"] = np.array(f[41:65], dtype=np.int32)
    h["threshold"] = f[65]
    h["path_bound"] = f[66]
    gk = ["chunk_off", "chunk_bytes", "n_slots", "n_leaf_slots", "depth", "n_trees"]
    h["groups"] = [
        dict(zip(gk, struct.unpack_from(_GROUP_FMT, blob, h["groups_off"] + 32 * g)[:6])) for g in range(h["n_groups"])
    ]
    return h


# ---------------------------------------------------------------------------------------------------------------------
# Path table for exact TreeSHAP (layout in ``csrc/forest_paths.h``)
# ---------------------------------------------------------------------------------------------------------------------
PATHS_MAGIC = b"B2FPATHS"
PATHS_VERSION = 1
PATHS_HEADER_BYTES = 256
PATH_RECORD_BYTES = 24
PATH_ELEM_BYTES = 48
PATHS_MAX_LEN = 24  # bias + at most 23 fields
PE_BIAS, PE_NUM, PE_CAT, PE_HAS_HI = 0, 1, 2, 4
BIAS_FIELD = 0xFF
_PATHS_HEADER_FMT = "<8s" + "I" * 10 + "dd" + "Q" * 4  # 96 bytes, padded to 256
_PATH_RECORD = np.dtype([("first", "<u4"), ("len", "<u4"), ("tree", "<u4"), ("reserved", "<u4"), ("leaf", "<f8")])
_PATH_ELEM = np.dtype([("field", "<u4"), ("kind", "<u4"), ("lo", "<f4"), ("hi", "<f4"), ("mask", "<u4", (4,)),
                       ("zero_fraction", "<f8"), ("inv_zero_fraction", "<f8")])
assert _PATH_RECORD.itemsize == PATH_RECORD_BYTES and _PATH_ELEM.itemsize == PATH_ELEM_BYTES


def blob_fingerprint(blob: bytes) -> int:
    """64-bit fingerprint of a forest blob: sum over its little-endian 64-bit words w_i of splitmix64(w_i ^ i * golden), mod
    2^64 (``b2f_model_attach_explainer`` computes the same over the model's blob to tie a path table to its forest)."""
    w = np.frombuffer(blob, dtype="<u8").astype(np.uint64)
    z = w ^ (np.arange(w.size, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15))
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = z ^ (z >> np.uint64(31))
    return int(z.sum(dtype=np.uint64))


def _tree_paths(tree, col_word, col_code, col_is_cat, leaf_value):
    """One sklearn ``Tree`` -> (per (leaf, ancestor) pair arrays, leaf node ids), vectorised over the tree's leaves.

    Pair k belongs to leaf ``pair_leaf[k]`` (an index into the returned leaves) and says: at ``node``, the path goes to
    ``child``.  The condition a row must meet there is expressed on the node's request field (``col_word``)."""
    left = tree.children_left.astype(np.int64)
    right = tree.children_right.astype(np.int64)
    cover = tree.weighted_n_node_samples.astype(np.float64)
    n = left.shape[0]
    parent = np.full(n, -1, dtype=np.int64)
    internal = np.nonzero(left != -1)[0]
    parent[left[internal]] = internal
    parent[right[internal]] = internal
    leaves = np.nonzero(left == -1)[0]
    pair_leaf, pair_node, pair_child = [], [], []
    cur = leaves.copy()
    idx = np.arange(leaves.size)
    while cur.size:
        p = parent[cur]
        up = p >= 0
        cur, idx, p = cur[up], idx[up], p[up]
        pair_leaf.append(idx)
        pair_node.append(p)
        pair_child.append(cur)
        cur = p
    pl = np.concatenate(pair_leaf) if pair_leaf else np.zeros(0, np.int64)
    pn = np.concatenate(pair_node) if pair_node else np.zeros(0, np.int64)
    pc = np.concatenate(pair_child) if pair_child else np.zeros(0, np.int64)
    col = tree.feature[pn].astype(np.int64)
    thr = tree.threshold[pn].astype(np.float64)
    go_right = pc == right[pn]
    return dict(leaf=pl, field=col_word[col], is_cat=col_is_cat[col], code=col_code[col], thr=thr, right=go_right,
                zf=cover[pc] / cover[pn]), leaves, leaf_value[leaves].astype(np.float64), cover


def flatten_explainer(pipeline, flat: FlatForest | None = None) -> bytes:
    """Fitted reference-style Pipeline -> path table for ``b2f_model_attach_explainer`` (layout in ``csrc/forest_paths.h``).

    One path per leaf of every classifier tree, its nodes merged by request field as in GPUTreeShap (Mitchell et al., PeerJ
    CS 2022): per field the product of ``cover(child) / cover(parent)`` over the path's nodes on it (cover =
    ``tree_.weighted_n_node_samples``) and the condition a row must meet to follow the path at all of them -- a float32
    interval ``[lo, hi)`` under the prediction kernels' compare for a numeric field, a 128-bit mask over ``code + 1`` (bit 0 =
    unknown / missing) for a categorical one.  A categorical field is ONE player however many one-hot columns its nodes
    test.  ``flat``: the pipeline's ``flatten_pipeline`` result when the caller already has it (its blob is fingerprinted)."""
    if flat is None:
        flat = flatten_pipeline(pipeline)
    pre = pipeline.named_steps["preprocessor"]
    clf = pipeline.named_steps["classifier"]
    _, _, categories, _, col_word, col_code, col_is_cat, _, _ = _describe_preprocessor(pre)
    if any(len(c) > 127 for c in categories):
        raise NotImplementedError("explanations need categorical fields of at most 127 categories (a 128-bit code mask)")
    n_cat, n_num = len(flat.cat_features), len(flat.num_features)
    if flat.agg_mode == AGG_RF_MEAN:
        trees = [e.tree_ for e in clf.estimators_]
        denom, init = float(len(trees)), 0.0

        def leaf_values(t):
            v = t.value[:, 0, :]
            s = v.sum(axis=1)
            return v[:, 1] / np.where(s == 0.0, 1.0, s)

    else:
        trees = [e.tree_ for e in clf.estimators_[:, 0]]
        denom, init = 1.0, parse_header(flat.blob)["init_raw"]
        lr = np.float64(clf.learning_rate)

        def leaf_values(t):
            return lr * t.value[:, 0, 0].astype(np.float64)

    recs, elems, expected = [], [], []
    n_elems = 0
    for ti, t in enumerate(trees):
        pr, leaves, lv, cover = _tree_paths(t, col_word, col_code, col_is_cat, leaf_values(t))
        # v(empty set) of this tree: every leaf weighted by its cover share
        expected.append(float(np.dot(lv, cover[leaves] / cover[0])))
        if pr["leaf"].size == 0:
            continue  # a single-leaf tree moves only the base value
        order = np.lexsort((pr["field"], pr["leaf"]))
        pr = {k: v[order] for k, v in pr.items()}
        key = pr["leaf"] * 64 + pr["field"]
        start = np.nonzero(np.r_[True, key[1:] != key[:-1]])[0]
        # numeric: the left branch needs x < t', the right one x >= t' (or unordered)
        t32 = strict_upper_f32(pr["thr"])
        lo = np.where(pr["right"] & ~pr["is_cat"], t32, np.float32(-np.inf)).astype(np.float32)
        hi = np.where(~pr["right"] & ~pr["is_cat"], t32, np.float32(np.inf)).astype(np.float32)
        has_hi = (~pr["right"] & ~pr["is_cat"]).astype(np.uint32)
        # categorical: the one-hot column is 1 iff code == the column's code; left iff that value <= thr.  Bit c + 1 of the
        # mask: code c follows the path here (c = -1: unknown, and every code no node tests)
        left_if_match = 1.0 <= pr["thr"]
        left_if_other = 0.0 <= pr["thr"]
        other_ok = np.where(pr["right"], ~left_if_other, left_if_other)
        match_ok = np.where(pr["right"], ~left_if_match, left_if_match)
        mask = np.where(other_ok[:, None], np.uint32(0xFFFFFFFF), np.uint32(0)).repeat(4, axis=1).astype(np.uint32)
        bit = pr["code"] + 1
        rows = np.nonzero(pr["is_cat"])[0]
        w, b = bit[rows] // 32, (bit[rows] % 32).astype(np.uint32)
        one = np.left_shift(np.uint32(1), b)
        mask[rows, w] = np.where(match_ok[rows], mask[rows, w] | one, mask[rows, w] & ~one)
        mask[~pr["is_cat"]] = 0
        # merge by (leaf, field)
        m_zf = np.multiply.reduceat(pr["zf"], start)
        m_lo = np.maximum.reduceat(lo, start)
        m_hi = np.minimum.reduceat(hi, start)
        m_has_hi = np.bitwise_or.reduceat(has_hi, start)
        m_mask = np.bitwise_and.reduceat(mask, start, axis=0)
        m_field = pr["field"][start]
        m_cat = pr["is_cat"][start]
        m_leaf = pr["leaf"][start]
        counts = np.bincount(m_leaf, minlength=leaves.size)
        have = np.nonzero(counts)[0]
        lens = counts[have] + 1
        # element table of this tree: per path a bias element, then its merged fields
        e = np.zeros(int(lens.sum()), dtype=_PATH_ELEM)
        first = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
        pos = np.ones(e.size, dtype=bool)
        pos[first] = False
        bias = first
        e["field"][bias] = BIAS_FIELD
        e["kind"][bias] = PE_BIAS
        e["zero_fraction"][bias] = 1.0
        e["inv_zero_fraction"][bias] = 1.0
        body = np.nonzero(pos)[0]  # m_* are sorted by leaf then field: they fill the non-bias slots in order
        e["field"][body] = m_field
        e["kind"][body] = np.where(m_cat, PE_CAT, PE_NUM | (m_has_hi * PE_HAS_HI)).astype(np.uint32)
        e["lo"][body] = np.where(m_cat, np.float32(0), m_lo)
        e["hi"][body] = np.where(m_cat | (m_has_hi == 0), np.float32(0), m_hi)
        e["mask"][body] = m_mask
        e["zero_fraction"][body] = m_zf
        e["inv_zero_fraction"][body] = 1.0 / m_zf
        r = np.zeros(have.size, dtype=_PATH_RECORD)
        r["first"] = first + n_elems
        r["len"] = lens
        r["tree"] = ti
        r["leaf"] = lv[have]
        recs.append(r)
        elems.append(e)
        n_elems += e.size
    recs = np.concatenate(recs) if recs else np.zeros(0, dtype=_PATH_RECORD)
    elems = np.concatenate(elems) if elems else np.zeros(0, dtype=_PATH_ELEM)
    max_len = int(recs["len"].max()) if recs.size else 0
    if max_len > PATHS_MAX_LEN:
        raise NotImplementedError(f"merged path of {max_len} elements exceeds {PATHS_MAX_LEN}")
    ex = np.asarray(expected, dtype=np.float64)
    base = float(ex.sum() / denom) if flat.agg_mode == AGG_RF_MEAN else float(init + ex.sum())
    paths_off = PATHS_HEADER_BYTES
    elems_off = (paths_off + recs.nbytes + 15) // 16 * 16
    total = elems_off + elems.nbytes
    header = struct.pack(_PATHS_HEADER_FMT, PATHS_MAGIC, PATHS_VERSION, PATHS_HEADER_BYTES, n_cat, n_num, flat.agg_mode,
                         len(trees), recs.size, max_len, elems.size, 0, base, denom, blob_fingerprint(flat.blob), paths_off,
                         elems_off, total)
    out = bytearray(total)
    out[: len(header)] = header
    out[paths_off : paths_off + recs.nbytes] = recs.tobytes()
    out[elems_off:] = elems.tobytes()
    return bytes(out)


def parse_explainer(paths: bytes) -> dict:
    """Decode a path table (host-side mirror of ``forest_paths.h``): header fields plus ``paths`` / ``elems`` record arrays."""
    f = struct.unpack_from(_PATHS_HEADER_FMT, paths, 0)
    keys = ["magic", "version", "header_bytes", "n_cat", "n_num", "agg_mode", "n_trees", "n_paths", "max_len", "n_elems",
            "reserved0", "base_value", "denom", "fingerprint", "paths_off", "elems_off", "total_bytes"]
    h = dict(zip(keys, f))
    h["paths"] = np.frombuffer(paths, dtype=_PATH_RECORD, count=h["n_paths"], offset=h["paths_off"])
    h["elems"] = np.frombuffer(paths, dtype=_PATH_ELEM, count=h["n_elems"], offset=h["elems_off"])
    return h
