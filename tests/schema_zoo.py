"""Request schemas other than the credit-default one, and everything a test needs to hold the kernels to the library on
them (TEST INFRASTRUCTURE, no GPU).

The library accepts any reference-shaped pipeline (``ColumnTransformer([categorical: imputer + OneHotEncoder, numeric:
imputer])``, at most 23 raw fields), and each row layout and kernel has its own limits: the packed 64-byte row (exactly 9
categoricals of <= 126 categories), the rank layout (<= 16 categoricals in a 4- or 8-byte block, tested codes < 64, <= 128
pseudo-features), the path table's 128-bit code masks, the native encoder (<= 16 categoricals) and the moments kernel's
compiled-in count of categorical words per 16-byte vector.  The schemas here put set bits where the credit data never
does: packed field 4 across the word boundary, an 8-byte categorical block, codes >= 32 / 64 / 96 in the masks, fewer
fields than warps, more than 16 categoricals.

* ``SCHEMAS``: vocabulary size per categorical field and the number of numerics.
* ``make_frame``: a seeded synthetic frame (string categories, numerics of varied scale, a target that depends on high
  codes so the trees split on them).
* ``make_pipeline``: the reference shape, RandomForest or GBDT.
* ``edge_rows``: unknown / None / NaN / literal "missing" categories, NaN, +-0, +-3e38, 1e-45 and values on split
  thresholds (and one float32 ulp either side), generic over the schema.
* ``dense``: the oracles' input, ``preprocessor.transform(df)`` as dense float32 -- sklearn itself.
* ``tree_subset`` / ``tested_pairs``: a forest restricted to some of its trees, and the (field, code) pairs it tests.
"""

from __future__ import annotations

import copy

import numpy as np
import pandas as pd

TARGET = "target"

# name -> (vocabulary size per categorical field, number of numerics)
SCHEMAS = {
    # packed row: field 4 (bits 28..34) gets codes + 1 up to 126, across the 32-bit word boundary; fields 4, 6 and 8 have
    # codes >= 32, >= 64, >= 96 for the path table's mask words
    "packed_wide": ([2, 7, 4, 10, 126, 40, 64, 3, 100], 10),
    # rank layout: 16 categoricals (the maximum) in 60 bits -> the 8-byte categorical block; four fields of 64 categories
    # (codes 32..63 land in the high half of the kernel's 64-bit per-feature mask); 7 numerics: F = 23
    "rank_wide": ([64, 5, 64, 7, 3, 64, 6, 2, 64, 4, 7, 5, 3, 6, 2, 7], 7),
    # F = 3 fields: fewer than the 8 warps the interaction kernel spreads fields over
    "tiny": ([3], 2),
    # 17 categoricals: no rank layout and no native encoder
    "over16": ([3, 4, 5, 6, 2, 3, 4, 5, 6, 2, 3, 4, 5, 6, 2, 3, 8], 6),
}

# the moments kernel compiles NC = 0..4 categorical words per 16-byte vector q: between them these schemas give every NC
# at some q > 0 (n_cat 9: NC 1 at q = 2; 6: 2 at q = 1; 7: 3 at q = 1; 16: 4 at q = 1..3; any: 0)
MOMENT_N_CAT = (1, 6, 7, 9, 10, 11, 16)


def moments_schema(n_cat: int):
    return ([3 + (j % 5) for j in range(n_cat)], 23 - n_cat)


def cat_names(spec):
    return [f"cat_{j:02d}" for j in range(len(spec[0]))]


def num_names(spec):
    return [f"num_{k:02d}" for k in range(spec[1])]


def features(spec):
    return cat_names(spec) + num_names(spec)


def category(j: int, code: int) -> str:
    return f"f{j}_c{code:03d}"  # zero-padded: the encoder's sorted order is the code order


def make_codes_nums(spec, n: int, seed: int):
    """-> (codes int32 (n, n_cat), nums float64 (n, n_num)): uniform codes, numerics of scale 1e-3 .. 1e3 (some integer
    valued, so ties sit on split thresholds)."""
    vocab, n_num = spec
    rng = np.random.default_rng(seed)
    codes = np.stack([rng.integers(0, v, n) for v in vocab], axis=1).astype(np.int32) if vocab else np.zeros((n, 0), np.int32)
    nums = np.empty((n, n_num), dtype=np.float64)
    for k in range(n_num):
        scale = 10.0 ** ((k % 7) - 3)
        col = rng.normal(0.0, 1.0, n) * scale + (k - n_num / 2) * scale
        nums[:, k] = np.round(col) if k % 3 == 2 else col
    return codes, nums


def _target(spec, codes, nums, seed):
    """Each category gets its own effect; codes in the top quarter of a wide field get a large one, so splits on high codes
    carry information."""
    vocab, n_num = spec
    rng = np.random.default_rng(seed + 1)
    z = np.zeros(len(codes))
    for j, v in enumerate(vocab):
        eff = rng.normal(0.0, 0.6, v)
        if v >= 32:
            eff[(3 * v) // 4 :] += rng.choice([-1.5, 1.5], v - (3 * v) // 4)
        z += eff[codes[:, j]]
    for k in range(n_num):
        col = nums[:, k]
        z += 0.8 * np.tanh((col - np.median(col)) / (np.std(col) + 1e-12)) * (1 if k % 2 else -1)
    z += rng.logistic(0.0, 1.0, len(z))
    return (z > np.median(z)).astype(np.int64)


def frame_from_arrays(spec, codes, nums) -> pd.DataFrame:
    cols = {}
    for j, name in enumerate(cat_names(spec)):
        cats = np.array([category(j, c) for c in range(spec[0][j])], dtype=object)
        cols[name] = cats[codes[:, j]]
    for k, name in enumerate(num_names(spec)):
        cols[name] = nums[:, k]
    return pd.DataFrame(cols)


def make_frame(spec, n: int, seed: int = 0, target: bool = True) -> pd.DataFrame:
    codes, nums = make_codes_nums(spec, n, seed)
    df = frame_from_arrays(spec, codes, nums)
    if target:
        df[TARGET] = _target(spec, codes, nums, seed)
    return df


def make_pipeline(spec, kind: str = "rf", **params):
    from sklearn.compose import ColumnTransformer
    from sklearn.ensemble import GradientBoostingClassifier, RandomForestClassifier
    from sklearn.impute import SimpleImputer
    from sklearn.pipeline import Pipeline
    from sklearn.preprocessing import OneHotEncoder

    catp = Pipeline([("imputer", SimpleImputer(strategy="constant", fill_value="missing")), ("ohe", OneHotEncoder(handle_unknown="ignore"))])
    nump = Pipeline([("imputer", SimpleImputer(strategy="median"))])
    pre = ColumnTransformer([("categorical", catp, cat_names(spec)), ("numeric", nump, num_names(spec))])
    clf = RandomForestClassifier(n_jobs=-1, **params) if kind == "rf" else GradientBoostingClassifier(**params)
    return Pipeline([("preprocessor", pre), ("classifier", clf)])


def fit_pipeline(spec, train: pd.DataFrame, kind: str = "rf", **params):
    pipe = make_pipeline(spec, kind, **params)
    pipe.fit(train[features(spec)], train[TARGET].to_numpy())
    return pipe


def dense(pipe, df: pd.DataFrame) -> np.ndarray:
    """The forest's input for ``df``: sklearn's own transform, dense float32 (the oracles' X32)."""
    X = pipe.named_steps["preprocessor"].transform(df)
    X = X.toarray() if hasattr(X, "toarray") else np.asarray(X)
    return X.astype(np.float32)


def predict(pipe, df: pd.DataFrame):
    """-> (P(class 1) float64, label int32), what the library computes."""
    X = df[list(pipe.named_steps["preprocessor"].feature_names_in_)]
    return pipe.predict_proba(X)[:, 1], pipe.predict(X).astype(np.int32)


def edge_rows(spec, pipe, n: int = 400, seed: int = 7) -> pd.DataFrame:
    """Rows on every edge the preprocessing has, for any schema: unknown categories, None, NaN, the literal "missing",
    NaN numerics, +-0, +-3e38, 1e-45, and numerics exactly on a split threshold of ``pipe`` and one float32 ulp either side
    (as float32 and as the float64 threshold itself)."""
    from oracle import treewalk as tw

    rng = np.random.default_rng(seed)
    base = make_frame(spec, n, seed=seed + 100, target=False)
    for name in cat_names(spec):
        col = base[name].astype(object).to_numpy().copy()
        r = rng.random(n)
        col[r < 0.08] = "never_seen_category"
        col[(r >= 0.08) & (r < 0.13)] = None
        col[(r >= 0.13) & (r < 0.17)] = np.nan
        col[(r >= 0.17) & (r < 0.20)] = "missing"
        base[name] = pd.Series(col, dtype=object)
    dump = tw.dump_pipeline(pipe)
    n_ohe = int(dump["cat_offsets"][-1])
    nodes = np.nonzero((dump["left"] != -1) & (dump["feature"] >= n_ohe))[0]
    nums = num_names(spec)
    if len(nodes):
        pick = rng.choice(nodes, size=n, replace=True)
        for i in range(n):
            t64 = float(dump["threshold"][pick[i]])
            t = np.float32(t64)
            v = [t, np.nextafter(t, np.float32(np.inf)), np.nextafter(t, np.float32(-np.inf)), t64][i % 4]
            base.loc[i, nums[int(dump["feature"][pick[i]]) - n_ohe]] = float(v)
    for name in nums:
        col = base[name].to_numpy(dtype=np.float64).copy()
        r = rng.random(n)
        col[r < 0.05] = np.nan
        col[(r >= 0.05) & (r < 0.06)] = 0.0
        col[(r >= 0.06) & (r < 0.07)] = -0.0
        col[(r >= 0.07) & (r < 0.08)] = 3.0e38
        col[(r >= 0.08) & (r < 0.09)] = -3.0e38
        col[(r >= 0.09) & (r < 0.10)] = 1e-45
        base[name] = col
    return base


N_TRAIN = 8000

# model name -> (schema, kind, parameters); fitted on N_TRAIN rows of make_frame(schema, seed 0)
MODELS = {
    "packed_wide": ("packed_wide", "rf", dict(n_estimators=60, max_depth=8, random_state=0)),
    "packed_wide_gbdt": ("packed_wide", "gbdt", dict(n_estimators=30, max_depth=4, random_state=0)),
    "packed_wide_shallow": ("packed_wide", "rf", dict(n_estimators=6, max_depth=3, random_state=0)),
    "rank_wide_pool": ("rank_wide", "rf", dict(n_estimators=300, max_depth=6, random_state=0)),
    "tiny": ("tiny", "rf", dict(n_estimators=20, max_depth=5, random_state=0)),
    "tiny_gbdt": ("tiny", "gbdt", dict(n_estimators=12, max_depth=3, random_state=0)),
    "over16": ("over16", "rf", dict(n_estimators=40, max_depth=7, random_state=0)),
}

_FITTED = {}


def fitted(name: str):
    """-> (schema spec, fitted pipeline), cached for the session.  ``rank_wide`` / ``rank_wide_129``: trees of
    ``rank_wide_pool`` that test exactly 120 / 121 (field, code) pairs, i.e. 128 / 129 pseudo-features with the 8 slots of
    the 7 numerics."""
    if name not in _FITTED:
        if name in ("rank_wide", "rank_wide_129"):
            spec, pool = fitted("rank_wide_pool")
            trees = trees_for_pair_count(pool, 128 - ((spec[1] + 1) & ~1) + (name == "rank_wide_129"))
            assert trees is not None, "no tree subset of the pool tests exactly the pairs wanted"
            _FITTED[name] = (spec, tree_subset(pool, trees))
        else:
            schema, kind, params = MODELS[name]
            spec = SCHEMAS[schema]
            _FITTED[name] = (spec, fit_pipeline(spec, make_frame(spec, N_TRAIN, seed=0), kind, **params))
    return _FITTED[name]


def fitted_small(spec):
    """A two-tree forest on ``spec`` (for the kernels that only need the schema, such as the moments kernel)."""
    key = ("small", tuple(spec[0]), spec[1])
    if key not in _FITTED:
        _FITTED[key] = (spec, fit_pipeline(spec, make_frame(spec, 500, seed=0), "rf", n_estimators=2, max_depth=2, random_state=0))
    return _FITTED[key]


def tested_pairs(pipe, trees=None) -> set:
    """(field, code) pairs the trees' one-hot splits test (every tree when ``trees`` is None)."""
    from oracle import treeshap as ts
    from oracle import treewalk as tw

    dump = tw.dump_pipeline(pipe)
    fields = ts.column_fields(dump)
    offs = dump["cat_offsets"]
    n_ohe = int(offs[-1])
    out = set()
    for t in range(dump["n_trees"]) if trees is None else trees:
        lo, hi = int(dump["tree_off"][t]), int(dump["tree_off"][t + 1])
        f = dump["feature"][lo:hi][dump["left"][lo:hi] != -1]
        for c in f[f < n_ohe]:
            j = int(fields[c])
            out.add((j, int(c) - int(offs[j])))
    return out


def tree_pairs(pipe) -> list:
    n = len(pipe.named_steps["classifier"].estimators_)
    return [tested_pairs(pipe, [t]) for t in range(n)]


def tree_subset(pipe, trees):
    """A copy of a fitted RandomForest pipeline that keeps only ``trees`` (in that order)."""
    sub = copy.deepcopy(pipe)
    clf = sub.named_steps["classifier"]
    clf.estimators_ = [clf.estimators_[t] for t in trees]
    clf.n_estimators = len(trees)
    return sub


def trees_for_pair_count(pipe, want: int):
    """Trees of ``pipe`` chosen greedily so that they test exactly ``want`` distinct (field, code) pairs -> list of tree
    indices (None if no seeded tree order gets there)."""
    per = tree_pairs(pipe)
    rng = np.random.default_rng(0)
    for attempt in range(500):  # greedy over seeded tree orders until one lands exactly on `want`
        order = np.arange(len(per)) if attempt == 0 else rng.permutation(len(per))
        chosen, have = [], set()
        for t in order:
            if len(have | per[t]) <= want:
                chosen.append(int(t))
                have |= per[t]
            if len(have) == want:
                return chosen
    return None
