#!/usr/bin/env python
"""Freeze library outputs for the two detectors of ``CustomModel.predict`` into ``expected_detectors.npz``.

The reference ships no golden vectors (SURVEY.md section 4) and neither alibi-detect wrapper is installed, so what is
frozen are the outputs of the libraries that hold the arithmetic, computed on the frozen copy of the reference's own
``curated.csv`` / ``inference.csv`` (``tests/golden/curated.npz``, ``inference.npz``):

* outlier detector (reference ``02-register-model.ipynb:232-233,339``): ``-IsolationForest(n_estimators=100,
  random_state=0).fit(curated numerics).decision_function(X)`` on the first 3 000 curated rows and the 81 inference rows;
* drift detector (``:224-229,338``): per-feature statistic and float64 p-value of ``oracle.drift`` (scipy
  ``chi2_contingency`` / ``ks_2samp(method="exact")``) for three batches against the 30 000 curated rows.

Usage:  python tests/golden/make_golden_detectors.py      (needs no reference checkout)
"""

from __future__ import annotations

import os
import sys

import numpy as np
import scipy
import sklearn
from scipy import stats
from sklearn.ensemble import IsolationForest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import datasets, reference_pipeline as rp  # noqa: E402


def drift_batches(cur, inf):
    shifted = cur[rp.FEATURES].iloc[:500].copy()
    for name in rp.NUMERIC_FEATURES:
        shifted[name] = shifted[name] * 1.15 + 3.0
    shifted["sex"] = shifted["sex"].iloc[0]
    return {"head64": cur[rp.FEATURES].iloc[:64], "inference": inf[rp.FEATURES], "shifted500": shifted}


def drift_reference_values(ref, batch):
    """(statistic, p-value) per feature in rp.FEATURES order, float64, straight from scipy."""
    stat, p = np.zeros(len(rp.FEATURES)), np.zeros(len(rp.FEATURES))
    for i, name in enumerate(rp.FEATURES):
        if name in rp.CATEGORICAL_FEATURES:
            a = ref[name].astype(str).to_numpy()
            x = batch[name].astype(str).to_numpy()
            union = sorted(set(a.tolist()) | set(x.tolist()))
            r = stats.chi2_contingency(np.array([[np.sum(a == v) for v in union], [np.sum(x == v) for v in union]]))
            stat[i], p[i] = r[0], r[1]
        else:
            r = stats.ks_2samp(ref[name].to_numpy(float), batch[name].to_numpy(float), alternative="two-sided", method="exact")
            stat[i], p[i] = r.statistic, r.pvalue
    return stat, p


def main() -> None:
    cur, inf = datasets.load_curated(), datasets.load_inference()
    iso = IsolationForest(n_estimators=100, random_state=0).fit(cur[rp.NUMERIC_FEATURES].to_numpy())
    out = {
        "sklearn_version": np.array(sklearn.__version__),
        "scipy_version": np.array(scipy.__version__),
        "iforest_offset": np.array(iso.offset_),
        "iforest_score_head3000": -iso.decision_function(cur[rp.NUMERIC_FEATURES].iloc[:3000].to_numpy()),
        "iforest_score_inference": -iso.decision_function(inf[rp.NUMERIC_FEATURES].to_numpy()),
    }
    ref = cur[rp.FEATURES]
    for key, batch in drift_batches(cur, inf).items():
        stat, p = drift_reference_values(ref, batch)
        out[f"drift_stat_{key}"] = stat
        out[f"drift_p_{key}"] = p
        print(key, "min p", p.min(), "max p", p.max())
    np.savez_compressed(os.path.join(HERE, "expected_detectors.npz"), **out)
    print("expected_detectors.npz", os.path.getsize(os.path.join(HERE, "expected_detectors.npz")))


if __name__ == "__main__":
    main()
