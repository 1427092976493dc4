"""The decision-boundary fixtures really put rows on the boundary, and the exact reference agrees with sklearn.

``tests/decision_models.py`` builds the models; ``test_gpu_decisions.py`` runs them through every kernel.  Here, without
a GPU: exact-tie counts are above zero and sklearn sends every tie to class 0; near-tie rows have a float64 margin whose
sign depends on the summation order; the exact-sign reference equals sklearn's ``predict`` on every row outside the
rounding band; GBDT rows at ``raw == 0`` and at ``0 < raw <= 5.6e-17`` get label 1 with ``p1 == 0.5``; the outlier
threshold is a score many rows share."""

import numpy as np
import pytest

import decision_models as dm


@pytest.fixture(scope="module")
def frame(curated):
    from oracle import reference_pipeline as rp

    return curated[rp.FEATURES].iloc[3000:9000]


@pytest.mark.parametrize("n_trees", [2, 4, 100, 290])
def test_rf_exact_ties_are_ties_and_go_to_class_0(curated, frame, n_trees):
    pipe = dm.rf_exact_ties(curated, n_trees)
    p0, p1 = dm.leaf_terms(pipe, frame)
    margin = dm.exact_margin(p0, p1)
    tie = margin == 0.0
    assert tie.sum() >= 50
    # dyadic payloads: every order gives the same sum, so the float64 tie is the exact one
    assert (p1.sum(axis=1)[tie] == n_trees / 2).all() and (p1[:, ::-1].cumsum(axis=1)[:, -1][tie] == n_trees / 2).all()
    proba = pipe.predict_proba(frame)
    assert (proba[tie, 1] == 0.5).all() and (proba[tie, 0] == 0.5).all()
    label = pipe.predict(frame)
    assert (label[tie] == 0).all()
    assert (label == dm.exact_labels(p0, p1)).all()


@pytest.mark.parametrize("n_trees", [100, 290])
def test_rf_near_ties_depend_on_summation_order(curated, frame, n_trees):
    pipe = dm.rf_near_ties(curated, n_trees)
    p0, p1 = dm.leaf_terms(pipe, frame)
    assert (p0 + p1 == 1.0).all()  # each leaf's fractions add to exactly 1: the margin is 2 sum p1 - T
    margin = dm.exact_margin(p0, p1)
    near = np.abs(margin) <= dm.band(n_trees)
    assert near.sum() >= 30
    forward = np.array([sum(r) for r in p1])
    backward = np.array([sum(r[::-1]) for r in p1])
    pairwise = p1.sum(axis=1)
    warp = p1.reshape(len(p1), -1, 2).sum(axis=2).sum(axis=1)  # another grouping
    signs = np.stack([(2 * s - n_trees) > 0 for s in (forward, backward, pairwise, warp)])
    order_dependent = (signs != signs[0]).any(axis=0)
    assert order_dependent.sum() >= 10 and near[order_dependent].all()
    # sklearn (tree-order float64 sums) agrees with the exact sign everywhere outside the band; inside, it may not
    label = pipe.predict(frame)
    want = dm.exact_labels(p0, p1)
    assert (label[~near] == want[~near]).all()
    assert (label[near] != want[near]).any()


def test_rf_reference_matches_sklearn_outside_the_band(curated, frame, rf100d6):
    """On a model nobody edited, every row is outside the band and the exact reference is sklearn's predict."""
    p0, p1 = dm.leaf_terms(rf100d6, frame)
    margin = dm.exact_margin(p0, p1)
    assert (np.abs(margin) > dm.band(100)).all()
    assert (rf100d6.predict(frame) == dm.exact_labels(p0, p1)).all()


def test_gbdt_raw_zero_and_tiny_positive(curated, frame):
    pipe = dm.gbdt_zero_raw(curated)
    _, terms = dm.leaf_terms(pipe, frame)
    raw = dm.exact_margin(None, terms)
    zero = raw == 0.0
    tiny = (raw > 0.0) & (raw <= 5.6e-17)
    assert zero.sum() >= 10 and tiny.sum() >= 10
    assert (raw[tiny] == dm.TINY).all()
    label = pipe.predict(frame)
    p1 = pipe.predict_proba(frame)[:, 1]
    assert (label[zero | tiny] == 1).all() and (p1[zero | tiny] == 0.5).all()
    assert (label == dm.exact_labels(None, terms)).all()
    # sklearn's tree-order sum loses 2^-56 against +-1/8: the decision does not hinge on it
    assert (pipe.decision_function(frame)[tiny] >= 0.0).all()


def test_iforest_threshold_is_a_shared_score(curated, iforest):
    from oracle import reference_pipeline as rp

    x = curated[rp.NUMERIC_FEATURES].to_numpy()
    score = -iforest.decision_function(x)
    thr = dm.shared_outlier_score(score)
    at = score == thr
    assert at.sum() >= 20
    assert not (score[at] > thr).any()
    assert (score[at] > np.nextafter(thr, -np.inf)).all()
    assert not (score[at] > np.nextafter(thr, np.inf)).any()


def test_iforest_payloads_and_path_bound_reproduce_sklearn_flags(curated, iforest):
    """The blob's per-tree payloads, added in tree order at the leaves sklearn reaches, give sklearn's path-length sum to
    the last bit; ``s <= iforest_path_bound(thr)`` is sklearn's ``score > thr`` at, above and below a shared score."""
    from oracle import reference_pipeline as rp

    from databricks_kubernetes_mlops_poc_b200 import flatten

    x = curated[rp.NUMERIC_FEATURES].to_numpy()
    score = -iforest.decision_function(x)
    h = flatten.parse_header(flatten.flatten_isolation_forest(iforest, 9, 14, threshold=0.0))
    assert h["flags"] & flatten.HEADER_HAS_PATH_BOUND
    depths = np.zeros(len(x))
    for est, feats in zip(iforest.estimators_, iforest.estimators_features_):
        t = est.tree_
        depth = np.zeros(t.node_count)
        for i in range(t.node_count):
            if t.children_left[i] != -1:
                depth[t.children_left[i]] = depth[t.children_right[i]] = depth[i] + 1.0
        payload = (depth.astype(np.int64) + 1) + flatten._average_path_length(t.n_node_samples) - 1.0
        depths += payload[est.apply(x[:, feats].astype(np.float32))]
    assert (-(-(2 ** (-np.divide(depths, h["denom"]))) - h["init_raw"]) == score).all()
    thr0 = dm.shared_outlier_score(score)
    for thr in (thr0, float(np.nextafter(thr0, np.inf)), float(np.nextafter(thr0, -np.inf)), 0.0, 0.95):
        bound = flatten.iforest_path_bound(h["init_raw"], h["denom"], thr)
        assert ((depths <= bound) == (score > thr)).all()
