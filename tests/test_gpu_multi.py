"""Multi-GPU C-ABI paths (one process driving several handles).  On a box with one visible GPU the same single-process
paths run over TWO REPLICAS ON THAT GPU (devices [0, 0]: two handles, two sets of streams and staging, the same slicing /
dealing / merging code), so the driver's round-end `pytest -m gpu` exercises them too; only the NCCL communicator needs two
distinct devices (run `pytest tests/test_gpu_multi.py -m gpu` on a machine with two GPUs)."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _devices():
    from databricks_kubernetes_mlops_poc_b200.engine import device_count

    n = device_count()
    return list(range(n)) if n >= 2 else [0, 0]


def test_predict_multi_and_stream_across_gpus(curated, rf100d6):
    from databricks_kubernetes_mlops_poc_b200 import flatten, training
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.engine import EngineGroup
    from oracle import reference_pipeline as rp

    flat = flatten.flatten_pipeline(rf100d6)
    enc = RowEncoder(flat)
    grp = EngineGroup(flat, devices=_devices())
    try:
        want_p, want_l = rp.oracle_predict(rf100d6, curated)
        rows = enc.encode_frame(curated)
        p, l = grp.predict_rows(rows)  # one batch sliced over all GPUs
        assert np.abs(p - want_p).max() <= 1e-12 and (l == want_l).all()
        pk = enc.pack_rows(rows)
        p32 = np.full(len(rows), -1, dtype=np.float32)
        l32 = np.full(len(rows), -1, dtype=np.int32)
        grp.predict_stream(pk, 4096, p32, l32)  # batches dealt round-robin, a host thread per GPU
        assert np.abs(p32 - want_p).max() <= 2e-7 and (l32 == want_l).all()
        # ranked rows from a NUMA-striped pinned buffer (what the config-4 stream leg of the bench deals)
        rk = enc.rank_rows(rows)
        host = grp.pinned_striped(np.uint32, rk.shape, 4096)
        host[:] = rk
        p32[:] = -1
        l32[:] = -1
        grp.predict_stream(host, 4096, p32, l32)
        assert np.abs(p32 - want_p).max() <= 2e-7 and (l32 == want_l).all()
        assert all(e.info()["launches"] > 0 for e in grp.engines)
    finally:
        grp.close()


def test_moments_merge_over_nccl(curated, rf100d6):
    """b2f_comm_init_all + b2f_moments_multi: per-GPU moments of row slices, 576-byte ncclAllGather, Chan merge."""
    from databricks_kubernetes_mlops_poc_b200 import flatten, training
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.engine import EngineGroup, device_count

    flat = flatten.flatten_pipeline(rf100d6)
    enc = RowEncoder(flat)
    _, codes, nums = training.synth_arrays(curated, 300_007, seed=21)
    rows = enc.encode_arrays(codes, nums)
    f = rows.view(np.float32)[:, 9:23].astype(np.float64)
    for nccl in ((False, True) if device_count() >= 2 else (False,)):  # a communicator needs distinct devices
        grp = EngineGroup(flat, devices=_devices(), nccl=nccl)
        try:
            got = grp.moments(rows)
            assert (got[9:23, 0] == (~np.isnan(f)).sum(0)).all()
            assert np.allclose(got[9:23, 1], np.nanmean(f, 0), rtol=1e-10)
            assert np.allclose(got[9:23, 2] / got[9:23, 0], np.nanvar(f, 0), rtol=1e-9)
            assert np.allclose(got[:9, 1], codes.mean(0), rtol=1e-12)
        finally:
            grp.close()


def test_full_model_across_gpus(curated, iforest, rf100d6):
    """Classifier + outlier forest sliced over the GPUs (b2f_predict_multi_ex with b2f_scored_full records), the drift
    detector on device 1, and concurrent drift requests over the detector's handle pool."""
    from concurrent.futures import ThreadPoolExecutor
    from types import SimpleNamespace

    from oracle import drift as od
    from oracle import reference_pipeline as rp

    from databricks_kubernetes_mlops_poc_b200.drift import TabularDrift
    from databricks_kubernetes_mlops_poc_b200.engine import device_count
    from databricks_kubernetes_mlops_poc_b200.model import B200Model

    ref = curated[rp.FEATURES]
    m = B200Model.from_pipeline(rf100d6, outlier=SimpleNamespace(isolationforest=iforest, threshold=0.0), devices=_devices())
    try:
        for df in (ref, ref.iloc[:3], ref.iloc[:1001]):
            out = m.predict(df)
            want_p, _ = rp.oracle_predict(rf100d6, df)
            want_s = -iforest.decision_function(df[rp.NUMERIC_FEATURES].to_numpy())
            assert np.abs(np.asarray(out["predictions"]) - want_p).max() <= 1e-12
            assert out["outliers"] == (want_s > 0.0).astype(int).tolist()
        assert all(e.info()["launches"] > 0 and e.info()["outlier_trees"] == 100 for e in m.group.engines)
        for r in m.replicas:  # the server's per-GPU scoring path
            proba, flags = r.score(ref.iloc[:500])
            assert np.abs(proba - want_p[:500]).max() <= 1e-12 and (flags == (want_s[:500] > 0.0)).all()
    finally:
        m.close()
    det = TabularDrift(ref, rp.CATEGORICAL_FEATURES, device=_devices()[-1])
    try:
        batches = [ref.iloc[100 * k: 100 * k + 64 + k].reset_index(drop=True) for k in range(12)]
        want = [od.drift_scores(ref, b, rp.CATEGORICAL_FEATURES) for b in batches]
        with ThreadPoolExecutor(max_workers=6) as pool:
            got = list(pool.map(det.score, batches))
        for g, w in zip(got, want):
            assert np.abs(np.asarray(g) - np.asarray(w)).max() <= 1e-6
        assert det.launches == 2 * len(batches)
    finally:
        det.close()
