"""GPU parity: the CUDA path, called through the C ABI, against the oracle (sklearn itself + the frozen
golden outputs).  Bar: class labels bit-exact, |dP| <= 1e-6 (north_star); we assert 1e-12 for float64
outputs and 2e-7 for float32 outputs, far inside it."""

import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TOL64 = 1e-12
TOL32 = 2e-7


def _engine(pipe, device=0):
    from databricks_kubernetes_mlops_poc_b200 import flatten
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine

    flat = flatten.flatten_pipeline(pipe)
    return ForestEngine(flat, device), RowEncoder(flat)


def _check(pipe, frames, walk=None, rows_per_warp=None, kernel="warp"):
    from oracle import reference_pipeline as rp

    old = {k: os.environ.get(k) for k in ("B2F_FORCE_WALK", "B2F_ROWS_PER_WARP", "B2F_KERNEL")}
    try:
        os.environ["B2F_KERNEL"] = kernel  # "warp": one warp per row; "tile": one thread per row (large-batch kernel)
        if walk:
            os.environ["B2F_FORCE_WALK"] = walk
        if rows_per_warp:
            os.environ["B2F_ROWS_PER_WARP"] = str(rows_per_warp)
        eng, enc = _engine(pipe)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    try:
        if walk:
            assert eng.info()["walk"] == walk
        for df in frames:
            want_p, want_l = rp.oracle_predict(pipe, df)
            rows = enc.encode_frame(df)
            p64, l64 = eng.predict_rows(rows, np.float64)
            p32, l32 = eng.predict_rows(rows, np.float32)
            assert np.abs(p64 - want_p).max() <= TOL64
            assert np.abs(p32.astype(np.float64) - want_p).max() <= TOL32
            assert (l64 == want_l).all() and (l32 == want_l).all()
        return eng.info()
    finally:
        eng.close()


def test_rf100d6_all_reference_rows(curated, inference, adversarial, rf100d6):
    """All 30 000 curated.csv rows + the 80 inference.csv rows (other column order) + edge rows, and
    the library outputs frozen in tests/golden (pins that this box's refit is the one we froze)."""
    from oracle import datasets
    from oracle import reference_pipeline as rp

    exp = datasets.load_expected("rf100d6")
    p, l = rp.oracle_predict(rf100d6, curated)
    assert np.abs(p - exp["proba1"]).max() < 1e-13 and (l == exp["label"]).all()
    info = _check(rf100d6, [curated, inference, adversarial])
    assert info["walk"] == "smem", "100 x depth-6 forest must be shared-memory resident"

    eng, enc = _engine(rf100d6)
    try:
        p64, l64 = eng.predict_rows(enc.encode_frame(curated), np.float64)
        assert np.abs(p64 - exp["proba1"]).max() <= TOL64 and (l64 == exp["label"]).all()
        pi, li = eng.predict_rows(enc.encode_frame(inference), np.float64)
        assert np.abs(pi - exp["inf_proba1"]).max() <= TOL64 and (li == exp["inf_label"]).all()
    finally:
        eng.close()


@pytest.mark.parametrize("rpw", [1, 2, 4])
def test_rf100d6_rows_per_warp_variants(curated, adversarial, rf100d6, rpw):
    _check(rf100d6, [curated.iloc[:20011], adversarial], rows_per_warp=rpw)


def test_rf100d6_global_walk(curated, adversarial, rf100d6):
    _check(rf100d6, [curated.iloc[:8000], adversarial], walk="global")


def test_rf500d8_all_reference_rows(curated, inference, adversarial, rf500d8):
    from oracle import datasets

    exp = datasets.load_expected("rf500d8")
    info = _check(rf500d8, [curated, inference, adversarial])
    assert info["walk"] == "global"  # 160 480 nodes do not fit 227 KB
    eng, enc = _engine(rf500d8)
    try:
        p64, l64 = eng.predict_rows(enc.encode_frame(curated), np.float64)
        assert np.abs(p64 - exp["proba1"]).max() <= TOL64 and (l64 == exp["label"]).all()
    finally:
        eng.close()


def test_deep_forest(curated, adversarial):
    """max_depth 24 is the top of the reference's search space (01-train-model.ipynb:344)."""
    from oracle import reference_pipeline as rp

    pipe = rp.fit_reference_pipeline(curated.iloc[:6000], dict(n_estimators=37, max_depth=24, criterion="entropy", random_state=1))
    info = _check(pipe, [curated.iloc[6000:9000], adversarial])
    assert info["max_depth"] > 12


def test_stumps_and_single_tree(curated, adversarial):
    from oracle import reference_pipeline as rp

    for params in (dict(n_estimators=1, max_depth=1, random_state=0), dict(n_estimators=33, max_depth=1, random_state=0),
                   dict(n_estimators=32, max_depth=3, random_state=0)):
        pipe = rp.fit_reference_pipeline(curated.iloc[:3000], params)
        _check(pipe, [curated.iloc[3000:4000], adversarial])


def test_gbdt(curated, adversarial, gbdt_small):
    _check(gbdt_small, [curated.iloc[:5000], adversarial])
    _check(gbdt_small, [curated.iloc[:2000]], walk="global")


def test_batch_size_edges(curated, rf100d6):
    from oracle import reference_pipeline as rp

    eng, enc = _engine(rf100d6)
    try:
        want_p, want_l = rp.oracle_predict(rf100d6, curated)
        rows = enc.encode_frame(curated)
        for n in (0, 1, 2, 31, 32, 33, 131, 132 * 32 + 1, 147, 148 * 32 + 1, 16384, 24576, 24577, 30000):
            p, l = eng.predict_rows(rows[:n], np.float64)
            assert p.shape == (n,) and l.shape == (n,)
            if n:
                assert np.abs(p - want_p[:n]).max() <= TOL64 and (l == want_l[:n]).all()
        # outputs are optional
        p, l = eng.predict_rows(rows[:100], np.float64, want_label=False)
        assert l is None and np.abs(p - want_p[:100]).max() <= TOL64
    finally:
        eng.close()


def test_async_ring_and_multi(curated, rf100d6):
    from databricks_kubernetes_mlops_poc_b200.engine import EngineGroup
    from oracle import reference_pipeline as rp

    eng, enc = _engine(rf100d6)
    try:
        want_p, want_l = rp.oracle_predict(rf100d6, curated)
        n = 20000
        rows, proba, label = eng.staging(n)
        enc.encode_frame(curated.iloc[:n], out=rows)
        proba[:] = -1
        tickets = []
        # several requests in flight on the pinned ring, disjoint slices
        for lo in range(0, n, 5000):
            tickets.append(eng.predict_rows_async(rows[lo : lo + 5000], proba[lo : lo + 5000], label[lo : lo + 5000]))
        for t in tickets:
            eng.wait(t)
        assert np.abs(proba - want_p[:n]).max() <= TOL64 and (label == want_l[:n]).all()
    finally:
        eng.close()
    grp = EngineGroup(enc_flat(rf100d6), devices=[0])
    try:
        p, l = grp.predict_rows(enc.encode_frame(curated.iloc[:7001]))
        assert np.abs(p - want_p[:7001]).max() <= TOL64 and (l == want_l[:7001]).all()
    finally:
        grp.close()


def enc_flat(pipe):
    from databricks_kubernetes_mlops_poc_b200 import flatten

    return flatten.flatten_pipeline(pipe)


def test_full_size_properties(curated, rf100d6):
    """BASELINE config 2 size (65 536 rows): size-independent properties instead of a row-by-row oracle:
    run-to-run determinism, host-pipelined == device-resident single launch, permutation equivariance,
    and agreement with the oracle on a random 4 096-row sample."""
    from databricks_kubernetes_mlops_poc_b200 import training
    from oracle import reference_pipeline as rp

    eng, enc = _engine(rf100d6)
    try:
        n = 65536
        vocabs, codes, nums = training.synth_arrays(curated, n, seed=20240)
        rows = enc.encode_arrays(codes, nums)
        p1, l1 = eng.predict_rows(rows, np.float64)
        p2, l2 = eng.predict_rows(rows, np.float64)
        assert (p1 == p2).all() and (l1 == l2).all()
        # device-resident single launch
        d_rows = eng.device_alloc(rows.nbytes)
        d_p = eng.device_alloc(n * 8)
        d_l = eng.device_alloc(n * 4)
        eng.h2d(d_rows, rows)
        eng.predict_device(d_rows, n, d_p, True, d_l)
        eng.sync()
        p3 = np.empty(n, dtype=np.float64)
        l3 = np.empty(n, dtype=np.int32)
        eng.d2h(p3, d_p)
        eng.d2h(l3, d_l)
        for d in (d_rows, d_p, d_l):
            eng.device_free(d)
        assert np.abs(p3 - p1).max() <= 1e-15 and (l3 == l1).all()
        perm = np.random.default_rng(1).permutation(n)
        p4, l4 = eng.predict_rows(rows[perm], np.float64)
        assert np.abs(p4 - p1[perm]).max() <= 1e-15 and (l4 == l1[perm]).all()
        idx = np.sort(np.random.default_rng(2).choice(n, 4096, replace=False))
        df = training.arrays_to_frame(vocabs, codes[idx], nums[idx])
        want_p, want_l = rp.oracle_predict(rf100d6, df)
        assert np.abs(p1[idx] - want_p).max() <= TOL64 and (l1[idx] == want_l).all()
        assert ((p1 >= 0) & (p1 <= 1)).all()
    finally:
        eng.close()


def test_moments(curated, rf100d6):
    from databricks_kubernetes_mlops_poc_b200 import training
    from databricks_kubernetes_mlops_poc_b200.engine import moments_merge

    eng, enc = _engine(rf100d6)
    try:
        n = 200_003
        _, codes, nums = training.synth_arrays(curated, n, seed=20243)
        rows = enc.encode_arrays(codes, nums)
        got = eng.moments(rows)
        f = rows.view(np.float32)[:, 9:23].astype(np.float64)
        cnt = (~np.isnan(f)).sum(axis=0)
        mean = np.nanmean(f, axis=0)
        var = np.nanvar(f, axis=0)
        assert (got[9:23, 0] == cnt).all()
        assert np.allclose(got[9:23, 1], mean, rtol=1e-9, atol=0)
        assert np.allclose(got[9:23, 2] / cnt, var, rtol=1e-9, atol=0)
        c = codes.astype(np.float64)
        assert (got[:9, 0] == n).all()
        assert np.allclose(got[:9, 1], c.mean(axis=0), rtol=1e-10)
        assert np.allclose(got[:9, 2] / n, c.var(axis=0), rtol=1e-9)
        # split + Chan merge == whole
        a, b = eng.moments(rows[:70001]), eng.moments(rows[70001:])
        merged = moments_merge(np.stack([a, b]))
        assert np.allclose(merged[:23], got[:23], rtol=1e-10, atol=1e-12)
        # determinism
        assert (eng.moments(rows) == got).all()
        # tiny / empty
        assert (eng.moments(rows[:0])[:, 0] == 0).all()
        one = eng.moments(rows[:1])
        assert (one[:9, 1] == c[0]).all() and (one[:23, 2] == 0).all()
    finally:
        eng.close()


def test_model_predict_dict(curated, inference, rf100d6):
    """End to end through the plugin boundary: DataFrame in, dict out (CustomModel.predict)."""
    from databricks_kubernetes_mlops_poc_b200.model import B200Model
    from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES, ModelOutput
    from oracle import reference_pipeline as rp

    model = B200Model.from_pipeline(rf100d6, reference_frame=curated, devices=[0])
    try:
        for df in (curated.iloc[:257], inference):
            out = model.predict(df)
            want_p, want_l = rp.oracle_predict(rf100d6, df)
            assert set(out) == {"predictions", "outliers", "feature_drift_batch"}
            assert np.abs(np.asarray(out["predictions"]) - want_p).max() <= TOL64
            assert out["outliers"] == [0] * len(df)
            assert list(out["feature_drift_batch"]) == ALL_FEATURES
            ModelOutput.model_validate(out)
            assert (model.predict_label(df) == want_l).all()
        with pytest.raises(KeyError):
            model.predict([])
    finally:
        model.close()


def test_http_end_to_end_and_load_model(curated, rf100d6, tmp_path):
    """POST /predict served by the CUDA engine, model loaded through the drop-in load_model(dir)
    (cached forest blob + drift reference), answers == the reference CustomModel restatement."""
    from fastapi.testclient import TestClient

    from databricks_kubernetes_mlops_poc_b200 import flatten, load_model
    from databricks_kubernetes_mlops_poc_b200.model import save_model_dir
    from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES, sample_request
    from databricks_kubernetes_mlops_poc_b200.server import create_app
    from oracle.custom_model import ReferenceCustomModel

    save_model_dir(str(tmp_path), flatten.flatten_pipeline(rf100d6), reference_frame=curated)
    ref = ReferenceCustomModel(rf100d6, curated)
    os.environ["MODEL_DIRECTORY"] = str(tmp_path)
    try:
        with TestClient(create_app(loader=load_model), raise_server_exceptions=False) as c:
            body = curated[ALL_FEATURES].iloc[:64].to_dict(orient="records")
            r = c.post("/predict", json=body)
            assert r.status_code == 200
            got = r.json()
            want = ref.predict(None, curated[ALL_FEATURES].iloc[:64])
            assert np.abs(np.asarray(got["predictions"]) - np.asarray(want["predictions"])).max() <= TOL64
            assert got["outliers"] == [float(v) for v in want["outliers"]]
            for k in ALL_FEATURES:  # same scipy statistics on both sides, float32 p-values
                assert abs(got["feature_drift_batch"][k] - want["feature_drift_batch"][k]) <= 1e-6
            assert c.post("/predict", json=sample_request()).status_code == 200
            assert c.post("/predict", json=[]).status_code == 500
            assert c.post("/predict", json=[{"age": "old"}]).status_code == 422
    finally:
        os.environ.pop("MODEL_DIRECTORY", None)


# ----------------------------------------------------------------------------- tile kernel (one thread per row)
def test_tile_kernel_resident_rf100d6(curated, inference, adversarial, rf100d6):
    """Forest resident in the shared-memory ring: all reference rows + edges, every batch-size edge."""
    from oracle import reference_pipeline as rp

    _check(rf100d6, [curated, inference, adversarial], kernel="tile")
    want_p, want_l = rp.oracle_predict(rf100d6, curated)
    os.environ["B2F_KERNEL"] = "tile"
    try:
        eng, enc = _engine(rf100d6)
    finally:
        os.environ.pop("B2F_KERNEL")
    try:
        rows = enc.encode_frame(curated)
        for n in (1, 31, 32, 33, 511, 512, 513, 20000, 30000):
            p, l = eng.predict_rows(rows[:n], np.float64)
            assert np.abs(p - want_p[:n]).max() <= TOL64 and (l == want_l[:n]).all()
    finally:
        eng.close()


def test_tile_kernel_streams_big_forest(curated, adversarial, rf500d8):
    """160 480 nodes: the forest streams through the shared-memory ring (full/empty mbarriers), several passes."""
    _check(rf500d8, [curated, adversarial], kernel="tile")


def test_tile_kernel_gbdt_and_small_forests(curated, adversarial, gbdt_small):
    from oracle import reference_pipeline as rp

    _check(gbdt_small, [curated.iloc[:9000], adversarial], kernel="tile")
    for params in (dict(n_estimators=1, max_depth=1, random_state=0), dict(n_estimators=5, max_depth=3, random_state=0),
                   dict(n_estimators=37, max_depth=11, random_state=0)):
        pipe = rp.fit_reference_pipeline(curated.iloc[:3000], params)
        _check(pipe, [curated.iloc[3000:5000], adversarial], kernel="tile")


def test_kernel_auto_selection_agrees(curated, rf100d6):
    """Default engine: chunked host batches take the warp kernel, one big device-resident launch the tile
    kernel; same answers (to float64 summation-order noise)."""
    from databricks_kubernetes_mlops_poc_b200 import training

    eng, enc = _engine(rf100d6)
    try:
        _, codes, nums = training.synth_arrays(curated, 70000, seed=11)
        rows = enc.encode_arrays(codes, nums)
        big_p, big_l = eng.predict_rows(rows, np.float64)
        d_rows = eng.device_alloc(rows.nbytes)
        d_p = eng.device_alloc(len(rows) * 8)
        d_l = eng.device_alloc(len(rows) * 4)
        eng.h2d(d_rows, rows)
        eng.predict_device(d_rows, len(rows), d_p, True, d_l)  # one 70 000-row launch -> tile kernel
        eng.sync()
        p = np.empty(len(rows))
        l = np.empty(len(rows), dtype=np.int32)
        eng.d2h(p, d_p)
        eng.d2h(l, d_l)
        for d in (d_rows, d_p, d_l):
            eng.device_free(d)
        assert np.abs(p - big_p).max() <= 1e-14 and (l == big_l).all()
    finally:
        eng.close()


@pytest.mark.parametrize("kernel", ["warp", "tile"])
def test_packed_rows_give_identical_results(curated, adversarial, rf100d6, gbdt_small, kernel):
    """64-byte packed rows (one third fewer PCIe bytes) vs 96-byte rows: bit-identical outputs, both kernels."""
    os.environ["B2F_KERNEL"] = kernel
    try:
        for pipe in (rf100d6, gbdt_small):
            eng, enc = _engine(pipe)
            try:
                assert eng.info()["packed_ok"] == 1
                for df in (curated.iloc[:20000], adversarial):
                    a = enc.encode_frame(df)
                    b = enc.pack_rows(a)
                    pa, la = eng.predict_rows(a, np.float64)
                    pb, lb = eng.predict_rows(b, np.float64)
                    assert (pa == pb).all() and (la == lb).all()
                    pb32, _ = eng.predict_rows(b, np.float32)
                    assert (pb32 == pa.astype(np.float32)).all()
            finally:
                eng.close()
    finally:
        os.environ.pop("B2F_KERNEL")


def test_pairs_output_and_chunk_plan(curated, rf100d6):
    """b2f_predict_pairs ({proba, label} interleaved, one D2H per chunk) == the two-array path, for batch
    sizes on every side of the chunk-plan thresholds."""
    from databricks_kubernetes_mlops_poc_b200 import training

    eng, enc = _engine(rf100d6)
    try:
        _, codes, nums = training.synth_arrays(curated, 70001, seed=5)
        rows = enc.encode_arrays_packed(codes, nums)
        for n in (0, 1, 1000, 16384, 24576, 24577, 32767, 32768, 65536, 70001):
            p, l = eng.predict_rows(rows[:n], np.float32)
            out = eng.predict_pairs(rows[:n])
            assert out.shape == (n,)
            assert (out["proba1"] == p).all() and (out["label"] == l).all()
    finally:
        eng.close()


def test_split_kernel_small_batches(curated, adversarial, rf100d6, rf500d8, gbdt_small):
    """The latency kernel (tree groups of a row across the warps of a CTA, walked from global memory)."""
    from oracle import reference_pipeline as rp

    for pipe in (rf100d6, rf500d8, gbdt_small):
        _check(pipe, [curated.iloc[:777], adversarial], kernel="split")
    for params in (dict(n_estimators=1, max_depth=1, random_state=0), dict(n_estimators=999, max_depth=3, random_state=0),
                   dict(n_estimators=40, max_depth=20, random_state=0)):
        pipe = rp.fit_reference_pipeline(curated.iloc[:2500], params)
        _check(pipe, [curated.iloc[2500:2700], adversarial.iloc[:64]], kernel="split")
    # default selection: tiny batches -> split kernel, and it agrees with the warp kernel
    eng, enc = _engine(rf500d8)
    try:
        rows = enc.encode_frame(curated.iloc[:300])
        want_p, want_l = rp.oracle_predict(rf500d8, curated.iloc[:300])
        for n in (1, 2, 3, 16, 256, 300):
            before = eng.info()["launches_split"]
            p, l = eng.predict_rows(rows[:n], np.float64)
            assert eng.info()["launches_split"] == before + 1
            assert np.abs(p - want_p[:n]).max() <= TOL64 and (l == want_l[:n]).all()
            out = eng.predict_pairs(enc.pack_rows(rows[:n]))
            assert np.abs(out["proba1"] - want_p[:n]).max() <= TOL32 and (out["label"] == want_l[:n]).all()
    finally:
        eng.close()


def test_stream_dealer(curated, iforest, rf100d6):
    """b2f_predict_stream: batches dealt round-robin over the models (one host thread per GPU inside the call)."""
    from databricks_kubernetes_mlops_poc_b200 import _cabi, flatten, training
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.engine import EngineGroup, device_count

    flat = flatten.flatten_pipeline(rf100d6)
    enc = RowEncoder(flat)
    grp = EngineGroup(flat, devices=list(range(min(2, device_count()))))
    n = 50_003
    _, codes, nums = training.synth_arrays(curated, n, seed=9)
    rows = enc.encode_arrays_packed(codes, nums)
    try:
        want_p, want_l = grp.engines[0].predict_rows(rows, np.float32)
        for batch, inflight in ((4096, 2), (65536, 1), (1000, 8)):
            p = np.full(n, -1, dtype=np.float32)
            l = np.full(n, -1, dtype=np.int32)
            grp.predict_stream(rows, batch, p, l, inflight=inflight)
            assert (p == want_p).all() and (l == want_l).all()
    finally:
        grp.close()
    # records through the C ABI, dealt over two replicas (both on GPU 0 when it is the only one); 4 096 does not divide n, so
    # every batch has to land at its own record offset.  The expected records come from one engine, batch by batch, so that
    # each batch takes the same kernel (and float64 summation order) as in the stream.
    grp = EngineGroup(flat, devices=[0, 1] if device_count() >= 2 else [0, 0])
    try:
        grp.attach_outlier_forest(flatten.flatten_isolation_forest(iforest, 9, 14, threshold=0.0))
        one, batch = grp.engines[0], 4096
        for kind, score in ((_cabi.OUT_PAIRS, one.predict_pairs), (_cabi.OUT_FULL, one.predict_full)):
            want = np.concatenate([score(rows[lo:lo + batch]) for lo in range(0, n, batch)])
            out = np.zeros(n, dtype=want.dtype)
            _cabi.check(grp._lib.b2f_predict_stream(grp._handles, 2, _cabi.ptr(rows), n, batch, _cabi.ROWS_PACKED64, _cabi.ptr(out), kind, None, 2),
                        "b2f_predict_stream")
            for field in ("proba1", "label", "is_outlier", "outlier_score"):  # every field the kernels write
                if field in want.dtype.names:
                    assert (out[field] == want[field]).all(), (kind, field)
    finally:
        grp.close()


def test_c_abi_error_paths(curated, rf100d6):
    """Bad arguments come back as error codes with a message (-> RuntimeError in the shim -> HTTP 500), never a crash."""
    import ctypes as C

    from databricks_kubernetes_mlops_poc_b200 import _cabi, flatten
    from databricks_kubernetes_mlops_poc_b200._cabi import B2FError
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine

    lib = _cabi.load_library()
    flat = flatten.flatten_pipeline(rf100d6)
    buf = np.frombuffer(flat.blob, dtype=np.uint8)
    assert not lib.b2f_model_create(_cabi.ptr(buf), buf.size, 99)  # no such device
    assert b"device 99" in lib.b2f_last_error()
    bad = bytearray(flat.blob)
    bad[0] = 0
    badbuf = np.frombuffer(bytes(bad), dtype=np.uint8)
    assert not lib.b2f_model_create(_cabi.ptr(badbuf), badbuf.size, 0)
    assert b"magic" in lib.b2f_last_error()
    eng = ForestEngine(flat, 0)
    try:
        rows = np.zeros((4, 24), dtype=np.uint32)
        out = np.zeros(4, dtype=np.float32)
        assert lib.b2f_predict(eng.handle, None, 4, _cabi.ptr(out), None) < 0  # NULL rows
        assert lib.b2f_predict(eng.handle, _cabi.ptr(rows), -1, _cabi.ptr(out), None) < 0  # negative n
        assert lib.b2f_predict_ex(eng.handle, _cabi.ptr(rows), 4, 7, _cabi.ptr(out), 0, None) < 0  # unknown row format
        assert lib.b2f_predict(None, _cabi.ptr(rows), 4, _cabi.ptr(out), None) < 0  # NULL model
        with pytest.raises(ValueError):
            eng.predict_rows(np.zeros((4, 23), dtype=np.uint32))
        with pytest.raises(B2FError):
            eng.moments_allgather(np.zeros((24, 3)))  # communicator not initialised
        # still healthy afterwards
        p, _ = eng.predict_rows(rows, np.float32)
        assert p.shape == (4,) and np.isfinite(p).all()
    finally:
        eng.close()


def test_load_model_from_mlflow_layout(curated, rf100d6, tmp_path):
    """The reference's artefact directory: artifacts/classifier/model/model.pkl (02-register-model.ipynb:317-321)
    -> load_model flattens the pickled sklearn Pipeline and caches the forest blob next to it."""
    import joblib

    from databricks_kubernetes_mlops_poc_b200 import load_model
    from oracle import reference_pipeline as rp

    d = tmp_path / "artifacts" / "classifier" / "model"
    d.mkdir(parents=True)
    joblib.dump(rf100d6, d / "model.pkl")
    m = load_model(str(tmp_path))
    try:
        df = curated[rp.FEATURES].iloc[:300]
        want_p, _ = rp.oracle_predict(rf100d6, df)
        assert np.abs(np.asarray(m.predict(df)["predictions"]) - want_p).max() <= TOL64
        assert (tmp_path / "forest.b2f.npz").exists()
    finally:
        m.close()
    m2 = load_model(str(tmp_path))  # second load comes from the cached blob
    try:
        assert np.abs(m2.predict_proba1(df) - want_p).max() <= TOL64
    finally:
        m2.close()
