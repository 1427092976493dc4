"""Back-to-back launches of the rank kernel on one stream.  Consecutive launches overlap through programmatic dependent
launch, and each CTA reads its rows and walks before it waits for the previous launch.  These tests check what a caller
relies on: a chain computes exactly what isolated launches compute, and the last launch writing a buffer wins.  Both
forms of the kernel (resident forest, streamed forest) under the three launch set-ups: the dependency wait before the
stores (default), the wait at kernel entry (B2F_RANK_WAIT_FIRST=1) and no programmatic launch (B2F_NO_PDL=1)."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N = 65536  # the benchmark's batch: 2 048 tiles of 32 rows over every SM
POOL = 32
STEPS = 200
MODES = {"wait_before_stores": None, "wait_first": ("B2F_RANK_WAIT_FIRST", "1"), "no_pdl": ("B2F_NO_PDL", "1")}


@pytest.fixture(scope="module")
def gbdt100d6(curated):
    """The benchmark's model shape (100 trees, depth 6: the rank layout stays resident in shared memory)."""
    from oracle import reference_pipeline as rp

    tr, _ = rp.reference_split(curated)
    tr = tr.iloc[:4000]
    return rp.fit_gbdt_pipeline(tr, tr[rp.TARGET].to_numpy(), dict(n_estimators=100, max_depth=6, random_state=0))


def _engine(pipe, mode, monkeypatch):
    """A fresh engine: the launch set-up is read from the environment when the model is created."""
    from databricks_kubernetes_mlops_poc_b200 import flatten
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine

    for name, _ in filter(None, MODES.values()):
        monkeypatch.delenv(name, raising=False)
    if MODES[mode]:
        monkeypatch.setenv(*MODES[mode])
    flat = flatten.flatten_pipeline(pipe)
    return ForestEngine(flat, 0), RowEncoder(flat)


def _ranked_pool(enc, curated, seed):
    """(POOL, N, words) ranked rows: N rows drawn from the curated table, each batch a different permutation of them."""
    from oracle import reference_pipeline as rp

    rng = np.random.default_rng(seed)
    base = enc.rank_rows(enc.encode_frame(curated[rp.FEATURES].iloc[rng.integers(0, len(curated), N)]))
    return np.stack([base[rng.permutation(N)] for _ in range(POOL)])


def _bits_equal(a, b):
    return a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("which", ["gbdt100d6", "rf500d8"])
def test_chained_launches_equal_isolated(curated, gbdt100d6, rf500d8, which, mode, monkeypatch):
    from databricks_kubernetes_mlops_poc_b200._cabi import ROWS_RANKED

    pipe = {"gbdt100d6": gbdt100d6, "rf500d8": rf500d8}[which]
    eng, enc = _engine(pipe, mode, monkeypatch)
    d = []
    try:
        info = eng.info()
        assert info["rank_ok"] and bool(info["rank_stream"]) == (which == "rf500d8")
        rows = _ranked_pool(enc, curated, 11)
        rb = rows.shape[2] * 4
        d_rows, d_p, d_l = (eng.device_alloc(nb) for nb in (rows.nbytes, POOL * N * 8, POOL * N * 4))
        d += [d_rows, d_p, d_l]
        eng.h2d(d_rows, rows)
        # isolated: one launch per batch, each followed by a synchronise
        for b in range(POOL):
            eng.predict_device(d_rows + b * N * rb, N, d_p + b * N * 8, True, d_l + b * N * 4, fmt=ROWS_RANKED)
            eng.sync()
        want_p, want_l = np.empty(POOL * N), np.empty(POOL * N, dtype=np.int32)
        eng.d2h(want_p, d_p)
        eng.d2h(want_l, d_l)
        assert np.isfinite(want_p).all()
        # chained: STEPS launches back to back over the pool, no event or synchronise in between
        eng.h2d(d_p, np.full(POOL * N, np.nan))
        eng.h2d(d_l, np.full(POOL * N, -1, dtype=np.int32))
        l0 = eng.info()["launches_rank"]
        eng.predict_stream_timed(d_rows, N, POOL, d_p, True, d_l, STEPS, fmt=ROWS_RANKED, per_launch=False)
        assert eng.info()["launches_rank"] - l0 == STEPS
        got_p, got_l = np.empty_like(want_p), np.empty_like(want_l)
        eng.d2h(got_p, d_p)
        eng.d2h(got_l, d_l)
        assert _bits_equal(got_p, want_p) and _bits_equal(got_l, want_l)
    finally:
        for p in d:
            eng.device_free(p)
        eng.close()


@pytest.mark.parametrize("mode", ["wait_before_stores", "wait_first"])
@pytest.mark.parametrize("which", ["gbdt100d6", "rf500d8"])
def test_last_launch_into_a_buffer_wins(curated, gbdt100d6, rf500d8, which, mode, monkeypatch):
    """64 launches without a synchronise alternate two batches A, B into the SAME output buffers, B last."""
    from databricks_kubernetes_mlops_poc_b200._cabi import ROWS_RANKED

    pipe = {"gbdt100d6": gbdt100d6, "rf500d8": rf500d8}[which]
    eng, enc = _engine(pipe, mode, monkeypatch)
    d = []
    try:
        rows = _ranked_pool(enc, curated, 12)[:2]
        rb = rows.shape[2] * 4
        d_rows, d_p, d_l = (eng.device_alloc(nb) for nb in (rows.nbytes, N * 8, N * 4))
        d += [d_rows, d_p, d_l]
        eng.h2d(d_rows, rows)
        want = {}
        for b in (0, 1):
            eng.predict_device(d_rows + b * N * rb, N, d_p, True, d_l, fmt=ROWS_RANKED)
            eng.sync()
            p, lab = np.empty(N), np.empty(N, dtype=np.int32)
            eng.d2h(p, d_p)
            eng.d2h(lab, d_l)
            want[b] = (p, lab)
        assert (want[0][0] != want[1][0]).mean() > 0.5, "the two batches must score differently"
        for i in range(64):
            b = i % 2  # ... A, B: the last launch scores B
            eng.predict_device(d_rows + b * N * rb, N, d_p, True, d_l, fmt=ROWS_RANKED)
        eng.sync()
        got_p, got_l = np.empty(N), np.empty(N, dtype=np.int32)
        eng.d2h(got_p, d_p)
        eng.d2h(got_l, d_l)
        assert _bits_equal(got_p, want[1][0]) and _bits_equal(got_l, want[1][1])
    finally:
        for p in d:
            eng.device_free(p)
        eng.close()
