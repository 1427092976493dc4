"""The resident rank kernel walks only a forest's real tree groups and reads every tree's top two levels from its parameter
block (RParams::top_root / top_kids, B2F_RANK_TOP_TREES trees at most); larger forests stream.  These tests hold the kernel
to the numpy emulator of the rank layout (tests/rank_walk.py) across the shapes that change with that: tree counts that
leave 0 .. 3 stub trees in the last group, stumps (no level 1) and deep trees, the table's capacity plus one, batch sizes
from one row to two rounds per CTA, and back-to-back launches into one output buffer.  The emulator runs on its own
(against the library) without a GPU first, so a failure on the GPU points at the kernel, not at the layout."""

import numpy as np
import pytest

from rank_walk import walk_rank_layout

TOP_TREES = 288  # B2F_RANK_TOP_TREES (csrc/forest_predict_rank.cuh)
TOL64 = 1e-12
# (trees, depth): 1 .. 5 and 33 / 100 / 101 trees leave 3, 1, 0, 3 / 0 / 3 stub trees in the last group of 4; depth 1 is a
# stump (no level 1), depth 8 the deepest rank layout; TOP_TREES + 1 trees must stream (or refuse the rank layout)
FORESTS = [(1, 6), (3, 6), (4, 6), (5, 6), (33, 6), (100, 6), (101, 6), (5, 1), (33, 2), (33, 8), (TOP_TREES + 1, 3)]
BATCHES = (1, 31, 33, 4096, 65536, 90000)  # 90 000 > 132 SMs x 16 tiles x 32 rows: a second round per CTA on an H100
N_ROWS = max(BATCHES)


def _fid(f):
    return f"{f[0]}x{f[1]}"


@pytest.fixture(scope="module")
def train(curated):
    from oracle import reference_pipeline as rp

    tr, _ = rp.reference_split(curated)
    return tr.iloc[:3000]


_PIPES = {}


def _pipe(train, forest):
    """GBDT (the benchmark's model family) with `trees` trees of depth `depth`, fitted once per module."""
    from oracle import reference_pipeline as rp

    if forest not in _PIPES:
        trees, depth = forest
        _PIPES[forest] = rp.fit_gbdt_pipeline(train, train[rp.TARGET].to_numpy(), dict(n_estimators=trees, max_depth=depth, random_state=0))
    return _PIPES[forest]


def _enc(pipe):
    from databricks_kubernetes_mlops_poc_b200 import flatten
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder

    flat = flatten.flatten_pipeline(pipe)
    return flat, RowEncoder(flat)


@pytest.fixture(scope="module")
def frame(curated):
    """N_ROWS reference rows: the curated table, permuted, repeated."""
    from oracle import reference_pipeline as rp

    rng = np.random.default_rng(5)
    return curated[rp.FEATURES].iloc[rng.integers(0, len(curated), N_ROWS)].reset_index(drop=True)


@pytest.mark.parametrize("forest", FORESTS, ids=_fid)
def test_emulator_matches_library(train, curated, forest):
    """CPU only: the rank layout of each forest, walked by the emulator, scores like sklearn."""
    from oracle import reference_pipeline as rp

    pipe = _pipe(train, forest)
    flat, enc = _enc(pipe)
    info = enc.rank_info()
    assert info.ok and info.n_trees == forest[0] and info.depth == forest[1]
    df = curated[rp.FEATURES].iloc[:2000]
    want_p, want_l = rp.oracle_predict(pipe, df)
    p, lab = walk_rank_layout(enc.rank_layout(), info, flat.blob, enc.rank_rows(enc.encode_frame(df)))
    assert np.abs(p - want_p).max() <= TOL64 and (lab == want_l).all()


@pytest.mark.gpu
@pytest.mark.parametrize("forest", FORESTS, ids=_fid)
def test_rank_kernel_matches_emulator(train, frame, forest):
    """Every batch size, resident or streamed as the tree count decides, against the emulator; run to run bit-identical."""
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine

    flat, enc = _enc(_pipe(train, forest))
    info = enc.rank_info()
    rows = enc.rank_rows(enc.encode_frame(frame))
    want_p, want_l = walk_rank_layout(enc.rank_layout(), info, flat.blob, rows)
    eng = ForestEngine(flat, 0)
    try:
        ei = eng.info()
        assert ei["rank_ok"]
        assert bool(ei["rank_stream"]) == (forest[0] > TOP_TREES)  # every other forest here fits shared memory
        for n in BATCHES:
            p, lab = eng.predict_rows(rows[:n], np.float64)
            assert np.abs(p - want_p[:n]).max() <= TOL64, (n, float(np.abs(p - want_p[:n]).max()))
            assert (lab == want_l[:n]).all(), n
        p2, l2 = eng.predict_rows(rows, np.float64)
        assert np.array_equal(p.view(np.uint64), p2.view(np.uint64)) and (lab == l2).all()
    finally:
        eng.close()


@pytest.mark.gpu
def test_over_capacity_forest_refused_when_resident_is_forced(train, monkeypatch):
    """B2F_RANK_STREAM=0 forbids the streamed kernel: a forest the resident kernel cannot take gets no rank kernel."""
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine

    monkeypatch.setenv("B2F_RANK_STREAM", "0")
    flat, _ = _enc(_pipe(train, (TOP_TREES + 1, 3)))
    eng = ForestEngine(flat, 0)
    try:
        assert not eng.info()["rank_ok"]
    finally:
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("forest", [(5, 6), (101, 6), (5, 1), (TOP_TREES + 1, 3)], ids=_fid)
@pytest.mark.parametrize("n", [33, 90000])
def test_chained_launches_last_one_wins(train, frame, forest, n):
    """16 launches without a synchronise alternate two batches into the same output buffers; the last one's scores stay."""
    from databricks_kubernetes_mlops_poc_b200._cabi import ROWS_RANKED
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine

    flat, enc = _enc(_pipe(train, forest))
    info = enc.rank_info()
    rows = enc.rank_rows(enc.encode_frame(frame))
    batches = np.stack([rows[:n], rows[::-1][:n]])
    want = [walk_rank_layout(enc.rank_layout(), info, flat.blob, b) for b in batches]
    eng = ForestEngine(flat, 0)
    d = []
    try:
        rb = batches.shape[2] * 4
        d_rows, d_p, d_l = (eng.device_alloc(nb) for nb in (batches.nbytes, n * 8, n * 4))
        d += [d_rows, d_p, d_l]
        eng.h2d(d_rows, batches)
        for i in range(16):
            eng.predict_device(d_rows + (i % 2) * n * rb, n, d_p, True, d_l, fmt=ROWS_RANKED)  # ... A, B: B is last
        eng.sync()
        p, lab = np.empty(n), np.empty(n, dtype=np.int32)
        eng.d2h(p, d_p)
        eng.d2h(lab, d_l)
        assert np.abs(p - want[1][0]).max() <= TOL64 and (lab == want[1][1]).all()
    finally:
        for q in d:
            eng.device_free(q)
        eng.close()
