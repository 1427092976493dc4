"""The kernels' numpy emulators and the host encoders on request schemas other than the credit-default one
(tests/schema_zoo.py), against the library and the oracles, on a CPU-only box.  These run before the GPU file
(tests/test_gpu_schemas.py) so that a GPU failure on a schema points at a kernel, not at the flattener, the ranker or the
encoder.

Every schema's reason to exist is asserted first (test_schema_preconditions), so a change of the synthetic data cannot
make the other tests pass vacuously."""

import os
import subprocess
import sys

import numpy as np
import pytest

import schema_zoo as sz
from blob_walk import walk_blob
from path_walk import explain_paths
from path_walk_interactions import explain_interactions_paths
from path_walk_interventional import explain_interventional
from rank_walk import walk_rank_layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-12

MODELS = ["packed_wide", "packed_wide_gbdt", "rank_wide", "rank_wide_129", "tiny", "tiny_gbdt", "over16"]


def _enc(pipe):
    from databricks_kubernetes_mlops_poc_b200 import flatten
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder

    flat = flatten.flatten_pipeline(pipe)
    return flat, RowEncoder(flat)


def _frames(spec, pipe):
    return [sz.make_frame(spec, 1500, seed=5, target=False), sz.edge_rows(spec, pipe)]


def test_schema_preconditions():
    from oracle import treewalk as tw

    # packed_wide: the packed row, field 4 (bits 28..34) with code + 1 >= 16 on both sides of the word boundary, and
    # tested codes >= 32 / 64 / 96 (the path table's mask words y / z / w); no rank layout (tested codes >= 64)
    spec, pipe = sz.fitted("packed_wide")
    flat, enc = _enc(pipe)
    assert enc.packed_ok and [len(c) for c in flat.categories] == spec[0]
    df = sz.make_frame(spec, 1500, seed=5, target=False)
    rows = enc.encode_frame(df)
    assert (rows.view(np.int32)[:, 4] + 1 >= 16).any() and (rows.view(np.int32)[:, 4] + 1 >= 64).any()
    packed = enc.pack_rows(rows)
    assert (packed[:, 1] & 0x7).any() and (packed[:, 0] >> 28).any()  # field 4's bits in both words
    for m in ("packed_wide", "packed_wide_gbdt", "packed_wide_shallow"):
        codes = [c for _, c in sz.tested_pairs(sz.fitted(m)[1])]
        assert max(codes) >= 96 and any(64 <= c < 96 for c in codes) and any(32 <= c < 64 for c in codes), m
        info = _enc(sz.fitted(m)[1])[1].rank_info()
        assert not info.ok and (b"64-bit per-feature mask" in info.why or b"more than 128" in info.why), info.why
    # rank_wide: 16 categoricals in the 8-byte block, codes 63 and 32..62 tested, exactly 128 pseudo-features; 129 refused
    spec, pipe = sz.fitted("rank_wide")
    flat, enc = _enc(pipe)
    info = enc.rank_info()
    assert len(spec[0]) == 16 and info.ok and info.cat_bytes == 8 and info.row_bytes == 24
    assert ((spec[1] + 1) & ~1) + info.n_pairs == 128
    codes = [c for _, c in sz.tested_pairs(pipe)]
    assert 63 in codes and any(32 <= c < 63 for c in codes)
    info129 = _enc(sz.fitted("rank_wide_129")[1])[1].rank_info()
    assert not info129.ok and b"more than 128" in info129.why and info129.n_pairs == 121
    # tiny: F = 3 fields, fewer than the interaction kernel's 8 warps
    spec, pipe = sz.fitted("tiny")
    assert len(spec[0]) + spec[1] == 3 and tw.dump_pipeline(pipe)["n_trees"] == 20
    # over16: no rank layout, no native encoder
    spec, pipe = sz.fitted("over16")
    flat, enc = _enc(pipe)
    assert len(spec[0]) == 17 and not enc.packed_ok
    info = enc.rank_info()
    assert not info.ok and b"16 categorical" in info.why
    assert enc._native_handle() is None  # b2f_encoder_create refuses more than 16 categoricals
    # moments schemas: every NC = 0..4 at some vector q > 0
    seen = {min(4, max(0, n_cat - 4 * q)) for n_cat in sz.MOMENT_N_CAT for q in range(1, 6)}
    assert seen == {0, 1, 2, 3, 4}


@pytest.mark.parametrize("name", MODELS)
def test_blob_and_rank_walks_match_library(name):
    spec, pipe = sz.fitted(name)
    flat, enc = _enc(pipe)
    info = enc.rank_info()
    for df in _frames(spec, pipe):
        want_p, want_l = sz.predict(pipe, df)
        rows = enc.encode_frame(df)
        p, l = walk_blob(flat.blob, rows)
        assert np.abs(p - want_p).max() <= TOL and (l == want_l).all()
        if info.ok:
            p, l = walk_rank_layout(enc.rank_layout(), info, flat.blob, enc.rank_rows(rows))
            assert np.abs(p - want_p).max() <= TOL and (l == want_l).all()


@pytest.mark.parametrize("name", MODELS + ["packed_wide_shallow"])
def test_path_walk_matches_oracle(name):
    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer
    from oracle import treeshap as ts
    from oracle import treewalk as tw

    spec, pipe = sz.fitted(name)
    flat, enc = _enc(pipe)
    table = flatten_explainer(pipe, flat)
    dump, cov = tw.dump_pipeline(pipe), ts.dump_covers(pipe)
    for df in _frames(spec, pipe):
        df = df.iloc[:150]
        phi, base = explain_paths(table, flat.blob, enc.encode_frame(df))
        X = sz.dense(pipe, df)
        want, wbase = ts.tree_shap(dump, cov, X)
        assert abs(base - wbase) <= TOL and np.abs(phi - want).max() <= TOL
        p, _, raw = tw.walk_numpy(dump, X)
        assert np.abs(base + phi.sum(axis=1) - (p if flat.agg_mode == 0 else raw)).max() <= TOL
        if name in ("packed_wide_shallow", "tiny_gbdt"):
            bphi, bbase = ts.brute_force_shap(dump, cov, X)
            assert np.abs(phi - bphi).max() <= TOL and abs(base - bbase) <= TOL


@pytest.mark.parametrize("name", ["packed_wide_shallow", "rank_wide", "tiny", "tiny_gbdt"])
def test_interaction_and_interventional_walks_match_oracles(name):
    import treeshap_interactions as tsi
    import treeshap_interventional as tiv

    from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer
    from oracle import treeshap as ts
    from oracle import treewalk as tw

    spec, pipe = sz.fitted(name)
    flat, enc = _enc(pipe)
    table = flatten_explainer(pipe, flat)
    dump, cov = tw.dump_pipeline(pipe), ts.dump_covers(pipe)
    edge = sz.edge_rows(spec, pipe)
    x, z = edge.iloc[:30], sz.make_frame(spec, 12, seed=9, target=False)
    X, Z = sz.dense(pipe, x), sz.dense(pipe, z)
    rows = enc.encode_frame(x)
    phi2, base = explain_interactions_paths(table, flat.blob, rows)
    want2, wbase = tsi.tree_shap_interactions(dump, cov, X)
    assert abs(base - wbase) <= TOL and np.abs(phi2 - want2).max() <= TOL
    assert np.array_equal(phi2, phi2.transpose(0, 2, 1))
    phi, _ = explain_paths(table, flat.blob, rows)
    assert np.abs(phi2.sum(axis=2) - phi).max() <= TOL
    iphi, ibase, _ = explain_interventional(table, flat.blob, rows, enc.encode_frame(z))
    want, wbase = tiv.interventional_shap(dump, X, Z)
    assert abs(ibase - wbase) <= TOL and np.abs(iphi - want).max() <= TOL
    assert np.abs(ibase + iphi.sum(axis=1) - tiv.output(dump, X)).max() <= TOL


_ENCODER_CODE = r"""
import hashlib, sys
import numpy as np
import pandas as pd
sys.path.insert(0, %r); sys.path.insert(0, %r)
import schema_zoo as sz
from databricks_kubernetes_mlops_poc_b200 import flatten
from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
h = hashlib.sha256()
for name in ("packed_wide", "rank_wide"):
    spec, pipe = sz.fitted(name)
    enc = RowEncoder(flatten.flatten_pipeline(pipe))
    assert enc._native_handle() is not None
    edge = sz.edge_rows(spec, pipe, n=600)
    big = pd.concat([sz.make_frame(spec, 5000, seed=11, target=False), edge], ignore_index=True)
    arrow = big.copy()
    for c in sz.cat_names(spec):
        arrow[c] = arrow[c].astype("string[pyarrow]")
    # the portable encoder's view of the same frame: Arrow nulls are NaN (the imputer's "missing" semantics)
    portable = arrow.copy()
    for c in sz.cat_names(spec):
        portable[c] = pd.Series(arrow[c].to_numpy(dtype=object, na_value=np.nan), dtype=object)
    for n in (129, 143, 1024 + 7, 4096 + 15, len(big)):  # remainders of the encoder's 16-row blocks
        a, p = arrow.iloc[:n], portable.iloc[:n]
        want = enc.encode_frame(p)  # object columns: always the portable path
        # the native encoder itself, called directly so that a silent fall-back cannot compare the portable path with itself
        got = np.empty_like(want)
        assert enc._encode_native(a, got, fmt=0), (name, n, "96-byte rows refused")
        assert np.array_equal(got, want), (name, n, "96-byte rows")
        h.update(got.tobytes())
        if enc.packed_ok:
            got = np.empty((n, 16), dtype=np.uint32)
            assert enc._encode_native(a, got, fmt=1), (name, n, "packed rows refused")
            assert np.array_equal(got, enc.pack_rows(want)), (name, n, "packed rows")
            h.update(got.tobytes())
        if enc.ranked_ok:
            got = np.empty((n, enc.ranked_row_words), dtype=np.uint32)
            assert enc._encode_native(a, got, fmt=2), (name, n, "ranked rows refused")
            assert np.array_equal(got, enc.rank_rows(want)), (name, n, "ranked rows")
            h.update(got.tobytes())
print(h.hexdigest())
"""


def test_native_encoder_matches_portable():
    """The native encoder (csrc/row_encoder.h + host_simd.cpp: 9 fields across the packed word boundary, 16 fields in the
    ranked 8-byte block) writes the portable encoder's 96-byte, packed and ranked rows, at every SIMD level (B2F_SIMD caps
    it: 0 scalar, 1 at most AVX2, 2 AVX-512 where the CPU has it) and at every 16-row block remainder; all levels write
    the same bytes."""
    code = _ENCODER_CODE % (ROOT, os.path.join(ROOT, "tests"))
    digests = {}
    for level in ("0", "1", "2"):
        out = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, B2F_SIMD=level), capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, (level, out.stderr[-3000:])
        digests[level] = out.stdout.strip().splitlines()[-1]
    assert len(set(digests.values())) == 1, digests


def test_over16_portable_encoder():
    """17 categoricals: the native encoder refuses the schema, so large frames take the portable path and still encode
    every field (no field beyond the 16th dropped)."""
    spec, pipe = sz.fitted("over16")
    flat, enc = _enc(pipe)
    df = sz.make_frame(spec, 700, seed=3, target=False)
    rows = enc.encode_frame(df)
    codes, nums = sz.make_codes_nums(spec, 700, 3)
    assert np.array_equal(rows.view(np.int32)[:, :17], codes)
    assert np.array_equal(rows.view(np.float32)[:, 17:23], nums.astype(np.float32))
    p, l = walk_blob(flat.blob, rows)
    want_p, want_l = sz.predict(pipe, df)
    assert np.abs(p - want_p).max() <= TOL and (l == want_l).all()
