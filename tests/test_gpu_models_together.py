"""Every analysis kernel beside models of other shapes in one process.  A kernel's dynamic shared-memory limit belongs to
the kernel function on the device, not to a model, so a model that needs less must not lower it under a model that
needs more (``set_smem_limit`` in csrc/b2f_api.cu only ever raises it).

The models, fitted once per module:
  A  rf100d6, credit schema (F = 23), TreeSHAP length bucket 9
  B  8 trees of depth 12 on the credit schema, bucket 16 -- the only forest of the suite in that bucket
  C  37 trees of depth 24 (entropy), bucket 24, permutation scores above 48 KB of shared memory
  D  the zoo's ``tiny`` forest (F = 3, bucket 9, beside A) and ``packed_wide_gbdt`` (F = 19, the GBDT aggregation)

The tests: the 16-element TreeSHAP instances against their oracles (B); every analysis output of A, B and C recorded,
checked against the emulators, then D created with everything attached and checked, then A, B and C run again and equal
to the recording bit for bit; the same outputs from two handles called at the same time; and A's predict kernels
afterwards.  The bucket preconditions are asserted on the CPU in tests/test_models_together_cpu.py.

Bars as in the rest of the suite: float64 outputs 1e-12, labels exact, repeated runs bit for bit."""

import threading

import numpy as np
import pandas as pd
import pytest

import schema_zoo as sz

pytestmark = pytest.mark.gpu

TOL = 1e-12
B_PARAMS = dict(n_estimators=8, max_depth=12, random_state=0)  # fitted on curated.iloc[:6000]
C_PARAMS = dict(n_estimators=37, max_depth=24, criterion="entropy", random_state=1)  # fitted on curated.iloc[:6000]
SMALL = ("tiny", "packed_wide_gbdt")


def bucket(max_len: int) -> int:
    """The TreeSHAP instance (explain_kernel in csrc/explain_api.cuh) a path table of longest path ``max_len`` runs."""
    return 9 if max_len <= 9 else (16 if max_len <= 16 else 24)


def _bits(v):
    """The bytes of an output, field by field for a record array (its padding is not part of the result)."""
    v = np.asarray(v)
    return tuple(v[f].tobytes() for f in v.dtype.names) if v.dtype.names else v.tobytes()


def _assert_same_bits(got: dict, want: dict):
    assert got.keys() == want.keys()
    for k in want:
        assert _bits(got[k]) == _bits(want[k]), k


class _Model:
    """One forest's engine with an explainer, a background, an MMD reference and a trust reference attached; a fixed set
    of rows, grids, words and permutations; every analysis output on them, and the emulators' checks of those outputs."""

    def __init__(self, pipe, zoo: bool, frames: dict, k: int, pi_words=None, sample=16, cf_sample=16):
        from databricks_kubernetes_mlops_poc_b200 import dependence, importance, interaction, mmd
        from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
        from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine
        from databricks_kubernetes_mlops_poc_b200.flatten import flatten_explainer, flatten_pipeline, parse_explainer, parse_header

        import knn_walk

        self.pipe, self.zoo, self.k, self.sample, self.cf_sample = pipe, zoo, k, sample, cf_sample
        self.flat = flat = flatten_pipeline(pipe)
        self.blob, self.table = flat.blob, flatten_explainer(pipe, flat)
        self.max_len = parse_explainer(self.table)["max_len"]
        self.enc = enc = RowEncoder(flat)
        feats = flat.all_features
        cats, nums = list(flat.cat_features), list(flat.num_features)
        self.n_cat, self.n_num = len(cats), len(nums)
        self.F = self.n_cat + self.n_num
        self.impute = parse_header(self.blob)["impute"][self.n_cat:self.n_cat + self.n_num]

        self.frame = frames["X"][feats].reset_index(drop=True)
        self.rows = enc.encode_frame(self.frame)
        self.y = np.asarray(frames["y"], dtype=np.int32)
        self.bg_frame = frames["bg"][feats].reset_index(drop=True)
        self.bg_rows = enc.encode_frame(self.bg_frame)
        self.mmd_ref = enc.encode_frame(frames["mmd_ref"][feats])
        self.mmd_mean, self.mmd_scale = mmd.standardization(mmd.numerics(self.mmd_ref, self.n_cat, self.n_num, self.impute))
        self.subsets = mmd.draw_subsets(len(self.mmd_ref), len(self.rows), 16, 0)
        self.knn_ref = enc.encode_frame(frames["knn_ref"][feats])
        self.knn_cls = np.asarray(frames["knn_cls"], dtype=np.int32)
        knn_mean, knn_scale, self.knn_embed = knn_walk.embedding(self.knn_ref, self.n_cat, self.n_num, self.impute)

        # grids of one categorical and two numeric fields from the clean reference frame; pairs of them
        grid_src = frames["mmd_ref"]
        words = {}
        for f in (cats[0], nums[0], nums[-1]):
            words[f] = dependence.encode_grid(enc, f, dependence.grid_from_column(grid_src[f], f in cats, 12))
        self.probes, off = [], 0
        for f, w in words.items():
            self.probes.append((dependence.word_of(enc, f), off, len(w)))
            off += len(w)
        self.grid = np.concatenate(list(words.values()))
        self.pair_probes, pts, off = [], [], 0
        for a, b in ((cats[0], nums[0]), (nums[0], nums[-1])):
            p = interaction.cartesian(words[a][:6], words[b][:6])
            self.pair_probes.append((dependence.word_of(enc, a), dependence.word_of(enc, b), off, len(p)))
            pts.append(p)
            off += len(p)
        self.points = np.concatenate(pts)
        self.cf_words = sorted({self.n_cat + i for i in (0, 1, self.n_num - 1)})
        self.pi_words = list(range(self.F)) if pi_words is None else pi_words
        self.perm = importance.permutations(len(self.rows), 2, 0)

        self.eng = ForestEngine(flat, 0)
        try:
            self.eng.attach_explainer(self.table)
            self.eng.attach_background(self.bg_rows)
            self.sigma = self.eng.attach_mmd_reference(self.mmd_ref, self.mmd_mean, self.mmd_scale)
            self.eng.attach_knn_reference(self.knn_ref, self.knn_cls, knn_mean, knn_scale)
        except BaseException:
            self.eng.close()
            raise

    def _device(self, fn, shape):
        """``fn(rows_dev, n, out_dev)``, one of the *_device entry points, on the rows -> its output."""
        e, r = self.eng, np.ascontiguousarray(self.rows)
        out = np.empty(shape, dtype=np.float64)
        d_rows, d_out = e.device_alloc(r.nbytes), e.device_alloc(out.nbytes)
        try:
            e.h2d(d_rows, r)
            fn(d_rows, len(r), d_out)
            e.sync()
            e.d2h(out, d_out)
        finally:
            e.device_free(d_rows)
            e.device_free(d_out)
        return out

    def permutation_scores(self):
        return self.eng.permutation_scores(self.rows, self.y, self.perm, self.pi_words)

    def knn(self, k=None):
        return self.eng.knn(self.rows, self.k if k is None else k)

    def mmd(self):
        return self.eng.mmd_statistics(self.rows, self.subsets)

    def outputs(self) -> dict:
        e, r, n, F = self.eng, self.rows, len(self.rows), self.F
        out = {}
        out["phi"], out["base"] = e.explain_rows(r)
        out["phi2"], out["base2"] = e.explain_interactions_rows(r)
        out["iphi"], out["ibase"] = e.explain_interventional_rows(r)
        out["phi_dev"] = self._device(e.explain_device, (n, F))
        out["phi2_dev"] = self._device(e.explain_interactions_device, (n, F, F))
        out["iphi_dev"] = self._device(e.explain_interventional_device, (n, F))
        out["pd"] = e.partial_dependence_rows(r, self.probes, self.grid)
        out["pair"] = e.pair_dependence_rows(r, self.pair_probes, self.points)
        out["cf_p"], out["cf"] = e.counterfactual_rows(r, self.cf_words, 0.5)
        out["perm"], out["perm_base"] = self.permutation_scores()
        out["mmd_obs"], out["mmd_perm"] = self.mmd()
        out["knn_d"], out["knn_i"] = self.knn()
        return out

    def check(self, out: dict):
        """``out`` against the emulators on the first rows, and the TreeSHAP identities on every row."""
        import counterfactual_walk
        import dependence_walk
        import importance_walk
        import knn_walk
        import mmd_walk
        import pair_walk
        import path_walk
        import path_walk_interactions
        import path_walk_interventional

        from oracle import treewalk as tw

        s, r = self.sample, self.rows
        gbdt = self.flat.agg_mode != 0
        # TreeSHAP: the path-table emulators, local accuracy, symmetry, row sums; the device forms equal the host forms
        want, wbase = path_walk.explain_paths(self.table, self.blob, r[:s])
        assert abs(out["base"] - wbase) <= TOL and np.abs(out["phi"][:s] - want).max() <= TOL
        want2, _ = path_walk_interactions.explain_interactions_paths(self.table, self.blob, r[:s // 2])
        assert np.abs(out["phi2"][:s // 2] - want2).max() <= TOL and out["base2"] == out["base"]
        iwant, ibase, _ = path_walk_interventional.explain_interventional(self.table, self.blob, r[:s], self.bg_rows)
        assert abs(out["ibase"] - ibase) <= TOL and np.abs(out["iphi"][:s] - iwant).max() <= TOL
        if gbdt:
            X = sz.dense(self.pipe, self.frame) if self.zoo else tw.transform_dense(tw.dump_pipeline(self.pipe), *tw.encode_frame(tw.dump_pipeline(self.pipe), self.frame))
            target = tw.walk_numpy(tw.dump_pipeline(self.pipe), X)[2]
        else:
            target = self.eng.predict_rows(r, np.float64)[0]
        assert np.abs(out["base"] + out["phi"].sum(axis=1) - target).max() <= TOL
        assert np.abs(out["ibase"] + out["iphi"].sum(axis=1) - target).max() <= TOL
        assert np.array_equal(out["phi2"], out["phi2"].transpose(0, 2, 1))
        assert np.abs(out["phi2"].sum(axis=2) - out["phi"]).max() <= TOL
        for k in ("phi", "phi2", "iphi"):
            assert np.array_equal(out[k + "_dev"], out[k]), k
        # one- and two-way dependence
        assert np.abs(out["pd"][:s] - dependence_walk.pd_walk(self.blob, r[:s], self.probes, self.grid)[0]).max() <= TOL
        assert np.abs(out["pair"][:s] - pair_walk.pair_walk(self.blob, r[:s], self.pair_probes, self.points)[0]).max() <= TOL
        # counterfactuals: exact; a GBDT's p1 to 4 ulp (numpy's exp against CUDA's)
        c = self.cf_sample
        wp, wrec = counterfactual_walk.counterfactual(self.blob, r[:c], self.cf_words, 0.5)
        same = lambda a, b: a.shape == b.shape and bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))  # noqa: E731
        close = lambda a, b: np.allclose(a, b, rtol=1e-15, atol=0, equal_nan=True)  # noqa: E731
        assert (close if gbdt else same)(out["cf_p"][:c], wp)
        for f in ("value", "lower", "upper", "lower_p1", "upper_p1"):
            got = out["cf"][f][:c]
            assert same(np.isnan(got), np.isnan(wrec[f])) and (close if gbdt and f.endswith("p1") else same)(got, wrec[f]), f
        # permutation scores: counts exactly, loss sums to 1e-12 relative
        pw, pbase = importance_walk.permutation_scores(self.blob, r, self.y, self.perm, self.pi_words)
        for got, want_ in ((out["perm"], pw), (out["perm_base"], pbase)):
            for f in ("tp", "fp", "tn", "fn", "auc_u2"):
                assert np.array_equal(got[f], want_[f]), f
            for f in ("log_loss_sum", "brier_sum"):
                assert np.allclose(got[f], want_[f], rtol=1e-12, atol=1e-300), f
        # MMD statistics
        zr, cr = mmd_walk.embed(self.mmd_ref, self.n_cat, self.n_num, self.impute, self.mmd_mean, self.mmd_scale)
        zb, cb = mmd_walk.embed(r, self.n_cat, self.n_num, self.impute, self.mmd_mean, self.mmd_scale)
        mw, terms = mmd_walk.statistics(zr, cr, zb, cb, self.subsets, self.sigma)
        assert abs(out["mmd_obs"] - mw[0]) <= TOL * terms[0]
        assert (np.abs(out["mmd_perm"] - mw[1:]) <= TOL * terms[1:]).all()
        # k nearest reference rows: bit for bit
        zq, cq = self.knn_embed(r)
        zk, ck = self.knn_embed(self.knn_ref)
        with np.errstate(over="ignore", invalid="ignore"):
            kd, ki = knn_walk.neighbours(zq, cq, zk, ck, self.knn_cls, self.k)
        assert out["knn_d"].tobytes() == kd.tobytes() and np.array_equal(out["knn_i"], ki)

    def close(self):
        self.eng.close()


def _credit_frames(curated, adversarial, lo=20000):
    from oracle import reference_pipeline as rp

    knn_ref = curated.iloc[1000:3000]
    return dict(
        X=pd.concat([adversarial.iloc[:40], curated[rp.FEATURES].iloc[lo:lo + 24]], ignore_index=True),
        y=np.concatenate([np.arange(40) % 2, curated[rp.TARGET].iloc[lo:lo + 24].to_numpy()]),
        bg=curated[rp.FEATURES].iloc[5000:5024],
        mmd_ref=curated[rp.FEATURES].iloc[:300],
        knn_ref=knn_ref,
        knn_cls=knn_ref[rp.TARGET].to_numpy(),
    )


def _zoo_frames(spec, pipe):
    knn_ref = sz.make_frame(spec, 400, seed=21, target=False)
    return dict(
        X=pd.concat([sz.edge_rows(spec, pipe, n=40), sz.make_frame(spec, 24, seed=9, target=False)], ignore_index=True),
        y=np.arange(64) * 7 % 3 == 0,
        bg=sz.make_frame(spec, 24, seed=31, target=False),
        mmd_ref=sz.make_frame(spec, 300, seed=51, target=False),
        knn_ref=knn_ref,
        knn_cls=np.arange(400) % 3 == 0,
    )


@pytest.fixture(scope="module")
def large(rf100d6, curated, adversarial):
    """A, B and C with everything attached, their outputs recorded before any smaller model exists, and A's forest on a
    tile-kernel and a warp-kernel engine."""
    import os

    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine
    from oracle import reference_pipeline as rp

    fits = {"A": rf100d6,
            "B": rp.fit_reference_pipeline(curated.iloc[:6000], B_PARAMS),
            "C": rp.fit_reference_pipeline(curated.iloc[:6000], C_PARAMS)}
    models, kernels = {}, {}
    try:
        for name, pipe in fits.items():
            models[name] = _Model(pipe, False, _credit_frames(curated, adversarial), 64,
                                  pi_words=[0, 3, 9, 10, 12, 22] if name == "C" else None,
                                  sample=8 if name == "C" else 16, cf_sample=4 if name == "C" else 16)
        assert [bucket(models[n].max_len) for n in "ABC"] == [9, 16, 24]
        assert 10 <= models["B"].max_len <= 16
        for kernel in ("tile", "warp"):
            os.environ["B2F_KERNEL"] = kernel
            try:
                kernels[kernel] = ForestEngine(models["A"].flat, 0)
            finally:
                del os.environ["B2F_KERNEL"]
        recorded = {n: m.outputs() for n, m in models.items()}
        yield models, kernels, recorded
    finally:
        for x in list(models.values()) + list(kernels.values()):
            x.close()


@pytest.fixture(scope="module")
def small(large):
    """D: the tiny and the GBDT zoo models with everything attached, created after A, B and C have recorded."""
    models = {}
    try:
        for name in SMALL:
            spec, pipe = sz.fitted(name)
            models[name] = _Model(pipe, True, _zoo_frames(spec, pipe), 2)
        assert bucket(models["tiny"].max_len) == 9 and models["tiny"].F == 3
        yield models
    finally:
        for m in models.values():
            m.close()


def test_bucket16_against_the_oracles(large, curated, adversarial):
    """The 16-element TreeSHAP instances (K5, K5b, K5c; 96-byte and packed rows; host and device forms) on model B,
    with the bars and samples of test_gpu_schemas.py::test_explainers."""
    import treeshap_interactions as tsi
    import treeshap_interventional as tiv

    from databricks_kubernetes_mlops_poc_b200._cabi import ROWS_PACKED64, ROWS_WORDS24
    from oracle import reference_pipeline as rp
    from oracle import treeshap as ts
    from oracle import treewalk as tw

    models, _, _ = large
    B = models["B"]
    assert bucket(B.max_len) == 16 and B.enc.packed_ok
    eng, enc, pipe = B.eng, B.enc, B.pipe
    df = pd.concat([adversarial, curated[rp.FEATURES].iloc[14000:14000 + 4096 - len(adversarial)]], ignore_index=True)
    rows = enc.encode_frame(df)
    dump, cov = tw.dump_pipeline(pipe), ts.dump_covers(pipe)
    X = tw.transform_dense(dump, *tw.encode_frame(dump, df))
    target, _ = rp.oracle_predict(pipe, df)

    phi, base = eng.explain_rows(rows)
    assert phi.shape == (len(df), 23)
    assert np.abs(base + phi.sum(axis=1) - target).max() <= TOL
    want, wbase = ts.tree_shap(dump, cov, X[:120])
    assert abs(base - wbase) <= TOL and np.abs(phi[:120] - want).max() <= TOL

    n2 = 1024
    phi2, base2 = eng.explain_interactions_rows(rows[:n2])
    assert phi2.shape == (n2, 23, 23) and abs(base2 - base) <= TOL
    assert np.array_equal(phi2, phi2.transpose(0, 2, 1))
    assert np.abs(phi2.sum(axis=2) - phi[:n2]).max() <= TOL
    want2, _ = tsi.tree_shap_interactions(dump, cov, X[:24])
    assert np.abs(phi2[:24] - want2).max() <= TOL

    iphi, ibase = eng.explain_interventional_rows(rows)  # against the 24 background rows attached by the fixture
    assert np.abs(ibase + iphi.sum(axis=1) - target).max() <= TOL
    Z = tw.transform_dense(dump, *tw.encode_frame(dump, B.bg_frame))
    want, wbase = tiv.interventional_shap(dump, X[:40], Z)
    assert abs(ibase - wbase) <= TOL and np.abs(iphi[:40] - want).max() <= TOL

    pk = enc.pack_rows(rows)
    assert np.array_equal(eng.explain_rows(pk)[0], phi)
    assert np.array_equal(eng.explain_interactions_rows(pk[:n2])[0], phi2)
    assert np.array_equal(eng.explain_interventional_rows(pk)[0], iphi)

    host = {"phi": phi, "phi2": phi2, "iphi": iphi}
    variants = {"phi": (eng.explain_rows, eng.explain_device, (23,)),
                "phi2": (eng.explain_interactions_rows, eng.explain_interactions_device, (23, 23)),
                "iphi": (eng.explain_interventional_rows, eng.explain_interventional_device, (23,))}
    for n in (33, n2):  # several path ranges and the finishing kernel; one range
        for k, (on_host, fn, tail) in variants.items():
            want = on_host(rows[:n])[0]  # the host form of the same batch
            for fmt, r in ((ROWS_WORDS24, rows[:n]), (ROWS_PACKED64, pk[:n])):
                r = np.ascontiguousarray(r)
                got = np.empty((n,) + tail, dtype=np.float64)
                d_rows, d_out = eng.device_alloc(r.nbytes), eng.device_alloc(got.nbytes)
                try:
                    eng.h2d(d_rows, r)
                    fn(d_rows, n, d_out, fmt)
                    eng.sync()
                    eng.d2h(got, d_out)
                finally:
                    eng.device_free(d_rows)
                    eng.device_free(d_out)
                assert np.array_equal(got, want), (k, n, fmt)

    # small batches run several path ranges and the finishing kernels: the same values to the last bit or two
    for n in (1, 31, 33):
        for k, (fn, _, _) in variants.items():
            got = fn(rows[:n])[0]
            assert np.abs(got - host[k][:n]).max() <= 1e-14, (k, n)
            assert np.array_equal(got, fn(rows[:n])[0]), (k, n)
    # one interaction batch past B2F_INTER_CHUNK_ROWS (16 384 rows): the second chunk's row is row 0 again
    big = np.concatenate([rows] * 5)[:16385]
    phi2_big, _ = eng.explain_interactions_rows(big)
    assert np.array_equal(phi2_big, phi2_big.transpose(0, 2, 1))
    assert np.abs(phi2_big.sum(axis=2) - eng.explain_rows(big)[0]).max() <= TOL
    assert np.abs(phi2_big[:n2] - phi2).max() <= 1e-14
    assert np.abs(phi2_big[16384] - phi2[0]).max() <= 1e-14


def test_smaller_models_leave_larger_models_outputs_alone(large, small):
    """A, B and C's outputs are right; D attaches everything (every shared-memory limit it sets is below A, B and C's)
    and its outputs are right; then A, B and C give their recorded outputs bit for bit."""
    models, _, recorded = large
    for name, m in models.items():
        m.check(recorded[name])
    for name, m in small.items():
        m.check(m.outputs())
    for name, m in models.items():
        _assert_same_bits(m.outputs(), recorded[name])


def _together(job_a, job_b, calls=8):
    """Each job alone, then both from two threads started together, ``calls`` times each: every result equals the job's
    result alone, bit for bit."""
    alone = [job_a(), job_b()]
    barrier = threading.Barrier(2, timeout=120)
    results, errors = [[], []], []

    def run(i, job):
        try:
            barrier.wait()
            for _ in range(calls):
                results[i].append(job())
        except BaseException as e:  # re-raised below, in the test's thread
            errors.append(e)

    threads = [threading.Thread(target=run, args=(i, job)) for i, job in enumerate((job_a, job_b))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errors:
        raise errors[0]
    for i in range(2):
        assert len(results[i]) == calls
        for got in results[i]:
            assert [_bits(x) for x in got] == [_bits(x) for x in alone[i]], i


def test_two_handles_at_the_same_time(large, small):
    """Per-call limits: a depth-24 and a depth-5 forest's permutation scores, k = 64 on 23 fields and k = 2 on 3, and the
    MMD statistics of 23 and 3 fields, each pair on two handles at once."""
    models, _, _ = large
    tiny = small["tiny"]
    _together(models["C"].permutation_scores, tiny.permutation_scores)
    _together(lambda: models["A"].knn(64), lambda: tiny.knn(2))
    _together(models["A"].mmd, tiny.mmd)


def test_predict_kernels_beside_the_analysis_models(large, small, curated, adversarial):
    """After the attaches and calls above, A's tile, warp and rank kernels still give the library's answers."""
    from oracle import reference_pipeline as rp

    models, kernels, _ = large
    A = models["A"]
    df = pd.concat([adversarial, curated[rp.FEATURES].iloc[:3000]], ignore_index=True)
    want_p, want_l = rp.oracle_predict(A.pipe, df)
    rows = A.enc.encode_frame(df)
    for kernel, eng in kernels.items():
        p, lab = eng.predict_rows(rows, np.float64)
        assert np.abs(p - want_p).max() <= TOL and (lab == want_l).all(), kernel
    assert A.eng.info()["rank_ok"]
    l0 = A.eng.info()["launches_rank"]
    p, lab = A.eng.predict_rows(A.enc.rank_rows(rows), np.float64)
    assert np.abs(p - want_p).max() <= TOL and (lab == want_l).all()
    assert A.eng.info()["launches_rank"] > l0
