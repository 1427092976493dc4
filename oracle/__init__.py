"""CPU oracle for the credit-default scoring hot path.  TEST INFRASTRUCTURE ONLY.

This package restates, on the CPU, what the reference service computes for
``POST /predict`` (reference ``app/main.py:42-86`` -> ``CustomModel.predict``,
``databricks/src/02-register-model.ipynb:330-353`` -> the sklearn pipeline defined
at ``databricks/src/01-train-model.ipynb:195-231``).

It may be imported ONLY by ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` -- always as the
checker or the timed CPU baseline, never by the product package
(``databricks_kubernetes_mlops_poc_b200``), which has no CPU fallback.

Parity pinning status
---------------------
The reference repo holds NO golden vectors, known-answer tests or model
artefacts for this path (SURVEY.md section 4 / 8c): by the reference's own tests the
parity is "unpinned".  The arithmetic lives in un-vendored third-party
packages (scikit-learn==1.1.1 pinned at reference ``app/requirements.txt:14``;
this image has a newer scikit-learn -- the version is recorded in every golden
file).  The pins we build instead:

* ``oracle.reference_pipeline`` re-creates the reference pipeline definition
  verbatim and re-fits it with fixed seeds on the reference's own
  ``databricks/data/curated.csv`` split; the real library ``predict_proba`` is
  therefore the primary oracle ("outputs of the reference itself run here").
* ``oracle.treewalk`` (numpy) and ``oracle/c/forest_walk.c`` (C) restate the
  compiled part of the algorithm (impute -> one-hot -> float32 cast -> tree walk
  -> float64 mean / GBDT sum + expit) independently and are checked against the
  library to <= 1e-15.
* ``oracle.drift`` restates alibi-detect 0.12.0's ``TabularDrift.feature_score`` on top of the real scipy calls
  (chi-squared over the union of categories, exact two-sample K-S) -- the oracle of the GPU drift detector -- and
  restates scipy's own exact K-S recursion in plain Python, pinned bit for bit to the compiled scipy functions
  (``tests/test_drift_cpu.py``).  alibi-detect itself is neither vendored nor installed: against it the drift path
  is "parity unpinned".  The outlier detector's oracle is sklearn's ``IsolationForest`` itself.
* ``tests/golden/make_golden.py`` freezes inputs + library outputs into
  ``tests/golden/*.npz`` so a machine without a reference checkout can
  re-fit, verify the re-fit reproduces the frozen outputs, and then check the
  CUDA path against them.
"""
