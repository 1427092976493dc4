"""Measurement helper: timeline of one `B200Model.predict(DataFrame of 65 536 rows)` -- per chunk, when it was encoded, when its GPU
work was enqueued (b2f_scorer_trace) and when the caller had it back and its part of the list built.  Median over TRACE_STEPS."""
import json, os, sys, time
OUT = os.environ.get("B2F_TOOL_OUT", "tools_out")  # where the result file goes
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
from databricks_kubernetes_mlops_poc_b200 import _cabi, flatten, training
from databricks_kubernetes_mlops_poc_b200._pylists import ListBuilder
from databricks_kubernetes_mlops_poc_b200.model import B200Model
from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES

dist = bench.Dist(1, False, solo=True)
MODEL = os.environ.get("TRACE_MODEL", "gbdt100d6")
pipe, base = bench.get_pipeline(MODEL, dist)
flat = flatten.flatten_pipeline(pipe)
pv, pc, pn = training.synth_arrays(base, bench.BATCH, bench.DATA_SEED)
df = training.arrays_to_frame(pv, pc, pn)[ALL_FEATURES]
model = B200Model(flat, devices=[0], host_threads=int(os.environ.get("TRACE_THREADS", "0")))
for _ in range(20):
    model.predict(df)
sc = model.replicas[0]._scorer
lib = _cabi.load_library()
K = int(os.environ.get("TRACE_STEPS", "200"))
chunk_rows = int(os.environ.get("TRACE_CHUNK_ROWS", "0"))
rec = []
for _ in range(K):
    t0 = time.perf_counter()
    cols = model.encoder.frame_columns(df)
    t1 = time.perf_counter()
    n_chunks = sc.start(len(df), cols, out_mode=1, chunk_rows=chunk_rows)
    t2 = time.perf_counter()
    out = sc.results()
    step = sc.chunk_rows
    bounds = sc.bounds
    lb = ListBuilder(len(df))
    back, built = [], []
    for c in range(n_chunks):
        sc.wait(c)
        back.append(time.perf_counter())
        lb.fill(bounds[c], out[bounds[c]:bounds[c + 1]])
        built.append(time.perf_counter())
    tr = np.zeros(2 * n_chunks)
    lib.b2f_scorer_trace(sc._h, _cabi.ptr(tr), n_chunks)
    rec.append({"columns": 1e6 * (t1 - t0), "start_call": 1e6 * (t2 - t1), "encoded": tr[0::2].tolist(), "enqueued": tr[1::2].tolist(),
                "back": [1e6 * (b - t1) for b in back], "built": [1e6 * (b - t1) for b in built], "total": 1e6 * (built[-1] - t0)})
med = lambda key: np.median(np.asarray([r[key] for r in rec]), axis=0)
res = {"model": MODEL, "row_format": sc.last_fmt, "threads": sc.threads, "chunks": n_chunks, "chunk_rows": int(step), "bounds": list(bounds), "us_since_start": {k: np.round(med(k), 1).tolist() for k in ("encoded", "enqueued", "back", "built")},
       "columns_us": float(med("columns")), "start_call_us": float(med("start_call")), "total_us": float(med("total"))}
print(json.dumps(res, indent=1))
os.makedirs(OUT, exist_ok=True)
json.dump(res, open(os.path.join(OUT, f"scorer_trace_{MODEL}_f{sc.last_fmt}_c{chunk_rows}.json"), "w"), indent=1)
model.close()
