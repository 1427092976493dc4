"""Measurement helper: synchronous C-ABI call (b2f_predict_pairs, 65 536 pre-encoded ranked rows in pinned memory) under different
chunk plans (B2F_CHUNK_PLAN: shares of the batch in 1/1024ths, the last chunk takes the rest; "1024" = one chunk)."""
import json, os, sys, time
OUT = os.environ.get("B2F_TOOL_OUT", "tools_out")  # where the result file goes
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
from databricks_kubernetes_mlops_poc_b200 import _cabi, flatten, training
from databricks_kubernetes_mlops_poc_b200._cabi import SCORED_DTYPE
from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine

dist = bench.Dist(1, False, solo=True)
pipe, base = bench.get_pipeline("gbdt100d6", dist)
flat = flatten.flatten_pipeline(pipe)
enc = RowEncoder(flat)
_, codes, nums = training.synth_arrays(base, 4 * 65536, 5)
rows24 = enc.encode_arrays(codes, nums)
res = {}
for fmt_name in ("ranked", "packed64"):
    for plan in ("1024", "768", "512", "640", "384,384", "256,256,256", "512,256", "256,512", "128,384,384"):
        os.environ["B2F_CHUNK_PLAN"] = plan
        eng = ForestEngine(flat, device=0)
        rows = enc.rank_rows(rows24) if fmt_name == "ranked" else enc.pack_rows(rows24)
        h = eng.pinned("rows", rows.nbytes).view(np.uint32, rows.shape)
        h[:] = rows
        out = eng.pinned("out", len(rows) * 8).view(SCORED_DTYPE, (len(rows),))
        t = []
        for i in range(220):
            b = i % 4
            t0 = time.perf_counter()
            eng.predict_pairs(h[b * 65536:(b + 1) * 65536], out[b * 65536:(b + 1) * 65536])
            t.append(time.perf_counter() - t0)
        t = np.asarray(t[20:])
        res[f"{fmt_name}:{plan}"] = {"p50_us": 1e6 * float(np.median(t)), "mean_us": 1e6 * float(t.mean()), "rows_per_s": 65536 / float(t.mean())}
        print(fmt_name, plan, {k: round(v, 1) for k, v in res[f"{fmt_name}:{plan}"].items()}, flush=True)
        eng.close()
os.makedirs(OUT, exist_ok=True)
json.dump(res, open(os.path.join(OUT, "chunk_plan_sweep.json"), "w"), indent=1)
