"""Measurement helper: where should the split kernel (one CTA per 2 rows, latency form) hand over to the warp-per-row kernel?
Synchronous b2f_predict_pairs on pinned 64-byte rows, GBDT 100 x d6 and 500 x d8, by batch size, each kernel pinned (B2F_KERNEL)."""
import json, os, sys, time
OUT = os.environ.get("B2F_TOOL_OUT", "tools_out")  # where the result file goes
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
from databricks_kubernetes_mlops_poc_b200 import flatten, training
from databricks_kubernetes_mlops_poc_b200._cabi import SCORED_DTYPE
from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine

dist = bench.Dist(1, False, solo=True)
res = {}
for name in ("gbdt100d6", "gbdt500d8"):
    pipe, base = bench.get_pipeline(name, dist)
    flat = flatten.flatten_pipeline(pipe)
    enc = RowEncoder(flat)
    _, codes, nums = training.synth_arrays(base, 8192, 5)
    rows = enc.pack_rows(enc.encode_arrays(codes, nums))
    for kern in ("split", "warp", "auto"):
        if kern == "auto":
            os.environ.pop("B2F_KERNEL", None)
        else:
            os.environ["B2F_KERNEL"] = kern
        eng = ForestEngine(flat, device=0)
        h = eng.pinned("rows", rows.nbytes).view(np.uint32, rows.shape)
        h[:] = rows
        out = eng.pinned("out", len(rows) * 8).view(SCORED_DTYPE, (len(rows),))
        for n in (64, 128, 256, 512, 768, 1024, 1536, 2048, 3072, 4096, 8192):
            t = []
            for i in range(120):
                t0 = time.perf_counter()
                eng.predict_pairs(h[:n], out[:n])
                t.append(time.perf_counter() - t0)
            res[f"{name}:{kern}:{n}"] = 1e6 * float(np.median(t[20:]))
        print(name, kern, eng.info()["split_max_rows"], {n: round(res[f"{name}:{kern}:{n}"], 1) for n in (64, 128, 256, 512, 768, 1024, 1536, 2048, 3072, 4096, 8192)}, flush=True)
        eng.close()
os.makedirs(OUT, exist_ok=True)
json.dump(res, open(os.path.join(OUT, "split_threshold.json"), "w"), indent=1)
