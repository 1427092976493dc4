"""Measurement helper: where the time of the columnar request pipeline goes (threads x chunk size x row format)."""
import json, os, sys, time
OUT = os.environ.get("B2F_TOOL_OUT", "tools_out")  # where the result file goes
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
from databricks_kubernetes_mlops_poc_b200 import flatten, training
from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine, Scorer
from databricks_kubernetes_mlops_poc_b200.model import B200Model
from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES

d = bench.Dist(1, use_cuda=False, solo=True)
pipe, base = bench.get_pipeline("gbdt100d6", d)
flat = flatten.flatten_pipeline(pipe)
enc = RowEncoder(flat)
eng = ForestEngine(flat, 0)
df = training.synth_frame(base, 65536, bench.DATA_SEED)[ALL_FEATURES]
cols = enc.frame_columns(df)
res = {}
def med(f, n=30):
    f(); f()
    ts = []
    for _ in range(n):
        t0 = time.perf_counter(); f(); ts.append(time.perf_counter() - t0)
    return 1e6 * float(np.median(ts))
# pure encode (no GPU): b2f_encoder_encode into pinned memory, by thread count
out_rk = eng.pinned("probe_rk", 65536 * 32).view(np.uint32, (65536, 8))
from databricks_kubernetes_mlops_poc_b200 import encode as encmod
for th in (1, 4, 8, 16, 32, 64):
    encmod.NATIVE_THREADS = th
    res[f"encode_only_ranked_t{th}_us"] = med(lambda: enc._encode_native(df, out_rk, fmt=2), 15)
out_pk = eng.pinned("probe_pk", 65536 * 64).view(np.uint32, (65536, 16))
encmod.NATIVE_THREADS = 16
res["encode_only_packed_t16_us"] = med(lambda: enc._encode_native(df, out_pk, fmt=1), 15)
res["c_abi_ranked_65536_us"] = med(lambda: eng.predict_rows(out_rk, np.float64))
for th in (1, 8, 16, 32, 48):
    sc = Scorer(eng, enc, th)
    for chunk in (2048, 4096, 8192, 16384, 65536):
        def run():
            n_chunks = sc.start(65536, cols, out_mode=1, chunk_rows=chunk)
            t0 = time.perf_counter()
            sc.wait(0)
            t1 = time.perf_counter()
            sc.wait(n_chunks - 1)
            return t1 - t0
        run(); run()
        tot, first = [], []
        for _ in range(30):
            t0 = time.perf_counter(); f = run(); tot.append(time.perf_counter() - t0); first.append(f)
        res[f"scorer_t{th}_chunk{chunk}"] = {"total_us": 1e6 * float(np.median(tot)), "first_chunk_us": 1e6 * float(np.median(first))}
    # back-to-back vs after an idle gap (worker wake-up)
    def gap():
        time.sleep(0.003)
        t0 = time.perf_counter()
        n_chunks = sc.start(65536, cols, out_mode=1, chunk_rows=8192)
        sc.wait(n_chunks - 1)
        return time.perf_counter() - t0
    gap()
    res[f"scorer_t{th}_chunk8192_after_3ms_idle_us"] = 1e6 * float(np.median([gap() for _ in range(20)]))
    sc.close()
# plugin call by request size, pipeline vs general path (B200_SCORER=0)
for scorer in ("1", "0"):
    os.environ["B200_SCORER"] = scorer
    m = B200Model(flat, devices=[0])
    for n in (1, 16, 128, 256, 1024, 4096, 65536):
        sub = df.iloc[:n]
        res[f"predict_n{n}_scorer{scorer}_us"] = med(lambda: m.predict(sub), 30)
    m.close()
print(json.dumps(res, indent=1))
os.makedirs(OUT, exist_ok=True)
json.dump(res, open(os.path.join(OUT, "scorer_probe.json"), "w"), indent=1)
