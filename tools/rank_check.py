"""Measurement helper: parity + timing of k_forest_predict_rank against the tile kernel on the cfg2 workload."""
import json, os, sys, time
OUT = os.environ.get("B2F_TOOL_OUT", "tools_out")  # where the result file goes
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
from databricks_kubernetes_mlops_poc_b200 import flatten, training, _cabi
from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine
from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES

out = {}
d = bench.Dist(1, use_cuda=False, solo=True)
for name in sys.argv[1:] or ["gbdt100d6", "rf100d6"]:
    pipe, base = bench.get_pipeline(name, d)
    flat = flatten.flatten_pipeline(pipe)
    enc = RowEncoder(flat)
    POOL, B = 32, 65536
    vocabs, codes, nums = training.synth_arrays(base, POOL * B, 5)
    rows24 = enc.encode_arrays(codes, nums)
    res = {}
    for u in ("4", "8"):
        os.environ["B2F_RANK_U"] = u
        eng = ForestEngine(flat, 0)
        info = eng.info()
        res["rank_ok"] = info["rank_ok"]; res["rank_smem"] = info["rank_smem_bytes"]
        rk = enc.rank_rows(rows24)
        pk = enc.pack_rows(rows24)
        # parity: full batch 0 (65536 rows) + odd sizes, f64, vs sklearn
        df = training.arrays_to_frame(vocabs, codes[:B], nums[:B])[ALL_FEATURES]
        want = pipe.predict_proba(df)[:, 1]; wl = pipe.predict(df)
        for n in (1, 31, 33, 1000, 4737, 65536):
            p, l = eng.predict_rows(rk[:n], np.float64)
            err = float(np.abs(p - want[:n]).max()); ok = bool((l == wl[:n]).all())
            res[f"u{u}_n{n}"] = [err, ok]
        # timing: device resident, streaming pool
        for fmt, arr, key in ((2, rk, "rank"), (1, pk, "tile")):
            d_rows = eng.device_alloc(arr.nbytes); d_p = eng.device_alloc(POOL * B * 4); d_l = eng.device_alloc(POOL * B * 4)
            eng.h2d(d_rows, arr)
            eng.predict_stream_timed(d_rows, B, POOL, d_p, False, d_l, 20, fmt=fmt)
            ms_each, tot = eng.predict_stream_timed(d_rows, B, POOL, d_p, False, d_l, 200, fmt=fmt)
            _, tot2 = eng.predict_stream_timed(d_rows, B, POOL, d_p, False, d_l, 2000, fmt=fmt, per_launch=False)
            res[f"u{u}_{key}"] = {"per_launch_us": 1e3 * float(np.mean(ms_each)), "min_us": 1e3 * float(ms_each.min()),
                                  "step_us_with_events": 1e3 * tot / 200, "step_us_no_events": 1e3 * tot2 / 2000}
            if key == "rank":
                os.environ["B2F_NO_PDL"] = "1"
            for dd in (d_rows, d_p, d_l): eng.device_free(dd)
        eng.close()
    out[name] = res
print(json.dumps(out, indent=1))
os.makedirs(OUT, exist_ok=True)
json.dump(out, open(os.path.join(OUT, "rank_check.json"), "w"), indent=1)
