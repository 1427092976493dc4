"""Measurement helper for ncu: a handful of launches of one predict kernel on the cfg2 workload (65 536 rows, device resident).
usage: rank_one.py [model] [fmt: 2 ranked | 1 packed] [launches]"""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
from databricks_kubernetes_mlops_poc_b200 import flatten, training
from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine

name = sys.argv[1] if len(sys.argv) > 1 else "gbdt100d6"
fmt = int(sys.argv[2]) if len(sys.argv) > 2 else 2
launches = int(sys.argv[3]) if len(sys.argv) > 3 else 6
d = bench.Dist(1, use_cuda=False, solo=True)
pipe, base = bench.get_pipeline(name, d)
flat = flatten.flatten_pipeline(pipe)
enc = RowEncoder(flat)
POOL, B = 4, 65536
vocabs, codes, nums = training.synth_arrays(base, POOL * B, 5)
rows24 = enc.encode_arrays(codes, nums)
arr = enc.rank_rows(rows24) if fmt == 2 else enc.pack_rows(rows24)
eng = ForestEngine(flat, 0)
d_rows = eng.device_alloc(arr.nbytes); d_p = eng.device_alloc(POOL * B * 4); d_l = eng.device_alloc(POOL * B * 4)
eng.h2d(d_rows, arr)
ms, tot = eng.predict_stream_timed(d_rows, B, POOL, d_p, False, d_l, launches, fmt=fmt)
print("per launch us", (1e3 * ms).round(2).tolist())
eng.close()
