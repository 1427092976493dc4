"""Where do the slow steps of the plugin e2e come from?  (run on an H100; writes e2e_stalls.json under $B2F_TOOL_OUT, default tools_out/)

Runs `B200Model.predict(DataFrame of 65 536 rows)` K times under several conditions -- no clock sampler, `nvidia-smi -lms 100`
next to it (what bench.py does during its timed regions), `-lms 1000` -- and with different host-thread counts, and records the
per-step latency distribution, the phase breakdown of the slowest steps, page faults / context switches per step and the
cgroup's CPU-throttling counters around each loop."""
import gc
import json
import os
OUT = os.environ.get("B2F_TOOL_OUT", "tools_out")  # where the result file goes
import resource
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def cgroup_cpu():
    out = {}
    for p in ("/sys/fs/cgroup/cpu.max", "/sys/fs/cgroup/cpu.stat", "/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "/sys/fs/cgroup/cpu/cpu.stat"):
        try:
            out[p] = open(p).read().strip().replace("\n", "; ")
        except OSError:
            pass
    return out


def loop(model, df, K):
    lat, stages, flt, csw = [], [], [], []
    for _ in range(K):
        r0 = resource.getrusage(resource.RUSAGE_SELF)
        t = time.perf_counter()
        model.predict(df)
        lat.append(time.perf_counter() - t)
        r1 = resource.getrusage(resource.RUSAGE_SELF)
        flt.append(r1.ru_minflt - r0.ru_minflt)
        csw.append((r1.ru_nvcsw - r0.ru_nvcsw, r1.ru_nivcsw - r0.ru_nivcsw))
        stages.append(dict(model.last_timing or {}))
    lat = np.asarray(lat)
    order = np.argsort(lat)[::-1][:6]
    return {
        "mean_ms": 1e3 * float(lat.mean()), "p50_ms": 1e3 * float(np.percentile(lat, 50)), "p90_ms": 1e3 * float(np.percentile(lat, 90)),
        "p99_ms": 1e3 * float(np.percentile(lat, 99)), "max_ms": 1e3 * float(lat.max()),
        "steps_over_2x_p50": int((lat > 2 * np.percentile(lat, 50)).sum()),
        "rows_per_s_mean": 65536 / float(lat.mean()),
        "minor_faults_per_step_p50": float(np.median(flt)),
        "slowest": [{"step": int(i), "ms": 1e3 * float(lat[i]), "minor_faults": int(flt[i]), "ctx_switches_vol_invol": csw[i],
                     **{k: (round(1e3 * v, 3) if k.endswith("_s") else v) for k, v in stages[i].items()}} for i in order],
    }


def main():
    from databricks_kubernetes_mlops_poc_b200 import flatten, training
    from databricks_kubernetes_mlops_poc_b200.model import B200Model
    from databricks_kubernetes_mlops_poc_b200.schema import ALL_FEATURES

    K = int(os.environ.get("STALL_STEPS", "300"))
    dist = bench.Dist(1, False, solo=True)
    pipe, base = bench.get_pipeline("gbdt100d6", dist)
    flat = flatten.flatten_pipeline(pipe)
    pv, pc, pn = training.synth_arrays(base, bench.BATCH, bench.DATA_SEED)
    df = training.arrays_to_frame(pv, pc, pn)[ALL_FEATURES]
    res = {"cgroup_before": cgroup_cpu(), "cpus": os.cpu_count(), "affinity": len(os.sched_getaffinity(0))}
    from databricks_kubernetes_mlops_poc_b200 import engine as _engine

    variants = [(int(t), f) for t in os.environ.get("STALL_THREADS", "0,12,10").split(",") for f in os.environ.get("STALL_ROWS", "ranked,packed64").split(",")]
    for threads, rows in variants:
        _engine._FMT_OVERRIDE = {"ranked": _engine.ROWS_RANKED, "packed64": None}[rows]
        model = B200Model(flat, devices=[0], host_threads=threads)
        for _ in range(20):
            model.predict(df)
        gc.collect()
        gc.freeze()
        for name, lms in (("no_sampler", None), ("nvidia_smi_lms100", 100)):
            proc = None
            if lms:
                proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={bench.ClockSampler.Q}", "--format=csv,noheader,nounits", "-lms", str(lms)],
                                        stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
                time.sleep(0.3)
            c0 = cgroup_cpu()
            r = loop(model, df, K)
            r["cgroup_cpu_stat_before"] = c0.get("/sys/fs/cgroup/cpu.stat")
            r["cgroup_cpu_stat_after"] = cgroup_cpu().get("/sys/fs/cgroup/cpu.stat")
            if proc:
                proc.terminate()
                proc.wait(timeout=5)
            res[f"threads{threads or 'auto'}_{rows}_{name}"] = r
            print(threads, rows, name, model.last_timing.get("threads"), {k: round(r[k], 3) for k in ("mean_ms", "p50_ms", "p90_ms", "p99_ms", "max_ms", "steps_over_2x_p50")}, flush=True)
        model.close()
        gc.unfreeze()
    os.makedirs(OUT, exist_ok=True)
    json.dump(res, open(os.path.join(OUT, "e2e_stalls.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
