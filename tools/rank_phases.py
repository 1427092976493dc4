"""Where the time of a back-to-back rank-kernel step goes, per CTA and between launches.

Builds the library with -DB2F_RANK_PHASES into $B2F_TOOL_OUT/rank_phases_lib/ (never into the package's lib/): thread 0 of
every CTA of every launch then writes %globaltimer at entry, forest ready, rows staged, walk done, dependency wait released
and exit, plus its SM id.  Runs the benchmark's value leg with it -- GBDT 100 x depth 6, 65 536 ranked rows per launch, a
pool of 32 batches, 200 launches back to back on one stream -- once per placement of griddepcontrol.wait (before the stores:
default; at entry: B2F_RANK_WAIT_FIRST=1), and writes $B2F_TOOL_OUT/rank_phases.json:
  per placement  median per-CTA phase durations (split by the CTA's tile count), the gap between one launch's last CTA
                 exit and the next launch's first store, the step time (timestamps and CUDA events), the observed timer tick;
  device         GPU name and power limit.
The instrumented kernel does slightly more work than the product's (one timer read and store per phase per CTA and one
extra barrier before the exit mark): use its step time to compare placements, bench.py for the product's speed.

    python tools/rank_phases.py [--launches 200] [--reps 2]
"""

from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.abspath(os.environ.get("B2F_TOOL_OUT", "tools_out"))
CSRC = os.path.join(ROOT, "databricks_kubernetes_mlops_poc_b200", "csrc")
SLOTS = 8  # B2F_RANK_PHASE_SLOTS
ENTRY, FOREST, STAGED, WALKED, RELEASED, EXIT, SMID = range(7)
PLACEMENTS = {"wait_before_stores": None, "wait_first": "1"}


def build_instrumented() -> str:
    lib_dir = os.path.join(OUT, "rank_phases_lib")
    os.makedirs(lib_dir, exist_ok=True)
    so = os.path.join(lib_dir, "libb200forest.so")
    log = os.path.join(lib_dir, "build.log")
    with open(log, "w") as f:
        rc = subprocess.call(["make", "-s", "-C", CSRC, f"OUT={so}", f"HOSTOBJ={os.path.join(lib_dir, 'host_simd.o')}",
                              "EXTRA_NVCCFLAGS=-DB2F_RANK_PHASES", so], stdout=f, stderr=subprocess.STDOUT)
    if rc != 0:
        sys.stderr.write(open(log).read()[-4000:])
        raise SystemExit(f"instrumented build failed (rc={rc})")
    return so


def med(x) -> float | None:
    x = np.asarray(x, dtype=np.float64)
    return float(np.median(x)) if x.size else None


def analyse(rec: np.ndarray, wait_first: bool, tiles: np.ndarray) -> dict:
    """rec: (launches, ctas, SLOTS) uint64 records; tiles: (ctas,) tiles per CTA.  Times in microseconds."""
    t = rec[..., :EXIT + 1].astype(np.int64)
    t = (t - t[..., ENTRY].min()) / 1e3
    walk_from = np.maximum(t[..., STAGED], t[..., FOREST])
    if wait_first:
        phases = {"wait_blocked": t[..., RELEASED] - t[..., ENTRY], "stage_rows": t[..., STAGED] - t[..., RELEASED],
                  "walk": t[..., WALKED] - walk_from, "reduce_and_store": t[..., EXIT] - t[..., WALKED]}
    else:
        phases = {"stage_rows": t[..., STAGED] - t[..., ENTRY], "walk": t[..., WALKED] - walk_from,
                  "wait_blocked": t[..., RELEASED] - t[..., WALKED], "reduce_and_store": t[..., EXIT] - t[..., RELEASED]}
    phases["forest_ready_after_entry"] = t[..., FOREST] - t[..., ENTRY]
    phases["cta_lifetime"] = t[..., EXIT] - t[..., ENTRY]
    by_tiles = {}
    for k in sorted(set(tiles.tolist())):
        sel = tiles == k
        by_tiles[f"{k}_tiles"] = {"ctas": int(sel.sum()), **{name: med(v[:, sel]) for name, v in phases.items()}}
    first_entry, last_exit = t[..., ENTRY].min(axis=1), t[..., EXIT].max(axis=1)
    first_store = np.maximum(t[..., RELEASED], t[..., WALKED]).min(axis=1)  # a CTA stores once it has walked and its wait is released
    gap = first_store[1:] - last_exit[:-1]
    early = (t[1:, :, ENTRY] < last_exit[:-1, None]).mean(axis=1)  # share of launch N + 1's CTAs that started before N ended
    d = np.diff(np.sort(rec[..., :EXIT + 1].astype(np.int64), axis=-1), axis=-1)
    return {
        "median_per_cta_us": {name: med(v) for name, v in phases.items()},
        "median_per_cta_us_by_tiles": by_tiles,
        "gap_last_exit_to_next_first_store_us": {"median": med(gap), "p10": float(np.percentile(gap, 10)), "p90": float(np.percentile(gap, 90))},
        "next_launch_ctas_started_before_last_exit": med(early),
        "launch_span_us": med(last_exit - first_entry),
        "step_us_from_timestamps": med(np.diff(last_exit)),
        "sms_used": int(len(set(rec[..., SMID].ravel().tolist()))),
        "globaltimer_tick_ns_observed": int(d[d > 0].min()) if (d > 0).any() else None,
    }


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--reps", type=int, default=2, help="runs per placement, alternating")
    args = ap.parse_args()
    so = build_instrumented()

    from databricks_kubernetes_mlops_poc_b200 import _cabi

    _cabi.LIB_PATH = so  # every engine below binds the instrumented library
    lib = _cabi.load_library()
    lib.b2f_rank_phases_arm.restype = C.c_int
    lib.b2f_rank_phases_arm.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    import bench
    from databricks_kubernetes_mlops_poc_b200 import flatten
    from databricks_kubernetes_mlops_poc_b200.encode import RowEncoder
    from databricks_kubernetes_mlops_poc_b200.engine import ForestEngine

    dist = bench.Dist(1, use_cuda=False, solo=True)
    pipe, base = bench.get_pipeline("gbdt100d6", dist)
    flat = flatten.flatten_pipeline(pipe)
    enc = RowEncoder(flat)
    B, POOL, L = bench.BATCH, bench.POOL, args.launches
    _, _, _, rows24 = bench.make_batches(base, enc, POOL, bench.DATA_SEED)
    rows = enc.rank_rows(rows24)

    result = {"workload": f"gbdt100d6, {B} ranked rows per launch, pool of {POOL} batches, {L} launches back to back",
              "device": bench.device_record(0), "runs": {}}
    for rep in range(args.reps):
        for name, env in PLACEMENTS.items():
            if env is None:
                os.environ.pop("B2F_RANK_WAIT_FIRST", None)
            else:
                os.environ["B2F_RANK_WAIT_FIRST"] = env
            eng = ForestEngine(flat, 0)
            info = eng.info()
            assert info["rank_ok"] and not info["rank_stream"]
            ctas = min(info["sm_count"], (B + 31) // 32)
            n_tiles = (B + 31) // 32
            tiles = n_tiles // ctas + (np.arange(ctas) < n_tiles % ctas)
            d_rows, d_p, d_l = eng.device_alloc(rows.nbytes), eng.device_alloc(POOL * B * 4), eng.device_alloc(POOL * B * 4)
            d_rec = eng.device_alloc(L * ctas * SLOTS * 8)
            eng.h2d(d_rows, rows)
            eng.predict_stream_timed(d_rows, B, POOL, d_p, False, d_l, 20, fmt=_cabi.ROWS_RANKED, per_launch=False)  # warm-up
            _cabi.check(lib.b2f_rank_phases_arm(eng.handle, d_rec, L), "b2f_rank_phases_arm")
            _, ms_total = eng.predict_stream_timed(d_rows, B, POOL, d_p, False, d_l, L, fmt=_cabi.ROWS_RANKED, per_launch=False)
            _cabi.check(lib.b2f_rank_phases_arm(eng.handle, None, 0), "b2f_rank_phases_arm")
            rec = np.empty((L, ctas, SLOTS), dtype=np.uint64)
            eng.d2h(rec, d_rec)
            for p in (d_rows, d_p, d_l, d_rec):
                eng.device_free(p)
            eng.close()
            r = analyse(rec, env is not None, tiles)
            r["step_us_from_events"] = 1e3 * ms_total / L
            result["runs"].setdefault(name, []).append(r)
    os.environ.pop("B2F_RANK_WAIT_FIRST", None)
    result["summary"] = {name: {"step_us_from_events": med([r["step_us_from_events"] for r in runs]),
                                "gap_last_exit_to_next_first_store_us": med([r["gap_last_exit_to_next_first_store_us"]["median"] for r in runs]),
                                "median_per_cta_us": runs[-1]["median_per_cta_us"]}
                         for name, runs in result["runs"].items()}
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "rank_phases.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result["summary"], indent=1))


if __name__ == "__main__":
    main()
