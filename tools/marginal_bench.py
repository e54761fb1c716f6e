"""Timing of the covariance queries (aprilsam_b200_marginal_covariance / _relative_covariance) on an H100.

Workloads: the M3500 batch and the 100 k dense batch (bench.py's m3500_batch / manhattan_batch graphs).  After one
batch solve, each query runs --warmup times untimed and --reps times timed: device time from CUDA events on the
library's stream around the public call (asam_timer_start / _stop), wall time of the call (it ends in a device
synchronisation).  Per query: median, min and max of both, the path length in supernodes and columns, and the
bytes of L the path kernel reads (from the plan: columns js..c-1 of each front on the path, rows k..m-1 of column
k).  The card's name, power limit and clocks are read in the same run.  Writes results/marginal_bench.json.

    python tools/marginal_bench.py [--reps 20] [--warmup 3] [--out results/marginal_bench.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from aprilsam_b200 import capi, datasets  # noqa: E402
from aprilsam_b200 import harness as H  # noqa: E402
from support import margcheck as mc  # noqa: E402
from support.frontcheck import borrowed_plan, dev_api  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return dict(zip(q.split(","), (v.strip() for v in out[0].split(","))))
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        return {"error": str(e)}


def path_cost(plan, nodes):
    """(supernodes, columns, bytes of L read) summed over the paths of `nodes`."""
    recs, _, _ = mc.paths(plan, nodes)
    d = plan.descs()
    nsn = cols = byts = 0
    for r in recs:
        js = int(r["j0"])
        for s in mc.chain(d, int(r["sn0"])):
            m, c = 3 * int(d["mb"][s]), 3 * int(d["cb"][s])
            k = np.arange(js, c)
            nsn += 1
            cols += c - js
            byts += 8 * int((m - k).sum())
            js = 0
    return nsn, cols, byts


def stats(v):
    v = np.asarray(v)
    return {"median": float(np.median(v)), "min": float(v.min()), "max": float(v.max())}


def run(name, d, reps, warmup, rng):
    L = capi.lib()
    out = {}
    with H.Harness("b200") as h:
        h.load_full(d)
        h.batch()
        h.batch()
        dev = C.c_void_p(L.asam_dbg_dev_of_graph(h.graph_ptr()))
        plan = borrowed_plan(dev_api(), h.param_ptr())
        N = d.n_nodes
        queries = {"newest": [N - 1], "oldest": [0], "newest_oldest": [N - 1, 0],
                   "random64": sorted(rng.choice(N, 64, replace=False).tolist()), "relative": [0, N - 1]}
        for q, ids in queries.items():
            call = (lambda: h.relative_covariance(ids[0], ids[1])) if q == "relative" else \
                (lambda: h.marginal_covariance(ids))
            for _ in range(warmup):
                call()
            dev_ms, wall_ms = [], []
            for _ in range(reps):
                ms = C.c_float()
                L.asam_timer_start(dev)
                t0 = time.perf_counter()
                call()
                wall_ms.append(1e3 * (time.perf_counter() - t0))
                L.asam_timer_stop(dev, C.byref(ms))
                dev_ms.append(ms.value)
            nsn, cols, byts = path_cost(plan, ids)
            out[q] = {"poses": len(ids), "device_ms": stats(dev_ms), "wall_ms": stats(wall_ms),
                      "path_supernodes": nsn, "path_columns": cols, "L_bytes": byts, "reps": reps}
            print(name, q, json.dumps(out[q]), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--poses", type=int, default=100000)
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "marginal_bench.json"))
    a = ap.parse_args()
    if capi.lib().asam_device_count() <= 0:
        raise SystemExit("marginal_bench: no CUDA device")
    rng = np.random.default_rng(0)
    res = {"gpu": gpu_info()}
    m3500 = H.PoseGraphData.load(os.path.join(ROOT, "tests", "golden", "m3500.npz"))
    res["m3500_batch"] = run("m3500_batch", m3500, a.reps, a.warmup, rng)
    res["manhattan_batch"] = run("manhattan_batch", datasets.manhattan_dense(a.poses, seed=1), a.reps, a.warmup, rng)
    res["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
