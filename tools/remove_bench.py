"""Timing of factor removal (aprilsam_b200_remove_factors) on an H100, against what a caller does without it.

Workloads: the M3500 batch and the 100 k dense batch (bench.py's m3500_batch / manhattan_batch graphs).  After one
batch solve (and one more, warm), removals of three kinds, each kind --reps times on the same solver (every removal
takes a different factor, so each one is a real removal of the graph as it is then), after --warmup untimed ones:
  * "newest": the loop closure with the highest index (near the newest pose);
  * "deep": the loop closure with the lowest index (an old pose: a long root path, usually the full back-substitution);
  * "sixteen": 16 closures spread over the graph in one call.
Per removal: wall time of the call (it ends in a device synchronisation), device time from CUDA events on the
library's stream around it (asam_timer_start / _stop), the host incidence scan (host profile slot 22) and naffected.
The alternative is the splice followed by april_graph_cholesky: a param that never solved the graph takes the
factor out (the splice alone), then the solving param's batch call re-plans (reference ordering, symbolic analysis,
upload) and relinearises everything; its wall time, --batch-reps times.  nthreshold is set out of reach, so that no
removal escalates to a batch solve (checked).  The card's name, power limit and clocks are
read in the same run.  Writes results/remove_bench.json.

    python tools/remove_bench.py [--reps 5] [--warmup 2] [--batch-reps 3] [--out results/remove_bench.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from aprilsam_b200 import capi, datasets  # noqa: E402
from aprilsam_b200 import harness as H  # noqa: E402
from marginal_bench import gpu_info, stats  # noqa: E402


def closures(h):
    out = []
    for i in range(h.n_factors):
        _, a, b, _, _ = h.factor(i)
        if b >= 0 and abs(a - b) > 1:
            out.append(i)
    return out


def profile(L):
    p = (C.c_double * 24)()
    L.asam_dbg_profile(p, 0)
    return np.array(p[:])


def run(name, d, reps, warmup, batch_reps):
    L = capi.lib()
    L.asam_timer_start.argtypes = [C.c_void_p]
    L.asam_timer_stop.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    out = {"poses": d.n_nodes}
    with H.Harness("b200", nthreshold=1 << 30) as h:  # no escalation: every call is a removal, not a batch solve
        h.load_full(d)
        h.batch()
        h.batch()
        out["factors"] = h.n_factors
        dev = C.c_void_p(L.asam_dbg_dev_of_graph(h.graph_ptr()))
        picks = {"newest": lambda lc: [lc[-1]], "deep": lambda lc: [lc[0]],
                 "sixteen": lambda lc: [lc[i] for i in np.linspace(0, len(lc) - 1, 16).astype(int)]}
        for kind, pick in picks.items():
            dev_ms, wall_ms, scan_ms, naff = [], [], [], []
            for r in range(warmup + reps):
                idx = pick(closures(h))
                p0 = profile(L)
                ms = C.c_float()
                L.asam_timer_start(dev)
                t0 = time.perf_counter()
                h.remove_factors(idx)
                wall = 1e3 * (time.perf_counter() - t0)
                L.asam_timer_stop(dev, C.byref(ms))
                if r >= warmup:
                    wall_ms.append(wall)
                    dev_ms.append(ms.value)
                    scan_ms.append(float(profile(L)[22] - p0[22]))
                    naff.append(h.info()["naffected"])
                    assert profile(L)[10] == p0[10], "a removal escalated to a batch solve"
            rec = {"removal_wall_ms": stats(wall_ms), "removal_device_ms": stats(dev_ms),
                   "incidence_scan_host_ms": stats(scan_ms), "naffected": naff, "factors_per_call": len(pick(closures(h)))}
            out[kind] = rec
            print(name, kind, json.dumps(rec), flush=True)
        # the splice and a batch solve (re-plan) instead
        walls = []
        for _ in range(batch_reps):
            idx = [closures(h)[-1]]
            fresh = h.new_param()
            mine = h.swap_param(fresh)
            t0 = time.perf_counter()
            h.remove_factors(idx)  # never solved: the splice alone
            h.swap_param(mine)
            h.batch()
            walls.append(1e3 * (time.perf_counter() - t0))
            h.free_param(fresh)
        out["splice_then_batch_wall_ms"] = stats(walls)
        print(name, "splice_then_batch", json.dumps(out["splice_then_batch_wall_ms"]), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch-reps", type=int, default=3)
    ap.add_argument("--poses", type=int, default=100000)
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "remove_bench.json"))
    a = ap.parse_args()
    if capi.lib().asam_device_count() <= 0:
        raise SystemExit("remove_bench: no CUDA device")
    res = {"gpu": gpu_info()}
    m3500 = H.PoseGraphData.load(os.path.join(ROOT, "tests", "golden", "m3500.npz"))
    res["m3500_batch"] = run("m3500_batch", m3500, a.reps, a.warmup, a.batch_reps)
    res["manhattan_batch"] = run("manhattan_batch", datasets.manhattan_dense(a.poses, seed=1), a.reps, a.warmup,
                                 a.batch_reps)
    res["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
