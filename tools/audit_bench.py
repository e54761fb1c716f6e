"""Timing of the factor audit on an H100: aprilsam_b200_factor_residuals (every factor) and
aprilsam_b200_factor_outlier_scores (chosen factors).

Workloads: M3500, the sparse and the dense 100 k worlds (datasets.manhattan_sparse / manhattan_dense), each batch-solved
until the largest state change of a solve is below 1e-9 (at most --max-batches solves).  The scores test a factor
against the linearisation at the l_points, so they describe outliers only near convergence; after a single batch solve
from the initial guess many correct closures score high.
  * residuals of all factors: --warmup calls untimed, --reps timed; device time from CUDA events on the library's
    stream around the public call (asam_timer_start / _stop), wall time of the call (it ends in a synchronisation);
  * scores of every loop closure of M3500 (|a - b| > 1), and of 1 k loop closures drawn at random (seeded) on the
    100 k worlds, timed the same way.
The path walk behind the scores is one SM streaming each distinct pose's root path, so the cost follows the paths,
not the number of factors; scoring every factor of a 100 k graph is not measured here.  The card's name, power limit
and clocks are read in the same run.  Writes results/audit_bench.json.

    python tools/audit_bench.py [--reps 10] [--warmup 2] [--out results/audit_bench.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from aprilsam_b200 import capi, datasets  # noqa: E402
from aprilsam_b200 import harness as H  # noqa: E402
from candidate_bench import timed  # noqa: E402
from marginal_bench import gpu_info  # noqa: E402


def run(name, d, reps, warmup, n_closures, rng, max_batches):
    L = capi.lib()
    out = {"poses": int(d.n_nodes), "factors": int(d.n_edges)}
    with H.Harness("b200") as h:
        h.load_full(d)
        prev = h.states().copy()
        for nb in range(1, max_batches + 1):
            h.batch()
            st = h.states()
            dst = st - prev
            dst[:, 2] = (dst[:, 2] + np.pi) % (2 * np.pi) - np.pi  # a heading may come back wrapped by 2 pi
            step = float(np.abs(dst).max())
            if step < 1e-9:
                break
            prev = st.copy()
        out["batches"] = nb
        out["last_step"] = step
        dev = C.c_void_p(L.asam_dbg_dev_of_graph(h.graph_ptr()))
        res = h.factor_residuals()
        dev_ms, wall_ms = timed(L, dev, lambda: h.factor_residuals(), reps, warmup)
        out["residuals_all"] = {"count": int(len(res)), "device_ms": dev_ms, "wall_ms": wall_ms}
        closures = (np.flatnonzero(np.abs(d.eb - d.ea) > 1) + 1).astype(np.int32)  # factor 0 is load_full's prior
        if n_closures is not None and len(closures) > n_closures:
            closures = np.sort(rng.choice(closures, n_closures, replace=False)).astype(np.int32)
        try:
            d2, red = h.factor_outlier_scores(closures)
        except RuntimeError as e:  # a root front too large for the path walk's shared memory
            out["scores_closures"] = {"count": int(len(closures)), "refused": str(e)}
            print(name, json.dumps(out), flush=True)
            return out
        dev_ms, wall_ms = timed(L, dev, lambda: h.factor_outlier_scores(closures), reps, warmup)
        ends = np.r_[d.ea[closures - 1], d.eb[closures - 1]]
        out["scores_closures"] = {
            "count": int(len(closures)), "distinct_poses": int(len(np.unique(ends))),
            "device_ms": dev_ms, "wall_ms": wall_ms, "nan": int(np.isnan(d2).sum()),
            "d2_above_16.27": int((d2 > 16.27).sum()), "redundancy_min": float(np.nanmin(red)),
            "redundancy_max": float(np.nanmax(red))}
    print(name, json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--poses", type=int, default=100000)
    ap.add_argument("--closures", type=int, default=1000)
    ap.add_argument("--max-batches", type=int, default=30)
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "audit_bench.json"))
    a = ap.parse_args()
    if capi.lib().asam_device_count() <= 0:
        raise SystemExit("audit_bench: no CUDA device")
    rng = np.random.default_rng(0)
    res = {"gpu": gpu_info(), "reps": a.reps, "warmup": a.warmup}
    m3500 = H.PoseGraphData.load(os.path.join(ROOT, "tests", "golden", "m3500.npz"))
    res["m3500"] = run("m3500", m3500, a.reps, a.warmup, None, rng, a.max_batches)
    res["manhattan_sparse"] = run("manhattan_sparse", datasets.manhattan_sparse(a.poses, seed=1), a.reps, a.warmup,
                                  a.closures, rng, a.max_batches)
    res["manhattan_dense"] = run("manhattan_dense", datasets.manhattan_dense(a.poses, seed=1), a.reps, a.warmup,
                                 a.closures, rng, a.max_batches)
    res["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
