"""In-place relinearisation (aprilsam_b200_relinearize_poses) against batch escalations, on two replays, on an H100.

Replays (bench.py's replay workloads):
  * M3500 from pose 0 (3499 incremental steps);
  * the sparse 100 k world (datasets.manhattan_sparse(100000, seed=1)) brought to pose 50 000 as bench.py:replay_seek
    does (the first 50 000 poses loaded at once at ground truth, two batch solves), then 1000 steps.
Arms, each on a fresh harness:
  (a) as shipped: nthreshold 100, no escalation policy;
  (b) the work-ratio policy (aprilsam_b200_policy_work_ratio, ratio 1/3) and nthreshold 100;
  (c) the work-ratio policy, and after every step that leaves start_over above 100 the flagged poses
      (tr->linearized_nodes) relinearised in place; nthreshold INT_MAX - 1, so start_over never escalates.  (The
      policy escalates by setting start_over to INT_MAX, which exceeds INT_MAX - 1 but not INT_MAX.)
  (d) in-place relinearisation as in (c) without the policy: no batch solve after the first, which shows what the
      calls cost once the appended poses have made the top of the tree a chain.
Comparing (b) with (c) isolates the feature: both re-order when the policy says so, only (c) relinearises in place.
Per arm: replay wall time (the sum of the per-step call times; a step's time includes the relinearisation made after
it), latency per bucket (bench.py's buckets), the escalations (steps that ended in a batch solve) and the in-place
relinearisations with their wall time and the host incidence scan inside them (host profile slot 22), the final chi2,
the chi2 after one closing batch solve, and the largest state difference from arm (a) after that batch.
The card's name, power limit and SM clock are read in the same run.  Writes results/relin_bench.json.

    python tools/relin_bench.py [--steps 1000] [--out results/relin_bench.json]
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
from bench import BUCKETS, bucket_latency, replay_seek, step_buckets  # noqa: E402
from marginal_bench import gpu_info, stats  # noqa: E402

INT_MAX = 2**31 - 1
RELIN_AT = 100
ARMS = {"a_as_shipped": dict(nthreshold=100, policy=False, relin=False),
        "b_policy": dict(nthreshold=100, policy=True, relin=False),
        "c_policy_relin_in_place": dict(nthreshold=INT_MAX - 1, policy=True, relin=True),
        "d_relin_in_place_no_policy": dict(nthreshold=INT_MAX - 1, policy=False, relin=True)}


def profile(L):
    p = (C.c_double * 24)()
    L.asam_dbg_profile(p, 0)
    return np.array(p[:])


def run_arm(d, s0, s_end, arm):
    L = capi.lib()
    with H.Harness("b200", nthreshold=arm["nthreshold"]) as h:
        replay_seek(h, d, s0)
        if arm["policy"]:
            h.set_policy_ratio(1.0 / 3.0)
        if arm["relin"]:
            h.set_relin_in_place(RELIN_AT)
        ms, info, relin_ms, scan_ms = [], [], [], []
        t0 = time.perf_counter()
        for k in range(s0, s_end):
            p0, r0 = profile(L), h.relin_stats()
            _, m, i = h.replay_to(k + 1, want_chi2=False)
            p1, r1 = profile(L), h.relin_stats()
            ms.append(float(m[0]))
            info.append(i[0])
            if r1[0] > r0[0]:
                relin_ms.append(r1[1] - r0[1])
                scan_ms.append(float(p1[22] - p0[22]))
        wall = 1e3 * (time.perf_counter() - t0)
        ms, info = np.array(ms), np.array(info)
        chi2_end = h.chi2()
        h.batch()
        rec = {"steps": len(ms), "replay_ms": float(ms.sum()), "replay_wall_ms_python_loop": wall,
               "latency_by_bucket": bucket_latency(ms, info)}
        esc = ms[step_buckets(info) == BUCKETS.index("batch_escalation")]
        rec["escalations"] = {"count": int(esc.size), "ms": stats(esc.tolist()) if esc.size else None,
                              "total_ms": float(esc.sum())}
        rec["relin_in_place"] = {"count": len(relin_ms), "ms": stats(relin_ms) if relin_ms else None,
                                 "total_ms": float(np.sum(relin_ms)) if relin_ms else 0.0,
                                 "host_scan_ms": stats(scan_ms) if scan_ms else None,
                                 "host_scan_total_ms": float(np.sum(scan_ms)) if scan_ms else 0.0}
        rec["final_chi2"] = chi2_end
        rec["chi2_after_closing_batch"] = h.chi2()
        return rec, h.states()


def run(name, d, s0, s_end):
    out = {"poses": d.n_nodes, "window": [s0, s_end]}
    ref = None
    for arm_name, arm in ARMS.items():
        rec, st = run_arm(d, s0, s_end, arm)
        if ref is None:
            ref = st
        dd = st - ref
        dd[:, 2] = np.arctan2(np.sin(dd[:, 2]), np.cos(dd[:, 2]))
        rec["max_state_diff_from_a_after_batch"] = float(np.abs(dd).max())
        out[arm_name] = rec
        print(name, arm_name, json.dumps({k: rec[k] for k in ("replay_ms", "escalations", "relin_in_place",
                                                                "final_chi2", "chi2_after_closing_batch",
                                                                "max_state_diff_from_a_after_batch")}), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1000, help="steps of the 100 k replay")
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "relin_bench.json"))
    a = ap.parse_args()
    if capi.lib().asam_device_count() <= 0:
        raise SystemExit("relin_bench: no CUDA device")
    res = {"gpu": gpu_info(), "relin_at_start_over": RELIN_AT, "arms": ARMS}
    m3500 = H.PoseGraphData.load(os.path.join(ROOT, "tests", "golden", "m3500.npz"))
    res["m3500_replay"] = run("m3500_replay", m3500, 1, m3500.n_nodes)
    sparse = datasets.manhattan_sparse(100000, seed=1)
    res["sparse100k_replay"] = run("sparse100k_replay", sparse, 50000, 50000 + a.steps)
    res["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
