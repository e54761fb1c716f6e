#!/usr/bin/env python
"""Cost of robust loop closures on the GPU: plain vs robust arms, alternated on the same device.

    python tools/robust_bench.py [--poses 100000] [--solves 25] [--warm 5] [--out FILE]

  * 100 k dense batch (the bench.py manhattan_batch graph): every closure plain vs every closure Cauchy;
    per arm the median k_linearize time (CUDA events) and the median device-resident solve
    (k_linearize + k_factor + k_backsolve) and end-to-end batch call;
  * M3500 demo-protocol replay: scans plain vs robust (Cauchy, k = 0.5), steps/s over the whole replay and the
    median latency of the steps with naffected <= 5.  The replay runs twice per arm (the first is the warm-up).

Prints one JSON line with the GPU name, power limit and SM clock (nvidia-smi, read in the same call).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from aprilsam_b200 import capi, datasets  # noqa: E402
from aprilsam_b200 import harness as H  # noqa: E402

K_ROBUST = 0.5


def gpu_info() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True, check=True).stdout.strip().split(", ")
    return dict(zip(["gpu", "power_limit", "sm_clock", "sm_clock_max"], out))


def batch_arms(d, solves: int, warm: int) -> dict:
    L = capi.lib()
    arms = {"plain": 0, "cauchy": H.Harness.CAUCHY}
    hs = {}
    for name, loss in arms.items():
        h = H.Harness("b200")
        h.set_scan_loss(loss, K_ROBUST)
        h.load_full(d)
        h.batch()  # cold: plan
        L.asam_set_timing(L.asam_dbg_dev_of_graph(h.graph_ptr()), 1)
        hs[name] = h
    rec = {n: [] for n in arms}
    for i in range(warm + solves):
        for name, h in hs.items():  # alternated
            h.set_states(d.init)
            ms = h.batch()
            if i >= warm:
                lin, fac, bs = capi.kernel_ms(L.asam_dbg_dev_of_graph(h.graph_ptr()))
                rec[name].append((lin, lin + fac + bs, ms))
    out = {}
    for name, r in rec.items():
        a = np.array(r)
        out[name] = {"k_linearize_ms": float(np.median(a[:, 0])), "device_solve_ms": float(np.median(a[:, 1])),
                     "e2e_batch_ms": float(np.median(a[:, 2])), "solves": len(r)}
        hs[name].close()
    out["k_linearize_ratio"] = out["cauchy"]["k_linearize_ms"] / out["plain"]["k_linearize_ms"]
    out["device_solve_ratio"] = out["cauchy"]["device_solve_ms"] / out["plain"]["device_solve_ms"]
    return out


def replay_arms(m) -> dict:
    arms = {"plain": 0, "cauchy": H.Harness.CAUCHY}
    res = {}
    for rnd in range(2):
        hs = {}
        for name, loss in arms.items():
            h = H.Harness("b200")
            h.set_scan_loss(loss, K_ROBUST)
            h.replay_begin(m)
            hs[name] = h
        ms = {n: [] for n in arms}
        info = {n: [] for n in arms}
        for k in range(m.n_nodes):  # alternated step by step
            for name, h in hs.items():
                _, t, inf = h.replay_to(k + 1, want_chi2=False)
                ms[name].append(t[-1])
                info[name].append(inf[-1, 0])
        for name, h in hs.items():
            h.close()
            if rnd == 1:
                t, na = np.array(ms[name][1:]), np.array(info[name][1:])
                res[name] = {"steps_per_s": float(len(t) / (t.sum() / 1e3)),
                             "median_ms_naffected_le5": float(np.median(t[na <= 5])), "steps": int(len(t)),
                             "steps_naffected_le5": int((na <= 5).sum())}
    res["steps_per_s_ratio"] = res["cauchy"]["steps_per_s"] / res["plain"]["steps_per_s"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--poses", type=int, default=100000)
    ap.add_argument("--solves", type=int, default=25)
    ap.add_argument("--warm", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if capi.lib().asam_device_count() <= 0:
        raise SystemExit("robust_bench: no CUDA device")
    info = gpu_info()
    d = datasets.manhattan_dense(args.poses, seed=1)
    m = H.PoseGraphData.load(os.path.join(ROOT, "tests", "golden", "m3500.npz"))
    res = dict(info, k=K_ROBUST, batch_100k={"poses": d.n_nodes, "closures": int((np.abs(d.ea - d.eb) != 1).sum()),
                                              **batch_arms(d, args.solves, args.warm)},
               m3500_replay=replay_arms(m))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
