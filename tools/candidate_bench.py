"""Timing of the candidate query (aprilsam_b200_candidate_mahalanobis) on an H100, against the ways a caller had before.

Workloads: the M3500 batch and the 100 k dense batch (bench.py's m3500_batch / manhattan_batch graphs).  After one
batch solve, for K in {1, 16, 256, 4096} candidates in two patterns, seeded: the newest pose against random old poses
("newest_vs_old") and random pairs ("random_pairs"), W a fixed information matrix and z drawn around zero:
  * the query: --warmup calls untimed, --reps timed; device time from CUDA events on the library's stream around the
    public call (asam_timer_start / _stop) and wall time of the call (it ends in a device synchronisation);
  * K relative_covariance calls plus d2 on the host (numpy), wall time of one pass after a warm-up of a few calls;
    their Sigma_rel must equal the query's bit for bit, and the d2 difference is reported;
  * where the distinct poses number at most --max-gram, one marginal_covariance of the distinct poses, wall time of one
    call after one warm-up, and the largest difference of J Sigma_6 J' from it against the query's Sigma_rel.
The card's name, power limit and clocks are read in the same run.  Writes results/candidate_bench.json.

    python tools/candidate_bench.py [--reps 10] [--warmup 2] [--out results/candidate_bench.json]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from aprilsam_b200 import capi, datasets  # noqa: E402
from aprilsam_b200 import harness as H  # noqa: E402
from marginal_bench import gpu_info, stats  # noqa: E402
from support import emul  # noqa: E402

W_CAND = np.array([[400.0, 30.0, 0.0], [30.0, 250.0, 5.0], [0.0, 5.0, 2000.0]])
KS = (1, 16, 256, 4096)


def pattern(name, N, K, rng):
    if name == "newest_vs_old":
        a = np.full(K, N - 1)
        b = rng.choice(N - 1, K, replace=K > N - 1)
    else:
        a = rng.integers(0, N, K)
        b = rng.integers(0, N, K)
        b = np.where(a == b, (b + 1) % N, b)
    z = rng.normal(0, 0.3, (K, 3))
    return a.astype(np.int32), b.astype(np.int32), z, np.tile(W_CAND.reshape(9), (K, 1))


def host_d2(st, a, b, z, Winv, cov):
    pa, pb = st[a], st[b]
    _, _, r = emul.xyt_eval(pa, pb, z)
    return float(r @ np.linalg.solve(cov + Winv, r))


def timed(L, dev, call, reps, warmup):
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
    return stats(dev_ms), stats(wall_ms)


def run(name, d, reps, warmup, max_gram, rng):
    L = capi.lib()
    out = {}
    Winv = np.linalg.inv(W_CAND)
    with H.Harness("b200") as h:
        h.load_full(d)
        h.batch()
        h.batch()
        dev = C.c_void_p(L.asam_dbg_dev_of_graph(h.graph_ptr()))
        N = d.n_nodes
        st, lp = h.states(), h.l_points()
        for pat in ("newest_vs_old", "random_pairs"):
            for K in KS:
                a, b, z, W = pattern(pat, N, K, rng)
                d2, cov = h.candidate_mahalanobis(a, b, z, W, with_cov=True)
                q_dev, q_wall = timed(L, dev, lambda: h.candidate_mahalanobis(a, b, z, W), reps, warmup)
                rec = {"K": K, "distinct_poses": int(len(np.unique(np.r_[a, b]))), "query_device_ms": q_dev,
                       "query_wall_ms": q_wall}
                # K relative_covariance calls and d2 on the host
                for c in range(min(K, 3)):
                    h.relative_covariance(a[c], b[c])
                t0 = time.perf_counter()
                rel = np.array([h.relative_covariance(a[c], b[c]) for c in range(K)])
                hd2 = np.array([host_d2(st, a[c], b[c], z[c], Winv, rel[c]) for c in range(K)])
                rec["relative_loop_wall_ms"] = 1e3 * (time.perf_counter() - t0)
                rec["relative_bit_identical"] = bool(np.array_equal(rel.view(np.int64), cov.view(np.int64)))
                rec["d2_max_rel_diff_vs_host"] = float(np.max(np.abs(hd2 - d2) / np.maximum(np.abs(hd2), 1e-300)))
                ids = np.unique(np.r_[a, b])
                if len(ids) <= max_gram:
                    h.marginal_covariance(ids)
                    t0 = time.perf_counter()
                    S = h.marginal_covariance(ids)
                    rec["marginal_cov_wall_ms"] = 1e3 * (time.perf_counter() - t0)
                    pos = {int(v): i for i, v in enumerate(ids)}
                    worst = 0.0
                    for c in range(K):
                        ia, ib = pos[int(a[c])], pos[int(b[c])]
                        sel = np.r_[3 * ia:3 * ia + 3, 3 * ib:3 * ib + 3]
                        Ja, Jb, _ = emul.xyt_eval(lp[a[c]], lp[b[c]], np.zeros(3))
                        J = np.hstack([Ja, Jb])
                        R = J @ S[np.ix_(sel, sel)] @ J.T
                        worst = max(worst, float(np.abs(R - cov[c]).max() / np.abs(R).max()))
                    rec["sigma_rel_max_rel_diff_vs_marginal_cov"] = worst
                out[f"{pat}_K{K}"] = rec
                print(name, pat, json.dumps(rec), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--poses", type=int, default=100000)
    ap.add_argument("--max-gram", type=int, default=1024)
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "candidate_bench.json"))
    a = ap.parse_args()
    if capi.lib().asam_device_count() <= 0:
        raise SystemExit("candidate_bench: no CUDA device")
    rng = np.random.default_rng(0)
    res = {"gpu": gpu_info()}
    m3500 = H.PoseGraphData.load(os.path.join(ROOT, "tests", "golden", "m3500.npz"))
    res["m3500_batch"] = run("m3500_batch", m3500, a.reps, a.warmup, a.max_gram, rng)
    res["manhattan_batch"] = run("manhattan_batch", datasets.manhattan_dense(a.poses, seed=1), a.reps, a.warmup,
                                 a.max_gram, rng)
    res["gpu_after"] = gpu_info()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
