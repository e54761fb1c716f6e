"""Timing of the candidate compatibility query (aprilsam_b200_candidate_compatibility) on an H100, against the ways a
caller had before.

Workloads: the M3500 batch and the 100 k dense batch (bench.py's m3500_batch / manhattan_batch graphs).  After two
batch solves, for K in {16, 64, 256, 1024} candidates in the two patterns of candidate_bench.py, seeded: the newest
pose against random old poses ("newest_vs_old") and random pairs ("random_pairs"), W a fixed information matrix and z
drawn around zero:
  * the query with cross9: --warmup calls untimed, --reps timed; device time from CUDA events on the library's stream
    around the public call (asam_timer_start / _stop) and wall time of the call (it ends in a device synchronisation);
    the number of tiles at the default budget; at K = 1024 the device time of each kernel of one call
    (torch.profiler), which says whether the path walks or the per-pair blocks bound the query;
  * candidate_mahalanobis on the same K, timed the same way;
  * where 2K <= 1024: one marginal_covariance of the distinct poses plus C_ij and the 6 x 6 solves on the host
    (numpy), wall time of one pass after one warm-up, and the largest difference of d2 and C between the two routes
    (relative to the largest entry of each).
The card's name, power limit and clocks are read in the same run.  Writes results/compat_bench.json.

    python tools/compat_bench.py [--reps 10] [--warmup 2] [--out results/compat_bench.json]
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
from candidate_bench import W_CAND, pattern, timed  # noqa: E402
from marginal_bench import gpu_info  # noqa: E402
from support import emul  # noqa: E402

KS = (16, 64, 256, 1024)


def host_route(h, a, b, z, W, st, lp):
    """marginal_covariance of the distinct poses, then C_ij and the joint d2 of every pair on the host."""
    ids = np.unique(np.r_[a, b])
    S = h.marginal_covariance(ids)
    pos = {int(v): i for i, v in enumerate(ids)}
    K = len(a)
    J = np.zeros((K, 3, 3 * len(ids)))
    r = np.zeros((K, 3))
    for c in range(K):
        ia, ib = pos[int(a[c])], pos[int(b[c])]
        Ja, Jb, _ = emul.xyt_eval(lp[a[c]], lp[b[c]], np.zeros(3))
        J[c][:, 3 * ia:3 * ia + 3] = Ja
        J[c][:, 3 * ib:3 * ib + 3] = Jb
        r[c] = emul.xyt_eval(st[a[c]], st[b[c]], z[c])[2]
    JS = J @ S  # K x 3 x 3n
    Cx = np.einsum("iak,jbk->ijab", JS, J)
    Winv = np.linalg.inv(W_CAND)
    D = np.einsum("iiab->iab", Cx) + Winv  # S_i
    M = np.zeros((K, K, 6, 6))
    M[:, :, :3, :3] = D[:, None]
    M[:, :, 3:, 3:] = D[None, :]
    M[:, :, :3, 3:] = Cx
    M[:, :, 3:, :3] = Cx.transpose(1, 0, 2, 3)
    v = np.zeros((K, K, 6))
    v[:, :, :3] = r[:, None]
    v[:, :, 3:] = r[None, :]
    d2 = np.einsum("ijk,ijk->ij", v, np.linalg.solve(M, v[..., None])[..., 0])
    d2[np.arange(K), np.arange(K)] = [r[c] @ np.linalg.solve(D[c], r[c]) for c in range(K)]
    return d2, Cx


def n_tiles(h, a, b):
    from support import frontcheck as fc
    plan = fc.borrowed_plan(fc.dev_api(), h.param_ptr())
    L = plan.L
    ip = C.POINTER(C.c_int)
    return int(L.asam_dbg_plan_compat_tiles(plan.p, len(a), a.ctypes.data_as(ip), b.ctypes.data_as(ip),
                                            (256 << 20) // 8, None, 0))


def kernel_split(call):
    """Device time per kernel of one call (torch.profiler with CUDA activities), to say what bounds the query."""
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        out = {}
        for e in prof.key_averages():
            if e.key.startswith("k_marginal") or "marginal" in e.key:
                out[e.key.split("(")[0]] = {"calls": e.count, "device_ms": e.device_time_total / 1e3}
        return out
    except Exception as ex:  # the split is an explanation, not a measurement the rest depends on
        return {"error": repr(ex)}


def run(name, d, reps, warmup, rng):
    L = capi.lib()
    out = {}
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
                d2, cross = h.candidate_compatibility(a, b, z, W, with_cross=True)
                q_dev, q_wall = timed(L, dev, lambda: h.candidate_compatibility(a, b, z, W, with_cross=True), reps,
                                      warmup)
                c_dev, c_wall = timed(L, dev, lambda: h.candidate_mahalanobis(a, b, z, W), reps, warmup)
                ids = np.unique(np.r_[a, b])
                rec = {"K": K, "pairs": K * (K - 1) // 2, "distinct_poses": int(len(ids)), "tiles": n_tiles(h, a, b),
                       "query_device_ms": q_dev, "query_wall_ms": q_wall,
                       "candidate_mahalanobis_device_ms": c_dev, "candidate_mahalanobis_wall_ms": c_wall}
                if 2 * K <= 1024:
                    host_route(h, a[:2], b[:2], z[:2], W[:2], st, lp)
                    t0 = time.perf_counter()
                    hd2, hC = host_route(h, a, b, z, W, st, lp)
                    rec["marginal_cov_host_wall_ms"] = 1e3 * (time.perf_counter() - t0)
                    rec["d2_max_rel_diff_vs_host"] = float(np.abs(hd2 - d2).max() / np.abs(hd2).max())
                    rec["cross_max_rel_diff_vs_host"] = float(np.abs(hC - cross).max() / np.abs(hC).max())
                if K == KS[-1]:
                    rec["kernel_split"] = kernel_split(lambda: h.candidate_compatibility(a, b, z, W, with_cross=True))
                out[f"{pat}_K{K}"] = rec
                print(name, pat, json.dumps(rec), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--poses", type=int, default=100000)
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "compat_bench.json"))
    a = ap.parse_args()
    if capi.lib().asam_device_count() <= 0:
        raise SystemExit("compat_bench: no CUDA device")
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
