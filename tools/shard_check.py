#!/usr/bin/env python
"""Multi-GPU check (run under torchrun, one rank per GPU): the sharded batch solve of the dense
synthetic Manhattan graph must reproduce the single-GPU solve of the same rank.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        --master-port 29511 tools/shard_check.py --poses 30000
"""
from __future__ import annotations

import argparse
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from aprilsam_b200 import capi, datasets  # noqa: E402
from aprilsam_b200 import harness as H  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--poses", type=int, default=30000)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--robust", default=None, help="huber:K or cauchy:K: every loop closure a robust factor")
    args = ap.parse_args()
    loss, k = 0, 0.0
    if args.robust:
        name, k = args.robust.split(":")
        loss, k = {"huber": H.Harness.HUBER, "cauchy": H.Harness.CAUCHY}[name], float(k)
    import torch
    import torch.distributed as dist
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    rank, world = dist.get_rank(), dist.get_world_size()
    L = capi.lib()
    capi.comm_init_torch(dist, local)
    d = datasets.manhattan_dense(args.poses, seed=1)

    def run(shard: bool):
        capi.check(L.asam_comm_set_sharding(1 if shard else 0), "set_sharding")
        with H.Harness("b200") as h:
            h.set_scan_loss(loss, k)
            h.load_full(d)
            h.batch()  # cold: plan
            dev = L.asam_dbg_dev_of_graph(h.graph_ptr())
            L.asam_set_timing(dev, 1)
            ms, km = [], []
            import ctypes as C
            prof = (C.c_double * 24)()
            L.asam_dbg_profile(prof, 1)  # reset the host-side phase timers
            for _ in range(args.iters):
                h.set_states(d.init)
                dist.barrier()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                h.batch()
                ms.append((time.perf_counter() - t0) * 1e3)
                km.append(capi.kernel_ms(dev))
            L.asam_dbg_profile(prof, 1)
            if rank == 0:
                print(("sharded" if shard else "single ") + " host ms/call (rank 0): gather %.3f plan-check %.3f enqueue+verify %.3f wait+D2H %.3f "
                      "tree+update %.3f; cpus %d (affinity %d)" % (*[prof[i] / args.iters for i in (11, 12, 13, 14, 16)], os.cpu_count(),
                                                                  len(os.sched_getaffinity(0))), flush=True)
            return h.states(), h.chi2(), float(np.median(ms)), np.median(np.array(km), axis=0)

    s1, c1, t1, k1 = run(False)
    sN, cN, tN, kN = run(True)
    err = np.abs(sN - s1)
    err[:, 2] = np.abs((err[:, 2] + np.pi) % (2 * np.pi) - np.pi)
    rel = float(err.max() / max(1.0, np.abs(s1).max()))
    t = torch.tensor([rel, tN, t1], dtype=torch.float64, device=torch.device("cuda", local))
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    print(f"[rank {rank}/{world}] single-GPU {t1:.2f} ms (lin/fac/bs {k1[0]:.3f}/{k1[1]:.3f}/{k1[2]:.3f}) | sharded {tN:.2f} ms "
          f"(fac incl. exchange {kN[1]:.3f}, bs {kN[2]:.3f}) | rel state err {rel:.3e} | chi2 {c1:.9g} vs {cN:.9g}", flush=True)
    if rank == 0:
        print(f"RESULT world {world} poses {args.poses}: max rel err {t[0].item():.3e}; e2e ms single {t[2].item():.2f} -> sharded {t[1].item():.2f}",
              flush=True)
    dist.destroy_process_group()
    return 0 if t[0].item() < 1e-6 else 1


if __name__ == "__main__":
    sys.exit(main())
