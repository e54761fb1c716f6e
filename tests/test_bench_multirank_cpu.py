"""world_size-2 gloo test of bench.py's multi-rank aggregation (replicas only: no data-path
collective; the only exchange is barrier + max of the per-rank times)."""
import os
import socket
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, q):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    sys.path.insert(0, ROOT)
    import bench
    w, r, local, dist = bench.dist_setup(world, backend="gloo")
    assert (w, r) == (world, rank)
    # rank r needs (r+1) seconds for 10 steps -> the job takes 2 s -> 2 ranks * 10 steps / 2 s
    slowest = bench.barrier_max(dist, local, float(rank + 1))
    rate = bench.aggregate_rate(dist, local, w, 10, float(rank + 1))
    q.put((rank, slowest, rate))
    dist.destroy_process_group()


def test_two_rank_gloo_aggregation():
    torch = pytest.importorskip("torch")
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, slowest, rate in res:
        assert slowest == 2.0
        assert rate == 10.0


def test_reference_arm_json_contract():
    """`bench.py --impl reference` (the unmodified reference on host cores) prints ONE JSON line with the keys of
    the bench contract; the b200 arm refuses to run without a CUDA device (no CPU fallback)."""
    import json
    import subprocess
    sys.path.insert(0, ROOT)
    from aprilsam_b200 import harness as H
    if not H.available("reference"):
        pytest.skip("reference oracle not built")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload", "m3500_batch",
                        "--steps", "2", "--warmup", "1"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-1000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    j = json.loads(lines[0])
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "impl", "cpu_baseline", "e2e"):
        assert k in j, k
    assert j["impl"] == "reference" and j["dtype"] == "f64" and j["unit"] == "solves/s" and j["steps"] == 2
    assert j["cpu_baseline"]["kind"] == "reference" and j["cpu_baseline"]["cores"] == 1
    assert j["e2e"]["h2d_bytes_per_step"] == 0 and j["e2e"]["d2h_bytes_per_step"] == 0
    assert 5 < j["value"] < 500 and abs(j["value"] - j["e2e"]["value"]) < 1e-9
    import torch
    if not torch.cuda.is_available():
        r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "2", "--workload", "m3500_batch"],
                           capture_output=True, text=True, timeout=300)
        assert r.returncode != 0 and "no CUDA device" in (r.stderr + r.stdout)


def test_reference_arm_default_line_covers_all_four_workloads():
    """The default line (--workload all) headlines the batch solve of the synthetic Manhattan world and carries one
    record each for m3500_batch, m3500_replay (with the as-shipped wall-clock variant beside it) and manhattan_replay,
    every record with value / e2e / cpu_baseline; replay records with per-naffected-bucket latencies.  Small world here;
without --steps the sub-workloads keep their own windows (the whole M3500 replay)."""
    import json
    import subprocess
    sys.path.insert(0, ROOT)
    from aprilsam_b200 import harness as H
    if not H.available("reference"):
        pytest.skip("reference oracle not built")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--poses", "3000",
                        "--replay-from", "1500", "--warmup", "1"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-1000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    j = json.loads(lines[0])
    assert j["config"]["workload"] == "manhattan_batch" and j["steps"] == 20 and j["impl"] == "reference"
    assert set(j["workloads"]) == {"m3500_batch", "m3500_replay", "manhattan_replay"}
    for name, rec in j["workloads"].items():
        for k in ("value", "unit", "steps", "ms_per_step", "e2e", "cpu_baseline"):
            assert k in rec, (name, k)
        assert rec["value"] > 0
    rp = j["workloads"]["m3500_replay"]
    assert rp["steps"] == 3499 and set(rp["latency_by_bucket"]) == {"naffected_le5", "naffected_6_50", "naffected_gt50", "batch_escalation"}
    assert rp["latency_by_bucket"]["batch_escalation"]["steps"] == 49  # SURVEY.md section 8c: 49 batch escalations
    assert rp["latency_by_bucket"]["naffected_le5"]["steps"] > 2000
    assert rp["cpu_baseline_wallclock"]["value"] > 0
