#!/usr/bin/env python
"""Generate tests/golden/*.npz from the UNMODIFIED reference (oracle/_ref, deterministic clock).

Needs oracle/_ref, which oracle/Makefile builds where the reference sources are present.  The
fixtures let the parity tests run where the reference binary is absent.
  m3500_batch.npz    config 1/2: 6 consecutive april_graph_cholesky calls on the full graph
  m3500_replay.npz   config 3: demo-protocol pose-by-pose replay, chi2 / naffected / start_over
                     after every step, full state vectors at checkpoints
  tutorial.npz       the 6-pose dog-leg of examples/aprilsam_tutorial.c (incremental + batch)
  reference_runs.npz the output of every `ref_*` driver of tests/test_host_cpu.py and
                     tests/test_gpu_parity.py run on the reference, keys "<driver>__<name>"
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from aprilsam_b200.harness import Harness, PoseGraphData  # noqa: E402

G = os.path.join(ROOT, "tests", "golden")


def m3500_batch(d):
    h = Harness("reference")
    h.load_full(d)
    chi2 = [h.chi2()]
    states = []
    for _ in range(6):
        h.batch()
        chi2.append(h.chi2())
        states.append(h.states())
    order = h.ordering()
    parents = h.tree_parents()
    h.close()
    np.savez_compressed(os.path.join(G, "m3500_batch.npz"), chi2=np.array(chi2), states=np.array(states),
                        ordering=order, tree_parents=parents)
    print("m3500_batch chi2", chi2)


def m3500_replay(d):
    h = Harness("reference")
    h.replay_begin(d)
    checkpoints = [1, 2, 10, 100, 500, 1000, 2000, 3000, 3500]
    chi2, info, states = [], [], {}
    for cp in checkpoints:
        c, _, i = h.replay_to(cp)
        chi2.append(c)
        info.append(i)
        states[f"states_{cp}"] = h.states()
    chi2 = np.concatenate(chi2)
    info = np.concatenate(info)
    h.close()
    np.savez_compressed(os.path.join(G, "m3500_replay.npz"), chi2=chi2, naffected=info[:, 0].astype(np.int32),
                        start_over=info[:, 1].astype(np.int32), checkpoints=np.array(checkpoints), **states)
    print("m3500_replay final chi2", chi2[-1], "batch escalations", int((np.diff(info[:, 1]) < 0).sum()))


def tutorial():
    # examples/aprilsam_tutorial.c: 6 poses, unit odometry with small lateral noise, one closure
    init = np.array([[0, 0, 0], [1.0, 0.1, 0.0], [2.1, 0.3, 0.02], [3.0, 0.55, 0.03], [4.1, 0.6, 0.0], [5.0, 0.9, 0.05]])
    W = np.diag([100.0, 100.0, 1000.0]).reshape(-1)
    ea = np.array([0, 1, 2, 3, 4, 0], dtype=np.int32)
    eb = np.array([1, 2, 3, 4, 5, 5], dtype=np.int32)
    ez = np.array([[1, 0.15, 0.01], [1, 0.17, 0.0], [1, 0.2, 0.0], [1.02, 0.15, 0.0], [1, 0.2, -0.01], [5.0, 0.85, 0.012]])
    d = PoseGraphData(init, ea, eb, ez, np.tile(W, (6, 1)))
    out = {}
    for mode, batch_only in (("inc", False), ("batch", True)):
        h = Harness("reference")
        h.replay_begin(d)
        chi2, _, info = h.replay_to(6, batch_only=batch_only)
        out[f"{mode}_chi2"] = chi2
        out[f"{mode}_states"] = h.states()
        h.close()
    np.savez_compressed(os.path.join(G, "tutorial.npz"), init=init, ea=ea, eb=eb, ez=ez, eW=np.tile(W, (6, 1)), **out)
    print("tutorial", out["inc_chi2"], out["batch_chi2"])


def reference_runs():
    sys.path[:0] = [os.path.join(ROOT, "tests")]
    import test_gpu_parity
    import test_host_cpu
    out = {}
    for mod in (test_host_cpu, test_gpu_parity):
        for name, fn in sorted(vars(mod).items()):
            if name.startswith("ref_") and callable(fn) and name != "ref_manhattan_batch":
                print(name, flush=True)
                for k, v in fn("reference").items():
                    v = np.asarray(v)
                    if v.dtype.kind == "i" and v.size:  # orderings and counters: the smallest exact type
                        v = v.astype(np.result_type(np.min_scalar_type(v.min()), np.min_scalar_type(v.max())))
                    out[f"{name[4:]}__{k}"] = v
    np.savez_compressed(os.path.join(G, "reference_runs.npz"), **out)


if __name__ == "__main__":
    if "--reference-runs" in sys.argv:  # only the driver outputs; the other fixtures stay as committed
        reference_runs()
        sys.exit(0)
    d = PoseGraphData.load(os.path.join(G, "m3500.npz"))
    m3500_batch(d)
    m3500_replay(d)
    tutorial()
    reference_runs()
