"""The sharded batch solve (SURVEY.md section 8e) on ONE GPU: ranks are processes, NCCL is a loopback stand-in.

A sharded solve cuts the elimination tree into shards; each rank factors its own shards, the ranks broadcast the
shard roots' update matrices, every rank factors the supernodes above the cut (the top), back-solves the top and its
own shards, and the ranks broadcast the solution segments.  NCCL refuses two ranks on one device, so the tests load
tests/support/loopnccl.c in its place (same SONAME, host barriers over a shared file, copies on the caller's stream)
and run one process per rank on the same GPU (tests/support/shardrank.py).  Nothing here measures speed: two
processes time-sliced on one GPU say nothing about scaling over several.

Every rank is checked against what it computed, front by front, with the bounds of test_gpu_kernels.py:
  * the exchange: every rank's copy of a shard root's trailing columns and of a shard's solution segment equals the
    owner's bit for bit; the stand-in counted one broadcast per non-empty range and one all-reduce per solve;
  * every front the rank factored (its shards and the top): local backward error against a float64 re-assembly from
    the rank's Hessian and the children's update matrices as the rank holds them (exchanged ones included); y equals
    the fronts' rhs rows bit for bit; the back-substitution per supernode; the residual and the forward error of the
    whole x after the exchange;
  * against the single-GPU solve: states within 1e-12 relative on integer-valued systems (every sum of k_linearize
    exact), 1e-10 on others (the order of k_linearize's atomics moves the last bits of their Hessian); on the former the Hessians of all ranks and of the single-GPU solve are bit-identical, and so is every front whose own
    kernel path and team size, and those of every supernode below it, agree between the two solves;
  * failed pivots in a shard of either rank and in the top: every rank reads the same status word, naming the
    failing supernode, never an ancestor; the restored system then factors to the same bits as before.

CPU tests (not marked gpu) check the stand-in itself in host mode and that the graphs and world sizes below reach
every part of the sharded schedule on host plans, so the GPU tests cannot become vacuous.
"""
from __future__ import annotations

import ctypes as C
import json
import os
import sys
import time

import numpy as np
import pytest

from aprilsam_b200 import datasets
from aprilsam_b200 import harness as H
from conftest import ROOT
from support import frontcheck as fc
from support import shardrank as sr
from support.hostplan import HostPlan
from test_gpu_kernels import (BACKSOLVE_TOL, FACTOR_TOL, FORWARD_C, RESIDUAL_TOL, RHS_TOL, _clique, _graph, _truth,
                              pendant_graph, pendant_sizes, zoo)

STATE_TOL = 1e-12        # sharded vs single-GPU states, relative to max(1, |states|), integer-valued systems
STATE_TOL_FLOAT = 1e-10  # the same on float-valued systems, whose Hessian depends on the order of k_linearize's
                         # atomics in the last bits (observed 4.5e-12 on the 100 k world, H100 SXM at 700 W)
RESIDUAL_TOL_FLOAT = 1e-14  # residual of x after the exchange on float-valued systems: every rank linearises on its
                            # own, so x joins solutions of Hessians that differ in the last bits (observed 1.3e-15)
LAMBDA = 1.0             # Tikhonov term of the integer-valued solves: an integer, so the Hessian stays exact
HBM_ENV = {"ASAM_TEAM_ROOM": "1"}  # every team front of a crowded level scaled down to one CTA on cta_front's HBM path
CAUCHY = (H.Harness.CAUCHY, 1.0)


# ---------------------------------------------------------------------------------------------
# graphs
# ---------------------------------------------------------------------------------------------
def integer_graph(d, seed=0):
    """The structure of d as an integer-valued system: headings 0, integer positions, z and W (W SPD), so that
    every product and sum of k_linearize is exact and the Hessian does not depend on the order of its atomics."""
    rng = np.random.default_rng(seed)
    xy = np.round(d.truth[:, :2] if d.truth is not None else d.init[:, :2])
    init = np.c_[xy + rng.integers(-1, 2, xy.shape), np.zeros(len(xy))]
    ez = np.c_[xy[d.eb] - xy[d.ea], np.zeros(d.n_edges)]
    eW = np.tile([4.0, 1, 0, 1, 4, 0, 0, 0, 2], (d.n_edges, 1))
    return H.PoseGraphData(init, d.ea.copy(), d.eb.copy(), ez, eW, np.c_[xy, np.zeros(len(xy))])


def clique_graph(n=12, seed=0):
    """Every pose joined to every other: one supernode, whose root has no children."""
    rng = np.random.default_rng(seed)
    return _graph(rng, _truth(rng, n), _clique(np.arange(n)))


GRAPHS = {
    "int30k": lambda: integer_graph(datasets.manhattan_dense(30000, seed=1)),
    "m30k": lambda: datasets.manhattan_dense(30000, seed=1),
    "m100k": lambda: datasets.manhattan_dense(100000, seed=1),
    "int_pendants": lambda: integer_graph(pendant_graph(pendant_sizes())),
    "int2000": lambda: integer_graph(datasets.manhattan_dense(2000, seed=1)),
    "int_wide": lambda: integer_graph(zoo("wide")),
    "int_clique": lambda: integer_graph(clique_graph()),
}
_cache = {}


def graph(name):
    if name not in _cache:
        _cache[name] = GRAPHS[name]()
    return _cache[name]


# ---------------------------------------------------------------------------------------------
# host plans of a sharded solve
# ---------------------------------------------------------------------------------------------
def sharded_plans(d, world, env=None):
    ftype = np.r_[2, np.ones(d.n_edges, dtype=np.int32)].astype(np.int32)
    fa, fb = np.r_[0, d.ea].astype(np.int32), np.r_[-1, d.eb].astype(np.int32)
    old = {k: os.environ.get(k) for k in (env or {})}
    try:
        os.environ.update(env or {})
        return [HostPlan().build(d.n_nodes, ftype, fa, fb, world=world, rank=r) for r in range(world)]
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def shard_layout(plans):
    """(paths per rank {supernode: path}, shard roots, shard owners, bs-leaf counts) of host plans; paths as
    ShardSnapshot names them."""
    p0 = plans[0]
    desc = p0.descs()
    tabs = []
    for p in plans:
        G = {}
        for s, w in list(zip(p.array("tasks"), p.array("nwait"))) + list(zip(p.array("top_tasks"), p.array("top_nwait"))):
            G.setdefault(int(s), (int(w) >> 24) & 0x7f)
        leaf, top = set(int(s) for s in p.array("leaf_tasks")), set(int(s) for s in p.array("top_tasks"))
        t = {}
        for s in set(G) | leaf:
            g = G.get(s, 0)
            path = "leaf" if s in leaf else (f"team{g}" if g else ("cta_smem" if fc.fits_smem(int(desc["mb"][s])) else "cta_hbm"))
            t[s] = ("top:" if s in top else "") + path
        tabs.append(t)
    own, off, cnt = p0.array("shard_owner"), p0.array64("shard_off"), p0.array64("shard_cnt")
    c = 3 * desc["cb"].astype(np.int64)
    m = 3 * desc["mb"].astype(np.int64)
    ld = (m + 2) & ~1
    roots = [int(np.nonzero((desc["f_off"] + c * ld == off[i]) & ((m - c) * ld == cnt[i]))[0][0]) for i in range(len(own))]
    return tabs, roots, own, [p.info()["n_bs_leaf"] for p in plans], desc


# (graph, world, env) of the GPU jobs below
SOLVE_JOBS = {
    2: [("int30k", {}), ("int_pendants", {}), ("int2000", HBM_ENV), ("int_wide", {}), ("int_clique", {})],
    3: [("int30k", {}), ("int_pendants", {}), ("int2000", {}), ("int2000", HBM_ENV)],
}


def test_scenarios_reach_the_sharded_paths(built):
    """The graphs and world sizes of the GPU tests reach every part of the sharded schedule on host plans."""
    roots, tops, widest_top, several, bsl = set(), set(), 0, set(), []
    for world, jobs in SOLVE_JOBS.items():
        for name, env in jobs:
            tabs, rts, own, nbsl, desc = shard_layout(sharded_plans(graph(name), world, env))
            roots |= {tabs[own[i]][r] for i, r in enumerate(rts)}
            for t in tabs:
                tops |= {p[4:] for p in t.values() if p.startswith("top:")}
                widest_top = max([widest_top] + [3 * int(desc["cb"][s]) for s, p in t.items() if p.startswith("top:")])
            if len(own) > world and max(np.bincount(own, minlength=world)) > 1:
                several.add(world)
            if name == "int30k" and world == 3:
                bsl = nbsl
    assert several == {2, 3}, "one rank owns several shards at world 2 and at world 3"
    assert {"leaf", "cta_smem", "cta_hbm"} <= roots and any(p.startswith("team") for p in roots), roots
    assert {"cta_smem", "cta_hbm"} <= tops and any(p.startswith("team") for p in tops), tops
    assert widest_top > 96, "a top supernode is solved in several back-solve blocks"
    assert min(bsl) == 0 and max(bsl) > 0, f"back-solve leaf set empty on one rank, not on another: {bsl}"
    # the edges of the cut
    tabs, rts, own, _, _ = shard_layout(sharded_plans(graph("int_clique"), 2))
    assert len(rts) == 1 and list(own) == [0] and not any(p.startswith("top:") for t in tabs for p in t.values())
    assert tabs[1] == {}, "rank 1 owns nothing"
    plans = sharded_plans(graph("int_wide"), 2)
    tabs, rts, own, _, desc = shard_layout(plans)
    assert len(own) == 1 < 2 and int(desc["ch_cnt"][rts[0]]) == 0, "the split stops on a childless heaviest shard"
    assert len(shard_layout(sharded_plans(graph("int_pendants"), 2))[2]) >= 16 * 2, "the split stops at max_shards"
    # the workload bench.py --gpus 2 shards: the 1413-column merged root is in the top
    tabs, _, _, _, desc = shard_layout(sharded_plans(graph("m100k"), 2))
    root = int(np.nonzero(desc["parent"] < 0)[0][-1])
    assert tabs[0][root].startswith("top:") and 3 * int(desc["cb"][root]) == 1413, (tabs[0][root], desc["cb"][root])


def test_integer_graph_is_exact(built):
    """integer_graph really gives integer-valued Hessian contributions: the float64 Hessian of the reference equals
    its long-double twin entry by entry."""
    d = integer_graph(datasets.manhattan_dense(2000, seed=1))
    ftype = np.r_[2, np.ones(d.n_edges, dtype=np.int32)]
    fa, fb = np.r_[0, d.ea], np.r_[-1, d.eb]
    fz = np.vstack([[0, 0, 0], d.ez])
    fW = np.vstack([[1e4, 0, 0, 0, 1e4, 0, 0, 0, 1e3], d.eW])
    Ad, AdA, B, BA, (_, _, Hh, HA) = fc.linearize_ref(d.n_nodes, ftype, fa, fb, fz, fW, d.init, None, 0.0)
    for v in (Ad, B, Hh):
        assert np.array_equal(v, np.round(v)), "integer entries"
    for v in (AdA, BA, HA):
        assert np.abs(v).max() < 2.0 ** 40, "far from 2^53: every partial sum is exact"


# ---------------------------------------------------------------------------------------------
# the stand-in itself, in host mode (no GPU)
# ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def standin(tmp_path_factory):
    return sr.build_standin(str(tmp_path_factory.mktemp("loopnccl")))


def _run_selftest(standin, tmp_path, world, ranks, env_extra, timeout=60):
    spec = {"world": world, "standin": standin, "id_path": str(tmp_path / "rdv"), "out": str(tmp_path)}
    path = tmp_path / "spec.json"
    path.write_text(json.dumps(spec))
    env = dict(os.environ, LOOPNCCL_HOST="1", **env_extra)
    here = os.path.join(ROOT, "tests", "support", "shardrank.py")
    res = sr.run_ranks(lambda r: [sys.executable, here, "selftest", str(path), str(ranks[r])], len(ranks), env, timeout)
    return res, [dict(np.load(tmp_path / f"selftest_r{r}.npz")) if (tmp_path / f"selftest_r{r}.npz").exists() else None
                 for r in ranks]


@pytest.mark.parametrize("world", [2, 3])
def test_standin_host_mode(standin, tmp_path, world):
    """Broadcasts in place from every root (empty, small, and 7 windows long), all-reduces (int32 max / min,
    float64 sum, chunked beyond the window), and the counters, across `world` processes."""
    res, outs = _run_selftest(standin, tmp_path, world, list(range(world)), {"LOOPNCCL_WINDOW": "4096"})
    assert all(rc == 0 for rc, _ in res), res
    for r, o in enumerate(outs):
        for root in range(world):
            for n in sr.SELFTEST_SIZES:
                assert np.array_equal(o[f"b{root}_{n}"], sr.selftest_data(root, n)), (r, root, n)
        vals = [sr.selftest_data(q, 1000) for q in range(world)]
        assert np.array_equal(o["max"], np.max([v.astype(np.int32) for v in vals], axis=0))
        assert np.array_equal(o["min"], np.min([v.astype(np.int32) for v in vals], axis=0))
        ref = vals[0].copy()
        for v in vals[1:]:
            ref = ref + v  # rank order, as the stand-in sums
        assert np.array_equal(o["sum"], ref)
        nb = world * len(sr.SELFTEST_SIZES)
        assert list(o["stats"]) == [nb, world * 8 * sum(sr.SELFTEST_SIZES), 3, 3000], o["stats"]


def test_standin_missing_peer(standin, tmp_path):
    """A peer that never joins, and one that leaves before a broadcast: the call fails within the wait limit."""
    t0 = time.monotonic()
    res, outs = _run_selftest(standin, tmp_path, 2, [0], {"LOOPNCCL_TIMEOUT": "1"})
    assert res[0][0] == 3, res  # ncclCommInitRank failed (exit code 3 = the init returned an error)
    assert time.monotonic() - t0 < 30
    d2 = tmp_path / "leave"
    d2.mkdir()
    res, outs = _run_selftest(standin, d2, 2, [0, "1:leave"], {"LOOPNCCL_TIMEOUT": "1"})
    assert res[1][0] == 0 and res[0][0] == 4, res  # rank 0's broadcast failed (exit code 4), rank 1 left cleanly


# ---------------------------------------------------------------------------------------------
# GPU: the sharded solve, rank by rank
# ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def two_contexts(built):
    """The device must accept a context per process: skip if its compute mode is exclusive (read, never set)."""
    cu = C.CDLL("libcuda.so.1")
    dev, mode = C.c_int(), C.c_int()
    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(C.byref(dev), 0) == 0
    assert cu.cuDeviceGetAttribute(C.byref(mode), 20, dev) == 0  # CU_DEVICE_ATTRIBUTE_COMPUTE_MODE
    if mode.value != 0:
        pytest.skip(f"compute mode {mode.value} is not the default: two processes cannot share the GPU")


def run_sharded(standin, tmp_path, world, jobs, timeout=1800):
    """Run the jobs on `world` rank processes; returns {job name: [(report, arrays) per rank]}."""
    for job in jobs:
        if "graph_name" in job:
            p = tmp_path / f"{job['graph_name']}.npz"
            if not p.exists():
                graph(job["graph_name"]).save(str(p))
            job["graph"] = str(p)
    spec = {"world": world, "standin": standin, "id_path": str(tmp_path / "rdv"), "out": str(tmp_path), "jobs": jobs}
    path = tmp_path / "spec.json"
    path.write_text(json.dumps(spec))
    env = dict(os.environ, ASAM_DEVICE="0")
    here = os.path.join(ROOT, "tests", "support", "shardrank.py")
    t0 = time.monotonic()
    res = sr.run_ranks(lambda r: [sys.executable, here, str(path), str(r)], world, env, timeout)
    print(f"SHARDED world {world}: {len(jobs)} jobs in {time.monotonic() - t0:.1f} s")
    assert all(rc == 0 for rc, _ in res), "\n".join(f"--- rank {r}: exit {rc}\n{o[-4000:]}" for r, (rc, o) in enumerate(res))
    out = {}
    for job in jobs:
        out[job["name"]] = []
        for r in range(world):
            z = dict(np.load(tmp_path / f"{job['name']}_r{r}.npz"))
            out[job["name"]].append((json.loads(str(z.pop("report"))), z))
    return out


def state_err(a, b):
    e = np.abs(a - b)
    e[:, 2] = np.abs((e[:, 2] + np.pi) % (2 * np.pi) - np.pi)
    return float(e.max() / max(1.0, np.abs(b).max()))


def effective_paths(rep, owner_reps, shard_of):
    """{supernode: path} of the fronts a sharded solve of one rank holds: a shard's from its owner, the top's own."""
    out = {}
    for s, (_, p) in rep["digests"].items():
        if p.startswith("top:"):
            out[int(s)] = p[4:]
    for s, r in shard_of.items():
        out[s] = owner_reps[r]["digests"][str(s)][1]
    return out


def shard_members(parent, roots, owner):
    """{supernode: owning rank} of every supernode below a shard root."""
    kids = {}
    for s, p in enumerate(parent):
        kids.setdefault(p, []).append(s)
    out = {}
    for r, o in zip(roots, owner):
        stack = [r]
        while stack:
            s = stack.pop()
            out[s] = int(o)
            stack += kids.get(s, [])
    return out


def same_front_count(parent, eff_a, eff_b, dig_a, dig_b):
    """(compared, equal): supernodes whose own path and those of all their descendants agree in both solves, and
    how many of them hold the same bits in both."""
    ok = [True] * len(parent)
    for s in range(len(parent)):  # children have smaller ids
        ok[s] = ok[s] and s in eff_a and s in eff_b and eff_a[s] == eff_b[s]
        if parent[s] >= 0 and not ok[s]:
            ok[parent[s]] = False
    cmp = [s for s in range(len(parent)) if ok[s] and s in dig_a and s in dig_b]
    return len(cmp), sum(dig_a[s] == dig_b[s] for s in cmp), [s for s in cmp if dig_a[s] != dig_b[s]][:5]


def assert_sharded(name, ranks, exact, summary):
    """Every check of the module docstring on the reports of one job."""
    world = len(ranks)
    single = ranks[0][0].get("single")
    for k, run in enumerate(ranks[0][0]["runs"]):
        reps = [r[0]["runs"][k] for r in ranks]
        arrs = [r[1] for r in ranks]
        if not run["sharded"]:
            assert all(r["n_top"] == 0 and r["status"] == 0 for r in reps), f"{name} run {k}: the plan was not rebuilt"
            if single is not None and exact:  # the same plan and Hessian as the fresh single-GPU solve: the same bits
                assert all(np.array_equal(a[f"run{k}_states"], arrs[0]["single_states"]) for a in arrs), name
            continue
        tag = f"run{k}"
        what = f"{name} run {k}"
        own, q0, qn = arrs[0][f"{tag}_shard_owner"], arrs[0][f"{tag}_shard_q0"], arrs[0][f"{tag}_shard_qn"]
        cnt = arrs[0][f"{tag}_shard_cnt"]
        for a in arrs[1:]:
            for key in ("shard_owner", "shard_q0", "shard_qn", "shard_off", "shard_cnt"):
                assert np.array_equal(a[f"{tag}_{key}"], arrs[0][f"{tag}_{key}"]), (what, key)
        assert all(r["status"] == 0 for r in reps), (what, [r["status"] for r in reps])
        # the exchange
        for i in range(len(own)):
            assert all(r["xch"][i] == reps[int(own[i])]["xch"][i] for r in reps), (what, "update matrix", i)
            seg = slice(3 * int(q0[i]), 3 * int(q0[i] + qn[i]))
            for a in arrs:
                assert np.array_equal(a[f"{tag}_x"][seg].view(np.int64), arrs[int(own[i])][f"{tag}_x"][seg].view(np.int64)), \
                    (what, "solution segment", i)
        n_bc = int(np.count_nonzero(cnt)) + int(np.count_nonzero(qn))
        n_bytes = 8 * int(cnt.sum()) + 24 * int(qn.sum())
        for r, a in enumerate(arrs):
            assert list(a[f"{tag}_stats"][:3]) == [n_bc, n_bytes, 1], (what, r, a[f"{tag}_stats"], n_bc, n_bytes)
        # every front each rank factored
        for r, rep in enumerate(reps):
            c = rep["checks"]
            msg = f"{what} rank {r}: {json.dumps(c)}"
            assert c["factor"] < FACTOR_TOL and c["rhs"] < RHS_TOL and c["y_bad"] == 0, msg
            assert c["backsolve"] < BACKSOLVE_TOL and c["residual"] < (RESIDUAL_TOL if exact else RESIDUAL_TOL_FLOAT), msg
            assert c.get("forward_over_kappa_u", 0.0) <= FORWARD_C, msg
            for p, v in c["per_path"].items():
                rec = summary.setdefault(("top:" if p.startswith("top:") else "rank:") + p.replace("top:", ""),
                                         {"n": 0, "factor": 0.0, "rhs": 0.0, "backsolve": 0.0})
                rec["n"] += v["n"]
                for key in ("factor", "rhs", "backsolve"):
                    rec[key] = max(rec[key], v[key])
            summary["residual"] = max(summary.get("residual", 0.0), c["residual"])
            summary["forward_over_kappa_u"] = max(summary.get("forward_over_kappa_u", 0.0), c.get("forward_over_kappa_u", 0.0))
        # against the single-GPU solve
        if single is None:
            continue
        assert single["status"] == 0 and single["n_top"] == 0
        errs = [state_err(a[f"{tag}_states"], arrs[0]["single_states"]) for a in arrs]
        summary.setdefault("state_err", {})[what] = max(errs)
        assert max(errs) <= (STATE_TOL if exact else STATE_TOL_FLOAT), (what, errs)
        if not exact:
            continue
        assert all(r["hessian"] == single["hessian"] for r in reps), (what, "Hessian bits")
        assert all(r["desc"] == single["desc"] for r in reps), (what, "plan descriptors")
        parent = single["parent"]
        members = shard_members(parent, reps[0]["roots"], own)
        sdig = {int(s): v[0] for s, v in single["digests"].items()}
        spath = {int(s): v[1] for s, v in single["digests"].items()}
        cov = summary.setdefault("bit_identity", {})
        for r, rep in enumerate(reps):
            eff = effective_paths(rep, reps, members)
            dig = {int(s): v[0] for s, v in rep["digests"].items()}
            n, same, bad = same_front_count(parent, eff, spath, dig, sdig)
            assert same == n, (what, f"rank {r} vs single GPU: fronts differ", bad)
            cov[f"{what} rank {r} vs single"] = [n, len(dig)]
            for r2 in range(r + 1, world):
                eff2 = effective_paths(reps[r2], reps, members)
                dig2 = {int(s): v[0] for s, v in reps[r2]["digests"].items()}
                n2, same2, bad2 = same_front_count(parent, eff, eff2, dig, dig2)
                assert same2 == n2, (what, f"rank {r} vs rank {r2}: top fronts differ", bad2)
                cov[f"{what} rank {r} vs rank {r2}"] = [n2, len(set(dig) & set(dig2))]


def assert_marginals(ranks):
    """Covariance queries after each run of the sharded / one-GPU / sharded job: refused with the reason on every rank
    after a sharded solve, checked hop by hop after the one-GPU solve on the same context."""
    from test_gpu_marginals import DINV_C, GRAM_C, HOP_C
    for rep, _ in ranks:
        for run in rep["runs"]:
            m = run["marginals"]
            print("MARGCHECK sharded " + json.dumps(m))
            if run["sharded"]:
                assert all(e is not None and "sharded" in e for e in m["errors"]), m
            else:
                assert m["hops_bad"] == 0 and m["transpose_bad"] == 0 and m["symmetric"], m
                assert m["hop"] <= HOP_C and m["gram"] <= GRAM_C and m["dinv"] <= DINV_C, m


SUMMARY = {}


def _report(name):
    print(f"SHARDCHECK {name} " + json.dumps(SUMMARY.get(name, {}), default=str))


@pytest.mark.gpu
@pytest.mark.parametrize("world", sorted(SOLVE_JOBS))
def test_sharded_solves(two_contexts, standin, tmp_path, world):
    """Integer-valued graphs at world 2 and 3 (one rank owning several shards; shard roots and top fronts on every
    kernel path; the one-supernode graph; a cut that stops on a childless shard); at world 2 the 30 k world is solved
    sharded, on one GPU and sharded again in one process."""
    jobs = []
    for k, (name, env) in enumerate(SOLVE_JOBS[world]):
        jobs.append({"name": f"{name}_{k}", "kind": "solve", "graph_name": name, "env": env, "single": True,
                     "tikhonov": LAMBDA, "sharding": [1, 0, 1] if (name == "int30k" and world == 2) else [1],
                     "marginals": name == "int30k" and world == 2})
    out = run_sharded(standin, tmp_path, world, jobs)
    summary = SUMMARY.setdefault(f"world{world}", {})
    for job in jobs:
        ranks = out[job["name"]]
        summary.setdefault("seconds", {})[job["name"]] = max(r[0]["seconds"] for r in ranks)
        assert_sharded(job["name"], ranks, True, summary)
    _report(f"world{world}")
    if world == 2:
        assert_marginals(out["int30k_0"])
    cov = summary["bit_identity"]
    for job in jobs:  # every job compared some fronts bit for bit with the single-GPU solve
        assert sum(n for key, (n, _) in cov.items() if key.startswith(job["name"]) and key.endswith("vs single")) > 0, cov


@pytest.mark.gpu
def test_sharded_robust_cauchy(two_contexts, standin, tmp_path):
    """Every loop closure a Cauchy factor, 30 k world, two ranks (what the two-GPU robust test checks)."""
    jobs = [{"name": "cauchy", "kind": "solve", "graph_name": "m30k", "single": True, "robust": list(CAUCHY),
             "sharding": [1]}]
    out = run_sharded(standin, tmp_path, 2, jobs)
    summary = SUMMARY.setdefault("cauchy", {})
    assert_sharded("cauchy", out["cauchy"], False, summary)
    _report("cauchy")


@pytest.mark.gpu
def test_sharded_100k(two_contexts, standin, tmp_path):
    """The workload bench.py --gpus 2 shards: manhattan_dense(100000), the 1413-column merged root in the top."""
    jobs = [{"name": "m100k", "kind": "solve", "graph_name": "m100k", "single": True, "forward": False,
             "sharding": [1]}]
    out = run_sharded(standin, tmp_path, 2, jobs)
    summary = SUMMARY.setdefault("m100k", {})
    assert_sharded("m100k", out["m100k"], False, summary)
    assert any(r[0]["runs"][0]["bt_split"] for r in out["m100k"])
    _report("m100k")


@pytest.mark.gpu
def test_sharded_failed_pivots(two_contexts, standin, tmp_path):
    """A failed pivot in a leaf-kernel supernode of rank 0, in a team / HBM front of rank 1 and in a top supernode:
    every rank reads the same status word, 1 + the failing supernode the float64 elimination predicts; restored, the
    system factors to the bits of the clean run on every rank."""
    jobs = [{"name": "pivots", "kind": "pivots", "graph_name": "int30k", "tikhonov": 0.0}]
    ranks = run_sharded(standin, tmp_path, 2, jobs)["pivots"]
    reps = [r[0] for r in ranks]
    summary = SUMMARY.setdefault("pivots", {})
    assert all(r["plan_unchanged"] for r in reps), "the extra priors leave the plan unchanged"
    assert_sharded("pivots", [(dict(runs=[r["runs"][1]]), {k.replace("clean", "run0"): v for k, v in a.items()})
                              for r, a in zip(reps, [x[1] for x in ranks])], False, summary)
    who = [t["who"] for t in reps[0]["targets"]]
    assert who == ["rank0", "rank1", "top"], who
    for j, w in enumerate(who):
        recs = [r["targets"][j] for r in reps]
        sn = recs[0]["sn"]
        words = [t["status"] for t in recs]
        owner = 0 if w == "rank0" else (1 if w == "rank1" else 0)
        pred = recs[owner]["predicted"]
        summary.setdefault("targets", []).append({"who": w, "sn": sn, "path": recs[owner]["path"], "status": words,
                                                  "predicted": pred})
        assert pred is not None and pred[0] == sn, (w, sn, pred)
        assert words == [1 + sn] * len(recs), (w, sn, words)
        assert all(t["status_restored"] == 0 and t["restored_same_bits"] for t in recs), (w, recs)
    paths = [reps[o]["targets"][j]["path"] for j, o in ((0, 0), (1, 1))]
    assert paths[0] == "leaf" and (paths[1].startswith("team") or paths[1] == "cta_hbm"), paths
    _report("pivots")
