"""Incremental steps (april_graph_cholesky_inc) checked kernel by kernel, after EVERY step.

test_gpu_kernels.py checks batch solves front by front; incremental steps are most of the calls of a replay and
are built from other parts: k_linearize / k_step stage 2 at host-supplied points, new Hessian slots and cleared
ranges, descriptors patched in HBM, partial re-factorisation (keep), team fronts re-factored, the pruned
back-substitution (bfirst), the old-pose fallback and escalations to a batch.  After every step these tests check

  * the Hessian in HBM against a ledger of what the reference semantics prescribe (support/inccheck.py), entry by
    entry, with the bound of check_linearize;
  * the device copy of the plan (descriptors, int pool, node2q, q2node, factor slots) and of the factor mirror
    against the host's, bit for bit;
  * every front (local backward error) and y, bit for bit;
  * full-traversal, fallback and escalated steps: the back-substitution of every supernode and the long-double
    residual;
  * pruned steps: the rows [3 bfirst, c) of every listed supernode, that x outside the listed columns is
    bit-identical to x before the step, that every pose whose state changed equals l_point + x(HBM) bit for bit,
    and that no pose outside the listed columns changed.

The step record (asam_dbg_record_steps / asam_dbg_last_step) says what the host asked of the kernels; the tests
assert from it that the scenarios reach the paths they are written for.  CPU tests replay the same scripts through
HostPlan.append and assert the plan-level part of that coverage without a GPU, and show that each new check
catches a wrong result.

Bounds: the constants of test_gpu_kernels.py.  Worst values observed on an H100 80GB HBM3 over all scenarios and
switches: local backward error 1.8e-15 (factor) and 2.9e-15 (rhs); Hessian 6.1 u per sum of contributions;
back-substitution 1.5e-15 (full) and 3.0e-16 (pruned rows); residual 5.8e-16.
"""
from __future__ import annotations

import copy
import json
import os
import subprocess
import sys
from collections import Counter

import numpy as np
import pytest

from aprilsam_b200 import harness as H
from conftest import ROOT
from support import emul
from support import frontcheck as fc
from support import inccheck as ic
from test_gpu_kernels import (BACKSOLVE_TOL, FACTOR_TOL, LINEARIZE_C, RESIDUAL_TOL, RHS_TOL, _full_W, pendant_graph,
                              plan_of, zoo_graph)

LAM = 1e-4  # param->tikhanov of april_graph_cholesky_param_init
BIG = 5000  # above this many poses: listed supernodes every step, all fronts every 25 steps


# ---------------------------------------------------------------------------------------------
# scenario graphs and scripts (shared by the GPU runs and their CPU emulation)
# ---------------------------------------------------------------------------------------------
B_GRAPHS = {"root195": (4, 20, 45), "root198": (4, 20, 46)}
B_DEPTHS = (0, 1, 3)


def b_graph(name):
    return zoo_graph(*B_GRAPHS[name], seed=7)


C_SIZES = [14] + [1] * 4150  # one 14-pose pendant clique, then enough single-pose pendants for k_backsolve_leaf


def c_graph():
    return pendant_graph(C_SIZES, seed=5)


def _top(plan, N):
    """The last pose in the elimination order: the root path of every pose ends there."""
    return int(plan.array("q2node")[N - 1])


def _col(plan, pose, k):
    """The pose at column k of the supernode holding `pose`."""
    q = int(plan.array("node2q")[pose])
    s = int(plan.array("sn_of_q")[q])
    return int(plan.array("q2node")[int(plan.descs()["first"][s]) + k])


def b_steps(depth):
    """A pose hanging under the pose `depth` columns below the top of the root (c = m > 96) of the batch plan, then
    two more poses on top: the first re-factors the (team) root and back-solves it from a column inside a later
    96-column block; the second back-solves it from its last column."""
    return [lambda p, N: dict(new=1, edges=[(int(p.array("q2node")[N - 1 - depth]), N)]),
            lambda p, N: dict(new=1, edges=[(N - 1, N)]),
            lambda p, N: dict(new=1, edges=[(N - 1, N)])]


def c_steps():
    """Scripted edge steps after the batch of c_graph()."""
    nsp = (len(C_SIZES) + 29) // 30
    clique, single = nsp, nsp + 14  # first pose of the 14-clique; the first single-pose pendant

    def three(p, N):
        return dict(new=3, edges=[(_top(p, N), N), (N, N + 1), (N + 1, N + 2), (N, N + 2)], tag="multi_pose")

    def prior(p, N):
        return dict(priors=[N - 2], tag="prior_moved")

    def old_pair(p, N):
        return dict(edges=[(single, nsp - 1)], tag="old_pair")

    def edit(p, N):
        return dict(new=1, edges=[(_top(p, N), N)], edit=5, tag="edit")

    def grow(p, N):
        return dict(new=1, edges=[(_col(p, clique, 7), N)], tag="grow")

    def outgrow(p, N):
        e = [(single + 1, N + k) for k in range(22)] + [(N + k, N + k + 1) for k in range(21)]
        return dict(new=22, edges=e, tag="outgrow")

    def esc(p, N):
        return dict(new=1, edges=[(_top(p, N), N)], policy=1e-300, tag="escalate")

    def after(p, N):
        return dict(new=1, edges=[(_top(p, N), N)], policy=0.0, tag="after")

    return [three, prior, old_pair, edit] + [grow] * 6 + [outgrow, esc, after, after, after]


# ---------------------------------------------------------------------------------------------
# CPU: the scripts through HostPlan.append, with the marking and back-solve lists of solver.c
# ---------------------------------------------------------------------------------------------
def step_lists(p, N0, N, ft, fa, fb, F0):
    """One april_graph_cholesky_inc on a host plan: mark the root paths (old tree), append (or rebuild with the
    order kept: the old-pose fallback), then the back-solve list of a pruned step (solver.c).  Returns the step's
    kind, task list, keep and (bt, bfirst) as the solver would ask for them."""
    order, pos, ppos = p.array("order"), p.array("pos"), p.array("parent_pos")
    marked, new = [], set()
    for f in range(F0, len(ft)):
        for v in ([fa[f], fb[f]] if ft[f] == 1 else [fa[f]]):
            v = int(v)
            if v >= N0:
                new.add(v)
                continue
            while v not in marked:
                marked.append(v)
                pp = ppos[pos[v]]
                if pp < 0:
                    break
                v = int(order[pp])
    desc0, nbl0, nsn0 = p.descs(), p.info()["n_bs_leaf"], p.info()["nsn"]
    r = p.append(N, ft, fa, fb, sorted(marked))
    if r is None:
        p.build(N, ft, fa, fb, order_keep=order[:N0])
        return dict(kind="fallback", tasks=np.zeros(0, np.int32), nwait=np.zeros(0, np.int32),
                    keep=np.zeros(0, np.int32), bt=np.zeros(0, np.int32), bfirst=np.zeros(0, np.int32),
                    moved=False, bs_leaf_broken=False)
    tasks, nwait = r
    d = p.descs()
    out = dict(tasks=tasks, nwait=nwait, keep=p.last_keep,
               moved=any(s < nsn0 and d["f_off"][s] != desc0["f_off"][s] for s in tasks),
               bs_leaf_broken=nbl0 > 0 and p.info()["n_bs_leaf"] == 0)
    if len(marked) + len(new) > 5:
        out.update(kind="full", bt=np.zeros(0, np.int32), bfirst=np.zeros(0, np.int32))
        return out
    order, pos, ppos = p.array("order"), p.array("pos"), p.array("parent_pos")
    n2q, sn_of_q = p.array("node2q"), p.array("sn_of_q")
    children = {}
    for v in range(N):
        pp = ppos[pos[v]]
        if pp >= 0:
            children.setdefault(int(order[pp]), []).append(v)
    jf = {}
    for v in marked + sorted(new):
        for u in [v] + children.get(v, []):
            q = int(n2q[u])
            s0 = s = int(sn_of_q[q])
            while s >= 0 and s not in jf:
                jf[s] = int(d["cb"][s])
                s = int(d["parent"][s])
            jf[s0] = min(jf[s0], q - int(d["first"][s0]))
    bt = np.array(sorted(jf, reverse=True), np.int32)
    bfirst = np.array([jf[s] if jf[s] < d["cb"][s] else 0 for s in bt], np.int32)
    small = len(bt) <= 64 and len(tasks) <= 32 and all(((int(w) >> 24) & 0x7f) <= 1 for w in nwait)
    out.update(kind="k_step" if small else "pruned", bt=bt, bfirst=bfirst)
    return out


class Coverage:
    """What a sequence of steps reached, from step records (GPU) or step_lists (CPU)."""

    def __init__(self):
        self.kinds = Counter()
        self.items = Counter()
        self.edges = set()  # 3 bfirst mod 96 of pruned back-solves of supernodes with c > 96

    def add(self, rec, desc, npose_new, tag=None):
        self.kinds[rec["kind"]] += 1
        if rec.get("escalated"):
            self.kinds["escalated"] += 1
        G = [(int(w) >> 24) & 0x7f for w in rec["nwait"]]
        if rec["kind"] == "k_step" and np.any(rec["keep"] > 0):
            self.items["k_step_keep"] += 1
        if np.any(rec["keep"] > 0):
            self.items["keep"] += 1
        if any(g > 1 for g in G):
            self.items["team_refactored"] += 1
            if not np.any(rec["keep"][np.array(G) > 1] != 0):
                self.items["team_keep0"] += 1
        if rec.get("moved"):
            self.items["moved"] += 1
        if rec.get("bs_leaf_broken"):
            self.items["bs_leaf_broken"] += 1
        if npose_new > 1:
            self.items["multi_pose"] += 1
        if tag:
            self.items[tag] += 1
        if rec["kind"] in ("k_step", "pruned"):
            for s, b in zip(rec["bt"], rec["bfirst"]):
                c = 3 * int(desc["cb"][s])
                if c > 96 and b > 0:
                    self.edges.add((3 * int(b)) % 96)
                    if 3 * int(b) >= 96:
                        self.items["later_block"] += 1

    def summary(self):
        return dict(kinds=dict(self.kinds), items=dict(self.items), bfirst_edges=sorted(self.edges))


def factor_lists(d):
    ft = np.r_[2, np.ones(d.n_edges, dtype=np.int32)].astype(np.int32)
    return ft, np.r_[0, d.ea].astype(np.int32), np.r_[-1, d.eb].astype(np.int32)


def emulate_script(d, steps):
    """The script on host plans only (no numerics, no escalations).  Returns its Coverage."""
    ft, fa, fb = factor_lists(d)
    p = plan_of(d)
    N = d.n_nodes
    cov = Coverage()
    for st in steps:
        spec = st(p, N)
        N0, F0 = N, len(ft)
        N += spec.get("new", 0)
        e = spec.get("edges", [])
        pr = spec.get("priors", [])
        ft = np.r_[ft, np.ones(len(e), np.int32), np.full(len(pr), 2, np.int32)].astype(np.int32)
        fa = np.r_[fa, [a for a, _ in e], pr].astype(np.int32)
        fb = np.r_[fb, [b for _, b in e], np.full(len(pr), -1)].astype(np.int32)
        rec = step_lists(p, N0, N, ft, fa, fb, F0)
        cov.add(rec, p.descs(), N - N0, spec.get("tag"))
    return cov


def a_steps_cpu(m, n):
    """Plan-level emulation of the pose-by-pose replay of the first n poses (no escalations)."""
    db, estart = m.bucketed()
    ft, fa, fb = factor_lists(db.head(2))
    sub = db.head(2)
    p = plan_of(sub)
    cov = Coverage()
    F = len(ft)
    for k in range(2, n):
        e = slice(estart[k], estart[k + 1])
        ft = np.r_[ft, np.ones(estart[k + 1] - estart[k], np.int32)].astype(np.int32)
        fa = np.r_[fa, db.ea[e]].astype(np.int32)
        fb = np.r_[fb, db.eb[e]].astype(np.int32)
        rec = step_lists(p, k, k + 1, ft, fa, fb, F)
        cov.add(rec, p.descs(), 1)
        F = len(ft)
    return cov


def test_scripts_reach_the_incremental_paths_on_host_plans(m3500, built):
    """The plan-level coverage of every scenario, without a GPU: the GPU tests below assert the same items from
    the step records of the real runs, so they cannot become vacuous unnoticed."""
    a = a_steps_cpu(m3500, 400)
    assert a.kinds["k_step"] > 0 and a.items["k_step_keep"] > 0 and a.kinds["full"] > 0, a.summary()
    edges, later = set(), 0
    for name in B_GRAPHS:
        for depth in B_DEPTHS:
            b = emulate_script(b_graph(name), b_steps(depth))
            assert b.items["team_refactored"] > 0 and b.items["team_keep0"] > 0, (name, depth, b.summary())
            assert b.kinds["pruned"] > 0, (name, depth, b.summary())
            edges |= b.edges
            later += b.items["later_block"]
    assert edges >= {0, 93} and later > 0, edges
    c = emulate_script(c_graph(), c_steps())
    for item in ("multi_pose", "prior_moved", "moved", "bs_leaf_broken", "keep"):
        assert c.items[item] > 0, (item, c.summary())
    assert c.kinds["fallback"] == 1, c.summary()


# ---------------------------------------------------------------------------------------------
# CPU: the new checks catch wrong results
# ---------------------------------------------------------------------------------------------
def _emulated_zoo_steps():
    """Batch of a zoo graph, then one incremental step (a pose under the top of a 32-pose root: too wide to take the
    pose in, so the old root gets the new pose's supernode as parent), emulated: the plan, the Hessian
    (ledger-style, evaluation points per factor), the fronts, the pruned back-solve list."""
    d = zoo_graph(2, 10, 22, seed=3)
    ft, fa, fb = factor_lists(d)
    fz = np.vstack([[0, 0, 0], d.ez]); fW = np.vstack([[1e4, 0, 0, 0, 1e4, 0, 0, 0, 1e3], d.eW])
    p = plan_of(d)
    N0, F0 = d.n_nodes, len(ft)
    Hs = emul.Hessian(N0, p.info()["n_slots"]); Hs.reset(N0, LAM)
    Hs.linearize(range(F0), ft, fa, fb, fz, fW, d.init, d.init, p.array("node2q"), p.array("fslot"))
    fr = emul.Fronts(); fr.ensure(N0)
    emul.factor(fr, Hs, p.descs(), p.array("ipool"), p.array("q2node"), p.array("tasks"), p.array("nwait"))
    emul.backsolve(fr, p.descs(), p.array("ipool"), np.arange(p.info()["nsn"] - 1, -1, -1))
    x_before = fr.x.copy()
    top, below = _top(p, N0), int(p.array("q2node")[N0 - 2])  # a new pose on two edges: the old poses move
    rng = np.random.default_rng(1)
    lp = np.r_[d.init, d.init[top:top + 1] + 0.1]
    ft = np.r_[ft, 1, 1].astype(np.int32); fa = np.r_[fa, top, below].astype(np.int32)
    fb = np.r_[fb, N0, N0].astype(np.int32)
    fz = np.r_[fz, rng.standard_normal((2, 3))]; fW = np.r_[fW, _full_W(rng, 2)]
    desc0 = p.descs()
    rec = step_lists(p, N0, N0 + 1, ft, fa, fb, F0)
    assert rec["kind"] == "k_step" and len(rec["bt"]) > 0
    info = p.info()
    Hs.grow(N0 + 1, info["n_slots"]); fr.ensure(N0 + 1)
    pts = np.c_[lp[fa[F0:]], lp[fb[F0:]]]
    Hs.linearize(range(F0, F0 + 2), ft, fa, fb, fz, fW, lp, lp, p.array("node2q"), p.array("fslot"), pts=pts)
    desc, ipool = p.descs(), p.array("ipool")
    emul.factor(fr, Hs, desc, ipool, p.array("q2node"), rec["tasks"], rec["nwait"], keep=rec["keep"])
    fr_b = copy.deepcopy(fr)
    ic.backsolve(fr, desc, ipool, rec["bt"], rec["bfirst"])
    led = ic.Ledger(LAM)
    led.ft, led.fa, led.fb, led.fz, led.fW = ft, fa, fb, fz, fW
    led.pts = np.c_[lp[fa], np.where((fb >= 0)[:, None], lp[np.maximum(fb, 0)], 0.0)]
    led.lamv = np.r_[np.full(N0, LAM), 0.0]
    return dict(p=p, Hs=Hs, fr=fr, fr_b=fr_b, x_before=x_before[:3 * N0], rec=rec, led=led, desc0=desc0,
                factors=(ft, fa, fb, fz, fW), N=N0 + 1)


def test_incremental_checks_catch_faults(built):
    """On an emulated step the checks pass; a new factor's contribution dropped from one node, a descriptor with a
    stale parent, a pruned back-substitution that also rewrites the column before bfirst, and one that stops one
    column late each fail their check."""
    e = _emulated_zoo_steps()
    p, Hs, fr, rec, led, N = e["p"], e["Hs"], e["fr"], e["rec"], e["led"], e["N"]
    snap = fc.snapshot_from_emulation(p, Hs, fr)
    fslot = p.array("fslot")
    assert led.check(snap, fslot) < LINEARIZE_C
    host = ic.host_plan_arrays(p, e["factors"])
    assert ic.plan_mismatches(copy.deepcopy(host), host) == {}
    mask = ic.listed_columns(snap.desc, N, rec["bt"], rec["bfirst"])
    assert ic.check_backsolve_rows(snap, rec["bt"], rec["bfirst"]) < BACKSOLVE_TOL
    assert ic.check_pruned_x(e["x_before"], snap.x, mask) == 0
    assert any(b > 0 for b in rec["bfirst"])

    # 1. the new factor's contribution to the diagonal block of its new pose dropped
    m1 = copy.copy(snap)
    m1.Adiag = snap.Adiag.copy()
    m1.Adiag[N - 1] = 0.0
    assert led.check(m1, fslot) > 1e6 * LINEARIZE_C
    # 2. the old root's descriptor with its parent as it was before the step (-1: the patch did not arrive)
    d0, d1 = e["desc0"], p.descs()
    stale = [int(s) for s in rec["tasks"] if int(s) < len(d0["parent"]) and d0["parent"][s] != d1["parent"][s]]
    assert stale, "the step re-parents an old supernode"
    bad = copy.deepcopy(host)
    bad["sn"].reshape(-1, 12)[stale[0], 3] = d0["parent"][stale[0]]
    assert ic.plan_mismatches(bad, host) == {"sn": [(stale[0], 3)]}
    # 3. / 4. pruned back-substitutions that start one column early / one column late
    k = int(np.argmax(rec["bfirst"]))
    s, b = int(rec["bt"][k]), int(rec["bfirst"][k])
    for shift in (-1, 1):
        fr2 = copy.deepcopy(e["fr_b"])
        bf = rec["bfirst"].copy()
        bf[k] = b + shift
        ic.backsolve(fr2, snap.desc, snap.ipool, rec["bt"], bf)
        x2 = fr2.x[:3 * N].copy()
        if shift < 0:  # rewrites the column before bfirst: x outside the listed columns changed
            assert ic.check_pruned_x(e["x_before"], x2, mask) > 0
        else:  # stops one column late: row 3 bfirst of the supernode is stale
            m4 = copy.copy(snap)
            m4.x = x2
            first = int(snap.desc["first"][s])
            assert not np.array_equal(x2[3 * (first + b):3 * (first + b + 1)], snap.x[3 * (first + b):3 * (first + b + 1)])
            assert ic.check_backsolve_rows(m4, rec["bt"], rec["bfirst"]) > 1e3 * BACKSOLVE_TOL


# ---------------------------------------------------------------------------------------------
# GPU: every step checked
# ---------------------------------------------------------------------------------------------
class StepChecker:
    """Runs incremental calls on a live Harness and checks each one (see the module docstring)."""

    def __init__(self, h, lam=LAM):
        self.L = ic.dev_api()
        self.h = h
        self.dev = None
        self.ledger = ic.Ledger(lam)
        self.cov = Coverage()
        self.worst = Counter()
        self.nstep = 0
        self.factors = None

    def __enter__(self):  # step records on while the checker runs (they are process-wide)
        self.rec = ic.recording(self.L).__enter__()
        return self

    def __exit__(self, *exc):
        self.rec.__exit__(*exc)

    def _w(self, k, v):
        self.worst[k] = max(self.worst[k], float(v))

    def _sync_factors(self):
        """The caller's factors (what the device mirror must hold), read once and then as they are appended."""
        h = self.h
        if self.factors is None:
            self.factors = list(ic.factors_of(h))
        elif len(self.factors[0]) < h.n_factors:
            new = ic.factors_of(h, len(self.factors[0]))
            self.factors = [np.r_[a, b] for a, b in zip(self.factors, new)]

    def edited(self, i):
        self._sync_factors()
        _, _, _, z, W = self.h.factor(i)
        self.factors[3][i], self.factors[4][i] = z, W

    def batch(self, run=None):
        """An explicit batch solve (or `run`, a call that makes one), checked like a step that escalated."""
        n = self.h.n_nodes
        (run or self.h.batch)()
        self.dev = self.L.asam_dbg_dev_of_graph(self.h.graph_ptr())
        self.ledger.batch(self.h)
        self._check(dict(kind="batch", escalated=True), np.full((self.h.n_nodes, 3), np.nan), np.zeros(3 * n),
                    self.h.n_nodes, full=True, all_fronts=self.h.n_nodes <= BIG)

    def step(self, run, tag=None, all_fronts=None):
        h, L = self.h, self.L
        N0 = h.n_nodes
        x0 = np.zeros(3 * N0)
        fc._ok(L, L.asam_download_x(self.dev, 0, N0, x0.ctypes.data_as(fc._dp)), "download_x")
        st0 = h.states()
        plan = fc.borrowed_plan(L, h.param_ptr())
        desc0, nbl0, nsn0 = plan.descs(), plan.info()["n_bs_leaf"], plan.info()["nsn"]
        nb0 = ic.batch_count(L)
        run()
        N = h.n_nodes
        rec = ic.last_step(L, h.param_ptr())
        escalated = ic.batch_count(L) > nb0
        assert escalated == rec["escalated"] or rec["kind"] == "none", rec
        lp = h.l_points()
        if escalated:  # a batch solve ran last: every pose's state is l_point + x
            self.ledger.batch(h)
            st_before = np.full((N, 3), np.nan)
        else:  # a new pose's state at the call is its l_point
            st_before = np.r_[st0, lp[N0:]]
            self.ledger.add(h, lp, st_before)
        d = plan.descs()
        rec["moved"] = (not escalated and rec["kind"] != "fallback" and
                        any(s < nsn0 and d["f_off"][s] != desc0["f_off"][s] for s in rec["tasks"]))
        rec["bs_leaf_broken"] = not escalated and rec["kind"] != "fallback" and nbl0 > 0 and plan.info()["n_bs_leaf"] == 0
        self.cov.add(rec, d, N - N0, tag)
        self.nstep += 1
        big = N > BIG
        if all_fronts is None:
            all_fronts = not big or self.nstep % 25 == 0
        all_fronts = all_fronts or escalated  # (the step's task list names supernodes of the plan before the batch)
        full = escalated or rec["kind"] in ("full", "fallback")
        self._check(rec, st_before, x0, N, full=full, all_fronts=all_fronts)
        return rec

    def _check(self, rec, st_before, x0, N, full, all_fronts=True):
        h, L = self.h, self.L
        what = f"step {self.nstep} {rec['kind']}" + (" escalated" if rec.get("escalated") else "")
        listed = None
        if not all_fronts:
            listed = sorted(set(int(s) for s in rec.get("tasks", [])) | set(int(s) for s in rec.get("bt", [])))
        snap = ic.snapshot(h, L, which=listed)
        self._sync_factors()
        fslot = snap.plan.array("fslot")
        wf, wr, per = fc.check_fronts(snap, listed)
        assert wf < FACTOR_TOL and wr < RHS_TOL, (what, fc.describe(per))
        self._w("factor", wf); self._w("rhs", wr)
        ybad = (fc.check_y(snap) if listed is None else ic.check_y(snap, listed))
        assert ybad == 0, (what, ybad)
        lin = self.ledger.check(snap, fslot)
        self._w("linearize", lin)
        assert lin < LINEARIZE_C, (what, lin)
        bad = ic.plan_mismatches(ic.read_device_plan(L, self.dev, snap.plan, len(self.factors[0])),
                                 ic.host_plan_arrays(snap.plan, self.factors))
        assert bad == {}, (what, bad)
        n2q = snap.node2q
        if full:
            if listed is None:
                bs = fc.check_backsolve_local(snap)
                self._w("backsolve", bs)
                assert bs < BACKSOLVE_TOL, (what, bs)
                A, b = fc.system(snap, self.ledger.ft, self.ledger.fa, self.ledger.fb, fslot)
                res = ic.check_residual(A, b, snap.x)
                self._w("residual", res)
                assert res < RESIDUAL_TOL, (what, res)
            mask = np.ones(N, bool)
        else:
            bt, bf = rec["bt"], rec["bfirst"]
            bs = ic.check_backsolve_rows(snap, bt, bf)
            self._w("backsolve_pruned", bs)
            assert bs < BACKSOLVE_TOL, (what, bs)
            mask = ic.listed_columns(snap.desc, N, bt, bf)
            nx = ic.check_pruned_x(x0, snap.x, mask)
            assert nx == 0, (what, "x outside the listed columns changed", nx)
        st = h.states()
        sb = np.where(np.isnan(st_before), np.inf, st_before)
        wrong, outside, nchanged = ic.check_states(sb, st, h.l_points(), snap.x, n2q, mask)
        assert wrong == 0 and outside == 0, (what, "states", wrong, outside, nchanged)

    def report(self, name):
        out = dict(worst=dict(self.worst), steps=self.nstep, **self.cov.summary())
        print(f"KERNELCHECK incremental {name} " + json.dumps(out))
        return out


def run_replay_a(m, nthreshold):
    d = m.head(400)
    with H.Harness("b200", nthreshold=nthreshold) as h:
        with StepChecker(h) as chk:
            h.replay_begin(d)
            chk.batch(lambda: h.replay_to(1))
            for k in range(1, d.n_nodes):
                chk.step(lambda: h.replay_to(k + 1))
            return chk.report(f"A nthreshold={nthreshold}")


def _add_step(h, chk, spec, rng):
    """Add what one script step asks for (new poses near the pose they hang under, edges with measurements taken
    from the current states plus noise, priors at the current state plus noise) and run the incremental call."""
    N = h.n_nodes
    st = h.states()
    e = spec.get("edges", [])
    new = spec.get("new", 0)
    place = {}
    for a, b in e:
        if b >= N and b not in place:
            place[b] = (place[a] if a in place else st[a]) + np.r_[0.7 * rng.standard_normal(2), 0.2 * rng.standard_normal()]
    for k in range(new):
        h.add_node(place.get(N + k, st[-1]))
    pose = np.r_[st, np.array([place.get(N + k, st[-1]) for k in range(new)]).reshape(-1, 3)]
    for a, b in e:
        c, s = np.cos(pose[a, 2]), np.sin(pose[a, 2])
        dd = pose[b] - pose[a]
        z = np.r_[c * dd[0] + s * dd[1], -s * dd[0] + c * dd[1], emul.mod2pi(dd[2])] + 0.01 * rng.standard_normal(3)
        h.add_xyt(int(a), int(b), z, _full_W(rng, 1)[0])
    for a in spec.get("priors", []):
        assert not np.array_equal(st[a], h.l_points()[a]), "the prior's pose has moved since it was linearised"
        h.add_xytpos(int(a), st[a] + 0.01 * rng.standard_normal(3), _full_W(rng, 1)[0])
    if "edit" in spec:
        i = spec["edit"]
        _, _, _, z, W = h.factor(i)
        h.set_factor(i, z + 0.05, 2.0 * W)
        h.chi2()  # re-uploads the factor mirror; the Hessian must not change before the next batch
        chk.edited(i)
    if "policy" in spec:
        h.set_policy_ratio(spec["policy"])
    return chk.step(h.inc, spec.get("tag"))


def run_script(d, steps, name, seed=0, nthreshold=100):
    rng = np.random.default_rng(seed)
    with H.Harness("b200", nthreshold=nthreshold) as h:
        with StepChecker(h) as chk:
            h.load_full(d)
            chk.batch()
            for st in steps:
                plan = fc.borrowed_plan(chk.L, h.param_ptr())
                _add_step(h, chk, st(plan, h.n_nodes), rng)
            return chk.report(name)


def run_b():
    outs = []
    for name in B_GRAPHS:
        for depth in B_DEPTHS:
            outs.append(run_script(b_graph(name), b_steps(depth), f"B {name} depth={depth}"))
    return outs


def run_c():
    # escalations only where the script asks for one (the poses it adds start far from where they settle)
    return run_script(c_graph(), c_steps(), "C", nthreshold=1 << 30)


def assert_a(outs):
    kinds = sum((Counter(o["kinds"]) for o in outs), Counter())
    items = sum((Counter(o["items"]) for o in outs), Counter())
    assert kinds["k_step"] > 0 and items["k_step_keep"] > 0 and kinds["full"] > 0, (kinds, items)
    assert kinds["escalated"] > 0, kinds


def assert_b(outs):
    edges = set()
    for o in outs:
        assert o["items"].get("team_refactored", 0) > 0 and o["items"].get("team_keep0", 0) > 0, o
        assert o["kinds"].get("pruned", 0) > 0, o
        edges |= set(o["bfirst_edges"])
    assert edges >= {0, 93} and sum(o["items"].get("later_block", 0) for o in outs) > 0, edges


def assert_c(o):
    for item in ("multi_pose", "prior_moved", "moved", "bs_leaf_broken", "keep", "edit", "after"):
        assert o["items"].get(item, 0) > 0, (item, o)
    assert o["kinds"].get("fallback", 0) == 1 and o["kinds"].get("escalated", 0) == 1, o


@pytest.mark.gpu
def test_incremental_m3500_replay(m3500):
    """A. M3500, first 400 poses pose by pose: at the default nthreshold and at 10 (escalations mid-replay, steps
    continuing from the new batch plan)."""
    assert_a([run_replay_a(m3500, 100), run_replay_a(m3500, 10)])


@pytest.mark.gpu
def test_incremental_appends_into_team_root():
    """B. Batch, then poses appended under the top columns of a root front of c = m = 195 / 198."""
    assert_b(run_b())


@pytest.mark.gpu
def test_incremental_scripted_edge_steps():
    """C. Several poses in one call, a prior on a moved pose, the old-pose fallback, an edited z / W, a front that
    outgrows its reservation, a pendant that outgrows the warp back-solve, an escalation and steps after it."""
    assert_c(run_c())


@pytest.mark.gpu
def test_incremental_sparse_30k():
    """D. 29 700 poses of manhattan_sparse(30000) batch-solved at the ground truth, then 200 poses one by one."""
    from aprilsam_b200 import datasets
    d = datasets.manhattan_sparse(30000, seed=1)
    s0 = 29700
    sub = d.head(s0)
    with H.Harness("b200") as h:
        with StepChecker(h) as chk:
            h.replay_begin(d)
            h.load_full(sub)
            h.set_states(sub.truth)
            chk.batch()
            for k in range(s0, s0 + 200):
                chk.step(lambda: h.replay_to(k + 1, want_chi2=False), all_fronts=(k % 25 == 24))
            out = chk.report("D sparse30k")
    assert out["items"].get("team_refactored", 0) > 0, out


# ---------------------------------------------------------------------------------------------
# GPU: A-C under the switches of the incremental path (one process each: they are read at context creation)
# ---------------------------------------------------------------------------------------------
INC_SWITCHES = {"keep0": {"ASAM_KEEP": "0"}, "small_step0": {"ASAM_SMALL_STEP": "0"},
                "bs_threads128": {"ASAM_BS_THREADS": "128"}}


def _worker():
    m = H.PoseGraphData.load(os.path.join(ROOT, "tests", "golden", "m3500.npz"))
    out = dict(a=[run_replay_a(m, 100), run_replay_a(m, 10)], b=run_b(), c=run_c())
    print("RESULT " + json.dumps(out))


@pytest.mark.gpu
@pytest.mark.parametrize("switch", list(INC_SWITCHES))
def test_incremental_switches(switch):
    e = dict(os.environ)
    e.update(INC_SWITCHES[switch])
    here = os.path.dirname(os.path.abspath(__file__))
    code = f"import sys; sys.path[:0] = [{ROOT!r}, {here!r}]; import test_gpu_incremental as t; t._worker()"
    r = subprocess.run([sys.executable, "-c", code], env=e, capture_output=True, text=True, timeout=1800, cwd=ROOT)
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    print("\n".join(ln for ln in r.stdout.splitlines() if ln.startswith("KERNELCHECK")))
    out = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1][len("RESULT "):])
    assert_b(out["b"])
    assert_c(out["c"])
    kinds = sum((Counter(o["kinds"]) for o in out["a"]), Counter())
    assert kinds["escalated"] > 0 and kinds["full"] > 0, kinds
    if switch == "small_step0":
        assert kinds["k_step"] == 0 and kinds["pruned"] > 0, kinds
