"""The factorisation status on every batch kernel path and in incremental steps: failed pivots at chosen columns of chosen fronts, valid pivots across
the double range, and a clean context after a failure.

The status word (asam_factor_status, asam_download_x_status) is all that stands between an indefinite system and a
wrong solution returned without complaint.  Each kernel path computes its own Cholesky pivots and flags a failure with
its own atomicCAS(err, 0, 1 + s): panel_factor (cta_front in shared memory and out of HBM, the team diagonal block)
and the warp loop of k_factor_leaf.

How a failure is placed: the graph gets extra xytpos priors (SPD W; priors add no edges, so the plan is unchanged) on
the poses to be targeted and is solved once through the public API.  After that only the C-ABI is used on its device
context (april_graph_cholesky aborts the process on a failed pivot): the perturbed W of one prior is uploaded, the
Hessian reset and linearised, the system factored and back-solved, the status read.  A prior adds W to its pose's
diagonal block; changing W_kk so that A'_kk = -max(1, |A_kk|) makes the pivot of column k of that pose at most A'_kk < 0
whatever the Schur updates are, and leaves every column eliminated earlier alone.  The status must then be exactly
1 + s, s the supernode owning that column: its ancestors fail too (on NaNs), but only after s has set the word, and
independent subtrees do not fail.  The perturbed Hessian is read back and checked against the float64 expectation, and
the float64 elimination of it (support/pivotcheck.first_failure) must meet its first non-positive or NaN pivot exactly
at the (supernode, column) the test names.

After every failure the original system is restored and factored twice: status 0 both times, fronts, y and x
bit-identical between the two runs and -- when the restored Hessian is bit-identical to the baseline's -- to the
baseline, which itself passes the frontcheck bounds of test_gpu_kernels.py.  That is what shows that clear_status and
the kernels' own at-rest invariants (team barriers, stage flags, back-solve epochs) hold after a failure on every path.

Valid pivots: a pose held by a diagonal prior alone, with no Tikhonov term, has its pivots set to 2^-1074 ... DBL_MAX;
the status must be 0 and L_kk, y and x must be the float64 values.
"""
from __future__ import annotations

import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from aprilsam_b200 import harness as H
from conftest import ROOT
from support import emul
from support import frontcheck as fc
from support import pivotcheck as pc
from support.hostplan import HostPlan
from test_gpu_kernels import (BACKSOLVE_TOL, FACTOR_TOL, PRIOR_W, RESIDUAL_TOL, RHS_TOL, TEAM_ENV, ZOO, _full_W,
                              env_set, path_table, pendant_graph, pendant_sizes, zoo)
from test_gpu_solo_front import SOLO_ENV, solo_graph, staged_width

LAM = 1e-4  # the Tikhonov term of april_graph_cholesky_param_init

# ---------------------------------------------------------------------------------------------
# what is targeted: group -> (environment, [(graph, path, front selector)]); a group runs in one process
# ---------------------------------------------------------------------------------------------
_SMEM = [("smem159_c12", "cta_smem", 159), ("smem159_c3", "cta_smem", 159), ("smem_n51", "cta_smem", "n51")]
# team162_c48: all of c in the first 48-column diagonal block.  The status names a supernode, not a column, and a
# failed pivot turns every later column of its front NaN: in a wider front a later panel would flag the same 1 + s
# and hide a first block that flags nothing
_TEAM = [("team162_c48", "team", 162), ("team162_c51", "team", 162), ("team162_c99", "team", 162), ("wide", "team", None)]
GROUPS = {
    "leaf": ({}, [("pendants", "leaf", 48)]),
    "leaf63": ({"ASAM_LEAF_MAX_M": "63"}, [("pendants63", "leaf", 63)]),
    "cta_smem": ({}, _SMEM),
    "smem_mma2": ({"ASAM_SMEM_MMA": "2"}, _SMEM),
    "pb_smem24": ({"ASAM_PB_SMEM": "24"}, _SMEM),
    "cta_hbm": (SOLO_ENV, [("m162_c51", "cta_hbm", 162), ("m555_c90", "cta_hbm", 555), ("m903_c60", "cta_hbm", 903)]),
    **{f"team{g}": (TEAM_ENV[g], _TEAM) for g in (1, 2, 3, 5)},
    "team_full": ({}, _TEAM),
}
# device switches read once per process (process-wide __constant__ symbols, statics): these groups run in a subprocess
SUBPROCESS = {"leaf63", "smem_mma2", "pb_smem24"}
# the group that also carries the other kinds of failure (exact zeros, NaNs, two seeds) on one graph of its path
EXTRA_KINDS = {"leaf": "pendants", "cta_smem": "smem_n51", "cta_hbm": "m555_c90", "team_full": "wide"}
# pivots of the isolated pose in the valid-range cases, three per 3x3 block, and the prior's residual: at least 1 so
# that J'Wr does not underflow to 0 at 2^-1074, below 1 where W * r would overflow
EXTREME = [((2.0 ** -1074, 2.0 ** -1022, 2.0 ** -121), (1.5, -1.25, 1.0)),
           ((2.0 ** -120, 2.0 ** 120, 2.0 ** 121), (1.5, -1.25, 1.0)),
           ((2.0 ** 1023, np.finfo(np.float64).max, 1.0), (0.75, -0.625, 1.0))]


def graph(name):
    if name == "pendants":
        return pendant_graph(pendant_sizes())
    if name == "pendants63":
        return pendant_graph(pendant_sizes(True))
    return zoo(name) if name in ZOO else solo_graph(name)


def columns(path, m, c):
    """Columns of the target front (3 (q - first) + k) to fail, per path: both sides of the 3x3 and 12-column steps,
    the diagonal-block stages of team fronts, the first columns of later (staged) panels, the last column."""
    if path == "leaf":
        js = [0, 1, 2, c - 1]
    elif path == "cta_smem":
        js = [0, 1, 2, 11, 12, c - 1]
    elif path == "cta_hbm":
        w = staged_width(m)
        js = [0, 11, 12, w, 2 * w, c - 1]
    else:
        js = [0, 12, 24, 36, 47, 48, 96, c - 1]
    return sorted(set(j for j in js if 0 <= j < c))


def factor_list(d, priors):
    """(ftype, fa, fb, fz, fW) in the harness's order: load_full's prior on pose 0, the edges, then `priors`."""
    P = len(priors)
    ftype = np.r_[2, np.ones(d.n_edges, np.int32), np.full(P, 2)].astype(np.int32)
    fa = np.r_[0, d.ea, [i for i, _, _ in priors]].astype(np.int32)
    fb = np.r_[-1, d.eb, np.full(P, -1)].astype(np.int32)
    fz = np.vstack([[0.0, 0.0, 0.0], d.ez] + [z for _, z, _ in priors]) if P else np.vstack([[0.0, 0.0, 0.0], d.ez])
    fW = np.vstack([PRIOR_W, d.eW] + [W for _, _, W in priors]) if P else np.vstack([PRIOR_W, d.eW])
    return ftype, fa, fb, fz.reshape(-1, 3), fW.reshape(-1, 9)


class Target:
    """One graph of a group: the plan (priors included), the target front, the priors and the failure cases.

    A case is a dict: kind, s (target front), col (its column, or None), seeds [(node, k)] for negative pivots,
    W {factor: W} and lp {node: point} uploads that do not depend on the Hessian, lam, expect (supernodes whose
    1 + s the status may be), at (predicted (supernode, column) of the first failure, column None = any)."""

    def __init__(self, gname, path, sel, env, extra):
        self.name, self.path, self.env = gname, path, env
        self.d = d = graph(gname)
        p0 = self._plan([])
        pt = path_table(p0)
        cand = [(s, f) for s, f in pt.items() if f[0] == path or (path == "team" and f[0].startswith("team"))]
        if sel == "n51":
            cand = [(s, f) for s, f in cand if f[1] - f[2] == 51]
        elif sel is not None:
            cand = [(s, f) for s, f in cand if f[1] == sel]
        assert cand, (gname, path, sel, sorted(set(pt.values()))[:20])
        desc, q2node = p0.descs(), p0.array("q2node")
        # the widest front of the path that has a parent (a failure must not reach the ancestors first)
        self.s, (self.label, self.m, self.c, _) = max(cand, key=lambda t: (int(desc["parent"][t[0]]) >= 0, t[1][2], -t[0]))
        self.cols = columns(path, self.m, self.c)
        nodes = {j: pc.column(desc, q2node, self.s, j) for j in self.cols}
        self.cases = [dict(kind="negative", s=self.s, col=j, seeds=[nodes[j]], expect={self.s}, at=(self.s, j))
                      for j in self.cols]
        targets = {n for n, _ in nodes.values()}
        if extra:
            self._extra_cases(p0, desc, q2node, pt, targets)
        rng = np.random.default_rng(11)
        truth = d.truth if d.truth is not None else d.init
        self.priors = [(int(i), truth[i] + 0.01 * rng.standard_normal(3), _full_W(rng, 1)[0]) for i in sorted(targets)]
        if hasattr(self, "iso"):
            # the isolated pose's residual is >= 1 in every component, so that J'Wr stays non-zero down to W = 2^-1074
            k = [i for i, _, _ in self.priors].index(self.iso)
            self.priors[k] = (self.iso, d.init[self.iso] + np.array([1.5, -1.25, 1.0]), self.priors[k][2])
        self.prior_f = {i: 1 + d.n_edges + k for k, (i, _, _) in enumerate(self.priors)}
        self.factors = factor_list(d, self.priors)
        self.plan = self._plan(self.priors)

    def _plan(self, priors):
        ft, fa, fb, _, _ = factor_list(self.d, priors)
        with env_set(self.env):
            return HostPlan().build(self.d.n_nodes, ft, fa, fb)

    def _extra_cases(self, p0, desc, q2node, pt, targets):
        s, first, cb = self.s, int(desc["first"][self.s]), int(desc["cb"][self.s])
        node2q, sn_of_q = p0.array("node2q"), p0.array("sn_of_q")
        ft, fa, fb, _, _ = factor_list(self.d, [])
        # a NaN in W of an edge inside the target front: the front fails at the earlier pose of the edge
        own = lambda i: first <= node2q[i] < first + cb  # noqa: E731
        f = next(f for f in range(len(ft)) if ft[f] == 1 and own(fa[f]) and own(fb[f]))
        q = min(node2q[fa[f]], node2q[fb[f]])
        self.cases.append(dict(kind="nan_W", s=s, col=3 * int(q - first), edge=int(f), expect={s},
                               at=(s, 3 * int(q - first))))
        # a NaN l_point: the pose and its neighbours get NaN blocks; the first position among them fails
        i = int(q2node[first + cb // 2])
        nb = pc.neighbours((ft, fa, fb), i)
        qm = int(min(node2q[[i] + nb]))
        # the fronts of the pose and its neighbours lie on one root path: the first position fails first, with no
        # race against a failure in a disjoint subtree
        owners = {int(sn_of_q[node2q[v]]) for v in [i] + nb}
        assert owners <= {int(sn_of_q[qm]), *pc.ancestors(desc, int(sn_of_q[qm]))}, (self.name, owners)
        self.cases.append(dict(kind="nan_lp", s=int(sn_of_q[qm]), col=None, node=i, expect={int(sn_of_q[qm])},
                               at=(int(sn_of_q[qm]), None)))
        # two seeds: the target front and its parent (the descendant must be reported) ...
        par = int(desc["parent"][s])
        if par >= 0:
            pn = pc.column(desc, q2node, par, 0)
            targets.add(pn[0])
            self.cases.append(dict(kind="two_nested", s=s, col=0, seeds=[pc.column(desc, q2node, s, 0), pn],
                                   expect={s}, at=(s, 0)))
        if self.path == "leaf":
            # ... and two fronts in disjoint subtrees (either may be reported)
            anc = set(pc.ancestors(desc, s))
            other = next(t for t, f in sorted(pt.items()) if f[0] == "leaf" and t != s and t not in anc
                         and s not in pc.ancestors(desc, t) and f[2] >= 3)
            on = pc.column(desc, q2node, other, 0)
            targets.add(on[0])
            self.cases.append(dict(kind="two_disjoint", s=s, col=0, seeds=[pc.column(desc, q2node, s, 0), on],
                                   expect={s, other}, at=None))
            # exact zero pivots on the pose no factor touches (a root front of c = m = 3), no Tikhonov term:
            # W = 0 gives a00 == 0, diag(w, 0, w) gives d1 == 0, diag(w, w, 0) gives d2 == 0
            iso = self.d.n_nodes - 1
            si = int(sn_of_q[node2q[iso]])
            assert int(desc["mb"][si]) == 1 and int(desc["cb"][si]) == 1, "the last pose is isolated"
            assert pt[si][0] == "leaf", pt[si]
            targets.add(iso)
            self.iso, self.s_iso = iso, si
            for k in range(3):
                W = np.diag([0.0 if (j == k or k == 0) else 400.0 for j in range(3)]).reshape(9)
                self.cases.append(dict(kind="zero", s=si, col=k, Wiso=W, lam=0.0, expect={si}, at=(si, k)))

    # -- the uploads of a case --------------------------------------------------------------
    def uploads(self, case, Ad, lp):
        """({factor: W}, {node: l_point}) of a case; negative pivots are placed against the Hessian Ad of the
        unperturbed system (with its Tikhonov term)."""
        W, P = {}, {}
        _, _, _, _, fW = self.factors
        for node, k in case.get("seeds", []):
            f = self.prior_f[node]
            W[f] = pc.negative_W(fW[f], Ad[node][k, k], k)
        if "edge" in case:
            W[case["edge"]] = pc.nan_W(fW[case["edge"]])
        if "Wiso" in case:
            W[self.prior_f[self.iso]] = case["Wiso"]
        if "node" in case:
            P[case["node"]] = np.full(3, np.nan)
        return W, P

    def perturbed(self, W, P):
        """The factor list with the W uploads applied (the l_point uploads go to the points of hessian_ref)."""
        ft, fa, fb, fz, fW = self.factors
        fW = fW.copy()
        for f, w in W.items():
            fW[f] = w
        return (ft, fa, fb, fz, fW)

    def describe(self, case):
        """path, graph, m, c of the front the case fails, column, kind, expected status."""
        path, m, c, _ = path_table(self.plan)[case["s"]]
        return (f"{path} {self.name} s={case['s']} m={m} c={c} col={case['col']} kind={case['kind']} "
                f"expected={sorted(1 + s for s in case['expect'])}")


def targets_of(group):
    env, specs = GROUPS[group]
    return [Target(g, p, sel, env, EXTRA_KINDS.get(group) == g) for g, p, sel in specs]


# ---------------------------------------------------------------------------------------------
# CPU: the table is reached, the priors leave the plan alone, the float64 elimination fails where predicted
# ---------------------------------------------------------------------------------------------
PLAN_ARRAYS = ("order", "node2q", "q2node", "sn_of_q", "ipool", "tasks", "nwait", "btasks", "desc", "leaf_tasks")


@pytest.mark.parametrize("group", list(GROUPS))
def test_targets_reach_every_path(built, group):
    """Every (path, column) row of the target table exists in the host plans, with the switches of the group."""
    ts = targets_of(group)
    for t in ts:
        assert path_table(t.plan)[t.s][0] == t.label
        if group.startswith("team") and group != "team_full":
            assert t.label == group, (t.name, t.label)
        if group == "team_full":
            assert int(t.label[4:]) > 5 or t.name != "wide", t.label
        assert t.label == t.path or (t.path == "team" and t.label.startswith("team"))
        assert t.cols[0] == 0 and t.cols[-1] == t.c - 1
    by = {t.name: t for t in ts}
    if group in ("leaf", "leaf63"):
        assert by[ts[0].name].m == (48 if group == "leaf" else 63) and {1, 2} <= set(ts[0].cols)
    if group == "cta_smem":
        assert {(t.m, t.c) for t in ts} == {(159, 12), (159, 3), (126, 75)}
        assert {11, 12} <= set(by["smem_n51"].cols)
    if group == "cta_hbm":
        # the first columns of the 2nd and 3rd staged panel of 48 / 36 / 24 columns
        assert [staged_width(t.m) for t in ts] == [48, 36, 24]
        assert {36, 72} <= set(by["m555_c90"].cols) and {24, 48} <= set(by["m903_c60"].cols)
    if group.startswith("team"):
        assert {0, 12, 24, 36, 47, 48} <= set(by["wide"].cols) and 96 in by["wide"].cols
        assert by["team162_c48"].c == 48 and by["team162_c48"].cols == [0, 12, 24, 36, 47]
    if group in EXTRA_KINDS:
        kinds = {c["kind"] for t in ts for c in t.cases}
        assert {"negative", "nan_W", "nan_lp", "two_nested"} <= kinds
        if group == "leaf":
            assert {"zero", "two_disjoint"} <= kinds


@pytest.mark.parametrize("name", ["pendants", "smem_n51", "m555_c90", "wide"])
def test_priors_leave_the_plan_unchanged(built, name):
    group = next(g for g, n in EXTRA_KINDS.items() if n == name)
    t = next(t for t in targets_of(group) if t.name == name)
    base = t._plan([])
    assert len(t.priors) >= 4
    for a in PLAN_ARRAYS:
        assert np.array_equal(base.array(a), t.plan.array(a)), a
    F0 = 1 + t.d.n_edges
    assert np.array_equal(base.array("fslot")[:F0], t.plan.array("fslot")[:F0])


def _reference_hessian(t, factors, lam):
    return pc.hessian_ref(t.d.n_nodes, t.plan.info()["n_slots"], factors, t.plan.array("fslot"), t.d.init, lam)


@pytest.mark.parametrize("group", [g for g in GROUPS if g not in SUBPROCESS or g == "leaf63"])
def test_emulation_fails_where_predicted(built, group):
    """The float64 elimination of every perturbed system meets its first non-positive or NaN pivot exactly at the
    predicted (supernode, column): the expectations of the GPU tests are right without a GPU."""
    for t in targets_of(group):
        Ad0, Ao0, B0 = _reference_hessian(t, t.factors, LAM)
        base = pc.reference_fronts(t.plan, Ad0, Ao0, B0)
        for case in t.cases:
            W, P = t.uploads(case, Ad0, t.d.init)
            lam = case.get("lam", LAM)
            lp = t.d.init.copy()
            for i, v in P.items():
                lp[i] = v
            Ad, Ao, B = pc.hessian_ref(t.d.n_nodes, t.plan.info()["n_slots"], t.perturbed(W, P),
                                       t.plan.array("fslot"), lp, lam)
            dirty = _dirty(t, W, P) if lam == LAM else None
            got = pc.first_failure(t.plan, Ad, Ao, B, base if dirty is not None else None, dirty)
            assert got is not None, t.describe(case)
            if case["at"] is None:
                assert got[0] in case["expect"], (t.describe(case), got)
            else:
                s, col = case["at"]
                assert got[0] == s and (col is None or got[1] == col), (t.describe(case), got)


def _dirty(t, W, P):
    _, fa, fb, _, _ = t.factors
    out = set()
    for f in W:
        out |= {int(fa[f])} | ({int(fb[f])} if fb[f] >= 0 else set())
    for i in P:
        out |= {int(i), *pc.neighbours(t.factors, i)}
    return out


def test_zero_pivots_are_exact(built):
    """With no Tikhonov term the isolated pose's pivots are exactly 0.0 (a00, d1, d2 as the kernels compute them)."""
    t = next(t for t in targets_of("leaf") if t.name == "pendants")
    Ad0, _, _ = _reference_hessian(t, t.factors, 0.0)
    assert np.all(Ad0[t.iso] == np.asarray(t.factors[4][t.prior_f[t.iso]]).reshape(3, 3))
    zeros = [c for c in t.cases if c["kind"] == "zero"]
    assert len(zeros) == 3
    for case in zeros:
        W, P = t.uploads(case, Ad0, t.d.init)
        Ad, _, _ = _reference_hessian(t, t.perturbed(W, P), 0.0)
        k = case["col"]
        assert pc.pivot_of(Ad, t.iso, k) == 0.0 and all(pc.pivot_of(Ad, t.iso, j) > 0 for j in range(k)), k


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
def _bounds(snap, factors):
    ft, fa, fb, _, _ = factors
    wf, wr, per = fc.check_fronts(snap)
    A, b = fc.system(snap, ft, fa, fb, snap.plan.array("fslot"))
    return dict(factor=wf, rhs=wr, y_bad=fc.check_y(snap), backsolve=fc.check_backsolve_local(snap),
                residual=fc.check_residual(A, b, snap.x), paths=fc.describe(per))


def _bounds_ok(r):
    return (r["factor"] < FACTOR_TOL and r["rhs"] < RHS_TOL and r["y_bad"] == 0 and r["backsolve"] < BACKSOLVE_TOL
            and r["residual"] < RESIDUAL_TOL)


def _run_case(t, ctx, case, base, baseH, use_x_status):
    Ad0 = baseH[0]
    W, P = t.uploads(case, Ad0, ctx.lp)
    lam = case.get("lam", LAM)
    for f, w in W.items():
        ctx.set_W(f, w)
        assert np.array_equal(ctx.device_W(f), np.asarray(w, float).reshape(9), equal_nan=True)
    for i, v in P.items():
        ctx.set_lp(i, v)
    ctx.relinearize(lam)
    Hp = ctx.hessian()
    rec = dict(what=t.describe(case), col=case["col"], kind=case["kind"], expected=sorted(1 + s for s in case["expect"]))
    # the perturbation is where it was meant to be: the diagonal entries of the seeds are the float64 expectation,
    # and the float64 elimination of the device Hessian fails at the predicted place
    for node, k in case.get("seeds", []):
        want = -max(1.0, abs(Ad0[node][k, k]))
        assert abs(Hp[0][node][k, k] - want) <= 1e-12 * abs(want), (rec["what"], Hp[0][node][k, k], want)
    dirty = _dirty(t, W, P) if lam == LAM else None
    got = pc.first_failure(ctx.plan, *Hp, base.fronts if dirty is not None else None, dirty)
    rec["emulated"] = None if got is None else [int(got[0]), int(got[1])]
    ctx.factor()
    if use_x_status:
        _, rec["status"] = ctx.x_status()
    else:
        rec["status"] = ctx.status()
    # recovery: the original system, factored twice
    for f in W:
        ctx.set_W(f, t.factors[4][f])
    for i in P:
        ctx.set_lp(i, ctx.lp[i])
    ctx.relinearize(LAM)
    runs = []
    for _ in range(2):
        ctx.factor()
        st = ctx.status()
        runs.append((st, ctx.snapshot()))
    Hr = ctx.hessian()
    rec["recovered_status"] = [runs[0][0], runs[1][0]]
    rec["repeatable"] = pc.same_bits(runs[0][1], runs[1][1])
    rec["hessian_as_baseline"] = pc.same_hessian(Hr, baseH)
    if rec["hessian_as_baseline"]:
        rec["as_baseline"] = pc.same_bits(runs[0][1], base)
    else:
        r = _bounds(runs[0][1], t.factors)
        rec["as_baseline"] = _bounds_ok(r)
        rec["bounds"] = {k: v for k, v in r.items() if k != "paths"}
    return rec


def _extreme_cases(t, ctx, base):
    """The isolated pose held by a diagonal prior alone, no Tikhonov term, pivots across the double range."""
    out = []
    f = t.prior_f[t.iso]
    q = int(ctx.node2q[t.iso])
    for piv, r in EXTREME:
        ctx.set_W(f, np.diag(piv).reshape(9), z=ctx.lp[t.iso] + np.array(r))
        ctx.relinearize(0.0)
        Ad, _, B = ctx.hessian()
        ctx.factor()
        x, st = ctx.x_status()
        F, rhs = ctx.fronts([t.s_iso])[t.s_iso]
        y = ctx.vec("y")
        rec = dict(what=f"leaf pendants isolated pose pivots {[float(p).hex() for p in piv]}", status=st, ulps=[])
        ok = st == 0
        for k in range(3):
            a = Ad[t.iso][k, k]
            ok &= a == piv[k]
            b = B[t.iso][k]
            root = np.sqrt(a)
            ulp = lambda v, ref: float(abs(v - ref) / np.spacing(abs(ref))) if ref != 0 else (0.0 if v == 0 else np.inf)  # noqa: E731
            u = [ulp(F[k, k], root), ulp(y[3 * q + k], b / root), ulp(x[3 * q + k], b / a)]
            rec["ulps"].append(u)
            power_of_four = np.frexp(a)[1] % 2 == 1 and np.frexp(a)[0] == 0.5
            ok &= (u[0] == 0.0) if power_of_four else (u[0] <= 2.0)
            ok &= np.isfinite(y[3 * q + k]) and np.isfinite(x[3 * q + k]) and u[1] <= 4.0 and u[2] <= 8.0
            ok &= b != 0.0 and x[3 * q + k] != 0.0  # a residual >= 1: the y and x checks are not 0 == 0
        rec["ok"] = bool(ok)
        out.append(rec)
    ctx.set_W(f, t.factors[4][f])
    ctx.relinearize(LAM)
    ctx.factor()
    snap = ctx.snapshot()
    out.append(dict(what="leaf pendants after the valid-range cases", status=ctx.status(),
                    ok=bool(pc.same_hessian(ctx.hessian(), (base.Adiag, base.Aoff, base.B)) and pc.same_bits(snap, base))
                    or _bounds_ok(_bounds(snap, t.factors))))
    return out


def run_group(group):
    """Every target of a group on the GPU: one record per case (and per valid-range case)."""
    env, _ = GROUPS[group]
    out = []
    with env_set(env):
        for t in targets_of(group):
            with H.Harness("b200") as h:
                h.load_full(t.d)
                for i, z, W in t.priors:
                    h.add_xytpos(i, z, W)
                h.batch()
                ctx = pc.Context(h, LAM)
                for a, b in zip(ctx.factors, t.factors):
                    assert np.array_equal(np.asarray(a), np.asarray(b)), t.name
                ctx.relinearize()
                ctx.factor()
                _, st = ctx.x_status()
                base = ctx.snapshot()
                assert st == 0 and base.path(t.s) == t.label, (t.name, st, base.path(t.s), t.label)
                assert not hasattr(t, "iso") or base.path(t.s_iso) == "leaf", base.path(t.s_iso)
                r = _bounds(base, t.factors)
                print(f"PIVOTCHECK baseline {group} {t.name} " + json.dumps({k: v for k, v in r.items() if k != "paths"}))
                assert _bounds_ok(r), (group, t.name, r)
                baseH = (base.Adiag, base.Aoff, base.B)
                for n, case in enumerate(t.cases):
                    out.append(_run_case(t, ctx, case, base, baseH, use_x_status=(n == 0)))
                if hasattr(t, "iso"):
                    out += _extreme_cases(t, ctx, base)
    return out


def _worker(group):
    """Runs in a subprocess with the group's switches in its environment; prints one JSON line."""
    runs = {"steps": run_steps, "scaled": run_scaled}
    print("RESULT " + json.dumps(runs[group]() if group in runs else run_group(group)))


def _run_worker(group):
    """A group in a subprocess (with its switches; the public API aborts the process on a failed solve)."""
    e = dict(os.environ)
    e.update(GROUPS[group][0] if group in GROUPS else {})
    here = os.path.dirname(os.path.abspath(__file__))
    code = f"import sys; sys.path[:0] = [{ROOT!r}, {here!r}]; import test_gpu_pivots as t; t._worker({group!r})"
    r = subprocess.run([sys.executable, "-c", code], env=e, capture_output=True, text=True, timeout=1200, cwd=ROOT)
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1]
    return json.loads(line[len("RESULT "):])


def assert_records(group, recs):
    bad = []
    for r in recs:
        print(f"PIVOTCHECK {group} " + json.dumps(r))
        if "ok" in r:
            if not (r["ok"] and r["status"] == 0):
                bad.append(r)
            continue
        fine = (r["status"] in r["expected"] and r["emulated"] is not None and 1 + r["emulated"][0] in r["expected"]
                and r["recovered_status"] == [0, 0] and r["repeatable"] and r["as_baseline"])
        if r["kind"] not in ("two_disjoint", "nan_lp") and r["col"] is not None and r["emulated"] is not None:
            fine &= r["emulated"][1] == r["col"]
        if not fine:
            bad.append(r)
    assert recs and not bad, "\n".join(f"{r['what']}: status {r.get('status')} " + json.dumps(r) for r in bad)


@pytest.fixture
def device(built):
    """Skips on a machine without a CUDA device (the solver has no CPU path and aborts there)."""
    from aprilsam_b200 import capi
    if capi.lib().asam_device_count() <= 0:
        pytest.skip("no CUDA device")


@pytest.mark.gpu
@pytest.mark.parametrize("group", list(GROUPS))
def test_failed_pivots(device, group):
    """Status exactly 1 + s for every placed failure; a clean context after each."""
    recs = _run_worker(group) if group in SUBPROCESS else run_group(group)
    assert_records(group, recs)


# ---------------------------------------------------------------------------------------------
# incremental steps: k_step (keep = 0 and keep > 0) and asam_step_run (team fronts re-factored)
# ---------------------------------------------------------------------------------------------
# (kind of task, column): the first column the task re-eliminates (3 * poses kept), or its last column
STEP_TARGETS = [("keep", "first"), ("keep", "last"), ("keep0", "first"), ("keep0", "last")]


def _step_target(rec, desc, want, team=False):
    """(task s, column) of a recorded step for a STEP_TARGETS entry (team: a task of a team of CTAs), or None."""
    kind, where = want
    for s, w, kp in zip(rec["tasks"], rec["nwait"], rec["keep"]):
        s, kp = int(s), int(kp)
        if (kp > 0) != (kind == "keep") or (team and ((int(w) >> 24) & 0x7F) <= 1):
            continue
        c = 3 * int(desc["cb"][s])
        j = 3 * (kp >> 16) if where == "first" else c - 1
        if j < c:
            return s, j
    return None


def _step_state(L, dev, desc, N, tasks):
    y, x = np.zeros(3 * N), np.zeros(3 * N)
    fc._ok(L, L.asam_download_y(dev, 0, N, y.ctypes.data_as(fc._dp)), "download_y")
    fc._ok(L, L.asam_download_x(dev, 0, N, x.ctypes.data_as(fc._dp)), "download_x")
    return fc.read_fronts(L, dev, desc, sorted(set(int(s) for s in tasks))), y, x


def _same(u, v):
    return np.array_equal(np.asarray(u).view(np.int64), np.asarray(v).view(np.int64))


def _step_case(h, L, rec, want, what, team=False):
    """Re-issue the step just taken: unperturbed (must reproduce it bit for bit), then with a negative pivot at the
    wanted column (status 1 + s), then recover with a batch solve on the same context (checked as in check_solve)."""
    from test_gpu_kernels import assert_solve_ok, check_solve
    dev = C.c_void_p(L.asam_dbg_dev_of_graph(h.graph_ptr()))
    plan = fc.borrowed_plan(L, h.param_ptr())
    desc, q2node, N = plan.descs(), plan.array("q2node"), h.n_nodes
    factors = fc.factors_of(h)
    assert factors[0][0] == 2 and factors[1][0] == 0, "factor 0 is the prior on pose 0"
    s, j = _step_target(rec, desc, want, team)
    node, k = pc.column(desc, q2node, s, j)
    point = h.states()[node]
    out = dict(what=f"{what} {want[0]} task s={s} m={3 * int(desc['mb'][s])} c={3 * int(desc['cb'][s])} col={j}",
               expected=[1 + s])
    fr0, y0, x0 = _step_state(L, dev, desc, N, rec["tasks"])
    small = rec["kind"] == "k_step"
    kern, st, xo = pc.reissue_step(L, dev, rec, desc, 0, node, np.zeros(9), point, small)
    pc.restore_factor(L, dev, factors, 0)
    fr1, y1, x1 = _step_state(L, dev, desc, N, rec["tasks"])
    listed = True
    if xo is not None:
        off = 0
        for b, bf in zip(rec["bt"], rec["bfirst"]):
            first, c = int(desc["first"][b]), 3 * int(desc["cb"][b])
            listed &= _same(xo[off + 3 * int(bf):off + c], x1[3 * first + 3 * int(bf):3 * first + c])
            off += c
    out.update(kernel=kern, reissue_status=st, listed_x=bool(listed),
               reissue_same=bool(_same(y0, y1) and _same(x0, x1) and
                                 all(_same(fr0[t][0], fr1[t][0]) and _same(fr0[t][1], fr1[t][1]) for t in fr0)))
    Ad = np.zeros((N, 3, 3))
    fc._ok(L, L.asam_debug_read_hessian(dev, N, 0, Ad.ctypes.data_as(fc._dp), None, None), "read_hessian")
    W = np.zeros((3, 3))
    W[k, k] = -max(1.0, abs(Ad[node][k, k])) - Ad[node][k, k]
    _, out["status"], _ = pc.reissue_step(L, dev, rec, desc, 0, node, W, point, small)
    pc.restore_factor(L, dev, factors, 0)
    h.batch()
    res = check_solve(h)
    try:
        assert_solve_ok(res, what + " recovery")
        out["recovered"] = True
    except AssertionError:
        out["recovered"] = False
    return out


def run_steps():
    """M3500 pose by pose (k_step, keep = 0 and keep > 0), then the appends under a team-merged root front of
    c = m = 195 / 198 (asam_step_run: team fronts are not single-CTA steps).  One case per chosen step."""
    from support import inccheck as ic
    from test_gpu_incremental import B_GRAPHS, _add_step, b_graph, b_steps
    pc.dev_api()
    L = ic.dev_api()
    out = []
    m = H.PoseGraphData.load(os.path.join(ROOT, "tests", "golden", "m3500.npz")).head(400)
    wants = list(STEP_TARGETS)
    with H.Harness("b200") as h, ic.recording(L):
        h.replay_begin(m)
        h.replay_to(2)
        for n in range(2, m.n_nodes):
            h.replay_to(n + 1)
            if not wants:
                break
            rec = ic.last_step(L, h.param_ptr())
            if rec["kind"] != "k_step":
                continue
            desc = fc.borrowed_plan(L, h.param_ptr()).descs()
            if _step_target(rec, desc, wants[0]) is None:
                continue
            out.append(_step_case(h, L, rec, wants.pop(0), f"m3500 step {n}"))
    assert not wants, wants

    class _Steps:  # _add_step's step hook: just run the incremental call
        def step(self, run, tag=None):
            run()

    for name, where in zip(B_GRAPHS, ("first", "last")):
        rng = np.random.default_rng(0)
        with H.Harness("b200") as h, ic.recording(L):
            h.load_full(b_graph(name))
            h.batch()
            spec = b_steps(1)[0](fc.borrowed_plan(L, h.param_ptr()), h.n_nodes)
            _add_step(h, _Steps(), spec, rng)
            rec = ic.last_step(L, h.param_ptr())
            G = [(int(w) >> 24) & 0x7F for w in rec["nwait"]]
            assert rec["kind"] == "pruned" and max(G) > 1, (rec["kind"], G)
            out.append(_step_case(h, L, rec, ("keep0", where), f"B {name}", team=True))
    return out


def assert_steps(recs):
    bad = []
    for r in recs:
        print("PIVOTCHECK steps " + json.dumps(r))
        fine = (r["reissue_status"] == 0 and r["reissue_same"] and r["listed_x"] and r["status"] in r["expected"]
                and r["recovered"] and r["kernel"] == ("k_step" if r["what"].startswith("m3500") else "step_run"))
        if not fine:
            bad.append(r)
    kernels = {r["kernel"] for r in recs}
    assert recs and not bad and kernels == {"k_step", "step_run"}, (kernels, bad)


def test_step_rows_reached(m3500, built):
    """The step targets are reached on host plans: the M3500 replay has k_step steps with keep > 0 tasks, the appends
    under the team root re-factor a team front with keep = 0."""
    from test_gpu_incremental import B_GRAPHS, a_steps_cpu, b_graph, b_steps, emulate_script
    a = a_steps_cpu(m3500, 400)
    assert a.kinds["k_step"] > 0 and a.items["k_step_keep"] > 0, a.summary()
    for name in B_GRAPHS:
        b = emulate_script(b_graph(name), b_steps(1))
        assert b.items["team_refactored"] > 0 and b.items["team_keep0"] > 0, (name, b.summary())


@pytest.mark.gpu
def test_failed_pivots_in_steps(device):
    """A recorded step re-issued unperturbed reproduces its fronts, y and x bit for bit; re-issued with a negative
    pivot at a column it re-eliminates (keep = 0 and keep > 0 tasks, k_step and asam_step_run) it reports exactly
    1 + s; a batch solve on the same context then passes check_solve."""
    assert_steps(_run_worker("steps"))


# ---------------------------------------------------------------------------------------------
# valid pivots out of the float range: every W x 2^k, no Tikhonov term
# ---------------------------------------------------------------------------------------------
SCALED = {"pendants": ({}, "leaf"), "smem_n51": ({}, "cta_smem"), "m555_c90": (SOLO_ENV, "cta_hbm"),
          "team162_c51": ({}, "team")}
MIN_RANGE = 800


def scaled_graph(name):
    """(graph, extra priors): the factorless last pose of the pendant graph gets a prior (no Tikhonov term)."""
    d = graph(name)
    if name != "pendants":
        return d, []
    iso = d.n_nodes - 1
    return d, [(iso, d.init[iso] + np.array([0.5, -0.25, 0.125]), np.diag([100.0, 100.0, 10.0]).reshape(9))]


def scale_range(name, exact=False):
    """Widest even k such that the float64 reference of the system scaled by 2^+-k keeps every non-zero entry of the
    Hessian (and of the sums of its contributions), W, L, y and the update matrices normal and finite.  L and y scale
    by 2^(k/2), the rest by 2^k."""
    env, _ = SCALED[name]
    d, pri = scaled_graph(name)
    fl = factor_list(d, pri)
    with env_set(env):
        p = HostPlan().build(d.n_nodes, *fl[:3])
    S = p.info()["n_slots"]
    Ad, AdA, B, BA, (_, _, Hh, HA) = fc.linearize_ref(d.n_nodes, *fl, d.init, None, 0.0)
    e = np.nonzero(fl[0] == 1)[0]
    Ao = np.zeros((S, 3, 3))
    np.add.at(Ao, p.array("fslot")[e], Hh)
    fr = pc.reference_fronts(p, Ad, Ao, B)
    cb = p.descs()["cb"]
    half = np.concatenate([np.r_[np.tril(F[:, :3 * cb[s]]).ravel(), b[:3 * cb[s]]] for s, (F, b) in fr.items()])
    full = np.concatenate([np.r_[np.tril(F[3 * cb[s]:, 3 * cb[s]:]).ravel(), b[3 * cb[s]:]] for s, (F, b) in fr.items()]
                          + [v.ravel() for v in (Ad, AdA, Ao, B, BA, HA, fl[4])])
    lg = lambda v: np.log2(np.abs(v[v != 0]))  # noqa: E731
    lh, lf = lg(half), lg(full)
    assert np.isfinite(lh).all() and np.isfinite(lf).all()
    up = min(1024 - lf.max(), 2 * (1024 - lh.max()))
    down = min(1022 + lf.min(), 2 * (1022 + lh.min()))
    if exact:  # products of two L / y entries stay normal too: the device's rounding scales exactly
        down = min(down, 1022 + 2 * lh.min())
    return int(np.floor(min(up, down) - 1e-9)) // 2 * 2


def scaled_solve(name, k):
    """Batch solve with every W scaled by 2^k, no Tikhonov term: (states, check_solve result)."""
    from test_gpu_kernels import check_solve
    env, _ = SCALED[name]
    d, pri = scaled_graph(name)
    s = 2.0 ** k
    with env_set(env), H.Harness("b200") as h:
        h.set_tikhanov(0.0)
        h.load_full(H.PoseGraphData(d.init, d.ea, d.eb, d.ez, d.eW * s))
        _, _, _, z, W = h.factor(0)
        h.set_factor(0, z, W * s)
        for i, z, W in pri:
            h.add_xytpos(i, z, W * s)
        h.batch()
        return h.states(), check_solve(h, lam=0.0, forward=False)


def run_scaled():
    out = {}
    for name in SCALED:
        K, Kx = scale_range(name), scale_range(name, exact=True)
        st0, _ = scaled_solve(name, 0)
        # two unscaled solves differ by the order of k_linearize's atomic sums, amplified by the condition number
        d0 = scaled_solve(name, 0)[0] - st0
        d0[:, 2] = emul.mod2pi(d0[:, 2])
        spread = float(np.abs(d0).max() / max(1.0, np.abs(st0).max()))
        recs = []
        for k in sorted({-K, -Kx, -(K // 4) * 2, (K // 4) * 2, Kx, K}):
            st, res = scaled_solve(name, k)
            dd = st - st0
            dd[:, 2] = emul.mod2pi(dd[:, 2])
            res["k"] = k
            res["state_err"] = float(np.abs(dd).max() / max(1.0, np.abs(st0).max()))
            res["finite"] = bool(np.isfinite(st).all())
            recs.append(res)
        out[name] = dict(K=K, K_exact=Kx, spread=spread, runs=recs)
    return out


@pytest.mark.parametrize("name", list(SCALED))
def test_scaled_sweep_reaches_its_paths(built, name):
    """The scaled graphs reach their paths and the float64 reference stays normal over |k| >= 800."""
    env, path = SCALED[name]
    d, pri = scaled_graph(name)
    fl = factor_list(d, pri)
    with env_set(env):
        paths = {f[0] for f in path_table(HostPlan().build(d.n_nodes, *fl[:3])).values()}
    assert any(p == path or (path == "team" and p.startswith("team")) for p in paths), paths
    assert scale_range(name) >= MIN_RANGE, scale_range(name)


def test_reference_follows_the_scaled_sweep(m3500):
    """The reference (sqrt in double) follows the widest scaling of the sweep: same solution within 1e-12, chi2
    scaled by 2^k (test_gpu_kernels.test_reference_is_scale_invariant goes to |k| = 180)."""
    if not H.available("reference"):
        pytest.skip("reference oracle not built")
    from test_gpu_kernels import scaled_run
    K = scale_range("team162_c51")
    for d in (m3500.head(200), zoo("team162_c51")):
        st0, c0 = scaled_run("reference", d, 0)
        for k in (-K, K):
            st, c = scaled_run("reference", d, k)
            dd = st - st0
            dd[:, 2] = emul.mod2pi(dd[:, 2])
            assert np.abs(dd).max() / max(1.0, np.abs(st0).max()) < 1e-12, k
            assert abs(c / 2.0 ** k - c0) <= 1e-12 * c0, (k, c, c0)


@pytest.mark.gpu
def test_scaled_sweep(device):
    """Every W x 2^k at the widest even |k| the float64 reference allows (and half of it), no Tikhonov term, on
    graphs reaching leaf, cta_smem, cta_hbm and team: status 0 (the public API aborts otherwise), every check of
    check_solve (scale-free bounds, y bit for bit, back-substitution, determinism) and states within 1e-12 of k = 0
    (or within 10x the spread of two unscaled solves, where the condition number makes that larger).  The sweep also
    runs at K_exact, the widest |k| at which products of two L entries stay normal as well."""
    from test_gpu_kernels import assert_solve_ok
    out = _run_worker("scaled")
    for name, o in out.items():
        _, path = SCALED[name]
        assert o["K"] >= MIN_RANGE, (name, o["K"])
        for r in o["runs"]:
            print(f"PIVOTCHECK scaled {name} K={o['K']} " + json.dumps({k: v for k, v in r.items() if k != "paths"}))
            assert any(p == path or (path == "team" and p.startswith("team")) for p in r["per_path"]), r["paths"]
            # 1e-12, or 10x the spread of two unscaled solves where that is larger (the pendant graph, kappa ~ 1e9)
            tol = max(1e-12, 10 * o["spread"])
            assert r["finite"] and r["state_err"] < tol, (name, r["k"], r["state_err"], o["spread"])
            assert_solve_ok(r, f"{name} k={r['k']}")
