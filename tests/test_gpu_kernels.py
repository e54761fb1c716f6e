"""Kernel-level tests: every front of a solve checked against float64 / long-double references of the same
operation (tests/support/frontcheck.py), on graphs whose fronts sit on the branch edges of the kernels.

The parity tests compare node states after whole Gauss-Newton calls at 1e-6; a kernel that is slightly wrong
in one front can pass them.  These tests bound the LOCAL backward error of every front (independent of
cond(A), so the bound can be tight), require y to be the fronts' rhs rows bit for bit, check the
back-substitution per supernode and globally, the forward error against kappa_1 * u, the Hessian of
k_linearize entry by entry, and that the factorisation is deterministic.  CPU tests (not marked gpu) show that the checker catches wrong fronts
and that the graphs really reach every kernel path they are meant to reach.

Bounds: about 10x the worst value observed on an H100 with the kernels of this tree (constants below).
"""
from __future__ import annotations

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
from support.hostplan import HostPlan

# observed worst on an H100 (zoo, team sizes 1-28, leaf kernels, manhattan_dense 2000 / 30000, M3500 replay):
FACTOR_TOL = 1e-14      # local backward error of a front, relative to |F| + |L||L|'   (observed 1.5e-15)
RHS_TOL = 2e-14         # rhs rows of a front, componentwise                          (observed 2.1e-15)
BACKSOLVE_TOL = 1e-14   # L11' x1 = y1 - L21' x2, componentwise                       (observed 1.1e-15)
RESIDUAL_TOL = 1e-15    # |Ax - b| / (|A||x| + |b|)                                    (observed 7.2e-17)
FORWARD_C = 0.1         # |x - x_ref| / |x_ref| <= FORWARD_C * kappa_1 * u            (observed 0.008)
LINEARIZE_C = 200.0     # |H_dev - H_ref| <= LINEARIZE_C * u * sum |contributions|    (observed 18.5)
CHI2_TOL = 1e-13        # asam_chi2 against a long-double sum over factors, relative  (observed 1.9e-15)

PRIOR_W = np.array([1e4, 0, 0, 0, 1e4, 0, 0, 0, 1e3])


# ---------------------------------------------------------------------------------------------
# the front zoo
# ---------------------------------------------------------------------------------------------
def _meas(rng, truth, a, b, sigma=0.01):
    c, s = np.cos(truth[a, 2]), np.sin(truth[a, 2])
    d = truth[b] - truth[a]
    z = np.c_[c * d[:, 0] + s * d[:, 1], -s * d[:, 0] + c * d[:, 1], emul.mod2pi(d[:, 2])]
    return z + sigma * rng.standard_normal(z.shape)


def _full_W(rng, n):
    M = rng.standard_normal((n, 3, 3))
    return (30.0 * (M @ np.transpose(M, (0, 2, 1)) + 0.5 * np.eye(3))).reshape(n, 9)


def _graph(rng, truth, pairs, init_noise=0.02):
    """PoseGraphData from (a, b) pairs: full SPD W, a third of the edges reversed, the odometry chain
    duplicated where it is also a clique edge."""
    pairs = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    flip = rng.random(len(pairs)) < 0.33
    ea = np.where(flip, pairs[:, 1], pairs[:, 0]).astype(np.int32)
    eb = np.where(flip, pairs[:, 0], pairs[:, 1]).astype(np.int32)
    ez = _meas(rng, truth, ea, eb)
    eW = _full_W(rng, len(ea))
    order = np.lexsort((np.minimum(ea, eb), np.maximum(ea, eb)))
    init = truth + init_noise * rng.standard_normal(truth.shape)
    init[:, 2] = emul.mod2pi(init[:, 2])
    return H.PoseGraphData(init, ea[order], eb[order], ez[order], eW[order], truth.copy())


def _truth(rng, n):
    """Poses of a wandering walk from the origin (where the prior puts pose 0: a replay starting elsewhere would
    have to rotate the whole graph in one step and diverges); headings spread over the whole circle, several within
    1e-3 of +-pi (d_mod2pi wraps there)."""
    th = rng.uniform(-np.pi, np.pi, n)
    near = rng.choice(n, size=max(1, n // 8), replace=False)
    th[near] = np.where(rng.random(len(near)) < 0.5, np.pi, -np.pi) - np.sign(rng.standard_normal(len(near))) * 1e-3 * rng.random(len(near))
    th = emul.mod2pi(th)
    th[0] = 0.0
    xy = np.cumsum(rng.standard_normal((n, 2)), axis=0)
    return np.c_[xy - xy[0], th]


def _clique(ids):
    ids = np.asarray(ids)
    i, j = np.triu_indices(len(ids), 1)
    return np.c_[ids[i], ids[j]]


def _join(A, B):
    A, B = np.asarray(A), np.asarray(B)
    return np.c_[np.repeat(A, len(B)), np.tile(B, len(A))]


def zoo_graph(a, r, b, seed=0):
    """Cliques S1 (a poses) and S2 (b poses), both fully joined to the separator clique T (r poses), plus the
    odometry chain over all poses and the prior on pose 0: one front with c = 3a, m = 3(a + r) and the root
    front with c = m = 3(b + r)."""
    rng = np.random.default_rng(seed)
    n = a + r + b
    S1, T, S2 = np.arange(a), np.arange(a, a + r), np.arange(a + r, n)
    pairs = [_clique(S1), _clique(T), _clique(S2), _join(S1, T), _join(S2, T), np.c_[np.arange(n - 1), np.arange(1, n)]]
    return _graph(rng, _truth(rng, n), np.vstack(pairs))


def pendant_graph(sizes, per_spine=30, seed=0):
    """A spine (odometry chain) with a pendant clique of k poses, fully joined to one spine pose, for every k in
    `sizes`: thousands of small supernodes (c = 3k, m = 3(k + 1)), the workload of the warp-per-front kernels.  The
    last pose has no factor at all (held by the Tikhonov term alone): a root front of c = m = 3."""
    rng = np.random.default_rng(seed)
    nsp = (len(sizes) + per_spine - 1) // per_spine
    pairs = [np.c_[np.arange(nsp - 1), np.arange(1, nsp)]]
    nxt = nsp
    for i, k in enumerate(sizes):
        ids = np.arange(nxt, nxt + k)
        nxt += k
        pairs += [_clique(ids), _join(ids, [i // per_spine])]
    return _graph(rng, _truth(rng, nxt + 1), np.vstack([p for p in pairs if len(p)]))


# (a, r, b) per zoo graph and what it is for (m = 3(a+r) for the first front, 3(b+r) for the root)
ZOO = {
    # shared-memory cta_front: m = 159 (the largest that fits), c mod 12 in {0, 3, 9}; trailing n = 48 / 51
    "smem159_c12": (4, 49, 10),
    "smem159_c3": (1, 52, 2),
    "smem159_c9": (3, 50, 3),
    "smem_n48": (20, 16, 30),
    "smem_n51": (25, 17, 2),
    # team fronts, m = 162 (the first that does not fit), c in {3, 45, 48, 51, 93, 96, 99}
    "team162_c3": (1, 53, 2),
    "team162_c45": (15, 39, 2),
    "team162_c48": (16, 38, 2),
    "team162_c51": (17, 37, 2),
    "team162_c93": (31, 23, 2),
    "team162_c96": (32, 22, 2),
    "team162_c99": (33, 21, 2),
    # crew row chunks around 128 rows below the next panel: m - 48 + 1 in {127, 130}
    "team_chunk127": (20, 38, 2),
    "team_chunk130": (20, 39, 2),
    # back-solve blocks: root c = m > 96 with c mod 96 in {0, 3, 93}
    "bs_192": (4, 20, 44),
    "bs_195": (4, 20, 45),
    "bs_189": (4, 20, 43),
    # wide: several 256-row and 64-column tiles
    "wide": (120, 120, 120),
}


def zoo(name):
    return zoo_graph(*ZOO[name], seed=len(name))


def plan_of(d, env=None):
    """HostPlan of a graph (prior on pose 0 first, like the harness's load_full)."""
    ftype = np.r_[2, np.ones(d.n_edges, dtype=np.int32)].astype(np.int32)
    fa = np.r_[0, d.ea].astype(np.int32)
    fb = np.r_[-1, d.eb].astype(np.int32)
    old = {k: os.environ.get(k) for k in (env or {})}
    try:
        os.environ.update(env or {})
        return HostPlan().build(d.n_nodes, ftype, fa, fb)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def pendant_sizes(leaf63=False):
    """4200 pendants: fronts of m = 6, 45 and 48 (and 63 for the wider leaf limit)."""
    return [1, 14, 15, 20] * 1050 if leaf63 else [1, 14, 15] * 1400


def path_table(p):
    """{supernode: (path, m, c, children)} of a host plan, as frontcheck.Snapshot.path names the paths."""
    d = p.descs()
    leaf = set(int(s) for s in p.array("leaf_tasks"))
    G = {}
    for s, w in zip(p.array("tasks"), p.array("nwait")):
        G.setdefault(int(s), (int(w) >> 24) & 0x7f)
    out = {}
    for s in range(len(d["mb"])):
        m, c = 3 * int(d["mb"][s]), 3 * int(d["cb"][s])
        g = G.get(s, 0)
        path = "leaf" if s in leaf else (f"team{g}" if g else ("cta_smem" if fc.fits_smem(m // 3) else "cta_hbm"))
        out[s] = (path, m, c, int(d["ch_cnt"][s]))
    return out


TEAM_ENV = {g: {"ASAM_TEAM_ROOM": "1", "ASAM_TEAM_MIN": str(g)} for g in (1, 2, 3, 5)}


# ---------------------------------------------------------------------------------------------
# CPU: the zoo reaches every branch edge; the checker catches wrong fronts
# ---------------------------------------------------------------------------------------------
def test_zoo_covers_the_kernel_branch_edges(built):
    """Every row of the coverage table is present in the host plans of the zoo, so the GPU tests below can
    never become vacuous."""
    fronts = []
    for name in ZOO:
        fronts += list(path_table(plan_of(zoo(name))).values())
    smem = [f for f in fronts if f[0] == "cta_smem"]
    team = [f for f in fronts if f[0].startswith("team")]
    assert any(m == 159 for _, m, _, _ in smem)
    assert {c % 12 for _, m, c, _ in smem if m == 159 and c < m} >= {0, 3, 9}
    assert {m - c for _, m, c, _ in smem} >= {48, 51}
    assert any(m == c for _, m, c, _ in smem)
    assert any(0 < ch <= 24 for _, _, _, ch in smem)
    assert any(m == 162 for _, m, _, _ in team)
    assert not fc.fits_smem(54) and fc.fits_smem(53)
    assert {c for _, m, c, _ in team if m == 162} >= {3, 45, 48, 51, 93, 96, 99}
    assert any(m == c for _, m, c, _ in team)
    assert {m - 48 + 1 for _, m, c, _ in team if c > 48} >= {127, 130}
    assert any(m >= 700 for _, m, _, _ in team)
    assert {c % 96 for _, m, c, _ in team + smem if c > 96} >= {0, 3, 93}
    # team sizes: one CTA on the team path (G field 1), 2, 3, 5, and the full team_size()
    for g, env in TEAM_ENV.items():
        gs = {f[0] for f in path_table(plan_of(zoo("team162_c51"), env)).values() if f[0].startswith("team")}
        assert gs == {f"team{g}"}, (g, gs)
    assert any(int(f[0][4:]) >= 20 for f in team)
    # warp-per-front kernels: >= 4096 leaf supernodes, m = 6, 45, 48 (63 with ASAM_LEAF_MAX_M=63)
    p = plan_of(pendant_graph(pendant_sizes()))
    t = path_table(p)
    assert len(p.array("leaf_tasks")) >= 4096
    assert p.info()["n_bs_leaf"] >= 4096  # k_backsolve_leaf
    assert 3 in {m for path, m, _, _ in t.values() if path == "leaf"}  # the isolated pose
    assert {m for path, m, _, _ in t.values() if path == "leaf"} >= {6, 45, 48}
    assert max(ch for path, _, _, ch in t.values() if path == "cta_smem") > 24
    p63 = plan_of(pendant_graph(pendant_sizes(True)), {"ASAM_LEAF_MAX_M": "63"})
    assert 63 in {m for path, m, _, _ in path_table(p63).values() if path == "leaf"}


def _emulated_snapshot(d):
    p = plan_of(d)
    info = p.info()
    ftype = np.r_[2, np.ones(d.n_edges, dtype=np.int32)].astype(np.int32)
    fa = np.r_[0, d.ea].astype(np.int32); fb = np.r_[-1, d.eb].astype(np.int32)
    fz = np.vstack([[0, 0, 0], d.ez]); fW = np.vstack([PRIOR_W, d.eW])
    Hs = emul.Hessian(d.n_nodes, info["n_slots"]); Hs.reset(d.n_nodes, 1e-4)
    Hs.linearize(range(len(ftype)), ftype, fa, fb, fz, fW, d.init, d.init, p.array("node2q"), p.array("fslot"))
    fr = emul.Fronts(); fr.ensure(d.n_nodes)
    emul.factor(fr, Hs, p.descs(), p.array("ipool"), p.array("q2node"), p.array("tasks"), p.array("nwait"))
    emul.backsolve(fr, p.descs(), p.array("ipool"), p.array("btasks"))
    return fc.snapshot_from_emulation(p, Hs, fr), (ftype, fa, fb, fz, fW)


def _mutant(snap, s, F, rhs, y=None):
    import copy
    m = copy.copy(snap)
    m.fronts = dict(snap.fronts)
    m.fronts[s] = (F, rhs)
    if y is not None:
        m.y = y
    return m


def test_checker_catches_wrong_fronts(built):
    """The checker on fronts of the numpy emulation: they pass; a stale 12-column stage, a dropped trailing
    update of the last partial panel on one 64-row tile, and one y entry off by 1e-10 relative each fail."""
    d = zoo("team162_c51")
    snap, (ftype, fa, fb, fz, fW) = _emulated_snapshot(d)
    wf, wr, per = fc.check_fronts(snap)
    assert wf < FACTOR_TOL and wr < RHS_TOL, fc.describe(per)
    assert fc.check_y(snap) == 0
    assert fc.check_backsolve_local(snap) < BACKSOLVE_TOL
    A, b = fc.system(snap, ftype, fa, fb, snap.plan.array("fslot"))
    assert fc.check_residual(A, b, snap.x) < RESIDUAL_TOL
    xr, kappa = fc.reference_solution(A, b)
    assert fc.forward_error(snap.x, xr) <= FORWARD_C * kappa * fc.U
    s = max(range(snap.nsn), key=lambda t: (3 * int(snap.desc["cb"][t]) % 48 != 0, int(snap.desc["cb"][t])))
    F, rhs = snap.fronts[s]
    m, c = F.shape[0], 3 * int(snap.desc["cb"][s])
    assert c == 51 and m == 162
    # 1. columns [12, 24) of L factored from the trailing matrix as it was one 12-column stage earlier: the update of
    #    stage [0, 12) never reached them (a reader that took the stage flag before the data)
    F0, _ = fc.assemble(snap, s)
    Fp = F0.copy()
    for k in range(24):
        Fp[k, k] = np.sqrt(Fp[k, k])
        Fp[k + 1:, k] /= Fp[k, k]
        cols = np.arange(k + 1, m) if k >= 12 else np.r_[np.arange(k + 1, 12), np.arange(24, m)]
        Fp[np.ix_(np.arange(k + 1, m), cols)] -= np.outer(Fp[k + 1:, k], Fp[cols, k])
    Fs = F.copy()
    Fs[12:, 12:24] = np.tril(Fp[12:, 12:24])
    Fs[12:24, 12:24] += np.triu(F[12:24, 12:24], 1)
    wf1, _, _ = fc.check_fronts(_mutant(snap, s, Fs, rhs))
    # 2. last partial panel [48, 51): trailing update dropped for rows [c, c + 64)
    Fd = F.copy()
    Lp = F[:, 48:51]
    rows = np.arange(c, min(m, c + 64))
    Fd[np.ix_(rows, np.arange(c, m))] += np.tril(Lp[rows] @ Lp[c:].T, c)[:, :]
    Fd = np.where(np.tril(np.ones_like(Fd, dtype=bool)), Fd, F)
    wf2, _, _ = fc.check_fronts(_mutant(snap, s, Fd, rhs))
    # 3. one entry of y1 off by 1e-10 relative (front and y alike)
    r3 = rhs.copy(); y3 = snap.y.copy()
    k = int(np.argmax(np.abs(rhs[:c])))
    r3[k] *= 1 + 1e-10
    y3[3 * int(snap.desc["first"][s]) + k] = r3[k]
    _, wr3, _ = fc.check_fronts(_mutant(snap, s, F, r3, y3))
    assert wf1 > 100 * FACTOR_TOL and wf2 > 100 * FACTOR_TOL and wr3 > 10 * RHS_TOL, (wf1, wf2, wr3)


# ---------------------------------------------------------------------------------------------
# GPU: every front of a batch solve
# ---------------------------------------------------------------------------------------------
def check_solve(h, lam=1e-4, forward=True, determinism=True):
    """All checks of frontcheck on the solve a Harness just ran; returns the worst values (and the per-path
    report) as a dict.  With `determinism`, asam_factor_full + asam_backsolve_full run once more on the same
    Hessian: status 0, fronts and x bit-identical."""
    L = fc.dev_api()
    snap = fc.snapshot(h, L)
    ftype, fa, fb, fz, fW = fc.factors_of(h)
    fslot = snap.plan.array("fslot")
    wf, wr, per = fc.check_fronts(snap)
    A, b = fc.system(snap, ftype, fa, fb, fslot)
    res = {"factor": wf, "rhs": wr, "paths": fc.describe(per),
           "per_path": {p: [v["factor"][0], v["rhs"][0]] for p, v in per.items()},
           "y_bad": fc.check_y(snap), "backsolve": fc.check_backsolve_local(snap),
           "residual": fc.check_residual(A, b, snap.x),
           "linearize": fc.check_linearize(snap, ftype, fa, fb, fz, fW, h.l_points(), fslot, lam)}
    if forward:
        xr, kappa = fc.reference_solution(A, b)
        res["forward_over_kappa_u"] = fc.forward_error(snap.x, xr) / (kappa * fc.U)
    if determinism:
        dev = L.asam_dbg_dev_of_graph(h.graph_ptr())
        fc._ok(L, L.asam_factor_full(dev), "factor_full")
        fc._ok(L, L.asam_backsolve_full(dev), "backsolve_full")
        x2 = np.zeros_like(snap.x)
        fc._ok(L, L.asam_download_x(dev, 0, len(x2) // 3, x2.ctypes.data_as(fc._dp)), "download_x")
        import ctypes as C
        st = C.c_int()
        fc._ok(L, L.asam_factor_status(dev, C.byref(st)), "factor_status")
        again = fc.read_fronts(L, dev, snap.desc)
        same = all(np.array_equal(again[s][0].view(np.int64), snap.fronts[s][0].view(np.int64)) and
                   np.array_equal(again[s][1].view(np.int64), snap.fronts[s][1].view(np.int64)) for s in again)
        res["deterministic"] = bool(same and np.array_equal(x2.view(np.int64), snap.x.view(np.int64)) and st.value == 0)
    return res


def assert_solve_ok(res, what):
    msg = f"{what}:\n{res['paths']}\n{ {k: v for k, v in res.items() if k not in ('paths', 'per_path')} }"
    print(f"KERNELCHECK {what} " + json.dumps({k: v for k, v in res.items() if k != "paths"}))
    assert res["factor"] < FACTOR_TOL and res["rhs"] < RHS_TOL, msg
    assert res["y_bad"] == 0, msg
    assert res["backsolve"] < BACKSOLVE_TOL and res["residual"] < RESIDUAL_TOL, msg
    assert res["linearize"] < LINEARIZE_C, msg
    assert res.get("forward_over_kappa_u", 0.0) <= FORWARD_C, msg
    assert res.get("deterministic", True), msg


class env_set:
    """Environment variables the host plan reads on every build (team sizes, leaf limit)."""

    def __init__(self, env):
        self.env = env

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.env}
        os.environ.update(self.env)

    def __exit__(self, *exc):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def add_priors(h, d, seed=3):
    """Two priors with full W besides the one load_full puts on pose 0 (the last one on the pose 0 as well)."""
    rng = np.random.default_rng(seed)
    for i in (d.n_nodes // 2, 0):
        h.add_xytpos(i, d.truth[i] + 0.01 * rng.standard_normal(3) if d.truth is not None else d.init[i], _full_W(rng, 1)[0])


def batch_and_check(d, env=None, priors=True, **kw):
    with env_set(env or {}), H.Harness("b200") as h:
        h.load_full(d)
        if priors:
            add_priors(h, d)
        h.batch()
        return check_solve(h, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ZOO))
def test_zoo_fronts(name):
    assert_solve_ok(batch_and_check(zoo(name)), name)


@pytest.mark.gpu
@pytest.mark.parametrize("g", sorted(TEAM_ENV))
def test_team_sizes(g):
    for name in ("team162_c51", "wide"):
        res = batch_and_check(zoo(name), TEAM_ENV[g])
        assert f"team{g}" in res["per_path"], res["paths"]
        assert_solve_ok(res, f"{name} G={g}")


@pytest.mark.gpu
@pytest.mark.parametrize("leaf63", [False, True])
def test_leaf_kernels(leaf63):
    env = {"ASAM_LEAF_MAX_M": "63"} if leaf63 else {}
    res = batch_and_check(pendant_graph(pendant_sizes(leaf63)), env, forward=False)
    assert "leaf" in res["per_path"], res["paths"]
    assert_solve_ok(res, f"pendants leaf63={leaf63}")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2000, 30000])
def test_manhattan_fronts(n):
    from aprilsam_b200 import datasets
    assert_solve_ok(batch_and_check(datasets.manhattan_dense(n, seed=1), forward=(n <= 2000)), f"manhattan_dense({n})")


@pytest.mark.gpu
def test_chi2_long_double_and_deterministic():
    """asam_chi2 (the deterministic two-level reduction behind april_graph_chi2) against a long-double sum over
    the factors, and bit-identical on a second call."""
    d = zoo("team162_c51")
    with H.Harness("b200") as h:
        h.load_full(d)
        add_priors(h, d)
        h.batch()
        c1, c2 = h.chi2(), h.chi2()
        ref = fc.chi2_ref(*fc.factors_of(h), h.states())
    print(f"KERNELCHECK chi2 {c1!r} {float(ref)!r} rel {float(abs(np.longdouble(c1) - ref) / ref):.2e}")
    assert c1 == c2
    assert abs(np.longdouble(c1) - ref) <= CHI2_TOL * ref, (c1, float(ref))


# ---------------------------------------------------------------------------------------------
# GPU: incremental steps (partial re-factorisation, k_step)
# ---------------------------------------------------------------------------------------------
def replay_checked(d, nsteps, check_every=1):
    """Pose-by-pose replay; after every step the per-front check on all fronts (the step only ADDS the new
    factors' contributions to the Hessian in HBM, so the invariant holds at every step).  At the last step, the
    states the step changed must equal l_point + x of one full back-substitution."""
    worst_f = worst_r = 0.0
    L = fc.dev_api()
    with H.Harness("b200") as h:
        h.replay_begin(d)
        h.replay_to(2)
        for k in range(2, nsteps):
            before = h.states()
            h.replay_to(k + 1)
            if (k % check_every) == 0 or k == nsteps - 1:
                snap = fc.snapshot(h, L)
                wf, wr, per = fc.check_fronts(snap)
                assert wf < FACTOR_TOL and wr < RHS_TOL, (k, fc.describe(per))
                worst_f, worst_r = max(worst_f, wf), max(worst_r, wr)
        after = h.states()
        n = len(after)
        changed = np.nonzero(np.any(after != np.vstack([before, np.zeros((n - len(before), 3))]), axis=1))[0]
        dev = L.asam_dbg_dev_of_graph(h.graph_ptr())
        fc._ok(L, L.asam_backsolve_full(dev), "backsolve_full")
        x = np.zeros(3 * n)
        fc._ok(L, L.asam_download_x(dev, 0, n, x.ctypes.data_as(fc._dp)), "download_x")
        n2q = fc.borrowed_plan(L, h.param_ptr()).array("node2q")
        want = h.l_points()[changed] + x.reshape(-1, 3)[n2q[changed]]
        diff = after[changed] - want
        diff[:, 2] = emul.mod2pi(diff[:, 2])
        return after, worst_f, worst_r, len(changed), float(np.abs(diff).max(initial=0.0) / max(1.0, np.abs(want).max()))


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["m3500_400", "zoo"])
def test_incremental_fronts_and_pruned_backsolve(m3500, which):
    d = m3500.head(400) if which == "m3500_400" else zoo("team162_c51")
    _, wf, wr, nchanged, err = replay_checked(d, d.n_nodes)
    print(f"KERNELCHECK replay {which} " + json.dumps({"factor": wf, "rhs": wr, "changed": nchanged, "x_err": err}))
    assert nchanged > 0 and err < 1e-12, (nchanged, err)


# ---------------------------------------------------------------------------------------------
# GPU: pivots outside the float range
# ---------------------------------------------------------------------------------------------
def scaled_run(impl, d, k, chi2_ref=False):
    """Batch solve with every W (the prior's too) scaled by 2^k and no Tikhonov term: (states, chi2), and with
    chi2_ref also april_graph_chi2 in long double at the same states (frontcheck.chi2_ref)."""
    s = 2.0 ** k
    with H.Harness(impl) as h:
        h.set_tikhanov(0.0)
        h.load_full(H.PoseGraphData(d.init, d.ea, d.eb, d.ez, d.eW * s))
        _, _, _, z, W = h.factor(0)
        h.set_factor(0, z, W * s)
        h.batch()
        if chi2_ref:
            return h.states(), h.chi2(), fc.chi2_ref(*fc.factors_of(h), h.states())
        return h.states(), h.chi2()


def test_reference_is_scale_invariant(m3500):
    """The reference takes sqrt in double: scaling every W by 2^k (k even, |k| <= 180) leaves its solution
    unchanged and scales chi2 by 2^k, up to rounding, so the GPU test below may compare each scale with k = 0."""
    if not H.available("reference"):
        pytest.skip("reference oracle not built")
    for d in (m3500.head(200), zoo("team162_c51")):
        st0, c0 = scaled_run("reference", d, 0)
        for k in (-180, -140, 140, 180):
            st, c = scaled_run("reference", d, k)
            dd = st - st0
            dd[:, 2] = emul.mod2pi(dd[:, 2])
            assert np.abs(dd).max() / max(1.0, np.abs(st0).max()) < 1e-12, k
            assert abs(c / 2.0 ** k - c0) <= 1e-12 * c0, k


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["zoo", "m3500_200"])
def test_pivots_outside_float_range(m3500, which):
    """Every W (the prior's too) scaled by 2^k, no Tikhonov term: A and b scale by 2^k exactly and the solution
    does not change.  Pivots then leave the float range, where a single-precision seed of 1/sqrt is 0 or inf.

    Two solves of one system are not bit-identical (the order of k_linearize's atomic sums varies from run to run,
    DESIGN.md §7), and chi2 after one Gauss-Newton step moves with the last bits of the states (6e-11 relative on
    M3500 (200 poses) on an H100).  So each run's chi2 is checked at 1e-13 against the long-double chi2 at its own
    states and its own scaled W, and against k = 0 only through the states."""
    d = m3500.head(200) if which == "m3500_200" else zoo("team162_c51")
    st0, c0, r0 = scaled_run("b200", d, 0, chi2_ref=True)
    assert abs(np.longdouble(c0) - r0) <= 1e-13 * r0, (c0, float(r0))
    for k in (-180, -140, -120, 120, 140, 180):
        st, c, r = scaled_run("b200", d, k, chi2_ref=True)
        d_ = st - st0
        d_[:, 2] = emul.mod2pi(d_[:, 2])
        err = float(np.abs(d_).max() / max(1.0, np.abs(st0).max()))
        assert np.isfinite(st).all() and err < 1e-12, (k, err)
        assert np.isfinite(c) and abs(np.longdouble(c) - r) <= 1e-13 * r, (k, c, float(r))


# ---------------------------------------------------------------------------------------------
# GPU: the alternative kernel paths behind tuning switches (one process each: the device switches are read
# when a graph's context is created, some go to process-wide __constant__ symbols, some are cached in statics)
# ---------------------------------------------------------------------------------------------
SWITCH_ZOO = ("smem159_c12", "smem_n51", "team162_c51", "team_chunk130", "bs_195", "wide")
SWITCHES = {
    "pf_groups0": {"ASAM_PF_GROUPS": "0"}, "dmap_ahead0": {"ASAM_DMAP_AHEAD": "0"},
    "smem_mma2": {"ASAM_SMEM_MMA": "2"}, "pb_smem24": {"ASAM_PB_SMEM": "24"},
    "solo400": {"ASAM_SOLO_MAX_M": "400"}, "solo400_pb24": {"ASAM_SOLO_MAX_M": "400", "ASAM_SOLO_PB": "24"},
    "solo400_pb12": {"ASAM_SOLO_MAX_M": "400", "ASAM_SOLO_PB": "12"}, "tpw2": {"ASAM_TILES_PER_WORKER": "2"},
    "merge_pct0": {"ASAM_TEAM_MERGE_PCT": "0"}, "plan_threads1": {"ASAM_PLAN_THREADS": "1"},
    "bs_threads128": {"ASAM_BS_THREADS": "128"},
    "order_cp": {"ASAM_TASK_ORDER": "cp"}, "order_sim": {"ASAM_TASK_ORDER": "sim"},
}
REPLAY_SWITCHES = {"keep0": {"ASAM_KEEP": "0"}, "small_step0": {"ASAM_SMALL_STEP": "0"}}


def _worker(kind):
    """Runs in a subprocess with the switch in its environment; prints one JSON line."""
    if kind == "batch":
        from aprilsam_b200 import datasets
        out = {}
        for name in SWITCH_ZOO:
            out[name] = batch_and_check(zoo(name))
        out["manhattan2000"] = batch_and_check(datasets.manhattan_dense(2000, seed=1), forward=False)
    else:
        m = H.PoseGraphData.load(os.path.join(ROOT, "tests", "golden", "m3500.npz")).head(300)
        st, wf, wr, nch, err = replay_checked(m, m.n_nodes, check_every=10)
        out = {"states": st.tolist(), "factor": wf, "rhs": wr, "x_err": err}
    print("RESULT " + json.dumps(out))


def _run_worker(kind, env):
    e = dict(os.environ)
    e.update(env)
    here = os.path.dirname(os.path.abspath(__file__))
    code = f"import sys; sys.path[:0] = [{ROOT!r}, {here!r}]; import test_gpu_kernels as t; t._worker({kind!r})"
    r = subprocess.run([sys.executable, "-c", code], env=e, capture_output=True, text=True, timeout=1200, cwd=ROOT)
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1]
    return json.loads(line[len("RESULT "):])


@pytest.mark.gpu
@pytest.mark.parametrize("switch", list(SWITCHES))
def test_switch_paths(switch):
    out = _run_worker("batch", SWITCHES[switch])
    for name, res in out.items():
        assert_solve_ok(res, f"{switch} {name}")


@pytest.fixture(scope="module")
def default_replay():
    return _run_worker("replay", {})


@pytest.mark.gpu
@pytest.mark.parametrize("switch", list(REPLAY_SWITCHES))
def test_replay_switches_match_default(switch, default_replay):
    base = default_replay
    alt = _run_worker("replay", REPLAY_SWITCHES[switch])
    for o in (base, alt):
        assert o["factor"] < FACTOR_TOL and o["rhs"] < RHS_TOL and o["x_err"] < 1e-12, o
    a, b = np.array(alt["states"]), np.array(base["states"])
    d = a - b
    d[:, 2] = emul.mod2pi(d[:, 2])
    assert np.abs(d).max() / max(1.0, np.abs(b).max()) < 1e-12
