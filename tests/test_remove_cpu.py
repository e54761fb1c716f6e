"""Factor removal, host side (-m "not gpu"): plan_refactor's task lists, plan_remove_factors' compaction, and the
emulated kernels running a removal's re-factorisation on the Hessian of the remaining factors.

A removal changes no structure: the plan keeps its supernodes, fronts and slots, and only the supernodes on the root
paths of the removed factors' poses are re-factored, each from its first marked column (keep words).  The emulation
(support/emul.py) checks every kept column against a full elimination and the solution against a sparse solve.
"""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse.linalg as spl

from aprilsam_b200 import datasets
from support import emul
from support import removecheck as rc
from support.hostplan import HostPlan, lib

_ip = C.POINTER(C.c_int)


def _api():
    L = lib()
    L.asam_dbg_plan_refactor.argtypes = [C.c_void_p, _ip, C.c_int, _ip, _ip, _ip, C.c_int]
    L.asam_dbg_plan_remove_factors.argtypes = [C.c_void_p, C.c_int, _ip]
    return L


def _i(a):
    return a.ctypes.data_as(_ip)


def refactor(p, marked):
    L = _api()
    marked = np.ascontiguousarray(marked, np.int32)
    cap = 4 * p.info()["nsn"] + 16
    t, w, k = (np.zeros(cap, np.int32) for _ in range(3))
    nt = L.asam_dbg_plan_refactor(p.p, _i(marked), len(marked), _i(t), _i(w), _i(k), cap)
    return t[:nt].copy(), w[:nt].copy(), k[:nt].copy()


def remove(p, idx):
    L = _api()
    idx = np.ascontiguousarray(sorted(idx), np.int32)
    if L.asam_dbg_plan_remove_factors(p.p, len(idx), _i(idx)) != 0:
        raise RuntimeError(L.aprilsam_b200_last_error().decode())


def factor_arrays(d):
    E = d.n_edges
    ftype = np.r_[2, np.ones(E, np.int32)].astype(np.int32)
    fa = np.r_[0, d.ea].astype(np.int32)
    fb = np.r_[-1, d.eb].astype(np.int32)
    fz = np.vstack([[0, 0, 0], d.ez])
    fW = np.vstack([[1e4, 0, 0, 0, 1e4, 0, 0, 0, 1e3], d.eW])
    return ftype, fa, fb, fz, fW


def snapshot_arrays(p):
    return {k: p.array(k) for k in ("order", "pos", "node2q", "q2node", "parent_pos", "sn_of_q", "ipool", "tasks",
                                    "nwait", "btasks", "desc", "leaf_tasks")}


def closures(fa, fb, n):
    """n loop closures (|a - b| > 1), spread over the factor list"""
    lc = np.nonzero((fb >= 0) & (np.abs(fa - fb) > 1))[0]
    return [int(v) for v in lc[np.linspace(0, len(lc) - 1, n).astype(int)]]


@pytest.fixture(scope="module")
def team_world():
    """Manhattan world whose top fronts are team fronts (G >= 2) in the batch schedule."""
    return datasets.manhattan_dense(12000, seed=5)


@pytest.mark.parametrize("world", ["m3500", "dense2k", "dense12k"])
def test_refactor_lists(m3500, world):
    d = {"m3500": m3500, "dense2k": datasets.manhattan_dense(2000, seed=3),
         "dense12k": datasets.manhattan_dense(12000, seed=5)}[world]
    ftype, fa, fb, _, _ = factor_arrays(d)
    p = HostPlan().build(d.n_nodes, ftype, fa, fb)
    before = snapshot_arrays(p)
    teams = 0
    rng = np.random.default_rng(1)
    picks = [closures(fa, fb, 1), closures(fa, fb, 16), [1, 2, 3], list(rng.choice(len(ftype), 5, replace=False))]
    for idx in picks:
        ends = [int(fa[f]) for f in idx] + [int(fb[f]) for f in idx if fb[f] >= 0]
        marked = rc.root_paths(p, ends)
        t, w, k = refactor(p, marked)
        assert rc.refactor_contract(p, marked, t, w, k) == []
        teams += int((((w >> 24) & 0x7f) > 1).any())
    after = snapshot_arrays(p)
    for name in before:
        assert np.array_equal(before[name], after[name]), f"plan_refactor changed {name}"
    if world == "dense12k":
        assert teams > 0, "a removal near the top re-factors a team front"


def test_remove_compacts_fslot_only(m3500):
    ftype, fa, fb, _, _ = factor_arrays(m3500)
    p = HostPlan().build(m3500.n_nodes, ftype, fa, fb)
    before = snapshot_arrays(p)
    fs0, info0 = p.array("fslot"), p.info()
    idx = closures(fa, fb, 7) + [0]
    remove(p, idx)
    keep = np.ones(len(ftype), bool)
    keep[idx] = False
    assert np.array_equal(p.array("fslot"), fs0[keep])
    info1 = p.info()
    assert info1["n_factors"] == info0["n_factors"] - len(idx)
    assert {k: v for k, v in info1.items() if k != "n_factors"} == {k: v for k, v in info0.items() if k != "n_factors"}
    after = snapshot_arrays(p)
    for name in before:
        assert np.array_equal(before[name], after[name]), f"plan_remove_factors changed {name}"
    # invalid lists change nothing
    for bad in ([5, 5], [-1], [len(ftype) - len(idx)], [9, 3]):
        L = _api()
        arr = np.ascontiguousarray(bad, np.int32)
        assert L.asam_dbg_plan_remove_factors(p.p, len(arr), _i(arr)) == -1
        assert np.array_equal(p.array("fslot"), fs0[keep])


def _emulate_removals(d, n0, script, lam=1e-4):
    """Batch of the first n0 poses, then the script: ("add", n) appends poses up to n (with their edges), ("rm",
    [factor ids]) removes factors.  Every removal runs plan_refactor's lists through emul.factor with keep on the
    ledger Hessian of the remaining factors; the solution is checked against a sparse solve after each one."""
    db, estart = d.bucketed()
    E = estart[n0]
    ftype = np.r_[2, np.ones(E, np.int32)].astype(np.int32)
    fa = np.r_[0, db.ea[:E]].astype(np.int32)
    fb = np.r_[-1, db.eb[:E]].astype(np.int32)
    fz = np.vstack([[0, 0, 0], db.ez[:E]])
    fW = np.vstack([[1e4, 0, 0, 0, 1e4, 0, 0, 0, 1e3], db.eW[:E]])
    p = HostPlan().build(n0, ftype, fa, fb)
    lp = d.init.copy()
    N = n0

    def hessian(N):
        info = p.info()
        Hs = emul.Hessian(N, info["n_slots"])
        Hs.reset(n0, lam)
        Hs.linearize(range(len(ftype)), ftype, fa, fb, fz, fW, lp, lp, p.array("node2q"), p.array("fslot"))
        return Hs

    Hs = hessian(N)
    fr = emul.Fronts()
    fr.ensure(N)
    leaf = p.array("leaf_tasks")  # large graphs: k_factor_leaf runs these first
    if len(leaf):
        emul.factor(fr, Hs, p.descs(), p.array("ipool"), p.array("q2node"), leaf, None)
    emul.factor(fr, Hs, p.descs(), p.array("ipool"), p.array("q2node"), p.array("tasks"), p.array("nwait"), prior=leaf)
    kept = removals = 0
    for op, arg in script:
        if op == "add":
            e0, e1 = estart[N], estart[arg]
            F0 = len(ftype)
            ftype = np.r_[ftype, np.ones(e1 - e0, np.int32)].astype(np.int32)
            fa = np.r_[fa, db.ea[e0:e1]].astype(np.int32)
            fb = np.r_[fb, db.eb[e0:e1]].astype(np.int32)
            fz, fW = np.vstack([fz, db.ez[e0:e1]]), np.vstack([fW, db.eW[e0:e1]])
            ends = [v for f in range(F0, len(ftype)) for v in (fa[f], fb[f]) if v < N]
            marked = rc.root_paths(p, ends)
            r = p.append(arg, ftype, fa, fb, sorted(marked))
            assert r is not None
            tasks, nwait = r
            keep = p.last_keep
            N = arg
        else:
            idx = sorted(arg(ftype, fa, fb, N))
            ends = [int(fa[f]) for f in idx] + [int(fb[f]) for f in idx if fb[f] >= 0]
            marked = rc.root_paths(p, ends)
            remove(p, idx)
            m = np.ones(len(ftype), bool)
            m[idx] = False
            ftype, fa, fb, fz, fW = ftype[m], fa[m], fb[m], fz[m], fW[m]
            tasks, nwait, keep = refactor(p, marked)
            assert rc.refactor_contract(p, marked, tasks, nwait, keep) == []
            removals += 1
        Hs = hessian(N)
        fr.ensure(N)
        k0 = getattr(fr, "kept_cols", 0)
        emul.factor(fr, Hs, p.descs(), p.array("ipool"), p.array("q2node"), tasks, nwait, keep=keep)
        if op == "rm":
            kept += getattr(fr, "kept_cols", 0) - k0
            info = p.info()
            fslot = p.array("fslot")
            pairs = [(0, 0)] * info["n_slots"]
            for f in range(len(ftype)):
                if ftype[f] == 1:
                    pairs[fslot[f]] = (min(fa[f], fb[f]), max(fa[f], fb[f]))
            fr2 = emul.Fronts()
            fr2.F, fr2.rhs, fr2.y, fr2.x = fr.F, fr.rhs, fr.y.copy(), fr.x.copy()
            emul.backsolve(fr2, p.descs(), p.array("ipool"), np.arange(info["nsn"] - 1, -1, -1))
            A = Hs.dense(pairs)
            xs = spl.spsolve(A.tocsc(), Hs.B.reshape(-1))
            node2q = p.array("node2q")
            x = np.concatenate([fr2.x[3 * node2q[i]:3 * node2q[i] + 3] for i in range(N)])
            assert np.abs(x - xs).max() < 1e-8 * max(1.0, np.abs(xs).max())
    return removals, kept


def test_emulated_removals_in_m3500_replay(m3500):
    """Removals interleaved with appends: the removal's task list and keep words on the ledger Hessian of the
    remaining factors reproduce a full elimination of it."""
    def last_closure(ft, fa, fb, N):
        lc = np.nonzero((fb >= 0) & (np.abs(fa - fb) > 1))[0]
        return [int(lc[-1])]

    def deep_closure(ft, fa, fb, N):
        lc = np.nonzero((fb >= 0) & (np.abs(fa - fb) > 1) & (np.maximum(fa, fb) < 60))[0]
        return [int(lc[0])]

    def several(ft, fa, fb, N):
        lc = np.nonzero((fb >= 0) & (np.abs(fa - fb) > 1))[0]
        return [int(v) for v in lc[::max(1, len(lc) // 6)][:6]]

    script = [("rm", last_closure), ("add", 260), ("rm", deep_closure), ("add", 300), ("rm", several),
              ("add", 330), ("rm", last_closure), ("add", 360)]
    removals, kept = _emulate_removals(m3500, 240, script)
    assert removals == 4
    assert kept > 0, "some removal kept the leading columns of a marked supernode"


def test_emulated_removal_team_root(team_world):
    """A removal on a world whose root path runs through team fronts (whole fronts re-factored)."""
    d = team_world

    def top_closure(ft, fa, fb, N):
        lc = np.nonzero((fb >= 0) & (np.abs(fa - fb) > 1))[0]
        return [int(lc[-1]), int(lc[len(lc) // 2])]

    removals, _ = _emulate_removals(d, d.n_nodes, [("rm", top_closure)])
    assert removals == 1
