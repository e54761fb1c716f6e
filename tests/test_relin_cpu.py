"""In-place relinearisation, host side (-m "not gpu"): the dirty sets, plan_refactor's lists for their root paths, and
the emulated kernels running those lists on the Hessian rebuilt at the mixed evaluation points.

Relinearising poses P changes no structure.  The factors with a pose in P (R) move to the new l_points of P, so the
diagonal blocks of their poses (D: P and its factor neighbours) and the slots of R's two-pose factors change, and
nothing else.  Only the supernodes on the root paths of D are re-factored, each from its first marked column (keep
words); the emulation (support/emul.py) checks every kept column against a full elimination and the solution against
a sparse solve.
"""
import numpy as np
import pytest
import scipy.sparse.linalg as spl

from aprilsam_b200 import datasets
from support import emul
from support import relincheck as rl
from support import removecheck as rc
from support.hostplan import HostPlan
from test_remove_cpu import factor_arrays, refactor, remove, snapshot_arrays

LAM = 1e-4
PRIOR_W = np.array([1e4, 0, 0, 0, 1e4, 0, 0, 0, 1e3])


class Emulation:
    """A host plan, the factors with their evaluation points, l_points and states, and the emulated fronts."""

    def __init__(self, d, n0, rng):
        db, self.estart = d.bucketed()
        self.db = db
        E = self.estart[n0]
        self.ftype = np.r_[2, np.ones(E, np.int32)].astype(np.int32)
        self.fa = np.r_[0, db.ea[:E]].astype(np.int32)
        self.fb = np.r_[-1, db.eb[:E]].astype(np.int32)
        self.fz = np.vstack([[0, 0, 0], db.ez[:E]])
        self.fW = np.vstack([PRIOR_W, db.eW[:E]])
        self.p = HostPlan().build(n0, self.ftype, self.fa, self.fb)
        self.N, self.n0 = n0, n0
        self.lp = d.init.copy() + rng.normal(0, 0.02, d.init.shape)  # the batch's l_points
        self.st = self.lp.copy()
        self.pts = self._pts_at_lp(np.arange(len(self.ftype)))
        self.fr = emul.Fronts()
        self.fr.ensure(self.N)
        H = self.hessian()
        leaf = self.p.array("leaf_tasks")
        if len(leaf):
            emul.factor(self.fr, H, self.p.descs(), self.p.array("ipool"), self.p.array("q2node"), leaf, None)
        emul.factor(self.fr, H, self.p.descs(), self.p.array("ipool"), self.p.array("q2node"), self.p.array("tasks"),
                    self.p.array("nwait"), prior=leaf)
        self.H = H
        self.solve_all()
        self.kept = 0

    def _pts_at_lp(self, fs):
        fs = np.asarray(fs, int)
        b = np.maximum(self.fb[fs], 0)
        return np.where((self.fb[fs] >= 0)[:, None], np.c_[self.lp[self.fa[fs]], self.lp[b]],
                        np.c_[self.lp[self.fa[fs]], np.zeros((len(fs), 3))])

    def hessian(self):
        info = self.p.info()
        H = emul.Hessian(self.N, info["n_slots"])
        H.reset(self.n0, LAM)
        H.linearize(range(len(self.ftype)), self.ftype, self.fa, self.fb, self.fz, self.fW, self.lp, self.st,
                    self.p.array("node2q"), self.p.array("fslot"), pts=self.pts)
        return H

    def refactor_and_check(self, tasks, nwait, keep, H):
        self.fr.ensure(self.N)
        k0 = getattr(self.fr, "kept_cols", 0)
        emul.factor(self.fr, H, self.p.descs(), self.p.array("ipool"), self.p.array("q2node"), tasks, nwait, keep=keep)
        self.kept += getattr(self.fr, "kept_cols", 0) - k0
        self.H = H
        self.solve_all()

    def solve_all(self):
        """Full back-substitution; x against a sparse solve of the Hessian; states = l_point + x."""
        info = self.p.info()
        fslot = self.p.array("fslot")
        pairs = [(0, 0)] * info["n_slots"]
        for f in range(len(self.ftype)):
            if self.ftype[f] == 1:
                pairs[fslot[f]] = (min(self.fa[f], self.fb[f]), max(self.fa[f], self.fb[f]))
        fr2 = emul.Fronts()
        fr2.F, fr2.rhs, fr2.y, fr2.x = self.fr.F, self.fr.rhs, self.fr.y.copy(), self.fr.x.copy()
        emul.backsolve(fr2, self.p.descs(), self.p.array("ipool"), np.arange(info["nsn"] - 1, -1, -1))
        xs = spl.spsolve(self.H.dense(pairs).tocsc(), self.H.B.reshape(-1))
        node2q = self.p.array("node2q")
        x = np.concatenate([fr2.x[3 * node2q[i]:3 * node2q[i] + 3] for i in range(self.N)])
        assert np.abs(x - xs).max() < 1e-8 * max(1.0, np.abs(xs).max())
        self.x = x.reshape(-1, 3)
        self.st = self.lp[:self.N] + self.x
        self.st[:, 2] = emul.mod2pi(self.st[:, 2])

    def add(self, n):
        db, N = self.db, self.N
        e0, e1 = self.estart[N], self.estart[n]
        F0 = len(self.ftype)
        self.ftype = np.r_[self.ftype, np.ones(e1 - e0, np.int32)].astype(np.int32)
        self.fa = np.r_[self.fa, db.ea[e0:e1]].astype(np.int32)
        self.fb = np.r_[self.fb, db.eb[e0:e1]].astype(np.int32)
        self.fz, self.fW = np.vstack([self.fz, db.ez[e0:e1]]), np.vstack([self.fW, db.eW[e0:e1]])
        self.lp[N:n] = db.init[N:n]
        self.st = np.r_[self.st, self.lp[N:n]]
        ends = [v for f in range(F0, len(self.ftype)) for v in (self.fa[f], self.fb[f]) if v < N]
        r = self.p.append(n, self.ftype, self.fa, self.fb, sorted(rc.root_paths(self.p, ends)))
        assert r is not None
        self.N = n
        self.pts = np.r_[self.pts, self._pts_at_lp(np.arange(F0, len(self.ftype)))]
        self.refactor_and_check(r[0], r[1], self.p.last_keep, self.hessian())

    def add_prior(self, v):
        """A prior added by a step on an old pose, evaluated at the pose's state (its prior-table record)."""
        F0 = len(self.ftype)
        self.ftype = np.r_[self.ftype, 2].astype(np.int32)
        self.fa, self.fb = np.r_[self.fa, v].astype(np.int32), np.r_[self.fb, -1].astype(np.int32)
        self.fz, self.fW = np.vstack([self.fz, self.st[v] + 0.01]), np.vstack([self.fW, PRIOR_W * 0.2])
        r = self.p.append(self.N, self.ftype, self.fa, self.fb, sorted(rc.root_paths(self.p, [v])))
        assert r is not None
        self.pts = np.r_[self.pts, [np.r_[self.st[v], np.zeros(3)]]]
        self.refactor_and_check(r[0], r[1], self.p.last_keep, self.hessian())
        return F0

    def remove(self, idx):
        idx = sorted(idx)
        ends = [int(self.fa[f]) for f in idx] + [int(self.fb[f]) for f in idx if self.fb[f] >= 0]
        marked = rc.root_paths(self.p, ends)
        remove(self.p, idx)
        m = np.ones(len(self.ftype), bool)
        m[idx] = False
        for name in ("ftype", "fa", "fb", "fz", "fW", "pts"):
            setattr(self, name, getattr(self, name)[m])
        tasks, nwait, keep = refactor(self.p, marked)
        self.refactor_and_check(tasks, nwait, keep, self.hessian())

    def relinearize(self, P):
        """l_point = state on P; the factors with a pose in P move to the new points; only D and the dirty slots of
        the Hessian change; plan_refactor's lists for D's root paths re-factor it."""
        fslot = self.p.array("fslot")
        R, D, dslot = rl.dirty_sets(P, self.ftype, self.fa, self.fb, fslot)
        H0 = self.H
        self.lp[list(P)] = self.st[list(P)]
        self.pts[R] = self._pts_at_lp(R)
        H1 = self.hessian()
        od = np.ones(self.N, bool); od[D] = False
        os_ = np.ones(len(H1.Aoff), bool); os_[dslot] = False
        assert np.array_equal(H1.Adiag[od], H0.Adiag[od]) and np.array_equal(H1.B[od], H0.B[od]), "outside D"
        assert np.array_equal(H1.Aoff[os_], H0.Aoff[os_]), "outside the dirty slots"
        marked = rc.root_paths(self.p, D)
        tasks, nwait, keep = refactor(self.p, marked)
        assert rc.refactor_contract(self.p, marked, tasks, nwait, keep) == []
        self.refactor_and_check(tasks, nwait, keep, H1)
        return D

    def flagged(self, delta=0.1):
        """The poses a step would flag: |x| beyond delta_xy / delta_theta."""
        return [int(v) for v in np.nonzero((np.abs(self.x[:, :2]) > delta).any(1) | (np.abs(self.x[:, 2]) > delta))[0]]


def _worlds(m3500):
    return {"m3500": (m3500, 3500), "dense2k": (datasets.manhattan_dense(2000, seed=3), 2000),
            "dense12k": (datasets.manhattan_dense(12000, seed=5), 12000)}


@pytest.mark.parametrize("world", ["m3500", "dense2k", "dense12k"])
def test_relin_dirty_sets_and_lists(m3500, world):
    """D is P plus its factor neighbours; plan_refactor's lists for D's root paths keep the plan as it is and meet the
    contract; on the big world a relinearisation near the top re-factors a team front."""
    d, _ = _worlds(m3500)[world]
    ftype, fa, fb, _, _ = factor_arrays(d)
    p = HostPlan().build(d.n_nodes, ftype, fa, fb)
    before = snapshot_arrays(p)
    fslot = p.array("fslot")
    lc = np.nonzero((fb >= 0) & (np.abs(fa - fb) > 1))[0]
    N = d.n_nodes
    rng = np.random.default_rng(2)
    picks = [[N - 1], [int(fa[lc[0]])], [0], [int(fb[lc[-1]]), int(fa[lc[len(lc) // 2]])],
             list(rng.choice(N, 40, replace=False))]
    teams = 0
    for P in picks:
        R, D, dslot = rl.dirty_sets(P, ftype, fa, fb, fslot)
        nb = set(int(v) for p_ in P for f in range(len(ftype)) for v in (fa[f], fb[f])
                 if v >= 0 and p_ in (fa[f], fb[f]))
        assert set(D.tolist()) == set(int(v) for v in P) | nb
        assert all(fa[f] in P or fb[f] in P for f in R)
        marked = rc.root_paths(p, D)
        t, w, k = refactor(p, marked)
        assert rc.refactor_contract(p, marked, t, w, k) == []
        teams += int((((w >> 24) & 0x7f) > 1).any())
    after = snapshot_arrays(p)
    for name in before:
        assert np.array_equal(before[name], after[name]), f"plan_refactor changed {name}"
    if world == "dense12k":
        assert teams > 0, "a relinearisation near the top re-factors a team front"


@pytest.mark.parametrize("world", ["m3500", "dense2k", "dense12k"])
def test_emulated_relin_solves(m3500, world):
    """Relinearise chosen P at perturbed states (a new pose, an old one with closures, the pose with the batch prior, a
    pose with a step-added prior, many at once): the lists run with their keep words on the Hessian rebuilt at the
    mixed points match a sparse solve of that system."""
    d, _ = _worlds(m3500)[world]
    n = min(d.n_nodes, 600) if world == "m3500" else d.n_nodes
    rng = np.random.default_rng(4)
    em = Emulation(d.head(n) if n < d.n_nodes else d, n, rng)
    N = em.N
    em.st = em.st + rng.normal(0, 0.05, em.st.shape)  # states away from the l_points
    lc = np.nonzero((em.fb >= 0) & (np.abs(em.fa - em.fb) > 1))[0]
    em.relinearize([N - 1])
    em.relinearize([int(em.fa[lc[0]])])
    em.relinearize([0])
    if world != "dense12k":
        v = N // 3
        f = em.add_prior(v)
        em.st[v] += 0.03
        em.relinearize([v])
        assert np.array_equal(em.pts[f, :3], em.lp[v])
        em.relinearize(list(rng.choice(N, 25, replace=False)))
    assert em.kept > 0, "some relinearisation kept the leading columns of a marked supernode"


def test_emulated_relin_in_m3500_replay(m3500):
    """An emulated M3500 run where relinearisations of the flagged poses alternate with appends and removals."""
    rng = np.random.default_rng(7)
    em = Emulation(m3500, 200, rng)
    relins = 0
    for n in range(220, 420, 20):
        em.add(n)
        fl = em.flagged(0.02)
        if fl:
            em.relinearize(fl)
            relins += 1
        if n % 60 == 0:
            lc = np.nonzero((em.fb >= 0) & (np.abs(em.fa - em.fb) > 1))[0]
            em.remove([int(lc[-1])])
            fl = em.flagged(0.02)
            if fl:
                em.relinearize(fl[:10])
                relins += 1
    assert relins >= 5, relins


def test_counters_model():
    """The counter update of the contract on a small example: order kept, start_over down by the flagged hits."""
    so, rest, fl = rl.counters_after(5, [7, 3, 9, 1, 4], {7, 3, 9, 1, 4}, [9, 2, 7])
    assert so == 3 and rest == [3, 1, 4] and fl == {3, 1, 4}
