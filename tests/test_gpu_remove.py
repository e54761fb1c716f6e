"""Factor removal (aprilsam_b200_remove_factors) on the GPU, checked kernel by kernel after every removal.

After each removal RemovalChecker (built on test_gpu_incremental.StepChecker) checks
  * the Hessian in HBM against the ledger of the remaining factors (support/removecheck.py), entry by entry, with
    the bound of check_linearize; dirty slots that no remaining factor maps to read exactly +0.0; every entry outside
    the dirty poses and slots is bit-identical to before;
  * the device copy of the plan and of the compacted factor mirror against the host's, bit for bit;
  * every re-factored front (local backward error) and y; every other front bit-identical to before;
  * full traversals: the back-substitution of every supernode and the long-double residual of the ledger system;
    pruned ones: the rows [3 bfirst, c) of every listed supernode, x outside the listed columns unchanged;
  * every pose whose state changed equals l_point + x(HBM) bit for bit, and no pose outside the listed columns moved.

Bounds: the constants of test_gpu_kernels.py, as in test_gpu_incremental.py.
"""
from __future__ import annotations

import numpy as np
import pytest

from aprilsam_b200 import datasets
from aprilsam_b200 import harness as H
from support import frontcheck as fc
from support import inccheck as ic
from support import removecheck as rc
from test_gpu_incremental import LAM, StepChecker
from test_gpu_kernels import CHI2_TOL, LINEARIZE_C

pytestmark = pytest.mark.gpu

ic.STEP_KINDS.setdefault(5, "remove")
ic.STEP_KINDS.setdefault(6, "remove_full")


def _bits(a):
    return np.ascontiguousarray(a).view(np.int64)


class RemovalChecker(StepChecker):
    """StepChecker whose ledger knows removals and robust losses, with a checked removal call."""

    def __init__(self, h, lam=LAM):
        super().__init__(h, lam)
        self.ledger = rc.RemovalLedger(lam)
        self.kinds = []

    def _sync_factors(self):
        super()._sync_factors()
        for i in range(len(self.factors[0])):  # the device mirror holds the type codes (32 for robust factors)
            self.factors[0][i] = self.h.factor(i)[0]

    def remove(self, idx, keep=False):
        h, L = self.h, self.L
        N = h.n_nodes
        self._sync_factors()
        x0 = np.zeros(3 * N)
        fc._ok(L, L.asam_download_x(self.dev, 0, N, x0.ctypes.data_as(fc._dp)), "download_x")
        st0 = h.states()
        snap0 = ic.snapshot(h, L)
        fslot0 = snap0.plan.array("fslot")
        led = self.ledger
        dirty = sorted(set(int(led.fa[f]) for f in idx) | set(int(led.fb[f]) for f in idx if led.fb[f] >= 0))
        dslot = sorted(set(int(fslot0[f]) for f in idx if led.fb[f] >= 0))
        nb0 = ic.batch_count(L)
        h.remove_factors(idx, keep=keep)
        rec = ic.last_step(L, h.param_ptr())
        escalated = ic.batch_count(L) > nb0
        assert escalated == rec["escalated"], rec
        keepm = np.ones(len(self.factors[0]), bool)
        keepm[list(idx)] = False
        self.factors = [a[keepm] for a in self.factors]
        if escalated:
            led.batch(h)
            st_before = np.full((N, 3), np.nan)
        else:
            assert rec["kind"] in ("remove", "remove_full"), rec
            led.remove(idx)
            st_before = st0
        self.kinds.append(("escalated " if escalated else "") + rec["kind"])
        self.nstep += 1
        full = escalated or rec["kind"] == "remove_full"
        self._check(rec, st_before, x0, N, full=full, all_fronts=True)
        if not escalated:
            snap = ic.snapshot(h, L)
            fslot = snap.plan.array("fslot")
            live = set(int(s) for s, t in zip(fslot, led.ft) if t == 1)
            od = np.ones(N, bool); od[dirty] = False
            os_ = np.ones(len(snap.Aoff), bool); os_[dslot] = False
            assert np.array_equal(_bits(snap.Adiag[od]), _bits(snap0.Adiag[od])), "Adiag outside the dirty poses"
            assert np.array_equal(_bits(snap.B[od]), _bits(snap0.B[od])), "Bq outside the dirty poses"
            assert np.array_equal(_bits(snap.Aoff[os_]), _bits(snap0.Aoff[os_])), "Aoff outside the dirty slots"
            for s in dslot:
                if s not in live:
                    assert np.all(_bits(snap.Aoff[s]) == 0), f"dead slot {s} is not +0.0"
            tasks = set(int(t) for t in rec["tasks"])
            for s in range(snap.nsn):
                if s not in tasks:
                    F0, r0 = snap0.fronts[s]
                    F1, r1 = snap.fronts[s]
                    assert np.array_equal(_bits(F0), _bits(F1)) and np.array_equal(_bits(r0), _bits(r1)), \
                        f"unmarked front {s} changed"
            # x on the listed columns (all of them for a full traversal) against the ledger system
            A, b = fc.system(snap, led.ft, led.fa, led.fb, fslot)
            xr, kappa = fc.reference_solution(A, b)
            mask = np.ones(N, bool) if full else ic.listed_columns(snap.desc, N, rec["bt"], rec["bfirst"])
            m3 = np.repeat(mask, 3)
            err = float(np.abs(snap.x[m3].astype(np.longdouble) - xr[m3]).max() / np.abs(xr).max())
            assert err <= 0.1 * kappa * fc.U + 1e-15, (err, kappa)
        return rec


def _closures(h, lo=0):
    """Indices of the loop closures (|a - b| > 1) among factors [lo, F)."""
    out = []
    for i in range(lo, h.n_factors):
        t, a, b, _, _ = h.factor(i)
        if b >= 0 and abs(a - b) > 1:
            out.append(i)
    return out


# ---------------------------------------------------------------------------------------------
# scenarios on the M3500 replay: plain, robust, priors, several at once, small and large naffected, appends after
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("robust", [False, True])
def test_remove_scenarios_m3500(m3500, robust):
    d = m3500.head(600)
    with H.Harness("b200") as h:
        if robust:
            h.set_scan_loss(H.Harness.HUBER, 1.0)
        with RemovalChecker(h) as chk:
            h.replay_begin(d)
            chk.batch(lambda: h.replay_to(1))
            for k in range(1, 300):
                chk.step(lambda: h.replay_to(k + 1))
            lc = _closures(h)
            chk.remove([lc[-1]])                        # the newest closure
            chk.remove([_closures(h)[3]])               # a deep old closure
            lc = _closures(h)
            chk.remove(lc[5:80:9], keep=True)           # several at once, handed back to the caller
            # a prior added by a step, then removed: rebuilt at the state it was added at
            N = h.n_nodes
            st = h.states()
            p = h.add_xytpos(N - 40, st[N - 40] + 0.01, [2e3, 0, 0, 0, 2e3, 0, 0, 0, 1e3])
            h.add_node(st[-1] + [0.5, 0, 0])
            h.add_xyt(N - 1, N, [0.5, 0, 0], [100, 0, 0, 0, 100, 0, 0, 0, 50])
            chk.step(h.inc)
            chk.remove([p])
            # a parallel edge between the two newest poses: a short root path
            N = h.n_nodes
            h.add_node(h.states()[-1] + [0.5, 0, 0])
            h.add_xyt(N - 1, N, [0.5, 0, 0], [100, 0, 0, 0, 100, 0, 0, 0, 50])
            h.add_xyt(N - 1, N, [0.52, 0.01, 0], [80, 0, 0, 0, 80, 0, 0, 0, 40])
            chk.step(h.inc)
            chk.remove([h.n_factors - 1])
            # the batch prior on pose 0
            chk.remove([0])
            # appends after removals (a new pose with odometry and a closure each), then one through the old-pose
            # fallback (slots renumbered)
            for k in range(12):
                N = h.n_nodes
                st = h.states()
                h.add_node(st[-1] + [0.4, 0.1, 0.02])
                h.add_xyt(N - 1, N, [0.4, 0.1, 0.02], [100, 0, 0, 0, 100, 0, 0, 0, 50])
                c = N - 30 - 7 * k
                dd = st[-1] + [0.4, 0.1, 0.02] - st[c]
                cc, ss = np.cos(st[c, 2]), np.sin(st[c, 2])
                h.add_xyt(c, N, [cc * dd[0] + ss * dd[1], -ss * dd[0] + cc * dd[1], dd[2]], [20, 0, 0, 0, 20, 0, 0, 0, 10])
                chk.step(h.inc)
            chk.remove([_closures(h)[-2]])
            h.add_xyt(5, 250, [0, 0, 0], [10, 0, 0, 0, 10, 0, 0, 0, 5])
            rec = chk.step(h.inc)
            assert rec["kind"] == "fallback"
            chk.remove([h.n_factors - 1])
            # an escalation: the policy sends the removal to a batch solve of the reduced graph
            h.set_policy_ratio(1e-300)
            chk.remove([_closures(h)[10]])
            h.set_policy_ratio(0.0)
            kinds = chk.kinds
            assert "remove" in kinds and "remove_full" in kinds and any(k.startswith("escalated") for k in kinds), kinds


def test_remove_every_kth_closure_replay(m3500):
    """The M3500 replay with every 4th loop closure removed one step after it arrived."""
    d = m3500.head(700)
    with H.Harness("b200") as h:
        with RemovalChecker(h) as chk:
            h.replay_begin(d)
            chk.batch(lambda: h.replay_to(1))
            seen = 0
            for k in range(1, d.n_nodes):
                F0 = h.n_factors
                chk.step(lambda: h.replay_to(k + 1, want_chi2=False))
                for f in _closures(h, F0):
                    seen += 1
                    if seen % 4 == 0:
                        chk.remove([f])
                        break
            assert len(chk.kinds) > 20


def test_remove_team_root():
    """A dense world whose root path runs through team fronts: the removal re-factors them whole."""
    d = datasets.manhattan_dense(12000, seed=5)
    with H.Harness("b200") as h:
        h.load_full(d)
        with RemovalChecker(h) as chk:
            chk.batch()
            rec = chk.remove([_closures(h)[-1], _closures(h)[len(_closures(h)) // 2]])
            assert (((rec["nwait"] >> 24) & 0x7f) > 1).any(), "team entries in the task list"


# ---------------------------------------------------------------------------------------------
# integer-valued systems: exact round trips
# ---------------------------------------------------------------------------------------------
def _integer_graph(h, n=40, dup=False):
    """Poses on integer grid points with theta 0, integer z and diagonal integer W: every Jacobian, residual and
    Hessian entry is an integer, so any order of summation gives the same bits."""
    for i in range(n):
        h.add_node([float(i % 8), float(i // 8), 0.0])
    h.add_xytpos(0, [0, 0, 0], [16, 0, 0, 0, 16, 0, 0, 0, 8])
    W = [4, 0, 0, 0, 4, 0, 0, 0, 2]
    for i in range(1, n):
        a = i - 1 if i % 8 else i - 8
        h.add_xyt(a, i, [float(i % 8 - a % 8), float(i // 8 - a // 8), 0], W)
        if dup and i == 9:
            h.add_xyt(a, i, [1.0, 0.0, 0.0], [2, 0, 0, 0, 2, 0, 0, 0, 1])
    for i in range(8, n, 3):
        h.add_xyt(i - 8 + 1, i, [float(i % 8 - (i - 7) % 8), 1.0, 0.0], [2, 0, 0, 0, 2, 0, 0, 0, 2])


def test_round_trip_integer_system():
    L = ic.dev_api()
    with H.Harness("b200") as h:
        h.set_tikhanov(0.5)
        _integer_graph(h)
        h.batch()
        s0 = ic.snapshot(h, L)
        st0 = h.states()
        S0 = len(s0.Aoff)
        h.add_xyt(3, 30, [-5.0, 3.0, 0.0], [2, 0, 0, 0, 2, 0, 0, 0, 1])  # between two solved poses: the fallback
        h.inc()
        st_fb = h.states()
        h.remove_factors([h.n_factors - 1])
        s1 = ic.snapshot(h, L)
        assert np.array_equal(_bits(s1.Adiag), _bits(s0.Adiag))
        assert np.array_equal(_bits(s1.B), _bits(s0.B))
        assert np.array_equal(_bits(s1.Aoff[:S0]), _bits(s0.Aoff[:S0]))
        assert np.all(_bits(s1.Aoff[S0:]) == 0)
        st1 = h.states()
        moved = np.any(_bits(st1) != _bits(st_fb), axis=1)  # the poses the removal's traversal updated
        if h.info()["naffected"] > 5:
            assert moved.sum() > 0
            moved[:] = True
        assert np.abs(st1[moved] - st0[moved]).max() <= 1e-12 * max(1.0, np.abs(st0).max())


def test_parallel_edge_slot_exact():
    """Two factors on one slot; removing one leaves exactly the other's block (compared with a graph that never had
    it).  A repeated removal on a copy rebuilds the same bits."""
    L = ic.dev_api()
    with H.Harness("b200") as a, H.Harness("b200") as b, H.Harness("b200") as c:
        for h in (a, b, c):
            h.set_tikhanov(0.5)
        _integer_graph(a, dup=True)
        _integer_graph(c, dup=True)
        _integer_graph(b, dup=False)
        for h in (a, b, c):
            h.batch()
        dup = next(i for i in range(a.n_factors) if a.factor(i)[1:3] == (8, 9) and a.factor(i)[4][0] == 2.0)
        a.remove_factors([dup])
        c.remove_factors([dup])
        sa, sb, sc = ic.snapshot(a, L), ic.snapshot(b, L), ic.snapshot(c, L)
        fa_, fb_ = sa.plan.array("fslot"), sb.plan.array("fslot")
        assert a.n_factors == b.n_factors
        for f in range(a.n_factors):
            assert np.array_equal(_bits(sa.Aoff[fa_[f]]), _bits(sb.Aoff[fb_[f]])) if fa_[f] >= 0 else True
        assert np.array_equal(_bits(sa.Adiag), _bits(sb.Adiag)) and np.array_equal(_bits(sa.B), _bits(sb.B))
        for x, y in ((sa.Adiag, sc.Adiag), (sa.B, sc.B), (sa.Aoff, sc.Aoff)):
            assert np.array_equal(_bits(x), _bits(y)), "the same removal on a copy gives other bits"


def test_repeated_removal_same_bits(m3500):
    """The same removal on two copies of a graph rebuilds its dirty entries to the same bits (no atomics)."""
    L = ic.dev_api()
    d = m3500.head(300)
    with H.Harness("b200", nthreshold=1 << 30) as a, H.Harness("b200", nthreshold=1 << 30) as b:
        for h in (a, b):
            h.load_full(d)
            h.batch()
        idx = _closures(a)[::11]
        dirty = sorted(set(v for f in idx for v in a.factor(f)[1:3] if v >= 0))
        fs = fc.borrowed_plan(L, a.param_ptr()).array("fslot")
        slots = sorted(set(int(fs[f]) for f in idx))
        for h in (a, b):
            h.remove_factors(idx)
        sa, sb = ic.snapshot(a, L), ic.snapshot(b, L)
        for x, y in ((sa.Adiag[dirty], sb.Adiag[dirty]), (sa.B[dirty], sb.B[dirty]), (sa.Aoff[slots], sb.Aoff[slots])):
            assert np.array_equal(_bits(x), _bits(y))


# ---------------------------------------------------------------------------------------------
# after a removal: batch solves, chi2 and the queries
# ---------------------------------------------------------------------------------------------
def _copy_graph(src, dst):
    """dst gets src's poses (states) and factors, in order."""
    for p in src.states():
        dst.add_node(p)
    for i in range(src.n_factors):
        t, a, b, z, W = src.factor(i)
        if b >= 0:
            dst.add_xyt(a, b, z, W)
        else:
            dst.add_xytpos(a, z, W)


def test_batch_after_removal_matches_fresh_copy(m3500):
    d = m3500.head(500)
    with H.Harness("b200") as h, H.Harness("b200") as g:
        h.replay_begin(d)
        h.replay_to(400)
        lc = _closures(h)
        h.remove_factors(lc[::7])
        h.batch()
        _copy_graph(h, g)
        g.set_states(h.l_points())
        g.batch()
        assert np.array_equal(h.ordering(), g.ordering())
        ref = g.states()
        assert np.abs(h.states() - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())
        want = fc.chi2_ref(*ic.factors_of(h), h.states())
        assert abs(h.chi2() - float(want)) <= CHI2_TOL * float(want)


def test_queries_after_removal(m3500):
    d = m3500.head(120)
    with H.Harness("b200") as h:
        with RemovalChecker(h) as chk:
            h.replay_begin(d)
            chk.batch(lambda: h.replay_to(1))
            for k in range(1, d.n_nodes):
                chk.step(lambda: h.replay_to(k + 1))
            chk.remove([_closures(h)[-1], _closures(h)[2]])
            plan = fc.borrowed_plan(chk.L, h.param_ptr())
            N = h.n_nodes
            A, _ = chk.ledger.dense_ld(N, plan.info()["n_slots"], plan.array("fslot"), plan.array("node2q"))
            Sig = np.linalg.inv(A.astype(np.float64))
            ids = [0, 17, N // 2, N - 1]
            got = h.marginal_covariance(ids)
            I = np.concatenate([3 * p + np.arange(3) for p in ids])
            want = Sig[np.ix_(I, I)]
            assert np.abs(got - want).max() <= 1e-8 * np.abs(want).max()
            a, b = np.array([N - 1, 5]), np.array([3, -1])
            z = np.array([[0.1, 0.2, 0.05], [0.0, 0.1, 0.0]])
            W = np.array([np.diag([50.0, 50.0, 20.0]).reshape(9)] * 2)
            d2, cov = h.candidate_mahalanobis(a, b, z, W, with_cov=True)
            st, lp = h.states(), h.l_points()
            for c in range(2):
                ia = slice(3 * a[c], 3 * a[c] + 3)
                if b[c] < 0:
                    Srel = Sig[ia, ia]
                    r = z[c] - st[a[c]]
                else:
                    pa, pb = lp[a[c]], lp[b[c]]
                    from support import emul
                    Ja, Jb, _ = emul.xyt_eval(pa, pb, z[c])
                    J = np.c_[Ja, Jb]
                    idx = np.r_[3 * a[c] + np.arange(3), 3 * b[c] + np.arange(3)]
                    Srel = J @ Sig[np.ix_(idx, idx)] @ J.T
                    _, _, r = emul.xyt_eval(st[a[c]], st[b[c]], z[c])
                assert np.abs(cov[c] - Srel).max() <= 1e-8 * np.abs(Srel).max()
                if b[c] < 0:
                    r[2] = ((r[2] + np.pi) % (2 * np.pi)) - np.pi
                S = Srel + np.linalg.inv(W[c].reshape(3, 3))
                assert abs(d2[c] - r @ np.linalg.solve(S, r)) <= 1e-8 * max(1.0, abs(d2[c]))


# ---------------------------------------------------------------------------------------------
# errors: -1, the message, nothing changed, and the next call runs cleanly
# ---------------------------------------------------------------------------------------------
def _state(h, L):
    s = ic.snapshot(h, L)
    facs = [h.factor(i) for i in range(h.n_factors)]
    return dict(info=h.info(), nf=h.n_factors, states=h.states().copy(), Ad=s.Adiag.copy(), Ao=s.Aoff.copy(),
                B=s.B.copy(), x=s.x.copy(), fronts={k: (v[0].copy(), v[1].copy()) for k, v in s.fronts.items()},
                facs=[(t, a, b, z.tobytes(), W.tobytes()) for t, a, b, z, W in facs])


def _same(s0, s1):
    assert s0["info"] == s1["info"] and s0["nf"] == s1["nf"] and s0["facs"] == s1["facs"]
    for k in ("states", "Ad", "Ao", "B", "x"):
        assert np.array_equal(_bits(s0[k]), _bits(s1[k])), k
    for k in s0["fronts"]:
        assert np.array_equal(_bits(s0["fronts"][k][0]), _bits(s1["fronts"][k][0])), k


def _expect_error(h, L, idx, words):
    s0 = _state(h, L)
    with pytest.raises(RuntimeError) as e:
        h.remove_factors(idx)
    assert all(w in str(e.value) for w in words), str(e.value)
    _same(s0, _state(h, L))


def test_errors_change_nothing(m3500):
    L = ic.dev_api()
    d = m3500.head(80)
    with H.Harness("b200") as h:
        h.replay_begin(d)
        h.replay_to(60)
        F = h.n_factors
        _expect_error(h, L, [], ["n < 1"])
        _expect_error(h, L, [F], ["not in [0"])
        _expect_error(h, L, [-1], ["not in [0"])
        _expect_error(h, L, [4, 4], ["twice"])
        # a new pose whose only link is removed; a chain of new poses cut off
        N = h.n_nodes
        h.add_node(h.states()[-1] + [1, 0, 0])
        h.add_xyt(N - 1, N, [1, 0, 0], [10, 0, 0, 0, 10, 0, 0, 0, 5])
        h.inc()
        _expect_error(h, L, [h.n_factors - 1], ["pose %d" % N, "unconstrained"])
        h.add_node(h.states()[-1] + [1, 0, 0])
        h.add_xyt(N, N + 1, [1, 0, 0], [10, 0, 0, 0, 10, 0, 0, 0, 5])
        h.inc()
        _expect_error(h, L, [h.n_factors - 2], ["unconstrained"])
        # poses or factors added since the last solve
        h.add_node(h.states()[-1] + [1, 0, 0])
        h.add_xyt(N + 1, N + 2, [1, 0, 0], [10, 0, 0, 0, 10, 0, 0, 0, 5])
        _expect_error(h, L, [3], ["added since the last solve"])
        h.inc()
        # an edited factor on a removed factor's pose, re-checked by chi2 (stale mirror)
        lc = _closures(h)
        t, a, b, z, W = h.factor(lc[0])
        nb = next(i for i in range(h.n_factors) if i != lc[0] and a in h.factor(i)[1:3])
        _, _, _, z2, W2 = h.factor(nb)
        h.set_factor(nb, z2 + 0.01, W2)
        h.chi2()
        _expect_error(h, L, [lc[0]], ["edited"])
        h.batch()  # the batch relinearises: the removal is fine now
        h.remove_factors([lc[0]])
        # a dropped plan
        h.invalidate_plan()
        _expect_error(h, L, [3], ["invalidate_plan"])
        h.batch()
        # accepted: an old pose left with only lambda; a new pose kept by a prior
        N = h.n_nodes
        inc = [i for i in range(h.n_factors) if 20 in h.factor(i)[1:3]]
        h.remove_factors(inc)
        assert h.info()["factor_num"] == h.n_factors
        h.add_node(h.states()[-1] + [1, 0, 0])
        h.add_xyt(N - 1, N, [1, 0, 0], [10, 0, 0, 0, 10, 0, 0, 0, 5])
        h.add_xytpos(N, h.states()[-1], [10, 0, 0, 0, 10, 0, 0, 0, 5])
        h.inc()
        h.remove_factors([h.n_factors - 2])
        h.batch()
        assert np.all(np.isfinite(h.states()))


def test_never_solved_splice_and_other_params(m3500):
    L = ic.dev_api()
    d = m3500.head(100)
    with H.Harness("b200") as h:
        h.load_full(d)
        F = h.n_factors
        f5 = h.factor(5)
        h.remove_factors([3, 4], keep=True)  # never solved: the splice alone
        assert h.n_factors == F - 2 and h.factor(3)[1:3] == f5[1:3]
        h.batch()
        # a second param on the same graph solves it, then the first removes a factor
        other = h.new_param()
        mine = h.swap_param(other)
        h.batch()
        h.swap_param(mine)
        h.remove_factors([_closures(h)[0]])
        h.swap_param(other)
        st0 = h.states()
        h.add_node(st0[-1] + [1, 0, 0])
        h.add_xyt(d.n_nodes - 1, d.n_nodes, [1, 0, 0], [10, 0, 0, 0, 10, 0, 0, 0, 5])
        h.inc()
        assert "removed from this graph through another param" in h.last_error()
        assert np.array_equal(_bits(h.states()[:-1]), _bits(st0))
        with pytest.raises(RuntimeError, match="another param"):
            h.marginal_covariance([1])
        with pytest.raises(RuntimeError, match="another param"):
            h.remove_factors([1])
        h.batch()  # re-plans
        plan = fc.borrowed_plan(L, h.param_ptr())
        assert plan.info()["n_factors"] == h.n_factors
        h.marginal_covariance([1])
        with H.Harness("b200") as g:
            _copy_graph(h, g)
            g.set_states(h.l_points())
            g.batch()
            assert np.abs(h.states() - g.states()).max() <= 1e-12 * max(1.0, np.abs(g.states()).max())
        h.swap_param(mine)
        h.free_param(other)
