"""In-place relinearisation (aprilsam_b200_relinearize_poses) on the GPU, checked kernel by kernel after every call.

After each relinearisation RelinChecker (built on test_gpu_remove.RemovalChecker) checks
  * l_point = state on the relinearised poses P and nowhere else; order and plan unchanged;
  * the counters against the contract's model (support/relincheck.py): start_over, nlinearized_nodes and the order of
    the remaining tr->linearized_nodes, the solve's new flags appended behind them;
  * the Hessian in HBM against the ledger whose evaluation points moved with P, entry by entry, with the bound of
    check_linearize; every entry outside the dirty poses D and the dirty slots bit-identical to before;
  * the device copy of the plan and of the factor mirror against the host's, bit for bit;
  * every re-factored front (local backward error) and y; every front outside the task list bit-identical;
  * x against the ledger system (full and pruned traversals: the rows the back-substitution solved);
  * every pose whose state changed equals l_point + x(HBM) bit for bit, and no pose outside the listed columns moved.

Bounds: the constants of test_gpu_kernels.py, as in test_gpu_incremental.py.
"""
from __future__ import annotations

import numpy as np
import pytest

from aprilsam_b200 import datasets
from aprilsam_b200 import harness as H
from support import emul
from support import frontcheck as fc
from support import inccheck as ic
from support import relincheck as rl
from test_gpu_incremental import LAM
from test_gpu_kernels import CHI2_TOL
from test_gpu_remove import RemovalChecker, _closures, _copy_graph, _integer_graph, _same, _state

pytestmark = pytest.mark.gpu

ic.STEP_KINDS.setdefault(5, "remove")
ic.STEP_KINDS.setdefault(6, "remove_full")
ic.STEP_KINDS.setdefault(7, "relin")
ic.STEP_KINDS.setdefault(8, "relin_full")


def _bits(a):
    return np.ascontiguousarray(a).view(np.int64)


class RelinChecker(RemovalChecker):
    """RemovalChecker whose ledger follows relinearisations, with a checked relinearisation call."""

    def __init__(self, h, lam=LAM):
        super().__init__(h, lam)
        self.ledger = rl.RelinLedger(lam)

    def relin(self, ids=None):
        h, L = self.h, self.L
        N = h.n_nodes
        self._sync_factors()
        x0 = np.zeros(3 * N)
        fc._ok(L, L.asam_download_x(self.dev, 0, N, x0.ctypes.data_as(fc._dp)), "download_x")
        st0, lp0 = h.states(), h.l_points()
        info0, lin0, order0 = h.info(), h.linearized_nodes().tolist(), h.ordering()
        P = lin0 if ids is None else [int(v) for v in ids]
        snap0 = ic.snapshot(h, L)
        desc0 = snap0.plan.descs()
        led = self.ledger
        R, D, dslot = rl.dirty_sets(P, led.ft, led.fa, led.fb, snap0.plan.array("fslot"))
        nb0 = ic.batch_count(L)
        h.relinearize_poses(ids)
        rec = ic.last_step(L, h.param_ptr())
        escalated = ic.batch_count(L) > nb0
        assert escalated == rec["escalated"], rec
        if escalated:
            led.batch(h)
            st_before = np.full((N, 3), np.nan)
        else:
            assert rec["kind"] in ("relin", "relin_full"), rec
            lp = h.l_points()
            assert np.array_equal(_bits(lp[P]), _bits(st0[P])), "l_point = state on P"
            rest = np.ones(N, bool); rest[P] = False
            assert np.array_equal(_bits(lp[rest]), _bits(lp0[rest])), "l_points outside P"
            assert np.array_equal(h.ordering(), order0)
            assert h.info()["factor_num"] == info0["factor_num"] and h.info()["nreordering"] == info0["nreordering"]
            # counters: the contract's update, then the solve's own flags behind the remaining entries
            so, remaining, _ = rl.counters_after(info0["start_over"], lin0, lin0, P)
            lin1, info1 = h.linearized_nodes().tolist(), h.info()
            assert lin1[:len(remaining)] == remaining, (lin1[:20], remaining[:20])
            assert info1["nlinearized"] == len(lin1)
            assert info1["start_over"] == so + len(lin1) - len(remaining), (info1, so)
            led.relinearize(P, lp)
            st_before = st0
        self.kinds.append(("escalated " if escalated else "") + rec["kind"])
        self.nstep += 1
        full = escalated or rec["kind"] == "relin_full"
        self._check(rec, st_before, x0, N, full=full, all_fronts=True)
        if not escalated:
            snap = ic.snapshot(h, L)
            assert all(np.array_equal(desc0[k], snap.plan.descs()[k]) for k in desc0), "plan changed"
            od = np.ones(N, bool); od[D] = False
            os_ = np.ones(len(snap.Aoff), bool); os_[dslot] = False
            assert np.array_equal(_bits(snap.Adiag[od]), _bits(snap0.Adiag[od])), "Adiag outside D"
            assert np.array_equal(_bits(snap.B[od]), _bits(snap0.B[od])), "Bq outside D"
            assert np.array_equal(_bits(snap.Aoff[os_]), _bits(snap0.Aoff[os_])), "Aoff outside the dirty slots"
            tasks = set(int(t) for t in rec["tasks"])
            for s in range(snap.nsn):
                if s not in tasks:
                    F0, r0 = snap0.fronts[s]
                    F1, r1 = snap.fronts[s]
                    assert np.array_equal(_bits(F0), _bits(F1)) and np.array_equal(_bits(r0), _bits(r1)), \
                        f"unmarked front {s} changed"
            fslot = snap.plan.array("fslot")
            A, b = fc.system(snap, led.ft, led.fa, led.fb, fslot)
            xr, kappa = fc.reference_solution(A, b)
            mask = np.ones(N, bool) if full else ic.listed_columns(snap.desc, N, rec["bt"], rec["bfirst"])
            m3 = np.repeat(mask, 3)
            err = float(np.abs(snap.x[m3].astype(np.longdouble) - xr[m3]).max() / max(np.abs(xr).max(), 1e-300))
            assert err <= 0.1 * kappa * fc.U + 1e-15, (err, kappa)
        rec["D"], rec["R"] = D, R
        return rec


def _perturb(h, ids, scale, seed):
    st = h.states()
    st[ids] += np.random.default_rng(seed).normal(0, scale, (len(ids), 3))
    h.set_states(st)


# ---------------------------------------------------------------------------------------------
# scenarios on the M3500 replay
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("robust", [False, True])
def test_relin_scenarios_m3500(m3500, robust):
    d = m3500.head(500)
    with H.Harness("b200", nthreshold=1 << 30) as h:  # the flags accumulate: no escalation from start_over
        if robust:
            h.set_scan_loss(H.Harness.HUBER, 1.0)
        with RelinChecker(h) as chk:
            h.replay_begin(d)
            chk.batch(lambda: h.replay_to(1))
            for k in range(1, 300):
                chk.step(lambda: h.replay_to(k + 1))
            N = h.n_nodes
            rec = chk.relin([N - 1])                        # the newest pose: a short root path
            assert rec["kind"] == "relin", rec
            chk.relin([h.factor(_closures(h)[3])[1]])       # an old pose deep in the tree
            assert len(h.linearized_nodes()) > 0
            chk.relin(None)                                 # everything flagged, through the tree's own list
            assert h.info()["nlinearized"] == len(h.linearized_nodes())
            chk.relin([0])                                  # the pose with the batch prior
            # a prior added by a step, then its pose relinearised: the prior moves to the new l_point
            st = h.states()
            h.add_xytpos(N - 40, st[N - 40] + 0.01, [2e3, 0, 0, 0, 2e3, 0, 0, 0, 1e3])
            h.add_node(st[-1] + [0.5, 0, 0])
            h.add_xyt(N - 1, N, [0.5, 0, 0], [100, 0, 0, 0, 100, 0, 0, 0, 50])
            chk.step(h.inc)
            _perturb(h, [N - 40], 0.02, 1)
            chk.relin([N - 40, N])
            # appends after relinearisations (a new pose with odometry and a closure each)
            for k in range(8):
                N = h.n_nodes
                st = h.states()
                h.add_node(st[-1] + [0.4, 0.1, 0.02])
                h.add_xyt(N - 1, N, [0.4, 0.1, 0.02], [100, 0, 0, 0, 100, 0, 0, 0, 50])
                c = N - 30 - 7 * k
                dd = st[-1] + [0.4, 0.1, 0.02] - st[c]
                cc, ss = np.cos(st[c, 2]), np.sin(st[c, 2])
                h.add_xyt(c, N, [cc * dd[0] + ss * dd[1], -ss * dd[0] + cc * dd[1], dd[2]], [20, 0, 0, 0, 20, 0, 0, 0, 10])
                chk.step(h.inc)
                if k % 3 == 0:
                    chk.relin([N, c])
            # the old-pose fallback after relinearisations, then relinearisations and a removal after it
            h.add_xyt(5, 250, [0, 0, 0], [10, 0, 0, 0, 10, 0, 0, 0, 5])
            rec = chk.step(h.inc)
            assert rec["kind"] == "fallback"
            _perturb(h, [5, 250], 0.01, 2)
            chk.relin([5, 250])
            chk.remove([_closures(h)[-2]])
            chk.relin([h.n_nodes - 2])
            # an escalation: the policy sends the relinearisation to a batch solve
            h.set_policy_ratio(1e-300)
            chk.relin([h.n_nodes // 2])
            h.set_policy_ratio(0.0)
            kinds = chk.kinds
            assert "relin" in kinds and "relin_full" in kinds and any(k.startswith("escalated") for k in kinds), kinds


def test_relin_team_root():
    """A dense world whose root path runs through team fronts: the relinearisation re-factors them whole."""
    d = datasets.manhattan_dense(12000, seed=5)
    with H.Harness("b200") as h:
        h.load_full(d)
        with RelinChecker(h) as chk:
            chk.batch()
            top = int(h.ordering()[-1])
            _perturb(h, [top, d.n_nodes // 2], 0.01, 3)
            rec = chk.relin([top, d.n_nodes // 2])
            assert (((rec["nwait"] >> 24) & 0x7f) > 1).any(), "team entries in the task list"


def test_relin_replay_driver(m3500):
    """The M3500 replay with the flagged poses relinearised in place whenever start_over exceeds 20: every such call
    checked (Python loop), and the harness's own driver (h_set_relin_in_place) runs without an escalation."""
    d = m3500.head(400)
    L = ic.dev_api()
    with H.Harness("b200") as h:
        with RelinChecker(h) as chk:
            h.replay_begin(d)
            chk.batch(lambda: h.replay_to(1))
            relins = 0
            for k in range(1, d.n_nodes):
                rec = chk.step(lambda: h.replay_to(k + 1, want_chi2=False))
                assert not rec["escalated"]
                if h.info()["start_over"] > 20:
                    rec = chk.relin(None)
                    assert not rec["escalated"]
                    relins += 1
            assert relins > 0
            chk_chi2 = h.chi2()
    with H.Harness("b200") as h:
        h.set_relin_in_place(20)
        h.replay_begin(d)
        h.replay_to(1)
        nb0 = ic.batch_count(L)
        _, _, info = h.replay_to(d.n_nodes, want_chi2=False)
        assert ic.batch_count(L) == nb0, "an escalation from start_over"
        assert info[:, 1].max() <= 100
        calls, ms = h.relin_stats()
        assert calls > 0 and ms > 0
        assert abs(h.chi2() - chk_chi2) <= 1e-3 * chk_chi2


# ---------------------------------------------------------------------------------------------
# exactness
# ---------------------------------------------------------------------------------------------
def test_relin_at_l_point_is_exact():
    """On an integer-valued system, relinearising poses whose state equals their l_point rebuilds the batch's Hessian
    bit for bit, and a second such call leaves the Hessian, fronts, y and x bit-identical.  (The first call's fronts may
    differ from the batch's in the last bits: the batch factors through other kernel paths.)"""
    L = ic.dev_api()
    with H.Harness("b200") as h:
        h.set_tikhanov(0.5)
        _integer_graph(h)
        h.batch()
        h.set_states(h.l_points())
        sb = ic.snapshot(h, L)
        P = [3, 17, 39, 0]
        h.relinearize_poses(P)
        s0 = ic.snapshot(h, L)
        for a, b in ((sb.Adiag, s0.Adiag), (sb.B, s0.B), (sb.Aoff, s0.Aoff)):
            assert np.array_equal(_bits(a), _bits(b))
        assert np.abs(s0.x - sb.x).max() <= 1e-12 * max(1.0, np.abs(sb.x).max())
        h.set_states(h.l_points())
        h.relinearize_poses(P)
        s1 = ic.snapshot(h, L)
        for a, b in ((s0.Adiag, s1.Adiag), (s0.B, s1.B), (s0.Aoff, s1.Aoff), (s0.y, s1.y), (s0.x, s1.x)):
            assert np.array_equal(_bits(a), _bits(b))
        for k in s0.fronts:
            assert np.array_equal(_bits(s0.fronts[k][0]), _bits(s1.fronts[k][0]))
            assert np.array_equal(_bits(s0.fronts[k][1]), _bits(s1.fronts[k][1]))


def test_relin_repeat_same_bits(m3500):
    """The same relinearisation on two copies from the same states rebuilds its dirty entries to the same bits (no
    atomics; the batch before it may differ in the last bits elsewhere)."""
    L = ic.dev_api()
    d = m3500.head(300)
    with H.Harness("b200", nthreshold=1 << 30) as a, H.Harness("b200", nthreshold=1 << 30) as b:
        P = list(range(0, 300, 7))
        for h in (a, b):
            h.load_full(d)
            h.batch()
        _perturb(a, P, 0.02, 5)
        b.set_states(a.states())
        fs = fc.borrowed_plan(L, a.param_ptr()).array("fslot")
        _, D, dslot = rl.dirty_sets(P, *ic.factors_of(a)[:3], fs)
        for h in (a, b):
            h.relinearize_poses(P)
        sa, sb = ic.snapshot(a, L), ic.snapshot(b, L)
        assert np.array_equal(_bits(a.l_points()), _bits(b.l_points()))
        for x, y in ((sa.Adiag[D], sb.Adiag[D]), (sa.B[D], sb.B[D]), (sa.Aoff[dslot], sb.Aoff[dslot])):
            assert np.array_equal(_bits(x), _bits(y))


@pytest.mark.parametrize("world", ["integer", "m3500", "dense30k"])
def test_relin_everything_matches_batch(m3500, world):
    """Perturb the states and relinearise every pose: the states match a fresh copy's batch solve at those states, and
    so does chi2.  On an integer-valued system (poses moved by whole units) both Hessians are exact, so the two solves
    differ only in the factorisation's rounding: within 1e-12 relative.  Elsewhere the two Hessians are the same sums
    in other orders (fixed order here, the batch's atomics there); the rhs sums nearly cancel near an optimum, so their
    last-bit differences reach x amplified by the condition number: measured 2.4e-12 (M3500) and 7.2e-12 (30 k world)
    of the largest state after four batch solves from the initial guess; the bound is 1e-10.  On the 30 k world the
    tables (about 2F + slots entries) exceed half the pinned staging buffer and go up by direct copy, into device
    buffers grown for them."""
    with H.Harness("b200", nthreshold=1 << 30) as h, H.Harness("b200") as g:
        tol = 1e-10
        if world == "integer":
            h.set_tikhanov(0.5)
            g.set_tikhanov(0.5)
            _integer_graph(h)
            tol = 1e-12
        elif world == "m3500":
            d = m3500.head(1000)
            h.replay_begin(d)
            h.replay_to(d.n_nodes, want_chi2=False)
        else:
            d = datasets.manhattan_dense(30000, seed=2)
            h.load_full(d)
            h.set_states(d.truth)
        h.batch()
        h.batch()
        N = h.n_nodes
        h.relinearize_poses([N - 1])  # small tables first: the buffers grow at the big call
        if world == "integer":  # grid points moved by whole units: every Hessian entry stays an integer
            st = np.array([[i % 8, i // 8, 0.0] for i in range(N)])
            st[::3, 0] += 1.0
            st[1::4, 1] -= 1.0
            h.set_states(st)
        else:
            _perturb(h, list(range(N)), 1e-5, 6)
        st = h.states()
        h.relinearize_poses(np.arange(N))
        assert np.array_equal(_bits(h.l_points()), _bits(st))
        _copy_graph(h, g)
        g.set_states(h.l_points())
        g.batch()
        ref = g.states()
        assert np.abs(h.states() - ref).max() <= tol * max(1.0, np.abs(ref).max())
        want = fc.chi2_ref(*ic.factors_of(h), h.states())
        assert abs(h.chi2() - float(want)) <= CHI2_TOL * float(want)
        assert abs(h.chi2() - g.chi2()) <= CHI2_TOL * g.chi2()


# ---------------------------------------------------------------------------------------------
# the queries after a relinearisation
# ---------------------------------------------------------------------------------------------
def test_queries_after_relin(m3500):
    d = m3500.head(120)
    with H.Harness("b200") as h:
        with RelinChecker(h) as chk:
            h.replay_begin(d)
            chk.batch(lambda: h.replay_to(1))
            for k in range(1, d.n_nodes):
                chk.step(lambda: h.replay_to(k + 1))
            N = h.n_nodes
            _perturb(h, [5, 40, N - 1], 0.02, 8)
            chk.relin([5, 40, N - 1])
            plan = fc.borrowed_plan(chk.L, h.param_ptr())
            A, _ = chk.ledger.dense_ld(N, plan.info()["n_slots"], plan.array("fslot"), plan.array("node2q"))
            Sig = np.linalg.inv(A.astype(np.float64))
            ids = [0, 5, 40, N // 2, N - 1]
            got = h.marginal_covariance(ids)
            I = np.concatenate([3 * p + np.arange(3) for p in ids])
            want = Sig[np.ix_(I, I)]
            assert np.abs(got - want).max() <= 1e-8 * np.abs(want).max()
            a, b = np.array([N - 1, 40]), np.array([5, -1])
            z = np.array([[0.1, 0.2, 0.05], [0.0, 0.1, 0.0]])
            W = np.array([np.diag([50.0, 50.0, 20.0]).reshape(9)] * 2)
            d2, cov = h.candidate_mahalanobis(a, b, z, W, with_cov=True)
            st, lp = h.states(), h.l_points()
            for c in range(2):
                ia = slice(3 * a[c], 3 * a[c] + 3)
                if b[c] < 0:
                    Srel = Sig[ia, ia]
                    r = z[c] - st[a[c]]
                    r[2] = ((r[2] + np.pi) % (2 * np.pi)) - np.pi
                else:
                    Ja, Jb, _ = emul.xyt_eval(lp[a[c]], lp[b[c]], z[c])
                    J = np.c_[Ja, Jb]
                    idx = np.r_[3 * a[c] + np.arange(3), 3 * b[c] + np.arange(3)]
                    Srel = J @ Sig[np.ix_(idx, idx)] @ J.T
                    _, _, r = emul.xyt_eval(st[a[c]], st[b[c]], z[c])
                assert np.abs(cov[c] - Srel).max() <= 1e-8 * np.abs(Srel).max()
                S = Srel + np.linalg.inv(W[c].reshape(3, 3))
                assert abs(d2[c] - r @ np.linalg.solve(S, r)) <= 1e-8 * max(1.0, abs(d2[c]))


# ---------------------------------------------------------------------------------------------
# errors: -1, the message, nothing changed
# ---------------------------------------------------------------------------------------------
def _relin_state(h, L):
    s = _state(h, L)
    s.update(lp=h.l_points().copy(), lin=h.linearized_nodes().tolist())
    return s


def _expect_error(h, L, ids, words):
    s0 = _relin_state(h, L)
    with pytest.raises(RuntimeError) as e:
        h.relinearize_poses(ids)
    assert all(w in str(e.value) for w in words), str(e.value)
    s1 = _relin_state(h, L)
    _same(s0, s1)
    assert np.array_equal(_bits(s0["lp"]), _bits(s1["lp"])) and s0["lin"] == s1["lin"]


def test_errors_change_nothing(m3500):
    L = ic.dev_api()
    d = m3500.head(80)
    with H.Harness("b200") as h:
        h.replay_begin(d)
        h.replay_to(60)
        N = h.n_nodes
        _perturb(h, [3, 4], 0.01, 9)
        _expect_error(h, L, [], ["n < 1"])
        _expect_error(h, L, [N], ["not in [0", "entry 0"])
        _expect_error(h, L, [2, -1], ["not in [0", "entry 1"])
        _expect_error(h, L, [4, 7, 4], ["twice", "entry 2"])
        # poses or factors added since the last solve
        h.add_node(h.states()[-1] + [1, 0, 0])
        h.add_xyt(N - 1, N, [1, 0, 0], [10, 0, 0, 0, 10, 0, 0, 0, 5])
        _expect_error(h, L, [3], ["added since the last solve"])
        h.inc()
        # an edited factor on a dirty pose (a neighbour's factor, not in R), re-checked by chi2
        f = next(i for i in range(h.n_factors) if h.factor(i)[1:3] == (20, 21))
        _, _, _, z2, W2 = h.factor(f)
        h.set_factor(f, z2 + 0.01, W2)
        h.chi2()
        _expect_error(h, L, [19], ["factor %d" % f, "edited"])
        fs = fc.borrowed_plan(L, h.param_ptr()).array("fslot")
        far = next(p for p in range(h.n_nodes - 1, 0, -1)
                   if not {20, 21} & set(rl.dirty_sets([p], *ic.factors_of(h)[:3], fs)[1].tolist()))
        h.relinearize_poses([far])  # away from the edit: fine
        h.batch()
        h.relinearize_poses([19])
        # a replaced factor
        t, a, b, z, W = h.factor(10)
        h.replace_xyt(10, a, b + 1 if b + 1 < h.n_nodes else b - 2, z, W)
        h.chi2()
        _expect_error(h, L, [3], ["replaced"])
        # a dropped plan
        h.invalidate_plan()
        _expect_error(h, L, [3], ["invalidate_plan"])
        h.batch()
        h.relinearize_poses([3])
        assert np.all(np.isfinite(h.states()))


def test_never_solved_and_other_params(m3500):
    L = ic.dev_api()
    d = m3500.head(100)
    with H.Harness("b200") as h:
        h.load_full(d)
        with pytest.raises(RuntimeError, match="does not continue a solve"):
            h.relinearize_poses([3])
        h.batch()
        other = h.new_param()
        mine = h.swap_param(other)
        h.batch()
        h.swap_param(mine)
        _perturb(h, [7], 0.01, 10)
        h.relinearize_poses([7])
        h.swap_param(other)
        st0 = h.states()
        h.add_node(st0[-1] + [1, 0, 0])
        h.add_xyt(d.n_nodes - 1, d.n_nodes, [1, 0, 0], [10, 0, 0, 0, 10, 0, 0, 0, 5])
        h.inc()
        assert "relinearised in place through another param" in h.last_error()
        assert "removed" not in h.last_error()
        assert np.array_equal(_bits(h.states()[:-1]), _bits(st0))
        with pytest.raises(RuntimeError, match="relinearised in place through another param"):
            h.marginal_covariance([1])
        with pytest.raises(RuntimeError, match="relinearised in place through another param"):
            h.relinearize_poses([1])
        with pytest.raises(RuntimeError, match="relinearised in place through another param"):
            h.remove_factors([1])
        h.batch()  # re-plans
        h.marginal_covariance([1])
        h.relinearize_poses([1])
        h.swap_param(mine)
        h.free_param(other)
        s0 = _relin_state(h, L)
        with pytest.raises(RuntimeError, match="relinearised in place through another param"):
            h.relinearize_poses([1])
        _same(s0, _relin_state(h, L))
