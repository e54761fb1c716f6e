"""Robust loop-closure factors (type 32) on the GPU: k_linearize / k_step weight W by the loss at every linearisation,
k_chi2_partial sums 0.5 rho(s).

  1. an inactive loss (k = 1e100: w = 1, rho = s) reproduces the plain graph: batch iterations (states, chi2, the
     Hessian in HBM) and a 400-step replay (states, naffected, escalations) -- the type 1 / 2 paths and the incremental
     machinery are unchanged;
  2. the Hessian against float64 (frontcheck.linearize_ref fed W pre-weighted in numpy), s on both sides of k^2;
  3. IRLS batch iterations on M3500 with 50 false closures against the float64 oracle port step with numpy weights;
  4. incremental steps against a ledger in which each robust factor is weighted at the points of the step that added
     it and re-weighted at every batch; the {loss, k} records in HBM against the host;
  5. aprilsam_b200_factor_set_loss between calls;
  6. a sharded two-GPU batch solve with robust factors against the single-GPU solve.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from aprilsam_b200 import capi
from aprilsam_b200 import harness as H
from conftest import ROOT
from oracle import port
from support import emul
from support import frontcheck as fc
from support import inccheck as ic

pytestmark = pytest.mark.gpu

HUBER, CAUCHY = H.Harness.HUBER, H.Harness.CAUCHY
LAM = 1e-4
LINEARIZE_C = 200.0  # as tests/test_gpu_kernels.py
FLOSS = 10           # ASAM_DBG_BUF_FLOSS


# ---------------------------------------------------------------------------------------------
# float64 references
# ---------------------------------------------------------------------------------------------
def xyt_s(z, W, pa, pb):
    """s = r'Wr per factor, r the xyt residual at (pa, pb); W (F, 9).  X = W r first, like the kernels."""
    ca, sa = np.cos(pa[:, 2]), np.sin(pa[:, 2])
    dx, dy = pb[:, 0] - pa[:, 0], pb[:, 1] - pa[:, 1]
    r = np.c_[z[:, 0] - (ca * dx + sa * dy), z[:, 1] - (-sa * dx + ca * dy), emul.mod2pi(z[:, 2] - (pb[:, 2] - pa[:, 2]))]
    X = np.einsum("fij,fj->fi", W.reshape(-1, 3, 3), r)
    return r[:, 0] * X[:, 0] + r[:, 1] * X[:, 1] + r[:, 2] * X[:, 2]


def weight(loss, k, s):
    k2 = k * k
    return np.where(loss == HUBER, np.where(s <= k2, 1.0, k / np.sqrt(s)), 1.0 / (1.0 + s / k2))


def rho(loss, k, s):
    k2 = k * k
    return np.where(loss == HUBER, np.where(s <= k2, s, 2.0 * k * np.sqrt(s) - k2), k2 * np.log1p(s / k2))


def scans(d):
    return np.abs(d.ea - d.eb) != 1


def with_outliers(m, n_out=50, seed=50, span=100):
    """m plus n_out seeded false closures between poses more than `span` apart (z up to 10 m / any angle off, W of a
    real closure)."""
    rng = np.random.default_rng(seed)
    a = rng.integers(0, m.n_nodes, 8 * n_out)
    b = rng.integers(0, m.n_nodes, 8 * n_out)
    ok = np.abs(a - b) > span
    a, b = a[ok][:n_out], b[ok][:n_out]
    z = np.c_[rng.uniform(-10, 10, n_out), rng.uniform(-10, 10, n_out), rng.uniform(-np.pi, np.pi, n_out)]
    W = m.eW[rng.choice(np.nonzero(scans(m))[0], n_out)]
    return H.PoseGraphData(m.init, np.r_[m.ea, a].astype(np.int32), np.r_[m.eb, b].astype(np.int32),
                           np.r_[m.ez, z], np.r_[m.eW, W])


def reweighted(d, loss, k, st):
    """d with the W of every scan edge multiplied by its IRLS weight at the states st (plain for loss 0)."""
    if not loss:
        return d
    w = np.where(scans(d), weight(loss, k, xyt_s(d.ez, d.eW, st[d.ea], st[d.eb])), 1.0)
    return H.PoseGraphData(d.init, d.ea, d.eb, d.ez, d.eW * w[:, None])


def state_err(a, b):
    e = a - b
    e[:, 2] = emul.mod2pi(e[:, 2])
    return np.abs(e)


# ---------------------------------------------------------------------------------------------
# what is in HBM
# ---------------------------------------------------------------------------------------------
def hessian(h, L):
    """(Adiag, Aoff, B) as one float64 vector."""
    snap = ic.snapshot(h, L, which=[])
    return np.r_[snap.Adiag.ravel(), snap.Aoff.ravel(), snap.B.ravel()]


def hessian_spread(h, L):
    """Per entry of hessian(h): 8 u times the sum of the absolute values of its contributions with the plain W
    (w <= 1 for every loss).  k_linearize adds the contributions with floating-point atomics, whose order follows the
    timing of the warps; two runs that differ in that order agree within this bound."""
    snap = ic.snapshot(h, L, which=[])
    ftype, fa, fb, fz, fW = fc.factors_of(h)
    N, S = len(snap.Adiag), len(snap.Aoff)
    _, AdA, _, BA, (_, _, _, HA) = fc.linearize_ref(N, ftype, fa, fb, fz, fW, h.l_points(), None, LAM)
    AoA = np.zeros((S, 3, 3))
    e = ftype == 1
    np.add.at(AoA, snap.plan.array("fslot")[:len(ftype)][e], HA)
    return 8 * fc.U * np.r_[AdA.ravel(), AoA.ravel(), BA.ravel()] + np.finfo(float).tiny


def rel_state_diff(a, b):
    return float(state_err(a, b).max() / max(1.0, np.abs(b).max()))


def factor_losses(h, first=0):
    L = capi.lib()
    F = h.n_factors - first
    loss, k = np.zeros(F, np.int32), np.zeros(F)
    lo, kk = C.c_int(), C.c_double()
    for i in range(F):
        L.asam_dbg_factor_loss(C.c_void_p(h.graph_ptr()), first + i, C.byref(lo), C.byref(kk))
        loss[i], k[i] = lo.value, kk.value
    return loss, k


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


# ---------------------------------------------------------------------------------------------
# 1. an inactive loss is the plain factor
# ---------------------------------------------------------------------------------------------
# With k = 1e100 the weight is exactly 1 (Huber: s <= k^2; Cauchy: 1 + s/k^2 rounds to 1), so every robust lane feeds
# the same values as a plain lane.  The sums are still formed by floating-point atomics in warp-timing order, and the
# robust lanes take a little longer, so the comparison allows that reordering and no more; the runs print how many
# entries / steps came out bit for bit.
@pytest.mark.parametrize("loss", [HUBER, CAUCHY])
def test_inactive_loss_batch_matches_plain(m3500, loss):
    L = fc.dev_api()
    with H.Harness("b200") as p, H.Harness("b200") as r:
        p.load_full(m3500)
        r.set_scan_loss(loss, 1e100)
        r.load_full(m3500)
        rl, _ = factor_losses(r)
        assert (rl[1:] == np.where(scans(m3500), loss, 0)).all() and rl[1:].any()
        same = []
        for it in range(6):
            r.set_states(p.states())  # each iteration from the same point: rounding does not carry over
            p.batch()
            r.batch()
            Hp, Hr = hessian(p, L), hessian(r, L)
            bad = np.abs(Hr - Hp) > hessian_spread(p, L)
            assert not bad.any(), ("Hessian", it, int(bad.sum()))
            same.append(int(np.count_nonzero(bits(Hr) == bits(Hp))))
            assert rel_state_diff(r.states(), p.states()) < 1e-6, ("states", it)
            r.set_states(p.states())
            cp, cr = p.chi2(), r.chi2()  # k_chi2_partial / k_chi2_final reduce in a fixed order
            assert (cr == cp) if loss == HUBER else cr == pytest.approx(cp, rel=1e-14), ("chi2", it, cp, cr)
        print(f"ROBUSTCHECK inactive batch loss {loss}: Hessian entries bit-identical per iteration {same} of {len(Hp)}")


def test_inactive_loss_replay_matches_plain(m3500):
    """400 steps in lock step: states, naffected and the other tree counters, escalations; through k_step."""
    L = ic.dev_api()
    d = m3500.head(400)
    with H.Harness("b200") as p, H.Harness("b200") as r:
        r.set_scan_loss(HUBER, 1e100)
        p.replay_begin(d)
        r.replay_begin(d)
        small0 = None
        nbits = 0
        for k in range(d.n_nodes):
            out = []
            for h in (p, r):
                nb0 = ic.batch_count(L)
                chi2, _, info = h.replay_to(k + 1)
                out.append((h.states(), chi2[-1], info[-1].copy(), ic.batch_count(L) - nb0))
            (sp, cp, ip, bp), (sr, cr, ir, br) = out
            nbits += int(np.array_equal(bits(sr), bits(sp)))
            assert rel_state_diff(sr, sp) < 1e-8, ("states", k)
            # states may differ in the last bits (summation order), and chi2 follows them to first order
            assert cr == pytest.approx(cp, rel=1e-9), ("chi2", k)
            assert np.array_equal(ip, ir) and bp == br, ("tree / escalation", k, ip, ir, bp, br)
            if k == 0:
                small0 = capi.lib().asam_small_steps(L.asam_dbg_dev_of_graph(r.graph_ptr()))
        assert factor_losses(r)[0].any()
        small = capi.lib().asam_small_steps(L.asam_dbg_dev_of_graph(r.graph_ptr()))
        print(f"ROBUSTCHECK inactive replay: states bit-identical after {nbits} of {d.n_nodes} steps; "
              f"{small - small0} k_step launches")
        assert small > small0 + 50, (small0, small)


# ---------------------------------------------------------------------------------------------
# 2. the Hessian and chi2 against float64
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("loss", [HUBER, CAUCHY])
def test_robust_hessian_and_chi2_against_float64(m3500, loss):
    d = with_outliers(m3500.head(300), n_out=10, span=30)
    sc = scans(d)
    s0 = xyt_s(d.ez, d.eW, d.init[d.ea], d.init[d.eb])[sc]
    k = float(np.sqrt(np.median(s0)))  # s on both sides of k^2, across many decades
    assert (s0 < k * k).sum() > 20 and (s0 > k * k).sum() > 20 and s0.max() / s0.min() > 1e6
    with H.Harness("b200") as h:
        h.set_scan_loss(loss, k)
        h.load_full(d)
        h.batch()
        L = fc.dev_api()
        snap = fc.snapshot(h, L)
        ftype, fa, fb, fz, fW = fc.factors_of(h)
        lp = h.l_points()
        floss, fk = factor_losses(h)
        rob = floss != 0
        assert rob.sum() == sc.sum()
        fWe = fW.copy()
        fWe[rob] *= weight(floss[rob], fk[rob], xyt_s(fz[rob], fW[rob], lp[fa[rob]], lp[fb[rob]]))[:, None]
        lin = fc.check_linearize(snap, ftype, fa, fb, fz, fWe, lp, snap.plan.array("fslot"), LAM)
        print(f"ROBUSTCHECK linearize loss {loss}: {lin:.2f}")
        assert lin < LINEARIZE_C, lin
        # the plain formula must NOT pass: the weights are really applied
        assert fc.check_linearize(snap, ftype, fa, fb, fz, fW, lp, snap.plan.array("fslot"), LAM) > 1e6
        st = h.states()
        e = ftype == 1
        s = xyt_s(fz[e], fW[e], st[fa[e]], st[fb[e]])
        c, re_ = s.copy(), rob[e]
        c[re_] = rho(floss[e][re_], fk[e][re_], s[re_])
        want = float(fc.chi2_ref(ftype[~e], fa[~e], fb[~e], fz[~e], fW[~e], st)) + 0.5 * float(np.sum(c))
        assert h.chi2() == pytest.approx(want, rel=1e-12)


# ---------------------------------------------------------------------------------------------
# 3. IRLS batch iterations
# ---------------------------------------------------------------------------------------------
_CLEAN = {}


def clean_solution(m):
    """M3500 solved on the CPU in float64 (30 oracle-port Gauss-Newton steps from the VERTEX2 poses)."""
    if "m" not in _CLEAN:
        st = m.init.copy()
        for _ in range(30):
            st = port.batch_step(m, st, LAM)
        _CLEAN["m"] = st
    return _CLEAN["m"]


# RMS position distance (m) of the state after 6 iterations from the clean solution, by the float64 oracle port on
# the CPU (k = 0.5; inliers have s <= 0.21 at the clean solution; the GPU run reproduces these to the printed digits):
#   plain 38.220, Huber 34.936, Cauchy 0.861.
# Huber bounds the pull of each false closure but does not remove it: 50 closures as precise as the real ones still
# bend the trajectory.  Cauchy all but ignores them.
END_RATIO = {HUBER: 0.95, CAUCHY: 0.05}


def rms_distance(st, clean):
    e = state_err(st, clean)
    return float(np.sqrt(np.mean(e[:, 0] ** 2 + e[:, 1] ** 2)))


@pytest.mark.parametrize("loss", [HUBER, CAUCHY])
def test_irls_batch_iterations(m3500, loss):
    if not port.available():
        pytest.skip("oracle port not built")
    clean = clean_solution(m3500)
    d = with_outliers(m3500)
    k = 0.5
    end = {}
    for arm in (0, loss):
        with H.Harness("b200") as h:
            h.set_scan_loss(arm, k)
            h.load_full(d)
            h.set_states(clean)
            worst = 0.0
            for it in range(6):
                st0 = h.states()
                want = port.batch_step(reweighted(d, arm, k, st0), st0, LAM)
                h.batch()
                err = state_err(h.states(), want).max() / max(1.0, np.abs(want).max())
                worst = max(worst, err)
                assert err < 1e-6, (arm, it, err)
            end[arm] = rms_distance(h.states(), clean)
            print(f"ROBUSTCHECK irls loss {arm}: worst step error {worst:.2e}, end distance {end[arm]:.3f}")
    assert end[loss] < END_RATIO[loss] * end[0], end


# ---------------------------------------------------------------------------------------------
# 4. incremental steps
# ---------------------------------------------------------------------------------------------
class RobustLedger(ic.Ledger):
    """inccheck.Ledger with each robust factor's W weighted at its own points: at the batch that (re)linearised it,
    or at the step that added it."""

    def __init__(self, lam):
        super().__init__(lam)
        self.loss, self.k = np.zeros(0, np.int32), np.zeros(0)

    def _weigh(self, first):
        rob = np.nonzero(self.loss[first:] != 0)[0] + first
        p = self.pts[rob]
        self.fW[rob] *= weight(self.loss[rob], self.k[rob], xyt_s(self.fz[rob], self.fW[rob], p[:, :3], p[:, 3:]))[:, None]

    def batch(self, h):
        super().batch(h)
        self.loss, self.k = factor_losses(h)
        self._weigh(0)

    def add(self, h, lp, st):
        first = len(self.ft)
        super().add(h, lp, st)
        lo, kk = factor_losses(h, first)
        self.loss, self.k = np.r_[self.loss, lo], np.r_[self.k, kk]
        self._weigh(first)


@pytest.mark.parametrize("loss", [HUBER, CAUCHY])
def test_incremental_steps_weigh_at_their_points(m3500, loss):
    d = with_outliers(m3500.head(300), n_out=12, span=30)
    L = ic.dev_api()
    kinds = {}
    with H.Harness("b200") as h, ic.recording(L):
        h.set_scan_loss(loss, 0.5)
        h.replay_begin(d)
        led = RobustLedger(LAM)
        worst = 0.0
        for k in range(d.n_nodes):
            N0 = h.n_nodes
            st0 = h.states()
            nb0 = ic.batch_count(L)
            h.replay_to(k + 1, want_chi2=False)
            escalated = k == 0 or ic.batch_count(L) > nb0
            if escalated:
                led.batch(h)
                kinds["batch"] = kinds.get("batch", 0) + 1
            else:
                rec = ic.last_step(L, h.param_ptr())
                kinds[rec["kind"]] = kinds.get(rec["kind"], 0) + 1
                led.add(h, h.l_points(), np.r_[st0, h.l_points()[N0:]])
            snap = ic.snapshot(h, L, which=[])
            lin = led.check(snap, snap.plan.array("fslot"))
            worst = max(worst, lin)
            assert lin < LINEARIZE_C, (k, lin)
            F = h.n_factors
            if not led.loss.any():  # no robust factor yet: the context has no {loss, k} records
                continue
            dev = L.asam_dbg_dev_of_graph(h.graph_ptr())
            rec16 = np.zeros(2 * F)
            fc._ok(L, L.asam_debug_read_buffer(dev, FLOSS, 0, rec16.nbytes, rec16.ctypes.data_as(C.c_void_p)), "FLOSS")
            rob = led.loss != 0
            dev_rec = rec16.reshape(F, 2)[rob]
            assert np.array_equal(bits(dev_rec), bits(np.c_[led.loss[rob].astype(np.float64), led.k[rob]])), k
        print(f"ROBUSTCHECK incremental loss {loss}: worst {worst:.2f}, steps {kinds}")
    assert kinds.get("k_step", 0) > 20, kinds
    assert sum(v for key, v in kinds.items() if key not in ("k_step", "batch")) > 5, kinds


# ---------------------------------------------------------------------------------------------
# 5. edits of the loss
# ---------------------------------------------------------------------------------------------
def test_set_loss_between_batch_calls(m3500):
    d = with_outliers(m3500.head(600), n_out=15, span=50)
    L = fc.dev_api()
    with H.Harness("b200") as a, H.Harness("b200") as b:
        a.set_scan_loss(HUBER, 0.5)
        a.load_full(d)
        for _ in range(2):
            a.batch()
        rob = np.nonzero(factor_losses(a)[0])[0]
        for i in rob:
            assert a.set_loss(int(i), CAUCHY, 0.25) == 0
        st = a.states()
        b.set_scan_loss(CAUCHY, 0.25)
        b.load_full(d)
        b.set_states(st)
        for h in (a, b):
            h.batch()
        bad = np.abs(hessian(a, L) - hessian(b, L)) > hessian_spread(b, L)
        assert not bad.any(), int(bad.sum())
        assert rel_state_diff(a.states(), b.states()) < 1e-8
        b.set_states(a.states())  # chi2 at the same states: the same edited loss
        assert a.chi2() == pytest.approx(b.chi2(), rel=1e-14)


def test_set_loss_between_incremental_steps_waits_for_the_batch(m3500):
    """An edit between incremental steps leaves the Hessian alone until the next batch re-weights every factor."""
    d = with_outliers(m3500.head(200), n_out=8, span=30)
    L = ic.dev_api()
    with H.Harness("b200", nthreshold=10 ** 9) as h:
        h.set_scan_loss(HUBER, 0.5)
        h.replay_begin(d)
        led = RobustLedger(LAM)
        h.replay_to(1)
        led.batch(h)
        for k in range(1, 150):
            N0, st0 = h.n_nodes, h.states()
            h.replay_to(k + 1, want_chi2=False)
            led.add(h, h.l_points(), np.r_[st0, h.l_points()[N0:]])
        rob = np.nonzero(led.loss)[0]
        assert len(rob) > 5
        for i in rob:
            assert h.set_loss(int(i), CAUCHY, 0.05) == 0
        N0, st0 = h.n_nodes, h.states()
        h.replay_to(151, want_chi2=False)  # an incremental step: old factors keep their Huber weights
        led.add(h, h.l_points(), np.r_[st0, h.l_points()[N0:]])
        snap = ic.snapshot(h, L, which=[])
        assert led.check(snap, snap.plan.array("fslot")) < LINEARIZE_C
        h.batch()  # the batch re-weights every factor with the edited loss
        led.batch(h)
        assert (led.loss[rob] == CAUCHY).all()
        snap = ic.snapshot(h, L, which=[])
        assert led.check(snap, snap.plan.array("fslot")) < LINEARIZE_C


# ---------------------------------------------------------------------------------------------
# 6. two GPUs
# ---------------------------------------------------------------------------------------------
def test_sharded_two_gpu_robust_solve_matches_single_gpu():
    if capi.lib().asam_device_count() < 2:
        pytest.skip("needs two GPUs")
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port_ = s.getsockname()[1]
    s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(port_), os.path.join(ROOT, "tools", "shard_check.py"), "--poses", "30000",
           "--iters", "3", "--robust", "cauchy:0.5"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-2000:])
    assert "RESULT world 2" in r.stdout
