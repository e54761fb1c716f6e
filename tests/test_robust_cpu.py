"""Robust loop-closure factors on the host (-m "not gpu"): construction and validation, the eval / state_eval hooks
against a numpy formula, copy, the ".graph" round trip, april_graph_dof and the replay CLI's --robust argument.

A robust factor (type 32) is an xyt factor whose information matrix is weighted by an M-estimator at
s = r'Wr:  Huber w = 1 if s <= k^2 else k / sqrt(s), rho = s or 2 k sqrt(s) - k^2;
           Cauchy w = 1 / (1 + s / k^2), rho = k^2 log1p(s / k^2).
"""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from aprilsam_b200 import capi
from aprilsam_b200 import harness as H
from conftest import ROOT
from support import emul

HUBER, CAUCHY = H.Harness.HUBER, H.Harness.CAUCHY
ROBUST_TYPE = 32
W0 = np.array([[40.0, 3.0, 1.0], [3.0, 25.0, -2.0], [1.0, -2.0, 90.0]])


def last_error() -> str:
    return capi.lib().aprilsam_b200_last_error().decode()


def factor_loss(h, idx):
    loss, k = C.c_int(), C.c_double()
    t = capi.lib().asam_dbg_factor_loss(C.c_void_p(h.graph_ptr()), idx, C.byref(loss), C.byref(k))
    return t, loss.value, k.value


def xyt_residual(pa, pb, z):
    ca, sa = math.cos(pa[2]), math.sin(pa[2])
    dx, dy = pb[0] - pa[0], pb[1] - pa[1]
    return np.array([z[0] - (ca * dx + sa * dy), z[1] - (-sa * dx + ca * dy),
                     float(emul.mod2pi(np.array([z[2] - (pb[2] - pa[2])]))[0])])


def loss_ref(loss, k, s):
    """(w, rho) in float64, the formulas of the factor's documentation."""
    k2 = k * k
    if loss == HUBER:
        return (1.0, s) if s <= k2 else (k / math.sqrt(s), 2.0 * k * math.sqrt(s) - k2)
    return 1.0 / (1.0 + s / k2), k2 * math.log1p(s / k2)


def two_poses(pa=(0.0, 0.0, 0.3), pb=(2.0, 1.0, 0.9)):
    h = H.Harness("b200")
    h.add_node(np.array(pa))
    h.add_node(np.array(pb))
    return h


@pytest.mark.parametrize("loss,k", [(0, 1.0), (3, 1.0), (-1, 1.0), (HUBER, 0.0), (HUBER, -2.0), (CAUCHY, math.nan),
                                    (CAUCHY, math.inf), (HUBER, -math.inf)])
def test_create_rejects_invalid_loss(built, loss, k):
    with two_poses() as h:
        assert h.add_xyt_robust(0, 1, [1, 0, 0], W0, loss, k) == -1
        assert h.n_factors == 0
        assert "robust loss" in last_error()


def test_set_loss_validates(built):
    with two_poses() as h:
        plain = h.add_xyt(0, 1, [1, 0, 0], W0)
        rob = h.add_xyt_robust(0, 1, [1, 0, 0], W0, HUBER, 2.0)
        assert h.set_loss(plain, CAUCHY, 1.0) == -1
        assert "no robust loss" in last_error()
        for loss, k in ((0, 1.0), (3, 1.0), (HUBER, 0.0), (CAUCHY, math.nan), (CAUCHY, math.inf), (HUBER, -1.0)):
            assert h.set_loss(rob, loss, k) == -1, (loss, k)
            assert last_error()
            assert factor_loss(h, rob) == (ROBUST_TYPE, HUBER, 2.0)  # a rejected edit changes nothing
        assert h.set_loss(rob, CAUCHY, 0.25) == 0
        assert factor_loss(h, rob) == (ROBUST_TYPE, CAUCHY, 0.25)
        assert factor_loss(h, plain) == (1, 0, 0.0)


@pytest.mark.parametrize("loss", [HUBER, CAUCHY])
def test_eval_hooks_match_numpy(built, loss):
    """eval (l_point) and state_eval (state): xyt r and J, W_eff = w W, chi2 = rho(s); s on both sides of k^2."""
    pa, pb = np.array([0.1, -0.2, 0.3]), np.array([2.0, 1.0, 0.9])
    z = np.array([1.9, -0.4, 0.5])
    with two_poses(pa, pb) as h:
        r = xyt_residual(pa, pb, z)
        s = float(r @ W0 @ r)
        plain = h.add_xyt(0, 1, z, W0)
        for k in (0.1 * math.sqrt(s), 10.0 * math.sqrt(s), 1e100):
            idx = h.add_xyt_robust(0, 1, z, W0, loss, k)
            w, rho = loss_ref(loss, k, s)
            rp, Jap, Jbp, Wp, chi2p = h.eval(plain)
            for at_state in (False, True):
                rr, Ja, Jb, W, chi2 = h.eval(idx, at_state)
                np.testing.assert_array_equal(rr, rp)
                np.testing.assert_array_equal(Ja, Jap)
                np.testing.assert_array_equal(Jb, Jbp)
                np.testing.assert_allclose(rr, r, rtol=1e-14, atol=1e-15)
                np.testing.assert_allclose(W, w * W0, rtol=1e-14)
                assert chi2 == pytest.approx(rho, rel=1e-13)
            if k == 1e100:  # inactive loss: the plain factor bit for bit (Cauchy: w within an ulp)
                if loss == HUBER:
                    assert np.array_equal(W, Wp) and chi2 == chi2p
                else:
                    assert chi2 == pytest.approx(chi2p, rel=1e-14)
        # state_eval follows the states, eval the linearisation points
        h.set_states(np.array([pa, pb + [0.5, 0.0, 0.0]]))
        r2 = xyt_residual(pa, pb + [0.5, 0, 0], z)
        s2 = float(r2 @ W0 @ r2)
        idx = h.add_xyt_robust(0, 1, z, W0, loss, 0.5)
        assert h.eval(idx, True)[4] == pytest.approx(loss_ref(loss, 0.5, s2)[1], rel=1e-13)
        assert h.eval(idx, False)[4] == pytest.approx(loss_ref(loss, 0.5, s)[1], rel=1e-13)


def test_nan_residual_gives_nan_weight(built):
    with two_poses() as h:
        idx = h.add_xyt_robust(0, 1, [math.nan, 0, 0], W0, HUBER, 1.0)
        _, _, _, W, chi2 = h.eval(idx)
        assert np.isnan(W).all() and math.isnan(chi2)


@pytest.mark.parametrize("loss", [HUBER, CAUCHY])
def test_copy_duplicates_the_loss(built, loss):
    with two_poses() as h:
        idx = h.add_xyt_robust(0, 1, [1.5, 0.2, 0.1], W0, loss, 0.75)
        h.attr_put(h.FACTOR, idx, "type", "scan")
        c = h.copy_factor(idx)
        assert factor_loss(h, c) == (ROBUST_TYPE, loss, 0.75)
        t, a, b, z, W = h.factor(c)
        assert (t, a, b) == (ROBUST_TYPE, 0, 1)
        assert np.array_equal(z, [1.5, 0.2, 0.1]) and np.array_equal(W, W0.reshape(9))
        assert h.attr_get(h.FACTOR, c, "type") == "scan"
        for at_state in (False, True):
            e0, e1 = h.eval(idx, at_state), h.eval(c, at_state)
            assert all(np.array_equal(x, y) for x, y in zip(e0, e1))
        # the copy owns its loss: editing one leaves the other alone
        assert h.set_loss(c, HUBER if loss == CAUCHY else CAUCHY, 3.0) == 0
        assert factor_loss(h, idx) == (ROBUST_TYPE, loss, 0.75)


def test_graph_file_round_trip(built, tmp_path):
    rng = np.random.default_rng(7)
    path = str(tmp_path / "robust.graph")
    with H.Harness("b200") as h:
        for i in range(5):
            h.add_node(rng.standard_normal(3))
        h.add_xytpos(0, [0, 0, 0], np.diag([1e4, 1e4, 1e3]))
        want = []
        for i, (a, b, loss, k) in enumerate([(0, 1, 0, 0), (1, 3, HUBER, 0.1 + rng.random()),
                                             (4, 2, CAUCHY, 1e-3 * rng.random()), (3, 4, 0, 0), (0, 4, HUBER, 1e100)]):
            z = rng.standard_normal(3)
            M = rng.standard_normal((3, 3))
            W = M @ M.T + np.eye(3)
            idx = h.add_xyt(a, b, z, W) if loss == 0 else h.add_xyt_robust(a, b, z, W, loss, k)
            want.append((idx, a, b, z, W.reshape(9), loss, k))
        assert h.save(path)
        with H.Harness("b200") as g:
            assert g.load(path) == 5
            assert g.n_factors == h.n_factors == 6
            assert g.dof() == h.dof()
            for idx, a, b, z, W, loss, k in want:
                t, ga, gb, gz, gW = g.factor(idx)
                assert (t, ga, gb) == ((ROBUST_TYPE if loss else 1), a, b)
                assert gz.tobytes() == z.tobytes() and gW.tobytes() == W.tobytes()
                assert factor_loss(g, idx) == ((ROBUST_TYPE if loss else 1), loss, k)
            assert factor_loss(g, 0)[0] == 2


def test_dof_counts_robust_factors(built):
    with two_poses() as h:
        h.add_node(np.zeros(3))
        h.add_xytpos(0, [0, 0, 0], np.eye(3))
        assert h.dof() == 3 - 9
        h.add_xyt_robust(0, 1, [1, 0, 0], W0, CAUCHY, 1.0)
        h.add_xyt(1, 2, [1, 0, 0], W0)
        h.add_xyt_robust(0, 2, [1, 0, 0], W0, HUBER, 1.0)
        assert h.dof() == 12 - 9


@pytest.mark.parametrize("arg", ["huber", "huber:", "huber:0", "cauchy:-1", "cauchy:nan", "huber:inf",
                                 "tukey:1", "huber:1x", "Huber:1", ":1", None])
def test_replay_cli_rejects_malformed_robust(built, arg):
    cli = os.path.join(ROOT, "examples", "_build", "asam_replay")
    cmd = [cli, "--datapath", "unused.txt", "--robust"] + ([arg] if arg is not None else [])
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=60)
    assert p.returncode == 2
    assert "--robust expects huber:K or cauchy:K" in p.stderr
