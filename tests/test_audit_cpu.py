"""The maths of the factor audit (aprilsam_b200_factor_outlier_scores), no GPU.

  1. record maths: a numpy restatement of k_marginal_audit's per-record steps (N = W - W Sigma_rel W from its upper
     triangle, a 3 x 3 Cholesky of N, d2 = |L^-1 W r|^2, redundancy = 3 - tr(Sigma_rel W)) against a dense float64
     inverse, r' (W^-1 - Sigma_rel)^-1 r;
  2. the leave-one-out identity, exact in the linear model: on the M3500 system at the l_points, the audit d2 of a
     closure from Sigma = A^-1 and r_lin = r_e - J x equals the candidate d2 of the same closure against
     A_-f = A - J'WJ and r_loo = r_e - J x_-f, for plain and robust closures;
  3. the trace identity: sum_f (3 - redundancy_f) + lambda sum_i tr Sigma_ii = 3N, because tr(Sigma A) = 3N.
"""
from __future__ import annotations

import os

import numpy as np

from aprilsam_b200.harness import PoseGraphData

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAM = 1e-4
CHI2_3_999 = 16.27


def m3500_head(n):
    return PoseGraphData.load(os.path.join(ROOT, "tests", "golden", "m3500.npz")).head(n)


def wrap(t):
    return (t + np.pi) % (2 * np.pi) - np.pi


def xyt_eval(pa, pb, z):
    """r = z - h(a, b) (theta wrapped) and J = dh/d[a b] (3 x 6) of an xyt factor."""
    c, s = np.cos(pa[2]), np.sin(pa[2])
    dx, dy = pb[0] - pa[0], pb[1] - pa[1]
    h = np.array([c * dx + s * dy, -s * dx + c * dy, pb[2] - pa[2]])
    J = np.array([[-c, -s, -s * dx + c * dy, c, s, 0.0],
                  [s, -c, -c * dx - s * dy, -s, c, 0.0],
                  [0.0, 0.0, -1.0, 0.0, 0.0, 1.0]])
    r = z - h
    r[2] = wrap(r[2])
    return r, J


def system(d, pts, lam=LAM, weights=None):
    """A (3N x 3N) and g = sum J'W r_e of the graph's xyt factors at pts, plus lambda I; per factor (J, r_e, W_f)."""
    N = d.n_nodes
    A = lam * np.eye(3 * N)
    g = np.zeros(3 * N)
    recs = []
    for f in range(d.n_edges):
        a, b = int(d.ea[f]), int(d.eb[f])
        r, J = xyt_eval(pts[a], pts[b], d.ez[f])
        W = d.eW[f].reshape(3, 3) * (1.0 if weights is None else weights[f])
        idx = np.r_[3 * a:3 * a + 3, 3 * b:3 * b + 3]
        A[np.ix_(idx, idx)] += J.T @ W @ J
        g[idx] += J.T @ W @ r
        recs.append((idx, J, r, W))
    return A, g, recs


def audit_record(R, W, r):
    """k_marginal_audit's per-record maths, step by step in float64."""
    T = R @ W
    Nu = W - W @ T
    N = np.triu(Nu) + np.triu(Nu, 1).T
    u = W @ r
    L = np.linalg.cholesky(N)
    y = np.linalg.solve(L, u)
    return float(y @ y), 3.0 - float(np.trace(T))


def candidate_d2(R, W, r):
    return float(r @ np.linalg.solve(R + np.linalg.inv(W), r))


def closures(d, k, rng):
    far = np.flatnonzero(np.abs(d.eb - d.ea) > 1)
    return rng.choice(far, size=min(k, len(far)), replace=False)


def test_record_maths_against_dense_inverse():
    d = m3500_head(400)
    A, _, recs = system(d, d.init)
    Sig = np.linalg.inv(A)
    rng = np.random.default_rng(7)
    for f in closures(d, 40, rng):
        idx, J, r, W = recs[f]
        R = J @ Sig[np.ix_(idx, idx)] @ J.T
        R = (R + R.T) / 2
        d2, red = audit_record(R, W, r)
        ref = float(r @ np.linalg.solve(np.linalg.inv(W) - R, r))
        assert abs(d2 - ref) <= 1e-8 * max(1.0, abs(ref)), (f, d2, ref)
        assert 0.0 <= red <= 3.0 + 1e-12
        assert abs(red - (3.0 - np.trace(R @ W))) <= 1e-12


def _loo_check(d, weights, picks):
    # lambda = 1e-2 keeps A's condition number low enough that the float64 inverses on both sides hold 1e-9; the
    # identity itself holds for every lambda
    pts = d.init
    A, g, recs = system(d, pts, lam=1e-2, weights=weights)
    Sig = np.linalg.inv(A)
    x = Sig @ g
    worst = 0.0
    for f in picks:
        idx, J, r_e, W = recs[f]
        R = J @ Sig[np.ix_(idx, idx)] @ J.T
        R = (R + R.T) / 2
        d2_audit, _ = audit_record(R, W, r_e - J @ x[idx])
        Am = A.copy()
        Am[np.ix_(idx, idx)] -= J.T @ W @ J
        gm = g.copy()
        gm[idx] -= J.T @ W @ r_e
        xm = np.linalg.solve(Am, gm)
        Sm = np.linalg.inv(Am)
        Rm = J @ Sm[np.ix_(idx, idx)] @ J.T
        d2_cand = candidate_d2((Rm + Rm.T) / 2, W, r_e - J @ xm[idx])
        rel = abs(d2_audit - d2_cand) / max(d2_cand, 1e-300)
        worst = max(worst, rel)
        assert rel <= 1e-9, (f, d2_audit, d2_cand)
    return worst


def test_leave_one_out_identity():
    d = m3500_head(300)
    rng = np.random.default_rng(11)
    picks = closures(d, 12, rng)
    _loo_check(d, None, picks)
    # a robust closure: the Hessian holds w W; the identity holds with W_f = w W
    w = np.ones(d.n_edges)
    w[picks[:4]] = [0.3, 0.05, 1e-3, 0.7]
    _loo_check(d, w, picks[:4])


def test_planted_outlier_stands_out():
    d = m3500_head(300)
    rng = np.random.default_rng(5)
    f = int(closures(d, 1, rng)[0])
    d.ez[f] = d.ez[f] + np.array([3.0, -2.0, 0.8])
    A, g, recs = system(d, d.init)
    Sig = np.linalg.inv(A)
    x = Sig @ g
    idx, J, r_e, W = recs[f]
    R = J @ Sig[np.ix_(idx, idx)] @ J.T
    d2, _ = audit_record((R + R.T) / 2, W, r_e - J @ x[idx])
    assert d2 > CHI2_3_999


def test_trace_identity():
    d = m3500_head(250)
    A, _, recs = system(d, d.init)
    Sig = np.linalg.inv(A)
    total = 0.0
    for idx, J, r, W in recs:
        R = J @ Sig[np.ix_(idx, idx)] @ J.T
        total += 3.0 - audit_record((R + R.T) / 2, W, r)[1]
    total += LAM * np.trace(Sig)
    assert abs(total - 3 * d.n_nodes) <= 1e-9 * 3 * d.n_nodes
