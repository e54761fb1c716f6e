"""Candidate compatibility on the GPU (k_marginal_compat behind aprilsam_b200_candidate_compatibility).

  1. the diagonal: d2 and cross9 at (c, c) are candidate_mahalanobis' d2 and cov9 bit for bit; d2 is exactly
     symmetric and cross9 at (j, i) is the exact transpose of (i, j);
  2. accuracy: C_ij against J_i Sigma J_j' in long double with Sigma from marginal_covariance of the pair's poses
     (REL_C), d2_ij against [r_i; r_j]' S_ij^-1 [r_i; r_j] in long double within a d2_bound-style bound, and end to end
     against sparse LU columns of A^-1 within FORWARD_C kappa_1 u; on M3500, robust M3500, worlds with a pose under
     every kind of front (priors among the candidates) and the dense 100 k world's 9-hop paths;
  3. independence: a pair alone, inside a 1024-candidate request, reversed, shuffled, repeated and one pair per tile,
     bit for bit;
  4. against a real solve: after adding candidate i with april_graph_cholesky_inc, candidate_mahalanobis of j is
     d2_ij - d2_i within COND_C;
  5. planted aliasing end to end: gate, compatibility, greedy clique, add;
  6. nothing changes: the device state, a replay with queries interleaved, queries after incremental steps, a removal
     and an in-place relinearisation, and every refusal.
"""
from __future__ import annotations

import ctypes as C
import json
import math

import numpy as np
import pytest

from aprilsam_b200 import harness as H
from support import emul
from support import frontcheck as fc
from test_gpu_candidates import (LD, U, W_CAND, _bits, _ld_inv3, candidates, d2_bound, front_candidates,
                                 residual_ld, set_budget)
from test_gpu_kernels import add_priors, zoo
from test_gpu_marginals import FORWARD_C, REL_C, _device_state

CHI2_3_99 = 11.34
CHI2_6_99 = 16.81
CHI2_6_999 = 22.46
COND_C = 0.05  # |candidate d2 of j after adding i - (d2_ij - d2_i)| / (that d2 + 1e-3) on converged M3500
HUBER, CAUCHY = 1, 2


def compat(h, a, b, z, W):
    return h.candidate_compatibility(a, b, z, W, with_cross=True)


def _ld_solve(M, r):
    A = M.astype(LD).copy()
    x = r.astype(LD).copy()
    n = len(x)
    for k in range(n):
        for i in range(k + 1, n):
            f = A[i, k] / A[k, k]
            A[i, k:] -= f * A[k, k:]
            x[i] -= f * x[k]
    y = np.zeros(n, dtype=LD)
    for i in range(n - 1, -1, -1):
        y[i] = (x[i] - A[i, i + 1:] @ y[i + 1:]) / A[i, i]
    return y


def _jac(lp, a, b, poses):
    """J of candidate (a, b) over the 3 |poses| columns of poses (J = [I 0] for a prior)."""
    J = np.zeros((3, 3 * len(poses)), dtype=LD)
    ia = poses.index(a)
    if b < 0:
        J[:, 3 * ia:3 * ia + 3] = np.eye(3)
    else:
        Ja, Jb, _ = emul.xyt_eval(lp[a], lp[b], np.zeros(3))
        ib = poses.index(b)
        J[:, 3 * ia:3 * ia + 3] = Ja
        J[:, 3 * ib:3 * ib + 3] = Jb
    return J


def check_diagonal(h, a, b, z, W, d2, cross, tag=""):
    """Item 1: the diagonal against candidate_mahalanobis bit for bit, and the exact symmetries."""
    ref, cov = h.candidate_mahalanobis(a, b, z, W, with_cov=True)
    k = len(a)
    assert np.array_equal(_bits(np.diag(d2).copy()), _bits(ref)), tag
    assert np.array_equal(_bits(cross[np.arange(k), np.arange(k)]), _bits(cov)), tag
    assert np.array_equal(_bits(d2), _bits(d2.T)), tag
    assert np.array_equal(_bits(cross), _bits(cross.transpose(1, 0, 3, 2))), tag


def check_pairs(h, a, b, z, W, d2, cross, pairs, tag=""):
    """Item 2 for the pairs given: C_ij and d2_ij against long double from marginal_covariance of the pair's poses.
    Returns the worst shares of REL_C and of the d2 bound."""
    lp, st = h.l_points(), h.states()
    worst = {"rel_u": 0.0, "d2": 0.0}
    for i, j in pairs:
        i, j = int(i), int(j)
        ids = [int(a[i]), int(b[i]), int(a[j]), int(b[j])]
        poses = sorted({p for p in ids if p >= 0})
        Sig = h.marginal_covariance(poses).astype(LD)
        Ji, Jj = _jac(lp, ids[0], ids[1], poses), _jac(lp, ids[2], ids[3], poses)
        Cref = Ji @ Sig @ Jj.T
        scale = np.abs(Ji) @ np.abs(Sig) @ np.abs(Jj).T
        e = float(np.max(np.abs(cross[i, j].astype(LD) - Cref) / scale)) / U
        worst["rel_u"] = max(worst["rel_u"], e)
        assert e <= REL_C, (tag, i, j, e)
        Ri, Rj = Ji @ Sig @ Ji.T, Jj @ Sig @ Jj.T
        Wi, Wj = W[i].reshape(3, 3), W[j].reshape(3, 3)
        S = np.block([[Ri + _ld_inv3(Wi), Cref], [Cref.T, Rj + _ld_inv3(Wj)]])
        ri, si = residual_ld(st, ids[0], ids[1], z[i])
        rj, sj = residual_ld(st, ids[2], ids[3], z[j])
        v = np.r_[ri, rj]
        ref = float(v @ _ld_solve(S, v))
        S64 = np.asarray(S, dtype=np.float64)
        Sinv = np.linalg.norm(np.linalg.inv(S64), 2)
        sc = np.asarray(np.block([[np.abs(Ji) @ np.abs(Sig) @ np.abs(Ji).T, scale],
                                  [scale.T, np.abs(Jj) @ np.abs(Sig) @ np.abs(Jj).T]]), dtype=np.float64)
        winv = max(np.linalg.norm(np.linalg.inv(Wi), 2) * np.linalg.cond(Wi, 2),
                   np.linalg.norm(np.linalg.inv(Wj), 2) * np.linalg.cond(Wj, 2))
        dS = REL_C * U * float(np.linalg.norm(sc, 2)) + 8 * U * winv + 16 * U * float(np.linalg.norm(S64, 2))
        r_scale = float(np.linalg.norm(np.asarray(np.r_[si, sj], dtype=np.float64)))
        bnd = d2_bound(S64, Sinv, dS, ref, r_scale) + 8 * U * ref
        assert abs(d2[i, j] - ref) <= bnd, (tag, i, j, d2[i, j], ref, bnd)
        worst["d2"] = max(worst["d2"], abs(d2[i, j] - ref) / bnd if bnd > 0 else 0.0)
    print(f"COMPATCHECK {tag} " + json.dumps(worst))
    return worst


def end_to_end(h, a, b, z, W, d2, cross, pairs, tag=""):
    """C_ij and d2_ij against Sigma from sparse LU columns of A^-1 (A from the Hessian in HBM), within FORWARD_C
    kappa_1 u: C relative to sqrt(|Sigma_rel,i| |Sigma_rel,j|), d2 relative to cond(S_ij) d2."""
    import scipy.sparse.linalg as spl
    L = fc.dev_api()
    snap = fc.snapshot(h, L)
    ftype, fa, fb, _, _ = fc.factors_of(h)
    A, _ = fc.system(snap, ftype, fa, fb, snap.plan.array("fslot"))
    lu = spl.splu(A.tocsc())
    E0 = np.zeros(A.shape[0]); E0[0] = 1.0
    _, kappa = fc.reference_solution(A, E0, steps=0)
    lp, st = h.l_points(), h.states()
    used = sorted({int(p) for i, j in pairs for p in (a[i], b[i], a[j], b[j]) if p >= 0})
    q = snap.node2q[used].astype(np.int64)
    idx = (3 * q[:, None] + np.arange(3)).reshape(-1)
    E = np.zeros((A.shape[0], len(idx))); E[idx, np.arange(len(idx))] = 1.0
    Sig = lu.solve(E)[idx]
    worst = {"C": 0.0, "d2": 0.0}
    for i, j in pairs:
        i, j = int(i), int(j)
        Ji = np.asarray(_jac(lp, int(a[i]), int(b[i]), used), dtype=np.float64)
        Jj = np.asarray(_jac(lp, int(a[j]), int(b[j]), used), dtype=np.float64)
        Cref = Ji @ Sig @ Jj.T
        Ri, Rj = Ji @ Sig @ Ji.T, Jj @ Sig @ Jj.T
        norm = math.sqrt(np.abs(Ri).max() * np.abs(Rj).max())
        worst["C"] = max(worst["C"], float(np.abs(cross[i, j] - Cref).max() / norm / (kappa * U)))
        S = np.block([[Ri + np.linalg.inv(W[i].reshape(3, 3)), Cref], [Cref.T, Rj + np.linalg.inv(W[j].reshape(3, 3))]])
        ri, _ = residual_ld(st, int(a[i]), int(b[i]), z[i])
        rj, _ = residual_ld(st, int(a[j]), int(b[j]), z[j])
        v = np.asarray(np.r_[ri, rj], dtype=np.float64)
        ref = float(v @ np.linalg.solve(S, v))
        worst["d2"] = max(worst["d2"], abs(d2[i, j] - ref) / (np.linalg.cond(S, 1) * ref + 1e-300) / (kappa * U))
    print(f"COMPATCHECK {tag} end to end " + json.dumps(worst) + f" kappa_1 {kappa:.2e}")
    assert max(worst.values()) <= FORWARD_C, (tag, worst)


def sample_pairs(k, rng, n):
    i = rng.integers(0, k, n)
    j = rng.integers(0, k, n)
    keep = i != j
    return list(zip(np.minimum(i, j)[keep], np.maximum(i, j)[keep]))


# ---------------------------------------------------------------------------------------------------------------- 1, 2
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["m3500", "m3500_robust", "team162_c51", "bs_195", "wide"])
def test_accuracy(m3500, name):
    from test_gpu_audit import closures_of
    d = m3500 if name.startswith("m3500") else zoo(name)
    rng = np.random.default_rng(1)
    with H.Harness("b200") as h:
        h.load_full(d)
        add_priors(h, d)
        if name == "m3500_robust":
            for f in closures_of(d)[::3]:
                h.set_loss(int(f), HUBER if f % 2 else CAUCHY, 1.5)
        h.batch()
        snap = fc.snapshot(h, fc.dev_api())
        a, b, z, W = front_candidates(h, snap, rng)  # closures of the newest pose, pairs and priors, mixed
        d2, cross = compat(h, a, b, z, W)
        check_diagonal(h, a, b, z, W, d2, cross, name)
        k = len(a)
        pairs = sample_pairs(k, rng, 60)
        check_pairs(h, a, b, z, W, d2, cross, pairs, name)
        end_to_end(h, a, b, z, W, d2, cross, pairs, name)
        off = d2[~np.eye(k, dtype=bool)]
        assert np.all(np.isfinite(off))
        dg = np.diag(d2)
        assert np.all(d2 >= np.maximum(dg[:, None], dg[None, :]) * (1 - 1e-6) - 1e-12)


@pytest.mark.gpu
def test_dense_100k_nine_hops(built):
    from aprilsam_b200 import datasets
    from support import margcheck as mc
    from test_gpu_marginals import _path_snapshot
    d = datasets.manhattan_dense(100000, seed=1)
    N = d.n_nodes
    rng = np.random.default_rng(11)
    old = np.r_[0, rng.choice(np.arange(1, N - 1), 11, replace=False)]
    a = np.r_[np.full(len(old), N - 1), old[:4]].astype(np.int32)
    b = np.r_[old, np.full(4, -1)].astype(np.int32)
    z = rng.normal(0, 0.3, (len(a), 3))
    W = np.tile(W_CAND.reshape(9), (len(a), 1))
    with H.Harness("b200") as h:
        h.load_full(d)
        h.batch()
        snap = _path_snapshot(h, fc.dev_api(), np.array([0, N - 1], np.int32))
        assert {len(mc.chain(snap.desc, r["sn0"])) for r in mc.paths(snap.plan, np.array([0], np.int32))[0]} == {9}
        d2, cross = compat(h, a, b, z, W)
        check_diagonal(h, a, b, z, W, d2, cross, "dense100k")
        k = len(a)
        check_pairs(h, a, b, z, W, d2, cross, [(i, j) for i in range(k) for j in range(i + 1, k)][::3], "dense100k")


# ---------------------------------------------------------------------------------------------------------------- 3
@pytest.mark.gpu
def test_independent_of_request_order_and_tiles(m3500):
    rng = np.random.default_rng(5)
    with H.Harness("b200") as h:
        h.load_full(m3500)
        h.batch()
        a, b, z, W = candidates(m3500.n_nodes, rng, 1024)
        d2, cross = compat(h, a, b, z, W)
        assert np.all(np.isfinite(d2))
        again = compat(h, a, b, z, W)
        assert np.array_equal(_bits(again[0]), _bits(d2)) and np.array_equal(_bits(again[1]), _bits(cross))
        check_diagonal(h, a, b, z, W, d2, cross, "m3500_1024")
        for perm in (np.arange(len(a))[::-1], rng.permutation(len(a))):
            d2p, crossp = compat(h, a[perm], b[perm], z[perm], W[perm])
            assert np.array_equal(_bits(d2p), _bits(d2[np.ix_(perm, perm)]))
            assert np.array_equal(_bits(crossp), _bits(cross[np.ix_(perm, perm)]))
        for i, j in sample_pairs(len(a), rng, 24):
            s = np.array([i, j])
            d2s, crs = compat(h, a[s], b[s], z[s], W[s])
            assert np.array_equal(_bits(d2s), _bits(d2[np.ix_(s, s)])) and \
                np.array_equal(_bits(crs), _bits(cross[np.ix_(s, s)])), (i, j)
        sub = rng.choice(len(a), 24, replace=False)
        try:
            set_budget(1)  # one pair per tile
            d2s, crs = compat(h, a[sub], b[sub], z[sub], W[sub])
            set_budget(2 << 20)  # several tiles over the whole request
            d2m, crm = compat(h, a, b, z, W)
        finally:
            set_budget(0)
        assert np.array_equal(_bits(d2s), _bits(d2[np.ix_(sub, sub)])) and \
            np.array_equal(_bits(crs), _bits(cross[np.ix_(sub, sub)]))
        assert np.array_equal(_bits(d2m), _bits(d2)) and np.array_equal(_bits(crm), _bits(cross))
        check_pairs(h, a, b, z, W, d2, cross, sample_pairs(len(a), rng, 30), "m3500_1024")


# ---------------------------------------------------------------------------------------------------------------- 4
def predict(st, a, b):
    pa = [float(v) for v in st[a]]
    if b < 0:
        return np.array(pa)
    pb = [float(v) for v in st[b]]
    ca, sa = math.cos(pa[2]), math.sin(pa[2])
    dx, dy = pb[0] - pa[0], pb[1] - pa[1]
    return np.array([ca * dx + sa * dy, -sa * dx + ca * dy, pb[2] - pa[2]])


@pytest.mark.gpu
def test_against_adding_the_first_candidate(m3500):
    from test_gpu_audit import converge
    d = m3500.head(1000)
    rng = np.random.default_rng(9)
    worst = 0.0
    for t in range(4):
        with H.Harness("b200") as h:
            h.load_full(d)
            converge(h)
            st = h.states()
            N = d.n_nodes
            a = np.array([N - 1 - t, N - 3 - t], np.int32)
            b = np.array([int(rng.integers(0, N // 2)), int(rng.integers(0, N // 2))], np.int32)
            # i close to its prediction, so that adding it moves the states little and the second-order terms of h
            # (which the linear model leaves out: with r_i ~ N(0, 4 W^-1) they alone make a 3-10 % difference on
            # these loops in a dense float64 model) stay small; j drawn from its own S = Sigma_rel + W^-1, so that
            # d2_(j|i) is dominated by what adding i tells about j
            Winv = np.linalg.inv(W_CAND)
            W = np.tile(W_CAND.reshape(9), (2, 1))
            z = np.array([predict(st, a[c], b[c]) for c in range(2)])
            _, cov = h.candidate_mahalanobis(a, b, z, W, with_cov=True)
            z[0] += rng.multivariate_normal(np.zeros(3), 0.01 * Winv)
            z[1] += rng.multivariate_normal(np.zeros(3), cov[1] + Winv)
            d2 = h.candidate_compatibility(a, b, z, W)
            h.add_xyt(int(a[0]), int(b[0]), z[0], W_CAND.reshape(9))
            h.inc()
            ref = h.candidate_mahalanobis(a[1:], b[1:], z[1:], W[1:])[0]
            pred = d2[0, 1] - d2[0, 0]
            rel = abs(pred - ref) / (ref + 1e-3)
            worst = max(worst, rel)
            print(f"COMPATCHECK sequential {t}: d2_ij - d2_i {pred:.6g}, after adding i {ref:.6g}")
            assert rel <= COND_C, (t, pred, ref)
    print(f"COMPATCHECK sequential worst relative difference {worst:.3e}")


# ---------------------------------------------------------------------------------------------------------------- 5
ALIAS_LOOPS = ((200, 800), (300, 700))


def greedy_clique(ok):
    """The INTEGRATION caller's greedy maximum clique: candidates by decreasing number of compatible partners (ties by
    index), each kept when it is compatible with all kept so far."""
    deg = ok.sum(1)
    kept = []
    for c in sorted(range(len(ok)), key=lambda c: (-deg[c], c)):
        if all(ok[c, q] for q in kept):
            kept.append(c)
    return sorted(kept)


@pytest.mark.gpu
def test_planted_aliasing_caller_loop(m3500):
    d = m3500.head(1000)
    with H.Harness("b200") as h:
        h.load_full(d)
        h.batch()
        h.batch()
        st = h.states()
        for lo, hi in ALIAS_LOOPS:
            # true closures around the loop (z = the prediction at the states) and two aliased ones at (lo, hi) and
            # (lo + 1, hi + 1), shifted so that each alone has d2 = 9 but they pull the drift in opposite directions
            a = np.array([lo, lo + 1, lo - 1, lo + 2, lo + 3], np.int32)
            b = np.array([hi, hi + 1, hi - 1, hi + 2, hi + 3], np.int32)
            z = np.array([predict(st, a[c], b[c]) for c in range(len(a))])
            W = np.tile(W_CAND.reshape(9), (len(a), 1))
            _, cross = compat(h, a, b, z, W)
            Winv = np.linalg.inv(W_CAND)
            Si, Sj = cross[0, 0] + Winv, cross[1, 1] + Winv
            u = np.linalg.eigh(Si)[1][:, -1]
            for sign in (1.0, -1.0):
                uj = sign * (cross[0, 1].T @ np.linalg.solve(Si, u))
                zz = z.copy()
                zz[0] += 3.0 * u / math.sqrt(u @ np.linalg.solve(Si, u))
                zz[1] += 3.0 * uj / math.sqrt(uj @ np.linalg.solve(Sj, uj))
                d2 = h.candidate_compatibility(a[:2], b[:2], zz[:2], W[:2])
                print(f"COMPATCHECK alias ({lo}, {hi}) sign {sign:+.0f}: d2 {d2[0, 0]:.3f} {d2[1, 1]:.3f} "
                      f"joint {d2[0, 1]:.2f}")
                assert abs(d2[0, 0] - 9.0) < 1e-6 and abs(d2[1, 1] - 9.0) < 1e-6
                assert d2[0, 1] > CHI2_6_999 if sign < 0 else d2[0, 1] < CHI2_6_99, (lo, hi, sign, d2[0, 1])
            # the caller loop: gate, compatibility of the ones that passed, greedy clique, add
            gate = h.candidate_mahalanobis(a, b, zz, W)
            passed = np.flatnonzero(gate < CHI2_3_99)
            assert len(passed) == len(a)  # the aliased ones pass the gate on their own
            D = h.candidate_compatibility(a[passed], b[passed], zz[passed], W[passed])
            kept = passed[greedy_clique(D < CHI2_6_99)]
            assert sorted(kept.tolist()) == [2, 3, 4], (lo, hi, kept, D)
            for c in kept:
                h.add_xyt(int(a[c]), int(b[c]), zz[c], W[c])
            h.inc()
            st = h.states()


# ---------------------------------------------------------------------------------------------------------------- 6
@pytest.mark.gpu
def test_query_changes_nothing(m3500):
    rng = np.random.default_rng(2)
    with H.Harness("b200") as h:
        h.load_full(m3500.head(1500))
        h.batch()
        before, _ = _device_state(h)
        st, lp = h.states().copy(), h.l_points().copy()
        compat(h, *candidates(1500, rng, 300))
        after, _ = _device_state(h)
        assert all(np.array_equal(x, y) for x, y in zip(before, after))
        assert np.array_equal(st, h.states()) and np.array_equal(lp, h.l_points())


@pytest.mark.gpu
def test_replay_with_queries_takes_the_same_steps(m3500):
    d = m3500.head(600)
    runs = []
    for q in (False, True):
        rng = np.random.default_rng(3)
        with H.Harness("b200") as h:
            h.replay_begin(d)
            infos = []
            for k in range(50, 601, 50):
                _, _, inf = h.replay_to(k)
                infos.append(inf.copy())
                if q:
                    compat(h, *candidates(k, rng, 48))
            runs.append((h.states().copy(), infos))
    (s0, i0), (s1, i1) = runs
    assert all(np.array_equal(x, y) for x, y in zip(i0, i1))
    diff = s0 - s1
    diff[:, 2] = emul.mod2pi(diff[:, 2])
    assert np.abs(diff).max() < 1e-9  # k_linearize's atomic sums: solves agree to rounding, not bit for bit


@pytest.mark.gpu
def test_after_steps_removal_and_relinearisation(m3500):
    """Queries after incremental steps, a removal and an in-place relinearisation describe the system of that moment:
    the diagonal is that moment's candidate query, the pairs match that moment's marginal covariances."""
    from test_gpu_audit import factors_of
    d = m3500.head(400)
    rng = np.random.default_rng(4)
    with H.Harness("b200") as h:
        h.replay_begin(d)
        h.replay_to(300)
        for k in range(301, 401, 20):
            h.replay_to(k)
            q = candidates(k, rng, 24, newest=k - 1)
            d2, cross = compat(h, *q)
            check_diagonal(h, *q, d2, cross, f"step {k}")
            check_pairs(h, *q, d2, cross, sample_pairs(24, rng, 10), f"step {k}")
        t, a, b, _, _ = factors_of(h)
        cl = np.flatnonzero((t != 2) & (np.abs(b - a) > 1))
        h.remove_factors([int(cl[len(cl) // 2]), int(cl[-1])])
        q = candidates(h.n_nodes, rng, 24)
        d2, cross = compat(h, *q)
        check_diagonal(h, *q, d2, cross, "removal")
        check_pairs(h, *q, d2, cross, sample_pairs(24, rng, 10), "removal")
        N = h.n_nodes
        h.relinearize_poses([5, 60, N - 1])
        d2, cross = compat(h, *q)
        check_diagonal(h, *q, d2, cross, "relinearisation")
        check_pairs(h, *q, d2, cross, sample_pairs(24, rng, 10), "relinearisation")


@pytest.mark.gpu
def test_errors_change_nothing_and_leave_the_solver_usable(m3500):
    lib = H._load("b200")
    d = m3500.head(300)
    rng = np.random.default_rng(8)
    good = candidates(200, rng, 6)
    with H.Harness("b200") as h:
        h.replay_begin(d)
        with pytest.raises(RuntimeError, match="does not continue a solve"):
            compat(h, *good)
        h.replay_to(200)
        ref = compat(h, *good)
        before, _ = _device_state(h)
        ip, dp = C.POINTER(C.c_int), C.POINTER(C.c_double)
        a, b, z, W = good
        d2 = np.full((6, 6), 7.0)
        args = [x.ctypes.data_as(ip) for x in (a, b)] + [x.ctypes.data_as(dp) for x in (z, W, d2)]
        assert lib.h_candidate_compatibility(h.h, 0, *args, None) == -1
        assert "k < 1" in lib.aprilsam_b200_last_error().decode()
        for k in range(5):
            bad = list(args)
            bad[k] = None
            assert lib.h_candidate_compatibility(h.h, 6, *bad, None) == -1
            assert "NULL" in lib.aprilsam_b200_last_error().decode()
        assert lib.h_candidate_compatibility(h.h, 46341, *args, None) == -1
        assert "at most 46340" in lib.aprilsam_b200_last_error().decode()
        assert np.all(d2 == 7.0)  # refused before d2 is touched

        def expect(match, **kw):
            q = [x.copy() for x in good]
            for key, (c, v) in kw.items():
                q["abzW".index(key)][c] = v
            with pytest.raises(RuntimeError, match=match):
                compat(h, *q)

        expect(r"candidate_compatibility: candidate 3: node 200 is not in the solved graph", a=(3, 200))
        expect(r"candidate 4: node 10000 is not in the solved graph", b=(4, 10000))
        expect(r"candidate 2: b = -3", b=(2, -3))
        expect(r"candidate 5: a == b", b=(5, int(good[0][5])))
        expect(r"candidate 0: z is not finite", z=(0, [0.0, np.nan, 0.0]))
        expect(r"candidate 1: W is not symmetric positive definite", W=(1, [1, 0.5, 0, 0.4, 1, 0, 0, 0, 1]))
        after, _ = _device_state(h)
        assert all(np.array_equal(x, y) for x, y in zip(before, after))
        got = compat(h, *good)
        assert np.array_equal(_bits(got[0]), _bits(ref[0])) and np.array_equal(_bits(got[1]), _bits(ref[1]))
        h.invalidate_plan()
        with pytest.raises(RuntimeError, match="plan was dropped"):
            compat(h, *good)
        h.batch()
        n = h.n_nodes
        h.add_node(h.states()[n - 1])
        with pytest.raises(RuntimeError, match="added since the last solve"):
            compat(h, *good)
        h.add_xyt(n - 1, n, np.zeros(3), np.diag([100.0, 100.0, 1000.0]).reshape(9))
        h.inc()
        d2, cross = compat(h, *good)
        check_diagonal(h, *good, d2, cross, "after errors")
