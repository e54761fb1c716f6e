"""Candidate factors on the GPU (k_marginal_path / k_marginal_pairs behind aprilsam_b200_candidate_mahalanobis).

  1. accuracy: Sigma_rel against J Sigma_6 J' in long double with Sigma_6 from marginal_covariance([a, b]) (REL_C);
     a prior's Sigma_rel bit-identical to the diagonal block of marginal_covariance; d2 against r' S^-1 r in long
     double within the bound of `d2_bound`; end to end against sparse LU columns of A^-1 within FORWARD_C kappa_1 u;
     on M3500, on worlds with a pose under every kind of front and on the dense 100 k world's 9-hop paths;
  2. independence: alone, inside a 4096-candidate request, reversed, shuffled, one candidate per batch and call to
     call, bit for bit; relative_covariance(a, b) is the query's Sigma_rel;
  3. a z equal to the prediction at the states gives d2 = 0 exactly;
  4. a query changes nothing the solve path holds, and replays with queries take the same steps;
  5. the SLAM flow: closures of the newest pose after incremental steps, a general-fallback step and appends into
     the team-merged root;
  6. limits: more than 65535 distinct poses, many batches, two graphs in turn, the hop checks on the call's scratch;
  7. every error case.
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
from support import margcheck as mc
from test_gpu_kernels import add_priors, zoo
from test_gpu_marginals import FORWARD_C, HOP_C, REL_C, _device_state, _path_snapshot, pick_poses

LD = mc.LD
U = fc.U
W_CAND = np.array([[400.0, 30.0, 0.0], [30.0, 250.0, 5.0], [0.0, 5.0, 2000.0]])


def _lib():
    from aprilsam_b200 import capi
    return capi.lib()


def set_budget(nbytes):
    _lib().asam_dbg_set_candidate_budget(int(nbytes))


def candidates(N, rng, k, newest=None):
    """k candidates: the newest pose against random old ones, random pairs and priors, a third each, with z drawn
    around zero and W = W_CAND."""
    newest = N - 1 if newest is None else newest
    n1, n2 = k // 3, k // 3
    a = np.r_[np.full(n1, newest), rng.integers(0, N, n2), rng.integers(0, N, k - n1 - n2)]
    b = np.r_[rng.integers(0, newest, n1), rng.integers(0, N, n2), np.full(k - n1 - n2, -1)]
    b[n1:n1 + n2] = np.where(b[n1:n1 + n2] == a[n1:n1 + n2], (a[n1:n1 + n2] + 1) % N, b[n1:n1 + n2])
    z = rng.normal(0, 0.5, (k, 3))
    W = np.tile(W_CAND.reshape(9), (k, 1))
    return a.astype(np.int32), b.astype(np.int32), z, W


def query(h, a, b, z, W):
    return h.candidate_mahalanobis(a, b, z, W, with_cov=True)


def _ld_inv3(M):
    M = M.astype(LD)
    cols = []
    for e in np.eye(3, dtype=LD):
        cols.append(_ld_solve3(M, e))
    return np.array(cols, dtype=LD).T


def _ld_solve3(M, r):
    A = M.astype(LD).copy()
    x = r.astype(LD).copy()
    for k in range(3):
        for i in range(k + 1, 3):
            f = A[i, k] / A[k, k]
            A[i, k:] -= f * A[k, k:]
            x[i] -= f * x[k]
    y = np.zeros(3, dtype=LD)
    for i in (2, 1, 0):
        y[i] = (x[i] - A[i, i + 1:] @ y[i + 1:]) / A[i, i]
    return y


def residual_ld(st, a, b, z):
    """z - h(x) at the states in long double, theta wrapped."""
    z = z.astype(LD)
    pa = st[a].astype(LD)
    if b < 0:
        r = z - pa
    else:
        pb = st[b].astype(LD)
        ca, sa = np.cos(pa[2]), np.sin(pa[2])
        dx, dy = pb[0] - pa[0], pb[1] - pa[1]
        r = np.array([z[0] - (ca * dx + sa * dy), z[1] - (-sa * dx + ca * dy), z[2] - (pb[2] - pa[2])], dtype=LD)
    r[2] = (r[2] + LD(np.pi)) % LD(2 * np.pi) - LD(np.pi)
    return r, np.abs(z) + np.abs(st[a]).sum() + (np.abs(st[b]).sum() if b >= 0 else 0.0) + 2 * np.pi


def d2_bound(S, Sinv_norm, dS, d2, r_scale):
    """First-order bound on |d2 - r'S^-1 r| for d2 computed from S + dS and r + dr:
         ||S^-1|| ||dS|| d2            (the perturbation of S: Sigma_rel, W^-1, the sum and the 3x3 Cholesky)
       + 2 sqrt(d2 ||S^-1||) ||dr||    (||dr|| <= 8 u r_scale: the host's residual in double, libm trig included)
       + 8 u d2                        (the triangular solve and the sum of squares)"""
    return Sinv_norm * dS * d2 + 2 * math.sqrt(max(d2, 0.0) * Sinv_norm) * 8 * U * r_scale + 8 * U * d2


def check_accuracy(h, a, b, z, W, d2, cov, tag=""):
    """Item 1 for every candidate given: returns the worst shares of REL_C and of the d2 bound."""
    lp = h.l_points()
    st = h.states()
    worst = {"rel_u": 0.0, "d2": 0.0}
    for c in range(len(a)):
        A, B = int(a[c]), int(b[c])
        Wm = W[c].reshape(3, 3)
        Winv = _ld_inv3(Wm)
        kW = np.linalg.cond(Wm, 2)
        assert np.array_equal(cov[c], cov[c].T), c
        if B < 0:
            S3 = h.marginal_covariance([A])
            assert np.array_equal(cov[c].view(np.int64), S3.view(np.int64)), (tag, c)
            Rref = S3.astype(LD)
            dR = 0.0
        else:
            S6 = h.marginal_covariance([A, B]).astype(LD)
            Ja, Jb, _ = emul.xyt_eval(lp[A], lp[B], np.zeros(3))
            J = np.hstack([Ja, Jb]).astype(LD)
            Rref = J @ S6 @ J.T
            scale = np.abs(J) @ np.abs(S6) @ np.abs(J).T
            e = float(np.max(np.abs(cov[c].astype(LD) - Rref) / scale)) / U
            worst["rel_u"] = max(worst["rel_u"], e)
            assert e <= REL_C, (tag, c, e)
            dR = REL_C * U * float(np.linalg.norm(np.asarray(scale, dtype=np.float64), 2))
        S = Rref + Winv
        r, r_scale = residual_ld(st, A, B, z[c])
        ref = float(r @ _ld_solve3(S, r))
        S64 = np.asarray(S, dtype=np.float64)
        Sinv = np.linalg.norm(np.linalg.inv(S64), 2)
        dS = dR + 8 * U * kW * float(np.linalg.norm(np.asarray(Winv, dtype=np.float64), 2)) + \
            8 * U * float(np.linalg.norm(S64, 2))
        bnd = d2_bound(S64, Sinv, dS, ref, float(np.linalg.norm(np.asarray(r_scale, dtype=np.float64))))
        assert abs(d2[c] - ref) <= bnd, (tag, c, d2[c], ref, bnd)
        worst["d2"] = max(worst["d2"], abs(d2[c] - ref) / bnd if bnd > 0 else 0.0)
    print(f"CANDCHECK {tag} " + json.dumps(worst))
    return worst


def end_to_end(h, a, b, cov, tag=""):
    """Sigma_rel against J Sigma_6 J' with Sigma_6 from sparse LU columns of A^-1, within FORWARD_C kappa_1 u."""
    import scipy.sparse.linalg as spl
    L = fc.dev_api()
    snap = fc.snapshot(h, L)
    ftype, fa, fb, _, _ = fc.factors_of(h)
    A, _ = fc.system(snap, ftype, fa, fb, snap.plan.array("fslot"))
    lu = spl.splu(A.tocsc())
    lp = h.l_points()
    worst = 0.0
    E0 = np.zeros(A.shape[0]); E0[0] = 1.0
    _, kappa = fc.reference_solution(A, E0, steps=0)
    for c in range(len(a)):
        ids = [int(a[c])] + ([int(b[c])] if b[c] >= 0 else [])
        q = snap.node2q[ids].astype(np.int64)
        idx = (3 * q[:, None] + np.arange(3)).reshape(-1)
        E = np.zeros((A.shape[0], len(idx))); E[idx, np.arange(len(idx))] = 1.0
        S6 = lu.solve(E)[idx]
        if b[c] >= 0:
            Ja, Jb, _ = emul.xyt_eval(lp[ids[0]], lp[ids[1]], np.zeros(3))
            J = np.hstack([Ja, Jb])
            ref = J @ S6 @ J.T
        else:
            ref = S6
        worst = max(worst, float(np.abs(cov[c] - ref).max() / np.abs(ref).max() / (kappa * U)))
    print(f"CANDCHECK {tag} end to end {worst:.2e} kappa_1 u")
    assert worst <= FORWARD_C, worst


def front_candidates(h, snap, rng):
    """Closures from the newest pose to every pose of pick_poses (newest, oldest, team, leaf, wide back-solve
    blocks, j0 inside a block), pairs among them and priors on them."""
    p = pick_poses(h, snap)
    N = len(snap.q2node)
    p = np.unique(p)
    a = np.r_[np.full(len(p), N - 1), p, p]
    b = np.r_[p, np.roll(p, 1), np.full(len(p), -1)]
    keep = a != b
    a, b = a[keep], b[keep]
    z = rng.normal(0, 0.3, (len(a), 3))
    return a.astype(np.int32), b.astype(np.int32), z, np.tile(W_CAND.reshape(9), (len(a), 1))


# ---------------------------------------------------------------------------------------------
# 1. accuracy
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["m3500", "team162_c51", "bs_195", "wide"])
def test_accuracy(m3500, name):
    d = m3500 if name == "m3500" else zoo(name)
    rng = np.random.default_rng(1)
    with H.Harness("b200") as h:
        h.load_full(d)
        if name != "m3500":
            add_priors(h, d)
        h.batch()
        snap = fc.snapshot(h, fc.dev_api())
        a, b, z, W = front_candidates(h, snap, rng)
        d2, cov = query(h, a, b, z, W)
        check_accuracy(h, a, b, z, W, d2, cov, name)
        end_to_end(h, a, b, cov, name)


@pytest.mark.gpu
def test_dense_100k_nine_hops(built):
    """Closures of the newest pose with the oldest (9 hops) and random poses of the dense 100 k world, and priors."""
    from aprilsam_b200 import datasets
    d = datasets.manhattan_dense(100000, seed=1)
    N = d.n_nodes
    rng = np.random.default_rng(11)
    old = np.r_[0, rng.choice(np.arange(1, N - 1), 15, replace=False)]
    a = np.r_[np.full(len(old), N - 1), old[:4]].astype(np.int32)
    b = np.r_[old, np.full(4, -1)].astype(np.int32)
    z = rng.normal(0, 0.3, (len(a), 3))
    W = np.tile(W_CAND.reshape(9), (len(a), 1))
    with H.Harness("b200") as h:
        h.load_full(d)
        h.batch()
        L = fc.dev_api()
        snap = _path_snapshot(h, L, np.array([0, N - 1], np.int32))
        assert {len(mc.chain(snap.desc, r["sn0"])) for r in mc.paths(snap.plan, np.array([0], np.int32))[0]} == {9}
        d2, cov = query(h, a, b, z, W)
        check_accuracy(h, a, b, z, W, d2, cov, "dense100k")


# ---------------------------------------------------------------------------------------------
# 2. independence and 3. the exact case
# ---------------------------------------------------------------------------------------------
def _bits(x):
    return np.ascontiguousarray(x).view(np.int64)


@pytest.mark.gpu
def test_independent_of_request_order_and_batches(m3500):
    rng = np.random.default_rng(5)
    with H.Harness("b200") as h:
        h.load_full(m3500)
        h.batch()
        a, b, z, W = candidates(m3500.n_nodes, rng, 4096)
        d2, cov = query(h, a, b, z, W)
        out = np.c_[d2, cov.reshape(-1, 9)]
        assert np.all(np.isfinite(out))
        again = np.c_[query(h, a, b, z, W)[0], query(h, a, b, z, W)[1].reshape(-1, 9)]
        assert np.array_equal(_bits(out), _bits(again))
        for perm in (np.arange(len(a))[::-1], rng.permutation(len(a))):
            d2p, covp = query(h, a[perm], b[perm], z[perm], W[perm])
            assert np.array_equal(_bits(np.c_[d2p, covp.reshape(-1, 9)]), _bits(out[perm]))
        try:
            set_budget(1)  # one candidate per batch
            sub = rng.choice(len(a), 300, replace=False)
            d2s, covs = query(h, a[sub], b[sub], z[sub], W[sub])
        finally:
            set_budget(0)
        assert np.array_equal(_bits(np.c_[d2s, covs.reshape(-1, 9)]), _bits(out[sub]))
        for c in list(rng.choice(len(a), 24, replace=False)) + [0, len(a) - 1]:
            d2a, cova = query(h, a[c:c + 1], b[c:c + 1], z[c:c + 1], W[c:c + 1])
            assert np.array_equal(_bits(np.c_[d2a, cova.reshape(-1, 9)]), _bits(out[c:c + 1])), c
            if b[c] >= 0:
                assert np.array_equal(_bits(h.relative_covariance(a[c], b[c])), _bits(cov[c])), c
        check_accuracy(h, a[:40], b[:40], z[:40], W[:40], d2[:40], cov[:40], "m3500_4096_head")


@pytest.mark.gpu
def test_prediction_gives_zero(m3500):
    """z = h(x) at the states, computed in double with math.cos / math.sin (the C library's), gives d2 = 0."""
    with H.Harness("b200") as h:
        h.load_full(m3500.head(1000))
        h.batch()
        st = h.states()
        pairs = [(999, 0), (999, 500), (3, 998), (10, 11), (400, -1), (0, -1)]
        a, b, z = [], [], []
        for i, j in pairs:
            pa = [float(v) for v in st[i]]
            if j < 0:
                zz = pa
            else:
                pb = [float(v) for v in st[j]]
                ca, sa = math.cos(pa[2]), math.sin(pa[2])
                dx, dy = pb[0] - pa[0], pb[1] - pa[1]
                zz = [ca * dx + sa * dy, -sa * dx + ca * dy, pb[2] - pa[2]]
            a.append(i); b.append(j); z.append(zz)
        d2 = h.candidate_mahalanobis(a, b, np.array(z), np.tile(W_CAND.reshape(9), (len(a), 1)))
        assert np.all(d2 == 0.0), d2


# ---------------------------------------------------------------------------------------------
# 4. nothing changes
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_query_changes_nothing(m3500):
    rng = np.random.default_rng(2)
    with H.Harness("b200") as h:
        h.load_full(m3500.head(1500))
        h.batch()
        before, _ = _device_state(h)
        st, lp = h.states().copy(), h.l_points().copy()
        query(h, *candidates(1500, rng, 500))
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
                    query(h, *candidates(k, rng, 64))
            runs.append((h.states().copy(), infos))
    (s0, i0), (s1, i1) = runs
    assert all(np.array_equal(x, y) for x, y in zip(i0, i1))
    diff = s0 - s1
    diff[:, 2] = emul.mod2pi(diff[:, 2])
    assert np.abs(diff).max() < 1e-9  # k_linearize's atomic sums: solves agree to rounding, not bit for bit


# ---------------------------------------------------------------------------------------------
# 5. the SLAM flow
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_slam_flow(m3500):
    """Per step: the pose and its odometry, april_graph_cholesky_inc, then that step's closures between the new pose
    and old ones; then a general-fallback step; then appends into the team-merged root of dense2000."""
    from aprilsam_b200 import datasets
    rng = np.random.default_rng(6)
    with H.Harness("b200") as h:
        h.replay_begin(m3500.head(400))
        h.replay_to(300)
        for k in range(301, 401):
            h.replay_to(k)
            a, b = np.full(12, k - 1, np.int32), rng.integers(0, k - 1, 12).astype(np.int32)
            z, W = rng.normal(0, 0.3, (12, 3)), np.tile(W_CAND.reshape(9), (12, 1))
            d2, cov = query(h, a, b, z, W)
            if k % 25 == 0:
                check_accuracy(h, a, b, z, W, d2, cov, f"slam step {k}")
        h.add_xyt(10, 350, m3500.ez[0], np.diag([100.0, 100.0, 1000.0]).reshape(9))
        h.inc()
        a, b, z, W = candidates(400, rng, 30, newest=399)
        d2, cov = query(h, a, b, z, W)
        check_accuracy(h, a, b, z, W, d2, cov, "general fallback")
        end_to_end(h, a, b, cov, "general fallback")
    d = datasets.manhattan_dense(2000, seed=1)
    with H.Harness("b200") as h:
        h.replay_begin(d)
        h.replay_to(1900, batch_only=True)
        h.replay_to(2000)
        a, b, z, W = candidates(2000, rng, 30, newest=1999)
        d2, cov = query(h, a, b, z, W)
        check_accuracy(h, a, b, z, W, d2, cov, "team-merged root")


# ---------------------------------------------------------------------------------------------
# 6. limits
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_large_requests_on_100k(built):
    """70000 priors on distinct poses of the dense 100 k world (more than the 65535 of marginal_covariance), then
    4096 closures of the newest pose under a budget that forces many batches; samples bit for bit alone."""
    from aprilsam_b200 import datasets
    from test_candidates_cpu import batches
    d = datasets.manhattan_dense(100000, seed=1)
    N = d.n_nodes
    rng = np.random.default_rng(9)
    with H.Harness("b200") as h:
        h.load_full(d)
        h.batch()
        host = fc.borrowed_plan(fc.dev_api(), h.param_ptr())
        a = rng.choice(N, 70000, replace=False).astype(np.int32)
        b = np.full(len(a), -1, np.int32)
        z = rng.normal(0, 0.3, (len(a), 3))
        W = np.tile(W_CAND.reshape(9), (len(a), 1))
        nb = len(batches(host, a, b, (256 << 20) // 8))
        d2, cov = query(h, a, b, z, W)
        print(f"CANDLIMIT 70000 distinct poses in {nb} batches")
        assert np.all(np.isfinite(d2))
        for c in rng.choice(len(a), 8, replace=False):
            d2a, cova = query(h, a[c:c + 1], b[c:c + 1], z[c:c + 1], W[c:c + 1])
            assert _bits(d2a)[0] == _bits(d2[c:c + 1])[0] and np.array_equal(_bits(cova[0]), _bits(cov[c])), c
        a, b, z, W = candidates(N, rng, 4096)
        ref = query(h, a, b, z, W)
        budget = 64 << 20
        nb = len(batches(host, a, b, budget // 8))
        assert nb >= 4, nb
        try:
            set_budget(budget)
            got = query(h, a, b, z, W)
        finally:
            set_budget(0)
        print(f"CANDLIMIT 4096 candidates in {nb} batches")
        assert np.array_equal(_bits(got[0]), _bits(ref[0])) and np.array_equal(_bits(got[1]), _bits(ref[1]))
        sel = rng.choice(len(a), 12, replace=False)
        check_accuracy(h, a[sel], b[sel], z[sel], W[sel], ref[0][sel], ref[1][sel], "dense100k batches")


@pytest.mark.gpu
def test_two_graphs_query_in_turn(m3500, built):
    from aprilsam_b200 import datasets
    da = datasets.manhattan_dense(2000, seed=1)
    rng = np.random.default_rng(4)
    qa, qb = candidates(2000, rng, 200), candidates(m3500.n_nodes, rng, 200)

    def live(d):
        h = H.Harness("b200")
        h.load_full(d)
        h.batch()
        return h

    with live(da) as ha:
        alone = query(ha, *qa)
        with live(m3500) as hb:
            first_b = query(hb, *qb)
            for h, q, ref in ((ha, qa, alone), (hb, qb, first_b), (ha, qa, alone)):
                got = query(h, *q)
                assert np.array_equal(_bits(got[0]), _bits(ref[0])) and np.array_equal(_bits(got[1]), _bits(ref[1]))


@pytest.mark.gpu
def test_hop_checks_on_the_query_scratch(m3500):
    """margcheck's hop checks on the z and hop records this call left in its scratch (one batch)."""
    rng = np.random.default_rng(7)
    with H.Harness("b200") as h:
        h.load_full(m3500)
        h.batch()
        L = fc.dev_api()
        snap = fc.snapshot(h, L)
        a, b, z, W = front_candidates(h, snap, rng)
        query(h, a, b, z, W)
        poses = []
        for x in np.c_[a, b].reshape(-1):
            if x >= 0 and x not in poses:
                poses.append(int(x))
        recs, zt, ht = mc.paths(snap.plan, np.array(poses, np.int32))
        o = (C.c_int64 * 6)()
        _lib().asam_debug_marginal_pairs_layout(len(poses), zt, ht, len(a), o)
        dev = L.asam_dbg_dev_of_graph(h.graph_ptr())
        Z = mc._read(mc._api(L), dev, mc.DBG_BUF_MARG, o[2], np.zeros(zt))
        hop = mc._read(L, dev, mc.DBG_BUF_MARG, o[3], np.zeros((ht, 4), dtype=np.int32))
        assert mc.check_hops(snap.desc, recs, hop) == 0
        worst, where = mc.worst_hop(snap, recs, Z)
        print(f"CANDCHECK hop {worst / U:.2f} u at {where}")
        assert worst / U <= HOP_C, (worst / U, where)


# ---------------------------------------------------------------------------------------------
# 7. errors
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_errors_leave_the_solver_usable(m3500):
    lib = H._load("b200")
    d = m3500.head(300)
    rng = np.random.default_rng(8)
    good = candidates(200, rng, 6)
    with H.Harness("b200") as h:
        h.replay_begin(d)
        with pytest.raises(RuntimeError, match="does not continue a solve"):
            query(h, *good)
        h.replay_to(200)
        ip, dp = C.POINTER(C.c_int), C.POINTER(C.c_double)
        a, b, z, W = good
        d2 = np.zeros(6)
        args = [x.ctypes.data_as(ip) for x in (a, b)] + [x.ctypes.data_as(dp) for x in (z, W, d2)]
        assert lib.h_candidate_mahalanobis(h.h, 0, *args, None) == -1
        assert "k < 1" in lib.aprilsam_b200_last_error().decode()
        for k in range(5):
            bad = list(args)
            bad[k] = None
            assert lib.h_candidate_mahalanobis(h.h, 6, *bad, None) == -1
            assert "NULL" in lib.aprilsam_b200_last_error().decode()

        def expect(match, **kw):
            q = [x.copy() for x in good]
            for key, (c, v) in kw.items():
                q["abzW".index(key)][c] = v
            with pytest.raises(RuntimeError, match=match):
                query(h, *q)

        expect(r"candidate 3: node 200 is not in the solved graph", a=(3, 200))
        expect(r"candidate 1: node -2 is not in the solved graph", a=(1, -2))
        expect(r"candidate 4: node 10000 is not in the solved graph", b=(4, 10000))
        expect(r"candidate 2: b = -3", b=(2, -3))
        expect(r"candidate 5: a == b", b=(5, int(good[0][5])))
        expect(r"candidate 0: z is not finite", z=(0, [0.0, np.nan, 0.0]))
        expect(r"candidate 3: z is not finite", z=(3, [np.inf, 0.0, 0.0]))
        for Wbad in ([1, 0.5, 0, 0.4, 1, 0, 0, 0, 1], [1, 0, 0, 0, -1, 0, 0, 0, 1], [1, 2, 0, 2, 1, 0, 0, 0, 1],
                     [1, 0, 0, 0, 1, 0, 0, 0, np.nan], [0] * 9):
            expect(r"candidate 1: W is not symmetric positive definite", W=(1, Wbad))
        ref = query(h, *good)
        h.replay_to(250)
        query(h, *good)
        h.invalidate_plan()
        with pytest.raises(RuntimeError, match="plan was dropped"):
            query(h, *good)
        h.batch()
        n = h.n_nodes
        h.add_node(h.states()[n - 1])
        with pytest.raises(RuntimeError, match="added since the last solve"):
            query(h, *good)
        h.add_xyt(n - 1, n, np.zeros(3), np.diag([100.0, 100.0, 1000.0]).reshape(9))
        h.inc()
        d2, cov = query(h, *good)
        check_accuracy(h, *good, d2, cov, "after errors")
        assert ref[0].shape == d2.shape
