"""Candidate factors (aprilsam_b200_candidate_mahalanobis) without a GPU: the batches plan_candidate_batches gives, the
residual helper shared with the eval hooks, and k_marginal_pairs' arithmetic restated in numpy on fronts of the
emulation against the long-double definition from the dense inverse of the emulated Hessian."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from support import emul
from support import frontcheck as fc
from support import margcheck as mc
from test_marginal_cpu import _emulated, _plan

_ip, _dp = C.POINTER(C.c_int), C.POINTER(C.c_double)
LD = mc.LD


def batches(plan, a, b, budget):
    """plan_candidate_batches on a HostPlan: [(candidates [c0, c1), distinct poses, ia, ib)] per batch."""
    L = plan.L
    L.asam_dbg_plan_candidate_batches.argtypes = [C.c_void_p, C.c_int, _ip, _ip, C.c_int64, _ip, _ip, _ip, _ip, _ip]
    a = np.ascontiguousarray(a, dtype=np.int32)
    b = np.ascontiguousarray(b, dtype=np.int32)
    k = len(a)
    be, pe = np.zeros(k, np.int32), np.zeros(k, np.int32)
    poses, ia, ib = np.zeros(2 * k, np.int32), np.zeros(k, np.int32), np.zeros(k, np.int32)
    ptr = lambda x: x.ctypes.data_as(_ip)  # noqa: E731
    nb = L.asam_dbg_plan_candidate_batches(plan.p, k, ptr(a), ptr(b), int(budget), ptr(be), ptr(poses), ptr(pe),
                                           ptr(ia), ptr(ib))
    out = []
    for t in range(nb):
        c0, p0 = (int(be[t - 1]), int(pe[t - 1])) if t else (0, 0)
        out.append((c0, int(be[t]), poses[p0:int(pe[t])].copy(), ia[c0:be[t]].copy(), ib[c0:be[t]].copy()))
    return out


def path_doubles(plan, nodes):
    return mc.paths(plan, np.asarray(nodes, dtype=np.int32))[1] if len(nodes) else 0


def check_batches(plan, a, b, budget):
    """Every candidate in exactly one batch, in input order; distinct poses per batch (a pose repeated in a batch is
    walked once); ia / ib point at the candidate's poses; each batch's scratch within the budget unless it holds a
    single candidate; a batch closes only where its next candidate's new poses would exceed the budget."""
    bs = batches(plan, a, b, budget)
    assert bs[0][0] == 0 and bs[-1][1] == len(a)
    assert all(bs[t][1] == bs[t + 1][0] and bs[t][0] < bs[t][1] for t in range(len(bs) - 1))
    for t, (c0, c1, poses, ia, ib) in enumerate(bs):
        assert len(set(poses.tolist())) == len(poses)
        assert np.array_equal(poses[ia], a[c0:c1])
        assert np.array_equal(np.where(b[c0:c1] >= 0, poses[np.maximum(ib, 0)], -1), b[c0:c1])
        assert np.all((ib >= 0) == (b[c0:c1] >= 0))
        used = {int(x) for x in a[c0:c1]} | {int(x) for x in b[c0:c1] if x >= 0}
        assert used == set(poses.tolist())
        z = path_doubles(plan, poses)
        assert z <= budget or c1 - c0 == 1, (t, z, budget)
        if t + 1 < len(bs):
            nxt = [int(a[c1])] + ([int(b[c1])] if b[c1] >= 0 else [])
            grown = sorted(set(poses.tolist()) | set(nxt))
            assert path_doubles(plan, grown) > budget, t
    return bs


def candidate_sets(N, rng, k):
    old = rng.choice(N - 1, k, replace=True)
    newest = (np.full(k, N - 1), old)
    pairs = tuple(rng.choice(N, (2, k), replace=True))
    pairs = (pairs[0], np.where(pairs[0] == pairs[1], (pairs[1] + 1) % N, pairs[1]))
    prior = (rng.choice(N, k), np.full(k, -1))
    mixed = (np.r_[newest[0][:k // 2], prior[0][:k // 2]], np.r_[newest[1][:k // 2], prior[1][:k // 2]])
    return {"newest_vs_old": newest, "pairs": pairs, "priors": prior, "mixed": mixed}


@pytest.mark.parametrize("world", ["m3500", "dense2000", "dense12000"])
def test_batches(m3500, world):
    from aprilsam_b200 import datasets
    d = m3500 if world == "m3500" else datasets.manhattan_dense(int(world[5:]), seed=1)
    p = _plan(d)
    N = d.n_nodes
    rng = np.random.default_rng(3)
    for name, (a, b) in candidate_sets(N, rng, 600).items():
        a, b = np.asarray(a, np.int32), np.asarray(b, np.int32)
        whole = path_doubles(p, sorted({int(x) for x in a} | {int(x) for x in b if x >= 0}))
        one = check_batches(p, a, b, 1 << 40)
        assert len(one) == 1, name  # everything fits: one batch
        many = check_batches(p, a, b, whole // 7)
        assert len(many) >= 7, (name, len(many))
        single = check_batches(p, a, b, 1)
        assert len(single) == len(a), name  # nothing fits: one candidate per batch
        if name == "newest_vs_old":
            # the newest pose is listed once per batch, however many candidates share it
            assert all(int((poses == N - 1).sum()) == 1 for _, _, poses, _, _ in many)


def test_batches_are_a_function_of_the_ids(m3500):
    """The same ids give the same batches; a candidate's batch does not depend on candidates after it."""
    p = _plan(m3500)
    rng = np.random.default_rng(8)
    a = rng.choice(m3500.n_nodes, 400).astype(np.int32)
    b = np.where(rng.random(400) < 0.3, -1, (a + 1 + rng.choice(100, 400)) % m3500.n_nodes).astype(np.int32)
    budget = path_doubles(p, np.unique(np.r_[a, b[b >= 0]])) // 5
    x = batches(p, a, b, budget)
    y = batches(p, a, b, budget)
    assert len(x) == len(y) and all(all(np.array_equal(u, v) for u, v in zip(s, t)) for s, t in zip(x, y))
    head = batches(p, a[:250], b[:250], budget)
    full_ends = [c1 for _, c1, *_ in x if c1 < 250]
    assert [c1 for _, c1, *_ in head][:-1] == full_ends


# ---------------------------------------------------------------------------------------------
# the residual helper
# ---------------------------------------------------------------------------------------------
def test_residual_helper_is_the_eval_hooks(built):
    """The residual of graph.c's helper equals, bit for bit, the r of the xyt state_eval / eval hooks and of the
    xytpos eval hook, headings on both sides of +-pi included."""
    from aprilsam_b200 import harness as H
    from support.hostplan import lib
    L = lib()
    L.asam_dbg_residual.argtypes = [_dp, _dp, _dp, _dp]
    L.asam_dbg_residual.restype = None
    rng = np.random.default_rng(2)
    n = 40
    P = np.c_[rng.normal(0, 20, (n, 2)), rng.uniform(-np.pi, np.pi, n)]
    P[:6, 2] = [np.pi - 1e-12, -np.pi + 1e-12, np.pi - 1e-3, -np.pi, 3.0, -3.0]
    W = np.diag([100.0, 50.0, 1000.0]).reshape(9)

    def helper(z, pa, pb=None):
        r = np.zeros(3)
        args = [np.ascontiguousarray(v, dtype=np.float64) for v in (z, pa)]
        pbp = np.ascontiguousarray(pb, dtype=np.float64).ctypes.data_as(_dp) if pb is not None else None
        L.asam_dbg_residual(args[0].ctypes.data_as(_dp), args[1].ctypes.data_as(_dp), pbp, r.ctypes.data_as(_dp))
        return r

    with H.Harness("b200") as h:
        for x in P:
            h.add_node(x)
        xyt = []
        for k in range(120):
            i, j = rng.choice(n, 2, replace=False)
            z = np.r_[rng.normal(0, 5, 2), rng.uniform(-4, 4)]
            xyt.append((h.add_xyt(int(i), int(j), z, W), int(i), int(j), z))
        pos = []
        for i in range(n):
            z = np.r_[rng.normal(0, 5, 2), rng.uniform(-4, 4)]
            pos.append((h.add_xytpos(i, z, W), i, z))
        st = h.states()
        for idx, i, j, z in xyt:
            r_state = h.eval(idx, True)[0]
            r_lp = h.eval(idx, False)[0]  # l_points = states before any solve
            assert np.array_equal(helper(z, st[i], st[j]).view(np.int64), r_state.view(np.int64)), idx
            assert np.array_equal(r_lp.view(np.int64), r_state.view(np.int64))
        for idx, i, z in pos:
            assert np.array_equal(helper(z, st[i]).view(np.int64), h.eval(idx)[0].view(np.int64)), idx


# ---------------------------------------------------------------------------------------------
# k_marginal_pairs' arithmetic
# ---------------------------------------------------------------------------------------------
def pair_kernel(Saa, Sab, Sbb, J, r, Winv):
    """k_marginal_pairs' epilogue in float64, in its order: (d2, Sigma_rel); Sab None for a prior."""
    if Sab is None:
        R = Saa.copy()
    else:
        S6 = np.block([[Saa, Sab], [Sab.T, Sbb]])
        JS = np.zeros((3, 6))
        for r_ in range(3):
            for c in range(6):
                acc = 0.0
                for k in range(6):
                    acc += J[r_, k] * S6[k, c]
                JS[r_, c] = acc
        R = np.zeros((3, 3))
        for r_ in range(3):
            for c in range(r_, 3):
                acc = 0.0
                for k in range(6):
                    acc += JS[r_, k] * J[c, k]
                R[r_, c] = R[c, r_] = acc
    S = R + Winv
    if not S[0, 0] > 0:
        return np.nan, R
    l00 = np.sqrt(S[0, 0]); l10 = S[1, 0] / l00; l20 = S[2, 0] / l00
    e11 = S[1, 1] - l10 * l10
    l11 = np.sqrt(e11) if e11 > 0 else np.nan
    l21 = (S[2, 1] - l20 * l10) / l11
    e22 = (S[2, 2] - l20 * l20) - l21 * l21
    l22 = np.sqrt(e22) if e22 > 0 else np.nan
    y0 = r[0] / l00
    y1 = (r[1] - l10 * y0) / l11
    y2 = ((r[2] - l20 * y0) - l21 * y1) / l22
    return (y0 * y0 + y1 * y1) + y2 * y2, R


def solve3_ld(S, r):
    """r' S^-1 r in long double (Gaussian elimination without pivoting; S symmetric positive definite)."""
    A = S.astype(LD).copy()
    x = r.astype(LD).copy()
    for k in range(3):
        for i in range(k + 1, 3):
            f = A[i, k] / A[k, k]
            A[i, k:] -= f * A[k, k:]
            x[i] -= f * x[k]
    y = np.zeros(3, dtype=LD)
    for i in (2, 1, 0):
        y[i] = (x[i] - A[i, i + 1:] @ y[i + 1:]) / A[i, i]
    return LD(r.astype(LD) @ y)


@pytest.mark.parametrize("world", ["m3500_300", "dense_600"])
def test_pair_formula_equals_dense_inverse(m3500, world):
    """d2 and Sigma_rel from the pair kernel's order on the float64 walk over emulated fronts equal the long-double
    definition from the dense inverse A^-1 of the emulated Hessian.  Bounds: the walk's Sigma is within
    eps = 0.1 kappa_1(A) u of A^-1 relative to max |Sigma| (test_walk_equals_dense_inverse); Sigma_rel then within
    eps max|Sigma_6| (|J| 1 1' |J|') + 8 u |J||Sigma_6||J|'; d2 within ||S^-1|| ||dS|| d2 + 8 kappa_2(S) u d2 (first
    order in the perturbation dS of S = Sigma_rel + W^-1)."""
    from aprilsam_b200 import datasets
    d = m3500.head(300) if world == "m3500_300" else datasets.manhattan_dense(600, seed=2)
    p, snap, A = _emulated(d)
    N = d.n_nodes
    inv = np.linalg.inv(A)
    kappa = np.linalg.cond(A, 1)
    eps = 0.1 * kappa * fc.U
    rng = np.random.default_rng(4)
    cands = [(N - 1, int(j)) for j in rng.choice(N - 1, 12, replace=False)] + \
            [tuple(int(x) for x in rng.choice(N, 2, replace=False)) for _ in range(12)] + \
            [(int(i), -1) for i in rng.choice(N, 6, replace=False)]
    lp = d.init  # the emulation linearises at init, which are also the states
    worst = {"rel": 0.0, "d2": 0.0}
    for a, b in cands:
        ids = [a] if b < 0 else [a, b]
        recs, _, _ = mc.paths(p, np.array(ids, np.int32))
        Sw, _ = mc.walk(snap, recs)
        q = snap.node2q[ids].astype(np.int64)
        idx = (3 * q[:, None] + np.arange(3)).reshape(-1)
        ref6 = inv[np.ix_(idx, idx)].astype(LD)
        Wm = np.diag(rng.uniform([50, 50, 500], [500, 500, 5000]))
        Wm[0, 1] = Wm[1, 0] = 0.3 * np.sqrt(Wm[0, 0] * Wm[1, 1])
        Winv = np.linalg.inv(Wm)
        Winv = np.triu(Winv) + np.triu(Winv, 1).T
        if b < 0:
            r = rng.normal(0, 0.05, 3)
            d2, R = pair_kernel(Sw[:3, :3], None, None, None, r, Winv)
            Jl = np.eye(3, dtype=LD)
        else:
            Ja, Jb, _ = emul.xyt_eval(lp[a], lp[b], np.zeros(3))
            J = np.hstack([Ja, Jb])
            r = rng.normal(0, 0.05, 3)
            d2, R = pair_kernel(Sw[:3, :3], Sw[:3, 3:], Sw[3:, 3:], J, r, Winv)
            Jl = J.astype(LD)
        assert np.array_equal(R, R.T)
        Rref = Jl @ ref6 @ Jl.T
        aJ = np.abs(Jl)
        scale = float(np.abs(ref6).max())
        bound_R = eps * scale * (aJ @ np.ones_like(ref6) @ aJ.T) + 8 * fc.U * (aJ @ np.abs(ref6) @ aJ.T)
        assert np.all(np.abs(R.astype(LD) - Rref) <= bound_R), (a, b)
        Sref = Rref + Winv.astype(LD)
        d2ref = solve3_ld(Sref, r)
        S64 = np.asarray(Sref, dtype=np.float64)
        Sinv = np.linalg.norm(np.linalg.inv(S64), 2)
        dS = np.linalg.norm(np.asarray(bound_R, dtype=np.float64), 2)
        bound_d2 = (Sinv * dS + 8 * np.linalg.cond(S64, 2) * fc.U) * float(d2ref)
        assert abs(d2 - float(d2ref)) <= bound_d2, (a, b, d2, float(d2ref), bound_d2)
        worst["rel"] = max(worst["rel"], float(np.max(np.abs(R.astype(LD) - Rref) / bound_R)))
        worst["d2"] = max(worst["d2"], abs(d2 - float(d2ref)) / bound_d2)
    print(f"CANDCPU {world} kappa {kappa:.2e} worst share of the bound {worst}")
