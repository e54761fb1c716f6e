"""Candidate compatibility (aprilsam_b200_candidate_compatibility) without a GPU.

  1. pair maths: a numpy restatement of k_marginal_compat's per-pair steps (the cross blocks of Sigma, C_ij = J_i Sigma
     J_j', S_ij from each candidate's S = Sigma_rel + W^-1, the 6 x 6 Cholesky in the kernel's order, d2 = |L^-1 r|^2)
     against a dense float64 solve, on an M3500 head of 1000 poses with Sigma = A^-1 dense;
  2. the chain rule, exact in the linear model: d2_ij = d2_i + d2_(j|i), d2_(j|i) the candidate distance of j against
     A + J_i' W_i J_i with r_j moved by that system's update (JCBB's sequential form), and d2_ij >= max(d2_i, d2_j);
  3. planted aliasing: two neighbouring closures across a long loop, each shifted so that its own d2 is 9 (inside the
     99 % gate with 3 degrees of freedom), fail jointly when they pull the drift in opposite directions and pass when
     they pull it the same way;
  4. the tiles plan_compat_tiles gives: every pair once, each tile within its budget or a single pair, a pure function.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from support import margcheck as mc
from test_audit_cpu import m3500_head, system, xyt_eval
from test_marginal_cpu import _plan

W_CAND = np.array([[400.0, 30.0, 0.0], [30.0, 250.0, 5.0], [0.0, 5.0, 2000.0]])
CHI2_3_99 = 11.34
CHI2_6_99 = 16.81
CHI2_6_999 = 22.46


def candidate(pts, a, b, r, W=W_CAND):
    """(pose ids, J (None for a prior), r, W^-1) of a candidate; J at pts."""
    if b < 0:
        return ([a], None, np.asarray(r, float), np.linalg.inv(W))
    _, J = xyt_eval(pts[a], pts[b], np.zeros(3))
    return ([a, b], J, np.asarray(r, float), np.linalg.inv(W))


def sigma_rel(Sig, c):
    ids, J, _, _ = c
    idx = np.concatenate([np.arange(3 * p, 3 * p + 3) for p in ids])
    S = Sig[np.ix_(idx, idx)]
    return S if J is None else J @ S @ J.T


def pair_kernel(Sig, ci, cj):
    """k_marginal_compat's epilogue in float64, in its order: (d2, C_ij), with Sigma_rel of each candidate symmetrised
    from its upper triangle as k_marginal_pairs leaves it."""
    (pi, Ji, ri, Wi), (pj, Jj, rj, Wj) = ci, cj
    X = np.block([[Sig[3 * u:3 * u + 3, 3 * v:3 * v + 3] for v in pj] for u in pi])  # 3 ni x 3 nj
    ns = 3 * len(pj)
    if Ji is None:
        T = X[:3].copy()
    else:
        T = np.zeros((3, ns))
        for r in range(3):
            for c in range(ns):
                acc = 0.0
                for k in range(6):
                    acc += Ji[r, k] * X[k, c]
                T[r, c] = acc
    if Jj is None:
        Cm = T.copy()
    else:
        Cm = np.zeros((3, 3))
        for r in range(3):
            for c in range(3):
                acc = 0.0
                for k in range(6):
                    acc += T[r, k] * Jj[c, k]
                Cm[r, c] = acc
    Ri, Rj = (np.triu(sigma_rel(Sig, x)) + np.triu(sigma_rel(Sig, x), 1).T for x in (ci, cj))
    M = np.zeros((6, 6))
    M[:3, :3] = Ri + Wi
    M[3:, 3:] = Rj + Wj
    M[3:, :3] = Cm.T
    L = np.zeros((6, 6))
    for j in range(6):
        e = M[j, j]
        for k in range(j):
            e -= L[j, k] * L[j, k]
        L[j, j] = np.sqrt(e) if e > 0 else np.nan
        for i in range(j + 1, 6):
            v = M[i, j]
            for k in range(j):
                v -= L[i, k] * L[j, k]
            L[i, j] = v / L[j, j]
    rhs = np.r_[ri, rj]
    y = np.zeros(6)
    for i in range(6):
        v = rhs[i]
        for k in range(i):
            v -= L[i, k] * y[k]
        y[i] = v / L[i, i]
    d2 = y[0] * y[0]
    for i in range(1, 6):
        d2 += y[i] * y[i]
    return d2, Cm


def single_d2(Sig, c):
    R = sigma_rel(Sig, c)
    return float(c[2] @ np.linalg.solve(R + c[3], c[2]))


def dense_pair(Sig, ci, cj):
    """[r_i; r_j]' S_ij^-1 [r_i; r_j] and C_ij by dense float64 products and a dense solve."""
    idx = [np.concatenate([np.arange(3 * p, 3 * p + 3) for p in c[0]]) for c in (ci, cj)]
    Js = [np.eye(3) if c[1] is None else c[1] for c in (ci, cj)]
    Cm = Js[0] @ Sig[np.ix_(idx[0], idx[1])] @ Js[1].T
    S = np.block([[sigma_rel(Sig, ci) + ci[3], Cm], [Cm.T, sigma_rel(Sig, cj) + cj[3]]])
    v = np.r_[ci[2], cj[2]]
    return float(v @ np.linalg.solve(S, v)), Cm


# ---------------------------------------------------------------------------------------------
# 1. pair maths
# ---------------------------------------------------------------------------------------------
def test_pair_maths_against_dense_solve():
    d = m3500_head(1000)
    A, _, _ = system(d, d.init)
    Sig = np.linalg.inv(A)
    Sig = (Sig + Sig.T) / 2
    rng = np.random.default_rng(3)
    N = d.n_nodes
    cands = []
    for q in range(24):
        a = int(rng.integers(0, N))
        b = -1 if q % 4 == 3 else int((a + 1 + rng.integers(0, N - 1)) % N)
        cands.append(candidate(d.init, a, b, rng.normal(0, 0.5, 3)))
    worst = 0.0
    for i in range(len(cands)):
        for j in range(i + 1, len(cands)):
            d2, Cm = pair_kernel(Sig, cands[i], cands[j])
            ref, Cref = dense_pair(Sig, cands[i], cands[j])
            assert np.abs(Cm - Cref).max() <= 1e-10 * np.abs(Cref).max() + 1e-300, (i, j)
            rel = abs(d2 - ref) / ref
            worst = max(worst, rel)
            assert rel <= 1e-8, (i, j, d2, ref)
            # swapping the candidates transposes C and leaves d2
            d2s, Cs = pair_kernel(Sig, cands[j], cands[i])
            assert abs(d2s - d2) <= 1e-9 * d2 and np.abs(Cs - Cm.T).max() <= 1e-9 * np.abs(Cm).max()
    print(f"COMPATCPU pair maths: worst relative d2 difference {worst:.1e}")


def test_pair_of_priors_and_shared_poses():
    """Two priors use Sigma(a_i, a_j) alone; closures that share a pose use its diagonal block."""
    d = m3500_head(400)
    A, _, _ = system(d, d.init)
    Sig = np.linalg.inv(A)
    Sig = (Sig + Sig.T) / 2
    rng = np.random.default_rng(4)
    p1, p2 = candidate(d.init, 10, -1, rng.normal(0, 1, 3)), candidate(d.init, 300, -1, rng.normal(0, 1, 3))
    _, Cm = pair_kernel(Sig, p1, p2)
    assert np.array_equal(Cm, Sig[30:33, 900:903])
    c1, c2 = candidate(d.init, 5, 380, rng.normal(0, 1, 3)), candidate(d.init, 380, 7, rng.normal(0, 1, 3))
    d2, Cm = pair_kernel(Sig, c1, c2)
    ref, Cref = dense_pair(Sig, c1, c2)
    assert abs(d2 - ref) <= 1e-8 * ref and np.allclose(Cm, Cref, rtol=1e-9, atol=1e-12)
    # the same candidate twice: S_ij is singular in exact arithmetic only without W^-1; with it d2 is finite
    d2, _ = pair_kernel(Sig, c1, c1)
    assert np.isfinite(d2) and d2 >= single_d2(Sig, c1) * (1 - 1e-9)


# ---------------------------------------------------------------------------------------------
# 2. chain rule and bound
# ---------------------------------------------------------------------------------------------
def test_chain_rule_and_bound():
    # lambda = 1e-2 keeps A well enough conditioned for float64 inverses on both sides to hold 1e-9
    d = m3500_head(300)
    pts = d.init
    A, g, _ = system(d, pts, lam=1e-2)
    Sig = np.linalg.inv(A)
    x = Sig @ g
    rng = np.random.default_rng(12)
    N = d.n_nodes
    specs = [(299, int(rng.integers(0, 250))) for _ in range(6)] + \
        [(int(rng.integers(0, N)), int(rng.integers(0, N))) for _ in range(6)] + [(int(rng.integers(0, N)), -1)] * 3
    specs = [(a, b if b != a else (a + 1) % N) for a, b in specs]
    worst = 0.0
    for q, (a, b) in enumerate(specs):
        for q2, (a2, b2) in enumerate(specs):
            if q2 <= q:
                continue
            # linearised residuals at the update: r = z - h(pts) - J x with z drawn around the prediction
            ci = candidate(pts, a, b, np.zeros(3))
            cj = candidate(pts, a2, b2, np.zeros(3))
            re_i, re_j = rng.normal(0, 2, 3), rng.normal(0, 2, 3)
            Ji = np.eye(3) if ci[1] is None else ci[1]
            Jj = np.eye(3) if cj[1] is None else cj[1]
            ii = np.concatenate([np.arange(3 * p, 3 * p + 3) for p in ci[0]])
            ij = np.concatenate([np.arange(3 * p, 3 * p + 3) for p in cj[0]])
            ci = (ci[0], ci[1], re_i - Ji @ x[ii], ci[3])
            cj = (cj[0], cj[1], re_j - Jj @ x[ij], cj[3])
            d2_ij, _ = dense_pair(Sig, ci, cj)
            d2_i, d2_j = single_d2(Sig, ci), single_d2(Sig, cj)
            Wi = np.linalg.inv(ci[3])
            Ai = A.copy()
            Ai[np.ix_(ii, ii)] += Ji.T @ Wi @ Ji
            gi = g.copy()
            gi[ii] += Ji.T @ Wi @ re_i
            Sig_i = np.linalg.inv(Ai)
            xi = Sig_i @ gi
            cj_i = (cj[0], cj[1], re_j - Jj @ xi[ij], cj[3])
            d2_j_given_i = single_d2(Sig_i, cj_i)
            rel = abs(d2_ij - (d2_i + d2_j_given_i)) / d2_ij
            worst = max(worst, rel)
            assert rel <= 1e-9, (q, q2, d2_ij, d2_i, d2_j_given_i)
            assert d2_ij >= max(d2_i, d2_j) * (1 - 1e-12), (q, q2)
            d2_k, _ = pair_kernel(Sig, ci, cj)
            assert abs(d2_k - d2_ij) <= 1e-9 * d2_ij
    print(f"COMPATCPU chain rule: worst relative difference {worst:.1e}")


# ---------------------------------------------------------------------------------------------
# 3. planted aliasing
# ---------------------------------------------------------------------------------------------
def planted(Sig, ci, cj, sign):
    """Shift ci along the largest axis u of S_i and cj along the drift that u implies for it, C_ij' S_i^-1 u (times
    sign), each scaled so that its own d2 is 9.  Returns the two shifted candidates."""
    Si = sigma_rel(Sig, ci) + ci[3]
    Sj = sigma_rel(Sig, cj) + cj[3]
    _, Cm = dense_pair(Sig, ci, cj)
    u = np.linalg.eigh(Si)[1][:, -1]
    uj = sign * (Cm.T @ np.linalg.solve(Si, u))
    ri = 3.0 * u / np.sqrt(u @ np.linalg.solve(Si, u))
    rj = 3.0 * uj / np.sqrt(uj @ np.linalg.solve(Sj, uj))
    return (ci[0], ci[1], ri, ci[3]), (cj[0], cj[1], rj, cj[3])


ALIAS_LOOPS = ((200, 800), (300, 700))


def test_planted_aliasing():
    d = m3500_head(1000)
    A, _, _ = system(d, d.init)
    Sig = np.linalg.inv(A)
    Sig = (Sig + Sig.T) / 2
    for a, b in ALIAS_LOOPS:
        ci = candidate(d.init, a, b, np.zeros(3))
        cj = candidate(d.init, a + 1, b + 1, np.zeros(3))
        for sign in (-1.0, 1.0):
            pi, pj = planted(Sig, ci, cj, sign)
            d2_i, d2_j = single_d2(Sig, pi), single_d2(Sig, pj)
            assert abs(d2_i - 9.0) < 1e-9 and abs(d2_j - 9.0) < 1e-9
            assert d2_i < CHI2_3_99 and d2_j < CHI2_3_99
            joint, _ = pair_kernel(Sig, pi, pj)
            print(f"COMPATCPU alias ({a}, {b}) sign {sign:+.0f}: joint d2 {joint:.2f}")
            if sign < 0:
                assert joint > CHI2_6_999, (a, b, joint)
            else:
                assert joint < CHI2_6_99, (a, b, joint)


# ---------------------------------------------------------------------------------------------
# 4. tiles
# ---------------------------------------------------------------------------------------------
def tiles(plan, a, b, budget):
    L = plan.L
    ip = C.POINTER(C.c_int)
    L.asam_dbg_plan_compat_tiles.argtypes = [C.c_void_p, C.c_int, ip, ip, C.c_int64, ip, C.c_int]
    a = np.ascontiguousarray(a, dtype=np.int32)
    b = np.ascontiguousarray(b, dtype=np.int32)
    n = L.asam_dbg_plan_compat_tiles(plan.p, len(a), a.ctypes.data_as(ip), b.ctypes.data_as(ip), int(budget), None, 0)
    out = np.zeros((max(n, 1), 4), dtype=np.int32)
    m = L.asam_dbg_plan_compat_tiles(plan.p, len(a), a.ctypes.data_as(ip), b.ctypes.data_as(ip), int(budget),
                                     out.ctypes.data_as(ip), n)
    assert m == n
    return out[:n]


def tile_doubles(plan, a, b, t):
    i0, i1, j0, j1 = (int(v) for v in t)
    ids = np.r_[a[i0:i1], b[i0:i1], a[j0:j1], b[j0:j1]]
    poses = np.unique(ids[ids >= 0])
    return mc.paths(plan, poses.astype(np.int32))[1] + 10 * (i1 - i0) * (j1 - j0)


def check_tiles(plan, a, b, budget):
    ts = tiles(plan, a, b, budget)
    k = len(a)
    seen = np.zeros((k, k), dtype=np.int32)
    for t in ts:
        i0, i1, j0, j1 = (int(v) for v in t)
        assert 0 <= i0 < i1 <= k and 0 <= j0 < j1 <= k
        assert (i0, i1) == (j0, j1) or i1 <= j0, t
        blk = seen[i0:i1, j0:j1]
        if i0 == j0:
            blk[np.triu_indices(i1 - i0)] += 1
            npairs = (i1 - i0) * (i1 - i0 + 1) // 2
        else:
            blk += 1
            npairs = (i1 - i0) * (j1 - j0)
        assert npairs >= 1
        assert npairs == 1 or tile_doubles(plan, a, b, t) <= budget, (t, budget)
    assert np.array_equal(seen, np.triu(np.ones((k, k), dtype=np.int32))), "every pair i <= j exactly once"
    again = tiles(plan, a, b, budget)
    assert np.array_equal(ts, again)
    return ts


@pytest.mark.parametrize("world", ["m3500", "dense12000"])
def test_tiles(m3500, world):
    from aprilsam_b200 import datasets
    d = m3500 if world == "m3500" else datasets.manhattan_dense(12000, seed=1)
    p = _plan(d)
    N = d.n_nodes
    rng = np.random.default_rng(6)
    k = 160
    a = np.r_[np.full(k // 2, N - 1), rng.integers(0, N, k // 4), rng.integers(0, N, k - k // 2 - k // 4)]
    b = np.r_[rng.integers(0, N - 1, k // 2), rng.integers(0, N, k // 4), np.full(k - k // 2 - k // 4, -1)]
    b = np.where(a == b, (a + 1) % N, b)
    a, b = a.astype(np.int32), b.astype(np.int32)
    default = (256 << 20) // 8
    one = check_tiles(p, a, b, default)
    assert len(one) == 1 and tuple(one[0]) == (0, k, 0, k)
    whole = tile_doubles(p, a, b, (0, k, 0, k))
    for div in (2, 5, 17, 60):
        many = check_tiles(p, a, b, whole // div)
        assert len(many) > 1, div
    single = check_tiles(p, a[:30], b[:30], 1)  # below one pair: one pair per tile
    assert len(single) == 30 * 31 // 2
    # a block whose candidate alone exceeds its share pairs with the others one pair per tile
    big = mc.paths(p, np.array([N - 1, 0], np.int32))[1]
    check_tiles(p, a[:40], b[:40], 3 * big)
    # a pure function of the ids: a prefix tiles the same way at the default budget
    assert np.array_equal(tiles(p, a[:50], b[:50], default), [[0, 50, 0, 50]])


def test_layout_hook(built):
    """asam_debug_marginal_compat_layout: err and both outputs first, every table 256-byte aligned and in order."""
    from aprilsam_b200 import capi
    L = capi.lib()
    o = (C.c_int64 * 8)()
    L.asam_debug_marginal_compat_layout(7, 1000, 20, 12, 144, o)
    o = list(o)
    assert o[0] == 16 and o[1] == 16 + 10 * 12 * 8
    assert o[2] >= o[1] + 10 * 144 * 8 and all(v % 256 == 0 for v in o[2:])
    assert o == sorted(o) and o[7] >= o[6] + 2 * 12 * 4
