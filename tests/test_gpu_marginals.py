"""Marginal covariances on the GPU (k_marginal_path / k_marginal_gram behind aprilsam_b200_marginal_covariance).

  1. the kernels against a float64 walk over the SAME fronts read back from HBM, entry by entry within
     MARG_C * u * (sum of |terms|), on worlds whose fronts reach every factorisation path;
  2. end to end against columns of A^-1 from a sparse LU solve of the Hessian read back, within C * kappa_1 * u;
  3. exactly symmetric, bit-identical from call to call and with or without other poses in the request;
  4. a query changes nothing the solve path holds, and replays with queries take the same steps;
  5. the same after incremental steps; 6. the relative covariance against numpy; 7. every error case.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from aprilsam_b200 import harness as H
from support import emul
from support import frontcheck as fc
from support import margcheck as mc
from test_gpu_kernels import add_priors, path_table, pendant_graph, pendant_sizes, zoo

MARG_C = 1e5        # |Sigma_dev - Sigma_walk| <= MARG_C * u * sum |terms|  (observed 2.4e3 on an H100: the rounding
                    # of the triangular solves grows along the path, which the terms of the final sum do not show)
FORWARD_C = 0.1     # |Sigma_dev - Sigma_ref| / |Sigma_ref| <= FORWARD_C * kappa_1 * u


def pick_poses(h, snap, extra=()):
    """Newest, oldest, first and last position of supernodes, j0 inside a 96-column block, one pose below every
    kind of front and a repeated id."""
    d = snap.desc
    q2n = snap.q2node
    N = len(q2n)
    out = [N - 1, 0]
    paths = {}
    for s, (kind, m, c, _) in path_table(snap.plan).items():
        paths.setdefault(kind, s)
    for s in list(paths.values()) + [int(np.argmax(d["cb"]))]:
        first, cb = int(d["first"][s]), int(d["cb"][s])
        out += [int(q2n[first]), int(q2n[first + cb - 1])]
        if cb > 32:
            out.append(int(q2n[first + 16]))  # j0 = 48: middle of the first 96-column block
    out += list(extra)
    out.append(out[2])
    return np.array(out, dtype=np.int32)


def kernel_vs_walk(h, nodes=None, forward=True):
    L = fc.dev_api()
    snap = fc.snapshot(h, L)
    nodes = pick_poses(h, snap) if nodes is None else np.asarray(nodes, dtype=np.int32)
    S = h.marginal_covariance(nodes)
    recs, _, _ = mc.paths(snap.plan, nodes)
    W, T = mc.walk(snap, recs)
    tiny = np.finfo(float).tiny
    res = {"walk": float((np.abs(S - W) / np.maximum(fc.U * T, tiny)).max()), "n": len(nodes)}
    assert np.array_equal(S, S.T), "not exactly symmetric"
    if forward:
        import scipy.sparse.linalg as spl
        ftype, fa, fb, _, _ = fc.factors_of(h)
        A, _ = fc.system(snap, ftype, fa, fb, snap.plan.array("fslot"))
        q = snap.node2q[nodes].astype(np.int64)
        idx = (3 * q[:, None] + np.arange(3)).reshape(-1)
        E = np.zeros((A.shape[0], len(idx)))
        E[idx, np.arange(len(idx))] = 1.0
        X = spl.splu(A.tocsc()).solve(E)
        ref = X[idx]
        _, kappa = fc.reference_solution(A, E[:, 0], steps=0)
        res["forward_over_kappa_u"] = float(np.abs(S - ref).max() / np.abs(ref).max() / (kappa * fc.U))
    print("MARGCHECK " + str(res))
    assert res["walk"] <= MARG_C, res
    assert res.get("forward_over_kappa_u", 0.0) <= FORWARD_C, res
    return S


WORLDS = ["m3500", "smem159_c12", "team162_c51", "bs_195", "wide", "pendants", "dense2000"]


def world(name, m3500):
    from aprilsam_b200 import datasets
    if name == "m3500":
        return m3500
    if name == "pendants":
        return pendant_graph(pendant_sizes())
    if name == "dense2000":
        return datasets.manhattan_dense(2000, seed=1)
    return zoo(name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", WORLDS)
def test_kernel_and_end_to_end(m3500, name):
    d = world(name, m3500)
    with H.Harness("b200") as h:
        h.load_full(d)
        if name != "m3500":
            add_priors(h, d)
        h.batch()
        kernel_vs_walk(h, forward=name not in ("pendants",))


@pytest.mark.gpu
def test_exact_repeatable_and_independent(m3500):
    with H.Harness("b200") as h:
        h.load_full(m3500)
        h.batch()
        rng = np.random.default_rng(5)
        ids = rng.choice(m3500.n_nodes, 64, replace=False).astype(np.int32)
        S1 = h.marginal_covariance(ids)
        S2 = h.marginal_covariance(ids)
        assert np.array_equal(S1.view(np.int64), S2.view(np.int64))
        assert np.array_equal(S1, S1.T)
        for a, b in ((0, 0), (3, 17), (63, 1)):
            alone = h.marginal_covariance([ids[a], ids[b]]) if a != b else h.marginal_covariance([ids[a]])
            blk = S1[3 * a:3 * a + 3, 3 * b:3 * b + 3]
            got = alone[0:3, 3:6] if a != b else alone
            assert np.array_equal(got.view(np.int64), blk.view(np.int64)), (a, b)


def _device_state(h):
    L = fc.dev_api()
    snap = fc.snapshot(h, L)
    dev = L.asam_dbg_dev_of_graph(h.graph_ptr())
    parts = [snap.Adiag, snap.Aoff, snap.B, snap.y, snap.x] + [snap.fronts[s][k] for s in sorted(snap.fronts) for k in (0, 1)]
    return [np.ascontiguousarray(p).view(np.int64).copy() for p in parts], dev


@pytest.mark.gpu
def test_query_changes_nothing(m3500):
    with H.Harness("b200") as h:
        h.load_full(m3500.head(1500))
        h.batch()
        before, _ = _device_state(h)
        st = h.states().copy(); lp = h.l_points().copy()
        h.marginal_covariance(np.arange(0, 1500, 7))
        h.relative_covariance(3, 1400)
        after, _ = _device_state(h)
        assert all(np.array_equal(a, b) for a, b in zip(before, after))
        assert np.array_equal(st, h.states()) and np.array_equal(lp, h.l_points())


@pytest.mark.gpu
def test_replay_with_queries_takes_the_same_steps(m3500):
    d = m3500.head(600)
    runs = []
    for query in (False, True):
        with H.Harness("b200") as h:
            h.replay_begin(d)
            infos = []
            for k in range(50, 601, 50):
                _, _, inf = h.replay_to(k)
                infos.append(inf.copy())
                if query:
                    h.marginal_covariance([0, k - 1])
            runs.append((h.states().copy(), infos))
    (s0, i0), (s1, i1) = runs
    assert all(np.array_equal(a, b) for a, b in zip(i0, i1))
    diff = s0 - s1
    diff[:, 2] = emul.mod2pi(diff[:, 2])
    assert np.abs(diff).max() < 1e-9


@pytest.mark.gpu
def test_after_incremental_steps(m3500):
    with H.Harness("b200") as h:
        h.replay_begin(m3500.head(400))
        h.replay_to(400)
        kernel_vs_walk(h, [399, 0, 200, 398, 57, 57])
        # a general-fallback step: a factor between two solved poses
        h.add_xyt(10, 350, m3500.ez[0], np.diag([100.0, 100.0, 1000.0]).reshape(9))
        h.inc()
        kernel_vs_walk(h, [399, 10, 350, 0])


@pytest.mark.gpu
def test_appends_into_team_merged_root(built):
    from aprilsam_b200 import datasets
    d = datasets.manhattan_dense(2000, seed=1)
    with H.Harness("b200") as h:
        h.replay_begin(d)
        h.replay_to(1900, batch_only=True)
        h.replay_to(2000)
        kernel_vs_walk(h)


def _relative_ref(h, a, b, S6):
    lp = h.l_points()
    Ja, Jb, _ = emul.xyt_eval(lp[a], lp[b], np.zeros(3))
    J = np.hstack([Ja, Jb])
    return J @ S6 @ J.T


@pytest.mark.gpu
@pytest.mark.parametrize("prior", [True, False])
def test_relative_covariance(m3500, prior):
    d = m3500.head(500)
    with H.Harness("b200") as h:
        if prior:
            h.load_full(d)
        else:
            for p in d.init:
                h.add_node(p)
            for a, b, z, W in zip(d.ea, d.eb, d.ez, d.eW):
                h.add_xyt(int(a), int(b), z, W)
        h.batch()
        L = fc.dev_api()
        snap = fc.snapshot(h, L)
        ftype, fa, fb, _, _ = fc.factors_of(h)
        A, _ = fc.system(snap, ftype, fa, fb, snap.plan.array("fslot"))
        import scipy.sparse.linalg as spl
        for a, b in ((10, 480), (499, 0), (250, 251)):
            q = snap.node2q[[a, b]].astype(np.int64)
            idx = (3 * q[:, None] + np.arange(3)).reshape(-1)
            E = np.zeros((A.shape[0], 6)); E[idx, np.arange(6)] = 1.0
            S6 = spl.splu(A.tocsc()).solve(E)[idx]
            ref = _relative_ref(h, a, b, S6)
            got = h.relative_covariance(a, b)
            assert np.array_equal(got, got.T)
            err = np.abs(got - ref).max() / np.abs(ref).max()
            print(f"MARGREL prior={prior} ({a},{b}) err {err:.2e}")
            assert err < 1e-6, (a, b, err)


@pytest.mark.gpu
def test_errors_leave_the_solver_usable(m3500):
    lib = H._load("b200")
    d = m3500.head(300)
    with H.Harness("b200") as h:
        out = np.zeros(9 * 4)
        ids = np.array([0, 1], dtype=np.int32)
        dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int)
        # before any solve: no solver behind param
        h.replay_begin(d)
        with pytest.raises(RuntimeError, match="does not continue a solve"):
            h.marginal_covariance([0])
        h.replay_to(200)
        assert lib.h_marginal_cov(h.h, 0, ids.ctypes.data_as(ip), out.ctypes.data_as(dp)) == -1
        assert lib.h_marginal_cov(h.h, 2, None, out.ctypes.data_as(dp)) == -1
        assert lib.h_relative_cov(h.h, 0, 1, None) == -1
        for bad in ([-1], [200], [0, 10**6]):
            with pytest.raises(RuntimeError, match="not in the solved graph"):
                h.marginal_covariance(bad)
        with pytest.raises(RuntimeError, match="not in the solved graph"):
            h.relative_covariance(0, 200)
        h.replay_to(250)
        h.marginal_covariance([0, 249])
        h.invalidate_plan()
        with pytest.raises(RuntimeError, match="plan was dropped"):
            h.relative_covariance(0, 5)
        h.batch()
        h.marginal_covariance([0, 249])
        n = h.n_nodes
        h.add_node(h.states()[n - 1])
        with pytest.raises(RuntimeError, match="added since the last solve"):
            h.marginal_covariance([0])
        h.add_xyt(n - 1, n, np.zeros(3), np.diag([100.0, 100.0, 1000.0]).reshape(9))
        h.inc()
        kernel_vs_walk(h, [n, 0, 150])
        h.batch()
        kernel_vs_walk(h, [n, 0, 150])
