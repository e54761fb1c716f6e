"""Marginal covariances on the GPU (k_marginal_path / k_marginal_gram behind aprilsam_b200_marginal_covariance).

  1. hop by hop on the kernels' own intermediate results (tests/support/margcheck.py): every hop record equals the
     plan's root chain; every hop's local backward error, with its right-hand side rebuilt in long double from the
     kernel's z of the hop below; every Sigma_ij against Z_i'Z_j in long double; dinv against the fronts' pivots;
  2. the kernels against a float64 walk over the SAME fronts read back from HBM, entry by entry within
     MARG_C * u * (sum of |terms|), on worlds whose fronts reach every factorisation path and on worlds whose paths
     reach the path kernel's blocking edges (widths, rows below a block, path shapes, the 100 k world's 9 hops);
  3. end to end against columns of A^-1 from a sparse LU solve of the Hessian read back, within C * kappa_1 * u;
  4. exactly symmetric, bit-identical from call to call and with or without other poses in the request;
  5. a query changes nothing the solve path holds, and replays with queries take the same steps;
  6. the same after incremental steps; 7. the relative covariance against J Sigma J' in long double;
  8. the limits: the largest front the shared memory takes, a Gram grid beyond 2^20 CTAs, two graphs querying in
     turn in one process; 9. every error case.
"""
from __future__ import annotations

import ctypes as C
import json

import numpy as np
import pytest

from aprilsam_b200 import harness as H
from support import emul
from support import frontcheck as fc
from support import margcheck as mc
from test_gpu_kernels import _clique, _graph, _truth, add_priors, path_table, pendant_graph, pendant_sizes, zoo, zoo_graph

# observed worst on an H100 (80 GB, 700 W; every world of this file and the sharded job):
MARG_C = 4e4        # |Sigma_dev - Sigma_walk| <= MARG_C * u * sum |terms|     (observed 4.1e3 on the team-merged root: the
                    # rounding of the float64 walk grows along the path, which the terms of the final sum do not show;
                    # 2.2e5 through the hop of 2994 columns of the largest front, where only the hop checks apply)
HOP_C = 90.0        # local backward error of a hop, in u                       (observed 8.6)
GRAM_C = 90.0       # |Sigma_ij - Z_i'Z_j| / sum |terms|, in u                    (observed 8.6)
DINV_C = 30.0       # |dinv_k L_kk - 1|, in u                                     (observed 2.9)
FORWARD_C = 0.1     # |Sigma_dev - Sigma_ref| / |Sigma_ref| <= FORWARD_C * kappa_1 * u   (observed 0.0047)
REL_C = 8.0         # |relative_covariance - J Sigma J'| <= REL_C * u * |J||Sigma||J|'   (observed 0.76)


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


def assert_query(res):
    print("MARGCHECK " + json.dumps(res))
    assert res["hops_bad"] == 0 and res["transpose_bad"] == 0 and res["symmetric"], res
    assert res["hop"] <= HOP_C and res["gram"] <= GRAM_C and res["dinv"] <= DINV_C, res
    assert res.get("walk", 0.0) <= MARG_C, res
    assert res.get("forward_over_kappa_u", 0.0) <= FORWARD_C, res


def kernel_vs_walk(h, nodes=None, forward=True, snap=None, L=None, walk=True):
    L = L or fc.dev_api()
    snap = snap or fc.snapshot(h, L)
    nodes = pick_poses(h, snap) if nodes is None else np.asarray(nodes, dtype=np.int32)
    S, res = mc.query_report(h, L, snap, nodes)
    if walk:
        recs, _, _ = mc.paths(snap.plan, nodes)
        W, T = mc.walk(snap, recs)
        res["walk"] = float((np.abs(S - W) / np.maximum(fc.U * T, mc.TINY)).max())
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
    assert_query(res)
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
        _all_dinv(h)
        # a general-fallback step: a factor between two solved poses
        h.add_xyt(10, 350, m3500.ez[0], np.diag([100.0, 100.0, 1000.0]).reshape(9))
        h.inc()
        kernel_vs_walk(h, [399, 10, 350, 0])
        _all_dinv(h)


def _all_dinv(h):
    """dinv of every supernode after a replay: columns kept from earlier steps (keep > 0) as well."""
    L = fc.dev_api()
    snap = fc.snapshot(h, L)
    dinv = mc.read_dinv(L, L.asam_dbg_dev_of_graph(h.graph_ptr()), len(snap.q2node))
    e = mc.dinv_errors(snap, dinv, range(snap.nsn))
    print(f"MARGCHECK dinv of all {snap.nsn} supernodes {e:.2f} u")
    assert e <= DINV_C, e


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


# ---------------------------------------------------------------------------------------------
# the path kernel's edges (tests/test_marginal_cpu.py checks on host plans that these requests reach them)
# ---------------------------------------------------------------------------------------------
EDGE_WORLDS = {"c99": (33, 21, 2), "r42": (4, 42, 2), "r43": (4, 43, 2), "wide": (120, 120, 120), "pendants": None}
WIDTHS = (3, 24, 27, 96, 99, 192, 195, 285)  # hop widths c - js: 1 and 8 columns of a 24-column group, one block...


def edge_world(name):
    return pendant_graph(pendant_sizes()) if name == "pendants" else zoo_graph(*EDGE_WORLDS[name], seed=len(name))


def edge_poses(plan):
    """The newest and the oldest pose; in the three widest supernodes below a root, the poses at j0 = c - w for
    every width w of WIDTHS that fits; the first pose of every root, of the first and the last child of the root
    and of the first and the last leaf (warp) supernode."""
    d = plan.descs()
    q2n = plan.array("q2node")
    par = d["parent"]
    nsn = len(par)
    out = [len(q2n) - 1, 0]
    for s in sorted((s for s in range(nsn) if par[s] >= 0), key=lambda s: (-int(d["cb"][s]), s))[:3]:
        c, first = 3 * int(d["cb"][s]), int(d["first"][s])
        out += [int(q2n[first + (c - w) // 3]) for w in WIDTHS if w <= c]
    firsts = [s for s in range(nsn) if par[s] < 0]
    kids = [s for s in range(nsn) if par[s] >= 0 and par[par[s]] < 0]
    leaf = [int(s) for s in plan.array("leaf_tasks")]
    firsts += kids[:1] + kids[-1:] if len(kids) > 1 else []
    firsts += leaf[:1] + leaf[-1:]
    out += [int(q2n[int(d["first"][s])]) for s in firsts]
    return np.array(out, dtype=np.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(EDGE_WORLDS))
def test_path_kernel_edges(name):
    from test_gpu_kernels import plan_of
    d = edge_world(name)
    host = plan_of(d)
    want = mc.coverage(host, edge_poses(host), host.array("leaf_tasks"))
    with H.Harness("b200") as h:
        h.load_full(d)
        add_priors(h, d)
        h.batch()
        L = fc.dev_api()
        snap = fc.snapshot(h, L)
        nodes = edge_poses(snap.plan)
        assert mc.coverage(snap.plan, nodes, snap.leaf_tasks) == want  # the live plan reaches what the host plan does
        kernel_vs_walk(h, nodes, forward=name != "pendants", snap=snap, L=L)


def _path_snapshot(h, L, nodes):
    """A Snapshot holding only the fronts on the root paths of `nodes` (worlds too large to read whole)."""
    plan = fc.borrowed_plan(L, h.param_ptr())
    recs, _, _ = mc.paths(plan, nodes)
    desc = plan.descs()
    which = sorted({s for r in recs for s in mc.chain(desc, r["sn0"])})
    dev = L.asam_dbg_dev_of_graph(h.graph_ptr())
    return fc.Snapshot(plan, None, None, None, fc.read_fronts(L, dev, desc, which), None, None)


@pytest.mark.gpu
def test_dense_100k_nine_hops(built):
    """The oldest pose (9 hops), the newest (1) and 62 random poses of the dense 100 k world."""
    from aprilsam_b200 import datasets
    d = datasets.manhattan_dense(100000, seed=1)
    rng = np.random.default_rng(11)
    nodes = np.r_[0, d.n_nodes - 1, rng.choice(np.arange(1, d.n_nodes - 1), 62, replace=False)].astype(np.int32)
    with H.Harness("b200") as h:
        h.load_full(d)
        h.batch()
        L = fc.dev_api()
        snap = _path_snapshot(h, L, nodes)
        assert {len(mc.chain(snap.desc, r["sn0"])) for r in mc.paths(snap.plan, nodes[:2])[0]} == {1, 9}
        kernel_vs_walk(h, nodes, forward=False, snap=snap, L=L)


# ---------------------------------------------------------------------------------------------
# limits: shared memory, a large request, two graphs in one process
# ---------------------------------------------------------------------------------------------
def max_order(optin_bytes):
    """The largest front order m (a multiple of 3) with ASAM_MSMEM(m) doubles within optin_bytes."""
    fixed = mc.BSW * (mc.BSW + 1) + mc.BSW + 4 * mc.MROWS * 3
    m = (optin_bytes // 8 - fixed) // 6
    return m - m % 3


def smem_graph():
    """A front below the root of m = 3018 (c = 30), the largest the path kernel takes on an H100."""
    return zoo_graph(10, 996, 2, seed=1)


def clique_graph():
    """One front of m = 3021: one pose more than the shared memory of an H100 takes."""
    rng = np.random.default_rng(2)
    n = 1007
    return _graph(rng, _truth(rng, n), np.vstack([_clique(np.arange(n)), np.c_[np.arange(n - 1), np.arange(1, n)]]))


def _optin():
    import torch
    return int(torch.cuda.get_device_properties(0).shared_memory_per_block_optin)


@pytest.mark.gpu
def test_largest_front_the_shared_memory_takes(built):
    m_max = max_order(_optin())
    d = smem_graph()
    with H.Harness("b200") as h:
        h.load_full(d)
        h.batch()
        L = fc.dev_api()
        snap = fc.snapshot(h, L)
        assert snap.plan.info()["max_m"] == m_max, (snap.plan.info()["max_m"], m_max)
        s = next(s for s in range(snap.nsn) if 3 * int(snap.desc["mb"][s]) == m_max)
        first, c = int(snap.desc["first"][s]), 3 * int(snap.desc["cb"][s])
        nodes = [int(snap.q2node[first]), int(snap.q2node[first + c // 3 - 1]), d.n_nodes - 1, 0]
        kernel_vs_walk(h, nodes, snap=snap, L=L, walk=False)  # the walk's own rounding: see MARG_C
    with H.Harness("b200") as h:
        h.load_full(clique_graph())
        h.batch()
        for _ in range(2):
            with pytest.raises(RuntimeError, match="need .* KB of shared memory, the device offers"):
                h.marginal_covariance([0, 5])
        st = h.states().copy()
        h.batch()  # still solves
        assert np.all(np.isfinite(h.states())) and st.shape == h.states().shape
    with H.Harness("b200") as h:  # and the next graph still queries
        h.load_full(d.head(300))
        h.batch()
        h.marginal_covariance([0, 299])


@pytest.mark.gpu
def test_large_request(built):
    """1025 poses of dense2000: a Gram grid of more than 2^20 CTAs.  Every block against the float64 walk, a sample
    of blocks and poses hop by hop in long double; 65536 poses are refused before `out` is touched."""
    from aprilsam_b200 import datasets
    d = datasets.manhattan_dense(2000, seed=1)
    rng = np.random.default_rng(4)
    nodes = rng.choice(d.n_nodes, 1025, replace=False).astype(np.int32)
    n = len(nodes)
    assert n * n > 1 << 20
    with H.Harness("b200") as h:
        h.load_full(d)
        h.batch()
        L = fc.dev_api()
        snap = fc.snapshot(h, L)
        pairs = [(0, 0), (0, n - 1), (n - 1, n - 1)] + [tuple(sorted(p)) for p in rng.integers(0, n, (200, 2))]
        S, res = mc.query_report(h, L, snap, nodes, pairs=pairs, hop_poses=rng.choice(n, 64, replace=False))
        recs, _, _ = mc.paths(snap.plan, nodes)
        W, T = _dense_walk(snap, recs)
        res["walk"] = float((np.abs(S - W) / np.maximum(fc.U * T, mc.TINY)).max())
        assert_query(res)
        lib = H._load("b200")
        big = np.zeros(65536, dtype=np.int32)
        out = np.full(64, 7.0)
        assert lib.h_marginal_cov(h.h, len(big), big.ctypes.data_as(C.POINTER(C.c_int)),
                                  out.ctypes.data_as(C.POINTER(C.c_double))) == -1
        assert "invalid arguments" in lib.aprilsam_b200_last_error().decode()
        assert np.all(out == 7.0)


def _dense_walk(snap, recs):
    """mc.walk for many poses: the float64 columns of L^-1 of every pose in one dense matrix over the rows of the
    supernodes on their paths (zero above js), Sigma = Z'Z and the sum of |terms| = |Z|'|Z|."""
    rows = {}
    for r in recs:
        for s in mc.chain(snap.desc, r["sn0"]):
            rows.setdefault(s, len(rows))
    base = np.cumsum([0] + [3 * int(snap.desc["cb"][s]) for s in rows])
    Z = np.zeros((int(base[-1]), 3 * len(recs)))
    for i, r in enumerate(recs):
        for s, js, z in mc.pose_columns(snap, r):
            o = int(base[rows[s]])
            Z[o + js:o + 3 * int(snap.desc["cb"][s]), 3 * i:3 * i + 3] = z
    A = np.abs(Z)
    return Z.T @ Z, A.T @ A


@pytest.mark.gpu
def test_two_graphs_query_in_turn(m3500, built):
    """Graph A (the larger fronts) queries, then B, then A, then B, then A: every query succeeds and equals bit for bit
    the same query on the graph alone.  The shared-memory limit of k_marginal_path belongs to the function, not to a
    graph's context: B's query must not shrink it under A's next launch."""
    from aprilsam_b200 import datasets
    da = datasets.manhattan_dense(2000, seed=1)
    ids = {"a": np.array([0, 1999, 777, 1000], np.int32), "b": np.array([0, 3499, 1234], np.int32)}

    def live(d):
        h = H.Harness("b200")
        h.load_full(d)
        h.batch()
        return h

    with live(da) as ha:
        alone = ha.marginal_covariance(ids["a"])  # A's first query, no other graph in the process
        with live(m3500) as hb:
            ma = fc.borrowed_plan(fc.dev_api(), ha.param_ptr()).info()["max_m"]
            mb = fc.borrowed_plan(fc.dev_api(), hb.param_ptr()).info()["max_m"]
            assert ma > mb, (ma, mb)
            first_b = hb.marginal_covariance(ids["b"])
            for k, h, ref in (("a", ha, alone), ("b", hb, first_b), ("a", ha, alone)):
                got = h.marginal_covariance(ids[k])
                assert np.array_equal(got.view(np.int64), ref.view(np.int64)), k


@pytest.mark.gpu
def test_relative_covariance_long_double(built):
    """relative_covariance(a, b) = J Sigma J' in long double from marginal_covariance([a, b]) and the l_points,
    componentwise within REL_C u (|J||Sigma||J|'), headings within 1e-3 of +-pi included."""
    d0 = zoo("team162_c51")
    d = H.PoseGraphData(d0.truth.copy(), d0.ea, d0.eb, d0.ez, d0.eW, d0.truth.copy())  # l_points = truth
    with H.Harness("b200") as h:
        h.load_full(d)
        h.batch()
        lp = h.l_points()
        near = [int(i) for i in np.flatnonzero(np.pi - np.abs(lp[:, 2]) < 1e-3)]
        assert len(near) >= 2, near
        worst = 0.0
        for a, b in [(near[0], near[1]), (near[1], 0), (0, near[-1]), (3, d.n_nodes - 1), (10, 11)]:
            S6 = h.marginal_covariance([a, b]).astype(mc.LD)
            Ja, Jb, _ = emul.xyt_eval(lp[a], lp[b], np.zeros(3))
            J = np.hstack([Ja, Jb]).astype(mc.LD)
            ref = J @ S6 @ J.T
            scale = np.abs(J) @ np.abs(S6) @ np.abs(J).T
            got = h.relative_covariance(a, b)
            assert np.array_equal(got, got.T)
            worst = max(worst, float(np.max(np.abs(got.astype(mc.LD) - ref) / scale)) / fc.U)
        print(f"MARGCHECK relative covariance {worst:.2f} u")
        assert worst <= REL_C, worst
