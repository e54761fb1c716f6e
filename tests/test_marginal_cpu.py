"""Marginal covariances without a GPU: the root paths plan_marginal_paths gives, and the walk over them on fronts
of the numpy emulation against the dense inverse of the emulated Hessian."""
from __future__ import annotations

import numpy as np
import pytest

from support import emul
from support import frontcheck as fc
from support import margcheck as mc
from support.hostplan import HostPlan

PRIOR_W = np.array([1e4, 0, 0, 0, 1e4, 0, 0, 0, 1e3])


def _factors(d):
    ftype = np.r_[2, np.ones(d.n_edges, dtype=np.int32)].astype(np.int32)
    fa = np.r_[0, d.ea].astype(np.int32)
    fb = np.r_[-1, d.eb].astype(np.int32)
    return ftype, fa, fb


def _plan(d):
    return HostPlan().build(d.n_nodes, *_factors(d))


def _check_paths(p, nodes):
    recs, ztot, htot = mc.paths(p, nodes)
    d = p.descs()
    n2q = p.array("node2q")
    used = 0
    ext = np.zeros(len(recs), dtype=np.int64)
    for k, (node, r) in enumerate(zip(nodes, recs)):
        q = int(n2q[node])
        s0 = int(r["sn0"])
        assert int(d["first"][s0]) <= q < int(d["first"][s0]) + int(d["cb"][s0])
        assert int(r["j0"]) == 3 * (q - int(d["first"][s0]))
        ch = mc.chain(d, s0)
        assert int(r["nhop"]) == len(ch) and int(d["parent"][ch[-1]]) == -1
        assert int(r["hop0"]) == used
        used += len(ch)
        ext[k] = sum(3 * (3 * int(d["cb"][s]) - (int(r["j0"]) if h == 0 else 0)) for h, s in enumerate(ch))
    assert used == htot
    # scratch ranges: consecutive, disjoint, adding up to the total
    off = recs["zoff"].astype(np.int64)
    assert off[0] == 0 and np.all(off[1:] == off[:-1] + ext[:-1]) and off[-1] + ext[-1] == ztot


def test_paths_m3500(m3500):
    p = _plan(m3500)
    _check_paths(p, np.arange(m3500.n_nodes))


@pytest.mark.parametrize("n", [2000, 12000])
def test_paths_dense(built, n):
    from aprilsam_b200 import datasets
    d = datasets.manhattan_dense(n, seed=1)
    p = _plan(d)
    rng = np.random.default_rng(0)
    nodes = np.r_[0, n - 1, rng.integers(0, n, 300), 7, 7]
    _check_paths(p, nodes)


def test_paths_reject_bad_nodes(m3500):
    p = _plan(m3500)
    for bad in (-1, m3500.n_nodes):
        with pytest.raises(ValueError, match="not in the solved graph"):
            mc.paths(p, [0, bad])


def _emulated(d, lam=1e-4):
    p = _plan(d)
    info = p.info()
    ftype, fa, fb = _factors(d)
    fz = np.vstack([[0, 0, 0], d.ez]); fW = np.vstack([PRIOR_W, d.eW])
    Hs = emul.Hessian(d.n_nodes, info["n_slots"]); Hs.reset(d.n_nodes, lam)
    Hs.linearize(range(len(ftype)), ftype, fa, fb, fz, fW, d.init, d.init, p.array("node2q"), p.array("fslot"))
    fr = emul.Fronts(); fr.ensure(d.n_nodes)
    emul.factor(fr, Hs, p.descs(), p.array("ipool"), p.array("q2node"), p.array("tasks"), p.array("nwait"))
    emul.backsolve(fr, p.descs(), p.array("ipool"), p.array("btasks"))
    snap = fc.snapshot_from_emulation(p, Hs, fr)
    A, _ = fc.system(snap, ftype, fa, fb, p.array("fslot"))
    return p, snap, A.toarray()


@pytest.mark.parametrize("world", ["m3500_300", "dense_600"])
def test_walk_equals_dense_inverse(m3500, world):
    from aprilsam_b200 import datasets
    d = m3500.head(300) if world == "m3500_300" else datasets.manhattan_dense(600, seed=2)
    p, snap, A = _emulated(d)
    N = d.n_nodes
    rng = np.random.default_rng(1)
    nodes = np.r_[N - 1, 0, rng.integers(0, N, 20), 5, 5]
    recs, _, _ = mc.paths(p, nodes)
    S, _ = mc.walk(snap, recs)
    inv = np.linalg.inv(A)
    q = snap.node2q[nodes].astype(np.int64)
    idx = (3 * q[:, None] + np.arange(3)).reshape(-1)
    ref = inv[np.ix_(idx, idx)]
    kappa = np.linalg.cond(A, 1)
    err = np.abs(S - ref).max() / np.abs(ref).max()
    print(f"MARGCPU {world} err {err:.2e} kappa {kappa:.2e}")
    assert err <= 0.1 * kappa * fc.U, (err, kappa)


# ---------------------------------------------------------------------------------------------
# the hop-by-hop checks of the GPU tests catch wrong hops; the GPU worlds reach the kernels' edges
# ---------------------------------------------------------------------------------------------
def test_checker_catches_wrong_hops(built):
    """k_marginal_path's order restated in float64 on fronts of the numpy emulation passes every check; a dropped
    24-column group of one 128-row pass, a row scattered to the neighbouring parent row, a column solved with the
    previous block's reciprocal pivot and a Gram block without its lowest shared supernode each fail by more than
    100x the bound."""
    from test_gpu_kernels import zoo
    from test_gpu_marginals import GRAM_C, HOP_C
    d = zoo("team162_c99")  # a front of c = 99, m = 162 (blocks [0, 96) and [96, 99), 66 and 63 rows below)
    p, snap, _ = _emulated(d)
    desc = snap.desc
    s = int(np.argmax(desc["cb"] * (desc["parent"] >= 0)))
    first, c, m = int(desc["first"][s]), 3 * int(desc["cb"][s]), 3 * int(desc["mb"][s])
    assert (c, m) == (99, 162)
    dinv = np.zeros(3 * d.n_nodes)
    for t in range(snap.nsn):
        ft, ct = 3 * int(desc["first"][t]), 3 * int(desc["cb"][t])
        dinv[ft:ft + ct] = 1.0 / np.diag(snap.fronts[t][0])[:ct]
    root = int(np.flatnonzero(desc["parent"] < 0)[0])
    nodes = np.r_[snap.q2node[first], snap.q2node[first + 20], snap.q2node[int(desc["first"][root])]]
    recs, zt, ht = mc.paths(p, nodes)
    hop = mc.expected_hops(desc, recs, ht)

    def run(fault=None, k=0):
        Z = np.zeros(zt)
        for i, r in enumerate(recs):
            z = mc.kernel_path(snap, r, dinv, fault if i == k else None)
            Z[int(r["zoff"]):int(r["zoff"]) + len(z)] = z
        return Z

    Z = run()
    assert mc.check_hops(desc, recs, hop) == 0
    hop_ok, _ = mc.worst_hop(snap, recs, Z)
    gram_ok, ntr = mc.gram_errors(recs, hop, Z, mc.gram(recs, hop, Z))
    assert hop_ok <= HOP_C * fc.U and gram_ok <= GRAM_C * fc.U and ntr == 0, (hop_ok / fc.U, gram_ok / fc.U, ntr)
    worst = {}
    # 1. pose 0 (j0 = 0), block [0, 96): column group [24, 48) lost in the pass over rows 96..161
    worst["drop"], _ = mc.worst_hop(snap, recs, run(("drop", 0, 0, 0, 1)))
    # 2. the tenth row of u (the first hop's rows below c) scattered to the next row of the parent
    worst["scatter"], _ = mc.worst_hop(snap, recs, run(("scatter", 0, 9)))
    # 3. column 96 (the first of the second block) solved with the reciprocal pivot of column 0
    worst["pivot"], _ = mc.worst_hop(snap, recs, run(("pivot", 0, 1, 0)))
    # 4. Sigma without the lowest shared supernode: s for poses 0 and 1, the root for the others
    worst["gram"], _ = mc.gram_errors(recs, hop, Z, mc.gram(recs, hop, Z, skip_lowest=True))
    print("MARGMUTANTS " + str({k: v / fc.U for k, v in worst.items()}))
    assert worst["drop"] > 100 * HOP_C * fc.U and worst["scatter"] > 100 * HOP_C * fc.U, worst
    assert worst["pivot"] > 100 * HOP_C * fc.U and worst["gram"] > 100 * GRAM_C * fc.U, worst


def test_edge_worlds_reach_the_kernel_edges(built):
    """The requests of the GPU edge tests, on host plans: hop widths c - js in {3, 24, 27, 96, 99} and beyond 192
    with (c - js) mod 96 in {0, 3, 93}; rows below a block m - be in {0, 63, 66, 126, 129}; paths of one hop and
    of nine (the oldest pose of the dense 100 k world); two poses of one supernode with different j0; a path that is
    a suffix of another; a pair sharing only the root; a path from a leaf (warp) supernode."""
    from aprilsam_b200 import datasets
    from test_gpu_kernels import plan_of
    from test_gpu_marginals import EDGE_WORLDS, edge_poses, edge_world
    tot = dict(width=set(), below=set(), nhop=set(), same_sn=False, suffix=False, root_only=False, leaf_start=False)
    for name in EDGE_WORLDS:
        p = plan_of(edge_world(name))
        cov = mc.coverage(p, edge_poses(p), p.array("leaf_tasks"))
        for k, v in cov.items():
            tot[k] = tot[k] | v
    d = datasets.manhattan_dense(100000, seed=1)
    p = plan_of(d)
    tot["nhop"] |= mc.coverage(p, [0, d.n_nodes - 1])["nhop"]
    assert tot["width"] >= {3, 24, 27, 96, 99}, tot
    assert {w % 96 for w in tot["width"] if w >= 192} >= {0, 3, 93}, tot
    assert tot["below"] >= {0, 63, 66, 126, 129}, tot
    assert tot["nhop"] >= {1, 9}, tot
    assert all(tot[k] for k in ("same_sn", "suffix", "root_only", "leaf_start")), tot


def test_shared_memory_edge_worlds(built):
    """zoo_graph(10, 996, 2) has a front below the root of exactly m = 3018 (the largest k_marginal_path takes with
    227 KB of shared memory per block); a 1007-pose clique has max_m = 3021."""
    from test_gpu_kernels import plan_of
    from test_gpu_marginals import clique_graph, max_order, smem_graph
    assert max_order(227 * 1024) == 3018
    p = plan_of(smem_graph())
    d = p.descs()
    assert p.info()["max_m"] == 3018
    assert any(3 * int(d["mb"][s]) == 3018 and d["parent"][s] >= 0 for s in range(len(d["mb"])))
    assert plan_of(clique_graph()).info()["max_m"] == 3021


def test_max_m_follows_appends(m3500, built, monkeypatch):
    """After every plan_append of the M3500 replay and of the appends under team roots, max_m (which sizes
    k_marginal_path's shared memory) is 3 max(mb)."""
    import test_gpu_incremental as ti
    seen = []
    append = HostPlan.append

    def checked(self, *a, **k):
        r = append(self, *a, **k)
        if r is not None:
            seen.append((self.info()["max_m"], 3 * int(self.descs()["mb"].max())))
        return r

    monkeypatch.setattr(HostPlan, "append", checked)
    ti.a_steps_cpu(m3500, 400)
    for name in ti.B_GRAPHS:
        for depth in ti.B_DEPTHS:
            ti.emulate_script(ti.b_graph(name), ti.b_steps(depth))
    assert len(seen) > 400 and all(a == b for a, b in seen), [s for s in seen if s[0] != s[1]][:5]
