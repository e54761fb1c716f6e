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
