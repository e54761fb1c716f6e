"""Fronts that do not fit in shared memory and are factored by ONE CTA out of HBM (cta_front's HBM mode: staged
panel, tensor-pipe trailing update).  The batch schedule sends every front there whose team the level room scales
below two CTAs; ASAM_TEAM_ROOM=1 scales every team of a graph down that far, so the zoo graphs below put their
team-sized fronts on this path.

GPU tests check every front of such solves at the edges of the path (m just above the shared-memory limit, m where
the staged panel narrows below 48 columns, c = 3, c off the 12-column and panel grid, c over several panels, many
children, c = m) with the bounds of test_gpu_kernels.py: local backward error, y equal to the rhs rows bit for bit,
and a second factorisation bit-identical.  CPU tests check the routing of the host plan.
"""
from __future__ import annotations

import numpy as np
import pytest

from support import frontcheck as fc
from test_gpu_kernels import (_clique, _graph, _join, _truth, assert_solve_ok, batch_and_check, path_table, plan_of,
                              zoo, zoo_graph)

SOLO_ENV = {"ASAM_TEAM_ROOM": "1"}

# (a, r, b) of zoo_graph: first front c = 3a, m = 3(a + r); root front c = m = 3(b + r)
SOLO_ZOO = {
    "m162_c3": (1, 53, 2),
    "m162_c51": (17, 37, 2),
    "m165_c15": (5, 50, 2),
    "m168_c99": (33, 23, 2),
    "m555_c90": (30, 155, 2),   # staged panel of 36 columns: panels 36 + 36 + 18
    "m903_c60": (20, 281, 3),   # staged panel of 24 columns; root c = m = 852
}


def staged_width(m, smem_doubles=25600, solo_pb=48):
    """Widest staged panel of the HBM mode for a front of order m (cta_front: ldp = 4 mod 16 >= m + 2)."""
    ld = (m + 2) & ~1
    ldp = ((m + 2) & ~15) + (4 if ((m + 2) & 15) <= 4 else 20)
    pb = min((smem_doubles - (((ld + 1) // 2 + 2) & ~1)) // ldp, solo_pb)
    return pb - pb % 12 if pb >= 12 else pb - pb % 3


def many_children_graph(seed=5, k=48):
    """A root clique of 56 poses (with one more pose: c = m = 171, just too large for shared memory) with k pendant
    cliques of 3 poses, each joined to two poses of the root: one front in HBM with k children."""
    rng = np.random.default_rng(seed)
    n_root = 56
    pairs = [_clique(np.arange(n_root)), np.c_[np.arange(n_root - 1), np.arange(1, n_root)]]
    nxt = n_root
    for i in range(k):
        ids = np.arange(nxt, nxt + 3)
        nxt += 3
        pairs += [_clique(ids), _join(ids, [(2 * i) % n_root, (2 * i + 7) % n_root])]
    return _graph(rng, _truth(rng, nxt), np.vstack(pairs))


def solo_graph(name):
    if name == "many_children":
        return many_children_graph()
    return zoo_graph(*SOLO_ZOO[name], seed=len(name))


def hbm_fronts(d, env=SOLO_ENV):
    return [f for f in path_table(plan_of(d, env)).values() if f[0] == "cta_hbm"]


# ---------------------------------------------------------------------------------------------
# CPU: the graphs reach the edges they are meant to; the plan routes teams of one to cta_front
# ---------------------------------------------------------------------------------------------
def test_solo_zoo_covers_the_edges(built):
    fronts = {name: hbm_fronts(solo_graph(name)) for name in list(SOLO_ZOO) + ["many_children"]}
    mc = {(m, c) for fs in fronts.values() for _, m, c, _ in fs}
    assert {(162, 3), (162, 51), (165, 15), (168, 99), (555, 90), (903, 60)} <= mc, sorted(mc)
    assert staged_width(162) == 48 and staged_width(555) == 36 and staged_width(903) == 24
    assert any(c == m and c > 2 * staged_width(m) for m, c in mc)  # root fronts: c = m over several panels
    assert {c % 12 for _, c in mc} >= {3, 6}
    assert max(ch for _, m, c, ch in fronts["many_children"] if m == c) >= 40


def _G_by_sn(p):
    G = {}
    for s, w in zip(p.array("tasks"), p.array("nwait")):
        G.setdefault(int(s), (int(w) >> 24) & 0x7F)
    return G


def _assert_topological(p):
    d = p.descs()
    parent = d["parent"]
    pos = {}
    for k, s in enumerate(p.array("tasks")):
        pos.setdefault(int(s), k)
    for s, k in pos.items():
        par = int(parent[s])
        if par >= 0 and par in pos:
            assert pos[par] > k, (s, par)


@pytest.mark.parametrize("world", ["zoo_room1", "manhattan_dense_100k"])
def test_teams_of_one_go_to_cta_front(built, world):
    """Against the plan with ASAM_TEAM_MIN=1 (teams of one kept on the team code, G = 1): every front that does not
    fit in shared memory and has a team of one there gets task word G = 0; every other front keeps its team size."""
    if world == "zoo_room1":
        d, env = zoo("wide"), SOLO_ENV
    else:
        from aprilsam_b200 import datasets
        d, env = datasets.manhattan_dense(100000, seed=1), {}
    new, old = plan_of(d, env), plan_of(d, {**env, "ASAM_TEAM_MIN": "1"})
    Gn, Go = _G_by_sn(new), _G_by_sn(old)
    assert Gn.keys() == Go.keys()
    mb = new.descs()["mb"]
    routed = 0
    for s, g in Go.items():
        if g == 1:
            assert not fc.fits_smem(int(mb[s])) and Gn[s] == 0, (s, g, Gn[s])
            routed += 1
        else:
            assert Gn[s] == g, (s, g, Gn[s])
    assert routed > (500 if world != "zoo_room1" else 0)
    assert sorted(new.array("tasks")) == sorted(old.array("tasks"))
    _assert_topological(new)


# ---------------------------------------------------------------------------------------------
# GPU: every front of solves through the single-CTA HBM path
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SOLO_ZOO) + ["many_children"])
def test_solo_fronts(name):
    res = batch_and_check(solo_graph(name), SOLO_ENV, forward=(name not in ("m903_c60",)))
    assert "cta_hbm" in res["per_path"], res["paths"]
    assert_solve_ok(res, f"solo {name}")


@pytest.mark.gpu
def test_solo_manhattan_100k():
    """The 100 k dense world with its default schedule: 800-odd teams of one on the single-CTA path."""
    from aprilsam_b200 import datasets
    d = datasets.manhattan_dense(100000, seed=1)
    assert len(hbm_fronts(d, {})) > 500
    res = batch_and_check(d, forward=False)
    assert "cta_hbm" in res["per_path"], res["paths"]
    assert_solve_ok(res, "manhattan_dense(100000)")
