"""The factor maths of the host hooks against an exact reference over the edge corpus (-m "not gpu").

The eval hooks (host/graph.c: xyt_eval, xytpos_eval, robust_weigh) share the loss maths (include/asam_loss.h) with
k_linearize, k_step, k_hessian_rebuild and k_chi2_partial.  Here they are compared with support/factormath.py (mpmath)
on every factor of the corpus: r, J_a, J_b, W_eff = w W and chi2 = rho(s) within HOST_C u sum|terms|, and the loss on
its own within 4 ulp of the exact w(s), rho(s) (or DBL_MIN below DBL_MIN) for every accepted k.  Inside the band where
k^2 and s / k^2 are normal the Cauchy maths is bit for bit the formula it always was.
"""
import math

import numpy as np
import pytest

from aprilsam_b200 import harness as H
from support import factormath as fm

HOST_C = 32.0  # hooks vs exact, in u sum|terms|  (observed 3.2: x86-64, gcc 13.3 -O2, glibc 2.39 libm)
LOSS_ULPS = 4.0


def harness_of(g):
    h = H.Harness("b200")
    for p in g.poses:
        h.add_node(p)
    for t, a, b, z, W, loss, k in g.factors:
        if t == 2:
            idx = h.add_xytpos(a, z, W)
        elif t == 1:
            idx = h.add_xyt(a, b, z, W)
        else:
            idx = h.add_xyt_robust(a, b, z, W, loss, k)
        assert idx >= 0, h.last_error()
    return h


def hook_outputs(h, g, at_state=False):
    """What the eval (l_point) or state_eval (state) hooks return per factor; None where the hook is unset (priors
    have no state_eval)."""
    out = []
    for i, (t, a, b, *_rest) in enumerate(g.factors):
        ev = h.eval(i, at_state)
        if ev is None:
            assert at_state and t == 2
            out.append(None)
            continue
        r, J0, J1, W, chi2 = ev
        got = {"r": r, "Weff": W, "rho": [chi2]}
        if t != 2:
            got.update(Ja=J0, Jb=J1)
        out.append(got)
    return out


@pytest.fixture(scope="module")
def corpus_refs(built):
    out = []
    for g in fm.corpus():
        out.append((g, fm.graph_refs(g)))
    return out


def test_hooks_match_exact_reference(corpus_refs):
    """Every factor of the corpus: eval (l_point) and state_eval (state) hook outputs within HOST_C u sum|terms| of the
    exact values.  The states are moved off the l_points first, to poses whose references are computed separately, so
    that each hook is shown to read its own points (the prior's eval hook reads the state; it has no state_eval)."""
    bad, worst, n_state = [], 0.0, 0
    for g, refs in corpus_refs:
        moved = g.poses.copy()
        moved[:, :2] += 0.25
        moved[:, 2] = -moved[:, 2]  # the seam headings stay on the seam
        refs_state = fm.graph_refs(fm.Graph(g.name, moved, g.factors))
        with harness_of(g) as h:
            h.set_states(moved)
            for at_state, rf in ((False, refs), (True, refs_state)):
                for i, got in enumerate(hook_outputs(h, g, at_state)):
                    if got is None:
                        continue
                    n_state += at_state
                    # the prior's eval hook reads the state, like the reference's xytpos eval
                    e = fm.excess(got, (refs_state if g.factors[i][0] == 2 else rf)[i])
                    worst = max(worst, e)
                    if not e <= HOST_C:
                        bad.append((g.name, at_state, i, g.factors[i][0], g.factors[i][5], g.factors[i][6], e))
    print(f"hooks vs exact: worst {worst:.3g} u sum|terms|")
    assert n_state > 500
    assert not bad, bad[:10]


@pytest.mark.parametrize("loss", [fm.HUBER, fm.CAUCHY])
def test_loss_within_ulps_for_every_k(built, loss):
    """The isolated loss rows (r = (r0, 0, 0), W = diag(W00, 1, 1)): W_eff[1][1] = w and chi2 = rho within 4 ulp of
    w(s), rho(s) at the s the hooks form, for every k from the least subnormal to DBL_MAX, and with s on both sides of
    the exact k^2 where k * k is subnormal; never NaN."""
    g = fm.losses()
    bad = []
    with harness_of(g) as h:
        for i, (_, _, _, z, W, ls, k) in enumerate(g.factors):
            if ls != loss:
                continue
            s = fm.loss_s(z[0], W[0])
            w_ex, rho_ex = fm.loss_ref(ls, k, s)
            _, _, _, We, chi2 = h.eval(i)
            uw, ur = fm.ulps(We[1, 1], w_ex), fm.ulps(chi2, rho_ex)
            if not (uw <= LOSS_ULPS and ur <= LOSS_ULPS):
                bad.append((k, s, float(We[1, 1]), float(w_ex), uw, chi2, float(rho_ex), ur))
    assert not bad, bad


def _old_cauchy(k, s):
    k2 = k * k
    return 1.0 / (1.0 + s / k2), k2 * math.log1p(s / k2)


def test_cauchy_bits_unchanged_inside_the_band(built):
    """Where k^2 and s / k^2 are normal the hooks give the bits of 1 / (1 + s / k^2) and k^2 log1p(s / k^2)."""
    ks = [2.0 ** -511, 1e-150, 3e-80, 1e-3, 0.37, 1.0, 7.5, 1e20, 1e100, 1e146, 1.3e154]
    r0s = [0.0, 1e-100, 1e-30, 2.5e-8, 0.1, 1.0, 3.0, 1e5, 1e40, 1e150]
    rows = [(k, r0) for k in ks for r0 in r0s if fm.loss_band(k, r0 * r0) == "normal"]
    assert len(rows) > 60
    poses, factors = [], []
    for k, r0 in rows:
        p = np.array([float(len(poses)), 0.0, 0.0])
        factors.append((32, len(poses), len(poses) + 1, np.array([r0, 0.0, 0.0]), np.eye(3).reshape(9), fm.CAUCHY, k))
        poses += [p, p.copy()]
    g = fm.Graph("band", np.array(poses), factors)
    with harness_of(g) as h:
        for i, (k, r0) in enumerate(rows):
            w, rho = _old_cauchy(k, r0 * r0)
            _, _, _, We, chi2 = h.eval(i)
            assert We[1, 1] == w and chi2 == rho and math.copysign(1, chi2) == math.copysign(1, rho), (k, r0)


# ---------------------------------------------------------------------------------------------
# the checker and the corpus
# ---------------------------------------------------------------------------------------------
def test_checker_rejects_wrong_outputs():
    """8 ulp off the exact loss fails; the late-pose-first off-diagonal block fails; the other representative of r[2]
    fails away from the seam and passes on it."""
    w, rho = fm.loss_ref(fm.CAUCHY, 0.7, 1.3)
    for v in (w, rho):
        x = float(v)
        assert fm.ulps(x, v) <= 0.5
        assert fm.ulps(x + 8 * math.ulp(x), v) > LOSS_ULPS
    assert fm.ulps(float("nan"), w) == math.inf

    g = fm.shapes()
    t, a, b, z, W, loss, k = next(f for f in g.factors if f[0] == 1)
    for early in (True, False):
        ref = fm.factor_ref(t, z, W, g.poses[a], g.poses[b], a_early=early, a_lower=a < b)
        assert len(ref) == 1
        good = {"H": ref[0].val["H"]}
        assert fm.excess(good, ref) <= 1.0
        late_first = {"H": ref[0].val["H"].T}
        assert fm.excess(late_first, ref) > 1e6

    h = fm.headings()
    seam = away = 0
    for t, a, b, z, W, loss, k in h.factors:
        pb = None if b < 0 else h.poses[b]
        ref = fm.factor_ref(t, z, W, h.poses[a], pb)
        r = ref[0].val["r"].copy()
        other = r.copy()
        other[2] += -2 * math.pi if r[2] > 0 else 2 * math.pi
        if len(ref) == 1:
            away += 1
            assert fm.excess({"r": r}, ref) <= 1.0
            assert fm.excess({"r": other}, ref) > 1e6
        else:
            seam += 1
            assert fm.excess({"r": r}, ref) <= 1.0 and fm.excess({"r": other}, ref) <= 1.0
    assert seam > 20 and away > 20, (seam, away)


def test_corpus_reaches_every_edge():
    """Every Cauchy band and every Huber row, both sides of the seam on edges and priors, a hub of degree > 64, a slot
    of 40 or more factors, more than 32 distinct pose pairs besides, N not a multiple of 4, both orientations."""
    gs = {g.name: g for g in fm.corpus()}
    tags = set().union(*(t for g in gs.values() for t in g.tags.values()))
    for band in ("normal", "k2_inf", "k2_small", "t_small", "t_inf"):
        assert f"cauchy:{band}" in tags, band
    for side in ("below", "above"):  # s on both sides of the exact k^2 where k * k is subnormal
        assert {f"huber:straddle_{side}", f"cauchy:straddle_{side}"} <= tags, side
    assert {"a<b", "a>b", "prior_heading"} <= tags
    assert {f"W2^{e}" for e in (-500, -100, 0, 100, 500)} <= tags

    h = gs["headings"]
    sides = set()
    for t, a, b, z, W, loss, k in h.factors:
        ref = fm.factor_ref(t, z, W, h.poses[a], None if b < 0 else h.poses[b])
        if len(ref) == 2:
            sides.add((t, float(np.sign(ref[0].val["r"][2]))))
    assert {(1, 1.0), (1, -1.0), (2, 1.0), (2, -1.0)} <= sides, sides

    s = gs["shapes"]
    two = [(a, b) for t, a, b, *_ in s.factors if t != 2]
    hub = [(a, b) for a, b in two if 0 in (a, b)]
    assert len(hub) > 64 and {a == 0 for a, b in hub} == {True, False}
    pairs = {}
    for a, b in two:
        pairs[(min(a, b), max(a, b))] = pairs.get((min(a, b), max(a, b)), 0) + 1
    big = max(pairs, key=pairs.get)
    assert pairs[big] >= 40
    assert len({(a, b) for a, b in two if (min(a, b), max(a, b)) == big}) == 2  # both orientations
    assert len(pairs) > 32 + 64 and len(s.poses) % 4 != 0
