"""The factor maths of k_linearize, k_step, k_hessian_rebuild and k_chi2_partial against the exact reference over the
edge corpus.

Direct drives.  Each corpus graph (support/factormath.py) is solved once with well-posed values (z the relative poses,
W = I, a prior on every pose), so that the plan, the slots and the elimination order exist.  Then the corpus values of
z, W and the loss are written into the factors in place and h.chi2() re-uploads them (gctx_verify_factors) without
factoring anything, and the kernels are driven through the device C-ABI:

  * factor by factor: asam_hessian_reset(lambda = 0), then asam_linearize of that factor alone at explicit points, and
    again without them (edges at the l_points in HBM, priors at the states in HBM, moved off the l_points), then
    asam_hessian_rebuild of the same factor (its two poses and its slot); each read back and compared with factor_ref
    within GPU_C u sum|terms| (either representative of r[2] at the +-pi seam), and linearize with rebuild within the
    same bound;
  * the isolated loss rows (r = (r0, 0, 0) exactly, J = -I / I exactly): the (1, 1) entry of J_a'W_eff J_a is w itself
    and chi2 is 0.5 rho, so both are checked within 4 ulp of the exact w(s), rho(s) for every k;
  * whole graphs at once (a hub of 80 factors across warps, a slot of 44 parallel factors in both orientations, 37 more
    dirty slots, N not a multiple of 4): linearised and rebuilt, against the summed reference;
  * chi2 factor by factor: every corpus factor inactive (W = 0) but one, the priors at zero residual, so
    april_graph_chi2 is that factor's term alone.

End to end.  The SPD corpora (the loss rows without Cauchy k^2 = 0 at s = 0, and the kernel shapes) with their own
values: a batch solve; the loss rows appended pair by pair through incremental steps that must run as k_step; the hub
losing 12 factors (remove_factors) and then relinearised in place (relinearize_poses).  After each, the Hessian in HBM
against every factor evaluated at its own points, and chi2 at the states.

No call here factors a system that holds the rows whose W_eff was NaN before the loss was made total (Cauchy,
k^2 = 0, s = 0): those reach only the direct drives.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import pytest

from aprilsam_b200 import harness as H
from support import factormath as fm
from support import frontcheck as fc
from support import inccheck as ic

pytestmark = pytest.mark.gpu

GPU_C = 40.0   # kernels vs exact, in u sum|terms|  (observed 3.8 on an H100 80GB HBM3, 700 W: the shapes graph)
LOSS_ULPS = 4.0
_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)


def dev_api():
    L = fc.dev_api()
    L.asam_hessian_reset.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double]
    L.asam_linearize.argtypes = [C.c_void_p, C.c_int, C.c_int, _dp]
    L.asam_hessian_rebuild.argtypes = [C.c_void_p, C.c_int, _ip, _ip, C.c_int, _ip, _ip, C.c_int, _ip, _dp, _dp]
    return L


def _i32(v):
    return np.ascontiguousarray(v, dtype=np.int32)


class Drive:
    """A corpus graph in a solved harness, with the corpus values in place and direct access to the kernels."""

    def __init__(self, g: fm.Graph):
        self.g = g
        self.h = H.Harness("b200")
        h = self.h
        for p in g.poses:
            h.add_node(p)
        I9 = np.eye(3).reshape(9)
        for t, a, b, z, W, loss, k in g.factors:
            if t == 2:
                h.add_xytpos(a, g.poses[a], I9)
            elif t == 1:
                h.add_xyt(a, b, fm._rel(g.poses[a], g.poses[b]), I9)
            else:
                h.add_xyt_robust(a, b, fm._rel(g.poses[a], g.poses[b]), I9, fm.HUBER, 1.0)
        self.F0 = len(g.factors)
        for a in range(len(g.poses)):
            h.add_xytpos(a, g.poses[a], I9)
        h.batch()
        self.L = dev_api()
        self.dev = self.L.asam_dbg_dev_of_graph(h.graph_ptr())
        plan = fc.borrowed_plan(self.L, h.param_ptr())
        info = plan.info()
        self.N, self.S = info["N"], info["n_slots"]
        self.fslot = plan.array("fslot")
        self.node2q = plan.array("node2q")
        # the whole graph as the reference sees it: corpus factors, then the priors at zero residual
        self.full = fm.Graph(g.name, g.poses, list(g.factors) +
                             [(2, a, -1, g.poses[a].copy(), I9, 0, 0.0) for a in range(len(g.poses))])
        F = len(self.full.factors)
        self.pts = np.zeros((F, 6))
        for i, (t, a, b, *_r) in enumerate(self.full.factors):
            self.pts[i, :3] = g.poses[a]
            if b >= 0:
                self.pts[i, 3:] = g.poses[b]
        self.set_corpus(range(self.F0))
        h.set_states(g.poses)
        h.chi2()  # re-uploads the edited factors
        self.refs = fm.graph_refs(self.full, node2q=self.node2q)
        # the batch uploaded the l_points it linearised at, the corpus poses (nothing uploads them again here); the
        # states are moved off them for the HBM-points drive, so that a kernel reading the wrong array for a factor
        # type shows: priors are referenced at `moved`, two-pose factors at the poses
        self.moved = g.poses.copy()
        self.moved[:, :2] += 0.25
        self.moved[:, 2] = -self.moved[:, 2]
        self.refs_st = fm.graph_refs(fm.Graph(g.name, self.moved, self.full.factors), node2q=self.node2q)

    def close(self):
        self.h.close()

    def set_corpus(self, idx):
        for i in idx:
            t, a, b, z, W, loss, k = self.g.factors[i]
            self.h.set_factor(i, z, W)
            if t == 32:
                assert self.h.set_loss(i, loss, k) == 0

    def set_inactive(self, idx):
        for i in idx:
            t, a, b, z, W, loss, k = self.g.factors[i]
            self.h.set_factor(i, z, np.zeros(9))
            if t == 32:
                assert self.h.set_loss(i, fm.HUBER, 1.0) == 0

    def _ok(self, rc, what):
        fc._ok(self.L, rc, what)

    def read(self):
        Ad = np.zeros((self.N, 3, 3)); Ao = np.zeros((max(self.S, 1), 3, 3)); B = np.zeros((self.N, 3))
        self._ok(self.L.asam_debug_read_hessian(self.dev, self.N, self.S, Ad.ctypes.data_as(_dp),
                                                Ao.ctypes.data_as(_dp), B.ctypes.data_as(_dp)), "read_hessian")
        return Ad.reshape(self.N, 9), Ao.reshape(-1, 9), B

    def reset(self):
        self._ok(self.L.asam_hessian_reset(self.dev, self.N, self.S, self.N, 0.0), "hessian_reset")

    def linearize(self, first, count, explicit=True):
        """asam_linearize of factors [first, first + count): at self.pts, or (explicit=False) at the l_points in HBM for
        two-pose factors and the states in HBM for priors."""
        pts = np.ascontiguousarray(self.pts[first:first + count])
        self._ok(self.L.asam_linearize(self.dev, first, count, pts.ctypes.data_as(_dp) if explicit else None),
                 "linearize")

    def rebuild(self, fidx):
        """asam_hessian_rebuild of the factors fidx: every pose they touch, every slot they fill."""
        fidx = list(fidx)
        poses = sorted({p for i in fidx for p in (self.full.factors[i][1], self.full.factors[i][2]) if p >= 0})
        inc = {p: [] for p in poses}
        slots = {}
        for i in fidx:
            t, a, b = self.full.factors[i][:3]
            inc[a].append(i)
            if b >= 0:
                inc[b].append(i)
                slots.setdefault(int(self.fslot[i]), []).append(i)
        ent, pptr = [], [0]
        for p in poses:
            ent += inc[p]
            pptr.append(len(ent))
        sl = sorted(slots)
        sptr = [len(ent)]
        for s in sl:
            ent += slots[s]
            sptr.append(len(ent))
        ent_pts = np.ascontiguousarray(self.pts[ent])
        lam = np.zeros(max(len(poses), 1))
        self._ok(self.L.asam_hessian_rebuild(self.dev, len(poses), _i32(poses).ctypes.data_as(_ip),
                                             _i32(pptr).ctypes.data_as(_ip), len(sl), _i32(sl).ctypes.data_as(_ip),
                                             _i32(sptr).ctypes.data_as(_ip), len(ent), _i32(ent).ctypes.data_as(_ip),
                                             ent_pts.ctypes.data_as(_dp), lam.ctypes.data_as(_dp)), "hessian_rebuild")

    def got_of(self, i, Ad, Ao, B):
        t, a, b = self.full.factors[i][:3]
        got = {"Da": Ad[a][list(fm.PACK)], "ba": B[a]}
        if b >= 0:
            got.update(Db=Ad[b][list(fm.PACK)], bb=B[b], H=Ao[self.fslot[i]].reshape(3, 3))
        return got


@pytest.fixture(scope="module", params=["headings", "coordinates", "losses", "shapes"])
def drive(built, request):
    g = {"headings": fm.headings, "coordinates": fm.coordinates, "losses": fm.losses, "shapes": fm.shapes}[
        request.param]()
    d = Drive(g)
    yield d
    d.close()


def test_each_factor_linearize_and_rebuild(drive):
    """Every corpus factor alone through k_linearize (at explicit points, and at the l_points / states in HBM) and
    k_hessian_rebuild: its blocks, J'Wr and off-diagonal block within GPU_C u sum|terms| of the exact values, and the
    two kernels within the same bound of each other; the loss rows' w within 4 ulp."""
    d = drive
    kinds = ("linearize", "rebuild", "linearize_hbm")
    bad, worst, cross = [], dict.fromkeys(kinds, 0.0), 0.0
    d.h.set_states(d.moved)
    d.h.chi2()  # uploads the moved states
    for i in range(d.F0):
        got = {}
        for kind in kinds:
            d.reset()
            d.linearize(i, 1) if kind == "linearize" else d.rebuild([i]) if kind == "rebuild" else \
                d.linearize(i, 1, explicit=False)
            Ad, Ao, B = d.read()
            got[kind] = d.got_of(i, Ad, Ao, B)
            t, a, b, z, W, loss, k = d.g.factors[i]
            refs = d.refs_st[i] if kind == "linearize_hbm" and t == 2 else d.refs[i]
            e = fm.excess(got[kind], refs)
            worst[kind] = max(worst[kind], e)
            if not e <= GPU_C:
                bad.append((kind, i, t, loss, k, e))
            if d.g.name == "losses":
                w_ex, _ = fm.loss_ref(loss, k, fm.loss_s(z[0], W[0]))
                uw = fm.ulps(float(Ad[a][4]), w_ex)
                if not uw <= LOSS_ULPS:
                    bad.append((kind, i, "w", loss, k, float(z[0]), float(Ad[a][4]), float(w_ex), uw))
        # the two kernels against each other, factor by factor, within the same bound
        ref = d.refs[i][0]
        for q in got["linearize"]:
            e = np.abs(np.asarray(got["linearize"][q]) - np.asarray(got["rebuild"][q])) / (fm.U * ref.abs[q] + fm.DBL_MIN)
            cross = max(cross, math.inf if np.isnan(e).any() else float(e.max()))
    d.h.set_states(d.g.poses)
    d.h.chi2()
    print(f"{d.g.name}: worst u sum|terms| {worst}, linearize vs rebuild {cross:.3g}")
    assert cross <= GPU_C, cross
    assert not bad, bad[:12]


def test_whole_graph_linearize_and_rebuild(drive):
    """All factors at once (the warp aggregation of k_linearize, the per-lane sums of k_hessian_rebuild) against the
    summed reference.  The two kernels are also compared with each other here, but only against 2 GPU_C of the summed
    abs; the tight comparison of the two is factor by factor, in test_each_factor_linearize_and_rebuild."""
    d = drive
    F = len(d.full.factors)
    seam = [i for i in range(d.F0) if len(d.refs[i]) > 1]  # either representative: checked one by one above
    d.set_inactive(seam)
    d.h.chi2()
    Ad = np.zeros((d.N, 9)); AdA = np.zeros((d.N, 9)); B = np.zeros((d.N, 3)); BA = np.zeros((d.N, 3))
    Ao = np.zeros((max(d.S, 1), 9)); AoA = np.zeros((max(d.S, 1), 9))
    P = list(fm.PACK)
    for i, (t, a, b, *_r) in enumerate(d.full.factors):
        if i in seam:
            continue
        ref = d.refs[i][0]
        Ad[a, P] += ref.val["Da"]; AdA[a, P] += ref.abs["Da"]
        B[a] += ref.val["ba"]; BA[a] += ref.abs["ba"]
        if b >= 0:
            Ad[b, P] += ref.val["Db"]; AdA[b, P] += ref.abs["Db"]
            B[b] += ref.val["bb"]; BA[b] += ref.abs["bb"]
            Ao[d.fslot[i]] += ref.val["H"].ravel(); AoA[d.fslot[i]] += ref.abs["H"].ravel()
    # the float64 sums above round too: their error is within u times the summed abs
    out = {}
    for kind in ("linearize", "rebuild"):
        d.reset()
        d.linearize(0, F) if kind == "linearize" else d.rebuild(range(F))
        gAd, gAo, gB = d.read()
        e = max(float((np.abs(gAd[:, P] - Ad[:, P]) / (fm.U * AdA[:, P] + fm.DBL_MIN)).max()),
                float((np.abs(gAo - Ao) / (fm.U * AoA + fm.DBL_MIN)).max()),
                float((np.abs(gB - B) / (fm.U * BA + fm.DBL_MIN)).max()))
        out[kind] = (e, gAd[:, P], gAo, gB)
    d.set_corpus(seam)
    d.h.chi2()
    print(f"{d.g.name}: whole graph, u sum|terms|: linearize {out['linearize'][0]:.3g}, rebuild {out['rebuild'][0]:.3g}")
    assert out["linearize"][0] <= GPU_C and out["rebuild"][0] <= GPU_C, {k: v[0] for k, v in out.items()}
    lin, reb = out["linearize"], out["rebuild"]
    cross = max(float((np.abs(lin[1] - reb[1]) / (fm.U * AdA[:, P] + fm.DBL_MIN)).max()),
                float((np.abs(lin[2] - reb[2]) / (fm.U * AoA + fm.DBL_MIN)).max()),
                float((np.abs(lin[3] - reb[3]) / (fm.U * BA + fm.DBL_MIN)).max()))
    assert cross <= 2 * GPU_C, cross


def test_chi2_factor_by_factor(drive):
    """april_graph_chi2 with one corpus factor active at a time: 0.5 rho(s) (r'Wr for priors) within GPU_C u sum|terms|;
    the loss rows within 4 ulp of the exact 0.5 rho(s)."""
    d = drive
    h = d.h
    d.set_inactive(range(d.F0))
    assert h.chi2() == 0.0
    bad, worst = [], 0.0
    for i in range(d.F0):
        d.set_corpus([i])
        c = h.chi2()
        d.set_inactive([i])
        e = fm.excess({"chi2": [c]}, d.refs[i])
        worst = max(worst, e)
        if not e <= GPU_C:
            bad.append((i, d.g.factors[i][0], d.g.factors[i][5], d.g.factors[i][6], c, e))
        t, a, b, z, W, loss, k = d.g.factors[i]
        if d.g.name == "losses":
            _, rho_ex = fm.loss_ref(loss, k, fm.loss_s(z[0], W[0]))
            u = fm.ulps(2 * c, rho_ex)
            if not u <= LOSS_ULPS:
                bad.append((i, "rho", loss, k, float(z[0]), 2 * c, float(rho_ex), u))
    d.set_corpus(range(d.F0))
    print(f"{d.g.name}: chi2 worst u sum|terms| {worst:.3g}")
    assert not bad, bad[:12]


# ---------------------------------------------------------------------------------------------
# end to end: a batch, incremental appends (k_step), remove_factors and relinearize_poses
# ---------------------------------------------------------------------------------------------
LAM = 1e-4  # the Tikhonov term of a default param


class Expect:
    """The Hessian and chi2 the device must hold, from factor_ref of each factor at its own evaluation points."""

    def __init__(self, h, factors):
        self.h, self.factors = h, list(factors)
        self.L = ic.dev_api()
        self.cache = {}

    def ref(self, i, pa, pb, node2q):
        t, a, b, z, W, loss, k = self.factors[i]
        early = b < 0 or node2q[a] < node2q[b]
        key = (i, tuple(pa), None if pb is None else tuple(pb), early)
        if key not in self.cache:
            self.cache[key] = fm.factor_ref(t, z, W, pa, pb, loss, k, a_early=early, a_lower=b < 0 or a < b)
        return self.cache[key]

    def hessian_excess(self, pts, lamv):
        """max |device - exact| / (u sum|terms| + DBL_MIN) over Adiag (upper), Aoff and B; pts (F, 6) per factor."""
        h, L = self.h, self.L
        plan = fc.borrowed_plan(L, h.param_ptr())
        info = plan.info()
        N, S = info["N"], info["n_slots"]
        fslot, node2q = plan.array("fslot"), plan.array("node2q")
        P = list(fm.PACK)
        Ad = np.zeros((N, 9)); AdA = np.zeros((N, 9)); B = np.zeros((N, 3)); BA = np.zeros((N, 3))
        Ao = np.zeros((max(S, 1), 9)); AoA = np.zeros((max(S, 1), 9))
        for q in (0, 4, 8):
            Ad[:, q] += lamv; AdA[:, q] += lamv
        for i, (t, a, b, *_r) in enumerate(self.factors):
            refs = self.ref(i, pts[i, :3], None if b < 0 else pts[i, 3:], node2q)
            assert len(refs) == 1, "end-to-end corpora keep off the seam"
            ref = refs[0]
            Ad[a, P] += ref.val["Da"]; AdA[a, P] += ref.abs["Da"]
            B[a] += ref.val["ba"]; BA[a] += ref.abs["ba"]
            if b >= 0:
                Ad[b, P] += ref.val["Db"]; AdA[b, P] += ref.abs["Db"]
                B[b] += ref.val["bb"]; BA[b] += ref.abs["bb"]
                Ao[fslot[i]] += ref.val["H"].ravel(); AoA[fslot[i]] += ref.abs["H"].ravel()
        dev = L.asam_dbg_dev_of_graph(h.graph_ptr())
        gAd = np.zeros((N, 9)); gAo = np.zeros((max(S, 1), 9)); gB = np.zeros((N, 3))
        fc._ok(L, L.asam_debug_read_hessian(dev, N, S, gAd.ctypes.data_as(_dp), gAo.ctypes.data_as(_dp),
                                            gB.ctypes.data_as(_dp)), "read_hessian")
        e = [np.abs(gAd[:, P] - Ad[:, P]) / (fm.U * AdA[:, P] + fm.DBL_MIN),
             np.abs(gAo[:S] - Ao[:S]) / (fm.U * AoA[:S] + fm.DBL_MIN), np.abs(gB - B) / (fm.U * BA + fm.DBL_MIN)]
        return max(math.inf if np.isnan(x).any() else float(x.max(initial=0.0)) for x in e)

    def chi2_excess(self):
        st = self.h.states()
        val, A = [], 0.0
        for i, (t, a, b, *_r) in enumerate(self.factors):
            ref = self.ref(i, st[a], None if b < 0 else st[b], np.zeros(len(st), np.int32))[0]
            val.append(float(ref.val["chi2"][0]))
            A += float(ref.abs["chi2"][0])
        c = self.h.chi2()
        return abs(c - math.fsum(val)) / (fm.U * A + fm.DBL_MIN) if not math.isnan(c) else math.inf

    def lp_pts(self):
        """Evaluation points after a batch: l_points for two-pose factors, the states it linearised at for priors."""
        lp = self.h.l_points()
        return np.array([np.r_[lp[a], lp[b] if b >= 0 else np.zeros(3)] for t, a, b, *_r in self.factors])


def harness_with(g, factors):
    h = H.Harness("b200")
    for p in g.poses:
        h.add_node(p)
    for t, a, b, z, W, loss, k in factors:
        idx = h.add_xytpos(a, z, W) if t == 2 else h.add_xyt(a, b, z, W) if t == 1 else \
            h.add_xyt_robust(a, b, z, W, loss, k)
        assert idx >= 0
    return h


def spd_losses():
    """The loss rows a solver may be given (no Cauchy k^2 = 0 row at s = 0), a prior at zero residual on every pose."""
    g = fm.losses(nan_rows=False)
    I9 = np.eye(3).reshape(9)
    g.factors += [(2, a, -1, g.poses[a].copy(), I9, 0, 0.0) for a in range(len(g.poses))]
    return g


@pytest.mark.parametrize("name", ["losses", "shapes"])
def test_end_to_end_batch(built, name):
    """A batch solve of an SPD corpus with its own values: the Hessian it factored (at the l_points, lambda on the
    diagonal) and chi2 at the states it leaves against the exact reference."""
    g = spd_losses() if name == "losses" else fm.shapes()
    with harness_with(g, g.factors) as h:
        h.batch()
        ex = Expect(h, g.factors)
        e_h = ex.hessian_excess(ex.lp_pts(), np.full(len(g.poses), LAM))
        e_c = ex.chi2_excess()
    print(f"{name}: batch Hessian {e_h:.3g}, chi2 {e_c:.3g} u sum|terms|")
    assert e_h <= GPU_C and e_c <= GPU_C, (e_h, e_c)


def test_end_to_end_incremental_k_step(built):
    """The SPD loss rows appended pose pair by pose pair through april_graph_cholesky_inc after a batch of the first:
    after every step the Hessian in HBM against each factor evaluated where the step added it (an edge at the l_points,
    a prior at the state), and chi2.  Most steps must run as one k_step launch (step records)."""
    g = spd_losses()
    n_pairs = len(g.poses) // 2
    # per pair: its robust factor and its two priors, in the order they are appended
    rob = [f for f in g.factors if f[0] == 32]
    pri = {f[1]: f for f in g.factors if f[0] == 2}
    L = ic.dev_api()
    kinds, worst_h, worst_c = {}, 0.0, 0.0
    with H.Harness("b200") as h:
        factors, pts = [], []
        lamv = np.zeros(0)
        with ic.recording(L):
            for p in range(n_pairs):
                a, b = rob[p][1], rob[p][2]
                assert (a, b) == (2 * p, 2 * p + 1)
                h.add_node(g.poses[a]); h.add_node(g.poses[b])
                new = [rob[p], pri[a], pri[b]]
                for t, fa, fb, z, W, loss, k in new:
                    h.add_xytpos(fa, z, W) if t == 2 else h.add_xyt_robust(fa, fb, z, W, loss, k)
                factors += new
                if p == 0:
                    ex = Expect(h, factors)
                ex.factors = factors
                lp, st = h.l_points(), h.states()
                nb0 = ic.batch_count(L)
                if p == 0:
                    h.batch()
                else:
                    h.inc()
                    kind = ic.last_step(L, h.param_ptr())["kind"]
                    kinds[kind] = kinds.get(kind, 0) + 1
                if ic.batch_count(L) != nb0:
                    pts = list(ex.lp_pts())
                    lamv = np.full(h.n_nodes, LAM)
                else:
                    pts += [np.r_[lp[fa], lp[fb]] if t == 32 else np.r_[st[fa], np.zeros(3)]
                            for t, fa, fb, *_r in new]
                    lamv = np.r_[lamv, np.zeros(h.n_nodes - len(lamv))]
                worst_h = max(worst_h, ex.hessian_excess(np.array(pts), lamv))
                worst_c = max(worst_c, ex.chi2_excess())
    print(f"incremental: steps {kinds}, worst Hessian {worst_h:.3g}, chi2 {worst_c:.3g} u sum|terms|")
    assert kinds.get("k_step", 0) > n_pairs // 2, kinds
    assert worst_h <= GPU_C and worst_c <= GPU_C, (worst_h, worst_c)


def test_end_to_end_remove_and_relinearize_hub(built):
    """The shapes corpus solved, then 12 of the hub's factors removed (k_hessian_rebuild of the touched blocks), then the
    hub relinearised in place: after each, the Hessian in HBM against the remaining factors at the l_points and chi2."""
    g = fm.shapes()
    hub = [i for i, f in enumerate(g.factors) if f[0] != 2 and 0 in (f[1], f[2])]
    drop = hub[::7][:12]
    with harness_with(g, g.factors) as h:
        h.batch()
        keep = [f for i, f in enumerate(g.factors) if i not in drop]
        h.remove_factors(drop)
        assert h.n_factors == len(keep)
        ex = Expect(h, keep)
        lamv = np.full(len(g.poses), LAM)
        e_rm = (ex.hessian_excess(ex.lp_pts(), lamv), ex.chi2_excess())
        lp0 = h.l_points()[0].copy()
        h.relinearize_poses([0])
        assert not np.array_equal(h.l_points()[0], lp0)
        e_rl = (ex.hessian_excess(ex.lp_pts(), lamv), ex.chi2_excess())
    print(f"remove: Hessian {e_rm[0]:.3g}, chi2 {e_rm[1]:.3g}; relinearize: Hessian {e_rl[0]:.3g}, chi2 {e_rl[1]:.3g}")
    assert max(e_rm + e_rl) <= GPU_C, (e_rm, e_rl)
