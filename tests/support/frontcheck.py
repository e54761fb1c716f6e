"""Front-by-front check of the factorisation and solve kernels against float64 / long-double references.

TEST INFRASTRUCTURE.  `snapshot(h)` reads back what a live Harness left in HBM after a solve (Hessian, plan
descriptors + int pool, every front, y, x); the `check_*` functions compare it with plain references of the
same operation:

  * check_linearize: the Hessian against a float64 re-linearisation at the harness's l_points, each entry
    bounded by u times the sum of the absolute values of its contributions;
  * check_fronts: LOCAL backward error of every front.  The front is re-assembled in float64 from the device
    Hessian and the children's update matrices as the device left them; then
    tril(F) = tril([L11;L21][L11;L21]' + [0 0; 0 U]) and L11 y1 = b1, U_rhs = b2 - L21 y1 must hold, relative
    to |F| + |L||L|'.  Backward stability makes this independent of cond(A) (1e8 - 1e9 here);
  * check_y: y as downloaded equals the rhs rows of the fronts bit for bit;
  * check_backsolve: L11' x1 = y1 - L21' x2 per supernode (componentwise), and the global residual
    |Ax - b| / (|A||x| + |b|) accumulated in long double;
  * check_forward: |x - x_ref| / |x_ref| against C * kappa_1 * u, x_ref a sparse LU solve refined in long double.

Every check returns its worst value; `check_fronts` also returns the worst record per kernel path (leaf /
cta_front in shared memory / cta_front out of HBM / team of G) so that a failure names a kernel and a shape.
The same functions run on fronts produced by the numpy emulation (tests/support/emul.py), which is how the
CPU tests show that they detect wrong fronts.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import emul
from .hostplan import HostPlan, lib as hostlib

U = np.finfo(np.float64).eps / 2
_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)


def asam_ld(m):
    """ASAM_LD(m): m + 1 rounded up to even (column stride of a front; row m holds the rhs)."""
    return (m + 2) & ~1


def fits_smem(mb):
    m = 3 * mb
    return asam_ld(m) * m + (asam_ld(m) + 1) // 2 + 2 <= 25600


def dev_api():
    L = hostlib()
    L.asam_dbg_dev_of_graph.argtypes = [C.c_void_p]
    L.asam_dbg_dev_of_graph.restype = C.c_void_p
    L.asam_dbg_plan_of_param.argtypes = [C.c_void_p]
    L.asam_dbg_plan_of_param.restype = C.c_void_p
    L.asam_debug_read_hessian.argtypes = [C.c_void_p, C.c_int, C.c_int, _dp, _dp, _dp]
    L.asam_download_x.argtypes = [C.c_void_p, C.c_int, C.c_int, _dp]
    L.asam_download_y.argtypes = [C.c_void_p, C.c_int, C.c_int, _dp]
    L.asam_debug_read_front.argtypes = [C.c_void_p, C.c_int64, C.c_int64, _dp]
    L.asam_factor_full.argtypes = [C.c_void_p]
    L.asam_backsolve_full.argtypes = [C.c_void_p]
    L.asam_factor_status.argtypes = [C.c_void_p, _ip]
    L.asam_chi2.argtypes = [C.c_void_p, C.c_int, _dp]
    L.asam_last_error.restype = C.c_char_p
    return L


def borrowed_plan(L, param_ptr):
    """The plan a live solver owns, viewed through HostPlan (not destroyed by it)."""
    p = HostPlan.__new__(HostPlan)
    p.L = L
    p.p = C.c_void_p(L.asam_dbg_plan_of_param(param_ptr))
    p.close = lambda: None
    return p


def _ok(L, rc, what):
    if rc != 0:
        raise RuntimeError(f"{what} failed: {L.asam_last_error().decode()}")


# ---------------------------------------------------------------------------------------------
# what is in HBM
# ---------------------------------------------------------------------------------------------
class Snapshot:
    """Plan + Hessian + fronts + y + x of one solve.  fronts[s] = (F (m x m, [row, col]), rhs (m))."""

    def __init__(self, plan, Adiag, Aoff, B, fronts, y, x, lam=None):
        self.plan = plan
        self.desc = plan.descs()
        self.ipool = plan.array("ipool")
        self.q2node = plan.array("q2node")
        self.node2q = plan.array("node2q")
        self.tasks = plan.array("tasks")
        self.nwait = plan.array("nwait")
        self.leaf_tasks = plan.array("leaf_tasks")
        self.Adiag, self.Aoff, self.B = Adiag, Aoff, B
        self.fronts, self.y, self.x = fronts, y, x
        self.nsn = len(self.desc["mb"])

    def path(self, s):
        """Kernel path of supernode s in the batch schedule of the plan."""
        if s in self._leafset():
            return "leaf"
        G = self._team().get(s, 0)
        if G == 0:
            return "cta_smem" if fits_smem(int(self.desc["mb"][s])) else "cta_hbm"
        return f"team{G}"

    def _leafset(self):
        if not hasattr(self, "_ls"):
            self._ls = set(int(s) for s in self.leaf_tasks)
        return self._ls

    def _team(self):
        if not hasattr(self, "_tm"):
            self._tm = {}
            for s, w in zip(self.tasks, self.nwait):
                self._tm.setdefault(int(s), (int(w) >> 24) & 0x7f)
        return self._tm


def read_fronts(L, dev, desc, which=None):
    out = {}
    for s in (range(len(desc["mb"])) if which is None else which):
        m = 3 * int(desc["mb"][s])
        ld = asam_ld(m)
        buf = np.zeros(ld * m)
        _ok(L, L.asam_debug_read_front(dev, int(desc["f_off"][s]), ld * m, buf.ctypes.data_as(_dp)), "read_front")
        G = buf.reshape(m, ld).T  # column-major -> [row, col]
        out[int(s)] = (G[:m, :m].copy(), G[m, :m].copy())
    return out


def snapshot(h, L=None):
    L = L or dev_api()
    dev = L.asam_dbg_dev_of_graph(h.graph_ptr())
    plan = borrowed_plan(L, h.param_ptr())
    info = plan.info()
    N, S = info["N"], info["n_slots"]
    Ad = np.zeros((N, 3, 3)); Ao = np.zeros((max(S, 1), 3, 3)); B = np.zeros((N, 3))
    _ok(L, L.asam_debug_read_hessian(dev, N, S, Ad.ctypes.data_as(_dp), Ao.ctypes.data_as(_dp), B.ctypes.data_as(_dp)),
        "read_hessian")
    y = np.zeros(3 * N); x = np.zeros(3 * N)
    _ok(L, L.asam_download_y(dev, 0, N, y.ctypes.data_as(_dp)), "download_y")
    _ok(L, L.asam_download_x(dev, 0, N, x.ctypes.data_as(_dp)), "download_x")
    desc = plan.descs()
    return Snapshot(plan, Ad, Ao[:S], B, read_fronts(L, dev, desc), y, x)


def snapshot_from_emulation(plan, Hs, fr):
    """The same view of fronts produced by emul.factor / emul.backsolve."""
    desc = plan.descs()
    fronts = {s: (fr.F[int(desc["f_off"][s])].copy(), fr.rhs[int(desc["f_off"][s])].copy())
              for s in range(len(desc["mb"]))}
    N = plan.info()["N"]
    return Snapshot(plan, Hs.Adiag.copy(), Hs.Aoff.copy(), Hs.B.copy(), fronts, fr.y[:3 * N].copy(), fr.x[:3 * N].copy())


# ---------------------------------------------------------------------------------------------
# local backward error of every front
# ---------------------------------------------------------------------------------------------
def assemble(snap, s):
    """Front s in float64 from the Hessian and the children's update matrices as they are in `snap`."""
    d, ipool = snap.desc, snap.ipool
    rows, rel, children, a_slot, a_rb, a_cb = emul.seg_views(d, ipool, s)
    mb, cb, first = int(d["mb"][s]), int(d["cb"][s]), int(d["first"][s])
    m = 3 * mb
    F = np.zeros((m, m)); b = np.zeros(m)
    for k in range(cb):
        node = snap.q2node[first + k]
        F[3 * k:3 * k + 3, 3 * k:3 * k + 3] = np.triu(snap.Adiag[node]).T
        b[3 * k:3 * k + 3] = snap.B[node]
    for i in range(len(a_slot)):
        rb = int(a_rb[i]) & ~emul.TR_FLAG
        S = snap.Aoff[a_slot[i]]
        F[3 * rb:3 * rb + 3, 3 * int(a_cb[i]):3 * int(a_cb[i]) + 3] = S if (int(a_rb[i]) & emul.TR_FLAG) else S.T
    for cs in children:
        cs = int(cs)
        cmb, ccb = int(d["mb"][cs]), int(d["cb"][cs])
        if cmb == ccb:
            continue
        _, crel, *_ = emul.seg_views(d, ipool, cs)
        idx = (3 * crel[ccb:cmb].astype(np.int64)[:, None] + np.arange(3)).reshape(-1)
        CF, crhs = snap.fronts[cs]
        F[np.ix_(idx, idx)] += np.tril(CF[3 * ccb:, 3 * ccb:])
        b[idx] += crhs[3 * ccb:]
    return np.tril(F), b


def front_errors(snap, s):
    """(factor backward error, rhs backward error) of front s."""
    F0, b0 = assemble(snap, s)
    F, rhs = snap.fronts[s]
    m, c = F.shape[0], 3 * int(snap.desc["cb"][s])
    Lc = np.tril(F[:, :c])
    R = Lc @ Lc.T
    R[c:, c:] += np.tril(F[c:, c:])
    absLL = np.abs(Lc) @ np.abs(Lc).T
    scale = np.abs(F0).max(initial=0.0) + absLL.max(initial=0.0)
    e_f = np.abs(np.tril(F0 - R)).max(initial=0.0) / max(scale, np.finfo(float).tiny)
    y1 = rhs[:c]
    L11, L21 = Lc[:c], Lc[c:]
    r1 = np.abs(L11 @ y1 - b0[:c])
    d1 = np.abs(L11) @ np.abs(y1) + np.abs(b0[:c])
    r2 = np.abs(rhs[c:] - (b0[c:] - L21 @ y1))
    d2 = np.abs(b0[c:]) + np.abs(L21) @ np.abs(y1) + np.abs(rhs[c:])
    e_r = float(np.max(np.r_[r1, r2] / np.maximum(np.r_[d1, d2], np.finfo(float).tiny), initial=0.0))
    return float(e_f), e_r


def check_fronts(snap, which=None):
    """Worst local backward errors.  Returns (worst_factor, worst_rhs, per_path) with per_path[path] =
    dict(factor=(err, s, m, c, nch), rhs=(...), n=count)."""
    per = {}
    wf = wr = 0.0
    for s in (range(snap.nsn) if which is None else which):
        s = int(s)
        ef, er = front_errors(snap, s)
        p = snap.path(s)
        rec = per.setdefault(p, {"factor": (0.0,), "rhs": (0.0,), "n": 0})
        rec["n"] += 1
        shape = (s, 3 * int(snap.desc["mb"][s]), 3 * int(snap.desc["cb"][s]), int(snap.desc["ch_cnt"][s]))
        if ef >= rec["factor"][0]:
            rec["factor"] = (ef, *shape)
        if er >= rec["rhs"][0]:
            rec["rhs"] = (er, *shape)
        wf, wr = max(wf, ef), max(wr, er)
    return wf, wr, per


def describe(per):
    """One line per path: worst errors with supernode, m, c and children count."""
    out = []
    for p in sorted(per):
        f, r = per[p]["factor"], per[p]["rhs"]
        shape = (lambda t: f"s={t[1]} m={t[2]} c={t[3]} children={t[4]}" if len(t) > 1 else "-")
        out.append(f"{p}: {per[p]['n']} fronts, factor {f[0]:.2e} ({shape(f)}), rhs {r[0]:.2e} ({shape(r)})")
    return "\n".join(out)


def check_y(snap):
    """Number of y entries that differ from the rhs rows of their fronts (must be 0: bit for bit)."""
    bad = 0
    for s in range(snap.nsn):
        first, c = int(snap.desc["first"][s]), 3 * int(snap.desc["cb"][s])
        _, rhs = snap.fronts[s]
        bad += int(np.count_nonzero(snap.y[3 * first:3 * first + c].view(np.int64) != rhs[:c].view(np.int64)))
    return bad


# ---------------------------------------------------------------------------------------------
# back-substitution
# ---------------------------------------------------------------------------------------------
def check_backsolve_local(snap, which=None):
    """max over supernodes of |L11' x1 + L21' x2 - y1| / (|L11'||x1| + |L21'||x2| + |y1|), componentwise."""
    worst = 0.0
    for s in (range(snap.nsn) if which is None else which):
        s = int(s)
        rows, *_ = emul.seg_views(snap.desc, snap.ipool, s)
        mb, cb, first = int(snap.desc["mb"][s]), int(snap.desc["cb"][s]), int(snap.desc["first"][s])
        c = 3 * cb
        F, rhs = snap.fronts[s]
        L11, L21 = np.tril(F[:c, :c]), F[c:, :c]
        x1 = snap.x[3 * first:3 * first + c]
        x2 = (snap.x.reshape(-1, 3)[rows[cb:]].reshape(-1)) if mb > cb else np.zeros(0)
        r = L11.T @ x1 + L21.T @ x2 - rhs[:c]
        den = np.abs(L11.T) @ np.abs(x1) + np.abs(L21.T) @ np.abs(x2) + np.abs(rhs[:c])
        worst = max(worst, float(np.max(np.abs(r) / np.maximum(den, np.finfo(float).tiny))))
    return worst


def system(snap, ftype, fa, fb, fslot):
    """A (scipy CSR, elimination order q) and b from the Hessian in the snapshot; the off-diagonal blocks are
    placed from the factor list (node pairs), not from the plan's gather lists."""
    import scipy.sparse as sp
    N = len(snap.Adiag)
    n2q = snap.node2q.astype(np.int64)
    pr = np.repeat(np.arange(3), 3); pc = np.tile(np.arange(3), 3)
    D = np.triu(snap.Adiag) + np.transpose(np.triu(snap.Adiag, 1), (0, 2, 1))
    rows = [(3 * n2q[:, None] + pr).reshape(-1)]
    cols = [(3 * n2q[:, None] + pc).reshape(-1)]
    vals = [D.reshape(-1)]
    pair = (np.asarray(ftype) == 1)
    slots, first_f = np.unique(np.asarray(fslot)[pair], return_index=True)
    fidx = np.nonzero(pair)[0][first_f]
    lo = np.minimum(np.asarray(fa)[fidx], np.asarray(fb)[fidx]).astype(np.int64)
    hi = np.maximum(np.asarray(fa)[fidx], np.asarray(fb)[fidx]).astype(np.int64)
    Sb = snap.Aoff[slots].reshape(-1, 9)
    for (r_, c_, v) in ((3 * n2q[lo][:, None] + pr, 3 * n2q[hi][:, None] + pc, Sb),
                        (3 * n2q[hi][:, None] + pc, 3 * n2q[lo][:, None] + pr, Sb)):
        rows.append(r_.reshape(-1)); cols.append(c_.reshape(-1)); vals.append(v.reshape(-1))
    A = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(3 * N, 3 * N))
    b = np.zeros(3 * N)
    b.reshape(-1, 3)[n2q] = snap.B
    return A, b


def _matvec_ld(A, x):
    """A @ x with products and sums in long double."""
    coo = A.tocoo()
    out = np.zeros(A.shape[0], dtype=np.longdouble)
    np.add.at(out, coo.row, coo.data.astype(np.longdouble) * np.asarray(x, dtype=np.longdouble)[coo.col])
    return out


def check_residual(A, b, x):
    """|Ax - b|_inf / (|A|_inf |x|_inf + |b|_inf), residual in long double."""
    r = _matvec_ld(A, x) - b.astype(np.longdouble)
    An = float(np.abs(A).sum(axis=1).max())
    return float(np.abs(r).max() / (An * np.abs(x).max() + np.abs(b).max()))


def reference_solution(A, b, steps=3):
    """splu solve + iterative refinement with long-double residuals.  Returns (x_ref, kappa_1 estimate)."""
    import scipy.sparse.linalg as spl
    lu = spl.splu(A.tocsc())
    x = lu.solve(b).astype(np.longdouble)
    bl = b.astype(np.longdouble)
    for _ in range(steps):
        r = bl - _matvec_ld(A, x)
        x = x + lu.solve(np.asarray(r, dtype=np.float64)).astype(np.longdouble)
    n = A.shape[0]
    inv = spl.LinearOperator((n, n), matvec=lambda v: lu.solve(np.asarray(v, dtype=np.float64)),
                             rmatvec=lambda v: lu.solve(np.asarray(v, dtype=np.float64), trans="T"), dtype=np.float64)
    kappa = spl.onenormest(A.tocsc()) * spl.onenormest(inv)
    return x, float(kappa)


def forward_error(x, x_ref):
    return float(np.abs(np.asarray(x, dtype=np.longdouble) - x_ref).max() / np.abs(x_ref).max())


# ---------------------------------------------------------------------------------------------
# k_linearize and chi2
# ---------------------------------------------------------------------------------------------
def factors_of(h):
    """(ftype, fa, fb, fz (F,3), fW (F,9)) of the harness's graph; ftype 1 = xyt edge, 2 = xytpos prior."""
    F = h.n_factors
    ft = np.zeros(F, np.int32); fa = np.zeros(F, np.int32); fb = np.zeros(F, np.int32)
    fz = np.zeros((F, 3)); fW = np.zeros((F, 9))
    for i in range(F):
        _, a, b, z, W = h.factor(i)
        ft[i], fa[i], fb[i] = (1 if b >= 0 else 2), a, b
        fz[i], fW[i] = z, W
    return ft, fa, fb, fz, fW


def linearize_ref(N, ftype, fa, fb, fz, fW, lp, node2q, lam):
    """float64 Hessian (Adiag upper, Aoff [lower id][higher id] by slot order of first use, B) and, for every
    entry, the sum of the absolute values of its contributions.  Vectorised emul.Hessian.linearize."""
    ftype, fa, fb = (np.asarray(v) for v in (ftype, fa, fb))
    W = fW.reshape(-1, 3, 3)
    Ad = np.zeros((N, 3, 3)); AdA = np.zeros((N, 3, 3)); B = np.zeros((N, 3)); BA = np.zeros((N, 3))
    for k in range(3):
        Ad[:, k, k] += lam
        AdA[:, k, k] += lam
    pri = np.nonzero(ftype == 2)[0]
    if len(pri):
        a = fa[pri]
        p = lp[a]
        r = np.c_[fz[pri, 0] - p[:, 0], fz[pri, 1] - p[:, 1], emul.mod2pi(fz[pri, 2] - p[:, 2])]
        rA = np.c_[np.abs(fz[pri, :2]) + np.abs(p[:, :2]), np.abs(fz[pri, 2]) + np.abs(p[:, 2]) + 2 * np.pi]
        np.add.at(Ad, a, W[pri]); np.add.at(AdA, a, np.abs(W[pri]))
        np.add.at(B, a, np.einsum("fij,fj->fi", W[pri], r))
        np.add.at(BA, a, np.einsum("fij,fj->fi", np.abs(W[pri]), rA))
    e = np.nonzero(ftype == 1)[0]
    a, b = fa[e], fb[e]
    pa, pb, z, We = lp[a], lp[b], fz[e], W[e]
    ca, sa = np.cos(pa[:, 2]), np.sin(pa[:, 2])
    dx, dy = pb[:, 0] - pa[:, 0], pb[:, 1] - pa[:, 1]
    n = len(e)
    Ja = np.zeros((n, 3, 3)); Jb = np.zeros((n, 3, 3))
    Ja[:, 0] = np.c_[-ca, -sa, -sa * dx + ca * dy]
    Ja[:, 1] = np.c_[sa, -ca, -ca * dx - sa * dy]
    Ja[:, 2, 2] = -1.0
    Jb[:, 0] = np.c_[ca, sa, np.zeros(n)]
    Jb[:, 1] = np.c_[-sa, ca, np.zeros(n)]
    Jb[:, 2, 2] = 1.0
    JaA = np.abs(Ja).copy()
    JaA[:, 0, 2] = np.abs(sa * dx) + np.abs(ca * dy)
    JaA[:, 1, 2] = np.abs(ca * dx) + np.abs(sa * dy)
    JbA = np.abs(Jb)
    adx, ady = np.abs(pb[:, 0]) + np.abs(pa[:, 0]), np.abs(pb[:, 1]) + np.abs(pa[:, 1])
    r = np.c_[z[:, 0] - (ca * dx + sa * dy), z[:, 1] - (-sa * dx + ca * dy),
              emul.mod2pi(z[:, 2] - (pb[:, 2] - pa[:, 2]))]
    rA = np.c_[np.abs(z[:, 0]) + adx + ady, np.abs(z[:, 1]) + adx + ady,
               np.abs(z[:, 2]) + np.abs(pb[:, 2]) + np.abs(pa[:, 2]) + 2 * np.pi]
    T = lambda M: np.transpose(M, (0, 2, 1))  # noqa: E731
    JatW, JbtW = T(Ja) @ We, T(Jb) @ We
    JatWA, JbtWA = T(JaA) @ np.abs(We), T(JbA) @ np.abs(We)
    np.add.at(Ad, a, JatW @ Ja); np.add.at(AdA, a, JatWA @ JaA)
    np.add.at(Ad, b, JbtW @ Jb); np.add.at(AdA, b, JbtWA @ JbA)
    np.add.at(B, a, np.einsum("fij,fj->fi", JatW, r)); np.add.at(BA, a, np.einsum("fij,fj->fi", JatWA, rA))
    np.add.at(B, b, np.einsum("fij,fj->fi", JbtW, r)); np.add.at(BA, b, np.einsum("fij,fj->fi", JbtWA, rA))
    # off-diagonal block of the pair, stored [lower id][higher id]
    lo_first = (a < b)
    Hab = JatW @ Jb                 # rows of a, columns of b
    H = np.where(lo_first[:, None, None], Hab, T(Hab))
    HA = JatWA @ JbA
    HA = np.where(lo_first[:, None, None], HA, T(HA))
    return Ad, AdA, B, BA, (np.minimum(a, b), np.maximum(a, b), H, HA)


def check_linearize(snap, ftype, fa, fb, fz, fW, lp, fslot, lam):
    """max over entries of |dev - ref| / (u * sum |contributions|) for Adiag (upper), Aoff and B."""
    N = len(snap.Adiag)
    Ad, AdA, B, BA, (lo, hi, H, HA) = linearize_ref(N, ftype, fa, fb, fz, fW, lp, snap.node2q, lam)
    e = np.nonzero(np.asarray(ftype) == 1)[0]
    S = len(snap.Aoff)
    Ao = np.zeros((S, 3, 3)); AoA = np.zeros((S, 3, 3))
    sl = np.asarray(fslot)[e]
    np.add.at(Ao, sl, H); np.add.at(AoA, sl, HA)
    tri = np.triu(np.ones((3, 3), bool))
    tiny = np.finfo(float).tiny
    rd = (np.abs(snap.Adiag - Ad) / np.maximum(U * AdA, tiny))[:, tri].max(initial=0.0)
    ro = (np.abs(snap.Aoff - Ao) / np.maximum(U * AoA, tiny)).max(initial=0.0)
    rb = (np.abs(snap.B - B) / np.maximum(U * BA, tiny)).max(initial=0.0)
    return float(max(rd, ro, rb))



def chi2_ref(ftype, fa, fb, fz, fW, st):
    """april_graph_chi2 in long double at the states st: 0.5 r'Wr per xyt edge, r'Wr per xytpos prior
    (april_graph_xyt.c / april_graph_xytpos.c)."""
    tot = np.longdouble(0)
    ftype = np.asarray(ftype)
    two_pi, pi = 2 * np.longdouble(np.pi), np.longdouble(np.pi)
    for kind, w in ((1, np.longdouble(0.5)), (2, np.longdouble(1))):
        f = np.nonzero(ftype == kind)[0]
        if not len(f):
            continue
        pa = st[fa[f]].astype(np.longdouble)
        z = fz[f].astype(np.longdouble)
        if kind == 2:
            r = z - pa
        else:
            pb = st[fb[f]].astype(np.longdouble)
            ca, sa = np.cos(pa[:, 2]), np.sin(pa[:, 2])
            dx, dy = pb[:, 0] - pa[:, 0], pb[:, 1] - pa[:, 1]
            r = np.stack([z[:, 0] - (ca * dx + sa * dy), z[:, 1] - (-sa * dx + ca * dy), z[:, 2] - (pb[:, 2] - pa[:, 2])], 1)
        r[:, 2] = r[:, 2] + pi - two_pi * np.floor((r[:, 2] + pi) / two_pi) - pi
        W = fW[f].reshape(-1, 3, 3).astype(np.longdouble)
        tot += w * np.einsum("fi,fij,fj->", r, W, r)
    return tot
