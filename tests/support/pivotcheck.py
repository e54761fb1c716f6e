"""Failed and extreme pivots: place a non-positive (or NaN) pivot at a chosen column of a chosen front, predict the
status word the factorisation must report, and drive one device context through failure and recovery.

TEST INFRASTRUCTURE.
  * Context: the device context of a Harness after a batch solve, driven at the C-ABI (upload a factor's W or a
    pose's l_point, reset + linearise, factor + back-solve, read the status, the Hessian, the fronts, y and x).
    Failing systems never go through april_graph_cholesky: it aborts the process on a failed pivot by design;
  * negative_W: the W of a prior on a pose that makes column k of its diagonal block A'_kk = -max(1, |A_kk|), so the
    pivot of that column is at most A'_kk < 0 whatever the Schur updates are;
  * hessian_ref / first_failure: the float64 Hessian of a factor list and the first column, in the task order of the
    plan, whose pivot is not > 0 (NaN included): the supernode and the column a kernel must flag;
  * same_bits: fronts, y and x of two runs compared bit for bit.
"""
from __future__ import annotations

import ctypes as C
from types import SimpleNamespace

import numpy as np

from . import frontcheck as fc

_dp, _ip = fc._dp, fc._ip


def dev_api():
    L = fc.dev_api()
    L.asam_upload_factors.argtypes = [C.c_void_p, C.c_int, C.c_int, _ip, _ip, _ip, _dp, _dp]
    L.asam_upload_points.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, _dp]
    L.asam_hessian_reset.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double]
    L.asam_linearize.argtypes = [C.c_void_p, C.c_int, C.c_int, _dp]
    L.asam_download_x_status.argtypes = [C.c_void_p, C.c_int, C.c_int, _dp, _ip]
    L.asam_debug_read_buffer.argtypes = [C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_void_p]
    L.asam_step_begin.argtypes = [C.c_void_p]
    L.asam_step_run.argtypes = [C.c_void_p]
    L.asam_step_run_small.argtypes = [C.c_void_p, _dp, C.c_int, _ip]
    L.asam_factor.argtypes = [C.c_void_p, C.c_int, _ip, _ip, _ip]
    L.asam_backsolve.argtypes = [C.c_void_p, C.c_int, _ip, _ip]
    return L


# ---------------------------------------------------------------------------------------------
# re-issuing a recorded incremental step
# ---------------------------------------------------------------------------------------------
def reissue_step(L, dev, rec, desc, vehicle, node, W, point, small):
    """Run the factor and back-solve lists of a recorded step (inccheck.last_step) once more, as one step: the
    mirror of factor `vehicle` (an xytpos prior) is re-pointed at `node` with information W, and the step linearises
    that one factor, adding W to the node's diagonal block (W = 0 adds nothing: A + 0 = A bit for bit), then factors
    and back-solves the recorded lists: with k_step when `small` (the host's choice: only single-CTA tasks), with
    asam_step_run otherwise.  A keep word names the rows of the front BEFORE the step (kept poses << 16 | old block
    rows); that memory now holds the front after the step, so the re-issue keeps the same poses of a front of the
    current block rows.  The caller restores the vehicle's mirror.  Returns (kernel, status, x of the listed
    supernodes in list order or None)."""
    i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)  # noqa: E731
    tasks, nwait, keep, bt, bf = (i32(rec[k]) for k in ("tasks", "nwait", "keep", "bt", "bfirst"))
    keep = i32([(int(kp) & ~0xFFFF) | int(desc["mb"][s]) if kp else 0 for s, kp in zip(tasks, keep)])
    t, a, b = i32([2]), i32([node]), i32([-1])
    z = np.ascontiguousarray(point, dtype=np.float64).reshape(3)
    W = np.ascontiguousarray(W, dtype=np.float64).reshape(9)
    pts = np.r_[z, np.zeros(3)]
    fc._ok(L, L.asam_step_begin(dev), "step_begin")
    fc._ok(L, L.asam_upload_factors(dev, vehicle, 1, t.ctypes.data_as(_ip), a.ctypes.data_as(_ip),
                                    b.ctypes.data_as(_ip), z.ctypes.data_as(_dp), W.ctypes.data_as(_dp)), "upload")
    fc._ok(L, L.asam_linearize(dev, vehicle, 1, pts.ctypes.data_as(_dp)), "linearize")
    fc._ok(L, L.asam_factor(dev, len(tasks), tasks.ctypes.data_as(_ip), nwait.ctypes.data_as(_ip),
                            keep.ctypes.data_as(_ip)), "factor")
    fc._ok(L, L.asam_backsolve(dev, len(bt), bt.ctypes.data_as(_ip), bf.ctypes.data_as(_ip)), "backsolve")
    nx = int(sum(3 * int(desc["cb"][s]) for s in bt))
    xo = np.zeros(max(nx, 1))
    st = C.c_int()
    rc = L.asam_step_run_small(dev, xo.ctypes.data_as(_dp), nx, C.byref(st)) if small else 2
    if rc == 0:
        return "k_step", st.value, xo[:nx]
    if rc != 2:
        raise RuntimeError(f"step_run_small failed: {L.asam_last_error().decode()}")
    fc._ok(L, L.asam_step_run(dev), "step_run")
    fc._ok(L, L.asam_factor_status(dev, C.byref(st)), "factor_status")
    return "step_run", st.value, None


def restore_factor(L, dev, factors, f):
    """Put factor f of the device mirror back to the caller's factor."""
    ft, fa, fb, fz, fW = factors
    t, a, b = (np.array([v[f]], np.int32) for v in (ft, fa, fb))
    z, W = np.ascontiguousarray(fz[f]), np.ascontiguousarray(fW[f])
    fc._ok(L, L.asam_upload_factors(dev, int(f), 1, t.ctypes.data_as(_ip), a.ctypes.data_as(_ip),
                                    b.ctypes.data_as(_ip), z.ctypes.data_as(_dp), W.ctypes.data_as(_dp)), "upload")


# ---------------------------------------------------------------------------------------------
# the device context at the C-ABI
# ---------------------------------------------------------------------------------------------
class Context:
    """One graph's device context after a batch solve through the public API.  Factor f of the graph is factor f of
    the device mirror; the l_point mirror holds h.l_points()."""

    def __init__(self, h, lam):
        self.L = L = dev_api()
        self.lam = lam
        self.dev = C.c_void_p(L.asam_dbg_dev_of_graph(h.graph_ptr()))
        self.plan = fc.borrowed_plan(L, h.param_ptr())
        info = self.plan.info()
        self.N, self.S = info["N"], info["n_slots"]
        self.desc = self.plan.descs()
        self.factors = fc.factors_of(h)
        self.lp = h.l_points()
        self.fslot = self.plan.array("fslot")
        self.sn_of_q = self.plan.array("sn_of_q")
        self.node2q = self.plan.array("node2q")
        self.q2node = self.plan.array("q2node")

    def _ok(self, rc, what):
        fc._ok(self.L, rc, what)

    def device_W(self, f):
        out = np.zeros(9)
        self._ok(self.L.asam_debug_read_buffer(self.dev, 9, 72 * f, 72, out.ctypes.data_as(C.c_void_p)), "read W")
        return out

    def set_W(self, f, W, z=None):
        """Factor f of the mirror with information W (and measurement z, default the caller's)."""
        ft, fa, fb, fz, _ = self.factors
        t, a, b = (np.array([v[f]], np.int32) for v in (ft, fa, fb))
        z = np.ascontiguousarray(fz[f] if z is None else z, dtype=np.float64)
        W = np.ascontiguousarray(W, dtype=np.float64).reshape(9)
        self._ok(self.L.asam_upload_factors(self.dev, int(f), 1, t.ctypes.data_as(_ip), a.ctypes.data_as(_ip),
                                            b.ctypes.data_as(_ip), z.ctypes.data_as(_dp), W.ctypes.data_as(_dp)),
                 "upload_factors")

    def set_lp(self, i, p):
        p = np.ascontiguousarray(p, dtype=np.float64).reshape(3)
        self._ok(self.L.asam_upload_points(self.dev, 0, int(i), 1, p.ctypes.data_as(_dp)), "upload_points")

    def relinearize(self, lam=None):
        lam = self.lam if lam is None else lam
        self._ok(self.L.asam_hessian_reset(self.dev, self.N, self.S, self.N, lam), "hessian_reset")
        self._ok(self.L.asam_linearize(self.dev, 0, len(self.factors[0]), None), "linearize")

    def factor(self):
        self._ok(self.L.asam_factor_full(self.dev), "factor_full")
        self._ok(self.L.asam_backsolve_full(self.dev), "backsolve_full")

    def status(self):
        st = C.c_int()
        self._ok(self.L.asam_factor_status(self.dev, C.byref(st)), "factor_status")
        return st.value

    def x_status(self):
        x = np.zeros(3 * self.N)
        st = C.c_int()
        self._ok(self.L.asam_download_x_status(self.dev, 0, self.N, x.ctypes.data_as(_dp), C.byref(st)),
                 "download_x_status")
        return x, st.value

    def hessian(self):
        Ad = np.zeros((self.N, 3, 3)); Ao = np.zeros((max(self.S, 1), 3, 3)); B = np.zeros((self.N, 3))
        self._ok(self.L.asam_debug_read_hessian(self.dev, self.N, self.S, Ad.ctypes.data_as(_dp),
                                                Ao.ctypes.data_as(_dp), B.ctypes.data_as(_dp)), "read_hessian")
        return Ad, Ao[:self.S], B

    def vec(self, which):
        v = np.zeros(3 * self.N)
        fn = self.L.asam_download_y if which == "y" else self.L.asam_download_x
        self._ok(fn(self.dev, 0, self.N, v.ctypes.data_as(_dp)), f"download_{which}")
        return v

    def fronts(self, which=None):
        return fc.read_fronts(self.L, self.dev, self.desc, which)

    def snapshot(self):
        Ad, Ao, B = self.hessian()
        return fc.Snapshot(self.plan, Ad, Ao, B, self.fronts(), self.vec("y"), self.vec("x"))


def same_bits(a, b):
    """Snapshots a and b hold the same fronts, y and x, bit for bit."""
    eq = lambda u, v: np.array_equal(np.asarray(u).view(np.int64), np.asarray(v).view(np.int64))  # noqa: E731
    return (a.fronts.keys() == b.fronts.keys() and eq(a.y, b.y) and eq(a.x, b.x) and
            all(eq(a.fronts[s][0], b.fronts[s][0]) and eq(a.fronts[s][1], b.fronts[s][1]) for s in a.fronts))


def same_hessian(a, b):
    return all(np.array_equal(u.view(np.int64), v.view(np.int64)) for u, v in zip(a, b))


# ---------------------------------------------------------------------------------------------
# where a failure is placed
# ---------------------------------------------------------------------------------------------
def negative_W(W, A_kk, k):
    """W of an xytpos prior with W_kk changed so that the pose's A'_kk = -max(1, |A_kk|) (A_kk: the entry with W)."""
    W = np.array(W, dtype=np.float64).reshape(3, 3)
    W[k, k] += -max(1.0, abs(A_kk)) - A_kk
    return W.reshape(9)


def nan_W(W):
    """W with a NaN in entry (0, 0): every entry of J'WJ and J'Wr of the factor is NaN (0 * NaN = NaN)."""
    W = np.array(W, dtype=np.float64).reshape(9)
    W[0] = np.nan
    return W


def column(desc, q2node, s, j):
    """(node, k) of column j of the front of supernode s."""
    return int(q2node[int(desc["first"][s]) + j // 3]), j % 3


def ancestors(desc, s):
    out = []
    p = int(desc["parent"][s])
    while p >= 0:
        out.append(p)
        p = int(desc["parent"][p])
    return out


def neighbours(factors, i):
    ft, fa, fb = (np.asarray(v) for v in factors[:3])
    e = ft == 1
    return sorted(set(fb[e & (fa == i)].tolist()) | set(fa[e & (fb == i)].tolist()))


# ---------------------------------------------------------------------------------------------
# the float64 expectation
# ---------------------------------------------------------------------------------------------
def hessian_ref(N, S, factors, fslot, lp, lam):
    """(Adiag (full 3x3), Aoff by slot, B) of a factor list in float64 (frontcheck.linearize_ref; a prior's residual
    is taken at lp)."""
    ftype, fa, fb, fz, fW = factors
    Ad, _, B, _, (_, _, H, _) = fc.linearize_ref(N, ftype, fa, fb, fz, fW, lp, None, lam)
    e = np.nonzero(np.asarray(ftype) == 1)[0]
    Ao = np.zeros((S, 3, 3))
    np.add.at(Ao, np.asarray(fslot)[e], H)
    return Ad, Ao, B


def task_order(plan):
    """Supernodes in the order the batch schedule factors them: the leaf kernel's list, then k_factor's (a team's
    entries once)."""
    out, seen = [], set()
    for s in list(plan.array("leaf_tasks")) + list(plan.array("tasks")):
        if int(s) not in seen:
            seen.add(int(s))
            out.append(int(s))
    return out


def _eliminate(F, b, c):
    """Right-looking Cholesky of the first c columns in place; the first column whose pivot is not > 0, or None."""
    for k in range(c):
        d = F[k, k]
        if not d > 0:
            return k
        piv = np.sqrt(d)
        F[k, k] = piv
        F[k + 1:, k] /= piv
        b[k] /= piv
        lk = F[k + 1:, k]
        F[k + 1:, k + 1:] -= np.tril(np.outer(lk, lk))
        b[k + 1:] -= lk * b[k]
    return None


def _factor_front(F, b, c):
    """Blocked elimination of an SPD front (numpy Cholesky), falling back to column steps to locate a failure."""
    F11 = np.tril(F[:c, :c])
    try:
        L11 = np.linalg.cholesky(F11 + np.tril(F11, -1).T)
        ok = np.isfinite(L11).all()
    except np.linalg.LinAlgError:
        ok = False
    if not ok:
        return _eliminate(F, b, c)
    L21 = np.linalg.solve(L11, F[c:, :c].T).T
    y1 = np.linalg.solve(L11, b[:c])
    F[:c, :c] = L11
    F[c:, :c] = L21
    F[c:, c:] -= np.tril(L21 @ L21.T)
    b[c:] -= L21 @ y1
    b[:c] = y1
    return None


def first_failure(plan, Ad, Ao, B, base=None, dirty=None):
    """(supernode, column in its front) of the first pivot that is not > 0 in the batch task order, or None.  With
    `base` (fronts of an SPD run of the same plan) and `dirty` (nodes whose Hessian blocks differ from that run) only
    the supernodes owning a dirty node and their ancestors are eliminated again."""
    desc, q2node = plan.descs(), plan.array("q2node")
    ns = SimpleNamespace(desc=desc, ipool=plan.array("ipool"), q2node=q2node, Adiag=Ad, Aoff=Ao, B=B,
                         fronts=dict(base or {}))
    redo = None
    if dirty is not None:
        sn_of_q, node2q = plan.array("sn_of_q"), plan.array("node2q")
        redo = set()
        for i in dirty:
            s = int(sn_of_q[node2q[i]])
            redo |= {s, *ancestors(desc, s)}
    for s in task_order(plan):
        if redo is not None and s not in redo:
            continue
        F, b = fc.assemble(ns, s)
        k = _factor_front(F, b, 3 * int(desc["cb"][s]))
        if k is not None:
            return s, k
        ns.fronts[s] = (F, b)
    return None


def reference_fronts(plan, Ad, Ao, B):
    """All fronts of an SPD system in float64 (the `base` of first_failure)."""
    desc = plan.descs()
    ns = SimpleNamespace(desc=desc, ipool=plan.array("ipool"), q2node=plan.array("q2node"), Adiag=Ad, Aoff=Ao, B=B,
                         fronts={})
    for s in task_order(plan):
        F, b = fc.assemble(ns, s)
        k = _factor_front(F, b, 3 * int(desc["cb"][s]))
        assert k is None, f"reference system fails at supernode {s} column {k}"
        ns.fronts[s] = (F, b)
    return ns.fronts


def pivot_of(Ad, node, k):
    """The pivot of column k of an isolated pose (no off-diagonal blocks): what the closed-form 3x3 Cholesky of the
    kernels computes as a00, d1 or d2, in float64 and in the same operation order."""
    A = np.triu(Ad[node])
    a00, a10, a20, a11, a21, a22 = A[0, 0], A[0, 1], A[0, 2], A[1, 1], A[1, 2], A[2, 2]
    if k == 0:
        return a00
    r0 = 1.0 / np.sqrt(a00) if a00 > 0 else np.nan
    l10, l20 = a10 * r0, a20 * r0
    d1 = a11 - l10 * l10
    if k == 1:
        return d1
    r1 = 1.0 / np.sqrt(d1) if d1 > 0 else np.nan
    l21 = (a21 - l20 * l10) * r1
    return a22 - l20 * l20 - l21 * l21

