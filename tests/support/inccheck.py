"""Checks of incremental steps (april_graph_cholesky_inc) against references: what frontcheck does for batch solves,
extended to what an incremental step leaves in HBM.

TEST INFRASTRUCTURE.
  * Ledger: the Hessian an incremental solver must hold, factor by factor, each factor evaluated at its own points;
  * read_device_plan / plan_mismatches: the device copy of the plan and of the factor mirror against the host's;
  * last_step / batch_count: what the last incremental call asked of the kernels (step record), batches so far;
  * snapshot / check_y / check_backsolve_rows: the frontcheck views restricted to listed supernodes, and the rows
    [3 bfirst, c) that a pruned back-substitution must satisfy;
  * listed_columns / check_pruned_x / check_states: what a pruned step may and may not change;
  * backsolve: emul.backsolve for the lists of an incremental step, with bfirst.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import emul
from . import frontcheck as fc

_dp, _ip = fc._dp, fc._ip


def dev_api():
    L = fc.dev_api()
    L.asam_debug_read_buffer.argtypes = [C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_void_p]
    L.asam_dbg_record_steps.argtypes = [C.c_int]
    L.asam_dbg_last_step.argtypes = [C.c_void_p, _ip, _ip, _ip, _ip, C.c_int, _ip, _ip, C.c_int]
    L.asam_dbg_profile.argtypes = [_dp, C.c_int]
    return L


class recording:
    """Step records on for the duration of a `with` block (they are process-wide and off by default)."""

    def __init__(self, L):
        self.L = L

    def __enter__(self):
        self.L.asam_dbg_record_steps(1)
        return self

    def __exit__(self, *exc):
        self.L.asam_dbg_record_steps(0)


# ---------------------------------------------------------------------------------------------
# the Hessian of incremental steps
# ---------------------------------------------------------------------------------------------
def factors_of(h, first=0):
    """(ftype, fa, fb, fz (F,3), fW (F,9)) of factors [first, F) of the harness's graph; ftype 1 = xyt, 2 = xytpos."""
    F = h.n_factors - first
    ft = np.zeros(F, np.int32); fa = np.zeros(F, np.int32); fb = np.zeros(F, np.int32)
    fz = np.zeros((F, 3)); fW = np.zeros((F, 9))
    for i in range(F):
        _, a, b, z, W = h.factor(first + i)
        ft[i], fa[i], fb[i] = (1 if b >= 0 else 2), a, b
        fz[i], fW[i] = z, W
    return ft, fa, fb, fz, fW


def check_linearize_pts(snap, ftype, fa, fb, fz, fW, pts, fslot, lamv):
    """frontcheck.check_linearize with every factor evaluated at its own points (pts: F x 6, a then b) and lambda per
    pose.  frontcheck.linearize_ref runs on virtual poses 2f, 2f+1 (one pair per factor); its sums -- and the sums of
    the absolute values of the contributions -- are then added into the real poses."""
    ftype, fa, fb = (np.asarray(v) for v in (ftype, fa, fb))
    F, N = len(ftype), len(snap.Adiag)
    va, vb = 2 * np.arange(F), 2 * np.arange(F) + 1
    lpv = np.asarray(pts).reshape(2 * F, 3)
    Adv, AdAv, Bv, BAv, (_, _, Hv, HAv) = fc.linearize_ref(2 * F, ftype, va, np.where(ftype == 1, vb, -1), fz, fW,
                                                           lpv, None, 0.0)
    Ad = np.zeros((N, 3, 3)); AdA = np.zeros((N, 3, 3)); B = np.zeros((N, 3)); BA = np.zeros((N, 3))
    for k in range(3):
        Ad[:, k, k] += lamv
        AdA[:, k, k] += lamv
    e = np.nonzero(ftype == 1)[0]
    for src, dst in ((va, fa), (vb[e], fb[e])):
        np.add.at(Ad, dst, Adv[src]); np.add.at(AdA, dst, AdAv[src])
        np.add.at(B, dst, Bv[src]); np.add.at(BA, dst, BAv[src])
    # virtual a < b: H has the rows of a; the slot stores [lower id][higher id]
    T = lambda M: np.transpose(M, (0, 2, 1))  # noqa: E731
    swap = (fa[e] > fb[e])[:, None, None]
    H, HA = np.where(swap, T(Hv), Hv), np.where(swap, T(HAv), HAv)
    S = len(snap.Aoff)
    Ao = np.zeros((S, 3, 3)); AoA = np.zeros((S, 3, 3))
    sl = np.asarray(fslot)[e]
    np.add.at(Ao, sl, H); np.add.at(AoA, sl, HA)
    tri = np.triu(np.ones((3, 3), bool))
    tiny, U = np.finfo(float).tiny, fc.U
    rd = (np.abs(snap.Adiag - Ad) / np.maximum(U * AdA, tiny))[:, tri].max(initial=0.0)
    ro = (np.abs(snap.Aoff - Ao) / np.maximum(U * AoA, tiny)).max(initial=0.0)
    rb = (np.abs(snap.B - B) / np.maximum(U * BA, tiny)).max(initial=0.0)
    return float(max(rd, ro, rb))


class Ledger:
    """The Hessian an incremental solver must leave in HBM, kept factor by factor (aprilsam.c:505-542,
    solver.c): at a batch every factor is evaluated at the l_points with z / W as they are then, and every pose
    gets lambda; a factor added by an incremental call (or its old-pose fallback) is evaluated once -- an xyt edge
    at the l_points of its poses at that call, an xytpos prior at the state of its pose -- and added to what is
    there; poses added since the last batch get no lambda.  Later edits of z / W reach the Hessian only at the
    next batch."""

    def __init__(self, lam):
        self.lam = lam
        self.ft = np.zeros(0, np.int32); self.fa = np.zeros(0, np.int32); self.fb = np.zeros(0, np.int32)
        self.fz = np.zeros((0, 3)); self.fW = np.zeros((0, 9)); self.pts = np.zeros((0, 6))
        self.lamv = np.zeros(0)

    def batch(self, h):
        """After a batch solve (l_point = the states it linearised at)."""
        self.ft, self.fa, self.fb, self.fz, self.fW = factors_of(h)
        lp = h.l_points()
        self.pts = np.c_[lp[self.fa], np.where((self.fb >= 0)[:, None], lp[np.maximum(self.fb, 0)], 0.0)]
        self.lamv = np.full(h.n_nodes, float(self.lam))

    def add(self, h, lp, st):
        """After an incremental call without a batch: lp / st = l_points / states at the call."""
        ft, fa, fb, fz, fW = factors_of(h, len(self.ft))
        pts = np.where((ft == 1)[:, None], np.c_[lp[fa], lp[np.maximum(fb, 0)]], np.c_[st[fa], np.zeros((len(fa), 3))])
        self.ft, self.fa, self.fb = np.r_[self.ft, ft], np.r_[self.fa, fa], np.r_[self.fb, fb]
        self.fz, self.fW, self.pts = np.r_[self.fz, fz], np.r_[self.fW, fW], np.r_[self.pts, pts]
        self.lamv = np.r_[self.lamv, np.zeros(h.n_nodes - len(self.lamv))]

    def check(self, snap, fslot):
        return check_linearize_pts(snap, self.ft, self.fa, self.fb, self.fz, self.fW, self.pts, fslot, self.lamv)


# ---------------------------------------------------------------------------------------------
# the device copy of the plan and of the factor mirror; what an incremental step asked for
# ---------------------------------------------------------------------------------------------
DEV_BUFS = dict(sn=0, ipool=1, node2q=2, q2node=3, fslot=4, ftype=5, fa=6, fb=7, fz=8, fW=9)


def read_device_plan(L, dev, plan, n_factors):
    """The device buffers that mirror the host plan and the factor mirror, as long as the host's."""
    info = plan.info()
    n = dict(sn=12 * info["nsn"], ipool=info["ipool_n"], node2q=info["N"], q2node=info["N"], fslot=n_factors,
             ftype=n_factors, fa=n_factors, fb=n_factors, fz=3 * n_factors, fW=9 * n_factors)
    out = {}
    for k, cnt in n.items():
        a = np.zeros(cnt, np.float64 if k in ("fz", "fW") else np.int32)
        fc._ok(L, L.asam_debug_read_buffer(dev, DEV_BUFS[k], 0, a.nbytes, a.ctypes.data_as(C.c_void_p)), f"read {k}")
        out[k] = a
    return out


def host_plan_arrays(plan, factors):
    """The same arrays from the host plan and the host factor arrays (ftype, fa, fb, fz, fW)."""
    ft, fa, fb, fz, fW = factors
    F = len(ft)
    return dict(sn=plan.array("desc"), ipool=plan.array("ipool"), node2q=plan.array("node2q"),
                q2node=plan.array("q2node"), fslot=plan.array("fslot")[:F], ftype=np.asarray(ft, np.int32),
                fa=np.asarray(fa, np.int32), fb=np.asarray(fb, np.int32), fz=np.asarray(fz).reshape(-1),
                fW=np.asarray(fW).reshape(-1))


def plan_mismatches(dev_arrays, host_arrays):
    """{buffer: number of words that differ bit for bit (or 'length')} -- empty when the device copy is exact.  For
    descriptors, the differing (supernode, field) pairs are listed."""
    bad = {}
    for k, want in host_arrays.items():
        got = dev_arrays[k]
        if len(got) != len(want):
            bad[k] = "length"
            continue
        w = want.view(np.int64 if want.dtype == np.float64 else np.int32)
        g = got.view(np.int64 if got.dtype == np.float64 else np.int32)
        n = int(np.count_nonzero(w != g))
        if n:
            if k == "sn":
                diff = np.nonzero((w != g).reshape(-1, 12))
                bad[k] = sorted(set(zip(diff[0].tolist(), diff[1].tolist())))[:8]
            else:
                bad[k] = n
    return bad


STEP_KINDS = {0: "none", 1: "k_step", 2: "pruned", 3: "full", 4: "fallback"}


def last_step(L, param_ptr, cap=1 << 16):
    """What the last april_graph_cholesky_inc asked of the kernels (inside `recording`)."""
    hdr = np.zeros(4, np.int32)
    t, w, k = (np.zeros(cap, np.int32) for _ in range(3))
    bt, bf = np.zeros(cap, np.int32), np.zeros(cap, np.int32)
    rc = L.asam_dbg_last_step(param_ptr, hdr.ctypes.data_as(_ip), t.ctypes.data_as(_ip), w.ctypes.data_as(_ip),
                              k.ctypes.data_as(_ip), cap, bt.ctypes.data_as(_ip), bf.ctypes.data_as(_ip), cap)
    if rc != 0:
        raise RuntimeError("no solver on this param")
    nt, nb = min(int(hdr[2]), cap), min(int(hdr[3]), cap)
    return dict(kind=STEP_KINDS[int(hdr[0])], escalated=bool(hdr[1]), tasks=t[:nt], nwait=w[:nt], keep=k[:nt],
                bt=bt[:nb], bfirst=bf[:nb])


def batch_count(L):
    """Batch solves so far in this process (explicit or escalated): the host profile counter."""
    out = np.zeros(24)
    L.asam_dbg_profile(out.ctypes.data_as(_dp), 0)
    return int(out[9])


# ---------------------------------------------------------------------------------------------
# fronts, y and the back-substitution of listed supernodes
# ---------------------------------------------------------------------------------------------
def snapshot(h, L, which=None):
    """frontcheck.snapshot; with `which`, only the fronts of those supernodes and of their children."""
    if which is None:
        return fc.snapshot(h, L)
    dev = L.asam_dbg_dev_of_graph(h.graph_ptr())
    plan = fc.borrowed_plan(L, h.param_ptr())
    info = plan.info()
    N, S = info["N"], info["n_slots"]
    Ad = np.zeros((N, 3, 3)); Ao = np.zeros((max(S, 1), 3, 3)); B = np.zeros((N, 3))
    fc._ok(L, L.asam_debug_read_hessian(dev, N, S, Ad.ctypes.data_as(_dp), Ao.ctypes.data_as(_dp),
                                        B.ctypes.data_as(_dp)), "read_hessian")
    y = np.zeros(3 * N); x = np.zeros(3 * N)
    fc._ok(L, L.asam_download_y(dev, 0, N, y.ctypes.data_as(_dp)), "download_y")
    fc._ok(L, L.asam_download_x(dev, 0, N, x.ctypes.data_as(_dp)), "download_x")
    desc, ipool = plan.descs(), plan.array("ipool")
    want = set(int(s) for s in which)
    for s in list(want):
        want |= set(int(c) for c in emul.seg_views(desc, ipool, s)[2])
    return fc.Snapshot(plan, Ad, Ao[:S], B, fc.read_fronts(L, dev, desc, sorted(want)), y, x)


def check_y(snap, which):
    """frontcheck.check_y on the listed supernodes."""
    bad = 0
    for s in which:
        s = int(s)
        first, c = int(snap.desc["first"][s]), 3 * int(snap.desc["cb"][s])
        bad += int(np.count_nonzero(snap.y[3 * first:3 * first + c].view(np.int64) != snap.fronts[s][1][:c].view(np.int64)))
    return bad


def check_backsolve_rows(snap, which, bfirst):
    """Rows [3 bfirst[i], c) of L11' x1 + L21' x2 = y1 of supernode which[i], componentwise (frontcheck's measure):
    what a pruned back-substitution that starts at pose bfirst of the supernode must satisfy."""
    worst = 0.0
    for s, b in zip(which, bfirst):
        s, j = int(s), 3 * int(b)
        rows, *_ = emul.seg_views(snap.desc, snap.ipool, s)
        mb, cb, first = int(snap.desc["mb"][s]), int(snap.desc["cb"][s]), int(snap.desc["first"][s])
        c = 3 * cb
        F, rhs = snap.fronts[s]
        L11, L21 = np.tril(F[:c, :c]), F[c:, :c]
        x1 = snap.x[3 * first:3 * first + c]
        x2 = (snap.x.reshape(-1, 3)[rows[cb:]].reshape(-1)) if mb > cb else np.zeros(0)
        r = (L11.T @ x1 + L21.T @ x2 - rhs[:c])[j:]
        den = (np.abs(L11.T) @ np.abs(x1) + np.abs(L21.T) @ np.abs(x2) + np.abs(rhs[:c]))[j:]
        worst = max(worst, float(np.max(np.abs(r) / np.maximum(den, np.finfo(float).tiny), initial=0.0)))
    return worst


def check_residual(A, b, x):
    """frontcheck.check_residual, 0 for an exact zero residual (a graph whose solution is 0, e.g. one pose at its
    prior)."""
    return 0.0 if np.array_equal(A @ x, b) and not np.any(b) else fc.check_residual(A, b, x)


def listed_columns(desc, N, bt, bfirst):
    """Mask over elimination positions [0, N): the poses a pruned back-substitution (bt, bfirst) solves for."""
    mask = np.zeros(N, bool)
    for s, b in zip(bt, bfirst):
        first, cb = int(desc["first"][s]), int(desc["cb"][s])
        mask[first + int(b):first + cb] = True
    return mask


def check_pruned_x(x_before, x_after, mask):
    """Number of x entries at positions outside `mask` that are not bit-identical to their value before the step
    (positions that did not exist before count when they are outside the mask)."""
    n0 = len(x_before) // 3
    keep = ~mask[:n0]
    xb, xa = x_before.reshape(-1, 3)[keep], x_after.reshape(-1, 3)[:n0][keep]
    return int(np.count_nonzero(xb.view(np.int64) != xa.view(np.int64))) + int(np.count_nonzero(~mask[n0:]))


def check_states(st_before, st_after, lp, x, node2q, mask):
    """(poses whose state changed but is not l_point + x(HBM) bit for bit, poses that changed outside `mask`, poses
    that changed).  st_before holds a row per pose before the call (for a new pose: its l_point)."""
    changed = np.nonzero(np.any(st_before.view(np.int64) != st_after.view(np.int64), axis=1))[0]
    want = lp[changed] + x.reshape(-1, 3)[node2q[changed]]
    want[:, 2] = emul.mod2pi(want[:, 2])
    wrong = int(np.count_nonzero(np.any(want.view(np.int64) != st_after[changed].view(np.int64), axis=1)))
    return wrong, int(np.count_nonzero(~mask[node2q[changed]])), len(changed)


def backsolve(fr, desc, ipool, bt, bfirst):
    """k_backsolve of an incremental step (entries: supernode ids, parents first): entry i solves the columns of
    poses [bfirst[i], cb) of its supernode."""
    for s, b in zip(bt, bfirst):
        s, j = int(s), 3 * int(b)
        P = int(desc["parent"][s])
        rows, *_ = emul.seg_views(desc, ipool, s)
        mb, cb, first = int(desc["mb"][s]), int(desc["cb"][s]), int(desc["first"][s])
        c = 3 * cb
        Lf = fr.F[int(desc["f_off"][s])]
        xs = np.concatenate([fr.x[3 * int(r):3 * int(r) + 3] for r in rows[cb:]]) if mb > cb else np.zeros(0)
        w = fr.y[3 * first + j:3 * first + c] - Lf[c:, j:c].T @ xs
        fr.x[3 * first + j:3 * first + c] = np.linalg.solve(np.tril(Lf[j:c, j:c]).T, w)
        assert P < 0 or P in set(int(t) for t in bt), f"parent {P} of {s} not in the list"
