"""Checks of factor removals (aprilsam_b200_remove_factors) against references.

TEST INFRASTRUCTURE.
  * RemovalLedger: inccheck.Ledger that also forgets removed factors and knows robust losses; check() is inccheck's
    entry-by-entry bound with each robust factor's weighted W; hessian() is the system the solver must hold (every
    remaining factor at its own evaluation points, lambda on the poses of the last batch);
  * root_paths / refactor_lists: the marking of solver.c and plan_refactor's contract, from a host plan;
  * dense_ld: the ledger system as a dense long-double matrix in node order, for solves and inverses.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import emul
from . import frontcheck as fc
from . import inccheck as ic

U = fc.U


def losses_of(h, first=0):
    """(loss code, k) per factor [first, F) of the harness's graph ((0, 0) without a robust loss)."""
    L = ic.dev_api()
    L.asam_dbg_factor_loss.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_double)]
    out_l, out_k = [], []
    for i in range(first, h.n_factors):
        lo, k = C.c_int(), C.c_double()
        L.asam_dbg_factor_loss(h.graph_ptr(), i, C.byref(lo), C.byref(k))
        out_l.append(lo.value)
        out_k.append(k.value)
    return np.array(out_l, np.int32), np.array(out_k)


class RemovalLedger(ic.Ledger):
    """inccheck.Ledger plus removals and robust losses."""

    def __init__(self, lam):
        super().__init__(lam)
        self.loss = np.zeros(0, np.int32)
        self.lk = np.zeros(0)

    def batch(self, h):
        super().batch(h)
        self.loss, self.lk = losses_of(h)

    def add(self, h, lp, st):
        n0 = len(self.loss)
        super().add(h, lp, st)
        lo, k = losses_of(h, n0)
        self.loss, self.lk = np.r_[self.loss, lo], np.r_[self.lk, k]

    def remove(self, idx):
        keep = np.ones(len(self.ft), bool)
        keep[np.asarray(idx, int)] = False
        for name in ("ft", "fa", "fb", "fz", "fW", "pts", "loss", "lk"):
            setattr(self, name, getattr(self, name)[keep])

    def hessian(self, N, n_slots, fslot, node2q):
        """(Ad, AdA, B, BA, Ao, AoA): the Hessian the solver must hold (Ad upper triangle, Ao in slot orientation
        [lower id][higher id]) and sums of absolute values of the contributions' factors."""
        Ad = np.zeros((N, 3, 3)); AdA = np.zeros((N, 3, 3)); B = np.zeros((N, 3)); BA = np.zeros((N, 3))
        Ao = np.zeros((n_slots, 3, 3)); AoA = np.zeros((n_slots, 3, 3))
        for k in range(3):
            Ad[:len(self.lamv), k, k] += self.lamv
            AdA[:len(self.lamv), k, k] += self.lamv
        W = self.fW.reshape(-1, 3, 3)
        pr = np.nonzero(self.ft == 2)[0]
        if len(pr):
            p = self.pts[pr, :3]
            r = np.stack([self.fz[pr, 0] - p[:, 0], self.fz[pr, 1] - p[:, 1], emul.mod2pi(self.fz[pr, 2] - p[:, 2])], 1)
            a = self.fa[pr]
            np.add.at(Ad, a, np.triu(W[pr])); np.add.at(AdA, a, np.abs(np.triu(W[pr])))
            np.add.at(B, a, np.einsum("fij,fj->fi", W[pr], r))
            np.add.at(BA, a, np.einsum("fij,fj->fi", np.abs(W[pr]), np.abs(r)))
        e = np.nonzero(self.ft == 1)[0]
        if len(e):
            pa, pb, z = self.pts[e, :3], self.pts[e, 3:], self.fz[e]
            ca, sa = np.cos(pa[:, 2]), np.sin(pa[:, 2])
            dx, dy = pb[:, 0] - pa[:, 0], pb[:, 1] - pa[:, 1]
            n = len(e)
            Ja = np.zeros((n, 3, 3)); Jb = np.zeros((n, 3, 3))
            Ja[:, 0, 0], Ja[:, 0, 1], Ja[:, 0, 2] = -ca, -sa, -sa * dx + ca * dy
            Ja[:, 1, 0], Ja[:, 1, 1], Ja[:, 1, 2] = sa, -ca, -ca * dx - sa * dy
            Ja[:, 2, 2] = -1.0
            Jb[:, 0, 0], Jb[:, 0, 1], Jb[:, 1, 0], Jb[:, 1, 1], Jb[:, 2, 2] = ca, sa, -sa, ca, 1.0
            r = np.stack([z[:, 0] - (ca * dx + sa * dy), z[:, 1] - (-sa * dx + ca * dy),
                          emul.mod2pi(z[:, 2] - (pb[:, 2] - pa[:, 2]))], 1)
            We = self.effective_W().reshape(-1, 3, 3)[e]
            T = lambda M: np.transpose(M, (0, 2, 1))  # noqa: E731
            JatW, JbtW = T(Ja) @ We, T(Jb) @ We
            absJa, absJb, absW = np.abs(Ja), np.abs(Jb), np.abs(We)
            fa, fb = self.fa[e], self.fb[e]
            for J, JtW, aJ, node in ((Ja, JatW, absJa, fa), (Jb, JbtW, absJb, fb)):
                np.add.at(Ad, node, np.triu(JtW @ J)); np.add.at(AdA, node, np.triu(T(aJ) @ absW @ aJ))
                np.add.at(B, node, np.einsum("fij,fj->fi", JtW, r))
                np.add.at(BA, node, np.einsum("fij,fj->fi", T(aJ) @ absW, np.abs(r)))
            early_a = (node2q[fa] < node2q[fb])[:, None, None]
            H = np.where(early_a, JatW @ Jb, JbtW @ Ja)
            HA = np.where(early_a, T(absJa) @ absW @ absJb, T(absJb) @ absW @ absJa)
            early = np.where(early_a[:, 0, 0], fa, fb)
            tr = (early != np.minimum(fa, fb))[:, None, None]
            H, HA = np.where(tr, T(H), H), np.where(tr, T(HA), HA)
            sl = np.asarray(fslot)[e]
            np.add.at(Ao, sl, H); np.add.at(AoA, sl, HA)
        return Ad, AdA, B, BA, Ao, AoA

    def check(self, snap, fslot):
        """Worst |device - ledger| / (u * sum |contributions|) over every entry: inccheck's check with every robust
        factor's W scaled by its weight."""
        return ic.check_linearize_pts(snap, self.ft, self.fa, self.fb, self.fz, self.effective_W(), self.pts, fslot,
                                      self.lamv)

    def effective_W(self):
        """W per factor with a robust factor's IRLS weight at its evaluation points applied (what k_linearize uses)."""
        fW = self.fW.copy()
        for f in np.nonzero(self.loss != 0)[0]:
            _, _, r = emul.xyt_eval(self.pts[f, :3], self.pts[f, 3:], self.fz[f])
            W = self.fW[f].reshape(3, 3)
            s = float(r @ (W @ r))
            k = float(self.lk[f])
            w = (1.0 if s <= k * k else k / np.sqrt(s)) if self.loss[f] == 1 else 1.0 / (1.0 + s / (k * k))
            fW[f] = (W * w).reshape(9)
        return fW

    def dense_ld(self, N, n_slots, fslot, node2q):
        """(A, b) of the ledger system in node order (3 rows per pose), long double."""
        Ad, _, B, _, Ao, _ = self.hessian(N, n_slots, fslot, node2q)
        A = np.zeros((3 * N, 3 * N), np.longdouble)
        D = np.triu(Ad) + np.transpose(np.triu(Ad, 1), (0, 2, 1))
        for i in range(N):
            A[3 * i:3 * i + 3, 3 * i:3 * i + 3] = D[i]
        e = np.nonzero(self.ft == 1)[0]
        seen = set()
        for f in e:
            s = int(fslot[f])
            if s in seen:
                continue
            seen.add(s)
            lo, hi = int(min(self.fa[f], self.fb[f])), int(max(self.fa[f], self.fb[f]))
            A[3 * lo:3 * lo + 3, 3 * hi:3 * hi + 3] = Ao[s]
            A[3 * hi:3 * hi + 3, 3 * lo:3 * lo + 3] = Ao[s].T
        return A, B.reshape(-1).astype(np.longdouble)


def root_paths(plan, poses):
    """The marking of solver.c: every pose on the node-level root path of each pose (graph ids, first visit order)."""
    order, pos, ppos = plan.array("order"), plan.array("pos"), plan.array("parent_pos")
    marked, seen = [], set()
    for v in poses:
        v = int(v)
        while v not in seen:
            seen.add(v)
            marked.append(v)
            pp = ppos[pos[v]]
            if pp < 0:
                break
            v = int(order[pp])
    return marked


def refactor_contract(plan, marked, tasks, nwait, keep):
    """Violations of plan_refactor's contract (empty list = none): the tasks are exactly the supernodes holding a
    marked pose, children first; a team's entries are consecutive with the same G; a keep word names the first
    marked column and the block rows; nwait counts the marked children."""
    bad = []
    D = plan.descs()
    node2q, sn_of_q = plan.array("node2q"), plan.array("sn_of_q")
    ipool = plan.array("ipool")
    want = sorted(set(int(sn_of_q[node2q[v]]) for v in marked))
    distinct = []
    for s in tasks:
        if not distinct or distinct[-1] != int(s):
            distinct.append(int(s))
    if distinct != want:
        bad.append(f"tasks {distinct[:8]}... != marked supernodes {want[:8]}...")
    if len(set(distinct)) != len(distinct):
        bad.append("a supernode appears in two runs")
    first_col = {}
    for v in marked:
        q = int(node2q[v])
        s = int(sn_of_q[q])
        first_col[s] = min(first_col.get(s, 1 << 30), q - int(D["first"][s]))
    ms = set(want)
    i = 0
    while i < len(tasks):
        s = int(tasks[i])
        G = (int(nwait[i]) >> 24) & 0x7f
        j = i
        while j < len(tasks) and int(tasks[j]) == s:
            if ((int(nwait[j]) >> 24) & 0x7f) != G:
                bad.append(f"team of {s}: mixed G")
            j += 1
        if G > 1 and j - i != G:
            bad.append(f"team of {s}: {j - i} entries for G = {G}")
        if G <= 1 and j - i != 1:
            bad.append(f"supernode {s}: {j - i} entries without a team")
        children = emul.seg_views(D, ipool, s)[2]
        nm = sum(1 for c in children if int(c) in ms)
        if (int(nwait[i]) & 0xffff) != nm:
            bad.append(f"supernode {s}: nwait {int(nwait[i]) & 0xffff} != {nm} marked children")
        kw = int(keep[i])
        kb = first_col[s]
        if G > 1:
            if any(int(keep[t]) for t in range(i, j)):
                bad.append(f"team {s} keeps columns")
        elif kb > 0:
            if kw != ((kb << 16) | int(D["mb"][s])):
                bad.append(f"supernode {s}: keep {kw:#x} != ({kb} << 16) | {int(D['mb'][s])}")
        elif kw != 0:
            bad.append(f"supernode {s}: keep {kw:#x} with the first column marked")
        i = j
    pos = {s: k for k, s in enumerate(distinct)}
    for s in distinct:
        p = int(D["parent"][s])
        if p in pos and pos[p] < pos[s]:
            bad.append(f"parent {p} before child {s}")
    return bad
