"""Marginal covariances in float64 numpy from a factor's fronts, walking each pose's root path as the kernels do.

TEST INFRASTRUCTURE.  `paths(plan, nodes)` calls plan_marginal_paths through the library; `walk(snap, paths)`
solves L z = E_q supernode by supernode on the fronts of a frontcheck.Snapshot (dividing by the diagonal of L
where the kernel multiplies by its reciprocal from dinv) and returns Sigma = Z'Z over the shared supernodes
together with the sum of the absolute values of its terms (the componentwise scale of the kernel check).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import scipy.linalg as sla

from . import emul

PATH_DTYPE = np.dtype([("sn0", np.int32), ("j0", np.int32), ("hop0", np.int32), ("nhop", np.int32),
                       ("zoff", np.int64)])


def paths(plan, nodes):
    """plan_marginal_paths on a HostPlan: (records, z doubles, hops)."""
    L = plan.L
    L.asam_dbg_plan_marginal_paths.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.c_void_p,
                                               C.POINTER(C.c_int64)]
    nodes = np.ascontiguousarray(nodes, dtype=np.int32)
    out = np.zeros(len(nodes), dtype=PATH_DTYPE)
    tot = (C.c_int64 * 2)()
    rc = L.asam_dbg_plan_marginal_paths(plan.p, len(nodes), nodes.ctypes.data_as(C.POINTER(C.c_int)),
                                        out.ctypes.data, tot)
    if rc != 0:
        raise ValueError(L.aprilsam_b200_last_error().decode())
    return out, int(tot[0]), int(tot[1])


def chain(desc, s0):
    out = [int(s0)]
    while int(desc["parent"][out[-1]]) >= 0:
        out.append(int(desc["parent"][out[-1]]))
    return out


def pose_columns(snap, rec):
    """[(supernode, js, z (c - js) x 3)] of one pose: its three columns of L^-1 along the root path."""
    d, ipool = snap.desc, snap.ipool
    s, js = int(rec["sn0"]), int(rec["j0"])
    m = 3 * int(d["mb"][s])
    b = np.zeros((m, 3))
    b[js:js + 3] = np.eye(3)
    out = []
    while True:
        F, _ = snap.fronts[s]
        c = 3 * int(d["cb"][s])
        L11 = np.tril(F[:c, :c])[js:, js:]
        z = sla.solve_triangular(L11, b[js:c], lower=True)
        u = b[c:] - F[c:, js:c] @ z
        out.append((s, js, z))
        p = int(d["parent"][s])
        if p < 0:
            return out
        _, rel, *_ = emul.seg_views(d, ipool, s)
        cb, mb = int(d["cb"][s]), int(d["mb"][s])
        idx = (3 * rel[cb:mb].astype(np.int64)[:, None] + np.arange(3)).reshape(-1)
        b = np.zeros((3 * int(d["mb"][p]), 3))
        b[idx] = u
        s, js = p, 0


def walk(snap, recs):
    """(Sigma, sum of |terms|), both (3n x 3n), for the path records of n poses."""
    cols = [pose_columns(snap, r) for r in recs]
    n = len(recs)
    S = np.zeros((3 * n, 3 * n))
    A = np.zeros((3 * n, 3 * n))
    for i in range(n):
        hi = {s: (js, z) for s, js, z in cols[i]}
        for j in range(n):
            for s, js, zj in cols[j]:
                if s not in hi:
                    continue
                jsi, zi = hi[s]
                r0 = max(js, jsi)
                a, b = zi[r0 - jsi:], zj[r0 - js:]
                S[3 * i:3 * i + 3, 3 * j:3 * j + 3] += a.T @ b
                A[3 * i:3 * i + 3, 3 * j:3 * j + 3] += np.abs(a).T @ np.abs(b)
    return S, A
