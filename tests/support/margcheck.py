"""Marginal covariances in float64 numpy from a factor's fronts, walking each pose's root path as the kernels do,
and hop-by-hop checks of what k_marginal_path / k_marginal_gram wrote.

TEST INFRASTRUCTURE.  `paths(plan, nodes)` calls plan_marginal_paths through the library; `walk(snap, paths)`
solves L z = E_q supernode by supernode on the fronts of a frontcheck.Snapshot (dividing by the diagonal of L
where the kernel multiplies by its reciprocal from dinv) and returns Sigma = Z'Z over the shared supernodes
together with the sum of the absolute values of its terms (the componentwise scale of the kernel check).

The hop checks run on the kernel's own intermediate results, read back from the query scratch (`read_query`):

  * check_hops: every hop record (supernode, js, c, offset) equals the root chain of the plan, exactly;
  * hop_errors: LOCAL backward error of every hop.  b_h is rebuilt in long double from the kernel's z of the hop
    below (scattered through rel), then |L11 z_h - b_h[js:c]| <= C u (|L11||z_h| + S_h) componentwise, S_h the
    sum of |terms| that make up b_h.  The bound does not grow along the path (as check_backsolve_local);
  * gram_errors: every Sigma_ij against Z_i'Z_j in long double over the shared hops from max(js_i, js_j), relative
    to the sum of |terms|, and (j, i) the exact transpose of (i, j);
  * dinv_errors: |dinv_k L_kk - 1| / u for the columns of the given supernodes.

`kernel_path` restates k_marginal_path's blocked order in float64 (96-column blocks from js, reciprocal pivots,
128-row passes by four 24-column groups) with an optional fault, which is how the CPU tests show that the checks
catch wrong hops.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import scipy.linalg as sla

from . import emul

PATH_DTYPE = np.dtype([("sn0", np.int32), ("j0", np.int32), ("hop0", np.int32), ("nhop", np.int32),
                       ("zoff", np.int64)])
LD = np.longdouble
U = np.finfo(np.float64).eps / 2
BSW, MKG, MROWS = 96, 24, 128  # ASAM_BSW, ASAM_MKG, ASAM_MROWS of asam_kernels.cuh
DBG_BUF_DINV, DBG_BUF_MARG = 11, 12  # ASAM_DBG_BUF_DINV / _MARG of asam_cuda.h
TINY = np.finfo(float).tiny


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


def _scatter_index(desc, ipool, s):
    _, rel, *_ = emul.seg_views(desc, ipool, s)
    cb, mb = int(desc["cb"][s]), int(desc["mb"][s])
    return (3 * rel[cb:mb].astype(np.int64)[:, None] + np.arange(3)).reshape(-1)


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
        b = np.zeros((3 * int(d["mb"][p]), 3))
        b[_scatter_index(d, ipool, s)] = u
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


# ---------------------------------------------------------------------------------------------
# what the kernels left in the query scratch
# ---------------------------------------------------------------------------------------------
def _api(L):
    L.asam_debug_read_buffer.argtypes = [C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_void_p]
    L.asam_debug_marginal_layout.argtypes = [C.c_int, C.c_int64, C.c_int, C.POINTER(C.c_int64)]
    L.asam_debug_marginal_layout.restype = None
    return L


def _read(L, dev, buf, off, arr):
    if L.asam_debug_read_buffer(dev, buf, int(off), arr.nbytes, arr.ctypes.data_as(C.c_void_p)) != 0:
        raise RuntimeError(L.asam_last_error().decode())
    return arr


def layout(L, n, z_doubles, n_hops):
    """Byte offsets {out, paths, z, hops, total} of the scratch of a query (asam_debug_marginal_layout)."""
    o = (C.c_int64 * 5)()
    _api(L).asam_debug_marginal_layout(n, z_doubles, n_hops, o)
    return dict(zip(("out", "paths", "z", "hops", "total"), (int(v) for v in o)))


def read_query(L, dev, recs, z_doubles, n_hops):
    """(Z: z_doubles, hop records: n_hops x 4) of the last asam_marginal_cov on the device context `dev`."""
    o = layout(L, len(recs), z_doubles, n_hops)
    Z = _read(L, dev, DBG_BUF_MARG, o["z"], np.zeros(z_doubles))
    hop = _read(L, dev, DBG_BUF_MARG, o["hops"], np.zeros((n_hops, 4), dtype=np.int32))
    return Z, hop


def read_dinv(L, dev, N):
    return _read(_api(L), dev, DBG_BUF_DINV, 0, np.zeros(3 * N))


# ---------------------------------------------------------------------------------------------
# checks
# ---------------------------------------------------------------------------------------------
def expected_hops(desc, recs, n_hops):
    """The hop records k_marginal_path must write: (supernode, js, c, offset from zoff) along each root chain."""
    out = np.full((n_hops, 4), -1, dtype=np.int32)
    for r in recs:
        off = 0
        for h, s in enumerate(chain(desc, r["sn0"])):
            js = int(r["j0"]) if h == 0 else 0
            c = 3 * int(desc["cb"][s])
            out[int(r["hop0"]) + h] = (s, js, c, off)
            off += 3 * (c - js)
    return out


def check_hops(desc, recs, hop):
    """Number of hop records that differ from the plan's root chains (must be 0)."""
    return int(np.count_nonzero(np.any(hop != expected_hops(desc, recs, len(hop)), axis=1)))


def hop_errors(snap, rec, Z):
    """[(supernode, js, c, m, error)] per hop of one pose, error = max_k |L11 z_h - b_h[js:c]|_k /
    (|L11||z_h| + S_h)_k with b_h and S_h rebuilt in long double from the kernel's z of the hop below."""
    d, ipool = snap.desc, snap.ipool
    s, js = int(rec["sn0"]), int(rec["j0"])
    m = 3 * int(d["mb"][s])
    b = np.zeros((m, 3), dtype=LD)
    b[js:js + 3] = np.eye(3)
    S = np.abs(b)
    off = int(rec["zoff"])
    out = []
    while True:
        F = snap.fronts[s][0]
        c = 3 * int(d["cb"][s])
        z = Z[off:off + 3 * (c - js)].reshape(-1, 3).astype(LD)
        off += 3 * (c - js)
        L11 = np.tril(F[:c, :c])[js:, js:].astype(LD)
        r = np.abs(L11 @ z - b[js:c])
        den = np.abs(L11) @ np.abs(z) + S[js:c]
        out.append((s, js, c, m, float(np.max(r / np.maximum(den, TINY)))))
        p = int(d["parent"][s])
        if p < 0:
            return out
        L21 = F[c:, js:c].astype(LD)
        u = b[c:] - L21 @ z
        su = S[c:] + np.abs(L21) @ np.abs(z)
        idx = _scatter_index(d, ipool, s)
        m = 3 * int(d["mb"][p])
        b = np.zeros((m, 3), dtype=LD); b[idx] = u
        S = np.zeros((m, 3), dtype=LD); S[idx] = su
        s, js = p, 0


def worst_hop(snap, recs, Z):
    """(worst hop error, (node index, supernode, js, c, m) where it is)."""
    worst, where = 0.0, None
    for k, r in enumerate(recs):
        for s, js, c, m, e in hop_errors(snap, r, Z):
            if e >= worst:
                worst, where = e, (k, s, js, c, m)
    return worst, where


def _hop_maps(recs, hop):
    out = []
    for r in recs:
        h0, nh, zo = int(r["hop0"]), int(r["nhop"]), int(r["zoff"])
        out.append({int(hop[h0 + t, 0]): (int(hop[h0 + t, 1]), int(hop[h0 + t, 2]), zo + int(hop[h0 + t, 3]))
                    for t in range(nh)})
    return out


def _block(hi, hj, Z, dtype, skip_lowest=False):
    """(sum Z_i'Z_j, sum |Z_i|'|Z_j|) over the shared hops, rows from max(js_i, js_j)."""
    acc = np.zeros((3, 3), dtype=dtype)
    ab = np.zeros((3, 3), dtype=dtype)
    shared = [s for s in hj if s in hi]  # in path order: the lowest first
    for s in shared[1:] if skip_lowest else shared:
        jsi, c, oi = hi[s]
        jsj, _, oj = hj[s]
        r0 = max(jsi, jsj)
        zi = Z[oi + 3 * (r0 - jsi):oi + 3 * (c - jsi)].reshape(-1, 3).astype(dtype)
        zj = Z[oj + 3 * (r0 - jsj):oj + 3 * (c - jsj)].reshape(-1, 3).astype(dtype)
        acc += zi.T @ zj
        ab += np.abs(zi).T @ np.abs(zj)
    return acc, ab


def gram(recs, hop, Z, skip_lowest=False):
    """Sigma (3n x 3n) from Z in float64 over the shared hops; skip_lowest leaves the lowest shared supernode out
    (a fault the CPU tests inject)."""
    hm = _hop_maps(recs, hop)
    n = len(recs)
    S = np.zeros((3 * n, 3 * n))
    for i in range(n):
        for j in range(i, n):
            S[3 * i:3 * i + 3, 3 * j:3 * j + 3] = _block(hm[i], hm[j], Z, np.float64, skip_lowest)[0]
            S[3 * j:3 * j + 3, 3 * i:3 * i + 3] = S[3 * i:3 * i + 3, 3 * j:3 * j + 3].T
    return S


def gram_errors(recs, hop, Z, Sig, pairs=None):
    """(max |Sigma_ij - sum Z_i'Z_j| / sum |terms| over the blocks `pairs` (all i <= j by default), number of
    blocks (j, i) that are not the exact transpose of (i, j)).  Sums in long double over the shared hops."""
    hm = _hop_maps(recs, hop)
    n = len(recs)
    if pairs is None:
        pairs = [(i, j) for i in range(n) for j in range(i, n)]
    worst = 0.0
    for i, j in pairs:
        acc, ab = _block(hm[i], hm[j], Z, LD)
        blk = Sig[3 * i:3 * i + 3, 3 * j:3 * j + 3].astype(LD)
        worst = max(worst, float(np.max(np.abs(blk - acc) / np.maximum(ab, TINY))))
    ntr = sum(int(not np.array_equal(Sig[3 * i:3 * i + 3, 3 * j:3 * j + 3].view(np.int64),
                                     Sig[3 * j:3 * j + 3, 3 * i:3 * i + 3].T.view(np.int64))) for i, j in pairs)
    return worst, ntr


def dinv_errors(snap, dinv, sns):
    """max over the columns of the supernodes `sns` of |dinv_k L_kk - 1| / u (long double)."""
    worst = 0.0
    for s in sns:
        first, c = int(snap.desc["first"][s]), 3 * int(snap.desc["cb"][s])
        Lkk = np.diag(snap.fronts[s][0])[:c].astype(LD)
        e = np.abs(dinv[3 * first:3 * first + c].astype(LD) * Lkk - 1) / LD(U)
        worst = max(worst, float(e.max(initial=0.0)))
    return worst


# ---------------------------------------------------------------------------------------------
# k_marginal_path's order in float64 (CPU tests)
# ---------------------------------------------------------------------------------------------
def kernel_path(snap, rec, dinv, fault=None):
    """Z of one pose (3 doubles per scalar row of its path) in the order of k_marginal_path.  fault:
      ("drop", hop, block, pass, group): that column group's partial sums of that 128-row pass are lost;
      ("scatter", hop, row): that row of u goes to the parent row after its own;
      ("pivot", hop, block, col): that column is solved with the reciprocal pivot of the previous block."""
    d, ipool = snap.desc, snap.ipool
    s, js, h = int(rec["sn0"]), int(rec["j0"]), 0
    b = np.zeros((3 * int(d["mb"][s]), 3))
    b[js:js + 3] = np.eye(3)
    out = []
    while True:
        F = snap.fronts[s][0]
        m, c, first = F.shape[0], 3 * int(d["cb"][s]), 3 * int(d["first"][s])
        for bi, b0 in enumerate(range(js, c, BSW)):
            be = min(b0 + BSW, c)
            for k in range(b0, be):
                piv = dinv[first + k - (BSW if fault == ("pivot", h, bi, k - b0) else 0)]
                b[k] = b[k] * piv
                b[k + 1:be] -= np.outer(F[k + 1:be, k], b[k])
            for p, base in enumerate(range(be, m, MROWS)):
                rows = slice(base, min(base + MROWS, m))
                tot = np.zeros((rows.stop - base, 3))
                for kg in range(BSW // MKG):
                    k0, k1 = b0 + kg * MKG, min(b0 + (kg + 1) * MKG, be)
                    if k0 < k1 and fault != ("drop", h, bi, p, kg):
                        tot = tot + F[rows, k0:k1] @ b[k0:k1]
                b[rows] -= tot
        out.append(b[js:c].reshape(-1).copy())
        p = int(d["parent"][s])
        if p < 0:
            return np.concatenate(out)
        idx = _scatter_index(d, ipool, s)
        if fault is not None and fault[:2] == ("scatter", h):
            idx = idx.copy()
            idx[fault[2]] += 1
        bn = np.zeros((3 * int(d["mb"][p]), 3))
        bn[idx] = b[c:]
        b, s, js, h = bn, p, 0, h + 1


# ---------------------------------------------------------------------------------------------
# what a request reaches (coverage of the kernels' edges)
# ---------------------------------------------------------------------------------------------
def coverage(plan, nodes, leaf_sns=()):
    """What the paths of `nodes` reach: hop widths c - js, rows below each block m - be, path lengths, and
    whether the request has two poses in one supernode with different j0, a path that is a suffix of another,
    a pair sharing only the root and a path starting at a leaf (warp) supernode."""
    d = plan.descs()
    recs, _, _ = paths(plan, nodes)
    out = dict(width=set(), below=set(), nhop=set(), same_sn=False, suffix=False, root_only=False, leaf_start=False)
    chains = []
    j0s = {}
    leaf = set(int(s) for s in leaf_sns)
    for r in recs:
        ch = chain(d, r["sn0"])
        chains.append(ch)
        out["nhop"].add(len(ch))
        j0s.setdefault(ch[0], set()).add(int(r["j0"]))
        out["leaf_start"] |= ch[0] in leaf
        for h, s in enumerate(ch):
            js = int(r["j0"]) if h == 0 else 0
            c, m = 3 * int(d["cb"][s]), 3 * int(d["mb"][s])
            out["width"].add(c - js)
            out["below"] |= {m - min(b0 + BSW, c) for b0 in range(js, c, BSW)}
    out["same_sn"] = any(len(v) > 1 for v in j0s.values())
    sets = [tuple(c) for c in chains]
    for a in sets:
        for b in sets:
            if len(a) < len(b) and b[len(b) - len(a):] == a:
                out["suffix"] = True
            if a[-1] == b[-1] and len(a) > 1 and len(b) > 1 and a[-2] != b[-2]:
                out["root_only"] = True
    return out


def query_report(h, L, snap, nodes, pairs=None, hop_poses=None):
    """h.marginal_covariance(nodes), then every check above on what the kernels left in the scratch (against the
    fronts of `snap`, which must hold every supernode on the paths).  Returns (Sigma, worst values: hop and gram in
    units of u).  pairs / hop_poses: the blocks and poses checked in long double (all by default)."""
    dev = L.asam_dbg_dev_of_graph(h.graph_ptr())
    nodes = np.ascontiguousarray(nodes, dtype=np.int32)
    S = h.marginal_covariance(nodes)
    recs, zt, ht = paths(snap.plan, nodes)
    Z, hop = read_query(L, dev, recs, zt, ht)
    dinv = read_dinv(L, dev, len(snap.q2node))
    sns = sorted({s for r in recs for s in chain(snap.desc, r["sn0"])})
    sel = recs if hop_poses is None else recs[np.asarray(hop_poses)]
    hop_e, where = worst_hop(snap, sel, Z)
    gram_e, ntr = gram_errors(recs, hop, Z, S, pairs)
    return S, dict(n=len(nodes), hops_bad=check_hops(snap.desc, recs, hop), hop=hop_e / U, hop_at=where,
                   gram=gram_e / U, transpose_bad=ntr, dinv=dinv_errors(snap, dinv, sns),
                   symmetric=bool(np.array_equal(S, S.T)))
