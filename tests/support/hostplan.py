"""ctypes access to the host symbolic layer (asam_dbg_* exports; no GPU needed)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
LIBPATH = os.path.join(ROOT, "aprilsam_b200", "lib", "libaprilsam_b200.so")
_ip = C.POINTER(C.c_int)

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(LIBPATH, mode=os.RTLD_LOCAL | os.RTLD_NOW)
        L.asam_dbg_plan_create.restype = C.c_void_p
        L.asam_dbg_plan_destroy.argtypes = [C.c_void_p]
        L.asam_dbg_plan_build.argtypes = [C.c_void_p, C.c_int, C.c_int, _ip, _ip, _ip]
        L.asam_dbg_plan_build_sharded.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, _ip, _ip, _ip]
        L.asam_dbg_plan_build_with_order.argtypes = [C.c_void_p, C.c_int, C.c_int, _ip, _ip, _ip, _ip, C.c_int]
        L.asam_dbg_plan_append.argtypes = [C.c_void_p, C.c_int, C.c_int, _ip, _ip, _ip, _ip, C.c_int, _ip, _ip, _ip, C.c_int]
        L.asam_dbg_plan_info.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_double)]
        L.asam_dbg_plan_array.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int64)]
        L.asam_dbg_plan_array.restype = _ip
        L.asam_dbg_ref_ordering.argtypes = [C.c_int, _ip, _ip, _ip]
        L.asam_dbg_ref_ordering_explicit.argtypes = [C.c_int, _ip, _ip, _ip]
        L.aprilsam_b200_last_error.restype = C.c_char_p
        _lib = L
    return _lib


def _i(a):
    return a.ctypes.data_as(_ip)


ARR = dict(order=0, pos=1, node2q=2, q2node=3, parent_pos=4, fslot=5, sn_of_q=6, ipool=7, tasks=8, nwait=9,
           btasks=10, desc=11, leaf_tasks=12, top_tasks=13, top_nwait=14, shard_owner=15,
           shard_q0=16, shard_qn=17, shard_off=18, shard_cnt=19)
TR_FLAG = 1 << 30


class HostPlan:
    """The numeric plan exactly as it is uploaded to HBM (descriptors + int pool)."""

    def __init__(self):
        self.L = lib()
        self.p = C.c_void_p(self.L.asam_dbg_plan_create())

    def close(self):
        if self.p:
            self.L.asam_dbg_plan_destroy(self.p)
            self.p = None

    def __del__(self):
        self.close()

    def build(self, N, ftype, fa, fb, order_keep=None, world=1, rank=0):
        self.ftype = np.ascontiguousarray(ftype, dtype=np.int32)
        self.fa = np.ascontiguousarray(fa, dtype=np.int32)
        self.fb = np.ascontiguousarray(fb, dtype=np.int32)
        if world > 1:
            rc = self.L.asam_dbg_plan_build_sharded(self.p, world, rank, N, len(self.ftype), _i(self.ftype),
                                                    _i(self.fa), _i(self.fb))
        elif order_keep is None:
            rc = self.L.asam_dbg_plan_build(self.p, N, len(self.ftype), _i(self.ftype), _i(self.fa), _i(self.fb))
        else:
            ok = np.ascontiguousarray(order_keep, dtype=np.int32)
            rc = self.L.asam_dbg_plan_build_with_order(self.p, N, len(self.ftype), _i(self.ftype), _i(self.fa),
                                                       _i(self.fb), _i(ok), len(ok))
        if rc:
            raise RuntimeError(self.L.aprilsam_b200_last_error().decode())
        return self

    def append(self, N, ftype, fa, fb, marked):
        self.ftype = np.ascontiguousarray(ftype, dtype=np.int32)
        self.fa = np.ascontiguousarray(fa, dtype=np.int32)
        self.fb = np.ascontiguousarray(fb, dtype=np.int32)
        marked = np.ascontiguousarray(marked, dtype=np.int32)
        cap = N + 16
        tasks = np.zeros(cap, dtype=np.int32)
        nwait = np.zeros(cap, dtype=np.int32)
        keep = np.zeros(cap, dtype=np.int32)
        nt = self.L.asam_dbg_plan_append(self.p, N, len(self.ftype), _i(self.ftype), _i(self.fa), _i(self.fb),
                                         _i(marked), len(marked), _i(tasks), _i(nwait), _i(keep), cap)
        if nt == -2:
            return None
        if nt < 0:
            raise RuntimeError(self.L.aprilsam_b200_last_error().decode())
        self.last_keep = keep[:nt].copy()
        return tasks[:nt].copy(), nwait[:nt].copy()

    def info(self):
        a = (C.c_int64 * 16)()
        fl = C.c_double()
        self.L.asam_dbg_plan_info(self.p, a, C.byref(fl))
        keys = ["N", "nsn", "n_slots", "ipool_n", "arena_n", "max_m", "nnz_l_blocks", "n_levels", "n_factors", "n_bs_leaf"]
        d = {k: int(a[i]) for i, k in enumerate(keys)}
        d["flops"] = fl.value
        return d

    def array(self, name):
        n = C.c_int64()
        ptr = self.L.asam_dbg_plan_array(self.p, ARR[name], C.byref(n))
        if n.value == 0:
            return np.zeros(0, dtype=np.int32)
        return np.ctypeslib.as_array(ptr, shape=(n.value,)).copy()

    def array64(self, name):
        return self.array(name).view(np.int64)

    def descs(self):
        """Structured view of asam_sn_desc_t[]."""
        raw = self.array("desc").reshape(-1, 12)
        f_off = raw[:, 8:10].copy().view(np.int64).reshape(-1)
        return dict(first=raw[:, 0], cb=raw[:, 1], mb=raw[:, 2], parent=raw[:, 3], seg=raw[:, 4], ch_cnt=raw[:, 5],
                    a_cnt=raw[:, 6], level=raw[:, 7], f_off=f_off)


def ref_ordering(N, pairs_lo, pairs_hi, explicit=False):
    """Run the library's ordering on an undirected edge list (explicit: the O(sum d^2) cross-check)."""
    import scipy.sparse as sp
    A = sp.coo_matrix((np.ones(len(pairs_lo)), (pairs_lo, pairs_hi)), shape=(N, N))
    A = ((A + A.T) > 0).astype(np.int8).tocsr()
    A.setdiag(0)
    A.eliminate_zeros()
    A.sort_indices()
    ptr = A.indptr.astype(np.int32)
    idx = A.indices.astype(np.int32)
    out = np.zeros(N, dtype=np.int32)
    (lib().asam_dbg_ref_ordering_explicit if explicit else lib().asam_dbg_ref_ordering)(N, _i(ptr), _i(idx), _i(out))
    return out
