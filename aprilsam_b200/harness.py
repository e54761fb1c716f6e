"""ctypes wrapper around harness/harness.c (one C driver, built against either library).

`Harness("b200")` drives aprilsam_b200's drop-in library; `Harness("reference")` drives
the unmodified reference built by oracle/Makefile into oracle/_ref/ (deterministic
clock) and `Harness("reference_wallclock")` the reference exactly as shipped.  The
reference flavours are ORACLE / BASELINE tooling: only tests/, bench.py's reference
arm and __graft_entry__.smoke() may construct them.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_PATHS = {
    "b200": os.path.join(ROOT, "harness", "_build", "harness_b200.so"),
    "reference": os.path.join(ROOT, "oracle", "_ref", "harness_ref.so"),
    "reference_wallclock": os.path.join(ROOT, "oracle", "_ref", "harness_refwc.so"),
}

_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)


def _d(a):
    return a.ctypes.data_as(_dp)


def _i(a):
    return a.ctypes.data_as(_ip)


def available(impl: str) -> bool:
    return os.path.exists(_PATHS[impl])


_LIBS: dict[str, C.CDLL] = {}


def _load(impl: str) -> C.CDLL:
    if impl in _LIBS:
        return _LIBS[impl]
    path = _PATHS[impl]
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} missing - run `python -c 'import __graft_entry__ as g; g.build()'`")
    lib = C.CDLL(path, mode=os.RTLD_LOCAL | os.RTLD_NOW)
    lib.h_impl.restype = C.c_char_p
    lib.h_create.restype = C.c_void_p
    lib.h_create.argtypes = [C.c_double, C.c_double, C.c_int]
    lib.h_destroy.argtypes = [C.c_void_p]
    lib.h_set_tikhanov.argtypes = [C.c_void_p, C.c_double]
    for name in ("h_nnodes", "h_nfactors"):
        getattr(lib, name).argtypes = [C.c_void_p]
        getattr(lib, name).restype = C.c_int
    lib.h_add_node.argtypes = [C.c_void_p, _dp]
    lib.h_add_xyt.argtypes = [C.c_void_p, C.c_int, C.c_int, _dp, _dp]
    lib.h_add_xytpos.argtypes = [C.c_void_p, C.c_int, _dp, _dp]
    # entry points added with robust factors: a prebuilt reference harness (oracle/_ref/, kept where the reference
    # sources are absent) may predate them, and the reference flavours never call them
    for name, args in (("h_add_xyt_robust", [C.c_void_p, C.c_int, C.c_int, _dp, _dp, C.c_int, C.c_double]),
                       ("h_set_loss", [C.c_void_p, C.c_int, C.c_int, C.c_double]),
                       ("h_set_scan_loss", [C.c_void_p, C.c_int, C.c_double]),
                       ("h_eval", [C.c_void_p, C.c_int, C.c_int, _dp]),
                       ("h_copy_factor", [C.c_void_p, C.c_int]),
                       ("h_dof", [C.c_void_p])):
        if hasattr(lib, name):
            getattr(lib, name).argtypes = args
        elif impl == "b200":
            raise AttributeError(f"{path}: {name} missing - rebuild with aprilsam_b200.build")
    # covariance queries: only libraries that export them (never the reference build)
    for name, args in (("h_marginal_cov", [C.c_void_p, C.c_int, _ip, _dp]),
                       ("h_relative_cov", [C.c_void_p, C.c_int, C.c_int, _dp]),
                       ("h_candidate_mahalanobis", [C.c_void_p, C.c_int, _ip, _ip, _dp, _dp, _dp, _dp]),
                       ("h_candidate_compatibility", [C.c_void_p, C.c_int, _ip, _ip, _dp, _dp, _dp, _dp]),
                       ("h_factor_residuals", [C.c_void_p, C.c_int, C.c_int, _dp]),
                       ("h_factor_outlier_scores", [C.c_void_p, C.c_int, _ip, _dp, _dp, _dp]),
                       ("h_remove_factors", [C.c_void_p, C.c_int, _ip, C.c_int]),
                       ("h_relinearize_poses", [C.c_void_p, C.c_int, _ip])):
        if hasattr(lib, name):
            getattr(lib, name).argtypes = args
            getattr(lib, name).restype = C.c_int
    for name, args, res in (("h_param_create", [C.c_void_p], C.c_void_p), ("h_param_destroy", [C.c_void_p], None),
                            ("h_swap_param", [C.c_void_p, C.c_void_p], C.c_void_p),
                            ("h_set_relin_in_place", [C.c_void_p, C.c_int], None),
                            ("h_relin_stats", [C.c_void_p, _dp], None),
                            ("h_get_linearized", [C.c_void_p, _ip, C.c_int], C.c_int)):
        if hasattr(lib, name):
            getattr(lib, name).argtypes = args
            getattr(lib, name).restype = res
    if hasattr(lib, "aprilsam_b200_last_error"):
        lib.aprilsam_b200_last_error.restype = C.c_char_p
    lib.h_relinearize.argtypes = [C.c_void_p, C.c_int]
    lib.h_get.argtypes = [C.c_void_p, C.c_int, _dp]
    lib.h_set.argtypes = [C.c_void_p, C.c_int, _dp]
    lib.h_chi2.argtypes = [C.c_void_p]
    lib.h_chi2.restype = C.c_double
    for name in ("h_batch", "h_inc"):
        getattr(lib, name).argtypes = [C.c_void_p]
        getattr(lib, name).restype = C.c_double
    lib.h_info.argtypes = [C.c_void_p, _ip]
    lib.h_get_ordering.argtypes = [C.c_void_p, _ip, C.c_int]
    lib.h_get_ordering.restype = C.c_int
    lib.h_get_tree_parents.argtypes = [C.c_void_p, _ip, C.c_int]
    lib.h_get_tree_parents.restype = C.c_int
    lib.h_replay.argtypes = [C.c_void_p, C.c_int, _dp, _ip, _ip, _ip, _dp, _dp, C.c_int,
                             C.c_int, C.c_int, _dp, _dp, _ip]
    lib.h_replay.restype = C.c_int
    lib.h_graph.argtypes = [C.c_void_p]
    lib.h_graph.restype = C.c_void_p
    lib.h_param.argtypes = [C.c_void_p]
    lib.h_param.restype = C.c_void_p
    lib.h_load_full.argtypes = [C.c_void_p, C.c_int, _dp, C.c_int, _ip, _ip, _dp, _dp]
    lib.h_save.argtypes = [C.c_void_p, C.c_char_p]
    lib.h_load.argtypes = [C.c_void_p, C.c_char_p]
    lib.h_attr_put_string.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_char_p, C.c_char_p]
    lib.h_attr_put_u64.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_char_p, C.c_uint64]
    lib.h_attr_get.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_char_p]
    lib.h_attr_get.restype = C.c_void_p
    lib.h_factor.argtypes = [C.c_void_p, C.c_int, _dp]
    lib.h_set_factor.argtypes = [C.c_void_p, C.c_int, _dp, _dp]
    lib.h_replace_xyt.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, _dp, _dp]
    lib.h_invalidate_plan.argtypes = [C.c_void_p]
    lib.h_set_policy_ratio.argtypes = [C.c_void_p, C.c_double]
    lib.h_set_show_timing.argtypes = [C.c_void_p, C.c_int]
    lib.h_inc_solver.argtypes = [C.c_void_p]
    _LIBS[impl] = lib
    return lib


@dataclass
class PoseGraphData:
    """A pose graph in the reference demo's text-file terms (VERTEX2 / EDGE2)."""
    init: np.ndarray   # (N,3) float64  VERTEX2 x y theta
    ea: np.ndarray     # (E,) int32     EDGE2 IDout
    eb: np.ndarray     # (E,) int32     EDGE2 IDin
    ez: np.ndarray     # (E,3) float64  dx dy dth
    eW: np.ndarray     # (E,9) float64  row-major 3x3 as the demo loader fills it
    truth: np.ndarray | None = None  # (N,3) ground-truth poses in the frame of pose 0 (synthetic graphs only)

    @property
    def n_nodes(self) -> int:
        return int(self.init.shape[0])

    @property
    def n_edges(self) -> int:
        return int(self.ea.shape[0])

    def bucketed(self) -> tuple["PoseGraphData", np.ndarray]:
        """Edges stably bucketed by max(node id) -> (data, estart[N+1])."""
        key = np.maximum(self.ea, self.eb)
        order = np.argsort(key, kind="stable")
        d = PoseGraphData(self.init, self.ea[order].copy(), self.eb[order].copy(),
                          self.ez[order].copy(), self.eW[order].copy(), self.truth)
        estart = np.searchsorted(key[order], np.arange(self.n_nodes + 1), side="left").astype(np.int32)
        return d, estart

    def save(self, path: str) -> None:
        np.savez_compressed(path, init=self.init, ea=self.ea, eb=self.eb, ez=self.ez, eW=self.eW)

    @staticmethod
    def load(path: str) -> "PoseGraphData":
        z = np.load(path)
        return PoseGraphData(np.ascontiguousarray(z["init"], dtype=np.float64),
                             np.ascontiguousarray(z["ea"], dtype=np.int32),
                             np.ascontiguousarray(z["eb"], dtype=np.int32),
                             np.ascontiguousarray(z["ez"], dtype=np.float64),
                             np.ascontiguousarray(z["eW"], dtype=np.float64))

    def head(self, n: int) -> "PoseGraphData":
        """Sub-graph induced by the first n poses."""
        keep = (self.ea < n) & (self.eb < n)
        return PoseGraphData(self.init[:n].copy(), self.ea[keep].copy(), self.eb[keep].copy(),
                             self.ez[keep].copy(), self.eW[keep].copy(),
                             None if self.truth is None else self.truth[:n].copy())


class Harness:
    """One graph + one april_graph_cholesky_param_t, driven through the public C API."""

    def __init__(self, impl: str = "b200", delta_xy: float = 0.1, delta_theta: float = 0.1,
                 nthreshold: int = 100):
        self.impl = impl
        self.lib = _load(impl)
        self.h = C.c_void_p(self.lib.h_create(delta_xy, delta_theta, nthreshold))
        self._replay = None

    def close(self):
        if self.h:
            self.lib.h_destroy(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    # -- graph construction ------------------------------------------------------------
    def add_node(self, xyt) -> int:
        a = np.ascontiguousarray(xyt, dtype=np.float64)
        return self.lib.h_add_node(self.h, _d(a))

    def add_xyt(self, a: int, b: int, z, W) -> int:
        z = np.ascontiguousarray(z, dtype=np.float64)
        W = np.ascontiguousarray(W, dtype=np.float64).reshape(9)
        return self.lib.h_add_xyt(self.h, a, b, _d(z), _d(W))

    def add_xytpos(self, a: int, z, W) -> int:
        z = np.ascontiguousarray(z, dtype=np.float64)
        W = np.ascontiguousarray(W, dtype=np.float64).reshape(9)
        return self.lib.h_add_xytpos(self.h, a, _d(z), _d(W))

    # robust loop closures (aprilsam_b200 extension: the reference build returns -1 / ignores them)
    HUBER, CAUCHY = 1, 2

    def add_xyt_robust(self, a: int, b: int, z, W, loss: int, k: float) -> int:
        """aprilsam_b200_factor_xyt_robust_create + append; -1 (no factor) for an invalid loss / k."""
        z = np.ascontiguousarray(z, dtype=np.float64)
        W = np.ascontiguousarray(W, dtype=np.float64).reshape(9)
        return self.lib.h_add_xyt_robust(self.h, a, b, _d(z), _d(W), int(loss), float(k))

    def set_loss(self, idx: int, loss: int, k: float) -> int:
        """aprilsam_b200_factor_set_loss on factor idx: 0 ok, -1 otherwise."""
        return self.lib.h_set_loss(self.h, idx, int(loss), float(k))

    def set_scan_loss(self, loss: int, k: float = 0.0) -> None:
        """replay_to / load_full create every scan edge (|a - b| != 1) as a robust factor; loss 0 = plain xyt."""
        self.lib.h_set_scan_loss(self.h, int(loss), float(k))

    def eval(self, idx: int, at_state: bool = False):
        """The factor's eval (l_point) or state_eval (state) hook -> (r, J0, J1, W, chi2), None if unset."""
        out = np.zeros(31, dtype=np.float64)
        if self.lib.h_eval(self.h, idx, int(at_state), _d(out)) < 0:
            return None
        return out[:3].copy(), out[3:12].reshape(3, 3).copy(), out[12:21].reshape(3, 3).copy(), \
            out[21:30].reshape(3, 3).copy(), float(out[30])

    def copy_factor(self, idx: int) -> int:
        """Append factor->copy(factor); returns the new index."""
        return self.lib.h_copy_factor(self.h, idx)

    def dof(self) -> int:
        return self.lib.h_dof(self.h)

    def marginal_covariance(self, ids):
        """aprilsam_b200_marginal_covariance: (3n x 3n) covariance of the poses `ids` from the last solve's factor.
        Raises RuntimeError with the library's message when it returns -1."""
        ids = np.ascontiguousarray(ids, dtype=np.int32).reshape(-1)
        out = np.zeros((3 * len(ids), 3 * len(ids)), dtype=np.float64)
        if self.lib.h_marginal_cov(self.h, len(ids), _i(ids), _d(out)) != 0:
            raise RuntimeError(self.lib.aprilsam_b200_last_error().decode())
        return out

    def relative_covariance(self, a: int, b: int):
        """aprilsam_b200_relative_covariance: 3 x 3 covariance of pose b in pose a's frame."""
        out = np.zeros((3, 3), dtype=np.float64)
        if self.lib.h_relative_cov(self.h, int(a), int(b), _d(out)) != 0:
            raise RuntimeError(self.lib.aprilsam_b200_last_error().decode())
        return out

    def candidate_mahalanobis(self, a, b, z, W, with_cov: bool = False):
        """aprilsam_b200_candidate_mahalanobis: d2 (k,) of the candidate factors (a[c], b[c]; b[c] = -1 for a prior)
        with measurements z (k x 3) and information matrices W (k x 9 or k x 3 x 3); with_cov also returns
        Sigma_rel (k x 3 x 3).  Raises RuntimeError with the library's message when it returns -1."""
        a = np.ascontiguousarray(a, dtype=np.int32).reshape(-1)
        b = np.ascontiguousarray(b, dtype=np.int32).reshape(-1)
        k = len(a)
        if len(b) != k:
            raise ValueError(f"a has {k} ids, b {len(b)}")
        z = np.ascontiguousarray(z, dtype=np.float64).reshape(k, 3)
        W = np.ascontiguousarray(W, dtype=np.float64).reshape(k, 9)
        d2 = np.zeros(k, dtype=np.float64)
        cov = np.zeros((k, 3, 3), dtype=np.float64) if with_cov else None
        if self.lib.h_candidate_mahalanobis(self.h, k, _i(a), _i(b), _d(z), _d(W), _d(d2),
                                            _d(cov) if with_cov else None) != 0:
            raise RuntimeError(self.lib.aprilsam_b200_last_error().decode())
        return (d2, cov) if with_cov else d2

    def candidate_compatibility(self, a, b, z, W, with_cross: bool = False):
        """aprilsam_b200_candidate_compatibility: d2 (k, k) of the candidates' pairs (diagonal: each candidate's own
        candidate_mahalanobis d2; off the diagonal: the joint distance of the pair, 6 degrees of freedom); with_cross
        also returns C (k, k, 3, 3), the cross-covariances of the residuals (C[c, c] = Sigma_rel of c).  Candidates as
        for candidate_mahalanobis.  Raises RuntimeError with the library's message when it returns -1."""
        a = np.ascontiguousarray(a, dtype=np.int32).reshape(-1)
        b = np.ascontiguousarray(b, dtype=np.int32).reshape(-1)
        k = len(a)
        if len(b) != k:
            raise ValueError(f"a has {k} ids, b {len(b)}")
        z = np.ascontiguousarray(z, dtype=np.float64).reshape(k, 3)
        W = np.ascontiguousarray(W, dtype=np.float64).reshape(k, 9)
        n = max(k, 1)
        d2 = np.zeros((n, n), dtype=np.float64)
        cross = np.zeros((n, n, 3, 3), dtype=np.float64) if with_cross else None
        if self.lib.h_candidate_compatibility(self.h, k, _i(a), _i(b), _d(z), _d(W), _d(d2),
                                              _d(cross) if with_cross else None) != 0:
            raise RuntimeError(self.lib.aprilsam_b200_last_error().decode())
        return (d2[:k, :k], cross[:k, :k]) if with_cross else d2[:k, :k]

    def factor_residuals(self, first: int = 0, count=None):
        """aprilsam_b200_factor_residuals: (count, 6) rows {r[0], r[1], r[2], s = r'Wr, w, chi2} of factors
        [first, first + count) at the states (count None: up to the last factor).  Raises RuntimeError with the
        library's message when it returns -1."""
        if count is None:
            count = max(self.n_factors - int(first), 0)
        out = np.zeros((max(int(count), 1), 6), dtype=np.float64)
        if self.lib.h_factor_residuals(self.h, int(first), int(count), _d(out)) != 0:
            raise RuntimeError(self.lib.aprilsam_b200_last_error().decode())
        return out[:int(count)]

    def factor_outlier_scores(self, idx, with_cov: bool = False):
        """aprilsam_b200_factor_outlier_scores: (d2, redundancy), each (k,), the leave-one-out Mahalanobis distances
        and redundancies of factors idx against the last solve; with_cov also returns Sigma_rel (k x 3 x 3).  Raises
        RuntimeError with the library's message when it returns -1."""
        idx = np.ascontiguousarray(idx, dtype=np.int32).reshape(-1)
        k = len(idx)
        d2 = np.zeros(max(k, 1), dtype=np.float64)
        red = np.zeros(max(k, 1), dtype=np.float64)
        cov = np.zeros((max(k, 1), 3, 3), dtype=np.float64) if with_cov else None
        if self.lib.h_factor_outlier_scores(self.h, k, _i(idx), _d(d2), _d(red), _d(cov) if with_cov else None) != 0:
            raise RuntimeError(self.lib.aprilsam_b200_last_error().decode())
        return (d2[:k], red[:k], cov[:k]) if with_cov else (d2[:k], red[:k])

    def remove_factors(self, idx, keep: bool = False) -> None:
        """aprilsam_b200_remove_factors: take factors idx out of the graph (the others keep their order) and update the
        solution like an incremental step.  keep: the removed factors are handed back (and destroyed by the harness)
        instead of being destroyed by the library.  Raises RuntimeError with the library's message when it returns -1."""
        idx = np.ascontiguousarray(idx, dtype=np.int32).reshape(-1)
        if self.lib.h_remove_factors(self.h, len(idx), _i(idx), int(keep)) != 0:
            raise RuntimeError(self.lib.aprilsam_b200_last_error().decode())

    def relinearize_poses(self, ids=None) -> None:
        """aprilsam_b200_relinearize_poses: relinearise the poses `ids` in place (l_point = state) and update the
        solution like an incremental step.  ids None: the poses the tree has flagged, passing the tree's own list
        (tr->linearized_nodes).  Not the node hook `relinearize(i)`.  Raises RuntimeError with the library's message
        when it returns -1."""
        if ids is None:
            rc = self.lib.h_relinearize_poses(self.h, 0, None)
        else:
            ids = np.ascontiguousarray(ids, dtype=np.int32).reshape(-1)
            rc = self.lib.h_relinearize_poses(self.h, len(ids), _i(ids))
        if rc != 0:
            raise RuntimeError(self.lib.aprilsam_b200_last_error().decode())

    def set_relin_in_place(self, threshold: int) -> None:
        """replay_to relinearises the flagged poses in place after every step that leaves start_over above
        `threshold` (its time counts in the step's ms); a negative threshold (the default) turns it off."""
        self.lib.h_set_relin_in_place(self.h, int(threshold))

    def relin_stats(self) -> tuple[int, float]:
        """(relinearisations replay_to made, their wall ms)."""
        out = np.zeros(2, dtype=np.float64)
        self.lib.h_relin_stats(self.h, _d(out))
        return int(out[0]), float(out[1])

    def new_param(self) -> int:
        """A further april_graph_cholesky_param_t for this graph (same settings); swap it in with swap_param."""
        return self.lib.h_param_create(self.h)

    def swap_param(self, p: int) -> int:
        """Make p the param every call goes through; returns the one it replaces (free it with free_param)."""
        return self.lib.h_swap_param(self.h, C.c_void_p(p))

    def free_param(self, p: int) -> None:
        self.lib.h_param_destroy(C.c_void_p(p))

    def last_error(self) -> str:
        return self.lib.aprilsam_b200_last_error().decode()

    def relinearize(self, i: int):
        self.lib.h_relinearize(self.h, i)

    def load_full(self, d: PoseGraphData):
        self.lib.h_load_full(self.h, d.n_nodes, _d(d.init), d.n_edges, _i(d.ea), _i(d.eb), _d(d.ez), _d(d.eW))

    # -- files and attributes (aprilsam.h:185, :288-299) --------------------------------------
    GRAPH, NODE, FACTOR = 0, 1, 2

    def save(self, path: str) -> bool:
        return bool(self.lib.h_save(self.h, path.encode()))

    def load(self, path: str) -> int:
        """Replace the graph by the one stored in `path`; returns the node count (-1: failure)."""
        return self.lib.h_load(self.h, path.encode())

    def attr_put(self, which: int, idx: int, key: str, value) -> None:
        if isinstance(value, str):
            self.lib.h_attr_put_string(self.h, which, idx, key.encode(), value.encode())
        else:
            self.lib.h_attr_put_u64(self.h, which, idx, key.encode(), int(value))

    def attr_get(self, which: int, idx: int, key: str, kind: str = "string"):
        p = self.lib.h_attr_get(self.h, which, idx, key.encode())
        if not p:
            return None
        return C.cast(p, C.c_char_p).value.decode() if kind == "string" else C.cast(p, C.POINTER(C.c_uint64))[0]

    def factor(self, idx: int):
        out = np.zeros(14, dtype=np.float64)
        t = self.lib.h_factor(self.h, idx, _d(out))
        return t, int(out[0]), int(out[1]), out[2:5].copy(), out[5:14].copy()

    def set_factor(self, idx: int, z, W) -> None:
        """Overwrite z / W of factor idx in place (the caller-side edit the reference honours on the next batch call)."""
        z = np.ascontiguousarray(z, dtype=np.float64)
        W = np.ascontiguousarray(W, dtype=np.float64).reshape(9)
        self.lib.h_set_factor(self.h, idx, _d(z), _d(W))

    def replace_xyt(self, idx: int, a: int, b: int, z, W) -> None:
        z = np.ascontiguousarray(z, dtype=np.float64)
        W = np.ascontiguousarray(W, dtype=np.float64).reshape(9)
        self.lib.h_replace_xyt(self.h, idx, a, b, _d(z), _d(W))

    def invalidate_plan(self) -> None:
        """aprilsam_b200 extension: the next batch call orders + analyses again (no-op for the reference)."""
        self.lib.h_invalidate_plan(self.h)

    def set_policy_ratio(self, ratio: float) -> None:
        """aprilsam_b200 extension: deterministic escalation policy (no-op for the reference)."""
        self.lib.h_set_policy_ratio(self.h, ratio)

    def set_show_timing(self, on: bool) -> None:
        self.lib.h_set_show_timing(self.h, int(on))

    # -- state access ------------------------------------------------------------------
    @property
    def n_nodes(self) -> int:
        return self.lib.h_nnodes(self.h)

    @property
    def n_factors(self) -> int:
        return self.lib.h_nfactors(self.h)

    def _get(self, which: int) -> np.ndarray:
        out = np.empty((self.n_nodes, 3), dtype=np.float64)
        self.lib.h_get(self.h, which, _d(out))
        return out

    def _set(self, which: int, v):
        v = np.ascontiguousarray(v, dtype=np.float64).reshape(self.n_nodes, 3)
        self.lib.h_set(self.h, which, _d(v))

    def states(self):
        return self._get(0)

    def l_points(self):
        return self._get(1)

    def delta_X(self):
        return self._get(2)

    def set_states(self, v):
        self._set(0, v)

    def set_tikhanov(self, lam: float):
        self.lib.h_set_tikhanov(self.h, lam)

    # -- solver ------------------------------------------------------------------------
    def batch(self) -> float:
        """april_graph_cholesky(); returns host wall ms."""
        return self.lib.h_batch(self.h)

    def inc(self) -> float:
        """april_graph_cholesky_inc(); returns host wall ms."""
        return self.lib.h_inc(self.h)

    def chi2(self) -> float:
        return self.lib.h_chi2(self.h)

    def inc_solver(self) -> None:
        """april_graph_cholesky_inc_solver(graph, param, NULL)."""
        self.lib.h_inc_solver(self.h)

    def info(self) -> dict:
        a = np.zeros(8, dtype=np.int32)
        self.lib.h_info(self.h, _i(a))
        return dict(naffected=int(a[0]), start_over=int(a[1]), nlinearized=int(a[2]), tree_nnodes=int(a[3]),
                    root=int(a[4]), nreordering=int(a[5]), factor_num=int(a[6]))

    def ordering(self) -> np.ndarray:
        out = np.zeros(max(self.n_nodes, 1), dtype=np.int32)
        n = self.lib.h_get_ordering(self.h, _i(out), out.size)
        return out[:n]

    def tree_parents(self) -> np.ndarray:
        out = np.zeros(max(self.n_nodes, 1), dtype=np.int32)
        n = self.lib.h_get_tree_parents(self.h, _i(out), out.size)
        return out[:n]

    def linearized_nodes(self) -> np.ndarray:
        """tr->linearized_nodes: the poses flagged since the last batch solve, in the order they were flagged."""
        out = np.zeros(max(self.n_nodes, 1), dtype=np.int32)
        n = self.lib.h_get_linearized(self.h, _i(out), out.size)
        return out[:n]

    def graph_ptr(self) -> int:
        return self.lib.h_graph(self.h)

    def param_ptr(self) -> int:
        return self.lib.h_param(self.h)

    # -- demo-protocol replay ------------------------------------------------------------
    def replay_begin(self, d: PoseGraphData):
        self._replay = d.bucketed()

    def replay_to(self, step_end: int, batch_only: bool = False, want_chi2: bool = True):
        """Run demo steps up to (excluding) step_end; returns (chi2[], ms[], info[][8])."""
        d, estart = self._replay
        n = max(0, min(step_end, d.n_nodes))
        chi2 = np.zeros(n + 1, dtype=np.float64)
        ms = np.zeros(n + 1, dtype=np.float64)
        info = np.zeros((n + 1, 8), dtype=np.int32)
        done = self.lib.h_replay(self.h, d.n_nodes, _d(d.init), _i(estart), _i(d.ea), _i(d.eb), _d(d.ez),
                                 _d(d.eW), int(step_end), int(batch_only), int(want_chi2), _d(chi2), _d(ms),
                                 _i(info))
        return chi2[:done], ms[:done], info[:done]
