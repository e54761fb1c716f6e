"""ctypes declarations of the kernel-level C-ABI (include/asam_cuda.h) and of the test-only
accessors, for bench.py / tools / tests.  The product API is the C library itself; this module
only lets Python reach the device context a graph already owns."""
from __future__ import annotations

import ctypes as C
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBPATH = os.path.join(ROOT, "aprilsam_b200", "lib", "libaprilsam_b200.so")

_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)
_fp = C.POINTER(C.c_float)
_lib = None


def lib() -> C.CDLL:
    """The drop-in library.  Raises if it has not been built: there is no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIBPATH):
        raise FileNotFoundError(f"{LIBPATH} missing: run `python -m aprilsam_b200.build` (needs nvcc)")
    L = C.CDLL(LIBPATH, mode=os.RTLD_LOCAL | os.RTLD_NOW)
    L.asam_last_error.restype = C.c_char_p
    L.aprilsam_b200_last_error.restype = C.c_char_p
    L.asam_device_count.restype = C.c_int
    L.asam_dbg_dev_of_graph.argtypes = [C.c_void_p]
    L.asam_dbg_dev_of_graph.restype = C.c_void_p
    L.asam_dbg_plan_of_param.argtypes = [C.c_void_p]
    L.asam_dbg_plan_of_param.restype = C.c_void_p
    L.asam_dbg_plan_info.argtypes = [C.c_void_p, C.POINTER(C.c_int64), _dp]
    L.asam_hessian_reset.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double]
    L.asam_linearize.argtypes = [C.c_void_p, C.c_int, C.c_int, _dp]
    L.asam_factor_full.argtypes = [C.c_void_p]
    L.asam_backsolve_full.argtypes = [C.c_void_p]
    L.asam_sync.argtypes = [C.c_void_p]
    L.asam_counters.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
    L.asam_set_timing.argtypes = [C.c_void_p, C.c_int]
    L.asam_last_kernel_ms.argtypes = [C.c_void_p, _fp, _fp, _fp]
    L.asam_timer_start.argtypes = [C.c_void_p]
    L.asam_timer_stop.argtypes = [C.c_void_p, _fp]
    L.asam_l2_flush.argtypes = [C.c_void_p]
    L.asam_device_info.argtypes = [C.c_void_p, _ip, _ip, _ip, _ip]
    L.asam_factor_status.argtypes = [C.c_void_p, _ip]
    L.asam_download_x.argtypes = [C.c_void_p, C.c_int, C.c_int, _dp]
    L.asam_download_y.argtypes = [C.c_void_p, C.c_int, C.c_int, _dp]
    L.asam_debug_read_hessian.argtypes = [C.c_void_p, C.c_int, C.c_int, _dp, _dp, _dp]
    L.asam_debug_read_front.argtypes = [C.c_void_p, C.c_int64, C.c_int64, _dp]
    L.asam_comm_unique_id.argtypes = [C.c_void_p]
    L.asam_comm_init.argtypes = [C.c_int, C.c_int, C.c_void_p]
    L.asam_comm_destroy.restype = None
    L.asam_comm_info.argtypes = [_ip, _ip, _ip]
    L.asam_comm_set_sharding.argtypes = [C.c_int]
    L.asam_measure_fp64_peak.argtypes = [C.c_void_p, _dp]
    L.asam_small_steps.argtypes = [C.c_void_p]
    L.asam_small_steps.restype = C.c_int64
    L.asam_small_step_profile.argtypes = [C.c_void_p, _dp, C.c_int]
    L.asam_small_step_profile.restype = None
    L.asam_dbg_profile.argtypes = [_dp, C.c_int]
    L.asam_dbg_profile.restype = None
    L.asam_upload_loss.argtypes = [C.c_void_p, C.c_int, C.c_int, _ip, _dp]
    L.asam_debug_read_buffer.argtypes = [C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_void_p]
    L.asam_marginal_cov.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_int, _dp]
    L.asam_dbg_plan_marginal_paths.argtypes = [C.c_void_p, C.c_int, _ip, C.c_void_p, C.POINTER(C.c_int64)]
    L.aprilsam_b200_marginal_covariance.argtypes = [C.c_void_p, C.c_void_p, C.c_int, _ip, _dp]
    L.aprilsam_b200_relative_covariance.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, _dp]
    L.aprilsam_b200_candidate_mahalanobis.argtypes = [C.c_void_p, C.c_void_p, C.c_int, _ip, _ip, _dp, _dp, _dp, _dp]
    L.asam_marginal_pairs.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int,
                                      C.c_void_p, _dp]
    L.asam_dbg_plan_candidate_batches.argtypes = [C.c_void_p, C.c_int, _ip, _ip, C.c_int64, _ip, _ip, _ip, _ip, _ip]
    L.asam_dbg_set_candidate_budget.argtypes = [C.c_int64]
    L.asam_dbg_set_candidate_budget.restype = None
    L.asam_debug_marginal_pairs_layout.argtypes = [C.c_int, C.c_int64, C.c_int, C.c_int, C.POINTER(C.c_int64)]
    L.asam_debug_marginal_pairs_layout.restype = None
    L.asam_dbg_factor_loss.argtypes = [C.c_void_p, C.c_int, _ip, _dp]
    L.asam_chi2.argtypes = [C.c_void_p, C.c_int, _dp]
    L.aprilsam_b200_factor_residuals.argtypes = [C.c_void_p, C.c_int, C.c_int, _dp]
    L.aprilsam_b200_factor_outlier_scores.argtypes = [C.c_void_p, C.c_void_p, C.c_int, _ip, _dp, _dp, _dp]
    L.asam_factor_residuals.argtypes = [C.c_void_p, C.c_int, C.c_int, _dp]
    L.asam_marginal_audit.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int,
                                      C.c_void_p, _dp]
    L.asam_debug_marginal_audit_layout.argtypes = [C.c_int, C.c_int64, C.c_int, C.c_int, C.POINTER(C.c_int64)]
    L.asam_debug_marginal_audit_layout.restype = None
    L.aprilsam_b200_candidate_compatibility.argtypes = [C.c_void_p, C.c_void_p, C.c_int, _ip, _ip, _dp, _dp, _dp,
                                                        _dp]
    L.asam_marginal_compat.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int,
                                       C.c_int, C.c_void_p, _ip, _dp, _dp]
    L.asam_debug_marginal_compat_layout.argtypes = [C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int64,
                                                    C.POINTER(C.c_int64)]
    L.asam_debug_marginal_compat_layout.restype = None
    L.asam_dbg_plan_compat_tiles.argtypes = [C.c_void_p, C.c_int, _ip, _ip, C.c_int64, _ip, C.c_int]
    L.aprilsam_b200_remove_factors.argtypes = [C.c_void_p, C.c_void_p, C.c_int, _ip, C.c_void_p]
    L.aprilsam_b200_relinearize_poses.argtypes = [C.c_void_p, C.c_void_p, C.c_int, _ip]
    L.asam_hessian_rebuild.argtypes = [C.c_void_p, C.c_int, _ip, _ip, C.c_int, _ip, _ip, C.c_int, _ip, _dp, _dp]
    L.asam_dbg_plan_refactor.argtypes = [C.c_void_p, _ip, C.c_int, _ip, _ip, _ip, C.c_int]
    L.asam_dbg_plan_remove_factors.argtypes = [C.c_void_p, C.c_int, _ip]
    _lib = L
    return L


def comm_init_torch(dist, local_rank: int) -> None:
    """Create the library's NCCL communicator inside a torch.distributed job: rank 0 makes the
    128-byte id, torch broadcasts it, every rank joins (one process per GPU)."""
    import torch
    L = lib()
    world, rank = dist.get_world_size(), dist.get_rank()
    buf = (C.c_ubyte * 128)()
    if rank == 0:
        check(L.asam_comm_unique_id(buf), "asam_comm_unique_id")
    cuda = dist.get_backend() == "nccl"
    t = torch.tensor(list(buf), dtype=torch.uint8, device=torch.device("cuda", local_rank) if cuda else "cpu")
    dist.broadcast(t, src=0)
    raw = bytes(t.cpu().tolist())
    ident = (C.c_ubyte * 128).from_buffer_copy(raw)
    check(L.asam_comm_init(world, rank, ident), "asam_comm_init")


def check(rc: int, what: str = "asam call"):
    if rc != 0:
        raise RuntimeError(f"{what} failed: {lib().asam_last_error().decode()}")


def plan_info(plan_ptr) -> dict:
    a = (C.c_int64 * 16)()
    fl = C.c_double()
    lib().asam_dbg_plan_info(plan_ptr, a, C.byref(fl))
    keys = ["N", "nsn", "n_slots", "ipool_n", "arena_n", "max_m", "nnz_l_blocks", "n_levels", "n_factors"]
    d = {k: int(a[i]) for i, k in enumerate(keys)}
    d["flops"] = fl.value
    return d


def counters(dev) -> tuple[int, int, int]:
    a = (C.c_int64 * 3)()
    lib().asam_counters(dev, a)
    return int(a[0]), int(a[1]), int(a[2])


def kernel_ms(dev) -> tuple[float, float, float]:
    a, b, c = C.c_float(), C.c_float(), C.c_float()
    check(lib().asam_last_kernel_ms(dev, C.byref(a), C.byref(b), C.byref(c)), "asam_last_kernel_ms")
    return a.value, b.value, c.value
