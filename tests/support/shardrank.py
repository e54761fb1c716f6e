"""One rank of a sharded batch solve on one GPU, for tests/test_gpu_sharded.py.

TEST INFRASTRUCTURE.  The parent test starts one process per rank:

    python tests/support/shardrank.py SPEC.json RANK

with ASAM_DEVICE=0.  The process loads the loopback stand-in for NCCL (tests/support/loopnccl.c, SONAME
libnccl.so.2) with RTLD_GLOBAL BEFORE the solver's library, so the solver's dlopen("libnccl.so.2") resolves to it;
it must never import torch, which would load the real libnccl.so.2 first.  It joins the communicator
(asam_comm_init with the id the parent wrote: the path of a rendezvous file), runs the jobs of the spec and writes
what it read back and checked to <out>/<job>_r<rank>.npz.  The parent compares the ranks' files with each other and
with the single-GPU solve that rank 0 runs in its own process (asam_comm_set_sharding(0)).

Jobs:
  * "solve": a batch solve of a graph for every entry of `sharding` (1 = sharded, 0 = one GPU) in ONE harness (the
    plan is rebuilt at every switch).  After each sharded solve: ShardSnapshot checks of every front this rank
    factored (its shards and the top), y, the per-supernode back-substitution, the residual and the forward error
    of the whole x after the exchange; SHA-1 digests of the Hessian, of every front it factored, of the exchanged
    arena ranges; x, the states, the status word and the stand-in's counters of the solve;
  * "pivots": failed pivots placed in shard supernodes of chosen ranks and in a top supernode (extra SPD priors that
    leave the plan unchanged, W made negative at the C-ABI as in pivotcheck); the status word every rank reads, the
    float64 prediction of the owner, then the restored system against the clean run bit for bit.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SYNC_TIMEOUT = 1800.0  # the ranks meet between solves; one of them may still be checking the last one


# ---------------------------------------------------------------------------------------------
# parent side: build the stand-in, write the id, run the ranks
# ---------------------------------------------------------------------------------------------
def build_standin(outdir):
    """gcc the stand-in into outdir/libnccl.so.2 (SONAME libnccl.so.2); returns its path."""
    out = os.path.join(outdir, "libnccl.so.2")
    subprocess.run(["gcc", "-shared", "-fPIC", "-O2", "-Wall", "-Wl,-soname,libnccl.so.2", "-o", out,
                    os.path.join(HERE, "loopnccl.c"), "-ldl"], check=True, capture_output=True)
    return out


def unique_id(path):
    """The 128-byte id of the stand-in: the rendezvous file's path, NUL-padded."""
    raw = os.fsencode(path)
    assert len(raw) < 128, path
    return raw + b"\0" * (128 - len(raw))


def run_ranks(argv_of, world, env, timeout):
    """Start `world` processes (argv_of(rank)), wait for all of them, kill and reap whatever is left.  Returns
    [(returncode, output)] per rank; returncode None = killed at the timeout."""
    procs = []
    outs = [None] * world
    try:
        for r in range(world):
            procs.append(subprocess.Popen(argv_of(r), env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                                          text=True))
        end = time.monotonic() + timeout
        for r, p in enumerate(procs):
            try:
                outs[r] = p.communicate(timeout=max(1.0, end - time.monotonic()))[0]
            except subprocess.TimeoutExpired:
                p.kill()
                outs[r] = p.communicate()[0] + "\n[killed at the timeout]"
        return [(None if "[killed at the timeout]" in (o or "") else p.returncode, o) for p, o in zip(procs, outs)]
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
            p.wait()


# ---------------------------------------------------------------------------------------------
# child side
# ---------------------------------------------------------------------------------------------
def sha(*arrays):
    h = hashlib.sha1()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


class Rank:
    def __init__(self, spec, rank):
        self.spec, self.rank, self.world = spec, rank, spec["world"]
        self.standin = C.CDLL(spec["standin"], mode=os.RTLD_GLOBAL | os.RTLD_NOW)  # before the solver's library
        self.standin.loopnccl_stats.argtypes = [C.POINTER(C.c_longlong)]
        self.standin.loopnccl_sync.argtypes = [C.c_double]
        sys.path.insert(0, ROOT)
        sys.path.insert(0, os.path.dirname(HERE))
        from aprilsam_b200 import capi
        self.capi = capi
        self.L = capi.lib()
        ident = (C.c_ubyte * 128).from_buffer_copy(unique_id(spec["id_path"]))
        capi.check(self.L.asam_comm_init(self.world, rank, ident), "asam_comm_init")
        assert "torch" not in sys.modules
        from support import frontcheck as fc
        self.D = fc.dev_api()  # the same library, with the debug accessors' signatures (HostPlan, read-back)

    def stats(self):
        a = (C.c_longlong * 4)()
        self.standin.loopnccl_stats(a)
        return np.array(a[:], dtype=np.int64)

    def sync(self):
        rc = self.standin.loopnccl_sync(SYNC_TIMEOUT)
        if rc:
            raise RuntimeError(f"rank {self.rank}: the other ranks did not arrive (stand-in error {rc})")

    def set_sharding(self, on):
        self.capi.check(self.L.asam_comm_set_sharding(1 if on else 0), "asam_comm_set_sharding")


class ShardSnapshot:
    """frontcheck.Snapshot of ONE rank of a sharded solve.  `computed` = the supernodes this rank factored (its own
    shards' leaf and k_factor tasks, and the top); fronts holds them and the shard roots of every rank (their
    trailing columns are what the exchange brought); paths are named as frontcheck names them, with the top's
    prefixed "top:"."""

    def __init__(self, L, dev, plan, fc):
        info = plan.info()
        N, S = info["N"], info["n_slots"]
        self.plan = plan
        self.desc = plan.descs()
        self.nsn = len(self.desc["mb"])
        for k in ("ipool", "q2node", "node2q", "tasks", "nwait", "leaf_tasks", "top_tasks", "top_nwait",
                  "shard_owner", "shard_q0", "shard_qn", "fslot"):
            setattr(self, k, plan.array(k))
        self.shard_off, self.shard_cnt = plan.array64("shard_off"), plan.array64("shard_cnt")
        Ad = np.zeros((N, 3, 3)); Ao = np.zeros((max(S, 1), 3, 3)); B = np.zeros((N, 3))
        fc._ok(L, L.asam_debug_read_hessian(dev, N, S, Ad.ctypes.data_as(fc._dp), Ao.ctypes.data_as(fc._dp),
                                            B.ctypes.data_as(fc._dp)), "read_hessian")
        self.Adiag, self.Aoff, self.B = Ad, Ao[:S], B
        self.y = np.zeros(3 * N); self.x = np.zeros(3 * N)
        fc._ok(L, L.asam_download_y(dev, 0, N, self.y.ctypes.data_as(fc._dp)), "download_y")
        fc._ok(L, L.asam_download_x(dev, 0, N, self.x.ctypes.data_as(fc._dp)), "download_x")
        self.top = set(int(s) for s in self.top_tasks)
        self.own = set(int(s) for s in self.tasks) | set(int(s) for s in self.leaf_tasks)
        self.computed = sorted(self.top | self.own)
        self.roots = [self.root_of(i) for i in range(len(self.shard_owner))]
        self.fronts = fc.read_fronts(L, dev, self.desc, sorted(set(self.computed) | set(self.roots)))
        self.team = {}
        for s, w in list(zip(self.tasks, self.nwait)) + list(zip(self.top_tasks, self.top_nwait)):
            self.team.setdefault(int(s), (int(w) >> 24) & 0x7f)
        self.leafset = set(int(s) for s in self.leaf_tasks)
        self.fits_smem = fc.fits_smem
        self.xch = []
        for i in range(len(self.shard_owner)):
            buf = np.zeros(int(self.shard_cnt[i]))
            fc._ok(L, L.asam_debug_read_front(dev, int(self.shard_off[i]), len(buf), buf.ctypes.data_as(fc._dp)),
                   "read_front")
            self.xch.append(sha(buf))

    def root_of(self, i):
        """The supernode whose trailing columns are shard i's exchanged range."""
        d = self.desc
        ld = lambda m: (m + 2) & ~1  # noqa: E731
        c = 3 * d["cb"].astype(np.int64)
        m = 3 * d["mb"].astype(np.int64)
        hit = np.nonzero((d["f_off"] + c * ld(m) == self.shard_off[i]) & ((m - c) * ld(m) == self.shard_cnt[i]))[0]
        assert len(hit) == 1, (i, hit)
        return int(hit[0])

    def path(self, s):
        if s in self.leafset:
            p = "leaf"
        else:
            G = self.team.get(s, 0)
            p = f"team{G}" if G else ("cta_smem" if self.fits_smem(int(self.desc["mb"][s])) else "cta_hbm")
        return ("top:" if s in self.top else "") + p


def path_table(plan, fc):
    """{supernode: path} of every supernode of a single-GPU plan (frontcheck.Snapshot.path)."""
    snap = fc.Snapshot.__new__(fc.Snapshot)
    snap.desc, snap.tasks, snap.nwait, snap.leaf_tasks = plan.descs(), plan.array("tasks"), plan.array("nwait"), \
        plan.array("leaf_tasks")
    return {s: snap.path(s) for s in range(len(snap.desc["mb"]))}


def check_rank(snap, h, fc, forward):
    """frontcheck's checks restricted to what this rank computed; per path: worst factor, rhs and back-solve."""
    per = {}
    for s in snap.computed:
        ef, er = fc.front_errors(snap, s)
        eb = fc.check_backsolve_local(snap, [s])
        rec = per.setdefault(snap.path(s), {"n": 0, "factor": 0.0, "rhs": 0.0, "backsolve": 0.0})
        rec["n"] += 1
        rec["factor"], rec["rhs"], rec["backsolve"] = max(rec["factor"], ef), max(rec["rhs"], er), \
            max(rec["backsolve"], eb)
    y_bad = 0
    for s in snap.computed:
        first, c = int(snap.desc["first"][s]), 3 * int(snap.desc["cb"][s])
        y_bad += int(np.count_nonzero(snap.y[3 * first:3 * first + c].view(np.int64)
                                      != snap.fronts[s][1][:c].view(np.int64)))
    ftype, fa, fb, _, _ = fc.factors_of(h)
    A, b = fc.system(snap, ftype, fa, fb, snap.fslot)
    res = {"per_path": per, "y_bad": y_bad, "residual": fc.check_residual(A, b, snap.x),
           "factor": max([v["factor"] for v in per.values()], default=0.0),
           "rhs": max([v["rhs"] for v in per.values()], default=0.0),
           "backsolve": max([v["backsolve"] for v in per.values()], default=0.0)}
    if forward:
        xr, kappa = fc.reference_solution(A, b)
        res["forward_over_kappa_u"] = fc.forward_error(snap.x, xr) / (kappa * fc.U)
    return res


def front_digests(snap, which):
    return {int(s): [sha(snap.fronts[s][0], snap.fronts[s][1]), snap.path(s)] for s in which}


def load_graph(path):
    from aprilsam_b200.harness import PoseGraphData
    return PoseGraphData.load(path)


def new_harness(job, d):
    from aprilsam_b200 import harness as H
    h = H.Harness("b200")
    if job.get("robust"):
        h.set_scan_loss(*job["robust"])
    if job.get("tikhonov") is not None:
        h.set_tikhanov(job["tikhonov"])
    h.load_full(d)
    return h


def sharded_solve(R, h, d, fc, forward, out, tag):
    """One sharded batch solve from the graph's initial states; everything the parent compares goes into `out`."""
    L = R.D
    R.sync()
    h.set_states(d.init)
    s0 = R.stats()
    h.batch()
    s1 = R.stats()
    dev = C.c_void_p(L.asam_dbg_dev_of_graph(h.graph_ptr()))
    plan = fc.borrowed_plan(L, h.param_ptr())
    snap = ShardSnapshot(L, dev, plan, fc)
    st = C.c_int()
    fc._ok(L, L.asam_factor_status(dev, C.byref(st)), "factor_status")
    rep = {"sharded": True, "computed": len(snap.computed), "top": len(snap.top), "own": len(snap.own), "status": st.value,
           "n_shards": len(snap.shard_owner), "digests": front_digests(snap, snap.computed),
           "xch": snap.xch, "roots": snap.roots, "hessian": sha(snap.Adiag, snap.Aoff, snap.B), "desc": sha(plan.array("desc")),
           "n_bt": len(plan.array("btasks")), "bt_split": int(np.any(plan.array("btasks") >> 24)),
           "n_bs_leaf": plan.info()["n_bs_leaf"]}
    t0 = time.monotonic()
    rep["checks"] = check_rank(snap, h, fc, forward)
    rep["check_s"] = time.monotonic() - t0
    out[f"{tag}_x"] = snap.x
    out[f"{tag}_states"] = h.states()
    out[f"{tag}_stats"] = s1 - s0
    for k in ("shard_owner", "shard_q0", "shard_qn", "shard_off", "shard_cnt"):
        out[f"{tag}_{k}"] = getattr(snap, k)
    return rep, snap


def single_solve(R, h, d, fc, out, tag):
    """The single-GPU solve (sharding off) of the same harness."""
    L = R.D
    h.set_states(d.init)
    s0 = R.stats()
    h.batch()
    dev = C.c_void_p(L.asam_dbg_dev_of_graph(h.graph_ptr()))
    plan = fc.borrowed_plan(L, h.param_ptr())
    snap = fc.snapshot(h, L)
    paths = path_table(plan, fc)
    st = C.c_int()
    fc._ok(L, L.asam_factor_status(dev, C.byref(st)), "factor_status")
    out[f"{tag}_states"] = h.states()
    return {"sharded": False, "status": st.value, "hessian": sha(snap.Adiag, snap.Aoff, snap.B), "desc": sha(plan.array("desc")),
            "parent": [int(p) for p in snap.desc["parent"]], "n_top": len(plan.array("top_tasks")),
            "stats": (R.stats() - s0).tolist(),
            "digests": {s: [sha(snap.fronts[s][0], snap.fronts[s][1]), paths[s]] for s in range(snap.nsn)}}


def marginal_report(R, h, d, fc, sharded):
    """After a sharded solve: the errors of marginal_covariance and relative_covariance (a rank holds only its own
    shards' fronts).  After a single-GPU solve on the same context: the hop-by-hop checks of margcheck."""
    if sharded:
        errs = []
        for call in (lambda: h.marginal_covariance([0, d.n_nodes - 1]), lambda: h.relative_covariance(0, 1)):
            try:
                call()
                errs.append(None)
            except RuntimeError as e:
                errs.append(str(e))
        return {"errors": errs}
    from support import margcheck as mc
    nodes = [0, d.n_nodes - 1, d.n_nodes // 2, 17]
    _, res = mc.query_report(h, R.D, fc.snapshot(h, R.D), nodes)
    return res


def job_solve(R, job, fc):
    d = load_graph(job["graph"])
    out, rep = {}, {"runs": []}
    env = job.get("env") or {}
    os.environ.update(env)
    with new_harness(job, d) as h:
        for k, on in enumerate(job["sharding"]):
            R.set_sharding(on)
            if on:
                r, _ = sharded_solve(R, h, d, fc, job.get("forward", True), out, f"run{k}")
            else:
                R.sync()
                r = single_solve(R, h, d, fc, out, f"run{k}")
            if job.get("marginals"):
                r["marginals"] = marginal_report(R, h, d, fc, on)
            rep["runs"].append(r)
    if job.get("single") and R.rank == 0:  # in a harness of its own (a fresh plan)
        R.set_sharding(0)
        with new_harness(job, d) as h:
            rep["single"] = single_solve(R, h, d, fc, out, "single")
    for k in env:
        os.environ.pop(k, None)
    R.sync()
    return out, rep


# ---------------------------------------------------------------------------------------------
# failed pivots
# ---------------------------------------------------------------------------------------------
def choose_targets(tables, world):
    """Deterministic targets from every rank's path table ({supernode: path} of what it factored): a leaf-kernel
    supernode of rank 0 (else its deepest own one), a team / HBM / widest front of rank 1, a top supernode on a team
    path (else the widest top one)."""
    own = [{int(s): p for s, p in t.items() if not p.startswith("top:")} for t in tables]
    top = {int(s): p for s, p in tables[0].items() if p.startswith("top:")}
    out = []
    r0 = sorted(s for s, p in own[0].items() if p == "leaf") or sorted(own[0])
    if r0:
        out.append(("rank0", r0[0]))
    if world > 1:
        big = sorted(s for s, p in own[1].items() if p.startswith("team") or p == "cta_hbm")
        r1 = big or sorted(own[1])
        if r1:
            out.append(("rank1", r1[-1]))
    tops = sorted(s for s, p in top.items() if "team" in p) or sorted(top)
    if tops:
        out.append(("top", tops[0]))
    return out


def predict(snap, s, pc, fc):
    """First failing supernode in float64, eliminating s and its ancestors (ids ascending: children first) on top of
    this rank's clean fronts.  Only the owner of s (or any rank, for a top s) holds every child needed."""
    from types import SimpleNamespace
    Ad, Ao, B = snap["H"]
    ns = SimpleNamespace(desc=snap["base"].desc, ipool=snap["base"].ipool, q2node=snap["base"].q2node, Adiag=Ad,
                         Aoff=Ao, B=B, fronts=dict(snap["base"].fronts))
    for t in [s] + pc.ancestors(ns.desc, s):
        F, b = fc.assemble(ns, t)
        k = pc._factor_front(F, b, 3 * int(ns.desc["cb"][t]))
        if k is not None:
            return t, k
        ns.fronts[t] = (F, b)
    return None


def job_pivots(R, job, fc):
    from support import pivotcheck as pc
    d = load_graph(job["graph"])
    out, rep = {}, {"runs": [], "targets": []}
    R.set_sharding(1)
    tables_dir = os.path.join(R.spec["out"], job["name"] + "_tables")
    os.makedirs(tables_dir, exist_ok=True)
    with new_harness(job, d) as h:
        r0, snap0 = sharded_solve(R, h, d, fc, False, out, "plan")
        with open(os.path.join(tables_dir, f"r{R.rank}.json"), "w") as f:
            json.dump({int(s): snap0.path(s) for s in snap0.computed}, f)
        R.sync()
        tables = []
        for r in range(R.world):
            with open(os.path.join(tables_dir, f"r{r}.json")) as f:
                tables.append(json.load(f))
        targets = choose_targets(tables, R.world)
        q2node = snap0.q2node
        W = np.array([4.0, 1, 0, 1, 4, 0, 0, 0, 2])  # integer, SPD
        F0 = h.n_factors
        for j, (_, s) in enumerate(targets):
            node = int(q2node[int(snap0.desc["first"][s])])
            h.add_xytpos(node, d.init[node], W.reshape(3, 3))
        # the priors leave the plan unchanged; this clean run is the base of the restored system
        r1, snap1 = sharded_solve(R, h, d, fc, job.get("forward", True), out, "clean")
        rep["runs"] = [r0, r1]
        rep["plan_unchanged"] = r0["desc"] == r1["desc"] and r0["digests"].keys() == r1["digests"].keys()
        ctx = pc.Context(h, job.get("tikhonov") or 0.0)
        base_x = snap1.x.copy()
        for j, (who, s) in enumerate(targets):
            f = F0 + j
            node = int(q2node[int(snap1.desc["first"][s])])
            Ad, Ao, Bq = ctx.hessian()
            R.sync()
            ctx.set_W(f, pc.negative_W(W, float(Ad[node][0, 0]), 0))
            ctx.relinearize()
            s0 = R.stats()
            ctx.factor()
            st_fail = ctx.status()
            stats_fail = (R.stats() - s0).tolist()
            mine = s in snap1.top or s in snap1.own
            pred = None
            if mine:
                H_fail = ctx.hessian()
                p = predict({"H": H_fail, "base": snap1}, s, pc, fc)
                pred = None if p is None else [int(p[0]), int(p[1])]
            R.sync()
            ctx.set_W(f, W)
            ctx.relinearize()
            ctx.factor()
            st_ok = ctx.status()
            again = ShardSnapshot(R.D, ctx.dev, snap1.plan, fc)
            same = (front_digests(again, again.computed) == front_digests(snap1, snap1.computed)
                    and np.array_equal(again.x.view(np.int64), base_x.view(np.int64)) and again.xch == snap1.xch)
            rep["targets"].append({"who": who, "sn": int(s), "node": node, "path": snap1.path(s) if mine else None,
                                   "status": st_fail, "predicted": pred, "status_restored": st_ok,
                                   "restored_same_bits": bool(same), "stats": stats_fail})
    R.sync()
    return out, rep


# ---------------------------------------------------------------------------------------------
# the stand-in alone, in host mode (LOOPNCCL_HOST=1): tests/test_gpu_sharded.py::test_standin_*
# ---------------------------------------------------------------------------------------------
SELFTEST_SIZES = [0, 5, 3584]  # doubles; 3584 x 8 bytes = 7 windows of 4096 bytes


def selftest_data(rank, n):
    return np.random.default_rng(1000 * rank + n).standard_normal(n) * 1000.0


class _Uid(C.Structure):
    _fields_ = [("internal", C.c_char * 128)]


def selftest(spec, rank_arg):
    """Exit 0 after every operation, 3 if joining failed, 4 if a broadcast failed; "R:leave" joins and exits."""
    rank, leave = int(rank_arg.split(":")[0]), rank_arg.endswith(":leave")
    world = spec["world"]
    S = C.CDLL(spec["standin"])
    S.ncclCommInitRank.argtypes = [C.POINTER(C.c_void_p), C.c_int, _Uid, C.c_int]
    S.ncclBroadcast.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    S.ncclAllReduce.argtypes = S.ncclBroadcast.argtypes
    S.loopnccl_stats.argtypes = [C.POINTER(C.c_longlong)]
    comm = C.c_void_p()
    uid = _Uid()
    uid.internal = unique_id(spec["id_path"])
    if S.ncclCommInitRank(C.byref(comm), world, uid, rank):
        return 3
    if leave:
        return 0
    out = {}
    for root in range(world):
        for n in SELFTEST_SIZES:
            buf = selftest_data(root, n) if rank == root else np.full(n, -1.0)
            if S.ncclBroadcast(buf.ctypes.data, buf.ctypes.data, n, 8, root, comm, None):
                return 4
            out[f"b{root}_{n}"] = buf
    v = selftest_data(rank, 1000)
    for name, op in (("max", 2), ("min", 3)):
        a = v.astype(np.int32)
        if S.ncclAllReduce(a.ctypes.data, a.ctypes.data, len(a), 2, op, comm, None):
            return 5
        out[name] = a
    if S.ncclAllReduce(v.ctypes.data, v.ctypes.data, len(v), 8, 0, comm, None):
        return 5
    out["sum"] = v
    st = (C.c_longlong * 4)()
    S.loopnccl_stats(st)
    out["stats"] = np.array(st[:])
    np.savez(os.path.join(spec["out"], f"selftest_r{rank}.npz"), **out)
    S.ncclCommDestroy(comm)
    return 0


def main(argv):
    if argv[1] == "selftest":
        with open(argv[2]) as f:
            return selftest(json.load(f), argv[3])
    with open(argv[1]) as f:
        spec = json.load(f)
    rank = int(argv[2])
    R = Rank(spec, rank)
    from support import frontcheck as fc
    for job in spec["jobs"]:
        t0 = time.monotonic()
        out, rep = (job_pivots if job["kind"] == "pivots" else job_solve)(R, job, fc)
        rep["seconds"] = time.monotonic() - t0
        rep["total_stats"] = R.stats().tolist()
        out["report"] = np.array(json.dumps(rep))
        np.savez(os.path.join(spec["out"], f"{job['name']}_r{rank}.npz"), **out)
        print(f"rank {rank}: {job['name']} done in {rep['seconds']:.1f} s", flush=True)
    R.L.asam_comm_destroy()
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
