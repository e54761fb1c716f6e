// asam_cuda.cu -- C-ABI (include/asam_cuda.h) of the sm_90a CUDA implementation of the AprilSAM
// Gauss-Newton path: device context, HBM buffers, uploads/downloads, kernel launches.
// The kernels themselves are in asam_kernels.cuh.
//
// There is no CPU implementation of any of this in the product: if the CUDA runtime or a
// device is missing, asam_dev_create() fails and the host API aborts.

#include <cuda_runtime.h>

#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <mutex>
#include <vector>

#include "asam_cuda.h"

#define ASAM_EXPORT extern "C" __attribute__((visibility("default")))

// ------------------------------------------------------------------------------------------
// error plumbing
// ------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";

static int set_err(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return 1;
}

#define CK(call)                                                                              \
    do {                                                                                      \
        cudaError_t e_ = (call);                                                              \
        if (e_ != cudaSuccess)                                                                \
            return set_err("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
    } while (0)

ASAM_EXPORT const char *asam_last_error(void) { return g_err; }

// ------------------------------------------------------------------------------------------
// device context
// ------------------------------------------------------------------------------------------
struct Buf {
    void *p = nullptr;
    size_t cap = 0; // bytes
};

struct BatchItem {
    unsigned long long dst;
    unsigned int off;   // payload offset (copy items)
    unsigned int bytes; // multiple of 4
    unsigned int fill;  // 1 = fill with `val`
    unsigned int val;
};
#define ASAM_MAX_ITEMS 1024
#define ASAM_TABLE_BYTES (ASAM_MAX_ITEMS * sizeof(BatchItem))
#define ASAM_ITEM_CHUNK (8u << 10) // one k_scatter block per item: small chunks keep that kernel at a few microseconds

struct asam_dev {
    int device = 0;
    int n_sm = 0;
    cudaStream_t stream = nullptr;

    // graph mirror
    Buf f_type, f_a, f_b, f_z, f_W, f_slot;
    Buf f_loss; // double2 {loss, k} per factor: meaningful for robust factors only; allocated at the first
                // asam_upload_loss, so that graphs without robust factors allocate, move and read nothing more
    Buf lp, st, node2q, q2node;
    // hessian
    Buf Adiag, Aoff, Bq, y, x, dinv;
    // plan
    Buf sn, ipool, arena;
    Buf arrive, xdone, tbar, xblk;
    // task lists
    Buf tasks_full, nwait_full, btasks_full;
    int ntasks_full = 0;
    Buf leaf_tasks; // supernodes handled by k_factor_leaf before k_factor (batch solves of large graphs)
    int n_leaf = 0;
    int leaf_grid = 0, leaf_smem = 0;
    int bt_nleaf = 0; // the last bt_nleaf entries of btasks_full are back-solved by k_backsolve_leaf
    // multi-GPU shard schedule (asam_set_shard_schedule)
    int sharded = 0;
    Buf top_tasks, top_nwait;
    int n_top = 0;
    int n_shards = 0;
    int *sh_owner = nullptr, *sh_q0 = nullptr, *sh_qn = nullptr;
    long long *sh_off = nullptr, *sh_cnt = nullptr;
    int bsl_grid = 0, bsl_smem = 0;
    int bt_start = 0, bt_count = 0, bt_cap = 0; // btasks_full holds [bt_start, bt_start+bt_count)
    Buf tasks_tmp, nwait_tmp, btasks_tmp, keep_tmp;
    int keep_off = 0; // ASAM_KEEP=0: always re-factor whole fronts (A/B measurements)
    // misc
    Buf ctrl;     // int[8]: [0] ticket, [1] err, [2] ticket backsolve
    Buf partial;  // chi2 partial sums
    Buf patch_ids, patch_desc;
    Buf pts;
    Buf rb_int, rb_dbl; // tables of asam_hessian_rebuild
    int epoch = 0;

    // host->device traffic is BATCHED: small uploads and fills are queued in one pinned staging
    // buffer and reach HBM with a single cudaMemcpyAsync + one scatter kernel (k_scatter) right
    // before the next kernel launch / download -- an incremental step costs two API calls for all
    // of its ~15 small transfers.
    char *pin = nullptr;      // [item table | payload]
    size_t pin_cap = 0, pin_off = 0; // pin_off = payload bytes used
    char *dstage = nullptr;   // device mirror of the staging buffer
    struct BatchItem *items = nullptr;
    int n_items = 0;
    cudaEvent_t up_ev = nullptr;
    int up_busy = 0;
    char *pin_down = nullptr; // separate pinned buffer for downloads
    size_t pin_down_cap = 0;
    // deferred launches (asam_step_begin .. asam_step_run): kernels recorded, launched after ONE flush
    int defer = 0;
    struct Pending *pend = nullptr;
    int npend = 0;
    int step_seq = 0;  // sequence number of the last k_step launch (completion flag in pin_down)
    int pb_smem = 12;  // ASAM_PB_SMEM: panel width of shared-memory fronts
    int smem_mma = 1;  // ASAM_SMEM_MMA: 0 DFMA only, 1 tensor pipe for the kept-columns update, 2 for every panel update
    int solo_pb = 48;  // ASAM_SOLO_PB: staged panel width of single-CTA fronts that live in HBM
    int small_ok = 1;  // ASAM_SMALL_STEP=0 disables the fused small-step kernel (A/B measurements)
    int64_t n_small = 0;
    double small_us[8] = {0, 0, 0, 0, 0, 0, 0, 0}; // accumulated phases of k_step (device stamps) + host launch / wait

    // launch config
    int fac_threads = 256, fac_grid = 0, fac_smem = 0;
    int bs_threads = 256, bs_grid = 0, bs_smem = 0; // 8 warps: faster than 4 on M3500 and the 100 k world in A/B runs; ASAM_BS_THREADS=128 for comparison

    int64_t n_launch = 0, n_h2d = 0, n_d2h = 0;

    int timing = 0;
    cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    int ev_set[3] = {0, 0, 0};
    cudaEvent_t tev[2] = {nullptr, nullptr};
    Buf flush;
    int flush_val = 0;
    int trace_on = 0;
    Buf trace_fac, trace_bs;
    int trace_nfac = 0, trace_nbs = 0;
    Buf ptrace; // panel-step stamps of one team front (asam_set_panel_trace)
    int ptrace_sn = -1, ptrace_panels = 0;
    Buf marg;          // scratch of asam_marginal_cov, allocated at the first query
};

static int flush_uploads(asam_dev *d);
static int clear_status(asam_dev *d);

static int buf_reserve(asam_dev *d, Buf &b, size_t bytes, bool keep, bool zero_new)
{
    if (bytes <= b.cap)
        return 0;
    if (flush_uploads(d)) // queued items may point into the buffer that is about to move
        return 1;
    // growth in powers of two from 1 MiB: a replay grows ~25 buffers pose by pose, and every move costs a cudaMalloc, a stream
    // synchronisation and a cudaFree (with 4 KiB x 1.5 the M3500 replay moved a buffer ~350 times on its way to 3500 poses)
    size_t want = b.cap ? b.cap : ((size_t) 1 << 20);
    while (want < bytes)
        want *= 2;
    void *np = nullptr;
    CK(cudaMalloc(&np, want));
    if (zero_new)
        CK(cudaMemsetAsync(np, 0, want, d->stream));
    if (keep && b.p && b.cap)
        CK(cudaMemcpyAsync(np, b.p, b.cap, cudaMemcpyDeviceToDevice, d->stream));
    if (b.p) {
        CK(cudaStreamSynchronize(d->stream));
        CK(cudaFree(b.p));
    }
    b.p = np;
    b.cap = want;
    return 0;
}

__global__ void k_scatter(const BatchItem *items, const char *payload)
{
    const BatchItem it = items[blockIdx.x];
    unsigned int *dst = (unsigned int *) it.dst;
    const unsigned int words = it.bytes >> 2;
    if (it.fill) {
        for (unsigned int i = threadIdx.x; i < words; i += blockDim.x)
            dst[i] = it.val;
    } else {
        const unsigned int *src = (const unsigned int *) (payload + it.off);
        for (unsigned int i = threadIdx.x; i < words; i += blockDim.x)
            dst[i] = src[i];
    }
}

// Push everything queued so far to the device (one H2D copy + one scatter launch).
static int flush_uploads(asam_dev *d)
{
    if (d->n_items == 0)
        return 0;
    memcpy(d->pin, d->items, (size_t) d->n_items * sizeof(BatchItem));
    const size_t total = ASAM_TABLE_BYTES + d->pin_off;
    CK(cudaMemcpyAsync(d->dstage, d->pin, total, cudaMemcpyHostToDevice, d->stream));
    CK(cudaEventRecord(d->up_ev, d->stream));
    k_scatter<<<d->n_items, 256, 0, d->stream>>>((const BatchItem *) d->dstage, d->dstage + ASAM_TABLE_BYTES);
    CK(cudaGetLastError());
    d->n_launch++;
    d->n_items = 0;
    d->pin_off = 0;
    d->up_busy = 1;
    return 0;
}

static int batch_room(asam_dev *d, size_t bytes, int items)
{
    if (d->up_busy) { // the staging buffer is still being copied by the previous flush
        CK(cudaEventSynchronize(d->up_ev));
        d->up_busy = 0;
    }
    if (d->n_items + items > ASAM_MAX_ITEMS || ASAM_TABLE_BYTES + d->pin_off + bytes > d->pin_cap) {
        if (flush_uploads(d))
            return 1;
        CK(cudaEventSynchronize(d->up_ev));
        d->up_busy = 0;
    }
    return 0;
}

static int upload(asam_dev *d, void *dst, const void *src, size_t bytes)
{
    if (bytes == 0)
        return 0;
    d->n_h2d += (int64_t) bytes;
    if ((bytes & 3) || bytes > (d->pin_cap - ASAM_TABLE_BYTES) / 2) { // odd size or large: direct copy
        if (flush_uploads(d))
            return 1;
        CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, d->stream));
        return 0;
    }
    const int nitems = (int) ((bytes + ASAM_ITEM_CHUNK - 1) / ASAM_ITEM_CHUNK);
    if (batch_room(d, bytes + 16, nitems))
        return 1;
    const size_t off = (d->pin_off + 15) & ~(size_t) 15;
    memcpy(d->pin + ASAM_TABLE_BYTES + off, src, bytes);
    for (size_t o = 0; o < bytes; o += ASAM_ITEM_CHUNK) {
        BatchItem &it = d->items[d->n_items++];
        it.dst = (unsigned long long) ((char *) dst + o);
        it.off = (unsigned int) (off + o);
        it.bytes = (unsigned int) (bytes - o < ASAM_ITEM_CHUNK ? bytes - o : ASAM_ITEM_CHUNK);
        it.fill = 0;
        it.val = 0;
    }
    d->pin_off = off + bytes;
    return 0;
}

// Queue a fill of `bytes` (multiple of 4) at dst with the 32-bit pattern `val`.
static int queue_fill(asam_dev *d, void *dst, unsigned int val, size_t bytes)
{
    if (bytes == 0)
        return 0;
    const size_t chunk = 4 * ASAM_ITEM_CHUNK;
    const int nitems = (int) ((bytes + chunk - 1) / chunk);
    if (nitems > ASAM_MAX_ITEMS / 2) { // huge: plain memset in stream order
        if (flush_uploads(d))
            return 1;
        CK(cudaMemsetAsync(dst, (int) (val & 0xff), bytes, d->stream));
        return 0;
    }
    if (batch_room(d, 0, nitems))
        return 1;
    for (size_t o = 0; o < bytes; o += chunk) {
        BatchItem &it = d->items[d->n_items++];
        it.dst = (unsigned long long) ((char *) dst + o);
        it.off = 0;
        it.bytes = (unsigned int) (bytes - o < chunk ? bytes - o : chunk);
        it.fill = 1;
        it.val = val;
    }
    return 0;
}

static int download(asam_dev *d, void *dst, const void *src, size_t bytes)
{
    if (bytes == 0)
        return 0;
    if (flush_uploads(d))
        return 1;
    d->n_d2h += (int64_t) bytes;
    if (bytes <= d->pin_down_cap) {
        CK(cudaMemcpyAsync(d->pin_down, src, bytes, cudaMemcpyDeviceToHost, d->stream));
        CK(cudaStreamSynchronize(d->stream));
        memcpy(dst, d->pin_down, bytes);
    } else {
        CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, d->stream));
        CK(cudaStreamSynchronize(d->stream));
    }
    return 0;
}

#include <dlfcn.h>

#include "asam_kernels.cuh"

// wall-clock bound of every inter-CTA wait (see SpinClock): 20 s -- far above any real solve, far below
// the limits of the job schedulers around us
#define ASAM_SPIN_LIMIT_NS 20000000000LL

struct Pending {
    int kind; // 0 linearize, 1 factor, 2 backsolve, 3 Hessian rebuild
    int grid;
    int nleaf;
    LinArgs lin;
    FacArgs fac;
    BsArgs bs;
    RebuildArgs rb;
};
#define ASAM_MAX_PENDING 8

static int run_linearize(asam_dev *d, const LinArgs &a)
{
    if (d->timing)
        CK(cudaEventRecord(d->ev[0], d->stream));
    k_linearize<<<(a.f_count + 127) / 128, 128, 0, d->stream>>>(a);
    d->n_launch++;
    CK(cudaGetLastError());
    if (d->timing) {
        CK(cudaEventRecord(d->ev[1], d->stream));
        d->ev_set[0] = 1;
    }
    return 0;
}

static int run_rebuild(asam_dev *d, const RebuildArgs &a)
{
    const int warps = a.n_pose + (a.n_slot + 31) / 32;
    k_hessian_rebuild<<<(warps + 3) / 4, 128, 0, d->stream>>>(a);
    d->n_launch++;
    CK(cudaGetLastError());
    return 0;
}

static int run_factor(asam_dev *d, const FacArgs &a, int grid, int with_leaves = 0)
{
    if (d->timing)
        CK(cudaEventRecord(d->ev[2], d->stream));
    if (with_leaves && d->n_leaf > 0) {
        LeafArgs l;
        l.sn = a.sn;
        l.ipool = a.ipool;
        l.arena = a.arena;
        l.Adiag = a.Adiag;
        l.Aoff = a.Aoff;
        l.Bq = a.Bq;
        l.q2node = a.q2node;
        l.y = a.y;
        l.dinv = a.dinv;
        l.arrive = a.arrive;
        l.tasks = (const int *) d->leaf_tasks.p;
        l.ntasks = d->n_leaf;
        l.ctrl = a.ctrl;
        l.spin_limit = a.spin_limit;
        const int want = (d->n_leaf + ASAM_LEAF_WARPS - 1) / ASAM_LEAF_WARPS;
        k_factor_leaf<<<want < d->leaf_grid ? want : d->leaf_grid, 32 * ASAM_LEAF_WARPS, d->leaf_smem, d->stream>>>(l);
        d->n_launch++;
        CK(cudaGetLastError());
    }
    if (grid > 0) {
        k_factor<<<grid, d->fac_threads, d->fac_smem, d->stream>>>(a);
        d->n_launch++;
    }
    CK(cudaGetLastError());
    if (d->timing) {
        CK(cudaEventRecord(d->ev[3], d->stream));
        d->ev_set[1] = 1;
    }
    return 0;
}

static int run_backsolve(asam_dev *d, const BsArgs &a, int grid, int nleaf = 0)
{
    if (d->timing)
        CK(cudaEventRecord(d->ev[4], d->stream));
    if (grid > 0) {
        k_backsolve<<<grid, d->bs_threads, d->bs_smem, d->stream>>>(a);
        d->n_launch++;
        CK(cudaGetLastError());
    }
    if (nleaf > 0) { // same epoch: parents outside the leaf set were flagged by the launch above
        BsArgs l = a;
        l.btasks = a.btasks + a.ntasks;
        l.ntasks = nleaf;
        const int want = (nleaf + ASAM_BSL_WARPS - 1) / ASAM_BSL_WARPS;
        k_backsolve_leaf<<<want < d->bsl_grid ? want : d->bsl_grid, 32 * ASAM_BSL_WARPS, d->bsl_smem, d->stream>>>(l);
        d->n_launch++;
        CK(cudaGetLastError());
    }
    if (d->timing) {
        CK(cudaEventRecord(d->ev[5], d->stream));
        d->ev_set[2] = 1;
    }
    return 0;
}

static int defer_push(asam_dev *d, int kind, int grid, const LinArgs *lin, const FacArgs *fac, const BsArgs *bs,
                      int nleaf = 0)
{
    if (d->npend >= ASAM_MAX_PENDING)
        return set_err("too many deferred launches");
    Pending &p = d->pend[d->npend++];
    p.kind = kind;
    p.grid = grid;
    p.nleaf = nleaf;
    if (lin) p.lin = *lin;
    if (fac) p.fac = *fac;
    if (bs) p.bs = *bs;
    return 0;
}

// Record the kernels of one incremental step and launch them after a single upload flush.
ASAM_EXPORT int asam_step_begin(asam_dev_t *d)
{
    if (!d->pend)
        d->pend = (Pending *) malloc(sizeof(Pending) * ASAM_MAX_PENDING);
    d->defer = 1;
    d->npend = 0;
    return 0;
}

ASAM_EXPORT int asam_step_run(asam_dev_t *d)
{
    CK(cudaSetDevice(d->device));
    d->defer = 0;
    if (flush_uploads(d))
        return 1;
    for (int i = 0; i < d->npend; i++) {
        Pending &p = d->pend[i];
        int rc = p.kind == 0   ? run_linearize(d, p.lin)
                 : p.kind == 1 ? run_factor(d, p.fac, p.grid)
                 : p.kind == 2 ? run_backsolve(d, p.bs, p.grid, p.nleaf)
                               : run_rebuild(d, p.rb);
        if (rc)
            return rc;
    }
    d->npend = 0;
    return 0;
}

// A small incremental step in ONE launch (k_step): the uploads queued since asam_step_begin stay in
// the pinned staging buffer and are fetched by the kernel itself; the recorded linearize / factor /
// back-solve run inside that kernel; x of the back-solved supernodes (list order, 3*cb doubles each)
// and the status word come back through pinned memory, the host spins on a sequence flag.
// Preconditions (checked): exactly linearize + factor + backsolve recorded, no leaf kernels.  Not checked
// here, the caller's to ensure (solver.c does): every factor task a single-CTA front -- k_step is one CTA,
// a team task would wait for workers that never start.  Returns 2 if the step does not qualify (nothing
// launched; call asam_step_run instead).
ASAM_EXPORT int asam_step_small_supported(asam_dev_t *d) { return d->small_ok && !d->timing && !d->trace_on && !d->sharded; }

ASAM_EXPORT int asam_step_run_small(asam_dev_t *d, double *x_out, int x_doubles, int *status_out)
{
    CK(cudaSetDevice(d->device));
    if (!d->defer || d->npend != 3 || d->pend[0].kind != 0 || d->pend[1].kind != 1 || d->pend[2].kind != 2 ||
        d->pend[2].nleaf != 0 || (size_t) x_doubles * sizeof(double) + 64 > d->pin_down_cap || d->n_items <= 0)
        return 2;
    if (d->up_busy) { // an earlier flush may still be reading the staging buffer
        CK(cudaEventSynchronize(d->up_ev));
        d->up_busy = 0;
    }
    d->defer = 0;
    StepArgs a;
    memcpy(d->pin, d->items, (size_t) d->n_items * sizeof(BatchItem));
    a.host_in = (const uint4 *) d->pin;
    a.stage = (uint4 *) d->dstage;
    a.table_bytes = (unsigned int) (d->n_items * sizeof(BatchItem));
    a.payload_off = (unsigned int) ASAM_TABLE_BYTES;
    a.payload_bytes = (unsigned int) d->pin_off;
    a.n_items = d->n_items;
    a.lin = d->pend[0].lin;
    a.fac = d->pend[1].fac;
    a.bs = d->pend[2].bs;
    a.bs.smem_doubles = d->fac_smem / (int) sizeof(double); // the CTA's whole dynamic shared memory
    a.x_out = (double *) (d->pin_down + 64);
    a.done = (volatile int *) d->pin_down;
    a.seq = ++d->step_seq;
    struct timespec ts0, ts1, ts2;
    clock_gettime(CLOCK_MONOTONIC, &ts0);
    k_step<<<1, 256, d->fac_smem, d->stream>>>(a);
    CK(cudaGetLastError());
    clock_gettime(CLOCK_MONOTONIC, &ts1);
    d->n_launch++;
    d->n_small++;
    d->n_items = 0;
    d->pin_off = 0;
    d->npend = 0;
    d->n_d2h += (int64_t) x_doubles * 8 + 8;
    volatile int *done = (volatile int *) d->pin_down;
    for (long long spins = 0; done[0] != a.seq; ++spins) {
#if defined(__x86_64__)
        __builtin_ia32_pause();
#endif
        if ((spins & 0xffff) == 0xffff) { // a faulted launch never raises the flag
            cudaError_t q = cudaStreamQuery(d->stream);
            if (q != cudaSuccess && q != cudaErrorNotReady)
                return set_err("k_step failed: %s", cudaGetErrorString(q));
            if (q == cudaSuccess && done[0] != a.seq)
                return set_err("k_step finished without raising its flag");
        }
    }
    __sync_synchronize();
    clock_gettime(CLOCK_MONOTONIC, &ts2);
    {
        const volatile unsigned long long *st = (const volatile unsigned long long *) (d->pin_down + 8);
        for (int i = 0; i < 5; i++)
            d->small_us[i] += (double) (long long) (st[i + 1] - st[i]) * 1e-3;
        d->small_us[5] += (ts1.tv_sec - ts0.tv_sec) * 1e6 + (ts1.tv_nsec - ts0.tv_nsec) * 1e-3; // launch call
        d->small_us[6] += (ts2.tv_sec - ts1.tv_sec) * 1e6 + (ts2.tv_nsec - ts1.tv_nsec) * 1e-3; // flag wait
    }
    *status_out = done[1];
    memcpy(x_out, d->pin_down + 64, (size_t) x_doubles * sizeof(double));
    if (*status_out != 0)
        return clear_status(d);
    return 0;
}

// ------------------------------------------------------------------------------------------
// C-ABI
// ------------------------------------------------------------------------------------------
ASAM_EXPORT int asam_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess)
        return 0;
    return n;
}

ASAM_EXPORT int asam_dev_create(asam_dev_t **out)
{
    *out = nullptr;
    int n = 0;
    CK(cudaGetDeviceCount(&n));
    if (n <= 0)
        return set_err("no CUDA device");
    int dev = 0;
    const char *e = getenv("ASAM_DEVICE");
    if (!e)
        e = getenv("LOCAL_RANK");
    if (e)
        dev = atoi(e) % n;
    CK(cudaSetDevice(dev));
    asam_dev *d = new asam_dev();
    d->device = dev;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, dev));
    d->n_sm = prop.multiProcessorCount;
    CK(cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking));
    d->pin_cap = 8u << 20;
    CK(cudaMallocHost((void **) &d->pin, d->pin_cap));
    CK(cudaMalloc((void **) &d->dstage, d->pin_cap));
    d->items = (BatchItem *) malloc(ASAM_TABLE_BYTES);
    CK(cudaEventCreateWithFlags(&d->up_ev, cudaEventDisableTiming));
    d->pin_down_cap = 8u << 20;
    CK(cudaMallocHost((void **) &d->pin_down, d->pin_down_cap));
    for (int i = 0; i < 6; i++)
        CK(cudaEventCreate(&d->ev[i]));
    if (buf_reserve(d, d->ctrl, 8 * sizeof(int), false, true))
        return 1;

    // launch geometry: k_factor keeps a whole front in shared memory when it fits
    int max_optin = 0;
    CK(cudaDeviceGetAttribute(&max_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    // fronts up to m = 159 stay on chip (M3500's largest is 147).  The plan decides which fronts those are with the
    // same 200 KB (plan.c:front_fits_smem), so a device that offers less cannot run k_factor at all.
    const int want = 200 * 1024;
    if (want > max_optin - 1024)
        return set_err("k_factor needs %d KB of shared memory per block, the device offers %d KB", want / 1024,
                       (max_optin - 1024) / 1024);
    d->fac_smem = want;
    CK(cudaFuncSetAttribute(k_factor, cudaFuncAttributeMaxDynamicSharedMemorySize, d->fac_smem));
    int occ = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_factor, d->fac_threads, d->fac_smem));
    if (occ < 1)
        return set_err("k_factor does not fit on an SM");
    d->fac_grid = occ * d->n_sm;

    d->leaf_smem = ASAM_LEAF_WARPS * ASAM_LEAF_STRIDE * (int) sizeof(double);
    CK(cudaFuncSetAttribute(k_factor_leaf, cudaFuncAttributeMaxDynamicSharedMemorySize, d->leaf_smem));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_factor_leaf, 32 * ASAM_LEAF_WARPS, d->leaf_smem));
    if (occ < 1)
        return set_err("k_factor_leaf does not fit on an SM");
    d->leaf_grid = occ * d->n_sm;

    d->bsl_smem = ASAM_BSL_WARPS * ASAM_BSL_STRIDE * (int) sizeof(double);
    CK(cudaFuncSetAttribute(k_backsolve_leaf, cudaFuncAttributeMaxDynamicSharedMemorySize, d->bsl_smem));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_backsolve_leaf, 32 * ASAM_BSL_WARPS, d->bsl_smem));
    if (occ < 1)
        return set_err("k_backsolve_leaf does not fit on an SM");
    d->bsl_grid = occ * d->n_sm;

    if (getenv("ASAM_BS_THREADS"))
        d->bs_threads = atoi(getenv("ASAM_BS_THREADS")) >= 256 ? 256 : 128;
    d->bs_smem = 100 * 1024; // two CTAs per SM; L11 of a 96-column supernode stays on chip
    CK(cudaFuncSetAttribute(k_backsolve, cudaFuncAttributeMaxDynamicSharedMemorySize, d->bs_smem));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_backsolve, d->bs_threads, d->bs_smem));
    if (occ < 1)
        return set_err("k_backsolve does not fit on an SM");
    d->bs_grid = occ * d->n_sm;
    CK(cudaFuncSetAttribute(k_step, cudaFuncAttributeMaxDynamicSharedMemorySize, d->fac_smem));
    if (getenv("ASAM_SOLO_PB") && atoi(getenv("ASAM_SOLO_PB")) >= 12)
        d->solo_pb = atoi(getenv("ASAM_SOLO_PB")) / 12 * 12;
    if (getenv("ASAM_PB_SMEM") && atoi(getenv("ASAM_PB_SMEM")) >= 3)
        d->pb_smem = atoi(getenv("ASAM_PB_SMEM")) / 3 * 3;
    if (getenv("ASAM_SMEM_MMA"))
        d->smem_mma = atoi(getenv("ASAM_SMEM_MMA"));
    if (getenv("ASAM_DMAP_AHEAD")) {
        const int v = atoi(getenv("ASAM_DMAP_AHEAD")) != 0;
        CK(cudaMemcpyToSymbol(g_dmap_ahead, &v, sizeof(int)));
    }
    if (getenv("ASAM_PF_GROUPS")) {
        const int v = atoi(getenv("ASAM_PF_GROUPS")) != 0;
        CK(cudaMemcpyToSymbol(g_pf_groups, &v, sizeof(int)));
    }
    if (getenv("ASAM_KEEP"))
        d->keep_off = atoi(getenv("ASAM_KEEP")) == 0;
    if (getenv("ASAM_SMALL_STEP"))
        d->small_ok = atoi(getenv("ASAM_SMALL_STEP")) != 0;
    memset(d->pin_down, 0, 64);
    *out = d;
    return 0;
}

ASAM_EXPORT void asam_dev_destroy(asam_dev_t *d)
{
    if (!d)
        return;
    cudaSetDevice(d->device);
    cudaStreamSynchronize(d->stream);
    Buf *all[] = { &d->f_type, &d->f_a, &d->f_b, &d->f_z, &d->f_W, &d->f_slot, &d->f_loss, &d->lp, &d->st, &d->node2q, &d->q2node,
                   &d->Adiag, &d->Aoff, &d->Bq, &d->y, &d->x, &d->dinv, &d->sn, &d->ipool, &d->arena, &d->arrive,
                   &d->xdone, &d->xblk, &d->tbar, &d->tasks_full, &d->nwait_full, &d->btasks_full, &d->tasks_tmp, &d->nwait_tmp,
                   &d->btasks_tmp, &d->keep_tmp, &d->leaf_tasks, &d->top_tasks, &d->top_nwait, &d->ctrl, &d->partial, &d->patch_ids, &d->patch_desc, &d->pts, &d->rb_int, &d->rb_dbl, &d->flush, &d->trace_fac, &d->trace_bs, &d->ptrace, &d->marg };
    for (int i = 0; i < 2; i++)
        if (d->tev[i])
            cudaEventDestroy(d->tev[i]);
    for (Buf *b : all)
        if (b->p)
            cudaFree(b->p);
    if (d->pin)
        cudaFreeHost(d->pin);
    if (d->pin_down)
        cudaFreeHost(d->pin_down);
    if (d->dstage)
        cudaFree(d->dstage);
    if (d->up_ev)
        cudaEventDestroy(d->up_ev);
    free(d->items);
    free(d->pend);
    free(d->sh_owner); free(d->sh_q0); free(d->sh_qn); free(d->sh_off); free(d->sh_cnt);
    for (int i = 0; i < 6; i++)
        if (d->ev[i])
            cudaEventDestroy(d->ev[i]);
    cudaStreamDestroy(d->stream);
    delete d;
}

ASAM_EXPORT int asam_reserve(asam_dev_t *d, int n_nodes, int n_factors, int n_slots, int n_sn, int64_t ipool_ints,
                             int64_t arena_doubles)
{
    CK(cudaSetDevice(d->device));
    size_t N = (size_t) (n_nodes > 0 ? n_nodes : 0), Fn = (size_t) (n_factors > 0 ? n_factors : 0);
    size_t S = (size_t) (n_slots > 0 ? n_slots : 0), SN = (size_t) (n_sn > 0 ? n_sn : 0);
    int rc = 0;
    rc |= buf_reserve(d, d->f_type, Fn * sizeof(int), true, false);
    rc |= buf_reserve(d, d->f_a, Fn * sizeof(int), true, false);
    rc |= buf_reserve(d, d->f_b, Fn * sizeof(int), true, false);
    rc |= buf_reserve(d, d->f_slot, Fn * sizeof(int), true, false);
    rc |= buf_reserve(d, d->f_z, Fn * 3 * sizeof(double), true, false);
    rc |= buf_reserve(d, d->f_W, Fn * 9 * sizeof(double), true, false);
    if (d->f_loss.cap) // in use (asam_upload_loss): grows with the factor capacity
        rc |= buf_reserve(d, d->f_loss, Fn * 2 * sizeof(double), true, false);
    rc |= buf_reserve(d, d->lp, N * 3 * sizeof(double), true, false);
    rc |= buf_reserve(d, d->st, N * 3 * sizeof(double), true, false);
    rc |= buf_reserve(d, d->node2q, N * sizeof(int), true, false);
    rc |= buf_reserve(d, d->q2node, N * sizeof(int), true, false);
    rc |= buf_reserve(d, d->Adiag, N * 9 * sizeof(double), true, true);
    rc |= buf_reserve(d, d->Bq, N * 3 * sizeof(double), true, true);
    rc |= buf_reserve(d, d->y, N * 3 * sizeof(double), true, true);
    rc |= buf_reserve(d, d->x, N * 3 * sizeof(double), true, true);
    rc |= buf_reserve(d, d->dinv, N * 3 * sizeof(double), true, true);
    rc |= buf_reserve(d, d->Aoff, S * 9 * sizeof(double), true, true);
    rc |= buf_reserve(d, d->sn, SN * sizeof(asam_sn_desc_t), true, false);
    rc |= buf_reserve(d, d->arrive, SN * sizeof(int), true, true);
    rc |= buf_reserve(d, d->xdone, SN * sizeof(int), true, true);
    rc |= buf_reserve(d, d->xblk, SN * sizeof(int), true, true);
    rc |= buf_reserve(d, d->tbar, 2 * SN * sizeof(int), true, true);
    rc |= buf_reserve(d, d->ipool, (size_t) ipool_ints * sizeof(int), true, false);
    rc |= buf_reserve(d, d->arena, (size_t) arena_doubles * sizeof(double), true, false);
    return rc;
}

ASAM_EXPORT int asam_upload_factors(asam_dev_t *d, int first, int count, const int32_t *type, const int32_t *na,
                                    const int32_t *nb, const double *z3, const double *W9)
{
    if (count <= 0)
        return 0;
    size_t need = (size_t) first + count;
    if (need * sizeof(int) > d->f_type.cap)
        return set_err("asam_upload_factors: capacity (call asam_reserve)");
    int rc = 0;
    rc |= upload(d, (int *) d->f_type.p + first, type, count * sizeof(int));
    rc |= upload(d, (int *) d->f_a.p + first, na, count * sizeof(int));
    rc |= upload(d, (int *) d->f_b.p + first, nb, count * sizeof(int));
    rc |= upload(d, (double *) d->f_z.p + 3 * (size_t) first, z3, count * 3 * sizeof(double));
    rc |= upload(d, (double *) d->f_W.p + 9 * (size_t) first, W9, count * 9 * sizeof(double));
    return rc;
}

ASAM_EXPORT int asam_upload_loss(asam_dev_t *d, int first, int count, const int32_t *loss, const double *k)
{
    if (count <= 0)
        return 0;
    if (((size_t) first + count) * sizeof(int) > d->f_type.cap)
        return set_err("asam_upload_loss: capacity (call asam_reserve)");
    // first robust factor of this context: one record per factor of the reserved capacity
    if (buf_reserve(d, d->f_loss, d->f_type.cap / sizeof(int) * 2 * sizeof(double), true, false))
        return 1;
    // one 16-byte record per factor: the loss code travels as a double next to k
    std::vector<double> rec(2 * (size_t) count);
    for (int i = 0; i < count; i++) {
        rec[2 * (size_t) i] = (double) loss[i];
        rec[2 * (size_t) i + 1] = k[i];
    }
    return upload(d, (double *) d->f_loss.p + 2 * (size_t) first, rec.data(), rec.size() * sizeof(double));
}

ASAM_EXPORT int asam_upload_points(asam_dev_t *d, int which, int first, int count, const double *p3)
{
    if (count <= 0)
        return 0;
    Buf &b = which == 0 ? d->lp : d->st;
    if (((size_t) first + count) * 3 * sizeof(double) > b.cap)
        return set_err("asam_upload_points: capacity");
    return upload(d, (double *) b.p + 3 * (size_t) first, p3, (size_t) count * 3 * sizeof(double));
}

ASAM_EXPORT int asam_copy_points(asam_dev_t *d, int from, int to, int first, int count)
{
    if (count <= 0 || from == to)
        return 0;
    CK(cudaSetDevice(d->device));
    Buf &src = from == 0 ? d->lp : d->st, &dst = to == 0 ? d->lp : d->st;
    const size_t off = (size_t) first * 3 * sizeof(double), bytes = (size_t) count * 3 * sizeof(double);
    if (off + bytes > src.cap || off + bytes > dst.cap)
        return set_err("asam_copy_points: capacity");
    if (flush_uploads(d)) // the source may still be queued
        return 1;
    CK(cudaMemcpyAsync((char *) dst.p + off, (const char *) src.p + off, bytes, cudaMemcpyDeviceToDevice, d->stream));
    return 0;
}

ASAM_EXPORT int asam_upload_node2q(asam_dev_t *d, int first, int count, const int32_t *node2q)
{
    if (count <= 0)
        return 0;
    if (((size_t) first + count) * sizeof(int) > d->node2q.cap)
        return set_err("asam_upload_node2q: capacity");
    return upload(d, (int *) d->node2q.p + first, node2q, (size_t) count * sizeof(int));
}

ASAM_EXPORT int asam_upload_q2node(asam_dev_t *d, int first, int count, const int32_t *q2node)
{
    if (count <= 0)
        return 0;
    if (((size_t) first + count) * sizeof(int) > d->q2node.cap)
        return set_err("asam_upload_q2node: capacity");
    return upload(d, (int *) d->q2node.p + first, q2node, (size_t) count * sizeof(int));
}

ASAM_EXPORT int asam_upload_fslot(asam_dev_t *d, int first, int count, const int32_t *fslot)
{
    if (count <= 0)
        return 0;
    if (((size_t) first + count) * sizeof(int) > d->f_slot.cap)
        return set_err("asam_upload_fslot: capacity");
    return upload(d, (int *) d->f_slot.p + first, fslot, (size_t) count * sizeof(int));
}

ASAM_EXPORT int asam_upload_ipool(asam_dev_t *d, int64_t first, int64_t count, const int32_t *data)
{
    if (count <= 0)
        return 0;
    if ((size_t) (first + count) * sizeof(int) > d->ipool.cap)
        return set_err("asam_upload_ipool: capacity");
    return upload(d, (int *) d->ipool.p + first, data, (size_t) count * sizeof(int));
}

ASAM_EXPORT int asam_upload_desc(asam_dev_t *d, int n, const int32_t *sn_ids, const asam_sn_desc_t *desc)
{
    if (n <= 0)
        return 0;
    CK(cudaSetDevice(d->device));
    if (n <= 256) { // incremental step: each descriptor is one queued 48-byte copy
        for (int i = 0; i < n; i++)
            if (upload(d, (asam_sn_desc_t *) d->sn.p + sn_ids[i], &desc[i], sizeof(asam_sn_desc_t)))
                return 1;
        return 0;
    }
    if (buf_reserve(d, d->patch_ids, (size_t) n * sizeof(int), false, false))
        return 1;
    if (buf_reserve(d, d->patch_desc, (size_t) n * sizeof(asam_sn_desc_t), false, false))
        return 1;
    if (upload(d, d->patch_ids.p, sn_ids, (size_t) n * sizeof(int)))
        return 1;
    if (upload(d, d->patch_desc.p, desc, (size_t) n * sizeof(asam_sn_desc_t)))
        return 1;
    if (flush_uploads(d))
        return 1;
    k_apply_desc<<<(n + 127) / 128, 128, 0, d->stream>>>((asam_sn_desc_t *) d->sn.p, (const int *) d->patch_ids.p,
                                                         (const asam_sn_desc_t *) d->patch_desc.p, n);
    d->n_launch++;
    CK(cudaGetLastError());
    return 0;
}

ASAM_EXPORT int asam_hessian_reset(asam_dev_t *d, int n_nodes, int n_slots, int n_lambda, double lambda)
{
    CK(cudaSetDevice(d->device));
    size_t total = 9 * (size_t) n_nodes + 9 * (size_t) n_slots + 3 * (size_t) n_nodes;
    if (total == 0)
        return 0;
    if (flush_uploads(d))
        return 1;
    k_hessian_reset<<<(unsigned) ((total + 255) / 256), 256, 0, d->stream>>>(
        (double *) d->Adiag.p, (double *) d->Aoff.p, (double *) d->Bq.p, n_nodes, n_slots, n_lambda, lambda);
    d->n_launch++;
    CK(cudaGetLastError());
    return 0;
}

ASAM_EXPORT int asam_hessian_clear_range(asam_dev_t *d, int q_first, int q_count, int slot_first, int slot_count)
{
    CK(cudaSetDevice(d->device));
    int rc = 0;
    if (q_count > 0) {
        rc |= queue_fill(d, (double *) d->Adiag.p + 9 * (size_t) q_first, 0, (size_t) q_count * 9 * sizeof(double));
        rc |= queue_fill(d, (double *) d->Bq.p + 3 * (size_t) q_first, 0, (size_t) q_count * 3 * sizeof(double));
    }
    if (slot_count > 0)
        rc |= queue_fill(d, (double *) d->Aoff.p + 9 * (size_t) slot_first, 0, (size_t) slot_count * 9 * sizeof(double));
    return rc;
}

ASAM_EXPORT int asam_linearize(asam_dev_t *d, int f_first, int f_count, const double *pts6)
{
    if (f_count <= 0)
        return 0;
    CK(cudaSetDevice(d->device));
    LinArgs a;
    a.f_type = (const int *) d->f_type.p;
    a.f_a = (const int *) d->f_a.p;
    a.f_b = (const int *) d->f_b.p;
    a.f_slot = (const int *) d->f_slot.p;
    a.f_z = (const double *) d->f_z.p;
    a.f_W = (const double *) d->f_W.p;
    a.f_loss = (const double2 *) d->f_loss.p;
    a.lp = (const double *) d->lp.p;
    a.st = (const double *) d->st.p;
    a.pts = nullptr;
    if (pts6) {
        if (buf_reserve(d, d->pts, (size_t) f_count * 6 * sizeof(double), false, false))
            return 1;
        if (upload(d, d->pts.p, pts6, (size_t) f_count * 6 * sizeof(double)))
            return 1;
        a.pts = (const double *) d->pts.p;
    }
    a.node2q = (const int *) d->node2q.p;
    a.Adiag = (double *) d->Adiag.p;
    a.Aoff = (double *) d->Aoff.p;
    a.Bq = (double *) d->Bq.p;
    a.f_first = f_first;
    a.f_count = f_count;
    if (d->defer)
        return defer_push(d, 0, 0, &a, nullptr, nullptr);
    if (flush_uploads(d))
        return 1;
    return run_linearize(d, a);
}

ASAM_EXPORT int asam_hessian_rebuild(asam_dev_t *d, int n_pose, const int32_t *pose, const int32_t *pose_ptr, int n_slot,
                                     const int32_t *slot, const int32_t *slot_ptr, int n_ent, const int32_t *ent_f,
                                     const double *ent_pts, const double *lam)
{
    if (n_pose < 0 || n_slot < 0 || n_ent < 0)
        return set_err("asam_hessian_rebuild: %d poses, %d slots, %d entries", n_pose, n_slot, n_ent);
    if (n_pose == 0 && n_slot == 0)
        return 0;
    CK(cudaSetDevice(d->device));
    // ints: pose | pose_ptr | slot | slot_ptr | ent_f;  doubles: ent_pts | lam
    const size_t ni = (size_t) n_pose + (n_pose + 1) + n_slot + (n_slot + 1) + n_ent;
    const size_t nd = 6 * (size_t) n_ent + n_pose;
    if (buf_reserve(d, d->rb_int, ni * sizeof(int), false, false) ||
        buf_reserve(d, d->rb_dbl, (nd ? nd : 1) * sizeof(double), false, false))
        return 1;
    int *ip = (int *) d->rb_int.p;
    double *dp = (double *) d->rb_dbl.p;
    RebuildArgs a;
    a.f_type = (const int *) d->f_type.p;
    a.f_a = (const int *) d->f_a.p;
    a.f_b = (const int *) d->f_b.p;
    a.f_z = (const double *) d->f_z.p;
    a.f_W = (const double *) d->f_W.p;
    a.f_loss = (const double2 *) d->f_loss.p;
    a.node2q = (const int *) d->node2q.p;
    a.pose = ip;
    a.pose_ptr = ip + n_pose;
    a.slot = ip + 2 * (size_t) n_pose + 1;
    a.slot_ptr = a.slot + n_slot;
    a.ent_f = a.slot_ptr + n_slot + 1;
    a.ent_pts = dp;
    a.lam = dp + 6 * (size_t) n_ent;
    a.Adiag = (double *) d->Adiag.p;
    a.Aoff = (double *) d->Aoff.p;
    a.Bq = (double *) d->Bq.p;
    a.n_pose = n_pose;
    a.n_slot = n_slot;
    int rc = 0;
    if (n_pose > 0) {
        rc |= upload(d, (void *) a.pose, pose, (size_t) n_pose * sizeof(int));
        rc |= upload(d, (void *) a.pose_ptr, pose_ptr, (size_t) (n_pose + 1) * sizeof(int));
        rc |= upload(d, (void *) a.lam, lam, (size_t) n_pose * sizeof(double));
    }
    if (n_slot > 0) {
        rc |= upload(d, (void *) a.slot, slot, (size_t) n_slot * sizeof(int));
        rc |= upload(d, (void *) a.slot_ptr, slot_ptr, (size_t) (n_slot + 1) * sizeof(int));
    }
    if (n_ent > 0) {
        rc |= upload(d, (void *) a.ent_f, ent_f, (size_t) n_ent * sizeof(int));
        rc |= upload(d, (void *) a.ent_pts, ent_pts, 6 * (size_t) n_ent * sizeof(double));
    }
    if (rc)
        return 1;
    if (d->defer) {
        if (d->npend >= ASAM_MAX_PENDING)
            return set_err("too many deferred launches");
        Pending &p = d->pend[d->npend++];
        p.kind = 3;
        p.grid = 0;
        p.nleaf = 0;
        p.rb = a;
        return 0;
    }
    if (flush_uploads(d))
        return 1;
    return run_rebuild(d, a);
}

static int launch_factor(asam_dev *d, int ntasks, const int *tasks_dev, const int *nwait_dev, int with_leaves = 0,
                         const int *keep_dev = nullptr)
{
    if (ntasks <= 0 && !(with_leaves && d->n_leaf > 0))
        return 0;
    // ticket / team-barrier counters are left at zero by the previous launch (ticket_release,
    // team_leave); err is only ever non-zero on a fatal path (see clear_status)
    FacArgs a;
    a.sn = (const asam_sn_desc_t *) d->sn.p;
    a.ipool = (const int *) d->ipool.p;
    a.arena = (double *) d->arena.p;
    a.Adiag = (const double *) d->Adiag.p;
    a.Aoff = (const double *) d->Aoff.p;
    a.Bq = (const double *) d->Bq.p;
    a.q2node = (const int *) d->q2node.p;
    a.y = (double *) d->y.p;
    a.dinv = (double *) d->dinv.p;
    a.arrive = (int *) d->arrive.p;
    a.tbar = (int *) d->tbar.p;
    a.tasks = tasks_dev;
    a.nwait = nwait_dev;
    a.keep = keep_dev;
    a.ntasks = ntasks;
    a.ctrl = (int *) d->ctrl.p;
    a.smem_doubles = d->fac_smem / (int) sizeof(double);
    a.spin_limit = ASAM_SPIN_LIMIT_NS;
    a.solo_pb = d->solo_pb;
    a.smem_mma = d->smem_mma;
    a.pb_smem = d->pb_smem;
    a.trace = nullptr;
    if (d->trace_on) {
        if (buf_reserve(d, d->trace_fac, (size_t) ntasks * 8 * sizeof(unsigned long long), false, false))
            return 1;
        a.trace = (unsigned long long *) d->trace_fac.p;
        d->trace_nfac = ntasks;
    }
    a.ptrace = d->ptrace_sn >= 0 ? (unsigned long long *) d->ptrace.p : nullptr;
    a.ptrace_sn = d->ptrace_sn;
    a.ptrace_panels = d->ptrace_panels;
    int grid = d->fac_grid < ntasks ? d->fac_grid : ntasks;
    if (d->defer) {
        if (with_leaves && d->n_leaf > 0)
            return set_err("asam_factor_full inside asam_step_begin/asam_step_run");
        return defer_push(d, 1, grid, nullptr, &a, nullptr);
    }
    if (flush_uploads(d))
        return 1;
    return run_factor(d, a, grid, with_leaves);
}

static int launch_backsolve(asam_dev *d, int ntasks, const int *btasks_dev, int nleaf = 0, const int *bfirst_dev = nullptr)
{
    if (ntasks <= 0)
        return 0;
    ntasks -= nleaf; // the leaf part follows the main part in the list
    d->epoch++;
    BsArgs a;
    a.sn = (const asam_sn_desc_t *) d->sn.p;
    a.ipool = (const int *) d->ipool.p;
    a.arena = (const double *) d->arena.p;
    a.y = (const double *) d->y.p;
    a.dinv = (const double *) d->dinv.p;
    a.x = (double *) d->x.p;
    a.xdone = (int *) d->xdone.p;
    a.xblk = (int *) d->xblk.p;
    a.btasks = btasks_dev;
    a.bfirst = bfirst_dev;
    a.ntasks = ntasks;
    a.ctrl = (int *) d->ctrl.p;
    a.epoch = d->epoch;
    a.smem_doubles = d->bs_smem / (int) sizeof(double);
    a.spin_limit = ASAM_SPIN_LIMIT_NS;
    a.trace = nullptr;
    if (d->trace_on) {
        if (buf_reserve(d, d->trace_bs, (size_t) ntasks * 8 * sizeof(unsigned long long), false, false))
            return 1;
        a.trace = (unsigned long long *) d->trace_bs.p;
        d->trace_nbs = ntasks;
    }
    int grid = d->bs_grid < ntasks ? d->bs_grid : ntasks;
    if (d->defer)
        return defer_push(d, 2, grid, nullptr, nullptr, &a, nleaf);
    if (flush_uploads(d))
        return 1;
    return run_backsolve(d, a, grid, nleaf);
}

ASAM_EXPORT int asam_set_full_tasks(asam_dev_t *d, int ntasks, const int32_t *tasks, const int32_t *nwait,
                                    int nbtasks, const int32_t *btasks)
{
    CK(cudaSetDevice(d->device));
    size_t b = (size_t) ntasks * sizeof(int), bb = (size_t) nbtasks * sizeof(int);
    int headroom = nbtasks / 2 + 1024; // room to prepend supernodes of poses appended later
    if (buf_reserve(d, d->tasks_full, b, false, false) || buf_reserve(d, d->nwait_full, b, false, false) ||
        buf_reserve(d, d->btasks_full, bb + (size_t) headroom * sizeof(int), false, false))
        return 1;
    d->bt_cap = (int) (d->btasks_full.cap / sizeof(int));
    d->bt_start = d->bt_cap - nbtasks;
    d->bt_count = nbtasks;
    if (upload(d, d->tasks_full.p, tasks, b) || upload(d, d->nwait_full.p, nwait, b) ||
        upload(d, (int *) d->btasks_full.p + d->bt_start, btasks, bb))
        return 1;
    d->ntasks_full = ntasks;
    d->n_leaf = 0;
    d->bt_nleaf = 0;
    return 0;
}

// Supernodes of the batch schedule that k_factor_leaf handles (one warp per front) before
// k_factor runs the list given to asam_set_full_tasks; call after asam_set_full_tasks.
ASAM_EXPORT int asam_set_leaf_tasks(asam_dev_t *d, int n, const int32_t *tasks)
{
    CK(cudaSetDevice(d->device));
    d->n_leaf = 0;
    if (n <= 0)
        return 0;
    if (buf_reserve(d, d->leaf_tasks, (size_t) n * sizeof(int), false, false) ||
        upload(d, d->leaf_tasks.p, tasks, (size_t) n * sizeof(int)))
        return 1;
    d->n_leaf = n;
    return 0;
}

// The LAST n entries of the back-solve list (asam_set_full_tasks) go through k_backsolve_leaf.
ASAM_EXPORT int asam_set_bs_leaf_count(asam_dev_t *d, int n)
{
    if (n < 0 || n > d->bt_count)
        return set_err("asam_set_bs_leaf_count: %d of %d", n, d->bt_count);
    d->bt_nleaf = n;
    return 0;
}

ASAM_EXPORT int asam_btasks_prepend(asam_dev_t *d, int n, const int32_t *ids)
{
    if (n <= 0)
        return 0;
    CK(cudaSetDevice(d->device));
    if (d->bt_start < n) { // out of head-room: move the list to the end of a larger buffer
        if (flush_uploads(d))
            return 1;
        int newcap = 2 * (d->bt_count + n) + 1024;
        void *np = nullptr;
        CK(cudaMalloc(&np, (size_t) newcap * sizeof(int)));
        int newstart = newcap - d->bt_count;
        CK(cudaMemcpyAsync((int *) np + newstart, (int *) d->btasks_full.p + d->bt_start,
                           (size_t) d->bt_count * sizeof(int), cudaMemcpyDeviceToDevice, d->stream));
        CK(cudaStreamSynchronize(d->stream));
        CK(cudaFree(d->btasks_full.p));
        d->btasks_full.p = np;
        d->btasks_full.cap = (size_t) newcap * sizeof(int);
        d->bt_cap = newcap;
        d->bt_start = newstart;
    }
    d->bt_start -= n;
    d->bt_count += n;
    return upload(d, (int *) d->btasks_full.p + d->bt_start, ids, (size_t) n * sizeof(int));
}

// ------------------------------------------------------------------------------------------
// several GPUs: NCCL through dlopen (no link-time dependency; a copy already loaded by the host
// application, e.g. PyTorch's, is re-used because it has the same soname)
// ------------------------------------------------------------------------------------------
typedef struct ncclComm *nccl_comm_t;
typedef struct { char internal[128]; } nccl_uid_t;
struct NcclApi {
    void *h = nullptr;
    int (*GetUniqueId)(nccl_uid_t *) = nullptr;
    int (*CommInitRank)(nccl_comm_t *, int, nccl_uid_t, int) = nullptr;
    int (*CommDestroy)(nccl_comm_t) = nullptr;
    int (*Broadcast)(const void *, void *, size_t, int, int, nccl_comm_t, cudaStream_t) = nullptr;
    int (*AllReduce)(const void *, void *, size_t, int, int, nccl_comm_t, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    const char *(*GetErrorString)(int) = nullptr;
};
static NcclApi g_nccl;
static nccl_comm_t g_comm = nullptr;
static int g_world = 1, g_rank = 0, g_sharding = 0;
#define ASAM_NCCL_FLOAT64 8
#define ASAM_NCCL_INT32 2
#define ASAM_NCCL_SUM 0
#define ASAM_NCCL_MIN 3

#define NCK(call)                                                                                  \
    do {                                                                                           \
        int r_ = (call);                                                                           \
        if (r_ != 0)                                                                               \
            return set_err("%s:%d %s -> NCCL error %d (%s)", __FILE__, __LINE__, #call, r_,        \
                           g_nccl.GetErrorString ? g_nccl.GetErrorString(r_) : "?");               \
    } while (0)

static int nccl_load()
{
    if (g_nccl.h)
        return 0;
    void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h)
        h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h)
        return set_err("cannot load libnccl.so.2: %s", dlerror());
#define SYM(field, name)                                                  \
    *(void **) (&g_nccl.field) = dlsym(h, name);                          \
    if (!g_nccl.field)                                                    \
        return set_err("libnccl: symbol %s missing", name);
    SYM(GetUniqueId, "ncclGetUniqueId")
    SYM(CommInitRank, "ncclCommInitRank")
    SYM(CommDestroy, "ncclCommDestroy")
    SYM(Broadcast, "ncclBroadcast")
    SYM(AllReduce, "ncclAllReduce")
    SYM(GroupStart, "ncclGroupStart")
    SYM(GroupEnd, "ncclGroupEnd")
    SYM(GetErrorString, "ncclGetErrorString")
#undef SYM
    g_nccl.h = h;
    return 0;
}

static int select_device(int *dev_out)
{
    int n = 0;
    CK(cudaGetDeviceCount(&n));
    if (n <= 0)
        return set_err("no CUDA device");
    int dev = 0;
    const char *e = getenv("ASAM_DEVICE");
    if (!e)
        e = getenv("LOCAL_RANK");
    if (e)
        dev = atoi(e) % n;
    *dev_out = dev;
    return 0;
}

ASAM_EXPORT int asam_comm_unique_id(void *id128_out)
{
    if (nccl_load())
        return 1;
    nccl_uid_t id;
    NCK(g_nccl.GetUniqueId(&id));
    memcpy(id128_out, &id, sizeof(id));
    return 0;
}

ASAM_EXPORT int asam_comm_init(int world, int rank, const void *id128)
{
    if (world < 1 || rank < 0 || rank >= world)
        return set_err("asam_comm_init: bad world/rank %d/%d", world, rank);
    if (g_comm)
        return set_err("asam_comm_init: communicator already initialised");
    if (world == 1) {
        g_world = 1;
        g_rank = 0;
        return 0;
    }
    if (nccl_load())
        return 1;
    int dev = 0;
    if (select_device(&dev))
        return 1;
    CK(cudaSetDevice(dev));
    nccl_uid_t id;
    memcpy(&id, id128, sizeof(id));
    NCK(g_nccl.CommInitRank(&g_comm, world, id, rank));
    g_world = world;
    g_rank = rank;
    return 0;
}

ASAM_EXPORT void asam_comm_destroy(void)
{
    if (g_comm && g_nccl.CommDestroy)
        g_nccl.CommDestroy(g_comm);
    g_comm = nullptr;
    g_world = 1;
    g_rank = 0;
    g_sharding = 0;
}

ASAM_EXPORT int asam_comm_info(int *world, int *rank, int *sharding)
{
    if (world)
        *world = g_world;
    if (rank)
        *rank = g_rank;
    if (sharding)
        *sharding = g_sharding && g_world > 1;
    return 0;
}

ASAM_EXPORT int asam_comm_set_sharding(int enabled)
{
    if (enabled && (g_world <= 1 || !g_comm))
        return set_err("asam_comm_set_sharding: no communicator (asam_comm_init)");
    g_sharding = enabled ? 1 : 0;
    return 0;
}

ASAM_EXPORT int asam_set_shard_schedule(asam_dev_t *d, const asam_shard_sched_t *sh)
{
    CK(cudaSetDevice(d->device));
    d->sharded = 0;
    d->n_top = 0;
    d->n_shards = 0;
    free(d->sh_owner); free(d->sh_q0); free(d->sh_qn); free(d->sh_off); free(d->sh_cnt);
    d->sh_owner = d->sh_q0 = d->sh_qn = nullptr;
    d->sh_off = d->sh_cnt = nullptr;
    if (!sh)
        return 0;
    if (g_world <= 1 || !g_comm)
        return set_err("asam_set_shard_schedule: no communicator (asam_comm_init)");
    size_t b = (size_t) sh->n_top * sizeof(int);
    if (sh->n_top > 0) {
        if (buf_reserve(d, d->top_tasks, b, false, false) || buf_reserve(d, d->top_nwait, b, false, false) ||
            upload(d, d->top_tasks.p, sh->top_tasks, b) || upload(d, d->top_nwait.p, sh->top_nwait, b))
            return 1;
    }
    const int n = sh->n_shards;
    d->sh_owner = (int *) malloc(sizeof(int) * (size_t) (n + 1));
    d->sh_q0 = (int *) malloc(sizeof(int) * (size_t) (n + 1));
    d->sh_qn = (int *) malloc(sizeof(int) * (size_t) (n + 1));
    d->sh_off = (long long *) malloc(sizeof(long long) * (size_t) (n + 1));
    d->sh_cnt = (long long *) malloc(sizeof(long long) * (size_t) (n + 1));
    for (int i = 0; i < n; i++) {
        d->sh_owner[i] = sh->shard_owner[i];
        d->sh_q0[i] = sh->shard_q0[i];
        d->sh_qn[i] = sh->shard_qn[i];
        d->sh_off[i] = sh->shard_off[i];
        d->sh_cnt[i] = sh->shard_cnt[i];
        if (d->sh_owner[i] < 0 || d->sh_owner[i] >= g_world)
            return set_err("asam_set_shard_schedule: shard %d owner %d", i, d->sh_owner[i]);
    }
    d->n_top = sh->n_top;
    d->n_shards = n;
    d->sharded = 1;
    return 0;
}

// root fronts of the shards (which = 0) or their solution segments (which = 1): one grouped
// NCCL broadcast per shard on the library's stream, in place (same offsets on every rank)
static int shard_exchange(asam_dev *d, int which)
{
    if (!d->sharded || d->n_shards == 0)
        return 0;
    NCK(g_nccl.GroupStart());
    for (int i = 0; i < d->n_shards; i++) {
        void *p;
        size_t count;
        if (which == 0) {
            p = (double *) d->arena.p + d->sh_off[i];
            count = (size_t) d->sh_cnt[i];
        } else {
            p = (double *) d->x.p + 3 * (size_t) d->sh_q0[i];
            count = 3 * (size_t) d->sh_qn[i];
        }
        if (count == 0)
            continue;
        NCK(g_nccl.Broadcast(p, p, count, ASAM_NCCL_FLOAT64, d->sh_owner[i], g_comm, d->stream));
    }
    NCK(g_nccl.GroupEnd());
    d->n_launch++;
    return 0;
}

// Sharded solves: every rank reads the same status word, the one of the rank that owns the failure (each rank owns a
// copy of the caller's graph and takes the same action).  A failed pivot in a shard poisons the shard root's update
// matrix, which the exchange carries to every rank, so the other ranks fail a top ancestor of it; ancestors have
// larger ids than their descendants, so the smallest failing supernode is the owner's.  ctrl[7] = the word as a key
// (timeouts below failed pivots below a clean word), all-reduced (min), written back.
__global__ void k_status_flag(int *ctrl, int phase)
{
    if (phase == 0)
        ctrl[7] = ctrl[1] == 0 ? INT_MAX : ctrl[1];
    else
        ctrl[1] = ctrl[7] == INT_MAX ? 0 : ctrl[7];
}

static int shard_status_agree(asam_dev *d)
{
    if (!d->sharded)
        return 0;
    int *ctrl = (int *) d->ctrl.p;
    k_status_flag<<<1, 1, 0, d->stream>>>(ctrl, 0);
    NCK(g_nccl.AllReduce(ctrl + 7, ctrl + 7, 1, ASAM_NCCL_INT32, ASAM_NCCL_MIN, g_comm, d->stream));
    k_status_flag<<<1, 1, 0, d->stream>>>(ctrl, 1);
    CK(cudaGetLastError());
    d->n_launch += 3;
    return 0;
}

ASAM_EXPORT int asam_factor_full(asam_dev_t *d)
{
    CK(cudaSetDevice(d->device));
    if (!d->sharded)
        return launch_factor(d, d->ntasks_full, (const int *) d->tasks_full.p, (const int *) d->nwait_full.p, 1);
    if (d->defer)
        return set_err("sharded asam_factor_full inside asam_step_begin/asam_step_run");
    // own shards -> exchange of the shard roots' update matrices -> the supernodes above the cut
    const int timing = d->timing;
    if (flush_uploads(d))
        return 1;
    if (timing)
        CK(cudaEventRecord(d->ev[2], d->stream));
    d->timing = 0;
    int rc = launch_factor(d, d->ntasks_full, (const int *) d->tasks_full.p, (const int *) d->nwait_full.p, 1);
    if (!rc)
        rc = shard_exchange(d, 0);
    // arrivals of the shard roots at parents above the cut were counted before the exchange
    if (!rc && d->arrive.p && cudaMemsetAsync(d->arrive.p, 0, d->arrive.cap, d->stream) != cudaSuccess)
        rc = set_err("cudaMemsetAsync(arrive) failed");
    if (!rc)
        rc = launch_factor(d, d->n_top, (const int *) d->top_tasks.p, (const int *) d->top_nwait.p, 0);
    d->timing = timing;
    if (!rc && timing) {
        CK(cudaEventRecord(d->ev[3], d->stream));
        d->ev_set[1] = 1;
    }
    return rc;
}

ASAM_EXPORT int asam_factor(asam_dev_t *d, int ntasks, const int32_t *tasks, const int32_t *nwait, const int32_t *keep)
{
    if (ntasks <= 0)
        return 0;
    CK(cudaSetDevice(d->device));
    size_t b = (size_t) ntasks * sizeof(int);
    if (buf_reserve(d, d->tasks_tmp, b, false, false) || buf_reserve(d, d->nwait_tmp, b, false, false) ||
        buf_reserve(d, d->keep_tmp, b, false, false))
        return 1;
    if (upload(d, d->tasks_tmp.p, tasks, b) || upload(d, d->nwait_tmp.p, nwait, b))
        return 1;
    int any = 0;
    for (int t = 0; keep && t < ntasks; t++)
        any |= keep[t];
    if (any && !d->keep_off && upload(d, d->keep_tmp.p, keep, b))
        return 1;
    return launch_factor(d, ntasks, (const int *) d->tasks_tmp.p, (const int *) d->nwait_tmp.p, 0,
                         any && !d->keep_off ? (const int *) d->keep_tmp.p : nullptr);
}

ASAM_EXPORT int asam_backsolve_full(asam_dev_t *d)
{
    CK(cudaSetDevice(d->device));
    int rc = launch_backsolve(d, d->bt_count, (const int *) d->btasks_full.p + d->bt_start, d->bt_nleaf);
    if (!rc && d->sharded) {
        if (d->defer)
            return set_err("sharded asam_backsolve_full inside asam_step_begin/asam_step_run");
        rc = shard_exchange(d, 1); // every rank ends up with the whole solution
        if (!rc)
            rc = shard_status_agree(d);
    }
    return rc;
}

ASAM_EXPORT int asam_backsolve(asam_dev_t *d, int ntasks, const int32_t *btasks, const int32_t *bfirst)
{
    if (ntasks <= 0)
        return 0;
    CK(cudaSetDevice(d->device));
    size_t b = (size_t) ntasks * sizeof(int);
    if (buf_reserve(d, d->btasks_tmp, 2 * b, false, false))
        return 1;
    if (upload(d, d->btasks_tmp.p, btasks, b))
        return 1;
    // (bfirst holds with ASAM_KEEP=0 too: a front re-factored whole has the same L and y in the wanted columns)
    const bool part = bfirst != nullptr;
    if (part && upload(d, (int *) d->btasks_tmp.p + ntasks, bfirst, b))
        return 1;
    return launch_backsolve(d, ntasks, (const int *) d->btasks_tmp.p, 0, part ? (const int *) d->btasks_tmp.p + ntasks : nullptr);
}

ASAM_EXPORT int asam_download_x(asam_dev_t *d, int q_first, int q_count, double *x3)
{
    CK(cudaSetDevice(d->device));
    return download(d, x3, (const double *) d->x.p + 3 * (size_t) q_first, (size_t) q_count * 3 * sizeof(double));
}

ASAM_EXPORT int asam_download_y(asam_dev_t *d, int q_first, int q_count, double *y3)
{
    CK(cudaSetDevice(d->device));
    return download(d, y3, (const double *) d->y.p + 3 * (size_t) q_first, (size_t) q_count * 3 * sizeof(double));
}

ASAM_EXPORT int asam_chi2(asam_dev_t *d, int n_factors, double *chi2_out)
{
    *chi2_out = 0.0;
    if (n_factors <= 0)
        return 0;
    CK(cudaSetDevice(d->device));
    int nblk = (n_factors + 255) / 256;
    if (buf_reserve(d, d->partial, ((size_t) nblk + 1) * sizeof(double), false, false))
        return 1;
    double *partial = (double *) d->partial.p;
    if (flush_uploads(d))
        return 1;
    k_chi2_partial<<<nblk, 256, 0, d->stream>>>((const int *) d->f_type.p, (const int *) d->f_a.p,
                                                 (const int *) d->f_b.p, (const double *) d->f_z.p,
                                                 (const double *) d->f_W.p, (const double2 *) d->f_loss.p,
                                                 (const double *) d->st.p, n_factors, partial + 1);
    k_chi2_final<<<1, 256, 0, d->stream>>>(partial + 1, nblk, partial);
    d->n_launch += 2;
    CK(cudaGetLastError());
    return download(d, chi2_out, partial, sizeof(double));
}

static size_t align256(size_t v) { return (v + 255) & ~(size_t) 255; }

// Byte offsets in the query scratch: [err | out (3n x 3n)] [paths] [z] [hops]; err and out come back with one copy.
// o = {out, paths, z, hops, total}.
static void marg_layout(int n, int64_t z_doubles, int n_hops, size_t o[5])
{
    o[0] = 16;
    o[1] = align256(o[0] + 9 * (size_t) n * n * sizeof(double));
    o[2] = o[1] + align256((size_t) n * sizeof(asam_marg_path_t));
    o[3] = o[2] + align256((size_t) z_doubles * sizeof(double));
    o[4] = o[3] + align256(4 * (size_t) n_hops * sizeof(int));
}

ASAM_EXPORT void asam_debug_marginal_layout(int n, int64_t z_doubles, int n_hops, int64_t out5[5])
{
    size_t o[5];
    marg_layout(n, z_doubles, n_hops, o);
    for (int k = 0; k < 5; k++)
        out5[k] = (int64_t) o[k];
}

// Byte offsets in the scratch of a candidate query: [err | out (10 doubles per candidate)] [paths] [z] [hops] [pairs].
// o = {out, paths, z, hops, pairs, total}.
static void marg_pairs_layout(int n, int64_t z_doubles, int n_hops, int k, size_t o[6])
{
    o[0] = 16;
    o[1] = align256(o[0] + 10 * (size_t) k * sizeof(double));
    o[2] = o[1] + align256((size_t) n * sizeof(asam_marg_path_t));
    o[3] = o[2] + align256((size_t) z_doubles * sizeof(double));
    o[4] = o[3] + align256(4 * (size_t) n_hops * sizeof(int));
    o[5] = o[4] + align256((size_t) k * sizeof(asam_marg_pair_t));
}

ASAM_EXPORT void asam_debug_marginal_pairs_layout(int n, int64_t z_doubles, int n_hops, int k, int64_t out6[6])
{
    size_t o[6];
    marg_pairs_layout(n, z_doubles, n_hops, k, o);
    for (int q = 0; q < 6; q++)
        out6[q] = (int64_t) o[q];
}

// The dynamic shared memory limit of k_marginal_path is a property of the function on a device, shared by every
// context (one per graph) in the process.  It only grows, so a launch sized at or below any value set before stays
// valid while other threads query graphs with smaller fronts.
static std::mutex g_marg_smem_mu;
static std::vector<int> g_marg_smem; // per device: bytes k_marginal_path is set up for

static int marg_smem_reserve(int device, size_t smem, int max_m, const char *fn)
{
    std::lock_guard<std::mutex> lock(g_marg_smem_mu);
    if ((size_t) device >= g_marg_smem.size())
        g_marg_smem.resize((size_t) device + 1, 0);
    if (smem <= (size_t) g_marg_smem[device])
        return 0;
    int optin = 0;
    CK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
    if (smem > (size_t) optin)
        return set_err("%s: fronts of order %d need %zu KB of shared memory, the device offers %d KB", fn, max_m,
                       smem / 1024, optin / 1024);
    CK(cudaFuncSetAttribute(k_marginal_path, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
    g_marg_smem[device] = (int) smem;
    return 0;
}

ASAM_EXPORT int asam_marginal_cov(asam_dev_t *d, int n, const asam_marg_path_t *paths, int64_t z_doubles, int n_hops,
                                  int max_m, double *out)
{
    if (n < 1 || n > 65535 || !paths || !out || z_doubles < 3 || n_hops < n || max_m < 3)
        return set_err("asam_marginal_cov: invalid arguments (n %d, z %lld, hops %d, max_m %d)", n, (long long) z_doubles,
                       n_hops, max_m);
    CK(cudaSetDevice(d->device));
    const size_t smem = ASAM_MSMEM(max_m) * sizeof(double);
    if (marg_smem_reserve(d->device, smem, max_m, "asam_marginal_cov"))
        return 1;
    size_t lay[5];
    marg_layout(n, z_doubles, n_hops, lay);
    const size_t out_bytes = lay[0] + 9 * (size_t) n * n * sizeof(double);
    const size_t o_paths = lay[1], o_z = lay[2], o_hop = lay[3], total = lay[4];
    if (buf_reserve(d, d->marg, total, false, false))
        return 1;
    char *base = (char *) d->marg.p;
    if (flush_uploads(d))
        return 1;
    CK(cudaMemcpyAsync(base + o_paths, paths, (size_t) n * sizeof(asam_marg_path_t), cudaMemcpyHostToDevice, d->stream));
    CK(cudaMemsetAsync(base, 0, 16, d->stream));
    d->n_h2d += (int64_t) n * (int64_t) sizeof(asam_marg_path_t);
    MargArgs a;
    a.sn = (const asam_sn_desc_t *) d->sn.p;
    a.ipool = (const int *) d->ipool.p;
    a.arena = (const double *) d->arena.p;
    a.dinv = (const double *) d->dinv.p;
    a.paths = (const asam_marg_path_t *) (base + o_paths);
    a.pairs = nullptr;
    a.z = (double *) (base + o_z);
    a.hop = (int *) (base + o_hop);
    a.out = (double *) (base + 16);
    a.err = (int *) base;
    a.n = n;
    a.max_m = max_m;
    k_marginal_path<<<n, 256, smem, d->stream>>>(a);
    CK(cudaGetLastError());
    k_marginal_gram<<<dim3(n, n), 128, 0, d->stream>>>(a);
    CK(cudaGetLastError());
    d->n_launch += 2;
    std::vector<double> host(out_bytes / sizeof(double));
    if (download(d, host.data(), base, out_bytes))
        return 1;
    int err = 0;
    memcpy(&err, host.data(), sizeof(int));
    if (err)
        return set_err("asam_marginal_cov: %s", err == 1 ? "a front on a path is larger than max_m"
                                                          : "a path's length differs from the plan's");
    memcpy(out, host.data() + 2, 9 * (size_t) n * n * sizeof(double));
    return 0;
}

ASAM_EXPORT int asam_marginal_pairs(asam_dev_t *d, int n, const asam_marg_path_t *paths, int64_t z_doubles,
                                    int n_hops, int max_m, int k, const asam_marg_pair_t *pairs, double *out)
{
    if (n < 1 || !paths || z_doubles < 3 || n_hops < n || max_m < 3 || k < 1 || !pairs || !out)
        return set_err("asam_marginal_pairs: invalid arguments (n %d, z %lld, hops %d, max_m %d, k %d)", n,
                       (long long) z_doubles, n_hops, max_m, k);
    CK(cudaSetDevice(d->device));
    const size_t smem = ASAM_MSMEM(max_m) * sizeof(double);
    if (marg_smem_reserve(d->device, smem, max_m, "asam_marginal_pairs"))
        return 1;
    size_t lay[6];
    marg_pairs_layout(n, z_doubles, n_hops, k, lay);
    const size_t out_bytes = lay[0] + 10 * (size_t) k * sizeof(double);
    if (buf_reserve(d, d->marg, lay[5], false, false))
        return 1;
    char *base = (char *) d->marg.p;
    if (flush_uploads(d))
        return 1;
    CK(cudaMemcpyAsync(base + lay[1], paths, (size_t) n * sizeof(asam_marg_path_t), cudaMemcpyHostToDevice, d->stream));
    CK(cudaMemcpyAsync(base + lay[4], pairs, (size_t) k * sizeof(asam_marg_pair_t), cudaMemcpyHostToDevice, d->stream));
    CK(cudaMemsetAsync(base, 0, 16, d->stream));
    d->n_h2d += (int64_t) n * (int64_t) sizeof(asam_marg_path_t) + (int64_t) k * (int64_t) sizeof(asam_marg_pair_t);
    MargArgs a;
    a.sn = (const asam_sn_desc_t *) d->sn.p;
    a.ipool = (const int *) d->ipool.p;
    a.arena = (const double *) d->arena.p;
    a.dinv = (const double *) d->dinv.p;
    a.paths = (const asam_marg_path_t *) (base + lay[1]);
    a.pairs = (const asam_marg_pair_t *) (base + lay[4]);
    a.z = (double *) (base + lay[2]);
    a.hop = (int *) (base + lay[3]);
    a.out = (double *) (base + 16);
    a.err = (int *) base;
    a.n = n;
    a.max_m = max_m;
    k_marginal_path<<<n, 256, smem, d->stream>>>(a);
    CK(cudaGetLastError());
    k_marginal_pairs<<<k, 128, 0, d->stream>>>(a);
    CK(cudaGetLastError());
    d->n_launch += 2;
    std::vector<double> host(out_bytes / sizeof(double));
    if (download(d, host.data(), base, out_bytes))
        return 1;
    int err = 0;
    memcpy(&err, host.data(), sizeof(int));
    if (err)
        return set_err("asam_marginal_pairs: %s", err == 1 ? "a front on a path is larger than max_m"
                                                            : "a path's length differs from the plan's");
    memcpy(out, host.data() + 2, 10 * (size_t) k * sizeof(double));
    return 0;
}

// A non-zero status is fatal for the solve in flight; the control words (tickets, team barriers,
// arrival counters) may be mid-way, so put all of them back to their idle state.
static int clear_status(asam_dev *d)
{
    CK(cudaMemsetAsync(d->ctrl.p, 0, 8 * sizeof(int), d->stream));
    if (d->tbar.p)
        CK(cudaMemsetAsync(d->tbar.p, 0, d->tbar.cap, d->stream));
    if (d->arrive.p)
        CK(cudaMemsetAsync(d->arrive.p, 0, d->arrive.cap, d->stream));
    return 0;
}

ASAM_EXPORT int asam_factor_status(asam_dev_t *d, int *status_out)
{
    CK(cudaSetDevice(d->device));
    int ctrl[2] = { 0, 0 };
    if (download(d, ctrl, d->ctrl.p, 2 * sizeof(int)))
        return 1;
    *status_out = ctrl[1];
    if (ctrl[1] != 0)
        return clear_status(d);
    return 0;
}

ASAM_EXPORT int asam_debug_read_hessian(asam_dev_t *d, int n_nodes, int n_slots, double *Adiag9, double *Aoff9,
                                        double *Bq3)
{
    CK(cudaSetDevice(d->device));
    int rc = 0;
    if (Adiag9)
        rc |= download(d, Adiag9, d->Adiag.p, (size_t) n_nodes * 9 * sizeof(double));
    if (Aoff9)
        rc |= download(d, Aoff9, d->Aoff.p, (size_t) n_slots * 9 * sizeof(double));
    if (Bq3)
        rc |= download(d, Bq3, d->Bq.p, (size_t) n_nodes * 3 * sizeof(double));
    return rc;
}

ASAM_EXPORT int asam_debug_read_front(asam_dev_t *d, int64_t f_off, int64_t count, double *out)
{
    CK(cudaSetDevice(d->device));
    return download(d, out, (const double *) d->arena.p + f_off, (size_t) count * sizeof(double));
}

ASAM_EXPORT int asam_debug_read_buffer(asam_dev_t *d, int id, int64_t off, int64_t bytes, void *out)
{
    CK(cudaSetDevice(d->device));
    Buf *b = nullptr;
    switch (id) {
    case ASAM_DBG_BUF_SN: b = &d->sn; break;
    case ASAM_DBG_BUF_IPOOL: b = &d->ipool; break;
    case ASAM_DBG_BUF_NODE2Q: b = &d->node2q; break;
    case ASAM_DBG_BUF_Q2NODE: b = &d->q2node; break;
    case ASAM_DBG_BUF_FSLOT: b = &d->f_slot; break;
    case ASAM_DBG_BUF_FTYPE: b = &d->f_type; break;
    case ASAM_DBG_BUF_FA: b = &d->f_a; break;
    case ASAM_DBG_BUF_FB: b = &d->f_b; break;
    case ASAM_DBG_BUF_FZ: b = &d->f_z; break;
    case ASAM_DBG_BUF_FW: b = &d->f_W; break;
    case ASAM_DBG_BUF_FLOSS: b = &d->f_loss; break;
    case ASAM_DBG_BUF_DINV: b = &d->dinv; break;
    case ASAM_DBG_BUF_MARG: b = &d->marg; break;
    default: return set_err("asam_debug_read_buffer: unknown buffer id %d", id);
    }
    if (off < 0 || bytes < 0 || (size_t) (off + bytes) > b->cap)
        return set_err("asam_debug_read_buffer: [%lld, %lld) outside buffer %d of %zu bytes", (long long) off,
                       (long long) (off + bytes), id, b->cap);
    return download(d, out, (const char *) b->p + off, (size_t) bytes);
}

ASAM_EXPORT int asam_sync(asam_dev_t *d)
{
    CK(cudaSetDevice(d->device));
    if (flush_uploads(d))
        return 1;
    CK(cudaStreamSynchronize(d->stream));
    return 0;
}

// x[q_first .. q_first+q_count) and the factorisation status with ONE synchronisation.
ASAM_EXPORT int asam_download_x_status(asam_dev_t *d, int q_first, int q_count, double *x3, int *status_out)
{
    CK(cudaSetDevice(d->device));
    if (flush_uploads(d))
        return 1;
    const size_t xb = (size_t) q_count * 3 * sizeof(double);
    if (xb + 16 > d->pin_down_cap) {
        if (download(d, x3, (const double *) d->x.p + 3 * (size_t) q_first, xb))
            return 1;
        return asam_factor_status(d, status_out);
    }
    d->n_d2h += (int64_t) xb + 8;
    CK(cudaMemcpyAsync(d->pin_down, d->ctrl.p, 2 * sizeof(int), cudaMemcpyDeviceToHost, d->stream));
    if (xb)
        CK(cudaMemcpyAsync(d->pin_down + 16, (const double *) d->x.p + 3 * (size_t) q_first, xb, cudaMemcpyDeviceToHost,
                           d->stream));
    CK(cudaStreamSynchronize(d->stream));
    *status_out = ((const int *) d->pin_down)[1];
    memcpy(x3, d->pin_down + 16, xb);
    if (*status_out != 0)
        return clear_status(d);
    return 0;
}

ASAM_EXPORT int64_t asam_small_steps(asam_dev_t *d) { return d->n_small; }

// Accumulated microseconds of the fused small steps so far: [0] upload fetch + scatter, [1] linearize,
// [2] factor, [3] back-solve, [4] result write-back (device globaltimer), [5] host launch call, [6] host
// wait on the completion flag; reset = 1 zeroes the accumulators (diagnostics: tools/step_profile.py).
ASAM_EXPORT void asam_small_step_profile(asam_dev_t *d, double *out7, int reset)
{
    memcpy(out7, d->small_us, 7 * sizeof(double));
    if (reset)
        memset(d->small_us, 0, sizeof(d->small_us));
}

ASAM_EXPORT int asam_counters(asam_dev_t *d, int64_t *out3)
{
    out3[0] = d->n_launch;
    out3[1] = d->n_h2d;
    out3[2] = d->n_d2h;
    return 0;
}

// Generic device-side stopwatch on the library's stream (bench.py): asam_timer_start /
// asam_timer_stop bracket any sequence of asam_* calls; _stop synchronises and returns ms.
ASAM_EXPORT int asam_timer_start(asam_dev_t *d)
{
    CK(cudaSetDevice(d->device));
    if (flush_uploads(d))
        return 1;
    if (!d->tev[0]) {
        CK(cudaEventCreate(&d->tev[0]));
        CK(cudaEventCreate(&d->tev[1]));
    }
    CK(cudaEventRecord(d->tev[0], d->stream));
    return 0;
}

ASAM_EXPORT int asam_timer_stop(asam_dev_t *d, float *ms)
{
    CK(cudaSetDevice(d->device));
    CK(cudaEventRecord(d->tev[1], d->stream));
    CK(cudaEventSynchronize(d->tev[1]));
    CK(cudaEventElapsedTime(ms, d->tev[0], d->tev[1]));
    return 0;
}

// Evict the working set from L2 between timed iterations: overwrite a buffer larger than L2 (H100: 50 MB).
ASAM_EXPORT int asam_l2_flush(asam_dev_t *d)
{
    CK(cudaSetDevice(d->device));
    const size_t bytes = (size_t) 128 << 20;
    if (buf_reserve(d, d->flush, bytes, false, false) || flush_uploads(d))
        return 1;
    d->flush_val ^= 0x5a;
    CK(cudaMemsetAsync(d->flush.p, d->flush_val, bytes, d->stream));
    return 0;
}

// FP64 peak of this device, measured: a register-resident DFMA loop (8 independent chains per thread,
// 512 threads per SM) timed with CUDA events on the library's stream.  MEASURED_PEAKS.json carries HBM
// and bf16 figures only; the factorisation's second roofline (SURVEY.md section 8d) is the FP64 pipe.
__global__ void k_fp64_peak(double *out, int iters)
{
    double a[8], b = 1.000001, c = 0.5;
#pragma unroll
    for (int i = 0; i < 8; i++)
        a[i] = threadIdx.x + i;
    for (int it = 0; it < iters; it++)
#pragma unroll
        for (int i = 0; i < 8; i++)
            a[i] = fma(a[i], b, c);
    double s = 0;
#pragma unroll
    for (int i = 0; i < 8; i++)
        s += a[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

ASAM_EXPORT int asam_measure_fp64_peak(asam_dev_t *d, double *tflops_out)
{
    CK(cudaSetDevice(d->device));
    *tflops_out = 0.0;
    const int threads = 512, iters = 20000;
    if (buf_reserve(d, d->partial, (size_t) d->n_sm * threads * sizeof(double), false, false) || flush_uploads(d))
        return 1;
    if (!d->tev[0]) {
        CK(cudaEventCreate(&d->tev[0]));
        CK(cudaEventCreate(&d->tev[1]));
    }
    double best = 0.0;
    for (int rep = 0; rep < 4; rep++) { // first repetition = warm-up
        CK(cudaEventRecord(d->tev[0], d->stream));
        k_fp64_peak<<<d->n_sm, threads, 0, d->stream>>>((double *) d->partial.p, iters);
        CK(cudaGetLastError());
        CK(cudaEventRecord(d->tev[1], d->stream));
        CK(cudaEventSynchronize(d->tev[1]));
        float ms = 0.f;
        CK(cudaEventElapsedTime(&ms, d->tev[0], d->tev[1]));
        const double tf = 2.0 * 8 * iters * (double) threads * d->n_sm / (ms * 1e-3) * 1e-12;
        if (rep > 0 && tf > best)
            best = tf;
    }
    *tflops_out = best;
    return 0;
}

ASAM_EXPORT int asam_device_info(asam_dev_t *d, int *n_sm, int *fac_grid, int *fac_smem, int *bs_grid)
{
    *n_sm = d->n_sm;
    *fac_grid = d->fac_grid;
    *fac_smem = d->fac_smem;
    *bs_grid = d->bs_grid;
    return 0;
}

// Per-task timestamps (globaltimer ns) of the last k_factor (which=0) / k_backsolve (which=1)
// launch: 8 words per task (see asam_kernels.cuh).  Diagnostics only.
ASAM_EXPORT int asam_set_trace(asam_dev_t *d, int enabled)
{
    d->trace_on = enabled;
    return 0;
}

ASAM_EXPORT int asam_download_trace(asam_dev_t *d, int which, unsigned long long *out, int max_tasks)
{
    CK(cudaSetDevice(d->device));
    if (flush_uploads(d))
        return 1;
    int n = which == 0 ? d->trace_nfac : d->trace_nbs;
    Buf &b = which == 0 ? d->trace_fac : d->trace_bs;
    if (n > max_tasks)
        n = max_tasks;
    if (n <= 0 || !b.p)
        return 0;
    CK(cudaMemcpyAsync(out, b.p, (size_t) n * 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, d->stream));
    CK(cudaStreamSynchronize(d->stream));
    return 0;
}

// Panel-step stamps of team front `sn` (-1: off): 8 x uint64 per (panel, worker < 8); see team_front.
ASAM_EXPORT int asam_set_panel_trace(asam_dev_t *d, int sn, int max_panels)
{
    CK(cudaSetDevice(d->device));
    d->ptrace_sn = -1;
    if (sn < 0 || max_panels <= 0)
        return 0;
    const size_t bytes = (size_t) max_panels * 64 * sizeof(unsigned long long);
    if (buf_reserve(d, d->ptrace, bytes, false, false) || flush_uploads(d))
        return 1;
    CK(cudaMemsetAsync(d->ptrace.p, 0, bytes, d->stream));
    d->ptrace_sn = sn;
    d->ptrace_panels = max_panels;
    return 0;
}

ASAM_EXPORT int asam_download_panel_trace(asam_dev_t *d, unsigned long long *out, int max_panels)
{
    CK(cudaSetDevice(d->device));
    if (!d->ptrace.p || max_panels > d->ptrace_panels)
        return set_err("asam_download_panel_trace: no trace");
    if (flush_uploads(d))
        return 1;
    CK(cudaMemcpyAsync(out, d->ptrace.p, (size_t) max_panels * 64 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, d->stream));
    CK(cudaStreamSynchronize(d->stream));
    return 0;
}

ASAM_EXPORT int asam_set_timing(asam_dev_t *d, int enabled)
{
    d->timing = enabled;
    d->ev_set[0] = d->ev_set[1] = d->ev_set[2] = 0;
    return 0;
}

ASAM_EXPORT int asam_last_kernel_ms(asam_dev_t *d, float *lin_ms, float *fac_ms, float *bs_ms)
{
    CK(cudaSetDevice(d->device));
    if (flush_uploads(d))
        return 1;
    CK(cudaStreamSynchronize(d->stream));
    float *outs[3] = { lin_ms, fac_ms, bs_ms };
    for (int i = 0; i < 3; i++) {
        float ms = 0.f;
        if (d->ev_set[i])
            CK(cudaEventElapsedTime(&ms, d->ev[2 * i], d->ev[2 * i + 1]));
        if (outs[i])
            *outs[i] = ms;
    }
    return 0;
}
