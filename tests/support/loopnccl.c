/* loopnccl.c -- a loopback stand-in for NCCL, for tests only.
 *
 * The solver reaches NCCL through dlopen("libnccl.so.2") and eight symbols.  Built as a shared library with the
 * SONAME libnccl.so.2 and loaded (RTLD_GLOBAL) before the solver's library, this file takes NCCL's place, so that
 * the ranks of a sharded solve can be processes on ONE GPU (NCCL itself refuses two ranks on one device).
 *
 *   - unique id: the 128 bytes hold the path of a rendezvous file (NUL-terminated); the test writes it;
 *   - transport: that file, mapped with mmap: a header (barrier, join count) and a fixed data window
 *     (LOOPNCCL_WINDOW bytes, default 16 MiB); larger operations go through it in chunks;
 *   - eager operations: each one runs when it is called and a group is a no-op (every rank issues the same
 *     operations in the same order).  No GPU-side wait crosses processes: every dependency between ranks is a
 *     host barrier here;
 *   - device memory through the CUDA driver API (dlopen("libcuda.so.1")): copies run on the stream passed in,
 *     and that stream is synchronised before a call returns (the solver's stream is non-blocking, so a copy on
 *     the legacy stream would not be ordered before its next kernel).  LOOPNCCL_HOST=1 treats every pointer as
 *     host memory (tests of the stand-in itself, no GPU);
 *   - every barrier wait ends after LOOPNCCL_TIMEOUT seconds (default 60) with an error code, so a missing peer
 *     becomes a failed call, not a stuck process;
 *   - loopnccl_stats: broadcasts, bytes broadcast, all-reduces and elements all-reduced since the communicator
 *     was created (the tests prove with them that the exchange ran).
 *
 * Build: gcc -shared -fPIC -O2 -Wl,-soname,libnccl.so.2 -o libnccl.so.2 loopnccl.c -ldl
 */
#define _GNU_SOURCE
#include <dlfcn.h>
#include <errno.h>
#include <fcntl.h>
#include <sched.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <time.h>
#include <unistd.h>

/* NCCL's result, data type and reduction codes (nccl.h) */
enum { ncclSuccess = 0, ncclUnhandledCudaError = 1, ncclSystemError = 2, ncclInternalError = 3,
       ncclInvalidArgument = 4, ncclInvalidUsage = 5, ncclRemoteError = 6 };
enum { ncclInt8 = 0, ncclUint8 = 1, ncclInt32 = 2, ncclUint32 = 3, ncclInt64 = 4, ncclUint64 = 5, ncclFloat16 = 6,
       ncclFloat32 = 7, ncclFloat64 = 8 };
enum { ncclSum = 0, ncclProd = 1, ncclMax = 2, ncclMin = 3 };

typedef struct { char internal[128]; } ncclUniqueId;
typedef void *cudaStream_t;

#define HDR_BYTES 4096
typedef struct {
    int world;      /* set by the first rank to join */
    int joined;     /* ranks that have mapped the file */
    int count;      /* barrier: arrivals of the current generation */
    int gen;        /* barrier: generation */
    int64_t window; /* bytes of the data window */
} hdr_t;

typedef struct loop_comm {
    int world, rank, host;
    hdr_t *h;
    char *win;
    size_t map_bytes;
    int64_t window;
    double timeout_s;
} loop_comm_t;

static loop_comm_t *g_comm; /* the communicator of this process (loopnccl_sync) */
static long long g_stats[4];
static const char *g_last = "";

/* ---- CUDA driver API ------------------------------------------------------------------------------------------ */
typedef int (*cu_sync_t)(cudaStream_t);
typedef int (*cu_dtoh_t)(void *, unsigned long long, size_t, cudaStream_t);
typedef int (*cu_htod_t)(unsigned long long, const void *, size_t, cudaStream_t);
static cu_sync_t cu_sync;
static cu_dtoh_t cu_dtoh;
static cu_htod_t cu_htod;

static int cuda_load(void)
{
    if (cu_sync)
        return 0;
    void *h = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
    if (!h)
        return -1;
    cu_sync = (cu_sync_t) dlsym(h, "cuStreamSynchronize");
    cu_dtoh = (cu_dtoh_t) dlsym(h, "cuMemcpyDtoHAsync_v2");
    cu_htod = (cu_htod_t) dlsym(h, "cuMemcpyHtoDAsync_v2");
    return cu_sync && cu_dtoh && cu_htod ? 0 : -1;
}

/* device (or, in host mode, host) memory -> host */
static int to_host(loop_comm_t *c, void *dst, const void *src, size_t n, cudaStream_t s)
{
    if (c->host) {
        memcpy(dst, src, n);
        return 0;
    }
    if (cu_sync(s) || cu_dtoh(dst, (unsigned long long) (uintptr_t) src, n, s) || cu_sync(s)) {
        g_last = "loopnccl: device to host copy failed";
        return ncclUnhandledCudaError;
    }
    return 0;
}

static int from_host(loop_comm_t *c, void *dst, const void *src, size_t n, cudaStream_t s)
{
    if (c->host) {
        memcpy(dst, src, n);
        return 0;
    }
    if (cu_htod((unsigned long long) (uintptr_t) dst, src, n, s) || cu_sync(s)) {
        g_last = "loopnccl: host to device copy failed";
        return ncclUnhandledCudaError;
    }
    return 0;
}

/* ---- barrier -------------------------------------------------------------------------------------------------- */
static double now_s(void)
{
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (double) ts.tv_sec + 1e-9 * (double) ts.tv_nsec;
}

static int barrier(loop_comm_t *c, double timeout_s)
{
    hdr_t *h = c->h;
    const int gen = __atomic_load_n(&h->gen, __ATOMIC_ACQUIRE);
    if (__atomic_add_fetch(&h->count, 1, __ATOMIC_ACQ_REL) == c->world) {
        __atomic_store_n(&h->count, 0, __ATOMIC_RELAXED);
        __atomic_store_n(&h->gen, gen + 1, __ATOMIC_RELEASE);
        return 0;
    }
    const double end = now_s() + timeout_s;
    for (int spin = 0; __atomic_load_n(&h->gen, __ATOMIC_ACQUIRE) == gen; spin++) {
        if (spin < 1000) {
            sched_yield();
            continue;
        }
        if (now_s() > end) {
            g_last = "loopnccl: timed out waiting for a peer";
            return ncclRemoteError;
        }
        usleep(50);
    }
    return 0;
}

/* ---- NCCL entry points ---------------------------------------------------------------------------------------- */
const char *ncclGetErrorString(int r)
{
    switch (r) {
    case ncclSuccess: return "no error";
    case ncclInvalidArgument: return "invalid argument (loopnccl)";
    case ncclInvalidUsage: return "invalid usage (loopnccl)";
    default: return g_last[0] ? g_last : "loopnccl error";
    }
}

int ncclGetUniqueId(ncclUniqueId *id)
{
    const char *tmp = getenv("TMPDIR");
    memset(id, 0, sizeof(*id));
    snprintf(id->internal, sizeof(id->internal), "%s/loopnccl-%d-%ld", tmp ? tmp : "/tmp", (int) getpid(),
             (long) time(NULL));
    return ncclSuccess;
}

int ncclCommInitRank(loop_comm_t **out, int nranks, ncclUniqueId id, int rank)
{
    *out = NULL;
    if (nranks < 1 || rank < 0 || rank >= nranks)
        return ncclInvalidArgument;
    char path[129];
    memcpy(path, id.internal, 128);
    path[128] = 0;
    if (!path[0])
        return ncclInvalidArgument;
    const char *e = getenv("LOOPNCCL_HOST");
    const int host = e && atoi(e) != 0;
    if (!host && cuda_load()) {
        g_last = "loopnccl: cannot load libcuda.so.1";
        return ncclSystemError;
    }
    e = getenv("LOOPNCCL_WINDOW");
    int64_t window = e ? atoll(e) : (int64_t) 16 << 20;
    window = window < 64 ? 64 : (window & ~(int64_t) 7);
    e = getenv("LOOPNCCL_TIMEOUT");
    const double timeout_s = e ? atof(e) : 60.0;

    const size_t bytes = HDR_BYTES + (size_t) window;
    int fd = open(path, O_RDWR | O_CREAT, 0600);
    if (fd < 0) {
        g_last = "loopnccl: cannot open the rendezvous file";
        return ncclSystemError;
    }
    struct stat st;
    if (fstat(fd, &st) || ((size_t) st.st_size < bytes && ftruncate(fd, (off_t) bytes))) {
        close(fd);
        g_last = "loopnccl: cannot size the rendezvous file";
        return ncclSystemError;
    }
    void *p = mmap(NULL, bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    close(fd);
    if (p == MAP_FAILED) {
        g_last = "loopnccl: mmap failed";
        return ncclSystemError;
    }
    loop_comm_t *c = calloc(1, sizeof(*c));
    c->world = nranks;
    c->rank = rank;
    c->host = host;
    c->h = (hdr_t *) p;
    c->win = (char *) p + HDR_BYTES;
    c->map_bytes = bytes;
    c->window = window;
    c->timeout_s = timeout_s;
    int w0 = 0;
    int64_t win0 = 0;
    __atomic_compare_exchange_n(&c->h->world, &w0, nranks, 0, __ATOMIC_ACQ_REL, __ATOMIC_ACQUIRE);
    __atomic_compare_exchange_n(&c->h->window, &win0, window, 0, __ATOMIC_ACQ_REL, __ATOMIC_ACQUIRE);
    if (__atomic_load_n(&c->h->world, __ATOMIC_ACQUIRE) != nranks ||
        __atomic_load_n(&c->h->window, __ATOMIC_ACQUIRE) != window) {
        munmap(p, bytes);
        free(c);
        return ncclInvalidUsage;
    }
    __atomic_add_fetch(&c->h->joined, 1, __ATOMIC_ACQ_REL);
    int r = barrier(c, timeout_s); /* every rank has joined */
    if (r) {
        munmap(p, bytes);
        free(c);
        return r;
    }
    memset(g_stats, 0, sizeof(g_stats));
    g_comm = c;
    *out = c;
    return ncclSuccess;
}

int ncclCommDestroy(loop_comm_t *c)
{
    if (!c)
        return ncclSuccess;
    munmap(c->h, c->map_bytes);
    if (g_comm == c)
        g_comm = NULL;
    free(c);
    return ncclSuccess;
}

int ncclGroupStart(void) { return ncclSuccess; }
int ncclGroupEnd(void) { return ncclSuccess; }

static size_t type_size(int t)
{
    switch (t) {
    case ncclInt8: case ncclUint8: return 1;
    case ncclFloat16: return 2;
    case ncclInt32: case ncclUint32: case ncclFloat32: return 4;
    case ncclInt64: case ncclUint64: case ncclFloat64: return 8;
    default: return 0;
    }
}

/* root: its buffer -> window; barrier; others: window -> their buffer; barrier.  In place or not. */
int ncclBroadcast(const void *send, void *recv, size_t count, int type, int root, loop_comm_t *c, cudaStream_t s)
{
    const size_t sz = type_size(type);
    if (!c || !sz || root < 0 || root >= c->world)
        return ncclInvalidArgument;
    const size_t bytes = count * sz;
    g_stats[0]++;
    g_stats[1] += (long long) bytes;
    for (size_t off = 0; off < bytes; off += (size_t) c->window) {
        const size_t n = bytes - off < (size_t) c->window ? bytes - off : (size_t) c->window;
        int r = 0;
        if (c->rank == root)
            r = to_host(c, c->win, (const char *) send + off, n, s);
        if (r || (r = barrier(c, c->timeout_s)))
            return r;
        if (c->rank != root || send != recv)
            r = from_host(c, (char *) recv + off, c->win, n, s);
        if (r || (r = barrier(c, c->timeout_s)))
            return r;
    }
    return ncclSuccess;
}

#define REDUCE(T)                                                                                      \
    do {                                                                                               \
        T *o = (T *) out;                                                                              \
        for (int q = 0; q < c->world; q++) {                                                           \
            const T *v = (const T *) (c->win + (size_t) q * n * sz);                                   \
            for (size_t i = 0; i < n; i++) {                                                           \
                if (q == 0)                                                                            \
                    o[i] = v[i];                                                                       \
                else if (op == ncclSum)                                                                \
                    o[i] = o[i] + v[i];                                                                \
                else if (op == ncclMax)                                                                \
                    o[i] = v[i] > o[i] ? v[i] : o[i];                                                  \
                else                                                                                   \
                    o[i] = v[i] < o[i] ? v[i] : o[i];                                                  \
            }                                                                                          \
        }                                                                                              \
    } while (0)

/* every rank's slice -> its slot of the window; barrier; each rank reduces the slots in rank order (the same bits
 * on every rank); barrier; result -> recv */
int ncclAllReduce(const void *send, void *recv, size_t count, int type, int op, loop_comm_t *c, cudaStream_t s)
{
    const size_t sz = type_size(type);
    if (!c || !(type == ncclInt32 || type == ncclInt64 || type == ncclFloat64) ||
        !(op == ncclSum || op == ncclMax || op == ncclMin))
        return ncclInvalidArgument;
    g_stats[2]++;
    g_stats[3] += (long long) count;
    const size_t per = (size_t) c->window / ((size_t) c->world * sz); /* elements per chunk */
    if (per == 0)
        return ncclInvalidUsage;
    void *out = malloc(per * sz);
    int r = 0;
    for (size_t e0 = 0; e0 < count && !r; e0 += per) {
        const size_t n = count - e0 < per ? count - e0 : per;
        r = to_host(c, c->win + (size_t) c->rank * n * sz, (const char *) send + e0 * sz, n * sz, s);
        if (r || (r = barrier(c, c->timeout_s)))
            break;
        if (type == ncclInt32)
            REDUCE(int32_t);
        else if (type == ncclInt64)
            REDUCE(int64_t);
        else
            REDUCE(double);
        if ((r = barrier(c, c->timeout_s)))
            break;
        r = from_host(c, (char *) recv + e0 * sz, out, n * sz, s);
    }
    free(out);
    return r;
}

/* ---- test-only exports ---------------------------------------------------------------------------------------- */
/* out[0] broadcasts, out[1] bytes broadcast, out[2] all-reduces, out[3] elements all-reduced */
int loopnccl_stats(long long *out4)
{
    memcpy(out4, g_stats, sizeof(g_stats));
    return 0;
}

/* a host barrier of every rank of this process's communicator with its own time limit (the ranks of a test
 * meet here between solves, while one of them may be busy checking) */
int loopnccl_sync(double timeout_s)
{
    return g_comm ? barrier(g_comm, timeout_s) : ncclInvalidUsage;
}
