/* plan.c -- host-side symbolic analysis and numeric plan for the GPU multifrontal solver.
 *
 * Replaces, with its own algorithms, the symbolic half of the reference's batch step:
 *   node adjacency                     aprilsam.c:104-114 (smatd Asym)
 *   ordering                           aprilsam.c:121       -> ordering.c
 *   cs_schol (etree, post, counts)     csparse.c:1693-1716  -> block elimination tree + block
 *                                                             row structures computed directly
 *   search_tree_create_from_smat       aprilsam.c:613-657   -> parent_pos[] (node-level tree)
 * and adds what a GPU supernodal method needs: post-ordering, fundamental supernodes, frontal
 * matrix layout, child->parent relative indices, Hessian gather lists, a level schedule.
 *
 * plan_append() is the symbolic side of april_graph_cholesky_inc (aprilsam.c:393-498,
 * :908-987): new poses are appended at the end of the elimination order and only the
 * supernodes on root paths of the touched nodes change (they gain the new poses as rows).
 */
#define _POSIX_C_SOURCE 200809L
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "asam_host.h"

/* diagnostics: time spent in the phases of plan_append (ms), read by tools/gpu_diag.py */
static double g_plan_prof[8];
static double g_build_prof[8]; /* phases of plan_build (ms): see BUILD_LAP */
static double pp_now(void)
{
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6;
}
void asam_dbg_plan_profile(double *out, int reset)
{
    memcpy(out, g_plan_prof, sizeof(g_plan_prof));
    if (reset)
        memset(g_plan_prof, 0, sizeof(g_plan_prof));
}
void asam_dbg_build_profile(double *out, int reset)
{
    memcpy(out, g_build_prof, sizeof(g_build_prof));
    if (reset)
        memset(g_build_prof, 0, sizeof(g_build_prof));
}

#define RELAX_Z 2     /* relaxed amalgamation: missing block rows tolerated per merge */
#define RELAX_FILL 24 /* ... and explicit zero blocks (3x3) added per merge */
#define TEAM_MERGE_PCT 20     /* team-sized fronts: extra rows tolerated per merge, % of the front (0: off; swept 10 .. 60) */
#define TEAM_MERGE_MFLOP 400.0 /* ... and extra flops per merge (millions) */
#define ASAM_TEAM_ROOM 64        /* CTAs that the team fronts of one tree level may claim together (H100, 100 k dense world: 64 beats 80, 100 and 132) */
#define ASAM_BSLEAF_MAX 64       /* = ASAM_BSL_XS of k_backsolve_leaf: own columns / rows below */
#define ASAM_BSLEAF_MIN_COUNT 4096 /* measured: no gain on M3500-sized trees (the kernel boundary eats it) */
#define ASAM_LEAF_MAX_M_DEFAULT 63 /* <= ASAM_LEAF_M of k_factor_leaf (ASAM_LEAF_MAX_M overrides downwards, tuning) */
#define ASAM_LEAF_MIN_COUNT 4096 /* below this one k_factor launch does it all */
#define ASAM_SOLO_MAX_M_DEFAULT 0 /* see solo_max_m() */
#define PLAN_OMP_MIN_SN 8192 /* below this many supernodes the symbolic loops stay on one thread */
#define PLAN_OMP_THREADS 8 /* ASAM_PLAN_THREADS overrides (1: serial) */
#define ASAM_SHARD_TOL_DEFAULT 1.10 /* multi-GPU cut: heaviest rank's load / mean at which the splitting stops */
#define ASAM_TILES_PER_WORKER 1   /* trailing-update tiles per worker and panel that team_size() plans for */
#define MAX_SN_COLS 32 /* block columns per supernode: L11 (96x96) fits k_backsolve shared memory */

/* ---- pair map ---------------------------------------------------------------------------- */
static inline uint64_t mix64(uint64_t x)
{
    x ^= x >> 33;
    x *= 0xff51afd7ed558ccdULL;
    x ^= x >> 33;
    x *= 0xc4ceb9fe1a85ec53ULL;
    x ^= x >> 33;
    return x;
}

void pairmap_init(pairmap_t *m, int expect)
{
    int cap = 64;
    while (cap < 2 * expect + 16)
        cap *= 2;
    m->cap = cap;
    m->n = 0;
    m->keys = malloc(sizeof(uint64_t) * cap);
    m->vals = malloc(sizeof(int) * cap);
    memset(m->keys, 0xff, sizeof(uint64_t) * cap);
}

void pairmap_free(pairmap_t *m)
{
    free(m->keys);
    free(m->vals);
    memset(m, 0, sizeof(*m));
}

static void pairmap_grow(pairmap_t *m)
{
    pairmap_t n;
    pairmap_init(&n, m->cap);
    for (int i = 0; i < m->cap; i++) {
        if (m->keys[i] == UINT64_MAX)
            continue;
        uint64_t h = mix64(m->keys[i]) & (uint64_t) (n.cap - 1);
        while (n.keys[h] != UINT64_MAX)
            h = (h + 1) & (uint64_t) (n.cap - 1);
        n.keys[h] = m->keys[i];
        n.vals[h] = m->vals[i];
    }
    n.n = m->n;
    free(m->keys);
    free(m->vals);
    *m = n;
}

int pairmap_get_or_add(pairmap_t *m, int lo, int hi, int next_slot, int *created)
{
    if (2 * (m->n + 1) > m->cap)
        pairmap_grow(m);
    uint64_t key = ((uint64_t) (uint32_t) lo << 32) | (uint32_t) hi;
    uint64_t h = mix64(key) & (uint64_t) (m->cap - 1);
    while (m->keys[h] != UINT64_MAX) {
        if (m->keys[h] == key) {
            *created = 0;
            return m->vals[h];
        }
        h = (h + 1) & (uint64_t) (m->cap - 1);
    }
    m->keys[h] = key;
    m->vals[h] = next_slot;
    m->n++;
    *created = 1;
    return next_slot;
}

/* ---- helpers ------------------------------------------------------------------------------ */
static int cmp_int(const void *a, const void *b)
{
    int x = *(const int *) a, y = *(const int *) b;
    return (x > y) - (x < y);
}

static void sort_ints(int *p, int n)
{
    if (n < 2)
        return;
    if (n <= 24) { /* insertion sort: most lists are tiny */
        for (int i = 1; i < n; i++) {
            int v = p[i], j = i - 1;
            while (j >= 0 && p[j] > v) {
                p[j + 1] = p[j];
                j--;
            }
            p[j + 1] = v;
        }
        return;
    }
    qsort(p, n, sizeof(int), cmp_int);
}

static int sort_unique(int *p, int n)
{
    sort_ints(p, n);
    int k = 0;
    for (int i = 0; i < n; i++)
        if (k == 0 || p[k - 1] != p[i])
            p[k++] = p[i];
    return k;
}

static int find_sorted(const int *p, int n, int v)
{
    int lo = 0, hi = n - 1;
    while (lo <= hi) {
        int mid = (lo + hi) >> 1;
        if (p[mid] == v)
            return mid;
        if (p[mid] < v)
            lo = mid + 1;
        else
            hi = mid - 1;
    }
    return -1;
}

static void sn_host_free(sn_host_t *h)
{
    ivec_free(&h->rows);
    ivec_free(&h->rel);
    ivec_free(&h->children);
    ivec_free(&h->a_slot);
    ivec_free(&h->a_rb);
    ivec_free(&h->a_cb);
}

void plan_free(plan_t *pl)
{
    free(pl->order);
    free(pl->pos);
    free(pl->node2q);
    free(pl->q2node);
    free(pl->parent_pos);
    if (pl->pairs.keys)
        pairmap_free(&pl->pairs);
    free(pl->fslot);
    for (int s = 0; s < pl->nsn; s++)
        sn_host_free(&pl->snh[s]);
    free(pl->desc);
    free(pl->snh);
    free(pl->sn_of_q);
    free(pl->tasks);
    free(pl->nwait);
    free(pl->btasks);
    free(pl->leaf_tasks);
    free(pl->bs_leaf);
    free(pl->mark_idx);
    free(pl->top_tasks);
    free(pl->top_nwait);
    free(pl->shard_owner);
    free(pl->shard_off);
    free(pl->shard_cnt);
    free(pl->shard_q0);
    free(pl->shard_qn);
    ivec_free(&pl->ipool_host);
    memset(pl, 0, sizeof(*pl));
}

static void node_arrays_reserve(plan_t *pl, int N)
{
    if (N <= pl->node_cap)
        return;
    int cap = pl->node_cap ? pl->node_cap : 64;
    while (cap < N)
        cap *= 2;
    pl->order = realloc(pl->order, sizeof(int) * cap);
    pl->pos = realloc(pl->pos, sizeof(int) * cap);
    pl->node2q = realloc(pl->node2q, sizeof(int) * cap);
    pl->q2node = realloc(pl->q2node, sizeof(int) * cap);
    pl->parent_pos = realloc(pl->parent_pos, sizeof(int) * cap);
    pl->sn_of_q = realloc(pl->sn_of_q, sizeof(int) * cap);
    pl->node_cap = cap;
}

static void sn_arrays_reserve(plan_t *pl, int n)
{
    if (n <= pl->sn_cap)
        return;
    int cap = pl->sn_cap ? pl->sn_cap : 64;
    while (cap < n)
        cap *= 2;
    pl->desc = realloc(pl->desc, sizeof(asam_sn_desc_t) * cap);
    pl->snh = realloc(pl->snh, sizeof(sn_host_t) * cap);
    memset(pl->snh + pl->sn_cap, 0, sizeof(sn_host_t) * (cap - pl->sn_cap));
    memset(pl->desc + pl->sn_cap, 0, sizeof(asam_sn_desc_t) * (cap - pl->sn_cap));
    if (pl->bs_leaf) { /* supernodes created later are never in the back-solve leaf set */
        pl->bs_leaf = realloc(pl->bs_leaf, (size_t) cap + 1);
        memset(pl->bs_leaf + pl->sn_cap, 0, (size_t) (cap - pl->sn_cap) + 1);
    }
    pl->sn_cap = cap;
}

static void fslot_reserve(plan_t *pl, int n)
{
    if (n <= pl->fslot_cap)
        return;
    int cap = pl->fslot_cap ? pl->fslot_cap : 64;
    while (cap < n)
        cap *= 2;
    pl->fslot = realloc(pl->fslot, sizeof(int) * cap);
    pl->fslot_cap = cap;
}

/* rel[k] for k >= cb: index of the child's row in the parent's row list */
/* Largest front of the warp-per-front kernel.  Big trees are bound by CTA-time (every front the leaf kernel takes frees an
 * SM for a team front), small ones by their dependent chain, where
 * a longer leaf launch ahead of k_factor only adds to it: the wider limit from
 * ASAM_LEAF_WIDE_MIN_SN supernodes on.  ASAM_LEAF_MAX_M overrides (tuning). */
#define ASAM_LEAF_WIDE_MIN_SN 30000
static int leaf_max_m_for(int nsn)
{
    const char *e = getenv("ASAM_LEAF_MAX_M");
    if (e && atoi(e) >= 3 && atoi(e) <= ASAM_LEAF_MAX_M_DEFAULT)
        return atoi(e);
    return nsn >= ASAM_LEAF_WIDE_MIN_SN ? ASAM_LEAF_MAX_M_DEFAULT : 48;
}

static double host_now_ms(void)
{
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6;
}

static double host_spin(int iters)
{
    volatile double x = 1.0;
    for (int i = 0; i < iters; i++)
        x = x * 1.0000001 + 1e-9;
    return x;
}

int asam_host_threads(void)
{
    static int v = 0;
    if (v == 0) {
        const char *e = getenv("ASAM_PLAN_THREADS");
        int want = e && atoi(e) > 0 ? atoi(e) : PLAN_OMP_THREADS;
        want = want > 16 ? 16 : want;
        if (want > 1) {
            /* two threads spinning for a fixed count each: side by side that takes as long as one of them */
            const int iters = 40000;
            double t0 = host_now_ms();
            host_spin(iters);
            const double t1 = host_now_ms() - t0;
            double tp = 1e30;
            for (int rep = 0; rep < 3 && tp > 2.5 * t1 + 0.05; rep++) { /* (the first region also creates the threads) */
                t0 = host_now_ms();
#pragma omp parallel num_threads(2)
                host_spin(iters);
                const double t = host_now_ms() - t0;
                tp = t < tp ? t : tp;
            }
            if (tp > 2.5 * t1 + 0.05)
                want = 1;
            if (getenv("ASAM_PLAN_VERBOSE"))
                fprintf(stderr, "plan: host threads %d (one thread %.3f ms, two side by side %.3f ms)\n", want, t1, tp);
        }
        v = want;
    }
    return v;
}

static int plan_threads(void) { return asam_host_threads(); }

static int compute_rel(plan_t *pl, int s)
{
    sn_host_t *h = &pl->snh[s];
    int cb = pl->desc[s].cb;
    ivec_reserve(&h->rel, h->rows.n);
    h->rel.n = h->rows.n;
    for (int k = 0; k < cb && k < h->rows.n; k++)
        h->rel.p[k] = -1;
    int P = pl->desc[s].parent;
    if (P < 0) {
        if (h->rows.n != cb) {
            asam_set_error("plan: supernode %d has rows below but no parent", s);
            return 1;
        }
        return 0;
    }
    const ivec_t *pr = &pl->snh[P].rows;
    int j = 0;
    for (int k = cb; k < h->rows.n; k++) {
        int v = h->rows.p[k];
        while (j < pr->n && pr->p[j] < v)
            j++;
        if (j >= pr->n || pr->p[j] != v) {
            asam_set_error("plan: row %d of supernode %d missing in parent %d", v, s, P);
            return 1;
        }
        h->rel.p[k] = j;
    }
    return 0;
}

/* Serialise the index segment of supernode s at the tail of `buf`; sets desc.seg. */
static void emit_segment(plan_t *pl, int s, ivec_t *buf, int64_t base)
{
    sn_host_t *h = &pl->snh[s];
    asam_sn_desc_t *d = &pl->desc[s];
    d->seg = (int32_t) (base + buf->n);
    d->mb = h->rows.n;
    d->ch_cnt = h->children.n;
    d->a_cnt = h->a_slot.n;
    int need = buf->n + 2 * h->rows.n + h->children.n + 3 * h->a_slot.n;
    ivec_reserve(buf, need);
    const ivec_t *parts[6] = { &h->rows, &h->rel, &h->children, &h->a_slot, &h->a_rb, &h->a_cb };
    const int lens[6] = { h->rows.n, h->rows.n, h->children.n, h->a_slot.n, h->a_slot.n, h->a_slot.n };
    for (int i = 0; i < 6; i++) {
        if (lens[i] > 0) /* (an empty list may have no storage at all) */
            memcpy(buf->p + buf->n, parts[i]->p, sizeof(int) * (size_t) lens[i]);
        buf->n += lens[i];
    }
}

/* CTAs that share one front in k_factor: fronts that fit in shared memory (200 KB) take one.
 * Larger ones are bound by the LATENCY of their panel steps (two team barriers, the diagonal
 * block, one trailing tile per worker), not by throughput: the team gets one CTA per 256 x 64
 * tile of the first trailing update and no more, so that the fronts of one tree level find room
 * side by side on the SMs instead of queueing for each other's workers. */
static int front_fits_smem(int mb)
{
    int64_t m = 3 * (int64_t) mb;
    return (int64_t) ASAM_LD(m) * m + (ASAM_LD(m) + 1) / 2 + 2 <= 25600;
}

/* Fronts up to this order that do not fit in shared memory go to ONE CTA (cta_front's HBM mode) even where
 * their team would be larger; by default (0) only the fronts whose team the level room scales below two CTAs do
 * (build_schedule).  ASAM_SOLO_MAX_M overrides (tuning). */
static int solo_max_m(void)
{
    static int v = -1;
    if (v < 0) {
        const char *e = getenv("ASAM_SOLO_MAX_M");
        v = e ? atoi(e) : ASAM_SOLO_MAX_M_DEFAULT;
    }
    return v;
}

static int team_size(int mb, int cb, int cap)
{
    int64_t m = 3 * (int64_t) mb, c = 3 * (int64_t) cb;
    if (front_fits_smem(mb) || m <= solo_max_m())
        return 1;
    int64_t j0 = c < 48 ? c : 48, tiles = 0;
    for (int64_t cb0 = j0; cb0 < m; cb0 += 64)
        tiles += (m - cb0 + 1 + 255) / 256;
    int64_t chunks = 1 + (m - j0 + 1 + 127) / 128; /* look-ahead crew: the diagonal block + the 128-row chunks (ASAM_CROWS) */
    /* A panel step (diagonal block + row solves + barrier: the dependent chain) lasts several times as long as a
     * tensor-pipe tile: a worker outside the crew gets through several tiles per step, and a worker that has none left only
     * holds an SM that another front could use.  ASAM_TILES_PER_WORKER overrides (tuning). */
    static int tpw = 0;
    if (tpw == 0) {
        const char *e = getenv("ASAM_TILES_PER_WORKER");
        tpw = e && atoi(e) > 0 ? atoi(e) : ASAM_TILES_PER_WORKER;
    }
    int G = (int) ((tiles + tpw - 1) / tpw + chunks); /* the look-ahead crew (one CTA per chunk) takes no tiles */
    /* every worker of a team must be resident at the same time (spin barriers in a persistent,
     * non-cooperative launch): never more workers than the device seats CTAs of k_factor */
    if (cap < 2)
        cap = 2;
    if (cap > 120)
        cap = 120;
    if (G < 2)
        G = 2;
    if (G > cap)
        G = cap;
    return G;
}

/* nwait word of a task: bits 0-15 children to wait for, 16-23 worker index, 24-30 team size */
static inline int pack_nwait(int nw, int w, int G)
{
    if (nw < 0 || nw > 0xffff || w < 0 || w > 0xff || G < 0 || G > 0x7f)
        asam_fatal("plan: task word overflow (%d children in one launch, worker %d of %d): hub supernodes with more "
                   "than 65535 re-factored children are not supported", nw, w, G);
    return (nw & 0xffff) | (w << 16) | (G << 24);
}

static int plan_team_cap(const plan_t *pl) { return pl->max_team > 0 ? pl->max_team : 120; }

/* doubles of the arena a front of mb block rows occupies: the front itself and, for fronts that do not fit
 * in shared memory (team path), the two row-major panel buffers behind it (asam_kernels.cuh, ASAM_LDW) */
static int64_t front_doubles(int mb)
{
    int64_t m = 3 * (int64_t) mb;
    return (int64_t) ASAM_LD(m) * m + (front_fits_smem(mb) ? 0 : 2 * (m + 2) * 52);
}

/* ---- schedule: task lists of one batch solve ------------------------------------------------
 * Single GPU (world == 1): leaf set -> k_factor_leaf, everything else -> k_factor (level order,
 * teams expanded), back-solve list = [rest | leaf set], parents first.
 *
 * Several GPUs (world > 1, one process each, SURVEY.md section 8e): the elimination tree is cut into
 * disjoint subtrees ("shards") that are dealt to the ranks; a rank factors its own shards (same
 * two kernels), the shard roots' update matrices are exchanged (NCCL broadcast of the trailing
 * columns of each root front, same arena offsets on every rank), and every rank then factors the
 * supernodes above the cut ("top") redundantly.  The back-solve runs top + own shards; the
 * solution segments of the shards (contiguous q intervals: positions are a post-order) are
 * exchanged the same way.  Supernodes of other ranks' shards appear in no list of this rank. */
static double sn_work(const asam_sn_desc_t *d)
{
    double m = 3.0 * d->mb, c = 3.0 * d->cb;
    return c * m * m + 3.0e4; /* flops + a per-front latency floor */
}

void plan_work(const plan_t *pl, const int *tasks, int ntasks, double *step_work, int *step_fronts, double *batch_work,
               int *batch_fronts)
{
    double sw = 0.0, bw = 0.0;
    int sf = 0, last = -1;
    for (int t = 0; t < ntasks; t++) { /* the workers of a team are consecutive entries of one supernode */
        if (tasks[t] == last)
            continue;
        last = tasks[t];
        sw += sn_work(&pl->desc[last]);
        sf++;
    }
    for (int s = 0; s < pl->nsn; s++)
        bw += sn_work(&pl->desc[s]);
    *step_work = sw;
    *step_fronts = sf;
    *batch_work = bw;
    *batch_fronts = pl->nsn;
}

typedef struct {
    double key;
    int id;
} sn_key_t;

static int cmp_key_desc(const void *a, const void *b)
{
    const sn_key_t *x = a, *y = b;
    if (x->key != y->key)
        return x->key > y->key ? -1 : 1;
    return (x->id > y->id) - (x->id < y->id); /* deterministic */
}

/* Modelled duration (microseconds) of front s once its children are done, factored by g CTAs (least-squares
 * fits to device traces of the 100 k world, tools/panel_trace.py --dump-trace).  ASAM_TEAM_MODEL="a,b,c,d,e"
 * overrides the team coefficients (tuning).  A fit to H100 traces of the current team path (children ready ->
 * eliminated of the 943 team fronts, non-negative least squares: 24.8, 30.5, 11.4, 0.077, 0.228) tracks the
 * durations far better (median error 8 % against 22 %) but gave no shorter k_factor (7.14 / 7.18 ms against
 * 7.10 / 7.14 ms, H100 80GB HBM3 at 700 W); the ticket order only needs the relative durations. */
static double team_model[5] = { 21.5, 24.4, 11.6, 0.041, 0.0 };
static void team_model_init(void)
{
    static int done = 0;
    if (done)
        return;
    done = 1;
    const char *e = getenv("ASAM_TEAM_MODEL");
    if (e)
        sscanf(e, "%lf,%lf,%lf,%lf,%lf", &team_model[0], &team_model[1], &team_model[2], &team_model[3], &team_model[4]);
}

/* g: the team size, 0 for one CTA on cta_front */
static double front_lat_us(const plan_t *pl, int s, int g)
{
    const double m = 3.0 * pl->desc[s].mb, c = 3.0 * pl->desc[s].cb;
    if (m <= 48) /* (fitted on fronts of the leaf kernel when its limit was 48) */
        return 2.0 + 0.1 * c;
    if (front_fits_smem(pl->desc[s].mb))
        return 3.8 + 0.121 * m + 0.105 * c + 0.00508 * c * m;
    if (g < 1) /* front in HBM, one CTA (cta_front): non-negative least squares over a + b m + c' c + d c m, fitted to
                  the 816 such fronts of the 100 k world on an H100 80GB HBM3 at 400 W (tools/solo_trace.py): a = c' = 0,
                  median error 6 %, 90th percentile 15 % */
        return 0.119 * m + 0.00631 * c * m;
    double tiles = 0.0, crew = 0.0;
    const int npan = (int) ceil(c / 48.0);
    for (int k = 0; k < npan; k++) {
        const double r = m - 48.0 * (k + 1) > 0 ? m - 48.0 * (k + 1) : 0.0;
        tiles += r * r / 2.0 / (256.0 * 64.0);
        crew += 1.0 + ceil(r / 128.0);
    }
    return team_model[0] * npan + team_model[1] * tiles / g + team_model[2] * crew / g + team_model[3] * m +
           team_model[4] * m * m / 1024.0 / g;
}

/* ---- static list schedule --------------------------------------------------------------------------
 * The ticket order of k_factor decides when a front's CTAs are taken: a team whose tickets come up while
 * its children are still running spins on all its CTAs (on the 100 k world the nine fronts of order > 1000
 * each hold dozens of CTAs).
 * So the order is taken from a SIMULATION of the kernel: P resident CTAs, every front with its modelled
 * duration and team size, ready fronts started by priority (length of the dependent chain above them) as
 * CTAs become free; the order in which the simulation STARTS the fronts is the ticket order.  Children finish
 * before their parent starts in the simulation, so the order is topological; where the model is off the
 * kernel merely waits as it would have.  in[s] != 0: s is a task of this launch (others count as done). */
typedef struct {
    double key;
    int id;
} hp_t;

static void hp_push(hp_t *h, int *n, double key, int id, int maxheap)
{
    int i = (*n)++;
    h[i].key = key;
    h[i].id = id;
    while (i > 0) {
        int p = (i - 1) / 2;
        int better = maxheap ? (h[i].key > h[p].key || (h[i].key == h[p].key && h[i].id < h[p].id))
                             : (h[i].key < h[p].key || (h[i].key == h[p].key && h[i].id < h[p].id));
        if (!better)
            break;
        hp_t t = h[p]; h[p] = h[i]; h[i] = t;
        i = p;
    }
}

static hp_t hp_pop(hp_t *h, int *n, int maxheap)
{
    hp_t top = h[0];
    h[0] = h[--(*n)];
    int i = 0;
    for (;;) {
        int l = 2 * i + 1, r = l + 1, b = i;
        for (int c = l; c <= r; c++) {
            if (c >= *n)
                break;
            int better = maxheap ? (h[c].key > h[b].key || (h[c].key == h[b].key && h[c].id < h[b].id))
                                 : (h[c].key < h[b].key || (h[c].key == h[b].key && h[c].id < h[b].id));
            if (better)
                b = c;
        }
        if (b == i)
            break;
        hp_t t = h[b]; h[b] = h[i]; h[i] = t;
        i = b;
    }
    return top;
}

/* returns the number of entries written to out[] (= tasks with in[s] != 0) */
static int sim_order(const plan_t *pl, const char *in, const int *G_of, const double *lat, const double *prio, int P, int *out)
{
    const int nsn = pl->nsn;
    int *pending = calloc((size_t) nsn + 1, sizeof(int));
    hp_t *ready = malloc(sizeof(hp_t) * (size_t) (nsn + 1)), *events = malloc(sizeof(hp_t) * (size_t) (nsn + 1));
    int nready = 0, nev = 0, nout = 0, free_cta = P;
    for (int s = 0; s < nsn; s++)
        if (in[s] && pl->desc[s].parent >= 0 && in[pl->desc[s].parent])
            pending[pl->desc[s].parent]++;
    for (int s = 0; s < nsn; s++)
        if (in[s] && pending[s] == 0)
            hp_push(ready, &nready, prio[s], s, 1);
    double now = 0.0;
    for (;;) {
        while (nready > 0) {
            int s = ready[0].id, g = G_of[s] < 0 ? 1 : (G_of[s] > P ? P : G_of[s]);
            if (g > free_cta && nev > 0)
                break; /* tickets are strictly ordered: nothing overtakes a team that is gathering its CTAs */
            hp_pop(ready, &nready, 1);
            out[nout++] = s;
            free_cta -= g < free_cta ? g : free_cta;
            hp_push(events, &nev, now + lat[s], s, 0);
        }
        if (nev == 0)
            break;
        hp_t e = hp_pop(events, &nev, 0);
        now = e.key;
        {
            int s = e.id, g = G_of[s] < 0 ? 1 : (G_of[s] > P ? P : G_of[s]);
            free_cta += g;
            if (free_cta > P)
                free_cta = P;
            int par = pl->desc[s].parent;
            if (par >= 0 && in[par] && --pending[par] == 0)
                hp_push(ready, &nready, prio[par], par, 1);
        }
    }
    free(pending);
    free(ready);
    free(events);
    return nout;
}

static void build_schedule(plan_t *pl)
{
    const int nsn = pl->nsn, W = pl->world > 1 ? pl->world : 1, me = pl->world > 1 ? pl->rank : 0;
    free(pl->tasks); free(pl->nwait); free(pl->btasks); free(pl->leaf_tasks);
    free(pl->top_tasks); free(pl->top_nwait);
    free(pl->shard_owner); free(pl->shard_off); free(pl->shard_cnt); free(pl->shard_q0); free(pl->shard_qn);
    pl->top_tasks = pl->top_nwait = pl->shard_owner = pl->shard_q0 = pl->shard_qn = NULL;
    pl->shard_off = pl->shard_cnt = NULL;
    pl->n_top = pl->n_top_sn = pl->n_shards = 0;

    /* owner[s]: rank that factors s, -1 = top (every rank) */
    int *owner = malloc(sizeof(int) * (size_t) (nsn + 1));
    for (int s = 0; s < nsn; s++)
        owner[s] = 0;
    if (W > 1 && nsn > 0) {
        double *sub = malloc(sizeof(double) * (size_t) nsn); /* work of the subtree rooted at s */
        for (int s = 0; s < nsn; s++)
            sub[s] = sn_work(&pl->desc[s]);
        for (int s = 0; s < nsn; s++) /* children have smaller ids */
            if (pl->desc[s].parent >= 0)
                sub[pl->desc[s].parent] += sub[s];
        /* frontier of subtree roots; split the heaviest until the shards can be balanced */
        int *fr = malloc(sizeof(int) * (size_t) (nsn + 1)), nfr = 0;
        double total = 0.0;
        for (int s = 0; s < nsn; s++)
            if (pl->desc[s].parent < 0) {
                fr[nfr++] = s;
                total += sub[s];
            }
        for (int s = 0; s < nsn; s++)
            owner[s] = -2; /* undecided */
        const int max_shards = 16 * W;
        /* ASAM_SHARD_TOL: imbalance at which the splitting stops (tuning).  Every split moves one more front of the
         * dependent chain above the cut, where all ranks repeat it */
        const double shard_tol = getenv("ASAM_SHARD_TOL") ? atof(getenv("ASAM_SHARD_TOL")) : ASAM_SHARD_TOL_DEFAULT;
        double *load = malloc(sizeof(double) * (size_t) W);
        for (;;) {
            /* heaviest-first dealing (LPT) of the current frontier */
            for (int i = 1; i < nfr; i++) { /* insertion sort by (work desc, id asc): deterministic */
                int v = fr[i], j = i - 1;
                while (j >= 0 && (sub[fr[j]] < sub[v] || (sub[fr[j]] == sub[v] && fr[j] > v))) {
                    fr[j + 1] = fr[j];
                    j--;
                }
                fr[j + 1] = v;
            }
            for (int r = 0; r < W; r++)
                load[r] = 0.0;
            double shard_sum = 0.0;
            for (int i = 0; i < nfr; i++) {
                int best = 0;
                for (int r = 1; r < W; r++)
                    if (load[r] < load[best])
                        best = r;
                load[best] += sub[fr[i]];
                shard_sum += sub[fr[i]];
            }
            double mx = 0.0;
            for (int r = 0; r < W; r++)
                if (load[r] > mx)
                    mx = load[r];
            /* stop when balanced within 10 %, when there are plenty of shards, or when the heaviest
             * shard cannot be split (no children) */
            int h = fr[0];
            if (nfr >= W && mx <= shard_tol * shard_sum / W)
                break;
            if (nfr >= max_shards || pl->snh[h].children.n == 0)
                break;
            owner[h] = -1; /* the root of the heaviest shard moves above the cut */
            fr[0] = fr[nfr - 1];
            nfr--;
            for (int c = 0; c < pl->snh[h].children.n; c++)
                fr[nfr++] = pl->snh[h].children.p[c];
        }
        /* final dealing + shard descriptors */
        for (int r = 0; r < W; r++)
            load[r] = 0.0;
        pl->n_shards = nfr;
        pl->shard_owner = malloc(sizeof(int) * (size_t) (nfr + 1));
        pl->shard_off = malloc(sizeof(int64_t) * (size_t) (nfr + 1));
        pl->shard_cnt = malloc(sizeof(int64_t) * (size_t) (nfr + 1));
        pl->shard_q0 = malloc(sizeof(int) * (size_t) (nfr + 1));
        pl->shard_qn = malloc(sizeof(int) * (size_t) (nfr + 1));
        int *npose = calloc((size_t) nsn + 1, sizeof(int)); /* poses in the subtree of s */
        for (int s = 0; s < nsn; s++) {
            npose[s] += pl->desc[s].cb;
            if (pl->desc[s].parent >= 0)
                npose[pl->desc[s].parent] += npose[s];
        }
        for (int i = 0; i < nfr; i++) {
            int best = 0, s = fr[i];
            for (int r = 1; r < W; r++)
                if (load[r] < load[best])
                    best = r;
            load[best] += sub[s];
            owner[s] = best;
            const asam_sn_desc_t *d = &pl->desc[s];
            int64_t m = 3 * (int64_t) d->mb, c = 3 * (int64_t) d->cb, ld = ASAM_LD(m);
            pl->shard_owner[i] = best;
            pl->shard_off[i] = d->f_off + c * ld;   /* trailing columns: update matrix + rhs row */
            pl->shard_cnt[i] = (m - c) * ld;
            pl->shard_qn[i] = npose[s];
            pl->shard_q0[i] = d->first + d->cb - npose[s];
        }
        /* push ownership down the shards (parents have larger ids) */
        for (int s = nsn - 1; s >= 0; s--)
            if (owner[s] == -2)
                owner[s] = pl->desc[s].parent >= 0 ? owner[pl->desc[s].parent] : -1;
        free(npose);
        free(load);
        free(fr);
        free(sub);
    }

    /* leaf set: supernodes whose whole subtree consists of fronts small enough for the
     * warp-per-front kernels (children have smaller ids).  Only worth separate launches when
     * there are thousands of them. */
    char *leaf = calloc((size_t) nsn + 1, 1);
    int n_leaf_all = 0;
    const int leaf_max = leaf_max_m_for(nsn);
    for (int s = 0; s < nsn; s++) {
        int ok = 3 * pl->desc[s].mb <= leaf_max;
        for (int c = 0; ok && c < pl->snh[s].children.n; c++)
            ok = leaf[pl->snh[s].children.p[c]];
        leaf[s] = (char) ok;
        n_leaf_all += ok;
    }
    if (n_leaf_all < ASAM_LEAF_MIN_COUNT)
        memset(leaf, 0, (size_t) nsn);
    /* the warp-per-supernode BACK-SOLVE takes any downward-closed set with <= 64 own columns and
     * <= 64 rows below (a superset of the factor leaf set); it pays from a few dozen supernodes on:
     * a warp per supernode has everything fetched before its parent's flag arrives */
    free(pl->bs_leaf);
    pl->bs_leaf = calloc((size_t) pl->sn_cap + 1, 1);
    for (int s = 0; s < nsn; s++) {
        int ok = 3 * pl->desc[s].cb <= ASAM_BSLEAF_MAX && 3 * (pl->desc[s].mb - pl->desc[s].cb) <= ASAM_BSLEAF_MAX;
        for (int c = 0; ok && c < pl->snh[s].children.n; c++)
            ok = pl->bs_leaf[pl->snh[s].children.p[c]];
        pl->bs_leaf[s] = (char) ok;
    }

    /* Task order.  The persistent kernels hand out tasks in list order, so the list IS the schedule.  Plain
     * level order (every front of level l before any of level l+1) starts the deepest chain of the tree last
     * among its level-mates and leaves its top to run alone at the end, with most SMs spinning.
     * Critical-path-first instead: fronts are listed by
     * DESCENDING length of the dependent chain from them up to the root (their own modelled latency
     * included), which is still a topological order -- a child's chain is its parent's plus its own -- so a
     * waiting CTA only ever waits for tasks that were handed out before its own.  ASAM_TASK_ORDER=level keeps
     * the level order (A/B). */
    int *byl = malloc(sizeof(int) * (size_t) (nsn + 1));
    int order_mode = 0; /* 0 level, 1 chain length ("cp"), 2 simulated schedule ("sim"), 3 auto: cp or sim by load */
    int *bylv = malloc(sizeof(int) * (size_t) (nsn + 1)); /* plain level order: the back-substitution list (faster
                                                            * than the reversed chain order in A/B runs) */
    {
        int *cnt = calloc((size_t) pl->n_levels + 2, sizeof(int));
        for (int s = 0; s < nsn; s++)
            cnt[pl->desc[s].level + 1]++;
        for (int l = 0; l < pl->n_levels; l++)
            cnt[l + 1] += cnt[l];
        for (int s = 0; s < nsn; s++)
            bylv[cnt[pl->desc[s].level]++] = s;
        free(cnt);
    }
    {
        const char *eo = getenv("ASAM_TASK_ORDER");
        if (eo && strcmp(eo, "level") == 0) {
            memcpy(byl, bylv, sizeof(int) * (size_t) nsn);
        } else {
            order_mode = (eo && strcmp(eo, "cp") == 0) ? 1 : ((eo && strcmp(eo, "sim") == 0) ? 2 : 3);
        }
    }

    /* team sizes.  A front's team is bound by latency, not throughput (team_size()), so where one tree
     * level holds more team fronts than the SMs can seat side by side, smaller teams finish the
     * LEVEL sooner: CTA-time per front (G x duration) falls with G.  Scale the teams of such a level
     * down to the room there is (never below 2). */
    int *G_of = malloc(sizeof(int) * (size_t) (nsn + 1));
    {
        int64_t *want = calloc((size_t) pl->n_levels + 1, sizeof(int64_t));
        for (int s = 0; s < nsn; s++) {
            G_of[s] = (owner[s] == me || owner[s] == -1) && !leaf[s] ? team_size(pl->desc[s].mb, pl->desc[s].cb, plan_team_cap(pl)) : 1;
            if (G_of[s] > 1)
                want[pl->desc[s].level] += G_of[s];
        }
        int64_t room = ASAM_TEAM_ROOM < plan_team_cap(pl) ? ASAM_TEAM_ROOM : plan_team_cap(pl);
        const char *er = getenv("ASAM_TEAM_ROOM"); /* tuning knob (tools only) */
        if (er && atoi(er) > 0)
            room = atoi(er);
        /* A front scaled below a team of two is factored by ONE CTA on cta_front's HBM path (task word G = 0): it
         * pays where a level holds far more team fronts than SMs (the SM time per front is what limits the level,
         * not its latency), and one CTA needs none of the team protocol.  ASAM_TEAM_MIN=g (A/B) sets the smallest
         * team instead; with g = 1 such fronts run the team code alone (G = 1). */
        int gmin = 0;
        const char *em = getenv("ASAM_TEAM_MIN");
        if (em && atoi(em) >= 1)
            gmin = atoi(em);
        for (int s = 0; s < nsn; s++) {
            int64_t w = want[pl->desc[s].level];
            if (G_of[s] > 1 && w > room) {
                int g = (int) ((int64_t) G_of[s] * room / w);
                g = g < gmin ? gmin : g;
                G_of[s] = g >= 2 ? g : (gmin == 1 ? -1 : 1); /* -1: one CTA, team code path */
            }
        }
        free(want);
    }
    if (order_mode != 0) {
        /* modelled duration of every front once its children are done (microseconds; least-squares fit to device
         * traces of the 100 k world, tools/panel_trace.py --dump-trace: median error 8 % for shared-memory fronts,
         * 9 % for teams) and the length of the dependent chain from a front up to the root */
        double *lat_us = malloc(sizeof(double) * (size_t) (nsn + 1)), *up_us = malloc(sizeof(double) * (size_t) (nsn + 1));
        double work = 0.0, chain = 0.0;
        team_model_init();
        for (int s = nsn - 1; s >= 0; s--) { /* parents have larger ids */
            const int g = G_of[s] < 0 ? 1 : G_of[s];
            const double lat = front_lat_us(pl, s, G_of[s] == 1 ? 0 : g);
            lat_us[s] = lat;
            up_us[s] = lat + (pl->desc[s].parent >= 0 ? up_us[pl->desc[s].parent] : 0.0);
            if ((owner[s] == me || owner[s] == -1) && !leaf[s])
                work += lat * g;
            if (up_us[s] > chain)
                chain = up_us[s];
        }
        const int P = pl->n_cta > 0 ? pl->n_cta : 132;
        /* auto: where the SMs are far from saturated (M3500: 11 of 67 CTA-ms busy) spinning costs nothing and the
         * eager chain-length order starts parents soonest; where they are saturated, a team must not take its
         * CTAs before it can use them */
        const int use_sim = order_mode == 2 || (order_mode == 3 && work / P > 0.5 * chain);
        {
            sn_key_t *keys = malloc(sizeof(sn_key_t) * (size_t) (nsn + 1));
            for (int s = 0; s < nsn; s++) {
                keys[s].key = up_us[s];
                keys[s].id = s;
            }
            qsort(keys, (size_t) nsn, sizeof(sn_key_t), cmp_key_desc);
            for (int k = 0; k < nsn; k++)
                byl[k] = keys[k].id;
            free(keys);
        }
        if (use_sim) {
            /* ticket order of k_factor = start order of the simulated schedule; the main list (own fronts outside
             * the leaf set) and the part above a multi-GPU cut are separate launches, simulated separately; the
             * leaf set keeps the chain-length order (warp-sized tasks: nothing to gather) */
            char *in = calloc((size_t) nsn + 1, 1);
            int *ord = malloc(sizeof(int) * (size_t) (nsn + 1)), *pos_of = malloc(sizeof(int) * (size_t) (nsn + 1));
            int n1, n2;
            for (int s = 0; s < nsn; s++)
                in[s] = owner[s] == me && !leaf[s];
            n1 = sim_order(pl, in, G_of, lat_us, up_us, P, ord);
            for (int s = 0; s < nsn; s++)
                in[s] = owner[s] == -1;
            n2 = sim_order(pl, in, G_of, lat_us, up_us, P, ord + n1);
            for (int s = 0; s < nsn; s++)
                pos_of[s] = -1;
            for (int k = 0; k < n1 + n2; k++)
                pos_of[ord[k]] = k;
            /* byl: simulated tasks in start order, everything else (leaf set, other ranks) after them in the old order */
            int *nb = malloc(sizeof(int) * (size_t) (nsn + 1)), k2 = 0;
            for (int k = 0; k < n1 + n2; k++)
                nb[k2++] = ord[k];
            for (int k = 0; k < nsn; k++)
                if (pos_of[byl[k]] < 0)
                    nb[k2++] = byl[k];
            memcpy(byl, nb, sizeof(int) * (size_t) nsn);
            free(nb);
            free(in);
            free(ord);
            free(pos_of);
        }
        free(lat_us);
        free(up_us);
    }

    /* Back-solve entries of a supernode: one, or -- supernodes wider than one 96-column block (ASAM_BSW) in a
     * batch schedule -- one per block, last block first, each solved by its own CTA (cta_backsolve, blk_only).
     * Entry word: supernode | (block + 1) << 24.  ASAM_BS_SPLIT=0 switches the split off (A/B). */
    int bs_split = 1;
    {
        const char *eb = getenv("ASAM_BS_SPLIT");
        if (eb)
            bs_split = atoi(eb) != 0;
    }
    pl->bt_split = 0;
#define BS_NBLK(s_) ((bs_split && !pl->bs_leaf[s_] && 3 * pl->desc[s_].cb > 96 && pl->nsn < (1 << 24)) ? (3 * pl->desc[s_].cb + 95) / 96 : 1)
    int64_t n_local = 0, n_top = 0;
    int n_leaf = 0, n_main_sn = 0, n_top_sn = 0, n_bsl = 0, n_top_bt = 0;
    for (int s = 0; s < nsn; s++)
        n_bsl += owner[s] == me && pl->bs_leaf[s];
    if (n_bsl < ASAM_BSLEAF_MIN_COUNT) {
        memset(pl->bs_leaf, 0, (size_t) nsn);
        n_bsl = 0;
    }
    for (int s = 0; s < nsn; s++) {
        if (owner[s] == me) {
            if (leaf[s])
                n_leaf++;
            else
                n_local += G_of[s] < 0 ? 1 : G_of[s];
            if (!pl->bs_leaf[s])
                n_main_sn += BS_NBLK(s);
        } else if (owner[s] == -1) {
            n_top += G_of[s] < 0 ? 1 : G_of[s];
            n_top_sn++;
            n_top_bt += BS_NBLK(s);
        }
    }
    pl->ntasks = (int) n_local;
    pl->tasks = malloc(sizeof(int) * (size_t) (n_local + 1));
    pl->nwait = malloc(sizeof(int) * (size_t) (n_local + 1));
    pl->n_leaf = n_leaf;
    pl->leaf_tasks = malloc(sizeof(int) * (size_t) (n_leaf + 1));
    pl->n_top = (int) n_top;
    pl->n_top_sn = n_top_sn;
    pl->top_tasks = malloc(sizeof(int) * (size_t) (n_top + 1));
    pl->top_nwait = malloc(sizeof(int) * (size_t) (n_top + 1));
    pl->n_bs_leaf = n_bsl;
    pl->n_btasks = n_top_bt + n_main_sn + n_bsl;
    pl->btasks = malloc(sizeof(int) * (size_t) (pl->n_btasks + 1));
    /* back-solve list, parents first: [top | own shards outside the back-solve leaf set | that set].
     * Order inside a segment: by the modelled TIME of the longest chain below a supernode (its own solve included),
     * longest first -- a parent's chain is longer than any child's, so the order is topological, and the deep
     * chains do not queue behind the thousands of supernodes that merely share their height (level order: the
     * bottom of the longest chain of the 100 k world got its tickets late at every link).  ASAM_BS_ORDER=level
     * keeps the height order (A/B). */
    {
        const char *eb = getenv("ASAM_BS_ORDER");
        if (!(eb && strcmp(eb, "level") == 0) && nsn > 0) {
            double *down = calloc((size_t) nsn, sizeof(double));
            sn_key_t *keys = malloc(sizeof(sn_key_t) * (size_t) nsn);
            for (int s = 0; s < nsn; s++) { /* children have smaller ids: down[s] holds max over children here */
                if (!pl->bs_leaf[s]) /* (the warp-per-supernode set runs in a launch of its own, afterwards) */
                    down[s] += 5.0 + 0.17 * 3.0 * pl->desc[s].cb + 0.01 * 3.0 * pl->desc[s].mb;
                else
                    down[s] += 1e-3 * (pl->desc[s].level + 1);
                const int par = pl->desc[s].parent;
                if (par >= 0 && down[s] > down[par])
                    down[par] = down[s];
                keys[s].key = down[s];
                keys[s].id = s;
            }
            qsort(keys, (size_t) nsn, sizeof(sn_key_t), cmp_key_desc);
            for (int k = 0; k < nsn; k++)
                bylv[nsn - 1 - k] = keys[k].id; /* ascending: the list below is filled backwards */
            free(keys);
            free(down);
        }
    }
    int t = 0, tl = 0, tt = 0;
    int bt = n_top_bt - 1, bm = n_top_bt + n_main_sn - 1, bl = pl->n_btasks - 1;
    for (int k = 0; k < nsn; k++) { /* back-solve entries, filled backwards: parents first */
        int s = bylv[k];
        if (owner[s] == -1) {
            const int nb = BS_NBLK(s); /* block 0 lands last, the last block first */
            for (int b = 0; b < nb; b++)
                pl->btasks[bt--] = nb > 1 ? (s | ((b + 1) << 24)) : s;
            pl->bt_split |= nb > 1;
        } else if (owner[s] == me) {
            if (pl->bs_leaf[s]) {
                pl->btasks[bl--] = s;
            } else {
                const int nb = BS_NBLK(s);
                for (int b = 0; b < nb; b++)
                    pl->btasks[bm--] = nb > 1 ? (s | ((b + 1) << 24)) : s;
                pl->bt_split |= nb > 1;
            }
        }
    }
    for (int k = 0; k < nsn; k++) { /* factorisation tasks, children first */
        int s = byl[k];
        if (owner[s] == -1) {
            int nw = 0; /* children above the cut: the others were exchanged before this launch */
            for (int c = 0; c < pl->snh[s].children.n; c++)
                nw += owner[pl->snh[s].children.p[c]] == -1;
            int G = G_of[s] < 0 ? 1 : G_of[s];
            for (int w = 0; w < G; w++, tt++) {
                pl->top_tasks[tt] = s;
                pl->top_nwait[tt] = pack_nwait(nw, w, G > 1 ? G : (G_of[s] < 0 ? 1 : 0));
            }
            continue;
        }
        if (owner[s] != me)
            continue;
        if (leaf[s]) {
            pl->leaf_tasks[tl++] = s;
            continue;
        }
        /* nwait counts ALL children: those of the leaf set arrived in the earlier launch */
        int G = G_of[s] < 0 ? 1 : G_of[s];
        for (int w = 0; w < G; w++, t++) {
            pl->tasks[t] = s;
            pl->nwait[t] = pack_nwait(pl->desc[s].ch_cnt, w, G > 1 ? G : (G_of[s] < 0 ? 1 : 0));
        }
    }
#undef BS_NBLK
    free(G_of);
    free(byl);
    free(bylv);
    free(leaf);
    free(owner);
}

/* ---- batch build --------------------------------------------------------------------------- */
static int plan_build_impl(plan_t *pl, asam_dev_t *dev, int N, int n_factors, const int *ftype, const int *fa,
                           const int *fb, const int *order_keep, int N_keep)
{
    uint64_t keep_hash = pl->struct_hash;
    int keep_world = pl->world, keep_rank = pl->rank, keep_team = pl->max_team, keep_cta = pl->n_cta;
    plan_free(pl);
    pl->struct_hash = keep_hash;
    pl->world = keep_world;
    pl->rank = keep_rank;
    pl->max_team = keep_team;
    pl->n_cta = keep_cta;
    if (dev) { /* teams are sized for the CTAs this device actually seats (MIG slice, smaller part, ...) */
        int n_sm = 0, fac_grid = 0, fac_smem = 0, bs_grid = 0;
        if (asam_device_info(dev, &n_sm, &fac_grid, &fac_smem, &bs_grid) == 0 && fac_grid > 0)
            pl->max_team = fac_grid < 120 ? fac_grid : 120, pl->n_cta = fac_grid;
    }
    if (N <= 0)
        return 0;
    node_arrays_reserve(pl, N);
    fslot_reserve(pl, n_factors);
    pl->N = N;
    pl->n_factors = n_factors;

    double bt_ = pp_now(), bt2_;
#define BUILD_LAP(i)                 \
    do {                             \
        bt2_ = pp_now();             \
        g_build_prof[i] += bt2_ - bt_; \
        bt_ = bt2_;                  \
    } while (0)
    /* 1. unique node pairs -> Hessian slots */
    pairmap_init(&pl->pairs, n_factors);
    ivec_t plo = { 0 }, phi = { 0 };
    for (int f = 0; f < n_factors; f++) {
        if (asam_two_pose_type(ftype[f])) {
            int a = fa[f], b = fb[f];
            if (a == b || a < 0 || b < 0 || a >= N || b >= N) {
                asam_set_error("factor %d: bad node ids (%d,%d)", f, a, b);
                return 1;
            }
            int lo = a < b ? a : b, hi = a < b ? b : a, created;
            int slot = pairmap_get_or_add(&pl->pairs, lo, hi, pl->n_slots, &created);
            if (created) {
                ivec_push(&plo, lo);
                ivec_push(&phi, hi);
                pl->n_slots++;
            }
            pl->fslot[f] = slot;
        } else if (ftype[f] == APRIL_GRAPH_FACTOR_XYTPOS_TYPE) {
            if (fa[f] < 0 || fa[f] >= N) {
                asam_set_error("factor %d: bad node id %d", f, fa[f]);
                return 1;
            }
            pl->fslot[f] = -1;
        } else {
            asam_set_error("factor %d: unsupported factor type %d", f, ftype[f]);
            return 1;
        }
    }
    const int S = pl->n_slots;

    /* 2. adjacency CSR, ascending */
    int *adj_ptr = calloc((size_t) N + 1, sizeof(int));
    for (int s = 0; s < S; s++) {
        adj_ptr[plo.p[s] + 1]++;
        adj_ptr[phi.p[s] + 1]++;
    }
    for (int i = 0; i < N; i++)
        adj_ptr[i + 1] += adj_ptr[i];
    int *adj = malloc(sizeof(int) * (size_t) (2 * S + 1));
    int *fill = malloc(sizeof(int) * (size_t) N);
    memcpy(fill, adj_ptr, sizeof(int) * (size_t) N);
    for (int s = 0; s < S; s++) {
        adj[fill[plo.p[s]]++] = phi.p[s];
        adj[fill[phi.p[s]]++] = plo.p[s];
    }
    for (int i = 0; i < N; i++)
        sort_ints(adj + adj_ptr[i], adj_ptr[i + 1] - adj_ptr[i]);
    free(fill);

    BUILD_LAP(0); /* slots + adjacency */
    /* 3. elimination order */
    if (order_keep) {
        for (int p = 0; p < N_keep; p++)
            pl->order[p] = order_keep[p];
        for (int p = N_keep; p < N; p++)
            pl->order[p] = p;
    } else {
        int *ord = asam_ref_ordering(N, adj_ptr, adj);
        memcpy(pl->order, ord, sizeof(int) * (size_t) N);
        free(ord);
    }
    for (int p = 0; p < N; p++)
        pl->pos[pl->order[p]] = p;

    BUILD_LAP(1); /* ordering */
    /* 4. block symbolic factorisation in reference positions */
    int *parent = pl->parent_pos;
    int *head = malloc(sizeof(int) * (size_t) N), *tail = malloc(sizeof(int) * (size_t) N);
    int *next = malloc(sizeof(int) * (size_t) N), *nchild = calloc((size_t) N, sizeof(int));
    int *stamp = calloc((size_t) N, sizeof(int));
    int64_t *bptr = malloc(sizeof(int64_t) * ((size_t) N + 1));
    ivec_t bl = { 0 };
    for (int p = 0; p < N; p++)
        head[p] = tail[p] = next[p] = -1;
    bptr[0] = 0;
    for (int p = 0; p < N; p++) {
        int v = pl->order[p], start = bl.n, token = p + 1;
        stamp[p] = token;
        for (int e = adj_ptr[v]; e < adj_ptr[v + 1]; e++) {
            int pu = pl->pos[adj[e]];
            if (pu > p && stamp[pu] != token) {
                stamp[pu] = token;
                ivec_push(&bl, pu);
            }
        }
        for (int c = head[p]; c >= 0; c = next[c]) {
            for (int64_t e = bptr[c]; e < bptr[c + 1]; e++) {
                int x = bl.p[e];
                if (stamp[x] != token) {
                    stamp[x] = token;
                    ivec_push(&bl, x);
                }
            }
        }
        /* (the lists stay unsorted: only their sizes, their union and their minimum -- the parent -- are used; the
         * rows of a supernode are sorted once, in numeric positions, in step 7) */
        bptr[p + 1] = bl.n;
        int pmin = -1;
        for (int e = start; e < bl.n; e++)
            if (pmin < 0 || bl.p[e] < pmin)
                pmin = bl.p[e];
        parent[p] = pmin;
        if (parent[p] >= 0) {
            int P = parent[p];
            if (tail[P] < 0)
                head[P] = p;
            else
                next[tail[P]] = p;
            tail[P] = p;
            nchild[P]++;
        }
    }
    free(stamp);
    free(adj);
    free(adj_ptr);

    BUILD_LAP(2); /* block symbolic */
    /* 5. post-order -> numeric positions q.  Children are visited in ascending structure
     * size so that the child with the largest front is numbered right before its parent and can
     * share a supernode with it (step 6). */
    {
        int *kids = malloc(sizeof(int) * (size_t) N);
        for (int p = 0; p < N; p++) {
            int n = 0;
            for (int c = head[p]; c >= 0; c = next[c])
                kids[n++] = c;
            if (n < 2)
                continue;
            for (int i = 1; i < n; i++) { /* insertion sort by (|below|, position) */
                int v = kids[i], j = i - 1;
                int64_t kv = bptr[v + 1] - bptr[v];
                while (j >= 0 && (bptr[kids[j] + 1] - bptr[kids[j]]) > kv) {
                    kids[j + 1] = kids[j];
                    j--;
                }
                kids[j + 1] = v;
            }
            head[p] = kids[0];
            for (int i = 0; i + 1 < n; i++)
                next[kids[i]] = kids[i + 1];
            next[kids[n - 1]] = -1;
            tail[p] = kids[n - 1];
        }
        free(kids);
    }
    int *qpos = malloc(sizeof(int) * (size_t) N), *pofq = malloc(sizeof(int) * (size_t) N);
    {
        int *stack = malloc(sizeof(int) * (size_t) N), *it = malloc(sizeof(int) * (size_t) N);
        int q = 0;
        for (int r = 0; r < N; r++) {
            if (parent[r] >= 0)
                continue;
            int sp = 0;
            stack[sp] = r;
            it[sp] = head[r];
            sp++;
            while (sp > 0) {
                int c = it[sp - 1];
                if (c >= 0) {
                    it[sp - 1] = next[c];
                    stack[sp] = c;
                    it[sp] = head[c];
                    sp++;
                } else {
                    int p = stack[--sp];
                    qpos[p] = q;
                    pofq[q] = p;
                    q++;
                }
            }
        }
        free(stack);
        free(it);
    }
    for (int p = 0; p < N; p++) {
        pl->node2q[pl->order[p]] = qpos[p];
        pl->q2node[qpos[p]] = pl->order[p];
    }

    /* 6. supernodes: a node joins the supernode of the child numbered right before it when the
     * child's structure is the node's structure plus itself (fundamental), or misses at most
     * RELAX_Z block rows of it (relaxed amalgamation: a few explicit zero blocks buy fewer, fatter
     * fronts and a shorter dependency chain); width capped at MAX_SN_COLS. */
    int relax_z = RELAX_Z, relax_fill = RELAX_FILL; /* ASAM_RELAX_Z / ASAM_RELAX_FILL override (tuning) */
    if (getenv("ASAM_RELAX_Z"))
        relax_z = atoi(getenv("ASAM_RELAX_Z"));
    if (getenv("ASAM_RELAX_FILL"))
        relax_fill = atoi(getenv("ASAM_RELAX_FILL"));
    int team_merge_pct = TEAM_MERGE_PCT;
    double team_merge_mflop = TEAM_MERGE_MFLOP;
    if (getenv("ASAM_TEAM_MERGE_PCT"))
        team_merge_pct = atoi(getenv("ASAM_TEAM_MERGE_PCT"));
    if (getenv("ASAM_TEAM_MERGE_MFLOP"))
        team_merge_mflop = atof(getenv("ASAM_TEAM_MERGE_MFLOP"));
    pl->nsn = 0;
    pl->nnz_l_blocks = 0;
    pl->flops = 0.0;
    for (int q = 0; q < N; q++) {
        int p = pofq[q];
        int nb = (int) (bptr[p + 1] - bptr[p]);
        pl->nnz_l_blocks += 1 + nb;
        for (int k = 0; k < 3; k++) {
            double cnt = 3.0 * nb + 3 - k;
            pl->flops += cnt * cnt;
        }
        int merge = 0;
        if (q > 0 && pl->nsn > 0) {
            int pp = pofq[q - 1];
            int nbp = (int) (bptr[pp + 1] - bptr[pp]);
            int z = nb + 1 - nbp; /* block rows of {p} + below(p) missing from below(pp); >= 0 */
            int gcb = pl->desc[pl->nsn - 1].cb;
            if (parent[pp] == p && gcb < MAX_SN_COLS &&
                (z == 0 || (z <= relax_z && (int64_t) z * gcb <= relax_fill)))
                merge = 1;
            /* a fundamental chain whose front is processed by a CTA team anyway (it does not fit
             * in shared memory) is not capped: splitting it only adds levels and one full copy of
             * the update matrix per link */
            if (!merge && parent[pp] == p && z == 0 && !front_fits_smem(gcb + nbp))
                merge = 1;
            /* team-sized fronts along a chain: every front boundary costs the chain an extend-add pass, a
             * first panel without look-ahead, a ticket and a partly filled last panel, the
             * explicit zeros of a merge only tensor-pipe tiles spread over the whole team.  Merge while the
             * extra rows stay below team_merge_pct % of the front and the extra flops below team_merge_mflop. */
            if (!merge && parent[pp] == p && team_merge_pct > 0 && !front_fits_smem(gcb + nbp) &&
                (int64_t) z * 100 <= (int64_t) team_merge_pct * (gcb + nbp) &&
                27.0 * gcb * z * (2.0 * (gcb + nbp) + z) <= 1e6 * team_merge_mflop)
                merge = 1;
        }
        if (merge) {
            pl->desc[pl->nsn - 1].cb++;
        } else {
            sn_arrays_reserve(pl, pl->nsn + 1);
            asam_sn_desc_t *d = &pl->desc[pl->nsn];
            memset(d, 0, sizeof(*d));
            d->first = q;
            d->cb = 1;
            d->parent = -1;
            pl->nsn++;
        }
        pl->sn_of_q[q] = pl->nsn - 1;
    }

    BUILD_LAP(3); /* post-order + supernodes */
    /* 7. row lists, parents, children, levels */
    pl->max_m = 0;
    int max_m = 0;
    /* (per-supernode work, independent: split over a few host threads on large graphs, like the pose loops of solver.c) */
#pragma omp parallel for schedule(static, 256) reduction(max : max_m) if (pl->nsn >= PLAN_OMP_MIN_SN) num_threads(plan_threads())
    for (int s = 0; s < pl->nsn; s++) {
        asam_sn_desc_t *d = &pl->desc[s];
        sn_host_t *h = &pl->snh[s];
        int qt = d->first + d->cb - 1, pt = pofq[qt];
        int nb = (int) (bptr[pt + 1] - bptr[pt]);
        ivec_reserve(&h->rows, d->cb + nb);
        for (int k = 0; k < d->cb; k++)
            ivec_push(&h->rows, d->first + k);
        for (int64_t e = bptr[pt]; e < bptr[pt + 1]; e++)
            ivec_push(&h->rows, qpos[bl.p[e]]);
        /* positions on a root path are ordered alike in both numberings; be safe anyway */
        sort_ints(h->rows.p + d->cb, nb);
        d->mb = h->rows.n;
        if (3 * d->mb > max_m)
            max_m = 3 * d->mb;
        d->parent = nb > 0 ? pl->sn_of_q[h->rows.p[d->cb]] : -1;
    }
    pl->max_m = max_m;
    for (int s = 0; s < pl->nsn; s++) {
        int P = pl->desc[s].parent;
        if (P >= 0) {
            ivec_push(&pl->snh[P].children, s);
            int lv = pl->desc[s].level + 1;
            if (lv > pl->desc[P].level)
                pl->desc[P].level = lv; /* children have smaller ids: final when P is reached */
        }
    }
    pl->n_levels = 0;
    {
        int rel_bad = 0, n_levels = 0;
#pragma omp parallel for schedule(static, 256) reduction(| : rel_bad) reduction(max : n_levels) if (pl->nsn >= PLAN_OMP_MIN_SN) num_threads(plan_threads())
        for (int s = 0; s < pl->nsn; s++) {
            rel_bad |= compute_rel(pl, s);
            if (pl->desc[s].level + 1 > n_levels)
                n_levels = pl->desc[s].level + 1;
        }
        if (rel_bad)
            return 1;
        pl->n_levels = n_levels;
    }
    free(bptr);
    ivec_free(&bl);
    free(head);
    free(tail);
    free(next);
    free(nchild);
    free(qpos);
    free(pofq);

    BUILD_LAP(4); /* row lists, rel */
    /* 8. Hessian gather lists: the searches in parallel, the lists filled in slot order */
    {
        int *g_sn = malloc(sizeof(int) * (size_t) (S + 1)), *g_rb = malloc(sizeof(int) * (size_t) (S + 1)),
            *g_cb = malloc(sizeof(int) * (size_t) (S + 1));
        int bad_slot = -1;
#pragma omp parallel for schedule(static, 4096) reduction(max : bad_slot) if (S >= 8 * PLAN_OMP_MIN_SN) num_threads(plan_threads())
        for (int sl = 0; sl < S; sl++) {
            int lo = plo.p[sl], hi = phi.p[sl];
            int qlo = pl->node2q[lo], qhi = pl->node2q[hi];
            int qe = qlo < qhi ? qlo : qhi, ql = qlo < qhi ? qhi : qlo;
            int s = pl->sn_of_q[qe];
            const sn_host_t *h = &pl->snh[s];
            int rb = find_sorted(h->rows.p, h->rows.n, ql);
            if (rb < 0 && sl > bad_slot)
                bad_slot = sl;
            g_sn[sl] = s;
            g_rb[sl] = rb | (qe == qlo ? 0 : ASAM_TR_FLAG);
            g_cb[sl] = qe - pl->desc[s].first;
        }
        if (bad_slot >= 0) {
            asam_set_error("plan: Hessian block (%d,%d) not in the structure of supernode %d", plo.p[bad_slot], phi.p[bad_slot],
                           g_sn[bad_slot]);
            free(g_sn);
            free(g_rb);
            free(g_cb);
            return 1;
        }
        for (int sl = 0; sl < S; sl++) {
            sn_host_t *h = &pl->snh[g_sn[sl]];
            ivec_push(&h->a_slot, sl);
            ivec_push(&h->a_rb, g_rb[sl]);
            ivec_push(&h->a_cb, g_cb[sl]);
        }
        free(g_sn);
        free(g_rb);
        free(g_cb);
    }
    ivec_free(&plo);
    ivec_free(&phi);

    BUILD_LAP(5); /* gather lists */
    /* 9. layout + schedule */
    ivec_t seg = { 0 };
    pl->arena_n = 0;
    for (int s = 0; s < pl->nsn; s++) {
        emit_segment(pl, s, &seg, 0);
        pl->desc[s].f_off = pl->arena_n;
        pl->desc[s].reserved = front_doubles(pl->desc[s].mb); /* capacity of this allocation */
        pl->arena_n += pl->desc[s].reserved;
    }
    pl->ipool_n = seg.n;

    build_schedule(pl);

    BUILD_LAP(6); /* segments + schedule */
    /* host mirror of the device int pool (debug / tests) */
    ivec_free(&pl->ipool_host);
    ivec_reserve(&pl->ipool_host, seg.n);
    memcpy(pl->ipool_host.p, seg.p, sizeof(int) * (size_t) seg.n);
    pl->ipool_host.n = seg.n;
    if (!dev) {
        ivec_free(&seg);
        return 0;
    }

    /* 10. upload */
    int64_t ipool_cap = pl->ipool_n * 2 + 4096, arena_cap = pl->arena_n + pl->arena_n / 2 + 65536;
    int rc = asam_reserve(dev, N + N / 2 + 64, n_factors + n_factors / 2 + 64, S + S / 2 + 64,
                          pl->nsn + N / 2 + 64, ipool_cap, arena_cap);
    if (rc)
        return rc;
    int *ids = malloc(sizeof(int) * (size_t) pl->nsn);
    for (int s = 0; s < pl->nsn; s++)
        ids[s] = s;
    rc |= asam_upload_ipool(dev, 0, seg.n, seg.p);
    rc |= asam_upload_desc(dev, pl->nsn, ids, pl->desc);
    rc |= asam_upload_node2q(dev, 0, N, pl->node2q);
    rc |= asam_upload_q2node(dev, 0, N, pl->q2node);
    rc |= asam_upload_fslot(dev, 0, n_factors, pl->fslot);
    rc |= asam_set_full_tasks(dev, pl->ntasks, pl->tasks, pl->nwait, pl->n_btasks, pl->btasks);
    rc |= asam_set_leaf_tasks(dev, pl->n_leaf, pl->leaf_tasks);
    rc |= asam_set_bs_leaf_count(dev, pl->n_bs_leaf);
    if (pl->world > 1) {
        asam_shard_sched_t sh;
        memset(&sh, 0, sizeof(sh));
        sh.n_top = pl->n_top;
        sh.top_tasks = pl->top_tasks;
        sh.top_nwait = pl->top_nwait;
        sh.n_top_sn = pl->n_top_sn;
        sh.n_shards = pl->n_shards;
        sh.shard_owner = pl->shard_owner;
        sh.shard_off = pl->shard_off;
        sh.shard_cnt = pl->shard_cnt;
        sh.shard_q0 = pl->shard_q0;
        sh.shard_qn = pl->shard_qn;
        rc |= asam_set_shard_schedule(dev, &sh);
    } else {
        rc |= asam_set_shard_schedule(dev, NULL);
    }
    free(ids);
    ivec_free(&seg);
    BUILD_LAP(7); /* upload */
    return rc;
}

int plan_build(plan_t *pl, asam_dev_t *dev, int N, int n_factors, const int *ftype, const int *fa, const int *fb)
{
    return plan_build_impl(pl, dev, N, n_factors, ftype, fa, fb, NULL, 0);
}

int plan_build_with_order(plan_t *pl, asam_dev_t *dev, int N, int n_factors, const int *ftype, const int *fa,
                          const int *fb, const int *order_keep, int N_keep)
{
    int *keep = malloc(sizeof(int) * (size_t) (N_keep > 0 ? N_keep : 1));
    memcpy(keep, order_keep, sizeof(int) * (size_t) N_keep);
    int rc = plan_build_impl(pl, dev, N, n_factors, ftype, fa, fb, keep, N_keep);
    free(keep);
    return rc;
}

/* ---- incremental append ------------------------------------------------------------------- */
int plan_append(plan_t *pl, asam_dev_t *dev, int N, int n_factors, const int *ftype, const int *fa, const int *fb,
                const int *marked_old, int n_marked, int **tasks_out, int **nwait_out, int **keep_out, int *ntasks_out)
{
    const int N0 = pl->N, F0 = pl->n_factors, nsn0 = pl->nsn;
    double pp_t0 = pp_now();
    *tasks_out = *nwait_out = NULL;
    if (keep_out)
        *keep_out = NULL;
    *ntasks_out = 0;
    for (int f = F0; f < n_factors; f++) {
        if (asam_two_pose_type(ftype[f])) {
            if (fa[f] == fb[f] || fa[f] < 0 || fb[f] < 0 || fa[f] >= N || fb[f] >= N) {
                asam_set_error("factor %d: bad node ids (%d,%d)", f, fa[f], fb[f]);
                return 1;
            }
            if (fa[f] < N0 && fb[f] < N0)
                return 2; /* edge between two old poses: structure of old rows changes */
        } else if (ftype[f] == APRIL_GRAPH_FACTOR_XYTPOS_TYPE) {
            if (fa[f] < 0 || fa[f] >= N) {
                asam_set_error("factor %d: bad node id %d", f, fa[f]);
                return 1;
            }
        } else {
            asam_set_error("factor %d: unsupported factor type %d", f, ftype[f]);
            return 1;
        }
    }

    if (pl->world > 1) {
        asam_set_error("a batch solve sharded over %d GPUs cannot be continued incrementally (replicas only)", pl->world);
        return 1;
    }
    /* incremental steps grow supernodes: the per-block entries of the batch schedule's back-solve list are
     * replaced by one entry per supernode (parents first = descending id) once, at the first append */
    if (pl->bt_split) {
        int *plain = malloc(sizeof(int) * (size_t) (nsn0 + 1));
        for (int sx = 0; sx < nsn0; sx++)
            plain[sx] = nsn0 - 1 - sx;
        free(pl->btasks);
        pl->btasks = plain;
        pl->n_btasks = nsn0;
        pl->bt_split = 0;
        pl->n_bs_leaf = 0;
        if (dev && (asam_set_full_tasks(dev, pl->ntasks, pl->tasks, pl->nwait, pl->n_btasks, pl->btasks) ||
                    asam_set_bs_leaf_count(dev, 0)))
            return 1;
    }
    /* incremental steps run the whole schedule through k_factor / k_backsolve */
    if (pl->n_leaf > 0) {
        pl->n_leaf = 0;
        if (dev && asam_set_leaf_tasks(dev, 0, NULL))
            return 1;
    }

    /* grow node-indexed arrays: new poses are eliminated last, in id order */
    node_arrays_reserve(pl, N);
    fslot_reserve(pl, n_factors);
    const int nnew = N - N0;
    sn_arrays_reserve(pl, nsn0 + nnew);
    for (int i = N0; i < N; i++) {
        pl->order[i] = i;
        pl->pos[i] = i;
        pl->node2q[i] = i;
        pl->q2node[i] = i;
        pl->parent_pos[i] = -1;
        pl->sn_of_q[i] = -1; /* assigned below: joins the root supernode or gets a new one */
    }

    /* new Hessian slots */
    const int slot0 = pl->n_slots;
    ivec_t nlo = { 0 }, nhi = { 0 };
    for (int f = F0; f < n_factors; f++) {
        if (!asam_two_pose_type(ftype[f])) {
            pl->fslot[f] = -1;
            continue;
        }
        int a = fa[f], b = fb[f], lo = a < b ? a : b, hi = a < b ? b : a, created;
        int slot = pairmap_get_or_add(&pl->pairs, lo, hi, pl->n_slots, &created);
        if (created) {
            ivec_push(&nlo, lo);
            ivec_push(&nhi, hi);
            pl->n_slots++;
        }
        pl->fslot[f] = slot;
    }

    /* marked supernodes, ascending id (= children first) */
    int *msn = malloc(sizeof(int) * (size_t) (n_marked + 1));
    int nm = 0;
    for (int i = 0; i < n_marked; i++)
        if (marked_old[i] < N0)
            msn[nm++] = pl->sn_of_q[pl->node2q[marked_old[i]]];
    nm = sort_unique(msn, nm);
    /* sn -> index in msn or -1: kept across steps, all -1 between them (an O(nsn) fill per step is what made the
     * reference's incremental steps grow with the graph, SURVEY.md quirk 13) */
    if (pl->sn_cap > pl->mark_cap) {
        pl->mark_idx = realloc(pl->mark_idx, sizeof(int) * (size_t) pl->sn_cap);
        for (int s = pl->mark_cap; s < pl->sn_cap; s++)
            pl->mark_idx[s] = -1;
        pl->mark_cap = pl->sn_cap;
    }
    int *mark_idx = pl->mark_idx;
    for (int i = 0; i < nm; i++)
        mark_idx[msn[i]] = i;

    /* Partial re-factorisation: the columns of a marked supernode BEFORE its first marked pose are
     * unchanged by this step (their Hessian entries, their children and -- because a new pose reaches an
     * old column only through a marked one -- their rows), so the kernel keeps them (L and y) and
     * re-eliminates from the first marked column on.  keepb[i] = poses kept of marked supernode i,
     * oldmb[i] = its block rows before this step (the retained front still has that layout). */
    int *keepb = malloc(sizeof(int) * (size_t) (nm + 1)), *oldmb = malloc(sizeof(int) * (size_t) (nm + 1));
    for (int i = 0; i < nm; i++) {
        keepb[i] = pl->desc[msn[i]].cb;
        oldmb[i] = pl->snh[msn[i]].rows.n;
    }
    for (int i = 0; i < n_marked; i++)
        if (marked_old[i] < N0) {
            int q = pl->node2q[marked_old[i]], sidx = mark_idx[pl->sn_of_q[q]];
            int k = q - pl->desc[msn[sidx]].first;
            if (k < keepb[sidx])
                keepb[sidx] = k;
        }

    int rc = 0, bs_leaf_broken = 0;
    ivec_t *gain = calloc((size_t) nm + 1, sizeof(ivec_t));
    ivec_t *pend = calloc((size_t) nnew + 1, sizeof(ivec_t)); /* children of each new supernode */
    ivec_t *nbelow = calloc((size_t) nnew + 1, sizeof(ivec_t));

    /* seed gains with the new edges (old pose, new pose); new-new edges seed nbelow */
    for (int k = 0; k < nlo.n; k++) {
        int lo = nlo.p[k], hi = nhi.p[k];
        if (lo < N0) {
            int s = pl->sn_of_q[pl->node2q[lo]];
            if (mark_idx[s] < 0) {
                asam_set_error("plan_append: pose %d gets a new factor but is not marked", lo);
                rc = 1;
                goto done;
            }
            ivec_push(&gain[mark_idx[s]], hi);
        } else {
            ivec_push(&nbelow[lo - N0], hi);
        }
    }

    /* propagate gains up the marked sub-forest; grow row lists; re-place fronts */
    for (int i = 0; i < nm; i++) {
        int s = msn[i];
        sn_host_t *h = &pl->snh[s];
        asam_sn_desc_t *d = &pl->desc[s];
        for (int c = 0; c < h->children.n; c++) {
            int ci = mark_idx[h->children.p[c]];
            if (ci >= 0)
                for (int e = 0; e < gain[ci].n; e++)
                    ivec_push(&gain[i], gain[ci].p[e]);
        }
        gain[i].n = sort_unique(gain[i].p, gain[i].n);
        int old_mb = h->rows.n;
        for (int e = 0; e < gain[i].n; e++)
            ivec_push(&h->rows, gain[i].p[e]); /* new poses sort after every old row */
        d->mb = h->rows.n;
        if (3 * d->mb > pl->max_m)
            pl->max_m = 3 * d->mb;
        if (pl->n_bs_leaf > 0 && pl->bs_leaf[s] && 3 * (d->mb - d->cb) > ASAM_BSLEAF_MAX)
            bs_leaf_broken = 1; /* outgrew the warp kernel: everything goes through k_backsolve from now on */
        if (d->mb != old_mb && front_doubles(d->mb) > d->reserved) {
            /* the front outgrew its allocation: move it, with head-room for the poses that
             * later steps will append (the old space is reclaimed at the next batch) */
            int slack = d->mb / 4 > 4 ? d->mb / 4 : 4;
            d->reserved = front_doubles(d->mb + slack);
            d->f_off = pl->arena_n;
            pl->arena_n += d->reserved;
            keepb[i] = 0; /* the retained columns stay behind at the old place */
        }
        if (d->parent < 0 && gain[i].n > 0) { /* old root: hangs under the first new pose */
            ivec_push(&pend[gain[i].p[0] - N0], s); /* supernode id of that pose: set below */
            int top = pl->q2node[d->first + d->cb - 1];
            pl->parent_pos[pl->pos[top]] = gain[i].p[0]; /* pos == q == id for new poses */
        }
    }
    /* gather-list entries for the new (old,new) blocks */
    for (int k = 0; k < nlo.n; k++) {
        int lo = nlo.p[k], hi = nhi.p[k];
        if (lo >= N0)
            continue;
        int s = pl->sn_of_q[pl->node2q[lo]];
        sn_host_t *h = &pl->snh[s];
        int rb = find_sorted(h->rows.p, h->rows.n, hi);
        if (rb < 0) {
            asam_set_error("plan_append: internal (row %d not in supernode %d)", hi, s);
            rc = 1;
            goto done;
        }
        ivec_push(&h->a_slot, slot0 + k);
        ivec_push(&h->a_rb, rb); /* early = lo = lower id: no transpose */
        ivec_push(&h->a_cb, pl->node2q[lo] - pl->desc[s].first);
    }

    /* new poses, ascending.  A pose whose predecessor in the order tops a root supernode with
     * exactly the structure {pose} + below(pose) becomes one more COLUMN of that supernode
     * (fundamental merge) -- otherwise every step would add one more link to the chain at the top
     * of the tree; any other pose starts a singleton supernode. */
    int *nsid = malloc(sizeof(int) * (size_t) (nnew + 1));
    int ncreated = 0;
    for (int j = 0; j < nnew; j++) {
        int n = N0 + j;
        ivec_t *bel = &nbelow[j];
        int lvl = 0;
        for (int c = 0; c < pend[j].n; c++) {
            int X = pend[j].p[c];
            const sn_host_t *hx = &pl->snh[X];
            for (int e = pl->desc[X].cb; e < hx->rows.n; e++)
                if (hx->rows.p[e] != n)
                    ivec_push(bel, hx->rows.p[e]);
            if (pl->desc[X].level + 1 > lvl)
                lvl = pl->desc[X].level + 1;
        }
        bel->n = sort_unique(bel->p, bel->n);
        int R = n > 0 ? pl->sn_of_q[n - 1] : -1, sid = -1;
        if (R >= 0 && pl->desc[R].cb < MAX_SN_COLS && pl->desc[R].first + pl->desc[R].cb == n &&
            pl->snh[R].rows.n - pl->desc[R].cb == 1 + bel->n) {
            for (int c = 0; c < pend[j].n; c++)
                if (pend[j].p[c] == R)
                    sid = R;
        }
        if (sid >= 0) { /* n joins R: the row list already holds n right after R's columns */
            asam_sn_desc_t *d = &pl->desc[R];
            sn_host_t *h = &pl->snh[R];
            d->cb += 1;
            if (pl->n_bs_leaf > 0 && pl->bs_leaf[R] && 3 * d->cb > ASAM_BSLEAF_MAX)
                bs_leaf_broken = 1;
            for (int c = 0; c < pend[j].n; c++) {
                int X = pend[j].p[c];
                if (X == R)
                    continue;
                ivec_push(&h->children, X);
                pl->desc[X].parent = R;
            }
            if (lvl > d->level)
                d->level = lvl;
            d->parent = -1;
        } else {
            sid = pl->nsn++;
            ncreated++;
            asam_sn_desc_t *d = &pl->desc[sid];
            sn_host_t *h = &pl->snh[sid];
            memset(d, 0, sizeof(*d));
            d->first = n;
            d->cb = 1;
            d->parent = -1;
            d->level = lvl;
            h->rows.n = 0;
            ivec_push(&h->rows, n);
            for (int e = 0; e < bel->n; e++)
                ivec_push(&h->rows, bel->p[e]);
            h->children.n = 0;
            for (int c = 0; c < pend[j].n; c++) {
                ivec_push(&h->children, pend[j].p[c]);
                pl->desc[pend[j].p[c]].parent = sid;
            }
            h->a_slot.n = h->a_rb.n = h->a_cb.n = 0;
            d->mb = h->rows.n;
            if (3 * d->mb > pl->max_m)
                pl->max_m = 3 * d->mb;
            d->reserved = front_doubles(d->mb + 4);
            d->f_off = pl->arena_n;
            pl->arena_n += d->reserved;
        }
        nsid[j] = sid;
        pl->sn_of_q[n] = sid;
        if (bel->n > 0) {
            ivec_push(&pend[bel->p[0] - N0], sid);
            pl->parent_pos[n] = bel->p[0];
        }
        if (pl->desc[sid].level + 1 > pl->n_levels)
            pl->n_levels = pl->desc[sid].level + 1;
    }
    for (int k = 0; k < nlo.n; k++) { /* (new,new) blocks */
        int lo = nlo.p[k], hi = nhi.p[k];
        if (lo < N0)
            continue;
        int s = nsid[lo - N0];
        sn_host_t *h = &pl->snh[s];
        int rb = find_sorted(h->rows.p, h->rows.n, hi);
        if (rb < 0) {
            asam_set_error("plan_append: internal (row %d not in new supernode %d)", hi, s);
            rc = 1;
            free(nsid);
            goto done;
        }
        ivec_push(&h->a_slot, slot0 + k);
        ivec_push(&h->a_rb, rb);
        ivec_push(&h->a_cb, lo - pl->desc[s].first);
    }

    /* relative indices + segments of everything that changed */
    {
        int nt = nm + ncreated;
        int *tasks = malloc(sizeof(int) * (size_t) (nt + 1)), *nwait = malloc(sizeof(int) * (size_t) (nt + 1));
        int *keep = calloc((size_t) nt + 1, sizeof(int));
        for (int i = 0; i < nm; i++) {
            tasks[i] = msn[i];
            if (keepb[i] > 0 && keepb[i] < 0x7fff && oldmb[i] < 0xffff)
                keep[i] = (keepb[i] << 16) | oldmb[i];
        }
        for (int k = 0; k < ncreated; k++) { /* created supernodes have ids nsn0 .. nsn0+ncreated-1 */
            tasks[nm + k] = nsn0 + k;
            mark_idx[nsn0 + k] = nm + k;
        }
        for (int j = 0; j < nnew; j++) /* a pose may have joined a supernode that was not marked */
            if (mark_idx[nsid[j]] < 0) {
                asam_set_error("plan_append: pose %d joined unmarked supernode %d", N0 + j, nsid[j]);
                rc = 1;
            }
        free(nsid);
        ivec_t seg = { 0 };
        for (int t = 0; t < nt && !rc; t++)
            rc |= compute_rel(pl, tasks[t]);
        for (int t = 0; t < nt && !rc; t++) {
            int s = tasks[t], w = 0;
            for (int c = 0; c < pl->snh[s].children.n; c++)
                if (mark_idx[pl->snh[s].children.p[c]] >= 0)
                    w++;
            nwait[t] = pack_nwait(w, 0, 0);
            emit_segment(pl, s, &seg, pl->ipool_n);
        }
        if (!rc) {
            ivec_reserve(&pl->ipool_host, pl->ipool_host.n + seg.n);
            memcpy(pl->ipool_host.p + pl->ipool_host.n, seg.p, sizeof(int) * (size_t) seg.n);
            pl->ipool_host.n += seg.n;
        }
        if (!rc && !dev)
            pl->ipool_n += seg.n;
        if (!rc && !dev && bs_leaf_broken) /* (with a device: below, together with the device's count) */
            pl->n_bs_leaf = 0;
        g_plan_prof[0] += pp_now() - pp_t0; /* host symbolic */
        pp_t0 = pp_now();
        if (!rc && dev) {
            int64_t ipool_need = pl->ipool_n + seg.n;
            rc = asam_reserve(dev, N + 64, n_factors + 64, pl->n_slots + 64, pl->nsn + 64, ipool_need + ipool_need / 2,
                              pl->arena_n + pl->arena_n / 4);
            g_plan_prof[1] += pp_now() - pp_t0; /* asam_reserve */
            pp_t0 = pp_now();
            asam_sn_desc_t *dd = malloc(sizeof(asam_sn_desc_t) * (size_t) (nt + 1));
            for (int t = 0; t < nt; t++)
                dd[t] = pl->desc[tasks[t]];
            if (!rc)
                rc |= asam_upload_ipool(dev, pl->ipool_n, seg.n, seg.p);
            if (!rc)
                rc |= asam_upload_desc(dev, nt, tasks, dd);
            if (!rc && nnew > 0) {
                rc |= asam_upload_node2q(dev, N0, nnew, pl->node2q + N0);
                rc |= asam_upload_q2node(dev, N0, nnew, pl->q2node + N0);
            }
            if (!rc && ncreated > 0) { /* new supernodes are ancestors of all older ones */
                int *pre = malloc(sizeof(int) * (size_t) ncreated);
                for (int k = 0; k < ncreated; k++)
                    pre[k] = nsn0 + ncreated - 1 - k;
                rc |= asam_btasks_prepend(dev, ncreated, pre);
                free(pre);
            }
            if (!rc && bs_leaf_broken) {
                pl->n_bs_leaf = 0;
                rc |= asam_set_bs_leaf_count(dev, 0);
            }
            if (!rc)
                rc |= asam_upload_fslot(dev, F0, n_factors - F0, pl->fslot + F0);
            if (!rc)
                rc |= asam_hessian_clear_range(dev, N0, nnew, slot0, pl->n_slots - slot0);
            free(dd);
            pl->ipool_n += seg.n;
            g_plan_prof[2] += pp_now() - pp_t0; /* uploads */
        }
        ivec_free(&seg);
        if (rc) {
            free(tasks);
            free(nwait);
            free(keep);
        } else {
            /* expand big fronts into teams of consecutive entries */
            int total = 0;
            for (int t = 0; t < nt; t++)
                total += team_size(pl->desc[tasks[t]].mb, pl->desc[tasks[t]].cb, plan_team_cap(pl));
            if (total != nt) {
                int *t2 = malloc(sizeof(int) * (size_t) total), *w2 = malloc(sizeof(int) * (size_t) total);
                int *k2 = calloc((size_t) total, sizeof(int)); /* teams re-factor whole fronts */
                int k = 0;
                for (int t = 0; t < nt; t++) {
                    int G = team_size(pl->desc[tasks[t]].mb, pl->desc[tasks[t]].cb, plan_team_cap(pl));
                    for (int w = 0; w < G; w++, k++) {
                        t2[k] = tasks[t];
                        w2[k] = pack_nwait(nwait[t], w, G > 1 ? G : 0);
                        k2[k] = G > 1 ? 0 : keep[t];
                    }
                }
                free(tasks);
                free(nwait);
                free(keep);
                tasks = t2;
                nwait = w2;
                keep = k2;
                nt = total;
            }
            *tasks_out = tasks;
            *nwait_out = nwait;
            if (keep_out)
                *keep_out = keep;
            else
                free(keep);
            *ntasks_out = nt;
        }
    }
    pl->N = N;
    pl->n_factors = n_factors;
    pl->struct_hash = 0; /* appended order: never to be reused by a batch solve (it re-orders) */

done:
    for (int i = 0; i < nm; i++)
        ivec_free(&gain[i]);
    for (int j = 0; j < nnew; j++) {
        ivec_free(&pend[j]);
        ivec_free(&nbelow[j]);
    }
    for (int i = 0; i < nm; i++)
        mark_idx[msn[i]] = -1;
    for (int sx = nsn0; sx < nsn0 + nnew && sx < pl->mark_cap; sx++)
        mark_idx[sx] = -1;
    free(gain);
    free(pend);
    free(nbelow);
    free(msn);
    free(keepb);
    free(oldmb);
    ivec_free(&nlo);
    ivec_free(&nhi);
    return rc;
}
