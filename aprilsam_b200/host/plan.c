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
            double t0 = pp_now();
            host_spin(iters);
            const double t1 = pp_now() - t0;
            double tp = 1e30;
            for (int rep = 0; rep < 3 && tp > 2.5 * t1 + 0.05; rep++) { /* (the first region also creates the threads) */
                t0 = pp_now();
#pragma omp parallel num_threads(2)
                host_spin(iters);
                const double t = pp_now() - t0;
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
 * (team_sizes).  ASAM_SOLO_MAX_M overrides (tuning). */
static int solo_max_m(void)
{
    static int v = -1;
    if (v < 0) {
        const char *e = getenv("ASAM_SOLO_MAX_M");
        v = e ? atoi(e) : ASAM_SOLO_MAX_M_DEFAULT;
    }
    return v;
}

/* Returns the team word of a front, the G field of its task word (pack_nwait): 0 = one CTA on cta_front,
 * >= 2 = a team of G CTAs (team_front); team_sizes() may also scale a team to 1 = team_front on one CTA. */
static int team_size(int mb, int cb, int cap)
{
    int64_t m = 3 * (int64_t) mb, c = 3 * (int64_t) cb;
    if (front_fits_smem(mb) || m <= solo_max_m())
        return 0;
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

/* CTAs (= consecutive task entries) of a front of team word G */
static inline int front_ctas(int G) { return G > 1 ? G : 1; }

static int plan_team_cap(const plan_t *pl) { return pl->max_team > 0 ? pl->max_team : 120; }

/* doubles of the arena a front of mb block rows occupies: the front itself and, for fronts that do not fit
 * in shared memory (team path), the two row-major panel buffers behind it (asam_kernels.cuh, ASAM_LDW) */
static int64_t front_doubles(int mb)
{
    int64_t m = 3 * (int64_t) mb;
    return (int64_t) ASAM_LD(m) * m + (front_fits_smem(mb) ? 0 : 2 * (m + 2) * 52);
}

/* ---- schedule: task lists of one batch solve ------------------------------------------------
 * Single GPU (world == 1): leaf set -> k_factor_leaf, everything else -> k_factor (ticket order of
 * factor_order(), teams expanded), back-solve list = [rest | leaf set], parents first.
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

/* out[0 .. n) = 0 .. n-1 by descending key, ties by ascending id */
static void order_desc(const double *key, int n, int *out)
{
    sn_key_t *keys = malloc(sizeof(sn_key_t) * (size_t) (n + 1));
    for (int s = 0; s < n; s++) {
        keys[s].key = key[s];
        keys[s].id = s;
    }
    qsort(keys, (size_t) n, sizeof(sn_key_t), cmp_key_desc);
    for (int k = 0; k < n; k++)
        out[k] = keys[k].id;
    free(keys);
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

/* g: the team word (team_size()) */
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
static int sim_order(const plan_t *pl, const char *in, const int *G, const double *lat, const double *prio, int P, int *out)
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
            int s = ready[0].id, g = front_ctas(G[s]) < P ? front_ctas(G[s]) : P;
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
            int s = e.id, g = front_ctas(G[s]) < P ? front_ctas(G[s]) : P;
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

/* owner[s]: rank that factors s, -1 = top (every rank).  Several ranks: the cut and the shard descriptors of pl. */
static int *shard_cut(plan_t *pl, int W)
{
    const int nsn = pl->nsn;
    free(pl->shard_owner); free(pl->shard_off); free(pl->shard_cnt); free(pl->shard_q0); free(pl->shard_qn);
    pl->shard_owner = pl->shard_q0 = pl->shard_qn = NULL;
    pl->shard_off = pl->shard_cnt = NULL;
    pl->n_shards = 0;
    int *owner = calloc((size_t) nsn + 1, sizeof(int));
    if (W <= 1 || nsn == 0)
        return owner;
    double *sub = malloc(sizeof(double) * (size_t) nsn); /* work of the subtree rooted at s */
    for (int s = 0; s < nsn; s++)
        sub[s] = sn_work(&pl->desc[s]);
    for (int s = 0; s < nsn; s++) /* children have smaller ids */
        if (pl->desc[s].parent >= 0)
            sub[pl->desc[s].parent] += sub[s];
    /* frontier of subtree roots; split the heaviest until the shards can be balanced */
    int *fr = malloc(sizeof(int) * (size_t) (nsn + 1)), nfr = 0;
    for (int s = 0; s < nsn; s++)
        if (pl->desc[s].parent < 0)
            fr[nfr++] = s;
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
    return owner;
}

/* Returns the factor leaf set; sets the back-solve leaf set (pl->bs_leaf, pl->n_bs_leaf). */
static char *leaf_sets(plan_t *pl, const int *owner, int me)
{
    const int nsn = pl->nsn;
    /* factor leaf set: supernodes whose whole subtree consists of fronts small enough for the
     * warp-per-front kernels (children have smaller ids).  Only worth separate launches when
     * there are thousands of them. */
    char *leaf = calloc((size_t) nsn + 1, 1);
    int n_leaf = 0;
    const int leaf_max = leaf_max_m_for(nsn);
    for (int s = 0; s < nsn; s++) {
        int ok = 3 * pl->desc[s].mb <= leaf_max;
        for (int c = 0; ok && c < pl->snh[s].children.n; c++)
            ok = leaf[pl->snh[s].children.p[c]];
        leaf[s] = (char) ok;
        n_leaf += ok;
    }
    if (n_leaf < ASAM_LEAF_MIN_COUNT)
        memset(leaf, 0, (size_t) nsn);
    /* the warp-per-supernode BACK-SOLVE takes any downward-closed set with <= 64 own columns and
     * <= 64 rows below (a superset of the factor leaf set); it pays from a few dozen supernodes on:
     * a warp per supernode has everything fetched before its parent's flag arrives */
    free(pl->bs_leaf);
    pl->bs_leaf = calloc((size_t) pl->sn_cap + 1, 1);
    int n_bsl = 0;
    for (int s = 0; s < nsn; s++) {
        int ok = 3 * pl->desc[s].cb <= ASAM_BSLEAF_MAX && 3 * (pl->desc[s].mb - pl->desc[s].cb) <= ASAM_BSLEAF_MAX;
        for (int c = 0; ok && c < pl->snh[s].children.n; c++)
            ok = pl->bs_leaf[pl->snh[s].children.p[c]];
        pl->bs_leaf[s] = (char) ok;
        n_bsl += ok && owner[s] == me;
    }
    if (n_bsl < ASAM_BSLEAF_MIN_COUNT) {
        memset(pl->bs_leaf, 0, (size_t) nsn);
        n_bsl = 0;
    }
    pl->n_bs_leaf = n_bsl;
    return leaf;
}

/* Team word of every supernode (team_size(); 0 for the leaf set and other ranks' fronts).  A front's team is bound
 * by latency, not throughput (team_size()), so where one tree level holds more team fronts than the SMs can seat
 * side by side, smaller teams finish the LEVEL sooner: CTA-time per front (G x duration) falls with G.  The teams of
 * such a level are scaled down to the room there is. */
static int *team_sizes(const plan_t *pl, const int *owner, int me, const char *leaf)
{
    const int nsn = pl->nsn;
    int *G = malloc(sizeof(int) * (size_t) (nsn + 1));
    int64_t *want = calloc((size_t) pl->n_levels + 1, sizeof(int64_t));
    for (int s = 0; s < nsn; s++) {
        G[s] = (owner[s] == me || owner[s] == -1) && !leaf[s] ? team_size(pl->desc[s].mb, pl->desc[s].cb, plan_team_cap(pl)) : 0;
        if (G[s] >= 2)
            want[pl->desc[s].level] += G[s];
    }
    int64_t room = ASAM_TEAM_ROOM < plan_team_cap(pl) ? ASAM_TEAM_ROOM : plan_team_cap(pl);
    const char *er = getenv("ASAM_TEAM_ROOM"); /* tuning knob (tools only) */
    if (er && atoi(er) > 0)
        room = atoi(er);
    /* A front scaled below a team of two is factored by ONE CTA on cta_front's HBM path (word 0): it pays where a
     * level holds far more team fronts than SMs (the SM time per front is what limits the level, not its latency),
     * and one CTA needs none of the team protocol.  ASAM_TEAM_MIN=g (A/B) sets the smallest team instead; with
     * g = 1 such fronts run the team code alone (word 1). */
    int gmin = 0;
    const char *em = getenv("ASAM_TEAM_MIN");
    if (em && atoi(em) >= 1)
        gmin = atoi(em);
    for (int s = 0; s < nsn; s++) {
        int64_t w = want[pl->desc[s].level];
        if (G[s] >= 2 && w > room) {
            int g = (int) ((int64_t) G[s] * room / w);
            g = g < gmin ? gmin : g;
            G[s] = g >= 2 || gmin == 1 ? g : 0;
        }
    }
    free(want);
    return G;
}

/* Ticket order of k_factor (returned: every supernode once; the task lists take theirs in this order).  The
 * persistent kernels hand out tasks in list order, so the list IS the schedule.  Plain level order (every front
 * of level l before any of level l+1) starts the deepest chain of the tree last among its level-mates and leaves
 * its top to run alone at the end, with most SMs spinning.  Critical-path-first instead ("cp"): fronts are listed
 * by DESCENDING length of the dependent chain from them up to the root (their own modelled latency included),
 * which is still a topological order -- a child's chain is its parent's plus its own -- so a waiting CTA only ever
 * waits for tasks that were handed out before its own.  Where the SMs are saturated, the simulated schedule
 * ("sim", sim_order()) instead.  ASAM_TASK_ORDER=cp|sim forces one of the two. */
static int *factor_order(const plan_t *pl, const int *owner, int me, const char *leaf, const int *G)
{
    const int nsn = pl->nsn;
    const char *eo = getenv("ASAM_TASK_ORDER");
    const int force_cp = eo && strcmp(eo, "cp") == 0, force_sim = eo && strcmp(eo, "sim") == 0;
    /* modelled duration of every front once its children are done (microseconds; least-squares fit to device
     * traces of the 100 k world, tools/panel_trace.py --dump-trace: median error 8 % for shared-memory fronts,
     * 9 % for teams) and the length of the dependent chain from a front up to the root */
    double *lat_us = malloc(sizeof(double) * (size_t) (nsn + 1)), *up_us = malloc(sizeof(double) * (size_t) (nsn + 1));
    double work = 0.0, chain = 0.0;
    team_model_init();
    for (int s = nsn - 1; s >= 0; s--) { /* parents have larger ids */
        const double lat = front_lat_us(pl, s, G[s]);
        lat_us[s] = lat;
        up_us[s] = lat + (pl->desc[s].parent >= 0 ? up_us[pl->desc[s].parent] : 0.0);
        if ((owner[s] == me || owner[s] == -1) && !leaf[s])
            work += lat * front_ctas(G[s]);
        if (up_us[s] > chain)
            chain = up_us[s];
    }
    const int P = pl->n_cta > 0 ? pl->n_cta : 132;
    /* auto: where the SMs are far from saturated (M3500: 11 of 67 CTA-ms busy) spinning costs nothing and the
     * eager chain-length order starts parents soonest; where they are saturated, a team must not take its
     * CTAs before it can use them */
    const int use_sim = force_sim || (!force_cp && work / P > 0.5 * chain);
    int *ord = malloc(sizeof(int) * (size_t) (nsn + 1));
    order_desc(up_us, nsn, ord);
    if (use_sim) {
        /* ticket order of k_factor = start order of the simulated schedule; the main list (own fronts outside
         * the leaf set) and the part above a multi-GPU cut are separate launches, simulated separately; the
         * leaf set keeps the chain-length order (warp-sized tasks: nothing to gather) */
        char *in = calloc((size_t) nsn + 1, 1);
        int *sim = malloc(sizeof(int) * (size_t) (nsn + 1)), n;
        for (int s = 0; s < nsn; s++)
            in[s] = owner[s] == me && !leaf[s];
        n = sim_order(pl, in, G, lat_us, up_us, P, sim);
        for (int s = 0; s < nsn; s++)
            in[s] = owner[s] == -1;
        n += sim_order(pl, in, G, lat_us, up_us, P, sim + n);
        /* simulated tasks in start order, everything else (leaf set, other ranks) after them in chain-length order */
        memset(in, 0, (size_t) nsn);
        for (int k = 0; k < n; k++)
            in[sim[k]] = 1;
        for (int k = 0; k < nsn; k++)
            if (!in[ord[k]])
                sim[n++] = ord[k];
        free(ord);
        free(in);
        ord = sim;
    }
    free(lat_us);
    free(up_us);
    return ord;
}

/* Back-solve order (returned), parents first: by the modelled TIME of the longest chain below a supernode (its own
 * solve included), longest first -- a parent's chain is longer than any child's, so the order is topological, and
 * the deep chains do not queue behind the thousands of supernodes that merely share their height (level order: the
 * bottom of the longest chain of the 100 k world got its tickets late at every link). */
static int *backsolve_order(const plan_t *pl)
{
    const int nsn = pl->nsn;
    double *down = calloc((size_t) nsn + 1, sizeof(double));
    int *ord = malloc(sizeof(int) * (size_t) (nsn + 1));
    for (int s = 0; s < nsn; s++) { /* children have smaller ids: down[s] holds max over children here */
        if (!pl->bs_leaf[s]) /* (the warp-per-supernode set runs in a launch of its own, afterwards) */
            down[s] += 5.0 + 0.17 * 3.0 * pl->desc[s].cb + 0.01 * 3.0 * pl->desc[s].mb;
        else
            down[s] += 1e-3 * (pl->desc[s].level + 1);
        const int par = pl->desc[s].parent;
        if (par >= 0 && down[s] > down[par])
            down[par] = down[s];
    }
    order_desc(down, nsn, ord);
    free(down);
    return ord;
}

/* Back-solve entries of a supernode in a batch schedule: one, or -- supernodes wider than one 96-column block
 * (ASAM_BSW) -- one per block, each solved by its own CTA (cta_backsolve, blk_only).  Entry word:
 * supernode | (block + 1) << 24. */
static int bs_nblk(const plan_t *pl, int s)
{
    const int c = 3 * pl->desc[s].cb;
    return !pl->bs_leaf[s] && c > 96 && pl->nsn < (1 << 24) ? (c + 95) / 96 : 1;
}

/* Writes the front_ctas(G) task entries of front s (workers 0 .. G-1 of a team, consecutive); returns their number. */
static int emit_front(int *tasks, int *nwait, int s, int nw, int G)
{
    const int n = front_ctas(G);
    for (int w = 0; w < n; w++) {
        tasks[w] = s;
        nwait[w] = pack_nwait(nw, w, G);
    }
    return n;
}

/* The task lists of this rank: leaf_tasks (k_factor_leaf), tasks/nwait (k_factor: own fronts outside the leaf set)
 * and top_tasks/top_nwait (k_factor: the fronts above a multi-GPU cut), each in the ticket order `tick`; btasks =
 * [top | own shards outside the back-solve leaf set | that set], each segment in the back-solve order `bso`. */
static void emit_lists(plan_t *pl, const int *owner, int me, const char *leaf, const int *G, const int *tick,
                       const int *bso)
{
    const int nsn = pl->nsn;
    free(pl->tasks); free(pl->nwait); free(pl->btasks); free(pl->leaf_tasks); free(pl->top_tasks); free(pl->top_nwait);
    int n_local = 0, n_top = 0, n_leaf = 0, n_top_sn = 0, n_main_bt = 0, n_top_bt = 0;
    for (int s = 0; s < nsn; s++) {
        if (owner[s] == me) {
            if (leaf[s])
                n_leaf++;
            else
                n_local += front_ctas(G[s]);
            if (!pl->bs_leaf[s])
                n_main_bt += bs_nblk(pl, s);
        } else if (owner[s] == -1) {
            n_top += front_ctas(G[s]);
            n_top_sn++;
            n_top_bt += bs_nblk(pl, s);
        }
    }
    pl->ntasks = n_local;
    pl->tasks = malloc(sizeof(int) * (size_t) (n_local + 1));
    pl->nwait = malloc(sizeof(int) * (size_t) (n_local + 1));
    pl->n_leaf = n_leaf;
    pl->leaf_tasks = malloc(sizeof(int) * (size_t) (n_leaf + 1));
    pl->n_top = n_top;
    pl->n_top_sn = n_top_sn;
    pl->top_tasks = malloc(sizeof(int) * (size_t) (n_top + 1));
    pl->top_nwait = malloc(sizeof(int) * (size_t) (n_top + 1));
    pl->n_btasks = n_top_bt + n_main_bt + pl->n_bs_leaf;
    pl->btasks = malloc(sizeof(int) * (size_t) (pl->n_btasks + 1));
    pl->bt_split = 0;
    int at[3] = { 0, n_top_bt, n_top_bt + n_main_bt }; /* next entry of each back-solve segment */
    for (int k = 0; k < nsn; k++) {
        const int s = bso[k];
        if (owner[s] != me && owner[s] != -1)
            continue;
        const int seg = owner[s] == -1 ? 0 : pl->bs_leaf[s] ? 2 : 1, nb = bs_nblk(pl, s);
        for (int b = nb - 1; b >= 0; b--) /* the last block first */
            pl->btasks[at[seg]++] = nb > 1 ? (s | ((b + 1) << 24)) : s;
        pl->bt_split |= nb > 1;
    }
    int t = 0, tl = 0, tt = 0;
    for (int k = 0; k < nsn; k++) {
        const int s = tick[k];
        if (owner[s] == -1) {
            int nw = 0; /* children above the cut: the others were exchanged before this launch */
            for (int c = 0; c < pl->snh[s].children.n; c++)
                nw += owner[pl->snh[s].children.p[c]] == -1;
            tt += emit_front(pl->top_tasks + tt, pl->top_nwait + tt, s, nw, G[s]);
        } else if (owner[s] == me && leaf[s]) {
            pl->leaf_tasks[tl++] = s;
        } else if (owner[s] == me) { /* nwait counts ALL children: those of the leaf set arrived in the earlier launch */
            t += emit_front(pl->tasks + t, pl->nwait + t, s, pl->desc[s].ch_cnt, G[s]);
        }
    }
}

static void build_schedule(plan_t *pl)
{
    const int me = pl->world > 1 ? pl->rank : 0;
    int *owner = shard_cut(pl, pl->world > 1 ? pl->world : 1);
    char *leaf = leaf_sets(pl, owner, me);
    int *G = team_sizes(pl, owner, me, leaf);
    int *tick = factor_order(pl, owner, me, leaf, G);
    int *bso = backsolve_order(pl);
    emit_lists(pl, owner, me, leaf, G, tick, bso);
    free(bso);
    free(tick);
    free(G);
    free(leaf);
    free(owner);
}

/* ---- decisions shared by the batch build and the incremental append ------------------------------ */
/* Factors [f0, n_factors) on poses [0, N): a prior on one pose, or a two-pose factor on two distinct poses.  Returns 0,
 * 1 (error text set), or 2 for a two-pose factor between two poses below N0, which no incremental step can append. */
static int check_factors(int f0, int n_factors, int N, int N0, const int *ftype, const int *fa, const int *fb)
{
    for (int f = f0; f < n_factors; f++) {
        if (asam_two_pose_type(ftype[f])) {
            if (fa[f] == fb[f] || fa[f] < 0 || fb[f] < 0 || fa[f] >= N || fb[f] >= N) {
                asam_set_error("factor %d: bad node ids (%d,%d)", f, fa[f], fb[f]);
                return 1;
            }
            if (fa[f] < N0 && fb[f] < N0)
                return 2;
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
    return 0;
}

/* Hessian slots of the checked factors [f0, n_factors): one per distinct pose pair, -1 for a prior.  The pairs that
 * get a new slot are appended to (plo, phi) in slot order. */
static void assign_slots(plan_t *pl, int f0, int n_factors, const int *ftype, const int *fa, const int *fb, ivec_t *plo,
                         ivec_t *phi)
{
    fslot_reserve(pl, n_factors);
    for (int f = f0; f < n_factors; f++) {
        if (!asam_two_pose_type(ftype[f])) {
            pl->fslot[f] = -1;
            continue;
        }
        int a = fa[f], b = fb[f], lo = a < b ? a : b, hi = a < b ? b : a, created;
        int slot = pairmap_get_or_add(&pl->pairs, lo, hi, pl->n_slots, &created);
        if (created) {
            ivec_push(plo, lo);
            ivec_push(phi, hi);
            pl->n_slots++;
        }
        pl->fslot[f] = slot;
    }
}

/* A new supernode whose one column is position q, without a parent; returns its id. */
static int sn_create(plan_t *pl, int q)
{
    sn_arrays_reserve(pl, pl->nsn + 1);
    pl->desc[pl->nsn] = (asam_sn_desc_t) { .first = q, .cb = 1, .parent = -1 };
    return pl->nsn++;
}

/* Block rows of supernode s from its row list; the largest front order follows. */
static void sn_set_mb(plan_t *pl, int s)
{
    pl->desc[s].mb = pl->snh[s].rows.n;
    if (3 * pl->desc[s].mb > pl->max_m)
        pl->max_m = 3 * pl->desc[s].mb;
}

/* Places the front of supernode s at the end of the arena, with room for a front of mb_capacity block rows. */
static void front_place(plan_t *pl, int s, int mb_capacity)
{
    pl->desc[s].f_off = pl->arena_n;
    pl->desc[s].reserved = front_doubles(mb_capacity);
    pl->arena_n += pl->desc[s].reserved;
}

/* Supernode s is in the back-solve leaf set but no longer fits k_backsolve_leaf. */
static int bs_leaf_outgrown(const plan_t *pl, int s)
{
    const asam_sn_desc_t *d = &pl->desc[s];
    return pl->n_bs_leaf > 0 && pl->bs_leaf[s] &&
           (3 * d->cb > ASAM_BSLEAF_MAX || 3 * (d->mb - d->cb) > ASAM_BSLEAF_MAX);
}

/* Where the Hessian block of poses (lo, hi) goes: the supernode of the pose eliminated first (returned), its column *cb
 * there, and *rb, the block row of the other pose (-1: none), with ASAM_TR_FLAG where the slot is read transposed. */
static int gather_find(const plan_t *pl, int lo, int hi, int *rb, int *cb)
{
    int qlo = pl->node2q[lo], qhi = pl->node2q[hi];
    int qe = qlo < qhi ? qlo : qhi, ql = qlo < qhi ? qhi : qlo;
    int s = pl->sn_of_q[qe];
    const sn_host_t *h = &pl->snh[s];
    *rb = find_sorted(h->rows.p, h->rows.n, ql) | (qe == qlo ? 0 : ASAM_TR_FLAG);
    *cb = qe - pl->desc[s].first;
    return s;
}

static void gather_push(plan_t *pl, int s, int slot, int rb, int cb)
{
    sn_host_t *h = &pl->snh[s];
    ivec_push(&h->a_slot, slot);
    ivec_push(&h->a_rb, rb);
    ivec_push(&h->a_cb, cb);
}

/* ---- batch build --------------------------------------------------------------------------- */
static void build_lap(int i, double *t)
{
    const double now = pp_now();
    g_build_prof[i] += now - *t;
    *t = now;
}

/* Empties the plan for a rebuild.  What survives it: the structure hash and where the plan runs (world, rank, the
 * largest team and the resident CTAs, re-read from `dev` when there is one). */
static void plan_reset(plan_t *pl, asam_dev_t *dev)
{
    const uint64_t hash = pl->struct_hash;
    const int world = pl->world, rank = pl->rank, max_team = pl->max_team, n_cta = pl->n_cta;
    plan_free(pl);
    pl->struct_hash = hash;
    pl->world = world, pl->rank = rank;
    pl->max_team = max_team, pl->n_cta = n_cta;
    if (dev) { /* teams are sized for the CTAs this device actually seats (MIG slice, smaller part, ...) */
        int n_sm = 0, fac_grid = 0, fac_smem = 0, bs_grid = 0;
        if (asam_device_info(dev, &n_sm, &fac_grid, &fac_smem, &bs_grid) == 0 && fac_grid > 0)
            pl->max_team = fac_grid < 120 ? fac_grid : 120, pl->n_cta = fac_grid;
    }
}

/* Adjacency of the N poses from the slots' pose pairs, CSR with ascending lists (malloc'd) */
static void adjacency(int N, const ivec_t *plo, const ivec_t *phi, int **adj_ptr_out, int **adj_out)
{
    const int S = plo->n;
    int *adj_ptr = *adj_ptr_out = calloc((size_t) N + 1, sizeof(int));
    for (int s = 0; s < S; s++) {
        adj_ptr[plo->p[s] + 1]++;
        adj_ptr[phi->p[s] + 1]++;
    }
    for (int i = 0; i < N; i++)
        adj_ptr[i + 1] += adj_ptr[i];
    int *adj = *adj_out = malloc(sizeof(int) * (size_t) (2 * S + 1)), *fill = malloc(sizeof(int) * (size_t) N);
    memcpy(fill, adj_ptr, sizeof(int) * (size_t) N);
    for (int s = 0; s < S; s++) {
        adj[fill[plo->p[s]]++] = phi->p[s];
        adj[fill[phi->p[s]]++] = plo->p[s];
    }
    for (int i = 0; i < N; i++)
        sort_ints(adj + adj_ptr[i], adj_ptr[i + 1] - adj_ptr[i]);
    free(fill);
}

/* pl->order and pl->pos: the reference's elimination order, or order_keep for the first N_keep positions and the
 * other poses after them in id order */
static void elimination_order(plan_t *pl, const int *adj_ptr, const int *adj, const int *order_keep, int N_keep)
{
    const int N = pl->N;
    if (order_keep) {
        memcpy(pl->order, order_keep, sizeof(int) * (size_t) N_keep);
        for (int p = N_keep; p < N; p++)
            pl->order[p] = p;
    } else {
        int *ord = asam_ref_ordering(N, adj_ptr, adj);
        memcpy(pl->order, ord, sizeof(int) * (size_t) N);
        free(ord);
    }
    for (int p = 0; p < N; p++)
        pl->pos[pl->order[p]] = p;
}

/* Block elimination tree in reference positions p; the parents are pl->parent_pos.  The rows below column p are
 * bl[bptr[p] .. bptr[p+1]), unsorted: only their sizes, their union and their minimum (the parent) are used, and the
 * rows of a supernode are sorted once, in numeric positions, by sn_structure().  The children of p are head[p],
 * next[head[p]], ... (-1 ends the list).  post_order() numbers the tree: qpos[p] = q, pofq[q] = p. */
typedef struct {
    int64_t *bptr;
    ivec_t bl;
    int *head, *next;
    int *qpos, *pofq;
} etree_t;

static etree_t block_symbolic(plan_t *pl, const int *adj_ptr, const int *adj)
{
    const int N = pl->N;
    int *head = malloc(sizeof(int) * (size_t) N), *tail = malloc(sizeof(int) * (size_t) N);
    int *next = malloc(sizeof(int) * (size_t) N), *stamp = calloc((size_t) N, sizeof(int));
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
        bptr[p + 1] = bl.n;
        int pmin = -1;
        for (int e = start; e < bl.n; e++)
            if (pmin < 0 || bl.p[e] < pmin)
                pmin = bl.p[e];
        pl->parent_pos[p] = pmin;
        if (pmin >= 0) { /* p is the last child of pmin so far */
            if (tail[pmin] < 0)
                head[pmin] = p;
            else
                next[tail[pmin]] = p;
            tail[pmin] = p;
        }
    }
    free(tail); free(stamp);
    return (etree_t) { .bptr = bptr, .bl = bl, .head = head, .next = next };
}

/* Post-order of the tree -> numeric positions q (t->qpos, t->pofq, pl->node2q, pl->q2node).  Children are visited in
 * ascending structure size so that the child with the largest front is numbered right before its parent and can
 * share a supernode with it (supernodes()).  Uses up the child lists. */
static void post_order(plan_t *pl, etree_t *t)
{
    const int N = pl->N;
    int *head = t->head, *next = t->next;
    const int64_t *bptr = t->bptr;
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
    }
    free(kids);
    int *qpos = t->qpos = malloc(sizeof(int) * (size_t) N), *pofq = t->pofq = malloc(sizeof(int) * (size_t) N);
    int *stack = malloc(sizeof(int) * (size_t) N), q = 0;
    for (int r = 0; r < N; r++) {
        if (pl->parent_pos[r] >= 0)
            continue;
        int sp = 0;
        stack[0] = r;
        while (sp >= 0) { /* head[p]: the next child of p to visit */
            int p = stack[sp], c = head[p];
            if (c >= 0) {
                head[p] = next[c];
                stack[++sp] = c;
            } else {
                sp--;
                qpos[p] = q;
                pofq[q++] = p;
            }
        }
    }
    free(stack);
    for (int p = 0; p < N; p++) {
        pl->node2q[pl->order[p]] = qpos[p];
        pl->q2node[qpos[p]] = pl->order[p];
    }
}

/* Supernodes (and the statistics nnz_l_blocks, flops): a node joins the supernode of the child numbered right before
 * it when the child's structure is the node's structure plus itself (fundamental), or misses at most RELAX_Z block
 * rows of it (relaxed amalgamation: a few explicit zero blocks buy fewer, fatter fronts and a shorter dependency
 * chain); width capped at MAX_SN_COLS. */
static void supernodes(plan_t *pl, const etree_t *t)
{
    const int64_t *bptr = t->bptr;
    const int *pofq = t->pofq;
    const int *parent = pl->parent_pos;
    /* ASAM_RELAX_Z, ASAM_RELAX_FILL, ASAM_TEAM_MERGE_PCT and ASAM_TEAM_MERGE_MFLOP override (tuning) */
    const int relax_z = getenv("ASAM_RELAX_Z") ? atoi(getenv("ASAM_RELAX_Z")) : RELAX_Z;
    const int relax_fill = getenv("ASAM_RELAX_FILL") ? atoi(getenv("ASAM_RELAX_FILL")) : RELAX_FILL;
    const int team_merge_pct = getenv("ASAM_TEAM_MERGE_PCT") ? atoi(getenv("ASAM_TEAM_MERGE_PCT")) : TEAM_MERGE_PCT;
    const double team_merge_mflop =
        getenv("ASAM_TEAM_MERGE_MFLOP") ? atof(getenv("ASAM_TEAM_MERGE_MFLOP")) : TEAM_MERGE_MFLOP;
    for (int q = 0; q < pl->N; q++) {
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
        if (merge)
            pl->desc[pl->nsn - 1].cb++;
        else
            sn_create(pl, q);
        pl->sn_of_q[q] = pl->nsn - 1;
    }
}

/* Row lists, block rows, parents, children, levels and relative indices of every supernode */
static int sn_structure(plan_t *pl, const etree_t *t)
{
    const int64_t *bptr = t->bptr;
    const int *qpos = t->qpos, *pofq = t->pofq;
    /* (per-supernode work, independent: split over a few host threads on large graphs, like the pose loops of solver.c) */
#pragma omp parallel for schedule(static, 256) if (pl->nsn >= PLAN_OMP_MIN_SN) num_threads(asam_host_threads())
    for (int s = 0; s < pl->nsn; s++) {
        asam_sn_desc_t *d = &pl->desc[s];
        sn_host_t *h = &pl->snh[s];
        int qt = d->first + d->cb - 1, pt = pofq[qt];
        int nb = (int) (bptr[pt + 1] - bptr[pt]);
        ivec_reserve(&h->rows, d->cb + nb);
        for (int k = 0; k < d->cb; k++)
            ivec_push(&h->rows, d->first + k);
        for (int64_t e = bptr[pt]; e < bptr[pt + 1]; e++)
            ivec_push(&h->rows, qpos[t->bl.p[e]]);
        /* positions on a root path are ordered alike in both numberings; be safe anyway */
        sort_ints(h->rows.p + d->cb, nb);
        d->parent = nb > 0 ? pl->sn_of_q[h->rows.p[d->cb]] : -1;
    }
    for (int s = 0; s < pl->nsn; s++) {
        sn_set_mb(pl, s);
        int P = pl->desc[s].parent;
        if (P >= 0) {
            ivec_push(&pl->snh[P].children, s);
            int lv = pl->desc[s].level + 1;
            if (lv > pl->desc[P].level)
                pl->desc[P].level = lv; /* children have smaller ids: final when P is reached */
        }
    }
    int rel_bad = 0, n_levels = 0;
#pragma omp parallel for schedule(static, 256) reduction(| : rel_bad) reduction(max : n_levels) if (pl->nsn >= PLAN_OMP_MIN_SN) num_threads(asam_host_threads())
    for (int s = 0; s < pl->nsn; s++) {
        rel_bad |= compute_rel(pl, s);
        if (pl->desc[s].level + 1 > n_levels)
            n_levels = pl->desc[s].level + 1;
    }
    pl->n_levels = n_levels;
    return rel_bad;
}

/* Hessian gather lists: the searches in parallel, the lists filled in slot order */
static int gather_lists(plan_t *pl, const ivec_t *plo, const ivec_t *phi)
{
    const int S = pl->n_slots;
    int *g_sn = malloc(sizeof(int) * (size_t) (S + 1)), *g_rb = malloc(sizeof(int) * (size_t) (S + 1)),
        *g_cb = malloc(sizeof(int) * (size_t) (S + 1));
    int bad_slot = -1;
#pragma omp parallel for schedule(static, 4096) reduction(max : bad_slot) if (S >= 8 * PLAN_OMP_MIN_SN) num_threads(asam_host_threads())
    for (int sl = 0; sl < S; sl++) {
        g_sn[sl] = gather_find(pl, plo->p[sl], phi->p[sl], &g_rb[sl], &g_cb[sl]);
        if (g_rb[sl] < 0 && sl > bad_slot)
            bad_slot = sl;
    }
    if (bad_slot >= 0)
        asam_set_error("plan: Hessian block (%d,%d) not in the structure of supernode %d", plo->p[bad_slot],
                       phi->p[bad_slot], g_sn[bad_slot]);
    else
        for (int sl = 0; sl < S; sl++)
            gather_push(pl, g_sn[sl], sl, g_rb[sl], g_cb[sl]);
    free(g_sn); free(g_rb); free(g_cb);
    return bad_slot >= 0;
}

/* Index segments (into the host copy of the int pool) and arena places of every supernode, in id order */
static void layout(plan_t *pl)
{
    for (int s = 0; s < pl->nsn; s++) {
        emit_segment(pl, s, &pl->ipool_host, 0);
        front_place(pl, s, pl->desc[s].mb);
    }
    pl->ipool_n = pl->ipool_host.n;
}

/* Device buffers for the plan, with head-room for incremental steps, and the whole plan uploaded */
static int build_upload(plan_t *pl, asam_dev_t *dev)
{
    const int N = pl->N, n_factors = pl->n_factors, S = pl->n_slots;
    int64_t ipool_cap = pl->ipool_n * 2 + 4096, arena_cap = pl->arena_n + pl->arena_n / 2 + 65536;
    int rc = asam_reserve(dev, N + N / 2 + 64, n_factors + n_factors / 2 + 64, S + S / 2 + 64,
                          pl->nsn + N / 2 + 64, ipool_cap, arena_cap);
    if (rc)
        return rc;
    int *ids = malloc(sizeof(int) * (size_t) pl->nsn);
    for (int s = 0; s < pl->nsn; s++)
        ids[s] = s;
    rc |= asam_upload_ipool(dev, 0, pl->ipool_host.n, pl->ipool_host.p);
    rc |= asam_upload_desc(dev, pl->nsn, ids, pl->desc);
    rc |= asam_upload_node2q(dev, 0, N, pl->node2q);
    rc |= asam_upload_q2node(dev, 0, N, pl->q2node);
    rc |= asam_upload_fslot(dev, 0, n_factors, pl->fslot);
    rc |= asam_set_full_tasks(dev, pl->ntasks, pl->tasks, pl->nwait, pl->n_btasks, pl->btasks);
    rc |= asam_set_leaf_tasks(dev, pl->n_leaf, pl->leaf_tasks);
    rc |= asam_set_bs_leaf_count(dev, pl->n_bs_leaf);
    asam_shard_sched_t sh = { .n_top = pl->n_top, .top_tasks = pl->top_tasks, .top_nwait = pl->top_nwait,
                              .n_top_sn = pl->n_top_sn, .n_shards = pl->n_shards, .shard_owner = pl->shard_owner,
                              .shard_off = pl->shard_off, .shard_cnt = pl->shard_cnt, .shard_q0 = pl->shard_q0,
                              .shard_qn = pl->shard_qn };
    rc |= asam_set_shard_schedule(dev, pl->world > 1 ? &sh : NULL);
    free(ids);
    return rc;
}

static int plan_build_impl(plan_t *pl, asam_dev_t *dev, int N, int n_factors, const int *ftype, const int *fa,
                           const int *fb, const int *order_keep, int N_keep)
{
    plan_reset(pl, dev);
    if (N <= 0)
        return 0;
    int rc = check_factors(0, n_factors, N, 0, ftype, fa, fb);
    if (rc)
        return rc;
    node_arrays_reserve(pl, N);
    pl->N = N;
    pl->n_factors = n_factors;
    double t = pp_now();
    ivec_t plo = { 0 }, phi = { 0 }; /* pose pairs of the Hessian slots */
    int *adj_ptr, *adj;
    pairmap_init(&pl->pairs, n_factors);
    assign_slots(pl, 0, n_factors, ftype, fa, fb, &plo, &phi);
    adjacency(N, &plo, &phi, &adj_ptr, &adj);
    build_lap(0, &t);
    elimination_order(pl, adj_ptr, adj, order_keep, N_keep);
    build_lap(1, &t);
    etree_t et = block_symbolic(pl, adj_ptr, adj);
    free(adj_ptr); free(adj);
    build_lap(2, &t);
    post_order(pl, &et);
    free(et.head); free(et.next);
    supernodes(pl, &et);
    build_lap(3, &t);
    rc = sn_structure(pl, &et);
    free(et.bptr); ivec_free(&et.bl); free(et.qpos); free(et.pofq);
    build_lap(4, &t);
    if (rc == 0)
        rc = gather_lists(pl, &plo, &phi);
    ivec_free(&plo); ivec_free(&phi);
    if (rc)
        return rc;
    build_lap(5, &t);
    layout(pl);
    build_schedule(pl);
    build_lap(6, &t);
    if (dev) {
        rc = build_upload(pl, dev);
        build_lap(7, &t);
    }
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
/* One plan_append step: what its stages hand on.  pl->mark_idx (supernode -> index among the re-factored ones) is -1
 * between steps; a step sets it for the marked and the created supernodes only, and step_free() resets those. */
typedef struct {
    int N0, F0, nsn0, nnew, slot0; /* the plan before the step; new poses; first new Hessian slot */
    ivec_t nlo, nhi;        /* pose pairs of the new slots slot0, slot0 + 1, ... */
    int *msn, nm;           /* marked supernodes, ascending id (= children first) */
    ivec_t *gain;           /* per marked supernode: the new poses it gains as rows */
    ivec_t *pend, *nbelow;  /* per new pose: children of its supernode, its rows below */
    int ncreated;           /* supernodes created (ids nsn0, nsn0 + 1, ...) */
    int bs_leaf_broken;     /* a supernode outgrew k_backsolve_leaf: all go through k_backsolve from now on */
    int *tasks, *nwait, *keep, nt; /* the fronts to re-factor (keep: their keep words) */
} step_t;

static void step_free(plan_t *pl, step_t *st)
{
    for (int i = 0; i < st->nm; i++) {
        pl->mark_idx[st->msn[i]] = -1;
        ivec_free(&st->gain[i]);
    }
    for (int k = 0; k < st->ncreated; k++)
        pl->mark_idx[st->nsn0 + k] = -1;
    for (int j = 0; st->pend && j < st->nnew; j++) {
        ivec_free(&st->pend[j]);
        ivec_free(&st->nbelow[j]);
    }
    free(st->gain); free(st->pend); free(st->nbelow); free(st->msn);
    free(st->tasks); free(st->nwait); free(st->keep);
    ivec_free(&st->nlo); ivec_free(&st->nhi);
}

/* Incremental steps grow supernodes and run the whole schedule through k_factor / k_backsolve: at the first append the
 * batch back-solve list gets one entry per supernode (parents first = descending id), and the leaf launches go. */
static int step_form(plan_t *pl, asam_dev_t *dev)
{
    const int nsn = pl->nsn;
    if (pl->bt_split) {
        int *plain = malloc(sizeof(int) * (size_t) (nsn + 1));
        for (int sx = 0; sx < nsn; sx++)
            plain[sx] = nsn - 1 - sx;
        free(pl->btasks);
        pl->btasks = plain;
        pl->n_btasks = nsn;
        pl->bt_split = 0;
        pl->n_bs_leaf = 0;
        if (dev && (asam_set_full_tasks(dev, pl->ntasks, pl->tasks, pl->nwait, pl->n_btasks, pl->btasks) ||
                    asam_set_bs_leaf_count(dev, 0)))
            return 1;
    }
    if (pl->n_leaf > 0) {
        pl->n_leaf = 0;
        if (dev && asam_set_leaf_tasks(dev, 0, NULL))
            return 1;
    }
    return 0;
}

/* Node-indexed arrays for N poses and room for a supernode per new pose: new poses are eliminated last, in id order */
static void grow_arrays(plan_t *pl, int N, const step_t *st)
{
    node_arrays_reserve(pl, N);
    sn_arrays_reserve(pl, st->nsn0 + st->nnew);
    for (int i = st->N0; i < N; i++) {
        pl->order[i] = pl->pos[i] = pl->node2q[i] = pl->q2node[i] = i;
        pl->parent_pos[i] = pl->sn_of_q[i] = -1; /* sn_of_q: set by place_new_poses() */
    }
}

/* The marked supernodes, their mark_idx and their keep words.  Partial re-factorisation: the columns of a marked
 * supernode BEFORE its first marked pose are unchanged by this step (their Hessian entries, their children and --
 * because a new pose reaches an old column only through a marked one -- their rows), so the kernel keeps them (L and
 * y) and re-eliminates from the first marked column on: keep[i] = (poses kept << 16) | block rows before this step
 * (the retained front still has that layout), 0 = re-factor the whole front. */
static void mark_supernodes(plan_t *pl, step_t *st, const int *marked_old, int n_marked)
{
    st->msn = malloc(sizeof(int) * (size_t) (n_marked + 1));
    for (int i = 0; i < n_marked; i++)
        if (marked_old[i] < st->N0)
            st->msn[st->nm++] = pl->sn_of_q[pl->node2q[marked_old[i]]];
    st->nm = sort_unique(st->msn, st->nm);
    /* mark_idx is kept across steps, all -1 between them (an O(nsn) fill per step is what made the reference's
     * incremental steps grow with the graph, SURVEY.md quirk 13) */
    if (pl->sn_cap > pl->mark_cap) {
        pl->mark_idx = realloc(pl->mark_idx, sizeof(int) * (size_t) pl->sn_cap);
        for (int s = pl->mark_cap; s < pl->sn_cap; s++)
            pl->mark_idx[s] = -1;
        pl->mark_cap = pl->sn_cap;
    }
    for (int i = 0; i < st->nm; i++)
        pl->mark_idx[st->msn[i]] = i;
    st->gain = calloc((size_t) st->nm + 1, sizeof(ivec_t));
    st->keep = calloc((size_t) (st->nm + st->nnew) + 1, sizeof(int)); /* (created supernodes: 0) */
    for (int i = 0; i < st->nm; i++)
        st->keep[i] = pl->desc[st->msn[i]].cb;
    for (int i = 0; i < n_marked; i++)
        if (marked_old[i] < st->N0) {
            int q = pl->node2q[marked_old[i]], sidx = pl->mark_idx[pl->sn_of_q[q]];
            int k = q - pl->desc[st->msn[sidx]].first;
            if (k < st->keep[sidx])
                st->keep[sidx] = k;
        }
    for (int i = 0; i < st->nm; i++) {
        const int kept = st->keep[i], oldmb = pl->snh[st->msn[i]].rows.n;
        st->keep[i] = kept > 0 && kept < 0x7fff && oldmb < 0xffff ? (kept << 16) | oldmb : 0;
    }
}

/* The new poses that become rows of the marked supernodes: those of their new (old, new) blocks, and, up the marked
 * sub-forest, those of their marked children.  A front that outgrows its allocation moves; an old root hangs under
 * the first new pose it gains.  The (new, new) blocks seed the rows below the new poses. */
static int propagate_gains(plan_t *pl, step_t *st)
{
    const int N0 = st->N0;
    int *mark_idx = pl->mark_idx;
    st->pend = calloc((size_t) st->nnew + 1, sizeof(ivec_t));
    st->nbelow = calloc((size_t) st->nnew + 1, sizeof(ivec_t));
    for (int k = 0; k < st->nlo.n; k++) {
        int lo = st->nlo.p[k], hi = st->nhi.p[k];
        if (lo < N0) {
            int s = pl->sn_of_q[pl->node2q[lo]];
            if (mark_idx[s] < 0) {
                asam_set_error("plan_append: pose %d gets a new factor but is not marked", lo);
                return 1;
            }
            ivec_push(&st->gain[mark_idx[s]], hi);
        } else {
            ivec_push(&st->nbelow[lo - N0], hi);
        }
    }
    for (int i = 0; i < st->nm; i++) {
        int s = st->msn[i];
        sn_host_t *h = &pl->snh[s];
        asam_sn_desc_t *d = &pl->desc[s];
        ivec_t *gain = &st->gain[i];
        for (int c = 0; c < h->children.n; c++) {
            int ci = mark_idx[h->children.p[c]];
            if (ci >= 0)
                for (int e = 0; e < st->gain[ci].n; e++)
                    ivec_push(gain, st->gain[ci].p[e]);
        }
        gain->n = sort_unique(gain->p, gain->n);
        int old_mb = h->rows.n;
        for (int e = 0; e < gain->n; e++)
            ivec_push(&h->rows, gain->p[e]); /* new poses sort after every old row */
        sn_set_mb(pl, s);
        st->bs_leaf_broken |= bs_leaf_outgrown(pl, s);
        if (d->mb != old_mb && front_doubles(d->mb) > d->reserved) {
            /* the front outgrew its allocation: move it, with head-room for the poses that
             * later steps will append (the old space is reclaimed at the next batch) */
            front_place(pl, s, d->mb + (d->mb / 4 > 4 ? d->mb / 4 : 4));
            st->keep[i] = 0; /* the retained columns stay behind at the old place */
        }
        if (d->parent < 0 && gain->n > 0) { /* old root: hangs under the first new pose */
            ivec_push(&st->pend[gain->p[0] - N0], s); /* supernode id of that pose: set by place_new_poses() */
            int top = pl->q2node[d->first + d->cb - 1];
            pl->parent_pos[pl->pos[top]] = gain->p[0]; /* pos == q == id for new poses */
        }
    }
    return 0;
}

/* New poses, ascending.  A pose whose predecessor in the order tops a root supernode with exactly the structure
 * {pose} + below(pose) becomes one more COLUMN of that supernode (fundamental merge) -- otherwise every step would add
 * one more link to the chain at the top of the tree; any other pose starts a singleton supernode. */
static void place_new_poses(plan_t *pl, step_t *st)
{
    const int N0 = st->N0;
    for (int j = 0; j < st->nnew; j++) {
        int n = N0 + j;
        ivec_t *bel = &st->nbelow[j], *pend = &st->pend[j];
        int lvl = 0;
        for (int c = 0; c < pend->n; c++) {
            int X = pend->p[c];
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
            for (int c = 0; c < pend->n; c++)
                if (pend->p[c] == R)
                    sid = R;
        }
        if (sid >= 0) { /* n joins R: the row list already holds n right after R's columns */
            asam_sn_desc_t *d = &pl->desc[R];
            d->cb += 1;
            st->bs_leaf_broken |= bs_leaf_outgrown(pl, R);
            for (int c = 0; c < pend->n; c++) {
                int X = pend->p[c];
                if (X == R)
                    continue;
                ivec_push(&pl->snh[R].children, X);
                pl->desc[X].parent = R;
            }
            if (lvl > d->level)
                d->level = lvl;
            d->parent = -1;
        } else {
            sid = sn_create(pl, n);
            st->ncreated++;
            sn_host_t *h = &pl->snh[sid];
            pl->desc[sid].level = lvl;
            ivec_push(&h->rows, n);
            for (int e = 0; e < bel->n; e++)
                ivec_push(&h->rows, bel->p[e]);
            for (int c = 0; c < pend->n; c++) {
                ivec_push(&h->children, pend->p[c]);
                pl->desc[pend->p[c]].parent = sid;
            }
            sn_set_mb(pl, sid);
            front_place(pl, sid, pl->desc[sid].mb + 4);
        }
        pl->sn_of_q[n] = sid;
        if (bel->n > 0) {
            ivec_push(&st->pend[bel->p[0] - N0], sid);
            pl->parent_pos[n] = bel->p[0];
        }
        if (pl->desc[sid].level + 1 > pl->n_levels)
            pl->n_levels = pl->desc[sid].level + 1;
    }
}

/* Gather entries of the new slots: the (old, new) blocks, then the (new, new) ones */
static int gather_entries(plan_t *pl, const step_t *st)
{
    for (int pass = 0; pass < 2; pass++)
        for (int k = 0; k < st->nlo.n; k++) {
            int lo = st->nlo.p[k], hi = st->nhi.p[k], rb, cb;
            if ((lo >= st->N0) != pass)
                continue;
            int s = gather_find(pl, lo, hi, &rb, &cb);
            if (rb < 0) {
                asam_set_error("plan_append: internal (row %d not in %ssupernode %d)", hi, pass ? "new " : "", s);
                return 1;
            }
            gather_push(pl, s, st->slot0 + k, rb, cb);
        }
    return 0;
}

/* The fronts to re-factor, marked then created, with their child counts, relative indices and index segments
 * (appended to the host copy of the int pool); every new pose must be in one of them */
static int step_fronts(plan_t *pl, step_t *st)
{
    int rc = 0;
    st->nt = st->nm + st->ncreated;
    st->tasks = malloc(sizeof(int) * (size_t) (st->nt + 1));
    st->nwait = malloc(sizeof(int) * (size_t) (st->nt + 1));
    memcpy(st->tasks, st->msn, sizeof(int) * (size_t) st->nm);
    for (int k = 0; k < st->ncreated; k++) {
        st->tasks[st->nm + k] = st->nsn0 + k;
        pl->mark_idx[st->nsn0 + k] = st->nm + k;
    }
    for (int n = st->N0; n < st->N0 + st->nnew; n++) /* a pose may have joined a supernode that was not marked */
        if (pl->mark_idx[pl->sn_of_q[n]] < 0) {
            asam_set_error("plan_append: pose %d joined unmarked supernode %d", n, pl->sn_of_q[n]);
            rc = 1;
        }
    for (int t = 0; t < st->nt && !rc; t++)
        rc = compute_rel(pl, st->tasks[t]);
    for (int t = 0; t < st->nt && !rc; t++) {
        int s = st->tasks[t], w = 0;
        for (int c = 0; c < pl->snh[s].children.n; c++)
            if (pl->mark_idx[pl->snh[s].children.p[c]] >= 0)
                w++;
        st->nwait[t] = pack_nwait(w, 0, 0);
        emit_segment(pl, s, &pl->ipool_host, 0); /* the host pool holds pl->ipool_n ints before the step */
    }
    return rc;
}

/* What the step changed, to the device: segments and descriptors of the fronts, the new poses, the new supernodes at
 * the head of the back-solve list (ancestors of all older ones), the new factors' slots; new Hessian entries cleared */
static int step_upload(plan_t *pl, asam_dev_t *dev, const step_t *st, int N, int n_factors)
{
    double t = pp_now();
    const int nt = st->nt, nnew = st->nnew, ncreated = st->ncreated;
    const int64_t ipool_need = pl->ipool_host.n;
    int rc = asam_reserve(dev, N + 64, n_factors + 64, pl->n_slots + 64, pl->nsn + 64, ipool_need + ipool_need / 2,
                          pl->arena_n + pl->arena_n / 4);
    g_plan_prof[1] += pp_now() - t; /* asam_reserve */
    t = pp_now();
    asam_sn_desc_t *dd = malloc(sizeof(asam_sn_desc_t) * (size_t) (nt + 1));
    for (int k = 0; k < nt; k++)
        dd[k] = pl->desc[st->tasks[k]];
    if (!rc)
        rc |= asam_upload_ipool(dev, pl->ipool_n, ipool_need - pl->ipool_n, pl->ipool_host.p + pl->ipool_n);
    if (!rc)
        rc |= asam_upload_desc(dev, nt, st->tasks, dd);
    if (!rc && nnew > 0) {
        rc |= asam_upload_node2q(dev, st->N0, nnew, pl->node2q + st->N0);
        rc |= asam_upload_q2node(dev, st->N0, nnew, pl->q2node + st->N0);
    }
    if (!rc && ncreated > 0) {
        int *pre = malloc(sizeof(int) * (size_t) ncreated);
        for (int k = 0; k < ncreated; k++)
            pre[k] = st->nsn0 + ncreated - 1 - k;
        rc |= asam_btasks_prepend(dev, ncreated, pre);
        free(pre);
    }
    if (!rc && st->bs_leaf_broken)
        rc |= asam_set_bs_leaf_count(dev, 0);
    if (!rc)
        rc |= asam_upload_fslot(dev, st->F0, n_factors - st->F0, pl->fslot + st->F0);
    if (!rc)
        rc |= asam_hessian_clear_range(dev, st->N0, nnew, st->slot0, pl->n_slots - st->slot0);
    free(dd);
    g_plan_prof[2] += pp_now() - t; /* uploads */
    return rc;
}

/* Fronts that teams factor become consecutive task entries, one per worker (emit_front); teams re-factor whole fronts */
static void expand_teams(const plan_t *pl, step_t *st)
{
    int total = 0;
    for (int t = 0; t < st->nt; t++)
        total += front_ctas(team_size(pl->desc[st->tasks[t]].mb, pl->desc[st->tasks[t]].cb, plan_team_cap(pl)));
    if (total == st->nt)
        return;
    int *t2 = malloc(sizeof(int) * (size_t) total), *w2 = malloc(sizeof(int) * (size_t) total);
    int *k2 = calloc((size_t) total, sizeof(int)), k = 0;
    for (int t = 0; t < st->nt; t++) {
        const int G = team_size(pl->desc[st->tasks[t]].mb, pl->desc[st->tasks[t]].cb, plan_team_cap(pl));
        if (G == 0)
            k2[k] = st->keep[t];
        k += emit_front(t2 + k, w2 + k, st->tasks[t], st->nwait[t], G);
    }
    free(st->tasks); free(st->nwait); free(st->keep);
    st->tasks = t2;
    st->nwait = w2;
    st->keep = k2;
    st->nt = total;
}

int plan_append(plan_t *pl, asam_dev_t *dev, int N, int n_factors, const int *ftype, const int *fa, const int *fb,
                const int *marked_old, int n_marked, int **tasks_out, int **nwait_out, int **keep_out, int *ntasks_out)
{
    const double t0 = pp_now();
    *tasks_out = *nwait_out = NULL;
    if (keep_out)
        *keep_out = NULL;
    *ntasks_out = 0;
    step_t st = { .N0 = pl->N, .F0 = pl->n_factors, .nsn0 = pl->nsn, .nnew = N - pl->N };
    /* everything is checked before anything changes: after a 2 the caller rebuilds from this plan */
    int rc = check_factors(st.F0, n_factors, N, st.N0, ftype, fa, fb);
    if (rc == 0 && pl->world > 1) {
        asam_set_error("a batch solve sharded over %d GPUs cannot be continued incrementally (replicas only)", pl->world);
        rc = 1;
    }
    if (rc == 0)
        rc = step_form(pl, dev);
    if (rc == 0) {
        grow_arrays(pl, N, &st);
        st.slot0 = pl->n_slots;
        assign_slots(pl, st.F0, n_factors, ftype, fa, fb, &st.nlo, &st.nhi);
        mark_supernodes(pl, &st, marked_old, n_marked);
        rc = propagate_gains(pl, &st);
    }
    if (rc == 0) {
        place_new_poses(pl, &st);
        rc = gather_entries(pl, &st);
    }
    if (rc == 0) {
        rc = step_fronts(pl, &st);
        g_plan_prof[0] += pp_now() - t0; /* host symbolic */
    }
    if (rc == 0 && dev)
        rc = step_upload(pl, dev, &st, N, n_factors);
    if (rc == 0) {
        pl->ipool_n = pl->ipool_host.n;
        if (st.bs_leaf_broken)
            pl->n_bs_leaf = 0;
        expand_teams(pl, &st);
        *tasks_out = st.tasks;
        *nwait_out = st.nwait;
        *ntasks_out = st.nt;
        st.tasks = st.nwait = NULL;
        if (keep_out) {
            *keep_out = st.keep;
            st.keep = NULL;
        }
        pl->N = N;
        pl->n_factors = n_factors;
        pl->struct_hash = 0; /* appended order: never to be reused by a batch solve (it re-orders) */
    }
    step_free(pl, &st);
    return rc;
}

/* ---- steps without structural change (factor removal) ---------------------------------------- */
int plan_refactor(plan_t *pl, const int *marked, int n_marked, int **tasks_out, int **nwait_out, int **keep_out,
                  int *ntasks_out)
{
    step_t st = { .N0 = pl->N, .F0 = pl->n_factors, .nsn0 = pl->nsn };
    mark_supernodes(pl, &st, marked, n_marked);
    st.nt = st.nm;
    st.tasks = malloc(sizeof(int) * (size_t) (st.nt + 1));
    st.nwait = malloc(sizeof(int) * (size_t) (st.nt + 1));
    memcpy(st.tasks, st.msn, sizeof(int) * (size_t) st.nm);
    for (int t = 0; t < st.nt; t++) {
        int s = st.tasks[t], w = 0;
        for (int c = 0; c < pl->snh[s].children.n; c++)
            if (pl->mark_idx[pl->snh[s].children.p[c]] >= 0)
                w++;
        st.nwait[t] = pack_nwait(w, 0, 0);
    }
    expand_teams(pl, &st);
    *tasks_out = st.tasks;
    *nwait_out = st.nwait;
    *keep_out = st.keep;
    *ntasks_out = st.nt;
    st.tasks = st.nwait = st.keep = NULL;
    step_free(pl, &st);
    return 0;
}

int plan_remove_factors(plan_t *pl, asam_dev_t *dev, int n, const int *sorted_idx)
{
    if (n < 1) {
        asam_set_error("plan_remove_factors: n = %d", n);
        return 1;
    }
    for (int k = 0; k < n; k++)
        if (sorted_idx[k] < 0 || sorted_idx[k] >= pl->n_factors || (k > 0 && sorted_idx[k] <= sorted_idx[k - 1])) {
            asam_set_error("plan_remove_factors: index %d (entry %d) is not ascending in [0, %d)", sorted_idx[k], k,
                           pl->n_factors);
            return 1;
        }
    const int F = pl->n_factors, first = sorted_idx[0];
    for (int f = first, k = 0, out = first; f < F; f++) {
        if (k < n && sorted_idx[k] == f) {
            k++;
            continue;
        }
        pl->fslot[out++] = pl->fslot[f];
    }
    pl->n_factors = F - n;
    pl->struct_hash = 0; /* counts may match the next structure again (remove one, add one): never reuse */
    if (dev && pl->n_factors > first && asam_upload_fslot(dev, first, pl->n_factors - first, pl->fslot + first))
        return 1;
    return 0;
}

int plan_marginal_paths(const plan_t *pl, int n, const int *nodes, asam_marg_path_t *out, int64_t *z_total,
                        int *hop_total)
{
    int64_t z = 0, hops = 0;
    for (int i = 0; i < n; i++) {
        const int node = nodes[i];
        if (node < 0 || node >= pl->N) {
            asam_set_error("node %d is not in the solved graph (%d poses)", node, pl->N);
            return -1;
        }
        const int q = pl->node2q[node], s0 = pl->sn_of_q[q];
        out[i].sn0 = s0;
        out[i].j0 = 3 * (q - pl->desc[s0].first);
        out[i].hop0 = (int32_t) hops;
        out[i].zoff = z;
        int nh = 0;
        for (int s = s0, js = out[i].j0; s >= 0; s = pl->desc[s].parent, js = 0, nh++)
            z += 3 * (3 * (int64_t) pl->desc[s].cb - js);
        out[i].nhop = nh;
        hops += nh;
        if (hops > INT32_MAX) {
            asam_set_error("%d poses: their paths have more than 2^31 supernodes in all", n);
            return -1;
        }
    }
    *z_total = z;
    *hop_total = (int) hops;
    return 0;
}

/* doubles of query scratch (3 per scalar row of the root path) of the pose at elimination position q */
static int64_t marginal_path_doubles(const plan_t *pl, int q)
{
    int64_t z = 0;
    for (int s = pl->sn_of_q[q], js = 3 * (q - pl->desc[s].first); s >= 0; s = pl->desc[s].parent, js = 0)
        z += 3 * (3 * (int64_t) pl->desc[s].cb - js);
    return z;
}

/* scratch doubles of the poses of candidate (a, b) that the open batch does not hold yet (slot[node] < 0) */
static int64_t candidate_new_doubles(const plan_t *pl, const int *slot, int a, int b)
{
    int64_t z = slot[a] < 0 ? marginal_path_doubles(pl, pl->node2q[a]) : 0;
    if (b >= 0 && b != a && slot[b] < 0)
        z += marginal_path_doubles(pl, pl->node2q[b]);
    return z;
}

void plan_candidate_batches(const plan_t *pl, int k, const int *a, const int *b, int64_t budget, int *batch_end,
                            int *n_batches, int *poses, int *pose_end, int *ia, int *ib)
{
    int *slot = malloc(sizeof(int) * (size_t) (pl->N > 0 ? pl->N : 1));
    for (int i = 0; i < pl->N; i++)
        slot[i] = -1;
    int nb = 0, np = 0, p0 = 0, nc = 0; /* batches closed, poses listed, first pose of the open batch, its candidates */
    int64_t z = 0;
    for (int c = 0; c < k; c++) {
        int64_t ext = candidate_new_doubles(pl, slot, a[c], b[c]);
        if (nc > 0 && z + ext > budget) {
            for (int i = p0; i < np; i++)
                slot[poses[i]] = -1;
            batch_end[nb] = c;
            pose_end[nb++] = np;
            p0 = np;
            nc = 0;
            z = 0;
            ext = candidate_new_doubles(pl, slot, a[c], b[c]);
        }
        z += ext;
        if (slot[a[c]] < 0) {
            slot[a[c]] = np - p0;
            poses[np++] = a[c];
        }
        ia[c] = slot[a[c]];
        if (b[c] >= 0 && slot[b[c]] < 0) {
            slot[b[c]] = np - p0;
            poses[np++] = b[c];
        }
        ib[c] = b[c] >= 0 ? slot[b[c]] : -1;
        nc++;
    }
    if (nc > 0) {
        batch_end[nb] = k;
        pose_end[nb++] = np;
    }
    free(slot);
    *n_batches = nb;
}

/* scratch doubles of the distinct poses of candidates [c0, c1) and [d0, d1); slot (all -1) is left as it was found */
static int64_t compat_union_doubles(const plan_t *pl, int *slot, const int *a, const int *b, int c0, int c1, int d0,
                                    int d1)
{
    int64_t z = 0;
    for (int pass = 0; pass < 2; pass++)
        for (int h = 0; h < 2; h++)
            for (int c = h ? d0 : c0; c < (h ? d1 : c1); c++)
                for (int e = 0; e < 2; e++) {
                    const int node = e ? b[c] : a[c];
                    if (node < 0)
                        continue;
                    if (pass == 1) {
                        slot[node] = -1;
                    } else if (slot[node] < 0) {
                        slot[node] = 0;
                        z += marginal_path_doubles(pl, pl->node2q[node]);
                    }
                }
    return z;
}

/* the scratch of tile (I, J): the z rows of its distinct poses and 10 doubles per pair slot |I| x |J| */
static int64_t compat_tile_doubles(const plan_t *pl, int *slot, const int *a, const int *b, int i0, int i1, int j0,
                                   int j1)
{
    return compat_union_doubles(pl, slot, a, b, i0, i1, j0, j1) + 10 * (int64_t) (i1 - i0) * (int64_t) (j1 - j0);
}

static void compat_push(int **t, int *n, int *cap, int i0, int i1, int j0, int j1)
{
    if (*n == *cap) {
        *cap = *cap ? 2 * *cap : 16;
        *t = realloc(*t, sizeof(int) * 4 * (size_t) *cap);
    }
    int *q = *t + 4 * (size_t) (*n)++;
    q[0] = i0;
    q[1] = i1;
    q[2] = j0;
    q[3] = j1;
}

int plan_compat_tiles(const plan_t *pl, int k, const int *a, const int *b, int64_t budget, int **tiles_out)
{
    int *slot = malloc(sizeof(int) * (size_t) (pl->N > 0 ? pl->N : 1));
    for (int i = 0; i < pl->N; i++)
        slot[i] = -1;
    int *t = NULL, nt = 0, cap = 0;
    if (compat_tile_doubles(pl, slot, a, b, 0, k, 0, k) <= budget) {
        compat_push(&t, &nt, &cap, 0, k, 0, k);
    } else {
        /* blocks in input order: each within a quarter of the budget in z and half of it in pair slots, so that any
         * two of them make a tile within the budget */
        int *bend = malloc(sizeof(int) * (size_t) k), nb = 0, c0 = 0, p0 = 0, np = 0;
        int *bp = malloc(sizeof(int) * 2 * (size_t) k);
        int64_t z = 0;
        for (int c = 0; c < k; c++) {
            int64_t ext = candidate_new_doubles(pl, slot, a[c], b[c]);
            const int64_t n1 = c - c0 + 1;
            if (c > c0 && (z + ext > budget / 4 || 10 * n1 * n1 > budget / 2)) {
                for (int i = p0; i < np; i++)
                    slot[bp[i]] = -1;
                bend[nb++] = c;
                c0 = c;
                p0 = np;
                z = 0;
                ext = candidate_new_doubles(pl, slot, a[c], b[c]);
            }
            z += ext;
            for (int e = 0; e < 2; e++) {
                const int node = e ? b[c] : a[c];
                if (node >= 0 && slot[node] < 0) {
                    slot[node] = 0;
                    bp[np++] = node;
                }
            }
        }
        for (int i = p0; i < np; i++)
            slot[bp[i]] = -1;
        bend[nb++] = k;
        /* tiles (B_p, B_q), p <= q; a pair of blocks beyond the budget (one of them a single candidate that alone
         * exceeds its share) goes one pair per tile */
        for (int p = 0; p < nb; p++)
            for (int q = p; q < nb; q++) {
                const int i0 = p ? bend[p - 1] : 0, i1 = bend[p], j0 = q ? bend[q - 1] : 0, j1 = bend[q];
                if (p == q || compat_tile_doubles(pl, slot, a, b, i0, i1, j0, j1) <= budget) {
                    compat_push(&t, &nt, &cap, i0, i1, j0, j1);
                    continue;
                }
                for (int i = i0; i < i1; i++)
                    for (int j = j0; j < j1; j++)
                        compat_push(&t, &nt, &cap, i, i + 1, j, j + 1);
            }
        free(bend);
        free(bp);
    }
    free(slot);
    *tiles_out = t;
    return nt;
}
