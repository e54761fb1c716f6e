/* solver.c -- april_graph_cholesky / april_graph_cholesky_inc / april_graph_chi2 (host C).
 *
 * Host control plane of the drop-in.  It keeps the reference's observable protocol
 * (reference: aprilsam/aprilsam.c:45-597, :599-987) --
 *   - param bookkeeping (chol non-NULL after a batch, factor_num, nreordering, ordering, tr)
 *   - the node-level elimination tree `param->tr`, root-path marking, naffected
 *   - the back-substitution traversal rule of solve_node (full tree when naffected > 5,
 *     otherwise only marked nodes are updated), relinearisation counters, batch escalation
 * -- while every floating-point operation of the solve (linearisation, J'WJ assembly,
 * Cholesky factorisation, forward/backward substitution, chi2) runs in the CUDA kernels
 * behind include/asam_cuda.h.  The host only moves poses in and the solution out.
 *
 * Deliberate differences from the reference (SURVEY.md section 9):
 *   - the wall-clock escalation hack (aprilsam.c:556-559) is not reproduced (quirk 1);
 *   - a non-positive pivot aborts with a message instead of a NULL dereference (quirk 12);
 *   - param->A / B / y / delta_x stay NULL: the Hessian, rhs and factor live in HBM;
 *   - a factor added between two already-solved poses is handled exactly (full symbolic
 *     rebuild, no relinearisation) where the reference corrupts its tree (aprilsam.c:925-941).
 */
#include <limits.h>
#include <math.h>
#include <pthread.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "asam_host.h"

/* ---- errors -------------------------------------------------------------------------------- */
static __thread char g_error[512];

void asam_set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
}

void asam_fatal(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    fprintf(stderr, "aprilsam_b200: fatal: ");
    vfprintf(stderr, fmt, ap);
    fprintf(stderr, "\n");
    va_end(ap);
    abort();
}

ASAM_API const char *aprilsam_b200_last_error(void) { return g_error; }

/* ---- host phase profile (diagnostics; read with asam_dbg_profile) ----------------------------- */
static double g_prof[24];
static inline double prof_now(void)
{
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6;
}
#define PROF_BEGIN() double prof_t_ = prof_now()
#define PROF_LAP(idx)                   \
    do {                                \
        double n_ = prof_now();         \
        g_prof[idx] += n_ - prof_t_;    \
        prof_t_ = n_;                   \
    } while (0)

ASAM_API void asam_dbg_profile(double *out, int reset)
{
    memcpy(out, g_prof, sizeof(g_prof));
    if (reset)
        memset(g_prof, 0, sizeof(g_prof));
}

/* host threads for the per-node loops of a batch solve on a large graph (never for small ones: the
 * fork/join costs more than 3500 poses do) */
/* the fused small-step kernel (k_step) takes steps with at most this many fronts to re-factor /
 * supernodes to back-solve; anything larger has parallelism the persistent kernels exploit */
#define ASAM_SMALL_MAX_TASKS 32
#define ASAM_SMALL_MAX_BS 64

#define ASAM_OMP_MIN_NODES 16384
/* (thread count of the per-pose loops: asam_host_threads(), plan.c) */

#define DEV_OK(call)                                                                       \
    do {                                                                                   \
        if ((call) != 0)                                                                   \
            asam_fatal("%s failed: %s / %s", #call, asam_last_error(), g_error);           \
    } while (0)

/* ---- param->show_timing (aprilsam.c:317-318, :553-555, :587-588): phase table in the reference's
 * timeprofile_display format ("%2d %32s %15f ms %15f ms": this phase, cumulative), host phases plus
 * the device time of the three kernels (CUDA events on the library's stream) ------------------- */
typedef struct {
    const char *name[12];
    double t[12];
    int n;
} stamps_t;

static inline void stamp(stamps_t *sp, const char *name)
{
    if (sp->n < 12) {
        sp->name[sp->n] = name;
        sp->t[sp->n++] = prof_now();
    }
}

static void stamps_display(const stamps_t *sp, asam_dev_t *dev)
{
    for (int i = 0; i < sp->n; i++)
        printf("%2d %32s %15f ms %15f ms\n", i, sp->name[i], i ? sp->t[i] - sp->t[i - 1] : 0.0, sp->t[i] - sp->t[0]);
    float lin = 0, fac = 0, bs = 0;
    if (dev && asam_last_kernel_ms(dev, &lin, &fac, &bs) == 0)
        printf("   %32s %15f ms\n   %32s %15f ms\n   %32s %15f ms\n", "device: k_linearize", lin,
               "device: k_factor(+leaf)", fac, "device: k_backsolve(+leaf)", bs);
}

/* ---- per-graph device context ---------------------------------------------------------------- */
typedef struct gctx {
    april_graph_t *graph; /* NULL once the graph was destroyed */
    asam_dev_t *dev;
    int refs;
    int nf_dev; /* factors mirrored in HBM */
    int *ftype, *fa, *fb;
    double *zw; /* host mirror of what HBM holds: 12 doubles per factor (z[3], W[9]) */
    int32_t *floss; /* loss code and k per factor (0 / 0 without a robust loss); in HBM for robust factors */
    double *fk;
    int fcap;
    double *stage; /* host staging for poses */
    int stage_cap;
    struct gctx *next;
} gctx_t;

/* The registry is the only state shared between graphs: two threads may solve two different graphs
 * concurrently (as with the reference, whose solver state lives in graph + param), so lookups,
 * inserts and removals are serialised.  One graph is still one caller thread at a time. */
static gctx_t *g_ctx_list = NULL;
static pthread_mutex_t g_ctx_lock = PTHREAD_MUTEX_INITIALIZER;

static gctx_t *gctx_get(april_graph_t *g)
{
    pthread_mutex_lock(&g_ctx_lock);
    for (gctx_t *c = g_ctx_list; c; c = c->next)
        if (c->graph == g) {
            pthread_mutex_unlock(&g_ctx_lock);
            return c;
        }
    pthread_mutex_unlock(&g_ctx_lock);
    gctx_t *c = calloc(1, sizeof(*c));
    c->graph = g;
    if (asam_dev_create(&c->dev) != 0)
        asam_fatal("no usable CUDA device (%s); aprilsam_b200 has no CPU path", asam_last_error());
    c->refs = 1; /* the registry */
    pthread_mutex_lock(&g_ctx_lock);
    c->next = g_ctx_list;
    g_ctx_list = c;
    pthread_mutex_unlock(&g_ctx_lock);
    return c;
}

static void gctx_unref(gctx_t *c)
{
    pthread_mutex_lock(&g_ctx_lock);
    if (--c->refs > 0) {
        pthread_mutex_unlock(&g_ctx_lock);
        return;
    }
    for (gctx_t **pp = &g_ctx_list; *pp; pp = &(*pp)->next)
        if (*pp == c) {
            *pp = c->next;
            break;
        }
    pthread_mutex_unlock(&g_ctx_lock);
    free(c->zw);
    free(c->floss);
    free(c->fk);
    asam_dev_destroy(c->dev);
    free(c->ftype);
    free(c->fa);
    free(c->fb);
    free(c->stage);
    free(c);
}

void asam_graph_forget(april_graph_t *g)
{
    pthread_mutex_lock(&g_ctx_lock);
    gctx_t *hit = NULL;
    for (gctx_t *c = g_ctx_list; c; c = c->next)
        if (c->graph == g) {
            c->graph = NULL;
            hit = c;
            break;
        }
    pthread_mutex_unlock(&g_ctx_lock);
    if (hit)
        gctx_unref(hit);
}

static double *gctx_stage(gctx_t *c, int doubles)
{
    if (doubles > c->stage_cap) {
        c->stage_cap = doubles + doubles / 2 + 64;
        c->stage = realloc(c->stage, sizeof(double) * (size_t) c->stage_cap);
    }
    return c->stage;
}

static inline april_graph_node_t *node_at(april_graph_t *g, int i)
{
    return ((april_graph_node_t **) g->nodes->data)[i];
}

static inline april_graph_factor_t *factor_at(april_graph_t *g, int i)
{
    return ((april_graph_factor_t **) g->factors->data)[i];
}

/* Mirror factors [c->nf_dev, F) into HBM (append-only API: aprilsam.h has no removal). */
static void gctx_sync_factors(gctx_t *c, april_graph_t *g)
{
    int F = zarray_size(g->factors), N = zarray_size(g->nodes);
    if (F < c->nf_dev)
        asam_fatal("factors were removed from the graph (%d -> %d); not supported", c->nf_dev, F);
    if (F == c->nf_dev)
        return;
    if (F > c->fcap) {
        c->fcap = F + F / 2 + 64;
        c->ftype = realloc(c->ftype, sizeof(int) * (size_t) c->fcap);
        c->fa = realloc(c->fa, sizeof(int) * (size_t) c->fcap);
        c->fb = realloc(c->fb, sizeof(int) * (size_t) c->fcap);
        c->zw = realloc(c->zw, sizeof(double) * 12 * (size_t) c->fcap);
        c->floss = realloc(c->floss, sizeof(int32_t) * (size_t) c->fcap);
        c->fk = realloc(c->fk, sizeof(double) * (size_t) c->fcap);
    }
    int first = c->nf_dev, cnt = F - first;
    double *zw = malloc(sizeof(double) * 12 * (size_t) cnt);
    double *z = zw, *W = zw + 3 * (size_t) cnt;
    int robust = 0;
    for (int k = 0; k < cnt; k++) {
        april_graph_factor_t *f = factor_at(g, first + k);
        int i = first + k;
        if (asam_two_pose_type(f->type) && f->nnodes == 2) {
            c->fa[i] = f->nodes[0];
            c->fb[i] = f->nodes[1];
        } else if (f->type == APRIL_GRAPH_FACTOR_XYTPOS_TYPE && f->nnodes == 1) {
            c->fa[i] = f->nodes[0];
            c->fb[i] = -1;
        } else {
            asam_fatal("factor %d has type %d / %d nodes: only xyt (1), xytpos (2) and robust xyt (32) factors are "
                       "supported", i, f->type, f->nnodes);
        }
        c->ftype[i] = f->type;
        asam_factor_loss(f, &c->floss[i], &c->fk[i]);
        if (f->type == APRIL_GRAPH_FACTOR_XYT_ROBUST_TYPE && !c->floss[i])
            asam_fatal("factor %d: robust xyt factor without a loss (create it with "
                       "aprilsam_b200_factor_xyt_robust_create)", i);
        robust |= c->floss[i] != 0;
        const matd_t *Wm = f->u.common.W;
        if (!Wm || Wm->nrows != 3 || Wm->ncols != 3 || !f->u.common.z)
            asam_fatal("factor %d: W must be 3x3 and z non-NULL", i);
        memcpy(z + 3 * (size_t) k, f->u.common.z, 3 * sizeof(double));
        memcpy(W + 9 * (size_t) k, Wm->data, 9 * sizeof(double));
        memcpy(c->zw + 12 * (size_t) i, f->u.common.z, 3 * sizeof(double));
        memcpy(c->zw + 12 * (size_t) i + 3, Wm->data, 9 * sizeof(double));
        for (int j = 0; j < f->nnodes; j++)
            if (f->nodes[j] < 0 || f->nodes[j] >= N)
                asam_fatal("factor %d references node %d outside the graph (%d nodes)", i, f->nodes[j], N);
    }
    DEV_OK(asam_reserve(c->dev, N + 64, F + F / 4 + 64, 0, 0, 0, 0));
    DEV_OK(asam_upload_factors(c->dev, first, cnt, c->ftype + first, c->fa + first, c->fb + first, z, W));
    if (robust) /* graphs without robust factors never move loss records */
        DEV_OK(asam_upload_loss(c->dev, first, cnt, c->floss + first, c->fk + first));
    free(zw);
    c->nf_dev = F;
}

/* The reference reads every factor on every batch call (aprilsam.c:154-195), so a caller may edit
 * z / W in place between calls (re-weighting; robust factors of type 32 re-weight on the GPU at
 * every linearisation instead), change a robust factor's loss, or swap a factor for another one.
 * The HBM mirror is checked against the host structs on every batch call: factors [0, upto) whose
 * measurement or information matrix changed are re-uploaded; a change of type or node ids is
 * reported through the return value (the symbolic plan has to be rebuilt).  The check costs one
 * 96-byte compare per factor and is run WHILE the kernels of the call are in flight (see
 * april_graph_cholesky): in the common case -- nothing changed -- it is free.
 * Returns 0 = unchanged, 1 = values re-uploaded, 2 = structure changed (mirror updated). */
static int gctx_verify_factors(gctx_t *c, april_graph_t *g, int upto)
{
    int changed = 0, structural = 0;
    int lo = upto, hi = -1;
#pragma omp parallel for schedule(static) reduction(| : changed, structural) reduction(min : lo) reduction(max : hi) \
    if (upto >= 4 * ASAM_OMP_MIN_NODES) num_threads(asam_host_threads())
    for (int i = 0; i < upto; i++) {
        const april_graph_factor_t *f = factor_at(g, i);
        const matd_t *Wm = f->u.common.W;
        int na = f->nnodes > 0 ? f->nodes[0] : -1, nb = f->nnodes > 1 ? f->nodes[1] : -1;
        if (f->type != c->ftype[i] || na != c->fa[i] || nb != c->fb[i] || !Wm || !f->u.common.z) {
            structural = 1;
            continue;
        }
        double *m = c->zw + 12 * (size_t) i;
        int32_t loss;
        double k;
        asam_factor_loss(f, &loss, &k);
        if (memcmp(m, f->u.common.z, 3 * sizeof(double)) != 0 || memcmp(m + 3, Wm->data, 9 * sizeof(double)) != 0 ||
            loss != c->floss[i] || memcmp(&k, &c->fk[i], sizeof(double)) != 0) {
            memcpy(m, f->u.common.z, 3 * sizeof(double));
            memcpy(m + 3, Wm->data, 9 * sizeof(double));
            c->floss[i] = loss;
            c->fk[i] = k;
            changed = 1;
            if (i < lo)
                lo = i;
            if (i > hi)
                hi = i;
        }
    }
    if (structural)
        return 2;
    if (!changed)
        return 0;
    /* re-upload the dirty range [lo, hi] (edits are usually a contiguous run or everything) */
    int cnt = hi - lo + 1;
    double *zw = malloc(sizeof(double) * 12 * (size_t) cnt);
    double *z = zw, *W = zw + 3 * (size_t) cnt;
    int robust = 0;
    for (int k = 0; k < cnt; k++) {
        memcpy(z + 3 * (size_t) k, c->zw + 12 * (size_t) (lo + k), 3 * sizeof(double));
        memcpy(W + 9 * (size_t) k, c->zw + 12 * (size_t) (lo + k) + 3, 9 * sizeof(double));
        robust |= c->floss[lo + k] != 0;
    }
    DEV_OK(asam_upload_factors(c->dev, lo, cnt, c->ftype + lo, c->fa + lo, c->fb + lo, z, W));
    if (robust)
        DEV_OK(asam_upload_loss(c->dev, lo, cnt, c->floss + lo, c->fk + lo));
    free(zw);
    return 1;
}

/* ---- chi2 (april_graph.c:79-98) -------------------------------------------------------------- */
ASAM_API double april_graph_chi2(april_graph_t *g)
{
    int N = zarray_size(g->nodes), F = zarray_size(g->factors);
    if (F == 0)
        return 0.0;
    gctx_t *c = gctx_get(g);
    if (gctx_verify_factors(c, g, c->nf_dev < F ? c->nf_dev : F) == 2)
        c->nf_dev = 0; /* a factor was replaced: mirror everything again */
    gctx_sync_factors(c, g);
    double *st = gctx_stage(c, 3 * N);
    for (int i = 0; i < N; i++)
        memcpy(st + 3 * (size_t) i, node_at(g, i)->state, 3 * sizeof(double));
    DEV_OK(asam_reserve(c->dev, N + 64, 0, 0, 0, 0, 0));
    DEV_OK(asam_upload_points(c->dev, 1, 0, N, st));
    double chi2 = 0.0;
    DEV_OK(asam_chi2(c->dev, F, &chi2));
    return chi2;
}

/* ---- what the last incremental call asked of the kernels (tests; asam_dbg_record_steps) ------------- */
enum { STEP_NONE = 0, STEP_SMALL = 1, STEP_PRUNED = 2, STEP_FULL = 3, STEP_FALLBACK = 4 };

typedef struct step_rec {
    int kind, escalated, ntasks, nbt;
    int *tasks, *nwait, *keep, *bt, *bfirst;
    int tcap, bcap;
} step_rec_t;

static int g_record_steps = 0;

static void rec_tasks(step_rec_t *r, int n, const int *tasks, const int *nwait, const int *keep)
{
    if (n > r->tcap) {
        r->tcap = n + n / 2 + 16;
        r->tasks = realloc(r->tasks, sizeof(int) * (size_t) r->tcap);
        r->nwait = realloc(r->nwait, sizeof(int) * (size_t) r->tcap);
        r->keep = realloc(r->keep, sizeof(int) * (size_t) r->tcap);
    }
    r->ntasks = n;
    if (n > 0) {
        memcpy(r->tasks, tasks, sizeof(int) * (size_t) n);
        memcpy(r->nwait, nwait, sizeof(int) * (size_t) n);
        memcpy(r->keep, keep, sizeof(int) * (size_t) n);
    }
}

static void rec_bt(step_rec_t *r, int n, const int *bt, const int *bfirst)
{
    if (n > r->bcap) {
        r->bcap = n + n / 2 + 16;
        r->bt = realloc(r->bt, sizeof(int) * (size_t) r->bcap);
        r->bfirst = realloc(r->bfirst, sizeof(int) * (size_t) r->bcap);
    }
    r->nbt = n;
    if (n > 0) {
        memcpy(r->bt, bt, sizeof(int) * (size_t) n);
        memcpy(r->bfirst, bfirst, sizeof(int) * (size_t) n);
    }
}

/* ---- solver context (hangs off param->chol) -------------------------------------------------- */
#define SOLVER_MAGIC 0x41534d42u /* "ASMB" */

typedef struct solver {
    smatd_chol_t hdr; /* param->chol points here; must stay first */
    uint32_t magic;
    gctx_t *gc;
    plan_t plan;
    int plan_valid;
    double *x; /* solution in elimination (q) order */
    int xcap;
    int tree_fresh; /* param->tr is exactly the tree of `plan` as built by the last batch */
    int *scratch;
    int scratch_cap;
    int *sn_stamp, *sn_jf, *sn_bt; /* per-supernode scratch of the pruned back-substitution (no O(nsn) work per step) */
    int stamp_cap, stamp_epoch;
    aprilsam_b200_escalation_fn policy; /* deterministic escalation hook (aprilsam.h) */
    void *policy_user;
    step_rec_t rec; /* filled only while asam_dbg_record_steps is on */
} solver_t;

/* policies set before the first batch solve wait here for their solver (param -> fn) */
typedef struct pending_policy {
    april_graph_cholesky_param_t *param;
    aprilsam_b200_escalation_fn fn;
    void *user;
    struct pending_policy *next;
} pending_policy_t;
static pending_policy_t *g_pending_policy = NULL;

static solver_t *solver_of(april_graph_cholesky_param_t *param)
{
    solver_t *s = (solver_t *) param->chol;
    if (s && s->magic != SOLVER_MAGIC)
        asam_fatal("param->chol was not created by aprilsam_b200");
    return s;
}

static void solver_destroy(solver_t *s)
{
    if (!s)
        return;
    plan_free(&s->plan);
    if (s->gc)
        gctx_unref(s->gc);
    free(s->x);
    free(s->scratch);
    free(s->sn_stamp);
    free(s->sn_jf);
    free(s->sn_bt);
    free(s->rec.tasks);
    free(s->rec.nwait);
    free(s->rec.keep);
    free(s->rec.bt);
    free(s->rec.bfirst);
    s->magic = 0;
    free(s);
}

static solver_t *solver_get(april_graph_t *g, april_graph_cholesky_param_t *param)
{
    solver_t *s = solver_of(param);
    if (s && s->gc->graph != g) { /* param re-used on another graph */
        solver_destroy(s);
        s = NULL;
        param->chol = NULL;
    }
    if (!s) {
        s = calloc(1, sizeof(*s));
        s->magic = SOLVER_MAGIC;
        s->hdr.is_spd = 1;
        s->gc = gctx_get(g);
        pthread_mutex_lock(&g_ctx_lock);
        s->gc->refs++;
        for (pending_policy_t **pp = &g_pending_policy; *pp; pp = &(*pp)->next)
            if ((*pp)->param == param) {
                pending_policy_t *hit = *pp;
                s->policy = hit->fn;
                s->policy_user = hit->user;
                *pp = hit->next;
                free(hit);
                break;
            }
        pthread_mutex_unlock(&g_ctx_lock);
        param->chol = &s->hdr;
    }
    return s;
}

ASAM_API void aprilsam_b200_set_escalation_policy(april_graph_cholesky_param_t *param, aprilsam_b200_escalation_fn fn,
                                                  void *user)
{
    if (!param)
        return;
    if (param->chol) {
        solver_t *s = solver_of(param);
        s->policy = fn;
        s->policy_user = user;
        return;
    }
    pthread_mutex_lock(&g_ctx_lock);
    pending_policy_t *e = NULL;
    for (pending_policy_t **pp = &g_pending_policy; *pp; pp = &(*pp)->next)
        if ((*pp)->param == param) {
            e = *pp;
            if (!fn) { /* removal */
                *pp = e->next;
                free(e);
                pthread_mutex_unlock(&g_ctx_lock);
                return;
            }
            break;
        }
    if (fn) {
        if (!e) {
            e = calloc(1, sizeof(*e));
            e->param = param;
            e->next = g_pending_policy;
            g_pending_policy = e;
        }
        e->fn = fn;
        e->user = user;
    }
    pthread_mutex_unlock(&g_ctx_lock);
}

ASAM_API int aprilsam_b200_policy_work_ratio(const aprilsam_b200_step_cost_t *cost, void *user)
{
    double ratio = user ? *(const double *) user : 1.0 / 3.0;
    return cost->step_work > ratio * cost->batch_work;
}

ASAM_API void aprilsam_b200_invalidate_plan(april_graph_cholesky_param_t *param)
{
    solver_t *s = param && param->chol ? solver_of(param) : NULL;
    if (s) {
        s->plan_valid = 0;
        s->plan.struct_hash = 0;
        s->tree_fresh = 0;
    }
}

static double *solver_x(solver_t *s, int N)
{
    if (3 * N > s->xcap) {
        s->xcap = 3 * N + 3 * N / 2 + 64;
        s->x = realloc(s->x, sizeof(double) * (size_t) s->xcap);
    }
    return s->x;
}

static int *solver_scratch(solver_t *s, int n)
{
    if (n > s->scratch_cap) {
        s->scratch_cap = n + n / 2 + 64;
        s->scratch = realloc(s->scratch, sizeof(int) * (size_t) s->scratch_cap);
    }
    return s->scratch;
}

/* ---- param lifecycle (aprilsam.c:45-85) ------------------------------------------------------ */
ASAM_API void april_graph_cholesky_param_init(april_graph_cholesky_param_t *param)
{
    memset(param, 0, sizeof(*param));
    param->tikhanov = 0.0001;
    param->nreordering = 1;
}

ASAM_API void search_tree_destroy(search_tree_t *tr)
{
    if (!tr)
        return;
    for (int i = 0; i < tr->nalloc; i++)
        free(tr->nodes[i].children);
    free(tr->nodes);
    free(tr->linearized_nodes);
    free(tr);
}

ASAM_API void april_graph_cholesky_param_destory(april_graph_cholesky_param_t *param)
{
    if (!param)
        return;
    aprilsam_b200_set_escalation_policy(param->chol ? NULL : param, NULL, NULL); /* forget a policy that never met a solver */
    solver_destroy(solver_of(param));
    if (param->tr)
        search_tree_destroy(param->tr);
    free(param->delta_x);
    free(param->B);
    free(param->y);
    free(param->ordering);
    free(param);
}

/* ---- node-level elimination tree (aprilsam.c:613-657) ---------------------------------------- */
static void tree_add_child(search_tree_node_t *p, int child)
{
    if (p->nchildren >= p->nalloc) {
        p->nalloc = p->nalloc > 0 ? 2 * p->nalloc : 8;
        p->children = realloc(p->children, sizeof(int) * (size_t) p->nalloc);
    }
    p->children[p->nchildren++] = child;
}

static search_tree_t *tree_from_plan(const plan_t *pl, april_graph_t *g)
{
    int N = pl->N;
    search_tree_t *tr = calloc(1, sizeof(*tr));
    tr->nnodes = N;
    tr->nalloc = N;
    tr->nodes = calloc((size_t) N, sizeof(search_tree_node_t));
    tr->linearized_nodes = calloc((size_t) N, sizeof(int));
    for (int i = 0; i < N; i++) {
        /* child lists are allocated on first use (leaves never need one) */
        tr->nodes[i].parent = -1;
        tr->nodes[i].g_node = node_at(g, i);
        tr->nodes[i].g_node->UID = i; /* the reference overwrites UIDs too (:627-628) */
    }
    /* children are attached scanning positions downwards, like the reference (:635-652) */
    for (int ui = N - 2; ui >= 0; ui--) {
        int pp = pl->parent_pos[ui];
        if (pp < 0)
            continue;
        int child = pl->order[ui], par = pl->order[pp];
        tr->nodes[child].id = ui;
        tr->nodes[child].parent = par;
        tree_add_child(&tr->nodes[par], child);
    }
    tr->root = &tr->nodes[pl->order[N - 1]];
    tr->root->id = N - 1;
    return tr;
}

/* ---- pose transfer ----------------------------------------------------------------------------- */
static void check_nodes(april_graph_t *g, int first, int N)
{
    for (int i = first; i < N; i++) {
        april_graph_node_t *n = node_at(g, i);
        if (n->type != APRIL_GRAPH_NODE_XYT_TYPE || n->length != 3)
            asam_fatal("node %d has type %d: only xyt nodes (type 100) are supported", i, n->type);
    }
}

/* state <- l_point + dx (april_graph_xyt.c:302-314) */
static inline void apply_update(april_graph_node_t *n, const double *dx)
{
    if (isnan(dx[0]) || isnan(dx[1]) || isnan(dx[2]))
        return;
    for (int k = 0; k < 3; k++) {
        n->state[k] = n->l_point[k] + dx[k];
        n->delta_X[k] = dx[k];
    }
    n->state[2] = mod2pi(n->state[2]);
}

static uint64_t structure_hash(int N, int F, const int *ftype, const int *fa, const int *fb)
{
    uint64_t h = 1469598103934665603ULL ^ ((uint64_t) N << 32) ^ (uint64_t) F;
    for (int f = 0; f < F; f++) {
        uint64_t v = ((uint64_t) (uint32_t) fa[f] << 32) ^ (uint64_t) (uint32_t) fb[f] ^ ((uint64_t) ftype[f] << 60);
        h ^= v;
        h *= 1099511628211ULL;
        h ^= h >> 29;
    }
    return h ? h : 1;
}

static void report_factor_status(solver_t *s, int status, const char *where)
{
    if (status > 0) {
        s->hdr.is_spd = 0;
        asam_fatal("%s: information matrix is not positive definite (pivot <= 0 in supernode %d)", where,
                   status - 1);
    } else if (status == ASAM_STATUS_REMOTE) {
        s->hdr.is_spd = 0;
        asam_fatal("%s: another rank of the sharded solve reported a failed factorisation (not positive definite?)", where);
    } else if (status < 0) {
        asam_fatal("%s: internal scheduling error in the factorisation kernel (supernode %d)", where, -status - 1);
    }
}

static void check_factor_status(solver_t *s, const char *where)
{
    int status = 0;
    DEV_OK(asam_factor_status(s->gc->dev, &status));
    report_factor_status(s, status, where);
}

/* ---- batch Gauss-Newton step (aprilsam.c:87-375) ------------------------------------------------ */
ASAM_API void april_graph_cholesky(april_graph_t *graph, april_graph_cholesky_param_t *param)
{
    int N = zarray_size(graph->nodes), F = zarray_size(graph->factors);
    if (N == 0 || F == 0)
        return;
    if (!param->nreordering)
        asam_fatal("april_graph_cholesky: param->nreordering == 0 is not supported (the reference asserts)");

    PROF_BEGIN();
    g_prof[9] += 1;
    solver_t *s = solver_get(graph, param);
    gctx_t *c = s->gc;
    asam_dev_t *dev = c->dev;
    stamps_t tp = { .n = 0 };
    if (param->show_timing) {
        asam_set_timing(dev, 1);
        stamp(&tp, "begin");
    }
    int restarted = 0;
restart:;
    const int F_mirrored = c->nf_dev < F ? c->nf_dev : F; /* already in HBM: checked while the kernels run */
    gctx_sync_factors(c, graph);

    /* relinearise every node at its current state (:131-135) and stage the poses */
    /* (large graphs: the per-node loops of this function chase one pointer per pose into separately
     * malloc'd arrays -- they are split over a few host threads, SURVEY.md section 7 "host marshalling") */
    double *lp = gctx_stage(c, 3 * N);
    int bad_node = -1;
#pragma omp parallel for schedule(static) reduction(max : bad_node) if (N >= ASAM_OMP_MIN_NODES) num_threads(asam_host_threads())
    for (int i = 0; i < N; i++) {
        april_graph_node_t *n = node_at(graph, i);
        if (n->type != APRIL_GRAPH_NODE_XYT_TYPE || n->length != 3) {
            bad_node = i > bad_node ? i : bad_node; /* reported below */
            continue;
        }
        if (i + 16 < N) { /* every pose is three separate allocations: keep a few in flight */
            const april_graph_node_t *nx = node_at(graph, i + 16);
            __builtin_prefetch(nx);
            __builtin_prefetch(node_at(graph, i + 8)->state);
            __builtin_prefetch(node_at(graph, i + 8)->l_point, 1);
        }
        memcpy(n->l_point, n->state, 3 * sizeof(double));
        memcpy(lp + 3 * (size_t) i, n->state, 3 * sizeof(double));
    }
    if (bad_node >= 0)
        check_nodes(graph, bad_node, bad_node + 1); /* aborts with the message */

    PROF_LAP(11);
    /* ordering + symbolic analysis: cached while the factor structure is unchanged */
    /* the API is append-only and factor node ids are immutable, so a cached plan with the same
     * counts on the same graph has the same structure; the hash (O(F)) is only taken when the
     * counts changed */
    uint64_t h = (s->plan_valid && s->plan.N == N && s->plan.n_factors == F && s->plan.struct_hash != 0)
                     ? s->plan.struct_hash
                     : structure_hash(N, F, c->ftype, c->fa, c->fb);
    int plan_reused = 1;
    /* several GPUs (asam_comm_init + asam_comm_set_sharding): this rank factors its shards of the
     * elimination tree and the part above the cut; every rank calls april_graph_cholesky on its
     * own copy of the same graph */
    int cw = 1, cr = 0, csh = 0;
    asam_comm_info(&cw, &cr, &csh);
    const int want_world = csh ? cw : 1;
    if (!(s->plan_valid && s->plan.N == N && s->plan.n_factors == F && s->plan.struct_hash == h &&
          (s->plan.world > 1 ? s->plan.world : 1) == want_world && (want_world == 1 || s->plan.rank == cr))) {
        plan_reused = 0;
        s->plan.world = want_world;
        s->plan.rank = want_world > 1 ? cr : 0;
        if (plan_build(&s->plan, dev, N, F, c->ftype, c->fa, c->fb) != 0)
            asam_fatal("april_graph_cholesky: %s %s", g_error, asam_last_error());
        s->plan.struct_hash = h;
        s->plan_valid = 1;
    }
    plan_t *pl = &s->plan;
    PROF_LAP(12);
    if (param->show_timing)
        stamp(&tp, plan_reused ? "relinearize, plan (cached)" : "relinearize, ordering+symbolic");

    DEV_OK(asam_upload_points(dev, 0, 0, N, lp));
    DEV_OK(asam_copy_points(dev, 0, 1, 0, N)); /* state mirror = linearisation points, copied in HBM */
    DEV_OK(asam_hessian_reset(dev, N, pl->n_slots, N, param->tikhanov > 0 ? param->tikhanov : 0.0));
    DEV_OK(asam_linearize(dev, 0, F, NULL));
    DEV_OK(asam_factor_full(dev));
    DEV_OK(asam_backsolve_full(dev));
    PROF_LAP(13);
    /* the kernels are in flight: compare the factors HBM holds with the caller's structs (the reference
     * re-reads every factor on every call).  Nothing changed (the usual case): no cost.  Otherwise the
     * changed measurements are uploaded and the pipeline runs again; a replaced factor (other nodes or
     * type) also rebuilds the plan. */
    if (F_mirrored > 0 && !restarted) {
        int v = gctx_verify_factors(c, graph, F_mirrored);
        if (v) {
            int st_ = 0;
            DEV_OK(asam_factor_status(dev, &st_)); /* drain the stale run (its pivots may have failed) */
            restarted = 1;
            if (v == 2) {
                c->nf_dev = 0;
                s->plan_valid = 0;
                goto restart;
            }
            DEV_OK(asam_hessian_reset(dev, N, pl->n_slots, N, param->tikhanov > 0 ? param->tikhanov : 0.0));
            DEV_OK(asam_linearize(dev, 0, F, NULL));
            DEV_OK(asam_factor_full(dev));
            DEV_OK(asam_backsolve_full(dev));
        }
    }
    /* persistent state the incremental path continues from (:260-288) -- host-only work, done while the
     * kernels are still in flight */
    if (plan_reused && s->tree_fresh && param->tr && param->tr->nnodes == N) {
        /* same structure as the previous batch: same tree; only the per-solve labels reset */
        search_tree_t *tr = param->tr;
#pragma omp parallel for schedule(static) if (N >= ASAM_OMP_MIN_NODES) num_threads(asam_host_threads())
        for (int i = 0; i < N; i++) {
            tr->nodes[i].label_changed = 0;
            tr->nodes[i].label_relinearized = 0;
            tr->nodes[i].g_node = node_at(graph, i);
            tr->nodes[i].g_node->UID = i;
        }
        tr->start_over = tr->nlinearized_nodes = tr->naffected = tr->isam1_cnt = 0;
        tr->total_delta_xy = tr->total_delta_theta = 0.0;
    } else {
        if (param->tr)
            search_tree_destroy(param->tr);
        param->tr = tree_from_plan(pl, graph);
    }
    s->tree_fresh = 1;
    param->tr->delta_xy = param->delta_xy;
    param->tr->delta_theta = param->delta_theta;
    if (!(plan_reused && param->ordering && param->nreordering == N)) {
        free(param->ordering);
        param->ordering = malloc(sizeof(int) * (size_t) N);
    }
    memcpy(param->ordering, pl->order, sizeof(int) * (size_t) N);
    param->nreordering = N;
    param->factor_num = F;

    double *x = solver_x(s, N);
    int fstatus = 0;
    DEV_OK(asam_download_x_status(dev, 0, N, x, &fstatus));
    PROF_LAP(14);
    report_factor_status(s, fstatus, "april_graph_cholesky");
    PROF_LAP(15);
    if (param->show_timing)
        stamp(&tp, "H2D, kernels, D2H of solution");

    /* state = l_point + x (:311-315) */
#pragma omp parallel for schedule(static) if (N >= ASAM_OMP_MIN_NODES) num_threads(asam_host_threads())
    for (int i = 0; i < N; i++) {
        if (i + 16 < N) {
            __builtin_prefetch(node_at(graph, i + 16));
            __builtin_prefetch(node_at(graph, i + 8)->l_point);
            __builtin_prefetch(node_at(graph, i + 8)->state, 1);
            __builtin_prefetch(node_at(graph, i + 8)->delta_X, 1);
        }
        apply_update(node_at(graph, i), x + 3 * (size_t) pl->node2q[i]);
    }
    PROF_LAP(16);
    if (param->show_timing) {
        stamp(&tp, "tree, state update");
        stamps_display(&tp, dev);
    }
}

/* ---- incremental step ---------------------------------------------------------------------------- */

/* search_tree_append (aprilsam.c:908-987) driven by the plan's node-level parents. */
static void tree_reparent(search_tree_t *tr, int child_id, int parent_id, int ui)
{
    search_tree_node_t *child = &tr->nodes[child_id], *par = &tr->nodes[parent_id];
    child->id = ui;
    if (child->parent != -1) {
        if (child->parent == parent_id)
            return;
        /* detach from the old parent, keeping the sibling order */
        search_tree_node_t *old = &tr->nodes[child->parent];
        int at = -1;
        for (int i = 0; i < old->nchildren; i++)
            if (old->children[i] == child_id) {
                at = i;
                break;
            }
        if (at >= 0) {
            for (int i = at + 1; i < old->nchildren; i++)
                old->children[i - 1] = old->children[i];
            old->nchildren--;
        }
    }
    child->parent = parent_id;
    tree_add_child(par, child_id);
}

static void tree_append_from_plan(search_tree_t *tr, const plan_t *pl, const int *marked, int n_marked, int old_root_pos,
                                  int N)
{
    /* marked old nodes: only their parent may have changed (old roots gain one) */
    for (int i = 0; i < n_marked; i++) {
        int v = marked[i];
        int ui = pl->pos[v], pp = pl->parent_pos[ui];
        if (pp >= 0 && ui <= old_root_pos)
            tree_reparent(tr, v, pl->order[pp], ui);
    }
    /* new nodes except the last, scanning downwards like the reference (:962-983) */
    for (int ui = N - 2; ui > old_root_pos; ui--) {
        int pp = pl->parent_pos[ui];
        if (pp >= 0)
            tree_reparent(tr, pl->order[ui], pl->order[pp], ui);
    }
    tr->root = &tr->nodes[pl->order[N - 1]];
    tr->root->id = N - 1;
}

/* Back-substitution bookkeeping of solve_node (aprilsam.c:721-779) on the solution x. */
static void apply_solution(solver_t *s, search_tree_t *tr, const double *x, int qbase)
{
    const plan_t *pl = &s->plan;
    int *stack = solver_scratch(s, tr->nnodes + 8);
    int sp = 0;
    stack[sp++] = (int) (tr->root - tr->nodes);
    while (sp > 0) {
        int id = stack[--sp];
        search_tree_node_t *node = &tr->nodes[id];
        const double *xi = x + 3 * (size_t) (pl->node2q[id] - qbase);
        april_graph_node_t *gn = node->g_node;
        if (fabs(xi[0]) > tr->delta_xy || fabs(xi[1]) > tr->delta_xy || fabs(xi[2]) > tr->delta_theta) {
            if (!node->label_relinearized) {
                node->label_relinearized = 1;
                tr->linearized_nodes[tr->nlinearized_nodes++] = gn->UID;
                tr->start_over += 1;
                tr->total_delta_xy += fabs(xi[0]) + fabs(xi[1]);
            } else {
                tr->total_delta_xy += fabs(xi[0]) + fabs(xi[1]) - gn->delta_X[0] - gn->delta_X[1];
            }
        }
        gn->delta_X[0] = xi[0];
        gn->delta_X[1] = xi[1];
        gn->delta_X[2] = xi[2];
        if (tr->naffected > 5) {
            node->label_changed = 0;
        } else if (node->label_changed == 1) {
            node->label_changed = 0;
        } else {
            /* the reference compares delta_X with the value it has just stored into it, so
             * an unmarked node always stops the descent here (:761-770) */
            continue;
        }
        apply_update(gn, xi);
        for (int i = node->nchildren - 1; i >= 0; i--)
            stack[sp++] = node->children[i];
    }
}

static void inc_general_fallback(april_graph_t *graph, april_graph_cholesky_param_t *param, solver_t *s, int N, int F,
                                 int F0);

ASAM_API void april_graph_cholesky_inc(april_graph_t *graph, april_graph_cholesky_param_t *param)
{
    int N = zarray_size(graph->nodes), F = zarray_size(graph->factors);
    if (N == 0 || F == 0)
        return;
    if (!param->chol)
        return;
    if (param->factor_num == F)
        return;
    solver_t *s = solver_of(param);
    if (s->gc->graph != graph || !s->plan_valid || !param->tr)
        asam_fatal("april_graph_cholesky_inc: param does not continue a batch solve of this graph");
    gctx_t *c = s->gc;
    asam_dev_t *dev = c->dev;
    plan_t *pl = &s->plan;
    const int N0 = param->nreordering, F0 = param->factor_num;
    if (pl->N != N0 || pl->n_factors != F0)
        asam_fatal("april_graph_cholesky_inc: solver state out of sync (%d/%d nodes, %d/%d factors)", pl->N, N0,
                   pl->n_factors, F0);
    PROF_BEGIN();
    g_prof[8] += 1;
    stamps_t tp = { .n = 0 };
    if (param->show_timing) {
        asam_set_timing(dev, 1);
        stamp(&tp, "begin");
    }
    s->tree_fresh = 0;
    if (g_record_steps) {
        s->rec.kind = STEP_NONE;
        s->rec.escalated = 0;
        s->rec.ntasks = s->rec.nbt = 0;
    }
    check_nodes(graph, N0, N);
    gctx_sync_factors(c, graph);

    /* new poses are eliminated last, in id order (:393-397) */
    param->ordering = realloc(param->ordering, sizeof(int) * (size_t) N);
    for (int i = N0; i < N; i++)
        param->ordering[i] = i;

    /* grow the tree; new nodes start parentless (:453-477) */
    search_tree_t *tr = param->tr;
    int old_nnodes = tr->nnodes;
    int root_id = (int) (tr->root - tr->nodes);
    int old_root_pos = tr->root->id;
    tr->nnodes = N;
    if (tr->nnodes >= tr->nalloc) {
        int nalloc = tr->nnodes * 2;
        search_tree_node_t *tmp = calloc((size_t) nalloc, sizeof(search_tree_node_t));
        memcpy(tmp, tr->nodes, sizeof(search_tree_node_t) * (size_t) old_nnodes);
        free(tr->nodes);
        tr->nodes = tmp;
        tr->nalloc = nalloc;
        tr->linearized_nodes = realloc(tr->linearized_nodes, sizeof(int) * (size_t) nalloc);
    }
    tr->root = &tr->nodes[root_id];
    for (int i = old_nnodes; i < N; i++) {
        search_tree_node_t *tn = &tr->nodes[i];
        tn->nchildren = 0;
        tn->parent = -1;
        tn->g_node = node_at(graph, i);
        tn->g_node->UID = i;
        tn->id = i;
        tn->label_changed = 0;
        tn->label_relinearized = 0;
    }
    /* g_node pointers of old nodes stay valid: the graph owns the nodes */

    /* mark the root paths of every node a new factor touches (:482-498) */
    int *marked = solver_scratch(s, 2 * N + 16) + N + 8; /* upper half: apply_solution uses the lower */
    int n_marked = 0;
    tr->naffected = 0;
    for (int f = F0; f < F; f++) {
        int ends[2] = { c->fa[f], c->fb[f] };
        for (int z0 = 0; z0 < (asam_two_pose_type(c->ftype[f]) ? 2 : 1); z0++) {
            search_tree_node_t *node = &tr->nodes[ends[z0]];
            while (!node->label_changed) {
                node->label_changed = 1;
                tr->naffected++;
                marked[n_marked++] = (int) (node - tr->nodes);
                if (node->parent != -1)
                    node = &tr->nodes[node->parent];
                else
                    break;
            }
        }
    }

    /* evaluation points of the new factors: l_point for xyt (plain or robust), state for xytpos */
    int nf = F - F0;
    double *pts = gctx_stage(c, 6 * nf);
    for (int k = 0; k < nf; k++) {
        int f = F0 + k;
        if (asam_two_pose_type(c->ftype[f])) {
            memcpy(pts + 6 * (size_t) k, node_at(graph, c->fa[f])->l_point, 3 * sizeof(double));
            memcpy(pts + 6 * (size_t) k + 3, node_at(graph, c->fb[f])->l_point, 3 * sizeof(double));
        } else {
            memcpy(pts + 6 * (size_t) k, node_at(graph, c->fa[f])->state, 3 * sizeof(double));
            memset(pts + 6 * (size_t) k + 3, 0, 3 * sizeof(double));
        }
    }

    /* symbolic append + numeric re-factorisation of the marked supernodes */
    int *tasks = NULL, *nwait = NULL, *keep = NULL, ntasks = 0;
    PROF_LAP(0);
    int rc = plan_append(pl, dev, N, F, c->ftype, c->fa, c->fb, marked, n_marked, &tasks, &nwait, &keep, &ntasks);
    if (rc == 2) {
        if (g_record_steps)
            s->rec.kind = STEP_FALLBACK;
        inc_general_fallback(graph, param, s, N, F, F0);
        goto escalate;
    }
    if (rc != 0)
        asam_fatal("april_graph_cholesky_inc: %s %s", g_error, asam_last_error());
    if (g_record_steps)
        rec_tasks(&s->rec, ntasks, tasks, nwait, keep);
    int policy_escalate = 0;
    if (s->policy) {
        aprilsam_b200_step_cost_t cost;
        memset(&cost, 0, sizeof(cost));
        plan_work(pl, tasks, ntasks, &cost.step_work, &cost.step_fronts, &cost.batch_work, &cost.batch_fronts);
        cost.naffected = tr->naffected;
        cost.nnodes = N;
        cost.start_over = tr->start_over;
        policy_escalate = s->policy(&cost, s->policy_user) != 0;
    }
    PROF_LAP(1);
    if (param->show_timing)
        stamp(&tp, "mark paths, symbolic append");
    DEV_OK(asam_step_begin(dev)); /* record the step's kernels; one upload flush at asam_step_run */
    DEV_OK(asam_linearize(dev, F0, nf, pts));
    DEV_OK(asam_factor(dev, ntasks, tasks, nwait, keep));
    param->factor_num = F;
    PROF_LAP(2);

    /* tree append (:550) */
    tree_append_from_plan(tr, pl, marked, n_marked, old_root_pos, N);
    param->nreordering = N;
    PROF_LAP(3);

    /* solve (:563, :578-597): which supernodes does the traversal need? */
    {
        double *x = solver_x(s, N);
        int qbase = 0;
        int fstatus = 0;
        if (tr->naffected > 5) {
            if (g_record_steps)
                s->rec.kind = STEP_FULL;
            DEV_OK(asam_backsolve_full(dev));
            DEV_OK(asam_step_run(dev));
            DEV_OK(asam_download_x_status(dev, 0, N, x, &fstatus));
        } else {
            /* visited = marked nodes + their children; close under ancestors.  Per supernode the first
             * wanted pose: the back-substitution of a supernode stops there (cta_backsolve, jcol) */
            if (pl->sn_cap > s->stamp_cap) {
                s->sn_stamp = realloc(s->sn_stamp, sizeof(int) * (size_t) pl->sn_cap);
                s->sn_jf = realloc(s->sn_jf, sizeof(int) * (size_t) pl->sn_cap);
                s->sn_bt = realloc(s->sn_bt, sizeof(int) * 2 * (size_t) pl->sn_cap);
                memset(s->sn_stamp + s->stamp_cap, 0, sizeof(int) * (size_t) (pl->sn_cap - s->stamp_cap));
                s->stamp_cap = pl->sn_cap;
            }
            if (++s->stamp_epoch == INT_MAX) {
                memset(s->sn_stamp, 0, sizeof(int) * (size_t) s->stamp_cap);
                s->stamp_epoch = 1;
            }
            int *stamp = s->sn_stamp, *jf = s->sn_jf, *bt = s->sn_bt;
            const int ep = s->stamp_epoch;
            int nbt = 0, qmin = N;
            for (int i = 0; i < n_marked; i++) {
                search_tree_node_t *node = &tr->nodes[marked[i]];
                for (int ci = -1; ci < node->nchildren; ci++) {
                    int v = ci < 0 ? marked[i] : node->children[ci];
                    int q = pl->node2q[v], sn0 = pl->sn_of_q[q], sn = sn0;
                    while (sn >= 0 && stamp[sn] != ep) {
                        stamp[sn] = ep;
                        jf[sn] = pl->desc[sn].cb;
                        bt[nbt++] = sn;
                        if (pl->desc[sn].first < qmin)
                            qmin = pl->desc[sn].first;
                        sn = pl->desc[sn].parent;
                    }
                    if (q - pl->desc[sn0].first < jf[sn0])
                        jf[sn0] = q - pl->desc[sn0].first;
                }
            }
            /* parents before children: descending supernode id */
            for (int i = 1; i < nbt; i++) {
                int v = bt[i], j = i - 1;
                while (j >= 0 && bt[j] < v) {
                    bt[j + 1] = bt[j];
                    j--;
                }
                bt[j + 1] = v;
            }
            int *bfirst = bt + pl->sn_cap;
            for (int i = 0; i < nbt; i++)
                bfirst[i] = jf[bt[i]] < pl->desc[bt[i]].cb ? jf[bt[i]] : 0;
            DEV_OK(asam_backsolve(dev, nbt, bt, bfirst));
            /* a handful of single-CTA fronts: the whole step in ONE launch, results through pinned memory */
            int small = nbt <= ASAM_SMALL_MAX_BS && ntasks <= ASAM_SMALL_MAX_TASKS && asam_step_small_supported(dev);
            for (int t = 0; small && t < ntasks; t++)
                small = ((nwait[t] >> 24) & 0x7f) <= 1;
            if (small) {
                int xd = 0;
                for (int i = 0; i < nbt; i++)
                    xd += 3 * pl->desc[bt[i]].cb;
                double *xc = gctx_stage(c, 6 * nf + xd) + 6 * (size_t) nf; /* behind the evaluation points */
                int rs = asam_step_run_small(dev, xc, xd, &fstatus);
                if (rs == 0) {
                    for (int i = 0, off = 0; i < nbt; i++) {
                        const asam_sn_desc_t *sd = &pl->desc[bt[i]];
                        memcpy(x + 3 * (size_t) sd->first, xc + off, sizeof(double) * 3 * (size_t) sd->cb);
                        off += 3 * sd->cb;
                    }
                    qbase = 0;
                    g_prof[18] += 1;
                    g_prof[19] += ntasks;
                    g_prof[20] += nbt;
                    g_prof[21] += xd;
                } else if (rs == 2) {
                    small = 0;
                } else {
                    asam_fatal("april_graph_cholesky_inc: %s", asam_last_error());
                }
            }
            if (!small) {
                DEV_OK(asam_step_run(dev));
                qbase = qmin;
                DEV_OK(asam_download_x_status(dev, qbase, N - qbase, x, &fstatus));
            }
            if (g_record_steps) {
                s->rec.kind = small ? STEP_SMALL : STEP_PRUNED;
                rec_bt(&s->rec, nbt, bt, bfirst);
            }
        }
        PROF_LAP(4);
        report_factor_status(s, fstatus, "april_graph_cholesky_inc");
        PROF_LAP(5);
        if (param->show_timing)
            stamp(&tp, "H2D, kernels, D2H of solution");
        apply_solution(s, tr, x, qbase);
        PROF_LAP(6);
        if (tr->naffected > 5)
            g_prof[17] += 1;
        if (param->show_timing) {
            stamp(&tp, "solve_node bookkeeping");
            stamps_display(&tp, dev);
        }
    }
    free(tasks);
    free(nwait);
    free(keep);

    if (policy_escalate) /* the deterministic stand-in for the wall-clock rule (:556-559): same effect */
        param->tr->start_over = INT_MAX;

escalate:
    /* too many poses moved since the last batch: relinearise everything (:566-575) */
    if (param->tr->start_over > param->nthreshold) {
        free(param->ordering);
        param->ordering = NULL;
        struct timespec t0, t1;
        clock_gettime(CLOCK_MONOTONIC, &t0);
        april_graph_cholesky(graph, param);
        clock_gettime(CLOCK_MONOTONIC, &t1);
        param->batch_time = (t1.tv_sec - t0.tv_sec) * 1e3 + (t1.tv_nsec - t0.tv_nsec) * 1e-6;
        g_prof[7] += param->batch_time;
        g_prof[10] += 1;
        param->tr->start_over = 0;
        param->tr->nlinearized_nodes = 0;
        if (g_record_steps)
            solver_of(param)->rec.escalated = 1;
    }
}

/* A factor between two already-solved poses changes the structure of old rows and may
 * re-parent old nodes.  Keep the elimination order, rebuild the symbolic plan for the whole
 * graph and re-factor everything WITHOUT relinearising (the Hessian in HBM is kept and the
 * new factors are added to it), then solve like a full-traversal incremental step. */
static void inc_general_fallback(april_graph_t *graph, april_graph_cholesky_param_t *param, solver_t *s, int N, int F,
                                 int F0)
{
    gctx_t *c = s->gc;
    asam_dev_t *dev = c->dev;
    plan_t *pl = &s->plan;
    search_tree_t *old = param->tr;
    int N0 = pl->N, nf = F - F0;
    int old_slots = pl->n_slots;
    /* the slot numbering is rebuilt from the factor list in order, so old slots keep their ids */
    if (plan_build_with_order(pl, dev, N, F, c->ftype, c->fa, c->fb, param->ordering, N0) != 0)
        asam_fatal("april_graph_cholesky_inc: %s %s", g_error, asam_last_error());
    s->plan.struct_hash = 0; /* order differs from a fresh batch: never reuse for one */
    DEV_OK(asam_hessian_clear_range(dev, N0, N - N0, old_slots, pl->n_slots - old_slots));
    double *pts = c->stage; /* filled by the caller */
    DEV_OK(asam_linearize(dev, F0, nf, pts));
    DEV_OK(asam_factor_full(dev));
    DEV_OK(asam_backsolve_full(dev));
    double *x = solver_x(s, N);
    DEV_OK(asam_download_x(dev, 0, N, x));
    check_factor_status(s, "april_graph_cholesky_inc");

    search_tree_t *tr = tree_from_plan(pl, graph);
    tr->delta_xy = old->delta_xy;
    tr->delta_theta = old->delta_theta;
    tr->start_over = old->start_over;
    tr->total_delta_xy = old->total_delta_xy;
    tr->nlinearized_nodes = old->nlinearized_nodes;
    memcpy(tr->linearized_nodes, old->linearized_nodes, sizeof(int) * (size_t) old->nlinearized_nodes);
    for (int i = 0; i < old->nnodes && i < N; i++)
        tr->nodes[i].label_relinearized = old->nodes[i].label_relinearized;
    tr->naffected = old->naffected > 5 ? old->naffected : 6; /* force the full traversal */
    search_tree_destroy(old);
    param->tr = tr;
    param->factor_num = F;
    param->nreordering = N;
    apply_solution(s, tr, x, 0);
}

/* aprilsam.c:578-597.  Public in the reference header; with the factor in HBM there is
 * nothing for a caller to do with it beyond what april_graph_cholesky_inc already did, so it
 * re-runs the full back-substitution + bookkeeping on the current factor. */
ASAM_API void april_graph_cholesky_inc_solver(april_graph_t *graph, april_graph_cholesky_param_t *param, int *idxs)
{
    (void) idxs;
    if (!param->nreordering || !param->chol || !param->tr)
        return;
    solver_t *s = solver_of(param);
    if (s->gc->graph != graph || !s->plan_valid)
        return;
    int N = s->plan.N;
    double *x = solver_x(s, N);
    DEV_OK(asam_backsolve_full(s->gc->dev));
    DEV_OK(asam_download_x(s->gc->dev, 0, N, x));
    int keep = param->tr->naffected;
    param->tr->naffected = 6;
    apply_solution(s, param->tr, x, 0);
    param->tr->naffected = keep;
}

/* ---- test-only accessors (tools/gpu_diag.py, tests/) ------------------------------------------ */
ASAM_API void *asam_dbg_dev_of_graph(april_graph_t *g)
{
    for (gctx_t *c = g_ctx_list; c; c = c->next)
        if (c->graph == g)
            return c->dev;
    return NULL;
}

ASAM_API void *asam_dbg_plan_of_param(april_graph_cholesky_param_t *param)
{
    solver_t *s = param && param->chol ? solver_of(param) : NULL;
    return s ? (void *) &s->plan : NULL;
}

/* Step records: off by default (the solve path then only tests the flag). */
ASAM_API void asam_dbg_record_steps(int on) { g_record_steps = on != 0; }

/* The last april_graph_cholesky_inc on param: hdr = {kind (STEP_*), escalated to a batch, ntasks, nbt}; the factor
 * task list (tasks, nwait, keep: as given to asam_factor, up to tcap) and the back-solve list (bt, bfirst: as given
 * to asam_backsolve, up to bcap).  Returns -1 without a solver. */
ASAM_API int asam_dbg_last_step(april_graph_cholesky_param_t *param, int *hdr, int *tasks, int *nwait, int *keep,
                                int tcap, int *bt, int *bfirst, int bcap)
{
    solver_t *s = param && param->chol ? solver_of(param) : NULL;
    if (!s)
        return -1;
    const step_rec_t *r = &s->rec;
    hdr[0] = r->kind;
    hdr[1] = r->escalated;
    hdr[2] = r->ntasks;
    hdr[3] = r->nbt;
    int nt = r->ntasks < tcap ? r->ntasks : tcap, nb = r->nbt < bcap ? r->nbt : bcap;
    if (nt > 0) {
        memcpy(tasks, r->tasks, sizeof(int) * (size_t) nt);
        memcpy(nwait, r->nwait, sizeof(int) * (size_t) nt);
        memcpy(keep, r->keep, sizeof(int) * (size_t) nt);
    }
    if (nb > 0) {
        memcpy(bt, r->bt, sizeof(int) * (size_t) nb);
        memcpy(bfirst, r->bfirst, sizeof(int) * (size_t) nb);
    }
    return 0;
}
