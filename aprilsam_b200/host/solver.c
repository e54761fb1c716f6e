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
    /* per factor: re-uploaded by gctx_verify_factors (an edit of z / W / loss) since the last batch linearised it, so
     * HBM no longer holds what the Hessian was built from; all_stale: the mirror was rebuilt after a replaced factor */
    unsigned char *fstale;
    int n_stale, all_stale;
    unsigned remove_epoch; /* aprilsam_b200_remove_factors calls on this graph (solvers that missed one are stale) */
    unsigned relin_epoch;  /* aprilsam_b200_relinearize_poses calls on this graph (likewise) */
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
    free(c->fstale);
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

/* Mirror factors [c->nf_dev, F) into HBM (factors leave only through aprilsam_b200_remove_factors, which compacts the
 * mirror itself). */
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
        c->fstale = realloc(c->fstale, (size_t) c->fcap);
    }
    memset(c->fstale + c->nf_dev, 0, (size_t) (F - c->nf_dev));
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
            c->fstale[i] = 1;
            changed = 1;
            if (i < lo)
                lo = i;
            if (i > hi)
                hi = i;
        }
    }
    if (structural) {
        c->all_stale = 1;
        return 2;
    }
    if (!changed)
        return 0;
    c->n_stale = 1;
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
/* a step solved over a pruned traversal records its kind (STEP_PRUNED, STEP_REMOVE, STEP_RELIN), over the full one that
 * kind + 1 */
enum {
    STEP_NONE = 0, STEP_SMALL = 1, STEP_PRUNED = 2, STEP_FULL = 3, STEP_FALLBACK = 4, STEP_REMOVE = 5, STEP_REMOVE_FULL = 6,
    STEP_RELIN = 7, STEP_RELIN_FULL = 8
};

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
    /* what the Hessian in HBM was built from, for aprilsam_b200_remove_factors: the last batch put lam on the diagonal
     * of poses [0, lam_n); priors added by incremental steps were evaluated at the states staged then (pr_st, 3
     * doubles per entry, ascending factor index pr_f); a removal since the batch (removed) has left dead slots */
    double lam;
    int lam_n;
    int *pr_f;
    double *pr_st;
    int n_pr, pr_cap;
    int removed;
    unsigned epoch, relin_epoch; /* gc->remove_epoch / gc->relin_epoch as of this solver's last call */
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
    free(s->pr_f);
    free(s->pr_st);
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
        s->epoch = s->gc->remove_epoch;
        s->relin_epoch = s->gc->relin_epoch;
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

/* Why the Hessian and factor in HBM no longer describe what this solver last solved, or NULL: another param on the same
 * graph removed factors or relinearised poses since */
static const char *stale_reason(const solver_t *s)
{
    if (s->epoch != s->gc->remove_epoch)
        return "factors were removed from this graph through another param since this one last solved it";
    if (s->relin_epoch != s->gc->relin_epoch)
        return "poses of this graph were relinearised in place through another param since this one last solved it";
    return NULL;
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
    if (stale_reason(s)) { /* another solver removed factors (this plan may match the counts, not the graph) or relinearised */
        s->plan_valid = 0;
        s->tree_fresh = 0;
        s->epoch = c->remove_epoch;
        s->relin_epoch = c->relin_epoch;
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
    /* this linearisation is what a later removal rebuilds from */
    s->lam = param->tikhanov > 0 ? param->tikhanov : 0.0;
    s->lam_n = N;
    s->n_pr = 0;
    s->removed = 0;
    if (c->n_stale || c->all_stale) {
        memset(c->fstale, 0, (size_t) c->nf_dev);
        c->n_stale = c->all_stale = 0;
    }

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

/* The solve of an incremental step, a removal or an in-place relinearisation (:563, :578-597), after its
 * re-factorisation was recorded (asam_step_begin ... asam_factor): naffected > 5 back-substitutes every pose, otherwise
 * only the supernodes the traversal visits (the marked poses and their children, closed under ancestors), each from its
 * first wanted pose (bfirst).  Runs the recorded step, downloads x with the factorisation status and applies the
 * solution (apply_solution).  kind: STEP_PRUNED for april_graph_cholesky_inc, STEP_REMOVE / STEP_RELIN for the rebuild
 * steps, which never take the one-launch k_step (it knows only the kernels of a step) and leave the step counters of
 * the host profile alone.  stage_off: doubles of the staging area still in use. */
static void step_solve(april_graph_cholesky_param_t *param, solver_t *s, const int *marked, int n_marked, int ntasks,
                       const int *nwait, int kind, int stage_off, stamps_t *tp)
{
    PROF_BEGIN();
    gctx_t *c = s->gc;
    asam_dev_t *dev = c->dev;
    const plan_t *pl = &s->plan;
    search_tree_t *tr = param->tr;
    const int N = pl->N;
    const int rebuild = kind != STEP_PRUNED;
    const char *where = kind == STEP_REMOVE  ? "aprilsam_b200_remove_factors"
                        : kind == STEP_RELIN ? "aprilsam_b200_relinearize_poses"
                                             : "april_graph_cholesky_inc";
    double *x = solver_x(s, N);
    int qbase = 0;
    int fstatus = 0;
    if (tr->naffected > 5) {
        if (g_record_steps)
            s->rec.kind = kind + 1;
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
        int small = !rebuild && nbt <= ASAM_SMALL_MAX_BS && ntasks <= ASAM_SMALL_MAX_TASKS && asam_step_small_supported(dev);
        for (int t = 0; small && t < ntasks; t++)
            small = ((nwait[t] >> 24) & 0x7f) <= 1;
        if (small) {
            int xd = 0;
            for (int i = 0; i < nbt; i++)
                xd += 3 * pl->desc[bt[i]].cb;
            double *xc = gctx_stage(c, stage_off + xd) + stage_off; /* behind the evaluation points */
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
                asam_fatal("%s: %s", where, asam_last_error());
            }
        }
        if (!small) {
            DEV_OK(asam_step_run(dev));
            qbase = qmin;
            DEV_OK(asam_download_x_status(dev, qbase, N - qbase, x, &fstatus));
        }
        if (g_record_steps) {
            s->rec.kind = small ? STEP_SMALL : kind;
            rec_bt(&s->rec, nbt, bt, bfirst);
        }
    }
    if (!rebuild)
        PROF_LAP(4);
    report_factor_status(s, fstatus, where);
    if (!rebuild)
        PROF_LAP(5);
    if (param->show_timing)
        stamp(tp, "H2D, kernels, D2H of solution");
    apply_solution(s, tr, x, qbase);
    if (!rebuild) {
        PROF_LAP(6);
        if (tr->naffected > 5)
            g_prof[17] += 1;
    }
    if (param->show_timing) {
        stamp(tp, "solve_node bookkeeping");
        stamps_display(tp, dev);
    }
}

/* Priors added by incremental steps: the state each was evaluated at (a removal rebuilds them there) */
static void prior_record(solver_t *s, int f, const double *st)
{
    if (s->n_pr == s->pr_cap) {
        s->pr_cap = s->pr_cap ? 2 * s->pr_cap : 16;
        s->pr_f = realloc(s->pr_f, sizeof(int) * (size_t) s->pr_cap);
        s->pr_st = realloc(s->pr_st, sizeof(double) * 3 * (size_t) s->pr_cap);
    }
    s->pr_f[s->n_pr] = f;
    memcpy(s->pr_st + 3 * (size_t) s->n_pr++, st, 3 * sizeof(double));
}

/* The recorded state of prior f, or NULL for a prior present at the last batch (evaluated at its l_point) */
static const double *prior_point(const solver_t *s, int f)
{
    int lo = 0, hi = s->n_pr;
    while (lo < hi) {
        int mid = (lo + hi) / 2;
        if (s->pr_f[mid] < f)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo < s->n_pr && s->pr_f[lo] == f ? s->pr_st + 3 * (size_t) lo : NULL;
}

static void step_escalate(april_graph_t *graph, april_graph_cholesky_param_t *param);

/* The points factor f of the mirror was evaluated at for the Hessian in HBM (a then b): the l_points of its poses for an
 * xyt factor (plain or robust), the recorded state for a prior added by a step, the l_point of its pose for a prior
 * present at the last batch */
static void eval_point(const solver_t *s, april_graph_t *g, int f, double *pts6)
{
    const gctx_t *c = s->gc;
    if (asam_two_pose_type(c->ftype[f])) {
        memcpy(pts6, node_at(g, c->fa[f])->l_point, 3 * sizeof(double));
        memcpy(pts6 + 3, node_at(g, c->fb[f])->l_point, 3 * sizeof(double));
        return;
    }
    const double *st = prior_point(s, f);
    memcpy(pts6, st ? st : node_at(g, c->fa[f])->l_point, 3 * sizeof(double));
    memset(pts6 + 3, 0, 3 * sizeof(double));
}


ASAM_API void april_graph_cholesky_inc(april_graph_t *graph, april_graph_cholesky_param_t *param)
{
    int N = zarray_size(graph->nodes), F = zarray_size(graph->factors);
    if (N == 0 || F == 0)
        return;
    if (!param->chol)
        return;
    solver_t *s = solver_of(param);
    if (s->gc->graph == graph && stale_reason(s)) {
        asam_set_error("april_graph_cholesky_inc: %s; nothing was done (solve with april_graph_cholesky first)",
                       stale_reason(s));
        return;
    }
    if (param->factor_num == F)
        return;
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
            prior_record(s, f, pts + 6 * (size_t) k);
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

    step_solve(param, s, marked, n_marked, ntasks, nwait, STEP_PRUNED, 6 * nf, &tp);
    free(tasks);
    free(nwait);
    free(keep);

    if (policy_escalate) /* the deterministic stand-in for the wall-clock rule (:556-559): same effect */
        param->tr->start_over = INT_MAX;

escalate:
    step_escalate(graph, param);
}

/* too many poses moved since the last batch: relinearise everything (:566-575) */
static void step_escalate(april_graph_t *graph, april_graph_cholesky_param_t *param)
{
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
    if (s->removed) {
        /* a removal left slots that the rebuild dropped, so later slots were renumbered: the whole Hessian is
         * built again, every factor at the point it was evaluated at (no relinearisation) */
        double *all = malloc(sizeof(double) * 6 * (size_t) F);
        for (int f = 0; f < F; f++)
            eval_point(s, graph, f, all + 6 * (size_t) f);
        DEV_OK(asam_hessian_reset(dev, N, pl->n_slots, s->lam_n, s->lam));
        DEV_OK(asam_linearize(dev, 0, F, all));
        free(all);
        s->removed = 0;
    } else {
        DEV_OK(asam_hessian_clear_range(dev, N0, N - N0, old_slots, pl->n_slots - old_slots));
        double *pts = c->stage; /* filled by the caller */
        DEV_OK(asam_linearize(dev, F0, nf, pts));
    }
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

/* ---- factor removal (extension) ------------------------------------------------------------------------------ */
static gctx_t *gctx_find(april_graph_t *g)
{
    pthread_mutex_lock(&g_ctx_lock);
    gctx_t *hit = NULL;
    for (gctx_t *c = g_ctx_list; c; c = c->next)
        if (c->graph == g) {
            hit = c;
            break;
        }
    pthread_mutex_unlock(&g_ctx_lock);
    return hit;
}

/* Drop the removed factors (sorted[0..n), ascending) from the host mirror and upload what moved: HBM then holds the
 * remaining factors in their new order.  Values come from the mirror, not from the caller's structs, so an edit the
 * mirror has not seen yet stays unseen until the next batch checks it.  Factors not mirrored yet are skipped. */
static void gctx_remove_factors(gctx_t *c, int n, const int *sorted)
{
    int m = 0;
    while (m < n && sorted[m] < c->nf_dev)
        m++;
    if (m == 0)
        return;
    const int first = sorted[0], F = c->nf_dev;
    int out = first;
    for (int f = first, k = 0; f < F; f++) {
        if (k < m && sorted[k] == f) {
            k++;
            continue;
        }
        c->ftype[out] = c->ftype[f];
        c->fa[out] = c->fa[f];
        c->fb[out] = c->fb[f];
        memcpy(c->zw + 12 * (size_t) out, c->zw + 12 * (size_t) f, 12 * sizeof(double));
        c->floss[out] = c->floss[f];
        c->fk[out] = c->fk[f];
        c->fstale[out] = c->fstale[f];
        out++;
    }
    c->nf_dev = out;
    const int cnt = out - first;
    if (cnt <= 0)
        return;
    double *zw = malloc(sizeof(double) * 12 * (size_t) cnt);
    double *z = zw, *W = zw + 3 * (size_t) cnt;
    int robust = 0;
    for (int k = 0; k < cnt; k++) {
        memcpy(z + 3 * (size_t) k, c->zw + 12 * (size_t) (first + k), 3 * sizeof(double));
        memcpy(W + 9 * (size_t) k, c->zw + 12 * (size_t) (first + k) + 3, 9 * sizeof(double));
        robust |= c->floss[first + k] != 0;
    }
    DEV_OK(asam_upload_factors(c->dev, first, cnt, c->ftype + first, c->fa + first, c->fb + first, z, W));
    if (robust)
        DEV_OK(asam_upload_loss(c->dev, first, cnt, c->floss + first, c->fk + first));
    free(zw);
}

/* Take the factors out of graph->factors, the others keeping their order; hand them to the caller (factor_idx order)
 * or destroy them */
static void graph_splice(april_graph_t *g, int n, const int *factor_idx, const int *sorted,
                         april_graph_factor_t **removed_out)
{
    april_graph_factor_t **fs = (april_graph_factor_t **) g->factors->data;
    const int F = zarray_size(g->factors);
    for (int k = 0; k < n; k++) {
        if (removed_out)
            removed_out[k] = fs[factor_idx[k]];
        else
            fs[factor_idx[k]]->destroy(fs[factor_idx[k]]);
    }
    int out = sorted[0];
    for (int f = sorted[0], k = 0; f < F; f++) {
        if (k < n && sorted[k] == f) {
            k++;
            continue;
        }
        fs[out++] = fs[f];
    }
    g->factors->size = out;
}

static int cmp_int_asc(const void *a, const void *b)
{
    int x = *(const int *) a, y = *(const int *) b;
    return (x > y) - (x < y);
}

/* sorted lookup: index of v in p[0..n) or -1 */
static int find_int(const int *p, int n, int v)
{
    int lo = 0, hi = n;
    while (lo < hi) {
        int mid = (lo + hi) / 2;
        if (p[mid] < v)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo < n && p[lo] == v ? lo : -1;
}

/* Is every pose of `dirty` still anchored once the removed factors (rm[f] = 1) are gone: a pose with a Tikhonov term
 * (it existed at the last batch, lambda > 0) or a remaining prior, or one the remaining factors connect to such a pose?
 * Breadth-first from each dirty pose, stopping at the first anchored pose.  Returns the first pose left without an
 * anchor, or -1. */
static int unanchored_pose(const solver_t *s, int N, int F, const unsigned char *rm, const int *dirty, int n_dirty,
                           const unsigned char *dirty_prior)
{
    const gctx_t *c = s->gc;
    const int lam_on = s->lam > 0.0;
    int need = 0;
    for (int i = 0; i < n_dirty && !need; i++)
        need = !((lam_on && dirty[i] < s->lam_n) || dirty_prior[i]);
    if (!need)
        return -1;
    /* adjacency of the remaining factors; a prior marks its pose */
    int *deg = calloc((size_t) N + 1, sizeof(int));
    unsigned char *prior = calloc((size_t) N, 1);
    for (int f = 0; f < F; f++) {
        if (rm[f])
            continue;
        if (asam_two_pose_type(c->ftype[f])) {
            deg[c->fa[f] + 1]++;
            deg[c->fb[f] + 1]++;
        } else {
            prior[c->fa[f]] = 1;
        }
    }
    for (int i = 0; i < N; i++)
        deg[i + 1] += deg[i];
    int *adj = malloc(sizeof(int) * (size_t) (deg[N] + 1)), *fill = malloc(sizeof(int) * (size_t) N);
    memcpy(fill, deg, sizeof(int) * (size_t) N);
    for (int f = 0; f < F; f++)
        if (!rm[f] && asam_two_pose_type(c->ftype[f])) {
            adj[fill[c->fa[f]]++] = c->fb[f];
            adj[fill[c->fb[f]]++] = c->fa[f];
        }
    int *seen = calloc((size_t) N, sizeof(int)), *queue = fill; /* fill is free again */
    int bad = -1;
    for (int i = 0; i < n_dirty && bad < 0; i++) {
        int head = 0, tail = 0, found = 0;
        queue[tail++] = dirty[i];
        seen[dirty[i]] = i + 1;
        while (head < tail && !found) {
            int v = queue[head++];
            if ((lam_on && v < s->lam_n) || prior[v]) {
                found = 1;
                break;
            }
            for (int e = deg[v]; e < deg[v + 1]; e++)
                if (seen[adj[e]] != i + 1) {
                    seen[adj[e]] = i + 1;
                    queue[tail++] = adj[e];
                }
        }
        if (!found)
            bad = dirty[i];
    }
    free(deg);
    free(prior);
    free(adj);
    free(fill);
    free(seen);
    return bad;
}

/* ---- rebuild steps: the second half of a removal and of an in-place relinearisation ------------------------------- */
/* The Hessian entries a rebuild step overwrites and the factors they are summed from.  The caller names the dirty poses
 * and slots (ascending, distinct); rebuild_scan finds every factor on them with one pass over the factor list (O(F)),
 * rebuild_tables evaluates them, rebuild_step re-factors and solves. */
typedef struct rebuild {
    ivec_t dirty, dslot;
    int *pcnt, *scnt;      /* factors per dirty pose / dirty slot */
    unsigned char *dprior; /* per dirty pose: a prior sits on it */
    ivec_t hit;            /* (f, dirty pose index of a or -1, of b or -1, dirty slot index or -1) per factor found */
    int stale;             /* the first factor found whose mirror gctx_verify_factors re-uploaded since the last batch */
    /* the tables of asam_hessian_rebuild: entries [pptr[i], pptr[i+1]) for dirty pose i, [sptr[j], sptr[j+1]) for
     * dirty slot j (sptr[0] = pptr[n_dirty]), each a factor index and its evaluation points; lambda per dirty pose */
    int *pptr, *sptr, *ent_f, n_ent;
    double *ent_pts, *lamv;
} rebuild_t;

static void ivec_sort_unique(ivec_t *v)
{
    qsort(v->p, (size_t) v->n, sizeof(int), cmp_int_asc);
    int w = 0;
    for (int i = 0; i < v->n; i++)
        if (i == 0 || v->p[i] != v->p[i - 1])
            v->p[w++] = v->p[i];
    v->n = w;
}

static void rebuild_free(rebuild_t *rb)
{
    ivec_free(&rb->dirty);
    ivec_free(&rb->dslot);
    ivec_free(&rb->hit);
    free(rb->pcnt);
    free(rb->scnt);
    free(rb->dprior);
    free(rb->pptr);
    free(rb->sptr);
    free(rb->ent_f);
    free(rb->ent_pts);
    free(rb->lamv);
    memset(rb, 0, sizeof(*rb));
}

/* Per dirty pose and per dirty slot, its factors in index order, skipping those with rm[f] set (rm may be NULL) */
static void rebuild_scan(rebuild_t *rb, const solver_t *s, int F, const unsigned char *rm)
{
    const gctx_t *c = s->gc;
    const int *dirty = rb->dirty.p, *dslot = rb->dslot.p, n_dirty = rb->dirty.n, n_dslot = rb->dslot.n;
    rb->pcnt = calloc((size_t) n_dirty + 1, sizeof(int));
    rb->scnt = calloc((size_t) n_dslot + 1, sizeof(int));
    rb->dprior = calloc((size_t) n_dirty + 1, 1);
    rb->stale = -1;
    for (int f = 0; f < F; f++) {
        if (rm && rm[f])
            continue;
        int two = asam_two_pose_type(c->ftype[f]);
        int ia = find_int(dirty, n_dirty, c->fa[f]), ib = two ? find_int(dirty, n_dirty, c->fb[f]) : -1;
        if (ia < 0 && ib < 0)
            continue;
        int is = two && ia >= 0 && ib >= 0 ? find_int(dslot, n_dslot, s->plan.fslot[f]) : -1;
        if (c->fstale[f] && rb->stale < 0)
            rb->stale = f;
        ivec_push(&rb->hit, f);
        ivec_push(&rb->hit, ia);
        ivec_push(&rb->hit, ib);
        ivec_push(&rb->hit, is);
        if (ia >= 0)
            rb->pcnt[ia]++;
        if (ib >= 0)
            rb->pcnt[ib]++;
        if (is >= 0)
            rb->scnt[is]++;
        if (!two)
            rb->dprior[ia] = 1;
    }
}

/* The tables, every factor found at its evaluation point now (eval_point).  An entry holds the factor's index once the
 * n_rm factors rm_sorted[] (ascending) have left the list: the index after a removal's compaction. */
static void rebuild_tables(rebuild_t *rb, const solver_t *s, april_graph_t *g, int n_rm, const int *rm_sorted)
{
    const int n_dirty = rb->dirty.n, n_dslot = rb->dslot.n, n_hit = rb->hit.n / 4;
    int *pptr = malloc(sizeof(int) * ((size_t) n_dirty + 1)), *sptr = malloc(sizeof(int) * ((size_t) n_dslot + 1));
    pptr[0] = 0;
    for (int i = 0; i < n_dirty; i++)
        pptr[i + 1] = pptr[i] + rb->pcnt[i];
    sptr[0] = pptr[n_dirty];
    for (int i = 0; i < n_dslot; i++)
        sptr[i + 1] = sptr[i] + rb->scnt[i];
    const int n_ent = sptr[n_dslot];
    int *ent_f = malloc(sizeof(int) * ((size_t) n_ent + 1));
    double *ent_pts = malloc(sizeof(double) * 6 * ((size_t) n_ent + 1));
    double *lamv = malloc(sizeof(double) * ((size_t) n_dirty + 1));
    int *pcur = rb->pcnt, *scur = rb->scnt; /* the counts become fill cursors */
    memcpy(pcur, pptr, sizeof(int) * (size_t) n_dirty);
    memcpy(scur, sptr, sizeof(int) * (size_t) n_dslot);
    for (int h = 0; h < n_hit; h++) {
        const int *e = rb->hit.p + 4 * h;
        const int f = e[0], ia = e[1], ib = e[2], is = e[3];
        int below = 0, hi = n_rm; /* f less the removed factors before it */
        while (below < hi) {
            int mid = (below + hi) / 2;
            if (rm_sorted[mid] < f)
                below = mid + 1;
            else
                hi = mid;
        }
        double pts[6];
        eval_point(s, g, f, pts);
        int dst[3] = { ia >= 0 ? pcur[ia]++ : -1, ib >= 0 ? pcur[ib]++ : -1, is >= 0 ? scur[is]++ : -1 };
        for (int j = 0; j < 3; j++)
            if (dst[j] >= 0) {
                ent_f[dst[j]] = f - below;
                memcpy(ent_pts + 6 * (size_t) dst[j], pts, sizeof(pts));
            }
    }
    for (int i = 0; i < n_dirty; i++)
        lamv[i] = rb->dirty.p[i] < s->lam_n ? s->lam : 0.0;
    rb->pptr = pptr;
    rb->sptr = sptr;
    rb->ent_f = ent_f;
    rb->ent_pts = ent_pts;
    rb->lamv = lamv;
    rb->n_ent = n_ent;
}

/* Re-factor and solve a rebuild step whose uploads are recorded since asam_step_begin: mark the root paths of the dirty
 * poses as if factors had been added on them (:482-498), overwrite the dirty entries (asam_hessian_rebuild), re-factor
 * the marked supernodes (plan_refactor), solve like a step (step_solve with kind STEP_REMOVE or STEP_RELIN), then the
 * policy hook and the nthreshold escalation of a step. */
static void rebuild_step(rebuild_t *rb, april_graph_t *graph, april_graph_cholesky_param_t *param, solver_t *s, int kind,
                         stamps_t *tp)
{
    plan_t *pl = &s->plan;
    search_tree_t *tr = param->tr;
    const int N = pl->N;
    int *marked = solver_scratch(s, 2 * N + 16) + N + 8; /* upper half: apply_solution uses the lower */
    int n_marked = 0;
    tr->naffected = 0;
    for (int i = 0; i < rb->dirty.n; i++) {
        search_tree_node_t *node = &tr->nodes[rb->dirty.p[i]];
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
    int *tasks = NULL, *nwait = NULL, *keep = NULL, ntasks = 0;
    plan_refactor(pl, marked, n_marked, &tasks, &nwait, &keep, &ntasks);
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
    if (param->show_timing)
        stamp(tp, "scan, mark paths, rebuild tables");
    DEV_OK(asam_hessian_rebuild(s->gc->dev, rb->dirty.n, rb->dirty.p, rb->pptr, rb->dslot.n, rb->dslot.p, rb->sptr,
                                rb->n_ent, rb->ent_f, rb->ent_pts, rb->lamv));
    DEV_OK(asam_factor(s->gc->dev, ntasks, tasks, nwait, keep));
    step_solve(param, s, marked, n_marked, ntasks, nwait, kind, 0, tp);
    free(tasks);
    free(nwait);
    free(keep);
    if (policy_escalate)
        tr->start_over = INT_MAX;
    step_escalate(graph, param);
}

/* What a rebuild step needs of the solver it continues, checked before anything changes: NULL, or why not (and *tail,
 * the advice that follows it in the error text).  sharded: the text for a sharded batch solve. */
static const char *rebuild_refusal(const solver_t *s, april_graph_cholesky_param_t *param, april_graph_t *graph,
                                   const char *sharded, const char **tail)
{
    const gctx_t *c = s->gc;
    const int N = zarray_size(graph->nodes), F = zarray_size(graph->factors);
    *tail = "";
    if (c->graph != graph)
        return "param does not continue a solve of this graph";
    if (!s->plan_valid)
        return "the plan was dropped (aprilsam_b200_invalidate_plan); solve again first";
    if (stale_reason(s)) {
        *tail = "; solve with april_graph_cholesky first";
        return stale_reason(s);
    }
    if (s->plan.world > 1)
        return sharded;
    if (!param->tr || N != s->plan.N || F != s->plan.n_factors || F != param->factor_num || F != c->nf_dev)
        return "poses or factors were added since the last solve (call april_graph_cholesky_inc first)";
    if (c->all_stale)
        return "a factor was replaced since the last batch solve (its HBM mirror no longer matches the linearised "
               "Hessian); solve with april_graph_cholesky first";
    return NULL;
}

ASAM_API int aprilsam_b200_remove_factors(april_graph_t *graph, april_graph_cholesky_param_t *param, int n,
                                          const int *factor_idx, april_graph_factor_t **removed_out)
{
    const char *fn = "aprilsam_b200_remove_factors";
    if (!graph || !param || !factor_idx || n < 1) {
        asam_set_error("%s: NULL graph / param / factor_idx or n < 1", fn);
        return -1;
    }
    const int N = zarray_size(graph->nodes), F = zarray_size(graph->factors);
    int *idx = malloc(sizeof(int) * (size_t) n);
    for (int k = 0; k < n; k++) {
        if (factor_idx[k] < 0 || factor_idx[k] >= F) {
            asam_set_error("%s: factor index %d (entry %d) is not in [0, %d)", fn, factor_idx[k], k, F);
            free(idx);
            return -1;
        }
        idx[k] = factor_idx[k];
    }
    qsort(idx, (size_t) n, sizeof(int), cmp_int_asc);
    for (int k = 1; k < n; k++)
        if (idx[k] == idx[k - 1]) {
            asam_set_error("%s: factor index %d is listed twice", fn, idx[k]);
            free(idx);
            return -1;
        }
    if (!param->chol) { /* never solved: only the splice (and the mirror of a graph another param solved) */
        gctx_t *c = gctx_find(graph);
        if (c) {
            gctx_remove_factors(c, n, idx);
            c->remove_epoch++;
        }
        graph_splice(graph, n, factor_idx, idx, removed_out);
        free(idx);
        return 0;
    }
    solver_t *s = solver_of(param);
    gctx_t *c = s->gc;
    const char *tail, *why = rebuild_refusal(
                          s, param, graph,
                          "the last batch solve was sharded over several GPUs; removal continues single-GPU solves only",
                          &tail);
    if (why) {
        asam_set_error("%s: %s%s", fn, why, tail);
        free(idx);
        return -1;
    }

    /* ---- validation on the unchanged state: dirty poses and slots, the remaining factors on them ---- */
    plan_t *pl = &s->plan;
    double t_scan = prof_now();
    rebuild_t rb = { 0 };
    for (int k = 0; k < n; k++) {
        int f = idx[k];
        ivec_push(&rb.dirty, c->fa[f]);
        if (asam_two_pose_type(c->ftype[f])) {
            ivec_push(&rb.dirty, c->fb[f]);
            ivec_push(&rb.dslot, pl->fslot[f]);
        }
    }
    ivec_sort_unique(&rb.dirty);
    ivec_sort_unique(&rb.dslot);
    unsigned char *rm = calloc((size_t) F, 1);
    for (int k = 0; k < n; k++)
        rm[idx[k]] = 1;
    rebuild_scan(&rb, s, F, rm);
    int bad = rb.stale < 0 ? unanchored_pose(s, N, F, rm, rb.dirty.p, rb.dirty.n, rb.dprior) : -1;
    t_scan = prof_now() - t_scan;
    free(rm);
    if (rb.stale >= 0 || bad >= 0) {
        if (rb.stale >= 0)
            asam_set_error("%s: factor %d, which shares a pose with a removed factor, was edited since the last batch "
                           "solve (its HBM mirror no longer holds the values the Hessian was built from); solve with "
                           "april_graph_cholesky first", fn, rb.stale);
        else
            asam_set_error("%s: pose %d would be left unconstrained: it was created after the last batch solve and no "
                           "remaining factor connects it to a pose of that batch or to a prior", fn, bad);
        free(idx);
        rebuild_free(&rb);
        return -1;
    }

    /* ---- from here on the removal happens ---- */
    g_prof[22] += t_scan;
    g_prof[23] += 1;
    asam_dev_t *dev = c->dev;
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
    rebuild_tables(&rb, s, graph, n, idx); /* evaluation points read before the mirror moves */

    /* ---- compaction: graph, mirror (host and HBM), plan, prior table ---- */
    DEV_OK(asam_step_begin(dev)); /* one upload flush and one synchronisation for the whole removal */
    gctx_remove_factors(c, n, idx);
    if (plan_remove_factors(pl, dev, n, idx) != 0)
        asam_fatal("%s: %s %s", fn, g_error, asam_last_error());
    {
        int o = 0;
        for (int i = 0, k = 0; i < s->n_pr; i++) {
            while (k < n && idx[k] < s->pr_f[i])
                k++;
            if (k < n && idx[k] == s->pr_f[i])
                continue;
            s->pr_f[o] = s->pr_f[i] - k;
            memmove(s->pr_st + 3 * (size_t) o, s->pr_st + 3 * (size_t) i, 3 * sizeof(double));
            o++;
        }
        s->n_pr = o;
    }
    graph_splice(graph, n, factor_idx, idx, removed_out);
    param->factor_num = F - n;
    s->removed = 1;
    c->remove_epoch++;
    s->epoch = c->remove_epoch;

    /* ---- rebuild, re-factor the root paths, solve ---- */
    rebuild_step(&rb, graph, param, s, STEP_REMOVE, &tp);
    free(idx);
    rebuild_free(&rb);
    return 0;
}

/* ---- in-place relinearisation (extension) ---------------------------------------------------------------------- */
ASAM_API int aprilsam_b200_relinearize_poses(april_graph_t *graph, april_graph_cholesky_param_t *param, int n,
                                             const int *nodes)
{
    const char *fn = "aprilsam_b200_relinearize_poses";
    if (!graph || !param || !nodes || n < 1) {
        asam_set_error("%s: NULL graph / param / nodes or n < 1", fn);
        return -1;
    }
    const int N = zarray_size(graph->nodes), F = zarray_size(graph->factors);
    /* a copy first: nodes may be param->tr->linearized_nodes, which this call edits */
    int *P = malloc(sizeof(int) * (size_t) n);
    memcpy(P, nodes, sizeof(int) * (size_t) n);
    unsigned char *inP = calloc((size_t) N + 1, 1);
    for (int k = 0; k < n; k++) {
        int bad = P[k] < 0 || P[k] >= N;
        if (bad)
            asam_set_error("%s: pose id %d (entry %d) is not in [0, %d)", fn, P[k], k, N);
        else if ((bad = inP[P[k]]))
            asam_set_error("%s: pose id %d (entry %d) is listed twice", fn, P[k], k);
        if (bad) {
            free(P);
            free(inP);
            return -1;
        }
        inP[P[k]] = 1;
    }
    const char *tail = "", *why = "param does not continue a solve of this graph";
    if (param->chol)
        why = rebuild_refusal(solver_of(param), param, graph,
                              "the last batch solve was sharded over several GPUs; relinearisation in place continues "
                              "single-GPU solves only", &tail);
    if (why) {
        asam_set_error("%s: %s%s", fn, why, tail);
        free(P);
        free(inP);
        return -1;
    }
    solver_t *s = solver_of(param);
    gctx_t *c = s->gc;
    plan_t *pl = &s->plan;

    /* ---- validation on the unchanged state: R = the factors with a pose in P; D = their poses and P; the dirty slots
     * = the slots of R's two-pose factors; then every factor on D ---- */
    double t_scan = prof_now();
    rebuild_t rb = { 0 };
    for (int k = 0; k < n; k++)
        ivec_push(&rb.dirty, P[k]);
    for (int f = 0; f < F; f++) {
        if (asam_two_pose_type(c->ftype[f])) {
            if (inP[c->fa[f]] || inP[c->fb[f]]) {
                ivec_push(&rb.dirty, c->fa[f]);
                ivec_push(&rb.dirty, c->fb[f]);
                ivec_push(&rb.dslot, pl->fslot[f]);
            }
        }
    }
    ivec_sort_unique(&rb.dirty);
    ivec_sort_unique(&rb.dslot);
    rebuild_scan(&rb, s, F, NULL);
    t_scan = prof_now() - t_scan;
    if (rb.stale >= 0) {
        asam_set_error("%s: factor %d, on a pose whose blocks the relinearisation rebuilds, was edited since the last "
                       "batch solve (its HBM mirror no longer holds the values the Hessian was built from); solve with "
                       "april_graph_cholesky first", fn, rb.stale);
        free(P);
        free(inP);
        rebuild_free(&rb);
        return -1;
    }

    /* ---- from here on the relinearisation happens ---- */
    g_prof[22] += t_scan;
    g_prof[23] += 1;
    asam_dev_t *dev = c->dev;
    search_tree_t *tr = param->tr;
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
    /* counters: the poses of P that were flagged are flagged no more */
    int cleared = 0;
    for (int k = 0; k < n; k++)
        if (tr->nodes[P[k]].label_relinearized) {
            tr->nodes[P[k]].label_relinearized = 0;
            cleared++;
        }
    if (cleared) {
        int w = 0;
        for (int i = 0; i < tr->nlinearized_nodes; i++)
            if (!inP[tr->linearized_nodes[i]])
                tr->linearized_nodes[w++] = tr->linearized_nodes[i];
        tr->nlinearized_nodes = w;
        tr->start_over -= cleared;
    }
    /* l_point = state (the batch's copy, :131-135); a prior a step added on a pose of P moves with it */
    for (int k = 0; k < n; k++) {
        april_graph_node_t *nd = node_at(graph, P[k]);
        memcpy(nd->l_point, nd->state, 3 * sizeof(double));
    }
    for (int i = 0; i < s->n_pr; i++)
        if (inP[c->fa[s->pr_f[i]]])
            memcpy(s->pr_st + 3 * (size_t) i, node_at(graph, c->fa[s->pr_f[i]])->l_point, 3 * sizeof(double));
    rebuild_tables(&rb, s, graph, 0, NULL);
    c->relin_epoch++;
    s->relin_epoch = c->relin_epoch;

    /* ---- rebuild, re-factor the root paths, solve ---- */
    DEV_OK(asam_step_begin(dev)); /* one upload flush and one synchronisation */
    rebuild_step(&rb, graph, param, s, STEP_RELIN, &tp);
    free(P);
    free(inP);
    rebuild_free(&rb);
    return 0;
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

/* ---- marginal covariances (extension) ------------------------------------------------------------ */
/* The solver whose factor describes g as it is now, or NULL with the reason in the error text. */
static solver_t *marginal_solver(april_graph_t *g, april_graph_cholesky_param_t *param, const char *fn)
{
    if (!g || !param) {
        asam_set_error("%s: NULL graph or param", fn);
        return NULL;
    }
    solver_t *s = (solver_t *) param->chol;
    if (!s || s->magic != SOLVER_MAGIC || !s->gc || s->gc->graph != g) {
        asam_set_error("%s: param does not continue a solve of this graph", fn);
        return NULL;
    }
    if (!s->plan_valid) {
        asam_set_error("%s: the plan was dropped (aprilsam_b200_invalidate_plan); solve again first", fn);
        return NULL;
    }
    if (stale_reason(s)) {
        asam_set_error("%s: %s; solve with april_graph_cholesky first", fn, stale_reason(s));
        return NULL;
    }
    if (zarray_size(g->nodes) != s->plan.N || zarray_size(g->factors) != s->plan.n_factors ||
        zarray_size(g->factors) != param->factor_num) {
        asam_set_error("%s: nodes or factors were added since the last solve (%d / %d poses, %d / %d factors)", fn,
                       zarray_size(g->nodes), s->plan.N, zarray_size(g->factors), s->plan.n_factors);
        return NULL;
    }
    if (s->plan.world > 1) {
        asam_set_error("%s: the last batch solve was sharded over %d GPUs; a rank holds only its own shards' fronts", fn,
                       s->plan.world);
        return NULL;
    }
    return s;
}

static int marginal_run(solver_t *s, int n, const int *nodes, double *out, const char *fn)
{
    asam_marg_path_t *paths = malloc(sizeof(*paths) * (size_t) n);
    int64_t z = 0;
    int hops = 0, rc = -1;
    if (plan_marginal_paths(&s->plan, n, nodes, paths, &z, &hops) != 0) {
        char why[512];
        snprintf(why, sizeof(why), "%s", g_error);
        asam_set_error("%s: %s", fn, why);
    } else if (asam_marginal_cov(s->gc->dev, n, paths, z, hops, s->plan.max_m, out) != 0) {
        asam_set_error("%s: %s", fn, asam_last_error());
    } else {
        rc = 0;
    }
    free(paths);
    return rc;
}

ASAM_API int aprilsam_b200_marginal_covariance(april_graph_t *g, april_graph_cholesky_param_t *param, int n,
                                               const int *nodes, double *out)
{
    const char *fn = "aprilsam_b200_marginal_covariance";
    if (!nodes || !out || n < 1) {
        asam_set_error("%s: NULL nodes / out or n < 1", fn);
        return -1;
    }
    solver_t *s = marginal_solver(g, param, fn);
    return s ? marginal_run(s, n, nodes, out, fn) : -1;
}

/* ---- candidate factors: Sigma_rel and Mahalanobis distance (extension) ----------------------------------- */
int64_t asam_candidate_budget = ASAM_CANDIDATE_BUDGET;

/* J = [J_a J_b] (3 x 6, row-major) of an xyt factor between a and b at their l_points */
static void candidate_jacobian(april_graph_t *g, int a, int b, double *J)
{
    double Ja[9], Jb[9];
    asam_xyt_jacobians(node_at(g, a)->l_point, node_at(g, b)->l_point, Ja, Jb);
    for (int r = 0; r < 3; r++)
        for (int k = 0; k < 3; k++) {
            J[6 * r + k] = Ja[3 * r + k];
            J[6 * r + 3 + k] = Jb[3 * r + k];
        }
}

/* Winv = W^-1 (exactly symmetric) by W = L L'; 0 unless W is exactly symmetric and positive definite */
static int spd_inverse3(const double *W, double *Winv)
{
    for (int r = 0; r < 3; r++)
        for (int c = r + 1; c < 3; c++)
            if (!(W[3 * r + c] == W[3 * c + r]))
                return 0;
    double L[9] = { 0 }, X[9] = { 0 };
    for (int j = 0; j < 3; j++) {
        double d = W[4 * j];
        for (int k = 0; k < j; k++)
            d -= L[3 * j + k] * L[3 * j + k];
        if (!(d > 0.0) || !isfinite(d))
            return 0;
        L[4 * j] = sqrt(d);
        for (int i = j + 1; i < 3; i++) {
            double v = W[3 * i + j];
            for (int k = 0; k < j; k++)
                v -= L[3 * i + k] * L[3 * j + k];
            L[3 * i + j] = v / L[4 * j];
        }
    }
    /* X = L^-1 (lower triangular), W^-1 = X' X */
    for (int c = 0; c < 3; c++)
        for (int i = c; i < 3; i++) {
            double v = i == c ? 1.0 : 0.0;
            for (int k = c; k < i; k++)
                v -= L[3 * i + k] * X[3 * k + c];
            X[3 * i + c] = v / L[4 * i];
        }
    for (int r = 0; r < 3; r++)
        for (int c = r; c < 3; c++) {
            double acc = 0.0;
            for (int k = c; k < 3; k++)
                acc += X[3 * k + r] * X[3 * k + c];
            if (!isfinite(acc))
                return 0;
            Winv[3 * r + c] = Winv[3 * c + r] = acc;
        }
    return 1;
}

/* Sigma_rel (cov9, 9 doubles per candidate, may be NULL) and d2 of k candidates whose records hold J, r, Winv and
 * has_w (ids checked by the caller).  Runs the batches of plan_candidate_batches, one asam_marginal_pairs each. */
static int candidates_run(solver_t *s, int k, const int *a, const int *b, asam_marg_pair_t *rec, double *d2,
                          double *cov9, const char *fn)
{
    const plan_t *pl = &s->plan;
    int *batch_end = malloc(sizeof(int) * (size_t) k), *pose_end = malloc(sizeof(int) * (size_t) k);
    int *poses = malloc(sizeof(int) * 2 * (size_t) k), *ia = malloc(sizeof(int) * (size_t) k);
    int *ib = malloc(sizeof(int) * (size_t) k);
    asam_marg_path_t *paths = malloc(sizeof(*paths) * 2 * (size_t) k);
    double *out = malloc(sizeof(double) * 10 * (size_t) k);
    int nb = 0, rc = 0;
    plan_candidate_batches(pl, k, a, b, asam_candidate_budget / (int64_t) sizeof(double), batch_end, &nb, poses,
                           pose_end, ia, ib);
    for (int t = 0; t < nb && rc == 0; t++) {
        const int c0 = t ? batch_end[t - 1] : 0, c1 = batch_end[t];
        const int p0 = t ? pose_end[t - 1] : 0, n = pose_end[t] - p0;
        int64_t z = 0;
        int hops = 0;
        if (plan_marginal_paths(pl, n, poses + p0, paths, &z, &hops) != 0) {
            char why[512];
            snprintf(why, sizeof(why), "%s", g_error);
            asam_set_error("%s: %s", fn, why);
            rc = -1;
            break;
        }
        for (int c = c0; c < c1; c++) {
            rec[c].pa = ia[c];
            rec[c].pb = ib[c];
        }
        if (asam_marginal_pairs(s->gc->dev, n, paths, z, hops, pl->max_m, c1 - c0, rec + c0, out) != 0) {
            asam_set_error("%s: %s", fn, asam_last_error());
            rc = -1;
            break;
        }
        for (int c = c0; c < c1; c++) {
            d2[c] = out[10 * (size_t) (c - c0)];
            if (cov9)
                memcpy(cov9 + 9 * (size_t) c, out + 10 * (size_t) (c - c0) + 1, 9 * sizeof(double));
        }
    }
    free(batch_end);
    free(pose_end);
    free(poses);
    free(ia);
    free(ib);
    free(paths);
    free(out);
    return rc;
}

ASAM_API int aprilsam_b200_candidate_mahalanobis(april_graph_t *g, april_graph_cholesky_param_t *param, int k,
                                                 const int *a, const int *b, const double *z, const double *W,
                                                 double *d2, double *cov9)
{
    const char *fn = "aprilsam_b200_candidate_mahalanobis";
    if (k < 1 || !a || !b || !z || !W || !d2) {
        asam_set_error("%s: NULL a / b / z / W / d2 or k < 1", fn);
        return -1;
    }
    solver_t *s = marginal_solver(g, param, fn);
    if (!s)
        return -1;
    const int N = s->plan.N;
    asam_marg_pair_t *rec = calloc((size_t) k, sizeof(*rec));
    int rc = 0;
    for (int c = 0; c < k && rc == 0; c++) {
        const double *zc = z + 3 * (size_t) c;
        rc = -1;
        if (a[c] < 0 || a[c] >= N || b[c] >= N)
            asam_set_error("%s: candidate %d: node %d is not in the solved graph (%d poses)", fn, c,
                           a[c] < 0 || a[c] >= N ? a[c] : b[c], N);
        else if (b[c] < -1)
            asam_set_error("%s: candidate %d: b = %d; expected a pose id, or -1 for a prior on a", fn, c, b[c]);
        else if (a[c] == b[c])
            asam_set_error("%s: candidate %d: a == b (%d)", fn, c, a[c]);
        else if (!isfinite(zc[0]) || !isfinite(zc[1]) || !isfinite(zc[2]))
            asam_set_error("%s: candidate %d: z is not finite", fn, c);
        else if (!spd_inverse3(W + 9 * (size_t) c, rec[c].Winv))
            asam_set_error("%s: candidate %d: W is not symmetric positive definite", fn, c);
        else
            rc = 0;
        if (rc)
            break;
        rec[c].has_w = 1;
        const double *sa = node_at(g, a[c])->state;
        if (b[c] >= 0) {
            candidate_jacobian(g, a[c], b[c], rec[c].J);
            asam_xyt_residual(zc, sa, node_at(g, b[c])->state, rec[c].r);
        } else {
            asam_xytpos_residual(zc, sa, rec[c].r);
        }
    }
    if (rc == 0)
        rc = candidates_run(s, k, a, b, rec, d2, cov9, fn);
    free(rec);
    return rc;
}

ASAM_API int aprilsam_b200_relative_covariance(april_graph_t *g, april_graph_cholesky_param_t *param, int a, int b,
                                               double out9[9])
{
    const char *fn = "aprilsam_b200_relative_covariance";
    if (!out9) {
        asam_set_error("%s: NULL out9", fn);
        return -1;
    }
    solver_t *s = marginal_solver(g, param, fn);
    if (!s)
        return -1;
    for (int e = 0; e < 2; e++) {
        const int id = e ? b : a;
        if (id < 0 || id >= s->plan.N) {
            asam_set_error("%s: node %d is not in the solved graph (%d poses)", fn, id, s->plan.N);
            return -1;
        }
    }
    /* one candidate without W: Sigma_rel only */
    asam_marg_pair_t rec;
    memset(&rec, 0, sizeof(rec));
    candidate_jacobian(g, a, b, rec.J);
    double d2;
    return candidates_run(s, 1, &a, &b, &rec, &d2, out9, fn);
}
