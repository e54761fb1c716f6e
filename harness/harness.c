/* harness.c -- one driver source, two builds.
 *
 * A small C driver written ONLY against the public AprilSAM API (aprilsam.h): it is
 * compiled once against the reference's headers + oracle/_ref/libaprilsam_ref.so
 * (-DHARNESS_REFERENCE, see oracle/Makefile) and once against include/aprilsam/ +
 * libaprilsam_b200.so (see aprilsam_b200/build.py).  Python (ctypes) loads both and
 * runs them in lock-step on identical inputs, so parity tests, bench.py's reference
 * arm and the golden-vector generator all make exactly the calls a user of the
 * reference would make (zarray_add of nodes/factors, april_graph_cholesky{,_inc},
 * april_graph_chi2).
 *
 * The replay mirrors the reference demo's pose-by-pose protocol
 * (/root/reference/examples/aprilsam_demo.c:150-234): step k appends node k at its
 * VERTEX2 init; step 0 adds the xytpos prior W=diag(1e4,1e4,1e3), z=0 (:133-145);
 * every edge whose larger node id is k is appended in file order; an "odom" edge
 * (|a-b|==1, :83-87) first dead-reckons the new node's state from its neighbour and
 * relinearises it (:172-191); then step 0 calls april_graph_cholesky and every later
 * step april_graph_cholesky_inc (or always the batch call with batch_only) (:219-234).
 */
#define _POSIX_C_SOURCE 200809L
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "aprilsam.h"

#define H_EXPORT __attribute__((visibility("default")))

typedef struct hctx {
    april_graph_t *g;
    april_graph_cholesky_param_t *p;
    double last_ms;
    /* replay cursor */
    int next_step;
    /* loss / k of the robust factors h_replay and h_load_full create for "scan" edges (0: plain xyt) */
    int scan_loss;
    double scan_k;
    /* h_replay relinearises the flagged poses in place after a step whose start_over exceeds this (< 0: never) */
    int relin_threshold;
    int relin_calls;   /* those relinearisations so far, and their wall time */
    double relin_ms;
} hctx_t;

static double now_ms(void)
{
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6;
}

H_EXPORT const char *h_impl(void)
{
#ifdef HARNESS_REFERENCE
    return "reference";
#else
    return "b200";
#endif
}

H_EXPORT hctx_t *h_create(double delta_xy, double delta_theta, int nthreshold)
{
    hctx_t *h = calloc(1, sizeof(hctx_t));
    h->g = april_graph_create();
    h->p = calloc(1, sizeof(april_graph_cholesky_param_t));
    april_graph_cholesky_param_init(h->p);
    h->p->show_timing = 0;
    h->p->delta_xy = delta_xy;
    h->p->delta_theta = delta_theta;
    h->p->nthreshold = nthreshold;
    h->relin_threshold = -1;
    return h;
}

H_EXPORT void h_destroy(hctx_t *h)
{
    if (!h)
        return;
    april_graph_cholesky_param_destory(h->p); /* (sic) frees the param too */
    april_graph_destroy(h->g);
    free(h);
}

H_EXPORT void h_set_tikhanov(hctx_t *h, double lambda) { h->p->tikhanov = lambda; }

H_EXPORT int h_nnodes(hctx_t *h) { return zarray_size(h->g->nodes); }
H_EXPORT int h_nfactors(hctx_t *h) { return zarray_size(h->g->factors); }

static april_graph_node_t *node_at(hctx_t *h, int i)
{
    april_graph_node_t *n;
    zarray_get(h->g->nodes, i, &n);
    return n;
}

H_EXPORT int h_add_node(hctx_t *h, const double *xyt)
{
    april_graph_node_t *n = april_graph_node_xyt_create(xyt, xyt, xyt);
    zarray_add(h->g->nodes, &n);
    return zarray_size(h->g->nodes) - 1;
}

H_EXPORT int h_add_xyt(hctx_t *h, int a, int b, const double *z, const double *W9)
{
    matd_t *W = matd_create_data(3, 3, W9);
    april_graph_factor_t *f = april_graph_factor_xyt_create(a, b, z, NULL, W);
    zarray_add(h->g->factors, &f);
    matd_destroy(W);
    return zarray_size(h->g->factors) - 1;
}

/* a robust xyt factor (aprilsam_b200 extension); -1 and no factor in the reference build or for invalid loss / k */
H_EXPORT int h_add_xyt_robust(hctx_t *h, int a, int b, const double *z, const double *W9, int loss, double k)
{
#ifndef HARNESS_REFERENCE
    matd_t *W = matd_create_data(3, 3, W9);
    april_graph_factor_t *f = aprilsam_b200_factor_xyt_robust_create(a, b, z, NULL, W, loss, k);
    matd_destroy(W);
    if (!f)
        return -1;
    zarray_add(h->g->factors, &f);
    return zarray_size(h->g->factors) - 1;
#else
    (void) h, (void) a, (void) b, (void) z, (void) W9, (void) loss, (void) k;
    return -1;
#endif
}

/* aprilsam_b200_factor_set_loss on factor idx: 0 ok, -1 otherwise (always -1 in the reference build) */
H_EXPORT int h_set_loss(hctx_t *h, int idx, int loss, double k)
{
#ifndef HARNESS_REFERENCE
    april_graph_factor_t *f;
    zarray_get(h->g->factors, idx, &f);
    return aprilsam_b200_factor_set_loss(f, loss, k);
#else
    (void) h, (void) idx, (void) loss, (void) k;
    return -1;
#endif
}

/* from now on h_replay / h_load_full create every "scan" edge (|a-b| != 1) as a robust factor with this loss;
 * loss 0 = plain xyt (the default).  No-op in the reference build. */
H_EXPORT void h_set_scan_loss(hctx_t *h, int loss, double k)
{
    h->scan_loss = loss;
    h->scan_k = k;
}

static void add_edge(hctx_t *h, int a, int b, const double *z, const double *W9)
{
#ifndef HARNESS_REFERENCE
    if (h->scan_loss && abs(a - b) != 1) {
        if (h_add_xyt_robust(h, a, b, z, W9, h->scan_loss, h->scan_k) < 0) {
            fprintf(stderr, "harness: %s\n", aprilsam_b200_last_error());
            abort();
        }
        return;
    }
#endif
    h_add_xyt(h, a, b, z, W9);
}

H_EXPORT int h_add_xytpos(hctx_t *h, int a, const double *z, const double *W9)
{
    matd_t *W = matd_create_data(3, 3, W9);
    double zz[3] = { z[0], z[1], z[2] };
    april_graph_factor_t *f = april_graph_factor_xytpos_create(a, zz, NULL, W);
    zarray_add(h->g->factors, &f);
    matd_destroy(W);
    return zarray_size(h->g->factors) - 1;
}

H_EXPORT void h_relinearize(hctx_t *h, int i)
{
    april_graph_node_t *n = node_at(h, i);
    n->relinearize(n);
}

/* which: 0 state, 1 l_point, 2 delta_X, 3 init */
static double *node_vec(april_graph_node_t *n, int which)
{
    switch (which) {
    case 0: return n->state;
    case 1: return n->l_point;
    case 2: return n->delta_X;
    default: return n->init;
    }
}

H_EXPORT void h_get(hctx_t *h, int which, double *out)
{
    int N = zarray_size(h->g->nodes);
    for (int i = 0; i < N; i++)
        memcpy(&out[3 * i], node_vec(node_at(h, i), which), 3 * sizeof(double));
}

H_EXPORT void h_set(hctx_t *h, int which, const double *in)
{
    int N = zarray_size(h->g->nodes);
    for (int i = 0; i < N; i++)
        memcpy(node_vec(node_at(h, i), which), &in[3 * i], 3 * sizeof(double));
}

H_EXPORT double h_chi2(hctx_t *h) { return april_graph_chi2(h->g); }

H_EXPORT double h_batch(hctx_t *h)
{
    double t0 = now_ms();
    april_graph_cholesky(h->g, h->p);
    h->last_ms = now_ms() - t0;
    return h->last_ms;
}

H_EXPORT double h_inc(hctx_t *h)
{
    double t0 = now_ms();
    april_graph_cholesky_inc(h->g, h->p);
    h->last_ms = now_ms() - t0;
    return h->last_ms;
}

/* info[0]=naffected info[1]=start_over info[2]=nlinearized_nodes info[3]=tree nnodes
 * info[4]=root graph-node id info[5]=param->nreordering info[6]=param->factor_num */
H_EXPORT void h_info(hctx_t *h, int *info)
{
    memset(info, 0, 8 * sizeof(int));
    search_tree_t *tr = h->p->tr;
    if (tr) {
        info[0] = tr->naffected;
        info[1] = tr->start_over;
        info[2] = tr->nlinearized_nodes;
        info[3] = tr->nnodes;
        info[4] = tr->root ? (int) (tr->root - tr->nodes) : -1;
    }
    info[5] = h->p->nreordering;
    info[6] = h->p->factor_num;
}

/* tr->linearized_nodes (the poses flagged since the last batch, in flag order); returns how many */
H_EXPORT int h_get_linearized(hctx_t *h, int *out, int cap)
{
    search_tree_t *tr = h->p->tr;
    if (!tr)
        return 0;
    int n = tr->nlinearized_nodes < cap ? tr->nlinearized_nodes : cap;
    memcpy(out, tr->linearized_nodes, (size_t) (n > 0 ? n : 0) * sizeof(int));
    return n;
}

/* elimination ordering of the last batch/inc call: out[pos] = graph node id */
H_EXPORT int h_get_ordering(hctx_t *h, int *out, int cap)
{
    int n = h->p->nreordering;
    if (!h->p->ordering)
        return 0;
    if (n > cap)
        n = cap;
    memcpy(out, h->p->ordering, n * sizeof(int));
    return n;
}

/* parent[i] of every tree node (graph-node ids), -1 for the root */
H_EXPORT int h_get_tree_parents(hctx_t *h, int *out, int cap)
{
    search_tree_t *tr = h->p->tr;
    if (!tr)
        return 0;
    int n = tr->nnodes < cap ? tr->nnodes : cap;
    for (int i = 0; i < n; i++)
        out[i] = tr->nodes[i].parent;
    return n;
}

static void xyt_mul(const double *a, const double *b, double *r)
{
    double s = sin(a[2]), c = cos(a[2]);
    double x = c * b[0] - s * b[1] + a[0];
    double y = s * b[0] + c * b[1] + a[1];
    double t = a[2] + b[2];
    r[0] = x; r[1] = y; r[2] = t;
}

static void xyt_inv(const double *a, double *r)
{
    double s = sin(a[2]), c = cos(a[2]);
    r[0] = -s * a[1] - c * a[0];
    r[1] = -c * a[1] + s * a[0];
    r[2] = -a[2];
}

/* Demo-protocol replay of steps [h->next_step, step_end).
 *  init      3*N   VERTEX2 values
 *  estart    N+1   edges of step k are e in [estart[k], estart[k+1]) (bucketed by max id,
 *                  file order kept inside a bucket)
 *  ea,eb,ez(3E),eW(9E)
 * Per executed step s (index s - first step): chi2_out, ms_out, info_out[8*s..].
 * If states_out != NULL the full state vector after the LAST executed step is stored.
 * Returns the number of steps executed. */
H_EXPORT int h_replay(hctx_t *h, int N, const double *init, const int *estart, const int *ea,
                      const int *eb, const double *ez, const double *eW, int step_end,
                      int batch_only, int want_chi2, double *chi2_out, double *ms_out,
                      int *info_out)
{
    int done = 0;
    if (step_end > N)
        step_end = N;
    for (int k = h->next_step; k < step_end; k++, done++) {
        h_add_node(h, &init[3 * k]);
        if (k == 0) {
            double W[9] = { 10000, 0, 0, 0, 10000, 0, 0, 0, 1000 };
            double z[3] = { 0, 0, 0 };
            h_add_xytpos(h, 0, z, W);
        }
        for (int e = estart[k]; e < estart[k + 1]; e++) {
            int a = ea[e], b = eb[e];
            if (abs(a - b) == 1) { /* "odom": dead-reckon the newer node */
                april_graph_node_t *na = node_at(h, a), *nb = node_at(h, b);
                if (a < b) {
                    xyt_mul(na->state, &ez[3 * e], nb->state);
                    nb->relinearize(nb);
                } else {
                    double iz[3];
                    xyt_inv(&ez[3 * e], iz);
                    xyt_mul(nb->state, iz, na->state);
                    na->relinearize(na);
                }
            }
            add_edge(h, a, b, &ez[3 * e], &eW[9 * e]);
        }
        double ms;
        if (k == 0 || batch_only)
            ms = h_batch(h);
        else
            ms = h_inc(h);
#ifndef HARNESS_REFERENCE
        if (h->relin_threshold >= 0 && k > 0 && !batch_only && h->p->tr && h->p->tr->start_over > h->relin_threshold &&
            h->p->tr->nlinearized_nodes > 0) {
            double t0 = now_ms();
            if (aprilsam_b200_relinearize_poses(h->g, h->p, h->p->tr->nlinearized_nodes, h->p->tr->linearized_nodes)) {
                fprintf(stderr, "harness: %s\n", aprilsam_b200_last_error());
                abort();
            }
            double t = now_ms() - t0;
            h->relin_calls++;
            h->relin_ms += t;
            ms += t;
        }
#endif
        if (ms_out)
            ms_out[done] = ms;
        if (chi2_out)
            chi2_out[done] = want_chi2 ? april_graph_chi2(h->g) : 0.0;
        if (info_out)
            h_info(h, &info_out[8 * done]);
    }
    h->next_step = step_end > h->next_step ? step_end : h->next_step;
    return done;
}

/* Build the whole graph at once (config 1/2/4 protocol): all nodes at init, prior on
 * node 0, all edges in the given order.  No solve. */
H_EXPORT void h_load_full(hctx_t *h, int N, const double *init, int E, const int *ea,
                          const int *eb, const double *ez, const double *eW)
{
    for (int k = 0; k < N; k++)
        h_add_node(h, &init[3 * k]);
    double W[9] = { 10000, 0, 0, 0, 10000, 0, 0, 0, 1000 };
    double z[3] = { 0, 0, 0 };
    h_add_xytpos(h, 0, z, W);
    for (int e = 0; e < E; e++)
        add_edge(h, ea[e], eb[e], &ez[3 * e], &eW[9 * e]);
    h->next_step = N;
}

/* ---- files + attributes (aprilsam.h:185, :288-299): examples/aprilsam_graph_save_*.c in miniature ---- */
static void serial_init(void)
{
    static int done = 0;
    if (!done) {
        stype_register_basic_types();
        april_graph_stype_init();
        done = 1;
    }
}

H_EXPORT int h_save(hctx_t *h, const char *path)
{
    serial_init();
    return april_graph_save(h->g, path);
}

/* replaces the graph (the solver state starts over); returns the node count or -1 */
H_EXPORT int h_load(hctx_t *h, const char *path)
{
    serial_init();
    april_graph_t *g = april_graph_create_from_file(path);
    if (!g)
        return -1;
    april_graph_cholesky_param_destory(h->p);
    h->p = calloc(1, sizeof(april_graph_cholesky_param_t));
    april_graph_cholesky_param_init(h->p);
    april_graph_destroy(h->g);
    h->g = g;
    h->next_step = zarray_size(g->nodes);
    return zarray_size(g->nodes);
}

/* which: 0 graph, 1 node idx, 2 factor idx; string-valued attribute (stype "string") */
H_EXPORT void h_attr_put_string(hctx_t *h, int which, int idx, const char *key, const char *value)
{
    serial_init();
    stype_t *st = stype_get("string");
    if (which == 0) {
        april_graph_attr_put(h->g, st, key, strdup(value));
    } else if (which == 1) {
        april_graph_node_t *n;
        zarray_get(h->g->nodes, idx, &n);
        april_graph_node_attr_put(n, st, key, strdup(value));
    } else {
        april_graph_factor_t *f;
        zarray_get(h->g->factors, idx, &f);
        april_graph_factor_attr_put(f, st, key, strdup(value));
    }
}

H_EXPORT void h_attr_put_u64(hctx_t *h, int which, int idx, const char *key, uint64_t value)
{
    serial_init();
    stype_t *st = stype_get("uint64");
    uint64_t *v = malloc(sizeof(uint64_t));
    *v = value;
    if (which == 0) {
        april_graph_attr_put(h->g, st, key, v);
    } else if (which == 1) {
        april_graph_node_t *n;
        zarray_get(h->g->nodes, idx, &n);
        april_graph_node_attr_put(n, st, key, v);
    } else {
        april_graph_factor_t *f;
        zarray_get(h->g->factors, idx, &f);
        april_graph_factor_attr_put(f, st, key, v);
    }
}

/* returns the attribute's raw pointer (char* for "string", uint64_t* for "uint64") or NULL */
H_EXPORT const void *h_attr_get(hctx_t *h, int which, int idx, const char *key)
{
    if (which == 0)
        return april_graph_attr_get(h->g, key);
    if (which == 1) {
        april_graph_node_t *n;
        zarray_get(h->g->nodes, idx, &n);
        return april_graph_node_attr_get(n, key);
    }
    april_graph_factor_t *f;
    zarray_get(h->g->factors, idx, &f);
    return april_graph_factor_attr_get(f, key);
}

/* factor record for comparisons: out[0..1] node ids (-1 if unary), out[2..4] z, out[5..13] W; returns type */
H_EXPORT int h_factor(hctx_t *h, int idx, double *out)
{
    april_graph_factor_t *f;
    zarray_get(h->g->factors, idx, &f);
    out[0] = f->nodes[0];
    out[1] = f->nnodes > 1 ? f->nodes[1] : -1;
    memcpy(out + 2, f->u.common.z, 3 * sizeof(double));
    memcpy(out + 5, f->u.common.W->data, 9 * sizeof(double));
    return f->type;
}

/* the factor's host hook: which 0 = eval (at l_point), 1 = state_eval (at state).  out = r[3] | J_0[9] | J_1[9] |
 * W[9] | chi2 (J_1 zero for unary factors); returns the residual length, -1 if the hook is not set */
H_EXPORT int h_eval(hctx_t *h, int idx, int which, double *out)
{
    april_graph_factor_t *f;
    zarray_get(h->g->factors, idx, &f);
    april_graph_factor_eval_t *(*fn)(april_graph_factor_t *, april_graph_t *, april_graph_factor_eval_t *) =
        which ? f->state_eval : f->eval;
    if (!fn)
        return -1;
    april_graph_factor_eval_t *ev = fn(f, h->g, NULL);
    memset(out, 0, 31 * sizeof(double));
    memcpy(out, ev->r, 3 * sizeof(double));
    for (int j = 0; j < 2 && ev->jacobians[j]; j++)
        memcpy(out + 3 + 9 * j, ev->jacobians[j]->data, 9 * sizeof(double));
    memcpy(out + 21, ev->W->data, 9 * sizeof(double));
    out[30] = ev->chi2;
    int len = ev->length;
    april_graph_factor_eval_destroy(ev);
    return len;
}

/* append factor->copy(factor) of factor idx; returns the new index */
H_EXPORT int h_copy_factor(hctx_t *h, int idx)
{
    april_graph_factor_t *f;
    zarray_get(h->g->factors, idx, &f);
    april_graph_factor_t *c = f->copy(f);
    zarray_add(h->g->factors, &c);
    return zarray_size(h->g->factors) - 1;
}

H_EXPORT int h_dof(hctx_t *h) { return april_graph_dof(h->g); }

/* overwrite measurement and information matrix of factor idx IN PLACE (what a robust-kernel or
 * re-weighting loop around the reference does between batch calls) */
H_EXPORT void h_set_factor(hctx_t *h, int idx, const double *z, const double *W9)
{
    april_graph_factor_t *f;
    zarray_get(h->g->factors, idx, &f);
    memcpy(f->u.common.z, z, 3 * sizeof(double));
    memcpy(f->u.common.W->data, W9, 9 * sizeof(double));
}

/* replace factor idx by a new xyt factor between a and b (same count, other structure) */
H_EXPORT void h_replace_xyt(hctx_t *h, int idx, int a, int b, const double *z, const double *W9)
{
    april_graph_factor_t *old;
    zarray_get(h->g->factors, idx, &old);
    matd_t *W = matd_create_data(3, 3, W9);
    april_graph_factor_t *f = april_graph_factor_xyt_create(a, b, z, NULL, W);
    matd_destroy(W);
    zarray_set(h->g->factors, idx, &f, NULL);
    old->destroy(old);
}

/* aprilsam_b200 extensions (no-ops in the reference build) */
H_EXPORT void h_invalidate_plan(hctx_t *h)
{
#ifndef HARNESS_REFERENCE
    aprilsam_b200_invalidate_plan(h->p);
#else
    (void) h;
#endif
}

/* ratio > 0: deterministic escalation policy step_work > ratio * batch_work; <= 0: none */
H_EXPORT void h_set_policy_ratio(hctx_t *h, double ratio)
{
#ifndef HARNESS_REFERENCE
    static double ratios[64];
    static int next = 0;
    if (ratio > 0) {
        double *r = &ratios[next++ % 64];
        *r = ratio;
        aprilsam_b200_set_escalation_policy(h->p, aprilsam_b200_policy_work_ratio, r);
    } else {
        aprilsam_b200_set_escalation_policy(h->p, NULL, NULL);
    }
#else
    (void) h;
    (void) ratio;
#endif
}

/* aprilsam_b200_marginal_covariance / _relative_covariance / _candidate_mahalanobis (extensions; absent from the
 * reference build) */
#ifndef HARNESS_REFERENCE
H_EXPORT int h_marginal_cov(hctx_t *h, int n, const int *nodes, double *out)
{
    return aprilsam_b200_marginal_covariance(h->g, h->p, n, nodes, out);
}

H_EXPORT int h_relative_cov(hctx_t *h, int a, int b, double *out9)
{
    return aprilsam_b200_relative_covariance(h->g, h->p, a, b, out9);
}

H_EXPORT int h_candidate_mahalanobis(hctx_t *h, int k, const int *a, const int *b, const double *z, const double *W,
                                     double *d2, double *cov9)
{
    return aprilsam_b200_candidate_mahalanobis(h->g, h->p, k, a, b, z, W, d2, cov9);
}

/* aprilsam_b200_candidate_compatibility (d2: k x k; cross9: k x k x 9 or NULL) */
H_EXPORT int h_candidate_compatibility(hctx_t *h, int k, const int *a, const int *b, const double *z, const double *W,
                                       double *d2, double *cross9)
{
    return aprilsam_b200_candidate_compatibility(h->g, h->p, k, a, b, z, W, d2, cross9);
}

/* aprilsam_b200_factor_residuals (out: 6 doubles per factor) / _factor_outlier_scores */
H_EXPORT int h_factor_residuals(hctx_t *h, int first, int count, double *out)
{
    return aprilsam_b200_factor_residuals(h->g, first, count, (aprilsam_b200_factor_residual_t *) out);
}

H_EXPORT int h_factor_outlier_scores(hctx_t *h, int k, const int *idx, double *d2, double *redundancy, double *cov9)
{
    return aprilsam_b200_factor_outlier_scores(h->g, h->p, k, idx, d2, redundancy, cov9);
}

/* aprilsam_b200_remove_factors; keep = 1 hands the removed factors back and destroys them here (exercises both
 * ownership paths) */
H_EXPORT int h_remove_factors(hctx_t *h, int n, const int *idx, int keep)
{
    if (!keep)
        return aprilsam_b200_remove_factors(h->g, h->p, n, idx, NULL);
    april_graph_factor_t **out = calloc((size_t) (n > 0 ? n : 1), sizeof(*out));
    int rc = aprilsam_b200_remove_factors(h->g, h->p, n, idx, out);
    for (int k = 0; rc == 0 && k < n; k++)
        out[k]->destroy(out[k]);
    free(out);
    return rc;
}

/* aprilsam_b200_relinearize_poses; ids == NULL relinearises the poses the tree has flagged, passing
 * p->tr->linearized_nodes itself (the aliasing case) */
H_EXPORT int h_relinearize_poses(hctx_t *h, int n, const int *ids)
{
    if (!ids) {
        if (!h->p->tr)
            return aprilsam_b200_relinearize_poses(h->g, h->p, 0, NULL);
        return aprilsam_b200_relinearize_poses(h->g, h->p, h->p->tr->nlinearized_nodes, h->p->tr->linearized_nodes);
    }
    return aprilsam_b200_relinearize_poses(h->g, h->p, n, ids);
}

/* threshold >= 0: h_replay relinearises the flagged poses in place after every step that leaves start_over above it
 * (its time counts in the step's ms); < 0 (the default): never */
H_EXPORT void h_set_relin_in_place(hctx_t *h, int threshold) { h->relin_threshold = threshold; }

/* out[0] = relinearisations h_replay made, out[1] = their wall ms */
H_EXPORT void h_relin_stats(hctx_t *h, double *out)
{
    out[0] = h->relin_calls;
    out[1] = h->relin_ms;
}

/* further params on the same graph, for the tests of several solvers of one graph: h_swap_param makes one the
 * harness's param (every h_* call then goes through it) and returns the one it replaces */
H_EXPORT void *h_param_create(hctx_t *h)
{
    april_graph_cholesky_param_t *p = calloc(1, sizeof(*p));
    april_graph_cholesky_param_init(p);
    p->delta_xy = h->p->delta_xy;
    p->delta_theta = h->p->delta_theta;
    p->nthreshold = h->p->nthreshold;
    p->tikhanov = h->p->tikhanov;
    return p;
}

H_EXPORT void h_param_destroy(void *p) { april_graph_cholesky_param_destory(p); }

H_EXPORT void *h_swap_param(hctx_t *h, void *p)
{
    void *old = h->p;
    h->p = p;
    return old;
}
#endif

/* april_graph_cholesky_inc_solver (aprilsam.h:276): the reference never reads idxs (aprilsam.c:578-597) */
H_EXPORT void h_inc_solver(hctx_t *h) { april_graph_cholesky_inc_solver(h->g, h->p, NULL); }

H_EXPORT void h_set_show_timing(hctx_t *h, int on) { h->p->show_timing = on; }

H_EXPORT void *h_graph(hctx_t *h) { return h->g; }
H_EXPORT void *h_param(hctx_t *h) { return h->p; }
