/* graph.c -- graph / node / factor objects of the public API (host C).
 *
 * Mirrors the reference's object model so callers populate the graph exactly as before
 * (reference: aprilsam/april_graph.c:326-364, april_graph_xyt.c:271-295,420-438,
 * april_graph_xytpos.c:186-217).  Attributes, stype serialisation and file I/O are out of
 * scope this round (SURVEY.md section 8f); `attr` and `stype` stay NULL.
 *
 * The per-factor `eval` / `state_eval` and per-node `update` / `relinearize` function
 * pointers are provided because they are part of the public structs and callers use them
 * (the demo calls node->relinearize and factor->copy).  The SOLVER never calls eval /
 * state_eval / update: april_graph_cholesky{,_inc}() and april_graph_chi2() dispatch on the
 * type tags and do that arithmetic in the CUDA kernels.
 */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "aprilsam.h"
#include "asam_host.h"

/* ---- matd (common/matd.h) ------------------------------------------------------------ */
ASAM_API matd_t *matd_create(int rows, int cols)
{
    matd_t *m = calloc(1, sizeof(matd_t) + sizeof(double) * (size_t) rows * cols);
    m->nrows = rows;
    m->ncols = cols;
    return m;
}

ASAM_API matd_t *matd_create_data(int rows, int cols, const double *data)
{
    matd_t *m = matd_create(rows, cols);
    memcpy(m->data, data, sizeof(double) * (size_t) rows * cols);
    return m;
}

ASAM_API matd_t *matd_identity(int dim)
{
    matd_t *m = matd_create(dim, dim);
    for (int i = 0; i < dim; i++)
        MATD_EL(m, i, i) = 1.0;
    return m;
}

ASAM_API matd_t *matd_copy(const matd_t *m)
{
    return matd_create_data(m->nrows, m->ncols, m->data);
}

ASAM_API void matd_destroy(matd_t *m) { free(m); }

ASAM_API void APRILSAM_VERSION(void)
{
    printf("=========================\n");
    printf("| APRILSAM-B200 (sm_90a)  |\n");
    printf("=========================\n\n");
}

/* ---- graph --------------------------------------------------------------------------- */
ASAM_API april_graph_t *april_graph_create(void)
{
    april_graph_t *g = calloc(1, sizeof(april_graph_t));
    g->nodes = zarray_create(sizeof(april_graph_node_t *));
    g->factors = zarray_create(sizeof(april_graph_factor_t *));
    g->stype = &stype_april_graph; /* april_graph.c:334 */
    return g;
}

ASAM_API void april_graph_destroy(april_graph_t *g)
{
    if (!g)
        return;
    asam_graph_forget(g); /* drop the device mirror used by april_graph_chi2 */
    for (int i = 0; i < zarray_size(g->nodes); i++) {
        april_graph_node_t *n;
        zarray_get(g->nodes, i, &n);
        if (n && n->destroy)
            n->destroy(n);
    }
    for (int i = 0; i < zarray_size(g->factors); i++) {
        april_graph_factor_t *f;
        zarray_get(g->factors, i, &f);
        if (f && f->destroy)
            f->destroy(f);
    }
    zarray_destroy(g->nodes);
    zarray_destroy(g->factors);
    april_graph_attr_destroy(g->attr);
    free(g);
}

ASAM_API int april_graph_dof(april_graph_t *g)
{
    /* reference: april_graph.c:60-77 */
    int fdof = 0, sdof = 0;
    for (int i = 0; i < zarray_size(g->factors); i++) {
        april_graph_factor_t *f;
        zarray_get(g->factors, i, &f);
        fdof += f->length;
    }
    for (int i = 0; i < zarray_size(g->nodes); i++) {
        april_graph_node_t *n;
        zarray_get(g->nodes, i, &n);
        sdof += n->length;
    }
    return fdof - sdof;
}

ASAM_API void april_graph_factor_eval_destroy(april_graph_factor_eval_t *ev)
{
    if (!ev)
        return;
    if (ev->jacobians) {
        for (int i = 0; ev->jacobians[i]; i++)
            matd_destroy(ev->jacobians[i]);
        free(ev->jacobians);
    }
    free(ev->r);
    matd_destroy(ev->W);
    free(ev);
}

/* ---- xyt node ------------------------------------------------------------------------ */
static void node_xyt_update(april_graph_node_t *n, double *d)
{
    /* april_graph_xyt.c:302-314: skip on NaN, state = l_point + d, wrap theta */
    if (isnan(d[0]) || isnan(d[1]) || isnan(d[2]))
        return;
    for (int i = 0; i < 3; i++) {
        n->state[i] = n->l_point[i] + d[i];
        n->delta_X[i] = d[i];
    }
    n->state[2] = mod2pi(n->state[2]);
}

static void node_xyt_relinearize(april_graph_node_t *n) { memcpy(n->l_point, n->state, 3 * sizeof(double)); }

static void node_xyt_destroy(april_graph_node_t *n)
{
    free(n->state);
    free(n->init);
    free(n->truth);
    free(n->l_point);
    free(n->delta_X);
    april_graph_attr_destroy(n->attr);
    free(n);
}

static april_graph_node_t *node_xyt_copy(april_graph_node_t *n)
{
    april_graph_node_t *c = april_graph_node_xyt_create(n->state, n->init, n->truth);
    memcpy(c->l_point, n->l_point, 3 * sizeof(double));
    memcpy(c->delta_X, n->delta_X, 3 * sizeof(double));
    c->UID = n->UID;
    c->attr = asam_attr_dup(n->attr);
    return c;
}

static const double zero3[3] = { 0, 0, 0 };

ASAM_API april_graph_node_t *april_graph_node_xyt_create(const double *state, const double *init, const double *truth)
{
    april_graph_node_t *n = calloc(1, sizeof(april_graph_node_t));
    n->type = APRIL_GRAPH_NODE_XYT_TYPE;
    n->length = 3;
    n->state = doubles_dup(state, 3);
    n->init = doubles_dup(init, 3);   /* NULL stays NULL (april_graph_xyt.c:421-423) */
    n->truth = doubles_dup(truth, 3);
    n->l_point = doubles_dup(state, 3);
    n->delta_X = doubles_dup(zero3, 3);
    n->update = node_xyt_update;
    n->relinearize = node_xyt_relinearize;
    n->copy = node_xyt_copy;
    n->destroy = node_xyt_destroy;
    n->stype = &stype_april_node_xyt;
    return n;
}

/* ---- factors: host-side plug-in hooks ------------------------------------------------- */
static april_graph_factor_eval_t *eval_alloc(int nj)
{
    april_graph_factor_eval_t *ev = calloc(1, sizeof(*ev));
    ev->jacobians = calloc(nj + 1, sizeof(matd_t *));
    for (int i = 0; i < nj; i++)
        ev->jacobians[i] = matd_create(3, 3);
    ev->r = calloc(3, sizeof(double));
    ev->W = matd_create(3, 3);
    ev->length = 3;
    return ev;
}

static void eval_finish(april_graph_factor_eval_t *ev, const matd_t *W)
{
    memcpy(ev->W->data, W->data, 9 * sizeof(double));
    double X[3];
    for (int i = 0; i < 3; i++)
        X[i] = MATD_EL(W, i, 0) * ev->r[0] + MATD_EL(W, i, 1) * ev->r[1] + MATD_EL(W, i, 2) * ev->r[2];
    ev->chi2 = ev->r[0] * X[0] + ev->r[1] * X[1] + ev->r[2] * X[2];
}

void asam_xyt_jacobians(const double *pa, const double *pb, double *Ja, double *Jb)
{
    double ca = cos(pa[2]), sa = sin(pa[2]);
    double dx = pb[0] - pa[0], dy = pb[1] - pa[1];
    const double a[9] = { -ca, -sa, -sa * dx + ca * dy, sa, -ca, -ca * dx - sa * dy, 0, 0, -1 };
    const double b[9] = { ca, sa, 0, -sa, ca, 0, 0, 0, 1 };
    memcpy(Ja, a, sizeof(a));
    memcpy(Jb, b, sizeof(b));
}

void asam_xyt_residual(const double *z, const double *pa, const double *pb, double *r)
{
    double ca = cos(pa[2]), sa = sin(pa[2]);
    double dx = pb[0] - pa[0], dy = pb[1] - pa[1];
    r[0] = z[0] - (ca * dx + sa * dy);
    r[1] = z[1] - (-sa * dx + ca * dy);
    r[2] = mod2pi(z[2] - (pb[2] - pa[2]));
}

void asam_xytpos_residual(const double *z, const double *pa, double *r)
{
    r[0] = z[0] - pa[0];
    r[1] = z[1] - pa[1];
    r[2] = mod2pi(z[2] - pa[2]);
}

static april_graph_factor_eval_t *xyt_eval_at(april_graph_factor_t *f, const double *pa, const double *pb,
                                              april_graph_factor_eval_t *ev)
{
    if (!ev)
        ev = eval_alloc(2);
    asam_xyt_jacobians(pa, pb, ev->jacobians[0]->data, ev->jacobians[1]->data);
    asam_xyt_residual(f->u.common.z, pa, pb, ev->r);
    eval_finish(ev, f->u.common.W);
    return ev;
}

static april_graph_factor_eval_t *xyt_eval(april_graph_factor_t *f, april_graph_t *g, april_graph_factor_eval_t *ev)
{
    april_graph_node_t *na, *nb;
    zarray_get(g->nodes, f->nodes[0], &na);
    zarray_get(g->nodes, f->nodes[1], &nb);
    return xyt_eval_at(f, na->l_point, nb->l_point, ev);
}

static april_graph_factor_eval_t *xyt_state_eval(april_graph_factor_t *f, april_graph_t *g,
                                                 april_graph_factor_eval_t *ev)
{
    april_graph_node_t *na, *nb;
    zarray_get(g->nodes, f->nodes[0], &na);
    zarray_get(g->nodes, f->nodes[1], &nb);
    return xyt_eval_at(f, na->state, nb->state, ev);
}

static void factor_common_destroy(april_graph_factor_t *f)
{
    free(f->nodes);
    free(f->u.common.z);
    free(f->u.common.ztruth);
    matd_destroy(f->u.common.W);
    april_graph_attr_destroy(f->attr);
    free(f);
}

static april_graph_factor_t *xyt_copy(april_graph_factor_t *f)
{
    april_graph_factor_t *c =
        april_graph_factor_xyt_create(f->nodes[0], f->nodes[1], f->u.common.z, f->u.common.ztruth, f->u.common.W);
    c->attr = asam_attr_dup(f->attr);
    return c;
}

ASAM_API april_graph_factor_t *april_graph_factor_xyt_create(int a, int b, const double *z, const double *ztruth,
                                                            const matd_t *W)
{
    april_graph_factor_t *f = calloc(1, sizeof(*f));
    f->type = APRIL_GRAPH_FACTOR_XYT_TYPE;
    f->nnodes = 2;
    f->nodes = calloc(2, sizeof(int));
    f->nodes[0] = a;
    f->nodes[1] = b;
    f->length = 3;
    f->copy = xyt_copy;
    f->eval = xyt_eval;
    f->state_eval = xyt_state_eval;
    f->destroy = factor_common_destroy;
    f->u.common.z = doubles_dup(z, 3);
    f->u.common.ztruth = ztruth ? doubles_dup(ztruth, 3) : NULL;
    f->u.common.W = matd_copy(W);
    f->stype = &stype_april_factor_xyt;
    return f;
}

/* ---- robust xyt factor (extension, aprilsam.h): xyt + a loss the factor owns behind u.common.impl ---- */
typedef struct {
    int loss;
    double k;
} robust_loss_t;

static int loss_valid(int loss, double k)
{
    if (loss != APRILSAM_B200_LOSS_HUBER && loss != APRILSAM_B200_LOSS_CAUCHY) {
        asam_set_error("robust loss %d: expected %d (Huber) or %d (Cauchy)", loss, APRILSAM_B200_LOSS_HUBER,
                       APRILSAM_B200_LOSS_CAUCHY);
        return 0;
    }
    if (!(k > 0.0) || !isfinite(k)) {
        asam_set_error("robust loss scale k = %g: must be finite and > 0", k);
        return 0;
    }
    return 1;
}

void asam_factor_loss(const april_graph_factor_t *f, int32_t *loss, double *k)
{
    const robust_loss_t *r = f->type == APRIL_GRAPH_FACTOR_XYT_ROBUST_TYPE ? f->u.common.impl : NULL;
    *loss = r ? r->loss : 0;
    *k = r ? r->k : 0.0;
}

/* xyt evaluation -> W_eff = w W and chi2 = rho(s), s = r'Wr as eval_finish left it in chi2 (the same
 * arithmetic as k_linearize / k_chi2_partial) */
static april_graph_factor_eval_t *robust_weigh(const april_graph_factor_t *f, april_graph_factor_eval_t *ev)
{
    const robust_loss_t *r = f->u.common.impl;
    const double s = ev->chi2, k2 = r->k * r->k;
    double w, rho;
    if (r->loss == APRILSAM_B200_LOSS_HUBER) {
        w = s <= k2 ? 1.0 : r->k / sqrt(s);
        rho = s <= k2 ? s : 2.0 * r->k * sqrt(s) - k2;
    } else {
        w = 1.0 / (1.0 + s / k2);
        rho = k2 * log1p(s / k2);
    }
    for (int i = 0; i < 9; i++)
        ev->W->data[i] *= w;
    ev->chi2 = rho;
    return ev;
}

static april_graph_factor_eval_t *robust_eval(april_graph_factor_t *f, april_graph_t *g, april_graph_factor_eval_t *ev)
{
    return robust_weigh(f, xyt_eval(f, g, ev));
}

static april_graph_factor_eval_t *robust_state_eval(april_graph_factor_t *f, april_graph_t *g,
                                                    april_graph_factor_eval_t *ev)
{
    return robust_weigh(f, xyt_state_eval(f, g, ev));
}

static void robust_destroy(april_graph_factor_t *f)
{
    free(f->u.common.impl);
    factor_common_destroy(f);
}

static april_graph_factor_t *robust_copy(april_graph_factor_t *f)
{
    const robust_loss_t *r = f->u.common.impl;
    april_graph_factor_t *c = aprilsam_b200_factor_xyt_robust_create(f->nodes[0], f->nodes[1], f->u.common.z,
                                                                     f->u.common.ztruth, f->u.common.W, r->loss, r->k);
    c->attr = asam_attr_dup(f->attr);
    return c;
}

ASAM_API april_graph_factor_t *aprilsam_b200_factor_xyt_robust_create(int a, int b, const double *z,
                                                                     const double *ztruth, const matd_t *W, int loss,
                                                                     double k)
{
    if (!loss_valid(loss, k))
        return NULL;
    april_graph_factor_t *f = april_graph_factor_xyt_create(a, b, z, ztruth, W);
    robust_loss_t *r = malloc(sizeof(*r));
    r->loss = loss;
    r->k = k;
    f->type = APRIL_GRAPH_FACTOR_XYT_ROBUST_TYPE;
    f->u.common.impl = r;
    f->copy = robust_copy;
    f->eval = robust_eval;
    f->state_eval = robust_state_eval;
    f->destroy = robust_destroy;
    f->stype = &stype_april_factor_xyt_robust;
    return f;
}

ASAM_API int aprilsam_b200_factor_set_loss(april_graph_factor_t *f, int loss, double k)
{
    if (!f || f->type != APRIL_GRAPH_FACTOR_XYT_ROBUST_TYPE || !f->u.common.impl) {
        asam_set_error("aprilsam_b200_factor_set_loss: factor of type %d has no robust loss", f ? f->type : -1);
        return -1;
    }
    if (!loss_valid(loss, k))
        return -1;
    robust_loss_t *r = f->u.common.impl;
    r->loss = loss;
    r->k = k;
    return 0;
}

static april_graph_factor_eval_t *xytpos_eval(april_graph_factor_t *f, april_graph_t *g, april_graph_factor_eval_t *ev)
{
    if (!ev)
        ev = eval_alloc(1);
    for (int i = 0; i < 3; i++)
        MATD_EL(ev->jacobians[0], i, i) = 1.0;
    april_graph_node_t *na;
    zarray_get(g->nodes, f->nodes[0], &na);
    asam_xytpos_residual(f->u.common.z, na->state, ev->r);
    eval_finish(ev, f->u.common.W);
    return ev;
}

static april_graph_factor_t *xytpos_copy(april_graph_factor_t *f)
{
    april_graph_factor_t *c = april_graph_factor_xytpos_create(f->nodes[0], f->u.common.z, f->u.common.ztruth, f->u.common.W);
    c->attr = asam_attr_dup(f->attr);
    return c;
}

ASAM_API april_graph_factor_t *april_graph_factor_xytpos_create(int a, double *z, double *ztruth, matd_t *W)
{
    april_graph_factor_t *f = calloc(1, sizeof(*f));
    f->type = APRIL_GRAPH_FACTOR_XYTPOS_TYPE;
    f->nnodes = 1;
    f->nodes = calloc(1, sizeof(int));
    f->nodes[0] = a;
    f->length = 3;
    f->copy = xytpos_copy;
    f->eval = xytpos_eval;
    f->state_eval = NULL; /* reference leaves it unset too */
    f->destroy = factor_common_destroy;
    f->u.common.z = doubles_dup(z, 3);
    f->u.common.ztruth = ztruth ? doubles_dup(ztruth, 3) : NULL;
    f->u.common.W = matd_copy(W);
    f->stype = &stype_april_factor_xytpos;
    return f;
}
