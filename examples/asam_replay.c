/* asam_replay.c -- command-line driver of the drop-in library (SURVEY.md section 8f item 1).
 *
 *   asam_replay --datapath FILE [--batch_update_only] [--delta_xy 0.1] [--delta_theta 0.1]
 *               [--nthreshold 100] [--quiet] [--show_timing] [--save OUT.graph]
 *               [--robust huber:K | cauchy:K] [--relin-in-place N]
 *
 * FILE is a Manhattan-style text file (VERTEX2 id x y theta / EDGE2 a b dx dy dth I11 I12 I22 I33
 * I13 I23) or a ".graph" file in the stype framing.  The graph is then replayed pose by pose with
 * the protocol of the reference demo (examples/aprilsam_demo.c:150-234): step k appends pose k and
 * every factor whose larger pose id is k; the first step adds a prior on pose 0 and calls
 * april_graph_cholesky, every later step april_graph_cholesky_inc (or the batch call with
 * --batch_update_only); chi2 and the step time are printed per step.  --robust creates every "scan" factor
 * (a loop closure, |a - b| != 1) as a robust xyt factor with a Huber or Cauchy loss of scale K > 0, so that
 * a wrong closure cannot pull the trajectory towards it.  --relin-in-place N relinearises the poses the tree has
 * flagged (tr->linearized_nodes) in place, as one step, after every step that leaves start_over above N; combine it
 * with a high --nthreshold so that the batch escalation does not come first.
 * Written against include/aprilsam/aprilsam.h only: without --robust and --relin-in-place (aprilsam_b200
 * extensions) it links unchanged against the reference too.
 */
#define _POSIX_C_SOURCE 200809L
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "aprilsam.h"

static double now_ms(void)
{
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6;
}

static int ends_with(const char *s, const char *suffix)
{
    size_t n = strlen(s), m = strlen(suffix);
    return n >= m && !strcmp(s + n - m, suffix);
}

/* text loader: the information matrix is filled the way the demo does (upper triangle only) */
static april_graph_t *load_text(const char *path)
{
    FILE *f = fopen(path, "r");
    if (!f)
        return NULL;
    april_graph_t *g = april_graph_create();
    char tok[64];
    while (fscanf(f, "%63s", tok) == 1) {
        if (!strcmp(tok, "VERTEX2")) {
            int id;
            double p[3];
            if (fscanf(f, "%d %lf %lf %lf", &id, &p[0], &p[1], &p[2]) != 4)
                goto bad;
            april_graph_node_t *n = april_graph_node_xyt_create(p, p, p);
            zarray_add(g->nodes, &n);
        } else if (!strcmp(tok, "EDGE2")) {
            int a, b;
            double z[3], w[6];
            if (fscanf(f, "%d %d %lf %lf %lf %lf %lf %lf %lf %lf %lf", &a, &b, &z[0], &z[1], &z[2], &w[0], &w[1], &w[2],
                       &w[3], &w[4], &w[5]) != 11)
                goto bad;
            matd_t *W = matd_create(3, 3);
            W->data[0] = w[0]; W->data[1] = w[1]; W->data[4] = w[2];
            W->data[8] = w[3]; W->data[2] = w[4]; W->data[5] = w[5];
            april_graph_factor_t *fac = april_graph_factor_xyt_create(a, b, z, NULL, W);
            april_graph_factor_attr_put(fac, stype_get("string"), "type", strdup(abs(a - b) == 1 ? "odom" : "scan"));
            zarray_add(g->factors, &fac);
            matd_destroy(W);
        } else {
            goto bad;
        }
    }
    fclose(f);
    return g;
bad:
    fprintf(stderr, "%s: parse error near '%s'\n", path, tok);
    fclose(f);
    april_graph_destroy(g);
    return NULL;
}

/* "huber:K" or "cauchy:K" with a finite K > 0 -> loss code and K; -1 if malformed */
static int parse_robust(const char *s, int *loss, double *k)
{
    const char *colon = strchr(s, ':');
    if (!colon)
        return -1;
    size_t n = (size_t) (colon - s);
    if (n == 5 && !strncmp(s, "huber", 5))
        *loss = APRILSAM_B200_LOSS_HUBER;
    else if (n == 6 && !strncmp(s, "cauchy", 6))
        *loss = APRILSAM_B200_LOSS_CAUCHY;
    else
        return -1;
    char *end;
    *k = strtod(colon + 1, &end);
    if (end == colon + 1 || *end || !(*k > 0.0) || !isfinite(*k))
        return -1;
    return 0;
}

int main(int argc, char **argv)
{
    const char *path = NULL, *save = NULL;
    int batch_only = 0, quiet = 0, nthreshold = 100, show_timing = 0, robust_loss = 0, relin_in_place = -1;
    double delta_xy = 0.1, delta_theta = 0.1, robust_k = 0.0;
    for (int i = 1; i < argc; i++) {
        if (!strcmp(argv[i], "--robust")) {
            if (i + 1 >= argc || parse_robust(argv[i + 1], &robust_loss, &robust_k)) {
                fprintf(stderr, "%s: --robust expects huber:K or cauchy:K with a finite K > 0\n", argv[0]);
                return 2;
            }
            i++;
            continue;
        }
        if (!strcmp(argv[i], "--datapath") && i + 1 < argc) path = argv[++i];
        else if (!strcmp(argv[i], "--save") && i + 1 < argc) save = argv[++i];
        else if (!strcmp(argv[i], "--batch_update_only")) batch_only = 1;
        else if (!strcmp(argv[i], "--quiet")) quiet = 1;
        else if (!strcmp(argv[i], "--show_timing")) show_timing = 1;
        else if (!strcmp(argv[i], "--delta_xy") && i + 1 < argc) delta_xy = atof(argv[++i]);
        else if (!strcmp(argv[i], "--delta_theta") && i + 1 < argc) delta_theta = atof(argv[++i]);
        else if (!strcmp(argv[i], "--nthreshold") && i + 1 < argc) nthreshold = atoi(argv[++i]);
        else if (!strcmp(argv[i], "--relin-in-place") && i + 1 < argc && atoi(argv[i + 1]) >= 0)
            relin_in_place = atoi(argv[++i]);
        else {
            fprintf(stderr, "usage: %s --datapath FILE [--batch_update_only] [--delta_xy D] [--delta_theta D] "
                            "[--nthreshold N] [--quiet] [--save OUT.graph] [--robust huber:K | cauchy:K] "
                            "[--relin-in-place N]\n", argv[0]);
            return 2;
        }
    }
    if (!path) {
        fprintf(stderr, "%s: --datapath is required\n", argv[0]);
        return 2;
    }
    stype_register_basic_types();
    april_graph_stype_init();
    april_graph_t *all = ends_with(path, ".graph") ? april_graph_create_from_file(path) : load_text(path);
    if (!all) {
        fprintf(stderr, "cannot load %s\n", path);
        return 1;
    }
    const int N = zarray_size(all->nodes), F = zarray_size(all->factors);
    printf("%d nodes, %d factors\n", N, F);
    if (save && !april_graph_save(all, save))
        return 1;

    /* factors by the step that introduces them (larger pose id), file order inside a step */
    int *first = calloc((size_t) N + 2, sizeof(int)), *order = malloc(sizeof(int) * (size_t) (F + 1));
    for (int f = 0; f < F; f++) {
        april_graph_factor_t *fac;
        zarray_get(all->factors, f, &fac);
        int k = fac->nodes[0];
        for (int j = 1; j < fac->nnodes; j++)
            if (fac->nodes[j] > k)
                k = fac->nodes[j];
        first[k + 2]++;
    }
    for (int k = 0; k <= N; k++)
        first[k + 1] += first[k];
    for (int f = 0; f < F; f++) {
        april_graph_factor_t *fac;
        zarray_get(all->factors, f, &fac);
        int k = fac->nodes[0];
        for (int j = 1; j < fac->nnodes; j++)
            if (fac->nodes[j] > k)
                k = fac->nodes[j];
        order[first[k + 1]++] = f;
    }

    april_graph_t *g = april_graph_create();
    april_graph_cholesky_param_t *param = calloc(1, sizeof(*param));
    april_graph_cholesky_param_init(param);
    param->delta_xy = delta_xy;
    param->delta_theta = delta_theta;
    param->nthreshold = nthreshold;
    param->show_timing = show_timing; /* per-phase table after every solve (aprilsam.c:317) */
    double total = 0.0;
    int relins = 0;
    for (int k = 0; k < N; k++) {
        april_graph_node_t *src;
        zarray_get(all->nodes, k, &src);
        april_graph_node_t *n = april_graph_node_xyt_create(src->init ? src->init : src->state, src->init, src->truth);
        n->UID = k;
        zarray_add(g->nodes, &n);
        if (k == 0) { /* anchor the first pose (demo: W = diag(1e4, 1e4, 1e3), z = 0) */
            double z0[3] = { 0, 0, 0 }, w0[9] = { 1e4, 0, 0, 0, 1e4, 0, 0, 0, 1e3 };
            matd_t *W = matd_create_data(3, 3, w0);
            april_graph_factor_t *prior = april_graph_factor_xytpos_create(0, z0, NULL, W);
            zarray_add(g->factors, &prior);
            matd_destroy(W);
        }
        for (int e = first[k]; e < first[k + 1]; e++) {
            april_graph_factor_t *fac;
            zarray_get(all->factors, order[e], &fac);
            const char *type = april_graph_factor_attr_get(fac, "type");
            april_graph_factor_t *c;
            if (robust_loss && fac->type == APRIL_GRAPH_FACTOR_XYT_TYPE && type && !strcmp(type, "scan"))
                c = aprilsam_b200_factor_xyt_robust_create(fac->nodes[0], fac->nodes[1], fac->u.common.z,
                                                           fac->u.common.ztruth, fac->u.common.W, robust_loss, robust_k);
            else
                c = fac->copy(fac);
            if (c->nnodes == 2 && type && !strcmp(type, "odom")) {
                /* dead-reckon the new pose from its neighbour and relinearise it */
                int a = c->nodes[0], b = c->nodes[1];
                april_graph_node_t *na, *nb;
                zarray_get(g->nodes, a, &na);
                zarray_get(g->nodes, b, &nb);
                if (b == k) {
                    doubles_xyt_mul(na->state, c->u.common.z, nb->state);
                    nb->relinearize(nb);
                } else {
                    double inv[3];
                    doubles_xyt_inv(c->u.common.z, inv);
                    doubles_xyt_mul(nb->state, inv, na->state);
                    na->relinearize(na);
                }
            }
            zarray_add(g->factors, &c);
        }
        double t0 = now_ms();
        if (k == 0 || batch_only)
            april_graph_cholesky(g, param);
        else
            april_graph_cholesky_inc(g, param);
        if (relin_in_place >= 0 && k > 0 && !batch_only && param->tr->start_over > relin_in_place &&
            param->tr->nlinearized_nodes > 0) {
            if (aprilsam_b200_relinearize_poses(g, param, param->tr->nlinearized_nodes, param->tr->linearized_nodes)) {
                fprintf(stderr, "step %d: %s\n", k, aprilsam_b200_last_error());
                return 1;
            }
            relins++;
        }
        double dt = now_ms() - t0;
        total += dt;
        if (!quiet)
            printf("step %d: chi2 %.6f, %.3f ms (total %.1f ms)\n", k, april_graph_chi2(g), dt, total);
    }
    printf("final chi2 %.9f after %d steps, solver time %.1f ms\n", april_graph_chi2(g), N, total);
    if (relin_in_place >= 0)
        printf("%d in-place relinearisations\n", relins);
    april_graph_cholesky_param_destory(param);
    april_graph_destroy(g);
    april_graph_destroy(all);
    free(first);
    free(order);
    return 0;
}
