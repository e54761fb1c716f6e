/* debug.c -- test-only exports of the host symbolic layer (no GPU needed).
 *
 * tests/ (-m "not gpu") build plans through these entry points and replay them with a
 * numpy emulation of the kernels to check row structures, relative indices, gather lists
 * and the task schedule without a device.  Nothing here is on the solve path.
 */
#include <stdlib.h>
#include <string.h>

#include "asam_host.h"

ASAM_API void *asam_dbg_plan_create(void) { return calloc(1, sizeof(plan_t)); }

ASAM_API void asam_dbg_plan_destroy(void *p)
{
    if (!p)
        return;
    plan_free((plan_t *) p);
    free(p);
}

/* plan_marginal_paths on a plan: per node 6 ints {sn0, j0, hop0, nhop, zoff (int64)}; totals[0] = doubles of
 * scratch, totals[1] = hops */
ASAM_API int asam_dbg_plan_marginal_paths(void *p, int n, const int *nodes, asam_marg_path_t *out, int64_t *totals)
{
    int hops = 0;
    int rc = plan_marginal_paths((const plan_t *) p, n, nodes, out, &totals[0], &hops);
    totals[1] = hops;
    return rc;
}

/* plan_candidate_batches on a plan: returns the number of batches; batch_end / pose_end need k ints, poses 2k */
ASAM_API int asam_dbg_plan_candidate_batches(void *p, int k, const int *a, const int *b, int64_t budget_doubles,
                                             int *batch_end, int *poses, int *pose_end, int *ia, int *ib)
{
    int nb = 0;
    plan_candidate_batches((const plan_t *) p, k, a, b, budget_doubles, batch_end, &nb, poses, pose_end, ia, ib);
    return nb;
}

/* the residual helpers of graph.c: an xyt factor at (pa, pb), an xytpos factor at pa (pb NULL) */
ASAM_API void asam_dbg_residual(const double *z, const double *pa, const double *pb, double *r)
{
    if (pb)
        asam_xyt_residual(z, pa, pb, r);
    else
        asam_xytpos_residual(z, pa, r);
}

/* z scratch per batch of aprilsam_b200_candidate_mahalanobis in bytes; <= 0 restores the default */
ASAM_API void asam_dbg_set_candidate_budget(int64_t bytes)
{
    asam_candidate_budget = bytes > 0 ? bytes : ASAM_CANDIDATE_BUDGET;
}

ASAM_API int asam_dbg_plan_build(void *p, int N, int F, const int *ftype, const int *fa, const int *fb)
{
    return plan_build((plan_t *) p, NULL, N, F, ftype, fa, fb);
}

/* type of factor idx of g, and its loss code / k ((0, 0) without a robust loss) */
ASAM_API int asam_dbg_factor_loss(april_graph_t *g, int idx, int *loss, double *k)
{
    april_graph_factor_t *f;
    zarray_get(g->factors, idx, &f);
    int32_t l;
    asam_factor_loss(f, &l, k);
    *loss = l;
    return f->type;
}

/* multi-GPU schedule of rank `rank` of `world` (no device, no communicator needed) */
ASAM_API int asam_dbg_plan_build_sharded(void *p, int world, int rank, int N, int F, const int *ftype, const int *fa,
                                         const int *fb)
{
    plan_t *pl = (plan_t *) p;
    pl->world = world;
    pl->rank = rank;
    return plan_build(pl, NULL, N, F, ftype, fa, fb);
}

ASAM_API int asam_dbg_plan_build_with_order(void *p, int N, int F, const int *ftype, const int *fa, const int *fb,
                                            const int *order_keep, int N_keep)
{
    return plan_build_with_order((plan_t *) p, NULL, N, F, ftype, fa, fb, order_keep, N_keep);
}

/* returns ntasks (>= 0) or -rc */
ASAM_API int asam_dbg_plan_append(void *p, int N, int F, const int *ftype, const int *fa, const int *fb,
                                  const int *marked, int n_marked, int *tasks_out, int *nwait_out, int *keep_out, int cap)
{
    int *tasks = NULL, *nwait = NULL, *keep = NULL, nt = 0;
    int rc = plan_append((plan_t *) p, NULL, N, F, ftype, fa, fb, marked, n_marked, &tasks, &nwait, &keep, &nt);
    if (rc)
        return -rc;
    if (nt > cap)
        nt = cap;
    memcpy(tasks_out, tasks, sizeof(int) * (size_t) nt);
    memcpy(nwait_out, nwait, sizeof(int) * (size_t) nt);
    if (keep_out)
        memcpy(keep_out, keep, sizeof(int) * (size_t) nt);
    free(tasks);
    free(nwait);
    free(keep);
    return nt;
}

/* plan_refactor on a plan: returns ntasks (<= cap entries copied) */
ASAM_API int asam_dbg_plan_refactor(void *p, const int *marked, int n_marked, int *tasks_out, int *nwait_out,
                                    int *keep_out, int cap)
{
    int *tasks = NULL, *nwait = NULL, *keep = NULL, nt = 0;
    plan_refactor((plan_t *) p, marked, n_marked, &tasks, &nwait, &keep, &nt);
    int k = nt < cap ? nt : cap;
    memcpy(tasks_out, tasks, sizeof(int) * (size_t) k);
    memcpy(nwait_out, nwait, sizeof(int) * (size_t) k);
    memcpy(keep_out, keep, sizeof(int) * (size_t) k);
    free(tasks);
    free(nwait);
    free(keep);
    return nt;
}

/* plan_remove_factors on a plan (no device): 0, or -1 with the error text */
ASAM_API int asam_dbg_plan_remove_factors(void *p, int n, const int *sorted_idx)
{
    return plan_remove_factors((plan_t *) p, NULL, n, sorted_idx) ? -1 : 0;
}

/* info: N, nsn, n_slots, ipool_n, arena_n, max_m, nnz_l_blocks, n_levels, n_factors, n_bs_leaf */
ASAM_API void asam_dbg_plan_info(void *p, int64_t *info, double *flops)
{
    plan_t *pl = (plan_t *) p;
    info[0] = pl->N;
    info[1] = pl->nsn;
    info[2] = pl->n_slots;
    info[3] = pl->ipool_n;
    info[4] = pl->arena_n;
    info[5] = pl->max_m;
    info[6] = pl->nnz_l_blocks;
    info[7] = pl->n_levels;
    info[8] = pl->n_factors;
    info[9] = pl->n_bs_leaf;
    *flops = pl->flops;
}

/* which: 0 order 1 pos 2 node2q 3 q2node 4 parent_pos 5 fslot 6 sn_of_q 7 ipool 8 tasks 9 nwait
 * 10 btasks 11 desc (as int32 words, 12 per supernode) 12 leaf_tasks 13 top_tasks 14 top_nwait
 * 15 shard_owner 16 shard_q0 17 shard_qn 18 shard_off (int64 as 2 words) 19 shard_cnt (int64) */
ASAM_API const int *asam_dbg_plan_array(void *p, int which, int64_t *count)
{
    plan_t *pl = (plan_t *) p;
    switch (which) {
    case 0: *count = pl->N; return pl->order;
    case 1: *count = pl->N; return pl->pos;
    case 2: *count = pl->N; return pl->node2q;
    case 3: *count = pl->N; return pl->q2node;
    case 4: *count = pl->N; return pl->parent_pos;
    case 5: *count = pl->n_factors; return pl->fslot;
    case 6: *count = pl->N; return pl->sn_of_q;
    case 7: *count = pl->ipool_host.n; return pl->ipool_host.p;
    case 8: *count = pl->tasks ? pl->ntasks : 0; return pl->tasks;
    case 9: *count = pl->nwait ? pl->ntasks : 0; return pl->nwait;
    case 10: *count = pl->btasks ? pl->n_btasks : 0; return pl->btasks;
    case 11: *count = 12 * (int64_t) pl->nsn; return (const int *) pl->desc;
    case 12: *count = pl->leaf_tasks ? pl->n_leaf : 0; return pl->leaf_tasks;
    case 13: *count = pl->top_tasks ? pl->n_top : 0; return pl->top_tasks;
    case 14: *count = pl->top_nwait ? pl->n_top : 0; return pl->top_nwait;
    case 15: *count = pl->shard_owner ? pl->n_shards : 0; return pl->shard_owner;
    case 16: *count = pl->shard_q0 ? pl->n_shards : 0; return pl->shard_q0;
    case 17: *count = pl->shard_qn ? pl->n_shards : 0; return pl->shard_qn;
    case 18: *count = pl->shard_off ? 2 * (int64_t) pl->n_shards : 0; return (const int *) pl->shard_off;
    case 19: *count = pl->shard_cnt ? 2 * (int64_t) pl->n_shards : 0; return (const int *) pl->shard_cnt;
    default: *count = 0; return NULL;
    }
}

ASAM_API int asam_dbg_ref_ordering(int N, const int *adj_ptr, const int *adj, int *out)
{
    int *o = asam_ref_ordering(N, adj_ptr, adj);
    memcpy(out, o, sizeof(int) * (size_t) (N > 0 ? N : 0));
    free(o);
    return 0;
}

ASAM_API int asam_dbg_ref_ordering_explicit(int N, const int *adj_ptr, const int *adj, int *out)
{
    int *o = asam_ref_ordering_explicit(N, adj_ptr, adj);
    memcpy(out, o, sizeof(int) * (size_t) (N > 0 ? N : 0));
    free(o);
    return 0;
}

void asam_dbg_plan_profile(double *out, int reset);
ASAM_API void asam_dbg_plan_profile_get(double *out, int reset) { asam_dbg_plan_profile(out, reset); }

void asam_dbg_build_profile(double *out, int reset);
ASAM_API void asam_dbg_build_profile_get(double *out, int reset) { asam_dbg_build_profile(out, reset); }
