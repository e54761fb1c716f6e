/* asam_host.h -- internal declarations of the host side (C) of aprilsam_b200. */
#ifndef ASAM_HOST_H
#define ASAM_HOST_H

#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "aprilsam.h"
#include "asam_cuda.h"
#include "common/stype.h"

#define ASAM_API __attribute__((visibility("default")))

/* Factor types the solver treats as an xyt factor between two poses: plain xyt (1) and robust xyt (32).
 * Every host site that decides "one pose or two" asks this, never the type code itself. */
static inline int asam_two_pose_type(int type)
{
    return type == APRIL_GRAPH_FACTOR_XYT_TYPE || type == APRIL_GRAPH_FACTOR_XYT_ROBUST_TYPE;
}

/* ---- small containers ---------------------------------------------------------------- */
typedef struct {
    int *p;
    int n, cap;
} ivec_t;

static inline void ivec_reserve(ivec_t *v, int cap)
{
    if (cap <= v->cap)
        return;
    int c = v->cap ? v->cap : 8;
    while (c < cap)
        c *= 2;
    v->p = (int *) realloc(v->p, sizeof(int) * (size_t) c);
    v->cap = c;
}

static inline void ivec_push(ivec_t *v, int x)
{
    if (v->n == v->cap)
        ivec_reserve(v, v->n + 1);
    v->p[v->n++] = x;
}

static inline void ivec_free(ivec_t *v)
{
    free(v->p);
    v->p = NULL;
    v->n = v->cap = 0;
}

/* (lo,hi) node pair -> Hessian off-diagonal slot */
typedef struct {
    uint64_t *keys;
    int *vals;
    int cap, n; /* cap is a power of two */
} pairmap_t;

void pairmap_init(pairmap_t *m, int expect);
void pairmap_free(pairmap_t *m);
/* returns the slot of (lo,hi); *created = 1 if it was inserted with value `next_slot` */
int pairmap_get_or_add(pairmap_t *m, int lo, int hi, int next_slot, int *created);

/* Host threads for the symbolic loops: ASAM_PLAN_THREADS (default 8, capped at 16), or 1 when a short calibration at first
 * use finds that threads do not actually run side by side here (CPU quota of a container: eight threads on one core
 * made the plan build of the 100 k world four times SLOWER). */
int asam_host_threads(void);

/* ---- ordering (ordering.c) ----------------------------------------------------------- */
/* Reference-equivalent elimination order; adj lists ascending, no self loops.
 * Returns malloc'd order[pos] = node. */
int *asam_ref_ordering(int N, const int *adj_ptr, const int *adj);
int *asam_ref_ordering_explicit(int N, const int *adj_ptr, const int *adj); /* cross-check (tests) */

/* ---- symbolic plan (plan.c) ----------------------------------------------------------- */
#define ASAM_TR_FLAG (1 << 30) /* a_rb flag: gather the slot transposed */

typedef struct {
    ivec_t rows;     /* block rows in q positions, ascending; first cb = own columns  */
    ivec_t rel;      /* rel[k] = index of rows[k] in the parent's rows (k >= cb)       */
    ivec_t children; /* supernode ids                                                   */
    ivec_t a_slot, a_rb, a_cb;
} sn_host_t;

typedef struct {
    int N;        /* nodes covered by the plan                                        */
    int *order;   /* reference elimination position -> node (mirrors param->ordering)  */
    int *pos;     /* node -> reference position                                        */
    int *node2q;  /* node -> numeric position (post-order of the block etree)          */
    int *q2node;
    int *parent_pos; /* block etree in reference positions (node level), -1 = root     */
    int node_cap;

    pairmap_t pairs;
    int n_slots;
    int *fslot; /* per factor; -1 for unary factors */
    int fslot_cap;
    int n_factors; /* factors covered by the plan */

    int nsn, sn_cap;
    asam_sn_desc_t *desc;
    sn_host_t *snh;
    int *sn_of_q;
    int *mark_idx; /* plan_append scratch: supernode -> index among the marked ones, -1 between steps */
    int mark_cap;

    ivec_t ipool_host; /* host copy of the device int pool */
    int64_t ipool_n;  /* ints used in the device pool   */
    int64_t arena_n;  /* doubles used in the device arena */
    int max_m;        /* largest front order (scalars)  */

    /* full task lists (batch): ntasks entries of tasks/nwait (teams expanded), nsn of btasks */
    int *tasks, *nwait, *btasks;
    int ntasks;
    int *leaf_tasks; /* supernodes factored by k_factor_leaf before `tasks` (large graphs only) */
    int n_leaf;
    int n_btasks;    /* entries of btasks (>= the supernodes in it: wide supernodes have one entry per 96-column block) */
    int bt_split;    /* btasks holds per-block entries (batch schedule only; undone by the first plan_append) */
    char *bs_leaf;   /* per supernode: back-solved by k_backsolve_leaf (last n_bs_leaf entries of btasks) */
    int n_bs_leaf;

    /* multi-GPU sharding (world > 1): tasks / leaf_tasks / btasks then cover this rank's shards
     * (+ the top in btasks); see build_schedule() in plan.c */
    int world, rank;
    int max_team;   /* largest CTA team k_factor can seat (resident CTAs of the device; 0 = default) */
    int n_cta;      /* resident CTAs of k_factor on the device (0 = 132, the SMs of an H100): processors of the simulated schedule */
    int *top_tasks, *top_nwait;
    int n_top, n_top_sn;
    int n_shards;
    int *shard_owner, *shard_q0, *shard_qn;
    int64_t *shard_off, *shard_cnt;

    /* statistics of the last build */
    int64_t nnz_l_blocks; /* sum over nodes of (1 + |below|) */
    double flops;         /* sum over scalar columns of count^2 */
    int n_levels;

    /* structure cache */
    uint64_t struct_hash;
} plan_t;

void plan_free(plan_t *pl);

/* Build ordering + symbolic factorisation + supernodes + gather lists for the first
 * n_factors factors over N nodes and upload everything to `dev`.  ftype/fa/fb are the
 * factor type and node ids.  Returns 0 on success. */
int plan_build(plan_t *pl, asam_dev_t *dev, int N, int n_factors, const int *ftype, const int *fa, const int *fb);

/* Same, but keep a given elimination order for the first N_keep nodes (order_keep[pos]) and
 * append the remaining nodes in id order (used by the incremental fallback). */
int plan_build_with_order(plan_t *pl, asam_dev_t *dev, int N, int n_factors, const int *ftype, const int *fa,
                          const int *fb, const int *order_keep, int N_keep);

/* Incremental append: nodes [pl->N, N) and factors [pl->n_factors, n_factors) are new and
 * every new binary factor touches at least one new node.  marked_old = graph-node ids of
 * old nodes on the root paths (any order).  On return tasks_out/nwait_out (malloc'd, length
 * *ntasks_out) list the supernodes to re-factor, children first; keep_out (may be NULL) gets, per
 * task, (poses kept << 16) | block rows before the step, 0 = re-factor the whole front.
 * Returns 0 ok, 1 error, 2 = not an append-only update (caller falls back). */
int plan_append(plan_t *pl, asam_dev_t *dev, int N, int n_factors, const int *ftype, const int *fa, const int *fb,
                const int *marked_old, int n_marked, int **tasks_out, int **nwait_out, int **keep_out, int *ntasks_out);

/* Re-factorisation list of a step that changes no structure (aprilsam_b200_remove_factors): marked = graph-node ids on
 * the root paths (any order, all < pl->N).  tasks / nwait / keep (malloc'd, *ntasks_out entries) as plan_append gives
 * them: the supernodes holding a marked pose, children first, nwait counting their marked children, keep =
 * (poses before the first marked one << 16) | block rows, teams expanded (keep 0).  Emits no segments and uploads
 * nothing; the plan is left as it was.  Returns 0. */
int plan_refactor(plan_t *pl, const int *marked, int n_marked, int **tasks_out, int **nwait_out, int **keep_out,
                  int *ntasks_out);

/* Factors sorted_idx[0..n) (ascending, distinct, in [0, n_factors)) leave the plan: fslot and n_factors are compacted,
 * the order of the other factors kept, and fslot is uploaded from sorted_idx[0] on (dev may be NULL).  Hessian slots
 * stay; one that no remaining factor maps to is a dead zero block.  struct_hash becomes 0.  Nothing changes on an
 * invalid list: 1 and the error text. */
int plan_remove_factors(plan_t *pl, asam_dev_t *dev, int n, const int *sorted_idx);

/* Modelled cost (columns x rows^2 + a latency term per front, the measure build_schedule balances
 * shards with) of re-factoring the distinct supernodes in tasks[0..ntasks) and of factoring every
 * supernode of the plan; feeds the escalation policy hook (aprilsam.h). */
void plan_work(const plan_t *pl, const int *tasks, int ntasks, double *step_work, int *step_fronts, double *batch_work,
               int *batch_fronts);

/* Where each pose's columns of L^-1 live during a covariance query (asam_marginal_cov): for nodes[i], its
 * supernode sn0 and first scalar column j0 = 3 (q - first) in it, and its entries of the hop table and the
 * scratch (one hop per supernode from sn0 to the root; 3 doubles per scalar row, from j0 in sn0 and from 0
 * above).  A pure function of the plan.  Returns 0, or -1 (and the error text) for a node outside [0, pl->N). */
int plan_marginal_paths(const plan_t *pl, int n, const int *nodes, asam_marg_path_t *out, int64_t *z_total,
                        int *hop_total);

/* Batches of a candidate query (aprilsam_b200_candidate_mahalanobis): candidates c in input order, where candidate
 * c is a factor on poses a[c] and b[c] (b[c] = -1: a prior on a[c]; ids valid, checked by the caller).  A batch
 * closes before the candidate whose new poses would take the scratch of its distinct poses beyond `budget` doubles;
 * a batch always holds at least one candidate.  Batch t holds candidates [batch_end[t-1], batch_end[t]) and the
 * distinct poses poses[pose_end[t-1], pose_end[t]) in order of first use; ia[c] / ib[c] are the places of a[c] /
 * b[c] in that list (ib = -1 for a prior).  poses needs room for 2k ids, batch_end and pose_end for k.  A pure
 * function of the plan, the ids and the budget. */
void plan_candidate_batches(const plan_t *pl, int k, const int *a, const int *b, int64_t budget, int *batch_end,
                            int *n_batches, int *poses, int *pose_end, int *ia, int *ib);

/* Bytes of z scratch a batch of a candidate query may take (solver.c; tests lower it through debug.c) */
#define ASAM_CANDIDATE_BUDGET ((int64_t) 256 << 20)
extern int64_t asam_candidate_budget;

/* ---- solver context (solver.c) --------------------------------------------------------- */
void asam_graph_forget(april_graph_t *g);
/* graph.c: loss code and k of a factor; (0, 0) for factors without a robust loss */
void asam_factor_loss(const april_graph_factor_t *f, int32_t *loss, double *k);
/* graph.c: Jacobians of the xyt prediction (pose b in pose a's frame) at (pa, pb), row-major 3x3 */
void asam_xyt_jacobians(const double *pa, const double *pb, double *Ja, double *Jb);
/* graph.c: residual z - h(x) of an xyt factor at (pa, pb) and of an xytpos factor at pa, theta wrapped by mod2pi;
 * the eval hooks and the candidate query share them */
void asam_xyt_residual(const double *z, const double *pa, const double *pb, double *r);
void asam_xytpos_residual(const double *z, const double *pa, double *r);
/* serial.c */
extern const stype_t stype_april_graph, stype_april_graph_attr, stype_april_node_xyt, stype_april_factor_xyt,
    stype_april_factor_xytpos, stype_april_factor_xyt_robust;
april_graph_attr_t *asam_attr_dup(const april_graph_attr_t *a);
void asam_set_error(const char *fmt, ...);
void asam_fatal(const char *fmt, ...);

#endif
