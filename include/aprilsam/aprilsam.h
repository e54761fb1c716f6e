/* aprilsam.h -- public API of aprilsam_b200 (drop-in for AprilSAM's solver path).
 *
 * This header re-declares, from scratch, the part of the reference's public C API
 * that the Gauss-Newton path touches (reference: aprilsam/aprilsam.h).  Struct layouts
 * are ABI-identical on x86-64 (checked by the _Static_asserts at the bottom; offsets
 * from SURVEY.md section 8b) so a program written against the reference re-links against
 * libaprilsam_b200.so unchanged.  Each declaration cites the reference line it replaces.
 *
 * What runs where: every entry point below is host C; all arithmetic of
 * april_graph_cholesky{,_inc}() and april_graph_chi2() -- linearisation, J'WJ assembly,
 * sparse Cholesky, triangular solves -- runs in sm_90a CUDA kernels behind the C-ABI in
 * include/asam_cuda.h.  There is no CPU fallback: without a CUDA device the solver entry
 * points abort with a message.
 */
#ifndef APRILSAM_B200_APRILSAM_H
#define APRILSAM_B200_APRILSAM_H

#include <stdbool.h> /* the reference's headers pull it in; its examples rely on that */
#include <stdint.h>
#include <stdlib.h>

#include "common/doubles.h"
#include "common/matd.h"
#include "common/stype.h"
#include "common/zarray.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Types the reference exposes through pointers only; opaque here. */
typedef struct zhash zhash_t;
typedef struct smatd smatd_t;

/* reference: aprilsam/common/smatd.h:62-67.  In this library `u` is unused and the
 * object is the owner of the opaque GPU solver context (see aprilsam_b200/host). */
typedef struct {
    smatd_t *u;
    int is_spd;
} smatd_chol_t;

void APRILSAM_VERSION(void); /* aprilsam.h:44 */
int64_t utime_now(void);     /* common/time_util.h:45: microseconds since the epoch (the examples time with it) */

/* ---- attributes (aprilsam.h:46-61): string -> (stype, value) table ---------------- */
typedef struct april_graph_attr april_graph_attr_t;
struct april_graph_attr {
    zhash_t *hash; /* opaque: this library keeps a small insertion-ordered table behind it */
    const stype_t *stype;
};
april_graph_attr_t *april_graph_attr_create(void);          /* aprilsam.h:60 */
void april_graph_attr_destroy(april_graph_attr_t *attr);    /* aprilsam.h:61; NULL is fine */

/* ---- graph (aprilsam.h:64-72) ------------------------------------------------------ */
typedef struct april_graph april_graph_t;
struct april_graph {
    zarray_t *factors; /* of april_graph_factor_t*  */
    zarray_t *nodes;   /* of april_graph_node_t*    */
    april_graph_attr_t *attr;
    const stype_t *stype;
};

/* ---- factor evaluation record (aprilsam.h:75-89) ----------------------------------- */
typedef struct april_graph_factor_eval april_graph_factor_eval_t;
struct april_graph_factor_eval {
    double chi2;
    matd_t **jacobians; /* one per connected node, NULL-terminated */
    int length;
    double *r; /* residual, length x 1   */
    matd_t *W; /* information, length^2  */
};

#define APRIL_GRAPH_FACTOR_XYT_TYPE 1    /* aprilsam.h:91 */
#define APRIL_GRAPH_FACTOR_XYTPOS_TYPE 2 /* aprilsam.h:92 */
#define APRIL_GRAPH_NODE_XYT_TYPE 100    /* aprilsam.h:94 */

/* ---- factor (aprilsam.h:98-146) ---------------------------------------------------- */
typedef struct april_graph_factor april_graph_factor_t;
struct april_graph_factor {
    int type;
    int nnodes;
    int *nodes; /* indices into graph->nodes */
    int length; /* residual DOF */
    april_graph_attr_t *attr;

    april_graph_factor_t *(*copy)(april_graph_factor_t *factor);
    /* Host-side plug-in hooks kept for API compatibility.  The GPU solver does NOT call
     * them: it dispatches on `type` and evaluates xyt / xytpos factors in-kernel. */
    april_graph_factor_eval_t *(*eval)(april_graph_factor_t *factor, april_graph_t *graph,
                                       april_graph_factor_eval_t *eval);
    april_graph_factor_eval_t *(*state_eval)(april_graph_factor_t *factor, april_graph_t *graph,
                                             april_graph_factor_eval_t *eval);
    void (*destroy)(april_graph_factor_t *factor);

    union {
        struct {
            double *z;
            double *ztruth;
            matd_t *W;
            void *impl;
        } common;
        struct {
            april_graph_factor_t **factors;
            double *logw;
            int nfactors;
        } max;
        struct {
            void *impl;
        } impl;
    } u;

    const stype_t *stype;
};

/* ---- node (aprilsam.h:151-179) ----------------------------------------------------- */
typedef struct april_graph_node april_graph_node_t;
struct april_graph_node {
    int UID;
    int type;
    int length; /* DOF */

    double *state;   /* current estimate                      */
    double *init;
    double *truth;
    double *l_point; /* linearisation point                   */
    double *delta_X; /* last solved offset from l_point        */

    april_graph_attr_t *attr;

    april_graph_node_t *(*copy)(april_graph_node_t *node);
    void (*update)(april_graph_node_t *node, double *dstate); /* state = l_point + dstate */
    void (*relinearize)(april_graph_node_t *node);            /* l_point = state         */
    void (*destroy)(april_graph_node_t *node);

    void *impl;
    const stype_t *stype;
};

/* ---- graph lifecycle (aprilsam.h:184-188) ------------------------------------------ */
april_graph_t *april_graph_create(void);
void april_graph_destroy(april_graph_t *graph);
void april_graph_factor_eval_destroy(april_graph_factor_eval_t *eval);

/* ---- block elimination tree (aprilsam.h:190-228) ----------------------------------- */
typedef struct search_tree_node search_tree_node_t;
struct search_tree_node {
    int *children; /* graph-node ids */
    int parent;    /* graph-node id, -1 = none */
    int nalloc;
    int nchildren;
    int id; /* position in the elimination order */
    april_graph_node_t *g_node;
    int label_changed;      /* on a root path of a factor added this step */
    int label_relinearized; /* counted towards start_over since the last batch */
};

typedef struct search_tree search_tree_t;
struct search_tree {
    int nnodes;
    int nalloc;
    search_tree_node_t *root;
    search_tree_node_t *nodes; /* indexed by graph-node id */
    int start_over;
    int nlinearized_nodes;
    int *linearized_nodes;
    int isam1_cnt;
    int naffected;
    double delta_xy;
    double delta_theta;
    double total_delta_xy;
    double total_delta_theta;
};

void search_tree_destroy(search_tree_t *tr);

/* ---- solver parameters + persistent state (aprilsam.h:231-265) --------------------- */
typedef struct april_graph_cholesky_param april_graph_cholesky_param_t;
struct april_graph_cholesky_param {
    double tikhanov; /* lambda added to every diagonal entry at each batch solve */

    smatd_chol_t *chol; /* non-NULL once a batch solve has run (owns the GPU context) */
    int factor_num;     /* factors consumed so far */

    int *ordering;   /* ordering[pos] = graph-node id; owned by the param */
    int nreordering; /* non-zero = enabled; after a solve: node count at that solve */
    int show_timing;

    double *delta_x; /* unused (reference leaves it dangling, aprilsam.c:360-366) */
    double *B;       /* unused here: rhs lives in HBM */
    double *y;       /* unused here */
    smatd_t *A;      /* unused here: the block Hessian lives in HBM */

    search_tree_t *tr;

    double l_thresh;     /* unused by the reference solver */
    double delta_thresh; /* unused by the reference solver */
    int nthreshold;      /* batch re-solve when more than this many nodes moved */

    double batch_time;

    double delta_xy;    /* relinearisation thresholds */
    double delta_theta;
};

/* aprilsam.h:268-269 (the spelling "destory" is the reference's) */
void april_graph_cholesky_param_init(april_graph_cholesky_param_t *param);
void april_graph_cholesky_param_destory(april_graph_cholesky_param_t *param);

/* aprilsam.h:274-276 */
void april_graph_cholesky(april_graph_t *graph, april_graph_cholesky_param_t *param);
void april_graph_cholesky_inc(april_graph_t *graph, april_graph_cholesky_param_t *param);
void april_graph_cholesky_inc_solver(april_graph_t *graph, april_graph_cholesky_param_t *param, int *idxs);

/* aprilsam.h:280-281 */
int april_graph_dof(april_graph_t *graph);
double april_graph_chi2(april_graph_t *graph);

/* aprilsam.h:283-286 */
april_graph_node_t *april_graph_node_xyt_create(const double *state, const double *init, const double *truth);
april_graph_factor_t *april_graph_factor_xyt_create(int a, int b, const double *z, const double *ztruth, const matd_t *W);
april_graph_factor_t *april_graph_factor_xytpos_create(int a, double *z, double *ztruth, matd_t *W);

/* ---- files and attributes (aprilsam.h:185, :288-299; SURVEY.md section 8f) --------------
 * ".graph" files in the reference's stype framing (big-endian, self-describing); call
 * april_graph_stype_init() (and stype_register_basic_types() for "string"/"uint64" attribute
 * values) once before loading.  Values put into an attribute table are owned by it afterwards
 * (destroyed through their stype); a value replaced by a second put stays the caller's. */
april_graph_t *april_graph_create_from_file(const char *path); /* NULL on failure */
int april_graph_save(april_graph_t *graph, const char *path); /* 1 on success, 0 on failure */
void april_graph_stype_init(void);
void april_graph_attr_put(april_graph_t *graph, const stype_t *type, const char *key, void *data);
void *april_graph_attr_get(april_graph_t *graph, const char *key);
void april_graph_factor_attr_put(april_graph_factor_t *factor, const stype_t *type, const char *key, void *data);
void *april_graph_factor_attr_get(april_graph_factor_t *factor, const char *key);
void april_graph_node_attr_put(april_graph_node_t *node, const stype_t *type, const char *key, void *data);
void *april_graph_node_attr_get(april_graph_node_t *node, const char *key);

/* Last error text of this library on the calling thread ("" if none).  Extension: the
 * reference reports nothing (void returns, asserts, NULL dereference on non-SPD). */
const char *aprilsam_b200_last_error(void);

/* Drop the cached ordering + symbolic analysis of `param`: the next april_graph_cholesky() orders
 * and analyses the graph again, as the reference does on every call (aprilsam.c:104-128, :216-258).
 * Extension; never needed for correctness (the cache is keyed on the factor structure and factor
 * values are re-checked on every batch call) -- it exists so that the uncached cost can be measured. */
void aprilsam_b200_invalidate_plan(april_graph_cholesky_param_t *param);

/* ---- robust loop closures (extension) ----------------------------------------------------------
 * A type-32 factor is an xyt factor between two poses (same z, W, Jacobians and residual as type 1)
 * with an M-estimator loss of scale k > 0.  At s = r'Wr (r at the factor's evaluation point):
 *   Huber   w = 1 if s <= k^2, else k / sqrt(s)     rho = s if s <= k^2, else 2 k sqrt(s) - k^2
 *   Cauchy  w = 1 / (1 + s / k^2)                   rho = k^2 log1p(s / k^2)
 * Every linearisation uses W_eff = w W (iteratively reweighted least squares, no second-order term);
 * april_graph_chi2 counts 0.5 rho(s) at the states.  The eval / state_eval hooks return W_eff and
 * chi2 = rho(s).  w and rho are accurate for every finite k > 0 and every finite s >= 0: within a few ulp of
 * the exact value where that lies in [DBL_MIN, DBL_MAX / 4], within DBL_MIN of it below, never NaN.  So a
 * Cauchy loss may be switched off with k = DBL_MAX, and a tiny k leaves a factor at zero residual its full W.
 * Files holding such factors ("april_graph_factor_xyt_robust") are this library's own. */
#define APRIL_GRAPH_FACTOR_XYT_ROBUST_TYPE 32
enum { APRILSAM_B200_LOSS_HUBER = 1, APRILSAM_B200_LOSS_CAUCHY = 2 };
/* NULL (text in aprilsam_b200_last_error) unless loss is one of the above and k is finite and > 0 */
april_graph_factor_t *aprilsam_b200_factor_xyt_robust_create(int a, int b, const double *z, const double *ztruth,
                                                             const matd_t *W, int loss, double k);
/* change loss / k of a robust factor: 0 ok, -1 (and last_error) for another factor type or invalid values.
 * Like an edit of z / W: used from the next batch solve on, not by incremental steps before it. */
int aprilsam_b200_factor_set_loss(april_graph_factor_t *f, int loss, double k);

/* ---- marginal covariances (extension) ------------------------------------------------------------
 * Uncertainty of poses from the factor L the GPU holds after the last april_graph_cholesky() or
 * april_graph_cholesky_inc() of `graph` with `param`: Sigma = A^-1 of the system that solve factored, that is
 * J'WJ at each factor's evaluation point (its linearisation point, not `state`) plus tikhanov on the poses
 * that existed at the last batch solve (incremental steps give new poses no such term).  Nothing is
 * re-factored and nothing changes: not the graph, `param`, the tree, the solver's device state or what the
 * next call does.  The cost follows the root paths of the poses asked for.
 *
 * Absolute covariances of a graph without a prior are set mostly by tikhanov: about 1/tikhanov in the gauge
 * directions.  The relative covariance is free of the gauge; it is what gating a candidate loop closure by its
 * Mahalanobis distance needs.
 *
 * Both return 0, or -1 with the reason in aprilsam_b200_last_error() for NULL arguments or n < 1, node ids
 * outside the graph, a `param` that does not continue a solve of `graph`, a plan dropped by
 * aprilsam_b200_invalidate_plan, nodes or factors added since the last solve, or a sharded batch solve (a rank
 * holds only its own shards' fronts).
 *
 * out: (3n) x (3n), row-major; block (a, b) = cov(x_nodes[a], x_nodes[b]) in (x, y, theta) order.  Exactly
 * symmetric, the same on every call, and block (a, b) does not depend on the other nodes asked for. */
int aprilsam_b200_marginal_covariance(april_graph_t *graph, april_graph_cholesky_param_t *param, int n, const int *nodes,
                                      double *out);
/* Covariance (3 x 3, row-major) of pose b expressed in pose a's frame: J Sigma_ab J' with Sigma_ab the 6 x 6 joint
 * marginal of (a, b) and J = [J_a J_b] the Jacobians of an xyt factor between a and b at their l_points. */
int aprilsam_b200_relative_covariance(april_graph_t *graph, april_graph_cholesky_param_t *param, int a, int b,
                                      double out9[9]);
/* Mahalanobis distances of k candidate factors against the last solve, for gating loop closures.  Candidate c is
 * the factor the caller would add: an xyt factor between poses a[c] and b[c] (b[c] >= 0), or a prior (xytpos) on
 * pose a[c] (b[c] == -1), with measurement z (3k doubles) and information matrix W (9k doubles, row-major), the
 * same z and W that april_graph_factor_xyt_create / _xytpos_create take.  With r the factor's residual at the
 * current states (theta wrapped by mod2pi, as the eval hooks compute it) and
 *   Sigma_rel = J Sigma_ab J'  (J = [J_a J_b] at the l_points: exactly aprilsam_b200_relative_covariance(a, b))
 *   Sigma_rel = Sigma_aa       (a prior: the diagonal block of aprilsam_b200_marginal_covariance)
 * d2[c] = r' (Sigma_rel + W^-1)^-1 r, NaN if Sigma_rel + W^-1 is not numerically positive definite.  A caller
 * accepts a candidate when d2 is below a chi-square quantile with 3 degrees of freedom, for example 7.815 (95 %)
 * or 11.345 (99 %).  Without a prior in the graph Sigma_aa is mostly 1/tikhanov, so prior candidates are only
 * meaningful on graphs that hold a prior.
 *
 * cov9 (NULL allowed): Sigma_rel of every candidate, 9 doubles row-major, exactly symmetric.  A candidate's d2 and
 * Sigma_rel are the same alone or in any request, in any order, and from call to call.  The cost follows the
 * distinct poses: a pose that appears in many candidates is walked once.
 *
 * Returns 0, or -1 with the reason in aprilsam_b200_last_error() for the cases of the covariance queries above, and
 * for k < 1, NULL a / b / z / W / d2, b[c] < -1, a[c] == b[c], a non-finite z or a W that is not exactly symmetric
 * and positive definite; the message names the index of the candidate at fault.  d2 and cov9 are unspecified after
 * an error; the solver stays usable. */
int aprilsam_b200_candidate_mahalanobis(april_graph_t *graph, april_graph_cholesky_param_t *param, int k, const int *a,
                                        const int *b, const double *z, const double *W, double *d2, double *cov9);

/* ---- candidate compatibility (extension) ---------------------------------------------------------------------------
 * Which candidates can be true together.  aprilsam_b200_candidate_mahalanobis tests each candidate on its own; on a
 * long loop Sigma_rel is large, so a false closure from perceptual aliasing (a corridor, a row of doors, a repeated
 * room) passes that gate, and usually several pass together.  Their residuals share one drift, because the Sigma_rel of
 * neighbouring closures are strongly correlated: two closures that each sit inside their own ellipse can pull that
 * drift in opposite directions.  Testing them jointly catches this (pairwise compatibility and a maximum clique, as in
 * CCDA or PCM; or joint compatibility, JCBB).
 *
 * aprilsam_b200_candidate_compatibility: for k candidates exactly as aprilsam_b200_candidate_mahalanobis takes them
 * (a[c], b[c], z, W; b[c] = -1 for a prior on a[c]; r at the states, J at the l_points; the same validation and error
 * texts), with Sigma as aprilsam_b200_marginal_covariance defines it and J = [I 0] for a prior:
 *   C_ij = J_i Sigma_(a_i b_i),(a_j b_j) J_j'      the cross-covariance of the two residuals
 *   S_i  = Sigma_rel,i + W_i^-1
 *   d2[i*k + j] = [r_i; r_j]' S_ij^-1 [r_i; r_j],  S_ij = [S_i C_ij; C_ij' S_j]   (i != j)
 *   d2[c*k + c] = the d2 aprilsam_b200_candidate_mahalanobis returns for c, bit for bit.
 * d2 is k x k, row-major and exactly symmetric.  Compare an off-diagonal entry with a chi-square quantile with 6
 * degrees of freedom: 16.81 (99 %), 22.46 (99.9 %).  It is NaN when S_ij is not numerically positive definite (a
 * pivot of its 6 x 6 Cholesky is not > 0).  In the linear model d2[i*k + j] = d2_i + d2_(j|i), d2_(j|i) the candidate
 * distance of j against the solve with i added, and d2[i*k + j] >= max(d2_i, d2_j).
 *
 * cross9 (NULL allowed): C_ij for every ordered pair, k x k x 9 doubles, each block row-major; cross9 at (j, i) is the
 * exact transpose of (i, j), and cross9 at (c, c) is Sigma_rel of c, the cov9 of aprilsam_b200_candidate_mahalanobis,
 * bit for bit.  With it a caller can run JCBB on any subset: S of a set is these blocks plus W^-1 on the diagonal.
 *
 * An entry (i, j) depends only on candidates i and j: the same bits for the pair alone (k = 2), inside any request, in
 * any order (a permutation of the input permutes the matrix), under any tiling and from call to call.  The pairs are
 * computed in tiles whose query scratch stays within the candidate query's budget (256 MiB); each tile walks the root
 * paths of its distinct poses once, and when the whole request fits, every distinct pose is walked once.  The cost
 * grows with k^2 (one small 6 x 6 problem and up to four 3 x 3 blocks of Sigma per pair) plus the path walks; nothing
 * but the query scratch on the GPU is written.
 *
 * Returns 0, or -1 with the reason in aprilsam_b200_last_error() and nothing changed for everything
 * aprilsam_b200_candidate_mahalanobis refuses and for k > APRILSAM_B200_COMPAT_MAX_K (checked before d2 is touched):
 * the kernel indexes a tile's k x k pair slots with an int.  d2 and cross9 are unspecified after an error; the solver
 * stays usable. */
#define APRILSAM_B200_COMPAT_MAX_K 46340
int aprilsam_b200_candidate_compatibility(april_graph_t *graph, april_graph_cholesky_param_t *param, int k,
                                          const int *a, const int *b, const double *z, const double *W, double *d2,
                                          double *cross9);

/* ---- factor audit (extension) ------------------------------------------------------------------------------------
 * Which accepted factor has proved false.  A raw residual is the wrong test: the solve pulls the graph towards an
 * outlier, so its residual shrinks, and a factor the rest of the graph hardly checks looks good even when it is wrong.
 *
 * aprilsam_b200_factor_residuals: per factor f of [first, first + count), at the states (the values april_graph_chi2
 * sees): r = z - h(state) (theta wrapped by mod2pi, as the eval hooks compute it), s = r'Wr, the robust weight
 * w = w(s) of a robust factor (1 for other types) and chi2, the term april_graph_chi2 adds for f (0.5 s, 0.5 rho(s)
 * for a robust factor, s for a prior).  Summed in april_graph_chi2's order (256-factor blocks, each a 256-lane tree,
 * then a 256-lane tree over the blocks) the chi2 fields give april_graph_chi2 bit for bit.  Like april_graph_chi2 it
 * needs no solve and no param: it checks the factors against their HBM mirror (re-uploading edits), uploads the
 * states and runs one kernel.  Returns 0, or -1 with the reason in aprilsam_b200_last_error() for NULL arguments or a
 * range that is empty or not inside [0, F). */
typedef struct {
    double r[3];
    double s;
    double w;
    double chi2;
} aprilsam_b200_factor_residual_t;
int aprilsam_b200_factor_residuals(april_graph_t *graph, int first, int count, aprilsam_b200_factor_residual_t *out);

/* aprilsam_b200_factor_outlier_scores: the leave-one-out test of k factors of a solved graph (indices factor_idx[],
 * repeats allowed), with Sigma as aprilsam_b200_marginal_covariance defines it.  For factor f, with J = [J_a J_b] at
 * its evaluation point (the l_points), r its residual at the states, W_f the information matrix the Hessian holds
 * for it (W; w W for a robust factor, w at the evaluation point) and
 *   Sigma_rel = J Sigma_ab J'  (an xyt factor: exactly aprilsam_b200_relative_covariance(a, b))
 *   Sigma_rel = Sigma_aa       (a prior: the diagonal block of aprilsam_b200_marginal_covariance),
 *   d2[q]         = (W_f r)' N^-1 (W_f r),  N = W_f - W_f Sigma_rel W_f  (= r' (W_f^-1 - Sigma_rel)^-1 r)
 *   redundancy[q] = 3 - tr(Sigma_rel W_f).
 * In the linear model d2 is exactly the candidate distance (aprilsam_b200_candidate_mahalanobis) the factor would get
 * against the solve of the graph without it: compare it with a chi-square quantile with 3 degrees of freedom, for
 * example 16.27 (99.9 %).  The redundancy, in [0, 3], is how much of the factor the rest of the graph checks; summed
 * over all factors it gives the graph's degrees of freedom.  A bridge has redundancy 0 and cannot be tested: N is
 * singular and d2 is NaN (as for a non-positive pivot of N).  A factor with little redundancy gives a weak test.
 * r is taken at the states and J at the l_points: the test is the leave-one-out test of the linearised problem, so it
 * describes outliers only near convergence.  After a single solve from a poor initial guess, correct factors can
 * score high too; solve until the step is small before judging factors by d2.
 *
 * cov9 (NULL allowed): Sigma_rel, 9 doubles row-major.  A factor's outputs are the same alone or in any request, in
 * any order and batch split, and from call to call; nothing but the query scratch on the GPU is written.  The cost
 * follows the root paths of the factors' distinct poses: a pose near the leaves of a large graph has a long path, so
 * score the loop closures that aprilsam_b200_factor_residuals flags, not every factor of a large graph.
 *
 * Returns 0, or -1 with the reason in aprilsam_b200_last_error() and nothing changed for the cases of the covariance
 * queries above, and for k < 1, NULL factor_idx / d2 / redundancy, an index outside [0, F), a factor replaced since
 * the last solve, or a factor whose z / W / loss differs from the values the Hessian was built from (edited since the
 * last batch solve, whether or not april_graph_chi2 has re-checked it since); the message names the entry at
 * fault.  d2, redundancy and cov9 are unspecified after an error; the solver stays usable. */
int aprilsam_b200_factor_outlier_scores(april_graph_t *graph, april_graph_cholesky_param_t *param, int k,
                                        const int *factor_idx, double *d2, double *redundancy, double *cov9);

/* ---- factor removal (extension) --------------------------------------------------------------------------------
 * Take the n distinct factors factor_idx[] out of graph->factors; the others keep their order (later indices shift
 * down).  removed_out == NULL: the removed factors are destroyed through their destroy hook; otherwise removed_out[k]
 * receives factor factor_idx[k] and the caller owns it.
 *
 * If `param` has never solved `graph` (param->chol == NULL) this is the splice alone.  If it continues a batch or
 * incremental solve of `graph`, the solution is updated as an incremental step would update it, without
 * relinearising or re-ordering: the Hessian becomes the system of the remaining factors, each at its own evaluation
 * point (the l_points for xyt factors; for a prior, the l_point if it was there at the last batch solve, else the
 * state it was added at), plus the last batch's tikhanov on the poses that existed then; only the supernodes on the
 * root paths of the removed factors' poses are re-factored; label_changed, naffected (counted as if the removed
 * factors had been added by a step), the back-substitution rule (every pose when naffected > 5, otherwise the marked
 * paths, state = l_point + x), start_over, the nthreshold escalation and the escalation policy behave as in a step.
 * param->factor_num becomes F - n.  The elimination order and param->tr stay until the next batch solve, which
 * re-plans and takes the reference order of the reduced graph.  april_graph_chi2 and the queries above then work on
 * the reduced graph.
 *
 * Returns 0, or -1 with the reason in aprilsam_b200_last_error() and nothing changed (graph, param, device state) for:
 * NULL arguments or n < 1; an index outside [0, F) or listed twice; poses or factors added since the last solve (call
 * april_graph_cholesky_inc first); a plan dropped by aprilsam_b200_invalidate_plan; a sharded batch solve; a removal
 * that would leave a pose created since the last batch solve without any remaining factor connecting it to a pose of
 * that batch or to a prior (its pivot would be zero); a remaining factor on a removed factor's pose whose z / W /
 * loss was edited and re-checked (april_graph_chi2) since the last batch solve, so that HBM no longer holds the
 * values it was linearised with.
 *
 * Another param that solved the same graph no longer matches it: its next april_graph_cholesky re-plans, its
 * april_graph_cholesky_inc does nothing and sets aprilsam_b200_last_error, and its queries return -1, until then. */
int aprilsam_b200_remove_factors(april_graph_t *graph, april_graph_cholesky_param_t *param, int n, const int *factor_idx,
                                 april_graph_factor_t **removed_out);

/* ---- in-place relinearisation (extension) --------------------------------------------------------------------------
 * Relinearise the n distinct poses nodes[] (the set P) of a solved graph as one incremental step, without a batch
 * solve, a new ordering or a new plan -- what an incremental smoother does about drift instead of starting over.
 *
 * For every pose p of P, l_point = state (the copy april_graph_cholesky makes); no other l_point changes.  R is every
 * factor with a pose in P.  The dirty poses D are the poses of R's factors and P itself (a pose of P without factors
 * holds only its lambda); the dirty slots are the slots of R's two-pose factors.  Afterwards each factor is evaluated
 * where it was before (the l_points for xyt factors; for a prior, the l_point if it was there at the last batch solve,
 * else the state it was added at), except that R's factors are evaluated at the new l_points of P: a prior added by a
 * step on a pose of P moves to that pose's new l_point.  Every dirty pose is rebuilt from all its factors plus the last
 * batch's tikhanov if the pose existed then, every dirty slot from all its factors (fixed-order overwrites on the GPU);
 * nothing else in the Hessian is written.  The root paths of D are marked as if factors had been added on them
 * (label_changed, naffected), only their supernodes are re-factored, and the solve is a step's: the back-substitution
 * rule (every pose when naffected > 5, otherwise the marked paths, state = l_point + x), the escalation policy, the
 * nthreshold escalation and start_over.  The elimination order, the plan, param->tr, param->factor_num and
 * param->nreordering stay as they are.
 *
 * Counters, before the solve: every pose of P whose label_relinearized is set has it cleared and leaves
 * tr->linearized_nodes (the other entries keep their order); nlinearized_nodes and start_over drop by that count;
 * total_delta_xy / total_delta_theta stay.  The solve then flags poses as a step does, so a pose of P can be flagged
 * again.  nodes may be param->tr->linearized_nodes itself with n = param->tr->nlinearized_nodes ("relinearise what the
 * tree has flagged"): the list is copied before the tree is edited.
 *
 * Returns 0, or -1 with the reason in aprilsam_b200_last_error() and nothing changed (graph, param, device state) for:
 * NULL arguments or n < 1; an id outside [0, N) or listed twice; a param that does not continue a solve of this graph;
 * poses or factors added since the last solve (call april_graph_cholesky_inc first); a plan dropped by
 * aprilsam_b200_invalidate_plan; a sharded batch solve; a factor replaced since the last batch solve; a factor on a
 * dirty pose whose z / W / loss was edited and re-checked (april_graph_chi2) since the last batch solve, so that HBM no
 * longer holds the values its other contributions were built from.  Another param that solved the same graph becomes
 * stale as after a removal (its own error text names the relinearisation). */
int aprilsam_b200_relinearize_poses(april_graph_t *graph, april_graph_cholesky_param_t *param, int n, const int *nodes);

/* Relinearisation / re-ordering policy of april_graph_cholesky_inc().  The reference escalates an
 * incremental step to a full batch solve when `start_over > nthreshold` (kept) and, as shipped, also
 * when the step took longer than a third of the last batch solve by the WALL CLOCK
 * (aprilsam.c:556-559 "HACK", :569-572) -- results then depend on machine load.  This hook is the
 * deterministic replacement: after the symbolic update of every incremental step the policy sees the
 * modelled cost of that step next to the modelled cost of a batch solve of the whole graph (both from
 * the supernodal plan: sum over the fronts to (re-)factor of columns x rows^2 plus a per-front
 * latency term) and returns non-zero to escalate.  No policy (the default) = the reference with a
 * constant clock, which is what the parity tests pin. */
typedef struct {
    double step_work;   /* fronts re-factored by this step                                      */
    double batch_work;  /* every front of the current plan                                       */
    int step_fronts, batch_fronts;
    int naffected;      /* poses on the marked root paths (search_tree_t.naffected)              */
    int nnodes;         /* poses in the graph                                                    */
    int start_over;     /* poses relinearised since the last batch (compared with nthreshold)    */
} aprilsam_b200_step_cost_t;
typedef int (*aprilsam_b200_escalation_fn)(const aprilsam_b200_step_cost_t *cost, void *user);
/* fn == NULL removes the policy.  May be called before the first april_graph_cholesky(). */
void aprilsam_b200_set_escalation_policy(april_graph_cholesky_param_t *param, aprilsam_b200_escalation_fn fn,
                                         void *user);
/* Built-in policy, the reference's ratio made deterministic: escalate when
 * step_work > ratio * batch_work; `user` points to the ratio (double), NULL = 1/3. */
int aprilsam_b200_policy_work_ratio(const aprilsam_b200_step_cost_t *cost, void *user);

/* ---- ABI checks against the reference layout (SURVEY.md section 8b) ------------------ */
#if defined(__x86_64__) && !defined(__cplusplus)
#include <stddef.h>
_Static_assert(sizeof(zarray_t) == 24, "zarray_t");
_Static_assert(sizeof(aprilsam_b200_factor_residual_t) == 6 * sizeof(double), "aprilsam_b200_factor_residual_t");
_Static_assert(sizeof(april_graph_t) == 32, "april_graph_t");
_Static_assert(sizeof(april_graph_node_t) == 112 && offsetof(april_graph_node_t, state) == 16 &&
                   offsetof(april_graph_node_t, l_point) == 40 && offsetof(april_graph_node_t, delta_X) == 48 &&
                   offsetof(april_graph_node_t, update) == 72 && offsetof(april_graph_node_t, relinearize) == 80,
               "april_graph_node_t");
_Static_assert(sizeof(april_graph_factor_t) == 104 && offsetof(april_graph_factor_t, nodes) == 8 &&
                   offsetof(april_graph_factor_t, eval) == 40 && offsetof(april_graph_factor_t, u.common.z) == 64 &&
                   offsetof(april_graph_factor_t, u.common.W) == 80 && offsetof(april_graph_factor_t, stype) == 96,
               "april_graph_factor_t");
_Static_assert(sizeof(search_tree_node_t) == 40 && sizeof(search_tree_t) == 80, "search_tree");
_Static_assert(sizeof(april_graph_cholesky_param_t) == 128 && offsetof(april_graph_cholesky_param_t, chol) == 8 &&
                   offsetof(april_graph_cholesky_param_t, ordering) == 24 &&
                   offsetof(april_graph_cholesky_param_t, nreordering) == 32 &&
                   offsetof(april_graph_cholesky_param_t, tr) == 72 &&
                   offsetof(april_graph_cholesky_param_t, nthreshold) == 96 &&
                   offsetof(april_graph_cholesky_param_t, delta_xy) == 112,
               "april_graph_cholesky_param_t");
#endif

#ifdef __cplusplus
}
#endif
#endif
