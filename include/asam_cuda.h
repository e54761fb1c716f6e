/* asam_cuda.h -- C-ABI between the host solver (C) and the sm_90a CUDA kernels.
 *
 * Plain pointers and sizes only.  Every entry point returns 0 on success, non-zero on
 * failure (text via asam_last_error()).  All calls on one asam_dev_t must come from one
 * host thread (the reference library is single-threaded, SURVEY.md section 8b).
 *
 * Data model in HBM (all indices 32-bit, all arithmetic IEEE double):
 *   node i        graph->nodes index                         (reference: aprilsam.h:151-179)
 *   q = node2q[i] elimination position of node i (post-ordered block elimination tree)
 *   lp[3i], st[3i]        linearisation point / state mirrors   (april_graph_node_t.l_point/.state)
 *   factor f      type, node ids, z[3], W[9] mirrors            (april_graph_factor_t, aprilsam.h:98-146)
 *   Adiag[9i]     diagonal 3x3 block of node i of A = J'WJ (+lambda I), row-major, entries r<=c valid
 *   Aoff[9s]      off-diagonal block of node-pair slot s, stored [lower node id][higher node id]
 *   Bq[3i]        B = J'W r of node i                             (aprilsam.c:154-204)
 *   supernode s   consecutive positions first..first+cb-1 sharing one dense frontal matrix
 *                 F (m x m, column-major, m = 3*mb) + m rhs doubles at arena[f_off]:
 *                 columns [0,3cb) hold L after factorisation, the trailing block holds the
 *                 Schur complement ("update matrix") handed to the parent supernode.
 *   y[3q], x[3q]  forward-solve result and solution in elimination order (aprilsam.c:298)
 */
#ifndef ASAM_CUDA_H
#define ASAM_CUDA_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Leading dimension of a front of order m (rows 0..m-1 + the rhs row m), in doubles: m+1 rounded up to
 * even so that every column of the column-major front starts on a 16-byte boundary (the operands of the
 * trailing update travel to shared memory as bulk asynchronous copies, which need that). */
#define ASAM_LD(m) (((m) + 2) & ~1)

typedef struct asam_dev asam_dev_t;

/* Supernode descriptor as stored in HBM (48 bytes). `seg` is the offset into the int pool
 * of this supernode's index segment, laid out as
 *   rows[mb] | rel[mb] | children[ch_cnt] | a_slot[a_cnt] | a_rb[a_cnt] | a_cb[a_cnt]
 * rows = block-row list in q positions (first cb entries are the supernode's own columns),
 * rel[k] = index of rows[k] in the PARENT's row list (k >= cb), children = supernode ids,
 * (a_slot, a_rb, a_cb) = off-diagonal A blocks gathered into block (row a_rb, col a_cb);
 * bit 30 of a_rb is set when the column node is the higher node id (gather transposed). */
typedef struct asam_sn_desc {
    int32_t first, cb, mb, parent;
    int32_t seg, ch_cnt, a_cnt, level;
    int64_t f_off;
    int64_t reserved;
} asam_sn_desc_t;

const char *asam_last_error(void);

/* Context on the current CUDA device (env ASAM_DEVICE or LOCAL_RANK selects it). */
int asam_dev_create(asam_dev_t **out);
void asam_dev_destroy(asam_dev_t *d);
int asam_device_count(void);

/* Capacity management (grow-only; contents preserved). */
int asam_reserve(asam_dev_t *d, int n_nodes, int n_factors, int n_slots, int n_sn, int64_t ipool_ints,
                 int64_t arena_doubles);

/* Graph mirror.  Factors are appended; a removal (aprilsam_b200_remove_factors) uploads the compacted records again
 * from its first removed index on. */
int asam_upload_factors(asam_dev_t *d, int first, int count, const int32_t *type, const int32_t *na,
                        const int32_t *nb, const double *z3, const double *W9);
/* Losses of robust xyt factors (type 32): per factor one 16-byte record {loss code as a double, k}
 * (1 Huber, 2 Cauchy).  Only lanes of type-32 factors read it, so other factors may leave theirs unset. */
int asam_upload_loss(asam_dev_t *d, int first, int count, const int32_t *loss, const double *k);
/* which: 0 = l_point, 1 = state */
int asam_upload_points(asam_dev_t *d, int which, int first, int count, const double *p3);
/* copy poses [first, first+count) between the two mirrors inside HBM (which: 0 = l_point, 1 = state) */
int asam_copy_points(asam_dev_t *d, int from, int to, int first, int count);

/* Symbolic plan pieces. */
int asam_upload_node2q(asam_dev_t *d, int first, int count, const int32_t *node2q);
int asam_upload_q2node(asam_dev_t *d, int first, int count, const int32_t *q2node);
int asam_upload_fslot(asam_dev_t *d, int first, int count, const int32_t *fslot);
int asam_upload_ipool(asam_dev_t *d, int64_t first, int64_t count, const int32_t *data);
int asam_upload_desc(asam_dev_t *d, int n, const int32_t *sn_ids, const asam_sn_desc_t *desc);

/* A = 0 (diag = lambda on positions [0, n_lambda)), B = 0 for positions [0, n_nodes) and
 * slots [0, n_slots).  (aprilsam.c:152-153,197-204) */
int asam_hessian_reset(asam_dev_t *d, int n_nodes, int n_slots, int n_lambda, double lambda);
/* Zero a range of newly created positions / slots (incremental growth, no lambda). */
int asam_hessian_clear_range(asam_dev_t *d, int q_first, int q_count, int slot_first, int slot_count);

/* Factor removal (k_hessian_rebuild): OVERWRITE Adiag[9p] and Bq[3p] of the n_pose dirty poses pose[i] with lam[i] on
 * the diagonal plus the blocks of the entries [pose_ptr[i], pose_ptr[i+1]), and Aoff[9s] of the n_slot dirty slots
 * slot[i] with the off-diagonal blocks of the entries [slot_ptr[i], slot_ptr[i+1]) (+0.0 for none).  Entry e is factor
 * ent_f[e] of the HBM mirror, evaluated at ent_pts[6e..6e+6) (pose a, then pose b; a prior uses the first three), with
 * the maths of k_linearize.  Sums run in a fixed order, without atomics: the same tables give the same bits; nothing
 * outside the dirty sets is written.  Tables in host memory, uploaded with the queued uploads; may be recorded between
 * asam_step_begin and asam_step_run. */
int asam_hessian_rebuild(asam_dev_t *d, int n_pose, const int32_t *pose, const int32_t *pose_ptr, int n_slot,
                         const int32_t *slot, const int32_t *slot_ptr, int n_ent, const int32_t *ent_f,
                         const double *ent_pts, const double *lam);

/* Kernel 1: linearise factors [f_first, f_first+f_count) and scatter J'WJ / J'Wr into
 * Adiag/Aoff/Bq (replaces xyt_factor_eval + the assembly loop: april_graph_xyt.c:62-124,
 * april_graph_xytpos.c:63-102, aprilsam.c:154-195 and :508-542).  If pts6 != NULL it holds
 * per-factor evaluation points (a then b, host memory) overriding the lp/st mirrors. */
int asam_linearize(asam_dev_t *d, int f_first, int f_count, const double *pts6);

/* Kernel 2: multifrontal supernodal Cholesky + fused forward solve over the given
 * supernodes (children before parents).  nwait[t]: bits 0-15 = number of children of tasks[t]
 * that are themselves in the task list; bits 16-23 / 24-30 = worker index / team size when a
 * front too large for shared memory is shared by a team of CTAs (the team's entries must be
 * consecutive; 0 or 1 = single CTA).  Replaces cs_schol/cs_chol + forward solve
 * (csparse.c:462-513, smatd.c:1051-1073) and, with a subset, the un-eliminate /
 * re-eliminate of the incremental path (aprilsam.c:791-906). */
int asam_factor(asam_dev_t *d, int ntasks, const int32_t *tasks, const int32_t *nwait, const int32_t *keep);
/* Same, re-using the task list of the previous asam_factor_full upload. */
int asam_set_full_tasks(asam_dev_t *d, int ntasks, const int32_t *tasks, const int32_t *nwait,
                        int nbtasks, const int32_t *btasks);
/* Large graphs: supernodes (children first) whose fronts are at most 48 x 48 and whose whole
 * subtree is of that kind are factored by a warp-per-front kernel launched right before the list
 * above by asam_factor_full.  Call after asam_set_full_tasks; n = 0 disables. */
int asam_set_leaf_tasks(asam_dev_t *d, int n, const int32_t *tasks);
/* Back-substitution: the LAST n entries of the btasks list given to asam_set_full_tasks (a
 * downward-closed set of supernodes with <= 64 own columns and <= 64 rows below, parents first) are
 * solved by a warp-per-supernode kernel right after k_backsolve has done the rest.  n = 0: the whole
 * list goes through k_backsolve.  Call after asam_set_full_tasks. */
int asam_set_bs_leaf_count(asam_dev_t *d, int n);
int asam_factor_full(asam_dev_t *d);
/* Supernodes created after asam_set_full_tasks (poses appended by incremental steps) are
 * ancestors of everything older: prepend them (parents first) to the full back-solve list. */
int asam_btasks_prepend(asam_dev_t *d, int n, const int32_t *ids);

/* ---- several GPUs, one process per GPU (SURVEY.md section 8e) ---------------------------------
 * The communicator is process-wide (a process drives one GPU): rank 0 obtains a 128-byte id with
 * asam_comm_unique_id and ships it to the other ranks by any means (bench.py: torch.distributed),
 * every rank then calls asam_comm_init.  NCCL is loaded with dlopen("libnccl.so.2") -- the copy a
 * host application (PyTorch) already loaded is re-used.  With a communicator in place a batch solve
 * (april_graph_cholesky) may shard the elimination tree: asam_comm_set_sharding(1). */
int asam_comm_unique_id(void *id128_out);
int asam_comm_init(int world, int rank, const void *id128);
void asam_comm_destroy(void);
/* world = 1 without a communicator; *sharding = 1 if batch solves are to be sharded */
int asam_comm_info(int *world, int *rank, int *sharding);
int asam_comm_set_sharding(int enabled);

/* Schedule of a sharded batch solve on this rank.  The lists given to asam_set_full_tasks /
 * asam_set_leaf_tasks then cover this rank's shards only (btasks: top, then own shards, then own
 * leaf set); here come the supernodes above the cut (factored by every rank after the exchange)
 * and what is exchanged: for shard i, owner rank, the arena range holding the trailing columns of
 * its root front (update matrix + rhs row) and its interval of elimination positions (solution
 * segment).  asam_factor_full = own shards -> broadcast of the root fronts -> top;
 * asam_backsolve_full = top + own shards -> broadcast of the solution segments. */
typedef struct asam_shard_sched {
    int32_t n_top, n_top_sn;
    const int32_t *top_tasks, *top_nwait;
    int32_t n_shards;
    const int32_t *shard_owner;
    const int64_t *shard_off, *shard_cnt; /* arena doubles */
    const int32_t *shard_q0, *shard_qn;   /* positions */
} asam_shard_sched_t;
int asam_set_shard_schedule(asam_dev_t *d, const asam_shard_sched_t *sched /* NULL: not sharded */);

/* Kernel 3: back-substitution over the given supernodes (parents before children; the
 * list must be closed under ancestors).  (smatd.c:1075-1097, aprilsam.c:721-779) */
int asam_backsolve(asam_dev_t *d, int ntasks, const int32_t *btasks, const int32_t *bfirst);
int asam_backsolve_full(asam_dev_t *d);

/* Between asam_step_begin and asam_step_run, asam_linearize / asam_hessian_rebuild / asam_factor* / asam_backsolve* only
 * record their launch; asam_step_run pushes every queued upload with one copy and then launches
 * the recorded kernels in order (one incremental step = one H2D transfer). */
int asam_step_begin(asam_dev_t *d);
int asam_step_run(asam_dev_t *d);

/* A small incremental step in one launch (k_step: the queued uploads, linearize, factor and
 * back-solve recorded since asam_step_begin, all in one CTA; results through pinned memory, no
 * stream synchronisation).  x_out receives, in the order of the recorded back-solve list, the
 * 3*cb solution entries of every supernode in it (x_doubles in total).  Returns 0 ok, 2 = the
 * recorded step does not qualify (nothing was launched: call asam_step_run), 1 = error. */
int asam_step_small_supported(asam_dev_t *d);
int asam_step_run_small(asam_dev_t *d, double *x_out, int x_doubles, int *status_out);
int64_t asam_small_steps(asam_dev_t *d);
void asam_small_step_profile(asam_dev_t *d, double *out7, int reset);

/* Solution read-back: x in elimination order, positions [q_first, q_first+q_count). */
int asam_download_x(asam_dev_t *d, int q_first, int q_count, double *x3);
int asam_download_y(asam_dev_t *d, int q_first, int q_count, double *y3);
/* x and the factorisation status (see asam_factor_status) with a single synchronisation. */
int asam_download_x_status(asam_dev_t *d, int q_first, int q_count, double *x3, int *status_out);

/* Marginal covariances from the factor in the arena (Sigma = A^-1 = P' L^-T L^-1 P).  Pose i at elimination
 * position q lies in supernode sn0 at scalar column j0 = 3 (q - first); its three columns Z_i = L^-1 E_q are
 * non-zero only on the supernodes from sn0 to the root, and Sigma_ij = Z_i' Z_j sums over the supernodes the two
 * paths share.  The host (plan_marginal_paths) gives each pose its place in the scratch: entries
 * [hop0, hop0 + nhop) of the hop table and the doubles from zoff on, 3 per scalar row of its path (from j0 in
 * sn0, from 0 above). */
typedef struct asam_marg_path {
    int32_t sn0, j0;
    int32_t hop0, nhop;
    int64_t zoff;
} asam_marg_path_t;
/* One CTA per pose walks its path (k_marginal_path), one CTA per pair i <= j sums the shared part in a fixed
 * order (k_marginal_gram): out (3n x 3n, row-major, host memory) is exactly symmetric, the same from call to call,
 * and block (i, j) does not depend on the other poses of the request.  max_m: the plan's largest front order
 * (sizes shared memory).  Reads the plan, the arena and dinv; writes only its own scratch buffer, allocated at the
 * first call.  One synchronisation. */
int asam_marginal_cov(asam_dev_t *d, int n, const asam_marg_path_t *paths, int64_t z_doubles, int n_hops, int max_m,
                      double *out);
/* One candidate factor of asam_marginal_pairs: an xyt factor between the poses of paths[pa] and paths[pb], or a
 * prior on paths[pa] (pb = -1).  J = [J_a J_b] (3 x 6, row-major) at the l_points, r the residual at the states,
 * Winv the inverse of the factor's information matrix (exactly symmetric); has_w = 0: no W, d2 is NaN. */
typedef struct asam_marg_pair {
    int32_t pa, pb;
    int32_t has_w, pad;
    double J[18];
    double r[3];
    double Winv[9];
} asam_marg_pair_t;
/* k_marginal_path over the n distinct poses, then one CTA per candidate (k_marginal_pairs): the 3 x 3 blocks
 * Sigma_aa, Sigma_ab, Sigma_bb (bit-identical to the blocks of asam_marginal_cov), Sigma_rel = J Sigma_6 J' (Sigma_aa
 * for a prior), S = Sigma_rel + Winv and d2 = r' S^-1 r by a 3 x 3 Cholesky of S (NaN for a non-positive pivot).
 * out: 10 doubles per candidate, {d2, Sigma_rel (row-major, exactly symmetric)}, host memory.  A candidate's
 * output depends only on its own record.  Writes only the scratch buffer; one H2D copy per table and one
 * synchronisation. */
int asam_marginal_pairs(asam_dev_t *d, int n, const asam_marg_path_t *paths, int64_t z_doubles, int n_hops, int max_m,
                        int k, const asam_marg_pair_t *pairs, double *out);

/* One factor of asam_marginal_audit: an xyt factor between the poses of paths[pa] and paths[pb], or a prior on
 * paths[pa] (pb = -1).  J = [J_a J_b] (3 x 6, row-major) at the factor's evaluation point, r the residual at the
 * states, W the information matrix the Hessian holds for it (w W for a robust factor, w at the evaluation point). */
typedef struct asam_marg_audit {
    int32_t pa, pb;
    double J[18];
    double r[3];
    double W[9];
} asam_marg_audit_t;
/* k_marginal_path over the n distinct poses, then one CTA per factor (k_marginal_audit): Sigma_rel as
 * asam_marginal_pairs forms it (bit-identical for the same J and poses), N = W - W Sigma_rel W (exactly symmetric),
 * d2 = (W r)' N^-1 (W r) by a 3 x 3 Cholesky of N (NaN for a non-positive pivot) and redundancy = 3 - tr(Sigma_rel W).
 * out: 11 doubles per factor, {d2, redundancy, Sigma_rel (row-major)}, host memory.  A factor's output depends only on
 * its own record.  Writes only the scratch buffer; one H2D copy per table and one synchronisation. */
int asam_marginal_audit(asam_dev_t *d, int n, const asam_marg_path_t *paths, int64_t z_doubles, int n_hops, int max_m,
                        int k, const asam_marg_audit_t *recs, double *out);
/* One tile of a candidate compatibility query: k_marginal_path over the n distinct poses of the tile, k_marginal_pairs
 * over its nc = jo + nj records (recs[c].pa / pb index paths; has_w = 1), then one CTA per pair slot
 * (k_marginal_compat).  Records [0, ni) are the rows I, [jo, jo + nj) the columns J: jo = 0 is a diagonal tile
 * (nj = ni, J = I, pairs li < lj), jo = ni an off-diagonal one (every slot a pair); ni * nj <= INT32_MAX (one CTA per
 * slot).  ids: the a and b node ids of each record (2 ints), the key of a pair's canonical order.  For a pair (i, j):
 * the cross blocks of Sigma between the candidates' poses by marg_block, C_ij = J_i Sigma J_j' (J = [I 0] of a prior),
 * S = [S_i C_ij; C_ij' S_j] with S_c = Sigma_rel,c + Winv_c as k_marginal_pairs forms it, a 6 x 6 Cholesky of S and
 * d2 = |L^-1 [r_i; r_j]|^2 (NaN for a pivot that is not > 0).  out (host memory): k_marginal_pairs' 10 doubles per
 * record ({d2, Sigma_rel}, as asam_marginal_pairs returns them); cross (host memory): 10 doubles per slot
 * li * nj + lj, {d2, C_ij row-major} (unwritten for li >= lj of a diagonal tile).  A pair's output depends only on its
 * two records.  Writes only the scratch buffer; one H2D copy per table and one synchronisation. */
int asam_marginal_compat(asam_dev_t *d, int n, const asam_marg_path_t *paths, int64_t z_doubles, int n_hops, int max_m,
                         int ni, int nj, int jo, const asam_marg_pair_t *recs, const int *ids, double *out,
                         double *cross);

/* chi2 = sum 0.5 r'Wr (xyt, at state) + sum 0.5 rho(r'Wr) (robust xyt) + sum r'Wr (xytpos) over factors [0, n_factors)
 * using the st mirror (april_graph.c:79-98). Deterministic reduction. */
int asam_chi2(asam_dev_t *d, int n_factors, double *chi2_out);
/* Per factor of [first, first + count) at the st mirror: {r[3], s = r'Wr, w, chi2} (6 doubles, host memory), w the
 * robust weight of a type-32 factor (1 otherwise) and chi2 the exact term asam_chi2 adds for the factor.  One D2H copy
 * and one synchronisation. */
int asam_factor_residuals(asam_dev_t *d, int first, int count, double *out);

/* Status of the last factorisation: 0 ok, >0 = 1 + supernode id with a non-positive (or NaN) pivot,
 * <0 = internal dependency timeout.  A failed pivot turns its ancestors NaN, but they start only after their
 * children have arrived, so with one failure the status names the FIRST failing supernode, never an ancestor;
 * failures in disjoint subtrees report one of them.  A non-zero status, once read, resets the control words,
 * so the context can factor again (tests/test_gpu_pivots.py).  In a sharded solve every rank reads the same word, the
 * owner's: a failure in one rank's shard names that shard's supernode on every rank, and a timeout on any rank is a
 * timeout on every rank (tests/test_gpu_sharded.py). */
int asam_factor_status(asam_dev_t *d, int *status_out);

/* Debug / test access (not used on the solve path). */
int asam_debug_read_hessian(asam_dev_t *d, int n_nodes, int n_slots, double *Adiag9, double *Aoff9, double *Bq3);
int asam_debug_read_front(asam_dev_t *d, int64_t f_off, int64_t count, double *out);
/* bytes [off, off+bytes) of one device mirror of host state: the plan (descriptors, int pool, node2q,
 * q2node, factor slots) or the factor mirror (type, node ids, z, W, {loss, k} records); the reciprocal pivots
 * 1/L_kk (dinv, 3 doubles per pose in elimination order) or the scratch of the last asam_marginal_cov */
enum {
    ASAM_DBG_BUF_SN = 0, ASAM_DBG_BUF_IPOOL, ASAM_DBG_BUF_NODE2Q, ASAM_DBG_BUF_Q2NODE, ASAM_DBG_BUF_FSLOT,
    ASAM_DBG_BUF_FTYPE, ASAM_DBG_BUF_FA, ASAM_DBG_BUF_FB, ASAM_DBG_BUF_FZ, ASAM_DBG_BUF_FW, ASAM_DBG_BUF_FLOSS,
    ASAM_DBG_BUF_DINV, ASAM_DBG_BUF_MARG
};
int asam_debug_read_buffer(asam_dev_t *d, int id, int64_t off, int64_t bytes, void *out);
/* Byte offsets in the scratch of an asam_marginal_cov call with these arguments: {out (3n x 3n doubles), paths,
 * z, hops (4 ints each: supernode, js, c, offset of its rows from the pose's zoff), total}; the error word is at 0. */
void asam_debug_marginal_layout(int n, int64_t z_doubles, int n_hops, int64_t out5[5]);
/* The same for an asam_marginal_pairs call: {out (10 doubles per candidate), paths, z, hops, pairs, total}. */
void asam_debug_marginal_pairs_layout(int n, int64_t z_doubles, int n_hops, int k, int64_t out6[6]);
/* The same for an asam_marginal_audit call: {out (11 doubles per factor), paths, z, hops, records, total}. */
void asam_debug_marginal_audit_layout(int n, int64_t z_doubles, int n_hops, int k, int64_t out6[6]);
/* The same for an asam_marginal_compat tile of nc records and `slots` pair slots: {out (10 doubles per record), cross
 * (10 doubles per slot), paths, z, hops, records, ids, total}. */
void asam_debug_marginal_compat_layout(int n, int64_t z_doubles, int n_hops, int nc, int64_t slots, int64_t out8[8]);
int asam_sync(asam_dev_t *d);
/* Counters: [0] kernel launches since creation, [1] bytes H2D, [2] bytes D2H. */
int asam_counters(asam_dev_t *d, int64_t *out3);
/* Device-side time (ms) of the kernels launched by the last linearize / factor / backsolve
 * calls, measured with CUDA events on the library's stream (0 if timing disabled). */
int asam_set_timing(asam_dev_t *d, int enabled);
/* Per-task globaltimer stamps of the last k_factor (which=0) / k_backsolve (which=1) launch,
 * 8 x uint64 per task in task-list order (diagnostics only). */
int asam_set_trace(asam_dev_t *d, int enabled);
int asam_download_trace(asam_dev_t *d, int which, unsigned long long *out, int max_tasks);
/* Panel-step stamps of ONE team front of k_factor (sn < 0: off): per 48-column panel and worker < 8,
 * 8 x uint64 = iteration start, crew tiles done, block published / rows solved, trailing tiles done,
 * past the team barrier, m, team size, crew size (diagnostics: tools/panel_trace.py). */
int asam_set_panel_trace(asam_dev_t *d, int sn, int max_panels);
int asam_download_panel_trace(asam_dev_t *d, unsigned long long *out, int max_panels);
/* Device stopwatch on the library's stream around any sequence of calls; an L2 flush
 * (384 MiB overwrite) for cold-cache timing; launch geometry of the persistent kernels. */
int asam_timer_start(asam_dev_t *d);
int asam_timer_stop(asam_dev_t *d, float *ms);
int asam_l2_flush(asam_dev_t *d);
int asam_device_info(asam_dev_t *d, int *n_sm, int *fac_grid, int *fac_smem, int *bs_grid);
/* measured FP64 (DFMA) peak of the device in TFLOP/s: the factorisation's compute roofline (bench.py) */
int asam_measure_fp64_peak(asam_dev_t *d, double *tflops_out);
int asam_last_kernel_ms(asam_dev_t *d, float *lin_ms, float *fac_ms, float *bs_ms);

#ifdef __cplusplus
}
#endif
#endif
