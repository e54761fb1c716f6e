// asam_kernels.cuh -- device code of the AprilSAM Gauss-Newton path for sm_90a (H100).
//
//   k_linearize   one thread per factor: residual, Jacobians, J'WJ / J'Wr, atomically
//                 scattered into the block Hessian (Adiag / Aoff / Bq).  Robust xyt factors (type 32)
//                 scale W by their IRLS weight at the residual first.
//                 reference: april_graph_xyt.c:62-124, april_graph_xytpos.c:63-102,
//                            aprilsam.c:154-195 (batch), :508-542 (incremental)
//   k_factor      persistent, dependency-driven multifrontal supernodal Cholesky with the
//                 forward solve fused in (the rhs is carried as an extra ROW of each front).
//                 reference: csparse.c:462-513 (cs_chol), smatd.c:1051-1073, and for a
//                 subset of supernodes aprilsam.c:791-906 (reconstruct + re-eliminate)
//   k_backsolve   persistent, dependency-driven back-substitution L' x = y.
//                 reference: smatd.c:1075-1097, aprilsam.c:721-779
//   k_chi2_*      deterministic reduction of the factor energies at `state`.
//                 reference: april_graph.c:79-98, april_graph_xyt.c:126-188
//
// Front layout (arena[f_off ...], ld*m doubles): column-major, leading dimension
// ld = ASAM_LD(m) = m+1 rounded up to EVEN (every column starts 16-byte aligned: bulk async copies),
// m = 3*mb.  Rows 0..m-1 are the supernode's block rows, ROW m is the right-hand
// side.  After elimination of the first c = 3*cb columns: columns [0,c) hold L (L11 on top of
// L21) and, in row m, y1 = L11^-1 b1; the trailing (m-c) x (m-c) lower triangle holds the
// update matrix (Schur complement) and row m, columns [c,m), the updated rhs b2 - L21 y1 --
// both are scatter-added into the parent's front ("extend-add").
#pragma once

#include <cuda_runtime.h>

#include <cstdint>

#include "asam_cuda.h"
#include "asam_loss.h"

#define ASAM_TR_FLAG (1 << 30)
#define ASAM_MAX_CACHED_CHILDREN 24

// ------------------------------------------------------------------------------------------
// small device helpers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ double d_mod2pi(double v)
{
    // reference: common/math_util.h:113-122 (same constants, same operation order)
    const double twopi = 6.2831853071795862319959;
    const double pi = 3.141592653589793238462643383279502884196;
    double w = v + pi;
    return (w - twopi * floor(w / twopi)) - pi;
}

// C = A' * B for row-major 3x3 (matd_op("M'*M"): transpose then naive triple loop,
// reference common/matd.c:230-254)
__device__ __forceinline__ void d_atb(const double *A, const double *B, double *C)
{
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) {
            double acc = 0.0;
#pragma unroll
            for (int k = 0; k < 3; k++)
                acc += A[k * 3 + i] * B[k * 3 + j];
            C[i * 3 + j] = acc;
        }
}

__device__ __forceinline__ void d_ab(const double *A, const double *B, double *C)
{
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) {
            double acc = 0.0;
#pragma unroll
            for (int k = 0; k < 3; k++)
                acc += A[i * 3 + k] * B[k * 3 + j];
            C[i * 3 + j] = acc;
        }
}

__device__ __forceinline__ void d_av(const double *A, const double *v, double *r)
{
#pragma unroll
    for (int i = 0; i < 3; i++)
        r[i] = A[i * 3 + 0] * v[0] + A[i * 3 + 1] * v[1] + A[i * 3 + 2] * v[2];
}

// Residual + Jacobians of an xyt factor at (pa, pb)   (april_graph_xyt.c:62-124)
__device__ __forceinline__ void d_xyt_eval(const double *pa, const double *pb, const double *z, double *Ja,
                                           double *Jb, double *r)
{
    double ca, sa;
    sincos(pa[2], &sa, &ca);
    double dx = pb[0] - pa[0], dy = pb[1] - pa[1];
    double zh0 = ca * dx + sa * dy;
    double zh1 = -sa * dx + ca * dy;
    double zh2 = pb[2] - pa[2];
    Ja[0] = -ca; Ja[1] = -sa; Ja[2] = -sa * dx + ca * dy;
    Ja[3] = sa;  Ja[4] = -ca; Ja[5] = -ca * dx - sa * dy;
    Ja[6] = 0.0; Ja[7] = 0.0; Ja[8] = -1.0;
    Jb[0] = ca;  Jb[1] = sa;  Jb[2] = 0.0;
    Jb[3] = -sa; Jb[4] = ca;  Jb[5] = 0.0;
    Jb[6] = 0.0; Jb[7] = 0.0; Jb[8] = 1.0;
    r[0] = z[0] - zh0;
    r[1] = z[1] - zh1;
    r[2] = d_mod2pi(z[2] - zh2);
}

// Factor types (aprilsam.h): 1 xyt, 2 xytpos prior, 32 xyt with a robust loss.  Types 1 and 32 have the
// same two poses, Jacobians and residual; the loss only scales W.
__device__ __forceinline__ bool d_two_pose(const int type) { return type == 1 || type == 32; }

// 1/sqrt(a) for the Cholesky pivots: single-precision seed (MUFU.RSQ) + two Newton steps in double (relative
// error 2^-22 -> 2^-43 -> below 2^-53; one to two ulp after rounding).  Three of these are CHAINED in every
// 3x3 pivot block, i.e. they sit on the dependent chain of every panel of every front; the library rsqrt()
// (MUFU.RSQ64H + a longer refinement with range fix-ups) costs about twice as much.  The float seed only exists
// for a in the float range: information matrices carry units and the Tikhonov term may be 0, so a pivot can be
// anywhere in the double range (every W scaled by 2^k scales every pivot by 2^k).  A pivot outside [2^-120, 2^120]
// is brought into range by an even power of two, 4^h, and the result scaled back by 2^-h: both exact, and the
// seed and the Newton steps scale exactly too, so a system scaled by 4^h factors to the same bits scaled.  In-range
// pivots never take that branch; a <= 0, inf and NaN go to rsqrt() (the pivot check flags a <= 0).
__device__ __forceinline__ double d_rsqrt_in_range(const double a)
{
    double y = (double) rsqrtf((float) a);
    double e = fma(-a * y, y, 1.0);
    y = fma(0.5 * y, e, y);
    e = fma(-a * y, y, 1.0);
    y = fma(0.5 * y, e, y);
    return y;
}

__device__ __forceinline__ double d_rsqrt(const double a)
{
    if (!(a >= 0x1p-120 && a <= 0x1p120)) {
        if (!(a > 0.0 && a < INFINITY))
            return rsqrt(a);
        int ex;
        frexp(a, &ex);
        const int h = ex / 2; // a 4^-h has an exponent in {-1, 0, 1}
        return ldexp(d_rsqrt_in_range(ldexp(a, -2 * h)), -h);
    }
    return d_rsqrt_in_range(a);
}

__device__ __forceinline__ int ld_volatile(const int *p) { return *((const volatile int *) p); }

// Flags between the CTAs of a team: release on the writer's side, acquire on the reader's.  A thread that
// publishes for its CTA does so after a barrier, which makes the release cover the writes of every thread
// it synchronised with; a reader polls with plain volatile loads (an acquire load invalidates L1 on every poll),
// acquires once when the value is there and barriers behind that load.  Unlike __threadfence()
// (MEMBAR.SC.GPU + L1 invalidation on sm_90) these do not wait for a sequentially consistent order of all memory
// operations, and they sit on the dependent chain of every panel step.
__device__ __forceinline__ int ld_acquire(const int *p)
{
    int v;
    asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(int *p, const int v)
{
    asm volatile("st.release.gpu.global.b32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void red_release_add(int *p, const int v)
{
    asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

__device__ __forceinline__ unsigned long long d_now()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// Bounded spin: every wait on a counter/flag written by another CTA gives up after `limit_ns` of WALL
// time (globaltimer, sampled every 1024 polls), flags the error word and lets the launch drain -- a
// dependency bug must not hang the GPU, and a legitimately long factorisation (the root waits for the
// whole tree) must not be cut short by a poll count.
struct SpinClock {
    long long n = 0;
    unsigned long long t0 = 0;
};
__device__ __forceinline__ bool spin_over(SpinClock &c, long long limit_ns)
{
    if ((++c.n & 1023) != 0)
        return false;
    const unsigned long long now = d_now();
    if (c.t0 == 0) {
        c.t0 = now;
        return false;
    }
    return (long long) (now - c.t0) > limit_ns;
}

// k_linearize aggregates the per-node contributions inside the warp before touching HBM: lanes
// whose destination node matches (__match_any_sync) are summed with shuffles and only the lowest
// such lane issues the atomics.  Factors are listed by (max node id, min node id), so the closures
// of one pose sit in neighbouring lanes and would otherwise serialise on the same L2 address.

// ------------------------------------------------------------------------------------------
// kernel 1: linearise + scatter
// ------------------------------------------------------------------------------------------
struct LinArgs {
    const int *f_type, *f_a, *f_b, *f_slot;
    const double *f_z, *f_W;
    const double2 *f_loss; // {loss, k} per factor; read by robust factors (type 32) only
    const double *lp, *st;
    const double *pts; // optional, indexed from f_first
    const int *node2q;
    double *Adiag, *Aoff, *Bq;
    int f_first, f_count;
};

// one factor per lane; every lane of a warp must call this together (warp-wide match / shuffles)
__device__ __forceinline__ void linearize_body(const LinArgs &a, const int t)
{
    const bool live = t < a.f_count;
    const int f = a.f_first + (live ? t : 0);
    const int type = live ? a.f_type[f] : 0;
    const int na = live ? a.f_a[f] : -1;
    const int nb = (live && d_two_pose(type)) ? a.f_b[f] : -1;
    double z[3], W[9];
#pragma unroll
    for (int i = 0; i < 3; i++)
        z[i] = live ? a.f_z[3 * (size_t) f + i] : 0.0;
#pragma unroll
    for (int i = 0; i < 9; i++)
        W[i] = live ? a.f_W[9 * (size_t) f + i] : 0.0;

    // per-node contributions: packed upper triangle of the 3x3 block (6) + rhs (3)
    double ca9[9], cb9[9], H[9];
    bool has_off = false;
    if (live && type == 2) { // xytpos: J = I, r = z - state   (april_graph_xytpos.c:63-102)
        const double *src = a.pts ? (a.pts + 6 * (size_t) t) : (a.st + 3 * (size_t) na);
        const double r[3] = { z[0] - src[0], z[1] - src[1], d_mod2pi(z[2] - src[2]) };
        // J'W = W ; (J'W) J = W ; keep scalar row <= col  (aprilsam.c:171-172)
        ca9[0] = W[0]; ca9[1] = W[1]; ca9[2] = W[2]; ca9[3] = W[4]; ca9[4] = W[5]; ca9[5] = W[8];
        d_av(W, r, ca9 + 6);
    } else if (live) { // xyt factor (type 1 or 32)
        const int qa = a.node2q[na], qb = a.node2q[nb];
        double pa[3], pb[3];
        if (a.pts) {
            const double *src = a.pts + 6 * (size_t) t;
#pragma unroll
            for (int i = 0; i < 3; i++) { pa[i] = src[i]; pb[i] = src[3 + i]; }
        } else {
#pragma unroll
            for (int i = 0; i < 3; i++) { pa[i] = a.lp[3 * (size_t) na + i]; pb[i] = a.lp[3 * (size_t) nb + i]; }
        }
        double Ja[9], Jb[9], r[3], JatW[9], JbtW[9], D[9];
        d_xyt_eval(pa, pb, z, Ja, Jb, r);
        if (type == 32) { // robust: IRLS weight at r, W_eff = w W (no second-order term: stays PSD)
            const double2 lk = a.f_loss[f];
            double X[3];
            d_av(W, r, X);
            const double w = asam_loss_weight((int) lk.x, lk.y, r[0] * X[0] + r[1] * X[1] + r[2] * X[2]);
#pragma unroll
            for (int i = 0; i < 9; i++)
                W[i] *= w;
        }
        d_atb(Ja, W, JatW); // J_a' W
        d_atb(Jb, W, JbtW); // J_b' W
        // diagonal blocks: entries with scalar row <= col only (aprilsam.c:171-172)
        d_ab(JatW, Ja, D);
        ca9[0] = D[0]; ca9[1] = D[1]; ca9[2] = D[2]; ca9[3] = D[4]; ca9[4] = D[5]; ca9[5] = D[8];
        d_av(JatW, r, ca9 + 6);
        d_ab(JbtW, Jb, D);
        cb9[0] = D[0]; cb9[1] = D[1]; cb9[2] = D[2]; cb9[3] = D[4]; cb9[4] = D[5]; cb9[5] = D[8];
        d_av(JbtW, r, cb9 + 6);
        // off-diagonal block: the reference keeps (J_early' W J_late) where "early" is the node
        // eliminated first; the mirrored block is dropped (matters for non-symmetric W).
        if (qa < qb)
            d_ab(JatW, Jb, H);
        else
            d_ab(JbtW, Ja, H);
        const int early = qa < qb ? na : nb;
        if (early != (na < nb ? na : nb)) { // slot layout is S[lower node id][higher node id]
            double tsw;
            tsw = H[1]; H[1] = H[3]; H[3] = tsw;
            tsw = H[2]; H[2] = H[6]; H[6] = tsw;
            tsw = H[5]; H[5] = H[7]; H[7] = tsw;
        }
        has_off = true;
    }

    // scatter: diag block entries (r<=c) at offsets {0,1,2,4,5,8} of Adiag[9*node], rhs at Bq[3*node]
    {
        const bool act = live;
        double tmp[9];
#pragma unroll
        for (int i = 0; i < 9; i++)
            tmp[i] = live ? ca9[i] : 0.0;
        // aggregate the 9 values per destination node, then the leader writes to the two arrays
        const unsigned lane = threadIdx.x & 31;
        const unsigned m1 = __ballot_sync(0xffffffffu, act);
        if (act) {
            const unsigned peers = __match_any_sync(m1, na);
            const int leader = __ffs(peers) - 1;
            for (unsigned rem = peers & ~(1u << leader); rem; rem &= rem - 1) {
                const int src = __ffs(rem) - 1;
#pragma unroll
                for (int i = 0; i < 9; i++)
                    tmp[i] += __shfl_sync(peers, ca9[i], src);
            }
            if ((int) lane == leader) {
                double *Ad = a.Adiag + 9 * (size_t) na;
                atomicAdd(Ad + 0, tmp[0]); atomicAdd(Ad + 1, tmp[1]); atomicAdd(Ad + 2, tmp[2]);
                atomicAdd(Ad + 4, tmp[3]); atomicAdd(Ad + 5, tmp[4]); atomicAdd(Ad + 8, tmp[5]);
                double *Bn = a.Bq + 3 * (size_t) na;
                atomicAdd(Bn + 0, tmp[6]); atomicAdd(Bn + 1, tmp[7]); atomicAdd(Bn + 2, tmp[8]);
            }
        }
    }
    {
        const bool act = has_off;
        const unsigned lane = threadIdx.x & 31;
        const unsigned m1 = __ballot_sync(0xffffffffu, act);
        if (act) {
            double tmp[9];
#pragma unroll
            for (int i = 0; i < 9; i++)
                tmp[i] = cb9[i];
            const unsigned peers = __match_any_sync(m1, nb);
            const int leader = __ffs(peers) - 1;
            for (unsigned rem = peers & ~(1u << leader); rem; rem &= rem - 1) {
                const int src = __ffs(rem) - 1;
#pragma unroll
                for (int i = 0; i < 9; i++)
                    tmp[i] += __shfl_sync(peers, cb9[i], src);
            }
            if ((int) lane == leader) {
                double *Ad = a.Adiag + 9 * (size_t) nb;
                atomicAdd(Ad + 0, tmp[0]); atomicAdd(Ad + 1, tmp[1]); atomicAdd(Ad + 2, tmp[2]);
                atomicAdd(Ad + 4, tmp[3]); atomicAdd(Ad + 5, tmp[4]); atomicAdd(Ad + 8, tmp[5]);
                double *Bn = a.Bq + 3 * (size_t) nb;
                atomicAdd(Bn + 0, tmp[6]); atomicAdd(Bn + 1, tmp[7]); atomicAdd(Bn + 2, tmp[8]);
            }
            // off-diagonal slots are (almost always) unique per factor: plain atomics
            double *S = a.Aoff + 9 * (size_t) a.f_slot[f];
#pragma unroll
            for (int i = 0; i < 9; i++)
                atomicAdd(S + i, H[i]);
        }
    }
}

__global__ void __launch_bounds__(128) k_linearize(LinArgs a)
{
    linearize_body(a, blockIdx.x * blockDim.x + threadIdx.x);
}

__global__ void k_hessian_reset(double *Adiag, double *Aoff, double *Bq, int n_nodes, int n_slots, int n_lambda,
                                double lambda)
{
    size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    size_t nd = 9 * (size_t) n_nodes, no = 9 * (size_t) n_slots, nb = 3 * (size_t) n_nodes;
    if (i < nd) {
        int e = (int) (i % 9);
        int q = (int) (i / 9);
        Adiag[i] = ((e == 0 || e == 4 || e == 8) && q < n_lambda) ? lambda : 0.0;
    } else if (i < nd + no) {
        Aoff[i - nd] = 0.0;
    } else if (i < nd + no + nb) {
        Bq[i - nd - no] = 0.0;
    }
}

// ------------------------------------------------------------------------------------------
// factor removal: the touched Hessian entries recomputed from the factors that remain
// ------------------------------------------------------------------------------------------
struct RebuildArgs {
    const int *f_type, *f_a, *f_b;
    const double *f_z, *f_W;
    const double2 *f_loss;  // read by robust factors (type 32) only
    const int *node2q;
    const int *pose, *pose_ptr; // dirty pose i: incidence entries [pose_ptr[i], pose_ptr[i+1])
    const int *slot, *slot_ptr; // dirty slot i: entries [slot_ptr[i], slot_ptr[i+1])
    const int *ent_f;           // factor of each entry
    const double *ent_pts;      // 6 doubles per entry: evaluation points of pose a, then b (priors: a only)
    const double *lam;          // per dirty pose: the Tikhonov term on its diagonal
    double *Adiag, *Aoff, *Bq;
    int n_pose, n_slot;
};

// One factor at its evaluation points, with the maths of linearize_body: ca9 / cb9 = the upper triangle (r <= c) of
// J_a'WJ_a / J_b'WJ_b packed in 6 + J'Wr (3), H = the off-diagonal block, "early" pose first, stored
// [lower node id][higher node id].  A prior fills ca9 only.
__device__ __forceinline__ void rebuild_factor(const RebuildArgs &a, const int f, const double *pts, double *ca9,
                                               double *cb9, double *H)
{
    const int type = a.f_type[f];
    double z[3], W[9];
#pragma unroll
    for (int i = 0; i < 3; i++)
        z[i] = a.f_z[3 * (size_t) f + i];
#pragma unroll
    for (int i = 0; i < 9; i++)
        W[i] = a.f_W[9 * (size_t) f + i];
    if (type == 2) {
        const double r[3] = { z[0] - pts[0], z[1] - pts[1], d_mod2pi(z[2] - pts[2]) };
        ca9[0] = W[0]; ca9[1] = W[1]; ca9[2] = W[2]; ca9[3] = W[4]; ca9[4] = W[5]; ca9[5] = W[8];
        d_av(W, r, ca9 + 6);
        return;
    }
    const int na = a.f_a[f], nb = a.f_b[f];
    double Ja[9], Jb[9], r[3], JatW[9], JbtW[9], D[9];
    d_xyt_eval(pts, pts + 3, z, Ja, Jb, r);
    if (type == 32) {
        const double2 lk = a.f_loss[f];
        double X[3];
        d_av(W, r, X);
        const double w = asam_loss_weight((int) lk.x, lk.y, r[0] * X[0] + r[1] * X[1] + r[2] * X[2]);
#pragma unroll
        for (int i = 0; i < 9; i++)
            W[i] *= w;
    }
    d_atb(Ja, W, JatW);
    d_atb(Jb, W, JbtW);
    d_ab(JatW, Ja, D);
    ca9[0] = D[0]; ca9[1] = D[1]; ca9[2] = D[2]; ca9[3] = D[4]; ca9[4] = D[5]; ca9[5] = D[8];
    d_av(JatW, r, ca9 + 6);
    d_ab(JbtW, Jb, D);
    cb9[0] = D[0]; cb9[1] = D[1]; cb9[2] = D[2]; cb9[3] = D[4]; cb9[4] = D[5]; cb9[5] = D[8];
    d_av(JbtW, r, cb9 + 6);
    const int qa = a.node2q[na], qb = a.node2q[nb];
    if (qa < qb)
        d_ab(JatW, Jb, H);
    else
        d_ab(JbtW, Ja, H);
    const int early = qa < qb ? na : nb;
    if (early != (na < nb ? na : nb)) {
        double tsw;
        tsw = H[1]; H[1] = H[3]; H[3] = tsw;
        tsw = H[2]; H[2] = H[6]; H[6] = tsw;
        tsw = H[5]; H[5] = H[7]; H[7] = tsw;
    }
}

// One warp per dirty pose: its lanes take the pose's entries in turn, each lane sums its share in list order, a fixed
// butterfly adds the 32 partial sums, and lane 0 OVERWRITES Adiag (lambda + the sum on r <= c, 0 below) and Bq.  Then one
// thread per dirty slot overwrites Aoff with its entries' blocks summed in list order (+0.0 for none).  No atomics: the
// same lists give the same bits on every call; entries outside the lists are not touched.
__global__ void __launch_bounds__(128) k_hessian_rebuild(RebuildArgs a)
{
    const int gt = blockIdx.x * blockDim.x + threadIdx.x;
    const int w = gt >> 5, lane = gt & 31;
    double ca9[9], cb9[9], H[9];
    if (w < a.n_pose) {
        const int p = a.pose[w];
        double acc[9];
#pragma unroll
        for (int i = 0; i < 9; i++)
            acc[i] = 0.0;
        for (int e = a.pose_ptr[w] + lane; e < a.pose_ptr[w + 1]; e += 32) {
            const int f = a.ent_f[e];
            rebuild_factor(a, f, a.ent_pts + 6 * (size_t) e, ca9, cb9, H);
            const bool is_b = a.f_type[f] != 2 && a.f_a[f] != p;
#pragma unroll
            for (int i = 0; i < 9; i++)
                acc[i] += is_b ? cb9[i] : ca9[i];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
#pragma unroll
            for (int i = 0; i < 9; i++)
                acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], o);
        if (lane == 0) {
            const double l = a.lam[w];
            double *Ad = a.Adiag + 9 * (size_t) p;
            Ad[0] = l + acc[0]; Ad[1] = acc[1]; Ad[2] = acc[2];
            Ad[3] = 0.0; Ad[4] = l + acc[3]; Ad[5] = acc[4];
            Ad[6] = 0.0; Ad[7] = 0.0; Ad[8] = l + acc[5];
            double *Bn = a.Bq + 3 * (size_t) p;
            Bn[0] = acc[6]; Bn[1] = acc[7]; Bn[2] = acc[8];
        }
        return;
    }
    const int si = (w - a.n_pose) * 32 + lane;
    if (si >= a.n_slot)
        return;
    double S[9];
#pragma unroll
    for (int i = 0; i < 9; i++)
        S[i] = 0.0;
    for (int e = a.slot_ptr[si]; e < a.slot_ptr[si + 1]; e++) {
        rebuild_factor(a, a.ent_f[e], a.ent_pts + 6 * (size_t) e, ca9, cb9, H);
#pragma unroll
        for (int i = 0; i < 9; i++)
            S[i] += H[i];
    }
    double *Ao = a.Aoff + 9 * (size_t) a.slot[si];
#pragma unroll
    for (int i = 0; i < 9; i++)
        Ao[i] = S[i];
}

// ------------------------------------------------------------------------------------------
// kernel 2: persistent multifrontal factorisation (+ fused forward solve)
// ------------------------------------------------------------------------------------------
struct FacArgs {
    const asam_sn_desc_t *sn;
    const int *ipool;
    double *arena;
    const double *Adiag, *Aoff, *Bq;
    const int *q2node;
    double *y;
    double *dinv; // 1/L_kk in elimination order (used by k_backsolve)
    int *arrive;
    int *tbar; // team barrier counters, zeroed before the launch
    const int *tasks, *nwait; // nwait: bits 0-15 children in this launch, 16-23 worker, 24-30 team size
    const int *keep; // optional, per task: (poses kept << 16) | block rows of the retained front; see cta_front
    int ntasks;
    int *ctrl; // [0] ticket, [1] err
    int smem_doubles;
    long long spin_limit;
    unsigned long long *trace; // optional: 8 words per task
    int pb_smem;   // panel width of shared-memory fronts (multiple of 3)
    int smem_mma;  // shared-memory fronts on the FP64 tensor pipe: 1 = the one wide update of kept columns (incremental
                   // steps), 2 = also the 12-column panel updates, 0 = DFMA only
    int solo_pb; // widest staged panel of a front that one CTA handles out of HBM (multiple of ASAM_PB)
    unsigned long long *ptrace; // optional: panel-step stamps of supernode ptrace_sn, [panel][worker < 8][8]
    int ptrace_sn, ptrace_panels;
};

// Trailing update  C[i,j] -= sum_{p<pb} P[i,p] * P[j,p]  for j in [j0, m), i in [j, m]
// (row m = rhs row).  P holds the pb factored panel columns (leading dim ldp, row index =
// front row); C is the front (leading dim ld).  One warp per tile of TN columns, each lane R
// rows spaced 32 apart: conflict-free shared-memory reads for the row values, broadcast reads
// for the column values; R*TN accumulators per lane keep the FP64 pipe, not the shared-memory
// pipe, the limiter (2R + TN wavefronts feed R*TN warp-wide DFMAs per panel column).
// Out-of-range rows/columns are clamped for the loads and masked at the store.
template <int R, int TN>
__device__ __forceinline__ void trailing_update(double *C, int ld, const double *P, int ldp, int pb, int j0, int jend, int m,
                                                const int sub_warps = 0)
{
    // columns [j0, jend) (jend <= m), rows [j, m]; sub_warps > 0: only that many warps take part
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = sub_warps ? sub_warps : (blockDim.x >> 5);
    for (int tj = j0 + TN * warp; tj < jend; tj += TN * nwarps) {
        int jc[TN];
#pragma unroll
        for (int q = 0; q < TN; q++)
            jc[q] = min(tj + q, jend - 1);
        for (int ib = tj; ib <= m; ib += 32 * R) {
            double acc[R][TN];
            int irow[R], ic[R];
#pragma unroll
            for (int r = 0; r < R; r++) {
                irow[r] = ib + lane + 32 * r;
                ic[r] = min(irow[r], m);
#pragma unroll
                for (int q = 0; q < TN; q++)
                    acc[r][q] = 0.0;
            }
#pragma unroll 2
            for (int p = 0; p < pb; p++) {
                const double *pc = P + (size_t) p * ldp;
                double b[TN], av[R];
#pragma unroll
                for (int q = 0; q < TN; q++)
                    b[q] = pc[jc[q]];
#pragma unroll
                for (int r = 0; r < R; r++)
                    av[r] = pc[ic[r]];
#pragma unroll
                for (int r = 0; r < R; r++)
#pragma unroll
                    for (int q = 0; q < TN; q++)
                        acc[r][q] += av[r] * b[q];
            }
#pragma unroll
            for (int r = 0; r < R; r++)
#pragma unroll
                for (int q = 0; q < TN; q++) {
                    const int i = irow[r], j = tj + q;
                    if (i <= m && j < jend && i >= j)
                        C[i + (size_t) j * ld] -= acc[r][q];
                }
        }
    }
}

// D(8x8) += A(8x4, row) * B(4x8, col) on the FP64 tensor pipe.  Fragments: lane = 4*g + t holds A[g][t], B[t][g],
// D[g][2t], D[g][2t+1].
__device__ __forceinline__ void dmma_8x8x4(double &c0, double &c1, const double a, const double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

// The same trailing update on the FP64 tensor pipe, for fronts and panels in SHARED memory (any pb >= 1: the
// k dimension is padded with zeros in the fragments).  Work items are (8-column block, 32-row block) pairs of the
// lower trapezoid, dealt round-robin to the warps; per 4 panel columns 4 + 1 fragment loads feed 4 tensor
// instructions of 256 multiply-adds (trailing_update<2,8>: 10 loads per 512).  Rows beyond m and columns beyond
// jend are masked in the loads (no out-of-range reads) and at the store.
__device__ __forceinline__ void trailing_update_mma(double *C, const int ld, const double *P, const int ldp, const int pb,
                                                    const int j0, const int jend, const int m, const int sub_warps = 0)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = sub_warps ? sub_warps : (blockDim.x >> 5);
    const int g = lane >> 2, t = lane & 3;
    int pair = 0;
    for (int jb = j0; jb < jend; jb += 8) {
        for (int ib = jb; ib <= m; ib += 32, ++pair) {
            if (pair % nwarps != warp)
                continue;
            double acc[4][2];
#pragma unroll
            for (int mt = 0; mt < 4; mt++)
                acc[mt][0] = acc[mt][1] = 0.0;
            const bool jok = jb + g < jend;
            for (int kk = 0; kk < pb; kk += 4) {
                const bool kok = kk + t < pb;
                const size_t koff = (size_t) (kk + t) * ldp;
                const double bv = (kok && jok) ? P[(jb + g) + koff] : 0.0;
#pragma unroll
                for (int mt = 0; mt < 4; mt++) {
                    const int row = ib + 8 * mt + g;
                    const double av = (kok && row <= m) ? -P[row + koff] : 0.0;
                    dmma_8x8x4(acc[mt][0], acc[mt][1], av, bv);
                }
            }
#pragma unroll
            for (int mt = 0; mt < 4; mt++)
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const int i = ib + 8 * mt + g, j = jb + 2 * t + e;
                    if (i <= m && j < jend && i >= j)
                        C[i + (size_t) j * ld] += acc[mt][e];
                }
        }
    }
}

#define ASAM_PB 12 // panel width of the dense partial Cholesky (a multiple of 3)

// Dense partial Cholesky of one panel of pb (multiple of 3, <= ASAM_PB) columns [k0, k0+pb) of
// the front held in P (panel column p at P + p*ldp, indexed by front row; rows k0..m valid,
// row m = rhs).  Every pose contributes a 3x3 block column, so the panel is processed in
// 3-column steps with a CLOSED-FORM 3x3 Cholesky that every thread evaluates redundantly in
// registers (three chained reciprocal square roots, no warp/block hand-off), followed by the
// row TRSM (each thread owns rows) and the rank-3 update of the remaining panel columns.
// Two block barriers per 3 columns; the code stays small (this kernel executes straight-line
// code once per task, so instruction-cache footprint matters more than unrolling).
// sub_nt > 0: only the first sub_nt threads of the CTA take part (they synchronise on named barrier 1; the
// others must not call): a 48 x 48 block has work for two warps, and a barrier of two warps is far cheaper than one
// of eight -- there are 9 of them per 12 columns on the dependent chain of every panel.
__device__ __forceinline__ void bar_sub(const int nthreads) { asm volatile("bar.sync 1, %0;" ::"r"(nthreads) : "memory"); }

// (tuning switches live in CONSTANT memory: a __device__ global read inside panel_factor is a global load on the
// dependent chain of every 3x3 step)
__constant__ int g_pf_groups = 1; // ASAM_PF_GROUPS=0: one thread per row in the in-panel update of panel_factor (A/B)
__constant__ int g_dmap_ahead = 1; // ASAM_DMAP_AHEAD=0: destination maps child by child inside the extend-add loop (A/B)

__device__ __forceinline__ void panel_factor(double *P, int ldp, int k0, int pb, int m, int sn_id, int *err,
                                             double *dinv_out, const int sub_nt = 0)
{
    const int tid = threadIdx.x, nt = sub_nt ? sub_nt : blockDim.x;
#define PF_SYNC()            \
    do {                     \
        if (sub_nt)          \
            bar_sub(sub_nt); \
        else                 \
            __syncthreads(); \
    } while (0)
    for (int c0 = 0; c0 < pb; c0 += 3) {
        const int rb = k0 + c0; // front row of this 3x3 diagonal block
        double *p0 = P + (size_t) c0 * ldp, *p1 = p0 + ldp, *p2 = p1 + ldp;
        PF_SYNC(); // previous in-panel update (or trailing update) is complete
        const double a00 = p0[rb], a10 = p0[rb + 1], a20 = p0[rb + 2];
        const double a11 = p1[rb + 1], a21 = p1[rb + 2], a22 = p2[rb + 2];
        const double r0 = d_rsqrt(a00);
        const double l10 = a10 * r0, l20 = a20 * r0;
        const double d1 = a11 - l10 * l10;
        const double r1 = d_rsqrt(d1);
        const double l21 = (a21 - l20 * l10) * r1;
        const double d2 = a22 - l20 * l20 - l21 * l21;
        const double r2 = d_rsqrt(d2);
        if (tid == 0 && !(a00 > 0.0 && d1 > 0.0 && d2 > 0.0))
            atomicCAS(err, 0, 1 + sn_id);
        // rows below the block: x = row * L11^-T  (the thread keeps x for the update below)
        const int i_first = rb + 3 + tid;
        for (int i = i_first; i <= m; i += nt) {
            const double x0 = p0[i] * r0;
            const double x1 = (p1[i] - x0 * l10) * r1;
            const double x2 = (p2[i] - x0 * l20 - x1 * l21) * r2;
            p0[i] = x0;
            p1[i] = x1;
            p2[i] = x2;
        }
        PF_SYNC(); // every thread has read the diagonal block; L rows are visible
        if (tid == 0) {
            p0[rb] = a00 * r0; p0[rb + 1] = l10; p0[rb + 2] = l20;
            p1[rb + 1] = d1 * r1; p1[rb + 2] = l21;
            p2[rb + 2] = d2 * r2;
            if (dinv_out) {
                dinv_out[rb] = r0; dinv_out[rb + 1] = r1; dinv_out[rb + 2] = r2;
            }
        }
        // rank-3 update of the remaining panel columns jc in (c0+2, pb): rows i >= k0 + jc
        const int nrem = pb - (c0 + 3);
        const int nrow = m - (rb + 3) + 1; // rows below the 3x3 block (the rhs row included)
        if (nrem > 0 && nrow > 0) {
            // fewer rows than threads (diagonal blocks of team fronts, small fronts): the spare threads share the
            // columns of a row -- thread = (row, column group) -- instead of one thread walking all <= 9 of them
            int ng = g_pf_groups ? nt / nrow : 1;
            ng = ng > nrem ? nrem : ng;
            if (ng > 1) {
                const int gi = tid / nrow, ri = tid - gi * nrow;
                if (gi < ng) {
                    const int i = rb + 3 + ri;
                    const double x0 = p0[i], x1 = p1[i], x2 = p2[i];
                    const int jmax = min(nrem, ri + 1);
                    for (int jj = gi; jj < jmax; jj += ng) {
                        const int jr = rb + 3 + jj;
                        double *pj = P + (size_t) (c0 + 3 + jj) * ldp;
                        pj[i] -= x0 * p0[jr] + x1 * p1[jr] + x2 * p2[jr];
                    }
                }
            } else {
                for (int i = i_first; i <= m; i += nt) {
                    const double x0 = p0[i], x1 = p1[i], x2 = p2[i];
                    const int jmax = min(nrem, i - (rb + 3) + 1); // columns whose diagonal row <= i
                    for (int jj = 0; jj < jmax; jj++) {
                        const int jr = rb + 3 + jj; // front row (= column) of panel column c0+3+jj
                        double *pj = P + (size_t) (c0 + 3 + jj) * ldp;
                        pj[i] -= x0 * p0[jr] + x1 * p1[jr] + x2 * p2[jr];
                    }
                }
            }
        }
    }
    PF_SYNC();
#undef PF_SYNC
}

// ------------------------------------------------------------------------------------------
// Big fronts: a TEAM of G CTAs (consecutive tickets of the same supernode) factors one front that
// does not fit in shared memory.  The front stays in HBM/L2; phases are separated by a team
// barrier on a per-supernode counter (tbar; the last worker to leave a front zeroes it again):
//   every worker: wait for the children, zero + assemble + extend-add its OWN columns -> [barrier]
//   -> panel 0 by everybody -> [barrier] -> per panel k of <= ASAM_TPB columns: { a crew factors panel
//   k+1: worker 0 factors its diagonal block and publishes L11 in 12-column stages behind a release flag,
//   the other crew workers solve their row chunks stage by stage; the rest of the team applies panel k
//   to the trailing matrix in tiles, operands from the row-major panel workspace } -> [barrier]
// (DESIGN §4 has the details.)  Column / chunk / tile ownership is a fixed function of (worker, team
// size): deterministic.
// All reads of front data written by other workers bypass L1 (ld.global.cg).
// A supernode of this kind may be arbitrarily wide (host: fundamental chains of team-sized
// fronts are merged without a cap), e.g. the 1383-column root separator of the 100 k graph.
// ------------------------------------------------------------------------------------------
#define ASAM_TPB 48   // panel width of the team path
#define ASAM_TROWS 256
#define ASAM_TCOLS 64

#define ASAM_CROWS 128 // rows of one look-ahead crew item (row chunk of the next panel)

// ---- mbarrier / bulk asynchronous copy (TMA engine, 1-D) --------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned) __cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}

__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity)
{
    unsigned ok;
    long long tries = 0;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok)
                     : "r"(smem_u32(bar)), "r"(parity)
                     : "memory");
        if (!ok && ++tries > (1LL << 24)) // a copy that never completes must not hang the GPU: fail the launch loudly
            __trap();
    } while (!ok);
}

// global -> shared, `bytes` (multiple of 16) from a 16-byte aligned source to a 16-byte aligned
// destination; completion is counted on `bar` (complete_tx)
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, unsigned bytes, unsigned long long *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// Row-major PANEL WORKSPACE of a team front.  Behind the front (arena[f_off + ld*m ...]) sit two
// buffers of (m+2) rows x ASAM_LDW doubles; buffer k&1 holds the factored panel k by ROWS: row r of the front
// at W[r * ASAM_LDW .. + pb), zero up to the next multiple of 4.  A tile's operands -- a chunk of rows of the
// panel -- are then ONE contiguous block each: two bulk asynchronous copies per tile instead of one per panel
// column (96 small copies cost as much as staging by hand).  ASAM_LDW = 4 (mod 16) keeps the
// m8n8k4 fragment loads conflict free, and a row is 416 bytes: every row 16-byte aligned.
#define ASAM_LDW 52
#define ASAM_WS_DOUBLES(m) (2 * (size_t) ((m) + 2) * ASAM_LDW)

// C[rb0.., cb0..] -= L[rb0.., panel] * L[cb0.., panel]' with the panel taken from its row-major workspace Wk.
// out_mode 0: C is read from and written back to the front (trailing update); 1: C is read from the front and
// written to Out[ii + jj * ASAM_TPB] (the next panel's diagonal block, factored in diag_publish); 2: C is read from
// the front and written to Out[ii + jj * ASAM_TROWS] (rows of the next panel, solved in place by trsm_row_block; Out
// may alias Li).  FP64 tensor pipe (mma.sync.m8n8k4.f64): warp w owns the 8*MT-row strip w of the tile and all of
// its (at most 8) 8-column blocks; per 4 panel columns MT + 8 shared-memory fragment loads feed MT*8 tensor
// instructions.  The C values are fetched before the products and written after them.
template <int MT>
__device__ __noinline__ void tile_rm(double *F, const int ld, const double *Wk, const int pb4, const int cb0, const int ncol,
                                     const int rb0, const int nrow, const int out_mode, double *Out, double *Li, double *Lj,
                                     unsigned long long *bar, unsigned &parity)
{
    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const bool same = rb0 == cb0 && nrow >= ncol; // diagonal block: one operand
    __syncthreads(); // everybody is done with the previous contents of Li / Lj
    if (warp == 0) {
        asm volatile("fence.proxy.async;" ::: "memory");
        if (lane == 0) {
            const unsigned bi = (unsigned) nrow * ASAM_LDW * 8u, bj = same ? 0u : (unsigned) ncol * ASAM_LDW * 8u;
            mbar_expect_tx(bar, bi + bj);
            bulk_g2s(Li, Wk + (size_t) rb0 * ASAM_LDW, bi, bar);
            if (!same)
                bulk_g2s(Lj, Wk + (size_t) cb0 * ASAM_LDW, bj, bar);
        }
    }
    const double *Ljs = same ? Li : Lj;
    const int g = lane >> 2, t = lane & 3;
    const int r0 = warp * 8 * MT;
    const int nnt = (ncol + 7) >> 3;
    const int rowmax = rb0 + min(r0 + 8 * MT, nrow) - 1;
    const int nneed = (r0 < nrow && rowmax >= cb0) ? min(nnt, ((rowmax - cb0) >> 3) + 1) : 0;
    double acc[MT][8][2];
#pragma unroll
    for (int mt = 0; mt < MT; mt++)
#pragma unroll
        for (int q = 0; q < 8; q++)
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const int ii = r0 + 8 * mt + g, jj = 8 * q + 2 * t + e;
                const bool ok = q < nneed && ii < nrow && jj < ncol && rb0 + ii >= cb0 + jj;
                acc[mt][q][e] = ok ? __ldcg(&F[(rb0 + ii) + (size_t) (cb0 + jj) * ld]) : 0.0;
            }
    mbar_wait(bar, parity);
    parity ^= 1u;
    if (nneed > 0) {
        const double *ai = Li + (size_t) (r0 + g) * ASAM_LDW + t;
        const double *bj_ = Ljs + (size_t) g * ASAM_LDW + t;
#pragma unroll 2
        for (int kk = 0; kk < pb4; kk += 4) {
            double av[MT];
#pragma unroll
            for (int mt = 0; mt < MT; mt++)
                av[mt] = -ai[(size_t) (8 * mt) * ASAM_LDW + kk];
#pragma unroll
            for (int q = 0; q < 8; q++) {
                if (q < nneed) {
                    const double bv = bj_[(size_t) (8 * q) * ASAM_LDW + kk];
#pragma unroll
                    for (int mt = 0; mt < MT; mt++)
                        dmma_8x8x4(acc[mt][q][0], acc[mt][q][1], av[mt], bv);
                }
            }
        }
    }
    if (out_mode == 2)
        __syncthreads(); // Out may alias Li: every warp is done with its operand
    if (nneed > 0) {
#pragma unroll
        for (int mt = 0; mt < MT; mt++)
#pragma unroll
            for (int q = 0; q < 8; q++)
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const int ii = r0 + 8 * mt + g, jj = 8 * q + 2 * t + e;
                    if (q < nneed && ii < nrow && jj < ncol && rb0 + ii >= cb0 + jj) {
                        if (out_mode == 0)
                            F[(rb0 + ii) + (size_t) (cb0 + jj) * ld] = acc[mt][q][e];
                        else if (out_mode == 1)
                            Out[ii + jj * ASAM_TPB] = acc[mt][q][e];
                        else
                            Out[ii + jj * ASAM_TROWS] = acc[mt][q][e];
                    }
                }
    }
}

struct TeamCtx {
    int *tbar_s;
    int G, w, phase;
    long long spin_limit;
    int *err;
    int sn;
};

__device__ __forceinline__ bool team_barrier(TeamCtx &tc, int *s_flag)
{
    __syncthreads();
    if (threadIdx.x == 0) {
        red_release_add(tc.tbar_s, 1);
        const int target = (++tc.phase) * tc.G;
        SpinClock spins;
        int ok = 1;
        while (ld_volatile(tc.tbar_s) < target) {
            __nanosleep(20);
            if (spin_over(spins, tc.spin_limit) || ld_volatile(tc.err) < 0) {
                atomicCAS(tc.err, 0, -(1 + tc.sn));
                ok = 0;
                break;
            }
        }
        ld_acquire(tc.tbar_s);
        *s_flag = ok;
    } else {
        tc.phase++;
    }
    __syncthreads();
    return *s_flag != 0;
}

// Leaving a front: the counter stands at phase*G; every worker adds one more and the last one
// to do so zeroes it for the next launch (no host-side reset between launches).
__device__ __forceinline__ void team_leave(TeamCtx &tc)
{
    if (threadIdx.x == 0) {
        const int v = atomicAdd(tc.tbar_s, 1);
        if (v == tc.phase * tc.G + tc.G - 1)
            atomicExch(tc.tbar_s, 0);
    }
}

__device__ __forceinline__ bool team_owns(int col, int w, int G) { return ((col >> 2) % G) == w; }

// Cholesky of the pb x pb diagonal block held in shared memory (column-major, leading dimension ASAM_TPB),
// right-looking and blocked: 12-column sub-panels of closed-form 3x3 steps (panel_factor: every thread of the CTA
// takes part in the row solves and the in-panel rank-3 updates) followed by an update of the rest of the block on
// the FP64 tensor pipe -- no dot products of growing length on the dependent chain.  rdv[k] = 1 / L_kk.
// Ends with a CTA-wide barrier.
__device__ __forceinline__ void diag_factor_rl(double *D, int pb, double *rdv, int sn_id, int *err)
{
    constexpr int LDD = ASAM_TPB;
    constexpr int SUB = 256; // (64 = two warps on a named barrier was measured slower, see diag_publish)
    if (threadIdx.x < SUB) {
        for (int k1 = 0; k1 < pb; k1 += ASAM_PB) {
            const int pbb = min(ASAM_PB, pb - k1);
            panel_factor(D + (size_t) k1 * LDD, LDD, k1, pbb, pb - 1, sn_id, err, rdv, SUB);
            if (k1 + pbb < pb) {
                trailing_update_mma(D, LDD, D + (size_t) k1 * LDD, LDD, pbb, k1 + pbb, pb, pb - 1, SUB / 32);
                bar_sub(SUB);
            }
        }
    }
    __syncthreads();
}

// One row of the panel per thread: x = row * L11^-T.  The row lives in Li (column p at
// Li[tid + p*ASAM_TROWS]); it is processed 12 columns at a time in registers -- first the
// contributions of the columns already solved (L entries fetched two at a time, broadcast), then
// the 12x12 triangle fully unrolled.  Results go back to Li, to the front in HBM and to the row-major panel
// workspace (Wrow[0..pb), zero up to the next multiple of 4), where the next iteration's tiles fetch it as part of
// one contiguous block.
// one 12-column block [b0, b0+nb) of the row solve (needs x of the columns before b0 in Li and rows b0.. of the
// columns [0, b0+nb) of L11 in D)
__device__ __forceinline__ void trsm_row_block(double *Li, const double *D, const double *rdv, const int b0, const int nb,
                                               double *Frow, int ld, double *Wrow)
{
    const int tid = threadIdx.x;
    constexpr int LDD = ASAM_TPB;
    double r[12];
#pragma unroll
    for (int q = 0; q < 12; q++)
        r[q] = (q < nb) ? Li[tid + (b0 + q) * ASAM_TROWS] : 0.0;
    for (int p = 0; p < b0; p++) {
        const double xp = Li[tid + p * ASAM_TROWS];
        const double2 *Dp = reinterpret_cast<const double2 *>(D + p * LDD + b0);
#pragma unroll
        for (int q2 = 0; q2 < 6; q2++) {
            const double2 v = Dp[q2];
            r[2 * q2] -= xp * v.x;
            r[2 * q2 + 1] -= xp * v.y;
        }
    }
#pragma unroll
    for (int q = 0; q < 12; q++) {
        if (q < nb) {
            r[q] *= rdv[b0 + q];
#pragma unroll
            for (int q2 = q + 1; q2 < 12; q2++)
                r[q2] -= r[q] * D[(b0 + q2) + (b0 + q) * LDD];
        }
    }
#pragma unroll
    for (int q = 0; q < 12; q++)
        if (q < nb) {
            Li[tid + (b0 + q) * ASAM_TROWS] = r[q];
            Frow[(size_t) (b0 + q) * ld] = r[q];
            Wrow[b0 + q] = r[q];
        }
}

__device__ __forceinline__ void trsm_row(double *Li, const double *D, const double *rdv, int pb, double *Frow, int ld,
                                         double *Wrow)
{
    for (int b0 = 0; b0 < pb; b0 += 12)
        trsm_row_block(Li, D, rdv, b0, min(12, pb - b0), Frow, ld, Wrow);
    for (int q = pb; q < ((pb + 3) & ~3); q++)
        Wrow[q] = 0.0;
}

// returns false on abort
__device__ bool team_front(const FacArgs &a, const asam_sn_desc_t &d, int s, int nw, int w, int G, double *sm,
                           int *s_flag, unsigned long long *trow, unsigned long long *mbar, unsigned &mb_parity)
{
    // trow (worker 0, thread 0 only): [1] children ready, [2] assembled, [3] extend-added,
    // [4] eliminated; [7] high word: ns spent in the panel (diag + TRSM) phases
    const int tid = threadIdx.x, nt = blockDim.x;
    const int lane = tid & 31, warp = tid >> 5, nwarps = nt >> 5;
    const int m = 3 * d.mb, c = 3 * d.cb, ld = ASAM_LD(m);
    const int *seg = a.ipool + d.seg;
    const int *children = seg + 2 * d.mb;
    const int *a_slot = children + d.ch_cnt;
    const int *a_rb = a_slot + d.a_cnt;
    const int *a_cb = a_rb + d.a_cnt;
    double *F = a.arena + d.f_off;
    int *err = a.ctrl + 1;
    TeamCtx tc;
    tc.tbar_s = a.tbar + 2 * (size_t) s; // [2s] team barrier, [2s+1] crew barrier of the look-ahead
    tc.G = G;
    tc.w = w;
    tc.phase = 0;
    tc.spin_limit = a.spin_limit;
    tc.err = err;
    tc.sn = s;

    // ---- zero + assemble own columns ---------------------------------------------------------
    for (int j = warp; j < m; j += nwarps) {
        if (!team_owns(j, w, G))
            continue;
        for (int i = j + lane; i <= m; i += 32)
            F[i + (size_t) j * ld] = 0.0;
    }
    __syncthreads();
    for (int e = tid; e < d.cb * 9; e += nt) {
        int k = e / 9, p = (e % 9) / 3, q = e % 3;
        if (p >= q && team_owns(3 * k + q, w, G))
            F[(3 * k + p) + (size_t) (3 * k + q) * ld] = a.Adiag[9 * (size_t) a.q2node[d.first + k] + q * 3 + p];
    }
    for (int e = tid; e < c; e += nt)
        if (team_owns(e, w, G))
            F[m + (size_t) e * ld] = a.Bq[3 * (size_t) a.q2node[d.first + e / 3] + e % 3];
    for (int e = tid; e < d.a_cnt * 9; e += nt) {
        int i = e / 9, p = (e % 9) / 3, q = e % 3;
        const int col = 3 * a_cb[i] + q;
        if (!team_owns(col, w, G))
            continue;
        const int rbf = a_rb[i];
        const int rb = rbf & ~ASAM_TR_FLAG;
        const int si = (rbf & ASAM_TR_FLAG) ? (p * 3 + q) : (q * 3 + p);
        F[(3 * rb + p) + (size_t) col * ld] = a.Aoff[9 * (size_t) a_slot[i] + si];
    }
    // every worker waits for the children re-factored in this launch (the counter is zeroed by
    // worker 0 after the first team barrier, when nobody looks at it any more)
    if (nw > 0 && tid == 0) {
        SpinClock spins;
        int ok = 1;
        while (ld_volatile(&a.arrive[s]) < nw) {
            __nanosleep(20);
            if (spin_over(spins, a.spin_limit) || ld_volatile(err) < 0) {
                atomicCAS(err, 0, -(1 + s));
                ok = 0;
                break;
            }
        }
        __threadfence();
        *s_flag = ok;
    } else if (tid == 0) {
        *s_flag = 1;
    }
    __syncthreads();
    if (!*s_flag)
        return false;
    if (trow && tid == 0)
        trow[1] = trow[2] = d_now();

    // ---- extend-add into own columns -------------------------------------------------------
    int *dmap = (int *) sm; // ld ints
    for (int ci = 0; ci < d.ch_cnt; ++ci) {
        const asam_sn_desc_t cd = a.sn[children[ci]];
        const int cm = 3 * cd.mb, cc = 3 * cd.cb, cr = cm - cc, cld = ASAM_LD(cm);
        const double *CF = a.arena + cd.f_off;
        const int *crel = a.ipool + cd.seg + cd.mb;
        __syncthreads();
        for (int i = tid; i <= cr; i += nt)
            dmap[i] = (i < cr) ? 3 * crel[(cc + i) / 3] + (cc + i) % 3 : m;
        __syncthreads();
        for (int j = warp; j < cr; j += nwarps) {
            const int dj = dmap[j];
            if (!team_owns(dj, w, G))
                continue;
            const double *ccol = CF + (size_t) (cc + j) * cld + cc;
            double *fcol = F + (size_t) dj * ld;
            // the column is this worker's own and dmap is injective: the destination values are fetched
            // together with the child's (16 independent loads in flight per lane, one L2 round trip per
            // 256 rows) instead of one read-modify-write after the other
            for (int i0 = j + lane; i0 <= cr; i0 += 256) {
                double v[8], dv[8];
                int di[8];
#pragma unroll
                for (int u = 0; u < 8; u++) {
                    const bool ok = i0 + 32 * u <= cr;
                    v[u] = ok ? __ldcg(ccol + i0 + 32 * u) : 0.0;
                    di[u] = ok ? dmap[i0 + 32 * u] : -1;
                }
#pragma unroll
                for (int u = 0; u < 8; u++)
                    dv[u] = di[u] >= 0 ? __ldcg(fcol + di[u]) : 0.0;
#pragma unroll
                for (int u = 0; u < 8; u++)
                    if (di[u] >= 0)
                        fcol[di[u]] = dv[u] + v[u];
            }
        }
    }
    if (!team_barrier(tc, s_flag))
        return false;
    if (w == 0 && nw > 0 && tid == 0)
        a.arrive[s] = 0;
    unsigned long long t_panel = 0, t_mark = 0;
    if (trow && tid == 0)
        trow[3] = d_now();

    // ---- panels, with one panel of look-ahead ---------------------------------------------------
    // Panel k+1 is factored by a small CREW while the other workers are still applying panel k to
    // the rest of the trailing matrix.  In iteration k
    //   crew worker 0:   applies panel k to the 48x48 diagonal block of panel k+1, factors it (once)
    //                    and publishes L11 / 1/diag in 12-column stages, each behind a release flag
    //   crew worker w>0: applies panel k to its 128-row chunk of panel k+1's columns, keeps the rows in
    //                    shared memory and solves them stage by stage as the stages are published
    //   everybody else:  tiles of the trailing update with panel k right of panel k+1
    //   -> [team barrier]
    // so the dependent chain per panel is max(chunk update, block update + factorisation) + row solve
    // + one barrier, instead of factorisation + barrier + a whole trailing update + barrier.
    double *D = sm;                              // ASAM_TPB x ASAM_TPB diagonal block
    double *rdv = D + ASAM_TPB * ASAM_TPB;       // ASAM_TPB reciprocal diagonal entries
    // tile operands by rows from the panel workspace behind the front (Li: <= 256 x ASAM_LDW, Lj: <= 64 x ASAM_LDW);
    // Li also holds the rows being solved (column p at Li[tid + p * ASAM_TROWS])
    double *Li = rdv + ASAM_TPB;
    double *Lj = Li + ASAM_TROWS * ASAM_LDW;
    double *Wbase = F + (size_t) ld * m;
    auto Wbuf = [&](int panel_index) { return Wbase + (size_t) (panel_index & 1) * (m + 2) * ASAM_LDW; };
    double *dinv = a.dinv + 3 * (size_t) d.first;
    int *crew_bar = a.tbar + 2 * (size_t) s + 1; // flag: 8 * seq + the stages of the diagonal block published

    // C[rb0.., cb0..] -= L[rb0.., k0..k0+pb) * L[cb0.., k0..k0+pb)'  (lower trapezoid only), operands from the
    // row-major workspace of the panel at k0.  Dout != nullptr: the tile is the diagonal block of the next panel;
    // its values go straight into the shared-memory block that diag_publish factors, not back to the front
    auto tile = [&](int k0, int pb, int cb0, int ncol, int rb0, int nrow, double *Dout) {
        const double *Wk = Wbuf(k0 / ASAM_TPB);
        const int pb4 = (pb + 3) & ~3;
        if (Dout)
            tile_rm<1>(F, ld, Wk, pb4, cb0, ncol, rb0, nrow, 1, Dout, Li, Lj, mbar, mb_parity);
        else if (nrow <= 128)
            tile_rm<2>(F, ld, Wk, pb4, cb0, ncol, rb0, nrow, 0, nullptr, Li, Lj, mbar, mb_parity);
        else
            tile_rm<4>(F, ld, Wk, pb4, cb0, ncol, rb0, nrow, 0, nullptr, Li, Lj, mbar, mb_parity);
    };
    // diagonal block of the panel at k0 into D (every caller redundantly), the caller's row chunk
    // [rb0, rb0+256) below the block into Li while the block is being factored, then the rows
    auto panel = [&](int k0, int pb, int rb0) {
        __syncthreads();
        for (int e = tid; e < ASAM_TPB * ASAM_TPB; e += nt) {
            const int i = e % ASAM_TPB, j = e / ASAM_TPB;
            D[e] = (i >= j && i < pb && j < pb) ? __ldcg(&F[(k0 + i) + (size_t) (k0 + j) * ld]) : 0.0;
        }
        const int i = rb0 + tid;
        const bool row = rb0 >= 0 && i >= k0 + pb && i <= m;
        if (row)
            for (int j = 0; j < pb; j++)
                Li[tid + j * ASAM_TROWS] = __ldcg(&F[i + (size_t) (k0 + j) * ld]);
        __syncthreads();
        diag_factor_rl(D, pb, rdv, s, err);
        if (row)
            trsm_row(Li, D, rdv, pb, F + i + (size_t) k0 * ld, ld, Wbuf(0) + (size_t) i * ASAM_LDW);
    };
    auto writeback = [&](int k0, int pb) { // worker 0, after a team barrier: nobody reads the raw block any more
        for (int e = tid; e < pb * pb; e += nt) {
            const int i = e % pb, j = e / pb;
            if (i >= j)
                F[(k0 + i) + (size_t) (k0 + j) * ld] = D[i + j * ASAM_TPB];
        }
        for (int e = tid; e < pb; e += nt)
            dinv[k0 + e] = rdv[e];
    };

    // worker 0 of the crew: the diagonal block of the panel at k0 (already updated by its own tile) is factored
    // ONCE, blocked right-looking, and PUBLISHED IN STAGES: after each 12-column sub-panel its columns of L11 are
    // final and go to the front + 1/diag to dinv + the flag (8 * seq + stage); the crew solves the matching 12
    // columns of its rows while the next sub-panel is being factored, instead of starting when all 48 are done
    auto diag_publish = [&](int k0, int pb, int seq) {
        __syncthreads(); // D was zeroed before, and filled by, the tile that updated this block
        constexpr int LDD = ASAM_TPB;
        constexpr int SUB = 256; // threads that factor the block (one warp in registers, and 64 threads on a two-warp
                                 // barrier, were SLOWER: the publish / update loops want the threads more than the
                                 // barriers cost)
        int stage = 0;
        for (int k1 = 0; k1 < pb; k1 += ASAM_PB) {
            const int pbb = min(ASAM_PB, pb - k1);
            panel_factor(D + (size_t) k1 * LDD, LDD, k1, pbb, pb - 1, s, err, rdv, SUB);
            ++stage;
            for (int e = tid; e < pbb * pb; e += SUB) {
                const int j = k1 + e / pb, i = e % pb;
                if (i >= j)
                    F[(k0 + i) + (size_t) (k0 + j) * ld] = D[i + j * LDD];
            }
            for (int e = tid; e < pbb; e += SUB)
                dinv[k0 + k1 + e] = rdv[k1 + e];
            bar_sub(SUB);
            if (tid == 0)
                st_release(crew_bar, 8 * seq + stage);
            if (k1 + pbb < pb) {
                trailing_update_mma(D, LDD, D + (size_t) k1 * LDD, LDD, pbb, k1 + pbb, pb, pb - 1, SUB / 32);
                bar_sub(SUB);
            }
        }
        __syncthreads();
    };
    // the crew's rows (already updated, in Li) are solved 12 columns at a time, each stage as soon as worker 0 has
    // published the matching columns of L11
    auto rows_solve_staged = [&](int k0, int pb, int rb0, int seq, double *Wnext) {
        constexpr int LDD = ASAM_TPB;
        // Two groups of four warps.  LOADERS (warps 4-7): wait for the flag of stage s, fetch its 12 columns of L11
        // (one L2 round trip) into D and hand them over on named barrier 3 + s (they only arrive).  SOLVERS (warps
        // 0-3, one row each): pick the columns up and solve.  The loaders are already polling for stage s + 1 while
        // the solvers work on s: a stage costs the crew max(poll + fetch, solve) instead of their sum -- before,
        // a stage took longer than the block took to publish it, the row chunks finished well after the last
        // publish and the whole team waited for them.
        if (tid == 0)
            *s_flag = 1;
        __syncthreads();
        const int i = rb0 + tid;
        const bool row = tid < ASAM_CROWS && i <= m;
        int stage = 0;
        for (int b0 = 0; b0 < pb; b0 += ASAM_PB, ++stage) {
            const int nb = min(ASAM_PB, pb - b0);
            if (warp >= 4) {
                if (tid == 128 && *s_flag) {
                    SpinClock spins;
                    while (ld_volatile(crew_bar) < 8 * seq + stage + 1) {
                        __nanosleep(20);
                        if (spin_over(spins, a.spin_limit) || ld_volatile(err) < 0) {
                            atomicCAS(err, 0, -(1 + s));
                            *s_flag = 0;
                            break;
                        }
                    }
                    ld_acquire(crew_bar);
                }
                asm volatile("bar.sync 2, 128;" ::: "memory");
                if (*s_flag) {
                    for (int e = tid - 128; e < nb * ASAM_TPB; e += 128) {
                        const int j = b0 + e / ASAM_TPB, ii = e % ASAM_TPB;
                        D[ii + j * LDD] = (ii >= j && ii < pb) ? __ldcg(&F[(k0 + ii) + (size_t) (k0 + j) * ld]) : 0.0;
                    }
                    if (tid - 128 < nb)
                        rdv[b0 + tid - 128] = __ldcg(&dinv[k0 + b0 + tid - 128]);
                }
                __threadfence_block();
                asm volatile("bar.arrive %0, 256;" ::"r"(3 + stage) : "memory");
            } else {
                asm volatile("bar.sync %0, 256;" ::"r"(3 + stage) : "memory");
                if (row && *s_flag)
                    trsm_row_block(Li, D, rdv, b0, nb, F + i + (size_t) k0 * ld, ld, Wnext + (size_t) i * ASAM_LDW);
            }
        }
        if (row && *s_flag)
            for (int q = pb; q < ((pb + 3) & ~3); q++)
                Wnext[(size_t) i * ASAM_LDW + q] = 0.0;
        __syncthreads();
        return *s_flag != 0;
    };
    // prologue: panel 0 by everybody (row chunks of 256 from the panel's first row, round-robin)
    {
        const int pb = min(ASAM_TPB, c);
        if (trow && tid == 0)
            t_mark = d_now();
        const int nchunk = (m + 1 + ASAM_TROWS - 1) / ASAM_TROWS;
        bool first = true;
        for (int ch = w; ch < nchunk || first; ch += G) {
            panel(0, pb, ch < nchunk ? ch * ASAM_TROWS : -1);
            first = false;
        }
        if (!team_barrier(tc, s_flag))
            return false;
        if (trow && tid == 0)
            t_panel += d_now() - t_mark;
        if (w == 0)
            writeback(0, pb);
    }
    int seq = 0;
    const bool pt_on = a.ptrace && s == a.ptrace_sn && w < 8 && tid == 0;
    for (int k0 = 0; k0 < c; k0 += ASAM_TPB) {
        // panel trace (diagnostics): [0] iteration start, [1] own crew tiles done, [2] block factored and
        // published (w 0) / flag seen and rows solved (w > 0), [3] own trailing tiles done, [4] past the barrier
        unsigned long long *pt = (pt_on && k0 / ASAM_TPB < a.ptrace_panels) ? a.ptrace + ((size_t) (k0 / ASAM_TPB) * 8 + w) * 8 : nullptr;
        if (pt) {
            pt[0] = d_now();
            pt[1] = pt[2] = pt[3] = pt[0];
            pt[5] = (unsigned long long) m;
            pt[6] = (unsigned long long) G;
        }
        const int pb = min(ASAM_TPB, c - k0);
        const int kn0 = k0 + pb;                       // first trailing column = next panel
        const bool has_next = kn0 < c;
        const int pbn = has_next ? min(ASAM_TPB, c - kn0) : 0;
        // crew of the next panel: worker 0 owns its diagonal block, workers 1.. the 256-row chunks below
        const int ncrew = has_next ? 1 + (m - (kn0 + pbn) + 1 + ASAM_CROWS - 1) / ASAM_CROWS : 0;
        ++seq;
        if (w < ncrew) {
            // crew items: 0 = the diagonal block, i >= 1 = row chunk i-1; dealt round-robin (a team
            // scaled down by the host may be smaller than the crew), the block first
            if (trow && tid == 0)
                t_mark = d_now();
            if (w == 0) {
                __syncthreads(); // worker 0 has written the previous panel's block back
                for (int e = tid; e < ASAM_TPB * ASAM_TPB; e += nt)
                    D[e] = 0.0;
                tile(k0, pb, kn0, pbn, kn0, pbn, D);
                if (pt)
                    pt[1] = d_now();
                diag_publish(kn0, pbn, seq);
                if (pt)
                    pt[2] = d_now();
            }
            // fused crew item: the updated rows go from the tensor-pipe accumulators straight into shared
            // memory (no round trip through the front), are solved there against the published L11 and
            // leave once -- to the front (final L) and to the next panel's row-major workspace
            for (int it = (w == 0 ? G : w); it < ncrew; it += G) {
                const int rb0 = kn0 + pbn + (it - 1) * ASAM_CROWS;
                tile_rm<2>(F, ld, Wbuf(k0 / ASAM_TPB), (pb + 3) & ~3, kn0, pbn, rb0, min(ASAM_CROWS, m - rb0 + 1), 2, Li, Li,
                           Lj, mbar, mb_parity);
                if (pt && w > 0 && it == w)
                    pt[1] = d_now();
                if (!rows_solve_staged(kn0, pbn, rb0, seq, Wbuf(kn0 / ASAM_TPB)))
                    return false;
            }
            if (pt && w > 0)
                pt[2] = d_now();
            if (trow && tid == 0)
                t_panel += d_now() - t_mark;
        }

        // trailing update with panel k right of the next panel: tiles of TR rows x 64 columns over
        // the lower trapezoid (TR = 128 when 256-row tiles would leave workers idle).  The crew is
        // on the critical path already: the tiles go to the other workers only, unless the team is
        // all crew
        const int j0 = kn0 + pbn;
        const int nfree = (G - ncrew >= 2) ? G - ncrew : G, wfree = (G - ncrew >= 2) ? w - ncrew : w;
        int n256 = 0;
        for (int cb0 = j0; cb0 < m; cb0 += ASAM_TCOLS)
            n256 += (m - cb0 + 1 + 255) / 256;
        const int TR = (n256 < 2 * nfree) ? 128 : 256;
        if (wfree >= 0) {
            int u = 0;
            for (int cb0 = j0; cb0 < m; cb0 += ASAM_TCOLS)
                for (int rb0 = cb0; rb0 <= m; rb0 += TR, ++u)
                    if (u % nfree == wfree)
                        tile(k0, pb, cb0, min(ASAM_TCOLS, m - cb0), rb0, min(TR, m - rb0 + 1), nullptr);
        }
        if (pt)
            pt[3] = d_now();
        if (!team_barrier(tc, s_flag))
            return false;
        if (pt) {
            pt[4] = d_now();
            pt[7] = (unsigned long long) ncrew;
        }
    }
    if (w == 0 && tid == 0)
        atomicExch(crew_bar, 0); // everybody is past its last wait on the crew flag (team barrier above)

    if (trow && tid == 0) {
        trow[4] = d_now();
        trow[7] = (unsigned long long) (unsigned) m | (t_panel << 32);
    }
    // ---- publish ------------------------------------------------------------------------------------
    if (w == 0) {
        for (int e = tid; e < c; e += nt)
            a.y[3 * (size_t) d.first + e] = __ldcg(&F[m + (size_t) e * ld]);
        __syncthreads();
        if (tid == 0 && d.parent >= 0) {
            __threadfence();
            atomicAdd(&a.arrive[d.parent], 1);
        }
    }
    team_leave(tc);
    __syncthreads();
    return true;
}

// Persistent kernels take tickets from a counter in a.ctrl; the last CTA to leave zeroes the
// counter again, so back-to-back launches need no host-side reset (err stays 0 unless fatal).
__device__ __forceinline__ void ticket_release(int *ticket, int *done)
{
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(done, 1) == (int) gridDim.x - 1) {
            atomicExch(ticket, 0);
            atomicExch(done, 0);
        }
    }
}

// ncol columns of 2*nr2 doubles from src (leading dim lds) to dst (leading dim ldd), both 16-byte aligned, in
// 16-byte accesses with eight of them in flight per thread (a panel of a front in HBM to or from shared memory).
__device__ __forceinline__ void solo_copy(double *dst, const int ldd, const double *src, const int lds, const int nr2,
                                          const int ncol)
{
    const int n = nr2 * ncol, nt = blockDim.x;
    for (int e0 = threadIdx.x; e0 < n; e0 += 8 * nt) {
        double2 v[8];
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const int e = e0 + u * nt, p = e / nr2, r = e - p * nr2;
            if (e < n)
                v[u] = *(const double2 *) (src + 2 * r + (size_t) p * lds);
        }
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const int e = e0 + u * nt, p = e / nr2, r = e - p * nr2;
            if (e < n)
                *(double2 *) (dst + 2 * r + (size_t) p * ldd) = v[u];
        }
    }
}

// Trailing update of a front in HBM by one CTA:  F[i,j] -= sum_{p<pb} P[i,p] * P[j,p]  for j in [j0, m), i in [j, m]
// (row m = rhs).  P is the staged panel in shared memory (column p at P + p*ldp, indexed by front row, ldp = 4
// (mod 16)).  Tiles of 32 rows x 8 columns of the lower trapezoid on the FP64 tensor pipe, dealt to the warps
// round-robin with no barrier between them.  A warp issues the L2 loads of its NEXT tile's C before the products
// of the current one, so their latency hides behind the tensor instructions.
__device__ __forceinline__ void solo_tile_next(int &jb, int &ib, const int m, int n)
{
    for (; n > 0 && jb < m; --n) {
        ib += 32;
        if (ib > m) {
            jb += 8;
            ib = jb;
        }
    }
}

__device__ __noinline__ void solo_update(double *F, const int ld, const double *P, const int ldp, const int pb,
                                         const int j0, const int m)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int g = lane >> 2, t = lane & 3;
    auto load_c = [&](const int jb, const int ib, double (&v)[4][2]) {
#pragma unroll
        for (int mt = 0; mt < 4; mt++)
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const int i = ib + 8 * mt + g, j = jb + 2 * t + e;
                v[mt][e] = (jb < m && i <= m && j < m && i >= j) ? F[i + (size_t) j * ld] : 0.0;
            }
    };
    int jb = j0, ib = j0;
    solo_tile_next(jb, ib, m, warp);
    double cv[4][2];
    load_c(jb, ib, cv);
    while (jb < m) {
        int jn = jb, in = ib;
        solo_tile_next(jn, in, m, nwarps);
        double cn[4][2];
        load_c(jn, in, cn);
        double acc[4][2];
#pragma unroll
        for (int mt = 0; mt < 4; mt++)
            acc[mt][0] = acc[mt][1] = 0.0;
        const bool jok = jb + g < m;
        for (int kk = 0; kk < pb; kk += 4) {
            const bool kok = kk + t < pb;
            const size_t koff = (size_t) (kk + t) * ldp;
            const double bv = (kok && jok) ? P[(jb + g) + koff] : 0.0;
#pragma unroll
            for (int mt = 0; mt < 4; mt++) {
                const int row = ib + 8 * mt + g;
                const double av = (kok && row <= m) ? -P[row + koff] : 0.0;
                dmma_8x8x4(acc[mt][0], acc[mt][1], av, bv);
            }
        }
#pragma unroll
        for (int mt = 0; mt < 4; mt++)
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const int i = ib + 8 * mt + g, j = jb + 2 * t + e;
                if (i <= m && j < m && i >= j)
                    F[i + (size_t) j * ld] = cv[mt][e] + acc[mt][e];
                cv[mt][e] = cn[mt][e];
            }
        jb = jn;
        ib = in;
    }
}

// One front handled by ONE CTA (the front in shared memory when it fits, else in HBM with staged
// panels): zero + gather the Hessian entries, wait for the children of this launch, extend-add the
// children's update matrices, eliminate the supernode's columns, publish.  t = index in the task
// list (trace slot).  Returns false on abort.
// Partial re-factorisation (incremental steps, keepw != 0): the first `keep` columns of the front are
// unchanged by the step (host: plan_append), their L and y are still in the arena (front of order 3*old_mb at
// the same offset).  The front is assembled as usual, those columns are overwritten with the retained L, applied
// to the rest in ONE parallel pass, and only the columns from `keep` on go through the sequential elimination.
__device__ bool cta_front(const FacArgs &a, const int t, const int s, const int nw, const asam_sn_desc_t &d, double *sm,
                          asam_sn_desc_t *s_cd, int *s_abort, unsigned long long tr0, const int keepw = 0)
{
    const int tid = threadIdx.x, nt = blockDim.x;
    const int lane = tid & 31, warp = tid >> 5, nwarps = nt >> 5;
    int *err = a.ctrl + 1;
    unsigned long long tr1 = 0, tr2 = 0, tr3 = 0, tr4 = 0, accA = 0, accB = 0;
    const int m = 3 * d.mb, c = 3 * d.cb, ld = ASAM_LD(m);
    const int *seg = a.ipool + d.seg;
    const int *children = seg + 2 * d.mb;
    const int *a_slot = children + d.ch_cnt;
    const int *a_rb = a_slot + d.a_cnt;
    const int *a_cb = a_rb + d.a_cnt;
    double *Fg = a.arena + d.f_off;
    // shared-memory budget: front + destination map (ld ints) when the front fits
    const long long fsz = (long long) ld * m;
    const bool use_sm = fsz + (ld + 1) / 2 + 2 <= (long long) a.smem_doubles;
    double *F = use_sm ? sm : Fg;
    int *dmap = (int *) (sm + (use_sm ? fsz : 0)); // ld ints
    const int pboff = ((ld + 1) / 2 + 2) & ~1;      // HBM mode: the staged panel behind dmap, 16-byte aligned
    double *dinv = a.dinv + 3 * (size_t) d.first;   // 1/L_kk of this supernode's columns

    // ---- 1. zero the lower trapezoid (+ rhs row), gather the original entries ---------
    if (use_sm) {
        for (int i = tid; i < (int) fsz; i += nt)
            F[i] = 0.0;
    } else {
        for (int j = warp; j < m; j += nwarps)
            for (int i = j + lane; i <= m; i += 32)
                F[i + (size_t) j * ld] = 0.0;
    }
    for (int e = tid; e < d.ch_cnt && e < ASAM_MAX_CACHED_CHILDREN; e += nt)
        s_cd[e] = a.sn[children[e]];
    __syncthreads();
    // Destination maps of ALL children now (they are plan data, not results): their loads share the round trip of
    // the Hessian gather below and overlap the wait for the children, instead of costing every child one L2
    // round trip of its own on the dependent chain.  Needs room behind the front for sum(rows + 1) ints.
    __shared__ int s_doff[ASAM_MAX_CACHED_CHILDREN + 1];
    bool dmap_ahead = false;
    if (use_sm && g_dmap_ahead && d.ch_cnt > 0 && d.ch_cnt <= ASAM_MAX_CACHED_CHILDREN) {
        if (tid == 0) {
            int o = 0;
            for (int e = 0; e < d.ch_cnt; e++) {
                s_doff[e] = o;
                o += 3 * (s_cd[e].mb - s_cd[e].cb) + 1;
            }
            s_doff[d.ch_cnt] = o;
        }
        __syncthreads();
        dmap_ahead = (long long) s_doff[d.ch_cnt] <= 2 * ((long long) a.smem_doubles - fsz) - 2;
        if (dmap_ahead)
            for (int ci = 0; ci < d.ch_cnt; ++ci) {
                const int cc = 3 * s_cd[ci].cb, cr = 3 * s_cd[ci].mb - cc;
                const int *crel = a.ipool + s_cd[ci].seg + s_cd[ci].mb;
                int *dm = dmap + s_doff[ci];
                for (int i = tid; i <= cr; i += nt)
                    dm[i] = (i < cr) ? 3 * crel[(cc + i) / 3] + (cc + i) % 3 : m;
            }
    }
    for (int e = tid; e < d.cb * 9; e += nt) {
        int k = e / 9, p = (e % 9) / 3, q = e % 3; // F[row 3k+p, col 3k+q], p >= q
        if (p >= q)
            F[(3 * k + p) + (size_t) (3 * k + q) * ld] =
                a.Adiag[9 * (size_t) a.q2node[d.first + k] + q * 3 + p];
    }
    for (int e = tid; e < c; e += nt) // rhs row
        F[m + (size_t) e * ld] = a.Bq[3 * (size_t) a.q2node[d.first + e / 3] + e % 3];
    for (int e = tid; e < d.a_cnt * 9; e += nt) {
        int i = e / 9, p = (e % 9) / 3, q = e % 3; // late-node component p (row), early q (col)
        const int rbf = a_rb[i];
        const int rb = rbf & ~ASAM_TR_FLAG;
        // slot is S[lo id][hi id]; flag set when the early (column) node is the higher id
        const int si = (rbf & ASAM_TR_FLAG) ? (p * 3 + q) : (q * 3 + p);
        F[(3 * rb + p) + (size_t) (3 * a_cb[i] + q) * ld] = a.Aoff[9 * (size_t) a_slot[i] + si];
    }
    if (a.trace && tid == 0)
        tr1 = d_now();

    // ---- 2. wait for the children that are being re-factored in this launch ---------
    if (nw > 0 && tid == 0) {
        SpinClock spins;
        while (ld_volatile(&a.arrive[s]) < nw) {
            __nanosleep(32);
            if (spin_over(spins, a.spin_limit) || ld_volatile(err) < 0) {
                atomicCAS(err, 0, -(1 + s));
                *s_abort = 1;
                break;
            }
        }
        a.arrive[s] = 0;
        __threadfence();
    }
    __syncthreads();
    if (*s_abort)
        return false;
    if (a.trace && tid == 0)
        tr2 = d_now();

    // ---- 3. extend-add the children's update matrices (fixed order: deterministic) ----
    for (int ci = 0; ci < d.ch_cnt; ++ci) {
        const asam_sn_desc_t cd = ci < ASAM_MAX_CACHED_CHILDREN ? s_cd[ci] : a.sn[children[ci]];
        const int cm = 3 * cd.mb, cc = 3 * cd.cb, cr = cm - cc, cld = ASAM_LD(cm);
        const double *CF = a.arena + cd.f_off;
        const int *crel = a.ipool + cd.seg + cd.mb; // rel[]
        // destination row of child row cc+i (i in [0,cr]); the child's rhs row -> ours
        if (dmap_ahead) {
            dmap = (int *) (sm + fsz) + s_doff[ci];
        } else {
            for (int i = tid; i <= cr; i += nt)
                dmap[i] = (i < cr) ? 3 * crel[(cc + i) / 3] + (cc + i) % 3 : m;
            __syncthreads();
        }
        if (use_sm && cr <= 159) {
            // the whole update matrix in few round trips: four columns per warp and pass, up to
            // 160 rows each -> 20 independent loads in flight per lane (the critical path of a
            // small solve is a chain of these extend-adds, each bound by L2 latency, not bytes)
            for (int j0 = warp; j0 < cr; j0 += 4 * nwarps) {
                double v[4][5];
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    const int j = j0 + q * nwarps;
                    const double *ccol = CF + (size_t) (cc + min(j, cr - 1)) * cld + cc;
#pragma unroll
                    for (int u = 0; u < 5; u++) {
                        const int i = j + lane + 32 * u;
                        v[q][u] = (j < cr && i <= cr) ? __ldcg(ccol + i) : 0.0;
                    }
                }
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    const int j = j0 + q * nwarps;
                    if (j < cr) {
                        double *fcol = F + (size_t) dmap[j] * ld;
#pragma unroll
                        for (int u = 0; u < 5; u++) {
                            const int i = j + lane + 32 * u;
                            if (i <= cr)
                                fcol[dmap[i]] += v[q][u];
                        }
                    }
                }
            }
        } else {
            for (int j = warp; j < cr; j += nwarps) {
                const double *ccol = CF + (size_t) (cc + j) * cld + cc;
                double *fcol = F + (size_t) dmap[j] * ld;
                for (int i0 = j + lane; i0 <= cr; i0 += 256) { // sixteen independent loads in flight per lane
                    double v[8], dv[8];
                    int di[8];
#pragma unroll
                    for (int u = 0; u < 8; u++) {
                        const bool ok = i0 + 32 * u <= cr;
                        v[u] = ok ? __ldcg(ccol + i0 + 32 * u) : 0.0;
                        di[u] = ok ? dmap[i0 + 32 * u] : -1;
                    }
#pragma unroll
                    for (int u = 0; u < 8; u++)
                        dv[u] = di[u] >= 0 ? fcol[di[u]] : 0.0;
#pragma unroll
                    for (int u = 0; u < 8; u++)
                        if (di[u] >= 0)
                            fcol[di[u]] = dv[u] + v[u];
                }
            }
        }
        __syncthreads();
    }
    if (a.trace && tid == 0)
        tr3 = d_now();

    // ---- 4. eliminate this supernode's columns, panel by panel ------------------------
    int kstart = 0;
    if (use_sm && keepw != 0) {
        const int keep = 3 * (keepw >> 16), m_old = 3 * (keepw & 0xffff), ld_old = ASAM_LD(m_old);
        if (keep > 0 && keep < c && m_old <= m && keep <= m_old) {
            // retained L (rows j..m_old-1) and y (old rhs row) of the kept columns; the rows of the poses
            // appended since are structurally zero in them
            for (int j = warp; j < keep; j += nwarps) {
                const double *oc = Fg + (size_t) j * ld_old;
                double *nc = F + (size_t) j * ld;
                for (int i = j + lane; i < m; i += 32)
                    nc[i] = i < m_old ? oc[i] : 0.0;
                if (lane == 0)
                    nc[m] = oc[m_old];
            }
            __syncthreads();
            if (a.smem_mma)
                trailing_update_mma(F, ld, F, ld, keep, keep, m, m);
            else
                trailing_update<2, 8>(F, ld, F, ld, keep, keep, m, m);
            __syncthreads();
            kstart = keep;
        }
    }
    if (use_sm) {
        const int pbw = a.pb_smem; // panel width of shared-memory fronts (12; ASAM_PB_SMEM=24 for A/B)
        for (int k0 = kstart; k0 < c; k0 += pbw) {
            const int pb = min(pbw, c - k0);
            double *P = F + (size_t) k0 * ld; // panel columns live inside the front
            unsigned long long ta = 0, tb = 0;
            if (a.trace && tid == 0)
                ta = d_now();
            panel_factor(P, ld, k0, pb, m, s, err, dinv);
            if (a.trace && tid == 0) {
                tb = d_now();
                accA += tb - ta;
            }
            const int n = m - (k0 + pb);
            if (a.smem_mma >= 2 && n > 0) // (12-column panels were faster on the DFMA tiles in A/B runs)
                trailing_update_mma(F, ld, P, ld, pb, k0 + pb, m, m);
            else if (n > 48)
                trailing_update<2, 8>(F, ld, P, ld, pb, k0 + pb, m, m);
            else
                trailing_update<1, 4>(F, ld, P, ld, pb, k0 + pb, m, m);
            __syncthreads();
        }
    } else {
        // Front in HBM handled by this CTA alone (fronts whose team would be one CTA, and every such front
        // of an incremental step): the front stays in HBM/L2; one panel of up to a.solo_pb columns, rows
        // k0..m, is staged in shared memory, factored there in 12-column sub-panels with tensor-pipe updates
        // between them, written back, and applied to the trailing matrix by solo_update.  Nothing else reads
        // the front before it is published, so no flag or fence separates the steps: one CTA barrier after
        // the staging and one after the trailing update.
        // Staged copy: rows kr..m (kr = k0 rounded down to even) of panel column p at Pbuf[(row - kr) + p * ldp];
        // ldp = 4 (mod 16) keeps the m8n8k4 fragment loads free of bank conflicts.  Pst addresses it by front row.
        double *Pbuf = sm + pboff;
        const int ldp = ((m + 2) & ~15) + (((m + 2) & 15) <= 4 ? 4 : 20);
        int PB = (a.smem_doubles - pboff) / ldp;
        PB = PB > a.solo_pb ? a.solo_pb : PB;
        PB = PB >= ASAM_PB ? PB - (PB % ASAM_PB) : PB - (PB % 3);
        if (PB < 3) { // front too tall for even a 3-column panel (cannot happen below m ~ 8000)
            if (tid == 0)
                atomicCAS(err, 0, -(1 + s));
            return false;
        }
        for (int k0 = 0; k0 < c; k0 += PB) {
            const int pbw = min(PB, c - k0);
            const int kr = k0 & ~1, nr2 = (m - kr + 2) >> 1; // staged rows kr..kr+2*nr2-1 (<= ld-1): 16-byte pairs
            double *Pst = Pbuf - kr;
            solo_copy(Pbuf, ldp, F + kr + (size_t) k0 * ld, ld, nr2, pbw);
            __syncthreads();
            double *Cp = Pst - (size_t) k0 * ldp; // the staged panel addressed by front row and FRONT column
            for (int k1 = 0; k1 < pbw; k1 += ASAM_PB) {
                const int pb = min(ASAM_PB, pbw - k1);
                panel_factor(Pst + (size_t) k1 * ldp, ldp, k0 + k1, pb, m, s, err, dinv);
                if (k1 + pb < pbw) {
                    trailing_update_mma(Cp, ldp, Pst + (size_t) k1 * ldp, ldp, pb, k0 + k1 + pb, k0 + pbw, m);
                    __syncthreads();
                }
            }
            solo_copy(F + kr + (size_t) k0 * ld, ld, Pbuf, ldp, nr2, pbw); // L and the panel's y
            solo_update(F, ld, Pst, ldp, pbw, k0 + pbw, m);
            __syncthreads();
        }
    }
    if (a.trace && tid == 0)
        tr4 = d_now();

    // ---- 5. publish: the update matrix first (that is all the parent waits for), then y and
    // the L panel, which only the back-substitution and later incremental steps read ----------
    if (use_sm) {
        for (int j = c + warp; j < m; j += nwarps)
            for (int i = j + lane; i <= m; i += 32)
                Fg[i + (size_t) j * ld] = F[i + (size_t) j * ld];
    }
    __syncthreads();
    if (tid == 0 && d.parent >= 0) {
        __threadfence();
        atomicAdd(&a.arrive[d.parent], 1);
    }
    for (int e = tid; e < c; e += nt)
        a.y[3 * (size_t) d.first + e] = F[m + (size_t) e * ld];
    if (use_sm) {
        for (int j = warp; j < c; j += nwarps)
            for (int i = j + lane; i <= m; i += 32)
                Fg[i + (size_t) j * ld] = F[i + (size_t) j * ld];
    }
    __syncthreads();
    if (tid == 0) {
        if (a.trace) {
            unsigned smid;
            asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
            unsigned long long *tr = a.trace + 8 * (size_t) t;
            tr[0] = tr0; tr[1] = tr1; tr[2] = tr2; tr[3] = tr3; tr[4] = tr4; tr[5] = d_now();
            (void) smid;
            tr[6] = (unsigned long long) s | (accB << 32); // low: supernode, high: ns in panel TRSM
            tr[7] = (unsigned long long) (unsigned) m | (accA << 32); // low: m, high: ns in diag blocks
        }
    }
    __syncthreads();
    return true;
}

__global__ void __launch_bounds__(256, 1) k_factor(FacArgs a)
{
    extern __shared__ __align__(16) double sm[];
    __shared__ int s_task, s_abort;
    __shared__ asam_sn_desc_t s_cd[ASAM_MAX_CACHED_CHILDREN];
    __shared__ __align__(8) unsigned long long s_mbar; // completion of the bulk copies of one tile (team path)
    const int tid = threadIdx.x;
    unsigned mb_parity = 0;
    if (tid == 0)
        mbar_init(&s_mbar, 1);
    __syncthreads();
    for (;;) {
        if (tid == 0) {
            s_task = atomicAdd(&a.ctrl[0], 1);
            s_abort = 0;
        }
        __syncthreads();
        const int t = s_task;
        if (t >= a.ntasks)
            break;
        unsigned long long tr0 = 0;
        if (a.trace && tid == 0)
            tr0 = d_now();
        const int s = a.tasks[t];
        const int nwp = a.nwait[t];
        const int nw = nwp & 0xffff, tw = (nwp >> 16) & 0xff, tG = (nwp >> 24) & 0x7f;
        const asam_sn_desc_t d = a.sn[s];
        if (tG >= 1) { // one worker of a CTA team (a team of one runs the same panel code alone)
            unsigned long long *trow = (a.trace && tw == 0) ? a.trace + 8 * (size_t) t : nullptr;
            if (trow && tid == 0) {
                trow[0] = tr0; trow[1] = tr0;
            }
            if (!team_front(a, d, s, nw, tw, tG, sm, &s_abort, trow, &s_mbar, mb_parity))
                break;
            if (a.trace && tid == 0) {
                unsigned long long *tr = a.trace + 8 * (size_t) t;
                if (tw == 0) {
                    tr[5] = d_now();
                    tr[6] = (unsigned long long) s | ((unsigned long long) tG << 32);
                } else { // other workers: only the total
                    tr[0] = tr0; tr[1] = tr0; tr[2] = tr0; tr[3] = tr0; tr[4] = d_now(); tr[5] = tr[4];
                    tr[6] = (unsigned long long) s | ((unsigned long long) tG << 32);
                    tr[7] = (unsigned long long) (unsigned) (3 * d.mb);
                }
            }
            __syncthreads();
            continue;
        }
        if (!cta_front(a, t, s, nw, d, sm, s_cd, &s_abort, tr0, a.keep ? a.keep[t] : 0))
            break;
    }
    ticket_release(&a.ctrl[0], &a.ctrl[3]);
}

// ------------------------------------------------------------------------------------------
// kernel 2a: the leaves.  Large graphs have tens of thousands of supernodes with tiny fronts
// (100 k Manhattan: 36 k of 47 k have m < 49) at the bottom of the tree; one CTA per front
// wastes the SM on them.  Here every WARP takes tickets on its own and factors a whole front
// (m <= ASAM_LEAF_M) in its private slice of shared memory; the host hands this kernel the
// downward-closed set of supernodes whose whole subtree consists of such fronts, k_factor does
// the rest afterwards.  Same arithmetic as k_factor's shared-memory path (3-column closed-form
// steps, right-looking), same front layout, same arrival counters.
// ------------------------------------------------------------------------------------------
#define ASAM_LEAF_M 63   // (host: ASAM_LEAF_MAX_M_DEFAULT; 7 warps x 32.5 KB of shared memory)
#define ASAM_LEAF_WARPS 7
#define ASAM_LEAF_STRIDE (ASAM_LD(ASAM_LEAF_M) * ASAM_LEAF_M + ASAM_LEAF_M / 2 + 2) // doubles per warp (even)

struct LeafArgs {
    const asam_sn_desc_t *sn;
    const int *ipool;
    double *arena;
    const double *Adiag, *Aoff, *Bq;
    const int *q2node;
    double *y;
    double *dinv;
    int *arrive;
    const int *tasks; // children before parents
    int ntasks;
    int *ctrl; // [5] ticket, [6] done, [1] err
    long long spin_limit;
};

__global__ void __launch_bounds__(32 * ASAM_LEAF_WARPS, 1) k_factor_leaf(LeafArgs a)
{
    extern __shared__ __align__(16) double sm[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double *F = sm + (size_t) warp * ASAM_LEAF_STRIDE;
    int *dmap = (int *) (F + ASAM_LD(ASAM_LEAF_M) * ASAM_LEAF_M);
    int *err = a.ctrl + 1;
    for (;;) {
        int t = 0;
        if (lane == 0)
            t = atomicAdd(&a.ctrl[5], 1);
        t = __shfl_sync(0xffffffffu, t, 0);
        if (t >= a.ntasks)
            break;
        const int s = a.tasks[t];
        const asam_sn_desc_t d = a.sn[s];
        const int m = 3 * d.mb, c = 3 * d.cb, ld = ASAM_LD(m);
        if (m > ASAM_LEAF_M) { // host error
            if (lane == 0)
                atomicCAS(err, 0, -(1 + s));
            break;
        }
        const int *seg = a.ipool + d.seg;
        const int *children = seg + 2 * d.mb;
        const int *a_slot = children + d.ch_cnt;
        const int *a_rb = a_slot + d.a_cnt;
        const int *a_cb = a_rb + d.a_cnt;
        double *Fg = a.arena + d.f_off;
        const int fsz = ld * m;

        // ---- 1. zero, gather the original entries ------------------------------------------
        for (int i = lane; i < fsz; i += 32)
            F[i] = 0.0;
        __syncwarp();
        for (int e = lane; e < d.cb * 9; e += 32) {
            int k = e / 9, p = (e % 9) / 3, q = e % 3;
            if (p >= q)
                F[(3 * k + p) + (3 * k + q) * ld] = a.Adiag[9 * (size_t) a.q2node[d.first + k] + q * 3 + p];
        }
        for (int e = lane; e < c; e += 32)
            F[m + e * ld] = a.Bq[3 * (size_t) a.q2node[d.first + e / 3] + e % 3];
        for (int e = lane; e < d.a_cnt * 9; e += 32) {
            int i = e / 9, p = (e % 9) / 3, q = e % 3;
            const int rbf = a_rb[i];
            const int rb = rbf & ~ASAM_TR_FLAG;
            const int si = (rbf & ASAM_TR_FLAG) ? (p * 3 + q) : (q * 3 + p);
            F[(3 * rb + p) + (3 * a_cb[i] + q) * ld] = a.Aoff[9 * (size_t) a_slot[i] + si];
        }

        // ---- 2. wait for the children (all of them are tasks of this launch) -----------------
        int abort_ = 0;
        if (d.ch_cnt > 0) {
            if (lane == 0) {
                SpinClock spins;
                while (ld_volatile(&a.arrive[s]) < d.ch_cnt) {
                    __nanosleep(20);
                    if (spin_over(spins, a.spin_limit) || ld_volatile(err) < 0) {
                        atomicCAS(err, 0, -(1 + s));
                        abort_ = 1;
                        break;
                    }
                }
                a.arrive[s] = 0;
                __threadfence();
            }
            abort_ = __shfl_sync(0xffffffffu, abort_, 0);
        }
        if (abort_)
            break;
        __syncwarp();

        // ---- 3. extend-add --------------------------------------------------------------------
        for (int ci = 0; ci < d.ch_cnt; ++ci) {
            const asam_sn_desc_t cd = a.sn[children[ci]];
            const int cm = 3 * cd.mb, cc = 3 * cd.cb, cr = cm - cc, cld = ASAM_LD(cm);
            const double *CF = a.arena + cd.f_off + (size_t) cc * cld + cc; // (0,0) of the update matrix
            const int *crel = a.ipool + cd.seg + cd.mb;
            for (int i = lane; i <= cr; i += 32)
                dmap[i] = (i < cr) ? 3 * crel[(cc + i) / 3] + (cc + i) % 3 : m;
            __syncwarp();
            const int n = (cr + 1) * cr; // entries (i, j): i in [0, cr] (cr = rhs row), j in [0, cr)
            for (int e0 = lane; e0 < n; e0 += 128) {
                double v[4];
                int dst[4];
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const int e = e0 + 32 * u;
                    const int j = e / (cr + 1), i = e - j * (cr + 1);
                    const bool ok = e < n && i >= j;
                    v[u] = ok ? __ldcg(CF + i + (size_t) j * cld) : 0.0;
                    dst[u] = ok ? dmap[i] + dmap[j] * ld : -1;
                }
#pragma unroll
                for (int u = 0; u < 4; u++)
                    if (dst[u] >= 0)
                        F[dst[u]] += v[u];
            }
            __syncwarp();
        }

        // ---- 4. eliminate the c columns, 3 at a time ---------------------------------------
        double *dinv = a.dinv + 3 * (size_t) d.first;
        for (int k = 0; k < c; k += 3) {
            double *p0 = F + k * ld, *p1 = p0 + ld, *p2 = p1 + ld;
            const double a00 = p0[k], a10 = p0[k + 1], a20 = p0[k + 2];
            const double a11 = p1[k + 1], a21 = p1[k + 2], a22 = p2[k + 2];
            const double r0 = d_rsqrt(a00);
            const double l10 = a10 * r0, l20 = a20 * r0;
            const double d1 = a11 - l10 * l10;
            const double r1 = d_rsqrt(d1);
            const double l21 = (a21 - l20 * l10) * r1;
            const double d2 = a22 - l20 * l20 - l21 * l21;
            const double r2 = d_rsqrt(d2);
            if (lane == 0 && !(a00 > 0.0 && d1 > 0.0 && d2 > 0.0))
                atomicCAS(err, 0, 1 + s);
            __syncwarp(); // every lane has read the diagonal block
            for (int i = k + 3 + lane; i <= m; i += 32) {
                const double x0 = p0[i] * r0;
                const double x1 = (p1[i] - x0 * l10) * r1;
                const double x2 = (p2[i] - x0 * l20 - x1 * l21) * r2;
                p0[i] = x0;
                p1[i] = x1;
                p2[i] = x2;
            }
            if (lane == 0) {
                p0[k] = a00 * r0; p0[k + 1] = l10; p0[k + 2] = l20;
                p1[k + 1] = d1 * r1; p1[k + 2] = l21;
                p2[k + 2] = d2 * r2;
                dinv[k] = r0; dinv[k + 1] = r1; dinv[k + 2] = r2;
            }
            __syncwarp();
#pragma unroll 4
            for (int j = k + 3; j < m; ++j) {
                const double y0 = p0[j], y1 = p1[j], y2 = p2[j];
                double *cj = F + j * ld;
                for (int i = j + lane; i <= m; i += 32)
                    cj[i] -= p0[i] * y0 + p1[i] * y1 + p2[i] * y2;
            }
            __syncwarp();
        }

        // ---- 5. publish ------------------------------------------------------------------------
        for (int e = lane; e < c; e += 32)
            a.y[3 * (size_t) d.first + e] = F[m + e * ld];
        for (int i = lane; i < fsz; i += 32)
            Fg[i] = F[i];
        __syncwarp();
        if (lane == 0 && d.parent >= 0) {
            __threadfence();
            atomicAdd(&a.arrive[d.parent], 1);
        }
        __syncwarp();
    }
    ticket_release(&a.ctrl[5], &a.ctrl[6]);
}

// ------------------------------------------------------------------------------------------
// kernel 3: persistent back-substitution
// ------------------------------------------------------------------------------------------
struct BsArgs {
    const asam_sn_desc_t *sn;
    const int *ipool;
    const double *arena;
    const double *y;
    const double *dinv; // 1/L_kk written by k_factor
    double *x;
    int *xdone;
    const int *btasks;
    const int *bfirst; // optional, per task: first wanted pose of the supernode (see cta_backsolve, jcol)
    int *xblk;         // per supernode: (epoch << 8) | finished blocks (tasks that solve one block, see ASAM_BT_*)
    int ntasks;
    int *ctrl; // [2] ticket, [1] err
    int epoch;
    int smem_doubles;
    long long spin_limit;
    unsigned long long *trace;
};

// One supernode: x1 = L11^-T (y1 - L21' x2), x2 gathered from the ancestors' solution.
// The supernode's columns are solved in blocks of <= ASAM_BSW columns, last block first; for a
// block [b0, be) every row below it (later blocks and L21 alike) is "already known":
//   w = y[b0:be] - L[be:m, b0:be]' xf[be:m],   L[b0:be, b0:be]' x = w.
// Supernodes of the shared-memory path have one block (<= 96 columns); the wide supernodes of
// the team path (merged chains, up to the whole root separator) loop.
// Everything that does not depend on the parent (descriptor, row list, y, 1/diag and the L
// panel of the first block when it fits in shared memory) is fetched BEFORE waiting on the
// parent's flag.
#define ASAM_BSW 96
// back-solve task word: bits 0-23 supernode, bits 24-30 (one ASAM_BSW-column block of it) + 1, 0 = all of it
#define ASAM_BT_SN(e) ((e) & 0xffffff)
#define ASAM_BT_BLK(e) ((((e) >> 24) & 0x7f) - 1)

template <int U>
__device__ __forceinline__ double bs_dot(const double *lk, const double *xs, int n, int lane)
{
    double acc0 = 0.0, acc1 = 0.0;
    for (int i0 = lane; i0 < n; i0 += 32 * U) { // U independent loads in flight per lane
        double v[U];
#pragma unroll
        for (int u = 0; u < U; u++)
            v[u] = (i0 + 32 * u < n) ? lk[i0 + 32 * u] : 0.0;
#pragma unroll
        for (int u = 0; u < U; u += 2) {
            acc0 += v[u] * xs[min(i0 + 32 * u, n - 1)];
            acc1 += v[u + 1] * xs[min(i0 + 32 * (u + 1), n - 1)];
        }
    }
    acc0 += acc1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        acc0 += __shfl_down_sync(0xffffffffu, acc0, o);
    return acc0;
}

// One supernode of the back-substitution handled by ONE CTA (see the comment above).  t = index in the
// task list (trace slot).  Returns false on abort.
// jcol > 0 (incremental steps with the reference's pruned traversal, aprilsam.c:752-772): only x of the
// columns [jcol, c) is wanted -- back-substitution inside a supernode runs from its last column down, so it
// simply stops there (the columns before depend on these, not the other way round).
// blk_only >= 0 (wide supernodes of a batch solve, host: build_schedule): this task solves ONE ASAM_BSW-column
// block of the supernode; the blocks of a supernode are separate tasks (last block first) that run on
// different CTAs: every block first subtracts the ancestors' part (rows below the supernode) -- all blocks at
// once, as soon as the parent's flag is up -- and then the parts of the later blocks AS THEY FINISH
// (a.xblk[s] counts finished blocks, tagged with the launch epoch), so that the dependent chain per block is
// one 96 x 96 matrix-vector product and one triangular solve instead of a pass over everything below.
__device__ bool cta_backsolve(const BsArgs &a, const int t, const int s, double *sm, int *s_abort, const int jcol = 0,
                              const int blk_only = -1)
{
    const int tid = threadIdx.x, nt = blockDim.x;
    const int lane = tid & 31, warp = tid >> 5, nwarps = nt >> 5;
    int *err = a.ctrl + 1;
    unsigned long long tr0 = 0, tr1 = 0, tr2 = 0;
    if (a.trace && tid == 0)
        tr0 = d_now();
    const asam_sn_desc_t d = a.sn[s];
    const int m = 3 * d.mb, c = 3 * d.cb, r = m - c, ld = ASAM_LD(m);
    const int *rows = a.ipool + d.seg;
    const double *Lg = a.arena + d.f_off;
    const int bwmax = min(c, ASAM_BSW);
    if (m + 2 * bwmax + 2 > a.smem_doubles) { // host sizes shared memory for the largest front
        if (tid == 0)
            atomicCAS(err, 0, -(1 + s));
        return false;
    }
    double *xf = sm;          // x over the front's rows: [0,c) own columns, [c,m) ancestors
    double *w = sm + m;       // bwmax
    double *rd = w + bwmax;   // bwmax
    double *Ls = rd + bwmax;
    const long long room = (long long) a.smem_doubles - (m + 2 * bwmax);
    const int nblk = (c + ASAM_BSW - 1) / ASAM_BSW;

    const int blk_hi = blk_only >= 0 ? blk_only : nblk - 1, blk_lo = blk_only >= 0 ? blk_only : 0;
    for (int blk = blk_hi; blk >= blk_lo; --blk) {
        const int b0 = blk * ASAM_BSW, bw = min(ASAM_BSW, c - b0), be = b0 + bw, hb = m - b0;
        // staging mode: 2 = whole panel of the block (rows b0..m-1, ld lm), 1 = its diagonal
        // block only (ld lc), 0 = none.  Staged leading dimensions are ODD: the triangular
        // solve reads row k across columns, an even stride would pile the lanes onto a few banks
        if (be <= jcol)
            break; // nothing wanted in this block or the ones before it
        const int kmin = max(0, jcol - b0); // first wanted column of this block
        const int lm = hb | 1, lc = bw | 1;
        const int mode = ((long long) lm * bw <= room) ? 2 : (((long long) lc * bw <= room) ? 1 : 0);
        const int ll = mode == 2 ? lm : (mode == 1 ? lc : ld);
        if (blk != blk_hi)
            __syncthreads(); // the previous block is done with w / rd / Ls
        if (mode == 2) {
            for (int k = kmin + warp; k < bw; k += nwarps)
                for (int i = k + lane; i < hb; i += 32)
                    Ls[i + (size_t) k * lm] = Lg[(b0 + i) + (size_t) (b0 + k) * ld];
        } else if (mode == 1) {
            for (int k = kmin + warp; k < bw; k += nwarps)
                for (int i = k + lane; i < bw; i += 32)
                    Ls[i + (size_t) k * lc] = Lg[(b0 + i) + (size_t) (b0 + k) * ld];
        }
        for (int k = tid; k < bw; k += nt) {
            w[k] = a.y[3 * (size_t) d.first + b0 + k];
            rd[k] = a.dinv[3 * (size_t) d.first + b0 + k];
        }
        const double *L11 = mode ? Ls : (Lg + b0 + (size_t) b0 * ld); // (row, col) at L11[row + col*ll]

        if (blk == blk_hi) {
            if (a.trace && tid == 0)
                tr1 = d_now();
            if (d.parent >= 0 && tid == 0) {
                SpinClock spins;
                while (ld_volatile(&a.xdone[d.parent]) != a.epoch) {
                    __nanosleep(20);
                    if (spin_over(spins, a.spin_limit) || ld_volatile(err) < 0) {
                        atomicCAS(err, 0, -(1 + s));
                        *s_abort = 1;
                        break;
                    }
                }
                __threadfence();
            }
            __syncthreads();
            if (*s_abort)
                break;
            if (a.trace && tid == 0)
                tr2 = d_now();
            for (int i = tid; i < r; i += nt)
                xf[c + i] = __ldcg(&a.x[3 * (size_t) rows[d.cb + i / 3] + i % 3]);
        }
        __syncthreads();
        if (blk_only >= 0) {
            // (a) the ancestors' rows [c, m): available since the parent's flag
            if (r > 0) {
                for (int k = warp; k < bw; k += nwarps) {
                    const double *lk = (mode == 2) ? (Ls + (size_t) k * lm + (c - b0)) : (Lg + (size_t) (b0 + k) * ld + c);
                    const double acc = r > 512 ? bs_dot<16>(lk, xf + c, r, lane) : bs_dot<8>(lk, xf + c, r, lane);
                    if (lane == 0)
                        w[k] -= acc;
                }
            }
            // (b) the later blocks of this supernode, in the order they finish
            const int ep = a.epoch & 0xffffff;
            for (int b2 = nblk - 1; b2 > blk; --b2) {
                const int r0 = b2 * ASAM_BSW, n2 = min(ASAM_BSW, c - r0), need = nblk - b2;
                if (tid == 0) {
                    SpinClock spins;
                    for (;;) {
                        const int v = ld_volatile(&a.xblk[s]);
                        if ((int) ((unsigned) v >> 8) == ep && (v & 0xff) >= need)
                            break;
                        __nanosleep(20);
                        if (spin_over(spins, a.spin_limit) || ld_volatile(err) < 0) {
                            atomicCAS(err, 0, -(1 + s));
                            *s_abort = 1;
                            break;
                        }
                    }
                    __threadfence();
                }
                __syncthreads();
                if (*s_abort)
                    break;
                for (int i = tid; i < n2; i += nt)
                    xf[r0 + i] = __ldcg(&a.x[3 * (size_t) d.first + r0 + i]);
                __syncthreads();
                // 96 rows x ceil(bw / nwarps) columns per warp in rounds of six (two rounds with the default 8 warps):
                // 18 loads in flight per lane (the chain of a block is this product + the triangular solve)
                {
                    double xv[3];
#pragma unroll
                    for (int u = 0; u < 3; u++)
                        xv[u] = lane + 32 * u < n2 ? xf[r0 + lane + 32 * u] : 0.0;
#pragma unroll 1
                    for (int j0 = 0; j0 * nwarps < bw; j0 += 6) {
                        double lv[6][3];
#pragma unroll
                        for (int j = 0; j < 6; j++) {
                            const int k = warp + nwarps * (j0 + j);
                            const double *lk = (mode == 2) ? (Ls + (size_t) min(k, bw - 1) * lm + (r0 - b0))
                                                           : (Lg + (size_t) (b0 + min(k, bw - 1)) * ld + r0);
#pragma unroll
                            for (int u = 0; u < 3; u++)
                                lv[j][u] = (k < bw && lane + 32 * u < n2) ? lk[lane + 32 * u] : 0.0;
                        }
#pragma unroll
                        for (int j = 0; j < 6; j++) {
                            double acc = lv[j][0] * xv[0] + lv[j][1] * xv[1] + lv[j][2] * xv[2];
#pragma unroll
                            for (int o = 16; o > 0; o >>= 1)
                                acc += __shfl_down_sync(0xffffffffu, acc, o);
                            const int k = warp + nwarps * (j0 + j);
                            if (lane == 0 && k < bw)
                                w[k] -= acc;
                        }
                    }
                }
            }
            __syncthreads();
            if (*s_abort)
                break;
        }
        // w_k -= sum_{i >= be} L[i, b0+k] * xf[i]   (one warp per column)
        const int nr = blk_only >= 0 ? 0 : m - be;
        if (nr > 0) {
            for (int k = kmin + warp; k < bw; k += nwarps) {
                const double *lk = (mode == 2) ? (Ls + (size_t) k * lm + bw) : (Lg + (size_t) (b0 + k) * ld + be);
                const double acc = nr > 512 ? bs_dot<16>(lk, xf + be, nr, lane) : bs_dot<8>(lk, xf + be, nr, lane);
                if (lane == 0)
                    w[k] -= acc;
            }
            __syncthreads();
        }
        // L11' x = w, right-looking: x_k = w_k / L_kk, then w_j -= L[k, j] * x_k for j < k.
        // One warp, w in registers (lane l holds entries l, l+32, l+64), x_k travels by shuffle:
        // no shared-memory round trip on the dependent chain.
        if (warp == 0) {
            double wr[3];
#pragma unroll
            for (int t3 = 0; t3 < 3; t3++)
                wr[t3] = (lane + 32 * t3 < bw) ? w[lane + 32 * t3] : 0.0;
#pragma unroll 2
            for (int k = bw - 1; k >= kmin; --k) {
                const int ks = k >> 5;
                const double mine = ks == 0 ? wr[0] : (ks == 1 ? wr[1] : wr[2]);
                const double xk = __shfl_sync(0xffffffffu, mine, k & 31) * rd[k];
#pragma unroll
                for (int t3 = 0; t3 < 3; t3++) {
                    const int j = lane + 32 * t3;
                    if (j < k && j >= kmin)
                        wr[t3] -= L11[k + (size_t) j * ll] * xk;
                    else if (j == k)
                        wr[t3] = xk;
                }
            }
#pragma unroll
            for (int t3 = 0; t3 < 3; t3++) {
                const int k = lane + 32 * t3;
                if (k < bw && k >= kmin) {
                    a.x[3 * (size_t) d.first + b0 + k] = wr[t3];
                    xf[b0 + k] = wr[t3];
                }
            }
            __syncwarp();
        }
    }
    if (*s_abort)
        return false;
    if (warp == 0 && lane == 0) {
        __threadfence();
        if (blk_only >= 0)
            atomicExch(&a.xblk[s], ((a.epoch & 0xffffff) << 8) | (nblk - blk_only));
        if (blk_only <= 0)
            atomicExch(&a.xdone[s], a.epoch);
        if (a.trace) {
            unsigned long long *tr = a.trace + 8 * (size_t) t;
            tr[0] = tr0; tr[1] = tr1; tr[2] = tr2; tr[3] = d_now();
            tr[6] = (unsigned long long) s;
            tr[7] = (unsigned) m;
        }
    }
    __syncthreads();
    return true;
}

__global__ void __launch_bounds__(256, 2) k_backsolve(BsArgs a)
{
    extern __shared__ __align__(16) double sm[]; // xf[m] | w[bw] | rd[bw] | staged L (panel or L11 of one block)
    __shared__ int s_task, s_abort;
    const int tid = threadIdx.x, nt = blockDim.x;
    const int lane = tid & 31, warp = tid >> 5, nwarps = nt >> 5;
    int *err = a.ctrl + 1;

    for (;;) {
        if (tid == 0) {
            s_task = atomicAdd(&a.ctrl[2], 1);
            s_abort = 0;
        }
        __syncthreads();
        const int t = s_task;
        if (t >= a.ntasks)
            break;
        if (!cta_backsolve(a, t, ASAM_BT_SN(a.btasks[t]), sm, &s_abort, a.bfirst ? 3 * a.bfirst[t] : 0, ASAM_BT_BLK(a.btasks[t])))
            break;
    }
    ticket_release(&a.ctrl[2], &a.ctrl[4]);
}

// ------------------------------------------------------------------------------------------
// kernel 3a: back-substitution of the leaf set (see k_factor_leaf), one WARP per supernode,
// launched after k_backsolve has solved every other supernode with the same epoch.  The L panel
// (m x c, usually 48 x 9 or less) is staged in the warp's slice of shared memory when it fits,
// L21' x2 is one lane per column, the triangular solve runs in registers with shuffles.
// ------------------------------------------------------------------------------------------
#define ASAM_BSL_WARPS 8
#define ASAM_BSL_PANEL 1024                         // staged panel entries per warp
#define ASAM_BSL_XS 64                              // rows below the supernode (x2) per warp
#define ASAM_BSL_STRIDE (ASAM_BSL_PANEL + ASAM_BSL_XS) // doubles per warp

__global__ void __launch_bounds__(32 * ASAM_BSL_WARPS) k_backsolve_leaf(BsArgs a)
{
    extern __shared__ __align__(16) double sm[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double *Ls = sm + (size_t) warp * ASAM_BSL_STRIDE;
    double *xs = Ls + ASAM_BSL_PANEL;
    int *err = a.ctrl + 1;
    for (;;) {
        int t = 0;
        if (lane == 0)
            t = atomicAdd(&a.ctrl[5], 1);
        t = __shfl_sync(0xffffffffu, t, 0);
        if (t >= a.ntasks)
            break;
        const int s = ASAM_BT_SN(a.btasks[t]);
        const asam_sn_desc_t d = a.sn[s];
        const int m = 3 * d.mb, c = 3 * d.cb, r = m - c, ld = ASAM_LD(m);
        if (r > ASAM_BSL_XS || c > 64) { // host error: not a leaf-set supernode
            if (lane == 0)
                atomicCAS(err, 0, -(1 + s));
            break;
        }
        const int *rows = a.ipool + d.seg;
        const double *Lg = a.arena + d.f_off;
        const int lm = m | 1;
        const bool staged = lm * c <= ASAM_BSL_PANEL;
        if (staged) {
            for (int k = 0; k < c; k++)
                for (int i = k + lane; i < m; i += 32)
                    Ls[i + k * lm] = Lg[i + (size_t) k * ld];
        }
        const double *L = staged ? Ls : Lg;
        const int ll = staged ? lm : ld;
        double wr[2], rdv[2];
#pragma unroll
        for (int t2 = 0; t2 < 2; t2++) {
            const int k = lane + 32 * t2;
            wr[t2] = k < c ? a.y[3 * (size_t) d.first + k] : 0.0;
            rdv[t2] = k < c ? a.dinv[3 * (size_t) d.first + k] : 0.0;
        }
        int abort_ = 0;
        if (d.parent >= 0) {
            if (lane == 0) {
                SpinClock spins;
                while (ld_volatile(&a.xdone[d.parent]) != a.epoch) {
                    __nanosleep(20);
                    if (spin_over(spins, a.spin_limit) || ld_volatile(err) < 0) {
                        atomicCAS(err, 0, -(1 + s));
                        abort_ = 1;
                        break;
                    }
                }
                __threadfence();
            }
            abort_ = __shfl_sync(0xffffffffu, abort_, 0);
        }
        if (abort_)
            break;
        for (int i = lane; i < r; i += 32)
            xs[i] = __ldcg(&a.x[3 * (size_t) rows[d.cb + i / 3] + i % 3]);
        __syncwarp();
        // w_k -= sum_i L[c+i, k] xs[i]: one lane per column
#pragma unroll
        for (int t2 = 0; t2 < 2; t2++) {
            const int k = lane + 32 * t2;
            if (k < c) {
                const double *lk = L + c + (size_t) k * ll;
                double acc0 = 0.0, acc1 = 0.0;
                int i = 0;
#pragma unroll 4
                for (; i + 1 < r; i += 2) {
                    acc0 += lk[i] * xs[i];
                    acc1 += lk[i + 1] * xs[i + 1];
                }
                if (i < r)
                    acc0 += lk[i] * xs[i];
                wr[t2] -= acc0 + acc1;
            }
        }
        // L11' x = w in registers, x_k by shuffle
        for (int k = c - 1; k >= 0; --k) {
            const double mine = (k >> 5) == 0 ? wr[0] : wr[1];
            const double rk = (k >> 5) == 0 ? rdv[0] : rdv[1];
            const double xk = __shfl_sync(0xffffffffu, mine * rk, k & 31);
#pragma unroll
            for (int t2 = 0; t2 < 2; t2++) {
                const int j = lane + 32 * t2;
                if (j < k)
                    wr[t2] -= L[k + (size_t) j * ll] * xk;
                else if (j == k)
                    wr[t2] = xk;
            }
        }
#pragma unroll
        for (int t2 = 0; t2 < 2; t2++) {
            const int k = lane + 32 * t2;
            if (k < c)
                a.x[3 * (size_t) d.first + k] = wr[t2];
        }
        __syncwarp();
        if (lane == 0) {
            __threadfence();
            atomicExch(&a.xdone[s], a.epoch);
        }
        __syncwarp();
    }
    ticket_release(&a.ctrl[5], &a.ctrl[6]);
}

// ------------------------------------------------------------------------------------------
// kernel 4: a SMALL incremental step in one launch.
//
// The reference spends 18-60 us on an incremental step that touches a handful of poses
// (aprilsam.c:377-576; SURVEY.md section 7 "a GPU step must be a single small launch").  The general
// path costs five stream operations (H2D copy, scatter, k_linearize, k_factor, k_backsolve) plus two
// D2H copies and a stream synchronisation -- a dependent chain of launch latencies several times
// longer than the arithmetic.  Here ONE CTA does the whole step:
//   1. fetches the step's uploads (item table + payload queued by the host in PINNED memory) over
//      PCIe in one wave of 16-byte loads and scatters them to their places in HBM,
//   2. linearises the new factors,
//   3. re-factors the marked supernodes in list order (children first; all of them single-CTA fronts),
//   4. back-substitutes the visited supernodes in list order (parents first),
//   5. writes the solution of those supernodes and the status word straight into pinned host memory
//      and raises a sequence flag there -- the host spins on that flag instead of synchronising the
//      stream.
// The per-front / per-supernode code is the same device function the persistent kernels run
// (cta_front, cta_backsolve): the counters they wait on are already satisfied when they look.
// ------------------------------------------------------------------------------------------
struct StepArgs {
    const uint4 *host_in; // pinned host memory: [item table | payload]
    uint4 *stage;         // device mirror of it
    unsigned int table_bytes, payload_off, payload_bytes; // table = n_items * sizeof(BatchItem)
    int n_items;
    LinArgs lin;
    FacArgs fac;
    BsArgs bs;
    double *x_out;      // pinned host memory: x of the back-solved supernodes, in list order
    volatile int *done; // pinned host memory: [0] sequence number of the last finished step, [1] status,
                        // [2..15] as unsigned long long[7]: globaltimer at kernel start / uploads in place /
                        // linearised / factored / back-solved / results written (diagnostics)
    int seq;
};

__global__ void __launch_bounds__(256, 1) k_step(StepArgs a)
{
    extern __shared__ __align__(16) double sm[];
    __shared__ int s_abort;
    __shared__ asam_sn_desc_t s_cd[ASAM_MAX_CACHED_CHILDREN];
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nwarps = nt >> 5;
    volatile unsigned long long *stamps = (volatile unsigned long long *) (a.done + 2);
    if (tid == 0)
        stamps[0] = d_now();

    // ---- 1. uploads: host -> staging (all loads of a thread in flight before the first store) ----
    {
        const unsigned nt16 = (a.table_bytes + 15) >> 4, np16 = (a.payload_bytes + 15) >> 4, p0 = a.payload_off >> 4;
        const unsigned n16 = nt16 + np16;
        for (unsigned i0 = tid; i0 < n16; i0 += 4 * nt) {
            uint4 v[4];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const unsigned i = i0 + u * nt;
                if (i < n16)
                    v[u] = a.host_in[i < nt16 ? i : p0 + (i - nt16)];
            }
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const unsigned i = i0 + u * nt;
                if (i < n16)
                    a.stage[i < nt16 ? i : p0 + (i - nt16)] = v[u];
            }
        }
    }
    __syncthreads();
    {
        const BatchItem *items = (const BatchItem *) a.stage;
        const char *payload = (const char *) a.stage + a.payload_off;
        for (int it = warp; it < a.n_items; it += nwarps) {
            const BatchItem bi = items[it];
            unsigned int *dst = (unsigned int *) bi.dst;
            const unsigned int words = bi.bytes >> 2;
            if (bi.fill) {
                for (unsigned int i = lane; i < words; i += 32)
                    dst[i] = bi.val;
            } else {
                const unsigned int *src = (const unsigned int *) (payload + bi.off);
                for (unsigned int i = lane; i < words; i += 32)
                    dst[i] = __ldcg(src + i);
            }
        }
    }
    __threadfence();
    __syncthreads();
    if (tid == 0)
        stamps[1] = d_now();

    // ---- 2. new factors -----------------------------------------------------------------------
    for (int t0 = 0; t0 < a.lin.f_count; t0 += nt)
        linearize_body(a.lin, t0 + tid);
    __threadfence();
    __syncthreads();

    if (tid == 0)
        stamps[2] = d_now();

    // ---- 3. marked supernodes, children first ---------------------------------------------------
    bool ok = true;
    for (int t = 0; t < a.fac.ntasks && ok; ++t) {
        if (tid == 0)
            s_abort = 0;
        __syncthreads();
        const int s = a.fac.tasks[t];
        const int nwp = a.fac.nwait[t];
        const asam_sn_desc_t d = a.fac.sn[s];
        if (((nwp >> 24) & 0x7f) > 1) { // a team front: the host must not send it here
            if (tid == 0)
                atomicCAS(a.fac.ctrl + 1, 0, -(1 + s));
            ok = false;
            break;
        }
        ok = cta_front(a.fac, t, s, nwp & 0xffff, d, sm, s_cd, &s_abort, 0ULL, a.fac.keep ? a.fac.keep[t] : 0);
    }

    if (tid == 0)
        stamps[3] = d_now();

    // ---- 4. visited supernodes, parents first ---------------------------------------------------
    for (int t = 0; t < a.bs.ntasks && ok; ++t) {
        if (tid == 0)
            s_abort = 0;
        __syncthreads();
        ok = cta_backsolve(a.bs, t, ASAM_BT_SN(a.bs.btasks[t]), sm, &s_abort, a.bs.bfirst ? 3 * a.bs.bfirst[t] : 0);
    }
    __syncthreads();

    if (tid == 0)
        stamps[4] = d_now();

    // ---- 5. results to the host ---------------------------------------------------------------
    if (ok) {
        int off = 0;
        for (int t = 0; t < a.bs.ntasks; ++t) {
            const int s = ASAM_BT_SN(a.bs.btasks[t]);
            const int first = a.bs.sn[s].first, c = 3 * a.bs.sn[s].cb;
            for (int k = tid; k < c; k += nt)
                a.x_out[off + k] = __ldcg(&a.bs.x[3 * (size_t) first + k]);
            off += c;
        }
    }
    __threadfence_system();
    __syncthreads();
    if (tid == 0) {
        stamps[5] = d_now();
        a.done[1] = ld_volatile(a.fac.ctrl + 1);
        __threadfence_system();
        a.done[0] = a.seq;
    }
}

// ------------------------------------------------------------------------------------------
// chi2
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_chi2_partial(const int *f_type, const int *f_a, const int *f_b,
                                                      const double *f_z, const double *f_W, const double2 *f_loss,
                                                      const double *st, int n_factors, double *partial)
{
    __shared__ double red[256];
    int f = blockIdx.x * blockDim.x + threadIdx.x;
    double v = 0.0;
    if (f < n_factors) {
        int type = f_type[f];
        int na = f_a[f];
        double z[3], W[9], r[3];
#pragma unroll
        for (int i = 0; i < 3; i++)
            z[i] = f_z[3 * (size_t) f + i];
#pragma unroll
        for (int i = 0; i < 9; i++)
            W[i] = f_W[9 * (size_t) f + i];
        double scale;
        if (d_two_pose(type)) { // xyt at `state`, weight 0.5   (april_graph.c:86-89)
            int nb = f_b[f];
            double pa[3], pb[3], Ja[9], Jb[9];
#pragma unroll
            for (int i = 0; i < 3; i++) { pa[i] = st[3 * (size_t) na + i]; pb[i] = st[3 * (size_t) nb + i]; }
            d_xyt_eval(pa, pb, z, Ja, Jb, r);
            scale = 0.5;
        } else { // weight 1.0   (april_graph.c:90-93)
            r[0] = z[0] - st[3 * (size_t) na + 0];
            r[1] = z[1] - st[3 * (size_t) na + 1];
            r[2] = d_mod2pi(z[2] - st[3 * (size_t) na + 2]);
            scale = 1.0;
        }
        double X[3];
        d_av(W, r, X);
        const double s = r[0] * X[0] + r[1] * X[1] + r[2] * X[2];
        if (type == 32) { // robust xyt: 0.5 rho(s)
            const double2 lk = f_loss[f];
            v = scale * asam_loss_rho((int) lk.x, lk.y, s);
        } else {
            v = scale * s;
        }
    }
    red[threadIdx.x] = v;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o)
            red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0)
        partial[blockIdx.x] = red[0];
}

__global__ void __launch_bounds__(256) k_chi2_final(const double *partial, int n, double *out)
{
    __shared__ double red[256];
    double v = 0.0;
    for (int i = threadIdx.x; i < n; i += 256)
        v += partial[i];
    red[threadIdx.x] = v;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o)
            red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0)
        out[0] = red[0];
}

__global__ void k_apply_desc(asam_sn_desc_t *sn, const int *ids, const asam_sn_desc_t *desc, int n)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
        sn[ids[i]] = desc[i];
}

__global__ void k_clear_range(double *Adiag, double *Bq, double *Aoff, int q_first, int q_count, int s_first,
                              int s_count)
{
    size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    size_t nd = 9 * (size_t) q_count, nb = 3 * (size_t) q_count, no = 9 * (size_t) s_count;
    if (i < nd)
        Adiag[9 * (size_t) q_first + i] = 0.0;
    else if (i < nd + nb)
        Bq[3 * (size_t) q_first + (i - nd)] = 0.0;
    else if (i < nd + nb + no)
        Aoff[9 * (size_t) s_first + (i - nd - nb)] = 0.0;
}

// ------------------------------------------------------------------------------------------
// marginal covariances: Sigma = A^-1 = P' L^-T L^-1 P from the factor the last solve left in the arena
// ------------------------------------------------------------------------------------------
// Z_i = L^-1 E_q (three columns) is non-zero only on the supernodes from the pose's own up to the root, and
// the path is a chain: every supernode on it gets its right-hand side from exactly one child.  Neither kernel
// writes anything the solve path reads (arena, x, y, dinv, Hessian, control words): only the scratch below.
struct MargArgs {
    const asam_sn_desc_t *sn;
    const int *ipool;
    const double *arena;
    const double *dinv;
    const asam_marg_path_t *paths;
    const asam_marg_pair_t *pairs; // k_marginal_pairs: one record per candidate
    double *z;   // per pose: 3 doubles per scalar row of its path (row-major: row, column of E_q)
    int *hop;    // per hop: supernode, first row js, c, offset of its rows from the pose's zoff
    double *out; // k_marginal_gram: (3n x 3n) row-major; k_marginal_pairs: 10 doubles per candidate
    int *err;    // 0 ok, 1 front larger than max_m, 2 path length differs from the plan's
    int n, max_m;
};

#define ASAM_MLS (ASAM_BSW + 1) // leading dimension of the staged L11 block (odd: no bank conflicts)
#define ASAM_MKG 24             // columns of a block per thread group of the trailing update (4 groups x 24 = ASAM_BSW)
#define ASAM_MROWS 128          // rows of the trailing update per pass (2 per thread of a group)
#define ASAM_MSMEM(max_m) (6 * (size_t) (max_m) + ASAM_BSW * ASAM_MLS + ASAM_BSW + 4 * ASAM_MROWS * 3) // doubles

// One CTA per requested pose.  At each supernode s of its path (m rows, c own columns), with b the m x 3
// right-hand side: L11 z = b[js, c) block by block (ASAM_BSW columns, the diagonal block staged in shared
// memory and solved by one warp with the pivots 1/L_kk from dinv, as cta_backsolve uses them), after each block
// b[be, m) -= L[be:m, block] z_block by all threads (24 loads of L in flight per row and thread: the path is a
// dependent chain, latency is what counts).  Then z_s goes to the scratch and u = b[c, m) to the parent's rows
// through rel.
__global__ void __launch_bounds__(256) k_marginal_path(MargArgs a)
{
    extern __shared__ __align__(16) double sm[];
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nwarps = nt >> 5;
    const asam_marg_path_t P = a.paths[blockIdx.x];
    double *b = sm, *bn = sm + 3 * (size_t) a.max_m;
    double *Ls = bn + 3 * (size_t) a.max_m;
    double *rd = Ls + ASAM_BSW * ASAM_MLS;
    double *part = rd + ASAM_BSW; // [4 groups][ASAM_MROWS rows][3]
    int s = P.sn0, js = P.j0, h = 0;
    int64_t zo = P.zoff;
    asam_sn_desc_t d = a.sn[s];
    int m = 3 * d.mb;
    if (m > a.max_m) {
        if (tid == 0)
            atomicCAS(a.err, 0, 1);
        return;
    }
    for (int i = tid; i < 3 * m; i += nt)
        b[i] = 0.0;
    __syncthreads();
    if (tid < 3)
        b[3 * (js + tid) + tid] = 1.0;
    __syncthreads();
    for (;;) {
        const int c = 3 * d.cb, ld = ASAM_LD(m);
        const double *Lg = a.arena + d.f_off;
        for (int b0 = js; b0 < c; b0 += ASAM_BSW) {
            const int bw = min(ASAM_BSW, c - b0), be = b0 + bw;
            for (int k = warp; k < bw; k += nwarps)
                for (int j = k + lane; j < bw; j += 32)
                    Ls[j + k * ASAM_MLS] = Lg[(b0 + j) + (size_t) (b0 + k) * ld];
            for (int k = tid; k < bw; k += nt)
                rd[k] = a.dinv[3 * (size_t) d.first + b0 + k];
            __syncthreads();
            // L11 z = b, left to right: z_k = b_k / L_kk, then b_j -= L[j, k] z_k for j > k.  Lane l holds rows
            // l, l+32, l+64 of the block, z_k travels by shuffle.
            if (warp == 0) {
                double w[3][3];
#pragma unroll
                for (int t3 = 0; t3 < 3; t3++)
#pragma unroll
                    for (int e = 0; e < 3; e++)
                        w[t3][e] = lane + 32 * t3 < bw ? b[3 * (b0 + lane + 32 * t3) + e] : 0.0;
                for (int k = 0; k < bw; ++k) {
                    const int ks = k >> 5;
                    double zk[3];
#pragma unroll
                    for (int e = 0; e < 3; e++) {
                        const double mine = ks == 0 ? w[0][e] : (ks == 1 ? w[1][e] : w[2][e]);
                        zk[e] = __shfl_sync(0xffffffffu, mine, k & 31) * rd[k];
                    }
#pragma unroll
                    for (int t3 = 0; t3 < 3; t3++) {
                        const int j = lane + 32 * t3;
                        if (j > k && j < bw) {
                            const double l = Ls[j + k * ASAM_MLS];
#pragma unroll
                            for (int e = 0; e < 3; e++)
                                w[t3][e] -= l * zk[e];
                        } else if (j == k) {
#pragma unroll
                            for (int e = 0; e < 3; e++)
                                w[t3][e] = zk[e];
                        }
                    }
                }
#pragma unroll
                for (int t3 = 0; t3 < 3; t3++)
                    if (lane + 32 * t3 < bw)
#pragma unroll
                        for (int e = 0; e < 3; e++)
                            b[3 * (b0 + lane + 32 * t3) + e] = w[t3][e];
            }
            __syncthreads();
            // b[be, m) -= L[be:m, b0:be] z: thread = (row slot rs, column group kg), two rows per pass; the four
            // groups' partial sums are added in a fixed order
            const int rs = tid & 63, kg = tid >> 6, k0 = kg * ASAM_MKG, k1 = min(k0 + ASAM_MKG, bw);
            for (int base = be; base < m; base += ASAM_MROWS) {
                const int i0 = base + rs, i1 = i0 + 64;
                double a0[3] = {0.0, 0.0, 0.0}, a1[3] = {0.0, 0.0, 0.0};
                if (k0 < k1) {
                    double l0[ASAM_MKG], l1[ASAM_MKG];
#pragma unroll
                    for (int u = 0; u < ASAM_MKG; u++) {
                        const size_t col = (size_t) (b0 + k0 + u) * ld;
                        l0[u] = (k0 + u < k1 && i0 < m) ? Lg[i0 + col] : 0.0;
                        l1[u] = (k0 + u < k1 && i1 < m) ? Lg[i1 + col] : 0.0;
                    }
#pragma unroll
                    for (int u = 0; u < ASAM_MKG; u++) {
                        if (k0 + u < k1) {
                            const double *zk = b + 3 * (b0 + k0 + u);
#pragma unroll
                            for (int e = 0; e < 3; e++) {
                                a0[e] += l0[u] * zk[e];
                                a1[e] += l1[u] * zk[e];
                            }
                        }
                    }
                }
#pragma unroll
                for (int e = 0; e < 3; e++) {
                    part[(kg * ASAM_MROWS + rs) * 3 + e] = a0[e];
                    part[(kg * ASAM_MROWS + rs + 64) * 3 + e] = a1[e];
                }
                __syncthreads();
                for (int q = tid; q < 3 * ASAM_MROWS; q += nt) {
                    const int r = q / 3, e = q % 3, i = base + r;
                    if (i < m)
                        b[3 * i + e] -= ((part[r * 3 + e] + part[(ASAM_MROWS + r) * 3 + e]) +
                                         part[(2 * ASAM_MROWS + r) * 3 + e]) + part[(3 * ASAM_MROWS + r) * 3 + e];
                }
                __syncthreads();
            }
        }
        for (int i = tid; i < 3 * (c - js); i += nt)
            a.z[zo + i] = b[3 * js + i];
        if (tid == 0 && h < P.nhop) {
            int *hr = a.hop + 4 * ((size_t) P.hop0 + h);
            hr[0] = s; hr[1] = js; hr[2] = c; hr[3] = (int) (zo - P.zoff);
        }
        zo += 3 * (c - js);
        ++h;
        if (d.parent < 0)
            break;
        // u = b[c, m) into the parent's rows
        const int *rel = a.ipool + d.seg + d.mb;
        const int cb = d.cb, mb = d.mb;
        s = d.parent;
        d = a.sn[s];
        const int mp = 3 * d.mb;
        if (mp > a.max_m) {
            if (tid == 0)
                atomicCAS(a.err, 0, 1);
            return;
        }
        for (int i = tid; i < 3 * mp; i += nt)
            bn[i] = 0.0;
        __syncthreads();
        for (int q = tid; q < 9 * (mb - cb); q += nt) {
            const int row = 3 * cb + q / 3, e = q % 3;
            bn[3 * (3 * rel[row / 3] + row % 3) + e] = b[3 * row + e];
        }
        __syncthreads();
        double *t = b;
        b = bn;
        bn = t;
        m = mp;
        js = 0;
    }
    if (h != P.nhop && tid == 0)
        atomicCAS(a.err, 0, 2);
}

// Sigma_ij = Z_i' Z_j over the supernodes the two paths share (a common suffix of both hop lists: paths never meet
// again below their lowest common ancestor), from that ancestor up, each in rows [max(js_i, js_j), c).  Called by
// all 128 threads of a CTA; fixed striping and a fixed reduction tree, no floating-point atomics: the block depends
// only on the two poses.  Returns element tid (row-major) to threads tid < 9, for a diagonal block (diag) taken
// from the upper triangle, so that the block is exactly symmetric.
__device__ __forceinline__ double marg_block(const MargArgs &a, const asam_marg_path_t &Pi, const asam_marg_path_t &Pj,
                                             bool diag)
{
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5;
    __shared__ int s_ns;
    __shared__ double red[4][9];
    __shared__ double S[9];
    const int *hi = a.hop + 4 * (size_t) Pi.hop0, *hj = a.hop + 4 * (size_t) Pj.hop0;
    const int nmin = min(Pi.nhop, Pj.nhop);
    if (tid == 0)
        s_ns = nmin;
    __syncthreads();
    for (int t = tid; t < nmin; t += nt)
        if (hi[4 * (Pi.nhop - 1 - t)] != hj[4 * (Pj.nhop - 1 - t)])
            atomicMin(&s_ns, t);
    __syncthreads();
    double acc[9];
#pragma unroll
    for (int q = 0; q < 9; q++)
        acc[q] = 0.0;
    for (int t = s_ns - 1; t >= 0; --t) {
        const int *ri = hi + 4 * (Pi.nhop - 1 - t), *rj = hj + 4 * (Pj.nhop - 1 - t);
        const int c = ri[2], r0 = max(ri[1], rj[1]);
        const double *zi = a.z + Pi.zoff + ri[3] + 3 * (r0 - ri[1]);
        const double *zj = a.z + Pj.zoff + rj[3] + 3 * (r0 - rj[1]);
        for (int k = tid; k < c - r0; k += nt) {
            const double u0 = zi[3 * k], u1 = zi[3 * k + 1], u2 = zi[3 * k + 2];
            const double v0 = zj[3 * k], v1 = zj[3 * k + 1], v2 = zj[3 * k + 2];
            acc[0] += u0 * v0; acc[1] += u0 * v1; acc[2] += u0 * v2;
            acc[3] += u1 * v0; acc[4] += u1 * v1; acc[5] += u1 * v2;
            acc[6] += u2 * v0; acc[7] += u2 * v1; acc[8] += u2 * v2;
        }
    }
#pragma unroll
    for (int q = 0; q < 9; q++) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
            acc[q] += __shfl_down_sync(0xffffffffu, acc[q], o);
        if (lane == 0)
            red[warp][q] = acc[q];
    }
    __syncthreads();
    if (tid < 9)
        S[tid] = ((red[0][tid] + red[1][tid]) + red[2][tid]) + red[3][tid];
    __syncthreads();
    if (tid >= 9)
        return 0.0;
    const int r = tid / 3, q = tid % 3;
    return (diag && r > q) ? S[3 * q + r] : S[tid];
}

// One CTA per pair i <= j: block (i, j) from marg_block, (j, i) written as its exact transpose.
__global__ void __launch_bounds__(128) k_marginal_gram(MargArgs a)
{
    const int i = blockIdx.y, j = blockIdx.x, tid = threadIdx.x;
    if (i > j)
        return;
    const double v = marg_block(a, a.paths[i], a.paths[j], i == j);
    if (tid < 9) {
        const int r = tid / 3, q = tid % 3;
        const size_t n3 = 3 * (size_t) a.n;
        a.out[(3 * (size_t) i + r) * n3 + 3 * j + q] = v;
        a.out[(3 * (size_t) j + q) * n3 + 3 * i + r] = v;
    }
}

// One CTA per candidate factor (asam_marg_pair_t): Sigma_aa, and for a closure Sigma_ab and Sigma_bb, by marg_block
// (each bit-identical to the block asam_marginal_cov gives), then on one thread Sigma_rel = J Sigma_6 J' in the
// order of a row-major 3x6 by 6x6 by 6x3 product (symmetrised from its upper triangle; Sigma_aa itself for a
// prior), S = Sigma_rel + Winv, S = L L' and d2 = |L^-1 r|^2.  A pivot of S that is not > 0 gives NaN.  The output
// depends only on the candidate's own record: the same alone, in any request, order or batch.
__global__ void __launch_bounds__(128) k_marginal_pairs(MargArgs a)
{
    const int tid = threadIdx.x;
    const asam_marg_pair_t &pr = a.pairs[blockIdx.x];
    const int pa = pr.pa, pb = pr.pb;
    __shared__ double sg[3][9]; // Sigma_aa, Sigma_ab, Sigma_bb
    const asam_marg_path_t Pa = a.paths[pa];
    double v = marg_block(a, Pa, Pa, true);
    if (tid < 9)
        sg[0][tid] = v;
    if (pb >= 0) {
        const asam_marg_path_t Pb = a.paths[pb];
        v = marg_block(a, Pa, Pb, false);
        if (tid < 9)
            sg[1][tid] = v;
        v = marg_block(a, Pb, Pb, true);
        if (tid < 9)
            sg[2][tid] = v;
    }
    __syncthreads();
    if (tid != 0)
        return;
    double R[9];
    if (pb < 0) {
#pragma unroll
        for (int q = 0; q < 9; q++)
            R[q] = sg[0][q];
    } else {
        // Sigma_6 = [S_aa S_ab; S_ab' S_bb], entry (k, c)
        auto s6 = [&](int k, int c) -> double {
            if (k < 3)
                return c < 3 ? sg[0][3 * k + c] : sg[1][3 * k + c - 3];
            return c < 3 ? sg[1][3 * c + k - 3] : sg[2][3 * (k - 3) + c - 3];
        };
        double JS[18];
        for (int r = 0; r < 3; r++)
            for (int c = 0; c < 6; c++) {
                double acc = 0.0;
                for (int k = 0; k < 6; k++)
                    acc += pr.J[6 * r + k] * s6(k, c);
                JS[6 * r + c] = acc;
            }
        for (int r = 0; r < 3; r++)
            for (int c = r; c < 3; c++) {
                double acc = 0.0;
                for (int k = 0; k < 6; k++)
                    acc += JS[6 * r + k] * pr.J[6 * c + k];
                R[3 * r + c] = acc;
                R[3 * c + r] = acc;
            }
    }
    double *o = a.out + 10 * (size_t) blockIdx.x;
#pragma unroll
    for (int q = 0; q < 9; q++)
        o[1 + q] = R[q];
    double d2 = nan("");
    if (pr.has_w) {
        double S[9];
#pragma unroll
        for (int q = 0; q < 9; q++)
            S[q] = R[q] + pr.Winv[q];
        const double l00 = S[0] > 0.0 ? sqrt(S[0]) : nan("");
        const double l10 = S[3] / l00, l20 = S[6] / l00;
        const double e11 = S[4] - l10 * l10;
        const double l11 = e11 > 0.0 ? sqrt(e11) : nan("");
        const double l21 = (S[7] - l20 * l10) / l11;
        const double e22 = (S[8] - l20 * l20) - l21 * l21;
        const double l22 = e22 > 0.0 ? sqrt(e22) : nan("");
        const double y0 = pr.r[0] / l00;
        const double y1 = (pr.r[1] - l10 * y0) / l11;
        const double y2 = ((pr.r[2] - l20 * y0) - l21 * y1) / l22;
        d2 = (y0 * y0 + y1 * y1) + y2 * y2;
    }
    o[0] = d2;
}
