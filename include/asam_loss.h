/* asam_loss.h -- robust losses of type-32 factors (aprilsam.h): the IRLS weight w = rho'(s) and the cost rho(s) at
 * s = r'Wr, loss 1 Huber, 2 Cauchy, k > 0 and finite (checked where the loss is set).  One definition for the host
 * hooks (graph.c) and the kernels (k_linearize, k_step, k_hessian_rebuild, k_chi2_partial).
 *
 * Huber compares s with k^2 as written wherever k^2 is at least DBL_MIN (it may overflow to inf); where k * k is
 * subnormal or zero its rounding can be far from k^2, and s <= k^2 is decided as (s / k) / k <= 1 instead.
 *
 * Cauchy evaluates w = 1 / (1 + t) and rho = k^2 log1p(t), t = s / k^2, as written wherever k^2 and t are normal
 * doubles.  Outside that band k^2 overflows, underflows or loses bits, or t does: t is then formed as (s / k) / k,
 * and rho as s log1p(t) / t for k >= 1 (there t < 1) or as k (k log1p(t)) for k < 1, with log1p(t) = log(s) - 2 log(k)
 * where t overflows.  Over every finite s >= 0 and every accepted k both stay within a few ulp of the exact value,
 * or within DBL_MIN of it where that is below DBL_MIN, and neither is NaN.  A NaN s gives NaN for both. */
#ifndef ASAM_LOSS_H
#define ASAM_LOSS_H

#include <math.h>

#ifdef __CUDACC__
#define ASAM_LOSS_FN static __host__ __device__ __forceinline__
#else
#define ASAM_LOSS_FN static inline
#endif

ASAM_LOSS_FN int asam_loss_normal(const double x) { return x >= 0x1p-1022 && x <= 0x1.fffffffffffffp+1023; }

/* Huber: s <= k^2 */
ASAM_LOSS_FN int asam_huber_inside(const double k, const double k2, const double s)
{
    return k2 >= 0x1p-1022 ? s <= k2 : (s / k) / k <= 1.0;
}

ASAM_LOSS_FN double asam_loss_weight(const int loss, const double k, const double s)
{
    const double k2 = k * k;
    if (loss == 1)
        return asam_huber_inside(k, k2, s) ? 1.0 : k / sqrt(s);
    const double t = s / k2;
    if (asam_loss_normal(k2) && asam_loss_normal(t))
        return 1.0 / (1.0 + t);
    return 1.0 / (1.0 + (s / k) / k);
}

ASAM_LOSS_FN double asam_loss_rho(const int loss, const double k, const double s)
{
    const double k2 = k * k;
    if (loss == 1)
        return asam_huber_inside(k, k2, s) ? s : 2.0 * k * sqrt(s) - k2;
    const double t = s / k2;
    if (asam_loss_normal(k2) && asam_loss_normal(t))
        return k2 * log1p(t);
    const double u = (s / k) / k;
    if (k >= 1.0) /* k^2 overflows, or s / k^2 underflows: u < 1 and rho is s to within a factor 1 - u / 2 */
        return u > 0.0 ? s * (log1p(u) / u) : s;
    /* k^2 below DBL_MIN, or s / k^2 above DBL_MAX */
    const double L = u <= 0x1.fffffffffffffp+1023 ? log1p(u) : log(s) - 2.0 * log(k);
    return (k * L) * k;
}

#endif
