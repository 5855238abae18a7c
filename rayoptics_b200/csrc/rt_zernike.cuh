/*
 * rt_zernike.cuh -- the 37 Fringe (University of Arizona) Zernike polynomials of rt_grid_zernike,
 * evaluated at a ray's relative pupil coordinates (x, y); theta is measured from +x, so Z2 = x and
 * Z3 = y.  Kept in a header so that tests/hostsim can compile it for the host.
 *
 * Term j is R_n^m(rho) * (cos | sin)(m theta) with R_n^m(rho) = rho^m * P(rho^2); the table lists
 * the integer coefficients of P from the constant term up.  The evaluation is part of the arithmetic
 * contract (DESIGN.md section 4) and is restated in numpy by engine.zernike_terms:
 *   r2 = x*x + y*y;
 *   C1 = x, S1 = y, C(k+1) = C(k)*x - S(k)*y, S(k+1) = S(k)*x + C(k)*y   (k < 5);
 *   P by Horner in r2 from the highest coefficient: p = a_K, then p = p*r2 + a_k for k = K-1 ... 0;
 *   Z = P*C(m), P*S(m), or P when m = 0.
 * Every product is rounded once: the library is built with -fmad=false and nothing here uses
 * __fma_rn.
 */
#pragma once
#include <cuda_runtime.h>

namespace b200rt {

#define RT_ZERN_MAX_M 5

/* X(j, n, m, sin, coefficients of P from the constant term up), in Fringe order */
#define RT_FRINGE_TABLE(X)                                   \
    X( 1,  0, 0, 0, 1)                                       \
    X( 2,  1, 1, 0, 1)                                       \
    X( 3,  1, 1, 1, 1)                                       \
    X( 4,  2, 0, 0, -1, 2)                                   \
    X( 5,  2, 2, 0, 1)                                       \
    X( 6,  2, 2, 1, 1)                                       \
    X( 7,  3, 1, 0, -2, 3)                                   \
    X( 8,  3, 1, 1, -2, 3)                                   \
    X( 9,  4, 0, 0, 1, -6, 6)                                \
    X(10,  3, 3, 0, 1)                                       \
    X(11,  3, 3, 1, 1)                                       \
    X(12,  4, 2, 0, -3, 4)                                   \
    X(13,  4, 2, 1, -3, 4)                                   \
    X(14,  5, 1, 0, 3, -12, 10)                              \
    X(15,  5, 1, 1, 3, -12, 10)                              \
    X(16,  6, 0, 0, -1, 12, -30, 20)                         \
    X(17,  4, 4, 0, 1)                                       \
    X(18,  4, 4, 1, 1)                                       \
    X(19,  5, 3, 0, -4, 5)                                   \
    X(20,  5, 3, 1, -4, 5)                                   \
    X(21,  6, 2, 0, 6, -20, 15)                              \
    X(22,  6, 2, 1, 6, -20, 15)                              \
    X(23,  7, 1, 0, -4, 30, -60, 35)                         \
    X(24,  7, 1, 1, -4, 30, -60, 35)                         \
    X(25,  8, 0, 0, 1, -20, 90, -140, 70)                    \
    X(26,  5, 5, 0, 1)                                       \
    X(27,  5, 5, 1, 1)                                       \
    X(28,  6, 4, 0, -5, 6)                                   \
    X(29,  6, 4, 1, -5, 6)                                   \
    X(30,  7, 3, 0, 10, -30, 21)                             \
    X(31,  7, 3, 1, 10, -30, 21)                             \
    X(32,  8, 2, 0, -10, 60, -105, 56)                       \
    X(33,  8, 2, 1, -10, 60, -105, 56)                       \
    X(34,  9, 1, 0, 5, -60, 210, -280, 126)                  \
    X(35,  9, 1, 1, 5, -60, 210, -280, 126)                  \
    X(36, 10, 0, 0, -1, 30, -210, 560, -630, 252)            \
    X(37, 12, 0, 0, 1, -42, 420, -1680, 3150, -2772, 924)

/* P(r2) by Horner from the highest coefficient */
template <int K>
__device__ __forceinline__ double fringe_horner(const double (&a)[K], double r2)
{
    double p = a[K - 1];
#pragma unroll
    for (int k = K - 2; k >= 0; k--) p = p*r2 + a[k];
    return p;
}

/* Z_1 ... Z_{n_terms} at (x, y): put(j, Z_j) for j = 1 ... n_terms, in increasing j.  Terms past
 * n_terms are not formed. */
template <typename Put>
__device__ __forceinline__ void fringe_zernike(double x, double y, int n_terms, Put &&put)
{
    const double r2 = x*x + y*y;
    double C[RT_ZERN_MAX_M + 1], S[RT_ZERN_MAX_M + 1];
    C[0] = 1.0; S[0] = 0.0;            /* not used: m = 0 terms are P alone */
    C[1] = x; S[1] = y;
#pragma unroll
    for (int k = 1; k < RT_ZERN_MAX_M; k++) {
        C[k + 1] = C[k]*x - S[k]*y;
        S[k + 1] = S[k]*x + C[k]*y;
    }
#define RT_FRINGE_EVAL(j, n, m, s, ...)                                             \
    if (j <= n_terms) {                                                             \
        const double a_[] = {__VA_ARGS__};                                          \
        const double p_ = fringe_horner(a_, r2);                                    \
        put(j, (m) == 0 ? p_ : p_*((s) ? S[m] : C[m]));                             \
    }
    RT_FRINGE_TABLE(RT_FRINGE_EVAL)
#undef RT_FRINGE_EVAL
}

}  // namespace b200rt
