/*
 * tests/hostsim/zernike.cpp -- TEST INFRASTRUCTURE (see cuda_runtime.h here).
 * rayoptics_b200/csrc/rt_zernike.cuh compiled for the host, in a library of its own: the Fringe
 * table and fringe_zernike, point by point, for tests/test_zernike.py.
 */
#define RT_HOSTSIM 1
#include "cuda_runtime.h"
#include "../../rayoptics_b200/csrc/rt_zernike.cuh"

using namespace b200rt;

#define HOSTSIM_MAX_COEFS 8

extern "C" {

/* z: [n][n_terms] */
int hostsim_zernike_terms(int64_t n, const double *x, const double *y, int n_terms, double *z)
{
    for (int64_t r = 0; r < n; r++)
        fringe_zernike(x[r], y[r], n_terms, [&](int j, double v) { z[r*n_terms + j - 1] = v; });
    return 0;
}

/* the table (returns its rows): per term n, m, sin, number of coefficients and coefficients [37][HOSTSIM_MAX_COEFS] */
int hostsim_fringe_table(int32_t *n_out, int32_t *m_out, int32_t *sin_out, int32_t *n_coef, double *coef)
{
    int rows = 0;
#define HOSTSIM_ROW(j, n, m, s, ...)                                                   \
    {                                                                                 \
        const double a_[] = {__VA_ARGS__};                                            \
        const int k_ = (int)(sizeof a_/sizeof a_[0]);                                 \
        n_out[j - 1] = n; m_out[j - 1] = m; sin_out[j - 1] = s; n_coef[j - 1] = k_;   \
        for (int q = 0; q < k_; q++) coef[(j - 1)*HOSTSIM_MAX_COEFS + q] = a_[q];     \
        rows++;                                                                       \
    }
    RT_FRINGE_TABLE(HOSTSIM_ROW)
#undef HOSTSIM_ROW
    return rows;
}

}
