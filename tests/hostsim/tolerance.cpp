/*
 * tests/hostsim/tolerance.cpp -- TEST INFRASTRUCTURE (see cuda_runtime.h here).
 * rayoptics_b200/csrc/rt_tol.cuh compiled for the host, in a library of its own: the summands of the
 * tolerance records of rt_trace_grid_variants, for tests/test_tolerance.py.
 */
#define RT_HOSTSIM 1
#include "cuda_runtime.h"
#include "../../rayoptics_b200/csrc/rt_tol.cuh"

using namespace b200rt;

extern "C" {

/* n rays: ax, ay, op, dx, dy, dz [n] -> out [n][16]: the 12 summands of tol_summands at their record
 * columns (tol_sum_col), other columns 0 */
int hostsim_tol_summands(int64_t n, const double *ax, const double *ay, const double *op, const double *dx,
                         const double *dy, const double *dz, double *out)
{
    for (int64_t i = 0; i < n; i++) {
        double v[RT_TOL_ITEM_SUMS];
        const Vec3 d = {dx[i], dy[i], dz[i]};
        tol_summands(ax[i], ay[i], op[i], d, v);
        for (int k = 0; k < 24; k++) out[i*24 + k] = 0.0;
        for (int j = 0; j < RT_TOL_ITEM_SUMS; j++) out[i*24 + tol_sum_col(j)] = v[j];
    }
    return 0;
}

}
