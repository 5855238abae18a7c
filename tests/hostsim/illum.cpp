/*
 * tests/hostsim/illum.cpp -- TEST INFRASTRUCTURE (see cuda_runtime.h here).
 * rayoptics_b200/csrc/rt_illum.cuh compiled for the host, in a library of its own: the used-ray rule,
 * the derivative choice, J and the two-level sums, applied as k_illumination applies them, for
 * tests/test_relative_illumination.py.
 */
#define RT_HOSTSIM 1
#include "cuda_runtime.h"
#include <vector>

#include "../../rayoptics_b200/csrc/rt_illum.cuh"

using namespace b200rt;

extern "C" {

/* one tile: status, L, M [n][n] (ray (i, j) at i*n + j), x, y [n] -> record [10] as k_illumination
 * writes it; kinds [4]: how often each illum_deriv branch was taken, over both axes of every used ray */
int hostsim_illum_tile(int n, const int32_t *status, const double *L, const double *M, const double *x,
                       const double *y, double *record, int64_t *kinds)
{
    std::vector<double> col_abs(n), col_j(n);
    int64_t c[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int q = 0; q < 4; q++) kinds[q] = 0;
    auto pt = [&](int i, int j) {
        if (i < 0 || i >= n || j < 0 || j >= n) return IllumPt{0.0, 0.0, false};
        const int64_t r = (int64_t)i*n + j;
        return IllumPt{L[r], M[r], status[r] == 0};
    };
    for (int j = 0; j < n; j++) {
        IllumAcc acc{0.0, 0.0};
        const double y_m = j > 0 ? y[j - 1] : y[j], y_p = j + 1 < n ? y[j + 1] : y[j];
        for (int i = 0; i < n; i++) {
            const int64_t r = (int64_t)i*n + j;
            const int st = status[r];
            c[(st >= 0 && st <= 3) ? st : 4]++;
            c[6] += x[i]*x[i] + y[j]*y[j] <= 1.0;
            if (!illum_used(st, x[i], y[j])) continue;
            c[5]++;
            const double x_m = i > 0 ? x[i - 1] : x[i], x_p = i + 1 < n ? x[i + 1] : x[i];
            double d0, d1;
            kinds[illum_deriv(pt(i - 1, j), pt(i, j), pt(i + 1, j), x_m, x[i], x_p, &d0, &d1)]++;
            kinds[illum_deriv(pt(i, j - 1), pt(i, j), pt(i, j + 1), y_m, y[j], y_p, &d0, &d1)]++;
            if (!illum_term(acc, pt(i, j), pt(i - 1, j), pt(i + 1, j), pt(i, j - 1), pt(i, j + 1),
                            x_m, x[i], x_p, y_m, y[j], y_p))
                c[7]++;
        }
        col_abs[j] = acc.abs_j;
        col_j[j] = acc.j;
    }
    for (int q = 0; q < 8; q++) record[q] = (double)c[q];
    record[8] = illum_line_sum(col_abs.data(), n);
    record[9] = illum_line_sum(col_j.data(), n);
    return 0;
}

}
