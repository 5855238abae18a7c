/*
 * tests/hostsim/mtf.cpp -- TEST INFRASTRUCTURE (see cuda_runtime.h here).
 * rayoptics_b200/csrc/rt_mtf.cuh compiled for the host, in a library of its own: the used-ray rule,
 * the rounded product and the two-level sums, applied as k_mtf applies them, for tests/test_mtf.py.
 * The host has no sincospi: the stand-in below reduces x modulo 2 exactly and calls sin / cos, so
 * the phasor is checked against numpy to a tolerance only; the sums are checked bit for bit.
 */
#define RT_HOSTSIM 1
#define RT_HOSTSIM_SINCOSPI 1
#include "cuda_runtime.h"
#include <vector>

static inline void sincospi(double x, double *s, double *c)
{
    const double r = x - 2.0*std::rint(0.5*x);
    *s = std::sin(M_PI*r);
    *c = std::cos(M_PI*r);
}

#include "../../rayoptics_b200/csrc/rt_mtf.cuh"

using namespace b200rt;

extern "C" {

/* P: [n][n] complex (re, im) of one tile -> acf_x, acf_y [n] complex, s [1] complex, as k_mtf forms
 * them: each line with mtf_line_shift / mtf_line_sum, lines along y from the transposed copy */
int hostsim_mtf_sums(int n, const double *P, double *acf_x, double *acf_y, double *s)
{
    const MtfC *p = reinterpret_cast<const MtfC *>(P);
    std::vector<MtfC> pt((size_t)n*n), lines(n);
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) pt[(size_t)j*n + i] = p[(size_t)i*n + j];
    MtfC *cx = reinterpret_cast<MtfC *>(acf_x), *cy = reinterpret_cast<MtfC *>(acf_y);
    for (int k = 0; k < n; k++) {
        for (int l = 0; l < n; l++) lines[l] = mtf_line_shift(p + l, n, n, k);
        cx[k] = mtf_line_sum(lines.data(), 1, n);
        for (int l = 0; l < n; l++) lines[l] = mtf_line_shift(pt.data() + l, n, n, k);
        cy[k] = mtf_line_sum(lines.data(), 1, n);
    }
    for (int l = 0; l < n; l++) lines[l] = mtf_line_sum(p + l, n, n);
    *reinterpret_cast<MtfC *>(s) = mtf_line_sum(lines.data(), 1, n);
    return 0;
}

/* per ray: out[r] = P of the used rays (mtf_used, mtf_phasor with the stand-in sincospi), 0 else */
int hostsim_mtf_pupil(int64_t n, const int32_t *status, const double *opd, const double *x, const double *y,
                      double lambda, double *out)
{
    MtfC *o = reinterpret_cast<MtfC *>(out);
    for (int64_t r = 0; r < n; r++)
        o[r] = mtf_used(status[r], x[r], y[r]) ? mtf_phasor(opd[r], lambda) : MtfC{0.0, 0.0};
    return 0;
}

}
