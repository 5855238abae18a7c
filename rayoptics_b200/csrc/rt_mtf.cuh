/*
 * rt_mtf.cuh -- the pupil function and the ordered sums of rt_grid_pupil_function / rt_grid_mtf.
 * Kept in a header so that tests/hostsim can compile it for the host.
 *
 * Contract (DESIGN.md section 4), restated in numpy by engine.mtf_sums_host:
 *   a ray is used when its status is 0 and x*x + y*y <= 1 (the rule of rt_grid_zernike);
 *   its phasor is P = exp(2 pi i w), w = opd/lambda rounded once, evaluated as sincospi(2.0*w)
 *   (2.0*w is exact); an unused ray has P = +0.0 + 0.0i;
 *   the product a*conj(b) is re = ar*br + ai*bi, im = ai*br - ar*bi with every real product rounded
 *   once (the library is built with -fmad=false and nothing here uses __fma_rn);
 *   a line is added along its own axis in increasing index from +0.0, and the line sums are added in
 *   line order from +0.0 (mtf_line_shift / mtf_line_sum applied twice).
 */
#pragma once
#include <cuda_runtime.h>

namespace b200rt {

/* one complex128 value, laid out as numpy / torch store it (re, im); 16-byte aligned so that the
 * device moves it with one 128-bit access */
struct alignas(16) MtfC {
    double re, im;
};

__device__ __forceinline__ bool mtf_used(int status, double x, double y)
{
    return status == 0 && x*x + y*y <= 1.0;
}

#if defined(__CUDACC__) || defined(RT_HOSTSIM_SINCOSPI)
/* exp(2 pi i opd/lambda); the host build supplies its own sincospi */
__device__ __forceinline__ MtfC mtf_phasor(double opd, double lambda)
{
    const double w = opd/lambda;
    MtfC p;
    sincospi(2.0*w, &p.im, &p.re);
    return p;
}
#endif

__device__ __forceinline__ MtfC mtf_add(MtfC a, MtfC b)
{
    return MtfC{a.re + b.re, a.im + b.im};
}

/* a*conj(b), every real product rounded once */
__device__ __forceinline__ MtfC mtf_mul_conj(MtfC a, MtfC b)
{
    const double rr = a.re*b.re, ii = a.im*b.im, ir = a.im*b.re, ri = a.re*b.im;
    return MtfC{rr + ii, ir - ri};
}

/* one line at shift k: sum over i = 0 ... n-k-1 of p[(i+k)*stride]*conj(p[i*stride]), in increasing
 * i from +0.0 */
__device__ __forceinline__ MtfC mtf_line_shift(const MtfC *__restrict__ p, int64_t stride, int n, int k)
{
    MtfC acc{0.0, 0.0};
    const MtfC *a = p + (int64_t)k*stride;
#pragma unroll 4
    for (int i = 0; i < n - k; i++) acc = mtf_add(acc, mtf_mul_conj(a[(int64_t)i*stride], p[(int64_t)i*stride]));
    return acc;
}

/* sum over i = 0 ... n-1 of p[i*stride], in increasing i from +0.0 (a line of S = sum P, and the
 * line sums of every result in line order) */
__device__ __forceinline__ MtfC mtf_line_sum(const MtfC *__restrict__ p, int64_t stride, int n)
{
    MtfC acc{0.0, 0.0};
#pragma unroll 4
    for (int i = 0; i < n; i++) acc = mtf_add(acc, p[(int64_t)i*stride]);
    return acc;
}

}  // namespace b200rt
