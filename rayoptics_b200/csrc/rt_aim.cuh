/*
 * rt_aim.cuh -- chief-ray aiming of one field (rt_grid_aim_chief): the damped 2-D Newton iteration
 * of vigcalc.aim_chief_ray / aim_all_fields_batched, which finds the aim point on the paraxial
 * entrance pupil that puts the (0, 0) pupil ray through the vertex of the stop interface.
 *
 * The iteration, its termination rules and the 2x2 solve are part of the arithmetic contract
 * (DESIGN.md section 4); tests/aim_ref.py restates them in numpy.  Kept in a header so that
 * tests/hostsim can compile it for the host next to the per-ray code.
 */
#pragma once
#include "rt_grid.cuh"

namespace b200rt {

/* not NaN and not +-inf */
__device__ __forceinline__ bool aim_finite(double v) { return fabs(v) < CUDART_INF; }

/* Stop intercept (fx, fy) of the (0, 0) pupil ray of field f aimed at (aim_x, aim_y): the start
 * ray of grid_start_ray_at<false> with the trial aim in place of F.aim (epd_start_ray_aimed), traced by the general loop
 * through interface `stop` (o: first_surf 1, apertures not checked, intersect_obj on).  The loop
 * ends at the stop, so what happens behind it cannot fail the ray; its intercept there has the
 * bits a trace through the whole system records at segment `stop`.  false when the ray does not
 * reach the stop (n_seg <= stop, where aim_all_fields_batched sets NaN) or the intercept is not
 * finite.  Out of line: the iteration traces from four places and one copy of the loop serves them. */
__device__ __noinline__ bool aim_stop_xy(const rt_surface_desc *tab, const double *nrow, double wvl,
                                        const GridDev &G, int f, int stop, const rt_opts &o,
                                        double aim_x, double aim_y, double &fx, double &fy)
{
    Vec3 p0, d0;
    epd_start_ray_aimed(G, f, 0.0, 0.0, aim_x, aim_y, p0, d0);
    FullWriter fw = {nullptr, 0};
    RayResult R;
    trace_ray<false>(tab, nrow, wvl, stop + 1, o, p0, d0, fw, R);
    if (R.n_seg <= stop) return false;
    fx = R.p.x; fy = R.p.y;
    return aim_finite(fx) && aim_finite(fy);
}

/* max(|a|, |b|) of finite values: np.max(np.abs(f)) */
__device__ __forceinline__ double aim_norm(double a, double b)
{
    const double x = fabs(a), y = fabs(b);
    return x < y ? y : x;
}

/* J s = r for the 2x2 matrix [[a, b], [c, d]]: Gaussian elimination with partial pivoting
 * (the rows swap only when |c| > |a|), every operation rounded once:
 *   l = c/a   u = d - l*b   y1 = r1 - l*r0   s1 = y1/u   s0 = (r0 - b*s1)/a
 * false for a zero pivot or a step that is not finite.  With b = 0 and r0 = +-0 (a field on the
 * meridian: its stop intercept has x = +-0 whatever the y aim) this is s1 = r1/d exactly, the
 * value numpy's solve returns there. */
__device__ __forceinline__ bool aim_solve2(double a, double b, double c, double d, double r0, double r1,
                                           double &s0, double &s1)
{
    if (fabs(c) > fabs(a)) {
        double t;
        t = a; a = c; c = t;
        t = b; b = d; d = t;
        t = r0; r0 = r1; r1 = t;
    }
    if (a == 0.0) return false;
    const double l = c/a;
    const double u = d - l*b;
    if (u == 0.0) return false;
    const double y1 = r1 - l*r0;
    s1 = y1/u;
    s0 = (r0 - b*s1)/a;
    return aim_finite(s0) && aim_finite(s1);
}

/* Aim field f (rt_aim_term result; aim = (aim_x, aim_y), iters = accepted Newton steps):
 *   x = (0, 0); f(x) = aim_stop_xy at x; the first ray fails -> x = (0, 0), RT_AIM_FIRST_FAILED.
 *   up to max_iter times:
 *     max|f| < tol                                  -> RT_AIM_CONVERGED
 *     J[:, k] = (f(x + h e_k) - f)/h, the trial aims formed as (x0 + h, x1 + 0.0) and
 *     (x0 + 0.0, x1 + h); either ray fails          -> RT_AIM_DIFF_FAILED
 *     s = aim_solve2(J, -f) fails                   -> RT_AIM_SINGULAR
 *     lam = 1, 1/2, ... (20 trials): accept the first x + lam*s whose ray reaches the stop with
 *     max|f_new| < max|f|; none                     -> RT_AIM_NO_STEP
 *   the loop runs out                               -> RT_AIM_MAX_ITER
 * The field's x == 0 rule of aim_chief_ray (aim_x = 0) is the caller's. */
__device__ __forceinline__ int aim_chief_ray(const rt_surface_desc *tab, const double *nrow, double wvl,
                                             const GridDev &G, int f, int stop, const rt_opts &o, double h,
                                             double tol, int max_iter, double &aim_x, double &aim_y, int &iters)
{
    double x0 = 0.0, x1 = 0.0, f0, f1;
    aim_x = 0.0; aim_y = 0.0; iters = 0;
    if (!aim_stop_xy(tab, nrow, wvl, G, f, stop, o, x0, x1, f0, f1)) return RT_AIM_FIRST_FAILED;
    int term = RT_AIM_MAX_ITER;
#pragma unroll 1
    for (int it = 0; it < max_iter; it++) {
        const double m = aim_norm(f0, f1);
        if (m < tol) { term = RT_AIM_CONVERGED; break; }
        double ga0, ga1, gb0, gb1;
        if (!aim_stop_xy(tab, nrow, wvl, G, f, stop, o, x0 + h, x1 + 0.0, ga0, ga1) ||
            !aim_stop_xy(tab, nrow, wvl, G, f, stop, o, x0 + 0.0, x1 + h, gb0, gb1)) {
            term = RT_AIM_DIFF_FAILED;
            break;
        }
        const double j00 = (ga0 - f0)/h, j10 = (ga1 - f1)/h, j01 = (gb0 - f0)/h, j11 = (gb1 - f1)/h;
        double s0, s1;
        if (!aim_solve2(j00, j01, j10, j11, -f0, -f1, s0, s1)) { term = RT_AIM_SINGULAR; break; }
        double lam = 1.0;
        bool accepted = false;
#pragma unroll 1
        for (int bt = 0; bt < 20; bt++) {
            const double t0 = x0 + lam*s0, t1 = x1 + lam*s1;
            double n0, n1;
            if (aim_stop_xy(tab, nrow, wvl, G, f, stop, o, t0, t1, n0, n1) && aim_norm(n0, n1) < m) {
                x0 = t0; x1 = t1; f0 = n0; f1 = n1;
                accepted = true;
                break;
            }
            lam *= 0.5;
        }
        if (!accepted) { term = RT_AIM_NO_STEP; break; }
        iters++;
    }
    aim_x = x0; aim_y = x1;
    return term;
}

}  // namespace b200rt
