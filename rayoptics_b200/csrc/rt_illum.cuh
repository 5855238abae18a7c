/*
 * rt_illum.cuh -- the per-ray terms and ordered sums of rt_grid_illumination (relative illumination).
 * Kept in a header so that tests/hostsim can compile it for the host.
 *
 * Contract (DESIGN.md section 4), restated in numpy by engine.illumination_sums_host.  Each tile is an
 * n x n product grid of relative pupil coordinates (x[i], y[j]); per ray the trace gives its status
 * and the direction cosines L, M of its last segment.  The projected solid angle of the image-space
 * beam is Omega = integral over the unit disk of |d(L, M)/d(x, y)| dx dy, summed as:
 *   a ray is used when its status is 0 and x*x + y*y <= 1 (illum_used);
 *   for F in {L, M} its derivative along x is central (F[i+1] - F[i-1])/(x[i+1] - x[i-1]) when rays
 *   i-1 and i+1 both exist with status 0, else forward (F[i+1] - F[i])/(x[i+1] - x[i]) when ray i+1
 *   does, else backward (F[i] - F[i-1])/(x[i] - x[i-1]) when ray i-1 does, else it is not formed;
 *   the same along y (illum_deriv);
 *   J = Lx*My - Ly*Mx with each product rounded once (the library is built with -fmad=false and
 *   nothing here uses __fma_rn); a used ray with a derivative not formed is isolated and adds nothing;
 *   |J| and J of each column j are added along i in increasing i from +0.0 (illum_term), and the
 *   column sums in increasing j from +0.0 (illum_line_sum).
 */
#pragma once
#include <cuda_runtime.h>

namespace b200rt {

/* which difference illum_deriv formed */
enum { ILLUM_CENTRAL = 0, ILLUM_FORWARD = 1, ILLUM_BACKWARD = 2, ILLUM_NONE = 3 };

/* a neighbour of a ray along one pupil axis: its L, M, and ok when it exists and has status 0 */
struct IllumPt {
    double L, M;
    bool ok;
};

/* sum |J| and sum J of one column */
struct IllumAcc {
    double abs_j, j;
};

__device__ __forceinline__ bool illum_used(int status, double x, double y)
{
    return status == 0 && x*x + y*y <= 1.0;
}

/* dL/du and dM/du at the ray c (coordinate u0) from its neighbours m (u_m) and p (u_p) along one axis */
__device__ __forceinline__ int illum_deriv(IllumPt m, IllumPt c, IllumPt p, double u_m, double u0, double u_p,
                                           double *dL, double *dM)
{
    if (m.ok && p.ok) {
        const double h = u_p - u_m;
        *dL = (p.L - m.L)/h;
        *dM = (p.M - m.M)/h;
        return ILLUM_CENTRAL;
    }
    if (p.ok) {
        const double h = u_p - u0;
        *dL = (p.L - c.L)/h;
        *dM = (p.M - c.M)/h;
        return ILLUM_FORWARD;
    }
    if (m.ok) {
        const double h = u0 - u_m;
        *dL = (c.L - m.L)/h;
        *dM = (c.M - m.M)/h;
        return ILLUM_BACKWARD;
    }
    return ILLUM_NONE;
}

/* J = Lx*My - Ly*Mx, each product rounded once */
__device__ __forceinline__ double illum_jacobian(double Lx, double Ly, double Mx, double My)
{
    const double a = Lx*My, b = Ly*Mx;
    return a - b;
}

/* The term of a used ray c at (x0, y0) with its neighbours xm, xp along x (at x_m, x_p) and ym, yp along
 * y: |J| and J added to its column's chains.  Returns false, adding nothing, when the ray is isolated. */
__device__ __forceinline__ bool illum_term(IllumAcc &acc, IllumPt c, IllumPt xm, IllumPt xp, IllumPt ym, IllumPt yp,
                                           double x_m, double x0, double x_p, double y_m, double y0, double y_p)
{
    double Lx, Mx, Ly, My;
    if (illum_deriv(xm, c, xp, x_m, x0, x_p, &Lx, &Mx) == ILLUM_NONE) return false;
    if (illum_deriv(ym, c, yp, y_m, y0, y_p, &Ly, &My) == ILLUM_NONE) return false;
    const double J = illum_jacobian(Lx, Ly, Mx, My);
    acc.abs_j = acc.abs_j + fabs(J);
    acc.j = acc.j + J;
    return true;
}

/* sum over k = 0 ... n-1 of v[k], in increasing k from +0.0 (the column sums of a tile) */
__device__ __forceinline__ double illum_line_sum(const double *v, int n)
{
    double acc = 0.0;
    for (int k = 0; k < n; k++) acc = acc + v[k];
    return acc;
}

}  // namespace b200rt
