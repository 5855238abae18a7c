/*
 * rt_refocus.cuh -- the OPD of one traced ray against many reference spheres
 * (rt_trace_grid_opd_focus).  Kept in a header so that tests/hostsim can compile it for the host.
 *
 * Refocusing moves only the reference sphere, so the OPD splits as the reference's rapid-refocus
 * route splits it (raytr/waveabr.py: wave_abr_pre_calc / wave_abr_calc, :226-253, 310-353,
 * 427-488; restated in rayoptics_b200/waveabr.py): refocus_pre once per ray, refocus_opd once per
 * sphere.  Contract (DESIGN.md section 4):
 *   finite sphere: pre_opd = -n_obj*e1 - ray_op + n_img*ekp + cr_op, the expression order of
 *     wave_opd, so the tile's own sphere gives wave_opd's bits; F*F stands for the reference's F**2;
 *   infinite reference: pre_opd = -n_obj*e1 - W0, opd = pre_opd - n_img*numer/denom, which rounds
 *     like the reference's focus_wavefront, not like wave_abr_full_calc_inf_ref;
 *   every division is an IEEE division (no reciprocal of R is shared).
 * Sphere record S (RT_SPHERE_DOUBLES): 0-2 ref_dir, 3 ref_sphere_radius, 4 sign_soln (0 on tiles of
 * the infinite-reference variant), 5-7 image_pt.  The variant is the tile's: W[21] == 0.
 */
#pragma once
#include "rt_device.cuh"

namespace b200rt {

/* what refocus_opd needs of one ray: finite -> a = p_coord, b = b4_dir, s0 = dot(b4_dir, p_coord),
 * s1 = dot(p_coord, p_coord); infinite -> a = d_cr_b4 - d_b4*dot(d_b4, d_cr_b4), b = ray[-1].p,
 * s0 = 1 + dot(d_b4, d_cr_b4) */
struct RefocusRay {
    Vec3 a, b;
    double pre_opd, s0, s1, n_img;
    bool inf;
};

__device__ __forceinline__ RefocusRay refocus_pre(const double *__restrict__ W, const Vec3 &p1, const Vec3 &d0,
                                                  const Vec3 &pk, const Vec3 &dk, const Vec3 &pl,
                                                  const Vec3 &dl, double ray_op)
{
    RefocusRay q;
    const double n_obj = W[22], n_img = W[23];
    q.n_img = n_img;
    q.inf = W[21] == 0.0;
    if (q.inf) {
        double e1;
        const double W0 = inf_ref_w0(W, p1, d0, pl, dl, pk.x, pk.y, pk.z, dk, ray_op, e1);
        const Vec3 d_cr_b4 = {W[17], W[18], W[19]};
        const double dbc = dot3(dk, d_cr_b4);
        q.a = {d_cr_b4.x - dk.x*dbc, d_cr_b4.y - dk.y*dbc, d_cr_b4.z - dk.z*dbc};
        q.b = pl;
        q.s0 = 1 + dot3(dk, d_cr_b4);
        q.s1 = 0.0;
        q.pre_opd = -n_obj*e1 - W0;
        return q;
    }
    const Vec3 cr_p1 = {W[0], W[1], W[2]}, cr_d0 = {W[3], W[4], W[5]};
    const Vec3 cr_pk = {W[6], W[7], W[8]}, cr_dk = {W[9], W[10], W[11]};
    const double cr_op = W[12], cr_exp_dist = W[16];
    const Vec3 cr_exp_pt = {W[13], W[14], W[15]};
    const double e1 = eic_distance(p1, d0, cr_p1, cr_d0);
    const double ekp = eic_distance(pk, dk, cr_pk, cr_dk);
    const double dst = ekp - cr_exp_dist;
    const Vec3 eic_exp_pt = {pk.x - dst*dk.x, pk.y - dst*dk.y, pk.z - dst*dk.z};
    q.a = {eic_exp_pt.x - cr_exp_pt.x, eic_exp_pt.y - cr_exp_pt.y, eic_exp_pt.z - cr_exp_pt.z};
    q.b = dk;
    q.s0 = dot3(dk, q.a);
    q.s1 = dot3(q.a, q.a);
    q.pre_opd = -n_obj*e1 - ray_op + n_img*ekp + cr_op;
    return q;
}

/* the OPD of the ray of refocus_pre against the sphere record S */
__device__ __forceinline__ double refocus_opd(const RefocusRay &q, const double *__restrict__ S)
{
    if (q.inf) {
        const Vec3 ta = {q.b.x - S[5], q.b.y - S[6], q.b.z - S[7]};
        const double numer = dot3(q.a, ta);
        return q.pre_opd - q.n_img*numer/q.s0;
    }
    const Vec3 ref_dir = {S[0], S[1], S[2]};
    const double R = S[3], sign_soln = S[4];
    const double F = dot3(ref_dir, q.b) - q.s0/R;
    const double J = q.s1/R - 2.0*dot3(ref_dir, q.a);
    const double denom = F + sign_soln*sqrt(F*F + J/R);
    const double ep = (denom == 0.0) ? 0.0 : J/denom;
    return q.pre_opd - q.n_img*ep;
}

}  // namespace b200rt
