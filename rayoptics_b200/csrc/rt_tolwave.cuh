/*
 * rt_tolwave.cuh -- the RT_WAVE_DOUBLES record of one traced chief ray (rt_variants_wave: the wave
 * records of every perturbed prescription of a variant set, built on the device).  Kept in a header so
 * that tests/hostsim can compile it for the host and feed it the oracle's chief rays.
 *
 * Restates, for an image gap whose interface n_ifc - 2 has no decenter, what rayoptics_b200/waveabr.py
 * does on the host: transfer_to_exit_pupil, calculate_reference_sphere (image_pt_2d = image_delta =
 * None) and wave_record, both the finite sphere and the infinite-reference branch (radius
 * is_kinda_big).  Rounding contract (DESIGN.md section 2):
 *   element-wise numpy expressions unfused, in source order;
 *   np.linalg.norm and np.dot are the ddot FMA chain (dot3); normalize divides by the norm;
 *   -h/u and foc/d_z are single IEEE divisions;
 *   |u| < 1e-14 falls back to the paraxial exit-pupil distance.
 * rt.dot(v) of the infinite branch uses the interface's own rotation; the callers only get here with
 * the identity (has_tfrm == 0), for which every summation order gives the same bits.
 */
#pragma once
#include "rt_device.cuh"

namespace b200rt {

/* misc_math.is_kinda_big */
__device__ __forceinline__ bool tolwave_kinda_big(double x)
{
    return isinf(x) || fabs(x) > 1e8;
}

/* the record W and reference image point ref[2] of a chief ray: p1 = ray[1].p, d0 = ray[0].d,
 * pk / dk = ray[-2], pl / dl = ray[-1], cr_op its optical path; foc the focus shift; last the
 * descriptor of interface n_ifc - 2 (its t[2] is the image gap's thickness, its rt / t the last
 * local transform); exp_dist, n_obj, n_img the paraxial exit-pupil distance and |indices|.  A chief
 * ray that did not reach the image (status != 0) gives NaN everywhere. */
__device__ __forceinline__ void tolwave_record(int status, const Vec3 &p1, const Vec3 &d0, const Vec3 &pk,
                                               const Vec3 &dk, const Vec3 &pl, const Vec3 &dl, double cr_op,
                                               double foc, const rt_surface_desc &last, double exp_dist,
                                               double n_obj, double n_img, double *__restrict__ W,
                                               double *__restrict__ ref)
{
    if (status != RT_RAY_OK) {
        for (int k = 0; k < RT_WAVE_DOUBLES; k++) W[k] = (double)NAN;
        ref[0] = (double)NAN; ref[1] = (double)NAN;
        return;
    }
    /* transfer_to_exit_pupil */
    const double h = pk.y, u = dk.y;
    const double exp_dst = fabs(u) < 1e-14 ? exp_dist : -h/u;
    const Vec3 exp_pt = {pk.x + exp_dst*dk.x, pk.y + exp_dst*dk.y, pk.z + exp_dst*dk.z};
    /* calculate_reference_sphere */
    const double dist = foc/dl.z;
    const Vec3 image_pt = {pl.x + dist*dl.x, pl.y + dist*dl.y, pl.z + dist*dl.z};
    const double image_thi = last.t[2];
    const Vec3 v = {image_pt.x - exp_pt.x, image_pt.y - exp_pt.y, (image_pt.z + image_thi) - exp_pt.z};
    const double radius = sqrt(dot3(v, v));
    ref[0] = image_pt.x; ref[1] = image_pt.y;
    W[22] = n_obj; W[23] = n_img;
    W[0] = p1.x; W[1] = p1.y; W[2] = p1.z;
    W[3] = d0.x; W[4] = d0.y; W[5] = d0.z;
    if (tolwave_kinda_big(radius)) {
        /* wave_abr_full_calc_inf_ref: p_cr_b4 = rt.(ray[-2].p - t), d_cr_b4 = rt.ray[-2].d */
        const double *r = last.rt;
        const Vec3 q = {pk.x - last.t[0], pk.y - last.t[1], pk.z - last.t[2]};
        const Vec3 r0 = {r[0], r[1], r[2]}, r1 = {r[3], r[4], r[5]}, r2 = {r[6], r[7], r[8]};
        const Vec3 p_cr_b4 = {dot3(r0, q), dot3(r1, q), dot3(r2, q)};
        const Vec3 d_cr_b4 = {dot3(r0, dk), dot3(r1, dk), dot3(r2, dk)};
        const Vec3 mp = {-p_cr_b4.x, -p_cr_b4.y, -p_cr_b4.z};
        const double op_cr_b4 = dot3(d_cr_b4, mp);
        W[6] = pl.x; W[7] = pl.y; W[8] = pl.z;
        W[9] = dl.x; W[10] = dl.y; W[11] = dl.z;
        W[12] = cr_op + op_cr_b4;
        W[13] = image_pt.x; W[14] = image_pt.y; W[15] = image_pt.z;
        W[16] = 0.0;
        W[17] = d_cr_b4.x; W[18] = d_cr_b4.y; W[19] = d_cr_b4.z;
        W[20] = last.t[2];
        W[21] = 0.0;                     /* flag: infinite-reference variant */
        return;
    }
    const Vec3 ref_dir = radius == 0.0 ? v : Vec3{v.x/radius, v.y/radius, v.z/radius};
    W[6] = pk.x; W[7] = pk.y; W[8] = pk.z;
    W[9] = dk.x; W[10] = dk.y; W[11] = dk.z;
    W[12] = cr_op;
    W[13] = exp_pt.x; W[14] = exp_pt.y; W[15] = exp_pt.z;
    W[16] = exp_dst;
    W[17] = ref_dir.x; W[18] = ref_dir.y; W[19] = ref_dir.z;
    W[20] = radius;
    W[21] = ref_dir.z*dl.z < 0 ? -1.0 : 1.0;
}

}  // namespace b200rt
