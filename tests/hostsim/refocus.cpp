/*
 * tests/hostsim/refocus.cpp -- TEST INFRASTRUCTURE (see cuda_runtime.h here).
 * rayoptics_b200/csrc/rt_refocus.cuh compiled for the host, in a library of its own: the OPD of one
 * ray against many reference spheres, split as k_trace_grid[_lean]_opd_focus splits it, for
 * tests/test_through_focus_wavefront.py and the GPU file that checks the device against it.
 */
#define RT_HOSTSIM 1
#include "cuda_runtime.h"
#include "../../rayoptics_b200/csrc/rt_refocus.cuh"

using namespace b200rt;

extern "C" {

/* ray: p1, d0, pk, dk, pl, dl (18 doubles) of one traced ray; W its tile's RT_WAVE_DOUBLES record;
 * spheres [n][RT_SPHERE_DOUBLES] -> out [n]: refocus_pre once, refocus_opd per sphere */
int hostsim_refocus(const double *W, const double *ray, double ray_op, const double *spheres, int n, double *out)
{
    const Vec3 v[6] = {{ray[0], ray[1], ray[2]}, {ray[3], ray[4], ray[5]}, {ray[6], ray[7], ray[8]},
                       {ray[9], ray[10], ray[11]}, {ray[12], ray[13], ray[14]}, {ray[15], ray[16], ray[17]}};
    const RefocusRay q = refocus_pre(W, v[0], v[1], v[2], v[3], v[4], v[5], ray_op);
    for (int k = 0; k < n; k++) out[k] = refocus_opd(q, spheres + (int64_t)k*RT_SPHERE_DOUBLES);
    return 0;
}

}
