/*
 * tests/hostsim/tolwave.cpp -- TEST INFRASTRUCTURE (see cuda_runtime.h here).
 * rayoptics_b200/csrc/rt_tolwave.cuh compiled for the host, in a library of its own: the wave record of
 * one traced chief ray as k_variants_wave forms it, for tests/test_tolerance_wavefront.py.
 */
#define RT_HOSTSIM 1
#include "cuda_runtime.h"
#include "../../rayoptics_b200/csrc/rt_tolwave.cuh"

using namespace b200rt;

extern "C" {

/* n chief rays: ray [n][18] = p1, d0, pk, dk, pl, dl; op, status [n]; last: the descriptor of interface
 * n_ifc - 2; parax [3] -> W [n][RT_WAVE_DOUBLES], ref [n][2]; branch [n]: 1 infinite reference, 2 finite
 * with the paraxial exit-pupil fallback (|u| < 1e-14), 0 otherwise */
int hostsim_tolwave(int64_t n, const double *ray, const double *op, const int32_t *status,
                    const rt_surface_desc *last, double foc, const double *parax, double *W, double *ref,
                    int32_t *branch)
{
    for (int64_t i = 0; i < n; i++) {
        const double *r = ray + i*18;
        const Vec3 v[6] = {{r[0], r[1], r[2]}, {r[3], r[4], r[5]}, {r[6], r[7], r[8]},
                           {r[9], r[10], r[11]}, {r[12], r[13], r[14]}, {r[15], r[16], r[17]}};
        double *w = W + i*RT_WAVE_DOUBLES;
        tolwave_record(status[i], v[0], v[1], v[2], v[3], v[4], v[5], op[i], foc, *last, parax[0], parax[1],
                       parax[2], w, ref + i*2);
        branch[i] = status[i] != 0 ? 0 : (w[21] == 0.0 ? 1 : (std::fabs(v[3].y) < 1e-14 ? 2 : 0));
    }
    return 0;
}

}
