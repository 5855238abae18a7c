/*
 * tests/hostsim/aim.cpp -- TEST INFRASTRUCTURE (see cuda_runtime.h here).
 * rayoptics_b200/csrc/rt_aim.cuh compiled for the host, in a library of its own: the chief-ray
 * aiming of k_aim_chief field by field, for tests/test_field_map.py.
 */
#define RT_HOSTSIM 1
#include "cuda_runtime.h"
#include "../../rayoptics_b200/csrc/rt_aim.cuh"

using namespace b200rt;

extern "C" {

/* aim_chief_ray for every field of the grid described by g (pupil_kind RT_PUPIL_EPD), with the
 * options rt_grid_aim_chief passes.  aim: [n_fields][2]; term, iters: [n_fields]. */
int hostsim_aim_chief(const rt_surface_desc *surfs, int n_ifc, const double *n_by_wvl, const double *wvls,
                      const rt_grid_spec *g, int stop, int wvl_idx, double h, double tol, int max_iter,
                      double *aim, int32_t *term, int32_t *iters)
{
    if (g->pupil_kind != RT_PUPIL_EPD || stop < 1 || stop > n_ifc - 2) return -1;
    GridDev G;
    G.n_wvls = g->n_wvls; G.nx = g->nx; G.ny = g->ny;
    G.apply_vignetting = g->apply_vignetting; G.flip_z_dir = g->flip_z_dir; G.paired = g->paired;
    G.eprad = g->eprad; G.z_pupil = g->z_pupil; G.foc = g->foc;
    G.fields = g->fields; G.wvl_idx = g->wvl_idx;
    G.pupil_x = g->pupil_x; G.pupil_y = g->pupil_y; G.ref_img = g->ref_img; G.wave = g->wave;
    G.rays_per_tile = (int64_t)g->nx*g->ny; G.chunks_per_tile = 0;
    rt_opts o;
    o.eps = 1.0e-12; o.pt_inside_fuzz = -1.0; o.check_apertures = 0; o.intersect_obj = 1;
    o.filter_out_phantoms = 0; o.first_surf = 1; o.last_surf = stop; o.wvl_idx = wvl_idx;
    for (int f = 0; f < g->n_fields; f++) {
        int it = 0;
        term[f] = aim_chief_ray(surfs, n_by_wvl + (int64_t)wvl_idx*n_ifc, wvls ? wvls[wvl_idx] : 0.0, G, f, stop, o,
                                h, tol, max_iter, aim[2*f], aim[2*f + 1], it);
        iters[f] = it;
    }
    return 0;
}

}
