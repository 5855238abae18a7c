/*
 * rt_grid.cuh -- device-side description of a pupil grid and the generation of its
 * start rays (Field.apply_vignetting + ray_start_from_osp + the virtual-object flip of
 * trace_base; /root/reference/src/rayoptics/raytr/opticalspec.py:289-400,1339-1353,
 * raytr/trace.py:289-308).  Kept in a header so that tests/hostsim can compile it for
 * the host next to the per-ray code.
 */
#pragma once
#include "rt_device.cuh"

namespace b200rt {

struct GridDev {
    int32_t n_wvls, nx, ny, apply_vignetting, flip_z_dir, paired;
    double eprad, z_pupil, foc;
    const rt_field_desc *fields;
    const int32_t *wvl_idx;
    const double *pupil_x, *pupil_y, *ref_img, *wave;
    int64_t rays_per_tile, chunks_per_tile;
};

/* angular pupil specifications ('NA', 'f/#' in object space), opticalspec.py:368-398.
 * Out of line: the spatial ('epd') branch is the one every bundled model takes and it
 * keeps its code.  (pupil*slope)**2 is libm pow() in the reference, a product here:
 * tolerance parity for RT_PUPIL_FNO, bit-exact for RT_PUPIL_NA. */
__device__ __noinline__ void angular_start_dir(int pupil_kind, double scale, double pupx, double pupy,
                                               double crx, double cry, double *d /* [3] */)
{
    double pdx, pdy;
    if (pupil_kind == RT_PUPIL_NA) {
        pdx = scale*pupx; pdy = scale*pupy;
    } else {
        const double sx = pupx*scale, sy = pupy*scale;
        double hypt = sqrt(1 + sx*sx + sy*sy);
        pdx = scale*pupx/hypt; pdy = scale*pupy/hypt;
    }
    d[0] = pdx + crx; d[1] = pdy + cry;
    d[2] = sqrt(1 - __fma_rn(d[1], d[1], d[0]*d[0]));
}

/* start ray of grid ray (tile, loc).  pupil_kind (rt_pupil_kind) is a separate kernel
 * argument of the general kernels: the lean kernels are only launched for RT_PUPIL_EPD
 * grids (rt_trace_grid routes angular pupils to the general kernels), and keeping it
 * out of GridDev leaves their parameter layout -- and code -- untouched. */
template <bool LEAN>
__device__ __forceinline__ void grid_start_ray_at(const GridDev &G, int pupil_kind, int f, double pupx,
                                                  double pupy, bool apply_vignetting, Vec3 &p0, Vec3 &d0)
{
    const rt_field_desc &F = G.fields[f];
    /* Field.apply_vignetting, opticalspec.py:1339-1353 */
    if (apply_vignetting) {
        const double vlx = F.vlx, vux = F.vux, vly = F.vly, vuy = F.vuy;
        if (pupx < 0.0) { if (vlx != 0.0) pupx *= (1.0 - vlx); }
        else            { if (vux != 0.0) pupx *= (1.0 - vux); }
        if (pupy < 0.0) { if (vly != 0.0) pupy *= (1.0 - vly); }
        else            { if (vuy != 0.0) pupy *= (1.0 - vuy); }
    }
    p0.x = F.pt0[0]; p0.y = F.pt0[1]; p0.z = F.pt0[2];
    if (LEAN || pupil_kind == RT_PUPIL_EPD) {
        /* ray_start_from_osp 'epd' branch, opticalspec.py:354-366 */
        Vec3 pt1 = {G.eprad*pupx + F.aim[0], G.eprad*pupy + F.aim[1], G.z_pupil};
        Vec3 dv = {pt1.x - p0.x, pt1.y - p0.y, pt1.z - p0.z};
        d0 = LEAN ? normalize3_shared(dv) : normalize3(dv);
    } else if (pupil_kind == RT_PUPIL_WIDE) {
        /* wide-angle fields, opticalspec.py:342-358: pt1 = matmul(rot_d2s, eprad*[px, py, 0]),
         * pt1[2] -= obj2enp_dist, dir0 = normalize(pt1 - pt0).  rot is C-contiguous in numpy:
         * its matmul with a 3-vector rounds as fma(a2,v2, fma(a0,v0, a1*v1)) (table.py has_tfrm 2) */
        const double *a = F.rot;
        const double vx = G.eprad*pupx, vy = G.eprad*pupy, vz = G.eprad*0.0;
        Vec3 pt1 = {__fma_rn(a[2], vz, __fma_rn(a[0], vx, a[1]*vy)),
                    __fma_rn(a[5], vz, __fma_rn(a[3], vx, a[4]*vy)),
                    __fma_rn(a[8], vz, __fma_rn(a[6], vx, a[7]*vy))};
        pt1.z -= F.obj2enp;
        Vec3 dv = {pt1.x - p0.x, pt1.y - p0.y, pt1.z - p0.z};
        d0 = normalize3(dv);
    } else {
        double d[3];
        angular_start_dir(pupil_kind, G.eprad, pupx, pupy, F.aim[0], F.aim[1], d);
        d0.x = d[0]; d0.y = d[1]; d0.z = d[2];
    }
    /* trace_base virtual-object flip, trace.py:305-308 */
    if (d0.z*(double)G.flip_z_dir < 0) { d0.x = -d0.x; d0.y = -d0.y; d0.z = -d0.z; }
}

/* the start ray of grid_start_ray_at<false> for RT_PUPIL_EPD without vignetting, aimed at
 * (aim_x, aim_y) in place of the field's aim: the same expressions (rt_aim.cuh's trial rays) */
__device__ __forceinline__ void epd_start_ray_aimed(const GridDev &G, int f, double pupx, double pupy,
                                                    double aim_x, double aim_y, Vec3 &p0, Vec3 &d0)
{
    const rt_field_desc &F = G.fields[f];
    p0.x = F.pt0[0]; p0.y = F.pt0[1]; p0.z = F.pt0[2];
    Vec3 pt1 = {G.eprad*pupx + aim_x, G.eprad*pupy + aim_y, G.z_pupil};
    Vec3 dv = {pt1.x - p0.x, pt1.y - p0.y, pt1.z - p0.z};
    d0 = normalize3(dv);
    if (d0.z*(double)G.flip_z_dir < 0) { d0.x = -d0.x; d0.y = -d0.y; d0.z = -d0.z; }
}

template <bool LEAN>
__device__ __forceinline__ void grid_start_ray(const GridDev &G, int pupil_kind, int f, int64_t loc,
                                               Vec3 &p0, Vec3 &d0)
{
    const int i = (int)(loc/G.ny), j = (int)(loc - (int64_t)i*G.ny);
    const double pupx = G.pupil_x[(int64_t)f*G.nx + i];
    const double pupy = G.paired ? G.pupil_y[(int64_t)f*G.nx + i] : G.pupil_y[(int64_t)f*G.ny + j];
    grid_start_ray_at<LEAN>(G, pupil_kind, f, pupx, pupy, G.apply_vignetting != 0, p0, d0);
}

/* relative pupil coordinates of grid ray (tile, loc) as grid_start_ray uses them: pupil_x[i] and
 * pupil_y[j] (product grid) or pupil_y[i] (ray list) of field f, after Field.apply_vignetting
 * when the grid applies it */
__device__ __forceinline__ void grid_pupil_coords(const GridDev &G, int f, int64_t loc, double &pupx, double &pupy)
{
    const int i = (int)(loc/G.ny), j = (int)(loc - (int64_t)i*G.ny);
    pupx = G.pupil_x[(int64_t)f*G.nx + i];
    pupy = G.paired ? G.pupil_y[(int64_t)f*G.nx + i] : G.pupil_y[(int64_t)f*G.ny + j];
    if (G.apply_vignetting) {
        const rt_field_desc &F = G.fields[f];
        const double vlx = F.vlx, vux = F.vux, vly = F.vly, vuy = F.vuy;
        if (pupx < 0.0) { if (vlx != 0.0) pupx *= (1.0 - vlx); }
        else            { if (vux != 0.0) pupx *= (1.0 - vux); }
        if (pupy < 0.0) { if (vly != 0.0) pupy *= (1.0 - vly); }
        else            { if (vuy != 0.0) pupy *= (1.0 - vuy); }
    }
}

}  // namespace b200rt
