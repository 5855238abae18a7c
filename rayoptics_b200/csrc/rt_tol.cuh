/*
 * rt_tol.cuh -- the per-work-item record of rt_trace_grid_variants (tolerance analysis: many
 * perturbed prescriptions traced over one pupil grid).  The summands are kept host-compilable so
 * that tests/hostsim can form them from oracle-traced rays.
 *
 * Record (RT_TOL_DOUBLES), per work item of 32 rays in scratch and per (variant, tile) after
 * k_reduce_tol (DESIGN.md section 4):
 *   0-15  rt_trace_grid's summary layout: 0-4 counts by status class, 5-9 sum ax, ay, ax*ax, ay*ay,
 *         ax*ay, 10-13 min / max ax, ay, 14 sum op, 15 zero
 *   16-21 sum ux, uy, ux*ux, uy*uy, ax*ux, ay*uy with ux = dx/dz, uy = dy/dz of the last segment
 *   22    valid flag (scratch records; 0 in the reduced record)   23 zero
 * Only status-0 rays enter columns 5-21.  Every product is rounded once; the 12 sums of an item
 * are added by the halving tree of wfe_item_sums_store (x[i] + x[i+16], +8, +4, +2, +1), then
 * reduce_tile adds a tile's items in item order.  The spot sums are thus added exactly as
 * rt_trace_grid adds them, in either of its regimes.
 */
#pragma once
#include "rt_device.cuh"

namespace b200rt {

#define RT_TOL_ITEM_SUMS 12
#define RT_TOL_VALID 22

/* record column of sum j of tol_summands */
__host__ __device__ __forceinline__ constexpr int tol_sum_col(int j) { return j < 5 ? 5 + j : (j == 5 ? 14 : 10 + j); }

/* the 12 summands of one status-0 ray in tol_sum_col order: ax, ay, ax*ax, ay*ay, ax*ay, op, ux, uy,
 * ux*ux, uy*uy, ax*ux, ay*uy */
__host__ __device__ __forceinline__ void tol_summands(double ax, double ay, double op, const Vec3 &d,
                                                      double v[RT_TOL_ITEM_SUMS])
{
    const double ux = d.x/d.z, uy = d.y/d.z;
    v[0] = ax; v[1] = ay; v[2] = ax*ax; v[3] = ay*ay; v[4] = ax*ay; v[5] = op;
    v[6] = ux; v[7] = uy; v[8] = ux*ux; v[9] = uy*uy; v[10] = ax*ux; v[11] = ay*uy;
}

#ifdef __CUDACC__
/* the 16-value transposition of wfe_item_sums_store: after the 16 / 8 / 4 / 2 / 1 exchanges, even
 * lane 2g holds the warp sum of value 8*[bit 4] + 4*[bit 3] + 2*[bit 2] + [bit 1] of g = lane/2 */
__device__ __forceinline__ double item_sums16(const double (&v)[16], int lane)
{
    const bool h16 = lane & 16, h8 = lane & 8, h4 = lane & 4, h2 = lane & 2;
    double a[8];
#pragma unroll
    for (int k = 0; k < 8; k++)
        a[k] = (h16 ? v[8 + k] : v[k]) + __shfl_xor_sync(0xffffffffu, h16 ? v[k] : v[8 + k], 16);
    double b[4];
#pragma unroll
    for (int k = 0; k < 4; k++)
        b[k] = (h8 ? a[4 + k] : a[k]) + __shfl_xor_sync(0xffffffffu, h8 ? a[k] : a[4 + k], 8);
    const double c0 = (h4 ? b[2] : b[0]) + __shfl_xor_sync(0xffffffffu, h4 ? b[0] : b[2], 4);
    const double c1 = (h4 ? b[3] : b[1]) + __shfl_xor_sync(0xffffffffu, h4 ? b[1] : b[3], 4);
    double e = (h2 ? c1 : c0) + __shfl_xor_sync(0xffffffffu, h2 ? c0 : c1, 2);
    return e + __shfl_xor_sync(0xffffffffu, e, 1);
}

/* one work item's whole record (every column written, so scratch needs no clearing):
 * the sums by item_sums16, the counts by ballots, min / max ax, ay in 6 shuffles */
__device__ __forceinline__ void tol_item(bool have, int status, double ax, double ay, double op, const Vec3 &d,
                                         double *__restrict__ dst)
{
    const int lane = threadIdx.x & 31;
    const bool ok = have && status == RT_RAY_OK;
    double v[16];
    tol_summands(ax, ay, op, d, v);
    v[12] = 0.0; v[13] = 0.0; v[14] = 0.0; v[15] = 0.0;
#pragma unroll
    for (int k = 0; k < RT_TOL_ITEM_SUMS; k++) v[k] = ok ? v[k] : 0.0;
    const double e = item_sums16(v, lane);
    const int idx = ((lane >> 4) & 1)*8 + ((lane >> 3) & 1)*4 + ((lane >> 2) & 1)*2 + ((lane >> 1) & 1);
    if ((lane & 1) == 0 && idx < RT_TOL_ITEM_SUMS) dst[tol_sum_col(idx)] = e;
    /* min / max: the lower half-warp reduces ax, the upper ay; lanes 0 / 8 / 16 / 24 hold
     * min ax / max ax / min ay / max ay */
    const bool h16 = lane & 16, h8 = lane & 8;
    const double v0 = ok ? ax : CUDART_INF, v1 = ok ? ax : -CUDART_INF;
    const double v2 = ok ? ay : CUDART_INF, v3 = ok ? ay : -CUDART_INF;
    const double a0 = fmin(h16 ? v2 : v0, __shfl_xor_sync(0xffffffffu, h16 ? v0 : v2, 16));
    const double a1 = fmax(h16 ? v3 : v1, __shfl_xor_sync(0xffffffffu, h16 ? v1 : v3, 16));
    double b = __shfl_xor_sync(0xffffffffu, h8 ? a0 : a1, 8);
    b = h8 ? fmax(a1, b) : fmin(a0, b);
#pragma unroll
    for (int s = 4; s > 0; s >>= 1) {
        const double y = __shfl_xor_sync(0xffffffffu, b, s);
        b = h8 ? fmax(b, y) : fmin(b, y);
    }
    if ((lane & 7) == 0) dst[10 + (lane >> 3)] = b;
    /* odd lanes 1..9: the counts of status classes 0..4; 11: valid flag; 13, 15: the zero columns */
    const int ck = status == RT_RAY_OK ? 0 : (status <= RT_RAY_BLOCKED ? status : 4);
    double cnt = 0.0;
#pragma unroll
    for (int c = 0; c < 5; c++) {
        const unsigned m = __ballot_sync(0xffffffffu, have && ck == c);
        if (lane == 2*c + 1) cnt = (double)__popc(m);
    }
    if ((lane & 1) && lane <= 9) dst[lane >> 1] = cnt;
    if (lane == 11) dst[RT_TOL_VALID] = 1.0;
    if (lane == 13) dst[15] = 0.0;
    if (lane == 15) dst[23] = 0.0;
}
#endif

}  // namespace b200rt
