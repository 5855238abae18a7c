/*
 * b200rt.cu -- kernels and C ABI of libb200rt.so (see include/b200rt.h).
 *
 * Kernels (sm_90a, H100; fp64 vector pipe + coalesced SoA global traffic; no tensor
 * cores -- the path is not a contraction):
 *   k_trace_bundle<FULL,STAGE>  one ray per lane over caller-supplied start rays
 *   k_trace_grid<FULL,SUMMARY,STAGE>  start rays generated on device from the
 *                               (field, wavelength, pupil i, j) index, optional
 *                               per-chunk spot sums
 *   k_trace_grid[_lean]_focus   one trace, spot sums at up to RT_MAX_FOCUS image planes
 *   k_trace_grid[_lean]_wfe     one trace, per-tile sums of the OPD and its least-squares fits
 *   k_reduce_summary            fixed-order per-tile reduction of the chunk sums (_wfe: of the
 *                               wavefront-error sums)
 *   k_zernike_moments<ROWS>     per-chunk Gram matrix of [OPD, Fringe Zernike terms] from a grid
 *                               trace's per-ray opd / status; k_reduce_zernike adds the chunks
 *   k_aim_chief                 chief-ray aiming: the Newton iteration of rt_aim.cuh, one thread
 *                               per field
 *   k_pupil_function, k_mtf     pupil function of a grid trace's per-ray opd / status, and its
 *                               autocorrelation along both pupil axes, at every or at listed
 *                               shifts (rt_mtf.cuh)
 *   k_trace_grid[_lean]_opd_focus  one trace, the OPD of every ray against up to RT_MAX_FOCUS
 *                               reference spheres (rt_refocus.cuh)
 *   k_trace_grid_variants       the whole grid traced once per perturbed prescription of a
 *                               variant set, per-item records (rt_tol.cuh); k_reduce_tol
 *   k_variants_wave             the chief ray and wave record of every (variant, tile), one thread
 *                               each (rt_tolwave.cuh)
 *   k_trace_grid_variants_wfe   k_trace_grid_variants with the OPD epilogue against each variant's
 *                               wave records, per-item wavefront-error records; k_reduce_variants_wfe
 *   k_illumination              projected solid angle of every tile from a grid trace's per-ray
 *                               status and last directions, one CTA cluster per tile (rt_illum.cuh)
 *   k_dfma_peak                 fp64 FMA microbenchmark (roofline denominator)
 *
 * The surface table (n_ifc x rt_surface_desc + n_wvl x n_ifc indices) is staged
 * into shared memory once per CTA; CTAs are persistent (grid = SMs x resident
 * CTAs) and walk rays / chunks with a grid stride.
 */
#include <cuda_runtime.h>
#include <math_constants.h>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "rt_device.cuh"
#include "rt_lean.cuh"
#include "rt_grid.cuh"
#include "rt_zernike.cuh"
#include "rt_aim.cuh"
#include "rt_mtf.cuh"
#include "rt_refocus.cuh"
#include "rt_tol.cuh"
#include "rt_tolwave.cuh"
#include "rt_illum.cuh"
#include <cooperative_groups.h>

namespace cg = cooperative_groups;

using namespace b200rt;

#ifndef RT_BLOCK
#define RT_BLOCK 256          /* threads per CTA = rays per chunk */
#endif
#ifndef RT_LEAN_MIN_CTAS
#define RT_LEAN_MIN_CTAS 3   /* resident CTAs per SM the lean kernels are register-limited for */
#endif
#define RT_MAX_STAGE_BYTES (200*1024)

/* ------------------------------------------------------------------ errors */
static thread_local std::string g_err;
static thread_local int g_last_grid = 0;      /* CTAs of the grid kernel this thread launched last */
static thread_local int64_t g_item_off = 0;   /* doubles from scratch to the per-item sums (set by rt_trace_grid) */
static std::atomic<int64_t> g_launches{0};

static int fail(int code, const char *fmt, const char *a = "", const char *b = "")
{
    char buf[512];
    snprintf(buf, sizeof buf, fmt, a, b);
    g_err = buf;
    return code;
}

#define CUDA_TRY(expr)                                                            \
    do {                                                                          \
        cudaError_t e_ = (expr);                                                  \
        if (e_ != cudaSuccess)                                                    \
            return fail(RT_ERR_CUDA, "%s: %s", #expr, cudaGetErrorString(e_));    \
    } while (0)

struct DeviceGuard {
    int prev = -1;
    bool changed = false;
    explicit DeviceGuard(int dev)
    {
        if (cudaGetDevice(&prev) == cudaSuccess && prev != dev) {
            cudaSetDevice(dev);
            changed = true;
        }
    }
    ~DeviceGuard()
    {
        if (changed) cudaSetDevice(prev);
    }
};

/* ------------------------------------------------------------------ handles */
struct rt_table {
    int32_t device, n_ifc, n_wvl, sm_count;
    rt_surface_desc *d_surfs;
    double *d_n;
    double *d_wvl;           /* [n_wvl] wavelengths in nm (NaN until rt_table_set_wavelengths) */
    bool has_phase;
    size_t stage_bytes;      /* shared memory needed to stage the table */
    bool stage;              /* false: table too large, read it from global/L1 */
    bool lean;               /* all interfaces quadric, unrotated, max_aperture clipping only */
    bool lean_poly;          /* lean, with polynomial / toroid profiles (out-of-line Newton) */
    bool wave_ok;            /* interface n_ifc-2 carries no decenter: OPD epilogue applicable */
    size_t lean_bytes;       /* shared memory of the lean plan */
    bool dynamic;            /* grid kernels draw 32-ray work items from a counter (default) */
    unsigned long long *d_counters;     /* ring of RT_COUNTERS work counters */
    std::atomic<unsigned> next_counter;
};
#define RT_COUNTERS 64

struct rt_grid {
    int32_t device;
    int32_t n_fields, n_wvls, nx, ny;
    int32_t apply_vignetting, flip_z_dir, paired, pupil_kind;
    double eprad, z_pupil, foc;
    rt_field_desc *d_fields;
    int32_t *d_wvl_idx;
    double *d_pupil_x, *d_pupil_y, *d_ref_img, *d_wave;
    void *d_block;           /* the one device allocation the pointers above point into */
    int64_t rays_per_tile, chunks_per_tile, n_tiles, n_chunks, n_rays;
    std::vector<int32_t> h_wvl_idx;   /* host copy: range-checked against the table in rt_trace_grid */
    unsigned char *h_stage;           /* pinned image of d_block */
    cudaEvent_t uploaded;             /* last rt_grid_update copy */
    size_t b_fields, b_px, b_py, b_ref, b_wave, o_fields, o_px, o_py, o_ref, o_wave, o_wvl, total;
    /* rt_trace_grid_to_host: two internal streams + events (created on first use) */
    cudaStream_t side[2];
    cudaEvent_t ev_in, ev_side[2];
    bool side_ok;
};

/* the prescriptions of a tolerance analysis: n_var surface tables of one shape in one allocation */
struct rt_variants {
    int32_t device, n_ifc, n_wvl, n_var, sm_count;
    rt_surface_desc *d_surfs;           /* [n_var][n_ifc] */
    double *d_n;                        /* [n_var][n_wvl][n_ifc] */
    double *d_wvl;                      /* [n_wvl] wavelengths in nm (NaN when not given) */
    unsigned long long *d_counters;     /* ring of RT_COUNTERS work counters */
    void *d_block;
    std::atomic<unsigned> next_counter;
    std::vector<unsigned char> wave_ok; /* [n_var] rt_table::wave_ok of each variant */
};

/* what the grid kernel needs, passed by value */
/* ------------------------------------------------------------------ kernels */

/* Stage the table into shared memory (8-byte words, coalesced) or, for very
 * long systems, leave it in global memory (uniform loads hit L1). */
template <bool STAGE>
__device__ __forceinline__ void stage_table(const rt_surface_desc *g_surfs, const double *g_n,
                                            int n_ifc, int n_wvl, unsigned char *smem,
                                            const rt_surface_desc *&tab, const double *&ntab)
{
    if (STAGE) {
        const int words_s = n_ifc*(int)(sizeof(rt_surface_desc)/8);
        const int words_n = n_ifc*n_wvl;
        double *dst = reinterpret_cast<double *>(smem);
        const double *src = reinterpret_cast<const double *>(g_surfs);
        for (int i = threadIdx.x; i < words_s; i += blockDim.x) dst[i] = src[i];
        for (int i = threadIdx.x; i < words_n; i += blockDim.x) dst[words_s + i] = g_n[i];
        __syncthreads();
        tab = reinterpret_cast<const rt_surface_desc *>(smem);
        ntab = dst + words_s;
    } else {
        tab = g_surfs;
        ntab = g_n;
    }
}

/* NRML == false: a launch of output kind 0 (out_kind), whose normal and dst columns are NULL,
 * so that R.n and R.dst need not be formed */
template <bool NRML>
__device__ __forceinline__ void store_result(const rt_out &out, int64_t k, const RayResult &R)
{
    if (out.px) { out.px[k] = R.p.x; out.py[k] = R.p.y; out.pz[k] = R.p.z; }
    if (out.dx) { out.dx[k] = R.d.x; out.dy[k] = R.d.y; out.dz[k] = R.d.z; }
    if (NRML && out.nx) { out.nx[k] = R.n.x; out.ny[k] = R.n.y; out.nz[k] = R.n.z; }
    if (NRML && out.dst) out.dst[k] = R.dst;
    if (out.op) out.op[k] = R.op;
    if (out.status) out.status[k] = R.status;
    if (out.fail_surf) out.fail_surf[k] = R.fail_surf;
    if (out.n_seg) out.n_seg[k] = R.n_seg;
}

template <bool FULL, bool STAGE>
__global__ void __launch_bounds__(RT_BLOCK)
k_trace_bundle(const rt_surface_desc *__restrict__ g_surfs, const double *__restrict__ g_n,
               int n_ifc, int n_wvl, int64_t n_rays,
               const double *__restrict__ px, const double *__restrict__ py,
               const double *__restrict__ pz, const double *__restrict__ dx,
               const double *__restrict__ dy, const double *__restrict__ dz,
               const int32_t *__restrict__ wvl_idx, rt_opts o, rt_out out,
               const double *__restrict__ g_wvl)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const rt_surface_desc *tab;
    const double *ntab;
    stage_table<STAGE>(g_surfs, g_n, n_ifc, n_wvl, smem, tab, ntab);

    const int64_t step = (int64_t)gridDim.x*blockDim.x;
    for (int64_t r = (int64_t)blockIdx.x*blockDim.x + threadIdx.x; r < n_rays; r += step) {
        Vec3 p0 = {px[r], py[r], pz[r]};
        Vec3 d0 = {dx[r], dy[r], dz[r]};
        const int w = wvl_idx ? wvl_idx[r] : o.wvl_idx;
        FullWriter fw = {FULL ? out.full + r : nullptr, out.full_stride};
        RayResult R;
        trace_ray<FULL>(tab, ntab + (int64_t)w*n_ifc, g_wvl[w], n_ifc, o, p0, d0, fw, R);
        store_result<true>(out, r, R);
    }
}

/* ---- per-(field, wvl) spot sums.
 * Every thread keeps 15 running values in shared memory (acc[k*RT_BLOCK + tid],
 * conflict-free); when the CTA moves on to another tile (or finishes) each warp
 * shuffle-reduces its lanes and lane 0 writes one 16-double record (15 values +
 * a valid flag) to its slot of the tile.  Slots of a tile: RT_WARPS x SL,
 * SL = min(chunks_per_tile, RT_MAX_GRID); slot = local chunk when
 * chunks_per_tile <= gridDim.x (then a CTA never meets a tile twice), else
 * blockIdx.x (a CTA's chunks of one tile are consecutive => one record).  The
 * scratch buffer is zeroed before the launch, k_reduce_summary adds up the valid
 * records of a tile in slot order: bit-reproducible for a given launch shape,
 * and no CTA barrier / per-chunk shuffle traffic in the trace kernel. */
#define RT_WARPS (RT_BLOCK/32)
#define RT_MAX_GRID 2048
#define RT_ACC 15
#define RT_ACC_BYTES (RT_ACC*RT_BLOCK*sizeof(double))

__device__ __forceinline__ void acc_init(double *acc)
{
#pragma unroll
    for (int k = 0; k < RT_ACC; k++)
        acc[k*RT_BLOCK + threadIdx.x] =
            (k == 10 || k == 12) ? CUDART_INF : ((k == 11 || k == 13) ? -CUDART_INF : 0.0);
}

__device__ __forceinline__ void acc_add(double *acc, int status, double ax, double ay, double op)
{
    double *a = acc + threadIdx.x;
    const int ck = status == RT_RAY_OK ? 0 : (status <= RT_RAY_BLOCKED ? status : 4);
    a[ck*RT_BLOCK] += 1.0;
    if (status == RT_RAY_OK) {
        a[5*RT_BLOCK] += ax; a[6*RT_BLOCK] += ay;
        a[7*RT_BLOCK] += ax*ax; a[8*RT_BLOCK] += ay*ay; a[9*RT_BLOCK] += ax*ay;
        a[10*RT_BLOCK] = fmin(a[10*RT_BLOCK], ax); a[11*RT_BLOCK] = fmax(a[11*RT_BLOCK], ax);
        a[12*RT_BLOCK] = fmin(a[12*RT_BLOCK], ay); a[13*RT_BLOCK] = fmax(a[13*RT_BLOCK], ay);
        a[14*RT_BLOCK] += op;
    }
}

/* dynamic scheduling: only the order-independent columns (counts, min / max) go through the
 * per-thread accumulators; the floating-point sums are reduced per work item (item_sums) */
__device__ __forceinline__ void acc_add_exact(double *acc, int status, double ax, double ay)
{
    double *a = acc + threadIdx.x;
    const int ck = status == RT_RAY_OK ? 0 : (status <= RT_RAY_BLOCKED ? status : 4);
    a[ck*RT_BLOCK] += 1.0;
    if (status == RT_RAY_OK) {
        a[10*RT_BLOCK] = fmin(a[10*RT_BLOCK], ax); a[11*RT_BLOCK] = fmax(a[11*RT_BLOCK], ax);
        a[12*RT_BLOCK] = fmin(a[12*RT_BLOCK], ay); a[13*RT_BLOCK] = fmax(a[13*RT_BLOCK], ay);
    }
}

/* the six sums of one work item (32 rays) in 9 shuffles instead of 30: at the 16 / 8 / 4
 * exchanges every lane hands over the half of its values that its partner keeps, so after
 * three steps each lane owns ONE of (up to 8) values summed over 8 lanes; two more exchanges
 * finish that value.  The addition tree is fixed: same rays, same bits. */
#define RT_ITEM_SUMS 6
__device__ __forceinline__ void item_sums_store(bool ok, double ax, double ay, double op, double *dst)
{
    const int lane = threadIdx.x & 31;
    double v0 = ok ? ax : 0.0, v1 = ok ? ay : 0.0, v2 = ok ? ax*ax : 0.0, v3 = ok ? ay*ay : 0.0;
    double v4 = ok ? ax*ay : 0.0, v5 = ok ? op : 0.0, v6 = 0.0, v7 = 0.0;
    const bool h16 = lane & 16, h8 = lane & 8, h4 = lane & 4;
    /* 16: lower half-warp keeps v0..v3, upper keeps v4..v7 */
    double a0 = (h16 ? v4 : v0) + __shfl_xor_sync(0xffffffffu, h16 ? v0 : v4, 16);
    double a1 = (h16 ? v5 : v1) + __shfl_xor_sync(0xffffffffu, h16 ? v1 : v5, 16);
    double a2 = (h16 ? v6 : v2) + __shfl_xor_sync(0xffffffffu, h16 ? v2 : v6, 16);
    double a3 = (h16 ? v7 : v3) + __shfl_xor_sync(0xffffffffu, h16 ? v3 : v7, 16);
    /* 8: keep a0, a1 | a2, a3 */
    double b0 = (h8 ? a2 : a0) + __shfl_xor_sync(0xffffffffu, h8 ? a0 : a2, 8);
    double b1 = (h8 ? a3 : a1) + __shfl_xor_sync(0xffffffffu, h8 ? a1 : a3, 8);
    /* 4: keep b0 | b1 */
    double c = (h4 ? b1 : b0) + __shfl_xor_sync(0xffffffffu, h4 ? b0 : b1, 4);
    c = c + __shfl_xor_sync(0xffffffffu, c, 2);
    c = c + __shfl_xor_sync(0xffffffffu, c, 1);
    /* lane 4g holds value index 4*[bit 4] + 2*[bit 3] + [bit 2] of g = lane/4 */
    const int idx = ((lane >> 4) & 1)*4 + ((lane >> 3) & 1)*2 + ((lane >> 2) & 1);
    if ((lane & 3) == 0 && idx < RT_ITEM_SUMS) dst[idx] = c;
}

/* warp-reduce the accumulators into the warp's record of (tile, slot) and reset them */
__device__ __forceinline__ void acc_flush(double *acc, double *scratch, int64_t tile, int64_t slot,
                                          int64_t slots_per_tile)
{
    const int lane = threadIdx.x & 31;
    double *dst = scratch + ((tile*slots_per_tile + slot)*RT_WARPS + (threadIdx.x >> 5))*RT_SUMMARY_DOUBLES;
#pragma unroll
    for (int k = 0; k < RT_ACC; k++) {
        double x = acc[k*RT_BLOCK + threadIdx.x];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            double y = __shfl_down_sync(0xffffffffu, x, off);
            if (k == 10 || k == 12) x = fmin(x, y);
            else if (k == 11 || k == 13) x = fmax(x, y);
            else x = x + y;
        }
        if (lane == 0) dst[k] = x;
    }
    if (lane == 0) dst[RT_ACC] = 1.0;
    acc_init(acc);
}

/* per-chunk variant (chunk slots): the lanes' contributions are reduced straight
 * from registers; lanes without a ray contribute the identity */
__device__ __forceinline__ void warp_record_from_regs(bool have, int status, double ax, double ay,
                                                      double op, double *scratch, int64_t tile,
                                                      int64_t slot, int64_t slots_per_tile, int slice)
{
    const int lane = threadIdx.x & 31;
    double *dst = scratch + ((tile*slots_per_tile + slot)*RT_WARPS + slice)*RT_SUMMARY_DOUBLES;
    const bool ok = have && status == RT_RAY_OK;
#pragma unroll
    for (int k = 0; k < RT_ACC; k++) {
        double x;
        if (k < 5) {
            const int ck = status == RT_RAY_OK ? 0 : (status <= RT_RAY_BLOCKED ? status : 4);
            x = (have && ck == k) ? 1.0 : 0.0;
        } else if (k == 10 || k == 12) x = ok ? (k == 10 ? ax : ay) : CUDART_INF;
        else if (k == 11 || k == 13) x = ok ? (k == 11 ? ax : ay) : -CUDART_INF;
        else if (!ok) x = 0.0;
        else x = k == 5 ? ax : k == 6 ? ay : k == 7 ? ax*ax : k == 8 ? ay*ay : k == 9 ? ax*ay : op;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            double y = __shfl_down_sync(0xffffffffu, x, off);
            if (k == 10 || k == 12) x = fmin(x, y);
            else if (k == 11 || k == 13) x = fmax(x, y);
            else x = x + y;
        }
        if (lane == 0) dst[k] = x;
    }
    if (lane == 0) dst[RT_ACC] = 1.0;
}

/* ---- through-focus spot sums (rt_trace_grid_focus): every ray is traced once and its
 * transverse aberration is evaluated at n image planes.  Plane k's records reduce to the
 * summary a single-focus rt_trace_grid launch at foc[k] returns over the same chunk range:
 *  - chunk slots (the regime that launch would take): warp_record_from_regs's record, its sums
 *    with the same shuffle tree;
 *  - otherwise the per-item sums of item_sums_store (same tree, same item order in the
 *    reduction) plus one record per (tile, CTA, warp) holding the counts and the min / max,
 *    whose result does not depend on the order the rays are added in.
 * The per-thread shared-memory accumulators of the static schedule would need n x 15 doubles
 * per thread, so this path always draws work items from a counter (B200RT_STATIC is ignored). */
struct FocusPlanes {
    const double *foc;          /* [n] focus shifts: the kernel's shared-memory copy of FocusList */
    const double *ref;          /* DEVICE [n][n_fields][2] reference image points, or NULL (= 0) */
    int64_t n_tiles, n_items;   /* tiles of the grid; work items of the launch (one plane) */
    int32_t n, n_fields, chunk_slots, pad_;
};
struct FocusList { double v[RT_MAX_FOCUS]; };

/* constant-offset reads of the parameter array (a dynamically indexed kernel parameter would
 * be copied to local memory); blockDim.x >= RT_MAX_FOCUS */
__device__ __forceinline__ void stage_focus(const FocusList &L, int n, double *s)
{
#pragma unroll
    for (int k = 0; k < RT_MAX_FOCUS; k++)
        if ((int)threadIdx.x == k && k < n) s[k] = L.v[k];
    __syncthreads();
}

__device__ __forceinline__ void focus_item(const FocusPlanes &F, bool have, int status, const Vec3 &p,
                                           const Vec3 &d, double op, int f, int64_t tile, int64_t lc,
                                           int slice, unsigned long long item, bool chunk_slots, bool first,
                                           int64_t sl, double *scratch, double *item_sums)
{
    const int lane = threadIdx.x & 31;
    const bool ok = have && status == RT_RAY_OK;
    const int ck = status == RT_RAY_OK ? 0 : (status <= RT_RAY_BLOCKED ? status : 4);
    /* record column this lane writes: 10..13 min / max (lanes 0, 8, 16, 24), 0..4 the status
     * counts (lanes 1..5, the same on every plane), 15 the valid flag (lane 6) */
    double cnt = 0.0;
#pragma unroll
    for (int c = 0; c < 5; c++) {
        const unsigned m = __ballot_sync(0xffffffffu, have && ck == c);
        if (lane == c + 1) cnt = (double)__popc(m);
    }
    const int col = (lane & 7) == 0 ? 10 + (lane >> 3) : (lane >= 1 && lane <= 5) ? lane - 1 : (lane == 6 ? 15 : -1);
    const int64_t rec = chunk_slots ? (tile*sl + lc)*RT_WARPS + slice
                                    : (tile*sl + blockIdx.x)*RT_WARPS + (threadIdx.x >> 5);
    const bool h16 = lane & 16, h8 = lane & 8;
    for (int k = 0; k < F.n; k++) {
        const double rx = F.ref ? F.ref[((int64_t)k*F.n_fields + f)*2 + 0] : 0.0;
        const double ry = F.ref ? F.ref[((int64_t)k*F.n_fields + f)*2 + 1] : 0.0;
        /* the single-focus epilogue of grid_chunk_loop with G.foc -> foc[k] */
        const double dist = div_maybe_zero(F.foc[k], d.z);
        const double ax = (p.x + dist*d.x) - rx;
        const double ay = (p.y + dist*d.y) - ry;
        /* min / max in 6 shuffles: lower half-warp keeps x, upper y; then lanes 0-7 min, 8-15 max */
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
        double *dst = scratch + ((int64_t)k*F.n_tiles*sl*RT_WARPS + rec)*RT_SUMMARY_DOUBLES;
        double v = col >= 10 && col <= 13 ? b : (col == 15 ? 1.0 : cnt);
        if (chunk_slots) {
            /* the sums exactly as warp_record_from_regs forms them */
            const double s6[RT_ITEM_SUMS] = {ax, ay, ax*ax, ay*ay, ax*ay, op};
            const int scol[RT_ITEM_SUMS] = {5, 6, 7, 8, 9, 14};
#pragma unroll
            for (int j = 0; j < RT_ITEM_SUMS; j++) {
                double x = ok ? s6[j] : 0.0;
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) x = x + __shfl_down_sync(0xffffffffu, x, off);
                if (lane == 0) dst[scol[j]] = x;
            }
        } else {
            item_sums_store(ok, ax, ay, op, item_sums + ((int64_t)k*F.n_items + item)*RT_ITEM_SUMS);
            /* a warp's items come in increasing order, so it never returns to a tile it has left */
            if (!first && col >= 0 && col != 15) {
                const double o = dst[col];
                v = (col == 10 || col == 12) ? fmin(o, v) : (col == 11 || col == 13) ? fmax(o, v) : o + v;
            }
        }
        if (col >= 0) dst[col] = v;
    }
}

/* ---- wavefront-error sums (rt_trace_grid_wfe): per work item, the 13 sums of W = opd and the
 * relative pupil coordinates (x, y) of its status-0 rays (RT_WFE_DOUBLES columns 7-19), and per
 * (tile, CTA, warp) a record of the counts and min / max W, whose result does not depend on the
 * order the rays are added in.  Always drawn from a work counter. */
#define RT_WFE_ITEM_SUMS 13

/* the 13 sums of one work item in 8 + 4 + 2 + 1 + 1 = 16 shuffles: the transposition of
 * item_sums_store widened to 16 slots.  At the 16 / 8 / 4 / 2 exchanges every lane hands over the
 * half of its values that its partner keeps; the additions are the halving tree x[i] + x[i+16],
 * +8, +4, +2, +1 of every value (DESIGN.md section 4).  Summands, formed unfused in this order:
 * W, W*W, x*W, y*W, r2*W, x, y, x*x, x*y, y*y, x*r2, y*r2, r2*r2 with r2 = x*x + y*y; lanes
 * without a status-0 ray hold +0.0. */
__device__ __forceinline__ void wfe_item_sums_store(bool ok, double W, double x, double y, double *dst)
{
    const int lane = threadIdx.x & 31;
    const double r2 = x*x + y*y;
    double v[16];
    v[0] = W; v[1] = W*W; v[2] = x*W; v[3] = y*W; v[4] = r2*W;
    v[5] = x; v[6] = y; v[7] = x*x; v[8] = x*y; v[9] = y*y;
    v[10] = x*r2; v[11] = y*r2; v[12] = r2*r2; v[13] = 0.0; v[14] = 0.0; v[15] = 0.0;
#pragma unroll
    for (int k = 0; k < RT_WFE_ITEM_SUMS; k++) v[k] = ok ? v[k] : 0.0;
    const bool h16 = lane & 16, h8 = lane & 8, h4 = lane & 4, h2 = lane & 2;
    /* 16: lower half-warp keeps v0..v7, upper keeps v8..v15 */
    double a[8];
#pragma unroll
    for (int k = 0; k < 8; k++)
        a[k] = (h16 ? v[8 + k] : v[k]) + __shfl_xor_sync(0xffffffffu, h16 ? v[k] : v[8 + k], 16);
    /* 8: keep a0..a3 | a4..a7 */
    double b[4];
#pragma unroll
    for (int k = 0; k < 4; k++)
        b[k] = (h8 ? a[4 + k] : a[k]) + __shfl_xor_sync(0xffffffffu, h8 ? a[k] : a[4 + k], 8);
    /* 4: keep b0, b1 | b2, b3 */
    const double c0 = (h4 ? b[2] : b[0]) + __shfl_xor_sync(0xffffffffu, h4 ? b[0] : b[2], 4);
    const double c1 = (h4 ? b[3] : b[1]) + __shfl_xor_sync(0xffffffffu, h4 ? b[1] : b[3], 4);
    /* 2: keep c0 | c1 */
    double e = (h2 ? c1 : c0) + __shfl_xor_sync(0xffffffffu, h2 ? c0 : c1, 2);
    e = e + __shfl_xor_sync(0xffffffffu, e, 1);
    /* lane 2g holds value index 8*[bit 4] + 4*[bit 3] + 2*[bit 2] + [bit 1] of g = lane/2 */
    const int idx = ((lane >> 4) & 1)*8 + ((lane >> 3) & 1)*4 + ((lane >> 2) & 1)*2 + ((lane >> 1) & 1);
    if ((lane & 1) == 0 && idx < RT_WFE_ITEM_SUMS) dst[idx] = e;
}

/* one work item of the wavefront-error trace: its sums, and its counts / min / max folded into the
 * warp's record of the tile (overwritten when the warp meets the tile first) */
__device__ __forceinline__ void wfe_item(bool have, int status, double W, double x, double y, int64_t tile,
                                         bool first, int64_t sl, double *scratch, double *item_dst)
{
    const int lane = threadIdx.x & 31;
    const bool ok = have && status == RT_RAY_OK;
    wfe_item_sums_store(ok, W, x, y, item_dst);
    const int ck = status == RT_RAY_OK ? 0 : (status <= RT_RAY_BLOCKED ? status : 4);
    double cnt = 0.0;
#pragma unroll
    for (int c = 0; c < 5; c++) {
        const unsigned m = __ballot_sync(0xffffffffu, have && ck == c);
        if (lane == c + 1) cnt = (double)__popc(m);
    }
    /* min / max in 5 shuffles: the lower half-warp reduces min, the upper max; lanes 0 and 16 */
    const bool h16 = lane & 16;
    const double mn = ok ? W : CUDART_INF, mx = ok ? W : -CUDART_INF;
    const double got = __shfl_xor_sync(0xffffffffu, h16 ? mn : mx, 16);
    double b = h16 ? fmax(mx, got) : fmin(mn, got);
#pragma unroll
    for (int s = 8; s > 0; s >>= 1) {
        const double o = __shfl_xor_sync(0xffffffffu, b, s);
        b = h16 ? fmax(b, o) : fmin(b, o);
    }
    /* record column this lane writes: 5 min (lane 0), 6 max (lane 16), 0..4 the counts (lanes 1..5),
     * 20 the valid flag (lane 6) */
    const int col = lane == 0 ? 5 : lane == 16 ? 6 : (lane >= 1 && lane <= 5) ? lane - 1 : (lane == 6 ? 20 : -1);
    if (col < 0) return;
    double *dst = scratch + ((tile*sl + blockIdx.x)*RT_WARPS + (threadIdx.x >> 5))*RT_WFE_DOUBLES;
    double v = col == 5 || col == 6 ? b : (col == 20 ? 1.0 : cnt);
    /* a warp's items come in increasing order, so it never returns to a tile it has left */
    if (!first && col != 20) {
        const double o = dst[col];
        v = col == 5 ? fmin(o, v) : col == 6 ? fmax(o, v) : o + v;
    }
    dst[col] = v;
}

/* ---- OPD at many reference spheres (rt_trace_grid_opd_focus): per ray, refocus_pre once and
 * refocus_opd per plane (rt_refocus.cuh), after the trace and outside its interface loop */
struct RefocusPlanes {
    const double *spheres;      /* DEVICE [n][n_tiles][RT_SPHERE_DOUBLES] */
    double *planes;             /* DEVICE [n][n_rays]: plane pl of ray k of the range at pl*n_rays + k */
    int64_t n_rays, sphere_stride;     /* rays of the range; n_tiles*RT_SPHERE_DOUBLES */
    int32_t n, pad_;
};

/* the perturbed prescriptions of one rt_trace_grid_variants[_wfe] launch */
struct VariantPlan {
    double *items;              /* DEVICE [n_var][n_tiles][chunks_per_tile*RT_WARPS][RT_TOL_DOUBLES] (WFE:
                                 * [RT_WFE_DOUBLES]) */
    int32_t n_var, n_tiles;
    const double *wave;         /* WFE: DEVICE [n_var][n_tiles][RT_WAVE_DOUBLES] */
};

/* one work item of the variants wavefront-error trace: its whole RT_WFE_DOUBLES record (every
 * column written, so scratch needs no clearing) -- the 13 sums by wfe_item_sums_store's halving
 * tree, the counts by ballots, min / max W, the valid flag.  reduce_tile<WfeLayout> then adds a
 * (variant, tile)'s items in item order, as k_reduce_wfe adds rt_trace_grid_wfe's item sums. */
__device__ __forceinline__ void wfe_var_item(bool have, int status, double W, double x, double y,
                                             double *__restrict__ dst)
{
    const int lane = threadIdx.x & 31;
    const bool ok = have && status == RT_RAY_OK;
    wfe_item_sums_store(ok, W, x, y, dst + 7);
    const int ck = status == RT_RAY_OK ? 0 : (status <= RT_RAY_BLOCKED ? status : 4);
    double cnt = 0.0;
#pragma unroll
    for (int c = 0; c < 5; c++) {
        const unsigned m = __ballot_sync(0xffffffffu, have && ck == c);
        if (lane == 2*c + 1) cnt = (double)__popc(m);
    }
    /* min / max as wfe_item: the lower half-warp reduces min, the upper max; lanes 0 and 16 */
    const bool h16 = lane & 16;
    const double mn = ok ? W : CUDART_INF, mx = ok ? W : -CUDART_INF;
    const double got = __shfl_xor_sync(0xffffffffu, h16 ? mn : mx, 16);
    double b = h16 ? fmax(mx, got) : fmin(mn, got);
#pragma unroll
    for (int s = 8; s > 0; s >>= 1) {
        const double o = __shfl_xor_sync(0xffffffffu, b, s);
        b = h16 ? fmax(b, o) : fmin(b, o);
    }
    /* odd lanes 1..9: counts 0..4 (the even lanes < 26 hold the sums); 0 / 16: min / max;
     * 11: valid flag; 13, 15, 17: the zero columns 21-23 */
    if ((lane & 1) && lane <= 9) dst[lane >> 1] = cnt;
    if (lane == 0) dst[5] = b;
    if (lane == 16) dst[6] = b;
    if (lane == 11) dst[20] = 1.0;
    if (lane == 13) dst[21] = 0.0;
    if (lane == 15) dst[22] = 0.0;
    if (lane == 17) dst[23] = 0.0;
}

/* chunk loop shared by the general and the lean grid kernels: start ray ->
 * trace -> per-ray results -> transverse aberration (focus_pupil_coords,
 * analyses.py:561-580) -> spot sums.  FOCUS: the spot sums of the planes of *FP instead
 * (needs SUMMARY == false and a work counter).  WFE: the wavefront-error sums of wfe_item instead
 * (needs WAVE, SUMMARY == false and a work counter).  OPDF: the OPD against every sphere of *RP
 * instead of out.opd (needs WAVE alone).  NRML: see store_result.  VARIANTS: the chunk range once per prescription of *VP,
 * work item u of variant u / (items of the range); trace gets the variant as a seventh argument; no
 * per-ray outputs; the item's tol_item record instead (needs a work counter and nothing else); with
 * WAVE and WFE the OPD against the variant's own wave record of *VP and the item's wfe_var_item
 * record instead. */
template <bool SUMMARY, bool WAVE, bool FOCUS = false, bool NRML = true, bool WFE = false, bool OPDF = false,
          bool VARIANTS = false, typename TraceFn>
__device__ __forceinline__ void grid_chunk_loop(const GridDev &G, int64_t chunk_begin, int64_t chunk_end,
                                                const rt_out &out, double *scratch, double *acc,
                                                unsigned long long *work_counter, double *item_sums,
                                                TraceFn trace, const FocusPlanes *FP = nullptr,
                                                const RefocusPlanes *RP = nullptr, const VariantPlan *VP = nullptr)
{
    static_assert(!VARIANTS || (!SUMMARY && !FOCUS && !OPDF && WAVE == WFE), "VARIANTS writes its own records");
    static_assert(!WFE || (WAVE && !SUMMARY && !FOCUS), "WFE needs the OPD epilogue and no spot sums");
    static_assert(!OPDF || (WAVE && !SUMMARY && !FOCUS && !WFE), "OPDF needs the OPD epilogue alone");
    const int64_t tile0 = chunk_begin/G.chunks_per_tile;
    const int64_t ray0 = tile0*G.rays_per_tile + (chunk_begin - tile0*G.chunks_per_tile)*RT_BLOCK;
    const int64_t sl = G.chunks_per_tile < RT_MAX_GRID ? G.chunks_per_tile : RT_MAX_GRID;
    const bool chunk_slots = FOCUS ? FP->chunk_slots != 0 : G.chunks_per_tile <= (int64_t)gridDim.x;
    int64_t cur_tile = -1;
    if (SUMMARY && !chunk_slots) acc_init(acc);
    const unsigned long long per_var = (unsigned long long)(chunk_end - chunk_begin)*RT_WARPS;
    const unsigned long long n_items = VARIANTS ? per_var*(unsigned long long)VP->n_var : per_var;
    int64_t c = chunk_begin + blockIdx.x;
    int var = 0;
    for (;;) {
        int slice;                       /* which 32 rays of the chunk this warp takes */
        unsigned long long item = 0;
        if (work_counter) {
            /* dynamic scheduling, one work item = 32 consecutive rays: every warp draws its next
             * item from a global counter, so no warp idles while rays are left (the cost of a
             * chunk varies several-fold between the pupil centre and its clipped edge) */
            unsigned long long u = 0;
            if ((threadIdx.x & 31) == 0) u = atomicAdd(work_counter, 1ull);
            u = __shfl_sync(0xffffffffu, u, 0);
            if (u >= n_items) break;
            unsigned long long r = u;
            if (VARIANTS) {
                var = (int)(u/per_var);
                r = u - (unsigned long long)var*per_var;
            }
            c = chunk_begin + (int64_t)(r/RT_WARPS);
            slice = (int)(r % RT_WARPS);
            item = u;
        } else {
            if (c >= chunk_end) break;
            /* static round robin; the slice a warp takes is a hash of the chunk id, so that no
             * warp is stuck with the pupil-edge (cheap) or the centre (expensive) end of every chunk */
            slice = (int)(((threadIdx.x >> 5) + ((unsigned)c*0x9E3779B1u >> 27)) % RT_WARPS);
        }
        const int64_t tile = c/G.chunks_per_tile;
        const int64_t lc = c - tile*G.chunks_per_tile;
        const int64_t loc = lc*RT_BLOCK + slice*32 + (threadIdx.x & 31);
        const bool have = loc < G.rays_per_tile;
        if (SUMMARY && !chunk_slots && tile != cur_tile) {
            if (cur_tile >= 0) acc_flush(acc, scratch, cur_tile, blockIdx.x, sl);
            cur_tile = tile;
        }
        int status = RT_RAY_OK;
        double ax = 0.0, ay = 0.0, op = 0.0;
        Vec3 fp = {0.0, 0.0, 0.0}, fd = {0.0, 0.0, 0.0};     /* FOCUS: image point and direction */
        double wW = 0.0, wx = 0.0, wy = 0.0;                  /* WFE: opd, relative pupil coordinates */
        if (have) {
            const int f = (int)(tile/G.n_wvls);
            const int w = (int)(tile - (int64_t)f*G.n_wvls);
            const int64_t k = tile*G.rays_per_tile + loc - ray0;
            RayResult R;
            Vec3 d0;
            if constexpr (VARIANTS) trace(f, w, loc, k, R, d0, var);
            else trace(f, w, loc, k, R, d0);
            if (!VARIANTS) store_result<NRML>(out, k, R);
            status = R.status; op = R.op;
            if (FOCUS || VARIANTS) { fp = R.p; fd = R.d; }
            if (OPDF) {
                /* every plane of the ray: the sphere records of a work item's tile are warp-uniform loads */
                double *dst = RP->planes + k;
                if (R.status == RT_RAY_OK) {
                    const RefocusRay q = refocus_pre(G.wave + tile*RT_WAVE_DOUBLES, R.p1, d0, R.pk, R.dk, R.p, R.d, R.op);
                    const double *S = RP->spheres + tile*RT_SPHERE_DOUBLES;
                    for (int pl = 0; pl < RP->n; pl++)
                        dst[pl*RP->n_rays] = refocus_opd(q, S + pl*RP->sphere_stride);
                } else {
                    for (int pl = 0; pl < RP->n; pl++) dst[pl*RP->n_rays] = CUDART_NAN;
                }
            } else if (WAVE) {
                const double *wr = VARIANTS ? VP->wave + ((int64_t)var*VP->n_tiles + tile)*RT_WAVE_DOUBLES
                                            : G.wave + tile*RT_WAVE_DOUBLES;
                const double opd = (R.status == RT_RAY_OK)
                                       ? wave_opd(wr, R.p1, d0, R.pk, R.dk, R.p, R.d, R.op)
                                       : CUDART_NAN;
                if (!VARIANTS && (!WFE || out.opd)) out.opd[k] = opd;
                if (WFE) {
                    wW = opd;
                    grid_pupil_coords(G, f, loc, wx, wy);
                }
            }
            if ((VARIANTS && !WFE) || out.abr_x || SUMMARY) {
                const double rx = G.ref_img ? G.ref_img[tile*2 + 0] : 0.0;
                const double ry = G.ref_img ? G.ref_img[tile*2 + 1] : 0.0;
                double dist = div_maybe_zero(G.foc, R.d.z);
                ax = (R.p.x + dist*R.d.x) - rx;
                ay = (R.p.y + dist*R.d.y) - ry;
                if (!VARIANTS && out.abr_x) {
                    double sx = ax, sy = ay;
                    if ((out.flags & RT_OUT_ABR_NAN_STATUS) && status != RT_RAY_OK) {
                        sx = __longlong_as_double((long long)(RT_NAN_PAYLOAD_BASE | (unsigned long long)(status & 0xFFFF)));
                        sy = __longlong_as_double((long long)(RT_NAN_PAYLOAD_BASE | (unsigned long long)(R.fail_surf & 0xFFFF)));
                    }
                    out.abr_x[k] = sx; out.abr_y[k] = sy;
                }
                if (SUMMARY && !chunk_slots) {
                    if (work_counter) acc_add_exact(acc, status, ax, ay);
                    else acc_add(acc, status, ax, ay, op);
                }
            }
        }
        /* dynamic schedule: which warp adds which rays varies from run to run, so the sums of every
         * work item are stored on their own and k_reduce_summary adds them in item order --
         * the summary stays bit-reproducible */
        if (SUMMARY && !chunk_slots && work_counter)
            item_sums_store(have && status == RT_RAY_OK, ax, ay, op, item_sums + item*RT_ITEM_SUMS);
        if (SUMMARY && chunk_slots) warp_record_from_regs(have, status, ax, ay, op, scratch, tile, lc, sl, slice);
        if (FOCUS) {
            const bool first = tile != cur_tile;
            cur_tile = tile;
            focus_item(*FP, have, status, fp, fd, op, (int)(tile/G.n_wvls), tile, lc, slice, item, chunk_slots,
                       first, sl, scratch, item_sums);
        }
        if (WFE && !VARIANTS) {
            const bool first = tile != cur_tile;
            cur_tile = tile;
            wfe_item(have, status, wW, wx, wy, tile, first, sl, scratch, item_sums + item*RT_WFE_ITEM_SUMS);
        }
        /* a variant's items are its tiles' items in order: item u is record u */
        if (VARIANTS && !WFE) tol_item(have, status, ax, ay, op, fd, VP->items + item*RT_TOL_DOUBLES);
        if (VARIANTS && WFE) wfe_var_item(have, status, wW, wx, wy, VP->items + item*RT_WFE_DOUBLES);
        if (!work_counter) c += gridDim.x;
    }
    if (SUMMARY && !chunk_slots && cur_tile >= 0) acc_flush(acc, scratch, cur_tile, blockIdx.x, sl);
}

template <bool FULL, bool SUMMARY, bool STAGE, bool WAVE>
__global__ void __launch_bounds__(RT_BLOCK)
k_trace_grid(const rt_surface_desc *__restrict__ g_surfs, const double *__restrict__ g_n,
             int n_ifc, int n_wvl, GridDev G, int64_t chunk_begin, int64_t chunk_end,
             rt_opts o, rt_out out, double *__restrict__ scratch, const double *__restrict__ g_wvl,
             int pupil_kind, unsigned long long *work_counter, double *item_sums)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const rt_surface_desc *tab;
    const double *ntab;
    double *acc = reinterpret_cast<double *>(smem);          /* [RT_ACC][RT_BLOCK] when SUMMARY */
    stage_table<STAGE>(g_surfs, g_n, n_ifc, n_wvl, smem + (SUMMARY ? RT_ACC_BYTES : 0), tab, ntab);
    grid_chunk_loop<SUMMARY, WAVE>(G, chunk_begin, chunk_end, out, scratch, acc, work_counter, item_sums,
        [&](int f, int w, int64_t loc, int64_t k, RayResult &R, Vec3 &d0) {
            Vec3 p0;
            grid_start_ray<false>(G, pupil_kind, f, loc, p0, d0);
            FullWriter fw = {FULL ? out.full + k : nullptr, out.full_stride};
            const int wi = G.wvl_idx[w];
            trace_ray<FULL, WAVE>(tab, ntab + (int64_t)wi*n_ifc, g_wvl[wi], n_ifc, o, p0, d0, fw, R);
        });
}

/* through-focus instance of k_trace_grid (per-ray outputs of kind 0 only) */
template <bool STAGE>
__global__ void __launch_bounds__(RT_BLOCK)
k_trace_grid_focus(const rt_surface_desc *__restrict__ g_surfs, const double *__restrict__ g_n,
                   int n_ifc, int n_wvl, GridDev G, int64_t chunk_begin, int64_t chunk_end,
                   rt_opts o, rt_out out, double *__restrict__ scratch, const double *__restrict__ g_wvl,
                   int pupil_kind, unsigned long long *work_counter, double *item_sums,
                   FocusPlanes P, FocusList foc)
{
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ double s_foc[RT_MAX_FOCUS];
    const rt_surface_desc *tab;
    const double *ntab;
    stage_focus(foc, P.n, s_foc);
    stage_table<STAGE>(g_surfs, g_n, n_ifc, n_wvl, smem, tab, ntab);
    FocusPlanes F = P;
    F.foc = s_foc;
    grid_chunk_loop<false, false, true>(G, chunk_begin, chunk_end, out, scratch, nullptr, work_counter, item_sums,
        [&](int f, int w, int64_t loc, int64_t k, RayResult &R, Vec3 &d0) {
            Vec3 p0;
            grid_start_ray<false>(G, pupil_kind, f, loc, p0, d0);
            FullWriter fw = {nullptr, 0};
            const int wi = G.wvl_idx[w];
            trace_ray<false, false>(tab, ntab + (int64_t)wi*n_ifc, g_wvl[wi], n_ifc, o, p0, d0, fw, R);
        }, &F);
}

/* wavefront-error instance of k_trace_grid (per-ray outputs of kind 0, opd optional) */
template <bool STAGE>
__global__ void __launch_bounds__(RT_BLOCK)
k_trace_grid_wfe(const rt_surface_desc *__restrict__ g_surfs, const double *__restrict__ g_n,
                 int n_ifc, int n_wvl, GridDev G, int64_t chunk_begin, int64_t chunk_end,
                 rt_opts o, rt_out out, double *__restrict__ scratch, const double *__restrict__ g_wvl,
                 int pupil_kind, unsigned long long *work_counter, double *item_sums)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const rt_surface_desc *tab;
    const double *ntab;
    stage_table<STAGE>(g_surfs, g_n, n_ifc, n_wvl, smem, tab, ntab);
    grid_chunk_loop<false, true, false, true, true>(G, chunk_begin, chunk_end, out, scratch, nullptr, work_counter,
                                                    item_sums,
        [&](int f, int w, int64_t loc, int64_t k, RayResult &R, Vec3 &d0) {
            Vec3 p0;
            grid_start_ray<false>(G, pupil_kind, f, loc, p0, d0);
            FullWriter fw = {nullptr, 0};
            const int wi = G.wvl_idx[w];
            trace_ray<false, true>(tab, ntab + (int64_t)wi*n_ifc, g_wvl[wi], n_ifc, o, p0, d0, fw, R);
        });
}

/* OPD-at-many-spheres instance of k_trace_grid (per-ray outputs of kind 0) */
template <bool STAGE>
__global__ void __launch_bounds__(RT_BLOCK)
k_trace_grid_opd_focus(const rt_surface_desc *__restrict__ g_surfs, const double *__restrict__ g_n,
                       int n_ifc, int n_wvl, GridDev G, int64_t chunk_begin, int64_t chunk_end,
                       rt_opts o, rt_out out, const double *__restrict__ g_wvl, int pupil_kind,
                       unsigned long long *work_counter, RefocusPlanes P)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const rt_surface_desc *tab;
    const double *ntab;
    stage_table<STAGE>(g_surfs, g_n, n_ifc, n_wvl, smem, tab, ntab);
    grid_chunk_loop<false, true, false, true, false, true>(G, chunk_begin, chunk_end, out, nullptr, nullptr,
                                                           work_counter, nullptr,
        [&](int f, int w, int64_t loc, int64_t k, RayResult &R, Vec3 &d0) {
            Vec3 p0;
            grid_start_ray<false>(G, pupil_kind, f, loc, p0, d0);
            FullWriter fw = {nullptr, 0};
            const int wi = G.wvl_idx[w];
            trace_ray<false, true>(tab, ntab + (int64_t)wi*n_ifc, g_wvl[wi], n_ifc, o, p0, d0, fw, R);
        }, nullptr, &P);
}

/* every prescription of a variant set over the whole grid (rt_trace_grid_variants): the general
 * trace with the table read from global memory, since a warp's prescription changes from one work
 * item to the next.  g_surfs / g_n: the set's rows from the launch's first variant on */
__global__ void __launch_bounds__(RT_BLOCK)
k_trace_grid_variants(const rt_surface_desc *__restrict__ g_surfs, const double *__restrict__ g_n,
                      int n_ifc, int n_wvl, GridDev G, int64_t n_chunks, rt_opts o,
                      const double *__restrict__ g_wvl, int pupil_kind, unsigned long long *work_counter,
                      VariantPlan P)
{
    const rt_out out = {};
    grid_chunk_loop<false, false, false, false, false, false, true>(G, 0, n_chunks, out, nullptr, nullptr,
                                                                    work_counter, nullptr,
        [&](int f, int w, int64_t loc, int64_t k, RayResult &R, Vec3 &d0, int v) {
            Vec3 p0;
            grid_start_ray<false>(G, pupil_kind, f, loc, p0, d0);
            FullWriter fw = {nullptr, 0};
            const int wi = G.wvl_idx[w];
            trace_ray<false, false>(g_surfs + (int64_t)v*n_ifc, g_n + ((int64_t)v*n_wvl + wi)*n_ifc, g_wvl[wi],
                                    n_ifc, o, p0, d0, fw, R);
        }, nullptr, nullptr, &P);
}

/* k_trace_grid_variants with the OPD epilogue (rt_trace_grid_variants_wfe): each ray's OPD against
 * its variant's wave record of P.wave, per-item wavefront-error records */
__global__ void __launch_bounds__(RT_BLOCK)
k_trace_grid_variants_wfe(const rt_surface_desc *__restrict__ g_surfs, const double *__restrict__ g_n,
                          int n_ifc, int n_wvl, GridDev G, int64_t n_chunks, rt_opts o,
                          const double *__restrict__ g_wvl, int pupil_kind, unsigned long long *work_counter,
                          VariantPlan P)
{
    const rt_out out = {};
    grid_chunk_loop<false, true, false, false, true, false, true>(G, 0, n_chunks, out, nullptr, nullptr,
                                                                  work_counter, nullptr,
        [&](int f, int w, int64_t loc, int64_t k, RayResult &R, Vec3 &d0, int v) {
            Vec3 p0;
            grid_start_ray<false>(G, pupil_kind, f, loc, p0, d0);
            FullWriter fw = {nullptr, 0};
            const int wi = G.wvl_idx[w];
            trace_ray<false, true>(g_surfs + (int64_t)v*n_ifc, g_n + ((int64_t)v*n_wvl + wi)*n_ifc, g_wvl[wi],
                                   n_ifc, o, p0, d0, fw, R);
        }, nullptr, nullptr, &P);
}

/* the wave record of every (variant, tile) of rt_variants_wave, one thread each: the chief ray of
 * k_chief_ref (pupil (0, 0), no vignetting) at the tile's wavelength through the variant's rows,
 * then tolwave_record.  g_surfs / g_n: the set's rows from the launch's first variant on */
__global__ void k_variants_wave(const rt_surface_desc *__restrict__ g_surfs, const double *__restrict__ g_n,
                                int n_ifc, int n_wvl, GridDev G, int n_tiles, int n_var, int pupil_kind,
                                const double *__restrict__ g_wvl, rt_opts o, double exp_dist, double n_obj,
                                double n_img, double *__restrict__ wave, double *__restrict__ ref_img,
                                int32_t *__restrict__ status)
{
    const int64_t i = (int64_t)blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= (int64_t)n_var*n_tiles) return;
    const int v = (int)(i/n_tiles), tile = (int)(i - (int64_t)v*n_tiles);
    const int f = tile/G.n_wvls, w = tile - f*G.n_wvls;
    const rt_surface_desc *tab = g_surfs + (int64_t)v*n_ifc;
    const int wi = G.wvl_idx[w];
    Vec3 p0, d0;
    grid_start_ray_at<false>(G, pupil_kind, f, 0.0, 0.0, false, p0, d0);
    FullWriter fw = {nullptr, 0};
    RayResult R;
    trace_ray<false, true>(tab, g_n + ((int64_t)v*n_wvl + wi)*n_ifc, g_wvl[wi], n_ifc, o, p0, d0, fw, R);
    tolwave_record(R.status, R.p1, d0, R.pk, R.dk, R.p, R.d, R.op, G.foc, tab[n_ifc - 2], exp_dist, n_obj, n_img,
                   wave + i*RT_WAVE_DOUBLES, ref_img + i*2);
    status[i] = R.status;
}

/* ---- lean kernels: plan built in shared memory by the CTA (rt_lean.cuh) */
template <int OUT, bool POLY>
__global__ void __launch_bounds__(RT_BLOCK, POLY ? 2 : RT_LEAN_MIN_CTAS)
k_trace_bundle_lean(const rt_surface_desc *__restrict__ g_surfs, const double *__restrict__ g_n,
                    int n_ifc, int n_wvl, int64_t n_rays,
                    const double *__restrict__ px, const double *__restrict__ py,
                    const double *__restrict__ pz, const double *__restrict__ dx,
                    const double *__restrict__ dy, const double *__restrict__ dz,
                    const int32_t *__restrict__ wvl_idx, rt_opts o, rt_out out)
{
    extern __shared__ __align__(16) unsigned char smem[];
    LeanSurf *ls = reinterpret_cast<LeanSurf *>(smem);
    LeanIdx *li = reinterpret_cast<LeanIdx *>(ls + n_ifc);
    LeanPoly *lp = reinterpret_cast<LeanPoly *>(li + (size_t)n_ifc*n_wvl);      /* POLY instances only */
    build_plan(g_surfs, g_n, n_ifc, n_wvl, o, ls, li);
    if (POLY) build_poly_plan(g_surfs, n_ifc, lp);
    __syncthreads();

    const int64_t step = (int64_t)gridDim.x*blockDim.x;
    for (int64_t r = (int64_t)blockIdx.x*blockDim.x + threadIdx.x; r < n_rays; r += step) {
        Vec3 p0 = {px[r], py[r], pz[r]};
        Vec3 d0 = {dx[r], dy[r], dz[r]};
        const int w = wvl_idx ? wvl_idx[r] : o.wvl_idx;
        FullWriter fw = {OUT == 2 ? out.full + r : nullptr, out.full_stride};
        RayResult R;
        trace_ray_lean<OUT, false, POLY>(ls, li + (int64_t)w*n_ifc, lp, g_surfs, n_ifc, o, p0, d0, fw, R);
        store_result<(OUT >= 1)>(out, r, R);
    }
}

template <int OUT, bool SUMMARY, bool WAVE, bool POLY>
__global__ void __launch_bounds__(RT_BLOCK, POLY ? 2 : RT_LEAN_MIN_CTAS)
k_trace_grid_lean(const rt_surface_desc *__restrict__ g_surfs, const double *__restrict__ g_n,
                  int n_ifc, int n_wvl, GridDev G, int64_t chunk_begin, int64_t chunk_end,
                  rt_opts o, rt_out out, double *__restrict__ scratch, unsigned long long *work_counter,
                  double *item_sums)
{
    extern __shared__ __align__(16) unsigned char smem[];
    double *acc = reinterpret_cast<double *>(smem);          /* [RT_ACC][RT_BLOCK] when SUMMARY */
    LeanSurf *ls = reinterpret_cast<LeanSurf *>(smem + (SUMMARY ? RT_ACC_BYTES : 0));
    LeanIdx *li = reinterpret_cast<LeanIdx *>(ls + n_ifc);
    LeanPoly *lp = reinterpret_cast<LeanPoly *>(li + (size_t)n_ifc*n_wvl);      /* POLY instances only */
    build_plan(g_surfs, g_n, n_ifc, n_wvl, o, ls, li);
    if (POLY) build_poly_plan(g_surfs, n_ifc, lp);
    __syncthreads();
    grid_chunk_loop<SUMMARY, WAVE, false, (OUT >= 1)>(G, chunk_begin, chunk_end, out, scratch, acc, work_counter, item_sums,
        [&](int f, int w, int64_t loc, int64_t k, RayResult &R, Vec3 &d0) {
            Vec3 p0;
            grid_start_ray<true>(G, RT_PUPIL_EPD, f, loc, p0, d0);
            FullWriter fw = {OUT == 2 ? out.full + k : nullptr, out.full_stride};
            trace_ray_lean<OUT, WAVE, POLY>(ls, li + (int64_t)G.wvl_idx[w]*n_ifc, lp, g_surfs, n_ifc, o, p0, d0, fw, R);
        });
}

/* through-focus instance of k_trace_grid_lean (per-ray outputs of kind 0 only) */
template <bool POLY>
__global__ void __launch_bounds__(RT_BLOCK, POLY ? 2 : RT_LEAN_MIN_CTAS)
k_trace_grid_lean_focus(const rt_surface_desc *__restrict__ g_surfs, const double *__restrict__ g_n,
                        int n_ifc, int n_wvl, GridDev G, int64_t chunk_begin, int64_t chunk_end,
                        rt_opts o, rt_out out, double *__restrict__ scratch, unsigned long long *work_counter,
                        double *item_sums, FocusPlanes P, FocusList foc)
{
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ double s_foc[RT_MAX_FOCUS];
    LeanSurf *ls = reinterpret_cast<LeanSurf *>(smem);
    LeanIdx *li = reinterpret_cast<LeanIdx *>(ls + n_ifc);
    LeanPoly *lp = reinterpret_cast<LeanPoly *>(li + (size_t)n_ifc*n_wvl);      /* POLY instances only */
    build_plan(g_surfs, g_n, n_ifc, n_wvl, o, ls, li);
    if (POLY) build_poly_plan(g_surfs, n_ifc, lp);
    stage_focus(foc, P.n, s_foc);                /* its barrier also completes the plan */
    FocusPlanes F = P;
    F.foc = s_foc;
    grid_chunk_loop<false, false, true, false>(G, chunk_begin, chunk_end, out, scratch, nullptr, work_counter, item_sums,
        [&](int f, int w, int64_t loc, int64_t k, RayResult &R, Vec3 &d0) {
            Vec3 p0;
            grid_start_ray<true>(G, RT_PUPIL_EPD, f, loc, p0, d0);
            FullWriter fw = {nullptr, 0};
            trace_ray_lean<0, false, POLY>(ls, li + (int64_t)G.wvl_idx[w]*n_ifc, lp, g_surfs, n_ifc, o, p0, d0, fw, R);
        }, &F);
}

/* wavefront-error instance of k_trace_grid_lean (per-ray outputs of kind 0, opd optional) */
template <bool POLY>
__global__ void __launch_bounds__(RT_BLOCK, POLY ? 2 : RT_LEAN_MIN_CTAS)
k_trace_grid_lean_wfe(const rt_surface_desc *__restrict__ g_surfs, const double *__restrict__ g_n,
                      int n_ifc, int n_wvl, GridDev G, int64_t chunk_begin, int64_t chunk_end,
                      rt_opts o, rt_out out, double *__restrict__ scratch, unsigned long long *work_counter,
                      double *item_sums)
{
    extern __shared__ __align__(16) unsigned char smem[];
    LeanSurf *ls = reinterpret_cast<LeanSurf *>(smem);
    LeanIdx *li = reinterpret_cast<LeanIdx *>(ls + n_ifc);
    LeanPoly *lp = reinterpret_cast<LeanPoly *>(li + (size_t)n_ifc*n_wvl);      /* POLY instances only */
    build_plan(g_surfs, g_n, n_ifc, n_wvl, o, ls, li);
    if (POLY) build_poly_plan(g_surfs, n_ifc, lp);
    __syncthreads();
    grid_chunk_loop<false, true, false, false, true>(G, chunk_begin, chunk_end, out, scratch, nullptr, work_counter,
                                                     item_sums,
        [&](int f, int w, int64_t loc, int64_t k, RayResult &R, Vec3 &d0) {
            Vec3 p0;
            grid_start_ray<true>(G, RT_PUPIL_EPD, f, loc, p0, d0);
            FullWriter fw = {nullptr, 0};
            trace_ray_lean<0, true, POLY>(ls, li + (int64_t)G.wvl_idx[w]*n_ifc, lp, g_surfs, n_ifc, o, p0, d0, fw, R);
        });
}

/* OPD-at-many-spheres instance of k_trace_grid_lean (per-ray outputs of kind 0) */
template <bool POLY>
__global__ void __launch_bounds__(RT_BLOCK, POLY ? 2 : RT_LEAN_MIN_CTAS)
k_trace_grid_lean_opd_focus(const rt_surface_desc *__restrict__ g_surfs, const double *__restrict__ g_n,
                            int n_ifc, int n_wvl, GridDev G, int64_t chunk_begin, int64_t chunk_end,
                            rt_opts o, rt_out out, unsigned long long *work_counter, RefocusPlanes P)
{
    extern __shared__ __align__(16) unsigned char smem[];
    LeanSurf *ls = reinterpret_cast<LeanSurf *>(smem);
    LeanIdx *li = reinterpret_cast<LeanIdx *>(ls + n_ifc);
    LeanPoly *lp = reinterpret_cast<LeanPoly *>(li + (size_t)n_ifc*n_wvl);      /* POLY instances only */
    build_plan(g_surfs, g_n, n_ifc, n_wvl, o, ls, li);
    if (POLY) build_poly_plan(g_surfs, n_ifc, lp);
    __syncthreads();
    grid_chunk_loop<false, true, false, false, false, true>(G, chunk_begin, chunk_end, out, nullptr, nullptr,
                                                            work_counter, nullptr,
        [&](int f, int w, int64_t loc, int64_t k, RayResult &R, Vec3 &d0) {
            Vec3 p0;
            grid_start_ray<true>(G, RT_PUPIL_EPD, f, loc, p0, d0);
            FullWriter fw = {nullptr, 0};
            trace_ray_lean<0, true, POLY>(ls, li + (int64_t)G.wvl_idx[w]*n_ifc, lp, g_surfs, n_ifc, o, p0, d0, fw, R);
        }, nullptr, &P);
}

/* division self-test: div_shared/normalize3_shared against the IEEE `/` */
__global__ void k_selftest_division(uint64_t seed, int64_t n_per_thread, unsigned long long *mismatch)
{
    uint64_t x = seed + 0x9E3779B97F4A7C15ull*(uint64_t)(blockIdx.x*blockDim.x + threadIdx.x + 1);
    unsigned long long bad = 0;
    for (int64_t it = 0; it < n_per_thread; it++) {
        uint64_t r[4];
        for (int k = 0; k < 4; k++) {          /* splitmix64 */
            x += 0x9E3779B97F4A7C15ull;
            uint64_t z = x;
            z = (z ^ (z >> 30))*0xBF58476D1CE4E5B9ull;
            z = (z ^ (z >> 27))*0x94D049BB133111EBull;
            r[k] = z ^ (z >> 31);
        }
        /* operands: random mantissas, exponents spread over a window chosen by the draw:
         * mostly ordinary magnitudes, sometimes extreme (exercise the fallback) */
        const int mode = (int)(r[3] & 15);
        const int span = mode < 12 ? 40 : (mode < 15 ? 600 : 2046);
        double a[3], b;
        uint64_t bm = (r[3] >> 8) & 0xFFFFFFFFFFFFFull;
        if (((r[3] >> 4) & 15) == 0) bm = 0xFFFFFFFFFFFFFull;        /* all-ones mantissa */
        if (((r[3] >> 4) & 15) == 1) bm = 0;                          /* power of two */
        int be = 1023 + (int)((r[2] >> 40) % (uint64_t)span) - span/2;
        be = be < 0 ? 0 : (be > 2047 ? 2047 : be);
        b = __longlong_as_double((long long)(((r[2] & 1) << 63) | ((uint64_t)be << 52) | bm));
        for (int k = 0; k < 3; k++) {
            int ae = 1023 + (int)((r[k] >> 53) % (uint64_t)span) - span/2;
            ae = ae < 0 ? 0 : (ae > 2047 ? 2047 : ae);
            uint64_t am = r[k] & 0xFFFFFFFFFFFFFull;
            if (((r[k] >> 60) & 7) == 0) am = 0;
            a[k] = __longlong_as_double((long long)(((r[k] >> 52 & 1) << 63) | ((uint64_t)ae << 52) | am));
            if (mode == 7 && k == 2) a[k] = 0.0;
        }
        const double rr = rcp_refined(b);
        for (int k = 0; k < 3; k++) {
            double q1 = div_shared(a[k], b, rr), q2 = a[k]/b;
            if (__double_as_longlong(q1) != __double_as_longlong(q2) && !(isnan(q1) && isnan(q2))) bad++;
        }
        Vec3 v = {a[0], a[1], a[2]};
        if (mode < 12) {
            Vec3 n1 = normalize3_shared(v), n2 = normalize3(v);
            if (__double_as_longlong(n1.x) != __double_as_longlong(n2.x) ||
                __double_as_longlong(n1.y) != __double_as_longlong(n2.y) ||
                __double_as_longlong(n1.z) != __double_as_longlong(n2.z)) {
                if (!(isnan(n1.x) && isnan(n2.x)) ) bad++;
            }
        }
    }
    {   /* sqrt_near_one against sqrt for every bit pattern within 2048 ulps of 1 */
        long long k = (long long)((blockIdx.x*blockDim.x + threadIdx.x) % 4097) - 2048;
        double sv = __longlong_as_double(0x3FF0000000000000LL + k);
        if (__double_as_longlong(sqrt_near_one(sv)) != __double_as_longlong(sqrt(sv))) bad++;
    }
    if (bad) atomicAdd(mismatch, bad);
}

/* Fixed-order reduction of the valid records of each tile.  RT_RED_SPLIT CTAs per
 * tile each add up a contiguous range of records (thread t takes records t,
 * t+256, ... ascending, then a fixed binary tree over the 256 thread sums); the
 * CTA that finishes last (ticket) combines the RT_RED_SPLIT partials in order. */
#define RT_RED_THREADS 256
#define RT_RED_SPLIT 16

/* Record layouts of the reductions.  A record holds ACC accumulated columns, then (in scratch
 * records) a valid flag at column ACC; W doubles per record and per summary row.  SH: row stride
 * of reduce_tile's shared-memory tree. */
struct SpotLayout {        /* RT_SUMMARY_DOUBLES: spot sums */
    static constexpr int W = RT_SUMMARY_DOUBLES, ACC = RT_ACC, N_ITEM = RT_ITEM_SUMS, SH = RT_SUMMARY_DOUBLES + 1;
    static __device__ __forceinline__ constexpr bool is_min(int k) { return k == 10 || k == 12; }
    static __device__ __forceinline__ constexpr bool is_max(int k) { return k == 11 || k == 13; }
    /* column of per-item sum j: sum_x, sum_y, sum_xx, sum_yy, sum_xy, sum_op */
    static __device__ __forceinline__ constexpr int item_col(int j) { return j < 5 ? 5 + j : 14; }
};
struct WfeLayout {         /* RT_WFE_DOUBLES: wavefront-error sums */
    static constexpr int W = RT_WFE_DOUBLES, ACC = 20, N_ITEM = RT_WFE_ITEM_SUMS, SH = 21;
    static __device__ __forceinline__ constexpr bool is_min(int k) { return k == 5; }
    static __device__ __forceinline__ constexpr bool is_max(int k) { return k == 6; }
    static __device__ __forceinline__ constexpr int item_col(int j) { return 7 + j; }
};

struct TolLayout {         /* RT_TOL_DOUBLES: tolerance records; the records are work items */
    static constexpr int W = RT_TOL_DOUBLES, ACC = RT_TOL_VALID, N_ITEM = 1, SH = RT_TOL_VALID + 1;  /* no item sums */
    static __device__ __forceinline__ constexpr bool is_min(int k) { return k == 10 || k == 12; }
    static __device__ __forceinline__ constexpr bool is_max(int k) { return k == 11 || k == 13; }
    static __device__ __forceinline__ constexpr int item_col(int j) { return j; }
};

template <typename L>
__device__ __forceinline__ double red_op(int k, double a, double y)
{
    if (L::is_min(k)) return fmin(a, y);
    if (L::is_max(k)) return fmax(a, y);
    return a + y;
}

template <typename L>
__device__ __forceinline__ double red_identity(int k)
{
    return L::is_min(k) ? CUDART_INF : (L::is_max(k) ? -CUDART_INF : 0.0);
}

/* body of k_reduce_summary / k_reduce_wfe for the records of layout L.  FOCUS: the summary tiles
 * are n planes x n_tiles grid tiles (plane-major) and plane k's per-item sums start at
 * item_sums + k*plane_items*L::N_ITEM */
template <typename L, bool FOCUS>
__device__ __forceinline__ void reduce_tile(const double *__restrict__ scratch, int64_t recs_per_tile,
                                            double *partials, unsigned int *tickets,
                                            double *__restrict__ summary, const double *__restrict__ item_sums,
                                            int64_t chunk_begin, int64_t chunk_end, int64_t chunks_per_tile,
                                            int64_t n_tiles, int64_t plane_items)
{
    __shared__ double sh[RT_RED_THREADS][L::SH];
    __shared__ bool last;
    const int64_t tile = blockIdx.x/RT_RED_SPLIT;
    const int part = blockIdx.x%RT_RED_SPLIT;
    const int64_t plane = FOCUS ? tile/n_tiles : 0;
    const int64_t gtile = FOCUS ? tile - plane*n_tiles : tile;     /* the grid tile whose chunks it covers */
    if (FOCUS && item_sums) item_sums += plane*plane_items*L::N_ITEM;
    const int64_t per = (recs_per_tile + RT_RED_SPLIT - 1)/RT_RED_SPLIT;
    int64_t r0 = part*per, r1 = r0 + per;
    if (r1 > recs_per_tile) r1 = recs_per_tile;
    double x[L::ACC];
#pragma unroll
    for (int k = 0; k < L::ACC; k++) x[k] = red_identity<L>(k);
    for (int64_t r = r0 + threadIdx.x; r < r1; r += RT_RED_THREADS) {
        const double *p = scratch + (tile*recs_per_tile + r)*L::W;
        if (p[L::ACC] != 0.0) {
#pragma unroll
            for (int k = 0; k < L::ACC; k++) x[k] = red_op<L>(k, x[k], p[k]);
        }
    }
    if (item_sums) {
        /* the work items of this tile inside the launch's chunk range, in item order: thread t of
         * part p takes items t, t + 256, ... of the part's contiguous range */
        int64_t c0 = gtile*chunks_per_tile, c1 = c0 + chunks_per_tile;
        if (c0 < chunk_begin) c0 = chunk_begin;
        if (c1 > chunk_end) c1 = chunk_end;
        if (c1 > c0) {
            const int64_t i0 = (c0 - chunk_begin)*RT_WARPS, n_it = (c1 - c0)*RT_WARPS;
            const int64_t per_it = (n_it + RT_RED_SPLIT - 1)/RT_RED_SPLIT;
            int64_t a0 = part*per_it, a1 = a0 + per_it;
            if (a1 > n_it) a1 = n_it;
            int col[L::N_ITEM];
#pragma unroll
            for (int k = 0; k < L::N_ITEM; k++) col[k] = L::item_col(k);
            for (int64_t it = a0 + threadIdx.x; it < a1; it += RT_RED_THREADS) {
                const double *p = item_sums + (i0 + it)*L::N_ITEM;
#pragma unroll
                for (int k = 0; k < L::N_ITEM; k++) x[col[k]] += p[k];
            }
        }
    }
#pragma unroll
    for (int k = 0; k < L::ACC; k++) sh[threadIdx.x][k] = x[k];
    __syncthreads();
    for (int off = RT_RED_THREADS/2; off > 0; off >>= 1) {
        if (threadIdx.x < off) {
#pragma unroll
            for (int k = 0; k < L::ACC; k++)
                sh[threadIdx.x][k] = red_op<L>(k, sh[threadIdx.x][k], sh[threadIdx.x + off][k]);
        }
        __syncthreads();
    }
    double *mine = partials + ((int64_t)blockIdx.x)*L::W;
    if (threadIdx.x < L::ACC) mine[threadIdx.x] = sh[0][threadIdx.x];
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = (atomicAdd(&tickets[tile], 1u) == RT_RED_SPLIT - 1);
    __syncthreads();
    if (last && threadIdx.x < L::W) {
        __threadfence();
        const int k = threadIdx.x;
        double v = 0.0;
        if (k < L::ACC) {
            const volatile double *pp = partials + tile*RT_RED_SPLIT*L::W;
            v = pp[k];
            for (int j = 1; j < RT_RED_SPLIT; j++) v = red_op<L>(k, v, pp[j*L::W + k]);
        }
        summary[tile*L::W + k] = v;
    }
}

__global__ void __launch_bounds__(RT_RED_THREADS)
k_reduce_summary(const double *__restrict__ scratch, int64_t recs_per_tile, double *partials,
                 unsigned int *tickets, double *__restrict__ summary,
                 const double *__restrict__ item_sums, int64_t chunk_begin, int64_t chunk_end,
                 int64_t chunks_per_tile)
{
    reduce_tile<SpotLayout, false>(scratch, recs_per_tile, partials, tickets, summary, item_sums, chunk_begin,
                                   chunk_end, chunks_per_tile, 0, 0);
}

/* k_reduce_summary over the n planes x n_tiles summary tiles of rt_trace_grid_focus */
__global__ void __launch_bounds__(RT_RED_THREADS)
k_reduce_summary_focus(const double *__restrict__ scratch, int64_t recs_per_tile, double *partials,
                       unsigned int *tickets, double *__restrict__ summary,
                       const double *__restrict__ item_sums, int64_t chunk_begin, int64_t chunk_end,
                       int64_t chunks_per_tile, int64_t n_tiles, int64_t plane_items)
{
    reduce_tile<SpotLayout, true>(scratch, recs_per_tile, partials, tickets, summary, item_sums, chunk_begin,
                                  chunk_end, chunks_per_tile, n_tiles, plane_items);
}

/* k_reduce_summary for the wavefront-error records and item sums of rt_trace_grid_wfe */
__global__ void __launch_bounds__(RT_RED_THREADS)
k_reduce_wfe(const double *__restrict__ scratch, int64_t recs_per_tile, double *partials,
             unsigned int *tickets, double *__restrict__ summary,
             const double *__restrict__ item_sums, int64_t chunk_begin, int64_t chunk_end,
             int64_t chunks_per_tile)
{
    reduce_tile<WfeLayout, false>(scratch, recs_per_tile, partials, tickets, summary, item_sums, chunk_begin,
                                  chunk_end, chunks_per_tile, 0, 0);
}

/* k_reduce_summary for the per-item records of rt_trace_grid_variants: one summary tile per (variant,
 * grid tile), whose records are its work items in item order */
__global__ void __launch_bounds__(RT_RED_THREADS)
k_reduce_tol(const double *__restrict__ items, int64_t items_per_tile, double *partials, unsigned int *tickets,
             double *__restrict__ record)
{
    reduce_tile<TolLayout, false>(items, items_per_tile, partials, tickets, record, nullptr, 0, 0, 1, 0, 0);
}

/* k_reduce_tol for the per-item wavefront-error records of rt_trace_grid_variants_wfe */
__global__ void __launch_bounds__(RT_RED_THREADS)
k_reduce_variants_wfe(const double *__restrict__ items, int64_t items_per_tile, double *partials,
                      unsigned int *tickets, double *__restrict__ record)
{
    reduce_tile<WfeLayout, false>(items, items_per_tile, partials, tickets, record, nullptr, 0, 0, 1, 0, 0);
}

/* summary of an empty chunk range: zero counts / sums, identities in the min / max columns */
__global__ void k_summary_identity(double *__restrict__ summary, int64_t n)
{
    const int64_t i = (int64_t)blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int k = (int)(i % RT_SUMMARY_DOUBLES);
    summary[i] = (k == 10 || k == 12) ? CUDART_INF : ((k == 11 || k == 13) ? -CUDART_INF : 0.0);
}

/* k_summary_identity for wavefront-error records */
__global__ void k_wfe_identity(double *__restrict__ summary, int64_t n)
{
    const int64_t i = (int64_t)blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= n) return;
    summary[i] = red_identity<WfeLayout>((int)(i % RT_WFE_DOUBLES));
}

/* out[tile][k] = parts[0][tile][k] (+|min|max) parts[1][tile][k] ... in part order */
template <typename L>
__device__ __forceinline__ void combine_rows(const double *__restrict__ parts, int n_parts, int64_t n,
                                             double *__restrict__ out)
{
    const int64_t i = (int64_t)blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int k = (int)(i % L::W);
    double v = parts[i];
    for (int p = 1; p < n_parts; p++) v = red_op<L>(k, v, parts[(int64_t)p*n + i]);
    out[i] = v;
}

__global__ void k_combine_summaries(const double *__restrict__ parts, int n_parts, int64_t n,
                                    double *__restrict__ out)
{
    combine_rows<SpotLayout>(parts, n_parts, n, out);
}

__global__ void k_combine_wfe(const double *__restrict__ parts, int n_parts, int64_t n, double *__restrict__ out)
{
    combine_rows<WfeLayout>(parts, n_parts, n, out);
}

/* ---- Zernike moments (rt_grid_zernike): per tile the packed Gram matrix of the augmented row
 * a = [W, Z_1 ... Z_J] of its used rays (status 0, r2 <= 1).  One warp per chunk (256 rays of one
 * tile).  The warp evaluates a for 32 rays at a time, one ray per lane, into shared memory; then every
 * lane runs over those 32 rows in ray order and adds a_i*a_j into a fixed register block of ROWS x 8
 * entries of the triangle.  Every entry is thus one chain over the chunk's rays in ray order, from
 * +0.0 (DESIGN.md section 4); no atomics.  The chunk's record goes to scratch and k_reduce_zernike
 * adds the tile's chunk records in chunk order. */
#define RT_ZERN_WARPS 4          /* warps (= chunks) per CTA of k_zernike_moments */
#define RT_ZERN_ROW 41           /* shared row stride in doubles: 5 blocks of 8 columns + 1 (odd: stores by
                                  * 16 lanes to one column hit 16 distinct bank pairs) */
#define RT_ZERN_HEAD 9           /* record columns before the Gram block */

struct ZernLayout {        /* RT_ZERN_DOUBLES: Zernike moments */
    static constexpr int W = RT_ZERN_DOUBLES;
    static __device__ __forceinline__ constexpr bool is_min(int k) { return k == 6; }
    static __device__ __forceinline__ constexpr bool is_max(int k) { return k == 7; }
};

/* shared slot of column d of an augmented row: column-major over 5 blocks of 8, so that the 5 block
 * columns one lane-load instruction touches are adjacent (1 wavefront for the 8-wide block loads, at
 * most 2 for the row loads) */
__device__ __forceinline__ int zern_slot(int d) { return (d & 7)*5 + (d >> 3); }

/* ROWS: rows of the lane's register block (4 for J >= 24, 2 for J >= 8, else 1), so that the
 * triangle's n_blocks (n_blocks + 1)/2 pairs of 8-blocks x 8/ROWS parts fit in 32 lanes */
template <int ROWS>
__global__ void __launch_bounds__(RT_ZERN_WARPS*32, 3)
k_zernike_moments(GridDev G, int64_t chunk_begin, int64_t chunk_end, int n_terms, int n_blocks,
                  const int32_t *__restrict__ status, const double *__restrict__ opd, double *__restrict__ rec,
                  int64_t rec_stride)
{
    __shared__ double sh[RT_ZERN_WARPS][32*RT_ZERN_ROW];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t c = chunk_begin + (int64_t)blockIdx.x*RT_ZERN_WARPS + warp;
    if (c >= chunk_end) return;
    double *A = sh[warp];
    const int64_t tile = c/G.chunks_per_tile, lc = c - tile*G.chunks_per_tile;
    const int f = (int)(tile/G.n_wvls);
    const int64_t tile0 = chunk_begin/G.chunks_per_tile;
    const int64_t ray0 = tile0*G.rays_per_tile + (chunk_begin - tile0*G.chunks_per_tile)*RT_BLOCK;

    /* the lane's block: pair p of 8-blocks (I <= Jb, numbered Jb-major), rows ROWS*part ... of block I */
    constexpr int PARTS = 8/ROWS;
    const int p = lane/PARTS, part = lane - p*PARTS;
    int I = p, Jb = 0;
    while (Jb < 5 && I > Jb) { I -= Jb + 1; Jb++; }
    const bool active = Jb < n_blocks;
    if (!active) { I = 0; Jb = 0; }               /* computes a block it does not store */
    const int i0 = 8*I + ROWS*part, j0 = 8*Jb;
    int si[ROWS], sj[8];
#pragma unroll
    for (int k = 0; k < ROWS; k++) si[k] = zern_slot(i0 + k);
#pragma unroll
    for (int q = 0; q < 8; q++) sj[q] = zern_slot(j0 + q);

    double acc[ROWS][8];
#pragma unroll
    for (int k = 0; k < ROWS; k++)
#pragma unroll
        for (int q = 0; q < 8; q++) acc[k][q] = 0.0;
    int cnt[5] = {0, 0, 0, 0, 0}, n_used = 0;     /* lane 0's */
    double mn = CUDART_INF, mx = -CUDART_INF;
    const int n_cols = 8*n_blocks;
    double *row = A + lane*RT_ZERN_ROW;
    for (int s = 0; s < RT_WARPS; s++) {
        const int64_t loc = lc*RT_BLOCK + s*32 + lane;
        const bool have = loc < G.rays_per_tile;
        int st = 0;
        double W = 0.0, x = 0.0, y = 0.0;
        if (have) {
            const int64_t k = tile*G.rays_per_tile + loc - ray0;
            st = status[k];
            W = opd[k];
            grid_pupil_coords(G, f, loc, x, y);
        }
        const bool used = have && st == RT_RAY_OK && x*x + y*y <= 1.0;
        const int ck = (st >= 0 && st <= RT_RAY_BLOCKED) ? st : 4;
#pragma unroll
        for (int cl = 0; cl < 5; cl++) cnt[cl] += __popc(__ballot_sync(0xffffffffu, have && ck == cl));
        n_used += __popc(__ballot_sync(0xffffffffu, used));
        if (used) { mn = fmin(mn, W); mx = fmax(mx, W); }
        /* the augmented row of this lane's ray; +0.0 for a ray that is not used and past J */
        row[zern_slot(0)] = used ? W : 0.0;
        fringe_zernike(x, y, n_terms, [&](int j, double z) { row[zern_slot(j)] = used ? z : 0.0; });
        for (int d = n_terms + 1; d < n_cols; d++) row[zern_slot(d)] = 0.0;
        __syncwarp();
#pragma unroll 4
        for (int r = 0; r < 32; r++) {
            const double *ar = A + r*RT_ZERN_ROW;
            double ai[ROWS], aj[8];
#pragma unroll
            for (int k = 0; k < ROWS; k++) ai[k] = ar[si[k]];
#pragma unroll
            for (int q = 0; q < 8; q++) aj[q] = ar[sj[q]];
#pragma unroll
            for (int k = 0; k < ROWS; k++)
#pragma unroll
                for (int q = 0; q < 8; q++) acc[k][q] = acc[k][q] + ai[k]*aj[q];
        }
        __syncwarp();
    }
    double *out = rec + (c - chunk_begin)*rec_stride;
    if (active) {
#pragma unroll
        for (int k = 0; k < ROWS; k++)
#pragma unroll
            for (int q = 0; q < 8; q++) {
                const int i = i0 + k, j = j0 + q;
                if (i <= j && j <= n_terms) out[RT_ZERN_HEAD + j*(j + 1)/2 + i] = acc[k][q];
            }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        mn = fmin(mn, __shfl_xor_sync(0xffffffffu, mn, off));
        mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    }
    if (lane == 0) {
#pragma unroll
        for (int cl = 0; cl < 5; cl++) out[cl] = (double)cnt[cl];
        out[5] = (double)n_used;
        out[6] = mn;
        out[7] = mx;
        out[8] = 0.0;
    }
}

/* one thread per (tile, record column): the tile's chunk records inside the range added in chunk
 * order from +0.0 (counts too; column 6 fmin, 7 fmax).  Columns past the launch's record width and
 * tiles without chunks in the range get the identity.  The chain is sequential, so the loads of
 * RT_ZERN_RED_BATCH chunks are issued before their additions: one memory latency per batch. */
#define RT_ZERN_RED_THREADS 64
#define RT_ZERN_RED_BATCH 32
__global__ void __launch_bounds__(RT_ZERN_RED_THREADS)
k_reduce_zernike(const double *__restrict__ rec, int64_t rec_stride, int64_t chunk_begin, int64_t chunk_end,
                 int64_t chunks_per_tile, int64_t n_tiles, double *__restrict__ summary)
{
    const int64_t i = (int64_t)blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= n_tiles*RT_ZERN_DOUBLES) return;
    const int64_t tile = i/RT_ZERN_DOUBLES;
    const int k = (int)(i - tile*RT_ZERN_DOUBLES);
    double v = red_identity<ZernLayout>(k);
    if (k < rec_stride) {
        const int64_t c0 = tile*chunks_per_tile > chunk_begin ? tile*chunks_per_tile : chunk_begin;
        const int64_t c1 = (tile + 1)*chunks_per_tile < chunk_end ? (tile + 1)*chunks_per_tile : chunk_end;
        const double *p = rec + (c0 - chunk_begin)*rec_stride + k;
        int64_t c = c0;
        for (; c + RT_ZERN_RED_BATCH <= c1; c += RT_ZERN_RED_BATCH, p += RT_ZERN_RED_BATCH*rec_stride) {
            double b[RT_ZERN_RED_BATCH];
#pragma unroll
            for (int q = 0; q < RT_ZERN_RED_BATCH; q++) b[q] = p[q*rec_stride];
#pragma unroll
            for (int q = 0; q < RT_ZERN_RED_BATCH; q++) v = red_op<ZernLayout>(k, v, b[q]);
        }
        for (; c < c1; c++, p += rec_stride) v = red_op<ZernLayout>(k, v, *p);
    }
    summary[i] = v;
}

__global__ void k_zernike_identity(double *__restrict__ summary, int64_t n)
{
    const int64_t i = (int64_t)blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= n) return;
    summary[i] = red_identity<ZernLayout>((int)(i % RT_ZERN_DOUBLES));
}

__global__ void k_combine_zernike(const double *__restrict__ parts, int n_parts, int64_t n, double *__restrict__ out)
{
    combine_rows<ZernLayout>(parts, n_parts, n, out);
}

/* ---- diffraction MTF (rt_grid_pupil_function, rt_grid_mtf; rt_mtf.cuh).  Tiles of n x n rays,
 * ray (i, j) at i*n + j. */
#define RT_MTF_THREADS 256

/* one thread per ray: the phasor into P[tile][i*n + j] and its transposed copy PT[tile][j*n + i],
 * from which k_mtf reads the lines along y with coalesced loads */
__global__ void __launch_bounds__(RT_MTF_THREADS)
k_pupil_function(GridDev G, int64_t n_rays, const int32_t *__restrict__ status, const double *__restrict__ opd,
                 const double *__restrict__ wvl_sys, MtfC *__restrict__ P, MtfC *__restrict__ PT)
{
    const int64_t r = (int64_t)blockIdx.x*blockDim.x + threadIdx.x;
    if (r >= n_rays) return;
    const int n = G.nx;
    const int64_t tile = r/G.rays_per_tile, loc = r - tile*G.rays_per_tile;
    const int64_t i = loc/n, j = loc - i*n;
    const int f = (int)(tile/G.n_wvls);
    const double x = G.pupil_x[(int64_t)f*n + i], y = G.pupil_y[(int64_t)f*n + j];
    const MtfC p = mtf_used(status[r], x, y) ? mtf_phasor(opd[r], wvl_sys[tile]) : MtfC{0.0, 0.0};
    P[r] = p;
    PT[tile*G.rays_per_tile + j*n + i] = p;
}

/* One CTA per (tile, slot), slot = 0 ... 2m with m = n_shifts: slot s < m is Cx(shift s), m + s is
 * Cy(shift s), 2m the tile's record; shift s is shifts[s], or s itself when shifts is NULL (every
 * shift, rt_grid_mtf).  A thread per line (strided over the CTA) adds its line in index order;
 * thread 0 then adds the line sums in line order (rt_mtf.cuh).  Lines along x are the columns of P
 * and lines along y the columns of PT, so a warp's loads are always 32 adjacent values.  No
 * atomics, no scratch.  A listed shift outside [0, n-1] gives NaN. */
__global__ void __launch_bounds__(RT_MTF_THREADS)
k_mtf(GridDev G, const int32_t *__restrict__ status, const MtfC *__restrict__ P, const MtfC *__restrict__ PT,
      const int32_t *__restrict__ shifts, int n_shifts, MtfC *__restrict__ acf_x, MtfC *__restrict__ acf_y,
      double *__restrict__ rec)
{
    __shared__ MtfC lines[RT_MTF_MAX_RAYS];
    __shared__ int cnt[RT_MTF_THREADS][6];
    const int n = G.nx, m = n_shifts;
    const int64_t tile = blockIdx.x/(2*m + 1);
    const int slot = (int)(blockIdx.x - tile*(2*m + 1));
    const int64_t base = tile*G.rays_per_tile;
    if (slot < 2*m) {
        const bool ax = slot < m;
        const int s = ax ? slot : slot - m;
        const int k = shifts ? shifts[s] : s;
        MtfC *dst = (ax ? acf_x : acf_y) + tile*m + s;
        if (k < 0 || k >= n) {
            if (threadIdx.x == 0) *dst = MtfC{CUDART_NAN, CUDART_NAN};
            return;
        }
        const MtfC *src = (ax ? P : PT) + base;
        for (int l = threadIdx.x; l < n; l += blockDim.x) lines[l] = mtf_line_shift(src + l, n, n, k);
        __syncthreads();
        if (threadIdx.x == 0) *dst = mtf_line_sum(lines, 1, n);
        return;
    }
    /* the record: S = sum P (lines along x), the status classes and the used rays */
    const int f = (int)(tile/G.n_wvls);
    int c[6] = {0, 0, 0, 0, 0, 0};
    for (int l = threadIdx.x; l < n; l += blockDim.x) {
        lines[l] = mtf_line_sum(P + base + l, n, n);
        const double y = G.pupil_y[(int64_t)f*n + l];
        for (int i = 0; i < n; i++) {
            const int st = status[base + (int64_t)i*n + l];
            const int ck = (st >= 0 && st <= RT_RAY_BLOCKED) ? st : 4;
#pragma unroll
            for (int q = 0; q < 5; q++) c[q] += ck == q;          /* constant indices: c stays in registers */
            c[5] += mtf_used(st, G.pupil_x[(int64_t)f*n + i], y);
        }
    }
#pragma unroll
    for (int q = 0; q < 6; q++) cnt[threadIdx.x][q] = c[q];
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int t = 1; t < blockDim.x; t++)
#pragma unroll
            for (int q = 0; q < 6; q++) c[q] += cnt[t][q];
        const MtfC s = mtf_line_sum(lines, 1, n);
        double *out = rec + tile*RT_MTF_DOUBLES;
#pragma unroll
        for (int q = 0; q < 6; q++) out[q] = (double)c[q];
        out[6] = s.re;
        out[7] = s.im;
    }
}

/* ---- relative illumination (rt_grid_illumination; rt_illum.cuh).  Tiles of n x n rays, ray (i, j) at
 * i*n + j.  A tile's columns are split over a cluster of RT_ILLUM_CLUSTER_MAX CTAs at most, one thread per
 * column. */
#define RT_ILLUM_THREADS 128
#define RT_ILLUM_CLUSTER_MAX 8

/* one row of a column as a thread walks it: its pupil x, and status, L, M (status -1 past the grid's
 * edge); the lanes at a warp's edge also hold the ray beside them in the next warp's column (e*) */
struct IllumRow {
    int st, est;
    double x, L, M, eL, eM;
};

/* row i of the column that starts at ray `col` */
__device__ __forceinline__ IllumRow illum_row(const int32_t *__restrict__ status, const double *__restrict__ L,
                                              const double *__restrict__ M, const double *__restrict__ px,
                                              int64_t col, int n, int i, bool in, int de, bool edge)
{
    IllumRow w{-1, -1, 0.0, 0.0, 0.0, 0.0, 0.0};
    if (i < n) {
        const int64_t r = col + (int64_t)i*n;
        w.x = px[i];
        if (in) {
            w.st = status[r];
            w.L = L[r];
            w.M = M[r];
        }
        if (in && edge) {
            w.est = status[r + de];
            w.eL = L[r + de];
            w.eM = M[r + de];
        }
    }
    return w;
}

__device__ __forceinline__ IllumPt illum_pt(int st, double L, double M)
{
    return IllumPt{L, M, st == 0};
}

/* One cluster of CTAs per tile; CTA `rank` of the cluster takes columns rank*blockDim.x ..., one thread
 * per column.  Each thread walks its column in increasing i with rows i-1, i, i+1 in registers and rows
 * i+2, i+3 already loaded, so a warp's loads are 32 adjacent rays of one row; the neighbours along j come
 * from the adjacent lanes (the lanes at a warp's edge load theirs with the row).  The column chains and
 * the counts go to the shared memory of the cluster's first CTA, whose thread 0 adds the columns in
 * increasing j (rt_illum.cuh).  No atomics, no scratch. */
__global__ void __launch_bounds__(RT_ILLUM_THREADS)
k_illumination(GridDev G, const int32_t *__restrict__ status, const double *__restrict__ L,
               const double *__restrict__ M, double *__restrict__ rec)
{
    __shared__ double col_abs[RT_ILLUM_MAX_RAYS], col_j[RT_ILLUM_MAX_RAYS];
    __shared__ int cnt[RT_ILLUM_CLUSTER_MAX*RT_ILLUM_THREADS/32][8];
    cg::cluster_group cluster = cg::this_cluster();
    const int rank = (int)cluster.block_rank(), n_cta = (int)cluster.num_blocks();
    const int n = G.nx;
    const int64_t tile = blockIdx.x/n_cta;
    const int f = (int)(tile/G.n_wvls);
    const double *px = G.pupil_x + (int64_t)f*n, *py = G.pupil_y + (int64_t)f*n;
    const int lane = threadIdx.x & 31, de = lane == 0 ? -1 : 1;
    const int j = rank*blockDim.x + threadIdx.x;
    const bool in = j < n;
    const bool edge = (lane == 0 && j > 0) || (lane == 31 && j + 1 < n);
    const double y0 = in ? py[j] : 0.0;
    const double y_m = in && j > 0 ? py[j - 1] : y0, y_p = in && j + 1 < n ? py[j + 1] : y0;
    const int64_t col = tile*G.rays_per_tile + j;
    int c[8] = {0, 0, 0, 0, 0, 0, 0, 0};       /* status classes 0-4, used, disk, isolated */
    IllumRow r0{-1, -1, 0.0, 0.0, 0.0, 0.0, 0.0};
    IllumRow r1 = illum_row(status, L, M, px, col, n, 0, in, de, edge);
    IllumRow r2 = illum_row(status, L, M, px, col, n, 1, in, de, edge);
    IllumRow r3 = illum_row(status, L, M, px, col, n, 2, in, de, edge);
    IllumRow r4 = illum_row(status, L, M, px, col, n, 3, in, de, edge);
    IllumAcc acc{0.0, 0.0};
    /* unrolled by the window's length, so that the rows rotate by renaming: a copy would wait for the
     * load of row i+4 one iteration after it was issued */
#pragma unroll 5
    for (int i = 0; i < n; i++) {
        /* row i's neighbours along j */
        int st_m = __shfl_up_sync(0xffffffffu, r1.st, 1), st_p = __shfl_down_sync(0xffffffffu, r1.st, 1);
        double L_m = __shfl_up_sync(0xffffffffu, r1.L, 1), L_p = __shfl_down_sync(0xffffffffu, r1.L, 1);
        double M_m = __shfl_up_sync(0xffffffffu, r1.M, 1), M_p = __shfl_down_sync(0xffffffffu, r1.M, 1);
        if (lane == 0) {
            st_m = r1.est;
            L_m = r1.eL;
            M_m = r1.eM;
        }
        if (lane == 31) {
            st_p = r1.est;
            L_p = r1.eL;
            M_p = r1.eM;
        }
        const double x0 = r1.x, x_m = i > 0 ? r0.x : x0, x_p = i + 1 < n ? r2.x : x0;
        if (in) {
            const int ck = (r1.st >= 0 && r1.st <= RT_RAY_BLOCKED) ? r1.st : 4;
#pragma unroll
            for (int q = 0; q < 5; q++) c[q] += ck == q;          /* constant indices: c stays in registers */
            c[6] += x0*x0 + y0*y0 <= 1.0;
            if (illum_used(r1.st, x0, y0)) {
                c[5]++;
                if (!illum_term(acc, illum_pt(r1.st, r1.L, r1.M), illum_pt(r0.st, r0.L, r0.M),
                                illum_pt(r2.st, r2.L, r2.M), illum_pt(st_m, L_m, M_m), illum_pt(st_p, L_p, M_p),
                                x_m, x0, x_p, y_m, y0, y_p))
                    c[7]++;
            }
        }
        r0 = r1;
        r1 = r2;
        r2 = r3;
        r3 = r4;
        r4 = illum_row(status, L, M, px, col, n, i + 4, in, de, edge);
    }
#pragma unroll
    for (int q = 0; q < 8; q++) c[q] = __reduce_add_sync(0xffffffffu, c[q]);
    cluster.sync();                                     /* every CTA of the cluster has started */
    double *abs0 = cluster.map_shared_rank(col_abs, 0), *j0 = cluster.map_shared_rank(col_j, 0);
    int *cnt0 = cluster.map_shared_rank(&cnt[0][0], 0);
    if (in) {
        abs0[j] = acc.abs_j;
        j0[j] = acc.j;
    }
    if (lane == 0) {
        const int w = rank*(int)(blockDim.x/32) + (int)(threadIdx.x/32);
#pragma unroll
        for (int q = 0; q < 8; q++) cnt0[w*8 + q] = c[q];
    }
    cluster.sync();
    if (rank == 0 && threadIdx.x == 0) {
        for (int w = 1; w < n_cta*(int)(blockDim.x/32); w++)
#pragma unroll
            for (int q = 0; q < 8; q++) c[q] += cnt[w][q];
        double *out = rec + tile*RT_ILLUM_DOUBLES;
#pragma unroll
        for (int q = 0; q < 8; q++) out[q] = (double)c[q];
        out[8] = illum_line_sum(col_abs, n);
        out[9] = illum_line_sum(col_j, n);
    }
}

/* chief rays of all fields: pupil (0, 0), no vignetting, apertures not checked, general
 * per-ray code on the global table (bit-identical to the lean loop by construction, and
 * n_fields rays do not need the specialised kernel).  One thread per field. */
__global__ void k_chief_ref(const rt_surface_desc *__restrict__ g_surfs, const double *__restrict__ g_n,
                            int n_ifc, GridDev G, int n_fields, int pupil_kind, int wi,
                            const double *__restrict__ g_wvl, rt_opts o, double *__restrict__ ref_img,
                            double *__restrict__ ref_out)
{
    const int f = blockIdx.x*blockDim.x + threadIdx.x;
    if (f >= n_fields) return;
    Vec3 p0, d0;
    grid_start_ray_at<false>(G, pupil_kind, f, 0.0, 0.0, false, p0, d0);
    FullWriter fw = {nullptr, 0};
    RayResult R;
    trace_ray<false>(g_surfs, g_n + (int64_t)wi*n_ifc, g_wvl[wi], n_ifc, o, p0, d0, fw, R);
    for (int w = 0; w < G.n_wvls; w++) {
        ref_img[((int64_t)f*G.n_wvls + w)*2 + 0] = R.p.x;
        ref_img[((int64_t)f*G.n_wvls + w)*2 + 1] = R.p.y;
    }
    if (ref_out) { ref_out[f*2 + 0] = R.p.x; ref_out[f*2 + 1] = R.p.y; }
}

/* the chief rays of k_chief_ref, their image intercepts defocused to every plane with the
 * expression of the grid epilogue: ref_out[k][f] = p + (foc[k]/d_z) d.  blockDim.x = RT_MAX_FOCUS */
__global__ void __launch_bounds__(RT_MAX_FOCUS)
k_chief_ref_focus(const rt_surface_desc *__restrict__ g_surfs, const double *__restrict__ g_n,
                  int n_ifc, GridDev G, int n_fields, int pupil_kind, int wi,
                  const double *__restrict__ g_wvl, rt_opts o, FocusList foc, int n_foc,
                  double *__restrict__ ref_out)
{
    __shared__ double s_foc[RT_MAX_FOCUS];
    stage_focus(foc, n_foc, s_foc);
    const int f = blockIdx.x*blockDim.x + threadIdx.x;
    if (f >= n_fields) return;
    Vec3 p0, d0;
    grid_start_ray_at<false>(G, pupil_kind, f, 0.0, 0.0, false, p0, d0);
    FullWriter fw = {nullptr, 0};
    RayResult R;
    trace_ray<false>(g_surfs, g_n + (int64_t)wi*n_ifc, g_wvl[wi], n_ifc, o, p0, d0, fw, R);
    for (int k = 0; k < n_foc; k++) {
        const double dist = div_maybe_zero(s_foc[k], R.d.z);
        ref_out[((int64_t)k*n_fields + f)*2 + 0] = R.p.x + dist*R.d.x;
        ref_out[((int64_t)k*n_fields + f)*2 + 1] = R.p.y + dist*R.d.y;
    }
}

/* chief-ray aiming of every field of a grid (rt_grid_aim_chief): aim_chief_ray of rt_aim.cuh, one
 * thread per field, the table read from global memory as in k_chief_ref */
__global__ void k_aim_chief(const rt_surface_desc *__restrict__ g_surfs, const double *__restrict__ g_n,
                            int n_ifc, GridDev G, int n_fields, int stop, int wi,
                            const double *__restrict__ g_wvl, rt_opts o, double h, double tol, int max_iter,
                            double *__restrict__ aim_out, int32_t *__restrict__ term_out)
{
    const int f = blockIdx.x*blockDim.x + threadIdx.x;
    if (f >= n_fields) return;
    double ax, ay;
    int iters;
    const int term = aim_chief_ray(g_surfs, g_n + (int64_t)wi*n_ifc, g_wvl[wi], G, f, stop, o, h, tol, max_iter,
                                   ax, ay, iters);
    aim_out[f*2 + 0] = ax;
    aim_out[f*2 + 1] = ay;
    if (term_out) term_out[f] = term;
}

/* fp64 FMA microbenchmark: 8 independent chains per thread */
__global__ void __launch_bounds__(256) k_dfma_peak(double *out, int iters, double a, double b)
{
    double x0 = threadIdx.x, x1 = x0 + 1, x2 = x0 + 2, x3 = x0 + 3;
    double x4 = x0 + 4, x5 = x0 + 5, x6 = x0 + 6, x7 = x0 + 7;
    for (int i = 0; i < iters; i++) {
        x0 = __fma_rn(x0, a, b); x1 = __fma_rn(x1, a, b);
        x2 = __fma_rn(x2, a, b); x3 = __fma_rn(x3, a, b);
        x4 = __fma_rn(x4, a, b); x5 = __fma_rn(x5, a, b);
        x6 = __fma_rn(x6, a, b); x7 = __fma_rn(x7, a, b);
    }
    double s = ((x0 + x1) + (x2 + x3)) + ((x4 + x5) + (x6 + x7));
    if (s == 12345.678) out[blockIdx.x*blockDim.x + threadIdx.x] = s;
}

/* dependent-issue latency of the fp64 pipe: one warp, one chain of DFMAs, clock64 around it */
__global__ void k_dfma_latency(double *out, long long *cycles, int iters, double a, double b)
{
    double x = threadIdx.x;
    long long t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < iters; i++) x = __fma_rn(x, a, b);
    long long t1 = clock64();
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
    if (x == 12345.678) out[threadIdx.x] = x;
}

/* ------------------------------------------------------------ launch helpers */
/* records (16 doubles each): n_tiles x min(chunks_per_tile, RT_MAX_GRID) x RT_WARPS, then
 * the reduce kernel's partials (n_tiles x RT_RED_SPLIT records) and tickets */
static int64_t scratch_records(const rt_grid *g)
{
    const int64_t sl = g->chunks_per_tile < RT_MAX_GRID ? g->chunks_per_tile : RT_MAX_GRID;
    return g->n_tiles*sl*RT_WARPS;
}

/* doubles before the per-item sums: records, the reduce kernel's partials, tickets */
static int64_t scratch_head_doubles(const rt_grid *g)
{
    return (scratch_records(g) + g->n_tiles*RT_RED_SPLIT)*RT_SUMMARY_DOUBLES + g->n_tiles;
}

template <typename K>
static int persistent_grid(K kernel, size_t smem, int sm_count, int64_t work_items, int *grid)
{
    int per_sm = 0;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, RT_BLOCK, smem));
    if (per_sm < 1) per_sm = 1;
    int64_t g = (int64_t)sm_count*per_sm;
    if (g > work_items) g = work_items;
    if (g > RT_MAX_GRID) g = RT_MAX_GRID;
    if (g < 1) g = 1;
    *grid = (int)g;
    return RT_OK;
}

template <typename K>
static int prep_kernel(K kernel, size_t smem)
{
    if (smem > 48*1024)
        CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    return RT_OK;
}

static int check_opts(const rt_table *t, const rt_opts *o)
{
    if (!o) return fail(RT_ERR_INVALID, "opts is NULL");
    if (o->wvl_idx < 0 || o->wvl_idx >= t->n_wvl) return fail(RT_ERR_INVALID, "opts.wvl_idx out of range");
    return RT_OK;
}

template <bool FULL, bool STAGE>
static int launch_bundle(const rt_table *t, int64_t n_rays, const double *px, const double *py,
                         const double *pz, const double *dx, const double *dy, const double *dz,
                         const int32_t *wvl_idx, const rt_opts *o, const rt_out *out,
                         cudaStream_t stream)
{
    auto kern = k_trace_bundle<FULL, STAGE>;
    const size_t smem = STAGE ? t->stage_bytes : 0;
    int rc = prep_kernel(kern, smem);
    if (rc) return rc;
    int grid;
    rc = persistent_grid(kern, smem, t->sm_count, (n_rays + RT_BLOCK - 1)/RT_BLOCK, &grid);
    if (rc) return rc;
    kern<<<grid, RT_BLOCK, smem, stream>>>(t->d_surfs, t->d_n, t->n_ifc, t->n_wvl, n_rays,
                                           px, py, pz, dx, dy, dz, wvl_idx, *o, *out, t->d_wvl);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RT_OK;
}

/* work counter of one launch (NULL: static schedule, unless `always`): a slot of the table's ring,
 * zeroed on the stream */
static int launch_counter(const rt_table *t, cudaStream_t stream, unsigned long long **out, bool always = false)
{
    *out = nullptr;
    if (!t->dynamic && !always) return RT_OK;
    rt_table *tt = const_cast<rt_table *>(t);
    unsigned long long *c = t->d_counters + (tt->next_counter++ % RT_COUNTERS);
    CUDA_TRY(cudaMemsetAsync(c, 0, sizeof(unsigned long long), stream));
    *out = c;
    return RT_OK;
}

template <bool FULL, bool SUMMARY, bool STAGE, bool WAVE = false>
static int launch_grid(const rt_table *t, const rt_grid *g, const GridDev &G, int64_t cb, int64_t ce,
                       const rt_opts *o, const rt_out *out, double *scratch, cudaStream_t stream)
{
    auto kern = k_trace_grid<FULL, SUMMARY, STAGE, WAVE>;
    const size_t smem = (STAGE ? t->stage_bytes : 0) + (SUMMARY ? RT_ACC_BYTES : 0);
    int rc = prep_kernel(kern, smem);
    if (rc) return rc;
    int grid;
    rc = persistent_grid(kern, smem, t->sm_count, ce - cb, &grid);
    if (rc) return rc;
    unsigned long long *wc;
    rc = launch_counter(t, stream, &wc);
    if (rc) return rc;
    g_last_grid = grid;
    kern<<<grid, RT_BLOCK, smem, stream>>>(t->d_surfs, t->d_n, t->n_ifc, t->n_wvl, G, cb, ce, *o, *out,
                                           scratch, t->d_wvl, g->pupil_kind, wc,
                                           (wc && SUMMARY) ? scratch + g_item_off : nullptr);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RT_OK;
}

template <int OUT, bool POLY>
static int launch_bundle_lean_(const rt_table *t, int64_t n_rays, const double *px, const double *py,
                              const double *pz, const double *dx, const double *dy, const double *dz,
                              const int32_t *wvl_idx, const rt_opts *o, const rt_out *out,
                              cudaStream_t stream)
{
    auto kern = k_trace_bundle_lean<OUT, POLY>;   /* (lean kernels: no phase elements, no wavelengths) */
    const size_t smem = t->lean_bytes;
    int rc = prep_kernel(kern, smem);
    if (rc) return rc;
    int grid;
    rc = persistent_grid(kern, smem, t->sm_count, (n_rays + RT_BLOCK - 1)/RT_BLOCK, &grid);
    if (rc) return rc;
    kern<<<grid, RT_BLOCK, smem, stream>>>(t->d_surfs, t->d_n, t->n_ifc, t->n_wvl, n_rays,
                                           px, py, pz, dx, dy, dz, wvl_idx, *o, *out);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RT_OK;
}

template <int OUT, bool SUMMARY, bool WAVE, bool POLY>
static int launch_grid_lean_(const rt_table *t, const GridDev &G, int64_t cb, int64_t ce,
                            const rt_opts *o, const rt_out *out, double *scratch, cudaStream_t stream)
{
    auto kern = k_trace_grid_lean<OUT, SUMMARY, WAVE, POLY>;
    const size_t smem = t->lean_bytes + (SUMMARY ? RT_ACC_BYTES : 0);
    int rc = prep_kernel(kern, smem);
    if (rc) return rc;
    int grid;
    rc = persistent_grid(kern, smem, t->sm_count, ce - cb, &grid);
    if (rc) return rc;
    unsigned long long *wc;
    rc = launch_counter(t, stream, &wc);
    if (rc) return rc;
    g_last_grid = grid;
    kern<<<grid, RT_BLOCK, smem, stream>>>(t->d_surfs, t->d_n, t->n_ifc, t->n_wvl, G, cb, ce, *o, *out,
                                           scratch, wc, (wc && SUMMARY) ? scratch + g_item_off : nullptr);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RT_OK;
}

template <int OUT>
static int launch_bundle_lean(const rt_table *t, int64_t n_rays, const double *px, const double *py,
                              const double *pz, const double *dx, const double *dy, const double *dz,
                              const int32_t *wvl_idx, const rt_opts *o, const rt_out *out,
                              cudaStream_t stream)
{
    return t->lean_poly
        ? launch_bundle_lean_<OUT, true>(t, n_rays, px, py, pz, dx, dy, dz, wvl_idx, o, out, stream)
        : launch_bundle_lean_<OUT, false>(t, n_rays, px, py, pz, dx, dy, dz, wvl_idx, o, out, stream);
}

template <int OUT, bool SUMMARY, bool WAVE = false>
static int launch_grid_lean(const rt_table *t, const GridDev &G, int64_t cb, int64_t ce,
                            const rt_opts *o, const rt_out *out, double *scratch, cudaStream_t stream)
{
    return t->lean_poly ? launch_grid_lean_<OUT, SUMMARY, WAVE, true>(t, G, cb, ce, o, out, scratch, stream)
                        : launch_grid_lean_<OUT, SUMMARY, WAVE, false>(t, G, cb, ce, o, out, scratch, stream);
}

/* CTAs of the summary launch rt_trace_grid would make over [cb, ce) (per-ray outputs of kind 0):
 * that grid decides whether the summary records are per chunk */
static int single_focus_grid(const rt_table *t, const rt_grid *g, int64_t cb, int64_t ce, int *grid)
{
    int rc;
    if (t->lean && g->pupil_kind == RT_PUPIL_EPD) {
        const size_t smem = t->lean_bytes + RT_ACC_BYTES;
        auto kern = t->lean_poly ? k_trace_grid_lean<0, true, false, true> : k_trace_grid_lean<0, true, false, false>;
        if ((rc = prep_kernel(kern, smem))) return rc;
        return persistent_grid(kern, smem, t->sm_count, ce - cb, grid);
    }
    const size_t smem = (t->stage ? t->stage_bytes : 0) + RT_ACC_BYTES;
    auto kern = t->stage ? k_trace_grid<false, true, true, false> : k_trace_grid<false, true, false, false>;
    if ((rc = prep_kernel(kern, smem))) return rc;
    return persistent_grid(kern, smem, t->sm_count, ce - cb, grid);
}

template <typename K, typename... Args>
static int launch_item_kernel(K kern, size_t smem, const rt_table *t, const rt_grid *g, int64_t cb, int64_t ce,
                               bool chunk_slots, cudaStream_t stream, Args... args)
{
    int rc = prep_kernel(kern, smem);
    if (rc) return rc;
    int grid;
    if ((rc = persistent_grid(kern, smem, t->sm_count, ce - cb, &grid))) return rc;
    /* per-(tile, CTA, warp) records: blockIdx.x must stay below the slots of a tile */
    if (!chunk_slots && grid > g->chunks_per_tile) grid = (int)g->chunks_per_tile;
    kern<<<grid, RT_BLOCK, smem, stream>>>(args...);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RT_OK;
}

/* 0: p,d only; 1: + normal/dst; 2: whole ray */
static int out_kind(const rt_out *out)
{
    if (out->full) return 2;
    if (out->nx || out->ny || out->nz || out->dst) return 1;
    return 0;
}

static GridDev grid_dev(const rt_grid *g)
{
    GridDev G;
    G.n_wvls = g->n_wvls; G.nx = g->nx; G.ny = g->ny;
    G.apply_vignetting = g->apply_vignetting; G.flip_z_dir = g->flip_z_dir; G.paired = g->paired;
    G.eprad = g->eprad; G.z_pupil = g->z_pupil; G.foc = g->foc;
    G.fields = g->d_fields; G.wvl_idx = g->d_wvl_idx;
    G.pupil_x = g->d_pupil_x; G.pupil_y = g->d_pupil_y; G.ref_img = g->d_ref_img; G.wave = g->d_wave;
    G.rays_per_tile = g->rays_per_tile; G.chunks_per_tile = g->chunks_per_tile;
    return G;
}

/* the descriptor fields the kernels index or switch on, for rt_table_create / rt_variants_create */
static int check_descs(const char *fn, const rt_surface_desc *surfs, int64_t n)
{
    for (int64_t i = 0; i < n; i++) {
        const rt_surface_desc &s = surfs[i];
        if (s.profile < RT_PROFILE_SPHERICAL || s.profile > RT_PROFILE_THINLENS)
            return fail(RT_ERR_UNSUPPORTED, "%s: unknown profile id", fn);
        if (s.mode < RT_MODE_TRANSMIT || s.mode > RT_MODE_PHANTOM)
            return fail(RT_ERR_UNSUPPORTED, "%s: unknown interact mode", fn);
        if (s.n_coefs < 0 || s.n_coefs > RT_MAX_COEFS || s.n_apertures < 0 ||
            s.n_apertures > RT_MAX_APERTURES)
            return fail(RT_ERR_INVALID, "%s: coefficient / aperture count out of range", fn);
        if (s.phase_kind < RT_PHASE_NONE || s.phase_kind > RT_PHASE_RADIAL)
            return fail(RT_ERR_UNSUPPORTED, "%s: unknown phase element kind", fn);
        if (s.n_phase_coefs < 0 || s.n_phase_coefs > RT_MAX_PHASE_COEFS)
            return fail(RT_ERR_INVALID, "%s: phase coefficient count out of range", fn);
    }
    return RT_OK;
}

/* RT_ERR_UNSUPPORTED unless every variant of [var_begin, var_end) can carry the OPD epilogue (the
 * refusal of rt_trace_grid_wfe: >= 3 interfaces and no decenter on the last one before the image --
 * which also keeps the image gap of an infinite-reference tile untilted and undecentered) */
static int check_variants_wave(const char *fn, const rt_variants *v, int32_t var_begin, int32_t var_end)
{
    for (int32_t i = var_begin; i < var_end; i++)
        if (!v->wave_ok[i])
            return fail(RT_ERR_UNSUPPORTED, "%s: opd needs >= 3 interfaces and no decenter on the last one before "
                        "the image", fn);
    return RT_OK;
}

/* rt_trace_grid_variants[_wfe]: the argument checks, the scratch (item records | partials | tickets; both
 * records are 24 doubles) and the two launches.  wfe: the _wfe launch, whose wave records are `wave` */
template <typename Kern, typename Red>
static int variants_launch(const char *fn, Kern kern, Red red, bool wfe, const rt_variants *v, const rt_grid *g,
                           int32_t var_begin, int32_t var_end, const rt_opts *o, const double *wave, double *record,
                           void *scratch, void *stream)
{
    static_assert(RT_TOL_DOUBLES == RT_WFE_DOUBLES, "one scratch layout");
    if (!v || !g || !o) return fail(RT_ERR_INVALID, "%s: bad arguments", fn);
    if (var_begin < 0 || var_end > v->n_var || var_end < var_begin)
        return fail(RT_ERR_INVALID, "%s: variant range out of bounds", fn);
    if (var_end > var_begin && (!record || !scratch))
        return fail(RT_ERR_INVALID, "%s: record and scratch are required", fn);
    if (wfe && var_end > var_begin && !wave) return fail(RT_ERR_INVALID, "%s: wave records are required", fn);
    if (v->device != g->device)
        return fail(RT_ERR_INVALID, "%s: variants and grid on different devices", fn);
    if (o->wvl_idx < 0 || o->wvl_idx >= v->n_wvl) return fail(RT_ERR_INVALID, "opts.wvl_idx out of range");
    for (int32_t wi : g->h_wvl_idx)
        if (wi < 0 || wi >= v->n_wvl)
            return fail(RT_ERR_INVALID, "%s: the grid's wvl_idx is out of range for the variants", fn);
    if (wfe)
        if (int rc = check_variants_wave(fn, v, var_begin, var_end)) return rc;
    if (var_end == var_begin) return RT_OK;
    DeviceGuard guard(v->device);
    cudaStream_t s = (cudaStream_t)stream;
    const int32_t n_var = var_end - var_begin;
    const int64_t tiles = (int64_t)n_var*g->n_tiles;
    const int64_t n_items = n_var*g->n_chunks*RT_WARPS;
    double *items = (double *)scratch;
    double *partials = items + n_items*RT_TOL_DOUBLES;
    unsigned int *tickets = (unsigned int *)(partials + tiles*RT_RED_SPLIT*RT_TOL_DOUBLES);
    /* every item record is written by the trace and every partial before it is read: clear the tickets */
    CUDA_TRY(cudaMemsetAsync(tickets, 0, (size_t)tiles*sizeof(unsigned int), s));
    rt_variants *vv = const_cast<rt_variants *>(v);
    unsigned long long *wc = v->d_counters + (vv->next_counter++ % RT_COUNTERS);
    CUDA_TRY(cudaMemsetAsync(wc, 0, sizeof(unsigned long long), s));
    VariantPlan P;
    P.items = items; P.n_var = n_var; P.n_tiles = (int32_t)g->n_tiles; P.wave = wave;
    int grid;
    int rc = persistent_grid(kern, 0, v->sm_count, n_items/RT_WARPS, &grid);
    if (rc) return rc;
    kern<<<grid, RT_BLOCK, 0, s>>>(v->d_surfs + (int64_t)var_begin*v->n_ifc,
                                   v->d_n + (int64_t)var_begin*v->n_wvl*v->n_ifc, v->n_ifc,
                                   v->n_wvl, grid_dev(g), g->n_chunks, *o, v->d_wvl,
                                   g->pupil_kind, wc, P);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    red<<<(unsigned)(tiles*RT_RED_SPLIT), RT_RED_THREADS, 0, s>>>(
        items, g->chunks_per_tile*RT_WARPS, partials, tickets, record);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RT_OK;
}

/* ------------------------------------------------------------------ C ABI */
extern "C" {

int rt_abi_version(void) { return RT_ABI_VERSION; }
int32_t rt_chunk_rays(void) { return RT_BLOCK; }
const char *rt_last_error(void) { return g_err.c_str(); }
int64_t rt_launch_count(void) { return g_launches.load(); }

int rt_table_create(const rt_surface_desc *surfs, int32_t n_ifc, const double *n_by_wvl,
                    int32_t n_wvl, int32_t device, rt_table **out)
{
    if (!surfs || !n_by_wvl || !out || n_ifc < 2 || n_wvl < 1)
        return fail(RT_ERR_INVALID, "rt_table_create: bad arguments");
    int rc = check_descs("rt_table_create", surfs, n_ifc);
    if (rc) return rc;
    DeviceGuard guard(device);
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    rt_table *t = new (std::nothrow) rt_table();
    if (!t) return fail(RT_ERR_NOMEM, "rt_table_create: out of host memory");
    t->device = device; t->n_ifc = n_ifc; t->n_wvl = n_wvl;
    t->sm_count = prop.multiProcessorCount;
    t->d_surfs = nullptr; t->d_n = nullptr; t->d_wvl = nullptr; t->has_phase = false;
    t->stage_bytes = (size_t)n_ifc*sizeof(rt_surface_desc) + (size_t)n_ifc*n_wvl*sizeof(double);
    t->stage = t->stage_bytes <= RT_MAX_STAGE_BYTES - RT_ACC_BYTES;
    t->lean_bytes = (size_t)n_ifc*sizeof(LeanSurf) + (size_t)n_ifc*n_wvl*sizeof(LeanIdx);
    t->lean = t->lean_bytes <= RT_MAX_STAGE_BYTES - RT_ACC_BYTES;
    t->lean_poly = false;
    for (int i = 0; i < n_ifc; i++) {
        const rt_surface_desc &s = surfs[i];
        if (s.has_tfrm != 0 || s.n_apertures != 0) t->lean = false;
        if (s.phase_kind != RT_PHASE_NONE || s.profile == RT_PROFILE_THINLENS) { t->lean = false; t->has_phase = true; }
        if (s.profile > RT_PROFILE_CONIC) t->lean_poly = true;
    }
    if (t->lean_poly) {
        t->lean_bytes += (size_t)n_ifc*sizeof(LeanPoly);
        if (t->lean_bytes > RT_MAX_STAGE_BYTES - RT_ACC_BYTES) t->lean = false;
    }
    if (getenv("B200RT_NO_LEAN")) t->lean = false;
    /* grid kernels: warps draw 32-ray work items from a counter (B200RT_STATIC=1: fixed round robin
     * of chunks over CTAs, kept for comparison) */
    t->dynamic = getenv("B200RT_STATIC") == nullptr;
    t->d_counters = nullptr; t->next_counter = 0;
    {
        const rt_surface_desc &k = surfs[n_ifc >= 2 ? n_ifc - 2 : 0];
        t->wave_ok = n_ifc >= 3 && k.has_tfrm == 0 && k.t[0] == 0.0 && k.t[1] == 0.0;
    }
    cudaError_t e = cudaMalloc(&t->d_surfs, (size_t)n_ifc*sizeof(rt_surface_desc));
    if (e == cudaSuccess) e = cudaMalloc(&t->d_n, (size_t)n_ifc*n_wvl*sizeof(double));
    if (e == cudaSuccess)
        e = cudaMemcpy(t->d_surfs, surfs, (size_t)n_ifc*sizeof(rt_surface_desc), cudaMemcpyHostToDevice);
    if (e == cudaSuccess)
        e = cudaMemcpy(t->d_n, n_by_wvl, (size_t)n_ifc*n_wvl*sizeof(double), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMalloc(&t->d_wvl, (size_t)n_wvl*sizeof(double));
    if (e == cudaSuccess) e = cudaMalloc(&t->d_counters, RT_COUNTERS*sizeof(unsigned long long));
    if (e == cudaSuccess) {
        std::vector<double> nanv((size_t)n_wvl, (double)NAN);
        e = cudaMemcpy(t->d_wvl, nanv.data(), (size_t)n_wvl*sizeof(double), cudaMemcpyHostToDevice);
    }
    /* pageable copies: see rt_grid_create */
    if (e == cudaSuccess) e = cudaStreamSynchronize(cudaStreamLegacy);
    if (e != cudaSuccess) {
        cudaFree(t->d_surfs); cudaFree(t->d_n); cudaFree(t->d_wvl); cudaFree(t->d_counters); delete t;
        return fail(RT_ERR_CUDA, "rt_table_create: %s", cudaGetErrorString(e));
    }
    *out = t;
    return RT_OK;
}

int rt_table_destroy(rt_table *t)
{
    if (!t) return RT_OK;
    DeviceGuard guard(t->device);
    cudaFree(t->d_surfs);
    cudaFree(t->d_n);
    cudaFree(t->d_wvl);
    cudaFree(t->d_counters);
    delete t;
    return RT_OK;
}

int rt_table_set_wavelengths(rt_table *t, const double *wvl_nm)
{
    if (!t || !wvl_nm) return fail(RT_ERR_INVALID, "rt_table_set_wavelengths: bad arguments");
    DeviceGuard guard(t->device);
    CUDA_TRY(cudaMemcpy(t->d_wvl, wvl_nm, (size_t)t->n_wvl*sizeof(double), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaStreamSynchronize(cudaStreamLegacy));
    return RT_OK;
}

int rt_table_dims(const rt_table *t, int32_t *n_ifc, int32_t *n_wvl, int32_t *device)
{
    if (!t) return fail(RT_ERR_INVALID, "rt_table_dims: NULL table");
    if (n_ifc) *n_ifc = t->n_ifc;
    if (n_wvl) *n_wvl = t->n_wvl;
    if (device) *device = t->device;
    return RT_OK;
}

int rt_trace_bundle(const rt_table *t, int64_t n_rays, const double *px, const double *py,
                    const double *pz, const double *dx, const double *dy, const double *dz,
                    const int32_t *wvl_idx, const rt_opts *o, const rt_out *out, void *stream)
{
    if (!t || !out || n_rays < 0 || !px || !py || !pz || !dx || !dy || !dz)
        return fail(RT_ERR_INVALID, "rt_trace_bundle: bad arguments");
    int rc = check_opts(t, o);
    if (rc) return rc;
    if (n_rays == 0) return RT_OK;
    if (out->full && out->full_stride < n_rays)
        return fail(RT_ERR_INVALID, "rt_trace_bundle: full_stride < n_rays");
    DeviceGuard guard(t->device);
    cudaStream_t s = (cudaStream_t)stream;
    if (t->lean) {
        switch (out_kind(out)) {
        case 0: return launch_bundle_lean<0>(t, n_rays, px, py, pz, dx, dy, dz, wvl_idx, o, out, s);
        case 1: return launch_bundle_lean<1>(t, n_rays, px, py, pz, dx, dy, dz, wvl_idx, o, out, s);
        default: return launch_bundle_lean<2>(t, n_rays, px, py, pz, dx, dy, dz, wvl_idx, o, out, s);
        }
    }
    if (out->full) {
        return t->stage ? launch_bundle<true, true>(t, n_rays, px, py, pz, dx, dy, dz, wvl_idx, o, out, s)
                        : launch_bundle<true, false>(t, n_rays, px, py, pz, dx, dy, dz, wvl_idx, o, out, s);
    }
    return t->stage ? launch_bundle<false, true>(t, n_rays, px, py, pz, dx, dy, dz, wvl_idx, o, out, s)
                    : launch_bundle<false, false>(t, n_rays, px, py, pz, dx, dy, dz, wvl_idx, o, out, s);
}

int rt_grid_destroy(rt_grid *g)
{
    if (!g) return RT_OK;
    DeviceGuard guard(g->device);
    if (g->uploaded) { cudaEventSynchronize(g->uploaded); cudaEventDestroy(g->uploaded); }
    if (g->side_ok) {
        for (int k = 0; k < 2; k++) {
            cudaStreamSynchronize(g->side[k]); cudaStreamDestroy(g->side[k]); cudaEventDestroy(g->ev_side[k]);
        }
        cudaEventDestroy(g->ev_in);
    }
    cudaFree(g->d_block);
    cudaFreeHost(g->h_stage);
    delete g;
    return RT_OK;
}

static bool grid_spec_ok(const rt_grid_spec *spec)
{
    return spec && spec->n_fields >= 1 && spec->n_wvls >= 1 && spec->nx >= 1 && spec->ny >= 1 &&
           spec->fields && spec->wvl_idx && spec->pupil_x && spec->pupil_y &&
           !(spec->paired && spec->ny != 1) && spec->pupil_kind >= RT_PUPIL_EPD &&
           spec->pupil_kind <= RT_PUPIL_WIDE;
}

/* scalars of the description + the arrays into the pinned staging block (layout fixed at create) */
static void grid_fill(rt_grid *g, const rt_grid_spec *spec)
{
    g->apply_vignetting = spec->apply_vignetting; g->flip_z_dir = spec->flip_z_dir;
    g->pupil_kind = spec->pupil_kind;
    g->eprad = spec->eprad; g->z_pupil = spec->z_pupil; g->foc = spec->foc;
    unsigned char *st = g->h_stage;
    memcpy(st + g->o_fields, spec->fields, g->b_fields);
    memcpy(st + g->o_px, spec->pupil_x, g->b_px);
    memcpy(st + g->o_py, spec->pupil_y, g->b_py);
    if (spec->ref_img) memcpy(st + g->o_ref, spec->ref_img, g->b_ref);
    else memset(st + g->o_ref, 0, g->b_ref);
    if (g->b_wave) memcpy(st + g->o_wave, spec->wave, g->b_wave);
    memcpy(st + g->o_wvl, spec->wvl_idx, (size_t)g->n_wvls*sizeof(int32_t));
    g->h_wvl_idx.assign(spec->wvl_idx, spec->wvl_idx + g->n_wvls);
}

/* All arrays of the description live in ONE device allocation and travel as ONE copy from a
 * pinned staging block owned by the handle; rt_grid_update() re-uses both, so an analysis that
 * is called repeatedly pays one small asynchronous copy per call and no allocation. */
int rt_grid_create(const rt_grid_spec *spec, int32_t device, rt_grid **out)
{
    if (!grid_spec_ok(spec) || !out) return fail(RT_ERR_INVALID, "rt_grid_create: bad arguments");
    DeviceGuard guard(device);
    rt_grid *g = new (std::nothrow) rt_grid();
    if (!g) return fail(RT_ERR_NOMEM, "rt_grid_create: out of host memory");
    g->device = device;
    g->n_fields = spec->n_fields; g->n_wvls = spec->n_wvls; g->nx = spec->nx; g->ny = spec->ny;
    g->paired = spec->paired;
    g->rays_per_tile = (int64_t)spec->nx*spec->ny;
    g->chunks_per_tile = (g->rays_per_tile + RT_BLOCK - 1)/RT_BLOCK;
    g->n_tiles = (int64_t)spec->n_fields*spec->n_wvls;
    g->n_chunks = g->n_tiles*g->chunks_per_tile;
    g->n_rays = g->n_tiles*g->rays_per_tile;

    const size_t nf = (size_t)spec->n_fields, nw = (size_t)spec->n_wvls;
    g->b_fields = nf*sizeof(rt_field_desc);
    g->b_px = nf*spec->nx*sizeof(double);
    g->b_py = nf*(spec->paired ? spec->nx : spec->ny)*sizeof(double);
    g->b_ref = (size_t)g->n_tiles*2*sizeof(double);          /* zeros when spec->ref_img is NULL */
    g->b_wave = spec->wave ? (size_t)g->n_tiles*RT_WAVE_DOUBLES*sizeof(double) : 0;
    const size_t b_wvl = (nw*sizeof(int32_t) + 7)/8*8;
    g->o_fields = 0; g->o_px = g->o_fields + g->b_fields; g->o_py = g->o_px + g->b_px;
    g->o_ref = g->o_py + g->b_py; g->o_wave = g->o_ref + g->b_ref; g->o_wvl = g->o_wave + g->b_wave;
    g->total = g->o_wvl + b_wvl;
    g->d_block = nullptr; g->h_stage = nullptr; g->uploaded = nullptr; g->side_ok = false;
    cudaError_t e = cudaMallocHost((void **)&g->h_stage, g->total);
    if (e == cudaSuccess) e = cudaMalloc(&g->d_block, g->total);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&g->uploaded, cudaEventDisableTiming);
    if (e == cudaSuccess) {
        grid_fill(g, spec);
        e = cudaMemcpy(g->d_block, g->h_stage, g->total, cudaMemcpyHostToDevice);
    }
    /* callers launch on non-blocking streams: make the block visible to every stream */
    if (e == cudaSuccess) e = cudaStreamSynchronize(cudaStreamLegacy);
    if (e != cudaSuccess) {
        if (g->uploaded) cudaEventDestroy(g->uploaded);
        cudaFree(g->d_block);
        cudaFreeHost(g->h_stage);
        delete g;
        return fail(RT_ERR_CUDA, "rt_grid_create: %s", cudaGetErrorString(e));
    }
    unsigned char *base = (unsigned char *)g->d_block;
    g->d_fields = (rt_field_desc *)(base + g->o_fields);
    g->d_pupil_x = (double *)(base + g->o_px);
    g->d_pupil_y = (double *)(base + g->o_py);
    g->d_ref_img = (double *)(base + g->o_ref);
    g->d_wave = g->b_wave ? (double *)(base + g->o_wave) : nullptr;
    g->d_wvl_idx = (int32_t *)(base + g->o_wvl);
    *out = g;
    return RT_OK;
}

int rt_grid_update(rt_grid *g, const rt_grid_spec *spec, void *stream)
{
    if (!g || !grid_spec_ok(spec)) return fail(RT_ERR_INVALID, "rt_grid_update: bad arguments");
    if (spec->n_fields != g->n_fields || spec->n_wvls != g->n_wvls || spec->nx != g->nx ||
        spec->ny != g->ny || spec->paired != g->paired || (spec->wave != nullptr) != (g->b_wave != 0))
        return fail(RT_ERR_INVALID, "rt_grid_update: the new description has a different shape");
    DeviceGuard guard(g->device);
    CUDA_TRY(cudaEventSynchronize(g->uploaded));     /* the previous copy has left the staging block */
    grid_fill(g, spec);
    CUDA_TRY(cudaMemcpyAsync(g->d_block, g->h_stage, g->total, cudaMemcpyHostToDevice, (cudaStream_t)stream));
    CUDA_TRY(cudaEventRecord(g->uploaded, (cudaStream_t)stream));
    return RT_OK;
}

int rt_grid_dims(const rt_grid *g, int64_t *n_rays, int64_t *n_chunks, int32_t *chunk_rays)
{
    if (!g) return fail(RT_ERR_INVALID, "rt_grid_dims: NULL grid");
    if (n_rays) *n_rays = g->n_rays;
    if (n_chunks) *n_chunks = g->n_chunks;
    if (chunk_rays) *chunk_rays = RT_BLOCK;
    return RT_OK;
}

int64_t rt_grid_scratch_bytes(const rt_grid *g, int64_t chunk_begin, int64_t chunk_end)
{
    if (!g || chunk_end < chunk_begin) return 0;
    return (scratch_head_doubles(g) + (chunk_end - chunk_begin)*RT_WARPS*RT_ITEM_SUMS)*(int64_t)sizeof(double);
}

int rt_trace_grid(const rt_table *t, const rt_grid *g, int64_t chunk_begin, int64_t chunk_end,
                  const rt_opts *o, const rt_out *out, double *summary, void *scratch, void *stream)
{
    if (!t || !g || !out) return fail(RT_ERR_INVALID, "rt_trace_grid: bad arguments");
    if (t->device != g->device) return fail(RT_ERR_INVALID, "rt_trace_grid: table and grid on different devices");
    if (chunk_begin < 0 || chunk_end > g->n_chunks || chunk_end < chunk_begin)
        return fail(RT_ERR_INVALID, "rt_trace_grid: chunk range out of bounds");
    if (summary && !scratch) return fail(RT_ERR_INVALID, "rt_trace_grid: summary needs scratch");
    int rc = check_opts(t, o);
    if (rc) return rc;
    DeviceGuard guard(t->device);
    cudaStream_t s = (cudaStream_t)stream;
    for (int32_t wi : g->h_wvl_idx)
        if (wi < 0 || wi >= t->n_wvl)
            return fail(RT_ERR_INVALID, "rt_trace_grid: the grid's wvl_idx is out of range for this table");
    if (summary && chunk_begin == chunk_end) {
        /* an empty shard contributes the identity of every column (min / max: +-inf) */
        const int64_t n = g->n_tiles*RT_SUMMARY_DOUBLES;
        k_summary_identity<<<(unsigned)((n + 255)/256), 256, 0, s>>>(summary, n);
        g_launches++;
        CUDA_TRY(cudaGetLastError());
    }
    if (chunk_begin == chunk_end) return RT_OK;
    const GridDev G = grid_dev(g);
    double *scr = (double *)scratch;
    g_item_off = scratch_head_doubles(g);
    if (summary)
        CUDA_TRY(cudaMemsetAsync(scr, 0, (size_t)(t->dynamic ? rt_grid_scratch_bytes(g, chunk_begin, chunk_end)
                                                              : scratch_head_doubles(g)*(int64_t)sizeof(double)), s));
    const bool full = out->full != nullptr, summ = summary != nullptr, st = t->stage;
    const bool wave = out->opd != nullptr;
    /* angular pupil specifications are generated by the general kernels only (rt_grid.cuh) */
    const bool lean = t->lean && g->pupil_kind == RT_PUPIL_EPD;
    if (wave) {
        if (!g->d_wave) return fail(RT_ERR_INVALID, "rt_trace_grid: out.opd needs rt_grid_spec.wave");
        if (out_kind(out) != 0) return fail(RT_ERR_UNSUPPORTED, "rt_trace_grid: opd cannot be combined with normals / whole rays");
        if (!t->wave_ok)
            return fail(RT_ERR_UNSUPPORTED, "rt_trace_grid: opd needs >= 3 interfaces and no decenter on the last one before the image");
        if (lean) {
            rc = summ ? launch_grid_lean<0, true, true>(t, G, chunk_begin, chunk_end, o, out, scr, s)
                      : launch_grid_lean<0, false, true>(t, G, chunk_begin, chunk_end, o, out, scr, s);
        } else if (st) {
            rc = summ ? launch_grid<false, true, true, true>(t, g, G, chunk_begin, chunk_end, o, out, scr, s)
                      : launch_grid<false, false, true, true>(t, g, G, chunk_begin, chunk_end, o, out, scr, s);
        } else {
            rc = summ ? launch_grid<false, true, false, true>(t, g, G, chunk_begin, chunk_end, o, out, scr, s)
                      : launch_grid<false, false, false, true>(t, g, G, chunk_begin, chunk_end, o, out, scr, s);
        }
    } else if (lean) {
        const int kind = out_kind(out);
#define RT_LEAN_CASE(K, S)                                                                   \
        if (kind == K && summ == S)                                                          \
            rc = launch_grid_lean<K, S>(t, G, chunk_begin, chunk_end, o, out, scr, s);
        RT_LEAN_CASE(0, false) RT_LEAN_CASE(0, true) RT_LEAN_CASE(1, false)
        RT_LEAN_CASE(1, true) RT_LEAN_CASE(2, false) RT_LEAN_CASE(2, true)
#undef RT_LEAN_CASE
    } else {
#define RT_GRID_CASE(F, S, T)                                                               \
    if (full == F && summ == S && st == T)                                                  \
        rc = launch_grid<F, S, T>(t, g, G, chunk_begin, chunk_end, o, out, scr, s);
    RT_GRID_CASE(false, false, true)
    RT_GRID_CASE(false, true, true)
    RT_GRID_CASE(true, false, true)
    RT_GRID_CASE(true, true, true)
    RT_GRID_CASE(false, false, false)
    RT_GRID_CASE(false, true, false)
    RT_GRID_CASE(true, false, false)
    RT_GRID_CASE(true, true, false)
#undef RT_GRID_CASE
    }
    if (rc) return rc;
    if (summ) {
        const int64_t recs = scratch_records(g);
        double *partials = scr + recs*RT_SUMMARY_DOUBLES;
        unsigned int *tickets = (unsigned int *)(partials + g->n_tiles*RT_RED_SPLIT*RT_SUMMARY_DOUBLES);
        const bool chunk_slots = g->chunks_per_tile <= g_last_grid;
        k_reduce_summary<<<(unsigned)(g->n_tiles*RT_RED_SPLIT), RT_RED_THREADS, 0, s>>>(
            scr, recs/g->n_tiles, partials, tickets, summary,
            (t->dynamic && !chunk_slots) ? scr + scratch_head_doubles(g) : nullptr, chunk_begin, chunk_end,
            g->chunks_per_tile);
        g_launches++;
        CUDA_TRY(cudaGetLastError());
    }
    return RT_OK;
}

static int64_t first_ray_of_chunk(const rt_grid *g, int64_t c)
{
    const int64_t tile = c/g->chunks_per_tile, lc = c - tile*g->chunks_per_tile;
    const int64_t in_tile = lc*RT_BLOCK < g->rays_per_tile ? lc*RT_BLOCK : g->rays_per_tile;
    return tile*g->rays_per_tile + in_tile;
}

int64_t rt_trace_grid_to_host_scratch_bytes(const rt_grid *g, int32_t n_pieces)
{
    if (!g || n_pieces < 1) return 0;
    return 2*rt_grid_scratch_bytes(g, 0, g->n_chunks) +
           (int64_t)n_pieces*g->n_tiles*RT_SUMMARY_DOUBLES*(int64_t)sizeof(double);
}

/* The grid analyses' data path in one call: the chunk range is traced in n_pieces launches
 * alternating between two internal streams, and each piece's aberrations (NaN-coded status) go
 * device -> host right behind its trace, so the copy of one piece overlaps the trace of the
 * next without the caller issuing anything per piece. */
int rt_trace_grid_to_host(const rt_table *t, rt_grid *g, int64_t chunk_begin, int64_t chunk_end,
                          const rt_opts *o, double *d_abr_x, double *d_abr_y, double *h_abr_x,
                          double *h_abr_y, double *summary, void *scratch, int32_t n_pieces, void *stream)
{
    if (!t || !g || !d_abr_x || !d_abr_y || !h_abr_x || !h_abr_y || !scratch || n_pieces < 1)
        return fail(RT_ERR_INVALID, "rt_trace_grid_to_host: bad arguments");
    if (chunk_begin < 0 || chunk_end > g->n_chunks || chunk_end < chunk_begin)
        return fail(RT_ERR_INVALID, "rt_trace_grid_to_host: chunk range out of bounds");
    DeviceGuard guard(t->device);
    cudaStream_t s = (cudaStream_t)stream;
    if (!g->side_ok) {
        for (int k = 0; k < 2; k++) {
            CUDA_TRY(cudaStreamCreateWithFlags(&g->side[k], cudaStreamNonBlocking));
            CUDA_TRY(cudaEventCreateWithFlags(&g->ev_side[k], cudaEventDisableTiming));
        }
        CUDA_TRY(cudaEventCreateWithFlags(&g->ev_in, cudaEventDisableTiming));
        g->side_ok = true;
    }
    if (n_pieces > chunk_end - chunk_begin) n_pieces = (int32_t)(chunk_end - chunk_begin);
    if (n_pieces < 1) n_pieces = 1;
    const int64_t sb = rt_grid_scratch_bytes(g, 0, g->n_chunks);
    unsigned char *scr = (unsigned char *)scratch;
    double *partials = (double *)(scr + 2*sb);
    const int64_t tile_doubles = g->n_tiles*RT_SUMMARY_DOUBLES;
    const int64_t base = first_ray_of_chunk(g, chunk_begin);
    CUDA_TRY(cudaEventRecord(g->ev_in, s));                  /* grid upload, chief rays ... */
    for (int k = 0; k < 2; k++) CUDA_TRY(cudaStreamWaitEvent(g->side[k], g->ev_in, 0));
    for (int i = 0; i < n_pieces; i++) {
        const int64_t cb = chunk_begin + (chunk_end - chunk_begin)*i/n_pieces;
        const int64_t ce = chunk_begin + (chunk_end - chunk_begin)*(i + 1)/n_pieces;
        const int64_t a = first_ray_of_chunk(g, cb) - base, n = first_ray_of_chunk(g, ce) - first_ray_of_chunk(g, cb);
        cudaStream_t ss = g->side[i & 1];
        rt_out out;
        memset(&out, 0, sizeof out);
        out.abr_x = d_abr_x + a; out.abr_y = d_abr_y + a;
        out.flags = RT_OUT_ABR_NAN_STATUS;
        int rc = rt_trace_grid(t, g, cb, ce, o, &out, summary ? partials + i*tile_doubles : nullptr,
                               scr + (i & 1)*sb, ss);
        if (rc) return rc;
        CUDA_TRY(cudaMemcpyAsync(h_abr_x + a, d_abr_x + a, (size_t)n*sizeof(double), cudaMemcpyDeviceToHost, ss));
        CUDA_TRY(cudaMemcpyAsync(h_abr_y + a, d_abr_y + a, (size_t)n*sizeof(double), cudaMemcpyDeviceToHost, ss));
    }
    for (int k = 0; k < 2; k++) {
        CUDA_TRY(cudaEventRecord(g->ev_side[k], g->side[k]));
        CUDA_TRY(cudaStreamWaitEvent(s, g->ev_side[k], 0));
    }
    if (summary) return rt_combine_summaries(partials, n_pieces, g->n_tiles, summary, stream);
    return RT_OK;
}

int rt_grid_chief_ref(const rt_table *t, rt_grid *g, int32_t wvl_idx, double *ref_out, void *stream)
{
    if (!t || !g) return fail(RT_ERR_INVALID, "rt_grid_chief_ref: bad arguments");
    if (t->device != g->device) return fail(RT_ERR_INVALID, "rt_grid_chief_ref: table and grid on different devices");
    if (wvl_idx < 0 || wvl_idx >= t->n_wvl) return fail(RT_ERR_INVALID, "rt_grid_chief_ref: wvl_idx out of range");
    DeviceGuard guard(t->device);
    rt_opts o;
    o.eps = 1.0e-12; o.pt_inside_fuzz = -1.0; o.check_apertures = 0; o.intersect_obj = 1;
    o.filter_out_phantoms = 0; o.first_surf = 1; o.last_surf = t->n_ifc - 2; o.wvl_idx = wvl_idx;
    const int threads = 32, blocks = (g->n_fields + threads - 1)/threads;
    k_chief_ref<<<blocks, threads, 0, (cudaStream_t)stream>>>(t->d_surfs, t->d_n, t->n_ifc, grid_dev(g),
                                                              g->n_fields, g->pupil_kind, wvl_idx, t->d_wvl,
                                                              o, g->d_ref_img, ref_out);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RT_OK;
}

int rt_grid_aim_chief(const rt_table *t, const rt_grid *g, int32_t stop, int32_t wvl_idx, double h, double tol,
                      int32_t max_iter, double *aim_out, int32_t *term_out, void *stream)
{
    if (!t || !g) return fail(RT_ERR_INVALID, "rt_grid_aim_chief: table and grid are required");
    if (!aim_out) return fail(RT_ERR_INVALID, "rt_grid_aim_chief: aim_out is required");
    if (!(std::isfinite(h) && h > 0.0)) return fail(RT_ERR_INVALID, "rt_grid_aim_chief: h must be finite and positive");
    if (!(std::isfinite(tol) && tol > 0.0))
        return fail(RT_ERR_INVALID, "rt_grid_aim_chief: tol must be finite and positive");
    if (max_iter < 0) return fail(RT_ERR_INVALID, "rt_grid_aim_chief: max_iter must not be negative");
    if (g->pupil_kind != RT_PUPIL_EPD)
        return fail(RT_ERR_UNSUPPORTED, "rt_grid_aim_chief: only 'epd' pupils (RT_PUPIL_EPD) are aimed on the device");
    if (t->device != g->device) return fail(RT_ERR_INVALID, "rt_grid_aim_chief: table and grid on different devices");
    if (stop < 1 || stop > t->n_ifc - 2) return fail(RT_ERR_INVALID, "rt_grid_aim_chief: stop must be in 1 ... n_ifc - 2");
    if (wvl_idx < 0 || wvl_idx >= t->n_wvl) return fail(RT_ERR_INVALID, "rt_grid_aim_chief: wvl_idx out of range");
    if (g->n_fields == 0) return RT_OK;
    DeviceGuard guard(t->device);
    rt_opts o;     /* cuda_bundle_fn's trace: first_surf 1, apertures not checked, intersect_obj on */
    o.eps = 1.0e-12; o.pt_inside_fuzz = -1.0; o.check_apertures = 0; o.intersect_obj = 1;
    o.filter_out_phantoms = 0; o.first_surf = 1; o.last_surf = stop; o.wvl_idx = wvl_idx;
    const int threads = 32, blocks = (g->n_fields + threads - 1)/threads;
    k_aim_chief<<<blocks, threads, 0, (cudaStream_t)stream>>>(t->d_surfs, t->d_n, t->n_ifc, grid_dev(g), g->n_fields,
                                                              stop, wvl_idx, t->d_wvl, o, h, tol, max_iter, aim_out,
                                                              term_out);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RT_OK;
}

static int check_focus(const char *fn, const double *foc, int32_t n_foc, FocusList *L)
{
    if (n_foc < 1 || n_foc > RT_MAX_FOCUS) return fail(RT_ERR_INVALID, "%s: n_foc must be in [1, RT_MAX_FOCUS]", fn);
    if (!foc) return fail(RT_ERR_INVALID, "%s: foc is NULL", fn);
    memset(L, 0, sizeof *L);
    for (int k = 0; k < n_foc; k++) {
        if (!std::isfinite(foc[k])) return fail(RT_ERR_INVALID, "%s: foc holds a value that is not finite", fn);
        L->v[k] = foc[k];
    }
    return RT_OK;
}

int rt_grid_chief_ref_focus(const rt_table *t, const rt_grid *g, int32_t wvl_idx, const double *foc,
                            int32_t n_foc, double *ref_out, void *stream)
{
    FocusList L;
    int rc = check_focus("rt_grid_chief_ref_focus", foc, n_foc, &L);
    if (rc) return rc;
    if (!t || !g || !ref_out) return fail(RT_ERR_INVALID, "rt_grid_chief_ref_focus: bad arguments");
    if (t->device != g->device) return fail(RT_ERR_INVALID, "rt_grid_chief_ref_focus: table and grid on different devices");
    if (wvl_idx < 0 || wvl_idx >= t->n_wvl) return fail(RT_ERR_INVALID, "rt_grid_chief_ref_focus: wvl_idx out of range");
    DeviceGuard guard(t->device);
    rt_opts o;     /* as rt_grid_chief_ref */
    o.eps = 1.0e-12; o.pt_inside_fuzz = -1.0; o.check_apertures = 0; o.intersect_obj = 1;
    o.filter_out_phantoms = 0; o.first_surf = 1; o.last_surf = t->n_ifc - 2; o.wvl_idx = wvl_idx;
    const int threads = RT_MAX_FOCUS, blocks = (g->n_fields + threads - 1)/threads;
    k_chief_ref_focus<<<blocks, threads, 0, (cudaStream_t)stream>>>(t->d_surfs, t->d_n, t->n_ifc, grid_dev(g),
                                                                    g->n_fields, g->pupil_kind, wvl_idx, t->d_wvl,
                                                                    o, L, n_foc, ref_out);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RT_OK;
}

int64_t rt_grid_focus_scratch_bytes(const rt_grid *g, int32_t n_foc, int64_t chunk_begin, int64_t chunk_end)
{
    if (!g || n_foc < 1 || n_foc > RT_MAX_FOCUS || chunk_end < chunk_begin) return 0;
    return n_foc*rt_grid_scratch_bytes(g, chunk_begin, chunk_end);
}

/* scratch: records [n][n_tiles][slots][RT_WARPS][16] | partials [n*n_tiles][RT_RED_SPLIT][16] |
 * tickets [n*n_tiles] | per-item sums [n][items][RT_ITEM_SUMS] */
int rt_trace_grid_focus(const rt_table *t, const rt_grid *g, int64_t chunk_begin, int64_t chunk_end,
                        const rt_opts *o, const double *foc, int32_t n_foc, const double *ref_img,
                        const rt_out *out, double *summary, void *scratch, void *stream)
{
    FocusList L;
    int rc = check_focus("rt_trace_grid_focus", foc, n_foc, &L);
    if (rc) return rc;
    if (!summary) return fail(RT_ERR_INVALID, "rt_trace_grid_focus: summary is NULL");
    if (!out) return fail(RT_ERR_INVALID, "rt_trace_grid_focus: out is NULL");
    if (out->abr_x || out->abr_y || out->opd || out->full)
        return fail(RT_ERR_INVALID, "rt_trace_grid_focus: abr_x, abr_y, opd and full must be NULL (they depend on the plane)");
    if (out_kind(out) != 0)
        return fail(RT_ERR_INVALID, "rt_trace_grid_focus: normals and dst are not written by the through-focus trace");
    if (!t || !g || !scratch) return fail(RT_ERR_INVALID, "rt_trace_grid_focus: bad arguments");
    if (t->device != g->device) return fail(RT_ERR_INVALID, "rt_trace_grid_focus: table and grid on different devices");
    if (chunk_begin < 0 || chunk_end > g->n_chunks || chunk_end < chunk_begin)
        return fail(RT_ERR_INVALID, "rt_trace_grid_focus: chunk range out of bounds");
    if ((rc = check_opts(t, o))) return rc;
    for (int32_t wi : g->h_wvl_idx)
        if (wi < 0 || wi >= t->n_wvl)
            return fail(RT_ERR_INVALID, "rt_trace_grid_focus: the grid's wvl_idx is out of range for this table");
    DeviceGuard guard(t->device);
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t n_sum = (int64_t)n_foc*g->n_tiles;      /* summary tiles, plane-major */
    if (chunk_begin == chunk_end) {
        const int64_t n = n_sum*RT_SUMMARY_DOUBLES;
        k_summary_identity<<<(unsigned)((n + 255)/256), 256, 0, s>>>(summary, n);
        g_launches++;
        CUDA_TRY(cudaGetLastError());
        return RT_OK;
    }
    int single;
    if ((rc = single_focus_grid(t, g, chunk_begin, chunk_end, &single))) return rc;
    const bool chunk_slots = g->chunks_per_tile <= single;
    double *scr = (double *)scratch;
    const int64_t recs = scratch_records(g);                 /* per plane */
    double *partials = scr + n_foc*recs*RT_SUMMARY_DOUBLES;
    unsigned int *tickets = (unsigned int *)(partials + n_sum*RT_RED_SPLIT*RT_SUMMARY_DOUBLES);
    double *items = scr + n_foc*scratch_head_doubles(g);
    /* the per-item sums are all written by the trace: zero the records, partials and tickets only */
    CUDA_TRY(cudaMemsetAsync(scr, 0, (size_t)(n_foc*scratch_head_doubles(g))*sizeof(double), s));
    unsigned long long *wc;
    if ((rc = launch_counter(t, s, &wc, true))) return rc;
    FocusPlanes P;
    P.foc = nullptr; P.ref = ref_img; P.n_tiles = g->n_tiles;
    P.n_items = (chunk_end - chunk_begin)*RT_WARPS;
    P.n = n_foc; P.n_fields = g->n_fields; P.chunk_slots = chunk_slots; P.pad_ = 0;
    const GridDev G = grid_dev(g);
    /* angular pupil specifications are generated by the general kernels only (rt_grid.cuh) */
    if (t->lean && g->pupil_kind == RT_PUPIL_EPD) {
        auto kern = t->lean_poly ? k_trace_grid_lean_focus<true> : k_trace_grid_lean_focus<false>;
        rc = launch_item_kernel(kern, t->lean_bytes, t, g, chunk_begin, chunk_end, chunk_slots, s,
                                 t->d_surfs, t->d_n, t->n_ifc, t->n_wvl, G, chunk_begin, chunk_end, *o, *out,
                                 scr, wc, items, P, L);
    } else {
        auto kern = t->stage ? k_trace_grid_focus<true> : k_trace_grid_focus<false>;
        rc = launch_item_kernel(kern, t->stage ? t->stage_bytes : 0, t, g, chunk_begin, chunk_end, chunk_slots, s,
                                 t->d_surfs, t->d_n, t->n_ifc, t->n_wvl, G, chunk_begin, chunk_end, *o, *out,
                                 scr, t->d_wvl, g->pupil_kind, wc, items, P, L);
    }
    if (rc) return rc;
    k_reduce_summary_focus<<<(unsigned)(n_sum*RT_RED_SPLIT), RT_RED_THREADS, 0, s>>>(
        scr, recs/g->n_tiles, partials, tickets, summary, chunk_slots ? nullptr : items, chunk_begin, chunk_end,
        g->chunks_per_tile, g->n_tiles, P.n_items);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RT_OK;
}

/* the OPD of every ray against n_foc reference spheres (rt_refocus.cuh), one launch in the kernel
 * family rt_trace_grid takes for an opd launch; the schedule is rt_trace_grid's */
int rt_trace_grid_opd_focus(const rt_table *t, const rt_grid *g, int64_t chunk_begin, int64_t chunk_end,
                            const rt_opts *o, const double *spheres, int32_t n_foc, const rt_out *out,
                            double *opd_planes, void *stream)
{
    if (n_foc < 1 || n_foc > RT_MAX_FOCUS)
        return fail(RT_ERR_INVALID, "rt_trace_grid_opd_focus: n_foc must be in [1, RT_MAX_FOCUS]");
    if (!t || !g || !out || !spheres || (chunk_end > chunk_begin && !opd_planes))
        return fail(RT_ERR_INVALID, "rt_trace_grid_opd_focus: table, grid, out, spheres and opd_planes are required");
    if (out->opd || out->abr_x || out->abr_y || out->full)
        return fail(RT_ERR_INVALID, "rt_trace_grid_opd_focus: opd, abr_x, abr_y and full must be NULL");
    if (out_kind(out) != 0)
        return fail(RT_ERR_INVALID, "rt_trace_grid_opd_focus: normals and dst are not written");
    if (!g->d_wave)
        return fail(RT_ERR_INVALID, "rt_trace_grid_opd_focus: the grid has no wave records (rt_grid_spec.wave)");
    if (t->device != g->device)
        return fail(RT_ERR_INVALID, "rt_trace_grid_opd_focus: table and grid on different devices");
    if (chunk_begin < 0 || chunk_end > g->n_chunks || chunk_end < chunk_begin)
        return fail(RT_ERR_INVALID, "rt_trace_grid_opd_focus: chunk range out of bounds");
    int rc = check_opts(t, o);
    if (rc) return rc;
    for (int32_t wi : g->h_wvl_idx)
        if (wi < 0 || wi >= t->n_wvl)
            return fail(RT_ERR_INVALID, "rt_trace_grid_opd_focus: the grid's wvl_idx is out of range for this table");
    if (!t->wave_ok)
        return fail(RT_ERR_UNSUPPORTED, "rt_trace_grid_opd_focus: opd needs >= 3 interfaces and no decenter on the last one before the image");
    if (chunk_begin == chunk_end) return RT_OK;
    DeviceGuard guard(t->device);
    cudaStream_t s = (cudaStream_t)stream;
    RefocusPlanes P;
    P.spheres = spheres; P.planes = opd_planes;
    P.n_rays = first_ray_of_chunk(g, chunk_end) - first_ray_of_chunk(g, chunk_begin);
    P.sphere_stride = g->n_tiles*RT_SPHERE_DOUBLES;
    P.n = n_foc; P.pad_ = 0;
    const GridDev G = grid_dev(g);
    unsigned long long *wc;
    if ((rc = launch_counter(t, s, &wc))) return rc;
    int grid;
    /* angular pupil specifications are generated by the general kernels only (rt_grid.cuh) */
    if (t->lean && g->pupil_kind == RT_PUPIL_EPD) {
        auto kern = t->lean_poly ? k_trace_grid_lean_opd_focus<true> : k_trace_grid_lean_opd_focus<false>;
        if ((rc = prep_kernel(kern, t->lean_bytes))) return rc;
        if ((rc = persistent_grid(kern, t->lean_bytes, t->sm_count, chunk_end - chunk_begin, &grid))) return rc;
        kern<<<grid, RT_BLOCK, t->lean_bytes, s>>>(t->d_surfs, t->d_n, t->n_ifc, t->n_wvl, G, chunk_begin, chunk_end,
                                                   *o, *out, wc, P);
    } else {
        auto kern = t->stage ? k_trace_grid_opd_focus<true> : k_trace_grid_opd_focus<false>;
        const size_t smem = t->stage ? t->stage_bytes : 0;
        if ((rc = prep_kernel(kern, smem))) return rc;
        if ((rc = persistent_grid(kern, smem, t->sm_count, chunk_end - chunk_begin, &grid))) return rc;
        kern<<<grid, RT_BLOCK, smem, s>>>(t->d_surfs, t->d_n, t->n_ifc, t->n_wvl, G, chunk_begin, chunk_end, *o, *out,
                                          t->d_wvl, g->pupil_kind, wc, P);
    }
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RT_OK;
}

int rt_combine_summaries(const double *parts, int32_t n_parts, int64_t n_tiles, double *out, void *stream)
{
    if (!parts || !out || n_parts < 1 || n_tiles < 0)
        return fail(RT_ERR_INVALID, "rt_combine_summaries: bad arguments");
    if (n_tiles == 0) return RT_OK;
    const int64_t n = n_tiles*RT_SUMMARY_DOUBLES;
    k_combine_summaries<<<(unsigned)((n + 255)/256), 256, 0, (cudaStream_t)stream>>>(parts, n_parts, n, out);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RT_OK;
}

/* scratch of rt_trace_grid_wfe: records [n_tiles][slots][RT_WARPS][RT_WFE_DOUBLES] | partials
 * [n_tiles][RT_RED_SPLIT][RT_WFE_DOUBLES] | tickets [n_tiles] | per-item sums [items][RT_WFE_ITEM_SUMS] */
static int64_t wfe_head_doubles(const rt_grid *g)
{
    return (scratch_records(g) + g->n_tiles*RT_RED_SPLIT)*RT_WFE_DOUBLES + g->n_tiles;
}

int64_t rt_grid_wfe_scratch_bytes(const rt_grid *g, int64_t chunk_begin, int64_t chunk_end)
{
    if (!g || chunk_end < chunk_begin) return 0;
    return (wfe_head_doubles(g) + (chunk_end - chunk_begin)*RT_WARPS*RT_WFE_ITEM_SUMS)*(int64_t)sizeof(double);
}

int rt_trace_grid_wfe(const rt_table *t, const rt_grid *g, int64_t chunk_begin, int64_t chunk_end,
                      const rt_opts *o, const rt_out *out, double *summary, void *scratch, void *stream)
{
    if (!t || !g || !out) return fail(RT_ERR_INVALID, "rt_trace_grid_wfe: bad arguments");
    if (!summary || !scratch) return fail(RT_ERR_INVALID, "rt_trace_grid_wfe: summary and scratch are required");
    if (out->full) return fail(RT_ERR_INVALID, "rt_trace_grid_wfe: full must be NULL");
    if (!g->d_wave) return fail(RT_ERR_INVALID, "rt_trace_grid_wfe: the grid has no wave records (rt_grid_spec.wave)");
    if (t->device != g->device) return fail(RT_ERR_INVALID, "rt_trace_grid_wfe: table and grid on different devices");
    if (chunk_begin < 0 || chunk_end > g->n_chunks || chunk_end < chunk_begin)
        return fail(RT_ERR_INVALID, "rt_trace_grid_wfe: chunk range out of bounds");
    int rc = check_opts(t, o);
    if (rc) return rc;
    for (int32_t wi : g->h_wvl_idx)
        if (wi < 0 || wi >= t->n_wvl)
            return fail(RT_ERR_INVALID, "rt_trace_grid_wfe: the grid's wvl_idx is out of range for this table");
    if (out_kind(out) != 0) return fail(RT_ERR_UNSUPPORTED, "rt_trace_grid_wfe: opd cannot be combined with normals");
    if (!t->wave_ok)
        return fail(RT_ERR_UNSUPPORTED, "rt_trace_grid_wfe: opd needs >= 3 interfaces and no decenter on the last one before the image");
    DeviceGuard guard(t->device);
    cudaStream_t s = (cudaStream_t)stream;
    if (chunk_begin == chunk_end) {
        const int64_t n = g->n_tiles*RT_WFE_DOUBLES;
        k_wfe_identity<<<(unsigned)((n + 255)/256), 256, 0, s>>>(summary, n);
        g_launches++;
        CUDA_TRY(cudaGetLastError());
        return RT_OK;
    }
    double *scr = (double *)scratch;
    const int64_t recs = scratch_records(g);
    double *partials = scr + recs*RT_WFE_DOUBLES;
    unsigned int *tickets = (unsigned int *)(partials + g->n_tiles*RT_RED_SPLIT*RT_WFE_DOUBLES);
    double *items = scr + wfe_head_doubles(g);
    /* the per-item sums are all written by the trace: zero the records, partials and tickets only */
    CUDA_TRY(cudaMemsetAsync(scr, 0, (size_t)wfe_head_doubles(g)*sizeof(double), s));
    unsigned long long *wc;
    if ((rc = launch_counter(t, s, &wc, true))) return rc;
    const GridDev G = grid_dev(g);
    /* the kernel family rt_trace_grid takes for an opd launch; angular pupil specifications are
     * generated by the general kernels only (rt_grid.cuh) */
    if (t->lean && g->pupil_kind == RT_PUPIL_EPD) {
        auto kern = t->lean_poly ? k_trace_grid_lean_wfe<true> : k_trace_grid_lean_wfe<false>;
        rc = launch_item_kernel(kern, t->lean_bytes, t, g, chunk_begin, chunk_end, false, s,
                                t->d_surfs, t->d_n, t->n_ifc, t->n_wvl, G, chunk_begin, chunk_end, *o, *out,
                                scr, wc, items);
    } else {
        auto kern = t->stage ? k_trace_grid_wfe<true> : k_trace_grid_wfe<false>;
        rc = launch_item_kernel(kern, t->stage ? t->stage_bytes : 0, t, g, chunk_begin, chunk_end, false, s,
                                t->d_surfs, t->d_n, t->n_ifc, t->n_wvl, G, chunk_begin, chunk_end, *o, *out,
                                scr, t->d_wvl, g->pupil_kind, wc, items);
    }
    if (rc) return rc;
    k_reduce_wfe<<<(unsigned)(g->n_tiles*RT_RED_SPLIT), RT_RED_THREADS, 0, s>>>(
        scr, recs/g->n_tiles, partials, tickets, summary, items, chunk_begin, chunk_end, g->chunks_per_tile);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RT_OK;
}

/* ---- tolerance analysis: many prescriptions over one grid */
int rt_variants_create(const rt_surface_desc *surfs, int32_t n_ifc, const double *n_by_wvl, int32_t n_wvl,
                       int32_t n_var, const double *wvl_nm, int32_t device, rt_variants **out)
{
    if (!surfs || !n_by_wvl || !out || n_ifc < 2 || n_wvl < 1 || n_var < 1)
        return fail(RT_ERR_INVALID, "rt_variants_create: bad arguments");
    int rc = check_descs("rt_variants_create", surfs, (int64_t)n_var*n_ifc);
    if (rc) return rc;
    DeviceGuard guard(device);
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    const size_t b_s = (size_t)n_var*n_ifc*sizeof(rt_surface_desc);
    const size_t b_n = (size_t)n_var*n_wvl*n_ifc*sizeof(double), b_w = (size_t)n_wvl*sizeof(double);
    const size_t b_c = RT_COUNTERS*sizeof(unsigned long long);
    std::vector<unsigned char> h(b_s + b_n + b_w);
    memcpy(h.data(), surfs, b_s);
    memcpy(h.data() + b_s, n_by_wvl, b_n);
    for (int32_t w = 0; w < n_wvl; w++) {
        const double x = wvl_nm ? wvl_nm[w] : (double)NAN;
        memcpy(h.data() + b_s + b_n + (size_t)w*sizeof(double), &x, sizeof(double));
    }
    rt_variants *v = new (std::nothrow) rt_variants();
    if (!v) return fail(RT_ERR_NOMEM, "rt_variants_create: out of host memory");
    v->device = device; v->n_ifc = n_ifc; v->n_wvl = n_wvl; v->n_var = n_var;
    v->sm_count = prop.multiProcessorCount;
    v->wave_ok.resize((size_t)n_var);
    for (int32_t i = 0; i < n_var; i++) {      /* as rt_table_create's wave_ok */
        const rt_surface_desc &k = surfs[(int64_t)i*n_ifc + n_ifc - 2];
        v->wave_ok[i] = n_ifc >= 3 && k.has_tfrm == 0 && k.t[0] == 0.0 && k.t[1] == 0.0;
    }
    v->d_block = nullptr; v->next_counter = 0;
    cudaError_t e = cudaMalloc(&v->d_block, h.size() + b_c);
    if (e == cudaSuccess) e = cudaMemcpy(v->d_block, h.data(), h.size(), cudaMemcpyHostToDevice);
    /* pageable copies: see rt_grid_create */
    if (e == cudaSuccess) e = cudaStreamSynchronize(cudaStreamLegacy);
    if (e != cudaSuccess) {
        cudaFree(v->d_block); delete v;
        return fail(RT_ERR_CUDA, "rt_variants_create: %s", cudaGetErrorString(e));
    }
    unsigned char *base = (unsigned char *)v->d_block;
    v->d_surfs = (rt_surface_desc *)base;
    v->d_n = (double *)(base + b_s);
    v->d_wvl = (double *)(base + b_s + b_n);
    v->d_counters = (unsigned long long *)(base + b_s + b_n + b_w);
    *out = v;
    return RT_OK;
}

int rt_variants_destroy(rt_variants *v)
{
    if (!v) return RT_OK;
    DeviceGuard guard(v->device);
    cudaFree(v->d_block);
    delete v;
    return RT_OK;
}

/* scratch of rt_trace_grid_variants over n_var variants: item records [n_var][n_tiles][chunks_per_tile*RT_WARPS]
 * [RT_TOL_DOUBLES] | partials [n_var*n_tiles][RT_RED_SPLIT][RT_TOL_DOUBLES] | tickets [n_var*n_tiles] */
static int64_t tol_items(const rt_grid *g, int64_t n_var) { return n_var*g->n_chunks*RT_WARPS; }

int64_t rt_grid_variants_scratch_bytes(const rt_grid *g, int32_t n_var)
{
    if (!g || n_var < 0) return 0;
    const int64_t tiles = (int64_t)n_var*g->n_tiles;
    return ((tol_items(g, n_var) + tiles*RT_RED_SPLIT)*RT_TOL_DOUBLES + (tiles + 1)/2)*(int64_t)sizeof(double);
}

int rt_trace_grid_variants(const rt_variants *v, const rt_grid *g, int32_t var_begin, int32_t var_end,
                           const rt_opts *o, double *record, void *scratch, void *stream)
{
    return variants_launch("rt_trace_grid_variants", k_trace_grid_variants, k_reduce_tol, false, v, g, var_begin,
                           var_end, o, nullptr, record, scratch, stream);
}

int64_t rt_grid_variants_wfe_scratch_bytes(const rt_grid *g, int32_t n_var)
{
    return rt_grid_variants_scratch_bytes(g, n_var);      /* the same layout: RT_WFE_DOUBLES == RT_TOL_DOUBLES */
}

int rt_trace_grid_variants_wfe(const rt_variants *v, const rt_grid *g, int32_t var_begin, int32_t var_end,
                               const rt_opts *o, const double *wave, double *record, void *scratch, void *stream)
{
    return variants_launch("rt_trace_grid_variants_wfe", k_trace_grid_variants_wfe, k_reduce_variants_wfe, true, v, g,
                           var_begin, var_end, o, wave, record, scratch, stream);
}

int rt_variants_wave(const rt_variants *v, const rt_grid *g, int32_t var_begin, int32_t var_end, const double *parax,
                     double *wave, double *ref_img, int32_t *status, void *stream)
{
    if (!v || !g) return fail(RT_ERR_INVALID, "rt_variants_wave: bad arguments");
    if (var_begin < 0 || var_end > v->n_var || var_end < var_begin)
        return fail(RT_ERR_INVALID, "rt_variants_wave: variant range out of bounds");
    if (var_end > var_begin && (!parax || !wave || !ref_img || !status))
        return fail(RT_ERR_INVALID, "rt_variants_wave: parax, wave, ref_img and status are required");
    if (v->device != g->device)
        return fail(RT_ERR_INVALID, "rt_variants_wave: variants and grid on different devices");
    for (int32_t wi : g->h_wvl_idx)
        if (wi < 0 || wi >= v->n_wvl)
            return fail(RT_ERR_INVALID, "rt_variants_wave: the grid's wvl_idx is out of range for the variants");
    if (int rc = check_variants_wave("rt_variants_wave", v, var_begin, var_end)) return rc;
    if (var_end == var_begin) return RT_OK;
    DeviceGuard guard(v->device);
    /* the chief-ray options of waveabr.trace_chief_rays: trace_grid's defaults, apertures not checked */
    rt_opts o;
    o.eps = 1.0e-12; o.pt_inside_fuzz = -1.0;
    o.check_apertures = 0; o.intersect_obj = g->pupil_kind == RT_PUPIL_WIDE ? 0 : 1;
    o.filter_out_phantoms = 0; o.first_surf = 1; o.last_surf = v->n_ifc - 2; o.wvl_idx = 0;
    const int32_t n_var = var_end - var_begin;
    const int64_t n = (int64_t)n_var*g->n_tiles;
    const int threads = 128;
    k_variants_wave<<<(unsigned)((n + threads - 1)/threads), threads, 0, (cudaStream_t)stream>>>(
        v->d_surfs + (int64_t)var_begin*v->n_ifc, v->d_n + (int64_t)var_begin*v->n_wvl*v->n_ifc, v->n_ifc, v->n_wvl,
        grid_dev(g), (int)g->n_tiles, n_var, g->pupil_kind, v->d_wvl, o, parax[0], parax[1], parax[2], wave, ref_img,
        status);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RT_OK;
}

int rt_combine_wfe(const double *parts, int32_t n_parts, int64_t n_tiles, double *out, void *stream)
{
    if (!parts || !out || n_parts < 1 || n_tiles < 0) return fail(RT_ERR_INVALID, "rt_combine_wfe: bad arguments");
    if (n_tiles == 0) return RT_OK;
    const int64_t n = n_tiles*RT_WFE_DOUBLES;
    k_combine_wfe<<<(unsigned)((n + 255)/256), 256, 0, (cudaStream_t)stream>>>(parts, n_parts, n, out);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RT_OK;
}

/* doubles of one chunk record of rt_grid_zernike: the head and the packed Gram block of J terms */
static int64_t zern_rec_stride(int32_t n_terms)
{
    return RT_ZERN_HEAD + (int64_t)(n_terms + 1)*(n_terms + 2)/2;
}

int64_t rt_grid_zernike_scratch_bytes(const rt_grid *g, int64_t chunk_begin, int64_t chunk_end, int32_t n_terms)
{
    if (!g || chunk_begin < 0 || chunk_end < chunk_begin || chunk_end > g->n_chunks || n_terms < 1 ||
        n_terms > RT_ZERN_MAX_TERMS)
        return 0;
    return (chunk_end - chunk_begin)*zern_rec_stride(n_terms)*(int64_t)sizeof(double);
}

int rt_grid_zernike(const rt_grid *g, int64_t chunk_begin, int64_t chunk_end, int32_t n_terms,
                    const int32_t *status, const double *opd, double *summary, void *scratch, void *stream)
{
    if (!g || !summary) return fail(RT_ERR_INVALID, "rt_grid_zernike: grid and summary are required");
    if (n_terms < 1 || n_terms > RT_ZERN_MAX_TERMS) return fail(RT_ERR_INVALID, "rt_grid_zernike: n_terms must be 1 ... 37");
    if (chunk_begin < 0 || chunk_end > g->n_chunks || chunk_end < chunk_begin)
        return fail(RT_ERR_INVALID, "rt_grid_zernike: chunk range out of bounds");
    if (g->paired) return fail(RT_ERR_INVALID, "rt_grid_zernike: needs a product grid (paired = 0)");
    if (g->apply_vignetting)
        return fail(RT_ERR_INVALID, "rt_grid_zernike: the pupil coordinates must not be vignetted (apply_vignetting = 0)");
    if (chunk_end > chunk_begin && (!status || !opd || !scratch))
        return fail(RT_ERR_INVALID, "rt_grid_zernike: status, opd and scratch are required");
    DeviceGuard guard(g->device);
    cudaStream_t s = (cudaStream_t)stream;
    if (chunk_begin == chunk_end) {
        const int64_t n = g->n_tiles*RT_ZERN_DOUBLES;
        k_zernike_identity<<<(unsigned)((n + 255)/256), 256, 0, s>>>(summary, n);
        g_launches++;
        CUDA_TRY(cudaGetLastError());
        return RT_OK;
    }
    const int64_t stride = zern_rec_stride(n_terms);
    const int n_blocks = (n_terms + 1 + 7)/8, pairs = n_blocks*(n_blocks + 1)/2;
    const GridDev G = grid_dev(g);
    double *rec = (double *)scratch;
    const unsigned blocks = (unsigned)((chunk_end - chunk_begin + RT_ZERN_WARPS - 1)/RT_ZERN_WARPS);
    auto kern = pairs*8 <= 32 ? k_zernike_moments<1> : (pairs*4 <= 32 ? k_zernike_moments<2> : k_zernike_moments<4>);
    kern<<<blocks, RT_ZERN_WARPS*32, 0, s>>>(G, chunk_begin, chunk_end, n_terms, n_blocks, status, opd, rec, stride);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    const int64_t n = g->n_tiles*RT_ZERN_DOUBLES;
    k_reduce_zernike<<<(unsigned)((n + RT_ZERN_RED_THREADS - 1)/RT_ZERN_RED_THREADS), RT_ZERN_RED_THREADS, 0, s>>>(
        rec, stride, chunk_begin, chunk_end, g->chunks_per_tile, g->n_tiles, summary);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RT_OK;
}

int rt_combine_zernike(const double *parts, int32_t n_parts, int64_t n_tiles, double *out, void *stream)
{
    if (!parts || !out || n_parts < 1 || n_tiles < 0) return fail(RT_ERR_INVALID, "rt_combine_zernike: bad arguments");
    if (n_tiles == 0) return RT_OK;
    const int64_t n = n_tiles*RT_ZERN_DOUBLES;
    k_combine_zernike<<<(unsigned)((n + 255)/256), 256, 0, (cudaStream_t)stream>>>(parts, n_parts, n, out);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RT_OK;
}

/* the grid conditions of rt_grid_pupil_function / rt_grid_mtf */
static int mtf_check_grid(const rt_grid *g, const char *fn)
{
    if (!g) return fail(RT_ERR_INVALID, "%s: grid is required", fn);
    if (g->paired) return fail(RT_ERR_INVALID, "%s: needs a product grid (paired = 0)", fn);
    if (g->apply_vignetting)
        return fail(RT_ERR_INVALID, "%s: the pupil coordinates must not be vignetted (apply_vignetting = 0)", fn);
    if (g->nx != g->ny) return fail(RT_ERR_INVALID, "%s: needs a square grid (nx = ny)", fn);
    if (g->nx > RT_MTF_MAX_RAYS) return fail(RT_ERR_INVALID, "%s: nx exceeds RT_MTF_MAX_RAYS", fn);
    return RT_OK;
}

/* one k_mtf launch over n_shifts shifts per axis (shifts NULL: 0 ... n_shifts-1) */
static int launch_mtf(const rt_grid *g, const int32_t *status, const double *pupil, const double *pupil_t,
                      const int32_t *shifts, int32_t n_shifts, double *acf_x, double *acf_y, double *record,
                      void *stream)
{
    DeviceGuard guard(g->device);
    const int n = g->nx;
    const int threads = n >= RT_MTF_THREADS ? RT_MTF_THREADS : (n + 31)/32*32;
    k_mtf<<<(unsigned)(g->n_tiles*(2*(int64_t)n_shifts + 1)), threads, 0, (cudaStream_t)stream>>>(
        grid_dev(g), status, (const MtfC *)pupil, (const MtfC *)pupil_t, shifts, n_shifts, (MtfC *)acf_x,
        (MtfC *)acf_y, record);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RT_OK;
}

int rt_grid_pupil_function(const rt_grid *g, const int32_t *status, const double *opd, const double *wvl_sys,
                           double *pupil, double *pupil_t, void *stream)
{
    if (const int rc = mtf_check_grid(g, "rt_grid_pupil_function")) return rc;
    if (!status || !opd || !wvl_sys || !pupil || !pupil_t)
        return fail(RT_ERR_INVALID, "rt_grid_pupil_function: status, opd, wvl_sys, pupil and pupil_t are required");
    DeviceGuard guard(g->device);
    const int64_t n = g->n_rays;
    k_pupil_function<<<(unsigned)((n + RT_MTF_THREADS - 1)/RT_MTF_THREADS), RT_MTF_THREADS, 0, (cudaStream_t)stream>>>(
        grid_dev(g), n, status, opd, wvl_sys, (MtfC *)pupil, (MtfC *)pupil_t);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RT_OK;
}

int rt_grid_mtf(const rt_grid *g, const int32_t *status, const double *pupil, const double *pupil_t,
                double *acf_x, double *acf_y, double *record, void *stream)
{
    if (const int rc = mtf_check_grid(g, "rt_grid_mtf")) return rc;
    if (!status || !pupil || !pupil_t || !acf_x || !acf_y || !record)
        return fail(RT_ERR_INVALID, "rt_grid_mtf: status, pupil, pupil_t, acf_x, acf_y and record are required");
    return launch_mtf(g, status, pupil, pupil_t, nullptr, g->nx, acf_x, acf_y, record, stream);
}

int rt_grid_mtf_shifts(const rt_grid *g, const int32_t *status, const double *pupil, const double *pupil_t,
                       const int32_t *shifts, int32_t n_shifts, double *acf_x, double *acf_y, double *record,
                       void *stream)
{
    if (n_shifts < 0) return fail(RT_ERR_INVALID, "rt_grid_mtf_shifts: n_shifts out of range");
    if (const int rc = mtf_check_grid(g, "rt_grid_mtf_shifts")) return rc;
    if (!status || !pupil || !pupil_t || !record)
        return fail(RT_ERR_INVALID, "rt_grid_mtf_shifts: status, pupil, pupil_t and record are required");
    if (g->n_tiles*(2*(int64_t)n_shifts + 1) > INT32_MAX)
        return fail(RT_ERR_INVALID, "rt_grid_mtf_shifts: n_shifts out of range");
    if (n_shifts > 0 && (!shifts || !acf_x || !acf_y))
        return fail(RT_ERR_INVALID, "rt_grid_mtf_shifts: shifts, acf_x and acf_y are required when n_shifts > 0");
    return launch_mtf(g, status, pupil, pupil_t, shifts, n_shifts, acf_x, acf_y, record, stream);
}

int rt_grid_illumination(const rt_grid *g, const int32_t *status, const double *dx, const double *dy,
                         double *record, void *stream)
{
    const char *fn = "rt_grid_illumination";
    if (!g) return fail(RT_ERR_INVALID, "%s: grid is required", fn);
    if (g->paired) return fail(RT_ERR_INVALID, "%s: needs a product grid (paired = 0)", fn);
    if (g->apply_vignetting)
        return fail(RT_ERR_INVALID, "%s: the pupil coordinates must not be vignetted (apply_vignetting = 0)", fn);
    if (g->nx != g->ny) return fail(RT_ERR_INVALID, "%s: needs a square grid (nx = ny)", fn);
    if (g->nx < 2 || g->nx > RT_ILLUM_MAX_RAYS)
        return fail(RT_ERR_INVALID, "%s: nx must lie in 2 ... RT_ILLUM_MAX_RAYS", fn);
    if (!status || !dx || !dy || !record)
        return fail(RT_ERR_INVALID, "%s: status, dx, dy and record are required", fn);
    DeviceGuard guard(g->device);
    const int n = g->nx;
    /* at most RT_ILLUM_THREADS columns per CTA, whole warps: n <= 1024 needs at most 8 CTAs */
    const int n_cta = (n + RT_ILLUM_THREADS - 1)/RT_ILLUM_THREADS;
    const int threads = ((n + n_cta - 1)/n_cta + 31)/32*32;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(g->n_tiles*n_cta));
    cfg.blockDim = dim3((unsigned)threads);
    cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)n_cta;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    CUDA_TRY(cudaLaunchKernelEx(&cfg, k_illumination, grid_dev(g), status, dx, dy, record));
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    return RT_OK;
}

/* fp64 vector-pipe peak, measured with a DFMA chain kernel: the roofline
 * denominator for the register-resident trace (DESIGN.md "roofline"). */
int rt_measure_fp64_peak(int32_t device, double *tflops)
{
    if (!tflops) return fail(RT_ERR_INVALID, "rt_measure_fp64_peak: NULL output");
    DeviceGuard guard(device);
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    const int blocks = prop.multiProcessorCount*8, iters = 1 << 14;
    double *d_out;
    CUDA_TRY(cudaMalloc(&d_out, (size_t)blocks*256*sizeof(double)));
    cudaEvent_t e0, e1;
    CUDA_TRY(cudaEventCreate(&e0));
    CUDA_TRY(cudaEventCreate(&e1));
    double best = 0.0;
    for (int rep = 0; rep < 5; rep++) {
        CUDA_TRY(cudaEventRecord(e0));
        k_dfma_peak<<<blocks, 256>>>(d_out, iters, 0.999999, 1e-9);
        g_launches++;
        CUDA_TRY(cudaEventRecord(e1));
        CUDA_TRY(cudaEventSynchronize(e1));
        float ms = 0;
        CUDA_TRY(cudaEventElapsedTime(&ms, e0, e1));
        double fl = 2.0*8.0*(double)iters*256.0*blocks;
        double tf = fl/(ms*1e-3)/1e12;
        if (rep > 0 && tf > best) best = tf;
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(d_out);
    *tflops = best;
    return RT_OK;
}

/* Cycles between two DEPENDENT fp64 FMAs of one warp (the latency that the per-ray chains of
 * the trace kernels expose; DESIGN.md "what bounds the kernel"). */
int rt_measure_fp64_latency(int32_t device, double *cycles_per_dependent_dfma)
{
    if (!cycles_per_dependent_dfma) return fail(RT_ERR_INVALID, "rt_measure_fp64_latency: NULL output");
    DeviceGuard guard(device);
    double *d_out; long long *d_cyc;
    CUDA_TRY(cudaMalloc(&d_out, 32*sizeof(double)));
    CUDA_TRY(cudaMalloc(&d_cyc, sizeof(long long)));
    const int iters = 1 << 14;
    long long best = -1;
    for (int rep = 0; rep < 3; rep++) {
        k_dfma_latency<<<1, 32>>>(d_out, d_cyc, iters, 0.999999, 1e-9);
        g_launches++;
        long long c = 0;
        CUDA_TRY(cudaMemcpy(&c, d_cyc, sizeof c, cudaMemcpyDeviceToHost));
        if (best < 0 || c < best) best = c;
    }
    cudaFree(d_out); cudaFree(d_cyc);
    *cycles_per_dependent_dfma = (double)best/iters;
    return RT_OK;
}

/* Self-test of the shared-reciprocal division used by the lean kernels:
 * n_blocks x 256 threads x n_per_thread random operand sets (3 quotients + one
 * normalisation each) compared bit-for-bit with the IEEE `/`.  *mismatches
 * must come back 0. */
int rt_selftest_division(int32_t device, int32_t n_blocks, int64_t n_per_thread, uint64_t seed,
                         uint64_t *mismatches)
{
    if (!mismatches || n_blocks < 1 || n_per_thread < 1)
        return fail(RT_ERR_INVALID, "rt_selftest_division: bad arguments");
    DeviceGuard guard(device);
    unsigned long long *d_bad;
    CUDA_TRY(cudaMalloc(&d_bad, sizeof(unsigned long long)));
    CUDA_TRY(cudaMemset(d_bad, 0, sizeof(unsigned long long)));
    k_selftest_division<<<n_blocks, 256>>>(seed, n_per_thread, d_bad);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    unsigned long long bad = 0;
    CUDA_TRY(cudaMemcpy(&bad, d_bad, sizeof bad, cudaMemcpyDeviceToHost));
    cudaFree(d_bad);
    *mismatches = bad;
    return RT_OK;
}

}  /* extern "C" */
