/*
 * b200rt.h -- C ABI of libb200rt.so, the H100 (sm_90a) sequential real-ray
 * trace engine that replaces the hot path of mjhoptics/ray-optics:
 *
 *   rayoptics.raytr.raytrace.trace()/trace_raw()   src/rayoptics/raytr/raytrace.py:51-264
 *   and the per-ray loops stacked on it             src/rayoptics/raytr/trace.py:537-605,
 *                                                   src/rayoptics/raytr/analyses.py:212-230,437-455,666-696
 *
 * The reference is pure Python and has no FFI of its own; the binding a
 * maintainer would add is a ctypes stub (see INTEGRATION.md).  Every entry
 * point below takes plain pointers and sizes -- no torch / numpy types.
 *
 * Conventions
 *   - all functions return RT_OK (0) or a negative rt_error code; the message
 *     for the calling thread is available from rt_last_error().
 *   - per-ray failures (missed surface, TIR, blocked by an aperture) are DATA
 *     (`status`, `fail_surf` arrays), never C errors.  They map 1:1 onto the
 *     reference's TraceError subclasses (src/rayoptics/raytr/traceerror.py:11-52).
 *   - pointers documented "DEVICE" must be device pointers on the table's
 *     device; pointers documented "HOST" are host pointers that are read
 *     before the call returns.
 *   - the caller owns every ray / result buffer; the library owns only the
 *     immutable table / grid handles.  Launches are asynchronous on `stream`
 *     (a cudaStream_t passed as void*; NULL = legacy default stream).
 *   - all floating point is IEEE binary64; the arithmetic contract (which
 *     operations are fused) is stated in DESIGN.md and is what makes results
 *     bit-identical to the reference's numpy path.
 */
#ifndef B200RT_H
#define B200RT_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RT_ABI_VERSION 6
#define RT_MAX_COEFS 20     /* EvenPolynomial uses <=10, RadialPolynomial <=20 */
#define RT_MAX_PHASE_COEFS 10
#define RT_MAX_APERTURES 4  /* Surface.clear_apertures entries honoured per interface */
#define RT_SEG_DOUBLES 10   /* one ray segment = p[3], d[3], dst, nrml[3]  (raytr/__init__.py:36) */
#define RT_SUMMARY_DOUBLES 16
#define RT_WAVE_DOUBLES 24   /* per-(field, wvl) chief-ray / reference-sphere record, see rt_grid_spec.wave */
#define RT_MAX_FOCUS 64      /* image planes of one rt_trace_grid_focus call */
#define RT_WFE_DOUBLES 24    /* per-tile wavefront-error record of rt_trace_grid_wfe */
#define RT_ZERN_DOUBLES 752  /* per-tile Zernike moments record of rt_grid_zernike */
#define RT_ZERN_MAX_TERMS 37 /* Fringe Zernike terms of rt_grid_zernike */
#define RT_MTF_MAX_RAYS 1024 /* pupil samples per side of rt_grid_pupil_function / rt_grid_mtf */
#define RT_MTF_DOUBLES 8     /* per-tile record of rt_grid_mtf */
#define RT_SPHERE_DOUBLES 8  /* per-(plane, tile) reference-sphere record of rt_trace_grid_opd_focus */
#define RT_TOL_DOUBLES 24    /* per-(variant, tile) record of rt_trace_grid_variants */

/* error codes (function return values) */
enum rt_error {
    RT_OK = 0,
    RT_ERR_INVALID = -1,     /* bad argument */
    RT_ERR_CUDA = -2,        /* CUDA runtime error, text in rt_last_error() */
    RT_ERR_UNSUPPORTED = -3, /* interface type not representable in the table */
    RT_ERR_NOMEM = -4
};

/* SurfaceProfile subclasses, src/rayoptics/elem/profiles.py */
enum rt_profile {
    RT_PROFILE_SPHERICAL = 0,  /* profiles.py:218-416 */
    RT_PROFILE_CONIC = 1,      /* profiles.py:449-680 */
    RT_PROFILE_EVENPOLY = 2,   /* profiles.py:682-889 */
    RT_PROFILE_RADIALPOLY = 3, /* profiles.py:891-1116 */
    RT_PROFILE_YTOROID = 4,    /* profiles.py:1119-1372 */
    RT_PROFILE_XTOROID = 5,    /* profiles.py:1375-1437 */
    RT_PROFILE_THINLENS = 6    /* oprops/thinlens.py:130-137: plane z=0, normal (0,0,1) */
};

/* phase elements (Interface.phase_element), src/rayoptics/oprops/doe.py */
enum rt_phase {
    RT_PHASE_NONE = 0,
    RT_PHASE_HOE = 1,          /* HolographicElement, doe.py:326-395 (also every ThinLens) */
    RT_PHASE_GRATING = 2,      /* DiffractionGrating.phase_ludwig, doe.py:57-172 */
    RT_PHASE_RADIAL = 3        /* DiffractiveElement with radial_phase_fct, doe.py:28-54,214-323 */
};

/* Interface.interact_mode, src/rayoptics/seq/interface.py:42-49 */
enum rt_mode {
    RT_MODE_TRANSMIT = 0,
    RT_MODE_REFLECT = 1,
    RT_MODE_DUMMY = 2,
    RT_MODE_PHANTOM = 3
};

/* per-ray status; 1..4 are the TraceError subclasses of traceerror.py */
enum rt_status {
    RT_RAY_OK = 0,
    RT_RAY_MISSED = 1,     /* TraceMissedSurfaceError */
    RT_RAY_TIR = 2,        /* TraceTIRError */
    RT_RAY_BLOCKED = 3,    /* TraceRayBlockedError */
    RT_RAY_EVANESCENT = 4, /* TraceEvanescentRayError (phase element: sqrt of a negative, raytrace.py:41-48) */
    RT_RAY_NUMERIC = 5     /* the reference would raise an uncaught ValueError /
                              ZeroDivisionError (sqrt of a negative in
                              EvenPolynomial.df, profiles.py:870-873) */
};

/* pupil specification after the image-space substitution of opticalspec.py:311-325 */
enum rt_pupil_kind {
    RT_PUPIL_EPD = 0,   /* spatial: aim at the entrance pupil plane, opticalspec.py:329-366.
                           rt_field_desc: pt0 = -(obj_dist + z_enp) [d0x/d0z, d0y/d0z, 0], aim = aim_pt */
    RT_PUPIL_NA = 1,    /* angular, object-space NA: dir_tot = sin_ang*pupil + cr_dir, :368-398.
                           rt_field_desc: pt0 = object point p0, aim = chief ray direction d0[:2] */
    RT_PUPIL_FNO = 2,   /* angular, object-space f/#: pupil_dir = slope*pupil/hypt, :378-384 */
    RT_PUPIL_WIDE = 3   /* spatial, wide-angle fields (fov.is_wide_angle), opticalspec.py:342-358: the pupil
                           plane is normal to the chief ray.  rt_field_desc: pt0 = start point, rot = the
                           matrix rot_v1_into_v2(d0, z) that takes the pupil plane into surface-1
                           coordinates, obj2enp = -(obj_dist + z_enp) with z_enp the field's real entrance
                           pupil position (fld.aim_info, raytr/wideangle.py).  Traced with
                           intersect_obj = 0 and without the virtual-object flip (trace.py:299-303). */
};

/* Aperture subclasses, src/rayoptics/elem/surface.py:340-494 */
enum rt_aperture_type {
    RT_APERTURE_CIRCULAR = 1,    /* surface.py:397-431 */
    RT_APERTURE_RECTANGULAR = 2, /* surface.py:434-469 */
    RT_APERTURE_ELLIPTICAL = 3   /* surface.py:472-494: no point_inside() -> always blocks */
};

typedef struct rt_aperture_desc {
    int32_t type;           /* rt_aperture_type */
    int32_t is_obscuration; /* Aperture.is_obscuration */
    double a;               /* Circular.radius | x_half_width */
    double b;               /* y_half_width (unused for Circular) */
    double x_offset;        /* Aperture.x_offset */
    double y_offset;        /* Aperture.y_offset */
} rt_aperture_desc;

/* One entry of SequentialModel.path(wvl): (Intfc, Gap, Tfrm, Indx, Zdir),
 * src/rayoptics/optical/model_constants.py:12, seq/sequential.py:149-202.
 * The refractive index lives in the separate n_by_wvl table. */
typedef struct rt_surface_desc {
    int32_t profile;      /* rt_profile */
    int32_t mode;         /* rt_mode */
    int32_t z_dir;        /* path tuple Zdir: +1 / -1 */
    int32_t n_coefs;      /* profile.max_nonzero_coef (polynomial profiles) */
    int32_t has_tfrm;     /* 0: Tfrm rotation is the identity (only `t` is applied);
                             1: rotation stored Fortran-ordered in numpy (r.transpose() of a C array,
                                elem/transform.py:86) -> y_i = fma(a_i2,v2, fma(a_i1,v1, a_i0*v0));
                             2: C-contiguous in numpy -> y_i = fma(a_i2,v2, fma(a_i0,v0, a_i1*v1))
                             (the two roundings numpy/OpenBLAS dgemv produce; DESIGN.md) */
    int32_t n_apertures;  /* len(ifc.clear_apertures), 0 -> max_aperture test */
    double cv;            /* profile.cv */
    double cc;            /* profile.cc */
    double ec;            /* profile.ec (= cc + 1.0 evaluated by the host) */
    double cR;            /* toroid sweep curvature */
    double max_aperture;  /* Interface.max_aperture */
    double coefs[RT_MAX_COEFS];
    double rt[9];         /* Tfrm[0], row-major: applied as rt . (p - t) on the way to the NEXT interface */
    double t[3];          /* Tfrm[1] */
    rt_aperture_desc apertures[RT_MAX_APERTURES];
    /* phase element (hasattr(ifc, 'phase_element'), raytrace.py:205-210) */
    int32_t phase_kind;   /* rt_phase */
    int32_t phase_flags;  /* HOE: bit 0 ref_virtual, bit 1 obj_virtual */
    double phase_ref_wl;  /* HOE / radial DOE: ref_wl (nm); grating: _grating_spacing_nm */
    double phase_ref_pt[3];   /* HOE: ref_pt; grating: grating_normal */
    double phase_obj_pt[3];   /* HOE: obj_pt */
    double phase_order;   /* grating / radial DOE: order */
    int32_t n_phase_coefs;    /* radial DOE: len(coefficients) */
    int32_t phase_pad;
    double phase_coefs[RT_MAX_PHASE_COEFS];   /* radial DOE: r**2, r**4, ... coefficients */
} rt_surface_desc;

/* keyword arguments of trace_raw(), raytrace.py:83-121 */
typedef struct rt_opts {
    double eps;                  /* eps=1e-12 */
    double pt_inside_fuzz;       /* pt_inside_fuzz; <0 means None -> the 1e-5 default of point_inside() */
    int32_t check_apertures;     /* check_apertures=False */
    int32_t intersect_obj;       /* intersect_obj=True */
    int32_t filter_out_phantoms; /* filter_out_phantoms=False */
    int32_t first_surf;          /* first_surf (trace() default 1, trace_raw() default 0) */
    int32_t last_surf;           /* last_surf; <0 means None */
    int32_t wvl_idx;             /* row of n_by_wvl used when the per-ray wvl_idx pointer is NULL */
} rt_opts;

/* Result buffers of a bundle / grid trace; every pointer is DEVICE and
 * optional (NULL = not wanted).  Arrays hold one element per ray. */
typedef struct rt_out {
    /* last ray segment, i.e. ray[-1] of the (possibly partial) RayPkg */
    double *px, *py, *pz;   /* RaySeg.p    */
    double *dx, *dy, *dz;   /* RaySeg.d    */
    double *nx, *ny, *nz;   /* RaySeg.nrml */
    double *dst;            /* RaySeg.dst (0 unless the ray missed: then pp_dst, raytrace.py:232) */
    double *op;             /* op_delta on success, opl so far on failure (raytrace.py:236,261) */
    int32_t *status;        /* rt_status */
    int32_t *fail_surf;     /* TraceError.surf; -1 on success */
    int32_t *n_seg;         /* number of valid segments in `full` */
    /* whole ray, structure of arrays: full[(seg*RT_SEG_DOUBLES + c)*full_stride + ray],
     * c = 0..2 p, 3..5 d, 6 dst, 7..9 nrml; seg < n_ifc.  Segments >= n_seg are not written. */
    double *full;
    int64_t full_stride;    /* >= n_rays */
    /* transverse ray aberration at the image (grid traces only):
     * p + (foc/d_z) d - ref_img, analyses.py:561-580 */
    double *abr_x, *abr_y;
    /* optical path difference w.r.t. the chief ray on the reference sphere (grid traces
     * with rt_grid_spec.wave): wave_abr_full_calc_finite_pup, raytr/waveabr.py:255-305.
     * System units (mm); NaN for rays that do not reach the image. */
    double *opd;
    /* RT_OUT_* bits */
    int32_t flags;
    int32_t pad_;
} rt_out;

/* rt_out.flags */
#define RT_OUT_ABR_NAN_STATUS 1  /* grid traces: rays that do not reach the image get abr_x = quiet NaN
                                    whose low mantissa bits hold rt_status and abr_y = quiet NaN whose low
                                    bits hold fail_surf, so a consumer that only reads abr_x/abr_y (16 B/ray
                                    instead of 20) still gets both: status = isnan(x) ? bits(x) & 0xFFFF : 0 */
#define RT_NAN_PAYLOAD_BASE 0x7FF8000000000000ull

typedef struct rt_table rt_table;
typedef struct rt_grid rt_grid;
typedef struct rt_variants rt_variants;

/* ---- table: the compiled form of SequentialModel.path() for all wavelengths */

/* surfs: HOST [n_ifc]; n_by_wvl: HOST [n_wvl][n_ifc] refractive index following
 * each interface (path tuple Indx, unsigned; seq/sequential.py:259-274). */
int rt_table_create(const rt_surface_desc *surfs, int32_t n_ifc,
                    const double *n_by_wvl, int32_t n_wvl,
                    int32_t device, rt_table **out);
int rt_table_destroy(rt_table *table);
int rt_table_dims(const rt_table *table, int32_t *n_ifc, int32_t *n_wvl, int32_t *device);
/* wavelengths (nm) of the rows of n_by_wvl: needed only by phase elements (mu = wvl/ref_wl,
 * doe.py:384).  wvl_nm: HOST [n_wvl]. */
int rt_table_set_wavelengths(rt_table *table, const double *wvl_nm);

/* ---- bundle trace: replaces a Python loop over rt.trace()/trace_raw()
 * (raytrace.py:51-264; callers raytr/trace.py:250,310; analyses.py:458-510).
 * px..dz: DEVICE [n_rays] start point / direction cosines in the object
 * interface's coordinates; wvl_idx: DEVICE [n_rays] or NULL. */
int rt_trace_bundle(const rt_table *table, int64_t n_rays,
                    const double *px, const double *py, const double *pz,
                    const double *dx, const double *dy, const double *dz,
                    const int32_t *wvl_idx, const rt_opts *opts,
                    const rt_out *out, void *stream);

/* ---- grid trace: replaces trace.trace_grid / analyses.trace_ray_grid /
 * trace_ray_list / trace_ray_fan (raytr/trace.py:537-605, analyses.py:212-230,
 * 437-455,666-696) including the start-ray generation of
 * OpticalSpecs.ray_start_from_osp 'epd' branch (raytr/opticalspec.py:289-366),
 * Field.apply_vignetting (opticalspec.py:1339-1353) and the refocus /
 * transverse-aberration step (analyses.py:561-580). */

typedef struct rt_field_desc {
    double pt0[3];   /* ray start point on the object interface (opticalspec.py:361) */
    double aim[2];   /* fld.aim_info: aim point on the paraxial entrance pupil (opticalspec.py:357) */
    double vlx, vux, vly, vuy; /* Field vignetting factors */
    double rot[9];   /* RT_PUPIL_WIDE: rot_v1_into_v2(d0, [0,0,1]), row-major (C-contiguous in numpy) */
    double obj2enp;  /* RT_PUPIL_WIDE: -(fod.obj_dist + z_enp) */
} rt_field_desc;

typedef struct rt_grid_spec {
    int32_t n_fields, n_wvls;  /* tiles = n_fields * n_wvls, ordered field-major */
    int32_t nx, ny;            /* pupil samples per tile: x outer, y inner (trace.py:572-604) */
    const rt_field_desc *fields; /* HOST [n_fields] */
    const int32_t *wvl_idx;    /* HOST [n_wvls] rows of the table's n_by_wvl */
    const double *pupil_x;     /* HOST [n_fields][nx] relative pupil x before vignetting */
    const double *pupil_y;     /* HOST [n_fields][ny] */
    const double *ref_img;     /* HOST [n_fields][n_wvls][2] reference image point (ref_sphere[0]) or NULL (=0;
                                  rt_grid_chief_ref() can fill it on the device afterwards) */
    const double *wave;        /* HOST [n_fields][n_wvls][RT_WAVE_DOUBLES] or NULL.  Chief ray and reference
                                  sphere of each tile, what wave_abr_full_calc_finite_pup reads
                                  (raytr/waveabr.py:255-305, 24-76, 79-113):
                                  0-2 cr.ray[1].p   3-5 cr.ray[0].d   6-8 cr.ray[-2].p  9-11 cr.ray[-2].d
                                  12 cr_op  13-15 cr_exp_pt  16 cr_exp_dist  17-19 ref_dir
                                  20 ref_sphere_radius  21 sign_soln (+1/-1)  22 |n_obj|  23 |n_img|
                                  A record with [21] == 0 selects wave_abr_full_calc_inf_ref (waveabr.py:356-420,
                                  exit pupil beyond 1e8; image gap without tilt/decenter):
                                  0-2 cr.ray[1].p  3-5 cr.ray[0].d  6-8 cr.ray[-1].p  9-11 cr.ray[-1].d
                                  12 V_BE = cr_op + op_cr_b4  13-15 image_pt  17-19 d_cr_b4  20 t_z of the
                                  image gap  22 |n_obj|  23 |n_img| */
    int32_t apply_vignetting;  /* trace_base(apply_vignetting=...) trace.py:289-292 */
    int32_t flip_z_dir;        /* seq_model.z_dir[0]: dir0 is negated when dir0.z*z_dir < 0 (trace.py:305-308) */
    int32_t paired;            /* 0: product grid pupil_x[i] x pupil_y[j]; 1: ray list -- ny must be 1 and
                                  pupil_y is [n_fields][nx]: ray i uses (pupil_x[i], pupil_y[i])
                                  (trace_ray_list / trace_ray_fan, analyses.py:212-230,437-455) */
    int32_t pupil_kind;        /* rt_pupil_kind: which branch of ray_start_from_osp generates the rays */
    double eprad;              /* RT_PUPIL_EPD: pupil_value/2 (opticalspec.py:340); RT_PUPIL_NA: sin_ang = NA/n
                                  (:373-377); RT_PUPIL_FNO: slope = -1/(2 f/#) (:378-380) */
    double z_pupil;            /* fod.obj_dist + z_enp: z of the aim plane (opticalspec.py:360) */
    double foc;                /* focus shift used for abr_x/abr_y (analyses.py:572) */
} rt_grid_spec;

int rt_grid_create(const rt_grid_spec *spec, int32_t device, rt_grid **out);
int rt_grid_destroy(rt_grid *grid);
/* Replace the contents of `grid` by another description of the SAME shape (n_fields, n_wvls,
 * nx, ny, paired, wave present or not): one asynchronous host->device copy on `stream` from
 * the handle's pinned staging block, no allocation.  `spec` is read before the call returns;
 * launches on `stream` issued afterwards see the new description (launches on other streams
 * must be ordered after it by the caller). */
int rt_grid_update(rt_grid *grid, const rt_grid_spec *spec, void *stream);
/* total rays and the chunk geometry used for sharding / summaries */
int rt_grid_dims(const rt_grid *grid, int64_t *n_rays, int64_t *n_chunks, int32_t *chunk_rays);

/* Trace chunks [chunk_begin, chunk_end) of the grid.  A chunk is `chunk_rays`
 * consecutive rays of one (field, wvl) tile (the last chunk of a tile may be
 * short); flattened ray index = ((f*n_wvls + w)*nx + i)*ny + j.  Per-ray
 * outputs are indexed by (flattened ray index - first ray of chunk_begin).
 * summary: DEVICE [n_fields*n_wvls][RT_SUMMARY_DOUBLES] or NULL; receives this
 * call's partial per-tile sums (deterministic order):
 *   0 n_ok 1 n_missed 2 n_tir 3 n_blocked 4 n_other
 *   5 sum_x 6 sum_y 7 sum_xx 8 sum_yy 9 sum_xy (of abr_x/abr_y over ok rays)
 *   10 min_x 11 max_x 12 min_y 13 max_y 14 sum_op 15 reserved
 * scratch: DEVICE, rt_grid_scratch_bytes() bytes, needed when summary != NULL. */
int64_t rt_grid_scratch_bytes(const rt_grid *grid, int64_t chunk_begin, int64_t chunk_end);
int rt_trace_grid(const rt_table *table, const rt_grid *grid,
                  int64_t chunk_begin, int64_t chunk_end,
                  const rt_opts *opts, const rt_out *out,
                  double *summary, void *scratch, void *stream);

/* Grid trace with the results delivered to HOST memory -- the data path of the grid analyses
 * (spot diagrams: seq/sequential.py:1058-1085 evaluated for every field) in one call.  Chunks
 * [chunk_begin, chunk_end) are traced in n_pieces launches alternating between two streams
 * owned by the grid handle; each piece's transverse aberrations (RT_OUT_ABR_NAN_STATUS coding)
 * are copied device -> host right behind its trace, so copies and traces overlap.
 * d_abr_x/y: DEVICE staging [rays of the range]; h_abr_x/y: HOST, page-locked, same length;
 * summary: DEVICE [n_tiles][RT_SUMMARY_DOUBLES] or NULL; scratch: DEVICE,
 * rt_trace_grid_to_host_scratch_bytes(grid, n_pieces) bytes.  Work already queued on `stream`
 * (rt_grid_update, rt_grid_chief_ref) is waited for; when the call returns, `stream` waits for
 * all pieces: synchronising `stream` makes h_abr_* and summary valid. */
int64_t rt_trace_grid_to_host_scratch_bytes(const rt_grid *grid, int32_t n_pieces);
int rt_trace_grid_to_host(const rt_table *table, rt_grid *grid, int64_t chunk_begin, int64_t chunk_end,
                          const rt_opts *opts, double *d_abr_x, double *d_abr_y,
                          double *h_abr_x, double *h_abr_y, double *summary, void *scratch,
                          int32_t n_pieces, void *stream);

/* Reference image points without a host round trip: trace the (0, 0) pupil ray of every
 * field at row `wvl_idx` of the table (no vignetting, apertures not checked) and store its
 * image intercept (x, y) as the reference image point of every (field, wvl) tile of `grid` --
 * ref_sphere[0] of calculate_reference_sphere for image_pt_2d=None (raytr/waveabr.py:24-76,
 * raytr/trace.py:627-687 without the re-aiming).  One small launch on `stream`; later
 * rt_trace_grid calls on the same stream see the new points.  ref_out: DEVICE [n_fields][2]
 * or NULL, receives a copy. */
int rt_grid_chief_ref(const rt_table *table, rt_grid *grid, int32_t wvl_idx,
                      double *ref_out, void *stream);

/* ---- through focus (ABI 5): the spot sums of one grid trace at n_foc image planes.
 * Plane k is evaluated with the epilogue of rt_trace_grid at foc = foc[k]: each ray's
 * p + (foc[k]/d_z) d - ref_img[k][field].  Its summary row equals, column for column, the summary
 * rt_trace_grid returns over the same chunk range for a grid with foc = foc[k] and the same
 * reference points (both with the default dynamic schedule).  The through-focus trace always
 * draws work items from a counter, so B200RT_STATIC does not apply to it. */
/* chief-ray image intercepts defocused to every plane: ref_out[k][f] = p + (foc[k]/d_z) d of the
 * ray rt_grid_chief_ref traces (calculate_reference_sphere's image_pt, raytr/waveabr.py:24-76).
 * foc: HOST [n_foc]; ref_out: DEVICE [n_foc][n_fields][2].  The grid's own reference points are
 * not changed.  One launch on `stream`. */
int rt_grid_chief_ref_focus(const rt_table *table, const rt_grid *grid, int32_t wvl_idx,
                            const double *foc, int32_t n_foc, double *ref_out, void *stream);
/* DEVICE scratch bytes of rt_trace_grid_focus (n_foc times rt_grid_scratch_bytes); 0 for bad arguments */
int64_t rt_grid_focus_scratch_bytes(const rt_grid *grid, int32_t n_foc,
                                    int64_t chunk_begin, int64_t chunk_end);
/* foc: HOST [n_foc], finite, 1 <= n_foc <= RT_MAX_FOCUS; ref_img: DEVICE [n_foc][n_fields][2] or
 * NULL (= 0); summary: DEVICE [n_foc][n_tiles][RT_SUMMARY_DOUBLES] (required).  out: per-ray
 * results as rt_trace_grid (p, d, op, status, fail_surf, n_seg); abr_x/abr_y/opd/full/nx/ny/nz/dst
 * must be NULL.  RT_ERR_INVALID before any device work for bad arguments.  Two kernel launches
 * whatever n_foc is. */
int rt_trace_grid_focus(const rt_table *table, const rt_grid *grid,
                        int64_t chunk_begin, int64_t chunk_end, const rt_opts *opts,
                        const double *foc, int32_t n_foc, const double *ref_img,
                        const rt_out *out, double *summary, void *scratch, void *stream);

/* Combine n_parts partial summaries (chunk ranges of one grid, or the ranks' rows of an
 * all-gather): parts DEVICE [n_parts][n_tiles][RT_SUMMARY_DOUBLES] -> out DEVICE
 * [n_tiles][RT_SUMMARY_DOUBLES]; sums add in part order, the min / max columns take
 * min / max.  One launch on `stream`. */
int rt_combine_summaries(const double *parts, int32_t n_parts, int64_t n_tiles,
                         double *out, void *stream);

/* ---- wavefront error (ABI 6): the sums behind RMS / P-V wavefront error and its least-squares
 * fits on {1, x, y} and {1, x, y, r^2}, per tile, from one grid trace with the OPD epilogue.
 * W = the ray's opd (system units) as rt_trace_grid writes it; (x, y) = the ray's relative pupil
 * coordinates pupil_x[i], pupil_y[j] of its rt_grid_spec, after Field.apply_vignetting when the grid
 * applies it; r2 = x*x + y*y.  summary: DEVICE [n_tiles][RT_WFE_DOUBLES]:
 *   0 n_ok 1 n_missed 2 n_tir 3 n_blocked 4 n_other   (as the spot summary)
 *   5 min W 6 max W                                    (fmin / fmax: NaN skipped; +-inf without rays)
 *   7 sum W 8 sum W*W 9 sum x*W 10 sum y*W 11 sum r2*W
 *   12 sum x 13 sum y 14 sum x*x 15 sum x*y 16 sum y*y 17 sum x*r2 18 sum y*r2 19 sum r2*r2
 *   20-23 reserved (0)
 * Only status-0 rays enter columns 5-19; a status-0 ray with a NaN opd makes its tile's sums NaN.
 * The sums are added in the fixed order of DESIGN.md section 4 (32-ray work items drawn from a
 * counter, each summed by one shuffle tree and stored on its own): bit-reproducible.  B200RT_STATIC
 * does not apply. */
/* DEVICE scratch bytes of rt_trace_grid_wfe over [chunk_begin, chunk_end); 0 for bad arguments */
int64_t rt_grid_wfe_scratch_bytes(const rt_grid *grid, int64_t chunk_begin, int64_t chunk_end);
/* The grid must carry rt_grid_spec.wave.  out: per-ray results as rt_trace_grid (opd included,
 * all optional); out.full must be NULL.  summary and scratch are required.  RT_ERR_INVALID before
 * any device work for bad arguments.  Two kernel launches (one for an empty chunk range). */
int rt_trace_grid_wfe(const rt_table *table, const rt_grid *grid,
                      int64_t chunk_begin, int64_t chunk_end, const rt_opts *opts,
                      const rt_out *out, double *summary, void *scratch, void *stream);
/* rt_combine_summaries for wavefront-error records: parts DEVICE [n_parts][n_tiles][RT_WFE_DOUBLES]
 * -> out DEVICE [n_tiles][RT_WFE_DOUBLES]; sums and counts add in part order, column 5 takes fmin,
 * column 6 fmax.  One launch on `stream`. */
int rt_combine_wfe(const double *parts, int32_t n_parts, int64_t n_tiles, double *out, void *stream);

/* ---- Zernike moments (ABI 6, additive): the packed Gram matrix of a = [W, Z_1 ... Z_J] per tile,
 * the normal equations of a least-squares fit of the OPD on the first J Fringe Zernike terms
 * (csrc/rt_zernike.cuh).  status / opd: DEVICE per-ray arrays indexed as rt_trace_grid's outputs
 * over the same chunk range (rays_in_chunks(chunk_begin, chunk_end) entries; opd in system units).
 * (x, y) = the ray's relative pupil coordinates pupil_x[i], pupil_y[j] of its rt_grid_spec.  A ray
 * is used when its status is 0 and x*x + y*y <= 1.  summary: DEVICE [n_tiles][RT_ZERN_DOUBLES]:
 *   0-4 status-class counts of every ray (as the wavefront-error record)   5 n_used
 *   6 min W 7 max W over the used rays (fmin / fmax: NaN skipped; +-inf without used rays)   8 0
 *   9 + j*(j+1)/2 + i, i <= j <= J: sum of a_i*a_j over the used rays (a_0 = W, a_k = Z_k)
 *   later columns 0
 * Sum order (DESIGN.md section 4): products rounded once; per chunk of 256 rays of one tile every
 * entry is added in ray order from +0.0; the tile's chunk sums inside the range are added in chunk
 * order from +0.0.  Bit-reproducible, independent of the launch shape. */
/* DEVICE scratch bytes of rt_grid_zernike over [chunk_begin, chunk_end) with n_terms terms;
 * 0 for bad arguments or an empty range */
int64_t rt_grid_zernike_scratch_bytes(const rt_grid *grid, int64_t chunk_begin, int64_t chunk_end,
                                      int32_t n_terms);
/* The grid must be a product grid (paired = 0) without apply_vignetting; 1 <= n_terms <=
 * RT_ZERN_MAX_TERMS.  status, opd and scratch may be NULL only for an empty range; summary is
 * required.  RT_ERR_INVALID before any device work for bad arguments.  Two kernel launches (the
 * moments, their reduction), one for an empty chunk range. */
int rt_grid_zernike(const rt_grid *grid, int64_t chunk_begin, int64_t chunk_end, int32_t n_terms,
                    const int32_t *status, const double *opd, double *summary, void *scratch, void *stream);
/* rt_combine_summaries for Zernike moments records: parts DEVICE [n_parts][n_tiles][RT_ZERN_DOUBLES]
 * -> out DEVICE [n_tiles][RT_ZERN_DOUBLES]; sums and counts add in part order, column 6 takes fmin,
 * column 7 fmax.  One launch on `stream`. */
int rt_combine_zernike(const double *parts, int32_t n_parts, int64_t n_tiles, double *out, void *stream);

/* ---- chief-ray aiming (ABI 6, additive): the aim point of every field of a grid, found on the
 * device by the damped 2-D Newton iteration of vigcalc.aim_chief_ray / aim_all_fields_batched
 * (csrc/rt_aim.cuh; DESIGN.md section 4).  Per field, starting from aim (0, 0): the (0, 0) pupil ray
 * of the 'epd' start-ray rule (rt_field_desc pt0, the grid's eprad, z_pupil and flip_z_dir) with the
 * trial aim in place of rt_field_desc.aim is traced at row wvl_idx of the table with the general
 * loop (first_surf 1, apertures not checked, intersect_obj on) up to interface `stop`; the iteration
 * drives its (x, y) intercept there to 0.  h: the forward-difference step, 1e-4*max(1, enp_radius)
 * in aim_chief_ray; tol: max|intercept| below which a field has converged; max_iter: Newton steps.
 * aim_out: DEVICE [n_fields][2] receives the aim points (x = 0 is NOT forced for fields with
 * x = 0: aim_chief_ray applies that rule after its iteration, the caller does it after the copy);
 * term_out: DEVICE [n_fields] or NULL receives each field's rt_aim_term.  The grid's field records
 * are read, not changed.  One launch on `stream`, one thread per field.
 * RT_ERR_UNSUPPORTED before any device work when the grid's pupil_kind is not RT_PUPIL_EPD
 * (wide-angle fields and angular pupils stay with the host functions); RT_ERR_INVALID before any
 * device work when stop is not in 1 ... n_ifc - 2, wvl_idx is out of range, h or tol is not finite
 * and positive, max_iter < 0 or aim_out is NULL. */
enum rt_aim_term {
    RT_AIM_CONVERGED = 0,    /* max|intercept| < tol */
    RT_AIM_FIRST_FAILED = 1, /* the ray aimed at (0, 0) does not reach the stop: aim (0, 0) */
    RT_AIM_DIFF_FAILED = 2,  /* a forward-difference ray does not reach the stop */
    RT_AIM_SINGULAR = 3,     /* zero pivot in the 2x2 solve, or a step that is not finite */
    RT_AIM_NO_STEP = 4,      /* none of the 20 backtracking trials reduced max|intercept| (the usual
                                end for objects at infinity: the noise floor of the intercept) */
    RT_AIM_MAX_ITER = 5      /* max_iter Newton steps taken */
};
int rt_grid_aim_chief(const rt_table *table, const rt_grid *grid, int32_t stop, int32_t wvl_idx,
                      double h, double tol, int32_t max_iter, double *aim_out, int32_t *term_out,
                      void *stream);

/* ---- diffraction MTF (ABI 6, additive): the pupil function of every tile of a grid trace and its
 * autocorrelation along the two pupil axes (csrc/rt_mtf.cuh; DESIGN.md section 4).  The grid must be
 * a product grid (paired = 0) without apply_vignetting with nx = ny = n <= RT_MTF_MAX_RAYS; the whole
 * grid is processed (the autocorrelation needs every ray of a tile).  status / opd: DEVICE per-ray
 * arrays of an rt_trace_grid over all chunks (opd in system units); ray (i, j) of tile t is entry
 * t*n*n + i*n + j, at relative pupil coordinates (x, y) = (pupil_x[i], pupil_y[j]) of its field.  A
 * ray is used when its status is 0 and x*x + y*y <= 1.  RT_ERR_INVALID before any device work for a
 * bad grid or a NULL pointer.  One launch each on `stream`. */
/* wvl_sys: DEVICE [n_tiles] wavelength of each tile in system units.  pupil, pupil_t: DEVICE
 * [n_tiles][n][n] complex128 (re, im): pupil[t][i][j] = P = exp(2 pi i opd/wvl_sys) of a used ray
 * (sincospi(2.0*w), w = opd/wvl_sys rounded once), +0.0 otherwise; pupil_t[t][j][i] = the same value. */
int rt_grid_pupil_function(const rt_grid *grid, const int32_t *status, const double *opd, const double *wvl_sys,
                           double *pupil, double *pupil_t, void *stream);
/* pupil, pupil_t: rt_grid_pupil_function's outputs; status: the trace's.  acf_x, acf_y: DEVICE
 * [n_tiles][n] complex128: acf_x[t][k] = Cx(k) = sum over i < n-k and all j of P[i+k][j]*conj(P[i][j]),
 * acf_y the same along j.  record: DEVICE [n_tiles][RT_MTF_DOUBLES]:
 *   0-4 status-class counts of every ray (as the wavefront-error record)   5 n_used   6, 7 Re, Im S
 * with S = sum of P.  Sum order: products a*conj(b) as re = ar*br + ai*bi, im = ai*br - ar*bi, every
 * product rounded once; each line (fixed j for Cx and S, fixed i for Cy) added in increasing index
 * along the other axis from +0.0; the line sums added in line order from +0.0.  Bit-reproducible,
 * independent of the launch shape. */
int rt_grid_mtf(const rt_grid *grid, const int32_t *status, const double *pupil, const double *pupil_t,
                double *acf_x, double *acf_y, double *record, void *stream);
/* rt_grid_mtf at listed shifts only.  shifts: DEVICE [n_shifts], each in [0, n-1], any order,
 * duplicates allowed (an entry outside that range gives NaN).  acf_x, acf_y: DEVICE
 * [n_tiles][n_shifts] complex128; entry m is bit for bit rt_grid_mtf's entry shifts[m].  record: as
 * rt_grid_mtf.  n_shifts = 0 computes the record alone (shifts, acf_x and acf_y may be NULL).  One
 * launch on `stream`; RT_ERR_INVALID before any device work as rt_grid_mtf, and for n_shifts < 0. */
int rt_grid_mtf_shifts(const rt_grid *grid, const int32_t *status, const double *pupil, const double *pupil_t,
                       const int32_t *shifts, int32_t n_shifts, double *acf_x, double *acf_y,
                       double *record, void *stream);

/* ---- OPD at many reference spheres (ABI 6, additive): one trace of chunks [chunk_begin, chunk_end)
 * of a grid with rt_grid_spec.wave, and the OPD of every ray against n_foc reference spheres per tile
 * (csrc/rt_refocus.cuh; DESIGN.md section 4): the reference's wave_abr_pre_calc once per ray,
 * wave_abr_calc once per sphere.  The focus-independent columns of each tile's wave record are used
 * (finite: 0-16, 22, 23; infinite reference, [21] == 0: 0-12, 17-20, 22, 23).
 * spheres: DEVICE [n_foc][n_tiles][RT_SPHERE_DOUBLES], what calculate_reference_sphere changes with
 *   the focus: 0-2 ref_dir  3 ref_sphere_radius  4 sign_soln (+1/-1; 0 on infinite-reference tiles)
 *   5-7 image_pt.  A plane whose record equals the tile's own (wave 17-21) gives rt_trace_grid's opd
 *   bit for bit on finite tiles; infinite-reference tiles round as the reference's focus_wavefront.
 * 1 <= n_foc <= RT_MAX_FOCUS.  opd_planes: DEVICE [n_foc][n] with n the rays of the range: entry
 *   k*n + r is plane k's OPD (system units) of ray r of the range, indexed as rt_trace_grid's
 *   outputs; NaN on every plane for rays with status != 0.
 * out: per-ray results of kind 0 (p, d, op, status, fail_surf, n_seg); opd, abr_x, abr_y and full
 *   must be NULL.  opd_planes may be NULL for an empty range.  RT_ERR_INVALID for bad arguments and RT_ERR_UNSUPPORTED where rt_trace_grid's opd
 *   is unsupported, both before any device work.  One launch on `stream` (none for an empty range). */
int rt_trace_grid_opd_focus(const rt_table *table, const rt_grid *grid,
                            int64_t chunk_begin, int64_t chunk_end, const rt_opts *opts,
                            const double *spheres, int32_t n_foc,
                            const rt_out *out, double *opd_planes, void *stream);

/* ---- tolerance analysis: many perturbed prescriptions of one shape over one grid
 * rt_variants_create: n_var surface tables in one device allocation and one copy.
 *   surfs: HOST [n_var][n_ifc]; n_by_wvl: HOST [n_var][n_wvl][n_ifc]; wvl_nm: HOST [n_wvl] in nm, or
 *   NULL (phase elements then see NaN).  The handle is immutable and has its own work counters. */
int rt_variants_create(const rt_surface_desc *surfs, int32_t n_ifc, const double *n_by_wvl, int32_t n_wvl,
                       int32_t n_var, const double *wvl_nm, int32_t device, rt_variants **out);
int rt_variants_destroy(rt_variants *variants);
/* bytes of scratch rt_trace_grid_variants needs for n_var variants (proportional to the rays) */
int64_t rt_grid_variants_scratch_bytes(const rt_grid *grid, int32_t n_var);
/* The whole grid traced once per variant of [var_begin, var_end) in one persistent launch (the general
 * kernel, the table read from global memory), then one reduction.  The start rays, the reference image
 * points and foc are the grid's, shared by every variant; no per-ray data is written.
 * record: DEVICE [var_end - var_begin][n_tiles][RT_TOL_DOUBLES]:
 *   0-15  rt_trace_grid's summary layout (counts, sum x, y, xx, yy, xy, min / max x, y, sum op, 0);
 *         equal to rt_trace_grid's summary of a table of that variant alone (dynamic schedule)
 *   16-21 sum ux, uy, ux*ux, uy*uy, ax*ux, ay*uy over the status-0 rays: ux = dx/dz, uy = dy/dz of the
 *         last segment (one IEEE division each), (ax, ay) the transverse aberration
 *   22-23 zero
 * Sum order (DESIGN.md section 4): summands rounded once, the work-item halving tree, reduce_tile
 * over a tile's work items in item order.  RT_ERR_INVALID, before any device work, for a bad variant
 * range, NULL pointers, variants and grid on different devices, opts.wvl_idx or a grid wvl_idx out of
 * range.  Two launches on `stream` (none for an empty range). */
int rt_trace_grid_variants(const rt_variants *variants, const rt_grid *grid, int32_t var_begin, int32_t var_end,
                           const rt_opts *opts, double *record, void *scratch, void *stream);

/* ---- misc */
const char *rt_last_error(void);
int rt_abi_version(void);
/* rays per chunk (= threads per CTA of this build): the unit of rt_trace_grid's chunk ranges */
int32_t rt_chunk_rays(void);
/* number of kernel launches issued by this library in this process (bench.py's gpu_launches) */
int64_t rt_launch_count(void);
/* fp64 vector-pipe peak of `device` in TFLOP/s, measured with a chain of
 * independent DFMAs (the roofline denominator of the register-resident trace) */
int rt_measure_fp64_peak(int32_t device, double *tflops);
/* cycles between two dependent fp64 FMAs of one warp (dependent-issue latency of the fp64 pipe) */
int rt_measure_fp64_latency(int32_t device, double *cycles_per_dependent_dfma);
/* self-test of the shared-reciprocal division of the specialised kernels against
 * the IEEE division (n_blocks x 256 threads x n_per_thread operand sets);
 * *mismatches must come back 0 */
int rt_selftest_division(int32_t device, int32_t n_blocks, int64_t n_per_thread, uint64_t seed,
                         uint64_t *mismatches);

#ifdef __cplusplus
}
#endif
#endif /* B200RT_H */
