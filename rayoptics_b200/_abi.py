"""ctypes mirror of include/b200rt.h and the loader of libb200rt.so.

There is deliberately no fallback: if the CUDA shared object is missing or does
not export the ABI, importing the engine raises (the product path never routes
through a CPU implementation).
"""
from __future__ import annotations

import ctypes as C
import os

RT_ABI_VERSION = 6
RT_MAX_COEFS = 20
RT_MAX_PHASE_COEFS = 10
RT_MAX_APERTURES = 4
RT_SEG_DOUBLES = 10
RT_SUMMARY_DOUBLES = 16
RT_WAVE_DOUBLES = 24
RT_MAX_FOCUS = 64
RT_WFE_DOUBLES = 24
RT_ZERN_DOUBLES = 752
RT_ZERN_MAX_TERMS = 37
RT_MTF_MAX_RAYS = 1024
RT_MTF_DOUBLES = 8
RT_SPHERE_DOUBLES = 8
RT_TOL_DOUBLES = 24

# enum rt_profile
PROFILE_IDS = {'Spherical': 0, 'Conic': 1, 'EvenPolynomial': 2,
               'RadialPolynomial': 3, 'YToroid': 4, 'XToroid': 5, 'ThinLens': 6}
PHASE_IDS = {'HolographicElement': 1, 'DiffractionGrating': 2, 'DiffractiveElement': 3}
# enum rt_pupil_kind
PUPIL_EPD, PUPIL_NA, PUPIL_FNO, PUPIL_WIDE = 0, 1, 2, 3
# enum rt_mode
MODE_IDS = {'transmit': 0, 'reflect': 1, 'dummy': 2, 'phantom': 3}
# enum rt_status
RAY_OK, RAY_MISSED, RAY_TIR, RAY_BLOCKED, RAY_EVANESCENT, RAY_NUMERIC = range(6)
# enum rt_aim_term
AIM_CONVERGED, AIM_FIRST_FAILED, AIM_DIFF_FAILED, AIM_SINGULAR, AIM_NO_STEP, AIM_MAX_ITER = range(6)
# enum rt_aperture_type
APERTURE_IDS = {'Circular': 1, 'Rectangular': 2, 'Elliptical': 3}

c_double_p = C.POINTER(C.c_double)
c_int32_p = C.POINTER(C.c_int32)


class rt_aperture_desc(C.Structure):
    _fields_ = [('type', C.c_int32), ('is_obscuration', C.c_int32),
                ('a', C.c_double), ('b', C.c_double),
                ('x_offset', C.c_double), ('y_offset', C.c_double)]


class rt_surface_desc(C.Structure):
    _fields_ = [('profile', C.c_int32), ('mode', C.c_int32), ('z_dir', C.c_int32),
                ('n_coefs', C.c_int32), ('has_tfrm', C.c_int32), ('n_apertures', C.c_int32),
                ('cv', C.c_double), ('cc', C.c_double), ('ec', C.c_double), ('cR', C.c_double),
                ('max_aperture', C.c_double),
                ('coefs', C.c_double*RT_MAX_COEFS),
                ('rt', C.c_double*9), ('t', C.c_double*3),
                ('apertures', rt_aperture_desc*RT_MAX_APERTURES),
                ('phase_kind', C.c_int32), ('phase_flags', C.c_int32),
                ('phase_ref_wl', C.c_double),
                ('phase_ref_pt', C.c_double*3), ('phase_obj_pt', C.c_double*3),
                ('phase_order', C.c_double), ('n_phase_coefs', C.c_int32), ('phase_pad', C.c_int32),
                ('phase_coefs', C.c_double*RT_MAX_PHASE_COEFS)]


class rt_opts(C.Structure):
    _fields_ = [('eps', C.c_double), ('pt_inside_fuzz', C.c_double),
                ('check_apertures', C.c_int32), ('intersect_obj', C.c_int32),
                ('filter_out_phantoms', C.c_int32), ('first_surf', C.c_int32),
                ('last_surf', C.c_int32), ('wvl_idx', C.c_int32)]


class rt_out(C.Structure):
    _fields_ = [('px', C.c_void_p), ('py', C.c_void_p), ('pz', C.c_void_p),
                ('dx', C.c_void_p), ('dy', C.c_void_p), ('dz', C.c_void_p),
                ('nx', C.c_void_p), ('ny', C.c_void_p), ('nz', C.c_void_p),
                ('dst', C.c_void_p), ('op', C.c_void_p),
                ('status', C.c_void_p), ('fail_surf', C.c_void_p), ('n_seg', C.c_void_p),
                ('full', C.c_void_p), ('full_stride', C.c_int64),
                ('abr_x', C.c_void_p), ('abr_y', C.c_void_p), ('opd', C.c_void_p),
                ('flags', C.c_int32), ('pad_', C.c_int32)]


RT_OUT_ABR_NAN_STATUS = 1
RT_NAN_PAYLOAD_BASE = 0x7FF8000000000000


class rt_field_desc(C.Structure):
    _fields_ = [('pt0', C.c_double*3), ('aim', C.c_double*2),
                ('vlx', C.c_double), ('vux', C.c_double),
                ('vly', C.c_double), ('vuy', C.c_double),
                ('rot', C.c_double*9), ('obj2enp', C.c_double)]


class rt_grid_spec(C.Structure):
    _fields_ = [('n_fields', C.c_int32), ('n_wvls', C.c_int32),
                ('nx', C.c_int32), ('ny', C.c_int32),
                ('fields', C.POINTER(rt_field_desc)),
                ('wvl_idx', c_int32_p),
                ('pupil_x', c_double_p), ('pupil_y', c_double_p),
                ('ref_img', c_double_p), ('wave', c_double_p),
                ('apply_vignetting', C.c_int32), ('flip_z_dir', C.c_int32),
                ('paired', C.c_int32), ('pupil_kind', C.c_int32),
                ('eprad', C.c_double), ('z_pupil', C.c_double), ('foc', C.c_double)]


def make_opts(eps=1.0e-12, check_apertures=False, intersect_obj=True,
              filter_out_phantoms=False, first_surf=0, last_surf=None,
              pt_inside_fuzz=None, wvl_idx=0):
    """keyword arguments of trace_raw (raytrace.py:83-121) -> rt_opts"""
    return rt_opts(eps=float(eps),
                   pt_inside_fuzz=-1.0 if pt_inside_fuzz is None else float(pt_inside_fuzz),
                   check_apertures=int(bool(check_apertures)),
                   intersect_obj=int(bool(intersect_obj)),
                   filter_out_phantoms=int(bool(filter_out_phantoms)),
                   first_surf=int(first_surf),
                   last_surf=-1 if last_surf is None else int(last_surf),
                   wvl_idx=int(wvl_idx))


LIB_NAME = 'libb200rt.so'
EXPORTS = ['rt_table_create', 'rt_table_destroy', 'rt_table_dims', 'rt_table_set_wavelengths',
           'rt_trace_bundle', 'rt_grid_create', 'rt_grid_destroy', 'rt_grid_dims',
           'rt_grid_scratch_bytes', 'rt_trace_grid', 'rt_grid_chief_ref', 'rt_combine_summaries',
           'rt_grid_update', 'rt_trace_grid_to_host', 'rt_trace_grid_to_host_scratch_bytes',
           'rt_last_error', 'rt_abi_version', 'rt_chunk_rays', 'rt_launch_count', 'rt_measure_fp64_peak', 'rt_measure_fp64_latency',
           'rt_selftest_division', 'rt_grid_chief_ref_focus', 'rt_grid_focus_scratch_bytes',
           'rt_trace_grid_focus', 'rt_grid_wfe_scratch_bytes', 'rt_trace_grid_wfe', 'rt_combine_wfe',
           'rt_grid_zernike_scratch_bytes', 'rt_grid_zernike', 'rt_combine_zernike', 'rt_grid_aim_chief',
           'rt_grid_pupil_function', 'rt_grid_mtf', 'rt_grid_mtf_shifts', 'rt_trace_grid_opd_focus',
           'rt_variants_create', 'rt_variants_destroy', 'rt_grid_variants_scratch_bytes', 'rt_trace_grid_variants']

_lib = None


def lib_path():
    # B200RT_LIB: alternative build of the same ABI (kernel tuning experiments)
    return os.environ.get('B200RT_LIB') or os.path.join(
        os.path.dirname(os.path.abspath(__file__)), 'csrc', LIB_NAME)


class EngineError(RuntimeError):
    """A C-ABI call returned a negative rt_error code."""


def load_library():
    """dlopen libb200rt.so and declare signatures.  Raises if absent."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not os.path.exists(path):
        raise ImportError(
            f'{path} not found: build it with `python -c "import __graft_entry__ as g; g.build()"` '
            f'(or `make -C rayoptics_b200/csrc`).  There is no CPU fallback.')
    lib = C.CDLL(path)
    for name in EXPORTS:
        if not hasattr(lib, name):
            raise ImportError(f'{path} does not export {name}')
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    lib.rt_table_create.argtypes = [C.POINTER(rt_surface_desc), i32, c_double_p, i32, i32,
                                    C.POINTER(vp)]
    lib.rt_table_destroy.argtypes = [vp]
    lib.rt_table_dims.argtypes = [vp, c_int32_p, c_int32_p, c_int32_p]
    lib.rt_table_set_wavelengths.argtypes = [vp, c_double_p]
    lib.rt_table_set_wavelengths.restype = i32
    lib.rt_trace_bundle.argtypes = [vp, i64, vp, vp, vp, vp, vp, vp, vp,
                                    C.POINTER(rt_opts), C.POINTER(rt_out), vp]
    lib.rt_grid_create.argtypes = [C.POINTER(rt_grid_spec), i32, C.POINTER(vp)]
    lib.rt_grid_destroy.argtypes = [vp]
    lib.rt_grid_dims.argtypes = [vp, C.POINTER(i64), C.POINTER(i64), c_int32_p]
    lib.rt_grid_scratch_bytes.argtypes = [vp, i64, i64]
    lib.rt_grid_scratch_bytes.restype = i64
    lib.rt_trace_grid.argtypes = [vp, vp, i64, i64, C.POINTER(rt_opts), C.POINTER(rt_out),
                                  vp, vp, vp]
    lib.rt_grid_update.argtypes = [vp, C.POINTER(rt_grid_spec), vp]
    lib.rt_grid_update.restype = i32
    lib.rt_trace_grid_to_host_scratch_bytes.argtypes = [vp, i32]
    lib.rt_trace_grid_to_host_scratch_bytes.restype = i64
    lib.rt_trace_grid_to_host.argtypes = [vp, vp, i64, i64, C.POINTER(rt_opts), vp, vp, vp, vp, vp, vp, i32, vp]
    lib.rt_trace_grid_to_host.restype = i32
    lib.rt_grid_chief_ref.argtypes = [vp, vp, i32, vp, vp]
    lib.rt_grid_chief_ref.restype = i32
    lib.rt_grid_chief_ref_focus.argtypes = [vp, vp, i32, c_double_p, i32, vp, vp]
    lib.rt_grid_chief_ref_focus.restype = i32
    lib.rt_grid_focus_scratch_bytes.argtypes = [vp, i32, i64, i64]
    lib.rt_grid_focus_scratch_bytes.restype = i64
    lib.rt_trace_grid_focus.argtypes = [vp, vp, i64, i64, C.POINTER(rt_opts), c_double_p, i32, vp,
                                        C.POINTER(rt_out), vp, vp, vp]
    lib.rt_trace_grid_focus.restype = i32
    lib.rt_combine_summaries.argtypes = [vp, i32, i64, vp, vp]
    lib.rt_combine_summaries.restype = i32
    lib.rt_grid_wfe_scratch_bytes.argtypes = [vp, i64, i64]
    lib.rt_grid_wfe_scratch_bytes.restype = i64
    lib.rt_trace_grid_wfe.argtypes = [vp, vp, i64, i64, C.POINTER(rt_opts), C.POINTER(rt_out), vp, vp, vp]
    lib.rt_trace_grid_wfe.restype = i32
    lib.rt_combine_wfe.argtypes = [vp, i32, i64, vp, vp]
    lib.rt_combine_wfe.restype = i32
    lib.rt_grid_zernike_scratch_bytes.argtypes = [vp, i64, i64, i32]
    lib.rt_grid_zernike_scratch_bytes.restype = i64
    lib.rt_grid_zernike.argtypes = [vp, i64, i64, i32, vp, vp, vp, vp, vp]
    lib.rt_grid_zernike.restype = i32
    lib.rt_combine_zernike.argtypes = [vp, i32, i64, vp, vp]
    lib.rt_combine_zernike.restype = i32
    lib.rt_grid_aim_chief.argtypes = [vp, vp, i32, i32, C.c_double, C.c_double, i32, vp, vp, vp]
    lib.rt_grid_aim_chief.restype = i32
    lib.rt_grid_pupil_function.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    lib.rt_grid_pupil_function.restype = i32
    lib.rt_grid_mtf.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp]
    lib.rt_grid_mtf.restype = i32
    lib.rt_grid_mtf_shifts.argtypes = [vp, vp, vp, vp, vp, i32, vp, vp, vp, vp]
    lib.rt_grid_mtf_shifts.restype = i32
    lib.rt_trace_grid_opd_focus.argtypes = [vp, vp, i64, i64, C.POINTER(rt_opts), vp, i32, C.POINTER(rt_out), vp, vp]
    lib.rt_trace_grid_opd_focus.restype = i32
    lib.rt_variants_create.argtypes = [C.POINTER(rt_surface_desc), i32, c_double_p, i32, i32, c_double_p, i32,
                                       C.POINTER(vp)]
    lib.rt_variants_create.restype = i32
    lib.rt_variants_destroy.argtypes = [vp]
    lib.rt_variants_destroy.restype = i32
    lib.rt_grid_variants_scratch_bytes.argtypes = [vp, i32]
    lib.rt_grid_variants_scratch_bytes.restype = i64
    lib.rt_trace_grid_variants.argtypes = [vp, vp, i32, i32, C.POINTER(rt_opts), vp, vp, vp]
    lib.rt_trace_grid_variants.restype = i32
    lib.rt_last_error.restype = C.c_char_p
    lib.rt_abi_version.restype = i32
    lib.rt_chunk_rays.restype = i32
    lib.rt_launch_count.restype = i64
    lib.rt_measure_fp64_peak.argtypes = [i32, c_double_p]
    lib.rt_measure_fp64_peak.restype = i32
    lib.rt_measure_fp64_latency.argtypes = [i32, c_double_p]
    lib.rt_measure_fp64_latency.restype = i32
    lib.rt_selftest_division.argtypes = [i32, i32, i64, C.c_uint64, C.POINTER(C.c_uint64)]
    lib.rt_selftest_division.restype = i32
    for name in ('rt_table_create', 'rt_table_destroy', 'rt_table_dims', 'rt_trace_bundle',
                 'rt_grid_create', 'rt_grid_destroy', 'rt_grid_dims', 'rt_trace_grid'):
        getattr(lib, name).restype = i32
    if lib.rt_abi_version() != RT_ABI_VERSION:
        raise ImportError(f'{path}: ABI version {lib.rt_abi_version()} != {RT_ABI_VERSION}')
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        msg = load_library().rt_last_error()
        raise EngineError(f'libb200rt error {rc}: {msg.decode() if msg else ""}')
