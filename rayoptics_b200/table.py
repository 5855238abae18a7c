"""Surface table: the compiled form of ``SequentialModel.path(wvl)``.

Flattens the reference's path tuples ``(Intfc, Gap, Tfrm, Indx, Zdir)``
(/root/reference/src/rayoptics/seq/sequential.py:149-202,
optical/model_constants.py:12) into ``rt_surface_desc`` records plus an
``n_by_wvl[n_wvl][n_ifc]`` index table, and owns the device-side handle created
by ``rt_table_create``.  Works on the reference's own ``Surface``/profile
objects and on the mirrors in ``model.py`` alike: dispatch is by class *name*
and attribute (the "Interface protocol" row of SURVEY.md 8(b)).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _abi
from ._abi import (rt_surface_desc, RT_MAX_COEFS, RT_MAX_APERTURES, RT_MAX_PHASE_COEFS,
                   PROFILE_IDS, MODE_IDS, APERTURE_IDS, PHASE_IDS)


class _ThinLensProfile:
    cv = 0.0


def profile_fields(profile, pname):
    """``(cv, cc, ec)`` of a profile as the table stores them"""
    if pname in ('Spherical', 'ThinLens'):
        return float(profile.cv), 0.0, 1.0
    return float(profile.cv), float(profile.cc), float(profile.ec)


def set_transform(d, tfrm):
    """``rt``, ``t`` and ``has_tfrm`` of descriptor ``d`` from a path transform ``(rt, t)`` or None"""
    if tfrm is None:
        rt, t = np.identity(3), np.zeros(3)
    else:
        rt, t = np.asarray(tfrm[0], dtype=float), np.asarray(tfrm[1], dtype=float)
    if np.array_equal(rt, np.identity(3)):
        d.has_tfrm = 0
    elif rt.flags['C_CONTIGUOUS'] and not rt.flags['F_CONTIGUOUS']:
        d.has_tfrm = 2   # numpy takes the dgemv 't' path for rt.dot(v)
    else:
        d.has_tfrm = 1   # r.transpose() of a C array (elem/transform.py:86)
    for i in range(9):
        d.rt[i] = float(rt.reshape(-1)[i])
    for i in range(3):
        d.t[i] = float(t[i])


class UnsupportedInterfaceError(NotImplementedError):
    """The model contains an interface the table cannot represent (thin lens,
    diffractive/holographic phase element, user subclass ...)."""


def _describe_interface(seg, prev_n, prev_zdir):
    ifc, _gap, tfrm, n, z_dir = (tuple(seg) + (None,)*5)[:5]
    d = rt_surface_desc()
    if hasattr(ifc, 'phase_element'):   # same test as raytrace.py:205
        pe = ifc.phase_element
        kname = type(pe).__name__
        if kname not in PHASE_IDS:
            raise UnsupportedInterfaceError(
                f'{type(ifc).__name__} with a {kname} phase element is not supported by the surface table')
        d.phase_kind = PHASE_IDS[kname]
        if kname == 'HolographicElement':         # doe.py:326-395
            d.phase_flags = int(bool(pe.ref_virtual)) | (int(bool(pe.obj_virtual)) << 1)
            d.phase_ref_wl = float(pe.ref_wl)
            for i in range(3):
                d.phase_ref_pt[i] = float(pe.ref_pt[i])
                d.phase_obj_pt[i] = float(pe.obj_pt[i])
        elif kname == 'DiffractionGrating':       # doe.py:57-172 (phase() -> phase_ludwig)
            if getattr(ifc, 'interact_mode', None) not in ('transmit', 'reflect'):
                raise UnsupportedInterfaceError(
                    'DiffractionGrating on an interface that neither transmits nor reflects')
            d.phase_ref_wl = float(pe._grating_spacing_nm)
            d.phase_order = float(pe.order)
            for i in range(3):
                d.phase_ref_pt[i] = float(pe.grating_normal[i])
        else:                                     # DiffractiveElement, doe.py:214-323
            fct = getattr(pe, 'phase_fct', None)
            if getattr(fct, '__name__', None) != 'radial_phase_fct':
                raise UnsupportedInterfaceError(
                    'DiffractiveElement: only radial_phase_fct (doe.py:28-54) is compiled into the '
                    f'table, not {getattr(fct, "__name__", fct)!r}')
            cf = [float(c) for c in pe.coefficients]
            if len(cf) > RT_MAX_PHASE_COEFS:
                raise UnsupportedInterfaceError(
                    f'DiffractiveElement with {len(cf)} coefficients (max {RT_MAX_PHASE_COEFS})')
            d.phase_ref_wl = float(pe.ref_wl)
            d.phase_order = float(pe.order)
            d.n_phase_coefs = len(cf)
            for i, c in enumerate(cf):
                d.phase_coefs[i] = c
    profile = getattr(ifc, 'profile', None)
    pname = type(profile).__name__
    if type(ifc).__name__ == 'ThinLens':        # oprops/thinlens.py: no profile object
        pname = 'ThinLens'
        profile = _ThinLensProfile()
    if profile is None or pname not in PROFILE_IDS:
        raise UnsupportedInterfaceError(
            f'interface {type(ifc).__name__} / profile {pname} is not supported by the surface table')
    d.profile = PROFILE_IDS[pname]
    # raytrace.py:212-221: any unknown interact_mode passes the ray through
    d.mode = MODE_IDS.get(getattr(ifc, 'interact_mode', 'dummy'), MODE_IDS['dummy'])
    d.z_dir = int(z_dir if z_dir is not None else prev_zdir)
    d.cv, d.cc, d.ec = profile_fields(profile, pname)
    d.cR = float(getattr(profile, 'cR', 0.0))
    coefs = list(getattr(profile, 'coefs', []))
    k = getattr(profile, 'max_nonzero_coef', None)
    if k is None:
        k = 0
        for i, c in enumerate(coefs):
            if c != 0.0:
                k = i + 1
    if k > RT_MAX_COEFS:
        raise UnsupportedInterfaceError(f'{pname} with {k} coefficients (max {RT_MAX_COEFS})')
    d.n_coefs = int(k)
    for i in range(k):
        d.coefs[i] = float(coefs[i])
    d.max_aperture = float(getattr(ifc, 'max_aperture', 1.0))
    cas = list(getattr(ifc, 'clear_apertures', []) or [])
    if len(cas) > RT_MAX_APERTURES:
        raise UnsupportedInterfaceError(f'{len(cas)} clear apertures (max {RT_MAX_APERTURES})')
    d.n_apertures = len(cas)
    for i, ca in enumerate(cas):
        a = d.apertures[i]
        cname = type(ca).__name__
        if cname not in APERTURE_IDS:
            raise UnsupportedInterfaceError(f'aperture type {cname}')
        a.type = APERTURE_IDS[cname]
        a.is_obscuration = int(bool(getattr(ca, 'is_obscuration', False)))
        if cname == 'Circular':
            a.a, a.b = float(ca.radius), float(ca.radius)
        else:
            a.a, a.b = float(ca.x_half_width), float(ca.y_half_width)
        a.x_offset, a.y_offset = float(ca.x_offset), float(ca.y_offset)
    set_transform(d, tfrm)
    return d, float(n if n is not None else prev_n), d.z_dir


def describe_path(path):
    """path tuples -> (ctypes array of rt_surface_desc, list of indices)."""
    segs = list(path)
    arr = (rt_surface_desc*len(segs))()
    ns = []
    prev_n, prev_z = 1.0, 1
    for i, seg in enumerate(segs):
        d, prev_n, prev_z = _describe_interface(seg, prev_n, prev_z)
        arr[i] = d
        ns.append(prev_n)
    return arr, ns


def describe_model(seq_model, wvls=None):
    """All wavelengths of a sequential model -> (descs, n_by_wvl ndarray, wvls)."""
    if wvls is None:
        wvls = list(getattr(seq_model, 'wvlns', None) or [seq_model.central_wavelength()])
    descs = None
    rows = []
    for wl in wvls:
        if descs is None:
            descs, ns = describe_path(seq_model.path(wl))
        else:               # only the index column depends on the wavelength
            ns, prev_n = [], 1.0
            for seg in seq_model.path(wl):
                n = seg[3] if len(seg) > 3 else None
                prev_n = float(n if n is not None else prev_n)
                ns.append(prev_n)
        rows.append(ns)
    return descs, np.ascontiguousarray(np.array(rows, dtype=np.float64)), list(wvls)


class SurfaceTable:
    """Device-resident surface table (``rt_table*``) for one model.

    ``rt_table_create`` copies the descriptors to the device once; the handle
    is immutable and may be shared by threads / streams (SURVEY.md 8(b)).
    """

    def __init__(self, descs, n_by_wvl, wvls=None, device=0):
        lib = _abi.load_library()
        self.n_ifc = len(descs)
        self.n_by_wvl = np.ascontiguousarray(n_by_wvl, dtype=np.float64)
        assert self.n_by_wvl.shape[1] == self.n_ifc
        self.n_wvl = self.n_by_wvl.shape[0]
        self.wvls = list(wvls) if wvls is not None else list(range(self.n_wvl))
        self.descs = descs
        self.device = int(device)
        handle = C.c_void_p()
        _abi.check(lib.rt_table_create(descs, self.n_ifc,
                                       self.n_by_wvl.ctypes.data_as(_abi.c_double_p),
                                       self.n_wvl, self.device, C.byref(handle)))
        self._handle = handle
        self._lib = lib
        if wvls is not None and all(isinstance(w, (int, float)) for w in wvls):
            w = np.ascontiguousarray(wvls, dtype=np.float64)
            _abi.check(lib.rt_table_set_wavelengths(handle, w.ctypes.data_as(_abi.c_double_p)))

    @classmethod
    def from_model(cls, seq_model, wvls=None, device=0):
        descs, n_by_wvl, wvls = describe_model(seq_model, wvls)
        return cls(descs, n_by_wvl, wvls, device)

    @classmethod
    def from_path(cls, path, device=0, wvl=None):
        descs, ns = describe_path(path)
        return cls(descs, np.array([ns]), None if wvl is None else [float(wvl)], device)

    @property
    def handle(self):
        if self._handle is None:
            raise RuntimeError('SurfaceTable was destroyed')
        return self._handle

    def wvl_index(self, wvl):
        return self.wvls.index(wvl)

    def close(self):
        if getattr(self, '_handle', None) is not None:
            self._lib.rt_table_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
