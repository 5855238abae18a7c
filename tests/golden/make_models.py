#!/usr/bin/env python3
"""Write the model fixtures tests/golden/models/*.json (format b200rt-model-v1).

Runs ONLY in the build container: it reads the reference's bundled lens data
under /root/reference (which does not exist on the GPU box) and uses the
reference's own ``trace_raw`` (through oracle/ref_harness.py) for chief-ray
aiming and clear apertures.  The JSON it writes is committed, so tests, smoke()
and bench.py never need the reference tree.

Sources (numbers only; no reference source code is copied):
  singlet     /root/reference/src/rayoptics/models/singlet_f5.roa
  dblgauss    /root/reference/src/rayoptics/raytr/tests/ag_dblgauss_s.py  [cv, thi, n_d, V_d]
              + spec of /root/reference/src/rayoptics/codev/tests/ag_dblgauss.seq
              (EPD 50, fields 0/10/14 deg, VUY/VLY, WL 656.3 587.6 486.1, stop at surface 6)
  triplet     /root/reference/src/rayoptics/models/Sasian Triplet.roa
  rc          /root/reference/src/rayoptics/models/Ritchey_Chretien.roa (5 fields interpolated)
  cellphone   /root/reference/src/rayoptics/optical/tests/cell_phone_camera.roa (9 fields)
  cellphone_even  same lens, RadialPolynomial surfaces replaced by EvenPolynomial
              ones built from their even-order coefficients (synthetic)
  evenasph    /root/reference/src/rayoptics/zemax/tests/US08427765-1.ZMX geometry, with
              catalogue glasses replaced by (n_d, V_d) Cauchy models (approximate)
  zoom52      synthetic 50-surface stack (recipe below), 25 fields x 7 wavelengths
  fisheye     synthetic wide-angle lens (two negative menisci, stop, positive group; fields to 75
              degrees, fov.is_wide_angle): the real entrance pupil position of every field
              (fld.aim_info = z_enp) is found by the REFERENCE's own raytr/wideangle.py
              find_real_enp on the hybrid model
  threemir    /root/reference/src/rayoptics/codev/tests/threemir.seq (CODE V three-mirror
              compact: conic / aspheric mirrors, every surface decentered and tilted with
              'dec and return'), read by rayoptics_b200/seq.py
  edge_sphere, edge_conic, edge_even, edge_radial, edge_stops
              synthetic finite-conjugate lenses for the boundary rays of make_golden_edges.py
"""
import importlib.util
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh                      # noqa: E402
from rayoptics_b200 import model as M, roa, vigcalc, seq  # noqa: E402
from rayoptics_b200.opticalspec import (OpticalSpecs, WvlSpec, PupilSpec, FieldSpec,  # noqa: E402
                                        FocusRange)

REF = '/root/reference/src/rayoptics'
OUT = os.path.join(HERE, 'models')


def ref_trace_fn(sm, pt0, dir0, wvl, **kw):
    """trace() semantics of raytrace.py:51-80 on the reference's own trace_raw."""
    R = rh.ref()
    path = rh.ref_path(sm, wvl)
    kw.setdefault('first_surf', 1)
    kw.setdefault('last_surf', sm.get_num_surfaces() - 2)
    return R.raytrace.trace_raw(iter(path), np.array(pt0, dtype=float),
                                np.array(dir0, dtype=float), wvl, **kw)


def finish(opm, aim=True, apertures=True):
    opm.update_model()
    if aim:
        vigcalc.aim_all_fields(opm, ref_trace_fn)
    if apertures:
        vigcalc.set_clear_apertures(opm, ref_trace_fn)
    return opm


def dblgauss():
    spec = importlib.util.spec_from_file_location(
        'dblg', f'{REF}/raytr/tests/ag_dblgauss_s.py')
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    rows = [list(r) for r in mod.ag_dblgauss]
    rows[-2][1] += rows[-1][1]      # lump the defocus into the back focal distance,
    rows[-1][1] = 0.0               # as raytr/tests/test_sequential.py:26-27 does
    wvls = [656.3, 587.6, 486.1]
    sm = M.gen_sequence(rows, wvls=wvls, ref_wvl=1, stop_surface=6)
    sm.ifcs[6].interact_mode = 'dummy'      # STO plane (ag_dblgauss.seq:26-28)
    fields = [M.Field(y=0.0), M.Field(y=10.0000000023, vuy=0.2, vly=0.25),
              M.Field(y=14.0000000032, vuy=0.4, vly=0.4)]
    osp = OpticalSpecs(WvlSpec(wvls, 1), PupilSpec(('object', 'epd'), 50.0),
                       FieldSpec(('object', 'angle'), 14.0000000032, fields))
    return finish(M.OpticalModel(sm, osp, name='dblgauss'))


def from_roa(rel, name, n_fields=None, aim=False, apertures=False):
    opm = roa.open_roa(f'{REF}/{rel}')
    opm.name = name
    if n_fields is not None:
        fov = opm.optical_spec.field_of_view
        ymax = max(f.y for f in fov.fields)
        fov.fields = [M.Field(y=ymax*i/(n_fields - 1)) for i in range(n_fields)]
        aim = True
    return finish(opm, aim=aim, apertures=apertures)


def cellphone_even():
    opm = roa.open_roa(f'{REF}/optical/tests/cell_phone_camera.roa')
    opm.name = 'cellphone_even'
    for ifc in opm.seq_model.ifcs:
        p = ifc.profile
        if type(p).__name__ == 'RadialPolynomial':
            even = [p.coefs[i] if i < len(p.coefs) else 0.0 for i in range(1, 10, 2)]
            ifc.profile = M.EvenPolynomial(c=p.cv, ec=p.ec, coefs=even)
    fov = opm.optical_spec.field_of_view
    fov.fields = [M.Field(y=i/8) for i in range(9)]
    return finish(opm)


def evenasph():
    # geometry of zemax/tests/US08427765-1.ZMX (SURF 0..12); glasses -> (n_d, V_d)
    glass = {'J-LAK14': (1.6968, 55.5), 'L-TIM28': (1.68893, 31.1), 'SF11': (1.78472, 25.7),
             'TAF3': (1.8042, 46.5), 'TAFD30': (1.883, 40.8)}
    surf = [  # cv, thi, glass, evenasph(cc, coefs)
        (7.7669902912621352e-02, 3.34, 'J-LAK14', None),
        (2.8248587570621469e-02, 0.29, None, None),
        (7.2306579898770790e-02, 1.85, 'L-TIM28', None),
        (1.1178180192264700e-01, 4.25, None, (2.0e-2, [0.0, 1.10721e-5, 1.837e-7])),
        (0.0, 5.4, None, None),            # STOP
        (-1.2048192771084336e-01, 0.65, 'SF11', None),
        (-1.8660197798096658e-02, 0.22, None, None),
        (-2.6688017080330931e-02, 3.62, 'TAF3', None),
        (-8.5012326787384171e-02, 0.12, None, None),
        (4.8473097430925833e-03, 3.5, 'TAFD30', None),
        (-3.7707390648567117e-02, 21.25417782777, None, None)]
    ifcs = [M.Surface(lbl='Obj', interact_mode='dummy')]
    gaps = [M.Gap(1e10)]
    for i, (cv, thi, g, asp) in enumerate(surf):
        prf = M.Spherical(c=cv) if asp is None else M.EvenPolynomial(c=cv, cc=asp[0], coefs=asp[1])
        mode = 'dummy' if i == 4 else 'transmit'
        ifcs.append(M.Surface(profile=prf, interact_mode=mode))
        gaps.append(M.Gap(thi, M.AbbeGlass(*glass[g], label=g) if g else M.Air()))
    ifcs.append(M.Surface(lbl='Img', interact_mode='dummy'))
    wvls = [486.1327, 587.5618, 656.2725]
    sm = M.SequentialModel(ifcs, gaps, stop_surface=5, wvlns=wvls, ref_wvl=1)
    fields = [M.Field(y=13.6*i/8) for i in range(9)]
    osp = OpticalSpecs(WvlSpec(wvls, 1), PupilSpec(('image', 'f/#'), 2.1),
                       FieldSpec(('object', 'angle'), 13.6, fields))
    return finish(M.OpticalModel(sm, osp, name='evenasph'))


def zoom52():
    """Synthetic 50-surface stack: 12 weak air-spaced doublet cells (4 surfaces
    each) + one focusing singlet.  Deterministic, no RNG."""
    ifcs = [M.Surface(lbl='Obj', interact_mode='dummy')]
    gaps = [M.Gap(1e10)]
    crown, flint = M.AbbeGlass(1.62041, 60.3, 'crown'), M.AbbeGlass(1.60342, 38.0, 'flint')
    for c in range(12):
        s = 1.0 + 0.02*c
        cell = [(1/(150.0*s), 6.0, crown), (-1/(320.0*s), 1.5, None),
                (-1/(140.0*s), 3.0, flint), (1/(600.0*s), 6.0, None)]
        if c % 3 == 1:   # every third cell carries conic surfaces
            profs = [M.Conic(c=cell[0][0], cc=-0.4), M.Spherical(c=cell[1][0]),
                     M.Conic(c=cell[2][0], cc=0.25), M.Spherical(c=cell[3][0])]
        else:
            profs = [M.Spherical(c=k[0]) for k in cell]
        for prf, (cv, thi, g) in zip(profs, cell):
            ifcs.append(M.Surface(profile=prf))
            gaps.append(M.Gap(thi, g if g else M.Air()))
    ifcs.append(M.Surface(profile=M.Spherical(c=1/90.0)))
    gaps.append(M.Gap(7.0, crown))
    ifcs.append(M.Surface(profile=M.Spherical(c=-1/400.0)))
    gaps.append(M.Gap(100.0))
    ifcs.append(M.Surface(lbl='Img', interact_mode='dummy'))
    wvls = [656.3, 620.0, 587.6, 550.0, 520.0, 486.1, 450.0]
    sm = M.SequentialModel(ifcs, gaps, stop_surface=25, wvlns=wvls, ref_wvl=2)
    fields = [M.Field(y=3.0*i/24) for i in range(25)]
    osp = OpticalSpecs(WvlSpec(wvls, 2), PupilSpec(('object', 'epd'), 24.0),
                       FieldSpec(('object', 'angle'), 3.0, fields))
    opm = M.OpticalModel(sm, osp, name='zoom52')
    sm.gaps[-1].thi = float(osp.fod.img_dist)     # paraxial focus
    return finish(opm)


def exotic():
    """Synthetic model exercising everything the quadric lenses do not: Y/X toroids,
    even and radial polynomials, rectangular aperture with offset, circular
    obscuration, a phantom interface, tilted / decentered transforms in both
    numpy memory layouts (rayoptics_b200/table.py has_tfrm 1 and 2), finite object."""
    def rot(ax, ay):
        cx, sx, cy, sy = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay)
        Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
        Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
        return Rx @ Ry
    g1, g2 = M.AbbeGlass(1.6, 50.0, 'g1'), M.AbbeGlass(1.7, 30.0, 'g2')
    spec = [  # profile, mode, thi, medium, max_aperture
        (M.Spherical(0.0), 'dummy', 200.0, M.Air(), 50.0),
        (M.Conic(c=0.02, cc=-0.6), 'transmit', 6.0, g1, 14.0),
        (M.YToroid(c=-0.01, cR=-0.012, cc=0.2, coefs=[0.0, 2e-7]), 'transmit', 3.0, M.Air(), 14.0),
        (M.XToroid(c=0.015, cR=0.013, cc=-0.3, coefs=[0.0, -1e-7, 1e-10]), 'transmit', 5.0, g2, 13.0),
        (M.Spherical(0.0), 'phantom', 2.0, g2, 13.0),
        (M.EvenPolynomial(c=-0.025, cc=-0.4, coefs=[0.0, 1.5e-6, -2e-9, 1e-12]), 'transmit', 8.0, M.Air(), 12.0),
        (M.RadialPolynomial(c=0.03, ec=0.8, coefs=[0.0, 0.0, 2e-5, -3e-6, 1e-7]), 'transmit', 4.0, g1, 11.0),
        (M.Conic(c=-0.028, cc=0.5), 'transmit', 60.0, M.Air(), 11.0),
        (M.Spherical(0.0), 'dummy', 0.0, None, 30.0)]
    ifcs, gaps = [], []
    for prf, mode, thi, med, ap in spec:
        ifcs.append(M.Surface(profile=prf, interact_mode=mode, max_aperture=ap))
        if med is not None:
            gaps.append(M.Gap(thi, med))
    ifcs[2].clear_apertures = [M.Rectangular(12.0, 9.0, x_offset=0.5, y_offset=-0.4)]
    ifcs[5].clear_apertures = [M.Circular(11.5), M.Circular(1.2, is_obscuration=True, x_offset=0.3)]
    tf = []
    for i, g in enumerate(gaps):
        if i in (1, 2, 5, 6):
            R = rot(0.01*(i + 1)*(-1)**i, 0.008*(i + 2))
            rt = R.T if i % 2 else np.ascontiguousarray(R)     # F-ordered view / C array
            tf.append((rt, np.array([0.05*(i - 3), -0.03*i, g.thi])))
        else:
            tf.append((np.identity(3), np.array([0., 0., g.thi])))
    tf.append((np.identity(3), np.zeros(3)))
    wvls = [656.3, 587.6, 486.1]
    sm = M.SequentialModel(ifcs, gaps, stop_surface=None, wvlns=wvls, ref_wvl=1, lcl_tfrms=tf)
    sm.stop_surface = 4
    fields = [M.Field(y=0.0), M.Field(y=6.0), M.Field(x=4.0, y=-5.0)]
    osp = OpticalSpecs(WvlSpec(wvls, 1), PupilSpec(('object', 'epd'), 16.0),
                       FieldSpec(('object', 'height'), 6.0, fields))
    return finish(M.OpticalModel(sm, osp, name='exotic'), aim=False, apertures=False)


def diffractive():
    """Hybrid lens with the three diffractive phase elements of oprops/doe.py that have
    closed forms: radial-phase DiffractiveElement on a glass->air surface (bends to and
    from index 1, doe.py:296-299,319-321) and on an air->glass surface (no bends: the
    reference tests n_in only), a transmission DiffractionGrating and a reflective one
    on a concave mirror (z_dir flips, negative gap)."""
    g1, g2 = M.AbbeGlass(1.5168, 64.2, 'g1'), M.AbbeGlass(1.6, 40.0, 'g2')
    spec = [  # profile, mode, thi, medium, max_aperture, phase element
        (M.Spherical(0.0), 'dummy', 1e10, M.Air(), 1e9, None),
        (M.Spherical(0.02), 'transmit', 4.0, g1, 9.0, None),
        (M.Spherical(-0.01), 'transmit', 10.0, M.Air(), 9.0,
         M.DiffractiveElement(coefficients=[-1.0e-3, 1.0e-7, -2.0e-10], ref_wl=587.6, order=1)),
        (M.Conic(0.004, cc=-0.5), 'transmit', 3.0, g2, 9.0,
         M.DiffractiveElement(coefficients=[4.0e-4, -3.0e-8], ref_wl=550.0, order=-1)),
        (M.Spherical(0.0), 'transmit', 20.0, M.Air(), 9.0, None),
        (M.Spherical(0.0), 'transmit', 30.0, M.Air(), 12.0,
         M.DiffractionGrating(order=1, grating_lpmm=100.0, interact_mode='transmit')),
        (M.Spherical(-0.004), 'reflect', -60.0, M.Air(), 20.0,
         M.DiffractionGrating(order=-1, grating_normal=[0.2, 1.0, 0.05], grating_lpmm=150.0,
                              interact_mode='reflect')),
        (M.Spherical(0.0), 'dummy', 0.0, None, 60.0, None)]
    ifcs, gaps = [], []
    for prf, mode, thi, med, ap, pe in spec:
        sfc = M.Surface(profile=prf, interact_mode=mode, max_aperture=ap)
        if pe is not None:
            sfc.phase_element = pe
        ifcs.append(sfc)
        if med is not None:
            gaps.append(M.Gap(thi, med))
    wvls = [656.3, 587.6, 486.1]
    sm = M.SequentialModel(ifcs, gaps, stop_surface=1, wvlns=wvls, ref_wvl=1)
    fields = [M.Field(y=0.0), M.Field(y=1.0), M.Field(x=0.5, y=-1.0)]
    osp = OpticalSpecs(WvlSpec(wvls, 1), PupilSpec(('object', 'epd'), 12.0),
                       FieldSpec(('object', 'angle'), 1.0, fields))
    return finish(M.OpticalModel(sm, osp, name='diffractive'), aim=False, apertures=False)


def diffractive_wild():
    """Strong diffractive elements at steep angles: exercises the failure branches of
    oprops/doe.py (math.sqrt ValueError -> TraceEvanescentRayError in the DOE bends and
    roots, np.sqrt NaN propagation in the grating) against the reference itself."""
    g = M.ConstantIndex(1.7, 'n17')
    spec = [
        (M.Spherical(0.0), 'dummy', 20.0, M.Air(), 50.0, None),
        (M.Spherical(0.0), 'transmit', 5.0, g, 40.0,
         M.DiffractiveElement(coefficients=[4.0e-3, -2.0e-5], ref_wl=550.0, order=2)),
        (M.Spherical(0.01), 'transmit', 10.0, M.Air(), 40.0,
         M.DiffractiveElement(coefficients=[-3.0e-3, 2.0e-5, 1.0e-7], ref_wl=600.0, order=1)),
        (M.Spherical(0.0), 'transmit', 10.0, M.Air(), 60.0,
         M.DiffractionGrating(order=1, grating_normal=[0.0, 1.0, 0.0], grating_lpmm=800.0,
                              interact_mode='transmit')),
        (M.Spherical(0.002), 'reflect', -20.0, M.Air(), 80.0,
         M.DiffractionGrating(order=1, grating_normal=[1.0, 0.3, 0.0], grating_lpmm=500.0,
                              interact_mode='reflect')),
        (M.Spherical(0.0), 'dummy', 0.0, None, 400.0, None)]
    ifcs, gaps = [], []
    for prf, mode, thi, med, ap, pe in spec:
        sfc = M.Surface(profile=prf, interact_mode=mode, max_aperture=ap)
        if pe is not None:
            sfc.phase_element = pe
        ifcs.append(sfc)
        if med is not None:
            gaps.append(M.Gap(thi, med))
    wvls = [656.3, 587.6, 486.1]
    sm = M.SequentialModel(ifcs, gaps, stop_surface=1, wvlns=wvls, ref_wvl=1)
    fields = [M.Field(y=0.0), M.Field(y=4.0), M.Field(x=-3.0, y=2.0)]
    osp = OpticalSpecs(WvlSpec(wvls, 1), PupilSpec(('object', 'epd'), 24.0),
                       FieldSpec(('object', 'height'), 4.0, fields))
    return finish(M.OpticalModel(sm, osp, name='diffractive_wild'), aim=False, apertures=False)


def telecentric():
    """Image-space telecentric lens: aperture stop in the front focal plane of a
    two-element group, so the exit pupil is ~1e10+ mm away and the reference's
    wavefront code takes the INFINITE reference sphere branch
    (raytr/waveabr.py:206-253 `is_kinda_big(ref_sphere_radius)`, :356-420)."""
    g1, g2 = M.AbbeGlass(1.6204, 60.3, 'SK16'), M.AbbeGlass(1.6727, 32.2, 'SF5')

    def build(d_stop, bfl):
        spec = [(0.0, 'dummy', 1e10, M.Air(), None), (0.0, 'dummy', d_stop, M.Air(), None),
                (1/80.0, 'transmit', 7.0, g1, None), (-1/45.0, 'transmit', 2.5, g2, None),
                (-1/160.0, 'transmit', 30.0, M.Air(), None),
                (1/70.0, 'transmit', 6.0, g1, None), (0.0, 'transmit', bfl, M.Air(), None),
                (0.0, 'dummy', 0.0, None, None)]
        ifcs, gaps = [], []
        for cv, mode, thi, med, _ in spec:
            ifcs.append(M.Surface(profile=M.Spherical(cv), interact_mode=mode))
            if med is not None:
                gaps.append(M.Gap(thi, med))
        wvls = [656.3, 587.6, 486.1]
        sm = M.SequentialModel(ifcs, gaps, stop_surface=1, wvlns=wvls, ref_wvl=1)
        fields = [M.Field(y=0.0), M.Field(y=3.5), M.Field(y=5.0)]
        osp = OpticalSpecs(WvlSpec(wvls, 1), PupilSpec(('object', 'epd'), 10.0),
                           FieldSpec(('object', 'angle'), 5.0, fields))
        return M.OpticalModel(sm, osp, name='telecentric')

    # stop distance that sends the exit pupil to infinity (secant on 1/exp_dist), then
    # the paraxial image distance
    def inv_exp(d):
        opm = build(d, 50.0)
        opm.update_model()
        return 1.0/opm.optical_spec.fod.exp_dist
    d0, d1 = 30.0, 40.0
    f0, f1 = inv_exp(d0), inv_exp(d1)
    for _ in range(60):
        if f1 == f0:
            break
        d2 = d1 - f1*(d1 - d0)/(f1 - f0)
        d0, f0, d1, f1 = d1, f1, d2, inv_exp(d2)
        if abs(f1) < 1e-13:
            break
    opm = build(d1, 50.0)
    opm.update_model()
    opm = build(d1, opm.optical_spec.fod.img_dist if hasattr(opm.optical_spec.fod, 'img_dist')
                else opm.optical_spec.fod.bfl)
    return finish(opm)


def relay(pupil_key, pupil_value, name):
    """Finite-conjugate relay specified by an ANGULAR object-space pupil ('NA' or 'f/#'):
    the start rays take the angular branch of ray_start_from_osp (opticalspec.py:368-398)."""
    g = M.AbbeGlass(1.5168, 64.2, 'BK7')
    spec = [(0.0, 'dummy', 100.0, M.Air()), (1/55.0, 'transmit', 6.0, g), (-1/55.0, 'transmit', 12.0, M.Air()),
            (0.0, 'dummy', 12.0, M.Air()), (1/60.0, 'transmit', 6.0, g), (-1/50.0, 'transmit', 95.0, M.Air()),
            (0.0, 'dummy', 0.0, None)]
    ifcs, gaps = [], []
    for cv, mode, thi, med in spec:
        ifcs.append(M.Surface(profile=M.Spherical(cv), interact_mode=mode))
        if med is not None:
            gaps.append(M.Gap(thi, med))
    wvls = [656.3, 587.6, 486.1]
    sm = M.SequentialModel(ifcs, gaps, stop_surface=3, wvlns=wvls, ref_wvl=1)
    fields = [M.Field(y=0.0), M.Field(y=3.0), M.Field(x=2.0, y=-4.0)]
    osp = OpticalSpecs(WvlSpec(wvls, 1), PupilSpec(('object', pupil_key), pupil_value),
                       FieldSpec(('object', 'height'), 4.0, fields))
    return finish(M.OpticalModel(sm, osp, name=name), aim=False, apertures=True)


EDGE_PROFILES = {
    'sphere': lambda: M.Spherical(c=0.125),
    'conic': lambda: M.Conic(c=0.125, cc=-0.5),
    'even': lambda: M.EvenPolynomial(c=0.125, cc=-0.5, coefs=[0.0, 1e-4]),
    'radial': lambda: M.RadialPolynomial(c=0.125, ec=0.5, coefs=[0.0, 0.0, 1e-4]),
}


def edge_lens(kind):
    """Synthetic finite-conjugate lens for the boundary rays of make_golden_edges.py.  The object
    sits in an index-2 medium, so surface 1 (the profile under test, index 2 -> 1.5, radius 8,
    clear aperture 2) shows clipping, TIR (|sin I| > 3/4) and a miss (grazing at height ~8) to
    rays parallel to the axis.  cv = 1/8 and the indices 2 and 1.5 are chosen so that the
    quantities that decide (r**2 - L**2, n'**2 - n**2 sin**2 I, b**2 - a*c) cancel exactly for
    some start rays instead of only approximately.  Surface 2 is a plano 1.5 -> 1.75 interface
    that on-axis rays hit at its vertex."""
    n2, n15, n175 = M.ConstantIndex(2.0, 'n2'), M.ConstantIndex(1.5, 'n15'), M.ConstantIndex(1.75, 'n175')
    spec = [(M.Spherical(0.0), 'dummy', 10.0, n2, 1e3),
            (EDGE_PROFILES[kind](), 'transmit', 6.0, n15, 2.0),
            (M.Spherical(0.0), 'transmit', 5.0, n175, 20.0),
            (M.Spherical(0.0), 'dummy', 0.0, None, 1e3)]
    ifcs, gaps = [], []
    for prf, mode, thi, med, ap in spec:
        ifcs.append(M.Surface(profile=prf, interact_mode=mode, max_aperture=ap))
        if med is not None:
            gaps.append(M.Gap(thi, med))
    wvls = [587.6]
    sm = M.SequentialModel(ifcs, gaps, stop_surface=1, wvlns=wvls, ref_wvl=0)
    fields = [M.Field(y=0.0), M.Field(x=0.3, y=0.5)]
    osp = OpticalSpecs(WvlSpec(wvls, 0), PupilSpec(('object', 'epd'), 8.0),
                       FieldSpec(('object', 'height'), 0.5, fields))
    return finish(M.OpticalModel(sm, osp, name='edge_' + kind), aim=False, apertures=False)


def edge_stops():
    """Synthetic lens of plano interfaces with aperture lists (general kernel only): a
    rectangular stop with an offset, then an offset circular stop (inside the rectangle) with an
    offset circular obscuration.  Rays parallel to the axis keep their start x, y exactly up to
    the stops."""
    n15 = M.ConstantIndex(1.5, 'n15')
    spec = [('dummy', 10.0, M.Air()), ('transmit', 3.0, n15), ('transmit', 4.0, M.Air()),
            ('dummy', 0.0, None)]
    ifcs, gaps = [], []
    for mode, thi, med in spec:
        ifcs.append(M.Surface(profile=M.Spherical(0.0), interact_mode=mode, max_aperture=1e3))
        if med is not None:
            gaps.append(M.Gap(thi, med))
    ifcs[1].clear_apertures = [M.Rectangular(5.0, 4.0, x_offset=0.25, y_offset=-0.5)]
    ifcs[2].clear_apertures = [M.Circular(3.0, x_offset=0.3, y_offset=0.2),
                               M.Circular(1.0, is_obscuration=True, x_offset=-0.2, y_offset=0.1)]
    wvls = [587.6]
    sm = M.SequentialModel(ifcs, gaps, stop_surface=1, wvlns=wvls, ref_wvl=0)
    osp = OpticalSpecs(WvlSpec(wvls, 0), PupilSpec(('object', 'epd'), 6.0),
                       FieldSpec(('object', 'height'), 1.0, [M.Field(y=0.0), M.Field(y=1.0)]))
    return finish(M.OpticalModel(sm, osp, name='edge_stops'), aim=False, apertures=False)


def fisheye():
    import importlib
    import warnings
    from oracle import ref_model
    g1 = M.AbbeGlass(1.62041, 60.32, label='SK16')
    g2 = M.AbbeGlass(1.7847, 25.7, label='SF11')

    def build(img_thi):
        rows = [(0.0, 1e10, M.Air()),
                (1/45.0, 2.5, g1), (1/14.0, 11.0, M.Air()),
                (1/32.0, 2.0, g1), (1/10.5, 14.0, M.Air()),
                (0.0, 1.5, M.Air()),                                   # stop
                (1/38.0, 3.5, g1), (-1/15.0, 0.3, M.Air()),
                (1/22.0, 4.5, g1), (-1/11.0, 1.2, g2), (-1/36.0, img_thi, M.Air()),
                (0.0, 0.0, None)]
        ifcs, gaps = [], []
        for i, (cv, thi, med) in enumerate(rows):
            mode = 'dummy' if i in (0, 5, len(rows) - 1) else 'transmit'
            ifcs.append(M.Surface(profile=M.Spherical(c=cv), interact_mode=mode, max_aperture=30.0))
            if med is not None:
                gaps.append(M.Gap(thi, med))
        wv = [656.3, 587.6, 486.1]
        sm = M.SequentialModel(ifcs, gaps, stop_surface=5, wvlns=wv, ref_wvl=1)
        fields = [M.Field(0., 0.), M.Field(0., 35.), M.Field(0., 60.), M.Field(0., 75.)]
        osp = OpticalSpecs(WvlSpec(wv, 1), PupilSpec(('object', 'epd'), 2.0),
                           FieldSpec(('object', 'angle'), 75.0, fields, is_wide_angle=True),
                           FocusRange(0.0))
        opm = M.OpticalModel(sm, osp, name='fisheye')
        opm.update_model()
        return opm

    opm = build(build(20.0).optical_spec.fod.bfl)
    ref_model.modules()
    WA = importlib.import_module('rayoptics.raytr.wideangle')
    H = ref_model.HybridModel(opm)
    for f in opm.optical_spec.field_of_view.fields:
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            z_enp, rr = WA.find_real_enp(H, opm.seq_model.stop_surface, f, 587.6)
        assert rr.err is None
        f.aim_info = float(z_enp)
    return finish(opm, aim=False, apertures=True)


def threemir():
    opm = seq.open_seq(f'{REF}/codev/tests/threemir.seq')
    opm.name = 'threemir'
    return finish(opm, aim=True, apertures=True)


def main():
    os.makedirs(OUT, exist_ok=True)
    models = {
        'threemir': threemir,
        'fisheye': fisheye,
        'singlet': lambda: from_roa('models/singlet_f5.roa', 'singlet'),
        'dblgauss': dblgauss,
        'triplet': lambda: from_roa('models/Sasian Triplet.roa', 'triplet'),
        'rc': lambda: from_roa('models/Ritchey_Chretien.roa', 'rc', n_fields=5, apertures=True),
        'cellphone': lambda: from_roa('optical/tests/cell_phone_camera.roa', 'cellphone',
                                      n_fields=9),
        'cellphone_even': cellphone_even,
        'evenasph': evenasph,
        'zoom52': zoom52,
        # 3 ThinLens interfaces (HolographicElement phase), models/thin_triplet.roa
        'thin_triplet': lambda: from_roa('models/thin_triplet.roa', 'thin_triplet'),
        'exotic': exotic,
        'telecentric': telecentric,
        'relay_na': lambda: relay('NA', 0.07, 'relay_na'),
        'relay_fno': lambda: relay('f/#', 7.0, 'relay_fno'),
        'hybrid': lambda: from_roa('models/HybridAchromat.roa', 'hybrid'),
        'diffractive': diffractive,
        'diffractive_wild': diffractive_wild,
        **{'edge_' + k: (lambda k=k: edge_lens(k)) for k in EDGE_PROFILES},
        'edge_stops': edge_stops,
    }
    only = sys.argv[1:]
    for name, fn in models.items():
        if only and name not in only:
            continue
        opm = fn()
        opm.save(os.path.join(OUT, name + '.json'))
        fod = opm.optical_spec.fod
        print(f'{name:15s} n_ifc={opm.seq_model.get_num_surfaces():3d} efl={fod.efl:10.4f} '
              f'enp_dist={fod.enp_dist:10.4f} enp_r={fod.enp_radius:8.4f} '
              f'aims={[None if f.aim_info is None else np.round(f.aim_info, 6).tolist() for f in opm.optical_spec.fov.fields][:3]}')


if __name__ == '__main__':
    main()
