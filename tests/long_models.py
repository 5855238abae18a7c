"""Long-system fixtures (test helper, package only): built in memory, deterministic, no RNG, no
reference, so that nothing large is committed for them.  ``load(name)`` returns the model.

Each fixture is a periodic relay of weak singlets (f ~ 250 mm, spacing 60 mm < 4f, so the paraxial
rays stay bounded over hundreds of interfaces), a dummy stop in the middle, an 'epd' pupil, 3 fields
and the image at paraxial focus.  The sizes place the surface tables on the shared-memory budgets of
rt_table_create (csrc/b200rt.cu), 204 800 - 30 720 = 174 080 bytes (n_ifc counts the object and the
image, w is the number of wavelengths):

  long640   quadric, w = 5, n = 640: lean plan n (112 + 32 w) = 174 080 B, exactly the budget
  long360   quadric, w = 5, n = 360: lean plan 97 920 B (one summary CTA per SM, two of the rest)
  long320   Even / Radial polynomials, w = 3, n = 320: lean POLY plan n (448 + 32 w) = 174 080 B
  long256   general (a rectangular clear aperture, a tilted and decentered pair in both numpy
            layouts), w = 5, n = 256: staged table n (640 + 8 w) = 174 080 B

Every fixture clips the pupil edge mid-stack (max_aperture, status 3) and carries one steep
meniscus (radius 9 mm), where wild rays miss or are totally reflected.
"""
import numpy as np

from rayoptics_b200 import model as M
from rayoptics_b200.opticalspec import OpticalSpecs, WvlSpec, PupilSpec, FieldSpec

GLASS = M.AbbeGlass(1.5168, 64.2, 'BK7')
STEEP = M.AbbeGlass(1.7847, 25.7, 'SF11')
WVLS = {5: [656.3, 620.0, 587.6, 520.0, 486.1], 3: [656.3, 587.6, 486.1]}
R_LENS, T_GLASS, T_AIR = 250.0, 4.0, 56.0       # singlet radii, glass and air thicknesses (mm)
EPD, FIELD_DEG, AP = 12.0, 0.4, 40.0


def profile(kind, k, cv):
    """surface k of a singlet stack: the profile family the fixture stands for"""
    if kind == 'poly':
        if k % 4 == 0:
            return M.EvenPolynomial(c=cv, cc=-0.3, coefs=[0.0, 2e-9, -1e-13])
        if k % 4 == 2:
            return M.RadialPolynomial(c=cv, ec=0.9, coefs=[0.0, 0.0, 1e-9, 0.0, -2e-13])
        return M.Spherical(c=cv)
    if k % 3 == 0:
        return M.Conic(c=cv, cc=-0.5)
    return M.Spherical(c=cv)


def rows(n_ifc, kind):
    """(profile, interact_mode, thickness, medium) of interfaces 0 ... n_ifc - 2 (the image is
    added by build): singlets on both sides of a dummy stop, the steep meniscus in the first
    half, plano dummies to fill an odd count"""
    inner = n_ifc - 2                                # interfaces between object and image
    n_lens = (inner - 1 - 2)//2                      # - stop - meniscus
    fill = inner - 1 - 2 - 2*n_lens
    out = [(M.Spherical(0.0), 'dummy', 1e10, M.Air())]
    k = 0
    for i in range(n_lens):
        if i == n_lens//2:
            out.append((M.Spherical(0.0), 'dummy', T_AIR/2, M.Air()))               # the stop
        if i == n_lens//4:
            out.append((M.Spherical(1/9.0), 'transmit', 3.0, STEEP))
            out.append((M.Spherical(1/9.2), 'transmit', T_AIR, M.Air()))
        out.append((profile(kind, k, 1/R_LENS), 'transmit', T_GLASS, GLASS))
        out.append((profile(kind, k + 1, -1/R_LENS), 'transmit', T_AIR, M.Air()))
        k += 2
    for _ in range(fill):
        out.append((M.Spherical(0.0), 'dummy', 1.0, M.Air()))
    return out


def paraxial_heights(spec, wvl_n):
    """marginal ray height (EPD/2, object at infinity) at every interface of ``spec``"""
    y, u, n = EPD/2, 0.0, 1.0
    hs = [y]
    for j, (prf, mode, thi, med) in enumerate(spec):
        if j:
            n2 = med.rindex(wvl_n)
            if mode == 'transmit':
                u = (n*u - y*prf.cv*(n2 - n))/n2
            n = n2
            hs.append(y)
        y = y + thi*u if j else y
    return np.array(hs)


def build(name, n_ifc, n_wvl, kind, img_thi=None):
    spec = rows(n_ifc, kind)
    wvls = WVLS[n_wvl]
    stop = next(i for i, r in enumerate(spec) if r[1] == 'dummy' and i > 0)
    ys = paraxial_heights(spec, wvls[n_wvl//2])
    clip = 3*len(spec)//4                            # a lens surface behind the stop
    while spec[clip][1] != 'transmit':
        clip += 1
    ifcs, gaps = [], []
    for j, (prf, mode, thi, med) in enumerate(spec):
        ap = 1e10 if j == 0 else AP
        if j == clip:
            ap = 0.9*abs(ys[j])                      # the pupil edge is clipped here (status 3)
        ifcs.append(M.Surface(profile=prf, interact_mode=mode, max_aperture=ap))
        gaps.append(M.Gap(thi, med))
    gaps[-1].thi = 100.0 if img_thi is None else img_thi
    ifcs.append(M.Surface(lbl='Img', interact_mode='dummy', max_aperture=1e3))
    tf = None
    if kind == 'general':
        a = n_ifc//3
        ifcs[a].clear_apertures = [M.Rectangular(AP*0.9, AP*0.8, x_offset=0.3, y_offset=-0.2)]
        tf = []
        for i, g in enumerate(gaps):
            if i in (a + 10, a + 11):                # a tilted, decentered pair and its undoing
                s = 1 if i == a + 10 else -1
                cx, sx = np.cos(0.002*s), np.sin(0.002*s)
                R = np.array([[1.0, 0.0, 0.0], [0.0, cx, -sx], [0.0, sx, cx]])
                rt = R.T if s > 0 else np.ascontiguousarray(R)     # F-ordered view / C array
                tf.append((rt, np.array([0.05*s, -0.03*s, g.thi])))
            else:
                tf.append((np.identity(3), np.array([0., 0., g.thi])))
        tf.append((np.identity(3), np.zeros(3)))
    sm = M.SequentialModel(ifcs, gaps, stop_surface=stop, wvlns=wvls, ref_wvl=n_wvl//2, lcl_tfrms=tf)
    fields = [M.Field(y=0.0), M.Field(y=0.7*FIELD_DEG), M.Field(x=0.2*FIELD_DEG, y=FIELD_DEG)]
    osp = OpticalSpecs(WvlSpec(wvls, n_wvl//2), PupilSpec(('object', 'epd'), EPD),
                       FieldSpec(('object', 'angle'), FIELD_DEG, fields))
    opm = M.OpticalModel(sm, osp, name=name)
    opm.update_model()
    return opm


def long_model(name, n_ifc, n_wvl, kind):
    opm = build(name, n_ifc, n_wvl, kind)
    img = float(opm.optical_spec.fod.img_dist)       # paraxial focus
    opm = build(name, n_ifc, n_wvl, kind, img_thi=img)
    assert opm.seq_model.get_num_surfaces() == n_ifc
    return opm


MODELS = {
    'long640': (640, 5, 'quadric'),
    'long360': (360, 5, 'quadric'),
    'long320': (320, 3, 'poly'),
    'long256': (256, 5, 'general'),
}


def load(name):
    """a fresh model of the fixture ``name``"""
    return long_model(name, *MODELS[name])
