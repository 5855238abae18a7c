#!/usr/bin/env python3
"""Generate the boundary-ray vectors tests/golden/vectors/edges_<fixture>.npz.

Runs only where the reference tree exists, like make_golden.py: every ray is traced by the
reference's own ``trace_raw`` (oracle/ref_harness.py).  The kernels decide clipping, TIR and
misses with shortcuts that must agree with the reference exactly at the decision boundary
(the aperture band of rt_lean.cuh, the sign of the TIR argument, the sign of the discriminant),
and vertex / on-axis rays take special paths (plano shortcut, zero numerators, the r = 0 branch
of the radial polynomial).  Random rays practically never land there, so these rays are made to.

A *bisection family* is a one-parameter set of start rays (start height, start x or relative
pupil coordinate).  A coarse scan finds where the reference's (status, failing surface) changes
to the wanted outcome, bisection narrows that to two adjacent doubles, and K ``nextafter``
neighbours on each side are kept.  An *explicit family* is a fixed list of vertex / tiny-operand
rays.  Per ray the file stores, besides the make_golden.py record (p0, d0, wvl_idx, case, last,
op, status, fail_surf, n_seg, full, cases):

  family [n], step [n]   family index (``families``, JSON) and position relative to the flip
                         (-K..-1 on the first side, 0..K-1 on the second; 0 for explicit rays)
  q [n]                  the deciding quantity in units of its band / ulp (NaN where undefined):
                         aperture  (r**2 - L**2)/L**2 * 2**50, L = max_aperture + fuzz
                         list aperture  (|x - x_off| - (a + fuzz))/ulp(a + fuzz) resp. the same
                                   on sqrt(x**2 + y**2)
                         tir       (n'**2 - n**2 sin**2 I)/ulp(n'**2)
                         miss      (b**2 - a*c)/ulp(b**2) for quadrics, the sag argument
                                   (1 - ec cv**2 r**2)/ulp(1) for polynomials
  field [n], pupil [2, n] field index and relative pupil point of the rays made by
                         ``OpticalSpecs.ray_start_from_osp`` (field -1 otherwise); these rays
                         are traced as paired pupil lists by the grid kernels.

No random numbers: a re-run writes identical files.
"""
import json
import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh                 # noqa: E402
from rayoptics_b200 import model as M                # noqa: E402

OUT = os.path.join(HERE, 'vectors')
K = 16
N_SCAN = 400
BAND = 2.0**50


def cases_for(n_ifc):
    aps = dict(first_surf=1, last_surf=n_ifc - 2, check_apertures=True)
    return [aps, dict(aps, pt_inside_fuzz=1e-3), dict(aps, pt_inside_fuzz=0.0),
            dict(first_surf=1, last_surf=n_ifc - 2, check_apertures=False),
            dict(first_surf=0, last_surf=None, check_apertures=False)]


FUZZ = [1e-5, 1e-3, 0.0]          # pt_inside_fuzz of cases 0, 1, 2 (the reference's default first)
TILT = np.array([0.01, 0.02, 1.0])/np.linalg.norm([0.01, 0.02, 1.0])
AXIS = np.array([0.0, 0.0, 1.0])


def ray_y(x0, d):
    return lambda t: (np.array([x0, t, 0.0]), d.copy())


def ray_x(y0):
    return lambda t: (np.array([t, y0, 0.0]), AXIS.copy())


def ray_diag(ry):
    return lambda t: (np.array([t, ry*t, 0.0]), AXIS.copy())


def ray_pupil(opm, fi):
    osp, sm = opm.optical_spec, opm.seq_model
    fld = osp.field_of_view.fields[fi]

    def make(t):
        pt0, dir0 = osp.ray_start_from_osp(fld.apply_vignetting(np.array([0.0, t])), fld)
        if dir0[2]*sm.z_dir[0] < 0:
            dir0 = -dir0
        return pt0, dir0
    return make


class Tracer:
    def __init__(self, opm):
        self.sm = opm.seq_model
        self.n_ifc = self.sm.get_num_surfaces()
        self.cases = cases_for(self.n_ifc)
        self.wvl = self.sm.wvlns[0]
        self.path = rh.ref_path(self.sm, self.wvl)

    def __call__(self, pt0, dir0, ci):
        return rh.ref_trace(self.path, pt0, dir0, self.wvl, **self.cases[ci])


def flip(tr, make, ci, a, b, want):
    """Adjacent doubles lo < hi where the outcome (status, fail_surf) changes and the pair of
    outcomes is `want` (an unordered pair)."""
    def obs(t):
        r = tr(*make(t), ci)
        return (r['status'], r['fail_surf'])
    ts = np.linspace(a, b, N_SCAN)
    prev = obs(ts[0])
    for t0, t1 in zip(ts[:-1], ts[1:]):
        cur = obs(t1)
        if cur != prev and {prev, cur} == set(want):
            lo, hi, o_lo = float(t0), float(t1), prev
            while True:
                mid = lo + (hi - lo)/2
                if mid <= lo or mid >= hi:
                    return lo, hi
                if obs(mid) == o_lo:
                    lo = mid
                else:
                    hi = mid
        prev = cur
    raise RuntimeError(f'no flip {want} in [{a}, {b}] (case {ci})')


def neighbours(lo, hi):
    below, above = [lo], [hi]
    for _ in range(K - 1):
        below.append(float(np.nextafter(below[-1], -np.inf)))
        above.append(float(np.nextafter(above[-1], np.inf)))
    return below[::-1] + above, list(range(-K, 0)) + list(range(K))


def ulp(x):
    return float(np.spacing(abs(x)))


def q_aperture(sm, surf, fuzz, ray, n_seg):
    if n_seg <= surf:
        return np.nan
    x, y = ray[surf, 0], ray[surf, 1]
    L = sm.ifcs[surf].max_aperture + fuzz
    l2 = L*L
    return (x*x + y*y - l2)/l2*BAND


def q_list(sm, surf, ap, fuzz, ray, n_seg):
    if n_seg <= surf:
        return np.nan
    ca = sm.ifcs[surf].clear_apertures[ap]
    xa, ya = ray[surf, 0] - ca.x_offset, ray[surf, 1] - ca.y_offset
    if type(ca).__name__ == 'Circular':
        T = ca.radius + fuzz
        return (math.sqrt(xa*xa + ya*ya) - T)/ulp(T)
    Tx, Ty = ca.x_half_width + fuzz, ca.y_half_width + fuzz
    dx, dy = (abs(xa) - Tx)/ulp(Tx), (abs(ya) - Ty)/ulp(Ty)
    return dx if abs(dx) < abs(dy) else dy


def q_tir(tr, surf, ray, n_seg):
    if n_seg <= surf:
        return np.nan
    d, nrm = ray[surf - 1, 3:6], ray[surf, 7:10]
    n_in, n_out = tr.path[surf - 1][3], tr.path[surf][3]
    c = (d[0]*nrm[0] + d[1]*nrm[1] + d[2]*nrm[2])/math.sqrt(nrm[0]*nrm[0] + nrm[1]*nrm[1] + nrm[2]*nrm[2])
    arg = n_out*n_out - n_in*n_in*(1.0 - c*c)
    return arg/ulp(n_out*n_out)


def q_miss(tr, surf, ray, n_seg):
    """discriminant (quadrics) / sag argument (polynomials) at the first iterate"""
    if n_seg < surf:
        return np.nan
    p, d = ray[surf - 1, 0:3], ray[surf - 1, 3:6]
    t = tr.path[surf - 1][2][1]
    b4 = p - t
    pp = b4 + (-(b4[0]*d[0] + b4[1]*d[1] + b4[2]*d[2]))*d
    prf = tr.sm.ifcs[surf].profile
    cv = prf.cv
    kind = type(prf).__name__
    if kind == 'Spherical':
        cx2 = cv*(pp[0]*pp[0] + pp[1]*pp[1] + pp[2]*pp[2]) - 2*pp[2]
        b = cv*(d[0]*pp[0] + d[1]*pp[1] + d[2]*pp[2]) - d[2]
        return (b*b - cv*cx2)/ulp(b*b)
    if kind == 'Conic':
        ec = prf.ec
        ax2 = cv*(1. + prf.cc*d[2]*d[2])
        cx2 = cv*(pp[0]*pp[0] + pp[1]*pp[1] + ec*pp[2]*pp[2]) - 2.0*pp[2]
        b = cv*(d[0]*pp[0] + d[1]*pp[1] + ec*d[2]*pp[2]) - d[2]
        return (b*b - ax2*cx2)/ulp(b*b)
    if d[0] != 0.0 or d[1] != 0.0:       # Spencer's iterates move off the start point
        return np.nan
    r2 = pp[0]*pp[0] + pp[1]*pp[1]
    return (1. - prf.ec*cv*cv*r2)/ulp(1.0)


OK, MISS, TIR, BLOCK = 0, 1, 2, 3


def lens_families(opm):
    """Bisection and explicit families of the edge_<profile> lenses (make_models.edge_lens)."""
    sm = opm.seq_model
    fams = []
    for ci in (0, 1, 2):
        fams.append(dict(name=f'aperture_axial_c{ci}', case=ci, make=ray_y(0.0, AXIS), scan=(1.0, 3.0),
                         want=[(OK, -1), (BLOCK, 1)], q=('aperture', 1, FUZZ[ci])))
        fams.append(dict(name=f'aperture_tilted_c{ci}', case=ci, make=ray_y(0.1, TILT), scan=(0.5, 2.5),
                         want=[(OK, -1), (BLOCK, 1)], q=('aperture', 1, FUZZ[ci])))
    fams += [
        dict(name='tir_axial', case=3, make=ray_y(0.0, AXIS), scan=(4.0, 7.8),
             want=[(OK, -1), (TIR, 1)], q=('tir', 1)),
        dict(name='tir_tilted', case=4, make=ray_y(0.1, TILT), scan=(4.0, 7.8),
             want=[(OK, -1), (TIR, 1)], q=('tir', 1)),
        dict(name='miss_axial', case=3, make=ray_y(0.0, AXIS), scan=(6.0, 14.0),
             want=[(TIR, 1), (MISS, 1)], q=('miss', 1)),
        dict(name='miss_tilted', case=4, make=ray_y(0.1, TILT), scan=(6.0, 14.0),
             want=[(TIR, 1), (MISS, 1)], q=('miss', 1)),
    ]
    for fi in range(len(opm.optical_spec.field_of_view.fields)):
        fams += [
            dict(name=f'aperture_pupil_f{fi}', case=0, make=ray_pupil(opm, fi), scan=(0.0, 1.0),
                 want=[(OK, -1), (BLOCK, 1)], q=('aperture', 1, FUZZ[0]), field=fi),
            dict(name=f'tir_pupil_f{fi}', case=3, make=ray_pupil(opm, fi), scan=(0.0, 1.5),
                 want=[(OK, -1), (TIR, 1)], q=('tir', 1), field=fi),
        ]
    # on-axis / vertex rays with signed zeros, and tiny operands next to exact zeros
    z, t = 0.0, 1e-300
    starts = [(z, z), (-z, z), (z, -z), (-z, -z), (t, z), (z, -t), (t, t), (5e-324, z), (0.5, t), (t, 0.5)]
    dirs = [(z, z), (-z, -z), (t, z), (z, -t)]
    rays = [(np.array([x, y, 0.0]), np.array([dx, dy, 1.0])) for x, y in starts for dx, dy in dirs]
    for ci in range(5):
        fams.append(dict(name=f'vertex_c{ci}', case=ci, rays=rays))
    return fams


def stops_families(opm):
    """List-aperture families of edge_stops: each edge of the rectangle (offset), the offset
    circle and the offset obscuration, crossed by rays parallel to the axis."""
    fams = []
    for ci in (0, 1, 2):
        fams += [
            dict(name=f'rect_x_c{ci}', case=ci, make=ray_x(0.0), scan=(4.0, 6.0),
                 want=[(BLOCK, 2), (BLOCK, 1)], q=('list', 1, 0, FUZZ[ci])),
            dict(name=f'rect_y_c{ci}', case=ci, make=ray_y(0.0, AXIS), scan=(-5.5, -3.5),
                 want=[(BLOCK, 1), (BLOCK, 2)], q=('list', 1, 0, FUZZ[ci])),
            dict(name=f'circle_y_c{ci}', case=ci, make=ray_y(0.3, AXIS), scan=(2.0, 4.0),
                 want=[(OK, -1), (BLOCK, 2)], q=('list', 2, 0, FUZZ[ci])),
            dict(name=f'circle_diag_c{ci}', case=ci, make=ray_diag(0.75), scan=(-4.0, -1.5),
                 want=[(BLOCK, 2), (OK, -1)], q=('list', 2, 0, FUZZ[ci])),
            dict(name=f'obscuration_x_c{ci}', case=ci, make=ray_x(0.1), scan=(0.0, 1.5),
                 want=[(BLOCK, 2), (OK, -1)], q=('list', 2, 1, FUZZ[ci])),
        ]
    for fi in range(len(opm.optical_spec.field_of_view.fields)):
        fams.append(dict(name=f'circle_pupil_f{fi}', case=0, make=ray_pupil(opm, fi), scan=(0.5, 1.5),
                         want=[(OK, -1), (BLOCK, 2)], q=('list', 2, 0, FUZZ[0]), field=fi))
    return fams


def quantity(tr, spec, r):
    kind, surf = spec[0], spec[1]
    ray, n_seg = r['ray'], r['n_seg']
    if kind == 'aperture':
        return q_aperture(tr.sm, surf, spec[2], ray, n_seg)
    if kind == 'list':
        return q_list(tr.sm, surf, spec[2], spec[3], ray, n_seg)
    if kind == 'tir':
        return q_tir(tr, surf, ray, n_seg)
    return q_miss(tr, surf, ray, n_seg)


def build(name):
    opm = M.OpticalModel.load(os.path.join(HERE, 'models', name + '.json'))
    tr = Tracer(opm)
    fams = stops_families(opm) if name == 'edge_stops' else lens_families(opm)
    rays, meta = [], []
    for fid, f in enumerate(fams):
        if 'rays' in f:
            for p0, d0 in f['rays']:
                rays.append((p0, d0, f['case'], fid, 0, None, -1, (np.nan, np.nan)))
            continue
        lo, hi = flip(tr, f['make'], f['case'], *f['scan'], f['want'])
        ts, steps = neighbours(lo, hi)
        for t, s in zip(ts, steps):
            p0, d0 = f['make'](t)
            fi = f.get('field', -1)
            rays.append((p0, d0, f['case'], fid, s, f['q'], fi, (0.0, t) if fi >= 0 else (np.nan, np.nan)))
    n, n_ifc = len(rays), tr.n_ifc
    out = dict(p0=np.zeros((3, n)), d0=np.zeros((3, n)), wvl_idx=np.zeros(n, np.int32),
               case=np.zeros(n, np.int32), last=np.zeros((10, n)), op=np.zeros(n),
               status=np.zeros(n, np.int32), fail_surf=np.zeros(n, np.int32),
               n_seg=np.zeros(n, np.int32), full=np.full((n_ifc, 10, n), np.nan),
               family=np.zeros(n, np.int32), step=np.zeros(n, np.int32), q=np.full(n, np.nan),
               field=np.zeros(n, np.int32), pupil=np.zeros((2, n)))
    for k, (p0, d0, ci, fid, s, qs, fi, pup) in enumerate(rays):
        r = tr(p0, d0, ci)
        out['p0'][:, k], out['d0'][:, k], out['case'][k] = p0, d0, ci
        out['op'][k], out['status'][k] = r['op'], r['status']
        out['fail_surf'][k], out['n_seg'][k] = r['fail_surf'], r['n_seg']
        if r['n_seg'] > 0:
            out['last'][:, k] = r['ray'][-1]
        out['full'][:r['n_seg'], :, k] = r['ray']
        out['family'][k], out['step'][k], out['field'][k] = fid, s, fi
        out['pupil'][:, k] = pup
        if qs is not None:
            out['q'][k] = quantity(tr, qs, r)
    out['cases'] = np.array(json.dumps(tr.cases))
    out['families'] = np.array(json.dumps([{'name': f['name'], 'case': f['case'],
                                             'bisected': 'rays' not in f,
                                             'quantity': f['q'][0] if 'q' in f else None}
                                            for f in fams]))
    return out, fams


def main():
    names = sys.argv[1:] or ['edge_sphere', 'edge_conic', 'edge_even', 'edge_radial', 'edge_stops']
    for name in names:
        out, fams = build(name)
        np.savez_compressed(os.path.join(OUT, 'edges_' + name + '.npz'), **out)
        print(f'{name}: {out["status"].size} rays, status hist '
              f'{np.bincount(out["status"], minlength=6).tolist()}')
        for fid, f in enumerate(fams):
            sel = out['family'] == fid
            q = out['q'][sel]
            fin = q[np.isfinite(q)]
            print(f'  {f["name"]:22s} outcomes={sorted(set(zip(out["status"][sel], out["fail_surf"][sel])))} '
                  f'q in band={int((np.abs(fin) < 1).sum())} q==0: {int((fin == 0).sum())} '
                  f'q range=[{fin.min() if fin.size else np.nan:.3g}, {fin.max() if fin.size else np.nan:.3g}]')


if __name__ == '__main__':
    main()
