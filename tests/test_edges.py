"""Rays placed exactly at the decision boundaries of the trace (tests/golden/make_golden_edges.py):
the aperture band of the lean kernels, the sign of the TIR argument, the sign of the
discriminant, vertex / on-axis hits with signed zeros, tiny operands next to exact zeros and the
edges of aperture lists.  The reference's own results on these rays must be reproduced bit for
bit -- signed zeros included -- by the C oracle and by the device source compiled for the host
(general loop, lean and lean-poly loops, every output kind).  Random rays essentially never land
in these places, so the vectors also assert that they do land there."""
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN, load_model
from rayoptics_b200 import _abi, engine as E, table as T
from hostsim import build as HS

EDGE_NAMES = ['edge_sphere', 'edge_conic', 'edge_even', 'edge_radial', 'edge_stops']
LEAN_KIND = {'edge_sphere': 1, 'edge_conic': 1, 'edge_even': 2, 'edge_radial': 2, 'edge_stops': 0}


def load_edges(name):
    z = np.load(os.path.join(GOLDEN, 'vectors', 'edges_' + name + '.npz'))
    v = {k: z[k] for k in z.files}
    v['cases'] = json.loads(str(v['cases']))
    v['families'] = json.loads(str(v['families']))
    return v


def bits(a):
    """uint64 view with every NaN mapped to one pattern: NaNs compare by NaN-ness only"""
    a = np.ascontiguousarray(a, dtype=np.float64)
    b = a.view(np.uint64).copy()
    b[np.isnan(a)] = np.uint64(0x7FF8000000000000)
    return b


def signed_zero_rays(p0, d0):
    """The one known difference, in the sign of zero only.  The reference moves every ray into
    the next interface's coordinates with ``rt.dot(p - t)`` and ``rt.dot(d)`` even when ``rt`` is
    the identity; its sums 1*x + 0*y + 0*z turn x = -0.0 into +0.0.  The kernels and the oracle
    skip identity rotations (``has_tfrm == 0``), so a ray that starts on the axis with -0.0 in
    the same component of both start point and direction keeps -0.0 in the points, directions
    and normals along its path.  Values are otherwise identical."""
    nz = lambda a: (a == 0) & np.signbit(a)     # noqa: E731
    return (nz(p0[0]) & nz(d0[0])) | (nz(p0[1]) & nz(d0[1]))


def assert_bits(got, ref, what, zero_ok=None):
    """bitwise equality; `zero_ok` [n]: rays (last axis) allowed to differ in the sign of zero"""
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape, what
    if got.dtype.kind == 'f':
        diff = bits(got) != bits(ref)
        if zero_ok is not None:
            diff &= ~(zero_ok & (got == 0) & (ref == 0))
        if diff.any():
            k = np.argwhere(diff)[0]
            sign_only = np.array_equal(got, ref, equal_nan=True)
            pytest.fail(f'{what}: {int(diff.sum())} values differ{" only in the sign of zero" if sign_only else ""}, '
                        f'first at {k.tolist()}: {got[tuple(k)]!r} vs {ref[tuple(k)]!r}')
    else:
        assert np.array_equal(got, ref), what


def compare(r, v, idx, out_kind, what):
    """out_kind: 0 = last p, d; 1 = + dst, normal; 2 = + whole rays"""
    st = v['status'][idx]
    zero_ok = signed_zero_rays(v['p0'][:, idx], v['d0'][:, idx])
    assert_bits(r['status'], st, what + ' status')
    assert_bits(r['fail_surf'], np.where(st == 0, -1, v['fail_surf'][idx]), what + ' fail_surf')
    if r.get('n_seg') is not None:
        assert_bits(r['n_seg'], v['n_seg'][idx], what + ' n_seg')
    assert_bits(r['op'], v['op'][idx], what + ' op')
    assert_bits(r['last'][0:6], v['last'][0:6, idx], what + ' last p, d', zero_ok)
    if out_kind >= 1:
        assert_bits(r['last'][6:10], v['last'][6:10, idx], what + ' last dst, normal', zero_ok)
    if out_kind == 2:
        assert_bits(r['full'], v['full'][:, :, idx], what + ' full', zero_ok)


def by_case(v):
    for ci, case in enumerate(v['cases']):
        idx = np.nonzero(v['case'] == ci)[0]
        if idx.size:
            yield ci, case, idx


@pytest.fixture(scope='module')
def hostsim():
    HS.lib()
    return HS


@pytest.mark.parametrize('name', EDGE_NAMES)
def test_oracle_matches_edge_vectors(oracle, name):
    descs, n_by_wvl, wvls = T.describe_model(load_model(name).seq_model)
    v = load_edges(name)
    for ci, case, idx in by_case(v):
        r = oracle.trace_bundle(descs, n_by_wvl, v['p0'][:, idx], v['d0'][:, idx], v['wvl_idx'][idx],
                                _abi.make_opts(**case), want_full=True, wvls=wvls)
        compare(r, v, idx, 2, f'oracle case {ci}')


@pytest.mark.parametrize('name', EDGE_NAMES)
def test_device_source_matches_edge_vectors(hostsim, name):
    """general loop (kernel 0) and the lean loops; the lean-poly instance also runs the
    quadric-only tables, on which its quadric branch is the same code as the lean one's"""
    descs, n_by_wvl, wvls = T.describe_model(load_model(name).seq_model)
    kind = HS.lean_kind(descs)
    assert kind == LEAN_KIND[name]
    kernels = {0: [0], 1: [0, 1, 2], 2: [0, 2]}[kind]
    v = load_edges(name)
    for ci, case, idx in by_case(v):
        opts = _abi.make_opts(**case)
        for kern in kernels:
            for out_kind in (0, 1, 2):
                r = hostsim.trace_bundle(descs, n_by_wvl, v['p0'][:, idx], v['d0'][:, idx],
                                         v['wvl_idx'][idx], opts, kernel=kern, out_kind=out_kind, wvls=wvls)
                compare(r, v, idx, 1 if kern == 0 and out_kind < 2 else out_kind,
                        f'kernel {kern} out {out_kind} case {ci}')


def paired_specs(name, v, cls=E.PupilGridSpec, **kwargs):
    """(family index, grid of its pupil list as ONE paired tile, ray indices) for every family
    made by ray_start_from_osp; `cls`: PupilGridSpec or PupilGrid (kwargs: device)"""
    opm = load_model(name)
    osp, sm = opm.optical_spec, opm.seq_model
    for fid in np.unique(v['family'][v['field'] >= 0]):
        idx = np.nonzero(v['family'] == fid)[0]
        fi = int(v['field'][idx[0]])
        assert (v['field'][idx] == fi).all() and (v['case'][idx] == v['case'][idx[0]]).all()
        recs, eprad, z_pupil = osp.grid_fields([osp.field_of_view.fields[fi]])
        spec = cls(recs, [0], v['pupil'][0, idx], v['pupil'][1, idx], eprad, z_pupil,
                   flip_z_dir=sm.z_dir[0], paired=True, **kwargs)
        yield int(fid), spec, idx


@pytest.mark.parametrize('name', EDGE_NAMES)
def test_paired_pupil_lists_match_edge_vectors(hostsim, oracle, name):
    """The grid start rays of the paired pupil lists are the stored start rays (both instances of
    grid_start_ray and the oracle), and the oracle's grid trace gives the stored records."""
    descs, n_by_wvl, wvls = T.describe_model(load_model(name).seq_model)
    v = load_edges(name)
    n_lists = 0
    for fid, spec, idx in paired_specs(name, v):
        cs = spec.c_spec()
        p, d, _, _ = oracle.grid_start_rays(cs, 0, spec.n_rays)
        assert_bits(p, v['p0'][:, idx], 'oracle start p')
        assert_bits(d, v['d0'][:, idx], 'oracle start d')
        for lean in (False, True):
            pg, dg = hostsim.grid_start_rays(cs, 0, spec.n_rays, lean=lean)
            assert_bits(pg, v['p0'][:, idx], f'grid_start_ray(lean={lean}) p')
            assert_bits(dg, v['d0'][:, idx], f'grid_start_ray(lean={lean}) d')
        case = v['cases'][int(v['case'][idx[0]])]
        r = oracle.trace_grid(cs, descs, n_by_wvl, 0, spec.n_rays, _abi.make_opts(**case), wvls=wvls)
        compare(r, v, idx, 1, f'oracle grid, family {v["families"][fid]["name"]}')
        n_lists += 1
    assert n_lists >= 2


@pytest.mark.parametrize('name', EDGE_NAMES)
def test_edge_vectors_cover_the_boundaries(name):
    """Every bisected family straddles its flip with rays that are decided within a few ulps of
    the boundary (inside the 2**-50 band for the aperture test), and both outcomes appear."""
    v = load_edges(name)
    fams = v['families']
    assert len(fams) == v['family'].max() + 1
    for fid, f in enumerate(fams):
        sel = v['family'] == fid
        out = set(zip(v['status'][sel].tolist(), v['fail_surf'][sel].tolist()))
        if not f['bisected']:
            continue
        assert len(out) == 2, f['name']
        step = v['step'][sel]
        pair = [(int(v['status'][sel][step == s][0]), int(v['fail_surf'][sel][step == s][0])) for s in (-1, 0)]
        assert pair[0] != pair[1], f['name']
        q = v['q'][sel]
        if f['quantity'] is None or not np.isfinite(q).any():
            continue
        if f['quantity'] == 'aperture':
            band = np.abs(q) < 1
            assert ((q > -1) & (q <= 0)).any() and ((q > 0) & (q < 1)).any(), f['name']
            assert len(set(v['status'][sel][band].tolist())) == 2, f['name']
        else:
            assert np.nanmin(np.abs(q[step < 0])) <= 4 and np.nanmin(np.abs(q[step >= 0])) <= 4, f['name']
    # exact cancellations: r**2 == L**2, n'**2 - n**2 sin**2 I == 0, b**2 - a*c == 0,
    # |x - x_off| == a + fuzz ...
    kinds = {f['quantity'] for fid, f in enumerate(fams) if (v['q'][v['family'] == fid] == 0).any()}
    assert kinds >= ({'list'} if name == 'edge_stops' else {'aperture', 'tir'} | ({'miss'} if name == 'edge_sphere' else set()))


@pytest.mark.parametrize('name', [n for n in EDGE_NAMES if n != 'edge_stops'])
def test_edge_vectors_hit_vertices_with_signed_zeros(name):
    v = load_edges(name)
    vert = np.isin(v['family'], [i for i, f in enumerate(v['families']) if f['name'].startswith('vertex')])
    full = v['full'][:, :, vert]
    on_axis = (full[1:3, 0, :] == 0).all(0) & (full[1:3, 1, :] == 0).all(0)
    assert on_axis.sum() >= 20
    assert (np.signbit(v['p0'][0:2, vert]) & np.signbit(v['d0'][0:2, vert])).any()
    assert np.signbit(full[1:3, 7:9][:, :, on_axis]).any()          # normals (-cv*0, ...)
    tiny = (np.abs(v['p0'][0:2, vert]) < 1e-290) & (v['p0'][0:2, vert] != 0)
    assert tiny.any()
