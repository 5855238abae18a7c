"""Long systems (tests/long_models.py): surface tables that fill or overflow the
shared-memory budget of rt_table_create (csrc/b200rt.cu).

rt_table_create picks, from the table's size in bytes, how every later launch is made: the lean
kernels when their plan fits the budget RT_MAX_STAGE_BYTES - RT_ACC_BYTES (and the system has no
transforms, aperture lists or phase elements), else the general kernels with the table staged in
shared memory when it fits, else the general kernels reading the table from global memory.
``plan`` restates that choice from the struct sizes of a host compile of the headers and the
constants of the source text, and the fixtures are asserted to sit where they are meant to:
exactly at a budget, one wavelength row over it, or in the middle (long360).

The host-compiled per-ray loops (tests/hostsim) are held to the oracle bit for bit on these
tables, and the oracle to the reference's own trace_raw where the reference tree is present."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import long_models as LM
from conftest import ROOT, seeded_bundle
from rayoptics_b200 import _abi, table as T
from hostsim import build as HS
from test_hostsim import compare

SRC = os.path.join(ROOT, 'rayoptics_b200', 'csrc', 'b200rt.cu')
HOSTSIM = os.path.join(ROOT, 'tests', 'hostsim')
SIZES_LIB = os.path.join(HOSTSIM, '_build', 'libhostsim_sizes.so')
LONG_MODELS = ['long640', 'long360', 'long320', 'long256']

# (fixture, extra wavelength rows, regime, where the table sits)
PLACEMENTS = [
    ('long640', 0, 'lean', 'at'),             # lean quadric plan == budget
    ('long640', 1, 'unstaged', 'over'),       # one row more: neither plan fits
    ('long360', 0, 'lean', 'mid'),            # 97 920 B: one summary CTA per SM, two of the rest
    ('long320', 0, 'lean_poly', 'at'),        # lean POLY plan == budget
    ('long320', 1, 'unstaged', 'over'),
    ('long256', 0, 'staged', 'at'),           # general staged table == budget
    ('long256', 1, 'unstaged', 'over'),
]


def struct_sizes():
    """sizeof(rt_surface_desc), sizeof(LeanSurf), sizeof(LeanIdx), sizeof(LeanPoly) from a host
    compile of the headers (tests/hostsim/sizes.cpp, the flags of hostsim/build.py)"""
    srcs = [os.path.join(HOSTSIM, 'sizes.cpp'), os.path.join(HOSTSIM, 'cuda_runtime.h'),
            os.path.join(ROOT, 'include', 'b200rt.h')] + \
        [os.path.join(ROOT, 'rayoptics_b200', 'csrc', h) for h in ('rt_lean.cuh', 'rt_device.cuh')]
    os.makedirs(os.path.dirname(SIZES_LIB), exist_ok=True)
    if not os.path.exists(SIZES_LIB) or any(os.path.getmtime(s) > os.path.getmtime(SIZES_LIB) for s in srcs):
        subprocess.check_call(['g++', '-O2', '-std=c++17', '-DRT_HOSTSIM', '-fPIC', '-shared', '-I', HOSTSIM,
                               '-o', SIZES_LIB, srcs[0]])
    out = (C.c_int64*4)()
    assert C.CDLL(SIZES_LIB).hostsim_struct_sizes(out) == 0
    return dict(zip(('desc', 'lean_surf', 'lean_idx', 'lean_poly'), list(out)))


def source_constants():
    """RT_MAX_STAGE_BYTES, RT_BLOCK, RT_ACC and RT_ACC_BYTES as csrc/b200rt.cu defines them"""
    text = open(SRC).read()

    def define(name):
        m = re.search(r'^#define\s+' + name + r'\s+(\S+)', text, re.M)
        assert m, name
        assert re.fullmatch(r'[0-9()*+ ]+', m.group(1)), m.group(1)
        return int(eval(m.group(1)))
    assert re.search(r'^#define\s+RT_ACC_BYTES\s+\(RT_ACC\*RT_BLOCK\*sizeof\(double\)\)', text, re.M)
    k = dict(stage=define('RT_MAX_STAGE_BYTES'), block=define('RT_BLOCK'), acc=define('RT_ACC'))
    k['acc_bytes'] = k['acc']*k['block']*8
    k['budget'] = k['stage'] - k['acc_bytes']
    return k


def plan(descs, n_wvl, sizes=None, consts=None):
    """rt_table_create's choice for a table of ``descs`` with ``n_wvl`` index rows"""
    sz = sizes or struct_sizes()
    k = consts or source_constants()
    n = len(descs)
    stage_bytes = n*sz['desc'] + n*n_wvl*8
    lean_bytes = n*sz['lean_surf'] + n*n_wvl*sz['lean_idx']
    kind = HS.lean_kind(descs)                      # 0: general only, 1: lean, 2: lean POLY
    if kind == 2:
        lean_bytes += n*sz['lean_poly']
    lean = kind != 0 and lean_bytes <= k['budget']
    stage = stage_bytes <= k['budget']
    regime = ('lean_poly' if kind == 2 else 'lean') if lean else ('staged' if stage else 'unstaged')
    return dict(regime=regime, stage_bytes=stage_bytes, lean_bytes=lean_bytes, kind=kind,
                budget=k['budget'], acc_bytes=k['acc_bytes'],
                plan_bytes=lean_bytes if lean else (stage_bytes if stage else 0))


def table_args(name, extra_rows=0):
    """(model, descs, n_by_wvl, wvls) of a fixture, with ``extra_rows`` more index rows (the
    model's first wavelengths once more)"""
    opm = LM.load(name)
    wvls = list(opm.seq_model.wvlns) + list(opm.seq_model.wvlns[:extra_rows])
    descs, n_by_wvl, wvls = T.describe_model(opm.seq_model, wvls)
    return opm, descs, n_by_wvl, wvls


def test_struct_sizes_and_budget():
    """the sizes DESIGN.md §4 states, and the budget the fixtures were sized for"""
    assert struct_sizes() == dict(desc=640, lean_surf=112, lean_idx=32, lean_poly=336)
    k = source_constants()
    assert (k['stage'], k['acc_bytes'], k['budget']) == (204800, 30720, 174080)


@pytest.mark.parametrize('name,extra,regime,where', PLACEMENTS)
def test_fixture_sits_on_its_budget(name, extra, regime, where):
    opm, descs, n_by_wvl, wvls = table_args(name, extra)
    p = plan(descs, len(wvls))
    assert p['regime'] == regime, p
    budget = p['budget']
    if where == 'at':
        assert p['plan_bytes'] == budget, p
    elif where == 'over':
        assert p['stage_bytes'] > budget and (p['kind'] == 0 or p['lean_bytes'] > budget), p
        # the same model one row shorter sits exactly on a budget
        q = plan(descs, len(wvls) - 1)
        assert q['plan_bytes'] == budget and q['regime'] != 'unstaged', q
    else:
        # on an H100 (228 KB of shared memory per SM, 1 KB reserved per CTA; the GPU tests read both
        # from the device): one summary CTA per SM, two of the focus, wfe and bundle kernels
        smem_sm, reserved = 228*1024, 1024
        assert p['lean_bytes'] == 97920, p
        assert smem_sm//(p['lean_bytes'] + p['acc_bytes'] + reserved) == 1
        assert smem_sm//(p['lean_bytes'] + reserved) == 2


def test_fixture_shapes():
    """what the fixtures promise: interfaces, wavelengths, one aperture list and both transform
    layouts in the general one, no phase elements, a stop in the middle"""
    want = {'long640': (640, 5, 1), 'long360': (360, 5, 1), 'long320': (320, 3, 2), 'long256': (256, 5, 0)}
    for name, (n, w, kind) in want.items():
        opm = LM.load(name)
        descs, n_by_wvl, wvls = T.describe_model(opm.seq_model)
        assert (len(descs), len(wvls), HS.lean_kind(descs)) == (n, w, kind), name
        assert all(d.phase_kind == 0 and d.profile != 6 for d in descs)
        assert abs(opm.seq_model.stop_surface - n//2) <= 2
        assert opm.optical_spec.pupil.key[1] == 'epd' and len(opm.optical_spec.fov.fields) == 3
        if name == 'long256':
            assert {d.has_tfrm for d in descs} == {0, 1, 2}
            assert sum(d.n_apertures for d in descs) == 1
        if name == 'long320':
            assert {d.profile for d in descs} >= {2, 3}


@pytest.fixture(scope='module')
def hostsim():
    HS.lib()
    return HS


def option_cases(n_ifc):
    return (dict(first_surf=1, last_surf=n_ifc - 2, check_apertures=True),
            dict(first_surf=2, last_surf=n_ifc - 3, check_apertures=False, filter_out_phantoms=True,
                 intersect_obj=False))


@pytest.mark.parametrize('name', LONG_MODELS)
def test_host_loops_match_the_oracle(hostsim, oracle, name):
    """general, lean and lean POLY loops of the device source == oracle, bit for bit, for every
    output kind; the seeded rays reach the image, are clipped (status 3) and miss or are totally
    reflected at the steep meniscus"""
    opm, descs, n_by_wvl, wvls = table_args(name)
    n_ifc = len(descs)
    p0, d0, wv = seeded_bundle(opm, 400, np.random.default_rng(23))
    kind = HS.lean_kind(descs)
    seen = set()
    for case in option_cases(n_ifc):
        opts = _abi.make_opts(**case)
        ref = oracle.trace_bundle(descs, n_by_wvl, p0, d0, wv, opts, want_full=True, n_threads=4, wvls=wvls)
        seen |= set(np.unique(ref['status']).tolist())
        for kern in ([0] if kind == 0 else [0, kind]):
            for out_kind in ((2,) if kern == 0 else (0, 1, 2)):
                r = hostsim.trace_bundle(descs, n_by_wvl, p0, d0, wv, opts, kernel=kern, out_kind=out_kind,
                                         wvls=wvls)
                compare(r, ref, out_kind)
    assert {0, 3} <= seen and seen & {1, 2}, seen


@pytest.mark.parametrize('name', LONG_MODELS)
def test_oracle_against_reference_trace_raw(oracle, name):
    """the oracle == the reference's trace_raw on ~200 seeded rays per fixture"""
    from oracle import ref_harness as rh
    if not rh.available():
        pytest.skip('the reference tree is not present')
    opm = LM.load(name)
    sm = opm.seq_model
    n_ifc = sm.get_num_surfaces()
    kw = dict(first_surf=1, last_surf=n_ifc - 2, check_apertures=True)
    opts = _abi.make_opts(**kw)
    p0, d0, wv = seeded_bundle(opm, 200, np.random.default_rng(29))
    statuses = set()
    for wi, wvl in enumerate(sm.wvlns):
        idx = np.nonzero(wv == wi)[0]
        path = rh.ref_path(sm, wvl)
        descs, ns = T.describe_path(sm.path(wvl))
        for k in idx:
            a = rh.ref_trace(path, p0[:, k], d0[:, k], wvl, **kw)
            b = oracle.trace_ray(descs, ns, p0[:, k], d0[:, k], opts)
            assert a['status'] == b['status'], (name, k)
            assert a['n_seg'] == b['n_seg'], (name, k)
            assert np.array_equal(a['ray'], b['ray'], equal_nan=True), (name, k)
            assert a['op'] == b['op'] or (np.isnan(a['op']) and np.isnan(b['op'])), (name, k)
            statuses.add(int(a['status']))
    assert 0 in statuses and len(statuses) > 1, statuses
