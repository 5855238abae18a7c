"""GPU (H100): the CUDA kernels on the boundary rays of tests/golden/vectors/edges_*.npz (see
tests/test_edges.py and tests/golden/make_golden_edges.py), bit for bit against the reference's
own results.  Bundle launches run every eligible kernel -- lean or lean-poly, and the general
kernel forced with B200RT_NO_LEAN -- with last-segment-only and whole-ray outputs; grid launches
run the paired pupil lists that were bisected through ray_start_from_osp."""
import numpy as np
import pytest
import torch

from conftest import load_model
from test_edges import EDGE_NAMES, assert_bits, by_case, compare, load_edges, paired_specs
from rayoptics_b200 import _abi, engine as E, table as T

pytestmark = pytest.mark.gpu

LAST_ONLY = ('p', 'd', 'op', 'status', 'fail_surf', 'n_seg')


def np_(t):
    return t.detach().cpu().numpy()


def make_table(name, general, monkeypatch):
    if general:
        monkeypatch.setenv('B200RT_NO_LEAN', '1')
    tab = T.SurfaceTable.from_model(load_model(name).seq_model, device=0)
    monkeypatch.delenv('B200RT_NO_LEAN', raising=False)
    return tab


def records(r):
    n = r.status.shape[0]
    zero = np.zeros(n)
    dst = np_(r.dst)[None] if r.dst is not None else zero[None]
    nrml = np_(r.nrml) if r.nrml is not None else np.zeros((3, n))
    return {'status': np_(r.status), 'fail_surf': np_(r.fail_surf), 'n_seg': np_(r.n_seg),
            'op': np_(r.op), 'last': np.concatenate([np_(r.p), np_(r.d), dst, nrml]),
            'full': np_(r.full) if r.full is not None else None}


@pytest.mark.parametrize('general', [False, True], ids=['eligible', 'general'])
@pytest.mark.parametrize('name', EDGE_NAMES)
def test_cuda_bundles_match_edge_vectors(name, general, monkeypatch):
    tab = make_table(name, general, monkeypatch)
    v = load_edges(name)
    for ci, case, idx in by_case(v):
        args = (tab, v['p0'][:, idx], v['d0'][:, idx])
        r2 = E.trace_bundle(*args, wvl_idx=v['wvl_idx'][idx], full=True, **case)
        r1 = E.trace_bundle(*args, wvl_idx=v['wvl_idx'][idx], full=False, **case)
        r0 = E.trace_bundle(*args, wvl_idx=v['wvl_idx'][idx], outputs=LAST_ONLY, **case)
        torch.cuda.synchronize()
        for out_kind, r in ((2, r2), (1, r1), (0, r0)):
            compare(records(r), v, idx, out_kind, f'out {out_kind} case {ci}')


@pytest.mark.parametrize('general', [False, True], ids=['eligible', 'general'])
@pytest.mark.parametrize('name', EDGE_NAMES)
def test_cuda_paired_grids_match_edge_vectors(oracle, name, general, monkeypatch):
    """status, failing surface, p, d, op and transverse aberration of the paired pupil lists ==
    the reference (records) and the oracle (abr); NaN-coded status decodes to the same; the
    summary counts are the status histogram."""
    tab = make_table(name, general, monkeypatch)
    v = load_edges(name)
    n_lists = 0
    for fid, grid, idx in paired_specs(name, v, cls=E.PupilGrid, device=0):
        case = v['cases'][int(v['case'][idx[0]])]
        what = f'grid, family {v["families"][fid]["name"]}'
        r = E.trace_grid(tab, grid, **case)
        rn = E.trace_grid(tab, grid, outputs=('abr',), nan_status=True, **case)
        torch.cuda.synchronize()
        st = np_(r.status)
        compare({'status': st, 'fail_surf': np_(r.fail_surf), 'op': np_(r.op),
                 'last': np.concatenate([np_(r.p), np_(r.d), np.zeros((4, st.size))])}, v, idx, 0, what)
        ref = oracle.trace_grid(grid.c_spec(), tab.descs, tab.n_by_wvl, 0, grid.n_rays,
                                _abi.make_opts(**case), wvls=tab.wvls)
        abr = np_(r.abr)
        assert_bits(abr, ref['abr'], what + ' abr')
        nst, nfs = E.decode_nan_status(np_(rn.abr))
        assert_bits(nst, v['status'][idx], what + ' NaN-coded status')
        assert_bits(nfs, np.where(st == 0, -1, v['fail_surf'][idx]), what + ' NaN-coded fail_surf')
        ok = st == 0
        assert_bits(np_(rn.abr)[:, ok], abr[:, ok], what + ' abr (NaN-coded launch)')
        summ = np_(r.summary)
        assert summ.shape[0] == 1
        for k in range(5):
            assert summ[0, k] == (st == k).sum(), (what, k)
        assert len(set(st.tolist())) == 2
        n_lists += 1
    assert n_lists >= 2
