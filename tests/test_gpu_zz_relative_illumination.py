"""GPU: rt_grid_illumination against engine.illumination_sums_host fed the launch's own status and
directions, on the fixtures of test_gpu_zz_mtf.py; analyses.relative_illumination on the device against
its backend= route; launches, argument errors and repeatability across streams."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import PHASE_MODEL_NAMES, load_model
from rayoptics_b200 import _abi, engine as E, analyses as A
from rayoptics_b200.table import SurfaceTable
from test_gpu_zz_mtf import NAMES
from test_relative_illumination import IllumBackend

pytestmark = pytest.mark.gpu


def bits(v):
    """the bits of v, every NaN as numpy's (a used ray with a NaN direction, as diffractive_wild has, makes
    its tile's sums NaN; the device and numpy give that NaN different signs)"""
    v = np.asarray(v, dtype=np.float64)
    return np.ascontiguousarray(np.where(np.isnan(v), np.nan, v)).view(np.uint64).tolist()


def setup(name, n):
    opm = load_model(name)
    tab = SurfaceTable.from_model(opm.seq_model, device=0)
    grid = E.grid_for_model(opm, tab, n, pupil_range=(-1.0, 1.0), apply_vignetting=False, ref_img=None)
    return opm, tab, grid


def launch(tab, grid):
    res = E.BundleResult(grid.n_rays, tab.n_ifc, torch.device('cuda', 0), ('d', 'status'))
    rec = E.trace_grid_illumination(tab, grid, res=res)
    return rec.cpu().numpy(), res.status.cpu().numpy(), res.d.cpu().numpy()


@pytest.mark.parametrize('n', [2, 33, 64, 256, 1024])
@pytest.mark.parametrize('name', NAMES)
def test_record_equals_the_restatement(name, n):
    opm, tab, grid = setup(name, n)
    rec, status, d = launch(tab, grid)
    per = n*n
    for t in range(grid.n_tiles):
        f = t//grid.n_wvls
        sl = slice(t*per, (t + 1)*per)
        want = E.illumination_sums_host(status[sl].reshape(n, n), d[0, sl].reshape(n, n), d[1, sl].reshape(n, n),
                                        grid.pupil_x[f], grid.pupil_y[f])
        assert bits(rec[t]) == bits(want), (name, n, t)
    grid.close()


@pytest.mark.parametrize('name', [m for m in NAMES if m not in PHASE_MODEL_NAMES])
def test_device_equals_the_backend_route(name):
    opm = load_model(name)
    dev = A.relative_illumination(opm, 48)
    cpu = A.relative_illumination(opm, 48, backend=IllumBackend(opm))
    for k in ('record', 'ri', 'omega', 'f_number', 'fold', 'ri_poly', 'cra', 'chief_img', 'chief_dir'):
        assert bits(getattr(dev, k)) == bits(getattr(cpu, k)), k


def test_launches():
    opm, tab, grid = setup('dblgauss', 32)
    E.trace_grid_illumination(tab, grid)
    torch.cuda.synchronize()
    n0 = E.launch_count()
    E.trace_grid_illumination(tab, grid)                 # the trace and the sums
    assert E.launch_count() - n0 == 2
    n0 = E.launch_count()
    A.relative_illumination(opm, 32)                     # and the chief rays
    assert E.launch_count() - n0 == 3
    n0 = E.launch_count()
    A.relative_illumination(opm, 32, num_fields=4)       # and the aiming
    assert E.launch_count() - n0 == 4
    grid.close()


def test_bad_arguments_launch_nothing():
    lib = _abi.load_library()
    opm, tab, grid = setup('dblgauss', 8)
    dev = torch.device('cuda', 0)
    args, kw = E._grid_args(opm, tab.wvl_index, 8, None, None, None, (-1.0, 1.0), False)
    vign = E.PupilGrid(*args, device=0, **dict(kw, apply_vignetting=True))
    paired = E.PupilGrid(*args, device=0, **dict(kw, paired=True))
    rect = E.PupilGrid(args[0], args[1], args[2], args[3][:7], *args[4:], device=0, **kw)
    one = E.PupilGrid(args[0], args[1], args[2][:1], args[3][:1], *args[4:], device=0, **kw)
    big_px = E.accumulated_steps(-1.0, 1.0, 1025)
    big = E.PupilGrid(args[0], args[1], big_px, big_px, *args[4:], device=0, **kw)
    n = grid.n_rays
    st = torch.zeros(n, dtype=torch.int32, device=dev)
    L = torch.zeros(n, dtype=torch.float64, device=dev)
    rec = torch.zeros((grid.n_tiles, _abi.RT_ILLUM_DOUBLES), dtype=torch.float64, device=dev)
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())     # noqa: E731
    n0 = E.launch_count()
    for g, msg in ((vign, 'vignett'), (paired, 'product grid'), (rect, 'nx = ny'), (one, 'RT_ILLUM_MAX_RAYS'),
                   (big, 'RT_ILLUM_MAX_RAYS')):
        assert lib.rt_grid_illumination(g.handle, p(st), p(L), p(L), p(rec), None) == -1
        assert msg in lib.rt_last_error().decode(), msg
    a = [st, L, L, rec]
    for i in range(len(a)):
        b = [p(t) if j != i else None for j, t in enumerate(a)]
        assert lib.rt_grid_illumination(grid.handle, *b, None) == -1
        assert 'required' in lib.rt_last_error().decode()
    with pytest.raises(ValueError):
        E.grid_illumination(grid, st[1:], L, L)
    with pytest.raises(ValueError):
        A.relative_illumination(opm, 1025)
    assert E.launch_count() == n0
    for g in (grid, vign, paired, rect, one, big):
        g.close()


def test_repeatable_on_a_side_stream():
    opm = load_model('cellphone')
    a = A.relative_illumination(opm, 256)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        b = A.relative_illumination(opm, 256)
    s.synchronize()
    assert bits(a.record) == bits(b.record) and bits(a.ri) == bits(b.ri)
