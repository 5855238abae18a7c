"""GPU: the through-focus trace (rt_trace_grid_focus) against rt_trace_grid plane by plane.

Each plane's summary must equal, column for column, the summary of a single-focus grid trace at
that focus with the same reference points and chunk range: sums and counts as bit patterns,
min / max by == (fmin / fmax may return either signed zero)."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import load_model
from rayoptics_b200 import _abi, engine as E, analyses as A
from rayoptics_b200.table import SurfaceTable

pytestmark = pytest.mark.gpu

MODELS = ['dblgauss', 'evenasph', 'threemir', 'fisheye', 'relay_na']
SUM_COLS = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 14, 15]
MINMAX_COLS = [10, 11, 12, 13]


def planes(opm):
    """K = 7 focus shifts: 0, negative values and the model's focus_shift exactly"""
    fs = opm.optical_spec.defocus.focus_shift
    return [0.0, -0.05, 0.02, fs, -0.0, 0.1, -0.125]


def setup(name, num):
    opm = load_model(name)
    tab = SurfaceTable.from_model(opm.seq_model, device=0)
    grid = E.grid_for_model(opm, tab, num, ref_img=None)
    wi = tab.wvl_index(opm.seq_model.central_wavelength())
    return opm, tab, grid, wi


def single_focus_summary(opm, tab, num, foc, ref_k, n_wvls, c0, c1):
    ref = np.repeat(ref_k[:, None, :], n_wvls, axis=1)
    g1 = E.grid_for_model(opm, tab, num, foc=foc, ref_img=ref)
    r = E.trace_grid(tab, g1, c0, c1, outputs=(), summary=True)
    s = r.summary.cpu().numpy()
    g1.close()
    return s


def assert_same_summary(got, want, what):
    assert got[:, SUM_COLS].view(np.uint64).tolist() == want[:, SUM_COLS].view(np.uint64).tolist(), what
    assert (got[:, MINMAX_COLS] == want[:, MINMAX_COLS]).all(), what


def check_planes(name, num, chunk_range=None):
    opm, tab, grid, wi = setup(name, num)
    foc = planes(opm)
    ref = grid.chief_ref_focus(tab, wi, foc)
    c0, c1 = chunk_range if chunk_range is not None else (0, grid.n_chunks)
    summ = E.trace_grid_focus(tab, grid, foc, c0, c1, ref_img=ref).cpu().numpy()
    ref_h = ref.cpu().numpy()
    assert summ.shape == (len(foc), grid.n_tiles, 16)
    for k, f in enumerate(foc):
        want = single_focus_summary(opm, tab, num, f, ref_h[k], grid.n_wvls, c0, c1)
        assert_same_summary(summ[k], want, (name, num, k, f))
    assert (summ[:, :, 0].sum() > 0) == (c1 > c0)
    grid.close()


@pytest.mark.parametrize('num', [16, 768])          # one chunk per tile (per-chunk records) | work items
@pytest.mark.parametrize('name', MODELS)
def test_planes_equal_single_focus_traces(name, num):
    check_planes(name, num)


@pytest.mark.parametrize('name', ['dblgauss', 'threemir'])
def test_planes_equal_single_focus_traces_partial_range(name):
    opm, tab, grid, wi = setup(name, 48)
    n = grid.n_chunks
    grid.close()
    check_planes(name, 48, (3, n - 5))
    check_planes(name, 48, (2, 2))                    # empty range: identities


@pytest.mark.parametrize('name', ['dblgauss', 'threemir'])
def test_planes_between_sm_count_and_summary_ctas(name):
    """num 227: 202 chunks per tile, more than the SMs but no more than the CTAs of the summary launch
    (lean dblgauss: 3 per SM; general threemir: 2), so both launches keep per-chunk records.  Only a
    range that cuts tiles tells that regime from work items."""
    opm, tab, grid, wi = setup(name, 227)
    n, cpt = grid.n_chunks, grid.chunks_per_tile
    grid.close()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert sms < cpt <= 2*sms
    check_planes(name, 227, (3, n - 5))


@pytest.mark.parametrize('name', MODELS)
def test_chief_ref_focus(name):
    """plane k: the chief ray of rt_grid_chief_ref, defocused to foc[k] with p + (foc/d_z) d"""
    opm, tab, grid, wi = setup(name, 4)
    foc = planes(opm)
    dev = torch.device('cuda', 0)
    ref0 = torch.empty((grid.n_fields, 2), dtype=torch.float64, device=dev)
    grid.chief_ref(tab, wi, out=ref0)
    got = grid.chief_ref_focus(tab, wi, foc).cpu().numpy()
    ref0 = ref0.cpu().numpy()
    assert (got[0] == ref0).all() and (got[4] == ref0).all()       # foc = +-0
    if grid.pupil_kind != _abi.PUPIL_WIDE:       # (the grid trace starts wide-angle rays off the object)
        recs, eprad, z_pupil = opm.optical_spec.grid_fields(opm.optical_spec.field_of_view.fields)
        g0 = E.PupilGrid(recs, [wi], [0.0], [0.0], eprad, z_pupil, apply_vignetting=False,
                         flip_z_dir=opm.seq_model.z_dir[0], device=0)
        r0 = E.trace_grid(tab, g0, outputs=('p', 'd'), summary=False, check_apertures=False)
        p, d = r0.p.cpu().numpy(), r0.d.cpu().numpy()
        g0.close()
        assert p[:2].T.view(np.uint64).tolist() == ref0.view(np.uint64).tolist()
        for k, f in enumerate(foc):
            dist = f/d[2]
            want = np.stack([p[0] + dist*d[0], p[1] + dist*d[1]], axis=1)
            assert got[k].view(np.uint64).tolist() == want.view(np.uint64).tolist(), (name, k)
    grid.close()


@pytest.mark.parametrize('name', ['dblgauss', 'threemir'])
def test_per_ray_outputs_equal_trace_grid(name):
    opm, tab, grid, wi = setup(name, 40)
    c0, c1 = 1, grid.n_chunks - 1
    n = grid.rays_in_chunks(c0, c1)
    res = E.BundleResult(n, tab.n_ifc, torch.device('cuda', 0), ('p', 'd', 'status', 'op'))
    E.trace_grid_focus(tab, grid, [0.0, 0.1], c0, c1, res=res)
    want = E.trace_grid(tab, grid, c0, c1, outputs=('p', 'd', 'status', 'op'), summary=False)
    for key in ('p', 'd', 'status', 'op'):
        a, b = getattr(res, key).cpu().numpy(), getattr(want, key).cpu().numpy()
        assert a.tobytes() == b.tobytes(), key
    grid.close()


def test_through_focus_against_spot_diagrams():
    """through_focus plane k refers the aberrations to the chief ray defocused to foc[k];
    spot_diagram refers them to its image intercept.  Counts are equal, the centroids differ by the
    shift of the reference point, the RMS radii agree."""
    opm = load_model('dblgauss')
    foc = [-0.1, -0.03, 0.0, 0.04, 0.12]
    tf = A.through_focus(opm, 64, foc=foc)
    assert tf.summary['rms_radius'].shape == (5, tf.n_fields, tf.n_wvls)
    rms = []
    for k, f in enumerate(foc):
        sd = A.spot_diagram(opm, 64, foc=f)
        s = sd.summary
        for key in ('n_ok', 'n_missed', 'n_tir', 'n_blocked'):
            assert (tf.summary[key][k] == s[key]).all(), key
        shift = tf.ref_img[k] - sd.ref_img                   # [n_fields, 2]
        scale = np.maximum(np.abs(s['centroid_x']), s['rms_radius']) + np.abs(s['centroid_y'])
        np.testing.assert_allclose(tf.summary['centroid_x'][k] + shift[:, :1], s['centroid_x'], rtol=0,
                                   atol=1e-12*scale.max())
        np.testing.assert_allclose(tf.summary['centroid_y'][k] + shift[:, 1:], s['centroid_y'], rtol=0,
                                   atol=1e-12*scale.max())
        np.testing.assert_allclose(tf.summary['rms_radius'][k], s['rms_radius'], rtol=1e-12)
        rms.append(s['rms_radius'])
    assert (tf.best_index == np.argmin(np.array(rms), axis=0)).all()
    assert (tf.best_foc == np.array(foc)[tf.best_index]).all()
    assert len(set(tf.best_index.ravel().tolist())) >= 1


def test_launches_do_not_depend_on_the_number_of_planes():
    opm = load_model('dblgauss')
    A.through_focus(opm, 32, foc=[0.0, 0.1])             # grid / table set up
    counts = []
    for k in (2, 32):
        n0 = E.launch_count()
        A.through_focus(opm, 32, foc=np.linspace(-0.1, 0.1, k))
        counts.append(E.launch_count() - n0)
    assert counts[0] == counts[1] == 3, counts


def test_abi_argument_checks():
    lib = _abi.load_library()
    opm, tab, grid, wi = setup('dblgauss', 8)
    dev = torch.device('cuda', 0)
    opts = _abi.make_opts(first_surf=1, last_surf=tab.n_ifc - 2, check_apertures=True)
    summ = torch.empty((_abi.RT_MAX_FOCUS + 1, grid.n_tiles, 16), dtype=torch.float64, device=dev)
    scratch = torch.empty(lib.rt_grid_focus_scratch_bytes(grid.handle, 2, 0, grid.n_chunks)//8,
                          dtype=torch.float64, device=dev)
    abr = torch.empty((2, grid.n_rays), dtype=torch.float64, device=dev)
    ok_out = _abi.rt_out()
    bad_out = _abi.rt_out()
    bad_out.abr_x = C.c_void_p(abr[0].data_ptr())

    def call(foc, n, out=ok_out, summary=summ):
        f = np.ascontiguousarray(foc, dtype=np.float64)
        rc = lib.rt_trace_grid_focus(tab.handle, grid.handle, 0, grid.n_chunks, C.byref(opts),
                                     f.ctypes.data_as(_abi.c_double_p), n, None, C.byref(out),
                                     None if summary is None else C.c_void_p(summary.data_ptr()),
                                     C.c_void_p(scratch.data_ptr()), None)
        return rc, lib.rt_last_error().decode()
    n0 = E.launch_count()
    for args, msg in ((([0.0], 0), 'n_foc'), (([0.0]*65, 65), 'n_foc'), (([0.0, np.nan], 2), 'finite'),
                      (([0.0, np.inf], 2), 'finite'), (([0.0], 1, bad_out), 'abr_x'),
                      (([0.0], 1, ok_out, None), 'summary')):
        rc, err = call(*args)
        assert rc == -1 and msg in err, (args[1:], rc, err)
    assert E.launch_count() == n0
    assert lib.rt_grid_focus_scratch_bytes(grid.handle, 0, 0, grid.n_chunks) == 0
    assert lib.rt_grid_focus_scratch_bytes(grid.handle, 3, 0, grid.n_chunks) == \
        3*lib.rt_grid_scratch_bytes(grid.handle, 0, grid.n_chunks)
    ref = torch.empty((2, grid.n_fields, 2), dtype=torch.float64, device=dev)
    f = np.array([0.0, np.nan])
    assert lib.rt_grid_chief_ref_focus(tab.handle, grid.handle, wi, f.ctypes.data_as(_abi.c_double_p), 2,
                                       C.c_void_p(ref.data_ptr()), None) == -1
    grid.close()
