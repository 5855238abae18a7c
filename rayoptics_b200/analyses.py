"""Grid / list / fan analyses as single bundle launches.

The reference evaluates every analysis with a Python loop that traces one ray
per iteration (/root/reference/src/rayoptics/raytr/trace.py:537-605,
raytr/analyses.py:212-230,437-455,666-696; seq/sequential.py:1006-1085).  Here
the whole fields x wavelengths x pupil-grid index space is one ``rt_trace_grid``
launch; the start rays are generated on the device and only the requested
results come back to the host.

``spot_diagram`` is the engine-side equivalent of
``SequentialModel.trace_grid(spot, fi, num_rays=N, form='list',
append_if_none=False)`` evaluated for every field
(seq/sequential.py:1058-1085 with the ``spot`` filter of
mpl/axisarrayfigure.py:229-238): per field and wavelength the transverse ray
aberrations ``(dx, dy)`` of the rays that reach the image, referred to the
chief-ray image point at the central wavelength.
"""
from __future__ import annotations

import threading

import numpy as np
import torch

from . import engine as E
from .table import SurfaceTable
from .model import Field
from .opticalspec import grid_fields_of


class SpotDiagram:
    """Result of ``spot_diagram``.

    ``abr`` ``[2, n]``: host (pinned) array over the rays this process traced, flattened
    (field, wvl, i, j) order starting at ``first_ray``; rays that do not reach the image
    hold NaNs whose payloads are their status / failing surface (``status``, ``fail_surf``
    decode them on first use).  ``grids[fi][wi]``: ``[n_ok, 2]`` arrays of the rays that
    reach the image, in the reference's order (x outer, y inner) -- the ``form='list',
    append_if_none=False`` shape of seq/sequential.py:1058-1085 -- built lazily (whole grid
    only); ``summary``: dict of ``[n_fields, n_wvls]`` arrays (n_ok, n_blocked,
    centroid_x/y, rms_radius ...), combined over all ranks; ``ref_img``: ``[n_fields, 2]``
    chief-ray image points."""

    def __init__(self, abr, status, summary, ref_img, num_rays, n_fields, n_wvls, first_ray,
                 n_rays_total, io_bytes):
        self.abr, self._status, self.summary, self.ref_img = abr, status, summary, ref_img
        self._fail_surf = None
        self.num_rays, self.n_fields, self.n_wvls = num_rays, n_fields, n_wvls
        self.first_ray, self.n_rays_total = first_ray, n_rays_total
        self.io_bytes = io_bytes            # {'h2d': ..., 'd2h': ...} of this call
        self._grids = None

    def _decode(self):
        if self._status is None:
            self._status, self._fail_surf = E.decode_nan_status(self.abr)

    @property
    def status(self):
        self._decode()
        return self._status

    @property
    def fail_surf(self):
        self._decode()
        return self._fail_surf

    @property
    def grids(self):
        if self._grids is None:
            if self.first_ray != 0 or self.abr.shape[1] != self.n_rays_total:
                raise ValueError('per-tile lists need the whole grid on one process')
            ok = (self._status == 0) if self._status is not None else ~np.isnan(self.abr[0])
            per = self.num_rays*self.num_rays
            self._grids = []
            for fi in range(self.n_fields):
                row = []
                for wi in range(self.n_wvls):
                    sl = slice((fi*self.n_wvls + wi)*per, (fi*self.n_wvls + wi + 1)*per)
                    m = ok[sl]
                    row.append(np.stack([self.abr[0, sl][m], self.abr[1, sl][m]], axis=1))
                self._grids.append(row)
        return self._grids


_STREAMS = {}
# Re-used device blocks are per THREAD: two threads running analyses on one device must not share a
# grid block (one would trace the other's description) or staging buffers.  Tables are immutable and
# stay shared (SURVEY.md 8(b) "Threading").
_TLS = threading.local()


def _per_thread(name):
    d = getattr(_TLS, name, None)
    if d is None:
        d = {}
        setattr(_TLS, name, d)
    return d


def _side_streams(dev):
    if dev not in _STREAMS:
        _STREAMS[dev] = [torch.cuda.Stream(dev), torch.cuda.Stream(dev)]
    return _STREAMS[dev]


def _spec_key(opt_model, table, num_rays, fields, wvls, foc):
    """Everything the grid description is computed from, as a hashable key: while it does not
    change, the host-side description (start points, aim points, pupil tables) of the previous
    call is uploaded again instead of being recomputed."""
    osp, sm = opt_model.optical_spec, opt_model.seq_model
    fod = osp.fod if hasattr(osp, 'fod') else opt_model['analysis_results']['parax_data'].fod
    fkey = tuple((f.x, f.y, f.vux, f.vuy, f.vlx, f.vly,
                  None if f.aim_info is None else tuple(np.asarray(f.aim_info, dtype=float).ravel()))
                 for f in fields)
    fov, pup = osp.field_of_view, osp.pupil
    return (id(table), num_rays, fkey, tuple(wvls), foc, tuple(pup.key), pup.value, tuple(fov.key),
            fov.value, fov.is_relative, fov.is_wide_angle, sm.z_dir[0], sm.gaps[0].thi) + tuple(
                getattr(fod, a, None) for a in ('obj_dist', 'enp_dist', 'enp_radius', 'm', 'obj_na',
                                                'pr_ht0', 'pr_slp0', 'n_obj', 'n_img'))


def _reusable_grid(opt_model, table, num_rays, fields, wvls, foc):
    """The PupilGrid of this description: the device block and its pinned staging are allocated
    once per shape (``rt_grid_create``); every call uploads the description again (one
    asynchronous copy, ``rt_grid_update``) -- no cudaMalloc / cudaFree per analysis call -- and
    the host-side description itself is recomputed only when its inputs changed."""
    key = _spec_key(opt_model, table, num_rays, fields, wvls, foc)
    hit = _SPECS.get(key)
    if hit is None:
        args, kw = E._grid_args(opt_model, table.wvl_index, num_rays, fields, wvls, foc, (-1.0, 1.0), True)
        spec = E.PupilGridSpec(*args, **kw)
        if len(_SPECS) > 32:
            _SPECS.clear()
        hit = _SPECS[key] = (spec, args, kw)
    spec, args, kw = hit
    gkey = (int(table.device), spec.n_fields, spec.n_wvls, spec.nx, spec.ny, spec.paired, spec.wave is not None)
    grids = _per_thread('grids')     # shape key -> PupilGrid whose device block / pinned staging is re-used
    grid = grids.get(gkey)
    if grid is None or grid._handle is None:
        if len(grids) > 16:
            for g in grids.values():
                g.close()
            grids.clear()
        grid = grids[gkey] = E.PupilGrid(*args, device=table.device, **kw)
    else:
        grid.upload(spec)
    return grid, spec


_SPECS = {}


def _table_for(opt_model, table=None, device=0):
    if table is not None:
        return table
    sm = opt_model.seq_model
    cached = getattr(sm, '_b200_table', None)
    version = getattr(sm, '_version', None)
    built = None
    if version is None:
        # a model of the reference: no edit counter -- key the cache on the compiled
        # descriptor records themselves (every number the kernels can see; the reference's
        # own invalidation point is update_model(), seq/sequential.py:666-668)
        from .table import describe_model
        built = describe_model(sm)
        version = (bytes(built[0]), built[1].tobytes(), tuple(built[2]))
    if cached is None or cached[0] != version or cached[1].device != device:
        tab = SurfaceTable(*built, device=device) if built else SurfaceTable.from_model(sm, device=device)
        cached = (version, tab)
        sm._b200_table = cached
    return cached[1]


def chief_ray_image_points(opt_model, table, fields, wvl=None, foc=0.0, io=None):
    """Image intercept of the (0, 0) pupil ray of every field at ``wvl``
    (default: central wavelength): ``ref_sphere[0]`` of
    raytr/waveabr.py:24-76 for ``image_pt_2d=None``."""
    osp, sm = opt_model.optical_spec, opt_model.seq_model
    wvl = sm.central_wavelength() if wvl is None else wvl
    recs, eprad, z_pupil = grid_fields_of(opt_model, fields)
    g0 = E.PupilGrid(recs, [table.wvl_index(wvl)], [0.0], [0.0], eprad, z_pupil,
                     apply_vignetting=False, flip_z_dir=sm.z_dir[0], foc=foc, device=table.device)
    r0 = E.trace_grid(table, g0, outputs=('p',), summary=False, check_apertures=False)
    ref = r0.p[:2].t().contiguous().cpu().numpy()
    if io is not None:
        io['h2d'] += g0.host_bytes()
        io['d2h'] += ref.nbytes
    g0.close()
    return ref        # [n_fields, 2]


def spot_diagram(opt_model, num_rays=21, fields=None, wvls=None, foc=None, table=None,
                 device=0, pinned=None, shard=None, group=None, pieces=8, chunk_range=None, **kwargs):
    """Spot diagrams of all fields and wavelengths in one pass over the device.

    Host buffers in, host buffers out: the grid description goes to the device (one
    asynchronous copy into a re-used block), the chief-ray reference image points are
    computed there (``rt_grid_chief_ref``: no host round trip), ``rt_trace_grid`` generates
    and traces the rays, and the transverse aberrations come back into pinned host memory,
    16 B per ray (status / failing surface of the rays that do not arrive ride in the NaN
    payloads).  ``shard=(rank, world)`` traces only that rank's slice of the chunk space and
    all-gathers the per-(field, wvl) sums over ``group`` (parallel.py); ``chunk_range=(c0, c1)``
    overrides the equal-length slice (e.g. ``parallel.shard_chunks_weighted``).  ``pinned``:
    optional dict with a pinned host tensor ``abr`` ``[2, >=n]`` to re-use across calls.
    ``pieces``: the chunk range is traced in that many launches on two streams so that the
    device->host copy of one piece overlaps the trace of the next."""
    from .parallel import shard_chunks, gather_summaries
    osp, sm = opt_model.optical_spec, opt_model.seq_model
    table = _table_for(opt_model, table, device)
    fields = list(osp.field_of_view.fields if fields is None else fields)
    wvls = list(sm.wvlns if wvls is None else wvls)
    foc = osp.defocus.focus_shift if foc is None else foc
    io = {'h2d': 0, 'd2h': 0}
    dev = torch.device('cuda', table.device)
    with torch.cuda.device(dev):
        grid, spec = _reusable_grid(opt_model, table, num_rays, fields, wvls, foc)
        io['h2d'] += spec.host_bytes()
        ws = _per_thread('work').setdefault(table.device, {})     # re-used device staging buffers
        if ws.get('ref') is None or ws['ref'].shape[0] != len(fields):
            ws['ref'] = torch.empty((len(fields), 2), dtype=torch.float64, device=dev)
        ref_dev = ws['ref']
        grid.chief_ref(table, table.wvl_index(sm.central_wavelength()), out=ref_dev)
        c0, c1 = (0, grid.n_chunks) if shard is None else shard_chunks(grid.n_chunks, *shard)
        if chunk_range is not None:          # this rank's range, e.g. parallel.shard_chunks_weighted
            c0, c1 = chunk_range
        n = grid.rays_in_chunks(c0, c1)
        if pinned is None:
            pinned = {'abr': torch.empty((2, max(n, 1)), dtype=torch.float64).pin_memory()}
        h_abr = pinned['abr'][:, :n]
        # the chunk range is traced in `pieces` launches on two streams of the grid handle, each
        # followed by its device->host copy (rt_trace_grid_to_host): one C call, no per-piece Python
        summ, ws['trace'] = E.trace_grid_to_host(table, grid, pinned['abr'], c0, c1,
                                                 pieces=max(1, min(pieces, (c1 - c0)//64)),
                                                 workspace=ws.get('trace'), **kwargs)
        if shard is not None:
            summ = gather_summaries(summ, group)
        tail = torch.cat([summ.reshape(-1), ref_dev.reshape(-1)]).cpu().numpy()   # one small copy; waits
        torch.cuda.current_stream(dev).synchronize()
    summ_host = tail[:summ.numel()].reshape(summ.shape)
    ref = tail[summ.numel():].reshape(len(fields), 2).copy()
    stats_host = {k: np.asarray(v).reshape(len(fields), len(wvls))
                  for k, v in E.spot_statistics(summ_host).items()}
    io['d2h'] += h_abr.numel()*8 + tail.nbytes
    return SpotDiagram(h_abr.numpy(), None, stats_host, ref, num_rays, len(fields), len(wvls),
                       grid.first_ray_of_chunk(c0), grid.n_rays, io)


class ThroughFocus:
    """Result of ``through_focus``.

    ``foc`` ``[K]``: the focus shifts of the image planes; ``summary``: the ``spot_statistics``
    keys as ``[K, n_fields, n_wvls]`` arrays, combined over all ranks; ``ref_img``
    ``[K, n_fields, 2]``: the chief-ray image points defocused to each plane (the reference
    points of that plane's aberrations); ``best_index`` / ``best_foc`` ``[n_fields, n_wvls]``:
    the sampled plane of least ``rms_radius`` (-1 / NaN where no ray reaches the image)."""

    def __init__(self, foc, summary, ref_img, num_rays, n_fields, n_wvls):
        self.foc, self.summary, self.ref_img = foc, summary, ref_img
        self.num_rays, self.n_fields, self.n_wvls = num_rays, n_fields, n_wvls
        self.best_index, self.best_foc = best_focus(foc, summary['rms_radius'], summary['n_ok'])


def focus_planes(defocus, num_planes):
    """The planes of a FocusRange: ``defocus.get_focus(fr)`` for ``fr`` in ``linspace(-1, 1,
    num_planes)``.  A zero ``defocus_range`` would make every plane the same: ValueError."""
    if defocus.defocus_range == 0:
        raise ValueError('the model\'s defocus_range is 0: pass the focus shifts as foc=')
    return np.array([defocus.get_focus(fr) for fr in np.linspace(-1.0, 1.0, int(num_planes))])


def best_focus(foc, rms_radius, n_ok):
    """``(best_index, best_foc)`` over axis 0 of ``rms_radius`` ``[K, ...]``: the first plane of
    least RMS radius; -1 and NaN where no ray reaches the image (``n_ok`` is 0 on every plane)."""
    foc = np.asarray(foc, dtype=np.float64)
    rms = np.where(np.asarray(n_ok) > 0, np.asarray(rms_radius, dtype=np.float64), np.inf)
    rms = np.where(np.isnan(rms), np.inf, rms)
    idx = np.argmin(rms, axis=0)
    none = ~np.isfinite(rms).any(axis=0)
    idx = np.where(none, -1, idx)
    return idx, np.where(none, np.nan, foc[np.maximum(idx, 0)])


def through_focus(opt_model, num_rays=21, foc=None, num_planes=21, fields=None, wvls=None, table=None,
                  device=0, shard=None, group=None, chunk_range=None, **kwargs):
    """RMS spot size against focus for every field and wavelength, from one grid trace.

    The spot grid of ``spot_diagram`` is traced once and each ray's transverse aberration is
    evaluated at every focus shift of ``foc`` (default: ``focus_planes(osp.defocus,
    num_planes)``), referred to the chief ray at the central wavelength defocused to that plane
    (``calculate_reference_sphere``'s image point, raytr/waveabr.py:24-76).  Only the per-plane
    spot sums leave the device.  ``shard=(rank, world)`` / ``group`` / ``chunk_range`` as
    ``spot_diagram``: one all-gather of the ``[K*n_tiles, 16]`` sums whatever K is.  At most
    ``RT_MAX_FOCUS`` planes per call."""
    from .parallel import shard_chunks, gather_summaries
    osp, sm = opt_model.optical_spec, opt_model.seq_model
    foc = focus_planes(osp.defocus, num_planes) if foc is None else E._focus_array(foc)
    table = _table_for(opt_model, table, device)
    fields = list(osp.field_of_view.fields if fields is None else fields)
    wvls = list(sm.wvlns if wvls is None else wvls)
    dev = torch.device('cuda', table.device)
    with torch.cuda.device(dev):
        # the grid's own foc is not used by the through-focus trace
        grid, spec = _reusable_grid(opt_model, table, num_rays, fields, wvls, osp.defocus.focus_shift)
        ref_dev = grid.chief_ref_focus(table, table.wvl_index(sm.central_wavelength()), foc)
        c0, c1 = (0, grid.n_chunks) if shard is None else shard_chunks(grid.n_chunks, *shard)
        if chunk_range is not None:
            c0, c1 = chunk_range
        summ = E.trace_grid_focus(table, grid, foc, c0, c1, ref_img=ref_dev, **kwargs)
        if shard is not None:
            summ = gather_summaries(summ.reshape(-1, summ.shape[-1]), group)
        tail = torch.cat([summ.reshape(-1), ref_dev.reshape(-1)]).cpu().numpy()     # one small copy; waits
    k, nf, nw = len(foc), len(fields), len(wvls)
    summ_host = tail[:summ.numel()].reshape(k*nf*nw, -1)
    stats = {key: np.asarray(v).reshape(k, nf, nw) for key, v in E.spot_statistics(summ_host).items()}
    ref = tail[summ.numel():].reshape(k, nf, 2).copy()
    return ThroughFocus(foc, stats, ref, num_rays, nf, nw)


class WavefrontError:
    """Result of ``wavefront_error``: ``[n_fields, n_wvls]`` arrays, in waves, of

    ``rms`` (piston removed), ``pv``, ``rms_tilt`` / ``tilt_x`` / ``tilt_y`` (least-squares fit on
    {1, x, y}), ``rms_focus`` / ``focus`` (fit on {1, x, y, r^2}; coefficients at unit relative
    pupil), and the ray counts ``n_ok``, ``n_missed``, ``n_tir``, ``n_blocked``, ``n_other``
    (``engine.wavefront_statistics``).  ``summary``: the combined ``[n_tiles, RT_WFE_DOUBLES]``
    sums; ``ref_img`` ``[n_fields, n_wvls, 2]``: the reference image points; ``num_rays``: pupil
    samples per side."""

    def __init__(self, stats, summary, ref_img, num_rays, n_fields, n_wvls):
        self.stats = {k: np.asarray(v).reshape(n_fields, n_wvls) for k, v in stats.items()}
        for k, v in self.stats.items():
            setattr(self, k, v)
        self.summary, self.ref_img = summary, ref_img
        self.num_rays, self.n_fields, self.n_wvls = num_rays, n_fields, n_wvls


def _wavefront_pupil(opt_model, fld, num_rays):
    """pupil samples of ``RayGrid``: ``num_rays`` accumulated steps over the field's vignetting
    bounding box (Field.vignetting_bbox, oversize 1)"""
    poly = np.array([fld.apply_vignetting(list(pr)) for pr in opt_model.optical_spec.pupil.pupil_rays])
    lo, hi = poly.min(axis=0), poly.max(axis=0)
    return (E.accumulated_steps(lo[0], hi[0], num_rays), E.accumulated_steps(lo[1], hi[1], num_rays))


def _wfe_sums_host(spec, status, opd):
    """The ``[n_tiles, RT_WFE_DOUBLES]`` record of traced rays, formed on the host (the
    ``backend=`` test seam; the device forms it in ``rt_trace_grid_wfe``)."""
    from ._abi import RT_WFE_DOUBLES
    s = np.zeros((spec.n_tiles, RT_WFE_DOUBLES))
    per = spec.rays_per_tile
    for t in range(spec.n_tiles):
        f = t//spec.n_wvls
        gx, gy = np.meshgrid(spec.pupil_x[f], spec.pupil_y[f], indexing='ij')
        st, w = status[t*per:(t + 1)*per], opd[t*per:(t + 1)*per]
        ok = st == 0
        cls = np.where((st >= 0) & (st <= 3), st, 4)
        s[t, 0:5] = np.bincount(cls, minlength=5)[:5]
        x, y, w = gx.ravel()[ok], gy.ravel()[ok], w[ok]
        r2 = x*x + y*y
        s[t, 5] = np.fmin.reduce(w, initial=np.inf)
        s[t, 6] = np.fmax.reduce(w, initial=-np.inf)
        s[t, 7:20] = [v.sum() for v in (w, w*w, x*w, y*w, r2*w, x, y, x*x, x*y, y*y, x*r2, y*r2, r2*r2)]
    return s


def wavefront_grid_args(opt_model, table, num_rays, fields, wvls, foc, image_pt_2d=None, image_delta=None,
                        backend=None, ref_wvl_for_image_pt=None):
    """``(args, kw)`` of the PupilGridSpec / PupilGrid that ``wavefront_error`` traces: the chief rays
    and reference spheres of all tiles (one ``waveabr.setup_tiles`` call), each field's ``RayGrid``
    pupil samples, no vignetting applied.  ``ref_wvl_for_image_pt``: refer every wavelength to that
    wavelength's chief-ray image point (``setup_tiles``); by default each its own"""
    wave, ref_img, _ = W.setup_tiles(opt_model, table, fields, wvls, foc, image_pt_2d, image_delta,
                                     ref_wvl_for_image_pt=ref_wvl_for_image_pt,
                                     chief_tracer=None if backend is None else backend.chief_rays)
    return _wavefront_grid_args(opt_model, table, num_rays, fields, wvls, foc, wave, ref_img)


def _wavefront_grid_args(opt_model, table, num_rays, fields, wvls, foc, wave, ref_img):
    """the PupilGrid arguments of wavefront_grid_args for given tile records"""
    sm = opt_model.seq_model
    pupils = [_wavefront_pupil(opt_model, fld, num_rays) for fld in fields]
    recs, eprad, z_pupil = grid_fields_of(opt_model, fields)
    wvl_idx = [sm.index_for_wavelength(w) if table is None else table.wvl_index(w) for w in wvls]
    args = (recs, wvl_idx, np.array([p[0] for p in pupils]), np.array([p[1] for p in pupils]), eprad, z_pupil)
    return args, dict(ref_img=ref_img, apply_vignetting=False, flip_z_dir=sm.z_dir[0], foc=foc, wave=wave)


def wavefront_error(opt_model, num_rays=21, fields=None, wvls=None, foc=None, image_pt_2d=None,
                    image_delta=None, table=None, device=0, shard=None, group=None, chunk_range=None,
                    backend=None, **kwargs):
    """RMS and P-V wavefront error, with tilt and with tilt + focus removed, of every field and
    wavelength from one grid trace.

    Tile (field f, wavelength w) holds the rays of ``RayGrid(opt_model, f, w, foc,
    num_rays=num_rays)``: the same square grid over the field's vignetting bounding box, no
    vignetting applied, apertures checked, the same chief ray and reference sphere.  The chief rays
    and reference spheres of all tiles come from one ``waveabr.setup_tiles`` call, the OPDs are
    reduced on the device to per-tile sums (``rt_trace_grid_wfe``) and only those sums come back.
    ``shard=(rank, world)`` / ``group`` / ``chunk_range`` as ``spot_diagram``: one all-gather of
    the ``[n_tiles, RT_WFE_DOUBLES]`` sums.  ``backend``: the CPU test seam of ``RayGrid``.
    ``kwargs``: trace options (``check_apertures``, ...).  Returns a ``WavefrontError``."""
    from .parallel import shard_chunks, gather_summaries
    osp, sm = opt_model.optical_spec, opt_model.seq_model
    fields = list(osp.field_of_view.fields if fields is None else fields)
    wvls = list(sm.wvlns if wvls is None else wvls)
    foc = osp.defocus.focus_shift if foc is None else foc
    tab = None if backend is not None else _table_for(opt_model, table, device)
    args, grid_kw = wavefront_grid_args(opt_model, tab, num_rays, fields, wvls, foc, image_pt_2d, image_delta,
                                        backend)
    ref_img = grid_kw['ref_img']
    kwargs.setdefault('check_apertures', True)
    if backend is not None:
        spec = E.PupilGridSpec(*args, **grid_kw)
        r = backend.trace_tile(opt_model, spec, True, kwargs['check_apertures'])
        summ_host = _wfe_sums_host(spec, np.asarray(r['status']), np.asarray(r['opd']))
    else:
        dev = torch.device('cuda', tab.device)
        with torch.cuda.device(dev):
            grid = E.PupilGrid(*args, device=tab.device, **grid_kw)
            c0, c1 = (0, grid.n_chunks) if shard is None else shard_chunks(grid.n_chunks, *shard)
            if chunk_range is not None:
                c0, c1 = chunk_range
            summ = E.trace_grid_wfe(tab, grid, c0, c1, **kwargs)
            if shard is not None:
                summ = gather_summaries(summ, group)
            summ_host = summ.cpu().numpy()                 # one small copy; waits
            grid.close()
    lam = np.array([[opt_model.nm_to_sys_units(w) for w in wvls]]*len(fields)).ravel()
    stats = E.wavefront_statistics(summ_host, lam)
    return WavefrontError(stats, summ_host, ref_img, num_rays, len(fields), len(wvls))


class ZernikeFit:
    """Result of ``zernike_fit``: ``coef`` ``[n_fields, n_wvls, num_terms]``, the Fringe Zernike
    coefficients in waves (``coef[..., 0]`` is Z1, piston); ``[n_fields, n_wvls]`` arrays of
    ``rms_residual`` (sqrt(RSS/n_used), waves), ``rms`` (piston removed) and ``pv`` over the used
    rays (waves), ``n_used`` and the ray counts ``n_ok``, ``n_missed``, ``n_tir``, ``n_blocked``,
    ``n_other`` (``engine.zernike_statistics``).  ``summary``: the combined ``[n_tiles,
    RT_ZERN_DOUBLES]`` records; ``ref_img`` ``[n_fields, n_wvls, 2]``; ``num_rays``: pupil samples
    per side; ``num_terms``."""

    def __init__(self, stats, summary, ref_img, num_rays, num_terms, n_fields, n_wvls):
        self.coef = np.asarray(stats['coef']).reshape(n_fields, n_wvls, num_terms)
        self.stats = {k: np.asarray(v).reshape(n_fields, n_wvls) for k, v in stats.items() if k != 'coef'}
        for k, v in self.stats.items():
            setattr(self, k, v)
        self.summary, self.ref_img = summary, ref_img
        self.num_rays, self.num_terms, self.n_fields, self.n_wvls = num_rays, num_terms, n_fields, n_wvls


def _zernike_sums_host(spec, status, opd, n_terms):
    """The ``[n_tiles, RT_ZERN_DOUBLES]`` record of traced rays, formed on the host (the
    ``backend=`` test seam; the device forms it in ``rt_grid_zernike``)"""
    from ._abi import RT_ZERN_DOUBLES
    s = np.zeros((spec.n_tiles, RT_ZERN_DOUBLES))
    per = spec.rays_per_tile
    tri = [(i, j) for j in range(n_terms + 1) for i in range(j + 1)]
    cols = [E.zernike_gram_col(i, j) for i, j in tri]
    for t in range(spec.n_tiles):
        f = t//spec.n_wvls
        gx, gy = np.meshgrid(spec.pupil_x[f], spec.pupil_y[f], indexing='ij')
        x, y = gx.ravel(), gy.ravel()
        st, w = status[t*per:(t + 1)*per], opd[t*per:(t + 1)*per]
        used = (st == 0) & (x*x + y*y <= 1.0)
        cls = np.where((st >= 0) & (st <= 3), st, 4)
        s[t, 0:5] = np.bincount(cls, minlength=5)[:5]
        s[t, 5] = used.sum()
        s[t, 6] = np.fmin.reduce(w[used], initial=np.inf)
        s[t, 7] = np.fmax.reduce(w[used], initial=-np.inf)
        a = np.concatenate([w[used, None], E.zernike_terms(x[used], y[used], n_terms)], axis=1)
        g = a.T @ a
        s[t, cols] = [g[i, j] for i, j in tri]
    return s


def zernike_fit(opt_model, num_rays=64, num_terms=37, fields=None, wvls=None, foc=None, image_pt_2d=None,
                image_delta=None, table=None, device=0, shard=None, group=None, chunk_range=None,
                backend=None, **kwargs):
    """Fringe Zernike coefficients of the wavefront of every field and wavelength, from one grid
    trace.

    The rays are those of ``wavefront_error`` (``RayGrid``'s: a square grid over the field's
    vignetting bounding box, no vignetting applied, apertures checked, the same chief ray and
    reference sphere).  The fit is over the unit disk of relative pupil coordinates, restricted to
    the rays that arrive: a ray is used when its status is 0 and x^2 + y^2 <= 1.  The OPDs are
    reduced on the device to the Gram matrix of [W, Z_1 ... Z_num_terms] per tile
    (``rt_grid_zernike``) and only that comes back; the normal equations are solved on the host
    (``engine.zernike_statistics``).  ``num_terms``: 1 ... 37, the first Fringe terms.
    ``shard=(rank, world)`` / ``group`` / ``chunk_range`` as ``spot_diagram``: one all-gather of the
    ``[n_tiles, RT_ZERN_DOUBLES]`` records.  ``backend``: the CPU test seam of ``RayGrid``.
    ``kwargs``: trace options (``check_apertures``, ...).  Returns a ``ZernikeFit``."""
    from .parallel import shard_chunks, gather_summaries
    if not 1 <= num_terms <= E.RT_ZERN_MAX_TERMS:
        raise ValueError(f'num_terms must be 1 ... {E.RT_ZERN_MAX_TERMS}')
    osp, sm = opt_model.optical_spec, opt_model.seq_model
    fields = list(osp.field_of_view.fields if fields is None else fields)
    wvls = list(sm.wvlns if wvls is None else wvls)
    foc = osp.defocus.focus_shift if foc is None else foc
    tab = None if backend is not None else _table_for(opt_model, table, device)
    args, grid_kw = wavefront_grid_args(opt_model, tab, num_rays, fields, wvls, foc, image_pt_2d, image_delta,
                                        backend)
    ref_img = grid_kw['ref_img']
    kwargs.setdefault('check_apertures', True)
    if backend is not None:
        spec = E.PupilGridSpec(*args, **grid_kw)
        r = backend.trace_tile(opt_model, spec, True, kwargs['check_apertures'])
        summ_host = _zernike_sums_host(spec, np.asarray(r['status']), np.asarray(r['opd']), num_terms)
    else:
        dev = torch.device('cuda', tab.device)
        with torch.cuda.device(dev):
            grid = E.PupilGrid(*args, device=tab.device, **grid_kw)
            c0, c1 = (0, grid.n_chunks) if shard is None else shard_chunks(grid.n_chunks, *shard)
            if chunk_range is not None:
                c0, c1 = chunk_range
            summ = E.trace_grid_zernike(tab, grid, num_terms, c0, c1, **kwargs)
            if shard is not None:
                summ = gather_summaries(summ, group)
            summ_host = summ.cpu().numpy()                 # one small copy; waits
            grid.close()
    lam = np.array([[opt_model.nm_to_sys_units(w) for w in wvls]]*len(fields)).ravel()
    stats = E.zernike_statistics(summ_host, lam, num_terms)
    return ZernikeFit(stats, summ_host, ref_img, num_rays, num_terms, len(fields), len(wvls))


class MTF:
    """Result of ``mtf``, per field and wavelength.  Slices along the pupil axes: for fields on the y
    axis ``*_y`` is tangential and ``*_x`` sagittal.

    ``otf_x``, ``otf_y`` ``[n_fields, n_wvls, N]`` complex: the OTF against the pupil shift k =
    0 ... N-1 (``otf[..., 0]`` = 1); ``mtf_x``, ``mtf_y``: their moduli; ``freq_x``, ``freq_y``
    ``[n_fields, n_wvls, N]``: the frequency of each shift in cycles per system unit (NaN for tiles
    with an infinite reference sphere); ``cutoff`` ``[n_fields, n_wvls]``: 2 r_xp/(lambda |R|);
    ``strehl``: |sum P|^2/n_used^2 at the reference image point; ``n_used`` and the ray counts
    ``n_ok``, ``n_missed``, ``n_tir``, ``n_blocked``, ``n_other``; ``ref_img`` ``[n_fields, n_wvls,
    2]``; ``acf_x``, ``acf_y``, ``record``: the device's unnormalised autocorrelations and records.
    With ``freqs`` ``[K]``: ``otf_x_at``, ``otf_y_at``, ``mtf_x_at``, ``mtf_y_at`` ``[n_fields,
    n_wvls, K]``; polychromatic: ``poly_x``, ``poly_y`` ``[n_fields, K]`` and the weights ``wts``."""

    def __init__(self, **kw):
        for k, v in kw.items():
            setattr(self, k, v)


def _mtf_host(spec, status, opd, lam):
    """``(acf_x, acf_y, record)`` of traced rays, formed on the host (the ``backend=`` test seam; the
    device forms them in ``rt_grid_pupil_function`` and ``rt_grid_mtf``)"""
    n, per = spec.nx, spec.rays_per_tile
    acf_x = np.zeros((spec.n_tiles, n), dtype=np.complex128)
    acf_y = np.zeros((spec.n_tiles, n), dtype=np.complex128)
    rec = np.zeros((spec.n_tiles, E.RT_MTF_DOUBLES))
    for t in range(spec.n_tiles):
        f = t//spec.n_wvls
        gx, gy = np.meshgrid(spec.pupil_x[f], spec.pupil_y[f], indexing='ij')
        st, w = status[t*per:(t + 1)*per].reshape(n, n), opd[t*per:(t + 1)*per].reshape(n, n)
        P = E.pupil_function_host(st, w, gx, gy, lam[t])
        acf_x[t], acf_y[t], S = E.mtf_sums_host(P)
        cls = np.where((st >= 0) & (st <= 3), st, 4).ravel()
        rec[t, 0:5] = np.bincount(cls, minlength=5)[:5]
        rec[t, 5] = ((st == 0) & (gx*gx + gy*gy <= 1.0)).sum()
        rec[t, 6:8] = S.real, S.imag
    return acf_x, acf_y, rec


def mtf_frequencies(pupil, wave, lam, exp_radius):
    """``(freq [n_tiles, N], cutoff [n_tiles])`` of the shifts k = 0 ... N-1 along one pupil axis:
    nu_k = k*delta*r_xp/(lambda*|R|), delta = (pupil[-1] - pupil[0])/(N - 1) (relative pupil units,
    per field), R the tile's reference-sphere radius; NaN for tiles with an infinite reference sphere.
    ``pupil`` ``[n_fields, N]``; ``wave`` ``[n_fields, n_wvls, RT_WAVE_DOUBLES]``; ``lam`` ``[n_tiles]``
    in system units."""
    pupil = np.asarray(pupil, dtype=np.float64)
    nf, n = pupil.shape
    nw = wave.shape[1]
    delta = (pupil[:, -1] - pupil[:, 0])/(n - 1) if n > 1 else np.zeros(nf)
    R = np.abs(wave[:, :, 20]).ravel()
    scale = np.where(wave[:, :, 21].ravel() == 0.0, np.nan, exp_radius/(np.asarray(lam)*R))
    freq = np.arange(n)[None, :]*np.repeat(delta, nw)[:, None]*scale[:, None]
    return freq, 2.0*scale


def otf_at(freqs, freq, otf, cutoff):
    """complex OTF ``[n_tiles, K]`` at the frequencies ``freqs`` (>= 0), linear in nu between the
    native shifts ``freq`` ``[n_tiles, N]``; 0 past the last shift and past the tile's cutoff, NaN
    where the tile's frequencies are NaN"""
    freqs = np.asarray(freqs, dtype=np.float64).reshape(-1)
    out = np.empty((freq.shape[0], len(freqs)), dtype=np.complex128)
    for t in range(freq.shape[0]):
        if not np.isfinite(freq[t]).all() or not np.isfinite(cutoff[t]):
            out[t] = np.nan
            continue
        v = (np.interp(freqs, freq[t], otf[t].real, right=0.0)
             + 1j*np.interp(freqs, freq[t], otf[t].imag, right=0.0))
        out[t] = np.where(freqs > cutoff[t], 0.0, v)
    return out


def polychromatic_mtf(otf, wts):
    """|sum_w wts[w]*otf[..., w, :]|/sum wts: ``otf`` ``[n_fields, n_wvls, K]`` complex at common
    frequencies, referred to one image point -> ``[n_fields, K]``"""
    wts = np.asarray(wts, dtype=np.float64)
    return np.abs(np.einsum('fwk,w->fk', np.asarray(otf), wts))/wts.sum()


def mtf(opt_model, num_rays=64, fields=None, wvls=None, foc=None, image_pt_2d=None, image_delta=None,
        freqs=None, polychromatic=False, table=None, device=0, backend=None, **trace_kwargs):
    """Diffraction MTF along the two pupil axes and the Strehl ratio of every field and wavelength,
    from one grid trace.

    The rays are those of ``zernike_fit`` (``RayGrid``'s: ``num_rays`` x ``num_rays`` samples over
    the field's vignetting bounding box, no vignetting applied, apertures checked, the same chief ray
    and reference sphere); a ray is used when its status is 0 and x^2 + y^2 <= 1.  On the device the
    pupil function P = exp(2 pi i opd/lambda) of the used rays (0 elsewhere) is autocorrelated along
    pupil x and y in a fixed order (``rt_grid_mtf``, DESIGN.md section 4); only the ``[n_tiles, N]``
    autocorrelations and the ``[n_tiles, RT_MTF_DOUBLES]`` records come back.  OTF(k) = C(k)/C(0);
    the frequency of shift k is ``mtf_frequencies``'; the Strehl ratio is |sum P|^2/n_used^2, the
    discrete Fraunhofer PSF at the tile's reference image point over the unaberrated peak (tilt with
    respect to that point counts against it; ``image_pt_2d`` / ``image_delta`` move the point).

    The slices are along the pupil axes: for fields on the y axis ``y`` is tangential and ``x``
    sagittal.  ``freqs``: frequencies (cycles per system unit, >= 0) at which the OTF is also
    returned, interpolated linearly in nu.  ``polychromatic``: refer every wavelength to the chief-ray
    image point of the central wavelength (which must be among ``wvls``) and return |sum w OTF(nu)| /
    sum w at ``freqs`` (required), with w the model's spectral weights.  ``backend``: the CPU test seam
    of ``RayGrid``.  ``trace_kwargs``: trace options (``check_apertures``, ...).  Returns an ``MTF``."""
    if not 1 <= int(num_rays) <= E.RT_MTF_MAX_RAYS:
        raise ValueError(f'num_rays must be 1 ... {E.RT_MTF_MAX_RAYS}')
    if polychromatic and freqs is None:
        raise ValueError('polychromatic=True needs freqs=')
    if freqs is not None:
        freqs = np.asarray(freqs, dtype=np.float64).reshape(-1)
        if not (np.isfinite(freqs).all() and (freqs >= 0).all()):
            raise ValueError('freqs must be finite and >= 0')
    osp, sm = opt_model.optical_spec, opt_model.seq_model
    fields = list(osp.field_of_view.fields if fields is None else fields)
    wvls = list(sm.wvlns if wvls is None else wvls)
    foc = osp.defocus.focus_shift if foc is None else foc
    ref_wvl = None
    if polychromatic:
        ref_wvl = sm.central_wavelength()
        if ref_wvl not in wvls:
            raise ValueError('polychromatic=True needs the central wavelength among wvls')
    nf, nw, n = len(fields), len(wvls), int(num_rays)
    tab = None if backend is not None else _table_for(opt_model, table, device)
    args, grid_kw = wavefront_grid_args(opt_model, tab, n, fields, wvls, foc, image_pt_2d, image_delta, backend,
                                        ref_wvl_for_image_pt=ref_wvl)
    lam = np.array([[opt_model.nm_to_sys_units(w) for w in wvls]]*nf).ravel()
    trace_kwargs.setdefault('check_apertures', True)
    if backend is not None:
        spec = E.PupilGridSpec(*args, **grid_kw)
        r = backend.trace_tile(opt_model, spec, True, trace_kwargs['check_apertures'])
        acf_x, acf_y, rec = _mtf_host(spec, np.asarray(r['status']), np.asarray(r['opd']), lam)
    else:
        dev = torch.device('cuda', tab.device)
        with torch.cuda.device(dev):
            grid = E.PupilGrid(*args, device=tab.device, **grid_kw)
            cx, cy, rec_d, _ = E.trace_grid_mtf(tab, grid, lam, **trace_kwargs)
            host = torch.cat([torch.view_as_real(cx).reshape(-1), torch.view_as_real(cy).reshape(-1),
                              rec_d.reshape(-1)]).cpu().numpy()       # one small copy; waits
            grid.close()
        m = grid.n_tiles*n*2
        acf_x = host[:m].view(np.complex128).reshape(-1, n)
        acf_y = host[m:2*m].view(np.complex128).reshape(-1, n)
        rec = host[2*m:].reshape(-1, E.RT_MTF_DOUBLES)
    wave = grid_kw['wave']
    fod = opt_model['analysis_results']['parax_data'].fod
    freq_x, cutoff = mtf_frequencies(args[2], wave, lam, fod.exp_radius)
    freq_y, _ = mtf_frequencies(args[3], wave, lam, fod.exp_radius)
    with np.errstate(invalid='ignore', divide='ignore'):
        otf_x = acf_x/acf_x[:, :1].real                 # C(0) is real: every term of it is a*conj(a)
        otf_y = acf_y/acf_y[:, :1].real
        strehl = (rec[:, 6]**2 + rec[:, 7]**2)/rec[:, 5]**2
    shape = (nf, nw)
    out = dict(otf_x=otf_x.reshape(nf, nw, n), otf_y=otf_y.reshape(nf, nw, n),
               mtf_x=np.abs(otf_x).reshape(nf, nw, n), mtf_y=np.abs(otf_y).reshape(nf, nw, n),
               freq_x=freq_x.reshape(nf, nw, n), freq_y=freq_y.reshape(nf, nw, n),
               cutoff=cutoff.reshape(shape), strehl=strehl.reshape(shape), acf_x=acf_x, acf_y=acf_y,
               record=rec, ref_img=grid_kw['ref_img'], num_rays=n, n_fields=nf, n_wvls=nw, freqs=freqs,
               polychromatic=bool(polychromatic))
    for i, k in enumerate(E.MTF_RECORD[:6]):
        out[k] = rec[:, i].reshape(shape)
    if freqs is not None:
        for ax, o, fq in (('x', otf_x, freq_x), ('y', otf_y, freq_y)):
            at = otf_at(freqs, fq, o, cutoff).reshape(nf, nw, -1)
            out[f'otf_{ax}_at'], out[f'mtf_{ax}_at'] = at, np.abs(at)
        if polychromatic:
            region = osp.spectral_region
            wts = np.array([region.spectral_wts[list(region.wavelengths).index(w)] for w in wvls])
            out['wts'] = wts
            out['poly_x'] = polychromatic_mtf(out['otf_x_at'], wts)
            out['poly_y'] = polychromatic_mtf(out['otf_y_at'], wts)
    return MTF(**out)


class ThroughFocusWavefront:
    """Result of ``through_focus_wavefront``; plane k is focus shift ``foc[k]``.

    ``coef`` ``[K, n_fields, n_wvls, num_terms]``: Fringe Zernike coefficients in waves; ``rms``, ``pv``
    ``[K, n_fields, n_wvls]`` (piston removed, waves) and ``rms_wfe``: the RMS with piston and tilt
    removed (the 3-term fit's residual); ``strehl``: |sum P|^2/n_used^2 at plane k's reference point;
    ``ref_img`` ``[K, n_fields, n_wvls, 2]``; ``n_used`` and the ray counts ``n_ok``, ``n_missed``,
    ``n_tir``, ``n_blocked``, ``n_other`` ``[n_fields, n_wvls]`` (status does not depend on the focus);
    ``best_index_strehl`` / ``best_foc_strehl`` and ``best_index_rms`` / ``best_foc_rms`` ``[n_fields,
    n_wvls]``: the sampled plane of greatest Strehl ratio and of least ``rms_wfe`` (-1 / NaN where no
    ray is used).  With ``freqs`` ``[F]``: ``otf_x_at``, ``otf_y_at``, ``mtf_x_at``, ``mtf_y_at`` ``[K,
    n_fields, n_wvls, F]``, ``cutoff`` ``[K, n_fields, n_wvls]`` and ``shifts``, the pupil shifts whose
    autocorrelation was summed; polychromatic: ``poly_x``, ``poly_y`` ``[K, n_fields, F]`` and ``wts``.
    ``zernike_record``, ``mtf_record`` ``[K, n_tiles, ...]``, ``acf_x``, ``acf_y`` ``[K, n_tiles,
    len(shifts)]``: the raw device records."""

    def __init__(self, **kw):
        for k, v in kw.items():
            setattr(self, k, v)


def otf_shift_set(freqs, freq):
    """The native shifts ``otf_at`` reads to interpolate at ``freqs``: 0 and, for every tile (row of
    ``freq`` ``[..., N]`` with finite frequencies) and frequency, the two shifts of the bracket that
    ``np.interp`` finds in that row, widened by one on each side.  ``otf_at`` on the rows restricted to
    these shifts gives the same bits as on all N: the bracket, its slope and the end rules (the value
    at the last shift, 0 past it) are the same.  Sorted, unique, int."""
    freq = np.asarray(freq, dtype=np.float64)
    n = freq.shape[-1]
    rows = freq.reshape(-1, n)
    keep = {0}
    for row in rows[np.isfinite(rows).all(axis=1)]:
        j = np.searchsorted(row, np.asarray(freqs, dtype=np.float64), side='right') - 1
        for d in (-1, 0, 1, 2):
            keep.update(np.clip(j + d, 0, n - 1).tolist())
    return np.array(sorted(keep), dtype=np.int64)


def _opd_planes_host(opt_model, spec, fields, wvls, foc, full, op, status, pkgs):
    """``[K, n_rays]`` OPD of traced whole rays against every plane's reference sphere: the
    reference's rapid refocus, ``waveabr.wave_abr_pre_calc`` once per ray and ``wave_abr_calc`` per
    plane (the ``backend=`` seam of ``through_focus_wavefront``)"""
    fod = opt_model['analysis_results']['parax_data'].fod
    per, n_ifc = spec.rays_per_tile, full.shape[0]
    out = np.full((len(foc), spec.n_rays), np.nan)
    for t in range(spec.n_tiles):
        fi, wi = divmod(t, spec.n_wvls)
        fld, wvl = fields[fi], wvls[wi]
        crp, rs0 = pkgs[0][fi][wi]
        for r in range(t*per, (t + 1)*per):
            if status[r] != 0:
                continue
            ray = [[full[k, 0:3, r], full[k, 3:6, r], float(full[k, 6, r]), full[k, 7:10, r]] for k in range(n_ifc)]
            ray_pkg = (ray, float(op[r]), wvl)
            pre = W.wave_abr_pre_calc(fod, fld, wvl, foc[0], ray_pkg, crp, rs0)
            for k in range(len(foc)):
                out[k, r] = W.wave_abr_calc(fod, fld, wvl, foc[k], ray_pkg, crp, pre, pkgs[k][fi][wi][1])
    return out


def through_focus_wavefront(opt_model, num_rays=64, foc=None, num_planes=21, num_terms=9, freqs=None,
                            polychromatic=False, fields=None, wvls=None, image_pt_2d=None, image_delta=None,
                            table=None, device=0, backend=None, **trace_kwargs):
    """Zernike terms, RMS wavefront error, Strehl ratio and (with ``freqs``) the MTF of every field and
    wavelength at every focus shift of ``foc``, from one grid trace.

    The rays are those of ``zernike_fit`` and ``mtf`` (``RayGrid``'s ``num_rays`` x ``num_rays`` samples,
    no vignetting applied, apertures checked; a ray is used when its status is 0 and x^2 + y^2 <= 1).
    ``foc``: absolute focus shifts, as ``through_focus`` (default ``focus_planes(osp.defocus,
    num_planes)``), 1 ... RT_MAX_FOCUS of them.  The chief rays are traced once and give every plane's
    reference sphere (``waveabr.setup_tiles_focus``); one ``rt_trace_grid_opd_focus`` launch traces the
    grid and evaluates each ray's OPD against every sphere; then per plane ``rt_grid_zernike``
    (``num_terms``: 3 ... 37, default 9, through primary spherical), ``rt_grid_pupil_function`` and
    ``rt_grid_mtf_shifts`` at the pupil shifts that ``otf_at`` reads for ``freqs`` (none without them:
    the Strehl ratio needs the record only).  On finite-reference tiles plane k equals
    ``zernike_fit(foc=foc[k])`` and ``mtf(foc=foc[k])`` bit for bit; tiles with an infinite reference
    sphere round as the reference's ``focus_wavefront``.  ``polychromatic``: refer every wavelength to
    the central wavelength's chief-ray image point, as ``mtf``.  ``backend``: the CPU test seam (the
    reference's ``wave_abr_pre_calc`` / ``wave_abr_calc`` on traced whole rays).  ``trace_kwargs``:
    trace options.  Returns a ``ThroughFocusWavefront``."""
    n = int(num_rays)
    if not 1 <= n <= E.RT_MTF_MAX_RAYS:
        raise ValueError(f'num_rays must be 1 ... {E.RT_MTF_MAX_RAYS}')
    if not 3 <= int(num_terms) <= E.RT_ZERN_MAX_TERMS:
        raise ValueError(f'num_terms must be 3 ... {E.RT_ZERN_MAX_TERMS}')
    num_terms = int(num_terms)
    if polychromatic and freqs is None:
        raise ValueError('polychromatic=True needs freqs=')
    if freqs is not None:
        freqs = np.asarray(freqs, dtype=np.float64).reshape(-1)
        if not (np.isfinite(freqs).all() and (freqs >= 0).all()):
            raise ValueError('freqs must be finite and >= 0')
    osp, sm = opt_model.optical_spec, opt_model.seq_model
    foc = focus_planes(osp.defocus, num_planes) if foc is None else E._focus_array(foc)
    if not (1 <= len(foc) <= E._abi.RT_MAX_FOCUS and np.isfinite(foc).all()):
        raise ValueError(f'foc must hold 1 ... {E._abi.RT_MAX_FOCUS} finite focus shifts')
    fields = list(osp.field_of_view.fields if fields is None else fields)
    wvls = list(sm.wvlns if wvls is None else wvls)
    ref_wvl = None
    if polychromatic:
        ref_wvl = sm.central_wavelength()
        if ref_wvl not in wvls:
            raise ValueError('polychromatic=True needs the central wavelength among wvls')
    K, nf, nw = len(foc), len(fields), len(wvls)
    nt = nf*nw
    tab = None if backend is not None else _table_for(opt_model, table, device)
    wave, ref_img, spheres, pkgs = W.setup_tiles_focus(
        opt_model, tab, fields, wvls, foc, image_pt_2d, image_delta, ref_wvl_for_image_pt=ref_wvl,
        chief_tracer=None if backend is None else backend.chief_rays)
    args, grid_kw = _wavefront_grid_args(opt_model, tab, n, fields, wvls, foc[0], wave[0], ref_img[0])
    lam = np.array([[opt_model.nm_to_sys_units(w) for w in wvls]]*nf).ravel()
    fod = opt_model['analysis_results']['parax_data'].fod
    fx, cut, fy = zip(*[mtf_frequencies(args[2], wave[k], lam, fod.exp_radius)
                        + mtf_frequencies(args[3], wave[k], lam, fod.exp_radius)[:1] for k in range(K)])
    shifts = (np.zeros(0, dtype=np.int64) if freqs is None
              else otf_shift_set(freqs, np.concatenate([np.array(fx), np.array(fy)])))
    m = len(shifts)
    trace_kwargs.setdefault('check_apertures', True)
    if backend is not None:
        spec = E.PupilGridSpec(*args, **grid_kw)
        full, op, status = backend.trace_rays(opt_model, spec, trace_kwargs['check_apertures'])
        planes = _opd_planes_host(opt_model, spec, fields, wvls, foc, full, op, status, pkgs)
        zrec, acf_x, acf_y, mrec = [], [], [], []
        for k in range(K):
            zrec.append(_zernike_sums_host(spec, status, planes[k], num_terms))
            cx, cy, r = _mtf_host(spec, status, planes[k], lam)
            acf_x.append(cx[:, shifts])
            acf_y.append(cy[:, shifts])
            mrec.append(r)
        zrec, acf_x, acf_y, mrec = (np.array(v) for v in (zrec, acf_x, acf_y, mrec))
    else:
        dev = torch.device('cuda', tab.device)
        with torch.cuda.device(dev):
            grid = E.PupilGrid(*args, device=tab.device, **grid_kw)
            planes, res = E.trace_grid_opd_focus(tab, grid, spheres.reshape(K, nt, -1), **trace_kwargs)
            parts, pup = [], None
            sh_d = torch.as_tensor(shifts.astype(np.int32), device=dev)      # one upload for every plane
            for k in range(K):
                z = E.grid_zernike(grid, 0, grid.n_chunks, num_terms, res.status, planes[k])
                pup = E.grid_pupil_function(grid, res.status, planes[k], lam, out=pup)
                cx, cy, r = E.grid_mtf_shifts(grid, res.status, pup[0], pup[1], sh_d)
                parts += [z.reshape(-1), torch.view_as_real(cx).reshape(-1), torch.view_as_real(cy).reshape(-1),
                          r.reshape(-1)]
            host = torch.cat(parts).cpu().numpy()                  # one small copy; waits
            grid.close()
        sizes = (nt*E.RT_ZERN_DOUBLES, nt*m*2, nt*m*2, nt*E.RT_MTF_DOUBLES)
        per_plane = np.split(host, np.cumsum(sizes*K)[:-1])
        zrec = np.array(per_plane[0::4]).reshape(K, nt, E.RT_ZERN_DOUBLES)
        acf_x = np.array(per_plane[1::4]).view(np.complex128).reshape(K, nt, m)
        acf_y = np.array(per_plane[2::4]).view(np.complex128).reshape(K, nt, m)
        mrec = np.array(per_plane[3::4]).reshape(K, nt, E.RT_MTF_DOUBLES)
    lam_k = np.tile(lam, K)
    zs = E.zernike_statistics(zrec.reshape(K*nt, -1), lam_k, num_terms)
    z3 = E.zernike_statistics(zrec.reshape(K*nt, -1), lam_k, 3)
    shape = (K, nf, nw)
    with np.errstate(invalid='ignore', divide='ignore'):
        strehl = ((mrec[..., 6]**2 + mrec[..., 7]**2)/mrec[..., 5]**2).reshape(shape)
    rms_wfe = z3['rms_residual'].reshape(shape)
    n_used = zs['n_used'].reshape(shape)
    out = dict(foc=foc, coef=zs['coef'].reshape(shape + (num_terms,)), rms=zs['rms'].reshape(shape),
               pv=zs['pv'].reshape(shape), rms_wfe=rms_wfe, strehl=strehl, ref_img=ref_img,
               num_rays=n, num_terms=num_terms, n_fields=nf, n_wvls=nw, freqs=freqs, shifts=shifts,
               polychromatic=bool(polychromatic), zernike_record=zrec, mtf_record=mrec, acf_x=acf_x, acf_y=acf_y)
    for k in E.ZERN_STATISTICS[:6]:                   # the counts: status does not depend on the focus
        out[k] = zs[k].reshape(shape)[0]
    out['best_index_strehl'], out['best_foc_strehl'] = best_focus(foc, -strehl, n_used)
    out['best_index_rms'], out['best_foc_rms'] = best_focus(foc, rms_wfe, n_used)
    if freqs is not None:
        out['cutoff'] = np.array(cut).reshape(shape)
        for ax, acf, fq in (('x', acf_x, fx), ('y', acf_y, fy)):
            with np.errstate(invalid='ignore', divide='ignore'):
                otf = acf/acf[..., :1].real                # shift 0 leads the list: C(0) is real
            at = np.array([otf_at(freqs, fq[k][:, shifts], otf[k], cut[k]) for k in range(K)])
            out[f'otf_{ax}_at'] = at.reshape(shape + (-1,))
            out[f'mtf_{ax}_at'] = np.abs(out[f'otf_{ax}_at'])
        if polychromatic:
            region = osp.spectral_region
            wts = np.array([region.spectral_wts[list(region.wavelengths).index(w)] for w in wvls])
            out['wts'] = wts
            out['poly_x'] = np.array([polychromatic_mtf(out['otf_x_at'][k], wts) for k in range(K)])
            out['poly_y'] = np.array([polychromatic_mtf(out['otf_y_at'][k], wts) for k in range(K)])
    return ThroughFocusWavefront(**out)


class FieldMap:
    """Result of ``field_map``: a ``num_fields`` x ``num_fields`` grid of field points over the
    relative field [-1, 1]^2 (x outer, y inner).

    ``field_x``, ``field_y`` ``[n, n]``: the points' Field.x / Field.y (field-of-view units);
    ``traced`` ``[n, n]``: the point lies inside the unit circle of relative field and was aimed;
    ``valid`` ``[n, n]``: it was aimed and its chief ray reaches the image at every wavelength (the
    points with results); ``aim`` ``[n, n, 2]``: the aim points; ``img`` ``[n, n, n_wvls, 2]``: the
    real chief-ray image points (``ZernikeFit.ref_img``); ``parax_img`` ``[n, n, 2]``: the paraxial
    image points; ``distortion`` ``[n, n, n_wvls]`` in percent; ``coef`` ``[n, n, n_wvls,
    num_terms]`` Fringe Zernike coefficients, ``rms``, ``rms_residual``, ``pv`` ``[n, n, n_wvls]``, in
    waves; ``zernike``: the ``ZernikeFit`` of the valid points in row-major order of the map; ``wvls``.
    Entries without a result are NaN."""

    def __init__(self, **kw):
        for k, v in kw.items():
            setattr(self, k, v)


def paraxial_image_points(opt_model, fx, fy):
    """Paraxial image points ``[..., 2]`` of the fields (fx, fy) (field-of-view units): the chief
    ray's paraxial image height ``pr_ray[-1][HT]`` scaled linearly with the field variable the
    paraxial model is built on -- for object angles the slopes (d_x/d_z, d_y/d_z) of the object-space
    direction ``obj_coords`` gives the field, (tan a_x, tan a_y/cos a_x), against ``fod.pr_slp0``
    (tan(angle) on the x and y axes of the field); for object heights the height against
    ``fod.pr_ht0``.  NaN for every other field specification and for wide-angle fields."""
    from .firstorder import HT
    osp = opt_model.optical_spec
    fov, fod = osp.field_of_view, osp.fod
    fx, fy = np.asarray(fx, dtype=np.float64), np.asarray(fy, dtype=np.float64)
    scale = fov.value if fov.is_relative else 1.0
    key = tuple(fov.key)
    if fov.is_wide_angle or key not in (('object', 'angle'), ('object', 'height')):
        return np.full(fx.shape + (2,), np.nan)
    if key == ('object', 'angle'):
        ax, ay = np.deg2rad(scale*fx), np.deg2rad(scale*fy)
        dz = np.cos(ax)*np.cos(ay)
        ux, uy = np.sin(ax)*np.cos(ay)/dz, np.sin(ay)/dz
        umax = fod.pr_slp0
    else:
        ux, uy = scale*fx, scale*fy
        umax = fod.pr_ht0
    h = fod.pr_ray[-1][HT]
    return np.stack([h*ux/umax, h*uy/umax], axis=-1)


def field_map(opt_model, num_fields=9, num_rays=32, num_terms=37, wvls=None, foc=None, table=None, device=0,
              backend=None, **trace_kwargs):
    """Full-field maps of the wavefront (Fringe Zernike fit, RMS, P-V) and of distortion over a
    ``num_fields`` x ``num_fields`` grid of field points.

    The points are ``np.linspace(-1, 1, num_fields)`` in x (outer) and y (inner) of relative field,
    each a ``Field`` scaled by ``fov.max_field()[0]`` with zero vignetting factors; points with
    sqrt(x^2 + y^2) > 1 are not traced.  Steps: (1) the chief rays of all points are aimed on the
    device at the central wavelength (``vigcalc.aim_fields_on_device``: one launch); (2) one chief-ray
    launch (``waveabr.trace_chief_rays``) drops the points whose chief ray misses the image at any
    wavelength; (3) one ``zernike_fit`` over the remaining points.

    Distortion = 100 (|p_real| - |p_par|)/|p_par| with p_real the real chief ray's image point and
    p_par = ``paraxial_image_points`` (linear in the object-space chief-ray slope or object height): defined for object-angle and object-height fields that are not
    wide-angle, NaN for every other field specification (image heights included) and on the axis.
    ``backend``: the CPU test seam -- ``backend.aim_fields(opt_model, fields, wvl)`` aims like
    ``aim_fields_on_device``, ``backend.chief_rays`` / ``trace_tile`` as ``zernike_fit``'s.
    ``trace_kwargs``: trace options of ``zernike_fit``.  Returns a ``FieldMap``."""
    from . import vigcalc as V
    osp, sm = opt_model.optical_spec, opt_model.seq_model
    fov = osp.field_of_view
    n = int(num_fields)
    if n < 1:
        raise ValueError('num_fields must be at least 1')
    wvls = list(sm.wvlns if wvls is None else wvls)
    nw = len(wvls)
    rel = np.linspace(-1.0, 1.0, n)
    rx, ry = np.meshgrid(rel, rel, indexing='ij')
    scale = fov.max_field()[0]
    if fov.is_relative and fov.value != 0:
        scale = scale/fov.value
    field_x, field_y = scale*rx, scale*ry
    traced = np.sqrt(rx*rx + ry*ry) <= 1.0
    pts = [(i, j) for i in range(n) for j in range(n) if traced[i, j]]
    fields = [Field(x=float(field_x[i, j]), y=float(field_y[i, j]), fov=fov) for i, j in pts]
    tab = None if backend is not None else _table_for(opt_model, table, device)
    cwl = osp.spectral_region.central_wvl
    if backend is not None:
        backend.aim_fields(opt_model, fields, cwl)
    else:
        V.aim_fields_on_device(opt_model, fields, cwl, table=tab, device=device)
    if fields:
        _, _, status = (W.trace_chief_rays(opt_model, tab, fields, wvls) if backend is None
                        else backend.chief_rays(opt_model, fields, wvls))
        ok = (np.asarray(status).reshape(len(fields), nw) == 0).all(axis=1)
    else:
        ok = np.zeros(0, dtype=bool)
    kept = [fld for fld, k in zip(fields, ok) if k]
    where = [p for p, k in zip(pts, ok) if k]
    zf = None
    if kept:
        zf = zernike_fit(opt_model, num_rays, num_terms, fields=kept, wvls=wvls, foc=foc, table=table,
                         device=device, backend=backend, **trace_kwargs)
    nan = lambda *shape: np.full(shape, np.nan)        # noqa: E731
    aim, img, coef = nan(n, n, 2), nan(n, n, nw, 2), nan(n, n, nw, num_terms)
    rms, rms_res, pv = nan(n, n, nw), nan(n, n, nw), nan(n, n, nw)
    valid = np.zeros((n, n), dtype=bool)
    for (i, j), fld in zip(pts, fields):
        aim[i, j] = fld.aim_info
    for k, (i, j) in enumerate(where):
        valid[i, j] = True
        img[i, j], coef[i, j] = zf.ref_img[k], zf.coef[k]
        rms[i, j], rms_res[i, j], pv[i, j] = zf.rms[k], zf.rms_residual[k], zf.pv[k]
    parax = paraxial_image_points(opt_model, field_x, field_y)
    parax[~traced] = np.nan
    r_par = np.hypot(parax[..., 0], parax[..., 1])[..., None]
    r_real = np.hypot(img[..., 0], img[..., 1])
    with np.errstate(invalid='ignore', divide='ignore'):
        dist = np.where(r_par > 0, 100.0*(r_real - r_par)/r_par, np.nan)
    return FieldMap(field_x=field_x, field_y=field_y, traced=traced, valid=valid, aim=aim, img=img,
                    parax_img=parax, distortion=dist, coef=coef, rms=rms, rms_residual=rms_res, pv=pv,
                    zernike=zf, wvls=wvls, num_rays=num_rays, num_terms=num_terms)


class RelativeIllumination:
    """Result of ``relative_illumination``, per field and wavelength (``[n_fields, n_wvls]`` arrays).

    ``omega``: the projected solid angle of the image-space beam (steradians of direction-cosine area,
    in the image interface's frame); ``ri``: omega over the reference field's at the same wavelength;
    ``f_number``: the effective F-number 1/(2 |n'| sqrt(omega/pi)); ``fold``: 1 - |sum J|/sum |J|, nonzero
    where the pupil-to-direction map folds over; ``n_used``, ``n_disk``, ``n_isolated`` and the ray
    counts ``n_ok``, ``n_missed``, ``n_tir``, ``n_blocked``, ``n_other``; ``cra``: the chief ray's angle
    to the image interface's axis in degrees; ``chief_img`` ``[..., 2]`` and ``chief_dir`` ``[..., 3]``:
    its image point and last direction (NaN where the chief ray does not reach the image).
    ``ri_poly`` ``[n_fields]``: the spectrally weighted ratio with weights ``wts``; ``n_img`` ``[n_wvls]``:
    |n'|; ``fields``: the traced fields, ``ref_index``: the reference field's index among them;
    ``record``: the ``[n_tiles, RT_ILLUM_DOUBLES]`` device records."""

    def __init__(self, **kw):
        for k, v in kw.items():
            setattr(self, k, v)


def _illumination_host(spec, status, d):
    """The ``[n_tiles, RT_ILLUM_DOUBLES]`` records of traced rays, formed on the host (the ``backend=``
    test seam; the device forms them in ``rt_grid_illumination``)"""
    n, per = spec.nx, spec.rays_per_tile
    rec = np.zeros((spec.n_tiles, E.RT_ILLUM_DOUBLES))
    for t in range(spec.n_tiles):
        f = t//spec.n_wvls
        sl = slice(t*per, (t + 1)*per)
        rec[t] = E.illumination_sums_host(status[sl].reshape(n, n), d[0, sl].reshape(n, n),
                                          d[1, sl].reshape(n, n), spec.pupil_x[f], spec.pupil_y[f])
    return rec


def _aim(opt_model, fields, tab, device, backend):
    from . import vigcalc as V
    cwl = opt_model.optical_spec.spectral_region.central_wvl
    if backend is not None:
        backend.aim_fields(opt_model, fields, cwl)
    else:
        V.aim_fields_on_device(opt_model, fields, cwl, table=tab, device=device)


def relative_illumination(opt_model, num_rays=128, fields=None, wvls=None, num_fields=None, table=None, device=0,
                          backend=None, **trace_kwargs):
    """Relative illumination, effective F-number and chief-ray angle of every field and wavelength, from
    one grid trace.

    For a Lambertian object the image irradiance is proportional to the projected solid angle omega =
    integral of dL dM over the image-space beam (L, M: direction cosines in the image interface's frame),
    vignetting by the real apertures, pupil aberration and obliquity included, transmission left out.
    Each tile is a ``num_rays`` x ``num_rays`` grid over relative pupil [-1, 1]^2
    (``engine.accumulated_steps``), aimed at the field's aim point, no vignetting factors applied,
    apertures checked; omega = pi sum |J|/n_disk with J the Jacobian d(L, M)/d(x, y) of the used rays
    (``rt_grid_illumination``, DESIGN.md section 4).  RI is omega over the reference field's at the same
    wavelength; the reference field is the first field at (0, 0), or an axial field added to ``fields``
    and aimed like ``field_map``'s points.

    ``fields``: default the model's own; ``num_fields=K`` instead traces K points at relative field y =
    ``linspace(0, 1, K)``, scaled and aimed on the device as ``field_map``'s (not for wide-angle fields
    or angular pupils: NotImplementedError).  ``num_rays``: 2 ... RT_ILLUM_MAX_RAYS.  ``backend``: the
    CPU test seam -- ``backend.chief_rays`` as ``zernike_fit``'s, ``backend.aim_fields`` as
    ``field_map``'s, and ``backend.trace_directions(opt_model, spec, check_apertures)`` -> ``{'status',
    'd'}``.  ``trace_kwargs``: trace options (default ``check_apertures=True``).  Launches: the chief
    rays, the trace and the sums (plus the aiming of added fields).  Returns a
    ``RelativeIllumination``."""
    n = int(num_rays)
    if not 2 <= n <= E.RT_ILLUM_MAX_RAYS:
        raise ValueError(f'num_rays must be 2 ... {E.RT_ILLUM_MAX_RAYS}')
    osp, sm = opt_model.optical_spec, opt_model.seq_model
    fov = osp.field_of_view
    tab = None if backend is not None else _table_for(opt_model, table, device)
    if num_fields is not None:
        if fields is not None:
            raise ValueError('give fields or num_fields, not both')
        k = int(num_fields)
        if k < 1:
            raise ValueError('num_fields must be at least 1')
        scale = fov.max_field()[0]
        if fov.is_relative and fov.value != 0:
            scale = scale/fov.value
        fields = [Field(x=0.0, y=float(scale*r), fov=fov) for r in np.linspace(0.0, 1.0, k)]
        _aim(opt_model, fields, tab, device, backend)
    fields = list(fov.fields if fields is None else fields)
    ref = next((i for i, f in enumerate(fields) if f.x == 0 and f.y == 0), None)
    if ref is None:
        axial = Field(fov=fov)
        try:
            _aim(opt_model, [axial], tab, device, backend)
        except NotImplementedError as e:
            raise ValueError('relative_illumination: this model\'s fields cannot be aimed on the device; '
                             'pass fields= including an axial field (x = y = 0)') from e
        fields.append(axial)
        ref = len(fields) - 1
    wvls = list(sm.wvlns if wvls is None else wvls)
    nf, nw = len(fields), len(wvls)
    trace_kwargs.setdefault('check_apertures', True)
    full, _, cstatus = (W.trace_chief_rays(opt_model, tab, fields, wvls) if backend is None
                        else backend.chief_rays(opt_model, fields, wvls))
    wvl_index = sm.index_for_wavelength if tab is None else tab.wvl_index
    args, kw = E._grid_args(opt_model, wvl_index, n, fields, wvls, None, (-1.0, 1.0), False)
    if backend is not None:
        spec = E.PupilGridSpec(*args, **kw)
        r = backend.trace_directions(opt_model, spec, trace_kwargs['check_apertures'])
        rec = _illumination_host(spec, np.asarray(r['status']), np.asarray(r['d']))
    else:
        dev = torch.device('cuda', tab.device)
        with torch.cuda.device(dev):
            grid = E.PupilGrid(*args, device=tab.device, **kw)
            rec = E.trace_grid_illumination(tab, grid, **trace_kwargs).cpu().numpy()   # one small copy; waits
            grid.close()
    shape = (nf, nw)
    out = {k: rec[:, i].reshape(shape) for i, k in enumerate(E.ILLUM_RECORD[:8])}
    with np.errstate(invalid='ignore', divide='ignore'):
        omega = (np.pi*rec[:, 8]/rec[:, 6]).reshape(shape)
        ri = omega/omega[ref]
        fold = (1.0 - np.abs(rec[:, 9])/rec[:, 8]).reshape(shape)
        n_img = np.array([abs(sm.gaps[-1].medium.rindex(w)) for w in wvls])
        f_number = 1.0/(2.0*n_img*np.sqrt(omega/np.pi))
        region = osp.spectral_region
        wts = np.array([region.spectral_wts[list(region.wavelengths).index(w)] for w in wvls], dtype=np.float64)
        ri_poly = (omega @ wts)/(omega[ref] @ wts)
    last = np.asarray(full)[-1]                                   # [10, n_tiles]: the image segment
    ok = (np.asarray(cstatus).reshape(-1) == 0)[:, None]
    chief_img = np.where(ok, last[0:2].T, np.nan).reshape(nf, nw, 2)
    chief_dir = np.where(ok, last[3:6].T, np.nan).reshape(nf, nw, 3)
    cra = np.degrees(np.arctan2(np.hypot(chief_dir[..., 0], chief_dir[..., 1]), np.abs(chief_dir[..., 2])))
    out.update(omega=omega, ri=ri, f_number=f_number, fold=fold, ri_poly=ri_poly, wts=wts, n_img=n_img,
               cra=cra, chief_img=chief_img, chief_dir=chief_dir, record=rec, fields=fields, ref_index=ref,
               wvls=wvls, num_rays=n)
    return RelativeIllumination(**out)


# --------------------------------------------------------------------------
# RayFan / RayList / RayGrid: the reference's analysis classes
# (/root/reference/src/rayoptics/raytr/analyses.py:121-187,343-434,584-663) with
# the same constructor arguments and result attributes, each evaluated by one
# grid launch (chief rays: one more tiny launch).
# --------------------------------------------------------------------------
from . import waveabr as W                      # noqa: E402
from . import sampler                           # noqa: E402


def _resolve(opt_model, f, wl, foc):
    osp = opt_model.optical_spec
    fld = osp.field_of_view.fields[f] if isinstance(f, int) else f
    wvl = osp.spectral_region.central_wvl if wl is None else wl
    foc = osp.defocus.focus_shift if foc is None else foc
    return fld, wvl, foc


def _trace_pupil_points(opt_model, table, fld, wvl, foc, px, py, paired, apply_vignetting,
                        check_apertures, image_pt_2d, image_delta, want_opd, backend=None):
    """One (field, wvl) tile of pupil points -> host dict(pupil, abr, opd, status).
    ``backend``: test seam (object with ``chief_rays(opt_model, fields, wvls)`` and
    ``trace_tile(opt_model, spec, want_opd, check_apertures)``); None = the CUDA engine."""
    osp, sm = opt_model.optical_spec, opt_model.seq_model
    wave, ref_img, pkgs = W.setup_tiles(opt_model, table, [fld], [wvl], foc, image_pt_2d, image_delta,
                                        chief_tracer=None if backend is None else backend.chief_rays)
    recs, eprad, z_pupil = grid_fields_of(opt_model, [fld])
    if backend is not None:
        spec = E.PupilGridSpec(recs, [sm.index_for_wavelength(wvl)], px, py, eprad, z_pupil,
                               ref_img=ref_img, apply_vignetting=apply_vignetting,
                               flip_z_dir=sm.z_dir[0], foc=foc, paired=paired,
                               wave=wave if want_opd else None)
        out = backend.trace_tile(opt_model, spec, want_opd, check_apertures)
        out.update(ref_sphere=pkgs[0][0][1], chief_ray=pkgs[0][0][0])
        return out
    grid = E.PupilGrid(recs, [table.wvl_index(wvl)], px, py, eprad, z_pupil, ref_img=ref_img,
                       apply_vignetting=apply_vignetting, flip_z_dir=sm.z_dir[0], foc=foc,
                       paired=paired, wave=wave if want_opd else None, device=table.device)
    outs = ('abr', 'status') + (('opd',) if want_opd else ())
    res = E.trace_grid(table, grid, outputs=outs, summary=False, check_apertures=check_apertures)
    out = {'abr': res.abr.cpu().numpy(), 'status': res.status.cpu().numpy(),
           'opd': res.opd.cpu().numpy() if want_opd else None, 'ref_sphere': pkgs[0][0][1],
           'chief_ray': pkgs[0][0][0]}
    grid.close()
    return out


def _vignetted(fld, px, py, apply_vignetting):
    """pupil coordinates as the reference records them (after Field.apply_vignetting
    when it is applied: trace.trace_grid forwards the vignetted values)."""
    if not apply_vignetting:
        return np.array(px, dtype=float), np.array(py, dtype=float)
    vx, vy = np.array(px, dtype=float), np.array(py, dtype=float)
    for k in range(len(vx)):
        v = fld.apply_vignetting(np.array([vx[k], vy[k]]))
        vx[k], vy[k] = v[0], v[1]
    return vx, vy


class Ray:
    """A ray at the given field and wavelength (analyses.py:46-118): ``ray_seg`` (the
    segment at ``srf_indx``), ``ray_pkg`` when ``srf_save='all'``, ``t_abr`` the
    transverse aberration w.r.t. the reference image point."""

    def __init__(self, opt_model, p, f=0, wl=None, foc=None, image_pt_2d=None, image_delta=None,
                 srf_indx=-1, srf_save='single', output_filter=None, rayerr_filter=None,
                 color=None, clip_rays=False, table=None, device=0, tracer=None):
        self.opt_model = opt_model
        self.pupil = p
        self.fld, self.wvl, self.foc = _resolve(opt_model, f, wl, foc)
        self.image_pt_2d, self.image_delta = image_pt_2d, image_delta
        self.output_filter, self.rayerr_filter = output_filter, rayerr_filter
        self.clip_rays = clip_rays
        self.color = color
        self.srf_save, self.srf_indx = srf_save, srf_indx
        self._engine = dict(table=table, device=device, tracer=tracer)
        self.update_data()

    def update_data(self, **kwargs):
        from . import trace
        ref_sphere, cr_pkg = trace.setup_pupil_coords(self.opt_model, self.fld, self.wvl, self.foc,
                                                      image_pt=self.image_pt_2d,
                                                      image_delta=self.image_delta, **self._engine)
        build = kwargs.pop('build', 'rebuild')
        if build == 'rebuild':
            ray_pkg, ray_err = trace.trace_safe(self.opt_model, self.pupil, self.fld, self.wvl,
                                                self.output_filter, self.rayerr_filter,
                                                use_named_tuples=True,
                                                check_apertures=self.clip_rays, **self._engine,
                                                **kwargs)
            if ray_pkg is None:
                raise ray_err if ray_err is not None else RuntimeError('ray failed')
            self.ray_seg = ray_pkg.ray[self.srf_indx]
            if self.srf_save == 'all':
                self.ray_pkg = ray_pkg
        ray_seg = self.ray_seg
        dist = self.foc/ray_seg[1][2]
        defocused_pt = ray_seg[0] + dist*ray_seg[1]
        reference_image_pt = ref_sphere[0]
        self.t_abr = defocused_pt[:2] - reference_image_pt[:2]
        return self


class RayFan:
    """A fan of rays across the pupil (analyses.py:121-187).

    ``fan``: list of ``((pupil_x, pupil_y), (dx, dy, opd))`` for the rays that
    reach the image, ``opd`` in waves -- the output of ``focus_fan``
    (analyses.py:313-339)."""

    def __init__(self, opt_model, f=0, wl=None, foc=None, image_pt_2d=None, image_delta=None,
                 num_rays=21, xyfan='y', output_filter=None, rayerr_filter=None, color=None,
                 clip_rays=False, table=None, device=0, backend=None, **kwargs):
        self.opt_model = opt_model
        self._backend = backend
        self.fld, self.wvl, self.foc = _resolve(opt_model, f, wl, foc)
        self.image_pt_2d, self.image_delta = image_pt_2d, image_delta
        self.num_rays = num_rays
        self.xyfan = 0 if xyfan == 'x' else (1 if xyfan == 'y' else int(xyfan))
        self.color = color
        self.clip_rays = clip_rays
        self._table = None if backend is not None else _table_for(opt_model, table, device)
        self.update_data()

    def update_data(self, **kwargs):
        t = E.accumulated_steps(-1.0, 1.0, self.num_rays)
        zeros = E.accumulated_steps(0.0, 0.0, self.num_rays)
        px, py = (t, zeros) if self.xyfan == 0 else (zeros, t)
        r = _trace_pupil_points(self.opt_model, self._table, self.fld, self.wvl, self.foc, px, py,
                                True, True, self.clip_rays, self.image_pt_2d, self.image_delta, True,
                                backend=self._backend)
        convert_to_opd = 1/self.opt_model.nm_to_sys_units(self.wvl)
        vx, vy = _vignetted(self.fld, px, py, True)
        self.fan = [((vx[k], vy[k]), (r['abr'][0, k], r['abr'][1, k], convert_to_opd*r['opd'][k]))
                    for k in range(self.num_rays) if r['status'][k] == 0]
        return self


class RayList:
    """Rays from a list / generator of pupil coordinates (analyses.py:343-434).

    ``ray_abr``: ``[2, n_ok]`` transverse aberrations of the rays that reach the
    image (``np.rollaxis(focus_pupil_coords(...), 1)``, analyses.py:432)."""

    def __init__(self, opt_model, pupil_gen=None, pupil_coords=None, num_rays=21, f=0, wl=None,
                 foc=None, image_pt_2d=None, image_delta=None, output_filter=None,
                 rayerr_filter=None, clip_rays=False, apply_vignetting=True, table=None, device=0,
                 backend=None, **kwargs):
        self.opt_model = opt_model
        self._backend = backend
        if pupil_coords is not None and pupil_gen is None:
            self.pupil_coords, self.pupil_gen = pupil_coords, None
        else:
            if pupil_gen is None:
                grid_def = [np.array([-1., -1.]), np.array([1., 1.]), num_rays]
                pupil_gen = (sampler.csd_grid_ray_generator, (grid_def,), {})
            self.pupil_gen = pupil_gen
        self.fld, self.wvl, self.foc = _resolve(opt_model, f, wl, foc)
        self.image_pt_2d, self.image_delta = image_pt_2d, image_delta
        self.apply_vignetting = apply_vignetting
        # trace_pupil_coords defaults check_apertures to True when the key is absent;
        # RayList always passes clip_rays (analyses.py:389,554)
        self.clip_rays = clip_rays
        self._table = None if backend is not None else _table_for(opt_model, table, device)
        self.update_data()

    def update_data(self, **kwargs):
        if self.pupil_gen:
            fct, args, kwa = self.pupil_gen
            if fct in sampler._ARRAY_FORM and not kwa:      # whole sample set as one array
                self.pupil_coords = pts = sampler.sample_points(fct, *args)
            else:
                self.pupil_coords = fct(*args, **kwa)
                pts = None
        else:
            pts = None
        if pts is None:
            pts = np.array([np.array(p, dtype=float) for p in self.pupil_coords]).reshape(-1, 2)
        r = _trace_pupil_points(self.opt_model, self._table, self.fld, self.wvl, self.foc,
                                pts[:, 0], pts[:, 1], True, self.apply_vignetting, self.clip_rays,
                                self.image_pt_2d, self.image_delta, False, backend=self._backend)
        ok = r['status'] == 0
        self.ray_abr = r['abr'][:, ok]
        self.pupil = pts[ok].T
        return self


class RayGrid:
    """Square grid of rays over the vignetted pupil -> wavefront map
    (analyses.py:584-663).  ``grid``: ``[3, num, num]`` = pupil x, pupil y, OPD
    in waves (``value_if_none`` where the ray does not reach the image)."""

    def __init__(self, opt_model, f=0, wl=None, foc=None, image_pt_2d=None, image_delta=None,
                 output_filter=None, rayerr_filter=None, num_rays=21, clip_rays=True,
                 value_if_none=np.nan, oversize=1., table=None, device=0, backend=None, **kwargs):
        self.opt_model = opt_model
        self._backend = backend
        self.fld, self.wvl, self.foc = _resolve(opt_model, f, wl, foc)
        self.image_pt_2d, self.image_delta = image_pt_2d, image_delta
        self.num_rays, self.value_if_none, self.oversize = num_rays, value_if_none, oversize
        self.clip_rays = clip_rays
        self._table = None if backend is not None else _table_for(opt_model, table, device)
        self.update_data()

    def vignetting_bbox(self):
        """Field.vignetting_bbox (raytr/opticalspec.py:1326-1333)."""
        poly = [self.fld.apply_vignetting(list(pr)) for pr in self.opt_model.optical_spec.pupil.pupil_rays]
        poly = np.array(poly)
        return self.oversize*np.array([poly.min(axis=0), poly.max(axis=0)])

    def update_data(self, **kwargs):
        bbox = self.vignetting_bbox()
        n = self.num_rays
        px = E.accumulated_steps(bbox[0][0], bbox[1][0], n)
        py = E.accumulated_steps(bbox[0][1], bbox[1][1], n)
        # trace_ray_grid: apply_vignetting defaults to False (analyses.py:674)
        r = _trace_pupil_points(self.opt_model, self._table, self.fld, self.wvl, self.foc, px, py,
                                False, False, self.clip_rays, self.image_pt_2d, self.image_delta, True,
                                backend=self._backend)
        convert_to_opd = 1/self.opt_model.nm_to_sys_units(self.wvl)
        opd = np.where(r['status'] == 0, convert_to_opd*r['opd'], self.value_if_none).reshape(n, n)
        gx, gy = np.meshgrid(px, py, indexing='ij')
        self.grid = np.stack([gx, gy, opd])
        return self


# --- the functional forms of the analyses (analyses.py:233-273,513-542,699-732): one launch each,
#     same arguments and return values ---------------------------------------------------------
def _engine_kw(kwargs):
    return {k: kwargs.pop(k) for k in ('table', 'device', 'backend') if k in kwargs}


def _tile(opt_model, fld, wvl, foc, px, py, paired, apply_vignetting, check_apertures,
          image_pt_2d, image_delta, want_opd, eng):
    backend = eng.get('backend')
    table = None if backend is not None else _table_for(opt_model, eng.get('table'),
                                                        eng.get('device', 0))
    r = _trace_pupil_points(opt_model, table, fld, wvl, foc, px, py, paired, apply_vignetting,
                            check_apertures, image_pt_2d, image_delta, want_opd, backend=backend)
    fld.chief_ray, fld.ref_sphere = r['chief_ray'], r['ref_sphere']
    return r


def eval_fan(opt_model, fld, wvl, foc, xy, image_pt_2d=None, image_delta=None, num_rays=21,
             output_filter=None, rayerr_filter=None, **kwargs):
    """Trace a fan of rays and evaluate dx, dy, & OPD across the fan (analyses.py:233-273)."""
    eng = _engine_kw(kwargs)
    t = E.accumulated_steps(-1.0, 1.0, num_rays)
    zeros = E.accumulated_steps(0.0, 0.0, num_rays)
    px, py = (t, zeros) if xy == 0 else (zeros, t)
    apply_vig = kwargs.get('apply_vignetting', True)
    r = _tile(opt_model, fld, wvl, foc, px, py, True, apply_vig, kwargs.get('check_apertures', False),
              image_pt_2d, image_delta, True, eng)
    convert_to_opd = 1/opt_model.nm_to_sys_units(wvl)
    vx, vy = _vignetted(fld, px, py, apply_vig)
    return [((vx[k], vy[k]), (r['abr'][0, k], r['abr'][1, k], convert_to_opd*r['opd'][k]))
            for k in range(num_rays) if r['status'][k] == 0]


def eval_pupil_coords(opt_model, fld, wvl, foc, image_pt_2d=None, image_delta=None, num_rays=21,
                      **kwargs):
    """Trace a square grid of rays and return the transverse aberrations ``[n_ok, 2]``
    (analyses.py:513-542)."""
    eng = _engine_kw(kwargs)
    grid_def = [np.array([-1., -1.]), np.array([1., 1.]), num_rays]
    pts = sampler.square_grid_points(grid_def)
    r = _tile(opt_model, fld, wvl, foc, pts[:, 0], pts[:, 1], True,
              kwargs.get('apply_vignetting', True), kwargs.get('check_apertures', True),
              image_pt_2d, image_delta, False, eng)
    ok = r['status'] == 0
    return r['abr'][:, ok].T.copy()


def eval_wavefront(opt_model, fld, wvl, foc, image_pt_2d=None, image_delta=None, num_rays=21,
                   value_if_none=np.nan, **kwargs):
    """Trace a grid of rays over the vignetted pupil and evaluate the OPD: ``[num, num, 3]`` of
    (pupil x, pupil y, OPD in waves) (analyses.py:699-732)."""
    eng = _engine_kw(kwargs)
    bbox = fld.vignetting_bbox(opt_model['optical_spec']['pupil'], oversize=kwargs.get('oversize', 1.))
    px = E.accumulated_steps(bbox[0][0], bbox[1][0], num_rays)
    py = E.accumulated_steps(bbox[0][1], bbox[1][1], num_rays)
    r = _tile(opt_model, fld, wvl, foc, px, py, False, kwargs.get('apply_vignetting', False),
              kwargs.get('check_apertures', True), image_pt_2d, image_delta, True, eng)
    convert_to_opd = 1/opt_model.nm_to_sys_units(wvl)
    opd = np.where(r['status'] == 0, convert_to_opd*r['opd'], value_if_none).reshape(num_rays, num_rays)
    gx, gy = np.meshgrid(px, py, indexing='ij')
    return np.stack([gx, gy, opd], axis=2)


def select_plot_data(fan, xyfan, data_type):
    """Given a fan of data, select the sample points and the resulting data (analyses.py:190-199)"""
    f_x = np.array([p[xyfan] for p, val in fan])
    f_y = np.array([val[data_type] for p, val in fan])
    return f_x, f_y


def smooth_plot_data(f_x, f_y, num_points=100):
    """Interpolate fan data points and return a smoothed version (analyses.py:202-209)"""
    from scipy.interpolate import interp1d
    interpolator = interp1d(f_x, f_y, kind='cubic', assume_sorted=True)
    x_sample = np.linspace(f_x.min(), f_x.max(), num_points)
    return x_sample, interpolator(x_sample)


def update_psf_data(pupil_grid, build='rebuild'):
    """analyses.py:878-883"""
    pupil_grid.update_data(build=build)
    return calc_psf(pupil_grid.grid[2], pupil_grid.num_rays, pupil_grid.maxdim)


# the reference's per-ray loops of this module, batched (rayoptics_b200/trace.py)
from .trace import (analyses_trace_ray_fan as trace_ray_fan,       # noqa: E402
                    analyses_trace_ray_list as trace_ray_list,
                    analyses_trace_ray_grid as trace_ray_grid)


# --- trace once, refocus often (analyses.py:276-339,545-580,735-791): the first stage keeps the
#     whole rays of ONE launch (plus the focus-independent part of every OPD), the second stage is
#     host arithmetic on them -- no retrace when only ``foc`` / the image point changes.
#     (``eval_*`` above do both stages on the device and copy back 16-24 B per ray; these exist
#     for callers that hold on to the traced rays, e.g. the reference's focus sliders.)
def _stage_setup(opt_model, fld, wvl, foc, image_pt_2d, image_delta, kwargs):
    from . import trace as TR
    eng = {k: kwargs[k] for k in ('table', 'device', 'tracer') if k in kwargs}
    ref_sphere, cr_pkg = TR.setup_pupil_coords(opt_model, fld, wvl, foc, image_pt=image_pt_2d,
                                               image_delta=image_delta, **eng)
    return ref_sphere, cr_pkg


def _refocused(ray_pkg, foc, image_pt):
    seg = ray_pkg[0][-1]
    dist = foc/seg[1][2]
    defocused_pt = seg[0] + dist*seg[1]
    return defocused_pt - image_pt


def _pre_calc(opt_model, fld, wvl, foc, ray_pkg, cr_pkg, ref_sphere):
    if ray_pkg is None or isinstance(ray_pkg, Exception):
        return None
    fod = opt_model['analysis_results']['parax_data'].fod
    return W.wave_abr_pre_calc(fod, fld, wvl, foc, ray_pkg, cr_pkg, ref_sphere)


def trace_fan(opt_model, fld, wvl, foc, xy, image_pt_2d=None, image_delta=None, num_rays=21,
              output_filter=None, rayerr_filter=None, **kwargs):
    """Trace a fan of rays and precalculate data for rapid refocus later (analyses.py:276-310):
    ``(fan, upd_fan)`` = ``[[pupil_x, pupil_y, ray_pkg], ...]`` and the matching
    ``wave_abr_pre_calc`` tuples."""
    ref_sphere, cr_pkg = _stage_setup(opt_model, fld, wvl, foc, image_pt_2d, image_delta, kwargs)
    fld.chief_ray, fld.ref_sphere = cr_pkg, ref_sphere
    fan_start, fan_stop = np.array([0., 0.]), np.array([0., 0.])
    fan_start[xy], fan_stop[xy] = -1.0, 1.0
    fan = trace_ray_fan(opt_model, [fan_start, fan_stop, num_rays], fld, wvl, foc,
                        output_filter=output_filter, rayerr_filter=rayerr_filter, **kwargs)
    upd_fan = [_pre_calc(opt_model, fld, wvl, foc, fi[2], cr_pkg, ref_sphere) for fi in fan]
    return fan, upd_fan


def focus_fan(opt_model, fan_pkg, fld, wvl, foc, image_pt_2d=None, image_delta=None, **kwargs):
    """Refocus the fan of rays and return the transverse aberration and OPD (analyses.py:313-339):
    ``[((pupil_x, pupil_y), (dx, dy, opd in waves)), ...]``."""
    fod = opt_model['analysis_results']['parax_data'].fod
    fan, upd_fan = fan_pkg
    ref_sphere, cr_pkg = _stage_setup(opt_model, fld, wvl, foc, image_pt_2d, image_delta, kwargs)
    convert_to_opd = 1/opt_model.nm_to_sys_units(wvl)
    fan_data = []
    for (pupil_x, pupil_y, ray_pkg), pre in zip(fan, upd_fan):
        if ray_pkg is None or isinstance(ray_pkg, Exception):
            fan_data.append((pupil_x, pupil_y, np.nan))
            continue
        t_abr = _refocused(ray_pkg, foc, ref_sphere[0])
        opd = convert_to_opd*W.wave_abr_calc(fod, fld, wvl, foc, ray_pkg, cr_pkg, pre, ref_sphere)
        fan_data.append(((pupil_x, pupil_y), (t_abr[0], t_abr[1], opd)))
    return fan_data


def trace_pupil_coords(opt_model, pupil_coords, fld, wvl, foc, image_pt_2d=None, image_delta=None,
                       **kwargs):
    """Trace a list of rays and return data needed for rapid refocus (analyses.py:545-558)."""
    ref_sphere, cr_pkg = _stage_setup(opt_model, fld, wvl, foc, image_pt_2d, image_delta, kwargs)
    fld.chief_ray, fld.ref_sphere = cr_pkg, ref_sphere
    kwargs['check_apertures'] = kwargs.get('check_apertures', True)
    return trace_ray_list(opt_model, pupil_coords, fld, wvl, foc, **kwargs)


def focus_pupil_coords(opt_model, ray_list, fld, wvl, foc, image_pt_2d=None, image_delta=None,
                       **kwargs):
    """Given pre-traced rays and a reference sphere, return the transverse aberrations
    (analyses.py:561-580): ``[n, 2]`` (``nan`` entries for rays recorded as None)."""
    ref_sphere, cr_pkg = _stage_setup(opt_model, fld, wvl, foc, image_pt_2d, image_delta, kwargs)
    data = []
    for pupil_x, pupil_y, ray_pkg in ray_list:
        if ray_pkg is None:
            data.append(np.nan)
        else:
            t_abr = _refocused(ray_pkg, foc, ref_sphere[0])
            data.append((t_abr[0], t_abr[1]))
    return np.array(data)


def trace_wavefront(opt_model, fld, wvl, foc, image_pt_2d=None, image_delta=None, num_rays=21,
                    **kwargs):
    """Trace a grid of rays over the vignetted pupil and pre-calculate data needed for rapid
    refocus (analyses.py:735-766): ``(grid, upd_grid)``, rows of ``[pupil_x, pupil_y, ray_pkg]``."""
    ref_sphere, cr_pkg = _stage_setup(opt_model, fld, wvl, foc, image_pt_2d, image_delta, kwargs)
    fld.chief_ray, fld.ref_sphere = cr_pkg, ref_sphere
    vig_bbox = fld.vignetting_bbox(opt_model['optical_spec']['pupil'],
                                   oversize=kwargs.pop('oversize', 1.))
    kwargs['check_apertures'] = kwargs.get('check_apertures', True)
    grid = trace_ray_grid(opt_model, [vig_bbox[0], vig_bbox[1], num_rays], fld, wvl, foc, **kwargs)
    upd_grid = [[_pre_calc(opt_model, fld, wvl, foc, gij[2], cr_pkg, ref_sphere) for gij in row]
                for row in grid]
    return grid, upd_grid


def focus_wavefront(opt_model, grid_pkg, fld, wvl, foc, image_pt_2d=None, image_delta=None,
                    value_if_none=np.nan, **kwargs):
    """Given pre-traced rays and a reference sphere, return the rays' OPD (analyses.py:769-791):
    ``[num, num, 3]`` of (pupil x, pupil y, OPD in waves)."""
    fod = opt_model['analysis_results']['parax_data'].fod
    grid, upd_grid = grid_pkg
    ref_sphere, cr_pkg = _stage_setup(opt_model, fld, wvl, foc, image_pt_2d, image_delta, kwargs)
    convert_to_opd = 1/opt_model.nm_to_sys_units(wvl)
    out = []
    for row, upd_row in zip(grid, upd_grid):
        out_row = []
        for (pupil_x, pupil_y, ray_pkg), pre in zip(row, upd_row):
            if ray_pkg is None:
                out_row.append((pupil_x, pupil_y, value_if_none))
            else:
                opd = convert_to_opd*W.wave_abr_calc(fod, fld, wvl, foc, ray_pkg, cr_pkg, pre,
                                                     ref_sphere)
                out_row.append((pupil_x, pupil_y, opd))
        out.append(out_row)
    return np.array(out)


# --- raw ray list (analyses.py:458-510) ------------------------------------------------------
def _cuda_bundle_tracer(opt_model, table, p0, d0, wvl_idx, trace_kwargs):
    res = E.trace_bundle(table, p0, d0, wvl_idx=wvl_idx, full=True,
                         outputs=('op', 'status', 'fail_surf', 'n_seg'), **trace_kwargs)
    return {'full': res.full.cpu().numpy(), 'op': res.op.cpu().numpy(),
            'status': res.status.cpu().numpy(), 'fail_surf': res.fail_surf.cpu().numpy(),
            'n_seg': res.n_seg.cpu().numpy()}


def trace_list_of_rays(opt_model, rays, output_filter=None, rayerr_filter=None, table=None,
                       device=0, tracer=None, **kwargs):
    """Trace a list of rays ``(pt0, dir0, wvl)`` and return the ray packages in a list
    (analyses.py:458-510): one bundle launch instead of one ``trace()`` per ray, same
    ``output_filter`` / ``rayerr_filter`` conventions and the same list out."""
    from . import raytrace as RT
    from . import trace as TR
    sm = opt_model.seq_model
    rays = list(rays)
    if not rays:
        return []
    p0 = np.array([np.asarray(r[0], dtype=float) for r in rays]).T.copy()
    d0 = np.array([np.asarray(r[1], dtype=float) for r in rays]).T.copy()
    wvl_idx = np.array([sm.index_for_wavelength(r[2]) for r in rays], dtype=np.int32)
    kw = {k: v for k, v in kwargs.items() if k in TR._TRACE_RAW_KEYS}
    kw.setdefault('first_surf', 1)                       # raytrace.trace defaults (raytrace.py:77-79)
    kw.setdefault('last_surf', sm.get_num_surfaces() - 2)
    if tracer is None:
        table = _table_for(opt_model, table, device)
        tracer = _cuda_bundle_tracer
    r = tracer(opt_model, table, p0, d0, wvl_idx, kw)
    paths = {}
    ray_list = []
    for k, ray in enumerate(rays):
        wvl = ray[2]
        if wvl not in paths:
            paths[wvl] = list(sm.path(wvl))
        pkg, err = RT.package_ray(paths[wvl], r['full'][:, :, k], float(r['op'][k]),
                                  int(r['status'][k]), int(r['fail_surf'][k]), int(r['n_seg'][k]), wvl)
        if err is not None:
            if rayerr_filter == 'full':
                ray_list.append((ray, err))
            elif rayerr_filter == 'summary':
                err.ray_pkg = None
                ray_list.append((ray, err))
            continue
        pkg = TR.RayPkg(*pkg)
        if output_filter is None:
            ray_list.append(pkg)
        elif output_filter == 'last':
            rr, op_delta, w = pkg
            ray_list.append((rr[-1], op_delta, w))
        else:
            ray_list.append(output_filter(pkg))
    return ray_list


# --- PSF from a wavefront map (raytr/analyses.py:795-875) -------------------
def psf_sampling(n=None, n_pupil=None, n_airy=None):
    """Given 2 of (grid width, pupil samples, Airy-peak samples) compute the third
    (analyses.py:795-815)."""
    npa = n, n_pupil, n_airy
    i = npa.index(None)
    if i == 0:
        n = round((n_pupil*n_airy)/2.44)
    elif i == 1:
        n_pupil = round(2.44*n/n_airy)
    else:
        n_airy = round(2.44*n/n_pupil)
    return n, n_pupil, n_airy


def calc_psf_scaling(opt_model, fld, wvl, ndim, maxdim):
    """Input / output grid spacings of the FFT PSF (analyses.py:818-845): ``(delta_x, delta_xp)``,
    the linear grid spacing on the entrance pupil and on the image plane.  ``fld.ref_sphere``
    must be set (the analysis classes / ``trace.setup_pupil_coords`` do)."""
    fod = opt_model['analysis_results']['parax_data'].fod
    wl = opt_model.nm_to_sys_units(wvl)
    fill_factor = ndim/maxdim
    max_D = 2*fod.enp_radius/fill_factor
    delta_x = max_D/maxdim
    C = wl/fod.exp_radius
    delta_theta = (fill_factor*C)/2
    ref_sphere_radius = fld.ref_sphere[2]
    delta_xp = delta_theta*ref_sphere_radius
    return delta_x, delta_xp


def calc_psf(wavefront, ndim, maxdim, device=0):
    """Point spread function of a wavefront map (analyses.py:848-875): embed the
    ``ndim x ndim`` OPD map (waves, NaN = no data) in a ``maxdim`` grid, form the
    pupil function ``exp(2 pi i W)`` (entries equal to 1 are zeroed, as the
    reference does), FFT, normalise to the peak.  The FFT is ``torch.fft`` on the
    GPU (a plain library transform; tolerance vs numpy 1e-12)."""
    dev = torch.device('cuda', device)
    Wm = torch.zeros((maxdim, maxdim), dtype=torch.float64, device=dev)
    w = torch.as_tensor(np.nan_to_num(np.asarray(wavefront, dtype=np.float64)), device=dev)
    m2, nd2 = maxdim//2, ndim//2
    Wm[m2 - (nd2 - 1):m2 + (nd2 + 1), m2 - (nd2 - 1):m2 + (nd2 + 1)] = w
    phase = torch.exp(1j*2*np.pi*Wm.to(torch.complex128))
    phase = torch.where(phase == 1, torch.zeros_like(phase), phase)
    AP = torch.fft.fftshift(torch.fft.fft2(torch.fft.fftshift(phase))).abs()**2
    AP = AP/AP.max()
    return AP.cpu().numpy()


# ---------------------------------------------------------------- tolerance analysis
class TolMerit:
    """The spot merit of every variant of a tolerance run (``tol_merit``): ``merit`` / ``focus``
    ``[n_var]`` M(delta*) and delta*; ``merit0`` ``[n_var]`` M(0), at the grid's focus; ``n_ok``
    ``[n_var, n_fields]`` rays that reach the image (all wavelengths); ``centroid`` ``[n_var,
    n_fields, 2]`` the polychromatic centroid at delta*, ``centroid_shift`` the same minus variant 0's."""

    def __init__(self, merit, focus, merit0, n_ok, centroid):
        self.merit, self.focus, self.merit0, self.n_ok, self.centroid = merit, focus, merit0, n_ok, centroid
        self.centroid_shift = centroid - centroid[:1]


def _tol_moments(rec, wvl_wts):
    """per (variant, field) the spectrally weighted sums N, X1, U1, X2, XU, U2 (and for y) of the
    records ``[n_var, n_fields, n_wvls, RT_TOL_DOUBLES]``"""
    w = np.asarray(wvl_wts, dtype=np.float64)[None, None, :, None]
    s = (rec*w).sum(axis=2)
    return {'n': s[..., 0], 'x1': s[..., 5], 'y1': s[..., 6], 'x2': s[..., 7], 'y2': s[..., 8],
            'u1': s[..., 16], 'v1': s[..., 17], 'u2': s[..., 18], 'v2': s[..., 19],
            'xu': s[..., 20], 'yv': s[..., 21]}


def tol_sigma2(m, delta):
    """sigma_f^2(delta) ``[n_var, n_fields]``: the polychromatic mean square spot radius about the
    polychromatic centroid at defocus ``delta`` (``[n_var]`` or scalar) from the grid's focus,
    from the moments of ``_tol_moments``: X1 = x1 + delta u1, X2 = x2 + 2 delta xu + delta^2 u2"""
    d = np.asarray(delta, dtype=np.float64)
    d = d[:, None] if d.ndim else d
    n = m['n']
    with np.errstate(invalid='ignore', divide='ignore'):
        X1, Y1 = m['x1'] + d*m['u1'], m['y1'] + d*m['v1']
        X2 = m['x2'] + 2.0*d*m['xu'] + d*d*m['u2']
        Y2 = m['y2'] + 2.0*d*m['yv'] + d*d*m['v2']
        s2 = (X2 + Y2)/n - (X1*X1 + Y1*Y1)/(n*n)
    return np.where(n > 0, s2, np.nan)


def tol_merit(rec, wvl_wts, field_wts, compensate_focus=True):
    """``TolMerit`` of tolerance records ``[n_var, n_fields, n_wvls, RT_TOL_DOUBLES]``:
    M(delta) = sqrt(sum_f W_f sigma_f^2(delta) / sum_f W_f), quadratic in delta under the root;
    delta* = -B / 2A of M^2 = A delta^2 + B delta + C (0 where A <= 0 or not ``compensate_focus``).
    A field without rays makes its variant's merit NaN."""
    rec = np.asarray(rec, dtype=np.float64)
    m = _tol_moments(rec, wvl_wts)
    W = np.asarray(field_wts, dtype=np.float64)
    n = m['n']
    with np.errstate(invalid='ignore', divide='ignore'):
        a2 = (m['u2'] + m['v2'])/n - (m['u1']*m['u1'] + m['v1']*m['v1'])/(n*n)
        a1 = 2.0*(m['xu'] + m['yv'])/n - 2.0*(m['x1']*m['u1'] + m['y1']*m['v1'])/(n*n)
        A = (a2*W).sum(axis=1)/W.sum()
        B = (a1*W).sum(axis=1)/W.sum()
        focus = np.where(A > 0, -B/(2.0*A), 0.0) if compensate_focus else np.zeros(len(A))
    focus = np.where(np.isfinite(focus), focus, 0.0)

    def merit_at(d):
        return np.sqrt(np.maximum((tol_sigma2(m, d)*W).sum(axis=1)/W.sum(), 0.0))

    with np.errstate(invalid='ignore', divide='ignore'):
        cen = np.stack([(m['x1'] + focus[:, None]*m['u1'])/n, (m['y1'] + focus[:, None]*m['v1'])/n], axis=-1)
    return TolMerit(merit_at(focus), focus, merit_at(np.zeros(len(focus))), rec[..., 0].sum(axis=2), cen)


class WaveMerit:
    """The wavefront merit of every variant of a tolerance run (``wave_merit``), in waves: ``merit``
    ``[n_var]`` M; ``sigma`` / ``strehl`` ``[n_var, n_fields]`` the polychromatic RMS wavefront error
    sigma_f and its Marechal Strehl ratio exp(-(2 pi sigma_f)^2); ``n_ok`` ``[n_var, n_fields]`` rays that
    reach the image (all wavelengths); per tile ``[n_var, n_fields, n_wvls]``: ``rms`` the RMS wavefront
    error the merit uses (tilt and focus removed with the focus compensator, tilt removed without),
    ``focus`` the fitted focus coefficient on {1, x, y, r^2} (waves at unit relative pupil) and
    ``chief_status`` the status of the tile's chief ray (a tile whose chief ray fails is NaN)."""

    def __init__(self, merit, sigma, n_ok, rms, focus, chief_status):
        self.merit, self.sigma, self.n_ok, self.rms, self.focus = merit, sigma, n_ok, rms, focus
        self.strehl = np.exp(-(2.0*np.pi*sigma)**2)
        self.chief_status = chief_status


def wave_merit_of(rms, wvl_wts, field_wts):
    """``(M [n_var], sigma_f [n_var, n_fields])`` from per-tile RMS wavefront errors ``rms`` ``[n_var,
    n_fields, n_wvls]``: sigma_f^2 = sum_w S_w rms_fw^2 / sum_w S_w (spectral weights S), M = sqrt(sum_f
    W_f sigma_f^2 / sum_f W_f) (field weights W)"""
    w = np.asarray(wvl_wts, dtype=np.float64)
    W = np.asarray(field_wts, dtype=np.float64)
    s2 = (rms*rms*w).sum(axis=2)/w.sum()
    return np.sqrt((s2*W).sum(axis=1)/W.sum()), np.sqrt(s2)


def wave_merit(rec, lam, wvl_wts, field_wts, compensate_focus=True, chief_status=None):
    """``WaveMerit`` of wavefront-error records ``[n_var, n_fields, n_wvls, RT_WFE_DOUBLES]``
    (``engine.wavefront_statistics`` per tile; ``lam`` ``[n_wvls]`` the wavelengths in system units).
    With ``compensate_focus`` each tile's RMS has tilt and focus removed (``rms_focus``): every (field,
    wavelength) is refocused on its own, which is more optimistic than the spot criterion's one common
    defocus.  Without it tilt only (``rms_tilt``)."""
    rec = np.asarray(rec, dtype=np.float64)
    nv, nf, nw = rec.shape[:3]
    lam_t = np.broadcast_to(np.asarray(lam, dtype=np.float64)[None, None, :], (nv, nf, nw)).ravel()
    st = E.wavefront_statistics(rec.reshape(-1, rec.shape[-1]), lam_t)
    rms = st['rms_focus' if compensate_focus else 'rms_tilt'].reshape(nv, nf, nw)
    merit, sigma = wave_merit_of(rms, wvl_wts, field_wts)
    cs = np.zeros((nv, nf, nw), dtype=np.int32) if chief_status is None else np.asarray(chief_status)
    return WaveMerit(merit, sigma, rec[..., 0].sum(axis=2), rms, st['focus'].reshape(nv, nf, nw), cs)


class Sensitivity:
    """Result of ``tolerance_sensitivity``.  ``nominal`` / ``nominal_focus``: M and delta* of the
    nominal system; per tolerance ``merit_plus`` / ``merit_minus`` (at +-delta), ``delta_plus`` /
    ``delta_minus`` (their change of M), ``focus_plus`` / ``focus_minus``; ``estimated`` = M0 +
    sqrt(sum_i max(dM_i+, dM_i-, 0)^2); ``result``: the ``TolMerit`` of every variant (0 nominal,
    then +delta, -delta per tolerance).  With the wavefront criterion ``result`` is a ``WaveMerit``,
    the focus values are its per-tile ``focus`` coefficients and, since wavefront variances add,
    ``estimated`` = sqrt(M0^2 + sum_i max(M_i+^2 - M0^2, M_i-^2 - M0^2, 0))."""

    def __init__(self, tolerances, res):
        self.tolerances, self.result = list(tolerances), res
        if isinstance(res, WaveMerit):
            self._init_wave(res)
            return
        self.nominal, self.nominal_focus = float(res.merit[0]), float(res.focus[0])
        self.merit_plus, self.merit_minus = res.merit[1::2].copy(), res.merit[2::2].copy()
        self.focus_plus, self.focus_minus = res.focus[1::2].copy(), res.focus[2::2].copy()
        self.delta_plus, self.delta_minus = self.merit_plus - self.nominal, self.merit_minus - self.nominal
        worst = np.maximum(np.maximum(self.delta_plus, self.delta_minus), 0.0)
        self.estimated = self.nominal + float(np.sqrt(np.sum(worst*worst)))

    def _init_wave(self, res):
        self.nominal, self.nominal_focus = float(res.merit[0]), res.focus[0].copy()
        self.merit_plus, self.merit_minus = res.merit[1::2].copy(), res.merit[2::2].copy()
        self.focus_plus, self.focus_minus = res.focus[1::2].copy(), res.focus[2::2].copy()
        self.delta_plus, self.delta_minus = self.merit_plus - self.nominal, self.merit_minus - self.nominal
        m2 = self.nominal*self.nominal
        worst = np.maximum(np.maximum(self.merit_plus*self.merit_plus - m2, self.merit_minus*self.merit_minus - m2),
                           0.0)
        self.estimated = float(np.sqrt(m2 + np.sum(worst)))


class MonteCarlo:
    """Result of ``tolerance_monte_carlo``: ``values`` ``[num_trials, n_tol]`` the drawn changes;
    ``merit`` / ``focus`` ``[num_trials]``; ``nominal``; ``mean``, ``std`` and ``percentiles``
    {50, 80, 90, 98: M} of the trials' merits; ``result``: the ``TolMerit`` (variant 0 nominal).  With
    the wavefront criterion ``result`` is a ``WaveMerit`` and ``focus`` its per-tile ``focus``
    coefficients ``[num_trials, n_fields, n_wvls]``."""

    def __init__(self, tolerances, values, res):
        self.tolerances, self.values, self.result = list(tolerances), values, res
        self.nominal = float(res.merit[0])
        self.merit, self.focus = res.merit[1:].copy(), res.focus[1:].copy()
        self.mean, self.std = float(np.mean(self.merit)), float(np.std(self.merit))
        self.percentiles = {p: float(np.percentile(self.merit, p)) for p in (50, 80, 90, 98)}


def draw_tolerances(tolerances, num_trials, seed=0, distribution='normal'):
    """``[num_trials, n_tol]`` changes, trial-major from ``Generator(PCG64(seed))``: 'normal' with
    sigma = delta/2, truncated to +-delta by drawing again; 'uniform' on [-delta, delta]"""
    if distribution not in ('normal', 'uniform'):
        raise ValueError(f'unknown distribution {distribution!r}')
    rng = np.random.Generator(np.random.PCG64(seed))
    out = np.zeros((int(num_trials), len(tolerances)))
    for t in range(int(num_trials)):
        for i, tol in enumerate(tolerances):
            dl = abs(float(tol.delta))
            if distribution == 'uniform':
                out[t, i] = rng.uniform(-dl, dl)
                continue
            v = rng.normal(0.0, dl/2.0)
            while abs(v) > dl:
                v = rng.normal(0.0, dl/2.0)
            out[t, i] = v
    return out


def _tol_records(opt_model, change_sets, num_rays, fields, wvls, foc, table, device, backend, trace_kwargs):
    """``[n_var, n_fields, n_wvls, RT_TOL_DOUBLES]`` records of the nominal grid for every change
    set, and the spectral / field weights"""
    from . import tolerance as TOL
    from .table import describe_model
    osp, sm = opt_model.optical_spec, opt_model.seq_model
    fields = list(osp.field_of_view.fields if fields is None else fields)
    wvls = list(sm.wvlns if wvls is None else wvls)
    foc = osp.defocus.focus_shift if foc is None else foc
    region = osp.spectral_region
    wvl_wts = [region.spectral_wts[list(region.wavelengths).index(w)] for w in wvls]
    field_wts = [f.wt for f in fields]
    descs, n_by_wvl, all_wvls = describe_model(sm)
    var = [TOL.perturbed_descriptors(descs, n_by_wvl, ch, sm) for ch in change_sets]
    nb = np.stack([v[1] for v in var])
    args, kw = E._grid_args(opt_model, sm.index_for_wavelength, num_rays, fields, wvls, foc, (-1.0, 1.0), True)
    cwl = sm.index_for_wavelength(sm.central_wavelength())
    trace_kwargs.setdefault('check_apertures', True)
    if backend is not None:
        spec = E.PupilGridSpec(*args, **kw)
        ref = backend.chief_ref(descs, n_by_wvl, spec, cwl)
        spec = E.PupilGridSpec(*args, ref_img=np.repeat(ref[:, None, :], len(wvls), axis=1), **kw)
        rec = np.asarray(backend.trace_variants([v[0] for v in var], nb, spec))
    else:
        tab = _table_for(opt_model, table, device)
        dev = torch.device('cuda', tab.device)
        with torch.cuda.device(dev):
            grid = E.PupilGrid(*args, device=tab.device, **kw)
            grid.chief_ref(tab, cwl)
            vs = E.VariantSet([v[0] for v in var], nb, all_wvls, device=tab.device)
            rec = E.trace_grid_variants(vs, grid, **trace_kwargs).cpu().numpy()     # waits
            vs.close()
            grid.close()
    return rec.reshape(len(change_sets), len(fields), len(wvls), -1), wvl_wts, field_wts


def _tol_wave_records(opt_model, change_sets, num_rays, fields, wvls, foc, table, device, backend, trace_kwargs):
    """``[n_var, n_fields, n_wvls, RT_WFE_DOUBLES]`` wavefront-error records of every change set on the grid
    of ``wavefront_error`` (each field's ``RayGrid`` samples, no vignetting, each wavelength referred to
    its own chief ray), each variant's wave records built on the device; the chief rays' status
    ``[n_var, n_fields, n_wvls]``, the wavelengths in system units and the spectral / field weights"""
    from . import tolerance as TOL
    from .table import describe_model
    osp, sm = opt_model.optical_spec, opt_model.seq_model
    fields = list(osp.field_of_view.fields if fields is None else fields)
    wvls = list(sm.wvlns if wvls is None else wvls)
    foc = osp.defocus.focus_shift if foc is None else foc
    region = osp.spectral_region
    wvl_wts = [region.spectral_wts[list(region.wavelengths).index(w)] for w in wvls]
    field_wts = [f.wt for f in fields]
    descs, n_by_wvl, all_wvls = describe_model(sm)
    var = [TOL.perturbed_descriptors(descs, n_by_wvl, ch, sm) for ch in change_sets]
    nb = np.stack([v[1] for v in var])
    fod = opt_model['analysis_results']['parax_data'].fod
    parax = (fod.exp_dist, abs(fod.n_obj), abs(fod.n_img))       # nominal, as perturbed_model keeps it
    trace_kwargs.setdefault('check_apertures', True)
    if backend is not None:
        args, kw = _wavefront_grid_args(opt_model, None, num_rays, fields, wvls, foc, None, None)
        spec = E.PupilGridSpec(*args, **kw)
        wave, _, status = backend.variant_waves([v[0] for v in var], nb, spec, parax)
        rec = np.asarray(backend.trace_variants_wfe([v[0] for v in var], nb, spec, np.asarray(wave)))
        status = np.asarray(status)
    else:
        tab = _table_for(opt_model, table, device)
        args, kw = _wavefront_grid_args(opt_model, tab, num_rays, fields, wvls, foc, None, None)
        dev = torch.device('cuda', tab.device)
        with torch.cuda.device(dev):
            grid = E.PupilGrid(*args, device=tab.device, **kw)
            vs = E.VariantSet([v[0] for v in var], nb, all_wvls, device=tab.device)
            wave, _, status = vs.wave(grid, parax)
            rec = E.trace_grid_variants_wfe(vs, grid, wave, **trace_kwargs).cpu().numpy()     # waits
            status = status.cpu().numpy()
            vs.close()
            grid.close()
    lam = [opt_model.nm_to_sys_units(w) for w in wvls]
    n, nf, nw = len(change_sets), len(fields), len(wvls)
    return rec.reshape(n, nf, nw, -1), status.reshape(n, nf, nw), lam, wvl_wts, field_wts


def _tol_result(opt_model, tolerances, sets, criterion, num_rays, fields, wvls, foc, compensate_focus, table,
                device, backend, trace_kwargs):
    """the TolMerit (spot) or WaveMerit (wavefront) of every change set"""
    from . import tolerance as TOL
    for t in tolerances:
        TOL.check(opt_model.seq_model, t, criterion)
    if criterion == 'wavefront':
        TOL.check_wavefront_model(opt_model.seq_model)
        rec, st, lam, ww, fw = _tol_wave_records(opt_model, sets, num_rays, fields, wvls, foc, table, device,
                                                 backend, trace_kwargs)
        return wave_merit(rec, lam, ww, fw, compensate_focus, st)
    rec, ww, fw = _tol_records(opt_model, sets, num_rays, fields, wvls, foc, table, device, backend, trace_kwargs)
    return tol_merit(rec, ww, fw, compensate_focus)


def tolerance_sensitivity(opt_model, tolerances, num_rays=32, fields=None, wvls=None, foc=None,
                          compensate_focus=True, table=None, device=0, backend=None, criterion='spot',
                          **trace_kwargs):
    """Change of the spot merit for each tolerance at +delta and -delta, from one grid trace of all
    variants (``rt_trace_grid_variants``; variant 0 nominal, then +delta, -delta per tolerance).

    The merit M is the field-weighted RMS over fields of the polychromatic (spectral weights) RMS spot
    radius about its centroid, on the nominal pupil grid with the nominal aim, referred to the nominal
    chief rays (DESIGN.md section 4); with ``compensate_focus`` each variant is refocused to the
    delta* that minimises M, solved in closed form from the device sums (no second trace).  The
    perturbed systems keep the nominal apertures, vignetting and aim (``tolerance.perturbed_model``).
    ``backend``: the CPU test seam, ``backend.trace_variants(descs, n_by_wvl, grid_spec)`` returning
    the records and ``backend.chief_ref(descs, n_by_wvl, grid_spec, wvl_idx)`` the reference points.

    ``criterion='wavefront'``: the merit is the field-weighted RMS over fields of the polychromatic
    (spectral weights) RMS wavefront error in waves (``wave_merit``), on the grid of ``wavefront_error``
    (``RayGrid`` samples over each field's vignetting box, no vignetting, apertures checked), each
    wavelength of each variant referred to that variant's own chief ray and reference sphere, built on
    the device (``rt_variants_wave``) and traced with the OPD epilogue in one launch per batch
    (``rt_trace_grid_variants_wfe``).  The focus compensator removes a focus term per (field,
    wavelength) tile, fitted on {1, x, y, r^2}: each tile is refocused on its own, which is more
    optimistic than the spot criterion's one common delta*.  Decenters and tilts of interface n_ifc - 2
    and models whose OPD cannot be evaluated are refused (``tolerance.check``).  ``backend`` then
    provides ``variant_waves(descs, n_by_wvl, grid_spec, parax)`` -> (wave, ref_img, status) and
    ``trace_variants_wfe(descs, n_by_wvl, grid_spec, wave)`` -> the records."""
    sets = [[]]
    for t in tolerances:
        sets += [[(t, float(t.delta))], [(t, -float(t.delta))]]
    return Sensitivity(tolerances, _tol_result(opt_model, tolerances, sets, criterion, num_rays, fields, wvls, foc,
                                               compensate_focus, table, device, backend, trace_kwargs))


def tolerance_monte_carlo(opt_model, tolerances, num_trials=1000, seed=0, distribution='normal', num_rays=32,
                          fields=None, wvls=None, foc=None, compensate_focus=True, table=None, device=0,
                          backend=None, criterion='spot', **trace_kwargs):
    """Spot (or, with ``criterion='wavefront'``, RMS wavefront error) merit of ``num_trials`` randomly
    built systems: every trial draws every tolerance (``draw_tolerances``), and all trials (with the
    nominal system as variant 0) are traced over the nominal grid in one launch per batch.  Merit,
    criterion, focus compensation and ``backend`` as ``tolerance_sensitivity``.  The same seed gives
    the same result."""
    from . import tolerance as TOL
    for t in tolerances:
        TOL.check(opt_model.seq_model, t, criterion)
    values = draw_tolerances(tolerances, num_trials, seed, distribution)
    sets = [[]] + [list(zip(tolerances, row)) for row in values]
    return MonteCarlo(tolerances, values, _tol_result(opt_model, tolerances, sets, criterion, num_rays, fields, wvls,
                                                      foc, compensate_focus, table, device, backend, trace_kwargs))
