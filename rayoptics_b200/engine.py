"""Ray bundles and pupil grids on the GPU: PyTorch tensors in, C-ABI calls out.

PyTorch is plumbing here (device memory, streams); every ray is traced by the
hand-written sm_90a kernels in csrc/ through ``rt_trace_bundle`` /
``rt_trace_grid`` (include/b200rt.h).  Ray bundles are structure-of-arrays:
``p`` and ``d`` are ``[3, n]`` float64 tensors (row c = component c), so each
component is a contiguous array and every warp load/store is coalesced.

Replaces the per-ray Python loops of the reference:
``trace_list_of_rays`` (/root/reference/src/rayoptics/raytr/analyses.py:458-510),
``trace_grid`` (raytr/trace.py:563-605), ``trace_ray_grid`` (analyses.py:666-696).
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np
import torch

from . import _abi
from ._abi import (rt_out, rt_grid_spec, rt_field_desc, RT_SEG_DOUBLES, RT_SUMMARY_DOUBLES, RT_WFE_DOUBLES,
                   RT_ZERN_DOUBLES, RT_ZERN_MAX_TERMS, RT_MTF_DOUBLES, RT_MTF_MAX_RAYS, RT_SPHERE_DOUBLES,
                   RT_TOL_DOUBLES, RT_WAVE_DOUBLES, RT_ILLUM_DOUBLES, RT_ILLUM_MAX_RAYS)

SUMMARY_FIELDS = ('n_ok', 'n_missed', 'n_tir', 'n_blocked', 'n_other',
                  'sum_x', 'sum_y', 'sum_xx', 'sum_yy', 'sum_xy',
                  'min_x', 'max_x', 'min_y', 'max_y', 'sum_op', 'reserved')
# columns of a wavefront-error record (RT_WFE_DOUBLES, include/b200rt.h): W = OPD in system units,
# (x, y) relative pupil coordinates, r2 = x*x + y*y
WFE_FIELDS = ('n_ok', 'n_missed', 'n_tir', 'n_blocked', 'n_other', 'min_w', 'max_w',
              'sum_w', 'sum_ww', 'sum_xw', 'sum_yw', 'sum_r2w',
              'sum_x', 'sum_y', 'sum_xx', 'sum_xy', 'sum_yy', 'sum_xr2', 'sum_yr2', 'sum_r2r2',
              'reserved0', 'reserved1', 'reserved2', 'reserved3')
# min / max columns of the two record layouts, by record width
_MINMAX_COLS = {RT_SUMMARY_DOUBLES: ((10, 12), (11, 13)), RT_WFE_DOUBLES: ((5,), (6,)),
                RT_ZERN_DOUBLES: ((6,), (7,))}
_COMBINE_FN = {RT_SUMMARY_DOUBLES: 'rt_combine_summaries', RT_WFE_DOUBLES: 'rt_combine_wfe',
               RT_ZERN_DOUBLES: 'rt_combine_zernike'}


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream_ptr(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _as_soa(x, device, name):
    """[3, n] float64 device tensor (rows contiguous)."""
    if isinstance(x, (tuple, list)) and len(x) == 3 and torch.is_tensor(x[0]):
        x = torch.stack([xi.to(device=device, dtype=torch.float64) for xi in x])
    elif not torch.is_tensor(x):
        x = torch.as_tensor(np.ascontiguousarray(x, dtype=np.float64))
    if x.dim() != 2:
        raise ValueError(f'{name} must be 2-D')
    if x.shape[0] != 3 and x.shape[1] == 3:
        x = x.t()
    if x.shape[0] != 3:
        raise ValueError(f'{name} must have shape [3, n] or [n, 3]')
    return x.to(device=device, dtype=torch.float64).contiguous()


BUNDLE_OUTPUTS = ('p', 'd', 'nrml', 'dst', 'op', 'status', 'fail_surf', 'n_seg')
GRID_OUTPUTS = ('p', 'd', 'op', 'status', 'fail_surf', 'abr')


class BundleResult:
    """Structure-of-arrays result of a bundle / grid trace (device tensors).

    ``p``, ``d``, ``nrml``: ``[3, n]`` last ray segment (``ray[-1]`` of the
    reference's RayPkg); ``dst``, ``op``: ``[n]``; ``status``, ``fail_surf``,
    ``n_seg``: ``[n]`` int32; ``full``: ``[n_ifc, 10, n]`` whole rays;
    ``abr``: ``[2, n]`` transverse aberration (grid traces).  Only the
    ``outputs`` asked for are allocated and written (others are None)."""

    def __init__(self, n, n_ifc, device, outputs=BUNDLE_OUTPUTS, nan_status=False):
        self.nan_status = bool(nan_status)     # RT_OUT_ABR_NAN_STATUS: status / fail_surf ride in abr's NaNs
        f64 = dict(dtype=torch.float64, device=device)
        i32 = dict(dtype=torch.int32, device=device)
        want = set(outputs)
        unknown = want - set(BUNDLE_OUTPUTS) - {'full', 'abr', 'opd'}
        if unknown:
            raise ValueError(f'unknown outputs {sorted(unknown)}')
        self.n = n
        self.p = torch.empty((3, n), **f64) if 'p' in want else None
        self.d = torch.empty((3, n), **f64) if 'd' in want else None
        self.nrml = torch.empty((3, n), **f64) if 'nrml' in want else None
        self.dst = torch.empty(n, **f64) if 'dst' in want else None
        self.op = torch.empty(n, **f64) if 'op' in want else None
        self.status = torch.empty(n, **i32) if 'status' in want else None
        self.fail_surf = torch.empty(n, **i32) if 'fail_surf' in want else None
        self.n_seg = torch.empty(n, **i32) if 'n_seg' in want else None
        self.full = (torch.full((n_ifc, RT_SEG_DOUBLES, n), float('nan'), **f64)
                     if 'full' in want else None)
        self.abr = torch.empty((2, n), **f64) if 'abr' in want else None
        self.opd = torch.empty(n, **f64) if 'opd' in want else None
        self.summary = None

    def c_struct(self):
        o = rt_out()
        if self.p is not None:
            o.px, o.py, o.pz = (_ptr(self.p[i]) for i in range(3))
        if self.d is not None:
            o.dx, o.dy, o.dz = (_ptr(self.d[i]) for i in range(3))
        if self.nrml is not None:
            o.nx, o.ny, o.nz = (_ptr(self.nrml[i]) for i in range(3))
        o.dst, o.op = _ptr(self.dst), _ptr(self.op)
        o.status, o.fail_surf, o.n_seg = _ptr(self.status), _ptr(self.fail_surf), _ptr(self.n_seg)
        if self.full is not None:
            o.full = _ptr(self.full)
            o.full_stride = self.n
        if self.abr is not None:
            o.abr_x, o.abr_y = _ptr(self.abr[0]), _ptr(self.abr[1])
        o.opd = _ptr(self.opd)
        o.flags = _abi.RT_OUT_ABR_NAN_STATUS if self.nan_status else 0
        return o

    def bytes_per_ray(self):
        """bytes the kernel writes per ray for the allocated outputs"""
        b = 0
        for t in (self.p, self.d, self.nrml, self.abr, self.dst, self.op, self.status,
                  self.fail_surf, self.n_seg, self.opd):
            if t is not None:
                b += t.element_size()*(t.numel()//max(self.n, 1))
        return b

    def ok(self):
        return self.status == 0


def trace_bundle(table, p, d, wvl_idx=None, full=False, outputs=BUNDLE_OUTPUTS, **kwargs):
    """Trace ``n`` rays given start points / direction cosines in the object
    interface's coordinates.  ``kwargs`` are trace_raw's keyword arguments
    (eps, check_apertures, intersect_obj, filter_out_phantoms, first_surf,
    last_surf, pt_inside_fuzz) plus ``wvl`` / ``wvl_index`` for a
    single-wavelength bundle.  Asynchronous on the current CUDA stream."""
    lib = _abi.load_library()
    device = torch.device('cuda', table.device)
    p = _as_soa(p, device, 'p')
    d = _as_soa(d, device, 'd')
    n = p.shape[1]
    if d.shape[1] != n:
        raise ValueError('p and d must hold the same number of rays')
    wi = 0
    if 'wvl' in kwargs:
        wi = table.wvl_index(kwargs.pop('wvl'))
    wi = kwargs.pop('wvl_index', wi)
    opts = _abi.make_opts(wvl_idx=wi, **kwargs)
    if wvl_idx is not None:
        wvl_idx = torch.as_tensor(wvl_idx).to(device=device, dtype=torch.int32).contiguous()
        if wvl_idx.numel() != n:
            raise ValueError('wvl_idx must hold one entry per ray')
    res = BundleResult(n, table.n_ifc, device, tuple(outputs) + (('full',) if full else ()))
    out = res.c_struct()
    _abi.check(lib.rt_trace_bundle(table.handle, n, _ptr(p[0]), _ptr(p[1]), _ptr(p[2]),
                                   _ptr(d[0]), _ptr(d[1]), _ptr(d[2]), _ptr(wvl_idx),
                                   C.byref(opts), C.byref(out), _stream_ptr(device)))
    res._keep = (p, d, wvl_idx)   # inputs must outlive the asynchronous launch
    return res


def accumulated_steps(start, stop, num):
    """The reference's pupil sampling: ``start += step`` repeated (NOT linspace),
    /root/reference/src/rayoptics/raytr/trace.py:567-604."""
    return _accumulated_steps(float(start), float(stop), int(num)).copy()


@functools.lru_cache(maxsize=64)
def _accumulated_steps(start, stop, num):
    vals = np.empty(num)
    step = np.array((np.float64(stop) - np.float64(start))/(num - 1)) if num > 1 else np.float64(0.)
    x = np.float64(start)
    for i in range(num):
        vals[i] = x
        x = x + step
    return vals


def chunk_rays():
    """rays per chunk = threads per CTA of the loaded library (``rt_chunk_rays``; 256)"""
    return int(_abi.load_library().rt_chunk_rays())



class PupilGridSpec:
    """Host-side description of fields x wavelengths x (nx x ny) pupil rays
    (the arrays behind ``rt_grid_spec``; no CUDA involved).

    ``fields``: list of dicts / objects with ``pt0`` (3), ``aim`` (2), ``vlx,
    vux, vly, vuy`` (and optionally ``pupil_kind``, see ``rt_pupil_kind``: for the
    angular kinds ``pt0`` is the object point, ``aim`` the chief-ray direction
    cosines and ``eprad`` the sine / slope scale); ``pupil_x`` / ``pupil_y``: ``[n_fields, nx]`` / ``[n_fields,
    ny]`` relative pupil coordinates before vignetting (or 1-D, shared by all
    fields); ``wvl_idx``: rows of the table's index table; ``ref_img``:
    ``[n_fields, n_wvls, 2]`` reference image points or None."""

    def __init__(self, fields, wvl_idx, pupil_x, pupil_y, eprad, z_pupil, ref_img=None,
                 apply_vignetting=True, flip_z_dir=1, foc=0.0, paired=False, wave=None,
                 pupil_kind=None):
        nf = len(fields)
        if pupil_kind is None:      # records of OpticalSpecs.grid_fields carry it
            f0 = fields[0]
            pupil_kind = f0.get('pupil_kind', 0) if isinstance(f0, dict) else getattr(f0, 'pupil_kind', 0)
        self.pupil_kind = int(pupil_kind)
        self.paired = int(bool(paired))
        self.n_fields = nf
        self.wvl_idx = np.ascontiguousarray(wvl_idx, dtype=np.int32)
        self.n_wvls = len(self.wvl_idx)
        px = np.ascontiguousarray(pupil_x, dtype=np.float64)
        py = np.ascontiguousarray(pupil_y, dtype=np.float64)
        if px.ndim == 1:
            px = np.ascontiguousarray(np.broadcast_to(px, (nf, px.shape[0])))
        if py.ndim == 1:
            py = np.ascontiguousarray(np.broadcast_to(py, (nf, py.shape[0])))
        self.pupil_x, self.pupil_y = px, py
        self.nx, self.ny = px.shape[1], py.shape[1]
        if self.paired:          # ray list: (pupil_x[i], pupil_y[i]), one "row" of nx rays
            if py.shape[1] != px.shape[1]:
                raise ValueError('paired pupil lists need as many y as x coordinates')
            self.ny = 1
        self.fields = (rt_field_desc*nf)()
        for i, f in enumerate(fields):
            get = (lambda k, f=f: f[k]) if isinstance(f, dict) else (lambda k, f=f: getattr(f, k))
            for c in range(3):
                self.fields[i].pt0[c] = float(get('pt0')[c])
            for c in range(2):
                self.fields[i].aim[c] = float(get('aim')[c])
            for k in ('vlx', 'vux', 'vly', 'vuy'):
                setattr(self.fields[i], k, float(get(k)))
            if self.pupil_kind == _abi.PUPIL_WIDE:
                rot = np.asarray(get('rot'), dtype=float).reshape(9)
                for c in range(9):
                    self.fields[i].rot[c] = float(rot[c])
                self.fields[i].obj2enp = float(get('obj2enp'))
        self.ref_img = None
        if ref_img is not None:
            self.ref_img = np.ascontiguousarray(ref_img, dtype=np.float64).reshape(nf, self.n_wvls, 2)
        self.wave = None
        if wave is not None:
            self.wave = np.ascontiguousarray(wave, dtype=np.float64).reshape(
                nf, self.n_wvls, _abi.RT_WAVE_DOUBLES)
        self.eprad, self.z_pupil, self.foc = float(eprad), float(z_pupil), float(foc)
        # wide-angle fields: no virtual-object flip (trace.py:299-303)
        self.apply_vignetting = int(bool(apply_vignetting))
        self.flip_z_dir = 0 if self.pupil_kind == _abi.PUPIL_WIDE else int(flip_z_dir)
        self.chunk_rays = chunk_rays()
        self.rays_per_tile = self.nx*self.ny
        self.n_tiles = self.n_fields*self.n_wvls
        self.chunks_per_tile = (self.rays_per_tile + self.chunk_rays - 1)//self.chunk_rays
        self.n_chunks = self.n_tiles*self.chunks_per_tile
        self.n_rays = self.n_tiles*self.rays_per_tile

    def host_bytes(self):
        """bytes rt_grid_create copies to the device"""
        return (C.sizeof(rt_field_desc)*self.n_fields + self.wvl_idx.nbytes + self.pupil_x.nbytes
                + self.pupil_y.nbytes + (0 if self.ref_img is None else self.ref_img.nbytes)
                + (0 if self.wave is None else self.wave.nbytes))

    def c_spec(self):
        """The rt_grid_spec (host pointers into arrays owned by this object)."""
        s = rt_grid_spec()
        s.n_fields, s.n_wvls, s.nx, s.ny = self.n_fields, self.n_wvls, self.nx, self.ny
        s.fields = C.cast(self.fields, C.POINTER(rt_field_desc))
        s.wvl_idx = self.wvl_idx.ctypes.data_as(_abi.c_int32_p)
        s.pupil_x = self.pupil_x.ctypes.data_as(_abi.c_double_p)
        s.pupil_y = self.pupil_y.ctypes.data_as(_abi.c_double_p)
        s.ref_img = None if self.ref_img is None else self.ref_img.ctypes.data_as(_abi.c_double_p)
        s.wave = None if self.wave is None else self.wave.ctypes.data_as(_abi.c_double_p)
        s.apply_vignetting, s.flip_z_dir = self.apply_vignetting, self.flip_z_dir
        s.paired = self.paired
        s.pupil_kind = self.pupil_kind
        s.eprad, s.z_pupil, s.foc = self.eprad, self.z_pupil, self.foc
        return s

    def first_ray_of_chunk(self, chunk):
        tile, lc = divmod(chunk, self.chunks_per_tile)
        return tile*self.rays_per_tile + min(lc*self.chunk_rays, self.rays_per_tile)

    def rays_in_chunks(self, chunk_begin, chunk_end):
        return self.first_ray_of_chunk(chunk_end) - self.first_ray_of_chunk(chunk_begin)


class PupilGrid(PupilGridSpec):
    """A PupilGridSpec uploaded to the device (``rt_grid*``)."""

    def __init__(self, *args, device=0, **kwargs):
        super().__init__(*args, **kwargs)
        lib = _abi.load_library()
        self.device = int(device)
        spec = self.c_spec()
        handle = C.c_void_p()
        _abi.check(lib.rt_grid_create(C.byref(spec), self.device, C.byref(handle)))
        self._handle, self._lib = handle, lib
        n_rays, n_chunks, chunk = C.c_int64(), C.c_int64(), C.c_int32()
        _abi.check(lib.rt_grid_dims(handle, C.byref(n_rays), C.byref(n_chunks), C.byref(chunk)))
        assert (n_rays.value, n_chunks.value, chunk.value) == (self.n_rays, self.n_chunks,
                                                              self.chunk_rays)

    @property
    def handle(self):
        if self._handle is None:
            raise RuntimeError('PupilGrid was destroyed')
        return self._handle

    def shape_key(self):
        return (self.device, self.n_fields, self.n_wvls, self.nx, self.ny, self.paired,
                self.wave is not None)

    def update(self, *args, **kwargs):
        """Replace the description by another one of the same shape (``rt_grid_update``: one
        asynchronous copy on the current stream, no allocation).  Arguments as the constructor."""
        kwargs.pop('device', None)
        old = self.shape_key()
        PupilGridSpec.__init__(self, *args, **kwargs)
        if self.shape_key() != old:
            raise ValueError('PupilGrid.update: the new description has a different shape')
        spec = self.c_spec()
        with torch.cuda.device(self.device):
            _abi.check(self._lib.rt_grid_update(self.handle, C.byref(spec),
                                                _stream_ptr(torch.device('cuda', self.device))))
        return self

    def upload(self, spec):
        """``rt_grid_update`` from a PupilGridSpec built earlier (same shape)."""
        c = spec.c_spec()
        with torch.cuda.device(self.device):
            _abi.check(self._lib.rt_grid_update(self.handle, C.byref(c),
                                                _stream_ptr(torch.device('cuda', self.device))))
        self.foc, self.apply_vignetting = spec.foc, spec.apply_vignetting
        return self

    def chief_ref(self, table, wvl_idx, out=None):
        """Reference image points = image intercepts of the chief rays at row ``wvl_idx`` of
        the table, computed and stored on the device (``rt_grid_chief_ref``); ``out``:
        optional ``[n_fields, 2]`` float64 device tensor that receives a copy."""
        with torch.cuda.device(self.device):
            _abi.check(self._lib.rt_grid_chief_ref(table.handle, self.handle, int(wvl_idx), _ptr(out),
                                                   _stream_ptr(torch.device('cuda', self.device))))
        return out

    def chief_ref_focus(self, table, wvl_idx, foc, out=None):
        """The chief rays of ``chief_ref``, their image intercepts defocused to every focus shift
        of ``foc`` (``rt_grid_chief_ref_focus``): ``[K, n_fields, 2]`` float64 device tensor
        (``out`` if given).  The grid's own reference points are not changed."""
        foc = _focus_array(foc)
        if out is None:
            out = torch.empty((len(foc), self.n_fields, 2), dtype=torch.float64,
                              device=torch.device('cuda', self.device))
        with torch.cuda.device(self.device):
            _abi.check(self._lib.rt_grid_chief_ref_focus(
                table.handle, self.handle, int(wvl_idx), foc.ctypes.data_as(_abi.c_double_p), len(foc),
                _ptr(out), _stream_ptr(torch.device('cuda', self.device))))
        return out

    def close(self):
        if getattr(self, '_handle', None) is not None:
            self._lib.rt_grid_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def trace_grid(table, grid, chunk_begin=0, chunk_end=None, outputs=GRID_OUTPUTS, full=False,
               summary=True, res=None, nan_status=False, **kwargs):
    """Trace chunks ``[chunk_begin, chunk_end)`` of a PupilGrid.

    Returns a BundleResult whose per-ray tensors (``outputs``; pass ``()`` for
    summary-only, ``res=`` to reuse buffers) cover the rays of those chunks in flattened (field, wvl, i, j) order and whose
    ``summary`` is the ``[n_tiles, 16]`` partial per-(field, wvl) spot sums
    (SUMMARY_FIELDS).  Defaults follow the grid analyses of the reference:
    ``check_apertures=True`` (trace.py:583), ``first_surf=1``,
    ``last_surf=n_ifc-2`` (raytrace.py:77-79)."""
    lib = _abi.load_library()
    device = torch.device('cuda', table.device)
    if chunk_end is None:
        chunk_end = grid.n_chunks
    kwargs.setdefault('check_apertures', True)
    kwargs.setdefault('first_surf', 1)
    kwargs.setdefault('last_surf', table.n_ifc - 2)
    if grid.pupil_kind == _abi.PUPIL_WIDE:
        kwargs['intersect_obj'] = False          # trace_base, trace.py:299-300
    opts = _abi.make_opts(**kwargs)
    n = grid.rays_in_chunks(chunk_begin, chunk_end)
    if res is None:
        res = BundleResult(n, table.n_ifc, device, tuple(outputs) + (('full',) if full else ()),
                           nan_status=nan_status)
    elif res.n != n:
        raise ValueError('res was allocated for a different number of rays')
    out = res.c_struct()
    summ = scratch = None
    if summary:
        summ = torch.empty((grid.n_tiles, RT_SUMMARY_DOUBLES), dtype=torch.float64, device=device)
        nbytes = lib.rt_grid_scratch_bytes(grid.handle, chunk_begin, chunk_end)
        scratch = torch.empty(max(nbytes//8, 1), dtype=torch.float64, device=device)
    _abi.check(lib.rt_trace_grid(table.handle, grid.handle, chunk_begin, chunk_end,
                                 C.byref(opts), C.byref(out), _ptr(summ), _ptr(scratch),
                                 _stream_ptr(device)))
    res.summary = summ
    res._keep = scratch
    return res


def _focus_array(foc):
    return np.ascontiguousarray(np.atleast_1d(np.asarray(foc, dtype=np.float64)).ravel())


def trace_grid_focus(table, grid, foc, chunk_begin=0, chunk_end=None, ref_img=None, res=None, **kwargs):
    """Spot sums of chunks ``[chunk_begin, chunk_end)`` of a PupilGrid at every focus shift of
    ``foc`` from one trace (``rt_trace_grid_focus``): ``[K, n_tiles, 16]`` float64 device tensor
    whose row k is the ``trace_grid`` summary of the grid with ``foc = foc[k]``.  ``ref_img``:
    ``[K, n_fields, 2]`` device tensor of reference image points per plane (``chief_ref_focus``)
    or None (= 0).  ``res``: optional BundleResult that receives the per-ray ``p``, ``d``,
    ``op``, ``status``, ``fail_surf``, ``n_seg`` (the aberrations depend on the plane and are not
    written).  Trace defaults as ``trace_grid``.  Asynchronous on the current CUDA stream."""
    lib = _abi.load_library()
    device = torch.device('cuda', table.device)
    foc = _focus_array(foc)
    if chunk_end is None:
        chunk_end = grid.n_chunks
    kwargs.setdefault('check_apertures', True)
    kwargs.setdefault('first_surf', 1)
    kwargs.setdefault('last_surf', table.n_ifc - 2)
    if grid.pupil_kind == _abi.PUPIL_WIDE:
        kwargs['intersect_obj'] = False
    opts = _abi.make_opts(**kwargs)
    if res is None:
        res = BundleResult(0, table.n_ifc, device, ())
    elif res.n != grid.rays_in_chunks(chunk_begin, chunk_end):
        raise ValueError('res was allocated for a different number of rays')
    out = res.c_struct()
    if ref_img is not None:
        if tuple(ref_img.shape) != (len(foc), grid.n_fields, 2) or ref_img.dtype != torch.float64 \
                or ref_img.device != device or not ref_img.is_contiguous():
            raise ValueError('ref_img must be a contiguous float64 [K, n_fields, 2] tensor on the table\'s device')
    summ = torch.empty((len(foc), grid.n_tiles, RT_SUMMARY_DOUBLES), dtype=torch.float64, device=device)
    nbytes = lib.rt_grid_focus_scratch_bytes(grid.handle, len(foc), chunk_begin, chunk_end)
    scratch = torch.empty(max(nbytes//8, 1), dtype=torch.float64, device=device)
    _abi.check(lib.rt_trace_grid_focus(table.handle, grid.handle, chunk_begin, chunk_end, C.byref(opts),
                                       foc.ctypes.data_as(_abi.c_double_p), len(foc), _ptr(ref_img),
                                       C.byref(out), _ptr(summ), _ptr(scratch), _stream_ptr(device)))
    summ._keep = (scratch, ref_img)      # inputs / scratch must outlive the asynchronous launches
    return summ


def trace_grid_to_host(table, grid, h_abr, chunk_begin=0, chunk_end=None, pieces=8, summary=True,
                       workspace=None, **kwargs):
    """Trace chunks ``[chunk_begin, chunk_end)`` of a PupilGrid and deliver the transverse
    aberrations to page-locked HOST memory (``rt_trace_grid_to_host``): ``pieces`` launches on
    two library-owned streams, each followed by its device->host copy.  ``h_abr``: pinned
    ``[2, >= n]`` float64 tensor; rays that do not reach the image hold NaNs coding status /
    failing surface (``decode_nan_status``).  Returns ``(summary [n_tiles, 16] device tensor or
    None, workspace)``; pass ``workspace`` back in to re-use the device staging buffers.
    Asynchronous: synchronise the current stream before reading ``h_abr``."""
    lib = _abi.load_library()
    device = torch.device('cuda', table.device)
    if chunk_end is None:
        chunk_end = grid.n_chunks
    kwargs.setdefault('check_apertures', True)
    kwargs.setdefault('first_surf', 1)
    kwargs.setdefault('last_surf', table.n_ifc - 2)
    if grid.pupil_kind == _abi.PUPIL_WIDE:
        kwargs['intersect_obj'] = False
    opts = _abi.make_opts(**kwargs)
    n = grid.rays_in_chunks(chunk_begin, chunk_end)
    if not (h_abr.is_pinned() and h_abr.dtype == torch.float64 and h_abr.shape[0] == 2
            and h_abr.shape[1] >= n and h_abr.stride(1) == 1):
        raise ValueError('h_abr must be a pinned float64 tensor [2, >= n] with contiguous rows')
    pieces = max(1, min(int(pieces), chunk_end - chunk_begin))
    nbytes = lib.rt_trace_grid_to_host_scratch_bytes(grid.handle, pieces)
    ws = workspace
    if ws is None or ws['abr'].shape[1] < n or ws['scratch'].numel()*8 < nbytes or ws['device'] != device:
        ws = {'abr': torch.empty((2, max(n, 1)), dtype=torch.float64, device=device),
              'scratch': torch.empty(max(nbytes//8, 1), dtype=torch.float64, device=device),
              'device': device}
    summ = (torch.empty((grid.n_tiles, RT_SUMMARY_DOUBLES), dtype=torch.float64, device=device)
            if summary else None)
    _abi.check(lib.rt_trace_grid_to_host(table.handle, grid.handle, chunk_begin, chunk_end, C.byref(opts),
                                         _ptr(ws['abr'][0]), _ptr(ws['abr'][1]), _ptr(h_abr[0]),
                                         _ptr(h_abr[1]), _ptr(summ), _ptr(ws['scratch']), pieces,
                                         _stream_ptr(device)))
    return summ, ws


def decode_nan_status(abr):
    """``(status, fail_surf)`` int32 arrays from an ``abr`` ``[2, n]`` array written with
    ``nan_status=True`` (numpy, host): rays that reach the image have finite aberrations and
    status 0 / fail_surf -1; the others carry both numbers in the NaN payloads."""
    bits = np.ascontiguousarray(abr).view(np.uint64)
    bad = np.isnan(abr[0])
    status = np.where(bad, bits[0] & np.uint64(0xFFFF), 0).astype(np.int32)
    fs = (bits[1] & np.uint64(0xFFFF)).astype(np.int32)
    fail_surf = np.where(bad, np.where(fs >= 0x8000, fs - 0x10000, fs), -1).astype(np.int32)
    return status, fail_surf


def combine_summaries(parts, out=None):
    """Combine partial ``[n_tiles, 16]`` spot summaries, ``[n_tiles, RT_WFE_DOUBLES]``
    wavefront-error records or ``[n_tiles, RT_ZERN_DOUBLES]`` Zernike moments records (from chunk
    ranges / ranks; the layout is chosen by ``shape[-1]``): sums add in part order, min/max columns
    take min/max.  CUDA tensors: one ``rt_combine_summaries`` / ``rt_combine_wfe`` /
    ``rt_combine_zernike`` launch on the current stream; CPU tensors (gloo tests): torch."""
    parts = torch.stack(list(parts)) if not torch.is_tensor(parts) else parts
    width = parts.shape[-1]
    if width not in _MINMAX_COLS:
        raise ValueError(f'unknown summary width {width}')
    if parts.is_cuda:
        parts = parts.contiguous()
        if out is None:
            out = torch.empty(parts.shape[1:], dtype=parts.dtype, device=parts.device)
        lib = _abi.load_library()
        fn = getattr(lib, _COMBINE_FN[width])
        with torch.cuda.device(parts.device):
            _abi.check(fn(_ptr(parts), parts.shape[0], parts.shape[1], _ptr(out), _stream_ptr(parts.device)))
        out._keep = parts
        return out
    out = parts.sum(dim=0)
    mins, maxs = _MINMAX_COLS[width]
    for k in mins:
        out[:, k] = parts[:, :, k].min(dim=0).values
    for k in maxs:
        out[:, k] = parts[:, :, k].max(dim=0).values
    return out


def spot_statistics(summary):
    """Per-(field, wvl) spot centroid and RMS radius from a combined summary
    (torch tensor or numpy array ``[n_tiles, 16]``; same type out)."""
    s = summary
    if torch.is_tensor(s):
        n = s[:, 0].clamp(min=1.0)
        sqrt0 = lambda v: v.clamp(min=0.0).sqrt()      # noqa: E731
    else:
        n = np.maximum(s[:, 0], 1.0)
        sqrt0 = lambda v: np.sqrt(np.maximum(v, 0.0))  # noqa: E731
    cx, cy = s[:, 5]/n, s[:, 6]/n
    var = (s[:, 7] + s[:, 8])/n - (cx*cx + cy*cy)
    return {'n_ok': s[:, 0], 'n_missed': s[:, 1], 'n_tir': s[:, 2], 'n_blocked': s[:, 3],
            'centroid_x': cx, 'centroid_y': cy, 'rms_radius': sqrt0(var),
            'min_x': s[:, 10], 'max_x': s[:, 11], 'min_y': s[:, 12], 'max_y': s[:, 13],
            'mean_op': s[:, 14]/n}


def trace_grid_wfe(table, grid, chunk_begin=0, chunk_end=None, res=None, **kwargs):
    """Wavefront-error sums of chunks ``[chunk_begin, chunk_end)`` of a PupilGrid built with
    ``wave=`` records (``rt_trace_grid_wfe``): ``[n_tiles, RT_WFE_DOUBLES]`` float64 device tensor
    (WFE_FIELDS; ``wavefront_statistics`` turns it into numbers).  ``res``: optional BundleResult
    that receives per-ray outputs as ``trace_grid`` writes them (``opd`` included; no whole rays).
    Trace defaults as ``trace_grid``.  Asynchronous on the current CUDA stream."""
    lib = _abi.load_library()
    device = torch.device('cuda', table.device)
    if chunk_end is None:
        chunk_end = grid.n_chunks
    kwargs.setdefault('check_apertures', True)
    kwargs.setdefault('first_surf', 1)
    kwargs.setdefault('last_surf', table.n_ifc - 2)
    if grid.pupil_kind == _abi.PUPIL_WIDE:
        kwargs['intersect_obj'] = False
    opts = _abi.make_opts(**kwargs)
    if res is None:
        res = BundleResult(0, table.n_ifc, device, ())
    elif res.n != grid.rays_in_chunks(chunk_begin, chunk_end):
        raise ValueError('res was allocated for a different number of rays')
    out = res.c_struct()
    summ = torch.empty((grid.n_tiles, RT_WFE_DOUBLES), dtype=torch.float64, device=device)
    nbytes = lib.rt_grid_wfe_scratch_bytes(grid.handle, chunk_begin, chunk_end)
    scratch = torch.empty(max(nbytes//8, 1), dtype=torch.float64, device=device)
    _abi.check(lib.rt_trace_grid_wfe(table.handle, grid.handle, chunk_begin, chunk_end, C.byref(opts),
                                     C.byref(out), _ptr(summ), _ptr(scratch), _stream_ptr(device)))
    summ._keep = scratch          # scratch must outlive the asynchronous launches
    return summ


WFE_STATISTICS = ('n_ok', 'n_missed', 'n_tir', 'n_blocked', 'n_other', 'rms', 'pv', 'rms_tilt', 'tilt_x',
                  'tilt_y', 'rms_focus', 'focus')


def _fit(gram, rhs, sum_ww, n):
    """Least-squares fit from the normal equations of one tile: ``(coefficients, RSS)``; NaN
    when there are fewer rays than basis functions or the Gram matrix is rank deficient"""
    p = len(rhs)
    nan = (np.full(p, np.nan), np.nan)
    if not (n >= p) or not np.isfinite(gram).all() or not np.isfinite(rhs).all():
        return nan
    d = np.sqrt(np.diag(gram))
    if not (d > 0).all():
        return nan
    scaled = gram/np.outer(d, d)             # unit diagonal: its condition number is the fit's
    ev = np.linalg.eigvalsh(scaled)
    if not ev[0] > p*np.finfo(np.float64).eps*ev[-1]:
        return nan
    c = np.linalg.solve(scaled, rhs/d)/d
    return c, sum_ww - float(np.dot(c, rhs))


def wavefront_statistics(summary, wvl_sys):
    """Per-tile wavefront error from combined ``[n_tiles, RT_WFE_DOUBLES]`` records (numpy array
    or torch tensor; same type out, on the same device).  ``wvl_sys``: the wavelength in system
    units (``opt_model.nm_to_sys_units(wvl)``), a scalar or one value per tile; every result is
    in waves.

    ``rms``: sqrt(sum W^2/n - (sum W/n)^2), piston removed; ``pv``: max W - min W;
    ``rms_tilt``, ``tilt_x``, ``tilt_y``: least-squares fit of W on {1, x, y}, its residual
    sqrt(RSS/n) with RSS = sum W^2 - c.b from the 3 x 3 normal equations; ``rms_focus``,
    ``focus``: the same on {1, x, y, r^2} (4 x 4).  Coefficients are in waves at unit relative
    pupil.  A fit with fewer rays than basis functions or a rank-deficient Gram matrix is NaN;
    a tile without a status-0 ray is NaN everywhere except the counts."""
    is_t = torch.is_tensor(summary)
    s = (summary.detach().cpu().numpy() if is_t else np.asarray(summary, dtype=np.float64)).reshape(-1, RT_WFE_DOUBLES)
    lam = np.broadcast_to(np.asarray(wvl_sys, dtype=np.float64).reshape(-1), (s.shape[0],))
    n = s[:, 0]
    out = {k: s[:, i].copy() for i, k in enumerate(WFE_STATISTICS[:5])}
    for k in WFE_STATISTICS[5:]:
        out[k] = np.full(s.shape[0], np.nan)
    for t in range(s.shape[0]):
        (nt, sw, sww, sxw, syw, sr2w, sx, sy, sxx, sxy, syy, sxr2, syr2, sr2r2) = \
            (s[t, 0],) + tuple(s[t, 7:20])
        if not nt > 0:
            continue
        lt = lam[t]
        with np.errstate(invalid='ignore'):
            mean = sw/nt
            out['rms'][t] = np.sqrt(max(sww/nt - mean*mean, 0.0))/lt if np.isfinite(sww) else np.nan
        out['pv'][t] = (s[t, 6] - s[t, 5])/lt
        sr2 = sxx + syy
        g3 = np.array([[nt, sx, sy], [sx, sxx, sxy], [sy, sxy, syy]])
        c3, rss3 = _fit(g3, np.array([sw, sxw, syw]), sww, nt)
        out['rms_tilt'][t] = np.sqrt(max(rss3, 0.0)/nt)/lt if np.isfinite(rss3) else np.nan
        out['tilt_x'][t], out['tilt_y'][t] = c3[1]/lt, c3[2]/lt
        g4 = np.array([[nt, sx, sy, sr2], [sx, sxx, sxy, sxr2], [sy, sxy, syy, syr2], [sr2, sxr2, syr2, sr2r2]])
        c4, rss4 = _fit(g4, np.array([sw, sxw, syw, sr2w]), sww, nt)
        out['rms_focus'][t] = np.sqrt(max(rss4, 0.0)/nt)/lt if np.isfinite(rss4) else np.nan
        out['focus'][t] = c4[3]/lt
    if is_t:
        return {k: torch.as_tensor(v, device=summary.device) for k, v in out.items()}
    return out


# --- Fringe Zernike fits (rt_grid_zernike; the polynomials of csrc/rt_zernike.cuh) --------------
# (n, m, 'cos' | 'sin' | None, integer coefficients of P from the constant term up), Fringe order:
# Z_j = R_n^m(rho) * cos | sin(m theta), R_n^m(rho) = rho^m * P(rho^2), theta from +x
FRINGE_TERMS = (
    (0, 0, None, (1,)), (1, 1, 'cos', (1,)), (1, 1, 'sin', (1,)), (2, 0, None, (-1, 2)),
    (2, 2, 'cos', (1,)), (2, 2, 'sin', (1,)), (3, 1, 'cos', (-2, 3)), (3, 1, 'sin', (-2, 3)),
    (4, 0, None, (1, -6, 6)), (3, 3, 'cos', (1,)), (3, 3, 'sin', (1,)), (4, 2, 'cos', (-3, 4)),
    (4, 2, 'sin', (-3, 4)), (5, 1, 'cos', (3, -12, 10)), (5, 1, 'sin', (3, -12, 10)),
    (6, 0, None, (-1, 12, -30, 20)), (4, 4, 'cos', (1,)), (4, 4, 'sin', (1,)), (5, 3, 'cos', (-4, 5)),
    (5, 3, 'sin', (-4, 5)), (6, 2, 'cos', (6, -20, 15)), (6, 2, 'sin', (6, -20, 15)),
    (7, 1, 'cos', (-4, 30, -60, 35)), (7, 1, 'sin', (-4, 30, -60, 35)), (8, 0, None, (1, -20, 90, -140, 70)),
    (5, 5, 'cos', (1,)), (5, 5, 'sin', (1,)), (6, 4, 'cos', (-5, 6)), (6, 4, 'sin', (-5, 6)),
    (7, 3, 'cos', (10, -30, 21)), (7, 3, 'sin', (10, -30, 21)), (8, 2, 'cos', (-10, 60, -105, 56)),
    (8, 2, 'sin', (-10, 60, -105, 56)), (9, 1, 'cos', (5, -60, 210, -280, 126)),
    (9, 1, 'sin', (5, -60, 210, -280, 126)), (10, 0, None, (-1, 30, -210, 560, -630, 252)),
    (12, 0, None, (1, -42, 420, -1680, 3150, -2772, 924)))
ZERN_HEAD = 9            # record columns before the packed Gram block (include/b200rt.h)


def zernike_terms(x, y, n_terms=RT_ZERN_MAX_TERMS):
    """``[..., n_terms]`` Fringe Zernike terms Z_1 ... Z_n_terms at relative pupil coordinates
    ``(x, y)``, bit for bit as the device evaluates them (csrc/rt_zernike.cuh): r2 = x*x + y*y;
    C1 = x, S1 = y, C(k+1) = C(k)*x - S(k)*y, S(k+1) = S(k)*x + C(k)*y; P by Horner in r2 from the
    highest coefficient; Z = P*C(m), P*S(m) or P.  Every product is rounded once."""
    if not 1 <= n_terms <= RT_ZERN_MAX_TERMS:
        raise ValueError(f'n_terms must be 1 ... {RT_ZERN_MAX_TERMS}')
    x, y = np.broadcast_arrays(np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64))
    with np.errstate(all='ignore'):
        r2 = x*x + y*y
        C, S = [None, x], [None, y]
        for k in range(1, 5):
            C.append(C[k]*x - S[k]*y)
            S.append(S[k]*x + C[k]*y)
        out = np.empty(x.shape + (n_terms,))
        for j, (n, m, kind, a) in enumerate(FRINGE_TERMS[:n_terms]):
            p = np.full(x.shape, float(a[-1]))
            for c in a[-2::-1]:
                p = p*r2 + float(c)
            out[..., j] = p if m == 0 else p*(S[m] if kind == 'sin' else C[m])
    return out


def zernike_gram_col(i, j):
    """record column of the Gram entry sum a_i*a_j (a_0 = W, a_k = Z_k; symmetric in i, j)"""
    i, j = min(i, j), max(i, j)
    return ZERN_HEAD + j*(j + 1)//2 + i


def zernike_gram(record, n_terms):
    """``[..., n_terms + 1, n_terms + 1]`` symmetric Gram matrices of [W, Z_1 ... Z_n_terms] from
    ``[..., RT_ZERN_DOUBLES]`` records"""
    s = np.asarray(record, dtype=np.float64)
    idx = np.array([[zernike_gram_col(i, j) for j in range(n_terms + 1)] for i in range(n_terms + 1)])
    return s[..., idx]


def grid_zernike(grid, chunk_begin, chunk_end, n_terms, status, opd):
    """``rt_grid_zernike``: the ``[n_tiles, RT_ZERN_DOUBLES]`` Zernike moments record (float64
    device tensor) of chunks ``[chunk_begin, chunk_end)`` of a product PupilGrid without vignetting,
    from the per-ray ``status`` (int32) and ``opd`` (float64, system units) device tensors of a grid
    trace over the same chunks.  Asynchronous on the current CUDA stream."""
    lib = _abi.load_library()
    n = grid.rays_in_chunks(chunk_begin, chunk_end)
    for t, dt, name in ((status, torch.int32, 'status'), (opd, torch.float64, 'opd')):
        if not (torch.is_tensor(t) and t.is_cuda and t.dtype == dt and t.is_contiguous() and t.numel() == n):
            raise ValueError(f'{name} must be a contiguous {dt} CUDA tensor of the {n} rays of the chunk range')
    device = status.device
    summ = torch.empty((grid.n_tiles, RT_ZERN_DOUBLES), dtype=torch.float64, device=device)
    nbytes = lib.rt_grid_zernike_scratch_bytes(grid.handle, chunk_begin, chunk_end, n_terms)
    scratch = torch.empty(max(nbytes//8, 1), dtype=torch.float64, device=device)
    with torch.cuda.device(device):
        _abi.check(lib.rt_grid_zernike(grid.handle, chunk_begin, chunk_end, n_terms, _ptr(status), _ptr(opd),
                                       _ptr(summ), _ptr(scratch), _stream_ptr(device)))
    summ._keep = (scratch, status, opd)        # must outlive the asynchronous launches
    return summ


def trace_grid_zernike(table, grid, n_terms, chunk_begin=0, chunk_end=None, res=None, **kwargs):
    """Zernike moments of chunks ``[chunk_begin, chunk_end)`` of a PupilGrid built with ``wave=``
    records: ``trace_grid`` with the ``opd`` and ``status`` outputs into device buffers (``res``:
    an optional BundleResult with both, which keeps them), then ``grid_zernike``.  Returns the
    ``[n_tiles, RT_ZERN_DOUBLES]`` device tensor.  Trace defaults as ``trace_grid``."""
    if chunk_end is None:
        chunk_end = grid.n_chunks
    n = grid.rays_in_chunks(chunk_begin, chunk_end)
    if res is None:
        res = BundleResult(n, table.n_ifc, torch.device('cuda', table.device), ('opd', 'status'))
    elif res.opd is None or res.status is None:
        raise ValueError('res needs the opd and status outputs')
    trace_grid(table, grid, chunk_begin, chunk_end, summary=False, res=res, **kwargs)
    summ = grid_zernike(grid, chunk_begin, chunk_end, n_terms, res.status, res.opd)
    summ._keep = (summ._keep, res)
    return summ


ZERN_STATISTICS = ('n_ok', 'n_missed', 'n_tir', 'n_blocked', 'n_other', 'n_used', 'rms', 'pv', 'rms_residual')


def zernike_statistics(summary, wvl_sys, n_terms):
    """Per-tile Fringe Zernike fit from combined ``[n_tiles, RT_ZERN_DOUBLES]`` records (numpy
    array or torch tensor; same type out, on the same device).  ``wvl_sys``: the wavelength in
    system units, a scalar or one value per tile; results in waves.

    ``coef`` ``[n_tiles, n_terms]``: least-squares coefficients of W on Z_1 ... Z_n_terms over the
    used rays (``_fit`` on the normal equations); ``rms_residual``: sqrt(RSS/n_used); ``rms``:
    sqrt(sum W^2/n - (sum W/n)^2), piston removed; ``pv``: max W - min W; the counts.  A fit with
    fewer used rays than terms or a rank-deficient scaled Gram matrix is NaN; a tile without a used
    ray is NaN everywhere except the counts."""
    if not 1 <= n_terms <= RT_ZERN_MAX_TERMS:
        raise ValueError(f'n_terms must be 1 ... {RT_ZERN_MAX_TERMS}')
    is_t = torch.is_tensor(summary)
    s = (summary.detach().cpu().numpy() if is_t else np.asarray(summary, dtype=np.float64)).reshape(-1, RT_ZERN_DOUBLES)
    nt = s.shape[0]
    lam = np.broadcast_to(np.asarray(wvl_sys, dtype=np.float64).reshape(-1), (nt,))
    out = {k: s[:, i].copy() for i, k in enumerate(ZERN_STATISTICS[:6])}
    for k in ZERN_STATISTICS[6:]:
        out[k] = np.full(nt, np.nan)
    out['coef'] = np.full((nt, n_terms), np.nan)
    gram = zernike_gram(s, n_terms)
    for t in range(nt):
        n = s[t, 5]
        if not n > 0:
            continue
        g, lt = gram[t], lam[t]
        sww = g[0, 0]
        with np.errstate(invalid='ignore'):
            mean = g[0, 1]/n
            out['rms'][t] = np.sqrt(max(sww/n - mean*mean, 0.0))/lt if np.isfinite(sww) else np.nan
        out['pv'][t] = (s[t, 7] - s[t, 6])/lt
        c, rss = _fit(g[1:, 1:], g[0, 1:], sww, n)
        out['coef'][t] = c/lt
        out['rms_residual'][t] = np.sqrt(max(rss, 0.0)/n)/lt if np.isfinite(rss) else np.nan
    if is_t:
        return {k: torch.as_tensor(v, device=summary.device) for k, v in out.items()}
    return out


def aim_chief_rays(table, grid, stop, wvl_idx, h, tol=1e-13, max_iter=30):
    """``rt_grid_aim_chief``: the aim point of every field of a PupilGrid ('epd' pupil), found on the
    device by the Newton iteration of ``vigcalc.aim_chief_ray`` (csrc/rt_aim.cuh) at row ``wvl_idx``
    of the table with stop interface ``stop`` and forward-difference step ``h``.  Returns the device
    tensors ``aim`` ``[n_fields, 2]`` float64 (the x == 0 rule of ``aim_chief_ray`` not applied) and
    ``term`` ``[n_fields]`` int32 (``rt_aim_term``).  One launch, asynchronous on the current CUDA
    stream; the grid's field records are not changed."""
    lib = _abi.load_library()
    device = torch.device('cuda', table.device)
    aim = torch.empty((grid.n_fields, 2), dtype=torch.float64, device=device)
    term = torch.empty(grid.n_fields, dtype=torch.int32, device=device)
    with torch.cuda.device(device):
        _abi.check(lib.rt_grid_aim_chief(table.handle, grid.handle, int(stop), int(wvl_idx), float(h), float(tol),
                                         int(max_iter), _ptr(aim), _ptr(term), _stream_ptr(device)))
    return aim, term


# --- diffraction MTF (rt_grid_pupil_function, rt_grid_mtf; the sums of csrc/rt_mtf.cuh) -----------
MTF_RECORD = ('n_ok', 'n_missed', 'n_tir', 'n_blocked', 'n_other', 'n_used', 'sum_re', 'sum_im')


def _ray_tensor(t, dt, n, name):
    if not (torch.is_tensor(t) and t.is_cuda and t.dtype == dt and t.is_contiguous() and t.numel() == n):
        raise ValueError(f'{name} must be a contiguous {dt} CUDA tensor of {n} entries')


def grid_pupil_function(grid, status, opd, wvl_sys, out=None):
    """``rt_grid_pupil_function``: ``(pupil, pupil_t)``, ``[n_tiles, n, n]`` complex128 device tensors
    of the pupil function exp(2 pi i opd/wvl_sys) of every tile of a square product PupilGrid without
    vignetting (0 where a ray is not used: status != 0 or x^2 + y^2 > 1), ``pupil_t`` transposed in
    each tile.  ``status`` (int32), ``opd`` (float64, system units): the per-ray device tensors of a
    grid trace over all chunks; ``wvl_sys``: the wavelength in system units, a scalar or one value per
    tile.  ``out``: an earlier call's ``(pupil, pupil_t)`` to write into.  Asynchronous on the current
    CUDA stream."""
    lib = _abi.load_library()
    _ray_tensor(status, torch.int32, grid.n_rays, 'status')
    _ray_tensor(opd, torch.float64, grid.n_rays, 'opd')
    device = status.device
    lam = np.broadcast_to(np.asarray(wvl_sys, dtype=np.float64).reshape(-1), (grid.n_tiles,))
    lam = torch.tensor(lam, device=device)
    shape = (grid.n_tiles, grid.nx, grid.ny)
    if out is None:
        pupil = torch.empty(shape, dtype=torch.complex128, device=device)
        pupil_t = torch.empty(shape, dtype=torch.complex128, device=device)
    else:
        pupil, pupil_t = out
        for t, name in ((pupil, 'pupil'), (pupil_t, 'pupil_t')):
            _ray_tensor(t, torch.complex128, grid.n_rays, name)
    with torch.cuda.device(device):
        _abi.check(lib.rt_grid_pupil_function(grid.handle, _ptr(status), _ptr(opd), _ptr(lam), _ptr(pupil),
                                              _ptr(pupil_t), _stream_ptr(device)))
    pupil._keep = (status, opd, lam)           # must outlive the asynchronous launch
    return pupil, pupil_t


def grid_mtf(grid, status, pupil, pupil_t):
    """``rt_grid_mtf``: ``(acf_x, acf_y, record)`` of ``grid_pupil_function``'s outputs:
    ``[n_tiles, n]`` complex128 autocorrelations along pupil x and y against the shift k, and the
    ``[n_tiles, RT_MTF_DOUBLES]`` record (``MTF_RECORD``: status counts, n_used, Re / Im of sum P).
    Asynchronous on the current CUDA stream."""
    lib = _abi.load_library()
    _ray_tensor(status, torch.int32, grid.n_rays, 'status')
    for t, name in ((pupil, 'pupil'), (pupil_t, 'pupil_t')):
        _ray_tensor(t, torch.complex128, grid.n_rays, name)
    device = status.device
    acf_x = torch.empty((grid.n_tiles, grid.nx), dtype=torch.complex128, device=device)
    acf_y = torch.empty((grid.n_tiles, grid.nx), dtype=torch.complex128, device=device)
    rec = torch.empty((grid.n_tiles, RT_MTF_DOUBLES), dtype=torch.float64, device=device)
    with torch.cuda.device(device):
        _abi.check(lib.rt_grid_mtf(grid.handle, _ptr(status), _ptr(pupil), _ptr(pupil_t), _ptr(acf_x),
                                   _ptr(acf_y), _ptr(rec), _stream_ptr(device)))
    rec._keep = (status, pupil, pupil_t)
    return acf_x, acf_y, rec


def trace_grid_mtf(table, grid, wvl_sys, res=None, **kwargs):
    """Autocorrelations of the pupil functions of every tile of a square PupilGrid built with
    ``wave=`` records: ``trace_grid`` over all chunks with the ``opd`` and ``status`` outputs into
    device buffers (``res``: an optional BundleResult with both, which keeps them), then
    ``grid_pupil_function`` and ``grid_mtf`` -- three launches.  Returns ``(acf_x, acf_y, record,
    pupil)`` device tensors.  Trace defaults as ``trace_grid``."""
    if res is None:
        res = BundleResult(grid.n_rays, table.n_ifc, torch.device('cuda', table.device), ('opd', 'status'))
    elif res.opd is None or res.status is None:
        raise ValueError('res needs the opd and status outputs')
    trace_grid(table, grid, 0, grid.n_chunks, summary=False, res=res, **kwargs)
    pupil, pupil_t = grid_pupil_function(grid, res.status, res.opd, wvl_sys)
    acf_x, acf_y, rec = grid_mtf(grid, res.status, pupil, pupil_t)
    rec._keep = (rec._keep, res)
    return acf_x, acf_y, rec, pupil


def grid_mtf_shifts(grid, status, pupil, pupil_t, shifts):
    """``rt_grid_mtf_shifts``: ``grid_mtf`` at the listed shifts only -- ``(acf_x, acf_y, record)`` with
    ``acf_x``, ``acf_y`` ``[n_tiles, len(shifts)]`` complex128, entry m bit for bit ``grid_mtf``'s entry
    ``shifts[m]``.  ``shifts``: integers in [0, n-1], any order, duplicates allowed; none gives the
    record alone.  A contiguous int32 CUDA tensor is passed as it is, without the range check (an entry
    outside [0, n-1] gives NaN).  Asynchronous on the current CUDA stream."""
    lib = _abi.load_library()
    _ray_tensor(status, torch.int32, grid.n_rays, 'status')
    for t, name in ((pupil, 'pupil'), (pupil_t, 'pupil_t')):
        _ray_tensor(t, torch.complex128, grid.n_rays, name)
    device = status.device
    if torch.is_tensor(shifts) and shifts.is_cuda:
        _ray_tensor(shifts, torch.int32, shifts.numel(), 'shifts')
        sh_d = shifts
    else:
        sh = np.ascontiguousarray(np.asarray(shifts, dtype=np.int64).reshape(-1))
        if ((sh < 0) | (sh >= grid.nx)).any():
            raise ValueError(f'shifts must lie in [0, {grid.nx - 1}]')
        sh_d = torch.tensor(sh.astype(np.int32), device=device)
    m = sh_d.numel()
    acf_x = torch.empty((grid.n_tiles, m), dtype=torch.complex128, device=device)
    acf_y = torch.empty((grid.n_tiles, m), dtype=torch.complex128, device=device)
    rec = torch.empty((grid.n_tiles, RT_MTF_DOUBLES), dtype=torch.float64, device=device)
    with torch.cuda.device(device):
        _abi.check(lib.rt_grid_mtf_shifts(grid.handle, _ptr(status), _ptr(pupil), _ptr(pupil_t),
                                          _ptr(sh_d) if m else None, m,
                                          _ptr(acf_x) if m else None, _ptr(acf_y) if m else None, _ptr(rec),
                                          _stream_ptr(device)))
    rec._keep = (status, pupil, pupil_t, sh_d)
    return acf_x, acf_y, rec


def trace_grid_opd_focus(table, grid, spheres, chunk_begin=0, chunk_end=None, res=None, **kwargs):
    """The OPD of every ray of chunks ``[chunk_begin, chunk_end)`` of a PupilGrid built with ``wave=``
    records against K reference spheres per tile, from one trace (``rt_trace_grid_opd_focus``).
    ``spheres``: ``[K, n_tiles, RT_SPHERE_DOUBLES]`` records (``waveabr.setup_tiles_focus``), numpy or
    a float64 device tensor.  Returns ``(opd_planes, res)``: the ``[K, n]`` float64 device tensor (row k:
    plane k's OPD in system units, NaN where status != 0) and the BundleResult of the per-ray ``status``
    (``res``: one to write into, with any kind-0 outputs).  Trace defaults as ``trace_grid``.
    Asynchronous on the current CUDA stream."""
    lib = _abi.load_library()
    device = torch.device('cuda', table.device)
    if chunk_end is None:
        chunk_end = grid.n_chunks
    kwargs.setdefault('check_apertures', True)
    kwargs.setdefault('first_surf', 1)
    kwargs.setdefault('last_surf', table.n_ifc - 2)
    if grid.pupil_kind == _abi.PUPIL_WIDE:
        kwargs['intersect_obj'] = False
    opts = _abi.make_opts(**kwargs)
    n = grid.rays_in_chunks(chunk_begin, chunk_end)
    if res is None:
        res = BundleResult(n, table.n_ifc, device, ('status',))
    elif res.n != n:
        raise ValueError('res was allocated for a different number of rays')
    sph = spheres if torch.is_tensor(spheres) else torch.as_tensor(np.ascontiguousarray(spheres, dtype=np.float64))
    sph = sph.to(device=device, dtype=torch.float64).contiguous()
    k = sph.shape[0] if sph.dim() == 3 else 0
    if sph.dim() != 3 or tuple(sph.shape[1:]) != (grid.n_tiles, RT_SPHERE_DOUBLES):
        raise ValueError(f'spheres must have shape [K, {grid.n_tiles}, {RT_SPHERE_DOUBLES}]')
    planes = torch.empty((k, n), dtype=torch.float64, device=device)
    out = res.c_struct()
    _abi.check(lib.rt_trace_grid_opd_focus(table.handle, grid.handle, chunk_begin, chunk_end, C.byref(opts),
                                           _ptr(sph), k, C.byref(out), _ptr(planes), _stream_ptr(device)))
    planes._keep = sph                     # must outlive the asynchronous launch
    return planes, res


def pupil_function_host(status, opd, x, y, wvl_sys):
    """numpy pupil function of one tile: ``status`` / ``opd`` ``[n, n]``, ``x`` / ``y`` the relative
    pupil coordinates broadcast to ``[n, n]``; exp(2 pi i (w - rint w)), w = opd/wvl_sys, where
    status is 0 and x^2 + y^2 <= 1, else 0.  Within an ulp or two of the device's sincospi."""
    used = (np.asarray(status) == 0) & (x*x + y*y <= 1.0)
    with np.errstate(invalid='ignore'):
        w = np.asarray(opd, dtype=np.float64)/wvl_sys
        r = 2.0*np.pi*(w - np.rint(w))
        p = np.cos(r) + 1j*np.sin(r)
    return np.where(used, p, 0.0 + 0.0j)


def _line_sums_in_order(v):
    """``v [n_lines, ...]`` real: the sum over axis 0 from +0.0 in increasing index (a sequential
    chain, not numpy's pairwise sum)"""
    acc = np.zeros(v.shape[1:])
    for row in v:
        acc = acc + row
    return acc


def _autocorr_host(P):
    """Cx of ``P [n, n]`` in the order of rt_mtf.cuh: chains along axis 0 for every (k, line j) at
    once (row i of every chain added at step i), then the lines of each k in order"""
    n = P.shape[0]
    pr, pi = np.ascontiguousarray(P.real), np.ascontiguousarray(P.imag)
    acc_r, acc_i = np.zeros((n, n)), np.zeros((n, n))          # [k, j]
    for i in range(n):
        ar, ai, br, bi = pr[i:], pi[i:], pr[i], pi[i]            # a = P[i + k], b = P[i], k < n - i
        acc_r[:n - i] = acc_r[:n - i] + (ar*br + ai*bi)
        acc_i[:n - i] = acc_i[:n - i] + (ai*br - ar*bi)
    return _line_sums_in_order(acc_r.T) + 1j*_line_sums_in_order(acc_i.T)


def mtf_sums_host(P):
    """``(acf_x [n], acf_y [n], S)`` of one tile's ``[n, n]`` complex128 pupil function (x outer), bit
    for bit in the order of ``rt_grid_mtf`` (the ``backend=`` seam of ``analyses.mtf``)"""
    P = np.asarray(P, dtype=np.complex128)
    s_lines = _line_sums_in_order(P.real) + 1j*_line_sums_in_order(P.imag)       # line j: along i
    S = complex(_line_sums_in_order(s_lines.real[:, None])[0], _line_sums_in_order(s_lines.imag[:, None])[0])
    return _autocorr_host(P), _autocorr_host(P.T), S


# --- relative illumination (rt_grid_illumination; the sums of csrc/rt_illum.cuh) ---------------------
ILLUM_RECORD = ('n_ok', 'n_missed', 'n_tir', 'n_blocked', 'n_other', 'n_used', 'n_disk', 'n_isolated',
                'sum_abs_j', 'sum_j')


def grid_illumination(grid, status, dx, dy):
    """``rt_grid_illumination``: the ``[n_tiles, RT_ILLUM_DOUBLES]`` float64 device record
    (``ILLUM_RECORD``: status counts, n_used, n_disk, n_isolated, sum |J|, sum J) of the projected
    solid angle of every tile of a square product PupilGrid without vignetting, 2 <= n <=
    RT_ILLUM_MAX_RAYS.  ``status`` (int32), ``dx``, ``dy`` (float64, the last segment's direction
    cosines L, M): per-ray device tensors of a grid trace over all chunks.  Asynchronous on the current
    CUDA stream."""
    lib = _abi.load_library()
    _ray_tensor(status, torch.int32, grid.n_rays, 'status')
    _ray_tensor(dx, torch.float64, grid.n_rays, 'dx')
    _ray_tensor(dy, torch.float64, grid.n_rays, 'dy')
    device = status.device
    rec = torch.empty((grid.n_tiles, RT_ILLUM_DOUBLES), dtype=torch.float64, device=device)
    with torch.cuda.device(device):
        _abi.check(lib.rt_grid_illumination(grid.handle, _ptr(status), _ptr(dx), _ptr(dy), _ptr(rec),
                                            _stream_ptr(device)))
    rec._keep = (status, dx, dy)               # must outlive the asynchronous launch
    return rec


def trace_grid_illumination(table, grid, res=None, **kwargs):
    """The ``grid_illumination`` record of every tile of a square PupilGrid without vignetting:
    ``trace_grid`` over all chunks with the ``d`` and ``status`` outputs into device buffers (``res``: an
    optional BundleResult with both, which keeps them), then ``grid_illumination`` -- two launches.
    Trace defaults as ``trace_grid``."""
    if res is None:
        res = BundleResult(grid.n_rays, table.n_ifc, torch.device('cuda', table.device), ('d', 'status'))
    elif res.d is None or res.status is None:
        raise ValueError('res needs the d and status outputs')
    trace_grid(table, grid, 0, grid.n_chunks, summary=False, res=res, **kwargs)
    rec = grid_illumination(grid, res.status, res.d[0], res.d[1])
    rec._keep = (rec._keep, res)
    return rec


def _illum_deriv(ok, L, M, u):
    """``(dL, dM, kind)`` along axis 0 of ``[n, n]`` arrays (``u``: the coordinates of the rows) in the
    order of rt_illum.cuh's illum_deriv: kind 0 central, 1 forward, 2 backward, 3 not formed"""
    ok_m, ok_p = np.zeros_like(ok), np.zeros_like(ok)
    ok_m[1:], ok_p[:-1] = ok[:-1], ok[1:]
    u0 = u[:, None]
    u_m, u_p = np.concatenate([u[:1], u[:-1]])[:, None], np.concatenate([u[1:], u[-1:]])[:, None]
    kind = np.where(ok_m & ok_p, 0, np.where(ok_p, 1, np.where(ok_m, 2, 3)))
    out = []
    with np.errstate(invalid='ignore', divide='ignore', over='ignore'):
        for f in (L, M):
            f_m, f_p = f.copy(), f.copy()
            f_m[1:], f_p[:-1] = f[:-1], f[1:]
            out.append(np.select([kind == 0, kind == 1, kind == 2],
                                 [(f_p - f_m)/(u_p - u_m), (f_p - f)/(u_p - u0), (f - f_m)/(u0 - u_m)], 0.0))
    return out[0], out[1], kind


def illumination_sums_host(status, L, M, x, y):
    """The ``RT_ILLUM_DOUBLES`` record of one tile, bit for bit in the order of ``rt_grid_illumination``
    (the ``backend=`` seam of ``analyses.relative_illumination``).  ``status``, ``L``, ``M``: ``[n, n]``
    per-ray status and last-segment direction cosines, ray (i, j) at pupil (``x[i]``, ``y[j]``)."""
    st = np.asarray(status).reshape(len(x), len(y))
    L = np.asarray(L, dtype=np.float64).reshape(st.shape)
    M = np.asarray(M, dtype=np.float64).reshape(st.shape)
    x, y = np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)
    ok = st == 0
    disk = x[:, None]*x[:, None] + y[None, :]*y[None, :] <= 1.0
    used = ok & disk
    Lx, Mx, kx = _illum_deriv(ok, L, M, x)
    Ly, My, ky = (a.T for a in _illum_deriv(ok.T, L.T, M.T, y))
    formed = used & (kx != 3) & (ky != 3)
    with np.errstate(invalid='ignore', over='ignore'):
        a, b = Lx*My, Ly*Mx
        J = np.where(formed, a - b, 0.0)
    cols_abs = _line_sums_in_order(np.abs(J))           # column j: along i, increasing i, from +0.0
    cols_j = _line_sums_in_order(J)
    rec = np.zeros(RT_ILLUM_DOUBLES)
    cls = np.where((st >= 0) & (st <= 3), st, 4).ravel()
    rec[0:5] = np.bincount(cls, minlength=5)[:5]
    rec[5], rec[6], rec[7] = used.sum(), disk.sum(), (used & ~formed).sum()
    rec[8] = _line_sums_in_order(cols_abs[:, None])[0]
    rec[9] = _line_sums_in_order(cols_j[:, None])[0]
    return rec


def measure_fp64_peak(device=0):
    """TFLOP/s of the fp64 vector pipe (DFMA microbenchmark in the library)."""
    lib = _abi.load_library()
    v = C.c_double()
    _abi.check(lib.rt_measure_fp64_peak(int(device), C.byref(v)))
    return v.value


def measure_fp64_latency(device=0):
    """cycles between two dependent DFMAs of one warp (``rt_measure_fp64_latency``)"""
    lib = _abi.load_library()
    v = C.c_double()
    _abi.check(lib.rt_measure_fp64_latency(int(device), C.byref(v)))
    return v.value


# columns of a tolerance record (RT_TOL_DOUBLES, include/b200rt.h): the spot summary, then the sums of
# the last segment's slopes ux = dx/dz, uy = dy/dz that move the spot with the focus
TOL_FIELDS = SUMMARY_FIELDS + ('sum_ux', 'sum_uy', 'sum_uxux', 'sum_uyuy', 'sum_xux', 'sum_yuy',
                               'reserved0', 'reserved1')
# scratch of one trace_grid_variants launch is ~6 B per ray and variant; larger sets go in batches
VARIANT_SCRATCH_CAP = 1 << 30


class VariantSet:
    """``n_var`` surface tables of one shape on the device (``rt_variants*``): ``descs`` is a
    sequence of ``rt_surface_desc`` arrays (or one array of ``n_var * n_ifc``), ``n_by_wvl``
    ``[n_var, n_wvl, n_ifc]``.  One allocation and one copy; immutable."""

    def __init__(self, descs, n_by_wvl, wvls=None, device=0):
        lib = _abi.load_library()
        self.n_by_wvl = np.ascontiguousarray(n_by_wvl, dtype=np.float64)
        self.n_var, self.n_wvl, self.n_ifc = self.n_by_wvl.shape
        if isinstance(descs, C.Array) and len(descs) == self.n_var*self.n_ifc:
            flat = descs
        else:
            flat = (_abi.rt_surface_desc*(self.n_var*self.n_ifc))()
            size = C.sizeof(_abi.rt_surface_desc)*self.n_ifc
            for v, d in enumerate(descs):
                if len(d) != self.n_ifc:
                    raise ValueError('every variant needs n_ifc descriptors')
                C.memmove(C.addressof(flat) + v*size, d, size)
        w = None
        if wvls is not None and all(isinstance(x, (int, float)) for x in wvls):
            w = np.ascontiguousarray(wvls, dtype=np.float64)
        self.device = int(device)
        handle = C.c_void_p()
        _abi.check(lib.rt_variants_create(flat, self.n_ifc, self.n_by_wvl.ctypes.data_as(_abi.c_double_p),
                                          self.n_wvl, self.n_var,
                                          None if w is None else w.ctypes.data_as(_abi.c_double_p),
                                          self.device, C.byref(handle)))
        self._handle, self._lib = handle, lib

    @property
    def handle(self):
        if self._handle is None:
            raise RuntimeError('VariantSet was destroyed')
        return self._handle

    def wave(self, grid, parax, var_begin=0, var_end=None):
        """The wave records of variants ``[var_begin, var_end)`` on every tile of ``grid``, built on the
        device (``rt_variants_wave``): each variant's chief rays, reference spheres at ``grid.foc`` and
        ``waveabr.wave_record``.  ``parax``: the nominal ``(fod.exp_dist, |fod.n_obj|, |fod.n_img|)``.
        Returns ``(wave [n, n_tiles, RT_WAVE_DOUBLES], ref_img [n, n_tiles, 2], status [n, n_tiles])``
        device tensors; a tile whose chief ray does not reach the image has status != 0 and a NaN
        record.  Asynchronous on the current CUDA stream."""
        device = torch.device('cuda', self.device)
        var_end = self.n_var if var_end is None else int(var_end)
        n = max(var_end - int(var_begin), 0)
        wave = torch.empty((n, grid.n_tiles, RT_WAVE_DOUBLES), dtype=torch.float64, device=device)
        ref = torch.empty((n, grid.n_tiles, 2), dtype=torch.float64, device=device)
        status = torch.empty((n, grid.n_tiles), dtype=torch.int32, device=device)
        px = np.ascontiguousarray(parax, dtype=np.float64)
        if px.shape != (3,):
            raise ValueError('parax must be (exp_dist, |n_obj|, |n_img|)')
        _abi.check(self._lib.rt_variants_wave(self.handle, grid.handle, int(var_begin), var_end,
                                              px.ctypes.data_as(_abi.c_double_p), _ptr(wave), _ptr(ref),
                                              _ptr(status), _stream_ptr(device)))
        return wave, ref, status

    def close(self):
        if getattr(self, '_handle', None) is not None:
            self._lib.rt_variants_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def variant_batch(grid, n_var, cap=VARIANT_SCRATCH_CAP):
    """variants per ``rt_trace_grid_variants`` launch so that its scratch stays under ``cap`` bytes"""
    lib = _abi.load_library()
    per = max(1, int(lib.rt_grid_variants_scratch_bytes(grid.handle, 1)))
    return max(1, min(int(n_var), cap//per))


def trace_grid_variants(variants, grid, var_begin=0, var_end=None, cap=VARIANT_SCRATCH_CAP, **kwargs):
    """Tolerance records of variants ``[var_begin, var_end)`` of a VariantSet over the whole
    PupilGrid (``rt_trace_grid_variants``): ``[n, n_tiles, RT_TOL_DOUBLES]`` float64 device tensor
    (TOL_FIELDS).  The variants go in batches whose scratch stays under ``cap`` bytes (two launches
    per batch).  Trace defaults as ``trace_grid``.  Asynchronous on the current CUDA stream."""
    lib = _abi.load_library()
    device = torch.device('cuda', variants.device)
    var_end = variants.n_var if var_end is None else int(var_end)
    kwargs.setdefault('check_apertures', True)
    kwargs.setdefault('first_surf', 1)
    kwargs.setdefault('last_surf', variants.n_ifc - 2)
    if grid.pupil_kind == _abi.PUPIL_WIDE:
        kwargs['intersect_obj'] = False
    opts = _abi.make_opts(**kwargs)
    n = max(var_end - int(var_begin), 0)
    rec = torch.empty((n, grid.n_tiles, RT_TOL_DOUBLES), dtype=torch.float64, device=device)
    if n == 0:
        return rec
    batch = variant_batch(grid, n, cap)
    scratch = torch.empty(max(int(lib.rt_grid_variants_scratch_bytes(grid.handle, batch))//8, 1),
                          dtype=torch.float64, device=device)
    stream = _stream_ptr(device)
    for v0 in range(int(var_begin), var_end, batch):
        v1 = min(v0 + batch, var_end)
        _abi.check(lib.rt_trace_grid_variants(variants.handle, grid.handle, v0, v1, C.byref(opts),
                                              _ptr(rec[v0 - var_begin]), _ptr(scratch), stream))
    rec._keep = scratch            # scratch must outlive the asynchronous launches
    return rec


def trace_grid_variants_wfe(variants, grid, wave, var_begin=0, var_end=None, cap=VARIANT_SCRATCH_CAP, **kwargs):
    """Wavefront-error records of variants ``[var_begin, var_end)`` of a VariantSet over the whole
    PupilGrid (``rt_trace_grid_variants_wfe``): ``[n, n_tiles, RT_WFE_DOUBLES]`` float64 device tensor
    (WFE_FIELDS; ``wavefront_statistics`` turns it into numbers), each ray's OPD referred to its
    variant's record of ``wave`` ``[n, n_tiles, RT_WAVE_DOUBLES]`` (``VariantSet.wave`` of the same
    range).  Batches, trace defaults and stream as ``trace_grid_variants``."""
    lib = _abi.load_library()
    device = torch.device('cuda', variants.device)
    var_end = variants.n_var if var_end is None else int(var_end)
    kwargs.setdefault('check_apertures', True)
    kwargs.setdefault('first_surf', 1)
    kwargs.setdefault('last_surf', variants.n_ifc - 2)
    if grid.pupil_kind == _abi.PUPIL_WIDE:
        kwargs['intersect_obj'] = False
    opts = _abi.make_opts(**kwargs)
    n = max(var_end - int(var_begin), 0)
    rec = torch.empty((n, grid.n_tiles, RT_WFE_DOUBLES), dtype=torch.float64, device=device)
    if n == 0:
        return rec
    if tuple(wave.shape) != (n, grid.n_tiles, RT_WAVE_DOUBLES) or wave.dtype != torch.float64 \
            or wave.device != device or not wave.is_contiguous():
        raise ValueError('wave must be a contiguous float64 [n, n_tiles, RT_WAVE_DOUBLES] tensor on the '
                         'variants\' device')
    per = max(1, int(lib.rt_grid_variants_wfe_scratch_bytes(grid.handle, 1)))
    batch = max(1, min(n, cap//per))
    scratch = torch.empty(max(int(lib.rt_grid_variants_wfe_scratch_bytes(grid.handle, batch))//8, 1),
                          dtype=torch.float64, device=device)
    stream = _stream_ptr(device)
    for v0 in range(int(var_begin), var_end, batch):
        v1 = min(v0 + batch, var_end)
        i = v0 - int(var_begin)
        _abi.check(lib.rt_trace_grid_variants_wfe(variants.handle, grid.handle, v0, v1, C.byref(opts),
                                                  _ptr(wave[i]), _ptr(rec[i]), _ptr(scratch), stream))
    rec._keep = scratch            # scratch must outlive the asynchronous launches
    return rec


def launch_count():
    return int(_abi.load_library().rt_launch_count())


def _grid_args(opt_model, wvl_index, num_rays, fields, wvls, foc, pupil_range, apply_vignetting):
    osp, sm = opt_model.optical_spec, opt_model.seq_model
    fields = list(osp.field_of_view.fields if fields is None else fields)
    wvls = list(sm.wvlns if wvls is None else wvls)
    recs, eprad, z_pupil = osp.grid_fields(fields)
    foc = osp.defocus.focus_shift if foc is None else foc
    xs = accumulated_steps(pupil_range[0], pupil_range[1], num_rays)
    args = (recs, [wvl_index(w) for w in wvls], xs, xs, eprad, z_pupil)
    kw = dict(apply_vignetting=apply_vignetting, flip_z_dir=sm.z_dir[0], foc=foc)
    return args, kw


def grid_spec_for_model(opt_model, num_rays, fields=None, wvls=None, foc=None,
                        pupil_range=(-1.0, 1.0), apply_vignetting=True, ref_img=None):
    """Host-only PupilGridSpec of the reference's square-grid analyses (no CUDA)."""
    sm = opt_model.seq_model
    args, kw = _grid_args(opt_model, sm.index_for_wavelength, num_rays, fields, wvls, foc,
                          pupil_range, apply_vignetting)
    return PupilGridSpec(*args, ref_img=ref_img, **kw)


def grid_for_model(opt_model, table, num_rays, fields=None, wvls=None, foc=None,
                   pupil_range=(-1.0, 1.0), apply_vignetting=True, ref_img='chief'):
    """PupilGrid for the reference's square-grid analyses of a model:
    fields x wavelengths x (num_rays x num_rays) over relative pupil
    ``[-1, 1]^2`` with the reference's accumulated stepping
    (raytr/trace.py:563-605; seq/sequential.py:1058-1085).

    ``ref_img='chief'`` traces the (0, 0) pupil ray of every (field, wvl) first
    (one tiny grid launch) and uses its image intercept as the reference image
    point, as ``calculate_reference_sphere`` does (raytr/waveabr.py:24-76)."""
    args, kw = _grid_args(opt_model, table.wvl_index, num_rays, fields, wvls, foc, pupil_range,
                          apply_vignetting)
    ref = None
    if isinstance(ref_img, str) and ref_img == 'chief':
        g0 = PupilGrid(args[0], args[1], [0.0], [0.0], args[4], args[5], device=table.device,
                       **dict(kw, apply_vignetting=False))
        r0 = trace_grid(table, g0, outputs=('p',), summary=False, check_apertures=False)
        ref = r0.p[:2].t().contiguous().cpu().numpy().reshape(len(args[0]), len(args[1]), 2)
        g0.close()
    elif ref_img is not None:
        ref = ref_img
    return PupilGrid(*args, ref_img=ref, device=table.device, **kw)
