"""Chief-ray aiming and clear-aperture setting on top of a ``trace`` function.

Host-side model preparation (tens of rays per field, run once per model):

* ``aim_chief_ray``       /root/reference/src/rayoptics/raytr/trace.py:313-415,627-640
  (``iterate_ray``: find the entrance-pupil aim point that puts the ray through
  the centre of the stop surface)
* ``set_clear_apertures`` /root/reference/src/rayoptics/raytr/vigcalc.py:45-80
  (max radial height of the 5 boundary rays per field -> ``max_aperture``;
  the stop surface is set from the first field only)

``aim_all_fields_batched`` / ``set_clear_apertures_batched`` do the same with all fields
per bundle launch (SURVEY.md 8(f) rows 1 and 4).

The per-ray versions take the tracer as an argument (``trace_fn(seq_model, pt0, dir0, wvl,
**kw) -> (ray, op, wvl)``; the batched ones a ``bundle_fn``): the product passes the GPU drop-in
``rayoptics_b200.raytrace.trace``; the fixture generator, which runs where no
GPU exists, passes the reference's own ``trace``.  Not on the parity path --
their results are inputs shared by oracle and engine.
"""
from __future__ import annotations

import math

import numpy as np


def _wide(opt_model):
    return bool(opt_model.optical_spec.field_of_view.is_wide_angle)


def _launch(opt_model, dir0):
    """trace_base, trace.py:299-308: wide-angle rays start off the object surface and are never
    flipped; otherwise a ray running against z_dir means a virtual object and is reversed.
    Returns (dir0, trace keyword arguments)."""
    if _wide(opt_model):
        return dir0, {'intersect_obj': False}
    if dir0[2]*opt_model.seq_model.z_dir[0] < 0:
        dir0 = -dir0
    return dir0, {}


def _is_trace_error(e):
    """a per-ray failure (TraceError of this package or of the reference, by name: trace_fn may be
    either) as opposed to an engine failure"""
    return any(c.__name__ == 'TraceError' for c in type(e).__mro__)


def _stop_xy(opt_model, trace_fn, fld, wvl, aim, stop):
    osp = opt_model.optical_spec
    saved = fld.aim_info
    fld.aim_info = np.array(aim, dtype=float)
    try:
        pt0, dir0 = osp.ray_start_from_osp(np.array([0., 0.]), fld, 'rel pupil')
    finally:
        fld.aim_info = saved
    sm = opt_model.seq_model
    dir0, kw = _launch(opt_model, dir0)
    ray, _, _ = trace_fn(sm, pt0, dir0, wvl, **kw)
    p = ray[stop][0]
    return np.array([p[0], p[1]])


def aim_chief_ray(opt_model, fld, wvl, trace_fn, tol=1e-13, max_iter=30):
    """Aim point on the paraxial entrance pupil such that the (0, 0) pupil ray
    crosses the stop surface at its vertex.  Damped 2-D Newton iteration."""
    sm = opt_model.seq_model
    stop = sm.stop_surface
    if stop is None:
        return np.array([0., 0.])
    x = np.array([0., 0.])

    def f_at(v):
        try:
            return _stop_xy(opt_model, trace_fn, fld, wvl, v, stop)
        except Exception as e:  # a TraceError (this package's or the reference's, whatever the
            if not _is_trace_error(e):      # trace_fn raises): the trial ray did not reach the stop
                raise                       # anything else (engine, CUDA) stays loud
            return None

    f = f_at(x)
    if f is None:
        return x
    h = 1e-4*max(1.0, opt_model.optical_spec.fod.enp_radius)
    for _ in range(max_iter):
        if np.max(np.abs(f)) < tol:
            break
        J = np.zeros((2, 2))
        ok = True
        for k in range(2):
            dx = np.zeros(2)
            dx[k] = h
            fk = f_at(x + dx)
            if fk is None:
                ok = False
                break
            J[:, k] = (fk - f)/h
        if not ok:
            break
        try:
            step = np.linalg.solve(J, -f)
        except np.linalg.LinAlgError:
            break
        # backtracking: halve the step until the trial ray traces and improves
        lam, accepted = 1.0, False
        for _bt in range(20):
            f_new = f_at(x + lam*step)
            if f_new is not None and np.max(np.abs(f_new)) < np.max(np.abs(f)):
                x, f, accepted = x + lam*step, f_new, True
                break
            lam *= 0.5
        if not accepted:
            break
    if fld.x == 0.0:
        x[0] = 0.0
    return x


def aim_all_fields(opt_model, trace_fn, wvl=None):
    osp = opt_model.optical_spec
    wvl = osp.spectral_region.central_wvl if wvl is None else wvl
    if _wide(opt_model):        # aim_chief_ray, raytr/trace.py:634-635: the real entrance pupil search
        from . import wideangle
        wideangle.aim_wide_angle_fields(opt_model, wvl, trace_fn)
        return
    for fld in osp.field_of_view.fields:
        fld.aim_info = aim_chief_ray(opt_model, fld, wvl, trace_fn)


def trace_boundary_rays(opt_model, trace_fn, wvl=None):
    """raytr/trace.py:460-510: the pupil_rays of every field, with vignetting."""
    osp = opt_model.optical_spec
    sm = opt_model.seq_model
    wvl = osp.spectral_region.central_wvl if wvl is None else wvl
    rayset = []
    for fld in osp.field_of_view.fields:
        rim = []
        for pr in osp.pupil.pupil_rays:
            pupil = fld.apply_vignetting(list(pr))
            pt0, dir0 = osp.ray_start_from_osp(pupil, fld, 'rel pupil')
            dir0, kw = _launch(opt_model, dir0)
            try:
                ray, _, _ = trace_fn(sm, pt0, dir0, wvl, **kw)
            except Exception as e:       # TraceError: keep the partial ray
                if not _is_trace_error(e):
                    raise
                pkg = getattr(e, 'ray_pkg', None)
                ray = pkg[0] if pkg is not None else []
            rim.append(ray)
        rayset.append(rim)
    return rayset


def max_aperture_at_surf(rayset, i):
    """largest radial height at interface ``i`` over a set of boundary rays (per field, per pupil
    ray; ray packages or plain rays); None when a ray ended before ``i`` (vigcalc.py:31-42)"""
    max_ap = -1.0e+10
    for f in rayset:
        for p in f:
            ray = p.ray if hasattr(p, 'ray') else p
            if len(ray) > i:
                pt = ray[i][0]
                ap = math.sqrt(pt[0]**2 + pt[1]**2)
                if ap > max_ap:
                    max_ap = ap
            else:
                return None
    return max_ap


def _include_list(num_surfs, avoid_list, include_list):
    """vigcalc.py:60-66: everything, the given list, or everything but ``avoid_list``"""
    if avoid_list is not None:
        return [i for i in range(num_surfs) if i not in avoid_list]
    return range(num_surfs) if include_list is None else include_list


def set_clear_apertures(opt_model, trace_fn, wvl=None, avoid_list=None, include_list=None):
    """From the existing fields and vignetting, calculate clear apertures (vigcalc.py:45-80).
    The stop surface takes its aperture from the boundary rays of the first field."""
    sm = opt_model.seq_model
    include_list = _include_list(sm.get_num_surfaces(), avoid_list, include_list)
    rayset = trace_boundary_rays(opt_model, trace_fn, wvl)
    stop = sm.stop_surface
    for i in include_list:
        m = max_aperture_at_surf([rayset[0]] if i == stop else rayset, i)
        if m is not None:
            sm.ifcs[i].set_max_aperture(m)


# --- batched versions: all fields per launch --------------------------------------------------
def cuda_bundle_fn(opt_model, table=None, device=0):
    """``bundle_fn(p0 [3, n], d0 [3, n], wvl, last_surf) -> (full [n_ifc, 10, n], n_seg [n])``
    on the CUDA engine (whole rays: aiming and aperture setting read interior interfaces)."""
    from . import engine as E
    from .analyses import _table_for
    tab = _table_for(opt_model, table, device)

    def fn(p0, d0, wvl):
        w = np.full(p0.shape[1], tab.wvl_index(wvl), dtype=np.int32)
        r = E.trace_bundle(tab, p0, d0, wvl_idx=w, full=True, outputs=('n_seg',), first_surf=1,
                           last_surf=tab.n_ifc - 2, intersect_obj=not _wide(opt_model))
        return r.full.cpu().numpy(), r.n_seg.cpu().numpy()
    return fn


def _start_rays(opt_model, fields, aims, pupils):
    """(p0, d0) [3, n] for field k aimed at aims[k] with relative pupil pupils[k]"""
    osp, sm = opt_model.optical_spec, opt_model.seq_model
    p0, d0 = np.zeros((3, len(fields))), np.zeros((3, len(fields)))
    for k, (fld, aim, pupil) in enumerate(zip(fields, aims, pupils)):
        saved = fld.aim_info
        fld.aim_info = None if aim is None else np.array(aim, dtype=float)
        try:
            pt0, dir0 = osp.ray_start_from_osp(np.array(pupil, dtype=float), fld, 'rel pupil')
        finally:
            fld.aim_info = saved
        dir0, _ = _launch(opt_model, dir0)
        p0[:, k], d0[:, k] = pt0, dir0
    return p0, d0


def aim_all_fields_batched(opt_model, bundle_fn=None, wvl=None, tol=1e-13, max_iter=30, trace_fn=None):
    """``aim_chief_ray`` for every field at once (raytr/trace.py:313-415,627-640): each
    Newton iteration traces base + two finite-difference rays of ALL fields in one bundle,
    each backtracking round one more.  Same iteration as ``aim_chief_ray`` field by field,
    so the aim points are the same numbers.  Sets ``fld.aim_info``; returns the list."""
    osp, sm = opt_model.optical_spec, opt_model.seq_model
    stop = sm.stop_surface
    fields = list(osp.field_of_view.fields)
    nf = len(fields)
    if stop is None:
        for fld in fields:
            fld.aim_info = np.array([0., 0.])
        return [f.aim_info for f in fields]
    if _wide(opt_model):        # wide-angle fields: z_enp search on single rays (wideangle.py)
        from . import wideangle
        return wideangle.aim_wide_angle_fields(opt_model, wvl, trace_fn)
    if bundle_fn is None:
        bundle_fn = cuda_bundle_fn(opt_model)
    wvl = osp.spectral_region.central_wvl if wvl is None else wvl
    zero = [0., 0.]

    def stop_xy(idx, aims):
        """stop intercepts of the (0, 0) pupil rays of fields idx (NaN rows where a ray fails)"""
        p0, d0 = _start_rays(opt_model, [fields[i] for i in idx], aims, [zero]*len(idx))
        full, n_seg = bundle_fn(p0, d0, wvl)
        out = full[stop, 0:2, :].T.copy()
        out[n_seg <= stop] = np.nan
        return out

    x = np.zeros((nf, 2))
    f = stop_xy(range(nf), x)
    active = [i for i in range(nf) if np.isfinite(f[i]).all()]
    h = 1e-4*max(1.0, osp.fod.enp_radius)
    for _ in range(max_iter):
        active = [i for i in active if np.max(np.abs(f[i])) >= tol]
        if not active:
            break
        fx = stop_xy(active, [x[i] + [h, 0.] for i in active])
        fy = stop_xy(active, [x[i] + [0., h] for i in active])
        steps, keep = {}, []
        for k, i in enumerate(active):
            if not (np.isfinite(fx[k]).all() and np.isfinite(fy[k]).all()):
                continue
            J = np.stack([(fx[k] - f[i])/h, (fy[k] - f[i])/h], axis=1)
            try:
                steps[i] = np.linalg.solve(J, -f[i])
            except np.linalg.LinAlgError:
                continue
            keep.append(i)
        # backtracking, all still-unaccepted fields per launch
        lam = {i: 1.0 for i in keep}
        pending, accepted = list(keep), []
        for _bt in range(20):
            if not pending:
                break
            trial = stop_xy(pending, [x[i] + lam[i]*steps[i] for i in pending])
            nxt = []
            for k, i in enumerate(pending):
                if np.isfinite(trial[k]).all() and np.max(np.abs(trial[k])) < np.max(np.abs(f[i])):
                    x[i], f[i] = x[i] + lam[i]*steps[i], trial[k]
                    accepted.append(i)
                else:
                    lam[i] *= 0.5
                    nxt.append(i)
            pending = nxt
        active = accepted
    for i, fld in enumerate(fields):
        if fld.x == 0.0:
            x[i, 0] = 0.0
        fld.aim_info = x[i].copy()
    return [f.aim_info for f in fields]


def aim_fields_on_device(opt_model, fields, wvl=None, table=None, device=0, tol=1e-13, max_iter=30):
    """``aim_all_fields_batched`` for the given ``Field`` objects with the whole iteration on the
    device: one ``rt_grid_aim_chief`` launch (one thread per field, csrc/rt_aim.cuh) on the records
    of ``grid_fields_of`` and one small copy back, then the ``fld.x == 0`` rule.  Sets
    ``fld.aim_info``; returns the list.  A floating stop gives (0, 0) without a launch.  The
    iteration is ``aim_chief_ray``'s with its own 2x2 solve (DESIGN.md section 4): on-meridian fields
    get the aim points of ``aim_all_fields_batched`` bit for bit.  'epd' pupils only: wide-angle fields
    and angular pupils raise NotImplementedError."""
    from . import engine as E
    from .analyses import _table_for
    from .opticalspec import grid_fields_of
    osp, sm = opt_model.optical_spec, opt_model.seq_model
    fields = list(fields)
    stop = sm.stop_surface
    if stop is None or not fields:
        for fld in fields:
            fld.aim_info = np.array([0., 0.])
        return [f.aim_info for f in fields]
    if _wide(opt_model):
        raise NotImplementedError('aim_fields_on_device: wide-angle fields need the real entrance pupil search; '
                                  'use vigcalc.aim_all_fields_batched (wideangle.aim_wide_angle_fields)')
    recs, eprad, z_pupil = grid_fields_of(opt_model, fields)
    if recs[0]['pupil_kind'] != 0:
        raise NotImplementedError('aim_fields_on_device: angular pupils are not aimed on the device; '
                                  'use vigcalc.aim_all_fields_batched or aim_chief_ray')
    tab = _table_for(opt_model, table, device)
    wvl = osp.spectral_region.central_wvl if wvl is None else wvl
    wi = tab.wvl_index(wvl)
    h = 1e-4*max(1.0, osp.fod.enp_radius)
    grid = E.PupilGrid(recs, [wi], [0.0], [0.0], eprad, z_pupil, apply_vignetting=False,
                       flip_z_dir=sm.z_dir[0], device=tab.device)
    aim, _ = E.aim_chief_rays(tab, grid, stop, wi, h, tol, max_iter)
    x = aim.cpu().numpy()                        # one small copy; waits
    grid.close()
    for i, fld in enumerate(fields):
        if fld.x == 0.0:
            x[i, 0] = 0.0
        fld.aim_info = x[i].copy()
    return [f.aim_info for f in fields]


def set_clear_apertures_batched(opt_model, bundle_fn=None, wvl=None, avoid_list=None,
                                include_list=None):
    """``set_clear_apertures`` (raytr/vigcalc.py:45-80) with the 5 boundary rays of all
    fields in one bundle."""
    osp, sm = opt_model.optical_spec, opt_model.seq_model
    if bundle_fn is None:
        bundle_fn = cuda_bundle_fn(opt_model)
    wvl = osp.spectral_region.central_wvl if wvl is None else wvl
    fields = list(osp.field_of_view.fields)
    rays_f, rays_p = [], []
    for fld in fields:
        for pr in osp.pupil.pupil_rays:
            rays_f.append(fld)
            rays_p.append(fld.apply_vignetting(list(pr)))
    p0, d0 = _start_rays(opt_model, rays_f, [f.aim_info for f in rays_f], rays_p)
    full, n_seg = bundle_fn(p0, d0, wvl)
    per = len(osp.pupil.pupil_rays)
    r = np.sqrt(full[:, 0, :]*full[:, 0, :] + full[:, 1, :]*full[:, 1, :])      # [n_ifc, n]
    stop = sm.stop_surface
    for i in _include_list(sm.get_num_surfaces(), avoid_list, include_list):
        sel = slice(0, per) if i == stop else slice(None)
        if (n_seg[sel] <= i).any():           # a ray failed before this interface: keep the value
            continue
        sm.ifcs[i].set_max_aperture(float(r[i, sel].max()))


# --- vignetting factors from clear apertures (raytr/vigcalc.py:83-93,227-342,393-471) ----------
def _edge_pt_target(ifc, rel_dir):
    """Surface.edge_pt_target / Aperture.edge_pt_target (elem/surface.py:210-218,422-427,459-464)"""
    d = np.array(rel_dir, dtype=float)
    length = np.linalg.norm(d)
    d = d if length == 0.0 else d/length
    cas = getattr(ifc, 'clear_apertures', None) or []
    if cas:
        ca = cas[0]
        if type(ca).__name__ == 'Circular':
            return ca.radius*d
        return np.array([ca.x_half_width*d[0], ca.y_half_width*d[1]])
    return ifc.max_aperture*d


def iterate_pupil_ray(opt_model, indx, xy, start_r0, r_target, fld, wvl, **engine):
    """Pupil coordinate whose ray passes interface ``indx`` at radial height ``r_target``
    (vigcalc.py:393-471): scipy's secant ``newton`` with the reference's tolerance."""
    from scipy.optimize import newton
    from . import trace as TR
    from .raytrace import TraceError, TraceMissedSurfaceError

    def r_pupil_coordinate(xy_coord):
        rel_p1 = np.array([0., 0.])
        rel_p1[xy] = xy_coord
        try:
            ray_pkg = TR.trace_base(opt_model, rel_p1, fld, wvl, apply_vignetting=False,
                                    check_apertures=False, **engine)
        except TraceError as ray_error:
            ray_pkg = ray_error.ray_pkg
            limit = indx if isinstance(ray_error, TraceMissedSurfaceError) else indx - 1
            if ray_error.surf <= limit:
                ray_error.rel_p1 = rel_p1
                raise ray_error
        p = ray_pkg[0][indx][0]
        r_ray = math.copysign(math.sqrt(p[0]**2 + p[1]**2), r_target)
        return r_ray - r_target

    start_coords = np.array([0., 0.])
    if indx is None:                    # floating stop: use the entrance pupil for aiming
        start_coords[xy] = r_target
        return start_coords
    try:
        start_r, results = newton(r_pupil_coordinate, start_r0, tol=1e-6, disp=False,
                                  full_output=True)
    except TraceError as rt_err:
        start_r = 0.9*rt_err.rel_p1[xy]
    start_coords[xy] = start_r
    return start_coords


def calc_vignetted_ray(opm, xy, start_dir, fld, wvl, max_iter_count=50, **engine):
    """Find the limiting aperture along ``start_dir`` and return ``(vig, clip_indx, ray_pkg)``
    (vigcalc.py:248-342), same search: trace with clipping; when a surface blocks, iterate
    the pupil ray to its edge; stop when the same surface blocks twice or the ray passes."""
    from . import trace as TR
    from .raytrace import TraceError
    rel_p1 = np.array(start_dir, dtype=float)
    sm = opm.seq_model
    still_iterating, clip_indx, iter_count, ray_pkg = True, None, 0, None
    while still_iterating and iter_count < max_iter_count:
        iter_count += 1
        try:
            ray_pkg = TR.trace_base(opm, rel_p1, fld, wvl, apply_vignetting=False,
                                    check_apertures=True, pt_inside_fuzz=1e-4, **engine)
        except TraceError as ray_error:
            ray_pkg = ray_error.ray_pkg
            indx = ray_error.surf
            if indx == clip_indx:
                still_iterating = False
            else:
                r_target = _edge_pt_target(sm.ifcs[indx], start_dir)
                rel_p1 = iterate_pupil_ray(opm, indx, xy, rel_p1[xy], r_target[xy], fld, wvl, **engine)
                clip_indx = indx
        else:
            if clip_indx is not None:
                still_iterating = False
            else:                       # first pass succeeded: go to the edge of the stop
                stop_indx = sm.stop_surface
                if stop_indx is not None:
                    r_target = _edge_pt_target(sm.ifcs[stop_indx], start_dir)
                    rel_p1 = iterate_pupil_ray(opm, stop_indx, xy, rel_p1[xy], r_target[xy], fld,
                                               wvl, **engine)
                    clip_indx = stop_indx
                else:
                    still_iterating = False
    vig = 1.0 - (rel_p1[xy]/start_dir[xy])
    return vig, clip_indx, ray_pkg


def calc_vignetting_for_field(opm, fld, wvl, **kwargs):
    """vigcalc.py:227-245: the four pupil directions -> fld.vux, vlx, vuy, vly"""
    vg = {k: kwargs.pop(k) for k in ('max_iter_count',) if k in kwargs}
    pupil_starts = opm.optical_spec.pupil.pupil_rays[1:]
    vig_factors = [0.]*4
    for i in range(4):
        vig_factors[i] = calc_vignetted_ray(opm, i//2, pupil_starts[i], fld, wvl, **vg, **kwargs)[0]
    fld.vux, fld.vlx, fld.vuy, fld.vly = vig_factors


def set_vig(opm, **kwargs):
    """From the existing fields and clear apertures, calculate the vignetting factors
    (vigcalc.py:83-90).  ``tracer=`` / ``table=`` / ``device=`` select the engine
    (default: CUDA)."""
    osp = opm.optical_spec
    wvl = osp.spectral_region.central_wvl
    for fld in osp.field_of_view.fields:
        calc_vignetting_for_field(opm, fld, wvl, **kwargs)


def calc_vignetted_ray_by_bisection(opm, xy, start_dir, fld, wvl, max_iter_count=10, **engine):
    """The limiting aperture along ``start_dir`` by halving steps in the pupil
    (vigcalc.py:347-390): ``(vig, clip_indx, ray_pkg)``."""
    from . import trace as TR
    from .raytrace import TraceError
    rel_p1 = np.array(start_dir, dtype=float)
    clip_indx, ray_pkg, step_size = None, None, 1.0
    for _ in range(max_iter_count):
        step_size /= 2
        try:
            ray_pkg = TR.trace_base(opm, rel_p1, fld, wvl, apply_vignetting=False,
                                    check_apertures=True, pt_inside_fuzz=1e-4, **engine)
        except TraceError as ray_error:
            ray_pkg = TR.RayPkg(*ray_error.ray_pkg)
            clip_indx = ray_error.surf
            rel_p1 = -step_size*np.array(start_dir) + rel_p1
        else:
            rel_p1 = step_size*np.array(start_dir) + rel_p1
    vig = 1.0 - (rel_p1[xy]/start_dir[xy])
    return vig, clip_indx, ray_pkg


def _surface_od(ifc):
    """Surface.surface_od (elem/surface.py:181-196) without edge apertures"""
    cas = getattr(ifc, 'clear_apertures', None) or []
    od = 0
    for ca in cas:
        ap = (ca.radius if type(ca).__name__ == 'Circular'
              else max(ca.x_half_width, ca.y_half_width))
        od = max(od, ap)
    return od if cas else ifc.max_aperture


def paraxial_vignetting(opt_model, rel_fov=1):
    """Vignetting factors from the paraxial axial / chief rays and the surface apertures, no real
    ray involved (ParaxialModel.paraxial_vignetting, parax/paraxialdesign.py:1023-1050):
    ``((min lower ratio, interface), (min upper ratio, interface))``."""
    from .firstorder import HT
    sm = opt_model.seq_model
    fod = opt_model.optical_spec.fod
    ax, pr = fod.ax_ray, fod.pr_ray
    min_vly, min_vuy = (1, None), (1, None)
    for i, ifc in enumerate(sm.ifcs[:-1]):
        y = ax[i][HT]
        if y == 0:
            continue
        ybar = rel_fov*pr[i][HT]
        ratio = (_surface_od(ifc) - abs(ybar))/abs(y)
        if ratio <= 0:
            continue
        if ybar <= 0 and ratio < min_vly[0]:
            min_vly = ratio, i
        if ybar >= 0 and ratio < min_vuy[0]:
            min_vuy = ratio, i
    return min_vly, min_vuy


def apply_paraxial_vignetting(opt_model):
    """set ``vly`` / ``vuy`` of every field from ``paraxial_vignetting`` (raytr/trace.py:643-657)"""
    fov = opt_model.optical_spec.field_of_view
    max_field, _ = fov.max_field()
    for fld in fov.fields:
        rel_fov = math.sqrt(fld.x**2 + fld.y**2)
        if not fov.is_relative and max_field != 0:
            rel_fov = rel_fov/max_field
        min_vly, min_vuy = paraxial_vignetting(opt_model, rel_fov)
        if min_vly[1] is not None:
            fld.vly = 1 - min_vly[0]
        if min_vuy[1] is not None:
            fld.vuy = 1 - min_vuy[0]


def set_ape(opt_model, avoid_list=None, include_list=None, bundle_fn=None):
    """clear apertures from the existing fields and vignetting (vigcalc.py:83-99): the batched
    ``set_clear_apertures``, then the element model -- when the model has one (an unchanged
    ray-optics OpticalModel) -- is synchronised as the reference does"""
    set_clear_apertures_batched(opt_model, bundle_fn, avoid_list=avoid_list, include_list=include_list)
    try:
        em = opt_model['em']
    except (KeyError, TypeError, AttributeError):
        return
    em.sync_to_seq(opt_model['sm'])


def set_stop_aperture(opm, trace_fn=None, **engine):
    """Set the aperture of the stop surface to satisfy the pupil specification, then recompute
    the vignetting (vigcalc.py:104-115)."""
    from . import raytrace as RT
    sm = opm.seq_model
    opm.optical_spec.field_of_view.fields[0].clear_vignetting()      # fov['axis']
    set_clear_apertures(opm, RT.trace if trace_fn is None else trace_fn,
                        include_list=[sm.stop_surface])
    set_vig(opm, **engine)


def set_pupil(opm, use_parax=False, **engine):
    """From the existing stop size, calculate the pupil specification and the vignetting
    (vigcalc.py:118-224): the axial upper marginal ray is iterated through the edge of the stop;
    its object / image space segment gives the new EPD, NA or f/#."""
    from . import trace as TR
    from .firstorder import HT, SLP
    from .raytrace import TraceRayBlockedError
    sm, osp = opm.seq_model, opm.optical_spec
    if sm.stop_surface is None:
        print('floating stop surface')
        return
    idx_stop = sm.stop_surface
    fld_0, cwl, foc = osp.lookup_fld_wvl_focus(0)
    stop_radius = _surface_od(sm.ifcs[idx_stop])
    start_coords = iterate_pupil_ray(opm, idx_stop, 1, 1.0, stop_radius, fld_0, cwl, **engine)
    ray_pkg, ray_err = TR.trace_safe(opm, start_coords, fld_0, cwl, None, 'full',
                                     apply_vignetting=False, **engine)
    pupil = osp.pupil
    obj_img_key, pupil_spec = pupil.key
    pupil_value_orig = pupil.value
    fod = osp.fod
    ax_ray = fod.ax_ray
    wi = sm.index_for_wavelength(sm.central_wavelength())
    n0, nk = sm.rndx[0][wi], sm.rndx[-1][wi]              # central_rndx(0), central_rndx(-1)
    rs0, rs1, rsm2 = ray_pkg[0][0], ray_pkg[0][1], ray_pkg[0][-2]
    if use_parax:
        scale_ratio = stop_radius/ax_ray[idx_stop][HT]
        if obj_img_key == 'object':
            if pupil_spec == 'epd':
                pupil.value = scale_ratio*(2*fod.enp_radius)
            elif pupil_spec == 'NA':
                pupil.value = n0*rs0[1][1]
            elif pupil_spec == 'f/#':
                pupil.value = 1/(2*(scale_ratio*ax_ray[0][SLP]))
        elif obj_img_key == 'image':
            if pupil_spec == 'epd':
                pupil.value = scale_ratio*(2*fod.exp_radius)
            elif pupil_spec == 'NA':
                pupil.value = -nk*rsm2[1][1]
            elif pupil_spec == 'f/#':
                pupil.value = -1/(2*(scale_ratio*ax_ray[-1][SLP]))
    else:                                                   # the real marginal ray
        scale_ratio = rs1[0][1]/ax_ray[1][HT]
        if obj_img_key == 'object':
            if pupil_spec == 'epd':
                pupil.value *= scale_ratio
            elif pupil_spec == 'NA':
                pupil.value = n0*rs0[1][1]
            elif pupil_spec == 'f/#':
                pupil.value = 1/(2*(rs0[1][1]/rs0[1][2]))
        elif obj_img_key == 'image':
            if pupil_spec == 'epd':
                pupil.value = 2*rsm2[0][1]
            elif pupil_spec == 'NA':
                pupil.value = -nk*rsm2[1][1]
            elif pupil_spec == 'f/#':
                pupil.value = -1/(2*(scale_ratio*ax_ray[-1][SLP]))
    clipped = TR.trace_safe(opm, start_coords, fld_0, cwl, None, 'full', apply_vignetting=False,
                            check_apertures=True, **engine)
    if isinstance(clipped.err, TraceRayBlockedError):
        print(f'Axial bundle limited by surface {clipped.err.surf}, not stop surface.')
    if pupil_value_orig != pupil.value:
        opm.update_model()
        set_vig(opm, **engine)


# --- the same searches for ALL fields and pupil directions in lock step ----------------------
# Each (field, direction) search of calc_vignetted_ray / iterate_pupil_ray is a generator that
# yields the ray it wants traced and receives the result; the driver advances all of them
# together and traces each round's requests as (at most two) bundles.  The arithmetic of every
# search -- including scipy's secant iteration, restated step for step -- is that of the
# sequential code above, so the vignetting factors are the same numbers; only the number of
# launches changes (rounds instead of rounds x searches).

def cuda_ray_fn(opt_model, table=None, device=0):
    """``ray_fn(p0 [3, n], d0 [3, n], wvl, check_apertures, pt_inside_fuzz) -> dict`` of host
    arrays ``full [n_ifc, 10, n]``, ``n_seg``, ``status``, ``fail_surf`` on the CUDA engine."""
    from . import engine as E
    from .analyses import _table_for
    tab = _table_for(opt_model, table, device)

    def fn(p0, d0, wvl, check_apertures=False, pt_inside_fuzz=None):
        w = np.full(p0.shape[1], tab.wvl_index(wvl), dtype=np.int32)
        r = E.trace_bundle(tab, p0, d0, wvl_idx=w, full=True, outputs=('n_seg', 'status', 'fail_surf'),
                           first_surf=1, last_surf=tab.n_ifc - 2, check_apertures=check_apertures,
                           pt_inside_fuzz=pt_inside_fuzz, intersect_obj=not _wide(opt_model))
        return {'full': r.full.cpu().numpy(), 'n_seg': r.n_seg.cpu().numpy(),
                'status': r.status.cpu().numpy(), 'fail_surf': r.fail_surf.cpu().numpy()}
    return fn


class _RayAnswer:
    """what a search reads from one traced ray"""
    __slots__ = ('status', 'surf', 'full')

    def __init__(self, status, surf, full):
        self.status, self.surf, self.full = int(status), int(surf), full


def _secant(x0, tol=1e-6, maxiter=50):
    """scipy.optimize.newton(f, x0, tol=tol) without derivative (the secant branch of
    scipy/optimize/_zeros_py.py), as a generator: yields x, receives f(x), returns the root."""
    p0 = 1.0*x0
    eps = 1e-4
    p1 = x0*(1 + eps)
    p1 += (eps if p1 >= 0 else -eps)
    q0 = yield p0
    q1 = yield p1
    if abs(q1) < abs(q0):
        p0, p1, q0, q1 = p1, p0, q1, q0
    p = p1
    for _itr in range(maxiter):
        if q1 == q0:
            return (p1 + p0)/2.0
        if abs(q1) > abs(q0):
            p = (-q0/q1*p1 + p0)/(1 - q0/q1)
        else:
            p = (-q1/q0*p0 + p1)/(1 - q1/q0)
        if np.isclose(p, p1, rtol=0.0, atol=tol):
            return p
        p0, q0 = p1, q1
        p1 = p
        q1 = yield p1
    return p


def _pupil_ray_search(indx, xy, start_r0, r_target):
    """iterate_pupil_ray as a generator of ('free', rel_p1) requests; returns start_coords"""
    start_coords = np.array([0., 0.])
    if indx is None:
        start_coords[xy] = r_target
        return start_coords
    sec = _secant(start_r0)
    try:
        x = next(sec)
        while True:
            rel_p1 = np.array([0., 0.])
            rel_p1[xy] = x
            ans = yield ('free', rel_p1)
            if ans.status != 0:
                limit = indx if ans.status == 1 else indx - 1       # 1: TraceMissedSurfaceError
                if ans.surf <= limit:
                    start_coords[xy] = 0.9*rel_p1[xy]
                    return start_coords
            p = ans.full[indx, 0:3]
            r_ray = math.copysign(math.sqrt(p[0]**2 + p[1]**2), r_target)
            x = sec.send(r_ray - r_target)
    except StopIteration as done:
        start_coords[xy] = done.value
    return start_coords


def _vignetted_ray_search(sm, xy, start_dir, max_iter_count=50):
    """calc_vignetted_ray as a generator of ('clip' | 'free', rel_p1) requests; returns vig"""
    rel_p1 = np.array(start_dir, dtype=float)
    still_iterating, clip_indx, iter_count = True, None, 0
    while still_iterating and iter_count < max_iter_count:
        iter_count += 1
        ans = yield ('clip', rel_p1)
        if ans.status != 0:
            indx = ans.surf
            if indx == clip_indx:
                still_iterating = False
            else:
                r_target = _edge_pt_target(sm.ifcs[indx], start_dir)
                rel_p1 = yield from _pupil_ray_search(indx, xy, rel_p1[xy], r_target[xy])
                clip_indx = indx
        else:
            if clip_indx is not None:
                still_iterating = False
            else:
                stop_indx = sm.stop_surface
                if stop_indx is not None:
                    r_target = _edge_pt_target(sm.ifcs[stop_indx], start_dir)
                    rel_p1 = yield from _pupil_ray_search(stop_indx, xy, rel_p1[xy], r_target[xy])
                    clip_indx = stop_indx
                else:
                    still_iterating = False
    return 1.0 - (rel_p1[xy]/start_dir[xy])


def set_vig_batched(opm, ray_fn=None, wvl=None, max_iter_count=50):
    """``set_vig`` (raytr/vigcalc.py:83-90,227-342,393-471) with the four edge searches of every
    field advanced in lock step: each round traces the pending rays of all searches as one
    bundle per trace option.  Same vignetting factors as ``set_vig``.  Returns the number of
    bundle launches."""
    osp, sm = opm.optical_spec, opm.seq_model
    if ray_fn is None:
        ray_fn = cuda_ray_fn(opm)
    wvl = osp.spectral_region.central_wvl if wvl is None else wvl
    fields = list(osp.field_of_view.fields)
    starts = osp.pupil.pupil_rays[1:]
    searches, want, vig = {}, {}, {}
    for fi in range(len(fields)):
        for i in range(4):
            g = _vignetted_ray_search(sm, i//2, starts[i], max_iter_count)
            searches[(fi, i)] = g
            want[(fi, i)] = next(g)
    launches = 0
    while want:
        answers = {}
        for kind, opts in (('clip', dict(check_apertures=True, pt_inside_fuzz=1e-4)),
                           ('free', dict(check_apertures=False))):
            keys = [k for k, (kd, _) in want.items() if kd == kind]
            if not keys:
                continue
            flds = [fields[k[0]] for k in keys]
            p0, d0 = _start_rays(opm, flds, [f.aim_info for f in flds], [want[k][1] for k in keys])
            r = ray_fn(p0, d0, wvl, **opts)
            launches += 1
            for j, k in enumerate(keys):
                answers[k] = _RayAnswer(r['status'][j], r['fail_surf'][j], r['full'][:, :, j])
        for k, ans in answers.items():
            try:
                want[k] = searches[k].send(ans)
            except StopIteration as done:
                vig[k] = done.value
                del want[k]
    for fi, fld in enumerate(fields):
        fld.vux, fld.vlx, fld.vuy, fld.vly = (vig[(fi, i)] for i in range(4))
    return launches


# --- the bisection search as ONE launch ------------------------------------------------------
def cuda_tile_fn(opt_model, table=None, device=0):
    """``tile_fn(fields, wvl, px, py, **trace options) -> dict(status, fail_surf)``: the pupil points
    ``(px[k], py[k])`` (unvignetted, shared by all fields) of every field in one grid launch"""
    from . import engine as E
    from .analyses import _table_for
    from .opticalspec import grid_fields_of
    tab = _table_for(opt_model, table, device)
    sm = opt_model.seq_model

    def fn(fields, wvl, px, py, **opts):
        recs, eprad, z_pupil = grid_fields_of(opt_model, fields)
        grid = E.PupilGrid(recs, [tab.wvl_index(wvl)], px, py, eprad, z_pupil, apply_vignetting=False,
                           flip_z_dir=sm.z_dir[0], paired=True, device=tab.device)
        res = E.trace_grid(tab, grid, outputs=('status', 'fail_surf'), summary=False, **opts)
        out = {'status': res.status.cpu().numpy(), 'fail_surf': res.fail_surf.cpu().numpy()}
        grid.close()
        return out
    return fn


def bisection_tree(start_dir, levels):
    """Every pupil position ``calc_vignetted_ray_by_bisection`` can visit in ``levels`` halvings,
    in heap order (node i: blocked -> child 2i+1, passed -> child 2i+2), built with the search's own
    update expression so the doubles are the ones it would compute; the last level (never traced)
    holds the possible end positions.  ``[2**(levels+1) - 1, 2]``."""
    sd = np.array(start_dir, dtype=float)
    nodes = np.zeros((2**(levels + 1) - 1, 2))
    nodes[0] = sd
    step, first = 1.0, 0
    for level in range(levels):
        step /= 2
        for i in range(first, first + 2**level):
            nodes[2*i + 1] = -step*sd + nodes[i]
            nodes[2*i + 2] = step*sd + nodes[i]
        first += 2**level
    return nodes


def set_vig_by_bisection(opm, tile_fn=None, wvl=None, levels=10):
    """Vignetting factors of all fields by the bisection search (``calc_vignetted_ray_by_bisection``,
    vigcalc.py:347-390) in ONE launch: the search halves its step a fixed number of times, so the
    pupil positions it can visit form a binary tree known beforehand (2**levels - 1 per pupil
    direction); all of them, for the four directions of every field, are traced together
    (status only, 8 B per ray) and each search becomes a walk down its tree of results.  Same
    factors as the sequential search.  Sets ``vux, vlx, vuy, vly``; returns the limiting
    interface of every (field, direction)."""
    osp, sm = opm.optical_spec, opm.seq_model
    if tile_fn is None:
        tile_fn = cuda_tile_fn(opm)
    wvl = osp.spectral_region.central_wvl if wvl is None else wvl
    fields = list(osp.field_of_view.fields)
    starts = [np.array(sd, dtype=float) for sd in osp.pupil.pupil_rays[1:]]
    trees = [bisection_tree(sd, levels) for sd in starts]
    n_traced = 2**levels - 1
    px = np.concatenate([t[:n_traced, 0] for t in trees])
    py = np.concatenate([t[:n_traced, 1] for t in trees])
    r = tile_fn(fields, wvl, px, py, check_apertures=True, pt_inside_fuzz=1e-4)
    status = np.asarray(r['status']).reshape(len(fields), 4, n_traced)
    surf = np.asarray(r['fail_surf']).reshape(len(fields), 4, n_traced)
    clips = {}
    for fi, fld in enumerate(fields):
        vig = [0.]*4
        for di in range(4):
            node, clip = 0, None
            for _ in range(levels):
                if status[fi, di, node] != 0:
                    clip = int(surf[fi, di, node])
                    node = 2*node + 1
                else:
                    node = 2*node + 2
            xy = di//2
            vig[di] = 1.0 - (trees[di][node][xy]/starts[di][xy])
            clips[(fi, di)] = clip
        fld.vux, fld.vlx, fld.vuy, fld.vly = vig
    return clips


# --- the reference's own aiming iteration (raytr/trace.py:313-415) ----------------------------
def iterate_ray(opt_model, ifcx, xy_target, fld, wvl, trace_fn=None, full=False):
    """Iterate a ray to ``xy_target`` on interface ``ifcx``; returns the aim point on the
    paraxial entrance pupil plane -- ``iterate_ray`` of the reference with the same solvers
    (scipy ``newton`` in 1-D when field and target have x == 0, else ``fsolve`` with
    ``epsfcn = 1e-4 enp_radius``) on top of the engine's ``trace``: with the same residual
    function the iterates are the reference's (tests/test_trace_drivers.py runs the
    reference's own function text next to this one: identical result).

    Note for infinite conjugates: ``obj_coords`` returns the object point mirrored about the
    axis with respect to the ``pt0`` that ``ray_start_from_osp`` builds
    (opticalspec.py:1047-1051 vs :359-366), so the aim point found here has the opposite
    sign of the one ``ray_start_from_osp`` needs -- the aim points stored in the reference's
    ``.roa`` files have the consistent sign.  ``aim_chief_ray`` / ``aim_all_fields_batched``
    above iterate on ``ray_start_from_osp`` itself and reproduce the stored values."""
    from . import raytrace as RT
    if trace_fn is None:
        trace_fn = RT.trace
    seq_model, osp = opt_model.seq_model, opt_model.optical_spec
    fod = osp.fod
    pt0, d0 = osp.obj_coords(fld)
    coords, rr = _iterate_to_target(lambda p, d: trace_fn(seq_model, p, d, wvl), ifcx, xy_target,
                                    pt0, fod.obj_dist + fod.enp_dist, fod.enp_radius,
                                    not osp.field_of_view.is_wide_angle, seq_model.z_dir[0])
    return (coords, rr) if full else coords      # full: the reference's return value


def solver_gave_up(e):
    """is this RuntimeError scipy's own (an iteration that did not converge), as opposed to an
    engine / CUDA failure surfacing inside the residual function?  Only the former may be
    absorbed by the searches the way the reference absorbs it; the latter must stay loud."""
    msg = str(e)
    return (type(e) is RuntimeError
            and any(k in msg for k in ('onverge', 'olerance', 'erivative was zero', 'f(a) and f(b)')))


def _iterate_to_target(trace_one, ifcx, xy_target, pt0, obj2enp_dist, eprad, not_wa, z_dir0):
    """the solver part shared by ``iterate_ray`` and ``iterate_ray_raw`` (trace.py:313-415,
    866-957): returns ``(start_coords, (ray_pkg, error) of the last ray traced)``"""
    import warnings
    from scipy.optimize import newton, fsolve
    from . import raytrace as RT
    last = [None]

    def final_coord(pt1):
        v = pt1 - pt0
        dir0 = v/np.linalg.norm(v)
        if not_wa and dir0[2]*z_dir0 < 0:
            dir0 = -dir0
        try:
            pkg = trace_one(pt0, dir0)
        except RT.TraceError as ray_error:
            last[0] = (ray_error.ray_pkg, ray_error)
            if ray_error.surf < ifcx:
                raise ray_error
            return np.array([0., 0., 0.])
        last[0] = (pkg, None)
        return pkg[0][ifcx][0]

    def y_stop_coordinate(y1, y_target):
        return final_coord(np.array([0., y1, obj2enp_dist]))[1] - y_target

    def surface_coordinate(coord, target):
        fc = final_coord(np.array([coord[0], coord[1], obj2enp_dist]))
        return np.array([fc[0], fc[1]]) - target

    if ifcx is None:                       # floating stop: use the entrance pupil for aiming
        return np.array([0., 0.]) + xy_target, None
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        if pt0[0] == 0.0 and xy_target[0] == 0.0:
            try:
                start_y, results = newton(y_stop_coordinate, 0., args=(xy_target[1],), disp=False,
                                          full_output=True)
            except RuntimeError as e:
                if not solver_gave_up(e):
                    raise
                start_y = 0.0
            except RT.TraceError:
                start_y = 0.0
            return np.array([0., start_y]), last[0]
        try:
            coords = fsolve(surface_coordinate, np.array([0., 0.]), epsfcn=0.0001*eprad,
                            args=(np.array(xy_target, dtype=float),))
        except RT.TraceError:
            coords = np.array([0., 0.])
        return coords, last[0]


def iterate_ray_raw(pthlist, ifcx, xy_target, pt0, d0, obj2pup_dist, eprad, wvl, not_wa,
                    trace_raw_fn=None, **kwargs):
    """``iterate_ray`` on an explicit path list (trace.py:866-957): ``(start_coords, (ray_pkg,
    error))``.  Rays go through the drop-in ``raytrace.trace_raw`` (one single-ray launch each)."""
    from . import raytrace as RT
    trace_raw_fn = RT.trace_raw if trace_raw_fn is None else trace_raw_fn
    pthlist = list(pthlist)
    return _iterate_to_target(lambda p, d: trace_raw_fn(iter(pthlist), p, d, wvl), ifcx, xy_target,
                              np.array(pt0, dtype=float), obj2pup_dist, eprad, not_wa, pthlist[0][4])


def aim_chief_ray_like_reference(opt_model, fld, wvl=None, trace_fn=None):
    """``trace.aim_chief_ray`` (raytr/trace.py:627-640): aim at the centre of the stop surface"""
    sm = opt_model.seq_model
    wvl = sm.central_wavelength() if wvl is None else wvl
    return iterate_ray(opt_model, sm.stop_surface, np.array([0., 0.]), fld, wvl, trace_fn=trace_fn)
