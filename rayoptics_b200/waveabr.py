"""Chief rays, reference spheres and the per-tile records of the OPD epilogue.

Host side of the wavefront stage (SURVEY.md 8(f) row 2).  The per-ray OPD
(``wave_abr_full_calc_finite_pup``, /root/reference/src/rayoptics/raytr/waveabr.py:255-305)
is evaluated by the grid kernel; what it needs per (field, wavelength) tile is
computed here, once, with the reference's own expressions:

* chief ray = pupil (0, 0) traced whole (``trace_chief_ray``, raytr/trace.py:513-534)
  -- all tiles in one launch;
* ``transfer_to_exit_pupil`` (waveabr.py:79-113, interfaces without decenter);
* ``calculate_reference_sphere`` (waveabr.py:24-76).

Both branches of ``wave_abr_full_calc`` (waveabr.py:206-253) are covered: finite
reference spheres and -- for exit pupils farther than 1e8 (telecentric image
space) -- the infinite-reference variant (waveabr.py:356-420), the latter for an
image gap without tilt / decenter.
"""
from __future__ import annotations

import numpy as np

from . import engine as E
from .opticalspec import grid_fields_of
from ._abi import RT_WAVE_DOUBLES, RT_SPHERE_DOUBLES


def normalize(v):
    length = np.linalg.norm(v)
    return v if length == 0.0 else v/length


def is_kinda_big(x, kinda_big=1e8):
    """util/misc_math.py:22-29"""
    return bool(np.isinf(x) or np.abs(x) > kinda_big)


def transfer_to_exit_pupil(ray_seg, exp_dst_parax):
    """waveabr.py:79-113 for an exiting interface without decenter."""
    b4_pt, b4_dir = ray_seg
    h = b4_pt[1]
    u = b4_dir[1]
    if abs(u) < 1e-14:
        exp_dst = exp_dst_parax
    else:
        exp_dst = -h/u
    exp_pt = b4_pt + exp_dst*b4_dir
    return exp_pt, b4_dir, exp_dst, None, b4_pt, b4_dir


def trace_chief_rays(opt_model, table, fields, wvls):
    """Whole chief rays of every (field, wvl): one launch.  Returns
    ``full [n_ifc, 10, n_tiles]``, ``op [n_tiles]``, ``status [n_tiles]`` (numpy)."""
    osp, sm = opt_model.optical_spec, opt_model.seq_model
    recs, eprad, z_pupil = grid_fields_of(opt_model, fields)
    g0 = E.PupilGrid(recs, [table.wvl_index(w) for w in wvls], [0.0], [0.0], eprad, z_pupil,
                     apply_vignetting=True, flip_z_dir=sm.z_dir[0], device=table.device)
    r0 = E.trace_grid(table, g0, outputs=('op', 'status'), full=True, summary=False,
                      check_apertures=False)
    out = r0.full.cpu().numpy(), r0.op.cpu().numpy(), r0.status.cpu().numpy()
    g0.close()
    return out


def chief_ray_pkg(opt_model, full, op, wvl, tile):
    """(cr, cr_exp_seg) of one tile from the bundle output (trace.py:513-534)."""
    n_ifc = full.shape[0]
    ray = [[full[k, 0:3, tile].copy(), full[k, 3:6, tile].copy(), float(full[k, 6, tile]),
            full[k, 7:10, tile].copy()] for k in range(n_ifc)]
    cr = (ray, float(op[tile]), wvl)
    fod = opt_model['analysis_results']['parax_data'].fod
    cr_exp_seg = transfer_to_exit_pupil((ray[-2][0], ray[-2][1]), fod.exp_dist)
    return cr, cr_exp_seg


def calculate_reference_sphere(opt_model, fld, wvl, foc, chief_ray_pkg_, image_pt_2d=None,
                               image_delta=None):
    """waveabr.py:24-76 -> (image_pt, ref_dir, ref_sphere_radius, lcl_tfrm_last)."""
    cr, cr_exp_seg = chief_ray_pkg_
    ray = cr[0]
    if image_pt_2d is None:
        dist = foc/ray[-1][1][2]
        image_pt = ray[-1][0] + dist*ray[-1][1]
    else:
        image_pt = np.array([image_pt_2d[0], image_pt_2d[1], foc])
    if image_delta is not None:
        image_pt[:2] += image_delta
    seq_model = opt_model.seq_model
    lcl_tfrm_last = seq_model.lcl_tfrms[-2]
    image_thi = seq_model.gaps[-1].thi
    img_pt = np.array(image_pt)
    img_pt[2] += image_thi
    ref_sphere_vec = img_pt - cr_exp_seg[0]
    ref_sphere_radius = np.linalg.norm(ref_sphere_vec)
    ref_dir = normalize(ref_sphere_vec)
    return image_pt, ref_dir, ref_sphere_radius, lcl_tfrm_last


def wave_record(opt_model, chief_ray_pkg_, ref_sphere):
    """The RT_WAVE_DOUBLES record of a tile (layout: include/b200rt.h)."""
    cr, cr_exp_seg = chief_ray_pkg_
    ray, cr_op, _ = cr
    image_pt, ref_dir, radius, lcl_tfrm_last = ref_sphere
    fod = opt_model['analysis_results']['parax_data'].fod
    W = np.zeros(RT_WAVE_DOUBLES)
    if is_kinda_big(radius):
        # wave_abr_full_calc_inf_ref (waveabr.py:356-420): everything that depends on the
        # chief ray only, with the reference's expressions
        rt, t = lcl_tfrm_last
        if not np.array_equal(rt, np.identity(3)) or t[0] != 0.0 or t[1] != 0.0:
            raise NotImplementedError('infinite reference sphere with a tilted / decentered image gap')
        k = -2
        p_cr_b4, d_cr_b4 = rt.dot(ray[k][0] - t), rt.dot(ray[k][1])
        op_cr_b4 = np.dot(d_cr_b4, -p_cr_b4)
        W[0:3], W[3:6] = ray[1][0], ray[0][1]
        W[6:9], W[9:12] = ray[-1][0], ray[-1][1]
        W[12] = cr_op + op_cr_b4
        W[13:16] = image_pt
        W[17:20] = d_cr_b4
        W[20] = t[2]
        W[21] = 0.0                      # flag: infinite-reference variant
        W[22], W[23] = abs(fod.n_obj), abs(fod.n_img)
        return W
    W[0:3], W[3:6] = ray[1][0], ray[0][1]
    W[6:9], W[9:12] = ray[-2][0], ray[-2][1]
    W[12] = cr_op
    W[13:16] = cr_exp_seg[0]
    W[16] = cr_exp_seg[2]
    W[17:20] = ref_dir
    W[20] = radius
    W[21] = -1.0 if ref_dir[2]*ray[-1][1][2] < 0 else 1.0
    W[22], W[23] = abs(fod.n_obj), abs(fod.n_img)
    return W


def setup_tiles(opt_model, table, fields, wvls, foc, image_pt_2d=None, image_delta=None,
                ref_wvl_for_image_pt=None, chief_tracer=None):
    """Chief rays + reference spheres of all tiles.

    Returns ``(wave [n_f, n_w, 24], ref_img [n_f, n_w, 2], pkgs)`` where
    ``pkgs[f][w] = (chief_ray_pkg, ref_sphere)``.  ``ref_wvl_for_image_pt``: use
    the image point of that wavelength's chief ray for every wavelength (what
    ``SequentialModel.trace_fan/trace_grid`` do, seq/sequential.py:1015-1040)."""
    full, op, status = _chief_rays(opt_model, table, fields, wvls, chief_tracer)
    return _tiles_at(opt_model, full, op, fields, wvls, foc, image_pt_2d, image_delta, ref_wvl_for_image_pt)


def setup_tiles_focus(opt_model, table, fields, wvls, focs, image_pt_2d=None, image_delta=None,
                      ref_wvl_for_image_pt=None, chief_tracer=None):
    """``setup_tiles`` at every focus shift of ``focs`` from one chief-ray trace.

    Returns ``(wave [K, n_f, n_w, 24], ref_img [K, n_f, n_w, 2], spheres [K, n_f, n_w,
    RT_SPHERE_DOUBLES], pkgs)``: plane k's ``wave``, ``ref_img`` and ``pkgs[k]`` are
    ``setup_tiles(..., foc=focs[k])``'s, and its sphere records (``sphere_record``) the part of them
    that depends on the focus.  A tile
    whose reference sphere is finite at one plane and infinite at another raises ValueError."""
    full, op, status = _chief_rays(opt_model, table, fields, wvls, chief_tracer)
    waves, refs, spheres, all_pkgs = [], [], [], []
    for foc in focs:
        wave, ref_img, pkgs = _tiles_at(opt_model, full, op, fields, wvls, foc, image_pt_2d, image_delta,
                                        ref_wvl_for_image_pt)
        waves.append(wave)
        refs.append(ref_img)
        all_pkgs.append(pkgs)
        spheres.append([[sphere_record(wave[fi, wi], rs) for wi, (_, rs) in enumerate(row)]
                        for fi, row in enumerate(pkgs)])
    wave = np.array(waves)
    inf = wave[..., 21] == 0.0
    if (inf != inf[:1]).any():
        raise ValueError('a tile\'s reference sphere is finite at some focus shifts and infinite at others')
    return wave, np.array(refs), np.array(spheres), all_pkgs


def sphere_record(W, ref_sphere):
    """The RT_SPHERE_DOUBLES record of a tile (layout: include/b200rt.h rt_trace_grid_opd_focus) from its
    wave record ``W`` and ``calculate_reference_sphere``'s result: ref_dir, radius, sign_soln (0 on tiles
    of the infinite-reference variant), image_pt."""
    image_pt, ref_dir, radius, _ = ref_sphere
    S = np.zeros(RT_SPHERE_DOUBLES)
    S[0:3], S[3], S[4], S[5:8] = ref_dir, radius, W[21], image_pt
    return S


def _chief_rays(opt_model, table, fields, wvls, chief_tracer):
    # chief_tracer: test seam (the CPU suite feeds the oracle), same role as trace.py's tracer=
    full, op, status = (trace_chief_rays(opt_model, table, fields, wvls) if chief_tracer is None
                        else chief_tracer(opt_model, fields, wvls))
    if (status != 0).any():
        raise RuntimeError('a chief ray did not reach the image')
    return full, op, status


def _tiles_at(opt_model, full, op, fields, wvls, foc, image_pt_2d, image_delta, ref_wvl_for_image_pt):
    """the body of setup_tiles for traced chief rays"""
    nf, nw = len(fields), len(wvls)
    wave = np.zeros((nf, nw, RT_WAVE_DOUBLES))
    ref_img = np.zeros((nf, nw, 2))
    pkgs = []
    for fi, fld in enumerate(fields):
        row = []
        base_pt = image_pt_2d
        if ref_wvl_for_image_pt is not None and image_pt_2d is None:
            wi0 = wvls.index(ref_wvl_for_image_pt)
            crp = chief_ray_pkg(opt_model, full, op, wvls[wi0], fi*nw + wi0)
            base_pt = calculate_reference_sphere(opt_model, fld, wvls[wi0], foc, crp)[0]
        for wi, wvl in enumerate(wvls):
            crp = chief_ray_pkg(opt_model, full, op, wvl, fi*nw + wi)
            rs = calculate_reference_sphere(opt_model, fld, wvl, foc, crp, base_pt, image_delta)
            wave[fi, wi] = wave_record(opt_model, crp, rs)
            ref_img[fi, wi] = rs[0][:2]
            row.append((crp, rs))
        pkgs.append(row)
    return wave, ref_img, pkgs


# --- per-ray OPD on the host (for img_filter callbacks of trace.trace_fan/trace_grid;
#     the batched analyses use the kernel epilogue instead) ---------------------------------
def eic_distance(r, r0):
    """equally inclined chord distance, waveabr.py:117-132 (r = (p, d))"""
    e = (np.dot(r[1] + r0[1], r[0] - r0[0])/(1. + np.dot(r[1], r0[1])))
    return e


def ray_dist_to_perp_from_pt(r, pt):
    """distance along the ray ``r = (p, d)`` to the foot of the perpendicular from ``pt`` (waveabr.py:135-148)"""
    return np.dot(r[1], (pt - r[0]))


def ray_dist_to_perp_from_origin(r):
    """the same for the origin (waveabr.py:151-161)"""
    return np.dot(r[1], -r[0])


def dist_to_shortest_join(r1, r2):
    """points (and distances) of the closest join of two rays, waveabr.py:163-187"""
    p1, d1 = r1
    p2, d2 = r2
    del_p = p2 - p1
    n = np.cross(d1, d2)
    nn = np.dot(n, n)
    if nn == 0:
        t2 = np.dot((p1 - p2), d1)*np.dot(d1, d2)
        return (p1, 0), (p2 + t2*d2, t2)
    t1 = np.dot(np.cross(d2, n), del_p)/nn
    t2 = np.dot(np.cross(d1, n), del_p)/nn
    return (p1 + t1*d1, t1), (p2 + t2*d2, t2)


def wave_abr_full_calc_inf_ref(fod, fld, wvl, foc, ray_pkg, chief_ray_pkg_, ref_sphere):
    """waveabr.py:356-420 (Miks: infinite reference sphere), same expressions."""
    image_pt, ref_dir, ref_sphere_radius, lcl_tfrm_last = ref_sphere
    cr, cr_exp_seg = chief_ray_pkg_
    cr_ray, cr_op, _ = cr
    ray, ray_op, _ = ray_pkg
    k = -2
    n_obj, n_img = abs(fod.n_obj), abs(fod.n_img)
    e1 = eic_distance((ray[1][0], ray[0][1]), (cr_ray[1][0], cr_ray[0][1]))
    if lcl_tfrm_last is not None:
        rt, t = lcl_tfrm_last
        p_b4, d_b4 = rt.dot(ray[k][0] - t), rt.dot(ray[k][1])
        p_cr_b4, d_cr_b4 = rt.dot(cr_ray[k][0] - t), rt.dot(cr_ray[k][1])
    else:
        p_b4, d_b4 = ray[k][0], ray[k][1]
        p_cr_b4, d_cr_b4 = cr_ray[k][0], cr_ray[k][1]
    op_b4 = np.dot(d_b4, -p_b4)
    op_cr_b4 = np.dot(d_cr_b4, -p_cr_b4)
    P1, P2 = dist_to_shortest_join((cr_ray[-1][0], cr_ray[-1][1]), (ray[-1][0], ray[-1][1]))
    rF0 = (P1[0] + P2[0])/2
    V_B = ray_op + op_b4
    V_BE = cr_op + op_cr_b4
    W0 = V_B - V_BE + n_img*np.dot((d_b4 - d_cr_b4), rF0)
    ta = ray[-1][0] - image_pt
    numer = np.dot(d_cr_b4 - d_b4*np.dot(d_b4, d_cr_b4), ta)
    denom = 1 + np.dot(d_b4, d_cr_b4)
    W_inf = W0 + n_img*numer/denom
    return -n_obj*e1 - W_inf


def wave_abr_full_calc(fod, fld, wvl, foc, ray_pkg, chief_ray_pkg_, ref_sphere):
    """OPD of a ray w.r.t. the chief ray (``wave_abr_full_calc``, waveabr.py:206-253):
    finite reference sphere (``..._finite_pup``, :255-305, ``F**2`` on a numpy scalar
    included) or the infinite-reference variant.  System units."""
    from math import sqrt
    image_pt, ref_dir, ref_sphere_radius, lcl_tfrm_last = ref_sphere
    if is_kinda_big(ref_sphere_radius):
        return wave_abr_full_calc_inf_ref(fod, fld, wvl, foc, ray_pkg, chief_ray_pkg_, ref_sphere)
    cr, cr_exp_seg = chief_ray_pkg_
    cr_ray, cr_op, _ = cr
    cr_exp_pt, cr_exp_dir, cr_exp_dist, ifc, cr_b4_pt, cr_b4_dir = cr_exp_seg
    ray, ray_op, _ = ray_pkg
    k = -2
    e1 = eic_distance((ray[1][0], ray[0][1]), (cr_ray[1][0], cr_ray[0][1]))
    ekp = eic_distance((ray[k][0], ray[k][1]), (cr_ray[k][0], cr_ray[k][1]))
    b4_pt, b4_dir = ray[k][0], ray[k][1]            # transform_after_surface(None, ...)
    dst = ekp - cr_exp_dist
    eic_exp_pt = b4_pt - dst*b4_dir
    p_coord = eic_exp_pt - cr_exp_pt
    F = ref_dir.dot(b4_dir) - b4_dir.dot(p_coord)/ref_sphere_radius
    J = p_coord.dot(p_coord)/ref_sphere_radius - 2.0*ref_dir.dot(p_coord)
    sign_soln = -1 if ref_dir[2]*cr_ray[-1][1][2] < 0 else 1
    denom = F + sign_soln*sqrt(F**2 + J/ref_sphere_radius)
    ep = 0 if denom == 0 else J/denom
    n_obj = abs(fod.n_obj)
    n_img = abs(fod.n_img)
    opd = -n_obj*e1 - ray_op + n_img*ekp + cr_op - n_img*ep
    return opd


# --- focus-independent / focus-dependent halves of the OPD (rapid refocus without a retrace):
#     wave_abr_pre_calc / wave_abr_calc, waveabr.py:226-253 and their finite-pupil (:310-353) and
#     infinite-reference (:427-488) variants.  The split changes the rounding (the last
#     subtraction happens on ``pre_opd``), so the two halves are restated, not derived from the
#     full calculation above.
def _image_space_frame(ref_sphere, seg):
    """(p, d) of a ray segment in the coordinates of the image interface when the last gap has
    a transform (the infinite-reference variants), the segment itself otherwise"""
    lcl_tfrm_last = ref_sphere[3]
    if lcl_tfrm_last is None:
        return seg[0], seg[1]
    rt, t = lcl_tfrm_last
    return rt.dot(seg[0] - t), rt.dot(seg[1])


def wave_abr_pre_calc(fod, fld, wvl, foc, ray_pkg, chief_ray_pkg_, ref_sphere):
    """Everything of a ray's OPD that does not depend on the image point: the tuple the
    reference's ``focus_*`` functions hand back to ``wave_abr_calc``.
    finite pupil -> ``(pre_opd, p_coord, b4_pt, b4_dir)``;
    infinite reference -> ``(pre_opd, W0, p_b4, d_b4, p_cr_b4, d_cr_b4)``."""
    cr, cr_exp_seg = chief_ray_pkg_
    cr_ray, cr_op, _ = cr
    ray, ray_op, _ = ray_pkg
    k = -2
    n_obj, n_img = abs(fod.n_obj), abs(fod.n_img)
    e1 = eic_distance((ray[1][0], ray[0][1]), (cr_ray[1][0], cr_ray[0][1]))
    if is_kinda_big(ref_sphere[2]):
        p_b4, d_b4 = _image_space_frame(ref_sphere, ray[k])
        p_cr_b4, d_cr_b4 = _image_space_frame(ref_sphere, cr_ray[k])
        op_b4 = np.dot(d_b4, -p_b4)
        op_cr_b4 = np.dot(d_cr_b4, -p_cr_b4)
        P1, P2 = dist_to_shortest_join((cr_ray[-1][0], cr_ray[-1][1]), (ray[-1][0], ray[-1][1]))
        rF0 = (P1[0] + P2[0])/2
        V_B = ray_op + op_b4
        V_BE = cr_op + op_cr_b4
        W0 = V_B - V_BE + n_img*np.dot((d_b4 - d_cr_b4), rF0)
        return -n_obj*e1 - W0, W0, p_b4, d_b4, p_cr_b4, d_cr_b4
    cr_exp_pt, cr_exp_dist = cr_exp_seg[0], cr_exp_seg[2]
    ekp = eic_distance((ray[k][0], ray[k][1]), (cr_ray[k][0], cr_ray[k][1]))
    pre_opd = -n_obj*e1 - ray_op + n_img*ekp + cr_op
    b4_pt, b4_dir = ray[k][0], ray[k][1]            # transform_after_surface(None, ...)
    dst = ekp - cr_exp_dist
    eic_exp_pt = b4_pt - dst*b4_dir
    return pre_opd, eic_exp_pt - cr_exp_pt, b4_pt, b4_dir


def wave_abr_calc(fod, fld, wvl, foc, ray_pkg, chief_ray_pkg_, pre_opd_pkg, ref_sphere):
    """OPD of a ray from its ``wave_abr_pre_calc`` tuple and the (refocused / shifted)
    reference sphere.  System units."""
    from math import sqrt
    image_pt, ref_dir, ref_sphere_radius, _ = ref_sphere
    n_img = abs(fod.n_img)
    if is_kinda_big(ref_sphere_radius):
        pre_opd, W0, p_b4, d_b4, p_cr_b4, d_cr_b4 = pre_opd_pkg
        ta = ray_pkg[0][-1][0] - image_pt
        numer = np.dot(d_cr_b4 - d_b4*np.dot(d_b4, d_cr_b4), ta)
        denom = 1 + np.dot(d_b4, d_cr_b4)
        return pre_opd - n_img*numer/denom
    pre_opd, p_coord, b4_pt, b4_dir = pre_opd_pkg
    cr_ray = chief_ray_pkg_[0][0]
    F = ref_dir.dot(b4_dir) - b4_dir.dot(p_coord)/ref_sphere_radius
    J = p_coord.dot(p_coord)/ref_sphere_radius - 2.0*ref_dir.dot(p_coord)
    sign_soln = -1 if ref_dir[2]*cr_ray[-1][1][2] < 0 else 1
    denom = F + sign_soln*sqrt(F**2 + J/ref_sphere_radius)
    ep = 0 if denom == 0 else J/denom
    return pre_opd - n_img*ep
