"""Time chief-ray aiming on the device and the full-field map.

1. ``vigcalc.aim_fields_on_device`` against ``vigcalc.aim_all_fields_batched`` (CUDA bundles, the
   Newton iteration on the host) for 9 x 9, 17 x 17 and 33 x 33 field points over [-1, 1]^2 of the
   double Gauss and the zoom lens: synchronised wall clock, median of --reps after a warm-up;
2. ``k_aim_chief`` alone (``engine.aim_chief_rays`` on an uploaded grid), CUDA events;
3. ``analyses.field_map`` end to end at 9 x 9 points x 3 wavelengths x 32^2 rays and at 17 x 17 x
   64^2 on the double Gauss, split into aiming, chief rays + ``waveabr.setup_tiles`` (host), the opd
   trace and the Zernike moments.

Prints the card name, power limit and maximum SM clock of this run and writes one JSON line.

    python tools/bench_field_map.py [--reps 5] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_zernike import card, per_launch_ms, timed          # noqa: E402


def grid_fields(opm, n):
    from rayoptics_b200.model import Field
    fov = opm.optical_spec.field_of_view
    s = fov.max_field()[0]
    u = np.linspace(-1.0, 1.0, n)
    return [Field(x=float(s*a), y=float(s*b), fov=fov) for a in u for b in u]


def aiming(opm, n, reps, warmup, launches, rounds):
    from rayoptics_b200 import analyses as A, engine as E, vigcalc as V
    from rayoptics_b200.opticalspec import grid_fields_of
    fov = opm.optical_spec.field_of_view
    own = fov.fields
    fields = grid_fields(opm, n)
    fov.fields = fields
    try:
        V.aim_all_fields_batched(opm)
        t_host, host = timed(lambda: np.array(V.aim_all_fields_batched(opm)), reps)
    finally:
        fov.fields = own
    V.aim_fields_on_device(opm, fields)
    t_dev, dev = timed(lambda: np.array(V.aim_fields_on_device(opm, fields)), reps)
    on = np.array([f.x == 0.0 for f in fields])
    tab = A._table_for(opm)
    sm = opm.seq_model
    recs, eprad, z_pupil = grid_fields_of(opm, fields)
    wi = tab.wvl_index(opm.optical_spec.spectral_region.central_wvl)
    grid = E.PupilGrid(recs, [wi], [0.0], [0.0], eprad, z_pupil, apply_vignetting=False, flip_z_dir=sm.z_dir[0],
                       device=tab.device)
    h = 1e-4*max(1.0, opm.optical_spec.fod.enp_radius)
    k = per_launch_ms(lambda: E.aim_chief_rays(tab, grid, sm.stop_surface, wi, h), warmup, launches, rounds)
    grid.close()
    return {'fields': n*n, 'aim_fields_on_device_s': t_dev, 'aim_all_fields_batched_s': t_host,
            'ratio': t_host/t_dev, 'kernel_aim_chief_ms': k,
            'on_meridian_identical': bool(np.array_equal(dev[on].view(np.uint64), host[on].view(np.uint64))),
            'max_abs_aim_diff_mm': float(np.abs(dev - host).max())}


def field_map_split(opm, n, num_rays, reps):
    """field_map end to end and its steps, each synchronised, median of reps"""
    import torch
    from rayoptics_b200 import analyses as A, engine as E, vigcalc as V, waveabr as W
    wvls = list(opm.seq_model.wvlns)
    osp = opm.optical_spec
    A.field_map(opm, n, num_rays, 37)
    t_all, fm = timed(lambda: A.field_map(opm, n, num_rays, 37), reps)
    fov = osp.field_of_view
    from rayoptics_b200.model import Field
    pts = [Field(x=float(fm.field_x[i, j]), y=float(fm.field_y[i, j]), fov=fov)
           for i, j in zip(*np.nonzero(fm.traced))]
    tab = A._table_for(opm)
    t_aim, _ = timed(lambda: V.aim_fields_on_device(opm, pts), reps)
    t_chief, _ = timed(lambda: W.trace_chief_rays(opm, tab, pts, wvls), reps)
    foc = osp.defocus.focus_shift
    t_setup, (args, kw) = timed(lambda: A.wavefront_grid_args(opm, tab, num_rays, pts, wvls, foc), reps)
    grid = E.PupilGrid(*args, device=tab.device, **kw)
    res = E.BundleResult(grid.n_rays, tab.n_ifc, torch.device('cuda', tab.device), ('opd', 'status'))
    t_trace, _ = timed(lambda: E.trace_grid(tab, grid, res=res, summary=False, check_apertures=True), reps)
    t_mom, _ = timed(lambda: E.grid_zernike(grid, 0, grid.n_chunks, 37, res.status, res.opd), reps)
    grid.close()
    return {'points': int(fm.traced.sum()), 'wvls': len(wvls), 'num_rays': num_rays, 'field_map_s': t_all,
            'aim_s': t_aim, 'chief_rays_keep_check_s': t_chief, 'setup_tiles_host_s': t_setup,
            'opd_trace_s': t_trace, 'moments_s': t_mom}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--launches', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    from rayoptics_b200 import model as M
    if not torch.cuda.is_available():
        sys.exit('bench_field_map needs a CUDA device')
    rec = {'bench': 'field_map', 'card': card()}
    print(f'card (name, power limit, max SM clock): {rec["card"]}')
    models = {name: M.OpticalModel.load(os.path.join(ROOT, 'tests', 'golden', 'models', name + '.json'))
              for name in ('dblgauss', 'zoom52')}
    ok = True
    for name, opm in models.items():
        for n in (9, 17, 33):
            r = aiming(opm, n, a.reps, a.warmup, a.launches, a.rounds)
            ok &= r['on_meridian_identical'] and r['max_abs_aim_diff_mm'] <= 1e-4
            rec[f'aim_{name}_{n * n}'] = r
            print(f'{name} {n*n:5d} fields: device {r["aim_fields_on_device_s"]*1e3:9.3f} ms   host iteration '
                  f'{r["aim_all_fields_batched_s"]*1e3:9.3f} ms   ratio {r["ratio"]:7.1f}   k_aim_chief '
                  f'{r["kernel_aim_chief_ms"][0]:7.3f} ms   max |diff| {r["max_abs_aim_diff_mm"]:.2g} mm')
    for n, num in ((9, 32), (17, 64)):
        r = field_map_split(models['dblgauss'], n, num, a.reps)
        rec[f'field_map_{n}x{n}_{num}'] = r
        print(f'field_map dblgauss {n}x{n} ({r["points"]} points) x {r["wvls"]} wvls x {num}^2: '
              f'{r["field_map_s"]*1e3:9.3f} ms = aim {r["aim_s"]*1e3:.3f} + chief rays {r["chief_rays_keep_check_s"]*1e3:.3f} '
              f'+ setup_tiles {r["setup_tiles_host_s"]*1e3:.3f} + opd trace {r["opd_trace_s"]*1e3:.3f} '
              f'+ moments {r["moments_s"]*1e3:.3f} ms (steps timed separately)')
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')
    if not ok:
        sys.exit('device aims do not meet the agreement with aim_all_fields_batched')


if __name__ == '__main__':
    main()
