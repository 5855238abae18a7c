"""Wavefront tolerancing on the H100: sensitivity (20 tolerances, 41 variants) and a 1000-trial Monte Carlo
(1001 variants) on the double Gauss and zoom52 (3 fields x 3 wavelengths) at 32^2 and 64^2 rays per tile, with
the RMS wavefront error criterion.  Reports the end-to-end time, its host parts (variant descriptors; the
per-tile statistics and merit) and its device part (wave records + trace + reduce, CUDA events), and the
per-variant route (perturbed model, a SurfaceTable, waveabr.setup_tiles and rt_trace_grid_wfe per variant)
with the largest merit difference between the two routes (expected 0).  The per-variant route of the Monte
Carlo is timed on its first 101 variants.

    python tools/bench_tolerance_wavefront.py [--reps 3] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rayoptics_b200 import analyses as A, engine as E, model as M, tolerance as TOL, waveabr as WA  # noqa: E402
from rayoptics_b200.table import SurfaceTable, describe_model  # noqa: E402

PER_VARIANT_MAX = 101


def tolerances(sm, n):
    kinds = ['radius', 'thickness', 'tilt_x', 'decenter_y', 'index']
    out, i = [], 0
    while len(out) < n:
        k, s = kinds[i % len(kinds)], 1 + (i*3) % (len(sm.ifcs) - 3)
        i += 1
        if (k == 'thickness' and s > len(sm.gaps) - 1) or (k == 'radius' and sm.ifcs[s].profile.cv == 0.0):
            continue
        out.append(TOL.Tolerance(k, s, {'radius': 0.1, 'thickness': 0.02, 'index': 3e-4}.get(k, 0.01)))
    return out


def run(opm, fields, wvls, num_rays, sets, reps):
    sm, osp = opm.seq_model, opm.optical_spec
    foc = osp.defocus.focus_shift
    d0, n0, all_w = describe_model(sm)
    tab0 = SurfaceTable(d0, n0, all_w)
    args, kw = A._wavefront_grid_args(opm, tab0, num_rays, fields, wvls, foc, None, None)
    grid = E.PupilGrid(*args, **kw)
    region = osp.spectral_region
    ww = [region.spectral_wts[list(region.wavelengths).index(w)] for w in wvls]
    fw = [f.wt for f in fields]
    lam = [opm.nm_to_sys_units(w) for w in wvls]
    fod = opm['analysis_results']['parax_data'].fod
    parax = (fod.exp_dist, abs(fod.n_obj), abs(fod.n_img))
    best = None
    for _ in range(reps + 1):                      # the first pass warms up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        var = [TOL.perturbed_descriptors(d0, n0, ch, sm) for ch in sets]
        t1 = time.perf_counter()
        vs = E.VariantSet([v[0] for v in var], np.stack([v[1] for v in var]), all_w)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        wave, _, st = vs.wave(grid, parax)
        rec = E.trace_grid_variants_wfe(vs, grid, wave)
        e1.record()
        host = rec.cpu().numpy()
        t2 = time.perf_counter()
        res = A.wave_merit(host.reshape(len(sets), len(fields), len(wvls), -1), lam, ww, fw, True,
                           st.cpu().numpy().reshape(len(sets), len(fields), len(wvls)))
        t3 = time.perf_counter()
        vs.close()
        r = dict(end_to_end_s=t3 - t0, host_descriptors_s=t1 - t0, host_statistics_s=t3 - t2,
                 device_wave_trace_reduce_s=e0.elapsed_time(e1)*1e-3)
        if best is None or r['end_to_end_s'] < best['end_to_end_s']:
            best = r
    # per-variant route: a perturbed model, a table, the host reference spheres and one wfe trace per variant
    n_pv = min(len(sets), PER_VARIANT_MAX)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    merits = []
    for ch in sets[:n_pv]:
        pm = TOL.perturbed_model(opm, ch)
        tab = SurfaceTable.from_model(pm.seq_model)
        w_h, r_h, _ = WA.setup_tiles(pm, tab, fields, wvls, foc)
        g = E.PupilGrid(*args, **dict(kw, wave=w_h, ref_img=r_h))
        summ = E.trace_grid_wfe(tab, g).cpu().numpy()
        st = E.wavefront_statistics(summ, np.tile(lam, len(fields)))
        merits.append(A.wave_merit_of(st['rms_focus'].reshape(1, len(fields), len(wvls)), ww, fw)[0][0])
        g.close()
        tab.close()
    torch.cuda.synchronize()
    best['per_variant_route_s'] = time.perf_counter() - t0
    best['per_variant_route_variants'] = n_pv
    merits = np.array(merits)
    best['max_abs_merit_diff_waves'] = float(np.nanmax(np.abs(merits - res.merit[:n_pv])))
    best['nominal_merit_waves'] = float(res.merit[0])
    best['n_variants'] = len(sets)
    best['rays_per_variant'] = grid.n_rays
    grid.close()
    tab0.close()
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out', default=None, help='also write the results as JSON to this file')
    a = ap.parse_args()
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    out = {'gpu': gpu, 'results': []}
    for name in ('dblgauss', 'zoom52'):
        opm = M.OpticalModel.load(os.path.join(ROOT, 'tests', 'golden', 'models', f'{name}.json'))
        sm = opm.seq_model
        fields = list(opm.optical_spec.field_of_view.fields)[:3]
        wvls = list(sm.wvlns)
        wvls = [wvls[0], sm.central_wavelength(), wvls[-1]]
        tols = tolerances(sm, 20)
        sens = [[]] + [[(t, sg*t.delta)] for t in tols for sg in (1.0, -1.0)]
        vals = A.draw_tolerances(tols, 1000, seed=0)
        mc = [[]] + [list(zip(tols, row)) for row in vals]
        for num_rays in (32, 64):
            for label, sets in (('sensitivity', sens), ('monte_carlo_1000', mc)):
                r = run(opm, fields, wvls, num_rays, sets, a.reps)
                r.update(model=name, num_rays=num_rays, workload=label)
                print(json.dumps(r), flush=True)
                out['results'].append(r)
    print(gpu)
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
