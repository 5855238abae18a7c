"""Tolerance analysis on the H100: sensitivity (20 tolerances, 41 variants) and a 1000-trial Monte Carlo on
the double Gauss and zoom52 (3 fields x 3 wavelengths) at 32^2 and 64^2 rays per tile.  Reports the end-to-end
time, its host part (variant descriptors) and device part (trace + reduce, CUDA events), and the per-variant
route (a SurfaceTable per variant + rt_trace_grid_focus at that variant's refocused plane) with the merits
compared.

    python tools/bench_tolerance.py [--reps 3] [--out FILE]
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
from rayoptics_b200 import analyses as A, engine as E, model as M, tolerance as TOL  # noqa: E402
from rayoptics_b200.table import SurfaceTable, describe_model  # noqa: E402


def tolerances(sm, n):
    kinds = ['radius', 'thickness', 'tilt_x', 'decenter_y', 'index']
    out, i = [], 0
    while len(out) < n:
        k, s = kinds[i % len(kinds)], 1 + (i*3) % (len(sm.ifcs) - 2)
        i += 1
        if (k == 'thickness' and s > len(sm.gaps) - 1) or (k == 'radius' and sm.ifcs[s].profile.cv == 0.0):
            continue
        out.append(TOL.Tolerance(k, s, {'radius': 0.1, 'thickness': 0.02, 'index': 3e-4}.get(k, 0.01)))
    return out


def run(opm, fields, wvls, num_rays, sets, reps):
    sm, osp = opm.seq_model, opm.optical_spec
    d0, n0, all_w = describe_model(sm)
    tab0 = SurfaceTable(d0, n0, all_w)
    args, kw = E._grid_args(opm, sm.index_for_wavelength, num_rays, fields, wvls, None, (-1.0, 1.0), True)
    grid = E.PupilGrid(*args, **kw)
    grid.chief_ref(tab0, sm.index_for_wavelength(sm.central_wavelength()))
    region = osp.spectral_region
    ww = [region.spectral_wts[list(region.wavelengths).index(w)] for w in wvls]
    fw = [f.wt for f in fields]
    best = None
    for _ in range(reps + 1):                      # the first pass warms up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        var = [TOL.perturbed_descriptors(d0, n0, ch, sm) for ch in sets]
        t1 = time.perf_counter()
        vs = E.VariantSet([v[0] for v in var], np.stack([v[1] for v in var]), all_w)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rec = E.trace_grid_variants(vs, grid)
        e1.record()
        host = rec.cpu().numpy()
        res = A.tol_merit(host.reshape(len(sets), len(fields), len(wvls), -1), ww, fw)
        t2 = time.perf_counter()
        vs.close()
        r = dict(end_to_end_s=t2 - t0, host_descriptors_s=t1 - t0, device_trace_reduce_s=e0.elapsed_time(e1)*1e-3)
        if best is None or r['end_to_end_s'] < best['end_to_end_s']:
            best = r
    # per-variant route: a table per variant, one focus trace at its refocused plane
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    merits = []
    for v, ch in enumerate(sets):
        d, nb = TOL.perturbed_descriptors(d0, n0, ch, sm)
        tab = SurfaceTable(d, nb, all_w)
        summ = E.trace_grid_focus(tab, grid, [grid.foc + res.focus[v]]).cpu().numpy()
        s = summ.reshape(len(fields), len(wvls), 16)
        w = np.asarray(ww)
        n = (s[..., 0]*w).sum(1)
        x1, y1, x2 = (s[..., 5]*w).sum(1), (s[..., 6]*w).sum(1), ((s[..., 7] + s[..., 8])*w).sum(1)
        merits.append(np.sqrt(((x2/n - (x1*x1 + y1*y1)/(n*n))*np.asarray(fw)).sum()/sum(fw)))
        tab.close()
    torch.cuda.synchronize()
    best['per_variant_route_s'] = time.perf_counter() - t0
    merits = np.array(merits)
    best['max_rel_merit_diff'] = float(np.nanmax(np.abs(merits - res.merit)/merits))
    best['n_variants'] = len(sets)
    best['rays_per_variant'] = grid.n_rays
    grid.close()
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
