"""Time a through-focus curve: one ``analyses.through_focus`` call at K planes against K
``spot_diagram`` calls, on the double Gauss (3 fields x 3 wavelengths) at num_rays x num_rays
rays per tile.  Synchronised wall clock per call (both end in a device -> host copy), median of
--reps.  Prints the card name and power limit of this run, checks that plane 0 of through_focus
has the counts and RMS radii of the single-focus spot_diagram, and writes one JSON line.

    python tools/bench_through_focus.py [--num-rays 512] [--planes 1 8 32] [--reps 5] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def timed(fn, reps):
    import torch
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--num-rays', type=int, default=512)
    ap.add_argument('--planes', type=int, nargs='+', default=[1, 8, 32])
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    from rayoptics_b200 import model as M, analyses as A
    if not torch.cuda.is_available():
        sys.exit('bench_through_focus needs a CUDA device')
    opm = M.OpticalModel.load(os.path.join(ROOT, 'tests', 'golden', 'models', 'dblgauss.json'))
    rows = []
    for k in a.planes:
        foc = np.linspace(-0.1, 0.1, k) if k > 1 else np.array([0.0])
        A.through_focus(opm, a.num_rays, foc=foc)                        # warm-up of this shape
        A.spot_diagram(opm, a.num_rays, foc=float(foc[0]))
        t_tf, tf = timed(lambda: A.through_focus(opm, a.num_rays, foc=foc), a.reps)
        t_sd, sds = timed(lambda: [A.spot_diagram(opm, a.num_rays, foc=float(f)) for f in foc], a.reps)
        s0, t0 = sds[0].summary, tf.summary
        same = bool(all((t0[key][0] == s0[key]).all() for key in ('n_ok', 'n_missed', 'n_tir', 'n_blocked'))
                    and np.allclose(t0['rms_radius'][0], s0['rms_radius'], rtol=1e-12, atol=0))
        rows.append({'planes': int(k), 'through_focus_s': t_tf, 'spot_diagrams_s': t_sd,
                     'ratio': t_sd/t_tf, 'plane0_matches_spot_diagram': same})
        print(f'K={k:3d}  through_focus {t_tf*1e3:9.3f} ms   {k} x spot_diagram {t_sd*1e3:9.3f} ms   '
              f'ratio {t_sd/t_tf:6.2f}   plane 0 = spot_diagram: {same}')
    rec = {'bench': 'through_focus', 'model': 'dblgauss', 'num_rays': a.num_rays, 'card': card(),
           'rays_per_plane': int(tf.n_fields*tf.n_wvls*a.num_rays*a.num_rays), 'rows': rows}
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')
    if not all(r['plane0_matches_spot_diagram'] for r in rows):
        sys.exit('plane 0 does not match the single-focus spot diagram')


if __name__ == '__main__':
    main()
