#!/usr/bin/env python3
"""Are the committed golden vectors what the reference produces today?

Runs every generator under tests/golden/ (they import the reference from /root/reference and
write tests/golden/models, tests/golden/vectors, tests/golden/kat.json in place), compares
the regenerated files with the committed ones array by array, and puts the committed bytes back
whatever happens.  Build container only (the GPU box has no /root/reference).

    python tools/check_golden_reproducible.py        # exit 0: identical
"""
import glob
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, 'tests', 'golden')
GENERATORS = ('make_models.py', 'make_golden.py', 'make_golden_grids.py', 'make_golden_opd.py',
              'make_golden_analyses.py', 'make_golden_edges.py')


def arrays(path):
    z = np.load(path, allow_pickle=True)
    return {k: z[k] for k in z.files}


def same(a, b):
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    return np.array_equal(a, b, equal_nan=True) if a.dtype.kind in 'fiub' else bool((a == b).all())


def main():
    files = sorted(glob.glob(os.path.join(G, 'vectors', '*.npz')) + glob.glob(os.path.join(G, 'models', '*.json'))
                   + [os.path.join(G, 'kat.json')])
    committed = {f: open(f, 'rb').read() for f in files}
    before = {f: arrays(f) for f in files if f.endswith('.npz')}
    bad = []
    try:
        t0 = time.time()
        for script in GENERATORS:
            r = subprocess.run([sys.executable, os.path.join(G, script)], capture_output=True, text=True)
            print(f'{script:26s} rc={r.returncode}  {time.time() - t0:5.1f} s')
            if r.returncode:
                print(r.stderr[-2000:])
                bad.append((script, 'failed'))
        for f in files:
            if f.endswith('.npz'):
                new = arrays(f)
                if set(new) != set(before[f]):
                    bad.append((os.path.basename(f), 'keys'))
                    continue
                bad += [(os.path.basename(f), k) for k in new if not same(new[k], before[f][k])]
            elif open(f, 'rb').read() != committed[f]:
                bad.append((os.path.basename(f), 'text'))
    finally:
        for f, b in committed.items():
            with open(f, 'wb') as fh:
                fh.write(b)
    n_arr = sum(len(v) for v in before.values())
    print(f'{len(files)} files, {n_arr} arrays: ' + ('identical' if not bad else f'DIFFERENCES {bad}'))
    return 1 if bad else 0


if __name__ == '__main__':
    sys.exit(main())
