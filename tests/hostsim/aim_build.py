"""Build + ctypes wrapper of tests/hostsim/aim.cpp (TEST INFRASTRUCTURE): the chief-ray aiming of
csrc/rt_aim.cuh compiled for the host with the flags of build.py, in a library of its own."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, '_build', 'libhostsim_aim.so')
SOURCES = [os.path.join(HERE, 'aim.cpp'), os.path.join(HERE, 'cuda_runtime.h'),
           os.path.join(ROOT, 'include', 'b200rt.h')] + \
          [os.path.join(ROOT, 'rayoptics_b200', 'csrc', h) for h in ('rt_aim.cuh', 'rt_grid.cuh', 'rt_device.cuh')]

_lib = None


def build(force=False):
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    stale = force or not os.path.exists(LIB) or \
        any(os.path.getmtime(s) > os.path.getmtime(LIB) for s in SOURCES)
    if stale:
        subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-mfma', '-DRT_HOSTSIM',
                               '-fPIC', '-shared', '-I', HERE, '-o', LIB, SOURCES[0]])
    return LIB


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
    return _lib


def aim_chief(descs, n_by_wvl, wvls, spec, stop, wvl_idx, h, tol=1e-13, max_iter=30):
    """spec: rt_grid_spec (PupilGridSpec.c_spec()) -> (aim [n, 2], term [n], iters [n])"""
    n = spec.n_fields        # spec: rt_grid_spec
    nbw = np.ascontiguousarray(n_by_wvl, dtype=np.float64)
    wl = None if wvls is None else np.ascontiguousarray(wvls, dtype=np.float64)
    aim = np.full((n, 2), np.nan)
    term = np.full(n, -1, dtype=np.int32)
    iters = np.full(n, -1, dtype=np.int32)
    dp = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))      # noqa: E731
    ip = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))                               # noqa: E731
    rc = lib().hostsim_aim_chief(descs, C.c_int(len(descs)), dp(nbw), dp(wl), C.byref(spec), C.c_int(stop),
                                 C.c_int(wvl_idx), C.c_double(h), C.c_double(tol), C.c_int(max_iter),
                                 dp(aim), ip(term), ip(iters))
    assert rc == 0
    return aim, term, iters
