"""Build + ctypes wrapper of tests/hostsim/mtf.cpp (TEST INFRASTRUCTURE): the MTF header
csrc/rt_mtf.cuh compiled for the host with the flags of build.py, in a library of its own."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, '_build', 'libhostsim_mtf.so')
SOURCES = [os.path.join(HERE, 'mtf.cpp'), os.path.join(HERE, 'cuda_runtime.h'),
           os.path.join(ROOT, 'rayoptics_b200', 'csrc', 'rt_mtf.cuh')]

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


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def mtf_sums(P):
    """(acf_x [n], acf_y [n], S) of one tile's [n, n] complex pupil function, by the header"""
    P = np.ascontiguousarray(P, dtype=np.complex128)
    n = P.shape[0]
    cx, cy, s = np.full(n, np.nan + 0j), np.full(n, np.nan + 0j), np.full(1, np.nan + 0j)
    assert lib().hostsim_mtf_sums(C.c_int(n), _dp(P), _dp(cx), _dp(cy), _dp(s)) == 0
    return cx, cy, complex(s[0])


def pupil(status, opd, x, y, lam):
    """per-ray phasors of the used rays (the header's rule and mtf_phasor with a sin / cos stand-in)"""
    st = np.ascontiguousarray(status, dtype=np.int32).ravel()
    arrs = [np.ascontiguousarray(np.broadcast_to(v, st.shape), dtype=np.float64) for v in (opd, x, y)]
    out = np.full(len(st), np.nan + 0j)
    assert lib().hostsim_mtf_pupil(C.c_int64(len(st)), st.ctypes.data_as(C.POINTER(C.c_int32)),
                                   *(_dp(a) for a in arrs), C.c_double(lam), _dp(out)) == 0
    return out
