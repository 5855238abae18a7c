"""Build + ctypes wrapper of tests/hostsim/tolerance.cpp (TEST INFRASTRUCTURE): the tolerance header
csrc/rt_tol.cuh compiled for the host with the flags of build.py, in a library of its own."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, '_build', 'libhostsim_tolerance.so')
SOURCES = [os.path.join(HERE, 'tolerance.cpp'), os.path.join(HERE, 'cuda_runtime.h'),
           os.path.join(ROOT, 'rayoptics_b200', 'csrc', 'rt_tol.cuh'),
           os.path.join(ROOT, 'rayoptics_b200', 'csrc', 'rt_device.cuh'),
           os.path.join(ROOT, 'include', 'b200rt.h')]

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


def summands(ax, ay, op, dx, dy, dz):
    """``[n, 24]``: the summands of every ray at their record columns, by the header"""
    arrs = [np.ascontiguousarray(a, dtype=np.float64) for a in (ax, ay, op, dx, dy, dz)]
    n = len(arrs[0])
    out = np.zeros((n, 24))
    assert lib().hostsim_tol_summands(C.c_int64(n), *[_dp(a) for a in arrs], _dp(out)) == 0
    return out
