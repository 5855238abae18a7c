"""Build + ctypes wrapper of tests/hostsim/illum.cpp (TEST INFRASTRUCTURE): the relative-illumination
header csrc/rt_illum.cuh compiled for the host with the flags of build.py, in a library of its own."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, '_build', 'libhostsim_illum.so')
SOURCES = [os.path.join(HERE, 'illum.cpp'), os.path.join(HERE, 'cuda_runtime.h'),
           os.path.join(ROOT, 'rayoptics_b200', 'csrc', 'rt_illum.cuh')]

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


def illum_tile(status, L, M, x, y):
    """(record [RT_ILLUM_DOUBLES], kinds [4]) of one tile by the header: kinds counts the central,
    forward, backward and not-formed derivatives of the used rays over both axes"""
    n = len(x)
    st = np.ascontiguousarray(status, dtype=np.int32).reshape(n, n)
    L, M = (np.ascontiguousarray(a, dtype=np.float64).reshape(n, n) for a in (L, M))
    x, y = np.ascontiguousarray(x, dtype=np.float64), np.ascontiguousarray(y, dtype=np.float64)
    rec, kinds = np.full(10, np.nan), np.zeros(4, dtype=np.int64)
    assert lib().hostsim_illum_tile(C.c_int(n), st.ctypes.data_as(C.POINTER(C.c_int32)), _dp(L), _dp(M),
                                    _dp(x), _dp(y), _dp(rec), kinds.ctypes.data_as(C.POINTER(C.c_int64))) == 0
    return rec, kinds
