"""Build + ctypes wrapper of tests/hostsim/zernike.cpp (TEST INFRASTRUCTURE): the Fringe Zernike
header csrc/rt_zernike.cuh compiled for the host with the flags of build.py, in a library of its
own."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, '_build', 'libhostsim_zernike.so')
SOURCES = [os.path.join(HERE, 'zernike.cpp'), os.path.join(HERE, 'cuda_runtime.h'),
           os.path.join(ROOT, 'rayoptics_b200', 'csrc', 'rt_zernike.cuh')]
MAX_COEFS = 8

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


def _ip(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


def zernike_terms(x, y, n_terms):
    """``[n, n_terms]`` fringe_zernike at the points (x, y)"""
    x = np.ascontiguousarray(x, dtype=np.float64).ravel()
    y = np.ascontiguousarray(y, dtype=np.float64).ravel()
    z = np.full((len(x), n_terms), np.nan)
    assert lib().hostsim_zernike_terms(C.c_int64(len(x)), _dp(x), _dp(y), C.c_int(n_terms), _dp(z)) == 0
    return z


def fringe_table():
    """[(n, m, 'cos' | 'sin' | None, coefficients)] of RT_FRINGE_TABLE"""
    n, m, s, k = (np.zeros(37, np.int32) for _ in range(4))
    coef = np.zeros((37, MAX_COEFS))
    assert lib().hostsim_fringe_table(_ip(n), _ip(m), _ip(s), _ip(k), _dp(coef)) == 37
    return [(int(n[j]), int(m[j]), None if m[j] == 0 else ('sin' if s[j] else 'cos'),
             tuple(int(c) for c in coef[j, :k[j]])) for j in range(37)]
