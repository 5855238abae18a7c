"""Build + ctypes wrapper of tests/hostsim/refocus.cpp (TEST INFRASTRUCTURE): the refocus header
csrc/rt_refocus.cuh compiled for the host with the flags of build.py, in a library of its own."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, '_build', 'libhostsim_refocus.so')
SOURCES = [os.path.join(HERE, 'refocus.cpp'), os.path.join(HERE, 'cuda_runtime.h'),
           os.path.join(ROOT, 'rayoptics_b200', 'csrc', 'rt_refocus.cuh'),
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


def refocus(W, full, ray_op, spheres):
    """``[K]`` OPDs of one traced ray against ``spheres`` ``[K, RT_SPHERE_DOUBLES]``, by the header.
    ``full``: the ray's ``[n_ifc, 10]`` whole-ray record (p, d, dst, normal per interface); ``W``: its
    tile's wave record."""
    full = np.asarray(full, dtype=np.float64)
    ray = np.ascontiguousarray(np.concatenate([full[1, 0:3], full[0, 3:6], full[-2, 0:3], full[-2, 3:6],
                                               full[-1, 0:3], full[-1, 3:6]]))
    W = np.ascontiguousarray(W, dtype=np.float64)
    S = np.ascontiguousarray(spheres, dtype=np.float64)
    out = np.full(S.shape[0], np.nan)
    assert lib().hostsim_refocus(_dp(W), _dp(ray), C.c_double(ray_op), _dp(S), C.c_int(S.shape[0]), _dp(out)) == 0
    return out
