"""Build + ctypes wrapper of tests/hostsim/tolwave.cpp (TEST INFRASTRUCTURE): the wave-record header
csrc/rt_tolwave.cuh compiled for the host with the flags of build.py, in a library of its own."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, '_build', 'libhostsim_tolwave.so')
SOURCES = [os.path.join(HERE, 'tolwave.cpp'), os.path.join(HERE, 'cuda_runtime.h'),
           os.path.join(ROOT, 'rayoptics_b200', 'csrc', 'rt_tolwave.cuh'),
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


def records(full, op, status, last, foc, parax):
    """The wave records of chief rays by the header: ``full [n_ifc, 10, n]`` whole rays (the
    ``trace_chief_rays`` layout), ``op`` / ``status`` ``[n]``, ``last`` the ``rt_surface_desc`` of interface
    n_ifc - 2, ``parax`` (exp_dist, |n_obj|, |n_img|).  Returns ``(W [n, 24], ref [n, 2], branch [n])``."""
    n = full.shape[2]
    ray = np.ascontiguousarray(np.concatenate([full[1, 0:3], full[0, 3:6], full[-2, 0:3], full[-2, 3:6],
                                               full[-1, 0:3], full[-1, 3:6]], axis=0).T, dtype=np.float64)
    op = np.ascontiguousarray(op, dtype=np.float64)
    st = np.ascontiguousarray(status, dtype=np.int32)
    px = np.ascontiguousarray(parax, dtype=np.float64)
    W, ref, br = np.zeros((n, 24)), np.zeros((n, 2)), np.zeros(n, dtype=np.int32)
    assert lib().hostsim_tolwave(C.c_int64(n), _dp(ray), _dp(op), st.ctypes.data_as(C.POINTER(C.c_int32)),
                                 C.byref(last), C.c_double(foc), _dp(px), _dp(W), _dp(ref),
                                 br.ctypes.data_as(C.POINTER(C.c_int32))) == 0
    return W, ref, br
