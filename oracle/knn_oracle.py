"""ctypes front-end of the brute-force kNN oracle (oracle/knn_oracle.cpp) — TEST INFRASTRUCTURE ONLY.

Same names, arguments and flat return layout as the reference's simple_knn._C (ext.cpp:16-18), on numpy arrays:
    distCUDA2(points)                         -> float32 [P]
    distIndex2(points, K)                     -> (float32 [P*K], int32 [P*K])
    distIndexQ(points, q_indices, n_indices, K) -> (float32 [Q*K], int32 [Q*K])
Rows are sorted by (distance, index); see knn_oracle.cpp for the contract.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "knn_oracle.cpp")
LIB = os.path.join(HERE, "libknn_oracle.so")
_lib = None


def build(force: bool = False) -> str:
    if force or not os.path.isfile(LIB) or os.path.getmtime(LIB) < os.path.getmtime(SRC):
        cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fno-fast-math",
               "-fvisibility=hidden", "-o", LIB, SRC]
        subprocess.run(cmd, check=True)
    return LIB


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.ko_knn.restype = None
        _lib.ko_knn.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return _lib


def _np(x, dtype):
    if hasattr(x, "detach"):
        x = x.detach().cpu().numpy()
    return np.ascontiguousarray(x, dtype=dtype)


def _ptr(a):
    return None if a is None or a.size == 0 else a.ctypes.data


def knn(points, K, q_indices=None, n_indices=None, mean=False):
    """(dists [rows*K], indices [rows*K], mean3 [rows] or None)."""
    pts = _np(points, np.float32).reshape(-1, 3)
    P = pts.shape[0]
    q = None if q_indices is None else _np(q_indices, np.int32).reshape(-1)
    n = None if n_indices is None else _np(n_indices, np.int32).reshape(-1)
    rows = P if q is None else q.shape[0]
    d = np.empty(rows * K, np.float32)
    i = np.empty(rows * K, np.int32)
    m = np.empty(rows, np.float32) if mean else None
    lib().ko_knn(_ptr(pts), P, int(K), _ptr(q), -1 if q is None else q.shape[0], _ptr(n), -1 if n is None else n.shape[0],
                 _ptr(d), _ptr(i), _ptr(m))
    return d, i, m


def distCUDA2(points):
    return knn(points, 3, mean=True)[2]


def distIndex2(points, K):
    d, i, _ = knn(points, K)
    return d, i


def distIndexQ(points, q_indices, n_indices, K):
    d, i, _ = knn(points, K, q_indices, n_indices)
    return d, i
