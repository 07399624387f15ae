"""TEST INFRASTRUCTURE ONLY -- numpy/ctypes front end of oracle/knn_oracle.c, the CPU restatement of
`simple_knn._C.distCUDA2` (exact 3-nearest-neighbour mean squared distance) used to CHECK gaussianhaircut_b200/knn.py.
Only tests/ and tools/ import this; the product never does.

    build()                 gcc -> oracle/lib/libknn_oracle.so
    mean_dist3(points)      (P,3) float32 -> (P,) float32
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "knn_oracle.c")
LIB = os.path.join(HERE, "lib", "libknn_oracle.so")
_lib = None


def build(force: bool = False) -> str:
    if not force and os.path.isfile(LIB) and os.path.getmtime(LIB) >= os.path.getmtime(SRC):
        return LIB
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    # -ffp-contract=off: every float32 operation rounded on its own, like the kernels' intrinsics
    cmd = ["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-shared", "-fPIC", "-o", LIB, SRC, "-lm"]
    subprocess.run(cmd, check=True)
    return LIB


def _load():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(LIB)
        _lib.gho_knn_mean_dist3.restype = C.c_int
        _lib.gho_knn_mean_dist3.argtypes = [C.c_longlong, C.c_void_p, C.c_void_p]
    return _lib


def mean_dist3(points) -> np.ndarray:
    pts = np.ascontiguousarray(np.asarray(points, dtype=np.float32).reshape(-1, 3))
    out = np.empty(pts.shape[0], np.float32)
    if pts.shape[0] and _load().gho_knn_mean_dist3(pts.shape[0], pts.ctypes.data, out.ctypes.data) != 0:
        raise MemoryError("gho_knn_mean_dist3: out of memory")
    return out
