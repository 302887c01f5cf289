"""TEST INFRASTRUCTURE ONLY -- the float64 mesh_to_mesh_forward oracle.

oracle/mmi_oracle_scalar.c is the C restatement of op.cu written for a scalar type; this module compiles it as double
(the reference's double instantiation, with its points of rounding to float) and as float (only to check that source
against the pinned float oracle, oracle/mmi_oracle.c), and calls it per body like oracle/measure_oracle.py does.

    build()                                   -> oracle/_build/libmmi_oracle_f64.so, libmmi_oracle_scalar_f32.so
    mesh_to_mesh_forward(query, target, M)    float64 faces / barycentrics
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, 'mmi_oracle_scalar.c')
_LIBS = {}
VARIANTS = {np.dtype(np.float64): ('libmmi_oracle_f64.so', ['-DMMI_DOUBLE']),
            np.dtype(np.float32): ('libmmi_oracle_scalar_f32.so', [])}


def build(force: bool = False):
    out_dir = os.path.join(_HERE, '_build')
    os.makedirs(out_dir, exist_ok=True)
    for name, defs in VARIANTS.values():
        out = os.path.join(out_dir, name)
        if force or not os.path.exists(out) or os.path.getmtime(out) < os.path.getmtime(_SRC):
            subprocess.check_call(['gcc', '-O2', '-ffp-contract=off', '-fno-fast-math', '-shared', '-fPIC'] + defs +
                                  ['-o', out, _SRC, '-lm'])


def lib(dtype=np.float64):
    dtype = np.dtype(dtype)
    if dtype not in _LIBS:
        path = os.path.join(_HERE, '_build', VARIANTS[dtype][0])
        if not os.path.exists(path):
            build()
        L = ctypes.CDLL(path)
        L.mmi_oracle_scalar_forward.restype = ctypes.c_int
        L.mmi_oracle_scalar_forward.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                                ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        _LIBS[dtype] = L
    return _LIBS[dtype]


def mesh_to_mesh_forward(query: np.ndarray, target: np.ndarray, max_collisions: int = 16, dtype=np.float64):
    """query (B,Q,3,3), target (B,F,3,3), converted to `dtype` -> faces (B,Q*M) int64 (-1 empty), bcs (B,Q*M,2,3)."""
    dtype = np.dtype(dtype)
    query = np.ascontiguousarray(query, dtype)
    target = np.ascontiguousarray(target, dtype)
    B, Q = query.shape[:2]
    F = target.shape[1]
    M = max_collisions
    faces = np.full((B, Q * M), -1, np.int64)
    bcs = np.zeros((B, Q * M, 2, 3), dtype)
    L = lib(dtype)
    for b in range(B):
        L.mmi_oracle_scalar_forward(query[b].ctypes.data, target[b].ctypes.data, Q, F, M, faces[b].ctypes.data,
                                    bcs[b].ctypes.data)
    return faces, bcs


if __name__ == '__main__':
    build(force=True)
