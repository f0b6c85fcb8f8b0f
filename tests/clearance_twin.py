"""ctypes access to a g++ build of tests/cpu_twin/plan_clearance.cpp: the cell core of rda_plan_clearance
(plan_clearance.cuh) on the CPU — test infrastructure only."""
import ctypes as C

import numpy as np

import shim


def cells(G, h, cone, kind, A, b, pose):
    """sd of n cells for the body of canonical rows (G, h) (cone 0 polygon, 1 disc): kind [n], A [n, E, 2], b [n, E],
    pose [n, 3]; returns float64 [n]."""
    G = np.ascontiguousarray(G, np.float32).reshape(-1)
    h = np.ascontiguousarray(h, np.float32).reshape(-1)
    kind = np.ascontiguousarray(kind, np.int32)
    A = np.ascontiguousarray(A, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    pose = np.ascontiguousarray(pose, np.float32)
    n, E = A.shape[0], A.shape[1]
    out = np.zeros(n, np.float64)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    fn = shim.lib().twin_plan_clearance
    fn.restype = C.c_int
    rc = fn(p(G), p(h), C.c_int(h.shape[0]), C.c_int(cone), C.c_int(n), C.c_int(E), p(kind), p(A), p(b), p(pose), p(out))
    if rc != 0:
        raise RuntimeError(f'twin_plan_clearance: {rc}')
    return out
