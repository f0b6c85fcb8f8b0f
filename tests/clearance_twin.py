"""ctypes access to a g++ build of tests/cpu_twin/plan_clearance.cpp: the cell core of rda_plan_clearance
(plan_clearance.cuh) on the CPU — test infrastructure only.  Built on first use into tests/_build, or into a temporary
directory when the tree is read-only."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, 'cpu_twin', 'plan_clearance.cpp')
CSRC = os.path.join(ROOT, 'rda_planner_b200', 'csrc')
SO = os.path.join(HERE, '_build', 'libclearance_twin.so')

_lib = None


def build():
    deps = [SRC, os.path.join(ROOT, 'include', 'rda_b200.h')] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    if os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in deps):
        return SO
    so = SO
    if not os.access(HERE, os.W_OK):
        so = os.path.join(tempfile.mkdtemp(prefix='rda_clearance_twin_'), os.path.basename(SO))
    os.makedirs(os.path.dirname(so), exist_ok=True)
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-o', so, SRC])
    return so


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.twin_plan_clearance.restype = C.c_int
    return _lib


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
    rc = lib().twin_plan_clearance(p(G), p(h), C.c_int(h.shape[0]), C.c_int(cone), C.c_int(n), C.c_int(E), p(kind), p(A),
                                   p(b), p(pose), p(out))
    if rc != 0:
        raise RuntimeError(f'twin_plan_clearance: {rc}')
    return out
