"""ctypes access to a g++ build of tests/cpu_twin/world_obstacles.cpp, the CPU twin of the shared-world obstacle
selection (rda_convert_world_obstacles) — test infrastructure only.  Built on first use into tests/_build, or into a
temporary directory when the tree is read-only."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'cpu_twin', 'world_obstacles.cpp')
CSRC = os.path.join(os.path.dirname(HERE), 'rda_planner_b200', 'csrc')
INCLUDE = os.path.join(os.path.dirname(HERE), 'include', 'rda_b200.h')
SO = os.path.join(HERE, '_build', 'libworld_twin.so')

_lib = None


def build():
    deps = [SRC, INCLUDE] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    if os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in deps):
        return SO
    so = SO
    if not os.access(HERE, os.W_OK):
        so = os.path.join(tempfile.mkdtemp(prefix='rda_world_twin_'), os.path.basename(SO))
    os.makedirs(os.path.dirname(so), exist_ok=True)
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-shared', '-fPIC', '-o', so, SRC])
    return so


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        f = _lib.shim_convert_world_obstacles
        f.restype = C.c_int
        f.argtypes = [C.c_int] * 4 + [C.c_double, C.c_int, C.c_int] + [C.c_void_p] * 9
    return _lib


def convert_world_obstacles(world, w, N, T, E, dt, time_varying, order, state):
    """Robot at `state` in world `w` of `world` (dict from pack_worlds; w outside [0, W): empty list).
    Returns obs_A [N,Tc,E,2], obs_b [N,Tc,E], obs_kind [N], obs_count."""
    W = len(world['start']) - 1
    lo, hi = (int(world['start'][w]), int(world['start'][w + 1])) if 0 <= w < W else (0, 0)
    Tc = T + 1 if time_varying else 1
    A = np.zeros((N, Tc, E, 2), np.float32)
    b = np.zeros((N, Tc, E), np.float32)
    kind = np.zeros(N, np.int32)
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    i32 = lambda a: np.ascontiguousarray(a, np.int32)
    st = f32(np.ravel(state)[:3])
    k, nv = i32(world['kind'][lo:hi]), i32(world['nv'][lo:hi])
    xy, rad, vel = f32(world['xy'][lo:hi]), f32(world['radius'][lo:hi]), f32(world['vel'][lo:hi])
    p = lambda a: a.ctypes.data
    cnt = lib().shim_convert_world_obstacles(hi - lo, N, T, E, dt, int(time_varying), int(order), p(st), p(k), p(nv),
                                             p(xy), p(rad), p(vel), p(A), p(b), p(kind))
    return A, b, kind, cnt
