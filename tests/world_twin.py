"""ctypes access to a g++ build of tests/cpu_twin/world_obstacles.cpp, the CPU twin of the shared-world obstacle
selection (rda_convert_world_obstacles) — test infrastructure only."""
import ctypes as C

import numpy as np

import shim


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
    f = shim.lib().shim_convert_world_obstacles
    f.restype = C.c_int
    f.argtypes = [C.c_int] * 4 + [C.c_double, C.c_int, C.c_int] + [C.c_void_p] * 9
    cnt = f(hi - lo, N, T, E, dt, int(time_varying), int(order), p(st), p(k), p(nv), p(xy), p(rad), p(vel), p(A), p(b),
            p(kind))
    return A, b, kind, cnt
