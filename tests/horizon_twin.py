"""ctypes access to tests/cpu_twin/horizon_select.cpp, the brute-force CPU twin of rda_convert_world_obstacles_horizon
over one robot's list (its world's shapes, then its map-mates), and of the lower bounds its kernel prunes with — test
infrastructure only."""
import ctypes as C

import numpy as np

import fleet_obstacles_twin as ft
import shim

KEYS = ('kind', 'nv', 'xy', 'radius', 'vel')


def robot_list(world, fleet, robot_world, b):
    """Robot b's list in the layout of pack_worlds (one world), plus 'planned' [count] (1: a map-mate read along
    'plan_xy' [count,T+1,8,2] when fleet has plan_xy).  fleet None: the world's shapes only."""
    W = len(world['start']) - 1
    w = int(np.asarray(robot_world)[b]) if robot_world is not None else 0
    if fleet is None:
        lo, hi = (int(world['start'][w]), int(world['start'][w + 1])) if 0 <= w < W else (0, 0)
        lst = {k: np.asarray(world[k][lo:hi]) for k in KEYS}
        lst['planned'] = np.zeros(hi - lo, np.int32)
        return lst
    lst = ft.robot_list(world, fleet, robot_world, b)
    count = int(lst['start'][1])
    n_world = int(world['start'][w + 1] - world['start'][w]) if 0 <= w < W else 0
    lst['planned'] = np.zeros(count, np.int32)
    if 'plan_xy' in fleet:
        rw = np.asarray(robot_world)
        mates = np.nonzero(rw == w)[0] if 0 <= w < W else np.zeros(0, np.int64)
        mates = mates[mates != b]
        T1 = np.asarray(fleet['plan_xy']).shape[1]
        lst['planned'][n_world:] = 1
        plan = np.zeros((count, T1, 8, 2), np.float32)
        plan[n_world:] = np.asarray(fleet['plan_xy'])[mates]
        lst['plan_xy'] = plan
    return lst


def _args(lst, nom, ref, body):
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    i32 = lambda a: np.ascontiguousarray(a, np.int32)
    count = len(lst['kind'])
    arrs = [f32(nom), f32(ref), f32(body['xy']), i32(lst['kind']), i32(lst['nv']), f32(lst['xy']).reshape(-1),
            f32(lst['radius']), f32(lst['vel']).reshape(-1), i32(lst.get('planned', np.zeros(count))),
            f32(lst.get('plan_xy', np.zeros(1)))]
    arrs = [a if a.size else np.zeros(1, a.dtype) for a in arrs]
    p = [a.ctypes.data for a in arrs]
    return arrs, (p[0], p[1], int(body['kind']), int(body['nv']), p[2], float(body['radius'])) + tuple(p[3:])


_BODY = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_float] + [C.c_void_p] * 7


def select(lst, N, T, E, dt, time_varying, nom, ref, body):
    """What the kernel writes for one robot with list `lst` (robot_list), poses nom, ref [3,T+1] and body (robot_body
    format).  Returns obs_A [N,Tc,E,2], obs_b [N,Tc,E], obs_kind [N], obs_count, keys [count] (float64)."""
    count = len(lst['kind'])
    Tc = T + 1 if time_varying else 1
    A = np.zeros((N, Tc, E, 2), np.float32)
    bb = np.zeros((N, Tc, E), np.float32)
    kind = np.zeros(N, np.int32)
    keys = np.zeros(max(count, 1))
    keep, args = _args(lst, nom, ref, body)
    fn = shim.lib().shim_horizon_select
    fn.restype = C.c_int
    fn.argtypes = [C.c_int] * 4 + [C.c_double, C.c_int] + _BODY + [C.c_void_p] * 4
    cnt = fn(count, N, T, E, dt, int(time_varying), *args, keys.ctypes.data, A.ctypes.data, bb.ctypes.data,
             kind.ctypes.data)
    return A, bb, kind, cnt, keys[:count]


def bounds(lst, T, E, dt, time_varying, nom, ref, body):
    """The kernel's lower bounds of every entry: (one-disc bound of the horizon [count], bound of every pose [count])."""
    count = len(lst['kind'])
    lb_disc, lb_pose = np.zeros(max(count, 1)), np.zeros(max(count, 1))
    keep, args = _args(lst, nom, ref, body)
    fn = shim.lib().shim_horizon_bounds
    fn.restype = None
    fn.argtypes = [C.c_int] * 3 + [C.c_double, C.c_int] + _BODY + [C.c_void_p] * 2
    fn(count, T, E, dt, int(time_varying), *args, lb_disc.ctypes.data, lb_pose.ctypes.data)
    return lb_disc[:count], lb_pose[:count]


def exact_count(lst, N, T, E, dt, time_varying, nom, ref, body, tile=256):
    """How many entries of the list the kernel's scan evaluates with the exact key."""
    keep, args = _args(lst, nom, ref, body)
    fn = shim.lib().shim_horizon_exact_count
    fn.restype = C.c_int
    fn.argtypes = [C.c_int] * 4 + [C.c_double, C.c_int, C.c_int] + _BODY
    return fn(len(lst['kind']), N, T, E, dt, int(time_varying), tile, *args)
