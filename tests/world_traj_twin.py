"""ctypes access to tests/cpu_twin/world_traj.cpp, the CPU twin of rda_convert_world_obstacles_traj and
rda_convert_world_obstacles_horizon_traj over one robot's list (its world's shapes, then its map-mates), and of the
lower bounds the horizon kernel prunes with — test infrastructure only."""
import ctypes as C

import numpy as np

import horizon_twin as ht
import shim

_I, _D, _V = C.c_int, C.c_double, C.c_void_p


def robot_list(world, fleet, robot_world, b):
    """horizon_twin.robot_list (with 'planned' / 'plan_xy' for mates along their plans) plus 'traj' [count], each
    entry's trajectory index (world['traj'] for world shapes, -1 for map-mates), 'traj_xy' (world['traj_xy']) and
    'id' [count], each entry's obstacle id (the flat shape index, S + m for map-mate m)."""
    lst = ht.robot_list(world, fleet, robot_world, b)
    W = len(world['start']) - 1
    w = int(np.asarray(robot_world)[b]) if robot_world is not None else 0
    lo, hi = (int(world['start'][w]), int(world['start'][w + 1])) if 0 <= w < W else (0, 0)
    mates = np.zeros(0, np.int64)
    if fleet is not None and 0 <= w < W:
        rw = np.asarray(robot_world)
        mates = np.nonzero(rw == w)[0]
        mates = mates[mates != b]
    traj = np.asarray(world['traj'][lo:hi]) if 'traj' in world else np.full(hi - lo, -1)
    lst['traj'] = np.concatenate([traj, np.full(len(mates), -1)]).astype(np.int32)
    lst['traj_xy'] = np.asarray(world['traj_xy']) if 'traj_xy' in world else np.zeros((1, 1, 8, 2), np.float32)
    lst['id'] = np.concatenate([np.arange(lo, hi), int(world['start'][W]) + mates]).astype(np.int32)
    return lst


def _list_args(lst):
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    i32 = lambda a: np.ascontiguousarray(a, np.int32)
    count = len(lst['kind'])
    arrs = [i32(lst['kind']), i32(lst['nv']), f32(lst['xy']).reshape(-1), f32(lst['radius']),
            f32(lst['vel']).reshape(-1), i32(lst.get('planned', np.zeros(count))), f32(lst.get('plan_xy', np.zeros(1))),
            i32(lst['traj'])]
    arrs = [a if a.size else np.zeros(1, a.dtype) for a in arrs]
    txy = f32(lst['traj_xy'])
    keep = arrs + [txy]
    return keep, tuple(a.ctypes.data for a in arrs) + (len(txy), txy.ctypes.data)


def _outs(lst, N, T, E):
    Tc = T + 1
    return (np.zeros((N, Tc, E, 2), np.float32), np.zeros((N, Tc, E), np.float32), np.zeros(N, np.int32),
            np.zeros(N, np.int32))


def _ids(lst, src):
    return np.where(src >= 0, lst['id'][np.maximum(src, 0)] if len(lst['id']) else -1, -1).astype(np.int32)


def select(lst, N, T, E, dt, order, state):
    """What rda_convert_world_obstacles_traj writes for one robot at `state` (reference key when order, list order
    otherwise).  Returns obs_A [N,T+1,E,2], obs_b [N,T+1,E], obs_kind [N], obs_count, obs_id [N]."""
    A, b, kind, src = _outs(lst, N, T, E)
    keep, args = _list_args(lst)
    st = np.ascontiguousarray(np.ravel(state)[:3], np.float32)
    fn = shim.lib().shim_convert_traj_list
    fn.restype = C.c_int
    fn.argtypes = [_I] * 4 + [_D, _I, _V] + [_V] * 8 + [_I, _V] + [_V] * 4
    cnt = fn(len(lst['kind']), N, T, E, dt, int(order), st.ctypes.data, *args, A.ctypes.data, b.ctypes.data,
             kind.ctypes.data, src.ctypes.data)
    return A, b, kind, cnt, _ids(lst, src)


def _body(body):
    bxy = np.ascontiguousarray(body['xy'], np.float32)
    return bxy, (int(body['kind']), int(body['nv']), bxy.ctypes.data, float(body['radius']))


_BODY = [_I, _I, _V, C.c_float]


def horizon_select(lst, N, T, E, dt, nom, ref, body):
    """What rda_convert_world_obstacles_horizon_traj writes for one robot with poses nom, ref [3,T+1] and body
    (robot_body format).  Returns obs_A, obs_b, obs_kind, obs_count, obs_id as select, and keys [count] (float64)."""
    A, b, kind, src = _outs(lst, N, T, E)
    count = len(lst['kind'])
    keys = np.zeros(max(count, 1))
    keep, args = _list_args(lst)
    bxy, bargs = _body(body)
    nom, ref = np.ascontiguousarray(nom, np.float32), np.ascontiguousarray(ref, np.float32)
    fn = shim.lib().shim_horizon_traj_select
    fn.restype = C.c_int
    fn.argtypes = [_I] * 4 + [_D, _V, _V] + _BODY + [_V] * 8 + [_I, _V] + [_V] * 5
    cnt = fn(count, N, T, E, dt, nom.ctypes.data, ref.ctypes.data, *bargs, *args, keys.ctypes.data, A.ctypes.data,
             b.ctypes.data, kind.ctypes.data, src.ctypes.data)
    return A, b, kind, cnt, _ids(lst, src), keys[:count]


def bounds(lst, T, E, dt, nom, ref, body):
    """The horizon kernel's lower bounds of every entry: (one-disc bound [count], bound of every pose [count])."""
    count = len(lst['kind'])
    lb_disc, lb_pose = np.zeros(max(count, 1)), np.zeros(max(count, 1))
    keep, args = _list_args(lst)
    bxy, bargs = _body(body)
    nom, ref = np.ascontiguousarray(nom, np.float32), np.ascontiguousarray(ref, np.float32)
    fn = shim.lib().shim_horizon_traj_bounds
    fn.restype = None
    fn.argtypes = [_I] * 3 + [_D, _V, _V] + _BODY + [_V] * 8 + [_I, _V] + [_V] * 2
    fn(count, T, E, dt, nom.ctypes.data, ref.ctypes.data, *bargs, *args, lb_disc.ctypes.data, lb_pose.ctypes.data)
    return lb_disc[:count], lb_pose[:count]
