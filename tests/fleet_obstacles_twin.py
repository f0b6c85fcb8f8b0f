"""ctypes access to a g++ build of tests/cpu_twin/fleet_obstacles.cpp, the CPU twin of rda_fleet_shapes, and the
selection of rda_convert_fleet_obstacles restated as the world twin (world_twin) over each robot's list: its world's
shapes, then its map-mates — test infrastructure only."""
import ctypes as C

import numpy as np

import shim
import world_twin

KEYS = ('kind', 'nv', 'xy', 'radius', 'vel')


def fleet_shapes(state, cur_vel, body, dynamics):
    """state [B,3], cur_vel [B,2,T], body from frontend.robot_body -> dict kind, nv [B], xy [B,8,2], radius [B],
    vel [B,2] (host arrays)."""
    state = np.ascontiguousarray(state, np.float32)
    cur_vel = np.ascontiguousarray(cur_vel, np.float32)
    B, T = state.shape[0], cur_vel.shape[2]
    out = {'kind': np.zeros(B, np.int32), 'nv': np.zeros(B, np.int32), 'xy': np.zeros((B, 8, 2), np.float32),
           'radius': np.zeros(B, np.float32), 'vel': np.zeros((B, 2), np.float32)}
    bxy = np.ascontiguousarray(body['xy'], np.float32)
    p = lambda a: a.ctypes.data
    i, f, vp = C.c_int, C.c_float, C.c_void_p
    fn = shim.lib().shim_fleet_shapes
    fn.restype = None
    fn.argtypes = [i, i, i, i, i, vp, f, vp, vp, vp, vp, vp, vp, vp]
    fn(B, T, shim.DYN[dynamics], int(body['kind']), int(body['nv']), p(bxy), float(body['radius']), p(state), p(cur_vel),
       p(out['kind']), p(out['nv']), p(out['xy']), p(out['radius']), p(out['vel']))
    return out


def robot_list(world, fleet, robot_world, b):
    """Robot b's raw shapes in the layout of pack_worlds (one world): every shape of its world in world order, then
    every other robot of its world in ascending index.  A robot outside [0, W) has an empty list."""
    W = len(world['start']) - 1
    rw = np.asarray(robot_world)
    w = int(rw[b])
    if not 0 <= w < W:
        lo = hi = 0
        mates = np.zeros(0, np.int64)
    else:
        lo, hi = int(world['start'][w]), int(world['start'][w + 1])
        mates = np.nonzero(rw == w)[0]
        mates = mates[mates != b]
    out = {k: np.concatenate([np.asarray(world[k][lo:hi]), np.asarray(fleet[k])[mates]]) for k in KEYS}
    out['start'] = np.array([0, hi - lo + len(mates)], np.int32)
    return out


def convert_fleet_obstacles(world, fleet, robot_world, b, N, T, E, dt, time_varying, order, state):
    """What rda_convert_fleet_obstacles writes for robot b at `state`: the world twin over robot_list."""
    return world_twin.convert_world_obstacles(robot_list(world, fleet, robot_world, b), 0, N, T, E, dt, time_varying,
                                              order, state)
