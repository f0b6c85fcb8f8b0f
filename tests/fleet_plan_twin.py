"""ctypes access to a g++ build of tests/cpu_twin/fleet_plan.cpp, the CPU twin of rda_fleet_plan_shapes and of the
selection of rda_convert_fleet_plan_obstacles over each robot's list (its world's shapes, then its map-mates along their
plans) — test infrastructure only."""
import ctypes as C

import numpy as np

import fleet_obstacles_twin as ft
import shim


def fleet_plan_shapes(state, cur_vel, body, dynamics, dt, wheelbase, per_robot=None):
    """state [B,3], cur_vel [B,2,T], body from frontend.robot_body; per_robot None or a dict of host arrays 'dynamics'
    [B], 'wheelbase' [B], 'xy' [B,8,2], 'radius' [B] -> dict kind, nv [B], xy [B,8,2], radius [B], vel [B,2] and
    plan_xy [B,T+1,8,2] (host arrays)."""
    state = np.ascontiguousarray(state, np.float32)
    cur_vel = np.ascontiguousarray(cur_vel, np.float32)
    B, T = state.shape[0], cur_vel.shape[2]
    out = {'kind': np.zeros(B, np.int32), 'nv': np.zeros(B, np.int32), 'xy': np.zeros((B, 8, 2), np.float32),
           'radius': np.zeros(B, np.float32), 'vel': np.zeros((B, 2), np.float32),
           'plan_xy': np.zeros((B, T + 1, 8, 2), np.float32)}
    pr = {}
    if per_robot is not None:
        pr = {'dynamics': np.ascontiguousarray(per_robot['dynamics'], np.int32),
              'wheelbase': np.ascontiguousarray(per_robot['wheelbase'], np.float32),
              'xy': np.ascontiguousarray(per_robot['xy'], np.float32),
              'radius': np.ascontiguousarray(per_robot['radius'], np.float32)}
    bxy = np.ascontiguousarray(body['xy'], np.float32)
    p = lambda a: None if a is None else a.ctypes.data
    i, f, d, vp = C.c_int, C.c_float, C.c_double, C.c_void_p
    fn = shim.lib().shim_fleet_plan_shapes
    fn.restype = None
    fn.argtypes = [i, i, i, d, d, i, i, vp, f] + [vp] * 12
    fn(B, T, shim.DYN[dynamics], dt, wheelbase, int(body['kind']), int(body['nv']), p(bxy), float(body['radius']),
       p(pr.get('dynamics')), p(pr.get('wheelbase')), p(pr.get('xy')), p(pr.get('radius')), p(state), p(cur_vel),
       p(out['kind']), p(out['nv']), p(out['xy']), p(out['radius']), p(out['vel']), p(out['plan_xy']))
    return out


def convert_fleet_plan_obstacles(world, fleet, robot_world, b, N, T, E, dt, order, state):
    """What rda_convert_fleet_plan_obstacles writes for robot b at `state` (always time-varying): its list as
    fleet_obstacles_twin.robot_list builds it, the mates read along fleet['plan_xy'].  Returns obs_A [N,T+1,E,2],
    obs_b [N,T+1,E], obs_kind [N], obs_count."""
    lst = ft.robot_list(world, fleet, robot_world, b)
    count = int(lst['start'][1])
    rw = np.asarray(robot_world)
    W = len(world['start']) - 1
    w = int(rw[b])
    n_world = int(world['start'][w + 1] - world['start'][w]) if 0 <= w < W else 0
    mates = np.nonzero(rw == w)[0] if 0 <= w < W else np.zeros(0, np.int64)
    mates = mates[mates != b]
    planned = np.zeros(max(count, 1), np.int32)
    planned[n_world:count] = 1
    plan = np.zeros((max(count, 1), T + 1, 8, 2), np.float32)
    plan[n_world:count] = np.asarray(fleet['plan_xy'])[mates]
    A = np.zeros((N, T + 1, E, 2), np.float32)
    bb = np.zeros((N, T + 1, E), np.float32)
    kind = np.zeros(N, np.int32)
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    i32 = lambda a: np.ascontiguousarray(a, np.int32)
    st = f32(np.ravel(state)[:3])
    k, nv = i32(lst['kind']), i32(lst['nv'])
    xy, rad, vel = f32(lst['xy']), f32(lst['radius']), f32(lst['vel'])
    p = lambda a: a.ctypes.data
    fn = shim.lib().shim_convert_plan_list
    fn.restype = C.c_int
    fn.argtypes = [C.c_int] * 4 + [C.c_double, C.c_int] + [C.c_void_p] * 11
    cnt = fn(count, N, T, E, dt, int(order), p(st), p(k), p(nv), p(xy), p(rad), p(vel), p(planned), p(plan), p(A), p(bb),
             p(kind))
    return A, bb, kind, cnt
