"""ctypes access to a g++ build of tests/cpu_twin/fleet_paths.cpp, the CPU twin of the per-robot path kernels
(rda_pre_process_paths / rda_post_process_paths) — test infrastructure only."""
import ctypes as C

import numpy as np

import shim


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def _i32(a):
    return np.ascontiguousarray(a, np.int32)


def pre_process_paths(packed, dynamics, T, dt, L, state, cur_vel, ref_speed, robot_path, curve_index, start_index,
                      threshold=0.1, ind_range=10):
    """packed: dict from pack_paths; per-robot arrays state [B,3], cur_vel [B,2,T], ref_speed [B], robot_path,
    curve_index, start_index [B].  Returns nom_s [B,3,T+1], ref_s [B,3,T+1], near_index [B], solver_speed [B]."""
    state, cur_vel, ref_speed = _f32(state), _f32(cur_vel), _f32(ref_speed)
    B = state.shape[0]
    rp, ci, si = _i32(robot_path), _i32(curve_index), _i32(start_index)
    path, pc, cs, cg = _f32(packed['path']), _i32(packed['path_curve']), _i32(packed['curve_start']), \
        _i32(packed['curve_gear'])
    nom = np.zeros((B, 3, T + 1), np.float32)
    ref = np.zeros((B, 3, T + 1), np.float32)
    near = np.zeros(B, np.int32)
    speed = np.zeros(B, np.float32)
    p = lambda a: a.ctypes.data
    i, f, vp = C.c_int, C.c_float, C.c_void_p
    fn = shim.lib().shim_pre_process_paths
    fn.restype = None
    fn.argtypes = [i, i, i, f, f, vp, vp, vp, vp, i, vp, vp, vp, vp, vp, vp, f, i, vp, vp, vp, vp]
    fn(B, T, shim.DYN[dynamics], dt, L, p(state), p(cur_vel), p(ref_speed), p(path), len(pc) - 1, p(pc), p(cs), p(cg),
       p(rp), p(ci), p(si), threshold, ind_range, p(nom), p(ref), p(near), p(speed))
    return nom, ref, near, speed


def post_process_paths(packed, T, robot_path, goal_index_threshold, near_index, curve_index, u_opt):
    """Returns near_index, curve_index, u_opt, cur_vel, arrive after the end-of-curve and arrive rules (copies)."""
    near, ci, u = _i32(near_index).copy(), _i32(curve_index).copy(), _f32(u_opt).copy()
    rp, pc, cs = _i32(robot_path), _i32(packed['path_curve']), _i32(packed['curve_start'])
    B = len(near)
    cur_vel = np.zeros_like(u)
    arrive = np.zeros(B, np.int32)
    p = lambda a: a.ctypes.data
    i, vp = C.c_int, C.c_void_p
    fn = shim.lib().shim_post_process_paths
    fn.restype = None
    fn.argtypes = [i, i, i, vp, vp, vp, i, vp, vp, vp, vp, vp]
    fn(B, T, len(pc) - 1, p(pc), p(cs), p(rp), goal_index_threshold, p(near), p(ci), p(u), p(cur_vel), p(arrive))
    return near, ci, u, cur_vel, arrive
