"""Batched front end: the steps either side of the solve, on the device (SURVEY.md §8 f1-f3).

  pre_process_batch        MPC.pre_process                         (mpc.py:251-291, 338-438)
  convert_obstacles_batch  MPC.convert_rda_obstacle + RDA_solver.assign_obstacle_parameter
                           (mpc.py:189-218, 440-549; rda_solver.py:483-526)
  convert_world_obstacles_batch
                           the same over obstacle worlds of any size shared by many robots: each
                           robot's N nearest shapes of its world
  fleet_shapes_batch, convert_fleet_obstacles_batch
                           the same with the other robots of each world as moving obstacles
  fleet_plan_shapes_batch  the robots along their last plans, for convert_fleet_obstacles_batch(plan=True)
  convert_world_obstacles_horizon_batch
                           the world and fleet conversions in the horizon order: each robot's shapes sorted by the
                           smallest signed distance of its body over its nominal and reference poses
  pack_paths               a set of reference paths cut into single-gear curves (split_path, mpc.py:232-249),
                           in the layout the device reads
  BatchedMPC               MPC.control for B robots, on one reference path or each on its own path of a
                           shared set (mpc.py:127-187), closed loop without a host round trip

Thin wrappers over the C ABI (include/rda_b200.h, "front end"); no CPU fallback."""
import ctypes as C

import numpy as np
import torch

from . import _cabi
from .rda_solver import RDA_solver, canonical_polygon_rows


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _stream(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def path_tensor(ref_path, device):
    """list of (3|4, 1) waypoints (the reference's ref_path) or an array [P, >=3] -> float32 [P, 3]."""
    if isinstance(ref_path, torch.Tensor):
        return ref_path.to(device=device, dtype=torch.float32)[:, :3].contiguous()
    if isinstance(ref_path, (list, tuple)):
        arr = np.stack([np.asarray(p, float).reshape(-1)[:3] for p in ref_path])
    else:
        arr = np.asarray(ref_path, float)[:, :3]
    return torch.as_tensor(arr, dtype=torch.float32, device=device).contiguous()


def _path_rows(ref_path):
    """A reference path in any form path_tensor accepts -> float64 array [P, k], one waypoint per row with all its
    rows (x, y, heading and, when present, the gear flag)."""
    if isinstance(ref_path, torch.Tensor):
        return ref_path.detach().to('cpu', torch.float64).numpy().reshape(len(ref_path), -1)
    if isinstance(ref_path, (list, tuple)):
        if not ref_path:
            return np.zeros((0, 3))
        return np.stack([np.asarray(p, float).reshape(-1) for p in ref_path])
    return np.asarray(ref_path, float).reshape(len(ref_path), -1)


def pack_paths(paths, enable_reverse=False):
    """W reference paths, each in any form path_tensor accepts, -> dict of host arrays in the layout of
    rda_pre_process_paths: path [P,3] float32 (all waypoints, one flat list), curve_start [C+1], path_curve [W+1] and
    curve_gear [C] int32.  Each path is cut into single-gear curves as split_path does it (mpc.py:232-249): with
    enable_reverse a new curve starts wherever the gear flag, the last row of a waypoint, changes; without it every
    path is one curve of gear +1."""
    rows = [_path_rows(p) for p in paths]
    if not rows:
        raise ValueError('at least one path')
    curve_start, path_curve, gears = [0], [0], []
    for w, r in enumerate(rows):
        if len(r) == 0 or r.shape[1] < 3:
            raise ValueError(f'path {w} is empty or has fewer than 3 rows per waypoint')
        if enable_reverse:
            if r.shape[1] < 4:
                raise ValueError(f'path {w} has no gear row (enable_reverse reads the last of 4 rows)')
            flags = r[:, -1]
            cuts = [i for i in range(1, len(r)) if flags[i] != flags[i - 1]]
        else:
            flags, cuts = np.ones(len(r)), []
        base = curve_start[-1]
        for c in cuts + [len(r)]:
            curve_start.append(base + c)
        gears += [int(flags[c]) for c in [0] + cuts]
        path_curve.append(len(gears))
    if curve_start[-1] > np.iinfo(np.int32).max:
        raise ValueError('more than 2**31 - 1 waypoints')
    return {'path': np.concatenate([r[:, :3] for r in rows]).astype(np.float32),
            'curve_start': np.asarray(curve_start, np.int32), 'path_curve': np.asarray(path_curve, np.int32),
            'curve_gear': np.asarray(gears, np.int32)}


def _shape_arrays(*lead):
    return {'kind': np.zeros(lead, np.int32), 'nv': np.zeros(lead, np.int32),
            'xy': np.zeros(lead + (_cabi.MAX_EDGE, 2), np.float32), 'radius': np.zeros(lead, np.float32),
            'vel': np.zeros(lead + (2,), np.float32)}


def _pack_shape(out, at, o, max_edge_num):
    """One simulator obstacle into entry `at` of the shape arrays `out`."""
    vel = getattr(o, 'velocity', None)
    if vel is not None:
        out['vel'][at] = np.asarray(vel, float).reshape(-1)[:2]
    if o.cone_type == 'norm2':
        out['kind'][at] = _cabi.OBS_CIRCLE
        out['xy'][at + (0,)] = np.asarray(o.center, float).reshape(-1)[:2]
        out['radius'][at] = o.radius
    else:
        v = np.asarray(o.vertex, float)
        n = v.shape[1]
        if n > min(max_edge_num, _cabi.MAX_EDGE) or n < 3:
            raise ValueError(f'polygon with {n} vertices: 3..{min(max_edge_num, _cabi.MAX_EDGE)} supported')
        out['kind'][at] = _cabi.OBS_POLYGON
        out['nv'][at] = n
        out['xy'][at + (slice(0, n),)] = v[0:2].T


def _pack_trajectory(o, max_edge_num):
    """The trajectory of one simulator obstacle -> float32 [T+1, 8, 2], its shape at every stage in the world frame: a
    polygon's vertices (T+1 arrays 2 x nv, nv that of its vertex), a disc's centre in row 0 (centres 2 x (T+1))."""
    xy = None
    if o.cone_type == 'norm2':
        c = np.asarray(o.trajectory, float)
        if c.ndim != 2 or c.shape[0] != 2 or c.shape[1] < 1:
            raise ValueError(f'a disc trajectory is 2 x (T+1) centres, got shape {c.shape}')
        xy = np.zeros((c.shape[1], _cabi.MAX_EDGE, 2))
        xy[:, 0] = c.T
    else:
        nv = np.asarray(o.vertex).shape[1]
        stages = [np.asarray(v, float) for v in o.trajectory]
        if not stages:
            raise ValueError('a polygon trajectory has at least one stage')
        for t, v in enumerate(stages):
            if v.ndim != 2 or v.shape[0] < 2 or v.shape[1] != nv:
                raise ValueError(f'stage {t} of a polygon trajectory has shape {v.shape}: 2 x {nv} vertices, as its '
                                 'vertex, at every stage')
        if nv > min(max_edge_num, _cabi.MAX_EDGE):
            raise ValueError(f'polygon trajectory with {nv} vertices: 3..{min(max_edge_num, _cabi.MAX_EDGE)} supported')
        xy = np.zeros((len(stages), _cabi.MAX_EDGE, 2))
        for t, v in enumerate(stages):
            xy[t, :nv] = v[0:2].T
    if not np.all(np.isfinite(xy)):
        raise ValueError('a trajectory has non-finite values')
    return xy.astype(np.float32)


def pack_shapes(obstacle_lists, max_shapes=None, max_edge_num=_cabi.MAX_EDGE):
    """Per-instance lists of simulator obstacles (attributes cone_type, center, radius, vertex,
    velocity — what MPC.convert_rda_obstacle reads, mpc.py:189-208) -> dict of host arrays in
    the layout of rda_convert_obstacles.  Polygons with more than `max_edge_num` vertices are
    refused here (the kernel would write an all-zero obstacle for them)."""
    B = len(obstacle_lists)
    M = max_shapes or max(1, max(len(l) for l in obstacle_lists))
    if M > _cabi.MAX_SHAPES:
        raise ValueError(f'at most {_cabi.MAX_SHAPES} raw obstacles per instance')
    out = _shape_arrays(B, M)
    out['count'] = np.zeros(B, np.int32)
    for b, lst in enumerate(obstacle_lists):
        if len(lst) > M:
            raise ValueError('more obstacles than max_shapes')
        out['count'][b] = len(lst)
        for j, o in enumerate(lst):
            if getattr(o, 'trajectory', None) is not None:
                raise ValueError('obstacles with a trajectory are packed by pack_worlds (one world per robot, '
                                 'robot_world = arange(B), gives per-robot lists)')
            _pack_shape(out, (b, j), o, max_edge_num)
    return out


def pack_worlds(worlds, max_edge_num=_cabi.MAX_EDGE):
    """W lists of simulator obstacles (as pack_shapes takes them), each shared by any number of robots, of any
    size -> dict of host arrays in the layout of rda_convert_world_obstacles: kind, nv, xy, radius, vel over the
    flat list of all worlds' shapes, and start [W+1] (world w is shapes start[w]:start[w+1]).  The shape arrays
    have at least one entry, so that a set of empty worlds still has device buffers to point at.

    An obstacle may carry a `trajectory`, its predicted shape at every stage t = 0..T in the world frame: for a polygon
    T+1 vertex arrays 2 x nv (nv that of its vertex), for a disc the centres 2 x (T+1).  When one does, the dict also
    holds traj [S] int32 (each shape's trajectory, -1 for none) and traj_xy [K, T+1, 8, 2] float32 (trajectory k's
    stage-t vertices, or a disc's centre in row 0), the table of rda_convert_world_obstacles_traj; xy then holds stage 0
    and vel zero for the shapes with a trajectory.  Both may be overwritten on the device between control steps (a
    predictor's output) without packing again: keep the shape, the dtype and the storage.  Without trajectories the
    dict is exactly what it was."""
    sizes = [len(l) for l in worlds]
    if not sizes:
        raise ValueError('at least one world')
    start = np.zeros(len(worlds) + 1, np.int64)
    start[1:] = np.cumsum(sizes)
    if start[-1] > np.iinfo(np.int32).max:
        raise ValueError('more than 2**31 - 1 shapes')
    out = _shape_arrays(max(1, int(start[-1])))
    trajs = []
    for w, lst in enumerate(worlds):
        for j, o in enumerate(lst):
            _pack_shape(out, (int(start[w]) + j,), o, max_edge_num)
            if getattr(o, 'trajectory', None) is not None:
                trajs.append((int(start[w]) + j, _pack_trajectory(o, max_edge_num)))
    out['start'] = start.astype(np.int32)
    if trajs:
        stages = {len(xy) for _, xy in trajs}
        if len(stages) != 1:
            raise ValueError(f'trajectories of different stage counts {sorted(stages)}: every one has T+1 stages')
        out['traj'] = np.full(len(out['kind']), -1, np.int32)
        out['traj_xy'] = np.stack([xy for _, xy in trajs])
        for k, (at, xy) in enumerate(trajs):
            out['traj'][at] = k
            out['xy'][at] = xy[0]
            out['vel'][at] = 0
    return out


def _check_traj(world, T, time_varying, device=None):
    """Refuse, with a ValueError, a world with trajectories (pack_worlds) that a call with horizon T and time_varying
    cannot take: time-invariant output, traj_xy not [K, T+1, 8, 2], and with `device` (the conversions) traj_xy /
    traj that are not contiguous float32 / int32 [S] tensors on that device."""
    if not time_varying:
        raise ValueError('a world with trajectories needs time_varying=True: a trajectory is T+1 copies')
    txy, traj = world['traj_xy'], world['traj']
    if len(txy.shape) != 4 or txy.shape[1] != T + 1:
        raise ValueError(f"world['traj_xy'] has shape {tuple(txy.shape)}: [K, T+1, 8, 2] with T+1 = {T + 1} stages")
    if tuple(txy.shape[2:]) != (_cabi.MAX_EDGE, 2) or txy.shape[0] < 1:
        raise ValueError(f"world['traj_xy'] has shape {tuple(txy.shape)}: [K, T+1, {_cabi.MAX_EDGE}, 2], K >= 1")
    if tuple(traj.shape) != tuple(world['kind'].shape):
        raise ValueError(f"world['traj'] has shape {tuple(traj.shape)}: one entry per packed shape, "
                         f"{tuple(world['kind'].shape)}")
    if device is None:
        return
    for name, t, dtype in (('traj_xy', txy, torch.float32), ('traj', traj, torch.int32)):
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or t.device != device or not t.is_contiguous():
            raise ValueError(f"world['{name}'] must be a contiguous {dtype} tensor on {device}")


def _traj_args(world, T, time_varying, device):
    """(shape_traj, K, traj_xy) of a world with trajectories, checked against the call (_check_traj)."""
    _check_traj(world, T, time_varying, device)
    return _ptr(world['traj']), world['traj_xy'].shape[0], _ptr(world['traj_xy'])


def pre_process_batch(state, cur_vel, ref_speed, path, start_index, dynamics, dt, wheelbase, T,
                      threshold=0.1, ind_range=10):
    """CUDA tensors: state [B,3], cur_vel [B,2,T], ref_speed [B], path [P,3], start_index [B] int32.
    Returns nom_s [B,3,T+1], ref_s [B,3,T+1], near_index [B] int32."""
    lib = _cabi.load()
    dev = state.device
    B = state.shape[0]
    nom = torch.empty((B, 3, T + 1), dtype=torch.float32, device=dev)
    ref = torch.empty((B, 3, T + 1), dtype=torch.float32, device=dev)
    near = torch.empty(B, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _cabi.check(lib.rda_pre_process(B, T, _cabi.DYNAMICS[dynamics], dt, wheelbase, _ptr(state), _ptr(cur_vel),
                                        _ptr(ref_speed), _ptr(path), path.shape[0], _ptr(start_index), threshold,
                                        ind_range, _ptr(nom), _ptr(ref), _ptr(near), _stream(dev)), 'rda_pre_process')
    return nom, ref, near


def convert_obstacles_batch(shapes, state, N, T, E, dt, time_varying=False, order=True, ids=False):
    """shapes: dict of CUDA tensors (kind, nv [B,M] int32; xy [B,M,8,2]; radius [B,M]; vel [B,M,2];
    count [B] int32).  Returns obs_A [B,N,Tc,E,2], obs_b [B,N,Tc,E], obs_kind [B,N], obs_count [B], and with ids also
    obs_id [B,N] int32: the position of each slot's shape in the robot's list (-1 for an empty list), for
    RDA_solver.set_obstacle_ids."""
    lib = _cabi.load()
    dev = shapes['kind'].device
    B, M = shapes['kind'].shape
    Tc = T + 1 if time_varying else 1
    A = torch.empty((B, N, Tc, E, 2), dtype=torch.float32, device=dev)
    b = torch.empty((B, N, Tc, E), dtype=torch.float32, device=dev)
    kind = torch.empty((B, N), dtype=torch.int32, device=dev)
    count = torch.empty(B, dtype=torch.int32, device=dev)
    args = (B, M, N, T, E, dt, int(time_varying), int(order), _ptr(state), _ptr(shapes['kind']), _ptr(shapes['nv']),
            _ptr(shapes['xy']), _ptr(shapes['radius']), _ptr(shapes['vel']), _ptr(shapes['count']), _ptr(A), _ptr(b),
            _ptr(kind), _ptr(count))
    with torch.cuda.device(dev):
        if ids:
            obs_id = torch.empty((B, N), dtype=torch.int32, device=dev)
            _cabi.check(lib.rda_convert_obstacles_ids(*args, _ptr(obs_id), _stream(dev)), 'rda_convert_obstacles_ids')
            return A, b, kind, count, obs_id
        _cabi.check(lib.rda_convert_obstacles(*args, _stream(dev)), 'rda_convert_obstacles')
    return A, b, kind, count


def convert_world_obstacles_batch(world, state, robot_world, N, T, E, dt, time_varying=False, order=True, ids=False):
    """world: dict of CUDA tensors from pack_worlds (kind, nv [S] int32; xy [S,8,2]; radius [S]; vel [S,2];
    start [W+1] int32); robot_world [B] int32 or None (every robot in world 0).  Each robot gets the N nearest
    shapes of its world (order) or its first N, as convert_obstacles_batch would given the whole world as its
    list.  Returns obs_A [B,N,Tc,E,2], obs_b [B,N,Tc,E], obs_kind [B,N], obs_count [B] (the world sizes), and with ids
    also obs_id [B,N] int32: the flat index of each slot's shape in the packed worlds (-1 for an empty world), for
    RDA_solver.set_obstacle_ids.  A world with trajectories (traj, traj_xy) needs time_varying: its shapes are keyed
    by their stage 0 and written along their trajectories (rda_convert_world_obstacles_traj)."""
    lib = _cabi.load()
    dev = state.device
    B, W = state.shape[0], world['start'].shape[0] - 1
    Tc = T + 1 if time_varying else 1
    A = torch.empty((B, N, Tc, E, 2), dtype=torch.float32, device=dev)
    b = torch.empty((B, N, Tc, E), dtype=torch.float32, device=dev)
    kind = torch.empty((B, N), dtype=torch.int32, device=dev)
    count = torch.empty(B, dtype=torch.int32, device=dev)
    if 'traj' in world:
        traj = _traj_args(world, T, time_varying, dev)
        obs_id = torch.empty((B, N), dtype=torch.int32, device=dev) if ids else None
        with torch.cuda.device(dev):
            _cabi.check(lib.rda_convert_world_obstacles_traj(
                B, W, N, T, E, dt, int(time_varying), int(order), _ptr(state), _ptr(world['start']), _ptr(robot_world),
                _ptr(world['kind']), _ptr(world['nv']), _ptr(world['xy']), _ptr(world['radius']), _ptr(world['vel']),
                *(None,) * 8, _ptr(A), _ptr(b), _ptr(kind), _ptr(count), _ptr(obs_id), *traj, _stream(dev)),
                'rda_convert_world_obstacles_traj')
        return (A, b, kind, count, obs_id) if ids else (A, b, kind, count)
    if ids:
        obs_id = torch.empty((B, N), dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _cabi.check(lib.rda_convert_world_obstacles_ids(
                B, W, N, T, E, dt, int(time_varying), int(order), _ptr(state), _ptr(world['start']), _ptr(robot_world),
                _ptr(world['kind']), _ptr(world['nv']), _ptr(world['xy']), _ptr(world['radius']), _ptr(world['vel']),
                *(None,) * 8, _ptr(A), _ptr(b), _ptr(kind), _ptr(count), _ptr(obs_id), _stream(dev)),
                'rda_convert_world_obstacles_ids')
        return A, b, kind, count, obs_id
    with torch.cuda.device(dev):
        _cabi.check(lib.rda_convert_world_obstacles(B, W, N, T, E, dt, int(time_varying), int(order), _ptr(state),
                                                    _ptr(world['start']), _ptr(robot_world), _ptr(world['kind']),
                                                    _ptr(world['nv']), _ptr(world['xy']), _ptr(world['radius']),
                                                    _ptr(world['vel']), _ptr(A), _ptr(b), _ptr(kind), _ptr(count),
                                                    _stream(dev)),
                    'rda_convert_world_obstacles')
    return A, b, kind, count


def robot_body(car_tuple):
    """The robot body of car_tuple in its own frame, as one raw shape for the other robots of a fleet: dict kind
    (OBS_POLYGON / OBS_CIRCLE), nv, xy [8,2] float32, radius.  A polygon body is given by the vertices of its canonical
    rows (canonical_polygon_rows, the rows the solver holds), counter-clockwise, vertex i joining rows i-1 and i,
    computed in float64 and rounded to float32; a disc body by its centre (h0, h1) in xy[0] and its radius -h2."""
    G = np.asarray(car_tuple.G, float)
    h = np.asarray(car_tuple.h, float).reshape(-1)
    xy = np.zeros((_cabi.MAX_EDGE, 2), np.float32)
    if car_tuple.cone_type == 'norm2':
        xy[0] = h[:2]
        return {'kind': _cabi.OBS_CIRCLE, 'nv': 0, 'xy': xy, 'radius': float(np.float32(-h[2]))}
    G, h = canonical_polygon_rows(G, h)
    Gp, hp = np.roll(G, 1, axis=0), np.roll(h, 1)
    det = Gp[:, 0] * G[:, 1] - Gp[:, 1] * G[:, 0]
    V = np.stack([(hp * G[:, 1] - h * Gp[:, 1]) / det, (Gp[:, 0] * h - G[:, 0] * hp) / det], axis=1)
    xy[:len(V)] = V
    return {'kind': _cabi.OBS_POLYGON, 'nv': len(V), 'xy': xy, 'radius': 0.0}


def fleet_shapes_batch(state, cur_vel, body, dynamics, per_robot=None):
    """CUDA tensors state [B,3], cur_vel [B,2,T] (the controls each robot last applied in cur_vel[:, :, 0]); body from
    robot_body with xy a CUDA tensor.  Returns every robot as one raw shape for its map-mates, dict of CUDA tensors in
    the layout of pack_worlds without 'start': its body at its pose, moving with the world-frame velocity of its
    control.  per_robot: None, or a dict of CUDA tensors 'dynamics' int32 [B], 'xy' float32 [B,8,2] and 'radius' float32
    [B], each robot's own dynamics and body (robot classes; body gives the kind and vertex count of every robot)."""
    lib = _cabi.load()
    dev = state.device
    B, T = state.shape[0], cur_vel.shape[2]
    out = {'kind': torch.empty(B, dtype=torch.int32, device=dev), 'nv': torch.empty(B, dtype=torch.int32, device=dev),
           'xy': torch.empty((B, _cabi.MAX_EDGE, 2), dtype=torch.float32, device=dev),
           'radius': torch.empty(B, dtype=torch.float32, device=dev),
           'vel': torch.empty((B, 2), dtype=torch.float32, device=dev)}
    if per_robot is not None:
        with torch.cuda.device(dev):
            _cabi.check(lib.rda_fleet_shapes_per_robot(B, T, _ptr(per_robot['dynamics']), body['kind'], body['nv'],
                                                       _ptr(per_robot['xy']), _ptr(per_robot['radius']), _ptr(state),
                                                       _ptr(cur_vel), _ptr(out['kind']), _ptr(out['nv']), _ptr(out['xy']),
                                                       _ptr(out['radius']), _ptr(out['vel']), _stream(dev)),
                        'rda_fleet_shapes_per_robot')
        return out
    with torch.cuda.device(dev):
        _cabi.check(lib.rda_fleet_shapes(B, T, _cabi.DYNAMICS[dynamics], body['kind'], body['nv'], _ptr(body['xy']),
                                         body['radius'], _ptr(state), _ptr(cur_vel), _ptr(out['kind']), _ptr(out['nv']),
                                         _ptr(out['xy']), _ptr(out['radius']), _ptr(out['vel']), _stream(dev)),
                    'rda_fleet_shapes')
    return out


def fleet_plan_shapes_batch(state, cur_vel, body, dynamics, dt, wheelbase, per_robot=None):
    """fleet_shapes_batch (the same entries, bit for bit) plus 'plan_xy' [B,T+1,8,2]: each robot's body along its plan,
    at q(0) = state and q(t+1) = the model step from q(t) with cur_vel[:, :, min(t + 1, T - 1)] (column 0 is the control
    it has just applied).  per_robot: None, or a dict as for fleet_shapes_batch with also 'wheelbase' float32 [B]."""
    lib = _cabi.load()
    dev = state.device
    B, T = state.shape[0], cur_vel.shape[2]
    out = {'kind': torch.empty(B, dtype=torch.int32, device=dev), 'nv': torch.empty(B, dtype=torch.int32, device=dev),
           'xy': torch.empty((B, _cabi.MAX_EDGE, 2), dtype=torch.float32, device=dev),
           'radius': torch.empty(B, dtype=torch.float32, device=dev),
           'vel': torch.empty((B, 2), dtype=torch.float32, device=dev),
           'plan_xy': torch.empty((B, T + 1, _cabi.MAX_EDGE, 2), dtype=torch.float32, device=dev)}
    pr = per_robot or {}
    with torch.cuda.device(dev):
        _cabi.check(lib.rda_fleet_plan_shapes(B, T, _cabi.DYNAMICS[dynamics], dt, wheelbase, body['kind'], body['nv'],
                                              _ptr(body['xy']), body['radius'], _ptr(pr.get('dynamics')),
                                              _ptr(pr.get('wheelbase')), _ptr(pr.get('xy')), _ptr(pr.get('radius')),
                                              _ptr(state), _ptr(cur_vel), _ptr(out['kind']), _ptr(out['nv']),
                                              _ptr(out['xy']), _ptr(out['radius']), _ptr(out['vel']),
                                              _ptr(out['plan_xy']), _stream(dev)),
                    'rda_fleet_plan_shapes')
    return out


def fleet_csr(robot_world, W):
    """robot_world [B] int32 CUDA tensor -> (start [W+1], robots [B]) int32: the robots of world w are
    robots[start[w]:start[w+1]], in ascending order; robots outside [0, W) are in no world.  On the device, without a
    host synchronisation."""
    ordered, robots = torch.sort(robot_world, stable=True)
    bounds = torch.arange(W + 1, dtype=ordered.dtype, device=ordered.device)
    start = torch.searchsorted(ordered, bounds, out_int32=True)
    return start, robots.to(torch.int32)


def convert_fleet_obstacles_batch(world, state, robot_world, fleet, N, T, E, dt, time_varying=False, order=True,
                                  plan=False, ids=False):
    """convert_world_obstacles_batch with the robots as obstacles of each other: robot b chooses from every shape of
    its world followed by every other robot of its world in ascending index, fleet [m] being robot m's shape (from
    fleet_shapes_batch).  robot_world [B] int32 or None (every robot in world 0).  Returns obs_A [B,N,Tc,E,2], obs_b [B,N,Tc,E], obs_kind [B,N], obs_count [B] (world
    size plus the robots of the world minus one).  plan: the stage-t copy of a mate is its body along its plan,
    fleet['plan_xy'][m, t] (from fleet_plan_shapes_batch), instead of its shape moved at constant velocity; the same
    slots in the same order.  Needs time_varying.  ids: also returns obs_id [B,N] int32, each slot's obstacle: the flat
    index of a world shape, S + m for map-mate robot m (S the number of packed shapes), -1 for an empty list.  A world
    with trajectories: as convert_world_obstacles_batch."""
    if plan and not time_varying:
        raise ValueError('a fleet predicted along its plans needs time_varying=True')
    lib = _cabi.load()
    dev = state.device
    B, W = state.shape[0], world['start'].shape[0] - 1
    csr = fleet_csr(robot_world if robot_world is not None else torch.zeros(B, dtype=torch.int32, device=dev), W)
    Tc = T + 1 if time_varying else 1
    A = torch.empty((B, N, Tc, E, 2), dtype=torch.float32, device=dev)
    b = torch.empty((B, N, Tc, E), dtype=torch.float32, device=dev)
    kind = torch.empty((B, N), dtype=torch.int32, device=dev)
    count = torch.empty(B, dtype=torch.int32, device=dev)
    args = (B, W, N, T, E, dt, int(time_varying), int(order), _ptr(state), _ptr(world['start']), _ptr(robot_world),
            _ptr(world['kind']), _ptr(world['nv']), _ptr(world['xy']), _ptr(world['radius']), _ptr(world['vel']),
            _ptr(csr[0]), _ptr(csr[1]), _ptr(fleet['kind']), _ptr(fleet['nv']), _ptr(fleet['xy']), _ptr(fleet['radius']),
            _ptr(fleet['vel']))
    outs = (_ptr(A), _ptr(b), _ptr(kind), _ptr(count), _stream(dev))
    if 'traj' in world:
        traj = _traj_args(world, T, time_varying, dev)
        obs_id = torch.empty((B, N), dtype=torch.int32, device=dev) if ids else None
        with torch.cuda.device(dev):
            _cabi.check(lib.rda_convert_world_obstacles_traj(*args, _ptr(fleet['plan_xy']) if plan else None,
                                                             *outs[:4], _ptr(obs_id), *traj, outs[4]),
                        'rda_convert_world_obstacles_traj')
        return (A, b, kind, count, obs_id) if ids else (A, b, kind, count)
    with torch.cuda.device(dev):
        if ids:
            obs_id = torch.empty((B, N), dtype=torch.int32, device=dev)
            _cabi.check(lib.rda_convert_world_obstacles_ids(*args, _ptr(fleet['plan_xy']) if plan else None, *outs[:4],
                                                            _ptr(obs_id), outs[4]), 'rda_convert_world_obstacles_ids')
            return A, b, kind, count, obs_id
        if plan:
            _cabi.check(lib.rda_convert_fleet_plan_obstacles(*args, _ptr(fleet['plan_xy']), *outs),
                        'rda_convert_fleet_plan_obstacles')
        else:
            _cabi.check(lib.rda_convert_fleet_obstacles(*args, *outs), 'rda_convert_fleet_obstacles')
    return A, b, kind, count


def convert_world_obstacles_horizon_batch(world, nom_s, ref_s, body, robot_world, N, T, E, dt, time_varying=False,
                                          fleet=None, plan=False, per_robot=None, ids=False):
    """convert_world_obstacles_batch (fleet None) or convert_fleet_obstacles_batch (fleet from fleet_shapes_batch or,
    with plan, fleet_plan_shapes_batch) in the horizon order: each robot's shapes sorted by the smallest signed distance
    between its body and the shape's rows over its nominal and reference poses, nom_s, ref_s [B,3,T+1] CUDA tensors.
    body from robot_body with xy a CUDA tensor; per_robot None, or a dict with CUDA tensors 'xy' [B,8,2] and 'radius'
    [B], each robot's own body (body gives the kind and vertex count).  The same list, padding, outputs and obs_count
    as those calls; without a host synchronisation.  ids: also returns obs_id [B,N] int32, the ids of
    convert_fleet_obstacles_batch.  A world with trajectories: as convert_world_obstacles_batch, the horizon key taken
    over each trajectory's stage-t rows."""
    if plan and (fleet is None or not time_varying):
        raise ValueError('a fleet predicted along its plans needs a fleet and time_varying=True')
    lib = _cabi.load()
    dev = nom_s.device
    B, W = nom_s.shape[0], world['start'].shape[0] - 1
    Tc = T + 1 if time_varying else 1
    A = torch.empty((B, N, Tc, E, 2), dtype=torch.float32, device=dev)
    b = torch.empty((B, N, Tc, E), dtype=torch.float32, device=dev)
    kind = torch.empty((B, N), dtype=torch.int32, device=dev)
    count = torch.empty(B, dtype=torch.int32, device=dev)
    mates = (None,) * 8
    if fleet is not None:
        csr = fleet_csr(robot_world if robot_world is not None else torch.zeros(B, dtype=torch.int32, device=dev), W)
        mates = (_ptr(csr[0]), _ptr(csr[1]), _ptr(fleet['kind']), _ptr(fleet['nv']), _ptr(fleet['xy']),
                 _ptr(fleet['radius']), _ptr(fleet['vel']), _ptr(fleet['plan_xy']) if plan else None)
    pr = per_robot or {}
    args = (B, W, N, T, E, dt, int(time_varying), _ptr(nom_s), _ptr(ref_s), int(body['kind']), int(body['nv']),
            _ptr(body['xy']), float(body['radius']), _ptr(pr.get('xy')), _ptr(pr.get('radius')), _ptr(world['start']),
            _ptr(robot_world), _ptr(world['kind']), _ptr(world['nv']), _ptr(world['xy']), _ptr(world['radius']),
            _ptr(world['vel']), *mates, _ptr(A), _ptr(b), _ptr(kind), _ptr(count))
    if 'traj' in world:
        traj = _traj_args(world, T, time_varying, dev)
        obs_id = torch.empty((B, N), dtype=torch.int32, device=dev) if ids else None
        with torch.cuda.device(dev):
            _cabi.check(lib.rda_convert_world_obstacles_horizon_traj(*args, _ptr(obs_id), *traj, _stream(dev)),
                        'rda_convert_world_obstacles_horizon_traj')
        return (A, b, kind, count, obs_id) if ids else (A, b, kind, count)
    with torch.cuda.device(dev):
        if ids:
            obs_id = torch.empty((B, N), dtype=torch.int32, device=dev)
            _cabi.check(lib.rda_convert_world_obstacles_horizon_ids(*args, _ptr(obs_id), _stream(dev)),
                        'rda_convert_world_obstacles_horizon_ids')
            return A, b, kind, count, obs_id
        _cabi.check(lib.rda_convert_world_obstacles_horizon(*args, _stream(dev)), 'rda_convert_world_obstacles_horizon')
    return A, b, kind, count


def shapes_to_device(shapes, device):
    return {k: torch.as_tensor(v, device=device).contiguous() for k, v in shapes.items()}


class BatchedMPC:
    """MPC.control (mpc.py:127-187) for `batch` robots, every step on the device: pre_process -> obstacle conversion
    -> ADMM solve -> arrive rule.  Keyword set of the reference's MPC where it applies.

    Without `robot_path`, every robot follows the one reference path `ref_path`.  With `robot_path` [B], `ref_path`
    is a sequence of W paths and robot b follows path robot_path[b], as a batch of reference MPC objects that each own
    their ref_path; a robot whose robot_path is outside [0, W) has no path (its reference holds its state and it is
    reported as arrived).  With `enable_reverse` each waypoint carries a gear flag in its 4th row (+1 forward, -1
    reverse; mpc.py:139-144): every path is cut into single-gear curves (split_path, mpc.py:232-249), the solver's
    reference speed carries the gear's sign and a robot moves on to the next curve of its path when it reaches the end
    of the current one (mpc.py:166-183).  cur_index is relative to the robot's curve, curve_index to its path.

    control(avoid_fleet=True) makes the robots that share a map obstacles of each other: every other robot of the
    same map, its body at its current pose moving with the control it last applied, follows the map's shapes in the
    list each robot chooses its N nearest obstacles from (convert_fleet_obstacles_batch).  With
    fleet_prediction='plan' (and time_varying=True) each of them instead follows, stage by stage, the controls its own
    last solve kept (cur_vel): the same obstacles in the same slots, turning, braking and stopping as planned.

    update_parameter(robots=mask, max_speed=..., ro2=...) gives robots their own limits, weights and tunables, so that
    robots of different classes (fast and slow, loaded and empty) step in one fleet and one solve.

    With `robot_class` [B], car_tuple is a list of up to 16 car_tuples (robot classes of one cone_type and one number of
    canonical body rows) and robot b is of class robot_class[b]: its body, wheelbase, dynamics and limits (and its body
    and motion as others see it with avoid_fleet).  The handle is built with class 0, so an index outside the list means
    class 0.  set_robot_class moves robots between classes on the device.

    obstacle_order: True sorts each robot's obstacles by the reference's key (mpc.py:210-218, the distance from its
    position to a polygon's nearest vertex or a disc's centre), False keeps list order, and 'horizon' sorts them by how
    close the robot's horizon comes to them: the smallest signed distance between its body and the obstacle's rows over
    its nominal and reference poses (convert_world_obstacles_horizon_batch).  'horizon' takes world= (and avoid_fleet),
    not shapes=.

    warm_start: 'slot' (default, the reference's behaviour) leaves each slot's warm start (the ADMM multipliers of the
    last solve) in its slot, whichever obstacle the selection puts there next; 'obstacle' moves it with the obstacle
    (RDA_solver.set_obstacle_ids), and info['obs_id'] [B,N] says which obstacle each slot held.  An obstacle's identity
    is its list position: its flat index in the packed world (pack_worlds), S + m for map-mate robot m (S packed shapes),
    its position in a robot's shapes= list.  A caller who repacks a map must keep its order for the warm start to
    follow.  A step without obstacles gives every slot the id -1, so each slot starts cold when obstacles come back.

    A world from pack_worlds whose obstacles carry trajectories (traj, traj_xy) makes those shapes follow them over the
    horizon, the reference's time-varying rdaobs (MPC(rda_obstacle=True)): keyed by their stage 0, written along their
    stages, with every obstacle_order, avoid_fleet, fleet_prediction and warm_start, and time_varying=True.  The caller
    may overwrite world['traj_xy'] (and world['traj']) on the device between steps, e.g. with a predictor's output."""

    def __init__(self, car_tuple, ref_path, batch, receding=10, sample_time=0.1, iter_num=4,
                 enable_reverse=False, obstacle_order=True, max_edge_num=5, max_obs_num=5,
                 accelerated=True, goal_index_threshold=1, device=None, iter_threshold=0.2, robot_path=None,
                 robot_class=None, warm_start='slot', **kwargs):
        self.lib = _cabi.load()
        if warm_start not in ('slot', 'obstacle'):
            raise ValueError(f"warm_start is 'slot' or 'obstacle', not {warm_start!r}")
        self.warm_start = warm_start
        self.enable_reverse = bool(enable_reverse)
        self.classes = None
        if robot_class is not None:
            self.classes = list(car_tuple)
            if not self.classes:
                raise ValueError('robot_class needs at least one car_tuple')
            car_tuple = self.classes[0]
        if isinstance(obstacle_order, str) and obstacle_order != 'horizon':
            raise ValueError(f"obstacle_order is True, False or 'horizon', not {obstacle_order!r}")
        self.rda = RDA_solver(receding, car_tuple, max_edge_num, max_obs_num, iter_num=iter_num,
                              step_time=sample_time, iter_threshold=iter_threshold, accelerated=accelerated,
                              time_print=False, batch=batch, device=device, **kwargs)
        self.device = self.rda.device
        self.batch, self.T, self.dt = batch, receding, sample_time
        self.N, self.E = max_obs_num, self.rda.max_edge_num
        self.car_tuple = car_tuple
        self.dynamics, self.L = car_tuple.dynamics, float(car_tuple.wheelbase)
        self.obstacle_order = obstacle_order
        self.goal_index_threshold = goal_index_threshold
        self.update_ref_path(ref_path, robot_path)
        init_vel = kwargs.get('init_vel')
        self.cur_vel = torch.zeros((batch, 2, receding), dtype=torch.float32, device=self.device)
        if init_vel is not None:
            self.cur_vel[:] = torch.as_tensor(init_vel, dtype=torch.float32, device=self.device)
        self.arrive = torch.zeros(batch, dtype=torch.int32, device=self.device)
        self._empty = None
        self.body = robot_body(car_tuple)
        self.body['xy'] = torch.as_tensor(self.body['xy'], device=self.device)
        self._no_world = None
        self.per_robot = None
        if self.classes is not None:
            self.rda.set_robot_classes(self.classes, robot_class)
            bodies = [robot_body(c) for c in self.classes + [car_tuple]]
            self._class_nv = max(int(bd['nv']) for bd in bodies)
            dev = self.device
            # per class slot [K + 1] (slot K: class 0, the handle's own), uploaded once
            self._class_tables = {
                'dynamics': torch.tensor([_cabi.DYNAMICS[c.dynamics] for c in self.classes + [car_tuple]],
                                         dtype=torch.int32, device=dev),
                'wheelbase': torch.tensor([float(c.wheelbase) for c in self.classes + [car_tuple]], dtype=torch.float32,
                                          device=dev),
                'xy': torch.as_tensor(np.stack([bd['xy'] for bd in bodies]), device=dev),
                'radius': torch.tensor([bd['radius'] for bd in bodies], dtype=torch.float32, device=dev)}
            self._gather_classes()

    def _gather_classes(self):
        """Each robot's dynamics, wheelbase and body from its class, gathered on the device."""
        slot = self.rda.class_slot()
        self.per_robot = {k: v[slot].contiguous() for k, v in self._class_tables.items()}

    def set_robot_class(self, index, robots):
        """Move the robots of the bool mask robots [B] to class index ([B] or one index; outside the classes: class 0):
        their body, wheelbase, dynamics, max_speed and max_acce change from the next control call, their warm start is
        kept.  On the device, without a host synchronisation when index and robots are CUDA tensors."""
        if self.classes is None:
            raise RuntimeError('set_robot_class needs a fleet built with robot_class')
        self.rda.set_robot_class_index(index, torch.as_tensor(robots, dtype=torch.bool, device=self.device))
        self._gather_classes()

    def update_ref_path(self, ref_path, robot_path=None):
        """MPC.update_ref_path (mpc.py:220-227) for the whole fleet: replace the path set (one path, or W paths with
        robot_path [B] as in the constructor) and put every robot back at the start of its path's first curve.
        cur_vel is kept, as in the reference."""
        dev = self.device
        paths = [ref_path] if robot_path is None else list(ref_path)
        packed = {k: torch.as_tensor(v, device=dev).contiguous()
                  for k, v in pack_paths(paths, self.enable_reverse).items()}
        self.path, self.curve_start = packed['path'], packed['curve_start']
        self.path_curve, self.curve_gear = packed['path_curve'], packed['curve_gear']
        self.n_paths, self.n_curves = len(paths), packed['curve_gear'].shape[0]
        if robot_path is None:
            self.robot_path = torch.zeros(self.batch, dtype=torch.int32, device=dev)
        else:
            self.robot_path = torch.as_tensor(robot_path, dtype=torch.int32, device=dev).reshape(self.batch).contiguous()
        self.cur_index = torch.zeros(self.batch, dtype=torch.int32, device=dev)
        self.curve_index = torch.zeros(self.batch, dtype=torch.int32, device=dev)

    def set_robot_path(self, robot_path, robots):
        """Put the robots of the bool mask robots [B] on paths of the current set, robot_path [B] or one index for all
        of them, at the start of the path's first curve: MPC.update_ref_path on those robots' MPCs.  On the device,
        without a host synchronisation; an index outside [0, W) leaves the robot without a path."""
        dev = self.device
        robots = torch.as_tensor(robots, dtype=torch.bool, device=dev).reshape(self.batch)
        robot_path = torch.as_tensor(robot_path, dtype=torch.int32, device=dev)
        self.robot_path = torch.where(robots, robot_path, self.robot_path).contiguous()
        self.cur_index = self.cur_index.masked_fill(robots, 0)
        self.curve_index = self.curve_index.masked_fill(robots, 0)

    def update_parameter(self, robots=None, **kwargs):
        """MPC.update_parameter (mpc.py:229-230) for the whole fleet, or for the robots of the bool mask robots [B].
        With scalar tunables and no mask this is exactly assign_adjust_parameter (slack_gain, max_sd, min_sd, ro1, ro2;
        ws / wu ignored, as in the reference).  Otherwise the values go to the robots' own rows
        (RDA_solver.set_instance_parameters): scalars or [B] / [B, 2] per robot, array-likes or CUDA tensors, and also
        max_speed / max_acce (pairs) and ws / wu, so that one fleet can hold robots of different classes."""
        uniform = robots is None and all(k not in ('max_speed', 'max_acce') and not isinstance(v, torch.Tensor)
                                         and np.ndim(v) == 0 for k, v in kwargs.items())
        if uniform:
            self.rda.assign_adjust_parameter(**kwargs)
        else:
            self.rda.set_instance_parameters(robots, **kwargs)

    def _no_obstacles(self):
        if self._empty is None:
            B, N, E, dev = self.batch, max(self.N, 1), self.E, self.device
            self._empty = (torch.zeros((B, N, 1, E, 2), dtype=torch.float32, device=dev),
                           torch.zeros((B, N, 1, E), dtype=torch.float32, device=dev),
                           torch.zeros((B, N), dtype=torch.int32, device=dev),
                           torch.zeros(B, dtype=torch.int32, device=dev))
        return self._empty

    def control(self, state, ref_speed=5.0, shapes=None, time_varying=False, world=None, robot_world=None,
                avoid_fleet=False, clearance=False, fleet_prediction='velocity'):
        """state [B,3] (CUDA tensor or array), ref_speed scalar or [B], shapes: dict from
        pack_shapes / shapes_to_device (None: free space).  Instead of shapes, world: dict from
        pack_worlds / shapes_to_device, obstacle maps shared by the robots, with robot_world [B] the map of
        each robot (may be omitted with a single map).  avoid_fleet: every robot also sees the other robots of its map
        (without world: all robots, in an empty map) as moving obstacles; not with shapes.  fleet_prediction: how those
        robots move over the horizon, 'velocity' (at the constant velocity of the control each just applied) or 'plan'
        (along the controls its last solve kept, cur_vel; needs avoid_fleet and time_varying=True).  Returns (u0 [B,2], info)
        where info holds the solver's batched outputs plus 'arrive', 'nom_s', 'ref_s', 'cur_index', 'curve_index'.
        clearance: info also holds 'clearance' [B] and 'clearance_index' [B] of the plan just solved
        (RDA_solver.plan_clearance: the smallest signed distance between a robot's planned footprints and the obstacles
        it was given, negative inside one, and where it occurs).  No host sync."""
        dev, B, T = self.device, self.batch, self.T
        if fleet_prediction not in ('velocity', 'plan'):
            raise ValueError(f"fleet_prediction is 'velocity' or 'plan', not {fleet_prediction!r}")
        plan = fleet_prediction == 'plan'
        if plan and not avoid_fleet:
            raise ValueError("fleet_prediction='plan' predicts the map-mates of avoid_fleet=True")
        if plan and not time_varying:
            raise ValueError("fleet_prediction='plan' needs time_varying=True: the prediction is a trajectory")
        horizon = isinstance(self.obstacle_order, str)
        if horizon and shapes is not None:
            raise ValueError("obstacle_order='horizon' selects from worlds, not from shapes=: pass the lists as worlds "
                             "(world=pack_worlds(lists), one world per robot, robot_world=arange(B))")
        if avoid_fleet:
            if shapes is not None:
                raise ValueError('avoid_fleet takes its obstacles from world= (or an empty map), not from shapes')
            nv = self.body['nv'] if self.classes is None else self._class_nv
            if self.body['kind'] == _cabi.OBS_POLYGON and nv > self.E:
                raise ValueError(f'avoid_fleet: a robot body has {nv} vertices, more than '
                                 f'max_edge_num={self.E} obstacle rows')
            if world is None:
                if self._no_world is None:
                    self._no_world = shapes_to_device(pack_worlds([[]]), dev)
                world = self._no_world
        if shapes is not None and 'traj' in shapes:
            raise ValueError('obstacles with trajectories are selected from worlds, not from shapes=: pass the lists as '
                             'worlds (world=pack_worlds(lists), one world per robot, robot_world=arange(B))')
        if world is not None and 'traj' in world:
            _check_traj(world, T, time_varying)
        if world is not None:
            if shapes is not None:
                raise ValueError('pass either shapes or world, not both')
            if robot_world is None and world['start'].shape[0] != 2:
                raise ValueError('robot_world is required with more than one world')
            if robot_world is not None:
                robot_world = torch.as_tensor(robot_world, dtype=torch.int32, device=dev).reshape(B).contiguous()
        state = torch.as_tensor(state, dtype=torch.float32, device=dev).reshape(B, -1)[:, :3].contiguous()
        if not isinstance(ref_speed, torch.Tensor):
            ref_speed = torch.full((B,), float(ref_speed), dtype=torch.float32, device=dev) if np.isscalar(ref_speed) \
                else torch.as_tensor(ref_speed, dtype=torch.float32, device=dev)
        ref_speed = ref_speed.to(dtype=torch.float32).contiguous()
        nom_s = torch.empty((B, 3, T + 1), dtype=torch.float32, device=dev)
        ref_s = torch.empty((B, 3, T + 1), dtype=torch.float32, device=dev)
        near = torch.empty(B, dtype=torch.int32, device=dev)
        solver_speed = torch.empty(B, dtype=torch.float32, device=dev)          # gear_flag * ref_speed (mpc.py:161)
        paths = (_ptr(self.path), self.n_paths, _ptr(self.path_curve), _ptr(self.curve_start), _ptr(self.curve_gear),
                 _ptr(self.robot_path), _ptr(self.curve_index), _ptr(self.cur_index), 0.1, 10, _ptr(nom_s), _ptr(ref_s),
                 _ptr(near), _ptr(solver_speed), _stream(dev))
        with torch.cuda.device(dev):
            if self.per_robot is None:
                _cabi.check(self.lib.rda_pre_process_paths(
                    B, T, _cabi.DYNAMICS[self.dynamics], self.dt, self.L, _ptr(state), _ptr(self.cur_vel),
                    _ptr(ref_speed), *paths), 'rda_pre_process_paths')
            else:
                _cabi.check(self.lib.rda_pre_process_paths_per_robot(
                    B, T, _ptr(self.per_robot['dynamics']), self.dt, _ptr(self.per_robot['wheelbase']), _ptr(state),
                    _ptr(self.cur_vel), _ptr(ref_speed), *paths), 'rda_pre_process_paths_per_robot')
        self.cur_index = near
        ids = self.warm_start == 'obstacle'
        if (shapes is None and world is None) or self.N == 0:
            conv = self._no_obstacles() + ((torch.full((B, self.N), -1, dtype=torch.int32, device=dev),) if ids else ())
            time_varying = False
        elif horizon:
            fleet = None
            if avoid_fleet:
                fleet = fleet_shapes_batch(state, self.cur_vel, self.body, self.dynamics, self.per_robot) if not plan \
                    else fleet_plan_shapes_batch(state, self.cur_vel, self.body, self.dynamics, self.dt, self.L,
                                                 self.per_robot)
            conv = convert_world_obstacles_horizon_batch(world, nom_s, ref_s, self.body, robot_world, self.N, T, self.E,
                                                         self.dt, time_varying, fleet, plan, self.per_robot, ids)
        elif avoid_fleet:
            if plan:
                fleet = fleet_plan_shapes_batch(state, self.cur_vel, self.body, self.dynamics, self.dt, self.L,
                                                self.per_robot)
            else:
                fleet = fleet_shapes_batch(state, self.cur_vel, self.body, self.dynamics, self.per_robot)
            conv = convert_fleet_obstacles_batch(world, state, robot_world, fleet, self.N, T, self.E, self.dt,
                                                 time_varying, self.obstacle_order, plan, ids)
        elif world is not None:
            conv = convert_world_obstacles_batch(world, state, robot_world, self.N, T, self.E, self.dt, time_varying,
                                                 self.obstacle_order, ids)
        else:
            conv = convert_obstacles_batch(shapes, state, self.N, T, self.E, self.dt, time_varying, self.obstacle_order,
                                           ids)
        A, b, kind, count = conv[:4]
        obs_id = conv[4] if ids else None
        if ids:
            self.rda.set_obstacle_ids(obs_id)
        out = self.rda.iterative_solve_batch(nom_s, self.cur_vel, ref_s, solver_speed, A, b, kind, count, time_varying)
        with torch.cuda.device(dev):
            _cabi.check(self.lib.rda_post_process_paths(B, T, self.n_paths, _ptr(self.path_curve), _ptr(self.curve_start),
                                                        _ptr(self.robot_path), self.goal_index_threshold, _ptr(near),
                                                        _ptr(self.curve_index), _ptr(out['u']), _ptr(self.cur_vel),
                                                        _ptr(self.arrive), _stream(dev)), 'rda_post_process_paths')
        info = dict(out)
        info.update(arrive=self.arrive, nom_s=nom_s, ref_s=ref_s, cur_index=near, curve_index=self.curve_index)
        if ids:
            info['obs_id'] = obs_id
        if clearance:
            c = self.rda.plan_clearance()
            info.update(clearance=c['min'], clearance_index=c['index'])
        return out['u'][:, :, 0], info

    def advance(self, state):
        """One simulator step with the first control of the last solve (mpc.py:293-336), in place."""
        with torch.cuda.device(self.device):
            if self.per_robot is not None:
                _cabi.check(self.lib.rda_motion_predict_per_robot(
                    self.batch, self.T, _ptr(self.per_robot['dynamics']), self.dt, _ptr(self.per_robot['wheelbase']),
                    _ptr(self.cur_vel), _ptr(state), _stream(self.device)), 'rda_motion_predict_per_robot')
                return state
            _cabi.check(self.lib.rda_motion_predict(self.batch, self.T, _cabi.DYNAMICS[self.dynamics], self.dt, self.L,
                                                    _ptr(self.cur_vel), _ptr(state), _stream(self.device)),
                        'rda_motion_predict')
        return state

    def reset(self):
        self.rda.reset()
        self.cur_index.zero_()
        self.cur_vel.zero_()
        self.curve_index.zero_()
