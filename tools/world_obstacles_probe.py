"""Time rda_convert_world_obstacles (each robot's N nearest shapes of a shared obstacle map) on the GPU.

For B robots in ONE shared world of M boxes (N = 20, static and time-varying output), CUDA events around many
launches of the conversion alone; at each B the time of one warm-started BatchedMPC.control + advance step on the
M = 16384 map (bench.py's closed_loop shape: metric row T = 30, N = 20, E = 4, 50 ADMM iterations), so every
conversion time is also given as a fraction of that step; and at M = 64 with per-robot worlds, the existing
rda_convert_obstacles on the same inputs next to the new entry point.  Writes DIR/world_obstacles_probe.json with the
GPU's name and power limit read in the same run.

    python tools/world_obstacles_probe.py DIR [--batches 256,4096,16384] [--maps 64,1024,16384,65536]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
T, N, E, ITERS, DT = 30, 20, 4, 50, 0.1
STEP_MAP = 16384


def gpu_identity(index):
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader,nounits', '-i', str(index)],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(',')
        return {'name': q[0].strip(), 'power_limit_w': float(q[1])}
    except Exception:
        import torch
        return {'name': torch.cuda.get_device_name(index), 'power_limit_w': None}


def boxes(rng, lead, lo_x, hi_x):
    """2 x 1 m boxes of random yaw, centres lo_x..hi_x along the 60 m line and 1.8..6 m to either side."""
    ctr = np.stack([rng.uniform(lo_x, hi_x, lead), rng.uniform(1.8, 6, lead) * rng.choice([-1, 1], lead)], -1)
    yaw = rng.uniform(0, np.pi, lead)
    corners = np.array([[-1, -0.5], [1, -0.5], [1, 0.5], [-1, 0.5]])
    rot = np.stack([np.stack([np.cos(yaw), -np.sin(yaw)], -1), np.stack([np.sin(yaw), np.cos(yaw)], -1)], -2)
    xy = np.zeros(lead + (8, 2), np.float32)
    xy[..., :4, :] = ctr[..., None, :] + np.einsum('...ij,kj->...ki', rot, corners)
    return {'kind': np.zeros(lead, np.int32), 'nv': np.full(lead, 4, np.int32), 'xy': xy,
            'radius': np.zeros(lead, np.float32), 'vel': np.zeros(lead + (2,), np.float32)}


def event_ms(fn, dev, min_window_s=0.3):
    """Mean time of fn() over enough back-to-back launches to fill min_window_s, after a warm-up."""
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize(dev)
    reps = int(min(500, max(10, min_window_s / max(e0.elapsed_time(e1) * 1e-3, 1e-6))))
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize(dev)
    return e0.elapsed_time(e1) / reps, reps


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('out_dir')
    ap.add_argument('--batches', default='256,4096,16384')
    ap.add_argument('--maps', default='64,1024,16384,65536')
    args = ap.parse_args()
    import torch
    from rda_planner_b200 import _cabi
    from rda_planner_b200.frontend import BatchedMPC, _ptr, _stream
    from rda_planner_b200.scenarios import rectangle_robot
    assert torch.cuda.is_available(), 'the probe measures the GPU; there is nothing to measure without one'
    dev = torch.device('cuda:0')
    lib = _cabi.load()
    batches = [int(x) for x in args.batches.split(',')]
    maps = [int(x) for x in args.maps.split(',')]
    rng = np.random.default_rng(5)
    path = np.stack([np.arange(0, 60, 0.1), np.zeros(600), np.zeros(600)], 1)
    out = {'gpu': gpu_identity(0), 'N': N, 'E': E, 'T': T, 'shape': '2 x 1 m boxes (4 vertices)',
           'conversion': [], 'per_robot_m64': [], 'control_step': []}
    worlds = {}
    for M in maps:
        host = boxes(rng, (M,), 0.0, 60.0)
        worlds[M] = {k: torch.as_tensor(v, device=dev) for k, v in host.items()}
        worlds[M]['start'] = torch.as_tensor([0, M], dtype=torch.int32, device=dev)
    for B in batches:
        idx = rng.integers(0, 480, B)
        state = torch.as_tensor(path[idx] + rng.normal(0, [0.3, 0.3, 0.1], (B, 3)), dtype=torch.float32, device=dev)
        for tv in (0, 1):
            Tc = T + 1 if tv else 1
            A = torch.empty((B, N, Tc, E, 2), dtype=torch.float32, device=dev)
            b = torch.empty((B, N, Tc, E), dtype=torch.float32, device=dev)
            kind = torch.empty((B, N), dtype=torch.int32, device=dev)
            count = torch.empty(B, dtype=torch.int32, device=dev)
            outs = [_ptr(A), _ptr(b), _ptr(kind), _ptr(count), _stream(dev)]
            for M in maps:
                w = worlds[M]
                args_w = [_ptr(state), _ptr(w['start']), None, _ptr(w['kind']), _ptr(w['nv']), _ptr(w['xy']),
                          _ptr(w['radius']), _ptr(w['vel'])] + outs
                ms, reps = event_ms(lambda: _cabi.check(lib.rda_convert_world_obstacles(B, 1, N, T, E, DT, tv, 1, *args_w),
                                                        'rda_convert_world_obstacles'), dev)
                out['conversion'].append({'B': B, 'M': M, 'time_varying': bool(tv), 'ms': ms, 'launches': reps,
                                          'shape_keys_per_s': B * M / (ms * 1e-3)})
            # M = 64 per robot: the same inputs through both entry points
            per = {k: torch.as_tensor(v, device=dev) for k, v in boxes(rng, (B, 64), 0.0, 60.0).items()}
            per['count'] = torch.full((B,), 64, dtype=torch.int32, device=dev)
            starts = torch.arange(0, 64 * (B + 1), 64, dtype=torch.int32, device=dev)
            robot_world = torch.arange(B, dtype=torch.int32, device=dev)
            shp = [_ptr(per['kind']), _ptr(per['nv']), _ptr(per['xy']), _ptr(per['radius']), _ptr(per['vel'])]
            ms_old, _ = event_ms(lambda: _cabi.check(lib.rda_convert_obstacles(B, 64, N, T, E, DT, tv, 1, _ptr(state), *shp,
                                                                               _ptr(per['count']), *outs),
                                                     'rda_convert_obstacles'), dev)
            ref = [t.clone() for t in (A, b, kind, count)]
            ms_new, _ = event_ms(lambda: _cabi.check(lib.rda_convert_world_obstacles(B, B, N, T, E, DT, tv, 1, _ptr(state),
                                                                                     _ptr(starts), _ptr(robot_world), *shp,
                                                                                     *outs),
                                                     'rda_convert_world_obstacles'), dev)
            same = all(torch.equal(r, t) for r, t in zip(ref, (A, b, kind, count)))
            out['per_robot_m64'].append({'B': B, 'time_varying': bool(tv), 'rda_convert_obstacles_ms': ms_old,
                                         'rda_convert_world_obstacles_ms': ms_new, 'outputs_bit_identical': same})
            del A, b, kind, count
        # one warm-started control step that takes its obstacles from the shared map
        if STEP_MAP in worlds:
            bm = BatchedMPC(rectangle_robot(), path, B, receding=T, sample_time=DT, iter_num=ITERS, max_edge_num=E,
                            max_obs_num=N, iter_threshold=0.0, device=dev)
            bm.cur_index[:] = torch.as_tensor(np.maximum(idx - 3, 0), dtype=torch.int32)
            bm.cur_vel[:, 0, :] = 4.0
            st = state.clone()

            def step():
                bm.control(st, 4.0, world=worlds[STEP_MAP])
                bm.advance(st)
            ms, reps = event_ms(step, dev, min_window_s=1.0)
            u0, info = bm.control(st, 4.0, world=worlds[STEP_MAP])
            ok = bool(torch.isfinite(u0).all()) and int((info['status'] & 6).sum()) == 0
            out['control_step'].append({'B': B, 'M': STEP_MAP, 'ms': ms, 'steps': reps, 'mpc_steps_per_s': B / (ms * 1e-3),
                                        'finite_and_converged': ok})
            del bm
    steps = {r['B']: r['ms'] for r in out['control_step']}
    for r in out['conversion']:
        r['fraction_of_control_step'] = r['ms'] / steps[r['B']] if r['B'] in steps else 'not measured'
    out['what'] = ('conversion: one launch of rda_convert_world_obstacles (order = 1, every robot in the one world), '
                   'CUDA events; control_step: BatchedMPC.control(world=...) + advance, warm-started, 50 iterations; '
                   'fraction_of_control_step: conversion ms over control step ms at the same B (static map of '
                   f'{STEP_MAP} boxes for the step)')
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, 'world_obstacles_probe.json'), 'w') as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
