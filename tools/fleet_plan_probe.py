"""Measure the plan prediction of a fleet (fleet_prediction='plan') against the velocity prediction on the GPU.

  kernels   CUDA events over many launches of the plan pair (rda_fleet_plan_shapes + rda_convert_fleet_plan_obstacles)
            and the velocity pair (rda_fleet_shapes + rda_convert_fleet_obstacles), both time-varying, order = 1, at
            B in {256, 4 096, 16 384}, T = 30, N = 20, E = 4, worlds of 8 and 256 robots each on a map of 1 024 boxes;
            the two pairs alternated, three rounds each.
  steps     warm-started BatchedMPC.control + advance at B = 16 384 and 50 ADMM iterations, robots 6 m apart on the
            path in worlds of 8 on maps of 1 024 boxes: velocity with time_varying=False, velocity and plan with
            time_varying=True, alternated step by step in one session.
  safety    a closed loop of seeded crossings (three robots per world: one straight, one crossing at right angles, one
            turning left across both lanes, with random lags), run with each prediction and with the robots blind to
            each other: body overlaps of the executed poses, the smallest executed robot-to-robot signed distance
            (oracle.clearance on the host) and the share of plans whose clearance is below 0 and below min_sd.

Writes OUT/fleet_plan_probe.json with the GPU's name and power limit read in the same run.

    python tools/fleet_plan_probe.py OUT [--batches 256,4096,16384] [--safety-worlds 64] [--safety-steps 120]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from fleet_obstacles_probe import boxes  # noqa: E402
from world_obstacles_probe import event_ms, gpu_identity  # noqa: E402

T, N, E, ITERS, DT = 30, 20, 4, 50, 0.1


def kernels(torch, lib, dev, batches, gen, rng):
    from rda_planner_b200 import _cabi
    from rda_planner_b200.frontend import _ptr, _stream, fleet_csr, robot_body
    from rda_planner_b200.scenarios import rectangle_robot
    body = robot_body(rectangle_robot())
    bxy = torch.as_tensor(body['xy'], device=dev)
    path = np.stack([np.arange(0, 60, 0.1), np.zeros(600), np.zeros(600)], 1)
    rows, M = [], 1024
    for B in batches:
        idx = rng.integers(0, 480, B)
        state = torch.as_tensor(path[idx] + rng.normal(0, [0.3, 0.3, 0.1], (B, 3)), dtype=torch.float32, device=dev)
        cur_vel = torch.zeros((B, 2, T), device=dev)
        cur_vel[:, 0, :] = 4.0
        cur_vel[:, 1, :] = torch.rand((B, T), device=dev, generator=gen) * 0.4 - 0.2
        fl = {'kind': torch.empty(B, dtype=torch.int32, device=dev), 'nv': torch.empty(B, dtype=torch.int32, device=dev),
              'xy': torch.empty((B, 8, 2), device=dev), 'radius': torch.empty(B, device=dev),
              'vel': torch.empty((B, 2), device=dev), 'plan': torch.empty((B, T + 1, 8, 2), device=dev)}
        for R in (8, 256):
            if R > B:
                continue
            W = B // R
            rw = (torch.arange(B, device=dev) % W).to(torch.int32)
            start, robots = fleet_csr(rw, W)
            w = boxes(torch, W, M, dev, gen)
            outs = {p: (torch.empty((B, N, T + 1, E, 2), device=dev), torch.empty((B, N, T + 1, E), device=dev),
                        torch.empty((B, N), dtype=torch.int32, device=dev), torch.empty(B, dtype=torch.int32, device=dev))
                    for p in (False, True)}
            s = _stream(dev)
            common = lambda: (B, W, N, T, E, DT, 1, 1, _ptr(state), _ptr(w['start']), _ptr(rw), _ptr(w['kind']),  # noqa
                              _ptr(w['nv']), _ptr(w['xy']), _ptr(w['radius']), _ptr(w['vel']), _ptr(start),
                              _ptr(robots), _ptr(fl['kind']), _ptr(fl['nv']), _ptr(fl['xy']), _ptr(fl['radius']),
                              _ptr(fl['vel']))
            fleet_out = lambda: (_ptr(fl['kind']), _ptr(fl['nv']), _ptr(fl['xy']), _ptr(fl['radius']),  # noqa
                                 _ptr(fl['vel']))

            def velocity():
                _cabi.check(lib.rda_fleet_shapes(B, T, 0, body['kind'], body['nv'], _ptr(bxy), body['radius'],
                                                 _ptr(state), _ptr(cur_vel), *fleet_out(), s), 'rda_fleet_shapes')
                o = outs[False]
                _cabi.check(lib.rda_convert_fleet_obstacles(*common(), *(_ptr(x) for x in o), s),
                            'rda_convert_fleet_obstacles')

            def plan():
                _cabi.check(lib.rda_fleet_plan_shapes(B, T, 0, DT, 3.0, body['kind'], body['nv'], _ptr(bxy),
                                                      body['radius'], None, None, None, None, _ptr(state),
                                                      _ptr(cur_vel), *fleet_out(), _ptr(fl['plan']), s),
                            'rda_fleet_plan_shapes')
                o = outs[True]
                _cabi.check(lib.rda_convert_fleet_plan_obstacles(*common(), _ptr(fl['plan']), *(_ptr(x) for x in o), s),
                            'rda_convert_fleet_plan_obstacles')
            times = {'velocity': [], 'plan': []}
            for _ in range(3):
                for name, fn in (('velocity', velocity), ('plan', plan)):
                    times[name].append(event_ms(fn, dev)[0])
            torch.cuda.synchronize(dev)
            same = {k: bool(torch.equal(outs[False][k][:, :, :1] if k < 2 else outs[False][k],
                                        outs[True][k][:, :, :1] if k < 2 else outs[True][k])) for k in range(4)}
            rows.append({'B': B, 'robots_per_world': R, 'worlds': W, 'M': M,
                         'velocity_ms': times['velocity'], 'plan_ms': times['plan'],
                         'velocity_median_ms': float(np.median(times['velocity'])),
                         'plan_median_ms': float(np.median(times['plan'])),
                         'stage0_kind_count_bitwise_equal': all(same.values())})
            del outs, w
        torch.cuda.empty_cache()
    return rows


def steps(torch, dev, gen, rng, rounds=6):
    from rda_planner_b200.frontend import BatchedMPC
    from rda_planner_b200.scenarios import rectangle_robot
    B, R, M = 16384, 8, 1024
    W = B // R
    path = np.stack([np.arange(0, 60, 0.1), np.zeros(600), np.zeros(600)], 1)
    idx = (np.arange(B) // W) * 60 + rng.integers(0, 10, B)
    state0 = torch.as_tensor(path[idx] + rng.normal(0, [0.1, 0.1, 0.05], (B, 3)), dtype=torch.float32, device=dev)
    rw = (torch.arange(B, device=dev) % W).to(torch.int32)
    world = boxes(torch, W, M, dev, gen)
    configs = {'velocity_static': (False, 'velocity'), 'velocity_tv': (True, 'velocity'), 'plan_tv': (True, 'plan')}
    runs = {}
    for name, (tv, pred) in configs.items():
        bm = BatchedMPC(rectangle_robot(), path, B, receding=T, sample_time=DT, iter_num=ITERS, max_edge_num=E,
                        max_obs_num=N, iter_threshold=0.0, device=dev)
        bm.cur_index[:] = torch.as_tensor(np.maximum(idx - 3, 0), dtype=torch.int32)
        bm.cur_vel[:, 0, :] = 4.0
        st = state0.clone()
        for _ in range(3):                                          # warm start and warm up
            bm.control(st, 4.0, world=world, robot_world=rw, avoid_fleet=True, time_varying=tv, fleet_prediction=pred)
            bm.advance(st)
        runs[name] = (bm, st, tv, pred)
    torch.cuda.synchronize(dev)
    times = {k: [] for k in configs}
    finite = {k: True for k in configs}
    for _ in range(rounds):
        for name, (bm, st, tv, pred) in runs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            u0, _ = bm.control(st, 4.0, world=world, robot_world=rw, avoid_fleet=True, time_varying=tv,
                               fleet_prediction=pred)
            bm.advance(st)
            e1.record()
            torch.cuda.synchronize(dev)
            times[name].append(e0.elapsed_time(e1))
            finite[name] &= bool(torch.isfinite(u0).all())
    return {'B': B, 'robots_per_world': R, 'M': M, 'T': T, 'N': N, 'E': E, 'iters': ITERS,
            'ms_per_step': times, 'median_ms': {k: float(np.median(v)) for k, v in times.items()}, 'finite': finite,
            'what': 'BatchedMPC.control(avoid_fleet=True) + advance, warm-started, the three configurations alternated '
                    'step by step; CUDA events around each step'}


def _line(x0, y0, heading, n, step=0.25):
    return [np.array([[x0 + step * i * np.cos(heading)], [y0 + step * i * np.sin(heading)], [heading]])
            for i in range(n)]


def _arc(cx, cy, r, phi0, phi1, step=0.25):
    n = int(abs(phi1 - phi0) * r / step) + 1
    turn = 1.0 if phi1 > phi0 else -1.0
    return [np.array([[cx + r * np.cos(p)], [cy + r * np.sin(p)], [p + turn * np.pi / 2]])
            for p in np.linspace(phi0, phi1, n)]


def safety(torch, dev, worlds, n_steps, seed=3):
    """Three robots per world: 0 east along y = 0, 1 north along x = 0, 2 from the south-east turning left on an arc
    (centre (-8, -8), radius 10) that crosses both lanes, then west along y = 2; each starts `lag` metres further back,
    lags drawn per world so that many worlds meet at the crossing together."""
    from oracle import clearance as oc
    from rda_planner_b200.frontend import BatchedMPC, pack_worlds, shapes_to_device
    from rda_planner_b200.scenarios import rectangle_robot
    car = rectangle_robot(length=2.0, width=1.0, wheelbase=1.2, dynamics='diff', max_speed=(3, 1.5), max_acce=(3, 1.5))
    paths = [_line(-12.0, 0.0, 0.0, 200), _line(0.0, -12.0, np.pi / 2, 200),
             _arc(-8.0, -8.0, 10.0, 0.0, np.pi / 2) + _line(-8.25, 2.0, np.pi, 120)[1:]]
    rng = np.random.default_rng(seed)
    lag = rng.uniform(0.0, 4.0, (worlds, 3))
    B = 3 * worlds
    robot_path = np.tile([0, 1, 2], worlds)
    robot_world = np.repeat(np.arange(worlds), 3).astype(np.int32)
    start = np.zeros(B, np.int64)
    start[0::3] = np.round(lag[:, 0] / 0.25)                      # robots 0 and 1 begin 4 m nearer, robot 2 on its arc
    start[1::3] = np.round(lag[:, 1] / 0.25)
    start[2::3] = 0
    state0 = np.array([np.asarray(paths[p][int(s)], float).reshape(-1)[:3] for p, s in zip(robot_path, start)])
    state0[2::3, 1] -= lag[:, 2]                                   # robot 2 further back, south of its arc
    modes = {'plan': (True, 'plan'), 'velocity': (True, 'velocity'), 'blind': (False, 'velocity')}
    body_V = None
    out = {}
    for name, (avoid, pred) in modes.items():
        bm = BatchedMPC(car, paths, B, robot_path=robot_path, receding=12, sample_time=DT, iter_num=4, max_edge_num=4,
                        max_obs_num=3, iter_threshold=0.0, device=dev)
        bm.cur_index[:] = torch.as_tensor(start, dtype=torch.int32)
        body_V = bm.body['xy'][:bm.body['nv']].cpu().numpy().astype(float)
        min_sd = float(bm.rda.get_adjust_parameter()['min_sd'])
        state = torch.as_tensor(state0, dtype=torch.float32, device=dev)
        rw = torch.as_tensor(robot_world, device=dev)
        world = shapes_to_device(pack_worlds([[] for _ in range(worlds)]), dev)
        traj, clear = [state.cpu().numpy().copy()], []
        for _ in range(n_steps):
            _, info = bm.control(state, 2.0, time_varying=True, world=world, robot_world=rw, avoid_fleet=avoid,
                                 fleet_prediction=pred, clearance=avoid)
            if avoid:
                clear.append(info['clearance'].cpu().numpy())
            bm.advance(state)
            traj.append(state.cpu().numpy().copy())
        traj = np.stack(traj)
        pairs, dmin = set(), np.inf
        for s in traj:
            for w in range(worlds):
                P = [s[3 * w + i, :2] + body_V @ np.array([[np.cos(s[3 * w + i, 2]), np.sin(s[3 * w + i, 2])],
                                                           [-np.sin(s[3 * w + i, 2]), np.cos(s[3 * w + i, 2])]])
                     for i in range(3)]
                for i in range(3):
                    for j in range(i + 1, 3):
                        d = oc.polygons(P[i], P[j])
                        dmin = min(dmin, d)
                        if d < 0:
                            pairs.add((w, i, j))
        done = (traj[-1, 0::3, 0] > 4.0) & (traj[-1, 1::3, 1] > 4.0) & (traj[-1, 2::3, 0] < -6.0)
        rec = {'overlapping_pairs': len(pairs), 'pairs': 3 * worlds, 'worlds_with_overlap': len({p[0] for p in pairs}),
               'min_executed_signed_distance_m': float(dmin), 'worlds_all_past_crossing': int(done.sum())}
        if avoid:
            c = np.stack(clear)
            rec.update(plans=int(c.size), share_clearance_below_0=float((c < 0).mean()),
                       share_clearance_below_min_sd=float((c < min_sd).mean()), min_sd=min_sd)
        else:
            rec['clearance'] = 'not applicable: blind robots are given no obstacles'
        out[name] = rec
        del bm
    out['what'] = (f'{worlds} worlds of three robots (2 x 1 m diff-drive bodies, 2 m/s, T = 12, N = 3, 4 ADMM '
                   f'iterations, time-varying obstacles), {n_steps} closed-loop steps of 0.1 s, empty maps; a pair '
                   'overlaps when oracle.clearance.polygons < 0 at some executed step')
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('out_dir')
    ap.add_argument('--batches', default='256,4096,16384')
    ap.add_argument('--safety-worlds', type=int, default=64)
    ap.add_argument('--safety-steps', type=int, default=120)
    ap.add_argument('--skip', default='', help='comma-separated sections to skip: kernels, steps, safety')
    args = ap.parse_args()
    import torch
    from rda_planner_b200 import _cabi
    assert torch.cuda.is_available(), 'the probe measures the GPU; there is nothing to measure without one'
    dev = torch.device('cuda:0')
    lib = _cabi.load()
    gen = torch.Generator(device=dev)
    gen.manual_seed(5)
    rng = np.random.default_rng(5)
    skip = set(args.skip.split(','))
    out = {'gpu': gpu_identity(0), 'T': T, 'N': N, 'E': E}
    if 'kernels' not in skip:
        out['kernels'] = kernels(torch, lib, dev, [int(x) for x in args.batches.split(',')], gen, rng)
    if 'steps' not in skip:
        out['steps'] = steps(torch, dev, gen, rng)
    if 'safety' not in skip:
        out['safety'] = safety(torch, dev, args.safety_worlds, args.safety_steps)
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, 'fleet_plan_probe.json'), 'w') as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
