"""Measure world shapes along given trajectories (rda_convert_world_obstacles_traj / _horizon_traj) on the GPU.

Section conversion: B robots in ONE map of M 2 x 1 m boxes along a 60 m line (T = 30, N = 20, E = 4, time-varying),
a share of the boxes on trajectories, timed against the same map where those boxes move at a constant velocity with the
same stage 0 (the trajectories are that straight-line motion), the two alternated twice in one run, CUDA events, the
faster window of each; reference key and horizon order.  Section step: one warm-started BatchedMPC step (control +
advance, 50 ADMM iterations) at B = 16 384 both ways, alternated, medians.  Section study: a closed loop of robots that
cross pedestrians who walk arcs and stop, planned once against their true trajectories (updated in place each step)
and once against their current velocity; executed overlaps and the smallest executed signed distance.  With --parent
TREE (a built checkout of the parent commit), section parity dumps the existing world, fleet and horizon conversions'
outputs on seeded inputs from both trees and compares them bitwise, and section bench runs bench.py in both trees
(horizon_select_probe.bench).  Writes DIR/world_traj_probe.json with the GPU's name, power limit and maximum SM clock
read in the same call.

    python tools/world_traj_probe.py DIR [--sections conversion,step,study,parity,bench] [--parent TREE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, '..')
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from world_obstacles_probe import boxes  # noqa: E402
from horizon_select_probe import bench, gpu_identity, poses  # noqa: E402

T, N, E, DT = 30, 20, 4, 0.1


def traj_pair(rng, M, share):
    """(velocity map, trajectory map) host dicts: the same boxes, the first share * M of them moving; in the trajectory
    map those are on trajectories of the same straight-line motion (stage 0 the box, stage t moved by vel * t * dt)."""
    vel_map = dict(boxes(rng, (M,), 0.0, 60.0), start=np.array([0, M], np.int32))
    k = int(round(share * M))
    vel_map['vel'][:k] = rng.uniform(-1.5, 1.5, (k, 2)).astype(np.float32)
    traj_map = {key: v.copy() for key, v in vel_map.items()}
    if k:
        t = (np.arange(T + 1) * np.float32(DT)).astype(np.float32)
        off = vel_map['vel'][:k, None, :] * t[None, :, None]                           # [k, T+1, 2]
        txy = vel_map['xy'][:k, None, :, :] + off[:, :, None, :]
        txy[:, :, 4:] = 0
        traj_map['traj_xy'] = txy.astype(np.float32)
        traj_map['traj'] = np.full(M, -1, np.int32)
        traj_map['traj'][:k] = np.arange(k)
        traj_map['vel'][:k] = 0
    return vel_map, traj_map


def timed(fn, dev, window_s=0.3):
    """Time per call of fn() over a window of back-to-back calls (CUDA events), after one warm-up call."""
    import torch
    fn()
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize(dev)
    reps = int(min(200, max(1, window_s / max(e0.elapsed_time(e1) * 1e-3, 1e-6))))
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize(dev)
    return e0.elapsed_time(e1) / reps


def conversion(torch, dev, batches, maps, shares):
    from rda_planner_b200.frontend import convert_world_obstacles_batch, convert_world_obstacles_horizon_batch, \
        robot_body
    from rda_planner_b200.scenarios import rectangle_robot
    rng = np.random.default_rng(5)
    body = robot_body(rectangle_robot())
    dbody = dict(body, xy=torch.as_tensor(body['xy'], device=dev))
    rows = []
    for M in maps:
        for share in shares:
            pair = [{k: torch.as_tensor(v, device=dev) for k, v in m.items()} for m in traj_pair(rng, M, share)]
            for B in batches:
                nom, ref = (torch.as_tensor(a, device=dev) for a in poses(rng, B))
                state = nom[:, :, 0].contiguous()
                calls = {
                    'reference_key': [lambda w=w: convert_world_obstacles_batch(w, state, None, N, T, E, DT, True, True)
                                      for w in pair],
                    'horizon': [lambda w=w: convert_world_obstacles_horizon_batch(w, nom, ref, dbody, None, N, T, E, DT,
                                                                                  True) for w in pair]}
                for order, (f_vel, f_traj) in calls.items():
                    t_vel, t_traj = [], []
                    for _ in range(2):
                        t_vel.append(timed(f_vel, dev))
                        t_traj.append(timed(f_traj, dev))
                    a, b = f_vel(), f_traj()
                    same_kind = bool(torch.equal(a[2], b[2]) and torch.equal(a[3], b[3]))
                    rows.append({'B': B, 'M': M, 'share': share, 'order': order, 'velocity_ms': min(t_vel),
                                 'trajectory_ms': min(t_traj), 'same_obs_kind_and_count': same_kind,
                                 'max_row_gap': float(max((a[0] - b[0]).abs().max(), (a[1] - b[1]).abs().max()))})
                    print(rows[-1], flush=True)
    return rows


def step(torch, dev, B=16384, M=1024, share=0.25, reps=3):
    from rda_planner_b200.frontend import BatchedMPC
    from rda_planner_b200.scenarios import rectangle_robot
    rng = np.random.default_rng(9)
    path = [np.array([[x], [0.0], [0.0]]) for x in np.arange(0, 70, 0.5)]
    pair = [{k: torch.as_tensor(v, device=dev) for k, v in m.items()} for m in traj_pair(rng, M, share)]
    state0 = torch.as_tensor(np.c_[rng.uniform(0, 45, B), rng.normal(0, 0.3, B), np.zeros(B)], dtype=torch.float32,
                             device=dev)
    out = {'B': B, 'M': M, 'share': share, 'iterations': 50}
    for order in (True, 'horizon'):
        bms = [BatchedMPC(rectangle_robot(), path, B, receding=T, iter_num=50, iter_threshold=0.0, max_edge_num=E,
                          max_obs_num=N, obstacle_order=order) for _ in pair]
        states = [state0.clone() for _ in pair]
        times = [[], []]
        for i in range(reps + 1):
            for j, (bm, st, w) in enumerate(zip(bms, states, pair)):
                torch.cuda.synchronize(dev)
                t0 = time.perf_counter()
                bm.control(st, 3.0, world=w, time_varying=True)
                bm.advance(st)
                torch.cuda.synchronize(dev)
                if i:
                    times[j].append((time.perf_counter() - t0) * 1e3)
        out['reference_key' if order is True else 'horizon'] = {'velocity_ms': float(np.median(times[0])),
                                                                'trajectory_ms': float(np.median(times[1]))}
        print(order, out, flush=True)
    return out


def _ped(p0, th0, v, w, stop, t):
    """Position and velocity at time t of a pedestrian walking an arc (speed v, turn rate w) who stops at `stop`."""
    s = np.minimum(t, stop)
    if abs(w) < 1e-9:
        pos = p0 + v * s * np.array([np.cos(th0), np.sin(th0)])
    else:
        pos = p0 + v / w * np.array([np.sin(th0 + w * s) - np.sin(th0), np.cos(th0) - np.cos(th0 + w * s)])
    th = th0 + w * s
    vel = (v * np.array([np.cos(th), np.sin(th)])) if t < stop else np.zeros(2)
    return pos, vel


def study(torch, dev, B=64, P=3, steps=100, Tq=12, Nq=3, seed=3):
    """Robot b drives east along y = 0 at 2 m/s in its own world of P pedestrians (discs of 0.3 m) that start 3-5 m
    beside the lane, walk towards it on arcs at 1-1.5 m/s and stop after 1.5-4.5 s, some of them in the lane."""
    from oracle import clearance
    from rda_planner_b200.frontend import BatchedMPC, robot_body
    from rda_planner_b200.scenarios import rectangle_robot
    rng = np.random.default_rng(seed)
    car = rectangle_robot(length=2.0, width=1.0, wheelbase=1.2, dynamics='diff', max_speed=(3, 1.5), max_acce=(3, 1.5))
    body = robot_body(car)
    ob = {'disc': False, 'V': body['xy'][:body['nv']].astype(float)}
    path = [np.array([[x], [0.0], [0.0]]) for x in np.arange(-5, 60, 0.25)]
    side = rng.choice([-1.0, 1.0], (B, P))
    peds = [dict(p0=np.array([rng.uniform(4, 16), side[b, i] * rng.uniform(3, 5)]), th0=-side[b, i] * np.pi / 2
                 + rng.uniform(-0.4, 0.4), v=rng.uniform(1.0, 1.5), w=rng.uniform(-0.4, 0.4), stop=rng.uniform(1.5, 4.5))
            for b in range(B) for i in range(P)]
    S = B * P
    res = {}
    for mode in ('trajectory', 'velocity'):
        bm = BatchedMPC(car, path, B, receding=Tq, sample_time=DT, iter_num=4, max_edge_num=4, max_obs_num=Nq,
                        iter_threshold=0.0)
        state = torch.as_tensor(np.c_[np.zeros(B), np.zeros(B), np.zeros(B)], dtype=torch.float32, device=dev)
        world = {'kind': torch.ones(S, dtype=torch.int32, device=dev), 'nv': torch.zeros(S, dtype=torch.int32,
                                                                                           device=dev),
                 'xy': torch.zeros((S, 8, 2), device=dev), 'radius': torch.full((S,), 0.3, device=dev),
                 'vel': torch.zeros((S, 2), device=dev),
                 'start': torch.arange(0, S + 1, P, dtype=torch.int32, device=dev)}
        if mode == 'trajectory':
            world['traj'] = torch.arange(S, dtype=torch.int32, device=dev)
            world['traj_xy'] = torch.zeros((S, Tq + 1, 8, 2), device=dev)
        rw = torch.arange(B, dtype=torch.int32, device=dev)
        overlaps, dmin, step_ms = 0, np.inf, []
        for k in range(steps):
            now = k * DT
            xy = np.zeros((S, 8, 2), np.float32)
            vel = np.zeros((S, 2), np.float32)
            txy = np.zeros((S, Tq + 1, 8, 2), np.float32)
            for j, p in enumerate(peds):
                pos, v = _ped(p['p0'], p['th0'], p['v'], p['w'], p['stop'], now)
                xy[j, 0], vel[j] = pos, v
                if mode == 'trajectory':
                    for t in range(Tq + 1):
                        txy[j, t, 0] = _ped(p['p0'], p['th0'], p['v'], p['w'], p['stop'], now + t * DT)[0]
            if mode == 'trajectory':
                world['xy'].copy_(torch.as_tensor(xy))
                world['traj_xy'].copy_(torch.as_tensor(txy))          # the predictor's output, in place
            else:
                world['xy'].copy_(torch.as_tensor(xy))
                world['vel'].copy_(torch.as_tensor(vel))
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            bm.control(state, 2.0, world=world, robot_world=rw, time_varying=True)
            bm.advance(state)
            torch.cuda.synchronize(dev)
            step_ms.append((time.perf_counter() - t0) * 1e3)
            s = state.cpu().numpy().astype(float)
            for b in range(B):
                for i in range(P):
                    pos = _ped(**peds[b * P + i], t=now + DT)[0]
                    d = clearance.cell(ob, s[b], 1, np.array([[1, 0], [0, 1], [0, 0]], float),
                                       np.array([pos[0], pos[1], -0.3]))
                    dmin = min(dmin, d)
                    overlaps += int(d < 0)
        res[mode] = {'robot_pedestrian_steps_overlapping': overlaps, 'of': B * P * steps,
                     'smallest_executed_sd_m': float(dmin), 'median_step_ms': float(np.median(step_ms)),
                     'mean_final_x_m': float(state[:, 0].mean())}
        print(mode, res[mode], flush=True)
    res['what'] = study.__doc__
    return res


def parity_dump(path):
    """The existing world, fleet, fleet-plan and horizon conversions (with and without ids) on seeded inputs, saved to
    `path` (npz); runs with whichever rda_planner_b200 is first on sys.path."""
    import torch
    from rda_planner_b200.frontend import (convert_fleet_obstacles_batch, convert_world_obstacles_batch,
                                           convert_world_obstacles_horizon_batch, fleet_plan_shapes_batch,
                                           fleet_shapes_batch, robot_body)
    from rda_planner_b200.scenarios import rectangle_robot
    dev = torch.device('cuda:0')
    rng = np.random.default_rng(21)
    B, W = 512, 4
    world = {k: torch.as_tensor(v, device=dev) for k, v in boxes(rng, (W * 200,), 0.0, 60.0).items()}
    world['vel'][::3] = torch.as_tensor(rng.uniform(-1, 1, (len(world['vel'][::3]), 2)), dtype=torch.float32,
                                        device=dev)
    world['start'] = torch.arange(0, W * 200 + 1, 200, dtype=torch.int32, device=dev)
    state = torch.as_tensor(np.c_[rng.uniform(0, 60, B), rng.normal(0, 1, B), rng.uniform(-3, 3, B)],
                            dtype=torch.float32, device=dev)
    rw = torch.as_tensor(rng.integers(-1, W + 1, B), dtype=torch.int32, device=dev)
    cur_vel = torch.as_tensor(rng.uniform(-2, 2, (B, 2, T)), dtype=torch.float32, device=dev)
    nom, ref = (torch.as_tensor(a, device=dev) for a in poses(rng, B))
    body = robot_body(rectangle_robot())
    body['xy'] = torch.as_tensor(body['xy'], device=dev)
    fleet = fleet_shapes_batch(state, cur_vel, body, 'acker')
    plan = fleet_plan_shapes_batch(state, cur_vel, body, 'acker', DT, 3.0)
    out = {}
    for ids in (False, True):
        for order in (0, 1):
            for tv in (False, True):
                out[f'world_{ids}_{order}_{tv}'] = convert_world_obstacles_batch(world, state, rw, N, T, E, DT, tv,
                                                                                 order, ids)
                out[f'fleet_{ids}_{order}_{tv}'] = convert_fleet_obstacles_batch(world, state, rw, fleet, N, T, E, DT,
                                                                                 tv, order, False, ids)
            out[f'plan_{ids}_{order}'] = convert_fleet_obstacles_batch(world, state, rw, plan, N, T, E, DT, True, order,
                                                                       True, ids)
        for tv in (False, True):
            out[f'hor_{ids}_{tv}'] = convert_world_obstacles_horizon_batch(world, nom, ref, body, rw, N, T, E, DT, tv,
                                                                           ids=ids)
            out[f'hor_fleet_{ids}_{tv}'] = convert_world_obstacles_horizon_batch(world, nom, ref, body, rw, N, T, E,
                                                                                 DT, tv, fleet, ids=ids)
        out[f'hor_plan_{ids}'] = convert_world_obstacles_horizon_batch(world, nom, ref, body, rw, N, T, E, DT, True,
                                                                       plan, True, ids=ids)
    np.savez(path, **{f'{k}_{i}': t.cpu().numpy() for k, v in out.items() for i, t in enumerate(v)})


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('out_dir')
    ap.add_argument('--sections', default='conversion,step,study')
    ap.add_argument('--batches', default='256,4096,16384')
    ap.add_argument('--maps', default='1024,16384')
    ap.add_argument('--shares', default='0,0.25,1')
    ap.add_argument('--parent', help='a built checkout of the parent commit (sections parity and bench)')
    ap.add_argument('--dump', help=argparse.SUPPRESS)
    ap.add_argument('--root', help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.dump:
        if args.root:                                     # the parent's package instead of this tree's
            sys.path.insert(0, args.root)
        return parity_dump(args.dump)
    import torch
    assert torch.cuda.is_available(), 'the probe measures the GPU; there is nothing to measure without one'
    sections = set(args.sections.split(','))
    if sections & {'parity', 'bench'} and not args.parent:
        ap.error('sections parity and bench need --parent')
    dev = torch.device('cuda:0')
    os.makedirs(args.out_dir, exist_ok=True)
    path_json = os.path.join(args.out_dir, 'world_traj_probe.json')
    out = json.load(open(path_json)) if os.path.exists(path_json) else {}
    out.setdefault('calls', []).append({'gpu': gpu_identity(0), 'sections': sorted(sections)})
    out.update(N=N, E=E, T=T)
    if 'parity' in sections:
        mine, theirs = os.path.join(args.out_dir, 'parity_new.npz'), os.path.join(args.out_dir, 'parity_parent.npz')
        me = os.path.abspath(__file__)
        subprocess.check_call([sys.executable, me, args.out_dir, '--dump', os.path.abspath(mine)], cwd=ROOT)
        subprocess.check_call([sys.executable, me, args.out_dir, '--dump', os.path.abspath(theirs), '--root',
                               os.path.abspath(args.parent)], cwd=os.path.abspath(args.parent))
        a, b = np.load(mine), np.load(theirs)
        out['parent_parity'] = {'arrays': len(a.files), 'bitwise_equal': all(np.array_equal(a[k], b[k]) for k in a.files)
                                and sorted(a.files) == sorted(b.files)}
        os.remove(mine)
        os.remove(theirs)
        print(out['parent_parity'], flush=True)
    if 'bench' in sections:
        out['bench'] = bench(args.parent, args.out_dir)
    if 'conversion' in sections:
        out['conversion'] = conversion(torch, dev, [int(x) for x in args.batches.split(',')],
                                       [int(x) for x in args.maps.split(',')], [float(x) for x in args.shares.split(',')])
    if 'step' in sections:
        out['step'] = step(torch, dev)
    if 'study' in sections:
        out['study'] = study(torch, dev)
    json.dump(out, open(path_json, 'w'), indent=1)
    print(json.dumps({k: v for k, v in out.items() if k in ('calls', 'parent_parity')}))


if __name__ == '__main__':
    main()
