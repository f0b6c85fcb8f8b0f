"""Time obstacle_order='horizon' (rda_convert_world_obstacles_horizon) against the reference's key on the GPU.

For B robots in ONE shared world of M 2 x 1 m boxes along a 60 m line (N = 20, T = 30, E = 4, static and
time-varying output), the two conversions alternated in one run, CUDA events around many launches each; fleet rows
(worlds of 8 and 256 robots along their plans, 64 boxes per world); the share of shapes the kernel hands to the exact
key, counted by the CPU twin on a sample of robots; and one warm-started BatchedMPC step per B (50 iterations) on the
16 384-box map with each order (sections conversion, fleet, step).  Section study: closed loops that compare the two
orders at N = 4, 6 and 10 (the corridor map with clutter, and three-robot fleet crossings among clutter).  With
--parent TREE (a built checkout of the parent commit), section parity dumps the reference-key conversions' outputs on
seeded inputs from both trees and compares them bitwise, and section bench runs bench.py in both trees, alternated
twice, and compares their --dump-outputs.  Each call merges its sections into DIR/horizon_select_probe.json, with the
GPU's name, power limit and maximum SM clock read in the same call.

    python tools/horizon_select_probe.py DIR [--sections conversion,fleet,step,study,parity,bench]
                                             [--batches 256,4096,16384] [--maps 64,1024,16384] [--parent TREE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, '..')
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from world_obstacles_probe import boxes, event_ms  # noqa: E402

T, N, E, ITERS, DT = 30, 20, 4, 50, 0.1
STEP_MAP = 16384


def gpu_identity(index):
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader,nounits',
                        '-i', str(index)], capture_output=True, text=True, timeout=30).stdout.strip().split(',')
    return {'name': q[0].strip(), 'power_limit_w': float(q[1]), 'max_sm_clock_mhz': float(q[2])}


def poses(rng, B):
    """nom (3 m/s) and ref (4 m/s) along the 60 m line from random starts."""
    x0 = rng.uniform(0, 48, B)
    y0 = rng.normal(0, 0.3, B)
    t = np.arange(T + 1) * DT
    nom = np.stack([x0[:, None] + 3 * t, np.repeat(y0[:, None], T + 1, 1), np.zeros((B, T + 1))], 1)
    ref = np.stack([x0[:, None] + 4 * t, np.zeros((B, T + 1)), np.zeros((B, T + 1))], 1)
    return nom.astype(np.float32), ref.astype(np.float32)


def parity_dump(path):
    """The reference-key conversions (world, fleet, fleet along plans) on seeded inputs, saved to `path` (npz); runs
    with whichever rda_planner_b200 is first on sys.path."""
    import torch
    from rda_planner_b200.frontend import (convert_fleet_obstacles_batch, convert_world_obstacles_batch,
                                           fleet_plan_shapes_batch, fleet_shapes_batch, robot_body)
    from rda_planner_b200.scenarios import rectangle_robot
    dev = torch.device('cuda:0')
    rng = np.random.default_rng(12)
    B, W = 1024, 8
    world = {k: torch.as_tensor(v, device=dev) for k, v in boxes(rng, (W * 300,), 0.0, 60.0).items()}
    world['start'] = torch.arange(0, W * 300 + 1, 300, dtype=torch.int32, device=dev)
    state = torch.as_tensor(np.c_[rng.uniform(0, 60, B), rng.normal(0, 1, B), rng.uniform(-3, 3, B)],
                            dtype=torch.float32, device=dev)
    rw = torch.as_tensor(rng.integers(-1, W + 1, B), dtype=torch.int32, device=dev)
    cur_vel = torch.as_tensor(rng.uniform(-2, 2, (B, 2, T)), dtype=torch.float32, device=dev)
    body = robot_body(rectangle_robot())
    body['xy'] = torch.as_tensor(body['xy'], device=dev)
    out = {}
    for order in (0, 1):
        for tv in (False, True):
            out[f'world_{order}_{tv}'] = convert_world_obstacles_batch(world, state, rw, N, T, E, DT, tv, order)
            fleet = fleet_shapes_batch(state, cur_vel, body, 'acker')
            out[f'fleet_{order}_{tv}'] = convert_fleet_obstacles_batch(world, state, rw, fleet, N, T, E, DT, tv, order)
        plan = fleet_plan_shapes_batch(state, cur_vel, body, 'acker', DT, 3.0)
        out[f'plan_{order}'] = convert_fleet_obstacles_batch(world, state, rw, plan, N, T, E, DT, True, order, True)
    np.savez(path, **{f'{k}_{i}': t.cpu().numpy() for k, v in out.items() for i, t in enumerate(v)})


def _map_distance(ht, lst, states, body):
    """Signed distance of the body at each executed pose states [B,3] to every shape of the map `lst` (the CPU twin's
    exact key with the pose as its only column: plan_clearance_cell on each shape's rows).  Returns [B]."""
    out = np.empty(len(states))
    for b, st in enumerate(states):
        col = np.repeat(np.asarray(st, np.float32).reshape(3, 1), 2, 1)
        keys = ht.select(lst, 1, 1, E, DT, False, col, col, body)[4]
        out[b] = keys.min() if len(keys) else np.inf
    return out


def _box(x0, y0, x1, y1):
    from collections import namedtuple
    Obs = namedtuple('Obs', 'center radius vertex cone_type velocity')
    return Obs(None, None, np.array([[x0, x1, x1, x0], [y0, y0, y1, y1]], float), 'Rpositive', np.zeros((2, 1)))


def study(torch, dev, ht, Ns=(4, 6, 10), steps=200, seed=7):
    """Closed loops, reference key against 'horizon', at each N.
    corridor: 64 robots on the corridor (two 70 x 2 m walls 4 m either side of y = 20) with 1 x 1 m boxes inside it
    (off the centre line, which the robots must pass) and 2 x 2 m clutter outside it within 35 m, 140 shapes; T = 15,
    10 ADMM iterations, 4 m/s.  Contacts and the smallest executed signed distance are measured against the whole
    map at every executed pose.
    crossing: 32 worlds of three 2 x 1 m diff-drive robots (east, north, and one turning left across both lanes, as
    tools/fleet_plan_probe.py's safety section) among 40 boxes per world beside the lanes, avoid_fleet with the plan
    prediction, T = 12, 4 ADMM iterations, 2 m/s; robot-robot overlaps with oracle.clearance.polygons."""
    from oracle import clearance as oc
    from rda_planner_b200.frontend import BatchedMPC, pack_worlds, robot_body, shapes_to_device
    from rda_planner_b200.scenarios import rectangle_robot
    from fleet_plan_probe import _arc, _line
    rng = np.random.default_rng(seed)
    res = {'corridor': [], 'crossing': []}
    # ---- corridor ----
    inside = [_box(x, y, x + 1, y + 1) for x, y in zip(rng.uniform(8, 56, 14), rng.choice([17.2, 21.8], 14))]
    outside = [_box(x, y, x + 2, y + 2) for x, y in zip(rng.uniform(-5, 63, 124), rng.choice([-1, 1], 124) *
                                                        rng.uniform(7, 30, 124) + 20)]
    outside = [o for o in outside if o.vertex[1].max() < 13.5 or o.vertex[1].min() > 26.5]
    shapes = [_box(-5, 14, 65, 16), _box(-5, 24, 65, 26)] + inside + outside
    world_h = pack_worlds([shapes])
    lst = ht.robot_list(world_h, None, None, 0)
    world = shapes_to_device(world_h, dev)
    car = rectangle_robot()
    body = robot_body(car)
    B = 64
    path = np.stack([np.arange(0, 64, 0.1), np.full(640, 20.0), np.zeros(640)], 1)
    start = np.c_[rng.uniform(0, 6, B), 20 + rng.uniform(-1, 1, B), rng.uniform(-0.2, 0.2, B)].astype(np.float32)
    for n_obs in Ns:
        for order in (True, 'horizon'):
            bm = BatchedMPC(car, path, B, receding=15, sample_time=DT, iter_num=10, max_edge_num=E, max_obs_num=n_obs,
                            iter_threshold=0.0, device=dev, obstacle_order=order)
            min_sd = float(bm.rda.get_adjust_parameter()['min_sd'])
            st = torch.as_tensor(start, device=dev)
            clear, dist, ms = [], [], []
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for _ in range(steps):
                e0.record()
                _, info = bm.control(st, 4.0, world=world, clearance=True)
                bm.advance(st)
                e1.record()
                torch.cuda.synchronize(dev)
                ms.append(e0.elapsed_time(e1))
                clear.append(info['clearance'].cpu().numpy())
                dist.append(_map_distance(ht, lst, st.cpu().numpy(), body))
            c, d = np.stack(clear), np.stack(dist)
            res['corridor'].append({'N': n_obs, 'order': str(order), 'robots': B, 'steps': steps,
                                    'robot_steps_in_contact': int((d < 0).sum()), 'robots_ever_in_contact':
                                    int((d < 0).any(0).sum()), 'min_executed_signed_distance_m': float(d.min()),
                                    'share_plans_clearance_below_0': float((c < 0).mean()),
                                    'share_plans_clearance_below_min_sd': float((c < min_sd).mean()), 'min_sd': min_sd,
                                    'arrived': int(bm.arrive.sum()), 'median_step_ms': float(np.median(ms[5:]))})
            print(res['corridor'][-1], flush=True)
            del bm
    # ---- fleet crossing among clutter ----
    worlds = 32
    car = rectangle_robot(length=2.0, width=1.0, wheelbase=1.2, dynamics='diff', max_speed=(3, 1.5), max_acce=(3, 1.5))
    body_V = robot_body(car)['xy'][:4].astype(float)
    paths = [_line(-12.0, 0.0, 0.0, 200), _line(0.0, -12.0, np.pi / 2, 200),
             _arc(-8.0, -8.0, 10.0, 0.0, np.pi / 2) + _line(-8.25, 2.0, np.pi, 120)[1:]]
    lag = rng.uniform(0.0, 4.0, (worlds, 3))
    Bc = 3 * worlds
    robot_path = np.tile([0, 1, 2], worlds)
    robot_world = np.repeat(np.arange(worlds), 3).astype(np.int32)
    st0 = np.zeros(Bc, np.int64)
    st0[0::3] = np.round(lag[:, 0] / 0.25)
    st0[1::3] = np.round(lag[:, 1] / 0.25)
    state0 = np.array([np.asarray(paths[p][int(k)], float).reshape(-1)[:3] for p, k in zip(robot_path, st0)])
    state0[2::3, 1] -= lag[:, 2]
    clutter = []
    for _ in range(worlds):
        xy = rng.uniform(-14, 14, (200, 2))
        keep = [(x, y) for x, y in xy if min(abs(y), abs(x), abs(np.hypot(x + 8, y + 8) - 10)) > 3.0 and
                not (x < -6 and abs(y - 2) < 3)][:40]
        clutter.append([_box(x, y, x + 1, y + 1) for x, y in keep])
    cworld_h = pack_worlds(clutter)
    cworld = shapes_to_device(cworld_h, dev)
    cbody = robot_body(car)
    for n_obs in Ns:
        for order in (True, 'horizon'):
            bm = BatchedMPC(car, paths, Bc, robot_path=robot_path, receding=12, sample_time=DT, iter_num=4,
                            max_edge_num=E, max_obs_num=n_obs, iter_threshold=0.0, device=dev, obstacle_order=order)
            bm.cur_index[:] = torch.as_tensor(st0, dtype=torch.int32)
            min_sd = float(bm.rda.get_adjust_parameter()['min_sd'])
            st = torch.as_tensor(state0, dtype=torch.float32, device=dev)
            rw = torch.as_tensor(robot_world, device=dev)
            traj, clear, ms = [], [], []
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for _ in range(120):
                e0.record()
                _, info = bm.control(st, 2.0, time_varying=True, world=cworld, robot_world=rw, avoid_fleet=True,
                                     fleet_prediction='plan', clearance=True)
                bm.advance(st)
                e1.record()
                torch.cuda.synchronize(dev)
                ms.append(e0.elapsed_time(e1))
                clear.append(info['clearance'].cpu().numpy())
                traj.append(st.cpu().numpy().copy())
            traj, c = np.stack(traj), np.stack(clear)
            pairs, dmin = set(), np.inf
            for s in traj[::2]:
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
            md = np.stack([np.array([_map_distance(ht, ht.robot_list(cworld_h, None, robot_world, b), s[b:b + 1],
                                                   cbody)[0] for b in range(Bc)]) for s in traj[::4]])
            done = (traj[-1, 0::3, 0] > 4.0) & (traj[-1, 1::3, 1] > 4.0) & (traj[-1, 2::3, 0] < -6.0)
            res['crossing'].append({'N': n_obs, 'order': str(order), 'worlds': worlds, 'steps': 120,
                                    'overlapping_robot_pairs': len(pairs), 'pairs': 3 * worlds,
                                    'min_robot_robot_signed_distance_m': float(dmin),
                                    'robot_map_contacts_every_4th_step': int((md < 0).sum()),
                                    'min_robot_map_signed_distance_m': float(md.min()),
                                    'share_plans_clearance_below_0': float((c < 0).mean()),
                                    'share_plans_clearance_below_min_sd': float((c < min_sd).mean()), 'min_sd': min_sd,
                                    'worlds_all_past_crossing': int(done.sum()), 'median_step_ms': float(np.median(ms[5:]))})
            print(res['crossing'][-1], flush=True)
            del bm
    res['what'] = study.__doc__
    return res


def bench(parent, out_dir):
    """bench.py --no-cpu-baseline --no-probes --dump-outputs in this tree and in `parent`, alternated twice; the
    solves/s of each run, and u, s, status, iters of the dumps compared bitwise (the dumps are deleted after)."""
    import shutil
    runs, cmp = [], {}
    dumps = {who: os.path.abspath(os.path.join(out_dir, f'bench_dump_{who}')) for who in ('change', 'parent')}
    for i in range(2):
        for who, tree in (('change', ROOT), ('parent', parent)):
            r = subprocess.run([sys.executable, 'bench.py', '--gpus', '1', '--steps', '5', '--warmup', '3',
                                '--no-cpu-baseline', '--no-probes', '--dump-outputs', dumps[who]],
                               cwd=os.path.abspath(tree), capture_output=True, text=True, check=True)
            res = json.loads(r.stdout.strip().splitlines()[-1])
            runs.append({'tree': who, 'run': i, 'solves_per_s': res['value'], 'ms_per_step': res['ms_per_step']})
            print(runs[-1], flush=True)
    for k in ('u', 's', 'status', 'iters'):
        a, b = np.load(os.path.join(dumps['change'], k + '.npy')), np.load(os.path.join(dumps['parent'], k + '.npy'))
        cmp[k] = 'bitwise equal' if np.array_equal(a, b) else f'differ: max {float(np.abs(a - b).max())}'
    for d in dumps.values():
        shutil.rmtree(d)
    return {'runs': runs, 'dump_outputs': cmp, 'what': bench.__doc__}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('out_dir')
    ap.add_argument('--sections', default='conversion,fleet,step,study')
    ap.add_argument('--batches', default='256,4096,16384')
    ap.add_argument('--maps', default='64,1024,16384')
    ap.add_argument('--parent', help='a built checkout of the parent commit (sections parity and bench)')
    ap.add_argument('--dump', help=argparse.SUPPRESS)
    ap.add_argument('--root', help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.dump:
        if args.root:                                     # the parent's package instead of this tree's
            sys.path.insert(0, args.root)
        return parity_dump(args.dump)
    import torch
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import horizon_twin as ht
    from rda_planner_b200.frontend import (BatchedMPC, convert_fleet_obstacles_batch, convert_world_obstacles_batch,
                                           convert_world_obstacles_horizon_batch, fleet_plan_shapes_batch, robot_body)
    from rda_planner_b200.scenarios import rectangle_robot
    assert torch.cuda.is_available(), 'the probe measures the GPU; there is nothing to measure without one'
    sections = set(args.sections.split(','))
    if sections & {'parity', 'bench'} and not args.parent:
        ap.error('sections parity and bench need --parent')
    dev = torch.device('cuda:0')
    os.makedirs(args.out_dir, exist_ok=True)
    path_json = os.path.join(args.out_dir, 'horizon_select_probe.json')
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
    if 'study' in sections:
        out['study'] = study(torch, dev, ht)
    rng = np.random.default_rng(5)
    body = robot_body(rectangle_robot())
    dbody = dict(body, xy=torch.as_tensor(body['xy'], device=dev))
    worlds, hosts = {}, {}
    for M in [int(x) for x in args.maps.split(',')]:
        hosts[M] = dict(boxes(rng, (M,), 0.0, 60.0), start=np.array([0, M], np.int32))
        worlds[M] = {k: torch.as_tensor(v, device=dev) for k, v in hosts[M].items()}
    for key in ('conversion', 'fleet', 'control_step'):
        if key.split('_')[-1] in sections or key in sections:
            out[key] = []
    for B in [int(x) for x in args.batches.split(',')] if sections & {'conversion', 'fleet', 'step'} else []:
        nom, ref = poses(rng, B)
        dnom, dref = torch.as_tensor(nom, device=dev), torch.as_tensor(ref, device=dev)
        state = dnom[:, :, 0].contiguous()
        for M, w in worlds.items() if 'conversion' in sections else ():
            for tv in (False, True):
                old = lambda: convert_world_obstacles_batch(w, state, None, N, T, E, DT, tv, True)
                new = lambda: convert_world_obstacles_horizon_batch(w, dnom, dref, dbody, None, N, T, E, DT, tv)
                times = {'reference_key_ms': [], 'horizon_ms': []}
                for _ in range(2):                                  # alternated
                    times['reference_key_ms'].append(event_ms(old, dev)[0])
                    times['horizon_ms'].append(event_ms(new, dev)[0])
                lst = ht.robot_list(hosts[M], None, None, 0)
                share = np.mean([ht.exact_count(lst, N, T, E, DT, tv, nom[b], ref[b], body) / M
                                 for b in rng.integers(0, B, 8)])
                out['conversion'].append(dict(B=B, M=M, time_varying=tv, exact_key_share=float(share), **times))
                print(out['conversion'][-1], flush=True)
        # fleet rows: worlds of R robots along their plans, 64 boxes per world
        for R in (8, 256) if 'fleet' in sections else ():
            W = B // R
            fw = {k: torch.as_tensor(v, device=dev) for k, v in boxes(rng, (W * 64,), 0.0, 60.0).items()}
            fw['start'] = torch.arange(0, W * 64 + 1, 64, dtype=torch.int32, device=dev)
            rw = torch.arange(B, dtype=torch.int32, device=dev) // R
            cur_vel = torch.full((B, 2, T), 3.0, device=dev)
            cur_vel[:, 1] = 0.0
            plan = fleet_plan_shapes_batch(state, cur_vel, dbody, 'acker', DT, 3.0)
            old = lambda: convert_fleet_obstacles_batch(fw, state, rw, plan, N, T, E, DT, True, True, True)
            new = lambda: convert_world_obstacles_horizon_batch(fw, dnom, dref, dbody, rw, N, T, E, DT, True, plan, True)
            times = {'reference_key_ms': [], 'horizon_ms': []}
            for _ in range(2):
                times['reference_key_ms'].append(event_ms(old, dev)[0])
                times['horizon_ms'].append(event_ms(new, dev)[0])
            out['fleet'].append(dict(B=B, robots_per_world=R, boxes_per_world=64, prediction='plan', **times))
            print(out['fleet'][-1], flush=True)
        if 'step' in sections and STEP_MAP in worlds:
            path = np.stack([np.arange(0, 80, 0.1), np.zeros(800), np.zeros(800)], 1)
            for order in (True, 'horizon'):
                bm = BatchedMPC(rectangle_robot(), path, B, receding=T, sample_time=DT, iter_num=ITERS, max_edge_num=E,
                                max_obs_num=N, iter_threshold=0.0, device=dev, obstacle_order=order)
                bm.cur_index[:] = torch.as_tensor(np.maximum((nom[:, 0, 0] * 10).astype(int) - 3, 0), dtype=torch.int32)
                bm.cur_vel[:, 0, :] = 3.0
                st = state.clone()

                def step():
                    bm.control(st, 3.0, world=worlds[STEP_MAP])
                    bm.advance(st)
                ms, reps = event_ms(step, dev, min_window_s=1.0)
                # what the solve was given: the conversion alone at the step's poses, and how close the kept obstacles
                # are to the nominal poses (plan_clearance per slot, smallest over t)
                _, info = bm.control(st, 3.0, world=worlds[STEP_MAP])
                wm = worlds[STEP_MAP]
                if order is True:
                    conv = lambda: convert_world_obstacles_batch(wm, st, None, N, T, E, DT, False, True)
                else:
                    conv = lambda: convert_world_obstacles_horizon_batch(wm, info['nom_s'], info['ref_s'], dbody, None,
                                                                         N, T, E, DT, False)
                conv_ms = event_ms(conv, dev)[0]
                slot = bm.rda.plan_clearance(s=info['nom_s'], per_cell=True)['map'].amin(2).cpu().numpy()
                out['control_step'].append({'B': B, 'M': STEP_MAP, 'order': str(order), 'ms': ms, 'steps': reps,
                                            'conversion_ms': conv_ms, 'rest_of_step_ms': ms - conv_ms,
                                            'kept_slots_overlapping_nom_per_robot': float((slot < 0).sum(1).mean()),
                                            'kept_slots_within_1m_of_nom_per_robot': float((slot < 1).sum(1).mean())})
                print(out['control_step'][-1], flush=True)
                del bm
    out['what'] = ('conversion / fleet: one launch of each conversion, CUDA events, the two alternated twice; '
                   'exact_key_share: shapes given the exact key over M, CPU twin of the kernel scan on 8 robots; '
                   'control_step: BatchedMPC.control(world=...) + advance, warm-started, 50 iterations, each order, '
                   'with the conversion timed alone at the step\'s poses and the kept slots\' clearance at nom_s; '
                   'study, parity, bench: see their own "what"; calls: the GPU identity of each call and its sections')
    with open(path_json, 'w') as f:
        json.dump(out, f, indent=1)
    print(json.dumps({k: v for k, v in out.items() if k in ('calls', 'parent_parity')}))


if __name__ == '__main__':
    main()
