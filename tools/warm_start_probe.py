"""Measure the warm start that follows the obstacles (BatchedMPC(warm_start='obstacle'), rda_set_obstacle_ids) against
the reference's slot behaviour on the GPU.

  remap     CUDA events over back-to-back rda_set_obstacle_ids calls that move every instance's slots (two id sets
            that are permutations of each other, alternated) at B = 16 384, T = 30, N = 20, E = 4 and at config E's
            shape (B = 8 192 on one GPU, T = 40, N = 128, E = 8), next to a solve of one ADMM iteration (rda_solve with
            iter_num = 1: begin, one iteration, finish) of the same handle.
  loops     closed loops with 'slot' and 'obstacle' alternated step by step in one session, on two scenes:
              world     bench.py's closed_loop scene as one shared world: robots on a 60 m line among 2 x 1 m boxes
                        (a map of 1 024 boxes), obstacle_order=True, N = 20, T = 30;
              crossing  the fleet crossing of tools/fleet_plan_probe.py: three robots per world crossing each other,
                        avoid_fleet with fleet_prediction='plan', N = 3, T = 12, empty maps.
            With iter_num = 50 and iter_threshold = 0.2: the mean ADMM iterations per step, the mean over steps of the
            slowest robot's iterations (a step lasts until its slowest robot stops) and the step time (CUDA events).  With iter_num = 4 and no early stop: the mean resi_pri / resi_dual, the smallest plan clearance
            (rda_plan_clearance over each solved plan) and the number of plans whose clearance is below 0; the
            smallest executed signed distance (the pose each step was planned from, against the obstacles that step
            was given) and the number of executed poses closer than 0 (contacts).  Churn: the share of slots whose obstacle id differs from the last step's (ids of
            the 'obstacle' run).

Writes OUT/warm_start_probe.json with the GPU's name and power limit read in the same run.

    python tools/warm_start_probe.py OUT [--steps 60] [--robots 1024] [--worlds 64] [--only-remap]

The same study at small B on the CPU with the float64 oracle: tools/warm_start_cpu_study.py.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from fleet_plan_probe import _arc, _line  # noqa: E402
from world_obstacles_probe import event_ms, gpu_identity  # noqa: E402


def remap(torch, dev, B=16384, T=30, N=20, E=4):
    from rda_planner_b200.rda_solver import RDA_solver
    from rda_planner_b200.scenarios import make_instance, rectangle_robot
    from rda_planner_b200.rda_solver import pack_obstacles
    U = 64
    insts = [make_instance(9000 + i, T=T, N=N, E=E) for i in range(U)]
    packs = [pack_obstacles(list(i['obstacles']), T, N, E) for i in insts]
    pick = np.arange(B) % U
    t = lambda a: torch.as_tensor(np.asarray(a)[pick], device=dev).contiguous()
    inp = dict(nom_s=t(np.stack([i['nom_s'] for i in insts]).astype(np.float32)),
               nom_u=t(np.stack([i['nom_u'] for i in insts]).astype(np.float32)),
               ref_s=t(np.stack([i['ref'] for i in insts]).astype(np.float32)),
               ref_speed=t(np.array([i['ref_speed'] for i in insts], np.float32)),
               obs_A=t(np.stack([p[0] for p in packs])), obs_b=t(np.stack([p[1] for p in packs])),
               obs_kind=t(np.stack([p[2] for p in packs])), obs_count=t(np.array([p[3] for p in packs], np.int32)))
    g = RDA_solver(T, rectangle_robot(), max_edge_num=E, max_obs_num=N, iter_num=1, iter_threshold=0.0,
                   time_print=False, batch=B, device=dev)
    g.iterative_solve_batch(**inp)
    rng = np.random.default_rng(0)
    ids = [torch.as_tensor(np.stack([rng.permutation(N) for _ in range(B)]).astype(np.int32), device=dev)
           for _ in range(2)]
    g.set_obstacle_ids(ids[0])
    k = [0]

    def move():
        k[0] ^= 1
        g.set_obstacle_ids(ids[k[0]])
    return {'shape': {'B': B, 'T': T, 'N': N, 'E': E}, 'remap_ms': event_ms(move, dev),
            'solve_one_iteration_ms': event_ms(lambda: g.iterative_solve_batch(**inp), dev),
            'what': 'rda_set_obstacle_ids moving every slot of every instance, against rda_solve with iter_num = 1'}


def world_scene(torch, dev, robots, rng):
    from rda_planner_b200.frontend import pack_worlds, shapes_to_device
    from collections import namedtuple
    Obs = namedtuple('Obs', 'cone_type center radius vertex velocity')
    path = np.stack([np.arange(0, 60, 0.1), np.zeros(600), np.zeros(600)], 1)
    corners = np.array([[-1, -0.5], [1, -0.5], [1, 0.5], [-1, 0.5]])
    boxes = []
    for _ in range(1024):
        c = np.array([rng.uniform(0, 64), rng.uniform(1.8, 6) * rng.choice([-1, 1])])
        y = rng.uniform(0, np.pi)
        R = np.array([[np.cos(y), -np.sin(y)], [np.sin(y), np.cos(y)]])
        boxes.append(Obs('Rpositive', None, None, (c[:, None] + R @ corners.T), np.zeros(2)))
    world = shapes_to_device(pack_worlds([boxes]), dev)
    idx = rng.integers(0, 480, robots)
    state0 = path[idx] + rng.normal(0, [0.3, 0.3, 0.1], (robots, 3))
    return dict(path=path, world=world, state0=state0, start=np.maximum(idx - 3, 0), speed=4.0,
                mpc=dict(receding=30, max_obs_num=20, max_edge_num=4, sample_time=0.1),
                control=dict(world=world))


def crossing_scene(torch, dev, worlds, rng):
    from rda_planner_b200.frontend import pack_worlds, shapes_to_device
    paths = [_line(-12.0, 0.0, 0.0, 200), _line(0.0, -12.0, np.pi / 2, 200),
             _arc(-8.0, -8.0, 10.0, 0.0, np.pi / 2) + _line(-8.25, 2.0, np.pi, 120)[1:]]
    lag = rng.uniform(0.0, 4.0, (worlds, 3))
    B = 3 * worlds
    robot_path = np.tile([0, 1, 2], worlds)
    start = np.zeros(B, np.int64)
    start[0::3] = np.round(lag[:, 0] / 0.25)
    start[1::3] = np.round(lag[:, 1] / 0.25)
    state0 = np.array([np.asarray(paths[p][int(s)], float).reshape(-1)[:3] for p, s in zip(robot_path, start)])
    state0[2::3, 1] -= lag[:, 2]
    world = shapes_to_device(pack_worlds([[] for _ in range(worlds)]), dev)
    rw = torch.as_tensor(np.repeat(np.arange(worlds), 3).astype(np.int32), device=dev)
    return dict(path=paths, robot_path=robot_path, state0=state0, start=start, speed=2.0,
                mpc=dict(receding=12, max_obs_num=3, max_edge_num=4, sample_time=0.1),
                control=dict(world=world, robot_world=rw, avoid_fleet=True, fleet_prediction='plan', time_varying=True))


def loops(torch, dev, scene, steps, iter_num, thr):
    """The scene's closed loop with 'slot' and 'obstacle' stepped alternately (one fleet each)."""
    from rda_planner_b200.frontend import BatchedMPC
    from rda_planner_b200.scenarios import rectangle_robot
    car = rectangle_robot() if 'robot_path' not in scene else \
        rectangle_robot(length=2.0, width=1.0, wheelbase=1.2, dynamics='diff', max_speed=(3, 1.5), max_acce=(3, 1.5))
    B = len(scene['state0'])
    run = {}
    for mode in ('slot', 'obstacle'):
        kw = dict(robot_path=scene['robot_path']) if 'robot_path' in scene else {}
        bm = BatchedMPC(car, scene['path'], B, iter_num=iter_num, iter_threshold=thr, device=dev, warm_start=mode,
                        **scene['mpc'], **kw)
        bm.cur_index[:] = torch.as_tensor(scene['start'], dtype=torch.int32)
        run[mode] = dict(bm=bm, state=torch.as_tensor(scene['state0'], dtype=torch.float32, device=dev), ms=[], iters=[],
                         rp=[], rd=[], clear=[], ids=[], exec=[], itmax=[])
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for step in range(steps):
        for mode, r in run.items():
            torch.cuda.synchronize(dev)
            e0.record()
            _, info = r['bm'].control(r['state'], scene['speed'], clearance=True, **scene['control'])
            e1.record()
            # the executed pose (the state this step was planned from) against the obstacles it was given, the
            # time-varying ones at their stage-0 copy
            T1 = r['bm'].T + 1
            ex = r['bm'].rda.plan_clearance(r['state'][:, :, None].expand(-1, -1, T1).contiguous())['min']
            r['exec'].append(ex.cpu().numpy())
            r['bm'].advance(r['state'])
            torch.cuda.synchronize(dev)
            if step >= 2:
                r['ms'].append(e0.elapsed_time(e1))
            r['iters'].append(info['iters'].float().mean().item())
            r['itmax'].append(int(info['iters'].max()))
            r['rp'].append(info['resi_pri'].float().mean().item())
            r['rd'].append(info['resi_dual'].float().mean().item())
            r['clear'].append(info['clearance'].cpu().numpy())
            if 'obs_id' in info:
                r['ids'].append(info['obs_id'].cpu().numpy())
    out = {}
    for mode, r in run.items():
        c = np.stack(r['clear'])
        out[mode] = {'mean_admm_iterations': float(np.mean(r['iters'])),
                     'mean_of_the_slowest_robots_iterations': float(np.mean(r['itmax'])), 'ms_per_control_step': float(np.median(r['ms'])),
                     'mean_resi_pri': float(np.mean(r['rp'])), 'mean_resi_dual': float(np.mean(r['rd'])),
                     'min_plan_clearance_m': float(c[np.isfinite(c)].min()) if np.isfinite(c).any() else None,
                     'plans_below_0': int((c < 0).sum()), 'plans': int(c.size)}
        x = np.stack(r['exec'])
        out[mode].update(min_executed_signed_distance_m=float(x[np.isfinite(x)].min()) if np.isfinite(x).any() else None,
                         contacts=int((x < 0).sum()), executed_poses=int(x.size))
    ids = run['obstacle']['ids']
    if len(ids) > 1:
        ch = [float(np.mean(a != b)) for a, b in zip(ids[:-1], ids[1:])]
        out['churn'] = {'mean_share_of_slots_changing_owner': float(np.mean(ch)), 'max_share': float(np.max(ch))}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out')
    ap.add_argument('--steps', type=int, default=60)
    ap.add_argument('--robots', type=int, default=1024)
    ap.add_argument('--worlds', type=int, default=64)
    ap.add_argument('--only-remap', action='store_true', help='the remap timings only')
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('warm_start_probe needs a GPU')
    dev = torch.device('cuda:0')
    res = {'gpu': gpu_identity(0), 'remap': remap(torch, dev),
           'remap_config_E': remap(torch, dev, B=8192, T=40, N=128, E=8)}
    if a.only_remap:
        res['gpu_after'] = gpu_identity(0)
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'warm_start_probe.json'), 'w') as f:
            json.dump(res, f, indent=1)
        print(json.dumps(res, indent=1))
        return
    for name, make, n in (('world', world_scene, a.robots), ('crossing', crossing_scene, a.worlds)):
        res[name] = {}
        for label, it, thr in (('early_stop_50_0.2', 50, 0.2), ('fixed_4', 4, 0.0)):
            scene = make(torch, dev, n, np.random.default_rng(7))
            res[name][label] = loops(torch, dev, scene, a.steps, it, thr)
    res['gpu_after'] = gpu_identity(0)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'warm_start_probe.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
