"""Time rda_plan_clearance and measure what it reports in a closed loop.

Kernel time from CUDA events over many launches (RDA_solver.plan_clearance on the last begin's obstacles, s = nom_s), with
and without the per-cell map, at three shapes: the metric row (B = 16 384, T = 30, N = 20 static polygons, E = 4),
config C's moving discs (B = 512, T = 30, N = 20 per-stage copies, E = 3) and config E's shape (B = 1 024 per GPU, T = 40,
N = 128, E = 8).  Bytes are the algorithm's from the shapes (s, the obstacle rows and kinds read, the map and the minimum
written), cells N * (T + 1) per instance.  Then the warm-started BatchedMPC step of bench.py's closed_loop shape
(B = 16 384, 50 ADMM iterations), control + advance, with and without clearance=True alternated step by step in one
session, and the share of robots whose plan clearance is below 0 and below min_sd at each step.  Writes
OUT/plan_clearance_probe.json with the GPU's name and power limit read in the same run.

    python tools/plan_clearance_probe.py OUT [--steps 6] [--launches 200]
"""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, '..')
sys.path.insert(0, ROOT)
sys.path.insert(1, HERE)


def kernel_row(name, cfg_name, B, unique, launches, dev):
    import torch
    from rda_planner_b200.rda_solver import RDA_solver, pack_obstacles
    from rda_planner_b200.scenarios import CONFIGS, config_instance, rectangle_robot
    c = CONFIGS[cfg_name]
    T, N, E = c['T'], c['N'], c['E']
    insts = [config_instance(cfg_name, 9000 + i) for i in range(unique)]
    packs = [pack_obstacles(list(i['obstacles']), T, N, E) for i in insts]
    tv = bool(packs[0][4])
    host = dict(nom_s=np.stack([i['nom_s'] for i in insts]), nom_u=np.stack([i['nom_u'] for i in insts]),
                ref_s=np.stack([i['ref'] for i in insts]), ref_speed=np.array([i['ref_speed'] for i in insts]),
                obs_A=np.stack([p[0] for p in packs]), obs_b=np.stack([p[1] for p in packs]),
                obs_kind=np.stack([p[2] for p in packs]), obs_count=np.array([p[3] for p in packs]))
    inp = {k: torch.as_tensor(v[np.arange(B) % unique], device=dev).contiguous() for k, v in host.items()}
    inp = {k: v.float() if v.is_floating_point() else v.int() for k, v in inp.items()}
    g = RDA_solver(T, rectangle_robot(dynamics=c['dynamics']), max_edge_num=E, max_obs_num=N, iter_num=1,
                   iter_threshold=0.0, time_print=False, batch=B, device=dev)
    g.begin(inp['nom_s'], inp['nom_u'], inp['ref_s'], inp['ref_speed'], inp['obs_A'], inp['obs_b'], inp['obs_kind'],
            inp['obs_count'], tv)
    Tc = T + 1 if tv else 1
    row = {'shape': name, 'B': B, 'T': T, 'N': N, 'E': E, 'time_varying': tv, 'cells': B * N * (T + 1)}
    for per_cell in (False, True):
        for _ in range(5):
            out = g.plan_clearance(inp['nom_s'], per_cell=per_cell)
        torch.cuda.synchronize(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            out = g.plan_clearance(inp['nom_s'], per_cell=per_cell)
        e1.record()
        torch.cuda.synchronize(dev)
        ms = e0.elapsed_time(e1) / launches
        nbytes = (B * 3 * (T + 1) * 4 + B * N * Tc * E * 3 * 4 + B * N * 4 + B * 4 + B * 8
                  + (B * N * (T + 1) * 4 if per_cell else 0))
        key = 'with_map' if per_cell else 'min_only'
        row[key] = {'ms': ms, 'bytes': nbytes, 'GB_per_s': nbytes / (ms * 1e-3) / 1e9,
                    'Gcells_per_s': row['cells'] / (ms * 1e-3) / 1e9}
    row['share_below_0'] = float((out['min'] < 0).float().mean())
    del g
    torch.cuda.empty_cache()
    return row


def closed_loop(dev, steps):
    """bench.py closed_loop_probe's fleet, alternating control steps without and with clearance=True."""
    import torch
    from rda_planner_b200.frontend import BatchedMPC
    from rda_planner_b200.scenarios import rectangle_robot
    T, N, E, B, ITERS = 30, 20, 4, 16384, 50
    rng = np.random.default_rng(77)
    path = np.stack([np.arange(0, 60, 0.1), np.zeros(600), np.zeros(600)], 1)
    bm = BatchedMPC(rectangle_robot(), path, B, receding=T, sample_time=0.1, iter_num=ITERS, max_edge_num=E,
                    max_obs_num=N, iter_threshold=0.0, device=dev)
    idx = rng.integers(0, 480, B)
    state = torch.as_tensor(path[idx] + rng.normal(0, [0.3, 0.3, 0.1], (B, 3)), dtype=torch.float32, device=dev)
    bm.cur_index[:] = torch.as_tensor(np.maximum(idx - 3, 0), dtype=torch.int32)
    bm.cur_vel[:, 0, :] = 4.0
    M = N
    ctr = path[idx][:, None, :2] + np.stack([rng.uniform(2, 14, (B, M)), rng.uniform(1.8, 6, (B, M)) * rng.choice([-1, 1], (B, M))], -1)
    yaw = rng.uniform(0, np.pi, (B, M))
    corners = np.array([[-1, -0.5], [1, -0.5], [1, 0.5], [-1, 0.5]])
    rot = np.stack([np.stack([np.cos(yaw), -np.sin(yaw)], -1), np.stack([np.sin(yaw), np.cos(yaw)], -1)], -2)
    xy = np.zeros((B, M, 8, 2), np.float32)
    xy[:, :, :4] = ctr[:, :, None, :] + np.einsum('bmij,kj->bmki', rot, corners)
    shapes = {'kind': np.zeros((B, M), np.int32), 'nv': np.full((B, M), 4, np.int32), 'xy': xy,
              'radius': np.zeros((B, M), np.float32), 'vel': np.zeros((B, M, 2), np.float32),
              'count': np.full(B, M, np.int32)}
    shapes = {k: torch.as_tensor(v, device=dev) for k, v in shapes.items()}
    min_sd = float(bm.rda.get_adjust_parameter()['min_sd'])
    bm.control(state, 4.0, shapes, clearance=True)
    bm.advance(state)
    torch.cuda.synchronize(dev)
    times = {False: [], True: []}
    quality = []
    for k in range(2 * steps):
        with_c = bool(k % 2)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _, info = bm.control(state, 4.0, shapes, clearance=with_c)
        bm.advance(state)
        e1.record()
        torch.cuda.synchronize(dev)
        times[with_c].append(e0.elapsed_time(e1))
        if with_c:
            c = info['clearance']
            quality.append({'step': k, 'share_below_0': float((c < 0).float().mean()),
                            'share_below_min_sd': float((c < min_sd).float().mean()),
                            'min': float(c.min())})
    return {'B': B, 'T': T, 'N': N, 'E': E, 'iters': ITERS, 'min_sd': min_sd,
            'ms_per_step_without': times[False], 'ms_per_step_with': times[True],
            'median_ms_without': float(np.median(times[False])), 'median_ms_with': float(np.median(times[True])),
            'quality_per_step': quality,
            'what': 'BatchedMPC.control + advance (50 warm-started ADMM iterations), alternated without / with '
                    'clearance=True in one session; CUDA events around each step'}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out')
    ap.add_argument('--steps', type=int, default=6)
    ap.add_argument('--launches', type=int, default=200)
    args = ap.parse_args()
    import torch
    from world_obstacles_probe import gpu_identity
    dev = torch.device('cuda:0')
    res = {'gpu': gpu_identity(0), 'kernel': []}
    res['kernel'].append(kernel_row('metric row', 'metric', 16384, 2048, args.launches, dev))
    res['kernel'].append(kernel_row('config C (moving discs)', 'C', 512, 256, args.launches, dev))
    res['kernel'].append(kernel_row('config E shape', 'E', 1024, 64, args.launches, dev))
    res['closed_loop'] = closed_loop(dev, args.steps)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'plan_clearance_probe.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
