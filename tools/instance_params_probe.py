"""Time the solve with and without a per-instance parameter table (RDA_solver.set_instance_parameters).

bench.py's metric row: B = 16 384 instances (bench band, seeds 9000.., 2 048 unique instances tiled), T = 30, N = 20,
E = 4, 50 ADMM iterations from a cold start, early stop off.  Three arms on one handle, alternated round by round:
no table, a table holding the handle's own values, and a mixed table (three parameter sets dealt round-robin).  Per arm:
the whole rda_solve (CUDA events around cold_start + solve) and, through the phase API, the device time of k_su and of
the cell phase (every launch of rda_step_lammuz) per ADMM iteration.  Writes DIR/instance_params_probe.json with the
GPU's name and power limit read in the same run, and checks that the uniform table gives the bits of no table.

    python tools/instance_params_probe.py DIR [--batch 16384] [--rounds 5]
"""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..'))
sys.path.insert(0, HERE)
from world_obstacles_probe import gpu_identity  # noqa: E402

T, N, E, ITERS, UNIQUE = 30, 20, 4, 50, 2048
SETS = [dict(max_speed=(10, 1), max_acce=(10, 0.5)),
        dict(max_speed=(6, 0.7), max_acce=(4, 0.3), ws=2, wu=0.5, slack_gain=5, max_sd=0.8, min_sd=0.2, ro1=100, ro2=2),
        dict(max_speed=(3, 0.5), max_acce=(2, 0.2), ws=0.5, wu=2, slack_gain=12, max_sd=1.5, min_sd=0.05, ro1=300,
             ro2=0.5)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out')
    ap.add_argument('--batch', type=int, default=16384)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    import torch
    from rda_planner_b200.rda_solver import RDA_solver, pack_obstacles
    from rda_planner_b200.scenarios import make_instance, rectangle_robot
    dev = torch.device('cuda:0')
    B = args.batch
    insts = [make_instance(9000 + i, T=T, N=N, E=E) for i in range(min(UNIQUE, B))]
    packs = [pack_obstacles(list(i['obstacles']), T, N, E) for i in insts]
    host = dict(nom_s=np.stack([i['nom_s'] for i in insts]), nom_u=np.stack([i['nom_u'] for i in insts]),
                ref_s=np.stack([i['ref'] for i in insts]), ref_speed=np.array([i['ref_speed'] for i in insts]),
                obs_A=np.stack([p[0] for p in packs]), obs_b=np.stack([p[1] for p in packs]),
                obs_kind=np.stack([p[2] for p in packs]), obs_count=np.array([p[3] for p in packs]))
    inp = {k: torch.as_tensor(v[np.arange(B) % len(v)], device=dev).contiguous() for k, v in host.items()}
    inp = {k: v.float() if v.is_floating_point() else v.int() for k, v in inp.items()}
    g = RDA_solver(T, rectangle_robot(), max_edge_num=E, max_obs_num=N, iter_num=ITERS, iter_threshold=0.0,
                   time_print=False, batch=B, device=dev)
    which = torch.arange(B, device=dev) % len(SETS)

    def arm(name):
        g.clear_instance_parameters()
        if name == 'uniform':
            g.set_instance_parameters()
        elif name == 'mixed':
            for k, s in enumerate(SETS):
                g.set_instance_parameters(robots=which == k, **s)

    ev = lambda: torch.cuda.Event(enable_timing=True)

    def solve_ms():
        e0, e1 = ev(), ev()
        g.cold_start()
        e0.record()
        out = g.iterative_solve_batch(**inp)
        e1.record()
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1), {k: v.clone() for k, v in out.items()}

    def phase_ms():
        g.cold_start()
        g.begin(inp['nom_s'], inp['nom_u'], inp['ref_s'], inp['ref_speed'], inp['obs_A'], inp['obs_b'], inp['obs_kind'],
                inp['obs_count'], False, 0.0)
        evs = [(ev(), ev(), ev()) for _ in range(ITERS)]
        for a, b, c in evs:
            a.record()
            g.step_su()
            b.record()
            g.step_lammuz()
            c.record()
        g.finish()
        torch.cuda.synchronize(dev)
        return (sum(a.elapsed_time(b) for a, b, _ in evs) / ITERS, sum(b.elapsed_time(c) for _, b, c in evs) / ITERS)

    arms = ['none', 'uniform', 'mixed']
    res = {a: {'solve_ms': [], 'k_su_ms_per_iter': [], 'cells_ms_per_iter': []} for a in arms}
    outs = {}
    for a in arms:                                   # warm-up of every arm
        arm(a)
        solve_ms()
        phase_ms()
    for r in range(args.rounds):
        for a in (arms if r % 2 == 0 else arms[::-1]):
            arm(a)
            ms, outs[a] = solve_ms()
            su, cells = phase_ms()
            res[a]['solve_ms'].append(ms)
            res[a]['k_su_ms_per_iter'].append(su)
            res[a]['cells_ms_per_iter'].append(cells)
    same = all(torch.equal(outs['none'][k], outs['uniform'][k]) for k in ('u', 's', 'status', 'iters'))
    summary = {a: {k + '_median': float(np.median(v)) for k, v in r.items()} for a, r in res.items()}
    for a in ('uniform', 'mixed'):
        summary[a]['solve_vs_none_pct'] = 100.0 * (summary[a]['solve_ms_median'] / summary['none']['solve_ms_median'] - 1)
    doc = {'gpu': gpu_identity(0), 'workload': {'batch': B, 'unique': min(UNIQUE, B), 'T': T, 'N': N, 'E': E,
                                               'iters': ITERS, 'cold_start': True, 'early_stop': False},
           'rounds': args.rounds, 'arms': res, 'summary': summary, 'uniform_table_bitwise_equal_to_none': same}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'instance_params_probe.json'), 'w') as f:
        json.dump(doc, f, indent=1)
    print(json.dumps({'gpu': doc['gpu'], 'summary': summary, 'uniform_bitwise': same}))


if __name__ == '__main__':
    main()
