"""Time the solve with and without robot classes (RDA_solver.set_robot_classes).

bench.py's metric row: B = 16 384 instances (bench band, seeds 9000.., 2 048 unique instances tiled), T = 30, N = 20,
E = 4, 50 ADMM iterations from a cold start, early stop off, handle body the rear-axle rectangle.  Arms on one handle,
alternated round by round: no class table ('none'), no classes but a per-instance table of the handle's own limits
('table', which every class table installs as well: the price of the table alone), a one-class table equal to the handle's body ('own') and the four
R = 4 bodies of tests/golden/make_oracle_fixture_bodies.py dealt round-robin ('mixed': acker L = 3, diff, omni, acker
L = 2.5 with its own limits).  Per arm: the whole rda_solve (CUDA events around cold_start + solve), the device time of
k_su and of the cell phase per ADMM iteration (phase API), and the su-QP interior point iterations of the solve
(counters[3]), which separates the cost of different problems from the cost of reading the class.  Writes
DIR/robot_classes_probe_<tag>.json with the GPU's name and power limit read in the same run.

--tree runs the package of another checkout (a parent build, for the 'none' arm: a parent-versus-change comparison in
one session alternates processes of the two trees and compares their u, s, status and iters, saved with --save).

    python tools/robot_classes_probe.py DIR [--tree ROOT] [--arms none,table,own,mixed] [--tag T] [--rounds 5] [--save]
    python tools/robot_classes_probe.py DIR --merge profiles/robot_classes_h100.json

--merge collects DIR's robot_classes_probe_<tag>.json files into one profile and compares the saved 'none' outputs of
every parent<i> / change<i> pair bitwise (u, s, status, iters).
"""
import argparse
import importlib.util
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, '..')
T, N, E, ITERS, UNIQUE = 30, 20, 4, 50, 2048
FOUR = ['rect_rear', 'rect_centred', 'omni_centred', 'offset_box']


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out')
    ap.add_argument('--tree', default=ROOT)
    ap.add_argument('--arms', default='none,table,own,mixed')
    ap.add_argument('--tag', default='change')
    ap.add_argument('--batch', type=int, default=16384)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--save', action='store_true')
    ap.add_argument('--merge')
    args = ap.parse_args()
    if args.merge:
        return merge(args.out, args.merge)
    sys.path.insert(0, os.path.abspath(args.tree))
    sys.path.insert(1, HERE)
    import torch
    from rda_planner_b200 import _cabi
    from rda_planner_b200.rda_solver import RDA_solver, pack_obstacles
    from rda_planner_b200.scenarios import make_instance, rectangle_robot
    from world_obstacles_probe import gpu_identity
    spec = importlib.util.spec_from_file_location('bodies', os.path.join(ROOT, 'tests', 'golden', 'make_oracle_fixture_bodies.py'))
    bodies = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bodies)
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
    rect = rectangle_robot()
    g = RDA_solver(T, rect, max_edge_num=E, max_obs_num=N, iter_num=ITERS, iter_threshold=0.0, time_print=False,
                   batch=B, device=dev)
    four = [bodies.body(n) for n in FOUR]
    four[3] = four[3]._replace(max_speed=[8, 0.9], max_acce=[6, 0.4])
    deal = torch.arange(B, device=dev, dtype=torch.int32) % len(four)

    def arm(name):
        if name == 'none':
            if hasattr(g, 'clear_robot_classes'):
                g.clear_robot_classes()
                g.clear_instance_parameters()
        elif name == 'table':
            g.clear_robot_classes()
            g.clear_instance_parameters()
            g.set_instance_parameters()
        elif name == 'own':
            g.set_robot_classes([rect], torch.zeros(B, dtype=torch.int32, device=dev))
        elif name == 'mixed':
            g.set_robot_classes(four, deal)

    ev = lambda: torch.cuda.Event(enable_timing=True)

    def solve_ms():
        e0, e1 = ev(), ev()
        g.cold_start()
        e0.record()
        out = g.iterative_solve_batch(**inp)
        e1.record()
        torch.cuda.synchronize(dev)
        su_iters = int(g.state_buffer(_cabi.BUF_COUNTERS)[3])
        return e0.elapsed_time(e1), {k: v.clone() for k, v in out.items()}, su_iters

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

    arms = args.arms.split(',')
    res = {a: {'solve_ms': [], 'k_su_ms_per_iter': [], 'cells_ms_per_iter': [], 'su_ipm_iters': []} for a in arms}
    outs = {}
    for a in arms:                                   # warm-up of every arm
        arm(a)
        solve_ms()
        phase_ms()
    for r in range(args.rounds):
        for a in (arms if r % 2 == 0 else arms[::-1]):
            arm(a)
            ms, outs[a], su_iters = solve_ms()
            su, cells = phase_ms()
            res[a]['solve_ms'].append(ms)
            res[a]['k_su_ms_per_iter'].append(su)
            res[a]['cells_ms_per_iter'].append(cells)
            res[a]['su_ipm_iters'].append(su_iters)
    summary = {a: {k + '_median': float(np.median(v)) for k, v in r.items()} for a, r in res.items()}
    for a in arms:
        s = res[a]['solve_ms']
        summary[a]['solve_ms_spread_pct'] = 100.0 * (max(s) - min(s)) / float(np.median(s))
        summary[a]['solves_per_s'] = B / (summary[a]['solve_ms_median'] / 1e3)
    if 'none' in arms:
        for a in arms:
            summary[a]['solve_vs_none_pct'] = 100.0 * (summary[a]['solve_ms_median'] / summary['none']['solve_ms_median'] - 1)
    checks = {}
    if 'own' in arms and 'none' in arms:
        checks['own_bitwise_equal_to_none'] = all(torch.equal(outs['none'][k], outs['own'][k])
                                                  for k in ('u', 's', 'status', 'iters'))
    if 'mixed' in arms:
        checks['mixed_status_ok'] = bool(((outs['mixed']['status'] & 7) == 0).float().mean().item() > 0.9)
    os.makedirs(args.out, exist_ok=True)
    if args.save and 'none' in arms:
        torch.save({k: outs['none'][k].cpu() for k in ('u', 's', 'status', 'iters')},
                   os.path.join(args.out, f'robot_classes_none_{args.tag}.pt'))
    doc = {'gpu': gpu_identity(0), 'tree': args.tag,
           'workload': {'batch': B, 'unique': min(UNIQUE, B), 'T': T, 'N': N, 'E': E, 'iters': ITERS, 'cold_start': True,
                        'early_stop': False, 'mixed_classes': FOUR},
           'rounds': args.rounds, 'arms': res, 'summary': summary, 'checks': checks}
    with open(os.path.join(args.out, f'robot_classes_probe_{args.tag}.json'), 'w') as f:
        json.dump(doc, f, indent=1)
    print(json.dumps({'tag': args.tag, 'gpu': doc['gpu'], 'summary': summary, 'checks': checks}))


def merge(src, dst):
    import glob
    import torch
    runs = [json.load(open(f)) for f in sorted(glob.glob(os.path.join(src, 'robot_classes_probe_*.json')))]
    bitwise = {}
    for r in runs:
        tag = r['tree']
        if tag.startswith('change'):
            par = os.path.join(src, f'robot_classes_none_parent{tag[6:]}.pt')
            cha = os.path.join(src, f'robot_classes_none_{tag}.pt')
            if os.path.exists(par) and os.path.exists(cha):
                a, b = torch.load(par), torch.load(cha)
                bitwise[tag] = {k: bool(torch.equal(a[k], b[k])) for k in a}
    doc = {'what': 'tools/robot_classes_probe.py: parent build (arm none) and this change (arms none, own, mixed) in '
                   'alternated processes of one session; --merge of their outputs',
           'gpu': runs[0]['gpu'], 'workload': runs[0]['workload'], 'rounds': runs[0]['rounds'],
           'runs': {r['tree']: {'summary': r['summary'], 'checks': r['checks'],
                                'solve_ms': {a: v['solve_ms'] for a, v in r['arms'].items()}} for r in runs},
           'parent_vs_change_none_bitwise': bitwise}
    with open(dst, 'w') as f:
        json.dump(doc, f, indent=1)
    print(json.dumps({'runs': list(doc['runs']), 'bitwise': bitwise}))


if __name__ == '__main__':
    main()
