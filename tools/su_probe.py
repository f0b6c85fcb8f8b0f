"""Time the su-QP kernel (k_su) per launch, and the cell phase next to it, at bench.py's shape on the GPU.

B = 16 384 unique metric-row instances (T = 30, N = 20 polygons, E = 4, 50 ADMM iterations, early stop off, cold start)
through the phase API (rda_begin / rda_step_su / rda_step_lammuz / rda_finish), the whole batch on one stream.  CUDA
events around every rda_step_su (k_su) and rda_step_lammuz (cell passes + finalize) of ADMM iterations 2 to 50, over
--solves whole solves after one warm-up solve.  Also recorded: the su-QP interior point iterations, su-QP solves and
pruned solves repeated with all hinges (the library's counters after the last solve), and the GPU's name and power limit
read in the same run.

    python tools/su_probe.py OUT.json [--batch 16384] [--solves 2] [--repeats 3] [--lib LABEL=PATH ...]

Every measurement runs in a process of its own.  With --lib, each library (loaded through RDA_B200_LIB) is measured
--repeats times, the libraries alternating (A B A B ...), so that two builds are compared in one session on one card;
without --lib, the library build.py makes from the tree.  The inputs are generated once and shared by every run.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)


def child(args):
    """One measurement in this process: prints one JSON line."""
    import torch
    import bench
    bench.load_library()
    from rda_planner_b200 import _cabi
    from rda_planner_b200.rda_solver import RDA_solver
    from rda_planner_b200.scenarios import rectangle_robot
    dev = torch.device('cuda:0')
    host = np.load(args.inputs)
    inp = {k: torch.from_numpy(host[k]).to(dev) for k in host.files}
    B = inp['nom_s'].shape[0]
    solver = RDA_solver(bench.T, rectangle_robot(), max_edge_num=bench.E, max_obs_num=bench.N, iter_num=bench.ITERS,
                        iter_threshold=0.0, time_print=False, batch=B, device=dev)
    iters = bench.ITERS

    def solve():
        ev = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(iters)]
        solver.cold_start()
        solver.begin(inp['nom_s'], inp['nom_u'], inp['ref_s'], inp['ref_speed'], inp['obs_A'], inp['obs_b'],
                     inp['obs_kind'], inp['obs_count'], False, 0.0)
        for i in range(iters):
            ev[i][0].record(); solver.step_su(); ev[i][1].record(); solver.step_lammuz(); ev[i][2].record()
        solver.finish()
        torch.cuda.synchronize(dev)
        return ([ev[i][0].elapsed_time(ev[i][1]) for i in range(1, iters)],
                [ev[i][1].elapsed_time(ev[i][2]) for i in range(1, iters)])
    solve()
    su, cells = [], []
    for _ in range(args.solves):
        a, b = solve()
        su += a; cells += b
    cnt = solver.state_buffer(_cabi.BUF_COUNTERS).cpu().numpy().astype(np.int64)
    line = {'k_su_ms_per_launch': float(np.mean(su)), 'k_su_ms_per_launch_median': float(np.median(su)),
            'cells_ms_per_launch': float(np.mean(cells)), 'launches_timed': len(su),
            'su_ipm_iterations': int(cnt[3]), 'su_solves': int(cnt[4]), 'su_pruned_solves_repeated': int(cnt[5]),
            'counters': cnt.tolist(), 'gpu': bench.gpu_identity(0)}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('out', nargs='?', help='JSON file to write')
    ap.add_argument('--batch', type=int, default=16384)
    ap.add_argument('--solves', type=int, default=2, help='timed solves per run (after one warm-up solve)')
    ap.add_argument('--repeats', type=int, default=3, help='runs per library')
    ap.add_argument('--lib', action='append', default=[], metavar='LABEL=PATH', help='library to measure (repeatable)')
    ap.add_argument('--child', action='store_true', help=argparse.SUPPRESS)
    ap.add_argument('--inputs', help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args)
    if not args.out:
        ap.error('OUT.json is required')
    libs = [tuple(x.split('=', 1)) for x in args.lib] or [('tree', None)]
    for label, path in libs:
        if path is not None and not os.path.exists(path):
            ap.error(f'--lib {label}: {path} does not exist')
    import bench
    with tempfile.TemporaryDirectory(prefix='su_probe_') as tmp:
        inputs = os.path.join(tmp, 'inputs.npz')
        np.savez(inputs, **bench.build_inputs(args.batch, 1000 * 9))        # bench.py's instances (rank 0)
        runs = []
        for r in range(args.repeats):
            for label, path in libs:
                env = dict(os.environ)
                if path is not None:
                    env['RDA_B200_LIB'] = os.path.abspath(path)
                out = subprocess.run([sys.executable, os.path.abspath(__file__), '--child', '--inputs', inputs,
                                      '--solves', str(args.solves)], env=env, capture_output=True, text=True)
                if out.returncode != 0:
                    sys.stderr.write(out.stderr)
                    raise SystemExit(f'su_probe: run {r} of {label} failed ({out.returncode})')
                line = json.loads(out.stdout.strip().splitlines()[-1])
                line.update(label=label, repeat=r)
                runs.append(line)
                print(json.dumps({k: line[k] for k in ('label', 'repeat', 'k_su_ms_per_launch', 'cells_ms_per_launch',
                                                        'su_ipm_iterations', 'su_pruned_solves_repeated')}), flush=True)
    summary = {}
    for label, _ in libs:
        ks = [x['k_su_ms_per_launch'] for x in runs if x['label'] == label]
        cs = [x['cells_ms_per_launch'] for x in runs if x['label'] == label]
        summary[label] = {'k_su_ms_median': float(np.median(ks)), 'k_su_ms_min': min(ks), 'k_su_ms_max': max(ks),
                          'cells_ms_median': float(np.median(cs)), 'cells_ms_min': min(cs), 'cells_ms_max': max(cs)}
    res = {'what': 'k_su and cell phase per launch, CUDA events, ADMM iterations 2-50, phase API, one stream',
           'shape': {'batch': args.batch, 'T': bench.T, 'N': bench.N, 'E': bench.E, 'admm_iterations': bench.ITERS,
                     'unique_instances': args.batch, 'timed_solves_per_run': args.solves},
           'gpu': runs[0]['gpu'], 'order': [x['label'] for x in runs], 'summary': summary, 'runs': runs}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps(summary))


if __name__ == '__main__':
    main()
