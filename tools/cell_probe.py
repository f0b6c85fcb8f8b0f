"""Time every kernel of the cell phase per ADMM iteration at bench.py's shape on the GPU (torch.profiler, CUDA activities).

B = 16 384 unique metric-row instances (T = 30, N = 20 polygons, E = 4, 50 ADMM iterations, early stop off, cold start)
through the phase API (rda_begin / rda_step_su / rda_step_lammuz / rda_finish), the whole batch on one stream, with the
rear-axle rectangle or (--body disc) bench.py's disc body of radius 1.2 m.  The
profiler records ADMM iterations 2 to 50 of --solves whole solves after one unprofiled warm-up solve; the device time of
each kernel is summed by a stable name (k_cells_fast<4,4,true>, k_cells_mid, ...) and divided by the ADMM iterations
recorded.  Also recorded: the library's counters after the last solve (cells resolved by the closed forms, by the
cooperative pass, failed), a SHA-256 of u, s, status, iters and every state plane after the last solve (so that two
libraries can be compared bit for bit in the same run), and the GPU's name and power limit read in the same run.

    python tools/cell_probe.py OUT.json [--body rectangle|disc] [--batch 16384] [--solves 2] [--repeats 3] [--lib LABEL=PATH ...]

Every measurement runs in a process of its own, with the profiler on (the per-kernel times are the profiler's; the
headline step time is bench.py's, taken without it).  With --lib, each library (loaded through RDA_B200_LIB) is measured
--repeats times, the libraries alternating (A B A B ...), so that two builds are compared in one session on one card;
without --lib, the library build.py makes from the tree.  The inputs are generated once and shared by every run.
"""
import argparse
import hashlib
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

# the kernels of rda_step_lammuz (rda_kernels.cu, step_lammuz_part), polygon and disc body; the tails run the cells the
# first pass declines
CELL_KERNELS = ['k_heading', 'k_cells_coh', 'k_cells_fast<4,4,true>', 'k_cells_fast<4,4,false>', 'k_cells_fast<8,8,false>',
                'k_cells_mid', 'k_cells_extra', 'k_cells_slow_coop', 'k_cells_dr', 'k_cells_dr_mid', 'k_cells_dr_slow_coop',
                'k_finalize']
TAIL_KERNELS = ['k_cells_fast<4,4,true>', 'k_cells_mid', 'k_cells_extra', 'k_cells_slow_coop', 'k_cells_dr_mid',
                'k_cells_dr_slow_coop']
# what the digest covers: the outputs that do not depend on the order of float atomics, and every state plane
DIGEST_OUTPUTS = ('u', 's', 'status', 'iters')
DIGEST_PLANES = ('LAM', 'MU', 'Z', 'XI', 'ZETA', 'DIS', 'COEF', 'PREF', 'CUR_S', 'CUR_U')


def body(name):
    from rda_planner_b200.scenarios import disc_robot, rectangle_robot
    return disc_robot(radius=1.2, wheelbase=2.0, dynamics='diff') if name == 'disc' else rectangle_robot()


def stable_name(name):
    """'void (anonymous namespace)::k_cells_fast<4, 4, true>((anonymous namespace)::DevPtrs, ...)' -> 'k_cells_fast<4,4,true>'"""
    m = re.search(r'\b(k_\w+)(<[^()]*?>)?\(', name)
    if not m:
        return name
    return m.group(1) + (m.group(2) or '').replace(' ', '')


def child(args):
    """One measurement in this process: prints one JSON line."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    import bench
    bench.load_library()
    from rda_planner_b200 import _cabi
    from rda_planner_b200.rda_solver import RDA_solver
    dev = torch.device('cuda:0')
    host = np.load(args.inputs)
    inp = {k: torch.from_numpy(host[k]).to(dev) for k in host.files}
    B = inp['nom_s'].shape[0]
    solver = RDA_solver(bench.T, body(args.body), max_edge_num=bench.E, max_obs_num=bench.N, iter_num=bench.ITERS,
                        iter_threshold=0.0, time_print=False, batch=B, device=dev)
    iters = bench.ITERS

    def solve(prof):
        solver.cold_start()
        solver.begin(inp['nom_s'], inp['nom_u'], inp['ref_s'], inp['ref_speed'], inp['obs_A'], inp['obs_b'],
                     inp['obs_kind'], inp['obs_count'], False, 0.0)
        solver.step_su(); solver.step_lammuz()
        torch.cuda.synchronize(dev)
        if prof is not None:
            prof.start()
        for _ in range(1, iters):
            solver.step_su(); solver.step_lammuz()
        torch.cuda.synchronize(dev)
        if prof is not None:
            prof.stop()
        out = solver.finish()
        torch.cuda.synchronize(dev)
        return out
    solve(None)
    us, launches = {}, {}
    for _ in range(args.solves):
        prof = profile(activities=[ProfilerActivity.CUDA])
        out = solve(prof)
        for e in prof.events():
            if e.device_type != DeviceType.CUDA:
                continue
            k = stable_name(e.name)
            us[k] = us.get(k, 0.0) + e.time_range.elapsed_us()
            launches[k] = launches.get(k, 0) + 1
    n_it = args.solves * (iters - 1)
    ms = {k: v / 1000.0 / n_it for k, v in us.items()}
    cnt = solver.state_buffer(_cabi.BUF_COUNTERS).cpu().numpy().astype(np.int64)
    arrays = [out[k] for k in DIGEST_OUTPUTS] + [solver.state_buffer(getattr(_cabi, 'BUF_' + k)) for k in DIGEST_PLANES]
    sha = hashlib.sha256()
    for a in arrays:
        sha.update(a.contiguous().cpu().numpy().tobytes())
    line = {'ms_per_iteration': ms, 'launches_per_iteration': {k: v / n_it for k, v in launches.items()},
            'cell_phase_ms': sum(ms.get(k, 0.0) for k in CELL_KERNELS),
            'tail_ms': sum(ms.get(k, 0.0) for k in TAIL_KERNELS),
            'iterations_recorded': n_it, 'counters': cnt.tolist(), 'sha256': sha.hexdigest(),
            'gpu': bench.gpu_identity(0)}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('out', nargs='?', help='JSON file to write')
    ap.add_argument('--body', choices=['rectangle', 'disc'], default='rectangle')
    ap.add_argument('--batch', type=int, default=16384)
    ap.add_argument('--solves', type=int, default=2, help='profiled solves per run (after one warm-up solve)')
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
    with tempfile.TemporaryDirectory(prefix='cell_probe_') as tmp:
        inputs = os.path.join(tmp, 'inputs.npz')
        np.savez(inputs, **bench.build_inputs(args.batch, 1000 * 9))        # bench.py's instances (rank 0)
        runs = []
        for r in range(args.repeats):
            for label, path in libs:
                env = dict(os.environ)
                if path is not None:
                    env['RDA_B200_LIB'] = os.path.abspath(path)
                out = subprocess.run([sys.executable, os.path.abspath(__file__), '--child', '--inputs', inputs,
                                      '--solves', str(args.solves), '--body', args.body], env=env, capture_output=True, text=True)
                if out.returncode != 0:
                    sys.stderr.write(out.stderr)
                    raise SystemExit(f'cell_probe: run {r} of {label} failed ({out.returncode})')
                line = json.loads(out.stdout.strip().splitlines()[-1])
                line.update(label=label, repeat=r)
                runs.append(line)
                print(json.dumps({'label': label, 'repeat': r, 'cell_phase_ms': line['cell_phase_ms'],
                                  'tail_ms': line['tail_ms'], 'sha256': line['sha256'], 'counters': line['counters'],
                                  **{k: round(v, 4) for k, v in line['ms_per_iteration'].items()}}), flush=True)
    summary = {}
    for label, _ in libs:
        mine = [x for x in runs if x['label'] == label]
        names = sorted({k for x in mine for k in x['ms_per_iteration']})
        per = {}
        for k in names + ['cell_phase_ms', 'tail_ms']:
            v = [x[k] if k in ('cell_phase_ms', 'tail_ms') else x['ms_per_iteration'].get(k, 0.0) for x in mine]
            per[k] = {'median': float(np.median(v)), 'min': min(v), 'max': max(v)}
        summary[label] = per
    res = {'what': 'device time per ADMM iteration of each kernel, torch.profiler (CUDA activities), ADMM iterations 2-50, '
                   'phase API, one stream',
           'body': args.body,
           'shape': {'batch': args.batch, 'T': bench.T, 'N': bench.N, 'E': bench.E, 'admm_iterations': bench.ITERS,
                     'unique_instances': args.batch, 'profiled_solves_per_run': args.solves},
           'tail_kernels': TAIL_KERNELS,
           'same_sha256_and_counters': len({(x['sha256'], tuple(x['counters'])) for x in runs}) == 1,
           'gpu': runs[0]['gpu'], 'order': [x['label'] for x in runs], 'summary': summary, 'runs': runs}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps({lb: {k: round(v['median'], 4) for k, v in s.items()} for lb, s in summary.items()}))


if __name__ == '__main__':
    main()
