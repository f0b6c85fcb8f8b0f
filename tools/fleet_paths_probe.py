"""Time the per-robot path kernels (rda_pre_process_paths, rda_post_process_paths) on the GPU.

At B robots (default 16 384) on W paths of a shared set (W = 1, 1 024, 16 384; 600-waypoint random paths of 1 to 4
curves, robots anywhere along them; T = 30), CUDA events around many launches of each kernel alone.  Then bench.py's
closed_loop shape (B robots, T = 30, N = 20 boxes per robot, E = 4, 50 ADMM iterations, warm-started
BatchedMPC.control + advance) with every robot on one 60 m line against every robot on its own translated copy of it,
its boxes translated with it.  Writes DIR/fleet_paths_probe.json with the GPU's name and power limit read in the same
run.

    python tools/fleet_paths_probe.py DIR [--batch 16384] [--paths 1,1024,16384]
"""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..'))
sys.path.insert(0, HERE)
from world_obstacles_probe import event_ms, gpu_identity  # noqa: E402

T, N, E, ITERS, DT, P = 30, 20, 4, 50, 0.1, 600


def random_set(rng, W):
    """W paths of P waypoints (random walks, 0.1 m steps) cut into 1 to 4 curves of alternating gear."""
    from rda_planner_b200.frontend import pack_paths
    paths = []
    for _ in range(W):
        head = np.cumsum(rng.normal(0, 0.02, P)) + rng.uniform(-np.pi, np.pi)
        xy = np.cumsum(0.1 * np.stack([np.cos(head), np.sin(head)], 1), 0) + rng.uniform(-100, 100, 2)
        gear = np.ones(P)
        for c in np.sort(rng.choice(np.arange(1, P), int(rng.integers(0, 4)), replace=False)):
            gear[c:] *= -1
        paths.append(np.concatenate([xy, head[:, None], gear[:, None]], 1))
    return pack_paths(paths, enable_reverse=True)


def closed_loop_step(dev, B, per_robot):
    """ms of one warm-started control + advance in bench.py's closed_loop shape."""
    import torch
    from rda_planner_b200.frontend import BatchedMPC
    from rda_planner_b200.scenarios import rectangle_robot
    rng = np.random.default_rng(77)
    line = np.stack([np.arange(0, 60, 0.1), np.zeros(600), np.zeros(600)], 1)
    idx = rng.integers(0, 480, B)
    off = np.stack([50.0 * (np.arange(B) % 64), 20.0 * (np.arange(B) // 64), np.zeros(B)], 1) if per_robot \
        else np.zeros((B, 3))
    kw = dict(receding=T, sample_time=DT, iter_num=ITERS, max_edge_num=E, max_obs_num=N, iter_threshold=0.0,
              device=dev)
    if per_robot:
        bm = BatchedMPC(rectangle_robot(), [line + o for o in off], B, robot_path=np.arange(B), **kw)
    else:
        bm = BatchedMPC(rectangle_robot(), line, B, **kw)
    state = torch.as_tensor(line[idx] + off + rng.normal(0, [0.3, 0.3, 0.1], (B, 3)), dtype=torch.float32, device=dev)
    bm.cur_index[:] = torch.as_tensor(np.maximum(idx - 3, 0), dtype=torch.int32)
    bm.cur_vel[:, 0, :] = 4.0
    ctr = line[idx][:, None, :2] + off[:, None, :2] + \
        np.stack([rng.uniform(2, 14, (B, N)), rng.uniform(1.8, 6, (B, N)) * rng.choice([-1, 1], (B, N))], -1)
    yaw = rng.uniform(0, np.pi, (B, N))
    corners = np.array([[-1, -0.5], [1, -0.5], [1, 0.5], [-1, 0.5]])
    rot = np.stack([np.stack([np.cos(yaw), -np.sin(yaw)], -1), np.stack([np.sin(yaw), np.cos(yaw)], -1)], -2)
    xy = np.zeros((B, N, 8, 2), np.float32)
    xy[:, :, :4] = ctr[:, :, None, :] + np.einsum('bmij,kj->bmki', rot, corners)
    shapes = {'kind': np.zeros((B, N), np.int32), 'nv': np.full((B, N), 4, np.int32), 'xy': xy,
              'radius': np.zeros((B, N), np.float32), 'vel': np.zeros((B, N, 2), np.float32),
              'count': np.full(B, N, np.int32)}
    shapes = {k: torch.as_tensor(v, device=dev) for k, v in shapes.items()}

    def step():
        bm.control(state, 4.0, shapes)
        bm.advance(state)
    ms, reps = event_ms(step, dev, min_window_s=2.0)
    u0, info = bm.control(state, 4.0, shapes)
    ok = bool(torch.isfinite(u0).all()) and int((info['status'] & 6).sum()) == 0
    return {'B': B, 'paths': B if per_robot else 1, 'ms': ms, 'steps': reps, 'mpc_steps_per_s': B / (ms * 1e-3),
            'finite_and_converged': ok}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('out_dir')
    ap.add_argument('--batch', type=int, default=16384)
    ap.add_argument('--paths', default='1,1024,16384')
    args = ap.parse_args()
    import torch
    from rda_planner_b200 import _cabi
    from rda_planner_b200.frontend import _ptr, _stream
    assert torch.cuda.is_available(), 'the probe measures the GPU; there is nothing to measure without one'
    dev = torch.device('cuda:0')
    lib = _cabi.load()
    B = args.batch
    rng = np.random.default_rng(5)
    out = {'gpu': gpu_identity(0), 'B': B, 'T': T, 'waypoints_per_path': P, 'kernels': [], 'closed_loop': []}
    for W in (int(x) for x in args.paths.split(',')):
        pk = random_set(rng, W)
        d = {k: torch.as_tensor(v, device=dev) for k, v in pk.items()}
        rp = rng.integers(0, W, B).astype(np.int32)
        ci = np.zeros(B, np.int32)
        start, state = np.zeros(B, np.int32), np.zeros((B, 3), np.float32)
        for b in range(B):
            lo, hi = pk['path_curve'][rp[b]], pk['path_curve'][rp[b] + 1]
            ci[b] = rng.integers(0, hi - lo)
            cs, ce = pk['curve_start'][lo + ci[b]], pk['curve_start'][lo + ci[b] + 1]
            start[b] = rng.integers(0, ce - cs)
            state[b] = pk['path'][cs + start[b]] + rng.normal(0, [0.3, 0.3, 0.1])
        t = lambda a: torch.as_tensor(a, device=dev)
        rp_d, ci_d, st_d, state_d = t(rp), t(ci), t(start), t(state)
        vel = torch.full((B, 2, T), 0.0, dtype=torch.float32, device=dev)
        vel[:, 0] = 4.0
        speed = torch.full((B,), 4.0, dtype=torch.float32, device=dev)
        nom = torch.empty((B, 3, T + 1), dtype=torch.float32, device=dev)
        ref, near, sp = torch.empty_like(nom), torch.empty(B, dtype=torch.int32, device=dev), torch.empty_like(speed)
        u = torch.randn((B, 2, T), device=dev)
        cur_vel, arrive = torch.empty_like(u), torch.empty_like(near)
        s = _stream(dev)
        pre = lambda: _cabi.check(lib.rda_pre_process_paths(
            B, T, 0, DT, 3.0, _ptr(state_d), _ptr(vel), _ptr(speed), _ptr(d['path']), W, _ptr(d['path_curve']),
            _ptr(d['curve_start']), _ptr(d['curve_gear']), _ptr(rp_d), _ptr(ci_d), _ptr(st_d), 0.1, 10, _ptr(nom),
            _ptr(ref), _ptr(near), _ptr(sp), s), 'rda_pre_process_paths')
        pre_ms, pre_n = event_ms(pre, dev)
        near0, ci0 = near.clone(), ci_d.clone()

        def post():                                   # from the same indices every launch
            near.copy_(near0)
            ci_d.copy_(ci0)
            _cabi.check(lib.rda_post_process_paths(B, T, W, _ptr(d['path_curve']), _ptr(d['curve_start']), _ptr(rp_d),
                                                   1, _ptr(near), _ptr(ci_d), _ptr(u), _ptr(cur_vel), _ptr(arrive), s),
                        'rda_post_process_paths')
        copies_ms, _ = event_ms(lambda: (near.copy_(near0), ci_d.copy_(ci0)), dev)
        post_ms, post_n = event_ms(post, dev)
        out['kernels'].append({'W': W, 'pre_ms': pre_ms, 'pre_launches': pre_n, 'post_ms': post_ms - copies_ms,
                               'post_launches': post_n, 'post_ms_including_index_reset': post_ms})
    for per_robot in (False, True):
        out['closed_loop'].append(closed_loop_step(dev, B, per_robot))
    step = out['closed_loop'][0]['ms']
    for r in out['kernels']:
        r['fraction_of_closed_loop_step'] = (r['pre_ms'] + r['post_ms']) / step
    out['what'] = ('kernels: CUDA events around back-to-back launches of each entry point alone (post: minus the two '
                   'index copies that reset its inputs every launch); closed_loop: BatchedMPC.control + advance, '
                   'warm-started, 50 iterations, one shared 60 m line against one translated copy per robot; '
                   'fraction_of_closed_loop_step: pre + post over the one-path step')
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, 'fleet_paths_probe.json'), 'w') as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
