"""Time the fleet obstacle selection (rda_fleet_shapes + rda_convert_fleet_obstacles) on the GPU.

For B robots split into worlds of R robots, each world a map of M boxes (N = 20, static and time-varying output),
CUDA events around many launches of the two kernels (the world -> robots lists are built once, outside the window);
a warm-started BatchedMPC.control + advance step at B = 16 384 (2 048 worlds of 8 robots 6 m apart on the path, each
world a map of 1 024 boxes; bench.py's closed_loop shape: T = 30, N = 20, E = 4, 50 ADMM iterations) with and without
avoid_fleet.  Worlds whose
maps would hold more than MAX_SHAPES boxes in all are not measured.  Writes DIR/fleet_obstacles_probe.json with the
GPU's name and power limit read in the same run.

    python tools/fleet_obstacles_probe.py DIR [--batches 256,4096,16384] [--per-world 1,16,256,B] [--maps 0,1024,16384]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from world_obstacles_probe import event_ms, gpu_identity  # noqa: E402

T, N, E, ITERS, DT = 30, 20, 4, 50, 0.1
MAX_SHAPES = 1 << 24


def boxes(torch, W, M, dev, gen):
    """W maps of M 2 x 1 m boxes of random yaw, centres along a 60 m line and 1.8..6 m to either side, on the device."""
    S = max(1, W * M)
    ctr = torch.stack([torch.rand(S, device=dev, generator=gen) * 60,
                       (1.8 + 4.2 * torch.rand(S, device=dev, generator=gen))
                       * torch.where(torch.rand(S, device=dev, generator=gen) < 0.5, -1.0, 1.0)], -1)
    yaw = torch.rand(S, device=dev, generator=gen) * np.pi
    corners = torch.tensor([[-1, -0.5], [1, -0.5], [1, 0.5], [-1, 0.5]], device=dev)
    c, s = torch.cos(yaw)[:, None], torch.sin(yaw)[:, None]
    xy = torch.zeros((S, 8, 2), device=dev)
    xy[:, :4, 0] = ctr[:, None, 0] + c * corners[:, 0] - s * corners[:, 1]
    xy[:, :4, 1] = ctr[:, None, 1] + s * corners[:, 0] + c * corners[:, 1]
    i32 = torch.int32
    return {'kind': torch.zeros(S, dtype=i32, device=dev), 'nv': torch.full((S,), 4, dtype=i32, device=dev),
            'xy': xy.contiguous(), 'radius': torch.zeros(S, device=dev), 'vel': torch.zeros((S, 2), device=dev),
            'start': torch.arange(W + 1, dtype=i32, device=dev) * M}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('out_dir')
    ap.add_argument('--batches', default='256,4096,16384')
    ap.add_argument('--per-world', default='1,16,256,B')
    ap.add_argument('--maps', default='0,1024,16384')
    args = ap.parse_args()
    import torch
    from rda_planner_b200 import _cabi
    from rda_planner_b200.frontend import BatchedMPC, _ptr, _stream, fleet_csr, robot_body
    from rda_planner_b200.scenarios import rectangle_robot
    assert torch.cuda.is_available(), 'the probe measures the GPU; there is nothing to measure without one'
    dev = torch.device('cuda:0')
    lib = _cabi.load()
    gen = torch.Generator(device=dev)
    gen.manual_seed(5)
    rng = np.random.default_rng(5)
    body = robot_body(rectangle_robot())
    bxy = torch.as_tensor(body['xy'], device=dev)
    path = np.stack([np.arange(0, 60, 0.1), np.zeros(600), np.zeros(600)], 1)
    out = {'gpu': gpu_identity(0), 'N': N, 'E': E, 'T': T, 'shape': '2 x 1 m boxes (4 vertices); robots: the '
           '4.6 x 1.6 m rectangle_robot body', 'conversion': [], 'control_step': []}
    for B in [int(x) for x in args.batches.split(',')]:
        idx = rng.integers(0, 480, B)
        state = torch.as_tensor(path[idx] + rng.normal(0, [0.3, 0.3, 0.1], (B, 3)), dtype=torch.float32, device=dev)
        cur_vel = torch.zeros((B, 2, T), device=dev)
        cur_vel[:, 0, :] = 4.0
        fl = {'kind': torch.empty(B, dtype=torch.int32, device=dev), 'nv': torch.empty(B, dtype=torch.int32, device=dev),
              'xy': torch.empty((B, 8, 2), device=dev), 'radius': torch.empty(B, device=dev),
              'vel': torch.empty((B, 2), device=dev)}
        for R in [B if x == 'B' else int(x) for x in args.per_world.split(',')]:
            if R > B:
                continue
            W = B // R
            rw = (torch.arange(B, device=dev) % W).to(torch.int32)
            start, robots = fleet_csr(rw, W)
            for M in [int(x) for x in args.maps.split(',')]:
                rec = {'B': B, 'robots_per_world': R, 'worlds': W, 'M': M}
                if W * M > MAX_SHAPES:
                    out['conversion'] += [dict(rec, time_varying=bool(tv), ms='not measured (maps too large)')
                                          for tv in (0, 1)]
                    continue
                w = boxes(torch, W, M, dev, gen)
                for tv in (0, 1):
                    Tc = T + 1 if tv else 1
                    A = torch.empty((B, N, Tc, E, 2), device=dev)
                    b = torch.empty((B, N, Tc, E), device=dev)
                    kind = torch.empty((B, N), dtype=torch.int32, device=dev)
                    count = torch.empty(B, dtype=torch.int32, device=dev)
                    s = _stream(dev)

                    def both():
                        _cabi.check(lib.rda_fleet_shapes(B, T, 0, body['kind'], body['nv'], _ptr(bxy), body['radius'],
                                                         _ptr(state), _ptr(cur_vel), _ptr(fl['kind']), _ptr(fl['nv']),
                                                         _ptr(fl['xy']), _ptr(fl['radius']), _ptr(fl['vel']), s),
                                    'rda_fleet_shapes')
                        _cabi.check(lib.rda_convert_fleet_obstacles(
                            B, W, N, T, E, DT, tv, 1, _ptr(state), _ptr(w['start']), _ptr(rw), _ptr(w['kind']),
                            _ptr(w['nv']), _ptr(w['xy']), _ptr(w['radius']), _ptr(w['vel']), _ptr(start),
                            _ptr(robots), _ptr(fl['kind']), _ptr(fl['nv']), _ptr(fl['xy']), _ptr(fl['radius']),
                            _ptr(fl['vel']), _ptr(A), _ptr(b), _ptr(kind), _ptr(count), s), 'rda_convert_fleet_obstacles')
                    ms, reps = event_ms(both, dev)
                    assert int(count[0]) == M + R - 1
                    out['conversion'].append(dict(rec, time_varying=bool(tv), ms=ms, launches=reps,
                                                  keys_per_s=B * (M + R - 1) / (ms * 1e-3)))
                    del A, b, kind, count
                del w
        torch.cuda.empty_cache()
    # warm-started control steps at B = 16 384: worlds of 8 robots 6 m apart along the path, each on a map of 1 024 boxes
    B, R, M = 16384, 8, 1024
    W = B // R
    idx = (np.arange(B) // W) * 60 + rng.integers(0, 10, B)
    state0 = torch.as_tensor(path[idx] + rng.normal(0, [0.1, 0.1, 0.05], (B, 3)), dtype=torch.float32, device=dev)
    rw = (torch.arange(B, device=dev) % W).to(torch.int32)
    world = boxes(torch, W, M, dev, gen)
    for avoid in (False, True):
        bm = BatchedMPC(rectangle_robot(), path, B, receding=T, sample_time=DT, iter_num=ITERS, max_edge_num=E,
                        max_obs_num=N, iter_threshold=0.0, device=dev)
        bm.cur_index[:] = torch.as_tensor(np.maximum(idx - 3, 0), dtype=torch.int32)
        bm.cur_vel[:, 0, :] = 4.0
        st = state0.clone()

        def step():
            bm.control(st, 4.0, world=world, robot_world=rw, avoid_fleet=avoid)
            bm.advance(st)
        ms, reps = event_ms(step, dev, min_window_s=1.0)
        u0, info = bm.control(st, 4.0, world=world, robot_world=rw, avoid_fleet=avoid)
        out['control_step'].append({'B': B, 'robots_per_world': R, 'M': M, 'avoid_fleet': avoid, 'ms': ms,
                                    'steps': reps, 'mpc_steps_per_s': B / (ms * 1e-3),
                                    'finite': bool(torch.isfinite(u0).all())})
        del bm
    out['what'] = ('conversion: one rda_fleet_shapes + one rda_convert_fleet_obstacles launch (order = 1, acker), '
                   'CUDA events, B robots in B / R worlds of R robots, each world a map of M boxes; keys_per_s: '
                   'B (M + R - 1) / time.  control_step: BatchedMPC.control(world=..., robot_world=...) + advance, '
                   'warm-started, 50 iterations, static maps, worlds of 8 robots 6 m apart')
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, 'fleet_obstacles_probe.json'), 'w') as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
