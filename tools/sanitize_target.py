"""Small target for compute-sanitizer (memcheck / racecheck): short batched solves covering polygon and
disc obstacles, static and moving, the two-stream sub-batch path (forced on this small batch; the interior point pass
is the warp-cooperative one), a disc body, and the front-end kernels through one closed-loop step of BatchedMPC."""
import os
import sys

os.environ['RDA_B200_SPLIT_MIN'] = '2'

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from rda_planner_b200.rda_solver import RDA_solver, pack_obstacles  # noqa: E402
from rda_planner_b200.scenarios import rectangle_robot, make_instance  # noqa: E402

for kind, moving in (('polygon', False), ('circle', True)):
    T, N, B = 10, 6, 48      # N*T multiple of 4: the persistent kernel stages its state with bulk (TMA) copies
    car = rectangle_robot()
    insts = [make_instance(40 + i, T=T, N=N, E=4, kind=kind, moving=moving, lateral=(0.3, 3.5)) for i in range(B)]
    packs = [pack_obstacles(list(i['obstacles']), T, N, 4) for i in insts]
    tv = any(p[4] for p in packs)
    if tv:      # all instances must share the layout: expand static ones
        packs = [(np.repeat(p[0], T + 1, 1) if not p[4] else p[0], np.repeat(p[1], T + 1, 1) if not p[4] else p[1], p[2], p[3], True)
                 for p in packs]
    g = RDA_solver(T, car, 4, N, iter_num=4, iter_threshold=0.0, time_print=False, batch=B)
    out = g.iterative_solve_batch(np.stack([i['nom_s'] for i in insts]), np.stack([i['nom_u'] for i in insts]),
                                  np.stack([i['ref'] for i in insts]), np.array([4.0] * B), np.stack([p[0] for p in packs]),
                                  np.stack([p[1] for p in packs]), np.stack([p[2] for p in packs]),
                                  np.array([p[3] for p in packs]), tv)
    torch.cuda.synchronize()
    print(kind, 'ok', bool(torch.isfinite(out['u']).all()), int((out['status'] & 6).sum()))

# disc body (cone_type 'norm2'): k_cells_dr / k_cells_dr_mid / k_cells_dr_slow_coop
from rda_planner_b200.scenarios import disc_robot  # noqa: E402
T, N, B = 8, 4, 24
insts = [make_instance(140 + i, T=T, N=N, E=4, kind='polygon' if i % 2 else 'circle', lateral=(0.3, 3.0), dynamics='diff') for i in range(B)]
packs = [pack_obstacles(list(i['obstacles']), T, N, 4) for i in insts]
g = RDA_solver(T, disc_robot(radius=1.1, center=(0.2, 0.0), wheelbase=2.0, dynamics='diff'), 4, N, iter_num=3, iter_threshold=0.0,
               time_print=False, batch=B)
out = g.iterative_solve_batch(np.stack([i['nom_s'] for i in insts]), np.stack([i['nom_u'] for i in insts]),
                              np.stack([i['ref'] for i in insts]), np.array([4.0] * B), np.stack([p[0] for p in packs]),
                              np.stack([p[1] for p in packs]), np.stack([p[2] for p in packs]), np.array([p[3] for p in packs]), False)
torch.cuda.synchronize()
print('disc body ok', bool(torch.isfinite(out['u']).all()), int((out['status'] & 6).sum()))

# front end: pre_process, obstacle conversion (sorted, padded, moving), arrive rule, model step
from collections import namedtuple  # noqa: E402
from rda_planner_b200.frontend import BatchedMPC, pack_shapes, shapes_to_device  # noqa: E402
Obs = namedtuple('Obs', 'center radius vertex cone_type velocity')
path = np.stack([np.arange(0, 20, 0.1), np.zeros(200), np.zeros(200)], 1)
B, T, N = 33, 10, 5
rng = np.random.default_rng(5)
lists = []
for b in range(B):
    obs = []
    for j in range(int(rng.integers(0, 9))):
        c = np.array([[rng.uniform(2, 18)], [rng.uniform(2, 5) * rng.choice([-1, 1])]])
        vel = rng.uniform(-0.4, 0.4, (2, 1)) if j % 2 else np.zeros((2, 1))
        if j % 3 == 0:
            obs.append(Obs(c, 0.6, None, 'norm2', vel))
        else:
            ang = np.sort(rng.uniform(0, 2 * np.pi, 4))[::(-1 if j % 2 else 1)]
            obs.append(Obs(None, None, c + 0.8 * np.vstack([np.cos(ang), np.sin(ang)]), 'Rpositive', vel))
    lists.append(obs)
bm = BatchedMPC(rectangle_robot(), path, B, receding=T, iter_num=3, max_edge_num=4, max_obs_num=N, iter_threshold=0.0)
state = torch.as_tensor(path[rng.integers(0, 199, B)] + rng.normal(0, 0.2, (B, 3)), dtype=torch.float32, device='cuda')
bm.cur_index[:] = torch.as_tensor(rng.integers(150, 199, B), dtype=torch.int32)
shapes = shapes_to_device(pack_shapes(lists, 10), 'cuda')
for _ in range(2):
    u0, info = bm.control(state, 4.0, shapes, time_varying=True)
    bm.advance(state)
torch.cuda.synchronize()
print('front end ok', bool(torch.isfinite(u0).all()), int(info['arrive'].sum()))
