"""k_convert_world_obstacles through the C ABI (rda_convert_world_obstacles): against its CPU twin on shared and
per-robot worlds of any size, against rda_convert_obstacles where both apply, config E's 128 polytopes through the
solver, and BatchedMPC on a shared map against one host mpc.MPC per robot."""
import copy
import os
from collections import namedtuple

import numpy as np
import pytest
import torch

import world_twin
from rda_planner_b200.scenarios import config_instance, rectangle_robot

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
PATH = list(np.load(os.path.join(HERE, 'golden', 'path_track_ref.npy'), allow_pickle=True))
PATH_ARR = np.stack([np.asarray(p, float).reshape(-1)[:3] for p in PATH])
Obs = namedtuple('Obs', 'center radius vertex cone_type velocity')
DEV = torch.device('cuda:0')
DT = 0.1
DT32 = float(np.float32(DT))          # the kernel's float dt, widened: the twin gets the same value


def _dev(host):
    from rda_planner_b200.frontend import shapes_to_device
    return shapes_to_device(host, DEV)


def _shared_world(rng, count, lo=0.0, hi=200.0):
    """`count` shapes scattered over a square map: discs and 3..8-gons, CW and CCW, a third moving, some exact
    duplicates."""
    obs = []
    for j in range(count):
        vel = rng.uniform(-1, 1, (2, 1)) if j % 3 == 1 else np.zeros((2, 1))
        if j % 11 == 10:
            obs.append(obs[int(rng.integers(0, len(obs)))])
            continue
        c = rng.uniform(lo, hi, (2, 1))
        if j % 4 == 0:
            obs.append(Obs(c, float(rng.uniform(0.3, 1.5)), None, 'norm2', vel))
        else:
            n = int(rng.integers(3, 9))
            ang = np.linspace(0, 2 * np.pi, n, endpoint=False) + rng.uniform(0, 1)
            if j % 2:
                ang = ang[::-1]
            obs.append(Obs(None, None, c + rng.uniform(0.4, 2.0) * np.vstack([np.cos(ang), np.sin(ang)]), 'Rpositive', vel))
    return obs


def _case(name, rng):
    """(worlds, robot_world [B] or None, state [B,3] float32, E)."""
    if name == 'shared':                                          # (a) one world of ~5000 shapes, 300 robots in it
        worlds = [_shared_world(rng, 5000)]
        state = np.c_[rng.uniform(0, 200, (300, 2)), rng.uniform(-np.pi, np.pi, 300)].astype(np.float32)
        return worlds, None, state, 8
    if name == 'config_e':                                        # (b) per-robot worlds of config E's 128 polytopes
        insts = [config_instance('E', s) for s in range(12)]
        return ([i['obstacles'] for i in insts], np.arange(12, dtype=np.int32),
                np.stack([i['state'] for i in insts]).astype(np.float32), 8)
    # (c) mixed sizes, empty worlds, robots whose world index is outside [0, W)
    sizes = [0, 1, 19, 20, 128, 300, 0, 1500, 64, 257]
    worlds = [_shared_world(rng, n, 0.0, 60.0) for n in sizes]
    B = 64
    rw = rng.integers(0, len(sizes), B).astype(np.int32)
    rw[:4] = [-1, len(sizes), 1 << 30, -(1 << 30)]
    state = np.c_[rng.uniform(0, 60, (B, 2)), np.zeros(B)].astype(np.float32)
    return worlds, rw, state, 8


@pytest.mark.parametrize('N', [1, 20, 128])
@pytest.mark.parametrize('tv,order', [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize('name', ['shared', 'config_e', 'mixed'])
def test_world_kernel_matches_cpu_twin(name, tv, order, N):
    from rda_planner_b200.frontend import convert_world_obstacles_batch, pack_worlds
    worlds, rw, state, E = _case(name, np.random.default_rng({'shared': 1, 'config_e': 2, 'mixed': 3}[name]))
    T = 10
    host = pack_worlds(worlds)
    A, b, kind, count = convert_world_obstacles_batch(_dev(host), torch.as_tensor(state, device=DEV),
                                                      None if rw is None else torch.as_tensor(rw, device=DEV),
                                                      N, T, E, DT, tv, order)
    A, b, kind, count = A.cpu().numpy(), b.cpu().numpy(), kind.cpu().numpy(), count.cpu().numpy()
    for i in range(state.shape[0]):
        w = 0 if rw is None else int(rw[i])
        A1, b1, k1, c1 = world_twin.convert_world_obstacles(host, w, N, T, E, DT32, tv, order, state[i])
        assert count[i] == c1 == (len(worlds[w]) if 0 <= w < len(worlds) else 0), i
        assert list(kind[i]) == list(k1), i
        np.testing.assert_array_equal(A[i], A1)
        np.testing.assert_allclose(b[i], b1, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize('tv,order', [(False, True), (True, True), (True, False)])
def test_world_kernel_equals_per_robot_kernel(tv, order):
    """Each robot's world is its own list of <= 64 shapes: bit for bit what rda_convert_obstacles writes."""
    from rda_planner_b200.frontend import convert_obstacles_batch, convert_world_obstacles_batch, pack_shapes, pack_worlds
    rng = np.random.default_rng(12)
    B, T, N, E = 97, 10, 20, 8
    lists = [_shared_world(rng, int(c), 0.0, 40.0) for c in rng.integers(0, 65, B)]
    lists[0], lists[1] = [], _shared_world(rng, 64, 0.0, 40.0)
    state = torch.as_tensor(np.c_[rng.uniform(0, 40, (B, 2)), np.zeros(B)].astype(np.float32), device=DEV)
    ref = convert_obstacles_batch(_dev(pack_shapes(lists, 64)), state, N, T, E, DT, tv, order)
    got = convert_world_obstacles_batch(_dev(pack_worlds(lists)), state, torch.arange(B, dtype=torch.int32, device=DEV),
                                        N, T, E, DT, tv, order)
    for r, g in zip(ref, got):
        assert torch.equal(r, g)


def test_config_e_worlds_through_the_solver():
    """Config E (128 polytopes, N = 128, E = 8) in list order: the kernel's arrays against pack_obstacles of the same
    instances, then 3 iterations of the batched solve on each."""
    from rda_planner_b200.frontend import convert_world_obstacles_batch, pack_worlds
    from rda_planner_b200.rda_solver import RDA_solver, pack_obstacles
    insts = [config_instance('E', s) for s in range(8)]
    B, T, N, E = len(insts), 40, 128, 8
    host = pack_worlds([i['obstacles'] for i in insts])
    state = torch.as_tensor(np.stack([i['state'] for i in insts]).astype(np.float32), device=DEV)
    A, b, kind, count = convert_world_obstacles_batch(_dev(host), state, torch.arange(B, dtype=torch.int32, device=DEV),
                                                      N, T, E, DT, False, False)
    packed = [pack_obstacles(list(i['obstacles']), T, N, E) for i in insts]
    Ah = np.stack([p[0] for p in packed]); bh = np.stack([p[1] for p in packed])
    assert not any(p[4] for p in packed) and list(count.cpu().numpy()) == [p[3] for p in packed] == [128] * B
    np.testing.assert_array_equal(kind.cpu().numpy(), np.stack([p[2] for p in packed]))
    # the kernel builds rows from float32 vertices, the host from float64 ones: with coordinates up to V, a row
    # a = (dy, -dx) carries the vertices' rounding, eps32 * V, and b = a . p that times |p| ~ V
    V = float(np.abs(host['xy']).max())
    eps = float(np.finfo(np.float32).eps)
    np.testing.assert_allclose(A.cpu().numpy(), Ah, rtol=1e-6, atol=2 * eps * V)
    np.testing.assert_allclose(b.cpu().numpy(), bh, rtol=1e-6, atol=4 * eps * V * V)
    nom_s = np.stack([i['nom_s'] for i in insts]); nom_u = np.stack([i['nom_u'] for i in insts])
    ref_s = np.stack([i['ref'] for i in insts]); speed = np.array([i['ref_speed'] for i in insts])
    outs = []
    for obs_A, obs_b in ((A, b), (Ah, bh)):
        s = RDA_solver(T, rectangle_robot(), max_edge_num=E, max_obs_num=N, iter_num=3, iter_threshold=0.0,
                       time_print=False, batch=B, device=DEV)
        o = s.iterative_solve_batch(nom_s, nom_u, ref_s, speed, obs_A, obs_b, kind, count, False)
        outs.append({k: v.cpu().numpy() for k, v in o.items() if isinstance(v, torch.Tensor)})
    for o in outs:
        assert np.all(o['status'] & 7 == 0), o['status']
    np.testing.assert_allclose(outs[0]['u'], outs[1]['u'], atol=1e-3)
    np.testing.assert_allclose(outs[0]['s'], outs[1]['s'], atol=1e-3)


def test_batched_mpc_on_a_shared_map_matches_host_front_end():
    """Four robots on the path_track reference share one map of 400 shapes (a third moving), 4 control steps:
    BatchedMPC.control(world=...) against one host mpc.MPC per robot that gets the whole map as obstacle_list."""
    from rda_planner_b200.frontend import BatchedMPC, pack_worlds
    from rda_planner_b200.mpc import MPC
    rng = np.random.default_rng(8)
    obs = []
    for j in range(400):                                        # beside the path, never on it
        c = PATH_ARR[int(rng.integers(0, len(PATH_ARR))), :2].reshape(2, 1) + rng.uniform(2.5, 6.0, (2, 1)) * rng.choice([-1, 1], (2, 1))
        vel = rng.uniform(-0.5, 0.5, (2, 1)) if j % 3 == 1 else np.zeros((2, 1))
        if j % 3 == 0:
            obs.append(Obs(c, float(rng.uniform(0.3, 1.0)), None, 'norm2', vel))
        else:
            n = int(rng.integers(3, 5))
            ang = np.linspace(0, 2 * np.pi, n, endpoint=False) + rng.uniform(0, 1)
            if j % 2:
                ang = ang[::-1]
            obs.append(Obs(None, None, c + rng.uniform(0.5, 1.2) * np.vstack([np.cos(ang), np.sin(ang)]), 'Rpositive', vel))
    obs = [o._replace(center=None if o.center is None else o.center.astype(np.float32).astype(float),
                      vertex=None if o.vertex is None else o.vertex.astype(np.float32).astype(float),
                      velocity=o.velocity.astype(np.float32).astype(float)) for o in obs]
    car = rectangle_robot()
    T, N, E, steps = 10, 4, 4, 4
    starts = [0, 25, 40, len(PATH) - 12]
    B = len(starts)
    states = np.stack([PATH_ARR[i] + np.array([0.2, -0.1, 0.05]) for i in starts]).astype(np.float32)
    kw = dict(receding=T, sample_time=DT, iter_num=3, max_edge_num=E, max_obs_num=N, iter_threshold=0.0)
    bm = BatchedMPC(car, PATH, B, **kw)
    bm.cur_index[:] = torch.as_tensor(starts, dtype=torch.int32)
    hosts = []
    for i in starts:
        m = MPC(car, copy.deepcopy(PATH), time_print=False, **kw)
        m.cur_index = i
        hosts.append(m)
    dev_state = torch.as_tensor(states, device=DEV)
    host_state = [states[i].astype(float).reshape(3, 1) for i in range(B)]
    world = _dev(pack_worlds([obs]))
    with pytest.raises(ValueError):
        bm.control(dev_state, 4.0, world, world=world)
    for k in range(steps):
        u0, info = bm.control(dev_state, 4.0, time_varying=True, world=world)
        u0 = u0.cpu().numpy()
        arrive = info['arrive'].cpu().numpy()
        for i, m in enumerate(hosts):
            uh, ih = m.control(host_state[i], 4.0, obs)
            assert bool(arrive[i]) == ih['arrive']
            assert int(info['cur_index'][i]) == m.cur_index
            np.testing.assert_allclose(u0[i], uh[:, 0], atol=2e-3)
            s = host_state[i]
            host_state[i] = s + 0.1 * np.array([[uh[0, 0] * np.cos(s[2, 0])], [uh[0, 0] * np.sin(s[2, 0])], [uh[0, 0] * np.tan(uh[1, 0]) / 3.0]])
        bm.advance(dev_state)
        np.testing.assert_allclose(dev_state.cpu().numpy(), np.hstack(host_state).T, atol=2e-3)


def test_batched_mpc_needs_robot_world_with_several_maps():
    from rda_planner_b200.frontend import BatchedMPC, pack_worlds
    bm = BatchedMPC(rectangle_robot(), PATH, 2, receding=8, iter_num=2, max_obs_num=3, max_edge_num=4)
    two = _dev(pack_worlds([_shared_world(np.random.default_rng(0), 5, 0, 60), []]))
    state = torch.as_tensor(np.stack([PATH_ARR[0], PATH_ARR[5]]).astype(np.float32), device=DEV)
    with pytest.raises(ValueError):
        bm.control(state, 4.0, world=two)
    u0, info = bm.control(state, 4.0, world=two, robot_world=[1, 0])
    assert info['arrive'].shape == (2,)
