"""Robots of a fleet as moving obstacles of each other on the device (rda_fleet_shapes, rda_convert_fleet_obstacles):
the kernels against their CPU twins on random fleets, the one-robot-per-world case against rda_convert_world_obstacles,
a 16 384-robot fleet against each world alone, BatchedMPC(avoid_fleet=True) against host MPCs handed the other robots
as obstacle tuples, a step without host synchronisation, and two robots that meet at a crossing."""
import copy
from collections import namedtuple

import numpy as np
import pytest
import torch

import fleet_obstacles_twin as ft
from rda_planner_b200.frontend import (BatchedMPC, convert_fleet_obstacles_batch, convert_world_obstacles_batch,
                                       fleet_shapes_batch, pack_worlds, robot_body, shapes_to_device)
from rda_planner_b200.mpc import MPC
from rda_planner_b200.scenarios import disc_robot, rectangle_robot

pytestmark = pytest.mark.gpu
Obs = namedtuple('Obs', 'center radius vertex cone_type velocity')
DEV = torch.device('cuda:0')
DT = 0.1
DT32 = float(np.float32(DT))
KEYS = ('kind', 'nv', 'xy', 'radius', 'vel')


def _t(a, dtype=None):
    return torch.as_tensor(np.asarray(a), device=DEV, dtype=dtype).contiguous()


def _dev_body(body):
    return dict(body, xy=_t(body['xy']))


def _world(rng, count, lo, hi):
    """`count` shapes over a square: discs and 3..8-gons, CW and CCW, a third moving, some exact duplicates."""
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
            obs.append(Obs(None, None, c + rng.uniform(0.4, 2.0) * np.vstack([np.cos(ang), np.sin(ang)]), 'Rpositive',
                           vel))
    return obs


def _fleet(rng, B, W, span):
    rw = rng.integers(0, W, B).astype(np.int32)
    rw[:4] = [-1, W, 1 << 30, -(1 << 30)]                       # in no world
    state = np.c_[rng.uniform(0, span, (B, 2)), rng.uniform(-np.pi, np.pi, B)].astype(np.float32)
    cur_vel = rng.uniform(-2, 2, (B, 2, 6)).astype(np.float32)
    cur_vel[rng.random(B) < 0.1, 0, 0] = 0.0                       # standing (or arrived)
    slow = rng.random(B) < 0.1
    cur_vel[slow, 0, 0] = rng.uniform(-0.01, 0.01, int(slow.sum()))  # below the moving threshold
    return rw, state, cur_vel


def _run(world_dev, state, rw, cur_vel, body, dyn, N, T, E, tv, order):
    st = _t(state)
    fleet = fleet_shapes_batch(st, _t(cur_vel), _dev_body(body), dyn)
    out = convert_fleet_obstacles_batch(world_dev, st, _t(rw), fleet, N, T, E, DT, tv, order)
    return {k: v.cpu().numpy() for k, v in fleet.items()}, [o.cpu().numpy() for o in out]


@pytest.mark.parametrize('N', [1, 20, 128])
@pytest.mark.parametrize('tv,order', [(False, False), (False, True), (True, False), (True, True)])
def test_fleet_kernels_match_cpu_twins(tv, order, N):
    """~1 000 robots in six worlds of 0 to 2 000 shapes (and robots in none); rectangle body, acker."""
    rng = np.random.default_rng(31)
    sizes = [0, 2000, 17, 400, 1, 1200]
    worlds = [_world(rng, n, 0.0, 80.0) for n in sizes]
    host = pack_worlds(worlds)
    B, T, E = 1000, 6, 8
    rw, state, cur_vel = _fleet(rng, B, len(sizes), 80.0)
    body = robot_body(rectangle_robot())
    fleet, (A, b, kind, count) = _run(shapes_to_device(host, DEV), state, rw, cur_vel, body, 'acker', N, T, E, tv, order)
    want = ft.fleet_shapes(state, cur_vel, body, 'acker')
    for k in ('kind', 'nv', 'radius'):
        np.testing.assert_array_equal(fleet[k], want[k])
    np.testing.assert_allclose(fleet['xy'], want['xy'], rtol=1e-6, atol=1e-5)
    np.testing.assert_allclose(fleet['vel'], want['vel'], rtol=1e-6, atol=1e-6)
    for i in range(B):                                             # selection and rows from the kernel's own shapes
        A1, b1, k1, c1 = ft.convert_fleet_obstacles(host, fleet, rw, i, N, T, E, DT32, tv, order, state[i])
        w = int(rw[i])
        assert count[i] == c1 == ((sizes[w] + int((rw == w).sum()) - 1) if 0 <= w < len(sizes) else 0), i
        assert list(kind[i]) == list(k1), i
        np.testing.assert_array_equal(A[i], A1)
        np.testing.assert_allclose(b[i], b1, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize('dyn,body', [('diff', 'disc'), ('omni', 'disc'), ('omni', 'rectangle')])
def test_fleet_shapes_of_other_bodies_match_twin(dyn, body):
    rng = np.random.default_rng(7)
    B = 4096
    _, state, cur_vel = _fleet(rng, B, 1, 500.0)
    bd = robot_body(disc_robot(0.7, (0.2, -0.1)) if body == 'disc' else rectangle_robot())
    got = fleet_shapes_batch(_t(state), _t(cur_vel), _dev_body(bd), dyn)
    want = ft.fleet_shapes(state, cur_vel, bd, dyn)
    for k in KEYS:
        np.testing.assert_allclose(got[k].cpu().numpy(), want[k], rtol=1e-6, atol=1e-4 if k == 'xy' else 1e-6)


@pytest.mark.parametrize('tv,order', [(False, True), (True, True), (True, False)])
def test_one_robot_per_world_equals_world_conversion(tv, order):
    rng = np.random.default_rng(12)
    B, T, N, E = 97, 10, 20, 8
    lists = [_world(rng, int(c), 0.0, 40.0) for c in rng.integers(0, 300, B)]
    lists[0] = []
    world = shapes_to_device(pack_worlds(lists), DEV)
    state = _t(np.c_[rng.uniform(0, 40, (B, 2)), rng.uniform(-3, 3, B)].astype(np.float32))
    rw = torch.arange(B, dtype=torch.int32, device=DEV)
    rw[5] = -1
    ref = convert_world_obstacles_batch(world, state, rw, N, T, E, DT, tv, order)
    fleet = fleet_shapes_batch(state, _t(rng.uniform(-2, 2, (B, 2, T)).astype(np.float32)),
                               _dev_body(robot_body(rectangle_robot())), 'acker')
    got = convert_fleet_obstacles_batch(world, state, rw, fleet, N, T, E, DT, tv, order)
    for r, g in zip(ref, got):
        assert torch.equal(r, g)


def test_16384_robots_in_64_worlds_equal_each_world_alone():
    """64 worlds of 1 024 shapes and 256 robots each (robots interleaved across the batch): every robot's arrays are
    bit for bit what the same kernels write when its world is converted as a batch of its own."""
    rng = np.random.default_rng(64)
    W, per, S, N, T, E = 64, 256, 1024, 20, 5, 8
    B = W * per
    rw = rng.permutation(np.repeat(np.arange(W, dtype=np.int32), per))
    worlds = [_world(rng, S, 0.0, 100.0) for _ in range(W)]
    host = pack_worlds(worlds)
    state = np.c_[rng.uniform(0, 100, (B, 2)), rng.uniform(-np.pi, np.pi, B)].astype(np.float32)
    cur_vel = rng.uniform(-2, 2, (B, 2, T)).astype(np.float32)
    body = robot_body(rectangle_robot())
    _, full = _run(shapes_to_device(host, DEV), state, rw, cur_vel, body, 'acker', N, T, E, True, True)
    assert (full[3] == S + per - 1).all()
    for w in range(W):
        idx = np.nonzero(rw == w)[0]
        one = {k: host[k][host['start'][w]:host['start'][w + 1]] for k in KEYS}
        one['start'] = np.array([0, S], np.int32)
        _, alone = _run(shapes_to_device(one, DEV), state[idx], np.zeros(per, np.int32), cur_vel[idx], body, 'acker',
                        N, T, E, True, True)
        for f, a in zip(full, alone):
            np.testing.assert_array_equal(f[idx], a)


# ---- BatchedMPC(avoid_fleet=True) ----------------------------------------------------------------------------------
def _line(x0, y0, heading, n, step=0.5):
    return [np.array([[x0 + step * i * np.cos(heading)], [y0 + step * i * np.sin(heading)], [heading]])
            for i in range(n)]


def _host_obstacle(body, s, u):
    """Robot at host state s (3, 1) that last applied u (2, 1), as a host simulator reports it (acker / diff)."""
    th = float(s[2, 0])
    R = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
    vel = float(u[0, 0]) * np.array([[np.cos(th)], [np.sin(th)]])
    V = s[:2] + R @ body['xy'][:body['nv']].astype(float).T
    return Obs(None, None, V, 'Rpositive', vel)


def test_closed_loop_with_fleet_avoidance_matches_host_mpcs():
    """Six robots on their own paths in two shared maps, time-varying obstacles, 4 steps: each host mpc.MPC gets its
    map plus the other robots of its map, built from the host states and controls."""
    car = rectangle_robot()
    T, N, E, steps, speed = 10, 4, 4, 4, 3.0
    rng = np.random.default_rng(9)
    maps = [_world(rng, 60, -5.0, 40.0), _world(rng, 30, -5.0, 40.0)]
    maps = [[o for o in m if o.center is None or abs(o.center[1, 0]) > 9] for m in maps]      # off the lanes
    maps = [[o for o in m if o.vertex is None or (np.abs(o.vertex[1]).min() > 9 and o.vertex.shape[1] <= E)]
            for m in maps]
    maps = [[o._replace(center=None if o.center is None else o.center.astype(np.float32).astype(float),
                        vertex=None if o.vertex is None else o.vertex.astype(np.float32).astype(float),
                        velocity=o.velocity.astype(np.float32).astype(float)) for o in m] for m in maps]
    paths = [_line(0.0, -3.0, 0.0, 80), _line(0.0, 0.0, 0.0, 80), _line(0.0, 3.0, 0.02, 80), _line(2.0, -6.0, 0.3, 80)]
    robot_path = [0, 1, 2, 0, 3, 1]
    robot_world = [0, 0, 0, 1, 1, 1]
    starts = [4, 2, 6, 3, 0, 8]
    B = len(robot_path)
    kw = dict(receding=T, sample_time=DT, iter_num=3, max_edge_num=E, max_obs_num=N, iter_threshold=0.0)
    bm = BatchedMPC(car, paths, B, robot_path=robot_path, **kw)
    bm.cur_index[:] = _t(starts, torch.int32)
    hosts, host_state = [], []
    for b in range(B):
        m = MPC(car, copy.deepcopy(paths[robot_path[b]]), time_print=False, **kw)
        m.cur_index = starts[b]
        hosts.append(m)
        wp = np.asarray(paths[robot_path[b]][starts[b]], float).reshape(-1)[:3]
        host_state.append((wp + np.array([0.1, -0.05, 0.02])).reshape(3, 1))
    host_u = [np.zeros((2, 1)) for _ in range(B)]
    body = bm.body
    body_h = dict(body, xy=body['xy'].cpu().numpy())
    world = shapes_to_device(pack_worlds(maps), DEV)
    dev_state = _t(np.hstack(host_state).T.astype(np.float32))
    for k in range(steps):
        u0, info = bm.control(dev_state, speed, time_varying=True, world=world, robot_world=robot_world,
                              avoid_fleet=True)
        u0 = u0.cpu().numpy()
        assert list(info['status'].cpu().numpy() & 6) == [0] * B
        mates = [_host_obstacle(body_h, host_state[m], host_u[m]) for m in range(B)]
        new_u = []
        for b, m in enumerate(hosts):
            others = [mates[j] for j in range(B) if robot_world[j] == robot_world[b] and j != b]
            uh, ih = m.control(host_state[b], speed, maps[robot_world[b]] + others)
            assert bool(info['arrive'][b]) == ih['arrive']
            assert int(info['cur_index'][b]) == m.cur_index
            np.testing.assert_allclose(u0[b], uh[:, 0], atol=2e-3, err_msg=f'{k} {b}')
            new_u.append(uh[:, :1])
        for b in range(B):
            s, u = host_state[b], new_u[b]
            host_state[b] = s + DT * np.array([[u[0, 0] * np.cos(s[2, 0])], [u[0, 0] * np.sin(s[2, 0])],
                                               [u[0, 0] * np.tan(u[1, 0]) / car.wheelbase]])
        host_u = new_u
        bm.advance(dev_state)
        np.testing.assert_allclose(dev_state.cpu().numpy(), np.hstack(host_state).T, atol=2e-3)


def test_fleet_step_needs_no_host_sync():
    car = rectangle_robot()
    B = 48
    paths = [_line(0.0, -1.0, 0.0, 50), _line(0.0, 2.5, 0.05, 50)]
    bm = BatchedMPC(car, paths, B, robot_path=np.arange(B) % 2, receding=8, iter_num=2, max_edge_num=4,
                    max_obs_num=4)
    world = shapes_to_device(pack_worlds([_world(np.random.default_rng(0), 50, 0, 30), []]), DEV)
    rw = _t(np.arange(B) % 3 - (np.arange(B) == 7), torch.int32)       # worlds 0, 1 and none (2, -1)
    state = _t(np.stack([[0.3 * (b % 16), 0.0, 0.0] for b in range(B)]).astype(np.float32))
    bm.control(state, 2.0, world=world, robot_world=rw, avoid_fleet=True)
    bm.control(state, 2.0, avoid_fleet=True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        u0, info = bm.control(state, 2.0, world=world, robot_world=rw, time_varying=True, avoid_fleet=True)
        bm.advance(state)
        u1, _ = bm.control(state, 2.0, avoid_fleet=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(u0).all()) and bool(torch.isfinite(u1).all())


def _corners(body, s):
    th = float(s[2])
    R = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
    return np.asarray(s[:2], float) + body['xy'][:body['nv']].astype(float) @ R.T


def _overlap(P, Q):
    """Separating-axis test of two convex polygons [n, 2]."""
    for poly in (P, Q):
        e = np.roll(poly, -1, axis=0) - poly
        for n in np.stack([e[:, 1], -e[:, 0]], 1):
            if (P @ n).max() < (Q @ n).min() or (Q @ n).max() < (P @ n).min():
                return False
    return True


CROSS = dict(speed=2.0, start=8.0, lag=1.0, steps=100)


def _crossing(avoid, lag=None):
    """Two robots on perpendicular lanes at the same speed, `start` m and `start` + `lag` m before the crossing: without
    seeing each other they are there together (the bodies are 2 m long)."""
    car = rectangle_robot(length=2.0, width=1.0, wheelbase=1.2, dynamics='diff', max_speed=(3, 1.5), max_acce=(3, 1.5))
    L = CROSS['start']
    L1 = L + (CROSS['lag'] if lag is None else lag)
    n = int(4 * L / 0.25)
    paths = [_line(-L, 0.0, 0.0, n, step=0.25), _line(0.0, -L1, np.pi / 2, n, step=0.25)]
    bm = BatchedMPC(car, paths, 2, robot_path=[0, 1], receding=12, sample_time=DT, iter_num=4, max_edge_num=4,
                    max_obs_num=3, iter_threshold=0.0)
    state = _t(np.array([[-L, 0.0, 0.0], [0.0, -L1, np.pi / 2]], np.float32))
    body = dict(bm.body, xy=bm.body['xy'].cpu().numpy())
    traj = [state.cpu().numpy().copy()]
    for _ in range(CROSS['steps']):
        bm.control(state, CROSS['speed'], time_varying=True, avoid_fleet=avoid)
        bm.advance(state)
        traj.append(state.cpu().numpy().copy())
    traj = np.stack(traj)
    hit = [_overlap(_corners(body, s[0]), _corners(body, s[1])) for s in traj]
    return traj, hit


def test_two_robots_at_a_crossing_avoid_each_other():
    traj, hit = _crossing(False)
    assert any(hit)                                                  # blind to each other, they collide
    traj, hit = _crossing(True)
    assert not any(hit)
    assert traj[-1, 0, 0] > 4.0 and traj[-1, 1, 1] > 4.0              # both well past the crossing
