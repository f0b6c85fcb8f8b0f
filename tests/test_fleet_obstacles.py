"""Robots of a fleet as moving obstacles of each other (rda_fleet_shapes, rda_convert_fleet_obstacles): the CPU twin
of the body placement (tests/cpu_twin/fleet_obstacles.cpp) against numpy, each robot's selection (the world twin over
its world's shapes followed by its map-mates) against the host front end given the same robots as obstacle tuples,
the world -> robots lists, BatchedMPC's refusals and the entry points' usage errors.  No GPU."""
import ctypes
from collections import namedtuple

import numpy as np
import pytest
import torch

import fleet_obstacles_twin as ft
from rda_planner_b200 import _cabi
from rda_planner_b200 import frontend
from rda_planner_b200.frontend import fleet_csr, pack_worlds, robot_body
from rda_planner_b200.mpc import MPC
from rda_planner_b200.rda_solver import pack_obstacles
from rda_planner_b200.scenarios import rectangle_robot

car = namedtuple('car', 'G h cone_type wheelbase max_speed max_acce dynamics')
Obs = namedtuple('Obs', 'center radius vertex cone_type velocity')
DISC = car(np.array([[1.0, 0], [0, 1], [0, 0]]), np.array([0.0, 0.0, -0.6]), 'norm2', 1.0, [2, 2], [1, 1], 'omni')
PENTAGON_V = np.array([[0.9, 0.0], [0.3, 0.7], [-0.6, 0.5], [-0.6, -0.5], [0.3, -0.7]])


class _NoSolver:
    def __init__(self, *a, **k):
        pass


def _pentagon(dynamics):
    # rows of the counter-clockwise pentagon: edge i -> i+1 has outward normal (dy, -dx)
    V = PENTAGON_V
    E = np.roll(V, -1, axis=0) - V
    G = np.stack([E[:, 1], -E[:, 0]], 1)
    h = (G * V).sum(1)
    return car(G, h, 'Rpositive', 1.0, [2, 2], [1, 1], dynamics)


def _f32(a):
    return np.asarray(a, float).astype(np.float32).astype(float)


def numpy_shape(body, state, u, dynamics):
    """Robot at `state` with applied control u = (v, w or psi) as the obstacle tuple a host MPC would be handed."""
    px, py, th = (float(x) for x in state)
    R = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
    d = u[1] if dynamics == 'omni' else th
    vel = _f32(u[0] * np.array([[np.cos(d)], [np.sin(d)]]))
    if body['kind'] == _cabi.OBS_CIRCLE:
        c = _f32(np.array([[px], [py]]) + R @ body['xy'][0].astype(float).reshape(2, 1))
        return Obs(c, float(body['radius']), None, 'norm2', vel)
    V = body['xy'][:body['nv']].astype(float).T
    return Obs(None, None, _f32(np.array([[px], [py]]) + R @ V), 'Rpositive', vel)


def test_robot_body_is_the_counter_clockwise_outline():
    rect = robot_body(rectangle_robot())
    G, h = np.asarray(rectangle_robot().G, float), np.asarray(rectangle_robot().h, float).reshape(-1)
    V = rect['xy'][:rect['nv']].astype(float)
    assert rect['kind'] == _cabi.OBS_POLYGON and rect['nv'] == 4 and not rect['xy'][4:].any()
    assert np.all(V @ G.T <= h + 1e-6)                                            # every vertex inside every row
    assert np.sum([np.isclose(V @ G[j], h[j], atol=1e-6).sum() for j in range(4)]) == 8   # two per edge
    x, y = V[:, 0], V[:, 1]
    assert 0.5 * np.sum(x * np.roll(y, -1) - np.roll(x, -1) * y) > 0               # counter-clockwise
    pent = robot_body(_pentagon('diff'))
    np.testing.assert_allclose(pent['xy'][:5], PENTAGON_V, atol=1e-6)
    disc = robot_body(DISC)
    assert disc['kind'] == _cabi.OBS_CIRCLE and disc['nv'] == 0 and disc['radius'] == np.float32(0.6)
    assert not disc['xy'].any()


@pytest.mark.parametrize('dynamics', ['acker', 'diff', 'omni'])
@pytest.mark.parametrize('body', ['pentagon', 'disc'])
def test_twin_fleet_shapes_match_numpy(body, dynamics):
    rng = np.random.default_rng(3)
    bd = robot_body(_pentagon(dynamics) if body == 'pentagon' else DISC._replace(h=np.array([0.2, -0.1, -0.6])))
    B, T = 40, 6
    state = np.c_[rng.uniform(-50, 50, (B, 2)), rng.uniform(-np.pi, np.pi, B)].astype(np.float32)
    cur_vel = rng.uniform(-2, 2, (B, 2, T)).astype(np.float32)
    cur_vel[:8, 0, 0] = 0.0                                       # standing still
    cur_vel[8:16, 0, 0] = rng.uniform(-0.01, 0.01, 8)             # below the 0.01 moving threshold
    got = ft.fleet_shapes(state, cur_vel, bd, dynamics)
    assert (got['kind'] == bd['kind']).all() and (got['nv'] == bd['nv']).all()
    for m in range(B):
        o = numpy_shape(bd, state[m], cur_vel[m, :, 0].astype(float), dynamics)
        np.testing.assert_allclose(got['vel'][m], o.velocity.ravel(), rtol=1e-6, atol=1e-7)
        if body == 'disc':
            np.testing.assert_allclose(got['xy'][m, 0], o.center.ravel(), rtol=1e-6, atol=1e-6)
            assert got['radius'][m] == np.float32(0.6) and not got['xy'][m, 1:].any()
        else:
            np.testing.assert_allclose(got['xy'][m, :5], o.vertex.T, rtol=1e-6, atol=1e-6)
            assert got['radius'][m] == 0 and not got['xy'][m, 5:].any()
    assert not got['vel'][:8].any()
    assert (np.hypot(got['vel'][8:16, 0], got['vel'][8:16, 1]) <= 0.01).all()


def _world(rng, count, spread):
    obs = []
    for j in range(count):
        vel = rng.uniform(-1, 1, (2, 1)) if j % 2 else np.zeros((2, 1))
        c = rng.uniform(-spread, spread, (2, 1))
        if j % 3 == 0:
            obs.append(Obs(_f32(c), float(np.float32(rng.uniform(0.3, 1.0))), None, 'norm2', _f32(vel)))
        else:
            n = int(rng.integers(3, 6))
            ang = np.linspace(0, 2 * np.pi, n, endpoint=False) + rng.uniform(0, 1)
            if j % 4 == 1:
                ang = ang[::-1]
            obs.append(Obs(None, None, _f32(c + rng.uniform(0.4, 1.5) * np.vstack([np.cos(ang), np.sin(ang)])),
                           'Rpositive', _f32(vel)))
    return obs


def _fleet_case(rng, body_car):
    """Four worlds (40 shapes and 5 robots, an empty map with 3, 25 shapes and one robot, 10 shapes and none) and two
    robots outside them.  Then two exact key ties between a world shape and a map-mate."""
    worlds = [_world(rng, 40, 12.0), [], _world(rng, 25, 12.0), _world(rng, 10, 12.0)]
    rw = np.array([0, 1, 0, 2, 0, -1, 1, 0, 4, 1, 0], np.int32)
    B = len(rw)
    state = np.c_[rng.uniform(-5, 5, (B, 2)), rng.uniform(-np.pi, np.pi, B)].astype(np.float32)
    cur_vel = rng.uniform(-1.5, 1.5, (B, 2, 6)).astype(np.float32)
    cur_vel[3, 0, 0] = 0.0
    cur_vel[4, 0, 0] = 0.004
    # ties: robot 0 at the origin; robot 2 placed with heading 0 (exact rotation) 3 m along +x; a world shape mirrored
    # across the line y = x sits at exactly the same key
    state[0] = (0.0, 0.0, 0.3)
    state[2] = (3.0, 0.0, 0.0)
    bd = robot_body(body_car)
    mate = numpy_shape(bd, state[2], cur_vel[2, :, 0].astype(float), body_car.dynamics)
    if mate.cone_type == 'norm2':
        twin = Obs(mate.center[::-1].copy(), mate.radius, None, 'norm2', np.zeros((2, 1)))
    else:
        twin = Obs(None, None, mate.vertex[::-1].copy(), 'Rpositive', np.zeros((2, 1)))
    worlds[0] = worlds[0][:20] + [twin] + worlds[0][20:]
    return worlds, rw, state, cur_vel, bd


@pytest.mark.parametrize('order', [True, False])
@pytest.mark.parametrize('N', [6, 30])
@pytest.mark.parametrize('body', ['rectangle', 'disc'])
def test_each_robot_matches_host_front_end_with_its_mates_as_obstacles(body, N, order):
    rng = np.random.default_rng(11)
    body_car = rectangle_robot() if body == 'rectangle' else DISC
    dyn = body_car.dynamics
    worlds, rw, state, cur_vel, bd = _fleet_case(rng, body_car)
    T, E = 6, 5
    world = pack_worlds(worlds)
    fleet = ft.fleet_shapes(state, cur_vel, bd, dyn)
    mates_obs = [numpy_shape(bd, state[m], cur_vel[m, :, 0].astype(float), dyn) for m in range(len(rw))]
    for b in range(len(rw)):
        w = int(rw[b])
        inside = 0 <= w < len(worlds)
        obs = (list(worlds[w]) + [mates_obs[m] for m in range(len(rw)) if rw[m] == w and m != b]) if inside else []
        m = MPC(car(None, None, 'Rpositive', 3.0, [10, 1], [10, 0.5], dyn), [], receding=T, sample_time=0.1,
                solver_cls=_NoSolver)
        st = state[b].astype(float).reshape(3, 1)
        m.state = st
        rda_obs = m.convert_rda_obstacle(obs, st, order)
        tv = any(isinstance(o.A, list) for o in rda_obs[:N])
        A, bb, kind, cnt = ft.convert_fleet_obstacles(world, fleet, rw, b, N, T, E, 0.1, tv, order, state[b])
        assert cnt == len(obs), b
        if not obs:
            assert not A.any() and not bb.any() and list(kind) == [_cabi.OBS_POLYGON] * N
            continue
        Ah, bh, kh, ch, tvh = pack_obstacles(list(rda_obs), T, N, E)
        assert ch == cnt
        assert list(kind) == list(kh), b
        np.testing.assert_allclose(A, Ah, atol=1e-5)
        np.testing.assert_allclose(bb, bh, atol=1e-4)
    # the tie: robot 0's list has the mirrored world shape (position 20) before robot 2, at the same key
    m = MPC(car(None, None, 'Rpositive', 3.0, [10, 1], [10, 0.5], dyn), [], receding=T, solver_cls=_NoSolver)
    m.state = state[0].astype(float).reshape(3, 1)
    lst = ft.robot_list(world, fleet, rw, 0)
    assert int(lst['start'][1]) == 41 + 4                         # 41 shapes, then robots 2, 4, 7, 10
    keys = [m.rda_obs_distance(o) for o in m.convert_rda_obstacle(worlds[0] + [mates_obs[2]], m.state)]
    assert keys[20] == keys[41]


def test_world_robot_lists():
    rw = torch.tensor([2, 0, -1, 2, 5, 0, 2, 3, 0], dtype=torch.int32)
    start, robots = fleet_csr(rw, 4)
    assert start.dtype == torch.int32 and robots.dtype == torch.int32
    assert start.tolist() == [1, 4, 4, 7, 8]                     # robots 2 (-1) and 4 (5) lie outside [start[0], start[W])
    got = robots.tolist()
    assert got[1:4] == [1, 5, 8] and got[4:7] == [0, 3, 6] and got[7:8] == [7]
    assert sorted(got) == list(range(9))
    start1, robots1 = fleet_csr(torch.zeros(5, dtype=torch.int32), 1)
    assert start1.tolist() == [0, 5] and robots1.tolist() == [0, 1, 2, 3, 4]


class _StubSolver:
    """Enough of RDA_solver for BatchedMPC's argument checks, without a device."""
    def __init__(self, receding, car_tuple, max_edge_num, max_obs_num, **kw):
        self.device = torch.device('cpu')
        self.max_edge_num = max(max_edge_num, 3)


def test_batched_mpc_refusals(monkeypatch):
    monkeypatch.setattr(frontend, 'RDA_solver', _StubSolver)
    path = np.stack([np.arange(10.0), np.zeros(10), np.zeros(10)], 1)
    bm = frontend.BatchedMPC(rectangle_robot(), path, 2, receding=4, max_edge_num=4, max_obs_num=3)
    state = np.zeros((2, 3), np.float32)
    shapes = frontend.pack_shapes([[], []])
    with pytest.raises(ValueError, match='shapes'):
        bm.control(state, 1.0, shapes=shapes, avoid_fleet=True)
    small = frontend.BatchedMPC(_pentagon('diff'), path, 2, receding=4, max_edge_num=4, max_obs_num=3)
    with pytest.raises(ValueError, match='max_edge_num=4'):
        small.control(state, 1.0, avoid_fleet=True)


def test_fleet_usage_errors_are_return_codes():
    """Checked before any device work, so this runs without a GPU."""
    lib = _cabi.load()
    fs = lib.rda_fleet_shapes
    fake = ctypes.c_void_p(256)
    P, D = _cabi.OBS_POLYGON, _cabi.OBS_CIRCLE
    nul = [None] * 8
    assert fs(0, 4, 0, P, 4, None, 0.0, *nul) == -1                 # B < 1
    assert fs(4, 0, 0, P, 4, None, 0.0, *nul) == -1                 # T < 1
    assert fs(4, 4, 3, P, 4, None, 0.0, *nul) == -1                 # unknown dynamics
    assert fs(4, 4, 0, 2, 4, None, 0.0, *nul) == -1                 # unknown body kind
    assert fs(4, 4, 0, P, 2, None, 0.0, *nul) == -2                 # polygon below 3 vertices
    assert fs(4, 4, 0, P, _cabi.MAX_EDGE + 1, None, 0.0, *nul) == -2
    assert fs(4, 4, 0, D, 0, None, 0.0, *nul) == -1                 # disc without a radius
    assert fs(4, 4, 0, P, 4, None, 0.0, *nul) == -1                 # missing pointers
    cf = lib.rda_convert_fleet_obstacles
    assert cf(0, 1, 5, 10, 4, 0.1, 0, 1, *[None] * 20) == -1        # B < 1
    assert cf(4, 1, _cabi.MAX_WORLD_SLOTS + 1, 10, 4, 0.1, 0, 1, *[None] * 20) == -2
    assert cf(4, 1, 5, 10, 2, 0.1, 0, 1, *[None] * 20) == -2        # E < 3
    if torch.cuda.is_available():                     # below, a missing check would launch on placeholder pointers
        return
    for missing in range(8):                                        # body_xy, state, cur_vel or an output
        p = [fake] * 8
        p[missing] = None
        assert fs(4, 4, 0, P, 4, p[0], 0.0, *p[1:], None) == -1, missing
    ptrs = [fake] * 19 + [None]
    for missing in [0, 1] + list(range(3, 19)):                     # all but robot_world (2), which may be NULL
        p = list(ptrs)
        p[missing] = None
        assert cf(4, 1, 5, 10, 4, 0.1, 0, 1, *p) == -1, missing
