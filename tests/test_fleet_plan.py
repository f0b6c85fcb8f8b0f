"""Robots of a fleet as obstacles of each other predicted along their plans (rda_fleet_plan_shapes,
rda_convert_fleet_plan_obstacles): the CPU twin of the rollout and placement (tests/cpu_twin/fleet_plan.cpp) against a
numpy restatement built on the host MPC's own model steps, each robot's selection against the host front end handed the
reference-terms list (its world's shapes, then every map-mate as an rdaobs whose A and b are lists of T+1 arrays),
BatchedMPC's refusals and the entry points' usage errors.  No GPU."""
import ctypes
from collections import namedtuple

import numpy as np
import pytest
import torch

import fleet_obstacles_twin as ft
import fleet_plan_twin as fp
from rda_planner_b200 import _cabi
from rda_planner_b200 import frontend
from rda_planner_b200.frontend import pack_worlds, robot_body
from rda_planner_b200.mpc import MPC, rdaobs
from rda_planner_b200.rda_solver import pack_obstacles
from rda_planner_b200.scenarios import rectangle_robot

car = namedtuple('car', 'G h cone_type wheelbase max_speed max_acce dynamics')
Obs = namedtuple('Obs', 'center radius vertex cone_type velocity')
DISC = car(np.array([[1.0, 0], [0, 1], [0, 0]]), np.array([0.2, -0.1, -0.6]), 'norm2', 1.0, [2, 2], [1, 1], 'omni')
PENTAGON_V = np.array([[0.9, 0.0], [0.3, 0.7], [-0.6, 0.5], [-0.6, -0.5], [0.3, -0.7]])
DT = 0.1


class _NoSolver:
    def __init__(self, *a, **k):
        pass


def _pentagon(dynamics):
    V = PENTAGON_V
    E = np.roll(V, -1, axis=0) - V
    G = np.stack([E[:, 1], -E[:, 0]], 1)
    return car(G, (G * V).sum(1), 'Rpositive', 1.0, [2, 2], [1, 1], dynamics)


def _f32(a):
    return np.asarray(a, float).astype(np.float32).astype(float)


def _host_mpc(dynamics, L, T):
    return MPC(car(None, None, 'Rpositive', L, [10, 1], [10, 0.5], dynamics), [], receding=T, sample_time=DT,
               solver_cls=_NoSolver)


def numpy_poses(state, u, dynamics, L):
    """q(0) = state, q(t+1) = the host model step (mpc.MPC.motion_predict_model_*) with u[:, min(t + 1, T - 1)]."""
    T = u.shape[1]
    m = _host_mpc(dynamics, L, T)
    q = np.asarray(state, float).reshape(3, 1)
    poses = [q]
    for t in range(T):
        c = min(t + 1, T - 1)
        v = np.asarray(u, float)[:, c:c + 1]
        if dynamics == 'acker':
            q = m.motion_predict_model_acker(q, v, L, DT)
        elif dynamics == 'diff':
            q = m.motion_predict_model_diff(q, v, DT)
        else:
            q = m.motion_predict_model_omni(q, v, DT)
        poses.append(q)
    return poses


def numpy_place(body, q):
    """The body at pose q in float64: polygon vertices [2, nv] or the disc centre [2, 1]."""
    th = float(q[2, 0])
    R = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
    n = 1 if body['kind'] == _cabi.OBS_CIRCLE else body['nv']
    return q[:2] + R @ np.asarray(body['xy'][:n], float).T


def numpy_plan(body, state, u, dynamics, L):
    """[T+1, 8, 2] float64: the body at every predicted pose, rows beyond the shape's zero."""
    out = np.zeros((u.shape[1] + 1, 8, 2))
    for t, q in enumerate(numpy_poses(state, u, dynamics, L)):
        V = numpy_place(body, q)
        out[t, :V.shape[1]] = V.T
    return out


def mate_rdaobs(m, body, plan):
    """A map-mate predicted along its plan in the reference's terms: rdaobs with A and b lists of T+1 arrays, the rows of
    its float32 shape at each stage (MPC.convert_inequal_*, standing), and its stage-0 centre or vertices."""
    A, b = [], []
    if body['kind'] == _cabi.OBS_CIRCLE:
        for p in plan:
            At, bt = m.convert_inequal_circle(_f32(p[0]).reshape(2, 1), float(body['radius']))
            A.append(At)
            b.append(bt)
        return rdaobs(A, b, 'norm2', _f32(plan[0, 0]).reshape(2, 1), None)
    nv = body['nv']
    for p in plan:
        At, bt = m.convert_inequal_polygon(_f32(p[:nv]).T)
        A.append(At)
        b.append(bt)
    return rdaobs(A, b, 'Rpositive', None, _f32(plan[0, :nv]).T)


@pytest.mark.parametrize('dynamics', ['acker', 'diff', 'omni'])
@pytest.mark.parametrize('body', ['pentagon', 'disc'])
def test_twin_plan_matches_numpy(body, dynamics):
    rng = np.random.default_rng(5)
    bd = robot_body(_pentagon(dynamics) if body == 'pentagon' else DISC)
    B, T, L = 40, 12, 1.7
    state = np.c_[rng.uniform(-50, 50, (B, 2)), rng.uniform(-np.pi, np.pi, B)].astype(np.float32)
    cur_vel = rng.uniform(-2, 2, (B, 2, T)).astype(np.float32)
    cur_vel[:4] = 0.0                                              # arrived: zero controls, standing still
    cur_vel[4:8, 0] = 1.5                                          # turning at constant steering / rate / direction
    cur_vel[4:8, 1] = 0.4
    got = fp.fleet_plan_shapes(state, cur_vel, bd, dynamics, DT, L)
    vel_mode = ft.fleet_shapes(state, cur_vel, bd, dynamics)
    for k in ('kind', 'nv', 'xy', 'radius', 'vel'):
        np.testing.assert_array_equal(got[k], vel_mode[k])
    np.testing.assert_array_equal(got['plan_xy'][:, 0], vel_mode['xy'])        # stage 0: bit for bit
    for m in range(B):
        want = numpy_plan(bd, state[m], cur_vel[m], dynamics, L)
        np.testing.assert_allclose(got['plan_xy'][m], want, rtol=1e-6, atol=2e-5, err_msg=str(m))
    assert (got['plan_xy'][:4] == got['plan_xy'][:4, :1]).all()               # arrived robots stand still
    if body == 'disc':
        assert not got['plan_xy'][..., 1:, :].any()
        return
    # the turning robots' footprints rotate from stage to stage as their heading does (omni robots do not turn)
    edge = got['plan_xy'][4:8, :, 1].astype(float) - got['plan_xy'][4:8, :, 0].astype(float)
    ang = np.unwrap(np.arctan2(edge[..., 1], edge[..., 0]), axis=1)
    w = float(np.float32(0.4))
    rate = {'acker': 1.5 * np.tan(w) / L, 'diff': w, 'omni': 0.0}[dynamics]
    np.testing.assert_allclose(ang - ang[:, :1], np.broadcast_to(rate * DT * np.arange(T + 1), ang.shape), atol=1e-4)


def test_twin_plan_per_robot_dynamics_and_bodies():
    """Each robot's own dynamics, wheelbase and body equal a one-robot call with those as the scalars."""
    rng = np.random.default_rng(8)
    B, T = 30, 8
    names = ['acker', 'diff', 'omni']
    dyn = rng.integers(0, 3, B).astype(np.int32)
    L = rng.uniform(0.5, 3.0, B).astype(np.float32)
    pent = robot_body(_pentagon('acker'))
    xy = np.repeat(pent['xy'][None], B, 0) * rng.uniform(0.5, 2.0, (B, 1, 1)).astype(np.float32)
    state = np.c_[rng.uniform(-20, 20, (B, 2)), rng.uniform(-np.pi, np.pi, B)].astype(np.float32)
    cur_vel = rng.uniform(-2, 2, (B, 2, T)).astype(np.float32)
    per = {'dynamics': dyn, 'wheelbase': L, 'xy': xy, 'radius': np.zeros(B, np.float32)}
    got = fp.fleet_plan_shapes(state, cur_vel, pent, 'acker', DT, 1.0, per)
    for m in range(B):
        one = fp.fleet_plan_shapes(state[m:m + 1], cur_vel[m:m + 1], dict(pent, xy=xy[m]), names[dyn[m]], DT,
                                   float(L[m]))
        for k in one:
            np.testing.assert_array_equal(got[k][m], one[k][0])


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


@pytest.mark.parametrize('order', [True, False])
@pytest.mark.parametrize('N', [6, 30])
@pytest.mark.parametrize('body', ['rectangle', 'disc'])
def test_each_robot_matches_host_front_end_with_planned_mates(body, N, order):
    """Four worlds (40 shapes and 5 robots, an empty map with 3, 25 shapes and one robot, 10 shapes and none) and two
    robots outside them; some robots turning, one arrived."""
    rng = np.random.default_rng(21)
    body_car = rectangle_robot() if body == 'rectangle' else DISC
    dyn, L = body_car.dynamics, float(body_car.wheelbase)
    worlds = [_world(rng, 40, 12.0), [], _world(rng, 25, 12.0), _world(rng, 10, 12.0)]
    rw = np.array([0, 1, 0, 2, 0, -1, 1, 0, 4, 1, 0], np.int32)
    B, T, E = len(rw), 6, 5
    state = np.c_[rng.uniform(-5, 5, (B, 2)), rng.uniform(-np.pi, np.pi, B)].astype(np.float32)
    cur_vel = rng.uniform(-1.5, 1.5, (B, 2, T)).astype(np.float32)
    cur_vel[2, 0], cur_vel[2, 1] = 1.2, 0.5                      # turning
    cur_vel[4] = 0.0                                              # arrived
    bd = robot_body(body_car)
    world = pack_worlds(worlds)
    fleet = fp.fleet_plan_shapes(state, cur_vel, bd, dyn, DT, L)
    plans = [numpy_plan(bd, state[m], cur_vel[m], dyn, L) for m in range(B)]
    for b in range(B):
        w = int(rw[b])
        inside = 0 <= w < len(worlds)
        m = _host_mpc(dyn, L, T)
        st = state[b].astype(float).reshape(3, 1)
        m.state = st
        lst = list(m.convert_rda_obstacle(worlds[w], st, False)) if inside else []
        lst += [mate_rdaobs(m, bd, plans[j]) for j in range(B) if inside and rw[j] == w and j != b]
        if order:
            lst.sort(key=m.rda_obs_distance)
        A, bb, kind, cnt = fp.convert_fleet_plan_obstacles(world, fleet, rw, b, N, T, E, DT, order, state[b])
        assert cnt == len(lst), b
        if not lst:
            assert not A.any() and not bb.any() and list(kind) == [_cabi.OBS_POLYGON] * N
            continue
        Ah, bh, kh, ch, tvh = pack_obstacles(lst, T, N, E)
        if not tvh:                                               # only static shapes in the first N: one copy for all
            Ah, bh = np.repeat(Ah, T + 1, 1), np.repeat(bh, T + 1, 1)
        assert ch == cnt and list(kind) == list(kh), b
        np.testing.assert_allclose(A, Ah, atol=1e-5, err_msg=str(b))
        np.testing.assert_allclose(bb, bh, atol=1e-4, err_msg=str(b))


class _StubSolver:
    """Enough of RDA_solver for BatchedMPC's argument checks, without a device."""
    def __init__(self, receding, car_tuple, max_edge_num, max_obs_num, **kw):
        self.device = torch.device('cpu')
        self.max_edge_num = max(max_edge_num, 3)


def test_batched_mpc_refuses_plan_misuse(monkeypatch):
    monkeypatch.setattr(frontend, 'RDA_solver', _StubSolver)
    path = np.stack([np.arange(10.0), np.zeros(10), np.zeros(10)], 1)
    bm = frontend.BatchedMPC(rectangle_robot(), path, 2, receding=4, max_edge_num=4, max_obs_num=3)
    state = np.zeros((2, 3), np.float32)
    with pytest.raises(ValueError, match="'velocity' or 'plan'"):
        bm.control(state, 1.0, avoid_fleet=True, time_varying=True, fleet_prediction='plans')
    with pytest.raises(ValueError, match='avoid_fleet'):
        bm.control(state, 1.0, time_varying=True, fleet_prediction='plan')
    with pytest.raises(ValueError, match='time_varying=True'):
        bm.control(state, 1.0, avoid_fleet=True, fleet_prediction='plan')
    with pytest.raises(ValueError, match='shapes'):
        bm.control(state, 1.0, shapes=frontend.pack_shapes([[], []]), avoid_fleet=True, time_varying=True,
                   fleet_prediction='plan')
    with pytest.raises(ValueError, match='time_varying=True'):
        frontend.convert_fleet_obstacles_batch(None, None, None, None, 3, 4, 4, DT, False, True, plan=True)


def test_fleet_plan_usage_errors_are_return_codes():
    """Checked before any device work, so this runs without a GPU."""
    lib = _cabi.load()
    fs = lib.rda_fleet_plan_shapes
    fake = ctypes.c_void_p(256)
    P, D = _cabi.OBS_POLYGON, _cabi.OBS_CIRCLE

    def shapes(B=4, T=4, dyn=0, kind=P, nv=4, radius=0.0, per=(None,) * 4, ptrs=None):
        p = [fake] * 9 if ptrs is None else ptrs                  # body_xy, state, cur_vel, 5 outputs, plan_xy
        return fs(B, T, dyn, DT, 1.0, kind, nv, p[0], radius, *per, *p[1:], None)

    assert shapes(B=0) == -1 and shapes(T=0) == -1
    assert shapes(dyn=3) == -1 and shapes(dyn=-1) == -1                 # unknown dynamics
    assert shapes(kind=2) == -1                                          # unknown body kind
    assert shapes(nv=2) == -2 and shapes(nv=_cabi.MAX_EDGE + 1) == -2    # polygon outside 3..8 vertices
    assert shapes(kind=D, nv=0, radius=0.0) == -1                        # disc without a radius
    assert shapes(ptrs=[fake] * 8 + [ctypes.c_void_p(260)]) == -1        # plan_xy not 16-byte aligned
    cf = lib.rda_convert_fleet_plan_obstacles
    full = [fake] * 16                                                   # state .. fleet_vel, plan, 4 outputs
    assert cf(4, 1, 5, 10, 4, DT, 1, 1, *full[:15], None, *full[:4], None) == -1      # no plan
    assert cf(4, 1, 5, 10, 4, DT, 0, 1, *[fake] * 20, None) == -1      # time_varying = 0
    assert cf(0, 1, 5, 10, 4, DT, 1, 1, *[fake] * 20, None) == -1      # B < 1
    assert cf(4, 1, _cabi.MAX_WORLD_SLOTS + 1, 10, 4, DT, 1, 1, *[fake] * 20, None) == -2
    assert cf(4, 1, 5, 10, 2, DT, 1, 1, *[fake] * 20, None) == -2      # E < 3
    if torch.cuda.is_available():                     # below, a missing check would launch on placeholder pointers
        return
    for missing in range(8):                                             # body_xy, state, cur_vel or an output
        p = [fake] * 9
        p[missing] = None
        assert shapes(ptrs=p) == -1, missing
    assert shapes(per=(fake, fake, None, None), ptrs=[fake] * 8 + [None]) == -1   # plan_xy
    for missing in [0, 1] + list(range(3, 20)):                          # all but robot_world (2), which may be NULL
        p = [fake] * 20
        p[missing] = None
        assert cf(4, 1, 5, 10, 4, DT, 1, 1, *p, None) == -1, missing
