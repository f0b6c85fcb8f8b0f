"""Robots of a fleet as obstacles of each other predicted along their plans, on the device (rda_fleet_plan_shapes,
rda_convert_fleet_plan_obstacles, BatchedMPC.control(fleet_prediction='plan')): the kernels against their CPU twins with
one body and with robot classes, a 16 384-robot fleet against each world alone, the same slots as the velocity
prediction, a closed loop against host MPCs handed the reference-terms list, a step without host synchronisation and in
a CUDA graph, and a robot that turns across another's lane."""
import copy
from collections import namedtuple

import numpy as np
import pytest
import torch

import fleet_plan_twin as fp
from rda_planner_b200.frontend import (BatchedMPC, convert_fleet_obstacles_batch, fleet_plan_shapes_batch,
                                       fleet_shapes_batch, pack_worlds, robot_body, shapes_to_device)
from rda_planner_b200.mpc import MPC, rdaobs
from rda_planner_b200.scenarios import rectangle_robot

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


def _fleet(rng, B, W, span, T):
    rw = rng.integers(0, W, B).astype(np.int32)
    rw[:4] = [-1, W, 1 << 30, -(1 << 30)]                       # in no world
    state = np.c_[rng.uniform(0, span, (B, 2)), rng.uniform(-np.pi, np.pi, B)].astype(np.float32)
    cur_vel = rng.uniform(-2, 2, (B, 2, T)).astype(np.float32)
    cur_vel[rng.random(B) < 0.1] = 0.0                             # arrived
    return rw, state, cur_vel


def _classes(rng, B, body):
    """Per-robot dynamics, wheelbase and body (the same kind and vertex count, scaled) as robot classes give them."""
    return {'dynamics': rng.integers(0, 3, B).astype(np.int32), 'wheelbase': rng.uniform(0.8, 3.0, B).astype(np.float32),
            'xy': (np.repeat(body['xy'][None], B, 0) * rng.uniform(0.5, 1.5, (B, 1, 1))).astype(np.float32),
            'radius': np.zeros(B, np.float32)}


def _run(world_dev, state, rw, cur_vel, body, dyn, L, N, T, E, order, per=None):
    st = _t(state)
    pr = None if per is None else {k: _t(v) for k, v in per.items()}
    fleet = fleet_plan_shapes_batch(st, _t(cur_vel), _dev_body(body), dyn, DT, L, pr)
    out = convert_fleet_obstacles_batch(world_dev, st, _t(rw), fleet, N, T, E, DT, True, order, plan=True)
    return {k: v.cpu().numpy() for k, v in fleet.items()}, [o.cpu().numpy() for o in out]


@pytest.mark.parametrize('classes', [False, True])
@pytest.mark.parametrize('N', [1, 20, 128])
@pytest.mark.parametrize('order', [False, True])
def test_plan_kernels_match_cpu_twins(order, N, classes):
    """~600 robots in six worlds of 0 to 2 000 shapes (and robots in none); rectangle body, acker or mixed classes."""
    rng = np.random.default_rng(41)
    sizes = [0, 2000, 17, 400, 1, 1200]
    host = pack_worlds([_world(rng, n, 0.0, 80.0) for n in sizes])
    B, T, E, L = 600, 6, 8, 2.5
    rw, state, cur_vel = _fleet(rng, B, len(sizes), 80.0, T)
    body = robot_body(rectangle_robot())
    per = _classes(rng, B, body) if classes else None
    fleet, (A, b, kind, count) = _run(shapes_to_device(host, DEV), state, rw, cur_vel, body, 'acker', L, N, T, E, order,
                                      per)
    want = fp.fleet_plan_shapes(state, cur_vel, body, 'acker', DT32, L, per)
    for k in ('kind', 'nv', 'radius'):
        np.testing.assert_array_equal(fleet[k], want[k])
    np.testing.assert_array_equal(fleet['plan_xy'][:, 0], fleet['xy'])          # stage 0 is the fleet shape
    for k in ('xy', 'vel', 'plan_xy'):
        np.testing.assert_allclose(fleet[k], want[k], rtol=1e-6, atol=1e-5)
    for i in range(B):                                             # selection and rows from the kernel's own shapes
        A1, b1, k1, c1 = fp.convert_fleet_plan_obstacles(host, fleet, rw, i, N, T, E, DT32, order, state[i])
        w = int(rw[i])
        assert count[i] == c1 == ((sizes[w] + int((rw == w).sum()) - 1) if 0 <= w < len(sizes) else 0), i
        assert list(kind[i]) == list(k1), i
        np.testing.assert_array_equal(A[i], A1)
        np.testing.assert_allclose(b[i], b1, rtol=1e-6, atol=1e-6)


def test_16384_robots_in_64_worlds_equal_each_world_alone():
    """64 worlds of 1 024 shapes and 256 robots each (interleaved across the batch), plan mode, mixed classes: every
    robot's arrays are bit for bit what the same kernels write when its world is converted as a batch of its own."""
    rng = np.random.default_rng(64)
    W, per_w, S, N, T, E = 64, 256, 1024, 20, 5, 8
    B = W * per_w
    rw = rng.permutation(np.repeat(np.arange(W, dtype=np.int32), per_w))
    host = pack_worlds([_world(rng, S, 0.0, 100.0) for _ in range(W)])
    state = np.c_[rng.uniform(0, 100, (B, 2)), rng.uniform(-np.pi, np.pi, B)].astype(np.float32)
    cur_vel = rng.uniform(-2, 2, (B, 2, T)).astype(np.float32)
    body = robot_body(rectangle_robot())
    per = _classes(rng, B, body)
    fleet, full = _run(shapes_to_device(host, DEV), state, rw, cur_vel, body, 'acker', 3.0, N, T, E, True, per)
    assert (full[3] == S + per_w - 1).all()
    for w in range(W):
        idx = np.nonzero(rw == w)[0]
        one = {k: host[k][host['start'][w]:host['start'][w + 1]] for k in KEYS}
        one['start'] = np.array([0, S], np.int32)
        f1, alone = _run(shapes_to_device(one, DEV), state[idx], np.zeros(per_w, np.int32), cur_vel[idx], body, 'acker',
                         3.0, N, T, E, True, {k: v[idx] for k, v in per.items()})
        np.testing.assert_array_equal(fleet['plan_xy'][idx], f1['plan_xy'])
        for f, a in zip(full, alone):
            np.testing.assert_array_equal(f[idx], a)


@pytest.mark.parametrize('order', [False, True])
def test_same_slots_as_velocity_prediction(order):
    """Against avoid_fleet's velocity prediction on the same inputs (time-varying output): the same kinds, counts and
    stage-0 copies bit for bit.  In worlds 0 and 1 (maps of 0 and 60 shapes) every robot drives straight at constant controls, so there every
    copy of every slot agrees within float32 rounding (world shapes: bit for bit).

    Tolerance for the straight robots.  Let e = 2^-24 (float32 unit roundoff), X the largest coordinate magnitude of a
    placed vertex (start and travel), d the largest distance a robot travels over the horizon and l the longest body
    edge.  Velocity mode places each vertex once in float32 (error <= X e) and moves it by fl(v cos th) t dt (error
    <= d e); plan mode rolls the pose out in double and rounds each stage's vertex once (error <= X e).  So a vertex
    differs by at most dv = (2 X + d) e.  A row is an edge vector (a_i = (dy, -dx)): it differs by at most 2 dv, plus its
    own float32 rounding l e.  b_i = a_i . p_i differs by at most 2 dv X + l dv + its rounding l X e.  A disc's centre
    row differs by at most dv.  Every bound is doubled for the double-precision steps in between."""
    rng = np.random.default_rng(17)
    W, B, T, N, E, span, vmax = 3, 300, 12, 20, 8, 40.0, 2.0
    host = pack_worlds([_world(rng, n, 0.0, span) for n in (0, 60, 5)])
    rw, state, cur_vel = _fleet(rng, B, W, span, T)
    straight = (rw == 0) | (rw == 1)
    dyn = 'diff'
    v = (rng.uniform(0.1, vmax, B) * rng.choice([-1, 1], B)).astype(np.float32)    # above the 0.01 moving threshold
    cur_vel[straight, 0, :] = v[straight, None]                    # constant speed, no turn
    cur_vel[straight, 1, :] = 0.0
    body = robot_body(rectangle_robot(dynamics=dyn))
    world = shapes_to_device(host, DEV)
    st, cv, bd, rwd = _t(state), _t(cur_vel), _dev_body(body), _t(rw)
    vel = convert_fleet_obstacles_batch(world, st, rwd, fleet_shapes_batch(st, cv, bd, dyn), N, T, E, DT, True, order)
    plan = convert_fleet_obstacles_batch(world, st, rwd, fleet_plan_shapes_batch(st, cv, bd, dyn, DT, 3.0), N, T, E, DT,
                                         True, order, plan=True)
    vel, plan = [o.cpu().numpy() for o in vel], [o.cpu().numpy() for o in plan]
    np.testing.assert_array_equal(vel[2], plan[2])                 # obs_kind
    np.testing.assert_array_equal(vel[3], plan[3])                 # obs_count
    np.testing.assert_array_equal(vel[0][:, :, 0], plan[0][:, :, 0])
    np.testing.assert_array_equal(vel[1][:, :, 0], plan[1][:, :, 0])
    eps = 2.0 ** -24
    d = vmax * T * DT
    V = body['xy'][:body['nv']].astype(float)
    ell = float(np.max(np.linalg.norm(np.roll(V, -1, axis=0) - V, axis=1)))
    X = span + float(np.max(np.linalg.norm(V, axis=1))) + d
    dv = 2 * (2 * X + d) * eps
    tol_A = 2 * (2 * dv + ell * eps)
    tol_b = 2 * (2 * dv * X + ell * dv + ell * X * eps)
    np.testing.assert_allclose(plan[0][straight], vel[0][straight], rtol=0, atol=tol_A)
    np.testing.assert_allclose(plan[1][straight], vel[1][straight], rtol=0, atol=tol_b)
    moved = (plan[1][straight] != vel[1][straight]).any(axis=(2, 3))
    assert moved.sum() > 100                                        # the comparison covers mates' later copies
    turning = ~straight & (rw == 2)                                 # and the prediction does change for the others
    assert np.abs(plan[1][turning] - vel[1][turning]).max() > 100 * tol_b


# ---- BatchedMPC(avoid_fleet=True, fleet_prediction='plan') --------------------------------------------------------
def _line(x0, y0, heading, n, step=0.5):
    return [np.array([[x0 + step * i * np.cos(heading)], [y0 + step * i * np.sin(heading)], [heading]])
            for i in range(n)]


def _arc(cx, cy, r, phi0, phi1, step=0.25):
    """Waypoints on the circle (cx, cy, r) from angle phi0 to phi1, heading along the direction of travel."""
    n = int(abs(phi1 - phi0) * r / step) + 1
    turn = 1.0 if phi1 > phi0 else -1.0
    return [np.array([[cx + r * np.cos(p)], [cy + r * np.sin(p)], [p + turn * np.pi / 2]])
            for p in np.linspace(phi0, phi1, n)]


def _host_plan_obstacle(m, body, s, u):
    """A map-mate at host state s (3, 1) with host control sequence u (2, T), predicted along its plan, as the reference's
    rdaobs with A and b lists of T+1 arrays (the host model step, the body placed in float64)."""
    T = u.shape[1]
    q, A, b, V0 = s, [], [], None
    for t in range(T + 1):
        th = float(q[2, 0])
        R = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
        V = q[:2] + R @ body['xy'][:body['nv']].astype(float).T
        V0 = V if V0 is None else V0
        At, bt = m.convert_inequal_polygon(V)
        A.append(At)
        b.append(bt)
        if t < T:
            c = min(t + 1, T - 1)
            q = m.motion_predict_model_acker(q, u[:, c:c + 1], m.L, m.dt)
    return rdaobs(A, b, 'Rpositive', None, V0)


def test_closed_loop_with_plan_prediction_matches_host_mpcs():
    """Six robots on their own paths (two of them arcs) in two shared maps, time-varying obstacles, 4 steps: each host
    mpc.MPC(rda_obstacle=True) is handed the reference-terms list built from host states and host control sequences:
    its map's shapes converted by the MPC itself, then every other robot of its map along its plan, sorted stably by
    rda_obs_distance."""
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
    paths = [_line(0.0, -3.0, 0.0, 80), _arc(0.0, 30.0, 30.0, -np.pi / 2, -np.pi / 2 + 0.9),
             _line(0.0, 3.0, 0.02, 80), _arc(0.0, -34.0, 30.0, np.pi / 2, np.pi / 2 - 0.9)]
    robot_path = [0, 1, 2, 0, 3, 1]
    robot_world = [0, 0, 0, 1, 1, 1]
    starts = [4, 2, 6, 3, 0, 8]
    B = len(robot_path)
    kw = dict(receding=T, sample_time=DT, iter_num=3, max_edge_num=E, max_obs_num=N, iter_threshold=0.0)
    bm = BatchedMPC(car, paths, B, robot_path=robot_path, **kw)
    bm.cur_index[:] = _t(starts, torch.int32)
    hosts, host_state = [], []
    for b in range(B):
        m = MPC(car, copy.deepcopy(paths[robot_path[b]]), time_print=False, rda_obstacle=True, **kw)
        m.cur_index = starts[b]
        hosts.append(m)
        wp = np.asarray(paths[robot_path[b]][starts[b]], float).reshape(-1)[:3]
        host_state.append((wp + np.array([0.1, -0.05, 0.02])).reshape(3, 1))
    body = dict(bm.body, xy=bm.body['xy'].cpu().numpy())
    world = shapes_to_device(pack_worlds(maps), DEV)
    dev_state = _t(np.hstack(host_state).T.astype(np.float32))
    turned = 0.0
    for k in range(steps):
        u0, info = bm.control(dev_state, speed, time_varying=True, world=world, robot_world=robot_world,
                              avoid_fleet=True, fleet_prediction='plan')
        u0 = u0.cpu().numpy()
        assert list(info['status'].cpu().numpy() & 6) == [0] * B
        mates = [_host_plan_obstacle(hosts[j], body, host_state[j], np.asarray(hosts[j].cur_vel_array, float))
                 for j in range(B)]
        turned = max(turned, max(float(np.abs(np.asarray(h.cur_vel_array)[1]).max()) for h in hosts))
        new_u = []
        for b, m in enumerate(hosts):
            m.state = host_state[b]
            lst = list(m.convert_rda_obstacle(maps[robot_world[b]], host_state[b], False))
            lst += [mates[j] for j in range(B) if robot_world[j] == robot_world[b] and j != b]
            lst.sort(key=m.rda_obs_distance)
            uh, ih = m.control(host_state[b], speed, lst)
            assert bool(info['arrive'][b]) == ih['arrive']
            assert int(info['cur_index'][b]) == m.cur_index
            np.testing.assert_allclose(u0[b], uh[:, 0], atol=2e-3, err_msg=f'{k} {b}')
            new_u.append(uh[:, :1])
        for b in range(B):
            s, u = host_state[b], new_u[b]
            host_state[b] = s + DT * np.array([[u[0, 0] * np.cos(s[2, 0])], [u[0, 0] * np.sin(s[2, 0])],
                                               [u[0, 0] * np.tan(u[1, 0]) / car.wheelbase]])
        bm.advance(dev_state)
        np.testing.assert_allclose(dev_state.cpu().numpy(), np.hstack(host_state).T, atol=2e-3)
    assert turned > 0.05                                             # the plans handed over do steer


def _plan_fleet(B=48):
    car = rectangle_robot()
    paths = [_line(0.0, -1.0, 0.0, 50), _arc(0.0, 22.5, 20.0, -np.pi / 2, 0.0)]
    bm = BatchedMPC(car, paths, B, robot_path=np.arange(B) % 2, receding=8, iter_num=2, max_edge_num=4, max_obs_num=4)
    world = shapes_to_device(pack_worlds([_world(np.random.default_rng(0), 50, 0, 30), []]), DEV)
    rw = _t(np.arange(B) % 3 - (np.arange(B) == 7), torch.int32)       # worlds 0, 1 and none (2, -1)
    state = _t(np.stack([[0.3 * (b % 16), 2.5 * (b % 2), 0.0] for b in range(B)]).astype(np.float32))
    return bm, world, rw, state


def test_plan_step_needs_no_host_sync():
    bm, world, rw, state = _plan_fleet()
    kw = dict(time_varying=True, avoid_fleet=True, fleet_prediction='plan')
    bm.control(state, 2.0, world=world, robot_world=rw, **kw)
    bm.control(state, 2.0, **kw)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        u0, info = bm.control(state, 2.0, world=world, robot_world=rw, **kw)
        bm.advance(state)
        u1, _ = bm.control(state, 2.0, **kw)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(u0).all()) and bool(torch.isfinite(u1).all())


def test_plan_step_in_a_cuda_graph_replays_the_eager_step():
    """Two identical fleets step eagerly; then one step (control + advance) of the first is captured and replayed while
    the second takes the same step eagerly: the replay gives the eager step's outputs bit for bit.  (One replay per
    capture: control() rebinds cur_index to the tensor it just wrote, so a graph keeps reading the index it was
    recorded with.)"""
    fleets = [_plan_fleet() for _ in range(2)]
    kw = dict(time_varying=True, avoid_fleet=True, fleet_prediction='plan')
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for bm, world, rw, state in fleets:
            for _ in range(2):
                bm.control(state, 2.0, world=world, robot_world=rw, **kw)
                bm.advance(state)
    side.synchronize()
    bm, world, rw, state = fleets[0]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            u_g, info_g = bm.control(state, 2.0, world=world, robot_world=rw, **kw)
            bm.advance(state)
    torch.cuda.current_stream().wait_stream(side)
    bm2, world2, rw2, state2 = fleets[1]
    graph.replay()
    u_e, info_e = bm2.control(state2, 2.0, world=world2, robot_world=rw2, **kw)
    bm2.advance(state2)
    torch.cuda.synchronize()
    assert torch.equal(u_g, u_e) and torch.equal(info_g['u'], info_e['u']) and torch.equal(info_g['s'], info_e['s'])
    assert torch.equal(state, state2) and torch.equal(bm.cur_vel, bm2.cur_vel)
    assert torch.equal(info_g['cur_index'], info_e['cur_index'])


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


def turning_crossing(prediction, avoid=True, steps=100):
    """Robot 0 drives east along y = 0 from x = -8; robot 1 comes from the south and turns left on an arc of radius 10
    (centre (-8, -8)) that crosses robot 0's lane at x = -2, heading north-west, then drives west along y = 2.  At the
    same speed both reach the crossing within a second of each other.  Returns the executed poses [steps + 1, 2, 3] and,
    per step, whether the bodies overlap."""
    car = rectangle_robot(length=2.0, width=1.0, wheelbase=1.2, dynamics='diff', max_speed=(3, 1.5), max_acce=(3, 1.5))
    paths = [_line(-8.0, 0.0, 0.0, 160, step=0.25),
             _arc(-8.0, -8.0, 10.0, 0.0, np.pi / 2) + _line(-8.25, 2.0, np.pi, 80, step=0.25)[1:]]
    bm = BatchedMPC(car, paths, 2, robot_path=[0, 1], receding=12, sample_time=DT, iter_num=4, max_edge_num=4,
                    max_obs_num=3, iter_threshold=0.0)
    state = _t(np.array([[-8.0, 0.0, 0.0], [2.0, -8.0, np.pi / 2]], np.float32))
    body = dict(bm.body, xy=bm.body['xy'].cpu().numpy())
    traj = [state.cpu().numpy().copy()]
    for _ in range(steps):
        bm.control(state, 2.0, time_varying=True, avoid_fleet=avoid, fleet_prediction=prediction if avoid else 'velocity')
        bm.advance(state)
        traj.append(state.cpu().numpy().copy())
    traj = np.stack(traj)
    return traj, [_overlap(_corners(body, s[0]), _corners(body, s[1])) for s in traj]


def test_a_robot_turning_across_a_lane_is_avoided_along_its_plan():
    traj, hit = turning_crossing('plan')
    assert not any(hit)
    assert traj[-1, 0, 0] > 4.0 and traj[-1, 1, 1] > 1.0 and traj[-1, 1, 0] < -6.0   # both well past the crossing
