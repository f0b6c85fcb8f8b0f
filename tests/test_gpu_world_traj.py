"""World shapes along given trajectories on the device (rda_convert_world_obstacles_traj,
rda_convert_world_obstacles_horizon_traj, BatchedMPC.control(world=...) with traj / traj_xy): both entry points
against the CPU twin (tests/cpu_twin/world_traj.cpp) on worlds, fleets at constant velocity and along plans, ids, robot
class bodies, robots outside every world, empty worlds and a 16 384-shape map; a BatchedMPC step against
iterative_solve_batch fed the twin's rows; its clearance report against oracle/clearance.py; updates of traj_xy in place,
without a host synchronisation and inside a captured graph."""
import numpy as np
import pytest
import torch

import fleet_plan_twin as fp
import world_traj_twin as wt
from oracle import clearance
from test_world_traj import TObs, _oracle_body, traj_world
from rda_planner_b200.frontend import (BatchedMPC, convert_fleet_obstacles_batch, convert_world_obstacles_batch,
                                       convert_world_obstacles_horizon_batch, pack_worlds, robot_body, shapes_to_device)
from rda_planner_b200.scenarios import rectangle_robot

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
DT = float(np.float32(0.1))


def _t(a, dtype=None):
    return torch.as_tensor(np.asarray(a), device=DEV, dtype=dtype).contiguous()


def _poses(rng, B, T, lo, hi):
    t = np.arange(T + 1) * DT
    out = []
    for _ in range(2):
        p0 = rng.uniform(lo, hi, (B, 2))
        th = rng.uniform(-np.pi, np.pi, B)
        v = rng.uniform(0, 5, B)
        out.append(np.stack([p0[:, :1] + v[:, None] * t * np.cos(th)[:, None],
                             p0[:, 1:] + v[:, None] * t * np.sin(th)[:, None], th[:, None] + 0.2 * t], 1)
                   .astype(np.float32))
    out[0][1, 0, 3] = np.nan
    return out


def _case(rng, B, T, E, sizes=(120, 30, 0)):
    worlds = [traj_world(rng, n, T, E, span=10.0, origin=(0.0, 0.0)) for n in sizes]
    world = pack_worlds(worlds)
    if 'traj' in world:
        world['traj'][np.nonzero(world['traj'] >= 0)[0][:2]] = [-3, 10 ** 6]     # out of range: no trajectory
    rw = (np.arange(B) % len(sizes)).astype(np.int32)
    rw[3], rw[4] = -1, 7                                                    # in no world
    return world, rw


def _fleet(rng, B, T, body, mode, classes):
    if mode == 'world':
        return None, None
    state = np.c_[rng.uniform(-10, 10, (B, 2)), rng.uniform(-np.pi, np.pi, B)].astype(np.float32)
    cur_vel = rng.uniform(-2, 2, (B, 2, T)).astype(np.float32)
    per = None
    if classes:
        scale = rng.uniform(0.5, 1.5, (B, 1, 1)).astype(np.float32)
        per = {'xy': (body['xy'][None] * scale).astype(np.float32), 'radius': np.zeros(B, np.float32),
               'dynamics': np.zeros(B, np.int32), 'wheelbase': np.full(B, 3.0, np.float32)}
    fleet = fp.fleet_plan_shapes(state, cur_vel, body, 'acker', DT, 3.0, per)
    if mode != 'plan':
        del fleet['plan_xy']
    return fleet, per


def _check_slots(got, want, keys=None):
    """Every slot bitwise; in the horizon order a slot may hold another entry whose key is within 1e-12 (the kernel's
    and the twin's keys may differ in the last bits)."""
    A, b, kind, cnt, ids = got
    tA, tb, tkind, tcnt, tids = want
    assert cnt == tcnt
    for n in range(len(kind)):
        if np.array_equal(A[n], tA[n]) and np.array_equal(b[n], tb[n]) and kind[n] == tkind[n] and ids[n] == tids[n]:
            continue
        assert keys is not None, n
        k = dict(zip(keys[1], keys[0]))
        assert abs(k[int(ids[n])] - k[int(tids[n])]) <= 1e-12 * max(1.0, abs(k[int(tids[n])])), n


@pytest.mark.parametrize('mode', ['world', 'velocity', 'plan'])
@pytest.mark.parametrize('order', [False, True])
@pytest.mark.parametrize('ids', [False, True])
def test_reference_key_matches_twin(mode, order, ids):
    rng = np.random.default_rng(10 * order + 3 * ids + len(mode))
    B, T, E, N = 40, 8, 8, 12
    world, rw = _case(rng, B, T, E)
    body = robot_body(rectangle_robot())
    fleet, _ = _fleet(rng, B, T, body, mode, False)
    state = np.c_[rng.uniform(-10, 10, (B, 2)), rng.uniform(-np.pi, np.pi, B)].astype(np.float32)
    dw = shapes_to_device(world, DEV)
    if fleet is None:
        out = convert_world_obstacles_batch(dw, _t(state), _t(rw), N, T, E, DT, True, order, ids)
    else:
        out = convert_fleet_obstacles_batch(dw, _t(state), _t(rw), {k: _t(v) for k, v in fleet.items()}, N, T, E, DT,
                                            True, order, mode == 'plan', ids)
    out = [o.cpu().numpy() for o in out]
    for r in range(B):
        lst = wt.robot_list(world, fleet, rw, r)
        want = wt.select(lst, N, T, E, DT, order, state[r])
        got = [o[r] for o in out[:4]] + [out[4][r] if ids else want[4]]
        _check_slots(got, want)


@pytest.mark.parametrize('mode', ['world', 'velocity', 'plan'])
@pytest.mark.parametrize('classes', [False, True])
def test_horizon_order_matches_twin(mode, classes):
    rng = np.random.default_rng(40 + classes + len(mode))
    B, T, E, N = 32, 8, 8, 10
    world, rw = _case(rng, B, T, E)
    body = robot_body(rectangle_robot())
    fleet, per = _fleet(rng, B, T, body, mode, classes)
    nom, ref = _poses(rng, B, T, -10, 10)
    dev_fleet = None if fleet is None else {k: _t(v) for k, v in fleet.items()}
    dev_per = None if per is None else {'xy': _t(per['xy']), 'radius': _t(per['radius'])}
    out = convert_world_obstacles_horizon_batch(shapes_to_device(world, DEV), _t(nom), _t(ref),
                                                dict(body, xy=_t(body['xy'])), _t(rw), N, T, E, DT, True, dev_fleet,
                                                mode == 'plan', dev_per, ids=True)
    out = [o.cpu().numpy() for o in out]
    for r in range(B):
        lst = wt.robot_list(world, fleet, rw, r)
        bb = body if per is None else dict(body, xy=per['xy'][r])
        want = wt.horizon_select(lst, N, T, E, DT, nom[r], ref[r], bb)
        _check_slots([o[r] for o in out], want[:5], (want[5], lst['id']))


def test_16384_shape_map_with_a_quarter_on_trajectories():
    rng = np.random.default_rng(5)
    S, B, T, N, E = 16384, 128, 30, 20, 4
    obs = []
    for j in range(S):
        c = rng.uniform(0, 400, 2)
        w, h = rng.uniform(0.5, 3, 2)
        box = np.array([[c[0], c[0] + w, c[0] + w, c[0]], [c[1], c[1], c[1] + h, c[1] + h]], np.float32).astype(float)
        tr = None
        if j % 4 == 0:
            d = rng.uniform(-1.5, 1.5, 2) * DT
            tr = [(box + (t * d).reshape(2, 1)).astype(np.float32).astype(float) for t in range(T + 1)]
        obs.append(TObs(None, None, box, 'Rpositive', np.zeros((2, 1)), tr))
    world = pack_worlds([obs])
    assert len(world['traj_xy']) == S // 4
    nom, ref = _poses(rng, B, T, 20, 380)
    state = nom[:, :, 0].copy()
    body = robot_body(rectangle_robot())
    dw = shapes_to_device(world, DEV)
    ref_key = [o.cpu().numpy() for o in convert_world_obstacles_batch(dw, _t(state), None, N, T, E, DT, True, True,
                                                                      ids=True)]
    hor = [o.cpu().numpy() for o in convert_world_obstacles_horizon_batch(
        dw, _t(nom), _t(ref), dict(body, xy=_t(body['xy'])), None, N, T, E, DT, True, ids=True)]
    lst = wt.robot_list(world, None, None, 0)
    for r in [0, 1] + list(range(32, B, 32)):
        _check_slots([o[r] for o in ref_key], wt.select(lst, N, T, E, DT, True, state[r]))
        want = wt.horizon_select(lst, N, T, E, DT, nom[r], ref[r], body)
        _check_slots([o[r] for o in hor], want[:5], (want[5], lst['id']))


def _line(x0, y0, heading, n, step=0.5):
    return [np.array([[x0 + i * step * np.cos(heading)], [y0 + i * step * np.sin(heading)], [heading]]) for i in range(n)]


def _mpc(B, T, N, E, order, warm_start):
    return BatchedMPC(rectangle_robot(), _line(-12, 0, 0.0, 200), B, receding=T, iter_num=3, max_edge_num=E,
                      max_obs_num=N, iter_threshold=0.0, obstacle_order=order, warm_start=warm_start)


def _step_case(seed=0, B=24, T=8):
    rng = np.random.default_rng(seed)
    world = pack_worlds([traj_world(rng, 40, T, 8, span=8.0, origin=(0.0, 0.0))])
    state = np.c_[rng.uniform(-10, -6, B), rng.uniform(-2, 2, B), rng.uniform(-0.3, 0.3, B)].astype(np.float32)
    return world, state


@pytest.mark.parametrize('order', [True, 'horizon'])
@pytest.mark.parametrize('warm_start', ['slot', 'obstacle'])
def test_batched_mpc_step_equals_solve_fed_the_twin_rows(order, warm_start):
    B, T, N, E = 24, 8, 6, 8
    world, state0 = _step_case()
    dw = shapes_to_device(world, DEV)
    bms = [_mpc(B, T, N, E, order, warm_start) for _ in range(2)]
    states = [_t(state0) for _ in range(2)]
    body = robot_body(rectangle_robot())
    for bm, st in zip(bms, states):                                   # one identical step on both
        bm.control(st, 3.0, world=dw, time_varying=True)
        bm.advance(st)
    torch.cuda.synchronize()
    _, info = bms[0].control(states[0], 3.0, world=dw, time_varying=True, clearance=True)
    st = states[1].cpu().numpy()
    nom, ref = info['nom_s'].cpu().numpy(), info['ref_s'].cpu().numpy()
    lst = wt.robot_list(world, None, None, 0)
    rows = [wt.select(lst, N, T, E, DT, True, st[r]) if order is True else
            wt.horizon_select(lst, N, T, E, DT, nom[r], ref[r], body)[:5] for r in range(B)]
    A, b, kind, cnt, ids = (np.stack([r[i] for r in rows]) for i in range(5))
    if warm_start == 'obstacle':
        assert torch.equal(info['obs_id'].cpu(), torch.as_tensor(ids))
        bms[1].rda.set_obstacle_ids(_t(ids))
    out = bms[1].rda.iterative_solve_batch(info['nom_s'], bms[1].cur_vel, info['ref_s'],
                                           torch.full((B,), 3.0, device=DEV), _t(A), _t(b), _t(kind), _t(cnt), True)
    for k in ('u', 's', 'status', 'iters'):
        assert torch.equal(out[k], info[k]), k
    # clearance: the signed distance of the planned body to each slot's stage-t trajectory shape
    s = info['s'].cpu().numpy()
    ob = _oracle_body(body)
    got = info['clearance'].cpu().numpy()
    for r in range(B):
        want = min(clearance.cell(ob, s[r, :, t].astype(float), int(kind[r, n]), A[r, n, t], b[r, n, t])
                   for n in range(min(N, cnt[r])) for t in range(T + 1))
        assert abs(got[r] - want) <= 1e-4 * max(1.0, abs(want)), (r, got[r], want)


def test_in_place_trajectory_update_needs_no_repack_and_no_host_sync():
    B, T, N, E = 24, 8, 6, 8
    world, state0 = _step_case(1)
    moved = dict(world, traj_xy=world['traj_xy'].copy())
    moved['traj_xy'][..., 1] += np.float32(0.75)                 # every trajectory shifted north
    dw = shapes_to_device(world, DEV)
    bm_a, bm_b, bm_c = (_mpc(B, T, N, E, True, 'obstacle') for _ in range(3))
    sa, sb, sc = _t(state0), _t(state0), _t(state0)
    bm_a.control(sa, 3.0, world=dw, time_varying=True)
    bm_b.control(sb, 3.0, world=shapes_to_device(world, DEV), time_varying=True)
    bm_c.control(sc, 3.0, world=shapes_to_device(world, DEV), time_varying=True)
    new_xy = _t(moved['traj_xy'])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        dw['traj_xy'].copy_(new_xy)                              # a predictor's output, written in place
        ua, ia = bm_a.control(sa, 3.0, world=dw, time_varying=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    ub, ib = bm_b.control(sb, 3.0, world=shapes_to_device(moved, DEV), time_varying=True)
    uc, ic = bm_c.control(sc, 3.0, world=shapes_to_device(world, DEV), time_varying=True)     # without the update
    torch.cuda.synchronize()
    for k in ('u', 's', 'status', 'iters', 'obs_id'):
        assert torch.equal(ia[k], ib[k]), k
    assert not torch.equal(ia['u'], ic['u'])                 # the update was read


def test_graph_step_replays_the_eager_step_with_updated_trajectories():
    B, T, N, E = 24, 8, 6, 8
    world, state0 = _step_case(2)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    runs = []
    with torch.cuda.stream(side):
        for _ in range(2):
            bm, dw, st = _mpc(B, T, N, E, 'horizon', 'obstacle'), shapes_to_device(world, DEV), _t(state0)
            for _ in range(2):
                bm.control(st, 3.0, world=dw, time_varying=True)
                bm.advance(st)
            runs.append((bm, dw, st))
    side.synchronize()
    bm, dw, st = runs[0]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            u_g, info_g = bm.control(st, 3.0, world=dw, time_varying=True)
            bm.advance(st)
    torch.cuda.current_stream().wait_stream(side)
    shift = torch.tensor([0.5, -0.25], device=DEV)
    dw['traj_xy'][:, 1:] += shift                                  # new predictions after capture
    graph.replay()
    bm2, dw2, st2 = runs[1]
    dw2['traj_xy'][:, 1:] += shift
    u_e, info_e = bm2.control(st2, 3.0, world=dw2, time_varying=True)
    bm2.advance(st2)
    torch.cuda.synchronize()
    for k in ('u', 's', 'status', 'iters', 'obs_id'):
        assert torch.equal(info_g[k], info_e[k]), k
    assert torch.equal(st, st2) and torch.equal(bm.cur_vel, bm2.cur_vel)


def test_batched_mpc_takes_a_trajectory_world_with_every_option():
    B, T, N, E = 12, 8, 4, 8
    world, state0 = _step_case(3, B)
    dw = shapes_to_device(world, DEV)
    for order in (True, False, 'horizon'):
        for fleet, pred in ((False, 'velocity'), (True, 'velocity'), (True, 'plan')):
            for ws in ('slot', 'obstacle'):
                bm = _mpc(B, T, N, E, order, ws)
                u, info = bm.control(_t(state0), 3.0, world=dw, time_varying=True, avoid_fleet=fleet,
                                     fleet_prediction=pred, clearance=True)
                assert bool(torch.isfinite(u).all()) and bool(torch.isfinite(info['clearance']).all())
    with pytest.raises(ValueError, match='time_varying'):
        _mpc(B, T, N, E, True, 'slot').control(_t(state0), 3.0, world=dw)
