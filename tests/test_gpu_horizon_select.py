"""obstacle_order='horizon' on the device (rda_convert_world_obstacles_horizon, BatchedMPC(obstacle_order='horizon')):
the kernel against the brute-force CPU twin slot by slot, bitwise, on worlds, fleets at constant velocity and along
plans, robot classes, robots outside every world, a 16 384-shape map and a world of exact ties; the selection against
the clearance report of a BatchedMPC step; and closed loops on worlds, fleets and classes."""
import numpy as np
import pytest
import torch

import fleet_plan_twin as fp
import horizon_twin as ht
from test_horizon_select import Obs, _polygon, corridor_world
from rda_planner_b200.frontend import (BatchedMPC, convert_world_obstacles_horizon_batch, pack_worlds, robot_body,
                                       shapes_to_device)
from rda_planner_b200.scenarios import disc_robot, rectangle_robot

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
DT = float(np.float32(0.1))          # the float32 dt the kernel reads, so that the twin offsets stages alike


def _t(a, dtype=None):
    return torch.as_tensor(np.asarray(a), device=DEV, dtype=dtype).contiguous()


def _shapes(rng, count, lo, hi, E):
    obs = []
    for j in range(count):
        vel = rng.uniform(-1.5, 1.5, (2, 1)) if j % 3 == 1 else np.zeros((2, 1))
        c = rng.uniform(lo, hi, 2)
        if j % 4 == 0:
            obs.append(Obs(c.reshape(2, 1), float(rng.uniform(0.2, 1.5)), None, 'norm2', vel))
        else:
            obs.append(Obs(None, None, _polygon(rng, c, int(rng.integers(3, E + 1)), rng.uniform(0.3, 2.0)), 'Rpositive',
                           vel))
    return obs


def _poses(rng, B, T, lo, hi):
    """nom, ref [B,3,T+1]: straight lines with a turn, headings beyond +-pi; robot 1 has non-finite columns, robot 2
    none at all."""
    t = np.arange(T + 1) * DT
    out = []
    for _ in range(2):
        p0 = rng.uniform(lo, hi, (B, 2))
        th = rng.uniform(-4 * np.pi, 4 * np.pi, B)
        v = rng.uniform(0, 6, B)
        s = np.stack([p0[:, :1] + v[:, None] * t * np.cos(th)[:, None], p0[:, 1:] + v[:, None] * t * np.sin(th)[:, None],
                      th[:, None] + 0.2 * t], 1)
        out.append(s.astype(np.float32))
    out[0][1, 0, 3] = np.nan
    out[1][1, 2, T] = np.inf
    out[0][2] = np.nan
    out[1][2] = np.nan
    return out


def _compare(got, lst, N, T, E, tv, nom, ref, body):
    """Kernel outputs of one robot against the twin: every slot bitwise, or a swap of two entries whose keys are within
    1e-12 relative.  Returns the number of swapped slots."""
    A, b, kind, cnt = got
    tA, tb, tkind, tcnt, keys = ht.select(lst, N, T, E, DT, tv, nom, ref, body)
    assert cnt == tcnt
    same = [np.array_equal(A[n], tA[n]) and np.array_equal(b[n], tb[n]) and kind[n] == tkind[n] for n in range(N)]
    if all(same):
        return 0
    count = len(keys)
    order = np.argsort(keys, kind='stable')
    fA, fb, _, _, _ = ht.select(lst, count, T, E, DT, tv, nom, ref, body)     # rows of every entry in sorted order
    swaps = 0
    for n in np.nonzero(~np.array(same))[0]:
        k0 = keys[order[min(n, count - 1)]]
        m = [i for i in range(count) if np.array_equal(A[n], fA[i]) and np.array_equal(b[n], fb[i])]
        assert m and any(abs(keys[order[i]] - k0) <= 1e-12 * max(1.0, abs(k0)) for i in m), \
            f'slot {n}: twin key {k0!r}, the kernel wrote the rows of sorted positions {m[:4]} with keys ' \
            f'{[float(keys[order[i]]) for i in m[:4]]}; kinds {kind[:8]} / {tkind[:8]}'
        swaps += 1
    return swaps


def _case(mode, tv, N, classes, seed=0, B=48, T=12, E=8):
    rng = np.random.default_rng(seed)
    worlds = [_shapes(rng, 300, -20, 20, E), _shapes(rng, 40, -20, 20, E), []]
    world = pack_worlds(worlds)
    rw = (np.arange(B) % 3).astype(np.int32)
    rw[3], rw[4] = -1, 7                                           # in no world
    nom, ref = _poses(rng, B, T, -15, 15)
    car = rectangle_robot()
    body = robot_body(car)
    per = None
    if classes:
        scale = rng.uniform(0.5, 1.5, (B, 1, 1)).astype(np.float32)
        per = {'xy': (body['xy'][None] * scale).astype(np.float32), 'radius': np.zeros(B, np.float32)}
    fleet = None
    if mode != 'world':
        state = np.c_[rng.uniform(-15, 15, (B, 2)), rng.uniform(-np.pi, np.pi, B)].astype(np.float32)
        cur_vel = rng.uniform(-2, 2, (B, 2, T)).astype(np.float32)
        bxy = {'xy': per['xy'], 'radius': per['radius'], 'dynamics': np.zeros(B, np.int32),
               'wheelbase': np.full(B, 3.0, np.float32)} if classes else None
        fleet = fp.fleet_plan_shapes(state, cur_vel, body, 'acker', DT, 3.0, bxy)   # its shapes are fleet_shapes'
        if mode != 'plan':
            del fleet['plan_xy']
    dev_world = shapes_to_device(world, DEV)
    dev_fleet = None if fleet is None else {k: _t(v) for k, v in fleet.items()}
    dev_per = None if per is None else {k: _t(v) for k, v in per.items()}
    out = convert_world_obstacles_horizon_batch(dev_world, _t(nom), _t(ref), dict(body, xy=_t(body['xy'])), _t(rw), N,
                                                T, E, DT, tv, dev_fleet, mode == 'plan', dev_per)
    out = [o.cpu().numpy() for o in out]
    swaps = 0
    for b in range(B):
        lst = ht.robot_list(world, fleet, rw, b)
        bb = body if per is None else dict(body, xy=per['xy'][b])
        swaps += _compare([o[b] for o in out], lst, N, T, E, tv, nom[b], ref[b], bb)
    return swaps


@pytest.mark.parametrize('N', [1, 20, 128])
@pytest.mark.parametrize('mode, tv', [('world', False), ('world', True), ('velocity', False), ('velocity', True),
                                      ('plan', True)])                  # plans are trajectories: time-varying only
def test_kernel_matches_brute_force_twin(N, tv, mode):
    swaps = _case(mode, tv, N, classes=False, seed=N + tv)
    print(f'swapped slots within 1e-12: {swaps}')


@pytest.mark.parametrize('mode', ['world', 'plan'])
def test_kernel_matches_twin_with_class_bodies(mode):
    swaps = _case(mode, True, 20, classes=True, seed=3)
    print(f'swapped slots within 1e-12: {swaps}')


def test_kernel_matches_twin_with_small_caps_and_a_disc_body():
    """E = 4 and a disc body: the <4, 4> instantiation."""
    rng = np.random.default_rng(11)
    B, T, N, E = 32, 10, 8, 4
    world = pack_worlds([_shapes(rng, 500, -20, 20, E)])
    nom, ref = _poses(rng, B, T, -15, 15)
    body = robot_body(disc_robot(0.8, center=(0.2, 0.0)))
    out = convert_world_obstacles_horizon_batch(shapes_to_device(world, DEV), _t(nom), _t(ref),
                                                dict(body, xy=_t(body['xy'])), None, N, T, E, DT, True)
    out = [o.cpu().numpy() for o in out]
    for b in range(B):
        _compare([o[b] for o in out], ht.robot_list(world, None, None, 0), N, T, E, True, nom[b], ref[b], body)


def test_16384_shape_map_prunes_almost_everything():
    rng = np.random.default_rng(5)
    S, B, T, N, E = 16384, 256, 30, 20, 4
    obs = []
    for j in range(S):
        c = rng.uniform(0, 400, 2)
        w, h = rng.uniform(0.5, 3, 2)
        obs.append(Obs(None, None, np.array([[c[0], c[0] + w, c[0] + w, c[0]], [c[1], c[1], c[1] + h, c[1] + h]]),
                       'Rpositive', np.zeros((2, 1))))
    world = pack_worlds([obs])
    nom, ref = _poses(rng, B, T, 20, 380)
    body = robot_body(rectangle_robot())
    out = convert_world_obstacles_horizon_batch(shapes_to_device(world, DEV), _t(nom), _t(ref),
                                                dict(body, xy=_t(body['xy'])), None, N, T, E, DT, False)
    out = [o.cpu().numpy() for o in out]
    exact = []
    lst = ht.robot_list(world, None, None, 0)
    for b in [1, 2] + list(range(16, B, 16)):                     # 1: non-finite columns, 2: no finite pose at all
        _compare([o[b] for o in out], lst, N, T, E, False, nom[b], ref[b], body)
        if b != 2:                                                # its keys are all +inf: nothing to prune
            exact.append(ht.exact_count(lst, N, T, E, DT, False, nom[b], ref[b], body) / S)
    print(f'share of shapes given the exact key: {np.mean(exact):.4f}')
    assert np.mean(exact) < 0.05


def test_world_of_exact_ties():
    """Duplicated shapes and discs on a circle around a robot standing still: equal keys go to the lower index."""
    rng = np.random.default_rng(8)
    B, T, N, E = 8, 6, 20, 4
    base = [Obs(np.array([[5 * np.cos(a)], [5 * np.sin(a)]]), 1.0, None, 'norm2', np.zeros((2, 1)))
            for a in np.linspace(0, 2 * np.pi, 12, endpoint=False)]
    box = Obs(None, None, np.array([[2.0, 3.0, 3.0, 2.0], [-0.5, -0.5, 0.5, 0.5]]), 'Rpositive', np.zeros((2, 1)))
    obs = [base[i % 12] if i % 3 else box for i in range(600)]
    world = pack_worlds([obs])
    nom = np.zeros((B, 3, T + 1), np.float32)
    nom[:, 2] = rng.uniform(-np.pi, np.pi, (B, 1))
    ref = nom.copy()
    body = robot_body(disc_robot(0.5))
    out = convert_world_obstacles_horizon_batch(shapes_to_device(world, DEV), _t(nom), _t(ref),
                                                dict(body, xy=_t(body['xy'])), None, N, T, E, DT, False)
    out = [o.cpu().numpy() for o in out]
    for b in range(B):
        assert _compare([o[b] for o in out], ht.robot_list(world, None, None, 0), N, T, E, False, nom[b], ref[b],
                        body) == 0


def _line(x0, y0, heading, n, step=0.5):
    return [np.array([[x0 + i * step * np.cos(heading)], [y0 + i * step * np.sin(heading)], [heading]]) for i in range(n)]


def test_selection_agrees_with_the_clearance_report():
    """After a step with 'horizon', plan_clearance at nom_s and at ref_s gives, per slot, the smallest distance over t:
    non-decreasing over the kept slots and equal to the twin's key of the shape in that slot."""
    rng = np.random.default_rng(2)
    B, T, N, E = 16, 10, 6, 4
    car = rectangle_robot()
    bm = BatchedMPC(car, _line(0, 20, 0.0, 200), B, receding=T, iter_num=2, max_edge_num=E, max_obs_num=N,
                    obstacle_order='horizon')
    extra = [Obs(None, None, np.array([[x, x + 1, x + 1, x], [y, y, y + 1, y + 1]], float), 'Rpositive',
                 np.zeros((2, 1))) for x, y in rng.uniform([0, 10], [60, 30], (40, 2)) if abs(y - 20) > 2.5]
    world = corridor_world(extra)
    state = np.c_[rng.uniform(5, 50, B), rng.uniform(19, 21, B), rng.uniform(-0.2, 0.2, B)].astype(np.float32)
    _, info = bm.control(_t(state), 3.0, world=shapes_to_device(world, DEV))
    per = [bm.rda.plan_clearance(s=info[k], per_cell=True)['map'].cpu().numpy() for k in ('nom_s', 'ref_s')]
    slot = np.minimum(per[0], per[1]).min(2)                          # [B, N]
    body = robot_body(car)
    for b in range(B):
        lst = ht.robot_list(world, None, None, 0)
        keys = ht.select(lst, N, T, E, DT, False, info['nom_s'][b].cpu().numpy(), info['ref_s'][b].cpu().numpy(),
                         body)[4]
        kept = np.sort(keys)[:N]
        assert np.all(np.diff(slot[b]) >= -1e-5)
        np.testing.assert_allclose(slot[b], kept, atol=1e-5)


@pytest.mark.parametrize('setup', ['world', 'fleet_velocity', 'fleet_plan', 'classes'])
def test_closed_loop_with_horizon_order(setup):
    rng = np.random.default_rng(4)
    B, T, N, E = 24, 10, 6, 4
    kw = dict(receding=T, iter_num=2, max_edge_num=E, max_obs_num=N, obstacle_order='horizon')
    paths = [_line(0, 20, 0.0, 200), _line(60, 21, np.pi, 200)]
    robot_path = np.arange(B) % 2
    if setup == 'classes':
        cars = [rectangle_robot(), rectangle_robot(length=3.0, width=1.2, wheelbase=2.0)]
        bm = BatchedMPC(cars, paths, B, robot_path=robot_path, robot_class=np.arange(B) % 2, **kw)
    else:
        bm = BatchedMPC(rectangle_robot(), paths, B, robot_path=robot_path, **kw)
    world = shapes_to_device(corridor_world(), DEV)
    state = _t(np.c_[np.where(robot_path == 0, 2.0, 58.0) + rng.uniform(-1, 1, B), 20 + 0.5 * (robot_path == 1),
                     np.where(robot_path == 0, 0.0, np.pi)].astype(np.float32))
    avoid = setup != 'world'
    pred = 'plan' if setup == 'fleet_plan' else 'velocity'
    for _ in range(4):
        u0, info = bm.control(state, 3.0, world=world, avoid_fleet=avoid, time_varying=setup != 'world',
                              fleet_prediction=pred, robot_world=_t(np.arange(B) % 3, torch.int32), clearance=True) \
            if setup != 'world' else bm.control(state, 3.0, world=world, clearance=True)
        assert torch.isfinite(u0).all() and torch.isfinite(info['s']).all()
        bm.advance(state)
    assert torch.isfinite(state).all()
