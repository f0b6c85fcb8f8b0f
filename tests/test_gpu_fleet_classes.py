"""-m gpu: robot classes in the batched front end: the per-robot entry points (rda_pre_process_paths_per_robot,
rda_motion_predict_per_robot, rda_fleet_shapes_per_robot) against the scalar ones, BatchedMPC(robot_class=...) against one
fleet per class, avoid_fleet with each robot's own body and motion, set_robot_class mid-run without a host
synchronisation, and a class change between warm-started solves on the coherent routing."""
import gc

import numpy as np
import pytest
import torch

from rda_planner_b200 import _cabi
from rda_planner_b200.frontend import BatchedMPC, convert_fleet_obstacles_batch, fleet_shapes_batch, pack_paths, pack_worlds, robot_body, \
    shapes_to_device
from rda_planner_b200.scenarios import disc_robot, rectangle_robot
from test_gpu_instance_params import _inputs, _path, _solve, _solver, _world
from test_robot_classes import BODIES, disc_classes

pytestmark = pytest.mark.gpu
KW = dict(receding=10, sample_time=0.1, iter_num=3, max_edge_num=4, max_obs_num=4, iter_threshold=0.0)


def fleet_classes():
    """acker (the rear-axle rectangle), diff (centred box of the diff examples), omni (centred box of the omni examples)."""
    return [BODIES.body('rect_rear'), BODIES.body('rect_centred'), BODIES.body('omni_centred')]


def _ptr(t):
    return t.data_ptr()


def _state(B, seed=5):
    rng = np.random.default_rng(seed)
    s = np.stack([rng.uniform(0, 3, B), rng.uniform(-1.5, 1.5, B), rng.uniform(-0.3, 0.3, B)], 1)
    return torch.as_tensor(s, dtype=torch.float32, device='cuda')


@pytest.mark.parametrize('dyn', ['acker', 'diff', 'omni'])
def test_per_robot_entry_points_equal_the_scalar_ones_with_uniform_arrays(dyn):
    lib = _cabi.load()
    B, T, dt, L = 64, 10, 0.1, 2.5
    st = _state(B)
    vel = torch.as_tensor(np.random.default_rng(1).uniform(-1, 1, (B, 2, T)), dtype=torch.float32, device='cuda')
    spd = torch.full((B,), 3.0, device='cuda')
    dyn_b = torch.full((B,), _cabi.DYNAMICS[dyn], dtype=torch.int32, device='cuda')
    L_b = torch.full((B,), L, dtype=torch.float32, device='cuda')
    p = {k: torch.as_tensor(v, device='cuda').contiguous() for k, v in pack_paths([_path()]).items()}
    zi = torch.zeros(B, dtype=torch.int32, device='cuda')
    res = []
    for per in (False, True):
        nom, ref = torch.empty((B, 3, T + 1), device='cuda'), torch.empty((B, 3, T + 1), device='cuda')
        near, sp = torch.empty(B, dtype=torch.int32, device='cuda'), torch.empty(B, device='cuda')
        tail = (_ptr(st), _ptr(vel), _ptr(spd), _ptr(p['path']), 1, _ptr(p['path_curve']), _ptr(p['curve_start']),
                _ptr(p['curve_gear']), _ptr(zi), _ptr(zi), _ptr(zi), 0.1, 10, _ptr(nom), _ptr(ref), _ptr(near), _ptr(sp),
                None)
        if per:
            assert lib.rda_pre_process_paths_per_robot(B, T, _ptr(dyn_b), dt, _ptr(L_b), *tail) == 0
        else:
            assert lib.rda_pre_process_paths(B, T, _cabi.DYNAMICS[dyn], dt, L, *tail) == 0
        s2 = st.clone()
        if per:
            assert lib.rda_motion_predict_per_robot(B, T, _ptr(dyn_b), dt, _ptr(L_b), _ptr(vel), _ptr(s2), None) == 0
        else:
            assert lib.rda_motion_predict(B, T, _cabi.DYNAMICS[dyn], dt, L, _ptr(vel), _ptr(s2), None) == 0
        body = robot_body(rectangle_robot())
        body['xy'] = torch.as_tensor(body['xy'], device='cuda')
        per_robot = {'dynamics': dyn_b, 'xy': body['xy'].expand(B, 8, 2).contiguous(),
                     'radius': torch.zeros(B, device='cuda')} if per else None
        fl = fleet_shapes_batch(st, vel, body, dyn, per_robot)
        torch.cuda.synchronize()
        res.append([nom, ref, near, sp, s2] + [fl[k] for k in ('kind', 'nv', 'xy', 'radius', 'vel')])
    for a, b in zip(*res):
        assert torch.equal(a, b)


@pytest.mark.parametrize('kind', ['polygon', 'disc'])
def test_per_robot_fleet_shapes_equal_one_call_per_class(kind):
    """Each robot is placed with its own body and moves with its own dynamics' world-frame velocity."""
    B, T = 30, 10
    classes = fleet_classes() if kind == 'polygon' else disc_classes()
    st = _state(B, 9)
    vel = torch.as_tensor(np.random.default_rng(2).uniform(-1, 1, (B, 2, T)), dtype=torch.float32, device='cuda')
    bm = BatchedMPC(classes, _path(), B, robot_class=np.arange(B) % len(classes), **KW)
    mixed = fleet_shapes_batch(st, vel, bm.body, bm.dynamics, bm.per_robot)
    for k, c in enumerate(classes):
        body = robot_body(c)
        body['xy'] = torch.as_tensor(body['xy'], device='cuda')
        one = fleet_shapes_batch(st, vel, body, c.dynamics)
        rows = torch.arange(k, B, len(classes), device='cuda')
        for key in ('kind', 'nv', 'xy', 'radius', 'vel'):
            assert torch.equal(mixed[key][rows], one[key][rows]), (k, key)
    # against numpy for the velocity: v0 along the control angle v1 for omni, along the heading for the others
    u0, u1 = vel[:, 0, 0].double().cpu().numpy(), vel[:, 1, 0].double().cpu().numpy()
    th = st[:, 2].double().cpu().numpy()
    for b in range(B):
        c = classes[b % len(classes)]
        d = u1[b] if c.dynamics == 'omni' else th[b]
        want = (u0[b] * np.cos(d), u0[b] * np.sin(d))
        np.testing.assert_allclose(mixed['vel'][b].double().cpu().numpy(), want, atol=1e-5)


@pytest.mark.parametrize('avoid', [False, True])
def test_mixed_fleet_steps_like_one_fleet_per_class(avoid):
    """20 closed-loop steps on a shared world: an acker / diff / omni fleet in one BatchedMPC against one BatchedMPC per
    class.  Without avoid_fleet every row is bitwise that of its class's fleet.  With avoid_fleet each robot's obstacle
    list holds its map-mates with their own class bodies and velocities: checked against a fleet of per-class bodies
    built from the same fleet shapes."""
    B, steps = 12, 20
    classes = fleet_classes()
    idx = np.arange(B) % 3
    world = shapes_to_device(pack_worlds([_world()]), 'cuda')
    st0 = _state(B, 3)
    bm = BatchedMPC(classes, _path(), B, robot_class=idx, **KW)
    st = st0.clone()
    us = []
    for _ in range(steps):
        u, info = bm.control(st, 3.0, world=world, avoid_fleet=avoid)
        assert bool(torch.isfinite(info['u']).all())
        us.append(u.clone())
        bm.advance(st)
    if avoid:
        # the obstacle lists of the next step: map shapes, then the map-mates, each with its own class body and velocity
        fl = fleet_shapes_batch(st, bm.cur_vel, bm.body, bm.dynamics, bm.per_robot)
        stitched = {k: v.clone() for k, v in fl.items()}
        for k, c in enumerate(classes):
            body = robot_body(c)
            body['xy'] = torch.as_tensor(body['xy'], device='cuda')
            one = fleet_shapes_batch(st, bm.cur_vel, body, c.dynamics)
            rows = torch.arange(k, B, 3, device='cuda')
            for key in stitched:
                stitched[key][rows] = one[key][rows]
        got = convert_fleet_obstacles_batch(world, st, None, fl, KW['max_obs_num'], KW['receding'], 4, KW['sample_time'])
        want = convert_fleet_obstacles_batch(world, st, None, stitched, KW['max_obs_num'], KW['receding'], 4,
                                             KW['sample_time'])
        for a, b in zip(got, want):
            assert torch.equal(a, b)
        return
    for k, c in enumerate(classes):
        one = BatchedMPC(c, _path(), B, **KW)
        s1 = st0.clone()
        rows = torch.arange(k, B, 3, device='cuda')
        for t in range(steps):
            u, _ = one.control(s1, 3.0, world=world)
            assert torch.equal(u[rows], us[t][rows]), (k, t)
            one.advance(s1)
        assert torch.equal(s1[rows], st[rows]), k
        del one
    gc.collect()


def test_set_robot_class_mid_run_needs_no_host_sync():
    B = 24
    classes = fleet_classes()
    classes[2] = classes[2]._replace(max_speed=[2.0, 0.4], max_acce=[1.0, 0.2])
    bm = BatchedMPC(classes, _path(), B, robot_class=np.zeros(B, int), **KW)
    world = shapes_to_device(pack_worlds([_world()]), 'cuda')
    st = _state(B, 4)
    bm.control(st, 3.0, world=world)
    keep = (torch.arange(B, device='cuda') % 4) == 3
    bm.update_parameter(robots=keep, max_speed=torch.tensor([5.0, 0.8], device='cuda').expand(B, 2))
    move = (torch.arange(B, device='cuda') % 2) == 0
    to = torch.full((B,), 2, dtype=torch.int64, device='cuda')
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        bm.set_robot_class(to, move)
        u, info = bm.control(st, 3.0, world=world)
        bm.advance(st)
        bm.rda.set_robot_class_index(torch.full((B,), 1 << 40, dtype=torch.int64, device='cuda'), ~move & ~keep)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.equal(bm.per_robot['dynamics'][move].cpu(), torch.full((int(move.sum()),), 2, dtype=torch.int32))
    ms = bm.rda.instance_parameters()['max_speed']
    assert bool((ms[move] == torch.tensor([2.0, 0.4], device='cuda')).all())
    assert bool((ms[keep & ~move] == torch.tensor([5.0, 0.8], device='cuda')).all())      # not moved: override kept
    assert bool((info['u'][move][:, 0].abs() <= 2.0 + 1e-5).all())
    # a 64-bit index far outside the classes means the handle's class (0), not a wrapped valid class
    assert bool((bm.rda.robot_class_index()[~move & ~keep] == -1).all())


def test_class_change_between_warm_solves_on_the_coherent_routing():
    """A robot whose class changes keeps its warm start (and the coherent pass' feat hint): the robots that did not move
    give the bits of a run where nobody moved, the moved ones solve without a kept-previous status."""
    B, T, N = 16384, 30, 20
    classes = fleet_classes()
    inp, tv = _inputs(B, T, N, seed=2500)
    first = torch.zeros(B, dtype=torch.int32, device='cuda')
    move = (torch.arange(B, device='cuda') % 5) == 0
    second = torch.where(move, torch.arange(B, device='cuda', dtype=torch.int32) % 3, first)
    res = {}
    for change in (False, True):
        g = _solver({}, classes[0], T, N, B, 8)
        g.set_robot_classes(classes, first)
        _solve(g, inp, tv)
        if change:
            g.set_robot_class_index(second)
        res[change] = _solve(g, inp, tv)
        del g
        gc.collect()
    stay = ~move | (second == 0)
    for k in ('u', 's', 'status', 'iters'):
        assert torch.equal(res[True][k][stay], res[False][k][stay]), k
    moved = move & (second != 0)
    assert bool(torch.isfinite(res[True]['u'][moved]).all())
    assert float(((res[True]['status'][moved] & 2) == 0).float().mean()) > 0.99
