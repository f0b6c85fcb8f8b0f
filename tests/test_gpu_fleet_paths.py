"""A fleet on its own reference paths on the H100: the path kernels (k_pre_process_paths, k_post_process_paths) against
the CPU twin (tests/cpu_twin/fleet_paths.cpp) on random fleets, their scale invariance, the old single-path entry
points as their W = 1 case, and BatchedMPC(robot_path=...) in closed loop against one host mpc.MPC per robot driving
the same solver, with update_ref_path and set_robot_path in the middle of the loop."""
import copy
import os
from collections import namedtuple

import numpy as np
import pytest
import torch

import fleet_twin
from rda_planner_b200 import _cabi
from rda_planner_b200.frontend import BatchedMPC, _ptr, _stream, pack_paths, pack_worlds
from rda_planner_b200.mpc import MPC
from rda_planner_b200.scenarios import rectangle_robot

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
PATH = list(np.load(os.path.join(HERE, 'golden', 'path_track_ref.npy'), allow_pickle=True))
DEV = torch.device('cuda:0')
Obs = namedtuple('Obs', 'center radius vertex cone_type velocity')
L, DT = 3.0, 0.1


def _dev(packed):
    return {k: torch.as_tensor(v, device=DEV).contiguous() for k, v in packed.items()}


def random_path(rng, n, curves):
    """n waypoints (random walk, 0.1-0.5 m steps) cut into `curves` single-gear curves (alternating gears)."""
    curves = min(curves, n)
    head = np.cumsum(rng.normal(0, 0.15, n)) + rng.uniform(-np.pi, np.pi)
    step = rng.uniform(0.1, 0.5, n)
    xy = np.cumsum(np.stack([step * np.cos(head), step * np.sin(head)], 1), 0) + rng.uniform(-30, 30, 2)
    cuts = np.sort(rng.choice(np.arange(1, n), curves - 1, replace=False)) if curves > 1 else np.array([], int)
    gear = np.ones(n) * rng.choice([-1.0, 1.0])
    for c in cuts:
        gear[c:] *= -1
    return np.concatenate([xy, head[:, None], gear[:, None]], 1).astype(np.float32).astype(float)


def random_fleet(rng, B, W, max_len=600, no_path=True):
    paths = [random_path(rng, int(rng.integers(1, max_len + 1)), int(rng.integers(1, 5))) for _ in range(W)]
    pk = pack_paths(paths, enable_reverse=True)
    robot_path = rng.integers(0, W, B).astype(np.int32)
    if no_path:
        robot_path[rng.random(B) < 0.03] = -1
        robot_path[rng.random(B) < 0.02] = W + 3
    curve_index = np.zeros(B, np.int32)
    start, state, near_in = np.zeros(B, np.int32), np.zeros((B, 3), np.float32), np.zeros(B, np.int32)
    for b in range(B):
        w = robot_path[b] if 0 <= robot_path[b] < W else 0
        lo, hi = pk['path_curve'][w], pk['path_curve'][w + 1]
        c = int(rng.integers(0, hi - lo))
        curve_index[b] = c if rng.random() > 0.05 else c + int(rng.choice([-3, 7]))     # clamped on the device
        cs, ce = pk['curve_start'][lo + c], pk['curve_start'][lo + c + 1]
        i = int(rng.integers(0, ce - cs))
        start[b] = max(0, i - int(rng.integers(0, 6)))
        state[b] = pk['path'][cs + i] + rng.normal(0, [0.3, 0.3, 0.2])
        near_in[b] = i if rng.random() < 0.5 else max(0, ce - cs - int(rng.integers(0, 3)))   # often at the end
    return pk, robot_path, curve_index, start, state, near_in


def pre_paths(pkd, W, dyn, T, state, cur_vel, speed, robot_path, curve_index, start):
    lib = _cabi.load()
    B = state.shape[0]
    nom = torch.empty((B, 3, T + 1), dtype=torch.float32, device=DEV)
    ref = torch.empty_like(nom)
    near = torch.empty(B, dtype=torch.int32, device=DEV)
    sp = torch.empty(B, dtype=torch.float32, device=DEV)
    _cabi.check(lib.rda_pre_process_paths(B, T, _cabi.DYNAMICS[dyn], DT, L, _ptr(state), _ptr(cur_vel), _ptr(speed),
                                          _ptr(pkd['path']), W, _ptr(pkd['path_curve']), _ptr(pkd['curve_start']),
                                          _ptr(pkd['curve_gear']), _ptr(robot_path), _ptr(curve_index), _ptr(start),
                                          0.1, 10, _ptr(nom), _ptr(ref), _ptr(near), _ptr(sp), _stream(DEV)),
                'rda_pre_process_paths')
    return nom, ref, near, sp


def post_paths(pkd, W, T, robot_path, thr, near, curve_index, u):
    B = near.shape[0]
    near, ci, u = near.clone(), curve_index.clone(), u.clone()
    cur_vel = torch.empty_like(u)
    arrive = torch.empty(B, dtype=torch.int32, device=DEV)
    _cabi.check(_cabi.load().rda_post_process_paths(B, T, W, _ptr(pkd['path_curve']), _ptr(pkd['curve_start']),
                                                    _ptr(robot_path), thr, _ptr(near), _ptr(ci), _ptr(u), _ptr(cur_vel),
                                                    _ptr(arrive), _stream(DEV)), 'rda_post_process_paths')
    return near, ci, u, cur_vel, arrive


def _t(a, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(a), device=DEV, dtype=dtype)


@pytest.mark.parametrize('dyn', ['acker', 'diff', 'omni'])
def test_path_kernels_match_twin_on_random_fleets(dyn):
    rng = np.random.default_rng({'acker': 1, 'diff': 2, 'omni': 3}[dyn])
    B, W, T = 2000, 97, 12
    pk, robot_path, curve_index, start, state, near_in = random_fleet(rng, B, W)
    vel = np.stack([rng.uniform(-3, 5, (B, T)), rng.uniform(-0.4, 0.4, (B, T))], 1).astype(np.float32)
    speed = rng.uniform(1, 5, B).astype(np.float32)
    pkd = _dev(pk)
    nom, ref, near, sp = pre_paths(pkd, W, dyn, T, _t(state), _t(vel), _t(speed), _t(robot_path), _t(curve_index),
                                   _t(start))
    n1, r1, k1, s1 = fleet_twin.pre_process_paths(pk, dyn, T, DT, L, state, vel, speed, robot_path, curve_index, start)
    np.testing.assert_array_equal(near.cpu().numpy(), k1)
    np.testing.assert_array_equal(sp.cpu().numpy(), s1)
    np.testing.assert_allclose(nom.cpu().numpy(), n1, atol=2e-5)
    np.testing.assert_allclose(ref.cpu().numpy(), r1, atol=2e-5)
    assert (s1 < 0).sum() > B // 5 and (k1 > 0).sum() > B // 2
    u = rng.normal(0, 1, (B, 2, T)).astype(np.float32)
    for thr in (1, 3):
        got = post_paths(pkd, W, T, _t(robot_path), thr, _t(near_in), _t(curve_index), _t(u))
        want = fleet_twin.post_process_paths(pk, T, robot_path, thr, near_in, curve_index, u)
        for g, w_ in zip(got, want):
            np.testing.assert_array_equal(g.cpu().numpy(), w_)
        moved = want[1] != curve_index
        assert moved.sum() > B // 20 and want[4].sum() > B // 20


def test_fleet_of_16384_on_1024_paths_equals_each_robot_alone():
    """Bitwise: every robot of a B = 16 384, W = 1 024 launch gives exactly what it gives launched alone on a store
    that holds only its own path."""
    rng = np.random.default_rng(9)
    B, W, T = 16384, 1024, 10
    pk, robot_path, curve_index, start, state, near_in = random_fleet(rng, B, W, no_path=False)
    vel = np.stack([rng.uniform(-3, 5, (B, T)), rng.uniform(-0.4, 0.4, (B, T))], 1).astype(np.float32)
    speed = rng.uniform(1, 5, B).astype(np.float32)
    u = rng.normal(0, 1, (B, 2, T)).astype(np.float32)
    st, vl, spd, ci, si, nr, uu = (_t(a) for a in (state, vel, speed, curve_index, start, near_in, u))
    rp = _t(robot_path)
    pkd = _dev(pk)
    nom, ref, near, sp = pre_paths(pkd, W, 'acker', T, st, vl, spd, rp, ci, si)
    post = post_paths(pkd, W, T, rp, 1, nr, ci, uu)
    one = []
    for w in range(W):
        lo, hi = pk['path_curve'][w], pk['path_curve'][w + 1]
        cs = pk['curve_start'][lo:hi + 1]
        one.append(_dev({'path': pk['path'][cs[0]:cs[-1]], 'path_curve': np.array([0, hi - lo], np.int32),
                         'curve_start': (cs - cs[0]).astype(np.int32), 'curve_gear': pk['curve_gear'][lo:hi]}))
    zero = torch.zeros(1, dtype=torch.int32, device=DEV)
    a_nom, a_ref = torch.empty_like(nom), torch.empty_like(ref)
    a_near, a_sp = torch.empty_like(near), torch.empty_like(sp)
    a_post = [nr.clone(), ci.clone(), uu.clone(), torch.empty_like(uu), torch.empty_like(near)]
    lib = _cabi.load()
    s = _stream(DEV)
    for b in range(B):
        p = one[robot_path[b]]
        _cabi.check(lib.rda_pre_process_paths(1, T, 0, DT, L, _ptr(st[b]), _ptr(vl[b]), _ptr(spd[b:]), _ptr(p['path']),
                                              1, _ptr(p['path_curve']), _ptr(p['curve_start']), _ptr(p['curve_gear']),
                                              _ptr(zero), _ptr(ci[b:]), _ptr(si[b:]), 0.1, 10, _ptr(a_nom[b]),
                                              _ptr(a_ref[b]), _ptr(a_near[b:]), _ptr(a_sp[b:]), s), 'pre alone')
        _cabi.check(lib.rda_post_process_paths(1, T, 1, _ptr(p['path_curve']), _ptr(p['curve_start']), _ptr(zero), 1,
                                               _ptr(a_post[0][b:]), _ptr(a_post[1][b:]), _ptr(a_post[2][b]),
                                               _ptr(a_post[3][b]), _ptr(a_post[4][b:]), s), 'post alone')
    for x, y in zip((nom, ref, near, sp) + tuple(post), (a_nom, a_ref, a_near, a_sp) + tuple(a_post)):
        assert torch.equal(x, y)
    assert int((post[1] != ci).sum()) > 100 and int(post[4].sum()) > 100


@pytest.mark.parametrize('reverse', [False, True])
def test_old_entry_points_are_the_one_path_case(reverse):
    """rda_pre_process / rda_post_process (one curve) and rda_pre_process_curves / rda_post_process_gear (one path of
    several curves) equal rda_pre_process_paths / rda_post_process_paths with W = 1, bitwise."""
    rng = np.random.default_rng(4)
    B, T = 4096, 15
    pk, _, curve_index, start, state, near_in = random_fleet(rng, B, 1, max_len=400, no_path=False)
    if not reverse:
        pk = pack_paths([pk['path']])
        curve_index[:] = 0
        start = np.minimum(start, len(pk['path']) - 1)
        near_in[::7] = len(pk['path']) - 1 - rng.integers(0, 3, len(near_in[::7]))       # at the end of the path
    C = len(pk['curve_gear'])
    vel = np.stack([rng.uniform(-3, 5, (B, T)), rng.uniform(-0.4, 0.4, (B, T))], 1).astype(np.float32)
    speed = rng.uniform(1, 5, B).astype(np.float32)
    u = rng.normal(0, 1, (B, 2, T)).astype(np.float32)
    st, vl, spd, ci, si, nr, uu = (_t(a) for a in (state, vel, speed, curve_index, start, near_in, u))
    pkd = _dev(pk)
    lib = _cabi.load()
    nom, ref, near, sp = pre_paths(pkd, 1, 'diff', T, st, vl, spd, None, ci, si)
    post = post_paths(pkd, 1, T, None, 2, nr, ci, uu)
    o_nom, o_ref, o_near = torch.empty_like(nom), torch.empty_like(ref), torch.empty_like(near)
    o_nr, o_ci, o_u = nr.clone(), ci.clone(), uu.clone()
    o_vel, o_arr = torch.empty_like(uu), torch.empty_like(near)
    s = _stream(DEV)
    if reverse:
        _cabi.check(lib.rda_pre_process_curves(B, T, 1, DT, L, _ptr(st), _ptr(vl), _ptr(spd), _ptr(pkd['path']), C,
                                               _ptr(pkd['curve_start']), _ptr(ci), _ptr(si), 0.1, 10, _ptr(o_nom),
                                               _ptr(o_ref), _ptr(o_near), s), 'rda_pre_process_curves')
        _cabi.check(lib.rda_post_process_gear(B, T, C, _ptr(pkd['curve_start']), 2, _ptr(o_nr), _ptr(o_ci), _ptr(o_u),
                                              _ptr(o_vel), _ptr(o_arr), s), 'rda_post_process_gear')
        gear = pkd['curve_gear'][(pkd['path_curve'][0] + ci.long().clamp(0, C - 1))].float()
        assert torch.equal(sp, spd * gear) and bool((gear < 0).any())
    else:
        _cabi.check(lib.rda_pre_process(B, T, 1, DT, L, _ptr(st), _ptr(vl), _ptr(spd), _ptr(pkd['path']),
                                        len(pk['path']), _ptr(si), 0.1, 10, _ptr(o_nom), _ptr(o_ref), _ptr(o_near), s),
                    'rda_pre_process')
        _cabi.check(lib.rda_post_process(B, T, len(pk['path']), 2, _ptr(o_nr), _ptr(o_u), _ptr(o_vel), _ptr(o_arr), s),
                    'rda_post_process')
        assert torch.equal(sp, spd)
    for x, y in zip((nom, ref, near) + tuple(post), (o_nom, o_ref, o_near, o_nr, o_ci, o_u, o_vel, o_arr)):
        assert torch.equal(x, y)
    assert int(post[4].sum()) > 0


# ---- BatchedMPC on a fleet of paths, through the solver -------------------------------------------------------
def _line(x0, y0, heading, n, step=0.5, gear=1.0):
    return [np.array([[x0 + step * i * np.cos(heading)], [y0 + step * i * np.sin(heading)], [heading], [gear]])
            for i in range(n)]


def _gear_path():
    """5 m forward, 4 m in reverse and forward again along y = 1 (three curves)."""
    pts = [(0.2 * i, 1.0) for i in range(26)] + [(5.0 - 0.2 * i, -1.0) for i in range(1, 21)] + \
          [(1.0 + 0.2 * i, 1.0) for i in range(1, 16)]
    return [np.array([[x], [1.0], [0.0], [g]]) for x, g in pts]


def _world():
    rng = np.random.default_rng(8)
    obs = []
    for j in range(40):
        c = np.array([[rng.uniform(-2, 25)], [rng.choice([-1, 1]) * rng.uniform(4.5, 9)]])
        if j % 2:
            obs.append(Obs(c, float(rng.uniform(0.3, 0.8)), None, 'norm2', np.zeros((2, 1))))
        else:
            ang = np.linspace(0, 2 * np.pi, 4, endpoint=False) + rng.uniform(0, 1)
            obs.append(Obs(None, None, c + 0.7 * np.vstack([np.cos(ang), np.sin(ang)]), 'Rpositive', np.zeros((2, 1))))
    return [o._replace(center=None if o.center is None else o.center.astype(np.float32).astype(float),
                       vertex=None if o.vertex is None else o.vertex.astype(np.float32).astype(float)) for o in obs]


def _acker_step(s, u):
    return s + DT * np.array([[u[0, 0] * np.cos(s[2, 0])], [u[0, 0] * np.sin(s[2, 0])], [u[0, 0] * np.tan(u[1, 0]) / L]])


def test_fleet_closed_loop_with_path_updates_matches_host_mpcs():
    """Eight robots on three paths (one with gear changes) in one shared obstacle map, 30 steps, against one host
    mpc.MPC per robot driving the same solver.  At step 10 set_robot_path moves three robots to other paths of the
    set near where they are; at step 20 update_ref_path replaces the whole set.  The host MPCs' paths are restored before each call
    (INTEGRATION.md §3, deviation (i))."""
    car = rectangle_robot()
    T, N, E, steps, speed = 8, 4, 4, 30, 2.0
    paths = [_line(0.0, -1.0, 0.0, 50), _gear_path(), _line(0.0, 2.5, 0.05, 50)]
    paths2 = [_line(-1.0, 0.0, 0.05, 30, step=2.0), _line(0.0, -2.0, -0.03, 30, step=2.0)]
    robot_path = [0, 1, 2, 1, 0, 2, 1, 0]
    starts = [(0, 0), (0, 3), (0, 4), (1, 2), (0, 20), (0, 10), (2, 5), (0, 38)]      # (curve, index)
    B = len(robot_path)
    kw = dict(receding=T, sample_time=DT, iter_num=2, max_edge_num=E, max_obs_num=N, iter_threshold=0.0,
              enable_reverse=True)
    obs = _world()
    world = _dev(pack_worlds([obs]))
    bm = BatchedMPC(car, paths, B, robot_path=robot_path, **kw)
    hosts, host_state, st0 = [], [], []
    for b, (c, i) in enumerate(starts):
        m = MPC(car, copy.deepcopy(paths[robot_path[b]]), time_print=False, **kw)
        m.curve_index, m.cur_index = c, i
        hosts.append(m)
        wp = np.asarray(m.curve_list[c][i], float).reshape(-1)[:3]
        st0.append(wp + np.array([0.05, 0.03, 0.01]))
        host_state.append(st0[-1].reshape(3, 1).copy())
    host_paths = [paths[w] for w in robot_path]
    bm.curve_index[:] = _t([c for c, _ in starts], torch.int32)
    bm.cur_index[:] = _t([i for _, i in starts], torch.int32)
    dev_state = _t(np.stack(st0).astype(np.float32))
    switched = 0
    for k in range(steps):
        if k == 10:
            moved, to = np.array([0, 2, 1]), np.array([2, 0, 0])
            mask = np.zeros(B, bool)
            mask[moved] = True
            new = np.zeros(B, np.int32)
            new[moved] = to
            bm.set_robot_path(_t(new), _t(mask))
            for b, w in zip(moved, to):
                hosts[b].update_ref_path(copy.deepcopy(paths[w]))
                host_paths[b] = paths[w]
        if k == 20:
            new = [1, 0, 1, 0, 0, 1, 1, 0]
            bm.update_ref_path(paths2, robot_path=new)
            for b, m in enumerate(hosts):
                m.update_ref_path(copy.deepcopy(paths2[new[b]]))
                host_paths[b] = paths2[new[b]]
        u0, info = bm.control(dev_state, speed, world=world)
        u0 = u0.cpu().numpy()
        for b, m in enumerate(hosts):
            m.ref_path = copy.deepcopy(host_paths[b])
            m.curve_list = m.split_path(m.ref_path)
            before = m.curve_index
            uh, ih = m.control(host_state[b], speed, obs)
            switched += int(m.curve_index != before)
            if m.curve_index >= len(m.curve_list):
                m.curve_index = len(m.curve_list) - 1      # the reference raises IndexError on its next call
                m.cur_index = len(m.curve_list[-1]) - 1
            assert bool(info['arrive'][b]) == ih['arrive'], (k, b)
            assert int(info['curve_index'][b]) == m.curve_index, (k, b)
            assert int(info['cur_index'][b]) == m.cur_index, (k, b)
            np.testing.assert_allclose(u0[b], uh[:, 0], atol=3e-3, err_msg=f'{k} {b}')
            host_state[b] = _acker_step(host_state[b], uh)
        bm.advance(dev_state)
        np.testing.assert_allclose(dev_state.cpu().numpy(), np.hstack(host_state).T, atol=3e-3)
    assert switched >= 2


def test_one_path_through_robot_path_equals_single_path_mpc():
    """All robots on path 0 of a one-path set equal the single-path BatchedMPC, bitwise, over 10 steps."""
    car = rectangle_robot()
    B, T = 64, 10
    kw = dict(receding=T, sample_time=DT, iter_num=3, max_edge_num=4, max_obs_num=4, iter_threshold=0.0)
    rng = np.random.default_rng(6)
    idx = rng.integers(0, len(PATH) - 5, B)
    arr = np.stack([np.asarray(p, float).reshape(-1)[:3] for p in PATH])
    st = _t((arr[idx] + rng.normal(0, [0.2, 0.2, 0.05], (B, 3))).astype(np.float32))
    world = _dev(pack_worlds([_world()]))
    a = BatchedMPC(car, PATH, B, **kw)
    b = BatchedMPC(car, [PATH], B, robot_path=np.zeros(B, np.int32), **kw)
    for m in (a, b):
        m.cur_index[:] = _t(np.maximum(idx - 2, 0), torch.int32)
    sa, sb = st.clone(), st.clone()
    for _ in range(10):
        ua, ia = a.control(sa, 3.0, world=world)
        ub, ib = b.control(sb, 3.0, world=world)
        assert torch.equal(ua, ub)
        for key in ('u', 's', 'arrive', 'nom_s', 'ref_s', 'cur_index', 'curve_index', 'status'):
            assert torch.equal(ia[key], ib[key]), key
        a.advance(sa)
        b.advance(sb)
    assert torch.equal(sa, sb)


def test_multi_path_step_needs_no_host_sync():
    car = rectangle_robot()
    B = 32
    paths = [_line(0.0, -1.0, 0.0, 50), _gear_path(), _line(0.0, 2.5, 0.05, 50)]
    bm = BatchedMPC(car, paths, B, robot_path=np.arange(B) % 4, receding=8, iter_num=2, max_edge_num=4,
                    max_obs_num=4, enable_reverse=True)
    world = _dev(pack_worlds([_world()]))
    state = _t(np.stack([[0.2 * (b % 8), 0.0, 0.0] for b in range(B)]).astype(np.float32))
    mask = _t(np.arange(B) % 3 == 0)
    new = _t(np.full(B, 2, np.int32))
    bm.control(state, 2.0, world=world)                                   # first call: allocations, graph keys
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        bm.set_robot_path(new, mask)
        u0, info = bm.control(state, 2.0, world=world)
        bm.advance(state)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(u0).all())
    no_path = [b for b in range(B) if b % 4 == 3 and b % 3]              # path index 3 of 3 paths, not moved
    assert bool(info['arrive'][no_path].all())
