"""A fleet on its own reference paths (rda_pre_process_paths / rda_post_process_paths): the CPU twin
(tests/cpu_twin/fleet_paths.cpp) against independent host front ends (mpc.MPC, one per robot) in a closed loop
without a solver, against the reference goldens with the golden path inside a larger set, and for robots without a
path; pack_paths against split_path; the entry points' usage errors.  No GPU."""
import copy
import ctypes
import json
import os

import numpy as np
import pytest
import torch

import fleet_twin
from rda_planner_b200 import _cabi
from rda_planner_b200.frontend import pack_paths
from rda_planner_b200.mpc import MPC

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, 'golden', 'boundary_golden.json')))
PATH = list(np.load(os.path.join(HERE, 'golden', 'path_track_ref.npy'), allow_pickle=True))
PATH_ARR = np.stack([np.asarray(p, float).reshape(-1)[:3] for p in PATH])
TOL = 2e-5
L, DT = 3.0, 0.1


class _Car:
    G = h = None
    cone_type, wheelbase, max_speed, max_acce = 'Rpositive', L, [10, 1], [10, 0.5]

    def __init__(self, dynamics):
        self.dynamics = dynamics


class _ScriptedSolver:
    """Stands in for RDA_solver: records what MPC.control hands to iterative_solve and returns scripted controls."""

    def __init__(self, *a, **k):
        self.u = None
        self.seen = None
        self.owner = None

    def iterative_solve(self, nom_s, cur_vel, ref_traj, ref_speed, obs, **kw):
        self.seen = dict(nom_s=np.array(nom_s, float), ref=np.hstack([np.asarray(r, float)[0:3] for r in ref_traj]),
                         speed=float(ref_speed), near=self.owner.cur_index)
        return self.u.copy(), {}


def with_gear(path, gear=1.0):
    return [np.vstack([np.asarray(p, float).reshape(-1, 1)[:3], [[gear]]]) for p in path]


def fwd_rev_fwd(x0=0.0, y0=0.0):
    """5 m forward along +x, 4 m in reverse, forward again: three curves (as the gear test of the batched MPC)."""
    pts = [(x0 + 0.2 * i, 1.0) for i in range(26)] + [(x0 + 5.0 - 0.2 * i, -1.0) for i in range(1, 21)] + \
          [(x0 + 1.0 + 0.2 * i, 1.0) for i in range(1, 16)]
    return [np.array([[x], [y0], [0.0], [g]]) for x, g in pts]


def line(n, x0, y0, heading, step=0.25):
    return [np.array([[x0 + step * i * np.cos(heading)], [y0 + step * i * np.sin(heading)], [heading], [1.0]])
            for i in range(n)]


def golden_reverse_path():
    """The path of the reference's split_path record: gear +1 for 5 waypoints, then -1 (tests/golden)."""
    return [np.array([[float(i)], [0.0], [0.0], [1.0 if i < 5 else -1.0]]) for i in range(9)]


# ---- pack_paths ----------------------------------------------------------------------------------------------
def _split_reference(path):
    m = MPC(_Car('acker'), path, receding=4, solver_cls=_ScriptedSolver, enable_reverse=True)
    return m.curve_list


@pytest.mark.parametrize('form', ['list', 'array', 'tensor'])
def test_pack_paths_matches_split_path(form):
    paths = [golden_reverse_path(), fwd_rev_fwd(3.0, 2.0), with_gear(PATH), line(1, 0, 0, 0.3),
             with_gear(PATH[:2], -1.0), golden_reverse_path()[::-1]]
    assert [len(c) for c in _split_reference(paths[0])] == GOLD['split_path']
    conv = {'list': lambda p: p, 'array': lambda p: np.hstack(p).T,
            'tensor': lambda p: torch.as_tensor(np.hstack(p).T)}[form]
    pk = pack_paths([conv(p) for p in paths], enable_reverse=True)
    assert all(pk[k].dtype == np.int32 for k in ('curve_start', 'path_curve', 'curve_gear'))
    assert pk['path'].dtype == np.float32 and pk['path'].shape == (sum(len(p) for p in paths), 3)
    assert len(pk['path_curve']) == len(paths) + 1
    for w, p in enumerate(paths):
        curves = _split_reference(copy.deepcopy(p))
        lo, hi = pk['path_curve'][w], pk['path_curve'][w + 1]
        assert hi - lo == len(curves)
        for c, ref in zip(range(lo, hi), curves):
            got = pk['path'][pk['curve_start'][c]:pk['curve_start'][c + 1]]
            np.testing.assert_array_equal(got, np.hstack(ref)[:3].T.astype(np.float32))
            assert pk['curve_gear'][c] == ref[0][-1, 0]
    assert pk['curve_start'][0] == 0 and pk['curve_start'][-1] == len(pk['path'])


def test_pack_paths_without_reverse_is_one_forward_curve_per_path():
    paths = [PATH, fwd_rev_fwd(), line(1, 0, 0, 0)]
    pk = pack_paths(paths)
    assert list(pk['path_curve']) == [0, 1, 2, 3]
    assert list(pk['curve_gear']) == [1, 1, 1]
    assert list(pk['curve_start']) == [0, len(PATH), len(PATH) + 61, len(PATH) + 62]
    np.testing.assert_array_equal(pk['path'][:len(PATH)], PATH_ARR.astype(np.float32))


def test_pack_paths_rejects_what_the_reference_cannot_follow():
    with pytest.raises(ValueError):
        pack_paths([])
    with pytest.raises(ValueError):
        pack_paths([PATH, []])                                  # the reference crashes on an empty path
    with pytest.raises(ValueError):
        pack_paths([fwd_rev_fwd(), PATH], enable_reverse=True)  # PATH's waypoints have no gear row
    with pytest.raises(ValueError):
        pack_paths([np.zeros((0, 4))], enable_reverse=True)


# ---- closed loop without a solver ----------------------------------------------------------------------------
def _fleet_paths():
    return [with_gear(PATH), fwd_rev_fwd(), line(40, 5.0, -3.0, 0.7), line(1, 2.0, 2.0, -0.4),
            line(2, -1.0, 4.0, 2.5)]


# (path, curve, index) of the 16 robots; every path has robots at its start and near its end
STARTS = [(0, 0, 0), (0, 0, 60), (0, 0, 121), (0, 0, 130),
          (1, 0, 0), (1, 0, 20), (1, 1, 12), (1, 2, 3),
          (2, 0, 0), (2, 0, 17), (2, 0, 33),
          (3, 0, 0), (3, 0, 0),
          (4, 0, 0), (4, 0, 1), (1, 2, 12)]


@pytest.mark.parametrize('enable_reverse', [False, True])
@pytest.mark.parametrize('dyn', ['acker', 'diff'])
def test_closed_loop_matches_one_host_mpc_per_robot(enable_reverse, dyn):
    """16 robots on 5 paths, 60 steps with scripted controls; the next state of each robot is its reference two
    columns ahead (plus a fixed offset), so robots move along their paths, switch curves and arrive.  The host MPCs'
    paths are restored before each call: the reference rewrites an exhausted path's last heading in place and keeps
    that across calls, which the device does only within one call (INTEGRATION.md §3, deviation (i))."""
    T, steps, speed, thr = 8, 60, 4.0, 1
    paths = _fleet_paths()
    B = len(STARTS)
    pk = pack_paths(paths, enable_reverse)
    hosts, state = [], np.zeros((B, 3), np.float32)
    for b, (w, c, i) in enumerate(STARTS):
        m = MPC(_Car(dyn), copy.deepcopy(paths[w]), receding=T, sample_time=DT, enable_reverse=enable_reverse,
                goal_index_threshold=thr, solver_cls=_ScriptedSolver)
        m.rda.owner = m
        curve = m.curve_list[c] if enable_reverse else m.ref_path
        if not enable_reverse:
            i += sum(len(x) for x in _split_reference(copy.deepcopy(paths[w]))[:c])
            c = 0
        m.cur_index = min(i, len(curve) - 1)
        if enable_reverse:
            m.curve_index = c
        hosts.append(m)
        state[b] = np.asarray(curve[m.cur_index], float).reshape(-1)[:3] + [0.05, -0.03, 0.02]
    robot_path = np.array([w for w, _, _ in STARTS], np.int32)
    curve_index = np.array([m.curve_index if enable_reverse else 0 for m in hosts], np.int32)
    cur_index = np.array([m.cur_index for m in hosts], np.int32)
    cur_vel = np.zeros((B, 2, T), np.float32)
    switches = arrivals = 0
    for k in range(steps):
        u = np.stack([np.vstack([2.0 + 0.3 * np.sin(0.7 * k + b) + 0.01 * np.arange(T),
                                 0.2 * np.cos(0.3 * k + 2 * b) - 0.005 * np.arange(T)]) for b in range(B)])
        u = u.astype(np.float32)
        nom, ref, near, solver_speed = fleet_twin.pre_process_paths(pk, dyn, T, DT, L, state, cur_vel,
                                                                    np.full(B, speed, np.float32), robot_path,
                                                                    curve_index, cur_index)
        near, curve_index, u_kept, cur_vel, arrive = fleet_twin.post_process_paths(pk, T, robot_path, thr, near,
                                                                                   curve_index, u)
        for b, m in enumerate(hosts):
            m.ref_path = copy.deepcopy(paths[STARTS[b][0]])
            if enable_reverse:
                m.curve_list = m.split_path(m.ref_path)
            m.rda.u = u[b].astype(float)
            before = m.curve_index if enable_reverse else 0
            _, info = m.control(state[b].astype(float).reshape(3, 1), speed, [])
            seen = m.rda.seen
            np.testing.assert_allclose(nom[b], seen['nom_s'], atol=TOL, err_msg=f'{k} {b}')
            np.testing.assert_allclose(ref[b], seen['ref'], atol=TOL, err_msg=f'{k} {b}')
            assert solver_speed[b] == np.float32(seen['speed']), (k, b)
            assert bool(arrive[b]) == info['arrive'], (k, b)
            np.testing.assert_array_equal(cur_vel[b], np.asarray(m.cur_vel_array, np.float32))
            np.testing.assert_array_equal(u_kept[b], np.asarray(m.cur_vel_array, np.float32))
            if enable_reverse and m.curve_index >= len(m.curve_list):
                # past the last curve: the reference would raise IndexError on its next call; the device keeps the
                # robot on its last curve at the closest waypoint it found
                m.curve_index, m.cur_index = len(m.curve_list) - 1, seen['near']
            if enable_reverse:
                switches += int(m.curve_index != before)
            arrivals += int(info['arrive'])
            assert int(near[b]) == m.cur_index, (k, b)
            assert int(curve_index[b]) == (m.curve_index if enable_reverse else 0), (k, b)
            state[b] = seen['ref'][:, 2] + [0.02, -0.01, 0.005]
        cur_index = near
    assert arrivals >= 3 * steps
    if enable_reverse:
        assert switches >= 4


def test_pre_process_matches_reference_goldens_inside_a_path_set():
    """The golden path as path 2 of 4, the other paths of different lengths before and after it."""
    rng = np.random.default_rng(1)
    other = lambda n: [np.array([[x], [y], [h]]) for x, y, h in rng.uniform(-20, 20, (n, 3))]
    pk = pack_paths([other(7), other(31), PATH, other(3)])
    for rec in GOLD['pre_process']:
        T = rec['T']
        nom, ref, near, speed = fleet_twin.pre_process_paths(
            pk, rec['dynamics'], T, 0.1, L, np.ravel(rec['state'])[None, :3], np.array(rec['vel'])[None],
            np.array([4.0]), [2], [0], [rec['index']])
        np.testing.assert_allclose(nom[0], rec['state_pre'], atol=TOL)
        np.testing.assert_allclose(ref[0], rec['ref'], atol=TOL)
        assert near[0] == rec['new_index'] and speed[0] == 4.0


@pytest.mark.parametrize('dyn', ['acker', 'diff', 'omni'])
def test_robots_without_a_path(dyn):
    """robot_path outside [0, W): the nominal rollout as usual, a reference holding the current state, index 0 and
    gear +1, then zero controls and arrive; robots with a path in the same batch are unaffected."""
    T = 6
    rng = np.random.default_rng(2)
    pk = pack_paths([fwd_rev_fwd(), PATH], enable_reverse=False)
    robot_path = np.array([-1, 2, 1, 1 << 30, 0], np.int32)
    B = len(robot_path)
    state = np.stack([PATH_ARR[5] + rng.normal(0, 0.2, 3) for _ in range(B)]).astype(np.float32)
    vel = np.stack([np.vstack([rng.uniform(1, 3, T), rng.uniform(-0.2, 0.2, T)]) for _ in range(B)]).astype(np.float32)
    nom, ref, near, speed = fleet_twin.pre_process_paths(pk, dyn, T, DT, L, state, vel, np.full(B, -3.0, np.float32),
                                                         robot_path, np.full(B, 5, np.int32), np.full(B, 4, np.int32))
    for b in (0, 1, 3):
        m = MPC(_Car(dyn), [], receding=T, sample_time=DT, solver_cls=_ScriptedSolver)
        m.cur_vel_array = vel[b].astype(float)
        cur, cols = state[b].astype(float).reshape(3, 1), [state[b].astype(float).reshape(3, 1)]
        model = {'acker': lambda s, v: m.motion_predict_model_acker(s, v, L, DT),
                 'diff': lambda s, v: m.motion_predict_model_diff(s, v, DT),
                 'omni': lambda s, v: m.motion_predict_model_omni(s, v, DT)}[dyn]
        for t in range(T):
            cur = model(cur, m.cur_vel_array[:, t:t + 1])
            cols.append(cur)
        np.testing.assert_allclose(nom[b], np.hstack(cols), atol=TOL)
        np.testing.assert_array_equal(ref[b], np.repeat(state[b][:, None], T + 1, 1))
        assert near[b] == 0 and speed[b] == -3.0
    assert near[2] >= 4 and near[4] >= 4                                   # robots with a path
    u = rng.normal(0, 1, (B, 2, T)).astype(np.float32)
    near2, ci, u2, cur_vel, arrive = fleet_twin.post_process_paths(pk, T, robot_path, 1, np.zeros(B, np.int32),
                                                                   np.zeros(B, np.int32), u)
    assert list(arrive) == [1, 1, 0, 1, 0]
    assert not u2[[0, 1, 3]].any() and not cur_vel[[0, 1, 3]].any()
    np.testing.assert_array_equal(u2[[2, 4]], u[[2, 4]])
    np.testing.assert_array_equal(cur_vel, u2)
    assert not near2.any() and not ci.any()


def test_path_usage_errors_are_return_codes():
    """Checked before any device work, so this runs without a GPU."""
    lib = _cabi.load()
    pre, post = lib.rda_pre_process_paths, lib.rda_post_process_paths
    fake = ctypes.c_void_p(256)
    # pre: B, T, dynamics, dt, L, state, cur_vel, ref_speed, path, W, path_curve, curve_start, curve_gear, robot_path,
    # curve_index, start_index, threshold, ind_range, nom_s, ref_s, near_index, solver_speed, stream
    nul = [None] * 4
    assert pre(0, 8, 0, 0.1, 3.0, *nul, 1, *[None] * 6, 0.1, 10, *nul, None) == -1          # B < 1
    assert pre(4, 0, 0, 0.1, 3.0, *nul, 1, *[None] * 6, 0.1, 10, *nul, None) == -1          # T < 1
    assert pre(4, 8, 3, 0.1, 3.0, *nul, 1, *[None] * 6, 0.1, 10, *nul, None) == -1          # unknown dynamics
    assert pre(4, 8, 0, 0.1, 3.0, *[fake] * 4, 0, *[fake] * 6, 0.1, 10, *[fake] * 4, None) == -1   # W < 1
    # post: B, T, W, path_curve, curve_start, robot_path, goal_index_threshold, near_index, curve_index, u_opt,
    # cur_vel, arrive, stream
    assert post(0, 8, 1, fake, fake, fake, 1, fake, fake, fake, fake, fake, None) == -1      # B < 1
    assert post(4, 0, 1, fake, fake, fake, 1, fake, fake, fake, fake, fake, None) == -1      # T < 1
    assert post(4, 8, 0, fake, fake, fake, 1, fake, fake, fake, fake, fake, None) == -1      # W < 1
    if torch.cuda.is_available():                     # below, a missing check would launch on placeholder pointers
        return
    pre_ptrs = list(range(5, 9)) + list(range(10, 13)) + [18, 19, 20]      # required pointer arguments
    for missing in pre_ptrs:
        args = [4, 8, 0, 0.1, 3.0] + [fake] * 4 + [2] + [fake] * 6 + [0.1, 10] + [fake] * 4 + [None]
        args[missing] = None
        assert pre(*args) == -1, missing
    for missing in (3, 4, 7, 8, 9):
        args = [4, 8, 2, fake, fake, fake, 1, fake, fake, fake, fake, fake, None]
        args[missing] = None
        assert post(*args) == -1, missing
