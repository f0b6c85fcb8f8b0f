"""Obstacle selection from shared worlds of any size (rda_convert_world_obstacles): the CPU twin
(tests/cpu_twin/world_obstacles.cpp) against the host front end (mpc.MPC.convert_rda_obstacle over the whole list,
then pack_obstacles) and against the per-robot core; pack_worlds; the entry point's usage errors.  No GPU."""
import ctypes
from collections import namedtuple

import numpy as np
import pytest

import shim
import world_twin
from rda_planner_b200 import _cabi
from rda_planner_b200.frontend import pack_shapes, pack_worlds
from rda_planner_b200.mpc import MPC
from rda_planner_b200.rda_solver import pack_obstacles

car = namedtuple('car', 'G h cone_type wheelbase max_speed max_acce dynamics')
Obs = namedtuple('Obs', 'center radius vertex cone_type velocity')
STATE = np.array([[10.0], [5.0], [0.3]])


class _NoSolver:
    def __init__(self, *a, **k):
        pass


def world_of(rng, count, origin=(10.0, 5.0), spread=30.0, max_nv=5):
    """`count` shapes around `origin`: discs and polygons, clockwise and counter-clockwise, static and moving, with
    exact duplicates and shapes at exactly the same distance from `origin` (sort ties), float32-exact."""
    ox, oy = origin
    obs = []
    for j in range(count):
        vel = rng.uniform(-1, 1, (2, 1)) if j % 2 else np.zeros((2, 1))
        if j % 7 == 6 and obs:                                          # exact duplicate of an earlier shape
            obs.append(obs[int(rng.integers(0, len(obs)))])
            continue
        if j % 5 == 4:                                                  # disc on an axis at a distance used twice
            d = float(1 + (j // 10) % 4)
            cx, cy = [(ox + d, oy), (ox - d, oy), (ox, oy + d), (ox, oy - d)][(j // 5) % 4]
            obs.append(Obs(np.array([[cx], [cy]]), 0.25, None, 'norm2', vel))
            continue
        c = np.array([[ox], [oy]]) + rng.uniform(-spread, spread, (2, 1))
        if j % 3 == 0:
            obs.append(Obs(c, float(rng.uniform(0.3, 1.5)), None, 'norm2', vel))
        else:
            n = int(rng.integers(3, max_nv + 1))
            ang = np.linspace(0, 2 * np.pi, n, endpoint=False) + rng.uniform(0, 1)
            if j % 2:
                ang = ang[::-1]                                         # clockwise input
            obs.append(Obs(None, None, c + rng.uniform(0.5, 2.0) * np.vstack([np.cos(ang), np.sin(ang)]), 'Rpositive',
                           vel))
    return [o._replace(center=None if o.center is None else o.center.astype(np.float32).astype(float),
                       vertex=None if o.vertex is None else o.vertex.astype(np.float32).astype(float),
                       velocity=o.velocity.astype(np.float32).astype(float)) for o in obs]


def test_world_generator_has_ties():
    obs = world_of(np.random.default_rng(0), 200)
    m = MPC(car(None, None, 'Rpositive', 3.0, [10, 1], [10, 0.5], 'acker'), [], receding=4, solver_cls=_NoSolver)
    m.state = STATE
    keys = [m.rda_obs_distance(o) for o in m.convert_rda_obstacle(obs, STATE, False)]
    assert len(set(keys)) < len(keys) - 40


@pytest.mark.parametrize('order', [False, True])
@pytest.mark.parametrize('count', [0, 1, 19, 20, 65, 128, 1000])
def test_twin_matches_host_front_end_on_the_whole_list(order, count):
    """Sorting the whole world by distance (stable: ties keep list order), first N, padding by repetition."""
    T, N, E = 6, 20, 5
    rng = np.random.default_rng(500 + count)
    obs = world_of(rng, count)
    m = MPC(car(None, None, 'Rpositive', 3.0, [10, 1], [10, 0.5], 'acker'), [], receding=T, sample_time=0.1,
            solver_cls=_NoSolver)
    m.state = STATE
    rda_obs = m.convert_rda_obstacle(obs, STATE, order)
    tv = any(isinstance(o.A, list) for o in rda_obs[:N])
    world = pack_worlds([obs])
    assert int(world['start'][1]) == count
    A, b, kind, cnt = world_twin.convert_world_obstacles(world, 0, N, T, E, 0.1, tv, order, STATE)
    assert cnt == count
    if count == 0:
        assert not A.any() and not b.any() and list(kind) == [_cabi.OBS_POLYGON] * N
        return
    Ah, bh, kh, ch, tvh = pack_obstacles(list(rda_obs), T, N, E)
    assert tvh == tv and ch == count
    assert list(kind) == list(kh)
    np.testing.assert_allclose(A, Ah, atol=1e-5)
    np.testing.assert_allclose(b, bh, atol=1e-4)


@pytest.mark.parametrize('tv,order', [(False, True), (True, True), (True, False)])
def test_twin_matches_per_robot_core_up_to_64_shapes(tv, order):
    T, N, E = 7, 9, 6
    rng = np.random.default_rng(21)
    for count in (0, 1, 8, 9, 33, 64):
        obs = world_of(rng, count)
        state = np.array([10.0 + rng.normal(0, 3), 5.0 + rng.normal(0, 3), 0.0], np.float32)
        one = {k: v[0] for k, v in pack_shapes([obs], 64).items()}
        A1, b1, k1, c1 = shim.convert_obstacles(one, N, T, E, 0.1, tv, order, state)
        A, b, kind, cnt = world_twin.convert_world_obstacles(pack_worlds([obs]), 0, N, T, E, 0.1, tv, order, state)
        assert cnt == c1 == count
        assert list(kind) == list(k1)
        np.testing.assert_array_equal(A, A1)
        np.testing.assert_array_equal(b, b1)


def test_pack_worlds_offsets_and_shapes():
    rng = np.random.default_rng(4)
    worlds = [world_of(rng, 3), [], world_of(rng, 5), world_of(rng, 1)]
    w = pack_worlds(worlds)
    assert w['start'].dtype == np.int32 and list(w['start']) == [0, 3, 3, 8, 9]
    assert w['kind'].shape == (9,) and w['xy'].shape == (9, _cabi.MAX_EDGE, 2) and w['vel'].shape == (9, 2)
    for i, lst in enumerate(worlds):
        if not lst:
            continue
        per = pack_shapes([lst])
        lo, hi = w['start'][i], w['start'][i + 1]
        for k in ('kind', 'nv', 'xy', 'radius', 'vel'):
            np.testing.assert_array_equal(w[k][lo:hi], per[k][0])
    empty = pack_worlds([[], []])                         # still one (unused) entry to point at
    assert list(empty['start']) == [0, 0, 0] and empty['kind'].shape == (1,)
    with pytest.raises(ValueError):
        pack_worlds([])


@pytest.mark.parametrize('n', [2, 9])
def test_pack_worlds_rejects_what_pack_shapes_rejects(n):
    ang = np.linspace(0, 2 * np.pi, n, endpoint=False)
    bad = Obs(None, None, np.vstack([np.cos(ang), np.sin(ang)]), 'Rpositive', np.zeros((2, 1)))
    good = world_of(np.random.default_rng(1), 4)
    with pytest.raises(ValueError):
        pack_shapes([good + [bad]])
    with pytest.raises(ValueError):
        pack_worlds([good, good + [bad]])
    five = Obs(None, None, np.vstack([np.cos(ang[:5]), np.sin(ang[:5])]), 'Rpositive', None) if n == 9 else None
    if five is not None:                                  # max_edge_num below the polygon's vertex count
        with pytest.raises(ValueError):
            pack_shapes([[five]], max_edge_num=4)
        with pytest.raises(ValueError):
            pack_worlds([[five]], max_edge_num=4)


def test_world_usage_errors_are_return_codes():
    """Checked before any device work, so this runs without a GPU."""
    lib = _cabi.load()
    f = lib.rda_convert_world_obstacles
    nul = [None] * 13
    assert f(0, 1, 5, 10, 4, 0.1, 0, 1, *nul) == -1                           # B < 1
    assert f(4, 0, 5, 10, 4, 0.1, 0, 1, *nul) == -1                           # W < 1
    assert f(4, 1, 0, 10, 4, 0.1, 0, 1, *nul) == -1                           # N < 1
    assert f(4, 1, 5, 0, 4, 0.1, 0, 1, *nul) == -1                            # T < 1
    assert f(4, 1, _cabi.MAX_WORLD_SLOTS + 1, 10, 4, 0.1, 0, 1, *nul) == -2   # N above the limit
    assert f(4, 1, 5, 10, 2, 0.1, 0, 1, *nul) == -2                           # E < 3
    assert f(4, 1, 5, 10, _cabi.MAX_EDGE + 1, 0.1, 0, 1, *nul) == -2          # E > RDA_MAX_EDGE
    assert f(4, 1, 5, 10, 4, 0.1, 0, 1, *nul) == -1                           # missing pointers
    import torch
    if torch.cuda.is_available():                     # below, a missing check would launch on placeholder pointers
        return
    fake = ctypes.c_void_p(256)
    ptrs = [fake] * 12 + [None]
    for missing in range(1, 12):                                              # each required pointer (robot_world, 2, may be NULL)
        if missing == 2:
            continue
        p = list(ptrs)
        p[missing] = None
        assert f(4, 1, 5, 10, 4, 0.1, 0, 1, *p) == -1, missing
    p = list(ptrs)
    p[0] = None                                                               # no state to sort by
    assert f(4, 1, 5, 10, 4, 0.1, 0, 1, *p) == -1
