"""World shapes along given trajectories on the CPU: the twin of rda_convert_world_obstacles_traj and
rda_convert_world_obstacles_horizon_traj (tests/cpu_twin/world_traj.cpp) against the reference's statement of such a
world (each trajectory shape an rdaobs with lists of T+1 rows, the others through MPC.convert_rda_obstacle, sorted by
the stage-0 key, then pack_obstacles) and against the float64 horizon key of oracle/clearance.py; trajectories that
stand still against the static shapes, bit for bit; the horizon bounds; pack_worlds; usage errors."""
import ctypes
from collections import namedtuple

import numpy as np
import pytest

import horizon_twin as ht
import world_traj_twin as wt
import world_twin
from oracle import clearance
from rda_planner_b200 import _cabi
from rda_planner_b200.frontend import BatchedMPC, pack_shapes, pack_worlds, robot_body
from rda_planner_b200.mpc import MPC, polygon_halfspaces, rdaobs
from rda_planner_b200.rda_solver import pack_obstacles
from rda_planner_b200.scenarios import disc_robot, rectangle_robot

car = namedtuple('car', 'G h cone_type wheelbase max_speed max_acce dynamics')
TObs = namedtuple('TObs', 'center radius vertex cone_type velocity trajectory')
DT = float(np.float32(0.1))
STATE = np.array([[10.0], [5.0], [0.3]])
F32 = lambda a: np.asarray(a, np.float32).astype(float)


class _NoSolver:
    def __init__(self, *a, **k):
        pass


def _polygon(rng, c, n, size, ccw=None):
    ang = np.sort(rng.uniform(0, 2 * np.pi, n))
    while np.min(np.diff(np.r_[ang, ang[0] + 2 * np.pi])) < 0.3:
        ang = np.sort(rng.uniform(0, 2 * np.pi, n))
    v = np.asarray(c).reshape(2, 1) + size * np.vstack([np.cos(ang), np.sin(ang)])
    return v[:, ::-1] if (rng.random() < 0.5 if ccw is None else not ccw) else v


def _arc(rng, T, c0):
    """Stage offsets [T+1, 2] and headings [T+1] of a walk along an arc that may stop."""
    v, w = rng.uniform(0.3, 2.0), rng.uniform(-1.5, 1.5)
    th0 = rng.uniform(-np.pi, np.pi)
    stop = int(rng.integers(1, T + 2))
    p, th = np.zeros((T + 1, 2)), np.zeros(T + 1)
    th[0] = th0
    for t in range(1, T + 1):
        go = t < stop
        th[t] = th[t - 1] + (w * DT if go else 0.0)
        p[t] = p[t - 1] + (v * DT * np.array([np.cos(th[t - 1]), np.sin(th[t - 1])]) if go else 0.0)
    return p + np.asarray(c0).reshape(1, 2), th - th0


def traj_world(rng, count, T, E=8, span=12.0, origin=(10.0, 5.0), still=False):
    """`count` obstacles: static, moving at a velocity and along trajectories (a polygon turning along an arc, a disc
    walking an arc and stopping), polygons of 3..E vertices in either orientation, float32-exact.  still: every
    trajectory stands at the shape's position."""
    obs = []
    for j in range(count):
        c = np.asarray(origin) + rng.uniform(-span, span, 2)
        disc = j % 4 == 0
        mode = j % 3                                        # 0 static, 1 velocity, 2 trajectory
        vel = F32(rng.uniform(-1.5, 1.5, (2, 1))) if mode == 1 else np.zeros((2, 1))
        if disc:
            ctr, rad = F32(c.reshape(2, 1)), float(np.float32(rng.uniform(0.2, 1.5)))
            tr = None
            if mode == 2:
                p, _ = _arc(rng, T, c)
                tr = F32(np.tile(c.reshape(1, 2), (T + 1, 1)).T if still else p.T)
                ctr = tr[:, :1].copy()
            obs.append(TObs(ctr, rad, None, 'norm2', vel, tr))
            continue
        n = int(rng.integers(3, E + 1))
        body = _polygon(rng, (0.0, 0.0), n, rng.uniform(0.3, 2.0))
        vert = F32(body + c.reshape(2, 1))
        tr = None
        if mode == 2:
            p, th = _arc(rng, T, c)
            tr = []
            for t in range(T + 1):
                R = np.array([[np.cos(th[t]), -np.sin(th[t])], [np.sin(th[t]), np.cos(th[t])]])
                tr.append(vert if still else F32(R @ body + p[t].reshape(2, 1)))
            vert = tr[0]
        obs.append(TObs(None, None, vert, 'Rpositive', vel, tr))
    return obs


def reference_list(obs, T, order, state=STATE):
    """The reference's statement of a world with trajectories: each trajectory shape an rdaobs whose A and b are lists of
    T+1 stage rows (polygon_halfspaces of the stage vertices, disc rows of the stage centre), the others through
    MPC.convert_rda_obstacle, sorted (stable) by rda_obs_distance of the stage-0 shape."""
    m = MPC(car(None, None, 'Rpositive', 3.0, [10, 1], [10, 0.5], 'acker'), [], receding=T, sample_time=DT,
            solver_cls=_NoSolver)
    m.state = state
    out = []
    for o in obs:
        if o.trajectory is None:
            out.append(m.convert_rda_obstacle([o], state, False)[0])
        elif o.cone_type == 'norm2':
            A0 = np.array([[1, 0], [0, 1], [0, 0]])
            out.append(rdaobs([A0] * (T + 1), [np.vstack((o.trajectory[:, t:t + 1], [[-o.radius]]))
                                                for t in range(T + 1)], 'norm2', o.trajectory[:, :1], None))
        else:
            rows = [polygon_halfspaces(np.asarray(v)) for v in o.trajectory]
            out.append(rdaobs([r[0] for r in rows], [r[1] for r in rows], 'Rpositive', None, o.trajectory[0]))
    if order:
        out.sort(key=m.rda_obs_distance)
    return out


def _packed_reference(obs, T, N, E, order):
    Ah, bh, kh, ch, tvh = pack_obstacles(reference_list(obs, T, order), T, N, E)
    if not tvh:
        Ah, bh = np.repeat(Ah, T + 1, axis=1), np.repeat(bh, T + 1, axis=1)
    return Ah, bh, kh, ch


@pytest.mark.parametrize('order', [False, True])
@pytest.mark.parametrize('count', [0, 1, 7, 20, 90])
def test_twin_matches_reference_statement(order, count):
    T, N, E = 8, 12, 8
    rng = np.random.default_rng(100 + count + order)
    obs = traj_world(rng, count, T, E)
    world = pack_worlds([obs])
    lst = wt.robot_list(world, None, None, 0)
    A, b, kind, cnt, ids = wt.select(lst, N, T, E, DT, order, STATE)
    assert cnt == count
    if count == 0:
        assert not A.any() and not b.any() and np.all(kind == _cabi.OBS_POLYGON) and np.all(ids == -1)
        return
    Ah, bh, kh, ch = _packed_reference(obs, T, N, E, order)
    assert ch == count and list(kind) == list(kh)
    np.testing.assert_allclose(A, Ah, atol=1e-5)
    np.testing.assert_allclose(b, bh, atol=1e-4)
    assert np.all((ids >= 0) & (ids < count))


def test_out_of_range_trajectory_indices_mean_none():
    """A traj value outside [0, K) is the shape's own xy and vel (pack_worlds: stage 0, standing)."""
    T, N, E = 6, 30, 8
    rng = np.random.default_rng(7)
    obs = traj_world(rng, 30, T, E)
    world = pack_worlds([obs])
    K = len(world['traj_xy'])
    has = np.nonzero(world['traj'] >= 0)[0]
    bad = {int(has[0]): K, int(has[1]): -7, int(has[2]): 2 ** 31 - 1}
    for j, v in bad.items():
        world['traj'][j] = v
    ref = [o._replace(trajectory=None) if j in bad else o for j, o in enumerate(obs)]     # at stage 0, standing
    for order in (False, True):
        A, b, kind, cnt, _ = wt.select(wt.robot_list(world, None, None, 0), N, T, E, DT, order, STATE)
        Ah, bh, kh, _ = _packed_reference(ref, T, N, E, order)
        assert list(kind) == list(kh)
        np.testing.assert_allclose(A, Ah, atol=1e-5)
        np.testing.assert_allclose(b, bh, atol=1e-4)


def _static_twin(obs):
    return [o._replace(trajectory=None) for o in obs]


@pytest.mark.parametrize('order', [False, True])
def test_standing_trajectory_is_the_static_shape_bit_for_bit(order):
    T, N, E = 7, 16, 8
    rng = np.random.default_rng(11)
    obs = traj_world(rng, 60, T, E, still=True)
    world = pack_worlds([obs])
    static = pack_worlds([_static_twin(obs)])
    assert 'traj' in world and 'traj' not in static
    for k in ('kind', 'nv', 'xy', 'radius', 'vel', 'start'):
        np.testing.assert_array_equal(world[k], static[k])
    for state in (STATE, np.array([0.0, 0.0, 0.0]), np.array([20.0, -3.0, 1.0])):
        A, b, kind, cnt, ids = wt.select(wt.robot_list(world, None, None, 0), N, T, E, DT, order, state)
        As, bs, ks, cs = world_twin.convert_world_obstacles(static, 0, N, T, E, DT, True, order, state)
        assert cnt == cs and np.array_equal(kind, ks)
        assert np.array_equal(A, As) and np.array_equal(b, bs)
        A2, b2, k2, c2, ids2 = wt.select(wt.robot_list(static, None, None, 0), N, T, E, DT, order, state)
        assert np.array_equal(ids, ids2)


def _bodies(rng):
    poly = np.zeros((8, 2), np.float32)
    ang = np.sort(rng.uniform(0, 2 * np.pi, 5))
    poly[:5] = (np.c_[np.cos(ang), np.sin(ang)] * rng.uniform(0.8, 1.6) + [0.7, 0.1]).astype(np.float32)
    return {'rect': robot_body(rectangle_robot()),
            'poly5': {'kind': _cabi.OBS_POLYGON, 'nv': 5, 'xy': poly, 'radius': 0.0},
            'disc': robot_body(disc_robot(0.9, center=(0.3, -0.1)))}


def _poses(rng, T, origin=(10.0, 5.0), span=6.0, broken=True):
    out = []
    for _ in range(2):
        p0 = np.asarray(origin) + rng.uniform(-span, span, 2)
        th, v = rng.uniform(-4 * np.pi, 4 * np.pi), rng.uniform(0, 6)
        t = np.arange(T + 1) * DT
        out.append(np.vstack([p0[0] + v * t * np.cos(th), p0[1] + v * t * np.sin(th), th + 0.3 * t]).astype(np.float32))
    if broken:
        out[0][0, 2] = np.nan
        out[1][2, T] = np.inf
    return out


def test_standing_trajectory_horizon_order_is_the_static_shape_bit_for_bit():
    T, N, E = 6, 10, 8
    rng = np.random.default_rng(12)
    obs = traj_world(rng, 50, T, E, still=True)
    world, static = pack_worlds([obs]), pack_worlds([_static_twin(obs)])
    for name, body in _bodies(rng).items():
        nom, ref = _poses(rng, T)
        A, b, kind, cnt, ids, keys = wt.horizon_select(wt.robot_list(world, None, None, 0), N, T, E, DT, nom, ref, body)
        As, bs, ks, cs, keys_s = ht.select(ht.robot_list(static, None, None, 0), N, T, E, DT, True, nom, ref, body)
        assert cnt == cs and np.array_equal(kind, ks), name
        assert np.array_equal(A, As) and np.array_equal(b, bs), name
        assert np.array_equal(keys, keys_s), name
        order = np.argsort(keys_s, kind='stable')
        assert np.array_equal(ids, order[np.minimum(np.arange(N), cnt - 1)]), name


def _oracle_body(body):
    xy = np.asarray(body['xy'], np.float32).astype(float)
    if body['kind'] == _cabi.OBS_CIRCLE:
        return {'disc': True, 'c': xy[0], 'r': float(np.float32(body['radius']))}
    return {'disc': False, 'V': xy[:int(body['nv'])]}


def _rows_of_every_entry(lst, T, E):
    """Each entry's T+1 stage rows, from the twin in list order with one slot per entry."""
    rows = []
    for j in range(len(lst['kind'])):
        one = {k: (v[j:j + 1] if k not in ('traj_xy',) else v) for k, v in lst.items() if k != 'plan_xy'}
        if 'plan_xy' in lst:
            one['plan_xy'] = lst['plan_xy'][j:j + 1]
        one['id'] = np.zeros(1, np.int32)
        A, b, _, _, _ = wt.select(one, 1, T, E, DT, False, np.zeros(3))
        rows.append((A[0], b[0]))
    return rows


@pytest.mark.parametrize('body_name', ['rect', 'poly5', 'disc'])
def test_horizon_twin_matches_float64_key(body_name):
    T, N, E = 8, 6, 8
    rng = np.random.default_rng(200 + len(body_name))
    body = _bodies(rng)[body_name]
    obs = traj_world(rng, 40, T, E, span=6.0)
    world = pack_worlds([obs])
    lst = wt.robot_list(world, None, None, 0)
    nom, ref = _poses(rng, T)
    A, b, kind, cnt, ids, keys = wt.horizon_select(lst, N, T, E, DT, nom, ref, body)
    rows = _rows_of_every_entry(lst, T, E)
    ob = _oracle_body(body)
    okeys = np.full(cnt, np.inf)
    for j in range(cnt):
        for s in (nom, ref):
            for t in range(T + 1):
                if np.all(np.isfinite(s[:, t])):
                    okeys[j] = min(okeys[j], clearance.cell(ob, s[:, t], int(lst['kind'][j]), rows[j][0][t],
                                                            rows[j][1][t]))
    assert np.all(np.isfinite(keys))
    assert np.all(np.abs(keys - okeys) <= 1e-9 * np.maximum(1, np.abs(okeys)))
    tw = np.argsort(keys, kind='stable')
    for n in range(N):
        j = tw[min(n, cnt - 1)]
        assert ids[n] == j and kind[n] == lst['kind'][j]
        assert np.array_equal(A[n], rows[j][0]) and np.array_equal(b[n], rows[j][1])
    lb_disc, lb_pose = wt.bounds(lst, T, E, DT, nom, ref, body)
    assert np.all(lb_disc <= keys) and np.all(lb_pose <= keys)
    on = lst['traj'] >= 0
    assert np.all(lb_disc[on] == -np.inf)                   # no one-disc bound for a trajectory


def test_horizon_bounds_with_non_finite_stages():
    T, E = 6, 8
    rng = np.random.default_rng(31)
    obs = traj_world(rng, 60, T, E, span=4.0)
    world = pack_worlds([obs])
    on = np.nonzero(world['traj'] >= 0)[0]
    bad = [(world['traj'][on[0]], 3, 0, 0, np.nan), (world['traj'][on[1]], 0, 1, 1, np.inf),
           (world['traj'][on[2]], T, 0, 1, -np.inf)]
    for k, t, v, c, val in bad:
        world['traj_xy'][k, t, v, c] = val
    lst = wt.robot_list(world, None, None, 0)
    for body in _bodies(rng).values():
        nom, ref = _poses(rng, T, span=3.0)
        keys = wt.horizon_select(lst, 4, T, E, DT, nom, ref, body)[5]
        lb_disc, lb_pose = wt.bounds(lst, T, E, DT, nom, ref, body)
        assert not np.any(lb_disc > keys) and not np.any(lb_pose > keys)
        for k, *_ in bad:
            j = int(np.nonzero(lst['traj'] == k)[0][0])
            assert lb_pose[j] == -np.inf and lb_disc[j] == -np.inf
        assert np.any(keys < 0.5)


def test_pack_worlds_trajectory_layout():
    T = 5
    rng = np.random.default_rng(3)
    obs = traj_world(rng, 24, T)
    w = pack_worlds([obs[:10], [], obs[10:]])
    has = [j for j, o in enumerate(obs) if o.trajectory is not None]
    assert w['traj'].dtype == np.int32 and w['traj'].shape == (24,)
    assert w['traj_xy'].dtype == np.float32 and w['traj_xy'].shape == (len(has), T + 1, 8, 2)
    assert list(np.nonzero(w['traj'] >= 0)[0]) == has and list(w['traj'][has]) == list(range(len(has)))
    for k, j in enumerate(has):
        o = obs[j]
        if o.cone_type == 'norm2':
            np.testing.assert_array_equal(w['traj_xy'][k, :, 0], np.asarray(o.trajectory, np.float32).T)
            assert not w['traj_xy'][k, :, 1:].any()
        else:
            nv = o.vertex.shape[1]
            for t in range(T + 1):
                np.testing.assert_array_equal(w['traj_xy'][k, t, :nv], np.asarray(o.trajectory[t], np.float32).T)
            assert not w['traj_xy'][k, :, nv:].any()
        np.testing.assert_array_equal(w['xy'][j], w['traj_xy'][k, 0])
        assert not w['vel'][j].any()
    assert set(pack_worlds([[o for o in obs if o.trajectory is None]])) == {'kind', 'nv', 'xy', 'radius', 'vel',
                                                                             'start'}


def test_pack_worlds_refuses_bad_trajectories():
    T = 4
    rng = np.random.default_rng(5)
    obs = traj_world(rng, 12, T)
    poly = next(o for o in obs if o.trajectory is not None and o.cone_type == 'Rpositive')
    disc = next(o for o in obs if o.trajectory is not None and o.cone_type == 'norm2')
    with pytest.raises(ValueError, match='stage counts'):
        pack_worlds([[poly, disc._replace(trajectory=disc.trajectory[:, :T])]])
    with pytest.raises(ValueError, match='vertices'):
        pack_worlds([[poly._replace(trajectory=poly.trajectory[:2] + [poly.trajectory[2][:, :-1]] +
                                    poly.trajectory[3:])]])
    bad = [np.array(v) for v in poly.trajectory]
    bad[1][0, 0] = np.nan
    with pytest.raises(ValueError, match='non-finite'):
        pack_worlds([[poly._replace(trajectory=bad)]])
    c = np.array(disc.trajectory)
    c[1, 2] = np.inf
    with pytest.raises(ValueError, match='non-finite'):
        pack_worlds([[disc._replace(trajectory=c)]])
    big = next(o for o in obs if o.cone_type == 'Rpositive' and o.vertex.shape[1] > 4 and o.trajectory is not None) \
        if any(o.cone_type == 'Rpositive' and o.vertex.shape[1] > 4 and o.trajectory is not None for o in obs) else None
    ang = np.linspace(0, 2 * np.pi, 6, endpoint=False)
    hexa = np.vstack([np.cos(ang), np.sin(ang)])
    big = big or TObs(None, None, hexa, 'Rpositive', np.zeros((2, 1)), [hexa] * (T + 1))
    with pytest.raises(ValueError):
        pack_worlds([[big]], max_edge_num=4)
    with pytest.raises(ValueError, match='pack_worlds'):
        pack_shapes([[poly]])


def _mpc_without_device(order=True, T=5):
    mpc = BatchedMPC.__new__(BatchedMPC)
    mpc.obstacle_order = order
    mpc.device, mpc.batch, mpc.T = None, 2, T
    return mpc


def test_batched_mpc_refuses_trajectory_worlds_it_cannot_take():
    """Checked before any device work, on a constructed object without a device."""
    T = 5
    world = pack_worlds([traj_world(np.random.default_rng(2), 6, T)])
    for order in (True, False, 'horizon'):
        with pytest.raises(ValueError, match='time_varying'):
            _mpc_without_device(order, T).control(np.zeros((2, 3)), world=world)
        short = dict(world, traj_xy=world['traj_xy'][:, :T])
        with pytest.raises(ValueError, match='stages'):
            _mpc_without_device(order, T).control(np.zeros((2, 3)), world=short, time_varying=True)
    with pytest.raises(ValueError, match='shapes='):
        _mpc_without_device(True, T).control(np.zeros((2, 3)), shapes=world, time_varying=True)


def _traj_call(lib, horizon, **kw):
    vp = ctypes.c_void_p
    buf = ctypes.create_string_buffer(8192)
    p = ctypes.cast(buf, vp)
    aligned = ctypes.c_void_p((ctypes.addressof(buf) + 15) // 16 * 16)
    head = dict(B=2, W=1, N=4, T=5, E=4, dt=0.1, tv=1)
    if horizon:
        head.update(nom=p, ref=p, bkind=_cabi.OBS_POLYGON, bnv=4, bxy=p, brad=0.0, bxy_b=None, brad_b=None)
    else:
        head.update(order=1, state=p)
    args = dict(head, start=p, rw=None, kind=p, nv=p, xy=p, rad=p, vel=p, fstart=None, frobot=None, fkind=None,
                fnv=None, fxy=None, frad=None, fvel=None, fplan=None, A=p, b=p, okind=p, ocount=p, oid=None,
                traj=p, K=3, traj_xy=aligned)
    args.update(kw)
    f = lib.rda_convert_world_obstacles_horizon_traj if horizon else lib.rda_convert_world_obstacles_traj
    return f(*args.values(), None), aligned


@pytest.mark.parametrize('horizon', [False, True])
def test_traj_usage_errors_are_return_codes(horizon):
    """Checked before any launch, so this runs without a GPU."""
    lib = _cabi.load()
    aligned = _traj_call(lib, horizon, B=0)[1]
    misaligned = ctypes.c_void_p(aligned.value + 4)
    assert _traj_call(lib, horizon, traj=None)[0] == _cabi.E_ARG
    assert _traj_call(lib, horizon, traj_xy=None)[0] == _cabi.E_ARG
    assert _traj_call(lib, horizon, traj_xy=misaligned)[0] == _cabi.E_ARG
    assert _traj_call(lib, horizon, K=0)[0] == _cabi.E_ARG
    assert _traj_call(lib, horizon, tv=0)[0] == _cabi.E_ARG
    assert _traj_call(lib, horizon, B=0)[0] == _cabi.E_ARG
    assert _traj_call(lib, horizon, start=None)[0] == _cabi.E_ARG
    assert _traj_call(lib, horizon, N=_cabi.MAX_WORLD_SLOTS + 1)[0] == _cabi.E_UNSUPPORTED
    assert _traj_call(lib, horizon, E=9)[0] == _cabi.E_UNSUPPORTED
    p = ctypes.cast(ctypes.create_string_buffer(64), ctypes.c_void_p)
    assert _traj_call(lib, horizon, fstart=p)[0] == _cabi.E_ARG    # a fleet without its arrays
    assert _traj_call(lib, horizon, fplan=p)[0] == _cabi.E_ARG     # plans without a fleet


def test_new_symbols_are_exported():
    lib = _cabi.load()
    for name in ('rda_convert_world_obstacles_traj', 'rda_convert_world_obstacles_horizon_traj'):
        assert name in _cabi.EXPORTS
        assert getattr(lib, name).restype is ctypes.c_int


def test_conversions_refuse_trajectory_tables_they_cannot_read():
    """traj_xy / traj of the wrong shape, dtype, layout or device are ValueErrors before any launch (CPU tensors here:
    the robots' device is the CPU, so this runs without a GPU)."""
    import torch
    from rda_planner_b200.frontend import convert_world_obstacles_batch
    T = 5
    world = {k: torch.as_tensor(v) for k, v in pack_worlds([traj_world(np.random.default_rng(4), 9, T)]).items()}
    state = torch.zeros((2, 3))
    bad = {'float64': dict(traj_xy=world['traj_xy'].double()),
           'rows': dict(traj_xy=world['traj_xy'][:, :, :4].contiguous()),
           'strided': dict(traj_xy=world['traj_xy'].transpose(2, 3).contiguous().transpose(2, 3)),
           'int64': dict(traj=world['traj'].long()),
           'length': dict(traj=world['traj'][:-1].contiguous()),
           'host': dict(traj_xy=world['traj_xy'].numpy())}
    for name, change in bad.items():
        with pytest.raises(ValueError, match='traj'):
            convert_world_obstacles_batch(dict(world, **change), state, None, 4, T, 8, DT, True)
        print(name, 'refused')
