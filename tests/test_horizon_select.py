"""obstacle_order='horizon' on the CPU: the brute-force twin of rda_convert_world_obstacles_horizon against a numpy
oracle built on oracle/clearance.py, the lower bounds its kernel prunes with against the exact keys, the corridor map
where the reference's key drops both walls, and usage errors of the C ABI and of BatchedMPC."""
import ctypes
from collections import namedtuple

import numpy as np
import pytest

import fleet_plan_twin as fp
import horizon_twin as ht
import world_twin
from oracle import clearance
from rda_planner_b200 import _cabi
from rda_planner_b200.frontend import pack_worlds, robot_body
from rda_planner_b200.scenarios import disc_robot, rectangle_robot

Obs = namedtuple('Obs', 'center radius vertex cone_type velocity')
DT = 0.1


def _polygon(rng, c, n, size):
    ang = np.sort(rng.uniform(0, 2 * np.pi, n))
    while np.min(np.diff(np.r_[ang, ang[0] + 2 * np.pi])) < 0.3:
        ang = np.sort(rng.uniform(0, 2 * np.pi, n))
    r = size * rng.uniform(0.6, 1.0)
    v = np.asarray(c).reshape(2, 1) + r * np.vstack([np.cos(ang), np.sin(ang)])
    return v[:, ::-1] if rng.random() < 0.5 else v                     # either orientation


def _world(rng, count, span, E, moving=True):
    """count shapes over [-span, span]^2: discs and polygons of 3..E vertices, a third moving."""
    obs = []
    for j in range(count):
        vel = rng.uniform(-1.5, 1.5, (2, 1)) if moving and j % 3 == 1 else np.zeros((2, 1))
        c = rng.uniform(-span, span, 2)
        if j % 4 == 0:
            obs.append(Obs(c.reshape(2, 1), float(rng.uniform(0.2, 1.5)), None, 'norm2', vel))
        else:
            obs.append(Obs(None, None, _polygon(rng, c, int(rng.integers(3, E + 1)), rng.uniform(0.3, 2.5)),
                           'Rpositive', vel))
    return pack_worlds([obs])


def _poses(rng, T, span, broken=True):
    """nom, ref [3, T+1] float32: headings beyond +-pi, and (broken) one non-finite column in each."""
    out = []
    for _ in range(2):
        p0 = rng.uniform(-span / 2, span / 2, 2)
        th = rng.uniform(-4 * np.pi, 4 * np.pi)
        v = rng.uniform(0, 8)
        t = np.arange(T + 1) * DT
        s = np.vstack([p0[0] + v * t * np.cos(th), p0[1] + v * t * np.sin(th), th + 0.3 * t])
        out.append(s.astype(np.float32))
    if broken:
        out[0][0, 2 % (T + 1)] = np.nan
        out[1][2, T] = np.inf
    return out


def _bodies(rng):
    poly = np.zeros((8, 2), np.float32)
    ang = np.sort(rng.uniform(0, 2 * np.pi, 5))
    poly[:5] = (np.c_[np.cos(ang), np.sin(ang)] * rng.uniform(0.8, 1.6) + [0.7, 0.1]).astype(np.float32)
    return {'rect': robot_body(rectangle_robot()),
            'poly5': {'kind': _cabi.OBS_POLYGON, 'nv': 5, 'xy': poly, 'radius': 0.0},
            'disc': robot_body(disc_robot(0.9, center=(0.3, -0.1)))}


def _oracle_body(body):
    xy = np.asarray(body['xy'], np.float32).astype(float)
    if body['kind'] == _cabi.OBS_CIRCLE:
        return {'disc': True, 'c': xy[0], 'r': float(np.float32(body['radius']))}
    return {'disc': False, 'V': xy[:int(body['nv'])]}


def _all_rows(lst, T, E, tv):
    """Rows of every entry in list order (the existing twins, order off): A [count,Tc,E,2], b [count,Tc,E]."""
    count = len(lst['kind'])
    if lst['planned'].any():
        A = np.zeros((count, T + 1, E, 2), np.float32)
        b = np.zeros((count, T + 1, E), np.float32)
        for j in range(count):
            one = {k: np.asarray(lst[k][j:j + 1]) for k in ht.KEYS}
            one['planned'] = lst['planned'][j:j + 1]
            one['plan_xy'] = lst['plan_xy'][j:j + 1]
            A[j], b[j] = _plan_rows(one, T, E)
        return A, b
    world = dict({k: lst[k] for k in ht.KEYS}, start=np.array([0, count], np.int32))
    A, b, _, _ = world_twin.convert_world_obstacles(world, 0, count, T, E, DT, tv, False, np.zeros(3))
    return A, b


def _plan_rows(one, T, E):
    """Stage rows of one map-mate along its plan (fleet_plan_twin's list conversion, order off)."""
    import ctypes as C
    import shim
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    i32 = lambda a: np.ascontiguousarray(a, np.int32)
    A = np.zeros((1, T + 1, E, 2), np.float32)
    b = np.zeros((1, T + 1, E), np.float32)
    kind = np.zeros(1, np.int32)
    arrs = [f32(np.zeros(3)), i32(one['kind']), i32(one['nv']), f32(one['xy']), f32(one['radius']), f32(one['vel']),
            i32(one['planned']), f32(one['plan_xy'])]
    fn = shim.lib().shim_convert_plan_list
    fn.restype = C.c_int
    fn.argtypes = [C.c_int] * 4 + [C.c_double, C.c_int] + [C.c_void_p] * 11
    fn(1, 1, T, E, DT, 0, *[a.ctypes.data for a in arrs], A.ctypes.data, b.ctypes.data, kind.ctypes.data)
    return A[0], b[0]


def _oracle_keys(lst, T, E, tv, nom, ref, body):
    count = len(lst['kind'])
    A, b = _all_rows(lst, T, E, tv)
    ob = _oracle_body(body)
    keys = np.full(count, np.inf)
    for j in range(count):
        for s in (nom, ref):
            for t in range(T + 1):
                if not np.all(np.isfinite(s[:, t])):
                    continue
                c = t if tv else 0
                keys[j] = min(keys[j], clearance.cell(ob, s[:, t], int(lst['kind'][j]), A[j, c], b[j, c]))
    return keys, A, b


def _check_against_oracle(lst, N, T, E, tv, nom, ref, body):
    A, b, kind, cnt, keys = ht.select(lst, N, T, E, DT, tv, nom, ref, body)
    count = len(lst['kind'])
    assert cnt == count
    okeys, rowsA, rowsb = _oracle_keys(lst, T, E, tv, nom, ref, body)
    fin = np.isfinite(okeys)
    assert np.array_equal(fin, np.isfinite(keys))
    assert np.all(np.abs(keys[fin] - okeys[fin]) <= 1e-9 * np.maximum(1, np.abs(okeys[fin])))
    if count == 0:
        assert not A.any() and not b.any() and np.all(kind == _cabi.OBS_POLYGON)
        return keys
    tw = np.argsort(keys, kind='stable')
    orc = np.argsort(okeys, kind='stable')
    Tc = T + 1 if tv else 1
    for n in range(N):
        slot = min(n, count - 1)
        j = tw[slot]
        assert np.array_equal(A[n], rowsA[j, :Tc]) and np.array_equal(b[n], rowsb[j, :Tc])
        assert kind[n] == lst['kind'][j]
        if orc[slot] != j:                                        # only where the two keys are within rounding
            assert abs(okeys[orc[slot]] - okeys[j]) <= 1e-7, (n, okeys[orc[slot]], okeys[j])
    return keys


@pytest.mark.parametrize('count', [0, 1, 5, 6, 1000])
@pytest.mark.parametrize('tv', [False, True])
@pytest.mark.parametrize('body_name', ['rect', 'poly5', 'disc'])
def test_twin_matches_oracle(count, tv, body_name):
    rng = np.random.default_rng(count * 7 + tv * 3 + len(body_name))
    N, E = 5, 8
    T = 4 if count == 1000 else 8
    span = 30.0 if count == 1000 else 8.0
    body = _bodies(rng)[body_name]
    world = _world(rng, count, span, E)
    lst = ht.robot_list(world, None, None, 0)
    nom, ref = _poses(rng, T, span)
    keys = _check_against_oracle(lst, N, T, E, tv, nom, ref, body)
    if count:
        assert np.isfinite(keys).all()


@pytest.mark.parametrize('body_name', ['rect', 'disc'])
def test_twin_matches_oracle_four_rows(body_name):
    """E = 4: the <4, 4> caps; polygons of more than four vertices have no rows and a key of +inf."""
    rng = np.random.default_rng(41)
    body = _bodies(rng)[body_name]
    world = _world(rng, 40, 8.0, 6)
    lst = ht.robot_list(world, None, None, 0)
    nom, ref = _poses(rng, 6, 8.0)
    keys = _check_against_oracle(lst, 6, 6, 4, True, nom, ref, body)
    assert np.array_equal(np.isinf(keys), (lst['kind'] == _cabi.OBS_POLYGON) & (lst['nv'] > 4))


def test_twin_matches_oracle_with_map_mates_along_plans():
    rng = np.random.default_rng(5)
    T, E, N = 6, 8, 4
    body = robot_body(rectangle_robot())
    world = _world(rng, 12, 10.0, E)
    B = 6
    state = np.c_[rng.uniform(-8, 8, (B, 2)), rng.uniform(-np.pi, np.pi, B)].astype(np.float32)
    cur_vel = rng.uniform(-2, 2, (B, 2, T)).astype(np.float32)
    fleet = fp.fleet_plan_shapes(state, cur_vel, body, 'acker', DT, 3.0)
    rw = np.zeros(B, np.int32)
    rw[5] = -1                                                    # in no world: an empty list
    for b in range(B):
        lst = ht.robot_list(world, fleet, rw, b)
        assert len(lst['kind']) == (0 if b == 5 else 12 + 4)
        nom, ref = _poses(rng, T, 10.0, broken=b == 1)
        _check_against_oracle(lst, N, T, E, True, nom, ref, body)


def test_no_finite_pose_keeps_list_order():
    rng = np.random.default_rng(9)
    world = _world(rng, 12, 8.0, 8)
    lst = ht.robot_list(world, None, None, 0)
    nom = np.full((3, 7), np.nan, np.float32)
    A, b, kind, cnt, keys = ht.select(lst, 5, 6, 8, DT, False, nom, nom, robot_body(rectangle_robot()))
    assert np.all(np.isinf(keys))
    assert np.array_equal(kind, lst['kind'][:5])


def _bound_cases(rng):
    """Worlds for the bound: random shapes near and at 60 m, and shapes touching or overlapping the poses."""
    T = 8
    for span, off in ((8.0, 0.0), (8.0, 60.0), (2.0, 0.0)):
        world = _world(rng, 200, span, 8)
        world['xy'][world['kind'] == _cabi.OBS_POLYGON] += np.float32(off)
        world['xy'][world['kind'] == _cabi.OBS_CIRCLE, 0] += np.float32(off)
        nom, ref = _poses(rng, T, span)
        nom[:2] += np.float32(off)
        ref[:2] += np.float32(off)
        yield world, T, nom, ref


def test_lower_bounds_never_exceed_the_exact_key():
    rng = np.random.default_rng(17)
    seen_useful = 0
    for world, T, nom, ref in _bound_cases(rng):
        lst = ht.robot_list(world, None, None, 0)
        for body in _bodies(rng).values():
            for tv in (False, True):
                keys = ht.select(lst, 4, T, 8, DT, tv, nom, ref, body)[4]
                lb_disc, lb_pose = ht.bounds(lst, T, 8, DT, tv, nom, ref, body)
                assert np.all(lb_disc <= keys) and np.all(lb_pose <= keys)
                assert np.any(keys < 0) or np.min(keys) < 0.5            # touching or overlapping pairs occur
                seen_useful += int(np.sum(lb_pose > keys - 1.0))
    assert seen_useful > 1000                                      # the bound is tight enough to prune


def test_lower_bounds_with_map_mates_along_plans():
    rng = np.random.default_rng(23)
    T = 8
    body = robot_body(rectangle_robot())
    B = 12
    state = np.c_[rng.uniform(-4, 4, (B, 2)) + 60, rng.uniform(-np.pi, np.pi, B)].astype(np.float32)
    cur_vel = rng.uniform(-3, 3, (B, 2, T)).astype(np.float32)
    fleet = fp.fleet_plan_shapes(state, cur_vel, body, 'diff', DT, 1.0)
    world = _world(rng, 30, 6.0, 8)
    world['xy'][world['kind'] == _cabi.OBS_POLYGON] += np.float32(60)
    world['xy'][world['kind'] == _cabi.OBS_CIRCLE, 0] += np.float32(60)
    rw = np.zeros(B, np.int32)
    for b in range(B):
        lst = ht.robot_list(world, fleet, rw, b)
        nom, ref = _poses(rng, T, 6.0)
        nom[:2] += np.float32(60)
        ref[:2] += np.float32(60)
        keys = ht.select(lst, 4, T, 8, DT, True, nom, ref, body)[4]
        lb_disc, lb_pose = ht.bounds(lst, T, 8, DT, True, nom, ref, body)
        assert np.all(lb_disc <= keys) and np.all(lb_pose <= keys)
        assert np.any(keys < 0)                                    # overlapping mates are among them


def corridor_world(extra=()):
    """The reference's corridor: two 70 x 2 m walls 4 m either side of y = 20, and boxes beside it within 35 m."""
    box = lambda x0, y0, x1, y1: Obs(None, None, np.array([[x0, x1, x1, x0], [y0, y0, y1, y1]], float), 'Rpositive',
                                     np.zeros((2, 1)))
    walls = [box(-5, 14, 65, 16), box(-5, 24, 65, 26)]
    clutter = [box(30 + dx, y, 31 + dx, y + 1) for dx in (-12, -6, 0, 6, 12) for y in (6, 33)]
    return pack_worlds([walls + clutter + list(extra)])


def test_corridor_keeps_both_walls_and_the_reference_key_drops_them():
    T, N, E = 10, 6, 4
    world = corridor_world()
    lst = ht.robot_list(world, None, None, 0)
    t = np.arange(T + 1) * DT
    nom = np.vstack([30 + 3 * t, np.full(T + 1, 20.0), np.zeros(T + 1)]).astype(np.float32)
    ref = np.vstack([30 + 5 * t, np.full(T + 1, 20.0), np.zeros(T + 1)]).astype(np.float32)
    body = robot_body(rectangle_robot())
    keys = ht.select(lst, N, T, E, DT, False, nom, ref, body)[4]
    chosen = set(np.argsort(keys, kind='stable')[:N].tolist())
    assert {0, 1} <= chosen
    vertex_key = np.array([np.min(np.hypot(lst['xy'][j, :4, 0] - 30, lst['xy'][j, :4, 1] - 20))
                           for j in range(len(lst['kind']))])
    ref_chosen = set(np.argsort(vertex_key, kind='stable')[:N].tolist())
    assert not ({0, 1} & ref_chosen)
    # the world twin with the reference key makes the same choice
    A, b, kind, _ = world_twin.convert_world_obstacles(world, 0, N, T, E, DT, False, True, nom[:, 0])
    wallA, _, _, _ = world_twin.convert_world_obstacles(world, 0, 2, T, E, DT, False, False, nom[:, 0])
    assert not any(np.array_equal(A[n], wallA[k]) for n in range(N) for k in range(2))


def _cabi_call(lib, **kw):
    vp = ctypes.c_void_p
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.cast(buf, vp)
    args = dict(B=2, W=1, N=4, T=5, E=4, dt=0.1, tv=0, nom=p, ref=p, bkind=_cabi.OBS_POLYGON, bnv=4, bxy=p, brad=0.0,
                bxy_b=None, brad_b=None, start=p, rw=None, kind=p, nv=p, xy=p, rad=p, vel=p, fstart=None, frobot=None,
                fkind=None, fnv=None, fxy=None, frad=None, fvel=None, fplan=None, A=p, b=p, okind=p, ocount=p)
    args.update(kw)
    return lib.rda_convert_world_obstacles_horizon(*args.values(), None)


def test_usage_errors_are_return_codes():
    """Checked before any launch, so this runs without a GPU."""
    lib = _cabi.load()
    assert _cabi_call(lib, nom=None) == _cabi.E_ARG
    assert _cabi_call(lib, ref=None) == _cabi.E_ARG
    assert _cabi_call(lib, bxy=None) == _cabi.E_ARG
    assert _cabi_call(lib, A=None) == _cabi.E_ARG
    assert _cabi_call(lib, start=None) == _cabi.E_ARG
    assert _cabi_call(lib, B=0) == _cabi.E_ARG
    assert _cabi_call(lib, N=_cabi.MAX_WORLD_SLOTS + 1) == _cabi.E_UNSUPPORTED
    assert _cabi_call(lib, E=2) == _cabi.E_UNSUPPORTED
    assert _cabi_call(lib, E=9) == _cabi.E_UNSUPPORTED
    assert _cabi_call(lib, bnv=9) == _cabi.E_UNSUPPORTED
    assert _cabi_call(lib, bkind=_cabi.OBS_CIRCLE, brad=0.0) == _cabi.E_ARG
    p = ctypes.cast(ctypes.create_string_buffer(64), ctypes.c_void_p)
    assert _cabi_call(lib, fstart=p) == _cabi.E_ARG                # a fleet without its arrays
    assert _cabi_call(lib, fplan=p) == _cabi.E_ARG                 # plans without a fleet


def test_batched_mpc_refuses_shapes_and_unknown_orders():
    from rda_planner_b200.frontend import BatchedMPC
    with pytest.raises(ValueError, match='obstacle_order'):
        BatchedMPC(rectangle_robot(), np.zeros((3, 3)), 2, obstacle_order='nearest')
    # the shapes= refusal is checked before any device work, on a constructed object without a device
    mpc = BatchedMPC.__new__(BatchedMPC)
    mpc.obstacle_order = 'horizon'
    mpc.device, mpc.batch, mpc.T = None, 2, 5
    with pytest.raises(ValueError, match='pack_worlds'):
        mpc.control(np.zeros((2, 3)), shapes={'kind': None})


def test_non_finite_shapes_are_never_pruned():
    """A NaN or infinite vertex, centre or radius gives a bound of -inf, whatever the exact key is.  (A NaN velocity is
    not "moving" for obstacle_rows, so such a shape stands still in its rows and in its bound alike.)"""
    rng = np.random.default_rng(31)
    world = _world(rng, 40, 8.0, 8)
    bad = [(0, 'xy', (0, 0, 0), np.nan), (2, 'xy', (2, 1, 1), np.inf),
           (4, 'radius', (4,), np.nan), (5, 'xy', (5, 2, 0), np.nan)]
    for j, key, at, v in bad:
        world[key][at] = v
    lst = ht.robot_list(world, None, None, 0)
    nom, ref = _poses(rng, 6, 8.0, broken=False)
    for tv in (False, True):
        lb_disc, lb_pose = ht.bounds(lst, 6, 8, DT, tv, nom, ref, robot_body(rectangle_robot()))
        for j, key, _, _ in bad:
            assert lb_disc[j] == -np.inf and lb_pose[j] == -np.inf, (j, key, tv)
