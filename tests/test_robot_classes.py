"""Robot classes of a handle (rda_set_robot_classes / rda_set_robot_class_index, RDA_solver.set_robot_classes) without a
GPU: whole solves of the g++ build of the kernels' cores with each instance's class picked by the kernels' own helpers
(class_slot, su_params_class; tests/cpu_twin/robot_classes.cpp), a mixed batch of four bodies against the committed
float64 oracle traces, the host-side checks of the Python layer, and the usage errors of the C entry points."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest

import class_twin
from oracle import cpu_port
from rda_planner_b200 import _cabi
from rda_planner_b200.rda_solver import pack_obstacles, robot_class_table
from rda_planner_b200.scenarios import car, disc_robot, make_instance, rectangle_robot

HERE = os.path.dirname(os.path.abspath(__file__))
TRAJ_TOL, RESI_RTOL = 1e-3, 2e-3          # as tests/test_robot_bodies.py


def _bodies():
    spec = importlib.util.spec_from_file_location('make_bodies', os.path.join(HERE, 'golden', 'make_oracle_fixture_bodies.py'))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


BODIES = _bodies()
# the R = 4 bodies of oracle_bodies.npz: acker L = 3, diff, omni, acker L = 2.5 (reference point outside the body)
FOUR = ['rect_rear', 'rect_centred', 'omni_centred', 'offset_box']


def batch_inputs(B, T, N, seed=0, kind='polygon', moving=False):
    insts = [make_instance(seed + i, T=T, N=N, E=4, lateral=(0.3, 3.0), kind=kind, moving=moving) for i in range(B)]
    packed = [pack_obstacles(list(i['obstacles']), T, N, 4) for i in insts]
    return dict(nom_s=np.stack([i['nom_s'] for i in insts]), nom_u=np.stack([i['nom_u'] for i in insts]),
                ref_s=np.stack([i['ref'] for i in insts]), ref_speed=np.array([i['ref_speed'] for i in insts]),
                obs_A=np.stack([p[0] for p in packed]), obs_b=np.stack([p[1] for p in packed]),
                obs_kind=np.stack([p[2] for p in packed]), obs_count=np.array([p[3] for p in packed])), packed[0][4]


def same_bits(a, b, rows=None):
    for k in ('u', 's', 'iters', 'resi_pri', 'resi_dual'):
        x = a[k] if rows is None else a[k][rows]
        assert np.array_equal(x.view(np.int32), b[k].view(np.int32)), k


def polygon_classes():
    """Three classes of the handle's R = 4 and cone: bodies, dynamics, wheelbases and limits all differ."""
    return [BODIES.body('rect_centred'),
            car(*BODIES.body('omni_centred')[:4], [6, 0.7], [4, 0.3], 'omni'),
            car(*BODIES.body('offset_box')[:4], [8, 0.9], [6, 0.4], 'acker')]


def disc_classes():
    return [disc_robot(0.6, (0.2, 0.0), dynamics='diff'), disc_robot(1.2, (-0.3, 0.1), wheelbase=2.0, dynamics='acker',
                                                                     max_speed=(6, 0.7), max_acce=(4, 0.3)),
            disc_robot(0.9, dynamics='omni')]


def _one(inp, b):
    return {k: np.asarray(v)[b:b + 1] for k, v in inp.items()}


@pytest.mark.parametrize('kind', ['polygon', 'disc'])
def test_robots_of_the_handles_class_give_the_bits_of_no_class_table(kind):
    """A class equal to the handle's car_tuple (and indices outside the table) solves like no class table at all."""
    handle = rectangle_robot() if kind == 'polygon' else disc_robot(0.8)
    T, N, B = 10, 4, 6
    inp, tv = batch_inputs(B, T, N, seed=11, kind='polygon' if kind == 'polygon' else 'circle')
    none = class_twin.solve_batch(handle, T, N, 4, time_varying=tv, iter_num=5, threads=1, **inp)
    own = class_twin.solve_batch(handle, T, N, 4, time_varying=tv, iter_num=5, threads=1, classes=[handle],
                                 robot_class=np.zeros(B, np.int32), **inp)
    outside = class_twin.solve_batch(handle, T, N, 4, time_varying=tv, iter_num=5, threads=1, classes=[handle],
                                     robot_class=np.array([-1, 1, 7, -100, 2, 1 << 30]), **inp)
    same_bits(own, none)
    same_bits(outside, none)


@pytest.mark.parametrize('kind,lean2', [('polygon', '0'), ('polygon', '1'), ('disc', '0')])
def test_mixed_batch_equals_uniform_solves_of_each_class(monkeypatch, kind, lean2):
    """Instance b of a mixed batch has the bits of a solve with its class's car_tuple; an index outside the table is the
    handle's car_tuple."""
    monkeypatch.setenv('RDA_PORT_LEAN2', lean2)
    handle = rectangle_robot() if kind == 'polygon' else disc_robot(0.8)
    classes = polygon_classes() if kind == 'polygon' else disc_classes()
    T, N, B = 10, 4, 8
    inp, tv = batch_inputs(B, T, N, seed=21, kind='polygon' if kind == 'polygon' else 'circle')
    idx = np.array([0, 1, 2, 3, -1, 2, 1, 0], np.int32)
    mixed = class_twin.solve_batch(handle, T, N, 4, time_varying=tv, iter_num=6, threads=1, classes=classes,
                                   robot_class=idx, **inp)
    for b in range(B):
        c = classes[idx[b]] if 0 <= idx[b] < len(classes) else handle
        one = cpu_port.solve_batch(c, T, N, 4, time_varying=tv, iter_num=6, threads=1, **_one(inp, b))
        same_bits(mixed, one, rows=slice(b, b + 1))


def four_body_batch():
    """The instances of make_oracle_fixture_bodies.instance for FOUR in one batch, packed time-varying (omni_centred's
    obstacles move; static obstacles become T + 1 equal copies)."""
    T, N = BODIES.T, BODIES.N
    rows = []
    for name in FOUR:
        _, inst = BODIES.instance(name)
        A, b, kd, count, tv = pack_obstacles(list(inst['obstacles']), T, N, 4)
        if not tv:
            A, b = np.repeat(A, T + 1, axis=1), np.repeat(b, T + 1, axis=1)
        rows.append((inst, A, b, kd, count))
    inp = dict(nom_s=np.stack([r[0]['nom_s'] for r in rows]), nom_u=np.stack([r[0]['nom_u'] for r in rows]),
               ref_s=np.stack([r[0]['ref'] for r in rows]), ref_speed=np.array([r[0]['ref_speed'] for r in rows]),
               obs_A=np.stack([r[1] for r in rows]), obs_b=np.stack([r[2] for r in rows]),
               obs_kind=np.stack([r[3] for r in rows]), obs_count=np.array([r[4] for r in rows]))
    return [BODIES.body(n) for n in FOUR], inp


@pytest.mark.parametrize('lean2', ['0', '1'])
def test_four_body_mixed_batch_matches_committed_oracle_traces(monkeypatch, lean2):
    """Every ADMM iteration of the cold call in oracle_bodies.npz, for a batch whose instances are four classes with the
    rear-axle rectangle as the handle's body, tolerances of test_robot_bodies."""
    monkeypatch.setenv('RDA_PORT_LEAN2', lean2)
    z = np.load(os.path.join(HERE, 'golden', 'oracle_bodies.npz'))
    cars, inp = four_body_batch()
    idx = np.arange(4, dtype=np.int32)
    for it in range(1, BODIES.ITERS + 1):
        r = class_twin.solve_batch(cars[0], BODIES.T, BODIES.N, 4, time_varying=True, iter_num=it, threads=1,
                                   classes=cars, robot_class=idx, **inp)
        for b, name in enumerate(FOUR):
            assert r['cell_failures'][b, 0] == 0
            ds = np.abs(r['s'][b] - z[f'{name}_c0_s'][it - 1]).max()
            du = np.abs(r['u'][b] - z[f'{name}_c0_u'][it - 1]).max()
            assert ds < TRAJ_TOL and du < TRAJ_TOL, (name, it, ds, du)
            for k in ('resi_pri', 'resi_dual'):
                ref = z[f'{name}_c0_{k}'][it - 1]
                assert abs(float(r[k][b]) - ref) <= RESI_RTOL * (1 + ref), (name, it, k)


def test_host_checks_name_the_offending_class():
    rect = rectangle_robot()
    R = 4
    ok = polygon_classes()
    assert robot_class_table(ok, 'Rpositive', R)[2].dynamics == _cabi.DYNAMICS['acker']
    with pytest.raises(ValueError, match='robot class 1: cone_type'):
        robot_class_table([rect, disc_robot(1.0)], 'Rpositive', R)
    with pytest.raises(ValueError, match='robot class 1: 6 canonical body rows'):
        robot_class_table([rect, BODIES.body('hexagon')], 'Rpositive', R)
    with pytest.raises(ValueError, match='robot class 0: unknown dynamics'):
        robot_class_table([rect._replace(dynamics='tank')], 'Rpositive', R)
    with pytest.raises(ValueError, match='robot class 2: wheelbase'):
        robot_class_table([rect, rect, rect._replace(wheelbase=0.0)], 'Rpositive', R)
    with pytest.raises(ValueError, match='robot class 0: wheelbase'):
        robot_class_table([rect._replace(wheelbase=float('nan'), dynamics='diff')], 'Rpositive', R)
    with pytest.raises(ValueError, match='robot class 1: max_speed'):
        robot_class_table([rect, rect._replace(max_speed=[-1, 1])], 'Rpositive', R)
    with pytest.raises(ValueError, match='at most 16 robot classes'):
        robot_class_table([rect] * 17, 'Rpositive', R)
    # disc classes: any centre and radius, three rows
    assert len(robot_class_table(disc_classes(), 'norm2', 3)) == 3
    with pytest.raises(ValueError, match='robot class 0: cone_type'):
        robot_class_table([rect], 'norm2', 3)


def test_usage_errors_are_return_codes_not_exceptions():
    """Both entry points check their handle before any device work, so this runs without a GPU."""
    lib = _cabi.load()
    arr = robot_class_table([rectangle_robot()], 'Rpositive', 4)
    idx = (ctypes.c_int32 * 4)()
    assert lib.rda_set_robot_classes(None, 1, arr, None) == _cabi.E_ARG
    assert lib.rda_set_robot_classes(None, 0, None, None) == _cabi.E_ARG
    assert lib.rda_set_robot_class_index(None, idx, None) == _cabi.E_ARG
    assert lib.rda_set_robot_class_index(None, None, None) == _cabi.E_ARG
