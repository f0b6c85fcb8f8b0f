"""-m gpu: robot classes (RDA_solver.set_robot_classes, rda_set_robot_classes / rda_set_robot_class_index) on every routing
of the solve: a mixed batch against handles built with each row's class, the handle's own class against no table, the
g++ twin, the committed float64 traces of four bodies, the phase API, graph replay and the usage errors of the C ABI."""
import ctypes
import gc
import os

import numpy as np
import pytest
import torch

import class_twin
from rda_planner_b200 import _cabi
from rda_planner_b200.rda_solver import robot_class_table
from rda_planner_b200.scenarios import car, disc_robot, make_instance, rectangle_robot
from test_gpu_instance_params import _assert_same, _inputs, _pack, _solve, _solver
from test_robot_classes import BODIES, FOUR, disc_classes, four_body_batch, polygon_classes

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
TRAJ_TOL, RESI_RTOL = 1e-3, 2e-3          # as tests/test_gpu_robot_bodies.py


def hexagon_classes():
    """R = 6 (k_cells_fast<8, 8>): the hexagon of the body fixture and a copy scaled by 0.7 with its own kinematics."""
    hexa = BODIES.body('hexagon')
    G, h = np.asarray(hexa.G, float), np.asarray(hexa.h, float)
    return [hexa, car(G, 0.7 * h, 'Rpositive', 0.0, [6, 0.7], [4, 0.3], 'diff')]


ROUTINGS = {                                     # name: (env, B, T, N, handle, classes)
    'small': ({}, 192, 12, 6, rectangle_robot, polygon_classes),
    'streaming': ({'RDA_B200_SMALL': '0'}, 256, 12, 6, rectangle_robot, polygon_classes),
    'split_extra': ({'RDA_B200_SMALL': '0', 'RDA_B200_SPLIT_MIN': '2', 'RDA_B200_EXTRA_MIN': '1'}, 1024, 12, 6,
                    rectangle_robot, polygon_classes),
    'coherent': ({}, 16384, 30, 20, rectangle_robot, polygon_classes),
    'hexagon': ({'RDA_B200_SMALL': '0'}, 256, 12, 6, lambda: BODIES.body('hexagon'), hexagon_classes),
    'disc': ({'RDA_B200_SMALL': '0'}, 256, 12, 6, lambda: disc_robot(0.8), disc_classes),
}


def _index(B, K):
    # every class, the handle's own (K and -1: outside the table), on both sides of each sub-batch boundary
    return (torch.arange(B, device='cuda', dtype=torch.int32) * 7 + 3) % (K + 2) - 1


@pytest.mark.parametrize('routing', list(ROUTINGS))
def test_mixed_batch_equals_a_handle_per_class(routing):
    env, B, T, N, handle, classes = ROUTINGS[routing]
    handle, classes = handle(), classes()
    K = len(classes)
    kind = 'circle' if routing == 'disc' else 'polygon'
    inp, tv = _inputs(B, T, N, seed=1300, kind=kind)
    idx = _index(B, K)
    g = _solver(env, handle, T, N, B, 8)
    g.set_robot_classes(classes, idx)
    mixed = _solve(g, inp, tv)
    launches = g.launch_count()
    del g
    for k, c in enumerate(classes + [handle]):
        u = _solver(env, c, T, N, B, 8)
        uni = _solve(u, inp, tv)
        sel = torch.nonzero((idx == k) if k < K else ((idx < 0) | (idx >= K))).flatten()
        assert sel.numel() > 0
        _assert_same(mixed, uni, sel)
        del u
        gc.collect()
    print(f'\n{routing}: B = {B}, {K} classes, launches {launches}')


@pytest.mark.parametrize('routing', ['small', 'streaming', 'coherent', 'disc'])
def test_table_of_the_handles_own_class_equals_no_table(routing):
    env, B, T, N, handle, _ = ROUTINGS[routing]
    handle = handle()
    inp, tv = _inputs(B, T, N, seed=1500, kind='circle' if routing == 'disc' else 'polygon')
    g = _solver(env, handle, T, N, B, 8)
    a = _solve(g, inp, tv)
    g.cold_start()
    g.set_robot_classes([handle], torch.zeros(B, dtype=torch.int32, device='cuda'))
    b = _solve(g, inp, tv)
    _assert_same(a, b)
    g.cold_start()
    g.set_robot_class_index(torch.full((B,), 5, dtype=torch.int32, device='cuda'))     # outside the table
    _assert_same(a, _solve(g, inp, tv))
    g.cold_start()
    g.clear_robot_classes()
    _assert_same(a, _solve(g, inp, tv))
    del g
    gc.collect()


@pytest.mark.parametrize('kind', ['polygon', 'disc'])
def test_kernels_match_the_twin(kind):
    """The kernels against the g++ twin on the bench band (obstacles 1.8-6 m beside the path), with the tolerance of
    test_gpu_instance_params' twin comparison."""
    T, N, B, iters = 12, 6, 48, 6
    handle = rectangle_robot() if kind == 'polygon' else disc_robot(0.8)
    classes = polygon_classes() if kind == 'polygon' else disc_classes()
    insts = [make_instance(1700 + i, T=T, N=N, E=4, kind='polygon' if kind == 'polygon' else 'circle') for i in range(B)]
    host, tv = _pack(insts, T, N)
    inp = {k: torch.as_tensor(v, device='cuda') for k, v in host.items()}
    idx = _index(B, len(classes))
    g = _solver({}, handle, T, N, B, iters)
    g.set_robot_classes(classes, idx.cpu().numpy())
    o = _solve(g, inp, tv)
    r = class_twin.solve_batch(handle, T, N, 4, time_varying=tv, iter_num=iters, classes=classes,
                               robot_class=idx.cpu().numpy(), **host)
    for k in ('u', 's'):
        d = np.abs(o[k].double().cpu().numpy() - r[k]).max(axis=tuple(range(1, r[k].ndim)))
        print(f'\n{kind} {k}: largest gap to the twin {d.max():.1e} (instance {int(d.argmax())}, class {int(idx[d.argmax()])})')
        assert d.max() < 3 * TRAJ_TOL, (k, d.max())


@pytest.mark.parametrize('routing', ['small', 'stream'])
def test_four_body_batch_matches_committed_oracle_traces(monkeypatch, routing):
    """Cold call, warm call and a call after reset() (k_reset's mu'h with each class's h) of a batch of the four R = 4
    bodies, with the tolerances of test_gpu_robot_bodies; rect_centred's later calls are checked for status only there."""
    z = np.load(os.path.join(HERE, 'golden', 'oracle_bodies.npz'))
    cars, inp = four_body_batch()
    env = {} if routing == 'small' else {'RDA_B200_SMALL': '0'}
    g = _solver(env, cars[0], BODIES.T, BODIES.N, 4, BODIES.ITERS)
    g.set_robot_classes(cars, np.arange(4))
    dev = {k: torch.as_tensor(np.ascontiguousarray(v), device='cuda') for k, v in inp.items()}
    for call in range(3):
        if call == 2:
            g.reset()
        o = _solve(g, dev, True)
        for b, name in enumerate(FOUR):
            assert int(o['status'][b]) & 7 == 0
            if call > 0 and name == 'rect_centred':
                continue
            s, u = o['s'][b].double().cpu().numpy(), o['u'][b].double().cpu().numpy()
            ds = np.abs(s - z[f'{name}_c{call}_s'][-1]).max()
            du = np.abs(u - z[f'{name}_c{call}_u'][-1]).max()
            tol = TRAJ_TOL if call == 0 else 3 * TRAJ_TOL
            assert ds < tol and du < tol, (name, call, ds, du)
            for k in ('resi_pri', 'resi_dual'):
                ref = z[f'{name}_c{call}_{k}'][-1]
                assert abs(float(o[k][b]) - ref) <= (1 if call == 0 else 3) * RESI_RTOL * (1 + ref), (name, call, k)


def test_phase_api_equals_solve():
    env, B, T, N, handle, classes = ROUTINGS['streaming']
    handle, classes = handle(), classes()
    inp, tv = _inputs(B, T, N, seed=1900)
    idx = _index(B, len(classes))
    g = _solver(env, handle, T, N, B, 6)
    g.set_robot_classes(classes, idx)
    a = _solve(g, inp, tv)
    g.cold_start()
    g.begin(**inp, time_varying=tv)
    for _ in range(6):
        g.step_su()
        g.step_lammuz()
    _assert_same(a, {k: v.clone() for k, v in g.finish().items()})


def test_graph_replay_sees_a_class_index_changed_after_capture():
    env, B, T, N, handle, classes = ROUTINGS['streaming']
    handle, classes = handle(), classes()
    inp, tv = _inputs(B, T, N, seed=2100)
    first, second = _index(B, len(classes)), torch.flip(_index(B, len(classes)), [0]).contiguous()
    res = {}
    for graph in (False, True):
        g = _solver(env, handle, T, N, B, 6, graph=graph)
        g.set_robot_classes(classes, first)
        _solve(g, inp, tv)                       # captured here with graph=True
        g.cold_start()
        g.set_robot_class_index(second)
        res[graph] = _solve(g, inp, tv)
        del g
    _assert_same(res[True], res[False])


def test_c_abi_return_codes_on_a_handle():
    g = _solver({}, rectangle_robot(), 8, 4, 4, 2)
    lib, h = g.lib, g._h
    good = robot_class_table(polygon_classes(), 'Rpositive', 4)
    assert lib.rda_set_robot_classes(h, 17, good, None) == _cabi.E_ARG
    assert lib.rda_set_robot_classes(h, -1, good, None) == _cabi.E_ARG
    for field, value in (('dynamics', 3), ('dynamics', -1), ('wheelbase', float('inf'))):
        bad = robot_class_table(polygon_classes(), 'Rpositive', 4)
        setattr(bad[1], field, value)
        assert lib.rda_set_robot_classes(h, 3, bad, None) == _cabi.E_ARG, field
    bad = robot_class_table(polygon_classes(), 'Rpositive', 4)
    bad[2].wheelbase = 0.0                          # class 2 is acker
    assert lib.rda_set_robot_classes(h, 3, bad, None) == _cabi.E_ARG
    bad = robot_class_table(polygon_classes(), 'Rpositive', 4)
    for j in range(8):
        bad[0].G[j] = 0.0                           # not a polygon
    assert lib.rda_set_robot_classes(h, 3, bad, None) == _cabi.E_UNSUPPORTED
    disc = robot_class_table(disc_classes(), 'norm2', 3)
    assert lib.rda_set_robot_classes(h, 3, disc, None) == _cabi.E_UNSUPPORTED    # a disc in a polygon handle
    assert lib.rda_set_robot_classes(h, 3, good, None) == 0
    assert lib.rda_set_robot_classes(h, 0, None, None) == 0
    idx = torch.zeros(4, dtype=torch.int32, device='cuda')
    assert lib.rda_set_robot_class_index(h, ctypes.c_void_p(idx.data_ptr()), None) == 0
    assert lib.rda_set_robot_class_index(h, None, None) == 0
    torch.cuda.synchronize()
