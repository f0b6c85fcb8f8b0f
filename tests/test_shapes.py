"""Whole solves at the horizon lengths T and obstacle counts N where the kernels change shape — T = 1 and 2, N*T below one
warp, T = 31..33, 64, 65 and 100, N = 33 and 64 (more than 32 hinges per stage), the disc body at T = 1, 33 and N*T = 28 —
on the g++ build of the kernels' cores, against every ADMM iteration of the float64 oracle traces of
tests/golden/make_oracle_fixture_shapes.py.  The polygon-body cases run twice: with the streaming cell passes and with the
port's emulation of the coherent pipeline (RDA_PORT_LEAN2=1)."""
import importlib.util
import os

import numpy as np
import pytest

from oracle import cpu_port
from rda_planner_b200.rda_solver import pack_obstacles
from test_robot_bodies import TRAJ_TOL, RESI_RTOL

HERE = os.path.dirname(os.path.abspath(__file__))
# t65 (T = 65, N = 2, seed 7067) is compared after 3 ADMM iterations instead of 4: its su-QP is degenerate in the steering
# of stages 14..23 (DESIGN.md §0 item 5), so the last iteration's steering is decided by each solver's stopping point rather
# than by the problem.  The CPU port's gap to the oracle there, controls u[1] at stages 16, 23, 14, 14 after iterations 1..4:
# 4.4e-6, 1.9e-5, 1.2e-4, 1.1e-3 (x4 to x9 per iteration; states 2e-6 .. 8.3e-5, resi_pri / resi_dual within 2e-6 relative
# at every iteration, so the cells agree).  The oracle is the less determined side: solving its own su-QP to su_tol = 1e-11
# instead of 1e-12 moves its steering by 3.4e-4 already at iteration 1 (stage 17) and by 1.1e-3 at iteration 3 (stage 14),
# 75 times the port's gap at iteration 1.  The gap is a flat direction of the su-QP amplified by the ADMM map, not a bug of
# the cores, and up to iteration 3 TRAJ_TOL still bounds it with a margin of eight.  t100 (T = 100, N = 4 discs, seed 9701)
# has the same flat steering at stage 17: the port is 5.5e-6 off after iteration 1 and 2.7e-3 after iteration 2, and the
# oracle's own su_tol = 1e-11 solve is 1.6e-4 and 2.3e-3 off its 1e-12 one there, so it is compared after one iteration.
COMPARE_AT = {'t65': 3, 't100': 1}


def _gen():
    spec = importlib.util.spec_from_file_location('make_shapes', os.path.join(HERE, 'golden', 'make_oracle_fixture_shapes.py'))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


SHAPES = _gen()


def traces():
    return np.load(os.path.join(HERE, 'golden', 'oracle_shapes.npz'))


def batch(name, seeds=None):
    """(car, inputs of solve_batch / iterative_solve_batch, time_varying) of the case's instances, one per seed."""
    T, N = SHAPES.CASES[name][:2]
    seeds = SHAPES.CASES[name][4] if seeds is None else seeds
    insts = [SHAPES.instance(name, s) for s in seeds]
    packs = [pack_obstacles(list(x['obstacles']), T, N, SHAPES.E) for x in insts]
    st = lambda k: np.stack([x[k] for x in insts])
    inp = dict(nom_s=st('nom_s'), nom_u=st('nom_u'), ref_s=st('ref'), ref_speed=np.array([x['ref_speed'] for x in insts]),
               obs_A=np.stack([p[0] for p in packs]), obs_b=np.stack([p[1] for p in packs]),
               obs_kind=np.stack([p[2] for p in packs]), obs_count=np.array([p[3] for p in packs], np.int32))
    return SHAPES.car(name), inp, packs[0][4]


def coherent(name):
    """The coherent pipeline runs for the polygon body at E = 4 with static obstacles; without a polygon among them it has
    no cell to resolve."""
    _, _, obs, body, _ = SHAPES.CASES[name]
    return body == 'rect' and obs in ('polygon', 'mixed')


PORT_CASES = [(n, '0') for n in SHAPES.CASES] + [(n, '1') for n in SHAPES.CASES if coherent(n)]


@pytest.mark.parametrize('name,lean2', PORT_CASES)
def test_port_matches_committed_shape_traces(monkeypatch, name, lean2):
    """Every ADMM iteration of every instance of the case against the CPU port (which always starts cold), with the
    tolerances of test_gpu_parity.py, and no cell the port's cores gave up on; t65 up to iteration 3 (COMPARE_AT)."""
    monkeypatch.setenv('RDA_PORT_LEAN2', lean2)
    z = traces()
    T, N = SHAPES.CASES[name][:2]
    car, inp, tv = batch(name)
    B = len(inp['nom_s'])
    worst = [0.0, 0.0]
    for it in range(1, COMPARE_AT.get(name, SHAPES.ITERS) + 1):
        r = cpu_port.solve_batch(car, T, N, SHAPES.E, time_varying=tv, iter_num=it, threads=1, **inp)
        assert (r['cell_failures'][:, 0] == 0).all(), (name, it)
        for i in range(B):
            ds = np.abs(r['s'][i] - z[f'{name}_s'][i, it - 1]).max()
            du = np.abs(r['u'][i] - z[f'{name}_u'][i, it - 1]).max()
            worst = [max(worst[0], ds), max(worst[1], du)]
            assert ds < TRAJ_TOL and du < TRAJ_TOL, (name, i, it, ds, du)
            for k in ('resi_pri', 'resi_dual'):
                ref = z[f'{name}_{k}'][i, it - 1]
                assert abs(float(r[k][i]) - ref) <= RESI_RTOL * (1 + ref), (name, i, it, k, float(r[k][i]), ref)
    print(f'\n{name} (T = {T}, N = {N}, {B} instances, lean2 {lean2}): largest gap to the oracle, states {worst[0]:.1e}, '
          f'controls {worst[1]:.1e}')
