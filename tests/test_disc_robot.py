"""Disc body (car_tuple.cone_type 'norm2', reference RDA_planner/rda_solver.py:1034-1039, :419): the two-cone cell
solver of csrc/cell_disc_robot.cuh against the numpy oracle in the ORIGINAL (lam, mu, z) variables (oracle/cell_generic.py,
SLSQP with both second-order cones), and the whole ADMM loop against OracleRDA."""
import importlib.util
import os

import numpy as np
import pytest

import shim
from oracle.cell_generic import solve_cell_generic, cell_objective
from oracle.cell_geo import solve_cell_geo_disc
from oracle.rda_oracle import OracleRDA
from oracle import cpu_port
from rda_planner_b200.scenarios import disc_robot, make_instance
from rda_planner_b200.rda_solver import pack_obstacles

HERE = os.path.dirname(os.path.abspath(__file__))
G_DISC = np.array([[1.0, 0.0], [0.0, 1.0], [0.0, 0.0]])


def _rect_rows(cx, cy, w, h, ang):
    c, s = np.cos(ang), np.sin(ang)
    V = np.array([[-w / 2, -h / 2], [w / 2, -h / 2], [w / 2, h / 2], [-w / 2, h / 2]]) @ np.array([[c, s], [-s, c]]) + [cx, cy]
    A, b = [], []
    for i in range(4):
        e = V[(i + 1) % 4] - V[i]
        n = np.array([e[1], -e[0]])
        A.append(n)
        b.append(n @ V[i])
    return np.array(A, np.float32).astype(float), np.array(b, np.float32).astype(float)


def _random_cell(rng, k):
    circ = k % 3 == 2
    h = np.array([*(rng.uniform(-0.5, 0.5, 2) if k % 2 else np.zeros(2)), -rng.uniform(0.3, 1.5)])
    if circ:
        ctr, rad = rng.uniform(-4, 4, 2), rng.uniform(0.3, 1.5)
        A = np.array([[1.0, 0], [0, 1], [0, 0], [0, 0]])
        b = np.array([ctr[0], ctr[1], -rad, 0.0]).astype(np.float32).astype(float)
    else:
        A, b = _rect_rows(rng.uniform(-4, 4), rng.uniform(-4, 4), rng.uniform(0.5, 3), rng.uniform(0.5, 3), rng.uniform(0, 3))
    p, phi = rng.uniform(-0.5, 0.5, 2), rng.uniform(-3, 3)
    dbar, zeta = rng.uniform(0.1, 1.0), rng.uniform(-0.5, 0.5) * (k % 4 != 0)
    xi = rng.uniform(-0.3, 0.3, 2) * (k % 5 in (1, 2))
    return circ, h, A, b, p, phi, dbar, zeta, xi


def test_disc_robot_cell_matches_generic_oracle():
    rng = np.random.default_rng(7)
    paths = {}
    for k in range(24):
        circ, h, A, b, p, phi, dbar, zeta, xi = _random_cell(rng, k)
        ref = solve_cell_generic(A, b, circ, G_DISC, h, p, phi, dbar, zeta, xi, 1.0, robot_cone='norm2')
        o_ref = cell_objective(A, b, G_DISC, h, p, phi, dbar, zeta, xi, 1.0, ref['lam'], ref['mu'], ref['z'])
        # cone membership of the oracle's own answer (guards the restatement): |mu[0:2]| <= -mu[2]
        assert np.hypot(ref['mu'][0], ref['mu'][1]) <= -ref['mu'][2] + 1e-7
        for prec, tol in (('d', 4e-5), ('f', 3e-4), ('barrier_d', 4e-5)):
            kk = shim.cell_disc_robot(h, int(circ), A, b, p, phi, dbar, zeta, xi, 1.0, prec=prec)
            assert kk['path'] != 5
            paths[kk['path']] = paths.get(kk['path'], 0) + 1
            assert np.hypot(kk['mu'][0], kk['mu'][1]) <= -kk['mu'][2] + 1e-6
            np.testing.assert_allclose(kk['lam'], ref['lam'], atol=tol)
            np.testing.assert_allclose(kk['mu'], ref['mu'], atol=tol)
            assert abs(kk['z'] - ref['z']) < tol
            if prec != 'f':
                # SLSQP is the less accurate of the two on active cells: the kernel's point must not be worse in the
                # reference objective (:399-406)
                o_k = cell_objective(A, b, G_DISC, h, p, phi, dbar, zeta, xi, 1.0, kk['lam'], kk['mu'], kk['z'])
                assert o_k <= o_ref + 1e-8
    # plain inactive cells, searched closed forms (edge / point contacts: 1, overlap cases: 4), and — with the closed forms
    # switched off ('barrier_d') — the two-cone programmes of both stages (2: max-margin stage, 3: active hinge)
    assert paths.get(0, 0) > 10 and paths.get(1, 0) > 10 and paths.get(4, 0) >= 2 and paths.get(3, 0) > 6 and paths.get(2, 0) > 3, paths


def test_disc_robot_oracle_shortcut_equals_generic():
    rng = np.random.default_rng(11)
    hit = 0
    for k in range(18):
        circ, h, A, b, p, phi, dbar, zeta, xi = _random_cell(rng, k)
        xi = np.zeros(2)
        st = {}
        r1 = solve_cell_geo_disc(A, b, circ, G_DISC, h, p, phi, dbar, zeta, xi, 1.0, stats=st)
        if 'geo_disc_inactive' not in st:
            continue
        hit += 1
        r2 = solve_cell_generic(A, b, circ, G_DISC, h, p, phi, dbar, zeta, xi, 1.0, robot_cone='norm2')
        np.testing.assert_allclose(r1['lam'], r2['lam'], atol=2e-5)
        np.testing.assert_allclose(r1['mu'], r2['mu'], atol=2e-5)
        assert abs(r1['z'] - r2['z']) < 2e-5
    assert hit >= 5


def _gen():
    spec = importlib.util.spec_from_file_location('make_dr', os.path.join(HERE, 'golden', 'make_oracle_fixture_disc_robot.py'))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _batch_inputs(inst, T, N):
    A, b, kd, count, tv = pack_obstacles(list(inst['obstacles']), T, N, 4)
    return dict(nom_s=inst['nom_s'][None], nom_u=inst['nom_u'][None], ref_s=inst['ref'][None], ref_speed=[inst['ref_speed']],
                obs_A=A[None], obs_b=b[None], obs_kind=kd[None], obs_count=[count]), tv


S_TOL, U_TOL, R_RTOL = 5e-4, 2e-3, 2e-3


def _check(name, it, z, s, u, rp, rd):
    k = it - 1
    assert np.abs(s - z[f'{name}_s'][k]).max() < S_TOL, (name, it, 's', np.abs(s - z[f'{name}_s'][k]).max())
    assert np.abs(u - z[f'{name}_u'][k]).max() < U_TOL, (name, it, 'u', np.abs(u - z[f'{name}_u'][k]).max())
    assert abs(rp - z[f'{name}_resi_pri'][k]) <= R_RTOL * (1 + z[f'{name}_resi_pri'][k]), (name, it, 'resi_pri')
    assert abs(rd - z[f'{name}_resi_dual'][k]) <= R_RTOL * (1 + z[f'{name}_resi_dual'][k]), (name, it, 'resi_dual')


def test_disc_robot_pipeline_matches_live_oracle():
    """Whole ADMM loop with a disc body, oracle run live (small case): compiled port of the kernels' cores (float32 state)
    vs OracleRDA (float64)."""
    m = _gen()
    car, inst, T, N, iters = m.instance('a')
    ref = [inst['ref'][:, t:t + 1] for t in range(T + 1)]
    o = OracleRDA(T, car, max_edge_num=4, max_obs_num=N, iter_num=iters, iter_threshold=0.0)
    uo, io = o.iterative_solve(inst['nom_s'], inst['nom_u'], ref, inst['ref_speed'], list(inst['obstacles']))
    inp, tv = _batch_inputs(inst, T, N)
    r = cpu_port.solve_batch(car, T, N, 4, time_varying=tv, iter_num=iters, **inp)
    assert r['cell_failures'][0, 0] == 0
    np.testing.assert_allclose(r['u'][0], uo, atol=1e-3)
    np.testing.assert_allclose(r['s'][0], np.hstack(io['opt_state_list']), atol=S_TOL)
    assert abs(r['resi_dual'][0] - io['resi_dual']) < R_RTOL * (1 + io['resi_dual'])
    assert abs(r['resi_pri'][0] - io['resi_pri']) < R_RTOL * (1 + io['resi_pri'])
    assert o.cell_stats.get('generic', 0) > 0          # the instance does exercise the two-cone programmes


@pytest.mark.parametrize('name', ['a', 'b', 'c', 'd', 'e'])
def test_disc_robot_port_matches_committed_oracle_traces(name):
    """Every ADMM iteration against tests/golden/oracle_disc_robot.npz (polygon / disc / moving-disc obstacles, centred
    and off-centre bodies, all three motion models)."""
    m = _gen()
    z = np.load(os.path.join(HERE, 'golden', 'oracle_disc_robot.npz'))
    car, inst, T, N, iters = m.instance(name)
    inp, tv = _batch_inputs(inst, T, N)
    for it in range(1, iters + 1):
        r = cpu_port.solve_batch(car, T, N, 4, time_varying=tv, iter_num=it, threads=1, **inp)
        assert r['cell_failures'][0, 0] == 0
        _check(name, it, z, r['s'][0], r['u'][0], float(r['resi_pri'][0]), float(r['resi_dual'][0]))


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['a', 'b', 'c', 'd', 'e'])
def test_gpu_disc_robot_matches_committed_oracle_traces(name):
    """The CUDA path (k_cells_dr / k_cells_dr_mid / k_cells_dr_slow_coop behind the C ABI) through the phase API, every
    iteration."""
    from rda_planner_b200.rda_solver import RDA_solver
    m = _gen()
    z = np.load(os.path.join(HERE, 'golden', 'oracle_disc_robot.npz'))
    car, inst, T, N, iters = m.instance(name)
    inp, tv = _batch_inputs(inst, T, N)
    g = RDA_solver(T, car, max_edge_num=4, max_obs_num=N, iter_num=iters, iter_threshold=0.0, time_print=False, batch=1)
    g.begin(inp['nom_s'], inp['nom_u'], inp['ref_s'], inp['ref_speed'], inp['obs_A'], inp['obs_b'], inp['obs_kind'], inp['obs_count'],
            tv, 0.0)
    for it in range(1, iters + 1):
        g.step_su()
        g.step_lammuz()
        o = g.finish()
        assert int((o['status'] & 6).sum()) == 0
        _check(name, it, z, o['s'][0].double().cpu().numpy(), o['u'][0].double().cpu().numpy(), float(o['resi_pri'][0]),
               float(o['resi_dual'][0]))
    # the reference-facing single-instance API (numpy in / out), last iterate
    ref = [inst['ref'][:, t:t + 1] for t in range(T + 1)]
    g2 = RDA_solver(T, car, max_edge_num=4, max_obs_num=N, iter_num=iters, iter_threshold=0.0, time_print=False)
    u, info = g2.iterative_solve(inst['nom_s'], inst['nom_u'], ref, inst['ref_speed'], list(inst['obstacles']))
    _check(name, iters, z, np.hstack(info['opt_state_list']), u, info['resi_pri'], info['resi_dual'])


@pytest.mark.gpu
def test_gpu_disc_robot_batch_equals_cpu_build_of_the_same_cores():
    """A batch of 96 instances (metric shape, disc body): every instance of the CUDA batch against the g++ build of the same
    cores, and the batch dimension itself (instance i of the batch == instance i alone)."""
    import torch
    from rda_planner_b200.rda_solver import RDA_solver
    T, N, B, iters = 30, 20, 96, 6
    car = disc_robot(radius=1.1, center=(0.2, 0.0), wheelbase=2.0, dynamics='diff')
    insts = [make_instance(900 + i, T=T, N=N, E=4, lateral=(0.3, 3.5), kind='polygon' if i % 2 else 'circle', dynamics='diff')
             for i in range(B)]
    packs = [pack_obstacles(list(x['obstacles']), T, N, 4) for x in insts]
    f = lambda k: np.stack([x[k] for x in insts]).astype(np.float32)
    inp = dict(nom_s=f('nom_s'), nom_u=f('nom_u'), ref_s=f('ref'), ref_speed=np.array([x['ref_speed'] for x in insts], np.float32),
               obs_A=np.stack([p[0] for p in packs]), obs_b=np.stack([p[1] for p in packs]), obs_kind=np.stack([p[2] for p in packs]),
               obs_count=np.array([p[3] for p in packs], np.int32))
    g = RDA_solver(T, car, max_edge_num=4, max_obs_num=N, iter_num=iters, iter_threshold=0.0, time_print=False, batch=B)
    o = g.iterative_solve_batch(**{k: torch.as_tensor(v, device='cuda') for k, v in inp.items()})
    assert int((o['status'] & 6).sum()) == 0
    r = cpu_port.solve_batch(car, T, N, 4, iter_num=iters, **inp)
    ds = np.abs(o['s'].cpu().numpy() - r['s']).reshape(B, -1).max(axis=1)
    assert np.median(ds) < 2e-4 and np.quantile(ds, 0.9) < 2e-3, (np.median(ds), ds.max())
    g1 = RDA_solver(T, car, max_edge_num=4, max_obs_num=N, iter_num=iters, iter_threshold=0.0, time_print=False, batch=1)
    for i in (0, 37, 95):
        o1 = g1.iterative_solve_batch(**{k: torch.as_tensor(v[i:i + 1], device='cuda') for k, v in inp.items()})
        assert float((o1['s'][0] - o['s'][i]).abs().max()) < 1e-5
        g1.cold_start()
