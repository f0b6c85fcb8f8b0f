"""Per-instance limits, weights and tunables (rda_set_instance_params, RDA_solver.set_instance_parameters) without a GPU:
whole solves of the g++ build of the kernels' cores with each instance's row selected by the kernels' own helpers
(su_params_row, inst_ro2; tests/cpu_twin/instance_params.cpp), the table builder of the Python layer on CPU tensors, and
the usage errors of the C entry point."""
import ctypes

import numpy as np
import pytest
import torch

import instance_twin
from oracle import cpu_port
from oracle.rda_oracle import OracleRDA
from rda_planner_b200 import _cabi
from rda_planner_b200.rda_solver import INSTANCE_COLUMNS, pack_obstacles, update_instance_table
from rda_planner_b200.scenarios import disc_robot, make_instance, rectangle_robot

TRAJ_TOL, RESI_RTOL = 1e-3, 2e-3          # as tests/test_gpu_parity.py (<= 6 ADMM iterations)
DT = 0.1
TUN_DEFAULTS = dict(slack_gain=8, max_sd=1.0, min_sd=0.1, ro1=200, ro2=1, ws=1, wu=1)


def row_of(car, dt=DT, **kw):
    """The table row of a handle constructed with car and kw, rounded to float32 as rda_config / rda_tunables hold it."""
    p = dict(TUN_DEFAULTS, **kw)
    ms, ma = np.asarray(car.max_speed, float), np.asarray(car.max_acce, float)
    return np.float32([ms[0], ms[1], ma[0] * dt, ma[1] * dt, p['ws'], p['wu'], p['slack_gain'], p['max_sd'],
                       p['min_sd'], p['ro1'], p['ro2']])


def batch_inputs(B, T, N, seed=0, kind='polygon', dyn='acker', moving=False):
    insts = [make_instance(seed + i, T=T, N=N, E=4, lateral=(0.3, 3.0), kind=kind, dynamics=dyn, moving=moving)
             for i in range(B)]
    packed = [pack_obstacles(list(i['obstacles']), T, N, 4) for i in insts]
    tv = packed[0][4]
    return dict(nom_s=np.stack([i['nom_s'] for i in insts]), nom_u=np.stack([i['nom_u'] for i in insts]),
                ref_s=np.stack([i['ref'] for i in insts]), ref_speed=np.array([i['ref_speed'] for i in insts]),
                obs_A=np.stack([p[0] for p in packed]), obs_b=np.stack([p[1] for p in packed]),
                obs_kind=np.stack([p[2] for p in packed]), obs_count=np.array([p[3] for p in packed])), tv, insts


def same_bits(a, b):
    for k in ('u', 's', 'iters', 'resi_pri', 'resi_dual'):
        assert np.array_equal(a[k].view(np.int32), b[k].view(np.int32)), k


# four parameter sets that differ in every column (car limits and tunables)
SETS = [
    (dict(max_speed=(10, 1), max_acce=(10, 0.5)), dict()),
    (dict(max_speed=(6, 0.7), max_acce=(4, 0.3)), dict(ws=2, wu=0.5, slack_gain=5, max_sd=0.8, min_sd=0.2, ro1=100, ro2=2)),
    (dict(max_speed=(3, 0.5), max_acce=(2, 0.2)), dict(ws=0.5, wu=2, slack_gain=12, max_sd=1.5, min_sd=0.05, ro1=300,
                                                       ro2=0.5)),
    (dict(max_speed=(8, 0.9), max_acce=(6, 0.4)), dict(ws=1.5, wu=1.2, slack_gain=3, max_sd=0.6, min_sd=0.15, ro1=50,
                                                       ro2=1.5)),
]


@pytest.mark.parametrize('body,dyn,accelerated,moving', [
    ('polygon', 'acker', True, False), ('polygon', 'diff', True, False), ('polygon', 'omni', False, False),
    ('polygon', 'acker', False, True), ('disc', 'diff', True, False), ('disc', 'omni', False, True),
])
def test_uniform_table_equals_no_table(body, dyn, accelerated, moving):
    """A table holding the handle's own values gives the same bits as no table (u, s, residuals, iterations)."""
    T, N, B = 8, 3, 5
    car = rectangle_robot(dynamics=dyn) if body == 'polygon' else disc_robot(radius=1.1, dynamics=dyn)
    inp, tv, _ = batch_inputs(B, T, N, seed=40, kind='circle' if moving else 'polygon', dyn=dyn, moving=moving)
    kw = dict(slack_gain=6, ro2=1.3)
    a = cpu_port.solve_batch(car, T, N, 4, time_varying=tv, iter_num=5, accelerated=accelerated, threads=1, **inp, **kw)
    table = np.tile(row_of(car, **kw), (B, 1))
    b = instance_twin.solve_batch(car, T, N, 4, time_varying=tv, iter_num=5, accelerated=accelerated, threads=1,
                                  inst=table, **inp, **kw)
    same_bits(a, b)
    assert np.array_equal(a['cell_failures'], b['cell_failures'])


@pytest.mark.parametrize('body', ['polygon', 'disc'])
def test_mixed_table_equals_uniform_solves(body):
    """K parameter sets dealt round-robin over a batch: instance b of the mixed solve equals instance b of the uniform
    solve of the whole batch with set b % K, bit for bit."""
    T, N, B, K = 8, 3, 8, len(SETS)
    mk = (lambda **c: rectangle_robot(**c)) if body == 'polygon' else (lambda **c: disc_robot(radius=1.1, **c))
    inp, tv, _ = batch_inputs(B, T, N, seed=60)
    table = np.stack([row_of(mk(**SETS[b % K][0]), **SETS[b % K][1]) for b in range(B)])
    assert all(len(set(table[:K, c])) == K for c in range(_cabi.INST_PARAMS))      # every column differs
    mixed = instance_twin.solve_batch(mk(), T, N, 4, time_varying=tv, iter_num=6, threads=1, inst=table, **inp)
    for k in range(K):
        uni = cpu_port.solve_batch(mk(**SETS[k][0]), T, N, 4, time_varying=tv, iter_num=6, threads=1, **inp,
                                   **SETS[k][1])
        for b in range(k, B, K):
            for key in ('u', 's', 'iters', 'resi_pri', 'resi_dual'):
                assert np.array_equal(mixed[key][b], uni[key][b]), (k, b, key)
    assert not np.array_equal(mixed['u'][1], cpu_port.solve_batch(mk(), T, N, 4, time_varying=tv, iter_num=6, threads=1,
                                                                  **inp)['u'][1])


@pytest.mark.parametrize('k', [1, 2, 3])
def test_instances_with_own_values_match_oracle(k):
    """Small instances whose row holds non-default limits and tunables against OracleRDA constructed with them."""
    T, N, iters = 8, 3, 5
    carc, tun = SETS[k]
    car = rectangle_robot(**carc)
    inp, tv, insts = batch_inputs(3, T, N, seed=80 + 7 * k)
    table = np.stack([row_of(rectangle_robot(), **{})] + [row_of(car, **tun)] * 2)
    r = instance_twin.solve_batch(rectangle_robot(), T, N, 4, time_varying=tv, iter_num=iters, threads=1, inst=table,
                                  **inp)
    for b in (1, 2):
        inst = insts[b]
        ref = [inst['ref'][:, t:t + 1] for t in range(T + 1)]
        o = OracleRDA(T, car, max_edge_num=4, max_obs_num=N, iter_num=iters, iter_threshold=0.0, **tun)
        uo, io = o.iterative_solve(inst['nom_s'], inst['nom_u'], ref, inst['ref_speed'], list(inst['obstacles']))
        np.testing.assert_allclose(r['u'][b], uo, atol=TRAJ_TOL)
        np.testing.assert_allclose(r['s'][b], np.hstack(io['opt_state_list']), atol=TRAJ_TOL)
        assert abs(r['resi_dual'][b] - io['resi_dual']) <= RESI_RTOL * (1 + io['resi_dual'])
        assert abs(r['resi_pri'][b] - io['resi_pri']) <= RESI_RTOL * (1 + io['resi_pri'])
        assert np.all(np.abs(r['u'][b]) <= np.asarray(car.max_speed, np.float32)[:, None] + 1e-5)


# ---- the table builder of the Python layer (CPU tensors) ----------------------------------------------------------
def base_table(B=4):
    return torch.as_tensor(np.tile(row_of(rectangle_robot()), (B, 1)))


def test_table_broadcasting_and_mask():
    t0 = base_table()
    t = update_instance_table(t0, DT, ro2=2.5, max_speed=(5, 0.5), max_acce=[[1, 0.1], [2, 0.2], [3, 0.3], [4, 0.4]],
                              ws=np.array([1.0, 2.0, 3.0, 4.0]))
    assert torch.equal(t0, base_table())                       # input untouched
    assert torch.all(t[:, _cabi.IP_RO2] == 2.5)
    assert torch.all(t[:, _cabi.IP_MAX_SPEED0] == 5) and torch.all(t[:, _cabi.IP_MAX_SPEED1] == 0.5)
    assert t[:, _cabi.IP_ACCE_BOUND0].tolist() == [float(np.float32(a * DT)) for a in (1.0, 2.0, 3.0, 4.0)]
    assert t[:, _cabi.IP_ACCE_BOUND1].tolist() == [float(np.float32(a * DT)) for a in (0.1, 0.2, 0.3, 0.4)]
    assert t[:, _cabi.IP_WS].tolist() == [1, 2, 3, 4]
    assert torch.equal(t[:, _cabi.IP_SLACK_GAIN], t0[:, _cabi.IP_SLACK_GAIN])
    mask = np.array([True, False, True, False])
    m = update_instance_table(t, DT, robots=mask, ro1=torch.tensor([7.0, 8.0, 9.0, 10.0]), min_sd=0.05)
    assert m[:, _cabi.IP_RO1].tolist() == [7, 200, 9, 200]
    assert m[:, _cabi.IP_MIN_SD].tolist() == [float(np.float32(0.05)), float(np.float32(0.1))] * 2
    assert torch.equal(m[:, _cabi.IP_RO2], t[:, _cabi.IP_RO2])
    # a tensor max_acce is rounded like a host one
    tt = update_instance_table(t0, DT, max_acce=torch.tensor([0.7, 0.3], dtype=torch.float64))
    th = update_instance_table(t0, DT, max_acce=(0.7, 0.3))
    assert torch.equal(tt, th)


@pytest.mark.parametrize('kw,msg', [
    (dict(ro2=0.0), '> 0'), (dict(ro1=-1), '> 0'), (dict(max_speed=(1, 0)), '> 0'), (dict(max_acce=(np.inf, 1)), 'finite'),
    (dict(slack_gain=-0.1), '>= 0'), (dict(ws=np.nan), 'finite'), (dict(wu=-1), '>= 0'),
    (dict(min_sd=0.9, max_sd=0.5), 'min_sd'), (dict(ro2=[1, 2]), 'shape'), (dict(max_speed=3.0), 'shape'),
    (dict(ro2=torch.ones(3)), 'shape'), (dict(ro2=torch.ones(4, dtype=torch.int32)), 'floating'),
])
def test_table_validation(kw, msg):
    with pytest.raises(ValueError, match=msg):
        update_instance_table(base_table(), DT, **kw)


def test_table_rejects_unknown_keys_and_bad_masks():
    with pytest.raises(TypeError):
        update_instance_table(base_table(), DT, z_theta=0.3)
    with pytest.raises(ValueError):
        update_instance_table(base_table(), DT, robots=[1, 0, 1, 0], ro2=2)
    with pytest.raises(ValueError):
        update_instance_table(base_table(), DT, robots=[True, False], ro2=2)
    assert sorted(INSTANCE_COLUMNS) == sorted(['max_speed', 'max_acce', 'ws', 'wu', 'slack_gain', 'max_sd', 'min_sd',
                                               'ro1', 'ro2'])


def test_assign_adjust_parameter_merges_only_named_columns():
    """With a table installed, assign_adjust_parameter writes the columns it names for every instance (what the
    reference's update_parameter does on each robot's MPC) and leaves the other per-instance values alone."""
    t = update_instance_table(base_table(), DT, robots=[True, False, True, False], max_speed=(4, 0.4), ro1=[1, 2, 3, 4],
                              ro2=3.0)
    merged = update_instance_table(t, DT, validate=False, ro2=0.5, slack_gain=9)
    assert torch.all(merged[:, _cabi.IP_RO2] == 0.5) and torch.all(merged[:, _cabi.IP_SLACK_GAIN] == 9)
    for c in range(_cabi.INST_PARAMS):
        if c not in (_cabi.IP_RO2, _cabi.IP_SLACK_GAIN):
            assert torch.equal(merged[:, c], t[:, c]), c


def test_set_instance_params_usage_errors():
    """A NULL handle is RDA_E_ARG (-1), with or without a table; nothing reaches the device."""
    lib = _cabi.load()
    assert lib.rda_set_instance_params(None, None, None) == -1
    assert lib.rda_set_instance_params(None, ctypes.c_void_p(16), None) == -1
