"""-m gpu: per-instance limits, weights and tunables (RDA_solver.set_instance_parameters, rda_set_instance_params) on every
routing of the solve, against uniform solves, the g++ build of the same cores and the fleet front end."""
import gc
from collections import namedtuple

import numpy as np
import pytest
import torch

import instance_twin
from rda_planner_b200.frontend import BatchedMPC, pack_worlds, shapes_to_device
from rda_planner_b200.rda_solver import RDA_solver, pack_obstacles
from rda_planner_b200.scenarios import disc_robot, make_instance, rectangle_robot

pytestmark = pytest.mark.gpu
SWITCHES = ('RDA_B200_SMALL', 'RDA_B200_LEAN2', 'RDA_B200_EXTRA_MIN', 'RDA_B200_SPLIT_MIN', 'RDA_B200_SPLIT_PARTS')
KEYS = ('u', 's', 'status', 'iters')
RESI_ATOL = 4e-6            # residuals are summed by float atomics in no fixed order (DESIGN.md §8)
TRAJ_TOL = 1e-3             # as tests/test_gpu_parity.py
# parameter sets that differ in every column: (car limits, tunables)
SETS = [
    (dict(max_speed=(10, 1), max_acce=(10, 0.5)), dict()),
    (dict(max_speed=(6, 0.7), max_acce=(4, 0.3)), dict(ws=2, wu=0.5, slack_gain=5, max_sd=0.8, min_sd=0.2, ro1=100, ro2=2)),
    (dict(max_speed=(3, 0.5), max_acce=(2, 0.2)), dict(ws=0.5, wu=2, slack_gain=12, max_sd=1.5, min_sd=0.05, ro1=300,
                                                       ro2=0.5)),
]


def _pack(insts, T, N):
    packs = [pack_obstacles(list(i['obstacles']), T, N, 4) for i in insts]
    return dict(nom_s=np.stack([i['nom_s'] for i in insts]).astype(np.float32),
                nom_u=np.stack([i['nom_u'] for i in insts]).astype(np.float32),
                ref_s=np.stack([i['ref'] for i in insts]).astype(np.float32),
                ref_speed=np.array([i['ref_speed'] for i in insts], np.float32),
                obs_A=np.stack([p[0] for p in packs]), obs_b=np.stack([p[1] for p in packs]),
                obs_kind=np.stack([p[2] for p in packs]), obs_count=np.array([p[3] for p in packs], np.int32)), packs[0][4]


def _inputs(B, T, N, unique=64, seed=300, **kw):
    inp, tv = _pack([make_instance(seed + i, T=T, N=N, E=4, lateral=(0.3, 3.0), **kw) for i in range(min(B, unique))],
                    T, N)
    return {k: torch.as_tensor(v[np.arange(B) % len(v)], device='cuda') for k, v in inp.items()}, tv


def _solver(env, car, T, N, B, iters, **kw):
    with pytest.MonkeyPatch.context() as mp:
        for k in SWITCHES:
            mp.delenv(k, raising=False)
        for k, v in env.items():
            mp.setenv(k, v)
        return RDA_solver(T, car, max_edge_num=4, max_obs_num=N, iter_num=iters, iter_threshold=0.0, time_print=False,
                          batch=B, **kw)


def _solve(g, inp, tv, **kw):
    return {k: v.clone() for k, v in g.iterative_solve_batch(**inp, time_varying=tv, **kw).items()}


def _assert_same(a, b, idx=None):
    sel = (lambda x: x) if idx is None else (lambda x: x[idx])
    for k in KEYS:
        assert torch.equal(sel(a[k]), sel(b[k])), k
    for k in ('resi_pri', 'resi_dual'):
        x, y = sel(a[k]), sel(b[k])
        assert bool(((x - y).abs() <= RESI_ATOL * (1 + y.abs())).all()), k


ROUTINGS = {                                     # name: (env, B, T, N)
    'small': ({}, 192, 12, 6),
    'streaming': ({'RDA_B200_SMALL': '0'}, 256, 12, 6),
    'split_extra': ({'RDA_B200_SMALL': '0', 'RDA_B200_SPLIT_MIN': '2', 'RDA_B200_EXTRA_MIN': '1'}, 1024, 12, 6),
    'coherent': ({}, 16384, 30, 20),
}


@pytest.mark.parametrize('case', list(ROUTINGS) + ['disc', 'moving', 'su_fp32'])
def test_uniform_table_equals_no_table(case):
    env, B, T, N = ROUTINGS.get(case, ({'RDA_B200_SMALL': '0'}, 256, 12, 6))
    car = disc_robot(radius=1.1, dynamics='diff') if case == 'disc' else rectangle_robot()
    inp, tv = _inputs(B, T, N, kind='circle' if case == 'moving' else 'polygon', moving=case == 'moving')
    g = _solver(env, car, T, N, B, 8, su_fp64=case != 'su_fp32', ro2=1.3, slack_gain=6)
    a = _solve(g, inp, tv)
    g.cold_start()
    g.set_instance_parameters()                  # a table holding the handle's own values
    b = _solve(g, inp, tv)
    _assert_same(a, b)
    del g
    gc.collect()


@pytest.mark.parametrize('case', ['small', 'split_extra'])
def test_mixed_table_equals_uniform_solves(case):
    env, B, T, N = ROUTINGS[case]
    K = len(SETS)
    inp, tv = _inputs(B, T, N, seed=700)
    g = _solver(env, rectangle_robot(), T, N, B, 6)
    idx = torch.arange(B, device='cuda') % K
    ms = torch.tensor([c['max_speed'] for c, _ in SETS], dtype=torch.float64, device='cuda')[idx]
    ma = torch.tensor([c['max_acce'] for c, _ in SETS], dtype=torch.float64, device='cuda')[idx]
    tun = {k: [dict(dict(ws=1, wu=1, slack_gain=8, max_sd=1.0, min_sd=0.1, ro1=200, ro2=1), **t)[k] for _, t in SETS]
           for k in ('ws', 'wu', 'slack_gain', 'max_sd', 'min_sd', 'ro1', 'ro2')}
    g.set_instance_parameters(max_speed=ms, max_acce=ma, **{k: np.asarray(v)[idx.cpu().numpy()] for k, v in tun.items()})
    mixed = _solve(g, inp, tv)
    for k, (carc, t) in enumerate(SETS):
        u = _solver(env, rectangle_robot(**carc), T, N, B, 6, **t)
        uni = _solve(u, inp, tv)
        sel = torch.nonzero(idx == k).flatten()
        for key in KEYS:
            assert torch.equal(mixed[key][sel], uni[key][sel]), (k, key)
        del u
    gc.collect()


def test_gpu_matches_port_with_the_same_table_and_respects_each_row():
    T, N, B, iters = 12, 6, 48, 6
    inp, tv = _inputs(B, T, N, seed=900)
    g = _solver({}, rectangle_robot(), T, N, B, iters)
    plain = _solve(g, inp, tv)
    tight = (torch.arange(B, device='cuda') % 2) == 1
    g.cold_start()
    g.set_instance_parameters(robots=tight, max_speed=(2.5, 0.3), max_acce=(1.5, 0.15), ro2=2.0, slack_gain=4)
    out = _solve(g, inp, tv)
    p = g.instance_parameters()
    table = torch.cat([p['max_speed'], p['acce_bound']] + [p[k][:, None] for k in ('ws', 'wu', 'slack_gain', 'max_sd',
                                                                                    'min_sd', 'ro1', 'ro2')], 1)
    host = {k: v.cpu().numpy() for k, v in inp.items()}
    port = instance_twin.solve_batch(rectangle_robot(), T, N, 4, **host, time_varying=tv, iter_num=iters,
                                     inst=table.cpu().numpy())
    np.testing.assert_allclose(out['u'].cpu().numpy(), port['u'], atol=3 * TRAJ_TOL)
    np.testing.assert_allclose(out['s'].cpu().numpy(), port['s'], atol=3 * TRAJ_TOL)
    solved = tight & ((out['status'] & 2) == 0)                 # an su-QP that failed keeps the previous nominal
    assert int(solved.sum()) >= int(tight.sum()) - 2
    u = out['u'][solved]
    assert bool((u[:, 0].abs() <= 2.5 + 1e-5).all()) and bool((u[:, 1].abs() <= 0.3 + 1e-5).all())
    du = u[:, :, 1:] - u[:, :, :-1]
    assert bool((du[:, 0].abs() <= np.float32(0.15) + 1e-5).all()) and bool((du[:, 1].abs() <= np.float32(0.015) + 1e-5).all())
    assert not torch.equal(out['u'][tight], plain['u'][tight])
    assert torch.equal(out['u'][~tight], plain['u'][~tight])


def test_phase_api_graph_replay_reset_and_cold_start_see_the_table():
    T, N, B, iters = 10, 5, 96, 4
    inp, tv = _inputs(B, T, N, seed=1100)
    mask = (torch.arange(B, device='cuda') % 3) == 0
    ref = _solver({'RDA_B200_SMALL': '0'}, rectangle_robot(), T, N, B, iters)
    ref.set_instance_parameters(robots=mask, ro2=2.5, max_speed=(4.0, 0.6))
    want = _solve(ref, inp, tv)
    # phase API
    ph = _solver({'RDA_B200_SMALL': '0'}, rectangle_robot(), T, N, B, iters)
    ph.set_instance_parameters(robots=mask, ro2=0.7)
    ph.set_instance_parameters(robots=mask, ro2=2.5, max_speed=(4.0, 0.6))       # an update of the installed table
    ph.reset()
    ph.cold_start()                                                             # neither touches the table
    ph.begin(inp['nom_s'], inp['nom_u'], inp['ref_s'], inp['ref_speed'], inp['obs_A'], inp['obs_b'], inp['obs_kind'],
             inp['obs_count'], tv, 0.0)
    for _ in range(iters):
        ph.step_su()
        ph.step_lammuz()
    _assert_same({k: v.clone() for k, v in ph.finish().items()}, want)
    # graph replay: captured with the first table, replayed after an update
    gr = _solver({'RDA_B200_SMALL': '0'}, rectangle_robot(), T, N, B, iters, graph=True)
    gr.set_instance_parameters(robots=mask, ro2=0.7)
    first = _solve(gr, inp, tv)
    gr.cold_start()
    gr.set_instance_parameters(robots=mask, ro2=2.5, max_speed=(4.0, 0.6))
    second = _solve(gr, inp, tv)
    assert len(gr._graphs) == 1                                                 # replayed, not captured again
    _assert_same(second, want)
    assert not torch.equal(first['u'][mask], second['u'][mask])
    gr.cold_start()
    gr.clear_instance_parameters()
    plain = _solve(_solver({'RDA_B200_SMALL': '0'}, rectangle_robot(), T, N, B, iters), inp, tv)
    _assert_same(_solve(gr, inp, tv), plain)


Obs = namedtuple('Obs', 'center radius vertex cone_type velocity')
FAST, SLOW = dict(max_speed=(6, 1), max_acce=(6, 0.5)), dict(max_speed=(2, 0.4), max_acce=(1.5, 0.2))


def _world():
    rng = np.random.default_rng(21)
    return [Obs(np.array([[rng.uniform(2, 30)], [rng.choice([-1, 1]) * rng.uniform(2.5, 5)]]),
                float(rng.uniform(0.3, 0.8)), None, 'norm2', np.zeros((2, 1))) for _ in range(20)]


def _path():
    return [np.array([[0.5 * i], [0.0], [0.0]]) for i in range(120)]


def test_mixed_fleet_equals_one_fleet_per_class():
    """Two robot classes in one BatchedMPC (update_parameter with a mask) step exactly like two fleets of one class each;
    every robot keeps its own speed limit."""
    B, steps = 16, 6
    kw = dict(receding=10, sample_time=0.1, iter_num=3, max_edge_num=4, max_obs_num=4, iter_threshold=0.0)
    world = shapes_to_device(pack_worlds([_world()]), 'cuda')
    slow = (torch.arange(B, device='cuda') % 2) == 1
    rng = np.random.default_rng(5)
    st = torch.as_tensor(np.stack([[rng.uniform(0, 3), rng.uniform(-1, 1), rng.uniform(-0.2, 0.2)] for _ in range(B)]),
                         dtype=torch.float32, device='cuda')
    mixed = BatchedMPC(rectangle_robot(**FAST), _path(), B, **kw)
    mixed.update_parameter(robots=slow, **SLOW)
    fast_f = BatchedMPC(rectangle_robot(**FAST), _path(), B // 2, **kw)
    slow_f = BatchedMPC(rectangle_robot(**SLOW), _path(), B // 2, **kw)
    sm, sf, ss = st.clone(), st[~slow].clone(), st[slow].clone()
    for _ in range(steps):
        um, im = mixed.control(sm, 5.0, world=world)
        uf, _ = fast_f.control(sf, 5.0, world=world)
        us, _ = slow_f.control(ss, 5.0, world=world)
        assert torch.equal(um[~slow], uf) and torch.equal(um[slow], us)
        assert bool((im['u'][slow][:, 0].abs() <= 2 + 1e-5).all())
        mixed.advance(sm)
        fast_f.advance(sf)
        slow_f.advance(ss)
    assert torch.equal(sm[~slow], sf) and torch.equal(sm[slow], ss)
    assert float(im['u'][~slow][:, 0].abs().max()) > 2.5          # the fast class does use its higher limit


def test_update_parameter_with_tensors_needs_no_host_sync():
    B = 32
    bm = BatchedMPC(rectangle_robot(), _path(), B, receding=8, iter_num=2, max_edge_num=4, max_obs_num=4)
    world = shapes_to_device(pack_worlds([_world()]), 'cuda')
    state = torch.zeros((B, 3), dtype=torch.float32, device='cuda')
    mask = (torch.arange(B, device='cuda') % 3) == 0
    ro2 = torch.full((B,), 2.0, device='cuda')
    ms = torch.tensor([3.0, 0.5], device='cuda').expand(B, 2)
    bm.control(state, 3.0, world=world)
    bm.update_parameter(robots=mask, ro2=torch.full((B,), 1.5, device='cuda'))    # first use: creates the table
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        bm.update_parameter(robots=mask, ro2=ro2, max_speed=ms)
        u0, info = bm.control(state, 3.0, world=world)
        bm.advance(state)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    p = bm.rda.instance_parameters()
    assert bool((p['ro2'][mask] == 2.0).all()) and bool((p['ro2'][~mask] == 1.0).all())
    assert bool((info['u'][mask][:, 0].abs() <= 3.0 + 1e-5).all())
