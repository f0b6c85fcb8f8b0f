"""-m gpu: the code paths that only large batches select, at the sizes that select them.

The library picks kernels by batch size (DESIGN.md §5): the single-launch k_admm_small up to 2 x SMs instances, two
sub-batches on two streams from 2 048, k_cells_extra (and the cooperative pass reading its list) from 3 000 instances per
sub-batch, the coherent first pass (k_cells_coh) from 8 192, and grid-stride loops that wrap once a sub-batch has more
than 16 x SMs x 128 cells.  The headline figure of bench.py (B = 16 384) runs all of them.

Instances never interact, so a batch made of copies of a few unique instances must give every copy the bits of the same
instances solved in a small batch that is forced through the same passes (RDA_B200_SMALL / _LEAN2 / _EXTRA_MIN /
_SPLIT_MIN); only the residuals, summed by float atomics in no fixed order, may differ in the last bits.  On top of that
the headline path is compared end to end with the float64 oracle trace tests/golden/oracle_metric50.npz and with the g++
build of the same cores (oracle/cpu_port, RDA_PORT_LEAN2=1 emulates the coherent pipeline)."""
import gc
import json
import os

import numpy as np
import pytest
import torch

from rda_planner_b200.scenarios import config_instance, disc_robot, make_instance, rectangle_robot

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
T, N, E = 30, 20, 4                  # the metric shape of bench.py
UNIQUE, B_HEAD = 2048, 16384         # bench.py's first 2 048 instances (seeds 9000..), tiled 8x to the headline batch
SWITCHES = ('RDA_B200_SMALL', 'RDA_B200_LEAN2', 'RDA_B200_EXTRA_MIN', 'RDA_B200_SPLIT_MIN', 'RDA_B200_SPLIT_PARTS')
# the small batch runs the passes the large one selects by size: streaming kernels, coherent pass, k_cells_extra
SAME_PASSES = {'RDA_B200_SMALL': '0', 'RDA_B200_LEAN2': '1', 'RDA_B200_EXTRA_MIN': '1'}
KEYS = ('u', 's', 'status', 'iters')
RESIDUALS = ('resi_pri', 'resi_dual')


def _state_ids():
    from rda_planner_b200 import _cabi
    return {'LAM': _cabi.BUF_LAM, 'MU': _cabi.BUF_MU, 'Z': _cabi.BUF_Z, 'XI': _cabi.BUF_XI, 'ZETA': _cabi.BUF_ZETA,
            'DIS': _cabi.BUF_DIS, 'COEF': _cabi.BUF_COEF, 'PREF': _cabi.BUF_PREF, 'CUR_S': _cabi.BUF_CUR_S,
            'CUR_U': _cabi.BUF_CUR_U}


def _pack(insts, T, N, E):
    from rda_planner_b200.rda_solver import pack_obstacles
    packs = [pack_obstacles(list(i['obstacles']), T, N, E) for i in insts]
    return dict(nom_s=np.stack([i['nom_s'] for i in insts]).astype(np.float32),
                nom_u=np.stack([i['nom_u'] for i in insts]).astype(np.float32),
                ref_s=np.stack([i['ref'] for i in insts]).astype(np.float32),
                ref_speed=np.array([i['ref_speed'] for i in insts], np.float32),
                obs_A=np.stack([p[0] for p in packs]), obs_b=np.stack([p[1] for p in packs]),
                obs_kind=np.stack([p[2] for p in packs]), obs_count=np.array([p[3] for p in packs], np.int32))


def _tile(inp, B):
    """Instance p of the batch is unique instance p % U."""
    U = len(inp['ref_speed'])
    return {k: v[np.arange(B) % U] for k, v in inp.items()}


def _dev(inp):
    return {k: torch.as_tensor(v, device='cuda') for k, v in inp.items()}


@pytest.fixture(scope='module')
def metric():
    """bench.py's metric instances 0..2047 (bench band, seeds 9000..), generated once per module."""
    return _pack([make_instance(9000 + i, T=T, N=N, E=E) for i in range(UNIQUE)], T, N, E)


def _run(env, car, shape, inp, iters, thr=0.0, calls=2, tv=False, phase=False, **kw):
    """Construct a solver with the environment switches `env` (read by rda_create), run `calls` solves of `iters`
    iterations (cold, then warm-started) or, with phase=True, one solve through the phase API.  Returns the outputs of
    every call, the persistent state and statistics after the last one, and the launch count; the handle is released."""
    from rda_planner_b200 import _cabi
    from rda_planner_b200.rda_solver import RDA_solver
    Ts, Ns, Es = shape
    B = len(inp['ref_speed'])
    with pytest.MonkeyPatch.context() as mp:
        for k in SWITCHES:
            mp.delenv(k, raising=False)
        for k, v in env.items():
            mp.setenv(k, v)
        g = RDA_solver(Ts, car, max_edge_num=Es, max_obs_num=Ns, iter_num=iters, iter_threshold=thr, time_print=False,
                       batch=B, **kw)
    dev = _dev(inp)
    outs = []
    if phase:
        g.begin(dev['nom_s'], dev['nom_u'], dev['ref_s'], dev['ref_speed'], dev['obs_A'], dev['obs_b'], dev['obs_kind'],
                dev['obs_count'], tv, thr)
        for _ in range(iters):
            g.step_su()
            g.step_lammuz()
        outs.append({k: v.clone() for k, v in g.finish().items()})
    else:
        for _ in range(calls):
            outs.append({k: v.clone() for k, v in g.iterative_solve_batch(**dev, time_varying=tv).items()})
    state = {name: g.state_buffer(b).reshape(B, -1).clone() for name, b in _state_ids().items()}
    res = {'outs': outs, 'state': state, 'counters': g.state_buffer(_cabi.BUF_COUNTERS).cpu().numpy(),
           'launches': g.launch_count()}
    torch.cuda.synchronize()
    del g, dev
    gc.collect()
    return res


def _assert_copies_equal(big, small, what):
    """Every instance p of the large batch against instance p % U of the small one, bit for bit."""
    B, U = big.shape[0], small.shape[0]
    ref = small.reshape(U, -1)[torch.arange(B, device=small.device) % U]
    got = big.reshape(B, -1)
    if not torch.equal(got, ref):
        bad = (got != ref).any(1).nonzero().flatten()
        gap = float((got.double() - ref.double()).abs().max())
        raise AssertionError(f'{what}: {bad.numel()} of {B} instances differ from their unique instance '
                             f'(first at {bad[:8].tolist()}, max gap {gap:.3e})')


def _check_invariance(big, small, name):
    assert big['launches'] == small['launches'], (name, big['launches'], small['launches'])
    for call, (ob, os_) in enumerate(zip(big['outs'], small['outs'])):
        for k in KEYS:
            _assert_copies_equal(ob[k], os_[k], f'{name} call {call} {k}')
        B, U = ob['u'].shape[0], os_['u'].shape[0]
        idx = torch.arange(B, device=ob['u'].device) % U
        for k in RESIDUALS:     # float atomics: summation order is not fixed
            assert torch.allclose(ob[k], os_[k][idx], rtol=1e-4, atol=1e-6), (name, call, k)
    for k in big['state']:
        _assert_copies_equal(big['state'][k], small['state'][k], f'{name} state {k}')


def _q(x):
    x = np.asarray(x, float)
    return {'median': float(np.median(x)), 'p90': float(np.quantile(x, .9)), 'p99': float(np.quantile(x, .99)),
            'max': float(x.max())}


def _port(car, shape, inp, iters, tv=False, lean2=True, **kw):
    from oracle import cpu_port
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv('RDA_PORT_LEAN2', '1' if lean2 else '0')
        return cpu_port.solve_batch(car, *shape, **inp, time_varying=tv, iter_num=iters, **kw)


def _assert_port_gaps(ds, du):
    """Bounds on the distribution of the per-instance gaps to the port: the bulk as in the existing batch-against-port
    tests (median 2e-4), the tail through its 99th percentile and the share of instances beyond 3e-3.  A few instances in
    two thousand exceed 3e-3 (headline: 1 after 2 iterations, 4 after 4).  Their gap is 1e-10 after the first iteration
    and opens in the second with the same value on every GPU path (k_admm_small, the search pass, the coherent pass), so
    it is the GPU and the g++ build rounding differently, not a pass that large batches select.  On some of them the port
    is the side far from the float64 oracle (metric seed 9705 after 2 iterations: port 3.1e-3 in states, GPU 5e-4), on
    others the GPU (seed 10830: 1.4e-3 in states and 3.0e-3 in controls after 2 iterations, 3e-4 and 7e-4 after 4), and on
    some the port's own two cell pipelines differ by 1e-2 after 4 iterations (seed 10987)."""
    for name, x in (('state', ds), ('control', du)):
        assert np.median(x) <= 2e-4 and np.quantile(x, .99) <= 1e-3, (name, _q(x))
        assert np.count_nonzero(x > 3e-3) <= 0.005 * len(x), (name, np.nonzero(x > 3e-3)[0].tolist())


def _port_gaps(gpu, port, U):
    """Per unique instance: max |s - s_port| and max |u - u_port| of the first U instances of a GPU batch."""
    ds = np.abs(gpu['s'][:U].double().cpu().numpy() - port['s']).reshape(U, -1).max(1)
    du = np.abs(gpu['u'][:U].double().cpu().numpy() - port['u']).reshape(U, -1).max(1)
    return ds, du


# ---------------------------------------------------------------------------------------------------- (a) invariance
@pytest.mark.parametrize('thr', [0.0, 0.2])
def test_headline_batch_equals_its_unique_instances(metric, thr):
    """B = 16 384 with default settings (two sub-batches of 8 192: coherent pass, k_cells_extra, the cooperative pass
    reading its list, wrapped grid-stride loops), 8 iterations cold then a warm-started call, against the 2 048 unique
    instances at B = 2 048 forced through the same passes.  thr = 0.2: instances that stop early are skipped by the
    uniform early exit of k_cells_coh, and every copy must stop at the same iteration."""
    car = rectangle_robot()
    small = _run(SAME_PASSES, car, (T, N, E), metric, 8, thr)
    big = _run({}, car, (T, N, E), _tile(metric, B_HEAD), 8, thr)
    _check_invariance(big, small, f'headline thr={thr}')
    for out in big['outs']:
        assert int((out['status'] & 6).sum()) == 0, 'an instance kept a previous iterate'
    c = big['counters']
    assert c[1] > 0 and c[2] == 0, ('the extra / cooperative passes must resolve cells, none may fail', c[:3].tolist())
    if thr > 0:     # the early exit must actually be taken: some copies stop before the last iteration
        stopped = int(((big['outs'][0]['status'] & 8) != 0).sum())
        early = int((big['outs'][0]['iters'] < 8).sum())
        assert 0 < early < B_HEAD and stopped >= early, (stopped, early)


# ------------------------------------------------------------------------------- (b) oracle, (c) CPU port, headline
def _oracle_positions(B, sms, nb):
    """24 places of the headline batch (two sub-batches of nb): first and last, both sides of the sub-batch boundary, and
    instances whose cells straddle or follow the wraps of the grid-stride loops (16 x SMs CTAs, kernels.cu grid_for):
    k_cells_fast / k_cells_dr at 128 threads per cell, k_begin / k_finish at 256 threads per state entry."""
    cell_sweep = 16 * sms * 128 // (N * T)           # first instance of a sub-batch not finished by the first cell sweep
    state_sweep = 16 * sms * 256 // (3 * (T + 1))
    pos = [0, B - 1, nb - 1, nb]
    for p0 in (0, nb):
        for m in (1, 2, 5, 12):
            pos += [p0 + m * cell_sweep, p0 + m * cell_sweep + 1]
        pos += [p0 + state_sweep, p0 + state_sweep + 1]
    assert len(set(pos)) == 24 and max(pos) < B, pos
    assert cell_sweep + 1 < nb
    return np.array(pos)


@pytest.fixture(scope='module')
def headline_runs(metric):
    """The headline batch with the 24 oracle instances placed inside it, solved cold for 1, 2, 4 and 8 iterations."""
    z = np.load(os.path.join(HERE, 'golden', 'oracle_metric50.npz'))
    orc = _pack([make_instance(int(sd), T=T, N=N, E=E, lateral=tuple(l)) for sd, l in zip(z['seeds'], z['lateral'])], T, N, E)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    pos = _oracle_positions(B_HEAD, sms, B_HEAD // 2)
    inp = _tile(metric, B_HEAD)
    for k in inp:
        inp[k][pos] = orc[k]
    # for the port comparison: one copy of every unique instance that no oracle instance replaced
    copies = np.arange(B_HEAD).reshape(-1, UNIQUE)
    free = ~np.isin(copies, pos)
    pick = copies[free.argmax(0), np.arange(UNIQUE)]
    assert free.any(0).all()
    from rda_planner_b200 import _cabi
    from rda_planner_b200.rda_solver import RDA_solver
    with pytest.MonkeyPatch.context() as mp:
        for k in SWITCHES:
            mp.delenv(k, raising=False)
        g = RDA_solver(T, rectangle_robot(), max_edge_num=E, max_obs_num=N, iter_num=8, iter_threshold=0.0,
                       time_print=False, batch=B_HEAD)
    dev = _dev(inp)
    runs = {}
    for k in (1, 2, 4, 8):
        g.cold_start()
        out = g.iterative_solve_batch(**dev, iter_num=k)
        runs[k] = {n: v.clone() for n, v in out.items()}
        runs[k]['d'] = g.state_buffer(_cabi.BUF_DIS, (B_HEAD, T)).clone()
    torch.cuda.synchronize()
    del g, dev
    gc.collect()
    return {'oracle': z, 'pos': pos, 'pick': pick, 'runs': runs, 'sms': sms}


def test_headline_batch_against_the_float64_oracle(headline_runs):
    """The 24 instances of oracle_metric50.npz inside the B = 16 384 batch, against the float64 trace after 1, 2, 4 and 8
    iterations, within the bounds of test_gpu_parity50.py for those iterations."""
    z, pos = headline_runs['oracle'], headline_runs['pos']
    rows = []
    for k, out in headline_runs['runs'].items():
        sel = torch.as_tensor(pos, device=out['u'].device)
        o = {n: v[sel].double().cpu().numpy() for n, v in out.items()}
        assert int((out['status'][sel] & 6).sum()) == 0, k
        ds = np.abs(o['s'] - z['s'][:, k - 1]).reshape(24, -1).max(1)
        du = np.abs(o['u'] - z['u'][:, k - 1]).reshape(24, -1).max(1)
        dd = np.abs(o['d'] - z['d'][:, k - 1]).reshape(24, -1).max(1)
        rp = np.abs(o['resi_pri'] - z['resi_pri'][:, k - 1]) / (1 + z['resi_pri'][:, k - 1])
        rd = np.abs(o['resi_dual'] - z['resi_dual'][:, k - 1]) / (1 + z['resi_dual'][:, k - 1])
        rows.append({'iteration': k, 'state_gap': _q(ds), 'control_gap': _q(du), 'd_gap': _q(dd),
                     'resi_pri_rel_gap': _q(rp), 'resi_dual_rel_gap': _q(rd)})
        assert ds.max() < 1e-3 and du.max() < 5e-3 and dd.max() < 5e-3, (k, pos[ds.argmax()], ds.max(), du.max(), dd.max())
        assert rp.max() < 2e-3 and rd.max() < 2e-3, (k, rp.max(), rd.max())
    print(json.dumps({'headline_vs_oracle': {'batch': B_HEAD, 'sms': headline_runs['sms'], 'positions': pos.tolist(),
                                             'rows': rows}}))


@pytest.mark.parametrize('iters', [2, 4])
def test_headline_batch_against_the_cpu_port(metric, headline_runs, iters):
    """The 2 048 unique instances through the g++ build of the same cores with the coherent pipeline emulated
    (RDA_PORT_LEAN2=1), against their copies in the B = 16 384 batch."""
    out = headline_runs['runs'][iters]
    sel = torch.as_tensor(headline_runs['pick'], device=out['u'].device)
    port = _port(rectangle_robot(), (T, N, E), metric, iters)
    ds, du = _port_gaps({k: out[k][sel] for k in ('s', 'u')}, port, UNIQUE)
    print(json.dumps({'headline_vs_port': {'iterations': iters, 'instances': UNIQUE, 'state_gap': _q(ds), 'control_gap': _q(du)}}))
    _assert_port_gaps(ds, du)


# ------------------------------------------------------------------------------------ (d) the other streaming variants
def test_disc_body_headline_batch(metric):
    """Disc body (k_cells_dr, k_cells_dr_mid, k_cells_dr_slow_coop) at B = 16 384 against B = 2 048, and against the port."""
    car = disc_robot(radius=1.1, center=(0.2, 0.0), wheelbase=3.0, dynamics='acker')
    small = _run({'RDA_B200_SMALL': '0'}, car, (T, N, E), metric, 4)
    big = _run({}, car, (T, N, E), _tile(metric, B_HEAD), 4)
    _check_invariance(big, small, 'disc body')
    port = _port(car, (T, N, E), metric, 2, lean2=False)
    ref = _run({'RDA_B200_SMALL': '0'}, car, (T, N, E), metric, 2, calls=1)     # same instances, 2 iterations
    ds, du = _port_gaps(ref['outs'][0], port, UNIQUE)
    print(json.dumps({'disc_body_vs_port': {'iterations': 2, 'state_gap': _q(ds), 'control_gap': _q(du)}}))
    _assert_port_gaps(ds, du)


def test_moving_discs_large_batch():
    """Moving discs (per-stage obstacle copies, coherent pass skipped) at B = 8 192 against the 1 024 unique instances
    forced through k_cells_extra in two sub-batches, and against the port."""
    U, B = 1024, 8192
    inst = _pack([make_instance(1500 + i, T=T, N=N, E=E, kind='circle', moving=True, lateral=(0.3, 3.5)) for i in range(U)],
                 T, N, E)
    assert inst['obs_A'].shape[2] == T + 1
    car = rectangle_robot()
    env = {'RDA_B200_SMALL': '0', 'RDA_B200_EXTRA_MIN': '1', 'RDA_B200_SPLIT_MIN': '2'}
    small = _run(env, car, (T, N, E), inst, 4, tv=True)
    big = _run({}, car, (T, N, E), _tile(inst, B), 4, tv=True)
    _check_invariance(big, small, 'moving discs')
    assert big['counters'][1] > 0 and big['counters'][2] == 0
    port = _port(car, (T, N, E), inst, 2, tv=True, lean2=False)
    ref = _run(env, car, (T, N, E), inst, 2, calls=1, tv=True)
    ds, du = _port_gaps(ref['outs'][0], port, U)
    print(json.dumps({'moving_discs_vs_port': {'iterations': 2, 'state_gap': _q(ds), 'control_gap': _q(du)}}))
    _assert_port_gaps(ds, du)


def test_config_d_shape_with_wrapped_grid():
    """Config D's shape (T = 30, N = 64 hulls of up to 8 faces: k_cells_fast<8, 8, false>), 256 unique instances tiled to
    4 096: 3.9 M cells per sub-batch, many sweeps of the grid-stride loops.  The small batch is split into two parts too."""
    from rda_planner_b200.scenarios import CONFIGS
    c = CONFIGS['D']
    U, B, shape = 256, 4096, (c['T'], c['N'], c['E'])
    inst = _pack([config_instance('D', 7000 + i) for i in range(U)], *shape)
    car = rectangle_robot(dynamics=c['dynamics'])
    assert B // 2 * c['N'] * c['T'] > 4 * 16 * torch.cuda.get_device_properties(0).multi_processor_count * 128
    small = _run({'RDA_B200_SMALL': '0', 'RDA_B200_SPLIT_MIN': '2'}, car, shape, inst, 4, **c['tun'])
    big = _run({}, car, shape, _tile(inst, B), 4, **c['tun'])
    _check_invariance(big, small, 'config D')
    port = _port(car, shape, inst, 2, lean2=False, **c['tun'])
    ref = _run({'RDA_B200_SMALL': '0'}, car, shape, inst, 2, calls=1, **c['tun'])
    ds, du = _port_gaps(ref['outs'][0], port, U)
    print(json.dumps({'config_d_vs_port': {'iterations': 2, 'state_gap': _q(ds), 'control_gap': _q(du)}}))
    _assert_port_gaps(ds, du)


def test_float32_su_headline_batch(metric):
    """su_fp64=False (k_su<float>) at B = 16 384 against B = 2 048 through the same passes."""
    car = rectangle_robot()
    small = _run(SAME_PASSES, car, (T, N, E), metric, 4, su_fp64=False)
    big = _run({}, car, (T, N, E), _tile(metric, B_HEAD), 4, su_fp64=False)
    _check_invariance(big, small, 'float32 su-QP')


# ---------------------------------------------------------------------------------- (e) more than 65 535 per launch
@pytest.fixture(scope='module')
def config_a():
    from rda_planner_b200.scenarios import CONFIGS
    c = CONFIGS['A']
    shape = (c['T'], c['N'], c['E'])
    return shape, c['tun'], _pack([config_instance('A', 3000 + i) for i in range(257)], *shape)


def test_phase_api_above_65535_instances(config_a):
    """65 553 instances of config A's shape in one launch of every kernel (the phase API runs the batch as one part):
    the coherent pass used to be launched with one grid row per instance, which gridDim.y caps at 65 535."""
    shape, tun, inst = config_a
    car = rectangle_robot()
    small = _run(SAME_PASSES, car, shape, inst, 2, phase=True, **tun)
    big = _run({}, car, shape, _tile(inst, 65536 + 17), 2, phase=True, **tun)
    _check_invariance(big, small, 'phase API, B = 65 553')


def test_solve_with_sub_batches_above_65535_instances(config_a):
    """2 x 65 553 instances through iterative_solve_batch: two sub-batches, each above 65 535 instances."""
    shape, tun, inst = config_a
    car = rectangle_robot()
    small = _run(dict(SAME_PASSES, RDA_B200_SPLIT_MIN='2'), car, shape, inst, 2, **tun)
    big = _run({}, car, shape, _tile(inst, 2 * 65536 + 34), 2, **tun)
    _check_invariance(big, small, 'solve, B = 131 106')
