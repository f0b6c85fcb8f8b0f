"""-m gpu: the cell passes hand the cells they decline to the next pass as packed records (CellRec, rda_kernels.cu).

A record carries every value of a cell the passes read from the state planes besides the obstacle rows, so a later pass
runs the same cell arithmetic on the same bits whether it reads the record or the planes.  At the headline shape (bench.py's
first 2 048 instances tiled 8x to B = 16 384, phase API, one stream) the whole persistent state after ADMM iterations 1, 2
and 8 must be bitwise equal, copy for copy, to the unique instances solved in a small batch forced through the same passes.
For the rectangle those are the coherent pass, the listed first pass, the searched pass, k_cells_extra and the cooperative
pass; for bench.py's disc body k_cells_dr, k_cells_dr_mid and k_cells_dr_slow_coop.  The state includes COEF and PREF, which
the end-of-solve outputs do not show.  The cold start's first iteration, in which the rectangle's coherent pass has no
support-vertex pairs and declines every cell, must resolve every cell once: no record may be lost for want of room."""
import gc

import numpy as np
import pytest
import torch

from rda_planner_b200.scenarios import disc_robot, make_instance, rectangle_robot

pytestmark = pytest.mark.gpu
T, N, E = 30, 20, 4
UNIQUE, B_HEAD = 2048, 16384
SWITCHES = ('RDA_B200_SMALL', 'RDA_B200_LEAN2', 'RDA_B200_EXTRA_MIN', 'RDA_B200_SPLIT_MIN', 'RDA_B200_SPLIT_PARTS')
# body -> (car tuple, the switches that send the small batch through the headline batch's passes)
BODIES = {'rectangle': (rectangle_robot, {'RDA_B200_SMALL': '0', 'RDA_B200_LEAN2': '1', 'RDA_B200_EXTRA_MIN': '1'}),
          'disc': (lambda: disc_robot(radius=1.2, wheelbase=2.0, dynamics='diff'), {'RDA_B200_SMALL': '0'})}
CHECKPOINTS = (1, 2, 8)
STATE = ('LAM', 'MU', 'Z', 'ZETA', 'XI', 'COEF', 'PREF')


@pytest.fixture(scope='module')
def metric():
    """bench.py's metric instances 0..2047 (seeds 9000..)."""
    from rda_planner_b200.rda_solver import pack_obstacles
    insts = [make_instance(9000 + i, T=T, N=N, E=E) for i in range(UNIQUE)]
    packs = [pack_obstacles(list(i['obstacles']), T, N, E) for i in insts]
    return dict(nom_s=np.stack([i['nom_s'] for i in insts]).astype(np.float32),
                nom_u=np.stack([i['nom_u'] for i in insts]).astype(np.float32),
                ref_s=np.stack([i['ref'] for i in insts]).astype(np.float32),
                ref_speed=np.array([i['ref_speed'] for i in insts], np.float32),
                obs_A=np.stack([p[0] for p in packs]), obs_b=np.stack([p[1] for p in packs]),
                obs_kind=np.stack([p[2] for p in packs]), obs_count=np.array([p[3] for p in packs], np.int32))


def _solver(body, env, B):
    from rda_planner_b200.rda_solver import RDA_solver
    with pytest.MonkeyPatch.context() as mp:
        for k in SWITCHES:
            mp.delenv(k, raising=False)
        for k, v in env.items():
            mp.setenv(k, v)
        return RDA_solver(T, BODIES[body][0](), max_edge_num=E, max_obs_num=N, iter_num=max(CHECKPOINTS),
                          iter_threshold=0.0, time_print=False, batch=B)


def _phase(body, env, inp, B, visit):
    """Cold start, begin, then ADMM iterations through the phase API; visit(iteration, solver) at every checkpoint."""
    g = _solver(body, env, B)
    dev = {k: torch.as_tensor(v[np.arange(B) % UNIQUE], device='cuda') for k, v in inp.items()}
    g.cold_start()
    g.begin(dev['nom_s'], dev['nom_u'], dev['ref_s'], dev['ref_speed'], dev['obs_A'], dev['obs_b'], dev['obs_kind'],
            dev['obs_count'], False, 0.0)
    for it in range(1, max(CHECKPOINTS) + 1):
        g.step_su()
        g.step_lammuz()
        if it in CHECKPOINTS:
            visit(it, g)
    torch.cuda.synchronize()
    del g, dev
    gc.collect()


def _state(g, B):
    from rda_planner_b200 import _cabi
    return {k: g.state_buffer(getattr(_cabi, 'BUF_' + k)).reshape(B, -1).clone() for k in STATE}


def _counters(g):
    from rda_planner_b200 import _cabi
    return g.state_buffer(_cabi.BUF_COUNTERS).cpu().numpy().astype(np.int64)


def _headline_state_matches_unique_instances(metric, body):
    """B = 16 384 copies of 2 048 unique instances: LAM, MU, Z, ZETA, XI, COEF and PREF after ADMM iterations 1, 2 and 8
    bitwise equal to the small batch run through the same passes, and every pass resolving 8x the small batch's cells."""
    small = {}
    _phase(body, BODIES[body][1], metric, UNIQUE, lambda it, g: small.__setitem__(it, (_state(g, UNIQUE), _counters(g))))
    idx = torch.arange(B_HEAD, device='cuda') % UNIQUE
    seen = []

    def check(it, g):
        state, cnt = _state(g, B_HEAD), _counters(g)
        ref_state, ref_cnt = small[it]
        for k in STATE:
            got, ref = state[k], ref_state[k][idx]
            if not torch.equal(got, ref):
                bad = (got != ref).any(1).nonzero().flatten()
                raise AssertionError(f'iteration {it} {k}: {bad.numel()} of {B_HEAD} copies differ from their unique '
                                     f'instance (first at {bad[:8].tolist()})')
        # cells resolved by the closed forms / by the cooperative pass / failed
        assert (cnt[:3] == (B_HEAD // UNIQUE) * ref_cnt[:3]).all(), (it, cnt[:3].tolist(), ref_cnt[:3].tolist())
        seen.append(it)
    _phase(body, {}, metric, B_HEAD, check)
    assert seen == list(CHECKPOINTS)


def _cold_start_resolves_every_cell_once(metric, body):
    """The first iteration after a cold start resolves every cell of the 16 384 instances exactly once."""
    live = int((metric['obs_count'][np.arange(B_HEAD) % UNIQUE] > 0).sum())
    res = {}

    def first(it, g):
        if it == 1:
            res['cnt'] = _counters(g)
    _phase(body, {}, metric, B_HEAD, first)
    cnt = res['cnt']
    assert int(cnt[0] + cnt[1] + cnt[2]) == live * N * T, (cnt[:3].tolist(), live * N * T)


def test_headline_state_matches_unique_instances(metric):
    _headline_state_matches_unique_instances(metric, 'rectangle')


def test_disc_headline_state_matches_unique_instances(metric):
    _headline_state_matches_unique_instances(metric, 'disc')


def test_cold_start_every_cell_declined_fits(metric):
    """The rectangle's coherent pass declines every cell (no support-vertex pairs yet); the later passes resolve each once."""
    _cold_start_resolves_every_cell_once(metric, 'rectangle')


def test_disc_cold_start_every_cell_resolved_once(metric):
    _cold_start_resolves_every_cell_once(metric, 'disc')
