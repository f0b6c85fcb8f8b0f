"""The su-QP kernels on their own: k_su (one warp per instance) and the su-QP of the persistent kernel k_admm_small, one
solve with inputs set directly, against the CPU build of the same core (su_solver.cuh under g++, one lane) and the dense
float64 oracle.  The CPU build is the tight reference: a difference from it is a warp or device effect (stage ownership
by lane, warp reductions, gains written by lane 0, the compact hinge list, the device reciprocal, the workspace in shared
memory), not an algorithm effect.

The solve is driven through the phase API: begin() with zero obstacles stages the nominal and the reference, the hinge
inputs (BUF_COEF), their positions (BUF_PREF) and the initial safety distances (BUF_DIS) are loaded directly (k_begin
writes none of them), step_su() runs k_su once.  k_admm_small runs one ADMM iteration with obs_count = 0, which skips
the cells, so its result is the su-QP solution.  Counters: [3] interior point iterations, [4] solves, [5] pruned solves
repeated with all hinges."""
import contextlib
import os

import numpy as np
import pytest
import torch

import su_cases as sc
from test_su_restarts import fixture_cases

pytestmark = pytest.mark.gpu

# The device returns s, u and d in float32, so they are compared with the CPU build's solution rounded to float32, in
# units of its float32 spacing (at least 2^-23): `_ulps`.  Measured on an H100 (80 GB HBM3, 700 W) over every case of this
# file: the float64 kernels agree with the float64 CPU build after rounding in 357 of 359 solves, the largest gap is
# 0.0078 (a value near zero), and every batch took exactly the CPU build's interior point iterations.  The float32
# kernels against the float32 CPU build: median 62, largest 4.75e4 spacings; 2 of 16 batches differ by one iteration
# (float32 rounding and contraction differ between the device and the host).  Bounds: about 10 x the largest gap.
GAP_F64 = 0.1
GAP_F32 = 5e5
TOL_F32 = 1e-3           # float32 kernels against the oracle (the CPU float32 build's bound)


@contextlib.contextmanager
def _env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update({k: str(v) for k, v in kv.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _stack(probs):
    return {k: np.stack([np.asarray(p[k], np.float32) for p in probs]) for k in ('cur_s', 'cur_u', 'ref_s', 'dis', 'pref', 'coef')} | \
        {'vref': np.array([p['vref'] for p in probs], np.float32)}


def gpu(probs, dyn='acker', acc=True, fp64=True, tun=sc.TUN, prune=sc.PRUNE, kernel='k_su'):
    """One su-QP solve of every problem (same T, N) in one batch: dict of s [B,3,T+1], u [B,2,T], d [B,T], status [B],
    counters [8], cur_s / cur_u (the persistent nominal after the solve)."""
    from rda_planner_b200 import _cabi
    from rda_planner_b200.rda_solver import RDA_solver
    from rda_planner_b200.scenarios import rectangle_robot
    T, N, B = probs[0]['T'], probs[0]['N'], len(probs)
    x = _stack(probs)
    with _env(RDA_B200_SU_PRUNE=prune, RDA_B200_SMALL=1 if kernel == 'small' else 0):
        g = RDA_solver(T, rectangle_robot(dynamics=dyn), max_edge_num=4, max_obs_num=N, batch=B, accelerated=acc,
                       su_fp64=fp64, device='cuda:0', time_print=False, iter_threshold=0.0,
                       **{k: tun[k] for k in ('slack_gain', 'max_sd', 'min_sd', 'ro1', 'ro2', 'wu')})
    obs = {}
    if N > 0:
        obs = dict(obs_A=np.zeros((B, N, 1, 4, 2), np.float32), obs_b=np.zeros((B, N, 1, 4), np.float32),
                   obs_kind=np.zeros((B, N), np.int32), obs_count=np.zeros(B, np.int32))
    args = (x['cur_s'], x['cur_u'], x['ref_s'], x['vref'])

    def load():
        if N > 0:
            g.load_state_buffer(_cabi.BUF_COEF, x['coef'])
        g.load_state_buffer(_cabi.BUF_PREF, x['pref'])
        g.load_state_buffer(_cabi.BUF_DIS, x['dis'])
        g.load_state_buffer(_cabi.BUF_COUNTERS, np.zeros(8, np.int32))

    if kernel == 'small':
        load()
        out = g.iterative_solve_batch(*args, **obs, iter_num=1, iter_threshold=0.0)
        assert g.launch_count() == 1          # k_admm_small and nothing else
    else:
        g.begin(*args, **obs)
        load()
        g.step_su()
        out = g.finish()
    torch.cuda.synchronize()
    r = {k: out[k].cpu().numpy().astype(float) for k in ('s', 'u')}
    r['status'] = out['status'].cpu().numpy()
    r['d'] = g.state_buffer(_cabi.BUF_DIS, (B, T)).cpu().numpy().astype(float)
    r['counters'] = g.state_buffer(_cabi.BUF_COUNTERS).cpu().numpy()
    r['cur_s'] = g.state_buffer(_cabi.BUF_CUR_S, (B, 3, T + 1)).cpu().numpy()
    r['cur_u'] = g.state_buffer(_cabi.BUF_CUR_U, (B, 2, T)).cpu().numpy()
    r['d32'] = g.state_buffer(_cabi.BUF_DIS, (B, T)).cpu().numpy()
    return r


def _ulps(r, b, ref):
    """Largest gap of instance b's (s, u, d) to ref rounded to float32, in units of max(float32 spacing, 2^-23)."""
    g = 0.0
    for k, v in zip('sud', ref):
        c = np.reshape(np.asarray(v, np.float32), r[k][b].shape)
        if c.size:
            g = max(g, float((np.abs(r[k][b] - c) / np.maximum(np.spacing(np.abs(c)), 2.0 ** -23)).max()))
    return g


GAPS = []      # (case, gap) of every comparison with the CPU build; (case + " iterations", GPU - CPU total) per batch


def check(probs, r, dyn='acker', acc=True, fp64=True, tun=sc.TUN, prune=sc.PRUNE, case=''):
    """Every instance against the CPU build in the kernel's precision (GAP_F64 / GAP_F32, `_ulps`): every solve converged
    and counted, and as many repeated as on the CPU build."""
    T, N = probs[0]['T'], probs[0]['N']
    P = sc.params(T, N, dyn, int(acc), prune, tun)
    its = restarts = 0
    for b, p in enumerate(probs):
        s, u, d, st, it, rep = sc.cpu(p, P, prec='d' if fp64 else 'f')
        assert st == 0 and r['status'][b] == 0, (case, b, st, r['status'][b])
        its += it
        restarts += rep['restarts']
        g = _ulps(r, b, (s, u, d))
        GAPS.append((('abs f64 ' if fp64 else 'abs f32 ') + case, max(float(np.abs(r[k][b] - np.reshape(np.float32(v), r[k][b].shape)).max(initial=0.0)) for k, v in zip('sud', (s, u, d)))))
        GAPS.append((('f64 ' if fp64 else 'f32 ') + case, g))
        assert g <= (GAP_F64 if fp64 else GAP_F32), (case, b, g)
    assert r['counters'][4] == len(probs) and r['counters'][5] == restarts, (case, r['counters'])
    GAPS.append((('f64 ' if fp64 else 'f32 ') + case + ' iterations', int(r['counters'][3]) - its))
    return its


def check_oracle(probs, r, acc=True, tun=sc.TUN, n=2):
    """The first n instances against the dense float64 oracle, at the CPU build's bounds (tests/test_su_restarts.py)."""
    from test_su_restarts import _tol
    for b, p in enumerate(probs[:n]):
        so, uo, do, info = sc.oracle(p, acc, tun).su_prob_solve()
        assert info['status'] in ('optimal', 'optimal_inaccurate'), info['status']
        for k, v, t in zip('sud', (so, uo, do), _tol(p['T'])):
            np.testing.assert_allclose(r[k][b], np.reshape(v, r[k][b].shape), atol=t, err_msg=f'{b} {k}')


@pytest.mark.parametrize('T', [1, 2, 31, 32, 33, 64, 65, 100])
def test_horizons(T):
    """Lanes own 0 to 4 stages; the rate rows of stage 0 are dead."""
    probs = [sc.problem(9000 + 10 * T + b, T, 3) for b in range(8)]
    r = gpu(probs)
    check(probs, r, case=f'T={T} N=3')
    if T <= 33:
        check_oracle(probs, r)


@pytest.mark.parametrize('N', [0, 1, 2, 3, 31, 32, 33, 64, 65, 128, 256])
def test_obstacle_counts(N):
    """1 to 8 hinge mask words; N <= 2 keeps every hinge (the two nearest); N = 0 has no d rows."""
    T = 4
    probs = [sc.problem(9500 + 10 * N + b, T, N, near=min(N, 6)) for b in range(8)]
    r = gpu(probs)
    check(probs, r, case=f'T={T} N={N}')
    if 0 < N * T <= 256:
        check_oracle(probs, r, n=1)


def test_joint_33_by_33():
    probs = [sc.problem(9900 + b, 33, 33, near=8) for b in range(6)]
    r = gpu(probs)
    check(probs, r, case='T=33 N=33')
    check_oracle(probs, r, n=1)


@pytest.mark.parametrize('fp64', [True, False])
@pytest.mark.parametrize('dyn,acc,prune', [('acker', True, sc.PRUNE), ('acker', True, 0.0), ('acker', False, sc.PRUNE),
                                            ('diff', True, sc.PRUNE), ('diff', False, sc.PRUNE),
                                            ('omni', True, sc.PRUNE), ('omni', False, sc.PRUNE), ('omni', True, 0.0)])
def test_configurations(dyn, acc, prune, fp64):
    T, N = 12, 8
    probs = [sc.problem(9700 + b, T, N, dyn=dyn) for b in range(16)]
    r = gpu(probs, dyn, acc, fp64, prune=prune)
    check(probs, r, dyn, acc, fp64, prune=prune, case=f'{dyn} acc={acc} prune={prune} fp64={fp64}')


@pytest.mark.parametrize('tun', ['TUN_C', 'TUN_D'])
def test_config_c_and_d_tunables(tun):
    T, N = 30, 20
    probs = [sc.problem(9800 + b, T, N, near=6) for b in range(8)]
    r = gpu(probs, tun=getattr(sc, tun))
    check(probs, r, tun=getattr(sc, tun), case=tun)


@pytest.mark.parametrize('acc', [True, False])
def test_more_than_32_hinges_per_stage(acc):
    """tests/test_su_many_hinges.py on the device: T = 8, N = 64 with 40 near activity, so that pruning keeps more than
    32 hinges at every stage, spread over both mask words."""
    probs = [sc.problem(seed, 8, 64, near=40) for seed in (61, 62, 63, 64)]
    P = sc.params(8, 64)
    pos = sc.rollout(probs[0], P)
    kept = [sum(not sc.left_out(probs[0], pos, t, o) for o in range(64)) for t in range(8)]
    assert min(kept) > 32 and max(kept) < 64, kept
    r = gpu(probs, acc=acc)
    check(probs, r, acc=acc, case=f'many hinges acc={acc}')
    check_oracle(probs, r, acc=acc)


@pytest.mark.parametrize('T,N', list(sc.RESTARTS))
def test_repeated_pruned_solves(T, N):
    """Hinges left out at the nominal rollout and violated at the pruned optimum (tests/su_cases.py: RESTARTS): exactly
    the planted instances repeat their solve, the result is the optimum with all hinges (oracle) and the unpruned
    solve's; with pruning off nothing repeats."""
    cases = sc.RESTARTS[(T, N)]
    probs = [sc.restart_problem(T, N, seed, cells) for seed, cells in cases]
    planted = sum(1 for _, cells in cases if cells)
    r = gpu(probs)
    check(probs, r, case=f'restarts T={T} N={N}')
    assert r['counters'][5] == planted, r['counters']
    r0 = gpu(probs, prune=0.0)
    check(probs, r0, prune=0.0, case=f'restarts unpruned T={T} N={N}')
    assert r0['counters'][5] == 0, r0['counters']
    from test_su_restarts import _tol
    for k, t in zip('sud', _tol(T)):
        np.testing.assert_allclose(r[k], r0[k], atol=t)
    check_oracle(probs, r, n=len(probs) if T * N <= 500 else 2)


def test_pruned_attempt_stopped_by_its_iteration_cap():
    """su_cases.CAPPED: the pruned attempt stops at its cap of 24 iterations on the CPU build; the device repeats the same
    solve (counters[5]) and ends at the oracle's optimum."""
    T, N, seed = sc.CAPPED
    probs = [sc.restart_problem(T, N, seed, [])]
    r = gpu(probs)
    check(probs, r, case='capped')
    assert r['counters'][5] == 1 and r['counters'][3] >= 24, r['counters']
    check_oracle(probs, r, n=1)


def test_config_d_and_e_sizes_against_the_committed_oracle_solves():
    from test_su_restarts import _tol
    by_size = {}
    for c in fixture_cases():
        by_size.setdefault((c[1]['T'], c[1]['N']), []).append(c)
    for (T, N), cases in by_size.items():
        tun = cases[0][2]
        assert all(c[2] is tun for c in cases)
        probs = [c[1] for c in cases]
        for fp64 in (True, False):
            r = gpu(probs, tun=tun, fp64=fp64)
            assert r['counters'][5] == sum(c[3] for c in cases), r['counters']
            for b, (name, p, _, _, ref, _) in enumerate(cases):
                for k, v, t in zip('sud', ref, _tol(T) if fp64 else (TOL_F32,) * 3):
                    np.testing.assert_allclose(r[k][b], np.reshape(v, r[k][b].shape), atol=t, err_msg=f'{name} fp64={fp64} {k}')
            check(probs, r, fp64=fp64, tun=tun, case=f'fixture T={T} N={N} fp64={fp64}')


@pytest.mark.parametrize('prune', [sc.PRUNE, 0.0])
def test_non_finite_inputs_keep_the_previous_nominal(prune):
    """A NaN g_x and an Inf c0: RDA_ST_SU_NONFINITE, the persistent nominal and safety distances bitwise unchanged; the
    other instances bitwise as in the batch without the two.  With pruning a hinge whose c0 is +Inf is left out and its
    check passes (l = +Inf), so the instance solves without it, as the CPU build does."""
    from rda_planner_b200 import _cabi
    T, N = 12, 8
    probs = [sc.problem(9600 + b, T, N) for b in range(6)]
    probs[1]['coef'][3, 2, 5] = np.nan
    probs[4]['coef'][2, 6, 3] = np.inf
    r = gpu(probs, prune=prune)
    good = [0, 2, 3, 5]
    r1 = gpu([probs[b] for b in good], prune=prune)
    P = sc.params(T, N, prune=prune)
    bad = []
    for b in (1, 4):
        s, u, d, st, _, _ = sc.cpu(probs[b], P)
        if st == 2:
            bad.append(b)
            assert r['status'][b] & _cabi.ST_SU_NONFINITE, (b, r['status'][b])
            assert np.array_equal(r['cur_s'][b], probs[b]['cur_s'].astype(np.float32))
            assert np.array_equal(r['cur_u'][b], probs[b]['cur_u'].astype(np.float32))
            assert np.array_equal(r['d32'][b], probs[b]['dis'].astype(np.float32))
        else:
            assert r['status'][b] == 0 and _ulps(r, b, (s, u, d)) <= GAP_F64
    assert 1 in bad and (prune > 0 or 4 in bad), bad
    for i, b in enumerate(good):
        for k in ('s', 'u', 'd', 'status'):
            assert np.array_equal(r[k][b], r1[k][i]), (b, k)


def test_batch_position_does_not_change_a_solve():
    T, N, B = 12, 8, 301
    probs = [sc.problem(20000 + b, T, N) for b in range(B)]
    for b in (0, B // 2, B - 1):
        probs[b] = sc.problem(777, T, N)
    r = gpu(probs)
    assert r['counters'][4] == B
    for k in ('s', 'u', 'd', 'status'):
        assert np.array_equal(r[k][0], r[k][B // 2]) and np.array_equal(r[k][0], r[k][B - 1]), k


@pytest.mark.parametrize('fp64', [True, False])
@pytest.mark.parametrize('T,N', [(33, 33), (64, 3), (12, 8)])
def test_persistent_kernel_su_qp_matches_k_su(T, N, fp64):
    """k_admm_small's su-QP (workspace and hinge arrays in shared memory) against k_su on the same inputs and both
    against the CPU build.  N T = 1089 stages the per-cell arrays by the threads, 192 and 96 by bulk copies."""
    probs = [sc.problem(30000 + b, T, N, near=min(N, 6)) for b in range(4)]
    small = gpu(probs, fp64=fp64, kernel='small')
    ksu = gpu(probs, fp64=fp64)
    for r in (small, ksu):
        check(probs, r, fp64=fp64, case=f'{"small" if r is small else "k_su"} T={T} N={N} fp64={fp64}')
    # the same core and the same arithmetic: bitwise equal on the H100
    for k in ('s', 'u', 'd', 'status', 'counters'):
        assert np.array_equal(small[k], ksu[k]), k


def test_report_gaps():
    """Prints the measured gaps (run with -s); the bounds above are set from them."""
    for prec in ('f64', 'f32'):
        g = [x for c, x in GAPS if c.startswith(prec) and not c.endswith('iterations')]
        it = [x for c, x in GAPS if c.startswith(prec) and c.endswith('iterations')]
        if g:
            print(f'\n{prec} largest absolute gap: {max(x for c, x in GAPS if c.startswith("abs " + prec)):.3g}')
            print(f'{prec} kernels vs CPU build: {len(g)} solves, gap in float32 spacings max {max(g):.3g}, '
                  f'p50 {np.median(g):.3g}, p99 {np.quantile(g, 0.99):.3g}, nonzero {sum(1 for x in g if x > 0)}')
            print(f'{prec} batches whose iteration total differs from the CPU build: {sum(1 for x in it if x)} of {len(it)}: {it}')
    for c, x in GAPS:
        print('GAP', c, x)
