"""The pruned su-QP solve of the CPU build of su_solver.cuh (accelerated mode): hinges far from activity at the nominal
rollout are left out of the interior point iteration and checked at its solution; a violated one repeats the solve
with every hinge.  The problems of tests/su_cases.py: RESTARTS plant such hinges; the solution of the repeated solve
must be the optimum of the problem with all hinges (the dense float64 oracle) and of the unpruned solve.  Also the
config D and E sizes against the committed oracle solves (tests/golden/oracle_su.npz)."""
import os

import numpy as np
import pytest

import su_cases as sc

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'oracle_su.npz')


def _tol(T):
    """Bounds of the CPU build against the oracle (s, u, d): test_host_cores.py at T <= 12 and, at T = 30-40, the gap of
    the core to a 1e-13 solve (test_su_core_is_closer_to_the_optimum_than_a_1e9_oracle_solve_at_metric_size)."""
    return (2e-5, 2e-5, 2e-5) if T <= 12 else (5e-5, 5e-4, 5e-4)


def _close(got, ref, tol, what=''):
    for a, b, t, k in zip(got, ref, tol, 'sud'):
        np.testing.assert_allclose(a, np.reshape(b, np.shape(a)), atol=t, err_msg=f'{what} {k}')


@pytest.mark.parametrize('T,N', list(sc.RESTARTS))
def test_pruned_solve_is_repeated_when_a_left_out_hinge_is_violated(T, N):
    P, P0 = sc.params(T, N), sc.params(T, N, prune=0.0)
    for seed, cells in sc.RESTARTS[(T, N)]:
        p = sc.restart_problem(T, N, seed, cells)
        pos = sc.rollout(p, P)
        assert all(sc.left_out(p, pos, t, o) for t, o in cells)
        s, u, d, st, it, rep = sc.cpu(p, P)
        assert st == 0, (seed, st, it)
        assert rep == {'restarts': int(bool(cells)), 'verified': 1, 'violated': int(bool(cells)), 'capped': 0}, (seed, rep)
        s0, u0, d0, st0, _, rep0 = sc.cpu(p, P0)
        assert st0 == 0 and rep0['restarts'] == 0 and rep0['verified'] == 0
        _close((s, u, d), (s0, u0, d0), _tol(T), f'seed {seed}: pruned vs unpruned')
        so, uo, do, info = sc.oracle(p).su_prob_solve()
        assert info['status'] in ('optimal', 'optimal_inaccurate'), info['status']
        _close((s, u, d), (so, uo, do), _tol(T), f'seed {seed}: vs oracle')


def test_float32_build_repeats_the_same_pruned_solves():
    for (T, N), cases in sc.RESTARTS.items():
        P = sc.params(T, N)
        for seed, cells in cases:
            p = sc.restart_problem(T, N, seed, cells)
            s, u, d, st, it, rep = sc.cpu(p, P, prec='f')
            sd, ud, dd, _, _, _ = sc.cpu(p, P)
            assert st == 0 and rep['restarts'] == int(bool(cells)), (T, N, seed, st, rep)
            _close((s, u, d), (sd, ud, dd), (1e-3, 1e-3, 1e-3), f'{T} {N} {seed}')


def test_iteration_cap_of_the_pruned_attempt_repeats_the_solve_with_all_hinges():
    """With max_iter below the pruned attempt's cap of 24 both attempts stop at the cap: the repeat is reported as
    caused by the cap, never by the verification, and every iteration of both attempts is counted."""
    T, N = 12, 40
    p = sc.restart_problem(T, N, *sc.RESTARTS[(T, N)][0])
    P = sc.params(T, N, max_iter=6)
    s, u, d, st, it, rep = sc.cpu(p, P)
    assert st == 1 and it == 12 and rep == {'restarts': 1, 'verified': 0, 'violated': 0, 'capped': 1}, (st, it, rep)
    assert np.all(np.isfinite(s)) and np.all(np.isfinite(u)) and np.all(np.isfinite(d))


def test_pruned_attempt_stopped_by_its_iteration_cap_is_repeated_with_all_hinges():
    """A problem whose pruned attempt does not converge within its 24 iterations (su_cases.CAPPED): the repeat is caused by
    the cap, not by the check of the left-out hinges, and ends at the optimum with all hinges."""
    T, N, seed = sc.CAPPED
    p = sc.restart_problem(T, N, seed, [])
    s, u, d, st, it, rep = sc.cpu(p, sc.params(T, N))
    assert st == 0 and it >= 24 and rep == {'restarts': 1, 'verified': 0, 'violated': 0, 'capped': 1}, (st, it, rep)
    so, uo, do, info = sc.oracle(p).su_prob_solve()
    _close((s, u, d), (so, uo, do), _tol(T), 'capped')
    s0, u0, d0, st0, _, rep0 = sc.cpu(p, sc.params(T, N, prune=0.0))
    assert st0 == 0 and rep0['restarts'] == 0
    _close((s, u, d), (s0, u0, d0), _tol(T), 'capped vs unpruned')


def fixture_cases():
    f = np.load(FIXTURE)
    out = []
    for name in f['names']:
        name = str(name)
        p = {k: f[f'{name}_{k}'].astype(float) for k in ('cur_s', 'cur_u', 'ref_s', 'dis', 'pref', 'coef')}
        T, N = p['dis'].shape[0], p['coef'].shape[1]
        p.update(T=T, N=N, dyn='acker', vref=float(f[f'{name}_vref']))
        ref = tuple(f[f'{name}_{k}'] for k in 'sud')
        out.append((name, p, getattr(sc, str(f[f'{name}_tun'])), len(f[f'{name}_cells']) > 0, ref, float(f[f'{name}_merit'])))
    return out


def test_config_d_and_e_sizes_match_the_committed_oracle_solves():
    """T = 30 / N = 64 (config D's tunables) and T = 40 / N = 128, each near activity and with planted hinges that
    repeat the pruned solve; the float32 build within 1e-3."""
    cases = fixture_cases()
    assert {c[0] for c in cases} == {'D', 'D_restart', 'E', 'E_restart'}
    for name, p, tun, restart, ref, merit in cases:
        assert merit < 1e-6, (name, merit)
        P = sc.params(p['T'], p['N'], tun=tun)
        s, u, d, st, it, rep = sc.cpu(p, P)
        assert st == 0 and rep['restarts'] == int(restart), (name, st, it, rep)
        _close((s, u, d), ref, _tol(p['T']), name)
        s, u, d, st, it, rep = sc.cpu(p, P, prec='f')
        assert st in (0, 1) and rep['restarts'] == int(restart), (name, st, it, rep)
        _close((s, u, d), ref, (1e-3, 1e-3, 1e-3), name + ' float32')
