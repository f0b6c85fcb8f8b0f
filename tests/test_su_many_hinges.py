"""The su-QP core (csrc/su_solver.cuh, CPU build) with more obstacles than one hinge-mask word holds, against the dense
oracle QP (oracle/qp_ipm.py through OracleRDA.su_prob_solve).  N = 64 hinges per stage, 40 of them near activity: with
pruning (accelerated mode) every stage keeps more than 32 hinges spread over both mask words, a different set at every
stage; without acceleration every hinge is a plain quadratic and all 64 are kept."""
import numpy as np
import pytest

import shim
from oracle.rda_oracle import OracleRDA
from rda_planner_b200.scenarios import rectangle_robot, make_instance

T, N, NEAR = 8, 64, 40
PRUNE, DMAX = 0.5, 1.0


def _f32(a):
    return np.asarray(a, np.float32).astype(float)


def _problem(seed):
    """Nominal trajectory of a generated instance; N hinge rows per stage with unit normals, NEAR of them (a random set
    per stage) with margins in [-0.5, 1] at the nominal point and the others with margins in [2.6, 3.5]."""
    rng = np.random.default_rng(seed)
    inst = make_instance(seed, T=T, N=4, E=4, lateral=(0.3, 3.5))
    ang = rng.uniform(-np.pi, np.pi, (N, T))
    margin = rng.uniform(2.6, 3.5, (N, T))
    for t in range(T):
        margin[rng.permutation(N)[:NEAR], t] = rng.uniform(-0.5, 1.0, NEAR)
    return {'nom_s': _f32(inst['nom_s']), 'nom_u': _f32(inst['nom_u']), 'ref': _f32(inst['ref']),
            'vref': float(np.float32(inst['ref_speed'])), 'dis': _f32(rng.uniform(0.1, 1.0, T)),
            'pref': _f32(inst['nom_s'][0:2, 1:] + rng.normal(0, 0.05, (2, T))),
            'hx': _f32(np.cos(ang)), 'hy': _f32(np.sin(ang)), 'hc': _f32(margin),
            'gx': _f32(rng.normal(0, 0.3, (N, T))), 'gy': _f32(rng.normal(0, 0.3, (N, T)))}


def _oracle(p, acc):
    """OracleRDA whose su-QP has exactly the kernel's hinge rows: lam'A = (hx, hy), lam'b = lam'A pref - hc, mu = z =
    zeta = 0, xi = (gx, gy)."""
    o = OracleRDA(T, rectangle_robot(), max_edge_num=4, max_obs_num=N, accelerated=acc)
    o.assign_state_parameter(p['nom_s'], p['nom_u'], p['dis'])
    o.ref_s, o.ref_speed = p['ref'], p['vref']
    o.para_obsA_lam[:, 1:, 0], o.para_obsA_lam[:, 1:, 1] = p['hx'], p['hy']
    o.para_obsb_lam[:, 1:] = p['hx'] * p['pref'][0] + p['hy'] * p['pref'][1] - p['hc']
    o.para_xi[:, 1:, 0], o.para_xi[:, 1:, 1] = p['gx'], p['gy']
    return o


def _kept_per_stage(o, p):
    """Hinges the pruning rule keeps at every stage, evaluated on the rollout of the linearised model the core starts from."""
    s = o.para_s[:, 0].copy()
    kept = []
    for t in range(T):
        A, B, C = o.lin[t]
        s = A @ s + B @ o.para_u[:, t] + C
        lp = p['hx'][:, t] * (s[0] - p['pref'][0, t]) + p['hy'][:, t] * (s[1] - p['pref'][1, t]) + p['hc'][:, t]
        kept.append(int(((lp - DMAX <= PRUNE) | (lp <= np.sort(lp)[1])).sum()))
    return kept


@pytest.mark.parametrize('accelerated', [1, 0])
@pytest.mark.parametrize('seed', [61, 62])
def test_su_core_with_more_than_32_hinges_matches_dense_oracle(accelerated, seed):
    p = _problem(seed)
    o = _oracle(p, bool(accelerated))
    if accelerated:
        kept = _kept_per_stage(o, p)
        assert min(kept) > 32 and max(kept) < N, kept
    s_o, u_o, d_o, info = o.su_prob_solve()
    assert info['status'] in ('optimal', 'optimal_inaccurate'), info['status']
    P = shim.SuParams(T=T, N=N, dynamics=shim.DYN['acker'], accelerated=accelerated, dt=0.1, L=3.0,
                      umax=(shim.C.c_float * 2)(10, 1), ab=(shim.C.c_float * 2)(1.0, 0.05), ws=1, wu=1, slack_gain=8,
                      dmin=0.1, dmax=DMAX, ro1=200, ro2=1, max_iter=40, mu0=1.0, prune=PRUNE)
    for prec, tol in (('d', 2e-5), ('f', 1e-3)):
        s, u, d, st, it = shim.su(P, o.para_s, o.para_u, o.ref_s, o.ref_speed, o.para_dis, p['hx'], p['hy'], p['hc'],
                                  p['gx'], p['gy'], p['pref'], prec=prec)
        assert st == 0 and it < 40, (prec, st, it)
        np.testing.assert_allclose(s, s_o, atol=tol)
        np.testing.assert_allclose(u, u_o, atol=tol)
        np.testing.assert_allclose(d, d_o.ravel(), atol=tol)
