"""su-QP problems with their inputs set directly, shared by the tests of the CPU build of the su-QP core
(tests/test_su_restarts.py) and of the device kernels (tests/test_gpu_su_qp.py), and by the fixture generator
tests/golden/make_oracle_fixture_su.py.

A problem is what k_su reads for one instance: the nominal (cur_s, cur_u: linearisation point and start of the
rollout), the reference (ref_s, ref_speed), the initial safety distances (dis), the positions the hinge offsets refer
to (pref) and the hinge inputs coef = (a_x, a_y, c0, g_x, g_y), [5][N][T].  Every value is rounded to float32 first,
as the device buffers hold them, so that the CPU build, the oracle and the kernels solve the same problem."""
import numpy as np

import shim
from oracle.rda_oracle import OracleRDA
from rda_planner_b200.scenarios import rectangle_robot, make_instance

PRUNE = 0.5                          # the library's default hinge pruning margin (rda_create)
TUN = dict(slack_gain=8.0, max_sd=1.0, min_sd=0.1, ro1=200.0, ro2=1.0, wu=1.0)
TUN_C = dict(TUN, min_sd=0.5, wu=0.2)          # config C's tunables
TUN_D = dict(TUN, slack_gain=13.0)             # config D's tunables


def _f32(a):
    return np.asarray(a, np.float32).astype(float)


def problem(seed, T, N, dyn='acker', near=None, v_nom=None, near_margin=(-0.5, 1.0)):
    """Nominal trajectory of a generated instance and N hinge rows per stage with unit normals: `near` of them (a random
    set per stage, default min(N, 3)) with margins in `near_margin` at the nominal point, the others in [2.6, 3.5] (far
    from activity: left out by the pruning).  v_nom below the reference speed moves the optimum away from the nominal."""
    rng = np.random.default_rng(seed)
    inst = make_instance(seed, T=T, N=4, E=4, dynamics=dyn, lateral=(0.3, 3.5), v_nom=v_nom)
    near = min(N, 3) if near is None else near
    ang = rng.uniform(-np.pi, np.pi, (N, T))
    margin = rng.uniform(2.6, 3.5, (N, T))
    for t in range(T):
        margin[rng.permutation(N)[:near], t] = rng.uniform(*near_margin, near)
    coef = np.stack([np.cos(ang), np.sin(ang), margin, rng.normal(0, 0.3, (N, T)), rng.normal(0, 0.3, (N, T))])
    return {'T': T, 'N': N, 'dyn': dyn, 'cur_s': _f32(inst['nom_s']), 'cur_u': _f32(inst['nom_u']),
            'ref_s': _f32(inst['ref']), 'vref': float(np.float32(inst['ref_speed'])), 'dis': _f32(rng.uniform(0.1, 1.0, T)),
            'pref': _f32(inst['nom_s'][0:2, 1:] + rng.normal(0, 0.05, (2, T))), 'coef': _f32(coef)}


def params(T, N, dyn='acker', acc=1, prune=PRUNE, tun=TUN, max_iter=40):
    """The SuParams the library builds (su_params in rda_kernels.cu) for rectangle_robot(dyn) at step time 0.1."""
    car = rectangle_robot(dynamics=dyn)
    ab = [np.float32(a * 0.1) for a in car.max_acce]
    return shim.SuParams(T=T, N=N, dynamics=shim.DYN[dyn], accelerated=acc, dt=0.1, L=car.wheelbase,
                         umax=(shim.C.c_float * 2)(*car.max_speed), ab=(shim.C.c_float * 2)(*ab), ws=1, wu=tun['wu'],
                         slack_gain=tun['slack_gain'], dmin=tun['min_sd'], dmax=tun['max_sd'], ro1=tun['ro1'],
                         ro2=tun['ro2'], max_iter=max_iter, mu0=1.0, prune=prune)


def cpu(p, P, prec='d'):
    """The CPU build of su_solver.cuh: (s, u, d, status, iterations, report) as shim.su."""
    return shim.su(P, p['cur_s'], p['cur_u'], p['ref_s'], p['vref'], p['dis'], *p['coef'], p['pref'], prec=prec, report=True)


def oracle(p, acc=True, tun=TUN):
    """OracleRDA whose su-QP has exactly the kernel's hinge rows: lam'A = (a_x, a_y), lam'b = lam'A pref - c0,
    mu = z = zeta = 0, xi = (g_x, g_y)."""
    T, N = p['T'], p['N']
    o = OracleRDA(T, rectangle_robot(dynamics=p['dyn']), max_edge_num=4, max_obs_num=N, accelerated=acc,
                  **{k: tun[k] for k in ('slack_gain', 'max_sd', 'min_sd', 'ro1', 'ro2', 'wu')})
    o.assign_state_parameter(p['cur_s'], p['cur_u'], p['dis'][None, :])
    o.ref_s, o.ref_speed = p['ref_s'], p['vref']
    hx, hy, hc, gx, gy = p['coef']
    if N:
        o.para_obsA_lam[:, 1:, 0], o.para_obsA_lam[:, 1:, 1] = hx, hy
        o.para_obsb_lam[:, 1:] = hx * p['pref'][0] + hy * p['pref'][1] - hc
        o.para_xi[:, 1:, 0], o.para_xi[:, 1:, 1] = gx, gy
    return o


def rollout(p, P):
    """Positions [2][T] of the linearised model's rollout from the nominal: where the pruning rule evaluates the hinges."""
    s = cpu(p, _no_iter(P))[0]
    return s[0:2, 1:]


def _no_iter(P):
    Q = shim.SuParams.from_buffer_copy(P)
    Q.max_iter = 0
    return Q


def left_out(p, pos, t, o, prune=PRUNE, dmax=1.0):
    """Whether the pruning rule leaves hinge o of stage t out of the interior point iteration at rollout positions pos."""
    hx, hy, hc = p['coef'][0:3, :, t]
    lp = hx * (pos[0, t] - p['pref'][0, t]) + hy * (pos[1, t] - p['pref'][1, t]) + hc
    return bool(lp[o] - dmax > prune and lp[o] > np.sort(lp)[1])


def plant(p, P, cells):
    """Hinges left out at the nominal rollout but violated at the pruned optimum.  For every (t, o) in `cells` hinge o of
    stage t is replaced by a row whose normal points against the move of stage t from the rollout to the optimum of the
    problem without it, placed 0.02 beyond the pruning margin at the rollout.  Returns the new problem and, per cell, the
    planted hinge's value l at that optimum (negative where the move is longer than the margin)."""
    q = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in p.items()}
    pos = rollout(q, P)
    s, _, d, st, _, rep = cpu(q, P)
    assert st == 0 and rep['restarts'] == 0, ('the base problem must not repeat its pruned solve', st, rep)
    for t, o in cells:
        mv = s[0:2, t + 1] - pos[:, t]
        a = -mv / np.linalg.norm(mv)
        a = _f32(a / np.linalg.norm(a))
        dpos = pos[:, t] - q['pref'][:, t]
        hc = P.dmax + P.prune + 0.02 - float(a @ dpos)
        q['coef'][0, o, t], q['coef'][1, o, t], q['coef'][2, o, t] = a[0], a[1], np.float32(hc)
        q['coef'][3:5, o, t] = 0.0
        assert left_out(q, pos, t, o, P.prune, P.dmax), (t, o)
    hx, hy, hc = q['coef'][0:3]
    lv = [float(hx[o, t] * (s[0, t + 1] - q['pref'][0, t]) + hy[o, t] * (s[1, t + 1] - q['pref'][1, t]) + hc[o, t] - d[t])
          for t, o in cells]
    return q, lv


# Problems whose pruned solve must be repeated, per (T, N): (seed, planted (t, o) cells).  Together they leave out and
# violate a hinge at o < 32 and at o >= 32 (both sides of the mask word boundary at one stage too), at a stage t >= 32,
# and at exactly one stage; an instance without planted hinges completes each batch.
RESTARTS = {
    (12, 40): [(102, [(11, 5)]), (104, [(11, 35), (10, 38)]), (104, [(11, 31), (11, 32)]), (103, [])],
    (40, 5): [(100, [(39, 4)]), (101, [(39, 4)]), (102, [])],
    (33, 33): [(101, [(32, 32)]), (103, [(32, 32)]), (104, [])],
}


def restart_problem(T, N, seed, cells, tun=TUN):
    """A restart problem of RESTARTS: the optimum moves far from the nominal (nominal speed 0.5, reference speed 4,
    hinges near activity with margins in [0.8, 1.4]); with no cells the problem itself, which converges unrepeated."""
    p = problem(seed, T, N, v_nom=0.5, near_margin=(0.8, 1.4))
    return plant(p, params(T, N, tun=tun), cells)[0] if cells else p

# (T, N, seed) of a restart_problem (no planted hinge) whose pruned attempt stops at its iteration cap of 24 and is
# repeated with all hinges: the one such problem among 1 800 generated ones (300 per family of six).
CAPPED = (30, 20, 50244)
