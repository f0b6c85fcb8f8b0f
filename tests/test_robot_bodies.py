"""Polygon robot bodies other than the rear-axle rectangle (tests/golden/make_oracle_fixture_bodies.py: centred boxes of the
diff-drive and omni examples, triangles, pentagon / hexagon / octagon, bodies whose reference point lies outside them) on the
g++ build of the kernels' cores: the (lam, mu, z) cell cores against the generic solver in the reference's original variables,
the coherent first pass at R = 3 and with outside reference points, and whole solves of the CPU port against committed float64
oracle traces, with and without the emulated coherent pipeline."""
import importlib.util
import os

import numpy as np
import pytest
from scipy.optimize import minimize

import shim
from oracle import cpu_port
from oracle.cell_generic import solve_cell_generic, cell_objective
from rda_planner_b200.mpc import polygon_halfspaces
from rda_planner_b200.rda_solver import canonical_polygon_rows, pack_obstacles
from test_cells_vs_generic import TOL, OBJ_TOL, _random_cell

HERE = os.path.dirname(os.path.abspath(__file__))
TRAJ_TOL, RESI_RTOL = 1e-3, 2e-3          # as tests/test_gpu_parity.py (<= 6 ADMM iterations)


def _gen():
    spec = importlib.util.spec_from_file_location('make_bodies', os.path.join(HERE, 'golden', 'make_oracle_fixture_bodies.py'))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


BODIES = _gen()
NAMES = list(BODIES.BODIES)


def _refine(A, b, circ, G, h, p, phi, dbar, zeta, xi, ro2, points):
    """Referee of an ACTIVE cell (z = 0) where the core and the generic solve disagree: the reference objective minimised
    again in float64 from each given (lam, mu), SLSQP at ftol 1e-16, every candidate (the given points included) projected
    onto the feasible set first (lam >= 0 or -lam in the cone, mu >= 0, |A'lam| <= 1).  Returns (f*, x*, |grad f(x*)|)."""
    E = A.shape[0]
    b = b.ravel()
    f = lambda x: cell_objective(A, b, G, h, p, phi, dbar, zeta, xi, ro2, x[:E], x[E:], 0.0)
    live = np.linalg.norm(A, axis=1) > 0
    bounds = [(None, None) if circ and i < 3 else ((0, None) if live[i] and not circ else (0, 0)) for i in range(E)]
    bounds += [(0, None)] * G.shape[0]
    cons = [{'type': 'ineq', 'fun': lambda x: 1.0 - np.sum((A.T @ x[:E]) ** 2)}]
    if circ:
        cons.append({'type': 'ineq', 'fun': lambda x: -x[2] - np.hypot(x[0], x[1])})

    def feasible(x):
        x = x.copy()
        x[E:] = np.maximum(x[E:], 0.0)
        if circ:
            x[2] = min(x[2], -np.hypot(x[0], x[1]))
        else:
            x[:E] = np.maximum(x[:E], 0.0)
        n = np.linalg.norm(A.T @ x[:E])
        if n > 1:
            x[:E] /= n
        return x
    cands = []
    for x0 in points:
        cands.append(feasible(x0))
        r = minimize(f, x0, bounds=bounds, constraints=cons, method='SLSQP', options={'ftol': 1e-16, 'maxiter': 2000})
        cands.append(feasible(r.x))
    x = min(cands, key=f)
    eps = 1e-7
    grad = np.array([(f(x + eps * e) - f(x - eps * e)) / (2 * eps) for e in np.eye(len(x))])
    return f(x), x, np.linalg.norm(grad)


def _cell_case(k, rng):
    kind = 'circle' if k % 5 == 4 else 'polygon'
    return kind, _random_cell(rng, k, kind)


@pytest.mark.parametrize('name', NAMES)
def test_cell_cores_equal_generic_solver_for_every_body(name):
    """shim.cell in float64 / float32 and the lean first passes (<4,4> with padded robot rows when R < 4, <8,8>) on far, near /
    active, overlapping and tilted (xi != 0) cells, polygon (3-4 rows) and disc obstacles.  Where the core and the generic solve
    disagree beyond the tolerances of test_cells_vs_generic.py, a refined float64 solve of the same cell decides: the core must
    be within TOL of the refined optimum, and its objective above it by no more than OBJ_TOL plus what its point error explains
    to first order.  Measured over the nine bodies (60 cells each): every disagreement is on an active cell; where the points
    differ by up to 8e-6 (overlap and disc cells of the outside-reference bodies) the generic solve is the one away from the
    refined optimum, and where the float64 core's objective is up to 1.6e-8 above (edge-contact closed forms of the triangles,
    whose root is resolved to a tangential residual of 1e-9) its point is within 2e-8 of the refined one."""
    car = BODIES.body(name)
    G, h = np.asarray(car.G, float), np.asarray(car.h, float).ravel()
    R = G.shape[0]
    rng = np.random.default_rng(sum(map(ord, name)))
    n = 60
    seen = {'active': 0, 'inactive': 0, 'tilted': 0, 'paths': set(), 'refereed': 0, 'lean4': 0, 'lean8': 0}
    worst = {}
    for k in range(n):
        kind, (A, b, p, phi, dbar, zeta, xi, ro2) = _cell_case(k, rng)
        circ = kind == 'circle'
        r = solve_cell_generic(A, b, circ, G, h, p, phi, dbar, zeta, xi, ro2)
        fo = cell_objective(A, b.ravel(), G, h, p, phi, dbar, zeta, xi, ro2, r['lam'], r['mu'], r['z'])
        seen['active' if r['active'] else 'inactive'] += 1
        seen['tilted'] += bool(np.any(xi != 0))
        ref = None
        for prec in ('d', 'f', 'lean4', 'lean8'):
            if prec == 'lean4' and R > 4:
                continue
            kk = shim.cell(G, h, int(circ), A, b, p, phi, dbar, zeta, xi, ro2, prec=prec)
            if prec.startswith('lean'):
                if kk['path'] == 6:                      # declined: the searched pass takes the cell
                    continue
                seen[prec] += 1
                assert not r['active'] and not np.any(xi != 0), (k, prec)
            else:
                assert kk['path'] != 5, (k, prec)
                seen['paths'].add(kk['path'])
            tol, otol = (TOL['f'], OBJ_TOL['f']) if prec != 'd' else (TOL['d'], OBJ_TOL['d'])
            lam, mu = kk['lam'][:A.shape[0]], kk['mu'][:R]
            fk = cell_objective(A, b.ravel(), G, h, p, phi, dbar, zeta, xi, ro2, lam, mu, kk['z'])
            gap = max(np.abs(lam - r['lam']).max(), np.abs(mu - r['mu']).max(), abs(kk['z'] - r['z']))
            if gap >= tol or fk - fo >= otol * (1 + fo):
                assert r['active'], (k, prec, gap, fk - fo)        # inactive cells: closed-form tie-break, no referee
                if ref is None:
                    ref = _refine(A, b, circ, G, h, p, phi, dbar, zeta, xi, ro2,
                                  [np.concatenate([r['lam'], r['mu']]), np.concatenate([lam, mu])])
                    seen['refereed'] += 1
                fs, xs, gn = ref
                dk = np.abs(np.concatenate([lam, mu]) - xs).max()
                assert dk < tol, (k, prec, 'core away from the refined optimum', dk, gap)
                assert fk - fs < otol * (1 + fs) + gn * dk * np.sqrt(len(xs)), (k, prec, fk - fs, dk)
                gap = dk
            worst[prec] = max(worst.get(prec, 0.0), gap)
            if circ:
                assert np.hypot(lam[0], lam[1]) <= -lam[2] + 1e-6 and np.hypot(lam[0], lam[1]) <= 1 + 1e-5
            else:
                assert (lam >= -1e-7).all() and np.linalg.norm(A.T @ lam) <= 1 + 1e-5
            assert (mu >= -1e-7).all() and kk['z'] >= 0
    print(f'\n{name} (R = {R}): largest (lam, mu, z) gap to the float64 reference per core {worst}; cells {seen}')
    assert seen['active'] > n // 6 and seen['inactive'] > n // 5 and seen['tilted'] > n // 4 and len(seen['paths']) >= 2
    assert seen['lean8'] > n // 6 and (R > 4 or seen['lean4'] > n // 6)


def _lean2_cases(G, h, seed, count):
    rng = np.random.default_rng(seed)
    made = 0
    while made < count:
        n = int(rng.integers(3, 5))
        c = rng.uniform(20, 50, 2)
        ang = np.sort(rng.uniform(0, 2 * np.pi, n))
        if np.min(np.diff(np.concatenate([ang, [ang[0] + 2 * np.pi]]))) < 0.3:
            continue
        V = c[:, None] + rng.uniform(0.5, 2.5) * np.vstack([np.cos(ang), np.sin(ang)])
        A, b = canonical_polygon_rows(*polygon_halfspaces(V))
        A4 = np.zeros((4, 2)); b4 = np.zeros(4); A4[:n] = A; b4[:n] = b
        a = rng.uniform(0, 2 * np.pi)
        p = c + rng.uniform(3, 9) * np.array([np.cos(a), np.sin(a)])
        phi = rng.uniform(-3.1, 3.1)
        dbar, zeta = rng.uniform(0.1, 1.0), rng.uniform(-0.2, 0.2)
        r0 = shim.cell(G, h, 0, A4, b4, p, phi, dbar, zeta, (0, 0), 1.0, prec='lean4')
        feat = int(r0['hm0'])
        if r0['path'] != 0 or not feat & 0x40:
            continue
        scale = rng.choice([0.01, 0.05, 0.3, 1.5])
        made += 1
        yield A4, b4, n, feat, p + rng.normal(0, scale, 2), phi + rng.normal(0, 0.3 * scale), dbar, zeta, rng


@pytest.mark.parametrize('name', ['triangle', 'triangle_out', 'offset_box'])
def test_coherent_pass_with_three_rows_and_outside_reference_points(name):
    """cell_lean2<4,4> (the coherent pass k_cells_coh runs for R <= 4) with the cached feature pair, a wrong pair and invalid
    bytes: it matches the float64 core or declines, never accepts a wrong pair with a wrong answer, and always declines a
    robot vertex index jb in R..7."""
    car = BODIES.body(name)
    G, h = canonical_polygon_rows(car.G, car.h)
    R = G.shape[0]
    keys = ('z', 'zeta_new', 'ax', 'ay', 'c0', 'gx', 'gy')
    hit = miss = wrong_acc = 0
    worst = 0.0
    for A4, b4, n, feat, p1, phi1, dbar, zeta, rng in _lean2_cases(G, h, 40 + R, 300):
        truth = shim.cell(G, h, 0, A4, b4, p1, phi1, dbar, zeta, (0, 0), 1.0, prec='d')
        for f in (feat, 0x40 | (int(rng.integers(0, n)) << 3) | int(rng.integers(0, R))):
            r = shim.cell_lean2(G, h, A4, b4, f, p1, phi1, dbar, zeta)
            if f == feat:
                hit += r['path'] != 6
                miss += r['path'] == 6
            if r['path'] == 6:
                continue
            wrong_acc += f != feat
            assert r['feat'] & 0x40 and truth['path'] == 0
            assert r['feat'] & 7 < R
            gap = max(abs(r[k] - truth[k]) for k in keys)
            worst = max(worst, gap)
            assert gap < 5e-5, (name, f, gap)
            np.testing.assert_allclose(r['lam'], truth['lam'][:4], atol=2e-5 * (1 + np.abs(truth['lam']).max()))
            np.testing.assert_allclose(r['mu'][:R], truth['mu'], atol=2e-5 * (1 + np.abs(truth['mu']).max()))
            assert np.all(r['mu'][R:] == 0)
        for jb in range(R, 8):                          # robot vertex beyond the body: always declined
            assert shim.cell_lean2(G, h, A4, b4, 0x40 | (feat & 0x38) | jb, p1, phi1, dbar, zeta)['path'] == 6
    print(f'\n{name} (R = {R}): cached pair accepted {hit}, declined {miss}, wrong pairs accepted (correctly) {wrong_acc}; '
          f'largest gap to the float64 core {worst:.1e}')
    assert hit > 5 * miss and wrong_acc > 0


def _inputs(name):
    car, inst = BODIES.instance(name)
    T, N = BODIES.T, BODIES.N
    A, b, kd, count, tv = pack_obstacles(list(inst['obstacles']), T, N, 4)
    return car, dict(nom_s=inst['nom_s'][None], nom_u=inst['nom_u'][None], ref_s=inst['ref'][None],
                     ref_speed=[inst['ref_speed']], obs_A=A[None], obs_b=b[None], obs_kind=kd[None], obs_count=[count]), tv


@pytest.mark.parametrize('lean2', ['0', '1'])
def test_port_matches_committed_oracle_traces_for_every_body(monkeypatch, lean2):
    """Every ADMM iteration of the first (cold) call in tests/golden/oracle_bodies.npz against the CPU port, which always starts
    cold; RDA_PORT_LEAN2=1 emulates the coherent pipeline where the library runs it (E <= 4, R <= 4, static polygons)."""
    monkeypatch.setenv('RDA_PORT_LEAN2', lean2)
    z = np.load(os.path.join(HERE, 'golden', 'oracle_bodies.npz'))
    hits = {}
    for name in NAMES:
        car, inp, tv = _inputs(name)
        worst = [0.0, 0.0]
        for it in range(1, BODIES.ITERS + 1):
            r = cpu_port.solve_batch(car, BODIES.T, BODIES.N, 4, time_varying=tv, iter_num=it, threads=1, **inp)
            assert r['cell_failures'][0, 0] == 0
            ds = np.abs(r['s'][0] - z[f'{name}_c0_s'][it - 1]).max()
            du = np.abs(r['u'][0] - z[f'{name}_c0_u'][it - 1]).max()
            worst = [max(worst[0], ds), max(worst[1], du)]
            assert ds < TRAJ_TOL and du < TRAJ_TOL, (name, it, ds, du)
            for k in ('resi_pri', 'resi_dual'):
                ref = z[f'{name}_c0_{k}'][it - 1]
                assert abs(float(r[k][0]) - ref) <= RESI_RTOL * (1 + ref), (name, it, k)
        hits[name] = int(r['cell_failures'][0, 1]) if lean2 == '1' else 0
        print(f'\n{name}: largest gap to the oracle, states {worst[0]:.1e}, controls {worst[1]:.1e}'
              + (f'; cells resolved by the coherent pass in the last solve {hits[name]}' if lean2 == '1' else ''))
    if lean2 == '1':
        for name in NAMES:
            R = np.asarray(BODIES.body(name).G).shape[0]
            static = BODIES.CASES[name][1] != 'moving'
            assert (hits[name] > 0) == (R <= 4 and static), (name, hits[name])
