"""Plan clearance (rda_plan_clearance) without a GPU: the float64 reference oracle/clearance.py against known answers and
against independent solvers, and the g++ build of the kernel's cell core (plan_clearance.cuh) against the reference on
random cells of every body of the body fixture family."""
import numpy as np
import pytest
from scipy.optimize import minimize

import clearance_cases as cc
import clearance_twin
from oracle import clearance as ref
from rda_planner_b200 import _cabi
from rda_planner_b200.mpc import polygon_halfspaces
from rda_planner_b200.rda_solver import robot_body
from rda_planner_b200.scenarios import disc_robot, rectangle_robot

E = 4


def _box(x0, x1, y0, y1):
    A, b = polygon_halfspaces(np.array([[x0, x1, x1, x0], [y0, y0, y1, y1]]))
    return A, b.ravel()


def _rect():
    G, h, _ = robot_body(rectangle_robot())
    return ref.body_from_halfspaces(G, h), G, h


def _disc(x, y, r):
    return np.array([[1.0, 0], [0, 1.0], [0, 0]]), np.array([x, y, -r])


def _support(V, w):
    return np.max(V @ w)


def _by_directions(P, Q, qr=0.0, pr=0.0):
    """The definition maximised over 3600 directions, then refined around the best one: P, Q vertex arrays (or a single
    centre with radius pr / qr)."""
    f = lambda a: (-_support(P, -np.array([np.cos(a), np.sin(a)])) - pr
                   - _support(Q, np.array([np.cos(a), np.sin(a)])) - qr)
    ang = np.linspace(-np.pi, np.pi, 3600, endpoint=False)
    a0 = ang[np.argmax([f(a) for a in ang])]
    lo, hi = a0 - 2e-3, a0 + 2e-3           # golden-section search: the maximum sits on a kink, where Brent's steps stall
    g = (np.sqrt(5.0) - 1) / 2
    for _ in range(80):
        a, b = hi - g * (hi - lo), lo + g * (hi - lo)
        if f(a) < f(b):
            lo = a
        else:
            hi = b
    return max(f(a0), f(0.5 * (lo + hi)))


def test_box_to_box_gap():
    body, _, _ = _rect()
    A, b = _box(6.0, 8.0, -1.0, 1.0)
    # the rear-axle rectangle spans x in [-0.8, 3.8]: gap 6.0 - 3.8 (tests/test_oracle.py)
    assert abs(ref.cell(body, [0, 0, 0], 0, A, b) - (6.0 - np.float32(3.8))) < 1e-7


def test_disc_to_box():
    body, _, _ = _rect()
    A, b = _disc(7.0, 0.0, 1.5)
    assert abs(ref.cell(body, [0, 0, 0], 1, A, b) - (7.0 - 1.5 - np.float32(3.8))) < 1e-7
    # a disc body against a box, and against a disc
    G, h, _ = robot_body(disc_robot(radius=0.5, center=(1.0, 0.0)))
    d = ref.body_from_halfspaces(G, h, disc=True)
    A, b = _box(3.0, 4.0, -1.0, 1.0)
    assert abs(ref.cell(d, [0, 0, 0], 0, A, b) - 1.5) < 1e-12
    A, b = _disc(1.0, 3.0, 1.0)
    assert abs(ref.cell(d, [0, 0, 0], 1, A, b) - 1.5) < 1e-12
    # heading pi / 2 turns the off-centre disc to (0, 1): sqrt(5) from the obstacle's centre (1, 3)
    assert abs(ref.cell(d, [0, 0, np.pi / 2], 1, A, b) - (np.sqrt(5.0) - 0.5 - 1.0)) < 1e-6


def test_containment():
    body, _, _ = _rect()
    V = body['V']
    x0, x1, y0, y1 = V[:, 0].min(), V[:, 0].max(), V[:, 1].min(), V[:, 1].max()
    # body inside a 20 x 20 box: the cheapest way out is through the nearest side
    A, b = _box(-10, 10, -10, 10)
    want = max(x0 - 10, -x1 - 10, y0 - 10, -y1 - 10)
    assert abs(ref.cell(body, [0, 0, 0], 0, A, b) - want) < 1e-7          # rows rounded to float32
    # a small box inside the body: pushed out through the nearest body side
    A, b = _box(1.0, 2.0, -0.2, 0.2)
    want = max(x0 - 2.0, 1.0 - x1, y0 - 0.2, -0.2 - y1)
    assert abs(ref.cell(body, [0, 0, 0], 0, A, b) - want) < 1e-7          # rows rounded to float32
    # both against the definition
    for A, b in (_box(-10, 10, -10, 10), _box(1.0, 2.0, -0.2, 0.2)):
        Q = ref.obstacle_polygon(A, b)[0]
        assert abs(ref.cell(body, [0, 0, 0], 0, A, b) - _by_directions(V, Q)) < 1e-9


def test_touching_sets_give_zero():
    body, _, _ = _rect()
    x1 = body['V'][:, 0].max()
    A, b = _box(float(x1), float(x1) + 2.0, -0.5, 0.5)
    assert abs(ref.cell(body, [0, 0, 0], 0, A, b)) < 1e-12
    c = np.float32(x1 + 1.25)
    A, b = _disc(float(c), 0.0, float(c) - float(x1))           # both float32 exactly (the kernels' inputs)
    assert abs(ref.cell(body, [0, 0, 0], 1, A, b)) < 1e-12


def _world_sets(car, kind, A, b, pose):
    G, h, cone = cc.body_rows(car)
    body = ref.body_from_halfspaces(G, h, cone == _cabi.ROBOT_DISC)
    x, y, th = (float(v) for v in pose)
    Rm = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
    if body['disc']:
        P, pr = (np.array([x, y]) + Rm @ body['c'])[None, :], body['r']
    else:
        P, pr = np.array([x, y]) + body['V'] @ Rm.T, 0.0
    if kind == _cabi.OBS_CIRCLE:
        Q, qr = np.asarray(b, float)[None, :2], -float(b[2])
    else:
        Q, qr = ref.obstacle_polygon(A, b)[0], 0.0
    return body, P, pr, Q, qr


def test_reference_against_independent_solvers():
    """Separated pairs: min |x - y| over the points of both sets (SLSQP); overlapping pairs: the definition maximised
    over sampled directions."""
    rng = np.random.default_rng(5)
    seen = {'sep': 0, 'ovl': 0}
    for name, car in cc.bodies().items():
        kinds, A, b, pose, _ = cc.random_cells(rng, car, 16)
        for k in range(len(kinds)):
            body, P, pr, Q, qr = _world_sets(car, kinds[k], A[k], b[k], pose[k])
            d = ref.cell(body, pose[k], kinds[k], A[k], b[k])
            if d > 1e-3:
                seen['sep'] += 1
                # a point of each set: a convex combination of a polygon's vertices, or centre + radius * u, |u| <= 1
                def point(X, rad, z):
                    return z @ X if len(X) > 1 else X[0] + rad * z
                nP, nQ = (len(P) if len(P) > 1 else 2), (len(Q) if len(Q) > 1 else 2)
                cons, bounds = [], []
                for X, n_, off in ((P, nP, 0), (Q, nQ, nP)):
                    sl = slice(off, off + n_)
                    if len(X) > 1:
                        cons.append({'type': 'eq', 'fun': lambda z, sl=sl: np.sum(z[sl]) - 1.0})
                        bounds += [(0.0, 1.0)] * n_
                    else:
                        cons.append({'type': 'ineq', 'fun': lambda z, sl=sl: 1.0 - np.sum(z[sl] ** 2)})
                        bounds += [(-1.0, 1.0)] * 2
                gap = lambda z: point(P, pr, z[:nP]) - point(Q, qr, z[nP:])
                feasible = lambda z: all(abs(c['fun'](z)) < 1e-7 if c['type'] == 'eq' else c['fun'](z) > -1e-7 for c in cons)
                best = np.inf
                for start in range(4):                 # the best feasible result of a few starts
                    w = rng.dirichlet(np.ones(nP + nQ)) if start else np.ones(nP + nQ)
                    z0 = np.r_[w[:nP] / w[:nP].sum() if len(P) > 1 else np.zeros(2),
                               w[nP:] / w[nP:].sum() if len(Q) > 1 else np.zeros(2)]
                    r = minimize(lambda z: gap(z) @ gap(z), z0, constraints=cons, bounds=bounds, method='SLSQP',
                                 options={'ftol': 1e-14, 'maxiter': 1000})
                    if feasible(r.x):
                        best = min(best, np.sqrt(r.fun))
                # a feasible pair is never closer than the distance, and the best one found comes within 1e-5
                assert -1e-5 <= best - d < 1e-5 * max(1.0, d), (name, k, best, d)      # constraints met to 1e-7 at 60 m
            elif d < -1e-3:
                seen['ovl'] += 1
                # no direction does better than the reference, and the best sampled one comes within 1e-7
                sampled = _by_directions(P, Q, qr, pr)
                assert -1e-12 <= d - sampled < 1e-7, (name, k, d, sampled)
    assert seen['sep'] > 50 and seen['ovl'] > 30, seen


@pytest.mark.parametrize('name', list(cc.bodies()))
def test_core_matches_reference(name):
    """The g++ build of the kernel's cell core against the float64 reference, to 1e-9 (both take the float32 inputs and
    the body as the kernels hold it)."""
    car = cc.bodies()[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    kinds, A, b, pose, target = cc.random_cells(rng, car, 320)
    G, h, cone = cc.body_rows(car)
    got = clearance_twin.cells(G, h, cone, kinds, A, b, pose)
    body = ref.body_from_halfspaces(G, h, cone == _cabi.ROBOT_DISC)
    want = np.array([ref.cell(body, pose[k], kinds[k], A[k], b[k]) for k in range(len(kinds))])
    err = np.abs(got - want) / np.maximum(1.0, np.abs(want))
    assert err.max() < 1e-9, (err.max(), int(err.argmax()))
    # what the cells cover
    assert (want > 20).any() and ((want > 0) & (want < 1e-3)).sum() >= 5
    assert ((want < 0) & (want > -0.05)).sum() >= 10 and (want < -0.3).sum() >= 10
    assert (np.abs(pose[:, :2]) > 55).all() and pose[:, 2].min() < -2.5 and pose[:, 2].max() > 2.5
    assert (kinds == _cabi.OBS_CIRCLE).any()
    rows = (np.linalg.norm(A, axis=2) > 0).sum(1)[kinds == _cabi.OBS_POLYGON]
    assert set(range(3, 9)) <= set(rows.tolist())
