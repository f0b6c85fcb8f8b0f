"""Random (body, pose, obstacle) cells for the plan clearance tests (test infrastructure only): the polygon bodies of
tests/golden/make_oracle_fixture_bodies.py and centred / off-centre discs; obstacles of 3..8 rows, discs, and
canonicalised walls and wedges; separations from 50 m down to 1e-4 m, shallow and deep overlaps and containment;
poses at 60 m coordinates with headings across +-pi.  Obstacles are placed by bisection of their offset along a random
direction on the g++ build of the core (clearance_twin), so that the separations land where they are asked for."""
import importlib.util
import os

import numpy as np

import clearance_twin
from rda_planner_b200 import _cabi
from rda_planner_b200.mpc import polygon_halfspaces
from rda_planner_b200.rda_solver import canonical_polygon_rows, robot_body
from rda_planner_b200.scenarios import disc_robot

HERE = os.path.dirname(os.path.abspath(__file__))
E = 8


def _fixture():
    spec = importlib.util.spec_from_file_location('make_bodies', os.path.join(HERE, 'golden', 'make_oracle_fixture_bodies.py'))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def bodies():
    """name -> car_tuple: every body of the body fixture family, a centred and an off-centre disc."""
    fx = _fixture()
    out = {name: fx.body(name) for name in fx.BODIES}
    out['disc_centred'] = disc_robot(radius=0.9)
    out['disc_offset'] = disc_robot(radius=0.7, center=(1.2, -0.3))
    return out


def body_rows(car):
    """(G, h, cone) as the kernels take them."""
    G, h, cone = robot_body(car)
    return G, h, cone


def _shape(rng, style):
    """Obstacle rows (kind, A [E, 2], b [E]) around the origin, which lies inside it."""
    A = np.zeros((E, 2))
    b = np.zeros(E)
    if style == 'disc':
        A[:3] = [[1, 0], [0, 1], [0, 0]]
        b[:3] = [0.0, 0.0, -rng.uniform(0.2, 2.0)]
        return _cabi.OBS_CIRCLE, A, b
    if style in ('wall', 'wedge'):
        ang = rng.uniform(-np.pi, np.pi)
        rows = [[np.cos(ang), np.sin(ang)]]
        if style == 'wedge':
            ang2 = ang + rng.uniform(0.6, 2.4) * rng.choice([-1, 1])
            rows.append([np.cos(ang2), np.sin(ang2)])
        Ar, br = canonical_polygon_rows(np.array(rows), np.full(len(rows), 0.3), bound=12.0)
        A[:len(Ar)], b[:len(br)] = Ar, br
        return _cabi.OBS_POLYGON, A, b
    if style == 'big':
        # an octagon inscribed in an ellipse of semi-axes >= 6 m: it contains every body centred at the origin
        n = E
        ang = np.linspace(0, 2 * np.pi, n, endpoint=False) + rng.uniform(-0.1, 0.1, n)
        ax, ay = rng.uniform(6.0, 10.0, 2)
    else:
        n = int(rng.integers(3, E + 1))
        ang = np.sort(rng.uniform(0, 2 * np.pi - 0.05 * n, n)) + 0.05 * np.arange(n)    # no two vertices too close
        ax, ay = rng.uniform(0.3, 2.5, 2) if style != 'tiny' else rng.uniform(0.05, 0.15, 2)
    V = np.stack([ax * np.cos(ang), ay * np.sin(ang)])
    Ar, br = polygon_halfspaces(V)
    sc = rng.uniform(0.5, 3.0)                               # rows need not be unit
    A[:n], b[:n] = Ar * sc, br.ravel() * sc
    return _cabi.OBS_POLYGON, A, b


def _moved(kind, A, b, d):
    """The obstacle translated by d."""
    b = b.copy()
    if kind == _cabi.OBS_CIRCLE:
        b[:2] += d
    else:
        live = np.linalg.norm(A, axis=1) > 0
        b[live] += A[live] @ d
    return b


def random_cells(rng, car, n):
    """n cells for body car: kind [n], A [n, E, 2], b [n, E], pose [n, 3] (float32) and the separation asked for [n]."""
    G, h, cone = body_rows(car)
    if cone == _cabi.ROBOT_DISC:
        centre = np.asarray(h, float).ravel()[:2]
    else:
        V = np.array([np.linalg.solve(np.array([G[j - 1], G[j]]), np.array([h[j - 1], h[j]])) for j in range(len(G))])
        centre = V.mean(0)
    kinds = np.zeros(n, np.int32)
    A = np.zeros((n, E, 2))
    b0 = np.zeros((n, E))
    pose = np.zeros((n, 3))
    target = np.zeros(n)
    u = np.zeros((n, 2))
    base = np.zeros((n, 2))
    for k in range(n):
        cat = k % 8
        style = rng.choice(['poly', 'poly', 'poly', 'disc', 'wall', 'wedge'])
        if cat == 6:
            style = 'tiny' if k % 16 == 6 else 'big'
        kinds[k], A[k], b0[k] = _shape(rng, style)
        pose[k] = [rng.choice([-1, 1]) * (60 + rng.uniform(-3, 3)), rng.choice([-1, 1]) * (60 + rng.uniform(-3, 3)),
                   rng.uniform(-np.pi, np.pi)]
        c, s = np.cos(pose[k, 2]), np.sin(pose[k, 2])
        base[k] = pose[k, :2] + np.array([[c, -s], [s, c]]) @ centre
        a = rng.uniform(-np.pi, np.pi)
        u[k] = [np.cos(a), np.sin(a)]
        target[k] = (10 ** rng.uniform(-4, np.log10(50)) if cat < 4 else -10 ** rng.uniform(-4, -1.3) if cat == 4
                     else -rng.uniform(0.1, 0.6) if cat == 5 else np.nan if cat == 6 else 0.0)
    # bisection of the offset t along u: sd(t) = target (containment cells stay at t = 0)
    lo, hi = np.zeros(n), np.full(n, 150.0)
    pose32 = pose.astype(np.float32)

    def place(t):
        return np.stack([_moved(kinds[k], A[k], b0[k], base[k] + t[k] * u[k]) for k in range(n)])
    for _ in range(40):
        mid = 0.5 * (lo + hi)
        d = clearance_twin.cells(G, h, cone, kinds, A, place(mid), pose32)
        up = d < target
        lo = np.where(up, mid, lo)
        hi = np.where(up, hi, mid)
    t = np.where(np.isnan(target), 0.0, hi)
    return kinds, A.astype(np.float32), place(t).astype(np.float32), pose32, target
