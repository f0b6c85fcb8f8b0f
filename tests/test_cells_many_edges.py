"""The (lam, mu, z) cell cores at the obstacle layouts other than E = 4 — E = 3 (config C), 5..7 (half-space sets) and 8 (lidar
hulls and polytopes of configs D and E) — against the generic solver in the reference's original variables
(oracle/cell_generic.py), on the g++ build of the kernels' cores: shim.cell in float64 and float32, the first pass
cell_lean<8,8> (cell_lean<4,4> at E = 3) and the disc body's core.  Polygons of 3..E vertices padded with zero rows, from the
families of tests/golden/make_oracle_fixture_edges.py: near-regular, random angles (slivers), a corner with an edge of
1e-4..1e-1 m (the contact is placed at that corner), nearly collinear consecutive vertices, and thin polygons down to an
aspect ratio of 1e-2.  Rows keep their length (the edge's length, as the reference's gen_inequal_global), so lam of a short
row is large: lam is compared in the scale of its row where the row is shorter than 1 (|A_i| |dlam_i|; rows of length >= 1
as they are)."""
import importlib.util
import os

import numpy as np
import pytest

import shim
from oracle.cell_generic import solve_cell_generic, cell_objective
from rda_planner_b200.rda_solver import canonical_polygon_rows
from rda_planner_b200.scenarios import rectangle_robot
from test_cells_vs_generic import TOL, OBJ_TOL
from test_robot_bodies import _refine

HERE = os.path.dirname(os.path.abspath(__file__))
FALLBACK = {'cells': 0}                # cells whose lam the direction / support-value comparison decided
FEAS = 1e-5                             # |A'lam| <= 1 + FEAS, lam, mu >= -1e-7, z >= 0 for every core
DISC_TOL = {'d': 1e-4, 'f': 3e-4}       # test_disc_robot.py's, with 'd' at 1e-4: the generic two-cone solve is accurate to 6e-5 at flat vertices
# float32 places the vertex between two rows delta apart to eps |b| / delta along them (8 mm at delta = 2e-4 and |b| = 30),
# and so the direction of a contact at that vertex: TOL['f'] holds down to delta = FLAT and grows as FLAT / delta below
FLAT = 1e-3
G_DISC = np.array([[1.0, 0.0], [0.0, 1.0], [0.0, 0.0]])
H_DISC = np.array([0.4, 0.1, -0.9])


def _gen():
    spec = importlib.util.spec_from_file_location('make_edges', os.path.join(HERE, 'golden', 'make_oracle_fixture_edges.py'))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


EDGES = _gen()
FAMILIES, polygon, rows = EDGES.FAMILIES, EDGES.polygon, EDGES.rows


def _body_vertices(G, h):
    G, h = canonical_polygon_rows(G, h)
    h = h.ravel()
    R = G.shape[0]
    return np.array([np.linalg.solve(G[[(j - 1) % R, j]], h[[(j - 1) % R, j]]) for j in range(R)])


def _facets(A, b):
    """Every row a facet: consecutive rows meet at a vertex that lies inside every other row.  Rounding the rows to float32
    can cut off an edge shorter than about eps |b| / delta (delta: angle to the neighbouring row); the cores take the rows
    of a polygon to be its edges in order (canonical_polygon_rows), so such a set is drawn again."""
    n = A.shape[0]
    for i in range(n):
        a = (i - 1) % n
        x = np.linalg.solve(A[[a, i]], b[[a, i]])
        if np.any(A @ x - b > 1e-9 * (1 + np.abs(b))):
            return False
    return True


def _cell(rng, k, E, families, Y=None):
    """One cell: a polygon of `families` (cycled by k) at a random place of the world, its contact vertex (the short edge's
    corner for 'short') facing the robot along a direction drawn inside that vertex's normal cone, in the regime k // len % 3:
    far (4..12 m), near (0.2..3 m: hinges become active) or overlapping (0..1 m deep).  Y: body vertices (polygon body), or
    None for the disc body H_DISC."""
    fam = families[k % len(families)]
    regime = (k // len(families)) % 3
    nv = int(rng.integers(4 if fam in ('short', 'collinear') else 3, E + 1))
    while True:
        V, kv = polygon(rng, fam, nv, rng.uniform(0.5, 2.0))
        V = V + rng.uniform(-30, 30, 2)[:, None]
        A, b = rows(V, E)
        A = A.astype(np.float32).astype(float)           # the rows both solvers see are the float32 the kernels store
        b = b.astype(np.float32).astype(float)
        if _facets(A[:nv], b[:nv]):
            break
    ep, en = V[:, kv] - V[:, kv - 1], V[:, (kv + 1) % nv] - V[:, kv]
    a0, a1 = np.arctan2(-ep[0], ep[1]), np.arctan2(-en[0], en[1])          # outward normals (e_y, -e_x) of the two edges
    ang = a0 + rng.uniform(0.05, 0.95) * np.mod(a1 - a0, 2 * np.pi)
    v = np.array([np.cos(ang), np.sin(ang)])
    dist = (rng.uniform(4, 12), rng.uniform(0.2, 3.0), -rng.uniform(0.0, 1.0))[regime]
    phi = rng.uniform(-np.pi, np.pi)
    c, s = np.cos(phi), np.sin(phi)
    Rm = np.array([[c, -s], [s, c]])
    if Y is None:
        p = V[:, kv] + (dist - H_DISC[2]) * v - Rm @ H_DISC[:2]
    else:
        Yw = Y @ Rm.T
        p = V[:, kv] + dist * v - Yw[np.argmin(Yw @ v)]
    dbar = rng.uniform(0.1, 1.0)
    zeta = rng.normal(0, 0.3) * (rng.random() < 0.7)
    xi = rng.normal(0, 0.2, 2) * (rng.random() < 0.5)
    ro2 = (0.5, 1.0, 5.0)[int(rng.integers(0, 3))]
    return fam, regime, A, b, p, phi, dbar, zeta, xi, ro2


def _flatness(A):
    """Smallest sine of the angle between consecutive live rows: the flattest vertex of the polygon."""
    n = A[np.linalg.norm(A, axis=1) > 0]
    n = n / np.linalg.norm(n, axis=1)[:, None]
    m = np.roll(n, -1, axis=0)
    return np.min(n[:, 0] * m[:, 1] - n[:, 1] * m[:, 0])


def _lam_gap(A, b, p, lam, ref, tol):
    """Gap of lam to ref, in the scale of each row where the row is shorter than 1.  Where it is tol or more, the
    multipliers may still be the same LP vertex solution (min lam'(b - A p) s.t. A'lam = v, lam >= 0) reached in a way that
    rounds differently: at a nearly flat vertex (two rows delta apart) lam is 1/delta times as sensitive as v, and across a
    short edge two vertex solutions differ in lam'(b - A p) by less than the LP's tolerance.  There the direction A'lam and
    the support value lam'(b - A p) must agree instead."""
    gap = np.max(np.abs(lam - ref) * np.minimum(1.0, np.linalg.norm(A, axis=1)))
    if gap < tol:
        return gap
    c = b - A @ p
    alt = max(np.abs(A.T @ (lam - ref)).max(), abs((lam - ref) @ c) / (1 + abs(ref @ c)))
    FALLBACK['cells'] += alt < tol
    return min(gap, alt)


def _check_feasible(A, lam, mu, z, where):
    assert (lam >= -1e-7).all() and np.linalg.norm(A.T @ lam) <= 1 + FEAS, (where, lam, np.linalg.norm(A.T @ lam))
    assert (mu >= -1e-7).all() and z >= 0, (where, mu, z)


def _compare(A, b, G, h, p, phi, dbar, zeta, xi, ro2, r, fo, kk, tol, otol, where, ref):
    """(lam, mu, z) gap of one core's answer to the generic solve, or to the referee's refined optimum where an active cell's
    optimum is not unique to the tolerance.  Returns (gap, ref)."""
    lam, mu = kk['lam'], kk['mu']
    fk = cell_objective(A, b, G, h, p, phi, dbar, zeta, xi, ro2, lam, mu, kk['z'])
    gap = max(_lam_gap(A, b, p, lam, r['lam'], tol), np.abs(mu - r['mu']).max(), abs(kk['z'] - r['z']))
    if gap >= tol or fk - fo >= otol * (1 + fo):
        assert r['active'], (where, 'inactive cell off the generic solve', gap, fk - fo)
        if ref is None:
            ref = _refine(A, b, False, G, h, p, phi, dbar, zeta, xi, ro2,
                          [np.concatenate([r['lam'], r['mu']]), np.concatenate([lam, mu])])
        fs, xs, gn = ref
        E = A.shape[0]
        dk = max(_lam_gap(A, b, p, lam, xs[:E], tol), np.abs(mu - xs[E:]).max())
        assert dk < tol, (where, 'core away from the refined optimum', dk, gap)
        assert fk - fs < otol * (1 + fs) + gn * dk * np.sqrt(len(xs)), (where, fk - fs, dk)
        gap = dk
    return gap, ref


LAYOUTS = [(3, ('regular', 'random', 'thin'), 90), (5, FAMILIES, 150), (6, FAMILIES, 120),
           (7, FAMILIES, 90), (8, FAMILIES, 180)]


@pytest.mark.parametrize('E,families,n', LAYOUTS)
def test_cell_cores_equal_generic_solver_at_every_obstacle_layout(E, families, n):
    """shim.cell ('d', 'f') and the first pass cell_lean<8,8> (and <4,4> at E = 3) on every family, every regime, three values
    of ro2, tilted and untilted xi: feasibility of the reference's constraints (:408-419), the reference objective (:399-406)
    within OBJ_TOL of the generic optimum, and (lam, mu, z) within test_cells_vs_generic's TOL.  A disagreement on an active
    cell goes to the referee of test_robot_bodies.py (a refined float64 solve)."""
    car = rectangle_robot()
    G, h = np.asarray(car.G, float), np.asarray(car.h, float).ravel()
    Y = _body_vertices(G, h)
    rng = np.random.default_rng(700 + E)
    leans = ('lean4', 'lean8') if E <= 4 else ('lean8',)
    fb0 = FALLBACK['cells']
    worst = {}
    seen = {'active': 0, 'inactive': 0, 'tilted': 0, 'refereed': 0, 'paths': {}, 'lean': 0, 'flat': 0}
    for k in range(n):
        fam, regime, A, b, p, phi, dbar, zeta, xi, ro2 = _cell(rng, k, E, families, Y)
        r = solve_cell_generic(A, b, False, G, h, p, phi, dbar, zeta, xi, ro2)
        fo = cell_objective(A, b, G, h, p, phi, dbar, zeta, xi, ro2, r['lam'], r['mu'], r['z'])
        seen['active' if r['active'] else 'inactive'] += 1
        seen['tilted'] += bool(np.any(xi != 0))
        ref = None
        for prec in ('d', 'f') + leans:
            kk = shim.cell(G, h, 0, A, b, p, phi, dbar, zeta, xi, ro2, prec=prec)
            where = (E, k, fam, regime, prec)
            if prec.startswith('lean'):
                if kk['path'] == 6:                     # declined: the searched passes take the cell
                    continue
                seen['lean'] += 1
                assert not r['active'] and not np.any(xi != 0), where
            else:
                assert kk['path'] != 5, where            # 5: the core gave up (keep-previous)
                seen['paths'][kk['path']] = seen['paths'].get(kk['path'], 0) + 1
            _check_feasible(A, kk['lam'], kk['mu'], kk['z'], where)
            tol, otol = (TOL['d'], OBJ_TOL['d']) if prec == 'd' else (TOL['f'] * max(1.0, FLAT / _flatness(A)), OBJ_TOL['f'])
            gap, ref = _compare(A, b, G, h, p, phi, dbar, zeta, xi, ro2, r, fo, kk, tol, otol, where, ref)
            key = (prec, fam)
            worst[key] = max(worst.get(key, 0.0), gap)
            seen['flat'] += prec == 'f' and tol > TOL['f']
        seen['refereed'] += ref is not None
    print(f'\nE = {E}: cells {seen}; lam decided by direction and support value (flat vertices) {FALLBACK["cells"] - fb0}')
    for prec in ('d', 'f') + leans:
        print(f'  {prec:6s} largest (lam, mu, z) gap per family ' +
              ', '.join(f'{f} {worst.get((prec, f), 0):.1e}' for f in families))
    assert seen['active'] > n // 6 and seen['inactive'] > n // 5 and seen['tilted'] > n // 4 and seen['lean'] > n // 8


@pytest.mark.parametrize('E', [3, 5, 8])
def test_disc_body_core_equals_generic_solver_at_every_obstacle_layout(E):
    """cell_disc_robot.cuh (float64 and float32) on the same families and regimes, against the generic solver with the body's
    second-order cone (robot_cone='norm2'), with the tolerances of test_disc_robot.py."""
    rng = np.random.default_rng(750 + E)
    families = ('regular', 'random', 'thin') if E == 3 else FAMILIES
    n = 45
    worst = {'d': 0.0, 'f': 0.0}
    paths = {}
    for k in range(n):
        fam, regime, A, b, p, phi, dbar, zeta, xi, ro2 = _cell(rng, k, E, families)
        r = solve_cell_generic(A, b, False, G_DISC, H_DISC, p, phi, dbar, zeta, xi, ro2, robot_cone='norm2')
        fo = cell_objective(A, b, G_DISC, H_DISC, p, phi, dbar, zeta, xi, ro2, r['lam'], r['mu'], r['z'])
        for prec in ('d', 'f'):
            where = (E, k, fam, regime, prec)
            kk = shim.cell_disc_robot(H_DISC, 0, A, b, p, phi, dbar, zeta, xi, ro2, prec=prec)
            assert kk['path'] != 5, where
            paths[kk['path']] = paths.get(kk['path'], 0) + 1
            lam, mu = kk['lam'], kk['mu']
            assert (lam >= -1e-7).all() and np.linalg.norm(A.T @ lam) <= 1 + FEAS, (where, np.linalg.norm(A.T @ lam))
            assert np.hypot(mu[0], mu[1]) <= -mu[2] + 1e-6 and kk['z'] >= 0, where
            gap = max(_lam_gap(A, b, p, lam, r['lam'], DISC_TOL[prec]), np.abs(mu - r['mu']).max(), abs(kk['z'] - r['z']))
            assert gap < DISC_TOL[prec], (where, gap, lam, r['lam'], mu, r['mu'])
            fk = cell_objective(A, b, G_DISC, H_DISC, p, phi, dbar, zeta, xi, ro2, lam, mu, kk['z'])
            assert fk - fo < OBJ_TOL[prec] * (1 + fo) + (1e-8 if prec == 'd' else 0), (where, fk - fo)
            worst[prec] = max(worst[prec], gap)
    print(f'\ndisc body, E = {E}: largest (lam, mu, z) gap {worst}; paths {paths}')
    assert paths.get(0, 0) > 5 and len(paths) >= 3


def _short_edge_hull():
    """The 8-row hull of the lidar sweep that exposed the fault: row 1 is 1.2e-4 m long and 0.3 degrees from row 2."""
    A = np.array([[-0.5666298866271973, 0.6087350249290466], [-0.00011136163811897859, 5.21551955898758e-05],
                  [-0.010576426982879639, 0.004885288421064615], [-0.19758541882038116, 0.06841594725847244],
                  [-1.0235785245895386, -0.26850950717926025], [-0.05887073278427124, -0.05940302461385727],
                  [-0.24856291711330414, -0.44017377495765686], [2.1059153079986572, 0.08599788695573807]])
    b = np.array([14.311259269714355, 0.0021503260359168053, 0.20355620980262756, 3.5787549018859863,
                  12.555319786071777, 0.3448127806186676, -0.15827348828315735, -28.809101104736328])
    return A, b


def test_far_cell_at_the_corner_of_a_short_hull_edge():
    """A far, inactive cell whose contact is the corner at the end of a 1.2e-4 m edge.  In float32 the support of the direction
    v went to the edge's other end, a vertex between two rows 0.3 degrees apart, and the LP-vertex multipliers there put
    |A'lam| = 26.5 on the short row alone.  Every core that resolves the cell must give the generic solve's multipliers: row
    0 and the short row."""
    car = rectangle_robot()
    G, h = np.asarray(car.G, float), np.asarray(car.h, float).ravel()
    A, b = _short_edge_hull()
    p, phi = np.array([-20.943758010864258, 13.519454956054688]), -2.1441547870635986
    dbar, zeta, xi, ro2 = 0.44385185837745667, 0.25531163811683655, np.zeros(2), 5.0
    r = solve_cell_generic(A, b, False, G, h, p, phi, dbar, zeta, xi, ro2)
    assert not r['active'] and r['lam'][0] > 0.4 and r['lam'][1] > 5000
    for prec in ('d', 'f', 'lean8'):
        kk = shim.cell(G, h, 0, A, b, p, phi, dbar, zeta, xi, ro2, prec=prec)
        if prec == 'lean8' and kk['path'] == 6:         # the first pass hands the cell to the searched passes ('f')
            continue
        assert kk['path'] == 0, prec
        _check_feasible(A, kk['lam'], kk['mu'], kk['z'], prec)
        tol = TOL['d'] if prec == 'd' else TOL['f']
        assert np.max(np.abs(kk['lam'] - r['lam']) * np.minimum(1, np.linalg.norm(A, axis=1))) < tol, (prec, kk['lam'], r['lam'])
        assert np.abs(kk['lam'] - r['lam']).max() < tol * (1 + np.abs(r['lam']).max()), prec
        assert np.abs(kk['mu'] - r['mu']).max() < tol and abs(kk['z'] - r['z']) < tol, prec


def test_four_row_closed_forms_at_short_edge_corners():
    """E = 4: quadrilaterals made of a triangle and a short edge at one of its corners, with the contact at that corner, far and
    near, untilted: the first pass cell_lean<4,4> and the coherent pass cell_lean2<4,4> (with the feature pair cell_lean<4,4>
    hands it): feasible multipliers whose direction A'lam is the float64 core's; the float64 core against the generic solver on
    every fourth cell."""
    car = rectangle_robot()
    G, h = np.asarray(car.G, float), np.asarray(car.h, float).ravel()
    Gc, hc = canonical_polygon_rows(G, h)
    hc = hc.ravel()
    Y = _body_vertices(G, h)
    rng = np.random.default_rng(704)
    worst = {'d': 0.0, 'f': 0.0, 'lean4': 0.0, 'lean2': 0.0}
    counts = {k: 0 for k in worst}
    for k in range(400):
        fam, regime, A, b, p, phi, dbar, zeta, _, ro2 = _cell(rng, k, 4, ('short',), Y)
        if regime == 2:
            continue
        xi = np.zeros(2)
        truth = shim.cell(Gc, hc, 0, A, b, p, phi, dbar, zeta, xi, ro2, prec='d')
        if k % 4 == 0:                                  # the float64 core itself against the generic solver
            r = solve_cell_generic(A, b, False, Gc, hc, p, phi, dbar, zeta, xi, ro2)
            fo = cell_objective(A, b, Gc, hc, p, phi, dbar, zeta, xi, ro2, r['lam'], r['mu'], r['z'])
            gap, _ = _compare(A, b, Gc, hc, p, phi, dbar, zeta, xi, ro2, r, fo, truth, TOL['d'], OBJ_TOL['d'], (k, 'd'), None)
            worst['d'] = max(worst['d'], gap)
            counts['d'] += 1
        outs = {prec: shim.cell(Gc, hc, 0, A, b, p, phi, dbar, zeta, xi, ro2, prec=prec) for prec in ('f', 'lean4')}
        if outs['lean4']['path'] == 0 and int(outs['lean4']['hm0']) & 0x40:
            outs['lean2'] = shim.cell_lean2(Gc, hc, A, b, int(outs['lean4']['hm0']), p, phi, dbar, zeta)
        for prec, kk in outs.items():
            if kk['path'] == 6:
                continue
            counts[prec] += 1
            _check_feasible(A, kk['lam'][:4], kk['mu'][:4], kk['z'], (k, prec))
            # the fault's signature is |A'lam| far above 1; the direction A'lam is what the su-QP receives
            gap = np.abs(A.T @ (kk['lam'][:4] - truth['lam'])).max()
            assert gap < TOL['f'], (k, prec, gap, kk['lam'], truth['lam'])
            worst[prec] = max(worst[prec], gap)
    print(f'\nE = 4 short-edge corners: cells per core {counts}; largest gap of A\'lam to the float64 core {worst}')
    assert min(counts[k] for k in ('f', 'lean4', 'lean2')) > 100 and counts['d'] > 50


def test_port_matches_committed_edge_traces():
    """Every ADMM iteration of the cases of tests/golden/oracle_edges.npz (E = 3, 5, 6, 8, short-edge hulls) against the CPU
    port, with the tolerances of test_gpu_parity.py."""
    from oracle import cpu_port
    from rda_planner_b200.rda_solver import pack_obstacles
    from test_robot_bodies import TRAJ_TOL, RESI_RTOL
    z = np.load(os.path.join(HERE, 'golden', 'oracle_edges.npz'))
    for name, (E, _, T, N) in EDGES.CASES.items():
        car, inst, _ = EDGES.instance(name)
        A, b, kd, count, tv = pack_obstacles(list(inst['obstacles']), T, N, E)
        inp = dict(nom_s=inst['nom_s'][None], nom_u=inst['nom_u'][None], ref_s=inst['ref'][None], ref_speed=[inst['ref_speed']],
                   obs_A=A[None], obs_b=b[None], obs_kind=kd[None], obs_count=[count])
        worst = [0.0, 0.0]
        for it in range(1, EDGES.ITERS + 1):
            r = cpu_port.solve_batch(car, T, N, E, time_varying=tv, iter_num=it, threads=1, **inp)
            assert r['cell_failures'][0, 0] == 0
            ds = np.abs(r['s'][0] - z[f'{name}_s'][it - 1]).max()
            du = np.abs(r['u'][0] - z[f'{name}_u'][it - 1]).max()
            worst = [max(worst[0], ds), max(worst[1], du)]
            assert ds < TRAJ_TOL and du < TRAJ_TOL, (name, it, ds, du)
            for k in EDGES.RESI[name]:
                ref = z[f'{name}_{k}'][it - 1]
                assert abs(float(r[k][0]) - ref) <= RESI_RTOL * (1 + ref), (name, it, k, float(r[k][0]), ref)
        print(f'\n{name} (E = {E}): largest gap to the oracle, states {worst[0]:.1e}, controls {worst[1]:.1e}')
