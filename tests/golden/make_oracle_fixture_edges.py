"""Generate tests/golden/oracle_edges.npz: float64 oracle traces (OracleRDA, every ADMM iteration of one cold call) of planning
instances whose obstacles have other row counts than 4 — E = 3 (config C), 5 and 6 (half-space sets), 8 (lidar hulls and
polytopes of configs D and E) — with polygons of 3..E vertices from the families of polygon() below, short-edge hulls
included, and discs.  The active cells go through oracle/cell_generic.py (SLSQP), which is why the traces are committed
instead of recomputed by the test suite.  The module also holds the polygon families the cell tests draw from.  Run in the
build container:
    python tests/golden/make_oracle_fixture_edges.py            (139 s on 8 cores)
"""
import os
import sys
from multiprocessing import Pool

os.environ.setdefault('OMP_NUM_THREADS', '1')
os.environ.setdefault('OPENBLAS_NUM_THREADS', '1')
import numpy as np  # noqa: E402

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', '..')
sys.path.insert(0, ROOT)

FAMILIES = ('regular', 'random', 'short', 'collinear', 'thin')


def polygon(rng, family, nv, r=1.0):
    """Convex polygon of nv vertices around the origin (2 x nv, counter-clockwise) and the index of a vertex of interest.
    regular: near-regular; random: random angles on a circle (slivers); short: a corner with an edge of 1e-4..1e-1 m whose
    far end is a nearly flat vertex (the short row and the next one are 1e-3..3e-2 rad apart, as on a lidar hull), returned
    index = that corner; collinear: a nearly flat vertex on an edge (pushed out by 1e-2..5e-2 of the edge); thin: on an
    ellipse of aspect ratio down to 1e-2.  short and collinear need nv >= 4."""
    if family == 'regular':
        ang = np.linspace(0, 2 * np.pi, nv, endpoint=False) + rng.uniform(0, 2 * np.pi)
        ang += rng.uniform(-0.15, 0.15, nv) * 2 * np.pi / nv
        V = r * np.stack([np.cos(ang), np.sin(ang)])
        return V, int(rng.integers(nv))
    if family == 'random':
        while True:
            ang = np.sort(rng.uniform(0, 2 * np.pi, nv))
            if np.min(np.diff(np.append(ang, ang[0] + 2 * np.pi))) > 1e-2:
                break
        return r * np.stack([np.cos(ang), np.sin(ang)]), int(rng.integers(nv))
    if family == 'thin':
        ang = np.sort(np.linspace(0, 2 * np.pi, nv, endpoint=False) + rng.uniform(-0.2, 0.2, nv) + rng.uniform(0, 2 * np.pi))
        asp = 10 ** rng.uniform(-2, -0.5)
        c, s = np.cos(rng.uniform(0, np.pi)), np.sin(rng.uniform(0, np.pi))
        V = np.array([[c, -s], [s, c]]) @ np.stack([r * np.cos(ang), r * asp * np.sin(ang)])
        return V, int(rng.integers(nv))
    assert nv >= 4, (family, nv)
    base, _ = polygon(rng, 'regular', nv - 1, r)
    k = int(rng.integers(nv - 1))
    P, Q = base[:, k], base[:, (k + 1) % (nv - 1)]
    e = Q - P
    el = np.linalg.norm(e)
    u, n = e / el, np.array([e[1], -e[0]]) / el                 # edge direction, outward normal (counter-clockwise)
    if family == 'collinear':
        new = P + rng.uniform(0.2, 0.8) * e + 10 ** rng.uniform(-2, -1.3) * el * n
        return np.insert(base, k + 1, new, axis=1), k + 1
    # short: corner P, short edge P -> X turned outwards by delta, X nearly on the line P -> Q; in half of the cases the
    # short edge X -> P ends at the corner instead, X nearly on the line from the previous vertex
    L, delta = 10 ** rng.uniform(-4, -1), 10 ** rng.uniform(-3, np.log10(3e-2))
    if rng.random() < 0.5:
        X = P + L * (np.cos(delta) * u + np.sin(delta) * n)
        return np.insert(base, k + 1, X, axis=1), k
    e = P - base[:, k - 1]
    u, n = e / np.linalg.norm(e), np.array([e[1], -e[0]]) / np.linalg.norm(e)
    X = P - L * (np.cos(delta) * u - np.sin(delta) * n)
    return np.insert(base, k, X, axis=1), k + 1


def rows(V, E):
    """polygon_halfspaces rows of V (one per edge, row length = edge length) padded with zero rows to E."""
    from rda_planner_b200.mpc import polygon_halfspaces
    A, b = polygon_halfspaces(V)
    nv = A.shape[0]
    return np.vstack([A, np.zeros((E - nv, 2))]), np.concatenate([b.ravel(), np.zeros(E - nv)])


T, N, ITERS = 10, 5, 5
# name: (E, seed, T, N); e5 has N*E*T = 250 (not a multiple of 4): k_admm_small copies its state with threads
CASES = {'e3': (3, 8301, 12, 4), 'e5': (5, 8302, T, N), 'e6': (6, 8303, 12, 4), 'e8': (8, 8304, T, N),
         'e8_short': (8, 8305, 12, 6)}

# residuals the tests compare.  e8_short's rows are as short as 5e-4 m, so lam there is ~2e3 (1/|A_i| times a unit-row
# multiplier) and the float32 lam state resolves it to ~1e-4.  resi_dual, the squared change of lam, falls from 1e6 to 2
# between iterations 1 and 3, and at that size its float32 resolution (measured: 1.7e-2 relative, CPU port against the
# oracle) is above RESI_RTOL: its states, controls and resi_pri are compared, resi_dual is not.
RESI = {name: ('resi_pri',) if name == 'e8_short' else ('resi_pri', 'resi_dual') for name in CASES}


def instance(name):
    """(car, inst, E): make_instance's corridor with the polygons replaced by polygon()'s families at the same centres (short-
    edge hulls on every slot of 'e8_short'), and discs on the odd slots of the other cases."""
    from rda_planner_b200.scenarios import make_instance, rectangle_robot, rdaobs
    E, seed, T_, N_ = CASES[name]
    car = rectangle_robot()
    inst = make_instance(seed, T=T_, N=N_, E=E, lateral=(0.3, 3.0), kind='polygon')
    disc = make_instance(seed, T=T_, N=N_, E=E, lateral=(0.3, 3.0), kind='circle')
    rng = np.random.default_rng(seed)
    obs = []
    for o in range(N_):
        if o % 2 == 1 and name != 'e8_short':
            obs.append(disc['obstacles'][o])
            continue
        fam = 'short' if name == 'e8_short' else FAMILIES[(o // 2) % len(FAMILIES)]
        nv = int(rng.integers(3, E + 1))
        if fam in ('short', 'collinear'):
            nv = max(nv, 4)
        if nv > E:
            fam, nv = 'regular', E
        V, _ = polygon(rng, fam, nv, rng.uniform(0.6, 1.8))
        V = V + np.mean(inst['obstacles'][o].vertex, axis=1).reshape(2, 1)
        A, b = rows(V, nv)
        obs.append(rdaobs(A, b.reshape(-1, 1), 'Rpositive', None, V))
    inst['obstacles'] = obs
    return car, inst, E


def run(name):
    from oracle.rda_oracle import OracleRDA
    car, inst, E = instance(name)
    T_ = CASES[name][2]
    ref = [inst['ref'][:, t:t + 1] for t in range(T_ + 1)]
    o = OracleRDA(T_, car, max_edge_num=E, max_obs_num=CASES[name][3], iter_num=ITERS, iter_threshold=0.0)
    o.iterative_solve(inst['nom_s'], inst['nom_u'], ref, inst['ref_speed'], list(inst['obstacles']))
    tr = o.trace
    out = {'s': np.stack([x[0] for x in tr]), 'u': np.stack([x[1] for x in tr]),
           'resi_dual': np.array([x[2] for x in tr]), 'resi_pri': np.array([x[3] for x in tr])}
    return name, out, str(o.cell_stats)


if __name__ == '__main__':
    with Pool(len(CASES)) as pool:
        res = pool.map(run, list(CASES), chunksize=1)
    flat = {}
    for name, out, stats in res:
        for k, v in out.items():
            flat[f'{name}_{k}'] = v
        print(name, stats)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'oracle_edges.npz')
    np.savez_compressed(path, **flat)
    print('wrote', path)
