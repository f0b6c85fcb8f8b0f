"""Generate tests/golden/oracle_bodies.npz: float64 oracle traces (OracleRDA, every ADMM iteration) of one planning instance
per polygon robot body of BODIES below — the rear-axle rectangle every other test uses, the centred bodies of the reference's
diff-drive and omni examples (wheelbase 0), triangles (R = 3), pentagon / hexagon / octagon (R = 5, 6, 8) and bodies whose
reference point lies OUTSIDE them.  Per body: a cold call, a warm-started second call on the same inputs and a third call
after reset() (which keeps mu, z, zeta and rebuilds lam'b from mu'h).  The active cells go through oracle/cell_generic.py
(SLSQP), which is why the traces are committed instead of recomputed by the test suite.  Run in the build container:
    python tests/golden/make_oracle_fixture_bodies.py            (~2 min on 5 cores)
"""
import os
import sys
from multiprocessing import Pool

os.environ.setdefault('OMP_NUM_THREADS', '1')
os.environ.setdefault('OPENBLAS_NUM_THREADS', '1')
import numpy as np  # noqa: E402

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', '..')
sys.path.insert(0, ROOT)


def _ellipse(cx, cy, ax, ay, deg):
    """Vertices on an ellipse at the given angles (degrees, increasing): a convex polygon, counter-clockwise."""
    a = np.radians(np.asarray(deg, float))
    return np.stack([cx + ax * np.cos(a), cy + ay * np.sin(a)])


def _box(x0, x1, y0, y1):
    return np.array([[x0, x1, x1, x0], [y0, y0, y1, y1]], float)


# name: (vertices 2 x R, counter-clockwise in the body frame; dynamics; wheelbase)
BODIES = {
    'rect_rear': (_box(-0.8, 3.8, -0.8, 0.8), 'acker', 3.0),                     # rectangle_robot(): the control
    'rect_centred': (_box(-2.3, 2.3, -0.8, 0.8), 'diff', 0.0),                   # example/*/*_diff.yaml
    'omni_centred': (_box(-1.5, 1.5, -0.8, 0.8), 'omni', 0.0),                   # example/*/*_omni.yaml
    'triangle': (np.array([[-1.0, 2.6, 0.2], [-0.9, -0.2, 1.1]]), 'acker', 2.0),
    'triangle_out': (np.array([[0.6, 3.2, 1.0], [-0.8, 0.1, 1.0]]), 'diff', 0.0),   # reference point outside
    'offset_box': (_box(0.5, 3.0, -0.6, 0.6), 'acker', 2.5),                     # reference point outside
    'pentagon': (_ellipse(0.9, 0.1, 2.2, 0.9, [-100, -20, 35, 110, 190]), 'diff', 0.0),
    'hexagon': (_ellipse(1.1, -0.05, 2.4, 0.85, [-130, -70, -5, 60, 120, 175]), 'acker', 2.8),
    'octagon': (_ellipse(0.7, 0.12, 1.9, 0.95, [-160, -115, -62, -20, 25, 80, 118, 150]), 'omni', 0.0),
}
# the same body with its rows in another order: starting at another vertex, and clockwise
ROW_ORDER_BODY = 'pentagon'


def body(name, dynamics=None):
    """Car tuple (scenarios.car) of body `name`: rows of polygon_halfspaces, i.e. counter-clockwise, row i = edge i -> i+1."""
    from rda_planner_b200.scenarios import car
    from rda_planner_b200.mpc import polygon_halfspaces
    vert, dyn, wheelbase = BODIES[name]
    G, h = polygon_halfspaces(vert)
    return car(G, h, 'Rpositive', wheelbase, [10, 1], [10, 0.5], dynamics or dyn)


def row_orders(name=ROW_ORDER_BODY):
    """(label, G, h) of the body with its rows rotated by two places, and listed clockwise."""
    c = body(name)
    G, h = np.asarray(c.G, float), np.asarray(c.h, float).reshape(-1, 1)
    return [('rotated', np.roll(G, -2, axis=0), np.roll(h, -2, axis=0)), ('clockwise', G[::-1].copy(), h[::-1].copy())]


T, N, ITERS = 12, 6, 6
# name: seed, obstacles ('mixed': polygons and discs alternately, 'moving': moving discs)
CASES = {
    'rect_rear': (7101, 'mixed'), 'rect_centred': (7102, 'mixed'), 'omni_centred': (7103, 'moving'),
    'triangle': (7104, 'mixed'), 'triangle_out': (7105, 'mixed'), 'offset_box': (7106, 'mixed'),
    'pentagon': (7107, 'mixed'), 'hexagon': (7108, 'moving'), 'octagon': (7109, 'mixed'),
}


def instance(name):
    """(car, inst) on the harsh band lateral = (0.3, 3.5): obstacles beside and on the path."""
    from rda_planner_b200.scenarios import make_instance
    seed, kind = CASES[name]
    car = body(name)
    kw = dict(T=T, N=N, E=4, lateral=(0.3, 3.5), dynamics=car.dynamics)
    if kind == 'moving':
        return car, make_instance(seed, kind='circle', moving=True, **kw)
    poly = make_instance(seed, kind='polygon', **kw)
    disc = make_instance(seed, kind='circle', **kw)       # same nominal path and reference (drawn before the obstacles)
    poly['obstacles'] = [(poly if o % 2 == 0 else disc)['obstacles'][o] for o in range(N)]
    return car, poly


def run(name):
    from oracle.rda_oracle import OracleRDA
    car, inst = instance(name)
    ref = [inst['ref'][:, t:t + 1] for t in range(T + 1)]
    o = OracleRDA(T, car, max_edge_num=4, max_obs_num=N, iter_num=ITERS, iter_threshold=0.0)
    out = {}
    for call in range(3):
        if call == 2:
            o.reset()
        o.iterative_solve(inst['nom_s'], inst['nom_u'], ref, inst['ref_speed'], list(inst['obstacles']))
        tr = o.trace
        out[f'c{call}_s'] = np.stack([x[0] for x in tr])
        out[f'c{call}_u'] = np.stack([x[1] for x in tr])
        out[f'c{call}_resi_dual'] = np.array([x[2] for x in tr])
        out[f'c{call}_resi_pri'] = np.array([x[3] for x in tr])
    return name, out, str(o.cell_stats)


if __name__ == '__main__':
    with Pool(5) as pool:
        res = pool.map(run, list(CASES), chunksize=1)
    flat = {}
    for name, out, stats in res:
        for k, v in out.items():
            flat[f'{name}_{k}'] = v
        print(name, stats)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'oracle_bodies.npz')
    np.savez_compressed(path, **flat)
    print('wrote', path)
