"""The warm-start study of tools/warm_start_probe.py at small B on the CPU, with the float64 oracle (oracle/rda_oracle.py)
as the solver: no GPU involved.

Scene: robots driving east along y = 0 at 3 m/s through a shared world of 2 x 1 m boxes of random yaw, centred 1.6 to
5 m to either side of the line (1.0 x 0.6 m acker bodies, T = 10, N = 6, E = 4, dt = 0.1).  Every step each robot's N
obstacles are the N nearest by the reference's key (obstacle_key, stable order), the nominal is the rollout of its last
controls from its state, the reference the line ahead of its projection.  The loop of each robot runs twice, with the
warm start left in its slot ('slot', the reference) and moved with the obstacles ('obstacle': remap_oracle_slots with
the list positions as ids), each with the early-stop rule (iter_threshold 0.2, at most 20 ADMM iterations) and with 4
fixed iterations.  Reported: churn (share of slots whose obstacle changes from one step to the next), mean ADMM
iterations per step, mean resi_pri / resi_dual, the smallest executed signed distance between the robot body at its
pose and any box of the world (oracle.clearance.polygons), and the number of executed poses closer than 0 (contacts).

    python tools/warm_start_cpu_study.py OUT [--robots 8] [--steps 30] [--procs 8]
"""
import argparse
import json
import os
import sys
from multiprocessing import Pool

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

T, N, E, DT, SPEED = 10, 6, 4, 0.1, 3.0


def world(seed=7, count=48, length=60.0):
    from rda_planner_b200.scenarios import rect_vertices
    from rda_planner_b200.mpc import polygon_halfspaces, rdaobs
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(count):
        c = (rng.uniform(0, length), rng.uniform(1.6, 5.0) * rng.choice([-1, 1]))
        V = rect_vertices(c[0], c[1], 2.0, 1.0, rng.uniform(0, np.pi))
        A, b = polygon_halfspaces(V)
        out.append(rdaobs(A, b, 'Rpositive', None, V))
    return out


def run_robot(args):
    """One robot's closed loop in one warm-start mode and one iteration setting."""
    r, mode, iter_num, thr, steps = args
    import obstacle_ids_twin as oi
    from oracle import clearance as oc
    from oracle.rda_oracle import OracleRDA
    from rda_planner_b200.frontend import pack_worlds, robot_body
    from rda_planner_b200.scenarios import rectangle_robot, rollout
    car = rectangle_robot(length=1.0, width=0.6, wheelbase=0.6)
    boxes = world()
    packed = pack_worlds([boxes])
    lst = {k: packed[k] for k in oi.KEYS}
    body = robot_body(car)['xy'][:4].astype(float)
    polys = [np.asarray(o.vertex, float).T for o in boxes]
    rng = np.random.default_rng(100 + r)
    state = np.array([rng.uniform(0, 10), rng.normal(0, 0.3), rng.normal(0, 0.05)])
    u = np.vstack([np.full(T, SPEED), np.zeros(T)])
    o = OracleRDA(T, car, max_edge_num=E, max_obs_num=N, iter_num=iter_num, step_time=DT, iter_threshold=thr)
    prev, rec = None, {'iters': [], 'resi_pri': [], 'resi_dual': [], 'sd': [], 'churn': []}
    for _ in range(steps):
        pos = oi.kept_positions(oi.reference_keys(lst, state.astype(np.float32)), N)
        if prev is not None:
            rec['churn'].append(float(np.mean(prev != pos)))
            if mode == 'obstacle':
                oi.remap_oracle_slots(o, prev, pos)
        nom_s = rollout(state, u, DT, car.wheelbase, car.dynamics)
        x0 = state[0]
        ref = [np.array([[x0 + SPEED * DT * t], [0.0], [0.0]]) for t in range(T + 1)]
        u, info = o.iterative_solve(nom_s, u, ref, SPEED, [boxes[int(j)] for j in pos])
        u = np.asarray(u, float)
        rec['iters'].append(len(o.trace))
        rec['resi_pri'].append(float(info['resi_pri']))
        rec['resi_dual'].append(float(info['resi_dual']))
        c, s = np.cos(state[2]), np.sin(state[2])
        P = state[:2] + body @ np.array([[c, s], [-s, c]])
        rec['sd'].append(min(oc.polygons(P, Q) for Q in polys))
        state = rollout(state, u[:, :1], DT, car.wheelbase, car.dynamics)[:, 1]
        prev = pos
    return r, mode, iter_num, rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out')
    ap.add_argument('--robots', type=int, default=8)
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--procs', type=int, default=8)
    a = ap.parse_args()
    settings = (('early_stop_20_0.2', 20, 0.2), ('fixed_4', 4, 0.0))
    jobs = [(r, mode, it, thr, a.steps) for _, it, thr in settings for mode in ('slot', 'obstacle') for r in range(a.robots)]
    with Pool(a.procs) as pool:
        done = pool.map(run_robot, jobs)
    res = {'what': __doc__.split('\n\n')[1].replace('\n', ' '), 'robots': a.robots, 'steps': a.steps,
           'device': 'CPU, float64 oracle'}
    for label, it, _ in settings:
        res[label] = {}
        for mode in ('slot', 'obstacle'):
            recs = [d[3] for d in done if d[1] == mode and d[2] == it]
            cat = lambda k: np.concatenate([np.asarray(x[k], float) for x in recs])
            sd = cat('sd')
            res[label][mode] = {'mean_admm_iterations': float(cat('iters').mean()),
                                'mean_resi_pri': float(cat('resi_pri').mean()),
                                'mean_resi_dual': float(cat('resi_dual').mean()),
                                'min_executed_signed_distance_m': float(sd.min()),
                                'contacts': int((sd < 0).sum()), 'executed_poses': int(sd.size),
                                'churn': float(cat('churn').mean())}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'warm_start_cpu_study.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
