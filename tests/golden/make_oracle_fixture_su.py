"""Generate tests/golden/oracle_su.npz: single su-QP solves of the dense float64 oracle (OracleRDA.su_prob_solve,
oracle/qp_ipm.py) at the sizes of configs D (T=30, N=64, slack_gain 13) and E (T=40, N=128), where one oracle solve
takes minutes.  Per size a problem near activity and one whose pruned solve must be repeated: a hinge left out at the
nominal rollout is violated at the pruned optimum (tests/su_cases.py: plant).  The inputs are stored with the
solutions, so the tests need neither the oracle nor the generator.  Run in the build container:
    python tests/golden/make_oracle_fixture_su.py            (~10 min on 4 cores)
"""
import os
import sys
from multiprocessing import Pool

os.environ.setdefault('OMP_NUM_THREADS', '2')
os.environ.setdefault('OPENBLAS_NUM_THREADS', '2')
import numpy as np  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..'))
sys.path.insert(0, os.path.join(HERE, '..'))
import su_cases as sc  # noqa: E402

# name, T, N, tunables, seed, near hinges per stage, planted hinge slots (empty: no planted hinge)
CASES = [('D', 30, 64, 'TUN_D', 8100, 20, ()), ('D_restart', 30, 64, 'TUN_D', 8200, 3, (40,)),
         ('E', 40, 128, 'TUN', 8300, 40, ()), ('E_restart', 40, 128, 'TUN', 8400, 3, (70, 5))]


def make(case):
    """The problem of a case; for a restart case the first seed from `seed` on whose base problem converges without a
    repeat and whose planted hinges (slots `slots`, at the stages that move most) are all violated at its optimum."""
    name, T, N, tun, seed, near, slots = case
    P = sc.params(T, N, tun=getattr(sc, tun))
    if not slots:
        return sc.problem(seed, T, N, near=near), []
    for sd in range(seed, seed + 50):
        p = sc.problem(sd, T, N, v_nom=0.5, near_margin=(0.8, 1.4))
        s, _, _, st, _, rep = sc.cpu(p, P)
        if st != 0 or rep['restarts']:
            continue
        mv = np.linalg.norm(s[0:2, 1:] - sc.rollout(p, P), axis=0)
        cells = list(zip(np.argsort(-mv)[:len(slots)].tolist(), slots))
        try:
            q, lv = sc.plant(p, P, cells)
        except AssertionError:
            continue
        r = sc.cpu(q, P)
        if r[3] == 0 and r[5]['restarts'] == 1 and max(lv) < -0.05:
            return q, cells
    raise RuntimeError(f'no restart instance for {name}')


def run(case):
    name, T, N, tun = case[:4]
    p, cells = make(case)
    s, u, d, info = sc.oracle(p, True, getattr(sc, tun)).su_prob_solve()
    print(name, info['status'], info['iters'], f"merit {info['merit']:.2e}", cells, flush=True)
    return name, p, cells, s, u, np.ravel(d), info


if __name__ == '__main__':
    with Pool(len(CASES)) as pool:
        res = pool.map(run, CASES, chunksize=1)
    flat = {'names': np.array([r[0] for r in res])}
    for (name, p, cells, s, u, d, info), case in zip(res, CASES):
        flat.update({f'{name}_{k}': np.asarray(p[k], np.float32) for k in ('cur_s', 'cur_u', 'ref_s', 'dis', 'pref', 'coef')})
        flat[f'{name}_vref'] = p['vref']
        flat[f'{name}_tun'] = case[3]
        flat[f'{name}_cells'] = np.array(cells, np.int32).reshape(-1, 2)
        flat.update({f'{name}_s': s, f'{name}_u': u, f'{name}_d': d, f'{name}_merit': info['merit'],
                     f'{name}_status': info['status']})
    out = os.path.join(HERE, 'oracle_su.npz')
    np.savez_compressed(out, **flat)
    print('wrote', out)
