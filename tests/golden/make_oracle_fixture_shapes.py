"""Generate tests/golden/oracle_shapes.npz: float64 oracle traces (OracleRDA, every ADMM iteration of one cold call,
iter_threshold = 0) at the horizon lengths T and obstacle counts N where the kernels change shape: T = 1 and 2, N*T below
one warp (several instances per warp on the streaming path), stage ownership by lane at T = 31..33, 64, 65 and 100, more than
32 hinges per stage (N = 33, 64), the disc body's passes at T = 1, 33 and N*T < 32, and the largest layout of the persistent
kernel k_admm_small at T = 10 next to the first one that does not fit.  Each case lists its seeds; the cases
that share warps on the streaming path have several distinct instances, each with its own trace.  The active cells go
through oracle/cell_generic.py (SLSQP), which is why the traces are committed instead of recomputed by the test suite.  The
archive is written with fixed zip timestamps, so a rerun reproduces it bit for bit.  Run in the build container:
    python tests/golden/make_oracle_fixture_shapes.py            (about 17 min on 8 cores)
"""
import io
import os
import sys
import zipfile
from multiprocessing import Pool

os.environ.setdefault('OMP_NUM_THREADS', '1')
os.environ.setdefault('OPENBLAS_NUM_THREADS', '1')
import numpy as np  # noqa: E402

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', '..')
sys.path.insert(0, ROOT)

ITERS, E, LATERAL = 4, 4, (0.3, 3.0)
DISC_BODY = dict(radius=1.0, center=(0.3, 0.0), wheelbase=2.0, dynamics='diff')
# name: (T, N, obstacles, body, seeds).  obstacles: 'polygon' (make_instance's boxes), 'circle' (discs), 'moving' (moving
# discs: per-stage rows), 'mixed' (boxes on the even slots, discs on the odd ones); body: 'rect' (rectangle_robot) or 'disc'
# (DISC_BODY).  The cases of several seeds put more than one instance into a warp of the streaming cell pass.
CASES = {
    't1': (1, 1, 'polygon', 'rect', tuple(range(9101, 9107))),
    't2': (2, 3, 'mixed', 'rect', tuple(range(9201, 9207))),
    't3_moving': (3, 1, 'moving', 'rect', (9301,)),
    'warp_mix': (7, 4, 'mixed', 'rect', tuple(range(9401, 9406))),
    't31': (31, 5, 'mixed', 'rect', (9501,)),
    't32': (32, 4, 'mixed', 'rect', (9502,)),
    't33': (33, 3, 'mixed', 'rect', (9503,)),
    't64': (64, 2, 'polygon', 'rect', (9601,)),
    't65': (65, 2, 'polygon', 'rect', (7067,)),
    't100': (100, 4, 'circle', 'rect', (9701,)),
    'n33': (8, 33, 'polygon', 'rect', (9801,)),
    'n64': (5, 64, 'polygon', 'rect', (9802,)),
    'disc_t1': (1, 2, 'mixed', 'disc', (9901,)),
    'disc_t33': (33, 3, 'mixed', 'disc', (9902,)),
    'disc_mix': (7, 4, 'mixed', 'disc', tuple(range(9911, 9916))),
    # the largest layout of k_admm_small at T = 10 and the first that does not fit its 200 KB of shared memory (rda_create's
    # small_L.total with the float64 su-QP: 203 904 and 204 864 bytes), obstacles spread wide so that a few of them
    # constrain the plan
    'small_max': (10, 177, 'polygon', 'rect', (9991,)),
    'small_over': (10, 178, 'polygon', 'rect', (9992,)),
}
WIDE = {'small_max': (2.0, 30.0), 'small_over': (2.0, 30.0)}        # lateral band of make_instance where not LATERAL


def car(name):
    from rda_planner_b200.scenarios import disc_robot, rectangle_robot
    return disc_robot(**DISC_BODY) if CASES[name][3] == 'disc' else rectangle_robot()


def instance(name, seed):
    """make_instance's corridor at the case's shape; 'mixed' takes the boxes of kind='polygon' on the even slots and the
    discs of kind='circle' (same seed) on the odd ones."""
    from rda_planner_b200.scenarios import make_instance
    T, N, obs, _, _ = CASES[name]
    kw = dict(T=T, N=N, E=E, lateral=WIDE.get(name, LATERAL), dynamics=car(name).dynamics)
    if obs == 'mixed':
        poly, disc = make_instance(seed, kind='polygon', **kw), make_instance(seed, kind='circle', **kw)
        poly['obstacles'] = [disc['obstacles'][o] if o % 2 else poly['obstacles'][o] for o in range(N)]
        return poly
    return make_instance(seed, kind='circle' if obs in ('circle', 'moving') else 'polygon', moving=obs == 'moving', **kw)


def run(job):
    from oracle.rda_oracle import OracleRDA
    name, seed = job
    T, N = CASES[name][:2]
    inst = instance(name, seed)
    ref = [inst['ref'][:, t:t + 1] for t in range(T + 1)]
    o = OracleRDA(T, car(name), max_edge_num=E, max_obs_num=N, iter_num=ITERS, iter_threshold=0.0)
    o.iterative_solve(inst['nom_s'], inst['nom_u'], ref, inst['ref_speed'], list(inst['obstacles']))
    tr = o.trace
    return job, dict(s=np.stack([x[0] for x in tr]), u=np.stack([x[1] for x in tr]),
                     resi_dual=np.array([x[2] for x in tr]), resi_pri=np.array([x[3] for x in tr])), str(o.cell_stats)


def save(path, arrays):
    """np.savez_compressed with a fixed timestamp on every member."""
    with zipfile.ZipFile(path, 'w', zipfile.ZIP_DEFLATED) as zf:
        for key, val in arrays.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(val), allow_pickle=False)
            info = zipfile.ZipInfo(key + '.npy', date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


if __name__ == '__main__':
    jobs = [(name, seed) for name, c in CASES.items() for seed in c[4]]
    jobs.sort(key=lambda j: -CASES[j[0]][0] * CASES[j[0]][1])         # the long ones first
    with Pool(os.cpu_count()) as pool:
        res = {job: (out, stats) for job, out, stats in pool.imap_unordered(run, jobs)}
    flat = {}
    for name, (T, N, obs, body, seeds) in CASES.items():
        # per case: [seed, iteration, ...] traces, the seeds and the generator arguments
        for k in ('s', 'u', 'resi_dual', 'resi_pri'):
            flat[f'{name}_{k}'] = np.stack([res[(name, s)][0][k] for s in seeds])
        flat[f'{name}_seeds'] = np.array(seeds, np.int64)
        flat[f'{name}_args'] = np.array(f'T={T} N={N} E={E} obstacles={obs} body={body} lateral={WIDE.get(name, LATERAL)} '
                                        f'iters={ITERS}')
        for s in seeds:
            print(name, s, res[(name, s)][1])
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'oracle_shapes.npz')
    save(path, flat)
    print('wrote', path)
