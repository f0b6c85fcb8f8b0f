"""-m gpu: whole solves at the horizon lengths T and obstacle counts N where the kernels change shape, on every routing, against
the float64 oracle traces of tests/golden/make_oracle_fixture_shapes.py.  The shapes reach what the metric shape does not:
  - N*T < 32 (t1, t2, t3_moving, warp_mix, disc_t1, disc_mix): on the streaming path one warp of k_cells_fast / k_cells_dr
    holds the cells of several instances, and each instance's residuals are summed by the per-thread branch;
  - T = 1, 2, 31, 32, 33, 64, 65, 100: the su-QP's stage ownership by lane in the whole loop, and k_cells_coh's (o, t) from
    (rem + 0.5) * invT with tiles of ceil(N*T / 128) cells, last tile partly empty;
  - N = 33, 64: more than 32 hinges per stage, so the su-QP's hinge mask has two words, with coefficients from real cell
    passes;
  - k_admm_small at T = 1 and 2, N*T not a multiple of 32 or of 4 (staging by threads), at its largest layout and at the
    first layout that does not fit its 200 KB of shared memory (small_max, small_over), which falls back to streaming;
  - the disc body's passes k_cells_dr* at T = 1, 33 and N*T = 28.
Every cell and every per-instance residual of the warp-sharing shapes against the float64 generic solver, the per-instance
early stop against the oracle's decision on its own trace, the plan clearance of every final plan against oracle/clearance.py,
and k_remap_slots above its 256 threads per CTA against the numpy slot rule."""
import numpy as np
import pytest

from oracle import clearance as ref_clearance
from rda_planner_b200 import _cabi
from rda_planner_b200.rda_solver import RDA_solver
from clearance_cases import body_rows
from test_gpu_obstacle_edges import KNOBS, ROUTING_ENV, _buf, check_every_cell
from test_gpu_obstacle_ids import check_remap_kernel
from test_gpu_parity import TRAJ_TOL, RESI_RTOL
from test_shapes import SHAPES, COMPARE_AT, batch, coherent, traces

pytestmark = pytest.mark.gpu
# rda_create runs k_admm_small when small_L.total <= 200 * 1024 = 204 800 bytes (rda_kernels.cu, small_layout: the six
# per-cell state arrays, the su-QP workspace and its per-hinge arrays, one flag per cell).  At E = R = 4 and the float64
# su-QP (RDA_solver's default):
#   t100 (T = 100, N = 4, N*T = 400)        124 944 B
#   small_max (T = 10, N = 177, N*T = 1770) 203 904 B: the largest N that fits at T = 10
#   small_over (T = 10, N = 178)            204 864 B: falls back to the streaming kernels
# every other case of the table stays below 76 000 B.  The disc body never runs k_admm_small (rb.disc).
FALLS_BACK = {'small_over'}
# n33 is compared after 3 iterations on the device.  Its gap to the oracle in the controls, stream routing, after iterations
# 1..4: 1.2e-6, 8.4e-6, 3.0e-5, 6.1e-4, and resi_dual within 1e-5 relative up to iteration 3, then 0.8556 against 0.8649
# (1.1 %) at iteration 4, the same on every routing.  Every one of its 264 cells of the second cell step agrees with the
# float64 generic solver (largest lam / mu / z gap 8e-6) and its residuals with their float64 recomputation, so the fourth
# iteration amplifies a float32 difference twentyfold rather than computing a wrong cell; the CPU port stays within
# 4e-5 of the oracle there.
GPU_COMPARE_AT = dict(COMPARE_AT, n33=3)
ROUTINGS = ('small', 'small_threads', 'stream', 'extra', 'split', 'split3')
WARP_SHARING = ('warp_mix', 't1', 't2', 'disc_mix')


def _solver(monkeypatch, routing, name, B, iters=SHAPES.ITERS):
    T, N = SHAPES.CASES[name][:2]
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in ROUTING_ENV[routing].items():
        monkeypatch.setenv(k, v)
    return RDA_solver(T, SHAPES.car(name), max_edge_num=SHAPES.E, max_obs_num=N, iter_num=iters, iter_threshold=0.0,
                      time_print=False, batch=B)


def _tiled(inp, B):
    """The case's instances repeated to B instances (instance i is seed i % len(seeds))."""
    n = len(inp['nom_s'])
    idx = np.arange(B) % n
    return {k: np.asarray(v)[idx] for k, v in inp.items()}


def _check_clearance(g, name, s, inp, tv):
    """k_plan_clearance on the final plans s: every (slot, stage) value and the per-instance minimum against the float64
    reference oracle/clearance.py."""
    G, h, cone = body_rows(SHAPES.car(name))
    out = g.plan_clearance(per_cell=True)
    s = s.double().cpu().numpy()
    got = out['map'].cpu().numpy()
    want = ref_clearance.plan_clearance(ref_clearance.body_from_halfspaces(G, h, cone == _cabi.ROBOT_DISC), s,
                                        inp['obs_A'].astype(np.float32), inp['obs_b'].astype(np.float32), inp['obs_kind'],
                                        inp['obs_count'], tv)
    fin = np.isfinite(want)
    assert np.array_equal(fin, np.isfinite(got))
    err = np.abs(got[fin] - want[fin]) / np.maximum(1.0, np.abs(want[fin]))
    assert err.max() < 2e-6, (name, err.max())
    wmin = want.reshape(len(want), -1).min(1)
    gmin = out['min'].cpu().numpy()
    assert (np.abs(gmin - wmin) / np.maximum(1.0, np.abs(wmin)) < 2e-6).all(), (name, gmin, wmin)
    return float(wmin.min())


WHOLE = [(n, r) for n in SHAPES.CASES for r in ROUTINGS] + [(n, 'coherent') for n in SHAPES.CASES if coherent(n)]


@pytest.mark.parametrize('name,routing', WHOLE)
def test_whole_solves_match_committed_oracle_traces(monkeypatch, name, routing):
    """A cold solve of every instance of the case (repeated to two instances where it has one, three for the split in three
    parts), last compared iterate against OracleRDA with the tolerances of test_gpu_parity.py and status & 7 == 0.  Which path
    ran is read from the launch count: 1 is k_admm_small, which the small routings must take exactly where the layout fits
    (and the body is a polygon).  The streaming routing also checks the plan clearance of the final plans."""
    z = traces()
    T, N, _, body, seeds = SHAPES.CASES[name]
    car, inp, tv = batch(name)
    B = max(len(seeds), 3 if routing == 'split3' else 2)
    inp = _tiled(inp, B)
    it = GPU_COMPARE_AT.get(name, SHAPES.ITERS)
    g = _solver(monkeypatch, routing, name, B, iters=it)
    o = g.iterative_solve_batch(**inp, time_varying=tv)
    launches = g.launch_count()
    cnt = _buf(g, 'COUNTERS').astype(int)
    worst = [0.0, 0.0, 0.0]
    for i in range(B):
        k = i % len(seeds)
        assert int(o['status'][i]) & 7 == 0, (i, int(o['status'][i]))
        ds = np.abs(o['s'][i].double().cpu().numpy() - z[f'{name}_s'][k, it - 1]).max()
        du = np.abs(o['u'][i].double().cpu().numpy() - z[f'{name}_u'][k, it - 1]).max()
        assert ds < TRAJ_TOL and du < TRAJ_TOL, (i, ds, du)
        for key in ('resi_pri', 'resi_dual'):
            ref = z[f'{name}_{key}'][k, it - 1]
            rel = abs(float(o[key][i]) - ref) / (1 + ref)
            assert rel <= RESI_RTOL, (i, key, float(o[key][i]), ref)
            worst[2] = max(worst[2], rel)
        worst[:2] = [max(worst[0], ds), max(worst[1], du)]
    clear = _check_clearance(g, name, o['s'], inp, tv) if routing == 'stream' else None
    small = routing.startswith('small') and body == 'rect' and name not in FALLS_BACK
    print(f'\n{name} (T = {T}, N = {N}, N*T = {N * T}, B = {B}, {body} body) {routing}: launches {launches} '
          f'({"k_admm_small" if launches == 1 else "streaming"}); gap to the oracle after {it} iterations: states {worst[0]:.1e}, '
          f'controls {worst[1]:.1e}, residuals {worst[2]:.1e} relative; cells per pass fast / searched / failed '
          f'{cnt[:3].tolist()}' + ('' if clear is None else f'; smallest plan clearance {clear:.3f} m'))
    assert (launches == 1) == small, (launches, small)
    if routing == 'small' and name == 'small_max':
        assert N * T >= 400 and launches == 1
    if routing == 'small' and name == 'small_over':
        assert launches > 1
    assert cnt[2] == 0


CELL_RUNS = [(n, 'stream') for n in WARP_SHARING] + [(n, 'coherent') for n in WARP_SHARING if coherent(n)]


@pytest.mark.parametrize('name,routing', CELL_RUNS)
def test_every_cell_and_instance_residual_at_warp_sharing_shapes(monkeypatch, name, routing):
    """Phase API, two ADMM iterations on every instance of the case in one batch (distinct seeds, so a residual summed into
    the wrong instance changes a value): every cell of the second cell step against the float64 generic solver, and each
    instance's resi_pri / resi_dual from finish() against their float64 recomputation from the kernels' own multipliers
    (test_gpu_obstacle_edges.check_every_cell).  N*T < 32: on the streaming path a warp holds cells of several instances."""
    T, N, _, body, seeds = SHAPES.CASES[name]
    car, inp, _ = batch(name)
    inp = {k: np.asarray(v, np.float32) if np.asarray(v).dtype == np.float64 else np.asarray(v) for k, v in inp.items()}
    assert N * T < 32 and len(seeds) > 1
    cnt = check_every_cell(monkeypatch, routing, car, body == 'disc', inp, T, N, SHAPES.E,
                           f'{name}: T = {T}, N = {N}, {len(seeds)} instances, cells of {min(len(seeds), -(-32 // (N * T)))} '
                           f'instances in the first warp')
    assert cnt[2] == 0


def _stop_threshold(z, name):
    """A threshold at which the instances of the case stop at different iterations by the oracle's rule (resi_dual < thr and
    resi_pri < thr after an iteration, :594), at least 5 % away from every residual the rule compares, and the oracle's
    stop iteration of each instance (ITERS + 1: runs to the end)."""
    m = np.maximum(z[f'{name}_resi_dual'], z[f'{name}_resi_pri'])              # [instance, iteration]
    vals = np.unique(m)
    best = None
    for lo, hi in zip(vals[:-1], vals[1:]):
        thr = float(np.sqrt(lo * hi))
        if hi < 1.1 * lo or (np.abs(m - thr) < 0.05 * thr).any():
            continue
        below = m < thr
        stop = np.where(below.any(1), below.argmax(1) + 1, SHAPES.ITERS + 1)
        if best is None or len(set(stop)) > len(set(best[1])):
            best = (thr, stop)
    return best


EARLY = [(n, r) for n in WARP_SHARING for r in ('stream', 'small')] + [(n, 'coherent') for n in WARP_SHARING if coherent(n)]


@pytest.mark.parametrize('name,routing', EARLY)
def test_per_instance_early_stop_at_warp_sharing_shapes(monkeypatch, name, routing):
    """With a threshold at which the instances stop at different iterations, each instance's iteration count and early-stop
    flag (status & 8) must be the oracle's decision on its own trace, and its plan the oracle's at that iteration."""
    z = traces()
    T, N, _, body, seeds = SHAPES.CASES[name]
    best = _stop_threshold(z, name)
    assert best is not None, name
    thr, stop = best
    assert len(set(stop)) >= 2, (name, stop)
    car, inp, tv = batch(name)
    g = _solver(monkeypatch, routing, name, len(seeds))
    o = g.iterative_solve_batch(**inp, time_varying=tv, iter_threshold=thr)
    iters, status = o['iters'].cpu().numpy(), o['status'].cpu().numpy()
    for i in range(len(seeds)):
        want = min(stop[i], SHAPES.ITERS)
        assert int(iters[i]) == want and bool(status[i] & 8) == (stop[i] <= SHAPES.ITERS), (i, int(iters[i]), int(status[i]), stop[i])
        ds = np.abs(o['s'][i].double().cpu().numpy() - z[f'{name}_s'][i, want - 1]).max()
        du = np.abs(o['u'][i].double().cpu().numpy() - z[f'{name}_u'][i, want - 1]).max()
        assert ds < TRAJ_TOL and du < TRAJ_TOL, (i, ds, du)
    print(f'\n{name} {routing}: threshold {thr:.3g}, iterations per instance {iters.tolist()} (oracle {stop.tolist()}), '
          f'launches {g.launch_count()}')


@pytest.mark.parametrize('T,E,disc', [(1, 4, False), (33, 8, True)])
def test_remap_slots_above_one_cta_of_threads(T, E, disc):
    """k_remap_slots at N = 300 slots, above its 256 threads per CTA, at T = 1 and T = 33, against the numpy slot rule of
    obstacle_ids_twin, bit for bit (test_gpu_obstacle_ids.check_remap_kernel)."""
    check_remap_kernel(6, T, 300, E, disc, 300 + T)
