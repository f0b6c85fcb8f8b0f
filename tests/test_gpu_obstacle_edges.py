"""-m gpu: obstacle layouts other than E = 4 on the device — E = 3 (config C), 5, 6 (half-space sets) and 8 (lidar hulls and
polytopes of configs D and E).  At these layouts rows_preload and k_cells_fast<4,4> take their scalar branch (E = 3), E > 4 runs
k_cells_fast<8,8> and cell_store reads the previous duals back from the lam / mu planes (rec_duals() is false), k_admm_small
copies its state with threads where N*E*T is not a multiple of 4, and the disc body's passes k_cells_dr* see rows other than 4.
Every cell of a batch against the float64 generic solver, a property test of every cell at the config D shape, and whole solves
against the committed oracle traces of tests/golden/make_oracle_fixture_edges.py."""
import os

import numpy as np
import pytest
import torch

from oracle.cell_generic import solve_cell_generic
from rda_planner_b200.rda_solver import canonical_polygon_rows, pack_obstacles
from rda_planner_b200.scenarios import disc_robot, make_instance, rectangle_robot, rdaobs
from test_cells_vs_generic import TOL
from test_cells_many_edges import EDGES, FLAT, _flatness, _lam_gap
from test_robot_bodies import BODIES, _refine
from test_gpu_parity import TRAJ_TOL, RESI_RTOL

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROUTING_ENV = {                     # environment read by rda_create
    'small': {'RDA_B200_SMALL': '1'},
    'small_threads': {'RDA_B200_SMALL': '1', 'RDA_B200_SMALL_BULK': '0'},
    'stream': {'RDA_B200_SMALL': '0'},
    'extra': {'RDA_B200_SMALL': '0', 'RDA_B200_EXTRA_MIN': '1'},
    'split': {'RDA_B200_SMALL': '0', 'RDA_B200_SPLIT_MIN': '2', 'RDA_B200_SPLIT_PARTS': '2'},
    'split3': {'RDA_B200_SMALL': '0', 'RDA_B200_SPLIT_MIN': '2', 'RDA_B200_SPLIT_PARTS': '3'},
    'coherent': {'RDA_B200_SMALL': '0', 'RDA_B200_LEAN2': '1'},     # polygon body, E <= 4: k_cells_coh first
}
KNOBS = ('RDA_B200_SMALL', 'RDA_B200_LEAN2', 'RDA_B200_EXTRA_MIN', 'RDA_B200_SMALL_BULK', 'RDA_B200_SPLIT_MIN',
         'RDA_B200_SPLIT_PARTS')
DISC_H = (0.3, 0.0, -1.0)


def _car(body):
    if body == 'disc':
        return disc_robot(radius=-DISC_H[2], center=DISC_H[:2], wheelbase=2.0, dynamics='diff')
    return rectangle_robot() if body == 'rect' else BODIES.body(body)


def _solver(monkeypatch, routing, car, T, N, E, iters, B):
    from rda_planner_b200.rda_solver import RDA_solver
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in ROUTING_ENV[routing].items():
        monkeypatch.setenv(k, v)
    return RDA_solver(T, car, max_edge_num=E, max_obs_num=N, iter_num=iters, iter_threshold=0.0, time_print=False, batch=B)


def _batch(car, B, T, N, E, seed0, lateral=(0.2, 2.5)):
    """B instances: on the even slots polygons of 3..E vertices of every family of make_oracle_fixture_edges.polygon (short-
    edge hulls included) at make_instance's obstacle centres, discs on the odd slots."""
    insts = []
    for i in range(B):
        rng = np.random.default_rng(seed0 + i)
        kw = dict(T=T, N=N, E=E, lateral=lateral, dynamics=car.dynamics)
        poly, disc = make_instance(seed0 + i, kind='polygon', **kw), make_instance(seed0 + i, kind='circle', **kw)
        obs = []
        for o in range(N):
            if o % 2:
                obs.append(disc['obstacles'][o])
                continue
            fam = EDGES.FAMILIES[(i * N + o) // 2 % len(EDGES.FAMILIES)]
            nv = int(rng.integers(4 if fam in ('short', 'collinear') else 3, E + 1)) if E >= 4 else 3
            if nv < 4 and fam in ('short', 'collinear'):
                fam = 'regular'
            V, _ = EDGES.polygon(rng, fam, nv, rng.uniform(0.6, 1.8))
            V = V + np.mean(poly['obstacles'][o].vertex, axis=1).reshape(2, 1)
            A, b = EDGES.rows(V, nv)
            obs.append(rdaobs(A, b.reshape(-1, 1), 'Rpositive', None, V))
        poly['obstacles'] = obs
        insts.append(poly)
    packs = [pack_obstacles(list(x['obstacles']), T, N, E) for x in insts]
    f = lambda k: np.stack([x[k] for x in insts]).astype(np.float32)
    return dict(nom_s=f('nom_s'), nom_u=f('nom_u'), ref_s=f('ref'), ref_speed=np.array([x['ref_speed'] for x in insts], np.float32),
                obs_A=np.stack([p[0] for p in packs]), obs_b=np.stack([p[1] for p in packs]),
                obs_kind=np.stack([p[2] for p in packs]), obs_count=np.array([p[3] for p in packs], np.int32))


def _cuda(inp):
    return {k: torch.as_tensor(v, device='cuda') for k, v in inp.items()}


def _buf(g, which):
    from rda_planner_b200 import _cabi
    return g.state_buffer(getattr(_cabi, 'BUF_' + which)).double().cpu().numpy()


CELL_CASES = [(E, body, routing) for E in (3, 5, 8) for body in ('rect', 'hexagon') for routing in ('stream', 'extra')]
CELL_CASES += [(E, 'disc', 'stream') for E in (3, 5, 8)]


@pytest.mark.parametrize('E,body,routing', CELL_CASES)
def test_every_cell_equals_generic_solver(monkeypatch, E, body, routing):
    """Every cell of the second cell step of a batch of B = 4, T = 8, N = 4 against the float64 generic solver
    (check_every_cell)."""
    B, T, N = 4, 8, 4
    car = _car(body)
    disc = body == 'disc'
    # the disc body is narrower than the rectangle: a closer band gives it active cells, which the searched passes take
    inp = _batch(car, B, T, N, E, 9300 + 10 * E, lateral=(0.0, 1.2) if disc else (0.2, 2.5))
    cnt = check_every_cell(monkeypatch, routing, car, disc, inp, T, N, E, f'E = {E}, {body}')
    assert cnt[2] == 0 and cnt[1] > 0                   # the searched passes saw cells of this layout


def check_every_cell(monkeypatch, routing, car, disc, inp, T, N, E, label):
    """Phase API, two ADMM iterations.  Every cell of the second cell step against solve_cell_generic in float64 on the float32
    inputs the kernels read: lam (E rows), mu (R rows), z, zeta_new, xi_new = xi + Hm, the su-QP coefficients rebuilt by
    DESIGN.md §2 (a = lam'A, c0 relative to pref, g = mu'G + xi_new), and the per-instance residuals of finish() against their
    float64 recomputation from the kernels' own multipliers.  Tolerances of test_gpu_robot_bodies.py; lam compared as in
    test_cells_many_edges.py (row scale, flat vertices, the float32 tolerance grown below FLAT).  Returns the cell counters
    of the two cell steps (fast, searched, failed, ...)."""
    B, ro2 = len(inp['nom_s']), 1.0
    G, h = (np.asarray(car.G, float), np.asarray(car.h, float)) if disc else canonical_polygon_rows(car.G, car.h)
    h = np.asarray(h).ravel()
    R = G.shape[0]
    g = _solver(monkeypatch, routing, car, T, N, E, 2, B)
    g.begin(**_cuda(inp), time_varying=False, iter_threshold=0.0)
    g.step_su(); g.step_lammuz()
    g.step_su()
    base = g.launch_count()
    before = {k: _buf(g, k) for k in ('CUR_S', 'DIS', 'ZETA', 'XI', 'LAM', 'MU', 'Z')}
    g.step_lammuz()
    launches = g.launch_count() - base
    after = {k: _buf(g, k) for k in ('LAM', 'MU', 'Z', 'ZETA', 'XI', 'COEF', 'PREF', 'COUNTERS')}
    out = {k: v.double().cpu().numpy() for k, v in g.finish().items()}
    cs = before['CUR_S'].reshape(B, 3, T + 1)
    dis = before['DIS'].reshape(B, T)
    zeta0, xi0 = before['ZETA'].reshape(B, N, T), before['XI'].reshape(B, 2, N, T)
    lam0, mu0, z0 = before['LAM'].reshape(B, N, E, T), before['MU'].reshape(B, N, R, T), before['Z'].reshape(B, N, T)
    lam1, mu1, z1 = after['LAM'].reshape(B, N, E, T), after['MU'].reshape(B, N, R, T), after['Z'].reshape(B, N, T)
    zeta1, xi1 = after['ZETA'].reshape(B, N, T), after['XI'].reshape(B, 2, N, T)
    coef, pref = after['COEF'].reshape(B, 5, N, T), after['PREF'].reshape(B, 2, T)
    A_all, b_all = inp['obs_A'].astype(float), inp['obs_b'].astype(float)
    worst = {k: 0.0 for k in ('lam_mu_z', 'zeta', 'xi', 'a', 'c0', 'g')}
    refereed = active = flat = 0
    for bi in range(B):
        hm2 = dual = 0.0
        for o in range(N):
            A, b = A_all[bi, o, 0], b_all[bi, o, 0]
            circ = int(inp['obs_kind'][bi, o]) == 1
            tol = TOL['f'] if circ else TOL['f'] * max(1.0, FLAT / _flatness(A))
            flat += tol > TOL['f']
            for t in range(T):
                p = cs[bi, 0:2, t + 1].copy()
                phi, dbar, zeta, xi = cs[bi, 2, t], dis[bi, t], zeta0[bi, o, t], xi0[bi, :, o, t].copy()
                c, s = np.cos(phi), np.sin(phi)
                Rm = np.array([[c, -s], [s, c]])
                r = solve_cell_generic(A, b, circ, G, h, p, phi, dbar, zeta, xi, ro2, robot_cone='norm2' if disc else 'Rpositive')
                active += r['active']
                lam, mu, z = lam1[bi, o, :, t], mu1[bi, o, :, t], z1[bi, o, t]
                lgap = np.abs(lam - r['lam']).max() if circ else _lam_gap(A, b, p, lam, r['lam'], tol)
                gap = max(lgap, np.abs(mu - r['mu']).max(), abs(z - r['z']))
                rl, rm, rz = r['lam'], r['mu'], r['z']
                if gap >= tol and r['active'] and not disc:     # the referee of test_robot_bodies decides which side is off
                    refereed += 1
                    fs, xs, gn = _refine(A, b, circ, G, h, p, phi, dbar, zeta, xi, ro2,
                                         [np.concatenate([rl, rm]), np.concatenate([lam, mu])])
                    rl, rm = xs[:E], xs[E:]
                    lgap = np.abs(lam - rl).max() if circ else _lam_gap(A, b, p, lam, rl, tol)
                    gap = max(lgap, np.abs(mu - rm).max(), abs(z - rz))
                assert gap < tol, (bi, o, t, 'lam/mu/z', gap, lam, rl, mu, rm, z, rz)
                if not circ:
                    assert (lam >= -1e-7).all() and np.linalg.norm(A.T @ lam) <= 1 + 1e-5, (bi, o, t, lam)
                worst['lam_mu_z'] = max(worst['lam_mu_z'], gap)
                # zeta / xi updates and su-QP coefficients from the kernel's own multipliers where the split of lam
                # across rows is not unique to the tolerance (flat vertices): they depend on lam only through A'lam, lam'b
                rl = lam if lgap < tol and np.abs(lam - rl).max() >= tol else rl
                scale = 1.0 + np.abs(A @ p - b).sum() + np.abs(h).sum()
                Hm = G.T @ rm + (A @ Rm).T @ rl
                zn = zeta + rl @ (A @ p - b) - rm @ h - dbar - rz
                xn = xi + Hm
                a = A.T @ rl
                c0 = rl @ (A @ pref[bi, :, t] - b) - rm @ h - rz + zn
                gg = G.T @ rm + xn
                gs = tol * (1 + np.abs(A).sum() + np.abs(G).sum())
                checks = {'zeta': (zeta1[bi, o, t], zn, tol * scale), 'xi': (xi1[bi, :, o, t], xn, gs),
                          'a': (coef[bi, 0:2, o, t], a, tol * (1 + np.abs(A).sum())), 'c0': (coef[bi, 2, o, t], c0, tol * scale),
                          'g': (coef[bi, 3:5, o, t], gg, gs)}
                for k, (got, want, tk) in checks.items():
                    d = np.abs(np.asarray(got) - want).max()
                    assert d < tk, (bi, o, t, k, got, want)
                    worst[k] = max(worst[k], d)
                hk = G.T @ mu + (A @ Rm).T @ lam
                hm2 += hk @ hk
                dual += np.sum((lam - lam0[bi, o, :, t]) ** 2) + np.sum((mu - mu0[bi, o, :, t]) ** 2) + (z - z0[bi, o, t]) ** 2
        assert abs(out['resi_pri'][bi] - np.sqrt(hm2)) <= 1e-3 * (1 + np.sqrt(hm2)), (bi, out['resi_pri'][bi], np.sqrt(hm2))
        assert abs(out['resi_dual'][bi] - dual / N) <= 1e-3 * (1 + dual / N), (bi, out['resi_dual'][bi], dual / N)
    cnt = after['COUNTERS'].astype(int)
    print(f'\n{label} (R = {R}), {routing}: largest gap to the float64 reference {worst}; {B * N * T} cells, {active} '
          f'active, {refereed} refereed, obstacles with a vertex flatter than {FLAT}: {flat}; cells per pass fast / searched / '
          f'failed {cnt[:3].tolist()}, launches of the cell step {launches}')
    return cnt


def test_config_d_shape_every_cell_feasible(monkeypatch):
    """Config D's shape (T = 30, N = 64 lidar hulls of 3..8 vertices, E = 8) at B = 8 192: the batch is split in two and each
    sub-batch of 4 096 runs k_cells_extra ahead of the cooperative pass.  After three ADMM iterations every cell must satisfy
    the reference's constraints: |A'lam| <= 1 + 1e-4 and lam >= 0 (polygons), |lam[0:2]| <= -lam[2] (discs), mu, z >= 0."""
    import bench
    from rda_planner_b200.scenarios import CONFIGS
    cfg = CONFIGS['D']
    T, N, E, B = cfg['T'], cfg['N'], cfg['E'], 8192
    inp = bench.build_inputs(B, 4400, config='D')
    car = rectangle_robot()
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    from rda_planner_b200.rda_solver import RDA_solver
    g = RDA_solver(T, car, max_edge_num=E, max_obs_num=N, iter_num=3, iter_threshold=0.0, time_print=False, batch=B)
    dev = _cuda(inp)
    g.begin(**dev, time_varying=False, iter_threshold=0.0)
    for _ in range(3):
        g.step_su()
        g.step_lammuz()
    from rda_planner_b200 import _cabi
    lam = g.state_buffer(_cabi.BUF_LAM).reshape(B, N, E, T)
    mu = g.state_buffer(_cabi.BUF_MU)
    z = g.state_buffer(_cabi.BUF_Z)
    cnt = g.state_buffer(_cabi.BUF_COUNTERS).cpu().tolist()
    out = g.finish()
    A = dev['obs_A'][:, :, 0].float()                                      # [B, N, E, 2]
    a = torch.einsum('bnet,bnex->bntx', lam, A)
    na = a.norm(dim=-1)                                                    # [B, N, T]
    poly = (dev['obs_kind'] == 0)[:, :, None].expand_as(na)
    circ = ~poly
    worst = float(na[poly].max()) if bool(poly.any()) else 0.0
    assert worst <= 1 + 1e-4, worst
    assert float(lam.permute(0, 1, 3, 2)[poly].min()) >= -1e-7
    if bool(circ.any()):
        lc = lam.permute(0, 1, 3, 2)[circ]
        assert bool((lc[:, 0:2].norm(dim=-1) <= -lc[:, 2] + 1e-5).all())
    assert float(mu.min()) >= -1e-7 and float(z.min()) >= 0
    assert int((out['status'] & 6).sum()) == 0
    print(f'\nconfig D shape, B = {B}: {B * N * T} cells, largest |A\'lam| {worst:.7f}; cells per pass over three iterations '
          f'fast / searched / failed {cnt[:3]}, launches {g.launch_count()}')
    assert cnt[2] == 0 and cnt[1] > 0


def _traces():
    return np.load(os.path.join(HERE, 'golden', 'oracle_edges.npz'))


TRACE_CASES = [(n, r) for n in EDGES.CASES for r in ('small', 'stream', 'extra', 'split')] + [('e3', 'small_threads')]


@pytest.mark.parametrize('name,routing', TRACE_CASES)
def test_whole_solves_match_committed_oracle_traces(monkeypatch, name, routing):
    """A cold solve of each case of oracle_edges.npz, the instance twice in a batch of 2 (the split routing runs one per sub-batch),
    last iterate against OracleRDA with the tolerances of test_gpu_parity.py: k_admm_small with bulk staging (N*E*T and N*R*T
    multiples of 4) and with thread copies (e5: N*E*T = 250; e3 with the bulk engine switched off), the streaming kernels,
    k_cells_extra, and the two-stream split."""
    z = _traces()
    car, inst, E = EDGES.instance(name)
    _, _, T, N = EDGES.CASES[name]
    A, b, kd, count, tv = pack_obstacles(list(inst['obstacles']), T, N, E)
    inp = dict(nom_s=inst['nom_s'][None], nom_u=inst['nom_u'][None], ref_s=inst['ref'][None], ref_speed=[inst['ref_speed']],
               obs_A=A[None], obs_b=b[None], obs_kind=kd[None], obs_count=[count])
    inp = {k: np.concatenate([np.asarray(v)] * 2) for k, v in inp.items()}
    g = _solver(monkeypatch, routing, car, T, N, E, EDGES.ITERS, 2)
    o = g.iterative_solve_batch(**inp, time_varying=tv)
    launches = g.launch_count()
    for i in range(2):
        assert int(o['status'][i]) & 7 == 0
        ds = np.abs(o['s'][i].double().cpu().numpy() - z[f'{name}_s'][-1]).max()
        du = np.abs(o['u'][i].double().cpu().numpy() - z[f'{name}_u'][-1]).max()
        assert ds < TRAJ_TOL and du < TRAJ_TOL, (i, ds, du)
        for k in EDGES.RESI[name]:
            ref = z[f'{name}_{k}'][-1]
            assert abs(float(o[k][i]) - ref) <= RESI_RTOL * (1 + ref), (i, k, float(o[k][i]), ref)
    print(f'\n{name} (E = {E}) {routing}: gap to the oracle, states {ds:.1e}, controls {du:.1e}; launches {launches}')
    assert (launches == 1) == routing.startswith('small')
