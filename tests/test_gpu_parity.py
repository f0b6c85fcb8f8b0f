"""-m gpu: the CUDA path through the C ABI (librda_b200.so) against the oracle, plus
size-independent properties at the full benchmark size."""
import numpy as np
import pytest
import torch

from rda_planner_b200.scenarios import rectangle_robot, make_instance

pytestmark = pytest.mark.gpu

# Stated float32 tolerances (BASELINE.json north_star: "match ... to a stated fp32 tolerance"):
TRAJ_TOL = 1e-3      # states (m, rad) and controls, absolute, after <= 6 ADMM iterations; 2e-3 after 8 (the ADMM map
                     # amplifies float32 rounding of the cell pass on instances with overlap cells, DESIGN.md §5;
                     # tests/test_gpu_parity50.py bounds the whole distribution up to 50 iterations)
RESI_RTOL = 2e-3     # residuals, relative


def _solvers(T, N, iters, dyn='acker', **kw):
    from rda_planner_b200.rda_solver import RDA_solver
    from oracle.rda_oracle import OracleRDA
    car = rectangle_robot(dynamics=dyn)
    g = RDA_solver(T, car, max_edge_num=4, max_obs_num=N, iter_num=iters, iter_threshold=kw.pop('thr', 0.0),
                   time_print=False, **kw)
    o = OracleRDA(T, car, max_edge_num=4, max_obs_num=N, iter_num=iters, iter_threshold=g.iter_threshold,
                  **{k: v for k, v in kw.items() if k in ('accelerated', 'ro1', 'ro2', 'slack_gain', 'min_sd', 'max_sd', 'ws', 'wu')})
    return car, g, o


@pytest.mark.parametrize('seed,T,N,iters,kind,dyn,moving', [
    (3, 10, 4, 4, 'polygon', 'acker', False),      # BASELINE configs[0] geometry (path_track)
    (11, 10, 5, 6, 'polygon', 'acker', False),     # obstacles on the path: active hinges, overlap
    (13, 10, 5, 6, 'circle', 'acker', False),
    (14, 10, 5, 6, 'polygon', 'diff', False),
    (15, 10, 5, 6, 'polygon', 'omni', False),
    (17, 12, 5, 5, 'circle', 'acker', True),       # moving discs: per-stage obstacle copies
    (18, 12, 5, 5, 'polygon', 'diff', True),
    (16, 20, 10, 8, 'polygon', 'acker', False),    # BASELINE configs[1] size (corridor)
])
def test_trajectory_matches_oracle(seed, T, N, iters, kind, dyn, moving):
    car, g, o = _solvers(T, N, iters, dyn)
    inst = make_instance(seed, T=T, N=N, E=4, lateral=(0.3, 3.5), kind=kind, dynamics=dyn, moving=moving)
    ref = [inst['ref'][:, t:t + 1] for t in range(T + 1)]
    ug, ig = g.iterative_solve(inst['nom_s'], inst['nom_u'], ref, inst['ref_speed'], list(inst['obstacles']))
    uo, io = o.iterative_solve(inst['nom_s'], inst['nom_u'], ref, inst['ref_speed'], list(inst['obstacles']))
    assert ig['status'] & 7 == 0
    tol = TRAJ_TOL if iters <= 6 else 2 * TRAJ_TOL
    np.testing.assert_allclose(ug, uo, atol=tol)
    np.testing.assert_allclose(np.hstack(ig['opt_state_list']), np.hstack(io['opt_state_list']), atol=tol)
    assert abs(ig['resi_dual'] - io['resi_dual']) <= RESI_RTOL * (1 + io['resi_dual'])
    assert abs(ig['resi_pri'] - io['resi_pri']) <= RESI_RTOL * (1 + io['resi_pri'])


def test_non_accelerated_mode_and_tunables():
    car, g, o = _solvers(8, 3, 4, accelerated=False, ro1=1, slack_gain=5, min_sd=0.2)
    inst = make_instance(21, T=8, N=3, E=4, lateral=(0.5, 3.0))
    ref = [inst['ref'][:, t:t + 1] for t in range(9)]
    ug, ig = g.iterative_solve(inst['nom_s'], inst['nom_u'], ref, 4.0, list(inst['obstacles']))
    uo, io = o.iterative_solve(inst['nom_s'], inst['nom_u'], ref, 4.0, list(inst['obstacles']))
    np.testing.assert_allclose(ug, uo, atol=TRAJ_TOL)
    p = g.get_adjust_parameter()
    assert p['ro1'] == 1 and p['slack_gain'] == 5 and abs(p['min_sd'] - 0.2) < 1e-7
    g.assign_adjust_parameter(ro1=150, max_sd=0.8)
    assert g.get_adjust_parameter()['ro1'] == 150


def test_warm_start_across_calls_reset_and_early_stop():
    """Second control step reuses lam/mu/z/xi/zeta/d (never cleared, SURVEY §9.8 quirk 5); reset()
    clears only lam'A, lam'b (:1060-1068); early stop follows :594-596."""
    car, g, o = _solvers(8, 3, 3)
    a = make_instance(31, T=8, N=3, E=4, lateral=(0.5, 3.0))
    ref = [a['ref'][:, t:t + 1] for t in range(9)]
    for k in range(3):
        if k == 2:
            g.reset(); o.reset()
        ug, ig = g.iterative_solve(a['nom_s'], a['nom_u'], ref, 4.0, list(a['obstacles']))
        uo, io = o.iterative_solve(a['nom_s'], a['nom_u'], ref, 4.0, list(a['obstacles']))
        np.testing.assert_allclose(ug, uo, atol=TRAJ_TOL)
    car, g, o = _solvers(8, 3, 10, thr=0.5)
    ug, ig = g.iterative_solve(a['nom_s'], a['nom_u'], ref, 4.0, list(a['obstacles']))
    uo, io = o.iterative_solve(a['nom_s'], a['nom_u'], ref, 4.0, list(a['obstacles']))
    assert ig['iterations'] == len(o.trace) and ig['iterations'] < 10
    np.testing.assert_allclose(ug, uo, atol=TRAJ_TOL)


def test_empty_and_short_obstacle_lists():
    car, g, o = _solvers(6, 3, 2)
    a = make_instance(41, T=6, N=2, E=4, lateral=(0.5, 3.0))
    ref = [a['ref'][:, t:t + 1] for t in range(7)]
    ug, ig = g.iterative_solve(a['nom_s'], a['nom_u'], ref, 4.0, list(a['obstacles']))      # padded by repetition
    uo, io = o.iterative_solve(a['nom_s'], a['nom_u'], ref, 4.0, list(a['obstacles']))
    np.testing.assert_allclose(ug, uo, atol=TRAJ_TOL)
    ug, ig = g.iterative_solve(a['nom_s'], a['nom_u'], ref, 4.0, [])                        # stale terms quirk
    uo, io = o.iterative_solve(a['nom_s'], a['nom_u'], ref, 4.0, [])
    np.testing.assert_allclose(ug, uo, atol=TRAJ_TOL)
    assert ig['resi_pri'] == 0 and ig['resi_dual'] == 0


def test_mpc_front_end_on_gpu_matches_oracle_backed_front_end():
    """example/path_track geometry: MPC.control for a few steps, CUDA solver vs oracle solver."""
    import os
    from collections import namedtuple
    from RDA_planner.mpc import MPC
    from oracle.rda_oracle import OracleRDA
    here = os.path.dirname(os.path.abspath(__file__))
    path = list(np.load(os.path.join(here, 'golden', 'path_track_ref.npy'), allow_pickle=True))
    Obs = namedtuple('Obs', 'center radius vertex cone_type velocity')
    obs = [Obs(np.array([[20.], [34.]]), 1.5, None, 'norm2', np.zeros((2, 1))),
           Obs(np.array([[10.5], [44.5]]), 1.0, None, 'norm2', np.zeros((2, 1))),
           Obs(None, None, np.array([[12., 14, 14, 12], [41, 41, 39, 39]]), 'Rpositive', np.zeros((2, 1)))]
    car = rectangle_robot()
    import copy
    kw = dict(receding=10, sample_time=0.1, iter_num=2, ro1=300, max_edge_num=4, max_obs_num=4, slack_gain=8)
    mg = MPC(car, copy.deepcopy(path), **kw)
    mo = MPC(car, copy.deepcopy(path), solver_cls=OracleRDA, **kw)
    state = np.array([[10.], [42.], [1.57]])
    for k in range(3):
        ug, ig = mg.control(state.copy(), 4, obs)
        uo, io = mo.control(state.copy(), 4, obs)
        np.testing.assert_allclose(ug, uo, atol=2e-3)
        th = state[2, 0]
        state = state + 0.1 * np.array([[uo[0, 0] * np.cos(th)], [uo[0, 0] * np.sin(th)], [uo[0, 0] * np.tan(uo[1, 0]) / 3.0]])


def _batch_inputs(B, T, N, seed0, **kw):
    from rda_planner_b200.rda_solver import pack_obstacles
    insts = [make_instance(seed0 + i, T=T, N=N, E=4, **kw) for i in range(B)]
    packs = [pack_obstacles(list(i['obstacles']), T, N, 4) for i in insts]
    return insts, dict(nom_s=np.stack([i['nom_s'] for i in insts]), nom_u=np.stack([i['nom_u'] for i in insts]),
                       ref_s=np.stack([i['ref'] for i in insts]), ref_speed=np.array([i['ref_speed'] for i in insts]),
                       obs_A=np.stack([p[0] for p in packs]), obs_b=np.stack([p[1] for p in packs]),
                       obs_kind=np.stack([p[2] for p in packs]), obs_count=np.array([p[3] for p in packs]))


def test_batch_equals_single_instances_and_cpu_port():
    """Instances of a batch do not interact; the compiled CPU port (same cores) agrees."""
    from rda_planner_b200.rda_solver import RDA_solver
    from oracle import cpu_port
    T, N, B, iters = 12, 6, 37, 6
    car = rectangle_robot()
    insts, inp = _batch_inputs(B, T, N, 500, lateral=(0.3, 3.5))
    gb = RDA_solver(T, car, 4, N, iter_num=iters, iter_threshold=0.0, time_print=False, batch=B)
    out = {k: v.clone() for k, v in gb.iterative_solve_batch(**inp).items()}
    assert int((out['status'] & 7).sum()) == 0
    port = cpu_port.solve_batch(car, T, N, 4, **inp, iter_num=iters)
    # nvcc and g++ contract multiply-adds differently; on the most sensitive instance of this (harsh)
    # batch the gap reaches 1e-3 after 6 iterations, hence 3x the oracle tolerance here
    np.testing.assert_allclose(out["u"].cpu().numpy(), port["u"], atol=3 * TRAJ_TOL)
    np.testing.assert_allclose(out["s"].cpu().numpy(), port["s"], atol=3 * TRAJ_TOL)
    g1 = RDA_solver(T, car, 4, N, iter_num=iters, iter_threshold=0.0, time_print=False)
    for i in (0, 17, 36):
        g1.cold_start()
        ref = [insts[i]['ref'][:, t:t + 1] for t in range(T + 1)]
        u1, _ = g1.iterative_solve(insts[i]['nom_s'], insts[i]['nom_u'], ref, 4.0, list(insts[i]['obstacles']))
        np.testing.assert_allclose(out['u'][i].cpu().numpy(), u1, atol=1e-6)


def test_full_size_properties():
    """BASELINE metric size (T=30, N=20, 50 iterations), B=256: finite, bounds respected, deterministic,
    permutation-equivariant over instances, invariant to duplicating the last obstacle slot."""
    from rda_planner_b200.rda_solver import RDA_solver
    T, N, B = 30, 20, 256
    car = rectangle_robot()
    insts, inp = _batch_inputs(B, T, N, 9000)
    g = RDA_solver(T, car, 4, N, iter_num=50, iter_threshold=0.0, time_print=False, batch=B)
    a = {k: v.clone() for k, v in g.iterative_solve_batch(**inp).items()}
    assert torch.isfinite(a['u']).all() and torch.isfinite(a['s']).all()
    assert int((a['status'] & 6).sum()) == 0
    assert float(a['u'][:, 0].abs().max()) <= 10 + 1e-4 and float(a['u'][:, 1].abs().max()) <= 1 + 1e-4
    du = (a['u'][:, :, 1:] - a['u'][:, :, :-1]).abs()
    assert float(du[:, 0].max()) <= 1.0 + 1e-4 and float(du[:, 1].max()) <= 0.05 + 1e-4
    assert (a['iters'] == 50).all()
    g.cold_start()
    b = {k: v.clone() for k, v in g.iterative_solve_batch(**inp).items()}
    assert torch.equal(a['u'], b['u']) and torch.equal(a['s'], b['s'])            # deterministic
    perm = np.random.default_rng(0).permutation(B)
    g.cold_start()
    c = g.iterative_solve_batch(**{k: v[perm] for k, v in inp.items()})
    assert torch.equal(c['u'], a['u'][torch.as_tensor(perm, device=a['u'].device)])
    # early stop enabled: every instance stops with both residuals below the threshold or runs out
    g.cold_start()
    d = g.iterative_solve_batch(**inp, iter_threshold=0.2)
    stopped = (d['status'] & 8) != 0
    assert bool(((d['resi_pri'] < 0.2) & (d['resi_dual'] < 0.2))[stopped].all())
    assert bool((d['iters'][~stopped] == 50).all())


def test_golden_trajectory_fixture():
    """Committed oracle output at the metric size (tests/golden/oracle_metric_T30N20.npz, made by
    tests/golden/make_oracle_fixture.py) after 6 ADMM iterations."""
    import os
    from rda_planner_b200.rda_solver import RDA_solver
    here = os.path.dirname(os.path.abspath(__file__))
    fx = np.load(os.path.join(here, 'golden', 'oracle_metric_T30N20.npz'))
    T, N = 30, 20
    car = rectangle_robot()
    inst = make_instance(int(fx['seed']), T=T, N=N, E=4)
    ref = [inst['ref'][:, t:t + 1] for t in range(T + 1)]
    g = RDA_solver(T, car, 4, N, iter_num=int(fx['iters']), iter_threshold=0.0, time_print=False)
    u, info = g.iterative_solve(inst['nom_s'], inst['nom_u'], ref, inst['ref_speed'], list(inst['obstacles']))
    np.testing.assert_allclose(u, fx['u'], atol=TRAJ_TOL)
    np.testing.assert_allclose(np.hstack(info['opt_state_list']), fx['s'], atol=TRAJ_TOL)


def test_golden_trajectory_fixture_moving_circles():
    """BASELINE configs[2] geometry: T=30, 20 moving discs, min_sd=0.5, wu=0.2
    (tests/golden/oracle_circles_T30N20.npz, made by tests/golden/make_oracle_fixture_circles.py)."""
    import os
    from rda_planner_b200.rda_solver import RDA_solver
    here = os.path.dirname(os.path.abspath(__file__))
    fx = np.load(os.path.join(here, 'golden', 'oracle_circles_T30N20.npz'))
    T, N = 30, 20
    car = rectangle_robot(max_acce=(10, 1.0))
    inst = make_instance(int(fx['seed']), T=T, N=N, E=4, kind='circle', moving=True, lateral=(1.0, 6.0))
    ref = [inst['ref'][:, t:t + 1] for t in range(T + 1)]
    g = RDA_solver(T, car, 4, N, iter_num=int(fx['iters']), iter_threshold=0.0, time_print=False, min_sd=0.5, wu=0.2)
    u, info = g.iterative_solve(inst['nom_s'], inst['nom_u'], ref, inst['ref_speed'], list(inst['obstacles']))
    np.testing.assert_allclose(u, fx['u'], atol=TRAJ_TOL)
    np.testing.assert_allclose(np.hstack(info['opt_state_list']), fx['s'], atol=TRAJ_TOL)


def test_cuda_graph_capture_replays_identically():
    """rda_solve enqueues only kernels on the caller's stream (no sync, no allocation): it can be
    captured in a CUDA graph and replayed."""
    from rda_planner_b200.rda_solver import RDA_solver
    T, N, B = 12, 6, 64
    car = rectangle_robot()
    insts, inp = _batch_inputs(B, T, N, 700, lateral=(0.5, 3.5))
    g = RDA_solver(T, car, 4, N, iter_num=5, iter_threshold=0.0, time_print=False, batch=B)
    dev = {k: torch.as_tensor(v, device='cuda', dtype=torch.int32 if 'kind' in k or 'count' in k else torch.float32)
           for k, v in inp.items()}
    eager = {k: v.clone() for k, v in g.iterative_solve_batch(**dev).items()}
    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream):
        g.cold_start()
        g.iterative_solve_batch(**dev)               # warm-up on the side stream
        stream.synchronize()
        with torch.cuda.graph(graph, stream=stream):
            g.cold_start()
            out = g.iterative_solve_batch(**dev)
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out['u'], eager['u']) and torch.equal(out['s'], eager['s'])


@pytest.mark.parametrize('kind,moving', [('polygon', False), ('circle', True)])
def test_two_stream_split_is_invisible(monkeypatch, kind, moving):
    """rda_solve runs large batches as two halves on two streams (fork/join by events).  Forced here
    on a small odd batch (RDA_B200_SPLIT_MIN): outputs and persistent state must be bit-identical to
    the single-stream order, eagerly and when captured in a CUDA graph."""
    from rda_planner_b200.rda_solver import RDA_solver
    from rda_planner_b200 import _cabi
    T, N, B = 12, 6, 37
    monkeypatch.setenv('RDA_B200_SMALL', '0')          # the streaming kernels, not the single-launch path of small batches
    car = rectangle_robot()
    insts, inp = _batch_inputs(B, T, N, 1500, lateral=(0.3, 3.5), kind=kind, moving=moving)
    dev = {k: torch.as_tensor(v, device='cuda', dtype=torch.int32 if 'kind' in k or 'count' in k else torch.float32)
           for k, v in inp.items()}
    res = {}
    for name, split_min, parts in (('whole', '1000000', '2'), ('split', '2', '2'), ('split3', '2', '3')):
        monkeypatch.setenv('RDA_B200_SPLIT_MIN', split_min)
        monkeypatch.setenv('RDA_B200_SPLIT_PARTS', parts)
        g = RDA_solver(T, car, 4, N, iter_num=5, iter_threshold=0.0, time_print=False, batch=B)
        out = {k: v.clone() for k, v in g.iterative_solve_batch(**dev, time_varying=moving).items()}
        out2 = {k: v.clone() for k, v in g.iterative_solve_batch(**dev, time_varying=moving).items()}     # warm-started second call
        state = {b: g.state_buffer(b).clone() for b in (_cabi.BUF_LAM, _cabi.BUF_MU, _cabi.BUF_Z, _cabi.BUF_XI,
                                                        _cabi.BUF_ZETA, _cabi.BUF_DIS)}
        res[name] = (out, out2, state, g)
    assert res['split'][3].launch_count() > 1.9 * res['whole'][3].launch_count() - 4
    for name in ('split', 'split3'):
        for call in (0, 1):
            w, sp = res['whole'][call], res[name][call]
            for k in ('u', 's', 'status', 'iters'):
                assert torch.equal(w[k], sp[k]), (name, call, k, float((w[k].float() - sp[k].float()).abs().max()))
            for k in ('resi_pri', 'resi_dual'):     # float atomics: summation order is not fixed
                assert torch.allclose(w[k], sp[k], rtol=1e-4, atol=1e-6), (name, call, k)
        for b in res['whole'][2]:
            assert torch.equal(res['whole'][2][b], res[name][2][b]), (name, b)
    g = res['split'][3]
    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream):
        g.cold_start()
        g.iterative_solve_batch(**dev, time_varying=moving)
        stream.synchronize()
        with torch.cuda.graph(graph, stream=stream):
            g.cold_start()
            out = g.iterative_solve_batch(**dev, time_varying=moving)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out['u'], res['whole'][0]['u']) and torch.equal(out['s'], res['whole'][0]['s'])


def test_float32_su_mode_and_residual_gap():
    """BASELINE configs[4] asks for a float32-vs-float64 comparison: su-QP interior point in float32
    (su_fp64=False) against the default float64 arithmetic on the same instances."""
    from rda_planner_b200.rda_solver import RDA_solver
    T, N, B = 20, 10, 128
    car = rectangle_robot()
    insts, inp = _batch_inputs(B, T, N, 800)
    out = {}
    for fp64 in (True, False):
        g = RDA_solver(T, car, 4, N, iter_num=6, iter_threshold=0.0, time_print=False, batch=B, su_fp64=fp64)
        out[fp64] = {k: v.clone() for k, v in g.iterative_solve_batch(**inp).items()}
    gap = (out[True]['u'] - out[False]['u']).abs().flatten(1).max(1).values
    assert torch.isfinite(out[False]['u']).all()
    assert float(gap.median()) < 5e-3
    rp = (out[True]['resi_pri'] - out[False]['resi_pri']).abs() / (1 + out[True]['resi_pri'])
    assert float(rp.median()) < 1e-2


def test_large_polytopes_config():
    """BASELINE configs[3]/[4] shapes: convex hulls with up to 8 faces, T=40, N=32 (E=8 code paths,
    two stages per lane in the su kernel); GPU against the compiled CPU port of the same cores."""
    from rda_planner_b200.rda_solver import RDA_solver, pack_obstacles
    from oracle import cpu_port
    T, N, E, B, iters = 40, 32, 8, 8, 4
    car = rectangle_robot()
    insts = [make_instance(900 + i, T=T, N=N, E=E, lateral=(1.0, 8.0)) for i in range(B)]
    packs = [pack_obstacles(list(i['obstacles']), T, N, E) for i in insts]
    inp = dict(nom_s=np.stack([i['nom_s'] for i in insts]), nom_u=np.stack([i['nom_u'] for i in insts]),
               ref_s=np.stack([i['ref'] for i in insts]), ref_speed=np.array([i['ref_speed'] for i in insts]),
               obs_A=np.stack([p[0] for p in packs]), obs_b=np.stack([p[1] for p in packs]),
               obs_kind=np.stack([p[2] for p in packs]), obs_count=np.array([p[3] for p in packs]))
    g = RDA_solver(T, car, E, N, iter_num=iters, iter_threshold=0.0, time_print=False, batch=B, slack_gain=13)
    out = g.iterative_solve_batch(**inp)
    port = cpu_port.solve_batch(car, T, N, E, **inp, iter_num=iters, slack_gain=13)
    assert int((out['status'] & 6).sum()) == 0
    np.testing.assert_allclose(out['u'].cpu().numpy(), port['u'], atol=3 * TRAJ_TOL)
    np.testing.assert_allclose(out['s'].cpu().numpy(), port['s'], atol=3 * TRAJ_TOL)


def test_coherent_first_pass_matches_the_search_pass(monkeypatch):
    """RDA_B200_LEAN2=1 (cell_lean2.cuh: cached support-vertex pair + separating-slab certificate, per-obstacle
    precomputed geometry) against the default search pass on the same batch.  The two differ at float
    rounding level per cell, so the comparison is made after few iterations; the coherent pass must
    actually resolve most cells from the second iteration on."""
    from rda_planner_b200.rda_solver import RDA_solver
    from rda_planner_b200 import _cabi
    T, N, B, iters = 12, 6, 96, 4
    monkeypatch.setenv('RDA_B200_SMALL', '0')
    car = rectangle_robot()
    insts, inp = _batch_inputs(B, T, N, 2500, lateral=(1.0, 5.0))
    res = {}
    for flag in ('0', '1'):
        monkeypatch.setenv('RDA_B200_LEAN2', flag)
        g = RDA_solver(T, car, 4, N, iter_num=iters, iter_threshold=0.0, time_print=False, batch=B)
        res[flag] = ({k: v.clone() for k, v in g.iterative_solve_batch(**inp).items()}, g.launch_count())
    assert res['1'][1] > res['0'][1]                       # extra launches of the coherent pipeline
    assert int((res['1'][0]['status'] & 7).sum()) == 0
    du = (res['0'][0]['u'] - res['1'][0]['u']).abs().flatten(1).max(1).values
    assert float(du.median()) < 2e-5 and float(du.max()) < 3 * TRAJ_TOL


def test_graph_replay_of_the_single_instance_api():
    """RDA_solver(graph=True): the reference-signature call stages its inputs in persistent device buffers and replays
    one CUDA graph per control step; results and warm-start evolution must be bit-identical to eager launches."""
    from rda_planner_b200.rda_solver import RDA_solver
    T, N = 10, 5
    car = rectangle_robot()
    gs = [RDA_solver(T, car, 4, N, iter_num=4, iter_threshold=0.0, time_print=False, graph=g) for g in (False, True)]
    for k in range(4):
        inst = make_instance(40 + k, T=T, N=N, E=4, lateral=(0.3, 3.0))
        ref = [inst['ref'][:, t:t + 1] for t in range(T + 1)]
        outs = [g.iterative_solve(inst['nom_s'], inst['nom_u'], ref, 4.0, list(inst['obstacles'])) for g in gs]
        assert np.array_equal(outs[0][0], outs[1][0]), k
        assert np.array_equal(np.hstack(outs[0][1]['opt_state_list']), np.hstack(outs[1][1]['opt_state_list']))
        assert abs(outs[0][1]['resi_pri'] - outs[1][1]['resi_pri']) <= 1e-5 * (1 + outs[0][1]['resi_pri'])
    assert len(gs[1]._graphs) == 1


@pytest.mark.parametrize('kind,moving,dyn,N,fp64', [('polygon', False, 'acker', 6, True), ('circle', True, 'diff', 5, True),
                                                     ('polygon', False, 'omni', 0, True), ('polygon', False, 'acker', 6, False)])
def test_persistent_small_kernel_equals_streaming_kernels(monkeypatch, kind, moving, dyn, N, fp64):
    """SURVEY §8 f4: small batches run the whole ADMM loop in ONE launch, one CTA per instance, state in shared memory
    (k_admm_small).  Same device functions as the streaming kernels: trajectories, residuals, early stop and the
    persistent warm-start state must agree to float32 rounding, cold and warm-started."""
    from rda_planner_b200.rda_solver import RDA_solver
    from rda_planner_b200 import _cabi
    T, B = 10, 9
    car = rectangle_robot(dynamics=dyn)
    insts, inp = _batch_inputs(B, T, max(N, 1), 3100, lateral=(0.3, 3.5), kind=kind, moving=moving, dynamics=dyn)
    dev = {k: torch.as_tensor(v, device='cuda', dtype=torch.int32 if 'kind' in k or 'count' in k else torch.float32)
           for k, v in inp.items()}
    if N == 0:
        dev = {k: v for k, v in dev.items() if not k.startswith('obs_')}
    res = {}
    for mode in ('0', '1'):
        monkeypatch.setenv('RDA_B200_SMALL', mode)
        g = RDA_solver(T, car, 4, N, iter_num=6, iter_threshold=0.3, time_print=False, batch=B, su_fp64=fp64)
        out = {k: v.clone() for k, v in g.iterative_solve_batch(**dev, time_varying=moving).items()}
        out2 = {k: v.clone() for k, v in g.iterative_solve_batch(**dev, time_varying=moving).items()}
        bufs = (_cabi.BUF_DIS, _cabi.BUF_CUR_S) if N == 0 else (_cabi.BUF_LAM, _cabi.BUF_MU, _cabi.BUF_Z, _cabi.BUF_XI, _cabi.BUF_ZETA,
                                                               _cabi.BUF_DIS, _cabi.BUF_COEF)
        state = {b: g.state_buffer(b).clone() for b in bufs}
        res[mode] = (out, out2, state, g.launch_count())
    assert res['1'][3] == 1 and res['0'][3] > 5
    for call in (0, 1):
        a, b = res['0'][call], res['1'][call]
        if fp64:
            assert torch.equal(a['iters'], b['iters']), (call, a['iters'], b['iters'])
            assert torch.equal(a['status'], b['status'])
        else:       # float32 su-QP (looser interior point tolerances): same code in both paths, only finiteness and closeness
            assert float((a['u'] - b['u']).abs().max()) < 5e-3 and int((b['status'] & 6).sum()) == 0
            continue
        # the streaming path resolves most cells in the lean first pass, the single-launch kernel in the general closed
        # forms: same arithmetic step by step but not the same rounding, amplified by the warm-started second call
        for k in ('u', 's'):
            # (6.5e-5 on positions of ~20 m was seen after 6 iterations: 30 ulps; the parity tolerance to the oracle is 1e-3)
            assert float((a[k] - b[k]).abs().max()) < (1e-4 if call == 0 else 5e-4), (call, k, float((a[k] - b[k]).abs().max()))
        for k in ('resi_pri', 'resi_dual'):
            assert torch.allclose(a[k], b[k], rtol=1e-3, atol=1e-4), (call, k)
    for k in res['0'][2]:
        assert float((res['0'][2][k] - res['1'][2][k]).abs().max()) < (1e-3 if fp64 else 5e-2), k

