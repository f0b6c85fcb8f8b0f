"""Plan clearance on the device (rda_plan_clearance, RDA_solver.plan_clearance, BatchedMPC.control(clearance=True)): the
kernel against the float64 reference on random cells with static and time-varying obstacle copies, the minimum and its
index against numpy on the kernel's own map (padding, obs_count 0 and > N), robot classes against one handle per class,
bitwise repeatability and CUDA-graph replay, a control step without host synchronisation, usage errors, the two robots
at a crossing, and a fleet at the bench's closed-loop shape against the host separating-axis test."""
import ctypes as C

import numpy as np
import pytest
import torch

import clearance_cases as cc
from oracle import clearance as ref
from rda_planner_b200 import _cabi
from rda_planner_b200.frontend import BatchedMPC
from rda_planner_b200.rda_solver import RDA_solver
from rda_planner_b200.scenarios import rectangle_robot
from test_gpu_fleet_obstacles import CROSS, DT, _corners, _line, _overlap

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


def _solver(car, B, T, N, E):
    return RDA_solver(T, car, max_edge_num=E, max_obs_num=N, iter_num=1, iter_threshold=0.0, time_print=False, batch=B,
                      device=DEV)


def _batch(rng, car, B, N, T, tv, E=cc.E):
    """Inputs of a batch built from random cells: pose (b, t) of one cell each, obstacle copies re-based from other cells
    onto the pose they are paired with.  Returns s [B, 3, T+1] and obs_A, obs_b, obs_kind (float32 / int32)."""
    T1, Tc = T + 1, T + 1 if tv else 1
    kinds, A, b, pose, _ = cc.random_cells(rng, car, B * T1)
    s = pose.reshape(B, T1, 3).transpose(0, 2, 1).copy()
    fits = np.nonzero((np.linalg.norm(A, axis=2) > 0).sum(1) <= E)[0]      # obstacles of at most E rows
    oA = np.zeros((B, N, Tc, E, 2), np.float32)
    ob = np.zeros((B, N, Tc, E), np.float32)
    ok = np.zeros((B, N), np.int32)
    for bb in range(B):
        for o in range(N):
            src0 = int(rng.choice(fits))
            for c in range(Tc):
                src = src0 if c == 0 or rng.random() < 0.3 else int(rng.choice(fits))
                src = src if kinds[src] == kinds[src0] else src0          # one kind per slot
                d = s[bb, :2, c].astype(float) - pose[src, :2].astype(float)
                oA[bb, o, c] = A[src, :E]
                ob[bb, o, c] = cc._moved(kinds[src], A[src, :E].astype(float), b[src, :E].astype(float), d)
            ok[bb, o] = kinds[src0]
    return s, oA, ob, ok


def _begin(g, s, oA, ob, ok, count, tv):
    B, _, T1 = s.shape
    g.begin(s, np.zeros((B, 2, T1 - 1), np.float32), s, np.zeros(B, np.float32), oA, ob, ok, count, tv)


@pytest.mark.parametrize('name', ['rect_rear', 'triangle_out', 'octagon', 'disc_offset'])
@pytest.mark.parametrize('tv', [False, True])
def test_kernel_matches_reference(name, tv):
    car = cc.bodies()[name]
    B, N, T = 6, 5, 6
    rng = np.random.default_rng(sum(map(ord, name)) + tv)
    s, oA, ob, ok = _batch(rng, car, B, N, T, tv)
    count = np.array([N, 3, N + 4, 1, N, 2], np.int32)
    g = _solver(car, B, T, N, cc.E)
    _begin(g, s, oA, ob, ok, count, tv)
    out = g.plan_clearance(s, per_cell=True)
    got = out['map'].cpu().numpy()
    G, h, cone = cc.body_rows(car)
    want = ref.plan_clearance(ref.body_from_halfspaces(G, h, cone == _cabi.ROBOT_DISC), s, oA, ob, ok, count, tv)
    fin = np.isfinite(want)
    assert np.array_equal(fin, np.isfinite(got))
    err = np.abs(got[fin] - want[fin]) / np.maximum(1.0, np.abs(want[fin]))
    assert err.max() < 2e-6, err.max()
    assert (want[fin] < 0).any() and (want[fin] > 0).any()


def _argmin(m):
    """(min, index) of each row of a [B, N, T+1] map as rda_plan_clearance defines them."""
    flat = m.reshape(m.shape[0], -1)
    if flat.shape[1] == 0:
        return np.full(m.shape[0], np.inf, np.float32), np.full(m.shape[0], -1, np.int32)
    i = np.argmin(flat, 1)
    v = flat[np.arange(len(flat)), i]
    return v, np.where(np.isfinite(v), i, -1).astype(np.int32)


@pytest.mark.parametrize('tv', [False, True])
def test_min_and_index_are_exact(tv):
    car = rectangle_robot()
    B, N, T = 12, 4, 5
    rng = np.random.default_rng(3 + tv)
    s, oA, ob, ok = _batch(rng, car, B, N, T, tv, E=4)
    count = np.array([0, 1, 2, N, N + 1, 100, -3, N, 3, 1, 0, N], np.int32)
    # ties: the same obstacle in every slot of instance 3 gives equal values, the smallest index (slot 0) wins
    oA[3], ob[3], ok[3] = oA[3, :1], ob[3, :1], ok[3, :1]
    g = _solver(car, B, T, N, 4)
    _begin(g, s, oA, ob, ok, count, tv)
    out = g.plan_clearance(s, per_cell=True)
    m = out['map'].cpu().numpy()
    v, i = _argmin(m)
    assert np.array_equal(out['min'].cpu().numpy(), v)
    assert np.array_equal(out['index'].cpu().numpy(), i)
    valid = np.minimum(np.maximum(count, 0), N)
    for bb in range(B):
        assert np.isinf(m[bb, valid[bb]:]).all() and np.isfinite(m[bb, :valid[bb]]).all()
    assert i[0] == -1 and np.isinf(v[0]) and i[6] == -1 and i[10] == -1
    assert np.array_equal(m[3, 0], m[3, 3]) and i[3] < T + 1
    # without the map, the same minimum
    out2 = g.plan_clearance(s)
    assert 'map' not in out2 and torch.equal(out2['min'], out['min']) and torch.equal(out2['index'], out['index'])


def test_classes_match_one_handle_per_class():
    bodies = cc.bodies()
    base = bodies['rect_rear']
    classes = [bodies['rect_centred'], bodies['omni_centred'], bodies['offset_box']]
    B, N, T = 16, 4, 5
    rng = np.random.default_rng(11)
    s, oA, ob, ok = _batch(rng, base, B, N, T, True, E=4)
    count = np.full(B, N, np.int32)
    cls = (np.arange(B) % 5 - 1).astype(np.int64)                         # -1 and 3: the handle's own body
    g = _solver(base, B, T, N, 4)
    g.set_robot_classes(classes, cls)
    _begin(g, s, oA, ob, ok, count, True)
    got = g.plan_clearance(s, per_cell=True)
    for k, car in enumerate(classes + [base]):
        h = _solver(car, B, T, N, 4)
        _begin(h, s, oA, ob, ok, count, True)
        want = h.plan_clearance(s, per_cell=True)
        rows = np.nonzero((cls == k) if k < len(classes) else ((cls < 0) | (cls >= len(classes))))[0]
        for key in ('map', 'min', 'index'):
            assert torch.equal(got[key][rows], want[key][rows]), (k, key)


def test_repeatable_and_graph_replay():
    car = cc.bodies()['hexagon']
    B, N, T = 64, 6, 8
    rng = np.random.default_rng(4)
    s, oA, ob, ok = _batch(rng, car, B, N, T, False)
    count = rng.integers(0, N + 2, B).astype(np.int32)
    g = _solver(car, B, T, N, cc.E)
    _begin(g, s, oA, ob, ok, count, False)
    st = torch.as_tensor(s, device=DEV)
    a = g.plan_clearance(st, per_cell=True)
    b = g.plan_clearance(st, per_cell=True)
    for k in a:
        assert torch.equal(a[k], b[k])
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            c = g.plan_clearance(st, per_cell=True)
    torch.cuda.current_stream().wait_stream(side)
    for k in c:
        c[k].fill_(7)
    graph.replay()
    torch.cuda.synchronize()
    for k in a:
        assert torch.equal(a[k], c[k]), k


def test_usage_errors():
    car = rectangle_robot()
    g = _solver(car, 2, 4, 3, 4)
    with pytest.raises(RuntimeError):
        g.plan_clearance()                          # no solve yet
    s = np.zeros((2, 3, 5), np.float32)
    oA, ob = np.zeros((2, 3, 1, 4, 2), np.float32), np.zeros((2, 3, 1, 4), np.float32)
    _begin(g, s, oA, ob, np.zeros((2, 3), np.int32), np.zeros(2, np.int32), False)
    with pytest.raises(ValueError):
        g.plan_clearance(np.zeros((2, 3, 4), np.float32))
    lib, vp = g.lib, C.c_void_p
    t = {k: torch.zeros(n, device=DEV) for k, n in (('s', 30), ('d', 30), ('m', 2))}
    idx = torch.zeros(2, dtype=torch.int32, device=DEV)
    inp = _cabi.Inputs()
    for k in ('obs_A', 'obs_b', 'obs_kind', 'obs_count'):
        setattr(inp, k, g._keep[k].data_ptr())
    p = lambda x: vp(x.data_ptr())
    ok = lambda h, i, s_, d, m, ix: lib.rda_plan_clearance(h, i, s_, d, m, ix, None)
    assert ok(g._h, C.byref(inp), p(t['s']), p(t['d']), p(t['m']), p(idx)) == 0
    assert ok(None, C.byref(inp), p(t['s']), None, p(t['m']), p(idx)) == _cabi.E_ARG
    assert ok(g._h, None, p(t['s']), None, p(t['m']), p(idx)) == _cabi.E_ARG
    assert ok(g._h, C.byref(inp), None, None, p(t['m']), p(idx)) == _cabi.E_ARG
    assert ok(g._h, C.byref(inp), p(t['s']), None, None, p(idx)) == _cabi.E_ARG
    assert ok(g._h, C.byref(inp), p(t['s']), None, p(t['m']), None) == _cabi.E_ARG
    for k in ('obs_A', 'obs_b', 'obs_kind', 'obs_count'):
        bad = _cabi.Inputs()
        for j in ('obs_A', 'obs_b', 'obs_kind', 'obs_count'):
            setattr(bad, j, None if j == k else g._keep[j].data_ptr())
        assert ok(g._h, C.byref(bad), p(t['s']), None, p(t['m']), p(idx)) == _cabi.E_ARG, k
    torch.cuda.synchronize()


def test_control_with_clearance_needs_no_host_sync():
    car = rectangle_robot()
    B = 32
    paths = [_line(0.0, -1.0, 0.0, 50), _line(0.0, 2.5, 0.05, 50)]
    bm = BatchedMPC(car, paths, B, robot_path=np.arange(B) % 2, receding=8, iter_num=2, max_edge_num=4, max_obs_num=4)
    state = torch.as_tensor(np.stack([[0.3 * (b % 16), 0.0, 0.0] for b in range(B)]), dtype=torch.float32, device=DEV)
    twin = BatchedMPC(car, paths, B, robot_path=np.arange(B) % 2, receding=8, iter_num=2, max_edge_num=4, max_obs_num=4)
    for m in (bm, twin):                      # the first call uploads the empty map
        m.control(state, 2.0, avoid_fleet=True)
    u_plain, info_plain = twin.control(state, 2.0, avoid_fleet=True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        u0, info = bm.control(state, 2.0, avoid_fleet=True, clearance=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert 'clearance' not in info_plain
    assert torch.equal(u0, u_plain) and torch.equal(info['s'], info_plain['s'])     # the plan itself does not change
    c = bm.rda.plan_clearance(per_cell=True)
    assert torch.equal(info['clearance'], c['min']) and torch.equal(info['clearance_index'], c['index'])


def test_crossing_stage0_clearance_is_the_body_distance():
    """The two robots of the crossing (tests/test_gpu_fleet_obstacles.py) with avoid_fleet=True: at every step the
    stage-0 clearance of each robot to its map-mate is the polygon distance of the two bodies there."""
    car = rectangle_robot(length=2.0, width=1.0, wheelbase=1.2, dynamics='diff', max_speed=(3, 1.5), max_acce=(3, 1.5))
    L, L1 = CROSS['start'], CROSS['start'] + CROSS['lag']
    n = int(4 * L / 0.25)
    paths = [_line(-L, 0.0, 0.0, n, step=0.25), _line(0.0, -L1, np.pi / 2, n, step=0.25)]
    bm = BatchedMPC(car, paths, 2, robot_path=[0, 1], receding=12, sample_time=DT, iter_num=4, max_edge_num=4,
                    max_obs_num=3, iter_threshold=0.0)
    state = torch.as_tensor(np.array([[-L, 0.0, 0.0], [0.0, -L1, np.pi / 2]], np.float32), device=DEV)
    body = dict(bm.body, xy=bm.body['xy'].cpu().numpy())
    closest = np.inf
    for _ in range(CROSS['steps']):
        now = state.cpu().numpy().astype(float)
        _, info = bm.control(state, CROSS['speed'], time_varying=True, avoid_fleet=True, clearance=True)
        m = bm.rda.plan_clearance(per_cell=True)['map'].cpu().numpy()
        s = info['s'].cpu().numpy().astype(float)
        for b in range(2):
            want = ref.polygons(_corners(body, s[b, :, 0]), _corners(body, now[1 - b]))
            assert abs(m[b, 0, 0] - want) < 1e-4 * max(1.0, abs(want)), (b, m[b, 0, 0], want)
            assert np.isinf(m[b, 1:]).all()                  # one map-mate, in slot 0
            closest = min(closest, want)
        assert np.array_equal(info['clearance'].cpu().numpy(), m.reshape(2, -1).min(1))
        bm.advance(state)
    assert 0 < closest < 2.0                                 # they did come close


def test_fleet_at_the_bench_closed_loop_shape_agrees_with_host_sat():
    T, N, E, B = 30, 20, 4, 16384
    rng = np.random.default_rng(77)
    path = np.stack([np.arange(0, 60, 0.1), np.zeros(600), np.zeros(600)], 1)
    bm = BatchedMPC(rectangle_robot(), path, B, receding=T, sample_time=0.1, iter_num=50, max_edge_num=E,
                    max_obs_num=N, iter_threshold=0.0, device=DEV)
    idx = rng.integers(0, 480, B)
    state = torch.as_tensor(path[idx] + rng.normal(0, [0.3, 0.3, 0.1], (B, 3)), dtype=torch.float32, device=DEV)
    bm.cur_index[:] = torch.as_tensor(np.maximum(idx - 3, 0), dtype=torch.int32)
    bm.cur_vel[:, 0, :] = 4.0
    ctr = path[idx][:, None, :2] + np.stack([rng.uniform(2, 14, (B, N)), rng.uniform(-3, 3, (B, N))], -1)
    yaw = rng.uniform(0, np.pi, (B, N))
    corners = np.array([[-1, -0.5], [1, -0.5], [1, 0.5], [-1, 0.5]])
    rot = np.stack([np.stack([np.cos(yaw), -np.sin(yaw)], -1), np.stack([np.sin(yaw), np.cos(yaw)], -1)], -2)
    xy = np.zeros((B, N, 8, 2), np.float32)
    xy[:, :, :4] = ctr[:, :, None, :] + np.einsum('bmij,kj->bmki', rot, corners)
    shapes = {'kind': np.zeros((B, N), np.int32), 'nv': np.full((B, N), 4, np.int32), 'xy': xy,
              'radius': np.zeros((B, N), np.float32), 'vel': np.zeros((B, N, 2), np.float32),
              'count': np.full(B, N, np.int32)}
    shapes = {k: torch.as_tensor(v, device=DEV) for k, v in shapes.items()}
    body = dict(bm.body, xy=bm.body['xy'].cpu().numpy())
    checked = 0
    for step in range(2):
        _, info = bm.control(state, 4.0, shapes, clearance=True)
        c = bm.rda.plan_clearance(per_cell=True)
        m, s = c['map'].cpu().numpy(), info['s'].cpu().numpy()
        A, b = (bm.rda._keep[k].cpu().numpy() for k in ('obs_A', 'obs_b'))
        assert np.array_equal(info['clearance'].cpu().numpy(), m.reshape(B, -1).min(1))
        for r in rng.choice(B, 48, replace=False):
            for o in range(N):
                Q = ref.obstacle_polygon(A[r, o, 0], b[r, o, 0])[0]
                for t in range(0, T + 1, 3):
                    d = m[r, o, t]
                    if abs(d) < 1e-4:
                        continue
                    hit = _overlap(_corners(body, s[r, :, t].astype(float)), Q)
                    assert hit == (d < 0), (step, r, o, t, d)
                    checked += 1
        bm.advance(state)
    assert checked > 10000
