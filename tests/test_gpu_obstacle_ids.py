"""Warm start that follows the obstacles on the device (rda_set_obstacle_ids, the rda_convert_*_ids calls,
BatchedMPC(warm_start='obstacle')): the remap kernel against the numpy rule bit for bit; solves whose slots are permuted
at every call against solves in a stable order, on every routing; the id conversions against the existing calls and the
twins' selection; the float64 oracle with its warm start remapped alike; and a captured graph against eager calls."""
import numpy as np
import pytest
import torch

import obstacle_ids_twin as oi
from test_obstacle_ids import _world
from oracle.rda_oracle import OracleRDA
from rda_planner_b200 import _cabi
from rda_planner_b200.frontend import (BatchedMPC, convert_fleet_obstacles_batch, convert_obstacles_batch,
                                       convert_world_obstacles_batch, convert_world_obstacles_horizon_batch,
                                       fleet_plan_shapes_batch, fleet_shapes_batch, pack_shapes, pack_worlds,
                                       robot_body, shapes_to_device)
from rda_planner_b200.rda_solver import RDA_solver, pack_obstacles
from rda_planner_b200.scenarios import disc_robot, make_instance, rectangle_robot

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
DT = float(np.float32(0.1))
SLOT_BUFS = {'LAM': (_cabi.BUF_LAM, 'E'), 'MU': (_cabi.BUF_MU, 'R'), 'Z': (_cabi.BUF_Z, 1), 'XI': (_cabi.BUF_XI, 'xi'),
             'ZETA': (_cabi.BUF_ZETA, 1), 'COEF': (_cabi.BUF_COEF, 'coef')}
INSTANCE_BUFS = {'DIS': _cabi.BUF_DIS, 'PREF': _cabi.BUF_PREF, 'CUR_S': _cabi.BUF_CUR_S, 'CUR_U': _cabi.BUF_CUR_U}


def _t(a, dtype=None):
    return torch.as_tensor(np.asarray(a), device=DEV, dtype=dtype).contiguous()


def _slot_view(x, kind, B, N, T, E, R):
    """A slot-indexed buffer as [B, N, ...] (slot axis second)."""
    if kind == 'E':
        return x.reshape(B, N, E * T)
    if kind == 'R':
        return x.reshape(B, N, R * T)
    if kind == 1:
        return x.reshape(B, N, T)
    planes = 2 if kind == 'xi' else 5
    return np.moveaxis(x.reshape(B, planes, N, T), 1, 2).reshape(B, N, planes * T)


@pytest.mark.parametrize('N,E,disc', [(5, 4, False), (20, 4, False), (7, 8, True), (256, 3, False), (300, 3, False)])
def test_remap_kernel_is_the_numpy_rule_bit_for_bit(N, E, disc):
    check_remap_kernel(48, 6, N, E, disc, N + E)


def check_remap_kernel(B, T, N, E, disc, seed):
    """k_remap_slots on random slot states and random id lists against the numpy rule of obstacle_ids_twin, bit for bit."""
    rng = np.random.default_rng(seed)
    car = disc_robot() if disc else rectangle_robot()
    g = RDA_solver(T, car, max_edge_num=E, max_obs_num=N, iter_num=1, time_print=False, batch=B, device=DEV)
    R = 3 if disc else 4
    before = {}
    for name, bid in list((k, v[0]) for k, v in SLOT_BUFS.items()) + list(INSTANCE_BUFS.items()):
        v = rng.standard_normal(g.buffer_count(bid)).astype(np.float32)
        g.load_state_buffer(bid, v)
        before[name] = v
    prev = np.stack([rng.integers(-1, N + 3, N) for _ in range(B)]).astype(np.int32)
    cur = np.stack([rng.integers(-1, N + 3, N) for _ in range(B)]).astype(np.int32)
    cur[0] = prev[0]                                              # an instance whose slots keep their state
    cur[1, N // 2:] = cur[1, N // 2 - 1] if N > 1 else cur[1]     # a padded tail
    launches = g.launch_count()
    g.set_obstacle_ids(prev)                                      # stores only
    for name, (bid, _) in SLOT_BUFS.items():
        np.testing.assert_array_equal(g.state_buffer(bid).cpu().numpy(), before[name])
    g.set_obstacle_ids(cur)
    torch.cuda.synchronize()
    assert g.launch_count() == launches
    for name, (bid, kind) in SLOT_BUFS.items():
        got = _slot_view(g.state_buffer(bid).cpu().numpy(), kind, B, N, T, E, R)
        old = _slot_view(before[name], kind, B, N, T, E, R)
        for b in range(B):
            want = oi.remap(old[b], oi.slot_source(prev[b], cur[b]))
            np.testing.assert_array_equal(got[b], want, err_msg=f'{name} instance {b}')
    for name, bid in INSTANCE_BUFS.items():
        np.testing.assert_array_equal(g.state_buffer(bid).cpu().numpy(), before[name])
    # None forgets: the next call stores again and moves nothing
    g.set_obstacle_ids(None)
    snap = {name: g.state_buffer(bid).clone() for name, (bid, _) in SLOT_BUFS.items()}
    g.set_obstacle_ids(prev)
    for name, (bid, _) in SLOT_BUFS.items():
        assert torch.equal(g.state_buffer(bid), snap[name])


def _instances(U, T, N, E, kind='polygon'):
    insts = [make_instance(700 + i, T=T, N=N, E=E, lateral=(0.3, 3.0), **({'kind': 'circle', 'moving': True}
                                                                           if kind == 'moving' else {}))
             for i in range(U)]
    tv = kind == 'moving'
    packs = [pack_obstacles(list(i['obstacles']), T, N, E) for i in insts]
    A = np.stack([p[0] for p in packs])
    if tv and A.shape[2] == 1:
        A = np.repeat(A, T + 1, axis=2)
    bb = np.stack([p[1] for p in packs])
    if tv and bb.shape[2] == 1:
        bb = np.repeat(bb, T + 1, axis=2)
    return dict(nom_s=np.stack([i['nom_s'] for i in insts]).astype(np.float32),
                nom_u=np.stack([i['nom_u'] for i in insts]).astype(np.float32),
                ref_s=np.stack([i['ref'] for i in insts]).astype(np.float32),
                ref_speed=np.array([i['ref_speed'] for i in insts], np.float32),
                obs_A=A.astype(np.float32), obs_b=bb.astype(np.float32), obs_kind=np.stack([p[2] for p in packs]),
                obs_count=np.array([p[3] for p in packs], np.int32)), tv


@pytest.mark.parametrize('B,body,kind', [(64, 'polygon', 'static'), (64, 'polygon', 'moving'), (1024, 'polygon', 'static'),
                                         (1024, 'disc', 'static'), (1024, 'polygon', 'moving'), (4096, 'polygon', 'static'),
                                         (8192, 'polygon', 'static'), (1024, 'polygon', 'early_stop')])
def test_permuted_slots_with_ids_solve_as_the_stable_order(B, body, kind):
    # 'early_stop': the reference's early-stop rule, with a threshold (1.0) that stops these instances within the same 8
    # iterations, so that the iteration counts compared below are the instances' own
    T, N, E, calls = 30, 20, 4, 3
    iters, thr = (8, 1.0) if kind == 'early_stop' else (8, 0.0)
    U = 64
    base, tv = _instances(U, T, N, E, 'moving' if kind == 'moving' else 'polygon')
    inp = {k: v[np.arange(B) % U] for k, v in base.items()}
    assert (inp['obs_count'] == N).all()                          # no padding: every slot holds its own obstacle
    car = disc_robot() if body == 'disc' else rectangle_robot()
    mk = lambda: RDA_solver(T, car, max_edge_num=E, max_obs_num=N, iter_num=iters, iter_threshold=thr,
                            time_print=False, batch=B, device=DEV)
    stable, moved = mk(), mk()
    rng = np.random.default_rng(B)
    dev = {k: _t(v) for k, v in inp.items()}
    worst_u = worst_s = 0.0
    for call in range(calls):
        perm = np.stack([rng.permutation(N) for _ in range(B)]) if call else np.tile(np.arange(N), (B, 1))
        pidx = torch.as_tensor(perm, device=DEV, dtype=torch.long)
        gather = lambda x: torch.gather(x, 1, pidx.reshape(B, N, *([1] * (x.dim() - 2))).expand_as(x)).contiguous()
        pd = dict(dev, obs_A=gather(dev['obs_A']), obs_b=gather(dev['obs_b']), obs_kind=gather(dev['obs_kind']))
        a = {k: v.clone() for k, v in stable.iterative_solve_batch(**dev, time_varying=tv).items()}
        moved.set_obstacle_ids(_t(perm, torch.int32))
        m = {k: v.clone() for k, v in moved.iterative_solve_batch(**pd, time_varying=tv).items()}
        torch.cuda.synchronize()
        assert torch.equal(a['status'], m['status']), call
        assert torch.equal(a['iters'], m['iters']), call
        worst_u = max(worst_u, float((a['u'] - m['u']).abs().max()))
        worst_s = max(worst_s, float((a['s'] - m['s']).abs().max()))
    print(f'B={B} {body} {kind}: max |du| {worst_u:.3g}, max |ds| {worst_s:.3g}, mean iterations '
          f'{float(a["iters"].float().mean()):.2f}')
    if kind == 'early_stop':
        assert len(torch.unique(a['iters'])) > 1 and int(a['iters'].min()) < iters   # stopped by the rule, at various counts
    assert worst_s < 1e-3 and worst_u < 1e-2, (worst_s, worst_u)


def test_oracle_with_remapped_warm_start_follows_the_device():
    T, N, E, iters, U = 10, 4, 4, 4, 3
    base, _ = _instances(U, T, N, E)
    car = rectangle_robot()
    g = RDA_solver(T, car, max_edge_num=E, max_obs_num=N, iter_num=iters, iter_threshold=0.0, time_print=False,
                   batch=U, device=DEV)
    orc = [OracleRDA(T, car, max_edge_num=E, max_obs_num=N, iter_num=iters, iter_threshold=0.0) for _ in range(U)]
    insts = [make_instance(700 + i, T=T, N=N, E=E, lateral=(0.3, 3.0)) for i in range(U)]
    rng = np.random.default_rng(1)
    prev = None
    worst = 0.0
    for call in range(3):
        perm = np.stack([rng.permutation(N) for _ in range(U)]).astype(np.int32)
        pA = np.take_along_axis(base['obs_A'], perm[:, :, None, None, None].astype(np.int64), 1)
        pb = np.take_along_axis(base['obs_b'], perm[:, :, None, None].astype(np.int64), 1)
        pk = np.take_along_axis(base['obs_kind'], perm.astype(np.int64), 1)
        g.set_obstacle_ids(perm)
        out = g.iterative_solve_batch(base['nom_s'], base['nom_u'], base['ref_s'], base['ref_speed'], pA, pb, pk,
                                      base['obs_count'])
        s = out['s'].cpu().numpy()
        for i, o in enumerate(orc):
            if prev is not None:
                oi.remap_oracle_slots(o, prev[i], perm[i])
            ref = [insts[i]['ref'][:, t:t + 1] for t in range(T + 1)]
            _, info = o.iterative_solve(insts[i]['nom_s'], insts[i]['nom_u'], ref, insts[i]['ref_speed'],
                                        [insts[i]['obstacles'][j] for j in perm[i]])
            worst = max(worst, float(np.abs(np.hstack(info['opt_state_list']) - s[i]).max()))
        prev = perm
    print(f'device vs float64 oracle with remapped warm start: max |ds| {worst:.3g}')
    assert worst < 1e-3, worst


def _robots(rng, B, span):
    return np.column_stack([rng.uniform(-span, span, (B, 2)), rng.uniform(-3, 3, B)]).astype(np.float32)


def test_id_conversions_write_the_existing_rows_and_the_twins_ids():
    rng = np.random.default_rng(5)
    T, E, N, B = 8, 4, 6, 24
    worlds = [_world(rng, 40, moving=True), _world(rng, 5), []]
    world_h = pack_worlds(worlds)
    world = shapes_to_device(world_h, DEV)
    robot_world_h = rng.integers(-1, 3, B).astype(np.int32)
    robot_world = _t(robot_world_h)
    state_h = _robots(rng, B, 15.0)
    state = _t(state_h)
    body = robot_body(rectangle_robot(length=1.0, width=0.6))
    body['xy'] = _t(body['xy'])
    cur_vel = _t(rng.uniform(-1, 1, (B, 2, T)).astype(np.float32))

    def same(plain, with_ids, want_ids):
        for x, y in zip(plain, with_ids[:4]):
            assert torch.equal(x, y)
        np.testing.assert_array_equal(with_ids[4].cpu().numpy(), want_ids)

    for order in (0, 1):
        for tv in (0, 1):
            same(convert_world_obstacles_batch(world, state, robot_world, N, T, E, DT, tv, order),
                 convert_world_obstacles_batch(world, state, robot_world, N, T, E, DT, tv, order, ids=True),
                 oi.world_ids(world_h, state_h, robot_world_h, N, order))
            fleet = fleet_shapes_batch(state, cur_vel, body, 'acker')
            fleet_h = {k: v.cpu().numpy() for k, v in fleet.items()}
            same(convert_fleet_obstacles_batch(world, state, robot_world, fleet, N, T, E, DT, tv, order),
                 convert_fleet_obstacles_batch(world, state, robot_world, fleet, N, T, E, DT, tv, order, ids=True),
                 oi.world_ids(world_h, state_h, robot_world_h, N, order, fleet_h))
        plan = fleet_plan_shapes_batch(state, cur_vel, body, 'acker', DT, 1.0)
        plan_h = {k: v.cpu().numpy() for k, v in plan.items() if k != 'plan_xy'}
        same(convert_fleet_obstacles_batch(world, state, robot_world, plan, N, T, E, DT, 1, order, plan=True),
             convert_fleet_obstacles_batch(world, state, robot_world, plan, N, T, E, DT, 1, order, plan=True, ids=True),
             oi.world_ids(world_h, state_h, robot_world_h, N, order, plan_h))
    # horizon order, world and fleet
    nom_h = np.repeat(state_h[:, :, None], T + 1, axis=2) + rng.normal(0, 0.3, (B, 3, T + 1)).astype(np.float32)
    ref_h = nom_h + np.float32(0.5)
    nom, ref = _t(nom_h), _t(ref_h)
    body_h = dict(body, xy=body['xy'].cpu().numpy())
    fleet = fleet_shapes_batch(state, cur_vel, body, 'acker')
    fleet_h = {k: v.cpu().numpy() for k, v in fleet.items()}
    for fl, flh in ((None, None), (fleet, fleet_h)):
        same(convert_world_obstacles_horizon_batch(world, nom, ref, body, robot_world, N, T, E, DT, 0, fl),
             convert_world_obstacles_horizon_batch(world, nom, ref, body, robot_world, N, T, E, DT, 0, fl, ids=True),
             oi.horizon_ids(world_h, nom_h, ref_h, body_h, robot_world_h, N, T, E, DT, 0, flh))
    # per-robot lists: the position in the list
    lists = [_world(rng, int(rng.integers(0, 12))) for _ in range(B)]
    shapes_h = pack_shapes(lists, max_edge_num=E)
    shapes = shapes_to_device(shapes_h, DEV)
    for order in (0, 1):
        want = np.stack([oi.kept_positions(oi.reference_keys({k: shapes_h[k][b, :len(lists[b])] for k in oi.KEYS},
                                                             state_h[b]) if order else
                                           np.arange(len(lists[b]), dtype=float), N) for b in range(B)])
        same(convert_obstacles_batch(shapes, state, N, T, E, DT, 1, order),
             convert_obstacles_batch(shapes, state, N, T, E, DT, 1, order, ids=True), want)


def _fleet_run(warm_start, steps=4, clear=False, **kw):
    rng = np.random.default_rng(2)
    B, T, N = 16, 10, 4
    path = np.stack([np.linspace(0, 40, 60), np.zeros(60), np.zeros(60)])
    world = shapes_to_device(pack_worlds([_world(rng, 30, spread=15.0)]), DEV)
    mpc = BatchedMPC(rectangle_robot(length=1.0, width=0.6, wheelbase=0.6), path, B, receding=T, max_obs_num=N,
                     max_edge_num=4, iter_num=4, device=DEV, **({'warm_start': warm_start} if warm_start else {}))
    state = _t(np.column_stack([rng.uniform(0, 5, B), rng.uniform(-3, 3, B), np.zeros(B)]).astype(np.float32))
    outs = []
    for k in range(steps):
        u, info = mpc.control(state, 2.0, world=world, avoid_fleet=True)
        outs.append({key: info[key].clone() for key in ('u', 's', 'status', 'iters') + (('obs_id',) if 'obs_id' in info
                                                                                          else ())})
        if clear and k == 1:
            mpc.rda.set_obstacle_ids(None)
        mpc.advance(state)
    return outs


def test_batched_mpc_warm_start_option():
    plain = _fleet_run(None)
    for outs in (_fleet_run('slot'), _fleet_run('slot', clear=True)):
        for a, b in zip(plain, outs):
            for k in ('u', 's', 'status', 'iters'):
                assert torch.equal(a[k], b[k]), k
    follow = _fleet_run('obstacle')
    assert all('obs_id' in o for o in follow)
    assert all(((o['obs_id'] >= -1)).all() for o in follow)
    assert all((o['status'] & (_cabi.ST_SU_NONFINITE | _cabi.ST_CELL_FALLBACK) == 0).all() for o in follow)
    with pytest.raises(ValueError):
        BatchedMPC(rectangle_robot(), np.zeros((3, 5)), 2, warm_start='id', device=DEV)


def _slot_obstacles(keep, b):
    """The obstacle list the device solved instance b with, as the oracle takes it: one object per slot from the rows
    the conversion wrote (the padding copies included, as assign_obstacle_parameter pads), none for an empty list."""
    from rda_planner_b200.mpc import rdaobs
    if int(keep['obs_count'][b]) == 0:
        return []
    A, bb, kind = (keep[k][b].double().cpu().numpy() for k in ('obs_A', 'obs_b', 'obs_kind'))
    return [rdaobs(A[n, 0], bb[n, 0].reshape(-1, 1), 'norm2' if int(kind[n]) == _cabi.OBS_CIRCLE else 'Rpositive',
                   None, None) for n in range(A.shape[0])]


@pytest.mark.parametrize('avoid_fleet', [False, True])
def test_batched_mpc_obstacle_warm_start_follows_the_oracle(avoid_fleet):
    """BatchedMPC(warm_start='obstacle') over a closed loop, against one float64 oracle per robot that solves each step
    with the device's nominal, reference and obstacle rows and moves its warm start by info['obs_id'] (the same rule,
    remap_oracle_slots).  A second oracle per robot keeps the warm start in its slot: the loop must change slot owners,
    and following the ids must matter, for the comparison to mean something."""
    rng = np.random.default_rng(21)
    T, N, E, iters, steps = 10, 4, 4, 4, 6
    car = rectangle_robot(length=1.0, width=0.6, wheelbase=0.6)
    path = np.stack([np.linspace(0, 60, 240), np.zeros(240), np.zeros(240)])
    if avoid_fleet:
        # five robots in an empty map, the faster ones behind: every robot sees its four mates, and the order of their
        # distances changes as they overtake
        B, world = 5, None
        state = _t(np.column_stack([np.linspace(6, 0, B), np.linspace(-0.8, 0.8, B), np.zeros(B)]).astype(np.float32))
        speed = _t(np.linspace(0.5, 3.0, B).astype(np.float32))
    else:
        B, world = 4, shapes_to_device(pack_worlds([_world(rng, 40, spread=12.0)]), DEV)
        state = _t(np.column_stack([np.linspace(0, 6, B), rng.uniform(-1, 1, B), np.zeros(B)]).astype(np.float32))
        speed = _t(np.full(B, 2.0, np.float32))
    mpc = BatchedMPC(car, path, B, receding=T, max_obs_num=N, max_edge_num=E, iter_num=iters, iter_threshold=0.0,
                     device=DEV, warm_start='obstacle')
    mk = lambda: OracleRDA(T, car, max_edge_num=E, max_obs_num=N, iter_num=iters, step_time=0.1, iter_threshold=0.0)
    follow, stay = [mk() for _ in range(B)], [mk() for _ in range(B)]
    prev, worst, worst_stay, moved = None, 0.0, 0.0, 0
    for _ in range(steps):
        nom_u = mpc.cur_vel.double().cpu().numpy()
        _, info = mpc.control(state, speed, world=world, avoid_fleet=avoid_fleet)
        keep = mpc.rda._keep                                    # the tensors the solve read
        ids = info['obs_id'].cpu().numpy()
        s_dev = info['s'].double().cpu().numpy()
        nom_s, ref_s = info['nom_s'].double().cpu().numpy(), info['ref_s'].double().cpu().numpy()
        for b in range(B):
            if prev is not None:
                oi.remap_oracle_slots(follow[b], prev[b], ids[b])
                moved += int(np.count_nonzero(oi.slot_source(prev[b], ids[b]) != np.arange(N)))
            ref = [ref_s[b][:, t:t + 1] for t in range(T + 1)]
            for o, gap in ((follow[b], 'follow'), (stay[b], 'stay')):
                _, oinfo = o.iterative_solve(nom_s[b], nom_u[b], ref, float(speed[b]), _slot_obstacles(keep, b))
                d = float(np.abs(np.hstack(oinfo['opt_state_list']) - s_dev[b]).max())
                if gap == 'follow':
                    worst = max(worst, d)
                else:
                    worst_stay = max(worst_stay, d)
        prev = ids
        mpc.advance(state)
    print(f'avoid_fleet={avoid_fleet}: {moved} slots moved; max |ds| to the oracle {worst:.3g} with the ids followed, '
          f'{worst_stay:.3g} with the warm start left in its slot')
    assert moved > 0
    assert worst < 1e-3, worst
    assert worst_stay > 1e-3, worst_stay                       # the bound tells the two warm starts apart


def test_captured_graph_replays_the_id_call_and_the_solve():
    T, N, E, B = 30, 20, 4, 1024
    base, _ = _instances(64, T, N, E)
    inp = {k: _t(v[np.arange(B) % 64]) for k, v in base.items()}
    rng = np.random.default_rng(9)
    perm = _t(np.stack([rng.permutation(N) for _ in range(B)]).astype(np.int32))
    ident = _t(np.tile(np.arange(N, dtype=np.int32), (B, 1)))
    pidx = perm.long()
    gather = lambda x: torch.gather(x, 1, pidx.reshape(B, N, *([1] * (x.dim() - 2))).expand_as(x)).contiguous()
    pinp = dict(inp, obs_A=gather(inp['obs_A']), obs_b=gather(inp['obs_b']), obs_kind=gather(inp['obs_kind']))
    mk = lambda: RDA_solver(T, rectangle_robot(), max_edge_num=E, max_obs_num=N, iter_num=6, iter_threshold=0.0,
                            time_print=False, batch=B, device=DEV)
    eager, cap = mk(), mk()
    for g in (eager, cap):
        g.set_obstacle_ids(ident)
        g.iterative_solve_batch(**inp)
    eager.set_obstacle_ids(perm)
    want = {k: v.clone() for k, v in eager.iterative_solve_batch(**pinp).items()}
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            cap.set_obstacle_ids(perm)
            out = cap.iterative_solve_batch(**pinp)
    torch.cuda.current_stream(DEV).wait_stream(side)
    graph.replay()
    torch.cuda.synchronize()
    for k in ('u', 's', 'status', 'iters'):
        assert torch.equal(out[k], want[k]), k
