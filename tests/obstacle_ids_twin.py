"""The slot match of rda_set_obstacle_ids restated in numpy, ctypes access to its g++ twin (tests/cpu_twin/obstacle_ids.cpp),
and the obstacle ids the world, fleet and horizon selections keep, restated from the twins' keys — test infrastructure
only."""
import ctypes as C

import numpy as np

import fleet_obstacles_twin as ft
import horizon_twin as ht
import shim

KEYS = ('kind', 'nv', 'xy', 'radius', 'vel')


def slot_source(prev, cur):
    """numpy restatement: src [N], the slot of prev whose state slot n of cur takes (-1: cold start).  Copy k of id X in
    cur (k = how many slots before n carry X) takes copy k of X in prev."""
    prev, cur = np.asarray(prev, np.int64), np.asarray(cur, np.int64)
    N = len(cur)
    rank = np.array([np.count_nonzero(cur[:n] == cur[n]) for n in range(N)], np.int64)
    src = np.full(N, -1, np.int64)
    for n in range(N):
        if cur[n] < 0:
            continue
        at = np.flatnonzero(prev == cur[n])
        if rank[n] < len(at):
            src[n] = at[rank[n]]
    return src


def remap(state, src):
    """Per-slot state [N, ...] moved by src (slot_source): rows of src, zeros where src < 0."""
    state = np.asarray(state)
    out = np.zeros_like(state)
    ok = src >= 0
    out[ok] = state[src[ok]]
    return out


ORACLE_SLOT_STATE = ('para_lam', 'para_mu', 'para_z', 'para_xi', 'para_zeta', 'para_obsA_lam', 'para_obsb_lam')


def remap_oracle_slots(o, prev_ids, ids):
    """The rule of rda_set_obstacle_ids on an OracleRDA, in float64: every per-slot warm-start array (slot axis first)
    moved by slot_source(prev_ids, ids), the constructor's zeros where nothing matches.  Returns src."""
    src = slot_source(prev_ids, ids)
    for name in ORACLE_SLOT_STATE:
        setattr(o, name, remap(getattr(o, name), src))
    return src


def twin_slot_source(prev, cur):
    prev, cur = np.ascontiguousarray(prev, np.int32), np.ascontiguousarray(cur, np.int32)
    src = np.zeros(len(cur), np.int32)
    fn = shim.lib().shim_obstacle_slot_source
    fn.restype = None
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    fn(prev.ctypes.data, cur.ctypes.data, len(cur), src.ctypes.data)
    return src


def reference_keys(lst, state):
    """obstacle_key of every entry of a list (pack_worlds layout, one world) seen from state [3]."""
    count = len(lst['kind'])
    keys = np.zeros(max(count, 1))
    kind = np.ascontiguousarray(lst['kind'], np.int32)
    nv = np.ascontiguousarray(lst['nv'], np.int32)
    xy = np.ascontiguousarray(lst['xy'], np.float32)
    if count:
        fn = shim.lib().shim_obstacle_keys
        fn.restype = None
        fn.argtypes = [C.c_int, C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        fn(count, float(np.float32(state[0])), float(np.float32(state[1])), kind.ctypes.data, nv.ctypes.data,
           xy.ctypes.data, keys.ctypes.data)
    return keys[:count]


def kept_positions(keys, N):
    """The list positions of the N slots: stable ascending order of keys, the last repeated past the list."""
    count = len(keys)
    if count == 0:
        return np.full(N, -1, np.int64)
    order = np.argsort(keys, kind='stable')
    return order[np.minimum(np.arange(N), count - 1)]


def list_ids(world, robot_world, b, fleet=None):
    """The obstacle id of every entry of robot b's list: the flat world index of its world's shapes, then S + m for its
    map-mates m (S = world['start'][-1]) when fleet is given."""
    W = len(world['start']) - 1
    w = int(np.asarray(robot_world)[b]) if robot_world is not None else 0
    lo, hi = (int(world['start'][w]), int(world['start'][w + 1])) if 0 <= w < W else (0, 0)
    ids = list(range(lo, hi))
    if fleet is not None and 0 <= w < W:
        rw = np.asarray(robot_world)
        ids += [int(world['start'][-1]) + int(m) for m in np.nonzero(rw == w)[0] if m != b]
    return np.asarray(ids, np.int64)


def world_ids(world, state, robot_world, N, order=True, fleet=None):
    """obs_id [B, N] of rda_convert_world_obstacles_ids with the reference key (order) or list order."""
    B = len(state)
    out = np.zeros((B, N), np.int64)
    for b in range(B):
        if fleet is None:
            W = len(world['start']) - 1
            w = int(np.asarray(robot_world)[b]) if robot_world is not None else 0
            lo, hi = (int(world['start'][w]), int(world['start'][w + 1])) if 0 <= w < W else (0, 0)
            lst = {k: np.asarray(world[k][lo:hi]) for k in KEYS}
        else:
            lst = ft.robot_list(world, fleet, robot_world if robot_world is not None else np.zeros(B, np.int32), b)
        keys = reference_keys(lst, state[b]) if order else np.arange(len(lst['kind']), dtype=float)
        pos = kept_positions(keys, N)
        ids = list_ids(world, robot_world, b, fleet)
        out[b] = np.where(pos >= 0, ids[np.maximum(pos, 0)] if len(ids) else -1, -1)
    return out


def horizon_ids(world, nom_s, ref_s, body, robot_world, N, T, E, dt, tv, fleet=None):
    """obs_id [B, N] of rda_convert_world_obstacles_horizon_ids, from the horizon twin's exact keys."""
    B = len(nom_s)
    out = np.zeros((B, N), np.int64)
    for b in range(B):
        lst = ht.robot_list(world, fleet, robot_world, b)
        keys = ht.select(lst, N, T, E, dt, tv, nom_s[b], ref_s[b], body)[4]
        pos = kept_positions(keys, N)
        ids = list_ids(world, robot_world, b, fleet)
        out[b] = np.where(pos >= 0, ids[np.maximum(pos, 0)] if len(ids) else -1, -1)
    return out
