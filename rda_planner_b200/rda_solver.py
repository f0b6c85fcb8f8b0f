"""RDA_solver — the drop-in for RDA_planner.rda_solver.RDA_solver, backed by sm_90a kernels.

Mirror of the reference's RDA_planner/rda_solver.py (class RDA_solver): constructor :18-22
(+ tunables :185-201, ws/wu :218-219), iterative_solve :573-610, assign_adjust_parameter
:426-434, get_adjust_parameter :1055-1056, reset :1060-1068.  numpy in / numpy out at this
level, exactly like the reference; all arithmetic runs in librda_b200.so (include/rda_b200.h)
on the current CUDA device, with PyTorch used only for device memory and streams.

New surface (absent in the reference, required by BASELINE.json): `batch` > 1 and
`iterative_solve_batch` on CUDA tensors — B independent planning instances that share
(T, N, E, robot, dynamics) and keep their own warm-start state on the device.
"""
import ctypes as C
import time

import numpy as np
import torch

from . import _cabi


def _as_cuda_f32(x, device):
    return torch.as_tensor(x, dtype=torch.float32, device=device).contiguous()


# Half-size [m] of the square (centred on the robot) that closes unbounded half-space sets in canonical_polygon_rows.
# The kernels work in float32 relative to the robot: a vertex L metres away turns a direction error of one ulp into
# L * 1e-7 m of margin, so the square is kept as small as a planning horizon allows and grown only when the set does
# not reach into it (then the obstacle is too far to matter).
HALFSPACE_BOUND = 100.0
HALFSPACE_BOUND_MAX = 1.0e5
_CANONICAL_SEEN = set()      # (A bytes, b bytes) of row sets already verified to be closed counter-clockwise polygons


def canonical_polygon_rows(A, b, bound=None, center=None):
    """Rows of a convex set {x: Ax <= b} ordered counter-clockwise by normal angle so that vertex i joins rows i-1 and
    i — the layout the kernels' closest-point geometry needs.  A no-op for the output of mpc.py:476-510 (closed convex
    polygon, rows already in order).  Anything else the reference accepts through rda_obstacle=True (mpc.py:150-155:
    the caller's own (A, b) tuples) is reduced to that case by clipping: rows in any order, redundant rows (dropped:
    their multipliers are zero at every optimum), and UNBOUNDED sets (a wall, a wedge, a strip), which are closed by
    the sides of the square |x - center|_inf <= bound (center: the robot position, default the origin; bound: default
    HALFSPACE_BOUND, grown 4x until the set reaches into the square) — exact as long as the closest obstacle point to
    the robot does not lie on one of those artificial sides.  Original rows keep their scaling.  Raises ValueError for
    an empty set."""
    A = np.asarray(A, float)
    b = np.asarray(b, float).reshape(-1)
    n = A.shape[0]
    def one_turn(M):
        # consecutive normals turn left AND the turning angles add up to a single 2 pi (no double winding)
        m = M.shape[0]
        d = M[np.arange(m) - 1, 0] * M[:, 1] - M[np.arange(m) - 1, 1] * M[:, 0]
        if m < 3 or not np.all(d > 0):
            return False
        a = np.arctan2(M[:, 1], M[:, 0])
        turn = np.mod(a - np.roll(a, 1), 2 * np.pi)
        return abs(turn.sum() - 2 * np.pi) < 1e-6
    def every_row_is_an_edge(M, c):
        # vertex i = rows i-1 and i; every vertex must satisfy all rows, and consecutive vertices must differ
        Mp, cp = np.roll(M, 1, axis=0), np.roll(c, 1)
        det = Mp[:, 0] * M[:, 1] - Mp[:, 1] * M[:, 0]
        V = np.stack([(cp * M[:, 1] - c * Mp[:, 1]) / det, (Mp[:, 0] * c - M[:, 0] * cp) / det], axis=1)
        slack = c[None, :] - V @ M.T
        scale = np.linalg.norm(M, axis=1)[None, :] * (1.0 + np.abs(V).max())
        if np.any(slack < -1e-9 * scale):
            return False
        return bool(np.all(np.linalg.norm(np.roll(V, -1, axis=0) - V, axis=1) > 1e-9 * (1.0 + np.abs(V).max())))
    # the common case — the output of mpc.py:476-510, unchanged from one control step to the next for static obstacles — is
    # recognised once and remembered by content (a dozen small numpy calls per obstacle would otherwise cost more than the
    # whole solve of the path_track example)
    key = (A.tobytes(), b.tobytes()) if A.size <= 64 else None
    if key is not None and key in _CANONICAL_SEEN:
        return A, b
    live = np.linalg.norm(A, axis=1) > 0
    if live.all() and one_turn(A) and every_row_is_an_edge(A, b):
        if key is not None:
            if len(_CANONICAL_SEEN) > 65536:
                _CANONICAL_SEEN.clear()
            _CANONICAL_SEEN.add(key)
        return A, b
    if np.any(b[~live] < 0):
        raise ValueError('obstacle half-spaces describe an empty set (0 <= b violated by a zero row)')
    ctr = np.zeros(2) if center is None else np.asarray(center, float).reshape(-1)[:2]
    if bound is None or bound > 0:
        # first square of half-size `bound` (default HALFSPACE_BOUND), grown 4x while the set does not reach into it
        L = float(HALFSPACE_BOUND if bound is None else bound)
        while True:
            try:
                return canonical_polygon_rows(A, b, bound=-L, center=ctr)
            except ValueError:
                if L >= HALFSPACE_BOUND_MAX:
                    raise
                L *= 4.0
    L = -float(bound)            # negative: exactly this size, no growth (internal)
    # Sutherland-Hodgman clipping of the square by every row; each vertex carries the row of the edge that STARTS there
    # (-1..-4: the artificial sides of the square)
    poly = [(ctr + np.array([-L, -L]), -1), (ctr + np.array([L, -L]), -2), (ctr + np.array([L, L]), -3),
            (ctr + np.array([-L, L]), -4)]
    for r in np.nonzero(live)[0]:
        a, c = A[r], b[r]
        tol = 1e-12 * np.linalg.norm(a) * (L + np.abs(ctr).max())
        out = []
        for k in range(len(poly)):
            (P, tag), (Q, _) = poly[k], poly[(k + 1) % len(poly)]
            sp, sq = a @ P - c, a @ Q - c
            if sp <= tol:
                out.append((P, tag))
                if sq > tol:
                    out.append((P + (Q - P) * (sp / (sp - sq)), int(r)))
            elif sq <= tol:
                out.append((P + (Q - P) * (sp / (sp - sq)), tag))
        poly = out
        if len(poly) < 3:
            raise ValueError('obstacle half-spaces describe an empty set inside |x| <= %g' % L)
    # drop zero-length edges (a row that only touches a vertex)
    keep = [k for k in range(len(poly))
            if np.linalg.norm(poly[(k + 1) % len(poly)][0] - poly[k][0]) > 1e-9 * (1.0 + 1e-4 * (L + np.abs(ctr).max()))]
    poly = [poly[k] for k in keep]
    if len(poly) < 3:
        raise ValueError('obstacle half-spaces describe a set without interior')
    box = {-1: (np.array([0.0, -1.0]), L - ctr[1]), -2: (np.array([1.0, 0.0]), L + ctr[0]),
           -3: (np.array([0.0, 1.0]), L + ctr[1]), -4: (np.array([-1.0, 0.0]), L - ctr[0])}
    rows = [(A[t], b[t]) if t >= 0 else box[t] for _, t in poly]
    An = np.array([r[0] for r in rows], float)
    bn = np.array([r[1] for r in rows], float)
    if not one_turn(An):
        raise ValueError('obstacle half-spaces could not be reduced to a closed convex polygon')
    return An, bn


def pack_obstacles(obstacle_list, T, N, E, center=None, bound=None):
    """assign_obstacle_parameter (rda_solver.py:483-526): pad a short list by repeating its
    last element (mutating the caller's list, as the reference does), truncate a long one,
    zero-pad rows to E.  center: robot position, only used to close unbounded half-space sets
    (canonical_polygon_rows).  Returns (A [N,Tc,E,2], b [N,Tc,E], kind [N], count, time_varying)."""
    count = len(obstacle_list)
    if 0 < count < N:
        obstacle_list += [obstacle_list[-1]] * (N - count)
    number = min(len(obstacle_list), N)
    tv = any(isinstance(o.A, list) for o in obstacle_list[:number])
    Tc = T + 1 if tv else 1
    A = np.zeros((N, Tc, E, 2), np.float32)
    b = np.zeros((N, Tc, E), np.float32)
    kind = np.zeros(N, np.int32)
    for i in range(number):
        o = obstacle_list[i]
        circle = o.cone_type != 'Rpositive'
        kind[i] = _cabi.OBS_CIRCLE if circle else _cabi.OBS_POLYGON
        for t in range(Tc):
            At = o.A[t] if isinstance(o.A, list) else o.A
            bt = o.b[t] if isinstance(o.b, list) else o.b
            At = np.asarray(At, float)
            bt = np.asarray(bt, float).reshape(-1)
            if not circle:
                At, bt = canonical_polygon_rows(At, bt, bound=bound, center=center)
            en = At.shape[0]
            if en > E:
                raise ValueError(f'obstacle with {en} edges exceeds max_edge_num={E}'
                                 + (' (an unbounded half-space set is closed by up to four sides of a large square: '
                                    'raise max_edge_num accordingly)' if en > np.asarray(o.A[t] if isinstance(o.A, list) else o.A).shape[0] else ''))
            A[i, t, :en] = At
            b[i, t, :en] = bt
    return A, b, kind, count, tv


# Per-instance parameters (RDA_solver.set_instance_parameters): key -> columns of the table (include/rda_b200.h, RDA_IP_*)
INSTANCE_COLUMNS = {'max_speed': (_cabi.IP_MAX_SPEED0, _cabi.IP_MAX_SPEED1),
                    'max_acce': (_cabi.IP_ACCE_BOUND0, _cabi.IP_ACCE_BOUND1),
                    'ws': (_cabi.IP_WS,), 'wu': (_cabi.IP_WU,), 'slack_gain': (_cabi.IP_SLACK_GAIN,),
                    'max_sd': (_cabi.IP_MAX_SD,), 'min_sd': (_cabi.IP_MIN_SD,), 'ro1': (_cabi.IP_RO1,),
                    'ro2': (_cabi.IP_RO2,)}
_POSITIVE = ('max_speed', 'max_acce', 'ro1', 'ro2')
_NON_NEGATIVE = ('slack_gain', 'ws', 'wu')


def _host_instance_value(key, value, B):
    """A host-given per-instance value, checked: float64 array of shape () / (B,) (scalar keys) or (2,) / (B, 2)
    (max_speed, max_acce)."""
    a = np.asarray(value, dtype=float)
    pair = len(INSTANCE_COLUMNS[key]) == 2
    shapes = ((2,), (B, 2)) if pair else ((), (B,))
    if a.shape not in shapes:
        raise ValueError(f'{key}: expected shape {" or ".join(str(x) for x in shapes)}, got {a.shape}')
    if not np.all(np.isfinite(a)):
        raise ValueError(f'{key}: values must be finite')
    if key in _POSITIVE and not np.all(a > 0):
        raise ValueError(f'{key}: values must be > 0')
    if key in _NON_NEGATIVE and not np.all(a >= 0):
        raise ValueError(f'{key}: values must be >= 0')
    return a


def update_instance_table(table, dt, robots=None, validate=True, **values):
    """A per-instance parameter table float32 [B, RDA_INST_PARAMS] (columns RDA_IP_*) with `values` written into the
    rows of the bool mask `robots` [B] (None: every row); returns a new tensor on table's device, the input is left as
    it is.  Keys of INSTANCE_COLUMNS; each value is a scalar (a pair for max_speed / max_acce) for every selected row,
    or [B] ([B, 2]) per row, as an array-like or a tensor.  max_acce is stored as acce_bound = max_acce * dt, formed in
    float64 and rounded to float32 as the constructor does.  Host-given values are checked (finite; max_speed,
    max_acce, ro1, ro2 > 0; slack_gain, ws, wu >= 0; min_sd <= max_sd when both are given); tensors only for shape and
    dtype, so that a call whose values and mask are all device tensors never waits for the device."""
    B, dev = table.shape[0], table.device
    unknown = sorted(set(values) - set(INSTANCE_COLUMNS))
    if unknown:
        raise TypeError(f'unknown per-instance parameter(s) {unknown}; known: {sorted(INSTANCE_COLUMNS)}')
    if robots is not None:
        robots = torch.as_tensor(robots, device=dev)
        if robots.dtype != torch.bool or robots.shape != (B,):
            raise ValueError(f'robots: expected a bool mask of shape ({B},), got {robots.dtype} {tuple(robots.shape)}')
    host = {}
    cols = {}       # column -> python float or float32 tensor [B]
    for key, v in values.items():
        pair = len(INSTANCE_COLUMNS[key]) == 2
        if isinstance(v, torch.Tensor):
            shapes = ((2,), (B, 2)) if pair else ((), (B,))
            if tuple(v.shape) not in shapes or not v.is_floating_point():
                raise ValueError(f'{key}: expected a floating tensor of shape {" or ".join(str(x) for x in shapes)}, '
                                 f'got {v.dtype} {tuple(v.shape)}')
            v = v.to(device=dev, dtype=torch.float64)
            if key == 'max_acce':
                v = v * float(dt)
            v = v.to(torch.float32)
            for j, c in enumerate(INSTANCE_COLUMNS[key]):
                x = v[..., j] if pair else v
                cols[c] = x.expand(B) if x.dim() == 0 else x
            continue
        a = _host_instance_value(key, v, B) if validate else np.asarray(v, dtype=float)
        host[key] = a
        if key == 'max_acce':
            a = a * float(dt)
        a = a.astype(np.float32)
        for j, c in enumerate(INSTANCE_COLUMNS[key]):
            x = a[..., j] if pair else a
            cols[c] = float(x) if x.ndim == 0 else torch.as_tensor(x, device=dev)
    if validate and 'min_sd' in host and 'max_sd' in host:
        if not np.all(np.broadcast_to(host['min_sd'], (B,)) <= np.broadcast_to(host['max_sd'], (B,))):
            raise ValueError('min_sd must not exceed max_sd')
    out = table.clone()
    for c, x in cols.items():
        if robots is None:
            out[:, c] = x
        else:
            out[:, c] = torch.where(robots, x, out[:, c])
    return out


def robot_body(car_tuple):
    """(G, h, robot cone) of a car_tuple's body as the kernels take it: a polygon's rows in canonical counter-clockwise
    order (canonical_polygon_rows), or the disc G = [[1,0],[0,1],[0,0]], h = (cx, cy, -r) of cone_type 'norm2'."""
    G = np.asarray(car_tuple.G, float)
    h = np.asarray(car_tuple.h, float).reshape(-1)
    if car_tuple.cone_type == 'norm2':
        # disc body (cone_cp_array(-mu, 'norm2'), :1034-1039) as ir-sim describes it: |y - (h0, h1)| <= -h2
        if G.shape != (3, 2) or np.abs(G - np.array([[1.0, 0], [0, 1], [0, 0]])).max() > 1e-9 or not h[2] < 0:
            raise NotImplementedError("norm2 robot: only the disc G = [[1,0],[0,1],[0,0]], h = (cx, cy, -r) is supported")
        return G, h, _cabi.ROBOT_DISC
    if car_tuple.cone_type == 'Rpositive':
        G, h = canonical_polygon_rows(G, h)
        return G, h, _cabi.ROBOT_POLYGON
    raise ValueError(f'unknown robot cone type {car_tuple.cone_type!r}')


def robot_class_table(car_tuples, cone_type, R):
    """The rda_robot_class array of car_tuples (at most RDA_MAX_ROBOT_CLASSES) for a solver whose body has cone_type and
    R canonical rows; raises ValueError naming the first class the kernels cannot take."""
    K = len(car_tuples)
    if K > _cabi.MAX_ROBOT_CLASSES:
        raise ValueError(f'at most {_cabi.MAX_ROBOT_CLASSES} robot classes, got {K}')
    arr = (_cabi.RobotClass * max(K, 1))()
    for k, car in enumerate(car_tuples):
        if car.cone_type != cone_type:
            raise ValueError(f'robot class {k}: cone_type {car.cone_type!r} differs from the solver\'s {cone_type!r}')
        G, h, _ = robot_body(car)
        if G.shape[0] != R:
            raise ValueError(f'robot class {k}: {G.shape[0]} canonical body rows, the solver has {R}')
        if car.dynamics not in _cabi.DYNAMICS:
            raise ValueError(f'robot class {k}: unknown dynamics {car.dynamics!r}')
        L = float(car.wheelbase)
        if not np.isfinite(L) or (car.dynamics == 'acker' and not L > 0):
            raise ValueError(f'robot class {k}: wheelbase must be finite, and > 0 for acker (got {car.wheelbase})')
        for key in ('max_speed', 'max_acce'):
            try:
                _host_instance_value(key, np.asarray(getattr(car, key), float).reshape(-1)[:2], 1)
            except ValueError as e:
                raise ValueError(f'robot class {k}: {e}') from None
        arr[k].dynamics, arr[k].wheelbase = _cabi.DYNAMICS[car.dynamics], L
        for j in range(R):
            arr[k].G[2 * j], arr[k].G[2 * j + 1], arr[k].h[j] = G[j, 0], G[j, 1], h[j]
    return arr


class RDA_solver:
    def __init__(self, receding, car_tuple, max_edge_num=5, max_obs_num=5, iter_num=2, step_time=0.1,
                 iter_threshold=0.2, process_num=4, accelerated=True, time_print=True, batch=1,
                 device=None, su_fp64=True, z_theta=0.5, graph=False, **kwargs):
        """kwargs: slack_gain (8), max_sd (1.0), min_sd (0.1), ro1 (200), ro2 (1), ws (1), wu (1)
        — rda_solver.py:24-31.  `process_num` is accepted for compatibility and ignored.
        graph=True replays the launches of a solve from a CUDA graph (captured on first use per set of input
        buffers / iteration count): the single-instance API then copies its inputs into persistent device
        buffers, so every control step after the first is one graph launch."""
        if not torch.cuda.is_available():
            raise RuntimeError('rda_planner_b200 needs a CUDA device (H100); there is no CPU fallback')
        self.lib = _cabi.load()
        self.device = torch.device(device if device is not None else f'cuda:{torch.cuda.current_device()}')
        self.T = receding
        self.car_tuple = car_tuple
        self.L = car_tuple.wheelbase
        self.max_obs_num = max_obs_num
        self.max_edge_num = max(max_edge_num, 3)
        self.dynamics = car_tuple.dynamics
        self.iter_num = iter_num
        self.dt = step_time
        self.iter_threshold = iter_threshold
        self.accelerated = accelerated
        self.process_num = process_num
        self.time_print = time_print
        self.batch = batch
        self.ws = kwargs.get('ws', 1)
        self.wu = kwargs.get('wu', 1)
        G, h, robot_cone = robot_body(car_tuple)
        R = G.shape[0]
        if R > _cabi.MAX_ROBOT_EDGE or self.max_edge_num > _cabi.MAX_EDGE:
            raise ValueError('at most 8 robot edges / obstacle edges are supported')
        cfg = _cabi.Config()
        cfg.batch, cfg.receding, cfg.max_obs_num = batch, receding, max_obs_num
        cfg.max_edge_num, cfg.robot_edges = self.max_edge_num, R
        cfg.dynamics = _cabi.DYNAMICS[self.dynamics]
        cfg.accelerated = int(bool(accelerated))
        cfg.su_fp64 = int(bool(su_fp64))
        cfg.step_time, cfg.wheelbase = step_time, float(self.L)
        ms = np.asarray(car_tuple.max_speed, float).reshape(-1)
        ma = np.asarray(car_tuple.max_acce, float).reshape(-1)
        for k in range(2):
            cfg.max_speed[k] = ms[k]
            cfg.acce_bound[k] = ma[k] * step_time                      # :44
        cfg.ws, cfg.wu = self.ws, self.wu
        cfg.robot_cone = robot_cone
        for j in range(R):
            cfg.G[2 * j], cfg.G[2 * j + 1], cfg.h[j] = G[j, 0], G[j, 1], h[j]
        self._tun = _cabi.Tunables(kwargs.get('slack_gain', 8), kwargs.get('max_sd', 1.0),
                                   kwargs.get('min_sd', 0.1), kwargs.get('ro1', 200),
                                   kwargs.get('ro2', 1), z_theta)
        # the values as the caller gave them (the device copy is float32): get_adjust_parameter returns these
        self._tun_py = {k: kwargs.get(k, dflt) for k, dflt in (('slack_gain', 8), ('max_sd', 1.0), ('min_sd', 0.1),
                                                                ('ro1', 200), ('ro2', 1))}
        # closing square of unbounded half-space obstacles (canonical_polygon_rows): 1.5 x what the robot can reach within the
        # horizon plus body and safety distance, at least 30 m — small, because far vertices cost float32 precision
        self._hs_bound = max(30.0, 1.5 * (receding * step_time * float(abs(ms[0])) + 8.0))
        self._cfg = cfg
        self._h = C.c_void_p()
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.rda_create(C.byref(cfg), C.byref(self._tun), C.byref(self._h)), 'rda_create')
        B, T = batch, receding
        dev = self.device
        self._out = {
            'u': torch.empty((B, 2, T), dtype=torch.float32, device=dev),
            's': torch.empty((B, 3, T + 1), dtype=torch.float32, device=dev),
            'resi_pri': torch.empty(B, dtype=torch.float32, device=dev),
            'resi_dual': torch.empty(B, dtype=torch.float32, device=dev),
            'status': torch.empty(B, dtype=torch.int32, device=dev),
            'iters': torch.empty(B, dtype=torch.int32, device=dev),
        }
        self._keep = None
        self._keep_tv = 0
        self.obstacle_num = 0
        self.use_graph = bool(graph)
        self._graphs = {}
        self._static = None
        self._inst = None           # the installed per-instance table [B, RDA_INST_PARAMS] (set_instance_parameters)
        self._classes = None        # the installed robot classes (set_robot_classes): car_tuples
        self._class_index = None    # their index [B] (int32 CUDA tensor)
        self._class_limits = None   # max_speed, max_acce of each class slot [K + 1, 2] (float64 CUDA tensors)

    def __del__(self):
        try:
            if getattr(self, '_h', None) is not None and self._h.value:
                self.lib.rda_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass

    # ------------------------------------------------------------------ tunables
    def assign_adjust_parameter(self, **kwargs):
        """slack_gain, max_sd, min_sd, ro1, ro2 (ws/wu silently ignored, as in :426-434)."""
        t = self._tun
        t.slack_gain = kwargs.get('slack_gain', t.slack_gain)
        t.max_sd = kwargs.get('max_sd', t.max_sd)
        t.min_sd = kwargs.get('min_sd', t.min_sd)
        t.ro1 = kwargs.get('ro1', t.ro1)
        t.ro2 = kwargs.get('ro2', t.ro2)
        for k in self._tun_py:
            if k in kwargs:
                self._tun_py[k] = kwargs[k]
        _cabi.check(self.lib.rda_set_tunables(self._h, C.byref(t)), 'rda_set_tunables')
        if self._inst is not None:
            # what the reference's update_parameter does on every robot's MPC: the named tunables of every instance
            named = {k: float(getattr(t, k)) for k in self._tun_py if k in kwargs}
            if named:
                self._install(update_instance_table(self._inst, self.dt, validate=False, **named))

    # ------------------------------------------------------------------ per-instance parameters
    def _uniform_table(self):
        """The handle's current limits, weights and tunables as a table [B, RDA_INST_PARAMS] on the device (column
        fills, no host-to-device copy)."""
        cfg, t = self._cfg, self._tun
        row = [cfg.max_speed[0], cfg.max_speed[1], cfg.acce_bound[0], cfg.acce_bound[1], cfg.ws, cfg.wu,
               t.slack_gain, t.max_sd, t.min_sd, t.ro1, t.ro2]
        table = torch.empty((self.batch, _cabi.INST_PARAMS), dtype=torch.float32, device=self.device)
        for c, v in enumerate(row):
            table[:, c] = float(v)
        return table

    def _install(self, table):
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.rda_set_instance_params(self._h, C.c_void_p(table.data_ptr()), self._stream()),
                        'rda_set_instance_params')
        if self._inst is None:
            self._graphs.clear()        # captured launches carry "no table"; an update of an installed table is seen
        self._inst = table              # the copy into the handle's storage reads it on the current stream

    def set_instance_parameters(self, robots=None, **values):
        """Give instances their own limits, weights and tunables: max_speed, max_acce (pairs), ws, wu, slack_gain,
        max_sd, min_sd, ro1, ro2 — each a scalar (pair) for every selected instance or [B] ([B, 2]) per instance, as
        an array-like or a CUDA tensor; robots: bool mask [B] that restricts the update (None: all).  The first call
        starts from the handle's current values.  From the next solve on, instance b solves with its row as if it had
        been constructed with those values (update_instance_table gives the checks).  Without host synchronisation when
        every value and the mask are CUDA tensors."""
        base = self._inst if self._inst is not None else self._uniform_table()
        self._install(update_instance_table(base, self.dt, robots, **values))

    def clear_instance_parameters(self):
        """Back to the handle's values (constructor / assign_adjust_parameter) for every instance."""
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.rda_set_instance_params(self._h, None, self._stream()), 'rda_set_instance_params')
        if self._inst is not None:
            self._graphs.clear()
        self._inst = None

    def instance_parameters(self):
        """The values each instance solves with, dict of CUDA tensors: max_speed, acce_bound, max_acce (acce_bound / dt)
        [B, 2] and ws, wu, slack_gain, max_sd, min_sd, ro1, ro2 [B]."""
        table = self._inst if self._inst is not None else self._uniform_table()
        out = {k: table[:, list(c)] if len(c) == 2 else table[:, c[0]] for k, c in INSTANCE_COLUMNS.items()}
        out['acce_bound'] = out.pop('max_acce')
        out['max_acce'] = (out['acce_bound'].double() / self.dt).float()
        return {k: v.clone() for k, v in out.items()}

    # ------------------------------------------------------------------ robot classes
    def set_robot_classes(self, car_tuples, robot_class):
        """Give each instance the body, wheelbase, dynamics and limits of a robot class: car_tuples is a list of at most
        16 car_tuples (G h cone_type wheelbase max_speed max_acce dynamics) with the constructor's cone_type and as many
        canonical rows (canonical_polygon_rows) as its body; robot_class [B] picks instance b's class, as an array-like
        or an integer CUDA tensor.  An index outside [0, len(car_tuples)) means the constructor's car_tuple.  Each
        instance's max_speed / max_acce become those of its class through set_instance_parameters (gathered on the
        device); a later set_instance_parameters still overrides them.  Raises ValueError naming the offending class.
        A set-up call: the classes and their limits are uploaded before it returns (the host waits for that copy);
        set_robot_class_index then moves robots between classes without host synchronisation."""
        car_tuples = list(car_tuples)
        arr = robot_class_table(car_tuples, self.car_tuple.cone_type, self._cfg.robot_edges)
        K = len(car_tuples)
        index = self._class_index_tensor(robot_class, K)
        with torch.cuda.device(self.device):
            rc = self.lib.rda_set_robot_classes(self._h, K, arr, self._stream())
            if rc == _cabi.E_UNSUPPORTED:
                raise ValueError('robot class body not accepted: its rows must describe a closed convex polygon '
                                 '(or the disc of cone_type norm2)')
            _cabi.check(rc, 'rda_set_robot_classes')
        self._graphs.clear()        # captured launches carry the number of classes
        self._classes = car_tuples
        # max_speed / max_acce of each class slot [K + 1, 2] (slot K: the constructor's car_tuple), uploaded once here so
        # that moving robots between classes gathers on the device only
        cars = car_tuples + [self.car_tuple]
        pair = lambda key: torch.tensor(np.array([np.asarray(getattr(c, key), float).reshape(-1)[:2] for c in cars]),
                                        dtype=torch.float64, device=self.device)
        self._class_limits = (pair('max_speed'), pair('max_acce'))
        self._class_index = None
        self._install_class_index(index, None)

    def set_robot_class_index(self, robot_class, robots=None):
        """Move instances to other classes of the installed set (set_robot_classes): robot_class [B] (or one index),
        applied to the robots of the bool mask robots [B] (None: all).  The robots whose class changes get their new
        class's max_speed / max_acce; the others keep their rows.  Without host synchronisation when robot_class and
        robots are CUDA tensors; a captured graph sees the new index."""
        if self._classes is None:
            raise RuntimeError('set_robot_classes first')
        index = self._class_index_tensor(robot_class)
        if robots is not None:
            robots = torch.as_tensor(robots, device=self.device)
            if robots.dtype != torch.bool or robots.shape != (self.batch,):
                raise ValueError(f'robots: expected a bool mask of shape ({self.batch},), got {robots.dtype} '
                                 f'{tuple(robots.shape)}')
            index = torch.where(robots, index, self._class_index).contiguous()
        self._install_class_index(index, self._class_index)

    def clear_robot_classes(self):
        """Back to the constructor's body, wheelbase, dynamics and limits for every instance."""
        if self._classes is not None and self._inst is not None:
            self._apply_class_limits(torch.full((self.batch,), -1, dtype=torch.int32, device=self.device))
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.rda_set_robot_class_index(self._h, None, self._stream()), 'rda_set_robot_class_index')
            _cabi.check(self.lib.rda_set_robot_classes(self._h, 0, None, self._stream()), 'rda_set_robot_classes')
        self._graphs.clear()
        self._classes = self._class_index = None

    def robot_class_index(self):
        """The installed class index [B] (a copy; -1 for an index outside the classes), or None."""
        return None if self._class_index is None else self._class_index.clone()

    def class_slot(self, index=None):
        """Slot of each instance in tables of K + 1 class rows [B] (int64, on the device): its class, or K for an index
        outside the classes (the constructor's car_tuple)."""
        index = self._class_index if index is None else index
        K = len(self._classes)
        return torch.where((index >= 0) & (index < K), index, torch.full_like(index, K)).long()

    def _class_index_tensor(self, robot_class, K=None):
        """robot_class as int32 [B] on the device, every value outside [0, K) made -1 before the narrowing (so that a
        wide integer cannot wrap into a valid class)."""
        B, K = self.batch, len(self._classes) if K is None else K
        if isinstance(robot_class, torch.Tensor):
            if robot_class.dim() not in (0, 1) or (robot_class.dim() == 1 and robot_class.shape != (B,)) \
                    or robot_class.is_floating_point() or robot_class.dtype == torch.bool:
                raise ValueError(f'robot_class: expected an integer tensor of shape ({B},), got {robot_class.dtype} '
                                 f'{tuple(robot_class.shape)}')
            x = robot_class.to(self.device).expand(B)
            return torch.where((x >= 0) & (x < K), x, torch.full_like(x, -1)).to(torch.int32).contiguous()
        a = np.asarray(robot_class)
        if a.ndim == 0:
            a = np.full(B, a)
        if a.shape != (B,) or not np.issubdtype(a.dtype, np.integer):
            raise ValueError(f'robot_class: expected integers of shape ({B},), got {a.dtype} {a.shape}')
        a = np.where((a >= 0) & (a < K), a, -1).astype(np.int32)
        return torch.as_tensor(a, device=self.device)

    def _apply_class_limits(self, index, robots=None):
        """max_speed / max_acce of each instance's class (the constructor's for an index outside the classes) into the
        rows of the robots of mask robots (None: all) of the per-instance table, gathered on the device."""
        slot = self.class_slot(index)
        ms, ma = self._class_limits
        self.set_instance_parameters(robots, max_speed=ms[slot], max_acce=ma[slot])

    def _install_class_index(self, index, previous):
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.rda_set_robot_class_index(self._h, C.c_void_p(index.data_ptr()), self._stream()),
                        'rda_set_robot_class_index')
        if previous is None:
            self._graphs.clear()    # captured launches carry "no classes"; a later index is seen by a replay
        self._class_index = index   # the copy into the handle's storage reads it on the current stream
        self._apply_class_limits(index, None if previous is None else self.class_slot(index) != self.class_slot(previous))

    # ------------------------------------------------------------------ warm start that follows the obstacles
    def set_obstacle_ids(self, ids):
        """ids [B, N] (array-like or CUDA tensor, int32 values; < 0: no obstacle): the obstacle each slot holds in the next
        solve, as the *_batch conversions return them with ids=True.  When ids of an earlier call are held, each
        instance's per-slot warm start (lam, mu, z, xi, zeta and the su-QP coefficients) moves with its obstacles: the
        k-th slot carrying id X takes the state of the k-th slot that carried X; a slot without a match starts cold.
        The first call only stores the ids; None forgets them (the reference's behaviour: the state stays in its slot).
        reset() and cold_start() keep them.  One kernel on the current stream, no host synchronisation."""
        with torch.cuda.device(self.device):
            if ids is None:
                _cabi.check(self.lib.rda_set_obstacle_ids(self._h, None, self._stream()), 'rda_set_obstacle_ids')
                self._keep_ids = None
                return
            t = torch.as_tensor(ids, device=self.device).to(torch.int32).reshape(self.batch, self.max_obs_num)
            t = t.contiguous()
            if self.max_obs_num == 0:
                return
            _cabi.check(self.lib.rda_set_obstacle_ids(self._h, C.c_void_p(t.data_ptr()), self._stream()),
                        'rda_set_obstacle_ids')
            self._keep_ids = t          # read asynchronously on the current stream

    def get_adjust_parameter(self):
        t = _cabi.Tunables()
        _cabi.check(self.lib.rda_get_tunables(self._h, C.byref(t)), 'rda_get_tunables')
        out = dict(self._tun_py)          # exact Python values, as the reference returns them (:1055-1056)
        for k in out:                      # ... unless the handle was changed behind this object's back
            if abs(float(getattr(t, k)) - float(out[k])) > 1e-6 * (1 + abs(float(out[k]))):
                out[k] = float(getattr(t, k))
        out.update(ws=self.ws, wu=self.wu)
        return out

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def reset(self):
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.rda_reset(self._h, self._stream()), 'rda_reset')

    def cold_start(self):
        """Extension: forget every warm-start quantity (constructor state)."""
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.rda_cold_start(self._h, self._stream()), 'rda_cold_start')

    def buffer_count(self, buf_id):
        ptr, cnt = C.c_void_p(), C.c_size_t()
        _cabi.check(self.lib.rda_get_buffer(self._h, buf_id, C.byref(ptr), C.byref(cnt)), 'rda_get_buffer')
        return cnt.value

    def state_buffer(self, buf_id, shape=None):
        """Copy of a persistent device buffer (checkpointing / tests)."""
        dtype = torch.int32 if buf_id == _cabi.BUF_COUNTERS else torch.float32
        out = torch.empty(self.buffer_count(buf_id), dtype=dtype, device=self.device)
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.rda_copy_buffer(self._h, buf_id, out.data_ptr(), 0, self._stream()),
                        'rda_copy_buffer')
        return out if shape is None else out.reshape(shape)

    def load_state_buffer(self, buf_id, values):
        """Overwrite a persistent device buffer (resume / tests)."""
        dtype = torch.int32 if buf_id == _cabi.BUF_COUNTERS else torch.float32
        src = torch.as_tensor(values, dtype=dtype, device=self.device).contiguous().reshape(-1)
        if src.numel() != self.buffer_count(buf_id):
            raise ValueError('wrong element count')
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.rda_copy_buffer(self._h, buf_id, src.data_ptr(), 1, self._stream()),
                        'rda_copy_buffer')
        self._keep_state = src

    # ------------------------------------------------------------------ solve
    def _inputs(self, nom_s, nom_u, ref_s, ref_speed, obs_A, obs_b, obs_kind, obs_count, time_varying):
        B, T, N, E = self.batch, self.T, self.max_obs_num, self.max_edge_num
        dev = self.device
        t = {
            'nom_s': _as_cuda_f32(nom_s, dev).reshape(B, 3, T + 1),
            'nom_u': _as_cuda_f32(nom_u, dev).reshape(B, 2, T),
            'ref_s': _as_cuda_f32(ref_s, dev).reshape(B, 3, T + 1),
            'ref_speed': _as_cuda_f32(ref_speed, dev).reshape(B),
        }
        Tc = T + 1 if time_varying else 1
        if N > 0:
            t['obs_A'] = _as_cuda_f32(obs_A, dev).reshape(B, N, Tc, E, 2)
            t['obs_b'] = _as_cuda_f32(obs_b, dev).reshape(B, N, Tc, E)
            t['obs_kind'] = torch.as_tensor(obs_kind, dtype=torch.int32, device=dev).reshape(B, N).contiguous()
            t['obs_count'] = torch.as_tensor(obs_count, dtype=torch.int32, device=dev).reshape(B).contiguous()
        inp = _cabi.Inputs()
        for k in ('nom_s', 'nom_u', 'ref_s', 'ref_speed', 'obs_A', 'obs_b', 'obs_kind', 'obs_count'):
            setattr(inp, k, t[k].data_ptr() if k in t else None)
        inp.obs_time_varying = int(bool(time_varying))
        self._keep = t          # the kernels read these buffers asynchronously
        self._keep_tv = inp.obs_time_varying
        return inp

    def _outputs(self):
        o = _cabi.Outputs()
        o.u_opt, o.s_opt = self._out['u'].data_ptr(), self._out['s'].data_ptr()
        o.resi_pri, o.resi_dual = self._out['resi_pri'].data_ptr(), self._out['resi_dual'].data_ptr()
        o.status, o.iters = self._out['status'].data_ptr(), self._out['iters'].data_ptr()
        return o

    def iterative_solve_batch(self, nom_s, nom_u, ref_s, ref_speed, obs_A=None, obs_b=None, obs_kind=None,
                              obs_count=None, time_varying=False, iter_num=None, iter_threshold=None):
        """B instances at once.  Arguments are array-likes or CUDA tensors with the layouts of
        include/rda_b200.h; returns a dict of CUDA tensors (u [B,2,T], s [B,3,T+1], resi_pri,
        resi_dual, status, iters) valid on the current stream.  No host synchronisation."""
        inp = self._inputs(nom_s, nom_u, ref_s, ref_speed, obs_A, obs_b, obs_kind, obs_count, time_varying)
        out = self._outputs()
        it = self.iter_num if iter_num is None else iter_num
        thr = self.iter_threshold if iter_threshold is None else iter_threshold
        if self.use_graph:
            # one graph per (input buffers, iteration count, threshold): the launches read the inputs through
            # their addresses, so a replay is valid exactly while the caller reuses the same tensors
            key = (tuple(int(getattr(inp, k) or 0) for k in ('nom_s', 'nom_u', 'ref_s', 'ref_speed', 'obs_A', 'obs_b',
                                                              'obs_kind', 'obs_count')), int(inp.obs_time_varying), int(it), float(thr))
            g = self._graphs.get(key)
            if g is None:
                cur = torch.cuda.current_stream(self.device)
                side = torch.cuda.Stream(self.device)
                side.wait_stream(cur)
                g = torch.cuda.CUDAGraph()
                with torch.cuda.stream(side):
                    with torch.cuda.graph(g, stream=side):
                        _cabi.check(self.lib.rda_solve(self._h, C.byref(inp), C.byref(out), int(it), float(thr),
                                                       self._stream()), 'rda_solve (graph capture)')
                cur.wait_stream(side)
                if len(self._graphs) >= 8:
                    self._graphs.pop(next(iter(self._graphs)))
                self._graphs[key] = (g, self._keep)          # keep the captured input tensors alive
                g = self._graphs[key]
            g[0].replay()
            return self._out
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.rda_solve(self._h, C.byref(inp), C.byref(out), int(it), float(thr),
                                           self._stream()), 'rda_solve')
        return self._out

    # phase API (rda_begin / rda_step_su / rda_step_lammuz / rda_finish): unit tests, profiling
    def begin(self, nom_s, nom_u, ref_s, ref_speed, obs_A=None, obs_b=None, obs_kind=None, obs_count=None,
              time_varying=False, iter_threshold=None):
        inp = self._inputs(nom_s, nom_u, ref_s, ref_speed, obs_A, obs_b, obs_kind, obs_count, time_varying)
        thr = self.iter_threshold if iter_threshold is None else iter_threshold
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.rda_begin(self._h, C.byref(inp), float(thr), self._stream()), 'rda_begin')

    def step_su(self):
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.rda_step_su(self._h, self._stream()), 'rda_step_su')

    def step_lammuz(self):
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.rda_step_lammuz(self._h, self._stream()), 'rda_step_lammuz')

    def finish(self):
        out = self._outputs()
        with torch.cuda.device(self.device):
            _cabi.check(self.lib.rda_finish(self._h, C.byref(out), self._stream()), 'rda_finish')
        return self._out

    def launch_count(self):
        return self.lib.rda_last_launch_count(self._h)

    def plan_clearance(self, s=None, per_cell=False):
        """How close each plan comes to its obstacles (rda_plan_clearance): the signed distance between the robot body
        (its class's, or the constructor's) placed at every pose s[b, :, t] and every obstacle the last solve (or begin)
        received, at that obstacle's stage-t copy; negative where the body overlaps the obstacle (minus the penetration
        depth).  The pose is the true footprint of column t: position and heading of the same column.  s: CUDA tensor
        or array-like [B, 3, T+1]; default the last solve's s (e.g. pass nom_s, or the current state repeated, for a
        check at the current pose).  Returns a dict of CUDA tensors: 'min' [B] float32 (the smallest distance of the
        instance, +inf without obstacles) and 'index' [B] int32 (the smallest o * (T+1) + t attaining it, -1 without
        obstacles), plus 'map' [B, N, T+1] (padding slots +inf) with per_cell.  Nothing the solver holds changes; no
        host synchronisation.  Raises before the first solve."""
        if self._keep is None:
            raise RuntimeError('plan_clearance needs the obstacles of a solve: call a solve (or begin) first')
        B, T, N, dev = self.batch, self.T, self.max_obs_num, self.device
        if s is None:
            s = self._out['s']
        else:
            s = _as_cuda_f32(s, dev)
            if tuple(s.shape) != (B, 3, T + 1):
                raise ValueError(f's: expected shape ({B}, 3, {T + 1}), got {tuple(s.shape)}')
        out = {'min': torch.empty(B, dtype=torch.float32, device=dev),
               'index': torch.empty(B, dtype=torch.int32, device=dev)}
        if per_cell:
            out['map'] = torch.empty((B, N, T + 1), dtype=torch.float32, device=dev)
        inp = _cabi.Inputs()
        for k in ('obs_A', 'obs_b', 'obs_kind', 'obs_count'):
            setattr(inp, k, self._keep[k].data_ptr() if k in self._keep else None)
        inp.obs_time_varying = self._keep_tv
        with torch.cuda.device(dev):
            _cabi.check(self.lib.rda_plan_clearance(self._h, C.byref(inp), C.c_void_p(s.data_ptr()),
                                                    C.c_void_p(out['map'].data_ptr()) if per_cell else None,
                                                    C.c_void_p(out['min'].data_ptr()),
                                                    C.c_void_p(out['index'].data_ptr()), self._stream()),
                        'rda_plan_clearance')
        return out

    def _solve_static(self, nom_s, nom_u, ref, ref_speed, A, b, kind, count, tv):
        """graph=True, single instance: inputs are staged into persistent device buffers (one pinned host block, one
        H2D copy each) so that the captured graph of the solve can be replayed every control step."""
        T, N, E, dev = self.T, self.max_obs_num, self.max_edge_num, self.device
        Tc = T + 1 if tv else 1
        if self._static is None or self._static['Tc'] != Tc:
            z = lambda *sh, dt=torch.float32: torch.zeros(sh, dtype=dt, device=dev)
            self._static = {'Tc': Tc, 'nom_s': z(1, 3, T + 1), 'nom_u': z(1, 2, T), 'ref_s': z(1, 3, T + 1), 'ref_speed': z(1),
                            'obs_A': z(1, max(N, 1), Tc, E, 2), 'obs_b': z(1, max(N, 1), Tc, E),
                            'obs_kind': z(1, max(N, 1), dt=torch.int32), 'obs_count': z(1, dt=torch.int32)}
            self._graphs.clear()
        st = self._static
        st['nom_s'].copy_(torch.as_tensor(nom_s, dtype=torch.float32)[None])
        st['nom_u'].copy_(torch.as_tensor(nom_u, dtype=torch.float32)[None])
        st['ref_s'].copy_(torch.as_tensor(ref, dtype=torch.float32)[None])
        st['ref_speed'].fill_(ref_speed)
        if N > 0:
            st['obs_A'].copy_(torch.as_tensor(A, dtype=torch.float32)[None])
            st['obs_b'].copy_(torch.as_tensor(b, dtype=torch.float32)[None])
            st['obs_kind'].copy_(torch.as_tensor(kind, dtype=torch.int32)[None])
        st['obs_count'].fill_(int(count))
        return self.iterative_solve_batch(st['nom_s'], st['nom_u'], st['ref_s'], st['ref_speed'],
                                          st['obs_A'] if N > 0 else None, st['obs_b'] if N > 0 else None,
                                          st['obs_kind'] if N > 0 else None, st['obs_count'] if N > 0 else None, tv)

    def iterative_solve(self, nom_s, nom_u, ref_states, ref_speed, obstacle_list, **kwargs):
        """Reference signature (:573): numpy in, (u (2,T) ndarray, info dict) out."""
        if self.batch != 1:
            raise RuntimeError('iterative_solve is the single-instance API; use iterative_solve_batch')
        T, N, E = self.T, self.max_obs_num, self.max_edge_num
        start = time.time()
        ref = np.hstack(ref_states)[0:3, :]                                     # :580
        if N > 0:
            A, b, kind, count, tv = pack_obstacles(obstacle_list, T, N, E, center=np.asarray(nom_s, float)[0:2, 0],
                                                   bound=self._hs_bound)
        else:
            A = b = kind = None
            count, tv = len(obstacle_list), False
        self.obstacle_num = len(obstacle_list)
        if self.use_graph:
            res = self._solve_static(np.asarray(nom_s, float), np.asarray(nom_u, float), ref, float(ref_speed), A, b, kind,
                                     count, tv)
        else:
            res = self.iterative_solve_batch(np.asarray(nom_s, float)[None], np.asarray(nom_u, float)[None],
                                             ref[None], np.array([ref_speed], float),
                                             None if A is None else A[None], None if b is None else b[None],
                                             None if kind is None else kind[None], np.array([count]), tv)
        u = res['u'][0].double().cpu().numpy()
        s = res['s'][0].double().cpu().numpy()
        info = {'ref_traj_list': ref_states, 'opt_state_list': [s[:, t:t + 1] for t in range(T + 1)],
                'iteration_time': time.time() - start,
                'resi_dual': float(res['resi_dual'][0]), 'resi_pri': float(res['resi_pri'][0]),
                'status': int(res['status'][0]), 'iterations': int(res['iters'][0])}
        if self.time_print:
            print('iterations:', info['iterations'], ' time:', info['iteration_time'])
        return u, info
