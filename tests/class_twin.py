"""ctypes access to a g++ build of tests/cpu_twin/robot_classes.cpp: the g++ build of the kernels' cores (oracle/cpu_port)
with robot classes, each instance's class picked by the kernels' own helpers — test infrastructure only.  Built on first
use into tests/_build, or into a temporary directory when the tree is read-only."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import cpu_port
from rda_planner_b200 import _cabi
from rda_planner_b200.rda_solver import robot_class_table

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, 'cpu_twin', 'robot_classes.cpp')
CSRC = os.path.join(ROOT, 'rda_planner_b200', 'csrc')
SO = os.path.join(HERE, '_build', 'libclass_twin.so')

_lib = None


def build():
    deps = [SRC, os.path.join(ROOT, 'include', 'rda_b200.h'), os.path.join(ROOT, 'oracle', 'cpu_port', 'rda_cpu_port.cpp')]
    deps += [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    if os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in deps):
        return SO
    so = SO
    if not os.access(HERE, os.W_OK):
        so = os.path.join(tempfile.mkdtemp(prefix='rda_class_twin_'), os.path.basename(SO))
    os.makedirs(os.path.dirname(so), exist_ok=True)
    subprocess.check_call(['g++', '-O3', '-std=c++17', '-fopenmp', '-shared', '-fPIC', '-o', so, SRC])
    return so


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.twin_solve_batch_cls.restype = C.c_int
    return _lib


def solve_batch(car, T, N, E, nom_s, nom_u, ref_s, ref_speed, obs_A, obs_b, obs_kind, obs_count, time_varying=False,
                iter_num=50, iter_threshold=0.0, dt=0.1, accelerated=True, threads=0, classes=(), robot_class=None, **kw):
    """oracle.cpu_port.solve_batch with robot classes: car is the handle's car_tuple, classes a list of car_tuples and
    robot_class [B] (or None) the class of each instance, as RDA_solver.set_robot_classes installs them."""
    G = np.asarray(car.G, float)
    h = np.asarray(car.h, float).ravel()
    B = int(np.asarray(nom_s).shape[0])
    cfg = cpu_port._Config()
    cfg.batch, cfg.receding, cfg.max_obs_num, cfg.max_edge_num, cfg.robot_edges = B, T, N, E, G.shape[0]
    cfg.dynamics, cfg.accelerated, cfg.su_fp64 = cpu_port._DYN[car.dynamics], int(accelerated), 1
    cfg.step_time, cfg.wheelbase = dt, float(car.wheelbase)
    for k in range(2):
        cfg.max_speed[k] = float(car.max_speed[k])
        cfg.acce_bound[k] = float(car.max_acce[k]) * dt
    cfg.ws, cfg.wu = kw.get('ws', 1), kw.get('wu', 1)
    for j in range(G.shape[0]):
        cfg.G[2 * j], cfg.G[2 * j + 1], cfg.h[j] = G[j, 0], G[j, 1], h[j]
    cfg.robot_cone = 1 if getattr(car, 'cone_type', 'Rpositive') == 'norm2' else 0
    tun = cpu_port._Tunables(kw.get('slack_gain', 8), kw.get('max_sd', 1.0), kw.get('min_sd', 0.1), kw.get('ro1', 200),
                             kw.get('ro2', 1), kw.get('z_theta', 0.5))
    classes = list(classes)
    table = robot_class_table(classes, getattr(car, 'cone_type', 'Rpositive'), G.shape[0])
    # the limits each class puts into the per-instance table (max_acce * dt in float64, rounded to float32)
    limits = np.array([[float(c.max_speed[0]), float(c.max_speed[1]), float(c.max_acce[0]) * dt, float(c.max_acce[1]) * dt]
                       for c in classes] or [[0, 0, 0, 0]], np.float32)
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    i32 = lambda a: np.ascontiguousarray(a, np.int32)
    arrs = [f32(nom_s), f32(nom_u), f32(ref_s), f32(ref_speed), f32(obs_A), f32(obs_b), i32(obs_kind), i32(obs_count)]
    rc_arr = None if robot_class is None else i32(robot_class)
    if rc_arr is not None and rc_arr.shape != (B,):
        raise ValueError(f'robot_class: expected shape ({B},), got {rc_arr.shape}')
    u = np.zeros((B, 2, T), np.float32)
    s = np.zeros((B, 3, T + 1), np.float32)
    rp = np.zeros(B, np.float32)
    rd = np.zeros(B, np.float32)
    it = np.zeros(B, np.int32)
    fails = np.zeros((B, 4), np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = lib().twin_solve_batch_cls(C.byref(cfg), C.byref(tun), C.c_int(B), *[p(a) for a in arrs],
                                    C.c_int(int(time_varying)), C.c_int(iter_num), C.c_float(iter_threshold), p(u),
                                    p(s), p(rp), p(rd), p(it), p(fails), C.c_int(threads), C.c_int(len(classes)),
                                    table, p(limits), None if rc_arr is None else p(rc_arr))
    if rc != 0:
        raise RuntimeError(f'twin_solve_batch_cls: {rc}')
    return {'u': u, 's': s, 'resi_pri': rp, 'resi_dual': rd, 'iters': it, 'cell_failures': fails}
