"""ctypes access to the robot-class twin of the CPU twin library (tests/cpu_twin/robot_classes.cpp): the g++ build of the
kernels' cores (oracle/cpu_port) with robot classes, each instance's class picked by the kernels' own helpers — test
infrastructure only."""
import ctypes as C

import numpy as np

import shim
from oracle import cpu_port
from rda_planner_b200.rda_solver import robot_class_table


def solve_batch(car, T, N, E, nom_s, nom_u, ref_s, ref_speed, obs_A, obs_b, obs_kind, obs_count, time_varying=False,
                iter_num=50, iter_threshold=0.0, dt=0.1, accelerated=True, threads=0, classes=(), robot_class=None, **kw):
    """oracle.cpu_port.solve_batch with robot classes: car is the handle's car_tuple, classes a list of car_tuples and
    robot_class [B] (or None) the class of each instance, as RDA_solver.set_robot_classes installs them."""
    B = int(np.asarray(nom_s).shape[0])
    cfg, tun = cpu_port._config(car, T, N, E, B, dt, accelerated, **kw)
    arrs = cpu_port._inputs(nom_s, nom_u, ref_s, ref_speed, obs_A, obs_b, obs_kind, obs_count)
    classes = list(classes)
    table = robot_class_table(classes, getattr(car, 'cone_type', 'Rpositive'), cfg.robot_edges)
    # the limits each class puts into the per-instance table (max_acce * dt in float64, rounded to float32)
    limits = np.array([[float(c.max_speed[0]), float(c.max_speed[1]), float(c.max_acce[0]) * dt, float(c.max_acce[1]) * dt]
                       for c in classes] or [[0, 0, 0, 0]], np.float32)
    rc_arr = None if robot_class is None else np.ascontiguousarray(robot_class, np.int32)
    if rc_arr is not None and rc_arr.shape != (B,):
        raise ValueError(f'robot_class: expected shape ({B},), got {rc_arr.shape}')
    out = cpu_port._outputs(B, T)
    p = cpu_port._p
    fn = shim.lib().twin_solve_batch_cls
    fn.restype = C.c_int
    rc = fn(C.byref(cfg), C.byref(tun), C.c_int(B), *map(p, arrs), C.c_int(int(time_varying)), C.c_int(iter_num),
            C.c_float(iter_threshold), *map(p, out.values()), C.c_int(threads), C.c_int(len(classes)), table, p(limits),
            None if rc_arr is None else p(rc_arr))
    if rc != 0:
        raise RuntimeError(f'twin_solve_batch_cls: {rc}')
    return out
