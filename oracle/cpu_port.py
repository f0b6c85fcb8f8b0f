"""TEST / BASELINE INFRASTRUCTURE — Python wrapper of oracle/cpu_port (compiled C++/OpenMP port
of the hot path: same algorithm as the CUDA kernels, run on the host cores).  Used by bench.py
as the CPU baseline / reference arm and by tests as a fast cross-check of the numpy oracle."""
import ctypes as C
import os

import numpy as np

from rda_planner_b200._cabi import DYNAMICS as _DYN

from . import build_port


class _Config(C.Structure):
    _fields_ = [('batch', C.c_int), ('receding', C.c_int), ('max_obs_num', C.c_int),
                ('max_edge_num', C.c_int), ('robot_edges', C.c_int), ('dynamics', C.c_int),
                ('accelerated', C.c_int), ('su_fp64', C.c_int), ('step_time', C.c_float),
                ('wheelbase', C.c_float), ('max_speed', C.c_float * 2), ('acce_bound', C.c_float * 2),
                ('ws', C.c_float), ('wu', C.c_float), ('G', C.c_float * 16), ('h', C.c_float * 8),
                ('robot_cone', C.c_int)]


class _Tunables(C.Structure):
    _fields_ = [('slack_gain', C.c_float), ('max_sd', C.c_float), ('min_sd', C.c_float),
                ('ro1', C.c_float), ('ro2', C.c_float), ('z_theta', C.c_float)]


_LIB = None


def _lib():
    """Build (if stale) and load the port ONCE per process — never inside a timed loop."""
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build_port.build())
        _LIB.port_solve_batch.restype = C.c_int
    return _LIB


def host_threads():
    """Threads this process may really use: min(affinity mask, cgroup CPU quota), with the raw numbers.
    os.cpu_count() reports the machine, not the lease: a 1-GPU lease of a 128-core box is typically pinned
    or quota-limited to a fraction of it, and oversubscribing OpenMP threads makes the baseline noisy."""
    import math
    import os
    aff = len(os.sched_getaffinity(0)) if hasattr(os, 'sched_getaffinity') else (os.cpu_count() or 1)
    quota = None
    try:
        q, per = open('/sys/fs/cgroup/cpu.max').read().split()[:2]
        if q != 'max':
            quota = float(q) / float(per)
    except Exception:
        try:
            q = int(open('/sys/fs/cgroup/cpu/cpu.cfs_quota_us').read())
            per = int(open('/sys/fs/cgroup/cpu/cpu.cfs_period_us').read())
            if q > 0:
                quota = q / per
        except Exception:
            pass
    eff = aff if quota is None else max(1, min(aff, int(math.floor(quota + 1e-9))))
    return {'effective': eff, 'affinity': aff, 'cgroup_quota': quota, 'os_cpu_count': os.cpu_count()}


def _config(car, T, N, E, B, dt, accelerated, **kw):
    """The rda_config / rda_tunables pair of a solve of B instances: car's body, dynamics and limits, the weights and
    tunables of kw (ws, wu, slack_gain, max_sd, min_sd, ro1, ro2, z_theta; RDA_solver's defaults for those left out)."""
    G = np.asarray(car.G, float); h = np.asarray(car.h, float).ravel()
    cfg = _Config()
    cfg.batch, cfg.receding, cfg.max_obs_num, cfg.max_edge_num, cfg.robot_edges = B, T, N, E, G.shape[0]
    cfg.dynamics, cfg.accelerated, cfg.su_fp64 = _DYN[car.dynamics], int(accelerated), 1
    cfg.step_time, cfg.wheelbase = dt, float(car.wheelbase)
    for k in range(2):
        cfg.max_speed[k] = float(car.max_speed[k])
        cfg.acce_bound[k] = float(car.max_acce[k]) * dt
    cfg.ws, cfg.wu = kw.get('ws', 1), kw.get('wu', 1)
    for j in range(G.shape[0]):
        cfg.G[2 * j], cfg.G[2 * j + 1], cfg.h[j] = G[j, 0], G[j, 1], h[j]
    cfg.robot_cone = 1 if getattr(car, 'cone_type', 'Rpositive') == 'norm2' else 0
    tun = _Tunables(kw.get('slack_gain', 8), kw.get('max_sd', 1.0), kw.get('min_sd', 0.1), kw.get('ro1', 200),
                    kw.get('ro2', 1), kw.get('z_theta', 0.5))
    return cfg, tun


def _inputs(nom_s, nom_u, ref_s, ref_speed, obs_A, obs_b, obs_kind, obs_count):
    """The input arrays of port_solve_batch, contiguous, in its argument order."""
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    i32 = lambda a: np.ascontiguousarray(a, np.int32)
    return [f32(nom_s), f32(nom_u), f32(ref_s), f32(ref_speed), f32(obs_A), f32(obs_b), i32(obs_kind), i32(obs_count)]


def _outputs(B, T):
    """Zeroed output arrays of port_solve_batch, in its argument order, under the keys solve_batch returns."""
    return {'u': np.zeros((B, 2, T), np.float32), 's': np.zeros((B, 3, T + 1), np.float32),
            'resi_pri': np.zeros(B, np.float32), 'resi_dual': np.zeros(B, np.float32), 'iters': np.zeros(B, np.int32),
            'cell_failures': np.zeros((B, 4), np.int32)}


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def solve_batch(car, T, N, E, nom_s, nom_u, ref_s, ref_speed, obs_A, obs_b, obs_kind, obs_count,
                time_varying=False, iter_num=50, iter_threshold=0.0, dt=0.1, accelerated=True, threads=0,
                **kw):
    lib = _lib()
    B = int(np.asarray(nom_s).shape[0])
    cfg, tun = _config(car, T, N, E, B, dt, accelerated, **kw)
    arrs = _inputs(nom_s, nom_u, ref_s, ref_speed, obs_A, obs_b, obs_kind, obs_count)
    out = _outputs(B, T)
    rc = lib.port_solve_batch(C.byref(cfg), C.byref(tun), C.c_int(B), *map(_p, arrs), C.c_int(int(time_varying)),
                              C.c_int(iter_num), C.c_float(iter_threshold), *map(_p, out.values()), C.c_int(threads))
    if rc != 0:
        raise RuntimeError(f'port_solve_batch: {rc}')
    return out
