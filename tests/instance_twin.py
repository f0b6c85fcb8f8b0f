"""ctypes access to the instance-parameter twin of the CPU twin library (tests/cpu_twin/instance_params.cpp): the g++
build of the kernels' cores (oracle/cpu_port) with a per-instance parameter table, each instance's row selected by the
kernels' own helpers — test infrastructure only."""
import ctypes as C

import numpy as np

import shim
from oracle import cpu_port

INST_PARAMS = 11


def solve_batch(car, T, N, E, nom_s, nom_u, ref_s, ref_speed, obs_A, obs_b, obs_kind, obs_count, time_varying=False,
                iter_num=50, iter_threshold=0.0, dt=0.1, accelerated=True, threads=0, inst=None, **kw):
    """oracle.cpu_port.solve_batch with inst: None, or a table [B, RDA_INST_PARAMS] (float32, columns RDA_IP_*) whose
    row b replaces the limits, weights and tunables of car / kw for instance b, as rda_set_instance_params does."""
    B = int(np.asarray(nom_s).shape[0])
    cfg, tun = cpu_port._config(car, T, N, E, B, dt, accelerated, **kw)
    arrs = cpu_port._inputs(nom_s, nom_u, ref_s, ref_speed, obs_A, obs_b, obs_kind, obs_count)
    if inst is not None:
        inst = np.ascontiguousarray(inst, np.float32)
        if inst.shape != (B, INST_PARAMS):
            raise ValueError(f'inst: expected shape ({B}, {INST_PARAMS}), got {inst.shape}')
    out = cpu_port._outputs(B, T)
    p = cpu_port._p
    fn = shim.lib().twin_solve_batch_inst
    fn.restype = C.c_int
    rc = fn(C.byref(cfg), C.byref(tun), C.c_int(B), *map(p, arrs), C.c_int(int(time_varying)), C.c_int(iter_num),
            C.c_float(iter_threshold), *map(p, out.values()), C.c_int(threads), None if inst is None else p(inst))
    if rc != 0:
        raise RuntimeError(f'twin_solve_batch_inst: {rc}')
    return out
