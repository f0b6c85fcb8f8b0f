"""ctypes access to tests/_build/librda_twins.so: the g++ build of the CUDA kernels' numerical cores (oracle/cpu_port)
linked with every CPU twin of tests/cpu_twin — test infrastructure only.  This module builds and loads the library; the
*_twin modules wrap their own entry points of it.  A new twin is one tests/cpu_twin/*.cpp file."""
import ctypes as C
import glob
import os
import sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import build_port
from rda_planner_b200._cabi import DYNAMICS as DYN

SO = os.path.join(HERE, '_build', 'librda_twins.so')


class SuParams(C.Structure):
    _fields_ = [('T', C.c_int), ('N', C.c_int), ('dynamics', C.c_int), ('accelerated', C.c_int),
                ('dt', C.c_float), ('L', C.c_float), ('umax', C.c_float * 2), ('ab', C.c_float * 2),
                ('ws', C.c_float), ('wu', C.c_float), ('slack_gain', C.c_float), ('dmin', C.c_float),
                ('dmax', C.c_float), ('ro1', C.c_float), ('ro2', C.c_float), ('max_iter', C.c_int),
                ('mu0', C.c_float), ('prune', C.c_float)]


def build(force=False):
    srcs = [build_port.SRC] + sorted(glob.glob(os.path.join(HERE, 'cpu_twin', '*.cpp')))
    return build_port.build_so(srcs, SO, force)


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def cell(G, h, kind, A, b, p, phi, dbar, zeta, xi, ro2, theta=0.5, prec='d'):
    G = _f32(G); h = _f32(np.ravel(h)); A = _f32(A); b = _f32(np.ravel(b))
    out = np.zeros(28)
    fn = getattr(lib(), 'shim_cell_' + prec)
    fn.restype = C.c_int
    rc = fn(_p(G), _p(h), C.c_int(G.shape[0]), C.c_int(kind), C.c_int(A.shape[0]), _p(A), _p(b),
            C.c_double(p[0]), C.c_double(p[1]), C.c_double(phi), C.c_double(dbar), C.c_double(zeta),
            C.c_double(xi[0]), C.c_double(xi[1]), C.c_double(ro2), C.c_double(theta), _p(out))
    assert rc == 0, rc
    E, R = A.shape[0], G.shape[0]
    keys = ['z', 'zeta_new', 'xi0', 'xi1', 'ax', 'ay', 'c0', 'gx', 'gy', 'hm0', 'hm1', 'path']
    r = {k: out[16 + i] for i, k in enumerate(keys)}
    r['lam'] = out[:E].copy(); r['mu'] = out[8:8 + R].copy(); r['path'] = int(r['path'])
    return r


def cell_disc_robot(h, kind, A, b, p, phi, dbar, zeta, xi, ro2, theta=0.5, prec='d'):
    """Cell of a DISC body (cone_type 'norm2', G = [[1,0],[0,1],[0,0]], h = (cx, cy, -r)): cell_disc_robot.cuh."""
    h = _f32(np.ravel(h)); A = _f32(A); b = _f32(np.ravel(b))
    out = np.zeros(28)
    fn = getattr(lib(), 'shim_cell_dr_' + prec)      # prec 'barrier_d': searched closed forms off (float64)
    fn.restype = C.c_int
    rc = fn(_p(h), C.c_int(kind), C.c_int(A.shape[0]), _p(A), _p(b), C.c_double(p[0]), C.c_double(p[1]), C.c_double(phi),
            C.c_double(dbar), C.c_double(zeta), C.c_double(xi[0]), C.c_double(xi[1]), C.c_double(ro2), C.c_double(theta), _p(out))
    assert rc == 0, rc
    E = A.shape[0]
    keys = ['z', 'zeta_new', 'xi0', 'xi1', 'ax', 'ay', 'c0', 'gx', 'gy', 'hm0', 'hm1', 'path']
    r = {k: out[16 + i] for i, k in enumerate(keys)}
    r['lam'] = out[:E].copy(); r['mu'] = out[8:11].copy(); r['path'] = int(r['path'])
    return r


def su(params, lins, linu, ref, vref, dis, hx, hy, hc, gx, gy, pref, prec='d', report=False):
    """One su-QP solve: (s, u, d, status, interior point iterations); with report=True also a dict of the pruned
    solve's repeat: restarts (1: repeated with all hinges), verified (the pruned attempt converged and its left-out
    hinges were checked), violated (that check found one with l < 0), capped (the repeat was caused by the pruned
    attempt's iteration cap, not by the check)."""
    T, N = params.T, params.N
    lins = _f64(np.asarray(lins).T); linu = _f64(np.asarray(linu).T); ref = _f64(np.asarray(ref).T)
    pref = _f64(np.asarray(pref).T); dis = _f64(np.ravel(dis))
    hx, hy, hc, gx, gy = (_f32(np.asarray(a).reshape(N, T)) for a in (hx, hy, hc, gx, gy))
    s = np.zeros((T + 1, 3)); u = np.zeros((T, 2)); d = np.zeros(T)
    it = C.c_int(0)
    rep = np.zeros(3, np.int32)
    fn = getattr(lib(), ('shim_su_report_' if report else 'shim_su_') + prec)
    fn.restype = C.c_int
    extra = (_p(rep),) if report else ()
    st = fn(C.byref(params), _p(lins), _p(linu), _p(ref), C.c_double(vref), _p(dis), _p(hx), _p(hy), _p(hc),
            _p(gx), _p(gy), _p(pref), _p(s), _p(u), _p(d), C.byref(it), *extra)
    out = (s.T.copy(), u.T.copy(), d, st, it.value)
    if not report:
        return out
    r = {'restarts': int(rep[0]), 'verified': int(rep[1]), 'violated': int(rep[2])}
    r['capped'] = int(r['restarts'] == 1 and r['verified'] == 0)
    return out + (r,)


# ---- front end cores (frontend.cuh) ----
def pre_process(dynamics, T, dt, L, state, vel, ref_speed, path, start_index, threshold=0.1, ind_range=10):
    state, vel, path = _f32(np.ravel(state)[:3]), _f32(vel), _f32(path)
    nom = np.zeros((3, T + 1), np.float32)
    ref = np.zeros((3, T + 1), np.float32)
    f = lib().shim_pre_process
    f.restype = C.c_int
    f.argtypes = [C.c_int, C.c_int, C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_int,
                  C.c_int, C.c_double, C.c_int, C.c_void_p, C.c_void_p]
    near = f(DYN[dynamics], T, dt, L, state.ctypes.data, vel.ctypes.data, ref_speed, path.ctypes.data, path.shape[0],
             start_index, threshold, ind_range, nom.ctypes.data, ref.ctypes.data)
    return nom, ref, near


def convert_obstacles(shapes, N, T, E, dt, time_varying, order, state):
    """shapes: dict of arrays kind [M], nv [M], xy [M,8,2], radius [M], vel [M,2], count."""
    M = len(shapes['kind'])
    Tc = T + 1 if time_varying else 1
    A = np.zeros((N, Tc, E, 2), np.float32)
    b = np.zeros((N, Tc, E), np.float32)
    kind = np.zeros(N, np.int32)
    st = _f32(np.ravel(state)[:3])
    k = np.ascontiguousarray(shapes['kind'], np.int32)
    nv = np.ascontiguousarray(shapes['nv'], np.int32)
    xy, rad, vel = _f32(shapes['xy']), _f32(shapes['radius']), _f32(shapes['vel'])
    f = lib().shim_convert_obstacles
    f.restype = C.c_int
    f.argtypes = [C.c_int] * 4 + [C.c_double, C.c_int, C.c_int] + [C.c_void_p] * 6 + [C.c_int] + [C.c_void_p] * 3
    cnt = f(M, N, T, E, dt, int(time_varying), int(order), st.ctypes.data, k.ctypes.data, nv.ctypes.data, xy.ctypes.data,
            rad.ctypes.data, vel.ctypes.data, int(shapes['count']), A.ctypes.data, b.ctypes.data, kind.ctypes.data)
    return A, b, kind, cnt


def cell_lean2(G, h, A, b, feat, p, phi, dbar, zeta, theta=0.5):
    """Coherent first pass (cell_lean2.cuh, E = R = 4 build): dict like cell(), plus 'feat'; path 6 = declined."""
    G = _f32(G); h = _f32(np.ravel(h)); A = _f32(A); b = _f32(np.ravel(b))
    out = np.zeros(28)
    fn = lib().shim_cell_lean2_4
    fn.restype = C.c_int
    rc = fn(_p(G), _p(h), C.c_int(G.shape[0]), C.c_int(A.shape[0]), _p(A), _p(b), C.c_int(int(feat)), C.c_double(p[0]),
            C.c_double(p[1]), C.c_double(phi), C.c_double(dbar), C.c_double(zeta), C.c_double(theta), _p(out))
    assert rc == 0, rc
    E, R = A.shape[0], G.shape[0]
    r = {'z': out[16], 'zeta_new': out[17], 'ax': out[20], 'ay': out[21], 'c0': out[22], 'gx': out[23], 'gy': out[24],
         'feat': int(out[25]), 'path': int(out[27]), 'lam': out[:E].copy(), 'mu': out[8:8 + R].copy()}
    return r
