"""ctypes binding of include/rda_b200.h (librda_b200.so, built in-tree by build.py).

There is NO CPU fallback: importing this module without the built CUDA library, or
creating a solver without a CUDA device, raises."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('RDA_B200_LIB') or os.path.join(_HERE, 'librda_b200.so')      # override: tuning experiments only

MAX_EDGE = 8
MAX_ROBOT_EDGE = 8
DYNAMICS = {'acker': 0, 'diff': 1, 'omni': 2}
OBS_POLYGON, OBS_CIRCLE = 0, 1
ROBOT_POLYGON, ROBOT_DISC = 0, 1
E_ARG, E_UNSUPPORTED, E_NOMEM = -1, -2, -3
ST_SU_NOT_CONVERGED, ST_SU_NONFINITE, ST_CELL_FALLBACK, ST_EARLY_STOP = 1, 2, 4, 8
(BUF_LAM, BUF_MU, BUF_Z, BUF_XI, BUF_ZETA, BUF_DIS, BUF_COEF, BUF_PREF, BUF_CUR_S, BUF_CUR_U,
 BUF_COUNTERS) = range(11)
# columns of a per-instance parameter row (rda_set_instance_params)
(IP_MAX_SPEED0, IP_MAX_SPEED1, IP_ACCE_BOUND0, IP_ACCE_BOUND1, IP_WS, IP_WU, IP_SLACK_GAIN, IP_MAX_SD, IP_MIN_SD, IP_RO1,
 IP_RO2) = range(11)
INST_PARAMS = 11
MAX_ROBOT_CLASSES = 16


class Config(C.Structure):
    _fields_ = [('batch', C.c_int), ('receding', C.c_int), ('max_obs_num', C.c_int),
                ('max_edge_num', C.c_int), ('robot_edges', C.c_int), ('dynamics', C.c_int),
                ('accelerated', C.c_int), ('su_fp64', C.c_int), ('step_time', C.c_float),
                ('wheelbase', C.c_float), ('max_speed', C.c_float * 2), ('acce_bound', C.c_float * 2),
                ('ws', C.c_float), ('wu', C.c_float), ('G', C.c_float * (MAX_ROBOT_EDGE * 2)),
                ('h', C.c_float * MAX_ROBOT_EDGE), ('robot_cone', C.c_int)]


class Tunables(C.Structure):
    _fields_ = [('slack_gain', C.c_float), ('max_sd', C.c_float), ('min_sd', C.c_float),
                ('ro1', C.c_float), ('ro2', C.c_float), ('z_theta', C.c_float)]


class RobotClass(C.Structure):
    _fields_ = [('dynamics', C.c_int), ('wheelbase', C.c_float), ('G', C.c_float * (MAX_ROBOT_EDGE * 2)),
                ('h', C.c_float * MAX_ROBOT_EDGE)]


class Inputs(C.Structure):
    _fields_ = [('nom_s', C.c_void_p), ('nom_u', C.c_void_p), ('ref_s', C.c_void_p),
                ('ref_speed', C.c_void_p), ('obs_A', C.c_void_p), ('obs_b', C.c_void_p),
                ('obs_kind', C.c_void_p), ('obs_count', C.c_void_p), ('obs_time_varying', C.c_int)]


class Outputs(C.Structure):
    _fields_ = [('u_opt', C.c_void_p), ('s_opt', C.c_void_p), ('resi_pri', C.c_void_p),
                ('resi_dual', C.c_void_p), ('status', C.c_void_p), ('iters', C.c_void_p)]


EXPORTS = ['rda_create', 'rda_destroy', 'rda_set_tunables', 'rda_get_tunables', 'rda_reset',
           'rda_cold_start', 'rda_solve', 'rda_begin', 'rda_step_su', 'rda_step_lammuz', 'rda_finish',
           'rda_get_buffer', 'rda_copy_buffer', 'rda_last_launch_count', 'rda_version',
           'rda_pre_process', 'rda_convert_obstacles', 'rda_post_process', 'rda_motion_predict',
           'rda_pre_process_curves', 'rda_post_process_gear', 'rda_convert_world_obstacles',
           'rda_pre_process_paths', 'rda_post_process_paths', 'rda_fleet_shapes', 'rda_convert_fleet_obstacles',
           'rda_set_instance_params', 'rda_set_robot_classes', 'rda_set_robot_class_index',
           'rda_pre_process_paths_per_robot', 'rda_motion_predict_per_robot', 'rda_fleet_shapes_per_robot',
           'rda_plan_clearance', 'rda_fleet_plan_shapes', 'rda_convert_fleet_plan_obstacles',
           'rda_convert_world_obstacles_horizon', 'rda_set_obstacle_ids', 'rda_convert_obstacles_ids',
           'rda_convert_world_obstacles_ids', 'rda_convert_world_obstacles_horizon_ids',
           'rda_convert_world_obstacles_traj', 'rda_convert_world_obstacles_horizon_traj']
MAX_SHAPES = 64
MAX_WORLD_SLOTS = 256

_lib = None


def load():
    """Load librda_b200.so; raise (never fall back) when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f'{LIB_PATH} is missing: build the sm_90a CUDA library first '
            '(python -c "import __graft_entry__ as g; g.build()" or python -m rda_planner_b200.build). '
            'rda_planner_b200 has no CPU fallback.')
    lib = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    lib.rda_create.argtypes = [C.POINTER(Config), C.POINTER(Tunables), C.POINTER(vp)]
    lib.rda_destroy.argtypes = [vp]
    lib.rda_set_tunables.argtypes = [vp, C.POINTER(Tunables)]
    lib.rda_get_tunables.argtypes = [vp, C.POINTER(Tunables)]
    lib.rda_set_instance_params.argtypes = [vp, vp, vp]
    lib.rda_set_robot_classes.argtypes = [vp, C.c_int, C.POINTER(RobotClass), vp]
    lib.rda_set_robot_class_index.argtypes = [vp, vp, vp]
    lib.rda_set_obstacle_ids.argtypes = [vp, vp, vp]
    lib.rda_reset.argtypes = [vp, vp]
    lib.rda_cold_start.argtypes = [vp, vp]
    lib.rda_solve.argtypes = [vp, C.POINTER(Inputs), C.POINTER(Outputs), C.c_int, C.c_float, vp]
    lib.rda_begin.argtypes = [vp, C.POINTER(Inputs), C.c_float, vp]
    lib.rda_step_su.argtypes = [vp, vp]
    lib.rda_step_lammuz.argtypes = [vp, vp]
    lib.rda_finish.argtypes = [vp, C.POINTER(Outputs), vp]
    lib.rda_get_buffer.argtypes = [vp, C.c_int, C.POINTER(vp), C.POINTER(C.c_size_t)]
    lib.rda_copy_buffer.argtypes = [vp, C.c_int, vp, C.c_int, vp]
    lib.rda_last_launch_count.argtypes = [vp]
    lib.rda_plan_clearance.argtypes = [vp, C.POINTER(Inputs), vp, vp, vp, vp, vp]
    lib.rda_version.restype = C.c_char_p
    i, f = C.c_int, C.c_float
    lib.rda_pre_process.argtypes = [i, i, i, f, f, vp, vp, vp, vp, i, vp, f, i, vp, vp, vp, vp]
    lib.rda_convert_obstacles.argtypes = [i, i, i, i, i, f, i, i] + [vp] * 12
    lib.rda_convert_world_obstacles.argtypes = [i, i, i, i, i, f, i, i] + [vp] * 13
    lib.rda_post_process.argtypes = [i, i, i, i, vp, vp, vp, vp, vp]
    lib.rda_pre_process_curves.argtypes = [i, i, i, f, f, vp, vp, vp, vp, i, vp, vp, vp, f, i, vp, vp, vp, vp]
    lib.rda_post_process_gear.argtypes = [i, i, i, vp, i, vp, vp, vp, vp, vp, vp]
    lib.rda_pre_process_paths.argtypes = [i, i, i, f, f, vp, vp, vp, vp, i, vp, vp, vp, vp, vp, vp, f, i, vp, vp, vp, vp,
                                          vp]
    lib.rda_post_process_paths.argtypes = [i, i, i, vp, vp, vp, i, vp, vp, vp, vp, vp, vp]
    lib.rda_motion_predict.argtypes = [i, i, i, f, f, vp, vp, vp]
    lib.rda_pre_process_paths_per_robot.argtypes = [i, i, vp, f, vp, vp, vp, vp, vp, i, vp, vp, vp, vp, vp, vp, f, i, vp,
                                                    vp, vp, vp, vp]
    lib.rda_motion_predict_per_robot.argtypes = [i, i, vp, f, vp, vp, vp, vp]
    lib.rda_fleet_shapes_per_robot.argtypes = [i, i, vp, i, i, vp, vp, vp, vp] + [vp] * 6
    lib.rda_fleet_shapes.argtypes = [i, i, i, i, i, vp, f] + [vp] * 8
    lib.rda_convert_fleet_obstacles.argtypes = [i, i, i, i, i, f, i, i] + [vp] * 20
    lib.rda_fleet_plan_shapes.argtypes = [i, i, i, f, f, i, i, vp, f] + [vp] * 13
    lib.rda_convert_fleet_plan_obstacles.argtypes = [i, i, i, i, i, f, i, i] + [vp] * 21
    lib.rda_convert_world_obstacles_horizon.argtypes = [i, i, i, i, i, f, i, vp, vp, i, i, vp, f] + [vp] * 22
    lib.rda_convert_obstacles_ids.argtypes = [i, i, i, i, i, f, i, i] + [vp] * 13
    lib.rda_convert_world_obstacles_ids.argtypes = [i, i, i, i, i, f, i, i] + [vp] * 22
    lib.rda_convert_world_obstacles_horizon_ids.argtypes = [i, i, i, i, i, f, i, vp, vp, i, i, vp, f] + [vp] * 23
    lib.rda_convert_world_obstacles_traj.argtypes = [i, i, i, i, i, f, i, i] + [vp] * 21 + [vp, i, vp, vp]
    lib.rda_convert_world_obstacles_horizon_traj.argtypes = ([i, i, i, i, i, f, i, vp, vp, i, i, vp, f] + [vp] * 22 +
                                                             [vp, i, vp, vp])
    for name in EXPORTS:
        if name != 'rda_version':
            getattr(lib, name).restype = C.c_int
    _lib = lib
    return lib


def check(rc, what):
    if rc == 0:
        return
    if rc < 0:
        names = {-1: 'RDA_E_ARG (bad argument)', -2: 'RDA_E_UNSUPPORTED', -3: 'RDA_E_NOMEM'}
        raise RuntimeError(f'{what}: {names.get(rc, rc)}')
    raise RuntimeError(f'{what}: CUDA error {rc}')
