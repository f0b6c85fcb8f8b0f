/* rda_b200.h — C ABI of the B200-native RDA ADMM-MPC hot path.
 *
 * The reference (hanruihua/RDA-planner) has no FFI: its boundary is the Python class
 * RDA_planner/rda_solver.py::RDA_solver (constructor :18-22, iterative_solve :573-610,
 * assign_adjust_parameter :426-434, get_adjust_parameter :1055-1056, reset :1060-1068).
 * Each entry point below replaces the reference code cited next to it.  All pointers in
 * rda_inputs / rda_outputs are DEVICE pointers to float32 arrays owned by the caller
 * (PyTorch); the handle owns only the persistent warm-start state the reference keeps in
 * cvxpy Parameters (rda_solver.py:112-182).  No entry point throws, allocates host memory
 * per call, synchronises the device (except create/destroy/export) or falls back to the
 * CPU.  Return value: 0 ok, <0 usage error (RDA_E_*), >0 a cudaError_t.
 */
#ifndef RDA_B200_H
#define RDA_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RDA_MAX_EDGE 8        /* max_edge_num  (obstacle rows)  */
#define RDA_MAX_ROBOT_EDGE 8  /* rows of car_tuple.G            */

enum { RDA_DYN_ACKER = 0, RDA_DYN_DIFF = 1, RDA_DYN_OMNI = 2 };       /* rda_solver.py:446-451 */
enum { RDA_OBS_POLYGON = 0, RDA_OBS_CIRCLE = 1 };                     /* cone flag :158,:512   */
enum { RDA_ROBOT_POLYGON = 0, RDA_ROBOT_DISC = 1 };                   /* car_tuple.cone_type 'Rpositive' / 'norm2', :1034-1039 */
enum { RDA_E_ARG = -1, RDA_E_UNSUPPORTED = -2, RDA_E_NOMEM = -3 };

/* per-instance status bits (device word), mirroring the reference's keep-previous-iterate
 * rules (rda_solver.py:696-700, :791-793) */
enum { RDA_ST_SU_NOT_CONVERGED = 1, RDA_ST_SU_NONFINITE = 2, RDA_ST_CELL_FALLBACK = 4,
       RDA_ST_EARLY_STOP = 8 };

typedef struct rda_config {
  int batch;          /* B planning instances sharing this configuration (reference: 1)  */
  int receding;       /* T   rda_solver.py:34                                            */
  int max_obs_num;    /* N   :38                                                         */
  int max_edge_num;   /* E   :39   (<= RDA_MAX_EDGE)                                      */
  int robot_edges;    /* R = G.shape[0] (<= RDA_MAX_ROBOT_EDGE); 3 for a disc body          */
  int dynamics;       /* RDA_DYN_*  :40                                                  */
  int accelerated;    /* :47                                                             */
  int su_fp64;        /* 1: su-QP interior point arithmetic in float64 (default), 0: float32 */
  float step_time;    /* dt  :43                                                         */
  float wheelbase;    /* L   :36                                                         */
  float max_speed[2]; /* :37                                                             */
  float acce_bound[2];/* max_acce * dt  :44                                              */
  float ws, wu;       /* :218-219 (fixed at construction, as in the reference)           */
  float G[RDA_MAX_ROBOT_EDGE * 2]; /* robot half-spaces, rows CCW (car_tuple.G)          */
  float h[RDA_MAX_ROBOT_EDGE];     /* car_tuple.h                                        */
  int robot_cone;     /* RDA_ROBOT_*: polygon body (rows of G counter-clockwise) or the disc body
                         G = [[1,0],[0,1],[0,0]], h = (cx, cy, -r) of cone_type 'norm2' (:1034-1039) */
} rda_config;

typedef struct rda_tunables {   /* rda_solver.py:185-201, :426-434 */
  float slack_gain, max_sd, min_sd, ro1, ro2;
  float z_theta;        /* tie-break of the slack z in [0, stuff] (DESIGN.md §3); 0.5 default */
} rda_tunables;

/* Columns of a per-instance parameter row (rda_set_instance_params): the limits and weights of rda_config and the
 * tunables of rda_tunables that one instance of a batch may hold on its own.  The body, wheelbase and dynamics come
 * per instance from a robot class (rda_set_robot_classes); only z_theta, T, N, E, dt, the robot cone and R stay per
 * handle. */
enum { RDA_IP_MAX_SPEED0 = 0, RDA_IP_MAX_SPEED1 = 1, /* rda_config.max_speed                   */
       RDA_IP_ACCE_BOUND0 = 2, RDA_IP_ACCE_BOUND1 = 3, /* rda_config.acce_bound (max_acce * dt) */
       RDA_IP_WS = 4, RDA_IP_WU = 5,                 /* rda_config.ws, wu                      */
       RDA_IP_SLACK_GAIN = 6, RDA_IP_MAX_SD = 7, RDA_IP_MIN_SD = 8, RDA_IP_RO1 = 9, RDA_IP_RO2 = 10 };
#define RDA_INST_PARAMS 11

/* A robot class: the part of a car_tuple (G h cone_type wheelbase max_speed max_acce dynamics) that the per-instance
 * parameter table does not hold.  G and h use the handle's robot_edges rows and robot_cone, as in rda_config. */
#define RDA_MAX_ROBOT_CLASSES 16
typedef struct rda_robot_class {
  int dynamics;                    /* RDA_DYN_*                                   */
  float wheelbase;                 /* L; > 0 for RDA_DYN_ACKER                    */
  float G[RDA_MAX_ROBOT_EDGE * 2]; /* robot half-spaces, rows CCW                 */
  float h[RDA_MAX_ROBOT_EDGE];
} rda_robot_class;

/* Inputs of one batched solve.  Layouts (row-major, last index fastest):
 *   nom_s  [B][3][T+1]   nominal states   (iterative_solve arg nom_s,  :573,:584)
 *   nom_u  [B][2][T]     nominal controls (arg nom_u)
 *   ref_s  [B][3][T+1]   reference states (arg ref_states, :580)
 *   ref_speed [B]        (:581)
 *   obs_A  [B][N][Tc][E][2], obs_b [B][N][Tc][E]   half-spaces per obstacle slot and copy
 *          (assign_obstacle_parameter :483-526; rows zero-padded; Tc = T+1 if
 *          obs_time_varying else 1)
 *   obs_kind [B][N] int32 RDA_OBS_*;  obs_count [B] int32 = len(obstacle_list) before padding
 *          (0 => LamMuZ/xi/zeta skipped for that instance, :625)                              */
typedef struct rda_inputs {
  const float *nom_s, *nom_u, *ref_s, *ref_speed;
  const float *obs_A, *obs_b;
  const int32_t *obs_kind, *obs_count;
  int obs_time_varying;
} rda_inputs;

/* Outputs (device): u_opt [B][2][T], s_opt [B][3][T+1] (solution of the last su-QP, :603-610),
 * resi_pri [B], resi_dual [B] (:604-608), status [B] int32 (RDA_ST_*), iters [B] int32.     */
typedef struct rda_outputs {
  float *u_opt, *s_opt, *resi_pri, *resi_dual;
  int32_t *status, *iters;
} rda_outputs;

typedef struct rda_handle rda_handle;

/* RDA_solver.__init__ / definition() (:18-78, :112-201): allocate persistent state, set the
 * reference initial values (all zero, para_dis = 1). */
int rda_create(const rda_config *cfg, const rda_tunables *tun, rda_handle **out);
int rda_destroy(rda_handle *h);
/* assign_adjust_parameter (:426-434) / get_adjust_parameter (:1055-1056) */
int rda_set_tunables(rda_handle *h, const rda_tunables *tun);
int rda_get_tunables(const rda_handle *h, rda_tunables *tun);
/* Per-instance limits, weights and tunables.  params: DEVICE pointer to float32 [B][RDA_INST_PARAMS]
 * (column order RDA_IP_*), copied asynchronously on cuda_stream into storage the handle owns (allocated on the
 * first call, freed by rda_destroy); from the next solve / phase call on, instance b uses row b instead of the
 * handle's rda_config / rda_tunables values.  params = NULL: back to the handle's values for every instance.
 * rda_set_tunables keeps updating the handle's values (rda_get_tunables returns them) while a table is installed,
 * but the table wins for its columns; rda_reset and rda_cold_start leave the table alone.  The values are not
 * checked: that is the caller's side (RDA_solver.set_instance_parameters). */
int rda_set_instance_params(rda_handle *h, const float *params, void *cuda_stream);
/* Robot classes of the handle: classes[0..K) (HOST array, read before the call returns) are checked and uploaded into
 * device storage the handle owns (allocated on the first call for RDA_MAX_ROBOT_CLASSES, freed by rda_destroy).  Each
 * class must have the handle's robot_cone and robot_edges rows; a disc class may have its own centre and radius.  A set-up
 * call: ordered on cuda_stream, not graph-capturable.  K = 0 removes the classes.  Returns RDA_E_ARG for K outside
 * [0, RDA_MAX_ROBOT_CLASSES], dynamics outside RDA_DYN_*, a non-finite wheelbase or an acker class with wheelbase <= 0;
 * RDA_E_UNSUPPORTED for a body the handle's cone and row count cannot take.  Nothing is installed on an error. */
int rda_set_robot_classes(rda_handle *h, int K, const rda_robot_class *classes, void *cuda_stream);
/* The kernel variant (with or without classes) and K are fixed in the launches when a solve is recorded into a CUDA
 * graph: a graph captured before the first rda_set_robot_class_index, after rda_set_robot_class_index(NULL), or before
 * rda_set_robot_classes changed K must be captured again.  A new index copied into the same storage is seen by a
 * replay. */
/* The class of each instance: robot_class is a DEVICE pointer to int32 [B], copied asynchronously on cuda_stream into
 * storage the handle owns (graph-capturable).  From the next solve / phase call on, instance b solves with the body,
 * wheelbase and dynamics of class robot_class[b]; an index outside [0, K) means the handle's own rda_config body,
 * wheelbase and dynamics (decided on the device).  robot_class = NULL: the handle's own for every instance.
 * rda_reset and rda_cold_start leave the classes and the index alone. */
int rda_set_robot_class_index(rda_handle *h, const int32_t *robot_class, void *cuda_stream);
/* Warm start that follows the obstacles (DESIGN.md §7.4).  The front ends choose each instance's obstacles again at every
 * step, so slot n holds whichever obstacle ranks n; by default (as in the reference, assign_obstacle_parameter :483-526)
 * the warm-start state stays in its slot.  obs_id: DEVICE pointer to int32 [B][N], the obstacle that slot n of instance b
 * holds in the next solve (the rda_convert_*_ids calls write them; values < 0: no obstacle, never matched).  When the
 * handle holds the ids of an earlier call, each instance's per-slot state moves with its obstacles: the k-th slot (in
 * slot order) carrying id X takes the state of the k-th slot that carried X, so the padding copies of a repeated last
 * obstacle match copy to copy; a slot without a match gets the values rda_cold_start writes.  The moved state is
 * everything indexed by slot that a solve leaves behind: RDA_BUF_LAM, MU, Z, XI, ZETA, all five planes of COEF, and the
 * coherent pass's support-vertex hints; per-instance state (DIS, PREF, CUR_S, CUR_U, status) stays.  Then the handle
 * keeps obs_id for the next call.  The first call after rda_create or after obs_id = NULL only stores the ids; NULL
 * forgets them (back to the slot behaviour).  rda_reset and rda_cold_start keep the ids.  One kernel on cuda_stream
 * for the whole batch (none when storing), no host synchronisation, no allocation after the first call (the id storage),
 * CUDA-graph capturable (whether a call stores or moves is decided on the host and fixed in a captured graph); not
 * counted in rda_last_launch_count.  RDA_E_UNSUPPORTED for N above 4096 (the kernel's ids in 48 KB of shared memory). */
int rda_set_obstacle_ids(rda_handle *h, const int32_t *obs_id, void *cuda_stream);
/* RDA_solver.reset (:1060-1068): clears lam'A and lam'b only. */
int rda_reset(rda_handle *h, void *cuda_stream);
/* Clear ALL warm-start state back to the constructor values (extension; used by benchmarks). */
int rda_cold_start(rda_handle *h, void *cuda_stream);
/* iterative_solve (:573-610): iter_num ADMM iterations (early stop per instance when both
 * residuals < iter_threshold, :594), enqueued on cuda_stream, no host synchronisation. */
int rda_solve(rda_handle *h, const rda_inputs *in, const rda_outputs *out, int iter_num,
              float iter_threshold, void *cuda_stream);
/* How close each plan comes to its obstacles: for every instance b, stage t = 0..T and obstacle slot o, the signed
 * distance between the robot body placed at the pose s[b][:][t] and obstacle o as the solver receives it at stage t
 * (copy t of obs_A / obs_b when obs_time_varying, else copy 0):
 *     sd(P, Q) = max over unit w of ( min_{x in P} w.x - max_{y in Q} w.y ),
 * the Euclidean distance of disjoint sets and minus the penetration depth of overlapping ones.  The pose is the true
 * footprint of column t (position and heading of the same column), not the solver's pairing of the heading of column
 * t with the position of column t+1.  The body is the instance's robot class's (rda_set_robot_class_index) or the
 * handle's; polygon obstacles are the closed counter-clockwise rows the solve takes, discs rows [[1,0],[0,1],[0,0]] with
 * b = (cx, cy, -r).  Slots o >= min(obs_count[b], N) (the padding copies) are +inf.
 *   s [B][3][T+1] (e.g. rda_outputs.s_opt or rda_inputs.nom_s); dist [B][N][T+1] or NULL;
 *   min_dist [B]: the minimum of the float32 values of instance b over its valid cells, +inf without one;
 *   min_index [B]: the smallest o * (T+1) + t attaining it, -1 without a valid cell.  Cells of a non-finite pose
 *   are written but do not take part in the minimum.
 * Reads only the obstacle fields of `in`; touches no warm-start state, counter or rda_last_launch_count.  One kernel
 * on cuda_stream, no host synchronisation, CUDA-graph capturable; results are bitwise reproducible.  RDA_E_ARG for a
 * NULL h, in, s, min_dist or min_index, or NULL obstacle arrays when N > 0. */
int rda_plan_clearance(rda_handle *h, const rda_inputs *in, const float *s /* [B][3][T+1] */,
                       float *dist /* [B][N][T+1] or NULL */, float *min_dist /* [B] */,
                       int32_t *min_index /* [B] */, void *cuda_stream);
/* Single phases, for unit tests and profiling: begin (load nominal + obstacles), one su-QP
 * (su_prob_solve :692-700 + assign_state_parameter :436-460), one LamMuZ + multiplier update
 * (:702-741, :529-542, :639-690), and the output stage. */
int rda_begin(rda_handle *h, const rda_inputs *in, float iter_threshold, void *cuda_stream);
int rda_step_su(rda_handle *h, void *cuda_stream);
int rda_step_lammuz(rda_handle *h, void *cuda_stream);
int rda_finish(rda_handle *h, const rda_outputs *out, void *cuda_stream);

/* Persistent buffers (device pointers, float32 unless noted), for tests / checkpointing:
 * ids below; returns element count in *count. */
enum { RDA_BUF_LAM = 0,   /* [B][N][E][T]  columns 1..T of para_lam (:141)   */
       RDA_BUF_MU = 1,    /* [B][N][R][T]                        (:142)      */
       RDA_BUF_Z = 2,     /* [B][N][T]                           (:143)      */
       RDA_BUF_XI = 3,    /* [B][2][N][T]  rows 1..T of para_xi  (:144)      */
       RDA_BUF_ZETA = 4,  /* [B][N][T]                           (:145)      */
       RDA_BUF_DIS = 5,   /* [B][T]        para_dis              (:119)      */
       RDA_BUF_COEF = 6,  /* [B][5][N][T]  su-QP hinge inputs: a_x, a_y (lam'A :172), c0, g_x, g_y */
       RDA_BUF_PREF = 7,  /* [B][2][T]     positions c0 refers to            */
       RDA_BUF_CUR_S = 8, /* [B][3][T+1]   current nominal (para_s :117)     */
       RDA_BUF_CUR_U = 9, /* [B][2][T]     para_u (:118)                     */
       RDA_BUF_COUNTERS = 10 /* int32 [8]: cells fast, cells slow, cells fallback, su iterations ... */
};
int rda_get_buffer(rda_handle *h, int id, void **dev_ptr, size_t *count);
/* Copy a persistent buffer to (to_handle = 0) or from (to_handle = 1) caller-owned device
 * memory of the same element count, asynchronously on cuda_stream (checkpoint / resume). */
int rda_copy_buffer(rda_handle *h, int id, void *user_dev_ptr, int to_handle, void *cuda_stream);

/* number of kernels the last rda_solve / phase call enqueued (for bench.py's gpu_launches) */
int rda_last_launch_count(const rda_handle *h);
const char *rda_version(void);

/* ------------------------------------------------------------------------------------------
 * Front end: the steps either side of the solve, batched and stateless (SURVEY.md §8 f1-f3).
 * All pointers are DEVICE pointers; every call only enqueues one kernel on cuda_stream.
 * ------------------------------------------------------------------------------------------ */
#define RDA_MAX_SHAPES 64     /* raw obstacles per instance handed to rda_convert_obstacles (only there) */
#define RDA_MAX_WORLD_SLOTS 256 /* N accepted by rda_convert_world_obstacles (worlds: any size) */

/* MPC.pre_process (mpc.py:251-291) with closest_point :338-353, inter_point :355-383,
 * range_cir_seg :385-423, wraptopi :431-438 and motion_predict_model_* :293-336, for B
 * robots on ONE reference path (rda_pre_process_paths below lets each robot follow its own).
 *   state [B][3]; cur_vel [B][2][T] (the controls of the previous step, MPC.cur_vel_array);
 *   ref_speed [B] (already multiplied by the gear); path [P][3] (x, y, heading);
 *   start_index [B] (MPC.cur_index; NULL = 0); threshold / ind_range: closest_point kwargs
 *   (0.1 / 10).  Out: nom_s, ref_s [B][3][T+1] (the solver's nom_s / ref_s), near_index [B]
 *   (the new MPC.cur_index).                                                              */
int rda_pre_process(int B, int T, int dynamics, float dt, float wheelbase, const float *state,
                    const float *cur_vel, const float *ref_speed, const float *path, int P,
                    const int32_t *start_index, float threshold, int ind_range, float *nom_s,
                    float *ref_s, int32_t *near_index, void *cuda_stream);

/* MPC.convert_rda_obstacle (mpc.py:189-218: conversion + optional distance sort) with
 * convert_inequal_circle :440-458, convert_inequal_polygon :460-474, gen_inequal_global
 * :476-510, is_convex_and_ordered :518-549, followed by RDA_solver.assign_obstacle_parameter
 * (rda_solver.py:483-526: keep the first N, pad a short list by repeating its last element,
 * zero rows beyond the shape's own).  Up to M <= RDA_MAX_SHAPES raw shapes per instance:
 *   shape_kind [B][M] RDA_OBS_*; shape_nv [B][M] vertices of a polygon (3..E);
 *   shape_xy [B][M][RDA_MAX_EDGE][2] polygon vertices, or the disc centre in entry 0;
 *   shape_radius [B][M]; shape_vel [B][M][2]; shape_count [B]; state [B][3] (sort key origin,
 *   may be NULL when order = 0).  time_varying selects the output layout (T+1 copies per
 *   obstacle, moved by velocity * t * dt when |velocity| > 0.01, or one copy at t = 0).
 * Out: obs_A, obs_b, obs_kind, obs_count exactly as rda_inputs expects them.              */
int rda_convert_obstacles(int B, int M, int N, int T, int E, float dt, int time_varying, int order,
                          const float *state, const int32_t *shape_kind, const int32_t *shape_nv,
                          const float *shape_xy, const float *shape_radius, const float *shape_vel,
                          const int32_t *shape_count, float *obs_A, float *obs_b, int32_t *obs_kind,
                          int32_t *obs_count, void *cuda_stream);

/* The same conversion when robots share obstacle WORLDS of any size, as MPC.control receives
 * everything the simulator knows: convert_rda_obstacle (mpc.py:189-218) over the robot's whole
 * world, stable-sorted by rda_obs_distance when order != 0, then assign_obstacle_parameter
 * (rda_solver.py:483-526) keeps the first N and pads by repeating the last.  Per robot the
 * result equals rda_convert_obstacles given that robot's world as its list, without the
 * RDA_MAX_SHAPES limit and without a private copy per robot.
 *   shape_kind, shape_nv, shape_xy, shape_radius, shape_vel: ONE flat list of S shapes, per-shape
 *   layout as rda_convert_obstacles ([S], [S], [S][RDA_MAX_EDGE][2], [S], [S][2]);
 *   world_start [W+1]: world w is shapes [world_start[w], world_start[w+1]);
 *   robot_world [B]: the world of each robot (NULL: all in world 0; outside [0, W): no obstacles);
 *   state [B][3]: sort key origin (may be NULL when order = 0).
 * N <= RDA_MAX_WORLD_SLOTS.  obs_count [B] receives the world size (len(obstacle_list)); a robot
 * whose world is empty gets all-zero slots.  Out: obs_A, obs_b, obs_kind, obs_count exactly as
 * rda_inputs expects them.                                                                 */
int rda_convert_world_obstacles(int B, int W, int N, int T, int E, float dt, int time_varying, int order,
                                const float *state, const int32_t *world_start, const int32_t *robot_world,
                                const int32_t *shape_kind, const int32_t *shape_nv, const float *shape_xy,
                                const float *shape_radius, const float *shape_vel, float *obs_A,
                                float *obs_b, int32_t *obs_kind, int32_t *obs_count, void *cuda_stream);

/* A FLEET that avoids itself: robots that share a world see each other as moving obstacles, as each reference MPC
 * receives the other agents from its simulator (the dynamic_obs example: obs(center, radius, vertex, cone_type,
 * velocity), predicted at constant velocity, mpc.py:440-474).
 * rda_fleet_shapes writes every robot as one raw shape (layout of rda_convert_world_obstacles, [B] entries): the
 * robot body (RDA_OBS_POLYGON: body_nv counter-clockwise vertices body_xy [body_nv][2] in the body frame, 3..8;
 * RDA_OBS_CIRCLE: centre body_xy[0..1], body_radius > 0) placed at the pose state [B][3] (p + R(theta) v), with the
 * world-frame velocity of the first control of cur_vel [B][2][T], the one rda_motion_predict moved the robot with:
 * v (cos theta, sin theta) for acker / diff, v (cos psi, sin psi) for omni (mpc.py:293-336).
 * rda_convert_fleet_obstacles is rda_convert_world_obstacles over a longer list per robot: every shape of its world
 * in world order, then every other robot of the same world in ascending robot index, whose shapes are entry m of
 * fleet_kind, fleet_nv, fleet_xy, fleet_radius, fleet_vel (rda_fleet_shapes' outputs).  The robots of world w are
 * fleet_robot [fleet_start[w], fleet_start[w+1]) (fleet_start [W+1], fleet_robot [B]), in ascending order, and must
 * be exactly the robots whose robot_world is w: a stable sort of robot_world and a search for 0..W give both.
 * Sort key, stable order, the first N, padding, rows and time_varying layout are those of rda_convert_world_obstacles;
 * obs_count [B] receives the world size plus the robots of the world minus one.  A robot whose robot_world is outside
 * [0, W) neither sees nor is seen.  rda_convert_world_obstacles is this call without the fleet.                */
int rda_fleet_shapes(int B, int T, int dynamics, int body_kind, int body_nv, const float *body_xy,
                     float body_radius, const float *state, const float *cur_vel, int32_t *shape_kind,
                     int32_t *shape_nv, float *shape_xy, float *shape_radius, float *shape_vel, void *cuda_stream);
/* rda_fleet_shapes for a fleet of several robot classes: dynamics int32 [B], body_xy float32 [B][RDA_MAX_EDGE][2]
 * (polygon: the body_nv vertices, disc: the centre in row 0) and body_radius float32 [B] per robot (device).  The kind
 * and vertex count stay one per fleet, as the handle's cone and R do.  dynamics values are the caller's to check. */
int rda_fleet_shapes_per_robot(int B, int T, const int32_t *dynamics, int body_kind, int body_nv, const float *body_xy,
                               const float *body_radius, const float *state, const float *cur_vel, int32_t *shape_kind,
                               int32_t *shape_nv, float *shape_xy, float *shape_radius, float *shape_vel,
                               void *cuda_stream);
int rda_convert_fleet_obstacles(int B, int W, int N, int T, int E, float dt, int time_varying, int order,
                                const float *state, const int32_t *world_start, const int32_t *robot_world,
                                const int32_t *shape_kind, const int32_t *shape_nv, const float *shape_xy,
                                const float *shape_radius, const float *shape_vel, const int32_t *fleet_start,
                                const int32_t *fleet_robot, const int32_t *fleet_kind, const int32_t *fleet_nv,
                                const float *fleet_xy, const float *fleet_radius, const float *fleet_vel,
                                float *obs_A, float *obs_b, int32_t *obs_kind, int32_t *obs_count,
                                void *cuda_stream);

/* A fleet that avoids each other's PLANS: every map-mate is a time-varying obstacle that follows the controls its last
 * solve kept (cur_vel [B][2][T]) instead of moving at the constant velocity of the first one.  In the reference's terms
 * each mate is an rdaobs whose A and b are lists of T+1 arrays (rda_solver.py:501-526), the rows of its body at its
 * predicted pose of each stage.
 * rda_fleet_plan_shapes writes what rda_fleet_shapes writes (bit for bit) and plan_xy [B][T+1][RDA_MAX_EDGE][2]
 * (16-byte aligned): robot m's body placed at q_m(t), with q_m(0) = state[m] and, for t = 0..T-1,
 * q_m(t+1) = motion_predict(q_m(t), cur_vel[m][:, c]), c = min(t + 1, T - 1), in double (column 0 is the control
 * rda_motion_predict has just applied, so the rest of the plan starts at column 1; the last column is held).  Stage 0 is
 * bit for bit the shape_xy of the same robot.  The dynamics, wheelbase and body are the scalars (checked as for
 * rda_fleet_shapes), or per robot when dynamics_b int32 [B], wheelbase_b float32 [B], body_xy_b float32
 * [B][RDA_MAX_EDGE][2] or body_radius_b float32 [B] are given (device; NULL: the scalar; values the caller's to check).
 * rda_convert_fleet_plan_obstacles is rda_convert_fleet_obstacles, the same list, keys (from the stage-0 shapes), order,
 * padding, obs_kind and obs_count, except that the stage-t copy of a mate's slot is the rows of its plan_xy[t] shape
 * standing still (fleet_plan_xy: rda_fleet_plan_shapes' plan_xy).  World shapes keep their constant-velocity rows.  The
 * prediction is a trajectory, so time_varying must be non-zero (RDA_E_ARG otherwise).  Neither call allocates, syncs
 * the host or breaks graph capture.                                                                              */
int rda_fleet_plan_shapes(int B, int T, int dynamics, float dt, float wheelbase, int body_kind, int body_nv,
                          const float *body_xy, float body_radius, const int32_t *dynamics_b, const float *wheelbase_b,
                          const float *body_xy_b, const float *body_radius_b, const float *state, const float *cur_vel,
                          int32_t *shape_kind, int32_t *shape_nv, float *shape_xy, float *shape_radius,
                          float *shape_vel, float *plan_xy, void *cuda_stream);
int rda_convert_fleet_plan_obstacles(int B, int W, int N, int T, int E, float dt, int time_varying, int order,
                                     const float *state, const int32_t *world_start, const int32_t *robot_world,
                                     const int32_t *shape_kind, const int32_t *shape_nv, const float *shape_xy,
                                     const float *shape_radius, const float *shape_vel, const int32_t *fleet_start,
                                     const int32_t *fleet_robot, const int32_t *fleet_kind, const int32_t *fleet_nv,
                                     const float *fleet_xy, const float *fleet_radius, const float *fleet_vel,
                                     const float *fleet_plan_xy, float *obs_A, float *obs_b, int32_t *obs_kind,
                                     int32_t *obs_count, void *cuda_stream);

/* HORIZON ORDER: rda_convert_world_obstacles / rda_convert_fleet_obstacles / rda_convert_fleet_plan_obstacles with each
 * robot's shapes chosen by how close its horizon comes to them instead of the reference's sort key (DESIGN.md §7.3).
 * The list is the same (the world's shapes, then, with a fleet, the map-mates in ascending index); shape j's key is
 *   min over the finite pose columns q of nom_s[b][:, t] and ref_s[b][:, t], t = 0..T, of sd(body at q, shape j at t)
 * where sd is rda_plan_clearance's signed distance and "shape j at t" the rows written for it (copy t when
 * time_varying, copy 0 otherwise).  A column with a non-finite entry takes no part; without any, every key is +inf and
 * the order is list order.  Stable ascending order, the first N, padding, obs_kind, obs_count and the rows are those of
 * the calls above, and so are their arguments, except:
 *   nom_s, ref_s [B][3][T+1]: the solver's nominal and reference poses (rda_pre_process_paths' outputs);
 *   the robot body in the format of rda_fleet_shapes (body_kind RDA_OBS_POLYGON: body_nv counter-clockwise vertices
 *   body_xy [body_nv][2], 3..8; RDA_OBS_CIRCLE: centre body_xy[0..1], body_radius > 0), or per robot body_xy_b
 *   [B][RDA_MAX_EDGE][2] / body_radius_b [B] (device; NULL: the one body; values the caller's to check);
 *   fleet_start NULL: no fleet, and the other fleet pointers are not read; fleet_plan_xy NULL: mates at constant
 *   velocity, else along their plans (needs a fleet and time_varying).
 * Usage errors are return codes: RDA_E_ARG for a NULL pointer or a bad body, RDA_E_UNSUPPORTED for N above
 * RDA_MAX_WORLD_SLOTS, E outside 3..8 or a polygon body outside 3..8 vertices.  No allocation, host sync or graph break. */
int rda_convert_world_obstacles_horizon(int B, int W, int N, int T, int E, float dt, int time_varying,
                                        const float *nom_s, const float *ref_s, int body_kind, int body_nv,
                                        const float *body_xy, float body_radius, const float *body_xy_b,
                                        const float *body_radius_b, const int32_t *world_start,
                                        const int32_t *robot_world, const int32_t *shape_kind, const int32_t *shape_nv,
                                        const float *shape_xy, const float *shape_radius, const float *shape_vel,
                                        const int32_t *fleet_start, const int32_t *fleet_robot,
                                        const int32_t *fleet_kind, const int32_t *fleet_nv, const float *fleet_xy,
                                        const float *fleet_radius, const float *fleet_vel, const float *fleet_plan_xy,
                                        float *obs_A, float *obs_b, int32_t *obs_kind, int32_t *obs_count,
                                        void *cuda_stream);

/* The conversions above that also say which obstacle went where, for rda_set_obstacle_ids: obs_A, obs_b, obs_kind and
 * obs_count are those of the existing call, bit for bit, and obs_id [B][N] (device) receives each slot's obstacle id:
 *   rda_convert_obstacles_ids: the position j of the shape in the robot's list (shape_kind[b][j] ...);
 *   rda_convert_world_obstacles_ids: the arguments of rda_convert_fleet_plan_obstacles, where fleet_start = NULL means a
 *     world only (the other fleet pointers are then not read) and fleet_plan_xy = NULL mates at constant velocity; the id
 *     is the flat shape index s for a world shape and world_start[W] + m for map-mate robot m;
 *   rda_convert_world_obstacles_horizon_ids: rda_convert_world_obstacles_horizon, with the same ids.
 * A robot with an empty list gets -1 in every slot.  Identity is list position: a caller who repacks a map must keep its
 * order for the warm start to follow.  Usage errors as the existing calls, and RDA_E_ARG for obs_id = NULL. */
int rda_convert_obstacles_ids(int B, int M, int N, int T, int E, float dt, int time_varying, int order,
                              const float *state, const int32_t *shape_kind, const int32_t *shape_nv,
                              const float *shape_xy, const float *shape_radius, const float *shape_vel,
                              const int32_t *shape_count, float *obs_A, float *obs_b, int32_t *obs_kind,
                              int32_t *obs_count, int32_t *obs_id, void *cuda_stream);
int rda_convert_world_obstacles_ids(int B, int W, int N, int T, int E, float dt, int time_varying, int order,
                                    const float *state, const int32_t *world_start, const int32_t *robot_world,
                                    const int32_t *shape_kind, const int32_t *shape_nv, const float *shape_xy,
                                    const float *shape_radius, const float *shape_vel, const int32_t *fleet_start,
                                    const int32_t *fleet_robot, const int32_t *fleet_kind, const int32_t *fleet_nv,
                                    const float *fleet_xy, const float *fleet_radius, const float *fleet_vel,
                                    const float *fleet_plan_xy, float *obs_A, float *obs_b, int32_t *obs_kind,
                                    int32_t *obs_count, int32_t *obs_id, void *cuda_stream);
int rda_convert_world_obstacles_horizon_ids(int B, int W, int N, int T, int E, float dt, int time_varying,
                                            const float *nom_s, const float *ref_s, int body_kind, int body_nv,
                                            const float *body_xy, float body_radius, const float *body_xy_b,
                                            const float *body_radius_b, const int32_t *world_start,
                                            const int32_t *robot_world, const int32_t *shape_kind,
                                            const int32_t *shape_nv, const float *shape_xy, const float *shape_radius,
                                            const float *shape_vel, const int32_t *fleet_start,
                                            const int32_t *fleet_robot, const int32_t *fleet_kind,
                                            const int32_t *fleet_nv, const float *fleet_xy, const float *fleet_radius,
                                            const float *fleet_vel, const float *fleet_plan_xy, float *obs_A,
                                            float *obs_b, int32_t *obs_kind, int32_t *obs_count, int32_t *obs_id,
                                            void *cuda_stream);

/* WORLD SHAPES ALONG TRAJECTORIES: a world shape may follow a given trajectory over the horizon (a predictor's output
 * for a pedestrian, a vehicle, a forklift) instead of standing still or translating at its constant velocity.  In the
 * reference's terms such a shape is rdaobs(A = [A_0 .. A_T], b = [b_0 .. b_T]) of its stage shapes (MPC(rda_obstacle=
 * True), rda_solver.py:501-526).  The two calls take the arguments of rda_convert_world_obstacles_ids /
 * rda_convert_world_obstacles_horizon_ids (fleet_start = NULL: no fleet; fleet_plan_xy = NULL: mates at constant
 * velocity; obs_id = NULL: no ids) plus the trajectory table (device):
 *   shape_traj int32 [S]: the trajectory of each packed shape; a value outside [0, K) means none (the shape's own
 *   shape_xy and shape_vel, exactly as the calls above; decided on the device);
 *   traj_xy float32 [K][T+1][RDA_MAX_EDGE][2], 16-byte aligned: trajectory k's shape at stage t in the world frame,
 *   a polygon's shape_nv vertices (either orientation, as shape_xy) or a disc's centre in row 0 (the radius stays
 *   shape_radius).
 * For a shape with trajectory k, traj_xy[k] replaces its shape_xy and shape_vel everywhere: its stage-t rows are
 * obstacle rows of traj_xy[k][t] standing still (no velocity threshold), its reference key (order != 0) is taken from
 * traj_xy[k][0], and its horizon key uses its stage-t rows.  It gets no one-disc bound in the horizon order, only the
 * bound of every pose.  Slots, padding, obs_kind, obs_count and ids (the flat shape index) keep their meaning.  Both
 * arrays may be rewritten on the device between calls; a captured graph reads the new values on replay.
 * Usage errors are return codes: RDA_E_ARG for NULL shape_traj or traj_xy, an unaligned traj_xy, K < 1 or
 * time_varying == 0 (a trajectory has T+1 copies); the rest as in the calls they extend.  No allocation, host sync or
 * graph break. */
int rda_convert_world_obstacles_traj(int B, int W, int N, int T, int E, float dt, int time_varying, int order,
                                     const float *state, const int32_t *world_start, const int32_t *robot_world,
                                     const int32_t *shape_kind, const int32_t *shape_nv, const float *shape_xy,
                                     const float *shape_radius, const float *shape_vel, const int32_t *fleet_start,
                                     const int32_t *fleet_robot, const int32_t *fleet_kind, const int32_t *fleet_nv,
                                     const float *fleet_xy, const float *fleet_radius, const float *fleet_vel,
                                     const float *fleet_plan_xy, float *obs_A, float *obs_b, int32_t *obs_kind,
                                     int32_t *obs_count, int32_t *obs_id, const int32_t *shape_traj, int K,
                                     const float *traj_xy, void *cuda_stream);
int rda_convert_world_obstacles_horizon_traj(int B, int W, int N, int T, int E, float dt, int time_varying,
                                             const float *nom_s, const float *ref_s, int body_kind, int body_nv,
                                             const float *body_xy, float body_radius, const float *body_xy_b,
                                             const float *body_radius_b, const int32_t *world_start,
                                             const int32_t *robot_world, const int32_t *shape_kind,
                                             const int32_t *shape_nv, const float *shape_xy, const float *shape_radius,
                                             const float *shape_vel, const int32_t *fleet_start,
                                             const int32_t *fleet_robot, const int32_t *fleet_kind,
                                             const int32_t *fleet_nv, const float *fleet_xy, const float *fleet_radius,
                                             const float *fleet_vel, const float *fleet_plan_xy, float *obs_A,
                                             float *obs_b, int32_t *obs_kind, int32_t *obs_count, int32_t *obs_id,
                                             const int32_t *shape_traj, int K, const float *traj_xy,
                                             void *cuda_stream);

/* Arrive rule of MPC.control (mpc.py:170-185, single gear): instances whose near_index >=
 * P - goal_index_threshold get u_opt = 0 and arrive = 1; cur_vel (may be NULL) receives the
 * controls kept as the next step's nominal (mpc.py:186).  u_opt, cur_vel [B][2][T].        */
int rda_post_process(int B, int T, int P, int goal_index_threshold, const int32_t *near_index,
                     float *u_opt, float *cur_vel, int32_t *arrive, void *cuda_stream);

/* Gear changes (enable_reverse, mpc.py:139-144, :166-183, split_path :232-249).  The reference path is cut into
 * n_curves single-gear curves, curve c = waypoints [curve_start[c], curve_start[c+1]) of `path`; every robot follows
 * curve curve_index[b].  rda_pre_process_curves is rda_pre_process on the robot's current curve (near_index is
 * relative to the curve).  rda_post_process_gear applies mpc.py:166-185: at the end of a curve the robot switches
 * to the next one (cur_index back to 0, controls kept); past the last curve the controls are zeroed and arrive is
 * set (curve_index then stays on the last curve: the reference would raise IndexError on the next call).
 * gear [B] (output) is the gear flag (+1 / -1) of the robot's curve BEFORE the update; the caller multiplies the
 * solver's reference speed with it (mpc.py:161). */
int rda_pre_process_curves(int B, int T, int dynamics, float dt, float wheelbase, const float *state,
                           const float *cur_vel, const float *ref_speed, const float *path, int n_curves,
                           const int32_t *curve_start, const int32_t *curve_index, const int32_t *start_index,
                           float threshold, int ind_range, float *nom_s, float *ref_s, int32_t *near_index,
                           void *cuda_stream);
int rda_post_process_gear(int B, int T, int n_curves, const int32_t *curve_start, int goal_index_threshold,
                          int32_t *near_index, int32_t *curve_index, float *u_opt, float *cur_vel,
                          int32_t *arrive, void *cuda_stream);

/* A FLEET on its own reference paths: each robot follows its own path, picked from a shared set of W paths, as
 * a batch of reference MPC objects each owning its ref_path (mpc.py:67-125, update_ref_path :220-227).  The
 * rda_pre_process / rda_pre_process_curves / rda_post_process / rda_post_process_gear calls above are the W = 1
 * case of these two.
 *   path [P][3]: the waypoints of all paths, one flat list; every path is cut into single-gear curves
 *   (split_path, mpc.py:232-249; without enable_reverse a path is one curve of gear +1):
 *   path_curve [W+1]: path w is curves [path_curve[w], path_curve[w+1]);
 *   curve_start [C+1]: curve c is waypoints [curve_start[c], curve_start[c+1]) of `path`;
 *   curve_gear [C]: +1 forward, -1 reverse;
 *   robot_path [B]: the path of each robot (NULL: all on path 0);
 *   curve_index [B]: the robot's curve, relative to its path (NULL: 0; out of range: clamped into the path);
 *   start_index / near_index [B]: MPC.cur_index, relative to the robot's curve (start_index NULL: 0).
 * rda_pre_process_paths is rda_pre_process on each robot's curve; solver_speed [B] (may be NULL) receives the
 * solver's reference speed gear * ref_speed (mpc.py:161).  rda_post_process_paths applies mpc.py:166-185: at the
 * end of a curve that is not its path's last, the robot moves to the next curve (near_index 0, controls kept);
 * past its path's last curve the controls are zeroed and arrive is set, and curve_index stays on that last curve.
 * cur_vel (may be NULL) receives the controls kept; arrive may be NULL.
 * A robot whose robot_path is outside [0, W), or whose path has no curve, has NO PATH (decided on the device, so
 * that the host never reads robot_path): nom_s is its rollout as usual, every column of ref_s is its current state,
 * near_index is 0 and its gear +1; rda_post_process_paths then zeroes its controls and sets arrive.           */
int rda_pre_process_paths(int B, int T, int dynamics, float dt, float wheelbase, const float *state,
                          const float *cur_vel, const float *ref_speed, const float *path, int W,
                          const int32_t *path_curve, const int32_t *curve_start, const int32_t *curve_gear,
                          const int32_t *robot_path, const int32_t *curve_index, const int32_t *start_index,
                          float threshold, int ind_range, float *nom_s, float *ref_s, int32_t *near_index,
                          float *solver_speed, void *cuda_stream);
/* rda_pre_process_paths with each robot's own dynamics (int32 [B], RDA_DYN_*) and wheelbase (float32 [B]), device
 * arrays (robot classes); the scalar entry point is this one with uniform arrays. */
int rda_pre_process_paths_per_robot(int B, int T, const int32_t *dynamics, float dt, const float *wheelbase,
                                    const float *state, const float *cur_vel, const float *ref_speed, const float *path,
                                    int W, const int32_t *path_curve, const int32_t *curve_start,
                                    const int32_t *curve_gear, const int32_t *robot_path, const int32_t *curve_index,
                                    const int32_t *start_index, float threshold, int ind_range, float *nom_s,
                                    float *ref_s, int32_t *near_index, float *solver_speed, void *cuda_stream);
int rda_post_process_paths(int B, int T, int W, const int32_t *path_curve, const int32_t *curve_start,
                           const int32_t *robot_path, int goal_index_threshold, int32_t *near_index,
                           int32_t *curve_index, float *u_opt, float *cur_vel, int32_t *arrive,
                           void *cuda_stream);

/* state [B][3] advanced in place by one step of the nonlinear model with the first control of
 * u_opt [B][2][T] (mpc.py:293-336; what the examples' simulator does between control calls). */
int rda_motion_predict(int B, int T, int dynamics, float dt, float wheelbase, const float *u_opt,
                       float *state, void *cuda_stream);
/* rda_motion_predict with each robot's own dynamics (int32 [B]) and wheelbase (float32 [B]), device arrays. */
int rda_motion_predict_per_robot(int B, int T, const int32_t *dynamics, float dt, const float *wheelbase,
                                 const float *u_opt, float *state, void *cuda_stream);

#ifdef __cplusplus
}
#endif
#endif
