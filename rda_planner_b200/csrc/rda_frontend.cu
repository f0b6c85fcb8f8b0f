// rda_frontend.cu — batched kernels for the steps either side of the solver (SURVEY.md §8 rows f1-f3):
// reference pre-processing, obstacle conversion, the arrive rule and the state advance of the closed
// loop.  Stateless C ABI (include/rda_b200.h, "front end" section); the per-instance arithmetic lives in
// frontend.cuh, shared with the CPU tests.  These passes are tiny next to the solve (one thread or one
// small CTA per instance, a few hundred bytes each); they exist so that a closed-loop step never leaves
// the device.
#include <cuda_runtime.h>
#include "../../include/rda_b200.h"
#include "rda_hd.h"
#include "frontend.cuh"
#include "horizon_key.cuh"

using namespace rda;

#define RDA_CUDA(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return (int)e_; } while (0)

namespace {

// MPC.pre_process on the single-gear curve each robot follows (mpc.py:139-144, :251-291), and the solver's reference
// speed gear * ref_speed (mpc.py:161).  A robot whose path index is outside [0, W) has no path: its nominal rollout as
// usual, a reference that holds its current state, near_index 0 and gear +1.  dyn_b / L_b [B]: each robot's own dynamics
// and wheelbase (robot classes), or NULL: the scalars for every robot.
__global__ void k_pre_process_paths(int B, int T, int dynamics, float dt, float L, const int* dyn_b, const float* L_b,
                                    const float* state,
                                    const float* cur_vel, const float* ref_speed, const float* path, int P, int W,
                                    int n_curves, const int* path_curve, const int* curve_start, const int* curve_gear,
                                    const int* robot_path, const int* curve_index, const int* start_index,
                                    float threshold, int ind_range, float* nom_s, float* ref_s, int* near_index,
                                    float* solver_speed) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int w = robot_path ? robot_path[b] : 0;
  if (dyn_b) dynamics = dyn_b[b];
  if (L_b) L = L_b[b];
  const float* st = state + 3 * (size_t)b;
  const float* vel = cur_vel + (size_t)b * 2 * T;
  float* nom = nom_s + (size_t)b * 3 * (T + 1);
  float* ref = ref_s + (size_t)b * 3 * (T + 1);
  PathCurve cv;
  int near = 0, gear = 1;
  if (w >= 0 && w < W &&
      resolve_curve(w, curve_index ? curve_index[b] : 0, path_curve, n_curves, curve_start, P, curve_gear, &cv)) {
    near = pre_process_one(dynamics, T, (double)dt, (double)L, st, vel, (double)ref_speed[b], path + 3 * (size_t)cv.first,
                           cv.len, start_index ? start_index[b] : 0, (double)threshold, ind_range, nom, ref);
    gear = cv.gear;
  } else {
    hold_state_one(dynamics, T, (double)dt, (double)L, st, vel, nom, ref);
  }
  near_index[b] = near;
  if (solver_speed) solver_speed[b] = ref_speed[b] * (float)gear;
}

// one CTA per instance: keys -> stable ranks -> rows of the N slots.  kIds: also the list position of each slot's
// shape into obs_id [B][N] (-1 for an empty list).
template <bool kIds>
__device__ __forceinline__ void convert_obstacles(int B, int M, int N, int T, int E, float dt, int time_varying, int order,
                                                  const float* state, const int* shape_kind, const int* shape_nv,
                                                  const float* shape_xy, const float* shape_radius, const float* shape_vel,
                                                  const int* shape_count, float* obs_A, float* obs_b, int* obs_kind,
                                                  int* obs_count, int* obs_id) {
  __shared__ double keys[RDA_MAX_SHAPES];
  __shared__ int sorted[RDA_MAX_SHAPES];
  const int b = blockIdx.x;
  if (b >= B) return;
  const int j = threadIdx.x;
  int count = shape_count[b];
  if (count > M) count = M;
  if (count < 0) count = 0;
  const size_t sb = (size_t)b * M;
  if (j < count) keys[j] = order ? obstacle_key(shape_kind[sb + j], shape_nv[sb + j], shape_xy + (sb + j) * RDA_MAX_EDGE * 2,
                                               (double)state[3 * b], (double)state[3 * b + 1])
                                 : (double)j;
  __syncthreads();
  if (j < count) {
    int before = 0;
    for (int i = 0; i < count; ++i)
      if (keys[i] < keys[j] || (keys[i] == keys[j] && i < j)) ++before;
    sorted[before] = j;
  }
  __syncthreads();
  if (j == 0) obs_count[b] = count;
  const int Tc = time_varying ? T + 1 : 1;
  for (int n = j; n < N; n += blockDim.x) {
    float* A = obs_A + ((size_t)b * N + n) * Tc * E * 2;
    float* bb = obs_b + ((size_t)b * N + n) * Tc * E;
    if (count == 0) {
      for (int i = 0; i < Tc * E; ++i) { A[2 * i] = 0.f; A[2 * i + 1] = 0.f; bb[i] = 0.f; }
      obs_kind[(size_t)b * N + n] = RDA_OBS_POLYGON;
      if (kIds) obs_id[(size_t)b * N + n] = -1;
      continue;
    }
    const int src = sorted[n < count ? n : count - 1];
    if (kIds) obs_id[(size_t)b * N + n] = src;
    const int kind = shape_kind[sb + src], nv = shape_nv[sb + src];
    const float* xy = shape_xy + (sb + src) * RDA_MAX_EDGE * 2;
    const double rad = shape_radius[sb + src];
    const double vx = shape_vel[(sb + src) * 2], vy = shape_vel[(sb + src) * 2 + 1];
    obs_kind[(size_t)b * N + n] = kind;
    for (int t = 0; t < Tc; ++t) obstacle_rows(kind, nv, xy, rad, vx, vy, t, (double)dt, E, A + (size_t)t * E * 2, bb + (size_t)t * E);
  }
}

__global__ void __launch_bounds__(RDA_MAX_SHAPES)
k_convert_obstacles(int B, int M, int N, int T, int E, float dt, int time_varying, int order, const float* state,
                    const int* shape_kind, const int* shape_nv, const float* shape_xy, const float* shape_radius,
                    const float* shape_vel, const int* shape_count, float* obs_A, float* obs_b, int* obs_kind,
                    int* obs_count) {
  convert_obstacles<false>(B, M, N, T, E, dt, time_varying, order, state, shape_kind, shape_nv, shape_xy, shape_radius,
                           shape_vel, shape_count, obs_A, obs_b, obs_kind, obs_count, nullptr);
}

__global__ void __launch_bounds__(RDA_MAX_SHAPES)
k_convert_obstacles_ids(int B, int M, int N, int T, int E, float dt, int time_varying, int order, const float* state,
                        const int* shape_kind, const int* shape_nv, const float* shape_xy, const float* shape_radius,
                        const float* shape_vel, const int* shape_count, float* obs_A, float* obs_b, int* obs_kind,
                        int* obs_count, int* obs_id) {
  convert_obstacles<true>(B, M, N, T, E, dt, time_varying, order, state, shape_kind, shape_nv, shape_xy, shape_radius,
                          shape_vel, shape_count, obs_A, obs_b, obs_kind, obs_count, obs_id);
}

// Shared worlds: one CTA per robot scans its world in tiles of kWorldTile shapes, one key per thread, and keeps the
// N first (key, index) pairs of the stable order sorted in shared memory.  Only shapes that beat the current N-th
// pair are compacted; they are ranked among themselves and merged with the kept list by binary search (every
// element's new position is its rank in its own list plus its rank in the other).  A tile's indices all exceed the
// kept ones, so once N are kept a shape beats the N-th only with a strictly smaller key: after the first tiles a
// shape costs its key and nothing else.  The world is read by every robot in it and stays in L2.
constexpr int kWorldTile = 256;

__device__ __forceinline__ int world_rank(const double* key, const int* idx, int n, double k, int i) {
  int lo = 0, hi = n;                                  // number of pairs in the sorted list before (k, i)
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (obstacle_before(key[mid], idx[mid], k, i)) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// The raw shapes a robot chooses from: its world's shapes [first, first + n_world), then, with a fleet, its map-mates:
// the robots of fleet_robot [mate0, mate0 + mates + 1) other than the robot itself, whose shapes are entry m of the
// fleet arrays.  Each world's robots are listed in ascending order, so skipping the robot is one comparison.
struct ShapeList {
  int first, n_world, mate0, mates;
};

__device__ __forceinline__ size_t list_entry(const ShapeList& L, int i, const int* fleet_robot, int b, int B,
                                             bool* mate) {
  *mate = i >= L.n_world;
  if (!*mate) return (size_t)L.first + i;
  const int p = L.mate0 + (i - L.n_world);
  int m = fleet_robot[p];
  if (m >= b) m = fleet_robot[p + 1];
  return (size_t)(m < 0 ? 0 : (m >= B ? B - 1 : m));   // a malformed list never reads outside the fleet
}

// The candidates of a tile, c (ckey, cidx) pairs in any order, ranked among themselves into (skey, sidx) and merged with
// the nk kept pairs of buffer cur into buffer cur ^ 1, the first N kept.  Every element's new position is its rank in
// its own list plus its rank in the other.  Ends with a barrier of the CTA.
__device__ __forceinline__ void world_merge(int tid, int c, int N, double* kkey, int* kidx, const double* ckey,
                                            const int* cidx, double* skey, int* sidx, int& nk, int& cur) {
  if (tid < c) {                                       // rank among the candidates: sorted copy
    const double k = ckey[tid];
    const int ix = cidx[tid];
    int r = 0;
    for (int j = 0; j < c; ++j) r += obstacle_before(ckey[j], cidx[j], k, ix);
    skey[r] = k; sidx[r] = ix;
  }
  __syncthreads();
  const int nxt = cur ^ 1;
  const double* ok = kkey + cur * N;
  const int* oi = kidx + cur * N;
  if (tid < c) {
    const int p = tid + world_rank(ok, oi, nk, skey[tid], sidx[tid]);
    if (p < N) { kkey[nxt * N + p] = skey[tid]; kidx[nxt * N + p] = sidx[tid]; }
  }
  for (int j = tid; j < nk; j += kWorldTile) {
    const int p = j + world_rank(skey, sidx, c, ok[j], oi[j]);
    if (p < N) { kkey[nxt * N + p] = ok[j]; kidx[nxt * N + p] = oi[j]; }
  }
  nk = nk + c < N ? nk + c : N;
  cur = nxt;
  __syncthreads();
}

// The trajectory of world shape s: its stages traj_xy [k][0..T] ([T+1][RDA_MAX_EDGE][2] each) when k = shape_traj[s]
// is in [0, K), else NULL (the shape's own xy and vel).
__device__ __forceinline__ const float* world_traj(const int* shape_traj, int K, const float* traj_xy, int T1, size_t s) {
  const int k = shape_traj[s];
  return k >= 0 && k < K ? traj_xy + (size_t)k * T1 * RDA_MAX_EDGE * 2 : nullptr;
}

// The current shape of world shape s: stage 0 of its trajectory, else its own xy.
__device__ __forceinline__ const float* world_xy0(const int* shape_traj, int K, const float* traj_xy, int T1,
                                                  const float* shape_xy, size_t s) {
  const float* tr = world_traj(shape_traj, K, traj_xy, T1, s);
  return tr ? tr : shape_xy + s * RDA_MAX_EDGE * 2;
}

// The rows of the N slots of robot b: slot n is the list entry kept_idx[n] (list order when kept_idx is NULL), the
// last one repeated past the list, all-zero rows for an empty list.  kPlan: map-mates are read along fleet_plan_xy.
// kTraj: world shapes with a trajectory (world_traj) are read along it (time-varying output only).
template <bool kPlan, bool kTraj>
__device__ __forceinline__ void world_slots(int tid, int b, int B, int N, int T, int E, float dt, int time_varying,
                                            int count, const ShapeList& L, const int* kept_idx, const int* shape_kind,
                                            const int* shape_nv, const float* shape_xy, const float* shape_radius,
                                            const float* shape_vel, const int* fleet_robot, const int* fleet_kind,
                                            const int* fleet_nv, const float* fleet_xy, const float* fleet_radius,
                                            const float* fleet_vel, const float* fleet_plan_xy, float* obs_A,
                                            float* obs_b, int* obs_kind, const int* shape_traj, int K,
                                            const float* traj_xy) {
  const int Tc = time_varying ? T + 1 : 1;
  for (int q = tid; q < N * Tc; q += kWorldTile) {     // one (slot, stage) copy per thread
    const int n = q / Tc, t = q - n * Tc;
    float* A = obs_A + (((size_t)b * N + n) * Tc + t) * E * 2;
    float* bb = obs_b + (((size_t)b * N + n) * Tc + t) * E;
    if (count == 0) {
      for (int r = 0; r < E; ++r) { A[2 * r] = 0.f; A[2 * r + 1] = 0.f; bb[r] = 0.f; }
      if (t == 0) obs_kind[(size_t)b * N + n] = RDA_OBS_POLYGON;
      continue;
    }
    const int slot = n < count ? n : count - 1;        // pad by repeating the last
    int src = kept_idx ? kept_idx[slot] : slot;
    if (src < 0 || src >= count) src = count - 1;      // NaN keys have no order; never read outside the list
    bool mate;
    const size_t s = list_entry(L, src, fleet_robot, b, B, &mate);
    const int kind = (mate ? fleet_kind : shape_kind)[s];
    if (t == 0) obs_kind[(size_t)b * N + n] = kind;
    const float* xy = (mate ? fleet_xy : shape_xy) + s * RDA_MAX_EDGE * 2;
    double vx = 0.0, vy = 0.0;
    const float* tr = kTraj && !mate ? world_traj(shape_traj, K, traj_xy, T + 1, s) : nullptr;
    if (kPlan && mate) {                               // a map-mate along its plan: its stage-t shape, standing
      xy = fleet_plan_xy + (s * (T + 1) + t) * RDA_MAX_EDGE * 2;
    } else if (kTraj && tr) {                          // a world shape along its trajectory: likewise
      xy = tr + (size_t)t * RDA_MAX_EDGE * 2;
    } else {
      const float* vel = (mate ? fleet_vel : shape_vel) + 2 * s;
      vx = vel[0]; vy = vel[1];
    }
    obstacle_rows(kind, (mate ? fleet_nv : shape_nv)[s], xy, (mate ? fleet_radius : shape_radius)[s], vx, vy, t,
                  (double)dt, E, A, bb);
  }
}

// The obstacle id of each of the N slots world_slots writes for robot b, into obs_id [B][N]: the flat shape index of a
// world shape, mate_base + m for map-mate robot m, -1 for an empty list.
__device__ __forceinline__ void world_slot_ids(int tid, int b, int B, int N, int count, const ShapeList& L,
                                               const int* kept_idx, const int* fleet_robot, int mate_base, int* obs_id) {
  for (int n = tid; n < N; n += kWorldTile) {
    int id = -1;
    if (count > 0) {
      int src = kept_idx ? kept_idx[n < count ? n : count - 1] : (n < count ? n : count - 1);
      if (src < 0 || src >= count) src = count - 1;
      bool mate;
      const size_t s = list_entry(L, src, fleet_robot, b, B, &mate);
      id = mate ? mate_base + (int)s : (int)s;
    }
    obs_id[(size_t)b * N + n] = id;
  }
}

// kPlan: map-mates are read along their plans, fleet_plan_xy [B][T+1][RDA_MAX_EDGE][2] (time-varying output only);
// the variant without plans never reads it, and compiles to the code it had before plans existed.
// kIds: also the slots' obstacle ids (world_slots) into obs_id.
// kTraj: world shapes with a trajectory are keyed by its stage 0 and written along it (world_traj; time-varying output
// only); the variant without never reads shape_traj / traj_xy, and compiles to the code it had before trajectories.
template <bool kPlan, bool kIds, bool kTraj>
__device__ __forceinline__ void convert_world(int B, int W, int N, int T, int E, float dt, int time_varying, int order,
                                              const float* state, const int* world_start, const int* robot_world,
                                              const int* shape_kind, const int* shape_nv, const float* shape_xy,
                                              const float* shape_radius, const float* shape_vel, const int* fleet_start,
                                              const int* fleet_robot, const int* fleet_kind, const int* fleet_nv,
                                              const float* fleet_xy, const float* fleet_radius, const float* fleet_vel,
                                              const float* fleet_plan_xy, float* obs_A, float* obs_b, int* obs_kind,
                                              int* obs_count, int* obs_id, const int* shape_traj, int K,
                                              const float* traj_xy) {
  // dynamic shared memory (order != 0): kept keys [2][N], candidate keys [2][tile], kept indices [2][N],
  // candidate indices [2][tile]; the kept list is double-buffered, candidates are gathered then sorted
  extern __shared__ double sh[];
  __shared__ int n_cand[3];                            // candidate counter of tile k is n_cand[k % 3]
  const int b = blockIdx.x;
  if (b >= B) return;
  const int tid = threadIdx.x;
  const int w = robot_world ? robot_world[b] : 0;
  ShapeList L = {0, 0, 0, 0};
  if (w >= 0 && w < W) {
    L.first = world_start[w];
    L.n_world = world_start[w + 1] - L.first;
    if (L.n_world < 0) L.n_world = 0;
    if (fleet_start) {                                 // NULL: no fleet, the world's shapes only
      L.mate0 = fleet_start[w];
      L.mates = fleet_start[w + 1] - L.mate0 - 1;
      if (L.mates < 0) L.mates = 0;
    }
  }
  const int count = L.n_world + L.mates;               // positions in the list: world shapes, then map-mates
  int cur = 0;
  int* kept_idx = nullptr;
  if (order && count > 0) {
    double* kkey = sh;                                 // [2][N]
    double* ckey = kkey + 2 * N;                       // gathered [tile], sorted [tile]
    double* skey = ckey + kWorldTile;
    int* kidx = (int*)(skey + kWorldTile);             // [2][N]
    int* cidx = kidx + 2 * N;
    int* sidx = cidx + kWorldTile;
    const double sx = state[3 * b], sy = state[3 * b + 1];
    if (tid == 0) n_cand[0] = 0;
    __syncthreads();
    int nk = 0;                                        // pairs kept so far (uniform across the CTA)
    for (int base = 0, tile = 0; base < count; base += kWorldTile, tile = tile == 2 ? 0 : tile + 1) {
      const int i = base + tid;
      if (i < count) {
        bool mate;
        const size_t s = list_entry(L, i, fleet_robot, b, B, &mate);
        const double key = obstacle_key((mate ? fleet_kind : shape_kind)[s], (mate ? fleet_nv : shape_nv)[s],
                                        kTraj && !mate ? world_xy0(shape_traj, K, traj_xy, T + 1, shape_xy, s)
                                                       : (mate ? fleet_xy : shape_xy) + s * RDA_MAX_EDGE * 2,
                                        sx, sy);
        if (nk < N || key < kkey[cur * N + N - 1]) {
          const int p = atomicAdd(&n_cand[tile], 1);
          ckey[p] = key; cidx[p] = i;
        }
      }
      // the next tile's counter was last read two tiles ago, before the previous barrier, and is next
      // incremented after the barrier below
      if (tid == 0) n_cand[tile == 2 ? 0 : tile + 1] = 0;
      __syncthreads();
      const int c = n_cand[tile];
      if (c == 0) continue;
      world_merge(tid, c, N, kkey, kidx, ckey, cidx, skey, sidx, nk, cur);
    }
    kept_idx = kidx + cur * N;
  }
  if (tid == 0) obs_count[b] = count;
  world_slots<kPlan, kTraj>(tid, b, B, N, T, E, dt, time_varying, count, L, kept_idx, shape_kind, shape_nv, shape_xy,
                            shape_radius, shape_vel, fleet_robot, fleet_kind, fleet_nv, fleet_xy, fleet_radius,
                            fleet_vel, fleet_plan_xy, obs_A, obs_b, obs_kind, shape_traj, K, traj_xy);
  if (kIds) world_slot_ids(tid, b, B, N, count, L, kept_idx, fleet_robot, world_start[W], obs_id);
}

// The parameter lists of the world kernels and the arguments that forward them.  The launchers
// (launch_world_obstacles, launch_world_obstacles_horizon) name their parameters alike and forward them with the same
// macros; all four are undefined after the launchers.
#define RDA_WORLD_PARAMS                                                                                               \
  int B, int W, int N, int T, int E, float dt, int time_varying, int order, const float *state, const int *world_start, \
      const int *robot_world, const int *shape_kind, const int *shape_nv, const float *shape_xy,                       \
      const float *shape_radius, const float *shape_vel, const int *fleet_start, const int *fleet_robot,                 \
      const int *fleet_kind, const int *fleet_nv, const float *fleet_xy, const float *fleet_radius,                      \
      const float *fleet_vel, const float *fleet_plan_xy, float *obs_A, float *obs_b, int *obs_kind, int *obs_count
#define RDA_WORLD_ARGS                                                                                                 \
  B, W, N, T, E, dt, time_varying, order, state, world_start, robot_world, shape_kind, shape_nv, shape_xy, shape_radius, \
      shape_vel, fleet_start, fleet_robot, fleet_kind, fleet_nv, fleet_xy, fleet_radius, fleet_vel, fleet_plan_xy,      \
      obs_A, obs_b, obs_kind, obs_count

// The trajectory table (kTraj), last so that the parameters before it keep their offsets in every variant
#define RDA_TRAJ_PARAMS const int *shape_traj, int K, const float *traj_xy
#define RDA_TRAJ_ARGS shape_traj, K, traj_xy

template <bool kPlan, bool kTraj>
__global__ void __launch_bounds__(kWorldTile) k_convert_world_obstacles(RDA_WORLD_PARAMS, RDA_TRAJ_PARAMS) {
  convert_world<kPlan, false, kTraj>(RDA_WORLD_ARGS, nullptr, RDA_TRAJ_ARGS);
}
template <bool kPlan, bool kTraj>
__global__ void __launch_bounds__(kWorldTile) k_convert_world_obstacles_ids(RDA_WORLD_PARAMS, int* obs_id,
                                                                             RDA_TRAJ_PARAMS) {
  convert_world<kPlan, true, kTraj>(RDA_WORLD_ARGS, obs_id, RDA_TRAJ_ARGS);
}

// Horizon order (rda_convert_world_obstacles_horizon): the tiles, candidates and merge of k_convert_world_obstacles
// with the key of horizon_key.cuh, the smallest signed distance of the robot's body over its nominal and reference
// poses.  Each tile goes in three steps:
//  1. a thread per shape: once N pairs are kept, a shape whose lower bound (the one-disc bound of the whole horizon,
//     then the bound of every pose) is >= the N-th kept key cannot enter, as every later shape has a larger index and
//     loses ties; the others are listed as survivors;
//  2. a warp per survivor: one lane per pose (2 (T + 1) poses), each the stage shape's rows and plan_clearance_cell,
//     and the warp's minimum: the exact key; keys that beat the N-th become candidates;
//  3. the merge of k_convert_world_obstacles.
// The selection is therefore that of sorting every exact key.  EC / RC: compile-time caps of the obstacle rows and
// body vertices (plan_clearance_cell).  The body (the one body, or body_xy_b [b] / body_radius_b [b]) and the horizon
// disc are staged once in shared memory.
#define RDA_HORIZON_PARAMS                                                                                             \
  int B, int W, int N, int T, int E, float dt, int time_varying, const float *nom_s, const float *ref_s, int body_kind, \
      int body_nv, const float *body_xy, float body_radius, const float *body_xy_b, const float *body_radius_b,        \
      const int *world_start, const int *robot_world, const int *shape_kind, const int *shape_nv,                      \
      const float *shape_xy, const float *shape_radius, const float *shape_vel, const int *fleet_start,                \
      const int *fleet_robot, const int *fleet_kind, const int *fleet_nv, const float *fleet_xy,                       \
      const float *fleet_radius, const float *fleet_vel, const float *fleet_plan_xy, float *obs_A, float *obs_b,        \
      int *obs_kind, int *obs_count
#define RDA_HORIZON_ARGS                                                                                               \
  B, W, N, T, E, dt, time_varying, nom_s, ref_s, body_kind, body_nv, body_xy, body_radius, body_xy_b, body_radius_b,     \
      world_start, robot_world, shape_kind, shape_nv, shape_xy, shape_radius, shape_vel, fleet_start, fleet_robot,      \
      fleet_kind, fleet_nv, fleet_xy, fleet_radius, fleet_vel, fleet_plan_xy, obs_A, obs_b, obs_kind, obs_count

template <int EC, int RC, bool kPlan, bool kIds, bool kTraj>
__device__ __forceinline__ void convert_world_horizon(RDA_HORIZON_PARAMS, int* obs_id, RDA_TRAJ_PARAMS) {
  // dynamic shared memory: as k_convert_world_obstacles, then the survivors of a tile [tile]
  extern __shared__ double sh[];
  __shared__ int n_surv, n_cand;
  __shared__ RobotGeom body;
  __shared__ double hor[4];                            // horizon disc centre, radius; body reach
  const int b = blockIdx.x;
  if (b >= B) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int w = robot_world ? robot_world[b] : 0;
  ShapeList L = {0, 0, 0, 0};
  if (w >= 0 && w < W) {
    L.first = world_start[w];
    L.n_world = world_start[w + 1] - L.first;
    if (L.n_world < 0) L.n_world = 0;
    if (fleet_start) {
      L.mate0 = fleet_start[w];
      L.mates = fleet_start[w + 1] - L.mate0 - 1;
      if (L.mates < 0) L.mates = 0;
    }
  }
  const int count = L.n_world + L.mates;
  const int T1 = T + 1;
  const double dtd = dt;
  int cur = 0;
  int* kept_idx = nullptr;
  if (count > 0) {
    double* kkey = sh;                                 // [2][N]
    double* ckey = kkey + 2 * N;                       // gathered [tile], sorted [tile]
    double* skey = ckey + kWorldTile;
    int* kidx = (int*)(skey + kWorldTile);             // [2][N]
    int* cidx = kidx + 2 * N;
    int* sidx = cidx + kWorldTile;
    int* surv = sidx + kWorldTile;                     // [tile]
    const float* nom = nom_s + (size_t)b * 3 * T1;
    const float* ref = ref_s + (size_t)b * 3 * T1;
    if (tid == 0) {
      body_geom(body_kind, body_nv, body_xy_b ? body_xy_b + (size_t)b * RDA_MAX_EDGE * 2 : body_xy,
                body_radius_b ? body_radius_b[b] : body_radius, &body);
      hor[3] = body_reach(body);
      if (horizon_disc(nom, ref, T, &hor[0], &hor[1], &hor[2]) == 0) hor[2] = -1;   // no finite pose: keys +inf
    }
    int nk = 0;                                        // pairs kept so far (uniform across the CTA)
    for (int base = 0; base < count; base += kWorldTile) {
      if (tid == 0) { n_surv = 0; n_cand = 0; }
      __syncthreads();                                 // also: the previous tile's counters have been read
      const double thr = nk < N ? INFINITY : kkey[cur * N + N - 1];
      const int i = base + tid;
      if (i < count) {
        bool mate;
        const size_t s = list_entry(L, i, fleet_robot, b, B, &mate);
        bool keep = nk < N;
        if (!keep && hor[2] >= 0) {                    // without a finite pose every key is +inf and loses to the kept
          const float* vel = (mate ? fleet_vel : shape_vel) + 2 * s;
          const RawShape r = {(mate ? fleet_kind : shape_kind)[s], (mate ? fleet_nv : shape_nv)[s],
                              (mate ? fleet_xy : shape_xy) + s * RDA_MAX_EDGE * 2,
                              (double)(mate ? fleet_radius : shape_radius)[s], (double)vel[0], (double)vel[1],
                              kPlan && mate ? fleet_plan_xy + s * T1 * RDA_MAX_EDGE * 2
                              : kTraj && !mate ? world_traj(shape_traj, K, traj_xy, T1, s) : nullptr};
          keep = horizon_disc_bound(r, time_varying, T, dtd, E, hor[0], hor[1], hor[2], hor[3]) < thr &&
                 horizon_bound(r, time_varying, T, dtd, E, nom, ref, hor[3], thr) < thr;
        }
        if (keep) surv[atomicAdd(&n_surv, 1)] = i;
      }
      __syncthreads();
      const int ns = n_surv;
      for (int k = warp; k < ns; k += kWorldTile / 32) {   // a warp per survivor, a lane per pose
        const int ix = surv[k];
        bool mate;
        const size_t s = list_entry(L, ix, fleet_robot, b, B, &mate);
        const float* vel = (mate ? fleet_vel : shape_vel) + 2 * s;
        const RawShape r = {(mate ? fleet_kind : shape_kind)[s], (mate ? fleet_nv : shape_nv)[s],
                            (mate ? fleet_xy : shape_xy) + s * RDA_MAX_EDGE * 2,
                            (double)(mate ? fleet_radius : shape_radius)[s], (double)vel[0], (double)vel[1],
                            kPlan && mate ? fleet_plan_xy + s * T1 * RDA_MAX_EDGE * 2
                            : kTraj && !mate ? world_traj(shape_traj, K, traj_xy, T1, s) : nullptr};
        double key = INFINITY;
        for (int q = lane; q < 2 * T1; q += 32) {
          const float* p = q < T1 ? nom : ref;
          const int t = q < T1 ? q : q - T1;
          if (!pose_finite(p, T1, t)) continue;
          const double v = horizon_cell<EC, RC>(body, r, time_varying ? t : 0, dtd, E, p[t], p[T1 + t], p[2 * T1 + t]);
          if (v < key) key = v;
        }
        for (int off = 16; off > 0; off >>= 1) {
          const double o = __shfl_xor_sync(0xffffffffu, key, off);
          key = o < key ? o : key;
        }
        if (lane == 0 && (nk < N || key < thr)) {
          const int p = atomicAdd(&n_cand, 1);
          ckey[p] = key; cidx[p] = ix;
        }
      }
      __syncthreads();
      const int c = n_cand;
      if (c > 0) world_merge(tid, c, N, kkey, kidx, ckey, cidx, skey, sidx, nk, cur);
    }
    kept_idx = kidx + cur * N;
  }
  if (tid == 0) obs_count[b] = count;
  world_slots<kPlan, kTraj>(tid, b, B, N, T, E, dt, time_varying, count, L, kept_idx, shape_kind, shape_nv, shape_xy,
                            shape_radius, shape_vel, fleet_robot, fleet_kind, fleet_nv, fleet_xy, fleet_radius,
                            fleet_vel, fleet_plan_xy, obs_A, obs_b, obs_kind, shape_traj, K, traj_xy);
  if (kIds) world_slot_ids(tid, b, B, N, count, L, kept_idx, fleet_robot, world_start[W], obs_id);
}

template <int EC, int RC, bool kPlan, bool kTraj>
__global__ void __launch_bounds__(kWorldTile) k_convert_world_obstacles_horizon(RDA_HORIZON_PARAMS, RDA_TRAJ_PARAMS) {
  convert_world_horizon<EC, RC, kPlan, false, kTraj>(RDA_HORIZON_ARGS, nullptr, RDA_TRAJ_ARGS);
}
template <int EC, int RC, bool kPlan, bool kTraj>
__global__ void __launch_bounds__(kWorldTile) k_convert_world_obstacles_horizon_ids(RDA_HORIZON_PARAMS, int* obs_id,
                                                                                     RDA_TRAJ_PARAMS) {
  convert_world_horizon<EC, RC, kPlan, true, kTraj>(RDA_HORIZON_ARGS, obs_id, RDA_TRAJ_ARGS);
}

// Each robot of a fleet as a raw shape for its map-mates (fleet_shape), one thread per robot: its body at its pose,
// moving with the first control of cur_vel, the one rda_motion_predict moved it with.  dyn_b [B], body_xy_b [B][8][2] and
// body_radius_b [B]: each robot's own dynamics and body (robot classes), or NULL: the scalars / the one body for every robot.
// kPlan: also each robot's body along its plan, plan_xy [B][T+1][RDA_MAX_EDGE][2] (16-byte aligned; fleet_plan, serial
// over T in the robot's thread), with time step dt and wheelbase L, or L_b [B] per robot.  The variant without plans
// never reads them, and compiles to the code it had before plans existed.
template <bool kPlan>
__global__ void k_fleet_shapes(int B, int T, int dynamics, int body_kind, int body_nv, const float* body_xy,
                               float body_radius, const int* dyn_b, const float* body_xy_b, const float* body_radius_b,
                               const float* state, const float* cur_vel, int* shape_kind,
                               int* shape_nv, float* shape_xy, float* shape_radius, float* shape_vel, float dt, float L,
                               const float* L_b, float* plan_xy) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float* u = cur_vel + (size_t)b * 2 * T;
  if (dyn_b) dynamics = dyn_b[b];
  if (body_xy_b) body_xy = body_xy_b + (size_t)b * RDA_MAX_EDGE * 2;
  if (body_radius_b) body_radius = body_radius_b[b];
  fleet_shape(dynamics, body_kind, body_nv, body_xy, body_radius, state + 3 * (size_t)b, (double)u[0], (double)u[T],
              shape_kind + b, shape_nv + b, shape_xy + (size_t)b * RDA_MAX_EDGE * 2, shape_radius + b,
              shape_vel + 2 * (size_t)b);
  if (!kPlan) return;
  if (L_b) L = L_b[b];
  fleet_plan(dynamics, (double)dt, (double)L, body_kind, body_nv, body_xy, state + 3 * (size_t)b, u, T,
             plan_xy + (size_t)b * (T + 1) * RDA_MAX_EDGE * 2);
}

// End-of-curve and arrive rules of MPC.control (mpc.py:166-185) on each robot's own curve and path, one thread per
// robot.  At the end of a curve that is not its path's last the robot moves on to the next curve (cur_index back to 0,
// controls kept); past its path's last curve, or without a path, its controls are zeroed and arrive is set.  cur_vel
// (may be NULL) receives the controls kept (mpc.py:186).  near_index and curve_index are only written on a curve
// switch, which a path of one curve never makes.
__global__ void k_post_process_paths(int B, int T, int P, int W, int n_curves, const int* path_curve,
                                     const int* curve_start, const int* robot_path, int goal_index_threshold,
                                     int* near_index, int* curve_index, float* u_opt, float* cur_vel, int* arrive) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int w = robot_path ? robot_path[b] : 0;
  PathCurve cv;
  bool arr = true;
  if (w >= 0 && w < W &&
      resolve_curve(w, curve_index ? curve_index[b] : 0, path_curve, n_curves, curve_start, P, nullptr, &cv)) {
    arr = false;
    if (near_index[b] >= cv.len - goal_index_threshold) {
      if (cv.index + 1 < cv.count) { curve_index[b] = cv.index + 1; near_index[b] = 0; }   // next curve
      else arr = true;                                                                     // past the last curve
    }
  }
  float* u = u_opt + (size_t)b * 2 * T;
  for (int i = 0; i < 2 * T; ++i) {
    if (arr) u[i] = 0.f;
    if (cur_vel) cur_vel[(size_t)b * 2 * T + i] = u[i];
  }
  if (arrive) arrive[b] = arr ? 1 : 0;
}

// dyn_b / L_b [B]: each robot's own dynamics and wheelbase, or NULL: the scalars for every robot
__global__ void k_motion_predict(int B, int T, int dynamics, float dt, float L, const int* dyn_b, const float* L_b,
                                 const float* u_opt, float* state) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  if (dyn_b) dynamics = dyn_b[b];
  if (L_b) L = L_b[b];
  const double s[3] = {state[3 * b], state[3 * b + 1], state[3 * b + 2]};
  double o[3];
  motion_predict(dynamics, (double)dt, (double)L, s, (double)u_opt[(size_t)b * 2 * T], (double)u_opt[(size_t)b * 2 * T + T], o);
  state[3 * b] = (float)o[0]; state[3 * b + 1] = (float)o[1]; state[3 * b + 2] = (float)o[2];
}

// The checks of the trajectory table (traj: the _traj entry points): both arrays, traj_xy 16-byte aligned, K >= 1 and
// time-varying output.
bool traj_args_ok(bool traj, int time_varying, const int32_t* shape_traj, int K, const float* traj_xy) {
  return !traj || (shape_traj && traj_xy && !((uintptr_t)traj_xy & 15) && K >= 1 && time_varying);
}

// Argument checks and launch of k_convert_world_obstacles.  Without `fleet` the fleet pointers are NULL and each robot
// chooses from its world's shapes only; fleet_plan_xy (fleet only, time-varying output only) may be NULL.  With `traj`
// world shapes may follow the trajectories of (shape_traj, K, traj_xy); without, those are not read.
int launch_world_obstacles(bool fleet, bool traj, int B, int W, int N, int T, int E, float dt, int time_varying, int order,
                           const float* state, const int32_t* world_start, const int32_t* robot_world,
                           const int32_t* shape_kind, const int32_t* shape_nv, const float* shape_xy,
                           const float* shape_radius, const float* shape_vel, const int32_t* fleet_start,
                           const int32_t* fleet_robot, const int32_t* fleet_kind, const int32_t* fleet_nv,
                           const float* fleet_xy, const float* fleet_radius, const float* fleet_vel,
                           const float* fleet_plan_xy, float* obs_A, float* obs_b, int32_t* obs_kind,
                           int32_t* obs_count, int32_t* obs_id, const int32_t* shape_traj, int K,
                           const float* traj_xy, cudaStream_t stream) {
  if (B < 1 || W < 1 || N < 1 || T < 1) return RDA_E_ARG;
  if (N > RDA_MAX_WORLD_SLOTS || E < 3 || E > RDA_MAX_EDGE) return RDA_E_UNSUPPORTED;
  if (!world_start || !shape_kind || !shape_nv || !shape_xy || !shape_radius || !shape_vel) return RDA_E_ARG;
  if (!obs_A || !obs_b || !obs_kind || !obs_count || (order && !state)) return RDA_E_ARG;
  if (fleet && (!fleet_start || !fleet_robot || !fleet_kind || !fleet_nv || !fleet_xy || !fleet_radius || !fleet_vel))
    return RDA_E_ARG;
  if (fleet_plan_xy && (!fleet || !time_varying)) return RDA_E_ARG;
  if (!traj_args_ok(traj, time_varying, shape_traj, K, traj_xy)) return RDA_E_ARG;
  const size_t smem = order ? (size_t)(2 * N + 2 * kWorldTile) * (sizeof(double) + sizeof(int)) : 0;
  const bool plan = fleet_plan_xy != nullptr;
  if (obs_id) {
    auto k = traj ? (plan ? k_convert_world_obstacles_ids<true, true> : k_convert_world_obstacles_ids<false, true>)
                  : (plan ? k_convert_world_obstacles_ids<true, false> : k_convert_world_obstacles_ids<false, false>);
    k<<<B, kWorldTile, smem, stream>>>(RDA_WORLD_ARGS, obs_id, RDA_TRAJ_ARGS);
  } else {
    auto k = traj ? (plan ? k_convert_world_obstacles<true, true> : k_convert_world_obstacles<false, true>)
                  : (plan ? k_convert_world_obstacles<true, false> : k_convert_world_obstacles<false, false>);
    k<<<B, kWorldTile, smem, stream>>>(RDA_WORLD_ARGS, RDA_TRAJ_ARGS);
  }
  RDA_CUDA(cudaGetLastError());
  return 0;
}

// Argument checks and launch of k_convert_world_obstacles_horizon.  fleet_start NULL: no fleet (the other fleet
// pointers are then not read); fleet_plan_xy (fleet only, time-varying output only) may be NULL; traj as for
// launch_world_obstacles.
int launch_world_obstacles_horizon(bool traj, int B, int W, int N, int T, int E, float dt, int time_varying, const float* nom_s,
                                   const float* ref_s, int body_kind, int body_nv, const float* body_xy,
                                   float body_radius, const float* body_xy_b, const float* body_radius_b,
                                   const int32_t* world_start, const int32_t* robot_world, const int32_t* shape_kind,
                                   const int32_t* shape_nv, const float* shape_xy, const float* shape_radius,
                                   const float* shape_vel, const int32_t* fleet_start, const int32_t* fleet_robot,
                                   const int32_t* fleet_kind, const int32_t* fleet_nv, const float* fleet_xy,
                                   const float* fleet_radius, const float* fleet_vel, const float* fleet_plan_xy,
                                   float* obs_A, float* obs_b, int32_t* obs_kind, int32_t* obs_count,
                                   int32_t* obs_id, const int32_t* shape_traj, int K, const float* traj_xy,
                                   cudaStream_t stream) {
  if (B < 1 || W < 1 || N < 1 || T < 1) return RDA_E_ARG;
  if (N > RDA_MAX_WORLD_SLOTS || E < 3 || E > RDA_MAX_EDGE) return RDA_E_UNSUPPORTED;
  if (body_kind == RDA_OBS_POLYGON) {
    if (body_nv < 3 || body_nv > RDA_MAX_ROBOT_EDGE) return RDA_E_UNSUPPORTED;
  } else if (body_kind != RDA_OBS_CIRCLE || (!body_radius_b && !(body_radius > 0.f))) {
    return RDA_E_ARG;
  }
  if ((!body_xy && !body_xy_b) || !nom_s || !ref_s) return RDA_E_ARG;
  if (!world_start || !shape_kind || !shape_nv || !shape_xy || !shape_radius || !shape_vel) return RDA_E_ARG;
  if (!obs_A || !obs_b || !obs_kind || !obs_count) return RDA_E_ARG;
  const bool fleet = fleet_start != nullptr;
  if (fleet && (!fleet_robot || !fleet_kind || !fleet_nv || !fleet_xy || !fleet_radius || !fleet_vel)) return RDA_E_ARG;
  if (fleet_plan_xy && (!fleet || !time_varying)) return RDA_E_ARG;
  if (!traj_args_ok(traj, time_varying, shape_traj, K, traj_xy)) return RDA_E_ARG;
  const bool small = E <= 4 && (body_kind == RDA_OBS_CIRCLE || body_nv <= 4);
  const bool plan = fleet_plan_xy != nullptr;
  const size_t smem = (size_t)(2 * N + 2 * kWorldTile) * (sizeof(double) + sizeof(int)) + kWorldTile * sizeof(int);
  if (obs_id) {
    auto k = traj ? (small ? (plan ? k_convert_world_obstacles_horizon_ids<4, 4, true, true>
                                   : k_convert_world_obstacles_horizon_ids<4, 4, false, true>)
                           : (plan ? k_convert_world_obstacles_horizon_ids<8, 8, true, true>
                                   : k_convert_world_obstacles_horizon_ids<8, 8, false, true>))
                  : (small ? (plan ? k_convert_world_obstacles_horizon_ids<4, 4, true, false>
                                   : k_convert_world_obstacles_horizon_ids<4, 4, false, false>)
                           : (plan ? k_convert_world_obstacles_horizon_ids<8, 8, true, false>
                                   : k_convert_world_obstacles_horizon_ids<8, 8, false, false>));
    k<<<B, kWorldTile, smem, stream>>>(RDA_HORIZON_ARGS, obs_id, RDA_TRAJ_ARGS);
  } else {
    auto k = traj ? (small ? (plan ? k_convert_world_obstacles_horizon<4, 4, true, true>
                                   : k_convert_world_obstacles_horizon<4, 4, false, true>)
                           : (plan ? k_convert_world_obstacles_horizon<8, 8, true, true>
                                   : k_convert_world_obstacles_horizon<8, 8, false, true>))
                  : (small ? (plan ? k_convert_world_obstacles_horizon<4, 4, true, false>
                                   : k_convert_world_obstacles_horizon<4, 4, false, false>)
                           : (plan ? k_convert_world_obstacles_horizon<8, 8, true, false>
                                   : k_convert_world_obstacles_horizon<8, 8, false, false>));
    k<<<B, kWorldTile, smem, stream>>>(RDA_HORIZON_ARGS, RDA_TRAJ_ARGS);
  }
  RDA_CUDA(cudaGetLastError());
  return 0;
}

#undef RDA_WORLD_PARAMS
#undef RDA_WORLD_ARGS
#undef RDA_HORIZON_PARAMS
#undef RDA_HORIZON_ARGS
#undef RDA_TRAJ_PARAMS
#undef RDA_TRAJ_ARGS

}  // namespace

extern "C" {

int rda_pre_process(int B, int T, int dynamics, float dt, float wheelbase, const float* state, const float* cur_vel,
                    const float* ref_speed, const float* path, int P, const int32_t* start_index, float threshold,
                    int ind_range, float* nom_s, float* ref_s, int32_t* near_index, void* stream) {
  if (B < 1 || T < 1 || P < 1 || dynamics < 0 || dynamics > 2) return RDA_E_ARG;
  if (!state || !cur_vel || !ref_speed || !path || !nom_s || !ref_s || !near_index) return RDA_E_ARG;
  k_pre_process_paths<<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
      B, T, dynamics, dt, wheelbase, nullptr, nullptr, state, cur_vel, ref_speed, path, P, 1, 1, nullptr, nullptr, nullptr, nullptr,
      nullptr, start_index, threshold, ind_range, nom_s, ref_s, near_index, nullptr);
  RDA_CUDA(cudaGetLastError());
  return 0;
}

int rda_pre_process_curves(int B, int T, int dynamics, float dt, float wheelbase, const float* state, const float* cur_vel,
                           const float* ref_speed, const float* path, int n_curves, const int32_t* curve_start,
                           const int32_t* curve_index, const int32_t* start_index, float threshold, int ind_range,
                           float* nom_s, float* ref_s, int32_t* near_index, void* stream) {
  if (B < 1 || T < 1 || n_curves < 1 || dynamics < 0 || dynamics > 2) return RDA_E_ARG;
  if (!state || !cur_vel || !ref_speed || !path || !curve_start || !curve_index || !nom_s || !ref_s || !near_index) return RDA_E_ARG;
  k_pre_process_paths<<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
      B, T, dynamics, dt, wheelbase, nullptr, nullptr, state, cur_vel, ref_speed, path, 0, 1, n_curves, nullptr, curve_start, nullptr,
      nullptr, curve_index, start_index, threshold, ind_range, nom_s, ref_s, near_index, nullptr);
  RDA_CUDA(cudaGetLastError());
  return 0;
}

int rda_pre_process_paths(int B, int T, int dynamics, float dt, float wheelbase, const float* state, const float* cur_vel,
                          const float* ref_speed, const float* path, int W, const int32_t* path_curve,
                          const int32_t* curve_start, const int32_t* curve_gear, const int32_t* robot_path,
                          const int32_t* curve_index, const int32_t* start_index, float threshold, int ind_range,
                          float* nom_s, float* ref_s, int32_t* near_index, float* solver_speed, void* stream) {
  if (B < 1 || T < 1 || W < 1 || dynamics < 0 || dynamics > 2) return RDA_E_ARG;
  if (!state || !cur_vel || !ref_speed || !path || !path_curve || !curve_start || !curve_gear) return RDA_E_ARG;
  if (!nom_s || !ref_s || !near_index) return RDA_E_ARG;
  k_pre_process_paths<<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
      B, T, dynamics, dt, wheelbase, nullptr, nullptr, state, cur_vel, ref_speed, path, 0, W, 0, path_curve, curve_start,
      curve_gear, robot_path, curve_index, start_index, threshold, ind_range, nom_s, ref_s, near_index, solver_speed);
  RDA_CUDA(cudaGetLastError());
  return 0;
}

int rda_pre_process_paths_per_robot(int B, int T, const int32_t* dynamics, float dt, const float* wheelbase,
                                    const float* state, const float* cur_vel, const float* ref_speed, const float* path,
                                    int W, const int32_t* path_curve, const int32_t* curve_start,
                                    const int32_t* curve_gear, const int32_t* robot_path, const int32_t* curve_index,
                                    const int32_t* start_index, float threshold, int ind_range, float* nom_s,
                                    float* ref_s, int32_t* near_index, float* solver_speed, void* stream) {
  if (B < 1 || T < 1 || W < 1 || !dynamics || !wheelbase) return RDA_E_ARG;
  if (!state || !cur_vel || !ref_speed || !path || !path_curve || !curve_start || !curve_gear) return RDA_E_ARG;
  if (!nom_s || !ref_s || !near_index) return RDA_E_ARG;
  k_pre_process_paths<<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
      B, T, 0, dt, 0.f, dynamics, wheelbase, state, cur_vel, ref_speed, path, 0, W, 0, path_curve, curve_start,
      curve_gear, robot_path, curve_index, start_index, threshold, ind_range, nom_s, ref_s, near_index, solver_speed);
  RDA_CUDA(cudaGetLastError());
  return 0;
}

int rda_post_process_gear(int B, int T, int n_curves, const int32_t* curve_start, int goal_index_threshold,
                          int32_t* near_index, int32_t* curve_index, float* u_opt, float* cur_vel, int32_t* arrive,
                          void* stream) {
  if (B < 1 || T < 1 || n_curves < 1 || !curve_start || !near_index || !curve_index || !u_opt) return RDA_E_ARG;
  k_post_process_paths<<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
      B, T, 0, 1, n_curves, nullptr, curve_start, nullptr, goal_index_threshold, near_index, curve_index, u_opt, cur_vel,
      arrive);
  RDA_CUDA(cudaGetLastError());
  return 0;
}

int rda_post_process_paths(int B, int T, int W, const int32_t* path_curve, const int32_t* curve_start,
                           const int32_t* robot_path, int goal_index_threshold, int32_t* near_index,
                           int32_t* curve_index, float* u_opt, float* cur_vel, int32_t* arrive, void* stream) {
  if (B < 1 || T < 1 || W < 1 || !path_curve || !curve_start || !near_index || !curve_index || !u_opt) return RDA_E_ARG;
  k_post_process_paths<<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
      B, T, 0, W, 0, path_curve, curve_start, robot_path, goal_index_threshold, near_index, curve_index, u_opt, cur_vel,
      arrive);
  RDA_CUDA(cudaGetLastError());
  return 0;
}

int rda_convert_obstacles(int B, int M, int N, int T, int E, float dt, int time_varying, int order, const float* state,
                          const int32_t* shape_kind, const int32_t* shape_nv, const float* shape_xy,
                          const float* shape_radius, const float* shape_vel, const int32_t* shape_count, float* obs_A,
                          float* obs_b, int32_t* obs_kind, int32_t* obs_count, void* stream) {
  if (B < 1 || N < 1 || T < 1 || M < 1) return RDA_E_ARG;
  if (M > RDA_MAX_SHAPES || E < 3 || E > RDA_MAX_EDGE) return RDA_E_UNSUPPORTED;
  if (!shape_kind || !shape_nv || !shape_xy || !shape_radius || !shape_vel || !shape_count) return RDA_E_ARG;
  if (!obs_A || !obs_b || !obs_kind || !obs_count || (order && !state)) return RDA_E_ARG;
  k_convert_obstacles<<<B, RDA_MAX_SHAPES, 0, (cudaStream_t)stream>>>(B, M, N, T, E, dt, time_varying, order, state, shape_kind,
                                                                     shape_nv, shape_xy, shape_radius, shape_vel,
                                                                     shape_count, obs_A, obs_b, obs_kind, obs_count);
  RDA_CUDA(cudaGetLastError());
  return 0;
}

int rda_convert_world_obstacles(int B, int W, int N, int T, int E, float dt, int time_varying, int order,
                                const float* state, const int32_t* world_start, const int32_t* robot_world,
                                const int32_t* shape_kind, const int32_t* shape_nv, const float* shape_xy,
                                const float* shape_radius, const float* shape_vel, float* obs_A, float* obs_b,
                                int32_t* obs_kind, int32_t* obs_count, void* stream) {
  return launch_world_obstacles(false, false, B, W, N, T, E, dt, time_varying, order, state, world_start, robot_world,
                                shape_kind, shape_nv, shape_xy, shape_radius, shape_vel, nullptr, nullptr, nullptr,
                                nullptr, nullptr, nullptr, nullptr, nullptr, obs_A, obs_b, obs_kind, obs_count,
                                nullptr, nullptr, 0, nullptr, (cudaStream_t)stream);
}

int rda_fleet_shapes(int B, int T, int dynamics, int body_kind, int body_nv, const float* body_xy, float body_radius,
                     const float* state, const float* cur_vel, int32_t* shape_kind, int32_t* shape_nv, float* shape_xy,
                     float* shape_radius, float* shape_vel, void* stream) {
  if (B < 1 || T < 1 || dynamics < 0 || dynamics > 2) return RDA_E_ARG;
  if (body_kind == RDA_OBS_POLYGON) {
    if (body_nv < 3 || body_nv > RDA_MAX_EDGE) return RDA_E_UNSUPPORTED;
  } else if (body_kind != RDA_OBS_CIRCLE || !(body_radius > 0.f)) {
    return RDA_E_ARG;
  }
  if (!body_xy || !state || !cur_vel || !shape_kind || !shape_nv || !shape_xy || !shape_radius || !shape_vel)
    return RDA_E_ARG;
  k_fleet_shapes<false><<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(B, T, dynamics, body_kind, body_nv, body_xy,
                                                                     body_radius, nullptr, nullptr, nullptr, state, cur_vel,
                                                                     shape_kind, shape_nv, shape_xy, shape_radius, shape_vel,
                                                                     0.f, 0.f, nullptr, nullptr);
  RDA_CUDA(cudaGetLastError());
  return 0;
}

int rda_fleet_shapes_per_robot(int B, int T, const int32_t* dynamics, int body_kind, int body_nv, const float* body_xy,
                               const float* body_radius, const float* state, const float* cur_vel, int32_t* shape_kind,
                               int32_t* shape_nv, float* shape_xy, float* shape_radius, float* shape_vel, void* stream) {
  if (B < 1 || T < 1 || !dynamics) return RDA_E_ARG;
  if (body_kind == RDA_OBS_POLYGON) {
    if (body_nv < 3 || body_nv > RDA_MAX_EDGE) return RDA_E_UNSUPPORTED;
  } else if (body_kind != RDA_OBS_CIRCLE) {
    return RDA_E_ARG;
  }
  if (!body_xy || !body_radius || !state || !cur_vel || !shape_kind || !shape_nv || !shape_xy || !shape_radius ||
      !shape_vel)
    return RDA_E_ARG;
  k_fleet_shapes<false><<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(B, T, 0, body_kind, body_nv, nullptr, 0.f, dynamics,
                                                                     body_xy, body_radius, state, cur_vel, shape_kind,
                                                                     shape_nv, shape_xy, shape_radius, shape_vel, 0.f, 0.f,
                                                                     nullptr, nullptr);
  RDA_CUDA(cudaGetLastError());
  return 0;
}

int rda_convert_fleet_obstacles(int B, int W, int N, int T, int E, float dt, int time_varying, int order,
                                const float* state, const int32_t* world_start, const int32_t* robot_world,
                                const int32_t* shape_kind, const int32_t* shape_nv, const float* shape_xy,
                                const float* shape_radius, const float* shape_vel, const int32_t* fleet_start,
                                const int32_t* fleet_robot, const int32_t* fleet_kind, const int32_t* fleet_nv,
                                const float* fleet_xy, const float* fleet_radius, const float* fleet_vel, float* obs_A,
                                float* obs_b, int32_t* obs_kind, int32_t* obs_count, void* stream) {
  return launch_world_obstacles(true, false, B, W, N, T, E, dt, time_varying, order, state, world_start, robot_world,
                                shape_kind, shape_nv, shape_xy, shape_radius, shape_vel, fleet_start, fleet_robot,
                                fleet_kind, fleet_nv, fleet_xy, fleet_radius, fleet_vel, nullptr, obs_A, obs_b,
                                obs_kind, obs_count, nullptr, nullptr, 0, nullptr, (cudaStream_t)stream);
}

int rda_fleet_plan_shapes(int B, int T, int dynamics, float dt, float wheelbase, int body_kind, int body_nv,
                          const float* body_xy, float body_radius, const int32_t* dynamics_b, const float* wheelbase_b,
                          const float* body_xy_b, const float* body_radius_b, const float* state, const float* cur_vel,
                          int32_t* shape_kind, int32_t* shape_nv, float* shape_xy, float* shape_radius,
                          float* shape_vel, float* plan_xy, void* stream) {
  if (B < 1 || T < 1 || (!dynamics_b && (dynamics < 0 || dynamics > 2))) return RDA_E_ARG;
  if (body_kind == RDA_OBS_POLYGON) {
    if (body_nv < 3 || body_nv > RDA_MAX_EDGE) return RDA_E_UNSUPPORTED;
  } else if (body_kind != RDA_OBS_CIRCLE || (!body_radius_b && !(body_radius > 0.f))) {
    return RDA_E_ARG;
  }
  if ((!body_xy && !body_xy_b) || !state || !cur_vel || !shape_kind || !shape_nv || !shape_xy || !shape_radius ||
      !shape_vel || !plan_xy || ((uintptr_t)plan_xy & 15))
    return RDA_E_ARG;
  k_fleet_shapes<true><<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
      B, T, dynamics, body_kind, body_nv, body_xy, body_radius, dynamics_b, body_xy_b, body_radius_b, state, cur_vel,
      shape_kind, shape_nv, shape_xy, shape_radius, shape_vel, dt, wheelbase, wheelbase_b, plan_xy);
  RDA_CUDA(cudaGetLastError());
  return 0;
}

int rda_convert_fleet_plan_obstacles(int B, int W, int N, int T, int E, float dt, int time_varying, int order,
                                     const float* state, const int32_t* world_start, const int32_t* robot_world,
                                     const int32_t* shape_kind, const int32_t* shape_nv, const float* shape_xy,
                                     const float* shape_radius, const float* shape_vel, const int32_t* fleet_start,
                                     const int32_t* fleet_robot, const int32_t* fleet_kind, const int32_t* fleet_nv,
                                     const float* fleet_xy, const float* fleet_radius, const float* fleet_vel,
                                     const float* fleet_plan_xy, float* obs_A, float* obs_b, int32_t* obs_kind,
                                     int32_t* obs_count, void* stream) {
  if (!fleet_plan_xy) return RDA_E_ARG;
  return launch_world_obstacles(true, false, B, W, N, T, E, dt, time_varying, order, state, world_start, robot_world,
                                shape_kind, shape_nv, shape_xy, shape_radius, shape_vel, fleet_start, fleet_robot,
                                fleet_kind, fleet_nv, fleet_xy, fleet_radius, fleet_vel, fleet_plan_xy, obs_A, obs_b,
                                obs_kind, obs_count, nullptr, nullptr, 0, nullptr, (cudaStream_t)stream);
}

int rda_convert_world_obstacles_horizon(int B, int W, int N, int T, int E, float dt, int time_varying,
                                        const float* nom_s, const float* ref_s, int body_kind, int body_nv,
                                        const float* body_xy, float body_radius, const float* body_xy_b,
                                        const float* body_radius_b, const int32_t* world_start,
                                        const int32_t* robot_world, const int32_t* shape_kind, const int32_t* shape_nv,
                                        const float* shape_xy, const float* shape_radius, const float* shape_vel,
                                        const int32_t* fleet_start, const int32_t* fleet_robot,
                                        const int32_t* fleet_kind, const int32_t* fleet_nv, const float* fleet_xy,
                                        const float* fleet_radius, const float* fleet_vel, const float* fleet_plan_xy,
                                        float* obs_A, float* obs_b, int32_t* obs_kind, int32_t* obs_count,
                                        void* stream) {
  return launch_world_obstacles_horizon(false, B, W, N, T, E, dt, time_varying, nom_s, ref_s, body_kind, body_nv, body_xy,
                                        body_radius, body_xy_b, body_radius_b, world_start, robot_world, shape_kind,
                                        shape_nv, shape_xy, shape_radius, shape_vel, fleet_start, fleet_robot,
                                        fleet_kind, fleet_nv, fleet_xy, fleet_radius, fleet_vel, fleet_plan_xy, obs_A,
                                        obs_b, obs_kind, obs_count, nullptr, nullptr, 0, nullptr, (cudaStream_t)stream);
}

int rda_convert_obstacles_ids(int B, int M, int N, int T, int E, float dt, int time_varying, int order,
                              const float* state, const int32_t* shape_kind, const int32_t* shape_nv,
                              const float* shape_xy, const float* shape_radius, const float* shape_vel,
                              const int32_t* shape_count, float* obs_A, float* obs_b, int32_t* obs_kind,
                              int32_t* obs_count, int32_t* obs_id, void* stream) {
  if (B < 1 || N < 1 || T < 1 || M < 1) return RDA_E_ARG;
  if (M > RDA_MAX_SHAPES || E < 3 || E > RDA_MAX_EDGE) return RDA_E_UNSUPPORTED;
  if (!shape_kind || !shape_nv || !shape_xy || !shape_radius || !shape_vel || !shape_count) return RDA_E_ARG;
  if (!obs_A || !obs_b || !obs_kind || !obs_count || !obs_id || (order && !state)) return RDA_E_ARG;
  k_convert_obstacles_ids<<<B, RDA_MAX_SHAPES, 0, (cudaStream_t)stream>>>(B, M, N, T, E, dt, time_varying, order, state,
                                                                         shape_kind, shape_nv, shape_xy, shape_radius,
                                                                         shape_vel, shape_count, obs_A, obs_b, obs_kind,
                                                                         obs_count, obs_id);
  RDA_CUDA(cudaGetLastError());
  return 0;
}

int rda_convert_world_obstacles_ids(int B, int W, int N, int T, int E, float dt, int time_varying, int order,
                                    const float* state, const int32_t* world_start, const int32_t* robot_world,
                                    const int32_t* shape_kind, const int32_t* shape_nv, const float* shape_xy,
                                    const float* shape_radius, const float* shape_vel, const int32_t* fleet_start,
                                    const int32_t* fleet_robot, const int32_t* fleet_kind, const int32_t* fleet_nv,
                                    const float* fleet_xy, const float* fleet_radius, const float* fleet_vel,
                                    const float* fleet_plan_xy, float* obs_A, float* obs_b, int32_t* obs_kind,
                                    int32_t* obs_count, int32_t* obs_id, void* stream) {
  if (!obs_id) return RDA_E_ARG;
  return launch_world_obstacles(fleet_start != nullptr, false, B, W, N, T, E, dt, time_varying, order, state, world_start,
                                robot_world, shape_kind, shape_nv, shape_xy, shape_radius, shape_vel, fleet_start,
                                fleet_robot, fleet_kind, fleet_nv, fleet_xy, fleet_radius, fleet_vel, fleet_plan_xy,
                                obs_A, obs_b, obs_kind, obs_count, obs_id, nullptr, 0, nullptr, (cudaStream_t)stream);
}

int rda_convert_world_obstacles_horizon_ids(int B, int W, int N, int T, int E, float dt, int time_varying,
                                            const float* nom_s, const float* ref_s, int body_kind, int body_nv,
                                            const float* body_xy, float body_radius, const float* body_xy_b,
                                            const float* body_radius_b, const int32_t* world_start,
                                            const int32_t* robot_world, const int32_t* shape_kind,
                                            const int32_t* shape_nv, const float* shape_xy, const float* shape_radius,
                                            const float* shape_vel, const int32_t* fleet_start,
                                            const int32_t* fleet_robot, const int32_t* fleet_kind,
                                            const int32_t* fleet_nv, const float* fleet_xy, const float* fleet_radius,
                                            const float* fleet_vel, const float* fleet_plan_xy, float* obs_A,
                                            float* obs_b, int32_t* obs_kind, int32_t* obs_count, int32_t* obs_id,
                                            void* stream) {
  if (!obs_id) return RDA_E_ARG;
  return launch_world_obstacles_horizon(false, B, W, N, T, E, dt, time_varying, nom_s, ref_s, body_kind, body_nv, body_xy,
                                        body_radius, body_xy_b, body_radius_b, world_start, robot_world, shape_kind,
                                        shape_nv, shape_xy, shape_radius, shape_vel, fleet_start, fleet_robot,
                                        fleet_kind, fleet_nv, fleet_xy, fleet_radius, fleet_vel, fleet_plan_xy, obs_A,
                                        obs_b, obs_kind, obs_count, obs_id, nullptr, 0, nullptr, (cudaStream_t)stream);
}

int rda_convert_world_obstacles_traj(int B, int W, int N, int T, int E, float dt, int time_varying, int order,
                                     const float* state, const int32_t* world_start, const int32_t* robot_world,
                                     const int32_t* shape_kind, const int32_t* shape_nv, const float* shape_xy,
                                     const float* shape_radius, const float* shape_vel, const int32_t* fleet_start,
                                     const int32_t* fleet_robot, const int32_t* fleet_kind, const int32_t* fleet_nv,
                                     const float* fleet_xy, const float* fleet_radius, const float* fleet_vel,
                                     const float* fleet_plan_xy, float* obs_A, float* obs_b, int32_t* obs_kind,
                                     int32_t* obs_count, int32_t* obs_id, const int32_t* shape_traj, int K,
                                     const float* traj_xy, void* stream) {
  return launch_world_obstacles(fleet_start != nullptr, true, B, W, N, T, E, dt, time_varying, order, state,
                                world_start, robot_world, shape_kind, shape_nv, shape_xy, shape_radius, shape_vel,
                                fleet_start, fleet_robot, fleet_kind, fleet_nv, fleet_xy, fleet_radius, fleet_vel,
                                fleet_plan_xy, obs_A, obs_b, obs_kind, obs_count, obs_id, shape_traj, K, traj_xy,
                                (cudaStream_t)stream);
}

int rda_convert_world_obstacles_horizon_traj(int B, int W, int N, int T, int E, float dt, int time_varying,
                                             const float* nom_s, const float* ref_s, int body_kind, int body_nv,
                                             const float* body_xy, float body_radius, const float* body_xy_b,
                                             const float* body_radius_b, const int32_t* world_start,
                                             const int32_t* robot_world, const int32_t* shape_kind,
                                             const int32_t* shape_nv, const float* shape_xy, const float* shape_radius,
                                             const float* shape_vel, const int32_t* fleet_start,
                                             const int32_t* fleet_robot, const int32_t* fleet_kind,
                                             const int32_t* fleet_nv, const float* fleet_xy, const float* fleet_radius,
                                             const float* fleet_vel, const float* fleet_plan_xy, float* obs_A,
                                             float* obs_b, int32_t* obs_kind, int32_t* obs_count, int32_t* obs_id,
                                             const int32_t* shape_traj, int K, const float* traj_xy, void* stream) {
  return launch_world_obstacles_horizon(true, B, W, N, T, E, dt, time_varying, nom_s, ref_s, body_kind, body_nv,
                                        body_xy, body_radius, body_xy_b, body_radius_b, world_start, robot_world,
                                        shape_kind, shape_nv, shape_xy, shape_radius, shape_vel, fleet_start,
                                        fleet_robot, fleet_kind, fleet_nv, fleet_xy, fleet_radius, fleet_vel,
                                        fleet_plan_xy, obs_A, obs_b, obs_kind, obs_count, obs_id, shape_traj, K,
                                        traj_xy, (cudaStream_t)stream);
}

int rda_post_process(int B, int T, int P, int goal_index_threshold, const int32_t* near_index, float* u_opt,
                     float* cur_vel, int32_t* arrive, void* stream) {
  if (B < 1 || T < 1 || !near_index || !u_opt) return RDA_E_ARG;
  // one curve of P waypoints: the kernel never switches curves, so near_index is only read
  k_post_process_paths<<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
      B, T, P, 1, 1, nullptr, nullptr, nullptr, goal_index_threshold, const_cast<int32_t*>(near_index), nullptr, u_opt,
      cur_vel, arrive);
  RDA_CUDA(cudaGetLastError());
  return 0;
}

int rda_motion_predict(int B, int T, int dynamics, float dt, float wheelbase, const float* u_opt, float* state,
                       void* stream) {
  if (B < 1 || T < 1 || dynamics < 0 || dynamics > 2 || !u_opt || !state) return RDA_E_ARG;
  k_motion_predict<<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(B, T, dynamics, dt, wheelbase, nullptr, nullptr,
                                                                       u_opt, state);
  RDA_CUDA(cudaGetLastError());
  return 0;
}

int rda_motion_predict_per_robot(int B, int T, const int32_t* dynamics, float dt, const float* wheelbase,
                                 const float* u_opt, float* state, void* stream) {
  if (B < 1 || T < 1 || !dynamics || !wheelbase || !u_opt || !state) return RDA_E_ARG;
  k_motion_predict<<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(B, T, 0, dt, 0.f, dynamics, wheelbase, u_opt, state);
  RDA_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
