// CPU twin of the trajectory variants of k_convert_world_obstacles and k_convert_world_obstacles_horizon
// (rda_frontend.cu, rda_convert_world_obstacles_traj / _horizon_traj) over one robot's list — test infrastructure only.
// An independent restatement of the selection, as world_obstacles.cpp and horizon_select.cpp: keys of every entry,
// std::stable_sort, the first N slots padded by repeating the last, rows from the same obstacle_rows / stage_rows cores.
//
// Entry j of the list: kind, nv, radius [count], xy [count][8][2], vel [count][2]; planned[j] != 0: a map-mate along
// plan_xy [count][T+1][8][2]; otherwise traj[j] in [0, K): a world shape along traj_xy [K][T+1][8][2], keyed by its
// stage 0; any other traj[j]: the shape's own xy and vel.  Always time-varying: obs_A [N][T+1][E][2], obs_b [N][T+1][E],
// obs_kind [N], and src [N] the list position written into each slot (-1 for an empty list).  Return count.
#include <algorithm>
#include <cstddef>
#include <vector>
#include "../../rda_planner_b200/csrc/horizon_key.cuh"

using namespace rda;

namespace {

// the entry's stage shapes: NULL for a shape at its xy and vel
const float* stages(int j, int T, const int* planned, const float* plan_xy, const int* traj, int K,
                    const float* traj_xy) {
  const size_t st = (size_t)(T + 1) * RDA_MAX_EDGE * 2;
  if (planned[j]) return plan_xy + j * st;
  if (traj[j] >= 0 && traj[j] < K) return traj_xy + traj[j] * st;
  return nullptr;
}

RawShape entry(int j, int T, const int* kind, const int* nv, const float* xy, const float* radius, const float* vel,
               const int* planned, const float* plan_xy, const int* traj, int K, const float* traj_xy) {
  return {kind[j], nv[j], xy + (size_t)j * RDA_MAX_EDGE * 2, (double)radius[j], (double)vel[2 * j],
          (double)vel[2 * j + 1], stages(j, T, planned, plan_xy, traj, K, traj_xy)};
}

void write_slots(const std::vector<int>& idx, int count, int N, int T, int E, double dt, const int* kind, const int* nv,
                 const float* xy, const float* radius, const float* vel, const int* planned, const float* plan_xy,
                 const int* traj, int K, const float* traj_xy, float* obs_A, float* obs_b, int* obs_kind, int* src) {
  const int Tc = T + 1;
  for (int n = 0; n < N; ++n) {
    float* A = obs_A + (size_t)n * Tc * E * 2;
    float* b = obs_b + (size_t)n * Tc * E;
    if (count == 0) {
      std::fill(A, A + (size_t)Tc * E * 2, 0.f);
      std::fill(b, b + (size_t)Tc * E, 0.f);
      obs_kind[n] = RDA_OBS_POLYGON;
      src[n] = -1;
      continue;
    }
    const int j = idx[n < count ? n : count - 1];
    src[n] = j;
    obs_kind[n] = kind[j];
    const RawShape s = entry(j, T, kind, nv, xy, radius, vel, planned, plan_xy, traj, K, traj_xy);
    for (int t = 0; t < Tc; ++t) stage_rows(s, t, dt, E, A + (size_t)t * E * 2, b + (size_t)t * E);
  }
}

}  // namespace

// The reference key (order != 0, from the robot's position state[0..1]) or list order.
extern "C" int shim_convert_traj_list(int count, int N, int T, int E, double dt, int order, const float* state,
                                      const int* kind, const int* nv, const float* xy, const float* radius,
                                      const float* vel, const int* planned, const float* plan_xy, const int* traj, int K,
                                      const float* traj_xy, float* obs_A, float* obs_b, int* obs_kind, int* src) {
  if (count < 0) count = 0;
  std::vector<int> idx(count);
  for (int j = 0; j < count; ++j) idx[j] = j;
  if (order) {
    std::vector<double> keys(count);
    for (int j = 0; j < count; ++j) {
      const float* st = stages(j, T, planned, plan_xy, traj, K, traj_xy);
      keys[j] = obstacle_key(kind[j], nv[j], st ? st : xy + (size_t)j * RDA_MAX_EDGE * 2, state[0], state[1]);
    }
    std::stable_sort(idx.begin(), idx.end(), [&](int a, int b) { return keys[a] < keys[b]; });
  }
  write_slots(idx, count, N, T, E, dt, kind, nv, xy, radius, vel, planned, plan_xy, traj, K, traj_xy, obs_A, obs_b,
              obs_kind, src);
  return count;
}

// The horizon order: nom, ref [3][T+1]; body in the robot_body format.  Also keys [count], every entry's exact key.
extern "C" int shim_horizon_traj_select(int count, int N, int T, int E, double dt, const float* nom, const float* ref,
                                        int body_kind, int body_nv, const float* body_xy, float body_radius,
                                        const int* kind, const int* nv, const float* xy, const float* radius,
                                        const float* vel, const int* planned, const float* plan_xy, const int* traj,
                                        int K, const float* traj_xy, double* keys, float* obs_A, float* obs_b,
                                        int* obs_kind, int* src) {
  if (count < 0) count = 0;
  RobotGeom rb;
  body_geom(body_kind, body_nv, body_xy, body_radius, &rb);
  const bool small = E <= 4 && (body_kind == RDA_OBS_CIRCLE || body_nv <= 4);
  std::vector<int> idx(count);
  for (int j = 0; j < count; ++j) {
    idx[j] = j;
    const RawShape s = entry(j, T, kind, nv, xy, radius, vel, planned, plan_xy, traj, K, traj_xy);
    keys[j] = small ? horizon_key<4, 4>(rb, s, 1, T, dt, E, nom, ref) : horizon_key<8, 8>(rb, s, 1, T, dt, E, nom, ref);
  }
  std::stable_sort(idx.begin(), idx.end(), [&](int a, int b) { return keys[a] < keys[b]; });
  write_slots(idx, count, N, T, E, dt, kind, nv, xy, radius, vel, planned, plan_xy, traj, K, traj_xy, obs_A, obs_b,
              obs_kind, src);
  return count;
}

// The kernel's two lower bounds of every entry: lb_disc [count] (one disc of the whole horizon; -inf for an entry with
// stage shapes) and lb_pose [count] (every pose on its own).
extern "C" void shim_horizon_traj_bounds(int count, int T, int E, double dt, const float* nom, const float* ref,
                                         int body_kind, int body_nv, const float* body_xy, float body_radius,
                                         const int* kind, const int* nv, const float* xy, const float* radius,
                                         const float* vel, const int* planned, const float* plan_xy, const int* traj,
                                         int K, const float* traj_xy, double* lb_disc, double* lb_pose) {
  RobotGeom rb;
  body_geom(body_kind, body_nv, body_xy, body_radius, &rb);
  const double reach = body_reach(rb);
  double hx, hy, hr;
  const bool any = horizon_disc(nom, ref, T, &hx, &hy, &hr) > 0;
  for (int j = 0; j < count; ++j) {
    const RawShape s = entry(j, T, kind, nv, xy, radius, vel, planned, plan_xy, traj, K, traj_xy);
    lb_disc[j] = any ? horizon_disc_bound(s, 1, T, dt, E, hx, hy, hr, reach) : INFINITY;
    lb_pose[j] = horizon_bound(s, 1, T, dt, E, nom, ref, reach, -INFINITY);
  }
}
