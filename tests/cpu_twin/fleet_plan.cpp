// CPU twin of the plan mode of k_fleet_shapes and k_convert_world_obstacles (rda_frontend.cu) — test infrastructure
// only.  The body placement and the rollout are the same fleet_shape / fleet_plan cores, one robot per loop step; the
// selection is an independent restatement over one robot's list (as world_obstacles.cpp): keys of every entry,
// std::stable_sort, first N slots padded by repeating the last, rows from obstacle_rows.
#include <algorithm>
#include <cstddef>
#include <vector>
#include "../../rda_planner_b200/csrc/frontend.cuh"

// state [B][3], cur_vel [B][2][T]; body_xy [RDA_MAX_EDGE][2] or, when body_xy_b is not NULL, [B][RDA_MAX_EDGE][2];
// dyn_b, L_b, radius_b [B] or NULL (the scalar).  Out: kind, nv, radius [B], xy [B][RDA_MAX_EDGE][2], vel [B][2],
// plan_xy [B][T+1][RDA_MAX_EDGE][2].
extern "C" void shim_fleet_plan_shapes(int B, int T, int dynamics, double dt, double L, int body_kind, int body_nv,
                                       const float* body_xy, float body_radius, const int* dyn_b, const float* L_b,
                                       const float* body_xy_b, const float* radius_b, const float* state,
                                       const float* cur_vel, int* kind, int* nv, float* xy, float* radius, float* vel,
                                       float* plan_xy) {
  for (int b = 0; b < B; ++b) {
    const float* u = cur_vel + (size_t)b * 2 * T;
    const int dyn = dyn_b ? dyn_b[b] : dynamics;
    const float* bxy = body_xy_b ? body_xy_b + (size_t)b * RDA_MAX_EDGE * 2 : body_xy;
    rda::fleet_shape(dyn, body_kind, body_nv, bxy, radius_b ? radius_b[b] : body_radius, state + 3 * (size_t)b, u[0],
                     u[T], kind + b, nv + b, xy + (size_t)b * RDA_MAX_EDGE * 2, radius + b, vel + 2 * (size_t)b);
    rda::fleet_plan(dyn, dt, L_b ? (double)L_b[b] : L, body_kind, body_nv, bxy, state + 3 * (size_t)b, u, T,
                    plan_xy + (size_t)b * (T + 1) * RDA_MAX_EDGE * 2);
  }
}

// One robot's list of `count` raw shapes (kind, nv, radius [count], xy [count][RDA_MAX_EDGE][2], vel [count][2]);
// entries with planned[j] != 0 are map-mates whose stage-t shape is plan_xy [count][T+1][RDA_MAX_EDGE][2] at [j][t],
// standing.  Always time-varying: out obs_A [N][T+1][E][2], obs_b [N][T+1][E], obs_kind [N].  Returns count.
extern "C" int shim_convert_plan_list(int count, int N, int T, int E, double dt, int order, const float* state,
                                      const int* kind, const int* nv, const float* xy, const float* radius,
                                      const float* vel, const int* planned, const float* plan_xy, float* obs_A,
                                      float* obs_b, int* obs_kind) {
  if (count < 0) count = 0;
  std::vector<int> idx(count);
  for (int j = 0; j < count; ++j) idx[j] = j;
  if (order) {
    std::vector<double> keys(count);
    for (int j = 0; j < count; ++j)
      keys[j] = rda::obstacle_key(kind[j], nv[j], xy + (size_t)j * RDA_MAX_EDGE * 2, state[0], state[1]);
    std::stable_sort(idx.begin(), idx.end(), [&](int a, int b) { return keys[a] < keys[b]; });
  }
  const int Tc = T + 1;
  for (int n = 0; n < N; ++n) {
    float* A = obs_A + (size_t)n * Tc * E * 2;
    float* b = obs_b + (size_t)n * Tc * E;
    if (count == 0) {
      std::fill(A, A + (size_t)Tc * E * 2, 0.f);
      std::fill(b, b + (size_t)Tc * E, 0.f);
      obs_kind[n] = RDA_OBS_POLYGON;
      continue;
    }
    const int src = idx[n < count ? n : count - 1];
    obs_kind[n] = kind[src];
    for (int t = 0; t < Tc; ++t) {
      if (planned[src])
        rda::obstacle_rows(kind[src], nv[src], plan_xy + ((size_t)src * Tc + t) * RDA_MAX_EDGE * 2, radius[src], 0.0,
                           0.0, t, dt, E, A + (size_t)t * E * 2, b + (size_t)t * E);
      else
        rda::obstacle_rows(kind[src], nv[src], xy + (size_t)src * RDA_MAX_EDGE * 2, radius[src], vel[2 * src],
                           vel[2 * src + 1], t, dt, E, A + (size_t)t * E * 2, b + (size_t)t * E);
    }
  }
  return count;
}
