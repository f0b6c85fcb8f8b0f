// CPU twin of k_pre_process_paths and k_post_process_paths (rda_frontend.cu) — test infrastructure only.
// The per-robot steps are restated here over the same resolve_curve and pre_process_one cores the kernels use:
// the path, curve and gear of each robot, the rollout and held reference of a robot without a path, and the
// end-of-curve and arrive rules (mpc.py:139-185).  Layouts and arguments as rda_pre_process_paths /
// rda_post_process_paths (include/rda_b200.h), on host arrays.
#include "../../rda_planner_b200/csrc/frontend.cuh"

namespace {

bool curve_of(int w, int W, int c, const int* path_curve, const int* curve_start, const int* curve_gear,
              rda::PathCurve* cv) {
  if (w < 0 || w >= W) return false;
  return rda::resolve_curve(w, c, path_curve, 0, curve_start, 0, curve_gear, cv);
}

}  // namespace

extern "C" void shim_pre_process_paths(int B, int T, int dynamics, float dt, float L, const float* state,
                                       const float* cur_vel, const float* ref_speed, const float* path, int W,
                                       const int* path_curve, const int* curve_start, const int* curve_gear,
                                       const int* robot_path, const int* curve_index, const int* start_index,
                                       float threshold, int ind_range, float* nom_s, float* ref_s, int* near_index,
                                       float* solver_speed) {
  const int S = T + 1;
  for (int b = 0; b < B; ++b) {
    const float* st = state + 3 * b;
    const float* vel = cur_vel + (size_t)b * 2 * T;
    float* nom = nom_s + (size_t)b * 3 * S;
    float* ref = ref_s + (size_t)b * 3 * S;
    rda::PathCurve cv;
    if (curve_of(robot_path[b], W, curve_index[b], path_curve, curve_start, curve_gear, &cv)) {
      near_index[b] = rda::pre_process_one(dynamics, T, (double)dt, (double)L, st, vel, (double)ref_speed[b],
                                           path + 3 * (size_t)cv.first, cv.len, start_index[b], (double)threshold,
                                           ind_range, nom, ref);
      solver_speed[b] = ref_speed[b] * (float)cv.gear;
      continue;
    }
    // no path: rollout with the previous controls, reference = the current state, index 0, gear +1
    double cur[3] = {st[0], st[1], st[2]};
    for (int r = 0; r < 3; ++r)
      for (int j = 0; j < S; ++j) ref[r * S + j] = st[r];
    for (int r = 0; r < 3; ++r) nom[r * S] = st[r];
    for (int i = 0; i < T; ++i) {
      double nxt[3];
      rda::motion_predict(dynamics, (double)dt, (double)L, cur, vel[i], vel[T + i], nxt);
      for (int r = 0; r < 3; ++r) { cur[r] = nxt[r]; nom[r * S + i + 1] = (float)nxt[r]; }
    }
    near_index[b] = 0;
    solver_speed[b] = ref_speed[b];
  }
}

extern "C" void shim_post_process_paths(int B, int T, int W, const int* path_curve, const int* curve_start,
                                        const int* robot_path, int goal_index_threshold, int* near_index,
                                        int* curve_index, float* u_opt, float* cur_vel, int* arrive) {
  for (int b = 0; b < B; ++b) {
    rda::PathCurve cv;
    bool arrived = true;
    if (curve_of(robot_path[b], W, curve_index[b], path_curve, curve_start, nullptr, &cv)) {
      const bool end_of_curve = near_index[b] >= cv.len - goal_index_threshold;
      const bool last_curve = cv.index == cv.count - 1;
      arrived = end_of_curve && last_curve;
      if (end_of_curve && !last_curve) {
        curve_index[b] = cv.index + 1;
        near_index[b] = 0;
      }
    }
    for (int i = 0; i < 2 * T; ++i) {
      float& u = u_opt[(size_t)b * 2 * T + i];
      if (arrived) u = 0.f;
      cur_vel[(size_t)b * 2 * T + i] = u;
    }
    arrive[b] = arrived ? 1 : 0;
  }
}
