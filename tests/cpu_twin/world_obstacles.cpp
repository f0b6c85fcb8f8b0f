// CPU twin of k_convert_world_obstacles (rda_frontend.cu), one robot per call — test infrastructure only.
// An independent restatement of the selection: keys of the robot's whole world, std::stable_sort by key
// (ties keep list order, as Python's list.sort in MPC.convert_rda_obstacle), first N slots padded by
// repeating the last; rows from the same obstacle_rows core the kernel uses.
#include <algorithm>
#include <vector>
#include "../../rda_planner_b200/csrc/frontend.cuh"

// world: `count` shapes (kind [count], nv [count], xy [count][RDA_MAX_EDGE][2], radius [count], vel [count][2]).
// Out: obs_A [N][Tc][E][2], obs_b [N][Tc][E], obs_kind [N].  Returns count (obs_count).
extern "C" int shim_convert_world_obstacles(int count, int N, int T, int E, double dt, int time_varying, int order,
                                            const float* state, const int* kind, const int* nv, const float* xy,
                                            const float* radius, const float* vel, float* obs_A, float* obs_b,
                                            int* obs_kind) {
  if (count < 0) count = 0;
  std::vector<int> idx(count);
  for (int j = 0; j < count; ++j) idx[j] = j;
  if (order) {
    std::vector<double> keys(count);
    for (int j = 0; j < count; ++j)
      keys[j] = rda::obstacle_key(kind[j], nv[j], xy + (size_t)j * RDA_MAX_EDGE * 2, state[0], state[1]);
    std::stable_sort(idx.begin(), idx.end(), [&](int a, int b) { return keys[a] < keys[b]; });
  }
  const int Tc = time_varying ? T + 1 : 1;
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
    for (int t = 0; t < Tc; ++t)
      rda::obstacle_rows(kind[src], nv[src], xy + (size_t)src * RDA_MAX_EDGE * 2, radius[src], vel[2 * src],
                         vel[2 * src + 1], t, dt, E, A + (size_t)t * E * 2, b + (size_t)t * E);
  }
  return count;
}
