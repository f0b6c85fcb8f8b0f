// CPU twin of the slot match of rda_set_obstacle_ids (obstacle_ids.cuh), and the reference's sort key of raw shapes for
// restating which list entries a selection keeps — test infrastructure only.
#include "../../rda_planner_b200/csrc/frontend.cuh"
#include "../../rda_planner_b200/csrc/obstacle_ids.cuh"

// prev, cur [N] -> src [N] (-1: cold start)
extern "C" void shim_obstacle_slot_source(const int* prev, const int* cur, int N, int* src) {
  for (int n = 0; n < N; ++n) src[n] = rda::obstacle_slot_source(prev, cur, N, n);
}

// obstacle_key (as k_convert_world_obstacles computes it) of `count` raw shapes seen from (sx, sy)
extern "C" void shim_obstacle_keys(int count, double sx, double sy, const int* kind, const int* nv, const float* xy,
                                   double* keys) {
  for (int j = 0; j < count; ++j) keys[j] = rda::obstacle_key(kind[j], nv[j], xy + (size_t)j * RDA_MAX_EDGE * 2, sx, sy);
}
