// CPU twin of k_fleet_shapes (rda_frontend.cu) — test infrastructure only: the same fleet_shape core, one robot per
// loop step.  The selection over a robot's world and map-mates is checked with the world twin
// (world_obstacles.cpp) on the concatenated list.
#include <cstddef>
#include "../../rda_planner_b200/csrc/frontend.cuh"

// state [B][3], cur_vel [B][2][T]; body_xy [RDA_MAX_EDGE][2].  Out: kind, nv, radius [B], xy [B][RDA_MAX_EDGE][2],
// vel [B][2].
extern "C" void shim_fleet_shapes(int B, int T, int dynamics, int body_kind, int body_nv, const float* body_xy,
                                  float body_radius, const float* state, const float* cur_vel, int* kind, int* nv,
                                  float* xy, float* radius, float* vel) {
  for (int b = 0; b < B; ++b) {
    const float* u = cur_vel + (size_t)b * 2 * T;
    rda::fleet_shape(dynamics, body_kind, body_nv, body_xy, body_radius, state + 3 * (size_t)b, u[0], u[T], kind + b,
                     nv + b, xy + (size_t)b * RDA_MAX_EDGE * 2, radius + b, vel + 2 * (size_t)b);
  }
}
