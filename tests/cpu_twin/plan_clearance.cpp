// CPU twin of rda_plan_clearance's cell core (plan_clearance.cuh) — test infrastructure only.  The body is stored by
// robot_geom_from_halfspaces, as rda_create does, and each cell goes through plan_clearance_cell with the caps the
// kernel launch picks (4 / 4 when E <= 4 and R <= 4, else 8 / 8).
#include "../../rda_planner_b200/csrc/plan_clearance.cuh"

using namespace rda;

// n cells: kind [n], A [n][E][2], b [n][E], pose [n][3] -> out [n] (float64, before the kernel's rounding to float32)
extern "C" int twin_plan_clearance(const float* G, const float* h, int R, int cone, int n, int E, const int* kind,
                                   const float* A, const float* b, const float* pose, double* out) {
  RobotGeom rb;
  const int rc = robot_geom_from_halfspaces(G, h, R, &rb, cone);
  if (rc) return rc;
  if (E < 1 || E > RDA_MAX_EDGE) return RDA_E_ARG;
  const bool small = E <= 4 && R <= 4;
  for (int k = 0; k < n; ++k) {
    const float* Ak = A + (size_t)k * E * 2;
    const float* bk = b + (size_t)k * E;
    const float* p = pose + 3 * (size_t)k;
    out[k] = small ? plan_clearance_cell<4, 4>(rb, kind[k], E, Ak, bk, p[0], p[1], p[2])
                   : plan_clearance_cell<8, 8>(rb, kind[k], E, Ak, bk, p[0], p[1], p[2]);
  }
  return 0;
}
