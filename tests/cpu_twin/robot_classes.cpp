// CPU twin of the robot classes of a handle (rda_set_robot_classes / rda_set_robot_class_index) — test infrastructure
// only.  The g++ build of the kernels' cores (oracle/cpu_port) solves with one rda_config per call; this twin gives
// instance b the body, wheelbase, dynamics and limits of its class, picked with the helpers the kernels use: class_slot
// for the slot (an index outside [0, K) is the handle's own) and su_params_class for the su-QP's dynamics and wheelbase.
// Each instance is then solved on its own: instances of a batch never interact.  Layouts as port_solve_batch;
// robot_class may be NULL (the handle's own for every instance, port_solve_batch itself).
#include <cstring>
#include "../../oracle/cpu_port/rda_cpu_port.h"
#include "../../rda_planner_b200/csrc/su_solver.cuh"

using namespace rda;

// limits: [K][4] max_speed[2], acce_bound[2] of each class (the per-instance table columns the classes set)
extern "C" int twin_solve_batch_cls(const rda_config* cfg, const rda_tunables* tun, int B, const float* nom_s,
                                    const float* nom_u, const float* ref_s, const float* ref_speed, const float* obs_A,
                                    const float* obs_b, const int* obs_kind, const int* obs_count, int tv, int iter_num,
                                    float thr, float* u_opt, float* s_opt, float* resi_pri, float* resi_dual,
                                    int* iters_out, int* fails_out, int nthreads, int K, const rda_robot_class* classes,
                                    const float* limits, const int* robot_class) {
  if (!robot_class)
    return port_solve_batch(cfg, tun, B, nom_s, nom_u, ref_s, ref_speed, obs_A, obs_b, obs_kind, obs_count, tv, iter_num,
                            thr, u_opt, s_opt, resi_pri, resi_dual, iters_out, fails_out, nthreads);
  const size_t T = cfg->receding, N = cfg->max_obs_num, E = cfg->max_edge_num, Tc = tv ? T + 1 : 1;
  for (int b = 0; b < B; ++b) {
    const int slot = class_slot(robot_class, K, b);
    rda_config c = *cfg;
    c.batch = 1;
    if (slot < K) {
      const rda_robot_class& k = classes[slot];
      SuParams P;
      P.dynamics = cfg->dynamics; P.L = cfg->wheelbase;
      su_params_class(P, ClassKin{k.dynamics, k.wheelbase});
      c.dynamics = P.dynamics; c.wheelbase = P.L;
      memcpy(c.G, k.G, sizeof(c.G));
      memcpy(c.h, k.h, sizeof(c.h));
      c.max_speed[0] = limits[4 * slot]; c.max_speed[1] = limits[4 * slot + 1];
      c.acce_bound[0] = limits[4 * slot + 2]; c.acce_bound[1] = limits[4 * slot + 3];
    }
    const int rc = port_solve_batch(
        &c, tun, 1, nom_s + b * 3 * (T + 1), nom_u + b * 2 * T, ref_s + b * 3 * (T + 1), ref_speed + b,
        obs_A ? obs_A + b * N * Tc * E * 2 : nullptr, obs_b ? obs_b + b * N * Tc * E : nullptr,
        obs_kind ? obs_kind + b * N : nullptr, obs_count ? obs_count + b : nullptr, tv, iter_num, thr,
        u_opt + b * 2 * T, s_opt + b * 3 * (T + 1), resi_pri + b, resi_dual + b, iters_out ? iters_out + b : nullptr,
        fails_out ? fails_out + 4 * b : nullptr, nthreads);
    if (rc) return rc;
  }
  return 0;
}
