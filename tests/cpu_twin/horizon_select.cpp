// CPU twin of k_convert_world_obstacles_horizon (rda_frontend.cu) — test infrastructure only.  Brute force over one
// robot's list: the exact key (horizon_key.cuh) of every entry, std::stable_sort, the first N slots padded by repeating
// the last, rows from stage_rows.  Also the lower bounds the kernel prunes with, and how many entries the kernel's tile
// scan hands to the exact key.
#include <algorithm>
#include <cstddef>
#include <vector>
#include "../../rda_planner_b200/csrc/horizon_key.cuh"

using namespace rda;

namespace {

// entry j of the list: kind, nv, radius [count], xy [count][8][2], vel [count][2]; planned[j] != 0: a map-mate along
// plan_xy [count][T+1][8][2]
RawShape entry(int j, int T, const int* kind, const int* nv, const float* xy, const float* radius, const float* vel,
               const int* planned, const float* plan_xy) {
  return {kind[j], nv[j], xy + (size_t)j * RDA_MAX_EDGE * 2, (double)radius[j], (double)vel[2 * j],
          (double)vel[2 * j + 1], planned && planned[j] ? plan_xy + (size_t)j * (T + 1) * RDA_MAX_EDGE * 2 : nullptr};
}

double exact_key(const RobotGeom& rb, bool small, const RawShape& s, int tv, int T, double dt, int E, const float* nom,
                 const float* ref) {
  return small ? horizon_key<4, 4>(rb, s, tv, T, dt, E, nom, ref) : horizon_key<8, 8>(rb, s, tv, T, dt, E, nom, ref);
}

}  // namespace

// nom, ref [3][T+1]; body in the robot_body format.  Out: keys [count], obs_A [N][Tc][E][2], obs_b [N][Tc][E],
// obs_kind [N].  Returns count.
extern "C" int shim_horizon_select(int count, int N, int T, int E, double dt, int tv, const float* nom, const float* ref,
                                   int body_kind, int body_nv, const float* body_xy, float body_radius, const int* kind,
                                   const int* nv, const float* xy, const float* radius, const float* vel,
                                   const int* planned, const float* plan_xy, double* keys, float* obs_A, float* obs_b,
                                   int* obs_kind) {
  if (count < 0) count = 0;
  RobotGeom rb;
  body_geom(body_kind, body_nv, body_xy, body_radius, &rb);
  const bool small = E <= 4 && (body_kind == RDA_OBS_CIRCLE || body_nv <= 4);
  std::vector<int> idx(count);
  for (int j = 0; j < count; ++j) {
    idx[j] = j;
    keys[j] = exact_key(rb, small, entry(j, T, kind, nv, xy, radius, vel, planned, plan_xy), tv, T, dt, E, nom, ref);
  }
  std::stable_sort(idx.begin(), idx.end(), [&](int a, int b) { return keys[a] < keys[b]; });
  const int Tc = tv ? T + 1 : 1;
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
    const RawShape s = entry(src, T, kind, nv, xy, radius, vel, planned, plan_xy);
    for (int t = 0; t < Tc; ++t) stage_rows(s, t, dt, E, A + (size_t)t * E * 2, b + (size_t)t * E);
  }
  return count;
}

// The kernel's two lower bounds of every entry: lb_disc [count] (one disc of the whole horizon) and lb_pose [count]
// (every pose on its own).
extern "C" void shim_horizon_bounds(int count, int T, int E, double dt, int tv, const float* nom, const float* ref,
                                    int body_kind, int body_nv, const float* body_xy, float body_radius,
                                    const int* kind, const int* nv, const float* xy, const float* radius,
                                    const float* vel, const int* planned, const float* plan_xy, double* lb_disc,
                                    double* lb_pose) {
  RobotGeom rb;
  body_geom(body_kind, body_nv, body_xy, body_radius, &rb);
  const double reach = body_reach(rb);
  double hx, hy, hr;
  const bool any = horizon_disc(nom, ref, T, &hx, &hy, &hr) > 0;
  for (int j = 0; j < count; ++j) {
    const RawShape s = entry(j, T, kind, nv, xy, radius, vel, planned, plan_xy);
    lb_disc[j] = any ? horizon_disc_bound(s, tv, T, dt, E, hx, hy, hr, reach) : INFINITY;
    lb_pose[j] = horizon_bound(s, tv, T, dt, E, nom, ref, reach, -INFINITY);
  }
}

// How many entries the kernel's scan evaluates exactly: tiles of `tile` entries in list order, every entry until N are
// kept, then those whose bounds are below the N-th kept key at the start of their tile.
extern "C" int shim_horizon_exact_count(int count, int N, int T, int E, double dt, int tv, int tile, const float* nom,
                                        const float* ref, int body_kind, int body_nv, const float* body_xy,
                                        float body_radius, const int* kind, const int* nv, const float* xy,
                                        const float* radius, const float* vel, const int* planned,
                                        const float* plan_xy) {
  RobotGeom rb;
  body_geom(body_kind, body_nv, body_xy, body_radius, &rb);
  const bool small = E <= 4 && (body_kind == RDA_OBS_CIRCLE || body_nv <= 4);
  const double reach = body_reach(rb);
  double hx, hy, hr;
  const bool any = horizon_disc(nom, ref, T, &hx, &hy, &hr) > 0;
  std::vector<double> kept;                            // the N smallest keys so far, ascending
  int exact = 0;
  for (int base = 0; base < count; base += tile) {
    const bool full = (int)kept.size() >= N;
    const double thr = full ? kept[N - 1] : INFINITY;
    for (int j = base; j < count && j < base + tile; ++j) {
      const RawShape s = entry(j, T, kind, nv, xy, radius, vel, planned, plan_xy);
      if (full && (!any || !(horizon_disc_bound(s, tv, T, dt, E, hx, hy, hr, reach) < thr) ||
                   !(horizon_bound(s, tv, T, dt, E, nom, ref, reach, thr) < thr)))
        continue;
      ++exact;
      kept.push_back(exact_key(rb, small, s, tv, T, dt, E, nom, ref));
    }
    std::stable_sort(kept.begin(), kept.end());
    if ((int)kept.size() > N) kept.resize(N);
  }
  return exact;
}
