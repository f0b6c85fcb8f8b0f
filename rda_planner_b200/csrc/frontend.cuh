// frontend.cuh — the steps either side of the solver, batched (SURVEY.md §8 rows f1-f3).
//
//   pre_process_one     MPC.pre_process / closest_point / inter_point / range_cir_seg / wraptopi and the
//                       motion_predict_model_* rollouts          (mpc.py:251-291, 293-336, 338-438)
//   obstacle_key, obstacle_rows
//                       MPC.convert_rda_obstacle / rda_obs_distance / convert_inequal_circle /
//                       convert_inequal_polygon / gen_inequal_global / is_convex_and_ordered
//                       (mpc.py:189-218, 440-549) followed by RDA_solver.assign_obstacle_parameter
//                       (rda_solver.py:483-526: truncate to N, pad by repeating the last, zero rows to E)
//   motion_predict      one step of the nonlinear model (mpc.py:293-336)
//
// Same host/device convention as the solver cores: plain functions compiled by nvcc for the kernels
// (rda_frontend.cu) and by g++ for the CPU tests, which check them against values produced by
// executing the reference's own numpy helpers (tests/golden/boundary_golden.json).
// Arithmetic is double (the reference's), inputs and outputs are the float32 arrays of the C ABI.
#pragma once
#include <math.h>
#include "rda_hd.h"

namespace rda {

#define RDA_PI_D 3.14159265358979323846

// mpc.py:431-438 — whole turns, closed interval [-pi, pi]
RDA_HD double wrap_to_pi_d(double a) {
  if (!(a == a) || a > 1e9 || a < -1e9) return a;
  while (a > RDA_PI_D) a -= 2 * RDA_PI_D;
  while (a < -RDA_PI_D) a += 2 * RDA_PI_D;
  return a;
}

// mpc.py:293-336
RDA_HD void motion_predict(int dynamics, double dt, double L, const double s[3], double v0, double v1,
                                  double out[3]) {
  if (dynamics == RDA_DYN_ACKER) {
    out[0] = s[0] + v0 * cos(s[2]) * dt; out[1] = s[1] + v0 * sin(s[2]) * dt; out[2] = s[2] + v0 * tan(v1) / L * dt;
  } else if (dynamics == RDA_DYN_DIFF) {
    out[0] = s[0] + v0 * cos(s[2]) * dt; out[1] = s[1] + v0 * sin(s[2]) * dt; out[2] = s[2] + v1 * dt;
  } else {
    out[0] = s[0] + dt * (v0 * cos(v1)); out[1] = s[1] + dt * (v0 * sin(v1)); out[2] = s[2];
  }
}

// far intersection of the circle (c, r) with the segment p0 -> p1 (mpc.py:385-423); false: none
RDA_HD bool seg_circle_exit_d(double cx, double cy, double r, double p0x, double p0y, double p1x, double p1y,
                                     double* hx, double* hy) {
  const double dx = p1x - p0x, dy = p1y - p0y;
  if (sqrt(dx * dx + dy * dy) == 0) return false;
  const double fx = p0x - cx, fy = p0y - cy;
  const double qa = dx * dx + dy * dy;
  const double qb = 2 * fx * dx + 2 * fy * dy;
  const double qc = fx * fx + fy * fy - r * r;
  const double disc = qb * qb - 4 * qa * qc;
  if (disc < 0) return false;
  const double tf = (-qb + sqrt(disc)) / (2 * qa);
  if (tf >= 0 && tf <= 1) { *hx = p0x + tf * dx; *hy = p0y + tf * dy; return true; }
  return false;
}

// One instance of MPC.pre_process.  path [P][3] (x, y, heading), vel [2][T] (row stride T),
// nom_s / ref_s [3][T+1] (row stride T+1).  Returns the index of the closest waypoint (the new
// cur_index, mpc.py:155).  Reproduced on purpose:
//  * the arc-length stepping continues from `start_index`, not from the closest waypoint (:276-283);
//  * the first reference point is the closest waypoint itself, heading not unwrapped (:258-262);
//  * once the path is exhausted every later reference point IS the last waypoint, whose heading the
//    reference overwrites in place (:285-286, :379-383): all those columns (and column 0 when the
//    closest waypoint is the last one) end up with the heading written by the final step.
RDA_HD int pre_process_one(int dynamics, int T, double dt, double L, const float* state, const float* vel,
                                  double ref_speed, const float* path, int P, int start_index, double threshold,
                                  int ind_range, float* nom_s, float* ref_s) {
  const int S = T + 1;
  // closest_point (mpc.py:338-353)
  double best = 1e300;
  int near = start_index;
  for (int k = 0; k < ind_range; ++k) {
    const int idx = start_index + k;
    if (idx >= P) break;
    const double ex = (double)state[0] - path[3 * idx], ey = (double)state[1] - path[3 * idx + 1];
    const double dk = sqrt(ex * ex + ey * ey);
    if (dk < best) {
      best = dk; near = idx;
      if (dk < threshold) break;
    }
  }
  double cur[3] = {state[0], state[1], state[2]};
  double ref[3] = {0, 0, 0};
  if (P > 0) { const int n = near < P ? near : P - 1; ref[0] = path[3 * n]; ref[1] = path[3 * n + 1]; ref[2] = path[3 * n + 2]; }
  for (int r = 0; r < 3; ++r) { nom_s[r * S] = (float)cur[r]; ref_s[r * S] = (float)ref[r]; }
  double end_h = P > 0 ? (double)path[3 * (P - 1) + 2] : 0.0;     // heading of the last waypoint (mutable)
  int first_alias = S;                                               // first column that is the last waypoint
  int ci = start_index;
  const double step = ref_speed * dt;
  for (int i = 0; i < T; ++i) {
    double nxt[3];
    motion_predict(dynamics, dt, L, cur, vel[i], vel[T + i], nxt);
    cur[0] = nxt[0]; cur[1] = nxt[1]; cur[2] = nxt[2];
    // inter_point (mpc.py:355-383)
    bool found = false;
    while (ci + 1 <= P - 1) {
      const float* a = path + 3 * ci;
      const float* c = path + 3 * (ci + 1);
      double hx, hy;
      if (!seg_circle_exit_d(ref[0], ref[1], step, a[0], a[1], c[0], c[1], &hx, &hy)) { ++ci; continue; }
      const double turn = wrap_to_pi_d((double)c[2] - (double)a[2]);
      ref[0] = hx; ref[1] = hy; ref[2] = wrap_to_pi_d((double)a[2] + turn / 2);
      found = true;
      break;
    }
    if (!found && P > 0) {
      end_h = wrap_to_pi_d(end_h);
      ref[0] = path[3 * (P - 1)]; ref[1] = path[3 * (P - 1) + 1]; ref[2] = end_h;
      if (first_alias == S) first_alias = i + 1;
    }
    ref[2] = cur[2] + wrap_to_pi_d(ref[2] - cur[2]);
    if (!found) end_h = ref[2];
    for (int r = 0; r < 3; ++r) { nom_s[r * S + i + 1] = (float)cur[r]; ref_s[r * S + i + 1] = (float)ref[r]; }
  }
  for (int j = first_alias; j < S; ++j) ref_s[2 * S + j] = (float)end_h;
  if (P > 0 && near == P - 1) ref_s[2 * S] = (float)end_h;
  return near;
}

// A robot without a reference path: the nominal rollout of pre_process_one, and a reference that holds the robot's
// current state in every column.
RDA_HD void hold_state_one(int dynamics, int T, double dt, double L, const float* state, const float* vel,
                           float* nom_s, float* ref_s) {
  const int S = T + 1;
  double cur[3] = {state[0], state[1], state[2]};
  for (int r = 0; r < 3; ++r) {
    nom_s[r * S] = state[r];
    for (int j = 0; j < S; ++j) ref_s[r * S + j] = state[r];
  }
  for (int i = 0; i < T; ++i) {
    double nxt[3];
    motion_predict(dynamics, dt, L, cur, vel[i], vel[T + i], nxt);
    for (int r = 0; r < 3; ++r) { cur[r] = nxt[r]; nom_s[r * S + i + 1] = (float)cur[r]; }
  }
}

// ---- reference path sets ----------------------------------------------------------------------
// W paths in one flat waypoint list path [P][3], each cut into single-gear curves (split_path, mpc.py:232-249):
// path w is curves [path_curve[w], path_curve[w+1]), curve c is waypoints [curve_start[c], curve_start[c+1]) with
// gear curve_gear[c] (+1 / -1).  NULL tables describe a single path: path_curve NULL = one path of n_curves
// curves, curve_start NULL = one curve of P waypoints, curve_gear NULL = gear +1.
struct PathCurve {
  int index;   // curve index relative to the path, clamped into [0, count)
  int count;   // curves of the path
  int first;   // first waypoint of the curve in the flat list
  int len;     // waypoints of the curve
  int gear;    // +1 forward, -1 reverse
};

// The curve a robot on path w (0 <= w < W) with relative curve index c follows.  Out-of-range c is clamped to the
// path's first or last curve.  Returns false for a path without curves.
RDA_HD bool resolve_curve(int w, int c, const int* path_curve, int n_curves, const int* curve_start, int P,
                          const int* curve_gear, PathCurve* out) {
  const int c0 = path_curve ? path_curve[w] : 0;
  const int nc = path_curve ? path_curve[w + 1] - c0 : n_curves;
  if (nc < 1) return false;
  c = c < 0 ? 0 : (c >= nc ? nc - 1 : c);
  const int g = c0 + c;
  out->index = c;
  out->count = nc;
  out->first = curve_start ? curve_start[g] : 0;
  out->len = curve_start ? curve_start[g + 1] - out->first : P;
  out->gear = curve_gear ? curve_gear[g] : 1;
  return true;
}

// ---- obstacles ------------------------------------------------------------------------------
// One raw shape: kind RDA_OBS_POLYGON (nv vertices xy[2 i], xy[2 i + 1]) or RDA_OBS_CIRCLE (centre xy[0..1],
// radius), constant velocity (vx, vy).

// sort key of convert_rda_obstacle(obstacle_order=True): mpc.py:210-218
RDA_HD double obstacle_key(int kind, int nv, const float* xy, double sx, double sy) {
  if (kind == RDA_OBS_CIRCLE) {
    const double dx = sx - xy[0], dy = sy - xy[1];
    return sqrt(dx * dx + dy * dy);
  }
  double best = 1e300;
  for (int i = 0; i < nv; ++i) {
    const double dx = sx - xy[2 * i], dy = sy - xy[2 * i + 1];
    const double d = sqrt(dx * dx + dy * dy);
    if (d < best) best = d;
  }
  return best;
}

// rows (A [E][2], b [E]) of one shape at stage t (mpc.py:440-510): the shape is translated by
// velocity * (t * dt) when it moves faster than 0.01, vertices are put in counter-clockwise order
// (mpc.py:480-486, 518-549), row i is the outward normal of edge i -> i+1; rows >= nv are zero
// (rda_solver.py:509-510, 523-524).
RDA_HD void obstacle_rows(int kind, int nv, const float* xy, double radius, double vx, double vy, int t, double dt,
                                 int E, float* A, float* b) {
  for (int i = 0; i < E; ++i) { A[2 * i] = 0.f; A[2 * i + 1] = 0.f; b[i] = 0.f; }
  const bool moving = sqrt(vx * vx + vy * vy) > 0.01;
  const double ox = moving ? vx * (t * dt) : 0.0, oy = moving ? vy * (t * dt) : 0.0;
  if (kind == RDA_OBS_CIRCLE) {
    if (E < 3) return;
    A[0] = 1.f; A[3] = 1.f;
    b[0] = (float)((double)xy[0] + ox); b[1] = (float)((double)xy[1] + oy); b[2] = (float)(-radius);
    return;
  }
  if (nv < 3 || nv > E) return;
  double px[RDA_MAX_EDGE], py[RDA_MAX_EDGE];
  for (int i = 0; i < nv; ++i) { px[i] = (double)xy[2 * i] + ox; py[i] = (double)xy[2 * i + 1] + oy; }
  // orientation: sign of the first non-zero turn; a later turn of the other sign means "not convex",
  // which the reference only warns about and then leaves the order alone (mpc.py:480-486, 518-549)
  int sign = 0;
  bool convex = true;
  for (int i = 0; i < nv; ++i) {
    const int j = (i + 1) % nv, k = (i + 2) % nv;
    const double cr = (px[j] - px[i]) * (py[k] - py[i]) - (py[j] - py[i]) * (px[k] - px[i]);
    if (cr == 0) continue;
    if (sign == 0) sign = cr > 0 ? 1 : -1;
    else if ((cr > 0) != (sign > 0)) convex = false;
  }
  if (!convex) sign = 0;
  if (sign < 0) {
    for (int i = 0; i < nv / 2; ++i) {
      const double tx = px[i], ty = py[i];
      px[i] = px[nv - 1 - i]; py[i] = py[nv - 1 - i];
      px[nv - 1 - i] = tx; py[nv - 1 - i] = ty;
    }
  }
  for (int i = 0; i < nv; ++i) {
    const int j = (i + 1) % nv;
    const double ex = px[j] - px[i], ey = py[j] - py[i];
    const double a0 = ey, a1 = -ex;
    A[2 * i] = (float)a0; A[2 * i + 1] = (float)a1;
    b[i] = (float)(a0 * px[i] + a1 * py[i]);
  }
}

// The body (body frame: polygon vertices body_xy [nv][2], counter-clockwise, or the disc centre body_xy[0..1]) placed
// at the pose (px, py, th): p + R(th) v in double, rounded to float32.  Entries of xy beyond the shape's own are zero,
// as the host packing leaves them.
RDA_HD void place_body(int body_kind, int body_nv, const float* body_xy, double px, double py, double th, float* xy) {
  const double c = cos(th), s = sin(th);
  const int n = body_kind == RDA_OBS_CIRCLE ? 1 : body_nv;
  for (int i = 0; i < RDA_MAX_EDGE; ++i) {
    if (i < n) {
      const double bx = body_xy[2 * i], by = body_xy[2 * i + 1];
      xy[2 * i] = (float)(px + (c * bx - s * by));
      xy[2 * i + 1] = (float)(py + (s * bx + c * by));
    } else {
      xy[2 * i] = 0.f; xy[2 * i + 1] = 0.f;
    }
  }
}

// A robot of a fleet as one raw shape for its map-mates: the body (body_radius: the disc's) placed at the pose `state`
// (place_body), moving with the world-frame velocity of its control (v0, v1) as motion_predict moves it: v0 (cos, sin)
// of the heading for acker / diff, of the control angle v1 for omni (mpc.py:293-336).
RDA_HD void fleet_shape(int dynamics, int body_kind, int body_nv, const float* body_xy, float body_radius,
                        const float* state, double v0, double v1, int* kind, int* nv, float* xy, float* radius,
                        float* vel) {
  const double th = state[2];
  place_body(body_kind, body_nv, body_xy, state[0], state[1], th, xy);
  *kind = body_kind;
  *nv = body_kind == RDA_OBS_CIRCLE ? 0 : body_nv;
  *radius = body_kind == RDA_OBS_CIRCLE ? body_radius : 0.f;
  const double dir = dynamics == RDA_DYN_OMNI ? v1 : th;
  vel[0] = (float)(v0 * cos(dir));
  vel[1] = (float)(v0 * sin(dir));
}

// A robot of a fleet predicted along its plan, as the stage-t shapes of a time-varying obstacle for its map-mates:
// q(0) = state, q(t+1) = motion_predict(q(t), u[:, c]) with c = min(t + 1, T - 1) for t = 0..T-1, in double (column 0
// of u [2][T] (row stride T) is the control the robot has just applied, so its plan goes on from column 1 and holds its
// last column); stage t is the body placed at q(t) (place_body), written to plan_xy [T+1][RDA_MAX_EDGE][2].  Stage 0 is
// bit for bit the xy of fleet_shape at the same state.  On the device plan_xy must be 16-byte aligned: each stage is
// stored as four 16-byte vectors.
RDA_HD void fleet_plan(int dynamics, double dt, double L, int body_kind, int body_nv, const float* body_xy,
                       const float* state, const float* u, int T, float* plan_xy) {
  double q[3] = {state[0], state[1], state[2]};
  for (int t = 0;; ++t) {
    float xy[2 * RDA_MAX_EDGE];
    place_body(body_kind, body_nv, body_xy, q[0], q[1], q[2], xy);
    float* out = plan_xy + (size_t)t * 2 * RDA_MAX_EDGE;
#ifdef __CUDA_ARCH__
    for (int i = 0; i < 2 * RDA_MAX_EDGE; i += 4)
      *reinterpret_cast<float4*>(out + i) = make_float4(xy[i], xy[i + 1], xy[i + 2], xy[i + 3]);
#else
    for (int i = 0; i < 2 * RDA_MAX_EDGE; ++i) out[i] = xy[i];
#endif
    if (t == T) break;
    const int c = t + 1 < T ? t + 1 : T - 1;
    double nxt[3];
    motion_predict(dynamics, dt, L, q, u[c], u[T + c], nxt);
    q[0] = nxt[0]; q[1] = nxt[1]; q[2] = nxt[2];
  }
}

// the order of the stable sort by key: ties go to the lower list index
RDA_HD bool obstacle_before(double ka, int ia, double kb, int ib) { return ka < kb || (ka == kb && ia < ib); }

// Which raw shape fills slot n of an instance (stable ascending order of the keys when `order`,
// otherwise list order; slots beyond the list repeat its last element): returns -1 for an empty list.
// keys[] is scratch of at least `count` doubles already filled by the caller when order != 0.
RDA_HD int obstacle_slot_source(int n, int count, int order, const double* keys) {
  if (count <= 0) return -1;
  const int want = n < count ? n : count - 1;
  if (!order) return want;
  // rank selection: the shape with exactly `want` shapes before it in stable order
  for (int i = 0; i < count; ++i) {
    int before = 0;
    for (int j = 0; j < count; ++j)
      if (keys[j] < keys[i] || (keys[j] == keys[i] && j < i)) ++before;
    if (before == want) return i;
  }
  return want;
}

}  // namespace rda
