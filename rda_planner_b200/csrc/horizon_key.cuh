// horizon_key.cuh — the sort key of obstacle_order='horizon' (rda_convert_world_obstacles_horizon) and the lower bound
// that lets the kernel skip it.  DESIGN.md §7.3.
//
//   key(j) = min over the poses q in { nom_s[:, t], ref_s[:, t] : t = 0..T } of sd(body at q, shape j at stage t)
//
// "Shape j at stage t" is exactly the rows the conversion writes for it (obstacle_rows of copy t when time-varying,
// copy 0 otherwise; a map-mate along its plan: its plan_xy[t] shape standing), and sd is plan_clearance_cell, the core
// of rda_plan_clearance.  A pose column with a non-finite entry takes no part; without any the key is +inf.
//
// The bound: the body lies within `reach` of its pose, the stage shape's rows within a disc (shape_disc), and sd is
// monotone under inclusion, so sd >= |c - p| - r - reach.  The disc covers the polygon the float32 rows describe, not
// only the raw vertices: rounding a row to float32 moves its vertices by up to about 5 * 2^-24 |v| / sin(turn), and the
// disc's radius carries 16 * 2^-24 |v|max / sin(smallest turn).  Shapes where that is not a small, safe number (a turn
// below 1e-6, an edge shorter than 1e3 margins, a non-convex or unordered polygon, whose rows are no convex polygon, a
// non-finite vertex, centre or radius) get an infinite disc and are never pruned, and a bound that comes out NaN is -inf.  disc_bound also subtracts 1e-9 of the magnitudes involved for the float64
// rounding of the exact key.
//
// Plain functions compiled by nvcc for the kernel (rda_frontend.cu) and by g++ for the CPU twin
// (tests/cpu_twin/horizon_select.cpp), which evaluate the same arithmetic.
#pragma once
#include <math.h>
#include "rda_hd.h"
#include "frontend.cuh"
#include "plan_clearance.cuh"

namespace rda {

// One raw shape of a robot's list: a world shape or a map-mate moving at (vx, vy), or a map-mate along its plan
// (plan: [T+1][RDA_MAX_EDGE][2], its stage-t shape standing).
struct RawShape {
  int kind, nv;
  const float* xy;
  double radius, vx, vy;
  const float* plan;
};

// the stage-t rows of the shape, as the conversion writes them (A [E][2], b [E])
RDA_HD void stage_rows(const RawShape& s, int t, double dt, int E, float* A, float* b) {
  if (s.plan)
    obstacle_rows(s.kind, s.nv, s.plan + (size_t)t * 2 * RDA_MAX_EDGE, s.radius, 0.0, 0.0, t, dt, E, A, b);
  else
    obstacle_rows(s.kind, s.nv, s.xy, s.radius, s.vx, s.vy, t, dt, E, A, b);
}

// The robot body of the robot_body format (polygon: nv counter-clockwise vertices xy [nv][2]; disc: centre xy[0..1],
// radius) as plan_clearance_cell reads it.
RDA_HD void body_geom(int kind, int nv, const float* xy, float radius, RobotGeom* g) {
  const bool disc = kind == RDA_OBS_CIRCLE;
  g->disc = disc ? 1 : 0;
  g->R = disc ? 3 : nv;
  g->cx = disc ? xy[0] : 0.f;
  g->cy = disc ? xy[1] : 0.f;
  g->rad = disc ? radius : 0.f;
  for (int j = 0; j < RDA_MAX_ROBOT_EDGE; ++j) {
    const bool v = !disc && j < nv;
    g->yx[j] = v ? xy[2 * j] : 0.f;
    g->yy[j] = v ? xy[2 * j + 1] : 0.f;
    g->nx[j] = g->ny[j] = g->h[j] = 0.f;
    g->gnorm[j] = 1.f;
  }
}

// radius of the body about its pose
RDA_HD double body_reach(const RobotGeom& g) {
  if (g.disc) return sqrt((double)g.cx * g.cx + (double)g.cy * g.cy) + (double)g.rad;
  double r = 0;
  for (int j = 0; j < g.R && j < RDA_MAX_ROBOT_EDGE; ++j) r = rmax(r, sqrt((double)g.yx[j] * g.yx[j] + (double)g.yy[j] * g.yy[j]));
  return r;
}

// A disc (cx, cy, r) that holds the shape whose rows obstacle_rows builds from (kind, nv, xy, radius) moved by at most
// `spread` (the rounding margin grows with the coordinates).  r = -inf: the shape has no rows (its sd is +inf);
// r = +inf: no safe disc.
struct ShapeDisc {
  double cx, cy, r;
};

RDA_HD ShapeDisc shape_disc(int kind, int nv, const float* xy, double radius, int E, double spread) {
  const double u = 1.0 / 16777216.0;                   // 2^-24, float32's unit roundoff
  if (kind == RDA_OBS_CIRCLE) {                        // rows b = (cx, cy, -r), the centre rounded to float32
    const double cx = xy[0], cy = xy[1];
    if (!(finite_(cx) && finite_(cy) && finite_(radius))) return {0.0, 0.0, INFINITY};
    return {cx, cy, radius + 2 * u * (fabs(cx) + fabs(cy) + 2 * spread)};
  }
  if (nv < 3 || nv > E) return {0.0, 0.0, -INFINITY};
  for (int i = 0; i < 2 * nv; ++i)                      // a non-finite vertex: no safe disc (rmin / rmax drop NaN)
    if (!finite_(xy[i])) return {0.0, 0.0, INFINITY};
  double lx = INFINITY, hx = -INFINITY, ly = INFINITY, hy = -INFINITY;
  for (int i = 0; i < nv; ++i) {
    lx = rmin(lx, (double)xy[2 * i]); hx = rmax(hx, (double)xy[2 * i]);
    ly = rmin(ly, (double)xy[2 * i + 1]); hy = rmax(hy, (double)xy[2 * i + 1]);
  }
  const double cx = 0.5 * (lx + hx), cy = 0.5 * (ly + hy);
  double r0 = 0, vmax = 0, smin = INFINITY, smax = -INFINITY, emin = INFINITY;
  for (int i = 0; i < nv; ++i) {
    const int j = i + 1 < nv ? i + 1 : 0, k = j + 1 < nv ? j + 1 : 0;
    const double x = xy[2 * i], y = xy[2 * i + 1];
    r0 = rmax(r0, sqrt((x - cx) * (x - cx) + (y - cy) * (y - cy)));
    vmax = rmax(vmax, sqrt(x * x + y * y));
    const double e1x = xy[2 * j] - x, e1y = xy[2 * j + 1] - y;
    const double e2x = (double)xy[2 * k] - xy[2 * j], e2y = (double)xy[2 * k + 1] - xy[2 * j + 1];
    const double l1 = sqrt(e1x * e1x + e1y * e1y), l2 = sqrt(e2x * e2x + e2y * e2y);
    const double s = (e1x * e2y - e1y * e2x) / (l1 * l2);    // sine of the turn at vertex j (NaN for a zero edge)
    smin = rmin(smin, s); smax = rmax(smax, s);
    emin = rmin(emin, l1);
  }
  const double turn = smin > 0 ? smin : -smax;         // every turn of one sign (either orientation) or no safe disc
  if (!(turn > 1e-6)) return {cx, cy, INFINITY};
  const double m = 16 * u * (vmax + spread) / turn;
  if (!(emin > 1e3 * m)) return {cx, cy, INFINITY};
  return {cx, cy, r0 + m};
}

// lower bound on the sd of a body within `reach` of (px, py) and a shape within the disc d; -inf where the arithmetic
// gives NaN (a non-finite velocity or body), so that such a shape is never pruned
RDA_HD double disc_bound(double px, double py, double reach, const ShapeDisc& d) {
  if (d.r == -INFINITY) return INFINITY;
  const double dx = px - d.cx, dy = py - d.cy;
  const double v = sqrt(dx * dx + dy * dy) - d.r - reach -
                   1e-9 * (1 + fabs(px) + fabs(py) + fabs(d.cx) + fabs(d.cy) + d.r + reach);
  return v == v ? v : -INFINITY;
}

// offset obstacle_rows applies to a shape moving at (vx, vy) at stage t
RDA_HD void stage_offset(double vx, double vy, int t, double dt, double* ox, double* oy) {
  const bool moving = sqrt(vx * vx + vy * vy) > 0.01;
  *ox = moving ? vx * (t * dt) : 0.0;
  *oy = moving ? vy * (t * dt) : 0.0;
}

RDA_HD bool pose_finite(const float* s, int T1, int t) {
  return finite_(s[t]) && finite_(s[T1 + t]) && finite_(s[2 * T1 + t]);
}

// The robot's horizon as one disc: the centre of the bounding box of its finite poses and their largest distance from
// it.  Returns the number of finite poses (0: no disc).
RDA_HD int horizon_disc(const float* nom, const float* ref, int T, double* cx, double* cy, double* r) {
  const int T1 = T + 1;
  double lx = INFINITY, hx = -INFINITY, ly = INFINITY, hy = -INFINITY;
  int n = 0;
  for (int q = 0; q < 2 * T1; ++q) {
    const float* s = q < T1 ? nom : ref;
    const int t = q < T1 ? q : q - T1;
    if (!pose_finite(s, T1, t)) continue;
    lx = rmin(lx, (double)s[t]); hx = rmax(hx, (double)s[t]);
    ly = rmin(ly, (double)s[T1 + t]); hy = rmax(hy, (double)s[T1 + t]);
    ++n;
  }
  *cx = 0.5 * (lx + hx); *cy = 0.5 * (ly + hy);
  double rr = 0;
  for (int q = 0; q < 2 * T1; ++q) {
    const float* s = q < T1 ? nom : ref;
    const int t = q < T1 ? q : q - T1;
    if (!pose_finite(s, T1, t)) continue;
    const double dx = s[t] - *cx, dy = s[T1 + t] - *cy;
    rr = rmax(rr, sqrt(dx * dx + dy * dy));
  }
  *r = rr;
  return n;
}

// One-disc bound of the whole horizon: the robot's horizon disc (hx, hy, hr) against one disc of the shape over every
// stage.  A map-mate along its plan has none (-inf: decided by horizon_bound).
RDA_HD double horizon_disc_bound(const RawShape& s, int tv, int T, double dt, int E, double hx, double hy, double hr,
                                 double reach) {
  if (s.plan) return -INFINITY;
  double ox = 0, oy = 0;
  if (tv) stage_offset(s.vx, s.vy, T, dt, &ox, &oy);
  const double half = 0.5 * sqrt(ox * ox + oy * oy);
  ShapeDisc d = shape_disc(s.kind, s.nv, s.xy, s.radius, E, 2 * half);
  d.cx += 0.5 * ox; d.cy += 0.5 * oy;
  if (d.r != -INFINITY) d.r += half;
  return disc_bound(hx, hy, hr + reach, d);
}

// Bound of every pose on its own: min over the finite poses of disc_bound(pose, the stage shape's disc).  Stops at
// the first pose whose bound is below `stop` and returns it (stop = -inf: the full minimum); +inf without poses.
RDA_HD double horizon_bound(const RawShape& s, int tv, int T, double dt, int E, const float* nom, const float* ref,
                            double reach, double stop) {
  const int T1 = T + 1;
  double ox = 0, oy = 0;
  if (tv) stage_offset(s.vx, s.vy, T, dt, &ox, &oy);
  const ShapeDisc d0 = s.plan ? ShapeDisc{0.0, 0.0, 0.0} : shape_disc(s.kind, s.nv, s.xy, s.radius, E,
                                                                     sqrt(ox * ox + oy * oy));
  double lb = INFINITY;
  for (int t = 0; t < T1; ++t) {
    const int c = tv ? t : 0;
    ShapeDisc d = d0;
    if (s.plan) {
      d = shape_disc(s.kind, s.nv, s.plan + (size_t)c * 2 * RDA_MAX_EDGE, s.radius, E, 0.0);
    } else {
      stage_offset(s.vx, s.vy, c, dt, &ox, &oy);
      d.cx += ox; d.cy += oy;
    }
    for (int h = 0; h < 2; ++h) {
      const float* p = h ? ref : nom;
      if (!pose_finite(p, T1, t)) continue;
      lb = rmin(lb, disc_bound(p[t], p[T1 + t], reach, d));
      if (lb < stop) return lb;
    }
  }
  return lb;
}

// sd of the body at the pose (px, py, th) and the stage-t shape
template <int EC, int RC>
RDA_HD double horizon_cell(const RobotGeom& rb, const RawShape& s, int t, double dt, int E, float px, float py, float th) {
  float A[2 * RDA_MAX_EDGE], b[RDA_MAX_EDGE];
  stage_rows(s, t, dt, E, A, b);
  return plan_clearance_cell<EC, RC>(rb, s.kind, E, A, b, px, py, th);
}

// The key, serially: pose q = 0..2T+1 is nom column q, then ref column q - (T+1); the kernel spreads q over a warp's
// lanes and takes the same minimum.
template <int EC, int RC>
RDA_HD double horizon_key(const RobotGeom& rb, const RawShape& s, int tv, int T, double dt, int E, const float* nom,
                          const float* ref) {
  const int T1 = T + 1;
  double key = INFINITY;
  for (int q = 0; q < 2 * T1; ++q) {
    const float* p = q < T1 ? nom : ref;
    const int t = q < T1 ? q : q - T1;
    if (!pose_finite(p, T1, t)) continue;
    const double v = horizon_cell<EC, RC>(rb, s, tv ? t : 0, dt, E, p[t], p[T1 + t], p[2 * T1 + t]);
    if (v < key) key = v;
  }
  return key;
}

}  // namespace rda
