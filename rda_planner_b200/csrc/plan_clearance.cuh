// plan_clearance.cuh — signed distance between the robot body at a planned pose and one obstacle (rda_plan_clearance).
//
//   sd(P, Q) = max over unit w of ( min_{x in P} w.x - max_{y in Q} w.y )
//
// the Euclidean distance of disjoint sets, minus the penetration depth (shortest separating translation) of overlapping
// ones.  P is the body of RobotGeom placed at the pose (x, y, heading) of ONE plan column, Q the obstacle's rows as the
// cell kernels read them: polygon rows closed counter-clockwise, row i joining vertices i and i+1, the first zero-norm row
// ending the polygon; a disc as rows [[1,0],[0,1],[0,0]], b = (cx, cy, -r).  float32 in and out, float64 inside, in
// coordinates relative to the pose (as frontend.cuh).  DESIGN.md §9.
//
// The geometry goes into a CellGeom<double> as cell_front builds it (same vertex construction), but by a routine of its
// own: its loops run to the compile-time caps EC / RC (obstacle rows, body vertices) with constant indices only, so
// that the whole geometry stays in registers (cell_front's loops to runtime bounds would put it in local memory), and
// the body's edge normals are formed from its float32 vertices in float64, so that every separating-axis gap is exact
// for the polygon the kernels hold (cell_front rotates the float32 normals of RobotGeom).  Sharing cell_front's code
// would change the registers of every cell pass; DESIGN.md §9.
#pragma once
#include "rda_hd.h"
#include "cell_solver.cuh"

namespace rda {

// squared distance of q to the segment a -> a + e
RDA_HD double clear_seg_d2(double qx, double qy, double ax, double ay, double ex, double ey) {
  const double rx = qx - ax, ry = qy - ay, e2 = ex * ex + ey * ey;
  const double t = e2 > 0 ? rclamp((rx * ex + ry * ey) / e2, 0.0, 1.0) : 0.0;
  const double dx = rx - t * ex, dy = ry - t * ey;
  return dx * dx + dy * dy;
}

// Signed distance of the point q to a convex polygon of n <= C vertices (vx, vy) with unit outward normals (nx, ny) of
// the edges i -> i+1: the largest edge gap when q is inside (<= 0), else the distance to the nearest edge.
template <int C>
RDA_HD double clear_point_polygon(double qx, double qy, int n, const double* vx, const double* vy, const double* nx,
                                  const double* ny) {
  double gap = -INFINITY;
#pragma unroll
  for (int i = 0; i < C; ++i)
    if (i < n) gap = rmax(gap, nx[i] * (qx - vx[i]) + ny[i] * (qy - vy[i]));
  if (!(gap > 0)) return gap;
  double d2 = INFINITY;
#pragma unroll
  for (int i = 0; i < C; ++i) {
    if (!(i < n)) continue;
    const int k = i + 1 < C ? i + 1 : 0;
    const double wx = i + 1 < n ? vx[k] : vx[0], wy = i + 1 < n ? vy[k] : vy[0];
    d2 = rmin(d2, clear_seg_d2(qx, qy, vx[i], vy[i], wx - vx[i], wy - vy[i]));
  }
  return sqrt(d2);
}

// sd of the body rb at pose (px, py, th) and the obstacle (kind, E rows A [E][2], b [E]); requires E <= EC, rb.R <= RC.
// A polygon obstacle with fewer than three rows has no extent: +inf.
template <int EC, int RC>
RDA_HD double plan_clearance_cell(const RobotGeom& rb, int kind, int E, const float* A, const float* b, float px, float py,
                                  float th) {
  const double c = cos((double)th), s = sin((double)th), pxd = px, pyd = py;
  CellGeom<double> g;     // only the first EC / RC entries are touched, with constant indices: registers
  // ---- obstacle, relative to the pose ----
  int ne = 0;
  if (kind == RDA_OBS_CIRCLE) {
    g.cx = (double)b[0] - pxd;
    g.cy = (double)b[1] - pyd;
    g.rad = -(double)b[2];
  } else {
    double brel[EC];
    double lnx = 0, lny = 0, lb = 0;         // the last row, which closes the polygon at vertex 0
    bool live = true;
#pragma unroll
    for (int i = 0; i < EC; ++i) {
      if (!(i < E && live)) continue;
      const double ax = A[2 * i], ay = A[2 * i + 1], n2 = ax * ax + ay * ay;
      if (!(n2 > 0)) { live = false; continue; }
      const double inv = 1.0 / sqrt(n2);
      g.nx[i] = ax * inv;
      g.ny[i] = ay * inv;
      brel[i] = ((double)b[i] - ax * pxd - ay * pyd) * inv;
      lnx = g.nx[i]; lny = g.ny[i]; lb = brel[i];
      ne = i + 1;
    }
    if (ne < 3) return INFINITY;
    // vertex i joins rows i-1 and i (cell_front)
#pragma unroll
    for (int i = 0; i < EC; ++i) {
      if (!(i < ne)) continue;
      const int a = i > 0 ? i - 1 : 0;
      const double pnx = i > 0 ? g.nx[a] : lnx, pny = i > 0 ? g.ny[a] : lny, pb = i > 0 ? brel[a] : lb;
      const double inv = 1.0 / (pnx * g.ny[i] - pny * g.nx[i]);
      g.vx[i] = (pb * g.ny[i] - brel[i] * pny) * inv;
      g.vy[i] = (pnx * brel[i] - g.nx[i] * pb) * inv;
    }
  }
  // ---- disc body: a point problem ----
  if (rb.disc) {
    const double qx = c * (double)rb.cx - s * (double)rb.cy, qy = s * (double)rb.cx + c * (double)rb.cy;
    if (kind == RDA_OBS_CIRCLE) return sqrt((qx - g.cx) * (qx - g.cx) + (qy - g.cy) * (qy - g.cy)) - g.rad - (double)rb.rad;
    return clear_point_polygon<EC>(qx, qy, ne, g.vx, g.vy, g.nx, g.ny) - (double)rb.rad;
  }
  // ---- polygon body: vertices rotated into the world frame, outward edge normals from them ----
  const int R = rb.R;
#pragma unroll
  for (int j = 0; j < RC; ++j) {
    if (!(j < R)) continue;
    const double yx = rb.yx[j], yy = rb.yy[j];
    g.yx[j] = c * yx - s * yy;
    g.yy[j] = s * yx + c * yy;
  }
#pragma unroll
  for (int j = 0; j < RC; ++j) {
    if (!(j < R)) continue;
    const int k = j + 1 < RC ? j + 1 : 0;
    const double fx = (j + 1 < R ? g.yx[k] : g.yx[0]) - g.yx[j], fy = (j + 1 < R ? g.yy[k] : g.yy[0]) - g.yy[j];
    const double inv = 1.0 / sqrt(fx * fx + fy * fy);
    g.mx[j] = fy * inv;
    g.my[j] = -fx * inv;
  }
  if (kind == RDA_OBS_CIRCLE)
    return clear_point_polygon<RC>(g.cx, g.cy, R, g.yx, g.yy, g.mx, g.my) - g.rad;
  // ---- two polygons: separating-axis gaps over the E + R edge normals ----
  double gap = -INFINITY;
#pragma unroll
  for (int i = 0; i < EC; ++i) {
    if (!(i < ne)) continue;
    double m = INFINITY;
#pragma unroll
    for (int j = 0; j < RC; ++j)
      if (j < R) m = rmin(m, g.nx[i] * (g.yx[j] - g.vx[i]) + g.ny[i] * (g.yy[j] - g.vy[i]));
    gap = rmax(gap, m);
  }
#pragma unroll
  for (int j = 0; j < RC; ++j) {
    if (!(j < R)) continue;
    double m = INFINITY;
#pragma unroll
    for (int i = 0; i < EC; ++i)
      if (i < ne) m = rmin(m, g.mx[j] * (g.vx[i] - g.yx[j]) + g.my[j] * (g.vy[i] - g.yy[j]));
    gap = rmax(gap, m);
  }
  // overlapping (or touching): the largest gap is minus the penetration depth
  if (!(gap > 0)) return gap;
  // disjoint: the nearest pair has a vertex of one polygon on an edge of the other
  double d2 = INFINITY;
#pragma unroll
  for (int i = 0; i < EC; ++i) {
    if (!(i < ne)) continue;
    const int k = i + 1 < EC ? i + 1 : 0;
    const double ex = (i + 1 < ne ? g.vx[k] : g.vx[0]) - g.vx[i], ey = (i + 1 < ne ? g.vy[k] : g.vy[0]) - g.vy[i];
#pragma unroll
    for (int j = 0; j < RC; ++j)
      if (j < R) d2 = rmin(d2, clear_seg_d2(g.yx[j], g.yy[j], g.vx[i], g.vy[i], ex, ey));
  }
#pragma unroll
  for (int j = 0; j < RC; ++j) {
    if (!(j < R)) continue;
    const int k = j + 1 < RC ? j + 1 : 0;
    const double fx = (j + 1 < R ? g.yx[k] : g.yx[0]) - g.yx[j], fy = (j + 1 < R ? g.yy[k] : g.yy[0]) - g.yy[j];
#pragma unroll
    for (int i = 0; i < EC; ++i)
      if (i < ne) d2 = rmin(d2, clear_seg_d2(g.vx[i], g.vy[i], g.yx[j], g.yy[j], fx, fy));
  }
  return sqrt(d2);
}

}  // namespace rda
