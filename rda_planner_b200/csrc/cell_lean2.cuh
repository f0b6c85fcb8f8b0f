// cell_lean2.cuh — coherent first pass of the (lam, mu, z) cell kernel, run by k_cells_coh (rda_kernels.cu).
//
// Same two closed-form cases as cell_lean.cuh (xi = 0, margin >= 0), restricted to clearly separated
// polygon/polygon cells, but without the search: the closest pair of two convex polygons always involves
// the obstacle's support vertex in the separating direction v and the robot's support vertex in -v (or an
// edge adjacent to one of them).  The pair of support-vertex indices found in the previous ADMM iteration
// (`feat`, one byte per cell) is tried first — 4 point-segment tests instead of 32 — and accepted through
// the separating-slab certificate
//       min_j v.Y_j - max_i v.V_i  >=  dist - tol          (always <= dist; equality iff the pair is closest)
// which costs nothing extra because both supports are needed for the multipliers anyway.  Everything that
// depends only on the obstacle (unit normals, vertices, inverse edge lengths, the 2x2 inverses that turn a
// direction into LP-vertex multipliers) is precomputed once per solve (ObstacleGeom, static obstacles);
// the robot-side counterparts are constants of the body (RobotAux).  A miss (pose moved to another feature
// pair, contact, active hinge, discs, time-varying obstacles) returns -1 and the caller runs cell_lean.
// Reference lines: rda_solver.py:389-421, 529-542, 639-690 (as cell_lean.cuh).
#pragma once
#include "rda_hd.h"
#include "cell_lean.cuh"

namespace rda {

#define RDA_FEAT_VALID 0x40

template <int EC>
struct ObstacleGeom {            // one polygon in ABSOLUTE coordinates
  float nx[EC], ny[EC], invn[EC];            // unit outward normal of row i, 1 / |A_i|
  float Vx[EC], Vy[EC];                      // vertex i joins rows i-1 and i
  float ie2[EC];                             // 1 / |V_{i+1} - V_i|^2 (edge i lies on row i)
  float pa0[EC], pa1[EC], pb0[EC], pb1[EC];  // at vertex i: v = alpha n_{i-1} + beta n_i, alpha = v.(pa0,pa1), beta = v.(pb0,pb1)
  int ne;                                    // live rows (0: not a usable polygon)
};

struct RobotAux {                // constants of the body (rows counter-clockwise, vertex j joins rows j-1 and j)
  float if2[RDA_MAX_ROBOT_EDGE];                                   // 1 / |y_{j+1} - y_j|^2
  float pa0[RDA_MAX_ROBOT_EDGE], pa1[RDA_MAX_ROBOT_EDGE];          // g = alpha n_{j-1} + beta n_j at vertex j
  float pb0[RDA_MAX_ROBOT_EDGE], pb1[RDA_MAX_ROBOT_EDGE];
  float ign[RDA_MAX_ROBOT_EDGE];                                   // 1 / |G_j|
};

inline void robot_aux_from_geom(const RobotGeom& rb, RobotAux* ra) {
  const int R = rb.R;
  for (int j = 0; j < RDA_MAX_ROBOT_EDGE; ++j) { ra->if2[j] = 0; ra->pa0[j] = ra->pa1[j] = ra->pb0[j] = ra->pb1[j] = 0; ra->ign[j] = 0; }
  for (int j = 0; j < R; ++j) {
    const int c = (j + 1) % R, a = (j + R - 1) % R;
    const double fx = (double)rb.yx[c] - rb.yx[j], fy = (double)rb.yy[c] - rb.yy[j];
    ra->if2[j] = (float)(1.0 / (fx * fx + fy * fy));
    const double anx = rb.nx[a], any = rb.ny[a], bnx = rb.nx[j], bny = rb.ny[j];
    const double det = anx * bny - any * bnx;
    ra->pa0[j] = (float)(bny / det); ra->pa1[j] = (float)(-bnx / det);
    ra->pb0[j] = (float)(-any / det); ra->pb1[j] = (float)(anx / det);
    ra->ign[j] = (float)(1.0 / rb.gnorm[j]);
  }
}

// Build ObstacleGeom from the padded rows of one polygon (A [E][2], b [E]); double arithmetic, once per solve.
template <int EC>
RDA_HD void obstacle_geometry(int E, const float* A, const float* b, ObstacleGeom<EC>& og) {
  double nx[EC], ny[EC], be[EC];
  int ne = 0;
  for (int i = 0; i < EC; ++i) {
    double ax = 0, ay = 0, bb = 0;
    if (i < E) { ax = A[2 * i]; ay = A[2 * i + 1]; bb = b[i]; }
    const double n2 = ax * ax + ay * ay;
    const bool live = (n2 > 0) && (ne == i);
    const double inv = live ? 1.0 / sqrt(n2) : 0.0;
    nx[i] = ax * inv; ny[i] = ay * inv; be[i] = bb * inv;
    og.nx[i] = (float)nx[i]; og.ny[i] = (float)ny[i]; og.invn[i] = (float)inv;
    og.Vx[i] = og.Vy[i] = og.ie2[i] = og.pa0[i] = og.pa1[i] = og.pb0[i] = og.pb1[i] = 0.f;
    if (live) ne = i + 1;
  }
  og.ne = ne >= 3 ? ne : 0;
  if (ne < 3) return;
  double Vx[EC], Vy[EC];
  bool ok = true;
  for (int i = 0; i < ne; ++i) {
    const int a = (i + ne - 1) % ne;
    const double det = nx[a] * ny[i] - ny[a] * nx[i];
    if (!(det > 1e-9)) ok = false;
    Vx[i] = (be[a] * ny[i] - be[i] * ny[a]) / det;
    Vy[i] = (nx[a] * be[i] - nx[i] * be[a]) / det;
    og.Vx[i] = (float)Vx[i]; og.Vy[i] = (float)Vy[i];
    og.pa0[i] = (float)(ny[i] / det); og.pa1[i] = (float)(-nx[i] / det);
    og.pb0[i] = (float)(-ny[a] / det); og.pb1[i] = (float)(nx[a] / det);
  }
  for (int i = 0; i < ne; ++i) {
    const int c = (i + 1) % ne;
    const double ex = Vx[c] - Vx[i], ey = Vy[c] - Vy[i];
    const double e2 = ex * ex + ey * ey;
    if (!(e2 > 0)) ok = false;
    og.ie2[i] = (float)(1.0 / e2);
  }
  if (!ok) og.ne = 0;
}

// register-array read with a run-time index (select chain; the arrays never leave registers)
template <int K>
RDA_HD float pick(const float (&a)[K], int i) {
  float r = a[0];
#pragma unroll
  for (int k = 1; k < K; ++k) r = (i == k) ? a[k] : r;
  return r;
}

// Returns the new feature byte (>= 0: resolved, outputs valid) or -1 (run cell_lean instead).
template <int EC, int RC>
RDA_HD int cell_lean2(const RobotGeom& rb, const RobotAux& ra, const ObstacleGeom<EC>& og, int feat, float px, float py,
                      float cphi, float sphi, float dbar, float zeta, float theta, LeanOut<EC, RC>& out) {
  const int ne = og.ne, R = rb.R;
  if (!(feat & RDA_FEAT_VALID) || ne < 3) return -1;
  const int ib = (feat >> 3) & 7, jb = feat & 7;
  if (ib >= ne || jb >= R) return -1;
  const float k0 = dbar - zeta;
  // robot vertices in the world frame and obstacle vertices, both relative to p
  float Yx[RC], Yy[RC], Vx[EC], Vy[EC];
#pragma unroll
  for (int j = 0; j < RC; ++j) {
    const float yx = rb.yx[j], yy = rb.yy[j];
    Yx[j] = cphi * yx - sphi * yy; Yy[j] = sphi * yx + cphi * yy;
  }
#pragma unroll
  for (int i = 0; i < EC; ++i) { Vx[i] = og.Vx[i] - px; Vy[i] = og.Vy[i] - py; }
  const int ia = (ib == 0) ? ne - 1 : ib - 1, ic = (ib + 1 == ne) ? 0 : ib + 1;
  const int ja = (jb == 0) ? R - 1 : jb - 1, jc = (jb + 1 == R) ? 0 : jb + 1;
  const float vbx = pick(Vx, ib), vby = pick(Vy, ib), vax = pick(Vx, ia), vay = pick(Vy, ia), vcx = pick(Vx, ic), vcy = pick(Vy, ic);
  const float ybx = pick(Yx, jb), yby = pick(Yy, jb), yax = pick(Yx, ja), yay = pick(Yy, ja), ycx = pick(Yx, jc), ycy = pick(Yy, jc);
  float best, bdx, bdy;
  {  // robot vertex jb against obstacle edges ia (V_ia -> V_ib) and ib (V_ib -> V_ic)
    float ex = vbx - vax, ey = vby - vay, rx = ybx - vax, ry = yby - vay;
    float t = rclamp((rx * ex + ry * ey) * og.ie2[ia], 0.f, 1.f);
    float dx = rx - t * ex, dy = ry - t * ey;
    best = (dx * dx + dy * dy) * ((t > 0.f && t < 1.f) ? 1.f : RDA_ENDPOINT_BIAS); bdx = dx; bdy = dy;
    ex = vcx - vbx; ey = vcy - vby; rx = ybx - vbx; ry = yby - vby;
    t = rclamp((rx * ex + ry * ey) * og.ie2[ib], 0.f, 1.f);
    dx = rx - t * ex; dy = ry - t * ey;
    float d2 = (dx * dx + dy * dy) * ((t > 0.f && t < 1.f) ? 1.f : RDA_ENDPOINT_BIAS);
    if (d2 < best) { best = d2; bdx = dx; bdy = dy; }
    // obstacle vertex ib against robot edges ja (Y_ja -> Y_jb) and jb (Y_jb -> Y_jc)
    float fx = ybx - yax, fy = yby - yay;
    rx = vbx - yax; ry = vby - yay;
    t = rclamp((rx * fx + ry * fy) * ra.if2[ja], 0.f, 1.f);
    dx = -(rx - t * fx); dy = -(ry - t * fy);
    d2 = (dx * dx + dy * dy) * ((t > 0.f && t < 1.f) ? 1.f : RDA_ENDPOINT_BIAS);
    if (d2 < best) { best = d2; bdx = dx; bdy = dy; }
    fx = ycx - ybx; fy = ycy - yby;
    rx = vbx - ybx; ry = vby - yby;
    t = rclamp((rx * fx + ry * fy) * ra.if2[jb], 0.f, 1.f);
    dx = -(rx - t * fx); dy = -(ry - t * fy);
    d2 = (dx * dx + dy * dy) * ((t > 0.f && t < 1.f) ? 1.f : RDA_ENDPOINT_BIAS);
    if (d2 < best) { best = d2; bdx = dx; bdy = dy; }
  }
  const float dist = sqrt_(best);
  if (!(dist > 1e-3f)) return -1;                 // contact or overlap: the full pass decides
  if (dist - k0 < 0.f) return -1;                 // active hinge: searched closed forms
  const float idist = 1.f / dist;
  const float v0 = bdx * idist, v1 = bdy * idist;
  // supports: obstacle in direction v, robot in direction g = -R'v (body frame)
  float sO = -1e30f;
  int ib2 = 0;
#pragma unroll
  for (int i = 0; i < EC; ++i) {
    const float sv = v0 * Vx[i] + v1 * Vy[i];
    if (i < ne && sv > sO) { sO = sv; ib2 = i; }
  }
  const float g0 = -(cphi * v0 + sphi * v1), g1 = -(-sphi * v0 + cphi * v1);
  float sR = -1e30f;
  int jb2 = 0;
#pragma unroll
  for (int j = 0; j < RC; ++j) {
    const float sv = g0 * rb.yx[j] + g1 * rb.yy[j];
    if (j < R && sv > sR) { sR = sv; jb2 = j; }
  }
  const float marg = -sO - sR;
  // separating-slab certificate: the slab of direction v between the two sets is as wide as the pair is far
  if (!(marg >= dist - 1e-5f * (1.f + dist))) return -1;
  // LP-vertex multipliers at the two support vertices (precomputed 2x2 inverses)
  const int ia2 = (ib2 == 0) ? ne - 1 : ib2 - 1;
  const float al = v0 * og.pa0[ib2] + v1 * og.pa1[ib2], be = v0 * og.pb0[ib2] + v1 * og.pb1[ib2];
  if (!lp_vertex_ok(og.nx[ia2], og.ny[ia2], og.nx[ib2], og.ny[ib2], v0, v1, al, be)) return -1;
  const float la = rmax(al, 0.f) * og.invn[ia2], lb = rmax(be, 0.f) * og.invn[ib2];
#pragma unroll
  for (int i = 0; i < EC; ++i) out.lam[i] = (i == ia2) ? la : ((i == ib2) ? lb : 0.f);
  const int ja2 = (jb2 == 0) ? R - 1 : jb2 - 1;
  const float am = g0 * ra.pa0[jb2] + g1 * ra.pa1[jb2], bm = g0 * ra.pb0[jb2] + g1 * ra.pb1[jb2];
  const float ma = rmax(am, 0.f) * ra.ign[ja2], mb = rmax(bm, 0.f) * ra.ign[jb2];
#pragma unroll
  for (int j = 0; j < RC; ++j) out.mu[j] = (j == ja2) ? ma : ((j == jb2) ? mb : 0.f);
  const float stuff = marg - k0;
  const float z = theta * rmax(stuff, 0.f);
  out.z = z;
  out.zeta_new = stuff - z;
  out.ax = v0; out.ay = v1;
  out.c0 = marg - z + out.zeta_new;
  out.gx = g0; out.gy = g1;
  return RDA_FEAT_VALID | (ib2 << 3) | jb2;
}

}  // namespace rda
