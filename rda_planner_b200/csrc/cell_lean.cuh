// cell_lean.cuh — first pass of the (lam, mu, z) cell kernel, specialised at compile time.
//
// Handles exactly the two closed-form cases that need no search (DESIGN.md §3, cases 1-2):
//   xi = 0, sets disjoint, margin >= 0  -> max-margin certificate = unit normal of the closest pair
//   xi = 0, sets overlap,  margin >= 0  -> v = 0
// i.e. the inactive cells, which are ~95 % of all cells.  Everything is written with compile-time
// loop bounds (EC obstacle rows, RC robot rows) and select chains instead of run-time indices, so
// that the whole per-cell geometry lives in registers (the generic cell_front keeps it in local
// memory).  Arithmetic mirrors cell_front / cell_back (cell_solver.cuh) step by step; the CPU tests
// compare the two on random cells.  Same reference lines: rda_solver.py:389-421, 529-542, 639-690.
#pragma once
#include "rda_hd.h"

namespace rda {

// A vertex-vertex pair and the neighbouring vertex-edge pair can tie in float32 when the foot of the
// perpendicular lies within sqrt(2 eps) |d| of the edge's end; the vertex-vertex direction is then off by up
// to 5e-4 rad and the margin by that times the edge length.  End-point candidates carry this relative
// handicap so that such ties go to the edge-interior pair, whose direction is the edge normal.
#define RDA_ENDPOINT_BIAS 1.0000006f

template <int EC, int RC>
struct LeanOut {
  float lam[EC];
  float mu[RC];
  float z, zeta_new, ax, ay, c0, gx, gy;
  int feat;      // 0x40 | obstacle support vertex << 3 | robot support vertex of a separated polygon pair, else 0 (cell_lean2.cuh)
};

// LP-vertex coefficients (al, be) of a direction v at a vertex with rows of unit normals n_a, n_b: false when v lies clearly
// outside the vertex's normal cone (the support went to the wrong end of a short edge) or al n_a + be n_b comes out longer
// than v by more than rounding (rows nearly parallel).  The first passes then decline the cell, and the searched passes
// resolve it (obs_vertex_lam, cell_solver.cuh).
RDA_HD bool lp_vertex_ok(float nax, float nay, float nbx, float nby, float v0, float v1, float al, float be) {
  if (rmin(al, be) < -1e-5f) return false;
  al = rmax(al, 0.f); be = rmax(be, 0.f);
  const float wx = al * nax + be * nbx, wy = al * nay + be * nby;
  return wx * wx + wy * wy <= (v0 * v0 + v1 * v1) * (1.f + 1e-5f);
}

// returns true when the cell is resolved (outputs valid); false -> next pass
template <int EC, int RC>
RDA_HD bool cell_lean(const RobotGeom& rb, int kind, int E, const float* A, const float* b, float px, float py,
                      float cphi, float sphi, float dbar, float zeta, float xi0, float xi1, float theta,
                      LeanOut<EC, RC>& out) {
  if (xi0 != 0.f || xi1 != 0.f) return false;
  const int R = rb.R;
  const float k0 = dbar - zeta;
  const float eps = 1e-5f;
  // ---- robot in the world frame (relative to p) ----
  float Yx[RC], Yy[RC], Mx[RC], My[RC];
#pragma unroll
  for (int j = 0; j < RC; ++j) {
    const float yx = rb.yx[j], yy = rb.yy[j], nx = rb.nx[j], ny = rb.ny[j];
    Yx[j] = cphi * yx - sphi * yy; Yy[j] = sphi * yx + cphi * yy;
    Mx[j] = cphi * nx - sphi * ny; My[j] = sphi * nx + cphi * ny;
  }
  float v0 = 0.f, v1 = 0.f;
  bool sep = false;
  float best = 1e30f, bdx = 0.f, bdy = 0.f;
  float sO = 0.f;                      // support of the obstacle in direction v (relative coordinates)
  float lamv[EC];
  int fi = -1, fj = -1;
#pragma unroll
  for (int i = 0; i < EC; ++i) lamv[i] = 0.f;
  if (kind == RDA_OBS_CIRCLE) {
    const float cx = b[0] - px, cy = b[1] - py, rad = -b[2];
    bool inside = true;
#pragma unroll
    for (int j = 0; j < RC; ++j) {
      if (j < R) {
        const float nxx = (j + 1 < RC) ? ((j + 1 < R) ? Yx[(j + 1) % RC] : Yx[0]) : Yx[0];
        const float nyy = (j + 1 < RC) ? ((j + 1 < R) ? Yy[(j + 1) % RC] : Yy[0]) : Yy[0];
        const float fx = nxx - Yx[j], fy = nyy - Yy[j];
        const float rx = cx - Yx[j], ry = cy - Yy[j];
        if (Mx[j] * rx + My[j] * ry > 0.f) inside = false;
        const float t = rclamp((rx * fx + ry * fy) / (fx * fx + fy * fy), 0.f, 1.f);
        const float dx = -(rx - t * fx), dy = -(ry - t * fy);
        const float d2 = dx * dx + dy * dy;
        if (d2 < best) { best = d2; bdx = dx; bdy = dy; }
      }
    }
    const float dc = sqrt_(best);
    sep = (!inside) && (dc > rad + eps);
    if (sep) {
      const float dd = dc - rad;
      if (dd - k0 < 0.f) return false;
      v0 = bdx / dc; v1 = bdy / dc;          // unit (bd / dc), as cell_front: (bd/dc*dd)/dd
      // cell_front rescales bd to length dd and divides by dist = dd: identical direction
      sO = v0 * cx + v1 * cy + rad * sqrt_(v0 * v0 + v1 * v1);
      lamv[0] = v0; lamv[1] = v1;
      if (EC > 2) lamv[2] = -sqrt_(v0 * v0 + v1 * v1);
    } else {
      if (k0 > 0.f) return false;
      sO = 0.f;
    }
  } else {
    // ---- polygon rows -> unit normals, offsets relative to p, vertices ----
    float nx[EC], ny[EC], invn[EC], brel[EC];
    int ne = 0;
#pragma unroll
    for (int i = 0; i < EC; ++i) {
      float ax = 0.f, ay = 0.f, bb = 0.f;
      if (i < E) { ax = A[2 * i]; ay = A[2 * i + 1]; bb = b[i]; }
      const float n2 = ax * ax + ay * ay;
      const bool live = (n2 > 0.f) && (ne == i);     // rows are contiguous; padding follows
      const float inv = live ? rsqrt_(n2) : 0.f;
      nx[i] = ax * inv; ny[i] = ay * inv; invn[i] = inv;
      brel[i] = (bb - ax * px - ay * py) * inv;
      if (live) ne = i + 1;
    }
    if (ne < 3) return false;
    // last live row (the "previous" row of vertex 0)
    float lnx = nx[0], lny = ny[0], lbr = brel[0];
#pragma unroll
    for (int i = 1; i < EC; ++i)
      if (i == ne - 1) { lnx = nx[i]; lny = ny[i]; lbr = brel[i]; }
    float Vx[EC], Vy[EC];
#pragma unroll
    for (int i = 0; i < EC; ++i) {
      const float pnx = (i == 0) ? lnx : nx[(i + EC - 1) % EC];
      const float pny = (i == 0) ? lny : ny[(i + EC - 1) % EC];
      const float pbr = (i == 0) ? lbr : brel[(i + EC - 1) % EC];
      const float det = pnx * ny[i] - pny * nx[i];
      const float inv = 1.f / det;
      Vx[i] = (pbr * ny[i] - brel[i] * pny) * inv;
      Vy[i] = (pnx * brel[i] - nx[i] * pbr) * inv;
    }
    // ---- closest pair and separating-axis test ----
    float dj2[RC], djx[RC], djy[RC];
#pragma unroll
    for (int j = 0; j < RC; ++j) dj2[j] = 1e30f;
#pragma unroll
    for (int i = 0; i < EC; ++i) {
      if (i < ne) {
        const float nvx = (i + 1 < EC && i + 1 < ne) ? Vx[(i + 1) % EC] : Vx[0];
        const float nvy = (i + 1 < EC && i + 1 < ne) ? Vy[(i + 1) % EC] : Vy[0];
        const float ex = nvx - Vx[i], ey = nvy - Vy[i];
        const float ie2 = 1.f / (ex * ex + ey * ey);
        float mins = 1e30f;
#pragma unroll
        for (int j = 0; j < RC; ++j) {
          if (j < R) {
            const float rx = Yx[j] - Vx[i], ry = Yy[j] - Vy[i];
            mins = rmin(mins, nx[i] * rx + ny[i] * ry);
            const float t = rclamp((rx * ex + ry * ey) * ie2, 0.f, 1.f);
            const float dx = rx - t * ex, dy = ry - t * ey;
            const float d2 = (dx * dx + dy * dy) * ((t > 0.f && t < 1.f) ? 1.f : RDA_ENDPOINT_BIAS);
            if (d2 < dj2[j]) { dj2[j] = d2; djx[j] = dx; djy[j] = dy; }
          }
        }
        if (mins > eps) sep = true;
      }
    }
#pragma unroll
    for (int j = 0; j < RC; ++j)
      if (j < R && dj2[j] < best) { best = dj2[j]; bdx = djx[j]; bdy = djy[j]; }
#pragma unroll
    for (int j = 0; j < RC; ++j) {
      if (j < R) {
        const float nxx = (j + 1 < RC && j + 1 < R) ? Yx[(j + 1) % RC] : Yx[0];
        const float nyy = (j + 1 < RC && j + 1 < R) ? Yy[(j + 1) % RC] : Yy[0];
        const float fx = nxx - Yx[j], fy = nyy - Yy[j];
        const float if2 = 1.f / (fx * fx + fy * fy);
        float mins = 1e30f;
#pragma unroll
        for (int i = 0; i < EC; ++i) {
          if (i < ne) {
            const float rx = Vx[i] - Yx[j], ry = Vy[i] - Yy[j];
            mins = rmin(mins, Mx[j] * rx + My[j] * ry);
            const float t = rclamp((rx * fx + ry * fy) * if2, 0.f, 1.f);
            const float dx = -(rx - t * fx), dy = -(ry - t * fy);
            const float d2 = (dx * dx + dy * dy) * ((t > 0.f && t < 1.f) ? 1.f : RDA_ENDPOINT_BIAS);
            if (d2 < best) { best = d2; bdx = dx; bdy = dy; }
          }
        }
        if (mins > eps) sep = true;
      }
    }
    if (sep) {
      const float dist = sqrt_(best);
      if (dist - k0 < 0.f) return false;
      v0 = bdx / dist; v1 = bdy / dist;
      // support vertex of the obstacle for v and the two rows adjacent to it (LP-vertex multipliers)
      float sb = -1e30f, anx = 0.f, any = 0.f, ain = 0.f, bnx = 0.f, bny = 0.f, bin = 0.f;
      int ia = 0, ib = 0;
#pragma unroll
      for (int i = 0; i < EC; ++i) {
        if (i < ne) {
          const float sv = v0 * Vx[i] + v1 * Vy[i];
          if (sv > sb) {
            sb = sv; ib = i; ia = (i == 0) ? ne - 1 : i - 1;
            bnx = nx[i]; bny = ny[i]; bin = invn[i];
            anx = (i == 0) ? lnx : nx[(i + EC - 1) % EC];
            any = (i == 0) ? lny : ny[(i + EC - 1) % EC];
          }
        }
      }
      // inverse norm of row ia
#pragma unroll
      for (int i = 0; i < EC; ++i)
        if (i == ia) ain = invn[i];
      sO = sb;
      fi = ib;
      const float det = anx * bny - any * bnx;
      const float al = (v0 * bny - v1 * bnx) / det;
      const float be = (anx * v1 - any * v0) / det;
      if (!lp_vertex_ok(anx, any, bnx, bny, v0, v1, al, be)) return false;
      const float la = rmax(al, 0.f) * ain, lb = rmax(be, 0.f) * bin;
#pragma unroll
      for (int i = 0; i < EC; ++i) lamv[i] = (i == ia) ? la : ((i == ib) ? lb : 0.f);
      if (ia == ib) { /* cannot happen for ne >= 3 */ }
    } else {
      if (k0 > 0.f) return false;
      sO = 0.f;                       // v = 0
    }
  }
  // ---- robot side: g = -R'v, multipliers of the two rows adjacent to its support vertex ----
  const float g0 = -(cphi * v0 + sphi * v1), g1 = -(-sphi * v0 + cphi * v1);
  float muv[RC];
#pragma unroll
  for (int j = 0; j < RC; ++j) muv[j] = 0.f;
  float sR = 0.f;
  if (g0 != 0.f || g1 != 0.f) {
    float sb = -1e30f, anx = 0.f, any = 0.f, agn = 1.f, bnx = 0.f, bny = 0.f, bgn = 1.f;
    int ja = 0, jb = 0;
    // last live robot row
    float lnx = rb.nx[0], lny = rb.ny[0], lgn = rb.gnorm[0];
#pragma unroll
    for (int j = 1; j < RC; ++j)
      if (j == R - 1) { lnx = rb.nx[j]; lny = rb.ny[j]; lgn = rb.gnorm[j]; }
#pragma unroll
    for (int j = 0; j < RC; ++j) {
      if (j < R) {
        const float sv = g0 * rb.yx[j] + g1 * rb.yy[j];
        if (sv > sb) {
          sb = sv; jb = j; ja = (j == 0) ? R - 1 : j - 1;
          bnx = rb.nx[j]; bny = rb.ny[j]; bgn = rb.gnorm[j];
          anx = (j == 0) ? lnx : rb.nx[(j + RC - 1) % RC];
          any = (j == 0) ? lny : rb.ny[(j + RC - 1) % RC];
          agn = (j == 0) ? lgn : rb.gnorm[(j + RC - 1) % RC];
        }
      }
    }
    sR = sb;
    fj = jb;
    const float det = anx * bny - any * bnx;
    const float al = (g0 * bny - g1 * bnx) / det;
    const float be = (anx * g1 - any * g0) / det;
    const float ma = rmax(al, 0.f) / agn, mb = rmax(be, 0.f) / bgn;
#pragma unroll
    for (int j = 0; j < RC; ++j) muv[j] = (j == ja) ? ma : ((j == jb) ? mb : 0.f);
  }
  // ---- multipliers and updates (cell_back with q = 0, xi = 0) ----
  const float marg = -sO - sR;
  const float stuff = marg - k0;
  const float z = theta * rmax(stuff, 0.f);
#pragma unroll
  for (int i = 0; i < EC; ++i) out.lam[i] = lamv[i];
#pragma unroll
  for (int j = 0; j < RC; ++j) out.mu[j] = muv[j];
  out.z = z;
  out.zeta_new = stuff - z;
  out.ax = v0; out.ay = v1;
  out.c0 = marg - z + out.zeta_new;
  out.gx = g0; out.gy = g1;
  out.feat = (fi >= 0 && fj >= 0) ? (0x40 | (fi << 3) | fj) : 0;
  return true;
}

}  // namespace rda
