// rda_hd.h — host/device portability shims.  The numerical cores (cell_solver.cuh,
// su_solver.cuh) are plain templates that compile both with nvcc for sm_90a (the
// product) and with g++ (tests/host_shim, CPU-only checks of the same arithmetic).
#pragma once
#include <math.h>
#include <stdint.h>
#include "../../include/rda_b200.h"

#if defined(__CUDACC__)
#define RDA_HD __host__ __device__ __forceinline__
#define RDA_HD_NOINLINE __host__ __device__ __noinline__
#else
#define RDA_HD inline
#define RDA_HD_NOINLINE
#endif

namespace rda {

// sum and product rounded on their own, never fused with a neighbouring operation into an FMA: they keep an expression's
// rounding where the compiler could otherwise contract differently (a factor of a constant +-1 folded away, an addend
// held in a register instead of memory)
RDA_HD float add_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
RDA_HD double add_rn(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
// a * b + c fused on the device, where the compiler could otherwise leave it unfused (both arms of a branch merged into
// one select); rounded twice on the host, as the host build computes it
RDA_HD float fma_dev(float a, float b, float c) {
#if defined(__CUDA_ARCH__)
  return __fmaf_rn(a, b, c);
#else
  return a * b + c;
#endif
}
RDA_HD double fma_dev(double a, double b, double c) {
#if defined(__CUDA_ARCH__)
  return __fma_rn(a, b, c);
#else
  return a * b + c;
#endif
}
RDA_HD float mul_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
RDA_HD double mul_rn(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
template <typename T> RDA_HD T rmin(T a, T b) { return a < b ? a : b; }
template <typename T> RDA_HD T rmax(T a, T b) { return a > b ? a : b; }
template <typename T> RDA_HD T rclamp(T x, T lo, T hi) { return x < lo ? lo : (x > hi ? hi : x); }
RDA_HD float rsqrt_(float x) { return 1.0f / sqrtf(x); }
RDA_HD double rsqrt_(double x) { return 1.0 / sqrt(x); }
RDA_HD float sqrt_(float x) { return sqrtf(x); }
RDA_HD double sqrt_(double x) { return sqrt(x); }
RDA_HD float abs_(float x) { return fabsf(x); }
RDA_HD double abs_(double x) { return fabs(x); }
// LP-vertex coefficients (al, be) >= 0 of a direction v in the unit normals n_a, n_b of a vertex's two rows: scaled back to
// |v| where al n_a + be n_b comes out longer than v by more than rounding (rows nearly parallel: the coefficients' rounding
// error is eps / sin(angle between the rows)), so that |A'lam| <= |v| <= 1 holds as the reference's constraint requires
template <typename T>
RDA_HD void cone_rescale(T nax, T nay, T nbx, T nby, T v0, T v1, T& al, T& be) {
  const T wx = al * nax + be * nbx, wy = al * nay + be * nby;
  const T w2 = wx * wx + wy * wy, v2 = v0 * v0 + v1 * v1;
  if (w2 > v2 * (T)(1 + 1e-5)) { const T f = sqrt_(v2 / w2); al *= f; be *= f; }
}
// reciprocal: on the device the hardware's double-precision reciprocal seed (MUFU.RCP64H, ~20 bits) refined by
// two Newton steps — 5 dependent instructions, no float <-> double conversions (the float-seed variant of round
// 1 spent 13 % of the su-QP kernel's stall samples on its two F2F conversions, profiles/ncu_r02_ksu_lines.md);
// arguments are positive normal numbers at every call site.  Plain division on the host.
RDA_HD float rcp_(float x) { return 1.0f / x; }
RDA_HD double rcp_(double x) {
#if defined(__CUDA_ARCH__)
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
  double e = fma(-x, r, 1.0);
  r = fma(r, e, r);
  e = fma(-x, r, 1.0);
  r = fma(r, e, r);
  return r;
#else
  return 1.0 / x;
#endif
}
// number of set bits
RDA_HD int popc_(unsigned m) {
#if defined(__CUDA_ARCH__)
  return __popc(m);
#else
  return __builtin_popcount(m);
#endif
}
RDA_HD bool finite_(float x) { return isfinite(x); }
RDA_HD bool finite_(double x) { return isfinite(x); }

// Single-lane context (host tests; also valid on the device for a thread-per-instance launch).
struct SeqCtx {
  RDA_HD int lane() const { return 0; }
  RDA_HD int nlanes() const { return 1; }
  RDA_HD void sync() const {}
  template <typename R> RDA_HD R sum(R x) const { return x; }
  template <typename R> RDA_HD R min(R x) const { return x; }
  template <typename R> RDA_HD R max(R x) const { return x; }
};

// Robot body (convex polygon, car_tuple.G/h with Rpositive cone), prepared once at
// rda_create: vertices y_j (vertex j joins rows j-1 and j, rda mpc.py:476-510 ordering),
// unit outward normals and row norms.
struct RobotGeom {
  int R;
  int disc;                 // 1: disc body (car_tuple.cone_type 'norm2', rda_solver.py:1034-1039): centre (cx, cy), radius rad
  float rad, cx, cy;
  float yx[RDA_MAX_ROBOT_EDGE], yy[RDA_MAX_ROBOT_EDGE];
  float nx[RDA_MAX_ROBOT_EDGE], ny[RDA_MAX_ROBOT_EDGE], gnorm[RDA_MAX_ROBOT_EDGE];
  float h[RDA_MAX_ROBOT_EDGE];
};

// Fill RobotGeom from (G, h); returns 0 or RDA_E_UNSUPPORTED when the rows do not describe a
// closed convex polygon listed counter-clockwise.
inline int robot_geom_from_halfspaces(const float* G, const float* h, int R, RobotGeom* out, int cone = RDA_ROBOT_POLYGON) {
  if (R < 3 || R > RDA_MAX_ROBOT_EDGE) return RDA_E_UNSUPPORTED;
  out->R = R;
  out->disc = 0; out->rad = 0.f; out->cx = 0.f; out->cy = 0.f;
  if (cone == RDA_ROBOT_DISC) {
    // ir-sim description of a circular body: G = [[1,0],[0,1],[0,0]], h = (cx, cy, -r); any other norm2 body is refused
    const float Gd[6] = {1.f, 0.f, 0.f, 1.f, 0.f, 0.f};
    if (R != 3) return RDA_E_UNSUPPORTED;
    for (int k = 0; k < 6; ++k) if (fabsf(G[k] - Gd[k]) > 1e-6f) return RDA_E_UNSUPPORTED;
    if (!(h[2] < 0.f)) return RDA_E_UNSUPPORTED;
    out->disc = 1; out->cx = h[0]; out->cy = h[1]; out->rad = -h[2];
    for (int j = 0; j < RDA_MAX_ROBOT_EDGE; ++j) { out->yx[j] = out->yy[j] = out->nx[j] = out->ny[j] = 0.f; out->gnorm[j] = 1.f; out->h[j] = j < 3 ? h[j] : 0.f; }
    return 0;
  }
  if (cone != RDA_ROBOT_POLYGON) return RDA_E_UNSUPPORTED;
  for (int j = 0; j < R; ++j) {
    double gx = G[2 * j], gy = G[2 * j + 1];
    double n = sqrt(gx * gx + gy * gy);
    if (!(n > 0)) return RDA_E_UNSUPPORTED;
    out->nx[j] = (float)(gx / n);
    out->ny[j] = (float)(gy / n);
    out->gnorm[j] = (float)n;
    out->h[j] = h[j];
  }
  for (int j = 0; j < R; ++j) {
    int a = (j + R - 1) % R;
    double ax = G[2 * a], ay = G[2 * a + 1], bx = G[2 * j], by = G[2 * j + 1];
    double det = ax * by - ay * bx;
    if (!(det > 1e-12)) return RDA_E_UNSUPPORTED;  // CCW rows => positive turn
    out->yx[j] = (float)((h[a] * by - h[j] * ay) / det);
    out->yy[j] = (float)((ax * h[j] - bx * h[a]) / det);
  }
  return 0;
}

}  // namespace rda
