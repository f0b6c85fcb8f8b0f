// TEST / BASELINE INFRASTRUCTURE (oracle/): CPU build of the numerical cores of
// rda_planner_b200/csrc (the same templates the CUDA kernels instantiate), compiled with g++.
//   * shim_cell_*, shim_su_*: single sub-problem entry points, used by tests/ to compare the kernel
//     arithmetic with the numpy oracle on a machine without a GPU;
//   * port_solve_batch: the whole ADMM loop of rda_kernels.cu (k_begin / k_su / k_cells /
//     k_finalize orchestration, float32 state, cold start) over a batch of instances with OpenMP
//     over instances — the compiled multi-core CPU baseline bench.py reports ("port"), and the
//     solver the CPU twins of tests/cpu_twin call per instance (declared in rda_cpu_port.h);
//   * shim_pre_process, shim_convert_obstacles: the front end cores, one instance per call.
// Built alone for bench.py (oracle/_build) and with tests/cpu_twin/*.cpp for the tests (tests/_build),
// both by oracle/build_port.py.  Never loaded by the product (rda_planner_b200/, RDA_planner/).
#include <vector>
#include <cstring>
#include <cmath>
#include <cstdlib>
#include <omp.h>
#include "../../rda_planner_b200/csrc/cell_solver.cuh"
#include "../../rda_planner_b200/csrc/cell_disc_robot.cuh"
#include "../../rda_planner_b200/csrc/su_solver.cuh"
#include "../../rda_planner_b200/csrc/cell_lean.cuh"
#include "../../rda_planner_b200/csrc/cell_lean2.cuh"
#include "rda_cpu_port.h"

using namespace rda;

template <typename Real>
static int cell_impl(const float* G, const float* h, int R, int kind, int E, const float* A, const float* b,
                     double px, double py, double phi, double dbar, double zeta, double xi0, double xi1,
                     double ro2, double theta, double* out /* lam[8] mu[8] z zeta_new xi0 xi1 ax ay c0 gx gy hm0 hm1 path */) {
  RobotGeom rb;
  int rc = robot_geom_from_halfspaces(G, h, R, &rb);
  if (rc) return rc;
  CellOut<Real> o;
  cell_solve<Real>(rb, kind, E, A, b, (Real)px, (Real)py, (Real)cos(phi), (Real)sin(phi), (Real)dbar,
                   (Real)zeta, (Real)xi0, (Real)xi1, (Real)ro2, (Real)theta, o);
  for (int i = 0; i < 8; ++i) out[i] = o.lam[i];
  for (int i = 0; i < 8; ++i) out[8 + i] = o.mu[i];
  double tail[] = {(double)o.z, (double)o.zeta_new, (double)o.xi0_new, (double)o.xi1_new, (double)o.ax,
                   (double)o.ay, (double)o.c0, (double)o.gx, (double)o.gy, (double)o.hm0, (double)o.hm1,
                   (double)o.path};
  memcpy(out + 16, tail, sizeof(tail));
  return 0;
}

// disc body (cone_type 'norm2'): h = (cx, cy, -r)
template <typename Real>
static int cell_dr_impl(const float* h, int kind, int E, const float* A, const float* b, double px, double py, double phi,
                        double dbar, double zeta, double xi0, double xi1, double ro2, double theta, double* out, int forms = 1) {
  const float Gd[6] = {1.f, 0.f, 0.f, 1.f, 0.f, 0.f};
  RobotGeom rb;
  int rc = robot_geom_from_halfspaces(Gd, h, 3, &rb, RDA_ROBOT_DISC);
  if (rc) return rc;
  CellOut<Real> o;
  cell_solve_dr<Real>(rb, kind, E, A, b, (Real)px, (Real)py, (Real)cos(phi), (Real)sin(phi), (Real)dbar,
                      (Real)zeta, (Real)xi0, (Real)xi1, (Real)ro2, (Real)theta, o, forms != 0);
  for (int i = 0; i < 8; ++i) out[i] = o.lam[i];
  for (int i = 0; i < 8; ++i) out[8 + i] = o.mu[i];
  double tail[] = {(double)o.z, (double)o.zeta_new, (double)o.xi0_new, (double)o.xi1_new, (double)o.ax,
                   (double)o.ay, (double)o.c0, (double)o.gx, (double)o.gy, (double)o.hm0, (double)o.hm1,
                   (double)o.path};
  memcpy(out + 16, tail, sizeof(tail));
  return 0;
}

// SeqCtx that also watches the su-QP's verification of the left-out hinges: its flag is the only integer that
// su_solve reduces with max(), so the call tells whether the pruned attempt converged and was verified (a repeat
// without that call was caused by the pruned attempt's iteration cap).  The solver's arithmetic is untouched.
struct SuProbeCtx : SeqCtx {
  mutable int verified = 0, violated = 0;
  template <typename R> R max(R x) const { return x; }
  int max(int x) const { ++verified; violated |= x; return x; }
};

template <typename Real>
static int su_impl(const SuParams* P, const double* lins, const double* linu, const double* ref, double vref,
                   const double* dis, const float* hx, const float* hy, const float* hc, const float* gx,
                   const float* gy, const double* pref, double* s, double* u, double* d, int* iters,
                   int* report /* restarts, verifications, violation found; may be null */) {
  const int T = P->T, N = P->N;
  SuWork<Real> W;
  size_t bytes = su_work_bytes<Real>(T, N);
  std::vector<char> buf(bytes + 64);
  char* base = (char*)(((uintptr_t)buf.data() + 63) & ~(uintptr_t)63);
  su_work_layout<Real>(T, N, &W, base);
  for (int i = 0; i < 3 * (T + 1); ++i) { W.lins[i] = (Real)lins[i]; W.ref[i] = (Real)ref[i]; }
  for (int i = 0; i < 2 * T; ++i) { W.linu[i] = (Real)linu[i]; W.pref[i] = (Real)pref[i]; }
  for (int i = 0; i < T; ++i) W.d[i] = (Real)dis[i];
  for (int i = 0; i < N * T; ++i) { W.hx[i] = hx[i]; W.hy[i] = hy[i]; W.hc[i] = hc[i]; }
  W.vref = (Real)vref;
  SuProbeCtx ctx;
  int st = su_solve<Real, SuProbeCtx>(*P, W, ctx, gx, gy, iters);
  for (int i = 0; i < 3 * (T + 1); ++i) s[i] = W.s[i];
  for (int i = 0; i < 2 * T; ++i) u[i] = W.u[i];
  for (int i = 0; i < T; ++i) d[i] = W.d[i];
  if (report) { report[0] = W.restarts; report[1] = ctx.verified; report[2] = ctx.violated; }
  return st;
}

template <int EC, int RC>
static int lean_impl(const float* G, const float* h, int R, int kind, int E, const float* A, const float* b, double px,
                     double py, double phi, double dbar, double zeta, double xi0, double xi1, double theta, double* out) {
  RobotGeom rb;
  int rc = robot_geom_from_halfspaces(G, h, R, &rb);
  if (rc) return rc;
  LeanOut<EC, RC> o;
  bool ok = cell_lean<EC, RC>(rb, kind, E, A, b, (float)px, (float)py, (float)cos(phi), (float)sin(phi), (float)dbar,
                              (float)zeta, (float)xi0, (float)xi1, (float)theta, o);
  for (int i = 0; i < 28; ++i) out[i] = 0;
  out[27] = ok ? 0 : 6;
  if (!ok) return 0;
  for (int i = 0; i < EC; ++i) out[i] = o.lam[i];
  for (int j = 0; j < RC; ++j) out[8 + j] = o.mu[j];
  out[16] = o.z; out[17] = o.zeta_new; out[18] = 0; out[19] = 0; out[20] = o.ax; out[21] = o.ay; out[22] = o.c0;
  out[23] = o.gx; out[24] = o.gy; out[25] = o.feat; out[26] = 0;
  return 0;
}

// coherent first pass (cell_lean2.cuh): out as lean_impl, out[25] = new feature byte, out[27] = 6 when declined
extern "C" int shim_cell_lean2_4(const float* G, const float* h, int R, int E, const float* A, const float* b, int feat,
                                 double px, double py, double phi, double dbar, double zeta, double theta, double* out) {
  RobotGeom rb;
  int rc = robot_geom_from_halfspaces(G, h, R, &rb);
  if (rc) return rc;
  RobotAux ra;
  robot_aux_from_geom(rb, &ra);
  ObstacleGeom<4> og;
  obstacle_geometry<4>(E, A, b, og);
  LeanOut<4, 4> o;
  int nf = cell_lean2<4, 4>(rb, ra, og, feat, (float)px, (float)py, (float)cos(phi), (float)sin(phi), (float)dbar,
                            (float)zeta, (float)theta, o);
  for (int i = 0; i < 28; ++i) out[i] = 0;
  out[27] = nf >= 0 ? 0 : 6;
  if (nf < 0) return 0;
  for (int i = 0; i < 4; ++i) out[i] = o.lam[i];
  for (int j = 0; j < 4; ++j) out[8 + j] = o.mu[j];
  out[16] = o.z; out[17] = o.zeta_new; out[20] = o.ax; out[21] = o.ay; out[22] = o.c0;
  out[23] = o.gx; out[24] = o.gy; out[25] = nf;
  return 0;
}

extern "C" {
int shim_cell_lean4(const float* G, const float* h, int R, int kind, int E, const float* A, const float* b, double px,
                    double py, double phi, double dbar, double zeta, double xi0, double xi1, double ro2, double theta,
                    double* out) {
  (void)ro2;
  return lean_impl<4, 4>(G, h, R, kind, E, A, b, px, py, phi, dbar, zeta, xi0, xi1, theta, out);
}
int shim_cell_lean8(const float* G, const float* h, int R, int kind, int E, const float* A, const float* b, double px,
                    double py, double phi, double dbar, double zeta, double xi0, double xi1, double ro2, double theta,
                    double* out) {
  (void)ro2;
  return lean_impl<8, 8>(G, h, R, kind, E, A, b, px, py, phi, dbar, zeta, xi0, xi1, theta, out);
}
int shim_cell_d(const float* G, const float* h, int R, int kind, int E, const float* A, const float* b,
                double px, double py, double phi, double dbar, double zeta, double xi0, double xi1, double ro2,
                double theta, double* out) {
  return cell_impl<double>(G, h, R, kind, E, A, b, px, py, phi, dbar, zeta, xi0, xi1, ro2, theta, out);
}
int shim_cell_f(const float* G, const float* h, int R, int kind, int E, const float* A, const float* b,
                double px, double py, double phi, double dbar, double zeta, double xi0, double xi1, double ro2,
                double theta, double* out) {
  return cell_impl<float>(G, h, R, kind, E, A, b, px, py, phi, dbar, zeta, xi0, xi1, ro2, theta, out);
}
int shim_cell_dr_d(const float* h, int kind, int E, const float* A, const float* b, double px, double py, double phi,
                   double dbar, double zeta, double xi0, double xi1, double ro2, double theta, double* out) {
  return cell_dr_impl<double>(h, kind, E, A, b, px, py, phi, dbar, zeta, xi0, xi1, ro2, theta, out);
}
// searched closed forms off: every cell that is not a plain inactive one goes through the two-cone barrier programmes
int shim_cell_dr_barrier_d(const float* h, int kind, int E, const float* A, const float* b, double px, double py, double phi,
                           double dbar, double zeta, double xi0, double xi1, double ro2, double theta, double* out) {
  return cell_dr_impl<double>(h, kind, E, A, b, px, py, phi, dbar, zeta, xi0, xi1, ro2, theta, out, 0);
}
int shim_cell_dr_f(const float* h, int kind, int E, const float* A, const float* b, double px, double py, double phi,
                   double dbar, double zeta, double xi0, double xi1, double ro2, double theta, double* out) {
  return cell_dr_impl<float>(h, kind, E, A, b, px, py, phi, dbar, zeta, xi0, xi1, ro2, theta, out);
}
int shim_su_d(const SuParams* P, const double* lins, const double* linu, const double* ref, double vref,
              const double* dis, const float* hx, const float* hy, const float* hc, const float* gx,
              const float* gy, const double* pref, double* s, double* u, double* d, int* iters) {
  return su_impl<double>(P, lins, linu, ref, vref, dis, hx, hy, hc, gx, gy, pref, s, u, d, iters, nullptr);
}
int shim_su_f(const SuParams* P, const double* lins, const double* linu, const double* ref, double vref,
              const double* dis, const float* hx, const float* hy, const float* hc, const float* gx,
              const float* gy, const double* pref, double* s, double* u, double* d, int* iters) {
  return su_impl<float>(P, lins, linu, ref, vref, dis, hx, hy, hc, gx, gy, pref, s, u, d, iters, nullptr);
}
// as shim_su_*, plus report[3]: restarts, verifications of the left-out hinges, violation found (SuProbeCtx)
int shim_su_report_d(const SuParams* P, const double* lins, const double* linu, const double* ref, double vref,
                     const double* dis, const float* hx, const float* hy, const float* hc, const float* gx,
                     const float* gy, const double* pref, double* s, double* u, double* d, int* iters, int* report) {
  return su_impl<double>(P, lins, linu, ref, vref, dis, hx, hy, hc, gx, gy, pref, s, u, d, iters, report);
}
int shim_su_report_f(const SuParams* P, const double* lins, const double* linu, const double* ref, double vref,
                     const double* dis, const float* hx, const float* hy, const float* hc, const float* gx,
                     const float* gy, const double* pref, double* s, double* u, double* d, int* iters, int* report) {
  return su_impl<float>(P, lins, linu, ref, vref, dis, hx, hy, hc, gx, gy, pref, s, u, d, iters, report);
}
}


// ------------------------------------------------------------------------------------------------
// Whole hot path on the CPU (mirrors rda_kernels.cu; see the kernel comments for reference lines).
// Layouts as in include/rda_b200.h.  Every instance starts cold (constructor state).
// ------------------------------------------------------------------------------------------------
extern "C" int port_solve_batch(const rda_config* cfg, const rda_tunables* tun, int B, const float* nom_s,
                                const float* nom_u, const float* ref_s, const float* ref_speed,
                                const float* obs_A, const float* obs_b, const int* obs_kind,
                                const int* obs_count, int tv, int iter_num, float thr, float* u_opt,
                                float* s_opt, float* resi_pri, float* resi_dual, int* iters_out, int* fails_out, int nthreads) {
  RobotGeom rb;
  int rc = robot_geom_from_halfspaces(cfg->G, cfg->h, cfg->robot_edges, &rb, cfg->robot_cone);
  if (rc) return rc;
  const int T = cfg->receding, N = cfg->max_obs_num, E = cfg->max_edge_num, R = cfg->robot_edges, NT = N * T;
  SuParams P;
  P.T = T; P.N = N; P.dynamics = cfg->dynamics; P.accelerated = cfg->accelerated;
  P.dt = cfg->step_time; P.L = cfg->wheelbase;
  P.umax[0] = cfg->max_speed[0]; P.umax[1] = cfg->max_speed[1];
  P.ab[0] = cfg->acce_bound[0]; P.ab[1] = cfg->acce_bound[1];
  P.ws = cfg->ws; P.wu = cfg->wu; P.slack_gain = tun->slack_gain; P.dmin = tun->min_sd; P.dmax = tun->max_sd;
  P.ro1 = tun->ro1; P.ro2 = tun->ro2; P.max_iter = 40;
  P.mu0 = 1.0f; P.prune = 0.5f;      // as the library (rda_kernels.cu: mu0, the default su_prune)
  const float theta = cfg->accelerated ? tun->z_theta : 1.0f;
  if (nthreads > 0) omp_set_num_threads(nthreads);
  const size_t bytes = su_work_bytes<double>(T, N);
#pragma omp parallel for schedule(dynamic, 1)
  for (int b = 0; b < B; ++b) {
    std::vector<char> buf(bytes + 64);
    char* base = (char*)(((uintptr_t)buf.data() + 63) & ~(uintptr_t)63);
    SuWork<double> W;
    su_work_layout<double>(T, N, &W, base);
    std::vector<float> lam((size_t)N * E * T, 0.f), mu((size_t)N * R * T, 0.f), z(NT, 0.f), xi(2 * NT, 0.f),
        zeta(NT, 0.f), dis(T, 1.f), coef(5 * (size_t)NT, 0.f), pref(2 * T, 0.f);
    const bool use_lean2 = getenv("RDA_PORT_LEAN2") && atoi(getenv("RDA_PORT_LEAN2")) != 0;
    std::vector<int> feat2(NT > 0 ? NT : 1, 0);
    std::vector<ObstacleGeom<4>> og2(N > 0 ? N : 1);
    RobotAux ra2;
    robot_aux_from_geom(rb, &ra2);
    long long coh_hits = 0;
    if (use_lean2 && E <= 4 && R <= 4 && !tv && !rb.disc)
      for (int o = 0; o < N; ++o) obstacle_geometry<4>(E, obs_A + ((size_t)b * N + o) * E * 2, obs_b + ((size_t)b * N + o) * E, og2[o]);
    std::vector<float> cs(nom_s + (size_t)b * 3 * (T + 1), nom_s + (size_t)(b + 1) * 3 * (T + 1));
    std::vector<float> cu(nom_u + (size_t)b * 2 * T, nom_u + (size_t)(b + 1) * 2 * T);
    const float* rf = ref_s + (size_t)b * 3 * (T + 1);
    float rp = 0.f, rd = 0.f;
    int it = 0, nfail = 0, first_fail = -1, su_iters = 0, su_bad = 0;
    for (it = 0; it < iter_num; ++it) {
      for (int i = 0; i < 3 * (T + 1); ++i) { int r = i / (T + 1), t = i % (T + 1); W.lins[3 * t + r] = cs[i]; W.ref[3 * t + r] = rf[i]; }
      for (int i = 0; i < 2 * T; ++i) { int r = i / T, t = i % T; W.linu[2 * t + r] = cu[i]; W.pref[2 * t + r] = pref[i]; }
      for (int t = 0; t < T; ++t) W.d[t] = dis[t];
      for (int i = 0; i < NT; ++i) { W.hx[i] = coef[i]; W.hy[i] = coef[NT + i]; W.hc[i] = coef[2 * NT + i]; }
      W.vref = ref_speed[b];
      SeqCtx ctx;
      int nit = 0;
      const int st = su_solve<double, SeqCtx>(P, W, ctx, coef.data() + 3 * NT, coef.data() + 4 * NT, &nit);
      su_iters += nit;
      if (st != 0) ++su_bad;
      if (st != 2) {
        for (int i = 0; i < 3 * (T + 1); ++i) { int r = i / (T + 1), t = i % (T + 1); cs[i] = (float)W.s[3 * t + r]; }
        for (int i = 0; i < 2 * T; ++i) { int r = i / T, t = i % T; cu[i] = (float)W.u[2 * t + r]; }
        for (int t = 0; t < T; ++t) dis[t] = (float)W.d[t];
      }
      double hm2 = 0, dual = 0;
      if (N > 0 && obs_count[b] != 0) {
        for (int o = 0; o < N; ++o)
          for (int t = 0; t < T; ++t) {
            int tc = tv ? t + 1 : 0, Tc = tv ? T + 1 : 1;
            size_t ob = ((size_t)b * N + o) * Tc + tc;
            float ph = cs[2 * (T + 1) + t];
            CellOut<float> out;
            // emulation of the coherent pipeline (RDA_PORT_LEAN2=1): k_cells_coh -> listed cell_lean -> generic solver, under the
            // library's condition (rda_create / step_lammuz_part: E <= 4, R <= 4, static polygons; padded rows are zero)
            bool lean_done = false;
            if (use_lean2 && !rb.disc && E <= 4 && R <= 4 && !tv && obs_kind[(size_t)b * N + o] == RDA_OBS_POLYGON) {
              LeanOut<4, 4> lo;
              int nf = -1;
              if (xi[o * T + t] == 0.f && xi[NT + o * T + t] == 0.f)
                nf = cell_lean2<4, 4>(rb, ra2, og2[o], feat2[o * T + t], cs[t + 1], cs[(T + 1) + t + 1], cosf(ph), sinf(ph), dis[t],
                                      zeta[o * T + t], theta, lo);
              if (nf < 0) {
                const bool ok1 = cell_lean<4, 4>(rb, RDA_OBS_POLYGON, E, obs_A + ob * E * 2, obs_b + ob * E, cs[t + 1], cs[(T + 1) + t + 1],
                                                 cosf(ph), sinf(ph), dis[t], zeta[o * T + t], xi[o * T + t], xi[NT + o * T + t], theta, lo);
                nf = ok1 ? lo.feat : -1;
              } else ++coh_hits;
              feat2[o * T + t] = nf >= 0 ? nf : 0;
              if (nf >= 0) {
                lean_done = true;
                for (int i = 0; i < 8; ++i) { out.lam[i] = i < 4 ? lo.lam[i] : 0.f; out.mu[i] = i < 4 ? lo.mu[i] : 0.f; }
                out.z = lo.z; out.zeta_new = lo.zeta_new; out.xi0_new = 0.f; out.xi1_new = 0.f; out.ax = lo.ax; out.ay = lo.ay;
                out.c0 = lo.c0; out.gx = lo.gx; out.gy = lo.gy; out.hm0 = 0.f; out.hm1 = 0.f; out.path = CELL_FAST_INACTIVE;
              }
            }
            if (rb.disc)
              cell_solve_dr<float>(rb, obs_kind[(size_t)b * N + o], E, obs_A + ob * E * 2, obs_b + ob * E, cs[t + 1],
                                   cs[(T + 1) + t + 1], cosf(ph), sinf(ph), dis[t], zeta[o * T + t], xi[o * T + t],
                                   xi[NT + o * T + t], (float)P.ro2, theta, out);
            else if (!lean_done)
            cell_solve<float>(rb, obs_kind[(size_t)b * N + o], E, obs_A + ob * E * 2, obs_b + ob * E, cs[t + 1],
                              cs[(T + 1) + t + 1], cosf(ph), sinf(ph), dis[t], zeta[o * T + t], xi[o * T + t],
                              xi[NT + o * T + t], (float)P.ro2, theta, out);
            if (out.path == CELL_FAILED) { dual = INFINITY; ++nfail; if (first_fail < 0) first_fail = (it * N + o) * T + t; continue; }
            float acc = 0.f;
            for (int i = 0; i < E; ++i) { float nv = out.lam[i], df = nv - lam[((size_t)o * E + i) * T + t]; acc += df * df; lam[((size_t)o * E + i) * T + t] = nv; }
            for (int j = 0; j < R; ++j) { float nv = out.mu[j], df = nv - mu[((size_t)o * R + j) * T + t]; acc += df * df; mu[((size_t)o * R + j) * T + t] = nv; }
            float dz = out.z - z[o * T + t];
            acc += dz * dz;
            z[o * T + t] = out.z;
            dual += acc;
            zeta[o * T + t] = out.zeta_new;
            xi[o * T + t] = out.xi0_new; xi[NT + o * T + t] = out.xi1_new;
            hm2 += out.hm0 * out.hm0 + out.hm1 * out.hm1;
            coef[o * T + t] = out.ax; coef[NT + o * T + t] = out.ay; coef[2 * NT + o * T + t] = out.c0;
            coef[3 * NT + o * T + t] = out.gx; coef[4 * NT + o * T + t] = out.gy;
            if (o == 0) { pref[t] = cs[t + 1]; pref[T + t] = cs[(T + 1) + t + 1]; }
          }
        rp = (float)sqrt(hm2); rd = (float)(dual / N);
      } else { rp = 0.f; rd = 0.f; }
      if (rd < thr && rp < thr) { ++it; break; }
    }
    for (int i = 0; i < 3 * (T + 1); ++i) s_opt[(size_t)b * 3 * (T + 1) + i] = cs[i];
    for (int i = 0; i < 2 * T; ++i) u_opt[(size_t)b * 2 * T + i] = cu[i];
    resi_pri[b] = rp; resi_dual[b] = rd;
    if (iters_out) iters_out[b] = it;
    if (fails_out) { fails_out[4 * b] = nfail; fails_out[4 * b + 1] = first_fail; fails_out[4 * b + 2] = su_iters; fails_out[4 * b + 3] = su_bad; if (use_lean2) fails_out[4 * b + 1] = (int)coh_hits; }
  }
  return 0;
}


// ---- front end cores (rda_planner_b200/csrc/frontend.cuh), one instance per call -----------------
#include "../../rda_planner_b200/csrc/frontend.cuh"

extern "C" int shim_pre_process(int dynamics, int T, double dt, double L, const float* state, const float* vel,
                                double ref_speed, const float* path, int P, int start_index, double threshold,
                                int ind_range, float* nom_s, float* ref_s) {
  return rda::pre_process_one(dynamics, T, dt, L, state, vel, ref_speed, path, P, start_index, threshold, ind_range,
                              nom_s, ref_s);
}

// Emulates k_convert_obstacles for one instance: M raw shapes -> N slots.
extern "C" int shim_convert_obstacles(int M, int N, int T, int E, double dt, int time_varying, int order, const float* state,
                                      const int* kind, const int* nv, const float* xy, const float* radius,
                                      const float* vel, int count, float* obs_A, float* obs_b, int* obs_kind) {
  if (count > M) count = M;
  std::vector<double> keys(count > 0 ? count : 1);
  for (int j = 0; j < count; ++j)
    keys[j] = order ? rda::obstacle_key(kind[j], nv[j], xy + (size_t)j * RDA_MAX_EDGE * 2, state[0], state[1]) : (double)j;
  const int Tc = time_varying ? T + 1 : 1;
  for (int n = 0; n < N; ++n) {
    float* A = obs_A + (size_t)n * Tc * E * 2;
    float* b = obs_b + (size_t)n * Tc * E;
    const int src = rda::obstacle_slot_source(n, count, 1, keys.data());
    if (src < 0) {
      for (int i = 0; i < Tc * E; ++i) { A[2 * i] = 0.f; A[2 * i + 1] = 0.f; b[i] = 0.f; }
      obs_kind[n] = RDA_OBS_POLYGON;
      continue;
    }
    obs_kind[n] = kind[src];
    for (int t = 0; t < Tc; ++t)
      rda::obstacle_rows(kind[src], nv[src], xy + (size_t)src * RDA_MAX_EDGE * 2, radius[src], vel[2 * src], vel[2 * src + 1], t,
                         dt, E, A + (size_t)t * E * 2, b + (size_t)t * E);
  }
  return count;
}
