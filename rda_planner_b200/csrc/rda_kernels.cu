// rda_kernels.cu — sm_90a kernels and the C ABI (include/rda_b200.h) of the RDA ADMM hot path.
//
// One ADMM iteration (rda_solver.py:612-637) is five launches on the caller's stream:
//   k_su      one warp per planning instance: su-QP (su_solver.cuh), state staged in shared memory
//   k_cells_fast / k_cells_mid   one thread per (instance, obstacle, stage) cell, k_cells_slow_coop one warp per cell:
//             (lam, mu, z) + xi/zeta update + residual partial sums + the next su-QP's hinge inputs (cell_solver.cuh)
//   k_finalize per instance: residuals, early-stop flag (:594-596)
// No host synchronisation, no allocation, CUDA-graph capturable.
#include <cuda_runtime.h>
#include <limits.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <new>
#include "rda_hd.h"
#include "cell_solver.cuh"
#include "su_solver.cuh"
#include "cell_lean.cuh"
#include "cell_lean2.cuh"
#include "cell_disc_robot.cuh"
#include "plan_clearance.cuh"
#include "obstacle_ids.cuh"

using namespace rda;

// byte offsets of the persistent kernel's shared-memory state (k_admm_small)
struct SmallLayout {
  int lam, mu, z, xi, zeta, dis, coef, pref, cur_s, cur_u, ref_s, misc, hs, su, wl, slow, total;
};

// A cell a cell pass declined, handed to the next pass: every value the cell's arithmetic reads from the state planes
// besides the obstacle rows.  Consecutive list entries are cells of unrelated instances, so gathering them again from the
// t-fastest planes would cost one 32-byte sector per scalar; a record is five 16-byte loads, consecutive across the warp.
// The previous duals (dual residual) are in the record when E <= 4 and R <= 4 (rec_duals); otherwise cell_store reads them
// from the planes.
struct __align__(16) CellRec {
  int cell, kind;                                    // b * N * T + o * T + t of the sub-batch, obstacle kind
  float px, py, cp, sp, dbar, zeta, xi0, xi1;        // as CellIn
  float lam[4], mu[4], z;                            // previous lam, mu, z of the cell
  int pad_;
};
static_assert(sizeof(CellRec) == 80, "CellRec: five 16-byte words");

struct rda_handle {
  rda_config cfg;
  rda_tunables tun;
  RobotGeom rb;
  int B, T, N, E, R;
  int sms;               // streaming multiprocessors of the device the handle was created on
  float *lam, *mu, *z, *xi, *zeta, *dis, *coef, *pref, *cur_s, *cur_u, *ref_s, *ref_speed;
  float *resi_acc, *resi_pri, *resi_dual;
  int *status, *iters, *done, *counters;
  // the declined cells of the cell passes as records, two lists of B * N * T (every cell may be declined: the cold
  // start's first iteration has no support-vertex pairs), used in turn (step_lammuz_part)
  CellRec *rec_a, *rec_b;
  char* su_ws;           // [B][su_ws_stride] global workspace of the su-QP interior point iteration (hinge slacks /
                         // multipliers)
  size_t su_ws_stride;
  // coherent first cell pass (cell_lean2.cuh; RDA_B200_LEAN2=1, E <= 4, R <= 4, static obstacles)
  int lean2;
  RobotAux ra;
  ObstacleGeom<4>* ogeo; // [B][N] per-obstacle geometry, rebuilt by every rda_begin / rda_solve
  unsigned char* feat;   // [B][N][T] support-vertex pair of the previous iteration (0: none)
  float* rot;            // [B][2][T] cos / sin of the nominal headings of this iteration
  const float *obs_A, *obs_b;
  const int *obs_kind, *obs_count;
  int obs_tv;
  float iter_threshold;
  int launches;
  int began;
  // rda_solve runs a large batch as `parts` contiguous sub-batches on as many streams (the caller's
  // and `side[]`), so that the latency-bound listed cell passes and the tail of the su-QP kernel of one
  // sub-batch overlap the kernels of the others
  cudaStream_t side[3];
  cudaEvent_t ev_fork, ev_join[3];
  // persistent single-launch ADMM for small batches (k_admm_small, SURVEY §8 f4)
  int small_mode;        // -1: batches up to small_max instances, 0: never, 1: always when the state fits (RDA_B200_SMALL)
  int small_max, small_ok, small_bulk;
  SmallLayout small_L;
  float su_prune;        // hinge pruning margin of the su-QP (su_solver.cuh; RDA_B200_SU_PRUNE, 0 = off)
  int extra_min;             // sub-batches of at least this many instances run k_cells_extra before the cooperative pass (RDA_B200_EXTRA_MIN)
  int split_min;        // smallest batch that is split (RDA_B200_SPLIT_MIN, default 2048)
  int parts;             // number of sub-batches, 1..4 (RDA_B200_SPLIT_PARTS, default 2)
  float* inst;           // [B][RDA_INST_PARAMS] per-instance limits, weights and tunables (rda_set_instance_params; allocated
                         // on the first call), read by the kernels while inst_on is set
  int inst_on;
  // robot classes (rda_set_robot_classes; allocated on the first call): tables [RDA_MAX_ROBOT_CLASSES + 1] whose slot ncls
  // holds the handle's own body, wheelbase and dynamics, and the class index [B] (rda_set_robot_class_index), read by
  // the kernels while cls_on is set and ncls > 0
  RobotGeom* cls_rb;
  RobotAux* cls_ra;
  ClassKin* cls_kin;
  int ncls;
  int* cls_idx;
  int cls_on;
  // the obstacle id of every slot in the last solve [B][N] (rda_set_obstacle_ids; allocated on the first call), held
  // while ids_on is set
  int* obs_id;
  int ids_on;
};

#define RDA_CUDA(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return (int)e_; } while (0)

namespace {

// The cooperative context of one whole warp (su_solver.cuh, coop_ipm.cuh): lanes, warp barrier, butterfly reductions.
struct WarpCtx {
  __device__ __forceinline__ int lane() const { return threadIdx.x & 31; }
  __device__ __forceinline__ int nlanes() const { return 32; }
  __device__ __forceinline__ void sync() const { __syncwarp(); }
  template <typename R> __device__ __forceinline__ R sum(R x) const {
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    return x;
  }
  template <typename R> __device__ __forceinline__ R min(R x) const {
    for (int o = 16; o > 0; o >>= 1) { R y = __shfl_xor_sync(0xffffffffu, x, o); x = y < x ? y : x; }
    return x;
  }
  template <typename R> __device__ __forceinline__ R max(R x) const {
    for (int o = 16; o > 0; o >>= 1) { R y = __shfl_xor_sync(0xffffffffu, x, o); x = y > x ? y : x; }
    return x;
  }
};

struct DevPtrs {
  float *lam, *mu, *z, *xi, *zeta, *dis, *coef, *pref, *cur_s, *cur_u, *ref_s, *ref_speed;
  float *resi_acc, *resi_pri, *resi_dual;
  int *status, *iters, *done, *counters;
  // lengths of the record lists of this sub-batch, the same for both bodies; k_finalize clears them:
  //   [0] first pass (k_cells_fast, k_cells_dr) -> searched pass (k_cells_mid, k_cells_dr_mid), in rec_b
  //   [1] searched pass -> last pass (k_cells_slow_coop, k_cells_dr_slow_coop) or k_cells_extra, in rec_a
  //   [2] coherent pass k_cells_coh -> listed first pass k_cells_fast<.., true>, in rec_a
  //   [3] k_cells_extra -> k_cells_slow_coop, in rec_b
  int* wl_count;
  const ObstacleGeom<4>* ogeo;
  unsigned char* feat;
  CellRec *rec_a, *rec_b;  // record lists of the cell passes (ping-pong, step_lammuz_part)
  char* su_ws;
  size_t su_ws_stride;
  const float *obs_A, *obs_b;
  const int *obs_kind, *obs_count;
  int obs_tv;
  int B, T, N, E, R;
  // per-instance limits, weights and tunables [B][RDA_INST_PARAMS] of this sub-batch (rda_set_instance_params), or
  // nullptr: the handle's values (the launch arguments) for every instance
  const float* inst;
  // the class index [B] of this sub-batch and the class tables [ncls + 1] (class_slot), or cls = nullptr: the
  // handle's body, wheelbase and dynamics (the launch arguments) for every instance.  The cell passes are compiled
  // for either case (template argument CLS, chosen at launch from cls).
  const int* cls;
  int ncls;
  const RobotGeom* cls_rb;
  const RobotAux* cls_ra;
  const ClassKin* cls_kin;
};

// The body of the instance in class-table slot `slot` (slot_of): its class's with a class table (CLS), else the
// handle's (rb, the launch argument).  Without a table the cells read the body from the kernel parameters as before.
template <bool CLS> __device__ __forceinline__ int slot_of(const DevPtrs& d, int b) {
  if constexpr (CLS) return class_slot(d.cls, d.ncls, b);
  else return 0;
}
template <bool CLS> __device__ __forceinline__ const RobotGeom& body_at(const DevPtrs& d, const RobotGeom& rb, int slot) {
  if constexpr (CLS) return d.cls_rb[slot];
  else return rb;
}
template <bool CLS> __device__ __forceinline__ const RobotAux& aux_at(const DevPtrs& d, const RobotAux& ra, int slot) {
  if constexpr (CLS) return d.cls_ra[slot];
  else return ra;
}

__global__ void k_begin(DevPtrs d, const float* nom_s, const float* nom_u, const float* ref_s,
                        const float* ref_speed) {
  const int T = d.T;
  const int per = 3 * (T + 1);
  const int total = d.B * per;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    d.cur_s[i] = nom_s[i];
    d.ref_s[i] = ref_s[i];
    int b = i / per, r = i - b * per;
    if (r < 2 * T) d.cur_u[b * 2 * T + r] = nom_u[b * 2 * T + r];
    if (r == 0) {
      d.ref_speed[b] = ref_speed[b];
      d.done[b] = 0; d.iters[b] = 0; d.status[b] = 0;
      d.resi_acc[2 * b] = 0; d.resi_acc[2 * b + 1] = 0;
      d.resi_pri[b] = 0; d.resi_dual[b] = 0;
    }
  }
}

// The su-QP of instance b: inputs from the persistent state (d), solve (su_solver.cuh), accepted result back.
// W is laid out by the caller (hs / hnu and the workspace may live in shared or global memory).
template <typename Real>
__device__ __forceinline__ void su_instance(const DevPtrs& d, const SuParams& Ph, int b, SuWork<Real>& W, WarpCtx& ctx) {
  // The instance's parameters in the workspace: a local copy would be held in registers across the whole solve (and
  // spill) or live in a stack frame read by local-memory loads.
  if (ctx.lane() == 0) {
    SuParams Pl = Ph;
    if (d.inst) su_params_row(Pl, d.inst + (size_t)b * RDA_INST_PARAMS);     // the instance's own row
    if (d.cls) su_params_class(Pl, d.cls_kin[class_slot(d.cls, d.ncls, b)]);  // its class's dynamics and wheelbase
    *W.par = Pl;
  }
  ctx.sync();
  const SuParams& P = *W.par;
  const int T = P.T, N = P.N, NT = N * T;
  const int lane = ctx.lane();
  const float* cs = d.cur_s + (size_t)b * 3 * (T + 1);   // [3][T+1]
  const float* cu = d.cur_u + (size_t)b * 2 * T;         // [2][T]
  const float* rf = d.ref_s + (size_t)b * 3 * (T + 1);
  for (int i = lane; i < 3 * (T + 1); i += 32) {
    int r = i / (T + 1), t = i - r * (T + 1);
    W.lins[3 * t + r] = cs[i];
    W.ref[3 * t + r] = rf[i];
  }
  for (int i = lane; i < 2 * T; i += 32) {
    int r = i / T, t = i - r * T;
    W.linu[2 * t + r] = cu[i];
    W.pref[2 * t + r] = d.pref[(size_t)b * 2 * T + i];
  }
  for (int t = lane; t < T; t += 32) W.d[t] = d.dis[(size_t)b * T + t];
  float* cf = d.coef + (size_t)b * 5 * NT;
  W.hx = cf; W.hy = cf + NT; W.hc = cf + 2 * NT;
  W.vref = d.ref_speed[b];
  ctx.sync();
  int iters = 0;
  int st = su_solve<Real, WarpCtx>(P, W, ctx, cf + 3 * NT, cf + 4 * NT, &iters);
  ctx.sync();
  // accept OPTIMAL and OPTIMAL_INACCURATE (iteration cap), else keep the previous nominal
  // ("No update of state and control vector", rda_solver.py:696-700)
  bool ok = st != 2;
  if (ok) {
    for (int i = lane; i < 3 * (T + 1); i += 32) {
      int r = i / (T + 1), t = i - r * (T + 1);
      float v = (float)W.s[3 * t + r];
      if (!isfinite(v)) ok = false;
    }
    for (int i = lane; i < 2 * T; i += 32) {
      int r = i / T, t = i - r * T;
      if (!isfinite((float)W.u[2 * t + r])) ok = false;
    }
    ok = ctx.min((int)ok) != 0;
  }
  if (ok) {
    float* ws = d.cur_s + (size_t)b * 3 * (T + 1);
    float* wu = d.cur_u + (size_t)b * 2 * T;
    for (int i = lane; i < 3 * (T + 1); i += 32) {
      int r = i / (T + 1), t = i - r * (T + 1);
      ws[i] = (float)W.s[3 * t + r];
    }
    for (int i = lane; i < 2 * T; i += 32) {
      int r = i / T, t = i - r * T;
      wu[i] = (float)W.u[2 * t + r];
    }
    for (int t = lane; t < T; t += 32) d.dis[(size_t)b * T + t] = (float)W.d[t];
  }
  if (lane == 0) {
    d.iters[b] += 1;
    int flag = 0;
    if (st == 1) flag |= RDA_ST_SU_NOT_CONVERGED;
    if (!ok) flag |= RDA_ST_SU_NONFINITE;
    if (flag) d.status[b] |= flag;
    atomicAdd(&d.counters[3], iters);
    atomicAdd(&d.counters[4], 1);
    if (W.restarts) atomicAdd(&d.counters[5], 1);      // pruned solve repeated with all hinges
  }
}

// ------------------------------------------------------------------------------------------------
// K1: su-QP, one warp per instance.
// ------------------------------------------------------------------------------------------------
template <typename Real>
__global__ void __launch_bounds__(32) k_su(DevPtrs d, SuParams P) {
  extern __shared__ __align__(16) char smem[];
  const int b = blockIdx.x;
  if (b >= d.B) return;
  if (d.done[b]) return;
  WarpCtx ctx;
  SuWork<Real> W;
  // per-hinge data stays in global memory (L2): every entry is touched only by the lane that owns
  // its stage, consecutive lanes read consecutive addresses (the compact hinge list: row k of every stage)
  su_work_layout<Real>(P.T, P.N, &W, smem, false, d.su_ws + (size_t)b * d.su_ws_stride);
  su_instance<Real>(d, P, b, W, ctx);
}

// inputs of one cell gathered from the persistent state
struct CellIn {
  int b, o, t, kind;
  size_t cell;
  float px, py, cp, sp, dbar, zeta, xi0, xi1;
  const float *A, *bb;
};

// the obstacle rows of cell (b, o, t) (as cell_load)
__device__ __forceinline__ void cell_rows(const DevPtrs& d, CellIn& c) {
  const int tc = d.obs_tv ? (c.t + 1) : 0;
  const int Tc = d.obs_tv ? (d.T + 1) : 1;
  const size_t ob = ((size_t)c.b * d.N + c.o) * Tc + tc;
  c.A = d.obs_A + ob * d.E * 2;
  c.bb = d.obs_b + ob * d.E;
}

__device__ __forceinline__ CellIn cell_load(const DevPtrs& d, long long idx) {
  const int T = d.T, N = d.N, E = d.E, NT = N * T;
  CellIn c;
  c.b = (int)(idx / NT);
  const int rem = (int)(idx - (long long)c.b * NT);
  c.o = rem / T; c.t = rem - c.o * T;
  const float* cs = d.cur_s + (size_t)c.b * 3 * (T + 1);
  c.px = cs[c.t + 1]; c.py = cs[(T + 1) + c.t + 1];
  sincosf(cs[2 * (T + 1) + c.t], &c.sp, &c.cp);      // NB column t (rda_solver.py:457-460)
  c.dbar = d.dis[(size_t)c.b * T + c.t];
  c.cell = (size_t)c.b * NT + (size_t)c.o * T + c.t;
  c.zeta = d.zeta[c.cell];
  const float* xi = d.xi + (size_t)c.b * 2 * NT;
  c.xi0 = xi[(size_t)c.o * T + c.t]; c.xi1 = xi[NT + (size_t)c.o * T + c.t];
  const int tc = d.obs_tv ? (c.t + 1) : 0;
  const int Tc = d.obs_tv ? (T + 1) : 1;
  const size_t ob = ((size_t)c.b * N + c.o) * Tc + tc;
  c.A = d.obs_A + ob * E * 2;
  c.bb = d.obs_b + ob * E;
  c.kind = d.obs_kind[(size_t)c.b * N + c.o];
  return c;
}

__device__ __forceinline__ bool rec_duals(const DevPtrs& d) { return d.E <= 4 && d.R <= 4; }

__device__ __forceinline__ CellRec cell_rec(const CellIn& c) {
  CellRec r;
  r.cell = (int)c.cell; r.kind = c.kind;
  r.px = c.px; r.py = c.py; r.cp = c.cp; r.sp = c.sp; r.dbar = c.dbar; r.zeta = c.zeta; r.xi0 = c.xi0; r.xi1 = c.xi1;
  r.pad_ = 0;
  return r;
}

__device__ __forceinline__ CellIn cell_from_rec(const DevPtrs& d, const CellRec& r) {
  const int T = d.T, NT = d.N * T;
  CellIn c;
  c.cell = (size_t)r.cell;
  c.b = r.cell / NT;
  const int rem = r.cell - c.b * NT;
  c.o = rem / T; c.t = rem - c.o * T;
  c.kind = r.kind;
  c.px = r.px; c.py = r.py; c.cp = r.cp; c.sp = r.sp; c.dbar = r.dbar; c.zeta = r.zeta; c.xi0 = r.xi0; c.xi1 = r.xi1;
  cell_rows(d, c);
  return c;
}

// the record of a cell the whole-batch pass declined, gathered again (from cache: the pass has just read the same values)
// rather than kept in registers through the cell's arithmetic
__device__ __forceinline__ CellRec cell_rec_load(const DevPtrs& d, long long idx) {
  const CellIn c = cell_load(d, idx);
  CellRec r = cell_rec(c);
  const int T = d.T, N = d.N, E = d.E, R = d.R;
  const float* lam = d.lam + ((size_t)c.b * N + c.o) * E * T + c.t;
  const float* mu = d.mu + ((size_t)c.b * N + c.o) * R * T + c.t;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    r.lam[i] = i < E ? lam[(size_t)i * T] : 0.f;
    r.mu[i] = i < R ? mu[(size_t)i * T] : 0.f;
  }
  r.z = d.z[c.cell];
  return r;
}

// the slot in `list` of the record of each lane with `need` set (one atomic per warp on *count), nullptr for the others.
// A pass that declines a listed cell copies its record over (from cache) instead of keeping it in registers through the
// cell's arithmetic.
__device__ __forceinline__ CellRec* rec_slot(bool need, CellRec* list, int* count) {
  const int lane = threadIdx.x & 31;
  const unsigned m = __ballot_sync(0xffffffffu, need);
  if (!m) return nullptr;
  const int leader = __ffs(m) - 1;
  int pos = 0;
  if (lane == leader) pos = atomicAdd(count, __popc(m));
  pos = __shfl_sync(0xffffffffu, pos, leader);
  return need ? list + pos + __popc(m & ((1u << lane) - 1)) : nullptr;
}

// write (lam, mu, z), the multiplier updates and the next su-QP's hinge inputs of one cell; prev: the cell's record, whose
// previous duals replace the planes' (the same values: a cell's duals are written only by the pass that resolves it)
__device__ __forceinline__ void cell_store(const DevPtrs& d, const CellIn& c, const CellOut<float>& out, float* hm2,
                                           float* dual, const CellRec* prev = nullptr) {
  const int T = d.T, N = d.N, E = d.E, R = d.R, NT = N * T;
  const bool pr = prev != nullptr && rec_duals(d);
  // dual residual |lam - lam_prev|^2 + |mu - mu_prev|^2 + |z - z_prev|^2 (:783-787)
  float* lam = d.lam + ((size_t)c.b * N + c.o) * E * T + c.t;
  float acc = 0.f;
  for (int i = 0; i < E; ++i) {
    float nv = out.lam[i];
    float df = nv - (pr ? prev->lam[i] : lam[(size_t)i * T]);
    acc += df * df;
    lam[(size_t)i * T] = nv;
  }
  float* mu = d.mu + ((size_t)c.b * N + c.o) * R * T + c.t;
  for (int j = 0; j < R; ++j) {
    float nv = out.mu[j];
    float df = nv - (pr ? prev->mu[j] : mu[(size_t)j * T]);
    acc += df * df;
    mu[(size_t)j * T] = nv;
  }
  float dz = out.z - (prev != nullptr ? prev->z : d.z[c.cell]);
  acc += dz * dz;
  d.z[c.cell] = out.z;
  *dual = acc;
  d.zeta[c.cell] = out.zeta_new;
  float* xi = d.xi + (size_t)c.b * 2 * NT;
  xi[(size_t)c.o * T + c.t] = out.xi0_new;
  xi[NT + (size_t)c.o * T + c.t] = out.xi1_new;
  *hm2 = out.hm0 * out.hm0 + out.hm1 * out.hm1;
  float* cf = d.coef + (size_t)c.b * 5 * NT + (size_t)c.o * T + c.t;
  cf[0] = out.ax;
  cf[NT] = out.ay;
  cf[2 * NT] = out.c0;
  cf[3 * NT] = out.gx;
  cf[4 * NT] = out.gy;
  if (c.o == 0) {
    d.pref[(size_t)c.b * 2 * T + c.t] = c.px;
    d.pref[(size_t)c.b * 2 * T + T + c.t] = c.py;
  }
}

// First pass: compile-time specialised lean solver (cell_lean.cuh), geometry in registers.
// LISTED: the cells come from the records in d.rec_a (what the coherent pass k_cells_coh declined) instead of the whole
// batch.  What this pass declines goes to d.rec_b as records.
template <int EC, int RC, bool LISTED, bool CLS>
__global__ void __launch_bounds__(128, (EC <= 4 ? 6 : 3)) k_cells_fast(DevPtrs d, RobotGeom rbh, float theta) {
  const int T = d.T, N = d.N, E = d.E, R = d.R;
  const int NT = N * T;
  const long long total = LISTED ? (long long)d.wl_count[2] : (long long)d.B * NT;
  const int lane = threadIdx.x & 31;
  for (long long base = (long long)blockIdx.x * blockDim.x; base < total; base += (long long)gridDim.x * blockDim.x) {
    const long long wi = base + threadIdx.x;
    long long idx = wi;
    bool live = idx < total;
    CellRec rec;
    if (LISTED && live) { rec = d.rec_a[wi]; idx = rec.cell; }      // listed cells are of live instances (k_cells_coh)
    int b = live ? (int)(idx / NT) : -1;
    float dual = 0.f;
    bool need = false;
    if (!LISTED && live && (d.done[b] || d.obs_count[b] == 0)) live = false;
    if (live) {
      CellIn c = LISTED ? cell_from_rec(d, rec) : cell_load(d, idx);
      const RobotGeom& rb = body_at<CLS>(d, rbh, slot_of<CLS>(d, c.b));
      // issue every global load of this cell before the arithmetic (memory-level parallelism): the
      // obstacle rows (128-bit loads when E == 4) and the previous duals needed for the residual
      float Ar[2 * EC], br[EC], lamo[EC], muo[RC];
      if (EC == 4 && E == 4) {
        const float4 a0 = __ldg(reinterpret_cast<const float4*>(c.A));
        const float4 a1 = __ldg(reinterpret_cast<const float4*>(c.A) + 1);
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(c.bb));
        Ar[0] = a0.x; Ar[1] = a0.y; Ar[2] = a0.z; Ar[3] = a0.w;
        Ar[(4) % (2 * EC)] = a1.x; Ar[(5) % (2 * EC)] = a1.y; Ar[(6) % (2 * EC)] = a1.z; Ar[(7) % (2 * EC)] = a1.w;
        br[0] = b0.x; br[1 % EC] = b0.y; br[2 % EC] = b0.z; br[3 % EC] = b0.w;
      } else {
#pragma unroll
        for (int i = 0; i < EC; ++i) {
          Ar[2 * i] = (i < E) ? __ldg(c.A + 2 * i) : 0.f;
          Ar[2 * i + 1] = (i < E) ? __ldg(c.A + 2 * i + 1) : 0.f;
          br[i] = (i < E) ? __ldg(c.bb + i) : 0.f;
        }
      }
      float zo;
      if (LISTED) {            // EC == RC == 4 (E <= 4, R <= 4): the previous duals are in the record
#pragma unroll
        for (int i = 0; i < EC; ++i) lamo[i] = (i < E) ? rec.lam[i % 4] : 0.f;
#pragma unroll
        for (int j = 0; j < RC; ++j) muo[j] = (j < R) ? rec.mu[j % 4] : 0.f;
        zo = rec.z;
      } else {
        const float* lamp = d.lam + ((size_t)c.b * N + c.o) * E * T + c.t;
        const float* mup = d.mu + ((size_t)c.b * N + c.o) * R * T + c.t;
#pragma unroll
        for (int i = 0; i < EC; ++i) lamo[i] = (i < E) ? lamp[(size_t)i * T] : 0.f;
#pragma unroll
        for (int j = 0; j < RC; ++j) muo[j] = (j < R) ? mup[(size_t)j * T] : 0.f;
        zo = d.z[c.cell];
      }
      LeanOut<EC, RC> o;
      const bool ok = cell_lean<EC, RC>(rb, c.kind, EC, Ar, br, c.px, c.py, c.cp, c.sp, c.dbar, c.zeta, c.xi0,
                                        c.xi1, theta, o);
      if (d.feat) d.feat[c.cell] = (unsigned char)(ok ? o.feat : 0);
      if (ok) {
        // dual residual |lam - lam_prev|^2 + |mu - mu_prev|^2 + |z - z_prev|^2 (:783-787)
        float* lam = d.lam + ((size_t)c.b * N + c.o) * E * T + c.t;
        float acc = 0.f;
#pragma unroll
        for (int i = 0; i < EC; ++i) {
          if (i < E) {
            const float df = o.lam[i] - lamo[i];
            acc += df * df;
            lam[(size_t)i * T] = o.lam[i];
          }
        }
        float* mu = d.mu + ((size_t)c.b * N + c.o) * R * T + c.t;
#pragma unroll
        for (int j = 0; j < RC; ++j) {
          if (j < R) {
            const float df = o.mu[j] - muo[j];
            acc += df * df;
            mu[(size_t)j * T] = o.mu[j];
          }
        }
        const float dz = o.z - zo;
        acc += dz * dz;
        d.z[c.cell] = o.z;
        dual = acc;
        d.zeta[c.cell] = o.zeta_new;
        // xi stays 0 (Hm + xi = 0 and xi was 0): nothing to write, Hm = 0
        float* cf = d.coef + (size_t)c.b * 5 * NT + (size_t)c.o * T + c.t;
        cf[0] = o.ax; cf[NT] = o.ay; cf[2 * NT] = o.c0; cf[3 * NT] = o.gx; cf[4 * NT] = o.gy;
        if (c.o == 0) {
          d.pref[(size_t)c.b * 2 * T + c.t] = c.px;
          d.pref[(size_t)c.b * 2 * T + T + c.t] = c.py;
        }
      } else {
        need = true;
      }
    }
    // the records of the cells for the second pass (one atomic per warp)
    if (CellRec* s = rec_slot(need, d.rec_b, &d.wl_count[0])) *s = LISTED ? d.rec_a[wi] : cell_rec_load(d, idx);
    const bool solved = live && !need;
    // dual-residual partial sums (Hm = 0 for every cell solved here): a warp spans at most two
    // instances when N*T >= 32
    if (LISTED) {            // listed cells are not contiguous: one atomic per cell
      if (solved) atomicAdd(&d.resi_acc[2 * b + 1], dual);
      unsigned fastl = __ballot_sync(0xffffffffu, solved);
      if (lane == 0 && fastl) atomicAdd(&d.counters[0], __popc(fastl));
      continue;
    }
    int b0 = __shfl_sync(0xffffffffu, b, 0);
    for (int pass = 0; pass < 2; ++pass) {
      bool mine = solved && ((pass == 0) ? (b == b0) : (b != b0));
      unsigned m = __ballot_sync(0xffffffffu, mine);
      if (m == 0) continue;
      float q = mine ? dual : 0.f;
      int leader = __ffs(m) - 1;
      int bl = __shfl_sync(0xffffffffu, b, leader);
      bool uniform = __all_sync(0xffffffffu, !mine || b == bl);
      if (uniform) {
        for (int o2 = 16; o2 > 0; o2 >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o2);
        if (lane == leader) atomicAdd(&d.resi_acc[2 * bl + 1], q);
      } else if (mine) {      // N*T < 32: several instances per warp
        atomicAdd(&d.resi_acc[2 * b + 1], q);
      }
    }
    unsigned fast = __ballot_sync(0xffffffffu, solved);
    if (lane == 0 && fast) atomicAdd(&d.counters[0], __popc(fast));
  }
}

// Per-obstacle geometry of the coherent pass, once per solve (static polygons; discs get ne = 0).
__global__ void k_obstacle_geometry(DevPtrs d, ObstacleGeom<4>* og) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= d.B * d.N) return;
  ObstacleGeom<4> g;
  if (d.obs_kind[i] == RDA_OBS_POLYGON && d.E <= 4) obstacle_geometry<4>(d.E, d.obs_A + (size_t)i * d.E * 2, d.obs_b + (size_t)i * d.E, g);
  else { obstacle_geometry<4>(0, nullptr, nullptr, g); }
  og[i] = g;
}

// cos / sin of the nominal headings (column t of cur_s, rda_solver.py:457-460), once per iteration for the
// coherent pass instead of one sincosf per cell
__global__ void k_heading(DevPtrs d, float* rot) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int T = d.T;
  if (i >= d.B * T) return;
  const int b = i / T, t = i - b * T;
  float sp, cp;
  sincosf(d.cur_s[(size_t)b * 3 * (T + 1) + 2 * (T + 1) + t], &sp, &cp);
  rot[(size_t)b * 2 * T + t] = cp;
  rot[(size_t)b * 2 * T + T + t] = sp;
}

// Coherent first pass (cell_lean2.cuh): one thread per cell tries the support-vertex pair of the previous
// iteration; what it declines goes to d.rec_a as records and through k_cells_fast<.., LISTED>.  Grid: one-dimensional,
// `tiles` = ceil(cells of one instance / 128) CTAs per instance, instance-major (blockIdx.x = b * tiles + tile,
// so any batch size fits; gridDim.y would cap it at 65 535) — no 64-bit index arithmetic, one instance per CTA
// (uniform early exit, one residual atomic per warp), 32-bit offsets inside the instance.
template <bool CLS>
__global__ void __launch_bounds__(128, 6) k_cells_coh(DevPtrs d, RobotGeom rbh, RobotAux rah, const float* __restrict__ rot,
                                                      float theta, float invT, int tiles) {
  constexpr int EC = 4, RC = 4;
  const int T = d.T, N = d.N, E = d.E, R = d.R, NT = N * T;
  const int b = blockIdx.x / tiles;
  if (d.done[b] || d.obs_count[b] == 0) return;             // uniform for the CTA
  // the body of the CTA's instance; the feat hint of a robot whose class changed is checked like any other
  // (cell_lean2 accepts a pair only through the separating-slab certificate)
  const int slot = slot_of<CLS>(d, b);
  const RobotGeom& rb = body_at<CLS>(d, rbh, slot);
  const RobotAux& ra = aux_at<CLS>(d, rah, slot);
  const int rem = (blockIdx.x - b * tiles) * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const bool live = rem < NT;
  float dual = 0.f;
  bool need = false, solved = false;
  CellRec rec;
  if (live) {
    int o = (int)(((float)rem + 0.5f) * invT);
    int t = rem - o * T;
    if (t < 0) { --o; t += T; } else if (t >= T) { ++o; t -= T; }
    const size_t ib = (size_t)b;
    const float* cs = d.cur_s + ib * 3 * (T + 1);
    const float* xi = d.xi + ib * 2 * NT;
    float* lamb = d.lam + ib * N * E * T;
    float* mub = d.mu + ib * N * R * T;
    float* zb = d.z + ib * NT;
    float* zetab = d.zeta + ib * NT;
    unsigned char* featb = d.feat + ib * NT;
    // every input of the cell, read coalesced here: a declined cell takes them to the later passes as its record
    const float xi0 = xi[rem], xi1 = xi[NT + rem];
    const int f = featb[rem];
    const float px = cs[t + 1], py = cs[(T + 1) + t + 1];
    const float cp = rot[ib * 2 * T + t], sp = rot[ib * 2 * T + T + t];
    const float dbar = d.dis[ib * T + t], zeta = zetab[rem];
    const int lo = o * E * T + t, mo = o * R * T + t;
    float lamo[EC], muo[RC];
#pragma unroll
    for (int i = 0; i < EC; ++i) lamo[i] = (i < E) ? lamb[lo + i * T] : 0.f;
#pragma unroll
    for (int j = 0; j < RC; ++j) muo[j] = (j < R) ? mub[mo + j * T] : 0.f;
    const float zo = zb[rem];
    int nf = -1;
    if (xi0 == 0.f && xi1 == 0.f && (f & RDA_FEAT_VALID)) {
      const ObstacleGeom<4>& og = d.ogeo[ib * N + o];         // same address for the T cells of an obstacle
      LeanOut<EC, RC> r;
      nf = cell_lean2<EC, RC>(rb, ra, og, f, px, py, cp, sp, dbar, zeta, theta, r);
      if (nf >= 0) {
        float acc = 0.f;
#pragma unroll
        for (int i = 0; i < EC; ++i) {
          if (i < E) { const float df = r.lam[i] - lamo[i]; acc += df * df; lamb[lo + i * T] = r.lam[i]; }
        }
#pragma unroll
        for (int j = 0; j < RC; ++j) {
          if (j < R) { const float df = r.mu[j] - muo[j]; acc += df * df; mub[mo + j * T] = r.mu[j]; }
        }
        const float dz = r.z - zo;
        acc += dz * dz;
        zb[rem] = r.z;
        dual = acc;
        zetab[rem] = r.zeta_new;
        float* cf = d.coef + ib * 5 * NT + rem;
        cf[0] = r.ax; cf[NT] = r.ay; cf[2 * NT] = r.c0; cf[3 * NT] = r.gx; cf[4 * NT] = r.gy;
        if (o == 0) {
          d.pref[ib * 2 * T + t] = px;
          d.pref[ib * 2 * T + T + t] = py;
        }
        if (nf != f) featb[rem] = (unsigned char)nf;
        solved = true;
      }
    }
    need = nf < 0;
    if (need) {
      rec.cell = b * NT + rem; rec.kind = d.obs_kind[ib * N + o];
      rec.px = px; rec.py = py; rec.cp = cp; rec.sp = sp; rec.dbar = dbar; rec.zeta = zeta; rec.xi0 = xi0; rec.xi1 = xi1;
#pragma unroll
      for (int i = 0; i < 4; ++i) { rec.lam[i] = lamo[i]; rec.mu[i] = muo[i]; }
      rec.z = zo; rec.pad_ = 0;
    }
  }
  if (CellRec* s = rec_slot(need, d.rec_a, &d.wl_count[2])) *s = rec;
  const unsigned fast = __ballot_sync(0xffffffffu, solved);
  if (fast) {
    float q = dual;
    for (int o2 = 16; o2 > 0; o2 >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o2);
    if (lane == 0) { atomicAdd(&d.resi_acc[2 * b + 1], q); atomicAdd(&d.counters[0], __popc(fast)); }
  }
}

// The rows of an obstacle copy into local arrays BEFORE the geometry: cell_front walks the rows in a loop that ends at the
// first zero row, so the compiler cannot hoist its loads — four dependent round trips to L2/HBM per cell.  With E == 4 (every
// reference example) three 128-bit loads fetch all of them at once; other row counts are loaded row by row up front.
struct RowsLocal { float A[2 * RDA_MAX_EDGE], b[RDA_MAX_EDGE]; };
__device__ __forceinline__ void rows_preload(const DevPtrs& d, const CellIn& c, RowsLocal& r) {
  if (d.E == 4) {
    const float4 a0 = __ldg(reinterpret_cast<const float4*>(c.A));
    const float4 a1 = __ldg(reinterpret_cast<const float4*>(c.A) + 1);
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(c.bb));
    r.A[0] = a0.x; r.A[1] = a0.y; r.A[2] = a0.z; r.A[3] = a0.w; r.A[4] = a1.x; r.A[5] = a1.y; r.A[6] = a1.z; r.A[7] = a1.w;
    r.b[0] = b0.x; r.b[1] = b0.y; r.b[2] = b0.z; r.b[3] = b0.w;
  } else {
#pragma unroll
    for (int i = 0; i < RDA_MAX_EDGE; ++i) {
      const bool in = i < d.E;
      r.A[2 * i] = in ? __ldg(c.A + 2 * i) : 0.f;
      r.A[2 * i + 1] = in ? __ldg(c.A + 2 * i + 1) : 0.f;
      r.b[i] = in ? __ldg(c.bb + i) : 0.f;
    }
  }
}

// Second pass: the searched closed forms (vertex / edge contact, overlap cases) for the cells the first pass declined (records
// in d.rec_b), one thread per record; the records of what is still unresolved go to d.rec_a.
template <bool CLS>
__global__ void __launch_bounds__(128) k_cells_mid(DevPtrs d, RobotGeom rbh, float ro2h, float theta) {
  const int count = d.wl_count[0];
  const int lane = threadIdx.x & 31;
  for (int base = blockIdx.x * blockDim.x; base < count; base += gridDim.x * blockDim.x) {
    const int wi = base + threadIdx.x;
    const bool live = wi < count;
    bool need = false;
    if (live) {
      CellIn c = cell_from_rec(d, d.rec_b[wi]);
      const float ro2 = inst_ro2(d.inst, c.b, ro2h);
      const RobotGeom& rb = body_at<CLS>(d, rbh, slot_of<CLS>(d, c.b));
      RowsLocal rows;
      rows_preload(d, c, rows);
      CellWork<float> w;
      cell_front<float>(rb, c.kind, d.E, rows.A, rows.b, c.px, c.py, c.cp, c.sp, c.dbar, c.zeta, c.xi0, c.xi1, ro2, w);
      if (w.have) {
        CellOut<float> out;
        cell_back<float>(rb, w, c.zeta, theta, out);
        float hm2 = 0.f, dual = 0.f;
        cell_store(d, c, out, &hm2, &dual, d.rec_b + wi);
        atomicAdd(&d.resi_acc[2 * c.b], hm2);
        atomicAdd(&d.resi_acc[2 * c.b + 1], dual);
      } else {
        need = true;
      }
    }
    if (CellRec* s = rec_slot(need, d.rec_a, &d.wl_count[1])) *s = d.rec_b[wi];
    unsigned solved = __ballot_sync(0xffffffffu, live && !need);
    if (lane == 0 && solved) atomicAdd(&d.counters[0], __popc(solved));
  }
}

// ------------------------------------------------------------------------------------------------
// Disc body (car_tuple.cone_type 'norm2', rda_solver.py:1034-1039; cell_disc_robot.cuh).  Three passes that hand
// their declined cells on as records, like the polygon passes: k_cells_dr solves every cell whose hinge is inactive in
// closed form (one thread per cell, coalesced like the first polygon pass) and lists the rest in d.rec_b;
// k_cells_dr_mid tries the searched closed forms of the listed cells, one cell per thread, and lists what is left in
// d.rec_a; k_cells_dr_slow_coop runs the two-cone barrier programmes of those, one cell per warp.
// ------------------------------------------------------------------------------------------------
template <bool CLS>
__global__ void __launch_bounds__(128) k_cells_dr(DevPtrs d, RobotGeom rbh, float ro2h, float theta) {
  const int NT = d.N * d.T;
  const long long total = (long long)d.B * NT;
  const int lane = threadIdx.x & 31;
  for (long long base = (long long)blockIdx.x * blockDim.x; base < total; base += (long long)gridDim.x * blockDim.x) {
    const long long idx = base + threadIdx.x;
    bool live = idx < total;
    const int b = live ? (int)(idx / NT) : -1;
    if (live && (d.done[b] || d.obs_count[b] == 0)) live = false;
    bool need = false;
    if (live) {
      CellIn c = cell_load(d, idx);
      const float ro2 = inst_ro2(d.inst, c.b, ro2h);
      const RobotGeom& rb = body_at<CLS>(d, rbh, slot_of<CLS>(d, c.b));
      CellWork<float> w;
      // first pass: the closed forms of the inactive hinge only (the searched ones run per listed cell in k_cells_dr_mid)
      cell_front_dr<float>(rb, c.kind, d.E, c.A, c.bb, c.px, c.py, c.cp, c.sp, c.dbar, c.zeta, c.xi0, c.xi1, ro2, w, false);
      if (w.have) {
        CellOut<float> out;
        cell_back_dr<float>(rb, w, c.zeta, theta, out);
        float hm2 = 0.f, dual = 0.f;
        cell_store(d, c, out, &hm2, &dual);
        atomicAdd(&d.resi_acc[2 * c.b], hm2);
        atomicAdd(&d.resi_acc[2 * c.b + 1], dual);
      } else {
        need = true;
      }
    }
    if (CellRec* s = rec_slot(need, d.rec_b, &d.wl_count[0])) *s = cell_rec_load(d, idx);
    const unsigned solved = __ballot_sync(0xffffffffu, live && !need);
    if (lane == 0 && solved) atomicAdd(&d.counters[0], __popc(solved));
  }
}

// Disc body, second pass: the searched closed forms (edge and point contacts, overlap cases; point contacts in float64) for the
// cells the first pass listed (records in d.rec_b), one thread per record; the records of what is left (0.01 % of the cells
// on the bench workload) go to the cooperative barrier pass through d.rec_a.
template <bool CLS>
__global__ void __launch_bounds__(128) k_cells_dr_mid(DevPtrs d, RobotGeom rbh, float ro2h, float theta) {
  const int count = d.wl_count[0];
  for (int base = blockIdx.x * blockDim.x; base < count; base += gridDim.x * blockDim.x) {
    const int wi = base + threadIdx.x;
    bool need = false;
    if (wi < count) {
      CellIn c = cell_from_rec(d, d.rec_b[wi]);
      const float ro2 = inst_ro2(d.inst, c.b, ro2h);
      const RobotGeom& rb = body_at<CLS>(d, rbh, slot_of<CLS>(d, c.b));
      CellWork<float> w;
      cell_front_dr<float>(rb, c.kind, d.E, c.A, c.bb, c.px, c.py, c.cp, c.sp, c.dbar, c.zeta, c.xi0, c.xi1, ro2, w, true);
      if (w.have) {
        CellOut<float> out;
        cell_back_dr<float>(rb, w, c.zeta, theta, out);
        float hm2 = 0.f, dual = 0.f;
        cell_store(d, c, out, &hm2, &dual, d.rec_b + wi);
        atomicAdd(&d.resi_acc[2 * c.b], hm2);
        atomicAdd(&d.resi_acc[2 * c.b + 1], dual);
        atomicAdd(&d.counters[0], 1);
      } else {
        need = true;
      }
    }
    if (CellRec* s = rec_slot(need, d.rec_a, &d.wl_count[1])) *s = d.rec_b[wi];
  }
}

// warps (cells) per CTA of the warp-cooperative passes k_cells_dr_slow_coop and k_cells_slow_coop
constexpr int COOP_WARPS = 4;

// one cell per WARP: the two-cone barrier iterations spread over the lanes, the problem in shared memory
template <bool CLS>
__global__ void __launch_bounds__(32 * COOP_WARPS) k_cells_dr_slow_coop(DevPtrs d, RobotGeom rbh, float ro2h, float theta) {
  __shared__ DiscSlowStore store[COOP_WARPS];
  const int count = d.wl_count[1];          // what k_cells_dr_mid left, in d.rec_a
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  DiscSlowStore& S = store[warp];
  WarpCtx ctx;
  for (int wi = blockIdx.x * COOP_WARPS + warp; wi < count; wi += gridDim.x * COOP_WARPS) {
    CellIn c;
    CellWork<float> w;
    w.have = false;
    int slot = 0;
    if (lane == 0) c = cell_from_rec(d, d.rec_a[wi]);
    if (CLS) slot = __shfl_sync(0xffffffffu, slot_of<CLS>(d, lane == 0 ? c.b : 0), 0);   // every lane takes part in the barrier solve
    const RobotGeom& rb = body_at<CLS>(d, rbh, slot);
    if (lane == 0) {
      const float ro2 = inst_ro2(d.inst, c.b, ro2h);
      // geometry only: the closed forms have been tried by k_cells_dr_mid
      cell_front_dr<float>(rb, c.kind, d.E, c.A, c.bb, c.px, c.py, c.cp, c.sp, c.dbar, c.zeta, c.xi0, c.xi1, ro2, w, false);
    }
    const int have = __shfl_sync(0xffffffffu, (int)w.have, 0);
    if (!have) {
      __syncwarp();
      cell_slow_dr<float, WarpCtx>(rb, w, S, ctx);
      __syncwarp();
    }
    if (lane == 0) {
      CellOut<float> out;
      cell_back_dr<float>(rb, w, c.zeta, theta, out);
      float hm2 = 0.f, dual = 0.f;
      if (out.path == CELL_FAILED) {
        // "Update Lam Mu Fail": previous duals kept, residual inf (:791-793)
        dual = INFINITY;
        atomicOr(&d.status[c.b], RDA_ST_CELL_FALLBACK);
      } else {
        // previous duals from the planes (the same values): read from the record, they stay live across the barrier
        // solve's calls and add 48 bytes of spills to this lane
        cell_store(d, c, out, &hm2, &dual);
      }
      atomicAdd(&d.resi_acc[2 * c.b], hm2);
      atomicAdd(&d.resi_acc[2 * c.b + 1], dual);
      atomicAdd(&d.counters[out.path == CELL_FAILED ? 2 : 1], 1);
    }
    __syncwarp();
  }
}

// Last pass, first half (with the cooperative interior point pass): the closed forms only the rare cells need (robot edge x
// obstacle edge, weighted maxima on monotone edges: cell_front<EXTRA>) for the cells the searched pass listed, one THREAD per
// cell — they resolve ~90 % of that list; the records of what is left (~0.01 % of all cells) go to k_cells_slow_coop through
// d.rec_b, which the searched pass has consumed by now.  (Doing these closed forms in lane 0 of the cooperative kernel was slow at
// 16 384 unique instances: ten thousand warps each waiting for one serial lane.)
template <bool CLS>
__global__ void __launch_bounds__(128) k_cells_extra(DevPtrs d, RobotGeom rbh, float ro2h, float theta) {
  const int count = d.wl_count[1];
  for (int base = blockIdx.x * blockDim.x; base < count; base += gridDim.x * blockDim.x) {
    const int wi = base + threadIdx.x;
    bool need = false;
    if (wi < count) {
      CellIn c = cell_from_rec(d, d.rec_a[wi]);
      const float ro2 = inst_ro2(d.inst, c.b, ro2h);
      const RobotGeom& rb = body_at<CLS>(d, rbh, slot_of<CLS>(d, c.b));
      RowsLocal rows;
      rows_preload(d, c, rows);
      CellWork<float> w;
      cell_front<float, true>(rb, c.kind, d.E, rows.A, rows.b, c.px, c.py, c.cp, c.sp, c.dbar, c.zeta, c.xi0, c.xi1, ro2, w);
      if (w.have) {
        CellOut<float> out;
        cell_back<float>(rb, w, c.zeta, theta, out);
        float hm2 = 0.f, dual = 0.f;
        cell_store(d, c, out, &hm2, &dual, d.rec_a + wi);
        atomicAdd(&d.resi_acc[2 * c.b], hm2);
        atomicAdd(&d.resi_acc[2 * c.b + 1], dual);
        atomicAdd(&d.counters[1], 1);
      } else {
        need = true;
      }
    }
    if (CellRec* s = rec_slot(need, d.rec_b, &d.wl_count[3])) *s = d.rec_a[wi];
  }
}

// Last pass, warp-cooperative: ONE cell per warp, the interior point iteration of coop_ipm.cuh spread over the lanes (rows,
// vector components and Newton-matrix entries), the problem in shared memory.  Round 1 measured it slower than one thread per
// cell — with 5 % of the cells in this pass; since the closed forms of round 2 leave 0.1 % (~13 000 cells at 16 384
// instances, three waves of warps) the pass is a pure latency tail, which is what cooperation shortens (DESIGN.md §3.1).
template <bool CLS>
__global__ void __launch_bounds__(32 * COOP_WARPS) k_cells_slow_coop(DevPtrs d, RobotGeom rbh, float ro2h, float theta, int from_extra) {
  __shared__ CellSlowStore store[COOP_WARPS];
  // from_extra: the records k_cells_extra left — d.rec_b (the first pass' list, consumed by now) with its own counter;
  // otherwise the searched pass' own leftovers in d.rec_a (small batches: one launch less, lane 0 runs the EXTRA closed forms)
  const int count = from_extra ? d.wl_count[3] : d.wl_count[1];
  const CellRec* list = from_extra ? d.rec_b : d.rec_a;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  CellSlowStore& S = store[warp];
  WarpCtx ctx;
  for (int wi = blockIdx.x * COOP_WARPS + warp; wi < count; wi += gridDim.x * COOP_WARPS) {
    CellIn c;
    CellWork<float> w;
    w.have = false;
    int slot = 0;
    if (lane == 0) c = cell_from_rec(d, list[wi]);
    if (CLS) slot = __shfl_sync(0xffffffffu, slot_of<CLS>(d, lane == 0 ? c.b : 0), 0);   // every lane takes part in the interior point solve
    const RobotGeom& rb = body_at<CLS>(d, rbh, slot);
    if (lane == 0) {
      const float ro2 = inst_ro2(d.inst, c.b, ro2h);
      cell_front<float, true>(rb, c.kind, d.E, c.A, c.bb, c.px, c.py, c.cp, c.sp, c.dbar, c.zeta, c.xi0, c.xi1, ro2, w);
    }
    const int have = __shfl_sync(0xffffffffu, (int)w.have, 0);
    if (!have) {
      __syncwarp();
      cell_slow<float, WarpCtx>(rb, w, S, ctx);
      __syncwarp();
    }
    if (lane == 0) {
      CellOut<float> out;
      cell_back<float>(rb, w, c.zeta, theta, out);
      float hm2 = 0.f, dual = 0.f;
      if (out.path == CELL_FAILED) {
        dual = INFINITY;
        atomicOr(&d.status[c.b], RDA_ST_CELL_FALLBACK);
      } else {
        cell_store(d, c, out, &hm2, &dual, list + wi);
      }
      atomicAdd(&d.resi_acc[2 * c.b], hm2);
      atomicAdd(&d.resi_acc[2 * c.b + 1], dual);
      atomicAdd(&d.counters[out.path == CELL_FAILED ? 2 : 1], 1);
    }
    __syncwarp();
  }
}

// per instance: residuals (:688, :735-739), early stop (:594-596), empty-list quirk (:564-568)
__device__ __forceinline__ void finalize_instance(const DevPtrs& d, const RobotGeom& rbh, float thr, int b) {
  const int T = d.T, N = d.N, NT = N * T, R = d.R;
  const float* rh = d.cls ? d.cls_rb[class_slot(d.cls, d.ncls, b)].h : rbh.h;
  float pri = 0.f, dual = 0.f;
  if (N > 0 && d.obs_count[b] != 0) {
    pri = sqrtf(d.resi_acc[2 * b]);
    dual = d.resi_acc[2 * b + 1] / (float)N;
  } else if (N > 0) {
    // obstacle list empty: only the LAST slot's lam'A and lam'b are cleared (loop-variable leak)
    int o = N - 1;
    float* cf = d.coef + (size_t)b * 5 * NT + (size_t)o * T;
    for (int t = 0; t < T; ++t) {
      const float* mu = d.mu + ((size_t)b * N + o) * R * T + t;
      float muh = 0.f;
      for (int j = 0; j < R; ++j) muh += mu[(size_t)j * T] * rh[j];
      size_t cell = (size_t)b * NT + (size_t)o * T + t;
      cf[t] = 0.f; cf[NT + t] = 0.f;
      cf[2 * NT + t] = -muh - d.z[cell] + d.zeta[cell];
    }
  }
  d.resi_acc[2 * b] = 0.f; d.resi_acc[2 * b + 1] = 0.f;
  d.resi_pri[b] = pri; d.resi_dual[b] = dual;
  if (dual < thr && pri < thr) { d.done[b] = 1; d.status[b] |= RDA_ST_EARLY_STOP; }
}

__global__ void k_finalize(DevPtrs d, RobotGeom rb, float thr) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b == 0) { d.wl_count[0] = 0; d.wl_count[1] = 0; d.wl_count[2] = 0; d.wl_count[3] = 0; }   // record lists consumed
  if (b >= d.B) return;
  if (d.done[b]) return;
  finalize_instance(d, rb, thr, b);
}

// ------------------------------------------------------------------------------------------------
// SURVEY.md §8 f4: the whole ADMM loop of one (small) instance in ONE launch, one CTA per instance, every piece of
// warm-start state staged in shared memory for the duration of the solve (HBM is touched once on the way in and
// once on the way out).  Warp 0 runs the su-QP (same code as k_su), all threads the closed forms of the cells (one
// cell per thread), all warps the interior point iteration of the cells those leave (one cell per warp, as
// k_cells_slow_coop), thread 0 the residual / early-stop rule.  The kernel reuses the device functions of the streaming kernels through a DevPtrs whose
// pointers address shared memory, so the arithmetic is identical; instances progress independently (no grid-wide
// barrier between the ADMM phases).
// ------------------------------------------------------------------------------------------------
// su_bytes, su_gbytes: the su-QP workspace and its per-hinge arrays (su_work_bytes with hinge_arrays = false)
static SmallLayout small_layout(int T, int N, int E, int R, size_t su_bytes, size_t su_gbytes) {
  SmallLayout L;
  size_t o = 0;
  auto take = [&](size_t bytes) { o = (o + 15) & ~(size_t)15; size_t r = o; o += bytes; return (int)r; };
  const size_t NT = (size_t)N * T;
  L.lam = take(4 * N * E * T); L.mu = take(4 * N * R * T); L.z = take(4 * NT); L.xi = take(8 * NT); L.zeta = take(4 * NT);
  L.dis = take(4 * T); L.coef = take(20 * NT); L.pref = take(8 * T); L.cur_s = take(12 * (T + 1)); L.cur_u = take(8 * T);
  L.ref_s = take(12 * (T + 1)); L.misc = take(128); L.hs = take(su_gbytes); L.su = take(su_bytes);
  // which cells the closed forms left (one flag per cell) and one interior point problem per warp (cooperative pass)
  L.wl = take(4 * (NT + 1)); L.slow = take(4 * sizeof(CellSlowStore));
  L.total = (int)((o + 15) & ~(size_t)15);
  return L;
}


// ---- bulk asynchronous copies (TMA engine, 1-D: no tensor map) with mbarrier completion -----------------------
// Used by the persistent kernel to stage an instance's warm-start state into shared memory and back: each array is one
// contiguous, 16-byte aligned block per instance, which is exactly the shape cp.async.bulk moves without any thread
// touching the data (SASS: UBLKCP).
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  unsigned ok = 0;
  do {
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void bulk_s2g(void* dst, const void* src, unsigned bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit_wait() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// Two resident CTAs per SM (small_max, and the staged state in shared memory): the register budget that leaves lets ptxas
// keep the su-QP's working set in registers (without the bound it settles at 168 and spills in the float64 build).
template <typename Real, bool CLS>
__global__ void __launch_bounds__(128, 2) k_admm_small(DevPtrs d, SuParams Ph, RobotGeom rbh, float theta, float thr,
                                                    int iter_num, SmallLayout L, const float* nom_s, const float* nom_u,
                                                    const float* ref_s, const float* ref_speed, rda_outputs out, int use_bulk) {
  extern __shared__ __align__(16) char smem[];
  const int b = blockIdx.x;
  if (b >= d.B) return;
  const int T = d.T, N = d.N, E = d.E, R = d.R, NT = N * T, tid = threadIdx.x, nth = blockDim.x;
  // the su-QP parameters and the cells' ro2: the handle's, or the instance's own row (rda_set_instance_params), read once
  SuParams P = Ph;
  if (d.inst) su_params_row(P, d.inst + (size_t)b * RDA_INST_PARAMS);
  const float ro2 = P.ro2;
  // the body, dynamics and wheelbase: the handle's, or the instance's class (rda_set_robot_classes), read once
  const int slot = slot_of<CLS>(d, b);
  const RobotGeom& rb = body_at<CLS>(d, rbh, slot);
  if (CLS) su_params_class(P, d.cls_kin[slot]);
  // ---- a one-instance view of the persistent state in shared memory ----
  DevPtrs ds = d;
  ds.B = 1;
  ds.inst = nullptr;      // P holds the row
  ds.cls = nullptr;       // ... and the class's kinematics; rb is its body
  ds.lam = (float*)(smem + L.lam); ds.mu = (float*)(smem + L.mu); ds.z = (float*)(smem + L.z); ds.xi = (float*)(smem + L.xi);
  ds.zeta = (float*)(smem + L.zeta); ds.dis = (float*)(smem + L.dis); ds.coef = (float*)(smem + L.coef);
  ds.pref = (float*)(smem + L.pref); ds.cur_s = (float*)(smem + L.cur_s); ds.cur_u = (float*)(smem + L.cur_u);
  ds.ref_s = (float*)(smem + L.ref_s);
  float* misc = (float*)(smem + L.misc);
  ds.resi_acc = misc; ds.resi_pri = misc + 2; ds.resi_dual = misc + 3; ds.ref_speed = misc + 4;
  ds.status = (int*)(misc + 5); ds.iters = (int*)(misc + 6); ds.done = (int*)(misc + 7);
  const size_t Tc = d.obs_tv ? T + 1 : 1;
  ds.obs_A = d.obs_A ? d.obs_A + (size_t)b * N * Tc * E * 2 : nullptr;
  ds.obs_b = d.obs_b ? d.obs_b + (size_t)b * N * Tc * E : nullptr;
  ds.obs_kind = d.obs_kind ? d.obs_kind + (size_t)b * N : nullptr;
  ds.obs_count = d.obs_count ? d.obs_count + b : nullptr;
  auto copy_in = [&](float* dst, const float* src, int n) { for (int i = tid; i < n; i += nth) dst[i] = src[i]; };
  auto copy_out = [&](float* dst, const float* src, int n) { for (int i = tid; i < n; i += nth) dst[i] = src[i]; };
  unsigned long long* bar = (unsigned long long*)(misc + 8);
  if (use_bulk) {
    // the six per-cell arrays (16-byte multiples, checked on the host) through the TMA engine, the rest by the threads
    if (tid == 0) mbar_init(bar, 1);
    __syncthreads();
    if (tid == 0) {
      const unsigned nle = N * E * T * 4, nmu = N * R * T * 4, nc = NT * 4;
      mbar_expect_tx(bar, nle + nmu + nc + 2 * nc + nc + 5 * nc);
      bulk_g2s(ds.lam, d.lam + (size_t)b * N * E * T, nle, bar);
      bulk_g2s(ds.mu, d.mu + (size_t)b * N * R * T, nmu, bar);
      bulk_g2s(ds.z, d.z + (size_t)b * NT, nc, bar);
      bulk_g2s(ds.xi, d.xi + (size_t)b * 2 * NT, 2 * nc, bar);
      bulk_g2s(ds.zeta, d.zeta + (size_t)b * NT, nc, bar);
      bulk_g2s(ds.coef, d.coef + (size_t)b * 5 * NT, 5 * nc, bar);
    }
  } else {
    copy_in(ds.lam, d.lam + (size_t)b * N * E * T, N * E * T); copy_in(ds.mu, d.mu + (size_t)b * N * R * T, N * R * T);
    copy_in(ds.z, d.z + (size_t)b * NT, NT); copy_in(ds.xi, d.xi + (size_t)b * 2 * NT, 2 * NT);
    copy_in(ds.zeta, d.zeta + (size_t)b * NT, NT); copy_in(ds.coef, d.coef + (size_t)b * 5 * NT, 5 * NT);
  }
  copy_in(ds.dis, d.dis + (size_t)b * T, T); copy_in(ds.pref, d.pref + (size_t)b * 2 * T, 2 * T);
  copy_in(ds.cur_s, nom_s + (size_t)b * 3 * (T + 1), 3 * (T + 1)); copy_in(ds.cur_u, nom_u + (size_t)b * 2 * T, 2 * T);
  copy_in(ds.ref_s, ref_s + (size_t)b * 3 * (T + 1), 3 * (T + 1));
  if (tid == 0) {
    misc[0] = 0.f; misc[1] = 0.f; misc[2] = 0.f; misc[3] = 0.f; misc[4] = ref_speed[b];
    ds.status[0] = 0; ds.iters[0] = 0; ds.done[0] = 0;
  }
  if (use_bulk) mbar_wait(bar, 0);
  __syncthreads();
  const bool has_obs = N > 0 && ds.obs_count[0] != 0;
  for (int it = 0; it < iter_num; ++it) {
    if (tid < 32) {
      WarpCtx ctx;
      SuWork<Real> W;
      su_work_layout<Real>(T, N, &W, smem + L.su, false, smem + L.hs);
      su_instance<Real>(ds, P, 0, W, ctx);
    }
    __syncthreads();
    if (has_obs) {
      // Residual terms are summed in a fixed order (per thread, then over the lanes, then warp by warp) so that a solve
      // reproduces its residuals bit for bit.  wl[1 + idx]: whether cell idx is left to the interior point pass below.
      int* wl = (int*)(smem + L.wl);
      const int warp = tid >> 5, lane = tid & 31, nwarps = nth >> 5;
      float hm2s = 0.f, duals = 0.f;
      for (int idx = tid; idx < NT; idx += nth) {
        CellIn c = cell_load(ds, idx);
        CellWork<float> w;
        cell_front<float, true>(rb, c.kind, E, c.A, c.bb, c.px, c.py, c.cp, c.sp, c.dbar, c.zeta, c.xi0, c.xi1, ro2, w);
        wl[1 + idx] = !w.have;
        if (!w.have) continue;
        CellOut<float> o;
        cell_back<float>(rb, w, c.zeta, theta, o);
        float hm2 = 0.f, dual = 0.f;
        cell_store(ds, c, o, &hm2, &dual);
        hm2s += hm2;
        duals += dual;
        atomicAdd(&d.counters[0], 1);
      }
      // the cells the closed forms left, in index order, the k-th to warp k % nwarps: interior point iteration spread over
      // the lanes (coop_ipm.cuh), the problem in shared memory — as k_cells_slow_coop of the streaming path
      __syncthreads();
      CellSlowStore& S = ((CellSlowStore*)(smem + L.slow))[warp];
      WarpCtx ctx;
      int rank = 0;
      for (int base = 0; base < NT; base += 32) {
        unsigned m = __ballot_sync(0xffffffffu, base + lane < NT && wl[1 + base + lane]);
        for (; m; m &= m - 1, ++rank) {
          if (rank % nwarps != warp) continue;
          const int idx = base + __ffs(m) - 1;
          CellIn c;
          CellWork<float> w;
          w.have = false;
          if (lane == 0) {
            c = cell_load(ds, idx);
            cell_front<float, true>(rb, c.kind, E, c.A, c.bb, c.px, c.py, c.cp, c.sp, c.dbar, c.zeta, c.xi0, c.xi1, ro2, w);
          }
          __syncwarp();
          cell_slow<float, WarpCtx>(rb, w, S, ctx);
          __syncwarp();
          if (lane == 0) {
            CellOut<float> o;
            cell_back<float>(rb, w, c.zeta, theta, o);
            float hm2 = 0.f, dual = 0.f;
            if (o.path == CELL_FAILED) {
              dual = INFINITY;
              atomicOr(&ds.status[0], RDA_ST_CELL_FALLBACK);
            } else {
              cell_store(ds, c, o, &hm2, &dual);
            }
            hm2s += hm2;
            duals += dual;
            atomicAdd(&d.counters[o.path == CELL_FAILED ? 2 : 1], 1);
          }
          __syncwarp();
        }
      }
      for (int o2 = 16; o2 > 0; o2 >>= 1) {
        hm2s += __shfl_xor_sync(0xffffffffu, hm2s, o2);
        duals += __shfl_xor_sync(0xffffffffu, duals, o2);
      }
      float* part = misc + 16;                       // [warp][2] sums of the (at most 4) warps
      if (lane == 0) { part[2 * warp] = hm2s; part[2 * warp + 1] = duals; }
      __syncthreads();
      if (tid == 0) {
        float hm2 = 0.f, dual = 0.f;
        for (int k = 0; k < nwarps; ++k) { hm2 += part[2 * k]; dual += part[2 * k + 1]; }
        ds.resi_acc[0] = hm2;
        ds.resi_acc[1] = dual;
      }
    }
    __syncthreads();
    if (tid == 0) finalize_instance(ds, rb, thr, 0);
    __syncthreads();
    if (ds.done[0]) break;
  }
  // ---- state and results back to HBM ----
  if (use_bulk) {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy writes visible to the copy engine
    __syncthreads();
    if (tid == 0) {
      const unsigned nle = N * E * T * 4, nmu = N * R * T * 4, nc = NT * 4;
      bulk_s2g(d.lam + (size_t)b * N * E * T, ds.lam, nle);
      bulk_s2g(d.mu + (size_t)b * N * R * T, ds.mu, nmu);
      bulk_s2g(d.z + (size_t)b * NT, ds.z, nc);
      bulk_s2g(d.xi + (size_t)b * 2 * NT, ds.xi, 2 * nc);
      bulk_s2g(d.zeta + (size_t)b * NT, ds.zeta, nc);
      bulk_s2g(d.coef + (size_t)b * 5 * NT, ds.coef, 5 * nc);
      bulk_commit_wait();
    }
  } else {
    copy_out(d.lam + (size_t)b * N * E * T, ds.lam, N * E * T); copy_out(d.mu + (size_t)b * N * R * T, ds.mu, N * R * T);
    copy_out(d.z + (size_t)b * NT, ds.z, NT); copy_out(d.xi + (size_t)b * 2 * NT, ds.xi, 2 * NT);
    copy_out(d.zeta + (size_t)b * NT, ds.zeta, NT); copy_out(d.coef + (size_t)b * 5 * NT, ds.coef, 5 * NT);
  }
  copy_out(d.dis + (size_t)b * T, ds.dis, T); copy_out(d.pref + (size_t)b * 2 * T, ds.pref, 2 * T);
  copy_out(d.cur_s + (size_t)b * 3 * (T + 1), ds.cur_s, 3 * (T + 1)); copy_out(d.cur_u + (size_t)b * 2 * T, ds.cur_u, 2 * T);
  copy_out(d.ref_s + (size_t)b * 3 * (T + 1), ds.ref_s, 3 * (T + 1));
  copy_out((float*)out.s_opt + (size_t)b * 3 * (T + 1), ds.cur_s, 3 * (T + 1));
  copy_out((float*)out.u_opt + (size_t)b * 2 * T, ds.cur_u, 2 * T);
  if (tid == 0) {
    d.ref_speed[b] = misc[4];
    d.resi_pri[b] = misc[2]; d.resi_dual[b] = misc[3]; d.resi_acc[2 * b] = 0.f; d.resi_acc[2 * b + 1] = 0.f;
    d.status[b] = ds.status[0]; d.iters[b] = ds.iters[0]; d.done[b] = ds.done[0];
    ((float*)out.resi_pri)[b] = misc[2]; ((float*)out.resi_dual)[b] = misc[3];
    ((int*)out.status)[b] = ds.status[0]; ((int*)out.iters)[b] = ds.iters[0];
  }
}

__global__ void k_finish(DevPtrs d, rda_outputs o) {
  const int T = d.T;
  const int per = 3 * (T + 1);
  const int total = d.B * per;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    o.s_opt[i] = d.cur_s[i];
    int b = i / per, r = i - b * per;
    if (r < 2 * T) o.u_opt[b * 2 * T + r] = d.cur_u[b * 2 * T + r];
    if (r == 0) {
      o.resi_pri[b] = d.resi_pri[b]; o.resi_dual[b] = d.resi_dual[b];
      o.status[b] = d.status[b]; o.iters[b] = d.iters[b];
    }
  }
}

// RDA_solver.reset (:1060-1068): lam'A = 0, lam'b = 0; mu, z, zeta, xi are NOT cleared.
__global__ void k_reset(DevPtrs d, RobotGeom rbh) {
  const int T = d.T, N = d.N, NT = N * T, R = d.R;
  const long long total = (long long)d.B * NT;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    int b = (int)(idx / NT);
    int rem = (int)(idx - (long long)b * NT);
    int o = rem / T, t = rem - o * T;
    const float* mu = d.mu + ((size_t)b * N + o) * R * T + t;
    const float* rh = d.cls ? d.cls_rb[class_slot(d.cls, d.ncls, b)].h : rbh.h;
    float muh = 0.f;
    for (int j = 0; j < R; ++j) muh += mu[(size_t)j * T] * rh[j];
    float* cf = d.coef + (size_t)b * 5 * NT + rem;
    cf[0] = 0.f; cf[NT] = 0.f;
    cf[2 * NT] = -muh - d.z[idx] + d.zeta[idx];
  }
}

__global__ void k_fill(float* p, float v, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}

// rda_set_obstacle_ids: one CTA per instance moves the per-slot warm start to the slots its obstacles went to.  The
// match (obstacle_ids.cuh) is one thread per slot on the ids in shared memory; an instance whose slots all keep their
// state stops there.  Otherwise the CTA copies the instance's per-slot planes into its own regions of the record lists,
// which the cell passes refill from scratch in every iteration (lam, mu: rec_a; z, zeta, xi, coef and feat: rec_b),
// then writes each moved slot from its source slot, or the cold-start zeros.  ids [B][N] (the handle's) receives cur.
constexpr int REMAP_THREADS = 256;
__global__ void __launch_bounds__(REMAP_THREADS) k_remap_slots(DevPtrs d, int* __restrict__ ids,
                                                               const int* __restrict__ cur_ids) {
  extern __shared__ int remap_sh[];                    // prev [N], cur [N], src [N]
  const int b = blockIdx.x, tid = threadIdx.x;
  const int N = d.N, T = d.T, E = d.E, R = d.R, NT = N * T;
  int* prev = remap_sh;
  int* cur = prev + N;
  int* src = cur + N;
  int* idb = ids + (size_t)b * N;
  for (int n = tid; n < N; n += REMAP_THREADS) { prev[n] = idb[n]; cur[n] = cur_ids[(size_t)b * N + n]; }
  __syncthreads();
  int moved = 0;
  for (int n = tid; n < N; n += REMAP_THREADS) {
    const int s = obstacle_slot_source(prev, cur, N, n);
    src[n] = s;
    moved |= s != n;
    idb[n] = cur[n];
  }
  if (!__syncthreads_or(moved)) return;
  float* lam = d.lam + (size_t)b * N * E * T;
  float* mu = d.mu + (size_t)b * N * R * T;
  // the nine [N][T] planes of the instance: z, zeta, xi (2), coef (5)
  auto plane = [&](int p) -> float* {
    return p == 0 ? d.z + (size_t)b * NT : p == 1 ? d.zeta + (size_t)b * NT
         : p < 4 ? d.xi + ((size_t)b * 2 + (p - 2)) * NT : d.coef + ((size_t)b * 5 + (p - 4)) * NT;
  };
  unsigned char* feat = d.feat ? d.feat + (size_t)b * NT : nullptr;
  float* sa = (float*)(d.rec_a + (size_t)b * NT);     // 20 floats per cell: lam, mu (E + R <= 16)
  float* sb = (float*)(d.rec_b + (size_t)b * NT);     // the nine planes, then feat (9 floats + 1 byte <= 20 floats)
  unsigned char* sf = (unsigned char*)(sb + 9 * NT);
  const int NET = N * E * T, NRT = N * R * T;
  for (int i = tid; i < NET; i += REMAP_THREADS) sa[i] = lam[i];
  for (int i = tid; i < NRT; i += REMAP_THREADS) sa[NET + i] = mu[i];
  for (int i = tid; i < 9 * NT; i += REMAP_THREADS) sb[i] = plane(i / NT)[i % NT];
  if (feat)
    for (int i = tid; i < NT; i += REMAP_THREADS) sf[i] = feat[i];
  __syncthreads();
  for (int i = tid; i < NET; i += REMAP_THREADS) {
    const int n = i / (E * T), s = src[n];
    if (s != n) lam[i] = s < 0 ? 0.f : sa[i + (s - n) * E * T];
  }
  for (int i = tid; i < NRT; i += REMAP_THREADS) {
    const int n = i / (R * T), s = src[n];
    if (s != n) mu[i] = s < 0 ? 0.f : sa[NET + i + (s - n) * R * T];
  }
  for (int i = tid; i < 9 * NT; i += REMAP_THREADS) {
    const int r = i % NT, n = r / T, s = src[n];
    if (s != n) plane(i / NT)[r] = s < 0 ? 0.f : sb[i + (s - n) * T];
  }
  if (feat)
    for (int i = tid; i < NT; i += REMAP_THREADS) {
      const int n = i / T, s = src[n];
      if (s != n) feat[i] = s < 0 ? (unsigned char)0 : sf[i + (s - n) * T];
    }
}

// (value, index) of two candidates: the smaller value, the smaller index among equal values (any reduction order gives
// the same result)
__device__ __forceinline__ void clear_min(float& v, int& i, float ov, int oi) {
  if (ov < v || (ov == v && oi < i)) { v = ov; i = oi; }
}

// rda_plan_clearance: one CTA per instance b, its threads striding over the N * (T + 1) cells c = o * (T + 1) + t (t
// fastest, the layout of dist), then the (value, index) minimum over each warp and over the CTA.  The body (the
// instance's class's, or the handle's rbh) is staged once in shared memory.
constexpr int CLEAR_THREADS = 128;
template <int EC, int RC>
__global__ void __launch_bounds__(CLEAR_THREADS) k_plan_clearance(const float* __restrict__ s, const float* __restrict__ obs_A,
                                                                  const float* __restrict__ obs_b,
                                                                  const int* __restrict__ obs_kind,
                                                                  const int* __restrict__ obs_count, int tv, int T, int N,
                                                                  int E, RobotGeom rbh, const int* __restrict__ cls,
                                                                  int ncls, const RobotGeom* __restrict__ cls_rb,
                                                                  float* __restrict__ dist, float* __restrict__ min_dist,
                                                                  int* __restrict__ min_index) {
  __shared__ RobotGeom body;
  __shared__ float wv[CLEAR_THREADS / 32];
  __shared__ int wi[CLEAR_THREADS / 32];
  const int b = blockIdx.x;
  if (threadIdx.x == 0) body = cls ? cls_rb[class_slot(cls, ncls, b)] : rbh;
  __syncthreads();
  const int T1 = T + 1, cells = N * T1;
  const int valid = N > 0 ? min(max(obs_count[b], 0), N) : 0;
  const size_t Tc = tv ? T1 : 1;
  const float* sb = s + (size_t)b * 3 * T1;
  float best = INFINITY;
  int bi = INT_MAX;
  for (int c = threadIdx.x; c < cells; c += CLEAR_THREADS) {
    const int o = c / T1, t = c - o * T1;
    float v = INFINITY;
    if (o < valid) {
      const size_t copy = ((size_t)b * N + o) * Tc + (tv ? t : 0);
      v = (float)plan_clearance_cell<EC, RC>(body, obs_kind[(size_t)b * N + o], E, obs_A + copy * E * 2, obs_b + copy * E,
                                             sb[t], sb[T1 + t], sb[2 * T1 + t]);
      clear_min(best, bi, v, c);
    }
    if (dist) dist[(size_t)b * cells + c] = v;
  }
  for (int off = 16; off > 0; off >>= 1)
    clear_min(best, bi, __shfl_xor_sync(0xffffffffu, best, off), __shfl_xor_sync(0xffffffffu, bi, off));
  if ((threadIdx.x & 31) == 0) { wv[threadIdx.x >> 5] = best; wi[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < CLEAR_THREADS / 32; ++w) clear_min(best, bi, wv[w], wi[w]);
    min_dist[b] = best;
    min_index[b] = bi == INT_MAX ? -1 : bi;
  }
}

// pointers of the sub-batch [b0, b0 + nb) (part selects its list counters)
DevPtrs dev_ptrs(const rda_handle* h, int b0, int nb, int part) {
  DevPtrs d;
  const size_t o = (size_t)b0, T = h->T, N = h->N, E = h->E, R = h->R, NT = N * T;
  const size_t Tc = h->obs_tv ? T + 1 : 1;
  d.lam = h->lam + o * N * E * T; d.mu = h->mu + o * N * R * T; d.z = h->z + o * NT; d.xi = h->xi + o * 2 * NT;
  d.zeta = h->zeta + o * NT; d.dis = h->dis + o * T; d.coef = h->coef + o * 5 * NT; d.pref = h->pref + o * 2 * T;
  d.cur_s = h->cur_s + o * 3 * (T + 1); d.cur_u = h->cur_u + o * 2 * T; d.ref_s = h->ref_s + o * 3 * (T + 1);
  d.ref_speed = h->ref_speed + o; d.resi_acc = h->resi_acc + 2 * o; d.resi_pri = h->resi_pri + o;
  d.resi_dual = h->resi_dual + o;
  d.status = h->status + o; d.iters = h->iters + o; d.done = h->done + o;
  d.counters = h->counters; d.wl_count = h->counters + 8 + 8 * part;     // part < 4, 8 counters each
  d.ogeo = h->ogeo ? h->ogeo + o * N : nullptr;
  d.feat = h->feat ? h->feat + o * NT : nullptr;
  d.rec_a = h->rec_a + o * NT; d.rec_b = h->rec_b + o * NT;
  d.su_ws = h->su_ws + o * h->su_ws_stride; d.su_ws_stride = h->su_ws_stride;
  d.obs_A = h->obs_A ? h->obs_A + o * N * Tc * E * 2 : nullptr;
  d.obs_b = h->obs_b ? h->obs_b + o * N * Tc * E : nullptr;
  d.obs_kind = h->obs_kind ? h->obs_kind + o * N : nullptr;
  d.obs_count = h->obs_count ? h->obs_count + o : nullptr;
  d.obs_tv = h->obs_tv;
  d.B = nb; d.T = h->T; d.N = h->N; d.E = h->E; d.R = h->R;
  d.inst = h->inst_on ? h->inst + o * RDA_INST_PARAMS : nullptr;
  d.cls = h->cls_on && h->ncls > 0 ? h->cls_idx + o : nullptr;
  d.ncls = h->ncls; d.cls_rb = h->cls_rb; d.cls_ra = h->cls_ra; d.cls_kin = h->cls_kin;
  return d;
}

DevPtrs dev_ptrs(const rda_handle* h) { return dev_ptrs(h, 0, h->B, 0); }

SuParams su_params(const rda_handle* h) {
  SuParams P;
  P.T = h->T; P.N = h->N; P.dynamics = h->cfg.dynamics; P.accelerated = h->cfg.accelerated;
  P.dt = h->cfg.step_time; P.L = h->cfg.wheelbase;
  P.umax[0] = h->cfg.max_speed[0]; P.umax[1] = h->cfg.max_speed[1];
  P.ab[0] = h->cfg.acce_bound[0]; P.ab[1] = h->cfg.acce_bound[1];
  P.ws = h->cfg.ws; P.wu = h->cfg.wu;
  P.slack_gain = h->tun.slack_gain; P.dmin = h->tun.min_sd; P.dmax = h->tun.max_sd;
  P.ro1 = h->tun.ro1; P.ro2 = h->tun.ro2;
  P.max_iter = 40;
  P.mu0 = 1.0f;
  P.prune = h->su_prune;
  return P;
}

// the variant of a kernel for the sub-batch d: with a class table or without (DevPtrs::cls)
template <typename K> K by_cls(const DevPtrs& d, K with_classes, K without) { return d.cls ? with_classes : without; }

int grid_for(long long n, int block, int sms) {
  long long g = (n + block - 1) / block;
  const long long cap = 16LL * sms;      // a few waves of the SMs; kernels grid-stride
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace

extern "C" {

const char* rda_version(void) { return "rda_b200 0.1 (sm_90a)"; }

int rda_create(const rda_config* cfg, const rda_tunables* tun, rda_handle** out) {
  if (!cfg || !tun || !out) return RDA_E_ARG;
  if (cfg->batch < 1 || cfg->receding < 1 || cfg->max_obs_num < 0) return RDA_E_ARG;
  if (cfg->max_edge_num < 3 || cfg->max_edge_num > RDA_MAX_EDGE) return RDA_E_UNSUPPORTED;
  if (cfg->dynamics < 0 || cfg->dynamics > 2) return RDA_E_ARG;
  rda_handle* h = new (std::nothrow) rda_handle();
  if (!h) return RDA_E_NOMEM;
  memset(h, 0, sizeof(*h));
  h->cfg = *cfg; h->tun = *tun;
  int rc = robot_geom_from_halfspaces(cfg->G, cfg->h, cfg->robot_edges, &h->rb, cfg->robot_cone);
  if (rc) { delete h; return rc; }
  h->B = cfg->batch; h->T = cfg->receding; h->N = cfg->max_obs_num; h->E = cfg->max_edge_num;
  h->R = cfg->robot_edges;
  const size_t B = h->B, T = h->T, N = h->N, E = h->E, R = h->R, NT = N * T;
  {
    // k_su keeps its workspace in shared memory, the hinge slacks / multipliers in a global slab per instance
    size_t g = 0;
    const size_t sm = cfg->su_fp64 ? su_work_bytes<double>((int)T, (int)N, false, &g) : su_work_bytes<float>((int)T, (int)N, false, &g);
    if (sm > 227 * 1024) { delete h; return RDA_E_UNSUPPORTED; }
    h->su_ws_stride = (g + 127) & ~(size_t)127;
  }
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) { delete h; return (int)e; }
  auto alloc = [&](float** p, size_t n) { if (e == cudaSuccess) e = cudaMalloc((void**)p, (n ? n : 1) * sizeof(float)); };
  alloc(&h->lam, B * N * E * T); alloc(&h->mu, B * N * R * T); alloc(&h->z, B * NT);
  alloc(&h->xi, B * 2 * NT); alloc(&h->zeta, B * NT); alloc(&h->dis, B * T);
  alloc(&h->coef, B * 5 * NT); alloc(&h->pref, B * 2 * T); alloc(&h->cur_s, B * 3 * (T + 1));
  alloc(&h->cur_u, B * 2 * T); alloc(&h->ref_s, B * 3 * (T + 1)); alloc(&h->ref_speed, B);
  alloc(&h->resi_acc, B * 2); alloc(&h->resi_pri, B); alloc(&h->resi_dual, B);
  alloc((float**)&h->status, B); alloc((float**)&h->iters, B); alloc((float**)&h->done, B);
  alloc((float**)&h->counters, 64);     // [0..7] statistics, [8 + 8 part ..] record list lengths of the sub-batches
  alloc((float**)&h->rec_a, B * NT * (sizeof(CellRec) / 4));
  alloc((float**)&h->rec_b, B * NT * (sizeof(CellRec) / 4));
  alloc((float**)&h->su_ws, B * (h->su_ws_stride / 4));
  if (e != cudaSuccess) { rda_destroy(h); return (int)e; }
  e = cfg->su_fp64 ? cudaFuncSetAttribute(k_su<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024)
                   : cudaFuncSetAttribute(k_su<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  if (e != cudaSuccess) { rda_destroy(h); return (int)e; }
  e = cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming);
  for (int p = 0; p < 3; ++p) {
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->side[p], cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->ev_join[p], cudaEventDisableTiming);
  }
  if (e != cudaSuccess) { rda_destroy(h); return (int)e; }
  // coherent first cell pass: on for batches whose sub-batches reach 4096 instances (at small batches its two extra
  // launches outweigh the saved work); RDA_B200_LEAN2=0/1 forces
  h->lean2 = h->B >= 8192 && h->E <= 4 && h->R <= 4 && h->N > 0 && !h->rb.disc;
  if (const char* l2 = getenv("RDA_B200_LEAN2")) h->lean2 = atoi(l2) != 0 && h->E <= 4 && h->R <= 4 && h->N > 0 && !h->rb.disc;
  if (h->lean2) {
    robot_aux_from_geom(h->rb, &h->ra);
    e = cudaMalloc((void**)&h->ogeo, B * N * sizeof(ObstacleGeom<4>));
    if (e == cudaSuccess) e = cudaMalloc((void**)&h->feat, B * NT ? B * NT : 1);
    if (e == cudaSuccess) e = cudaMalloc((void**)&h->rot, B * 2 * T * sizeof(float));
    if (e != cudaSuccess) { rda_destroy(h); return (int)e; }
  }
  h->split_min = 2048;
  h->parts = 2;
  h->su_prune = 0.5f;       // chosen by a sweep of 0.5, 1, 2 and off at B = 16384
  {
    size_t g = 0;
    const size_t sub = cfg->su_fp64 ? su_work_bytes<double>((int)T, (int)N, false, &g) : su_work_bytes<float>((int)T, (int)N, false, &g);
    h->small_L = small_layout((int)T, (int)N, (int)E, (int)R, sub, g);
    h->small_ok = h->small_L.total <= 200 * 1024 && !h->rb.disc;      // the persistent kernel has the polygon body's cells only
    h->small_mode = -1; h->small_max = 2 * h->sms;      // two resident CTAs per SM
    // bulk (TMA) staging needs every staged block to be a multiple of 16 bytes: N*E*T, N*R*T and N*T multiples of 4
    h->small_bulk = (N > 0) && ((N * E * T) % 4 == 0) && ((N * R * T) % 4 == 0) && ((N * T) % 4 == 0);
    if (const char* v = getenv("RDA_B200_SMALL_BULK")) { if (atoi(v) == 0) h->small_bulk = 0; }
    if (const char* v = getenv("RDA_B200_SMALL")) { int x = atoi(v); if (x >= -1 && x <= 1) h->small_mode = x; }
    if (const char* v = getenv("RDA_B200_SMALL_MAX")) { int x = atoi(v); if (x >= 1) h->small_max = x; }
    if (h->small_ok) {
      for (int c = 0; c < 2 && e == cudaSuccess; ++c) {
        if (cfg->su_fp64)
          e = cudaFuncSetAttribute(c ? k_admm_small<double, true> : k_admm_small<double, false>,
                                   cudaFuncAttributeMaxDynamicSharedMemorySize, h->small_L.total);
        else
          e = cudaFuncSetAttribute(c ? k_admm_small<float, true> : k_admm_small<float, false>,
                                   cudaFuncAttributeMaxDynamicSharedMemorySize, h->small_L.total);
      }
      if (e != cudaSuccess) { rda_destroy(h); return (int)e; }
    }
  }
  if (const char* v = getenv("RDA_B200_SU_PRUNE")) { float x = (float)atof(v); if (x >= 0.f) h->su_prune = x; }
  h->extra_min = 3000;
  if (const char* v = getenv("RDA_B200_EXTRA_MIN")) { int x = atoi(v); if (x >= 1) h->extra_min = x; }
  if (const char* sm = getenv("RDA_B200_SPLIT_MIN")) { int v = atoi(sm); if (v >= 2) h->split_min = v; }
  if (const char* sp = getenv("RDA_B200_SPLIT_PARTS")) { int v = atoi(sp); if (v >= 1 && v <= 4) h->parts = v; }
  rc = rda_cold_start(h, nullptr);
  if (rc) { rda_destroy(h); return rc; }
  e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { rda_destroy(h); return (int)e; }
  *out = h;
  return 0;
}

int rda_destroy(rda_handle* h) {
  if (!h) return RDA_E_ARG;
  float* bufs[] = {h->lam, h->mu, h->z, h->xi, h->zeta, h->dis, h->coef, h->pref, h->cur_s, h->cur_u,
                   h->ref_s, h->ref_speed, h->resi_acc, h->resi_pri, h->resi_dual, (float*)h->status,
                   (float*)h->iters, (float*)h->done, (float*)h->counters, (float*)h->su_ws};
  for (float* p : bufs) if (p) cudaFree(p);
  if (h->ogeo) cudaFree(h->ogeo);
  if (h->feat) cudaFree(h->feat);
  if (h->rec_a) cudaFree(h->rec_a);
  if (h->rec_b) cudaFree(h->rec_b);
  if (h->rot) cudaFree(h->rot);
  if (h->inst) cudaFree(h->inst);
  if (h->cls_rb) cudaFree(h->cls_rb);
  if (h->cls_ra) cudaFree(h->cls_ra);
  if (h->cls_kin) cudaFree(h->cls_kin);
  if (h->cls_idx) cudaFree(h->cls_idx);
  if (h->obs_id) cudaFree(h->obs_id);
  if (h->ev_fork) cudaEventDestroy(h->ev_fork);
  for (int p = 0; p < 3; ++p) {
    if (h->ev_join[p]) cudaEventDestroy(h->ev_join[p]);
    if (h->side[p]) cudaStreamDestroy(h->side[p]);
  }
  delete h;
  return 0;
}

int rda_set_tunables(rda_handle* h, const rda_tunables* tun) {
  if (!h || !tun) return RDA_E_ARG;
  h->tun = *tun;
  return 0;
}

int rda_get_tunables(const rda_handle* h, rda_tunables* tun) {
  if (!h || !tun) return RDA_E_ARG;
  *tun = h->tun;
  return 0;
}

int rda_set_instance_params(rda_handle* h, const float* params, void* stream) {
  if (!h) return RDA_E_ARG;
  if (!params) { h->inst_on = 0; return 0; }          // the storage stays for the next table
  if (!h->inst) RDA_CUDA(cudaMalloc((void**)&h->inst, (size_t)h->B * RDA_INST_PARAMS * sizeof(float)));
  RDA_CUDA(cudaMemcpyAsync(h->inst, params, (size_t)h->B * RDA_INST_PARAMS * sizeof(float), cudaMemcpyDeviceToDevice,
                           (cudaStream_t)stream));
  h->inst_on = 1;
  return 0;
}

int rda_set_robot_classes(rda_handle* h, int K, const rda_robot_class* classes, void* stream) {
  if (!h || K < 0 || K > RDA_MAX_ROBOT_CLASSES || (K > 0 && !classes)) return RDA_E_ARG;
  // slots 0..K-1: the classes, slot K: the handle's own body (an index outside [0, K))
  RobotGeom rb[RDA_MAX_ROBOT_CLASSES + 1];
  RobotAux ra[RDA_MAX_ROBOT_CLASSES + 1];
  ClassKin kin[RDA_MAX_ROBOT_CLASSES + 1];
  for (int k = 0; k < K; ++k) {
    const rda_robot_class& c = classes[k];
    if (c.dynamics < RDA_DYN_ACKER || c.dynamics > RDA_DYN_OMNI || !isfinite(c.wheelbase)) return RDA_E_ARG;
    if (c.dynamics == RDA_DYN_ACKER && !(c.wheelbase > 0.f)) return RDA_E_ARG;
  }
  for (int k = 0; k < K; ++k) {
    const int rc = robot_geom_from_halfspaces(classes[k].G, classes[k].h, h->R, &rb[k], h->cfg.robot_cone);
    if (rc) return rc;
    kin[k].dynamics = classes[k].dynamics; kin[k].L = classes[k].wheelbase;
  }
  rb[K] = h->rb;
  kin[K].dynamics = h->cfg.dynamics; kin[K].L = h->cfg.wheelbase;
  for (int k = 0; k <= K; ++k) {
    if (rb[k].disc) memset(&ra[k], 0, sizeof(RobotAux));      // the coherent pass, the only reader, takes polygons only
    else robot_aux_from_geom(rb[k], &ra[k]);
  }
  const size_t n = RDA_MAX_ROBOT_CLASSES + 1;
  if (!h->cls_rb) RDA_CUDA(cudaMalloc((void**)&h->cls_rb, n * sizeof(RobotGeom)));
  if (!h->cls_ra) RDA_CUDA(cudaMalloc((void**)&h->cls_ra, n * sizeof(RobotAux)));
  if (!h->cls_kin) RDA_CUDA(cudaMalloc((void**)&h->cls_kin, n * sizeof(ClassKin)));
  cudaStream_t s = (cudaStream_t)stream;
  // pageable host source: each copy has read it when the call returns
  RDA_CUDA(cudaMemcpyAsync(h->cls_rb, rb, (K + 1) * sizeof(RobotGeom), cudaMemcpyHostToDevice, s));
  RDA_CUDA(cudaMemcpyAsync(h->cls_ra, ra, (K + 1) * sizeof(RobotAux), cudaMemcpyHostToDevice, s));
  RDA_CUDA(cudaMemcpyAsync(h->cls_kin, kin, (K + 1) * sizeof(ClassKin), cudaMemcpyHostToDevice, s));
  h->ncls = K;
  return 0;
}

int rda_set_robot_class_index(rda_handle* h, const int32_t* robot_class, void* stream) {
  if (!h) return RDA_E_ARG;
  if (!robot_class) { h->cls_on = 0; return 0; }     // the storage stays for the next index
  if (!h->cls_idx) RDA_CUDA(cudaMalloc((void**)&h->cls_idx, (size_t)h->B * sizeof(int)));
  RDA_CUDA(cudaMemcpyAsync(h->cls_idx, robot_class, (size_t)h->B * sizeof(int), cudaMemcpyDeviceToDevice,
                           (cudaStream_t)stream));
  h->cls_on = 1;
  return 0;
}

int rda_set_obstacle_ids(rda_handle* h, const int32_t* obs_id, void* stream) {
  if (!h) return RDA_E_ARG;
  if (!obs_id) { h->ids_on = 0; return 0; }             // the storage stays for the next ids
  const size_t smem = (size_t)h->N * 3 * sizeof(int);
  if (smem > 48 * 1024) return RDA_E_UNSUPPORTED;
  const size_t n = (size_t)h->B * h->N;
  if (!h->obs_id) RDA_CUDA(cudaMalloc((void**)&h->obs_id, (n ? n : 1) * sizeof(int)));
  cudaStream_t s = (cudaStream_t)stream;
  if (!h->ids_on || h->N == 0) {
    RDA_CUDA(cudaMemcpyAsync(h->obs_id, obs_id, n * sizeof(int), cudaMemcpyDeviceToDevice, s));
    h->ids_on = 1;
    return 0;
  }
  k_remap_slots<<<h->B, REMAP_THREADS, smem, s>>>(dev_ptrs(h), h->obs_id, obs_id);
  RDA_CUDA(cudaGetLastError());
  return 0;
}

int rda_cold_start(rda_handle* h, void* stream) {
  if (!h) return RDA_E_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  const size_t B = h->B, T = h->T, N = h->N, E = h->E, R = h->R, NT = N * T;
  RDA_CUDA(cudaMemsetAsync(h->lam, 0, B * N * E * T * 4, s));
  RDA_CUDA(cudaMemsetAsync(h->mu, 0, B * N * R * T * 4, s));
  RDA_CUDA(cudaMemsetAsync(h->z, 0, B * NT * 4, s));
  RDA_CUDA(cudaMemsetAsync(h->xi, 0, B * 2 * NT * 4, s));
  RDA_CUDA(cudaMemsetAsync(h->zeta, 0, B * NT * 4, s));
  RDA_CUDA(cudaMemsetAsync(h->coef, 0, B * 5 * NT * 4, s));
  RDA_CUDA(cudaMemsetAsync(h->pref, 0, B * 2 * T * 4, s));
  RDA_CUDA(cudaMemsetAsync(h->cur_s, 0, B * 3 * (T + 1) * 4, s));
  RDA_CUDA(cudaMemsetAsync(h->cur_u, 0, B * 2 * T * 4, s));
  RDA_CUDA(cudaMemsetAsync(h->resi_acc, 0, B * 2 * 4, s));
  RDA_CUDA(cudaMemsetAsync(h->resi_pri, 0, B * 4, s));
  RDA_CUDA(cudaMemsetAsync(h->resi_dual, 0, B * 4, s));
  RDA_CUDA(cudaMemsetAsync(h->status, 0, B * 4, s));
  RDA_CUDA(cudaMemsetAsync(h->iters, 0, B * 4, s));
  RDA_CUDA(cudaMemsetAsync(h->done, 0, B * 4, s));
  RDA_CUDA(cudaMemsetAsync(h->counters, 0, 64 * 4, s));
  if (h->feat) RDA_CUDA(cudaMemsetAsync(h->feat, 0, B * NT, s));
  k_fill<<<grid_for((long long)(B * T), 256, h->sms), 256, 0, s>>>(h->dis, 1.0f, B * T);   // para_dis = 1 (:119)
  RDA_CUDA(cudaGetLastError());
  h->launches = 1;
  return 0;
}

int rda_reset(rda_handle* h, void* stream) {
  if (!h) return RDA_E_ARG;
  if (h->N == 0) return 0;
  DevPtrs d = dev_ptrs(h);
  k_reset<<<grid_for((long long)h->B * h->N * h->T, 256, h->sms), 256, 0, (cudaStream_t)stream>>>(d, h->rb);
  RDA_CUDA(cudaGetLastError());
  h->launches = 1;
  return 0;
}

// ---- the launches of one sub-batch [b0, b0 + nb) on stream s (part selects its list counters) ----
static int begin_part(rda_handle* h, const rda_inputs* in, int b0, int nb, int part, cudaStream_t s) {
  DevPtrs d = dev_ptrs(h, b0, nb, part);
  const size_t o = (size_t)b0, T = h->T;
  k_begin<<<grid_for((long long)nb * 3 * (h->T + 1), 256, h->sms), 256, 0, s>>>(
      d, (const float*)in->nom_s + o * 3 * (T + 1), (const float*)in->nom_u + o * 2 * T,
      (const float*)in->ref_s + o * 3 * (T + 1), (const float*)in->ref_speed + o);
  RDA_CUDA(cudaGetLastError());
  h->launches += 1;
  if (h->lean2 && !h->obs_tv && h->E <= 4 && h->R <= 4 && h->N > 0) {
    k_obstacle_geometry<<<(nb * h->N + 127) / 128, 128, 0, s>>>(d, h->ogeo + o * h->N);
    RDA_CUDA(cudaGetLastError());
    h->launches += 1;
  }
  return 0;
}

// The su-QP of a sub-batch: one warp (one CTA) per instance.
static int step_su_part(rda_handle* h, int b0, int nb, int part, cudaStream_t s) {
  DevPtrs d = dev_ptrs(h, b0, nb, part);
  SuParams P = su_params(h);
  const size_t smem1 = h->cfg.su_fp64 ? su_work_bytes<double>(h->T, h->N, false) : su_work_bytes<float>(h->T, h->N, false);
  if (smem1 > 227 * 1024) return RDA_E_UNSUPPORTED;
  if (h->cfg.su_fp64) k_su<double><<<nb, 32, smem1, s>>>(d, P);
  else k_su<float><<<nb, 32, smem1, s>>>(d, P);
  RDA_CUDA(cudaGetLastError());
  h->launches += 1;
  return 0;
}

static int step_lammuz_part(rda_handle* h, int b0, int nb, int part, cudaStream_t s) {
  DevPtrs d = dev_ptrs(h, b0, nb, part);
  if (h->N > 0) {
    const float theta = h->cfg.accelerated ? h->tun.z_theta : 1.0f;
    if (h->rb.disc) {
      by_cls(d, k_cells_dr<true>, k_cells_dr<false>)<<<grid_for((long long)nb * h->N * h->T, 128, h->sms), 128, 0, s>>>(d, h->rb, h->tun.ro2, theta);
      RDA_CUDA(cudaGetLastError());
      by_cls(d, k_cells_dr_mid<true>, k_cells_dr_mid<false>)<<<h->sms * 8, 128, 0, s>>>(d, h->rb, h->tun.ro2, theta);
      RDA_CUDA(cudaGetLastError());
      by_cls(d, k_cells_dr_slow_coop<true>, k_cells_dr_slow_coop<false>)<<<h->sms * 16, 32 * COOP_WARPS, 0, s>>>(d, h->rb, h->tun.ro2, theta);
      RDA_CUDA(cudaGetLastError());
      h->launches += 3;
      k_finalize<<<(nb + 127) / 128, 128, 0, s>>>(d, h->rb, h->iter_threshold);
      RDA_CUDA(cudaGetLastError());
      h->launches += 1;
      return 0;
    }
    if (h->lean2 && !h->obs_tv && h->E <= 4 && h->R <= 4) {
      k_heading<<<(nb * h->T + 255) / 256, 256, 0, s>>>(d, h->rot + (size_t)b0 * 2 * h->T);
      RDA_CUDA(cudaGetLastError());
      const int tiles = (h->N * h->T + 127) / 128;
      by_cls(d, k_cells_coh<true>, k_cells_coh<false>)<<<(unsigned)tiles * (unsigned)nb, 128, 0, s>>>(d, h->rb, h->ra, h->rot + (size_t)b0 * 2 * h->T, theta,
                                                                1.0f / (float)h->T, tiles);
      h->launches += 1;
      RDA_CUDA(cudaGetLastError());
      by_cls(d, k_cells_fast<4, 4, true, true>, k_cells_fast<4, 4, true, false>)<<<grid_for((long long)nb * h->N * h->T, 128, h->sms), 128, 0, s>>>(d, h->rb, theta);
      h->launches += 1;
    } else if (h->E <= 4 && h->R <= 4)
      by_cls(d, k_cells_fast<4, 4, false, true>, k_cells_fast<4, 4, false, false>)<<<grid_for((long long)nb * h->N * h->T, 128, h->sms), 128, 0, s>>>(d, h->rb, theta);
    else
      by_cls(d, k_cells_fast<8, 8, false, true>, k_cells_fast<8, 8, false, false>)<<<grid_for((long long)nb * h->N * h->T, 128, h->sms), 128, 0, s>>>(d, h->rb, theta);
    RDA_CUDA(cudaGetLastError());
    by_cls(d, k_cells_mid<true>, k_cells_mid<false>)<<<h->sms * 16, 128, 0, s>>>(d, h->rb, h->tun.ro2, theta);     // a few waves of the 6 resident CTAs per SM
    RDA_CUDA(cudaGetLastError());
    // the split costs a launch and pays from a few thousand instances on
    const int split = nb >= h->extra_min;
    if (split) {
      by_cls(d, k_cells_extra<true>, k_cells_extra<false>)<<<h->sms * 4, 128, 0, s>>>(d, h->rb, h->tun.ro2, theta);
      RDA_CUDA(cudaGetLastError());
      h->launches += 1;
    }
    by_cls(d, k_cells_slow_coop<true>, k_cells_slow_coop<false>)<<<h->sms * 16, 32 * COOP_WARPS, 0, s>>>(d, h->rb, h->tun.ro2, theta, split);
    RDA_CUDA(cudaGetLastError());
    h->launches += 3;
  }
  k_finalize<<<(nb + 127) / 128, 128, 0, s>>>(d, h->rb, h->iter_threshold);
  RDA_CUDA(cudaGetLastError());
  h->launches += 1;
  return 0;
}

static int finish_part(rda_handle* h, const rda_outputs* out, int b0, int nb, int part, cudaStream_t s) {
  DevPtrs d = dev_ptrs(h, b0, nb, part);
  const size_t o = (size_t)b0, T = h->T;
  rda_outputs po = *out;
  po.u_opt = (float*)out->u_opt + o * 2 * T;
  po.s_opt = (float*)out->s_opt + o * 3 * (T + 1);
  po.resi_pri = (float*)out->resi_pri + o;
  po.resi_dual = (float*)out->resi_dual + o;
  po.status = (int*)out->status + o;
  po.iters = (int*)out->iters + o;
  k_finish<<<grid_for((long long)nb * 3 * (h->T + 1), 256, h->sms), 256, 0, s>>>(d, po);
  RDA_CUDA(cudaGetLastError());
  h->launches += 1;
  return 0;
}

static int check_inputs(rda_handle* h, const rda_inputs* in, float iter_threshold) {
  if (!h || !in || !in->nom_s || !in->nom_u || !in->ref_s || !in->ref_speed) return RDA_E_ARG;
  if (h->N > 0 && (!in->obs_A || !in->obs_b || !in->obs_kind || !in->obs_count)) return RDA_E_ARG;
  h->obs_A = (const float*)in->obs_A; h->obs_b = (const float*)in->obs_b;
  h->obs_kind = (const int*)in->obs_kind; h->obs_count = (const int*)in->obs_count;
  h->obs_tv = in->obs_time_varying;
  h->iter_threshold = iter_threshold;
  return 0;
}

static int check_outputs(const rda_handle* h, const rda_outputs* out) {
  if (!h || !out || !out->u_opt || !out->s_opt || !out->resi_pri || !out->resi_dual || !out->status || !out->iters)
    return RDA_E_ARG;
  return 0;
}

int rda_begin(rda_handle* h, const rda_inputs* in, float iter_threshold, void* stream) {
  int rc = check_inputs(h, in, iter_threshold);
  if (rc) return rc;
  h->launches = 0;
  rc = begin_part(h, in, 0, h->B, 0, (cudaStream_t)stream);
  if (rc) return rc;
  h->began = 1;
  return 0;
}

int rda_step_su(rda_handle* h, void* stream) {
  if (!h || !h->began) return RDA_E_ARG;
  return step_su_part(h, 0, h->B, 0, (cudaStream_t)stream);
}

int rda_step_lammuz(rda_handle* h, void* stream) {
  if (!h || !h->began) return RDA_E_ARG;
  return step_lammuz_part(h, 0, h->B, 0, (cudaStream_t)stream);
}

int rda_finish(rda_handle* h, const rda_outputs* out, void* stream) {
  int rc = check_outputs(h, out);
  if (rc) return rc;
  return finish_part(h, out, 0, h->B, 0, (cudaStream_t)stream);
}

int rda_solve(rda_handle* h, const rda_inputs* in, const rda_outputs* out, int iter_num,
              float iter_threshold, void* stream) {
  if (iter_num < 1) return RDA_E_ARG;
  int rc = check_inputs(h, in, iter_threshold);
  if (rc) return rc;
  rc = check_outputs(h, out);
  if (rc) return rc;
  cudaStream_t s0 = (cudaStream_t)stream;
  h->launches = 0;
  h->began = 1;
  if (h->small_ok && (h->small_mode == 1 || (h->small_mode < 0 && h->B <= h->small_max))) {
    // the whole solve of every instance in one launch, state staged in shared memory (k_admm_small)
    DevPtrs d = dev_ptrs(h);
    SuParams P = su_params(h);
    const float theta = h->cfg.accelerated ? h->tun.z_theta : 1.0f;
    if (h->cfg.su_fp64)
      by_cls(d, k_admm_small<double, true>, k_admm_small<double, false>)<<<h->B, 128, h->small_L.total, s0>>>(d, P, h->rb, theta, iter_threshold, iter_num, h->small_L,
                                                              (const float*)in->nom_s, (const float*)in->nom_u, (const float*)in->ref_s,
                                                              (const float*)in->ref_speed, *out, h->small_bulk);
    else
      by_cls(d, k_admm_small<float, true>, k_admm_small<float, false>)<<<h->B, 128, h->small_L.total, s0>>>(d, P, h->rb, theta, iter_threshold, iter_num, h->small_L,
                                                             (const float*)in->nom_s, (const float*)in->nom_u, (const float*)in->ref_s,
                                                             (const float*)in->ref_speed, *out, h->small_bulk);
    RDA_CUDA(cudaGetLastError());
    h->launches = 1;
    return 0;
  }
  if (h->parts < 2 || h->B < h->split_min || h->B < h->parts) {
    rc = begin_part(h, in, 0, h->B, 0, s0);
    for (int i = 0; i < iter_num && !rc; ++i) {
      rc = step_su_part(h, 0, h->B, 0, s0);
      if (!rc) rc = step_lammuz_part(h, 0, h->B, 0, s0);
    }
    if (!rc) rc = finish_part(h, out, 0, h->B, 0, s0);
    return rc;
  }
  // Contiguous sub-batches, each an independent chain of launches: fork the side streams from the
  // caller's stream, enqueue the sub-batches alternately, join.  Instances never interact, so the
  // results do not depend on the split; fork and join are events only (CUDA-graph capturable).
  const int P = h->parts;
  int b0[5];
  for (int p = 0; p <= P; ++p) b0[p] = (int)((long long)h->B * p / P);
  cudaStream_t st[4];
  st[0] = s0;
  for (int p = 1; p < P; ++p) st[p] = h->side[p - 1];
  RDA_CUDA(cudaEventRecord(h->ev_fork, s0));
  for (int p = 1; p < P; ++p) RDA_CUDA(cudaStreamWaitEvent(st[p], h->ev_fork, 0));
  for (int p = 0; p < P && !rc; ++p) rc = begin_part(h, in, b0[p], b0[p + 1] - b0[p], p, st[p]);
  for (int i = 0; i < iter_num && !rc; ++i) {
    for (int p = 0; p < P && !rc; ++p) rc = step_su_part(h, b0[p], b0[p + 1] - b0[p], p, st[p]);
    for (int p = 0; p < P && !rc; ++p) rc = step_lammuz_part(h, b0[p], b0[p + 1] - b0[p], p, st[p]);
  }
  for (int p = 0; p < P && !rc; ++p) rc = finish_part(h, out, b0[p], b0[p + 1] - b0[p], p, st[p]);
  // always join, also on error, so that the caller's stream never outruns a side stream
  cudaError_t ej = cudaSuccess;
  for (int p = 1; p < P; ++p) {
    cudaError_t e1 = cudaEventRecord(h->ev_join[p - 1], st[p]);
    cudaError_t e2 = cudaStreamWaitEvent(s0, h->ev_join[p - 1], 0);
    if (ej == cudaSuccess) ej = e1 != cudaSuccess ? e1 : e2;
  }
  if (rc) return rc;
  return (int)ej;
}

int rda_get_buffer(rda_handle* h, int id, void** dev_ptr, size_t* count) {
  if (!h || !dev_ptr || !count) return RDA_E_ARG;
  const size_t B = h->B, T = h->T, N = h->N, E = h->E, R = h->R, NT = N * T;
  switch (id) {
    case RDA_BUF_LAM: *dev_ptr = h->lam; *count = B * N * E * T; break;
    case RDA_BUF_MU: *dev_ptr = h->mu; *count = B * N * R * T; break;
    case RDA_BUF_Z: *dev_ptr = h->z; *count = B * NT; break;
    case RDA_BUF_XI: *dev_ptr = h->xi; *count = B * 2 * NT; break;
    case RDA_BUF_ZETA: *dev_ptr = h->zeta; *count = B * NT; break;
    case RDA_BUF_DIS: *dev_ptr = h->dis; *count = B * T; break;
    case RDA_BUF_COEF: *dev_ptr = h->coef; *count = B * 5 * NT; break;
    case RDA_BUF_PREF: *dev_ptr = h->pref; *count = B * 2 * T; break;
    case RDA_BUF_CUR_S: *dev_ptr = h->cur_s; *count = B * 3 * (T + 1); break;
    case RDA_BUF_CUR_U: *dev_ptr = h->cur_u; *count = B * 2 * T; break;
    case RDA_BUF_COUNTERS: *dev_ptr = h->counters; *count = 8; break;
    default: return RDA_E_ARG;
  }
  return 0;
}

int rda_copy_buffer(rda_handle* h, int id, void* user, int to_handle, void* stream) {
  void* p = nullptr;
  size_t n = 0;
  int rc = rda_get_buffer(h, id, &p, &n);
  if (rc) return rc;
  if (!user) return RDA_E_ARG;
  RDA_CUDA(cudaMemcpyAsync(to_handle ? p : user, to_handle ? user : p, n * 4, cudaMemcpyDeviceToDevice,
                           (cudaStream_t)stream));
  return 0;
}

int rda_plan_clearance(rda_handle* h, const rda_inputs* in, const float* s, float* dist, float* min_dist,
                       int32_t* min_index, void* stream) {
  if (!h || !in || !s || !min_dist || !min_index) return RDA_E_ARG;
  if (h->N > 0 && (!in->obs_A || !in->obs_b || !in->obs_kind || !in->obs_count)) return RDA_E_ARG;
  const int* cls = h->cls_on && h->ncls > 0 ? h->cls_idx : nullptr;
  auto k = h->E <= 4 && h->R <= 4 ? k_plan_clearance<4, 4> : k_plan_clearance<8, 8>;
  k<<<h->B, CLEAR_THREADS, 0, (cudaStream_t)stream>>>(s, in->obs_A, in->obs_b, in->obs_kind, in->obs_count,
                                                     in->obs_time_varying, h->T, h->N, h->E, h->rb, cls, h->ncls,
                                                     h->cls_rb, dist, min_dist, min_index);
  RDA_CUDA(cudaGetLastError());
  return 0;
}

int rda_last_launch_count(const rda_handle* h) { return h ? h->launches : RDA_E_ARG; }

}  // extern "C"
