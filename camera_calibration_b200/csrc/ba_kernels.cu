// ba_kernels.cu -- the CUDA kernels of the bundle-adjustment path (sm_90a, FP64).
//
//   prepare_state_kernel        image_tr_global = camera_tr_rig * rig_tr_global, tangent frames
//   residual_jacobian_kernel    per observation: warm-started iterative projection, residual,
//                               Huber cost and (optionally) the analytic Jacobian rows
//   accumulate_scatter_kernel   J^T W J / J^T W r parts that group by point and by imageset
//   accumulate_cells_kernel     intrinsics x intrinsics (+ rig) blocks, grouped by B-spline cell
//   schur_* kernels             3x3 block factorisation, L^-1 B, back-substitution
//   update_* kernels            state retraction (JointOptimizationState::operator-=)
//   cost_compare_kernel         CostIsSmallerThan + totals, deterministic two-stage reduction
//
// Reference lines are cited at each kernel; paths relative to the reference repository
// (puzzlepaint/camera_calibration): applications/camera_calibration/src/camera_calibration (APP) and
// libvis/src/libvis (LV).

#include <algorithm>
#include <cstdlib>

#include "ba_device.cuh"
#include "ba_kernels.h"

namespace b200ba {

__device__ __forceinline__ int intr_col(const CamDev& c, int cell, int k);

// H(gi, gj) += v with gi, gj in the reference's global variable ordering; only the upper triangle
// is stored (lm_optimizer_update_accumulator.h:179,212,223): the pair is ordered first, then
// routed to the block-diagonal, off-diagonal or dense part (GetPartOfHAndB, :478-505).
__device__ __forceinline__ void add_H(const Layout& L, const SystemDev& sys, int gi, int gj, double v) {
  if (gi > gj) {
    const int t = gi;
    gi = gj;
    gj = t;
  }
  if (gj < L.nbd) {
    const int blk = gi / L.bs;
    const int a = gi - blk * L.bs, b = gj - blk * L.bs;  // same block by construction
    atomicAdd(&sys.Dblk[static_cast<int64_t>(blk) * L.dsz + a * L.bs - (a * (a - 1)) / 2 + (b - a)], v);
  } else if (gi < L.nbd) {
    atomicAdd(&sys.B[static_cast<int64_t>(gi) * L.nd + (gj - L.nbd)], v);
  } else {
    atomicAdd(&sys.C[static_cast<int64_t>(gi - L.nbd) * L.nd + (gj - L.nbd)], v);
  }
}
__device__ __forceinline__ void add_b(const Layout& L, const SystemDev& sys, int gi, double v) {
  if (gi < L.nbd)
    atomicAdd(&sys.bp[gi], v);
  else
    atomicAdd(&sys.bd[gi - L.nbd], v);
}

// ------------------------------------------------------------------------------------------
// prepare_state: composed poses + tangent frames
// ------------------------------------------------------------------------------------------
// image_tr_global = camera_tr_rig * rig_tr_global with Sophus' first-order renormalisation
// (APP/bundle_adjustment/joint_optimization.cc:277-280, sophus/so3.hpp:215-232); tangent
// frames of every control direction (joint_optimization.cc:254-270).
__global__ void prepare_state_kernel(ProblemDev pb, Layout L, StateDev st, int64_t n_control_total) {
  const int64_t tid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t n_pose = static_cast<int64_t>(L.n_imagesets) * L.n_cameras;
  if (tid < n_pose) {
    const int iset = static_cast<int>(tid / L.n_cameras);
    const int cam = static_cast<int>(tid % L.n_cameras);
    const double* a = st.camera_tr_rig + 7 * cam;
    const double* b = st.rig_tr_global + 7 * iset;
    const q4 qa{a[0], a[1], a[2], a[3]};
    const q4 qb{b[0], b[1], b[2], b[3]};
    double Ra[9];
    qrot(qa, Ra);
    const d3 t = mk3(a[4], a[5], a[6]) + rot_apply(Ra, mk3(b[4], b[5], b[6]));
    q4 q = qmul(qa, qb);
    const double sn = q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z;
    if (sn != 1.0) {
      const double s = 2.0 / (1.0 + sn);
      q.w *= s;
      q.x *= s;
      q.y *= s;
      q.z *= s;
    }
    double R[9];
    qrot(q, R);
    double* out = st.image_tr_global + 12 * tid;
#pragma unroll
    for (int i = 0; i < 9; ++i) out[i] = R[i];
    out[9] = t.x;
    out[10] = t.y;
    out[11] = t.z;
  }
  const int64_t k = tid - n_pose;
  if (k >= 0 && k < n_control_total) {
    // find the camera owning control point k (few cameras: linear scan)
    int cam = 0;
    int64_t local = k;
    for (int c = 0; c < L.n_cameras; ++c) {
      const int64_t G = static_cast<int64_t>(pb.cams[c].gw) * pb.cams[c].gh;
      if (local < G) {
        cam = c;
        break;
      }
      local -= G;
    }
    const CamDev& c = pb.cams[cam];
    const double* g = st.intrinsics + c.intr_off + 3 * local;
    d3 t1, t2;
    compute_tangents(mk3(g[0], g[1], g[2]), t1, t2);
    double* out = st.tangents + c.tan_off + 6 * local;
    out[0] = t1.x;
    out[1] = t1.y;
    out[2] = t1.z;
    out[3] = t2.x;
    out[4] = t2.y;
    out[5] = t2.z;
  }
}

void launch_prepare_state(const ProblemDev& pb, const Layout& L, const StateDev& st, int64_t n_control_total,
                          cudaStream_t s) {
  const int64_t n = static_cast<int64_t>(L.n_imagesets) * L.n_cameras + n_control_total;
  const int threads = 128;
  prepare_state_kernel<<<static_cast<unsigned>((n + threads - 1) / threads), threads, 0, s>>>(pb, L, st,
                                                                                              n_control_total);
}

// ------------------------------------------------------------------------------------------
// residual + Jacobian, one thread per observation
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void store_col(const ObsOut& out, int64_t n_obs, int64_t o, int col, double jx,
                                          double jy) {
  out.jac[(2 * static_cast<int64_t>(col)) * n_obs + o] = jx;
  out.jac[(2 * static_cast<int64_t>(col) + 1) * n_obs + o] = jy;
}

// AddReprojectionResidual (joint_optimization.cc:308-449) with the intrinsics / point
// Jacobians obtained analytically through the implicit function theorem at the converged
// projection (the reference differentiates numerically: joint_optimization.cc:357-376,
// models/central_grid.h:187-245, models/noncentral_generic.h:224-283).
//
// Two passes share this code. The MAIN pass (STRAGGLER = false) gives every observation a budget
// of kMainEvalBudget spline evaluations -- in the warm-started steady state all but a handful
// need exactly 2 -- and appends the rare observation that needs more (a point whose projection
// runs against the border of the calibrated area burns the reference's full 100 x 10 iteration
// allowance twice: ~400 evaluations) to a list instead of letting one lane hold its warp, block
// and ultimately the whole launch hostage. The STRAGGLER pass redoes the listed observations from
// scratch with an unlimited budget, two lanes per observation: lane 0 runs the warm-started
// attempt, lane 1 speculatively runs the reference's retry from the image centre; the result is
// exactly what the sequential reference procedure yields.
constexpr int kUnlimitedEvals = 1 << 30;
// ObsOut::has_jac states
constexpr uint8_t kJacNone = 0, kJacValid = 1, kJacPending = 2, kJacLate = 3;
static int g_main_eval_budget = 16;
void set_main_eval_budget(int b) { g_main_eval_budget = b < 1 ? 1 : b; }

// ---- chain rule to pose / rig / point (joint_optimization.cc:378-438) --------------------------
// For the left update q <- (1, delta) q: d(R(q) v)/d delta = -2 [R v]_x. R is the COMPOSED rotation
// image_tr_global; with a single camera the reference differentiates with it and an identity
// translation block (joint_optimization.cc:392-397, SURVEY appendix B.5), reproduced as is.
__device__ __forceinline__ void chain_rule(const Layout& L, const StateDev& st, int iset, int cam, const d3& point,
                                           const double* R, const d3& rp, const double P[2][3], double jp[2][3],
                                           double jo[2][6], double jr[2][6]) {
  if (L.rig_in_state) {
    const double* ca = st.camera_tr_rig + 7 * cam;
    const double* rb = st.rig_tr_global + 7 * static_cast<int64_t>(iset);
    double Rc[9], Rr[9];
    qrot(q4{ca[0], ca[1], ca[2], ca[3]}, Rc);
    qrot(q4{rb[0], rb[1], rb[2], rb[3]}, Rr);
    const d3 rrp = rot_apply(Rr, point);
    const d3 crp = rot_apply(Rc, rrp + mk3(rb[4], rb[5], rb[6]));
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      // PRc = P Rc
      const double a0 = P[r][0] * Rc[0] + P[r][1] * Rc[3] + P[r][2] * Rc[6];
      const double a1 = P[r][0] * Rc[1] + P[r][1] * Rc[4] + P[r][2] * Rc[7];
      const double a2 = P[r][0] * Rc[2] + P[r][1] * Rc[5] + P[r][2] * Rc[8];
      jo[r][0] = -2 * (a1 * rrp.z - a2 * rrp.y);
      jo[r][1] = -2 * (-a0 * rrp.z + a2 * rrp.x);
      jo[r][2] = -2 * (a0 * rrp.y - a1 * rrp.x);
      jo[r][3] = a0;
      jo[r][4] = a1;
      jo[r][5] = a2;
      jr[r][0] = -2 * (P[r][1] * crp.z - P[r][2] * crp.y);
      jr[r][1] = -2 * (-P[r][0] * crp.z + P[r][2] * crp.x);
      jr[r][2] = -2 * (P[r][0] * crp.y - P[r][1] * crp.x);
      jr[r][3] = P[r][0];
      jr[r][4] = P[r][1];
      jr[r][5] = P[r][2];
      jp[r][0] = a0 * Rr[0] + a1 * Rr[3] + a2 * Rr[6];
      jp[r][1] = a0 * Rr[1] + a1 * Rr[4] + a2 * Rr[7];
      jp[r][2] = a0 * Rr[2] + a1 * Rr[5] + a2 * Rr[8];
    }
  } else {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      jo[r][0] = -2 * (P[r][1] * rp.z - P[r][2] * rp.y);
      jo[r][1] = -2 * (-P[r][0] * rp.z + P[r][2] * rp.x);
      jo[r][2] = -2 * (P[r][0] * rp.y - P[r][1] * rp.x);
      jo[r][3] = P[r][0];
      jo[r][4] = P[r][1];
      jo[r][5] = P[r][2];
      jp[r][0] = P[r][0] * R[0] + P[r][1] * R[3] + P[r][2] * R[6];
      jp[r][1] = P[r][0] * R[1] + P[r][1] * R[4] + P[r][2] * R[7];
      jp[r][2] = P[r][0] * R[2] + P[r][1] * R[5] + P[r][2] * R[8];
#pragma unroll
      for (int j = 0; j < 6; ++j) jr[r][j] = 0.0;
    }
  }
}

// Compact mode: P of observation o and the [point | pose | rig] Jacobian blocks rebuilt from it.
__device__ __forceinline__ void compact_small_blocks(const ProblemDev& pb, const Layout& L, const StateDev& st,
                                                     const ObsOut& out, int64_t o, double jp[2][3], double jo[2][6],
                                                     double jr[2][6]) {
  const int64_t n = pb.n_obs;
  const int iset = static_cast<int>(pb.obs_imageset[o]);
  const int cam = static_cast<int>(pb.obs_camera[o]);
  const int pidx = static_cast<int>(pb.obs_point[o]);
  double P[2][3];
#pragma unroll
  for (int q = 0; q < 6; ++q) P[q / 3][q % 3] = out.cjac[static_cast<int64_t>(q) * n + o];
  const double* T = st.image_tr_global + 12 * (static_cast<int64_t>(iset) * L.n_cameras + cam);
  double R[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) R[i] = __ldg(T + i);
  const d3 point = ld3(st.points + 3 * static_cast<int64_t>(pidx));
  const d3 rp = rot_apply(R, point);
  chain_rule(L, st, iset, cam, point, R, rp, P, jp, jo, jr);
}

// one cubic B-spline basis weight (bspline_basis() for a single index)
__device__ __forceinline__ double bspline_w1(double u, int idx) {
  constexpr double k6 = 1.0 / 6.0;
  const double u2 = u * u, u3 = u2 * u, omu = 1.0 - u;
  return idx == 0 ? omu * omu * omu * k6
                  : (idx == 1 ? (3.0 * u3 - 6.0 * u2 + 4.0) * k6 : (idx == 2 ? (-3.0 * u3 + 3.0 * u2 + 3.0 * u + 1.0) * k6 : u3 * k6));
}

// Entry (rows x, y) of STORAGE column `col` of observation o: read from the expanded buffer, or rebuilt
// from the compact record (central-generic cameras only).
__device__ __forceinline__ void load_jcol(const ProblemDev& pb, const Layout& L, const StateDev& st, const ObsOut& out,
                                          int64_t o, int col, double& jx, double& jy) {
  const int64_t n = pb.n_obs;
  if (!out.compact) {
    jx = out.jac[(2 * static_cast<int64_t>(col)) * n + o];
    jy = out.jac[(2 * static_cast<int64_t>(col) + 1) * n + o];
    return;
  }
  if (col >= L.jc_intr) {
    const int k = col - L.jc_intr, cp = k >> 1, dsel = k & 1, xx = cp & 3, yy = cp >> 2;
    const CamDev& c = pb.cams[pb.obs_camera[o]];
    const double fu = out.cjac[12 * n + o], fv = out.cjac[13 * n + o];
    const double wk = bspline_w1(fu, xx) * bspline_w1(fv, yy);
    const double* tan = st.tangents + c.tan_off + 6 * (static_cast<int64_t>(out.cell[o]) + xx + static_cast<int64_t>(yy) * c.gw) + 3 * dsel;
    const d3 t = ld3(tan);
    const d3 m0 = mk3(out.cjac[6 * n + o], out.cjac[7 * n + o], out.cjac[8 * n + o]);
    const d3 m1 = mk3(out.cjac[9 * n + o], out.cjac[10 * n + o], out.cjac[11 * n + o]);
    jx = wk * dot3(m0, t);
    jy = wk * dot3(m1, t);
    return;
  }
  double jp[2][3], jo[2][6], jr[2][6];
  compact_small_blocks(pb, L, st, out, o, jp, jo, jr);
  // register arrays are indexed with compile-time constants only
  jx = jy = 0.0;
#pragma unroll
  for (int j = 0; j < 3; ++j)
    if (col == L.jc_point + j) {
      jx = jp[0][j];
      jy = jp[1][j];
    }
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    if (col == L.jc_pose + j) {
      jx = jo[0][j];
      jy = jo[1][j];
    }
    if (L.rig_in_state && col == L.jc_rig + j) {
      jx = jr[0][j];
      jy = jr[1][j];
    }
  }
}

template <int MODEL, bool JAC, bool STRAGGLER, bool COMPACT>
__device__ __forceinline__ void process_observation(const ProblemDev& pb, const Layout& L, const StateDev& st,
                                                    double2* __restrict__ last_projection, const ObsOut& out,
                                                    double huber, uint32_t* __restrict__ straggler_list,
                                                    int* __restrict__ straggler_count, int64_t o, int role,
                                                    int main_budget) {
  const int iset = static_cast<int>(pb.obs_imageset[o]);
  const int cam = static_cast<int>(pb.obs_camera[o]);
  const int pidx = static_cast<int>(pb.obs_point[o]);
  const float2 xyf = pb.obs_xy[o];
  const CamDev& c = pb.cams[cam];
  const int model = (MODEL >= 0) ? MODEL : c.model_type;

  const double* T = st.image_tr_global + 12 * (static_cast<int64_t>(iset) * L.n_cameras + cam);
  double R[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) R[i] = __ldg(T + i);
  const d3 tvec = mk3(__ldg(T + 9), __ldg(T + 10), __ldg(T + 11));
  const d3 point = ld3(st.points + 3 * static_cast<int64_t>(pidx));
  const d3 rp = rot_apply(R, point);
  const d3 lp = rp + tvec;

  // warm start (joint_optimization.cc:324-333)
  double2 lpj = last_projection[o];
  double px = lpj.x, py = lpj.y;
  if (!(px >= c.min_x && py >= c.min_y && px < c.max_x + 1 && py < c.max_y + 1) || isnan(px) || isnan(py)) {
    px = c.center_x;
    py = c.center_y;
  }

  const double* intr = st.intrinsics + c.intr_off;
  bool ok = false;
  int n_eval = 0;
  CentralEval ce;
  NoncentralEval ne;
  d3 nt1, nt2;
  double nR[2][2];
  const int budget = STRAGGLER ? kUnlimitedEvals : main_budget;
  int status = kProjFail;
  if (STRAGGLER && role == 1) {
    px = c.center_x;
    py = c.center_y;
  }
  if (model == B200BA_MODEL_CENTRAL_GENERIC) {
    const double ilen = rsqrt(dot3(lp, lp));
    const d3 dir = ilen * lp;
    status = central_project(c, intr, dir, px, py, ce, n_eval, budget);
    if (!STRAGGLER && status == kProjFail) {
      // backup: re-initialise at the centre of the calibrated area (joint_optimization.cc:334-342)
      px = c.center_x;
      py = c.center_y;
      status = central_project(c, intr, dir, px, py, ce, n_eval, budget);
    }
  } else if (model == B200BA_MODEL_NONCENTRAL_GENERIC) {
    const double* pgrid = intr + 3 * static_cast<int64_t>(c.gw) * c.gh;
    status = noncentral_project(c, intr, pgrid, lp, px, py, ne, nt1, nt2, nR, n_eval, budget);
    if (!STRAGGLER && status == kProjFail) {
      px = c.center_x;
      py = c.center_y;
      status = noncentral_project(c, intr, pgrid, lp, px, py, ne, nt1, nt2, nR, n_eval, budget);
    }
  } else {
    status = opencv_project(c, intr, lp, px, py) ? kProjOk : kProjFail;  // estimate ignored (central_opencv.h:61-67)
  }
  if (!STRAGGLER) {
    if (status == kProjUnfinished) {
      const int slot = atomicAdd(straggler_count, 1);
      straggler_list[slot] = static_cast<uint32_t>(o);
      if (JAC) out.has_jac[o] = kJacPending;
      return;  // every other output of this observation is written by the straggler pass
    }
    ok = status == kProjOk;
  } else {
    // lane 0 (warm) wins if it succeeded, else lane 1 (centre); the winner writes the outputs
    const bool mine = (role != 2) && status == kProjOk;
    const bool other = __shfl_xor_sync(0xffffffffu, mine ? 1 : 0, 1) != 0;
    if (role == 2) return;
    if (role == 0) {
      ok = mine;
      if (!mine && other) return;  // lane 1 reports the success
    } else {
      if (other || !mine) return;  // lane 0 succeeded, or both failed (lane 0 reports the failure)
      ok = true;
    }
  }
  if (out.evals) out.evals[o] = static_cast<uint16_t>(min(n_eval, 65535));

  if (!ok) {
    out.cost[o] = -1.0;  // AddInvalidResidual (LV/lm_optimizer_update_accumulator.h:158-160)
    out.residual[o] = nan("");
    out.residual[pb.n_obs + o] = nan("");
    if (JAC) {
      out.has_jac[o] = 0;
      out.cell[o] = -1;
    }
    return;
  }
  last_projection[o] = make_double2(px, py);
  const double rx = px - static_cast<double>(xyf.x);
  const double ry = py - static_cast<double>(xyf.y);
  out.residual[o] = rx;
  out.residual[pb.n_obs + o] = ry;
  out.cost[o] = huber_cost_sq(huber, rx * rx + ry * ry);
  if (!JAC) return;

  // ---- d pixel / d local_point (2x3) and d pixel / d intrinsics ---------------------------
  double P[2][3];
  const int jc_intr = L.jc_intr;
  int cell = 0;
  if (model == B200BA_MODEL_CENTRAL_GENERIC) {
    // M = (A^T A)^-1 A^T with A = d unproj / d pixel
    const double a00 = dot3(ce.ux, ce.ux), a01 = dot3(ce.ux, ce.uy), a11 = dot3(ce.uy, ce.uy);
    const double idet = 1.0 / (a00 * a11 - a01 * a01);
    const d3 M0 = idet * (a11 * ce.ux - a01 * ce.uy);
    const d3 M1 = idet * (a00 * ce.uy - a01 * ce.ux);
    const double ilen = rsqrt(dot3(lp, lp));
    const d3 d = ilen * lp;
    const double m0d = dot3(M0, d), m1d = dot3(M1, d);
    P[0][0] = (M0.x - m0d * d.x) * ilen;
    P[0][1] = (M0.y - m0d * d.y) * ilen;
    P[0][2] = (M0.z - m0d * d.z) * ilen;
    P[1][0] = (M1.x - m1d * d.x) * ilen;
    P[1][1] = (M1.y - m1d * d.y) * ilen;
    P[1][2] = (M1.z - m1d * d.z) * ilen;
    int x0, y0;
    double fu, fv;
    locate_support(c, px, py, x0, y0, fu, fv);
    cell = x0 + y0 * c.gw;
    if (COMPACT) {
      // d unproj / d G_k = w_k / |s| (I - u u^T) and M u = 0 (the columns of A are orthogonal to u), so
      // d pixel / d theta_k = w_k * Mn [t1 t2]_k with Mn = -M / |s|: the consumers rebuild the 32 columns
      const int64_t n = pb.n_obs;
      const double s = -ce.inv_n;
      out.cjac[0 * n + o] = P[0][0];
      out.cjac[1 * n + o] = P[0][1];
      out.cjac[2 * n + o] = P[0][2];
      out.cjac[3 * n + o] = P[1][0];
      out.cjac[4 * n + o] = P[1][1];
      out.cjac[5 * n + o] = P[1][2];
      out.cjac[6 * n + o] = s * M0.x;
      out.cjac[7 * n + o] = s * M0.y;
      out.cjac[8 * n + o] = s * M0.z;
      out.cjac[9 * n + o] = s * M1.x;
      out.cjac[10 * n + o] = s * M1.y;
      out.cjac[11 * n + o] = s * M1.z;
      out.cjac[12 * n + o] = fu;
      out.cjac[13 * n + o] = fv;
      out.cell[o] = cell;
      out.has_jac[o] = STRAGGLER ? kJacLate : kJacValid;
      return;
    }
    if (!L.localize_only) {
      double wx[4], dwx[4], wy[4], dwy[4];
      bspline_basis(fu, wx, dwx);
      bspline_basis(fv, wy, dwy);
      // d unproj / d G_k = w_k / |s| (I - u u^T) and M u = 0 (the columns of A are orthogonal to
      // u), so d pixel / d theta_k = -w_k / |s| * M [t1 t2]_k
      const double* tan = st.tangents + c.tan_off + 6 * static_cast<int64_t>(cell);
#pragma unroll 1
      for (int yy = 0; yy < 4; ++yy) {
        const double wyv = -sel4(wy, yy) * ce.inv_n;
#pragma unroll
        for (int xx = 0; xx < 4; ++xx) {
          const double wk = wx[xx] * wyv;
          const d3 t1 = ld3(tan + 6 * xx), t2 = ld3(tan + 6 * xx + 3);
          const int k = 2 * (xx + 4 * yy);
          store_col(out, pb.n_obs, o, jc_intr + k, wk * dot3(M0, t1), wk * dot3(M1, t1));
          store_col(out, pb.n_obs, o, jc_intr + k + 1, wk * dot3(M0, t2), wk * dot3(M1, t2));
        }
        tan += 6 * static_cast<int64_t>(c.gw);
      }
    }
  } else if (model == B200BA_MODEL_NONCENTRAL_GENERIC) {
    const double idet = 1.0 / (nR[0][0] * nR[1][1] - nR[0][1] * nR[1][0]);
    const double Ri00 = idet * nR[1][1], Ri01 = -idet * nR[0][1], Ri10 = -idet * nR[1][0], Ri11 = idet * nR[0][0];
    // d x / d p = R^-1 [t1 t2]^T
    P[0][0] = Ri00 * nt1.x + Ri01 * nt2.x;
    P[0][1] = Ri00 * nt1.y + Ri01 * nt2.y;
    P[0][2] = Ri00 * nt1.z + Ri01 * nt2.z;
    P[1][0] = Ri10 * nt1.x + Ri11 * nt2.x;
    P[1][1] = Ri10 * nt1.y + Ri11 * nt2.y;
    P[1][2] = Ri10 * nt1.z + Ri11 * nt2.z;
    int x0, y0;
    double fu, fv;
    locate_support(c, px, py, x0, y0, fu, fv);
    cell = x0 + y0 * c.gw;
    if (!L.localize_only) {
      double wx[4], dwx[4], wy[4], dwy[4];
      bspline_basis(fu, wx, dwx);
      bspline_basis(fv, wy, dwy);
      // d r / d direction (rows), through the normalisation of the interpolated direction
      d3 rd1, rd2;
      tangent_rows(ne.u, ne.o - lp, rd1, rd2);
      rd1 = ne.inv_n * (rd1 - dot3(rd1, ne.u) * ne.u);
      rd2 = ne.inv_n * (rd2 - dot3(rd2, ne.u) * ne.u);
      const double* tan = st.tangents + c.tan_off;
#pragma unroll 1
      for (int yy = 0; yy < 4; ++yy) {
        const double wyv = sel4(wy, yy);
#pragma unroll
        for (int xx = 0; xx < 4; ++xx) {
          const int64_t seq = cell + xx + static_cast<int64_t>(yy) * c.gw;
          const double wk = wx[xx] * wyv;
          const d3 t1 = ld3(tan + 6 * seq), t2 = ld3(tan + 6 * seq + 3);
          const d3 dk = ld3(intr + 3 * seq);
          const int k = 5 * (xx + 4 * yy);
          // LineJacobianWrtLocalUpdate (line_parametrization.h:123-135): direction DoF 0-1,
          // origin DoF 2-4 (along t1, t2 and the control direction)
          double dr0[5], dr1[5];
          dr0[0] = wk * dot3(rd1, t1);
          dr1[0] = wk * dot3(rd2, t1);
          dr0[1] = wk * dot3(rd1, t2);
          dr1[1] = wk * dot3(rd2, t2);
          dr0[2] = wk * dot3(nt1, t1);
          dr1[2] = wk * dot3(nt2, t1);
          dr0[3] = wk * dot3(nt1, t2);
          dr1[3] = wk * dot3(nt2, t2);
          dr0[4] = wk * dot3(nt1, dk);
          dr1[4] = wk * dot3(nt2, dk);
#pragma unroll
          for (int q = 0; q < 5; ++q)
            store_col(out, pb.n_obs, o, jc_intr + k + q, -(Ri00 * dr0[q] + Ri01 * dr1[q]),
                      -(Ri10 * dr0[q] + Ri11 * dr1[q]));
        }
      }
    }
  } else {
    double Jx[12], Jy[12];
    opencv_jacobians(intr, lp, P, Jx, Jy);
    if (!L.localize_only) {
#pragma unroll
      for (int k = 0; k < 12; ++k) store_col(out, pb.n_obs, o, jc_intr + k, Jx[k], Jy[k]);
    }
  }
  out.cell[o] = cell;
  // a late (straggler-pass) success is flagged separately: the main accumulation kernels may be
  // running concurrently and must not pick it up; accumulate_list_kernel folds it in afterwards
  out.has_jac[o] = STRAGGLER ? kJacLate : kJacValid;

  // ---- chain rule to pose / rig / point (joint_optimization.cc:378-438) ----------------------
  double jp[2][3], jo[2][6], jr[2][6];
  chain_rule(L, st, iset, cam, point, R, rp, P, jp, jo, jr);
  const int64_t stride = 2 * pb.n_obs;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    double* dst = out.jac + (2 * static_cast<int64_t>(L.jc_pose) + r) * pb.n_obs + o;
#pragma unroll
    for (int j = 0; j < 6; ++j) dst[j * stride] = jo[r][j];
    double* dp = out.jac + (2 * static_cast<int64_t>(L.jc_point) + r) * pb.n_obs + o;
#pragma unroll
    for (int j = 0; j < 3; ++j) dp[j * stride] = jp[r][j];
    if (L.rig_in_state) {
      double* dr = out.jac + (2 * static_cast<int64_t>(L.jc_rig) + r) * pb.n_obs + o;
#pragma unroll
      for (int j = 0; j < 6; ++j) dr[j * stride] = jr[r][j];
    }
  }
}

template <int MODEL, bool JAC, int MINB, bool STRAGGLER, bool COMPACT>
__global__ void __launch_bounds__(128, MINB)
    residual_jacobian_kernel(ProblemDev pb, Layout L, StateDev st, double2* __restrict__ last_projection,
                             ObsOut out, double huber, uint32_t* __restrict__ straggler_list,
                             int* __restrict__ straggler_count, int main_budget) {
  if (!STRAGGLER) {
    const int64_t o = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
    if (o >= pb.n_obs) return;
    process_observation<MODEL, JAC, false, COMPACT>(pb, L, st, last_projection, out, huber, straggler_list, straggler_count, o, 0,
                                           main_budget);
  } else {
    // two lanes per listed observation; the loop bound is warp-uniform so that the pair shuffle
    // inside process_observation always sees whole warps
    const int count = *straggler_count;
    const int lane = threadIdx.x & 31;
    const int64_t warp_id = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
    const int64_t stride = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 1;  // pairs per sweep
    for (int64_t base = warp_id * 16; base < count; base += stride) {
      int64_t pair = base + (lane >> 1);
      int role = lane & 1;  // 0 = warm-start attempt, 1 = speculative centre attempt
      if (pair >= count) {
        pair = count - 1;
        role = 2;  // muted lane: computes, never writes
      }
      process_observation<MODEL, JAC, true, COMPACT>(pb, L, st, last_projection, out, huber, straggler_list, straggler_count,
                                            straggler_list[pair], role, main_budget);
    }
  }
}

// Main pass: 128 threads per block; MINB = resident blocks per SM the kernel is compiled for (register budget
// 65536 / (128 * MINB)).
constexpr int kMainThreads = 128;

// Straggler pass geometry: a fixed grid that loops over the device-side list (its length is not
// known on the host without a sync); 2 lanes per listed observation.
constexpr int kStragglerBlocks = 1056;  // 8 per SM of an H100 (132 SMs): the cold first pass (every projection starts at last_projection = 0) defers many observations
constexpr int kStragglerThreads = 128;

template <int MODEL, bool JAC, int MINB>
static void launch_rj_model(const ProblemDev& pb, const Layout& L, const StateDev& st, double2* lp,
                            const ObsOut& out, double huber, uint32_t* list, int* count, cudaStream_t s,
                            cudaEvent_t main_done) {
  const unsigned blocks = static_cast<unsigned>((pb.n_obs + kMainThreads - 1) / kMainThreads);
  // central-generic Jacobians go to the compact records (out.compact is set for exactly these rigs)
  residual_jacobian_kernel<MODEL, JAC, MINB, false, (MODEL == B200BA_MODEL_CENTRAL_GENERIC && JAC)>
      <<<blocks, kMainThreads, 0, s>>>(pb, L, st, lp, out, huber, list, count, g_main_eval_budget);
  if (main_done) cudaEventRecord(main_done, s);  // between the main and the straggler pass
}

template <bool JAC>
static void launch_rj(int model, const ProblemDev& pb, const Layout& L, const StateDev& st, double2* lp,
                      const ObsOut& out, double huber, uint32_t* list, int* count, cudaStream_t s,
                      cudaEvent_t main_done) {
  if (pb.n_obs == 0) return;
  cudaMemsetAsync(count, 0, sizeof(int), s);
  switch (model) {
    case B200BA_MODEL_CENTRAL_GENERIC:
      launch_rj_model<B200BA_MODEL_CENTRAL_GENERIC, JAC, 4>(pb, L, st, lp, out, huber, list, count, s, main_done);
      break;
    case B200BA_MODEL_NONCENTRAL_GENERIC:
      launch_rj_model<B200BA_MODEL_NONCENTRAL_GENERIC, JAC, 3>(pb, L, st, lp, out, huber, list, count, s, main_done);
      break;
    case B200BA_MODEL_CENTRAL_OPENCV:
      launch_rj_model<B200BA_MODEL_CENTRAL_OPENCV, JAC, 4>(pb, L, st, lp, out, huber, list, count, s, main_done);
      break;
    default:
      launch_rj_model<-1, JAC, 3>(pb, L, st, lp, out, huber, list, count, s, main_done);
  }
}

template <bool JAC>
static void launch_stragglers(int model, const ProblemDev& pb, const Layout& L, const StateDev& st, double2* lp,
                              const ObsOut& out, double huber, uint32_t* list, int* count, cudaStream_t s) {
  if (pb.n_obs == 0) return;
  switch (model) {
    case B200BA_MODEL_CENTRAL_GENERIC:
      residual_jacobian_kernel<B200BA_MODEL_CENTRAL_GENERIC, JAC, 2, true, JAC>
          <<<kStragglerBlocks, kStragglerThreads, 0, s>>>(pb, L, st, lp, out, huber, list, count, 0);
      break;
    case B200BA_MODEL_NONCENTRAL_GENERIC:
      residual_jacobian_kernel<B200BA_MODEL_NONCENTRAL_GENERIC, JAC, 2, true, false>
          <<<kStragglerBlocks, kStragglerThreads, 0, s>>>(pb, L, st, lp, out, huber, list, count, 0);
      break;
    case B200BA_MODEL_CENTRAL_OPENCV:
      break;  // closed-form projection: the main pass never defers
    default:
      residual_jacobian_kernel<-1, JAC, 2, true, false><<<kStragglerBlocks, kStragglerThreads, 0, s>>>(pb, L, st, lp, out, huber,
                                                                                                    list, count, 0);
  }
}

void launch_residual_jacobian(int uniform_model, bool jac, const ProblemDev& pb, const Layout& L,
                              const StateDev& st, double2* last_projection, const ObsOut& out, double huber,
                              uint32_t* straggler_list, int* straggler_count, cudaStream_t s,
                              cudaEvent_t main_done) {
  if (jac)
    launch_rj<true>(uniform_model, pb, L, st, last_projection, out, huber, straggler_list, straggler_count, s, main_done);
  else
    launch_rj<false>(uniform_model, pb, L, st, last_projection, out, huber, straggler_list, straggler_count, s, main_done);
}

void launch_straggler_pass(int uniform_model, bool jac, const ProblemDev& pb, const Layout& L, const StateDev& st,
                           double2* last_projection, const ObsOut& out, double huber, uint32_t* straggler_list,
                           int* straggler_count, cudaStream_t s) {
  if (jac)
    launch_stragglers<true>(uniform_model, pb, L, st, last_projection, out, huber, straggler_list, straggler_count, s);
  else
    launch_stragglers<false>(uniform_model, pb, L, st, last_projection, out, huber, straggler_list, straggler_count, s);
}

// b200ba_get_jacobians in compact mode: materialise the expanded SoA buffer from the compact records.
__global__ void expand_jacobian_kernel(ProblemDev pb, Layout L, StateDev st, ObsOut out, double* __restrict__ jac) {
  const int64_t o = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int col = blockIdx.y;
  if (o >= pb.n_obs) return;
  double jx = 0.0, jy = 0.0;
  if (out.has_jac[o] == kJacValid || out.has_jac[o] == kJacLate) load_jcol(pb, L, st, out, o, col, jx, jy);
  jac[(2 * static_cast<int64_t>(col)) * pb.n_obs + o] = jx;
  jac[(2 * static_cast<int64_t>(col) + 1) * pb.n_obs + o] = jy;
}
void launch_expand_jacobian(const ProblemDev& pb, const Layout& L, const StateDev& st, const ObsOut& out, double* jac,
                            cudaStream_t s) {
  if (pb.n_obs == 0 || L.n_jcols == 0) return;
  dim3 grid(static_cast<unsigned>((pb.n_obs + 127) / 128), L.n_jcols);
  expand_jacobian_kernel<<<grid, 128, 0, s>>>(pb, L, st, out, jac);
}

// Folds the late successes of the straggler pass into the normal equations: one warp per listed
// observation walks the upper triangle of its column set [point 3 | pose 6 | rig 6 | intrinsics K]
// with FP64 atomics (LV/lm_optimizer_jtj_accumulator_base.h:287-412). The list is short in the
// steady state; generality over speed.
__global__ void accumulate_list_kernel(ProblemDev pb, Layout L, StateDev st, ObsOut out, SystemDev sys, double huber,
                                       const uint32_t* __restrict__ list, const int* __restrict__ count) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5;
  const int64_t n_warps = (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5;
  const int64_t n = pb.n_obs;
  for (int64_t li = warp; li < *count; li += n_warps) {
    const int64_t o = list[li];
    if (out.has_jac[o] != kJacLate) continue;
    const int cam = static_cast<int>(pb.obs_camera[o]);
    const int iset = static_cast<int>(pb.obs_imageset[o]);
    const int pidx = static_cast<int>(pb.obs_point[o]);
    const CamDev& c = pb.cams[cam];
    const int cell = out.cell[o];
    const double rx = out.residual[o], ry = out.residual[n + o];
    const double w = huber_weight_sq(huber, rx * rx + ry * ry);
    const int K = L.localize_only ? 0 : c.K;
    const int nc = 9 + (L.rig_in_state ? 6 : 0) + K;
    // column e of this observation: Jacobian storage column and global unknown index
    auto jcol = [&](int e) -> int {
      if (e < 9) return e;  // point 0-2, pose 3-8
      if (L.rig_in_state && e < 15) return L.jc_rig + (e - 9);
      return L.jc_intr + (e - (L.rig_in_state ? 15 : 9));
    };
    auto gidx = [&](int e) -> int {  // global index in the reference ordering
      if (e < 3) return L.g_point + 3 * pidx + e;
      if (e < 9) return L.g_pose + 6 * iset + (e - 3);
      if (L.rig_in_state && e < 15) return L.g_rig + 6 * cam + (e - 9);
      return L.g_intr + intr_col(c, cell, e - (L.rig_in_state ? 15 : 9));
    };
    for (int p = lane; p < nc * nc; p += 32) {
      const int i = p / nc, j = p - i * nc;
      if (j < i) continue;
      const int ci = jcol(i), cj = jcol(j);
      double ax, ay, bx, by;
      load_jcol(pb, L, st, out, o, ci, ax, ay);
      load_jcol(pb, L, st, out, o, cj, bx, by);
      const double v = w * (ax * bx + ay * by);
      add_H(L, sys, gidx(i), gidx(j), v);
    }
    for (int i = lane; i < nc; i += 32) {
      const int ci = jcol(i);
      double ax, ay;
      load_jcol(pb, L, st, out, o, ci, ax, ay);
      const double v = w * (ax * rx + ay * ry);
      add_b(L, sys, gidx(i), v);
    }
    __syncwarp();
    if (lane == 0) out.has_jac[o] = kJacValid;
  }
}
void launch_accumulate_list(const ProblemDev& pb, const Layout& L, const StateDev& st, const ObsOut& out,
                            const SystemDev& sys, double huber, const uint32_t* list, const int* count, cudaStream_t s) {
  if (pb.n_obs == 0) return;
  accumulate_list_kernel<<<296, 128, 0, s>>>(pb, L, st, out, sys, huber, list, count);
}

// ------------------------------------------------------------------------------------------
// accumulation
// ------------------------------------------------------------------------------------------
// Global dense column of intrinsics entry k of an observation (models/central_grid.h:213-215,
// models/noncentral_generic.h:242-245, models/central_opencv.h:143-145).
__device__ __forceinline__ int intr_col(const CamDev& c, int cell, int k) {
  if (c.model_type == B200BA_MODEL_CENTRAL_GENERIC) {
    const int cp = k >> 1;
    return c.upd_off + 2 * (cell + (cp & 3) + (cp >> 2) * c.gw) + (k & 1);
  } else if (c.model_type == B200BA_MODEL_NONCENTRAL_GENERIC) {
    const int cp = k / 5;
    return c.upd_off + 5 * (cell + (cp & 3) + (cp >> 2) * c.gw) + (k - 5 * cp);
  }
  return c.upd_off + k;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

// H += (w J)^T J, b += (w J)^T r (LV/lm_optimizer_jtj_accumulator_base.h:287-412,
// LV/lm_optimizer_update_accumulator.h:180-360) for the small per-observation blocks:
//   point x point (3x3), pose x pose (6x6), point x pose (3x6), {point, pose} x rig, and the
//   matching b entries -- 54 (+ 54 with a rig) FP64 atomics per observation.
// Which of them land in the block-diagonal, off-diagonal or dense part depends on the
// elimination order and is decided by add_H(). Everything involving intrinsics columns, and
// rig x rig, is left to accumulate_cells_kernel.
__global__ void __launch_bounds__(128)
    accumulate_scatter_kernel(ProblemDev pb, Layout L, StateDev st, ObsOut out, SystemDev sys, double huber) {
  const int64_t o = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t n = pb.n_obs;
  if (o >= n || out.has_jac[o] != kJacValid) return;
  const int iset = static_cast<int>(pb.obs_imageset[o]);
  const int cam = static_cast<int>(pb.obs_camera[o]);
  const int pidx = static_cast<int>(pb.obs_point[o]);
  const double rx = out.residual[o], ry = out.residual[n + o];
  const double w = huber_weight_sq(huber, rx * rx + ry * ry);
  double jpx[3], jpy[3], jox[6], joy[6], jrx6[6], jry6[6];
  if (out.compact) {
    double jp[2][3], jo[2][6], jr[2][6];
    compact_small_blocks(pb, L, st, out, o, jp, jo, jr);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      jpx[a] = jp[0][a];
      jpy[a] = jp[1][a];
    }
#pragma unroll
    for (int a = 0; a < 6; ++a) {
      jox[a] = jo[0][a];
      joy[a] = jo[1][a];
      jrx6[a] = jr[0][a];
      jry6[a] = jr[1][a];
    }
  } else {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      jpx[a] = out.jac[(2 * static_cast<int64_t>(L.jc_point + a)) * n + o];
      jpy[a] = out.jac[(2 * static_cast<int64_t>(L.jc_point + a) + 1) * n + o];
    }
#pragma unroll
    for (int a = 0; a < 6; ++a) {
      jox[a] = out.jac[(2 * static_cast<int64_t>(L.jc_pose + a)) * n + o];
      joy[a] = out.jac[(2 * static_cast<int64_t>(L.jc_pose + a) + 1) * n + o];
      if (L.rig_in_state) {
        jrx6[a] = out.jac[(2 * static_cast<int64_t>(L.jc_rig + a)) * n + o];
        jry6[a] = out.jac[(2 * static_cast<int64_t>(L.jc_rig + a) + 1) * n + o];
      }
    }
  }
  const int gp = L.g_point + 3 * pidx, go = L.g_pose + 6 * iset;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double wx_ = w * jpx[a], wy_ = w * jpy[a];
#pragma unroll
    for (int b = a; b < 3; ++b) add_H(L, sys, gp + a, gp + b, wx_ * jpx[b] + wy_ * jpy[b]);
#pragma unroll
    for (int b = 0; b < 6; ++b) add_H(L, sys, gp + a, go + b, wx_ * jox[b] + wy_ * joy[b]);
    add_b(L, sys, gp + a, wx_ * rx + wy_ * ry);
  }
#pragma unroll
  for (int a = 0; a < 6; ++a) {
    const double wx_ = w * jox[a], wy_ = w * joy[a];
#pragma unroll
    for (int b = a; b < 6; ++b) add_H(L, sys, go + a, go + b, wx_ * jox[b] + wy_ * joy[b]);
    add_b(L, sys, go + a, wx_ * rx + wy_ * ry);
  }
  if (L.rig_in_state) {
    const int gr = L.g_rig + 6 * cam;
#pragma unroll
    for (int b = 0; b < 6; ++b) {
      const double wx_ = w * jrx6[b], wy_ = w * jry6[b];
#pragma unroll
      for (int a = 0; a < 3; ++a) add_H(L, sys, gp + a, gr + b, wx_ * jpx[a] + wy_ * jpy[a]);
#pragma unroll
      for (int a = 0; a < 6; ++a) add_H(L, sys, go + a, gr + b, wx_ * jox[a] + wy_ * joy[a]);
    }
  }
}

void launch_accumulate_scatter(const ProblemDev& pb, const Layout& L, const StateDev& st, const ObsOut& out,
                               const SystemDev& sys, double huber, cudaStream_t s) {
  const int threads = 128;
  const unsigned blocks = static_cast<unsigned>((pb.n_obs + threads - 1) / threads);
  if (blocks == 0) return;
  accumulate_scatter_kernel<<<blocks, threads, 0, s>>>(pb, L, st, out, sys, huber);
}

// (rig U intrinsics) x (rig U intrinsics) and the matching b entries, grouped by (camera,
// cell): every observation of a cell touches the same 4x4 control points, so the block sums
// the rank-2 updates of a run of equal cells in registers and issues ONE set of FP64 atomics
// per run (neighbouring cells overlap in control points, hence atomics rather than stores).
// Observations are stored in a static cell-major order (sorted once, at b200ba_create, by the
// cell of the MEASURED pixel), so runs are long; an observation whose projection currently
// falls into a neighbouring cell merely starts a short run of its own -- no per-iteration sort.
// A block owns kCellChunk consecutive observations.
constexpr int kCellChunk = 128;
constexpr int kCellTile = 32;
constexpr int kCellThreads = 256;
constexpr uint32_t kInvalidKey = 0xffffffffu;

__device__ __forceinline__ uint32_t cell_key(const ProblemDev& pb, const ObsOut& out, int64_t pos) {
  if (out.has_jac[pos] != kJacValid) return kInvalidKey;
  return (pb.obs_camera[pos] << 24) | static_cast<uint32_t>(out.cell[pos]);  // <= 8 cameras, < 2^24 cells
}

template <int MAXPAIRS>
__global__ void __launch_bounds__(kCellThreads)
    accumulate_cells_kernel(ProblemDev pb, Layout L, StateDev st, ObsOut out, SystemDev sys, double huber) {
  extern __shared__ double smem[];
  static_assert(kCellTile == 32, "one lane per observation of a tile");
  const int64_t n = pb.n_obs;
  const int64_t begin = static_cast<int64_t>(blockIdx.x) * kCellChunk;
  const int64_t end = min(n, begin + kCellChunk);
  const int rigE = L.rig_in_state ? 6 : 0;
  const int Emax = rigE + L.Kmax;
  const int S = Emax | 1;                  // odd row stride: lane-per-observation stores are conflict-free
  double* sJx = smem;                      // [32][S]  sqrt(w) * J row x of [rig | intrinsics]
  double* sJy = sJx + kCellTile * S;       // [32][S]
  double* sR = sJy + kCellTile * S;        // [32][2]  sqrt(w) * r
  double* sPx = sR + 2 * kCellTile;        // [32][9]  sqrt(w) * J row x of [point 3 | pose 6]
  double* sPy = sPx + 9 * kCellTile;       // [32][9]
  __shared__ double sObs[kCellTile * 16];  // compact mode: sw, wx[4], wy[4], Mn[6] per observation of the tile
  __shared__ double sTan[96];              // compact mode: tangent frames of the run's 4x4 control points
  __shared__ uint32_t sKey[kCellTile];
  __shared__ int sPoint[kCellTile];
  __shared__ int sIset[kCellTile];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int kWarps = kCellThreads / 32;
  constexpr int kSlots = (kMaxK + 31) / 32;  // intrinsics columns per lane

  double acc[MAXPAIRS];
  double accb = 0;
  int pi[MAXPAIRS], pj[MAXPAIRS];

  int64_t pos = begin;
  while (pos < end) {
    const uint32_t key = cell_key(pb, out, pos);
    if (key == kInvalidKey) {  // no Jacobian for this observation (uniform across the block)
      ++pos;
      continue;
    }
    const int cam = static_cast<int>(key >> 24);
    const int cell = static_cast<int>(key & 0xffffffu);
    const CamDev& c = pb.cams[cam];
    const int K = L.localize_only ? 0 : c.K;
    const int E = rigE + K;
    const int npairs = E * (E + 1) / 2;
    // pair -> (i, j), i <= j, row-major over the upper triangle
#pragma unroll
    for (int q = 0; q < MAXPAIRS; ++q) {
      acc[q] = 0;
      const int p = threadIdx.x + q * kCellThreads;
      int i = 0, j = 0;
      if (p < npairs) {
        int lo = 0, hi = E - 1;  // row i starts at offset i*E - i(i-1)/2
        while (lo < hi) {
          const int mid = (lo + hi + 1) >> 1;
          if (mid * E - mid * (mid - 1) / 2 <= p) lo = mid; else hi = mid - 1;
        }
        i = lo;
        j = i + (p - (i * E - i * (i - 1) / 2));
      }
      pi[q] = i;
      pj[q] = j;
    }
    accb = 0;
    // dense column (offset inside a row of B / C) of the intrinsics entries this lane covers
    int gck[kSlots];
#pragma unroll
    for (int s = 0; s < kSlots; ++s) {
      const int kk = lane + 32 * s;
      gck[s] = (kk < K) ? (L.g_intr + intr_col(c, cell, kk) - L.nbd) : -1;
    }
    // walk the run in tiles of 32 observations (lane <-> observation while staging)
    bool run_done = false;
    while (!run_done && pos < end) {
      const int tile_n = static_cast<int>(min(static_cast<int64_t>(kCellTile), end - pos));
      __syncthreads();
      if (threadIdx.x < tile_n) sKey[threadIdx.x] = cell_key(pb, out, pos + threadIdx.x);
      __syncthreads();
      int run_n = 0;
      while (run_n < tile_n && sKey[run_n] == key) ++run_n;
      if (run_n < tile_n) run_done = true;
      // stage sqrt(w) * J: warp <-> column, lane <-> observation (coalesced column reads)
      if (out.compact) {
        // compact records: per-observation quantities first (one lane per observation), then the columns
        // are rebuilt from shared memory: J(k) = sw * wx * wy * Mn [t1 t2]_k
        if (warp == 0 && lane < run_n) {
          const int64_t o = pos + lane;
          const double rx = out.residual[o], ry = out.residual[n + o];
          const double sw = sqrt(huber_weight_sq(huber, rx * rx + ry * ry));
          double wx[4], dwx[4], wy[4], dwy[4];
          bspline_basis(out.cjac[12 * n + o], wx, dwx);
          bspline_basis(out.cjac[13 * n + o], wy, dwy);
          double* so = sObs + lane * 16;
          so[0] = sw;
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            so[1 + q] = wx[q];
            so[5 + q] = wy[q];
          }
#pragma unroll
          for (int q = 0; q < 6; ++q) so[9 + q] = out.cjac[static_cast<int64_t>(6 + q) * n + o];
          sR[2 * lane] = sw * rx;
          sR[2 * lane + 1] = sw * ry;
          sPoint[lane] = static_cast<int>(pb.obs_point[o]);
          sIset[lane] = static_cast<int>(pb.obs_imageset[o]);
        }
        if (warp == 1 && lane < run_n) {
          const int64_t o = pos + lane;
          const double rx = out.residual[o], ry = out.residual[n + o];
          const double sw = sqrt(huber_weight_sq(huber, rx * rx + ry * ry));
          double jp[2][3], jo[2][6], jr[2][6];
          compact_small_blocks(pb, L, st, out, o, jp, jo, jr);
#pragma unroll
          for (int q = 0; q < 3; ++q) {
            sPx[lane * 9 + q] = sw * jp[0][q];
            sPy[lane * 9 + q] = sw * jp[1][q];
          }
#pragma unroll
          for (int q = 0; q < 6; ++q) {
            sPx[lane * 9 + 3 + q] = sw * jo[0][q];
            sPy[lane * 9 + 3 + q] = sw * jo[1][q];
            if (rigE) {
              sJx[lane * S + q] = sw * jr[0][q];
              sJy[lane * S + q] = sw * jr[1][q];
            }
          }
        }
        if (threadIdx.x >= 64 && threadIdx.x < 64 + 96 && K > 0) {
          const int q = threadIdx.x - 64, cp = q / 6;
          sTan[q] = st.tangents[c.tan_off + 6 * (static_cast<int64_t>(cell) + (cp & 3) + static_cast<int64_t>(cp >> 2) * c.gw) + (q - 6 * cp)];
        }
        __syncthreads();
        if (lane < run_n) {
          const double* so = sObs + lane * 16;
          for (int k = warp; k < K; k += kWarps) {
            const int cp = k >> 1;
            const double wk = so[0] * so[1 + (cp & 3)] * so[5 + (cp >> 2)];
            const double* t = sTan + 6 * cp + 3 * (k & 1);
            sJx[lane * S + rigE + k] = wk * (so[9] * t[0] + so[10] * t[1] + so[11] * t[2]);
            sJy[lane * S + rigE + k] = wk * (so[12] * t[0] + so[13] * t[1] + so[14] * t[2]);
          }
        }
      } else if (lane < run_n) {
        const int64_t o = pos + lane;
        const double rx = out.residual[o], ry = out.residual[n + o];
        const double sw = sqrt(huber_weight_sq(huber, rx * rx + ry * ry));
        for (int e = warp; e < E; e += kWarps) {
          const int col = (e < rigE) ? (L.jc_rig + e) : (L.jc_intr + (e - rigE));
          sJx[lane * S + e] = sw * out.jac[(2 * static_cast<int64_t>(col)) * n + o];
          sJy[lane * S + e] = sw * out.jac[(2 * static_cast<int64_t>(col) + 1) * n + o];
        }
        for (int r9 = warp; r9 < 9; r9 += kWarps) {
          const int col = (r9 < 3) ? (L.jc_point + r9) : (L.jc_pose + (r9 - 3));
          sPx[lane * 9 + r9] = sw * out.jac[(2 * static_cast<int64_t>(col)) * n + o];
          sPy[lane * 9 + r9] = sw * out.jac[(2 * static_cast<int64_t>(col) + 1) * n + o];
        }
        if (warp == 0) {
          sR[2 * lane] = sw * rx;
          sR[2 * lane + 1] = sw * ry;
          sPoint[lane] = static_cast<int>(pb.obs_point[o]);
          sIset[lane] = static_cast<int>(pb.obs_imageset[o]);
        }
      }
      __syncthreads();
      // [point | pose] rows x intrinsics columns of the run. A warp takes one (observation, row)
      // pair at a time and its lanes the consecutive intrinsics columns of that ONE matrix row:
      // the warp-wide FP64 RED touches a few contiguous sectors instead of 32 scattered ones.
      if (K > 0) {
        for (int q = warp; q < run_n * 9; q += kWarps) {
          const int t = q / 9, r9 = q - 9 * t;
          const double px = sPx[t * 9 + r9], py = sPy[t * 9 + r9];
          const int grow = (r9 < 3) ? (L.g_point + 3 * sPoint[t] + r9) : (L.g_pose + 6 * sIset[t] + (r9 - 3));
          // intrinsics columns are dense and come last in both orderings: row < column always
          double* rowp = (grow < L.nbd) ? (sys.B + static_cast<int64_t>(grow) * L.nd)
                                        : (sys.C + static_cast<int64_t>(grow - L.nbd) * L.nd);
          const double* jx = sJx + t * S + rigE;
          const double* jy = sJy + t * S + rigE;
#pragma unroll
          for (int s = 0; s < kSlots; ++s) {
            const int kk = lane + 32 * s;
            if (kk < K) atomicAdd(rowp + gck[s], fma(px, jx[kk], py * jy[kk]));
          }
        }
      }
      // (rig U intrinsics)^2 and b: register accumulation over the run
#pragma unroll
      for (int q = 0; q < MAXPAIRS; ++q) {
        if (threadIdx.x + q * kCellThreads < npairs) {
          double a = acc[q];
          const double* xi = sJx + pi[q];
          const double* xj = sJx + pj[q];
          const double* yi = sJy + pi[q];
          const double* yj = sJy + pj[q];
          for (int t = 0; t < run_n; ++t) a = fma(xi[t * S], xj[t * S], fma(yi[t * S], yj[t * S], a));
          acc[q] = a;
        }
      }
      if (threadIdx.x < E) {
        double a = accb;
        for (int t = 0; t < run_n; ++t)
          a = fma(sJx[t * S + threadIdx.x], sR[2 * t], fma(sJy[t * S + threadIdx.x], sR[2 * t + 1], a));
        accb = a;
      }
      pos += run_n;
    }
    // flush the run
    auto gcol = [&](int e) -> int {  // rig and intrinsics are dense variables in both elimination orders
      return (e < rigE) ? (L.g_rig + 6 * cam + e) : (L.g_intr + intr_col(c, cell, e - rigE));
    };
#pragma unroll
    for (int q = 0; q < MAXPAIRS; ++q) {
      if (threadIdx.x + q * kCellThreads < npairs) {
        const int gi = gcol(pi[q]) - L.nbd, gj = gcol(pj[q]) - L.nbd;  // both dense, gi <= gj
        atomicAdd(&sys.C[static_cast<int64_t>(gi) * L.nd + gj], acc[q]);
      }
    }
    if (threadIdx.x < E) atomicAdd(&sys.bd[gcol(threadIdx.x) - L.nbd], accb);
  }
}

void launch_accumulate_cells(const ProblemDev& pb, const Layout& L, const StateDev& st, const ObsOut& out,
                             const SystemDev& sys, double huber, cudaStream_t s) {
  if (pb.n_obs == 0) return;
  const int rigE = L.rig_in_state ? 6 : 0;
  const int Emax = rigE + L.Kmax;
  if (Emax == 0) return;
  const int npairs = Emax * (Emax + 1) / 2;
  const int per_thread = (npairs + kCellThreads - 1) / kCellThreads;
  const size_t smem = (2 * static_cast<size_t>(kCellTile) * (Emax | 1) + 2 * kCellTile + 18 * kCellTile) * sizeof(double);
  const unsigned blocks = static_cast<unsigned>((pb.n_obs + kCellChunk - 1) / kCellChunk);
#define B200BA_LAUNCH_CELLS(MP)                                                                              \
  do {                                                                                                       \
    cudaFuncSetAttribute(accumulate_cells_kernel<MP>, cudaFuncAttributeMaxDynamicSharedMemorySize,           \
                         static_cast<int>(smem));                                                            \
    accumulate_cells_kernel<MP><<<blocks, kCellThreads, smem, s>>>(pb, L, st, out, sys, huber);              \
  } while (0)
  if (per_thread <= 1)
    B200BA_LAUNCH_CELLS(1);
  else if (per_thread <= 3)
    B200BA_LAUNCH_CELLS(3);
  else if (per_thread <= 4)
    B200BA_LAUNCH_CELLS(4);
  else if (per_thread <= 13)
    B200BA_LAUNCH_CELLS(13);
  else
    B200BA_LAUNCH_CELLS(15);
#undef B200BA_LAUNCH_CELLS
}

// ------------------------------------------------------------------------------------------
// Schur complement helpers (LV/lm_optimizer.h:1246-1369)
// ------------------------------------------------------------------------------------------
// Per block: L = chol(D_i + lambda I) (lower), Linv = L^-1 (packed lower, row-major), v = Linv b_i.
// D_i is stored as its packed upper triangle. A non-positive pivot raises *fail (the caller
// rejects the attempt like the reference rejects a NaN update).
template <int BS>
__global__ void schur_blocks_kernel(int n_blocks, const double* __restrict__ Dblk, const double* __restrict__ bp,
                                    double lambda, double* __restrict__ Linv, double* __restrict__ v, int* fail) {
  constexpr int DSZ = BS * (BS + 1) / 2;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_blocks) return;
  const double* D = Dblk + static_cast<int64_t>(DSZ) * p;
  double A[BS][BS], Lm[BS][BS], Li[BS][BS];
#pragma unroll
  for (int a = 0; a < BS; ++a)
#pragma unroll
    for (int b = a; b < BS; ++b) {
      const double d = D[a * BS - (a * (a - 1)) / 2 + (b - a)] + (a == b ? lambda : 0.0);
      A[a][b] = d;
      A[b][a] = d;
    }
  bool bad = false;
#pragma unroll
  for (int j = 0; j < BS; ++j) {
    double s = A[j][j];
#pragma unroll
    for (int k2 = 0; k2 < j; ++k2) s -= Lm[j][k2] * Lm[j][k2];
    if (!(s > 0)) bad = true;
    const double ljj = sqrt(s);
    Lm[j][j] = ljj;
#pragma unroll
    for (int i = j + 1; i < BS; ++i) {
      double t = A[i][j];
#pragma unroll
      for (int k2 = 0; k2 < j; ++k2) t -= Lm[i][k2] * Lm[j][k2];
      Lm[i][j] = t / ljj;
    }
  }
  if (bad) *fail = 1;
  // inverse of the lower-triangular factor by forward substitution, column by column
#pragma unroll
  for (int c2 = 0; c2 < BS; ++c2) {
#pragma unroll
    for (int i = 0; i < BS; ++i) {
      if (i < c2) {
        Li[i][c2] = 0;
      } else {
        double t = (i == c2) ? 1.0 : 0.0;
#pragma unroll
        for (int k2 = c2; k2 < i; ++k2) t -= Lm[i][k2] * Li[k2][c2];
        Li[i][c2] = t / Lm[i][i];
      }
    }
  }
  double* out = Linv + static_cast<int64_t>(DSZ) * p;
#pragma unroll
  for (int i = 0; i < BS; ++i)
#pragma unroll
    for (int j = 0; j <= i; ++j) out[(i * (i + 1)) / 2 + j] = Li[i][j];
#pragma unroll
  for (int i = 0; i < BS; ++i) {
    double t = 0;
#pragma unroll
    for (int j = 0; j <= i; ++j) t += Li[i][j] * bp[BS * p + j];
    v[BS * p + i] = t;
  }
}
void launch_schur_blocks(int bs, int n_blocks, const double* Dblk, const double* bp, double lambda, double* Linv,
                         double* v, int* fail, cudaStream_t s) {
  if (n_blocks == 0) return;
  if (bs == 3)
    schur_blocks_kernel<3><<<(n_blocks + 127) / 128, 128, 0, s>>>(n_blocks, Dblk, bp, lambda, Linv, v, fail);
  else
    schur_blocks_kernel<6><<<(n_blocks + 127) / 128, 128, 0, s>>>(n_blocks, Dblk, bp, lambda, Linv, v, fail);
}

// W = L^-1 B, BS rows per block. With D^-1 = L^-T L^-1 the contraction B^T D^-1 B
// (LV/lm_optimizer.h:1294-1311,1328) becomes the symmetric rank-k update W^T W.
template <int BS>
__global__ void schur_scale_rows_kernel(int nd, const double* __restrict__ B, const double* __restrict__ Linv,
                                        double* __restrict__ W) {
  constexpr int DSZ = BS * (BS + 1) / 2;
  const int p = blockIdx.y;
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= nd) return;
  const double* Li = Linv + static_cast<int64_t>(DSZ) * p;
  const int64_t r0 = static_cast<int64_t>(BS) * p * nd + col;
  double b[BS];
#pragma unroll
  for (int i = 0; i < BS; ++i) b[i] = B[r0 + static_cast<int64_t>(i) * nd];
#pragma unroll
  for (int i = 0; i < BS; ++i) {
    double t = 0;
#pragma unroll
    for (int j = 0; j <= i; ++j) t = fma(Li[(i * (i + 1)) / 2 + j], b[j], t);
    W[r0 + static_cast<int64_t>(i) * nd] = t;
  }
}
void launch_schur_scale_rows(int bs, int n_blocks, int nd, const double* B, const double* Linv, double* W,
                             cudaStream_t s) {
  if (n_blocks == 0 || nd == 0) return;
  dim3 grid((nd + 255) / 256, n_blocks);
  if (bs == 3)
    schur_scale_rows_kernel<3><<<grid, 256, 0, s>>>(nd, B, Linv, W);
  else
    schur_scale_rows_kernel<6><<<grid, 256, 0, s>>>(nd, B, Linv, W);
}

// x_b = L^-T y_b, y = v - W x_d (back-substitution, LV/lm_optimizer.h:1366-1367)
template <int BS>
__global__ void schur_backsub_kernel(int n_blocks, const double* __restrict__ Linv, const double* __restrict__ y,
                                     double* __restrict__ xp) {
  constexpr int DSZ = BS * (BS + 1) / 2;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_blocks) return;
  const double* Li = Linv + static_cast<int64_t>(DSZ) * p;
#pragma unroll
  for (int j = 0; j < BS; ++j) {
    double t = 0;
#pragma unroll
    for (int i = j; i < BS; ++i) t += Li[(i * (i + 1)) / 2 + j] * y[BS * p + i];
    xp[BS * p + j] = t;
  }
}
void launch_schur_backsub(int bs, int n_blocks, const double* Linv, const double* y, double* xp, cudaStream_t s) {
  if (n_blocks == 0) return;
  if (bs == 3)
    schur_backsub_kernel<3><<<(n_blocks + 127) / 128, 128, 0, s>>>(n_blocks, Linv, y, xp);
  else
    schur_backsub_kernel<6><<<(n_blocks + 127) / 128, 128, 0, s>>>(n_blocks, Linv, y, xp);
}

// ------------------------------------------------------------------------------------------
// Structured Schur contraction: S -= W^T W exploiting the exact zeros of B
// ------------------------------------------------------------------------------------------
// A pattern point is observed through a limited part of the image, so its three rows of the
// off-diagonal block B touch only the control points under those pixels (config 2: ~15 % of the
// 10 080 intrinsics columns). Schur blocks are grouped by image locality (host, at layout time);
// per group the union of non-zero dense columns is detected from B itself (exact, per build),
// the group's rows of W = L^-1 B are gathered into a compact k_g x m_g panel, a dense FP64
// rank-k update runs on the compact panel (library dsyrk, tensor-core DMMA) and the m_g x m_g
// result is scattered into S. Flops drop from n_d^2 * 3P to sum_g m_g^2 k_g (5x at config 2).

// flags[g][c] = 1 iff some row of group g has a non-zero in dense column c
__global__ void group_support_kernel(int bs, int nblocks, int nd, const double* __restrict__ B,
                                     const int* __restrict__ group_of_block, uint8_t* __restrict__ flags) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int blk0 = blockIdx.y * 8;
  if (c >= nd) return;
  for (int blk = blk0; blk < min(blk0 + 8, nblocks); ++blk) {
    bool nz = false;
    for (int r = 0; r < bs; ++r) nz |= (B[(static_cast<int64_t>(blk) * bs + r) * nd + c] != 0.0);
    if (nz) flags[static_cast<int64_t>(group_of_block[blk]) * nd + c] = 1;
  }
}
void launch_group_support(int bs, int nblocks, int nd, const double* B, const int* group_of_block, uint8_t* flags,
                          cudaStream_t s) {
  if (nblocks == 0 || nd == 0) return;
  dim3 grid((nd + 255) / 256, (nblocks + 7) / 8);
  group_support_kernel<<<grid, 256, 0, s>>>(bs, nblocks, nd, B, group_of_block, flags);
}

// cols[g][0 .. count[g]) = sorted dense columns flagged for group g (one block per group)
__global__ void compact_columns_kernel(int nd, const uint8_t* __restrict__ flags, int* __restrict__ cols,
                                       int* __restrict__ count) {
  const int g = blockIdx.x;
  const uint8_t* f = flags + static_cast<int64_t>(g) * nd;
  int* out = cols + static_cast<int64_t>(g) * nd;
  __shared__ int warp_sums[32];
  __shared__ int base;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int c0 = 0; c0 < nd; c0 += blockDim.x) {
    const int c = c0 + threadIdx.x;
    const int v = (c < nd && f[c]) ? 1 : 0;
    const unsigned bal = __ballot_sync(0xffffffffu, v);
    const int in_warp = __popc(bal & ((1u << lane) - 1));
    if (lane == 0) warp_sums[warp] = __popc(bal);
    __syncthreads();
    int off = base;
    for (int w = 0; w < warp; ++w) off += warp_sums[w];
    if (v) out[off + in_warp] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
      int tot = 0;
      for (int w = 0; w < nwarps; ++w) tot += warp_sums[w];
      base += tot;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) count[g] = base;
}
void launch_compact_columns(int ngroups, int nd, const uint8_t* flags, int* cols, int* count, cudaStream_t s) {
  if (ngroups == 0) return;
  compact_columns_kernel<<<ngroups, 1024, 0, s>>>(nd, flags, cols, count);
}

// Wc[(lb * BS + r) * ldw + j] = sum_k Linv[blk][r][k] * B[(blk * BS + k)][cols[j]]  for the blocks of one group
template <int BS>
__global__ void gather_scale_kernel(int nd, int m, int ldw, const double* __restrict__ B, const double* __restrict__ Linv,
                                    const int* __restrict__ blocks, const int* __restrict__ cols,
                                    double* __restrict__ Wc) {
  constexpr int DSZ = BS * (BS + 1) / 2;
  const int lb = blockIdx.y;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m) return;
  const int blk = blocks[lb];
  const int c = cols[j];
  const double* Li = Linv + static_cast<int64_t>(DSZ) * blk;
  double b[BS];
#pragma unroll
  for (int i = 0; i < BS; ++i) b[i] = B[(static_cast<int64_t>(blk) * BS + i) * nd + c];
#pragma unroll
  for (int i = 0; i < BS; ++i) {
    double t = 0;
#pragma unroll
    for (int q = 0; q <= i; ++q) t = fma(Li[(i * (i + 1)) / 2 + q], b[q], t);
    Wc[(static_cast<int64_t>(lb) * BS + i) * ldw + j] = t;
  }
}
void launch_gather_scale(int bs, int nblocks_in_group, int nd, int m, int ldw, const double* B, const double* Linv,
                         const int* blocks, const int* cols, double* Wc, cudaStream_t s) {
  if (nblocks_in_group == 0 || m == 0) return;
  dim3 grid((m + 255) / 256, nblocks_in_group);
  if (bs == 3)
    gather_scale_kernel<3><<<grid, 256, 0, s>>>(nd, m, ldw, B, Linv, blocks, cols, Wc);
  else
    gather_scale_kernel<6><<<grid, 256, 0, s>>>(nd, m, ldw, B, Linv, blocks, cols, Wc);
}

// S[cols[j] * nd + cols[i]] -= P[j * m + i] for i >= j (column-major lower triangles on both sides)
__global__ void scatter_sub_kernel(int nd, int m, const int* __restrict__ cols, const double* __restrict__ P,
                                   double* __restrict__ S) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int j = blockIdx.y;
  if (i >= m || i < j) return;
  S[static_cast<int64_t>(cols[j]) * nd + cols[i]] -= P[static_cast<int64_t>(j) * m + i];
}
void launch_scatter_sub(int nd, int m, const int* cols, const double* P, double* S, cudaStream_t s) {
  if (m == 0) return;
  dim3 grid((m + 255) / 256, m);
  scatter_sub_kernel<<<grid, 256, 0, s>>>(nd, m, cols, P, S);
}

// u = L^-T v  (= D^-1 b for the block), per block
template <int BS>
__global__ void block_solve_t_kernel(int n_blocks, const double* __restrict__ Linv, const double* __restrict__ v,
                                     double* __restrict__ u) {
  constexpr int DSZ = BS * (BS + 1) / 2;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_blocks) return;
  const double* Li = Linv + static_cast<int64_t>(DSZ) * p;
#pragma unroll
  for (int j = 0; j < BS; ++j) {
    double t = 0;
#pragma unroll
    for (int i = j; i < BS; ++i) t += Li[(i * (i + 1)) / 2 + j] * v[BS * p + i];
    u[BS * p + j] = t;
  }
}
void launch_block_solve_t(int bs, int n_blocks, const double* Linv, const double* v, double* u, cudaStream_t s) {
  if (n_blocks == 0) return;
  if (bs == 3)
    block_solve_t_kernel<3><<<(n_blocks + 127) / 128, 128, 0, s>>>(n_blocks, Linv, v, u);
  else
    block_solve_t_kernel<6><<<(n_blocks + 127) / 128, 128, 0, s>>>(n_blocks, Linv, v, u);
}

// x_b = u - L^-T (L^-1 t)   with t = B x_d  (back-substitution without materialising W)
template <int BS>
__global__ void block_backsub2_kernel(int n_blocks, const double* __restrict__ Linv, const double* __restrict__ u,
                                      const double* __restrict__ t, double* __restrict__ xb) {
  constexpr int DSZ = BS * (BS + 1) / 2;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_blocks) return;
  const double* Li = Linv + static_cast<int64_t>(DSZ) * p;
  double y[BS];
#pragma unroll
  for (int i = 0; i < BS; ++i) {
    double a = 0;
#pragma unroll
    for (int q = 0; q <= i; ++q) a += Li[(i * (i + 1)) / 2 + q] * t[BS * p + q];
    y[i] = a;
  }
#pragma unroll
  for (int j = 0; j < BS; ++j) {
    double a = 0;
#pragma unroll
    for (int i = j; i < BS; ++i) a += Li[(i * (i + 1)) / 2 + j] * y[i];
    xb[BS * p + j] = u[BS * p + j] - a;
  }
}
void launch_block_backsub2(int bs, int n_blocks, const double* Linv, const double* u, const double* t, double* xb,
                           cudaStream_t s) {
  if (n_blocks == 0) return;
  if (bs == 3)
    block_backsub2_kernel<3><<<(n_blocks + 127) / 128, 128, 0, s>>>(n_blocks, Linv, u, t, xb);
  else
    block_backsub2_kernel<6><<<(n_blocks + 127) / 128, 128, 0, s>>>(n_blocks, Linv, u, t, xb);
}

// S(i, i) = C(i, i) + lambda (LV/lm_optimizer.h:839-852: the damping is ADDED to the diagonal)
__global__ void add_diagonal_kernel(int n, double* M, int64_t ld, double lambda) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) M[static_cast<int64_t>(i) * ld + i] += lambda;
}
void launch_add_diagonal(int n, double* M, int64_t ld, double lambda, cudaStream_t s) {
  if (n == 0) return;
  add_diagonal_kernel<<<(n + 255) / 256, 256, 0, s>>>(n, M, ld, lambda);
}

// trace of H = sum of the block diagonals + sum diag(C) for the lambda initialisation
// (LV/lm_optimizer.h:766-781); single block, deterministic order.
__global__ void trace_kernel(int n_blocks, int bs, const double* __restrict__ Dblk, int nd,
                             const double* __restrict__ C, double* out) {
  __shared__ double sh[256];
  const int dsz = bs * (bs + 1) / 2;
  double a = 0;
  for (int p = threadIdx.x; p < n_blocks; p += blockDim.x) {
    const double* D = Dblk + static_cast<int64_t>(dsz) * p;
    for (int i = 0; i < bs; ++i) a += D[i * bs - (i * (i - 1)) / 2];
  }
  for (int i = threadIdx.x; i < nd; i += blockDim.x) a += C[static_cast<int64_t>(i) * nd + i];
  sh[threadIdx.x] = a;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = sh[0];
}
void launch_trace(int n_blocks, int bs, const double* Dblk, int nd, const double* C, double* out, cudaStream_t s) {
  trace_kernel<<<1, 256, 0, s>>>(n_blocks, bs, Dblk, nd, C, out);
}

// ------------------------------------------------------------------------------------------
// state retraction (JointOptimizationState::operator-=, joint_optimization.cc:172-214)
// ------------------------------------------------------------------------------------------
// ApplyLocalUpdateToQuaternion (local_parametrizations/quaternion_parametrization.h:39-60)
// keeps |update| and sin|u|/|u| in FLOAT; SE3d(q, t) then normalises the quaternion.
__device__ __forceinline__ void retract_pose(const double* src, double* dst, const double* delta) {
  const double u0 = -delta[0], u1 = -delta[1], u2 = -delta[2];
  q4 q{src[0], src[1], src[2], src[3]};
  const float norm_update = static_cast<float>(sqrt(u0 * u0 + u1 * u1 + u2 * u2));
  if (norm_update != 0.0f) {
    // float sin / cos of a float argument, correctly rounded via the double routines
    const float s = static_cast<float>(sin(static_cast<double>(norm_update)));
    const float cw = static_cast<float>(cos(static_cast<double>(norm_update)));
    const float sbu = s / norm_update;
    q4 uq{static_cast<double>(cw), static_cast<double>(sbu) * u0, static_cast<double>(sbu) * u1,
          static_cast<double>(sbu) * u2};
    q = qmul(uq, q);
  }
  const double nrm = sqrt(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
  dst[0] = q.w / nrm;
  dst[1] = q.x / nrm;
  dst[2] = q.y / nrm;
  dst[3] = q.z / nrm;
  dst[4] = src[4] - delta[3];
  dst[5] = src[5] - delta[4];
  dst[6] = src[6] - delta[5];
}

__global__ void update_state_kernel(ProblemDev pb, Layout L, StateDev src, StateDev dst, const double* __restrict__ x,
                                    int64_t n_control_total, int64_t n_param_total) {
  const int64_t tid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  // segment 0: point coordinates
  const int64_t n_pc = 3 * static_cast<int64_t>(L.n_points);
  if (tid < n_pc) {
    dst.points[tid] = src.points[tid] - x[L.g_point + tid];
    return;
  }
  int64_t k = tid - n_pc;
  // segment 1: imageset poses
  if (k < L.n_imagesets) {
    retract_pose(src.rig_tr_global + 7 * k, dst.rig_tr_global + 7 * k, x + L.g_pose + 6 * k);
    return;
  }
  k -= L.n_imagesets;
  // segment 2: camera_tr_rig (variables only when there is more than one camera)
  if (k < L.n_cameras) {
    if (L.rig_in_state) {
      retract_pose(src.camera_tr_rig + 7 * k, dst.camera_tr_rig + 7 * k, x + L.g_rig + 6 * k);
    } else {
      for (int i = 0; i < 7; ++i) dst.camera_tr_rig[7 * k + i] = src.camera_tr_rig[7 * k + i];
    }
    return;
  }
  k -= L.n_cameras;
  // segment 3: control points of the generic models (models/central_grid.h:168-184,
  // models/noncentral_generic.h:195-219)
  if (k < n_control_total) {
    int cam = 0;
    int64_t local = k;
    for (int c = 0; c < L.n_cameras; ++c) {
      const int64_t G = static_cast<int64_t>(pb.cams[c].gw) * pb.cams[c].gh;
      if (local < G) {
        cam = c;
        break;
      }
      local -= G;
    }
    const CamDev& c = pb.cams[cam];
    const double* g = src.intrinsics + c.intr_off + 3 * local;
    double* go = dst.intrinsics + c.intr_off + 3 * local;
    const d3 dir = mk3(g[0], g[1], g[2]);
    if (L.localize_only) {
      go[0] = dir.x;
      go[1] = dir.y;
      go[2] = dir.z;
      if (c.model_type == B200BA_MODEL_NONCENTRAL_GENERIC) {
        const int64_t G3 = 3 * static_cast<int64_t>(c.gw) * c.gh;
        for (int i = 0; i < 3; ++i) go[G3 + i] = g[G3 + i];
      }
      return;
    }
    d3 t1, t2;
    compute_tangents(dir, t1, t2);
    const double* dl = x + L.g_intr + c.upd_off + c.dof_per_point * local;
    const d3 nd_ = (dir + (-dl[0]) * t1) + (-dl[1]) * t2;
    const double nn = sqrt(dot3(nd_, nd_));
    go[0] = nd_.x / nn;
    go[1] = nd_.y / nn;
    go[2] = nd_.z / nn;
    if (c.model_type == B200BA_MODEL_NONCENTRAL_GENERIC) {
      const int64_t G3 = 3 * static_cast<int64_t>(c.gw) * c.gh;
      const d3 org = mk3(g[G3], g[G3 + 1], g[G3 + 2]);
      // ApplyLocalUpdateToLine (line_parametrization.h:107-120)
      const d3 no = ((org + (-dl[2]) * t1) + (-dl[3]) * t2) + (-dl[4]) * dir;
      go[G3] = no.x;
      go[G3 + 1] = no.y;
      go[G3 + 2] = no.z;
    }
    return;
  }
  k -= n_control_total;
  // segment 4: parametric models (models/central_opencv.h:91-94)
  if (k < n_param_total) {
    int cam = 0;
    int64_t local = k;
    for (int c = 0; c < L.n_cameras; ++c) {
      const int64_t np = (pb.cams[c].gw == 0) ? 12 : 0;
      if (local < np) {
        cam = c;
        break;
      }
      local -= np;
    }
    const CamDev& c = pb.cams[cam];
    const double d = L.localize_only ? 0.0 : x[L.g_intr + c.upd_off + local];
    dst.intrinsics[c.intr_off + local] = src.intrinsics[c.intr_off + local] - d;
  }
}
void launch_update_state(const ProblemDev& pb, const Layout& L, const StateDev& src, const StateDev& dst,
                         const double* x, int64_t n_control_total, int64_t n_param_total, cudaStream_t s) {
  const int64_t n = 3 * static_cast<int64_t>(L.n_points) + L.n_imagesets + L.n_cameras + n_control_total + n_param_total;
  update_state_kernel<<<static_cast<unsigned>((n + 127) / 128), 128, 0, s>>>(pb, L, src, dst, x, n_control_total,
                                                                             n_param_total);
}

// ------------------------------------------------------------------------------------------
// cost comparison (LV/lm_optimizer.h:993-1011) + totals; two deterministic stages
// ------------------------------------------------------------------------------------------
// out[0] = sum of trial costs over residuals valid in BOTH states, out[1] = same for the base
// state, out[2] = number of such residuals, out[3] = total trial cost (all valid trial
// residuals), out[4] = number of valid trial residuals, out[5] = sum |r|^2 of valid trial
// residuals (for the RMSE). base may be NULL (then out[1], out[2] refer to trial only).
// 2 blocks on each of the H100's 132 SMs (equal shares of the grid-stride loop); a compile-time constant,
// not the device's SM count, so that the summation order and hence the cost are the same on every GPU
constexpr int kReduceBlocks = 264;
constexpr int kReduceThreads = 256;
__global__ void __launch_bounds__(kReduceThreads)
    cost_reduce_stage1(int64_t n, const double* __restrict__ trial, const double* __restrict__ base,
                       const double* __restrict__ residual, double* __restrict__ partial) {
  double a[6] = {0, 0, 0, 0, 0, 0};
  for (int64_t o = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; o < n;
       o += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const double t = trial[o];
    const double b = base ? base[o] : 0.0;
    if (t >= 0 && b >= 0) {
      a[0] += t;
      a[1] += b;
      a[2] += 1;
    }
    if (t >= 0) {
      a[3] += t;
      a[4] += 1;
      if (residual) {
        const double rx = residual[o], ry = residual[n + o];
        a[5] += rx * rx + ry * ry;
      }
    }
  }
  __shared__ double sh[6][kReduceThreads];
#pragma unroll
  for (int q = 0; q < 6; ++q) sh[q][threadIdx.x] = a[q];
  __syncthreads();
  for (int s = kReduceThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
#pragma unroll
      for (int q = 0; q < 6; ++q) sh[q][threadIdx.x] += sh[q][threadIdx.x + s];
    }
    __syncthreads();
  }
  if (threadIdx.x < 6) partial[blockIdx.x * 6 + threadIdx.x] = sh[threadIdx.x][0];
}
__global__ void cost_reduce_stage2(int nblocks, const double* __restrict__ partial, double* __restrict__ out) {
  if (threadIdx.x < 6) {
    double a = 0;
    for (int b = 0; b < nblocks; ++b) a += partial[b * 6 + threadIdx.x];
    out[threadIdx.x] = a;
  }
}
void launch_cost_reduce(int64_t n, const double* trial, const double* base, const double* residual, double* partial,
                        double* out, cudaStream_t s) {
  cost_reduce_stage1<<<kReduceBlocks, kReduceThreads, 0, s>>>(n, trial, base, residual, partial);
  cost_reduce_stage2<<<1, 32, 0, s>>>(kReduceBlocks, partial, out);
}
int cost_reduce_partial_size() { return kReduceBlocks * 6; }

// ------------------------------------------------------------------------------------------
// stand-alone model evaluation (b200ba_project / b200ba_unproject)
// ------------------------------------------------------------------------------------------
__global__ void project_points_kernel(CamDev c, const double* __restrict__ intr, int64_t n,
                                      const double* __restrict__ lp, double* __restrict__ px, int32_t* ok) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const d3 p = mk3(lp[3 * i], lp[3 * i + 1], lp[3 * i + 2]);
  double x = px[2 * i], y = px[2 * i + 1];
  bool r = false;
  if (c.model_type == B200BA_MODEL_CENTRAL_GENERIC) {
    CentralEval e;
    int ne = 0;
    if (in_area(c, x, y)) r = central_project(c, intr, rsqrt(dot3(p, p)) * p, x, y, e, ne, kUnlimitedEvals) == kProjOk;
  } else if (c.model_type == B200BA_MODEL_NONCENTRAL_GENERIC) {
    NoncentralEval e;
    d3 t1, t2;
    double R[2][2];
    int ne = 0;
    if (in_area(c, x, y)) r = noncentral_project(c, intr, intr + 3 * static_cast<int64_t>(c.gw) * c.gh, p, x, y, e, t1, t2, R, ne, kUnlimitedEvals) == kProjOk;
  } else {
    r = opencv_project(c, intr, p, x, y);
  }
  px[2 * i] = x;
  px[2 * i + 1] = y;
  ok[i] = r ? 1 : 0;
}
void launch_project_points(const CamDev& c, const double* intr, int64_t n, const double* lp, double* px, int32_t* ok,
                           cudaStream_t s) {
  if (n == 0) return;
  project_points_kernel<<<static_cast<unsigned>((n + 127) / 128), 128, 0, s>>>(c, intr, n, lp, px, ok);
}

__global__ void unproject_pixels_kernel(CamDev c, const double* __restrict__ intr, int64_t n,
                                        const double* __restrict__ px, double* __restrict__ dirs,
                                        double* __restrict__ origins, int32_t* ok) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const double x = px[2 * i], y = px[2 * i + 1];
  d3 d = mk3(0, 0, 0), o = mk3(0, 0, 0);
  bool r = false;
  if (in_area(c, x, y)) {
    if (c.model_type == B200BA_MODEL_CENTRAL_GENERIC) {
      CentralEval e;
      central_eval(c, intr, x, y, e);
      d = e.u;
      r = true;
    } else if (c.model_type == B200BA_MODEL_NONCENTRAL_GENERIC) {
      NoncentralEval e;
      noncentral_eval(c, intr, intr + 3 * static_cast<int64_t>(c.gw) * c.gh, x, y, e);
      d = e.u;
      o = e.o;
      r = true;
    }
  }
  if (dirs) {
    dirs[3 * i] = d.x;
    dirs[3 * i + 1] = d.y;
    dirs[3 * i + 2] = d.z;
  }
  if (origins) {
    origins[3 * i] = o.x;
    origins[3 * i + 1] = o.y;
    origins[3 * i + 2] = o.z;
  }
  ok[i] = r ? 1 : 0;
}
void launch_unproject_pixels(const CamDev& c, const double* intr, int64_t n, const double* px, double* dirs,
                             double* origins, int32_t* ok, cudaStream_t s) {
  if (n == 0) return;
  unproject_pixels_kernel<<<static_cast<unsigned>((n + 127) / 128), 128, 0, s>>>(c, intr, n, px, dirs, origins, ok);
}

// ------------------------------------------------------------------------------------------
// calibration report (APP/calibration_report.cc:83-98, per camera :713-817)
// ------------------------------------------------------------------------------------------
// Everything below works on the device (cell-major) observation order, in which every camera is
// one contiguous range [cam_off[c], cam_off[c + 1]). Bin and cell indices depend on the last bit
// of the values they are computed from, so those expressions use __dmul_rn / __dadd_rn (no FMA
// contraction) and evaluate in the reference's order; the CPU side is compiled with
// -ffp-contract=off for the same reason.

// static_cast<int>(double) as x86-64 executes it (cvttsd2si): truncation toward zero, and INT_MIN
// for NaN and for values outside the int range, where CUDA's conversion would saturate instead.
__device__ __forceinline__ int report_trunc(double v) {
  return (v > -2147483649.0 && v < 2147483648.0) ? static_cast<int>(v) : INT_MIN;
}

// Eigen's Vector2d::norm(): sqrt(x * x + y * y) with no fused multiply-add
__device__ __forceinline__ double report_norm(double x, double y) {
  return sqrt(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)));
}

// ComputeAllReprojectionErrors (:101-148): local point from the image_tr_global cache, Project()
// (start at CenterOfCalibratedArea, no warm start; central_grid.h:79-97, noncentral_generic.h:88-93)
// with the projection code of the residual kernel. err = pixel - xy, NaN where Project fails.
__global__ void report_errors_kernel(ProblemDev pb, int n_cameras, StateDev st, double2* __restrict__ err,
                                     double* __restrict__ mag) {
  const int64_t o = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (o >= pb.n_obs) return;
  const int iset = static_cast<int>(pb.obs_imageset[o]);
  const int cam = static_cast<int>(pb.obs_camera[o]);
  const CamDev& c = pb.cams[cam];
  const double* T = st.image_tr_global + 12 * (static_cast<int64_t>(iset) * n_cameras + cam);
  double R[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) R[i] = __ldg(T + i);
  const d3 lp = rot_apply(R, ld3(st.points + 3 * static_cast<int64_t>(pb.obs_point[o]))) +
                mk3(__ldg(T + 9), __ldg(T + 10), __ldg(T + 11));
  const double* intr = st.intrinsics + c.intr_off;
  double px = c.center_x, py = c.center_y;
  bool ok;
  if (c.model_type == B200BA_MODEL_CENTRAL_GENERIC) {
    CentralEval e;
    int ne = 0;
    ok = central_project(c, intr, rsqrt(dot3(lp, lp)) * lp, px, py, e, ne, kUnlimitedEvals) == kProjOk;
  } else if (c.model_type == B200BA_MODEL_NONCENTRAL_GENERIC) {
    NoncentralEval e;
    d3 t1, t2;
    double Rn[2][2];
    int ne = 0;
    ok = noncentral_project(c, intr, intr + 3 * static_cast<int64_t>(c.gw) * c.gh, lp, px, py, e, t1, t2, Rn, ne,
                            kUnlimitedEvals) == kProjOk;
  } else {
    ok = opencv_project(c, intr, lp, px, py);
  }
  if (!ok) {
    err[o] = make_double2(nan(""), nan(""));
    mag[o] = nan("");
    return;
  }
  const float2 xy = pb.obs_xy[o];
  const double ex = px - static_cast<double>(xy.x), ey = py - static_cast<double>(xy.y);
  err[o] = make_double2(ex, ey);
  mag[o] = report_norm(ex, ey);
}

// count, sum and max of |e| per camera: two stages with a compile-time grid, like cost_reduce_stage1/2,
// so that the sum is the same on every GPU.
constexpr int kReportBlocks = 132;
constexpr int kReportThreads = 256;
__global__ void __launch_bounds__(kReportThreads)
    report_reduce_stage1(const int64_t* __restrict__ cam_off, const double* __restrict__ mag, double* __restrict__ partial) {
  const int cam = blockIdx.y;
  double cnt = 0, sum = 0, mx = 0;
  for (int64_t o = cam_off[cam] + blockIdx.x * static_cast<int64_t>(kReportThreads) + threadIdx.x; o < cam_off[cam + 1];
       o += static_cast<int64_t>(kReportBlocks) * kReportThreads) {
    const double m = mag[o];
    if (!isnan(m)) {
      cnt += 1;
      sum += m;
      mx = fmax(mx, m);
    }
  }
  __shared__ double sh[3][kReportThreads];
  sh[0][threadIdx.x] = cnt;
  sh[1][threadIdx.x] = sum;
  sh[2][threadIdx.x] = mx;
  __syncthreads();
  for (int s = kReportThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      sh[0][threadIdx.x] += sh[0][threadIdx.x + s];
      sh[1][threadIdx.x] += sh[1][threadIdx.x + s];
      sh[2][threadIdx.x] = fmax(sh[2][threadIdx.x], sh[2][threadIdx.x + s]);
    }
    __syncthreads();
  }
  if (threadIdx.x < 3) partial[(static_cast<int64_t>(cam) * kReportBlocks + blockIdx.x) * 3 + threadIdx.x] = sh[threadIdx.x][0];
}
__global__ void report_reduce_stage2(int n_cameras, const double* __restrict__ partial, ReportCam* __restrict__ rc) {
  const int cam = threadIdx.x;
  if (cam >= n_cameras) return;
  double cnt = 0, sum = 0, mx = 0;
  for (int b = 0; b < kReportBlocks; ++b) {
    const double* p = partial + (static_cast<int64_t>(cam) * kReportBlocks + b) * 3;
    cnt += p[0];
    sum += p[1];
    mx = fmax(mx, p[2]);
  }
  ReportCam& r = rc[cam];
  r.count = static_cast<long long>(cnt);
  r.sum = sum;
  r.max = mx;
  r.select_prefix = 0;
  r.select_rank = r.count / 2;
}

// Median (WriteReportInfoFile, :685-693: sorted(|e|)[count / 2]) by radix select on the bit patterns:
// non-negative doubles order like their uint64 patterns. 8 passes of 8 bits; pass p histograms digit
// 7 - p of the values whose higher digits equal the prefix chosen so far. Every range can select
// `ranks` ranks at once: slot s = range * ranks + j keeps its own prefix, rank and histogram.
constexpr int kSelectBlocks = 132;
__global__ void __launch_bounds__(kReportThreads)
    report_select_hist_kernel(int pass, int ranks, const int64_t* __restrict__ cam_off, const double* __restrict__ mag,
                              const ReportCam* __restrict__ rc, unsigned int* __restrict__ hist) {
  const int slot = blockIdx.y, cam = slot / ranks;
  __shared__ unsigned int h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  const int shift = 56 - 8 * pass;
  const unsigned long long prefix = rc[slot].select_prefix;
  for (int64_t o = cam_off[cam] + blockIdx.x * static_cast<int64_t>(kReportThreads) + threadIdx.x; o < cam_off[cam + 1];
       o += static_cast<int64_t>(kSelectBlocks) * kReportThreads) {
    const double m = mag[o];
    if (isnan(m)) continue;
    const unsigned long long bits = static_cast<unsigned long long>(__double_as_longlong(m));
    if (pass > 0 && ((bits ^ prefix) >> (shift + 8)) != 0) continue;
    atomicAdd(&h[(bits >> shift) & 255], 1u);
  }
  __syncthreads();
  if (h[threadIdx.x]) atomicAdd(&hist[slot * 256 + threadIdx.x], h[threadIdx.x]);
}
__global__ void report_select_scan_kernel(int pass, int n_slots, unsigned int* __restrict__ hist,
                                          ReportCam* __restrict__ rc) {
  const int slot = threadIdx.x;
  if (slot >= n_slots) return;
  ReportCam& r = rc[slot];
  unsigned int* h = hist + slot * 256;
  long long k = r.select_rank;
  int digit = 255;
  for (int d = 0; d < 256; ++d) {
    if (k < static_cast<long long>(h[d])) {
      digit = d;
      break;
    }
    k -= h[d];
  }
  for (int d = 0; d < 256; ++d) h[d] = 0;
  r.select_rank = k;
  r.select_prefix |= static_cast<unsigned long long>(digit) << (56 - 8 * pass);
  if (pass == 7) r.median = r.count > 0 ? __longlong_as_double(static_cast<long long>(r.select_prefix)) : nan("");
}

// ComputeReprojectionErrorHistogram (:151-168) with kHistResolution = 50, kHistExtent = 0.2f (:739-743):
// hx_f = (50 * 0.5f) * (e.x / extent + 1.f), hx = int(hx_f) - (hx_f < 0 ? 1.f : 0.f) (a float subtraction)
__device__ __forceinline__ int report_hist_bin(double e) {
  const double extent = static_cast<double>(0.2f);
  const double f = __dmul_rn(25.0, __dadd_rn(e / extent, 1.0));
  const int i = report_trunc(f);
  return f < 0 ? report_trunc(static_cast<double>(static_cast<float>(i) - 1.f)) : i;
}
constexpr int kHistBlocks = 66;
__global__ void __launch_bounds__(kReportThreads)
    report_hist_kernel(const int64_t* __restrict__ cam_off, const double2* __restrict__ err, int* __restrict__ hist) {
  const int cam = blockIdx.y;
  constexpr int kBins = B200BA_REPORT_HIST * B200BA_REPORT_HIST;
  __shared__ int h[kBins];
  for (int i = threadIdx.x; i < kBins; i += kReportThreads) h[i] = 0;
  __syncthreads();
  for (int64_t o = cam_off[cam] + blockIdx.x * static_cast<int64_t>(kReportThreads) + threadIdx.x; o < cam_off[cam + 1];
       o += static_cast<int64_t>(kHistBlocks) * kReportThreads) {
    const double2 e = err[o];
    if (isnan(e.x)) continue;
    const int hx = report_hist_bin(e.x), hy = report_hist_bin(e.y);
    if (hx >= 0 && hy >= 0 && hx < B200BA_REPORT_HIST && hy < B200BA_REPORT_HIST) atomicAdd(&h[hy * B200BA_REPORT_HIST + hx], 1);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kBins; i += kReportThreads)
    if (h[i]) atomicAdd(&hist[cam * kBins + i], h[i]);
}

// ComputeBiasedness (:171-351), one warp per (camera, bias cell). order lists the device positions of
// the cell's observations in the caller's order (cell_off: [n_cameras * 2500 + 1]). Lane 0 takes the
// Welford mean of |e| (libvis statistics.h:55-63) in that order; cells with fewer than 5 errors are
// skipped (kl = NaN). The lanes bin e * (1.25331 / mean) into the 8 x 8 table (:284-296), lane 0 sums
// P log(P / Q) over the non-empty bins in y-then-x order (:328-337).
__device__ __forceinline__ int report_bias_bin(double n) {
  // -1 * (n * (0.5 * 8) / 2.5 - 0.5 * 8), truncated, clamped to [0, 7]
  const double v = -__dadd_rn(__dmul_rn(n, 4.0) / 2.5, -4.0);
  return min(7, max(0, report_trunc(v)));
}
__global__ void __launch_bounds__(256)
    report_bias_kernel(int n_cells, const int* __restrict__ cell_off, const uint32_t* __restrict__ order,
                       const double2* __restrict__ err, const double* __restrict__ mag, const double* __restrict__ Q,
                       double* __restrict__ kl) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int cell = blockIdx.x * 8 + warp;
  __shared__ int bins[8][64];
  if (cell >= n_cells) return;
  const int a = cell_off[cell], b = cell_off[cell + 1];
  double mean = 0;
  unsigned int count = 0;
  if (lane == 0) {
    for (int i = a; i < b; ++i) {
      const double m = mag[order[i]];
      if (isnan(m)) continue;
      ++count;
      const double delta = m - mean;
      mean = __dadd_rn(mean, delta / static_cast<double>(count));
    }
  }
  count = __shfl_sync(0xffffffffu, count, 0);
  mean = __shfl_sync(0xffffffffu, mean, 0);
  if (count < 5) {
    if (lane == 0) kl[cell] = nan("");
    return;
  }
  bins[warp][lane] = 0;
  bins[warp][lane + 32] = 0;
  __syncwarp();
  const double s = 1.25331 / mean;
  for (int i = a + lane; i < b; i += 32) {
    const double2 e = err[order[i]];
    if (isnan(e.x)) continue;
    atomicAdd(&bins[warp][report_bias_bin(__dmul_rn(e.y, s)) * 8 + report_bias_bin(__dmul_rn(e.x, s))], 1);
  }
  __syncwarp();
  if (lane == 0) {
    const double total = static_cast<double>(count);
    double d = 0;
    for (int k = 0; k < 64; ++k) {
      const int c = bins[warp][k];
      if (c == 0) continue;
      const double P = c / total;
      d = __dadd_rn(d, __dmul_rn(P, log(P / Q[k])));
    }
    kl[cell] = d;
  }
}

// Biasedness = sorted(KL)[size / 2] over the cells that were not skipped: one block per camera sorts its
// (at most 2 500) values with a bitonic network in shared memory.
constexpr int kBiasSortN = 4096;
__global__ void __launch_bounds__(1024) report_bias_median_kernel(const double* __restrict__ kl, ReportCam* __restrict__ rc) {
  constexpr int kCells = kReportBiasCells * kReportBiasCells;
  const int cam = blockIdx.x;
  __shared__ double v[kBiasSortN];
  int valid = 0;
  for (int i = threadIdx.x; i < kBiasSortN; i += blockDim.x) {
    const double x = i < kCells ? kl[cam * kCells + i] : nan("");
    v[i] = isnan(x) ? INFINITY : x;
    valid += isnan(x) ? 0 : 1;
  }
  __shared__ int n_valid;
  if (threadIdx.x == 0) n_valid = 0;
  __syncthreads();
  atomicAdd(&n_valid, valid);
  for (int k = 2; k <= kBiasSortN; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      __syncthreads();
      for (int i = threadIdx.x; i < kBiasSortN; i += blockDim.x) {
        const int p = i ^ j;
        if (p > i) {
          const bool up = (i & k) == 0;
          const double x = v[i], y = v[p];
          if ((x > y) == up) {
            v[i] = y;
            v[p] = x;
          }
        }
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    rc[cam].biasedness_cells = n_valid;
    rc[cam].biasedness = n_valid > 0 ? v[n_valid / 2] : nan("");
  }
}

// ComputeApproximateFOV (:609-645) for central-generic cameras: Unproject at
// (min_x + 0.5f, 0.5f * height) and (max_x + 0.5f, 0.5f * height), angle between the normalised
// directions times width / (max_x - min_x) (a float ratio); vertically alike. -1 where an
// un-projection fails, for non-central cameras (as in the reference) and for OpenCV cameras (the model's
// iterative undistortion has no device code).
__device__ __forceinline__ bool report_unproject(const CamDev& c, const double* intr, float x, float y, d3& d) {
  if (!in_area(c, x, y)) return false;
  CentralEval e;
  central_eval(c, intr, x, y, e);
  d = rsqrt(dot3(e.u, e.u)) * e.u;
  return true;
}
__global__ void report_fov_kernel(ProblemDev pb, int n_cameras, StateDev st, ReportCam* __restrict__ rc) {
  const int cam = threadIdx.x;
  if (cam >= n_cameras) return;
  const CamDev& c = pb.cams[cam];
  double hfov = -1, vfov = -1;
  if (c.model_type == B200BA_MODEL_CENTRAL_GENERIC) {
    const double* intr = st.intrinsics + c.intr_off;
    d3 a, b;
    const float min_x = c.min_x + 0.5f, max_x = c.max_x + 0.5f, y = 0.5f * c.height;
    if (report_unproject(c, intr, min_x, y, a) && report_unproject(c, intr, max_x, y, b))
      hfov = acos(dot3(a, b)) * static_cast<double>(c.width / (max_x - min_x));
    const float min_y = c.min_y + 0.5f, max_y = c.max_y + 0.5f, x = 0.5f * c.width;
    if (report_unproject(c, intr, x, min_y, a) && report_unproject(c, intr, x, max_y, b))
      vfov = acos(dot3(a, b)) * static_cast<double>(c.height / (max_y - min_y));
  }
  rc[cam].hfov = hfov;
  rc[cam].vfov = vfov;
}

// count / sum / max in the fixed two-stage order and the exact median of the non-NaN mag values of
// every range [off[c], off[c + 1]), c < n_ranges (<= 32); results in rc[c].
void launch_report_statistics(int n_ranges, const int64_t* off, const double* mag, double* partial,
                              unsigned int* select_hist, ReportCam* rc, cudaStream_t s) {
  report_reduce_stage1<<<dim3(kReportBlocks, n_ranges), kReportThreads, 0, s>>>(off, mag, partial);
  report_reduce_stage2<<<1, 32, 0, s>>>(n_ranges, partial, rc);
  launch_report_select(n_ranges, 1, off, mag, select_hist, rc, s);
}

// The radix select of launch_report_statistics alone: rc[range * ranks + j].select_rank (set by the caller, prefix 0)
// becomes the value of that rank among the non-NaN mag of the range, in .median (its bits in .select_prefix).
void launch_report_select(int n_ranges, int ranks, const int64_t* off, const double* mag, unsigned int* select_hist,
                          ReportCam* rc, cudaStream_t s) {
  cudaMemsetAsync(select_hist, 0, sizeof(unsigned int) * 256 * n_ranges * ranks, s);
  for (int pass = 0; pass < 8; ++pass) {
    report_select_hist_kernel<<<dim3(kSelectBlocks, n_ranges * ranks), kReportThreads, 0, s>>>(pass, ranks, off, mag, rc,
                                                                                              select_hist);
    report_select_scan_kernel<<<1, 32, 0, s>>>(pass, n_ranges * ranks, select_hist, rc);
  }
}

void launch_calibration_report(const ProblemDev& pb, int n_cameras, const StateDev& st, const ReportDev& r,
                               cudaStream_t s) {
  launch_report_errors(pb, n_cameras, st, r, s);
  launch_report_statistics(n_cameras, r.cam_off, r.mag, r.partial, r.select_hist, r.cams, s);
  cudaMemsetAsync(r.hist, 0, sizeof(int) * n_cameras * B200BA_REPORT_HIST * B200BA_REPORT_HIST, s);
  report_hist_kernel<<<dim3(kHistBlocks, n_cameras), kReportThreads, 0, s>>>(r.cam_off, r.err, r.hist);
  const int n_cells = n_cameras * kReportBiasCells * kReportBiasCells;
  report_bias_kernel<<<(n_cells + 7) / 8, 256, 0, s>>>(n_cells, r.cell_off, r.cell_order, r.err, r.mag, r.Q, r.kl);
  report_bias_median_kernel<<<n_cameras, 1024, 0, s>>>(r.kl, r.cams);
  report_fov_kernel<<<1, 32, 0, s>>>(pb, n_cameras, st, r.cams);
}
int report_partial_size(int n_cameras) { return n_cameras * kReportBlocks * 3; }
void launch_report_errors(const ProblemDev& pb, int n_cameras, const StateDev& st, const ReportDev& r, cudaStream_t s) {
  const int64_t n = pb.n_obs;
  if (n > 0) report_errors_kernel<<<static_cast<unsigned>((n + 127) / 128), 128, 0, s>>>(pb, n_cameras, st, r.err, r.mag);
}

// ------------------------------------------------------------------------------------------
// outlier round of one camera (DeleteOutlierFeatures, APP/calibration.cc:62-184) on the report's errors
// ------------------------------------------------------------------------------------------
// The camera's observations are the device range [a, a + n). All arithmetic that decides a rank, a
// threshold or a colour is rounded operation by operation (no contraction), in the reference's order.

// |e| of the observations on used imagesets (NaN where the imageset is unused or Project failed)
__global__ void outlier_mag_kernel(ProblemDev pb, int64_t a, int64_t n, const double* __restrict__ rmag,
                                   const uint8_t* __restrict__ used, double* __restrict__ mag) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  mag[i] = used[pb.obs_imageset[a + i]] ? rmag[a + i] : nan("");
}

// ranks of the quartiles, reprojection_errors[0.25f * size + 0.5f] and [0.75f * size + 0.5f]: float
// arithmetic, truncated to size_t
__global__ void outlier_ranks_kernel(ReportCam* __restrict__ st) {
  const long long count = st[0].count;
  const float c = static_cast<float>(count);
  st[1] = st[0];
  st[0].select_rank = static_cast<long long>(__fadd_rn(__fmul_rn(0.25f, c), 0.5f));
  st[1].select_rank = static_cast<long long>(__fadd_rn(__fmul_rn(0.75f, c), 0.5f));
  st[0].select_prefix = st[1].select_prefix = 0;
}

// threshold = q3 + (double)factor * (q3 - q1)
__device__ __forceinline__ double outlier_threshold(const ReportCam* st, float factor) {
  const double q1 = st[0].median, q3 = st[1].median;
  return __dadd_rn(q3, __dmul_rn(static_cast<double>(factor), __dadd_rn(q3, -q1)));
}

// the pixel ((u32)x, (u32)y) of a feature, or -1 where a truncated coordinate is outside the image
__device__ __forceinline__ int64_t outlier_pixel(float2 xy, int w, int h) {
  const float tx = truncf(xy.x), ty = truncf(xy.y);
  if (!(tx >= 0.f && tx < static_cast<float>(w) && ty >= 0.f && ty < static_cast<float>(h))) return -1;
  return static_cast<int64_t>(ty) * w + static_cast<int64_t>(tx);
}

// remove = !ok || |e| > threshold for the observations on used imagesets; counts kept features per
// imageset, removed / failed features, and marks each pixel with 1 + the largest caller index removed there
__global__ void outlier_decide_kernel(ProblemDev pb, int64_t a, int64_t n, const double* __restrict__ rmag,
                                      const uint32_t* __restrict__ perm, OutlierDev d, float factor, int w, int h) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n || d.stats[0].count < 8) return;
  const int64_t o = a + i;
  const uint32_t iset = pb.obs_imageset[o];
  if (!d.used[iset]) return;
  const double m = rmag[o];
  if (!isnan(m) && !(m > outlier_threshold(d.stats, factor))) {
    atomicAdd(&d.kept[iset], 1);
    return;
  }
  const uint32_t caller = perm[o];
  d.remove[caller] = 1;
  atomicAdd(&d.counts[0], 1ull);
  if (isnan(m)) atomicAdd(&d.counts[1], 1ull);
  if (d.owner) {
    const int64_t p = outlier_pixel(pb.obs_xy[o], w, h);
    if (p >= 0) atomicMax(&d.owner[p], caller + 1);
  }
}

// the colour of the last removed feature (caller's order) at every marked pixel
__global__ void outlier_colour_kernel(ProblemDev pb, int64_t a, int64_t n, const double* __restrict__ rmag,
                                      const uint32_t* __restrict__ perm, OutlierDev d, int w, int h) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int64_t o = a + i;
  const int64_t p = outlier_pixel(pb.obs_xy[o], w, h);
  if (p < 0 || d.owner[p] != perm[o] + 1) return;
  const double m = rmag[o];
  uint8_t r = 255, g = 255, b = 255;
  if (isnan(m)) {
    r = g = b = 127;
  } else if (m > 10) {
    g = b = 0;
  } else if (m > 5) {
    g = 127;
    b = 0;
  } else if (m > 1) {
    b = 0;
  }
  d.image[3 * p] = r;
  d.image[3 * p + 1] = g;
  d.image[3 * p + 2] = b;
}

// imagesets left with fewer than 3 features of the camera become unused
__global__ void outlier_drop_kernel(int n_imagesets, OutlierDev d) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_imagesets || d.stats[0].count < 8) return;
  if (d.used[i] && d.kept[i] < 3) d.used[i] = 0;
}

void launch_delete_outliers(const ProblemDev& pb, int n_imagesets, const ReportDev& r, const uint32_t* perm,
                            int64_t a, int64_t n, float factor, int w, int h, const OutlierDev& d, cudaStream_t s) {
  const unsigned blocks = static_cast<unsigned>(std::max<int64_t>(1, (n + 255) / 256));
  outlier_mag_kernel<<<blocks, 256, 0, s>>>(pb, a, n, r.mag, d.used, d.mag);
  report_reduce_stage1<<<dim3(kReportBlocks, 1), kReportThreads, 0, s>>>(d.range, d.mag, d.partial);
  report_reduce_stage2<<<1, 32, 0, s>>>(1, d.partial, d.stats);
  outlier_ranks_kernel<<<1, 1, 0, s>>>(d.stats);
  launch_report_select(1, 2, d.range, d.mag, d.select_hist, d.stats, s);
  outlier_decide_kernel<<<blocks, 256, 0, s>>>(pb, a, n, r.mag, perm, d, factor, w, h);
  if (d.owner) outlier_colour_kernel<<<blocks, 256, 0, s>>>(pb, a, n, r.mag, perm, d, w, h);
  outlier_drop_kernel<<<std::max(1, (n_imagesets + 255) / 256), 256, 0, s>>>(n_imagesets, d);
}

// ------------------------------------------------------------------------------------------
// comparison of two central-generic models (CreateFittingErrorReport, APP/fitting_report.h:83-125,
// with parametric_r_dense = Identity and no border; called by tools/compare_calibrations.cc:68-72)
// ------------------------------------------------------------------------------------------
// One thread per pixel (x, y) of the image, in 2-D tiles so that a warp works on neighbouring pixels
// and therefore on the same control points:
//   A un-projects (x + 0.5f, y + 0.5f): outside A's calibrated area the pixel is skipped (NaN outputs);
//   B un-projects the same pixel: error = dir_B - dir_A, or +inf where B fails;
//   the two direction maxima over the pixels where both succeed;
//   B.Project(dir_A) from the centre of B's calibrated area (no warm start): e = pixel - projection.
// mag = |e| (NaN where A or Project fails) feeds launch_report_statistics.
// With `angles` set, the pass also writes _fitting_error_direction_angles.png (fitting_report.h:144-157), the one
// image that needs the two directions rather than their difference and depends on no maximum.
constexpr int kCompareTileX = 16, kCompareTileY = 8;
__device__ __forceinline__ bool compare_unproject(const CamDev& c, const double* __restrict__ grid, double x, double y,
                                                  d3& d) {
  if (!in_area(c, x, y)) return false;  // CentralGenericModel::Unproject (central_generic.h:97-105)
  CentralEval e;
  central_eval(c, grid, x, y, e);
  d = e.u;
  return true;
}
// std::min<int>(255, std::max<int>(0, 127 + 127 / (M_PI / 180.f * 0.025) * (g - f) + 0.5)) (fitting_report.h:155-156):
// evaluated left to right in double, converted to int as x86-64 does (INT_MIN for NaN, hence 0)
__device__ __forceinline__ uint8_t fitting_angle(double g, double f) {
  constexpr double kScale = 127 / (3.14159265358979323846 / static_cast<double>(180.f) * 0.025);
  const double v = __dadd_rn(__dadd_rn(127.0, __dmul_rn(kScale, __dsub_rn(g, f))), 0.5);
  return static_cast<uint8_t>(min(255, max(0, report_trunc(v))));
}
// kAngles: whether `angles` is set; a separate instance, so that the comparison alone keeps its register budget
template <bool kAngles>
__global__ void __launch_bounds__(kCompareTileX * kCompareTileY)
    compare_models_kernel(CamDev ca, const double* __restrict__ ga, CamDev cb, const double* __restrict__ gb,
                          double* __restrict__ mag, double* __restrict__ dir_err, double* __restrict__ rep_err,
                          unsigned long long* __restrict__ dir_max, uint8_t* __restrict__ angles) {
  const int x = blockIdx.x * kCompareTileX + threadIdx.x;
  const int y = blockIdx.y * kCompareTileY + threadIdx.y;
  const bool inside = x < ca.width && y < ca.height;
  double max_norm = 0, max_comp = 0;
  if (inside) {
    const int64_t p = static_cast<int64_t>(y) * ca.width + x;
    // the reference passes x + 0.5f (a float) where Unproject takes a double
    const double px = static_cast<double>(x + 0.5f), py = static_cast<double>(y + 0.5f);
    const double nan_v = nan("");
    double m = nan_v, ex = nan_v, ey = nan_v;
    d3 da;
    uint8_t ang0 = 0, ang1 = 0, ang2 = 0;  // (0, 0, 0) where A fails (error.hasNaN())
    if (compare_unproject(ca, ga, px, py, da)) {
      d3 db, err;
      if (compare_unproject(cb, gb, px, py, db)) {
        // __dsub_rn: the normalisation's product inside db must not be fused into this subtraction, so that
        // dir_B - dir_A is the difference of the two rounded directions (exactly 0 when A and B agree)
        err = mk3(__dsub_rn(db.x, da.x), __dsub_rn(db.y, da.y), __dsub_rn(db.z, da.z));
        max_comp = fmax(fabs(err.x), fmax(fabs(err.y), fabs(err.z)));
        // Vector3d::norm() in Eigen's order, no fused multiply-add
        max_norm = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(err.x, err.x), __dmul_rn(err.y, err.y)), __dmul_rn(err.z, err.z)));
      } else {
        err = mk3(INFINITY, INFINITY, INFINITY);
        // the reference reads its uninitialised fitted direction here; pinned as NaN, which gives (0, 0, 127)
        db = mk3(nan_v, nan_v, nan_v);
      }
      if (kAngles && !(isnan(err.x) || isnan(err.y) || isnan(err.z))) {
        ang0 = fitting_angle(atan2(da.z, da.x), atan2(db.z, db.x));
        ang1 = fitting_angle(atan2(da.y, da.z), atan2(db.y, db.z));
        ang2 = 127;
      }
      if (dir_err) {
        dir_err[3 * p] = err.x;
        dir_err[3 * p + 1] = err.y;
        dir_err[3 * p + 2] = err.z;
      }
      // CentralGridModel::Project (central_grid.h:79-97): normalise, start at CenterOfCalibratedArea()
      double qx = cb.center_x, qy = cb.center_y;
      CentralEval e;
      int ne = 0;
      if (central_project(cb, gb, rsqrt(dot3(da, da)) * da, qx, qy, e, ne, kUnlimitedEvals) == kProjOk) {
        ex = px - qx;
        ey = py - qy;
        m = report_norm(ex, ey);
      }
    } else if (dir_err) {
      dir_err[3 * p] = dir_err[3 * p + 1] = dir_err[3 * p + 2] = nan_v;
    }
    mag[p] = m;
    if (rep_err) {
      rep_err[2 * p] = ex;
      rep_err[2 * p + 1] = ey;
    }
    if (kAngles) {
      angles[3 * p] = ang0;
      angles[3 * p + 1] = ang1;
      angles[3 * p + 2] = ang2;
    }
  }
  // first stage of the maxima: the block's maximum, then one atomicMax per block on the bit patterns
  // (non-negative doubles order like their uint64 patterns; max is order-independent, so this is exact)
  for (int o = 16; o > 0; o >>= 1) {
    max_norm = fmax(max_norm, __shfl_xor_sync(0xffffffffu, max_norm, o));
    max_comp = fmax(max_comp, __shfl_xor_sync(0xffffffffu, max_comp, o));
  }
  constexpr int kWarps = kCompareTileX * kCompareTileY / 32;
  __shared__ double sh[2][kWarps];
  const int t = threadIdx.y * kCompareTileX + threadIdx.x;
  if ((t & 31) == 0) {
    sh[0][t >> 5] = max_norm;
    sh[1][t >> 5] = max_comp;
  }
  __syncthreads();
  if (t < 2) {
    double v = 0;
    for (int w = 0; w < kWarps; ++w) v = fmax(v, sh[t][w]);
    if (v > 0) atomicMax(dir_max + t, static_cast<unsigned long long>(__double_as_longlong(v)));
  }
}

// The other four images of CreateFittingErrorReport (fitting_report.h:141-177), one thread per pixel, from the
// comparison's dir_err and mag and the three maxima as the statistics left them on the device. Every value is
// evaluated in the reference's order and float/double mix and converted to u8 as x86-64 does (report_trunc, then the
// low byte):
//   magnitude     255.99f * (|e| / max_error_norm); 0 where e = +inf (B fails) and where 0 / 0;
//   direction     (255.99f / 2) * (min(max(e / max_error_component, -1), 1) + 1) per component, where std::min /
//                 std::max (Eigen's cwiseMin / cwiseMax) keep their first argument when a comparison sees NaN;
//   reprojection  max<float>(0, min<float>(255, 255.99f * |r| / reprojection_error_max)), |r| = 0 where A or
//   magnitude     Project fails (the reference's image holds zero there; mag holds NaN);
// and (0, 0, 0) for the first two where A fails (e = NaN). The reprojection-direction image is
// 127 + s * 127 * (sin, cos)(atan2(-r.y, -r.x)), 127, + 0.5f with the strength s = max(0, min(1, |r| / -1)): the tool
// passes max_visualization_extent_pixels = -1, so s = 0 for every |r| >= 0 and every pixel is (127, 127, 127).
constexpr int kFittingImageThreads = 256;
__global__ void __launch_bounds__(kFittingImageThreads)
    fitting_images_kernel(int64_t n, const double* __restrict__ dir_err, const double* __restrict__ mag,
                          const unsigned long long* __restrict__ dir_max, const ReportCam* __restrict__ stats,
                          uint8_t* __restrict__ magnitudes, uint8_t* __restrict__ directions,
                          uint8_t* __restrict__ rep_magnitudes, uint8_t* __restrict__ reprojections) {
  const int64_t p = static_cast<int64_t>(blockIdx.x) * kFittingImageThreads + threadIdx.x;
  if (p >= n) return;
  const double max_norm = __longlong_as_double(static_cast<long long>(dir_max[0]));
  const double max_comp = __longlong_as_double(static_cast<long long>(dir_max[1]));
  const double rep_max = stats->max;
  const double k = static_cast<double>(255.99f), k_half = static_cast<double>(255.99f / 2);
  const double e[3] = {dir_err[3 * p], dir_err[3 * p + 1], dir_err[3 * p + 2]};
  uint8_t m = 0, dir[3] = {0, 0, 0};
  if (!(isnan(e[0]) || isnan(e[1]) || isnan(e[2]))) {
    for (int c = 0; c < 3; ++c) {
      double r = __ddiv_rn(e[c], max_comp);
      r = r < -1.0 ? -1.0 : r;  // std::max(r, -1): r if the comparison is false, NaN included
      r = 1.0 < r ? 1.0 : r;    // std::min(r, 1)
      dir[c] = static_cast<uint8_t>(report_trunc(__dmul_rn(k_half, __dadd_rn(r, 1.0))));
    }
    const double norm = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(e[0], e[0]), __dmul_rn(e[1], e[1])), __dmul_rn(e[2], e[2])));
    m = static_cast<uint8_t>(report_trunc(__dmul_rn(k, __ddiv_rn(norm, max_norm))));
  }
  const double r_norm = isnan(mag[p]) ? 0.0 : mag[p];
  float v = __double2float_rn(__ddiv_rn(__dmul_rn(k, r_norm), rep_max));
  v = v < 255.f ? v : 255.f;  // std::min<float>(255, v): 255 for NaN
  v = 0.f < v ? v : 0.f;      // std::max<float>(0, v)
  magnitudes[p] = m;
  directions[3 * p] = dir[0];
  directions[3 * p + 1] = dir[1];
  directions[3 * p + 2] = dir[2];
  rep_magnitudes[p] = static_cast<uint8_t>(report_trunc(v));
  reprojections[3 * p] = reprojections[3 * p + 1] = reprojections[3 * p + 2] = 127;
}

void launch_compare_models(const CamDev& a, const double* ga, const CamDev& b, const double* gb, const CompareDev& d,
                           cudaStream_t s) {
  cudaMemsetAsync(d.dir_max, 0, 2 * sizeof(unsigned long long), s);  // the bits of +0.0
  const dim3 grid((a.width + kCompareTileX - 1) / kCompareTileX, (a.height + kCompareTileY - 1) / kCompareTileY);
  if (d.angles)
    compare_models_kernel<true><<<grid, dim3(kCompareTileX, kCompareTileY), 0, s>>>(a, ga, b, gb, d.mag, d.dir_err,
                                                                                 d.rep_err, d.dir_max, d.angles);
  else
    compare_models_kernel<false><<<grid, dim3(kCompareTileX, kCompareTileY), 0, s>>>(a, ga, b, gb, d.mag, d.dir_err,
                                                                                  d.rep_err, d.dir_max, nullptr);
  launch_report_statistics(1, d.range, d.mag, d.partial, d.select_hist, d.stats, s);
  if (d.magnitudes) {
    const int64_t n = static_cast<int64_t>(a.width) * a.height;
    fitting_images_kernel<<<static_cast<unsigned>((n + kFittingImageThreads - 1) / kFittingImageThreads),
                            kFittingImageThreads, 0, s>>>(n, d.dir_err, d.mag, d.dir_max, d.stats, d.magnitudes,
                                                          d.directions, d.rep_magnitudes, d.reprojections);
  }
}

// ------------------------------------------------------------------------------------------
// localization accuracy test (tools/localization_accuracy_test.cc:47-131): the draws of the 15 points of every
// trial, then one pose fit per trial (opengv's absolute_pose::optimize_nonlinear cost; the iteration and the random
// stream are specified in include/b200ba.h)
// ------------------------------------------------------------------------------------------
// (float)(h >> 40) * 2^-24f * extent: the first product is exact, the second rounds once
__device__ __forceinline__ float loc_coordinate(uint64_t h, float extent) {
  return __fmul_rn(static_cast<float>(h >> 40) * 0x1p-24f, extent);
}
// Eigen's normalized() without fused operations, v / sqrt((x^2 + y^2) + z^2), and v * s: the sample kernel and
// the pose kernel build p, f and u with these, so that u = f bit for bit where both models agree
__device__ __forceinline__ double loc_norm(d3 v) {
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(v.x, v.x), __dmul_rn(v.y, v.y)), __dmul_rn(v.z, v.z)));
}
__device__ __forceinline__ d3 loc_unit(d3 v, double n) { return mk3(__ddiv_rn(v.x, n), __ddiv_rn(v.y, n), __ddiv_rn(v.z, n)); }
__device__ __forceinline__ d3 loc_scaled(d3 v, double s) { return mk3(__dmul_rn(v.x, s), __dmul_rn(v.y, s), __dmul_rn(v.z, s)); }

// One thread per (trial, point): the draws until both models un-project the pixel (CentralGenericModel::Unproject
// succeeds exactly inside the calibrated area, central_generic.h:97-105), then p = s n and f.
constexpr int kLocSampleThreads = 128;
__global__ void __launch_bounds__(kLocSampleThreads)
    localization_sample_kernel(CamDev gt, const double* __restrict__ ggt, CamDev cm, const double* __restrict__ gcm,
                               int64_t trials, uint64_t seed_hash, double* __restrict__ p, double* __restrict__ f,
                               float* __restrict__ samples, unsigned long long* __restrict__ counts,
                               int* __restrict__ capped) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(kLocSampleThreads) + threadIdx.x;
  unsigned long long redraws = 0;
  if (i < trials * kLocPoints) {
    const uint64_t trial = static_cast<uint64_t>(i / kLocPoints), point = static_cast<uint64_t>(i % kLocPoints);
    const uint64_t key = (trial << 20) | (point << 16);
    const float w = static_cast<float>(gt.width), h = static_cast<float>(gt.height);
    int a = 0;
    float x = 0, y = 0;
    for (; a < kLocMaxDraws; ++a) {
      const uint64_t k = seed_hash ^ (key | (static_cast<uint64_t>(a) << 4));
      x = loc_coordinate(loc_splitmix64(k), w);
      y = loc_coordinate(loc_splitmix64(k ^ 1), h);
      if (in_area(gt, x, y) && in_area(cm, x, y)) break;
    }
    redraws = static_cast<unsigned long long>(a);
    const double nan_v = nan("");
    d3 pv = mk3(nan_v, nan_v, nan_v), fv = pv;
    float s = nan_v;
    if (a == kLocMaxDraws) {
      *capped = 1;
    } else {
      const uint64_t k = seed_hash ^ (key | (static_cast<uint64_t>(a) << 4) | 2);
      // kMinDistance + ((rand() % 10000) / 10000.f) * (kMaxDistance - kMinDistance) (:99), in float
      s = __fadd_rn(1.5f, __fmul_rn(__fdiv_rn(static_cast<float>(loc_splitmix64(k) % 10000), 10000.f), 1.0f));
      CentralEval e;
      central_eval(gt, ggt, x, y, e);
      const d3 n = loc_unit(e.u, loc_norm(e.u));  // gt_direction.normalize() (:96)
      central_eval(cm, gcm, x, y, e);
      const d3 m = loc_unit(e.u, loc_norm(e.u));  // compared_direction.normalized() (:103)
      pv = loc_scaled(n, static_cast<double>(s));
      const d3 sm = loc_scaled(m, static_cast<double>(s));
      fv = loc_unit(sm, loc_norm(sm));
    }
    p[3 * i] = pv.x;
    p[3 * i + 1] = pv.y;
    p[3 * i + 2] = pv.z;
    f[3 * i] = fv.x;
    f[3 * i + 1] = fv.y;
    f[3 * i + 2] = fv.z;
    if (samples) {
      samples[3 * i] = x;
      samples[3 * i + 1] = y;
      samples[3 * i + 2] = s;
    }
  }
  for (int o = 16; o > 0; o >>= 1) redraws += __shfl_xor_sync(0xffffffffu, redraws, o);
  if ((threadIdx.x & 31) == 0 && redraws) atomicAdd(counts, redraws);
}

// Residual of one point at x = (t, c): v = p - t, q = R(c)' v = ((1 - c'c) v + 2 c (c'v) - 2 c x v) / (1 + c'c),
// u = normalize(q), e = u - f. With J = 1: also dq/dx (3 x 6) through A = [-R(c)' | dq/dc] and
// du/dx = (A - u (u'A)) / |q|, dq/dc = (-2 v c' + 2 (c'v) I + 2 c v' + 2 [v]x - 2 q c') / (1 + c'c).
// e is computed with explicitly rounded operations in the oracle's order: the cost of the system (J = 1) and the
// trial cost (J = 0) at the same x are then the same number, as the LM's acceptance test assumes (with contractions
// chosen per call site, a trial could win by rounding alone and the fit would run to its iteration limit).
__device__ __forceinline__ double loc_dot(d3 a, d3 b) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a.x, b.x), __dmul_rn(a.y, b.y)), __dmul_rn(a.z, b.z));
}
__device__ __forceinline__ double loc_q(double one_m, double va, double cv2, double ca, double cxva, double inv_s) {
  return __dmul_rn(inv_s, __dsub_rn(__dadd_rn(__dmul_rn(one_m, va), __dmul_rn(cv2, ca)), __dmul_rn(2.0, cxva)));
}
template <bool J>
__device__ __forceinline__ void loc_residual(const double (&x)[6], d3 p, d3 f, d3& e, double (&du)[3][6]) {
  const d3 v = mk3(__dsub_rn(p.x, x[0]), __dsub_rn(p.y, x[1]), __dsub_rn(p.z, x[2]));
  const d3 c = mk3(x[3], x[4], x[5]);
  const double cc = loc_dot(c, c), cv = loc_dot(c, v), inv_s = __ddiv_rn(1.0, __dadd_rn(1.0, cc));
  const d3 cxv = mk3(__dsub_rn(__dmul_rn(c.y, v.z), __dmul_rn(c.z, v.y)), __dsub_rn(__dmul_rn(c.z, v.x), __dmul_rn(c.x, v.z)),
                     __dsub_rn(__dmul_rn(c.x, v.y), __dmul_rn(c.y, v.x)));
  const double one_m = __dsub_rn(1.0, cc), cv2 = 2.0 * cv;
  const d3 q = mk3(loc_q(one_m, v.x, cv2, c.x, cxv.x, inv_s), loc_q(one_m, v.y, cv2, c.y, cxv.y, inv_s),
                   loc_q(one_m, v.z, cv2, c.z, cxv.z, inv_s));
  const double nq = loc_norm(q);
  const d3 u = loc_unit(q, nq);
  e = mk3(__dsub_rn(u.x, f.x), __dsub_rn(u.y, f.y), __dsub_rn(u.z, f.z));
  if (!J) return;
  const double cs[3] = {c.x, c.y, c.z}, vs[3] = {v.x, v.y, v.z}, qs[3] = {q.x, q.y, q.z};
  const double inv_n = 1.0 / nq;
#pragma unroll
  for (int b = 0; b < 3; ++b) {
    // column b of -R' = -((1 - c'c) I + 2 c c' - 2 [c]x) / s and of dq/dc
    d3 rt = mk3(2.0 * c.x * cs[b], 2.0 * c.y * cs[b], 2.0 * c.z * cs[b]);
    d3 m = mk3(2.0 * (c.x * vs[b] - v.x * cs[b] - qs[0] * cs[b]), 2.0 * (c.y * vs[b] - v.y * cs[b] - qs[1] * cs[b]),
               2.0 * (c.z * vs[b] - v.z * cs[b] - qs[2] * cs[b]));
    if (b == 0) {
      rt.x += one_m;
      rt.y -= 2.0 * c.z;
      rt.z += 2.0 * c.y;
      m.x += 2.0 * cv;
      m.y += 2.0 * v.z;
      m.z -= 2.0 * v.y;
    } else if (b == 1) {
      rt.x += 2.0 * c.z;
      rt.y += one_m;
      rt.z -= 2.0 * c.x;
      m.x -= 2.0 * v.z;
      m.y += 2.0 * cv;
      m.z += 2.0 * v.x;
    } else {
      rt.x -= 2.0 * c.y;
      rt.y += 2.0 * c.x;
      rt.z += one_m;
      m.x += 2.0 * v.y;
      m.y -= 2.0 * v.x;
      m.z += 2.0 * cv;
    }
    const d3 at = (-inv_s) * rt, ac = inv_s * m;
    const d3 jt = inv_n * (at - dot3(u, at) * u), jc = inv_n * (ac - dot3(u, ac) * u);
    du[0][b] = jt.x;
    du[1][b] = jt.y;
    du[2][b] = jt.z;
    du[0][3 + b] = jc.x;
    du[1][3 + b] = jc.y;
    du[2][3 + b] = jc.z;
  }
}
// r = 1/2 |e|^2 = 1 - f'u for unit vectors; the point's term of F is r^2
__device__ __forceinline__ double loc_cost_term(d3 e) {
  const double r = 0.5 * __dadd_rn(__dadd_rn(__dmul_rn(e.x, e.x), __dmul_rn(e.y, e.y)), __dmul_rn(e.z, e.z));
  return r * r;
}
// sys = {F, grad F (6), H (21, lower triangle row by row)} of one point
constexpr int kLocSums = 28;
__device__ __forceinline__ int loc_h(int i, int j) { return 7 + i * (i + 1) / 2 + j; }
__device__ __forceinline__ void loc_point_system(const double (&x)[6], d3 p, d3 f, double (&sys)[kLocSums]) {
  d3 e;
  double du[3][6];
  loc_residual<true>(x, p, f, e, du);
  sys[0] = loc_cost_term(e);
  const double w = dot3(e, e);
  double a[6];
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    a[j] = du[0][j] * e.x + du[1][j] * e.y + du[2][j] * e.z;  // (J'e)_j
    sys[1 + j] = w * a[j];
  }
#pragma unroll
  for (int i = 0; i < 6; ++i)
#pragma unroll
    for (int j = 0; j <= i; ++j)
      sys[loc_h(i, j)] = w * (du[0][i] * du[0][j] + du[1][i] * du[1][j] + du[2][i] * du[2][j]) + 2.0 * a[i] * a[j];
}
// the same sum in every lane of the 16: a fixed xor butterfly (a + b == b + a, so all lanes agree bit for bit)
template <int N>
__device__ __forceinline__ void loc_reduce(double (&v)[N], unsigned mask) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1)
#pragma unroll
    for (int k = 0; k < N; ++k) v[k] += __shfl_xor_sync(mask, v[k], o);
}
// (H + lambda I) d = -g by Cholesky; false where H + lambda I is not positive definite
__device__ __forceinline__ bool loc_solve(const double (&sys)[kLocSums], double lambda, double (&d)[6]) {
  double L[21];
  bool ok = true;
#pragma unroll
  for (int i = 0; i < 6; ++i)
#pragma unroll
    for (int j = 0; j <= i; ++j) {
      double a = sys[loc_h(i, j)] + (i == j ? lambda : 0.0);
#pragma unroll
      for (int k = 0; k < j; ++k) a -= L[i * (i + 1) / 2 + k] * L[j * (j + 1) / 2 + k];
      if (i == j) {
        ok = ok && a > 0;
        L[i * (i + 1) / 2 + i] = sqrt(a);
      } else {
        L[i * (i + 1) / 2 + j] = a / L[j * (j + 1) / 2 + j];
      }
    }
  double y[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    double a = -sys[1 + i];
#pragma unroll
    for (int k = 0; k < i; ++k) a -= L[i * (i + 1) / 2 + k] * y[k];
    y[i] = a / L[i * (i + 1) / 2 + i];
  }
#pragma unroll
  for (int i = 5; i >= 0; --i) {
    double a = y[i];
#pragma unroll
    for (int k = i + 1; k < 6; ++k) a -= L[k * (k + 1) / 2 + i] * d[k];
    d[i] = a / L[i * (i + 1) / 2 + i];
  }
  return ok;
}

// 16 lanes per trial, two trials per warp; lane i < 15 owns point i, lane 15 adds zeros. Every lane holds the whole
// LM state (x, lambda, F, the reduced system) and factors H + lambda I itself, so the 16 lanes take the same branches.
constexpr int kLocPoseThreads = 128;
constexpr int kLocMaxIterations = 100;
__global__ void __launch_bounds__(kLocPoseThreads)
    localization_pose_kernel(int64_t trials, const double* __restrict__ p, const double* __restrict__ f,
                             double* __restrict__ poses, double* __restrict__ mag,
                             unsigned long long* __restrict__ counts) {
  const int64_t trial = (blockIdx.x * static_cast<int64_t>(kLocPoseThreads) + threadIdx.x) >> 4;
  const int lane = threadIdx.x & 15;
  const unsigned mask = 0xffffu << (threadIdx.x & 16);
  __shared__ unsigned long long block_iterations;
  __shared__ unsigned int block_max;
  if (threadIdx.x == 0) {
    block_iterations = 0;
    block_max = 0;
  }
  __syncthreads();
  if (trial < trials) {
    const bool own = lane < kLocPoints;
    d3 pi = mk3(0, 0, 0), fi = mk3(0, 0, 0);
    if (own) {
      const int64_t o = 3 * (trial * kLocPoints + lane);
      pi = ld3(p + o);
      fi = ld3(f + o);
    }
    double x[6] = {0, 0, 0, 0, 0, 0};
    double lambda = 0;
    int iterations = 0;
    for (int it = 0; it < kLocMaxIterations; ++it) {
      double sys[kLocSums];
      loc_point_system(x, pi, fi, sys);
      if (!own)
#pragma unroll
        for (int k = 0; k < kLocSums; ++k) sys[k] = 0;
      loc_reduce(sys, mask);
      const double cost = sys[0];
      if (cost == 0) break;
      if (it == 0) {
        double trace = 0;
#pragma unroll
        for (int i = 0; i < 6; ++i) trace += sys[loc_h(i, i)];
        lambda = static_cast<double>(0.001f) * trace / 6;
      }
      bool applied = false;
      double test_cost = cost;
      for (int attempt = 0; attempt < 10; ++attempt) {
        double d[6];
        if (!loc_solve(sys, lambda, d)) {
          lambda = 2.0 * lambda;
          continue;
        }
        double xt[6];
#pragma unroll
        for (int k = 0; k < 6; ++k) xt[k] = x[k] + d[k];
        d3 e;
        double unused[3][6];
        loc_residual<false>(xt, pi, fi, e, unused);
        double tc[1] = {own ? loc_cost_term(e) : 0.0};
        loc_reduce(tc, mask);
        if (tc[0] < cost) {
#pragma unroll
          for (int k = 0; k < 6; ++k) x[k] = xt[k];
          lambda = 0.5 * lambda;
          applied = true;
          ++iterations;
          test_cost = tc[0];
          break;
        }
        lambda = 2.0 * lambda;
      }
      if (!applied || test_cost == 0) break;
    }
    if (lane == 0) {
      if (poses)
#pragma unroll
        for (int k = 0; k < 6; ++k) poses[6 * trial + k] = x[k];
      // (float)translation.norm() (:115-116)
      const float err = static_cast<float>(loc_norm(mk3(x[0], x[1], x[2])));
      mag[trial] = static_cast<double>(err);
      atomicAdd(&block_iterations, static_cast<unsigned long long>(iterations));
      atomicMax(&block_max, static_cast<unsigned int>(iterations));
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (block_iterations) atomicAdd(counts + 1, block_iterations);
    atomicMax(counts + 2, static_cast<unsigned long long>(block_max));
  }
}

void launch_localization_sample(const CamDev& gt, const double* ggt, const CamDev& cmp, const double* gcmp,
                                int64_t trials, uint64_t seed, const LocalizationDev& d, cudaStream_t s) {
  cudaMemsetAsync(d.counts, 0, 3 * sizeof(unsigned long long), s);
  cudaMemsetAsync(d.capped, 0, sizeof(int), s);
  const int64_t n = trials * kLocPoints;
  const uint64_t seed_hash = loc_splitmix64(seed);
  localization_sample_kernel<<<static_cast<unsigned>((n + kLocSampleThreads - 1) / kLocSampleThreads),
                               kLocSampleThreads, 0, s>>>(gt, ggt, cmp, gcmp, trials, seed_hash, d.p, d.f, d.samples,
                                                          d.counts, d.capped);
}

void launch_localization_pose(int64_t trials, const LocalizationDev& d, cudaStream_t s) {
  constexpr int kTrialsPerBlock = kLocPoseThreads / 16;
  localization_pose_kernel<<<static_cast<unsigned>((trials + kTrialsPerBlock - 1) / kTrialsPerBlock), kLocPoseThreads,
                             0, s>>>(trials, d.p, d.f, d.poses, d.mag, d.counts);
  launch_report_statistics(1, d.range, d.mag, d.partial, d.select_hist, d.stats, s);
}

// ------------------------------------------------------------------------------------------
// reconstruction comparison (b200ba_compare_reconstructions; the sample loop of APP/tools/bundle_adjustment.cc:280-294)
// ------------------------------------------------------------------------------------------
// Unproject(x, y, Line3d*) of a CG / NCG / OpenCV model followed by the tool's direction().normalized(); origins are
// not used. The final normalisation is Eigen's: d / sqrt(|d|^2), |d|^2 without FMA.
__device__ __forceinline__ bool sweep_unproject(const CamDev& c, const double* __restrict__ intr, double x, double y,
                                                d3& d) {
  d3 u;
  if (c.model_type == B200BA_MODEL_CENTRAL_OPENCV) {
    if (!opencv_unproject(intr, x, y, u)) return false;
  } else {
    if (!in_area(c, x, y)) return false;
    if (c.model_type == B200BA_MODEL_CENTRAL_GENERIC) {
      CentralEval e;
      central_eval(c, intr, x, y, e);
      u = e.u;
    } else {
      d3 o;
      noncentral_line(c, intr, intr + 3 * static_cast<int64_t>(c.gw) * c.gh, x, y, o, u);
    }
  }
  const double n = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(u.x, u.x), __dmul_rn(u.y, u.y)), __dmul_rn(u.z, u.z)));
  d = mk3(u.x / n, u.y / n, u.z / n);
  return true;
}
// One thread per sample pixel (x, y) = (step i + 0.5, step j + 0.5) of the nx x ny sample grid, in 16 x 8 tiles. Pixels
// that both models un-project add 1 and d1 d2^T to the block's kSweepSums sums; the block reduces them by a fixed
// shared-memory tree into partial[block][kSweepSums] (the block's linear index), and sweep_stage2 adds the blocks in a
// fixed order. Nothing depends on scheduling, so repeated calls give the same bits.
constexpr int kSweepTileX = 16, kSweepTileY = 8, kSweepThreads = kSweepTileX * kSweepTileY;
__global__ void __launch_bounds__(kSweepThreads)
    reconstruction_sweep_kernel(CamDev c1, const double* __restrict__ intr1, CamDev c2,
                                const double* __restrict__ intr2, int step, int nx, int ny,
                                double* __restrict__ partial) {
  const int i = blockIdx.x * kSweepTileX + threadIdx.x, j = blockIdx.y * kSweepTileY + threadIdx.y;
  double s[kSweepSums];
#pragma unroll
  for (int k = 0; k < kSweepSums; ++k) s[k] = 0;
  if (i < nx && j < ny) {
    const double x = static_cast<double>(i) * step + 0.5, y = static_cast<double>(j) * step + 0.5;
    d3 d1, d2;
    if (sweep_unproject(c1, intr1, x, y, d1) && sweep_unproject(c2, intr2, x, y, d2)) {
      s[0] = 1;
      s[1] = d1.x * d2.x;
      s[2] = d1.x * d2.y;
      s[3] = d1.x * d2.z;
      s[4] = d1.y * d2.x;
      s[5] = d1.y * d2.y;
      s[6] = d1.y * d2.z;
      s[7] = d1.z * d2.x;
      s[8] = d1.z * d2.y;
      s[9] = d1.z * d2.z;
    }
  }
  __shared__ double sh[kSweepSums][kSweepThreads];
  const int t = threadIdx.y * kSweepTileX + threadIdx.x;
#pragma unroll
  for (int k = 0; k < kSweepSums; ++k) sh[k][t] = s[k];
  __syncthreads();
  for (int st = kSweepThreads / 2; st > 0; st >>= 1) {
    if (t < st) {
#pragma unroll
      for (int k = 0; k < kSweepSums; ++k) sh[k][t] += sh[k][t + st];
    }
    __syncthreads();
  }
  if (t < kSweepSums) partial[(static_cast<int64_t>(blockIdx.y) * gridDim.x + blockIdx.x) * kSweepSums + t] = sh[t][0];
}
// sums[k] = sum over the blocks of partial[b][k]: block k of the grid, thread t adds blocks t, t + 256, ... in order,
// then a fixed tree over the 256 threads.
__global__ void __launch_bounds__(kReportThreads)
    sweep_stage2(int64_t nblocks, const double* __restrict__ partial, double* __restrict__ sums) {
  const int k = blockIdx.x;
  double v = 0;
  for (int64_t b = threadIdx.x; b < nblocks; b += kReportThreads) v += partial[b * kSweepSums + k];
  __shared__ double sh[kReportThreads];
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int st = kReportThreads / 2; st > 0; st >>= 1) {
    if (threadIdx.x < st) sh[threadIdx.x] += sh[threadIdx.x + st];
    __syncthreads();
  }
  if (threadIdx.x == 0) sums[k] = sh[0];
}
// The per-pixel directions behind the sums: ok[2 p + k] and dirs[6 p + 3 k ..] of model k + 1 at sample p = j nx + i
// (0 where the model does not un-project the pixel).
__global__ void reconstruction_directions_kernel(CamDev c1, const double* __restrict__ intr1, CamDev c2,
                                                 const double* __restrict__ intr2, int step, int nx, int ny,
                                                 int32_t* __restrict__ ok, double* __restrict__ dirs) {
  const int64_t p = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (p >= static_cast<int64_t>(nx) * ny) return;
  const double x = static_cast<double>(p % nx) * step + 0.5, y = static_cast<double>(p / nx) * step + 0.5;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    d3 d = mk3(0, 0, 0);
    const bool r = sweep_unproject(k == 0 ? c1 : c2, k == 0 ? intr1 : intr2, x, y, d);
    ok[2 * p + k] = r ? 1 : 0;
    dirs[6 * p + 3 * k] = r ? d.x : 0.0;
    dirs[6 * p + 3 * k + 1] = r ? d.y : 0.0;
    dirs[6 * p + 3 * k + 2] = r ? d.z : 0.0;
  }
}
void launch_reconstruction_directions(const CamDev& c1, const double* intr1, const CamDev& c2, const double* intr2,
                                      int step, int nx, int ny, int32_t* ok, double* dirs, cudaStream_t s) {
  const int64_t n = static_cast<int64_t>(nx) * ny;
  reconstruction_directions_kernel<<<static_cast<unsigned>((n + 127) / 128), 128, 0, s>>>(c1, intr1, c2, intr2, step,
                                                                                          nx, ny, ok, dirs);
}
int64_t sweep_partial_blocks(int nx, int ny) {
  return static_cast<int64_t>((nx + kSweepTileX - 1) / kSweepTileX) * ((ny + kSweepTileY - 1) / kSweepTileY);
}
void launch_reconstruction_sweep(const CamDev& c1, const double* intr1, const CamDev& c2, const double* intr2,
                                 int step, int nx, int ny, double* partial, double* sums, cudaStream_t s) {
  const dim3 grid((nx + kSweepTileX - 1) / kSweepTileX, (ny + kSweepTileY - 1) / kSweepTileY);
  reconstruction_sweep_kernel<<<grid, dim3(kSweepTileX, kSweepTileY), 0, s>>>(c1, intr1, c2, intr2, step, nx, ny,
                                                                              partial);
  sweep_stage2<<<kSweepSums, kReportThreads, 0, s>>>(sweep_partial_blocks(nx, ny), partial, sums);
}

// ------------------------------------------------------------------------------------------
// centre-point analysis of a non-central camera (CreateCalibrationReportForCamera, APP/calibration_report.cc:839-982)
// ------------------------------------------------------------------------------------------
// The lines are evaluated once and stored (48 B per line: 55 MB for 1200 x 950, 576 MB for 4000 x 3000); every LM
// pass then streams them instead of re-evaluating two B-spline surfaces per line. DESIGN.md section 4 has the
// measured times of both: about equal, since a streaming pass is bound by the tangent frame's FP64 arithmetic. Each pixel of the calibrated rectangle lies in the calibrated area, so every Unproject
// of :847-856 succeeds and there is one line per rectangle pixel.
constexpr int kLineTileX = 16, kLineTileY = 8;
__global__ void __launch_bounds__(kLineTileX * kLineTileY)
    line_pass_kernel(CamDev c, const double* __restrict__ intr, double* __restrict__ lines) {
  const int rw = c.max_x - c.min_x + 1, rh = c.max_y - c.min_y + 1;
  const int lx = blockIdx.x * kLineTileX + threadIdx.x, ly = blockIdx.y * kLineTileY + threadIdx.y;
  if (lx >= rw || ly >= rh) return;
  // the reference passes x + 0.5f (a float) where Unproject takes a double
  const double px = static_cast<double>((c.min_x + lx) + 0.5f), py = static_cast<double>((c.min_y + ly) + 0.5f);
  d3 o, d;
  noncentral_line(c, intr, intr + 3 * static_cast<int64_t>(c.gw) * c.gh, px, py, o, d);
  const int64_t n = static_cast<int64_t>(rw) * rh, p = static_cast<int64_t>(ly) * rw + lx;
  lines[p] = o.x;
  lines[n + p] = o.y;
  lines[2 * n + p] = o.z;
  lines[3 * n + p] = d.x;
  lines[4 * n + p] = d.y;
  lines[5 * n + p] = d.z;
}
__device__ __forceinline__ void load_line(const double* __restrict__ lines, int64_t n, int64_t p, d3& o, d3& d) {
  o = mk3(lines[p], lines[n + p], lines[2 * n + p]);
  d = mk3(lines[3 * n + p], lines[4 * n + p], lines[5 * n + p]);
}

// One pass of CenterPointCostFunction::Compute (:56-80) at the centre c: sum over the lines of the per-line cost
// 1/2 (r1^2 + r2^2) (mode >= 0), of b = t1 r1 + t2 r2 (mode >= 1) and of H = t1 t1^T + t2 t2^T (mode 2), in the
// fixed two-stage order of report_reduce_stage1/2. The cost is written with non-fused operations, so that every mode
// computes the same bits for it: the trial cost of an accepted step IS the next iteration's cost, as in the reference.
template <int kMode>
__global__ void __launch_bounds__(kReportThreads)
    line_system_stage1(int64_t n, const double* __restrict__ lines, double cx, double cy, double cz,
                       double* __restrict__ partial) {
  double s[kLineSums];
#pragma unroll
  for (int k = 0; k < kLineSums; ++k) s[k] = 0;
  for (int64_t p = blockIdx.x * static_cast<int64_t>(kReportThreads) + threadIdx.x; p < n;
       p += static_cast<int64_t>(kReportBlocks) * kReportThreads) {
    d3 o, d, t1, t2;
    load_line(lines, n, p, o, d);
    compute_tangents(d, t1, t2);
    const d3 q = mk3(__dsub_rn(cx, o.x), __dsub_rn(cy, o.y), __dsub_rn(cz, o.z));
    const double r1 = dot3(t1, q), r2 = dot3(t2, q);
    s[0] += __dmul_rn(0.5, __dadd_rn(__dmul_rn(r1, r1), __dmul_rn(r2, r2)));
    if (kMode >= 1) {
      s[1] += t1.x * r1 + t2.x * r2;
      s[2] += t1.y * r1 + t2.y * r2;
      s[3] += t1.z * r1 + t2.z * r2;
    }
    if (kMode >= 2) {
      s[4] += t1.x * t1.x + t2.x * t2.x;
      s[5] += t1.x * t1.y + t2.x * t2.y;
      s[6] += t1.x * t1.z + t2.x * t2.z;
      s[7] += t1.y * t1.y + t2.y * t2.y;
      s[8] += t1.y * t1.z + t2.y * t2.z;
      s[9] += t1.z * t1.z + t2.z * t2.z;
    }
  }
  constexpr int kUsed = kMode == 0 ? 1 : (kMode == 1 ? 4 : kLineSums);
  __shared__ double sh[kUsed][kReportThreads];
#pragma unroll
  for (int k = 0; k < kUsed; ++k) sh[k][threadIdx.x] = s[k];
  __syncthreads();
  for (int st = kReportThreads / 2; st > 0; st >>= 1) {
    if (threadIdx.x < st) {
#pragma unroll
      for (int k = 0; k < kUsed; ++k) sh[k][threadIdx.x] += sh[k][threadIdx.x + st];
    }
    __syncthreads();
  }
  if (threadIdx.x < kLineSums) partial[blockIdx.x * kLineSums + threadIdx.x] = threadIdx.x < kUsed ? sh[threadIdx.x][0] : 0.0;
}
__global__ void line_system_stage2(const double* __restrict__ partial, double* __restrict__ sums) {
  const int k = threadIdx.x;
  if (k >= kLineSums) return;
  double v = 0;
  for (int b = 0; b < kReportBlocks; ++b) v += partial[b * kLineSums + k];
  sums[k] = v;
}
int line_system_partial_size() { return kReportBlocks * kLineSums; }
void launch_line_pass(const CamDev& c, const double* intr, const LineOffsetsDev& d, cudaStream_t s) {
  const int rw = c.max_x - c.min_x + 1, rh = c.max_y - c.min_y + 1;
  const dim3 grid((rw + kLineTileX - 1) / kLineTileX, (rh + kLineTileY - 1) / kLineTileY);
  line_pass_kernel<<<grid, dim3(kLineTileX, kLineTileY), 0, s>>>(c, intr, d.lines);
}
void launch_line_system(int mode, int64_t n, const double c[3], const LineOffsetsDev& d, cudaStream_t s) {
  if (mode == 0) line_system_stage1<0><<<kReportBlocks, kReportThreads, 0, s>>>(n, d.lines, c[0], c[1], c[2], d.partial);
  else if (mode == 1) line_system_stage1<1><<<kReportBlocks, kReportThreads, 0, s>>>(n, d.lines, c[0], c[1], c[2], d.partial);
  else line_system_stage1<2><<<kReportBlocks, kReportThreads, 0, s>>>(n, d.lines, c[0], c[1], c[2], d.partial);
  line_system_stage2<<<1, 32, 0, s>>>(d.partial, d.sums);
}

// :884-888 with no fused operation: parameter = d . (c - o), closest = o + parameter d, offset = closest - c
__device__ __forceinline__ d3 line_offset(d3 o, d3 d, d3 c, d3& closest) {
  const d3 q = mk3(__dsub_rn(c.x, o.x), __dsub_rn(c.y, o.y), __dsub_rn(c.z, o.z));
  const double t = __dadd_rn(__dadd_rn(__dmul_rn(d.x, q.x), __dmul_rn(d.y, q.y)), __dmul_rn(d.z, q.z));
  closest = mk3(__dadd_rn(o.x, __dmul_rn(t, d.x)), __dadd_rn(o.y, __dmul_rn(t, d.y)), __dadd_rn(o.z, __dmul_rn(t, d.z)));
  return mk3(__dsub_rn(closest.x, c.x), __dsub_rn(closest.y, c.y), __dsub_rn(closest.z, c.z));
}
// Vector3d::norm() in Eigen's order, no fused multiply-add
__device__ __forceinline__ double line_norm(d3 v) {
  return sqrt(__dadd_rn(__dadd_rn(__dmul_rn(v.x, v.x), __dmul_rn(v.y, v.y)), __dmul_rn(v.z, v.z)));
}

// :880-902: the line distance of every line into mag (statistics by launch_report_statistics) and the extent, an exact
// block maximum followed by one atomicMax per block on the bit pattern (non-negative doubles order like their uint64
// patterns; fmax skips NaN as the reference's std::max(extent, NaN) keeps extent)
__global__ void __launch_bounds__(kReportThreads)
    line_distances_kernel(int64_t n, const double* __restrict__ lines, double cx, double cy, double cz,
                          double* __restrict__ mag, unsigned long long* __restrict__ extent) {
  const int64_t p = blockIdx.x * static_cast<int64_t>(kReportThreads) + threadIdx.x;
  double ext = 0;
  if (p < n) {
    d3 o, d, closest;
    load_line(lines, n, p, o, d);
    const d3 off = line_offset(o, d, mk3(cx, cy, cz), closest);
    mag[p] = line_norm(off);
    ext = fmax(fabs(off.x), fmax(fabs(off.y), fabs(off.z)));
  }
  for (int o = 16; o > 0; o >>= 1) ext = fmax(ext, __shfl_xor_sync(0xffffffffu, ext, o));
  __shared__ double sh[kReportThreads / 32];
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = ext;
  __syncthreads();
  if (threadIdx.x == 0) {
    double v = 0;
    for (int w = 0; w < kReportThreads / 32; ++w) v = fmax(v, sh[w]);
    if (v > 0) atomicMax(extent, static_cast<unsigned long long>(__double_as_longlong(v)));
  }
}

// :870-871, :913-926 per image pixel: the offset (NaN outside the calibrated rectangle) and the colour
// 127 + 127 * offset_k / extent in double, converted as x86-64 converts double to u8 (truncation to int32, low byte;
// with extent 0 every channel is NaN and gives 0); black where the offset has a NaN
__global__ void __launch_bounds__(kLineTileX * kLineTileY)
    line_offsets_image_kernel(CamDev c, const double* __restrict__ lines, double cx, double cy, double cz,
                              const unsigned long long* __restrict__ extent, double* __restrict__ offsets,
                              uint8_t* __restrict__ img) {
  const int x = blockIdx.x * kLineTileX + threadIdx.x, y = blockIdx.y * kLineTileY + threadIdx.y;
  if (x >= c.width || y >= c.height) return;
  const double nan_v = nan("");
  d3 off = mk3(nan_v, nan_v, nan_v);
  if (x >= c.min_x && x <= c.max_x && y >= c.min_y && y <= c.max_y) {
    const int rw = c.max_x - c.min_x + 1;
    const int64_t n = static_cast<int64_t>(rw) * (c.max_y - c.min_y + 1);
    d3 o, d, closest;
    load_line(lines, n, static_cast<int64_t>(y - c.min_y) * rw + (x - c.min_x), o, d);
    off = line_offset(o, d, mk3(cx, cy, cz), closest);
  }
  const int64_t q = 3 * (static_cast<int64_t>(y) * c.width + x);
  if (offsets) {
    offsets[q] = off.x;
    offsets[q + 1] = off.y;
    offsets[q + 2] = off.z;
  }
  if (img) {
    uint8_t out[3] = {0, 0, 0};
    if (!isnan(off.x) && !isnan(off.y) && !isnan(off.z)) {
      const double e = __longlong_as_double(static_cast<long long>(*extent));
      out[0] = static_cast<uint8_t>(report_trunc(__dadd_rn(127.0, __ddiv_rn(__dmul_rn(127.0, off.x), e))));
      out[1] = static_cast<uint8_t>(report_trunc(__dadd_rn(127.0, __ddiv_rn(__dmul_rn(127.0, off.y), e))));
      out[2] = static_cast<uint8_t>(report_trunc(__dadd_rn(127.0, __ddiv_rn(__dmul_rn(127.0, off.z), e))));
    }
    img[q] = out[0];
    img[q + 1] = out[1];
    img[q + 2] = out[2];
  }
}

// :945-973: line i = iy * nx + ix of the .obj models is the pixel (min_x + ix * step, min_y + iy * step);
// obj[12 i ..]: point_a, point_b, closest point, origin
__global__ void line_obj_kernel(CamDev c, const double* __restrict__ lines, double cx, double cy, double cz, int step,
                                int nx, int64_t n_obj, double* __restrict__ obj) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n_obj) return;
  const int rw = c.max_x - c.min_x + 1;
  const int64_t n = static_cast<int64_t>(rw) * (c.max_y - c.min_y + 1);
  const int64_t p = (i / nx) * step * static_cast<int64_t>(rw) + (i % nx) * step;
  d3 o, d, closest;
  load_line(lines, n, p, o, d);
  const d3 off = line_offset(o, d, mk3(cx, cy, cz), closest);
  const double half = fmax(10.0, __dmul_rn(10.0, line_norm(off)));  // std::max<double>(10, 10 * norm)
  const d3 hd = mk3(__dmul_rn(half, d.x), __dmul_rn(half, d.y), __dmul_rn(half, d.z));
  double* out = obj + 12 * i;
  out[0] = __dadd_rn(closest.x, hd.x);
  out[1] = __dadd_rn(closest.y, hd.y);
  out[2] = __dadd_rn(closest.z, hd.z);
  out[3] = __dsub_rn(closest.x, hd.x);
  out[4] = __dsub_rn(closest.y, hd.y);
  out[5] = __dsub_rn(closest.z, hd.z);
  out[6] = closest.x;
  out[7] = closest.y;
  out[8] = closest.z;
  out[9] = o.x;
  out[10] = o.y;
  out[11] = o.z;
}

void launch_line_outputs(const CamDev& c, const double center[3], const LineOffsetsDev& d, int obj_step, int nx,
                         int64_t n_obj, cudaStream_t s) {
  const int64_t n = static_cast<int64_t>(c.max_x - c.min_x + 1) * (c.max_y - c.min_y + 1);
  cudaMemsetAsync(d.extent, 0, sizeof(unsigned long long), s);  // the bits of +0.0
  line_distances_kernel<<<static_cast<unsigned>((n + kReportThreads - 1) / kReportThreads), kReportThreads, 0, s>>>(
      n, d.lines, center[0], center[1], center[2], d.mag, d.extent);
  launch_report_statistics(1, d.range, d.mag, d.stat_partial, d.select_hist, d.stats, s);
  if (d.offsets || d.image) {
    const dim3 grid((c.width + kLineTileX - 1) / kLineTileX, (c.height + kLineTileY - 1) / kLineTileY);
    line_offsets_image_kernel<<<grid, dim3(kLineTileX, kLineTileY), 0, s>>>(c, d.lines, center[0], center[1], center[2],
                                                                            d.extent, d.offsets, d.image);
  }
  if (d.obj && n_obj > 0)
    line_obj_kernel<<<static_cast<unsigned>((n_obj + 127) / 128), 128, 0, s>>>(c, d.lines, center[0], center[1], center[2],
                                                                                obj_step, nx, n_obj, d.obj);
}

// ------------------------------------------------------------------------------------------
// report images (CreateCalibrationReportForCamera, APP/calibration_report.cc:713-838)
// ------------------------------------------------------------------------------------------
// Error maps (:354-603): every feature site owns its Voronoi cell; a pixel's colour is the sum over the
// cells of area(pixel n cell) * colour(cell), + 0.5, clamped to [0, 255.99] and truncated. The reference
// triangulates each cell with Boost.Polygon and rasterises the triangle fan on the CPU; here every pixel
// gathers the cells that can reach it and computes the exact partition:
//   1. counting sort of the sites into a uniform bucket grid (buckets listed in index order);
//   2. per 8 x 8 tile: the exact nearest site s0 of the tile centre (block-wide ring search), so that every
//      point of the tile is within U = |c - s0| + half diagonal of some site: only the sites within U of
//      the tile rectangle can own part of it, and they are read row of buckets by row of buckets (one
//      contiguous range of idx per row), the same sequence for every thread of the block (broadcast loads);
//   3. per pixel: the nearest site of its centre and of its four corners (integer squared distances in
//      quarter pixels, first site wins a tie). Cells are convex, so if the four corners share their nearest
//      site the pixel lies in that cell (the fast path). Otherwise the pixel's candidates are the sites whose
//      distance to the pixel square is at most the centre's nearest distance + sqrt(2)/2 px, and the square
//      is clipped, in double, by the bisector half-planes of every candidate pair; area * colour is summed
//      in the fixed candidate order.
// No atomics touch the images, so two calls give identical bytes.
constexpr int kVorTile = 8;
constexpr int kVorThreads = kVorTile * kVorTile;
constexpr int kVorMaxCand = 24;  // candidates held per slow pixel; beyond that the pixel re-reads the buckets
constexpr int kVorMaxPoly = 32;  // vertices of a clipped square (4 + one per cutting half-plane)

VoronoiGrid voronoi_grid_geometry(int64_t lo_x, int64_t lo_y, int64_t hi_x, int64_t hi_y) {
  VoronoiGrid g{};
  int64_t bs = 32;  // 8 pixels
  while (((hi_x - lo_x) / bs + 1) * ((hi_y - lo_y) / bs + 1) > kVoronoiMaxBuckets) bs *= 2;
  g.x0 = static_cast<int>(lo_x);
  g.y0 = static_cast<int>(lo_y);
  g.bs = static_cast<int>(bs);
  g.nx = static_cast<int>((hi_x - lo_x) / bs + 1);
  g.ny = static_cast<int>((hi_y - lo_y) / bs + 1);
  return g;
}

__device__ __forceinline__ int vor_bucket(const VoronoiGrid& g, int2 p) {
  return ((p.y - g.y0) / g.bs) * g.nx + (p.x - g.x0) / g.bs;
}
__global__ void vor_count_kernel(int64_t n, const int2* __restrict__ sites, VoronoiGrid g) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n || sites[i].x == kVoronoiNoSite) return;
  atomicAdd(&g.count[vor_bucket(g, sites[i])], 1);
}
__global__ void vor_scatter_kernel(int64_t n, const int2* __restrict__ sites, VoronoiGrid g) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n || sites[i].x == kVoronoiNoSite) return;
  const int b = vor_bucket(g, sites[i]);
  g.idx[g.off[b] + atomicAdd(&g.count[b], 1)] = static_cast<int>(i);
}
// the scatter's order inside a bucket depends on the atomics: sort every bucket by site index
__global__ void vor_sort_buckets_kernel(VoronoiGrid g) {
  const int64_t b = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (b >= static_cast<int64_t>(g.nx) * g.ny) return;
  int* v = g.idx + g.off[b];
  const int m = g.off[b + 1] - g.off[b];
  for (int i = 1; i < m; ++i) {
    const int x = v[i];
    int j = i - 1;
    while (j >= 0 && v[j] > x) {
      v[j + 1] = v[j];
      --j;
    }
    v[j + 1] = x;
  }
}

// exclusive scan of the bucket counts (1024 threads, 4 consecutive elements each per block)
constexpr int kScanThreads = kVoronoiScanChunk / 4;
__device__ __forceinline__ int vor_block_scan(int v, int& total) {
  __shared__ int warp_sum[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sum[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int s = warp_sum[lane];
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    warp_sum[lane] = s;
  }
  __syncthreads();
  const int excl = x - v + (warp > 0 ? warp_sum[warp - 1] : 0);
  total = warp_sum[31];
  __syncthreads();
  return excl;
}
__device__ __forceinline__ void vor_scan_chunk(int64_t n, const int* in, int* out, int base_add, int& total) {
  int v[4], s = 0;
  const int64_t base = static_cast<int64_t>(threadIdx.x) * 4;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    v[k] = base + k < n ? in[base + k] : 0;
    s += v[k];
  }
  int run = vor_block_scan(s, total) + base_add;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (base + k < n) out[base + k] = run;
    run += v[k];
  }
}
__global__ void __launch_bounds__(kScanThreads) vor_scan_blocks_kernel(int64_t n, const int* __restrict__ in, int* out,
                                                                       int* __restrict__ sums) {
  const int64_t b0 = static_cast<int64_t>(blockIdx.x) * kVoronoiScanChunk;
  int total;
  const int64_t m = n - b0 < kVoronoiScanChunk ? n - b0 : kVoronoiScanChunk;
  vor_scan_chunk(m, in + b0, out + b0, 0, total);
  if (threadIdx.x == 0) sums[blockIdx.x] = total;
}
__global__ void __launch_bounds__(kScanThreads) vor_scan_sums_kernel(int n_blocks, int* sums, int* total_out) {
  int total;
  vor_scan_chunk(n_blocks, sums, sums, 0, total);
  if (threadIdx.x == 0) *total_out = total;
}
__global__ void vor_scan_add_kernel(int64_t n, int* out, const int* __restrict__ sums) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < n) out[i] += sums[i / kVoronoiScanChunk];
}

__device__ __forceinline__ long long vor_d2(int ax, int ay, int bx, int by) {
  const long long dx = ax - bx, dy = ay - by;
  return dx * dx + dy * dy;
}
// squared distance from (x, y) to the box [x0, x1] x [y0, y1]
__device__ __forceinline__ long long vor_box_d2(int x, int y, int x0, int y0, int x1, int y1) {
  const long long dx = max(max(x0 - x, x - x1), 0), dy = max(max(y0 - y, y - y1), 0);
  return dx * dx + dy * dy;
}
__device__ __forceinline__ long long vor_block_min(long long v) {
  __shared__ long long sh[kVorThreads / 32];
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int t = threadIdx.y * kVorTile + threadIdx.x;
  if ((t & 31) == 0) sh[t >> 5] = v;
  __syncthreads();
  long long r = sh[0];
  for (int k = 1; k < kVorThreads / 32; ++k) r = min(r, sh[k]);
  __syncthreads();
  return r;
}
// cell k of the Chebyshev ring r around a bucket: top row, bottom row, left and right columns
__device__ __forceinline__ void vor_ring_cell(int r, int k, int& dx, int& dy) {
  if (k < 2 * r + 1) {
    dx = -r + k;
    dy = -r;
  } else if (k < 4 * r + 2) {
    dx = -r + (k - (2 * r + 1));
    dy = r;
  } else if (k < 6 * r + 1) {
    dx = -r;
    dy = -r + 1 + (k - (4 * r + 2));
  } else {
    dx = r;
    dy = -r + 1 + (k - (6 * r + 1));
  }
}
// keep the part of the convex polygon (x, y)[n] where a X + b Y <= c (Sutherland-Hodgman); writes (ox, oy)
__device__ __forceinline__ int vor_clip(const double* x, const double* y, int n, double a, double b, double c, double* ox,
                                        double* oy) {
  int m = 0;
  for (int k = 0; k < n; ++k) {
    const int k1 = k + 1 == n ? 0 : k + 1;
    const double f0 = a * x[k] + b * y[k] - c, f1 = a * x[k1] + b * y[k1] - c;
    if (f0 <= 0 && m < kVorMaxPoly) {
      ox[m] = x[k];
      oy[m] = y[k];
      ++m;
    }
    if (((f0 < 0 && f1 > 0) || (f0 > 0 && f1 < 0)) && m < kVorMaxPoly) {
      const double t = f0 / (f0 - f1);
      ox[m] = x[k] + t * (x[k1] - x[k]);
      oy[m] = y[k] + t * (y[k1] - y[k]);
      ++m;
    }
  }
  return m;
}

// The tile's candidate sites in the fixed order (rows of buckets, index order inside a row): f(site index, site)
// for every site whose squared distance to the tile rectangle is <= U2.
struct VorTile {
  int X0, Y0, X1, Y1;  // quarter-pixel rectangle of the tile (clipped to the image)
  double U2;
  int bx0, bx1, by0, by1;
};
template <class F>
__device__ __forceinline__ void vor_for_tile_sites(const VoronoiGrid& g, const VorTile& T, const int2* __restrict__ sites,
                                                   F f) {
  for (int by = T.by0; by <= T.by1; ++by) {
    const int row = by * g.nx;
    const int a = __ldg(g.off + row + T.bx0), b = __ldg(g.off + row + T.bx1 + 1);
    for (int j = a; j < b; ++j) {
      const int i = __ldg(g.idx + j);
      const int2 s = __ldg(sites + i);
      if (static_cast<double>(vor_box_d2(s.x, s.y, T.X0, T.Y0, T.X1, T.Y1)) > T.U2) continue;
      f(i, s);
    }
  }
}

// area of (cell of site i) n (pixel square), in pixels: the square [0, 4]^2 in quarter pixels relative to the
// pixel corner (qx, qy), clipped by the bisector of i and every other candidate j (enumerated by for_each_j)
template <class ForEachJ>
__device__ __forceinline__ double vor_cell_area(int i, int2 si, int qx, int qy, ForEachJ for_each_j) {
  double px[kVorMaxPoly], py[kVorMaxPoly], tx[kVorMaxPoly], ty[kVorMaxPoly];
  px[0] = 0; py[0] = 0; px[1] = 4; py[1] = 0; px[2] = 4; py[2] = 4; px[3] = 0; py[3] = 4;
  int n = 4;
  const long long rix = si.x - qx, riy = si.y - qy;
  for_each_j([&](int j, int2 sj) {
    if (j == i || n == 0) return;
    const long long rjx = sj.x - qx, rjy = sj.y - qy;
    if (rjx == rix && rjy == riy) {  // a repeated position: the lower index owns it
      if (j < i) n = 0;
      return;
    }
    // |q - r_i|^2 <= |q - r_j|^2  <=>  2 (r_j - r_i) . q <= |r_j|^2 - |r_i|^2
    const double c = static_cast<double>((rjx * rjx + rjy * rjy) - (rix * rix + riy * riy));
    n = vor_clip(px, py, n, 2.0 * static_cast<double>(rjx - rix), 2.0 * static_cast<double>(rjy - riy), c, tx, ty);
    for (int k = 0; k < n; ++k) {
      px[k] = tx[k];
      py[k] = ty[k];
    }
  });
  double area2 = 0;
  for (int k = 0; k < n; ++k) {
    const int k1 = k + 1 == n ? 0 : k + 1;
    area2 += px[k] * py[k1] - px[k1] * py[k];
  }
  return fabs(area2) * (0.5 / 16.0);
}

template <int NCH>
__global__ void __launch_bounds__(kVorThreads)
    voronoi_render_kernel(int w, int h, const int2* __restrict__ sites, const float* __restrict__ colors, VoronoiGrid g,
                          uint8_t* __restrict__ img0, uint8_t* __restrict__ img1) {
  const int tid = threadIdx.y * kVorTile + threadIdx.x;
  const int x = blockIdx.x * kVorTile + threadIdx.x, y = blockIdx.y * kVorTile + threadIdx.y;
  const bool inside = x < w && y < h;
  double acc[NCH];
#pragma unroll
  for (int k = 0; k < NCH; ++k) acc[k] = 0;
  const int n_sites = __ldg(g.off + static_cast<int64_t>(g.nx) * g.ny);
  if (n_sites > 0) {
    VorTile T;
    T.X0 = 4 * blockIdx.x * kVorTile;
    T.Y0 = 4 * blockIdx.y * kVorTile;
    T.X1 = 4 * min(static_cast<int>(blockIdx.x + 1) * kVorTile, w);
    T.Y1 = 4 * min(static_cast<int>(blockIdx.y + 1) * kVorTile, h);
    // 1. exact nearest site of the tile centre: rings of buckets until the ring is farther than the best
    const int cx = (T.X0 + T.X1) / 2, cy = (T.Y0 + T.Y1) / 2;
    const int cbx = min(g.nx - 1, (cx - g.x0) / g.bs), cby = min(g.ny - 1, (cy - g.y0) / g.bs);
    long long best = LLONG_MAX;
    for (int r = 0; r <= max(g.nx, g.ny); ++r) {
      if (r > 1 && best != LLONG_MAX) {
        const long long lb = static_cast<long long>(r - 1) * g.bs;
        if (lb * lb > best) break;
      }
      long long local = LLONG_MAX;
      const int cells = r == 0 ? 1 : 8 * r;
      for (int k = tid; k < cells; k += kVorThreads) {
        int dx = 0, dy = 0;
        if (r > 0) vor_ring_cell(r, k, dx, dy);
        const int bx = cbx + dx, by = cby + dy;
        if (bx < 0 || by < 0 || bx >= g.nx || by >= g.ny) continue;
        const int b = by * g.nx + bx;
        for (int j = __ldg(g.off + b); j < __ldg(g.off + b + 1); ++j) {
          const int2 s = __ldg(sites + __ldg(g.idx + j));
          local = min(local, vor_d2(s.x, s.y, cx, cy));
        }
      }
      best = min(best, vor_block_min(local));
    }
    // 2. every point of the tile is within U of s0
    const double U = sqrt(static_cast<double>(best)) +
                     0.5 * sqrt(static_cast<double>(T.X1 - T.X0) * (T.X1 - T.X0) + static_cast<double>(T.Y1 - T.Y0) * (T.Y1 - T.Y0));
    T.U2 = U * U * (1 + 1e-12) + 1e-6;
    T.bx0 = max(0, static_cast<int>(floor((T.X0 - U - g.x0) / g.bs)));
    T.bx1 = min(g.nx - 1, static_cast<int>(floor((T.X1 + U - g.x0) / g.bs)));
    T.by0 = max(0, static_cast<int>(floor((T.Y0 - U - g.y0) / g.bs)));
    T.by1 = min(g.ny - 1, static_cast<int>(floor((T.Y1 + U - g.y0) / g.bs)));
    // 3. nearest site of the pixel centre and of its four corners
    const int qx = 4 * x, qy = 4 * y;
    long long dc = LLONG_MAX, dk[4] = {LLONG_MAX, LLONG_MAX, LLONG_MAX, LLONG_MAX};
    int ik[4] = {-1, -1, -1, -1};
    vor_for_tile_sites(g, T, sites, [&](int i, int2 s) {
      dc = min(dc, vor_d2(s.x, s.y, qx + 2, qy + 2));
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const long long d = vor_d2(s.x, s.y, qx + 4 * (k & 1), qy + 4 * (k >> 1));
        if (d < dk[k]) {
          dk[k] = d;
          ik[k] = i;
        }
      }
    });
    const bool slow = inside && !(ik[0] == ik[1] && ik[0] == ik[2] && ik[0] == ik[3]);
    if (inside && !slow) {
#pragma unroll
      for (int k = 0; k < NCH; ++k) acc[k] = __ldg(colors + static_cast<int64_t>(ik[0]) * NCH + k);
    }
    if (__syncthreads_or(slow)) {
      // 4. the pixel's candidates: distance to the square <= centre's nearest distance + sqrt(2)/2 px
      const double bound = sqrt(static_cast<double>(dc)) + 2.0 * sqrt(2.0);
      const double bound2 = bound * bound * (1 + 1e-12) + 1e-6;
      int cand[kVorMaxCand];
      int nc = 0;
      bool overflow = false;
      vor_for_tile_sites(g, T, sites, [&](int i, int2 s) {
        if (!slow || static_cast<double>(vor_box_d2(s.x, s.y, qx, qy, qx + 4, qy + 4)) > bound2) return;
        if (nc < kVorMaxCand)
          cand[nc++] = i;
        else
          overflow = true;
      });
      if (slow) {
        auto add = [&](int i, double area) {
          if (area <= 0) return;
#pragma unroll
          for (int k = 0; k < NCH; ++k) acc[k] += area * static_cast<double>(__ldg(colors + static_cast<int64_t>(i) * NCH + k));
        };
        if (!overflow) {
          for (int a = 0; a < nc; ++a) {
            const int i = cand[a];
            add(i, vor_cell_area(i, __ldg(sites + i), qx, qy, [&](auto f) {
                  for (int b = 0; b < nc; ++b) f(cand[b], __ldg(sites + cand[b]));
                }));
          }
        } else {
          auto each = [&](auto f) {
            vor_for_tile_sites(g, T, sites, [&](int j, int2 s) {
              if (static_cast<double>(vor_box_d2(s.x, s.y, qx, qy, qx + 4, qy + 4)) <= bound2) f(j, s);
            });
          };
          each([&](int i, int2 s) { add(i, vor_cell_area(i, s, qx, qy, each)); });
        }
      }
    }
  }
  if (!inside) return;
  const int64_t p = 3 * (static_cast<int64_t>(y) * w + x);
  uint8_t* imgs[2] = {img0, img1};
#pragma unroll
  for (int m = 0; m < NCH / 3; ++m) {
    if (!imgs[m]) continue;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double v = fmin(fmax(acc[3 * m + k] + 0.5, 0.0), static_cast<double>(255.99f));
      imgs[m][p + k] = static_cast<uint8_t>(static_cast<int>(v));
    }
  }
}

void launch_render_voronoi(int w, int h, int64_t n, const int2* sites, const float* colors, int nch, const VoronoiGrid& g,
                           uint8_t* img0, uint8_t* img1, cudaStream_t s) {
  const int64_t nb = static_cast<int64_t>(g.nx) * g.ny;
  cudaMemsetAsync(g.count, 0, sizeof(int) * nb, s);
  if (n > 0) vor_count_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(n, sites, g);
  const int n_blocks = static_cast<int>((nb + kVoronoiScanChunk - 1) / kVoronoiScanChunk);
  vor_scan_blocks_kernel<<<n_blocks, kScanThreads, 0, s>>>(nb, g.count, g.off, g.scan_sums);
  vor_scan_sums_kernel<<<1, kScanThreads, 0, s>>>(n_blocks, g.scan_sums, g.off + nb);
  vor_scan_add_kernel<<<static_cast<unsigned>((nb + 255) / 256), 256, 0, s>>>(nb, g.off, g.scan_sums);
  cudaMemsetAsync(g.count, 0, sizeof(int) * nb, s);
  if (n > 0) vor_scatter_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(n, sites, g);
  vor_sort_buckets_kernel<<<static_cast<unsigned>((nb + 255) / 256), 256, 0, s>>>(g);
  const dim3 grid((w + kVorTile - 1) / kVorTile, (h + kVorTile - 1) / kVorTile);
  if (nch == 6)
    voronoi_render_kernel<6><<<grid, dim3(kVorTile, kVorTile), 0, s>>>(w, h, sites, colors, g, img0, img1);
  else
    voronoi_render_kernel<3><<<grid, dim3(kVorTile, kVorTile), 0, s>>>(w, h, sites, colors, g, img0, nullptr);
}

// CreateVoronoiDiagram (:362-384) and the colour computers (:547-558, :576-586) for one group of observations
// sharing the integer feature pixel ((int)x, (int)y): the first observation (caller's order) whose projection
// succeeded gives the site ((int)(4 x), (int)(4 y)) and, from its error e cast to float,
//   direction: theta = (double)atan2f(e.y, e.x); (127 + 127 sin theta, 127 + 127 cos theta, 127), in double
//   magnitude: f = min(1, (double)|e|_float / 0.5); (255.99f * f, 255.99f * (1 - f), 0), in double
// each rounded to float; no fused multiply-add anywhere.
__global__ void report_sites_kernel(ProblemDev pb, const double2* __restrict__ err, const double* __restrict__ mag,
                                    int64_t n_groups, const int* __restrict__ group_off,
                                    const uint32_t* __restrict__ group_obs, int2* __restrict__ sites,
                                    float* __restrict__ colors) {
  const int64_t g = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (g >= n_groups) return;
  int2 site = make_int2(kVoronoiNoSite, 0);
  float c[6] = {0, 0, 0, 0, 0, 0};
  for (int m = group_off[g]; m < group_off[g + 1]; ++m) {
    const uint32_t o = group_obs[m];
    if (isnan(mag[o])) continue;
    const float2 xy = pb.obs_xy[o];
    site = make_int2(__float2int_rz(4.f * xy.x), __float2int_rz(4.f * xy.y));
    const double2 e = err[o];
    const float ex = static_cast<float>(e.x), ey = static_cast<float>(e.y);
    const double theta = static_cast<double>(atan2f(ey, ex));
    c[0] = static_cast<float>(__dadd_rn(127.0, __dmul_rn(127.0, sin(theta))));
    c[1] = static_cast<float>(__dadd_rn(127.0, __dmul_rn(127.0, cos(theta))));
    c[2] = 127.f;
    const float norm = sqrtf(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)));
    const double f = fmin(1.0, static_cast<double>(norm) / 0.5);
    c[3] = static_cast<float>(__dmul_rn(static_cast<double>(255.99f), f));
    c[4] = static_cast<float>(__dmul_rn(static_cast<double>(255.99f), __dsub_rn(1.0, f)));
    c[5] = 0.f;
    break;
  }
  sites[g] = site;
#pragma unroll
  for (int k = 0; k < 6; ++k) colors[6 * g + k] = c[k];
}
void launch_report_sites(const ProblemDev& pb, const ReportDev& r, int64_t n_groups, const int* group_off,
                         const uint32_t* group_obs, int2* sites, float* colors, cudaStream_t s) {
  if (n_groups == 0) return;
  report_sites_kernel<<<static_cast<unsigned>((n_groups + 127) / 128), 128, 0, s>>>(pb, r.err, r.mag, n_groups, group_off,
                                                                                     group_obs, sites, colors);
}

// The observation-direction colour of a direction d (util.cc:190-229, tools/visualize_calibration.cc:84-93):
// ((70 * 255.99f) / 2.f) * (d + 1) (x, y) and ((270 * 255.99f) / 2.f) * (d + 1) (z) is a double that the reference
// converts to u8 as x86-64 does: truncation to int32, then the low byte (hence the stripes).
__device__ __forceinline__ void direction_colour(d3 d, uint8_t out[3]) {
  const double kxy = static_cast<double>((70 * 255.99f) / 2.f), kz = static_cast<double>((270 * 255.99f) / 2.f);
  out[0] = static_cast<uint8_t>(report_trunc(__dmul_rn(kxy, __dadd_rn(d.x, 1.0))));
  out[1] = static_cast<uint8_t>(report_trunc(__dmul_rn(kxy, __dadd_rn(d.y, 1.0))));
  out[2] = static_cast<uint8_t>(report_trunc(__dmul_rn(kz, __dadd_rn(d.z, 1.0))));
}

// VisualizeModelDirections (:1165-1190) with CreateObservationDirectionsImage (util.cc:190-229): the direction of
// (x + 0.5f, y + 0.5f) (the line direction for non-central models) in direction_colour, black where the un-projection
// fails.
constexpr int kDirTileX = 16, kDirTileY = 8;
__global__ void __launch_bounds__(kDirTileX * kDirTileY)
    observation_directions_kernel(CamDev c, const double* __restrict__ intr, uint8_t* __restrict__ img) {
  const int x = blockIdx.x * kDirTileX + threadIdx.x, y = blockIdx.y * kDirTileY + threadIdx.y;
  if (x >= c.width || y >= c.height) return;
  const double px = static_cast<double>(x + 0.5f), py = static_cast<double>(y + 0.5f);
  uint8_t out[3] = {0, 0, 0};
  if (in_area(c, px, py)) {
    d3 d;
    if (c.model_type == B200BA_MODEL_CENTRAL_GENERIC) {
      CentralEval e;
      central_eval(c, intr, px, py, e);
      d = e.u;
    } else {
      NoncentralEval e;
      noncentral_eval(c, intr, intr + 3 * static_cast<int64_t>(c.gw) * c.gh, px, py, e);
      d = e.u;
    }
    direction_colour(d, out);
  }
  const int64_t p = 3 * (static_cast<int64_t>(y) * c.width + x);
  img[p] = out[0];
  img[p + 1] = out[1];
  img[p + 2] = out[2];
}
void launch_observation_directions(const CamDev& c, const double* intr, uint8_t* img, cudaStream_t s) {
  const dim3 grid((c.width + kDirTileX - 1) / kDirTileX, (c.height + kDirTileY - 1) / kDirTileY);
  observation_directions_kernel<<<grid, dim3(kDirTileX, kDirTileY), 0, s>>>(c, intr, img);
}

// ---- VisualizeCameraModel (APP/tools/visualize_calibration.cc:39-96) for a libvis RadtanCamera8d -----------------------
// The orientation needs the mean un-normalised direction of the window x in [x0, w - 1], y in [y0, y1] to the right of
// the image centre, summed in row-major order as the reference sums it, so that the rotation does not depend on the launch
// shape: radtan8_window_kernel un-projects the window's pixels in parallel, radtan8_orientation_kernel adds them up on
// one thread (three independent accumulators) and forms the rotation, visualize_camera_kernel draws every pixel.
__global__ void radtan8_window_kernel(const double* __restrict__ params, int x0, int nx, int y0, int64_t n,
                                      double2* __restrict__ win) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int x = x0 + static_cast<int>(i % nx), y = y0 + static_cast<int>(i / nx);
  double ux, uy;
  radtan8_unproject(params, static_cast<double>(x + 0.5f), static_cast<double>(y + 0.5f), ux, uy);
  win[i] = make_double2(ux, uy);
}

// The rotation of VisualizeCameraModel (:48-82) from forward = Unproject(0.5f w, 0.5f h) and the window's directions,
// summed on one thread in row-major order (the z components, all 1, summed like the others), every operation but
// atan2 / sin / cos rounded on its own in Eigen's order: tiny images make the angle atan2 of two small numbers formed by
// cancellation, where any other order of the same operations moves the rotation by far more than an ulp. The block
// stages the directions through shared memory so that the summing thread waits on shared-memory rather than L2 latency.
constexpr int kWinThreads = 256, kWinChunk = 2048;
__global__ void __launch_bounds__(kWinThreads)
    radtan8_orientation_kernel(const double* __restrict__ params, int w, int h, int64_t n,
                               const double2* __restrict__ win, double* __restrict__ rot) {
  __shared__ double2 chunk[kWinChunk];
  double sx = 0, sy = 0, sz = 0;
  for (int64_t base = 0; base < n; base += kWinChunk) {
    const int m = static_cast<int>(min(static_cast<int64_t>(kWinChunk), n - base));
    __syncthreads();
    for (int i = threadIdx.x; i < m; i += kWinThreads) chunk[i] = win[base + i];
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll 8
      for (int i = 0; i < m; ++i) {
        const double2 d = chunk[i];
        sx = __dadd_rn(sx, d.x);
        sy = __dadd_rn(sy, d.y);
        sz = __dadd_rn(sz, 1.0);
      }
    }
  }
  if (threadIdx.x != 0) return;
  double fx, fy;
  radtan8_unproject(params, static_cast<double>(0.5f * static_cast<float>(w)),
                    static_cast<double>(0.5f * static_cast<float>(h)), fx, fy);
  // Quaterniond::FromTwoVectors(forward, e_z).toRotationMatrix() in Eigen's order: forward.normalized(); c = e_z . v0;
  // axis = v0 x e_z; s = sqrt((1 + c) * 2); q = (s * 0.5, axis * (1 / s)). Eigen's branch for c < -1 + 1e-12 cannot
  // be taken: the forward direction (u, 1) has c = 1 / |(u, 1)| > 0, or NaN.
  const double sq = __dadd_rn(__dadd_rn(__dmul_rn(fx, fx), __dmul_rn(fy, fy)), 1.0);
  double v0[3] = {fx, fy, 1.0};
  if (sq > 0) {
    const double n = sqrt(sq);
    for (int k = 0; k < 3; ++k) v0[k] = __ddiv_rn(v0[k], n);
  }
  const double c = __dadd_rn(__dadd_rn(__dmul_rn(0.0, v0[0]), __dmul_rn(0.0, v0[1])), __dmul_rn(1.0, v0[2]));
  const double axis[3] = {__dsub_rn(__dmul_rn(v0[1], 1.0), __dmul_rn(v0[2], 0.0)),
                          __dsub_rn(__dmul_rn(v0[2], 0.0), __dmul_rn(v0[0], 1.0)),
                          __dsub_rn(__dmul_rn(v0[0], 0.0), __dmul_rn(v0[1], 0.0))};
  const double s = sqrt(__dmul_rn(__dadd_rn(1.0, c), 2.0)), invs = __ddiv_rn(1.0, s);
  const double qw = __dmul_rn(s, 0.5), qx = __dmul_rn(axis[0], invs), qy = __dmul_rn(axis[1], invs),
               qz = __dmul_rn(axis[2], invs);
  const double tx = __dmul_rn(2.0, qx), ty = __dmul_rn(2.0, qy), tz = __dmul_rn(2.0, qz);
  const double twx = __dmul_rn(tx, qw), twy = __dmul_rn(ty, qw), twz = __dmul_rn(tz, qw);
  const double txx = __dmul_rn(tx, qx), txy = __dmul_rn(ty, qx), txz = __dmul_rn(tz, qx);
  const double tyy = __dmul_rn(ty, qy), tyz = __dmul_rn(tz, qy), tzz = __dmul_rn(tz, qz);
  const double F[9] = {__dsub_rn(1.0, __dadd_rn(tyy, tzz)), __dsub_rn(txy, twz), __dadd_rn(txz, twy),
                       __dadd_rn(txy, twz), __dsub_rn(1.0, __dadd_rn(txx, tzz)), __dsub_rn(tyz, twx),
                       __dsub_rn(txz, twy), __dadd_rn(tyz, twx), __dsub_rn(1.0, __dadd_rn(txx, tyy))};
  // right_sum / right_count, rotated by F; angle = atan2(-y, x); AngleAxisd(angle, e_z).toRotationMatrix() in Eigen's
  // order; rotation = right_rotation * forward_rotation, each entry's products added left to right
  const double count = static_cast<double>(n);
  const double m[3] = {__ddiv_rn(sx, count), __ddiv_rn(sy, count), __ddiv_rn(sz, count)};
  double r[3];
  for (int i = 0; i < 3; ++i)
    r[i] = __dadd_rn(__dadd_rn(__dmul_rn(F[3 * i], m[0]), __dmul_rn(F[3 * i + 1], m[1])), __dmul_rn(F[3 * i + 2], m[2]));
  const double angle = atan2(-r[1], r[0]);
  const double ca = cos(angle), sa = sin(angle);
  const double Rz[9] = {ca, -sa, 0.0, sa, ca, 0.0, 0.0, 0.0, __dadd_rn(__dsub_rn(1.0, ca), ca)};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      rot[3 * i + j] = __dadd_rn(__dadd_rn(__dmul_rn(Rz[3 * i], F[j]), __dmul_rn(Rz[3 * i + 1], F[3 + j])),
                                 __dmul_rn(Rz[3 * i + 2], F[6 + j]));
}

// Every pixel: d = Unproject(x + 0.5f, y + 0.5f), normalized() (d / sqrt(|d|^2), a zero vector unchanged), rotated
// (row-major R, the products of each row added left to right) and coloured with direction_colour. dirs (nullable):
// the rotated unit directions [h * w * 3].
__global__ void __launch_bounds__(kDirTileX * kDirTileY)
    visualize_camera_kernel(const double* __restrict__ params, int w, int h, const double* __restrict__ rot,
                            uint8_t* __restrict__ img, double* __restrict__ dirs) {
  const int x = blockIdx.x * kDirTileX + threadIdx.x, y = blockIdx.y * kDirTileY + threadIdx.y;
  if (x >= w || y >= h) return;
  double ux, uy;
  radtan8_unproject(params, static_cast<double>(x + 0.5f), static_cast<double>(y + 0.5f), ux, uy);
  double vx = ux, vy = uy, vz = 1.0;
  const double sq = __dadd_rn(__dadd_rn(__dmul_rn(ux, ux), __dmul_rn(uy, uy)), 1.0);
  if (sq > 0) {
    const double n = sqrt(sq);
    vx = __ddiv_rn(vx, n);
    vy = __ddiv_rn(vy, n);
    vz = __ddiv_rn(vz, n);
  }
  double r[3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
    r[i] = __dadd_rn(__dadd_rn(__dmul_rn(__ldg(rot + 3 * i), vx), __dmul_rn(__ldg(rot + 3 * i + 1), vy)),
                     __dmul_rn(__ldg(rot + 3 * i + 2), vz));
  uint8_t out[3];
  direction_colour(mk3(r[0], r[1], r[2]), out);
  const int64_t p = 3 * (static_cast<int64_t>(y) * w + x);
  img[p] = out[0];
  img[p + 1] = out[1];
  img[p + 2] = out[2];
  if (dirs) {
    dirs[p] = r[0];
    dirs[p + 1] = r[1];
    dirs[p + 2] = r[2];
  }
}

void launch_visualize_orientation(const double* params, int w, int h, double2* win, double* rot, cudaStream_t s) {
  const int x0 = std::min(w - 1, w / 2 + 11), y0 = std::max(0, h / 2 - 10), y1 = std::min(h - 1, h / 2 + 10);
  const int nx = w - x0;
  const int64_t n = static_cast<int64_t>(nx) * (y1 - y0 + 1);
  radtan8_window_kernel<<<static_cast<unsigned>((n + 127) / 128), 128, 0, s>>>(params, x0, nx, y0, n, win);
  radtan8_orientation_kernel<<<1, kWinThreads, 0, s>>>(params, w, h, n, win, rot);
}
void launch_visualize_camera(const double* params, int w, int h, const double* rot, uint8_t* img, double* dirs,
                             cudaStream_t s) {
  const dim3 grid((w + kDirTileX - 1) / kDirTileX, (h + kDirTileY - 1) / kDirTileY);
  visualize_camera_kernel<<<grid, dim3(kDirTileX, kDirTileY), 0, s>>>(params, w, h, rot, img, dirs);
}

// Generic small-block Schur preparation for b200ba_schur_solve (block size <= 6, arbitrary
// symmetric blocks like the reference's known-answer test): D^-1 by Gauss-Jordan with partial
// pivoting on the symmetrised block; DinvB = D^-1 B, Dinvb = D^-1 b1.
__global__ void generic_block_inverse_kernel(int bs, int nb, int nd, const double* __restrict__ D,
                                             const double* __restrict__ B, const double* __restrict__ b1,
                                             double* __restrict__ DinvB, double* __restrict__ Dinvb) {
  const int blk = blockIdx.x;
  __shared__ double inv[36];
  if (threadIdx.x == 0) {
    double a[6][12];
    for (int i = 0; i < bs; ++i)
      for (int j = 0; j < bs; ++j) {
        a[i][j] = (i <= j) ? D[(static_cast<int64_t>(blk) * bs + i) * bs + j] : D[(static_cast<int64_t>(blk) * bs + j) * bs + i];
        a[i][bs + j] = (i == j) ? 1.0 : 0.0;
      }
    for (int col = 0; col < bs; ++col) {
      int piv = col;
      for (int r = col + 1; r < bs; ++r)
        if (fabs(a[r][col]) > fabs(a[piv][col])) piv = r;
      if (piv != col)
        for (int j = 0; j < 2 * bs; ++j) {
          const double t = a[col][j];
          a[col][j] = a[piv][j];
          a[piv][j] = t;
        }
      const double ip = 1.0 / a[col][col];
      for (int j = 0; j < 2 * bs; ++j) a[col][j] *= ip;
      for (int r = 0; r < bs; ++r)
        if (r != col) {
          const double f = a[r][col];
          for (int j = 0; j < 2 * bs; ++j) a[r][j] -= f * a[col][j];
        }
    }
    for (int i = 0; i < bs; ++i)
      for (int j = 0; j < bs; ++j) inv[i * bs + j] = a[i][bs + j];
  }
  __syncthreads();
  for (int col = threadIdx.x; col < nd + 1; col += blockDim.x) {
    for (int r = 0; r < bs; ++r) {
      double s = 0;
      for (int k = 0; k < bs; ++k) {
        const double bv = (col < nd) ? B[(static_cast<int64_t>(blk) * bs + k) * nd + col] : b1[blk * bs + k];
        s += inv[r * bs + k] * bv;
      }
      if (col < nd)
        DinvB[(static_cast<int64_t>(blk) * bs + r) * nd + col] = s;
      else
        Dinvb[blk * bs + r] = s;
    }
  }
}
void launch_generic_block_inverse(int bs, int nb, int nd, const double* D, const double* B, const double* b1,
                                  double* DinvB, double* Dinvb, cudaStream_t s) {
  if (nb == 0) return;
  generic_block_inverse_kernel<<<nb, 128, 0, s>>>(bs, nb, nd, D, B, b1, DinvB, Dinvb);
}

// dst[i] = src[perm[i]] (gather) or dst[perm[i]] = src[i] (scatter) for double2 payloads: moves
// last_projection between the caller's observation order and the device's cell-major order.
__global__ void permute_double2_kernel(int64_t n, const uint32_t* __restrict__ perm, const double2* __restrict__ src,
                                       double2* __restrict__ dst, int scatter) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  if (scatter)
    dst[perm[i]] = src[i];
  else
    dst[i] = src[perm[i]];
}
void launch_permute_double2(int64_t n, const uint32_t* perm, const double2* src, double2* dst, bool scatter,
                            cudaStream_t s) {
  if (n == 0) return;
  permute_double2_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(n, perm, src, dst, scatter ? 1 : 0);
}

// mirror the valid (row <= col) triangle of a row-major square matrix into the other one
__global__ void symmetrize_kernel(int n, double* M) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = blockIdx.y * blockDim.y + threadIdx.y;
  if (i < n && j < n && i < j) M[static_cast<int64_t>(j) * n + i] = M[static_cast<int64_t>(i) * n + j];
}
void launch_symmetrize(int n, double* M, cudaStream_t s) {
  if (n == 0) return;
  dim3 block(32, 8);
  dim3 grid((n + 31) / 32, (n + 7) / 8);
  symmetrize_kernel<<<grid, block, 0, s>>>(n, M);
}

// ---- direction-grid fit (SURVEY.md 8f-4): CentralGenericBSplineDirectionCostFunction -----------
// (APP/models/central_generic.cc:152-228, residual / Jacobian of :86-150). One thread per sample
// (grid point, measured unit direction): r = normalise(sum w G) - m; d r / d (local update of
// control point k) = w_k / |s| (I - u u^T) [t1 t2]_k. A warp holds 32 consecutive samples of a
// raster scan, which almost always share the 4x4 support: the 3 x 32 Jacobians are staged in
// shared memory and lane L sums the (a <= c) pairs p = L, L + 32, ... of J^T J over the 32
// samples before ONE atomic per entry; a warp that straddles a cell border falls back to one set
// of atomics per sample. Not a hot path (<= 90 000 samples, <= 3 LM iterations per resampling).
__global__ void dirfit_tangents_kernel(int G, const double* __restrict__ grid, double* __restrict__ tan) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G) return;
  d3 t1, t2;
  compute_tangents(ld3(grid + 3 * static_cast<int64_t>(i)), t1, t2);
  double* o = tan + 6 * static_cast<int64_t>(i);
  o[0] = t1.x; o[1] = t1.y; o[2] = t1.z;
  o[3] = t2.x; o[4] = t2.y; o[5] = t2.z;
}

// support of grid point (gx, gy): top-left control point and the fractions in [0, 1)
// (ix = floor(g + 2), x0 = ix - 3, frac = g + 2 - x0 - 3: central_generic.cc:94-98 in the
// u-form of bspline_basis)
__device__ __forceinline__ void dirfit_locate(double g, int& i0, double& u) {
  const double f = floor(g + 2.0);
  i0 = static_cast<int>(f) - 3;
  u = (g + 2.0) - f;
}

constexpr int kDirfitRow = 33;  // padded row of the staged Jacobians (lane = sample)

template <bool JAC>
__global__ void __launch_bounds__(32) dirfit_kernel(int gw, int64_t n, const double* __restrict__ gp,
                                                    const double* __restrict__ dirs, const double* __restrict__ grid,
                                                    const double* __restrict__ tan, double* __restrict__ H,
                                                    double* __restrict__ b, int dof, double* __restrict__ cost) {
  __shared__ double sJ[JAC ? 96 * kDirfitRow : 1];
  __shared__ double sR[JAC ? 3 * kDirfitRow : 1];
  const int lane = threadIdx.x;
  const int64_t i = blockIdx.x * 32ll + lane;
  const bool active = i < n;
  int x0 = 0, y0 = 0;
  d3 r = mk3(0, 0, 0);
  if (active) {
    double fu, fv;
    dirfit_locate(gp[2 * i], x0, fu);
    dirfit_locate(gp[2 * i + 1], y0, fv);
    double wx[4], dwx[4], wy[4], dwy[4];
    bspline_basis(fu, wx, dwx);
    bspline_basis(fv, wy, dwy);
    d3 v, vx, vy;
    spline3(grid, gw, x0, y0, wx, dwx, wy, dwy, v, vx, vy);
    const double inv = 1.0 / sqrt(dot3(v, v));
    const d3 u = inv * v;
    r = u - mk3(dirs[3 * i], dirs[3 * i + 1], dirs[3 * i + 2]);
    cost[i] = 0.5 * dot3(r, r);
    if (JAC) {
#pragma unroll 1
      for (int k = 0; k < 16; ++k) {
        const int seq = (x0 + (k & 3)) + (y0 + (k >> 2)) * gw;
        const double w = sel4(wx, k & 3) * sel4(wy, k >> 2) * inv;
        const d3 t1 = ld3(tan + 6 * static_cast<int64_t>(seq)), t2 = ld3(tan + 6 * static_cast<int64_t>(seq) + 3);
        const d3 c1 = w * (t1 - dot3(u, t1) * u);
        const d3 c2 = w * (t2 - dot3(u, t2) * u);
        sJ[(0 * 32 + 2 * k) * kDirfitRow + lane] = c1.x;
        sJ[(1 * 32 + 2 * k) * kDirfitRow + lane] = c1.y;
        sJ[(2 * 32 + 2 * k) * kDirfitRow + lane] = c1.z;
        sJ[(0 * 32 + 2 * k + 1) * kDirfitRow + lane] = c2.x;
        sJ[(1 * 32 + 2 * k + 1) * kDirfitRow + lane] = c2.y;
        sJ[(2 * 32 + 2 * k + 1) * kDirfitRow + lane] = c2.z;
      }
    }
  }
  if (!JAC) return;
  if (!active) {
    for (int row = 0; row < 96; ++row) sJ[row * kDirfitRow + lane] = 0.0;
  }
  sR[0 * kDirfitRow + lane] = r.x;
  sR[1 * kDirfitRow + lane] = r.y;
  sR[2 * kDirfitRow + lane] = r.z;
  // inactive lanes adopt lane 0's support (their contributions are zero)
  const int key = x0 + y0 * gw;
  const int key0 = __shfl_sync(0xffffffffu, key, 0);
  const bool uniform = __all_sync(0xffffffffu, !active || key == key0);
  __syncwarp();
  if (uniform) {
    const int bx0 = __shfl_sync(0xffffffffu, x0, 0), by0 = __shfl_sync(0xffffffffu, y0, 0);
    auto gidx = [&](int a) { return 2 * ((bx0 + ((a >> 1) & 3)) + (by0 + (a >> 3)) * gw) + (a & 1); };
    // b: lane a owns entry a
    {
      double acc = 0;
      for (int q = 0; q < 3; ++q)
        for (int s2 = 0; s2 < 32; ++s2) acc = fma(sJ[(q * 32 + lane) * kDirfitRow + s2], sR[q * kDirfitRow + s2], acc);
      atomicAdd(&b[gidx(lane)], acc);
    }
    // H: pairs (a <= c) in row-major order of the upper triangle, p = lane, lane + 32, ...
    int a = 0, c = lane;  // pair index lane in row a = 0 (32 entries)
    for (int p = lane; p < 528; p += 32) {
      // advance (a, c) so that it is the p-th pair: rows have 32 - a entries
      while (c >= 32) {
        c = c - 32 + (a + 1);  // wrap into the next row, which starts at column a + 1
        ++a;
      }
      double acc = 0;
      for (int q = 0; q < 3; ++q) {
        const double* ja = sJ + (q * 32 + a) * kDirfitRow;
        const double* jc = sJ + (q * 32 + c) * kDirfitRow;
        for (int s2 = 0; s2 < 32; ++s2) acc = fma(ja[s2], jc[s2], acc);
      }
      atomicAdd(&H[static_cast<int64_t>(gidx(a)) * dof + gidx(c)], acc);
      c += 32;
    }
  } else if (active) {
    auto gidx = [&](int a) { return 2 * ((x0 + ((a >> 1) & 3)) + (y0 + (a >> 3)) * gw) + (a & 1); };
    for (int a = 0; a < 32; ++a) {
      const double j0 = sJ[(0 * 32 + a) * kDirfitRow + lane], j1 = sJ[(1 * 32 + a) * kDirfitRow + lane],
                   j2 = sJ[(2 * 32 + a) * kDirfitRow + lane];
      atomicAdd(&b[gidx(a)], fma(j0, r.x, fma(j1, r.y, j2 * r.z)));
      const int64_t rowoff = static_cast<int64_t>(gidx(a)) * dof;
      for (int c = a; c < 32; ++c)
        atomicAdd(&H[rowoff + gidx(c)], fma(j0, sJ[(0 * 32 + c) * kDirfitRow + lane],
                                            fma(j1, sJ[(1 * 32 + c) * kDirfitRow + lane],
                                                j2 * sJ[(2 * 32 + c) * kDirfitRow + lane])));
    }
  }
}

// deterministic sum of n doubles (one block)
__global__ void dirfit_sum_kernel(int64_t n, const double* __restrict__ v, double* __restrict__ out) {
  __shared__ double sh[1024];
  double acc = 0;
  for (int64_t i = threadIdx.x; i < n; i += 1024) acc += v[i];
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = sh[0];
}

// DirectionGridStateWithLocalUpdates::operator-= (central_generic.cc:65-80):
// d <- normalise(d - x0 t1 - x1 t2) with the tangents of the OLD direction
__global__ void dirfit_update_kernel(int G, const double* __restrict__ grid, const double* __restrict__ x,
                                     double* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= G) return;
  const d3 d = ld3(grid + 3 * static_cast<int64_t>(i));
  d3 t1, t2;
  compute_tangents(d, t1, t2);
  const d3 nd = (d + (-x[2 * i]) * t1) + (-x[2 * i + 1]) * t2;
  const double n = sqrt(dot3(nd, nd));
  out[3 * static_cast<int64_t>(i)] = nd.x / n;
  out[3 * static_cast<int64_t>(i) + 1] = nd.y / n;
  out[3 * static_cast<int64_t>(i) + 2] = nd.z / n;
}

void launch_dirfit_tangents(int G, const double* grid, double* tan, cudaStream_t s) {
  if (G > 0) dirfit_tangents_kernel<<<(G + 127) / 128, 128, 0, s>>>(G, grid, tan);
}
void launch_dirfit(bool jac, int gw, int64_t n, const double* gp, const double* dirs, const double* grid,
                   const double* tan, double* H, double* b, int dof, double* cost, double* cost_sum, cudaStream_t s) {
  if (n > 0) {
    const unsigned blocks = static_cast<unsigned>((n + 31) / 32);
    if (jac)
      dirfit_kernel<true><<<blocks, 32, 0, s>>>(gw, n, gp, dirs, grid, tan, H, b, dof, cost);
    else
      dirfit_kernel<false><<<blocks, 32, 0, s>>>(gw, n, gp, dirs, grid, tan, H, b, dof, cost);
  }
  dirfit_sum_kernel<<<1, 1024, 0, s>>>(n, cost, cost_sum);
}
void launch_dirfit_update(int G, const double* grid, const double* x, double* out, cudaStream_t s) {
  if (G > 0) dirfit_update_kernel<<<(G + 127) / 128, 128, 0, s>>>(G, grid, x, out);
}


// ------------------------------------------------------------------------------------------
// ChooseNiceCameraOrientation on the device (APP/models/central_generic.cc:570-621)
// ------------------------------------------------------------------------------------------
// One block per camera: forward = Unproject(image centre), right = mean Unproject over the 21-row strip to
// the right of the centre; rotation = Rz(angle) * FromTwoVectors(forward, e_z). The rotation is written
// to rot[9 * cam] (row-major); cameras that are not central-generic get the identity (the base class
// and the non-central model return it: camera_model.h:120-122, noncentral_generic.h:128-132).
__global__ void nice_orientation_kernel(ProblemDev pb, StateDev st, double* __restrict__ rot) {
  const int cam = blockIdx.x;
  const CamDev& c = pb.cams[cam];
  double* Rout = rot + 9 * cam;
  if (c.model_type != B200BA_MODEL_CENTRAL_GENERIC) {
    if (threadIdx.x < 9) Rout[threadIdx.x] = (threadIdx.x % 4 == 0) ? 1.0 : 0.0;
    return;
  }
  const double* grid = st.intrinsics + c.intr_off;
  __shared__ double sh[4][256];
  const int w = c.width, h = c.height;
  const int x0 = min(w - 1, w / 2 + 11), x1 = w - 1;
  const int y0 = max(0, h / 2 - 10), y1 = min(h - 1, h / 2 + 10);
  const int nx = x1 - x0 + 1, ny = y1 - y0 + 1;
  double sx = 0, sy = 0, sz = 0, cnt = 0;
  for (int i = threadIdx.x; i < nx * ny; i += blockDim.x) {
    const double px = static_cast<double>(x0 + i % nx) + 0.5, py = static_cast<double>(y0 + i / nx) + 0.5;
    if (!in_area(c, px, py)) continue;
    CentralEval e;
    central_eval(c, grid, px, py, e);
    sx += e.u.x;
    sy += e.u.y;
    sz += e.u.z;
    cnt += 1.0;
  }
  sh[0][threadIdx.x] = sx;
  sh[1][threadIdx.x] = sy;
  sh[2][threadIdx.x] = sz;
  sh[3][threadIdx.x] = cnt;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {  // fixed-order tree: deterministic
    if (threadIdx.x < o)
      for (int q = 0; q < 4; ++q) sh[q][threadIdx.x] += sh[q][threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  // the reference passes float pixel coordinates (0.5f * width())
  const double cx = static_cast<double>(0.5f * static_cast<float>(w)), cy = static_cast<double>(0.5f * static_cast<float>(h));
  d3 fwd = mk3(0, 0, 1);
  if (in_area(c, cx, cy)) {
    CentralEval e;
    central_eval(c, grid, cx, cy, e);
    fwd = e.u;
  }
  // Quaterniond::FromTwoVectors(forward, e_z)
  const d3 v0 = rsqrt(dot3(fwd, fwd)) * fwd;
  const double cc = v0.z;
  q4 q;
  if (cc < -1.0 + 1e-12) {
    d3 axis = cross3(v0, mk3(1, 0, 0));
    if (dot3(axis, axis) < 1e-12) axis = cross3(v0, mk3(0, 1, 0));
    axis = rsqrt(dot3(axis, axis)) * axis;
    q = q4{0.0, axis.x, axis.y, axis.z};
  } else {
    const d3 axis = cross3(v0, mk3(0, 0, 1));
    const double s2 = sqrt((1.0 + cc) * 2.0);
    q = q4{0.5 * s2, axis.x / s2, axis.y / s2, axis.z / s2};
  }
  double F[9];
  qrot(q, F);
  double Rz[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  if (sh[3][0] > 0) {
    const d3 mean = (1.0 / sh[3][0]) * mk3(sh[0][0], sh[1][0], sh[2][0]);
    const d3 frr = rot_apply(F, mean);
    const double angle = atan2(-frr.y, frr.x);
    const double ca = cos(angle), sa = sin(angle);
    Rz[0] = ca;
    Rz[1] = -sa;
    Rz[3] = sa;
    Rz[4] = ca;
  }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) Rout[3 * i + j] = Rz[3 * i] * F[j] + Rz[3 * i + 1] * F[3 + j] + Rz[3 * i + 2] * F[6 + j];
}

// Rotate(): every grid direction d <- rotation d; camera_tr_rig <- SE3(rotation, 0) * camera_tr_rig
// (APP/calibration.cc:246-252).
__global__ void apply_orientation_kernel(ProblemDev pb, StateDev st, const double* __restrict__ rot, int n_cameras) {
  const int cam = blockIdx.y;
  const CamDev& c = pb.cams[cam];
  if (c.model_type != B200BA_MODEL_CENTRAL_GENERIC) return;
  double R[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) R[i] = rot[9 * cam + i];
  const int64_t G = static_cast<int64_t>(c.gw) * c.gh;
  const int64_t k = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (k < G) {
    double* g = st.intrinsics + c.intr_off + 3 * k;
    const d3 r = rot_apply(R, mk3(g[0], g[1], g[2]));
    g[0] = r.x;
    g[1] = r.y;
    g[2] = r.z;
  }
  if (k == 0) {
    // rotation matrix -> unit quaternion (Eigen's QuaternionBase::operator=(MatrixBase))
    q4 q;
    const double t = R[0] + R[4] + R[8];
    if (t > 0) {
      const double s = sqrt(t + 1.0) * 2;
      q = q4{0.25 * s, (R[7] - R[5]) / s, (R[2] - R[6]) / s, (R[3] - R[1]) / s};
    } else {
      int i = 0;
      if (R[4] > R[0]) i = 1;
      if (R[8] > R[4 * i]) i = 2;
      const int j = (i + 1) % 3, kk = (i + 2) % 3;
      const double s = sqrt(R[4 * i] - R[4 * j] - R[4 * kk] + 1.0) * 2;
      double v[3];
      v[i] = 0.25 * s;
      v[j] = (R[3 * j + i] + R[3 * i + j]) / s;
      v[kk] = (R[3 * kk + i] + R[3 * i + kk]) / s;
      q = q4{(R[3 * kk + j] - R[3 * j + kk]) / s, v[0], v[1], v[2]};
    }
    const double qn = rsqrt(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
    q = q4{q.w * qn, q.x * qn, q.y * qn, q.z * qn};
    double* p = st.camera_tr_rig + 7 * cam;
    q4 r = qmul(q, q4{p[0], p[1], p[2], p[3]});
    // Sophus' product renormalises to first order when the squared norm is not exactly 1
    const double sn = r.w * r.w + r.x * r.x + r.y * r.y + r.z * r.z;
    if (sn != 1.0) {
      const double sc = 2.0 / (1.0 + sn);
      r = q4{r.w * sc, r.x * sc, r.y * sc, r.z * sc};
    }
    double Q[9];
    qrot(q, Q);
    const d3 tt = rot_apply(Q, mk3(p[4], p[5], p[6]));
    p[0] = r.w;
    p[1] = r.x;
    p[2] = r.y;
    p[3] = r.z;
    p[4] = tt.x;
    p[5] = tt.y;
    p[6] = tt.z;
  }
}

void launch_nice_orientation(const ProblemDev& pb, const StateDev& st, int n_cameras, double* rot, cudaStream_t s) {
  if (n_cameras <= 0) return;
  nice_orientation_kernel<<<n_cameras, 256, 0, s>>>(pb, st, rot);
  int64_t gmax = 1;
  for (int c = 0; c < n_cameras; ++c) gmax = std::max<int64_t>(gmax, static_cast<int64_t>(pb.cams[c].gw) * pb.cams[c].gh);
  dim3 grid(static_cast<unsigned>((gmax + 127) / 128), n_cameras);
  apply_orientation_kernel<<<grid, 128, 0, s>>>(pb, st, rot, n_cameras);
}


// ------------------------------------------------------------------------------------------
// FixVariable (LV/lm_optimizer.h:360-368, :1069-1121): the fixed unknowns are removed from the system.
// Here: their rows / columns of H are zeroed, the diagonal set to 1 and b to 0, so the solve returns a
// zero update for them and the remaining unknowns see exactly the thinned system.
// ------------------------------------------------------------------------------------------
__global__ void mask_fixed_blocks_kernel(Layout L, SystemDev sys, FixedRanges fr) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= L.nblocks) return;
  double* D = sys.Dblk + static_cast<int64_t>(L.dsz) * p;
  for (int a = 0; a < L.bs; ++a)
    for (int b = a; b < L.bs; ++b) {
      const bool fa = fr.has(L.bs * p + a), fb = fr.has(L.bs * p + b);
      if (fa || fb) D[a * L.bs - (a * (a - 1)) / 2 + (b - a)] = (a == b) ? 1.0 : 0.0;
    }
  for (int a = 0; a < L.bs; ++a)
    if (fr.has(L.bs * p + a)) sys.bp[L.bs * p + a] = 0.0;
}
__global__ void mask_fixed_B_kernel(Layout L, SystemDev sys, FixedRanges fr) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  const int row = blockIdx.y;
  if (col >= L.nd || row >= L.nbd) return;
  if (fr.has(row) || fr.has(L.nbd + col)) sys.B[static_cast<int64_t>(row) * L.nd + col] = 0.0;
}
__global__ void mask_fixed_C_kernel(Layout L, SystemDev sys, FixedRanges fr, double unit) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  const int row = blockIdx.y;
  if (col >= L.nd || row >= L.nd || col < row) return;
  const bool fr_ = fr.has(L.nbd + row), fc = fr.has(L.nbd + col);
  if (fr_ || fc) sys.C[static_cast<int64_t>(row) * L.nd + col] = (row == col) ? unit : 0.0;
  if (row == col && fr_) sys.bd[row] = 0.0;
}
void launch_mask_fixed(const Layout& L, const SystemDev& sys, const FixedRanges& fr, double unit, cudaStream_t s) {
  if (fr.n == 0) return;
  if (L.nblocks > 0) mask_fixed_blocks_kernel<<<(L.nblocks + 127) / 128, 128, 0, s>>>(L, sys, fr);
  if (L.nbd > 0 && L.nd > 0) {
    dim3 g((L.nd + 255) / 256, L.nbd);
    mask_fixed_B_kernel<<<g, 256, 0, s>>>(L, sys, fr);
  }
  if (L.nd > 0) {
    dim3 g((L.nd + 255) / 256, L.nd);
    mask_fixed_C_kernel<<<g, 256, 0, s>>>(L, sys, fr, unit);
  }
}

// ---- feature intersection (b200ba_intersect_features; APP/tools/intersect_datasets.cc:130-225) -------------------
// The reference erases features from std::vectors while it walks dataset 0 by index. Erasing keeps the order of the
// remaining elements, so every position in a current vector is the rank of an original index among the alive ones,
// and the same walk runs on the original arrays with one alive flag per feature:
//   - "the last index o with d <= best" is the last ALIVE original index with the smallest d <= thr2: an erased
//     feature's x is overwritten with NaN, so its d is NaN and never accepted;
//   - covered-index vectors of two passes of one fixed-point loop compare equal as positions exactly when they do as
//     original indices (nothing is erased inside the loop);
//   - after a rejection the reference erases the covered features and steps f back by one where covered[0] <= f,
//     then advances it by one. With covered[0] < f the element at f moved to f - 1, so the new f is the element after
//     the old f; with covered[0] == f it is the element after the erased one; with covered[0] > f, f + 1 is the next
//     element that is still there. In each case: the next alive original index after f. With covered[0] == -1 the
//     same f runs again, and after an acceptance the next alive index follows.
// Comparisons d <= thr2 (float d, double thr2) are d <= bound in float, bound = the largest float <= thr2.
constexpr int kIntersectMaxPasses = 100;
constexpr int kIntersectSmemBytes = 200 * 1024;  // lists up to 25600 features are staged in shared memory

// (float)(p.x - cx)^2 + (float)(p.y - cy)^2, each operation rounded on its own
__device__ __forceinline__ float intersect_d2(float2 p, float cx, float cy) {
  const float dx = __fsub_rn(p.x, cx), dy = __fsub_rn(p.y, cy);
  return __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
}

// The closest feature of pts [b, e) to (cx, cy) with d <= bound, ties to the later index; -1 if none. One warp; every
// lane returns the same index ((d, index) is reduced under one total order: smaller d first, then larger index).
__device__ int intersect_closest(const float2* pts, int b, int e, float cx, float cy, float bound, int lane) {
  float best = bound;
  int idx = -1;
#pragma unroll 4
  for (int k = b + lane; k < e; k += 32) {
    const float d = intersect_d2(pts[k], cx, cy);
    if (d <= best) {  // a lane sees its indices in increasing order, so a tie goes to the later one
      best = d;
      idx = k;
    }
  }
#pragma unroll
  for (int s = 16; s; s >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, s);
    const int oi = __shfl_xor_sync(0xffffffffu, idx, s);
    if (ob < best || (ob == best && oi > idx)) {
      best = ob;
      idx = oi;
    }
  }
  return idx;
}

// One CTA per list, one warp per dataset: warp w answers the closest-feature query of dataset w in every pass, and
// every thread then forms the same centre from the covered features in dataset order. The walk, the fixed-point loop
// and the acceptance are uniform over the CTA. Both loops are bounded: a pass loop by kIntersectMaxPasses, the walk by
// n0 advances plus one re-run per erased feature (a re-run without an erasure is the pinned "uncovered" case, which
// advances).
__global__ void __launch_bounds__(1024) intersect_walk_kernel(int D, const int64_t* __restrict__ off, float2* xy,
                                                              int use_smem, float bound, uint8_t* keep, float2* centres,
                                                              int* n_centres, unsigned long long* counts) {
  extern __shared__ float2 s_pts[];
  __shared__ int s_cov[32], s_old[32], s_b[33];
  const int64_t l = blockIdx.x;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t* o = off + l * D;
  const int64_t base = o[0];
  const int total = static_cast<int>(o[D] - base);
  float2* pts = xy + base;
  if (use_smem) {
    for (int k = threadIdx.x; k < total; k += blockDim.x) s_pts[k] = pts[k];
    pts = s_pts;
  }
  if (threadIdx.x <= D) s_b[threadIdx.x] = static_cast<int>(o[threadIdx.x] - base);
  __syncthreads();
  const int n0 = s_b[1], bw = s_b[w], ew = s_b[w + 1];
  uint8_t* alive = keep + base;
  float2* cent = centres + base;
  int nc = 0;
  unsigned long long uncovered = 0, capped = 0;
  int f = 0;
  while (f < n0) {
    float cx = pts[f].x, cy = pts[f].y;
    int k = -1;
    for (int pass = 1;; ++pass) {
      k = intersect_closest(pts, bw, ew, cx, cy, bound, lane);
      if (lane == 0) s_cov[w] = k;
      __syncthreads();
      float sx = 0.f, sy = 0.f;
      int count = 0;
      bool same = pass > 1;  // the first pass compares against an empty vector
      for (int i = 0; i < D; ++i) {
        const int ki = s_cov[i];
        if (ki >= 0) {
          const float2 p = pts[ki];
          sx = __fadd_rn(sx, p.x);
          sy = __fadd_rn(sy, p.y);
          ++count;
        }
        same = same && ki == s_old[i];
      }
      cx = __fdiv_rn(sx, static_cast<float>(count));
      cy = __fdiv_rn(sy, static_cast<float>(count));
      __syncthreads();  // s_cov and s_old are read by every thread before they change
      if (same) break;
      if (lane == 0) s_old[w] = k;
      if (pass == kIntersectMaxPasses) {
        ++capped;
        break;
      }
    }
    bool accept = true, any = false;
    for (int i = 0; i < D; ++i) {
      accept = accept && s_cov[i] >= 0;
      any = any || s_cov[i] >= 0;
    }
    const int c0 = s_cov[0];
    if (accept) {
      if (threadIdx.x == 0) cent[nc] = make_float2(cx, cy);
      ++nc;
    } else if (!any) {
      ++uncovered;
    } else if (lane == 0 && k >= 0) {
      pts[k].x = __int_as_float(0x7fc00000);
      alive[k] = 0;
    }
    __syncthreads();  // erasures are visible, and s_cov is read, before the next walk step
    if (accept || !any || c0 != -1) {
      ++f;
      while (f < n0 && !alive[f]) ++f;
    }
  }
  if (threadIdx.x == 0) {
    n_centres[l] = nc;
    if (uncovered) atomicAdd(counts, uncovered);
    if (capped) atomicAdd(counts + 1, capped);
  }
}

// The final pass: every alive feature of list l is kept where some accepted centre lies within thr2 of it.
__global__ void intersect_keep_kernel(int D, const int64_t* __restrict__ off, const float2* __restrict__ xy, float bound,
                                      const float2* __restrict__ centres, const int* __restrict__ n_centres,
                                      uint8_t* keep) {
  const int64_t l = blockIdx.x;
  const int64_t base = off[l * D], end = off[l * D + D];
  const int nc = n_centres[l];
  const float2* cent = centres + base;
  for (int64_t k = base + threadIdx.x; k < end; k += blockDim.x) {
    if (!keep[k]) continue;
    const float2 p = xy[k];
    uint8_t near = 0;
    for (int c = 0; c < nc; ++c) {
      const float2 q = __ldg(cent + c);
      if (intersect_d2(p, q.x, q.y) <= bound) {  // (c - p)^2 == (p - c)^2 bit for bit
        near = 1;
        break;
      }
    }
    keep[k] = near;
  }
}

void launch_intersect_features(int d, int64_t n_lists, int64_t max_list, const int64_t* off, float2* xy, float bound,
                               uint8_t* keep, float2* centres, int* n_centres, unsigned long long* counts,
                               cudaStream_t s) {
  if (n_lists == 0 || max_list == 0) return;
  const size_t bytes = sizeof(float2) * static_cast<size_t>(max_list);
  const bool use_smem = bytes <= static_cast<size_t>(kIntersectSmemBytes);
  if (use_smem && bytes > 48 * 1024)
    cudaFuncSetAttribute(intersect_walk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
  intersect_walk_kernel<<<static_cast<unsigned>(n_lists), 32 * d, use_smem ? bytes : 0, s>>>(
      d, off, xy, use_smem ? 1 : 0, bound, keep, centres, n_centres, counts);
  intersect_keep_kernel<<<static_cast<unsigned>(n_lists), 256, 0, s>>>(d, off, xy, bound, centres, n_centres, keep);
}

// ------------------------------------------------------------------------------------------
// synthetic pattern images (tools/render_synthetic_dataset.cc:202-291; the arithmetic is specified in
// include/b200ba.h). Every float and double operation that feeds a pixel is an explicit _rn intrinsic, so nvcc
// cannot contract it into a fused multiply-add; the library's global flags stay as they are.
// ------------------------------------------------------------------------------------------
// the float pose of one image: Rf (9, row-major), tf (3), then the inverse Rc (9), tc (3)
constexpr int kSynthPoseFloats = 24;
constexpr int kSynthClipCap = 20;  // Sutherland-Hodgman output of a 4-gon against 4 edges: at most 6, 9, 13, 19

// p_cam_i = ((R_i0 x + R_i1 y) + R_i2 z) + t_i (Eigen's 3 x 3 lazy product, then the translation)
__device__ __forceinline__ float synth_row(const float* r, float x, float y, float z) {
  return __fadd_rn(__fadd_rn(__fmul_rn(r[0], x), __fmul_rn(r[1], y)), __fmul_rn(r[2], z));
}

// the pixel range of one polygon, converted to int as x86-64 does (report_trunc) and clamped to the image
__device__ __forceinline__ int synth_lo(double v) { return max(0, report_trunc(v)); }
__device__ __forceinline__ int synth_hi(double v, int extent) { return min(extent - 1, report_trunc(v)); }

// One thread per (image, polygon): projects the vertices, stores the reference's clamped integer pixel range
// (x0, x1, y0, y1; empty when x0 > x1 or y0 > y1) and marks the polygon in the bitmap of every tile the range
// touches. Bit k of a tile's bitmap is polygon k, so a tile's polygons come out in generation order.
__global__ void synth_project_kernel(SynthParams p, int n_img, const float2* __restrict__ verts,
                                     const int8_t* __restrict__ nv, const float* __restrict__ poses,
                                     double2* __restrict__ proj, int4* __restrict__ range, uint32_t* bits) {
  const int64_t k = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (k >= static_cast<int64_t>(n_img) * p.n_poly) return;
  const int img = static_cast<int>(k / p.n_poly), poly = static_cast<int>(k % p.n_poly);
  const float* R = poses + static_cast<int64_t>(img) * kSynthPoseFloats;
  const float* t = R + 9;
  const int n = nv[poly];
  double min_x = 1.7976931348623157e308, min_y = 1.7976931348623157e308;
  double max_x = -1.7976931348623157e308, max_y = -1.7976931348623157e308;
  bool nan = false;
  for (int v = 0; v < n; ++v) {
    const float2 q = verts[poly * kSynthMaxVerts + v];
    const float X = __fadd_rn(synth_row(R, q.x, q.y, 0.f), t[0]);
    const float Y = __fadd_rn(synth_row(R + 3, q.x, q.y, 0.f), t[1]);
    const float Z = __fadd_rn(synth_row(R + 6, q.x, q.y, 0.f), t[2]);
    const double u = __fadd_rn(__fmul_rn(p.fx, __fdiv_rn(X, Z)), p.cx);
    const double w = __fadd_rn(__fmul_rn(p.fy, __fdiv_rn(Y, Z)), p.cy);
    proj[k * kSynthMaxVerts + v] = make_double2(u, w);
    nan |= u != u || w != w;
    min_x = u < min_x ? u : min_x;
    max_x = u > max_x ? u : max_x;
    min_y = w < min_y ? w : min_y;
    max_y = w > max_y ? w : max_y;
  }
  int4 r = make_int4(1, 0, 1, 0);  // empty
  if (!nan) r = make_int4(synth_lo(min_x), synth_hi(max_x, p.w), synth_lo(min_y), synth_hi(max_y, p.h));
  range[k] = r;
  if (r.x > r.y || r.z > r.w) return;
  uint32_t* b = bits + static_cast<int64_t>(img) * p.tiles_y * p.tiles_x * p.words + (poly >> 5);
  const uint32_t bit = 1u << (poly & 31);
  for (int ty = r.z / kSynthTile; ty <= r.w / kSynthTile; ++ty)
    for (int tx = r.x / kSynthTile; tx <= r.y / kSynthTile; ++tx)
      atomicOr(b + (static_cast<int64_t>(ty) * p.tiles_x + tx) * p.words, bit);
}

// libvis' LineLineIntersection (geometry.h:49-79) of the lines a0-a1 and b0-b1; *r is left alone only when the
// denominator is 0 (a non-finite quotient is stored before it is rejected)
__device__ __forceinline__ void synth_intersect(double2 a0, double2 a1, double2 b0, double2 b1, double2* r) {
  const double detL1 = __dsub_rn(__dmul_rn(a0.x, a1.y), __dmul_rn(a0.y, a1.x));
  const double detL2 = __dsub_rn(__dmul_rn(b0.x, b1.y), __dmul_rn(b0.y, b1.x));
  const double x1mx2 = __dsub_rn(a0.x, a1.x), x3mx4 = __dsub_rn(b0.x, b1.x);
  const double y1my2 = __dsub_rn(a0.y, a1.y), y3my4 = __dsub_rn(b0.y, b1.y);
  const double xnom = __dsub_rn(__dmul_rn(detL1, x3mx4), __dmul_rn(x1mx2, detL2));
  const double ynom = __dsub_rn(__dmul_rn(detL1, y3my4), __dmul_rn(y1my2, detL2));
  const double denom = __dsub_rn(__dmul_rn(x1mx2, y3my4), __dmul_rn(y1my2, x3mx4));
  if (denom == 0) return;
  r->x = __ddiv_rn(xnom, denom);
  r->y = __ddiv_rn(ynom, denom);
}

__device__ __forceinline__ double synth_dot(double2 a, double2 b) {
  return __dadd_rn(__dmul_rn(a.x, b.x), __dmul_rn(a.y, b.y));
}

// PolygonArea(ConvexClipPolygon(polygon, pixel square (x, y))) (geometry.h:147-207), in double with the float edge
// offset and the float orientation determinant of the reference
__device__ double synth_clip_area(const double2* __restrict__ poly, int n, int px, int py) {
  const double x = px, y = py;
  const double2 clip[4] = {make_double2(x, y), make_double2(__dadd_rn(x, 1.0), y),
                           make_double2(__dadd_rn(x, 1.0), __dadd_rn(y, 1.0)), make_double2(x, __dadd_rn(y, 1.0))};
  const float det = static_cast<float>(
      __dsub_rn(__dmul_rn(__dsub_rn(clip[1].x, clip[0].x), __dsub_rn(clip[2].y, clip[0].y)),
                __dmul_rn(__dsub_rn(clip[2].x, clip[0].x), __dsub_rn(clip[1].y, clip[0].y))));
  const int orientation = det > 0 ? 1 : -1;
  double2 buf[2][kSynthClipCap];
  const double2* in = poly;
  int n_in = n;
  for (int e = 0; e < 4; ++e) {
    const double2 s = clip[e], t = clip[(e + 1) & 3];
    const double2 right = make_double2(__dsub_rn(t.y, s.y), -__dsub_rn(t.x, s.x));
    const float edge_right = static_cast<float>(synth_dot(right, t));
    double2* out = buf[e & 1];
    int n_out = 0;
    for (int i = 0; i < n_in; ++i) {
      const double2 cur = in[i], prev = in[(i + n_in - 1) % n_in];
      const bool cur_in = orientation * (synth_dot(right, cur) > edge_right ? 1 : -1) < 0;
      if (cur_in) {
        if (orientation * (synth_dot(right, prev) > edge_right ? 1 : -1) > 0) {
          double2 r = prev;
          synth_intersect(prev, cur, t, s, &r);
          out[n_out++] = r;
        }
        out[n_out++] = cur;
      } else if (orientation * (synth_dot(right, prev) > edge_right ? 1 : -1) < 0) {
        double2 r = prev;
        synth_intersect(prev, cur, t, s, &r);
        out[n_out++] = r;
      }
    }
    in = out;
    n_in = n_out;
  }
  double sum = 0;
  for (int i = 0, j = n_in - 1; i < n_in; j = i++)
    sum = __dadd_rn(sum, __dmul_rn(__dsub_rn(in[i].x, in[j].x), __dadd_rn(in[i].y, in[j].y)));
  return fabs(__dmul_rn(0.5, sum));
}

// float -> u8 as x86-64 executes it: cvttss2si (truncation, INT_MIN outside the int range and for NaN), low byte
__device__ __forceinline__ uint8_t synth_u8(float v) {
  return static_cast<uint8_t>((v > -2147483649.f && v < 2147483648.f) ? static_cast<int>(v) : INT_MIN);
}

// One thread per pixel of a kSynthTile x kSynthTile tile: walks the tile's bitmap in polygon order, subtracts the
// clipped area of every polygon whose range holds the pixel, then composes the byte from the pixel's ray.
__global__ void __launch_bounds__(kSynthTile * kSynthTile, 3)
synth_render_kernel(SynthParams p, const float* __restrict__ poses, const int8_t* __restrict__ nv,
                    const double2* __restrict__ proj, const int4* __restrict__ range,
                    const uint32_t* __restrict__ bits, const uint8_t* __restrict__ pattern, uint8_t* images) {
  const int img = blockIdx.z;
  const int x = blockIdx.x * kSynthTile + threadIdx.x, y = blockIdx.y * kSynthTile + threadIdx.y;
  if (x >= p.w || y >= p.h) return;
  const uint32_t* b =
      bits + ((static_cast<int64_t>(img) * p.tiles_y + blockIdx.y) * p.tiles_x + blockIdx.x) * p.words;
  const int64_t pbase = static_cast<int64_t>(img) * p.n_poly;
  float rendering = 1.f;
  for (int wi = 0; wi < p.words; ++wi) {
    uint32_t m = b[wi];
    while (m) {
      const int poly = wi * 32 + __ffs(m) - 1;
      m &= m - 1;
      const int4 r = range[pbase + poly];
      if (x < r.x || x > r.y || y < r.z || y > r.w) continue;
      const double a = synth_clip_area(proj + (pbase + poly) * kSynthMaxVerts, nv[poly], x, y);
      rendering = __double2float_rn(__dsub_rn(static_cast<double>(rendering), a));
    }
  }
  // the ray of the pixel centre (UnprojectFromPixelCornerConv, then the inverse pose) meets the plane z = 0
  const float* Rc = poses + static_cast<int64_t>(img) * kSynthPoseFloats + 12;
  const float* tc = Rc + 9;
  const float lx = __fadd_rn(__fmul_rn(__fdiv_rn(1.f, p.fx), __fadd_rn(static_cast<float>(x), 0.5f)),
                             __fdiv_rn(-p.cx, p.fx));
  const float ly = __fadd_rn(__fmul_rn(__fdiv_rn(1.f, p.fy), __fadd_rn(static_cast<float>(y), 0.5f)),
                             __fdiv_rn(-p.cy, p.fy));
  float dx = synth_row(Rc, lx, ly, 1.f), dy = synth_row(Rc + 3, lx, ly, 1.f), dz = synth_row(Rc + 6, lx, ly, 1.f);
  const float n2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
  if (n2 > 0.f) {
    const float s = __fsqrt_rn(n2);
    dx = __fdiv_rn(dx, s);
    dy = __fdiv_rn(dy, s);
    dz = __fdiv_rn(dz, s);
  }
  const float offset = -0.f;
  const float num = __fadd_rn(offset, __fadd_rn(__fadd_rn(__fmul_rn(0.f, tc[0]), __fmul_rn(0.f, tc[1])),
                                                __fmul_rn(-1.f, tc[2])));
  const float den = __fadd_rn(__fadd_rn(__fmul_rn(0.f, dx), __fmul_rn(0.f, dy)), __fmul_rn(-1.f, dz));
  const float tt = __fdiv_rn(-num, den);
  const float X = __fadd_rn(tc[0], __fmul_rn(dx, tt)), Y = __fadd_rn(tc[1], __fmul_rn(dy, tt));
  const float lx2 = __fsub_rn(X, 0.f), ly2 = __fsub_rn(Y, -0.f);
  const float ix = __fadd_rn(__fmul_rn(1.f, lx2), __fmul_rn(0.f, ly2));
  const float iy = __fadd_rn(__fmul_rn(0.f, lx2), __fmul_rn(1.f, ly2));
  const float mx = __fmul_rn(__fdiv_rn(p.page_w, static_cast<float>(p.pattern_w)), ix);
  const float my = __fmul_rn(__fdiv_rn(p.page_h, static_cast<float>(p.pattern_h)), iy);
  const float cx = __fsub_rn(__fmul_rn(__fdiv_rn(__fsub_rn(mx, p.start_x), __fsub_rn(p.end_x, p.start_x)),
                                       static_cast<float>(p.squares_x)), 1.f);
  const float cy = __fsub_rn(__fmul_rn(__fdiv_rn(__fsub_rn(my, p.start_y), __fsub_rn(p.end_y, p.start_y)),
                                       static_cast<float>(p.squares_y)), 1.f);
  bool valid = cx >= -1.f && cy >= -1.f && cx <= static_cast<float>(p.squares_x) - 1.f &&
               cy <= static_cast<float>(p.squares_y) - 1.f;
  for (int k = 0; valid && k < p.num_tags; ++k) {
    const int4 tg = p.tags[k];
    if (cx >= static_cast<float>(tg.x - 1) && cy >= static_cast<float>(tg.y - 1) &&
        cx <= static_cast<float>(tg.x - 1 + tg.z) && cy <= static_cast<float>(tg.y - 1 + tg.w))
      valid = false;
  }
  uint8_t out = 0;
  if (valid) {
    const float v = __fmul_rn(255.99f, rendering);
    out = synth_u8(0.f < v ? v : 0.f);  // std::max<float>(0.f, v): NaN gives 0.f
  } else {
    const float qx = __fsub_rn(ix, 0.5f), qy = __fsub_rn(iy, 0.5f);
    if (qx >= 0.f && qy >= 0.f && qx < static_cast<float>(p.pattern_w - 1) &&
        qy < static_cast<float>(p.pattern_h - 1)) {
      const int jx = static_cast<int>(qx), jy = static_cast<int>(qy);
      const float fx = __fsub_rn(qx, static_cast<float>(jx)), fy = __fsub_rn(qy, static_cast<float>(jy));
      const float gx = __fsub_rn(1.f, fx), gy = __fsub_rn(1.f, fy);
      const uint8_t* row = pattern + static_cast<int64_t>(jy) * p.pattern_w + jx;
      const float v = __fadd_rn(
          __fadd_rn(__fadd_rn(__fmul_rn(__fmul_rn(gx, gy), static_cast<float>(row[0])),
                              __fmul_rn(__fmul_rn(fx, gy), static_cast<float>(row[1]))),
                    __fmul_rn(__fmul_rn(gx, fy), static_cast<float>(row[p.pattern_w]))),
          __fmul_rn(__fmul_rn(fx, fy), static_cast<float>(row[p.pattern_w + 1])));
      out = synth_u8(v);
    }
  }
  images[(static_cast<int64_t>(img) * p.h + y) * p.w + x] = out;
}

void launch_render_pattern(const SynthParams& p, int n_img, const float2* verts, const int8_t* nv, const float* poses,
                           const uint8_t* pattern, double2* proj, int4* range, uint32_t* bits, uint8_t* images,
                           cudaStream_t s) {
  if (n_img == 0) return;
  const int64_t n = static_cast<int64_t>(n_img) * p.n_poly;
  if (n > 0)
    synth_project_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(p, n_img, verts, nv, poses, proj,
                                                                               range, bits);
  synth_render_kernel<<<dim3(p.tiles_x, p.tiles_y, n_img), dim3(kSynthTile, kSynthTile), 0, s>>>(
      p, poses, nv, proj, range, bits, pattern, images);
}

// ------------------------------------------------------------------------------------------
// sub-pixel refinement of star-pattern features (feature_detector_tagged_pattern.cc:1427-1648 with the CPU path of
// cpu_refinement_by_matching.h and cpu_refinement_by_symmetry.h; the arithmetic is specified in include/b200ba.h).
// One warp per feature: lane l takes samples l, l + 32, ... in order and the sums are combined by an xor butterfly,
// so every lane holds the same bits and every LM decision is warp-uniform. The arithmetic goes through the _rn
// helpers of ba_common.h, which tests/refine_features_oracle.cc compiles too; nothing is contracted.
// ------------------------------------------------------------------------------------------
constexpr int kRefineWarps = 4;

__device__ __forceinline__ float refine_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = rf_add(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Image::ContainsPixelCenterConv
__device__ __forceinline__ bool refine_inside(const RefineParams& p, float x, float y) {
  return x >= 0.f && y >= 0.f && x < static_cast<float>(p.w - 1) && y < static_cast<float>(p.h - 1);
}

// hnorm(M (x, y, 1)), rows ((m0 x + m1 y) + m2)
__device__ __forceinline__ float2 refine_hnorm(const float* m, float x, float y) {
  const float u = rf_add(rf_add(rf_mul(m[0], x), rf_mul(m[1], y)), m[2]);
  const float v = rf_add(rf_add(rf_mul(m[3], x), rf_mul(m[4], y)), m[5]);
  const float w = rf_add(rf_add(rf_mul(m[6], x), rf_mul(m[7], y)), m[8]);
  return make_float2(rf_div(u, w), rf_div(v, w));
}

// PatternData::IsValidPatternCoord
__device__ __forceinline__ bool refine_valid_pattern(const RefineParams& p, float x, float y) {
  if (!(x >= -1.f && y >= -1.f && x <= rf_sub(static_cast<float>(p.squares_x), 1.f) &&
        y <= rf_sub(static_cast<float>(p.squares_y), 1.f)))
    return false;
  for (int k = 0; k < p.num_tags; ++k) {
    const int4 t = p.tags[k];
    if (x >= static_cast<float>(t.x - 1) && y >= static_cast<float>(t.y - 1) &&
        x <= static_cast<float>(t.x - 1 + t.z) && y <= static_cast<float>(t.y - 1 + t.w))
      return false;
  }
  return true;
}

// the gradient image's pixel (x, y) (feature_detector_tagged_pattern.cc:273-287), from the u8 bytes
__device__ __forceinline__ float2 refine_gradient(const uint8_t* __restrict__ im, int w, int h, int x, int y) {
  const int mx = max(0, x - 1), px = min(w - 1, x + 1), my = max(0, y - 1), py = min(h - 1, y + 1);
  const uint8_t* row = im + static_cast<int64_t>(y) * w;
  const float dx = rf_div(rf_sub(static_cast<float>(__ldg(row + px)), static_cast<float>(__ldg(row + mx))),
                          static_cast<float>(px - mx));
  const float dy = rf_div(rf_sub(static_cast<float>(__ldg(im + static_cast<int64_t>(py) * w + x)),
                                 static_cast<float>(__ldg(im + static_cast<int64_t>(my) * w + x))),
                          static_cast<float>(py - my));
  return make_float2(dx, dy);
}

// the four corners (x, y), (x + 1, y), (x, y + 1), (x + 1, y + 1) of channel 0 (and 1) of the image of kType:
// the u8 image (INTENSITIES, and matching), the gradient magnitude or the gradient (GRADIENTS_XY)
template <int kType>
__device__ __forceinline__ void refine_corners(const uint8_t* __restrict__ im, const RefineParams& p, int x, int y,
                                               float* c0, float* c1) {
  if (kType == B200BA_REFINE_INTENSITIES) {
    const uint8_t* row = im + static_cast<int64_t>(y) * p.w + x;
    c0[0] = __ldg(row);
    c0[1] = __ldg(row + 1);
    c0[2] = __ldg(row + p.w);
    c0[3] = __ldg(row + p.w + 1);
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 g = refine_gradient(im, p.w, p.h, x + (k & 1), y + (k >> 1));
      if (kType == B200BA_REFINE_GRADIENT_MAGNITUDE) {
        c0[k] = __fsqrt_rn(rf_add(rf_mul(g.x, g.x), rf_mul(g.y, g.y)));
      } else {
        c0[k] = g.x;
        c1[k] = g.y;
      }
    }
  }
}

// InterpolateBilinear: (((gx gy) c00 + (fx gy) c10) + (gx fy) c01) + (fx fy) c11
__device__ __forceinline__ float refine_value(float fx, float fy, const float* c) {
  const float gx = rf_sub(1.f, fx), gy = rf_sub(1.f, fy);
  return rf_add(rf_add(rf_add(rf_mul(rf_mul(gx, gy), c[0]), rf_mul(rf_mul(fx, gy), c[1])),
                       rf_mul(rf_mul(gx, fy), c[2])),
                rf_mul(rf_mul(fx, fy), c[3]));
}

// InterpolateBilinearWithJacobian: the value and (d/dx, d/dy)
__device__ __forceinline__ float refine_value_jac(float fx, float fy, const float* c, float* dx, float* dy) {
  const float gx = rf_sub(1.f, fx), gy = rf_sub(1.f, fy);
  const float top = rf_add(rf_mul(gx, c[0]), rf_mul(fx, c[1]));
  const float bottom = rf_add(rf_mul(gx, c[2]), rf_mul(fx, c[3]));
  *dx = rf_add(rf_mul(fy, rf_sub(c[3], c[2])), rf_mul(gy, rf_sub(c[1], c[0])));
  *dy = rf_sub(bottom, top);
  return rf_add(rf_mul(gy, top), rf_mul(fy, bottom));
}

// matching: the sum of squared residuals at (x, y, factor, bias); false when a sample leaves the image
__device__ __forceinline__ bool refine_match_cost(const RefineParams& p, const uint8_t* __restrict__ im,
                                                  const float2* __restrict__ samples, const float* tmpl, int lane,
                                                  float x, float y, float factor, float bias, float* cost) {
  const float h = static_cast<float>(p.half);
  float c = 0.f;
  bool out = false;
  for (int i = lane; i < p.n_match; i += 32) {
    const float2 s = __ldg(samples + i);
    const float sx = rf_add(x, rf_mul(h, s.x)), sy = rf_add(y, rf_mul(h, s.y));
    if (!refine_inside(p, sx, sy)) {
      out = true;
      break;
    }
    const int ix = static_cast<int>(sx), iy = static_cast<int>(sy);
    float cr[4];
    refine_corners<B200BA_REFINE_INTENSITIES>(im, p, ix, iy, cr, nullptr);
    const float v = refine_value(rf_sub(sx, static_cast<float>(ix)), rf_sub(sy, static_cast<float>(iy)), cr);
    const float r = rf_sub(rf_add(rf_mul(factor, v), bias), tmpl[i]);
    c = rf_add(c, rf_mul(r, r));
  }
  if (__any_sync(0xffffffffu, out)) return false;
  *cost = refine_warp_sum(c);
  return true;
}

// symmetry: the pixel positions of +-t under P
__device__ __forceinline__ void refine_sym_positions(const float* P, float tx, float ty, float2* a, float2* b) {
  *a = refine_hnorm(P, tx, ty);
  *b = refine_hnorm(P, -tx, -ty);
}

// d hnorm(P (t, 1)) / d(P00 P01 P02 P10 P11 P12 P20 P21) (cpu_refinement_by_symmetry.h:334-353), rows D[0..7], D[8..15]
__device__ __forceinline__ void refine_dpos(const float* P, float tx, float ty, float* D) {
  const float e0 = rf_div(1.f, rf_add(rf_add(rf_mul(P[6], tx), rf_mul(P[7], ty)), 1.f));
  const float e1 = rf_mul(rf_mul(-1.f, e0), e0);
  const float e2 = rf_mul(rf_add(rf_add(rf_mul(P[0], tx), rf_mul(P[1], ty)), P[2]), e1);
  const float e3 = rf_mul(rf_add(rf_add(rf_mul(P[3], tx), rf_mul(P[4], ty)), P[5]), e1);
  D[0] = rf_mul(tx, e0), D[1] = rf_mul(ty, e0), D[2] = e0, D[3] = 0.f, D[4] = 0.f, D[5] = 0.f;
  D[6] = rf_mul(tx, e2), D[7] = rf_mul(ty, e2);
  D[8] = 0.f, D[9] = 0.f, D[10] = 0.f, D[11] = D[0], D[12] = D[1], D[13] = D[2];
  D[14] = rf_mul(tx, e3), D[15] = rf_mul(ty, e3);
}

// symmetry: the pattern-space sample t_i = hnorm(M ((float)h s_i, 1))
__device__ __forceinline__ float2 refine_pattern_sample(const float* M, float h, float2 s) {
  return refine_hnorm(M, rf_mul(h, s.x), rf_mul(h, s.y));
}

// symmetry: the cost at P (ComputeCornerRefinementCost); false when a sample leaves the image
template <int kType>
__device__ __forceinline__ bool refine_sym_cost(const RefineParams& p, const uint8_t* __restrict__ im,
                                                const float2* __restrict__ samples, const float* M, const float* P,
                                                int lane, float* cost) {
  const float h = static_cast<float>(p.half);
  float c = 0.f;
  bool out = false;
  for (int i = lane; i < p.n_samples; i += 32) {
    const float2 t = refine_pattern_sample(M, h, __ldg(samples + i));
    float2 pa, pb;
    refine_sym_positions(P, t.x, t.y, &pa, &pb);
    if (!refine_inside(p, pa.x, pa.y) || !refine_inside(p, pb.x, pb.y)) {
      out = true;
      break;
    }
    float a0[4], a1[4], b0[4], b1[4];
    const int ax = static_cast<int>(pa.x), ay = static_cast<int>(pa.y);
    const int bx = static_cast<int>(pb.x), by = static_cast<int>(pb.y);
    refine_corners<kType>(im, p, ax, ay, a0, a1);
    refine_corners<kType>(im, p, bx, by, b0, b1);
    const float fax = rf_sub(pa.x, static_cast<float>(ax)), fay = rf_sub(pa.y, static_cast<float>(ay));
    const float fbx = rf_sub(pb.x, static_cast<float>(bx)), fby = rf_sub(pb.y, static_cast<float>(by));
    if (kType == B200BA_REFINE_GRADIENTS_XY) {
      const float r0 = rf_add(refine_value(fax, fay, a0), refine_value(fbx, fby, b0));
      const float r1 = rf_add(refine_value(fax, fay, a1), refine_value(fbx, fby, b1));
      c = rf_add(c, rf_add(rf_mul(r0, r0), rf_mul(r1, r1)));
    } else {
      const float r = rf_sub(refine_value(fax, fay, a0), refine_value(fbx, fby, b0));
      c = rf_add(c, rf_mul(r, r));
    }
  }
  if (__any_sync(0xffffffffu, out)) return false;
  *cost = refine_warp_sum(c);
  return true;
}

// symmetry: H (packed upper 8 x 8, 36), b (8) and the cost at P (ComputeCornerRefinementCostAndJacobian)
template <int kType>
__device__ __forceinline__ bool refine_sym_system(const RefineParams& p, const uint8_t* __restrict__ im,
                                                  const float2* __restrict__ samples, const float* M, const float* P,
                                                  int lane, float* H, float* b, float* cost) {
  const float h = static_cast<float>(p.half);
#pragma unroll
  for (int k = 0; k < 36; ++k) H[k] = 0.f;
#pragma unroll
  for (int k = 0; k < 8; ++k) b[k] = 0.f;
  float c = 0.f;
  bool out = false;
  for (int i = lane; i < p.n_samples; i += 32) {
    const float2 t = refine_pattern_sample(M, h, __ldg(samples + i));
    float2 pa, pb;
    refine_sym_positions(P, t.x, t.y, &pa, &pb);
    if (!refine_inside(p, pa.x, pa.y) || !refine_inside(p, pb.x, pb.y)) {
      out = true;
      break;
    }
    float a0[4], a1[4], b0[4], b1[4];
    const int ax = static_cast<int>(pa.x), ay = static_cast<int>(pa.y);
    const int bx = static_cast<int>(pb.x), by = static_cast<int>(pb.y);
    refine_corners<kType>(im, p, ax, ay, a0, a1);
    refine_corners<kType>(im, p, bx, by, b0, b1);
    const float fax = rf_sub(pa.x, static_cast<float>(ax)), fay = rf_sub(pa.y, static_cast<float>(ay));
    const float fbx = rf_sub(pb.x, static_cast<float>(bx)), fby = rf_sub(pb.y, static_cast<float>(by));
    float Da[16], Db[16];
    refine_dpos(P, t.x, t.y, Da);
    refine_dpos(P, -t.x, -t.y, Db);
    if (kType == B200BA_REFINE_GRADIENTS_XY) {
      float ga[4], gb[4];  // (channel 0 d/dx, d/dy, channel 1 d/dx, d/dy)
      const float va0 = refine_value_jac(fax, fay, a0, &ga[0], &ga[1]);
      const float va1 = refine_value_jac(fax, fay, a1, &ga[2], &ga[3]);
      const float vb0 = refine_value_jac(fbx, fby, b0, &gb[0], &gb[1]);
      const float vb1 = refine_value_jac(fbx, fby, b1, &gb[2], &gb[3]);
      const float r[2] = {rf_add(va0, vb0), rf_add(va1, vb1)};
#pragma unroll
      for (int row = 0; row < 2; ++row) {
        float J[8];
#pragma unroll
        for (int k = 0; k < 8; ++k)
          J[k] = rf_add(rf_add(rf_mul(ga[2 * row], Da[k]), rf_mul(ga[2 * row + 1], Da[8 + k])),
                        rf_add(rf_mul(gb[2 * row], Db[k]), rf_mul(gb[2 * row + 1], Db[8 + k])));
        int q = 0;
#pragma unroll
        for (int u = 0; u < 8; ++u)
#pragma unroll
          for (int v = u; v < 8; ++v, ++q) H[q] = rf_add(H[q], rf_mul(J[u], J[v]));
#pragma unroll
        for (int u = 0; u < 8; ++u) b[u] = rf_add(b[u], rf_mul(r[row], J[u]));
      }
      c = rf_add(c, rf_add(rf_mul(r[0], r[0]), rf_mul(r[1], r[1])));
    } else {
      float gax, gay, gbx, gby;
      const float va = refine_value_jac(fax, fay, a0, &gax, &gay);
      const float vb = refine_value_jac(fbx, fby, b0, &gbx, &gby);
      const float r = rf_sub(va, vb);
      float J[8];
#pragma unroll
      for (int k = 0; k < 8; ++k)
        J[k] = rf_sub(rf_add(rf_mul(gax, Da[k]), rf_mul(gay, Da[8 + k])),
                      rf_add(rf_mul(gbx, Db[k]), rf_mul(gby, Db[8 + k])));
      int q = 0;
#pragma unroll
      for (int u = 0; u < 8; ++u)
#pragma unroll
        for (int v = u; v < 8; ++v, ++q) H[q] = rf_add(H[q], rf_mul(J[u], J[v]));
#pragma unroll
      for (int u = 0; u < 8; ++u) b[u] = rf_add(b[u], rf_mul(r, J[u]));
      c = rf_add(c, rf_mul(r, r));
    }
  }
  if (__any_sync(0xffffffffu, out)) return false;
#pragma unroll
  for (int k = 0; k < 36; ++k) H[k] = refine_warp_sum(H[k]);
#pragma unroll
  for (int k = 0; k < 8; ++k) b[k] = refine_warp_sum(b[k]);
  *cost = refine_warp_sum(c);
  return true;
}

// RefineFeatureBySymmetry from the matching result m; returns the status and sets *pos and *final_cost
template <int kType>
__device__ __forceinline__ int refine_symmetry(const RefineParams& p, const uint8_t* __restrict__ im,
                                            const float2* __restrict__ samples, const float* M, const float* L,
                                            float mx, float my, float2* pos, float* final_cost) {
  const int lane = threadIdx.x & 31;
  float P[9];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    P[c] = rf_add(rf_add(rf_mul(1.f, L[c]), rf_mul(0.f, L[3 + c])), rf_mul(mx, L[6 + c]));
    P[3 + c] = rf_add(rf_add(rf_mul(0.f, L[c]), rf_mul(1.f, L[3 + c])), rf_mul(my, L[6 + c]));
    P[6 + c] = rf_add(rf_add(rf_mul(0.f, L[c]), rf_mul(0.f, L[3 + c])), rf_mul(1.f, L[6 + c]));
  }
  const float p22 = P[8];
#pragma unroll
  for (int k = 0; k < 9; ++k) P[k] = rf_div(P[k], p22);
  const float h = static_cast<float>(p.half);
  float lambda = -1.f, last = __int_as_float(0x7f800000), cost = 0.f;
  *pos = make_float2(mx, my);
  for (int iteration = 0; iteration < 30; ++iteration) {
    float H[36], b[8];
    if (!refine_sym_system<kType>(p, im, samples, M, P, lane, H, b, &cost)) return B200BA_REFINE_SYM_OUTSIDE;
    if (lambda < 0.f) {
      float d = H[0];
      for (int k = 1, q = 8; k < 8; q += 8 - k, ++k) d = rf_add(d, H[q]);
      lambda = rf_mul(rf_mul(0.001f, rf_div(1.f, 8.f)), d);
    }
    bool applied = false;
    for (int attempt = 0; attempt < 10; ++attempt) {
      float x[8];
      rf_ldlt_solve<8>(H, lambda, b, x);
      float T[9];
#pragma unroll
      for (int k = 0; k < 8; ++k) T[k] = rf_sub(P[k], x[k]);
      T[8] = P[8];
      float test_cost;
      if (!refine_sym_cost<kType>(p, im, samples, M, T, lane, &test_cost)) return B200BA_REFINE_SYM_OUTSIDE;
      if (test_cost < cost) {
        cost = test_cost;
        last = rf_add(rf_mul(x[2], x[2]), rf_mul(x[5], x[5]));
#pragma unroll
        for (int k = 0; k < 9; ++k) P[k] = T[k];
        lambda = rf_mul(lambda, 0.5f);
        applied = true;
        break;
      }
      lambda = rf_mul(lambda, 2.f);
    }
    *final_cost = cost;
    if (!applied) return B200BA_REFINE_ACCEPTED;
    *pos = make_float2(P[2], P[5]);
    if (fabsf(rf_sub(mx, P[2])) >= h || fabsf(rf_sub(my, P[5])) >= h) return B200BA_REFINE_SYM_LEFT_WINDOW;
  }
  return last < 1e-4f ? B200BA_REFINE_ACCEPTED : B200BA_REFINE_SYM_NOT_CONVERGED;
}

// kType: the refinement type (B200BA_REFINE_*)
template <int kType>
__global__ void __launch_bounds__(kRefineWarps * 32)
refine_features_kernel(RefineParams p, int64_t n, const b200ba_feature_prediction* __restrict__ pred,
                       const uint8_t* __restrict__ images, const float2* __restrict__ samples, float2* xy,
                       float* cost_out, int* status_out) {
  extern __shared__ float refine_templates[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t f = static_cast<int64_t>(blockIdx.x) * kRefineWarps + warp;
  if (f >= n) return;
  float* tmpl = refine_templates + warp * p.n_match;
  const b200ba_feature_prediction& pr = pred[f];
  const uint8_t* im = images + pr.image * static_cast<int64_t>(p.w) * p.h;
  const float h = static_cast<float>(p.half);
  const float x0 = pr.position[0], y0 = pr.position[1];
  float L[9], M[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) L[k] = pr.local_pixel_tr_pattern[k];
  rf_inverse3(L, M);
  int st = B200BA_REFINE_ACCEPTED;
  float final_cost = 0.f;
  float2 pos = make_float2(x0, y0);
  // pre-filter (:1443-1479)
  if (!(rf_sub(x0, h) >= 0.f && rf_sub(y0, h) >= 0.f && rf_add(x0, h) < static_cast<float>(p.w - 1) &&
        rf_add(y0, h) < static_cast<float>(p.h - 1))) {
    st = B200BA_REFINE_IMAGE_BORDER;
  } else {
    for (int corner = 0; corner < 4; ++corner) {
      const float2 o = refine_hnorm(M, corner % 2 == 0 ? h : -h, corner / 2 == 0 ? h : -h);
      if (!refine_valid_pattern(p, rf_add(static_cast<float>(pr.pattern_coordinate[0]), o.x),
                                rf_add(static_cast<float>(pr.pattern_coordinate[1]), o.y))) {
        st = B200BA_REFINE_OUTSIDE_PATTERN;
        break;
      }
    }
  }
  float mx = x0, my = y0;
  if (st == B200BA_REFINE_ACCEPTED) {
    // the template (cpu_refinement_by_matching.h:247-261)
    for (int i = lane; i < p.n_match; i += 32) {
      const float2 s = __ldg(samples + i);
      const float ox = rf_mul(h, s.x), oy = rf_mul(h, s.y);
      float sum = 0.f;
      for (int k = 0; k < 16; ++k) {
        const float2 q = refine_hnorm(M, rf_add(ox, -0.375f + 0.25f * (k % 4)), rf_add(oy, -0.375f + 0.25f * (k / 4)));
        sum = rf_add(sum, rf_pattern_intensity(p.num_star_segments, q.x, q.y));
      }
      tmpl[i] = sum;
    }
    __syncwarp();
    // factor and bias (:76-114)
    float s_qp = 0.f, s_p = 0.f, s_q = 0.f, s_pp = 0.f;
    bool out = false;
    for (int i = lane; i < p.n_match; i += 32) {
      const float2 s = __ldg(samples + i);
      const float sx = rf_add(x0, rf_mul(h, s.x)), sy = rf_add(y0, rf_mul(h, s.y));
      if (!refine_inside(p, sx, sy)) {
        out = true;
        break;
      }
      const int ix = static_cast<int>(sx), iy = static_cast<int>(sy);
      float cr[4];
      refine_corners<B200BA_REFINE_INTENSITIES>(im, p, ix, iy, cr, nullptr);
      const float v = refine_value(rf_sub(sx, static_cast<float>(ix)), rf_sub(sy, static_cast<float>(iy)), cr);
      const float q = tmpl[i];
      s_qp = rf_add(s_qp, rf_mul(q, v));
      s_p = rf_add(s_p, v);
      s_q = rf_add(s_q, q);
      s_pp = rf_add(s_pp, rf_mul(v, v));
    }
    if (__any_sync(0xffffffffu, out)) st = B200BA_REFINE_MATCH_OUTSIDE;
    s_qp = refine_warp_sum(s_qp);
    s_p = refine_warp_sum(s_p);
    s_q = refine_warp_sum(s_q);
    s_pp = refine_warp_sum(s_pp);
    const float nm = static_cast<float>(p.n_match);
    const float den = rf_sub(s_pp, rf_div(rf_mul(s_p, s_p), nm));
    float factor = fabsf(den) > 1e-6f ? rf_div(rf_sub(s_qp, rf_mul(rf_div(s_p, nm), s_q)), den) : 1.f;
    float bias = rf_mul(rf_div(1.f, nm), rf_sub(s_q, rf_mul(factor, s_p)));
    // LM on (x, y, factor, bias) (:306-417)
    float lambda = -1.f, last = __int_as_float(0x7f800000);
    bool converged = false;
    for (int iteration = 0; iteration < 50 && st == B200BA_REFINE_ACCEPTED; ++iteration) {
      float H[10], b[4], cost = 0.f;
#pragma unroll
      for (int k = 0; k < 10; ++k) H[k] = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) b[k] = 0.f;
      for (int i = lane; i < p.n_match; i += 32) {
        const float2 s = __ldg(samples + i);
        const float sx = rf_add(mx, rf_mul(h, s.x)), sy = rf_add(my, rf_mul(h, s.y));
        if (!refine_inside(p, sx, sy)) {
          out = true;
          break;
        }
        const int ix = static_cast<int>(sx), iy = static_cast<int>(sy);
        float cr[4], gx, gy;
        refine_corners<B200BA_REFINE_INTENSITIES>(im, p, ix, iy, cr, nullptr);
        const float v = refine_value_jac(rf_sub(sx, static_cast<float>(ix)), rf_sub(sy, static_cast<float>(iy)), cr,
                                         &gx, &gy);
        const float r = rf_sub(rf_add(rf_mul(factor, v), bias), tmpl[i]);
        const float J[4] = {rf_mul(factor, gx), rf_mul(factor, gy), v, 1.f};
        int q = 0;
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
          for (int w = u; w < 4; ++w, ++q) H[q] = rf_add(H[q], rf_mul(J[u], J[w]));
#pragma unroll
        for (int u = 0; u < 4; ++u) b[u] = rf_add(b[u], rf_mul(r, J[u]));
        cost = rf_add(cost, rf_mul(r, r));
      }
      if (__any_sync(0xffffffffu, out)) {
        st = B200BA_REFINE_MATCH_OUTSIDE;
        break;
      }
#pragma unroll
      for (int k = 0; k < 10; ++k) H[k] = refine_warp_sum(H[k]);
#pragma unroll
      for (int k = 0; k < 4; ++k) b[k] = refine_warp_sum(b[k]);
      cost = refine_warp_sum(cost);
      if (lambda < 0.f) lambda = rf_mul(rf_mul(0.001f, 0.5f), rf_add(rf_add(rf_add(H[0], H[4]), H[7]), H[9]));
      bool applied = false;
      for (int attempt = 0; attempt < 10; ++attempt) {
        float x[4];
        rf_ldlt_solve<4>(H, lambda, b, x);
        const float tx = rf_sub(mx, x[0]), ty = rf_sub(my, x[1]);
        const float tf = rf_sub(factor, x[2]), tb = rf_sub(bias, x[3]);
        float test_cost;
        if (!refine_match_cost(p, im, samples, tmpl, lane, tx, ty, tf, tb, &test_cost)) {
          st = B200BA_REFINE_MATCH_OUTSIDE;
          break;
        }
        if (test_cost < cost) {
          last = rf_add(rf_add(rf_add(rf_mul(x[0], x[0]), rf_mul(x[1], x[1])), rf_mul(x[2], x[2])),
                        rf_mul(x[3], x[3]));
          mx = tx, my = ty, factor = tf, bias = tb;
          lambda = rf_mul(lambda, 0.5f);
          applied = true;
          break;
        }
        lambda = rf_mul(lambda, 2.f);
      }
      if (st != B200BA_REFINE_ACCEPTED) break;
      if (!applied) {
        converged = true;
        break;
      }
      if (fabsf(rf_sub(x0, mx)) >= h || fabsf(rf_sub(y0, my)) >= h) st = B200BA_REFINE_MATCH_LEFT_WINDOW;
    }
    if (st == B200BA_REFINE_ACCEPTED) {
      if (static_cast<double>(last) < 1e-8) converged = true;
      if (!converged)
        st = B200BA_REFINE_MATCH_NOT_CONVERGED;
      else if (factor <= 0.f)
        st = B200BA_REFINE_MATCH_BAD_FACTOR;
    }
    pos = make_float2(mx, my);
  }
  if (kType != B200BA_REFINE_NO_REFINEMENT && st == B200BA_REFINE_ACCEPTED) {
    st = refine_symmetry<kType>(p, im, samples, M, L, mx, my, &pos, &final_cost);
    // :1626-1647
    const float dx = rf_sub(pos.x, mx), dy = rf_sub(pos.y, my);
    if (st == B200BA_REFINE_ACCEPTED && rf_add(rf_mul(dx, dx), rf_mul(dy, dy)) > 0.75f) st = B200BA_REFINE_INCONSISTENT;
  }
  if (lane == 0) {
    const bool ok = st == B200BA_REFINE_ACCEPTED;
    xy[f] = ok ? pos : make_float2(__int_as_float(0x7fc00000), __int_as_float(0x7fc00000));
    cost_out[f] = ok ? final_cost : -1.f;
    status_out[f] = st;
  }
}

void launch_refine_features(const RefineParams& p, int64_t n, const b200ba_feature_prediction* pred,
                            const uint8_t* images, const float2* samples, float2* xy, float* cost, int* status,
                            cudaStream_t s) {
  if (n == 0) return;
  const size_t smem = sizeof(float) * kRefineWarps * p.n_match;
  const unsigned blocks = static_cast<unsigned>((n + kRefineWarps - 1) / kRefineWarps);
  auto run = [&](auto kernel) {
    if (smem > 48 * 1024)
      cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    kernel<<<blocks, kRefineWarps * 32, smem, s>>>(p, n, pred, images, samples, xy, cost, status);
  };
  switch (p.type) {
    case B200BA_REFINE_GRADIENTS_XY: run(refine_features_kernel<B200BA_REFINE_GRADIENTS_XY>); break;
    case B200BA_REFINE_GRADIENT_MAGNITUDE: run(refine_features_kernel<B200BA_REFINE_GRADIENT_MAGNITUDE>); break;
    case B200BA_REFINE_INTENSITIES: run(refine_features_kernel<B200BA_REFINE_INTENSITIES>); break;
    default: run(refine_features_kernel<B200BA_REFINE_NO_REFINEMENT>); break;
  }
}

}  // namespace b200ba
