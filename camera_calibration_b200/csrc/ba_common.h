// ba_common.h -- structures shared by the host logic (ba_host.cu) and the kernels
// (ba_kernels.cu) of libb200ba.so. Not part of the public ABI (that is include/b200ba.h).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "../../include/b200ba.h"

namespace b200ba {

constexpr int kMaxCameras = 8;
constexpr int kMaxK = 80;  // IntrinsicsJacobianSize of the non-central model

// Device view of one camera (CameraModel base members + derived constants).
struct CamDev {
  int model_type;
  int width, height;
  int min_x, min_y, max_x, max_y;
  int gw, gh;
  // pixel -> grid map  g = 1 + gmul * (x - min)     (central_grid.h:150-154)
  double gmul_x, gmul_y;
  // PixelScaleToGridScaleX/Y: computed in FLOAT in the reference (central_grid.h:156-161)
  double sx, sy;
  // CenterOfCalibratedArea (camera_model.h:154-157)
  double center_x, center_y;
  int K;              // IntrinsicsJacobianSize: 32 / 80 / 12
  int dof_per_point;  // 2 / 5 / 0
  int64_t intr_off;   // offset of this camera's flat intrinsics in the state's intrinsics buffer
  int64_t tan_off;    // offset of its tangent frames (6 doubles per control point)
  int upd_off;        // offset of its update parameters relative to first_intrinsics
  int upd_count;      // update_parameter_count()
};

// Variable layout of JointOptimizationState (joint_optimization.cc:49-59,97-170) and of the
// block-diagonal / dense split of H (lm_optimizer.h:657-685):
//   eliminate_points:  [points 3P | rig_tr_global 6N | camera_tr_rig 6C (iff C > 1) | intrinsics]
//                      block part = points (3x3 blocks)
//   otherwise:         [rig_tr_global 6N | camera_tr_rig 6C (iff C > 1) | points 3P | intrinsics]
//                      block part = imageset poses (6x6 blocks)
// g_* are offsets in that global ordering; a dense index is (global - nbd).
struct Layout {
  int n_points, n_imagesets, n_cameras;
  int rig_in_state;     // n_cameras > 1
  int localize_only;
  int eliminate_points;
  int dof;              // all unknowns
  int bs;               // Schur block size: 3 (points) or 6 (poses)
  int nblocks;          // number of blocks: P or N
  int dsz;              // packed upper-triangle size of a block: bs (bs + 1) / 2
  int nbd;              // bs * nblocks (block-diagonal part)
  int nd;               // dense part
  int g_point, g_pose, g_rig, g_intr;  // global offsets of the variable groups
  int n_jcols;          // Jacobian columns stored per observation: 3 + 6 + (rig ? 6 : 0) + Kmax
  int Kmax;             // max IntrinsicsJacobianSize over cameras (0 when localize_only)
  int jc_point, jc_pose, jc_rig, jc_intr;  // first storage column of each part
};

struct ProblemDev {
  int64_t n_obs;
  const uint32_t* obs_imageset;
  const uint32_t* obs_camera;
  const uint32_t* obs_point;
  const float2* obs_xy;
  CamDev cams[kMaxCameras];
};

// One copy of the optimised state on the device.
struct StateDev {
  double* points;         // [3 * n_points]
  double* rig_tr_global;  // [7 * n_imagesets]
  double* camera_tr_rig;  // [7 * n_cameras]
  double* intrinsics;     // all cameras, CamDev::intr_off
  // derived, recomputed by prepare_state():
  double* image_tr_global;  // [n_imagesets * n_cameras][12]: R row-major (9), t (3)
  double* tangents;         // per control point t1 (3), t2 (3); CamDev::tan_off
};

// Per-observation outputs of the residual / Jacobian kernel.
struct ObsOut {
  double* residual;    // [2 * n_obs] SoA: rx[n_obs], ry[n_obs]
  double* cost;        // [n_obs], -1 = invalid residual
  double* jac;         // [2 * n_jcols][n_obs] SoA: row-x of column c at (2c) * n_obs, row-y at (2c+1) * n_obs
                       //   (NULL in compact mode, except while b200ba_get_jacobians expands it)
  // Compact mode (all cameras central-generic): instead of the 2 x (9 + 6 + 32) Jacobian entries the
  // kernel stores the 14 numbers they are all built from -- P = d pixel / d local_point (2x3), the two
  // rows of Mn = -(A^T A)^-1 A^T / |sum w G| (2x3) and the fractions (fu, fv) of the B-spline support;
  // consumers rebuild a column as  point / pose / rig: chain rule of P with the (L2-resident) poses,
  // intrinsics: w_k(fu, fv) * Mn [t1 t2]_k with the tangent frames. 116 B instead of 656 B per observation.
  double* cjac;        // [14][n_obs] SoA: P00 P01 P02 P10 P11 P12 | Mn00 Mn01 Mn02 Mn10 Mn11 Mn12 | fu fv
  int compact;
  int32_t* cell;       // [n_obs] top-left control point x0 + y0 * gw of the 4x4 support (generic models)
  uint8_t* has_jac;    // [n_obs]
  uint16_t* evals;     // [n_obs] spline evaluations spent by the projection LM (diagnostics; may be NULL)
};

// The normal equations on the device (all FP64). Everything that takes part in the
// cross-GPU reduction lives in ONE allocation so that a single all-reduce covers it.
struct SystemDev {
  double* base;     // the single allocation
  int64_t total;    // doubles
  double* Dblk;     // [nblocks][dsz]  packed upper triangle of each bs x bs block, row-major
  double* bp;       // [nbd]
  double* B;        // [nbd][nd]   row-major
  double* C;        // [nd][nd] row-major, row <= col valid (== column-major lower)
  double* bd;       // [nd]
  double* scalars;  // [8]: cost, n_valid, ...
};

// Calibration report (b200ba_calibration_report): per-camera results and scratch of the radix select.
constexpr int kReportBiasCells = 50;  // kBiasCellCount of ComputeBiasedness (calibration_report.cc:222)
struct ReportCam {
  long long count;
  double sum, max, median;
  double biasedness;
  int biasedness_cells;
  double hfov, vfov;
  unsigned long long select_prefix;  // bits of the median chosen so far
  long long select_rank;             // rank of the median among the values sharing that prefix
};
// Report-owned device buffers (allocated on the first report; none of them is read by the LM path).
struct ReportDev {
  double2* err;          // [n_obs] pixel - xy, device order; NaN where Project failed
  double* mag;           // [n_obs] |err|, NaN where Project failed
  int64_t* cam_off;      // [n_cameras + 1] range of each camera in the device order
  int* cell_off;         // [n_cameras * 2500 + 1] range of each (camera, bias cell) in cell_order
  uint32_t* cell_order;  // [n_obs] device positions by (camera, bias cell), caller's order inside a cell
  double* Q;             // [64] the normalised 8 x 8 Gaussian table, y-major
  double* partial;       // report_partial_size(n_cameras)
  unsigned int* select_hist;  // [n_cameras * 256]
  int* hist;             // [n_cameras * 2500] error histogram, [hy * 50 + hx]
  double* kl;            // [n_cameras * 2500] KL divergence per bias cell, NaN if skipped
  ReportCam* cams;       // [n_cameras]
};

// Outlier round of one camera (b200ba_delete_outliers): device buffers of one call. n is the camera's observation count.
struct OutlierDev {
  int64_t* range;               // [2] {0, n}
  double* mag;                  // [n] |e| on used imagesets where Project succeeded, else NaN
  double* partial;              // report_partial_size(1)
  unsigned int* select_hist;    // [2 * 256]
  ReportCam* stats;             // [2] count, q1 (.median of [0]) and q3 (.median of [1])
  uint8_t* used;                // [n_imagesets] imageset_used, in / out
  int* kept;                    // [n_imagesets] kept features of the camera
  unsigned long long* counts;   // [2] removed, failed
  uint8_t* remove;              // [n_obs] caller order
  uint32_t* owner;              // [w * h] 1 + the largest caller index removed at the pixel, or NULL (no image)
  uint8_t* image;               // [3 * w * h] or NULL
};

// Model comparison (b200ba_compare_models): device buffers of one call.
struct CompareDev {
  double* mag;                  // [w * h] |re-projection error|, NaN where A's un-projection or B's Project fails
  double* dir_err;              // [3 * w * h] dir_B - dir_A, or NULL
  double* rep_err;              // [2 * w * h] pixel - B.Project(dir_A), or NULL
  unsigned long long* dir_max;  // [2] bit patterns of max_error_norm, max_error_component
  int64_t* range;               // [2] {0, w * h}: the one range of launch_report_statistics
  double* partial;              // report_partial_size(1)
  unsigned int* select_hist;    // [256]
  ReportCam* stats;             // count / sum / max / median
  // the five images of b200ba_fitting_images, row-major, or all NULL (then dir_err may be NULL too)
  uint8_t* angles;              // [3 * w * h] _fitting_error_direction_angles.png, written by the comparison pass
  uint8_t* magnitudes;          // [w * h]     _fitting_error_magnitudes.png
  uint8_t* directions;          // [3 * w * h] _fitting_error_directions.png
  uint8_t* rep_magnitudes;      // [w * h]     _fitting_error_reprojection_magnitudes.png
  uint8_t* reprojections;       // [3 * w * h] _fitting_error_reprojections.png
};

// Localization accuracy test (b200ba_localization_accuracy): device buffers of one call.
constexpr int kLocPoints = 15;        // kPointCount (localization_accuracy_test.cc:77)
constexpr int kLocMaxDraws = 4096;    // draws per point before the call gives up (return code 4)
struct LocalizationDev {
  double* p;                   // [trials * 15 * 3] ground-truth points
  double* f;                   // [trials * 15 * 3] compared bearings
  float* samples;              // [trials * 15 * 3] x, y, distance, or NULL
  double* poses;               // [trials * 6] t, c, or NULL
  double* mag;                 // [trials] (double)(float)|t|
  unsigned long long* counts;  // [3] redraws, total iterations, max iterations
  int* capped;                 // 1 if some point was not drawn within kLocMaxDraws
  int64_t* range;              // [2] {0, trials}: the one range of launch_report_statistics
  double* partial;             // report_partial_size(1)
  unsigned int* select_hist;   // [256]
  ReportCam* stats;            // count / sum / max / median of the errors
};

// Reconstruction comparison (b200ba_compare_reconstructions): the count of sample pixels both models un-project and
// the nine entries of M = sum d1 d2^T, row-major.
constexpr int kSweepSums = 10;

// Centre-point analysis of a non-central camera (b200ba_line_offsets): device buffers of one call. The n lines are
// those of the pixels of the calibrated rectangle, p = (y - min_y) * rw + (x - min_x).
constexpr int kLineSums = 10;  // per LM pass: cost, b (3), H (6: 00 01 02 11 12 22)
struct LineOffsetsDev {
  double* lines;               // [6 * n] SoA: origin x, y, z, direction x, y, z
  double* partial;             // line_system_partial_size(): first stage of the LM sums
  double* sums;                // [kLineSums]
  double* mag;                 // [n] line distance |closest - centre|
  unsigned long long* extent;  // bit pattern of max_line_offset_extent
  int64_t* range;              // [2] {0, n}: the one range of launch_report_statistics
  double* stat_partial;        // report_partial_size(1)
  unsigned int* select_hist;   // [256]
  ReportCam* stats;            // count / sum / max / median of the line distances
  double* offsets;             // [3 * w * h] or NULL
  uint8_t* image;              // [3 * w * h] or NULL
  double* obj;                 // [12 * n_obj] or NULL
};

// Voronoi coverage renderer (b200ba_render_voronoi, b200ba_report_images). Sites are integer points in
// quarter-pixel units; a site whose x is kVoronoiNoSite is ignored. The sites are binned into a uniform
// grid of square buckets that covers the image and every site: bucket (bx, by) holds the sites with
// x0 + bx * bs <= x < x0 + (bx + 1) * bs (alike in y), listed in index order in idx[off[b], off[b + 1]).
constexpr int kVoronoiNoSite = INT32_MIN;
struct VoronoiGrid {
  int x0, y0;       // quarter-pixel origin
  int bs;           // bucket size in quarter pixels
  int nx, ny;       // buckets
  int* off;         // [nx * ny + 1]
  int* count;       // [nx * ny] scratch of the counting sort
  int* idx;         // [n_sites]
  int* scan_sums;   // [kVoronoiScanMax] scratch of the scan
};
constexpr int kVoronoiScanChunk = 4096;                                  // elements per block of the scan
constexpr int kVoronoiScanMax = 4096;                                    // blocks of the scan
constexpr int64_t kVoronoiMaxBuckets = int64_t(kVoronoiScanChunk) * kVoronoiScanMax - 1;

// Up to four ranges [lo, hi) of global unknown indices held fixed (debug_fix_* of OptimizeJointly).
struct FixedRanges {
  int n;
  int lo[4], hi[4];
  __host__ __device__ bool has(int g) const {
    for (int i = 0; i < n; ++i)
      if (g >= lo[i] && g < hi[i]) return true;
    return false;
  }
};

// SplitMix64, the mixing function of the counter-based random streams of b200ba_localization_accuracy and
// b200ba_synthetic_poses (include/b200ba.h)
__host__ __device__ __forceinline__ uint64_t loc_splitmix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// ---- feature refinement (b200ba_refine_features): functions the kernel and tests/refine_features_oracle.cc both
// compile, so that they agree bit for bit. On the device every operation is an explicit _rn intrinsic (nvcc cannot
// contract it into a fused multiply-add); the host compiles them with -ffp-contract=off.
__host__ __device__ __forceinline__ float rf_add(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ __forceinline__ float rf_sub(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
__host__ __device__ __forceinline__ float rf_mul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ __forceinline__ float rf_div(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}
__host__ __device__ __forceinline__ double rd_add(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ __forceinline__ double rd_sub(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
__host__ __device__ __forceinline__ double rd_mul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ __forceinline__ double rd_div(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}

__host__ __device__ __forceinline__ bool rf_sign_bit(float v) {
#ifdef __CUDA_ARCH__
  return __float_as_uint(v) >> 31;
#else
  uint32_t u;
  memcpy(&u, &v, sizeof u);
  return u >> 31;
#endif
}

// atan2 in float (the template's angle, PatternData::PatternIntensityAt). The device's atan2f and the C library's
// are different functions; this one is the project's own, so the kernel and the restatement agree. With
// a = min(|x|, |y|) / max(|x|, |y|) and s = a a, atan(a) = a + (a s) q(s) for a degree-7 polynomial q (Horner from
// the highest coefficient, fitted to the relative error on [0, 1]); then r = pi/2 - r when |y| > |x|, r = pi - r
// when x < 0, r = -r when y < 0 (sign bits, so -0 counts as negative). max(|x|, |y|) == 0 gives a = 0; NaN
// propagates. Its error against glibc's atan2f is stated in DESIGN.md section 7.
__host__ __device__ __forceinline__ float rf_atan2(float y, float x) {
  const float ax = fabsf(x), ay = fabsf(y);
  const float mx = ay > ax ? ay : ax, mn = ay > ax ? ax : ay;
  const float a = mx == 0.f ? 0.f : rf_div(mn, mx);
  const float s = rf_mul(a, a);
  float q = 0.00291985273f;
  q = rf_add(rf_mul(q, s), -0.0163645819f);
  q = rf_add(rf_mul(q, s), 0.0432064496f);
  q = rf_add(rf_mul(q, s), -0.0755176023f);
  q = rf_add(rf_mul(q, s), 0.106657945f);
  q = rf_add(rf_mul(q, s), -0.142110035f);
  q = rf_add(rf_mul(q, s), 0.199937671f);
  q = rf_add(rf_mul(q, s), -0.333331525f);
  float r = rf_add(a, rf_mul(rf_mul(a, s), q));
  if (ay > ax) r = rf_sub(1.57079637f, r);
  if (rf_sign_bit(x)) r = rf_sub(3.14159274f, r);
  if (rf_sign_bit(y)) r = -r;
  return r;
}

// (int)v as x86-64 converts (cvttss2si / cvttsd2si): truncation, INT_MIN outside the int range and for NaN
__host__ __device__ __forceinline__ int rf_trunc_int(float v) {
  return (v > -2147483904.f && v < 2147483648.f) ? static_cast<int>(v) : static_cast<int>(0x80000000u);
}
__host__ __device__ __forceinline__ int rd_trunc_int(double v) {
  return (v > -2147483649.0 && v < 2147483648.0) ? static_cast<int>(v) : static_cast<int>(0x80000000u);
}

// PatternData::PatternIntensityAt (feature_detector_tagged_pattern.h:115-130) with rf_atan2: 1 (white), 0 (black) or
// 0.5 (on the feature). The integer products wrap as two's complement.
__host__ __device__ __forceinline__ float rf_pattern_intensity(int num_star_segments, float x, float y) {
  const int kx = static_cast<int>(static_cast<uint32_t>(x > 0.f ? 1 : -1) *
                                  static_cast<uint32_t>(rf_trunc_int(rf_add(fabsf(x), 0.5f))));
  const int ky = static_cast<int>(static_cast<uint32_t>(y > 0.f ? 1 : -1) *
                                  static_cast<uint32_t>(rf_trunc_int(rf_add(fabsf(y), 0.5f))));
  const float cx = rf_sub(x, static_cast<float>(kx)), cy = rf_sub(y, static_cast<float>(ky));
  if (rf_add(rf_mul(cx, cx), rf_mul(cy, cy)) < 1e-8f) return 0.5f;
  float angle = static_cast<float>(rd_sub(static_cast<double>(rf_atan2(cy, cx)), 0.5 * 3.14159265358979323846));
  if (angle < 0.f) angle = static_cast<float>(rd_add(static_cast<double>(angle), 2 * 3.14159265358979323846));
  const double v = rd_div(static_cast<double>(rf_mul(static_cast<float>(num_star_segments), angle)),
                          2 * 3.14159265358979323846);
  return rd_trunc_int(v) % 2 == 0 ? 1.f : 0.f;
}

// The inverse of a row-major 3 x 3 float matrix by the adjugate over the determinant: cofactor
// c(i, j) = m(i1, j1) m(i2, j2) - m(i1, j2) m(i2, j1) with i1 = (i + 1) % 3, i2 = (i + 2) % 3 (j alike),
// det = (c(0, 0) m(0, 0) + c(0, 1) m(0, 1)) + c(0, 2) m(0, 2), inv(j, i) = c(i, j) * (1 / det).
__host__ __device__ __forceinline__ void rf_inverse3(const float* m, float* inv) {
  float c[9];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
      c[i * 3 + j] = rf_sub(rf_mul(m[i1 * 3 + j1], m[i2 * 3 + j2]), rf_mul(m[i1 * 3 + j2], m[i2 * 3 + j1]));
    }
  const float det = rf_add(rf_add(rf_mul(c[0], m[0]), rf_mul(c[1], m[1])), rf_mul(c[2], m[2]));
  const float invdet = rf_div(1.f, det);
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) inv[j * 3 + i] = rf_mul(c[i * 3 + j], invdet);
}

// Solves (A + lambda I) x = b for a symmetric N x N A given by its packed upper triangle in float (row-major:
// (0,0), (0,1), ..., (0,N-1), (1,1), ...), all in double, by an LDL^T factorisation without pivoting:
//   A'_ij = (double)A_ij, plus (double)lambda on the diagonal (the sum rounded to float first, as the float H_LM
//   of the reference is: A'_ii = (double)(float)(A_ii + lambda));
//   for j = 0..N-1: d_j = A'_jj - sum_{k<j} (L_jk L_jk) d_k, subtracting k = 0, 1, ... in order;
//     for i > j: v = A'_ji - sum_{k<j} (L_ik L_jk) d_k, alike, and L_ij = v / d_j when |d_j| > 0, else L_ij = v;
//   y_i = b_i - sum_{k<i} L_ik y_k (k ascending); z_i = y_i / d_i when |d_i| > DBL_MIN, else z_i = 0;
//   x_i = z_i - sum_{k>i} L_ki x_k (i descending, k ascending); returned as (float)x_i.
// A zero (or NaN) pivot is treated as Eigen 3.3's LDLT treats it: the column is not scaled, and the solution
// component is set to 0 (the pseudo-inverse of D). So A = 0 with lambda = 0, the LM's system in a textureless
// window, gives x = 0, a step that does not lower the cost.
template <int N>
__host__ __device__ __forceinline__ void rf_ldlt_solve(const float* A, float lambda, const float* b, float* x) {
  double L[N][N], d[N], y[N];
#pragma unroll
  for (int j = 0; j < N; ++j) {
    const int jj = j * N - j * (j - 1) / 2;  // packed index of (j, j)
    double dj = static_cast<double>(rf_add(A[jj], lambda));
#pragma unroll
    for (int k = 0; k < j; ++k) dj = rd_sub(dj, rd_mul(rd_mul(L[j][k], L[j][k]), d[k]));
    d[j] = dj;
#pragma unroll
    for (int i = j + 1; i < N; ++i) {
      double v = static_cast<double>(A[jj + (i - j)]);
#pragma unroll
      for (int k = 0; k < j; ++k) v = rd_sub(v, rd_mul(rd_mul(L[i][k], L[j][k]), d[k]));
      L[i][j] = fabs(dj) > 0.0 ? rd_div(v, dj) : v;
    }
  }
#pragma unroll
  for (int i = 0; i < N; ++i) {
    double v = static_cast<double>(b[i]);
#pragma unroll
    for (int k = 0; k < i; ++k) v = rd_sub(v, rd_mul(L[i][k], y[k]));
    y[i] = v;
  }
#pragma unroll
  for (int i = N - 1; i >= 0; --i) {
    double v = fabs(d[i]) > 2.2250738585072014e-308 ? rd_div(y[i], d[i]) : 0.0;
#pragma unroll
    for (int k = i + 1; k < N; ++k) v = rd_sub(v, rd_mul(L[k][i], y[k]));
    y[i] = v;
    x[i] = static_cast<float>(v);
  }
}

}  // namespace b200ba
