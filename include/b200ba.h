/*
 * b200ba.h -- C ABI of the CUDA (H100, sm_90a) joint-optimisation (bundle-adjustment) path.
 *
 * This is the drop-in boundary for ONE hot path of puzzlepaint/camera_calibration:
 *   double OptimizeJointly(Dataset&, BAState*, ...)            (reference:
 *     applications/camera_calibration/src/camera_calibration/bundle_adjustment/joint_optimization.h:53-70,
 *     implementation joint_optimization.cc:757-953)
 * and its GPU twin
 *   OptimizationReport CudaOptimizeJointly(...)               (reference:
 *     bundle_adjustment/cuda_joint_optimization.h:45-59).
 *
 * The reference has no C ABI; its seam is the C++ free function above plus the
 * CameraModel plugin (models/camera_model.h:42-204). A maintainer binds this
 * library by flattening Dataset / BAState into the POD structs below (see
 * INTEGRATION.md and include/b200ba_shim.hpp, which does exactly that behind the
 * reference's own signature).
 *
 * Conventions
 *   - plain pointers and sizes only; no C++ / torch types cross this line.
 *   - all functions return 0 on success, non-zero on error; b200ba_last_error()
 *     gives the message. Nothing here aborts (the reference CHECK()s).
 *   - the caller owns every host array for the duration of the call only; the
 *     handle owns all device memory, streams, cuBLAS/cuSOLVER handles and the
 *     NCCL communicator.
 *   - a handle is single-owner / not re-entrant, like the reference's cost
 *     function (models/central_grid.h:186).
 *   - quaternions are (w, x, y, z) followed by translation (x, y, z): the order
 *     of the reference's CUDA state upload (cuda_joint_optimization.cc:88-112).
 *     Eigen's coeffs() order is x,y,z,w -- convert at the shim.
 *   - pixels use the "pixel-corner" convention (camera_model.h:67-70).
 */
#ifndef B200BA_H_
#define B200BA_H_

#include <stdint.h>

#if defined(__GNUC__)
#define B200BA_API __attribute__((visibility("default")))
#else
#define B200BA_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* Values equal CameraModel::Type (models/camera_model.h:44-54). */
enum {
  B200BA_MODEL_CENTRAL_GENERIC = 0,
  B200BA_MODEL_NONCENTRAL_GENERIC = 1,
  B200BA_MODEL_CENTRAL_THIN_PRISM_FISHEYE = 2, /* not on the accelerated path */
  B200BA_MODEL_CENTRAL_OPENCV = 3,
  B200BA_MODEL_CENTRAL_RADIAL = 4 /* not on the accelerated path */
};

/* Values equal SchurMode (libvis lm_optimizer.h). All modes are numerically
 * interchangeable in the reference (test/central_generic_test.cc:77-91); this
 * library always stores the off-diagonal part densely on the device. */
enum {
  B200BA_SCHUR_DENSE = 0,
  B200BA_SCHUR_DENSE_CUDA = 1,
  B200BA_SCHUR_DENSE_ONTHEFLY = 2,
  B200BA_SCHUR_SPARSE = 3,
  B200BA_SCHUR_SPARSE_ONTHEFLY = 4
};

enum {
  B200BA_JACOBIAN_NUMERIC = 0, /* reference behaviour (finite differences); CPU oracle only */
  B200BA_JACOBIAN_ANALYTIC = 1 /* implicit-function-theorem Jacobian; the GPU path */
};

/* Static description of one camera (CameraModel base members,
 * models/camera_model.h:189-203, plus the grid resolution of the generic models). */
typedef struct b200ba_camera {
  int32_t model_type;
  int32_t width, height;
  int32_t calibration_min_x, calibration_min_y;
  int32_t calibration_max_x, calibration_max_y;
  int32_t grid_width, grid_height; /* 0 for parametric models */
} b200ba_camera;

/* Number of doubles in the flat intrinsics array of a camera:
 *   central-generic   : 3*gw*gh               (grid, row-major, xyz; central_grid.h m_grid)
 *   noncentral-generic: 3*gw*gh direction grid followed by 3*gw*gh point grid
 *   central-opencv    : 12  (fx fy cx cy k1..k6 p1 p2; central_opencv.cc:77-88)  */
B200BA_API int64_t b200ba_intrinsics_size(const b200ba_camera* cam);
/* update_parameter_count() of the model: 2*gw*gh / 5*gw*gh / 12. */
B200BA_API int32_t b200ba_update_parameter_count(const b200ba_camera* cam);

/* The constant part of a BA problem: the flattened Dataset (dataset.h:57-212)
 * restricted to used imagesets. Observations are listed in the reference's
 * residual order: imageset-major, then camera, then feature order
 * (joint_optimization.cc:273-290); obs_imageset must be non-decreasing and, within
 * an imageset, obs_camera non-decreasing. */
typedef struct b200ba_problem {
  int32_t n_cameras;
  const b200ba_camera* cameras;
  int32_t n_imagesets; /* used imagesets (sequential indices) */
  int32_t n_points;
  int64_t n_obs;
  const uint32_t* obs_imageset; /* [n_obs] */
  const uint32_t* obs_camera;   /* [n_obs] */
  const uint32_t* obs_point;    /* [n_obs]  PointFeature::index */
  const float* obs_xy;          /* [2*n_obs] PointFeature::xy (float, dataset.h:67) */
} b200ba_problem;

/* The optimised part of BAState (ba_state.h:79-96) + the warm-start cache
 * PointFeature::last_projection (dataset.h:79-83). Used for both input and output. */
typedef struct b200ba_state {
  double* points;            /* [3*n_points] */
  double* rig_tr_global;     /* [7*n_imagesets]  qw qx qy qz tx ty tz */
  double* camera_tr_rig;     /* [7*n_cameras] */
  double* const* intrinsics; /* [n_cameras] -> b200ba_intrinsics_size() doubles each */
  double* last_projection;   /* [2*n_obs]; may be NULL (= all zero on input, dropped on output) */
} b200ba_state;

/* Arguments of OptimizeJointly (joint_optimization.h:53-70) + the constants it
 * hard-codes (joint_optimization.cc:916-923, :346). */
typedef struct b200ba_options {
  int32_t max_iteration_count;
  double init_lambda;           /* < 0: initialise from H (lm_optimizer.h:766-781) */
  double numerical_diff_delta;  /* used by the numeric Jacobian mode only */
  double regularization_weight; /* the reference ignores it with an error log (:299-305); must be 0 */
  int32_t localize_only;
  int32_t eliminate_points;
  int32_t schur_mode;
  int32_t max_lm_attempts;      /* reference: 50 */
  double init_lambda_factor;    /* reference: 1e-5 */
  double huber_parameter;       /* reference: 1.0 */
  int32_t jacobian_mode;        /* B200BA_JACOBIAN_* */
  int32_t print_progress;
  /* the debug_* switches of OptimizeJointly (joint_optimization.h:63-68):
   *   debug_verify_cost: before optimising, the cost is evaluated without and with Jacobians, twice
   *     (LMOptimizer::VerifyCost, lm_optimizer.h:474-490); the call fails with code 5 where the
   *     reference CHECKs |cost1 - cost2| <= 1e-3 (joint_optimization.cc:866-876).
   *   debug_fix_*: the variables of the group are held fixed (LMOptimizer::FixVariable,
   *     joint_optimization.cc:878-903): their update is 0 and they are removed from the linear system
   *     (lm_optimizer.h:1069-1121). The reference then solves the thinned system densely; here the rows /
   *     columns are masked out of H, b and the Schur-complement path is kept (same solution). */
  int32_t debug_verify_cost;
  int32_t debug_fix_points;
  int32_t debug_fix_poses;
  int32_t debug_fix_rig_poses;
  int32_t debug_fix_intrinsics;
} b200ba_options;

B200BA_API void b200ba_default_options(b200ba_options* opt);

#define B200BA_MAX_TRACE 128

/* OptimizationReport (libvis lm_optimizer.h:55-77) + what OptimizeJointly returns
 * through its out-parameters, + a per-iteration trace for parity checks. */
typedef struct b200ba_report {
  double initial_cost;
  double final_cost;
  double final_lambda;
  int32_t num_iterations_performed;
  int32_t performed_an_iteration;
  double cost_and_jacobian_evaluation_time; /* seconds */
  double solve_time;                        /* seconds */
  int64_t n_valid;    /* residuals valid at the final state */
  int64_t n_invalid;
  double rmse;        /* sqrt(sum |pixel - xy|^2 / n_valid) at the final state (SURVEY 8d) */
  int32_t trace_len;
  double trace_cost[B200BA_MAX_TRACE];    /* cost after each outer iteration */
  double trace_lambda[B200BA_MAX_TRACE];  /* lambda after each outer iteration */
  int32_t trace_attempts[B200BA_MAX_TRACE]; /* LM attempts used by each outer iteration */
} b200ba_report;

typedef struct b200ba_handle b200ba_handle;

/* ---- lifetime ---------------------------------------------------------- */
/* device < 0: use the current CUDA device. Copies the problem to the device. */
B200BA_API int b200ba_create(const b200ba_problem* problem, int device, b200ba_handle** out);
B200BA_API void b200ba_destroy(b200ba_handle* h);
B200BA_API const char* b200ba_last_error(const b200ba_handle* h); /* h may be NULL: last create error */

/* ---- state transfer ------------------------------------------------------ */
B200BA_API int b200ba_set_state(b200ba_handle* h, const b200ba_state* state);
B200BA_API int b200ba_get_state(b200ba_handle* h, b200ba_state* state);

/* Device-side copy of the optimised state + last_projection held by the handle into a snapshot
 * slot / back (no host transfer). The reference keeps such a copy implicitly: LMOptimizer works
 * on `State test_state = *state` (libvis lm_optimizer.h:868) and the product writes a checkpoint
 * after every iteration (calibration.cc:240-243). */
B200BA_API int b200ba_snapshot_state(b200ba_handle* h);
B200BA_API int b200ba_restore_state(b200ba_handle* h);

/* ---- the hot path -------------------------------------------------------- */
/* Equivalent of OptimizeJointly (joint_optimization.cc:757-953) on the state held
 * by the handle; the state stays resident on the device between calls. */
B200BA_API int b200ba_optimize(b200ba_handle* h, const b200ba_options* opt, b200ba_report* report);

/* Convenience: set_state + optimize + get_state with HOST buffers, i.e. exactly
 * what a call of the reference's OptimizeJointly(Dataset&, BAState*) does. */
B200BA_API int b200ba_optimize_host(b200ba_handle* h, b200ba_state* state, const b200ba_options* opt,
                         b200ba_report* report);

/* RunBundleAdjustment (calibration.cc:187-304) on the state held by the handle: up to
 * max_iteration_count single LM iterations (lambda carried over, starting from opt->init_lambda, the
 * reference passes -1), after each one ChooseNiceCameraOrientation + Rotate + the camera_tr_rig update
 * for every camera (calibration.cc:245-252, models/central_generic.cc:570-621; skipped when
 * localize_only), stop as soon as cost >= last_cost - cost_reduction_threshold (:298-300). The state
 * never leaves the device; on_iteration (nullable) is called after every iteration -- the place for
 * the reference's per-iteration SaveBAState checkpoint via b200ba_get_state (:240-243) -- and stops
 * the loop by returning non-zero (the reference's 'q' key). With several ranks the call is collective. */
typedef struct b200ba_ba_report {
  double initial_cost, final_cost, final_lambda, rmse;
  int64_t n_valid, n_invalid;
  int32_t iterations;    /* LM iterations run (OptimizeJointly calls) */
  int32_t lm_attempts;   /* linear solves over all of them */
  double device_ms;      /* sum of the iterations' device times */
  double costs[B200BA_MAX_TRACE]; /* cost after each iteration */
} b200ba_ba_report;
B200BA_API int b200ba_run_bundle_adjustment(b200ba_handle* h, const b200ba_options* opt, int32_t max_iteration_count,
                                            double cost_reduction_threshold, b200ba_ba_report* report,
                                            int (*on_iteration)(void* user, int32_t iteration, double cost),
                                            void* user);

/* ---- calibration report ---------------------------------------------------- */
/* The numbers of CreateCalibrationReport (calibration_report.cc:83-98, per camera :713-817) for every
 * camera: every observation re-projected with Project (start at the centre of the calibrated area, no
 * warm start), then per camera the count / sum / max / median of |pixel - xy| over the successful
 * projections, the 50 x 50 error histogram (half extent 0.2f px), the biasedness (median KL divergence
 * of the per-cell error distributions from a Gaussian, 50 x 50 cells, cells with < 5 errors skipped)
 * and the approximate field of view. */
#define B200BA_REPORT_HIST 50
typedef struct b200ba_camera_report {
  int64_t reprojection_error_count;
  double reprojection_error_sum, reprojection_error_max, reprojection_error_median; /* median NaN if count == 0 */
  double biasedness;                 /* median KL divergence; NaN if no cell has >= 5 errors */
  int32_t biasedness_cells;          /* cells that entered the median */
  double horizontal_fov, vertical_fov; /* radians; -1 if not computed (non-central and OpenCV cameras) */
  int32_t histogram[B200BA_REPORT_HIST * B200BA_REPORT_HIST]; /* [hy * 50 + hx] */
} b200ba_camera_report;
/* CreateCalibrationReport's numbers (calibration_report.cc) for every camera, on the state held by the handle.
 * errors (nullable): [2*n_obs] pixel - xy in caller order, NaN where Project failed. Reads the state, writes none
 * of it (nor last_projection, nor what b200ba_get_jacobians reads). report_ms (nullable): device time. The
 * report's buffers are allocated on the first call. Single-rank handles only. */
B200BA_API int b200ba_calibration_report(b200ba_handle* h, b200ba_camera_report* reports /* [n_cameras] */,
                                         double* errors, double* report_ms);
/* The images of CreateCalibrationReportForCamera (calibration_report.cc:713-838) for one camera, each [h*w*3]
 * RGB row-major and nullable:
 *   observation_directions  the un-projected direction of every pixel (x + 0.5f, y + 0.5f), coloured
 *                           ((70*255.99f)/2.f)*(d+1) for x, y and ((270*255.99f)/2.f)*(d+1) for z, converted to u8
 *                           as x86-64 does (truncation to int32, low byte); black where the un-projection fails.
 *                           Central- and non-central-generic cameras only (returns 2 for others).
 *   error_directions,       Voronoi maps of the feature sites: the first successful projection (caller's order) per
 *   error_magnitudes        integer feature pixel ((int)x, (int)y) with 0 <= (int)x < 4w, 0 <= (int)y < 4h is a site
 *                           at the quarter pixel ((int)(4x), (int)(4y)), coloured by its error's direction or by its
 *                           magnitude (saturating at 0.5 px); a pixel is the sum of area(pixel n cell) * colour
 *                           over the cells, + 0.5, clamped to [0, 255.99] and truncated (exact partition).
 * n_sites (nullable): the number of sites; device_ms (nullable): device time. Uses the report's error pass and
 * buffers; reads the state and writes none of it (nor last_projection, nor what b200ba_get_jacobians reads).
 * Single-rank handles only; returns 2 for a bad camera index. */
B200BA_API int b200ba_report_images(b200ba_handle* h, int32_t camera, uint8_t* observation_directions,
                                    uint8_t* error_directions, uint8_t* error_magnitudes, int64_t* n_sites,
                                    double* device_ms);

/* ---- building blocks, exposed for parity tests and profiling -------------- */
/* One pass of JointOptimizationCostFunction::Compute<compute_jacobians>
 * (joint_optimization.cc:240-306) at the current state.
 *   residuals   [2*n_obs] out, nullable   pixel - xy
 *   costs       [n_obs]   out, nullable   Huber cost, -1 for invalid residuals
 *   total_cost            out, nullable
 * Updates last_projection on the device like the reference mutates the Dataset. */
B200BA_API int b200ba_evaluate(b200ba_handle* h, const b200ba_options* opt, int compute_jacobians,
                    double* residuals, double* costs, double* total_cost);

/* Per-observation Jacobians of the last b200ba_evaluate(compute_jacobians=1):
 *   j_point [n_obs*2*3], j_pose [n_obs*2*6], j_rig [n_obs*2*6] (nullable / zero if 1 camera),
 *   j_intr [n_obs*2*K], intr_index [n_obs*K] (global column of each entry), K = max over cameras
 *   of IntrinsicsJacobianSize (32 / 80 / 12). Row-major [obs][row][col]. */
B200BA_API int b200ba_get_jacobians(b200ba_handle* h, double* j_point, double* j_pose, double* j_rig,
                         double* j_intr, int32_t* intr_index, int32_t K);

/* Build H, b at the current state (hot loop 1) and download them as one dense
 * upper-triangular matrix in the reference's variable ordering
 * (joint_optimization.cc:49-59). H [n*n] row-major, b [n]; only for small problems. */
B200BA_API int b200ba_build_system(b200ba_handle* h, const b200ba_options* opt, int32_t n, double* H,
                        double* b, double* cost);
B200BA_API int32_t b200ba_degrees_of_freedom(const b200ba_handle* h, const b200ba_options* opt);

/* Stand-alone Schur-complement solve (libvis lm_optimizer.h:1246-1369) of
 *   [D B; B^T C] x = [b1; b2],  D block-diagonal with n_blocks blocks of block_size (<= 6).
 * Only the upper triangles of D blocks and C are read. Host buffers, row-major:
 *   D [n_blocks*bs*bs], B [(n_blocks*bs) * n_dense], C [n_dense*n_dense]. */
B200BA_API int b200ba_schur_solve(int device, int32_t block_size, int32_t n_blocks, int32_t n_dense,
                       const double* D, const double* B, const double* C, const double* b1,
                       const double* b2, double* x);

/* Stand-alone dense SPD solve A x = b on the in-tree kernels of the dense phase (blocked Cholesky with
 * FP64 tensor-core trailing updates, packed triangular solves): what replaces
 * `schur_M.selfadjointView<Upper>().ldlt().solve()` (libvis lm_optimizer.h:1361) inside b200ba_optimize.
 * A [n*n] symmetric, host; block_width a multiple of 128; the *_ms outputs (nullable) are device times.
 * Returns 4 if A is not positive definite. Tests / profiling. */
B200BA_API int b200ba_dense_cholesky_solve(int device, int32_t n, int32_t block_width, const double* A,
                                           const double* b, double* x, double* factor_ms, double* solve_ms);

/* CameraModel::ProjectWithInitialEstimate / Unproject for n points, on the device.
 * pixels is in/out (initial estimate / result); ok[i] = 1 on success. */
B200BA_API int b200ba_project(int device, const b200ba_camera* cam, const double* intrinsics, int64_t n,
                   const double* local_points, double* pixels, int32_t* ok);
B200BA_API int b200ba_unproject(int device, const b200ba_camera* cam, const double* intrinsics, int64_t n,
                     const double* pixels, double* directions, double* origins, int32_t* ok);

/* Voronoi coverage rendering, the renderer of b200ba_report_images' error maps. sites_q [2n]: integer sites in
 * quarter pixels, |x|, |y| <= 2^28 (a repeated position belongs to its lowest index); colors [3n]. image [h*w*3]
 * RGB row-major: per pixel the sum over the Voronoi cells of area(pixel n cell) * colour, + 0.5, clamped to
 * [0, 255.99] and truncated; no site gives black. device_ms (nullable): device time. Stand-alone (allocates,
 * computes, frees); returns 2 for a bad argument, 3 without a device. */
B200BA_API int b200ba_render_voronoi(int device, int32_t width, int32_t height, int64_t n_sites, const int32_t* sites_q,
                                     const float* colors, uint8_t* image, double* device_ms);

/* ---- calibration visualisation: VisualizeCameraModel (APP/tools/visualize_calibration.cc:39-96, the
 * --visualize_kalibr_calibration / --visualize_colmap_calibration tools) for a libvis RadtanCamera8d,
 * params = k1 k2 r1 r2 fx fy cx cy (libvis/camera.h: RadtanDistortion4 :500-591, PixelMapping4 :1011-1121).
 *   Unproject(x, y): n = (fx_inv x + cx_inv, fy_inv y + cy_inv), fx_inv = 1 / fx, cx_inv = -cx / fx (pixel-corner
 *     convention); then at most 5 Gauss-Newton steps from u = n: e = n - D(u), u += (J^T J)^-1 J^T e, Eigen's closed-form
 *     2 x 2 inverse (1 / det times the adjugate) and the products taken left to right; the iteration stops after the
 *     step whose e has |e|^2 < DBL_EPSILON. The direction is (u.x, u.y, 1). Where 5 steps do not converge it is the
 *     fifth iterate; where the iteration diverges it holds whatever IEEE arithmetic gives (NaN, inf).
 *   Orientation: F = FromTwoVectors(Unproject(0.5f w, 0.5f h), e_z); the directions of the window x in
 *     [min(w - 1, w/2 + 11), w - 1], y in [max(0, h/2 - 10), min(h - 1, h/2 + 10)] at (x + 0.5f, y + 0.5f), not
 *     normalised, are summed in row-major order (independent of the launch shape) and divided by their count, giving
 *     m; angle = atan2(-(F m).y, (F m).x); rotation = AngleAxisd(angle, e_z) F. Every operation but atan2, sin and cos
 *     is rounded on its own in Eigen's order (FromTwoVectors, toRotationMatrix, the products), because for tiny images
 *     the angle is atan2 of two small numbers formed by cancellation.
 *   Every pixel: d = rotation * Unproject(x + 0.5f, y + 0.5f).normalized() (division by sqrt of the squared norm; a
 *     zero or NaN vector is left as it is), coloured ((70 * 255.99f) / 2.f) * (d + 1) (x, y) and
 *     ((270 * 255.99f) / 2.f) * (d + 1) (z) in double and converted to u8 as b200ba_report_images' observation
 *     directions are: truncation to int32 with INT_MIN for NaN and out-of-range values, then the low byte (so a NaN
 *     direction is black). A forward direction or window sum that is not finite makes every pixel NaN, as in the
 *     reference.
 * Every value-path operation is rounded on its own (no fused multiply-add) in the reference's order, so that a
 * restatement in double reproduces each direction bit for bit given the rotation.
 * image [h*w*3] RGB row-major. rotation (nullable): [9] row-major. directions (nullable): [h*w*3] the rotated unit
 * directions. device_ms (nullable): device time. Stand-alone (allocates, computes, frees); returns 2 before any CUDA
 * call for a NULL params or image, width or height < 1 or > 2^24 or more than 2^31 pixels, a parameter that is not
 * finite, or fx == 0 or fy == 0 (the reference divides by zero there); 3 without a device. Repeated calls give
 * identical bytes. */
B200BA_API int b200ba_visualize_camera(int device, int32_t width, int32_t height, const double* params, uint8_t* image,
                                       double* rotation, double* directions, double* device_ms);

/* ---- model resampling (row f-4): CentralGenericModel::FitToPixelDirectionsImpl --------
 * (APP/models/central_generic.cc:551-568 with the cost function of :152-228 and the state of
 * :40-83). Levenberg-Marquardt over the direction grid -- 2 local DoF per control point in its
 * tangent frame -- so that the normalised B-spline un-projection at n grid points matches n unit
 * directions: LMOptimizer::Optimize(max_iteration_count, max_lm_attempts = 10, init_lambda = -1,
 * init_lambda_factor = 0.001f), quadratic loss (cost = 1/2 sum r^2 over the 3n scalar residuals),
 * dense solve. Called by FitToDenseModel / FitToPixelDirections when a model is resampled to
 * another grid resolution (APP/calibration.cc:373-522).
 *   grid         [3 * grid_width * grid_height] in/out, row-major, unit directions
 *   grid_points  [2 n] grid coordinates (PixelCornerConvToGridPoint of the sample pixels); each
 *                must have its 4x4 support inside the grid (1 <= g < size - 2)
 *   directions   [3 n] */
typedef struct b200ba_fit_report {
  double initial_cost;
  double final_cost;
  double final_lambda;
  int32_t num_iterations_performed;
  int32_t lm_attempts; /* total number of linear solves */
} b200ba_fit_report;
B200BA_API int b200ba_fit_directions(int device, int32_t grid_width, int32_t grid_height, double* grid, int64_t n,
                          const double* grid_points, const double* directions, int32_t max_iteration_count,
                          b200ba_fit_report* report);

/* ---- model comparison: CreateFittingErrorReport (APP/fitting_report.h:55-203) as the
 * --compare_calibrations tool runs it (APP/tools/compare_calibrations.cc:39-74: base = A, fitted = B,
 * rotation Identity, no border), numbers only. For every pixel (x, y) of the image: A un-projects
 * (x + 0.5f, y + 0.5f); where that succeeds, B un-projects the same pixel (direction error
 * dir_B - dir_A, +inf where B fails) and B projects A's direction (Project: start at the centre of B's
 * calibrated area, no warm start), the re-projection error being (x + 0.5f, y + 0.5f) - projection.
 * Both models must be central-generic, with the same width / height and grids of at least 4 x 4. */
typedef struct b200ba_fitting_report {
  int64_t reprojection_error_count;      /* pixels where A un-projects and B projects A's direction */
  double reprojection_error_sum, reprojection_error_max, reprojection_error_median; /* median NaN if count == 0 */
  double max_error_norm, max_error_component; /* over pixels where both un-projections succeed; 0 if none */
} b200ba_fitting_report;
/* Stand-alone (allocates, computes, frees). intr_a / intr_b: the grids [3 * grid_width * grid_height]; not
 * modified. direction_errors (nullable): [3*w*h] row-major (y, x), NaN where A fails, +inf where B fails.
 * reprojection_errors (nullable): [2*w*h], NaN where A or Project fails (the reference's image holds 0 there).
 * device_ms (nullable): device time of the comparison. Returns 2 for a bad argument, 3 without a device. */
B200BA_API int b200ba_compare_models(int device, const b200ba_camera* cam_a, const double* intr_a,
                                     const b200ba_camera* cam_b, const double* intr_b, b200ba_fitting_report* report,
                                     double* direction_errors, double* reprojection_errors, double* device_ms);
/* The comparison of b200ba_compare_models (same arguments and checks, the same report bit for bit) together with the
 * five images of CreateFittingErrorReport (fitting_report.h:135-184), row-major (y, x), all required:
 *   error_magnitudes        [h*w]    _fitting_error_magnitudes.png: 255.99f * (|e| / max_error_norm), e = dir_B - dir_A
 *   error_direction_angles  [h*w*3]  _fitting_error_direction_angles.png: per channel
 *                                    min(255, max(0, (int)(127 + 127 / (M_PI / 180.f * 0.025) * (atan2(a.z, a.x) -
 *                                    atan2(b.z, b.x)) + 0.5))), the same with atan2(.y, .z), and 127; a = dir_A, b = dir_B
 *   error_directions        [h*w*3]  _fitting_error_directions.png: (255.99f / 2) * (clamp(e / max_error_component,
 *                                    -1, 1) + 1) per component
 *   reprojection_magnitudes [h*w]    _fitting_error_reprojection_magnitudes.png:
 *                                    max<float>(0, min<float>(255, 255.99f * |r| / reprojection_error_max))
 *   reprojections           [h*w*3]  _fitting_error_reprojections.png: (127, 127, 127) everywhere (below)
 * with r = pixel - B.Project(dir_A). Every value is computed in the reference's order and float / double mix. Where the
 * reference's C++ is undefined, the result is what its x86-64 build computes:
 *   - every double / float -> u8 conversion, and the angle's double -> int, truncates to int32 with INT_MIN for NaN
 *     and out-of-range values, then keeps the low byte: so the magnitude is 0 where B fails (e = +inf) and where
 *     max_error_norm == 0 (0 / 0);
 *   - std::min / std::max and Eigen's cwiseMin / cwiseMax keep their first argument when a comparison involves NaN:
 *     where max_error_component == 0 a zero error gives NaN and the direction pixel is (0, 0, 0); where
 *     reprojection_error_max == 0 every reprojection magnitude is 255;
 *   - where B fails the reference reads an uninitialised fitted direction, pinned here as NaN: the angle pixel is
 *     (0, 0, 127); the direction pixel is (255, 255, 255) (e = +inf clamps to 1);
 *   - where A fails the magnitude, angle and direction pixels are 0 / (0, 0, 0), and the reprojection images see
 *     r = 0, as in the reference's image, which holds zero wherever Project fails or is not tried;
 *   - the reprojection-direction strength is max(0, min(1, |r| / -1)) = 0, because the tool passes
 *     max_visualization_extent_pixels = -1, so that image is uniformly (127, 127, 127), as the reference writes it.
 * device_ms (nullable): device time of the comparison and the images. Stand-alone; returns 2 for a bad argument
 * (also a NULL image) before any CUDA call, 3 without a device. Repeated calls give identical bytes. */
B200BA_API int b200ba_fitting_images(int device, const b200ba_camera* cam_a, const double* intr_a,
                                     const b200ba_camera* cam_b, const double* intr_b, b200ba_fitting_report* report,
                                     uint8_t* error_magnitudes, uint8_t* error_direction_angles,
                                     uint8_t* error_directions, uint8_t* reprojection_magnitudes,
                                     uint8_t* reprojections, double* device_ms);

/* ---- localization accuracy test (APP/tools/localization_accuracy_test.cc:47-131, --localization_accuracy_test):
 * what the difference between a ground-truth calibration and a compared calibration of one camera costs a camera
 * that is localized with the compared one. Every trial:
 *   1. draws 15 points: a float pixel (x, y) in [0, w] x [0, h] that BOTH models un-project (drawn again
 *      otherwise), the ground-truth unit direction n = normalize(u_gt) at a distance s, p = s n, and the compared
 *      bearing f = normalize(s normalize(u_cmp)) -- mathematically normalize(u_cmp); written with the operations
 *      that normalise the transformed point, so that two identical models give f = normalize(p) bit for bit;
 *   2. fits the pose x = (t, c) from x = 0, c the Cayley vector, R(c) = ((1 - c'c) I + 2 c c' + 2 [c]x) / (1 + c'c),
 *      u_i = normalize(R(c)' (p_i - t)), minimising opengv's absolute_pose::optimize_nonlinear cost
 *      F = sum_i (1 - f_i' u_i)^2, evaluated without cancellation as sum_i r_i^2, r_i = 1/2 |u_i - f_i|^2.
 *      The iteration is Levenberg-Marquardt on H = sum_i J_i' (|e_i|^2 I + 2 e_i e_i') J_i (the Hessian of F
 *      without its O(|e|^3) terms), e_i = u_i - f_i, J_i = du_i / d(t, c), step (H + lambda I) d = -grad F,
 *      x <- x + d; lambda_0 = 0.001f tr(H) / 6, at most 10 attempts per iteration (x0.5 on an accepted step, x2
 *      on a rejected step or a failed Cholesky factorisation), at most 100 iterations, stopping when an
 *      iteration accepts nothing or F == 0. The result is the minimiser of the reference's cost, not the point
 *      where the reference's MINPACK solver stops (that is reached early, at about twice the minimal cost);
 *   3. records error = (float)|t|, the camera-centre offset in metres.
 * The random stream is counter-based: with key = (trial << 20) | (point << 16) | (attempt << 4) | component and
 * SplitMix64(z) = { z += 0x9E3779B97F4A7C15; z = (z ^ z >> 30) * 0xBF58476D1CE4E5B9;
 *                   z = (z ^ z >> 27) * 0x94D049BB133111EB; return z ^ z >> 31; } (mod 2^64),
 * a draw is h = SplitMix64(SplitMix64(seed) ^ key), so it depends only on (seed, trial, point, attempt,
 * component). Attempt a of a point takes x = (float)(h_0 >> 40) * 2^-24f * (float)w and
 * y = (float)(h_1 >> 40) * 2^-24f * (float)h (component 0 and 1, float products); the attempt that both models
 * un-project takes the distance s = 1.5f + ((float)(h_2 % 10000) / 10000.f) * 1.0f (component 2). Examples, w = 640:
 *   seed 0, trial 0, point 0, attempt 0:  h_0 = 0xa706dd2f4d197e6f, x = 417.5670166015625,
 *                                         h_2 = 0xd7cc9674ff5ffa39, s = 1.7856999635696411 (k = 2857)
 *   seed 7, trial 12345, point 14, attempt 3:  h_0 = 0xe273e8e0afcdd023, x = 566.1318969726562
 * Both models must be central-generic (OpenCV models have no device un-projection; the reference never ends for a
 * non-central model, whose Unproject(x, y, Vec3d*) always fails), of one image size, with grids of at least
 * 4 x 4 and calibrated areas that intersect [0, w] x [0, h]. */
typedef struct b200ba_localization_report {
  int64_t trial_count;
  double average_error; /* metres: the mean of the float errors, a fixed-order double sum (the reference sums in
                           float, in order) */
  double median_error;  /* metres: sorted(errors)[trial_count / 2] */
  double max_error;     /* metres */
  int64_t total_iterations; /* accepted LM steps over all pose fits */
  int64_t redraws;          /* pixels drawn again because a model did not un-project them */
  int32_t max_iterations;   /* accepted LM steps of the longest pose fit */
} b200ba_localization_report;
/* Stand-alone (allocates, computes, frees); the grids gt_intr / intr [3 * grid_width * grid_height] are not
 * modified. errors (nullable): [trials] float. poses (nullable): [trials][6] t, c. samples (nullable):
 * [trials][15][3] float x, y, distance of the accepted draws. device_ms (nullable): device time of the test.
 * Returns 2 for a bad argument (before any CUDA call; also for trials < 1 or trials > 2^32), 3 without a device,
 * 4 when a point of a trial is still not un-projected by both models after 4096 draws. */
B200BA_API int b200ba_localization_accuracy(int device, const b200ba_camera* gt_cam, const double* gt_intr,
                                            const b200ba_camera* cam, const double* intr, int64_t trials,
                                            uint64_t seed, b200ba_localization_report* report, float* errors,
                                            double* poses, float* samples, double* device_ms);

/* ---- reconstruction comparison (APP/tools/bundle_adjustment.cc:223-392, --compare_reconstructions): how far two
 * bundle-adjusted reconstructions of one image sequence -- e.g. one per calibration of the camera -- drift apart.
 * Poses are [qw qx qy qz tx ty tz] (Sophus order: (a * b).q = normalize(a.q b.q), (a * b).t = a.t + R(a.q) b.t).
 *   1. G_k[i] = (camera_tr_rig_k * rig_tr_global_k[i])^-1 for every image i (image_used is not consulted); the
 *      centre c_k[i] = G_k[i].t = -R^T t of the composed pose.
 *   2. Scale: Umeyama with scaling from c_1 to c_2, in double (the reference runs it in float):
 *      s = lambda_max(N(S)) / sum_i |c_1[i] - mean c_1|^2, S = sum_i (c_2[i] - mean c_2)(c_1[i] - mean c_1)^T, where
 *      lambda_max(N(S)) is Horn's quaternion form of max over rotations R of tr(R^T S) (= Umeyama's tr(D S_sign)).
 *   3. Directions: every sample pixel (x + 0.5, y + 0.5), x = 0, step, ... < width, y likewise, that BOTH models
 *      un-project (Unproject(x, y, Line3d*): CG / NCG inside the calibrated area; OpenCV by the reference's
 *      UnprojectWithGaussNewton, parametric.h:60-148, whose iteration uses the exact derivative of the distortion);
 *      d_k = the unit line direction, normalised once more (origins are ignored). M = sum d1 d2^T on the device,
 *      one thread per sample pixel, summed in a fixed order (repeated calls give the same bits).
 *   4. R = intrinsics1_r_intrinsics2 = the exact minimiser of sum |R d2 - d1|^2 over rotations: the unit eigenvector
 *      of the largest eigenvalue of Horn's symmetric 4 x 4 matrix N(M) (cyclic Jacobi in double), as a rotation
 *      matrix. The reference reports the point where an LM run from the identity stops instead. rotation_cost is
 *      evaluated as direction_pairs - sum_ij R_ij M_ij, the identity for unit directions (absolute rounding error
 *      about direction_pairs * 2^-52).
 *   5. T = firstimage1_tr_firstimage2 = G1s[0].matrix() * [R 0; 0 1] * G2[0]^-1.matrix(), G1s = G_1 with its
 *      translations multiplied by s.
 *   6. endpoint_translation_difference e = |(T G2[n-1]).t - G1s[n-1].t|, evaluated as
 *      |R (R2_0^T (c_2[n-1] - c_2[0])) - s (R1_0^T (c_1[n-1] - c_1[0]))| with R_k0 the rotation of G_k[0]^-1 (the same
 *      number without forming T, so that two identical states give exactly 0); trajectory_length1 = sum_i
 *      |s c_1[i] - s c_1[i+1]|, trajectory_length2 = sum_i |c_2[i] - c_2[i+1]|; relative_endpoint_difference
 *      = e / (0.5 (trajectory_length1 + trajectory_length2)). */
typedef struct b200ba_reconstruction_comparison {
  int64_t direction_pairs;             /* sample pixels both models un-project */
  double direction_sums[9];            /* M = sum d1 d2^T, row-major */
  double intrinsics1_r_intrinsics2[9]; /* row-major: the minimiser of sum |R d2 - d1|^2 */
  double rotation_cost;                /* 1/2 sum |R d2 - d1|^2 at that R */
  double scale;                        /* s */
  double firstimage1_tr_firstimage2[16]; /* row-major 4 x 4 */
  double endpoint_translation_difference, trajectory_length1, trajectory_length2, relative_endpoint_difference;
} b200ba_reconstruction_comparison;
/* Stand-alone (allocates, computes, frees). cam1 / intr1 and cam2 / intr2: the single camera of each reconstruction,
 * central-generic, non-central-generic or central-OpenCV, of one image size. rig_tr_global1 / 2: [7 n_images];
 * camera_tr_rig1 / 2: [7]. device_ms (nullable): device time of the direction sweep. Returns 2 for a bad argument
 * before any CUDA call (a NULL pointer, another model type, a generic grid smaller than 4 x 4, different image sizes,
 * n_images < 2, pixel_step < 1, or all centres of one reconstruction equal: the reference divides by zero there),
 * 3 without a device, 4 when the rotation is not determined: fewer than two direction pairs or
 * lambda_1 - lambda_2 <= 64 * 2^-52 * |lambda_1| for the two largest eigenvalues of N(M) (this includes rank M < 2).
 * On 4, out holds the pairs and M. */
B200BA_API int b200ba_compare_reconstructions(int device, const b200ba_camera* cam1, const double* intr1,
                                              const b200ba_camera* cam2, const double* intr2, int32_t n_images,
                                              const double* rig_tr_global1, const double* camera_tr_rig1,
                                              const double* rig_tr_global2, const double* camera_tr_rig2,
                                              int32_t pixel_step, b200ba_reconstruction_comparison* out,
                                              double* device_ms);
/* The sample-pixel directions behind direction_sums, pixel by pixel (inspection and tests): for sample p = j nx + i,
 * nx = ceil(width / pixel_step), ok[2 p + k] = 1 where model k + 1 un-projects (step i + 0.5, step j + 0.5) and
 * directions[6 p + 3 k + c] its direction as step 3 defines it (0 otherwise). ok [2 nx ny], directions [6 nx ny].
 * The argument checks of b200ba_compare_reconstructions for the models and the step (2); 3 without a device. */
B200BA_API int b200ba_reconstruction_directions(int device, const b200ba_camera* cam1, const double* intr1,
                                                const b200ba_camera* cam2, const double* intr2, int32_t pixel_step,
                                                int32_t* ok, double* directions);
/* The host part of b200ba_compare_reconstructions (steps 1, 2 and 4-6) from given direction sums: fills every field
 * of out from direction_pairs and M [9]. Needs no device; returns 2 for a NULL pointer, n_images < 2 or coinciding
 * centres, 4 when the rotation is not determined (out then holds the pairs and M). */
B200BA_API int b200ba_reconstruction_alignment(int64_t direction_pairs, const double* direction_sums, int32_t n_images,
                                               const double* rig_tr_global1, const double* camera_tr_rig1,
                                               const double* rig_tr_global2, const double* camera_tr_rig2,
                                               b200ba_reconstruction_comparison* out);

/* ---- centre-point analysis of a non-central camera: the NoncentralGenericModel branch of
 * CreateCalibrationReportForCamera (APP/calibration_report.cc:839-982, with CenterPointCostFunction of :56-80).
 *   1. every pixel (x + 0.5f, y + 0.5f) of the calibrated area is un-projected to a line (o, d) (:847-856);
 *   2. the centre c closest to all lines: LMOptimizer<double>::Optimize(c = 0, max_iteration_count = 100,
 *      max_lm_attempts = 10, init_lambda = -1, init_lambda_factor = 0.001f) (:858-867) with two residuals per line,
 *      t1 . (c - o) and t2 . (c - o) in the line's tangent frame, quadratic loss (cost = 1/2 sum r^2);
 *   3. per line the offset closest - c, closest = o + (d . (c - o)) d, its norm (the line distance) and the largest
 *      |component| (:869-902); the statistics the reference computes but does not print (:904-911) are returned here;
 *   4. _line_offsets.png (:913-930): 127 + 127 * offset_k / max_line_offset_extent per channel in double, converted to
 *      u8 as x86-64 does (truncation to int32, low byte); black where there is no line;
 *   5. the lines of the .obj models (:932-973): every obj_step-th pixel from calibration_min in x and in y, half
 *      = max(10, 10 |closest - c|), point_a = closest + half d, point_b = closest - half d.
 * The model must be non-central-generic with grids of at least 4 x 4 and a calibrated area inside the image. */
typedef struct b200ba_line_offsets_report {
  double center[3];
  int64_t line_count;                      /* calibrated-area pixels whose Unproject succeeds */
  double line_distance_sum, line_distance_max, line_distance_median;  /* median NaN if count == 0 */
  double max_line_offset_extent;           /* max |component| of the offsets; 0 if none */
  double initial_cost, final_cost;         /* of the centre-point fit (quadratic loss: 1/2 sum r^2) */
  int32_t num_iterations_performed, lm_attempts;
} b200ba_line_offsets_report;
/* Stand-alone (allocates, computes, frees); intrinsics [6 * grid_width * grid_height] (direction grid, then point
 * grid) are not modified. image (nullable): [h*w*3] RGB row-major, _line_offsets.png. offsets (nullable): [3*w*h]
 * row-major (y, x), closest point on the line - centre, NaN where there is no line. obj_lines (nullable):
 * [n_obj][4][3] point_a, point_b, closest point, origin, in the reference's order (y outer, x inner); it must hold
 * ((max_x - min_x) / obj_step + 1) * ((max_y - min_y) / obj_step + 1) lines, and that count is written to n_obj
 * (nullable unless obj_lines is given). device_ms (nullable): device time of the analysis. Returns 2 for a bad
 * argument, 3 without a device. */
B200BA_API int b200ba_line_offsets(int device, const b200ba_camera* cam, const double* intrinsics,
                                   b200ba_line_offsets_report* report, uint8_t* image, double* offsets, int32_t obj_step,
                                   double* obj_lines, int64_t* n_obj, double* device_ms);

/* ---- feature intersection (APP/tools/intersect_datasets.cc:130-225, the feature level of --intersect_datasets):
 * of D feature lists of one (imageset, camera) -- one list per dataset, e.g. one per feature detector -- keep only the
 * features that every list detected. A "list" below is one such group of D lists (one per dataset); n_lists of them
 * are processed independently. thr2 = threshold * threshold in double (so a negative threshold acts as its absolute
 * value and a NaN threshold covers nothing). All coordinates are the given float xy.
 *   distance: d = (float)(x_o - c_x)^2 + (float)(y_o - c_y)^2 in float, each operation rounded on its own, compared
 *     with thr2 as a double.
 *   closest feature of dataset i to a centre c: the LAST index o, in list order among the features not yet erased,
 *     with d <= best, best starting at thr2 and taking every accepted d; so ties go to the later index, d == thr2 is
 *     covered and a NaN d never is. None (-1) where no d <= thr2.
 *   fixed-point loop of a centre: each pass finds the closest feature of every dataset, then sets the centre to the
 *     float sum of the covered features in dataset order divided by (float)count (0 / 0 = NaN when nothing is
 *     covered). It stops after the first pass whose covered-index vector equals the previous pass's (the first pass
 *     compares against an empty vector, so there are at least two passes), or after 100 passes, taking the 100th
 *     pass's result (the reference never ends on a loop that cycles without repeating its previous pass).
 *   walk: for f over dataset 0's features, from the feature's own xy: if every dataset covered a feature, the centre
 *     is accepted; otherwise every covered feature is erased and, where dataset 0 covered nothing (covered[0] == -1),
 *     the same f is walked again, else the next feature after f that is not erased. Accepted features stay and may be
 *     covered again by a later f.
 *   end: every feature whose distance to every accepted centre is > thr2 (or NaN) is erased.
 * Erasing only removes elements and keeps the order of the rest, so the walk is computed with one "alive" flag per
 * feature of the original order: the last index in list order is the last alive original index, and the next f is the
 * next alive feature after the current one. One rule of the reference never ends and is pinned here:
 *   - a rejected pass that covered nothing in any dataset (a feature with a NaN or infinite coordinate, a NaN
 *     threshold, or a centre that moved out of reach of everything) would re-run the same f forever; that f is
 *     rejected, left in place, and the walk moves on to the next feature. A rejection with covered[0] == -1 that
 *     erased features elsewhere is re-run as in the reference (it ends: every re-run erases at least one feature).
 * list_offsets [n_lists * D + 1]: list l, dataset i holds the features [list_offsets[l D + i], list_offsets[l D + i
 * + 1]) of xy [2 N] (x, y), N = list_offsets[n_lists D]; the offsets start at 0 and do not decrease, and one list
 * holds fewer than 2^31 features. The lists of one call must be independent (no feature in two lists); a caller with
 * tasks that share features runs them in order, one call after the other. keep [N]: 1 for a feature that survives,
 * else 0. report (nullable): the counts below. device_ms (nullable): device time of the intersection.
 * Stand-alone (allocates, computes, frees). Returns 2 for a bad argument before any CUDA call (n_datasets < 1 or
 * > 32, n_lists < 0 or >= 2^31, a NULL list_offsets, a NULL xy or keep with N > 0, offsets that do not start at 0 or
 * decrease, a list of 2^31 features or more), 3 without a device. Repeated calls give identical bytes. */
typedef struct b200ba_intersection_report {
  int64_t intersections;  /* accepted centres over all lists */
  int64_t kept;           /* features with keep == 1 */
  int64_t uncovered;      /* walks of a dataset-0 feature rejected with nothing covered, left in place (pinned above) */
  int64_t capped;         /* fixed-point loops stopped after 100 passes */
} b200ba_intersection_report;
B200BA_API int b200ba_intersect_features(int device, int32_t n_datasets, int64_t n_lists, const int64_t* list_offsets,
                                         const float* xy, double threshold, uint8_t* keep,
                                         b200ba_intersection_report* report, double* device_ms);

/* ---- synthetic calibration-pattern images (APP/tools/render_synthetic_dataset.cc, --render_synthetic_dataset): the
 * star pattern of a pattern YAML file (feature_detector_tagged_pattern.{h,cc}: PatternData) seen through a pinhole
 * camera from random poses, drawn with exact per-pixel area coverage so that the images carry no sampling bias.
 * All float operations below are rounded one by one in the order written (no fused multiply-add).
 *
 * The pattern. Its numbers are the floats the reference reads (`as<float>()`); at most B200BA_PATTERN_MAX_TAGS tags
 * are taken (more is refused with 2). pattern_w x pattern_h is the size of the pattern image (the PNG beside the
 * YAML file). A pattern coordinate c (features at integers) maps to pattern-image pixels (pixel-corner convention) as
 *   mm.x = start_x + ((c.x + 1) / (float)squares_x) * (end_x - start_x),  px.x = ((float)pattern_w / page_w) * mm.x
 * (y alike). The polygons are PatternData::ComputePatternGeometry without AprilTags, in generation order (features
 * y-major from (-1, -1), skipping features inside a tag, the black segments 0, 2, ... of each star whose middle
 * direction lies in the repeating area), each vertex mapped as above and lifted to z = 0. The star corners are
 * computed on the host with the C library's float sin / cos, as the reference computes them. Every polygon has 3 or 4
 * vertices. */
#define B200BA_PATTERN_MAX_TAGS 16
typedef struct b200ba_pattern_tag {
  int32_t x, y, width, height, index; /* tag_x, tag_y (squares), width, height (squares), index in its family */
} b200ba_pattern_tag;
typedef struct b200ba_pattern {
  int32_t squares_x, squares_y, num_star_segments, num_tags;
  float page_width_mm, page_height_mm, pattern_start_x_mm, pattern_start_y_mm, pattern_end_x_mm, pattern_end_y_mm;
  b200ba_pattern_tag tags[B200BA_PATTERN_MAX_TAGS];
} b200ba_pattern;
/* Poses (host only; the Python and C++ tools both call this). camera_tr_global [n][12]: the row-major rotation R
 * and the translation t of camera <- pattern, in double. Image i, attempt a (a = 0, 1, ...) draws from the stream of
 * b200ba_localization_accuracy with key = (i << 24) | (a << 4) | component, h = SplitMix64(SplitMix64(seed) ^ key):
 *   components 0-2: f_k = (float)(h_k % 10000) / 10000.f;
 *     t0 = (0.0 - (double)((-1.f + 2.f * f_0) * (float)pattern_w), 0.0 - (double)((-1.f + 2.f * f_1) *
 *          (float)pattern_h), 0.0 + (double)(500.f + 800.f * f_2));
 *   components 3-8: r_k = -1.0 + 2.0 * ((double)(h_k >> 11) * 2^-53) in [-1, 1); the tangent is
 *     (u, w) = 0.5 * (r_3 .. r_5, r_6 .. r_8) (Sophus order: translation part first).
 *   Sophus' SE3d::exp, in double with the C library's sin / cos: th2 = (wx wx + wy wy) + wz wz, th = sqrt(th2);
 *     th < 1e-10: im = (0.5 - (1/48) th2) + (1/3840) th2^2, re = (1 - 0.5 th2) + (1/384) th2^2, else
 *     im = sin(th / 2) / th, re = cos(th / 2) (th / 2 as 0.5 * th); q = (re, im wx, im wy, im wz);
 *     W = hat(w), W2 = W W (each entry a sum over k = 0, 1, 2 in order); V = rotation(q) when th < 1e-10, else
 *     (I + ((1 - cos th) / th2) W) + ((th - sin th) / (th2 th)) W2; t_exp = V u (each row (a0 u0 + a1 u1) + a2 u2).
 *   The pose is exp(tangent) * (I, t0) as Sophus composes it: t = t_exp + q.v where q.v = (v + re uv) + im_vec x uv,
 *     uv = 2 (im_vec x v) (Eigen's _transformVector, with the un-normalised q); then q is renormalised as SO3's *=:
 *     s = (x^2 + z^2) + (y^2 + w^2), q *= 2 / (1 + s) unless s == 1; R = rotation(q) with Eigen's toRotationMatrix
 *     (tx = 2x, twx = tx w, txx = tx x, ..., R00 = 1 - (tyy + tzz), R01 = txy - twz, ...).
 *   The pose is taken when, for some tag, the four corners of the tag's square (pattern coordinates (tag.x - 1,
 *   tag.y - 1) and (tag.x - 1 + width, tag.y - 1 + height), mapped as above) are all visible with border 0 to the
 *   float pose Rf = (float)R, tf = (float)t: p_cam_i = ((Rf_i0 x + Rf_i1 y) + Rf_i2 z) + tf_i, p_cam_z > 0 and the
 *   pixel (fx (p_cam_x / p_cam_z) + cx, fy (p_cam_y / p_cam_z) + cy) inside [0, width) x [0, height). Otherwise the
 *   attempt is drawn again. attempts (nullable): [n] the number of attempts of every image.
 * Worked examples (the fixture pattern of tests/golden/pattern, 1124 x 1590, 640 x 480, fx = fy = 480, cx = 320,
 * cy = 240):
 *   seed 0, image 0: attempt 0 has h_0 = 0xa706dd2f4d197e6f (k = 7055); 11 attempts show no whole tag; attempt 11
 *     (h_0 = 0x89c20cbbf41b13e7, k = 7431) is taken with t = (-88.31650879202545, -535.3216881191287,
 *     1468.5512805064373), R_00 = 0.9036277796763321;
 *   seed 7, image 3: attempt 0 (h_0 = 0x18080193089f89c2, k = 9218; h_3 = 0xfc9ef4a796148570) is taken with
 *     t = (-928.6952246323646, -359.4073177209594, 1231.647888783845), R_00 = 0.9714992824303272.
 * Returns 2 for a bad argument (NULL pointers, sizes below 1 or above 2^15, n < 1 or n >= 2^40, and the pattern and
 * camera checks of b200ba_render_pattern_images below), 4 when an image has no visible tag
 * after 4096 attempts (the reference would draw forever; camera_tr_global then holds the images before it).
 * The reference seeds rand() with the time and draws Eigen / Sophus Random(); this stream is seeded and repeatable. */
B200BA_API int b200ba_synthetic_poses(const b200ba_pattern* pattern, int32_t pattern_w, int32_t pattern_h,
                                      int32_t width, int32_t height, const float* fx_fy_cx_cy, int64_t n,
                                      uint64_t seed, double* camera_tr_global, int64_t* attempts);
/* Images. images [n][height][width] u8, one per pose of camera_tr_global [n][12] (as above). The float pose is
 * Rf = (float)R, tf = (float)t; the inverse is taken in double, R^T and ti = R^T (-t) (row i: (R_0i (-t0) +
 * R_1i (-t1)) + R_2i (-t2)), and cast to float afterwards (Rc, tc).
 *   Coverage (:202-243): a float image set to 1. For every polygon in generation order, every vertex p is projected
 *     in float (p_cam_i = ((Rf_i0 p.x + Rf_i1 p.y) + Rf_i2 p.z) + tf_i, pixel = (fx (p_cam_x / p_cam_z) + cx,
 *     fy (p_cam_y / p_cam_z) + cy)) and cast to double, without a visibility test: a vertex behind the camera is
 *     projected through its negative depth, exactly as the reference does. The pixel range is the bounding box
 *     of the vertices, converted to int as x86-64 does (truncation toward zero; INT_MIN for values outside the int
 *     range and for +-inf, so that a box reaching beyond 2^31 in x or y draws nothing and one reaching below -2^31
 *     starts at 0), clamped to [0, width - 1] x [0, height - 1]. A polygon with a NaN projected coordinate draws
 *     nothing (the pinned case; it needs p_cam_z == 0 and p_cam_x == 0 or p_cam_y == 0). For every pixel (x, y) of
 *     the range, rendering(x, y) = (float)((double)rendering(x, y) - A), A = libvis' PolygonArea of libvis'
 *     ConvexClipPolygon of the projected polygon against the pixel square (x, y), (x + 1, y), (x + 1, y + 1),
 *     (x, y + 1), in double, with its float edge offset and its IEEE comparisons (a NaN vertex counts as inside)
 *     and LineLineIntersection's result (the previous vertex where its denominator is 0, else the quotients, even
 *     non-finite ones); PolygonArea = |0.5 * sum_i (x_i - x_{i-1})
 *     (y_i + y_{i-1})| summed from i = 0 with i - 1 = last.
 *   Composition (:248-291): per pixel, the ray of (x + 0.5f, y + 0.5f) is d = Rc (x' , y', 1) with
 *     x' = (1.f / fx) (x + 0.5f) + (-cx / fx) (y alike; rows (a0 x' + a1 y') + a2), normalised as Eigen does
 *     (n2 = (dx dx + dy dy) + dz dz, d / sqrtf(n2) when n2 > 0), and meets the plane z = 0 (normal (0, 0, -1),
 *     offset -0.f) at t = -(offset + ((0 tx + 0 ty) + -1 tz)) / ((0 dx + 0 dy) + -1 dz), point = tc + d t
 *     (Eigen's ParametrizedLine::intersectionPoint). Its pattern-image coordinate is (1 (X - 0) + 0 (Y + 0), 0 (X - 0)
 *     + 1 (Y + 0)) (the normalised image axes), mm = (page_w / (float)pattern_w) * that, pattern coordinate =
 *     ((mm - start) / (end - start)) * (float)squares - 1. Inside IsValidPatternCoord (in [-1, squares - 1] and in
 *     no tag's [tag - 1, tag - 1 + size] box) the byte is u8(max(0.f, 255.99f * rendering)); else, at c = coordinate
 *     - 0.5f, if 0 <= c < (float)(pattern size - 1) it is libvis' InterpolateBilinear<float> of the pattern image
 *     (i = (int)c, f = c - i, (((1 - fx)(1 - fy)) p00 + (fx (1 - fy)) p10) + ((1 - fx) fy) p01) + (fx fy) p11),
 *     and 0 otherwise. u8(v) is static_cast<int>(v) as x86-64 executes it (truncation; INT_MIN for NaN, hence 0)
 *     reduced to its low byte.
 * pattern_image [pattern_h][pattern_w] grey u8. Images are rendered in chunks bounded in device memory (about
 * 512 MiB; the environment variable B200BA_SYNTH_CHUNK lowers the images per chunk), so any n works; the bytes do not
 * depend on the chunking. device_ms (nullable): device time of the rendering.
 * Stand-alone (allocates, computes, frees). Returns 2 for a bad argument before any CUDA call (NULL pointers, a
 * size below 1 or above 2^15, n < 0, num_tags outside [0, B200BA_PATTERN_MAX_TAGS], squares below 1,
 * num_star_segments below 2, odd or above 1024, more than 2^24 star segments ((squares_x + 1) (squares_y + 1)
 * num_star_segments / 2), a non-finite or zero focal length, a non-finite principal point), 3 without a device. Repeated calls give identical bytes. */
B200BA_API int b200ba_render_pattern_images(int device, const b200ba_pattern* pattern, const uint8_t* pattern_image,
                                            int32_t pattern_w, int32_t pattern_h, int32_t width, int32_t height,
                                            const float* fx_fy_cx_cy, int64_t n, const double* camera_tr_global,
                                            uint8_t* images, double* device_ms);

/* ---- sub-pixel refinement of star-pattern features (APP/feature_detection/feature_detector_tagged_pattern.cc:
 * 1427-1648, FeatureDetectorTaggedPattern::RefineFeatureDetections with the CPU path of
 * cpu_refinement_by_matching.h and cpu_refinement_by_symmetry.h). Every float operation below is rounded on its own
 * in the order written (no fused multiply-add); "(float)", "(double)" and "(int)" are C conversions ((int)
 * truncates; outside the int range and for NaN it gives INT_MIN, as x86-64 does).
 *
 * Samples (feature_detector_tagged_pattern.cc:239-248): n = (int)(8.0 * (2h + 1)^2 + 0.5) offsets in [-1, 1]^2,
 * h = window_half_extent. The reference calls srand(0) and then Vec2f::Random() per sample, x then y, each
 * coordinate -1.f + (2.f * (float)r) / (float)RAND_MAX (Eigen 3.3's float Random()) with r the next value of glibc's
 * rand(): the TYPE_3 additive generator of random_r (31 words, separation 3, seeded as srandom(1) because seed 0 is
 * taken as 1, 310 values discarded), restated here so that the samples do not depend on the platform's rand(). The
 * first sample is (0.68037546, -0.21123415). Matching uses the first n_m = (int)((1 / 8.) * n) = (2h + 1)^2
 * samples, symmetry all n. */
#define B200BA_REFINE_MAX_HALF_EXTENT 32
/* Returns 2 unless 1 <= window_half_extent <= B200BA_REFINE_MAX_HALF_EXTENT, n equals the count above and xy
 * ([n][2]) is given. Host only. */
B200BA_API int b200ba_feature_samples(int32_t window_half_extent, int32_t n, float* xy);

/* The refinement types, numbered as the reference's FeatureRefinement enum. */
#define B200BA_REFINE_GRADIENTS_XY 0
#define B200BA_REFINE_GRADIENT_MAGNITUDE 1
#define B200BA_REFINE_INTENSITIES 2
#define B200BA_REFINE_NO_REFINEMENT 3
/* Per-feature status: why a feature was rejected (final_cost -1, position NaN), or 0. */
#define B200BA_REFINE_ACCEPTED 0
#define B200BA_REFINE_IMAGE_BORDER 1        /* the window around the prediction leaves the image (:1448-1455) */
#define B200BA_REFINE_OUTSIDE_PATTERN 2     /* a window corner leaves the repeating pattern area (:1457-1474) */
#define B200BA_REFINE_MATCH_OUTSIDE 3       /* matching: a sample left the image (in a trial step) */
#define B200BA_REFINE_MATCH_LEFT_WINDOW 4   /* matching: the position moved >= h from the prediction */
#define B200BA_REFINE_MATCH_NOT_CONVERGED 5 /* matching: 50 iterations and a last step with |x|^2 >= 1e-8 */
#define B200BA_REFINE_MATCH_BAD_FACTOR 6    /* matching: the affine intensity factor is <= 0 */
#define B200BA_REFINE_SYM_OUTSIDE 7         /* symmetry: a sample left the image */
#define B200BA_REFINE_SYM_LEFT_WINDOW 8     /* symmetry: the position moved >= h from the matching result */
#define B200BA_REFINE_SYM_NOT_CONVERGED 9   /* symmetry: 30 iterations and a last translation step >= 1e-4f */
#define B200BA_REFINE_INCONSISTENT 10       /* symmetry and matching results lie more than 0.75 px^2 apart */
/* One predicted feature (the reference's FeatureDetection plus its image). position: pixel-centre convention
 * (pixel (0, 0)'s centre is (0, 0)). local_pixel_tr_pattern: row-major; it maps the local pattern coordinate
 * (0 at the feature, one unit per square) to the pixel offset from the feature. */
typedef struct b200ba_feature_prediction {
  int64_t image;                   /* index into images */
  float position[2];               /* x, y */
  int32_t pattern_coordinate[2];   /* the feature's integer pattern coordinate */
  float local_pixel_tr_pattern[9];
} b200ba_feature_prediction;
/* Refines every prediction, with the arithmetic of the reference's CPU path:
 *   Images: images [n_images][height][width] grey u8 (all one size). Bilinear interpolation (libvis'
 *     InterpolateBilinear / ...WithJacobian) at p: i = (int)p.x, j = (int)p.y, fx = p.x - (float)i, gx = 1 - fx
 *     (y alike); value = (((gx gy) v00 + (fx gy) v10) + (gx fy) v01) + (fx fy) v11; with the Jacobian instead
 *     top = gx v00 + fx v10, bottom = gx v01 + fx v11, value = gy top + fy bottom, d/dx = fy (v11 - v01) +
 *     gy (v10 - v00), d/dy = bottom - top, where for u8 images the differences are int subtractions converted to
 *     float. Gradient images are not stored: the pixel (x, y) of the gradient image is dx = ((float)I(x+, y) -
 *     (float)I(x-, y)) / (float)(x+ - x-) with x- = max(0, x - 1), x+ = min(W - 1, x + 1) (dy alike) and the
 *     gradient magnitude is sqrtf(dx dx + dy dy). A position p is inside when p.x >= 0, p.y >= 0,
 *     p.x < (float)(W - 1), p.y < (float)(H - 1).
 *   Pre-filter (:1443-1479): a prediction p passes when p.x - h >= 0, p.y - h >= 0, p.x + h < (float)(W - 1) and
 *     p.y + h < (float)(H - 1) (each in float), else status IMAGE_BORDER; then local_pattern_tr_pixel = the inverse
 *     of local_pixel_tr_pattern (rf_inverse3 of camera_calibration_b200/csrc/ba_common.h: the adjugate times
 *     1 / det), and each window corner c = (+-h, +-h) (corner k: x sign + for even k, y sign + for k < 2) maps to
 *     the pattern as hnorm(M (c, 1)) (rows ((m0 c.x + m1 c.y) + m2), hnorm divides x and y by z) plus
 *     (float)pattern_coordinate; it must satisfy PatternData::IsValidPatternCoord (in [-1, squares - 1] and in no
 *     tag's [tag - 1, tag - 1 + size] box), else status OUTSIDE_PATTERN.
 *   Matching (cpu_refinement_by_matching.h:232-417), on the u8 image with the first n_m samples s_i:
 *     template q_i = sum over k = 0..15 (in order, from 0.f) of PatternIntensityAt(hnorm(M (h s_i + o_k, 1))),
 *       o_k = (-0.375 + 0.25 (k % 4), -0.375 + 0.25 (k / 4)), h s_i = ((float)h s_i.x, (float)h s_i.y);
 *       PatternIntensityAt(p): c.x = p.x - (float)(sgn (int)(|p.x| + 0.5f)) with sgn = 1 for p.x > 0, else -1 (y
 *       alike); 0.5f when c.x c.x + c.y c.y < 1e-8f; else a = (float)((double)rf_atan2(c.y, c.x) - pi / 2),
 *       a = (float)((double)a + 2 pi) when a < 0, and 1.f when (int)((double)((float)num_star_segments * a) /
 *       (2 pi)) is even, else 0.f.
 *     sample positions are position + (float)h s_i (x and y each one addition); factor and bias start at
 *       factor = (S_qp - (S_p / n_m) S_q) / D when |D| > 1e-6f with D = S_pp - (S_p S_p) / n_m, else 1; bias =
 *       (1.f / n_m) (S_q - factor S_p); S_* are the sums of q p, p, q, p p over the samples (p the interpolated
 *       value) and n_m is converted to float.
 *     LM on (x, y, factor, bias), at most 50 iterations: residual r = (factor I + bias) - q_i, Jacobian
 *       (factor dI/dx, factor dI/dy, I, 1); H += J^T J (upper triangle, each entry J_a J_b added), b += r J,
 *       cost += r r. lambda = (0.001f * 0.5f) * (((H00 + H11) + H22) + H33) on the first iteration. Up to 10
 *       attempts: x = rf_ldlt_solve<4>(H, lambda, b) (ba_common.h: unpivoted LDL^T in double, a zero pivot's
 *       solution component set to 0 as Eigen's LDLT sets it); the trial is
 *       position - x[0..1], factor - x2, bias - x3; its cost (the sum of r r) below the current cost accepts it
 *       (last step = ((x0 x0 + x1 x1) + x2 x2) + x3 x3, lambda *= 0.5f), else lambda *= 2.f. No accepted
 *       attempt ends the loop as converged. After an accepted step, |x - x0| >= h or |y - y0| >= h (float, from
 *       the prediction) rejects with MATCH_LEFT_WINDOW. After the loop, not converged and (double)last >= 1e-8
 *       rejects with MATCH_NOT_CONVERGED, then factor <= 0 with MATCH_BAD_FACTOR. A sample outside the image in
 *       any cost evaluation rejects with MATCH_OUTSIDE.
 *   Symmetry (cpu_refinement_by_symmetry.h:40-580), skipped for NO_REFINEMENT (final_cost 0): the pattern
 *     samples are t_i = hnorm(M ((float)h s_i, 1)) for all n samples; P = T(m) * local_pixel_tr_pattern (each entry
 *     (T_r0 L_0c + T_r1 L_1c) + T_r2 L_2c, T = [1 0 m.x; 0 1 m.y; 0 0 1], m the matching result), then every entry
 *     divided by P22. Per sample a = hnorm(P (t_i, 1)) and b = hnorm(P (-t_i, 1)); both must be inside
 *     (SYM_OUTSIDE). INTENSITIES (u8 image) and GRADIENT_MAGNITUDE (gradient-magnitude image): r = I(a) - I(b),
 *     J = grad I(a) * D(a) - grad I(b) * D(b); GRADIENTS_XY (gradient image): r = g(a) + g(b) (2-vector),
 *     J = Grad g(a) D(a) + Grad g(b) D(b) (each entry (G_r0 D_0c + G_r1 D_1c)), its two rows added in turn. D(t) is
 *     d hnorm(P (t, 1)) / d(P00 P01 P02 P10 P11 P12 P20 P21): e0 = 1 / ((P20 t.x + P21 t.y) + 1), e1 = (-1 e0) e0,
 *     e2 = ((P00 t.x + P01 t.y) + P02) e1, e3 = ((P10 t.x + P11 t.y) + P12) e1; row 0 = (t.x e0, t.y e0, e0, 0, 0,
 *     0, t.x e2, t.y e2), row 1 = (0, 0, 0, t.x e0, t.y e0, e0, t.x e3, t.y e3). H += J^T J, b += r J, cost +=
 *     r r (r.x r.x + r.y r.y for GRADIENTS_XY). LM: at most 30 iterations, lambda = (0.001f * (1.f / 8)) *
 *     (diagonal sum, index order) on the first; up to 10 attempts of x = rf_ldlt_solve<8>, P - x (P22 kept),
 *     (a textureless window makes H = 0 and lambda = 0; the zero pivots give x = 0, so the LM ends converged at m
 *     with final_cost 0, as the reference's does),
 *     accepted when the trial cost is lower (last step = x2 x2 + x5 x5, lambda *= 0.5f, position = (P02, P12)),
 *     else lambda *= 2.f; no accepted attempt ends as converged; an accepted step with |P02 - m.x| >= h or
 *     |P12 - m.y| >= h rejects with SYM_LEFT_WINDOW; 30 iterations end converged only when last step < 1e-4f, else
 *     SYM_NOT_CONVERGED. final_cost is the cost at the result.
 *   Final test (:1626-1647): (dx dx + dy dy) > 0.75f between the symmetry and the matching result rejects with
 *     INCONSISTENT.
 *   Sums: every sum above over samples is taken in one order, that of one warp: lane l (0..31) adds samples l,
 *     l + 32, l + 64, ... in order into its own float accumulator (from 0.f), then the 32 lane values are
 *     combined by butterflies v_l = v_l + v_(l xor o) for o = 16, 8, 4, 2, 1. The reference adds into one running
 *     float sum per accumulator instead; the difference this order makes is stated in DESIGN.md section 7.
 *   Pinned here: the reference's pattern is d->patterns[0], one per call; its CUDA path handles at most 128
 *     features per call and only GRADIENTS_XY and INTENSITIES, neither applies. The LDL^T is unpivoted (Eigen's
 *     pivots), and the inverse and atan2 are this library's (ba_common.h).
 * Outputs: xy [n_features][2] (NaN for a rejected feature), final_cost [n_features] (-1 for a rejected feature;
 * the reference leaves a rejected feature's position partly written), status [n_features] (nullable), device_ms
 * (nullable): device time of the refinement kernels, without the uploads. samples: [n_samples][2], normally
 * b200ba_feature_samples(window_half_extent); callers may pass their own. Images go to the device in chunks bounded
 * in device memory (about 512 MiB; the environment variable B200BA_REFINE_CHUNK lowers the images per chunk), and the
 * features of a chunk in launches of at most 2^20 (80 bytes of device memory each), so any number of images and
 * features works; the outputs do not depend on the chunking or on the order of the features.
 * Stand-alone (allocates, computes, frees). Returns 2 for a bad argument before any CUDA call: NULL pointers, width
 * or height below 1 or above 2^15, n_images < 0, n_features < 0, the pattern checks of
 * b200ba_render_pattern_images, window_half_extent outside [1, B200BA_REFINE_MAX_HALF_EXTENT], n_samples other than
 * the count for it, an unknown refinement_type, an image index outside [0, n_images), a non-finite
 * local_pixel_tr_pattern entry. Returns 3 without a device. */
B200BA_API int b200ba_refine_features(int device, const b200ba_pattern* pattern, const uint8_t* images, int32_t width,
                                      int32_t height, int64_t n_images, const float* samples, int32_t n_samples,
                                      int32_t window_half_extent, int32_t refinement_type, int64_t n_features,
                                      const b200ba_feature_prediction* predictions, float* xy, float* final_cost,
                                      int32_t* status, double* device_ms);

/* ---- multi-GPU: imagesets sharded over ranks, one NCCL all-reduce per H/b build --- */
#define B200BA_NCCL_UNIQUE_ID_BYTES 128
B200BA_API int b200ba_nccl_unique_id(uint8_t id[B200BA_NCCL_UNIQUE_ID_BYTES]);
/* Every rank creates its handle from ITS shard of the observations (all ranks use the
 * same n_imagesets / n_points / cameras) and then joins the communicator. After that
 * b200ba_optimize / b200ba_optimize_host / b200ba_build_system are COLLECTIVE: every rank must
 * issue the same sequence of them with the same options. The first call after
 * b200ba_comm_init that needs the device layout (any of the above or b200ba_evaluate) also
 * all-reduces the bookkeeping that makes the ranks group the Schur blocks identically, so it
 * must be made by every rank too; later b200ba_evaluate / b200ba_get_state /
 * b200ba_get_jacobians calls are rank-local. */
B200BA_API int b200ba_comm_init(b200ba_handle* h, const uint8_t id[B200BA_NCCL_UNIQUE_ID_BYTES], int rank,
                     int n_ranks);

/* ---- instrumentation ------------------------------------------------------ */
/* Device-side timings (CUDA events on the handle's stream) of the last b200ba_optimize. */
typedef struct b200ba_timings {
  double jacobian_kernel_ms; /* sum over launches of the MAIN pass of the residual+Jacobian kernel */
  int32_t jacobian_kernel_launches;
  double accumulate_ms;      /* JtJ / Jtr accumulation kernels */
  double schur_ms;           /* D^-1, D^-1 B, B^T D^-1 B contraction */
  double factor_ms;          /* dense SPD factorisation + solves */
  double trial_cost_ms;      /* residual-only passes + comparison */
  double update_ms;          /* state retraction */
  double allreduce_ms;
  double total_ms;
  int64_t kernel_launches;   /* kernels of this library launched */
  double straggler_ms;       /* straggler passes of the residual/Jacobian kernel (observations whose
                                projection needs more than the main pass's evaluation budget) */
  double solve_ms;           /* triangular solves with the dense factor (part of factor_ms) */
  double contraction_flops;  /* FP64 flops of the Schur contraction S = C - W^T W actually issued (structured:
                                sum over groups of m_g^2 k_g; dense: n_d^2 * k), summed over LM attempts */
  double factor_flops;       /* n_d^3 / 3 per factorisation, summed over LM attempts */
  int32_t lm_attempts;       /* linear solves (LM attempts) of the last b200ba_optimize */
  int32_t build_count;       /* H / b builds (outer iterations) of the last b200ba_optimize */
} b200ba_timings;
B200BA_API int b200ba_get_timings(const b200ba_handle* h, b200ba_timings* t);

B200BA_API const char* b200ba_version(void);

/* ---- diagnostics (not part of the reference interface) ---------------------------------
 * Evaluation budget of the main residual/Jacobian pass (default 16 spline evaluations per
 * observation; what exceeds it is redone by the straggler pass). 1 sends every observation of
 * a generic camera through the straggler pass (tests). Process-wide. */
B200BA_API void b200ba_debug_set_eval_budget(int budget);
/* Spline evaluations the projection LM spent per observation in the last pass that wrote
 * Jacobians; counts [n_obs], caller's observation order. */
B200BA_API int b200ba_debug_eval_counts(b200ba_handle* h, uint16_t* counts);
/* One LM attempt's linear solve at the current state, with its intermediates: builds H, b (with the
 * debug_fix_* masks of opt) and solves (H + lambda I) x = b with the kernels b200ba_optimize uses
 * (B200BA_DENSE selects the in-tree or the cuBLAS / cuSOLVER dense phase). lambda < 0 means the LM's
 * first lambda, init_lambda_factor * trace(H) / dof. n = the number of unknowns. Outputs (host):
 *   H [n*n], b [n]   nullable; as b200ba_build_system returns them, from the same build
 *   S [n_d*n_d]      the reduced system C + lambda I - B^T (D + lambda I)^-1 B as the factorisation
 *                    receives it; column-major, lower triangle
 *   rhs [n_d]        the reduced right-hand side b_d - B^T (D + lambda I)^-1 b_p
 *   x [n]            the update, in b200ba_build_system's variable order
 *   lambda_used      nullable
 *   info [8]         positive definite (1 / 0), grouped contraction used, number of groups, and the
 *                    dense-phase variants in effect: GEMM tile (64 | 128 | 12816), panel version,
 *                    triangular-solve version, aux stream (1 / 0), block width (0 on the library path)
 * n_d = n minus the unknowns of the eliminated blocks (points, or poses without eliminate_points).
 * Returns 2 for a handle joined to a communicator. */
B200BA_API int b200ba_debug_solve_step(b200ba_handle* h, const b200ba_options* opt, double lambda, int32_t n,
                                       double* H, double* b, double* S, double* rhs, double* x,
                                       double* lambda_used, int32_t info[8]);
/* The retraction of one LM attempt (the reference's JointOptimizationState::operator-=) with the
 * caller's update x [n] (n = the number of unknowns, b200ba_build_system's variable order), from the
 * current state into the trial slot; the trial state is downloaded into out (last_projection is not
 * written). The current state is not changed. */
B200BA_API int b200ba_debug_apply_update(b200ba_handle* h, const b200ba_options* opt, const double* x, int32_t n,
                                         b200ba_state* out);
/* The LM's cost comparison (CostIsSmallerThan) and totals, on the caller's arrays: trial [n], base [n]
 * (nullable), residual [2n] as all x then all y (nullable); a negative cost marks an invalid residual.
 * out [6]: trial sum and base sum over the residuals valid in both, their count, total trial cost,
 * number of valid trial residuals, sum |r|^2 over those. Stand-alone; returns 3 without a device. */
B200BA_API int b200ba_debug_cost_compare(int device, int64_t n, const double* trial, const double* base,
                                         const double* residual, double out[6]);
/* ChooseNiceCameraOrientation applied to every camera of the current state, as
 * b200ba_run_bundle_adjustment does after each iteration (grids and camera_tr_rig are rotated);
 * rot [9 * n_cameras] receives each rotation, row-major (the identity for models other than
 * central-generic). */
B200BA_API int b200ba_debug_nice_orientation(b200ba_handle* h, double* rot);
/* Outcome of each LM attempt of the last b200ba_optimize, in order, over all its iterations. */
#define B200BA_LM_ACCEPTED 1       /* cost comparison accepted the update */
#define B200BA_LM_REJECTED_COST 2  /* cost comparison rejected the update */
#define B200BA_LM_REFUSED_PIVOT 3  /* factorisation met a non-positive pivot; the update was not evaluated */
/* Copies up to cap codes; returns the number of attempts (-1 for a NULL handle). */
B200BA_API int32_t b200ba_debug_lm_events(const b200ba_handle* h, int32_t* codes, int32_t cap);

#ifdef __cplusplus
}
#endif
#endif /* B200BA_H_ */
