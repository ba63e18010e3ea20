/*
 * ba_oracle.h -- C interface of the CPU oracle.
 *
 * TEST INFRASTRUCTURE ONLY. This is a dependency-free CPU restatement of the
 * reference's joint-optimisation path (puzzlepaint/camera_calibration,
 * OptimizeJointly and everything below it). Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it; the product
 * (camera_calibration_b200/) never does.
 *
 * Parity pinning: the reference itself cannot be built here (Eigen, Qt5, Boost,
 * OpenGV are absent -- SURVEY.md F9), so this restatement is pinned to the
 * reference through the known-answer vectors and thresholds of the reference's
 * own tests (tests/test_oracle_golden.py lists them with file:line).
 *
 * The POD types are those of the product's C ABI (include/b200ba.h) so that the
 * same flattened problem can be handed to both sides.
 */
#ifndef BA_ORACLE_H_
#define BA_ORACLE_H_

#include "../include/b200ba.h"

#ifdef __cplusplus
extern "C" {
#endif

/* OptimizeJointly (joint_optimization.cc:757-953). state is in/out. */
int oracle_optimize(const b200ba_problem* problem, b200ba_state* state,
                    const b200ba_options* opt, b200ba_report* report);
/* Outcome of each LM attempt of the last oracle_optimize (B200BA_LM_*; an update with a NaN is
 * B200BA_LM_REFUSED_PIVOT). Copies up to cap codes; returns the number of attempts. */
int32_t oracle_lm_events(int32_t* codes, int32_t cap);

/* JointOptimizationCostFunction::Compute<compute_jacobians> (joint_optimization.cc:240-306).
 * Outputs are nullable. Jacobian outputs as in b200ba_get_jacobians(); has_jacobian[i]=0
 * when the observation contributed its residual only (joint_optimization.cc:373-376,446-448). */
int oracle_evaluate(const b200ba_problem* problem, b200ba_state* state, const b200ba_options* opt,
                    int compute_jacobians, double* residuals, double* costs, double* total_cost,
                    double* j_point, double* j_pose, double* j_rig, double* j_intr,
                    int32_t* intr_index, int32_t K, int32_t* has_jacobian);

/* H (upper triangle, dense n*n row-major, reference variable ordering) and b. */
int oracle_build_system(const b200ba_problem* problem, b200ba_state* state,
                        const b200ba_options* opt, int32_t n, double* H, double* b, double* cost);
int32_t oracle_degrees_of_freedom(const b200ba_problem* problem, const b200ba_options* opt);

/* SolveWithSchurComplementDenseOffDiag (libvis lm_optimizer.h:1246-1369). */
int oracle_schur_solve(int32_t block_size, int32_t n_blocks, int32_t n_dense, const double* D,
                       const double* B, const double* C, const double* b1, const double* b2,
                       double* x);
/* LDLT(H.selfadjointView<Upper>()).solve(b) (libvis lm_optimizer.h:1022-1023). */
int oracle_solve_dense(int32_t n, const double* H, const double* b, double* x);

/* JointOptimizationState::operator-= (joint_optimization.cc:172-214). */
int oracle_apply_update(const b200ba_problem* problem, b200ba_state* state,
                        const b200ba_options* opt, const double* delta);

/* CameraModel::ProjectWithInitialEstimate / Unproject / UnprojectWithJacobian. */
int oracle_project(const b200ba_camera* cam, const double* intrinsics, int64_t n,
                   const double* local_points, double* pixels, int32_t* ok);
int oracle_unproject(const b200ba_camera* cam, const double* intrinsics, int64_t n,
                     const double* pixels, double* directions, double* origins, int32_t* ok);
/* jac: central [n*3*2] (d dir / d pixel), noncentral [n*6*2] (direction rows first). */
int oracle_unproject_jacobian(const b200ba_camera* cam, const double* intrinsics, int64_t n,
                              const double* pixels, double* directions, double* origins,
                              double* jac, int32_t* ok);

/* CentralGenericModel::FitToPixelDirectionsImpl (APP/models/central_generic.cc:551-568); the
 * arguments of b200ba_fit_directions. */
int oracle_fit_directions(int32_t grid_width, int32_t grid_height, double* grid, int64_t n,
                          const double* grid_points, const double* directions,
                          int32_t max_iteration_count, b200ba_fit_report* report);

/* b_spline.h: fast (EvalUniformCubicBSplineSurface :65-104) and slow (:168-186) evaluation
 * of a 3-vector grid at grid coordinates (x, y). */
int oracle_bspline_eval(int32_t gw, int32_t gh, const double* grid, double x, double y, int slow,
                        double out[3]);

/* HuberLoss (libvis loss_functions.h:94-133). */
double oracle_huber_cost(double huber, double residual);
double oracle_huber_weight(double huber, double residual);
double oracle_huber_cost_sq(double huber, double squared_residual);
double oracle_huber_weight_sq(double huber, double squared_residual);

/* CPU-baseline timing on a bounded sample (bench.py). Returns seconds, < 0 on error.
 *  - jacobian: one Compute<true> over the imagesets [first, first+count) accumulating into
 *    a private small system (the accumulation cost is included, the matrices are discarded);
 *  - residual: one Compute<false> over the same range;
 *  - contraction: B^T D^-1 B restricted to n_cols dense columns of a (3*n_points x n_cols) B;
 *  - ldlt: pivoted LDLT of an n x n SPD matrix + solve. */
double oracle_time_jacobian(const b200ba_problem* problem, b200ba_state* state,
                            const b200ba_options* opt, int32_t first_imageset, int32_t count,
                            int compute_jacobians);
double oracle_time_contraction(int32_t n_rows, int32_t n_cols);
double oracle_time_ldlt(int32_t n);

/* Full-size runs (bench.py --impl reference / cpu_baseline): host threads for the per-observation
 * pass and the blocked dense kernels (0 = all cores; 1 = single-threaded like the reference). */
int oracle_set_threads(int n);
void oracle_force_fast_dense(int on);
int oracle_schur_solve_fast(int32_t block_size, int32_t n_blocks, int32_t n_dense, const double* D,
                            const double* B, const double* C, const double* b1, const double* b2, double* x);


#ifdef __cplusplus
}
#endif
#endif
