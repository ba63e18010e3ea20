// ba_kernels.h -- launchers of the kernels in ba_kernels.cu (internal to libb200ba.so).
#pragma once
#include <vector>

#include "ba_common.h"

namespace b200ba {

void launch_prepare_state(const ProblemDev& pb, const Layout& L, const StateDev& st, int64_t n_control_total,
                          cudaStream_t s);
// uniform_model: the model type shared by all cameras, or -1 for a mixed rig (runtime switch)
void launch_residual_jacobian(int uniform_model, bool jac, const ProblemDev& pb, const Layout& L,
                              const StateDev& st, double2* last_projection, const ObsOut& out, double huber,
                              uint32_t* straggler_list, int* straggler_count, cudaStream_t s,
                              cudaEvent_t main_done = nullptr);
void launch_straggler_pass(int uniform_model, bool jac, const ProblemDev& pb, const Layout& L, const StateDev& st,
                           double2* last_projection, const ObsOut& out, double huber, uint32_t* straggler_list,
                           int* straggler_count, cudaStream_t s);
void launch_accumulate_list(const ProblemDev& pb, const Layout& L, const StateDev& st, const ObsOut& out,
                            const SystemDev& sys, double huber, const uint32_t* list, const int* count, cudaStream_t s);
void launch_expand_jacobian(const ProblemDev& pb, const Layout& L, const StateDev& st, const ObsOut& out, double* jac,
                            cudaStream_t s);
// evaluation budget of the main pass before an observation is deferred to the straggler pass
void set_main_eval_budget(int budget);
void launch_accumulate_scatter(const ProblemDev& pb, const Layout& L, const StateDev& st, const ObsOut& out,
                               const SystemDev& sys, double huber, cudaStream_t s);
void launch_accumulate_cells(const ProblemDev& pb, const Layout& L, const StateDev& st, const ObsOut& out,
                             const SystemDev& sys, double huber, cudaStream_t s);
void launch_schur_blocks(int bs, int n_blocks, const double* Dblk, const double* bp, double lambda, double* Linv,
                         double* v, int* fail, cudaStream_t s);
void launch_schur_scale_rows(int bs, int n_blocks, int nd, const double* B, const double* Linv, double* W,
                             cudaStream_t s);
void launch_schur_backsub(int bs, int n_blocks, const double* Linv, const double* y, double* xp, cudaStream_t s);
void launch_group_support(int bs, int nblocks, int nd, const double* B, const int* group_of_block, uint8_t* flags,
                          cudaStream_t s);
void launch_compact_columns(int ngroups, int nd, const uint8_t* flags, int* cols, int* count, cudaStream_t s);
void launch_gather_scale(int bs, int nblocks_in_group, int nd, int m, int ldw, const double* B, const double* Linv,
                         const int* blocks, const int* cols, double* Wc, cudaStream_t s);
void launch_scatter_sub(int nd, int m, const int* cols, const double* P, double* S, cudaStream_t s);
void launch_block_solve_t(int bs, int n_blocks, const double* Linv, const double* v, double* u, cudaStream_t s);
void launch_block_backsub2(int bs, int n_blocks, const double* Linv, const double* u, const double* t, double* xb,
                           cudaStream_t s);
void launch_add_diagonal(int n, double* M, int64_t ld, double lambda, cudaStream_t s);
void launch_trace(int n_blocks, int bs, const double* Dblk, int nd, const double* C, double* out, cudaStream_t s);
void launch_update_state(const ProblemDev& pb, const Layout& L, const StateDev& src, const StateDev& dst,
                         const double* x, int64_t n_control_total, int64_t n_param_total, cudaStream_t s);
void launch_cost_reduce(int64_t n, const double* trial, const double* base, const double* residual, double* partial,
                        double* out, cudaStream_t s);
int cost_reduce_partial_size();
void launch_project_points(const CamDev& c, const double* intr, int64_t n, const double* lp, double* px, int32_t* ok,
                           cudaStream_t s);
void launch_unproject_pixels(const CamDev& c, const double* intr, int64_t n, const double* px, double* dirs,
                             double* origins, int32_t* ok, cudaStream_t s);
// every statistic of the calibration report from the state st (its image_tr_global cache must be current)
void launch_calibration_report(const ProblemDev& pb, int n_cameras, const StateDev& st, const ReportDev& r,
                               cudaStream_t s);
int report_partial_size(int n_cameras);
// comparison of two central-generic models of the same image size (b200ba_compare_models); the grids a and b are
// on the device. With d's images set (d.dir_err is then required), also the five images of b200ba_fitting_images.
void launch_compare_models(const CamDev& a, const double* ga, const CamDev& b, const double* gb, const CompareDev& d,
                           cudaStream_t s);
// localization accuracy test (b200ba_localization_accuracy): the draws of every point (sets d.capped when a point
// needs more than kLocMaxDraws draws), then, after the caller has checked d.capped, the pose fits and the statistics
void launch_localization_sample(const CamDev& gt, const double* ggt, const CamDev& cmp, const double* gcmp,
                                int64_t trials, uint64_t seed, const LocalizationDev& d, cudaStream_t s);
void launch_localization_pose(int64_t trials, const LocalizationDev& d, cudaStream_t s);
// reconstruction comparison (b200ba_compare_reconstructions): over the nx x ny sample pixels (step i + 0.5,
// step j + 0.5), sums[0] = pixels both models un-project, sums[1 + 3 r + c] = sum of d1[r] d2[c] over them;
// partial holds sweep_partial_blocks(nx, ny) * kSweepSums doubles. intr1 / intr2 on the device.
int64_t sweep_partial_blocks(int nx, int ny);
void launch_reconstruction_sweep(const CamDev& c1, const double* intr1, const CamDev& c2, const double* intr2,
                                 int step, int nx, int ny, double* partial, double* sums, cudaStream_t s);
// the per-pixel un-projections of the same sample pixels: ok [2 nx ny], dirs [6 nx ny]
void launch_reconstruction_directions(const CamDev& c1, const double* intr1, const CamDev& c2, const double* intr2,
                                      int step, int nx, int ny, int32_t* ok, double* dirs, cudaStream_t s);
// centre-point analysis of a non-central camera (b200ba_line_offsets); intr on the device. launch_line_pass stores
// the line of every calibrated-rectangle pixel in d.lines; launch_line_system sums (mode 0) the cost, (1) + b,
// (2) + H at the centre c into d.sums; launch_line_outputs computes the distances and their statistics, the
// extent, and whichever of d.offsets / d.image / d.obj is set (obj: every obj_step-th pixel, nx per row, n_obj)
void launch_line_pass(const CamDev& c, const double* intr, const LineOffsetsDev& d, cudaStream_t s);
void launch_line_system(int mode, int64_t n, const double c[3], const LineOffsetsDev& d, cudaStream_t s);
int line_system_partial_size();
void launch_line_outputs(const CamDev& c, const double center[3], const LineOffsetsDev& d, int obj_step, int nx,
                         int64_t n_obj, cudaStream_t s);
// re-projection errors of every observation into r.err / r.mag (the first kernel of launch_calibration_report)
void launch_report_errors(const ProblemDev& pb, int n_cameras, const StateDev& st, const ReportDev& r, cudaStream_t s);
// the radix select of the report: rc[range * ranks + j].select_rank of every range [off[k], off[k + 1]) of the non-NaN
// mag, the value in rc[...].median (n_ranges * ranks <= 32)
void launch_report_select(int n_ranges, int ranks, const int64_t* off, const double* mag, unsigned int* select_hist,
                          ReportCam* rc, cudaStream_t s);
// outlier round of one camera (b200ba_delete_outliers) on the report's errors r.mag (launch_report_errors must have run):
// the camera is the device range [a, a + n); perm maps device positions to caller indices; w x h is its image size
void launch_delete_outliers(const ProblemDev& pb, int n_imagesets, const ReportDev& r, const uint32_t* perm,
                            int64_t a, int64_t n, float factor, int w, int h, const OutlierDev& d, cudaStream_t s);
// Voronoi coverage rendering of n sites (quarter-pixel int2, kVoronoiNoSite.x = skipped) with nch = 3 or 6 float
// colours per site into the RGB images img0 (channels 0-2) and img1 (channels 3-5, nch == 6), both [h * w * 3],
// nullable. g's geometry must be set (voronoi_grid_geometry) and its buffers allocated.
void launch_render_voronoi(int w, int h, int64_t n, const int2* sites, const float* colors, int nch, const VoronoiGrid& g,
                           uint8_t* img0, uint8_t* img1, cudaStream_t s);
// bucket grid over the quarter-pixel box [lo_x, hi_x] x [lo_y, hi_y] (which must contain the image)
VoronoiGrid voronoi_grid_geometry(int64_t lo_x, int64_t lo_y, int64_t hi_x, int64_t hi_y);
// sites and colours of the error maps of one camera: group_off [n_groups + 1] lists, per integer feature pixel, the
// device positions group_obs of its observations in the caller's order; the first one whose projection succeeded
// gives the group's site and its direction (colors[6g..6g+2]) and magnitude (colors[6g+3..6g+5]) colours
void launch_report_sites(const ProblemDev& pb, const ReportDev& r, int64_t n_groups, const int* group_off,
                         const uint32_t* group_obs, int2* sites, float* colors, cudaStream_t s);
// observation-direction image of one camera (VisualizeModelDirections): central- or non-central-generic
void launch_observation_directions(const CamDev& c, const double* intr, uint8_t* img, cudaStream_t s);
// VisualizeCameraModel of a libvis RadtanCamera8d (params [8] k1 k2 r1 r2 fx fy cx cy, on the device): the orientation
// rot [9] (window directions win: at most 21 * w), then the image [h * w * 3] and, dirs non-null, the rotated unit
// directions [h * w * 3]
void launch_visualize_orientation(const double* params, int w, int h, double2* win, double* rot, cudaStream_t s);
void launch_visualize_camera(const double* params, int w, int h, const double* rot, uint8_t* img, double* dirs,
                             cudaStream_t s);
// feature intersection of b200ba_intersect_features: n_lists independent lists of d datasets (off [n_lists * d + 1],
// xy [off[n_lists * d]] -- its erased features are overwritten with NaN), bound = the largest float <= thr2 (NaN for a
// NaN thr2), max_list = the largest list. keep [N] must hold 1 on entry; centres [N] and n_centres [n_lists] are
// scratch; counts [2] (uncovered walks, capped loops) are added to.
void launch_intersect_features(int d, int64_t n_lists, int64_t max_list, const int64_t* off, float2* xy, float bound,
                               uint8_t* keep, float2* centres, int* n_centres, unsigned long long* counts,
                               cudaStream_t s);
// synthetic pattern images of b200ba_render_pattern_images (the arithmetic is specified in include/b200ba.h)
constexpr int kSynthTile = 16;     // screen tiles of kSynthTile x kSynthTile pixels
constexpr int kSynthMaxVerts = 4;  // vertices of one pattern polygon
struct SynthParams {
  int w, h, tiles_x, tiles_y, words, n_poly;  // words: 32-bit words of one tile's polygon bitmap
  float fx, fy, cx, cy;
  int pattern_w, pattern_h, squares_x, squares_y, num_tags;
  float page_w, page_h, start_x, start_y, end_x, end_y;
  int4 tags[B200BA_PATTERN_MAX_TAGS];  // x, y, width, height
};
// n_img images of one chunk: verts [n_poly][kSynthMaxVerts] (pattern-image pixels, z = 0), nv [n_poly], poses
// [n_img][24] (Rf, tf, Rc, tc), pattern [pattern_h][pattern_w]; proj [n_img][n_poly][kSynthMaxVerts] and range
// [n_img][n_poly] are scratch, bits [n_img][tiles_y][tiles_x][words] must be zero on entry; images [n_img][h][w].
void launch_render_pattern(const SynthParams& p, int n_img, const float2* verts, const int8_t* nv, const float* poses,
                           const uint8_t* pattern, double2* proj, int4* range, uint32_t* bits, uint8_t* images,
                           cudaStream_t s);
// feature refinement of b200ba_refine_features (the arithmetic is specified in include/b200ba.h)
struct RefineParams {
  int w, h;                // image size
  int half;                // window_half_extent
  int n_samples, n_match;  // symmetry and matching sample counts
  int type;                // B200BA_REFINE_*
  int num_star_segments, squares_x, squares_y, num_tags;
  int4 tags[B200BA_PATTERN_MAX_TAGS];  // x, y, width, height
};
// n predictions whose image indices are relative to `images` ([..][h][w]); one warp per feature.
void launch_refine_features(const RefineParams& p, int64_t n, const b200ba_feature_prediction* pred,
                            const uint8_t* images, const float2* samples, float2* xy, float* cost, int* status,
                            cudaStream_t s);
void launch_generic_block_inverse(int bs, int nb, int nd, const double* D, const double* B, const double* b1,
                                  double* DinvB, double* Dinvb, cudaStream_t s);
void launch_symmetrize(int n, double* M, cudaStream_t s);
// direction-grid fit (b200ba_fit_directions)
void launch_dirfit_tangents(int G, const double* grid, double* tan, cudaStream_t s);
void launch_dirfit(bool jac, int gw, int64_t n, const double* gp, const double* dirs, const double* grid,
                   const double* tan, double* H, double* b, int dof, double* cost, double* cost_sum, cudaStream_t s);
void launch_dirfit_update(int G, const double* grid, const double* x, double* out, cudaStream_t s);
void launch_permute_double2(int64_t n, const uint32_t* perm, const double2* src, double2* dst, bool scatter,
                            cudaStream_t s);


void launch_mask_fixed(const Layout& L, const SystemDev& sys, const FixedRanges& fr, double unit, cudaStream_t s);
// ChooseNiceCameraOrientation + Rotate + camera_tr_rig update for every camera (rot: [9 * n_cameras] scratch)
void launch_nice_orientation(const ProblemDev& pb, const StateDev& st, int n_cameras, double* rot, cudaStream_t s);

// ---- dense phase (ba_dense.cu) ----------------------------------------------------------------
// Storage map of the reduced system S (n_d x n_d, column-major, lower triangle valid): columns are
// grouped in blocks of `nb`; block j lives in slot (j % ranks) * blocks_per_rank + j / ranks, so that
// the column blocks one rank owns in the block-cyclic distribution are CONTIGUOUS (one chunk of a
// reduce-scatter). With one rank the map is the identity. Rows are never permuted.
struct DenseMap {
  int nb;               // column-block width
  int ranks;            // R
  int blocks_per_rank;  // ceil(n_blocks / R)
  int64_t ld;           // leading dimension (>= n_d, even)
  __host__ __device__ __forceinline__ int slot(int block) const { return (block % ranks) * blocks_per_rank + block / ranks; }
  __host__ __device__ __forceinline__ int64_t col_offset(int c) const {
    const int b = c / nb;
    return (static_cast<int64_t>(slot(b)) * nb + (c - b * nb)) * ld;
  }
};

// One group of the grouped contraction (GemmArgs::groups): its compact panel W_g (k x m, row-major, leading
// dimension ld) at A + w_off, its column list at cols + cols_off, and the index of its first tile in the launch.
struct ContractGroup {
  int64_t w_off, cols_off, tile0;
  int m, k, ld;
  bool aligned;  // W_g is 16-byte aligned (even w_off and ld)
};

// C (+)= alpha * A B^T; A(i, k) at A[k * lda + i], B(j, k) at B[k * ldb + j], C(i, j) at C[j * ldc + i].
struct GemmArgs {
  int M, N, K;
  const double* A;
  int64_t lda;
  const double* B;
  int64_t ldb;
  double* C;
  int64_t ldc;
  double alpha, beta;
  bool a_aligned, b_aligned;  // 16-byte copies allowed (set by make_gemm_args)
  // scatter epilogue: C is the base of S, compact row / column i is dense column cols[i] (ascending)
  const int* cols;
  DenseMap map;
  int64_t n_tiles_lower;  // set by launch_dgemm_nt
  // owned-only trailing update of the block-cyclic factorisation: C = base of S, column n of the product is
  // global column col_base + n (rows likewise); tiles of column blocks owned by other ranks are skipped
  bool owned_only;
  int rank, col_base;
  // grouped contraction: C += alpha * W_g^T W_g (lower, scatter through each group's columns) for n_groups groups
  // in one launch; A = base of the panels, cols = base of the column lists, n_tiles_lower = total tile count.
  // Groups share entries of S, so the epilogue adds with FP64 reductions; beta, B, M, N, K are not used.
  const ContractGroup* groups;
  int n_groups;
};
inline bool gemm_operand_aligned(const double* p, int64_t ld) {
  return (reinterpret_cast<uintptr_t>(p) % 16 == 0) && (ld % 2 == 0);
}
// lower: only tiles / entries with i >= j (M == N); scatter: the scatter-subtract epilogue (implies lower).
// one_tile_per_cta: an ordinary grid instead of persistent CTAs (the factorisation's updates).
int launch_dgemm_nt(const GemmArgs& g, bool lower, bool scatter, cudaStream_t s, bool one_tile_per_cta = false);
// tiles of the LOWER enumeration of an M x N product (ContractGroup::tile0)
int64_t dgemm_lower_tiles(int M, int N);

// y += alpha B^T u (two stages, fixed order; partial: gemv_t_partial_size doubles) and t = B x for row-major B
int gemv_t_partial_size(int rows, int cols);
void launch_gemv_t(int rows, int cols, int64_t ld, const double* B, const double* u, double alpha, double* y, double* partial,
                   cudaStream_t s);
void launch_gemv_n(int rows, int cols, int64_t ld, const double* B, const double* x, double* t, cudaStream_t s);
void launch_add_diagonal_map(int n, double* S, const DenseMap& map, double lambda, cudaStream_t s);

// Context of the dense factorisation / solve (ba_dense.cu). The caller owns the buffers.
struct DenseCtx {
  int n = 0, NB = 256, nblk = 0, ntiles = 0;
  int rank = 0, ranks = 1;
  DenseMap map{};
  int64_t chunk = 0;                 // doubles per rank of the S allocation (reduce-scatter chunk)
  std::vector<int64_t> panel_off;    // [nblk + 1] offsets of the packed panels in Lpack
  std::vector<int> panel_h;          // [nblk] leading dimension (even) of each packed panel
  double* S = nullptr;               // ranks * chunk doubles
  double* Lpack = nullptr;           // panel_off[nblk] doubles: the factor; each panel is followed by the explicit
                                     // inverses of its NB / 128 diagonal tiles ([128 * 128] each)
  double* tmp = nullptr;             // [n] intermediate of the triangular solves
  int64_t* d_panel_off = nullptr;    // device copies for the backward step
  int* d_panel_h = nullptr;
  int* info = nullptr;               // device flag: non-positive pivot
  cudaStream_t s_main = nullptr, s_panel = nullptr, s_aux = nullptr;
  cudaEvent_t ev_ready[2] = {nullptr, nullptr}, ev_main[2] = {nullptr, nullptr}, ev_half2[2] = {nullptr, nullptr}, ev_misc = nullptr;
  // broadcast of `count` doubles from rank `root` on stream s (multi-GPU only)
  int (*bcast)(double* buf, size_t count, int root, cudaStream_t s, void* user) = nullptr;
  void* user = nullptr;
};
int dense_plan(DenseCtx* d, int n, int nb, int rank, int ranks);
int dense_factor(DenseCtx* d);
int dense_solve(DenseCtx* d, double* b);

}  // namespace b200ba
