// ba_host.cu -- host logic of libb200ba.so: the C ABI of include/b200ba.h, device memory
// management, the Levenberg-Marquardt control loop and the dense-algebra plumbing.
//
// What runs where
//   device, own kernels (ba_kernels.cu): residuals, Jacobians, J^T J accumulation, 3x3 block
//     factorisation, L^-1 B, state retraction, cost comparison.
//   device, libraries: the symmetric rank-k update S = C - W^T W (cublasDsyrk, a plain dense
//     FP64 contraction -- the reference uses cublasXtDgemm for it, LV/lm_optimizer.h:1371-1430)
//     and the dense SPD factorisation (cusolverDnDpotrf/potrs; scaffolding, see DESIGN.md).
//   host: the scalar LM decisions (accept / reject, lambda), exactly LV/lm_optimizer.h:628-991
//     as driven by APP/bundle_adjustment/joint_optimization.cc:905-940.
// There is NO CPU fallback: every entry point fails with an error if CUDA is unavailable.

#include <cublas_v2.h>
#include <cusolverDn.h>
#include <dlfcn.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <limits>
#include <string>
#include <vector>

#include "ba_kernels.h"

using namespace b200ba;

namespace {

std::string g_create_error;

struct NcclUniqueId {  // layout of ncclUniqueId (nccl.h): 128 opaque bytes, passed BY VALUE
  char internal[128];
};
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, NcclUniqueId, int) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*Broadcast)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*ReduceScatter)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
// ncclDataType_t / ncclRedOp_t values (nccl.h): ncclFloat64 = 8, ncclSum = 0
constexpr int kNcclDouble = 8;
constexpr int kNcclInt32 = 2;
constexpr int kNcclSum = 0;
constexpr int kNcclMax = 2;

NcclApi g_nccl;
bool load_nccl(std::string* err) {
  if (g_nccl.lib) return true;
  // Reuse the copy already mapped into the process (torch ships its own libnccl.so.2).
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  void* lib = nullptr;
  for (const char* n : names) {
    lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (lib) break;
  }
  if (!lib) {
    *err = std::string("cannot load libnccl: ") + dlerror();
    return false;
  }
  g_nccl.lib = lib;
  *reinterpret_cast<void**>(&g_nccl.GetUniqueId) = dlsym(lib, "ncclGetUniqueId");
  *reinterpret_cast<void**>(&g_nccl.CommInitRank) = dlsym(lib, "ncclCommInitRank");
  *reinterpret_cast<void**>(&g_nccl.AllReduce) = dlsym(lib, "ncclAllReduce");
  *reinterpret_cast<void**>(&g_nccl.Broadcast) = dlsym(lib, "ncclBroadcast");
  *reinterpret_cast<void**>(&g_nccl.ReduceScatter) = dlsym(lib, "ncclReduceScatter");
  *reinterpret_cast<void**>(&g_nccl.CommDestroy) = dlsym(lib, "ncclCommDestroy");
  *reinterpret_cast<void**>(&g_nccl.GetErrorString) = dlsym(lib, "ncclGetErrorString");
  if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllReduce || !g_nccl.Broadcast || !g_nccl.ReduceScatter ||
      !g_nccl.CommDestroy) {
    *err = "libnccl lacks a required symbol";
    g_nccl.lib = nullptr;
    return false;
  }
  return true;
}

constexpr int kMaxCholPanels = 1024;

enum Phase { PH_JAC = 0, PH_ACC, PH_SCHUR, PH_FACTOR, PH_TRIAL, PH_UPDATE, PH_ALLREDUCE, PH_STRAGGLER, PH_SOLVE, PH_COUNT };

}  // namespace

struct b200ba_handle {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t side_stream = nullptr;  // straggler pass of the Jacobian kernel, overlapped with accumulation
  cudaEvent_t straggler_done = nullptr;
  cublasHandle_t cublas = nullptr;
  cusolverDnHandle_t cusolver = nullptr;
  std::string error;

  // problem
  std::vector<b200ba_camera> cams_host;
  ProblemDev pb{};
  int n_cameras = 0, n_imagesets = 0, n_points = 0;
  int64_t n_obs = 0;
  int uniform_model = -1;
  int64_t n_control_total = 0, n_param_total = 0, intr_total = 0, tan_total = 0;
  uint32_t *d_obs_imageset = nullptr, *d_obs_camera = nullptr, *d_obs_point = nullptr;
  float2* d_obs_xy = nullptr;

  // state (two copies: current / trial)
  StateDev st[2]{};
  int cur = 0;
  double2* d_last_projection = nullptr;
  bool have_state = false;
  // device-side snapshot of (state, last_projection): b200ba_snapshot_state / b200ba_restore_state
  StateDev snap{};
  double2* d_snap_lp = nullptr;
  bool have_snapshot = false;

  // layout-dependent buffers
  Layout L{};
  bool have_layout = false;
  ObsOut out{};        // base evaluation (with Jacobians)
  ObsOut out_trial{};  // residual-only evaluation of the trial state
  SystemDev sys{};
  double *d_W = nullptr, *d_S = nullptr, *d_Linv = nullptr, *d_v = nullptr, *d_y = nullptr, *d_x = nullptr;
  double trace_H = 0;
  int64_t reduce_count = 0;  // doubles of sys.base covered by the per-build all-reduce
  double* d_potrf_work = nullptr;
  int potrf_lwork = 0;
  int chol_mode = -1;                     // B200BA_DIST_CHOL=0|1 overrides: 1 = column-block Cholesky (see factor_dense)
  int chol_nb = 512;                      // its panel width (B200BA_CHOL_NB)
  int *d_info = nullptr, *d_fail = nullptr;
  // Static cell-major processing order: device position -> index in the caller's (reference)
  // observation order. Computed once at create time from the cell of the measured pixel.
  std::vector<uint32_t> perm;
  uint32_t* d_perm = nullptr;
  double2* d_lp_stage = nullptr;  // last_projection in the caller's order (H2D / D2H staging)
  uint32_t* d_straggler_list = nullptr;  // observations deferred by the main pass of the Jacobian kernel
  int* d_straggler_count = nullptr;
  double *d_partial = nullptr, *d_scal = nullptr;
  double* d_rot = nullptr;  // [9 * n_cameras] rotations of ChooseNiceCameraOrientation
  double* h_scal = nullptr;  // pinned [16]
  int* h_flags = nullptr;    // pinned [2]

  // host copies of the observations (caller's order) for layout-time block grouping
  std::vector<uint32_t> h_obs_imageset, h_obs_camera, h_obs_point;
  std::vector<float> h_obs_xy;
  // structured Schur contraction (groups of Schur blocks with compacted column support)
  int group_blocks_n = 0;                 // blocks per group
  int n_groups = 0;
  std::vector<int> group_start;           // [n_groups + 1] into group_blocks
  std::vector<int> group_count;           // m_g of the current build
  int* d_group_of_block = nullptr;
  int* d_group_blocks = nullptr;
  uint8_t* d_flags = nullptr;
  int* d_cols = nullptr;
  int* d_count = nullptr;
  int* h_count = nullptr;                 // pinned
  double* d_Wc = nullptr;                 // 2 panels (double-buffered)
  double* d_P = nullptr;                  // 2 result buffers (double-buffered)
  size_t wc_stride = 0, p_stride = 0;
  cudaEvent_t ev_syrk[2] = {nullptr, nullptr}, ev_scatter[2] = {nullptr, nullptr}, ev_s_ready = nullptr;
  double* d_u = nullptr;
  bool use_grouped = false;
  // b200ba_debug_solve_step: host buffers that receive S (n_d x n_d, column-major) and the reduced right-hand side
  // between the Schur phase and the factorisation; null in every other call
  double* capture_S = nullptr;
  double* capture_rhs = nullptr;
  std::vector<int32_t> lm_events;         // B200BA_LM_* per LM attempt of the last b200ba_optimize
  std::vector<double> grp_sums;           // [sx | sy | count] per Schur block (see build_groups)
  int force_grouped = -1;                 // B200BA_GROUPED=0|1 overrides the cost model
  bool compact_j = true;                  // B200BA_COMPACT_J=0: expanded Jacobian buffer also for central-generic cameras

  // calibration report: allocated by the first b200ba_calibration_report
  ReportDev rep{};
  double2* d_rep_stage = nullptr;  // errors in the caller's order (D2H staging)
  bool have_report = false;
  // report images: observations grouped by (camera, integer feature pixel), allocated by the first
  // b200ba_report_images
  std::vector<int64_t> img_cam_groups;  // [n_cameras + 1] range of each camera's groups
  int* d_img_group_off = nullptr;       // [n_groups + 1] into d_img_group_obs
  uint32_t* d_img_group_obs = nullptr;  // device positions, the caller's order inside a group
  bool have_images = false;

  // multi-GPU
  void* comm = nullptr;
  int rank = 0, n_ranks = 1;

  // dense phase on the in-tree DMMA kernels (ba_dense.cu); B200BA_DENSE=lib selects the cuBLAS / cuSOLVER path
  bool own_dense = true;
  DenseCtx dn;
  int dense_planned_ranks = 0, dense_planned_n = -1;
  int dense_nb = 0;                     // column-block width of the factorisation (B200BA_DENSE_NB, multiple of 128); 0 = by rank count
  cudaStream_t panel_stream = nullptr;  // panel factorisations + broadcasts (look-ahead)
  cudaStream_t aux_stream = nullptr;    // second look-ahead update of the single-GPU factorisation
  int* d_ident_cols = nullptr;          // 0 .. nd - 1 (scatter epilogue of the dense contraction with several ranks)
  double* d_gemv_partial = nullptr;     // slab sums of the B^T u product

  // timings
  b200ba_timings timings{};
  struct Pending {
    int phase;
    cudaEvent_t a, b;
    bool own_a = true;  // false: `a` is another entry's `b` and is released there
  };
  std::vector<Pending> pending;
  std::vector<cudaEvent_t> event_pool;
};

namespace {

#define CUDA_TRY(h, expr)                                                                      \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      (h)->error = std::string(#expr) + ": " + cudaGetErrorString(_e);                         \
      return 1;                                                                                \
    }                                                                                          \
  } while (0)
#define CUBLAS_TRY(h, expr)                                                                    \
  do {                                                                                         \
    cublasStatus_t _s = (expr);                                                                \
    if (_s != CUBLAS_STATUS_SUCCESS) {                                                         \
      (h)->error = std::string(#expr) + ": cuBLAS status " + std::to_string(static_cast<int>(_s)); \
      return 1;                                                                                \
    }                                                                                          \
  } while (0)
#define CUSOLVER_TRY(h, expr)                                                                  \
  do {                                                                                         \
    cusolverStatus_t _s = (expr);                                                              \
    if (_s != CUSOLVER_STATUS_SUCCESS) {                                                       \
      (h)->error = std::string(#expr) + ": cuSOLVER status " + std::to_string(static_cast<int>(_s)); \
      return 1;                                                                                \
    }                                                                                          \
  } while (0)

template <class T>
int dev_alloc(b200ba_handle* h, T** p, size_t count) {
  if (*p) {
    cudaFree(*p);
    *p = nullptr;
  }
  if (count == 0) count = 1;
  CUDA_TRY(h, cudaMalloc(reinterpret_cast<void**>(p), count * sizeof(T)));
  return 0;
}

int64_t intrinsics_size(const b200ba_camera& c) {
  const int64_t G = static_cast<int64_t>(c.grid_width) * c.grid_height;
  switch (c.model_type) {
    case B200BA_MODEL_CENTRAL_GENERIC: return 3 * G;
    case B200BA_MODEL_NONCENTRAL_GENERIC: return 6 * G;
    default: return 12;
  }
}
int update_parameter_count(const b200ba_camera& c) {
  const int G = c.grid_width * c.grid_height;
  switch (c.model_type) {
    case B200BA_MODEL_CENTRAL_GENERIC: return 2 * G;
    case B200BA_MODEL_NONCENTRAL_GENERIC: return 5 * G;
    default: return 12;
  }
}
int jacobian_size(const b200ba_camera& c) {
  switch (c.model_type) {
    case B200BA_MODEL_CENTRAL_GENERIC: return 32;
    case B200BA_MODEL_NONCENTRAL_GENERIC: return 80;
    default: return 12;
  }
}

void fill_camdev(const b200ba_camera& c, CamDev* d) {
  d->model_type = c.model_type;
  d->width = c.width;
  d->height = c.height;
  d->min_x = c.calibration_min_x;
  d->min_y = c.calibration_min_y;
  d->max_x = c.calibration_max_x;
  d->max_y = c.calibration_max_y;
  d->gw = c.grid_width;
  d->gh = c.grid_height;
  const int aw = c.calibration_max_x + 1 - c.calibration_min_x;
  const int ah = c.calibration_max_y + 1 - c.calibration_min_y;
  d->gmul_x = (c.grid_width > 0) ? static_cast<double>(c.grid_width - 3) / aw : 0.0;
  d->gmul_y = (c.grid_height > 0) ? static_cast<double>(c.grid_height - 3) / ah : 0.0;
  // PixelScaleToGridScaleX/Y divide in float (APP/models/central_grid.h:156-161)
  d->sx = (c.grid_width > 0) ? static_cast<double>((c.grid_width - 3.f) / aw) : 0.0;
  d->sy = (c.grid_height > 0) ? static_cast<double>((c.grid_height - 3.f) / ah) : 0.0;
  d->center_x = 0.5f * static_cast<float>(c.calibration_min_x + c.calibration_max_x + 1);
  d->center_y = 0.5f * static_cast<float>(c.calibration_min_y + c.calibration_max_y + 1);
  d->K = jacobian_size(c);
  d->dof_per_point = c.model_type == B200BA_MODEL_CENTRAL_GENERIC ? 2 : (c.model_type == B200BA_MODEL_NONCENTRAL_GENERIC ? 5 : 0);
  d->upd_count = update_parameter_count(c);
}

int64_t align32(int64_t n) { return (n + 31) / 32 * 32; }

// ---- timing ----------------------------------------------------------------------------
cudaEvent_t get_event(b200ba_handle* h) {
  if (!h->event_pool.empty()) {
    cudaEvent_t e = h->event_pool.back();
    h->event_pool.pop_back();
    return e;
  }
  cudaEvent_t e;
  cudaEventCreate(&e);
  return e;
}
struct ScopedPhase {
  b200ba_handle* h;
  int phase;
  cudaEvent_t a;
  ScopedPhase(b200ba_handle* h_, int p) : h(h_), phase(p) {
    a = get_event(h);
    cudaEventRecord(a, h->stream);
  }
  ~ScopedPhase() {
    cudaEvent_t b = get_event(h);
    cudaEventRecord(b, h->stream);
    h->pending.push_back({phase, a, b, true});
  }
};
void resolve_timings(b200ba_handle* h) {
  for (auto& p : h->pending) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, p.a, p.b) == cudaSuccess) {
      switch (p.phase) {
        case PH_JAC: h->timings.jacobian_kernel_ms += ms; h->timings.jacobian_kernel_launches++; break;
        case PH_ACC: h->timings.accumulate_ms += ms; break;
        case PH_SCHUR: h->timings.schur_ms += ms; break;
        case PH_FACTOR: h->timings.factor_ms += ms; break;
        case PH_TRIAL: h->timings.trial_cost_ms += ms; break;
        case PH_UPDATE: h->timings.update_ms += ms; break;
        case PH_ALLREDUCE: h->timings.allreduce_ms += ms; break;
        case PH_STRAGGLER: h->timings.straggler_ms += ms; break;
        case PH_SOLVE: h->timings.solve_ms += ms; h->timings.factor_ms += ms; break;
      }
    }
    if (p.own_a) h->event_pool.push_back(p.a);
    h->event_pool.push_back(p.b);
  }
  h->pending.clear();
}
// All-reduces the centroid sums over the ranks (no-op without a communicator).
int reduce_group_sums(b200ba_handle* h) {
  if (h->n_ranks <= 1 || !h->comm || h->grp_sums.empty()) return 0;
  const size_t n = h->grp_sums.size();
  double* d = nullptr;
  CUDA_TRY(h, cudaMalloc(reinterpret_cast<void**>(&d), n * sizeof(double)));
  cudaMemcpy(d, h->grp_sums.data(), n * sizeof(double), cudaMemcpyHostToDevice);
  const int rc = g_nccl.AllReduce(d, d, n, kNcclDouble, kNcclSum, h->comm, h->stream);
  const cudaError_t ce = cudaStreamSynchronize(h->stream);
  if (rc == 0 && ce == cudaSuccess) cudaMemcpy(h->grp_sums.data(), d, n * sizeof(double), cudaMemcpyDeviceToHost);
  cudaFree(d);
  if (rc != 0 || ce != cudaSuccess) {
    h->error = "all-reduce of the group centroids failed";
    return 1;
  }
  return 0;
}

// Groups of Schur blocks for the structured contraction, from the centroid sums in h->grp_sums
// ([sx | sy | count] per block). Must produce the same grouping on every rank: the ranks split
// the GROUPS among themselves (solve_system), so a rank-dependent order would drop / repeat blocks.
int build_groups(b200ba_handle* h, bool allocate) {
  const Layout& L = h->L;
  const int nb = L.nblocks;
  int gb = (L.bs == 3) ? 96 : 48;  // ~288 rows per group
  if (const char* e = getenv("B200BA_GROUP_BLOCKS")) gb = std::max(1, atoi(e));
  h->group_blocks_n = gb;
  std::vector<int> order(nb);
  for (int i = 0; i < nb; ++i) order[i] = i;
  if (L.eliminate_points && nb > 0) {
    // order the pattern points along a Z-curve of the centroid of their measured pixels: points
    // that are neighbours in the image share most of their control-point support
    const double* sx = h->grp_sums.data();
    const double* sy = sx + nb;
    const double* cnt = sy + nb;
    const double qx = std::max(1.0, h->cams_host[0].width / 64.0), qy = std::max(1.0, h->cams_host[0].height / 64.0);
    std::vector<uint32_t> zkey(nb, 0);
    for (int p = 0; p < nb; ++p) {
      if (cnt[p] <= 0) continue;
      uint32_t ux = static_cast<uint32_t>(std::min(1023.0, std::max(0.0, sx[p] / cnt[p] / qx)));
      uint32_t uy = static_cast<uint32_t>(std::min(1023.0, std::max(0.0, sy[p] / cnt[p] / qy)));
      uint32_t z = 0;
      for (int b = 0; b < 10; ++b) z |= ((ux >> b) & 1u) << (2 * b) | ((uy >> b) & 1u) << (2 * b + 1);
      zkey[p] = z;
    }
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return zkey[a] < zkey[b]; });
  }
  h->n_groups = (nb + gb - 1) / gb;
  h->group_start.assign(h->n_groups + 1, 0);
  std::vector<int> gob(std::max(1, nb), 0);
  for (int g = 0; g < h->n_groups; ++g) {
    h->group_start[g] = g * gb;
    for (int i = g * gb; i < std::min(nb, (g + 1) * gb); ++i) gob[order[i]] = g;
  }
  h->group_start[h->n_groups] = nb;
  h->group_count.assign(std::max(1, h->n_groups), 0);
  if (allocate) {
    if (dev_alloc(h, &h->d_group_of_block, std::max(1, nb))) return 1;
    if (dev_alloc(h, &h->d_group_blocks, std::max(1, nb))) return 1;
    if (dev_alloc(h, &h->d_flags, static_cast<size_t>(std::max(1, h->n_groups)) * std::max(1, L.nd))) return 1;
    if (dev_alloc(h, &h->d_cols, static_cast<size_t>(std::max(1, h->n_groups)) * std::max(1, L.nd))) return 1;
    if (dev_alloc(h, &h->d_count, std::max(1, h->n_groups))) return 1;
    if (h->h_count) cudaFreeHost(h->h_count);
    CUDA_TRY(h, cudaMallocHost(reinterpret_cast<void**>(&h->h_count), std::max(1, h->n_groups) * sizeof(int)));
    h->wc_stride = static_cast<size_t>(gb) * L.bs * (std::max(1, L.nd) + 1);
    h->p_stride = static_cast<size_t>(std::max(1, L.nd)) * std::max(1, L.nd);
    if (dev_alloc(h, &h->d_Wc, 2 * h->wc_stride)) return 1;
    if (!h->own_dense && dev_alloc(h, &h->d_P, 2 * h->p_stride)) return 1;
    for (int i = 0; i < 2; ++i) {
      if (!h->ev_syrk[i]) CUDA_TRY(h, cudaEventCreateWithFlags(&h->ev_syrk[i], cudaEventDisableTiming));
      if (!h->ev_scatter[i]) CUDA_TRY(h, cudaEventCreateWithFlags(&h->ev_scatter[i], cudaEventDisableTiming));
    }
    if (!h->ev_s_ready) CUDA_TRY(h, cudaEventCreateWithFlags(&h->ev_s_ready, cudaEventDisableTiming));
    if (dev_alloc(h, &h->d_u, std::max(1, L.nbd))) return 1;
  }
  CUDA_TRY(h, cudaMemcpy(h->d_group_of_block, gob.data(), std::max(1, nb) * sizeof(int), cudaMemcpyHostToDevice));
  if (nb > 0) CUDA_TRY(h, cudaMemcpy(h->d_group_blocks, order.data(), nb * sizeof(int), cudaMemcpyHostToDevice));
  return 0;
}

// ---- dense phase buffers (own kernels) ------------------------------------------------------
int nccl_bcast_cb(double* buf, size_t count, int root, cudaStream_t s, void* user) {
  b200ba_handle* h = static_cast<b200ba_handle*>(user);
  const int rc = g_nccl.Broadcast(buf, buf, count, kNcclDouble, root, h->comm, s);
  if (rc != 0) {
    h->error = std::string("ncclBroadcast: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "error");
    return 1;
  }
  return 0;
}

// The streams and events the dense schedule (ba_dense.cu) runs on. The handle sets the streams to its own ones and
// creates the events it lacks on every plan; a stand-alone solve owns the streams as well.
cudaError_t dense_create(DenseCtx* d, bool own_streams) {
  cudaError_t e = cudaSuccess;
  if (own_streams) {
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);
    e = cudaStreamCreateWithFlags(&d->s_main, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaStreamCreateWithPriority(&d->s_panel, cudaStreamNonBlocking, hi);
    if (e == cudaSuccess) e = cudaStreamCreateWithPriority(&d->s_aux, cudaStreamNonBlocking, hi);
  }
  for (cudaEvent_t* ev : {&d->ev_ready[0], &d->ev_ready[1], &d->ev_main[0], &d->ev_main[1], &d->ev_half2[0],
                          &d->ev_half2[1], &d->ev_misc})
    if (e == cudaSuccess && !*ev) e = cudaEventCreateWithFlags(ev, cudaEventDisableTiming);
  return e;
}
void dense_release(DenseCtx* d, bool own_streams) {
  for (cudaEvent_t ev : {d->ev_ready[0], d->ev_ready[1], d->ev_main[0], d->ev_main[1], d->ev_half2[0], d->ev_half2[1],
                         d->ev_misc})
    if (ev) cudaEventDestroy(ev);
  if (own_streams)
    for (cudaStream_t s : {d->s_main, d->s_panel, d->s_aux})
      if (s) cudaStreamDestroy(s);
}

// (Re)plans the storage of S / the packed factor for the current (n_d, rank count).
int plan_dense(b200ba_handle* h) {
  if (!h->own_dense || !h->have_layout) return 0;
  const int nd = h->L.nd;
  if (h->dense_planned_n == nd && h->dense_planned_ranks == h->n_ranks) return 0;
  DenseCtx& d = h->dn;
  // one GPU: 512-wide block columns (fewer, longer panels); several ranks: 256, so that the block-cyclic distribution has enough blocks per rank and the broadcasts stay short
  const int nb = h->dense_nb > 0 ? h->dense_nb : (h->n_ranks == 1 ? 512 : 256);
  dense_plan(&d, nd, nb, h->rank, h->n_ranks);
  if (dev_alloc(h, &h->d_S, static_cast<size_t>(std::max<int64_t>(1, d.chunk * h->n_ranks)))) return 1;
  d.S = h->d_S;
  if (dev_alloc(h, &d.Lpack, static_cast<size_t>(std::max<int64_t>(1, d.panel_off[d.nblk])))) return 1;
  if (dev_alloc(h, &d.tmp, std::max(1, nd))) return 1;
  if (dev_alloc(h, &d.d_panel_off, d.panel_off.size())) return 1;
  if (dev_alloc(h, &d.d_panel_h, d.panel_h.size())) return 1;
  CUDA_TRY(h, cudaMemcpy(d.d_panel_off, d.panel_off.data(), d.panel_off.size() * sizeof(int64_t), cudaMemcpyHostToDevice));
  CUDA_TRY(h, cudaMemcpy(d.d_panel_h, d.panel_h.data(), d.panel_h.size() * sizeof(int), cudaMemcpyHostToDevice));
  {
    std::vector<int> ident(std::max(1, nd));
    for (int i = 0; i < nd; ++i) ident[i] = i;
    if (dev_alloc(h, &h->d_ident_cols, ident.size())) return 1;
    CUDA_TRY(h, cudaMemcpy(h->d_ident_cols, ident.data(), ident.size() * sizeof(int), cudaMemcpyHostToDevice));
  }
  if (dev_alloc(h, &h->d_gemv_partial, static_cast<size_t>(gemv_t_partial_size(h->L.nbd, std::max(1, nd))))) return 1;
  // the un-owned chunks of S are never written by the contraction of a single rank but are read by nobody either;
  // zero once so that partial sums start clean
  CUDA_TRY(h, cudaMemset(h->d_S, 0, static_cast<size_t>(std::max<int64_t>(1, d.chunk * h->n_ranks)) * sizeof(double)));
  d.info = h->d_info;
  d.s_main = h->stream;
  d.s_panel = h->panel_stream;
  d.s_aux = h->aux_stream;
  CUDA_TRY(h, dense_create(&d, /*own_streams=*/false));
  d.bcast = nccl_bcast_cb;
  d.user = h;
  h->dense_planned_n = nd;
  h->dense_planned_ranks = h->n_ranks;
  return 0;
}

// ---- layout / buffers ----------------------------------------------------------------------
int make_layout(b200ba_handle* h, const b200ba_options* opt) {
  if (opt->regularization_weight != 0) {
    // the reference logs an error and carries on without the term (joint_optimization.cc:299-305)
    static bool warned = false;
    if (!warned) fprintf(stderr, "[b200ba] regularization_weight is ignored (the term is disabled in the reference, joint_optimization.cc:299-305)\n");
    warned = true;
  }
  Layout L{};
  memset(&L, 0, sizeof(L));
  L.n_points = h->n_points;
  L.n_imagesets = h->n_imagesets;
  L.n_cameras = h->n_cameras;
  L.rig_in_state = h->n_cameras > 1;
  L.localize_only = opt->localize_only ? 1 : 0;
  L.eliminate_points = opt->eliminate_points ? 1 : 0;
  int n_intr = 0, kmax = 0;
  for (int c = 0; c < h->n_cameras; ++c) {
    n_intr += update_parameter_count(h->cams_host[c]);
    kmax = std::max(kmax, jacobian_size(h->cams_host[c]));
  }
  if (L.localize_only) {
    n_intr = 0;
    kmax = 0;
  }
  const int rig_dof = L.rig_in_state ? 6 * h->n_cameras : 0;
  // JointOptimizationState offsets (joint_optimization.cc:142-170)
  if (L.eliminate_points) {
    L.bs = 3;
    L.nblocks = h->n_points;
    L.g_point = 0;
    L.g_pose = 3 * h->n_points;
    L.g_rig = L.g_pose + 6 * h->n_imagesets;
    L.g_intr = L.g_rig + rig_dof;
  } else {
    L.bs = 6;
    L.nblocks = h->n_imagesets;
    L.g_pose = 0;
    L.g_rig = 6 * h->n_imagesets;
    L.g_point = L.g_rig + rig_dof;
    L.g_intr = L.g_point + 3 * h->n_points;
  }
  L.dsz = L.bs * (L.bs + 1) / 2;
  L.nbd = L.bs * L.nblocks;
  L.dof = 3 * h->n_points + 6 * h->n_imagesets + rig_dof + n_intr;
  L.nd = L.dof - L.nbd;
  L.Kmax = kmax;
  L.jc_point = 0;
  L.jc_pose = 3;
  L.jc_rig = 9;
  L.jc_intr = 9 + (L.rig_in_state ? 6 : 0);
  L.n_jcols = L.jc_intr + kmax;
  const bool same = h->have_layout && memcmp(&L, &h->L, sizeof(Layout)) == 0;
  if (same) return plan_dense(h);
  h->L = L;
  h->have_layout = true;
  h->dense_planned_n = -1;

  const int64_t n = h->n_obs;
  if (dev_alloc(h, &h->out.residual, 2 * n)) return 1;
  if (dev_alloc(h, &h->out.cost, n)) return 1;
  // compact Jacobian records when every camera is central-generic (B200BA_COMPACT_J=0 keeps the expanded buffer)
  h->out.compact = (h->uniform_model == B200BA_MODEL_CENTRAL_GENERIC && h->compact_j) ? 1 : 0;
  if (h->out.compact) {
    if (h->out.jac) cudaFree(h->out.jac);
    h->out.jac = nullptr;
    if (dev_alloc(h, &h->out.cjac, 14 * static_cast<size_t>(n))) return 1;
  } else {
    if (dev_alloc(h, &h->out.jac, 2 * static_cast<size_t>(L.n_jcols) * n)) return 1;
  }
  if (dev_alloc(h, &h->out.cell, n)) return 1;
  if (dev_alloc(h, &h->out.has_jac, n)) return 1;
  if (dev_alloc(h, &h->out.evals, n)) return 1;
  h->out_trial.evals = nullptr;
  if (dev_alloc(h, &h->out_trial.residual, 2 * n)) return 1;
  if (dev_alloc(h, &h->out_trial.cost, n)) return 1;
  h->out_trial.jac = nullptr;
  h->out_trial.cjac = nullptr;
  h->out_trial.compact = 0;
  h->out_trial.cell = nullptr;
  h->out_trial.has_jac = nullptr;

  // the normal equations: one allocation (one all-reduce)
  SystemDev& s = h->sys;
  // [D | b_p | B | b_d | scalars] are all-reduced after every build; C comes last and is NOT:
  // with several ranks each rank folds its partial C into its partial Schur complement, and the
  // all-reduce of S makes it global (see solve_system).
  const int64_t oD = 0;
  const int64_t obp = oD + align32(static_cast<int64_t>(L.dsz) * L.nblocks);
  const int64_t oB = obp + align32(L.nbd);
  const int64_t obd = oB + align32(static_cast<int64_t>(L.nbd) * L.nd);
  const int64_t osc = obd + align32(L.nd);
  const int64_t oC = osc + 32;
  s.total = oC + align32(static_cast<int64_t>(L.nd) * L.nd);
  h->reduce_count = oC;
  if (dev_alloc(h, &s.base, s.total)) return 1;
  s.Dblk = s.base + oD;
  s.bp = s.base + obp;
  s.B = s.base + oB;
  s.C = s.base + oC;
  s.bd = s.base + obd;
  s.scalars = s.base + osc;
  if (dev_alloc(h, &h->d_W, static_cast<size_t>(L.nbd) * L.nd)) return 1;
  if (!h->own_dense) {
    if (dev_alloc(h, &h->d_S, static_cast<size_t>(L.nd) * L.nd + L.nd)) return 1;  // + partial rhs tail
  } else if (plan_dense(h)) {
    return 1;
  }
  if (dev_alloc(h, &h->d_Linv, static_cast<size_t>(L.dsz) * L.nblocks)) return 1;
  if (dev_alloc(h, &h->d_v, L.nbd)) return 1;
  if (dev_alloc(h, &h->d_y, L.nbd)) return 1;
  if (dev_alloc(h, &h->d_x, L.dof)) return 1;
  int lwork = 0;
  CUSOLVER_TRY(h, cusolverDnDpotrf_bufferSize(h->cusolver, CUBLAS_FILL_MODE_LOWER, L.nd, h->d_S, std::max(1, L.nd), &lwork));
  {
    int lw2 = 0;
    const int nbp = std::max(1, std::min(L.nd, h->chol_nb));
    CUSOLVER_TRY(h, cusolverDnDpotrf_bufferSize(h->cusolver, CUBLAS_FILL_MODE_LOWER, nbp, h->d_S, std::max(1, L.nd), &lw2));
    lwork = std::max(lwork, lw2);
  }
  h->potrf_lwork = lwork;
  if (dev_alloc(h, &h->d_potrf_work, std::max(1, lwork))) return 1;

  // ---- groups of Schur blocks for the structured contraction ------------------------------------
  {
    // centroid sums of the measured pixels of every pattern point (this rank's observations;
    // b200ba_comm_init all-reduces them so that every rank derives the SAME grouping)
    const int nb = L.nblocks;
    h->grp_sums.assign(3 * static_cast<size_t>(std::max(1, nb)), 0.0);
    if (L.eliminate_points) {
      for (int64_t o = 0; o < h->n_obs; ++o) {
        const int p = static_cast<int>(h->h_obs_point[o]);
        h->grp_sums[p] += h->h_obs_xy[2 * o];
        h->grp_sums[nb + p] += h->h_obs_xy[2 * o + 1];
        h->grp_sums[2 * nb + p] += 1.0;
      }
    }
    if (reduce_group_sums(h)) return 1;
    if (build_groups(h, true)) return 1;
  }
  return 0;
}

int sync_stream(b200ba_handle* h) {
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  resolve_timings(h);
  return 0;
}

int all_reduce(b200ba_handle* h, double* buf, size_t count) {
  if (h->n_ranks <= 1 || !h->comm) return 0;
  ScopedPhase ph(h, PH_ALLREDUCE);
  int rc = g_nccl.AllReduce(buf, buf, count, kNcclDouble, kNcclSum, h->comm, h->stream);
  if (rc != 0) {
    h->error = std::string("ncclAllReduce: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "error");
    return 1;
  }
  return 0;
}

// One residual pass on state `which` into `out`; jac selects Compute<true>/<false>.
// overlap_stragglers: launch the straggler pass on the side stream and return without joining
// (the caller joins with join_stragglers() after independent work).
int evaluate_state(b200ba_handle* h, int which, bool jac, const ObsOut& out, double huber, int phase,
                   bool overlap_stragglers = false) {
  launch_prepare_state(h->pb, h->L, h->st[which], h->n_control_total, h->stream);
  h->timings.kernel_launches += 1;
  {
    // [a .. mid]: main pass (what `roofline` is quoted on)
    cudaEvent_t a = get_event(h), mid = get_event(h);
    cudaEventRecord(a, h->stream);
    launch_residual_jacobian(h->uniform_model, jac, h->pb, h->L, h->st[which], h->d_last_projection, out, huber,
                             h->d_straggler_list, h->d_straggler_count, h->stream, mid);
    if (h->n_obs == 0) cudaEventRecord(mid, h->stream);
    h->pending.push_back({phase, a, mid, true});
    cudaStream_t ss = overlap_stragglers ? h->side_stream : h->stream;
    if (overlap_stragglers) CUDA_TRY(h, cudaStreamWaitEvent(h->side_stream, mid, 0));
    cudaEvent_t s0 = get_event(h), s1 = get_event(h);
    cudaEventRecord(s0, ss);
    launch_straggler_pass(h->uniform_model, jac, h->pb, h->L, h->st[which], h->d_last_projection, out, huber,
                          h->d_straggler_list, h->d_straggler_count, ss);
    cudaEventRecord(s1, ss);
    h->pending.push_back({PH_STRAGGLER, s0, s1, true});
    h->straggler_done = s1;  // stays valid until the next resolve_timings()
    h->timings.kernel_launches += 2 * (h->n_obs > 0);
  }
  CUDA_TRY(h, cudaGetLastError());
  return 0;
}

// Hot loop 1: H, b at the current state (LV/lm_optimizer.h:706-716).
int build_system(b200ba_handle* h, double huber, double* cost, double* n_valid, const b200ba_options* fix = nullptr) {
  // The straggler pass (a handful of observations burning the reference's full iteration
  // allowance) runs on the side stream underneath the accumulation of everything else.
  if (evaluate_state(h, h->cur, true, h->out, huber, PH_JAC, /*overlap_stragglers=*/true)) return 1;
  {
    ScopedPhase ph(h, PH_ACC);
    CUDA_TRY(h, cudaMemsetAsync(h->sys.base, 0, h->sys.total * sizeof(double), h->stream));
    launch_accumulate_scatter(h->pb, h->L, h->st[h->cur], h->out, h->sys, huber, h->stream);
    if (!h->L.localize_only || h->L.rig_in_state) {
      launch_accumulate_cells(h->pb, h->L, h->st[h->cur], h->out, h->sys, huber, h->stream);
      h->timings.kernel_launches += 1;
    }
    // join, then fold in the stragglers that succeeded after all
    CUDA_TRY(h, cudaStreamWaitEvent(h->stream, h->straggler_done, 0));
    launch_accumulate_list(h->pb, h->L, h->st[h->cur], h->out, h->sys, huber, h->d_straggler_list, h->d_straggler_count, h->stream);
    h->timings.kernel_launches += 2;
    launch_cost_reduce(h->n_obs, h->out.cost, nullptr, h->out.residual, h->d_partial, h->sys.scalars, h->stream);
    // trace(H) of this rank's partial system, for the lambda initialisation (lm_optimizer.h:766-781)
    launch_trace(h->L.nblocks, h->L.bs, h->sys.Dblk, h->L.nd, h->sys.C, h->sys.scalars + 8, h->stream);
    h->timings.kernel_launches += 3;
  }
  CUDA_TRY(h, cudaGetLastError());
  // ONE all-reduce per build covers D, b_p, B, b_d, the cost scalars and the trace (SURVEY.md 8e)
  if (all_reduce(h, h->sys.base, static_cast<size_t>(h->reduce_count))) return 1;
  if (fix) {
    // FixVariable (joint_optimization.cc:878-903): mask the fixed unknowns out of H, b. The trace for the
    // lambda initialisation was taken from the full H, like the reference does before it thins the system.
    const Layout& L = h->L;
    FixedRanges fr{};
    auto add = [&](int g0, int count) {
      if (count > 0 && fr.n < 4) {
        fr.lo[fr.n] = g0;
        fr.hi[fr.n] = g0 + count;
        fr.n++;
      }
    };
    int n_intr = 0;
    for (int c = 0; c < h->n_cameras; ++c) n_intr += update_parameter_count(h->cams_host[c]);
    if (fix->debug_fix_points) add(L.g_point, 3 * L.n_points);
    if (fix->debug_fix_poses) add(L.g_pose, 6 * L.n_imagesets);
    if (fix->debug_fix_rig_poses && L.rig_in_state) add(L.g_rig, 6 * L.n_cameras);
    if (fix->debug_fix_intrinsics && !L.localize_only) add(L.g_intr, n_intr);
    // with several ranks C is a partial sum: rank 0 alone carries the unit diagonal of the fixed dense unknowns
    launch_mask_fixed(L, h->sys, fr, h->rank == 0 ? 1.0 : 0.0, h->stream);
    h->timings.kernel_launches += 3;
  }
  CUDA_TRY(h, cudaMemcpyAsync(h->h_scal, h->sys.scalars, 9 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if (h->n_groups > 0 && h->L.nd > 0 && h->force_grouped != 0) {
    // exact column support of every group of Schur blocks, from the (global) B itself
    ScopedPhase ph(h, PH_SCHUR);
    CUDA_TRY(h, cudaMemsetAsync(h->d_flags, 0, static_cast<size_t>(h->n_groups) * h->L.nd, h->stream));
    launch_group_support(h->L.bs, h->L.nblocks, h->L.nd, h->sys.B, h->d_group_of_block, h->d_flags, h->stream);
    launch_compact_columns(h->n_groups, h->L.nd, h->d_flags, h->d_cols, h->d_count, h->stream);
    CUDA_TRY(h, cudaMemcpyAsync(h->h_count, h->d_count, h->n_groups * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    h->timings.kernel_launches += 2;
  }
  if (sync_stream(h)) return 1;
  *cost = h->h_scal[3];
  *n_valid = h->h_scal[4];
  h->trace_H = h->h_scal[8];
  // cost model: grouped contraction sum_g k_g m_g^2 (+ scatter) against the dense n_d^2 * nbd
  h->use_grouped = false;
  if (h->n_groups > 0 && h->L.nd > 0 && h->force_grouped != 0) {
    double grouped = 0;
    for (int g = 0; g < h->n_groups; ++g) {
      const double kg = static_cast<double>(h->group_start[g + 1] - h->group_start[g]) * h->L.bs;
      const double mg = h->h_count[g];
      h->group_count[g] = h->h_count[g];
      grouped += mg * mg * (kg + 24.0);  // + ~24 flop-equivalents per scattered entry
    }
    const double dense = static_cast<double>(h->L.nd) * h->L.nd * h->L.nbd;
    h->use_grouped = (h->force_grouped == 1) || grouped < 0.6 * dense;
  }
  return 0;
}

__global__ void fold_panel_info_kernel(const int* __restrict__ panel_info, int n, int* __restrict__ info) {
  int worst = 0;
  for (int i = threadIdx.x; i < n; i += 32) worst = max(worst, panel_info[i] != 0 ? 1 : 0);
  for (int o = 16; o > 0; o >>= 1) worst = max(worst, __shfl_xor_sync(0xffffffffu, worst, o));
  if (threadIdx.x == 0) info[0] = worst;
}

// Cholesky factorisation of the reduced system S (column-major, lower) in place; info[0] != 0
// when a pivot was not positive.
//   default: cusolverDnDpotrf on the whole matrix (replicated on every rank).
//   B200BA_DIST_CHOL=1: right-looking factorisation over column blocks of width nb, dealt round-robin
//   to the ranks. The owner of block k factors its diagonal tile and solves the tile column below
//   it, broadcasts the finished column block (whole columns: contiguous in the column-major S),
//   then every rank applies the rank-nb update to the column blocks IT owns. Each rank thereby
//   does 1/N of the n^3/3 update flops instead of all of them, and ends with the complete L (its
//   own blocks computed, the others received), so the triangular solves stay local.
int factor_dense(b200ba_handle* h) {
  const Layout& L = h->L;
  const int nd = L.nd;
  const int nb = h->chol_nb;
  const int nblk = (nd + nb - 1) / nb;
  // Opt-in (B200BA_DIST_CHOL=1): the panel chain (potrf(nb) + trsm + broadcast per column block) is
  // serial without look-ahead, so the replicated potrf stays the default.
  bool blocked = (h->chol_mode == 1) && nd > nb;
  if (nblk > kMaxCholPanels) blocked = false;
  if (!blocked) {
    CUSOLVER_TRY(h, cusolverDnDpotrf(h->cusolver, CUBLAS_FILL_MODE_LOWER, nd, h->d_S, nd, h->d_potrf_work, h->potrf_lwork,
                                     h->d_info));
    return 0;
  }
  const double one = 1.0, minus_one = -1.0;
  int* panel_info = h->d_info + 2;
  CUDA_TRY(h, cudaMemsetAsync(panel_info, 0, nblk * sizeof(int), h->stream));
  for (int k = 0; k < nblk; ++k) {
    const int owner = k % h->n_ranks;
    const int j0 = k * nb, w = std::min(nb, nd - j0), below = nd - j0 - w;
    double* Akk = h->d_S + static_cast<size_t>(j0) * nd + j0;
    if (h->rank == owner) {
      CUSOLVER_TRY(h, cusolverDnDpotrf(h->cusolver, CUBLAS_FILL_MODE_LOWER, w, Akk, nd, h->d_potrf_work, h->potrf_lwork,
                                       panel_info + k));
      if (below > 0)  // L_below = A_below L_kk^-T
        CUBLAS_TRY(h, cublasDtrsm(h->cublas, CUBLAS_SIDE_RIGHT, CUBLAS_FILL_MODE_LOWER, CUBLAS_OP_T, CUBLAS_DIAG_NON_UNIT, below,
                                  w, &one, Akk, nd, Akk + w, nd));
    }
    if (h->n_ranks > 1 && h->comm) {
      double* col = h->d_S + static_cast<size_t>(j0) * nd;
      const int rc = g_nccl.Broadcast(col, col, static_cast<size_t>(nd) * w, kNcclDouble, owner, h->comm, h->stream);
      if (rc != 0) {
        h->error = std::string("ncclBroadcast: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "error");
        return 1;
      }
    }
    // trailing update of the column blocks this rank owns
    for (int j = k + 1; j < nblk; ++j) {
      if (j % h->n_ranks != h->rank) continue;
      const int c0 = j * nb, wj = std::min(nb, nd - c0);
      const double* Lj = h->d_S + static_cast<size_t>(j0) * nd + c0;  // rows c0.. of column block k
      CUBLAS_TRY(h, cublasDgemm(h->cublas, CUBLAS_OP_N, CUBLAS_OP_T, nd - c0, wj, w, &minus_one, Lj, nd, Lj, nd, &one,
                                h->d_S + static_cast<size_t>(c0) * nd + c0, nd));
    }
  }
  fold_panel_info_kernel<<<1, 32, 0, h->stream>>>(panel_info, nblk, h->d_info);
  if (h->n_ranks > 1 && h->comm) {
    // every rank must take the same branch of the LM loop
    const int rc = g_nccl.AllReduce(h->d_info, h->d_info, 1, kNcclInt32, kNcclMax, h->comm, h->stream);
    if (rc != 0) {
      h->error = "ncclAllReduce (factorisation status) failed";
      return 1;
    }
  }
  return 0;
}

// b200ba_debug_solve_step (one rank): downloads S + lambda I as the factorisation will see it, un-mapped to a plain
// column-major n_d x n_d array, and the reduced right-hand side.
int capture_reduced_system(b200ba_handle* h) {
  const Layout& L = h->L;
  const int nd = L.nd;
  if (nd > 0) {
    if (h->own_dense) {
      const DenseCtx& d = h->dn;
      for (int j = 0; j < d.nblk; ++j) {
        const int c0 = j * d.NB, w = std::min(d.NB, nd - c0);
        CUDA_TRY(h, cudaMemcpy2DAsync(h->capture_S + static_cast<size_t>(c0) * nd, static_cast<size_t>(nd) * sizeof(double),
                                      h->d_S + d.map.col_offset(c0), d.map.ld * sizeof(double),
                                      static_cast<size_t>(nd) * sizeof(double), w, cudaMemcpyDeviceToHost, h->stream));
      }
    } else {
      CUDA_TRY(h, cudaMemcpyAsync(h->capture_S, h->d_S, static_cast<size_t>(nd) * nd * sizeof(double), cudaMemcpyDeviceToHost,
                                  h->stream));
    }
    CUDA_TRY(h, cudaMemcpyAsync(h->capture_rhs, h->d_x + L.nbd, static_cast<size_t>(nd) * sizeof(double),
                                cudaMemcpyDeviceToHost, h->stream));
  }
  return sync_stream(h);
}

// Hot loop 2: Schur complement solve for a given lambda (LV/lm_optimizer.h:1246-1369).
// Leaves x = [x_points | x_dense] in d_x. *spd = 0 when a factorisation met a non-positive pivot.
int solve_system_own(b200ba_handle* h, double lambda, int* spd);

int solve_system(b200ba_handle* h, double lambda, int* spd) {
  if (h->own_dense) return solve_system_own(h, lambda, spd);
  const Layout& L = h->L;
  const double one = 1.0, minus_one = -1.0;
  bool grouped_done = false;
  if (h->use_grouped) {
    // ---- structured contraction: per group gather -> compact rank-k update -> scatter ----------
    ScopedPhase ph(h, PH_SCHUR);
    const double zero = 0.0;
    CUDA_TRY(h, cudaMemsetAsync(h->d_fail, 0, sizeof(int), h->stream));
    launch_schur_blocks(L.bs, L.nblocks, h->sys.Dblk, h->sys.bp, lambda, h->d_Linv, h->d_v, h->d_fail, h->stream);
    // S = C_r is copied on the side stream (0.4 ms of pure HBM traffic at config 2) underneath the
    // block factorisations and the first rank-k update; the scatters follow it in stream order.
    CUDA_TRY(h, cudaEventRecord(h->ev_s_ready, h->stream));  // everything that used S before is done
    CUDA_TRY(h, cudaStreamWaitEvent(h->side_stream, h->ev_s_ready, 0));
    CUDA_TRY(h, cudaMemcpyAsync(h->d_S, h->sys.C, static_cast<size_t>(L.nd) * L.nd * sizeof(double),
                                cudaMemcpyDeviceToDevice, h->side_stream));
    CUDA_TRY(h, cudaEventRecord(h->ev_s_ready, h->side_stream));
    launch_block_solve_t(L.bs, L.nblocks, h->d_Linv, h->d_v, h->d_u, h->stream);  // u = D^-1 b_block
    h->timings.kernel_launches += 2;
    // The compact rank-k updates (compute-bound, main stream) and the scatters into S (memory-
    // bound, side stream) are software-pipelined over two P / Wc buffers. All scatters run on the
    // side stream, hence in order: plain read-modify-write, no atomics.
    int it = 0;
    for (int g = h->rank; g < h->n_groups; g += h->n_ranks) {
      const int nblk = h->group_start[g + 1] - h->group_start[g];
      const int kg = nblk * L.bs, mg = h->group_count[g];
      if (mg == 0 || kg == 0) continue;
      h->timings.contraction_flops += static_cast<double>(mg) * mg * kg;
      const int b = it & 1;
      double* Wc = h->d_Wc + b * h->wc_stride;
      double* P = h->d_P + b * h->p_stride;
      const int* cols = h->d_cols + static_cast<size_t>(g) * L.nd;
      if (it >= 2) CUDA_TRY(h, cudaStreamWaitEvent(h->stream, h->ev_scatter[b], 0));  // buffer b is free again
      launch_gather_scale(L.bs, nblk, L.nd, mg, mg, h->sys.B, h->d_Linv, h->d_group_blocks + h->group_start[g], cols, Wc,
                          h->stream);
      // row-major Wc [kg x mg] is the column-major mg x kg panel: P = Wc^T Wc (lower)
      CUBLAS_TRY(h, cublasDsyrk(h->cublas, CUBLAS_FILL_MODE_LOWER, CUBLAS_OP_N, mg, kg, &one, Wc, mg, &zero, P, mg));
      CUDA_TRY(h, cudaEventRecord(h->ev_syrk[b], h->stream));
      CUDA_TRY(h, cudaStreamWaitEvent(h->side_stream, h->ev_syrk[b], 0));
      launch_scatter_sub(L.nd, mg, cols, P, h->d_S, h->side_stream);
      CUDA_TRY(h, cudaEventRecord(h->ev_scatter[b], h->side_stream));
      h->timings.kernel_launches += 2;
      ++it;
    }
    // join: every scatter has landed before S is used
    CUDA_TRY(h, cudaStreamWaitEvent(h->stream, h->ev_s_ready, 0));  // the copy (covers a rank without groups)
    for (int b = 0; b < 2 && b < it; ++b) CUDA_TRY(h, cudaStreamWaitEvent(h->stream, h->ev_scatter[b], 0));
    grouped_done = true;
  }
  if (grouped_done) {
    if (h->n_ranks > 1) {
      if (all_reduce(h, h->d_S, static_cast<size_t>(L.nd) * L.nd)) return 1;
    }
    ScopedPhase ph(h, PH_SCHUR);
    launch_add_diagonal(L.nd, h->d_S, L.nd, lambda, h->stream);
    // x_dense <- b_d - B^T u   (B is global after the per-build all-reduce: no partial sums here)
    CUDA_TRY(h, cudaMemcpyAsync(h->d_x + L.nbd, h->sys.bd, L.nd * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
    if (L.nbd > 0 && L.nd > 0)
      CUBLAS_TRY(h, cublasDgemv(h->cublas, CUBLAS_OP_N, L.nd, L.nbd, &minus_one, h->sys.B, L.nd, h->d_u, 1, &one,
                                h->d_x + L.nbd, 1));
    h->timings.kernel_launches += 1;
  } else {
    // Point range of this rank for the contraction: S = sum_r (C_r - W_r^T W_r) + lambda I, where
    // C_r is the rank's partial dense block and W_r the rows of W = L^-1 B of its points (B, D are
    // global after the per-build all-reduce). With one rank this is the plain S = C + lambda I - W^T W.
    const int p0 = static_cast<int>(static_cast<int64_t>(L.nblocks) * h->rank / h->n_ranks);
    const int p1 = static_cast<int>(static_cast<int64_t>(L.nblocks) * (h->rank + 1) / h->n_ranks);
    const int k_rows = L.bs * (p1 - p0);
    double* rhs_tail = h->d_S + static_cast<size_t>(L.nd) * L.nd;
    {
      ScopedPhase ph(h, PH_SCHUR);
      CUDA_TRY(h, cudaMemsetAsync(h->d_fail, 0, sizeof(int), h->stream));
      launch_schur_blocks(L.bs, L.nblocks, h->sys.Dblk, h->sys.bp, lambda, h->d_Linv, h->d_v, h->d_fail, h->stream);
      launch_schur_scale_rows(L.bs, L.nblocks, L.nd, h->sys.B, h->d_Linv, h->d_W, h->stream);
      CUDA_TRY(h, cudaMemcpyAsync(h->d_S, h->sys.C, static_cast<size_t>(L.nd) * L.nd * sizeof(double),
                                  cudaMemcpyDeviceToDevice, h->stream));
      CUDA_TRY(h, cudaMemsetAsync(rhs_tail, 0, L.nd * sizeof(double), h->stream));
      h->timings.kernel_launches += 2;
      if (k_rows > 0 && L.nd > 0) {
        h->timings.contraction_flops += static_cast<double>(L.nd) * L.nd * k_rows;
        const double zero = 0.0;
        const double* Wr = h->d_W + static_cast<size_t>(L.bs) * p0 * L.nd;
        // row-major W [nbd x nd] is the column-major nd x nbd matrix W^T: S -= W_r^T W_r (lower)
        CUBLAS_TRY(h, cublasDsyrk(h->cublas, CUBLAS_FILL_MODE_LOWER, CUBLAS_OP_N, L.nd, k_rows, &minus_one, Wr, L.nd,
                                  &one, h->d_S, L.nd));
        // partial reduced right-hand side: -W_r^T v_r
        CUBLAS_TRY(h, cublasDgemv(h->cublas, CUBLAS_OP_N, L.nd, k_rows, &minus_one, Wr, L.nd, h->d_v + L.bs * p0, 1, &zero,
                                  rhs_tail, 1));
      }
    }
    if (h->n_ranks > 1) {
      if (all_reduce(h, h->d_S, static_cast<size_t>(L.nd) * L.nd + L.nd)) return 1;
    }
    {
      ScopedPhase ph(h, PH_SCHUR);
      launch_add_diagonal(L.nd, h->d_S, L.nd, lambda, h->stream);
      // x_dense <- b_d - W^T v
      CUDA_TRY(h, cudaMemcpyAsync(h->d_x + L.nbd, h->sys.bd, L.nd * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
      CUBLAS_TRY(h, cublasDaxpy(h->cublas, L.nd, &one, rhs_tail, 1, h->d_x + L.nbd, 1));
      h->timings.kernel_launches += 1;
    }
  }
  if (h->capture_S && capture_reduced_system(h)) return 1;
  {
    ScopedPhase ph(h, PH_FACTOR);
    if (factor_dense(h)) return 1;
    h->timings.factor_flops += static_cast<double>(L.nd) * L.nd * L.nd / 3.0;
  }
  {
    ScopedPhase ph(h, PH_SOLVE);
    CUSOLVER_TRY(h, cusolverDnDpotrs(h->cusolver, CUBLAS_FILL_MODE_LOWER, L.nd, 1, h->d_S, L.nd, h->d_x + L.nbd, L.nd,
                                     h->d_info + 1));
  }
  if (grouped_done) {
    ScopedPhase ph(h, PH_SCHUR);
    // t = B x_d ; x_block = u - D^-1 t   (W is never materialised on this path)
    const double zero = 0.0;
    if (L.nbd > 0 && L.nd > 0)
      CUBLAS_TRY(h, cublasDgemv(h->cublas, CUBLAS_OP_T, L.nd, L.nbd, &one, h->sys.B, L.nd, h->d_x + L.nbd, 1, &zero,
                                h->d_y, 1));
    launch_block_backsub2(L.bs, L.nblocks, h->d_Linv, h->d_u, h->d_y, h->d_x, h->stream);
    h->timings.kernel_launches += 1;
  } else {
    ScopedPhase ph(h, PH_SCHUR);
    // y = v - W x_d ; x_p = L^-T y
    CUDA_TRY(h, cudaMemcpyAsync(h->d_y, h->d_v, L.nbd * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
    if (L.nbd > 0 && L.nd > 0)
      CUBLAS_TRY(h, cublasDgemv(h->cublas, CUBLAS_OP_T, L.nd, L.nbd, &minus_one, h->d_W, L.nd, h->d_x + L.nbd, 1, &one,
                                h->d_y, 1));
    launch_schur_backsub(L.bs, L.nblocks, h->d_Linv, h->d_y, h->d_x, h->stream);
    h->timings.kernel_launches += 1;
  }
  CUDA_TRY(h, cudaMemcpyAsync(h->h_flags, h->d_info, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(h->h_flags + 1, h->d_fail, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  if (sync_stream(h)) return 1;
  *spd = (h->h_flags[0] == 0 && h->h_flags[1] == 0) ? 1 : 0;
  return 0;
}

// The same solve on the in-tree kernels (ba_dense.cu): the contraction is a DMMA product whose epilogue
// scatters straight into S, the reduced system is factorised by a blocked right-looking Cholesky with
// look-ahead (block columns dealt cyclically to the ranks, panels broadcast over NVLink), the
// triangular solves run on the packed factor. With several ranks S is formed as partial sums
// S_r = C_r - sum_{g of r} W_g^T W_g that ONE reduce-scatter per attempt turns into the block columns each
// rank owns; nobody holds or reduces the whole matrix.
int solve_system_own(b200ba_handle* h, double lambda, int* spd) {
  const Layout& L = h->L;
  DenseCtx& d = h->dn;
  const int nd = L.nd, R = h->n_ranks;
  {
    ScopedPhase ph(h, PH_SCHUR);
    CUDA_TRY(h, cudaMemsetAsync(h->d_fail, 0, sizeof(int), h->stream));
    CUDA_TRY(h, cudaMemsetAsync(h->d_info, 0, sizeof(int), h->stream));
    launch_schur_blocks(L.bs, L.nblocks, h->sys.Dblk, h->sys.bp, lambda, h->d_Linv, h->d_v, h->d_fail, h->stream);
    // S <- C_r (this rank's partial dense block) through the storage map, on the side stream
    // underneath the block factorisations and the first gather
    CUDA_TRY(h, cudaEventRecord(h->ev_s_ready, h->stream));  // everything that used S before is done
    CUDA_TRY(h, cudaStreamWaitEvent(h->side_stream, h->ev_s_ready, 0));
    if (nd > 0) {
      if (R == 1) {
        CUDA_TRY(h, cudaMemcpy2DAsync(h->d_S, d.map.ld * sizeof(double), h->sys.C, static_cast<size_t>(nd) * sizeof(double),
                                      static_cast<size_t>(nd) * sizeof(double), nd, cudaMemcpyDeviceToDevice, h->side_stream));
      } else {
        for (int j = 0; j < d.nblk; ++j) {
          const int c0 = j * d.NB, w = std::min(d.NB, nd - c0);
          CUDA_TRY(h, cudaMemcpy2DAsync(h->d_S + d.map.col_offset(c0), d.map.ld * sizeof(double),
                                        h->sys.C + static_cast<size_t>(c0) * nd, static_cast<size_t>(nd) * sizeof(double),
                                        static_cast<size_t>(nd) * sizeof(double), w, cudaMemcpyDeviceToDevice, h->side_stream));
        }
      }
    }
    CUDA_TRY(h, cudaEventRecord(h->ev_s_ready, h->side_stream));
    launch_block_solve_t(L.bs, L.nblocks, h->d_Linv, h->d_v, h->d_u, h->stream);  // u = D^-1 b_block
    h->timings.kernel_launches += 2;
    bool joined = false;
    auto join_copy = [&]() {
      if (!joined) cudaStreamWaitEvent(h->stream, h->ev_s_ready, 0);
      joined = true;
    };
    if (h->use_grouped) {
      // structured contraction: per group gather -> DMMA rank-k update with the scatter epilogue
      int it = 0;
      for (int g = h->rank; g < h->n_groups; g += R) {
        const int nblk = h->group_start[g + 1] - h->group_start[g];
        const int kg = nblk * L.bs, mg = h->group_count[g];
        if (mg == 0 || kg == 0) continue;
        const int ldw = (mg + 1) / 2 * 2;
        double* Wc = h->d_Wc + (it & 1) * h->wc_stride;
        const int* cols = h->d_cols + static_cast<size_t>(g) * nd;
        launch_gather_scale(L.bs, nblk, nd, mg, ldw, h->sys.B, h->d_Linv, h->d_group_blocks + h->group_start[g], cols, Wc,
                            h->stream);
        join_copy();
        GemmArgs ga{};
        ga.M = ga.N = mg;
        ga.K = kg;
        ga.A = ga.B = Wc;
        ga.lda = ga.ldb = ldw;
        ga.C = h->d_S;
        ga.alpha = -1.0;
        ga.beta = 1.0;
        ga.a_aligned = ga.b_aligned = gemm_operand_aligned(Wc, ldw);
        ga.cols = cols;
        ga.map = d.map;
        if (launch_dgemm_nt(ga, true, true, h->stream)) {
          h->error = "dgemm_nt (contraction) launch failed";
          return 1;
        }
        h->timings.contraction_flops += static_cast<double>(mg) * mg * kg;
        h->timings.kernel_launches += 2;
        ++it;
      }
    } else if (L.nbd > 0 && nd > 0) {
      // dense contraction over this rank's slice of the Schur blocks: S_r -= W_r^T W_r
      const int p0 = static_cast<int>(static_cast<int64_t>(L.nblocks) * h->rank / R);
      const int p1 = static_cast<int>(static_cast<int64_t>(L.nblocks) * (h->rank + 1) / R);
      const int k_rows = L.bs * (p1 - p0);
      launch_schur_scale_rows(L.bs, L.nblocks, nd, h->sys.B, h->d_Linv, h->d_W, h->stream);
      h->timings.kernel_launches += 1;
      if (k_rows > 0) {
        const double* Wr = h->d_W + static_cast<size_t>(L.bs) * p0 * nd;
        join_copy();
        GemmArgs ga{};
        ga.M = ga.N = nd;
        ga.K = k_rows;
        ga.A = ga.B = Wr;
        ga.lda = ga.ldb = nd;
        ga.C = h->d_S;
        ga.ldc = d.map.ld;
        ga.alpha = -1.0;
        ga.beta = 1.0;
        ga.a_aligned = ga.b_aligned = gemm_operand_aligned(Wr, nd);
        ga.cols = h->d_ident_cols;
        ga.map = d.map;
        if (launch_dgemm_nt(ga, true, /*scatter=*/R > 1, h->stream)) {
          h->error = "dgemm_nt (contraction) launch failed";
          return 1;
        }
        h->timings.contraction_flops += static_cast<double>(nd) * nd * k_rows;
        h->timings.kernel_launches += 1;
      }
    }
    join_copy();
    if (h->rank == 0) launch_add_diagonal_map(nd, h->d_S, d.map, lambda, h->stream);
    // x_dense <- b_d - B^T u   (B, D, b are global after the per-build all-reduce)
    CUDA_TRY(h, cudaMemcpyAsync(h->d_x + L.nbd, h->sys.bd, nd * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
    if (L.nbd > 0 && nd > 0) launch_gemv_t(L.nbd, nd, nd, h->sys.B, h->d_u, -1.0, h->d_x + L.nbd, h->d_gemv_partial, h->stream);
    h->timings.kernel_launches += 4;
  }
  if (h->capture_S && capture_reduced_system(h)) return 1;
  if (R > 1 && nd > 0) {
    // partial sums -> the block columns each rank owns (in place: rank r keeps chunk r)
    ScopedPhase ph(h, PH_ALLREDUCE);
    const int rc = g_nccl.ReduceScatter(h->d_S, h->d_S + static_cast<size_t>(h->rank) * d.chunk, static_cast<size_t>(d.chunk),
                                        kNcclDouble, kNcclSum, h->comm, h->stream);
    if (rc != 0) {
      h->error = std::string("ncclReduceScatter: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "error");
      return 1;
    }
  }
  {
    ScopedPhase ph(h, PH_FACTOR);
    if (dense_factor(&d)) {
      if (h->error.empty()) h->error = "dense_factor: launch failed";
      return 1;
    }
    h->timings.factor_flops += static_cast<double>(nd) * nd * nd / 3.0;
    if (R > 1) {
      // every rank must take the same branch of the LM loop
      const int rc = g_nccl.AllReduce(h->d_info, h->d_info, 1, kNcclInt32, kNcclMax, h->comm, h->stream);
      if (rc != 0) {
        h->error = "ncclAllReduce (factorisation status) failed";
        return 1;
      }
    }
  }
  {
    ScopedPhase ph(h, PH_SOLVE);
    if (dense_solve(&d, h->d_x + L.nbd)) {
      h->error = "dense_solve: launch failed";
      return 1;
    }
    h->timings.kernel_launches += 4 * d.ntiles;
  }
  {
    ScopedPhase ph(h, PH_SCHUR);
    // t = B x_d ; x_block = u - D^-1 t   (W is never needed for the back-substitution)
    if (L.nbd > 0 && nd > 0)
      launch_gemv_n(L.nbd, nd, nd, h->sys.B, h->d_x + L.nbd, h->d_y, h->stream);
    else if (L.nbd > 0)
      CUDA_TRY(h, cudaMemsetAsync(h->d_y, 0, L.nbd * sizeof(double), h->stream));
    launch_block_backsub2(L.bs, L.nblocks, h->d_Linv, h->d_u, h->d_y, h->d_x, h->stream);
    h->timings.kernel_launches += 1;
  }
  CUDA_TRY(h, cudaMemcpyAsync(h->h_flags, h->d_info, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(h->h_flags + 1, h->d_fail, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  if (sync_stream(h)) return 1;
  *spd = (h->h_flags[0] == 0 && h->h_flags[1] == 0) ? 1 : 0;
  return 0;
}

int check_ready(b200ba_handle* h, const b200ba_options* opt) {
  if (!h) return 1;
  if (!opt) {
    h->error = "options are NULL";
    return 2;
  }
  if (!h->have_state) {
    h->error = "no state: call b200ba_set_state first";
    return 2;
  }
  CUDA_TRY(h, cudaSetDevice(h->device));
  return make_layout(h, opt);
}

void free_handle_buffers(b200ba_handle* h) {
  auto F = [](auto*& p) {
    if (p) cudaFree(p);
    p = nullptr;
  };
  F(h->d_obs_imageset); F(h->d_obs_camera); F(h->d_obs_point); F(h->d_obs_xy);
  for (int i = 0; i < 2; ++i) {
    F(h->st[i].points); F(h->st[i].rig_tr_global); F(h->st[i].camera_tr_rig); F(h->st[i].intrinsics);
    F(h->st[i].image_tr_global); F(h->st[i].tangents);
  }
  F(h->d_last_projection);
  F(h->snap.points); F(h->snap.rig_tr_global); F(h->snap.camera_tr_rig); F(h->snap.intrinsics); F(h->d_snap_lp);
  h->have_snapshot = false;
  F(h->out.residual); F(h->out.cost); F(h->out.jac); F(h->out.cjac); F(h->out.cell); F(h->out.has_jac); F(h->out.evals);
  F(h->out_trial.residual); F(h->out_trial.cost);
  F(h->sys.base); F(h->d_W); F(h->d_S); F(h->d_Linv); F(h->d_v); F(h->d_y); F(h->d_x); F(h->d_potrf_work);
  F(h->d_info); F(h->d_fail); F(h->d_straggler_list); F(h->d_straggler_count); F(h->d_perm); F(h->d_lp_stage);
  F(h->d_group_of_block); F(h->d_group_blocks); F(h->d_flags); F(h->d_cols); F(h->d_count); F(h->d_Wc); F(h->d_P); F(h->d_u);
  if (h->h_count) cudaFreeHost(h->h_count);
  h->h_count = nullptr;
  F(h->d_partial); F(h->d_scal); F(h->d_rot);
  F(h->rep.err); F(h->rep.mag); F(h->rep.cam_off); F(h->rep.cell_off); F(h->rep.cell_order); F(h->rep.Q);
  F(h->rep.partial); F(h->rep.select_hist); F(h->rep.hist); F(h->rep.kl); F(h->rep.cams); F(h->d_rep_stage);
  h->have_report = false;
  F(h->d_img_group_off); F(h->d_img_group_obs);
  h->have_images = false;
  F(h->dn.Lpack); F(h->dn.tmp); F(h->dn.d_panel_off); F(h->dn.d_panel_h); F(h->d_ident_cols); F(h->d_gemv_partial);
  h->dn.S = nullptr;
  h->dense_planned_n = -1;
  if (h->h_scal) cudaFreeHost(h->h_scal);
  if (h->h_flags) cudaFreeHost(h->h_flags);
  h->h_scal = nullptr;
  h->h_flags = nullptr;
}

// First b200ba_calibration_report: allocates the report's buffers and uploads what depends on the problem
// only -- the camera ranges of the device order, the ordering by (camera, bias cell) and the Gaussian table
// of ComputeBiasedness (calibration_report.cc:241-258, computed here with std::exp).
int setup_report(b200ba_handle* h) {
  if (h->have_report) return 0;
  const int64_t n = h->n_obs;
  const int nc = h->n_cameras;
  constexpr int kCells = kReportBiasCells * kReportBiasCells;
  // the device order is sorted by camera first (b200ba_create): each camera is one range
  std::vector<int64_t> cam_off(nc + 1, 0);
  for (int64_t o = 0; o < n; ++o) ++cam_off[h->h_obs_camera[o] + 1];
  for (int c = 0; c < nc; ++c) cam_off[c + 1] += cam_off[c];
  // bias cell of every observation (:225-235): step = (max - min) / 50.0 + 1e-7; the subtraction
  // xy - min is float - int in float, the division is in double, the conversion truncates
  std::vector<uint32_t> key(n);
  std::vector<int> cell_off(static_cast<size_t>(nc) * kCells + 1, 0);
  for (int64_t o = 0; o < n; ++o) {
    const uint32_t cam = h->h_obs_camera[o];
    const b200ba_camera& c = h->cams_host[cam];
    const double step_u = static_cast<double>(c.calibration_max_x - c.calibration_min_x) / kReportBiasCells + 1e-7;
    const double step_v = static_cast<double>(c.calibration_max_y - c.calibration_min_y) / kReportBiasCells + 1e-7;
    const float dx = h->h_obs_xy[2 * o] - static_cast<float>(c.calibration_min_x);
    const float dy = h->h_obs_xy[2 * o + 1] - static_cast<float>(c.calibration_min_y);
    const int cx = std::min(kReportBiasCells - 1, std::max(0, static_cast<int>(dx / step_u)));
    const int cy = std::min(kReportBiasCells - 1, std::max(0, static_cast<int>(dy / step_v)));
    key[o] = cam * kCells + cy * kReportBiasCells + cx;
    ++cell_off[key[o] + 1];
  }
  for (size_t k = 0; k + 1 < cell_off.size(); ++k) cell_off[k + 1] += cell_off[k];
  // stable counting sort by key: the caller's order inside each cell; entries are device positions
  std::vector<uint32_t> pos(n), order(n);
  for (int64_t i = 0; i < n; ++i) pos[h->perm[i]] = static_cast<uint32_t>(i);
  {
    std::vector<int> fill(cell_off.begin(), cell_off.end() - 1);
    for (int64_t o = 0; o < n; ++o) order[fill[key[o]]++] = pos[o];
  }
  // Q(x, y) = exp(-0.5 (dx^2 + dy^2)), dx = (2.5 / (0.5 * 8)) * (0.5 * 8 - (x + 0.5)), normalised; y-major
  double Q[64], q_sum = 0;
  for (int y = 0; y < 8; ++y)
    for (int x = 0; x < 8; ++x) {
      const double dx = (2.5 / (0.5 * 8)) * (0.5 * 8 - (x + 0.5));
      const double dy = (2.5 / (0.5 * 8)) * (0.5 * 8 - (y + 0.5));
      const double p = std::exp(-0.5 * (dx * dx + dy * dy));
      Q[y * 8 + x] = p;
      q_sum += p;
    }
  for (double& q : Q) q /= q_sum;
  ReportDev& r = h->rep;
  if (dev_alloc(h, &r.err, n) || dev_alloc(h, &r.mag, n) || dev_alloc(h, &r.cam_off, nc + 1) ||
      dev_alloc(h, &r.cell_off, cell_off.size()) || dev_alloc(h, &r.cell_order, n) || dev_alloc(h, &r.Q, 64) ||
      dev_alloc(h, &r.partial, report_partial_size(nc)) || dev_alloc(h, &r.select_hist, 256 * nc) ||
      dev_alloc(h, &r.hist, static_cast<size_t>(nc) * B200BA_REPORT_HIST * B200BA_REPORT_HIST) ||
      dev_alloc(h, &r.kl, static_cast<size_t>(nc) * kCells) || dev_alloc(h, &r.cams, nc) || dev_alloc(h, &h->d_rep_stage, n))
    return 1;
  CUDA_TRY(h, cudaMemcpy(r.cam_off, cam_off.data(), cam_off.size() * sizeof(int64_t), cudaMemcpyHostToDevice));
  CUDA_TRY(h, cudaMemcpy(r.cell_off, cell_off.data(), cell_off.size() * sizeof(int), cudaMemcpyHostToDevice));
  if (n > 0) CUDA_TRY(h, cudaMemcpy(r.cell_order, order.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice));
  CUDA_TRY(h, cudaMemcpy(r.Q, Q, sizeof(Q), cudaMemcpyHostToDevice));
  h->have_report = true;
  return 0;
}

// First b200ba_report_images: groups every camera's observations by their integer feature pixel
// ((int)x, (int)y) as CreateVoronoiDiagram de-duplicates them (calibration_report.cc:366-383), the caller's order
// inside a group. Its de-duplication image is 4W x 4H and indexed at (ix, iy), so observations outside
// 0 <= ix < 4W, 0 <= iy < 4H (undefined there) are left out.
int setup_images(b200ba_handle* h) {
  if (h->have_images) return 0;
  const int64_t n = h->n_obs;
  const int nc = h->n_cameras;
  std::vector<uint32_t> pos(n);
  for (int64_t i = 0; i < n; ++i) pos[h->perm[i]] = static_cast<uint32_t>(i);
  std::vector<std::pair<int64_t, uint32_t>> keyed;  // (camera-major key, caller index)
  keyed.reserve(n);
  for (int64_t o = 0; o < n; ++o) {
    const b200ba_camera& c = h->cams_host[h->h_obs_camera[o]];
    const float x = h->h_obs_xy[2 * o], y = h->h_obs_xy[2 * o + 1];
    if (!(x > -1.f && y > -1.f && x < 4.f * c.width && y < 4.f * c.height)) continue;
    const int64_t ix = static_cast<int>(x), iy = static_cast<int>(y);
    if (ix >= 4 * static_cast<int64_t>(c.width) || iy >= 4 * static_cast<int64_t>(c.height)) continue;
    const int64_t key = (static_cast<int64_t>(h->h_obs_camera[o]) << 40) | (iy * 4 * c.width + ix);
    keyed.emplace_back(key, static_cast<uint32_t>(o));
  }
  std::stable_sort(keyed.begin(), keyed.end(),
                   [](const std::pair<int64_t, uint32_t>& a, const std::pair<int64_t, uint32_t>& b) { return a.first < b.first; });
  std::vector<int> group_off;
  std::vector<uint32_t> group_obs(keyed.size());
  h->img_cam_groups.assign(nc + 1, 0);
  for (size_t k = 0; k < keyed.size(); ++k) {
    if (k == 0 || keyed[k].first != keyed[k - 1].first) {
      group_off.push_back(static_cast<int>(k));
      ++h->img_cam_groups[(keyed[k].first >> 40) + 1];
    }
    group_obs[k] = pos[keyed[k].second];
  }
  group_off.push_back(static_cast<int>(keyed.size()));
  for (int c = 0; c < nc; ++c) h->img_cam_groups[c + 1] += h->img_cam_groups[c];
  if (dev_alloc(h, &h->d_img_group_off, group_off.size()) || dev_alloc(h, &h->d_img_group_obs, group_obs.size())) return 1;
  CUDA_TRY(h, cudaMemcpy(h->d_img_group_off, group_off.data(), group_off.size() * sizeof(int), cudaMemcpyHostToDevice));
  if (!group_obs.empty())
    CUDA_TRY(h, cudaMemcpy(h->d_img_group_obs, group_obs.data(), group_obs.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  h->have_images = true;
  return 0;
}

// The CUDA state of one call that allocates, computes and frees: its first error, its device buffers, its timing
// events and its cuBLAS / cuSOLVER handles. Everything is released when the scope ends.
struct CallScope {
  std::string* error;  // receives the first error message
  int rc = 0;          // 1 after the first error
  std::vector<void*> buffers;
  cudaEvent_t events[3] = {};
  cublasHandle_t cublas = nullptr;
  cusolverDnHandle_t cusolver = nullptr;

  explicit CallScope(std::string* error_sink) : error(error_sink) {}
  CallScope(const CallScope&) = delete;
  CallScope& operator=(const CallScope&) = delete;
  ~CallScope() {
    for (void* p : buffers) cudaFree(p);
    for (cudaEvent_t e : events)
      if (e) cudaEventDestroy(e);
    if (cublas) cublasDestroy(cublas);
    if (cusolver) cusolverDnDestroy(cusolver);
  }
  // 3 without a device; otherwise selects `device` unless it is negative.
  int use_device(int device) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
      g_create_error = "no CUDA device available (this library has no CPU fallback)";
      return 3;
    }
    if (device >= 0) cudaSetDevice(device);
    return 0;
  }
  void fail(const char* message) {
    if (rc == 0) {
      *error = message;
      rc = 1;
    }
  }
  bool ok(cudaError_t e) {
    if (e != cudaSuccess) fail(cudaGetErrorString(e));
    return e == cudaSuccess;
  }
  template <class T>
  void alloc(T** p, size_t count) {
    if (ok(cudaMalloc(p, sizeof(T) * count))) buffers.push_back(*p);
  }
  // records timing event k on stream s; all events are created on the first call, so none is created inside a window
  void record(int k, cudaStream_t s) {
    for (cudaEvent_t& e : events)
      if (!e) ok(cudaEventCreate(&e));
    cudaEventRecord(events[k], s);
  }
  float elapsed_ms(int from, int to) {
    float ms = 0;
    ok(cudaEventElapsedTime(&ms, events[from], events[to]));
    return ms;
  }
  // cuBLAS / cuSOLVER on the legacy default stream; false after any error
  bool create_solvers() {
    if (rc == 0 && (cublasCreate(&cublas) != CUBLAS_STATUS_SUCCESS || cusolverDnCreate(&cusolver) != CUSOLVER_STATUS_SUCCESS))
      fail("cuBLAS / cuSOLVER initialisation failed");
    return rc == 0;
  }
};

// Device buffers of one Voronoi rendering: the bucket grid over a quarter-pixel box that contains the image
// and every site.
struct VoronoiRun {
  VoronoiGrid g{};
  int64_t nb = 0;
  void alloc(CallScope& cs, int64_t n, int64_t lo_x, int64_t lo_y, int64_t hi_x, int64_t hi_y) {
    g = voronoi_grid_geometry(lo_x, lo_y, hi_x, hi_y);
    nb = static_cast<int64_t>(g.nx) * g.ny;
    cs.alloc(&g.off, nb + 1);
    cs.alloc(&g.count, nb);
    cs.alloc(&g.idx, std::max<int64_t>(1, n));
    cs.alloc(&g.scan_sums, kVoronoiScanMax);
  }
  // sites that took part (those not marked kVoronoiNoSite); after the stream has finished
  cudaError_t n_valid(int64_t* out) {
    int v = 0;
    const cudaError_t e = cudaMemcpy(&v, g.off + nb, sizeof(int), cudaMemcpyDeviceToHost);
    *out = v;
    return e;
  }
};

// The buffers of launch_report_statistics over the one range {0, n}, with the range uploaded.
void alloc_range_statistics(CallScope& cs, int64_t n, int64_t** range, double** partial, unsigned int** select_hist,
                            ReportCam** stats) {
  cs.alloc(range, 2);
  cs.alloc(partial, report_partial_size(1));
  cs.alloc(select_hist, 256);
  cs.alloc(stats, 1);
  const int64_t r[2] = {0, n};
  if (cs.rc == 0) cs.ok(cudaMemcpy(*range, r, sizeof(r), cudaMemcpyHostToDevice));
}

struct LmResult {
  int iterations = 0, attempts = 0;
  double initial_cost = 0, final_cost = 0, lambda = 0;
};
// LMOptimizer::OptimizeImpl (LV/lm_optimizer.h:628-991) as the small dense fits call it: max_lm_attempts = 10,
// init_lambda = -1, init_lambda_factor = 0.001f. `system(k)` returns the cost at iteration k and builds what
// `solve(lambda)` factors; `init_lambda(factor)` derives lambda from the first system; `solve` returns false where the
// reference's update is NaN; `trial_cost()` evaluates the solved step and `accept()` takes it. The loop stops at the
// first error, which the callbacks record in `rc`.
template <class System, class InitLambda, class Solve, class TrialCost, class Accept>
LmResult small_lm(const int& rc, int max_iterations, System system, InitLambda init_lambda, Solve solve,
                  TrialCost trial_cost, Accept accept) {
  LmResult r;
  for (int iteration = 0; rc == 0 && iteration < max_iterations; ++iteration) {
    r.final_cost = system(iteration);
    if (rc) break;
    if (iteration == 0) r.initial_cost = r.final_cost;
    if (r.final_cost == 0) break;
    if (iteration == 0) {
      r.lambda = init_lambda(static_cast<double>(0.001f));  // the call sites pass a float literal
      if (rc) break;
    }
    bool applied = false;
    for (int attempt = 0; rc == 0 && attempt < 10; ++attempt) {
      r.attempts++;
      const bool solved = solve(r.lambda);
      if (rc) break;
      if (!solved) {
        r.lambda = 2.f * r.lambda;
        continue;
      }
      const double test_cost = trial_cost();
      if (rc) break;
      if (test_cost < r.final_cost) {  // CostIsSmallerThan: every residual is valid in both states
        accept();
        r.lambda = 0.5f * r.lambda;
        applied = true;
        r.iterations += 1;
        r.final_cost = test_cost;
        break;
      }
      r.lambda = 2.f * r.lambda;
    }
    if (!applied || r.final_cost == 0) break;
  }
  return r;
}

// H (row-major upper triangle, the reference's variable order) and b of the last build_system.
int download_system(b200ba_handle* h, double* H, double* b) {
  const Layout& L = h->L;
  const int n = L.dof;
  std::vector<double> D(static_cast<size_t>(L.dsz) * L.nblocks), bp(L.nbd), B(static_cast<size_t>(L.nbd) * L.nd),
      C(static_cast<size_t>(L.nd) * L.nd), bd(L.nd);
  CUDA_TRY(h, cudaMemcpy(D.data(), h->sys.Dblk, D.size() * sizeof(double), cudaMemcpyDeviceToHost));
  CUDA_TRY(h, cudaMemcpy(bp.data(), h->sys.bp, bp.size() * sizeof(double), cudaMemcpyDeviceToHost));
  CUDA_TRY(h, cudaMemcpy(B.data(), h->sys.B, B.size() * sizeof(double), cudaMemcpyDeviceToHost));
  CUDA_TRY(h, cudaMemcpy(C.data(), h->sys.C, C.size() * sizeof(double), cudaMemcpyDeviceToHost));
  CUDA_TRY(h, cudaMemcpy(bd.data(), h->sys.bd, bd.size() * sizeof(double), cudaMemcpyDeviceToHost));
  std::fill(H, H + static_cast<size_t>(n) * n, 0.0);
  for (int p = 0; p < L.nblocks; ++p) {
    const double* d = &D[static_cast<size_t>(L.dsz) * p];
    const int o = L.bs * p;
    for (int a2 = 0; a2 < L.bs; ++a2)
      for (int b2 = a2; b2 < L.bs; ++b2)
        H[static_cast<size_t>(o + a2) * n + o + b2] = d[a2 * L.bs - (a2 * (a2 - 1)) / 2 + (b2 - a2)];
  }
  for (int i = 0; i < L.nbd; ++i)
    for (int k = 0; k < L.nd; ++k) H[static_cast<size_t>(i) * n + L.nbd + k] = B[static_cast<size_t>(i) * L.nd + k];
  for (int i = 0; i < L.nd; ++i)
    for (int k = i; k < L.nd; ++k) H[static_cast<size_t>(L.nbd + i) * n + L.nbd + k] = C[static_cast<size_t>(i) * L.nd + k];
  for (int i = 0; i < L.nbd; ++i) b[i] = bp[i];
  for (int i = 0; i < L.nd; ++i) b[L.nbd + i] = bd[i];
  return 0;
}

}  // namespace

// ==============================================================================================
// C ABI
// ==============================================================================================
extern "C" {

const char* b200ba_version(void) { return "b200ba 0.1.0 (sm_90a, FP64)"; }

int64_t b200ba_intrinsics_size(const b200ba_camera* cam) { return cam ? intrinsics_size(*cam) : 0; }
int32_t b200ba_update_parameter_count(const b200ba_camera* cam) { return cam ? update_parameter_count(*cam) : 0; }

void b200ba_default_options(b200ba_options* o) {
  if (!o) return;
  o->max_iteration_count = 1;
  o->init_lambda = -1.0;
  o->numerical_diff_delta = 1e-4;   // APP/calibration.cc:201
  o->regularization_weight = 0.0;
  o->localize_only = 0;
  o->eliminate_points = 1;
  o->schur_mode = B200BA_SCHUR_DENSE;
  o->max_lm_attempts = 50;          // joint_optimization.cc:920
  o->init_lambda_factor = 1e-5;     // joint_optimization.cc:922
  o->huber_parameter = 1.0;         // joint_optimization.cc:346
  o->jacobian_mode = B200BA_JACOBIAN_ANALYTIC;
  o->print_progress = 0;
  o->debug_verify_cost = 0;
  o->debug_fix_points = o->debug_fix_poses = o->debug_fix_rig_poses = o->debug_fix_intrinsics = 0;
}

const char* b200ba_last_error(const b200ba_handle* h) { return h ? h->error.c_str() : g_create_error.c_str(); }

int b200ba_create(const b200ba_problem* p, int device, b200ba_handle** out) {
  if (!p || !out) {
    g_create_error = "NULL argument";
    return 2;
  }
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    g_create_error = "no CUDA device available (this library has no CPU fallback)";
    return 3;
  }
  if (p->n_cameras < 1 || p->n_cameras > kMaxCameras) {
    g_create_error = "n_cameras out of range (1..8)";
    return 2;
  }
  for (int c = 0; c < p->n_cameras; ++c) {
    const int t = p->cameras[c].model_type;
    if (t != B200BA_MODEL_CENTRAL_GENERIC && t != B200BA_MODEL_NONCENTRAL_GENERIC && t != B200BA_MODEL_CENTRAL_OPENCV) {
      g_create_error = "camera model not on the accelerated path (central-generic, noncentral-generic, central-opencv)";
      return 2;
    }
    if (t != B200BA_MODEL_CENTRAL_OPENCV && (p->cameras[c].grid_width < 4 || p->cameras[c].grid_height < 4)) {
      g_create_error = "generic models need a grid of at least 4x4 control points";
      return 2;
    }
  }
  if (p->n_obs >= (1LL << 31)) {
    g_create_error = "n_obs must be < 2^31";
    return 2;
  }
  for (int64_t o = 0; o < p->n_obs; ++o) {
    if (p->obs_imageset[o] >= static_cast<uint32_t>(p->n_imagesets) || p->obs_point[o] >= static_cast<uint32_t>(p->n_points) ||
        p->obs_camera[o] >= static_cast<uint32_t>(p->n_cameras)) {
      g_create_error = "observation index out of range";
      return 2;
    }
  }
  b200ba_handle* h = new b200ba_handle();
  auto fail = [&](int rc) {
    g_create_error = h->error;
    free_handle_buffers(h);
    if (h->cublas) cublasDestroy(h->cublas);
    if (h->cusolver) cusolverDnDestroy(h->cusolver);
    if (h->stream) cudaStreamDestroy(h->stream);
    if (h->side_stream) cudaStreamDestroy(h->side_stream);
    delete h;
    return rc;
  };
  if (device < 0) {
    if (cudaGetDevice(&device) != cudaSuccess) device = 0;
  }
  h->device = device;
#define TRYC(expr) \
  if ((expr) != 0) return fail(1)
  auto cuda_ok = [&](cudaError_t e, const char* what) {
    if (e != cudaSuccess) {
      h->error = std::string(what) + ": " + cudaGetErrorString(e);
      return 1;
    }
    return 0;
  };
  TRYC(cuda_ok(cudaSetDevice(device), "cudaSetDevice"));
  TRYC(cuda_ok(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking), "cudaStreamCreate"));
  TRYC(cuda_ok(cudaStreamCreateWithFlags(&h->side_stream, cudaStreamNonBlocking), "cudaStreamCreate"));
  if (cublasCreate(&h->cublas) != CUBLAS_STATUS_SUCCESS) {
    h->error = "cublasCreate failed";
    return fail(1);
  }
  cublasSetStream(h->cublas, h->stream);
  if (cusolverDnCreate(&h->cusolver) != CUSOLVER_STATUS_SUCCESS) {
    h->error = "cusolverDnCreate failed";
    return fail(1);
  }
  cusolverDnSetStream(h->cusolver, h->stream);

  h->n_cameras = p->n_cameras;
  h->n_imagesets = p->n_imagesets;
  h->n_points = p->n_points;
  h->n_obs = p->n_obs;
  h->cams_host.assign(p->cameras, p->cameras + p->n_cameras);
  h->uniform_model = h->cams_host[0].model_type;
  int upd = 0;
  for (int c = 0; c < p->n_cameras; ++c) {
    CamDev& d = h->pb.cams[c];
    fill_camdev(h->cams_host[c], &d);
    d.intr_off = h->intr_total;
    d.tan_off = h->tan_total;
    d.upd_off = upd;
    upd += d.upd_count;
    h->intr_total += intrinsics_size(h->cams_host[c]);
    const int64_t G = static_cast<int64_t>(d.gw) * d.gh;
    h->tan_total += 6 * G;
    h->n_control_total += G;
    if (d.gw == 0) h->n_param_total += 12;
    if (h->cams_host[c].model_type != h->uniform_model) h->uniform_model = -1;
  }
  const int64_t n = p->n_obs;
  TRYC(dev_alloc(h, &h->d_obs_imageset, n));
  TRYC(dev_alloc(h, &h->d_obs_camera, n));
  TRYC(dev_alloc(h, &h->d_obs_point, n));
  TRYC(dev_alloc(h, &h->d_obs_xy, n));
  if (n > 0) {
    // Static cell-major order: sort the observations ONCE by (camera, B-spline cell of the
    // measured pixel). Lanes of a warp then gather the same 4x4 control points (broadcast loads
    // instead of 32 scattered L1 wavefronts) and accumulate_cells_kernel sees long runs. The
    // C ABI keeps the reference's residual order: inputs are permuted here, per-observation
    // outputs are un-permuted on the way out.
    std::vector<uint32_t> key(n);
    for (int64_t o = 0; o < n; ++o) {
      const uint32_t cam = p->obs_camera[o];
      const CamDev& cd = h->pb.cams[cam];
      uint32_t cell = 0;
      if (cd.gw > 0) {
        const double gx = 1.0 + cd.gmul_x * (static_cast<double>(p->obs_xy[2 * o]) - cd.min_x);
        const double gy = 1.0 + cd.gmul_y * (static_cast<double>(p->obs_xy[2 * o + 1]) - cd.min_y);
        const int x0 = std::min(std::max(static_cast<int>(std::floor(gx)) - 1, 0), cd.gw - 4);
        const int y0 = std::min(std::max(static_cast<int>(std::floor(gy)) - 1, 0), cd.gh - 4);
        cell = static_cast<uint32_t>(x0 + y0 * cd.gw);
      }
      key[o] = (cam << 24) | cell;
    }
    h->perm.resize(n);
    for (int64_t o = 0; o < n; ++o) h->perm[o] = static_cast<uint32_t>(o);
    std::stable_sort(h->perm.begin(), h->perm.end(), [&](uint32_t a, uint32_t b) { return key[a] < key[b]; });
    std::vector<uint32_t> t32(n);
    std::vector<float> txy(2 * n);
    for (int64_t i = 0; i < n; ++i) t32[i] = p->obs_imageset[h->perm[i]];
    TRYC(cuda_ok(cudaMemcpy(h->d_obs_imageset, t32.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice), "H2D"));
    for (int64_t i = 0; i < n; ++i) t32[i] = p->obs_camera[h->perm[i]];
    TRYC(cuda_ok(cudaMemcpy(h->d_obs_camera, t32.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice), "H2D"));
    for (int64_t i = 0; i < n; ++i) t32[i] = p->obs_point[h->perm[i]];
    TRYC(cuda_ok(cudaMemcpy(h->d_obs_point, t32.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice), "H2D"));
    for (int64_t i = 0; i < n; ++i) {
      txy[2 * i] = p->obs_xy[2 * h->perm[i]];
      txy[2 * i + 1] = p->obs_xy[2 * h->perm[i] + 1];
    }
    TRYC(cuda_ok(cudaMemcpy(h->d_obs_xy, txy.data(), n * sizeof(float2), cudaMemcpyHostToDevice), "H2D"));
    TRYC(dev_alloc(h, &h->d_perm, n));
    TRYC(cuda_ok(cudaMemcpy(h->d_perm, h->perm.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice), "H2D"));
  }
  TRYC(dev_alloc(h, &h->d_lp_stage, n));
  if (n > 0) {
    h->h_obs_imageset.assign(p->obs_imageset, p->obs_imageset + n);
    h->h_obs_camera.assign(p->obs_camera, p->obs_camera + n);
    h->h_obs_point.assign(p->obs_point, p->obs_point + n);
    h->h_obs_xy.assign(p->obs_xy, p->obs_xy + 2 * n);
  }
  if (const char* e = getenv("B200BA_DENSE")) h->own_dense = !(strcmp(e, "lib") == 0 || strcmp(e, "0") == 0);
  if (const char* e = getenv("B200BA_DENSE_NB")) h->dense_nb = std::max(128, atoi(e) / 128 * 128);
  set_gemm_sm_reserve(getenv("B200BA_PANEL_SMS") ? atoi(getenv("B200BA_PANEL_SMS")) : 8);
  {
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);
    TRYC(cuda_ok(cudaStreamCreateWithPriority(&h->panel_stream, cudaStreamNonBlocking, hi), "cudaStreamCreate"));
    TRYC(cuda_ok(cudaStreamCreateWithPriority(&h->aux_stream, cudaStreamNonBlocking, hi), "cudaStreamCreate"));
  }
  if (const char* e = getenv("B200BA_GROUPED")) h->force_grouped = atoi(e);
  if (const char* e = getenv("B200BA_COMPACT_J")) h->compact_j = atoi(e) != 0;
  if (const char* e = getenv("B200BA_DIST_CHOL")) h->chol_mode = atoi(e);
  if (const char* e = getenv("B200BA_CHOL_NB")) h->chol_nb = std::max(32, atoi(e));
  h->pb.n_obs = n;
  h->pb.obs_imageset = h->d_obs_imageset;
  h->pb.obs_camera = h->d_obs_camera;
  h->pb.obs_point = h->d_obs_point;
  h->pb.obs_xy = h->d_obs_xy;
  for (int i = 0; i < 2; ++i) {
    TRYC(dev_alloc(h, &h->st[i].points, 3 * static_cast<size_t>(h->n_points)));
    TRYC(dev_alloc(h, &h->st[i].rig_tr_global, 7 * static_cast<size_t>(h->n_imagesets)));
    TRYC(dev_alloc(h, &h->st[i].camera_tr_rig, 7 * static_cast<size_t>(h->n_cameras)));
    TRYC(dev_alloc(h, &h->st[i].intrinsics, h->intr_total));
    TRYC(dev_alloc(h, &h->st[i].image_tr_global, 12 * static_cast<size_t>(h->n_imagesets) * h->n_cameras));
    TRYC(dev_alloc(h, &h->st[i].tangents, h->tan_total));
  }
  TRYC(dev_alloc(h, &h->d_last_projection, n));
  TRYC(cuda_ok(cudaMemset(h->d_last_projection, 0, std::max<int64_t>(1, n) * sizeof(double2)), "memset"));
  TRYC(dev_alloc(h, &h->d_straggler_list, n));
  TRYC(dev_alloc(h, &h->d_straggler_count, 1));
  TRYC(dev_alloc(h, &h->d_info, 2 + kMaxCholPanels));
  TRYC(dev_alloc(h, &h->d_fail, 1));
  TRYC(dev_alloc(h, &h->d_partial, cost_reduce_partial_size()));
  TRYC(dev_alloc(h, &h->d_scal, 16));
  TRYC(cuda_ok(cudaMallocHost(reinterpret_cast<void**>(&h->h_scal), 16 * sizeof(double)), "cudaMallocHost"));
  TRYC(cuda_ok(cudaMallocHost(reinterpret_cast<void**>(&h->h_flags), 4 * sizeof(int)), "cudaMallocHost"));
#undef TRYC
  *out = h;
  return 0;
}

void b200ba_destroy(b200ba_handle* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  if (h->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(h->comm);
  resolve_timings(h);
  for (auto e : h->event_pool) cudaEventDestroy(e);
  for (int i = 0; i < 2; ++i) {
    if (h->ev_syrk[i]) cudaEventDestroy(h->ev_syrk[i]);
    if (h->ev_scatter[i]) cudaEventDestroy(h->ev_scatter[i]);
  }
  if (h->ev_s_ready) cudaEventDestroy(h->ev_s_ready);
  free_handle_buffers(h);
  if (h->cublas) cublasDestroy(h->cublas);
  if (h->cusolver) cusolverDnDestroy(h->cusolver);
  if (h->stream) cudaStreamDestroy(h->stream);
  if (h->side_stream) cudaStreamDestroy(h->side_stream);
  if (h->panel_stream) cudaStreamDestroy(h->panel_stream);
  if (h->aux_stream) cudaStreamDestroy(h->aux_stream);
  dense_release(&h->dn, /*own_streams=*/false);
  delete h;
}

int b200ba_set_state(b200ba_handle* h, const b200ba_state* s) {
  if (!h) return 1;
  if (!s || !s->points || !s->rig_tr_global || !s->camera_tr_rig || !s->intrinsics) {
    h->error = "NULL state array";
    return 2;
  }
  CUDA_TRY(h, cudaSetDevice(h->device));
  StateDev& d = h->st[h->cur];
  CUDA_TRY(h, cudaMemcpyAsync(d.points, s->points, 3 * sizeof(double) * h->n_points, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(d.rig_tr_global, s->rig_tr_global, 7 * sizeof(double) * h->n_imagesets, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(d.camera_tr_rig, s->camera_tr_rig, 7 * sizeof(double) * h->n_cameras, cudaMemcpyHostToDevice, h->stream));
  for (int c = 0; c < h->n_cameras; ++c)
    CUDA_TRY(h, cudaMemcpyAsync(d.intrinsics + h->pb.cams[c].intr_off, s->intrinsics[c],
                                sizeof(double) * intrinsics_size(h->cams_host[c]), cudaMemcpyHostToDevice, h->stream));
  if (s->last_projection) {
    // caller's order -> device staging -> cell-major order (gather on the device)
    CUDA_TRY(h, cudaMemcpyAsync(h->d_lp_stage, s->last_projection, 2 * sizeof(double) * h->n_obs, cudaMemcpyHostToDevice, h->stream));
    launch_permute_double2(h->n_obs, h->d_perm, h->d_lp_stage, h->d_last_projection, /*scatter=*/false, h->stream);
  } else
    CUDA_TRY(h, cudaMemsetAsync(h->d_last_projection, 0, std::max<int64_t>(1, h->n_obs) * sizeof(double2), h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->have_state = true;
  return 0;
}

int b200ba_get_state(b200ba_handle* h, b200ba_state* s) {
  if (!h) return 1;
  if (!s || !h->have_state) {
    h->error = "no state";
    return 2;
  }
  CUDA_TRY(h, cudaSetDevice(h->device));
  const StateDev& d = h->st[h->cur];
  if (s->points) CUDA_TRY(h, cudaMemcpyAsync(s->points, d.points, 3 * sizeof(double) * h->n_points, cudaMemcpyDeviceToHost, h->stream));
  if (s->rig_tr_global) CUDA_TRY(h, cudaMemcpyAsync(s->rig_tr_global, d.rig_tr_global, 7 * sizeof(double) * h->n_imagesets, cudaMemcpyDeviceToHost, h->stream));
  if (s->camera_tr_rig) CUDA_TRY(h, cudaMemcpyAsync(s->camera_tr_rig, d.camera_tr_rig, 7 * sizeof(double) * h->n_cameras, cudaMemcpyDeviceToHost, h->stream));
  if (s->intrinsics)
    for (int c = 0; c < h->n_cameras; ++c)
      CUDA_TRY(h, cudaMemcpyAsync(s->intrinsics[c], d.intrinsics + h->pb.cams[c].intr_off,
                                  sizeof(double) * intrinsics_size(h->cams_host[c]), cudaMemcpyDeviceToHost, h->stream));
  if (s->last_projection) {
    launch_permute_double2(h->n_obs, h->d_perm, h->d_last_projection, h->d_lp_stage, /*scatter=*/true, h->stream);
    CUDA_TRY(h, cudaMemcpyAsync(s->last_projection, h->d_lp_stage, 2 * sizeof(double) * h->n_obs, cudaMemcpyDeviceToHost, h->stream));
  }
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  return 0;
}

// Device-side copy of the optimised state and the warm-start cache (no host round trip). Used to
// restart a trajectory from the same point (bench.py) and by callers that want to roll back.
static int copy_state_dev(b200ba_handle* h, const StateDev& src, const double2* src_lp, StateDev& dst, double2* dst_lp) {
  CUDA_TRY(h, cudaMemcpyAsync(dst.points, src.points, 3 * sizeof(double) * h->n_points, cudaMemcpyDeviceToDevice, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(dst.rig_tr_global, src.rig_tr_global, 7 * sizeof(double) * h->n_imagesets, cudaMemcpyDeviceToDevice, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(dst.camera_tr_rig, src.camera_tr_rig, 7 * sizeof(double) * h->n_cameras, cudaMemcpyDeviceToDevice, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(dst.intrinsics, src.intrinsics, sizeof(double) * h->intr_total, cudaMemcpyDeviceToDevice, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(dst_lp, src_lp, sizeof(double2) * std::max<int64_t>(1, h->n_obs), cudaMemcpyDeviceToDevice, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  return 0;
}

int b200ba_snapshot_state(b200ba_handle* h) {
  if (!h) return 1;
  if (!h->have_state) {
    h->error = "no state";
    return 2;
  }
  CUDA_TRY(h, cudaSetDevice(h->device));
  if (!h->snap.points) {
    if (dev_alloc(h, &h->snap.points, 3 * static_cast<size_t>(h->n_points))) return 1;
    if (dev_alloc(h, &h->snap.rig_tr_global, 7 * static_cast<size_t>(h->n_imagesets))) return 1;
    if (dev_alloc(h, &h->snap.camera_tr_rig, 7 * static_cast<size_t>(h->n_cameras))) return 1;
    if (dev_alloc(h, &h->snap.intrinsics, h->intr_total)) return 1;
    if (dev_alloc(h, &h->d_snap_lp, h->n_obs)) return 1;
  }
  if (copy_state_dev(h, h->st[h->cur], h->d_last_projection, h->snap, h->d_snap_lp)) return 1;
  h->have_snapshot = true;
  return 0;
}

int b200ba_restore_state(b200ba_handle* h) {
  if (!h) return 1;
  if (!h->have_snapshot) {
    h->error = "no snapshot: call b200ba_snapshot_state first";
    return 2;
  }
  CUDA_TRY(h, cudaSetDevice(h->device));
  return copy_state_dev(h, h->snap, h->d_snap_lp, h->st[h->cur], h->d_last_projection);
}

int b200ba_calibration_report(b200ba_handle* h, b200ba_camera_report* reports, double* errors, double* report_ms) {
  if (!h) return 1;
  if (!reports) {
    h->error = "reports is NULL";
    return 2;
  }
  if (h->comm || h->n_ranks > 1) {
    h->error = "b200ba_calibration_report: the handle is joined to a communicator and holds one shard of the "
               "observations; the report needs all of them (use a single-rank handle)";
    return 2;
  }
  if (!h->have_state) {
    h->error = "no state: call b200ba_set_state first";
    return 2;
  }
  CUDA_TRY(h, cudaSetDevice(h->device));
  if (setup_report(h)) return 1;
  const int nc = h->n_cameras;
  // prepare_state only refreshes the derived image_tr_global / tangents caches of the current state
  Layout L{};
  L.n_points = h->n_points;
  L.n_imagesets = h->n_imagesets;
  L.n_cameras = nc;
  cudaEvent_t a = get_event(h), b = get_event(h);
  cudaEventRecord(a, h->stream);
  launch_prepare_state(h->pb, L, h->st[h->cur], h->n_control_total, h->stream);
  launch_calibration_report(h->pb, nc, h->st[h->cur], h->rep, h->stream);
  cudaEventRecord(b, h->stream);
  CUDA_TRY(h, cudaGetLastError());
  constexpr int kBins = B200BA_REPORT_HIST * B200BA_REPORT_HIST;
  std::vector<ReportCam> rc(nc);
  std::vector<int32_t> hist(static_cast<size_t>(nc) * kBins);
  CUDA_TRY(h, cudaMemcpyAsync(rc.data(), h->rep.cams, nc * sizeof(ReportCam), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(hist.data(), h->rep.hist, hist.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
  if (errors && h->n_obs > 0) {
    launch_permute_double2(h->n_obs, h->d_perm, h->rep.err, h->d_rep_stage, /*scatter=*/true, h->stream);
    CUDA_TRY(h, cudaMemcpyAsync(errors, h->d_rep_stage, 2 * sizeof(double) * h->n_obs, cudaMemcpyDeviceToHost, h->stream));
  }
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  float ms = 0;
  CUDA_TRY(h, cudaEventElapsedTime(&ms, a, b));
  h->event_pool.push_back(a);
  h->event_pool.push_back(b);
  if (report_ms) *report_ms = ms;
  for (int c = 0; c < nc; ++c) {
    b200ba_camera_report& r = reports[c];
    r.reprojection_error_count = rc[c].count;
    r.reprojection_error_sum = rc[c].sum;
    r.reprojection_error_max = rc[c].max;
    r.reprojection_error_median = rc[c].median;
    r.biasedness = rc[c].biasedness;
    r.biasedness_cells = rc[c].biasedness_cells;
    r.horizontal_fov = rc[c].hfov;
    r.vertical_fov = rc[c].vfov;
    memcpy(r.histogram, hist.data() + static_cast<size_t>(c) * kBins, kBins * sizeof(int32_t));
  }
  return 0;
}

// The images of CreateCalibrationReportForCamera (calibration_report.cc:713-838) for one camera, from the report's
// error pass: the observation directions (:723-726) and the two Voronoi error maps (:758-787).
int b200ba_report_images(b200ba_handle* h, int32_t camera, uint8_t* observation_directions, uint8_t* error_directions,
                         uint8_t* error_magnitudes, int64_t* n_sites, double* device_ms) {
  if (!h) return 1;
  if (h->comm || h->n_ranks > 1) {
    h->error = "b200ba_report_images: the handle is joined to a communicator and holds one shard of the "
               "observations; the report needs all of them (use a single-rank handle)";
    return 2;
  }
  if (camera < 0 || camera >= h->n_cameras) {
    h->error = "b200ba_report_images: camera index out of range";
    return 2;
  }
  if (!h->have_state) {
    h->error = "no state: call b200ba_set_state first";
    return 2;
  }
  const b200ba_camera& cam = h->cams_host[camera];
  if (observation_directions && cam.model_type != B200BA_MODEL_CENTRAL_GENERIC &&
      cam.model_type != B200BA_MODEL_NONCENTRAL_GENERIC) {
    h->error = "b200ba_report_images: observation directions need a device un-projection, which exists for the "
               "central- and non-central-generic models only (pass NULL for this camera)";
    return 2;
  }
  CUDA_TRY(h, cudaSetDevice(h->device));
  if (setup_report(h) || setup_images(h)) return 1;
  const int nc = h->n_cameras;
  const int64_t g0 = h->img_cam_groups[camera], n_groups = h->img_cam_groups[camera + 1] - g0;
  const int64_t pixels = static_cast<int64_t>(cam.width) * cam.height;
  int2* d_sites = nullptr;
  float* d_colors = nullptr;
  uint8_t* d_img[3] = {nullptr, nullptr, nullptr};
  uint8_t* const out[3] = {observation_directions, error_directions, error_magnitudes};
  VoronoiRun vr;
  CallScope cs(&h->error);
  cs.alloc(&d_sites, std::max<int64_t>(1, n_groups));
  cs.alloc(&d_colors, 6 * std::max<int64_t>(1, n_groups));
  for (int k = 0; k < 3; ++k)
    if (out[k]) cs.alloc(&d_img[k], 3 * pixels);
  // the sites are ((int)(4 x), (int)(4 y)) with -1 < x < 4 W, -1 < y < 4 H
  if (cs.rc == 0) vr.alloc(cs, n_groups, -4, -4, 16 * static_cast<int64_t>(cam.width), 16 * static_cast<int64_t>(cam.height));
  if (cs.rc == 0) {
    Layout L{};
    L.n_points = h->n_points;
    L.n_imagesets = h->n_imagesets;
    L.n_cameras = nc;
    const CamDev& cd = h->pb.cams[camera];
    cs.record(0, h->stream);
    launch_prepare_state(h->pb, L, h->st[h->cur], h->n_control_total, h->stream);
    launch_report_errors(h->pb, nc, h->st[h->cur], h->rep, h->stream);
    launch_report_sites(h->pb, h->rep, n_groups, h->d_img_group_off + g0, h->d_img_group_obs, d_sites, d_colors, h->stream);
    launch_render_voronoi(cam.width, cam.height, n_groups, d_sites, d_colors, 6, vr.g, d_img[1], d_img[2], h->stream);
    if (d_img[0]) launch_observation_directions(cd, h->st[h->cur].intrinsics + cd.intr_off, d_img[0], h->stream);
    cs.record(1, h->stream);
    cs.ok(cudaGetLastError());
    cs.ok(cudaStreamSynchronize(h->stream));
  }
  if (cs.rc == 0) {
    for (int k = 0; k < 3; ++k)
      if (out[k]) cs.ok(cudaMemcpy(out[k], d_img[k], 3 * pixels, cudaMemcpyDeviceToHost));
    int64_t nv = 0;
    cs.ok(vr.n_valid(&nv));
    if (n_sites) *n_sites = nv;
    if (device_ms) *device_ms = cs.elapsed_ms(0, 1);
  }
  return cs.rc;
}

int32_t b200ba_degrees_of_freedom(const b200ba_handle* h, const b200ba_options* opt) {
  if (!h || !opt) return -1;
  int n_intr = 0;
  for (int c = 0; c < h->n_cameras; ++c) n_intr += update_parameter_count(h->cams_host[c]);
  return 3 * h->n_points + 6 * h->n_imagesets + (h->n_cameras > 1 ? 6 * h->n_cameras : 0) + (opt->localize_only ? 0 : n_intr);
}

// OptimizeJointly (joint_optimization.cc:757-953): a loop of single LM iterations, each being
// LMOptimizer::OptimizeImpl with max_iteration_count = 1 (LV/lm_optimizer.h:628-991).
int b200ba_optimize(b200ba_handle* h, const b200ba_options* opt, b200ba_report* report) {
  if (!h) return 1;
  if (!report) {
    h->error = "report is NULL";
    return 2;
  }
  if (int rc = check_ready(h, opt)) return rc;
  memset(report, 0, sizeof(*report));
  memset(&h->timings, 0, sizeof(h->timings));
  h->lm_events.clear();
  cudaEvent_t ev_total_a = get_event(h), ev_total_b = get_event(h);
  cudaEventRecord(ev_total_a, h->stream);
  const Layout& L = h->L;
  const double huber = opt->huber_parameter;
  double lambda = 0, init_lambda = opt->init_lambda;
  // on-the-fly block processing (pose elimination with an *OnTheFly Schur mode) starts from a fixed
  // lambda when none is handed in (joint_optimization.cc:801-804)
  if (!opt->eliminate_points && init_lambda < 0 &&
      (opt->schur_mode == B200BA_SCHUR_DENSE_ONTHEFLY || opt->schur_mode == B200BA_SCHUR_SPARSE_ONTHEFLY))
    init_lambda = 0.0001f;
  report->final_lambda = init_lambda;  // what optimizer.lambda() holds if no iteration changes it
  double final_cost = -1;
  // n_valid / sum |r|^2 of the CURRENT state, taken from the passes the LM loop makes anyway (the
  // base pass of a build, or the trial pass of an accepted step) -- no extra pass for statistics
  double stat_valid = 0, stat_sumsq = 0;
  bool have_stats = false;
  if (opt->debug_verify_cost) {
    // LMOptimizer::VerifyCost twice (joint_optimization.cc:866-876, lm_optimizer.h:474-490)
    double c[2] = {0, 0};
    for (int rep2 = 0; rep2 < 2; ++rep2) {
      double with_jac = 0;
      for (int jac = 0; jac < 2; ++jac) {
        if (evaluate_state(h, h->cur, jac != 0, jac ? h->out : h->out_trial, huber, PH_TRIAL)) return 1;
        const ObsOut& oo = jac ? h->out : h->out_trial;
        launch_cost_reduce(h->n_obs, oo.cost, nullptr, oo.residual, h->d_partial, h->d_scal, h->stream);
        if (all_reduce(h, h->d_scal, 6)) return 1;
        CUDA_TRY(h, cudaMemcpyAsync(h->h_scal, h->d_scal, 6 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
        if (sync_stream(h)) return 1;
        (jac ? with_jac : c[rep2]) = h->h_scal[3];
      }
      if (std::fabs(c[rep2] - with_jac) > 1e-3f)
        fprintf(stderr, "[b200ba] Cost differs when computed with or without Jacobians: %.12g vs %.12g\n", c[rep2], with_jac);
    }
    if (!(std::fabs(c[0] - c[1]) <= 1e-3f)) {
      h->error = "debug_verify_cost: two cost evaluations of the same state differ by more than 1e-3";
      return 5;
    }
  }
  const bool any_fixed = opt->debug_fix_points || opt->debug_fix_poses || opt->debug_fix_rig_poses || opt->debug_fix_intrinsics;
  for (int iteration = 0; iteration < opt->max_iteration_count; ++iteration) {
    double cost = 0, n_valid = 0;
    if (build_system(h, huber, &cost, &n_valid, any_fixed ? opt : nullptr)) return 1;
    h->timings.build_count += 1;
    stat_valid = h->h_scal[4];
    stat_sumsq = h->h_scal[5];
    have_stats = true;
    double last_cost = cost;
    if (iteration == 0) report->initial_cost = cost;
    if (cost == 0) {  // "Cost is zero, stopping." (lm_optimizer.h:755-760)
      final_cost = cost;
      break;
    }
    if (init_lambda >= 0) {
      lambda = init_lambda;
    } else {
      // lambda = init_lambda_factor * trace(H) / dof (lm_optimizer.h:766-781)
      lambda = opt->init_lambda_factor * h->trace_H / L.dof;
    }
    bool applied_update = false;
    int attempts = 0;
    for (int lm_iteration = 0; lm_iteration < opt->max_lm_attempts; ++lm_iteration) {
      ++attempts;
      h->timings.lm_attempts += 1;
      int spd = 1;
      if (solve_system(h, lambda, &spd)) return 1;
      if (!spd) {
        // A non-positive pivot: the analogue of the reference's NaN-update rejection
        // (lm_optimizer.h:905-913) -- increase the damping and retry.
        h->lm_events.push_back(B200BA_LM_REFUSED_PIVOT);
        lambda = 2.f * lambda;
        if (opt->print_progress) fprintf(stderr, "[b200ba]   [%d, %d] factorisation failed, new lambda %g\n", iteration + 1, lm_iteration + 1, lambda);
        continue;
      }
      const int trial = 1 - h->cur;
      {
        ScopedPhase ph(h, PH_UPDATE);
        launch_update_state(h->pb, L, h->st[h->cur], h->st[trial], h->d_x, h->n_control_total, h->n_param_total, h->stream);
        h->timings.kernel_launches += 1;
      }
      if (evaluate_state(h, trial, false, h->out_trial, huber, PH_TRIAL)) return 1;
      {
        ScopedPhase ph(h, PH_TRIAL);
        launch_cost_reduce(h->n_obs, h->out_trial.cost, h->out.cost, h->out_trial.residual, h->d_partial, h->d_scal, h->stream);
        h->timings.kernel_launches += 2;
      }
      if (all_reduce(h, h->d_scal, 6)) return 1;
      CUDA_TRY(h, cudaMemcpyAsync(h->h_scal, h->d_scal, 6 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
      if (sync_stream(h)) return 1;
      const double left = h->h_scal[0], right = h->h_scal[1], count = h->h_scal[2];
      const double trial_cost = h->h_scal[3];
      // CostIsSmallerThan (lm_optimizer.h:993-1011)
      if (count > 0 && left < right) {
        h->lm_events.push_back(B200BA_LM_ACCEPTED);
        h->cur = trial;
        stat_valid = h->h_scal[4];
        stat_sumsq = h->h_scal[5];
        lambda = 0.5f * lambda;
        applied_update = true;
        report->num_iterations_performed += 1;
        last_cost = trial_cost;
        if (opt->print_progress) fprintf(stderr, "[b200ba] [%d] update accepted, cost %.12g\n", iteration + 1, trial_cost);
        break;
      } else {
        h->lm_events.push_back(B200BA_LM_REJECTED_COST);
        lambda = 2.f * lambda;
        if (opt->print_progress) fprintf(stderr, "[b200ba]   [%d, %d of %d] update rejected (bad cost: %.12g), new lambda: %g\n", iteration + 1, lm_iteration + 1, opt->max_lm_attempts, trial_cost, lambda);
      }
    }
    final_cost = last_cost;
    init_lambda = lambda;
    report->final_lambda = lambda;
    if (report->trace_len < B200BA_MAX_TRACE) {
      report->trace_cost[report->trace_len] = last_cost;
      report->trace_lambda[report->trace_len] = lambda;
      report->trace_attempts[report->trace_len] = attempts;
      report->trace_len++;
    }
    if (!applied_update) break;
    report->performed_an_iteration = 1;
    if (last_cost == 0) break;
  }
  report->final_cost = final_cost;
  if (!have_stats) {
    // max_iteration_count == 0: statistics of the unchanged state need one residual-only pass
    if (evaluate_state(h, h->cur, false, h->out_trial, huber, PH_TRIAL)) return 1;
    launch_cost_reduce(h->n_obs, h->out_trial.cost, nullptr, h->out_trial.residual, h->d_partial, h->d_scal, h->stream);
    h->timings.kernel_launches += 2;
    if (all_reduce(h, h->d_scal, 6)) return 1;
    CUDA_TRY(h, cudaMemcpyAsync(h->h_scal, h->d_scal, 6 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    if (sync_stream(h)) return 1;
    stat_valid = h->h_scal[4];
    stat_sumsq = h->h_scal[5];
  }
  cudaEventRecord(ev_total_b, h->stream);
  if (sync_stream(h)) return 1;
  {
    float ms = 0;
    cudaEventElapsedTime(&ms, ev_total_a, ev_total_b);
    h->timings.total_ms = ms;
    h->event_pool.push_back(ev_total_a);
    h->event_pool.push_back(ev_total_b);
  }
  report->n_valid = static_cast<int64_t>(stat_valid);
  // with several ranks n_valid is global (all-reduced) while n_obs is this rank's shard
  report->n_invalid = (h->n_ranks > 1) ? -1 : (h->n_obs - report->n_valid);
  report->rmse = report->n_valid > 0 ? std::sqrt(stat_sumsq / stat_valid) : 0.0;
  report->cost_and_jacobian_evaluation_time = 1e-3 * (h->timings.jacobian_kernel_ms + h->timings.accumulate_ms + h->timings.trial_cost_ms);
  report->solve_time = 1e-3 * (h->timings.schur_ms + h->timings.factor_ms);
  return 0;
}

// RunBundleAdjustment (APP/calibration.cc:187-304) with the state resident on the device: single LM
// iterations with the lambda carried over, the re-orientation of every camera after each iteration
// (ChooseNiceCameraOrientation + camera_tr_rig update, calibration.cc:245-252) and the stopping
// criterion `cost >= last_cost - cost_reduction_threshold` (:298-300). Nothing but the scalars the
// stop rule needs crosses the PCIe bus between iterations.
int b200ba_run_bundle_adjustment(b200ba_handle* h, const b200ba_options* opt_in, int32_t max_iteration_count,
                                 double cost_reduction_threshold, b200ba_ba_report* out,
                                 int (*on_iteration)(void* user, int32_t iteration, double cost), void* user) {
  if (!h) return 1;
  if (!opt_in || !out) {
    h->error = "NULL argument";
    return 2;
  }
  memset(out, 0, sizeof(*out));
  b200ba_options opt = *opt_in;
  opt.max_iteration_count = 1;
  double lambda = opt_in->init_lambda;  // the reference starts from -1 (calibration.cc:203)
  double last_cost = INFINITY;
  b200ba_timings acc{};
  for (int iteration = 0; iteration < max_iteration_count; ++iteration) {
    opt.init_lambda = lambda;
    b200ba_report rep;
    if (int rc = b200ba_optimize(h, &opt, &rep)) return rc;
    lambda = rep.final_lambda;
    const double cost = rep.final_cost;
    if (iteration == 0) out->initial_cost = rep.initial_cost;
    out->final_cost = cost;
    out->final_lambda = lambda;
    out->rmse = rep.rmse;
    out->n_valid = rep.n_valid;
    out->n_invalid = rep.n_invalid;
    out->lm_attempts += rep.trace_len ? rep.trace_attempts[0] : 0;
    if (out->iterations < B200BA_MAX_TRACE) out->costs[out->iterations] = cost;
    out->iterations += 1;
    acc.total_ms += h->timings.total_ms;
    if (!opt.localize_only) {
      // beautify all camera orientations (calibration.cc:245-252)
      if (!h->d_rot && dev_alloc(h, &h->d_rot, 9 * static_cast<size_t>(h->n_cameras))) return 1;
      launch_nice_orientation(h->pb, h->st[h->cur], h->n_cameras, h->d_rot, h->stream);
      CUDA_TRY(h, cudaGetLastError());
    }
    if (on_iteration) {
      CUDA_TRY(h, cudaStreamSynchronize(h->stream));
      if (on_iteration(user, iteration, cost) != 0) break;  // the 'q' key of the reference (calibration.cc:293-295)
    }
    if (cost >= last_cost - cost_reduction_threshold) break;  // stopping criterion
    last_cost = cost;
  }
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  out->device_ms = acc.total_ms;
  return 0;
}

int b200ba_optimize_host(b200ba_handle* h, b200ba_state* state, const b200ba_options* opt, b200ba_report* report) {
  if (int rc = b200ba_set_state(h, state)) return rc;
  if (int rc = b200ba_optimize(h, opt, report)) return rc;
  return b200ba_get_state(h, state);
}

int b200ba_evaluate(b200ba_handle* h, const b200ba_options* opt, int compute_jacobians, double* residuals,
                    double* costs, double* total_cost) {
  if (int rc = check_ready(h, opt)) return rc;
  const int64_t n = h->n_obs;
  if (evaluate_state(h, h->cur, compute_jacobians != 0, h->out, opt->huber_parameter, PH_JAC)) return 1;
  launch_cost_reduce(n, h->out.cost, nullptr, h->out.residual, h->d_partial, h->d_scal, h->stream);
  CUDA_TRY(h, cudaMemcpyAsync(h->h_scal, h->d_scal, 6 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if (sync_stream(h)) return 1;
  if (residuals) {
    std::vector<double> tmp(2 * n);
    CUDA_TRY(h, cudaMemcpy(tmp.data(), h->out.residual, 2 * n * sizeof(double), cudaMemcpyDeviceToHost));
    for (int64_t i = 0; i < n; ++i) {
      residuals[2 * static_cast<int64_t>(h->perm[i])] = tmp[i];
      residuals[2 * static_cast<int64_t>(h->perm[i]) + 1] = tmp[n + i];
    }
  }
  if (costs) {
    std::vector<double> tmp(n);
    CUDA_TRY(h, cudaMemcpy(tmp.data(), h->out.cost, n * sizeof(double), cudaMemcpyDeviceToHost));
    for (int64_t i = 0; i < n; ++i) costs[h->perm[i]] = tmp[i];
  }
  if (total_cost) *total_cost = h->h_scal[3];
  return 0;
}

int b200ba_get_jacobians(b200ba_handle* h, double* j_point, double* j_pose, double* j_rig, double* j_intr,
                         int32_t* intr_index, int32_t K) {
  if (!h || !h->have_layout) return 1;
  CUDA_TRY(h, cudaSetDevice(h->device));
  const Layout& L = h->L;
  const int64_t n = h->n_obs;
  std::vector<double> jac(2 * static_cast<size_t>(L.n_jcols) * n);
  std::vector<int32_t> cell(n);
  std::vector<uint8_t> has(n);
  if (h->out.compact) {
    // rebuild the expanded buffer from the compact records (state of the evaluation = current state)
    double* tmp = nullptr;
    CUDA_TRY(h, cudaMalloc(reinterpret_cast<void**>(&tmp), std::max<size_t>(1, jac.size()) * sizeof(double)));
    launch_expand_jacobian(h->pb, L, h->st[h->cur], h->out, tmp, h->stream);
    cudaError_t e = cudaStreamSynchronize(h->stream);
    if (e == cudaSuccess) e = cudaMemcpy(jac.data(), tmp, jac.size() * sizeof(double), cudaMemcpyDeviceToHost);
    cudaFree(tmp);
    CUDA_TRY(h, e);
  } else
    CUDA_TRY(h, cudaMemcpy(jac.data(), h->out.jac, jac.size() * sizeof(double), cudaMemcpyDeviceToHost));
  CUDA_TRY(h, cudaMemcpy(cell.data(), h->out.cell, n * sizeof(int32_t), cudaMemcpyDeviceToHost));
  CUDA_TRY(h, cudaMemcpy(has.data(), h->out.has_jac, n, cudaMemcpyDeviceToHost));
  std::vector<uint32_t> cams(n);
  CUDA_TRY(h, cudaMemcpy(cams.data(), h->d_obs_camera, n * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  auto J = [&](int col, int r, int64_t i) { return jac[(2 * static_cast<size_t>(col) + r) * n + i]; };
  for (int64_t i = 0; i < n; ++i) {
    const int64_t o = h->perm[i];  // position i on the device holds the caller's observation o
    const bool v = has[i] == 1 || has[i] == 3;  // valid, or a late success of the straggler pass
    for (int r = 0; r < 2; ++r) {
      if (j_point) for (int j = 0; j < 3; ++j) j_point[(o * 2 + r) * 3 + j] = v ? J(L.jc_point + j, r, i) : 0.0;
      if (j_pose) for (int j = 0; j < 6; ++j) j_pose[(o * 2 + r) * 6 + j] = v ? J(L.jc_pose + j, r, i) : 0.0;
      if (j_rig) for (int j = 0; j < 6; ++j) j_rig[(o * 2 + r) * 6 + j] = (v && L.rig_in_state) ? J(L.jc_rig + j, r, i) : 0.0;
    }
    const CamDev& c = h->pb.cams[cams[i]];
    for (int k = 0; k < K; ++k) {
      const bool vk = v && !L.localize_only && k < c.K;
      if (j_intr) {
        j_intr[(o * 2 + 0) * K + k] = vk ? J(L.jc_intr + k, 0, i) : 0.0;
        j_intr[(o * 2 + 1) * K + k] = vk ? J(L.jc_intr + k, 1, i) : 0.0;
      }
      if (intr_index) {
        int idx = -1;
        if (vk) {
          int local;
          if (c.model_type == B200BA_MODEL_CENTRAL_GENERIC) {
            const int cp = k >> 1;
            local = 2 * (cell[i] + (cp & 3) + (cp >> 2) * c.gw) + (k & 1);
          } else if (c.model_type == B200BA_MODEL_NONCENTRAL_GENERIC) {
            const int cp = k / 5;
            local = 5 * (cell[i] + (cp & 3) + (cp >> 2) * c.gw) + (k - 5 * cp);
          } else {
            local = k;
          }
          idx = L.g_intr + c.upd_off + local;
        }
        intr_index[o * K + k] = idx;
      }
    }
  }
  return 0;
}

int b200ba_build_system(b200ba_handle* h, const b200ba_options* opt, int32_t n, double* H, double* b, double* cost) {
  if (int rc = check_ready(h, opt)) return rc;
  const Layout& L = h->L;
  if (n != L.dof) {
    h->error = "n does not equal the number of unknowns";
    return 2;
  }
  double c = 0, nv = 0;
  if (build_system(h, opt->huber_parameter, &c, &nv)) return 1;
  if (cost) *cost = c;
  return download_system(h, H, b);
}

// Diagnostics / tests: one LM attempt's linear solve at the current state (see the header).
int b200ba_debug_solve_step(b200ba_handle* h, const b200ba_options* opt, double lambda, int32_t n, double* H, double* b,
                            double* S, double* rhs, double* x, double* lambda_used, int32_t info[8]) {
  if (int rc = check_ready(h, opt)) return rc;
  const Layout& L = h->L;
  if (h->n_ranks > 1) {
    h->error = "b200ba_debug_solve_step: the handle is joined to a communicator";
    return 2;
  }
  if (n != L.dof || !S || !rhs || !x || !info) {
    h->error = "b200ba_debug_solve_step: n does not equal the number of unknowns, or a required output is NULL";
    return 2;
  }
  const bool any_fixed = opt->debug_fix_points || opt->debug_fix_poses || opt->debug_fix_rig_poses || opt->debug_fix_intrinsics;
  double cost = 0, n_valid = 0;
  if (build_system(h, opt->huber_parameter, &cost, &n_valid, any_fixed ? opt : nullptr)) return 1;
  if (H && b && download_system(h, H, b)) return 1;
  if (lambda < 0) lambda = opt->init_lambda_factor * h->trace_H / L.dof;
  int spd = 1;
  h->capture_S = S;
  h->capture_rhs = rhs;
  const int rc = solve_system(h, lambda, &spd);
  h->capture_S = h->capture_rhs = nullptr;
  if (rc) return rc;
  CUDA_TRY(h, cudaMemcpy(x, h->d_x, static_cast<size_t>(L.dof) * sizeof(double), cudaMemcpyDeviceToHost));
  if (lambda_used) *lambda_used = lambda;
  info[0] = spd;
  info[1] = h->use_grouped ? 1 : 0;
  info[2] = h->n_groups;
  dense_variants(&info[3], &info[4], &info[5], &info[6]);
  info[7] = h->own_dense ? h->dn.NB : 0;
  return 0;
}

// Diagnostics / tests: the retraction of one LM attempt (update_state_kernel) from the current state
// with the caller's update, downloaded from the trial slot. The current state is not changed.
int b200ba_debug_apply_update(b200ba_handle* h, const b200ba_options* opt, const double* x, int32_t n,
                              b200ba_state* out) {
  if (int rc = check_ready(h, opt)) return rc;
  const Layout& L = h->L;
  if (n != L.dof || !x || !out) {
    h->error = "b200ba_debug_apply_update: n does not equal the number of unknowns, or an argument is NULL";
    return 2;
  }
  CUDA_TRY(h, cudaMemcpyAsync(h->d_x, x, static_cast<size_t>(n) * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  launch_update_state(h->pb, L, h->st[h->cur], h->st[1 - h->cur], h->d_x, h->n_control_total, h->n_param_total,
                      h->stream);
  CUDA_TRY(h, cudaGetLastError());
  b200ba_state o = *out;
  o.last_projection = nullptr;  // the warm-start cache is not part of the retraction
  h->cur = 1 - h->cur;
  const int rc = b200ba_get_state(h, &o);
  h->cur = 1 - h->cur;
  return rc;
}

// Diagnostics / tests: launch_cost_reduce on caller's arrays (trial [n], base [n] or NULL,
// residual [2n] as all x then all y, or NULL); stand-alone, one scoped device call.
int b200ba_debug_cost_compare(int device, int64_t n, const double* trial, const double* base, const double* residual,
                              double out[6]) {
  if (n < 0 || (n > 0 && !trial) || !out) {
    g_create_error = "b200ba_debug_cost_compare: bad argument";
    return 2;
  }
  CallScope cs(&g_create_error);
  if (int rc = cs.use_device(device)) return rc;
  const size_t m = static_cast<size_t>(std::max<int64_t>(1, n));
  double *d_t = nullptr, *d_b = nullptr, *d_r = nullptr, *d_partial = nullptr, *d_out = nullptr;
  cs.alloc(&d_t, m);
  if (base) cs.alloc(&d_b, m);
  if (residual) cs.alloc(&d_r, 2 * m);
  cs.alloc(&d_partial, cost_reduce_partial_size());
  cs.alloc(&d_out, 6);
  if (cs.rc == 0 && n > 0) {
    cs.ok(cudaMemcpy(d_t, trial, n * sizeof(double), cudaMemcpyHostToDevice));
    if (base) cs.ok(cudaMemcpy(d_b, base, n * sizeof(double), cudaMemcpyHostToDevice));
    if (residual) cs.ok(cudaMemcpy(d_r, residual, 2 * n * sizeof(double), cudaMemcpyHostToDevice));
  }
  if (cs.rc == 0) {
    launch_cost_reduce(n, d_t, d_b, d_r, d_partial, d_out, 0);
    cs.ok(cudaGetLastError());
    cs.ok(cudaMemcpy(out, d_out, 6 * sizeof(double), cudaMemcpyDeviceToHost));
  }
  return cs.rc;
}

// Diagnostics / tests: ChooseNiceCameraOrientation of every camera applied to the current state, as
// b200ba_run_bundle_adjustment does after each iteration; rot [9 * n_cameras] receives the rotations.
int b200ba_debug_nice_orientation(b200ba_handle* h, double* rot) {
  if (!h) return 1;
  if (!rot || !h->have_state) {
    h->error = "b200ba_debug_nice_orientation: rot is NULL, or no state";
    return 2;
  }
  CUDA_TRY(h, cudaSetDevice(h->device));
  if (!h->d_rot && dev_alloc(h, &h->d_rot, 9 * static_cast<size_t>(h->n_cameras))) return 1;
  launch_nice_orientation(h->pb, h->st[h->cur], h->n_cameras, h->d_rot, h->stream);
  CUDA_TRY(h, cudaGetLastError());
  CUDA_TRY(h, cudaMemcpyAsync(rot, h->d_rot, 9 * sizeof(double) * h->n_cameras, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  return 0;
}

// Diagnostics / tests: the outcome of every LM attempt of the last b200ba_optimize (B200BA_LM_*).
int32_t b200ba_debug_lm_events(const b200ba_handle* h, int32_t* codes, int32_t cap) {
  if (!h) return -1;
  const int32_t n = static_cast<int32_t>(h->lm_events.size());
  for (int32_t i = 0; i < n && i < cap && codes; ++i) codes[i] = h->lm_events[i];
  return n;
}

// Diagnostics / tests: evaluation budget of the main Jacobian pass (default 16); 1 forces every
// observation of a generic camera through the straggler pass.
B200BA_API void b200ba_debug_set_eval_budget(int budget) { set_main_eval_budget(budget); }

// Diagnostics: spline evaluations spent per observation by the last pass that wrote Jacobians
// (caller's observation order). Not part of the reference interface.
B200BA_API int b200ba_debug_eval_counts(b200ba_handle* h, uint16_t* counts) {
  if (!h || !counts || !h->have_layout) return 1;
  std::vector<uint16_t> tmp(h->n_obs);
  CUDA_TRY(h, cudaMemcpy(tmp.data(), h->out.evals, h->n_obs * sizeof(uint16_t), cudaMemcpyDeviceToHost));
  for (int64_t i = 0; i < h->n_obs; ++i) counts[h->perm[i]] = tmp[i];
  return 0;
}

int b200ba_get_timings(const b200ba_handle* h, b200ba_timings* t) {
  if (!h || !t) return 1;
  *t = h->timings;
  return 0;
}

// ---- stand-alone dense SPD solve on the in-tree kernels (tests / profiling) ---------------------
// A: n x n symmetric (either major order), host. Factorises with the blocked Cholesky of ba_dense.cu
// (block width nb, a multiple of 128) and solves A x = b. Returns 4 when a pivot is not positive.
int b200ba_dense_cholesky_solve(int device, int32_t n, int32_t nb, const double* A, const double* b, double* x,
                                double* factor_ms, double* solve_ms) {
  if (n < 1 || nb < 128 || nb % 128 != 0 || !A || !b || !x) {
    g_create_error = "b200ba_dense_cholesky_solve: bad argument";
    return 2;
  }
  CallScope cs(&g_create_error);
  if (int rc = cs.use_device(device)) return rc;
  set_gemm_sm_reserve(getenv("B200BA_PANEL_SMS") ? atoi(getenv("B200BA_PANEL_SMS")) : 8);
  DenseCtx d;
  dense_plan(&d, n, nb, 0, 1);
  double* dA = nullptr;
  double* db = nullptr;
  cs.ok(dense_create(&d, /*own_streams=*/true));
  cs.alloc(&dA, static_cast<size_t>(n) * n);
  cs.alloc(&d.S, static_cast<size_t>(d.chunk));
  cs.alloc(&d.Lpack, static_cast<size_t>(d.panel_off[d.nblk]));
  cs.alloc(&d.tmp, static_cast<size_t>(n));
  cs.alloc(&d.d_panel_off, d.panel_off.size());
  cs.alloc(&d.d_panel_h, d.panel_h.size());
  cs.alloc(&db, static_cast<size_t>(n));
  cs.alloc(&d.info, 1);
  if (cs.rc == 0) {
    cs.ok(cudaMemcpy(dA, A, static_cast<size_t>(n) * n * sizeof(double), cudaMemcpyHostToDevice));
    cs.ok(cudaMemcpy(db, b, static_cast<size_t>(n) * sizeof(double), cudaMemcpyHostToDevice));
    cs.ok(cudaMemcpy(d.d_panel_off, d.panel_off.data(), d.panel_off.size() * sizeof(int64_t), cudaMemcpyHostToDevice));
    cs.ok(cudaMemcpy(d.d_panel_h, d.panel_h.data(), d.panel_h.size() * sizeof(int), cudaMemcpyHostToDevice));
    cs.ok(cudaMemset(d.S, 0, static_cast<size_t>(d.chunk) * sizeof(double)));
    cs.ok(cudaMemset(d.info, 0, sizeof(int)));
    cs.ok(cudaMemcpy2D(d.S, d.map.ld * sizeof(double), dA, static_cast<size_t>(n) * sizeof(double),
                       static_cast<size_t>(n) * sizeof(double), n, cudaMemcpyDeviceToDevice));
    cs.ok(cudaDeviceSynchronize());  // device-to-device copies are asynchronous; the work below runs on non-blocking streams
  }
  if (cs.rc == 0) {
    cs.record(0, d.s_main);
    if (dense_factor(&d)) cs.fail("b200ba_dense_cholesky_solve: kernel launch failed");
    cs.record(1, d.s_main);
    if (cs.rc == 0 && dense_solve(&d, db)) cs.fail("b200ba_dense_cholesky_solve: kernel launch failed");
    cs.record(2, d.s_main);
    cs.ok(cudaStreamSynchronize(d.s_main));
    cs.ok(cudaStreamSynchronize(d.s_panel));
  }
  if (cs.rc == 0) {
    if (factor_ms) *factor_ms = cs.elapsed_ms(0, 1);
    if (solve_ms) *solve_ms = cs.elapsed_ms(1, 2);
    int info = 0;
    cs.ok(cudaMemcpy(&info, d.info, sizeof(int), cudaMemcpyDeviceToHost));
    cs.ok(cudaMemcpy(x, db, static_cast<size_t>(n) * sizeof(double), cudaMemcpyDeviceToHost));
    if (cs.rc == 0 && info != 0) {
      g_create_error = "b200ba_dense_cholesky_solve: the matrix is not positive definite";
      cs.rc = 4;
    }
  }
  dense_release(&d, /*own_streams=*/true);
  return cs.rc;
}

// ---- stand-alone Schur solve (known-answer tests) ---------------------------------------------
int b200ba_schur_solve(int device, int32_t bs, int32_t nb, int32_t nd, const double* D, const double* B,
                       const double* C, const double* b1, const double* b2, double* x) {
  if (bs < 1 || bs > 6 || nb < 0 || nd < 1 || !D || !B || !C || !b1 || !b2 || !x) {
    g_create_error = "b200ba_schur_solve: bad argument";
    return 2;
  }
  CallScope cs(&g_create_error);
  if (int rc = cs.use_device(device)) return rc;
  const int nbd = bs * nb;
  double *dD = nullptr, *dB = nullptr, *dC = nullptr, *db1 = nullptr, *db2 = nullptr, *dDinvB = nullptr, *dDinvb = nullptr,
         *dwork = nullptr;
  int *dipiv = nullptr, *dinfo = nullptr;
  cs.alloc(&dD, std::max(1, nb * bs * bs));
  cs.alloc(&dB, std::max<size_t>(1, static_cast<size_t>(nbd) * nd));
  cs.alloc(&dC, static_cast<size_t>(nd) * nd);
  cs.alloc(&db1, std::max(1, nbd));
  cs.alloc(&db2, nd);
  cs.alloc(&dDinvB, std::max<size_t>(1, static_cast<size_t>(nbd) * nd));
  cs.alloc(&dDinvb, std::max(1, nbd));
  cs.alloc(&dipiv, nd);
  cs.alloc(&dinfo, 1);
  if (cs.rc == 0) {
    cs.ok(cudaMemcpy(dD, D, sizeof(double) * nb * bs * bs, cudaMemcpyHostToDevice));
    cs.ok(cudaMemcpy(dB, B, sizeof(double) * static_cast<size_t>(nbd) * nd, cudaMemcpyHostToDevice));
    cs.ok(cudaMemcpy(dC, C, sizeof(double) * static_cast<size_t>(nd) * nd, cudaMemcpyHostToDevice));
    cs.ok(cudaMemcpy(db1, b1, sizeof(double) * nbd, cudaMemcpyHostToDevice));
    cs.ok(cudaMemcpy(db2, b2, sizeof(double) * nd, cudaMemcpyHostToDevice));
  }
  if (cs.create_solvers()) {
    const double one = 1.0, m1 = -1.0;
    launch_symmetrize(nd, dC, 0);
    launch_generic_block_inverse(bs, nb, nd, dD, dB, db1, dDinvB, dDinvb, 0);
    if (nbd > 0) {
      // S = C - B^T D^-1 B ; sb = b2 - B^T D^-1 b1
      cublasDgemm(cs.cublas, CUBLAS_OP_N, CUBLAS_OP_T, nd, nd, nbd, &m1, dB, nd, dDinvB, nd, &one, dC, nd);
      cublasDgemv(cs.cublas, CUBLAS_OP_N, nd, nbd, &m1, dB, nd, dDinvb, 1, &one, db2, 1);
    }
    int lwork = 0;
    cusolverDnDgetrf_bufferSize(cs.cusolver, nd, nd, dC, nd, &lwork);
    cs.alloc(&dwork, std::max(1, lwork));
    cusolverDnDgetrf(cs.cusolver, nd, nd, dC, nd, dwork, dipiv, dinfo);
    cusolverDnDgetrs(cs.cusolver, CUBLAS_OP_N, nd, 1, dC, nd, dipiv, db2, nd, dinfo);
    if (nbd > 0) cublasDgemv(cs.cublas, CUBLAS_OP_T, nd, nbd, &m1, dDinvB, nd, db2, 1, &one, dDinvb, 1);
    cs.ok(cudaDeviceSynchronize());
    if (nbd > 0) cs.ok(cudaMemcpy(x, dDinvb, sizeof(double) * nbd, cudaMemcpyDeviceToHost));
    cs.ok(cudaMemcpy(x + nbd, db2, sizeof(double) * nd, cudaMemcpyDeviceToHost));
  }
  return cs.rc;
}

// ---- stand-alone model evaluation ------------------------------------------------------------------
static int model_io(int device, const b200ba_camera* cam, const double* intrinsics, int64_t n, const double* in,
                    int in_w, double* io_pixels, double* dirs, double* origins, int32_t* ok_out, bool project) {
  if (!cam || !intrinsics || n < 0) {
    g_create_error = "bad argument";
    return 2;
  }
  CallScope cs(&g_create_error);
  if (int rc = cs.use_device(device)) return rc;
  CamDev c{};
  fill_camdev(*cam, &c);
  const int64_t ni = intrinsics_size(*cam);
  double *dintr = nullptr, *din = nullptr, *dpx = nullptr, *ddir = nullptr, *dorg = nullptr;
  int32_t* dok = nullptr;
  const size_t nn = std::max<int64_t>(1, n);
  cs.alloc(&dintr, ni);
  cs.alloc(&din, in_w * nn);
  cs.alloc(&dpx, 2 * nn);
  cs.alloc(&ddir, 3 * nn);
  cs.alloc(&dorg, 3 * nn);
  cs.alloc(&dok, nn);
  if (cs.rc == 0) {
    cs.ok(cudaMemcpy(dintr, intrinsics, sizeof(double) * ni, cudaMemcpyHostToDevice));
    if (project) {
      cs.ok(cudaMemcpy(din, in, sizeof(double) * 3 * n, cudaMemcpyHostToDevice));
      cs.ok(cudaMemcpy(dpx, io_pixels, sizeof(double) * 2 * n, cudaMemcpyHostToDevice));
      launch_project_points(c, dintr, n, din, dpx, dok, 0);
    } else {
      cs.ok(cudaMemcpy(dpx, in, sizeof(double) * 2 * n, cudaMemcpyHostToDevice));
      launch_unproject_pixels(c, dintr, n, dpx, ddir, dorg, dok, 0);
    }
    cs.ok(cudaDeviceSynchronize());
    if (project) {
      cs.ok(cudaMemcpy(io_pixels, dpx, sizeof(double) * 2 * n, cudaMemcpyDeviceToHost));
    } else {
      if (dirs) cs.ok(cudaMemcpy(dirs, ddir, sizeof(double) * 3 * n, cudaMemcpyDeviceToHost));
      if (origins) cs.ok(cudaMemcpy(origins, dorg, sizeof(double) * 3 * n, cudaMemcpyDeviceToHost));
    }
    if (ok_out) cs.ok(cudaMemcpy(ok_out, dok, sizeof(int32_t) * n, cudaMemcpyDeviceToHost));
  }
  return cs.rc;
}

int b200ba_project(int device, const b200ba_camera* cam, const double* intrinsics, int64_t n,
                   const double* local_points, double* pixels, int32_t* ok) {
  return model_io(device, cam, intrinsics, n, local_points, 3, pixels, nullptr, nullptr, ok, true);
}
int b200ba_unproject(int device, const b200ba_camera* cam, const double* intrinsics, int64_t n, const double* pixels,
                     double* directions, double* origins, int32_t* ok) {
  return model_io(device, cam, intrinsics, n, pixels, 2, nullptr, directions, origins, ok, false);
}

// CentralGenericModel::FitToPixelDirectionsImpl (APP/models/central_generic.cc:551-568):
// LMOptimizer<double>::Optimize(max_iteration_count, max_lm_attempts = 10, init_lambda = -1,
// init_lambda_factor = 0.001f) over the direction grid (LV/lm_optimizer.h:628-991 without the
// Schur structure: SolveDensely). H (row-major upper == column-major lower) is built by
// dirfit_kernel<true>; every attempt factors a copy of H + lambda I with cuSOLVER.
int b200ba_fit_directions(int device, int32_t gw, int32_t gh, double* grid, int64_t n, const double* grid_points,
                          const double* directions, int32_t max_iteration_count, b200ba_fit_report* report) {
  if (gw < 4 || gh < 4 || !grid || n < 0 || (n > 0 && (!grid_points || !directions)) || !report) {
    g_create_error = "b200ba_fit_directions: bad argument";
    return 2;
  }
  for (int64_t i = 0; i < n; ++i) {
    const double gx = grid_points[2 * i], gy = grid_points[2 * i + 1];
    if (!(gx >= 1.0 && gx < gw - 2 && gy >= 1.0 && gy < gh - 2)) {
      g_create_error = "b200ba_fit_directions: a grid point has no complete 4x4 support";
      return 2;
    }
  }
  CallScope cs(&g_create_error);
  if (int rc = cs.use_device(device)) return rc;
  memset(report, 0, sizeof(*report));
  const int G = gw * gh, dof = 2 * G;
  const size_t nn = static_cast<size_t>(std::max<int64_t>(1, n));
  double *dgrid = nullptr, *dtrial = nullptr, *dtan = nullptr, *dgp = nullptr, *ddir = nullptr, *dH = nullptr,
         *dS = nullptr, *db = nullptr, *dx = nullptr, *dcost = nullptr, *dsum = nullptr, *dwork = nullptr;
  int* dinfo = nullptr;
  const size_t hsize = static_cast<size_t>(dof) * dof, hbytes = sizeof(double) * hsize;
  cs.alloc(&dgrid, 3 * G);
  cs.alloc(&dtrial, 3 * G);
  cs.alloc(&dtan, 6 * G);
  cs.alloc(&dgp, 2 * nn);
  cs.alloc(&ddir, 3 * nn);
  cs.alloc(&dH, hsize);
  cs.alloc(&dS, hsize);
  cs.alloc(&db, dof);
  cs.alloc(&dx, dof);
  cs.alloc(&dcost, nn);
  cs.alloc(&dsum, 2);
  cs.alloc(&dinfo, 2);
  int lwork = 0;
  if (cs.create_solvers()) {
    if (cusolverDnDpotrf_bufferSize(cs.cusolver, CUBLAS_FILL_MODE_LOWER, dof, dS, dof, &lwork) != CUSOLVER_STATUS_SUCCESS)
      cs.fail("cusolverDnDpotrf_bufferSize failed");
    cs.alloc(&dwork, std::max(1, lwork));
  }
  if (cs.rc == 0) {
    cs.ok(cudaMemcpy(dgrid, grid, sizeof(double) * 3 * G, cudaMemcpyHostToDevice));
    if (n > 0) {
      cs.ok(cudaMemcpy(dgp, grid_points, sizeof(double) * 2 * n, cudaMemcpyHostToDevice));
      cs.ok(cudaMemcpy(ddir, directions, sizeof(double) * 3 * n, cudaMemcpyHostToDevice));
    }
  }
  const LmResult lm = small_lm(
      cs.rc, max_iteration_count,
      [&](int) {  // H and b rebuilt at the current grid every iteration
        double cost = 0;
        launch_dirfit_tangents(G, dgrid, dtan, 0);
        cs.ok(cudaMemsetAsync(dH, 0, hbytes, 0));
        cs.ok(cudaMemsetAsync(db, 0, sizeof(double) * dof, 0));
        launch_dirfit(true, gw, n, dgp, ddir, dgrid, dtan, dH, db, dof, dcost, dsum, 0);
        cs.ok(cudaMemcpy(&cost, dsum, sizeof(double), cudaMemcpyDeviceToHost));
        return cost;
      },
      [&](double init_lambda_factor) {
        double trace = 0;  // the diagonal of J^T J is non-negative: sum |h_ii| = trace
        if (cublasDasum(cs.cublas, dof, dH, dof + 1, &trace) != CUBLAS_STATUS_SUCCESS) cs.fail("cublasDasum failed");
        return init_lambda_factor * trace / dof;
      },
      [&](double lambda) {
        cs.ok(cudaMemcpyAsync(dS, dH, hbytes, cudaMemcpyDeviceToDevice, 0));
        launch_add_diagonal(dof, dS, dof, lambda, 0);
        cs.ok(cudaMemcpyAsync(dx, db, sizeof(double) * dof, cudaMemcpyDeviceToDevice, 0));
        int info[2] = {0, 0};
        if (cusolverDnDpotrf(cs.cusolver, CUBLAS_FILL_MODE_LOWER, dof, dS, dof, dwork, lwork, dinfo) !=
                CUSOLVER_STATUS_SUCCESS ||
            cusolverDnDpotrs(cs.cusolver, CUBLAS_FILL_MODE_LOWER, dof, 1, dS, dof, dx, dof, dinfo + 1) !=
                CUSOLVER_STATUS_SUCCESS) {
          cs.fail("cuSOLVER potrf / potrs failed");
          return false;
        }
        cs.ok(cudaMemcpy(info, dinfo, sizeof(info), cudaMemcpyDeviceToHost));
        return info[0] == 0;  // false: not positive definite, the reference's NaN-update branch
      },
      [&] {
        double cost = 0;
        launch_dirfit_update(G, dgrid, dx, dtrial, 0);
        launch_dirfit(false, gw, n, dgp, ddir, dtrial, dtan, nullptr, nullptr, dof, dcost, dsum + 1, 0);
        cs.ok(cudaMemcpy(&cost, dsum + 1, sizeof(double), cudaMemcpyDeviceToHost));
        return cost;
      },
      [&] { std::swap(dgrid, dtrial); });
  report->initial_cost = lm.initial_cost;
  report->num_iterations_performed = lm.iterations;
  report->lm_attempts = lm.attempts;
  if (cs.rc == 0) {
    cs.ok(cudaGetLastError());
    cs.ok(cudaMemcpy(grid, dgrid, sizeof(double) * 3 * G, cudaMemcpyDeviceToHost));
    report->final_cost = lm.final_cost;
    report->final_lambda = lm.lambda;
  }
  return cs.rc;
}

// The argument checks of b200ba_compare_models and b200ba_fitting_images, which touch no CUDA state: the reference
// compares central-generic models only (compare_calibrations.cc:60-66) of one image size (fitting_report.h:65-66, a
// CHECK_EQ there). `fn` prefixes the message.
static int check_compare_arguments(const char* fn, const b200ba_camera* cam_a, const double* intr_a,
                                   const b200ba_camera* cam_b, const double* intr_b,
                                   const b200ba_fitting_report* report) {
  const std::string prefix = std::string(fn) + ": ";
  if (!cam_a || !intr_a || !cam_b || !intr_b || !report) {
    g_create_error = prefix + "a required argument is NULL";
    return 2;
  }
  if (cam_a->model_type != B200BA_MODEL_CENTRAL_GENERIC || cam_b->model_type != B200BA_MODEL_CENTRAL_GENERIC) {
    g_create_error = prefix + "calibration comparison is only implemented for CentralGenericModel";
    return 2;
  }
  if (cam_a->width != cam_b->width || cam_a->height != cam_b->height || cam_a->width < 1 || cam_a->height < 1) {
    g_create_error = prefix + "the models differ in image size (" + std::to_string(cam_a->width) + " x " +
                     std::to_string(cam_a->height) + " against " + std::to_string(cam_b->width) + " x " +
                     std::to_string(cam_b->height) + ")";
    return 2;
  }
  if (cam_a->grid_width < 4 || cam_a->grid_height < 4 || cam_b->grid_width < 4 || cam_b->grid_height < 4) {
    g_create_error = prefix + "a grid is smaller than 4 x 4";
    return 2;
  }
  return 0;
}

// The five images of b200ba_fitting_images, in the caller's memory.
struct FittingImagesOut {
  uint8_t *magnitudes, *angles, *directions, *rep_magnitudes, *reprojections;
};

// CreateFittingErrorReport(base = A, fitted = B, Identity) (APP/fitting_report.h:55-203) after the argument checks:
// the numbers, the per-pixel arrays that are asked for and, with `images`, the five images. The report does not
// depend on whether the images are computed.
static int run_comparison(int device, const b200ba_camera* cam_a, const double* intr_a, const b200ba_camera* cam_b,
                          const double* intr_b, b200ba_fitting_report* report, double* direction_errors,
                          double* reprojection_errors, const FittingImagesOut* images, double* device_ms) {
  CallScope cs(&g_create_error);
  if (int rc = cs.use_device(device)) return rc;
  CamDev ca{}, cb{};
  fill_camdev(*cam_a, &ca);
  fill_camdev(*cam_b, &cb);
  const int64_t n = static_cast<int64_t>(cam_a->width) * cam_a->height;
  const int64_t na = intrinsics_size(*cam_a), nb = intrinsics_size(*cam_b);
  double *dga = nullptr, *dgb = nullptr;
  CompareDev d{};
  cs.alloc(&dga, na);
  cs.alloc(&dgb, nb);
  cs.alloc(&d.mag, n);
  if (direction_errors || images) cs.alloc(&d.dir_err, 3 * n);
  if (reprojection_errors) cs.alloc(&d.rep_err, 2 * n);
  cs.alloc(&d.dir_max, 2);
  alloc_range_statistics(cs, n, &d.range, &d.partial, &d.select_hist, &d.stats);
  uint8_t* dimg = nullptr;  // the five images in one allocation: 1 + 3 + 3 + 1 + 3 bytes per pixel
  if (images) {
    cs.alloc(&dimg, 11 * n);
    if (dimg) {
      d.magnitudes = dimg;
      d.angles = dimg + n;
      d.directions = dimg + 4 * n;
      d.rep_magnitudes = dimg + 7 * n;
      d.reprojections = dimg + 8 * n;
    }
  }
  ReportCam stats{};
  unsigned long long dir_max[2] = {0, 0};
  if (cs.rc == 0) {
    cs.ok(cudaMemcpy(dga, intr_a, sizeof(double) * na, cudaMemcpyHostToDevice));
    cs.ok(cudaMemcpy(dgb, intr_b, sizeof(double) * nb, cudaMemcpyHostToDevice));
  }
  if (cs.rc == 0) {
    cs.record(0, 0);
    launch_compare_models(ca, dga, cb, dgb, d, 0);
    cs.record(1, 0);
    cs.ok(cudaGetLastError());
    cs.ok(cudaMemcpy(&stats, d.stats, sizeof(ReportCam), cudaMemcpyDeviceToHost));
    cs.ok(cudaMemcpy(dir_max, d.dir_max, sizeof(dir_max), cudaMemcpyDeviceToHost));
    if (direction_errors) cs.ok(cudaMemcpy(direction_errors, d.dir_err, sizeof(double) * 3 * n, cudaMemcpyDeviceToHost));
    if (reprojection_errors) cs.ok(cudaMemcpy(reprojection_errors, d.rep_err, sizeof(double) * 2 * n, cudaMemcpyDeviceToHost));
    if (images) {
      cs.ok(cudaMemcpy(images->magnitudes, d.magnitudes, n, cudaMemcpyDeviceToHost));
      cs.ok(cudaMemcpy(images->angles, d.angles, 3 * n, cudaMemcpyDeviceToHost));
      cs.ok(cudaMemcpy(images->directions, d.directions, 3 * n, cudaMemcpyDeviceToHost));
      cs.ok(cudaMemcpy(images->rep_magnitudes, d.rep_magnitudes, n, cudaMemcpyDeviceToHost));
      cs.ok(cudaMemcpy(images->reprojections, d.reprojections, 3 * n, cudaMemcpyDeviceToHost));
    }
  }
  if (cs.rc == 0) {
    if (device_ms) *device_ms = cs.elapsed_ms(0, 1);
    report->reprojection_error_count = stats.count;
    report->reprojection_error_sum = stats.sum;
    report->reprojection_error_max = stats.max;
    report->reprojection_error_median = stats.median;
    memcpy(&report->max_error_norm, &dir_max[0], sizeof(double));
    memcpy(&report->max_error_component, &dir_max[1], sizeof(double));
  }
  return cs.rc;
}

int b200ba_compare_models(int device, const b200ba_camera* cam_a, const double* intr_a, const b200ba_camera* cam_b,
                          const double* intr_b, b200ba_fitting_report* report, double* direction_errors,
                          double* reprojection_errors, double* device_ms) {
  if (int rc = check_compare_arguments("b200ba_compare_models", cam_a, intr_a, cam_b, intr_b, report)) return rc;
  return run_comparison(device, cam_a, intr_a, cam_b, intr_b, report, direction_errors, reprojection_errors, nullptr,
                        device_ms);
}

int b200ba_fitting_images(int device, const b200ba_camera* cam_a, const double* intr_a, const b200ba_camera* cam_b,
                          const double* intr_b, b200ba_fitting_report* report, uint8_t* error_magnitudes,
                          uint8_t* error_direction_angles, uint8_t* error_directions, uint8_t* reprojection_magnitudes,
                          uint8_t* reprojections, double* device_ms) {
  if (int rc = check_compare_arguments("b200ba_fitting_images", cam_a, intr_a, cam_b, intr_b, report)) return rc;
  if (!error_magnitudes || !error_direction_angles || !error_directions || !reprojection_magnitudes || !reprojections) {
    g_create_error = "b200ba_fitting_images: an image pointer is NULL";
    return 2;
  }
  const FittingImagesOut images{error_magnitudes, error_direction_angles, error_directions, reprojection_magnitudes,
                                reprojections};
  return run_comparison(device, cam_a, intr_a, cam_b, intr_b, report, nullptr, nullptr, &images, device_ms);
}

// The localization accuracy test (APP/tools/localization_accuracy_test.cc:47-131). The argument checks come first
// and touch no CUDA state. The sampling kernel runs first; a point that is not drawn within kLocMaxDraws ends the call
// with 4 before any fit, where the reference would loop forever.
int b200ba_localization_accuracy(int device, const b200ba_camera* gt_cam, const double* gt_intr, const b200ba_camera* cam,
                                 const double* intr, int64_t trials, uint64_t seed, b200ba_localization_report* report,
                                 float* errors, double* poses, float* samples, double* device_ms) {
  if (!gt_cam || !gt_intr || !cam || !intr || !report) {
    g_create_error = "b200ba_localization_accuracy: a required argument is NULL";
    return 2;
  }
  if (gt_cam->model_type != B200BA_MODEL_CENTRAL_GENERIC || cam->model_type != B200BA_MODEL_CENTRAL_GENERIC) {
    g_create_error = "b200ba_localization_accuracy: the localization accuracy test is only implemented for "
                     "CentralGenericModel";
    return 2;
  }
  if (gt_cam->width != cam->width || gt_cam->height != cam->height || gt_cam->width < 1 || gt_cam->height < 1) {
    g_create_error = "b200ba_localization_accuracy: The ground truth and compared camera models do not have the same "
                     "image size.";
    return 2;
  }
  if (gt_cam->grid_width < 4 || gt_cam->grid_height < 4 || cam->grid_width < 4 || cam->grid_height < 4) {
    g_create_error = "b200ba_localization_accuracy: a grid is smaller than 4 x 4";
    return 2;
  }
  if (trials < 1 || trials > (int64_t(1) << 32)) {
    g_create_error = "b200ba_localization_accuracy: trials must be in [1, 2^32]";
    return 2;
  }
  // pixels are drawn in [0, w] x [0, h]; a calibrated area is [min, max + 1) in x and y
  const double lo_x = std::max({0.0, double(gt_cam->calibration_min_x), double(cam->calibration_min_x)});
  const double lo_y = std::max({0.0, double(gt_cam->calibration_min_y), double(cam->calibration_min_y)});
  const double hi_x = std::min({double(gt_cam->width), gt_cam->calibration_max_x + 1.0, cam->calibration_max_x + 1.0});
  const double hi_y = std::min({double(gt_cam->height), gt_cam->calibration_max_y + 1.0, cam->calibration_max_y + 1.0});
  if (!(lo_x < hi_x && lo_y < hi_y)) {
    g_create_error = "b200ba_localization_accuracy: the calibrated areas of the two models do not intersect in the image";
    return 2;
  }
  CallScope cs(&g_create_error);
  if (int rc = cs.use_device(device)) return rc;
  CamDev cg{}, cc{};
  fill_camdev(*gt_cam, &cg);
  fill_camdev(*cam, &cc);
  const int64_t n = trials * kLocPoints;
  const int64_t ng = intrinsics_size(*gt_cam), nc = intrinsics_size(*cam);
  double *dgg = nullptr, *dgc = nullptr;
  LocalizationDev d{};
  cs.alloc(&dgg, ng);
  cs.alloc(&dgc, nc);
  cs.alloc(&d.p, 3 * n);
  cs.alloc(&d.f, 3 * n);
  if (samples) cs.alloc(&d.samples, 3 * n);
  if (poses) cs.alloc(&d.poses, 6 * trials);
  cs.alloc(&d.mag, trials);
  cs.alloc(&d.counts, 3);
  cs.alloc(&d.capped, 1);
  alloc_range_statistics(cs, trials, &d.range, &d.partial, &d.select_hist, &d.stats);
  if (cs.rc == 0) {
    cs.ok(cudaMemcpy(dgg, gt_intr, sizeof(double) * ng, cudaMemcpyHostToDevice));
    cs.ok(cudaMemcpy(dgc, intr, sizeof(double) * nc, cudaMemcpyHostToDevice));
  }
  int capped = 0;
  if (cs.rc == 0) {
    cs.record(0, 0);
    launch_localization_sample(cg, dgg, cc, dgc, trials, seed, d, 0);
    cs.ok(cudaGetLastError());
    cs.ok(cudaMemcpy(&capped, d.capped, sizeof(int), cudaMemcpyDeviceToHost));
  }
  if (cs.rc == 0 && capped) {
    g_create_error = "b200ba_localization_accuracy: a point was not un-projected by both models within " +
                     std::to_string(kLocMaxDraws) + " draws";
    return 4;
  }
  ReportCam stats{};
  unsigned long long counts[3] = {0, 0, 0};
  if (cs.rc == 0) {
    launch_localization_pose(trials, d, 0);
    cs.record(1, 0);
    cs.ok(cudaGetLastError());
    cs.ok(cudaMemcpy(&stats, d.stats, sizeof(ReportCam), cudaMemcpyDeviceToHost));
    cs.ok(cudaMemcpy(counts, d.counts, sizeof(counts), cudaMemcpyDeviceToHost));
    if (errors) {
      std::vector<double> mag(trials);
      cs.ok(cudaMemcpy(mag.data(), d.mag, sizeof(double) * trials, cudaMemcpyDeviceToHost));
      for (int64_t i = 0; i < trials; ++i) errors[i] = static_cast<float>(mag[i]);  // exact: mag holds floats
    }
    if (poses) cs.ok(cudaMemcpy(poses, d.poses, sizeof(double) * 6 * trials, cudaMemcpyDeviceToHost));
    if (samples) cs.ok(cudaMemcpy(samples, d.samples, sizeof(float) * 3 * n, cudaMemcpyDeviceToHost));
  }
  if (cs.rc == 0) {
    if (device_ms) *device_ms = cs.elapsed_ms(0, 1);
    b200ba_localization_report r{};
    r.trial_count = stats.count;
    r.average_error = stats.count > 0 ? stats.sum / static_cast<double>(stats.count) : std::nan("");
    r.median_error = stats.median;
    r.max_error = stats.max;
    r.total_iterations = static_cast<int64_t>(counts[1]);
    r.redraws = static_cast<int64_t>(counts[0]);
    r.max_iterations = static_cast<int32_t>(counts[2]);
    *report = r;
  }
  return cs.rc;
}

// ---- reconstruction comparison (APP/tools/bundle_adjustment.cc:223-392) -------------------------------------------
// R(q) of a unit quaternion (w, x, y, z), row-major
static void quat_matrix(const double* q, double R[9]) {
  const double w = q[0], x = q[1], y = q[2], z = q[3];
  R[0] = 1 - 2 * (y * y + z * z);
  R[1] = 2 * (x * y - w * z);
  R[2] = 2 * (x * z + w * y);
  R[3] = 2 * (x * y + w * z);
  R[4] = 1 - 2 * (x * x + z * z);
  R[5] = 2 * (y * z - w * x);
  R[6] = 2 * (x * z - w * y);
  R[7] = 2 * (y * z + w * x);
  R[8] = 1 - 2 * (x * x + y * y);
}

// image_tr_global = camera_tr_rig * rig_tr_global (Sophus: the product quaternion is normalised); its rotation R and
// the centre -R^T t of its inverse G
static void image_centre(const double* camera_tr_rig, const double* rig_tr_global, double R[9], double c[3]) {
  const double* a = camera_tr_rig;
  const double* b = rig_tr_global;
  double q[4] = {a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
                 a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                 a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3],
                 a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1]};
  const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  for (double& v : q) v /= n;
  double Ra[9];
  quat_matrix(a, Ra);
  double t[3];
  for (int r = 0; r < 3; ++r) t[r] = a[4 + r] + (Ra[3 * r] * b[4] + Ra[3 * r + 1] * b[5] + Ra[3 * r + 2] * b[6]);
  quat_matrix(q, R);
  for (int r = 0; r < 3; ++r) c[r] = -(R[r] * t[0] + R[3 + r] * t[1] + R[6 + r] * t[2]);
}

// Horn's quaternion method: for M = sum a b^T (a the targets, b the sources), the rotation R maximising tr(R^T M)
// = sum a^T R b is R(q) for the unit eigenvector q of the largest eigenvalue of the symmetric 4 x 4 matrix N(M), and
// that eigenvalue is the maximum. Cyclic Jacobi: a rotation is skipped where the off-diagonal entry is exactly zero, so
// a block-diagonal N (M symmetric) keeps its first row untouched and gives q = (1, 0, 0, 0) exactly.
static void horn_rotation(const double M[9], double R[9], double* lambda1, double* lambda2) {
  // S = M^T: S_ij = sum b_i a_j (Horn 1987, eq. 28 ff.)
  const double Sxx = M[0], Sxy = M[3], Sxz = M[6], Syx = M[1], Syy = M[4], Syz = M[7], Szx = M[2], Szy = M[5],
               Szz = M[8];
  double A[4][4] = {{Sxx + Syy + Szz, Syz - Szy, Szx - Sxz, Sxy - Syx},
                    {Syz - Szy, Sxx - Syy - Szz, Sxy + Syx, Szx + Sxz},
                    {Szx - Sxz, Sxy + Syx, -Sxx + Syy - Szz, Syz + Szy},
                    {Sxy - Syx, Szx + Sxz, Syz + Szy, -Sxx - Syy + Szz}};
  double V[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
  for (int sweep = 0; sweep < 64; ++sweep) {
    bool rotated = false;
    for (int p = 0; p < 3; ++p) {
      for (int r = p + 1; r < 4; ++r) {
        const double apq = A[p][r];
        if (apq == 0) continue;
        // negligible against both diagonal entries: set to zero (the classical Jacobi threshold)
        if (std::fabs(A[p][p]) + 1e3 * std::fabs(apq) == std::fabs(A[p][p]) &&
            std::fabs(A[r][r]) + 1e3 * std::fabs(apq) == std::fabs(A[r][r]) && sweep > 3) {
          A[p][r] = A[r][p] = 0;
          continue;
        }
        rotated = true;
        const double theta = (A[r][r] - A[p][p]) / (2 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1));
        const double c = 1 / std::sqrt(t * t + 1), s = t * c;
        for (int k = 0; k < 4; ++k) {  // A <- A J (columns p, r)
          const double akp = A[k][p], akr = A[k][r];
          A[k][p] = c * akp - s * akr;
          A[k][r] = s * akp + c * akr;
        }
        for (int k = 0; k < 4; ++k) {  // A <- J^T A (rows p, r)
          const double apk = A[p][k], ark = A[r][k];
          A[p][k] = c * apk - s * ark;
          A[r][k] = s * apk + c * ark;
        }
        A[p][r] = A[r][p] = 0;
        for (int k = 0; k < 4; ++k) {
          const double vkp = V[k][p], vkr = V[k][r];
          V[k][p] = c * vkp - s * vkr;
          V[k][r] = s * vkp + c * vkr;
        }
      }
    }
    if (!rotated) break;
  }
  int i1 = 0;
  for (int k = 1; k < 4; ++k)
    if (A[k][k] > A[i1][i1]) i1 = k;
  int i2 = i1 == 0 ? 1 : 0;
  for (int k = 0; k < 4; ++k)
    if (k != i1 && A[k][k] > A[i2][i2]) i2 = k;
  *lambda1 = A[i1][i1];
  *lambda2 = A[i2][i2];
  double q[4] = {V[0][i1], V[1][i1], V[2][i1], V[3][i1]};
  const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  for (double& v : q) v /= n;
  quat_matrix(q, R);
}

static double norm3(const double v[3]) { return std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }

static bool centres_coincide(int32_t n, const double* rig_tr_global, const double* camera_tr_rig) {
  double R[9], c0[3], c[3];
  image_centre(camera_tr_rig, rig_tr_global, R, c0);
  for (int32_t i = 1; i < n; ++i) {
    image_centre(camera_tr_rig, rig_tr_global + 7 * static_cast<int64_t>(i), R, c);
    if (c[0] != c0[0] || c[1] != c0[1] || c[2] != c0[2]) return false;
  }
  return true;
}

// argument checks of the host part; 0 or 2 (with g_create_error set)
static int alignment_arguments(const char* who, int32_t n_images, const double* rtg1, const double* ctr1, const double* rtg2,
                        const double* ctr2) {
  const std::string prefix = std::string(who) + ": ";
  if (!rtg1 || !ctr1 || !rtg2 || !ctr2) {
    g_create_error = prefix + "a required argument is NULL";
    return 2;
  }
  if (n_images < 2) {
    g_create_error = prefix + "the reconstructions need at least two images";
    return 2;
  }
  if (centres_coincide(n_images, rtg1, ctr1) || centres_coincide(n_images, rtg2, ctr2)) {
    g_create_error = prefix + "all camera centres of a reconstruction coincide";
    return 2;
  }
  return 0;
}

static int reconstruction_alignment(int64_t pairs, const double* M, int32_t n, const double* rtg1, const double* ctr1,
                             const double* rtg2, const double* ctr2, b200ba_reconstruction_comparison* out) {
  b200ba_reconstruction_comparison r{};
  r.direction_pairs = pairs;
  for (int k = 0; k < 9; ++k) r.direction_sums[k] = M[k];
  // step 1: rotations of G_k[i]^-1 and the centres
  std::vector<double> c1(3 * static_cast<size_t>(n)), c2(3 * static_cast<size_t>(n));
  double R1_0[9], R2_0[9], Rtmp[9];
  for (int32_t i = 0; i < n; ++i) {
    image_centre(ctr1, rtg1 + 7 * static_cast<int64_t>(i), i == 0 ? R1_0 : Rtmp, &c1[3 * i]);
    image_centre(ctr2, rtg2 + 7 * static_cast<int64_t>(i), i == 0 ? R2_0 : Rtmp, &c2[3 * i]);
  }
  // step 2: Umeyama's scale. Both sums are left undivided by n; their ratio is the same.
  double m1[3] = {0, 0, 0}, m2[3] = {0, 0, 0};
  for (int32_t i = 0; i < n; ++i)
    for (int k = 0; k < 3; ++k) {
      m1[k] += c1[3 * i + k];
      m2[k] += c2[3 * i + k];
    }
  for (int k = 0; k < 3; ++k) {
    m1[k] /= n;
    m2[k] /= n;
  }
  double S[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, V1[3] = {0, 0, 0};
  for (int32_t i = 0; i < n; ++i) {
    double a[3], b[3];
    for (int k = 0; k < 3; ++k) {
      a[k] = c2[3 * i + k] - m2[k];
      b[k] = c1[3 * i + k] - m1[k];
    }
    for (int row = 0; row < 3; ++row)
      for (int col = 0; col < 3; ++col) S[3 * row + col] += a[row] * b[col];
    for (int k = 0; k < 3; ++k) V1[k] += b[k] * b[k];
  }
  double Rs[9], ls1, ls2;
  horn_rotation(S, Rs, &ls1, &ls2);
  const double s = ls1 / ((V1[0] + V1[1]) + V1[2]);
  r.scale = s;
  // step 4: the intrinsics rotation
  double R[9], l1, l2;
  horn_rotation(M, R, &l1, &l2);
  for (int k = 0; k < 9; ++k) r.intrinsics1_r_intrinsics2[k] = R[k];
  double trRM = 0;
  for (int k = 0; k < 9; ++k) trRM += R[k] * M[k];
  r.rotation_cost = static_cast<double>(pairs) - trRM;
  if (pairs < 2 || !(l1 - l2 > 64 * std::numeric_limits<double>::epsilon() * std::fabs(l1))) {
    *out = b200ba_reconstruction_comparison{};
    out->direction_pairs = pairs;
    for (int k = 0; k < 9; ++k) out->direction_sums[k] = M[k];
    return 4;
  }
  // step 5: T = G1s[0] [R 0; 0 1] G2[0]^-1, G1s[0] = [R1_0^T | s c1[0]], G2[0]^-1 = [R2_0 | -R2_0 c2[0]]
  double A[16] = {0}, B[16] = {0}, C[16] = {0};
  for (int row = 0; row < 3; ++row) {
    for (int col = 0; col < 3; ++col) {
      A[4 * row + col] = R1_0[3 * col + row];
      C[4 * row + col] = R2_0[3 * row + col];
      B[4 * row + col] = R[3 * row + col];
    }
    A[4 * row + 3] = c1[row] * s;
    C[4 * row + 3] = -(R2_0[3 * row] * c2[0] + R2_0[3 * row + 1] * c2[1] + R2_0[3 * row + 2] * c2[2]);
  }
  A[15] = B[15] = C[15] = 1;
  double AB[16];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      double v = 0;
      for (int k = 0; k < 4; ++k) v += A[4 * i + k] * B[4 * k + j];
      AB[4 * i + j] = v;
    }
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      double v = 0;
      for (int k = 0; k < 4; ++k) v += AB[4 * i + k] * C[4 * k + j];
      r.firstimage1_tr_firstimage2[4 * i + j] = v;
    }
  // step 6
  const double* c1b = &c1[3 * (n - 1)];
  const double* c2b = &c2[3 * (n - 1)];
  double d1[3], d2[3], e[3];
  for (int k = 0; k < 3; ++k) {
    d1[k] = c1b[k] - c1[k];
    d2[k] = c2b[k] - c2[k];
  }
  double l1v[3], l2v[3];
  for (int row = 0; row < 3; ++row) {
    l1v[row] = R1_0[3 * row] * d1[0] + R1_0[3 * row + 1] * d1[1] + R1_0[3 * row + 2] * d1[2];
    l2v[row] = R2_0[3 * row] * d2[0] + R2_0[3 * row + 1] * d2[1] + R2_0[3 * row + 2] * d2[2];
  }
  for (int row = 0; row < 3; ++row)
    e[row] = (R[3 * row] * l2v[0] + R[3 * row + 1] * l2v[1] + R[3 * row + 2] * l2v[2]) - s * l1v[row];
  r.endpoint_translation_difference = norm3(e);
  double L1 = 0, L2 = 0;
  for (int32_t i = 0; i + 1 < n; ++i) {
    double a[3], b[3];
    for (int k = 0; k < 3; ++k) {
      a[k] = c1[3 * i + k] * s - c1[3 * (i + 1) + k] * s;
      b[k] = c2[3 * i + k] - c2[3 * (i + 1) + k];
    }
    L1 += norm3(a);
    L2 += norm3(b);
  }
  r.trajectory_length1 = L1;
  r.trajectory_length2 = L2;
  r.relative_endpoint_difference = r.endpoint_translation_difference / (0.5 * (L1 + L2));
  *out = r;
  return 0;
}

int b200ba_reconstruction_alignment(int64_t direction_pairs, const double* direction_sums, int32_t n_images,
                                    const double* rig_tr_global1, const double* camera_tr_rig1,
                                    const double* rig_tr_global2, const double* camera_tr_rig2,
                                    b200ba_reconstruction_comparison* out) {
  if (!direction_sums || !out) {
    g_create_error = "b200ba_reconstruction_alignment: a required argument is NULL";
    return 2;
  }
  if (int rc = alignment_arguments("b200ba_reconstruction_alignment", n_images, rig_tr_global1, camera_tr_rig1,
                                   rig_tr_global2, camera_tr_rig2))
    return rc;
  const int rc = reconstruction_alignment(direction_pairs, direction_sums, n_images, rig_tr_global1, camera_tr_rig1,
                                          rig_tr_global2, camera_tr_rig2, out);
  if (rc == 4) g_create_error = "b200ba_reconstruction_alignment: the intrinsics rotation is not determined";
  return rc;
}

// argument checks of the direction sweep; 0 or 2 (with g_create_error set)
static int sweep_arguments(const std::string& prefix, const b200ba_camera* cam1, const double* intr1,
                           const b200ba_camera* cam2, const double* intr2, int32_t pixel_step) {
  if (!cam1 || !intr1 || !cam2 || !intr2) {
    g_create_error = prefix + "a required argument is NULL";
    return 2;
  }
  for (const b200ba_camera* c : {cam1, cam2}) {
    if (c->model_type != B200BA_MODEL_CENTRAL_GENERIC && c->model_type != B200BA_MODEL_NONCENTRAL_GENERIC &&
        c->model_type != B200BA_MODEL_CENTRAL_OPENCV) {
      g_create_error = prefix + "the comparison is implemented for central-generic, non-central-generic and "
                                "central-OpenCV models";
      return 2;
    }
    if (c->model_type != B200BA_MODEL_CENTRAL_OPENCV && (c->grid_width < 4 || c->grid_height < 4)) {
      g_create_error = prefix + "a grid is smaller than 4 x 4";
      return 2;
    }
  }
  if (cam1->width != cam2->width || cam1->height != cam2->height || cam1->width < 1 || cam1->height < 1) {
    g_create_error = prefix + "the models differ in image size";
    return 2;
  }
  if (pixel_step < 1) {
    g_create_error = prefix + "pixel_step must be at least 1";
    return 2;
  }
  return 0;
}

int b200ba_compare_reconstructions(int device, const b200ba_camera* cam1, const double* intr1,
                                   const b200ba_camera* cam2, const double* intr2, int32_t n_images,
                                   const double* rig_tr_global1, const double* camera_tr_rig1,
                                   const double* rig_tr_global2, const double* camera_tr_rig2, int32_t pixel_step,
                                   b200ba_reconstruction_comparison* out, double* device_ms) {
  const std::string prefix = "b200ba_compare_reconstructions: ";
  if (!out) {
    g_create_error = prefix + "a required argument is NULL";
    return 2;
  }
  if (int rc = sweep_arguments(prefix, cam1, intr1, cam2, intr2, pixel_step)) return rc;
  if (int rc = alignment_arguments("b200ba_compare_reconstructions", n_images, rig_tr_global1, camera_tr_rig1,
                                   rig_tr_global2, camera_tr_rig2))
    return rc;
  CallScope cs(&g_create_error);
  if (int rc = cs.use_device(device)) return rc;
  CamDev c1{}, c2{};
  fill_camdev(*cam1, &c1);
  fill_camdev(*cam2, &c2);
  const int nx = (cam1->width + pixel_step - 1) / pixel_step, ny = (cam1->height + pixel_step - 1) / pixel_step;
  const int64_t n1 = intrinsics_size(*cam1), n2 = intrinsics_size(*cam2);
  double *d1 = nullptr, *d2 = nullptr, *partial = nullptr, *sums = nullptr;
  cs.alloc(&d1, n1);
  cs.alloc(&d2, n2);
  cs.alloc(&partial, sweep_partial_blocks(nx, ny) * kSweepSums);
  cs.alloc(&sums, kSweepSums);
  double h[kSweepSums] = {};
  if (cs.rc == 0) {
    cs.ok(cudaMemcpy(d1, intr1, sizeof(double) * n1, cudaMemcpyHostToDevice));
    cs.ok(cudaMemcpy(d2, intr2, sizeof(double) * n2, cudaMemcpyHostToDevice));
  }
  if (cs.rc == 0) {
    cs.record(0, 0);
    launch_reconstruction_sweep(c1, d1, c2, d2, pixel_step, nx, ny, partial, sums, 0);
    cs.record(1, 0);
    cs.ok(cudaGetLastError());
    cs.ok(cudaMemcpy(h, sums, sizeof(h), cudaMemcpyDeviceToHost));
  }
  if (cs.rc != 0) return cs.rc;
  if (device_ms) *device_ms = cs.elapsed_ms(0, 1);
  const int rc = reconstruction_alignment(static_cast<int64_t>(h[0]), h + 1, n_images, rig_tr_global1, camera_tr_rig1,
                                          rig_tr_global2, camera_tr_rig2, out);
  if (rc == 4) {
    g_create_error = prefix + "the intrinsics rotation is not determined (" + std::to_string(out->direction_pairs) +
                     " sample pixels that both models un-project; rank of sum d1 d2^T below 2)";
  }
  return rc;
}

int b200ba_reconstruction_directions(int device, const b200ba_camera* cam1, const double* intr1,
                                     const b200ba_camera* cam2, const double* intr2, int32_t pixel_step, int32_t* ok,
                                     double* directions) {
  const std::string prefix = "b200ba_reconstruction_directions: ";
  if (!ok || !directions) {
    g_create_error = prefix + "a required argument is NULL";
    return 2;
  }
  if (int rc = sweep_arguments(prefix, cam1, intr1, cam2, intr2, pixel_step)) return rc;
  CallScope cs(&g_create_error);
  if (int rc = cs.use_device(device)) return rc;
  CamDev c1{}, c2{};
  fill_camdev(*cam1, &c1);
  fill_camdev(*cam2, &c2);
  const int nx = (cam1->width + pixel_step - 1) / pixel_step, ny = (cam1->height + pixel_step - 1) / pixel_step;
  const int64_t n = static_cast<int64_t>(nx) * ny, n1 = intrinsics_size(*cam1), n2 = intrinsics_size(*cam2);
  double *d1 = nullptr, *d2 = nullptr, *ddirs = nullptr;
  int32_t* dok = nullptr;
  cs.alloc(&d1, n1);
  cs.alloc(&d2, n2);
  cs.alloc(&ddirs, 6 * n);
  cs.alloc(&dok, 2 * n);
  if (cs.rc == 0) {
    cs.ok(cudaMemcpy(d1, intr1, sizeof(double) * n1, cudaMemcpyHostToDevice));
    cs.ok(cudaMemcpy(d2, intr2, sizeof(double) * n2, cudaMemcpyHostToDevice));
  }
  if (cs.rc == 0) {
    launch_reconstruction_directions(c1, d1, c2, d2, pixel_step, nx, ny, dok, ddirs, 0);
    cs.ok(cudaGetLastError());
    cs.ok(cudaMemcpy(ok, dok, sizeof(int32_t) * 2 * n, cudaMemcpyDeviceToHost));
    cs.ok(cudaMemcpy(directions, ddirs, sizeof(double) * 6 * n, cudaMemcpyDeviceToHost));
  }
  return cs.rc;
}

// Stand-alone Voronoi coverage rendering (allocates, computes, frees): what b200ba_report_images renders its
// error maps with.
int b200ba_render_voronoi(int device, int32_t width, int32_t height, int64_t n_sites, const int32_t* sites_q,
                          const float* colors, uint8_t* image, double* device_ms) {
  constexpr int64_t kMaxCoord = int64_t(1) << 28;
  if (width < 1 || height < 1 || width > (1 << 24) || height > (1 << 24) || n_sites < 0 || n_sites > (int64_t(1) << 30) ||
      !image || (n_sites > 0 && (!sites_q || !colors))) {
    g_create_error = "b200ba_render_voronoi: bad argument";
    return 2;
  }
  int64_t lo_x = 0, lo_y = 0, hi_x = 4 * static_cast<int64_t>(width), hi_y = 4 * static_cast<int64_t>(height);
  for (int64_t i = 0; i < n_sites; ++i) {
    const int64_t x = sites_q[2 * i], y = sites_q[2 * i + 1];
    if (x < -kMaxCoord || x > kMaxCoord || y < -kMaxCoord || y > kMaxCoord) {
      g_create_error = "b200ba_render_voronoi: a site lies outside [-2^28, 2^28] quarter pixels";
      return 2;
    }
    lo_x = std::min(lo_x, x);
    lo_y = std::min(lo_y, y);
    hi_x = std::max(hi_x, x);
    hi_y = std::max(hi_y, y);
  }
  CallScope cs(&g_create_error);
  if (int rc = cs.use_device(device)) return rc;
  const int64_t pixels = static_cast<int64_t>(width) * height;
  const size_t nn = static_cast<size_t>(std::max<int64_t>(1, n_sites));
  int2* d_sites = nullptr;
  float* d_colors = nullptr;
  uint8_t* d_img = nullptr;
  VoronoiRun vr;
  cs.alloc(&d_sites, nn);
  cs.alloc(&d_colors, 3 * nn);
  cs.alloc(&d_img, 3 * pixels);
  if (cs.rc == 0) vr.alloc(cs, n_sites, lo_x, lo_y, hi_x, hi_y);
  if (cs.rc == 0 && n_sites > 0) {
    cs.ok(cudaMemcpy(d_sites, sites_q, sizeof(int2) * n_sites, cudaMemcpyHostToDevice));
    cs.ok(cudaMemcpy(d_colors, colors, sizeof(float) * 3 * n_sites, cudaMemcpyHostToDevice));
  }
  if (cs.rc == 0) {
    cs.record(0, 0);
    launch_render_voronoi(width, height, n_sites, d_sites, d_colors, 3, vr.g, d_img, nullptr, 0);
    cs.record(1, 0);
    cs.ok(cudaGetLastError());
    cs.ok(cudaMemcpy(image, d_img, 3 * pixels, cudaMemcpyDeviceToHost));
  }
  if (cs.rc == 0 && device_ms) *device_ms = cs.elapsed_ms(0, 1);
  return cs.rc;
}

// Stand-alone VisualizeCameraModel of a libvis RadtanCamera8d (APP/tools/visualize_calibration.cc:39-96): the
// orientation and the image on the device. The argument checks come first and touch no CUDA state.
int b200ba_visualize_camera(int device, int32_t width, int32_t height, const double* params, uint8_t* image,
                            double* rotation, double* directions, double* device_ms) {
  if (!params || !image) {
    g_create_error = "b200ba_visualize_camera: params and image are required";
    return 2;
  }
  if (width < 1 || height < 1 || width > (1 << 24) || height > (1 << 24) ||
      static_cast<int64_t>(width) * height > (int64_t(1) << 31)) {
    g_create_error = "b200ba_visualize_camera: width and height must be >= 1 and the image at most 2^31 pixels";
    return 2;
  }
  for (int k = 0; k < 8; ++k)
    if (!std::isfinite(params[k])) {
      g_create_error = "b200ba_visualize_camera: a parameter is not finite";
      return 2;
    }
  if (params[4] == 0 || params[5] == 0) {
    g_create_error = "b200ba_visualize_camera: fx and fy must not be 0";
    return 2;
  }
  CallScope cs(&g_create_error);
  if (int rc = cs.use_device(device)) return rc;
  const int64_t pixels = static_cast<int64_t>(width) * height;
  double* d_params = nullptr;
  double2* d_win = nullptr;
  double* d_rot = nullptr;
  uint8_t* d_img = nullptr;
  double* d_dirs = nullptr;
  cs.alloc(&d_params, 8);
  cs.alloc(&d_win, static_cast<size_t>(21) * width);  // the orientation window: at most 21 rows of at most width pixels
  cs.alloc(&d_rot, 9);
  cs.alloc(&d_img, 3 * pixels);
  if (directions) cs.alloc(&d_dirs, 3 * pixels);
  if (cs.rc == 0) cs.ok(cudaMemcpy(d_params, params, sizeof(double) * 8, cudaMemcpyHostToDevice));
  if (cs.rc == 0) {
    cs.record(0, 0);
    launch_visualize_orientation(d_params, width, height, d_win, d_rot, 0);
    launch_visualize_camera(d_params, width, height, d_rot, d_img, d_dirs, 0);
    cs.record(1, 0);
    cs.ok(cudaGetLastError());
    cs.ok(cudaMemcpy(image, d_img, 3 * pixels, cudaMemcpyDeviceToHost));
    if (rotation) cs.ok(cudaMemcpy(rotation, d_rot, sizeof(double) * 9, cudaMemcpyDeviceToHost));
    if (directions) cs.ok(cudaMemcpy(directions, d_dirs, sizeof(double) * 3 * pixels, cudaMemcpyDeviceToHost));
  }
  if (cs.rc == 0 && device_ms) *device_ms = cs.elapsed_ms(0, 1);
  return cs.rc;
}

// Stand-alone feature intersection of --intersect_datasets (APP/tools/intersect_datasets.cc:130-225): the walk and
// the final pass of every list on the device. The argument checks come first and touch no CUDA state.
int b200ba_intersect_features(int device, int32_t n_datasets, int64_t n_lists, const int64_t* list_offsets,
                              const float* xy, double threshold, uint8_t* keep, b200ba_intersection_report* report,
                              double* device_ms) {
  if (n_datasets < 1 || n_datasets > 32 || n_lists < 0 || n_lists >= (int64_t(1) << 31) || !list_offsets) {
    g_create_error = "b200ba_intersect_features: needs 1 <= n_datasets <= 32, 0 <= n_lists < 2^31 and list_offsets";
    return 2;
  }
  const int64_t n_off = n_lists * n_datasets;
  if (list_offsets[0] != 0) {
    g_create_error = "b200ba_intersect_features: list_offsets must start at 0";
    return 2;
  }
  int64_t max_list = 0;
  for (int64_t k = 0; k < n_off; ++k)
    if (list_offsets[k + 1] < list_offsets[k]) {
      g_create_error = "b200ba_intersect_features: list_offsets must not decrease";
      return 2;
    }
  for (int64_t l = 0; l < n_lists; ++l)
    max_list = std::max(max_list, list_offsets[(l + 1) * n_datasets] - list_offsets[l * n_datasets]);
  if (max_list >= (int64_t(1) << 31)) {
    g_create_error = "b200ba_intersect_features: a list holds 2^31 features or more";
    return 2;
  }
  const int64_t n = list_offsets[n_off];
  if (n > 0 && (!xy || !keep)) {
    g_create_error = "b200ba_intersect_features: xy and keep are required";
    return 2;
  }
  const double thr2 = threshold * threshold;
  float bound = static_cast<float>(thr2);  // the largest float <= thr2, so that float d <= bound iff (double)d <= thr2
  if (static_cast<double>(bound) > thr2) bound = std::nextafter(bound, -std::numeric_limits<float>::infinity());
  CallScope cs(&g_create_error);
  if (int rc = cs.use_device(device)) return rc;
  unsigned long long counts[2] = {0, 0};
  int64_t intersections = 0, kept = 0;
  if (n > 0) {
    int64_t* d_off = nullptr;
    float2* d_xy = nullptr;
    uint8_t* d_keep = nullptr;
    float2* d_cent = nullptr;
    int* d_nc = nullptr;
    unsigned long long* d_counts = nullptr;
    cs.alloc(&d_off, n_off + 1);
    cs.alloc(&d_xy, n);
    cs.alloc(&d_keep, n);
    cs.alloc(&d_cent, n);
    cs.alloc(&d_nc, n_lists);
    cs.alloc(&d_counts, 2);
    if (cs.rc == 0) cs.ok(cudaMemcpy(d_off, list_offsets, sizeof(int64_t) * (n_off + 1), cudaMemcpyHostToDevice));
    if (cs.rc == 0) cs.ok(cudaMemcpy(d_xy, xy, sizeof(float2) * n, cudaMemcpyHostToDevice));
    if (cs.rc == 0) cs.ok(cudaMemset(d_keep, 1, n));
    if (cs.rc == 0) cs.ok(cudaMemset(d_counts, 0, sizeof(counts)));
    if (cs.rc == 0) {
      cs.record(0, 0);
      launch_intersect_features(n_datasets, n_lists, max_list, d_off, d_xy, bound, d_keep, d_cent, d_nc, d_counts, 0);
      cs.record(1, 0);
      cs.ok(cudaGetLastError());
      cs.ok(cudaMemcpy(keep, d_keep, n, cudaMemcpyDeviceToHost));
      cs.ok(cudaMemcpy(counts, d_counts, sizeof(counts), cudaMemcpyDeviceToHost));
      std::vector<int> nc(n_lists);
      cs.ok(cudaMemcpy(nc.data(), d_nc, sizeof(int) * n_lists, cudaMemcpyDeviceToHost));
      for (int v : nc) intersections += v;
      for (int64_t k = 0; k < n; ++k) kept += keep[k];
    }
  }
  if (cs.rc == 0 && report) {
    report->intersections = intersections;
    report->kept = kept;
    report->uncovered = static_cast<int64_t>(counts[0]);
    report->capped = static_cast<int64_t>(counts[1]);
  }
  if (cs.rc == 0 && device_ms) *device_ms = n > 0 ? cs.elapsed_ms(0, 1) : 0.0;
  return cs.rc;
}

// ---- synthetic pattern images (--render_synthetic_dataset; the arithmetic is specified in include/b200ba.h) ----
namespace {
bool synth_valid_pattern_coord(const b200ba_pattern& p, float x, float y) {  // PatternData::IsValidPatternCoord
  if (!(x >= -1.f && y >= -1.f && x <= p.squares_x - 1.f && y <= p.squares_y - 1.f)) return false;
  for (int k = 0; k < p.num_tags; ++k) {
    const b200ba_pattern_tag& t = p.tags[k];
    if (x >= t.x - 1 && y >= t.y - 1 && x <= t.x - 1 + t.width && y <= t.y - 1 + t.height) return false;
  }
  return true;
}

// PatternData::GetStarCoord with square_length 1: float angle and float sin / cos, the offset in double
float2 synth_star_coord(int num_star_segments, float i, float center_x, float center_y) {
  const float angle = ((2 * M_PI) * i) / num_star_segments;
  float x = std::sin(angle), y = std::cos(angle);
  const float max_abs_x = std::max(std::fabs(x), std::fabs(y));
  x /= max_abs_x;
  y /= max_abs_x;
  return make_float2(static_cast<float>(center_x - 0.5 * x), static_cast<float>(center_y - 0.5 * y));
}

// pattern_to_pattern_image_coord of render_synthetic_dataset.cc:79-87, in float
float2 synth_pattern_to_image(const b200ba_pattern& p, int32_t pattern_w, int32_t pattern_h, float cx, float cy) {
  const float mx = p.pattern_start_x_mm + ((cx + 1.f) / static_cast<float>(p.squares_x)) *
                                              (p.pattern_end_x_mm - p.pattern_start_x_mm);
  const float my = p.pattern_start_y_mm + ((cy + 1.f) / static_cast<float>(p.squares_y)) *
                                              (p.pattern_end_y_mm - p.pattern_start_y_mm);
  return make_float2((static_cast<float>(pattern_w) / p.page_width_mm) * mx,
                     (static_cast<float>(pattern_h) / p.page_height_mm) * my);
}

// PatternData::ComputePatternGeometry (without AprilTags) in generation order, mapped to pattern-image pixels
void synth_geometry(const b200ba_pattern& p, int32_t pattern_w, int32_t pattern_h, std::vector<float2>* verts,
                    std::vector<int8_t>* nv) {
  const int n = p.num_star_segments;
  for (int y = -1; y < p.squares_y; ++y) {
    for (int x = -1; x < p.squares_x; ++x) {
      bool in_tag = false;
      for (int k = 0; k < p.num_tags && !in_tag; ++k) {
        const b200ba_pattern_tag& t = p.tags[k];
        in_tag = x >= t.x && y >= t.y && x <= t.x - 2 + t.width && y <= t.y - 2 + t.height;
      }
      if (in_tag) continue;
      for (int segment = 0; segment < n; segment += 2) {
        const float2 middle = synth_star_coord(n, segment + 0.5f, x, y);
        if (!synth_valid_pattern_coord(p, middle.x, middle.y)) continue;
        float2 poly[kSynthMaxVerts];
        int c = 0;
        poly[c++] = make_float2(x, y);
        poly[c++] = synth_star_coord(n, segment, x, y);
        const float angle1 = (2 * M_PI) * (segment) / n;
        const float angle2 = (2 * M_PI) * (segment + 1) / n;
        if (std::floor((angle1 - M_PI / 4) / (M_PI / 2)) != std::floor((angle2 - M_PI / 4) / (M_PI / 2))) {
          const float corner_angle = (M_PI / 4) + (M_PI / 2) * std::floor((angle2 - M_PI / 4) / (M_PI / 2));
          float corner_x = std::sin(corner_angle), corner_y = std::cos(corner_angle);
          const float normalizer = std::fabs(corner_x);
          corner_x /= normalizer;
          corner_y /= normalizer;
          poly[c++] = make_float2(static_cast<float>(x - 0.5 * corner_x), static_cast<float>(y - 0.5 * corner_y));
        }
        poly[c++] = synth_star_coord(n, segment + 1, x, y);
        for (int v = 0; v < kSynthMaxVerts; ++v)
          verts->push_back(v < c ? synth_pattern_to_image(p, pattern_w, pattern_h, poly[v].x, poly[v].y)
                                 : make_float2(0.f, 0.f));
        nv->push_back(static_cast<int8_t>(c));
      }
    }
  }
}

// Eigen's Quaternion::toRotationMatrix, row-major
void synth_rotation(double w, double x, double y, double z, double* R) {
  const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
  const double twx = tx * w, twy = ty * w, twz = tz * w;
  const double txx = tx * x, txy = ty * x, txz = tz * x;
  const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
  R[0] = 1 - (tyy + tzz), R[1] = txy - twz, R[2] = txz + twy;
  R[3] = txy + twz, R[4] = 1 - (txx + tzz), R[5] = tyz - twx;
  R[6] = txz - twy, R[7] = tyz + twx, R[8] = 1 - (txx + tyy);
}

void synth_cross(const double* a, const double* b, double* r) {
  r[0] = a[1] * b[2] - a[2] * b[1];
  r[1] = a[2] * b[0] - a[0] * b[2];
  r[2] = a[0] * b[1] - a[1] * b[0];
}

// attempt a of image i: exp(tangent) * (I, t0) as Sophus composes it; pose = [R row-major, t]
void synth_pose_attempt(uint64_t seed_hash, int64_t i, int a, int32_t pattern_w, int32_t pattern_h, double* pose) {
  uint64_t h[9];
  for (int c = 0; c < 9; ++c)
    h[c] = loc_splitmix64(seed_hash ^ ((static_cast<uint64_t>(i) << 24) | (static_cast<uint64_t>(a) << 4) | c));
  float f[3];
  for (int c = 0; c < 3; ++c) f[c] = static_cast<float>(h[c] % 10000) / 10000.f;
  const double t0[3] = {0.0 - static_cast<double>((-1.f + 2.f * f[0]) * static_cast<float>(pattern_w)),
                        0.0 - static_cast<double>((-1.f + 2.f * f[1]) * static_cast<float>(pattern_h)),
                        0.0 + static_cast<double>(500.f + 800.f * f[2])};
  double tan[6];
  for (int c = 0; c < 6; ++c) tan[c] = 0.5 * (-1.0 + 2.0 * (static_cast<double>(h[3 + c] >> 11) * 0x1p-53));
  const double* u = tan;
  const double* w = tan + 3;
  const double th2 = (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2];
  const double th = std::sqrt(th2);
  const double half = 0.5 * th;
  double im, re;
  if (th < 1e-10) {
    const double th4 = th2 * th2;
    im = (0.5 - (1.0 / 48.0) * th2) + (1.0 / 3840.0) * th4;
    re = (1.0 - 0.5 * th2) + (1.0 / 384.0) * th4;
  } else {
    im = std::sin(half) / th;
    re = std::cos(half);
  }
  const double qv[3] = {im * w[0], im * w[1], im * w[2]};
  const double qw = re;
  double V[9];
  if (th < 1e-10) {
    synth_rotation(qw, qv[0], qv[1], qv[2], V);
  } else {
    const double W[9] = {0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0};
    double W2[9];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) W2[r * 3 + c] = (W[r * 3] * W[c] + W[r * 3 + 1] * W[3 + c]) + W[r * 3 + 2] * W[6 + c];
    const double c1 = (1.0 - std::cos(th)) / th2, c2 = (th - std::sin(th)) / (th2 * th);
    for (int k = 0; k < 9; ++k) V[k] = ((k % 4 == 0 ? 1.0 : 0.0) + c1 * W[k]) + c2 * W2[k];
  }
  double t[3];
  for (int r = 0; r < 3; ++r) t[r] = (V[r * 3] * u[0] + V[r * 3 + 1] * u[1]) + V[r * 3 + 2] * u[2];
  double uv[3], uv2[3];
  synth_cross(qv, t0, uv);
  for (double& e : uv) e = e + e;
  synth_cross(qv, uv, uv2);
  for (int r = 0; r < 3; ++r) t[r] = t[r] + ((t0[r] + qw * uv[r]) + uv2[r]);
  double q[4] = {qv[0], qv[1], qv[2], qw};  // Eigen's coefficient order x, y, z, w
  const double s = (q[0] * q[0] + q[2] * q[2]) + (q[1] * q[1] + q[3] * q[3]);
  if (s != 1.0)
    for (double& e : q) e *= 2.0 / (1.0 + s);
  synth_rotation(q[3], q[0], q[1], q[2], pose);
  for (int r = 0; r < 3; ++r) pose[9 + r] = t[r];
}

// PinholeCamera4f::ProjectToPixelCornerConvIfVisible(p, 0) of the float pose
bool synth_visible(const float* Rf, const float* tf, const float* k, int32_t width, int32_t height, float x, float y) {
  float p[3];
  for (int r = 0; r < 3; ++r) p[r] = (((Rf[r * 3] * x) + (Rf[r * 3 + 1] * y)) + (Rf[r * 3 + 2] * 0.f)) + tf[r];
  if (p[2] <= 0.f) return false;
  const float u = k[0] * (p[0] / p[2]) + k[2], v = k[1] * (p[1] / p[2]) + k[3];
  return u >= 0.f && v >= 0.f && u < static_cast<float>(width) - 0.f && v < static_cast<float>(height) - 0.f;
}

// the float pose (Rf, tf) and the float inverse (Rc, tc) of one double pose
void synth_float_pose(const double* pose, float* out) {
  const double* R = pose;
  const double* t = pose + 9;
  for (int k = 0; k < 12; ++k) out[k] = static_cast<float>(pose[k]);
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) out[12 + r * 3 + c] = static_cast<float>(R[c * 3 + r]);
  for (int r = 0; r < 3; ++r) out[21 + r] = static_cast<float>((R[r] * -t[0] + R[3 + r] * -t[1]) + R[6 + r] * -t[2]);
}

// the checks of a pattern struct that b200ba_render_pattern_images and b200ba_refine_features share
const char* check_pattern_struct(const b200ba_pattern* p) {
  if (p->num_tags < 0 || p->num_tags > B200BA_PATTERN_MAX_TAGS) return "num_tags must lie in [0, B200BA_PATTERN_MAX_TAGS]";
  if (p->squares_x < 1 || p->squares_y < 1) return "squares_x and squares_y must be at least 1";
  if (p->num_star_segments < 2 || p->num_star_segments % 2 || p->num_star_segments > 1024)
    return "num_star_segments must be even and in [2, 1024]";
  if (int64_t(p->squares_x + 1) * (p->squares_y + 1) * (p->num_star_segments / 2) > (int64_t(1) << 24))
    return "the pattern has more than 2^24 star segments";
  return nullptr;
}

const char* synth_check_pattern(const b200ba_pattern* p, int32_t pattern_w, int32_t pattern_h, int32_t width,
                                int32_t height, const float* k) {
  if (!p || !k) return "pattern and fx_fy_cx_cy are required";
  if (pattern_w < 1 || pattern_h < 1 || width < 1 || height < 1 || pattern_w > 32768 || pattern_h > 32768 ||
      width > 32768 || height > 32768)
    return "sizes must lie in [1, 32768]";
  if (const char* e = check_pattern_struct(p)) return e;
  if (!std::isfinite(k[0]) || !std::isfinite(k[1]) || k[0] == 0.f || k[1] == 0.f || !std::isfinite(k[2]) ||
      !std::isfinite(k[3]))
    return "fx and fy must be finite and non-zero, cx and cy finite";
  return nullptr;
}
}  // namespace

int b200ba_synthetic_poses(const b200ba_pattern* pattern, int32_t pattern_w, int32_t pattern_h, int32_t width,
                           int32_t height, const float* fx_fy_cx_cy, int64_t n, uint64_t seed,
                           double* camera_tr_global, int64_t* attempts) {
  if (const char* e = synth_check_pattern(pattern, pattern_w, pattern_h, width, height, fx_fy_cx_cy)) {
    g_create_error = std::string("b200ba_synthetic_poses: ") + e;
    return 2;
  }
  if (n < 1 || n >= (int64_t(1) << 40) || !camera_tr_global) {
    g_create_error = "b200ba_synthetic_poses: needs 1 <= n < 2^40 and camera_tr_global";
    return 2;
  }
  const b200ba_pattern& p = *pattern;
  std::vector<float2> lo(p.num_tags), hi(p.num_tags);
  for (int k = 0; k < p.num_tags; ++k) {
    const b200ba_pattern_tag& t = p.tags[k];
    lo[k] = synth_pattern_to_image(p, pattern_w, pattern_h, t.x - 1, t.y - 1);
    hi[k] = synth_pattern_to_image(p, pattern_w, pattern_h, t.x - 1 + t.width, t.y - 1 + t.height);
  }
  const uint64_t seed_hash = loc_splitmix64(seed);
  for (int64_t i = 0; i < n; ++i) {
    double* pose = camera_tr_global + 12 * i;
    bool visible = false;
    int a = 0;
    for (; a < 4096 && !visible; ++a) {
      synth_pose_attempt(seed_hash, i, a, pattern_w, pattern_h, pose);
      float f[24];
      synth_float_pose(pose, f);
      for (int k = 0; k < p.num_tags && !visible; ++k)
        visible = synth_visible(f, f + 9, fx_fy_cx_cy, width, height, lo[k].x, lo[k].y) &&
                  synth_visible(f, f + 9, fx_fy_cx_cy, width, height, hi[k].x, lo[k].y) &&
                  synth_visible(f, f + 9, fx_fy_cx_cy, width, height, lo[k].x, hi[k].y) &&
                  synth_visible(f, f + 9, fx_fy_cx_cy, width, height, hi[k].x, hi[k].y);
    }
    if (attempts) attempts[i] = a;
    if (!visible) {
      g_create_error = "b200ba_synthetic_poses: no tag is visible after 4096 attempts";
      return 4;
    }
  }
  return 0;
}

int b200ba_render_pattern_images(int device, const b200ba_pattern* pattern, const uint8_t* pattern_image,
                                 int32_t pattern_w, int32_t pattern_h, int32_t width, int32_t height,
                                 const float* fx_fy_cx_cy, int64_t n, const double* camera_tr_global, uint8_t* images,
                                 double* device_ms) {
  if (const char* e = synth_check_pattern(pattern, pattern_w, pattern_h, width, height, fx_fy_cx_cy)) {
    g_create_error = std::string("b200ba_render_pattern_images: ") + e;
    return 2;
  }
  if (n < 0 || !pattern_image || (n > 0 && (!camera_tr_global || !images))) {
    g_create_error = "b200ba_render_pattern_images: needs n >= 0, pattern_image, camera_tr_global and images";
    return 2;
  }
  const b200ba_pattern& pat = *pattern;
  std::vector<float2> verts;
  std::vector<int8_t> nv;
  synth_geometry(pat, pattern_w, pattern_h, &verts, &nv);
  SynthParams sp{};
  sp.w = width;
  sp.h = height;
  sp.tiles_x = (width + kSynthTile - 1) / kSynthTile;
  sp.tiles_y = (height + kSynthTile - 1) / kSynthTile;
  sp.n_poly = static_cast<int>(nv.size());
  sp.words = std::max(1, (sp.n_poly + 31) / 32);
  sp.fx = fx_fy_cx_cy[0], sp.fy = fx_fy_cx_cy[1], sp.cx = fx_fy_cx_cy[2], sp.cy = fx_fy_cx_cy[3];
  sp.pattern_w = pattern_w, sp.pattern_h = pattern_h, sp.squares_x = pat.squares_x, sp.squares_y = pat.squares_y;
  sp.num_tags = pat.num_tags;
  sp.page_w = pat.page_width_mm, sp.page_h = pat.page_height_mm;
  sp.start_x = pat.pattern_start_x_mm, sp.start_y = pat.pattern_start_y_mm;
  sp.end_x = pat.pattern_end_x_mm, sp.end_y = pat.pattern_end_y_mm;
  for (int k = 0; k < pat.num_tags; ++k)
    sp.tags[k] = make_int4(pat.tags[k].x, pat.tags[k].y, pat.tags[k].width, pat.tags[k].height);
  // images per chunk: device memory bounded by about 512 MiB (B200BA_SYNTH_CHUNK caps the count)
  const int64_t pixels = static_cast<int64_t>(width) * height;
  const int64_t per_image = static_cast<int64_t>(sp.tiles_x) * sp.tiles_y * sp.words * 4 +
                            static_cast<int64_t>(sp.n_poly) * (kSynthMaxVerts * 16 + 16) + pixels + 96;
  int64_t chunk = std::max<int64_t>(1, (int64_t(512) << 20) / per_image);
  if (const char* e = getenv("B200BA_SYNTH_CHUNK")) chunk = std::max<int64_t>(1, std::min<int64_t>(chunk, atoll(e)));
  chunk = std::min<int64_t>(chunk, std::max<int64_t>(n, 1));
  chunk = std::min<int64_t>(chunk, 65535);
  CallScope cs(&g_create_error);
  if (int rc = cs.use_device(device)) return rc;
  if (n == 0) {
    if (device_ms) *device_ms = 0.0;
    return 0;
  }
  std::vector<float> poses(24 * n);
  for (int64_t i = 0; i < n; ++i) synth_float_pose(camera_tr_global + 12 * i, poses.data() + 24 * i);
  float2* d_verts = nullptr;
  int8_t* d_nv = nullptr;
  float* d_poses = nullptr;
  uint8_t* d_pattern = nullptr;
  double2* d_proj = nullptr;
  int4* d_range = nullptr;
  uint32_t* d_bits = nullptr;
  uint8_t* d_img = nullptr;
  const size_t bits_per_image = static_cast<size_t>(sp.tiles_x) * sp.tiles_y * sp.words;
  cs.alloc(&d_verts, std::max<size_t>(1, verts.size()));
  cs.alloc(&d_nv, std::max<size_t>(1, nv.size()));
  cs.alloc(&d_poses, poses.size());
  cs.alloc(&d_pattern, static_cast<size_t>(pattern_w) * pattern_h);
  cs.alloc(&d_proj, std::max<size_t>(1, static_cast<size_t>(chunk) * sp.n_poly * kSynthMaxVerts));
  cs.alloc(&d_range, std::max<size_t>(1, static_cast<size_t>(chunk) * sp.n_poly));
  cs.alloc(&d_bits, static_cast<size_t>(chunk) * bits_per_image);
  cs.alloc(&d_img, static_cast<size_t>(chunk) * pixels);
  if (cs.rc == 0 && !verts.empty())
    cs.ok(cudaMemcpy(d_verts, verts.data(), sizeof(float2) * verts.size(), cudaMemcpyHostToDevice));
  if (cs.rc == 0 && !nv.empty()) cs.ok(cudaMemcpy(d_nv, nv.data(), nv.size(), cudaMemcpyHostToDevice));
  if (cs.rc == 0) cs.ok(cudaMemcpy(d_poses, poses.data(), sizeof(float) * poses.size(), cudaMemcpyHostToDevice));
  if (cs.rc == 0)
    cs.ok(cudaMemcpy(d_pattern, pattern_image, static_cast<size_t>(pattern_w) * pattern_h, cudaMemcpyHostToDevice));
  double ms = 0.0;
  for (int64_t i0 = 0; i0 < n && cs.rc == 0; i0 += chunk) {
    const int m = static_cast<int>(std::min<int64_t>(chunk, n - i0));
    cs.record(0, 0);
    cs.ok(cudaMemsetAsync(d_bits, 0, sizeof(uint32_t) * bits_per_image * m, 0));
    launch_render_pattern(sp, m, d_verts, d_nv, d_poses + 24 * i0, d_pattern, d_proj, d_range, d_bits, d_img, 0);
    cs.record(1, 0);
    cs.ok(cudaGetLastError());
    cs.ok(cudaMemcpy(images + i0 * pixels, d_img, static_cast<size_t>(m) * pixels, cudaMemcpyDeviceToHost));
    if (cs.rc == 0) ms += cs.elapsed_ms(0, 1);
  }
  if (cs.rc == 0 && device_ms) *device_ms = ms;
  return cs.rc;
}

// ---- feature refinement (RefineFeatureDetections; the arithmetic is specified in include/b200ba.h) ----
namespace {
int refine_sample_count(int32_t h) { return static_cast<int>(8.0 * (2 * h + 1) * (2 * h + 1) + 0.5); }
}  // namespace

int b200ba_feature_samples(int32_t window_half_extent, int32_t n, float* xy) {
  if (window_half_extent < 1 || window_half_extent > B200BA_REFINE_MAX_HALF_EXTENT || !xy ||
      n != refine_sample_count(window_half_extent)) {
    g_create_error = "b200ba_feature_samples: needs 1 <= window_half_extent <= 32, n = (int)(8 (2h + 1)^2 + 0.5) "
                     "and xy";
    return 2;
  }
  // glibc's random_r, TYPE_3: srandom(1) (srand(0) seeds as 1), then 310 values discarded
  int32_t r[31];
  r[0] = 1;
  for (int i = 1; i < 31; ++i) {
    const int32_t hi = r[i - 1] / 127773, lo = r[i - 1] % 127773;
    int32_t word = 16807 * lo - 2836 * hi;
    if (word < 0) word += 2147483647;
    r[i] = word;
  }
  int f = 3, b = 0;
  auto next = [&]() {
    r[f] = static_cast<int32_t>(static_cast<uint32_t>(r[f]) + static_cast<uint32_t>(r[b]));
    const int32_t v = static_cast<int32_t>(static_cast<uint32_t>(r[f]) >> 1);
    f = (f + 1) % 31;
    b = (b + 1) % 31;
    return v;
  };
  for (int i = 0; i < 310; ++i) next();
  for (int64_t i = 0; i < 2 * static_cast<int64_t>(n); ++i)
    xy[i] = -1.f + (2.f * static_cast<float>(next())) / static_cast<float>(2147483647);
  return 0;
}

int b200ba_refine_features(int device, const b200ba_pattern* pattern, const uint8_t* images, int32_t width,
                           int32_t height, int64_t n_images, const float* samples, int32_t n_samples,
                           int32_t window_half_extent, int32_t refinement_type, int64_t n_features,
                           const b200ba_feature_prediction* predictions, float* xy, float* final_cost,
                           int32_t* status, double* device_ms) {
  const char* e = nullptr;
  if (!pattern || !samples || (n_features > 0 && (!images || !predictions || !xy || !final_cost)))
    e = "pattern, samples, and for n_features > 0 images, predictions, xy and final_cost are required";
  else if (width < 1 || height < 1 || width > 32768 || height > 32768)
    e = "width and height must lie in [1, 32768]";
  else if (n_images < 0 || n_features < 0)
    e = "n_images and n_features must not be negative";
  else if (window_half_extent < 1 || window_half_extent > B200BA_REFINE_MAX_HALF_EXTENT)
    e = "window_half_extent must lie in [1, B200BA_REFINE_MAX_HALF_EXTENT]";
  else if (n_samples != refine_sample_count(window_half_extent))
    e = "n_samples must be (int)(8 (2 window_half_extent + 1)^2 + 0.5)";
  else if (refinement_type < B200BA_REFINE_GRADIENTS_XY || refinement_type > B200BA_REFINE_NO_REFINEMENT)
    e = "unknown refinement_type";
  else
    e = check_pattern_struct(pattern);
  for (int64_t i = 0; !e && i < n_features; ++i) {
    const b200ba_feature_prediction& q = predictions[i];
    if (q.image < 0 || q.image >= n_images) e = "a prediction's image index lies outside [0, n_images)";
    for (int k = 0; !e && k < 9; ++k)
      if (!std::isfinite(q.local_pixel_tr_pattern[k])) e = "a prediction's local_pixel_tr_pattern is not finite";
  }
  if (e) {
    g_create_error = std::string("b200ba_refine_features: ") + e;
    return 2;
  }
  RefineParams rp{};
  rp.w = width, rp.h = height, rp.half = window_half_extent;
  rp.n_samples = n_samples;
  rp.n_match = static_cast<int>((1 / 8.) * n_samples);
  rp.type = refinement_type;
  rp.num_star_segments = pattern->num_star_segments;
  rp.squares_x = pattern->squares_x, rp.squares_y = pattern->squares_y, rp.num_tags = pattern->num_tags;
  for (int k = 0; k < pattern->num_tags; ++k)
    rp.tags[k] = make_int4(pattern->tags[k].x, pattern->tags[k].y, pattern->tags[k].width, pattern->tags[k].height);
  // images per chunk: device memory bounded by about 512 MiB (B200BA_REFINE_CHUNK caps the count)
  const int64_t pixels = static_cast<int64_t>(width) * height;
  int64_t chunk = std::max<int64_t>(1, (int64_t(512) << 20) / pixels);
  if (const char* env = getenv("B200BA_REFINE_CHUNK")) chunk = std::max<int64_t>(1, std::min<int64_t>(chunk, atoll(env)));
  chunk = std::min<int64_t>(chunk, std::max<int64_t>(n_images, 1));
  CallScope cs(&g_create_error);
  if (int rc = cs.use_device(device)) return rc;
  if (n_features == 0) {
    if (device_ms) *device_ms = 0.0;
    return 0;
  }
  // the features in image order (stable), so that each chunk's features are contiguous
  std::vector<int64_t> order(n_features);
  for (int64_t i = 0; i < n_features; ++i) order[i] = i;
  std::stable_sort(order.begin(), order.end(),
                   [&](int64_t a, int64_t b) { return predictions[a].image < predictions[b].image; });
  // features per launch: at most kMaxLaunch (80 B of device memory each), so any number of features works
  constexpr int64_t kMaxLaunch = int64_t(1) << 20;
  int64_t max_per_chunk = 0;
  for (int64_t lo = 0, i0 = 0; i0 < n_images; i0 += chunk) {
    int64_t hi = lo;
    while (hi < n_features && predictions[order[hi]].image < i0 + chunk) ++hi;
    max_per_chunk = std::max(max_per_chunk, std::min(hi - lo, kMaxLaunch));
    lo = hi;
  }
  uint8_t* d_img = nullptr;
  float2* d_samples = nullptr;
  b200ba_feature_prediction* d_pred = nullptr;
  float2* d_xy = nullptr;
  float* d_cost = nullptr;
  int* d_status = nullptr;
  cs.alloc(&d_img, static_cast<size_t>(chunk) * pixels);
  cs.alloc(&d_samples, static_cast<size_t>(n_samples));
  cs.alloc(&d_pred, static_cast<size_t>(max_per_chunk));
  cs.alloc(&d_xy, static_cast<size_t>(max_per_chunk));
  cs.alloc(&d_cost, static_cast<size_t>(max_per_chunk));
  cs.alloc(&d_status, static_cast<size_t>(max_per_chunk));
  if (cs.rc == 0) cs.ok(cudaMemcpy(d_samples, samples, sizeof(float2) * n_samples, cudaMemcpyHostToDevice));
  std::vector<b200ba_feature_prediction> pred(max_per_chunk);
  std::vector<float2> out_xy(max_per_chunk);
  std::vector<float> out_cost(max_per_chunk);
  std::vector<int> out_status(max_per_chunk);
  double ms = 0.0;
  for (int64_t lo = 0, i0 = 0; i0 < n_images && cs.rc == 0; i0 += chunk) {
    const int64_t m_img = std::min<int64_t>(chunk, n_images - i0);
    int64_t hi = lo;
    while (hi < n_features && predictions[order[hi]].image < i0 + m_img) ++hi;
    if (hi == lo) continue;
    cs.ok(cudaMemcpy(d_img, images + i0 * pixels, static_cast<size_t>(m_img) * pixels, cudaMemcpyHostToDevice));
    for (; lo < hi && cs.rc == 0; lo += kMaxLaunch) {
      const int64_t m = std::min(hi - lo, kMaxLaunch);
      for (int64_t k = 0; k < m; ++k) {
        pred[k] = predictions[order[lo + k]];
        pred[k].image -= i0;
      }
      cs.ok(cudaMemcpy(d_pred, pred.data(), sizeof(b200ba_feature_prediction) * m, cudaMemcpyHostToDevice));
      if (cs.rc != 0) break;
      cs.record(0, 0);
      launch_refine_features(rp, m, d_pred, d_img, d_samples, d_xy, d_cost, d_status, 0);
      cs.record(1, 0);
      cs.ok(cudaGetLastError());
      if (cs.rc == 0) cs.ok(cudaMemcpy(out_xy.data(), d_xy, sizeof(float2) * m, cudaMemcpyDeviceToHost));
      if (cs.rc == 0) cs.ok(cudaMemcpy(out_cost.data(), d_cost, sizeof(float) * m, cudaMemcpyDeviceToHost));
      if (cs.rc == 0) cs.ok(cudaMemcpy(out_status.data(), d_status, sizeof(int) * m, cudaMemcpyDeviceToHost));
      if (cs.rc != 0) break;
      ms += cs.elapsed_ms(0, 1);
      for (int64_t k = 0; k < m; ++k) {
        const int64_t i = order[lo + k];
        xy[2 * i] = out_xy[k].x;
        xy[2 * i + 1] = out_xy[k].y;
        final_cost[i] = out_cost[k];
        if (status) status[i] = out_status[k];
      }
    }
    lo = hi;
  }
  if (cs.rc == 0 && device_ms) *device_ms = ms;
  return cs.rc;
}

// Eigen::LDLT<MatrixXd, Lower>(A.selfadjointView<Upper>()).solve(b) for n = 3 (SolveDensely, LV/lm_optimizer.h:1022-1023):
// symmetric pivoting on the largest remaining |diagonal| entry as Eigen's left-looking factorisation sees it (the
// ORIGINAL values of the trailing diagonal), then x = P^T L^-T D^-1 L^-1 P b with 1 / d_i taken as 0 where
// |d_i| <= 1 / DBL_MAX. A is symmetric, row-major.
static void ldlt_solve3(const double A[3][3], const double b[3], double x[3]) {
  double L[3][3], od[3], col[3];
  int transp[3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j <= i; ++j) L[i][j] = A[j][i];
  for (int i = 0; i < 3; ++i) od[i] = L[i][i];
  for (int k = 0; k < 3; ++k) {
    int piv = k;
    for (int i = k + 1; i < 3; ++i)
      if (std::fabs(od[i]) > std::fabs(od[piv])) piv = i;
    transp[k] = piv;
    if (piv != k) {  // symmetric row / column swap k <-> piv on the lower triangle
      std::swap(od[k], od[piv]);
      for (int j = 0; j < k; ++j) std::swap(L[k][j], L[piv][j]);
      for (int i = piv + 1; i < 3; ++i) std::swap(L[i][k], L[i][piv]);
      std::swap(L[k][k], L[piv][piv]);
      for (int i = k + 1; i < piv; ++i) std::swap(L[i][k], L[piv][i]);
    }
    const double dk = L[k][k];
    if (std::fabs(dk) > 0) {
      for (int i = k + 1; i < 3; ++i) {
        col[i] = L[i][k];
        L[i][k] = col[i] / dk;
      }
      for (int i = k + 1; i < 3; ++i)
        for (int j = k + 1; j <= i; ++j) L[i][j] -= L[i][k] * col[j];
    }
  }
  double y[3] = {b[0], b[1], b[2]};
  for (int k = 0; k < 3; ++k) std::swap(y[k], y[transp[k]]);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < i; ++j) y[i] -= L[i][j] * y[j];
  const double tolerance = 1.0 / std::numeric_limits<double>::max();
  for (int i = 0; i < 3; ++i) y[i] = std::fabs(L[i][i]) > tolerance ? y[i] / L[i][i] : 0.0;
  for (int i = 2; i >= 0; --i)
    for (int j = 0; j < i; ++j) y[j] -= L[i][j] * y[i];
  for (int k = 2; k >= 0; --k) std::swap(y[k], y[transp[k]]);
  for (int i = 0; i < 3; ++i) x[i] = y[i];
}

// The NoncentralGenericModel branch of CreateCalibrationReportForCamera (APP/calibration_report.cc:839-982). The
// argument checks come first and touch no CUDA state. The LM loop is small_lm, LMOptimizer::OptimizeImpl
// (LV/lm_optimizer.h:628-991) as b200ba_fit_directions runs it; H = sum t1 t1^T + t2 t2^T does not depend on the centre,
// so it is summed once (the reference rebuilds the same matrix every iteration), and every iteration then needs one
// pass for b and the cost and every attempt one pass for the trial cost, each a sum of per-line costs.
int b200ba_line_offsets(int device, const b200ba_camera* cam, const double* intrinsics, b200ba_line_offsets_report* report,
                        uint8_t* image, double* offsets, int32_t obj_step, double* obj_lines, int64_t* n_obj,
                        double* device_ms) {
  if (!cam || !intrinsics || !report) {
    g_create_error = "b200ba_line_offsets: a required argument is NULL";
    return 2;
  }
  if (cam->model_type != B200BA_MODEL_NONCENTRAL_GENERIC) {
    g_create_error = "b200ba_line_offsets: the centre-point analysis is only defined for NoncentralGenericModel";
    return 2;
  }
  if (cam->grid_width < 4 || cam->grid_height < 4) {
    g_create_error = "b200ba_line_offsets: the grid is smaller than 4 x 4";
    return 2;
  }
  if (obj_step < 1 || (obj_lines && !n_obj)) {
    g_create_error = "b200ba_line_offsets: obj_step must be >= 1, and obj_lines needs n_obj";
    return 2;
  }
  // the reference writes every line's offset into an image of the camera's size (:870, :889)
  if (cam->calibration_min_x < 0 || cam->calibration_min_y < 0 || cam->calibration_max_x < cam->calibration_min_x ||
      cam->calibration_max_y < cam->calibration_min_y || cam->calibration_max_x >= cam->width ||
      cam->calibration_max_y >= cam->height) {
    g_create_error = "b200ba_line_offsets: the calibrated area is empty or not inside the image";
    return 2;
  }
  CallScope cs(&g_create_error);
  if (int rc = cs.use_device(device)) return rc;
  CamDev c{};
  fill_camdev(*cam, &c);
  const int rw = cam->calibration_max_x - cam->calibration_min_x + 1, rh = cam->calibration_max_y - cam->calibration_min_y + 1;
  const int64_t n = static_cast<int64_t>(rw) * rh, npx = static_cast<int64_t>(cam->width) * cam->height;
  const int nx = (rw - 1) / obj_step + 1, ny = (rh - 1) / obj_step + 1;
  const int64_t nobj = static_cast<int64_t>(nx) * ny;
  const int64_t ni = intrinsics_size(*cam);
  double* dintr = nullptr;
  LineOffsetsDev d{};
  cs.alloc(&dintr, ni);
  cs.alloc(&d.lines, 6 * n);
  cs.alloc(&d.partial, line_system_partial_size());
  cs.alloc(&d.sums, kLineSums);
  cs.alloc(&d.mag, n);
  cs.alloc(&d.extent, 1);
  alloc_range_statistics(cs, n, &d.range, &d.stat_partial, &d.select_hist, &d.stats);
  if (offsets) cs.alloc(&d.offsets, 3 * npx);
  if (image) cs.alloc(&d.image, 3 * npx);
  if (obj_lines) cs.alloc(&d.obj, 12 * nobj);
  if (cs.rc == 0) cs.ok(cudaMemcpy(dintr, intrinsics, sizeof(double) * ni, cudaMemcpyHostToDevice));
  b200ba_line_offsets_report rep{};
  double center[3] = {0, 0, 0};  // Vec3d::Zero() (:858)
  ReportCam stats{};
  unsigned long long extent_bits = 0;
  if (cs.rc == 0) {
    cs.record(0, 0);
    launch_line_pass(c, dintr, d, 0);
    auto pass = [&](int mode, const double* at, double* out) {
      launch_line_system(mode, n, at, d, 0);
      cs.ok(cudaMemcpy(out, d.sums, sizeof(double) * kLineSums, cudaMemcpyDeviceToHost));
    };
    // Optimize(&center, cost, max_iteration_count = 100, max_lm_attempts = 10, init_lambda = -1,
    // init_lambda_factor = 0.001f) (:859-867)
    double H[3][3] = {}, s[kLineSums] = {}, x[3], trial[3];
    const LmResult lm = small_lm(
        cs.rc, 100,
        [&](int iteration) {  // b and the cost at the centre; H does not depend on it and is summed once
          pass(iteration == 0 ? 2 : 1, center, s);
          if (iteration == 0) {
            H[0][0] = s[4]; H[0][1] = H[1][0] = s[5]; H[0][2] = H[2][0] = s[6];
            H[1][1] = s[7]; H[1][2] = H[2][1] = s[8]; H[2][2] = s[9];
          }
          return s[0];
        },
        [&](double init_lambda_factor) { return init_lambda_factor * (((0.0 + H[0][0]) + H[1][1]) + H[2][2]) / 3; },
        [&](double lambda) {
          double A[3][3];
          for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) A[i][j] = H[i][j] + (i == j ? lambda : 0.0);
          ldlt_solve3(A, s + 1, x);
          return !std::isnan(x[0]);  // false: the reference's NaN-update branch
        },
        [&] {
          for (int i = 0; i < 3; ++i) trial[i] = center[i] - x[i];
          double t[kLineSums];
          pass(0, trial, t);
          return t[0];
        },
        [&] { std::copy(trial, trial + 3, center); });
    rep.initial_cost = lm.initial_cost;
    rep.final_cost = lm.final_cost;
    rep.num_iterations_performed = lm.iterations;
    rep.lm_attempts = lm.attempts;
    launch_line_outputs(c, center, d, obj_step, nx, nobj, 0);
    cs.record(1, 0);
    cs.ok(cudaGetLastError());
    cs.ok(cudaMemcpy(&stats, d.stats, sizeof(ReportCam), cudaMemcpyDeviceToHost));
    cs.ok(cudaMemcpy(&extent_bits, d.extent, sizeof(extent_bits), cudaMemcpyDeviceToHost));
    if (offsets) cs.ok(cudaMemcpy(offsets, d.offsets, sizeof(double) * 3 * npx, cudaMemcpyDeviceToHost));
    if (image) cs.ok(cudaMemcpy(image, d.image, 3 * npx, cudaMemcpyDeviceToHost));
    if (obj_lines) cs.ok(cudaMemcpy(obj_lines, d.obj, sizeof(double) * 12 * nobj, cudaMemcpyDeviceToHost));
  }
  if (cs.rc == 0) {
    if (device_ms) *device_ms = cs.elapsed_ms(0, 1);
    std::copy(center, center + 3, rep.center);
    rep.line_count = stats.count;
    rep.line_distance_sum = stats.sum;
    rep.line_distance_max = stats.max;  // max is order-independent: the fixed-order reduction's max is exact
    rep.line_distance_median = stats.median;
    memcpy(&rep.max_line_offset_extent, &extent_bits, sizeof(double));
    *report = rep;
    if (n_obj) *n_obj = nobj;
  }
  return cs.rc;
}

// ---- multi-GPU -------------------------------------------------------------------------------------
int b200ba_nccl_unique_id(uint8_t id[B200BA_NCCL_UNIQUE_ID_BYTES]) {
  std::string err;
  if (!load_nccl(&err)) {
    g_create_error = err;
    return 1;
  }
  return g_nccl.GetUniqueId(id) == 0 ? 0 : 1;
}

int b200ba_comm_init(b200ba_handle* h, const uint8_t id[B200BA_NCCL_UNIQUE_ID_BYTES], int rank, int n_ranks) {
  if (!h) return 1;
  if (n_ranks <= 1) {
    h->rank = 0;
    h->n_ranks = 1;
    return 0;
  }
  std::string err;
  if (!load_nccl(&err)) {
    h->error = err;
    return 1;
  }
  CUDA_TRY(h, cudaSetDevice(h->device));
  NcclUniqueId uid;
  memcpy(uid.internal, id, 128);
  int rc = g_nccl.CommInitRank(&h->comm, n_ranks, uid, rank);
  if (rc != 0) {
    h->error = std::string("ncclCommInitRank: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "error");
    return 1;
  }
  h->rank = rank;
  h->n_ranks = n_ranks;
  if (plan_dense(h)) return 1;
  // every rank must derive the same groups of Schur blocks: reduce the centroid sums
  if (h->L.eliminate_points && h->L.nblocks > 0 && !h->grp_sums.empty()) {
    if (reduce_group_sums(h)) return 1;
    if (build_groups(h, false)) return 1;
  }
  return 0;
}

}  // extern "C"
