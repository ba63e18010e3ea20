// ba_dense.cu -- hand-written FP64 tensor-core (DMMA) kernels of the dense phase (sm_90a).
//
// The reduced system of the Schur-complement solve (LV/lm_optimizer.h:1246-1369) is formed and
// factorised with the kernels of this file instead of library calls:
//
//   dgemm_nt_kernel     C (+)= alpha * A B^T on 128 x 64 tiles, 32 x 32 warp tiles, FP64
//                       `mma.sync.m16n8k4` (SASS DMMA.16x8x4), operands staged through shared memory
//                       by a 4-stage cp.async pipeline. One kernel, three uses:
//                         * LOWER + plain epilogue: trailing update S22 -= L21 L21^T of the blocked Cholesky
//                           (the reference factors with Eigen's LDLT, LV/lm_optimizer.h:1361);
//                         * plain epilogue, K = N = 128: the panel solve L21 = A21 L11^-T as a product with the
//                           explicitly inverted diagonal tile;
//                         * LOWER + scatter epilogue: the structured Schur contraction S -= W_g^T W_g on the
//                           compact panel of one group of Schur blocks, scattered straight into S through
//                           the group's column list (the reference contracts with Eigen / cublasXtDgemm,
//                           LV/lm_optimizer.h:1328,1371-1430) -- no m_g x m_g temporary, no scatter pass;
//                           one launch covers every group (grouped mode: FP64 reductions into S).
//   potrf_trinv_tile_kernel
//                       Cholesky of one 128 x 128 diagonal tile + its explicit inverse (ba_tile.cuh).
//   small helpers       lambda on the diagonal, column-block copies.
//
// All operands of dgemm_nt are "k-strided": element (i, k) of A lives at A[k * lda + i] (i contiguous),
// which is what both a column-major panel of S and a row-major compact panel W_g[k][j] look like.
// C is column-major (element (i, j) at C[j * ldc + i]); for a symmetric result only i >= j is touched.

#include <algorithm>
#include <cstdio>

#include "ba_kernels.h"
#include "ba_tile.cuh"

namespace b200ba {

namespace {

constexpr int BM = 128;
constexpr int LDT = BM + 4;  // shared-memory row pitch: (k * LDT + m) mod 16 is distinct for k, m in 0..3 -> no bank conflicts
__host__ __device__ constexpr int gemm_threads(int bn) { return 4 * (bn / 32) * 32; }  // 4 x (bn / 32) warps, warp tile 32 x 32
constexpr size_t gemm_smem(int bn, int bk, int stages) {
  return static_cast<size_t>(stages) * bk * (LDT + bn + 4) * sizeof(double);
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, int src_bytes) {
  const unsigned s = static_cast<unsigned>(__cvta_generic_to_shared(smem));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async8(void* smem, const void* gmem, int src_bytes) {
  const unsigned s = static_cast<unsigned>(__cvta_generic_to_shared(smem));
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"(s), "l"(gmem), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}
// One m16n8k4 FP64 MMA (SASS DMMA.16x8x4: twice the FMAs per instruction of m8n8k4, which H100 issues at the
// same rate, so half the tensor pipe's peak is out of reach with m8n8k4). Fragments (lane = 4 lr + lc):
// a0 = A(m = lr, k = lc), a1 = A(lr + 8, lc), b = B(n = lr, k = lc), c[v0 + 2 v1] = C(m = lr + 8 v1, n = 2 lc + v0).
__device__ __forceinline__ void dmma1684(double& c0, double& c1, double& c2, double& c3, double a0, double a1, double b) {
  asm("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
      : "+d"(c0), "+d"(c1), "+d"(c2), "+d"(c3)
      : "d"(a0), "d"(a1), "d"(b));
}

// Loader of one operand's BK x W tiles (pitch W + 4): rows k0 .. k0 + BK of the k-strided matrix X (leading
// dimension ldx), columns i0 .. i0 + W, zero-filled beyond (rows, K). Everything that does not change along k --
// the source pointer of each of the thread's chunks, its byte count (row in range?), its shared-memory offset --
// is computed ONCE per tile in init(); issue() only advances the pointers by BK rows and checks k < K. (The first
// version recomputed the index arithmetic and four predicates per chunk in every k-iteration: with 2-4 warps per
// scheduler that integer latency was a third of all stall samples.) `aligned` = every 16-byte chunk is 16-byte
// aligned in global memory (even ldx, even i0, 16-byte aligned base); otherwise 8-byte copies.
template <int BK, int W, int THREADS>
struct TileLoader {
  static constexpr int LD = W + 4;
  static constexpr int CH = W / 2;               // 16-byte chunks per row
  static constexpr int KS16 = THREADS / CH;      // rows between two chunks of one thread (aligned path)
  static constexpr int KS8 = THREADS / W;        // ... (unaligned path)
  static constexpr int Q16 = BK / KS16, Q8 = BK / KS8;
  static_assert(THREADS % CH == 0 && THREADS % W == 0 && BK % KS16 == 0 && BK % KS8 == 0, "tile / thread count mismatch");
  // all chunks of a thread sit in the same column(s) and KS rows apart: one pointer, one byte count. X and ldx
  // are not kept: issue() takes them from the kernel arguments, which stay in the constant bank instead of
  // holding six registers through the main loop.
  const double* src;   // chunk of row k0 + kk0
  int off0, kk0, bytes;
  bool aligned;

  __device__ __forceinline__ void init(const double* __restrict__ X, int64_t ldx, int rows, int i0, bool al) {
    aligned = al;
    int i;
    if (al) {
      kk0 = threadIdx.x / CH;
      const int ch = threadIdx.x % CH;
      i = i0 + 2 * ch;
      off0 = kk0 * LD + 2 * ch;
      bytes = (i + 1 < rows) ? 16 : ((i < rows) ? 8 : 0);
    } else {
      kk0 = threadIdx.x / W;
      const int ii = threadIdx.x % W;
      i = i0 + ii;
      off0 = kk0 * LD + ii;
      bytes = (i < rows) ? 8 : 0;
    }
    src = X + static_cast<int64_t>(kk0) * ldx + min(i, max(rows - 1, 0));
  }
  // copies the tile whose first row is k0 into dst and advances to the next tile (X, ldx: those of init())
  __device__ __forceinline__ void issue(double* dst, int k0, int K, const double* __restrict__ X, int64_t ldx) {
    const double* p = src;
    if (aligned) {
#pragma unroll
      for (int q = 0; q < Q16; ++q) {
        const int nb = (k0 + kk0 + q * KS16 < K) ? bytes : 0;
        cp_async16(dst + off0 + q * KS16 * LD, nb ? p : X, nb);
        p += KS16 * ldx;
      }
    } else {
#pragma unroll
      for (int q = 0; q < Q8; ++q) {
        const int nb = (k0 + kk0 + q * KS8 < K) ? bytes : 0;
        cp_async8(dst + off0 + q * KS8 * LD, nb ? p : X, nb);
        p += KS8 * ldx;
      }
    }
    src += BK * ldx;
  }
};

}  // namespace

// C(i, j) at Cbase + col_off(j) + i, where col_off maps a column to its storage offset (see DenseMap).
// CTA tile 128 x BN_ (instantiated at BN_ = 64: 8 warps, two CTAs per SM so that one CTA's read-modify-write
// epilogue overlaps the other's tensor-core main loop).
template <bool LOWER, int EPI, int BN_, int BK, int STAGES>
__global__ void __launch_bounds__(gemm_threads(BN_), 2) dgemm_nt_kernel(GemmArgs g) {
  constexpr int THREADS = gemm_threads(BN_);
  constexpr int LDB = BN_ + 4;
  extern __shared__ __align__(16) double smem_d[];
  double* As = smem_d;
  double* Bs = smem_d + static_cast<size_t>(STAGES) * BK * LDT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wm = (warp & 3) * 32, wn = (warp >> 2) * 32;  // warp tile 32 (m) x 32 (n)
  const int lr = lane >> 2, lc = lane & 3;
  // Persistent CTAs (unless one_tile_per_cta): the grid is capped at two CTAs per SM and every CTA walks the
  // tile list with stride gridDim.x. LOWER: only the tiles that intersect i >= j, enumerated row by row:
  // row tm holds min(q (tm + 1), tiles_n) tiles with q = 128 / BN_.
  // EPI 3 (the grouped contraction): the tile list is the concatenation of every group's lower tiles, and each
  // tile takes its operand panel, sizes and column list from its group's entry of g.groups.
  constexpr int Q = BM / BN_;
  int M = g.M, N = g.N, K = g.K;
  const double* A = g.A;
  const double* Bop = g.B;
  int64_t lda = g.lda, ldb = g.ldb;
  const int* cols = g.cols;
  bool a_al = g.a_aligned, b_al = g.b_aligned;
  int tiles_m = (M + BM - 1) / BM, tiles_n = (N + BN_ - 1) / BN_;
  int t_full = min(tiles_m, tiles_n / Q);  // rows whose tile count is still growing
  int64_t tri = static_cast<int64_t>(Q) * t_full * (t_full + 1) / 2;
  const int64_t n_tiles = LOWER ? g.n_tiles_lower : static_cast<int64_t>(tiles_m) * tiles_n;
  for (int64_t tile_g = blockIdx.x; tile_g < n_tiles; tile_g += gridDim.x) {
    int64_t tile = tile_g;
    if (EPI == 3) {
      int lo = 0, hi = g.n_groups - 1;  // last group whose first tile is <= tile_g
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (g.groups[mid].tile0 <= tile_g) lo = mid; else hi = mid - 1;
      }
      const ContractGroup cg = g.groups[lo];
      tile = tile_g - cg.tile0;
      M = N = cg.m;
      K = cg.k;
      A = Bop = g.A + cg.w_off;
      lda = ldb = cg.ld;
      cols = g.cols + cg.cols_off;
      a_al = b_al = cg.aligned;
      tiles_m = (M + BM - 1) / BM;
      tiles_n = (N + BN_ - 1) / BN_;
      t_full = min(tiles_m, tiles_n / Q);
      tri = static_cast<int64_t>(Q) * t_full * (t_full + 1) / 2;
    }
    int tm, tn;
    if (LOWER) {
      if (tile < tri) {
        // largest tm with Q tm (tm + 1) / 2 <= tile
        tm = static_cast<int>((sqrt(8.0 * static_cast<double>(tile) / Q + 1.0) - 1.0) * 0.5);
        while (static_cast<int64_t>(Q) * tm * (tm + 1) / 2 > tile) --tm;
        while (static_cast<int64_t>(Q) * (tm + 1) * (tm + 2) / 2 <= tile) ++tm;
        tn = static_cast<int>(tile - static_cast<int64_t>(Q) * tm * (tm + 1) / 2);
      } else {
        const int64_t rest = tile - tri;
        tm = t_full + static_cast<int>(rest / tiles_n);
        tn = static_cast<int>(rest - static_cast<int64_t>(tm - t_full) * tiles_n);
      }
    } else {
      tm = static_cast<int>(tile / tiles_n);
      tn = static_cast<int>(tile - static_cast<int64_t>(tm) * tiles_n);
    }
    const int m0 = tm * BM, n0 = tn * BN_;
    if (EPI == 2) {
      // block-cyclic ownership of the column blocks: this rank updates only the tiles of its own blocks
      const int blk = (g.col_base + n0) / g.map.nb;
      if (blk % g.map.ranks != g.rank) continue;
    }
    __syncthreads();  // the previous tile's shared-memory stages are free

    double acc[4][4][2];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

    const int nk = (K + BK - 1) / BK;
    TileLoader<BK, BM, THREADS> la;
    TileLoader<BK, BN_, THREADS> lb;
    la.init(A, lda, M, m0, a_al);
    lb.init(Bop, ldb, N, n0, b_al);
#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
      if (s < nk) {
        la.issue(As + s * BK * LDT, s * BK, K, A, lda);
        lb.issue(Bs + s * BK * LDB, s * BK, K, Bop, ldb);
      }
      cp_async_commit();
    }
    for (int kt = 0; kt < nk; ++kt) {
      cp_async_wait<STAGES - 2>();
      __syncthreads();
      {
        // prefetch the tile STAGES - 1 ahead into the slot that was consumed in the previous iteration
        const int nt = kt + STAGES - 1;
        if (nt < nk) {
          const int s = nt % STAGES;
          la.issue(As + s * BK * LDT, nt * BK, K, A, lda);
          lb.issue(Bs + s * BK * LDB, nt * BK, K, Bop, ldb);
        }
        cp_async_commit();
      }
      const double* a_s = As + (kt % STAGES) * BK * LDT;
      const double* b_s = Bs + (kt % STAGES) * BK * LDB;
#pragma unroll
      for (int ks = 0; ks < BK / 4; ++ks) {
        // af[i] = A(row wm + 8 i + lr, k = 4 ks + lc), bf = B(column wn + 8 j + lr, same k). Rows 16 b .. 16 b + 15
        // of the warp tile are accumulator rows 2 b (m = lr) and 2 b + 1 (m = lr + 8): one m16n8k4 per (b, j).
        double af[4];
        const double* ap = a_s + (ks * 4 + lc) * LDT + wm + lr;
        const double* bp = b_s + (ks * 4 + lc) * LDB + wn + lr;
#pragma unroll
        for (int i = 0; i < 4; ++i) af[i] = ap[8 * i];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const double bf = bp[8 * j];
#pragma unroll
          for (int b = 0; b < 2; ++b)
            dmma1684(acc[2 * b][j][0], acc[2 * b][j][1], acc[2 * b + 1][j][0], acc[2 * b + 1][j][1], af[2 * b],
                     af[2 * b + 1], bf);
        }
      }
    }
    cp_async_wait<0>();

    // epilogue: accumulator (i, j) holds rows m0 + wm + 8 i + lr, columns n0 + wn + 8 j + 2 lc + {0, 1}.
    // Per output column the 4 read-modify-writes of a thread are issued as 4 loads, then 4 stores, so
    // that they overlap instead of forming a load -> store chain. EPI 3 adds alpha * acc with FP64 reductions
    // (RED.ADD.F64): tiles of different groups that hit one entry of S may run at the same time.
    constexpr bool SCATTER = EPI == 1 || EPI == 3;
    int rowidx[4];
    bool rowok[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = m0 + wm + 8 * i + lr;
      rowok[i] = m < M;
      rowidx[i] = SCATTER ? (rowok[i] ? __ldg(cols + m) : 0) : m;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int n = n0 + wn + 8 * j + 2 * lc + e;
        if (n >= N) continue;
        double* ccol = (EPI == 0) ? (g.C + static_cast<int64_t>(n) * g.ldc)
                                  : (SCATTER ? (g.C + g.map.col_offset(__ldg(cols + n)))
                                             : (g.C + g.map.col_offset(g.col_base + n) + g.col_base));
        bool ok[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) ok[i] = rowok[i] && !(LOWER && (m0 + wm + 8 * i + lr) < n);
        if (EPI == 3) {
#pragma unroll
          for (int i = 0; i < 4; ++i)
            if (ok[i]) atomicAdd(ccol + rowidx[i], g.alpha * acc[i][j][e]);
          continue;
        }
        double old[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) old[i] = (ok[i] && g.beta != 0.0) ? ccol[rowidx[i]] : 0.0;
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (ok[i]) ccol[rowidx[i]] = fma(g.beta, old[i], g.alpha * acc[i][j][e]);
      }
    }
  }  // tile loop
}

int64_t dgemm_lower_tiles(int M, int N) {
  constexpr int BN = 64, q = BM / BN;
  const int64_t tm = (M + BM - 1) / BM, tn = (N + BN - 1) / BN;
  const int64_t t_full = std::min<int64_t>(tm, tn / q);
  return q * t_full * (t_full + 1) / 2 + (tm - t_full) * tn;
}

int launch_dgemm_nt(const GemmArgs& g_in, bool lower, bool scatter, cudaStream_t s, bool one_tile_per_cta) {
  if (g_in.M <= 0 || g_in.N <= 0) return 0;
  // 128 x 64 tiles, BK 16 x 4 stages, 2 CTAs / SM
  constexpr int BN = 64, BK = 16, STAGES = 4;
  constexpr int T = gemm_threads(BN);
  constexpr int smem = static_cast<int>(gemm_smem(BN, BK, STAGES));
  static bool configured_dev[64] = {};
  static int sm_count[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  bool& configured = configured_dev[dev & 63];  // function attributes are per device
  if (!configured) {
    cudaFuncSetAttribute(dgemm_nt_kernel<true, 0, BN, BK, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(dgemm_nt_kernel<false, 0, BN, BK, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(dgemm_nt_kernel<true, 1, BN, BK, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(dgemm_nt_kernel<true, 2, BN, BK, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(dgemm_nt_kernel<true, 3, BN, BK, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaDeviceGetAttribute(&sm_count[dev & 63], cudaDevAttrMultiProcessorCount, dev);
    configured = true;
  }
  GemmArgs g = g_in;
  const bool tri_enum = lower || scatter || g.owned_only;
  int64_t n_tiles;
  if (g.groups) {
    n_tiles = g.n_tiles_lower;  // the sum of the groups' lower tile counts, set by the caller
    if (n_tiles <= 0 || g.n_groups <= 0) return 0;
  } else if (tri_enum) {
    n_tiles = dgemm_lower_tiles(g.M, g.N);
    g.n_tiles_lower = n_tiles;
  } else {
    n_tiles = static_cast<int64_t>((g.M + BM - 1) / BM) * ((g.N + BN - 1) / BN);
  }
  const int cap = std::max(1, sm_count[dev & 63] * 2);
  // one_tile_per_cta: an ordinary grid (the hardware scheduler can then hand SMs to a higher-priority stream
  // between tiles) instead of persistent CTAs
  const unsigned grid = static_cast<unsigned>(one_tile_per_cta ? n_tiles : std::min<int64_t>(n_tiles, cap));
  if (g.groups)
    dgemm_nt_kernel<true, 3, BN, BK, STAGES><<<grid, T, smem, s>>>(g);
  else if (g.owned_only)
    dgemm_nt_kernel<true, 2, BN, BK, STAGES><<<grid, T, smem, s>>>(g);
  else if (scatter)
    dgemm_nt_kernel<true, 1, BN, BK, STAGES><<<grid, T, smem, s>>>(g);
  else if (tri_enum)
    dgemm_nt_kernel<true, 0, BN, BK, STAGES><<<grid, T, smem, s>>>(g);
  else
    dgemm_nt_kernel<false, 0, BN, BK, STAGES><<<grid, T, smem, s>>>(g);
  return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

constexpr int PT = 128;  // diagonal tile size

// The blocked tile step (ba_tile.cuh): factor + inverse in one launch of 8 CTAs.
struct TileDeviceExec {
  tile::Thread t;
  template <class F>
  __host__ __device__ __forceinline__ void run(F f) {
#if defined(__CUDA_ARCH__)
    f(t, static_cast<int>(threadIdx.x));
    __syncthreads();
#else
    (void)f;
#endif
  }
};
__global__ void __launch_bounds__(tile::THREADS, 1)
    potrf_trinv_tile_kernel(const double* __restrict__ Ain, int64_t lda_in, int n, double* __restrict__ Lout, int64_t lda_out,
                            double* __restrict__ Linv, int* __restrict__ info) {
  extern __shared__ __align__(16) unsigned char tile_smem[];
  tile::Shared& sh = *reinterpret_cast<tile::Shared*>(tile_smem);
  TileDeviceExec ex;
  tile::potrf_trinv_program(ex, sh, Ain, lda_in, n, Lout, lda_out, Linv, static_cast<int>(blockIdx.x), info);
}
// Ain and Lout must not overlap (see ba_tile.cuh).
int launch_potrf_trinv_tile(const double* Ain, int64_t lda_in, int n, double* Lout, int64_t lda_out, double* Linv, int* info,
                            cudaStream_t s) {
  static bool configured_dev[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!configured_dev[dev & 63]) {
    cudaFuncSetAttribute(potrf_trinv_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(sizeof(tile::Shared)));
    configured_dev[dev & 63] = true;
  }
  potrf_trinv_tile_kernel<<<tile::CTAS, tile::THREADS, sizeof(tile::Shared), s>>>(Ain, lda_in, n, Lout, lda_out, Linv, info);
  return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

// ------------------------------------------------------------------------------------------
// small helpers
// ------------------------------------------------------------------------------------------
// S(c, c) += lambda through the storage map (LV/lm_optimizer.h:839-852: the damping is ADDED to the diagonal)
__global__ void add_diagonal_map_kernel(int n, double* S, DenseMap map, double lambda) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < n) S[map.col_offset(c) + c] += lambda;
}
void launch_add_diagonal_map(int n, double* S, const DenseMap& map, double lambda, cudaStream_t s) {
  if (n > 0) add_diagonal_map_kernel<<<(n + 255) / 256, 256, 0, s>>>(n, S, map, lambda);
}

// ------------------------------------------------------------------------------------------
// triangular solves with the packed factor
// ------------------------------------------------------------------------------------------
// The factor lives in packed block-column panels: panel k holds rows k0 .. n of the columns k0 .. k0 + NB
// (k0 = k * NB) column-major with leading dimension hk = even(n - k0); element L(i, c) = P_k[(c - k0) * hk +
// (i - k0)]. Every 128 x 128 diagonal tile also has its explicit inverse (Linv tiles, from potrf_trinv_tile).
//
// y_0 = Linv_0 b_0 (forward) or x_{T-1} = Linv_{T-1}^T y_{T-1} (backward, transpose): the first tile of each sweep
__global__ void trsv_store_tile_kernel(const double* __restrict__ Linv, const double* __restrict__ b, int live,
                                       double* __restrict__ out, bool transpose) {
  const int tid = threadIdx.x;
  if (tid >= live) return;
  double acc = 0.0;
  if (!transpose) {
    for (int c = 0; c <= tid; ++c) acc = fma(Linv[c * PT + tid], b[c], acc);
  } else {
    for (int i = tid; i < live; ++i) acc = fma(Linv[tid * PT + i], b[i], acc);
  }
  out[tid] = acc;
}

// The steps: the tile's solution arrives through global memory, so no CTA repeats the 128 x 128 product with the
// inverted diagonal tile before it touches its rows. Forward step t applies y_t to all rows below in 128-row CTAs
// (32 independent loads per thread and batch), and CTA 0 -- which owns exactly the rows of tile t + 1 -- goes on
// to y_{t+1} = Linv_{t+1} b_{t+1} with the inverse prefetched into shared memory by cp.async while the row update
// runs. One wave of at most 102 CTAs; nothing is computed twice.
constexpr int TS2_THREADS = 256;
constexpr int TS2_LD = PT + 2;  // pitch of the staged inverse (16-byte aligned columns)
constexpr size_t kTs2Smem = static_cast<size_t>(PT) * TS2_LD * sizeof(double);

__device__ __forceinline__ void stage_tile_async(double* dst, const double* __restrict__ src) {
  // 128 x 128 doubles, column c -> dst[c * TS2_LD ..]: 8192 chunks of 16 bytes
  for (int ch = threadIdx.x; ch < PT * PT / 2; ch += TS2_THREADS) {
    const int c = ch >> 6, i2 = (ch & 63) * 2;
    cp_async16(dst + c * TS2_LD + i2, src + c * PT + i2, 16);
  }
  cp_async_commit();
}

// forward: b_below -= L(below, tile t) y_t ; CTA 0: y_{t+1} = Linv_{t+1} b_{t+1}
__global__ void __launch_bounds__(TS2_THREADS, 1)
    trsv_forward2_kernel(const double* __restrict__ Lp /* L(row 0 below the tile, column 0 of the tile) */, int64_t hk,
                         int rows_below, const double* __restrict__ y_t, double* __restrict__ b_below,
                         const double* __restrict__ Linv_next, double* __restrict__ y_next) {
  extern __shared__ __align__(16) double ts2_smem[];
  __shared__ double ys[PT], part[2][PT], bs[PT];
  const int tid = threadIdx.x;
  const bool chain = blockIdx.x == 0;
  if (chain) stage_tile_async(ts2_smem, Linv_next);
  if (tid < PT) ys[tid] = y_t[tid];
  const int row = tid & (PT - 1), half = tid >> 7;
  const int r = blockIdx.x * PT + row;
  const bool live_row = r < rows_below;
  const double* lp = Lp + static_cast<int64_t>(half * 64) * hk + (live_row ? r : 0);
  __syncthreads();
  double acc0 = 0.0, acc1 = 0.0;
#pragma unroll
  for (int batch = 0; batch < 2; ++batch) {
    double l[32];
#pragma unroll
    for (int q = 0; q < 32; ++q) l[q] = live_row ? lp[static_cast<int64_t>(batch * 32 + q) * hk] : 0.0;
    const double* yc = ys + half * 64 + batch * 32;
#pragma unroll
    for (int q = 0; q < 32; q += 2) {
      acc0 = fma(l[q], yc[q], acc0);
      acc1 = fma(l[q + 1], yc[q + 1], acc1);
    }
  }
  part[half][row] = acc0 + acc1;
  __syncthreads();
  if (half == 0) {
    const double v = live_row ? b_below[r] - (part[0][row] + part[1][row]) : 0.0;
    if (chain)
      bs[row] = v;
    else if (live_row)
      b_below[r] = v;
  }
  if (!chain) return;
  cp_async_wait<0>();
  __syncthreads();
  // y_next(i) = sum_{c <= i} Linv(i, c) b(c): even / odd c per half
  double s0 = 0.0, s1 = 0.0;
  for (int c = half; c <= row; c += 4) {
    s0 = fma(ts2_smem[c * TS2_LD + row], bs[c], s0);
    if (c + 2 <= row) s1 = fma(ts2_smem[(c + 2) * TS2_LD + row], bs[c + 2], s1);
  }
  part[half][row] = s0 + s1;
  __syncthreads();
  if (half == 0 && live_row) y_next[row] = part[0][row] + part[1][row];
}

// backward: y_c -= sum_{i in tile t} L(i, c) x_i for the columns c left of the tile; CTA 0 (the columns of tile
// t - 1): x_{t-1} = Linv_{t-1}^T y_{t-1}. One warp per column (the rows of a column are contiguous), 16 columns
// per warp in two batches of 8 (32 loads in flight per lane).
__global__ void __launch_bounds__(TS2_THREADS, 1)
    trsv_backward2_kernel(const double* __restrict__ Lpack, const int64_t* __restrict__ panel_off,
                          const int* __restrict__ panel_h, int NB, int r0, int live, const double* __restrict__ x_t,
                          double* __restrict__ y /* full vector */, const double* __restrict__ Linv_prev,
                          double* __restrict__ x_prev /* at row r0 - 128 */) {
  extern __shared__ __align__(16) double ts2_smem[];
  __shared__ double xs[PT], ysm[PT], part[2][PT];
  const int tid = threadIdx.x;
  const bool chain = blockIdx.x == 0;
  if (chain) stage_tile_async(ts2_smem, Linv_prev);
  if (tid < PT) xs[tid] = (tid < live) ? x_t[tid] : 0.0;
  __syncthreads();
  const int warp = tid >> 5, lane = tid & 31;
  const int cbase = r0 - PT * (static_cast<int>(blockIdx.x) + 1);  // this CTA's 128 columns: cbase .. cbase + 127
#pragma unroll
  for (int batch = 0; batch < 2; ++batch) {
    double l[8][4];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int c = cbase + warp * 16 + batch * 8 + q;
      const int k = c / NB;
      const double* col = Lpack + panel_off[k] + static_cast<int64_t>(c - k * NB) * panel_h[k] + (r0 - k * NB);
#pragma unroll
      for (int u = 0; u < 4; ++u) l[q][u] = (lane + 32 * u < live) ? col[lane + 32 * u] : 0.0;
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      double acc = 0.0;
#pragma unroll
      for (int u = 0; u < 4; ++u) acc = fma(l[q][u], xs[lane + 32 * u], acc);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) {
        const int c = cbase + warp * 16 + batch * 8 + q;
        const double v = y[c] - acc;
        if (chain)
          ysm[c - cbase] = v;
        else
          y[c] = v;
      }
    }
  }
  if (!chain) return;
  cp_async_wait<0>();
  __syncthreads();
  // x_prev(j) = sum_{i >= j} Linv(i, j) y(i): column j of the staged inverse, even / odd i per half
  const int j = tid & (PT - 1), half = tid >> 7;
  double s0 = 0.0, s1 = 0.0;
  const double* colj = ts2_smem + j * TS2_LD;
  for (int i = j + half; i < PT; i += 4) {
    s0 = fma(colj[i], ysm[i], s0);
    if (i + 2 < PT) s1 = fma(colj[i + 2], ysm[i + 2], s1);
  }
  part[half][j] = s0 + s1;
  __syncthreads();
  if (half == 0) x_prev[j] = part[0][j] + part[1][j];
}

// ------------------------------------------------------------------------------------------
// host side: blocked right-looking Cholesky with look-ahead, block-cyclic over the ranks
// ------------------------------------------------------------------------------------------
int dense_plan(DenseCtx* d, int n, int nb, int rank, int ranks) {
  d->n = n;
  d->rank = rank;
  d->ranks = ranks;
  d->NB = nb;
  d->nblk = (n + nb - 1) / nb;
  d->ntiles = (n + PT - 1) / PT;
  d->map.nb = nb;
  d->map.ranks = ranks;
  d->map.blocks_per_rank = (d->nblk + ranks - 1) / ranks;
  d->map.ld = (n + 1) / 2 * 2;
  d->chunk = static_cast<int64_t>(d->map.blocks_per_rank) * nb * d->map.ld;
  d->panel_off.assign(d->nblk + 1, 0);
  d->panel_h.assign(std::max(1, d->nblk), 0);
  for (int k = 0; k < d->nblk; ++k) {
    const int hk = n - k * nb;
    d->panel_h[k] = (hk + 1) / 2 * 2;
    // a panel region = hk x NB factor columns followed by the inverses of its diagonal tiles: ONE broadcast
    d->panel_off[k + 1] = d->panel_off[k] + static_cast<int64_t>(d->panel_h[k]) * nb + static_cast<int64_t>(nb / PT) * PT * PT;
  }
  return 0;
}

// Factors the matrix held (lower triangle, storage map d->map) in d->S. On return every rank holds the
// complete factor in d->Lpack. Work is enqueued on d->s_main / d->s_panel; the caller synchronises.
//
// Schedule (right-looking, block columns of NB, owner(k) = k mod R). The whole critical path lives on the
// high-priority panel stream:
//     factor(k) -> broadcast(k) -> U(k, k+1) -> [wait rest(k-1)] -> U(k, k+2) -> factor(k+1) -> ...
// where U(k, j) applies panel k to block column j (each rank only for the blocks it owns). The bulk
//     rest(k) = U(k, j) for all owned j >= k + 3
// runs on the main stream as ordinary (non-persistent) grids, so the panel stream's CTAs take over SMs at
// tile granularity. Block column j thus receives its updates in panel order: rest(k) for k <= j - 3 (main stream,
// in order), then U(j-2, j) (after the wait for rest(j-3)), then U(j-1, j), then it is factored. rest(k) has a
// whole iteration of the chain to finish before anything waits for it: per iteration the cost is
// max(chain, rest) instead of chain + rest.
int dense_factor(DenseCtx* d) {
  const int n = d->n, NB = d->NB, R = d->ranks, me = d->rank;
  if (n == 0) return 0;
  const int sub_n = NB / PT;
  cudaStream_t sm = d->s_main, sp = d->s_panel;
  auto owner = [&](int k) { return k % R; };
  const bool use_aux = R == 1 && d->s_aux != nullptr;
  // S is ready when everything queued on s_main so far has run
  cudaEventRecord(d->ev_misc, sm);
  cudaStreamWaitEvent(sp, d->ev_misc, 0);

  // U(k, j_first .. j_last): one launch; owned_only = skip the tiles of column blocks other ranks own
  auto update = [&](int k, int j_first, int j_last, cudaStream_t st, bool owned_only) -> int {
    if (j_first >= d->nblk || j_first > j_last) return 0;
    const int k0 = k * NB, kw = std::min(NB, n - k0);
    const int j0 = j_first * NB;
    const int jn = std::min(n, (std::min(j_last, d->nblk - 1) + 1) * NB) - j0;
    if (jn <= 0) return 0;
    GemmArgs g{};
    g.M = n - j0;
    g.N = jn;
    g.K = kw;
    g.A = d->Lpack + d->panel_off[k] + (j0 - k0);
    g.lda = d->panel_h[k];
    g.B = g.A;
    g.ldb = g.lda;
    g.alpha = -1.0;
    g.beta = 1.0;
    g.a_aligned = g.b_aligned = gemm_operand_aligned(g.A, g.lda);
    if (owned_only) {
      g.C = d->S;
      g.map = d->map;
      g.owned_only = true;
      g.rank = me;
      g.col_base = j0;
    } else {
      g.C = d->S + d->map.col_offset(j0) + j0;
      g.ldc = d->map.ld;
    }
    return launch_dgemm_nt(g, /*lower=*/true, /*scatter=*/false, st, /*one_tile_per_cta=*/true);
  };

  for (int k = 0; k < d->nblk; ++k) {
    const int k0 = k * NB, kw = std::min(NB, n - k0), hk = d->panel_h[k], hlive = n - k0;
    double* P = d->Lpack + d->panel_off[k];
    if (owner(k) == me) {
      // Panel factorisation straight out of S: every diagonal tile goes through the blocked factor + inverse launch
      // (S -> P), the rows below it are solved OUT of place (S -> P: in place, the CTA of columns 0..63 of a row
      // block would overwrite operand columns the CTA of columns 64..127 still reads), and the panel-internal
      // update is applied to the remaining columns in S.
      const double* Sk = d->S + d->map.col_offset(k0) + k0;  // (i, c) of the block column at Sk[c * ld + i]
      double* Sk_w = d->S + d->map.col_offset(k0) + k0;
      const int64_t ld = d->map.ld;
      for (int sub = 0; sub < sub_n; ++sub) {
        const int c0 = sub * PT;
        if (c0 >= kw) break;
        const int live = std::min(PT, kw - c0);
        double* tile_out = P + static_cast<int64_t>(c0) * hk + c0;
        double* Li = P + static_cast<int64_t>(hk) * NB + static_cast<int64_t>(sub) * PT * PT;
        if (launch_potrf_trinv_tile(Sk + static_cast<int64_t>(c0) * ld + c0, ld, live, tile_out, hk, Li, d->info, sp)) return 1;
        const int below = hlive - c0 - PT;
        if (below > 0) {
          GemmArgs g{};  // rows below: X = A Linv^T
          g.M = below;
          g.N = PT;
          g.K = PT;
          g.A = Sk + static_cast<int64_t>(c0) * ld + c0 + PT;
          g.lda = ld;
          g.B = Li;
          g.ldb = PT;
          g.C = tile_out + PT;
          g.ldc = hk;
          g.alpha = 1.0;
          g.beta = 0.0;
          g.a_aligned = gemm_operand_aligned(g.A, g.lda);
          g.b_aligned = gemm_operand_aligned(g.B, g.ldb);
          if (launch_dgemm_nt(g, false, false, sp, true)) return 1;
          const int rest = kw - c0 - PT;  // remaining columns of this panel
          if (rest > 0) {
            GemmArgs u{};
            u.M = below;
            u.N = rest;
            u.K = PT;
            u.A = tile_out + PT;
            u.lda = hk;
            u.B = u.A;
            u.ldb = hk;
            u.C = Sk_w + static_cast<int64_t>(c0 + PT) * ld + (c0 + PT);
            u.ldc = ld;
            u.alpha = -1.0;
            u.beta = 1.0;
            u.a_aligned = u.b_aligned = gemm_operand_aligned(u.A, u.lda);
            if (launch_dgemm_nt(u, true, false, sp, true)) return 1;
          }
        }
      }
    }
    if (R > 1) {
      // the packed panel and the inverses of its diagonal tiles (stored right behind it) travel together
      if (d->bcast(P, static_cast<size_t>(hk) * NB + static_cast<size_t>(sub_n) * PT * PT, owner(k), sp, d->user)) return 1;
    }
    cudaEventRecord(d->ev_ready[k & 1], sp);
    // bulk of the trailing update on the main stream: owned blocks >= k + 3
    cudaStreamWaitEvent(sm, d->ev_ready[k & 1], 0);
    if (k + 3 < d->nblk && update(k, k + 3, d->nblk - 1, sm, R > 1)) return 1;
    cudaEventRecord(d->ev_main[k & 1], sm);  // rest(k) done
    if (use_aux) {
      // one GPU: U(k, k + 2) is not needed before factor(k + 1) -- it only sat on the panel stream because the stream
      // serialises. It runs beside the next panel factorisation on a third (high-priority) stream; the panel stream
      // picks it up again before U(k + 1, k + 2).
      if (k >= 1) cudaStreamWaitEvent(sp, d->ev_half2[(k - 1) & 1], 0);  // U(k - 1, k + 1) before U(k, k + 1)
      if (k + 1 < d->nblk && update(k, k + 1, k + 1, sp, false)) return 1;
      if (k + 2 < d->nblk) {
        cudaStreamWaitEvent(d->s_aux, d->ev_ready[k & 1], 0);
        if (k > 0) cudaStreamWaitEvent(d->s_aux, d->ev_main[(k - 1) & 1], 0);  // rest(k - 1) has applied panel k - 1 to block k + 2
        if (update(k, k + 2, k + 2, d->s_aux, false)) return 1;
      }
      cudaEventRecord(d->ev_half2[k & 1], d->s_aux);
      continue;
    }
    // the two next block columns on the panel stream (critical path)
    if (k + 1 < d->nblk && owner(k + 1) == me && update(k, k + 1, k + 1, sp, false)) return 1;
    if (k + 2 < d->nblk && owner(k + 2) == me) {
      if (k > 0) cudaStreamWaitEvent(sp, d->ev_main[(k - 1) & 1], 0);  // rest(k - 1) has applied panel k - 1 to block k + 2
      if (update(k, k + 2, k + 2, sp, false)) return 1;
    }
  }
  if (use_aux && d->nblk >= 1) cudaStreamWaitEvent(sp, d->ev_half2[(d->nblk - 1) & 1], 0);
  // the tail ran on the panel stream: join
  cudaEventRecord(d->ev_misc, sp);
  cudaStreamWaitEvent(sm, d->ev_misc, 0);
  return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

// Solves L L^T x = b in place (b on the device, length n) with the packed factor, on s_main.
int dense_solve(DenseCtx* d, double* b) {
  const int n = d->n, NB = d->NB;
  if (n == 0) return 0;
  cudaStream_t sm = d->s_main;
  auto linv_of = [&](int t) {
    const int k = (t * PT) / NB, sub = (t * PT - k * NB) / PT;
    return d->Lpack + d->panel_off[k] + static_cast<int64_t>(d->panel_h[k]) * NB + static_cast<int64_t>(sub) * PT * PT;
  };
  static bool configured_dev[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!configured_dev[dev & 63]) {
    cudaFuncSetAttribute(trsv_forward2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kTs2Smem));
    cudaFuncSetAttribute(trsv_backward2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kTs2Smem));
    configured_dev[dev & 63] = true;
  }
  const int T = d->ntiles;
  // forward: y_0 = Linv_0 b_0, then one launch per tile that has rows below it
  trsv_store_tile_kernel<<<1, PT, 0, sm>>>(linv_of(0), b, std::min(PT, n), d->tmp, false);
  for (int t = 0; t + 1 < T; ++t) {
    const int c0 = t * PT, k = c0 / NB, off = c0 - k * NB;
    const int rows_below = n - c0 - PT;
    const double* Lp = d->Lpack + d->panel_off[k] + static_cast<int64_t>(off) * d->panel_h[k] + off + PT;
    trsv_forward2_kernel<<<(rows_below + PT - 1) / PT, TS2_THREADS, kTs2Smem, sm>>>(Lp, d->panel_h[k], rows_below, d->tmp + c0,
                                                                                    b + c0 + PT, linv_of(t + 1), d->tmp + c0 + PT);
  }
  // backward: x_{T-1} = Linv^T y_{T-1}, then one launch per tile that has columns to its left
  {
    const int r0 = (T - 1) * PT;
    trsv_store_tile_kernel<<<1, PT, 0, sm>>>(linv_of(T - 1), d->tmp + r0, std::min(PT, n - r0), b + r0, true);
  }
  for (int t = T - 1; t >= 1; --t) {
    const int r0 = t * PT, live = std::min(PT, n - r0);
    trsv_backward2_kernel<<<r0 / PT, TS2_THREADS, kTs2Smem, sm>>>(d->Lpack, d->d_panel_off, d->d_panel_h, NB, r0, live, b + r0,
                                                                  d->tmp, linv_of(t - 1), b + r0 - PT);
  }
  return cudaGetLastError() == cudaSuccess ? 0 : 1;
}


// ------------------------------------------------------------------------------------------
// matrix-vector products with the off-diagonal block B [rows][ld] row-major (reduced right-hand side and
// back-substitution of the Schur solve, LV/lm_optimizer.h:1319,1366-1367). Fixed summation order.
// ------------------------------------------------------------------------------------------
// y[c] += alpha * sum_r B[r][c] u[r]: stage 1 sums 128-row slabs (coalesced along c), stage 2 the slabs
constexpr int GV_ROWS = 128;
__global__ void gemv_t_stage1_kernel(int rows, int cols, int64_t ld, const double* __restrict__ B,
                                     const double* __restrict__ u, double* __restrict__ partial) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int r0 = blockIdx.y * GV_ROWS, r1 = min(rows, r0 + GV_ROWS);
  if (c >= cols) return;
  double a0 = 0.0, a1 = 0.0;
  int r = r0;
  for (; r + 1 < r1; r += 2) {
    a0 = fma(B[static_cast<int64_t>(r) * ld + c], u[r], a0);
    a1 = fma(B[static_cast<int64_t>(r + 1) * ld + c], u[r + 1], a1);
  }
  if (r < r1) a0 = fma(B[static_cast<int64_t>(r) * ld + c], u[r], a0);
  partial[static_cast<int64_t>(blockIdx.y) * cols + c] = a0 + a1;
}
__global__ void gemv_t_stage2_kernel(int slabs, int cols, const double* __restrict__ partial, double alpha,
                                     double* __restrict__ y) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  double a = 0.0;
  for (int s = 0; s < slabs; ++s) a += partial[static_cast<int64_t>(s) * cols + c];
  y[c] = fma(alpha, a, y[c]);
}
// t[r] = sum_c B[r][c] x[c]: one warp per row
__global__ void gemv_n_kernel(int rows, int cols, int64_t ld, const double* __restrict__ B, const double* __restrict__ x,
                              double* __restrict__ t) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const double* row = B + static_cast<int64_t>(warp) * ld;
  double a0 = 0.0, a1 = 0.0;
  int c = lane;
  for (; c + 32 < cols; c += 64) {
    a0 = fma(row[c], x[c], a0);
    a1 = fma(row[c + 32], x[c + 32], a1);
  }
  if (c < cols) a0 = fma(row[c], x[c], a0);
  double a = a0 + a1;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if (lane == 0) t[warp] = a;
}
int gemv_t_partial_size(int rows, int cols) { return ((rows + GV_ROWS - 1) / GV_ROWS) * std::max(cols, 1); }
void launch_gemv_t(int rows, int cols, int64_t ld, const double* B, const double* u, double alpha, double* y, double* partial,
                   cudaStream_t s) {
  if (rows <= 0 || cols <= 0) return;
  const int slabs = (rows + GV_ROWS - 1) / GV_ROWS;
  dim3 grid((cols + 255) / 256, slabs);
  gemv_t_stage1_kernel<<<grid, 256, 0, s>>>(rows, cols, ld, B, u, partial);
  gemv_t_stage2_kernel<<<(cols + 255) / 256, 256, 0, s>>>(slabs, cols, partial, alpha, y);
}
void launch_gemv_n(int rows, int cols, int64_t ld, const double* B, const double* x, double* t, cudaStream_t s) {
  if (rows <= 0) return;
  gemv_n_kernel<<<(rows * 32 + 255) / 256, 256, 0, s>>>(rows, cols, ld, B, x, t);
}

}  // namespace b200ba
