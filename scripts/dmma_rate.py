#!/usr/bin/env python
"""Register-resident FP64 tensor-core throughput of the four f64 `mma.sync` shapes on one GPU.

    python scripts/dmma_rate.py [--iters N] [--json PATH]

Every warp runs CHAINS independent accumulator chains of one shape with no memory traffic inside the
timed loop, so what is measured is the rate at which the SM issues and retires that DMMA shape. The
geometries are those of `dgemm_nt_kernel`: 2 CTAs of 256 threads (128 x 64 tiles) or 1 CTA of 512 threads
(128 x 128 tiles) per SM, i.e. 16 warps, plus 8 warps per SM (one 256-thread CTA: what is left while the
other CTA of an SM runs its epilogue). FMA/clk/SM comes from the SM's own `clock64()` span over all CTAs resident on it;
TFLOP/s from CUDA events around the launch. The card name, power limit and SM clock are read with
`nvidia-smi` in the same call.

The kernel is compiled at run time with the flags of camera_calibration_b200/build.py into a temporary
directory (nothing is written to the tree).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SRC = r"""
#include <cstdio>
#include <cuda_runtime.h>

template <int S> struct Frag;  // S = 0: m8n8k4, 1: m16n8k4, 2: m16n8k8, 3: m16n8k16
template <> struct Frag<0> { static constexpr int NA = 1, NB = 1, NC = 2, FMA = 8 * 8 * 4; };
template <> struct Frag<1> { static constexpr int NA = 2, NB = 1, NC = 4, FMA = 16 * 8 * 4; };
template <> struct Frag<2> { static constexpr int NA = 4, NB = 2, NC = 4, FMA = 16 * 8 * 8; };
template <> struct Frag<3> { static constexpr int NA = 8, NB = 4, NC = 4, FMA = 16 * 8 * 16; };

template <int S>
__device__ __forceinline__ void mma(double* c, const double* a, const double* b);
template <>
__device__ __forceinline__ void mma<0>(double* c, const double* a, const double* b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(c[0]), "+d"(c[1]) : "d"(a[0]), "d"(b[0]));
}
template <>
__device__ __forceinline__ void mma<1>(double* c, const double* a, const double* b) {
  asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(b[0]));
}
template <>
__device__ __forceinline__ void mma<2>(double* c, const double* a, const double* b) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
               : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}
template <>
__device__ __forceinline__ void mma<3>(double* c, const double* a, const double* b) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
               "{%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
               : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                 "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

constexpr int CHAINS = 8;  // independent accumulators per warp

template <int S>
__global__ void __launch_bounds__(512) dmma_rate_kernel(int iters, double seed, double* out, long long* clk) {
  using F = Frag<S>;
  double a[F::NA], b[F::NB], c[CHAINS][F::NC];
  for (int i = 0; i < F::NA; ++i) a[i] = seed * (threadIdx.x + i);
  for (int i = 0; i < F::NB; ++i) b[i] = seed * (threadIdx.x - i);
  for (int q = 0; q < CHAINS; ++q)
    for (int i = 0; i < F::NC; ++i) c[q][i] = 0.0;
  __syncthreads();
  const long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int q = 0; q < CHAINS; ++q) mma<S>(c[q], a, b);
  }
  __syncthreads();
  const long long t1 = clock64();
  double s = 0.0;
  for (int q = 0; q < CHAINS; ++q)
    for (int i = 0; i < F::NC; ++i) s += c[q][i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0) {
    unsigned smid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    clk[3 * blockIdx.x] = t0;
    clk[3 * blockIdx.x + 1] = t1;
    clk[3 * blockIdx.x + 2] = smid;
  }
}

template <int S>
static int run_shape(int threads, int ctas_per_sm, int iters, float* ms, long long* clk_host, int* n_sm, int* fma) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 1;
  cudaDeviceGetAttribute(n_sm, cudaDevAttrMultiProcessorCount, dev);
  int resident = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, dmma_rate_kernel<S>, threads, 0);
  if (resident < ctas_per_sm) return 2;
  const int grid = *n_sm * ctas_per_sm;
  double* out = nullptr;
  long long* clk = nullptr;
  if (cudaMalloc(&out, sizeof(double) * grid * threads) != cudaSuccess) return 3;
  if (cudaMalloc(&clk, sizeof(long long) * 3 * grid) != cudaSuccess) return 3;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  dmma_rate_kernel<S><<<grid, threads>>>(iters / 10 + 1, 1e-3, out, clk);  // warm-up
  cudaEventRecord(e0);
  dmma_rate_kernel<S><<<grid, threads>>>(iters, 1e-3, out, clk);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  cudaEventElapsedTime(ms, e0, e1);
  cudaMemcpy(clk_host, clk, sizeof(long long) * 3 * grid, cudaMemcpyDeviceToHost);
  *fma = Frag<S>::FMA * CHAINS;  // per warp per iteration
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaFree(out);
  cudaFree(clk);
  return cudaGetLastError() == cudaSuccess ? 0 : 4;
}

extern "C" __attribute__((visibility("default"))) int dmma_rate(int shape, int threads, int ctas_per_sm, int iters,
                                                                float* ms, long long* clk, int* n_sm, int* fma) {
  switch (shape) {
    case 0: return run_shape<0>(threads, ctas_per_sm, iters, ms, clk, n_sm, fma);
    case 1: return run_shape<1>(threads, ctas_per_sm, iters, ms, clk, n_sm, fma);
    case 2: return run_shape<2>(threads, ctas_per_sm, iters, ms, clk, n_sm, fma);
    case 3: return run_shape<3>(threads, ctas_per_sm, iters, ms, clk, n_sm, fma);
  }
  return 5;
}
"""

SHAPES = ["m8n8k4", "m16n8k4", "m16n8k8", "m16n8k16"]
# (threads per CTA, CTAs per SM): the two occupancies of dgemm_nt_kernel
GEOMETRIES = [(256, 1), (256, 2), (512, 1)]


def _compile(tmp: str) -> str:
    from camera_calibration_b200 import build
    cu = os.path.join(tmp, "dmma_rate.cu")
    so = os.path.join(tmp, "libdmma_rate.so")
    with open(cu, "w") as f:
        f.write(SRC)
    r = subprocess.run([build.NVCC] + build.FLAGS + ["-shared", cu, "-o", so], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed:\n{r.stdout}\n{r.stderr}")
    return so


def _card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=10).stdout.strip()
    f = [v.strip() for v in out.split(",")]
    return dict(zip(q.split(","), f)) if len(f) == 4 else {"nvidia-smi": out}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20000)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        lib = C.CDLL(_compile(tmp))
        lib.dmma_rate.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_float),
                                  C.POINTER(C.c_longlong), C.POINTER(C.c_int), C.POINTER(C.c_int)]
        rows = []
        for threads, per_sm in GEOMETRIES:
            for s, name in enumerate(SHAPES):
                ms, n_sm, fma = C.c_float(0), C.c_int(0), C.c_int(0)
                clk = (C.c_longlong * (3 * 1024 * per_sm))()
                rc = lib.dmma_rate(s, threads, per_sm, args.iters, C.byref(ms), clk, C.byref(n_sm), C.byref(fma))
                if rc != 0:
                    raise RuntimeError(f"dmma_rate({name}, {threads}, {per_sm}) failed with {rc}")
                grid = n_sm.value * per_sm
                spans = {}
                for b in range(grid):
                    t0, t1, sm = clk[3 * b], clk[3 * b + 1], clk[3 * b + 2]
                    lo, hi, cnt = spans.get(sm, (t0, t1, 0))
                    spans[sm] = (min(lo, t0), max(hi, t1), cnt + 1)
                warps = threads // 32
                fma_sm_clk = [cnt * warps * args.iters * fma.value / (hi - lo) for lo, hi, cnt in spans.values()]
                total_fma = grid * warps * args.iters * fma.value
                rows.append({"shape": name, "threads": threads, "ctas_per_sm": per_sm, "warps_per_sm": warps * per_sm,
                             "fma_per_clk_sm": sorted(fma_sm_clk)[len(fma_sm_clk) // 2],
                             "tflops": 2.0 * total_fma / (ms.value * 1e-3) / 1e12, "ms": ms.value})
        card = _card()
    print(f"card: {card}")
    print(f"{'shape':>9} {'warps/SM':>8} {'FMA/clk/SM':>11} {'TFLOP/s':>8}")
    for r in rows:
        print(f"{r['shape']:>9} {r['warps_per_sm']:>8} {r['fma_per_clk_sm']:>11.1f} {r['tflops']:>8.2f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card, "rows": rows}, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
