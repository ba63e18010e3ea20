#!/usr/bin/env python
"""Device time of the stand-alone blocked Cholesky (`b200ba_dense_cholesky_solve`) at the bench's dense size.

    python scripts/dense_mma_timing.py [--lib PATH ...] [--n 13080] [--nb 512] [--reps 10] [--rounds 1]

Factorisation and triangular-solve device times (CUDA events inside the library) of a seeded SPD matrix,
median of --reps calls after two warm-up calls. Every library is timed in a subprocess of its own, so that
two builds (e.g. a parent commit's `libb200ba.so` and the current one) can be alternated in one run
(--rounds > 1 repeats the alternation). Default: the in-tree library.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def spd_matrix(n: int, seed: int = 0):
    """Symmetric random matrix shifted past its spectral radius: SPD, condition number about 10, O(n^2) to make."""
    import numpy as np
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((n, n))
    A += A.T
    A *= 0.5
    A[np.diag_indices(n)] += 1.2 * np.sqrt(2.0 * n)
    return A, rng.standard_normal(n)


def _child(lib_path: str, n: int, nb: int, reps: int) -> None:
    import numpy as np
    from camera_calibration_b200 import cabi
    lib = cabi.load_library(lib_path)
    A, b = spd_matrix(n)
    x = np.zeros(n)
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    fac, sol = [], []
    for i in range(reps + 2):
        fm, sm = C.c_double(0), C.c_double(0)
        rc = lib.b200ba_dense_cholesky_solve(0, n, nb, dp(A), dp(b), dp(x), C.byref(fm), C.byref(sm))
        if rc != 0:
            raise RuntimeError(f"b200ba_dense_cholesky_solve returned {rc}")
        if i >= 2:
            fac.append(fm.value)
            sol.append(sm.value)
    r = A @ x - b
    inf = lambda v: np.linalg.norm(v, np.inf)
    berr = float(inf(r) / (inf(A) * inf(x) + inf(b)))  # normwise backward error in the infinity norm
    print(json.dumps({"lib": lib_path, "n": n, "nb": nb, "reps": reps, "factor_ms_median": float(np.median(fac)),
                      "factor_ms_min": min(fac), "factor_ms_max": max(fac), "solve_ms_median": float(np.median(sol)),
                      "backward_error": berr}), flush=True)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=None, help="libb200ba.so to time (repeatable)")
    ap.add_argument("--n", type=int, default=13080)
    ap.add_argument("--nb", type=int, default=512)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    libs = args.lib or [os.path.join(ROOT, "camera_calibration_b200", "csrc", "libb200ba.so")]
    if args.child:
        _child(libs[0], args.n, args.nb, args.reps)
        return 0
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card}", flush=True)
    for _ in range(args.rounds):
        for lib in libs:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--lib", os.path.abspath(lib),
                                "--n", str(args.n), "--nb", str(args.nb), "--reps", str(args.reps)],
                               capture_output=True, text=True)
            if r.returncode != 0:
                sys.stderr.write(r.stdout + r.stderr)
                return r.returncode
            print(r.stdout.strip(), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
