"""Device time of b200ba_localization_accuracy (the --localization_accuracy_test: 15 rejection-sampled points and one
6-DoF pose fit per trial, then the statistics) for 10 000 trials (the reference's count) and 1 000 000 trials, with
the config-2 camera (synthetic.make_problem(2): 2050 x 1450, 84 x 60 grid) against a seeded perturbed copy of its
grid, after warm-up, as the median over repeats. Prints the card's name and power limit beside the result, and the
host time of the sequential CPU oracle of the pose fits (tests/localization_oracle.cc, compiled here into a
temporary directory) for the 10 000 trials' points; then one JSON line.

    python scripts/localization_timing.py [--repeats 20] [--warmup 3]
"""
import argparse
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from camera_calibration_b200 import api, synthetic  # noqa: E402


def config2_pair():
    sp = synthetic.make_problem(2)
    cam = sp.problem.cameras[0]
    models = []
    rng = np.random.default_rng(11)
    g = np.asarray(sp.gt_state.intrinsics[0], dtype=np.float64).reshape(cam.grid_height, cam.grid_width, 3)
    for grid in (g, g + 1e-4 * rng.standard_normal(g.shape)):
        m = api.CentralGenericModel(cam.grid_width, cam.grid_height, cam.calibration_min_x, cam.calibration_min_y,
                                    cam.calibration_max_x, cam.calibration_max_y, cam.width, cam.height)
        m.SetGrid(grid / np.linalg.norm(grid, axis=-1, keepdims=True))
        models.append(m)
    return models


def oracle_seconds(gt, cmp, trials):
    """Host wall time of the sequential oracle's pose fits on the points of `trials` trials (the points are taken
    from the device's samples, un-projected with numpy's float64 arithmetic through the CPU oracle)."""
    from oracle import oracle
    oracle.build()
    _, arrays, _ = api.LocalizationAccuracy(gt, cmp, trials=trials, with_trials=True)
    s = arrays["samples"].reshape(-1, 3)
    px = s[:, :2].astype(np.float64)
    unit = lambda v: v / np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])[:, None]
    sd = s[:, 2].astype(np.float64)[:, None]
    p = np.ascontiguousarray(unit(oracle.unproject(gt.c_camera(), gt.flat_intrinsics(), px)[0]) * sd)
    f = np.ascontiguousarray(unit(unit(oracle.unproject(cmp.c_camera(), cmp.flat_intrinsics(), px)[0]) * sd))
    out = tempfile.mkdtemp(prefix="localization_oracle_")
    try:
        so = os.path.join(out, "liblocalization_oracle.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC",
                               os.path.join(ROOT, "tests", "localization_oracle.cc"), "-o", so])
        lib = C.CDLL(so)
        D = C.POINTER(C.c_double)
        lib.oracle_localization_fit_batch.argtypes = [C.c_int64, D, D, C.c_int, D, D, C.POINTER(C.c_int32)]
        x = np.zeros((trials, 6))
        t0 = time.perf_counter()
        lib.oracle_localization_fit_batch(trials, p.ctypes.data_as(D), f.ctypes.data_as(D), 0, x.ctypes.data_as(D),
                                          None, None)
        return time.perf_counter() - t0
    finally:
        shutil.rmtree(out, True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print(f"card: {card[0] if card else 'unknown'}")
    gt, cmp = config2_pair()
    results = []
    for trials in (10000, 1000000):
        for _ in range(args.warmup):
            api.LocalizationAccuracy(gt, cmp, trials=trials)
        ms, wall = [], []
        for _ in range(args.repeats):
            t0 = time.perf_counter()
            report, _, m = api.LocalizationAccuracy(gt, cmp, trials=trials)
            wall.append(time.perf_counter() - t0)
            ms.append(m)
        ms, wall = np.array(ms), np.array(wall)
        res = {"trials": trials, "device_ms_median": float(np.median(ms)), "device_ms_min": float(ms.min()),
               "device_ms_max": float(ms.max()), "call_wall_ms_median": float(np.median(wall)) * 1e3,
               "repeats": args.repeats, "average_error_mm": 1000 * report.average_error,
               "median_error_mm": 1000 * report.median_error, "mean_iterations": report.total_iterations / trials,
               "max_iterations": int(report.max_iterations), "redraws": int(report.redraws)}
        line = (f"b200ba_localization_accuracy, config 2, {trials} trials: median {res['device_ms_median']:.3f} ms "
                f"device time (min {ms.min():.3f}, max {ms.max():.3f}, {args.repeats} repeats); "
                f"{res['call_wall_ms_median']:.1f} ms wall per call with allocation and copies; "
                f"average {res['average_error_mm']:.6g} mm, median {res['median_error_mm']:.6g} mm, "
                f"{res['mean_iterations']:.2f} iterations per fit (max {res['max_iterations']})")
        if trials == 10000:
            res["oracle_wall_s"] = oracle_seconds(gt, cmp, trials)
            line += f"; sequential CPU oracle of the fits {res['oracle_wall_s']:.3f} s wall"
        print(line)
        results.append(res)
    print(json.dumps({"card": card[0] if card else None, "results": results}))


if __name__ == "__main__":
    main()
