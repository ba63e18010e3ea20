"""Device time of b200ba_compare_models (the --compare_calibrations comparison: two B-spline un-projections
and one projection LM from the centre per pixel, then the statistics) for
  * config 2: the ground-truth model of synthetic.make_problem(2) against its perturbed initial intrinsics
    (2050 x 1450, 84 x 60 grid), and
  * a 4000 x 3000 pinhole camera (162 x 122 grid) against a seeded perturbed copy,
after warm-up, over repeats. Prints the card's name and power limit beside the result, then one JSON line.
``--with-oracle`` also times the sequential CPU oracle (un-project, un-project, project per pixel, as the
reference's loop does) over the same pixels.

    python scripts/compare_timing.py [--repeats 20] [--warmup 3] [--with-oracle]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from camera_calibration_b200 import api, cabi, synthetic  # noqa: E402


def _model(cam, grid):
    m = api.CentralGenericModel(cam.grid_width, cam.grid_height, cam.calibration_min_x, cam.calibration_min_y,
                                cam.calibration_max_x, cam.calibration_max_y, cam.width, cam.height)
    m.set_flat_intrinsics(np.asarray(grid, dtype=np.float64).reshape(-1))
    return m


def config2_pair():
    sp = synthetic.make_problem(2)
    cam = sp.problem.cameras[0]
    return "config2", _model(cam, sp.gt_state.intrinsics[0]), _model(cam, sp.init_state.intrinsics[0])


def large_pair():
    cam = synthetic.make_generic_camera(cabi.MODEL_CENTRAL_GENERIC, 4000, 3000, 25)
    a = synthetic.pinhole_direction_grid(cam, 1100.0 * 4000 / 2050)
    rng = np.random.default_rng(4000)
    b = a + 1e-3 * rng.standard_normal(a.shape)
    return "4000x3000", _model(cam, a), _model(cam, b / np.linalg.norm(b, axis=-1, keepdims=True))


def oracle_seconds(a, b):
    """Host wall time of the sequential CPU oracle over every pixel of the image."""
    from oracle import oracle
    oracle.build()
    ys, xs = np.meshgrid(np.arange(a.height()), np.arange(a.width()), indexing="ij")
    px = np.stack([xs.ravel() + 0.5, ys.ravel() + 0.5], -1)
    t0 = time.perf_counter()
    da, _, ok_a = oracle.unproject(a.c_camera(), a.flat_intrinsics(), px)
    oracle.unproject(b.c_camera(), b.flat_intrinsics(), px)
    oracle.project(b.c_camera(), b.flat_intrinsics(), da[ok_a])
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--with-oracle", action="store_true")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print(f"card: {card[0] if card else 'unknown'}")
    results = []
    for name, a, b in (config2_pair(), large_pair()):
        for _ in range(args.warmup):
            api.CompareModels(a, b)
        ms, wall = [], []
        for _ in range(args.repeats):
            t0 = time.perf_counter()
            report, _, _, m = api.CompareModels(a, b)
            wall.append(time.perf_counter() - t0)
            ms.append(m)
        ms, wall = np.array(ms), np.array(wall)
        n = a.width() * a.height()
        res = {"case": name, "pixels": n, "device_ms_median": float(np.median(ms)), "device_ms_min": float(ms.min()),
               "device_ms_max": float(ms.max()), "call_wall_ms_median": float(np.median(wall)) * 1e3,
               "repeats": args.repeats, "reprojection_error_count": int(report.reprojection_error_count),
               "max_error_norm": report.max_error_norm}
        line = (f"b200ba_compare_models, {name} ({n} pixels): median {res['device_ms_median']:.3f} ms device time "
                f"(min {ms.min():.3f}, max {ms.max():.3f}, {args.repeats} repeats); "
                f"{res['call_wall_ms_median']:.1f} ms wall per call with allocation and copies")
        if args.with_oracle:
            res["oracle_wall_s"] = oracle_seconds(a, b)
            line += f"; sequential CPU oracle {res['oracle_wall_s']:.2f} s wall"
        print(line)
        results.append(res)
    print(json.dumps({"card": card[0] if card else None, "results": results}))


if __name__ == "__main__":
    main()
