"""Device time of b200ba_line_offsets (the centre-point analysis of a non-central camera: one line per pixel of the
calibrated area, the LM fit of the centre, the offsets, the image and the .obj lines) for
  * config 3: the ground-truth model of synthetic.make_problem(3) (1200 x 950, 50 x 40 grid, 1.14 M lines), and
  * a seeded 4000 x 3000 non-central camera (162 x 122 grid, 12 M lines),
as the median over repeats after warm-up. Prints the card's name and power limit beside the result, the per-kernel
device times of one call (torch.profiler: the line pass evaluates both B-spline surfaces once, every LM pass streams
the stored lines), then one JSON line. ``--with-oracle`` also times the sequential restatement of
tests/test_line_offsets.py over the CPU oracle's un-projection.

    python scripts/line_offsets_timing.py [--repeats 20] [--warmup 3] [--with-oracle]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from collections import defaultdict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from camera_calibration_b200 import api, cabi, synthetic  # noqa: E402


def _model(cam, intrinsics):
    m = api.NoncentralGenericModel(cam.grid_width, cam.grid_height, cam.calibration_min_x, cam.calibration_min_y,
                                   cam.calibration_max_x, cam.calibration_max_y, cam.width, cam.height)
    m.set_flat_intrinsics(np.asarray(intrinsics, dtype=np.float64).reshape(-1))
    return m


def config3_model():
    # the camera does not depend on the imageset count or the lattice
    sp = synthetic.make_problem(3, n_imagesets=1, lattice=(25, 20))
    return "config3", _model(sp.problem.cameras[0], sp.gt_state.intrinsics[0])


def large_model():
    cam = synthetic.make_generic_camera(cabi.MODEL_NONCENTRAL_GENERIC, 4000, 3000, 25)
    dg = synthetic.pinhole_direction_grid(cam, 650.0 * 4000 / 1200)
    pg = 0.002 * np.random.default_rng(4000).uniform(-1.0, 1.0, dg.shape)
    return "4000x3000", _model(cam, np.concatenate([dg.reshape(-1), pg.reshape(-1)]))


def kernel_times(model):
    """Device time per kernel name over one call: {name: (calls, total ms)}."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        api.LineOffsets(model)
        torch.cuda.synchronize()
    out = defaultdict(lambda: [0, 0.0])
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and ("line" in e.name or "report_" in e.name):
            key = e.name.split("(")[0].replace("void ", "").replace("b200ba::", "")
            out[key][0] += 1
            out[key][1] += e.time_range.elapsed_us() / 1e3
    return {k: (v[0], v[1]) for k, v in out.items()}


def oracle_seconds(model):
    from oracle import oracle
    from tests import test_line_offsets as t
    oracle.build()
    t0 = time.perf_counter()
    t.restate(oracle, model)
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
    for name, model in (config3_model(), large_model()):
        for _ in range(args.warmup):
            api.LineOffsets(model)
        ms = []
        for _ in range(args.repeats):
            report, _, _, _, m = api.LineOffsets(model)
            ms.append(m)
        ms = np.array(ms)
        n = report.line_count
        res = {"case": name, "lines": int(n), "device_ms_median": float(np.median(ms)), "device_ms_min": float(ms.min()),
               "device_ms_max": float(ms.max()), "repeats": args.repeats,
               "iterations": int(report.num_iterations_performed), "lm_attempts": int(report.lm_attempts),
               "max_line_offset_extent": report.max_line_offset_extent, "center": list(report.center)}
        print(f"b200ba_line_offsets, {name} ({n} lines): median {res['device_ms_median']:.3f} ms device time "
              f"(min {ms.min():.3f}, max {ms.max():.3f}, {args.repeats} repeats); {res['iterations']} iterations, "
              f"{res['lm_attempts']} attempts")
        try:
            kt = kernel_times(model)
        except Exception as e:  # the breakdown is informative only
            print(f"  no per-kernel times: {e!r}")
            kt = {}
        res["kernels_ms"] = {k: {"calls": c, "total_ms": t} for k, (c, t) in sorted(kt.items())}
        for k, (c, t) in sorted(kt.items()):
            print(f"  {k}: {c} calls, {t:.3f} ms total, {t / c:.4f} ms each")
        if args.with_oracle:
            res["oracle_wall_s"] = oracle_seconds(model)
            print(f"  sequential restatement over the CPU oracle: {res['oracle_wall_s']:.2f} s wall")
        results.append(res)
    print(json.dumps({"card": card[0] if card else None, "results": results}))


if __name__ == "__main__":
    main()
