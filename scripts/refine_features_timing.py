"""Times b200ba_refine_features on the features of the --render_synthetic_dataset workload: the pattern of
tests/golden/pattern seen from 500 poses of b200ba_synthetic_poses (seed 0), at the tool's 640 x 480 camera
(fx = fy = 480) and at 2050 x 1450 (fx = fy = 1450, cx = 1025, cy = 725), images rendered on the device, every valid
feature predicted 3 px or less from its exact position (synthetic.pattern_feature_predictions).

Prints the GPU and its power limit, then per size and refinement type (h = 10, and h = 15 for intensities) the
feature count, the median device time of 20 calls after warm-up (each call refines every feature of the 500 images),
the accepted share, and the time of the reference-order restatement (tests/refine_features_oracle.cc, -O2, one CPU
thread) on 40 of the same features, scaled to all of them.

    python scripts/refine_features_timing.py
"""
import ctypes as C
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from camera_calibration_b200 import api, build, cabi, io, pipeline, synthetic  # noqa: E402

N_IMAGES, N_CALLS, N_RESTATED = 500, 20, 40
RUNS = (("gradients_xy", 10), ("gradient_magnitude", 10), ("intensities", 10), ("no_refinement", 10),
        ("intensities", 15))


def main():
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip())
    so = os.path.join(tempfile.mkdtemp(), "librefine_oracle.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I",
                           os.path.join(os.path.dirname(os.path.dirname(build.NVCC)), "include"),
                           os.path.join(ROOT, "tests", "refine_features_oracle.cc"), "-o", so])
    lib = C.CDLL(so)
    lib.oracle_refine.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                  C.c_int64, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    base = os.path.join(ROOT, "tests", "golden", "pattern", pipeline.SYNTHETIC_PATTERN_NAME)
    pattern, image = io.LoadPatternYAML(base + ".yaml"), io.ReadPNG(base + ".png")
    pattern_size = (image.shape[1], image.shape[0])
    p = api._pattern_struct(pattern)
    for size, k in (((640, 480), [480, 480, 320, 240]), ((2050, 1450), [1450, 1450, 1025, 725])):
        k = np.array(k, np.float32)
        poses, _ = api.SyntheticPoses(pattern, pattern_size, size, k, N_IMAGES, 0)
        gt = synthetic.pattern_feature_predictions(pattern, pattern_size, poses, k, size, 3.0, 0)
        rec = api._prediction_records(gt["image"], gt["prediction"], gt["pattern_coordinate"],
                                      gt["local_pixel_tr_pattern"])
        images, _ = api.RenderPatternImages(pattern, image, size, k, poses)
        sub = np.ascontiguousarray(rec[np.random.default_rng(0).permutation(len(rec))[:N_RESTATED]])
        for name, h in RUNS:
            for _ in range(3):
                xy, cost, st, _ = api.RefineFeatures(pattern, images, rec, name, h)
            times = [api.RefineFeatures(pattern, images, rec, name, h)[3] for _ in range(N_CALLS)]
            s = api.FeatureSamples(h)
            o_xy = np.zeros((N_RESTATED, 2), np.float32)
            o_cost = np.zeros(N_RESTATED, np.float32)
            o_status = np.zeros(N_RESTATED, np.int32)
            t0 = time.perf_counter()
            lib.oracle_refine(C.byref(p), images.ctypes.data, size[0], size[1], s.ctypes.data, len(s), h,
                              cabi.REFINEMENT_TYPES[name], N_RESTATED, sub.ctypes.data, 0, o_xy.ctypes.data,
                              o_cost.ctypes.data, o_status.ctypes.data)
            cpu = time.perf_counter() - t0
            print(f"{size[0]}x{size[1]} {name} h={h}: {len(rec)} features of {N_IMAGES} images, device median "
                  f"{np.median(times):.2f} ms (min {min(times):.2f}, max {max(times):.2f}), accepted "
                  f"{(st == 0).mean() * 100:.1f} %; restatement {cpu * 1e3 / N_RESTATED:.1f} ms per feature on one "
                  f"CPU thread ({N_RESTATED} features), {cpu / N_RESTATED * len(rec):.0f} s scaled to all")


if __name__ == "__main__":
    main()
