"""Times b200ba_render_pattern_images on the tool's workload: the pattern of tests/golden/pattern seen from 500 poses
of b200ba_synthetic_poses (seed 0), at the tool's 640 x 480 camera (fx = fy = 480) and at 2050 x 1450 (fx = fy = 1450,
cx = 1025, cy = 725).

Prints the GPU and its power limit, the median device time of 20 calls after warm-up (each call renders all 500
images), and the time of the sequential restatement (tests/render_synthetic_oracle.cc, -O2, one CPU thread) on the
first 20 of the same images, with its per-image time scaled to 500 images. The first 20 images of both agree byte
for byte. With --profile, also the mean time per call of each kernel under torch.profiler (in a run of its own:
synth_project_kernel projects and bins the polygons, synth_render_kernel clips and composes every pixel).

    python scripts/render_synthetic_timing.py [--profile]
"""
import argparse
import ctypes as C
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from camera_calibration_b200 import api, io, pipeline  # noqa: E402

N_IMAGES, N_CALLS, N_RESTATED = 500, 20, 20
KERNELS = ("synth_project_kernel", "synth_render_kernel")


def kernel_ms_per_call(call, repeats=5):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(repeats):
            call()
    out = {}
    for e in prof.key_averages():
        for k in KERNELS:
            if k in e.key:
                total = getattr(e, "self_device_time_total", None)
                if total is None:
                    total = e.self_cuda_time_total
                out[k] = out.get(k, 0.0) + total / 1e3 / repeats
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip())
    tmp = tempfile.mkdtemp()
    so = os.path.join(tmp, "liboracle.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "render_synthetic_oracle.cc"),
                           "-o", so])
    lib = C.CDLL(so)
    base = os.path.join(ROOT, "tests", "golden", "pattern", pipeline.SYNTHETIC_PATTERN_NAME)
    pattern, image = io.LoadPatternYAML(base + ".yaml"), io.ReadPNG(base + ".png")
    pattern_size = (image.shape[1], image.shape[0])
    for size, k in (((640, 480), [480, 480, 320, 240]), ((2050, 1450), [1450, 1450, 1025, 725])):
        k = np.array(k, np.float32)
        poses, attempts = api.SyntheticPoses(pattern, pattern_size, size, k, N_IMAGES, 0)
        for _ in range(3):
            images, _ = api.RenderPatternImages(pattern, image, size, k, poses)
        if args.profile:
            ms = kernel_ms_per_call(lambda: api.RenderPatternImages(pattern, image, size, k, poses))
            print(f"{size[0]}x{size[1]}: per call (mean of 5, ms): " +
                  ", ".join(f"{n} {ms.get(n, float('nan')):.2f}" for n in KERNELS))
            continue
        times = [api.RenderPatternImages(pattern, image, size, k, poses)[1] for _ in range(N_CALLS)]
        ref = np.zeros((N_RESTATED, size[1], size[0]), np.uint8)
        p = api._pattern_struct(pattern)
        sub = np.ascontiguousarray(poses[:N_RESTATED])
        t0 = time.perf_counter()
        lib.oracle_render(C.byref(p), C.c_void_p(image.ctypes.data), C.c_int32(pattern_size[0]),
                          C.c_int32(pattern_size[1]), C.c_int32(size[0]), C.c_int32(size[1]),
                          C.c_void_p(k.ctypes.data), C.c_int64(N_RESTATED), C.c_void_p(sub.ctypes.data),
                          C.c_void_p(ref.ctypes.data), None, None)
        cpu = time.perf_counter() - t0
        print(f"{size[0]}x{size[1]}: {N_IMAGES} images ({int(attempts.sum())} pose draws), device median "
              f"{np.median(times):.2f} ms (min {min(times):.2f}, max {max(times):.2f}); restatement "
              f"{cpu * 1e3 / N_RESTATED:.0f} ms per image on one CPU thread ({N_RESTATED} images), "
              f"{cpu / N_RESTATED * N_IMAGES:.0f} s scaled to {N_IMAGES}; first {N_RESTATED} identical: "
              f"{bool(np.array_equal(images[:N_RESTATED], ref))}")


if __name__ == "__main__":
    main()
