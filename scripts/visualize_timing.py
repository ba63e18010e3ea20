"""Device time of the calibration visualisation (b200ba_visualize_camera: VisualizeCameraModel of a radtan camera) at
752 x 480 (EuRoC), 2050 x 1450 (config 2) and 4000 x 3000, with the orientation's window sum split out.

    python scripts/visualize_timing.py [--repeats 20]

Prints the GPU's name and power limit, then one line per size: the median device time of `repeats` calls after two
warm-up calls (CUDA events around the call's kernels, as b200ba_visualize_camera reports it), and, from a second run of
`repeats` calls under torch.profiler, the mean time of each kernel: radtan8_window_kernel (the window's un-projections),
radtan8_orientation_kernel (the row-major window sum on one thread and the rotation) and visualize_camera_kernel (every
pixel). Needs a GPU; there is no CPU fallback.
"""
import argparse
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from camera_calibration_b200 import api  # noqa: E402

CASES = [
    ("752 x 480", 752, 480, [-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05, 458.654, 457.296, 367.215, 248.375]),
    ("2050 x 1450", 2050, 1450, [-0.12, 0.03, 1e-4, -2e-4, 1500.0, 1502.0, 1025.3, 724.8]),
    ("4000 x 3000", 4000, 3000, [-0.12, 0.03, 1e-4, -2e-4, 2900.0, 2905.0, 2001.3, 1498.7]),
]
KERNELS = ("radtan8_window_kernel", "radtan8_orientation_kernel", "visualize_camera_kernel")


def kernel_means_us(w, h, params, repeats):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(repeats):
            api.VisualizeCameraModel(w, h, params)
    out = {}
    for e in prof.key_averages():
        for k in KERNELS:
            if k in e.key:
                total = getattr(e, "self_device_time_total", None)
                if total is None:
                    total = e.self_cuda_time_total
                out[k] = total / e.count
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"GPU: {smi}")
    for name, w, h, params in CASES:
        for _ in range(2):
            api.VisualizeCameraModel(w, h, params)
        times = [api.VisualizeCameraModel(w, h, params)[3] for _ in range(args.repeats)]
        window = (w - min(w - 1, w // 2 + 11)) * (min(h - 1, h // 2 + 10) - max(0, h // 2 - 10) + 1)
        k = kernel_means_us(w, h, params, args.repeats)
        print(f"{name:12s}: {np.median(times):8.3f} ms (min {min(times):.3f}, max {max(times):.3f}); window {window} "
              f"pixels; per kernel (mean, us): " + ", ".join(f"{n} {k.get(n, float('nan')):.1f}" for n in KERNELS))


if __name__ == "__main__":
    main()
