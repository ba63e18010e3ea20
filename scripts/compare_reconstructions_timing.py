"""Device time of the reconstruction comparison's direction sweep (b200ba_compare_reconstructions), at the tool's pixel
step 10 and at step 1, for the config-2 camera (2050 x 1450, 84 x 60 grid) and a 4000 x 3000 camera, each compared
central-generic against central-generic and central-generic against OpenCV.

    python scripts/compare_reconstructions_timing.py [--repeats 20]

Prints the GPU's name and power limit, then one line per case: the median device time of `repeats` calls after two
warm-up calls (CUDA events around the sweep, as b200ba_compare_reconstructions reports it) and the sample pixels both
models un-project. Needs a GPU; there is no CPU fallback.
"""
import argparse
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from camera_calibration_b200 import api, cabi, synthetic  # noqa: E402


def cg_model(width, height, gw, gh, seed):
    """A smooth pinhole-with-distortion central-generic model of a width x height camera."""
    rng = np.random.default_rng(seed)
    f = 0.8 * width
    ys, xs = np.meshgrid(np.arange(gh), np.arange(gw), indexing="ij")
    cam = cabi.Camera()
    cam.calibration_max_x, cam.calibration_max_y, cam.grid_width, cam.grid_height = width - 1, height - 1, gw, gh
    px = synthetic.grid_point_to_pixel(cam, xs, ys)
    u = (px[0] - width / 2) / f
    v = (px[1] - height / 2) / f
    r2 = u * u + v * v
    k = 1 - 0.08 * r2 + 1e-4 * rng.standard_normal(u.shape)
    g = np.stack([u * k, v * k, np.ones_like(u)], axis=-1)
    m = api.CentralGenericModel(gw, gh, 0, 0, width - 1, height - 1, width, height)
    m.SetGrid(g / np.linalg.norm(g, axis=-1, keepdims=True))
    return m


def opencv_model(width, height):
    f = 0.8 * width
    return api.CentralOpenCVModel(width, height, [f, f, width / 2, height / 2, -0.08, 0.01, 0, 0, 0, 0, 1e-4, -1e-4])


def state(model, n=50, seed=0):
    rng = np.random.default_rng(seed)
    st = api.BAState()
    st.intrinsics = [model]
    q = rng.standard_normal((n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    st.rig_tr_global = np.concatenate([q, rng.uniform(-2, 2, (n, 3))], axis=1)
    st.image_used = [True] * n
    st.camera_tr_rig = np.array([synthetic.IDENTITY_POSE])
    return st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"GPU: {smi}")
    cases = [("config 2", 2050, 1450, 84, 60), ("4000 x 3000", 4000, 3000, 160, 120)]
    for name, w, h, gw, gh in cases:
        cg = cg_model(w, h, gw, gh, 1)
        for other_name, other in (("CG", cg_model(w, h, gw, gh, 2)), ("OpenCV", opencv_model(w, h))):
            s1, s2 = state(cg, seed=3), state(other, seed=3)
            for step in (10, 1):
                for _ in range(2):
                    api.CompareReconstructions(s1, s2, pixel_step=step)
                times, pairs = [], 0
                for _ in range(args.repeats):
                    r, ms = api.CompareReconstructions(s1, s2, pixel_step=step)
                    times.append(ms)
                    pairs = r.direction_pairs
                print(f"{name:12s} CG vs {other_name:6s} step {step:2d}: {np.median(times):9.3f} ms "
                      f"(min {min(times):.3f}, max {max(times):.3f}), {pairs} direction pairs")


if __name__ == "__main__":
    main()
