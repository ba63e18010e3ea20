"""Device time of b200ba_fitting_images (the --compare_calibrations comparison with its five images) next to
b200ba_compare_models alone, on the two cases of compare_timing.py:
  * config 2: the ground-truth model of synthetic.make_problem(2) against its perturbed initial intrinsics
    (2050 x 1450, 84 x 60 grid), and
  * a 4000 x 3000 pinhole camera (162 x 122 grid) against a seeded perturbed copy.
The two calls alternate after warm-up, so that both see the same clocks. Prints the card's name and power limit
beside the result, then one JSON line.

    python scripts/fitting_images_timing.py [--repeats 20] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402

from camera_calibration_b200 import api  # noqa: E402
from compare_timing import config2_pair, large_pair  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print(f"card: {card[0] if card else 'unknown'}")
    results = []
    for name, a, b in (config2_pair(), large_pair()):
        for _ in range(args.warmup):
            api.CompareModels(a, b)
            api.FittingImages(a, b)
        compare_ms, images_ms = [], []
        for _ in range(args.repeats):
            compare_ms.append(api.CompareModels(a, b)[3])
            images_ms.append(api.FittingImages(a, b)[2])
        compare_ms, images_ms = np.array(compare_ms), np.array(images_ms)
        n = a.width() * a.height()
        res = {"case": name, "pixels": n, "repeats": args.repeats,
               "compare_models_ms_median": float(np.median(compare_ms)),
               "fitting_images_ms_median": float(np.median(images_ms)),
               "fitting_images_ms_min": float(images_ms.min()), "fitting_images_ms_max": float(images_ms.max()),
               "images_added_ms": float(np.median(images_ms) - np.median(compare_ms))}
        print(f"{name} ({n} pixels): b200ba_fitting_images median {res['fitting_images_ms_median']:.3f} ms device time "
              f"(min {images_ms.min():.3f}, max {images_ms.max():.3f}); b200ba_compare_models alone "
              f"{res['compare_models_ms_median']:.3f} ms; the images add {res['images_added_ms']:.3f} ms "
              f"({args.repeats} alternated repeats)")
        results.append(res)
    print(json.dumps({"card": card[0] if card else None, "results": results}))


if __name__ == "__main__":
    main()
