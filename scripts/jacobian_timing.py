"""Device time of the residual / Jacobian kernel's main pass at full config 2 (955 157 observations, one
central-generic camera, 84 x 60 grid): ``BundleAdjuster.timings().jacobian_kernel_ms`` per launch over
repeated evaluations with Jacobians, after warm-up (the first evaluation starts every projection cold and is
not timed). Prints the card's name and power limit beside the result, then one JSON line.

    python scripts/jacobian_timing.py [--repeats 50] [--warmup 5] [--lib path/to/libb200ba.so]
                                      [--cache /tmp/config2.pkl]

``--lib`` times another build of the library (to compare two versions in one session, alternating runs);
``--cache`` keeps the generated problem in a pickle so that such runs generate it once.
"""
import argparse
import json
import os
import pickle
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from camera_calibration_b200 import api, cabi, synthetic  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--lib", default=None)
    ap.add_argument("--cache", default=None)
    args = ap.parse_args()
    if args.lib:
        cabi._LIB = cabi.load_library(os.path.abspath(args.lib))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    if args.cache and os.path.exists(args.cache):
        with open(args.cache, "rb") as f:
            sp = pickle.load(f)
    else:
        sp = synthetic.make_problem(2)
        if args.cache:
            with open(args.cache, "wb") as f:
                pickle.dump(sp, f)
    opt = cabi.default_options()
    with api.BundleAdjuster(sp.problem) as adj:
        adj.set_state(sp.init_state)
        for _ in range(args.warmup):
            adj.evaluate_device(opt, compute_jacobians=True)
        ms = []
        for _ in range(args.repeats):
            t0 = adj.timings()
            cost = adj.evaluate_device(opt, compute_jacobians=True)
            t1 = adj.timings()
            ms.append((t1.jacobian_kernel_ms - t0.jacobian_kernel_ms) /
                      max(1, t1.jacobian_kernel_launches - t0.jacobian_kernel_launches))
    ms = np.array(ms)
    lib = args.lib or "in-tree"
    print(f"card: {card[0] if card else 'unknown'}")
    print(f"residual/Jacobian main pass, config 2 ({sp.n_obs} observations, {lib}): median {np.median(ms):.4f} ms "
          f"(min {ms.min():.4f}, max {ms.max():.4f}, {args.repeats} evaluations); cost {cost:.12g}")
    print(json.dumps({"card": card[0] if card else None, "lib": lib, "n_obs": sp.n_obs,
                      "jacobian_kernel_ms_median": float(np.median(ms)), "jacobian_kernel_ms_min": float(ms.min()),
                      "jacobian_kernel_ms_max": float(ms.max()), "repeats": args.repeats, "cost": cost}))


if __name__ == "__main__":
    main()
