"""Device time of b200ba_calibration_report at full config 2 (955 157 observations, one central-generic
camera), after warm-up, over repeats. Prints the card's name and power limit beside the result, then one
JSON line.

    python scripts/report_timing.py [--repeats 20] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from camera_calibration_b200 import api, synthetic  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    sp = synthetic.make_problem(2)
    with api.BundleAdjuster(sp.problem) as adj:
        adj.set_state(sp.init_state)
        t0 = time.perf_counter()
        adj.calibration_report()  # first call: allocation + upload of the bias-cell ordering
        first_s = time.perf_counter() - t0
        for _ in range(args.warmup):
            adj.calibration_report()
        ms = np.array([adj.calibration_report()[2] for _ in range(args.repeats)])
        t0 = time.perf_counter()
        _, err, _ = adj.calibration_report(with_errors=True)
        with_errors_s = time.perf_counter() - t0
    print(f"card: {card[0] if card else 'unknown'}")
    print(f"b200ba_calibration_report, config 2 ({sp.n_obs} observations): median {np.median(ms):.3f} ms device time "
          f"(min {ms.min():.3f}, max {ms.max():.3f}, {args.repeats} repeats); first call {first_s * 1e3:.1f} ms wall; "
          f"with the error download {with_errors_s * 1e3:.1f} ms wall")
    print(json.dumps({"card": card[0] if card else None, "n_obs": sp.n_obs, "device_ms_median": float(np.median(ms)),
                      "device_ms_min": float(ms.min()), "device_ms_max": float(ms.max()), "repeats": args.repeats,
                      "first_call_wall_ms": first_s * 1e3, "with_errors_wall_ms": with_errors_s * 1e3,
                      "failed_projections": int(np.isnan(err[:, 0]).sum())}))


if __name__ == "__main__":
    main()
