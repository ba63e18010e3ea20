"""Device time of b200ba_report_images (all three images of one camera) and the time of the sequential CPU
restatement of the two Voronoi maps over the same sites, on the config-2 camera and on a 4000 x 3000 camera.

    python scripts/report_images_timing.py [--calls 20]

Prints the card name and power limit of the same run, and the median device time of the calls after one warm-up.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from camera_calibration_b200 import api, synthetic  # noqa: E402
from oracle import voronoi  # noqa: E402
from tests.test_report_images import report_sites  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def measure(label, problem, state, calls):
    with api.BundleAdjuster(problem) as adj:
        adj.set_state(state)
        _, err, _ = adj.calibration_report(True)
        adj.report_images(0)  # warm-up (first call groups the observations)
        ms = [adj.report_images(0)["device_ms"] for _ in range(calls)]
        n_sites = adj.report_images(0)["n_sites"]
    cam = problem.cameras[0]
    sel = np.nonzero(problem.obs_camera == 0)[0]
    sites, dcol, mcol = report_sites(problem.obs_xy[sel], err[sel], cam.width, cam.height)
    t0 = time.perf_counter()
    voronoi.render_voronoi(cam.width, cam.height, sites, dcol)
    voronoi.render_voronoi(cam.width, cam.height, sites, mcol)
    cpu_s = time.perf_counter() - t0
    return {"case": label, "width": cam.width, "height": cam.height, "observations": int(problem.n_obs),
            "sites": n_sites, "device_ms_median": float(np.median(ms)), "cpu_restatement_s": cpu_s}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    a = ap.parse_args()
    voronoi.build()
    print("card:", card())
    sp = synthetic.make_problem(2)
    print(json.dumps(measure("config 2", sp.problem, sp.init_state, a.calls)))
    sp = synthetic.make_problem(2, n_imagesets=60, lattice=(60, 45), image_size=(4000, 3000))
    print(json.dumps(measure("4000 x 3000", sp.problem, sp.init_state, a.calls)))


if __name__ == "__main__":
    main()
